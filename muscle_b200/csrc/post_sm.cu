// post_sm.cu -- launch surface of k_posterior_sm (post_kernel_sm.cuh)
#include "post_kernel_sm.cuh"
#include "launch.h"

template <bool MEGA, int CM, bool DUMP>
static void dispatch(int op, dim3 grid, size_t smem, cudaStream_t st, const PostParams *P, int *out)
	{
	if (op == 0)
		{
		cudaFuncSetAttribute(k_posterior_sm<MEGA, CM, DUMP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
		k_posterior_sm<MEGA, CM, DUMP><<<grid, 32*MB_WARPS_PER_BLOCK, smem, st>>>(*P);
		}
	else if (op == 1)
		{
		cudaFuncSetAttribute(k_posterior_sm<MEGA, CM, DUMP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
		cudaOccupancyMaxActiveBlocksPerMultiprocessor(out, k_posterior_sm<MEGA, CM, DUMP>, 32*MB_WARPS_PER_BLOCK, smem);
		}
	else
		*out = (int) sizeof(PostSmemHdr);
	}

template <bool MEGA, bool DUMP>
static bool dispatch_cm(int cm, int op, dim3 grid, size_t smem, cudaStream_t st, const PostParams *P, int *out)
	{
	switch (cm)
		{
		case 4:  dispatch<MEGA, 4, DUMP>(op, grid, smem, st, P, out); return true;
		case 8:  dispatch<MEGA, 8, DUMP>(op, grid, smem, st, P, out); return true;
		case 12: dispatch<MEGA, 12, DUMP>(op, grid, smem, st, P, out); return true;
		case 14: dispatch<MEGA, 14, DUMP>(op, grid, smem, st, P, out); return true;
		case 16: dispatch<MEGA, 16, DUMP>(op, grid, smem, st, P, out); return true;
		default: return false;
		}
	}

bool mb_post_sm_dispatch(bool mega, bool dump, int cm, int op, dim3 grid, size_t smem, cudaStream_t st,
  const PostParams *P, int *out)
	{
	if (mega)
		return dump ? dispatch_cm<true, true>(cm, op, grid, smem, st, P, out)
		            : dispatch_cm<true, false>(cm, op, grid, smem, st, P, out);
	return dump ? dispatch_cm<false, true>(cm, op, grid, smem, st, P, out)
	            : dispatch_cm<false, false>(cm, op, grid, smem, st, P, out);
	}
