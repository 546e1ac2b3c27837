// tree.cu -- the guide tree on the device (SURVEY.md section 8 f2).
//
// Replaces UPGMA5::FixEADistMx (upgma5.cpp:504-519: distance = 1 - EA) and UPGMA5::Run
// (upgma5.cpp:87-330) as MPCFlat::CalcGuideTree uses them (mpcflat.cpp:183-205, LINKAGE_Biased).
// The reference keeps, per matrix row, the distance to its nearest neighbour and does NOT refresh
// the rows whose nearest neighbour was one of the merged clusters (only the pointer is redirected,
// upgma5.cpp:248-259); ties are broken by scan order.  Both quirks decide which clusters merge, so
// the kernel reproduces the procedure literally: N-1 serial joins, each a few block-wide scans whose
// reductions return the LOWEST index among equal minima (= the reference's strict `<` in ascending
// index order).  One CTA of 1024 threads; the triangular matrix (2 MB at N=1000) stays in L2.
// The arithmetic is two fp32 multiplies, two adds and a halving per updated distance, never fused.
#include "engine.h"
#include <cfloat>
#include <cstring>

#define UP_THREADS 1024
#define UP_NONE 0xffffffffu

struct UpgmaParams
	{
	uint32_t n;
	int linkage;
	const float *ea;             // N(N-1)/2, row-major i<j
	float *dist;                 // triangle, subscript(i,j) = min + max(max-1)/2
	float *mindist; uint32_t *nn; uint32_t *nodeidx; float *height;
	uint32_t *left, *right; float *llen, *rlen;
	int *err;
	};

__device__ __forceinline__ uint32_t tri(uint32_t a, uint32_t b)          // UPGMA5::TriangleSubscript (upgma5.h:63-72)
	{
	return a >= b ? b + (a*(a - 1))/2 : a + (b*(b - 1))/2;
	}

// block-wide (value, index) minimum; equal values -> lower index (the reference's `d < best` scan)
__device__ __forceinline__ void block_argmin(float &v, uint32_t &idx, float *sv, uint32_t *si)
	{
	const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
		{
		const float ov = __shfl_xor_sync(MB_FULL, v, o);
		const uint32_t oi = __shfl_xor_sync(MB_FULL, idx, o);
		if (ov < v || (ov == v && oi < idx))
			{
			v = ov; idx = oi;
			}
		}
	if (lane == 0)
		{
		sv[wid] = v; si[wid] = idx;
		}
	__syncthreads();
	if (wid == 0)
		{
		v = lane < (UP_THREADS/32) ? sv[lane] : FLT_MAX;
		idx = lane < (UP_THREADS/32) ? si[lane] : UP_NONE;
#pragma unroll
		for (int o = 16; o > 0; o >>= 1)
			{
			const float ov = __shfl_xor_sync(MB_FULL, v, o);
			const uint32_t oi = __shfl_xor_sync(MB_FULL, idx, o);
			if (ov < v || (ov == v && oi < idx))
				{
				v = ov; idx = oi;
				}
			}
		if (lane == 0)
			{
			sv[0] = v; si[0] = idx;
			}
		}
	__syncthreads();
	v = sv[0]; idx = si[0];
	__syncthreads();
	}

__global__ void __launch_bounds__(UP_THREADS)
k_upgma(const UpgmaParams P)
	{
	__shared__ float sv[UP_THREADS/32];
	__shared__ uint32_t si[UP_THREADS/32];
	const uint32_t n = P.n;
	const uint32_t tid = threadIdx.x;
	// FixEADistMx + the initial triangle (upgma5.cpp:504-519,131-160); nearest neighbour of a row =
	// lowest index among its minima
	for (uint32_t i = tid; i < n; i += UP_THREADS)
		{
		float best = FLT_MAX;
		uint32_t bi = UP_NONE;
		for (uint32_t m = 0; m < n; ++m)
			{
			if (m == i)
				continue;
			const uint32_t a = min(i, m), b = max(i, m);
			const float e = P.ea[(uint64_t) a*n - (uint64_t) a*(a + 1)/2 + (b - a - 1)];
			if (!(e >= 0.0f && e <= 1.0f))
				*P.err = 1;                                  // the reference asserts 0 <= EA <= 1 (upgma5.cpp:512)
			const float d = __fsub_rn(1.0f, e);
			if (m < i)
				P.dist[tri(i, m)] = d;
			if (d < best)
				{
				best = d; bi = m;
				}
			}
		P.mindist[i] = best;
		P.nn[i] = bi;
		P.nodeidx[i] = i;
		}
	__syncthreads();
	const float c09 = __fsub_rn(1.0f, 0.1f);                     // `(1 - 0.1f)` of upgma5.cpp:240
	for (uint32_t k = 0; k + 1 < n; ++k)
		{
		// nearest pair (upgma5.cpp:176-194)
		float v = FLT_MAX;
		uint32_t lmin = UP_NONE;
		for (uint32_t j = tid; j < n; j += UP_THREADS)
			if (P.nodeidx[j] != UP_NONE)
				{
				const float d = P.mindist[j];
				if (d < v)
					{
					v = d; lmin = j;
					}
				}
		block_argmin(v, lmin, sv, si);
		const uint32_t rmin = P.nn[lmin];
		// distances to the new node, which overwrites the row of Lmin (upgma5.cpp:210-268)
		float nv = FLT_MAX;
		uint32_t nni = UP_NONE;
		for (uint32_t j = tid; j < n; j += UP_THREADS)
			{
			if (j == lmin || j == rmin || P.nodeidx[j] == UP_NONE)
				continue;
			const uint32_t vL = tri(lmin, j), vR = tri(rmin, j);
			const float dL = P.dist[vL], dR = P.dist[vR];
			float nd;
			if (P.linkage == MB200_LINKAGE_AVG)
				nd = __fmul_rn(__fadd_rn(dL, dR), 0.5f);
			else if (P.linkage == MB200_LINKAGE_MIN)
				nd = fminf(dL, dR);
			else if (P.linkage == MB200_LINKAGE_MAX)
				nd = fmaxf(dL, dR);
			else
				nd = __fadd_rn(__fmul_rn(0.1f, __fmul_rn(__fadd_rn(dL, dR), 0.5f)), __fmul_rn(c09, fminf(dL, dR)));
			if (P.nn[j] == rmin)
				P.nn[j] = lmin;
			P.dist[vL] = nd;
			if (nd < nv)
				{
				nv = nd; nni = j;
				}
			}
		block_argmin(nv, nni, sv, si);
		if (tid == 0)
			{
			const float dLR = P.dist[tri(lmin, rmin)];
			const float h = __fmul_rn(dLR, 0.5f);                  // dLR/2
			const uint32_t uL = P.nodeidx[lmin], uR = P.nodeidx[rmin];
			const float hL = uL < n ? 0.0f : P.height[uL - n];
			const float hR = uR < n ? 0.0f : P.height[uR - n];
			P.left[k] = uL; P.right[k] = uR;
			P.llen[k] = __fsub_rn(h, hL); P.rlen[k] = __fsub_rn(h, hR);
			P.height[k] = h;
			P.nodeidx[lmin] = n + k;
			P.nn[lmin] = nni;
			P.mindist[lmin] = nv;
			P.nodeidx[rmin] = UP_NONE;
			}
		__syncthreads();
		}
	}

extern "C" int mb200_guide_tree(mb200_ctx *ctx, const float *ea, int linkage, uint32_t *left, uint32_t *right,
  float *left_len, float *right_len)
	{
	if (!ctx || !left || !right || !left_len || !right_len)
		return mb_fail(ctx, MB200_EINVAL, "mb200_guide_tree: NULL argument");
	if (linkage < MB200_LINKAGE_MIN || linkage > MB200_LINKAGE_BIASED)
		return mb_fail(ctx, MB200_EINVAL, "mb200_guide_tree: unknown linkage %d", linkage);
	const uint32_t n = ctx->nseq;
	if (n < 2)
		return mb_fail(ctx, MB200_EINVAL, "mb200_guide_tree: need >= 2 sequences");
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	const uint64_t np = (uint64_t) n*(n - 1)/2;
	const float *d_ea;
	// scratch: [ea copy][triangle][mindist][nn][nodeidx][height][left][right][llen][rlen][err]
	const size_t need = 2*np*4 + 9*(size_t) n*4 + 256;
	ENSURE(ctx->d_join, need);
	char *p = (char *) ctx->d_join.p;
	float *d_eacopy = (float *) p;          p += np*4;
	UpgmaParams P;
	P.n = n; P.linkage = linkage;
	P.dist = (float *) p;                   p += np*4;
	P.mindist = (float *) p;                p += (size_t) n*4;
	P.nn = (uint32_t *) p;                  p += (size_t) n*4;
	P.nodeidx = (uint32_t *) p;             p += (size_t) n*4;
	P.height = (float *) p;                 p += (size_t) n*4;
	P.left = (uint32_t *) p;                p += (size_t) n*4;
	P.right = (uint32_t *) p;               p += (size_t) n*4;
	P.llen = (float *) p;                   p += (size_t) n*4;
	P.rlen = (float *) p;                   p += (size_t) n*4;
	P.err = (int *) p;
	if (ea != nullptr)
		{
		CU(cudaMemcpyAsync(d_eacopy, ea, np*4, cudaMemcpyHostToDevice, st));
		ctx->stats.h2d_bytes += np*4;
		d_ea = d_eacopy;
		}
	else
		{
		// the EA vector the posterior stage left on this device (store order == all-pairs order)
		const int rc = mb_store_require(ctx, "mb200_guide_tree", NEED_EA);
		if (rc != MB200_OK)
			return rc;
		d_ea = (const float *) ctx->d_ea.p;
		}
	P.ea = d_ea;
	CU(cudaMemsetAsync(P.err, 0, 4, st));
	k_upgma<<<1, UP_THREADS, 0, st>>>(P);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches++;
	CU(cudaMemcpyAsync(left, P.left, (size_t)(n - 1)*4, cudaMemcpyDeviceToHost, st));
	CU(cudaMemcpyAsync(right, P.right, (size_t)(n - 1)*4, cudaMemcpyDeviceToHost, st));
	CU(cudaMemcpyAsync(left_len, P.llen, (size_t)(n - 1)*4, cudaMemcpyDeviceToHost, st));
	CU(cudaMemcpyAsync(right_len, P.rlen, (size_t)(n - 1)*4, cudaMemcpyDeviceToHost, st));
	CU(cudaMemcpyAsync(ctx->h_pinned + 16, P.err, 4, cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));
	ctx->stats.d2h_bytes += 4*(size_t)(n - 1)*4 + 4;
	if (ctx->h_pinned[16] != 0)
		return mb_fail(ctx, MB200_EINVAL, "mb200_guide_tree: an EA value is outside [0,1] (the reference asserts, upgma5.cpp:512)");
	return MB200_OK;
	}
