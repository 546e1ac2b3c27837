// math.cu -- mb200_debug_math: k_posterior_sm's per-score arithmetic on caller-chosen inputs (test hook).
//
// Each op runs the production device code: LogAdd with its table built by mb_logadd_fill and its base read
// back by mb_logadd_make in this kernel's shared memory, exactly as k_posterior_sm sets them up, and the
// mb_post_prob / mb_keep_score decisions of the Backward pass and the compaction.  Operand a is either the
// caller's array or the floats whose bits are a_first_bits, a_first_bits + 1, ... (formed on the device, so
// that a sweep of every float in a range uploads nothing); operand b is an array or one scalar.
#include "engine.h"
#include <algorithm>

static const uint64_t kMathChunk = 1ull << 26;     // floats per launch and per copy back

__global__ void __launch_bounds__(256) k_debug_math(int op, uint32_t n, const float *a, uint32_t a_bits,
  const float *b, float b_scalar, MbHmm h, float *out)
	{
	__shared__ float4 coef[17];
	__shared__ uint32_t labase;
	mb_logadd_fill(coef, &labase);
	__syncthreads();
	const LogAdd la = mb_logadd_make(&labase);
	for (uint32_t k = blockIdx.x*blockDim.x + threadIdx.x; k < n; k += gridDim.x*blockDim.x)
		{
		const float x = a ? a[k] : __uint_as_float(a_bits + k);
		const float y = b ? b[k] : b_scalar;
		float r;
		switch (op)
			{
			case MB200_MATH_LOG_ADD:    r = la(x, y); break;
			case MB200_MATH_LOG_ADD_BA: r = la(y, x); break;
			case MB200_MATH_POST_PROB:  r = x < h.minScore ? 0.0f : mb_post_prob(x); break;
			default:                    r = x >= mb_keep_score(h) ? 1.0f : 0.0f; break;
			}
		out[k] = r;
		}
	}

extern "C" int mb200_debug_math(mb200_ctx *ctx, int op, uint64_t n, const float *a, uint32_t a_first_bits,
  const float *b, float b_scalar, float *out)
	{
	if (!ctx)
		return MB200_EINVAL;
	if (op < MB200_MATH_LOG_ADD || op > MB200_MATH_KEEP || (n > 0 && !out))
		return mb_fail(ctx, MB200_EINVAL, "mb200_debug_math: bad op %d or NULL out", op);
	if ((op == MB200_MATH_POST_PROB || op == MB200_MATH_KEEP) && !ctx->have_hmm)
		return mb_fail(ctx, MB200_EINVAL, "mb200_debug_math: op %d needs mb200_set_hmm first", op);
	if (n == 0)
		return MB200_OK;
	cudaSetDevice(ctx->device);
	const uint64_t chunk = std::min<uint64_t>(n, kMathChunk);
	ENSURE(ctx->d_math, 3*chunk*sizeof(float));
	float *d_out = (float *) ctx->d_math.p, *d_a = d_out + chunk, *d_b = d_a + chunk;
	for (uint64_t k0 = 0; k0 < n; k0 += chunk)
		{
		const uint32_t m = (uint32_t) std::min<uint64_t>(chunk, n - k0);
		if (a)
			CU(cudaMemcpyAsync(d_a, a + k0, m*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
		if (b)
			CU(cudaMemcpyAsync(d_b, b + k0, m*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
		const uint32_t blocks = std::min<uint32_t>((m + 255)/256, 8u*(uint32_t) ctx->prop.multiProcessorCount);
		k_debug_math<<<blocks, 256, 0, ctx->stream>>>(op, m, a ? d_a : nullptr, a_first_bits + (uint32_t) k0,
		  b ? d_b : nullptr, b_scalar, ctx->hmm, d_out);
		CU(cudaGetLastError());
		CU(cudaMemcpyAsync(out + k0, d_out, m*sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
		CU(cudaStreamSynchronize(ctx->stream));
		}
	return MB200_OK;
	}
