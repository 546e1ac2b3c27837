// relax.cu -- the consistency transform (one Jacobi iteration) on the device-resident store.
//
// Replaces MPCFlat::ConsIter (consflat.cpp:5-23) / MPCFlat::ConsPair (conspairflat.cpp:10-110) with
// RelaxFlat_ZX_ZY, RelaxFlat_XZ_ZY, RelaxFlat_XZ_YZ (relaxflat.cpp:4-94) and
// MySparseMx::UpdateFromPost (mysparsemx.cpp:87-113).
//
// Formulation.  The reference scatters P_XZ[i,k]*P_ZY[k,j] into a dense LX*LY scratch and then
// keeps only XY's own pattern.  Here every stored entry (i,j) of XY is owned by one thread that
// GATHERS its own sum: with both orientations of every pair in HBM, row i of S[x->z] and row j of
// S[y->z] are two short column-sorted lists and the contribution of z is their sparse dot product.
// For a fixed entry the reference adds the products in ascending z and, inside one z, in ascending
// k for all three of its loop nests; here z runs ascending, matches are visited k ascending, every
// product is one __fmul_rn and every accumulation one __fadd_rn, so the result is bit-identical
// (verified against the oracle and the compiled reference).
//
// Finding the matching k (round 2).  On real and synthetic posteriors a sparse row holds
// ~7 entries scattered over a span of ~55 columns (92 % of the rows are not contiguous), and a pair
// of rows (A_i, B_j) shares only ~0.7 columns per (entry, z): the round-1 kernel spent ~15 merge
// steps and ~30 gathered loads per (entry, z) to find them and was bound by L1 gather wavefronts.
// The pattern of the
// store never changes during consistency (mysparsemx.cpp:87-113), so the columns of every row, in
// both orientations, are encoded ONCE as bit masks over 32-column words
//      hdr[row]  = { slot of the row's first word, w0 | nw << 16 }      (w0 = first column / 32)
//      word[s]   = { mask of columns 32(w0+t)..+31, index of the first entry of that word }
// and a dot product becomes: intersect the two word ranges (1.6 words on average), AND the masks,
// and for every surviving bit (ascending = k ascending) fetch the two values by popcount.  That is
// ~6 loads and ~40 instructions per (entry, z) instead of ~30 and ~240.
//
// Relax is a sparse-sparse contraction (2 % density, scattered): tensor cores do not apply
// (DESIGN.md "relax is not a GEMM").
#include "engine.h"
#include <cub/cub.cuh>
#include <thrust/iterator/transform_iterator.h>
#include <algorithm>
#include <cstdlib>
#include <cstring>

// ---------------------------------------------------------------------------------------------
// column bit masks of one orientation.  Rows are addressed like the CSR offsets: slot
// rowbase[k] + i for row i of store pair k (the slot of the sentinel offset holds an empty row).
// One warp per pair, one lane per row.
__global__ void k_mask_count(uint32_t npairs, const uint64_t *__restrict__ rowbase, const uint32_t *__restrict__ rowoff,
  const uint64_t *__restrict__ entbase, const mb200_entry *__restrict__ entries, uint32_t *__restrict__ nw_out)
	{
	const uint32_t warp = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t nwarps = (gridDim.x*blockDim.x) >> 5;
	for (uint32_t k = warp; k < npairs; k += nwarps)
		{
		const uint64_t rb = rowbase[k];
		const uint32_t nrow = (uint32_t)(rowbase[k + 1] - rb) - 1;
		const uint32_t *ro = rowoff + rb;
		const mb200_entry *en = entries + entbase[k];
		for (uint32_t i = lane; i <= nrow; i += 32)
			{
			uint32_t nw = 0;
			if (i < nrow)
				{
				const uint32_t a = ro[i], b = ro[i + 1];
				if (b > a)
					nw = (en[b - 1].col >> 5) - (en[a].col >> 5) + 1;
				}
			nw_out[rb + i] = nw;
			}
		}
	}

__global__ void k_mask_fill(uint32_t npairs, const uint64_t *__restrict__ rowbase, const uint32_t *__restrict__ rowoff,
  const uint64_t *__restrict__ entbase, const mb200_entry *__restrict__ entries, const uint32_t *__restrict__ nw_in,
  const uint64_t *__restrict__ wslot, uint2 *__restrict__ hdr, uint2 *__restrict__ words)
	{
	const uint32_t warp = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t nwarps = (gridDim.x*blockDim.x) >> 5;
	for (uint32_t k = warp; k < npairs; k += nwarps)
		{
		const uint64_t rb = rowbase[k];
		const uint32_t nrow = (uint32_t)(rowbase[k + 1] - rb) - 1;
		const uint32_t *ro = rowoff + rb;
		const mb200_entry *en = entries + entbase[k];
		for (uint32_t i = lane; i <= nrow; i += 32)
			{
			const uint32_t nw = nw_in[rb + i];
			const uint32_t slot = (uint32_t) wslot[rb + i];
			uint32_t w0 = 0;
			if (nw > 0)
				{
				const uint32_t a = ro[i], b = ro[i + 1];
				w0 = en[a].col >> 5;
				uint32_t cur = w0, mask = 0, first = a;
				for (uint32_t e = a; e < b; ++e)
					{
					const uint32_t c = en[e].col;
					const uint32_t w = c >> 5;
					if (w != cur)
						{
						words[slot + (cur - w0)] = make_uint2(mask, first);
						for (uint32_t t = cur + 1; t < w; ++t)
							words[slot + (t - w0)] = make_uint2(0u, e);
						cur = w; mask = 0; first = e;
						}
					mask |= 1u << (c & 31);
					}
				words[slot + (cur - w0)] = make_uint2(mask, first);
				}
			hdr[rb + i] = make_uint2(slot, w0 | (nw << 16));
			}
		}
	}

struct WidenU32
	{
	__host__ __device__ uint64_t operator()(uint32_t v) const { return v; }
	};

static int build_masks_one(mb200_ctx *ctx, uint32_t np, uint64_t nslots, const uint64_t *rowbase, const uint32_t *rowoff,
  const mb200_entry *entries, DevBuf &d_hdr, DevBuf &d_words)
	{
	cudaStream_t st = ctx->stream;
	const int blocks = ctx->prop.multiProcessorCount*8;
	// d_tmp: nw per slot (u32); d_tmp2: exclusive scan (u64 per slot) followed by the cub scratch
	ENSURE(ctx->d_tmp, nslots*sizeof(uint32_t) + 64);
	uint32_t *d_nw = (uint32_t *) ctx->d_tmp.p;
	// 64-bit running sum of the 32-bit counts
	auto in64 = thrust::make_transform_iterator((const uint32_t *) d_nw, WidenU32());
	size_t tb = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, tb, in64, (uint64_t *) nullptr, (int64_t) nslots, st);
	const size_t scan_bytes = (nslots*sizeof(uint64_t) + 255)/256*256;
	ENSURE(ctx->d_tmp2, scan_bytes + tb + 64);
	uint64_t *d_slot = (uint64_t *) ctx->d_tmp2.p;
	void *d_scratch = (char *) ctx->d_tmp2.p + scan_bytes;
	k_mask_count<<<blocks, 256, 0, st>>>(np, rowbase, rowoff, (const uint64_t *) ctx->d_entbase.p, entries, d_nw);
	CU(cudaGetLastError());
	cub::DeviceScan::ExclusiveSum(d_scratch, tb, in64, d_slot, (int64_t) nslots, st);
	CU(cudaGetLastError());
	uint64_t last_slot = 0;
	uint32_t last_nw = 0;
	CU(cudaMemcpyAsync(&last_slot, d_slot + (nslots - 1), sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
	CU(cudaMemcpyAsync(&last_nw, d_nw + (nslots - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));
	const uint64_t nwords = last_slot + last_nw;
	if (nwords >= 0xffffffffull)
		return mb_fail(ctx, MB200_EOVERFLOW, "column masks need %llu words (32-bit slots)", (unsigned long long) nwords);
	ENSURE(d_hdr, nslots*sizeof(uint2));
	ENSURE(d_words, (nwords + 8)*sizeof(uint2));
	k_mask_fill<<<blocks, 256, 0, st>>>(np, rowbase, rowoff, (const uint64_t *) ctx->d_entbase.p, entries, d_nw, d_slot,
	  (uint2 *) d_hdr.p, (uint2 *) d_words.p);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches += 3;
	return MB200_OK;
	}

// the column masks of both orientations of a transposed store (mb_store_require)
int mb_build_masks(mb200_ctx *ctx)
	{
	const uint32_t np = (uint32_t) ctx->h_px.size();
	int rc = build_masks_one(ctx, np, ctx->h_rowbase.back(), (const uint64_t *) ctx->d_rowbase.p, (const uint32_t *) ctx->d_rowoff.p,
	  (const mb200_entry *) ctx->d_entries.p, ctx->d_mk_hdr, ctx->d_mk_words);
	if (rc != MB200_OK)
		return rc;
	rc = build_masks_one(ctx, np, ctx->h_tr_rowbase.back(), (const uint64_t *) ctx->d_tr_rowbase.p,
	  (const uint32_t *) ctx->d_tr_rowoff.p, (const mb200_entry *) ctx->d_tr_entries.p, ctx->d_tr_mk_hdr, ctx->d_tr_mk_words);
	if (rc != MB200_OK)
		return rc;
	CU(cudaStreamSynchronize(ctx->stream));
	return MB200_OK;
	}

// ---------------------------------------------------------------------------------------------
struct RelaxParams
	{
	uint32_t n;                       // sequences
	uint32_t nwork;                   // pairs to update
	const uint32_t *order;            // work list: all-pairs indexes in 2-D tile order
	const uint32_t *seqlen;
	const uint64_t *rowbase;  const uint32_t *rowoff;  const mb200_entry *entries;      // forward
	const uint64_t *trbase;   const mb200_entry *trentries;                             // transposed
	const uint2 *hdr, *words, *trhdr, *trwords;                                         // column masks
	const uint64_t *entbase;
	mb200_entry *out;                 // new values (same layout as entries)
	};

// operands of one z: S[x->z] (rows = positions of x) and S[y->z] (rows = positions of y)
struct ZDesc
	{
	const uint2 *hdrA, *wordsA; const mb200_entry *enA;
	const uint2 *hdrB, *wordsB; const mb200_entry *enB;
	};

#define RELAX_THREADS 256
#define RELAX_ZCHUNK 64
#ifndef RELAX_EPT
#define RELAX_EPT 4          // entries per thread held in registers per sweep
#endif

// MINB: resident CTAs/SM the register allocation is bounded for (sm_90a: 2: 96 registers, no spill;
// 3: 80, no spill; 4: 64, 56 bytes spilled).  The kernel is bound by gather latency, so occupancy
// wins over spills; 4 is the default (MB200_RELAX_OCC selects another).
template <int MINB>
__global__ void __launch_bounds__(RELAX_THREADS, MINB)
k_relax(const RelaxParams P)
	{
	__shared__ ZDesc zd[RELAX_ZCHUNK];
	if (blockIdx.x >= P.nwork)
		return;
	const uint32_t p = P.order[blockIdx.x];
	// invert p -> (x,y): find x with base(x) <= p < base(x+1)
	const uint32_t n = P.n;
	uint32_t x = 0;
		{
		// base(x) = x*n - x(x+1)/2 ; solve by a short search from the analytic estimate
		const double nn = (double) n - 0.5;
		double est = nn - sqrt(fmax(0.0, nn*nn - 2.0*(double) p));
		x = (uint32_t) fmin(fmax(est, 0.0), (double)(n - 2));
		while (x > 0 && (uint64_t) x*n - (uint64_t) x*(x + 1)/2 > p)
			--x;
		while (x + 1 < n - 1 && (uint64_t)(x + 1)*n - (uint64_t)(x + 1)*(x + 2)/2 <= p)
			++x;
		}
	const uint32_t y = x + 1 + (p - (uint32_t)((uint64_t) x*n - (uint64_t) x*(x + 1)/2));
	const uint32_t LX = P.seqlen[x];
	const uint32_t *ro = P.rowoff + P.rowbase[p];
	const uint64_t eb = P.entbase[p];
	const mb200_entry *en = P.entries + eb;
	mb200_entry *out = P.out + eb;
	const uint32_t nnz = ro[LX];
	const float fn = (float) n;

	for (uint32_t e0 = 0; e0 < nnz; e0 += RELAX_THREADS*RELAX_EPT)
		{
		// this thread's entries of the sweep: (row i, col j, accumulator)
		uint32_t ei[RELAX_EPT], ej[RELAX_EPT];
		float acc[RELAX_EPT];
		bool live[RELAX_EPT];
#pragma unroll
		for (int q = 0; q < RELAX_EPT; ++q)
			{
			const uint32_t e = e0 + q*RELAX_THREADS + threadIdx.x;
			live[q] = e < nnz;
			ei[q] = 0; ej[q] = 0; acc[q] = 0.0f;
			if (live[q])
				{
				const mb200_entry v = en[e];
				ej[q] = v.col;
				acc[q] = __fmul_rn(v.p, 2.0f);          // Z=X and Z=Y (conspairflat.cpp:26-30)
				// row of entry e: largest i with ro[i] <= e (binary search over LX+1 offsets)
				uint32_t lo = 0, hi = LX;
				while (hi - lo > 1)
					{
					const uint32_t mid = (lo + hi) >> 1;
					if (ro[mid] <= e) lo = mid; else hi = mid;
					}
				ei[q] = lo;
				}
			}
		for (uint32_t z0 = 0; z0 < n; z0 += RELAX_ZCHUNK)
			{
			__syncthreads();
			if (threadIdx.x < RELAX_ZCHUNK)
				{
				const uint32_t z = z0 + threadIdx.x;
				ZDesc d;
				d.hdrA = nullptr;
				if (z < n && z != x && z != y)
					{
					// S[x->z]: rows are positions of x
					if (x < z)
						{
						const uint32_t q = mb_pair_index(n, x, z);
						d.hdrA = P.hdr + P.rowbase[q]; d.wordsA = P.words; d.enA = P.entries + P.entbase[q];
						}
					else
						{
						const uint32_t q = mb_pair_index(n, z, x);
						d.hdrA = P.trhdr + P.trbase[q]; d.wordsA = P.trwords; d.enA = P.trentries + P.entbase[q];
						}
					// S[y->z]: rows are positions of y
					if (y < z)
						{
						const uint32_t q = mb_pair_index(n, y, z);
						d.hdrB = P.hdr + P.rowbase[q]; d.wordsB = P.words; d.enB = P.entries + P.entbase[q];
						}
					else
						{
						const uint32_t q = mb_pair_index(n, z, y);
						d.hdrB = P.trhdr + P.trbase[q]; d.wordsB = P.trwords; d.enB = P.trentries + P.entbase[q];
						}
					}
				zd[threadIdx.x] = d;
				}
			__syncthreads();
			const uint32_t zn = min((uint32_t) RELAX_ZCHUNK, n - z0);
			for (uint32_t zz = 0; zz < zn; ++zz)
				{
				const ZDesc d = zd[zz];
				if (d.hdrA == nullptr)
					continue;
				// The entries of a thread are independent chains, each three dependent gathers deep
				// (header -> mask word -> value).  The loads of one level are issued for ALL entries
				// before any is consumed, so RELAX_EPT x 2 loads are in flight per thread instead of one
				// (round-2 profile of the first version: 20.7 long-scoreboard stall cycles per issue).
				uint32_t slotA[RELAX_EPT], slotB[RELAX_EPT], lo[RELAX_EPT], hi[RELAX_EPT];
#pragma unroll
				for (int q = 0; q < RELAX_EPT; ++q)
					{
					uint2 hA = make_uint2(0u, 0u), hB = make_uint2(0u, 0u);
					if (live[q])
						{
						hA = d.hdrA[ei[q]];
						hB = d.hdrB[ej[q]];
						}
					const uint32_t w0A = hA.y & 0xffffu, w0B = hB.y & 0xffffu;
					lo[q] = max(w0A, w0B);
					hi[q] = min(w0A + (hA.y >> 16), w0B + (hB.y >> 16));
					slotA[q] = hA.x - w0A;                       // word w of the row lives at slot + w (mod 2^32)
					slotB[q] = hB.x - w0B;
					}
				uint2 a[RELAX_EPT], b[RELAX_EPT];
#pragma unroll
				for (int q = 0; q < RELAX_EPT; ++q)
					{
					a[q] = make_uint2(0u, 0u); b[q] = make_uint2(0u, 0u);
					if (lo[q] < hi[q])
						{
						a[q] = d.wordsA[slotA[q] + lo[q]];
						b[q] = d.wordsB[slotB[q] + lo[q]];
						}
					}
				float pa[RELAX_EPT], pb[RELAX_EPT];
				uint32_t m[RELAX_EPT];
#pragma unroll
				for (int q = 0; q < RELAX_EPT; ++q)
					{
					m[q] = a[q].x & b[q].x;
					pa[q] = 0.0f; pb[q] = 0.0f;
					if (m[q])
						{
						const uint32_t below = (m[q] & (0u - m[q])) - 1u;       // bits under the lowest common column
						pa[q] = d.enA[a[q].y + __popc(a[q].x & below)].p;
						pb[q] = d.enB[b[q].y + __popc(b[q].x & below)].p;
						}
					}
#pragma unroll
				for (int q = 0; q < RELAX_EPT; ++q)
					{
					float s = acc[q];
					if (m[q])
						{
						s = __fadd_rn(s, __fmul_rn(pa[q], pb[q]));                 // relaxflat.cpp:27,56,90
						uint32_t mm = m[q] & (m[q] - 1u);
						while (mm)                                                   // further common columns of the word (k ascending)
							{
							const uint32_t below = (mm & (0u - mm)) - 1u;
							const float xa = d.enA[a[q].y + __popc(a[q].x & below)].p;
							const float xb = d.enB[b[q].y + __popc(b[q].x & below)].p;
							s = __fadd_rn(s, __fmul_rn(xa, xb));
							mm &= mm - 1u;
							}
						}
					for (uint32_t w = lo[q] + 1; w < hi[q]; ++w)                   // further overlapping words (0.6 on average)
						{
						const uint2 a2 = d.wordsA[slotA[q] + w];
						const uint2 b2 = d.wordsB[slotB[q] + w];
						uint32_t mm = a2.x & b2.x;
						while (mm)
							{
							const uint32_t below = (mm & (0u - mm)) - 1u;
							const float xa = d.enA[a2.y + __popc(a2.x & below)].p;
							const float xb = d.enB[b2.y + __popc(b2.x & below)].p;
							s = __fadd_rn(s, __fmul_rn(xa, xb));
							mm &= mm - 1u;
							}
						}
					acc[q] = s;
					}
				}
			}
#pragma unroll
		for (int q = 0; q < RELAX_EPT; ++q)
			{
			if (live[q])
				{
				const uint32_t e = e0 + q*RELAX_THREADS + threadIdx.x;
				mb200_entry v;
				v.col = ej[q];
				v.p = __fdiv_rn(acc[q], fn);                    // mysparsemx.cpp:108
				out[e] = v;
				}
			}
		}
	}

// copy entries of pairs outside [p_lo,p_hi) unchanged into the new buffer
__global__ void k_copy_entries(uint64_t lo, uint64_t hi, const mb200_entry *__restrict__ src, mb200_entry *__restrict__ dst)
	{
	for (uint64_t k = lo + blockIdx.x*(uint64_t) blockDim.x + threadIdx.x; k < hi; k += (uint64_t) gridDim.x*blockDim.x)
		dst[k] = src[k];
	}

// Work order of the pairs of [p_lo,p_hi): 2-D tiles of the (x,y) triangle.  Every CTA streams
// S[x->z] and S[y->z] over all z; CTAs that are resident together start at z=0 and advance at about
// the same pace, so when they cover a compact tile of T x T pairs the 2T operand sequences of the
// current z are read from HBM once and then hit in the 50 MB L2 (row-major order would share x only).
#define RELAX_TILE 16
static int prepare_relax_order(mb200_ctx *ctx, uint32_t p_lo, uint32_t p_hi)
	{
	const uint32_t n = ctx->nseq;
	static uint32_t tile = 0;
	if (tile == 0)
		{
		const char *ev = getenv("MB200_RELAX_TILE");           // tuning hook
		tile = ev ? (uint32_t) std::max(1, atoi(ev)) : RELAX_TILE;
		}
	if (ctx->relax_order_n == n && ctx->relax_order_lo == p_lo && ctx->relax_order_hi == p_hi && ctx->d_relax_order.p)
		return MB200_OK;
	std::vector<uint32_t> order;
	order.reserve(p_hi - p_lo);
	const uint32_t T = tile;
	for (uint32_t tx = 0; tx < n; tx += T)
		for (uint32_t ty = tx; ty < n; ty += T)
			for (uint32_t x = tx; x < std::min(n, tx + T); ++x)
				for (uint32_t y = std::max(ty, x + 1); y < std::min(n, ty + T); ++y)
					{
					const uint32_t p = mb_pair_index(n, x, y);
					if (p >= p_lo && p < p_hi)
						order.push_back(p);
					}
	if (order.size() != (size_t)(p_hi - p_lo))
		return mb_fail(ctx, MB200_EINVAL, "relax work order covers %zu of %u pairs", order.size(), p_hi - p_lo);
	ENSURE(ctx->d_relax_order, order.size()*sizeof(uint32_t));
	CU(cudaMemcpyAsync(ctx->d_relax_order.p, order.data(), order.size()*sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
	CU(cudaStreamSynchronize(ctx->stream));
	ctx->stats.h2d_bytes += order.size()*sizeof(uint32_t);
	ctx->relax_order_n = n; ctx->relax_order_lo = p_lo; ctx->relax_order_hi = p_hi;
	return MB200_OK;
	}

extern "C" {

int mb200_consistency_iter(mb200_ctx *ctx, uint32_t p_lo, uint32_t p_hi)
	{
	if (!ctx)
		return MB200_EINVAL;
	int rc = mb_store_require(ctx, "mb200_consistency_iter", NEED_ALLPAIRS);
	if (rc != MB200_OK)
		return rc;
	const uint32_t n = ctx->nseq;
	const uint32_t np = (uint32_t) ctx->h_px.size();
	if (p_lo > p_hi || p_hi > np)
		return mb_fail(ctx, MB200_EINVAL, "pair range [%u,%u) invalid", p_lo, p_hi);
	if (n < 3)
		return MB200_OK;                       // MPCFlat::Consistency skips N<3 (mpcflat.cpp:176)
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	CU(cudaEventRecord(ctx->ev0, st));
	rc = mb_store_require(ctx, "mb200_consistency_iter", NEED_ALLPAIRS | FORM_MASKED);
	if (rc != MB200_OK)
		return rc;
	ENSURE(ctx->d_entries2, (ctx->store_nnz + 64)*sizeof(mb200_entry));
	CU(cudaEventRecord(ctx->ev1, st));
	if (p_hi > p_lo)
		{
		rc = prepare_relax_order(ctx, p_lo, p_hi);
		if (rc != MB200_OK)
			return rc;
		RelaxParams P;
		P.n = n; P.nwork = p_hi - p_lo;
		P.order = (const uint32_t *) ctx->d_relax_order.p;
		P.seqlen = (const uint32_t *) ctx->d_seqlen.p;
		P.rowbase = (const uint64_t *) ctx->d_rowbase.p;
		P.rowoff = (const uint32_t *) ctx->d_rowoff.p;
		P.entries = (const mb200_entry *) ctx->d_entries.p;
		P.trbase = (const uint64_t *) ctx->d_tr_rowbase.p;
		P.trentries = (const mb200_entry *) ctx->d_tr_entries.p;
		P.hdr = (const uint2 *) ctx->d_mk_hdr.p; P.words = (const uint2 *) ctx->d_mk_words.p;
		P.trhdr = (const uint2 *) ctx->d_tr_mk_hdr.p; P.trwords = (const uint2 *) ctx->d_tr_mk_words.p;
		P.entbase = (const uint64_t *) ctx->d_entbase.p;
		P.out = (mb200_entry *) ctx->d_entries2.p;
		CU(cudaEventRecord(ctx->ev1, st));
		static int occ = 0;
		if (occ == 0)
			{
			const char *ev = getenv("MB200_RELAX_OCC");        // tuning hooks
			occ = ev ? atoi(ev) : 4;
			}
		if (occ == 2)
			k_relax<2><<<p_hi - p_lo, RELAX_THREADS, 0, st>>>(P);
		else if (occ == 4)
			k_relax<4><<<p_hi - p_lo, RELAX_THREADS, 0, st>>>(P);
		else
			k_relax<3><<<p_hi - p_lo, RELAX_THREADS, 0, st>>>(P);
		CU(cudaGetLastError());
		ctx->stats.kernel_launches++;
		}
	CU(cudaEventRecord(ctx->ev2, st));
	// pairs outside the range keep their old values until the peers' results arrive
	uint64_t e_lo = 0, e_hi = 0;
	mb_store_entry_range(ctx, p_lo, p_hi, &e_lo, &e_hi);
	const int blocks = ctx->prop.multiProcessorCount*8;
	if (e_lo > 0)
		{
		k_copy_entries<<<blocks, 256, 0, st>>>(0, e_lo, (const mb200_entry *) ctx->d_entries.p, (mb200_entry *) ctx->d_entries2.p);
		ctx->stats.kernel_launches++;
		}
	if (e_hi < ctx->store_nnz)
		{
		k_copy_entries<<<blocks, 256, 0, st>>>(e_hi, ctx->store_nnz, (const mb200_entry *) ctx->d_entries.p, (mb200_entry *) ctx->d_entries2.p);
		ctx->stats.kernel_launches++;
		}
	CU(cudaGetLastError());
	CU(cudaEventRecord(ctx->ev3, st));
	CU(cudaStreamSynchronize(st));
	std::swap(ctx->d_entries, ctx->d_entries2);            // consflat.cpp:22
	mb_store_values_written(ctx);
	cudaEventElapsedTime(&ctx->stats.last_kernel_ms, ctx->ev1, ctx->ev2);
	cudaEventElapsedTime(&ctx->stats.last_total_ms, ctx->ev0, ctx->ev3);
	return MB200_OK;
	}

} // extern "C"
