// store.cu -- the device-resident sparse posterior store: its state (StoreState, engine.h), packing in
// pair order (export and the multi-GPU exchange image), loading a gathered image, values-only views,
// and the transposed orientation that the consistency kernel and the joins need, with the view of both
// orientations those kernels read (StoreView, common.cuh).
//
// Reference counterparts: the store replaces MPCFlat::m_SparsePosts1/2 (mpcflat.h:46-49); the wire
// format of one pair is MySparseMx's (mysparsemx.h:6-98).  The transposed orientation replaces the
// reference's three index-order variants of RelaxFlat (relaxflat.cpp:4,33,62) and the linear
// GetProb/GetColToRowLoHi scans (mysparsemx.cpp:44-62,238-268).
#include "engine.h"
#include <cub/cub.cuh>
#include <algorithm>
#include <cstring>
#include <numeric>

// ---------------------------------------------------------------------------------------------
// one warp per pair: copy the pair's entries to their packed position
__global__ void k_pack_entries(uint32_t npairs, const uint64_t *__restrict__ src_base,
  const uint64_t *__restrict__ dst_base, const uint32_t *__restrict__ nnz,
  const mb200_entry *__restrict__ src, mb200_entry *__restrict__ dst)
	{
	const uint32_t warp = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t nw = (gridDim.x*blockDim.x) >> 5;
	for (uint32_t k = warp; k < npairs; k += nw)
		{
		const mb200_entry *s = src + src_base[k];
		mb200_entry *d = dst + dst_base[k];
		const uint32_t n = nnz[k];
		for (uint32_t e = lane; e < n; e += 32)
			d[e] = s[e];
		}
	}

// nnz[k] = rowoff[rowbase[k] + LX_k]  (= rowoff[rowbase[k+1]-1])
__global__ void k_nnz_from_rowoff(uint32_t npairs, const uint64_t *__restrict__ rowbase,
  const uint32_t *__restrict__ rowoff, uint32_t *__restrict__ nnz, uint64_t *__restrict__ nnz64)
	{
	const uint32_t k = blockIdx.x*blockDim.x + threadIdx.x;
	if (k < npairs)
		{
		const uint32_t n = rowoff[rowbase[k + 1] - 1];
		nnz[k] = n;
		nnz64[k] = n;
		}
	}

__global__ void k_gather_values(uint64_t n, const mb200_entry *__restrict__ e, float *__restrict__ v)
	{
	for (uint64_t k = blockIdx.x*(uint64_t) blockDim.x + threadIdx.x; k < n; k += (uint64_t) gridDim.x*blockDim.x)
		v[k] = e[k].p;
	}

__global__ void k_scatter_values(uint64_t n, const float *__restrict__ v, mb200_entry *__restrict__ e)
	{
	for (uint64_t k = blockIdx.x*(uint64_t) blockDim.x + threadIdx.x; k < n; k += (uint64_t) gridDim.x*blockDim.x)
		e[k].p = v[k];
	}

// ---------------------------------------------------------------------------------------------
// Transposed orientation.  One warp per pair.
//  pass A: column histogram -> tr_rowoff (exclusive scan over LY+1 slots, done by the warp)
//  pass B: rows ascending, each entry goes to cursor[col]++ ; columns inside one row are distinct
//          and rows are visited in order, so every transposed row ends up sorted by original row.
// perm[t] = index (relative to the pair's entry base) of the forward entry stored at transposed t.
__global__ void k_transpose_pairs(uint32_t npairs, const uint32_t *__restrict__ px, const uint32_t *__restrict__ py,
  const uint32_t *__restrict__ seqlen, const uint64_t *__restrict__ rowbase, const uint32_t *__restrict__ rowoff,
  const uint64_t *__restrict__ entbase, const mb200_entry *__restrict__ entries,
  const uint64_t *__restrict__ tr_rowbase, uint32_t *__restrict__ tr_rowoff,
  mb200_entry *__restrict__ tr_entries, uint32_t *__restrict__ tr_perm)
	{
	const uint32_t warp = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t nw = (gridDim.x*blockDim.x) >> 5;
	for (uint32_t k = warp; k < npairs; k += nw)
		{
		const uint32_t LX = seqlen[px[k]], LY = seqlen[py[k]];
		const uint32_t *ro = rowoff + rowbase[k];
		const mb200_entry *en = entries + entbase[k];
		uint32_t *tro = tr_rowoff + tr_rowbase[k];
		mb200_entry *ten = tr_entries + entbase[k];
		uint32_t *perm = tr_perm + entbase[k];
		const uint32_t n = ro[LX];
		for (uint32_t c = lane; c <= LY; c += 32)
			tro[c] = 0;
		__syncwarp();
		for (uint32_t e = lane; e < n; e += 32)
			atomicAdd(&tro[en[e].col + 1], 1u);
		__syncwarp();
		// inclusive scan of tro[1..LY] in chunks of 32
		uint32_t carry = 0;
		for (uint32_t c0 = 1; c0 <= LY; c0 += 32)
			{
			const uint32_t c = c0 + lane;
			uint32_t v = c <= LY ? tro[c] : 0;
#pragma unroll
			for (int o = 1; o < 32; o <<= 1)
				{
				const uint32_t t = __shfl_up_sync(MB_FULL, v, o);
				if (lane >= (uint32_t) o)
					v += t;
				}
			v += carry;
			if (c <= LY)
				tro[c] = v;
			carry = __shfl_sync(MB_FULL, v, 31);
			}
		__syncwarp();
		// placement; tro[c] is used as the running cursor of column c and restored afterwards
		for (uint32_t i = 0; i < LX; ++i)
			{
			const uint32_t b = ro[i], eend = ro[i + 1];
			for (uint32_t e = b + lane; e < eend; e += 32)
				{
				const mb200_entry v = en[e];
				const uint32_t dst = tro[v.col]++;
				mb200_entry t; t.p = v.p; t.col = i;
				ten[dst] = t;
				perm[dst] = e;
				}
			__syncwarp();
			}
		// cursors now hold the END of each column == start of the next: shift back
		for (int64_t c0 = (int64_t) LY - 1 - ((int64_t)(LY - 1) % 32); c0 >= 0; c0 -= 32)
			{
			const int64_t c = c0 + lane;
			uint32_t v = 0;
			if (c < (int64_t) LY)
				v = tro[c];
			__syncwarp();
			if (c < (int64_t) LY)
				tro[c + 1] = v;
			__syncwarp();
			}
		if (lane == 0)
			tro[0] = 0;
		__syncwarp();
		}
	}

// tr_entries[t].p = entries[perm[t]].p; one warp per pair version (perm is relative to the pair's base)
__global__ void k_refresh_transposed_pairs(uint32_t npairs, const uint64_t *__restrict__ entbase,
  const uint32_t *__restrict__ nnz, const mb200_entry *__restrict__ entries, const uint32_t *__restrict__ perm,
  mb200_entry *__restrict__ tr_entries)
	{
	const uint32_t warp = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t nw = (gridDim.x*blockDim.x) >> 5;
	for (uint32_t k = warp; k < npairs; k += nw)
		{
		const uint64_t b = entbase[k];
		const uint32_t n = nnz[k];
		for (uint32_t t = lane; t < n; t += 32)
			tr_entries[b + t].p = entries[b + perm[b + t]].p;
		}
	}

// ---------------------------------------------------------------------------------------------
// the store's state (StoreState, engine.h) and its derived forms
static bool holds_allpairs(const mb200_ctx *ctx)
	{
	const StoreState &s = ctx->store;
	return s.pairs == PAIRS_RANGE && s.p_lo == 0 && s.p_hi == (uint64_t) ctx->nseq*(ctx->nseq - 1)/2;
	}

// pairs [p_lo,p_hi) of the row-major all-pairs order of n sequences, appended to px/py
static void allpairs_list(uint32_t n, uint32_t p_lo, uint32_t p_hi, std::vector<uint32_t> &px, std::vector<uint32_t> &py)
	{
	uint32_t p = 0;
	for (uint32_t i = 0; i < n && p < p_hi; ++i)
		for (uint32_t j = i + 1; j < n && p < p_hi; ++j, ++p)
			if (p >= p_lo)
				{
				px.push_back(i);
				py.push_back(j);
				}
	}

// first offset slot of every pair of the list and one past the last: LX+1 slots per pair
static std::vector<uint64_t> row_bases(const mb200_ctx *ctx, const std::vector<uint32_t> &px)
	{
	std::vector<uint64_t> rowbase(px.size() + 1, 0);
	for (size_t k = 0; k < px.size(); ++k)
		rowbase[k + 1] = rowbase[k] + ctx->h_len[px[k]] + 1;
	return rowbase;
	}

// Installs a new pair list: none, pairs [0,hi) of the caller's px/py (PAIRS_LIST, lo = 0), or the all-pairs
// range [lo,hi).  The store and the posterior plan of the old list go; the per-pair buffers of the store
// are sized and the list and its row bases uploaded.  A refused list leaves PAIRS_NONE.
int mb_store_set_pairs(mb200_ctx *ctx, StorePairs pairs, uint32_t lo, uint32_t hi, const uint32_t *px, const uint32_t *py)
	{
	ctx->store = StoreState{};
	ctx->plan.valid = false;
	ctx->h_px.clear();
	ctx->h_py.clear();
	ctx->h_rowbase.clear();
	if (pairs == PAIRS_NONE)
		return MB200_OK;
	if (pairs == PAIRS_LIST)
		{
		for (uint32_t k = 0; k < hi; ++k)
			if (px[k] >= ctx->nseq || py[k] >= ctx->nseq)
				return mb_fail(ctx, MB200_EINVAL, "pair %u references sequence out of range", k);
		ctx->h_px.assign(px, px + hi);
		ctx->h_py.assign(py, py + hi);
		}
	else
		allpairs_list(ctx->nseq, lo, hi, ctx->h_px, ctx->h_py);
	const uint32_t np = (uint32_t) ctx->h_px.size();
	ctx->h_rowbase = row_bases(ctx, ctx->h_px);
	ENSURE(ctx->d_px, np*sizeof(uint32_t));
	ENSURE(ctx->d_py, np*sizeof(uint32_t));
	ENSURE(ctx->d_rowbase, (np + 1)*sizeof(uint64_t));
	ENSURE(ctx->d_rowoff, ctx->h_rowbase[np]*sizeof(uint32_t));
	ENSURE(ctx->d_entbase, (np + 1)*sizeof(uint64_t));
	ENSURE(ctx->d_nnz, np*sizeof(uint32_t));
	ENSURE(ctx->d_ea, np*sizeof(float));
	cudaStream_t st = ctx->stream;
	CU(cudaMemcpyAsync(ctx->d_px.p, ctx->h_px.data(), np*sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(ctx->d_py.p, ctx->h_py.data(), np*sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(ctx->d_rowbase.p, ctx->h_rowbase.data(), (np + 1)*sizeof(uint64_t), cudaMemcpyHostToDevice, st));
	ctx->stats.h2d_bytes += 2ull*np*sizeof(uint32_t) + (np + 1)*sizeof(uint64_t);
	ctx->store = StoreState{pairs, lo, hi};
	return MB200_OK;
	}

// the inputs changed, or a posterior stage starts: the pair list and its plan stay
void mb_store_drop(mb200_ctx *ctx)
	{
	ctx->store.present = false;
	}

// a new store of the current pair list: computed by the posterior stage (raw layout, with its EA
// vector) or adopted as a packed image with its host index and no EA
void mb_store_fresh(mb200_ctx *ctx, bool adopted)
	{
	StoreState &s = ctx->store;
	s.present = true;
	s.ea_here = !adopted && holds_allpairs(ctx);
	s.form = adopted ? FORM_PACKED : FORM_RAW;
	s.index_valid = adopted;
	s.tr_stale = false;
	}

// the forward values changed in place (the pattern did not): the transposed copy is refreshed when next read
void mb_store_values_written(mb200_ctx *ctx)
	{
	ctx->store.tr_stale = true;
	}

// entries [e_lo,e_hi) of the pairs [p_lo,p_hi) of a packed store
void mb_store_entry_range(const mb200_ctx *ctx, uint32_t p_lo, uint32_t p_hi, uint64_t *e_lo, uint64_t *e_hi)
	{
	const size_t np = ctx->h_px.size();
	*e_lo = p_lo < np ? ctx->h_entbase[p_lo] : ctx->store_nnz;
	*e_hi = p_hi < np ? ctx->h_entbase[p_hi] : ctx->store_nnz;
	}

// h_nnz and, unless packing is about to compute them, h_entbase from the device
static int read_index(mb200_ctx *ctx, bool entbase)
	{
	const size_t np = ctx->h_px.size();
	ctx->h_nnz.resize(np);
	CU(cudaMemcpyAsync(ctx->h_nnz.data(), ctx->d_nnz.p, np*sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
	if (entbase)
		{
		ctx->h_entbase.resize(np);
		CU(cudaMemcpyAsync(ctx->h_entbase.data(), ctx->d_entbase.p, np*sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
		}
	CU(cudaStreamSynchronize(ctx->stream));
	ctx->store.index_valid = entbase;
	return MB200_OK;
	}

// make entbase the exclusive scan of nnz in store order (deterministic layout, no holes)
static int pack(mb200_ctx *ctx)
	{
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	const uint32_t np = (uint32_t) ctx->h_px.size();
	if (!ctx->store.index_valid)
		{
		const int rc = read_index(ctx, false);
		if (rc != MB200_OK)
			return rc;
		}
	std::vector<uint64_t> base(np + 1, 0);
	for (uint32_t k = 0; k < np; ++k)
		base[k + 1] = base[k] + ctx->h_nnz[k];
	const uint64_t total = base[np];
	ENSURE(ctx->d_tmp, (np + 1)*sizeof(uint64_t));
	CU(cudaMemcpyAsync(ctx->d_tmp.p, base.data(), (np + 1)*sizeof(uint64_t), cudaMemcpyHostToDevice, st));
	ENSURE(ctx->d_entries2, (total + 64)*sizeof(mb200_entry));
	const int blocks = ctx->prop.multiProcessorCount*8;
	k_pack_entries<<<blocks, 256, 0, st>>>(np, (const uint64_t *) ctx->d_entbase.p, (const uint64_t *) ctx->d_tmp.p,
	  (const uint32_t *) ctx->d_nnz.p, (const mb200_entry *) ctx->d_entries.p, (mb200_entry *) ctx->d_entries2.p);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches++;
	CU(cudaMemcpyAsync(ctx->d_entbase.p, ctx->d_tmp.p, np*sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
	CU(cudaStreamSynchronize(st));
	std::swap(ctx->d_entries, ctx->d_entries2);
	ctx->h_entbase.assign(base.begin(), base.begin() + np);
	ctx->store_nnz = total;
	ctx->store.index_valid = true;
	ctx->store.form = FORM_PACKED;
	return MB200_OK;
	}

static int build_transposed(mb200_ctx *ctx)
	{
	cudaStream_t st = ctx->stream;
	const uint32_t np = (uint32_t) ctx->h_px.size();
	std::vector<uint64_t> trb(np + 1, 0);
	for (uint32_t k = 0; k < np; ++k)
		trb[k + 1] = trb[k] + ctx->h_len[ctx->h_py[k]] + 1;
	ENSURE(ctx->d_tr_rowbase, (np + 1)*sizeof(uint64_t));
	ENSURE(ctx->d_tr_rowoff, trb[np]*sizeof(uint32_t));
	ENSURE(ctx->d_tr_entries, (ctx->store_nnz + 64)*sizeof(mb200_entry));
	ENSURE(ctx->d_tr_perm, (ctx->store_nnz + 64)*sizeof(uint32_t));
	CU(cudaMemcpyAsync(ctx->d_tr_rowbase.p, trb.data(), (np + 1)*sizeof(uint64_t), cudaMemcpyHostToDevice, st));
	const int blocks = ctx->prop.multiProcessorCount*8;
	k_transpose_pairs<<<blocks, 256, 0, st>>>(np, (const uint32_t *) ctx->d_px.p, (const uint32_t *) ctx->d_py.p,
	  (const uint32_t *) ctx->d_seqlen.p, (const uint64_t *) ctx->d_rowbase.p, (const uint32_t *) ctx->d_rowoff.p,
	  (const uint64_t *) ctx->d_entbase.p, (const mb200_entry *) ctx->d_entries.p,
	  (const uint64_t *) ctx->d_tr_rowbase.p, (uint32_t *) ctx->d_tr_rowoff.p,
	  (mb200_entry *) ctx->d_tr_entries.p, (uint32_t *) ctx->d_tr_perm.p);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches++;
	CU(cudaStreamSynchronize(st));
	ctx->h_tr_rowbase = trb;
	ctx->store.form = FORM_TRANSPOSED;
	ctx->store.tr_stale = false;
	return MB200_OK;
	}

static int refresh_transposed(mb200_ctx *ctx)
	{
	const uint32_t np = (uint32_t) ctx->h_px.size();
	const int blocks = ctx->prop.multiProcessorCount*8;
	k_refresh_transposed_pairs<<<blocks, 256, 0, ctx->stream>>>(np, (const uint64_t *) ctx->d_entbase.p,
	  (const uint32_t *) ctx->d_nnz.p, (const mb200_entry *) ctx->d_entries.p, (const uint32_t *) ctx->d_tr_perm.p,
	  (mb200_entry *) ctx->d_tr_entries.p);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches++;
	ctx->store.tr_stale = false;
	return MB200_OK;
	}

// Checks what `needs` asks of the store and builds the derived forms it lacks, in chain order
int mb_store_require(mb200_ctx *ctx, const char *who, unsigned needs)
	{
	StoreState &s = ctx->store;
	if ((needs & NEED_EA) && !(s.present && s.ea_here))
		return mb_fail(ctx, MB200_EINVAL, "%s: no all-pairs EA vector on this device "
		  "(mb200_posteriors_allpairs(0, npairs) must have run here, or pass ea)", who);
	if ((needs & NEED_ALLPAIRS) && !(s.present && holds_allpairs(ctx)))
		return mb_fail(ctx, MB200_EINVAL, "%s: the store must hold all N(N-1)/2 pairs "
		  "(mb200_posteriors_allpairs(0,npairs) or mb200_store_load_allpairs)", who);
	if (!s.present)
		return mb_fail(ctx, MB200_EINVAL, "no posterior store (run mb200_posteriors first)");
	const unsigned want = needs & 3;
	int rc = MB200_OK;
	if (want == FORM_MASKED && s.form < FORM_MASKED)
		{
		// the posterior scratch goes first: at C3 both stages fit one 80 GB device only without it
		CU(cudaStreamSynchronize(ctx->stream));
		mb_release_post_scratch(ctx);
		}
	if (want >= FORM_PACKED && s.form < FORM_PACKED && (rc = pack(ctx)) != MB200_OK)
		return rc;
	if (want >= FORM_TRANSPOSED && s.form < FORM_TRANSPOSED && (rc = build_transposed(ctx)) != MB200_OK)
		return rc;
	if (want >= FORM_TRANSPOSED && s.tr_stale && (rc = refresh_transposed(ctx)) != MB200_OK)
		return rc;
	if (want == FORM_MASKED && s.form < FORM_MASKED)
		{
		if ((rc = mb_build_masks(ctx)) != MB200_OK)
			return rc;
		s.form = FORM_MASKED;
		}
	if ((needs & NEED_INDEX) && !s.index_valid && (rc = read_index(ctx, true)) != MB200_OK)
		return rc;
	return MB200_OK;
	}

// mb_store_require(needs), then the kernels' view of the store: the transposed side is filled when `needs`
// asks for FORM_TRANSPOSED or more, the column masks when it asks for FORM_MASKED
int mb_store_view(mb200_ctx *ctx, const char *who, unsigned needs, StoreView *v)
	{
	const int rc = mb_store_require(ctx, who, needs);
	if (rc != MB200_OK)
		return rc;
	const unsigned want = needs & 3;
	*v = StoreView{};
	v->n = ctx->nseq;
	v->entbase = (const uint64_t *) ctx->d_entbase.p;
	v->fwd.rowbase = (const uint64_t *) ctx->d_rowbase.p;
	v->fwd.rowoff = (const uint32_t *) ctx->d_rowoff.p;
	v->fwd.entries = (const mb200_entry *) ctx->d_entries.p;
	if (want >= FORM_TRANSPOSED)
		{
		v->tr.rowbase = (const uint64_t *) ctx->d_tr_rowbase.p;
		v->tr.rowoff = (const uint32_t *) ctx->d_tr_rowoff.p;
		v->tr.entries = (const mb200_entry *) ctx->d_tr_entries.p;
		}
	if (want == FORM_MASKED)
		{
		v->fwd.hdr = (const uint2 *) ctx->d_mk_hdr.p;
		v->fwd.words = (const uint2 *) ctx->d_mk_words.p;
		v->tr.hdr = (const uint2 *) ctx->d_tr_mk_hdr.p;
		v->tr.words = (const uint2 *) ctx->d_tr_mk_words.p;
		}
	return MB200_OK;
	}

extern "C" {

int mb200_store_pack(mb200_ctx *ctx, const uint32_t **d_offsets, uint64_t *n_offsets,
  const mb200_entry **d_entries, uint64_t *n_entries)
	{
	if (!ctx)
		return MB200_EINVAL;
	const int rc = mb_store_require(ctx, "mb200_store_pack", FORM_PACKED);
	if (rc != MB200_OK)
		return rc;
	if (d_offsets)
		*d_offsets = (const uint32_t *) ctx->d_rowoff.p;
	if (n_offsets)
		*n_offsets = ctx->h_rowbase.back();
	if (d_entries)
		*d_entries = (const mb200_entry *) ctx->d_entries.p;
	if (n_entries)
		*n_entries = ctx->store_nnz;
	return MB200_OK;
	}

int mb200_export_all(mb200_ctx *ctx, uint32_t *offsets_concat, mb200_entry *entries_concat)
	{
	if (!ctx || !offsets_concat || !entries_concat)
		return mb_fail(ctx, MB200_EINVAL, "mb200_export_all: NULL argument");
	const int rc = mb_store_require(ctx, "mb200_export_all", FORM_PACKED);
	if (rc != MB200_OK)
		return rc;
	CU(cudaMemcpy(offsets_concat, ctx->d_rowoff.p, ctx->h_rowbase.back()*sizeof(uint32_t), cudaMemcpyDeviceToHost));
	CU(cudaMemcpy(entries_concat, ctx->d_entries.p, ctx->store_nnz*sizeof(mb200_entry), cudaMemcpyDeviceToHost));
	ctx->stats.d2h_bytes += ctx->h_rowbase.back()*sizeof(uint32_t) + ctx->store_nnz*sizeof(mb200_entry);
	return MB200_OK;
	}

// In-place exchange (multi-GPU): the gathered image is received directly into library-owned
// buffers, then adopted as the store -- no staging copy of a 10 GB image.
int mb200_store_exchange_begin(mb200_ctx *ctx, uint64_t n_offsets, uint64_t n_entries, uint32_t **d_offsets,
  mb200_entry **d_entries)
	{
	if (!ctx || !d_offsets || !d_entries || ctx->nseq < 2)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_exchange_begin: bad argument");
	cudaSetDevice(ctx->device);
	std::vector<uint32_t> px, py;
	allpairs_list(ctx->nseq, 0, (uint32_t)((uint64_t) ctx->nseq*(ctx->nseq - 1)/2), px, py);
	const uint64_t rows = row_bases(ctx, px).back();
	if (rows != n_offsets)
		return mb_fail(ctx, MB200_EINVAL, "offset image has %llu slots, all pairs need %llu",
		  (unsigned long long) n_offsets, (unsigned long long) rows);
	// the caller's own packed store (d_rowoff / d_entries) stays valid and readable until commit
	ENSURE(ctx->d_pack_off, n_offsets*sizeof(uint32_t));
	ENSURE(ctx->d_pack_ent, (n_entries + 64)*sizeof(mb200_entry));
	ctx->xchg_n_offsets = n_offsets;
	ctx->xchg_n_entries = n_entries;
	*d_offsets = (uint32_t *) ctx->d_pack_off.p;
	*d_entries = (mb200_entry *) ctx->d_pack_ent.p;
	return MB200_OK;
	}

// adopt d_pack_off / d_pack_ent (filled by the caller) as the store of all-pairs range [p_lo,p_hi)
static int adopt_image(mb200_ctx *ctx, uint32_t p_lo, uint32_t p_hi, uint64_t n_offsets, uint64_t n_entries)
	{
	// the image becomes the store's buffers and its pair list is installed before the checks: a refused image
	// leaves no store, like a failed posterior call, and d_rowoff needs no second buffer of the image's size
	std::swap(ctx->d_rowoff, ctx->d_pack_off);
	std::swap(ctx->d_entries, ctx->d_pack_ent);
	int rc = mb_store_set_pairs(ctx, PAIRS_RANGE, p_lo, p_hi);
	if (rc != MB200_OK)
		return rc;
	cudaStream_t st = ctx->stream;
	const uint32_t np = (uint32_t) ctx->h_px.size();
	if (ctx->h_rowbase[np] != n_offsets)
		return mb_fail(ctx, MB200_EINVAL, "offset image has %llu slots, pair range needs %llu",
		  (unsigned long long) n_offsets, (unsigned long long) ctx->h_rowbase[np]);
	ENSURE(ctx->d_tmp, (np + 1)*sizeof(uint64_t));
	k_nnz_from_rowoff<<<(np + 255)/256, 256, 0, st>>>(np, (const uint64_t *) ctx->d_rowbase.p,
	  (const uint32_t *) ctx->d_rowoff.p, (uint32_t *) ctx->d_nnz.p, (uint64_t *) ctx->d_tmp.p);
	CU(cudaGetLastError());
	size_t tb = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, tb, (uint64_t *) ctx->d_tmp.p, (uint64_t *) ctx->d_entbase.p, (int) np, st);
	ENSURE(ctx->d_tmp2, tb + 16);
	cub::DeviceScan::ExclusiveSum(ctx->d_tmp2.p, tb, (uint64_t *) ctx->d_tmp.p, (uint64_t *) ctx->d_entbase.p, (int) np, st);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches += 2;
	if ((rc = read_index(ctx, true)) != MB200_OK)
		return rc;
	const uint64_t tot = std::accumulate(ctx->h_nnz.begin(), ctx->h_nnz.end(), (uint64_t) 0);
	if (tot != n_entries)
		return mb_fail(ctx, MB200_EINVAL, "entry image has %llu entries, offsets say %llu",
		  (unsigned long long) n_entries, (unsigned long long) tot);
	ctx->store_nnz = tot;
	mb_store_fresh(ctx, true);
	return MB200_OK;
	}

int mb200_store_exchange_commit(mb200_ctx *ctx)
	{
	if (!ctx || ctx->xchg_n_offsets == 0)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_exchange_commit: no exchange in progress");
	cudaSetDevice(ctx->device);
	const uint64_t all = (uint64_t) ctx->nseq*(ctx->nseq - 1)/2;
	const int rc = adopt_image(ctx, 0, (uint32_t) all, ctx->xchg_n_offsets, ctx->xchg_n_entries);
	ctx->xchg_n_offsets = ctx->xchg_n_entries = 0;
	return rc;
	}

int mb200_store_load_allpairs(mb200_ctx *ctx, uint32_t p_lo, uint32_t p_hi, const uint32_t *d_offsets,
  uint64_t n_offsets, const mb200_entry *d_entries, uint64_t n_entries)
	{
	if (!ctx || !d_offsets || (!d_entries && n_entries > 0) || ctx->nseq < 2)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_load_allpairs: bad argument");
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	const uint64_t all = (uint64_t) ctx->nseq*(ctx->nseq - 1)/2;
	if (p_lo >= p_hi || p_hi > all)
		return mb_fail(ctx, MB200_EINVAL, "pair range [%u,%u) invalid", p_lo, p_hi);
	// the source image may alias our own buffers (single-rank round trip): stage before adopting
	ENSURE(ctx->d_pack_off, n_offsets*sizeof(uint32_t));
	ENSURE(ctx->d_pack_ent, (n_entries + 64)*sizeof(mb200_entry));
	CU(cudaMemcpyAsync(ctx->d_pack_off.p, d_offsets, n_offsets*sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
	if (n_entries)
		CU(cudaMemcpyAsync(ctx->d_pack_ent.p, d_entries, n_entries*sizeof(mb200_entry), cudaMemcpyDeviceToDevice, st));
	CU(cudaStreamSynchronize(st));
	return adopt_image(ctx, p_lo, p_hi, n_offsets, n_entries);
	}

int mb200_store_entries_ptr(mb200_ctx *ctx, mb200_entry **d_entries, uint64_t *n_entries)
	{
	if (!ctx || !d_entries)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_entries_ptr: NULL argument");
	const int rc = mb_store_require(ctx, "mb200_store_entries_ptr", FORM_PACKED);
	if (rc != MB200_OK)
		return rc;
	*d_entries = (mb200_entry *) ctx->d_entries.p;
	if (n_entries)
		*n_entries = ctx->store_nnz;
	return MB200_OK;
	}

int mb200_store_values_changed(mb200_ctx *ctx)
	{
	if (!ctx || !ctx->store.present)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_values_changed: no store");
	mb_store_values_written(ctx);
	return MB200_OK;
	}

int mb200_store_values(mb200_ctx *ctx, float *d_values_out, uint64_t n_entries)
	{
	if (!ctx || !d_values_out)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_values: NULL argument");
	const int rc = mb_store_require(ctx, "mb200_store_values", FORM_PACKED);
	if (rc != MB200_OK)
		return rc;
	if (n_entries != ctx->store_nnz)
		return mb_fail(ctx, MB200_EINVAL, "store has %llu entries, caller buffer %llu",
		  (unsigned long long) ctx->store_nnz, (unsigned long long) n_entries);
	k_gather_values<<<ctx->prop.multiProcessorCount*8, 256, 0, ctx->stream>>>(n_entries,
	  (const mb200_entry *) ctx->d_entries.p, d_values_out);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches++;
	CU(cudaStreamSynchronize(ctx->stream));
	return MB200_OK;
	}

int mb200_store_set_values(mb200_ctx *ctx, const float *d_values, uint64_t first_entry, uint64_t n_entries)
	{
	if (!ctx || !d_values)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_set_values: NULL argument");
	// refused rather than packed here: first_entry refers to the packed layout
	if (!ctx->store.present || ctx->store.form < FORM_PACKED)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_set_values: store must be packed (mb200_store_pack)");
	if (first_entry + n_entries > ctx->store_nnz)
		return mb_fail(ctx, MB200_EINVAL, "value range out of bounds");
	k_scatter_values<<<ctx->prop.multiProcessorCount*8, 256, 0, ctx->stream>>>(n_entries, d_values,
	  (mb200_entry *) ctx->d_entries.p + first_entry);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches++;
	CU(cudaStreamSynchronize(ctx->stream));
	mb_store_values_written(ctx);
	return MB200_OK;
	}

} // extern "C"
