// store.cu -- the device-resident sparse posterior store: packing in pair order (export and the
// multi-GPU exchange image), loading a gathered image, values-only views, and the transposed
// orientation that the consistency kernel needs.
//
// Reference counterparts: the store replaces MPCFlat::m_SparsePosts1/2 (mpcflat.h:46-49); the wire
// format of one pair is MySparseMx's (mysparsemx.h:6-98).  The transposed orientation replaces the
// reference's three index-order variants of RelaxFlat (relaxflat.cpp:4,33,62) and the linear
// GetProb/GetColToRowLoHi scans (mysparsemx.cpp:44-62,238-268).
#include "engine.h"
#include <cub/cub.cuh>
#include <algorithm>
#include <cstring>

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
// host helpers
int mb_store_pack_inplace(mb200_ctx *ctx)
	{
	// make entbase the exclusive scan of nnz in store order (deterministic layout, no holes)
	if (!ctx->store_valid)
		return mb_fail(ctx, MB200_EINVAL, "no posterior store (run mb200_posteriors first)");
	if (ctx->store_packed)
		return MB200_OK;
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	const uint32_t np = (uint32_t) ctx->h_px.size();
	ctx->h_nnz.resize(np);
	CU(cudaMemcpyAsync(ctx->h_nnz.data(), ctx->d_nnz.p, np*sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));
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
	ctx->h_index_valid = true;
	ctx->store_nnz = total;
	ctx->store_packed = true;
	ctx->store_tr_valid = false;
	ctx->store_masks_valid = false;
	return MB200_OK;
	}

int mb_store_build_transposed(mb200_ctx *ctx)
	{
	if (ctx->store_tr_valid)
		return MB200_OK;
	int rc = mb_store_pack_inplace(ctx);
	if (rc != MB200_OK)
		return rc;
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
	ctx->store_tr_valid = true;
	return MB200_OK;
	}

int mb_store_refresh_transposed(mb200_ctx *ctx)
	{
	const uint32_t np = (uint32_t) ctx->h_px.size();
	const int blocks = ctx->prop.multiProcessorCount*8;
	k_refresh_transposed_pairs<<<blocks, 256, 0, ctx->stream>>>(np, (const uint64_t *) ctx->d_entbase.p,
	  (const uint32_t *) ctx->d_nnz.p, (const mb200_entry *) ctx->d_entries.p, (const uint32_t *) ctx->d_tr_perm.p,
	  (mb200_entry *) ctx->d_tr_entries.p);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return MB200_OK;
	}

extern "C" {

int mb200_store_pack(mb200_ctx *ctx, const uint32_t **d_offsets, uint64_t *n_offsets,
  const mb200_entry **d_entries, uint64_t *n_entries)
	{
	if (!ctx)
		return MB200_EINVAL;
	const int rc = mb_store_pack_inplace(ctx);
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
	const int rc = mb_store_pack_inplace(ctx);
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
	uint64_t rows = 0;
	for (uint32_t i = 0; i + 1 < ctx->nseq; ++i)
		rows += (uint64_t)(ctx->h_len[i] + 1)*(ctx->nseq - 1 - i);
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
	cudaStream_t st = ctx->stream;
	const uint64_t all = (uint64_t) ctx->nseq*(ctx->nseq - 1)/2;
	std::vector<uint32_t> px, py;
	mb_allpairs_list(ctx->nseq, p_lo, p_hi, px, py);
	const uint32_t np = (uint32_t) px.size();
	std::vector<uint64_t> rowbase(np + 1, 0);
	for (uint32_t k = 0; k < np; ++k)
		rowbase[k + 1] = rowbase[k] + ctx->h_len[px[k]] + 1;
	if (rowbase[np] != n_offsets)
		return mb_fail(ctx, MB200_EINVAL, "offset image has %llu slots, pair range needs %llu",
		  (unsigned long long) n_offsets, (unsigned long long) rowbase[np]);
	ENSURE(ctx->d_px, np*sizeof(uint32_t));
	ENSURE(ctx->d_py, np*sizeof(uint32_t));
	ENSURE(ctx->d_rowbase, (np + 1)*sizeof(uint64_t));
	ENSURE(ctx->d_entbase, (np + 1)*sizeof(uint64_t));
	ENSURE(ctx->d_nnz, np*sizeof(uint32_t));
	ENSURE(ctx->d_ea, np*sizeof(float));
	ENSURE(ctx->d_tmp, (np + 1)*sizeof(uint64_t));
	CU(cudaMemcpyAsync(ctx->d_px.p, px.data(), np*sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(ctx->d_py.p, py.data(), np*sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(ctx->d_rowbase.p, rowbase.data(), (np + 1)*sizeof(uint64_t), cudaMemcpyHostToDevice, st));
	k_nnz_from_rowoff<<<(np + 255)/256, 256, 0, st>>>(np, (const uint64_t *) ctx->d_rowbase.p,
	  (const uint32_t *) ctx->d_pack_off.p, (uint32_t *) ctx->d_nnz.p, (uint64_t *) ctx->d_tmp.p);
	CU(cudaGetLastError());
	size_t tb = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, tb, (uint64_t *) ctx->d_tmp.p, (uint64_t *) ctx->d_entbase.p, (int) np, st);
	ENSURE(ctx->d_tmp2, tb + 16);
	cub::DeviceScan::ExclusiveSum(ctx->d_tmp2.p, tb, (uint64_t *) ctx->d_tmp.p, (uint64_t *) ctx->d_entbase.p, (int) np, st);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches += 2;
	std::vector<uint32_t> h_nnz(np);
	std::vector<uint64_t> h_entbase(np);
	CU(cudaMemcpyAsync(h_nnz.data(), ctx->d_nnz.p, np*sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	CU(cudaMemcpyAsync(h_entbase.data(), ctx->d_entbase.p, np*sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));
	uint64_t tot = 0;
	for (uint32_t k = 0; k < np; ++k)
		tot += h_nnz[k];
	if (tot != n_entries)
		return mb_fail(ctx, MB200_EINVAL, "entry image has %llu entries, offsets say %llu",
		  (unsigned long long) n_entries, (unsigned long long) tot);
	// everything validated: mutate the context
	std::swap(ctx->d_rowoff, ctx->d_pack_off);
	std::swap(ctx->d_entries, ctx->d_pack_ent);
	ctx->h_px.swap(px);
	ctx->h_py.swap(py);
	ctx->h_rowbase.swap(rowbase);
	ctx->h_nnz.swap(h_nnz);
	ctx->h_entbase.swap(h_entbase);
	ctx->plan_valid = false;
	ctx->h_index_valid = true;
	ctx->store_nnz = tot;
	ctx->store_valid = true;
	ctx->store_packed = true;
	ctx->store_tr_valid = false;
	ctx->store_masks_valid = false;
	ctx->tr_values_stale = false;
	ctx->store_allpairs = (p_lo == 0 && p_hi == all);
	ctx->ea_allpairs = false;          // the adopted image carries no EA values
	ctx->plan_is_allpairs = false;
	ctx->store_p_lo = p_lo;
	ctx->store_p_hi = p_hi;
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
	const int rc = mb_store_pack_inplace(ctx);
	if (rc != MB200_OK)
		return rc;
	*d_entries = (mb200_entry *) ctx->d_entries.p;
	if (n_entries)
		*n_entries = ctx->store_nnz;
	return MB200_OK;
	}

int mb200_store_values_changed(mb200_ctx *ctx)
	{
	if (!ctx || !ctx->store_valid)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_values_changed: no store");
	ctx->tr_values_stale = true;
	return MB200_OK;
	}

int mb200_store_values(mb200_ctx *ctx, float *d_values_out, uint64_t n_entries)
	{
	if (!ctx || !d_values_out)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_values: NULL argument");
	const int rc = mb_store_pack_inplace(ctx);
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
	if (!ctx->store_valid || !ctx->store_packed)
		return mb_fail(ctx, MB200_EINVAL, "mb200_store_set_values: store must be packed (mb200_store_pack)");
	if (first_entry + n_entries > ctx->store_nnz)
		return mb_fail(ctx, MB200_EINVAL, "value range out of bounds");
	k_scatter_values<<<ctx->prop.multiProcessorCount*8, 256, 0, ctx->stream>>>(n_entries, d_values,
	  (mb200_entry *) ctx->d_entries.p + first_entry);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches++;
	CU(cudaStreamSynchronize(ctx->stream));
	ctx->tr_values_stale = true;
	return MB200_OK;
	}

} // extern "C"
