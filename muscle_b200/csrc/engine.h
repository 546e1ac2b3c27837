// engine.h -- context layout shared by the host translation units of libmuscle_b200.so.
#pragma once
#include <vector>
#include "launch.h"

struct DevBuf
	{
	void  *p = nullptr;
	size_t cap = 0;
	int  ensure(size_t bytes);     // grow-only; 0 on success
	void release();
	};

struct PostDebug { float *fwd, *bwd, *post, *total; uint32_t pair; };

// What the sparse posterior store holds.  Only store.cu changes it (mb_store_* below).
enum StorePairs { PAIRS_NONE, PAIRS_LIST, PAIRS_RANGE };     // h_px/h_py: none, a caller's list, all pairs [p_lo,p_hi)
// derived forms in build order, each made from the one before: entries packed in store order without holes,
// the transposed orientation, the column masks of both orientations (relax.cu)
enum StoreForm { FORM_RAW, FORM_PACKED, FORM_TRANSPOSED, FORM_MASKED };
struct StoreState
	{
	StorePairs pairs = PAIRS_NONE;
	uint32_t p_lo = 0, p_hi = 0;
	bool present = false;             // the device holds the store of that pair list
	bool ea_here = false;             // d_ea holds the EA of all N(N-1)/2 pairs, computed on this device
	StoreForm form = FORM_RAW;
	bool index_valid = false;         // h_nnz / h_entbase match the device (always, once packed)
	bool tr_stale = false;            // forward values changed since the transposed copy was refreshed
	};
// mb_store_require(needs): the StoreForm a consumer reads, or'ed with: the store holds all N(N-1)/2 pairs,
// and their EA vector was computed here; the host index
constexpr unsigned NEED_ALLPAIRS = 4, NEED_EA = 8, NEED_INDEX = 16;

// Launch plan of the posterior stage: everything that depends only on the pair list, the forced width and
// R, the rows per lane per step of the emission mode (engine.cu build_plan; mb_store_set_pairs drops it)
struct PostClass                          // one size class
	{
	uint32_t chain0 = 0, nchains = 0;     // its chains: [chain0, chain0 + nchains) of d_chain
	uint32_t lxmax = 0, lymax = 0;
	uint64_t fsteps = 0;                  // most Forward steps of one chain, at R rows per step
	uint64_t rows = 0;                    // most rows of one chain (sum of LX)
	};
struct PostPlan
	{
	bool valid = false;
	int force_c = 0, R = 1;
	uint64_t cells = 0, est_entries = 0;
	PostClass cls[MB_MAX_C + 1];
	};

struct mb200_ctx
	{
	int device = 0;
	cudaDeviceProp prop;
	cudaStream_t stream = nullptr;
	cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;
	char err[512];
	mb200_stats stats = {};

	// HMM
	bool have_hmm = false;
	MbHmm hmm = {};
	uint8_t byte2class[256] = {};
	DevBuf d_matchT, d_insT;

	// sequences
	uint32_t nseq = 0;
	std::vector<uint8_t>  h_bytes;
	std::vector<uint64_t> h_off;
	std::vector<uint32_t> h_len;
	DevBuf d_codes, d_seqoff, d_seqlen;
	// Mega feature-profile emissions (mb200_set_seqs_mega): d_codes then holds 8 letters per position
	bool mega = false;
	uint32_t mega_nf = 0, mega_tsize = 0, mega_base[8] = {}, mega_alpha[8] = {};
	DevBuf d_megaT, d_insP;

	// the store: sparse posteriors of the listed pairs (replaces MPCFlat::m_SparsePosts1/2)
	StoreState store;
	std::vector<uint64_t> h_tr_rowbase;
	uint64_t store_nnz = 0;
	uint32_t nnz_per_row_cap = 12;    // entry pool sizing guess (retry with the exact count on overflow)
	std::vector<uint32_t> h_px, h_py;
	std::vector<uint64_t> h_rowbase;
	std::vector<uint32_t> h_nnz;
	std::vector<uint64_t> h_entbase;
	DevBuf d_px, d_py, d_order, d_chain;    // d_order: pairs chain after chain; d_chain: offsets of the chains in it
	DevBuf d_rowoff, d_rowbase, d_entries, d_cursor, d_entbase, d_nnz, d_ea;     // d_cursor: control block, see run_posteriors
	DevBuf d_entries2;                // second value buffer for the Jacobi update
	DevBuf d_pack_off, d_pack_ent;    // packed image for exchange/export
	uint64_t xchg_n_offsets = 0, xchg_n_entries = 0;      // sizes announced by mb200_store_exchange_begin
	// transposed orientation of every pair (rows = positions of Y) for the relax kernel
	DevBuf d_tr_rowoff, d_tr_rowbase, d_tr_entries, d_tr_perm;
	// column bit masks of every sparse row, both orientations (relax.cu): hdr = {first word slot,
	// w0 | nw << 16} per row, words = {mask of columns 32w..32w+31, index of the first such entry}
	DevBuf d_mk_hdr, d_mk_words, d_tr_mk_hdr, d_tr_mk_words;
	// relax work order (pairs of [p_lo,p_hi) in 2-D tile order) and the range it was built for
	DevBuf d_relax_order;
	uint32_t relax_order_n = 0, relax_order_lo = 0, relax_order_hi = 0;
	DevBuf d_tmp, d_tmp2;
	// device-resident MSAs (align.cu, SURVEY section 8 f3): position -> column of every residue
	// (same layout as d_codes) and, on the host, the column count of the MSA each sequence is in
	DevBuf d_p2c, d_join;             // d_join: per-join scratch (maps, Post, traceback, path)
	DevBuf d_stage;                   // BuildPost staging slots
	std::vector<uint32_t> h_msa_cols;
	bool msa_valid = false;
	uint32_t *h_pinned = nullptr;     // 64 words of pinned host memory for small read-backs

	PostPlan plan;
	uint64_t last_used_entries = 0;

	// per-warp scratch of the posterior kernel, one buffer per bin (PostParams fm, edge, rows, rowcnt, chainbuf)
	DevBuf d_post_scratch[MB_MAX_C + 1];
	static constexpr int kStreams = 4;          // column-width bins run concurrently to overlap their tails
	cudaStream_t aux[kStreams] = {};
	cudaEvent_t aux_done[kStreams] = {};
	DevBuf d_dbg;
	DevBuf d_math;                    // mb200_debug_math: one chunk of operands and results (math.cu)
	int debug_force_c = 0;
	int occ_cache[MB_MAX_C + 1] = {}, occ_cache_k = -1;     // resident CTAs/SM of k_posterior_sm per size class
	};

int mb_fail(mb200_ctx *ctx, int code, const char *fmt, ...);
// In a host function with a local `ctx` that returns an mb200 error code: fail on a CUDA error / a
// device allocation that cannot grow.
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
	return mb_fail(ctx, e_ == cudaErrorMemoryAllocation ? MB200_ENOMEM : MB200_ECUDA, \
	  "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } while (0)
#define ENSURE(buf, bytes) do { if ((buf).ensure(bytes) != 0) \
	return mb_fail(ctx, MB200_ENOMEM, "device allocation of %zu bytes failed (%s)", (size_t)(bytes), #buf); } while (0)
int mb_store_set_pairs(mb200_ctx *ctx, StorePairs pairs, uint32_t lo = 0, uint32_t hi = 0,
  const uint32_t *px = nullptr, const uint32_t *py = nullptr);
void mb_store_drop(mb200_ctx *ctx);
void mb_store_fresh(mb200_ctx *ctx, bool adopted);
void mb_store_values_written(mb200_ctx *ctx);
int mb_store_require(mb200_ctx *ctx, const char *who, unsigned needs);
int mb_store_view(mb200_ctx *ctx, const char *who, unsigned needs, StoreView *v);
void mb_store_entry_range(const mb200_ctx *ctx, uint32_t p_lo, uint32_t p_hi, uint64_t *e_lo, uint64_t *e_hi);
int mb_build_masks(mb200_ctx *ctx);             // relax.cu
void mb_release_post_scratch(mb200_ctx *ctx);
