// engine.cu -- host side of libmuscle_b200.so: context, uploads, work binning, launches, C ABI.
//
// The C ABI (include/muscle_b200.h) mirrors the reference's MPCFlat call sites; nothing here
// falls back to the CPU: without a CUDA device every entry point fails with MB200_ENODEV.
#include "engine.h"
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <numeric>

static char g_create_error[512] = "";

int mb_fail(mb200_ctx *ctx, int code, const char *fmt, ...)
	{
	char *dst = ctx ? ctx->err : g_create_error;
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(dst, 512, fmt, ap);
	va_end(ap);
	return code;
	}

int DevBuf::ensure(size_t need)
	{
	if (need <= cap)
		return 0;
	if (p)
		cudaFree(p);
	p = nullptr;
	cap = 0;
	size_t want = need + need/8 + 256;
	cudaError_t e = cudaMalloc(&p, want);
	if (e != cudaSuccess)
		{
		want = need;
		e = cudaMalloc(&p, want);
		}
	if (e != cudaSuccess)
		{
		cudaGetLastError();
		return -1;
		}
	cap = want;
	return 0;
	}

void DevBuf::release()
	{
	if (p)
		cudaFree(p);
	p = nullptr;
	cap = 0;
	}

// the per-warp scratch of the posterior kernel (sized from the free memory at launch, tens of GB on
// large all-pairs problems); the consistency stage frees it before it builds its own buffers so that
// both stages of a 1000-protein problem fit one 80 GB device.  The next posterior call reallocates it.
void mb_release_post_scratch(mb200_ctx *ctx)
	{
	for (DevBuf &b : ctx->d_post_scratch)
		b.release();
	}

extern "C" {

const char *mb200_version(void) { return "0.1.0 sm_90a"; }

const char *mb200_last_error(const mb200_ctx *ctx) { return ctx ? ctx->err : g_create_error; }

int mb200_create(int device, mb200_ctx **out)
	{
	mb200_ctx *ctx = nullptr;
	if (out == nullptr)
		return mb_fail(nullptr, MB200_EINVAL, "mb200_create: out is NULL");
	*out = nullptr;
	int ndev = 0;
	cudaError_t e = cudaGetDeviceCount(&ndev);
	if (e != cudaSuccess || ndev == 0)
		{
		cudaGetLastError();
		return mb_fail(nullptr, MB200_ENODEV, "no CUDA device (%s); libmuscle_b200 has no CPU path",
		  e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
		}
	if (device < 0 || device >= ndev)
		return mb_fail(nullptr, MB200_EINVAL, "device %d out of range (have %d)", device, ndev);
	ctx = new mb200_ctx();
	ctx->device = device;
	ctx->err[0] = 0;
	if (cudaSetDevice(device) != cudaSuccess || cudaGetDeviceProperties(&ctx->prop, device) != cudaSuccess)
		{
		mb_fail(nullptr, MB200_ECUDA, "cudaSetDevice(%d) failed: %s", device, cudaGetErrorString(cudaGetLastError()));
		delete ctx;
		return MB200_ECUDA;
		}
	if (ctx->prop.major != 9 || ctx->prop.minor != 0)
		{
		mb_fail(nullptr, MB200_ENODEV, "device %d is sm_%d%d; libmuscle_b200 is built for sm_90a (H100) only",
		  device, ctx->prop.major, ctx->prop.minor);
		delete ctx;
		return MB200_ENODEV;
		}
	cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
	cudaHostAlloc((void **) &ctx->h_pinned, 64*sizeof(uint32_t), cudaHostAllocDefault);
	cudaEventCreate(&ctx->ev0);
	cudaEventCreate(&ctx->ev1);
	cudaEventCreate(&ctx->ev2);
	cudaEventCreate(&ctx->ev3);
	for (int k = 0; k < mb200_ctx::kStreams; ++k)
		{
		cudaStreamCreateWithFlags(&ctx->aux[k], cudaStreamNonBlocking);
		cudaEventCreateWithFlags(&ctx->aux_done[k], cudaEventDisableTiming);
		}
	*out = ctx;
	return MB200_OK;
	}

void mb200_destroy(mb200_ctx *ctx)
	{
	if (!ctx)
		return;
	cudaSetDevice(ctx->device);
	cudaStreamSynchronize(ctx->stream);
	DevBuf *bufs[] = { &ctx->d_matchT, &ctx->d_insT, &ctx->d_codes, &ctx->d_seqoff, &ctx->d_seqlen, &ctx->d_px,
	  &ctx->d_py, &ctx->d_order, &ctx->d_chain,
	  &ctx->d_rowoff, &ctx->d_rowbase, &ctx->d_entries, &ctx->d_cursor, &ctx->d_entbase, &ctx->d_nnz,
	  &ctx->d_ea, &ctx->d_dbg, &ctx->d_pack_off, &ctx->d_pack_ent, &ctx->d_entries2,
	  &ctx->d_tr_rowoff, &ctx->d_tr_rowbase, &ctx->d_tr_entries, &ctx->d_tr_perm,
	  &ctx->d_tmp, &ctx->d_tmp2, &ctx->d_mk_hdr, &ctx->d_mk_words, &ctx->d_tr_mk_hdr, &ctx->d_tr_mk_words,
	  &ctx->d_relax_order, &ctx->d_p2c, &ctx->d_join, &ctx->d_stage, &ctx->d_megaT, &ctx->d_insP };
	if (ctx->h_pinned)
		cudaFreeHost(ctx->h_pinned);
	for (DevBuf *b : bufs)
		b->release();
	mb_release_post_scratch(ctx);
	for (int k = 0; k < mb200_ctx::kStreams; ++k)
		{
		cudaStreamSynchronize(ctx->aux[k]);
		cudaStreamDestroy(ctx->aux[k]);
		cudaEventDestroy(ctx->aux_done[k]);
		}
	cudaEventDestroy(ctx->ev0);
	cudaEventDestroy(ctx->ev1);
	cudaEventDestroy(ctx->ev2);
	cudaEventDestroy(ctx->ev3);
	cudaStreamDestroy(ctx->stream);
	delete ctx;
	}

int mb200_get_stats(const mb200_ctx *ctx, mb200_stats *out)
	{
	if (!ctx || !out)
		return MB200_EINVAL;
	*out = ctx->stats;
	return MB200_OK;
	}

// Pure host helper (no device needed; also exported for the CPU tests): bytes with the same insert
// score and the same match row AND column form one residue class; class ids are assigned in order
// of first appearance, rep[k] is the first byte of class k.
extern "C" int mb200_residue_classes(const float ins[256], const float match[65536], uint8_t byte2class[256],
  int *nclass_out, int rep_out[256])
	{
	if (!ins || !match || !byte2class || !nclass_out)
		return MB200_EINVAL;
	int nclass = 0;
	int rep[256];
	for (int b = 0; b < 256; ++b)
		{
		int found = -1;
		for (int k = 0; k < nclass && found < 0; ++k)
			{
			const int a = rep[k];
			if (memcmp(&ins[a], &ins[b], sizeof(float)) != 0)
				continue;
			if (memcmp(match + 256*a, match + 256*b, 256*sizeof(float)) != 0)
				continue;
			bool same = true;
			for (int r = 0; r < 256 && same; ++r)
				same = memcmp(&match[256*r + a], &match[256*r + b], sizeof(float)) == 0;
			if (same)
				found = k;
			}
		if (found < 0)
			{
			rep[nclass] = b;
			found = nclass++;
			}
		byte2class[b] = (uint8_t) found;
		}
	*nclass_out = nclass;
	if (rep_out)
		memcpy(rep_out, rep, sizeof(int)*256);
	return MB200_OK;
	}

// ------------------------------------------------------------------------------------------
// HMM tables: bytes with identical insert score and identical match row/column are merged into
// one residue class so that the device tables stay tiny (21 classes for proteins).
static int recode_seqs(mb200_ctx *ctx);

int mb200_set_hmm(mb200_ctx *ctx, const float start[5], const float trans[25], const float ins[256],
  const float match[65536], float min_sparse_score)
	{
	if (!ctx || !start || !trans || !ins || !match)
		return mb_fail(ctx, MB200_EINVAL, "mb200_set_hmm: NULL argument");
	cudaSetDevice(ctx->device);
	// validate before touching the context (a rejected table leaves the previous one in force)
	int nclass = 0;
	int rep[256];
	uint8_t byte2class[256];
	mb200_residue_classes(ins, match, byte2class, &nclass, rep);
	if (nclass > MB_MAX_K)
		return mb_fail(ctx, MB200_EALPHABET, "%d distinct residue classes in the HMM tables, device tables hold %d",
		  nclass, MB_MAX_K);
	MbHmm h = ctx->hmm;
	// state order M=0, IX=1, IY=2, JX=3, JY=4 (pairhmm.h:11-19); aliases of hmmscores.h:1-13
	h.tSM = start[0]; h.tSI = start[1]; h.tSJ = start[3];
	h.tMM = trans[0*5 + 0]; h.tMI = trans[0*5 + 1]; h.tMJ = trans[0*5 + 3];
	h.tII = trans[1*5 + 1]; h.tIM = trans[1*5 + 0];
	h.tJJ = trans[3*5 + 3]; h.tJM = trans[3*5 + 0];
	h.minScore = min_sparse_score;
	h.K = nclass;
	h.KS = nclass | 1;                 // odd row stride spreads match rows over the smem banks
	h.pad = byte2class[0];            // the reference reads byte 0 past the sequence end (bwdflat3.cpp:48,66)
	std::vector<float> insT(h.K), matchT((size_t) h.K*h.KS, 0.0f);
	for (int a = 0; a < h.K; ++a)
		{
		insT[a] = ins[rep[a]];
		for (int b = 0; b < h.K; ++b)
			matchT[(size_t) a*h.KS + b] = match[256*rep[a] + rep[b]];
		}
	ENSURE(ctx->d_insT, insT.size()*sizeof(float));
	ENSURE(ctx->d_matchT, matchT.size()*sizeof(float));
	CU(cudaMemcpyAsync(ctx->d_insT.p, insT.data(), insT.size()*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	CU(cudaMemcpyAsync(ctx->d_matchT.p, matchT.data(), matchT.size()*sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
	CU(cudaStreamSynchronize(ctx->stream));
	ctx->hmm = h;
	memcpy(ctx->byte2class, byte2class, sizeof(byte2class));
	ctx->have_hmm = true;
	mb_store_drop(ctx);
	if (ctx->nseq > 0)
		return recode_seqs(ctx);
	return MB200_OK;
	}

static int recode_seqs(mb200_ctx *ctx)
	{
	if (ctx->mega)
		return MB200_OK;                   // feature letters are not residue classes: nothing depends on the tables
	std::vector<uint8_t> codes(ctx->h_bytes.size());
	for (size_t k = 0; k < codes.size(); ++k)
		codes[k] = ctx->byte2class[ctx->h_bytes[k]];
	ENSURE(ctx->d_codes, codes.size() + 16);
	CU(cudaMemcpyAsync(ctx->d_codes.p, codes.data(), codes.size(), cudaMemcpyHostToDevice, ctx->stream));
	CU(cudaStreamSynchronize(ctx->stream));
	ctx->stats.h2d_bytes += codes.size();
	return MB200_OK;
	}

// Offsets of mb200_set_seqs / mb200_set_seqs_mega: every sequence non-empty and shorter than 2^31
static int check_offsets(mb200_ctx *ctx, uint32_t nseq, const uint64_t *offsets, const char *what)
	{
	for (uint32_t i = 0; i < nseq; ++i)
		{
		if (offsets[i + 1] <= offsets[i])
			return mb_fail(ctx, MB200_EINVAL, "%s %u is empty or offsets not increasing", what, i);
		if (offsets[i + 1] - offsets[i] > 0x7fffffffull)
			return mb_fail(ctx, MB200_EOVERFLOW, "%s %u too long", what, i);
		}
	return MB200_OK;
	}

// New sequences of either kind, validated: offsets from 0 and lengths on host and device, the statistics
// restart, and the pair list, the store and the MSAs of the old ones are dropped.  Enqueues uploads only.
static int install_seqs(mb200_ctx *ctx, uint32_t nseq, const uint64_t *offsets, bool mega)
	{
	ctx->nseq = nseq;
	ctx->mega = mega;
	ctx->h_off.assign(offsets, offsets + nseq + 1);
	for (auto &o : ctx->h_off)
		o -= offsets[0];
	ctx->h_len.resize(nseq);
	for (uint32_t i = 0; i < nseq; ++i)
		ctx->h_len[i] = (uint32_t)(offsets[i + 1] - offsets[i]);
	ctx->msa_valid = false;
	ENSURE(ctx->d_seqoff, (nseq + 1)*sizeof(uint64_t));
	ENSURE(ctx->d_seqlen, nseq*sizeof(uint32_t));
	CU(cudaMemcpyAsync(ctx->d_seqoff.p, ctx->h_off.data(), (nseq + 1)*sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->stream));
	CU(cudaMemcpyAsync(ctx->d_seqlen.p, ctx->h_len.data(), nseq*sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
	ctx->stats.h2d_bytes = (nseq + 1)*sizeof(uint64_t) + nseq*sizeof(uint32_t);
	ctx->stats.d2h_bytes = 0;
	mb_store_set_pairs(ctx, PAIRS_NONE);
	ctx->last_used_entries = 0;
	return MB200_OK;
	}

int mb200_set_seqs(mb200_ctx *ctx, uint32_t nseq, const uint8_t *bytes, const uint64_t *offsets)
	{
	if (!ctx || !bytes || !offsets || nseq == 0)
		return mb_fail(ctx, MB200_EINVAL, "mb200_set_seqs: bad argument");
	cudaSetDevice(ctx->device);
	// validate before touching the context (a failed call leaves the previous sequences usable)
	int rc = check_offsets(ctx, nseq, offsets, "sequence");
	if (rc != MB200_OK)
		return rc;
	ctx->h_bytes.assign(bytes + offsets[0], bytes + offsets[nseq]);
	rc = install_seqs(ctx, nseq, offsets, false);
	if (rc != MB200_OK)
		return rc;
	if (ctx->have_hmm)
		return recode_seqs(ctx);
	CU(cudaStreamSynchronize(ctx->stream));
	return MB200_OK;
	}

// Mega (Muscle-3D) feature profiles instead of residue bytes.  Replaces the emission side of
// Mega::CalcFwdFlat_mega / CalcBwdFlat_mega (fwdflat_mega.cpp:14, bwdflat_mega.cpp): the pair tables
// are pre-multiplied by the feature weights and the insert emission of every position is summed in
// feature order, with the same fp32 operations as Mega::GetMatchScore / GetInsScore (mega.cpp:273-359).
int mb200_set_seqs_mega(mb200_ctx *ctx, uint32_t nseq, const uint8_t *letters, const uint64_t *offsets,
  uint32_t nfeat, const uint32_t *alpha, const float *weights, const float *logprobs, const float *logprobmx)
	{
	if (!ctx || !letters || !offsets || !alpha || !weights || !logprobs || !logprobmx || nseq == 0)
		return mb_fail(ctx, MB200_EINVAL, "mb200_set_seqs_mega: bad argument");
	if (nfeat == 0 || nfeat > 8)
		return mb_fail(ctx, MB200_EALPHABET, "mb200_set_seqs_mega: %u features, the kernel handles 1..8", nfeat);
	cudaSetDevice(ctx->device);
	uint32_t tsize = 0, lsize = 0, base[8] = {}, lbase[8] = {};
	for (uint32_t f = 0; f < nfeat; ++f)
		{
		if (alpha[f] == 0 || alpha[f] > 256)
			return mb_fail(ctx, MB200_EALPHABET, "mb200_set_seqs_mega: feature %u has alphabet size %u", f, alpha[f]);
		base[f] = tsize; lbase[f] = lsize;
		tsize += alpha[f]*alpha[f];
		lsize += alpha[f];
		}
	if (tsize > 12*1024)
		return mb_fail(ctx, MB200_EALPHABET, "mb200_set_seqs_mega: pair tables of %u floats do not fit the kernel's shared memory", tsize);
	int rc = check_offsets(ctx, nseq, offsets, "profile");
	if (rc != MB200_OK)
		return rc;
	const uint64_t o0 = offsets[0], npos = offsets[nseq] - o0;
	std::vector<uint8_t> packed(npos*8, 0);
	std::vector<float> insP(npos);
	for (uint64_t r = 0; r < npos; ++r)
		{
		const uint8_t *col = letters + (o0 + r)*nfeat;
		float score = 0;
		for (uint32_t f = 0; f < nfeat; ++f)
			{
			if (col[f] >= alpha[f])
				return mb_fail(ctx, MB200_EINVAL, "profile position %llu: letter %u of feature %u outside its alphabet",
				  (unsigned long long) r, col[f], f);
			packed[r*8 + f] = col[f];
			const float term = logprobs[lbase[f] + col[f]]*weights[f];        // mega.cpp:283
			score += term;
			}
		insP[r] = score;
		}
	std::vector<float> T(tsize);
	for (uint32_t f = 0; f < nfeat; ++f)
		for (uint32_t k = 0; k < alpha[f]*alpha[f]; ++k)
			T[base[f] + k] = logprobmx[base[f] + k]*weights[f];                 // mega.cpp:355-356
	ctx->mega_nf = nfeat;
	ctx->mega_tsize = tsize;
	for (uint32_t f = 0; f < 8; ++f)
		{
		ctx->mega_base[f] = f < nfeat ? base[f] : 0;
		ctx->mega_alpha[f] = f < nfeat ? alpha[f] : 0;
		}
	ctx->h_bytes.clear();
	rc = install_seqs(ctx, nseq, offsets, true);
	if (rc != MB200_OK)
		return rc;
	ENSURE(ctx->d_codes, packed.size() + 16);
	ENSURE(ctx->d_insP, insP.size()*sizeof(float) + 16);
	ENSURE(ctx->d_megaT, T.size()*sizeof(float) + 16);
	cudaStream_t st = ctx->stream;
	CU(cudaMemcpyAsync(ctx->d_codes.p, packed.data(), packed.size(), cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(ctx->d_insP.p, insP.data(), insP.size()*sizeof(float), cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(ctx->d_megaT.p, T.data(), T.size()*sizeof(float), cudaMemcpyHostToDevice, st));
	CU(cudaStreamSynchronize(st));
	ctx->stats.h2d_bytes += packed.size() + insP.size()*4 + T.size()*4;
	return MB200_OK;
	}

// ------------------------------------------------------------------------------------------
// posterior stage
// A work unit of k_posterior_sm is a chain of pairs that share Y; the warp's wavefront fills and
// drains once per chain.  kChainRows bounds a chain's Forward rows (sum of LX+2) and so the per-warp
// Forward-M spill and candidate rows: at 1280 the C3 workload (1000 proteins of ~350 residues) runs
// chains of about 3.5 pairs and its scratch stays a small part of one 80 GB device.
static const uint64_t kChainRows = 1280;
// The plan of the installed pair list (PostPlan, engine.h): the column-width bins and, inside each, the
// chains in longest-first work order.  Cached across calls with the same pair list so that a repeated
// mb200_posteriors_allpairs() moves no host data.
static int build_plan(mb200_ctx *ctx, int force_c, int R)
	{
	const uint32_t np = (uint32_t) ctx->h_px.size();
	PostPlan &plan = ctx->plan;
	plan = PostPlan{};
	// reference overflow guard (fwdflat3.cpp:17-18); bin pairs by C = columns per lane
	std::vector<std::vector<uint32_t>> bins(MB_MAX_C + 1);
	for (uint32_t k = 0; k < np; ++k)
		{
		const uint32_t LX = ctx->h_len[ctx->h_px[k]], LY = ctx->h_len[ctx->h_py[k]];
		if ((double) LX*LY*5 + 100 > 2147483647.0)
			return mb_fail(ctx, MB200_EOVERFLOW, "HMM overflow, sequence lengths %u, %u (max ~21k)", LX, LY);
		plan.cells += (uint64_t) LX*LY;
		plan.est_entries += (uint64_t) LX*ctx->nnz_per_row_cap;
		int C = force_c > 0 ? force_c : (int) std::min<uint32_t>(MB_MAX_C, (LY + 31)/32);
		if (force_c <= 0)
			C = mb_post_sm_class(C);          // bins only size the shared-memory state
		bins[C].push_back(k);
		}
	// inside a bin, pairs with the same Y form chains (store order, at most kChainRows Forward rows and
	// MB_CHAIN_MAX pairs; pairs that need more than one strip stay alone); most cells first
	std::vector<uint32_t> order, chain;
	order.reserve(np);
	std::vector<int> open(ctx->nseq, -1);
	for (int C = 1; C <= MB_MAX_C; ++C)
		{
		PostClass &pc = plan.cls[C];
		std::vector<std::vector<uint32_t>> chains;
		std::vector<uint64_t> frows, fsteps, cost;
		for (uint32_t k : bins[C])
			{
			const uint32_t x = ctx->h_px[k], y = ctx->h_py[k];
			const uint32_t LX = ctx->h_len[x], LY = ctx->h_len[y];
			int &c = open[y];
			if (c < 0 || LY > 32u*C || frows[c] + LX + 2 > kChainRows || chains[c].size() == MB_CHAIN_MAX)
				{
				c = (int) chains.size();
				chains.emplace_back();
				frows.push_back(0);
				fsteps.push_back(0);
				cost.push_back(0);
				}
			chains[c].push_back(k);
			frows[c] += LX + 2;
			fsteps[c] += mb_fwd_steps(LX, R);
			cost[c] += (uint64_t) LX*LY;
			pc.lxmax = std::max(pc.lxmax, LX);
			pc.lymax = std::max(pc.lymax, LY);
			pc.fsteps = std::max<uint64_t>(pc.fsteps, fsteps[c]);
			pc.rows = std::max<uint64_t>(pc.rows, frows[c] - 2*chains[c].size());
			}
		for (uint32_t k : bins[C])
			open[ctx->h_py[k]] = -1;
		std::vector<uint32_t> idx(chains.size());
		std::iota(idx.begin(), idx.end(), 0u);
		std::stable_sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return cost[a] > cost[b]; });
		pc.chain0 = (uint32_t) chain.size();
		pc.nchains = (uint32_t) chains.size();
		for (uint32_t c : idx)
			{
			chain.push_back((uint32_t) order.size());
			order.insert(order.end(), chains[c].begin(), chains[c].end());
			}
		}
	chain.push_back((uint32_t) order.size());
	cudaStream_t st = ctx->stream;
	ENSURE(ctx->d_chain, chain.size()*sizeof(uint32_t));
	ENSURE(ctx->d_order, np*sizeof(uint32_t));
	CU(cudaMemcpyAsync(ctx->d_chain.p, chain.data(), chain.size()*sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(ctx->d_order.p, order.data(), np*sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	CU(cudaStreamSynchronize(st));     // host vectors above go out of scope
	ctx->stats.h2d_bytes += chain.size()*sizeof(uint32_t) + np*sizeof(uint32_t);
	plan.valid = true;
	plan.force_c = force_c;
	plan.R = R;
	return MB200_OK;
	}

// one launch of k_posterior_sm: the size class's instantiation, its dynamic shared memory and grid
struct ClassLaunch { const void *kern; size_t smem; uint32_t nblocks; PostParams P; };

// The launch of size class C with an entry pool of ent_cap entries.  Its per-warp scratch is one buffer
// whose warp count shrinks to fit 80 % of the free memory; free_b is that free memory, 0 = not known
// (it is asked for, and reset when a scratch buffer is (re)allocated).
static int class_launch(mb200_ctx *ctx, int C, const PostDebug *dbg, uint64_t ent_cap, size_t &free_b, ClassLaunch &L)
	{
	const PostClass &pc = ctx->plan.cls[C];
	const bool mega = ctx->mega;
	const bool dump = dbg != nullptr;
	const int CM = mb_post_sm_class(C);      // == C unless the width is forced
	L.kern = mb_post_sm_kernel(mega, dump, CM);
	if (!L.kern)
		return mb_fail(ctx, MB200_EINVAL, "k_posterior_sm has no instantiation for size class %d", CM);
	// floats of the emission table in shared memory (plain mode: {match, ins} pairs, see k_posterior_sm)
	const int tsize = mega ? (int) ctx->mega_tsize : 2*ctx->hmm.K*ctx->hmm.KS;
	L.smem = sizeof(PostSmemHdr) + (size_t)((tsize + 3) & ~3)*sizeof(float)
	  + (size_t) MB_WARPS_PER_BLOCK*(mega ? MB_SM_ARRAYS_MEGA : MB_SM_ARRAYS)*CM*32*sizeof(float);
	CU(cudaFuncSetAttribute(L.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) L.smem));
	if (ctx->occ_cache_k != tsize*2 + (mega ? 1 : 0))
		{
		memset(ctx->occ_cache, 0, sizeof ctx->occ_cache);
		ctx->occ_cache_k = tsize*2 + (mega ? 1 : 0);
		}
	int occ = 0;
	if (dump)          // another instantiation: not cached
		CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, L.kern, 32*MB_WARPS_PER_BLOCK, L.smem));
	else
		{
		if (ctx->occ_cache[C] == 0)
			{
			CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, L.kern, 32*MB_WARPS_PER_BLOCK, L.smem));
			ctx->occ_cache[C] = occ;
			}
		occ = ctx->occ_cache[C];
		}
	if (occ <= 0)
		return mb_fail(ctx, MB200_ECUDA, "k_posterior_sm (CM=%d) cannot be resident (smem %zu)", CM, L.smem);
	const uint32_t need_blocks = (pc.nchains + MB_WARPS_PER_BLOCK - 1)/MB_WARPS_PER_BLOCK;
	const uint32_t nblocks = std::max(1u, std::min((uint32_t) occ*ctx->prop.multiProcessorCount, need_blocks));
	const size_t nwarps = (size_t) nblocks*MB_WARPS_PER_BLOCK;
	// scratch geometry; shrink the resident warp count if the Forward-M spill would not fit
	PostParams &P = L.P;
	memset(&P, 0, sizeof P);
	P.lxmax = pc.lxmax;
	// Forward-M spill, R rows of W columns per step: a strip slot of fm_rows steps per strip of a
	// single pair, or the steps of a chain (at most its Forward steps + 30), which always has one strip
	const int R = ctx->plan.R;
	const uint32_t W = 32u*C;
	const uint32_t nstrips = (pc.lymax + W - 1)/W;
	P.fm_rows = mb_fwd_steps(pc.lxmax, R) + 31;
	P.fm_stride = std::max<size_t>((size_t) nstrips*P.fm_rows, pc.fsteps + 31)*R*W;
	P.edge_stride = 2*((size_t) pc.lxmax + 2);
	P.rows_stride = (size_t) pc.rows*MB_CAP;
	P.rowcnt_stride = ((size_t) pc.rows + 31)/16*16;
	// bytes per warp of the arrays fm, edge, rows, rowcnt and chainbuf
	const size_t bytes[5] = { P.fm_stride*4, P.edge_stride*16, P.rows_stride*8, P.rowcnt_stride,
	  (size_t) MB_CHAIN_BUF*4 };
	const size_t per_warp = bytes[0] + bytes[1] + bytes[2] + bytes[3] + bytes[4];
	size_t total_b = 0;
	if (free_b == 0)
		cudaMemGetInfo(&free_b, &total_b);
	DevBuf &scratch = ctx->d_post_scratch[C];
	const size_t held = scratch.cap;
	const size_t have = free_b + held;
	size_t use_warps = nwarps;
	if (per_warp*use_warps > have*8/10)
		use_warps = std::max<size_t>(MB_WARPS_PER_BLOCK, (have*8/10/per_warp)/MB_WARPS_PER_BLOCK*MB_WARPS_PER_BLOCK);
	L.nblocks = (uint32_t)(use_warps/MB_WARPS_PER_BLOCK);
	// one buffer holds the five arrays of all warps, each starting on a 256-byte boundary
	size_t off[6] = {};
	for (int a = 0; a < 5; ++a)
		off[a + 1] = off[a] + (bytes[a]*use_warps + 255)/256*256;
	ENSURE(scratch, off[5]);
	if (scratch.cap != held)
		free_b = 0;                        // it was (re)allocated: ask again for the next size class
	P.h = ctx->hmm;
	P.matchT = (const float *)(mega ? ctx->d_megaT.p : ctx->d_matchT.p);
	P.insT = (const float *)(mega ? ctx->d_insP.p : ctx->d_insT.p);
	P.mega_nf = ctx->mega_nf; P.mega_tsize = ctx->mega_tsize;
	memcpy(P.mega_base, ctx->mega_base, sizeof P.mega_base);
	memcpy(P.mega_alpha, ctx->mega_alpha, sizeof P.mega_alpha);
	P.codes = (const uint8_t *) ctx->d_codes.p;
	P.seqoff = (const uint64_t *) ctx->d_seqoff.p;
	P.seqlen = (const uint32_t *) ctx->d_seqlen.p;
	P.px = (const uint32_t *) ctx->d_px.p;
	P.py = (const uint32_t *) ctx->d_py.p;
	P.order = (const uint32_t *) ctx->d_order.p;
	P.chain = (const uint32_t *) ctx->d_chain.p + pc.chain0;
	P.nwork = pc.nchains;
	P.counter = (uint32_t *)((char *) ctx->d_cursor.p + 16) + C;
	P.fm = (float *)((char *) scratch.p + off[0]);
	P.edge = (float4 *)((char *) scratch.p + off[1]);
	P.rows = (mb200_entry *)((char *) scratch.p + off[2]);
	P.rowcnt = (uint8_t *)((char *) scratch.p + off[3]);
	P.chainbuf = (uint32_t *)((char *) scratch.p + off[4]);
	P.rowoff = (uint32_t *) ctx->d_rowoff.p;
	P.rowbase = (const uint64_t *) ctx->d_rowbase.p;
	P.entries = (mb200_entry *) ctx->d_entries.p;
	P.ent_cap = ent_cap;
	P.ent_cursor = (unsigned long long *) ctx->d_cursor.p;
	P.entbase = (uint64_t *) ctx->d_entbase.p;
	P.nnz = (uint32_t *) ctx->d_nnz.p;
	P.ea = (float *) ctx->d_ea.p;
	P.err = (int *)((char *) ctx->d_cursor.p + 8);
	if (dbg)
		{
		P.dbg_fwd = dbg->fwd; P.dbg_bwd = dbg->bwd; P.dbg_post = dbg->post; P.dbg_total = dbg->total;
		P.dbg_pair = dbg->pair;
		}
	P.cmax = (uint32_t) C;
	return MB200_OK;
	}

// The posterior stage over the installed pair list (mb_store_set_pairs)
static int run_posteriors(mb200_ctx *ctx, float *ea_out, const PostDebug *dbg, int force_c)
	{
	const uint32_t np = (uint32_t) ctx->h_px.size();
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	CU(cudaEventRecord(ctx->ev0, st));
	const PostPlan &plan = ctx->plan;
	if (!plan.valid || plan.force_c != force_c)
		{
		const int rc = build_plan(ctx, force_c, mb_post_rows(ctx->mega));
		if (rc != MB200_OK)
			return rc;
		}
	// one control block = { entry cursor u64, error flag i32, pad, work cursors u32[MB_MAX_C+1] }:
	// a single memset per attempt and a single 16-byte read-back
	const size_t cursor_bytes = 16 + (MB_MAX_C + 1)*sizeof(uint32_t);
	ENSURE(ctx->d_cursor, cursor_bytes);
	ctx->stats.cells = plan.cells;
	uint64_t est_entries = std::max(plan.est_entries, ctx->last_used_entries);

	bool done = false;
	for (int attempt = 0; attempt < 3; ++attempt)
		{
		ENSURE(ctx->d_entries, (est_entries + 64)*sizeof(mb200_entry));
		CU(cudaMemsetAsync(ctx->d_cursor.p, 0, cursor_bytes, st));
		CU(cudaEventRecord(ctx->ev1, st));
		for (int k = 0; k < mb200_ctx::kStreams; ++k)
			CU(cudaStreamWaitEvent(ctx->aux[k], ctx->ev1, 0));
		// widest bins first: they hold most of the work, the narrow ones fill the tails
		int nlaunched = 0;
		size_t free_b = 0;
		for (int C = MB_MAX_C; C >= 1; --C)
			{
			if (plan.cls[C].nchains == 0)
				continue;
			ClassLaunch L;
			const int rc = class_launch(ctx, C, dbg, est_entries, free_b, L);
			if (rc != MB200_OK)
				return rc;
			void *args[] = { &L.P };
			CU(cudaLaunchKernel(L.kern, dim3(L.nblocks), dim3(32*MB_WARPS_PER_BLOCK), args, L.smem,
			  ctx->aux[nlaunched++ % mb200_ctx::kStreams]));
			ctx->stats.kernel_launches++;
			}
		for (int k = 0; k < mb200_ctx::kStreams; ++k)
			{
			CU(cudaEventRecord(ctx->aux_done[k], ctx->aux[k]));
			CU(cudaStreamWaitEvent(st, ctx->aux_done[k], 0));
			}
		CU(cudaEventRecord(ctx->ev2, st));
		CU(cudaMemcpyAsync(ctx->h_pinned, ctx->d_cursor.p, 16, cudaMemcpyDeviceToHost, st));
		CU(cudaStreamSynchronize(st));
		unsigned long long used = 0;
		memcpy(&used, ctx->h_pinned, sizeof used);
		const int err = (int) ctx->h_pinned[2];
		ctx->stats.d2h_bytes += 16;
		ctx->store_nnz = used;
		if (err == MB200_ENOMEM && used > est_entries)
			{
			est_entries = used + used/16;     // the cursor counted everything: retry with the exact need
			ctx->last_used_entries = est_entries;
			continue;
			}
		if (err == MB200_EOVERFLOW)
			return mb_fail(ctx, MB200_EOVERFLOW, "a posterior row produced more than %d candidate entries", MB_CAP);
		if (err != 0)
			return mb_fail(ctx, err, "device error flag %d in k_posterior", err);
		done = true;
		break;
		}
	if (!done)
		return mb_fail(ctx, MB200_ENOMEM, "posterior entry pool still too small after re-sizing (%llu entries)",
		  (unsigned long long) est_entries);
	if (ea_out)
		{
		CU(cudaMemcpyAsync(ea_out, ctx->d_ea.p, np*sizeof(float), cudaMemcpyDeviceToHost, st));
		ctx->stats.d2h_bytes += np*sizeof(float);
		}
	CU(cudaEventRecord(ctx->ev3, st));
	CU(cudaStreamSynchronize(st));
	cudaEventElapsedTime(&ctx->stats.last_kernel_ms, ctx->ev1, ctx->ev2);
	cudaEventElapsedTime(&ctx->stats.last_total_ms, ctx->ev0, ctx->ev3);
	mb_store_fresh(ctx, false);
	return MB200_OK;
	}

// the new pair list of a posterior call, once there are tables and sequences
static int install_pairs(mb200_ctx *ctx, StorePairs pairs, uint32_t lo, uint32_t hi, const uint32_t *px, const uint32_t *py)
	{
	if (!ctx->have_hmm || ctx->nseq == 0)
		return mb_fail(ctx, MB200_EINVAL, "mb200_posteriors: call mb200_set_hmm and mb200_set_seqs first");
	cudaSetDevice(ctx->device);
	return mb_store_set_pairs(ctx, pairs, lo, hi, px, py);
	}

int mb200_posteriors(mb200_ctx *ctx, uint32_t npairs, const uint32_t *pair_x, const uint32_t *pair_y,
  uint32_t flags, float *ea_out)
	{
	if (!ctx || npairs == 0 || !pair_x || !pair_y)
		return mb_fail(ctx, MB200_EINVAL, "mb200_posteriors: bad argument");
	const int rc = install_pairs(ctx, PAIRS_LIST, 0, npairs, pair_x, pair_y);
	if (rc != MB200_OK)
		return rc;
	const int force_c = (int)((flags >> 8) & 0xff);
	if (force_c > MB_MAX_C)
		return mb_fail(ctx, MB200_EINVAL, "forced C %d > %d", force_c, MB_MAX_C);
	return run_posteriors(ctx, ea_out, nullptr, force_c);
	}

int mb200_posteriors_allpairs(mb200_ctx *ctx, uint32_t p_lo, uint32_t p_hi, float *ea_out)
	{
	if (!ctx || ctx->nseq < 2)
		return mb_fail(ctx, MB200_EINVAL, "mb200_posteriors_allpairs: need >= 2 sequences");
	const uint64_t npairs = (uint64_t) ctx->nseq*(ctx->nseq - 1)/2;
	if (p_lo >= p_hi || p_hi > npairs)
		return mb_fail(ctx, MB200_EINVAL, "pair range [%u,%u) invalid for %llu pairs", p_lo, p_hi,
		  (unsigned long long) npairs);
	const StoreState &s = ctx->store;
	int rc = MB200_OK;
	if (!(ctx->plan.valid && s.pairs == PAIRS_RANGE && s.p_lo == p_lo && s.p_hi == p_hi)
	  && (rc = install_pairs(ctx, PAIRS_RANGE, p_lo, p_hi, nullptr, nullptr)) != MB200_OK)
		return rc;
	mb_store_drop(ctx);
	return run_posteriors(ctx, ea_out, nullptr, 0);
	}

int mb200_calc_post_dense_pair(mb200_ctx *ctx, uint32_t npairs, const uint32_t *pair_x, const uint32_t *pair_y,
  uint32_t which, float *post_out, float *fwd_m_out, float *bwd_m_out, float *total_out)
	{
	if (!ctx || !post_out || !pair_x || !pair_y || which >= npairs || pair_x[which] >= ctx->nseq
	  || pair_y[which] >= ctx->nseq)
		return mb_fail(ctx, MB200_EINVAL, "mb200_calc_post_dense_pair: bad argument");
	cudaSetDevice(ctx->device);
	const size_t n = (size_t) ctx->h_len[pair_x[which]]*ctx->h_len[pair_y[which]];
	ENSURE(ctx->d_dbg, (3*n + 4)*sizeof(float));
	float *base = (float *) ctx->d_dbg.p;
	PostDebug dbg = { base, base + n, base + 2*n, base + 3*n, which };
	int rc = install_pairs(ctx, PAIRS_LIST, 0, npairs, pair_x, pair_y);
	if (rc == MB200_OK)
		rc = run_posteriors(ctx, nullptr, &dbg, ctx->debug_force_c);
	if (rc != MB200_OK)
		return rc;
	CU(cudaMemcpy(post_out, dbg.post, n*sizeof(float), cudaMemcpyDeviceToHost));
	if (fwd_m_out)
		CU(cudaMemcpy(fwd_m_out, dbg.fwd, n*sizeof(float), cudaMemcpyDeviceToHost));
	if (bwd_m_out)
		CU(cudaMemcpy(bwd_m_out, dbg.bwd, n*sizeof(float), cudaMemcpyDeviceToHost));
	if (total_out)
		CU(cudaMemcpy(total_out, dbg.total, sizeof(float), cudaMemcpyDeviceToHost));
	return MB200_OK;
	}

int mb200_calc_post_dense(mb200_ctx *ctx, uint32_t x, uint32_t y, float *post_out, float *fwd_m_out,
  float *bwd_m_out, float *total_out)
	{
	return mb200_calc_post_dense_pair(ctx, 1, &x, &y, 0, post_out, fwd_m_out, bwd_m_out, total_out);
	}

// test hook: the plan of the last posterior call, as the kernel reads it
int mb200_debug_plan(mb200_ctx *ctx, uint32_t *npairs, uint32_t *nchains, uint32_t *order, uint32_t *chain,
  uint32_t *bin_start, uint32_t *limits)
	{
	if (!ctx || !npairs || !nchains)
		return mb_fail(ctx, MB200_EINVAL, "mb200_debug_plan: bad argument");
	const PostPlan &plan = ctx->plan;
	if (!plan.valid)
		return mb_fail(ctx, MB200_EINVAL, "mb200_debug_plan: no plan (run a posterior stage first)");
	cudaSetDevice(ctx->device);
	const uint32_t np = (uint32_t) ctx->h_px.size(), nc = plan.cls[MB_MAX_C].chain0 + plan.cls[MB_MAX_C].nchains;
	*npairs = np;
	*nchains = nc;
	if (order)
		CU(cudaMemcpy(order, ctx->d_order.p, np*sizeof(uint32_t), cudaMemcpyDeviceToHost));
	if (chain)
		CU(cudaMemcpy(chain, ctx->d_chain.p, (nc + 1)*sizeof(uint32_t), cudaMemcpyDeviceToHost));
	if (bin_start)
		{
		for (int C = 0; C <= MB_MAX_C; ++C)
			bin_start[C] = plan.cls[C].chain0;          // first chain of size class C (class 0 is never used: 0)
		bin_start[MB_MAX_C + 1] = nc;
		}
	if (limits)
		{
		limits[0] = (uint32_t) kChainRows;
		limits[1] = MB_CHAIN_MAX;
		}
	return MB200_OK;
	}

// test hook: force the columns-per-lane of mb200_calc_post_dense (0 = automatic)
int mb200_debug_force_c(mb200_ctx *ctx, int c)
	{
	if (!ctx || c < 0 || c > MB_MAX_C)
		return MB200_EINVAL;
	ctx->debug_force_c = c;
	return MB200_OK;
	}

// test hook / tuning: expected sparse entries per posterior row used to size the entry pool
int mb200_set_nnz_per_row_cap(mb200_ctx *ctx, uint32_t cap)
	{
	if (!ctx || cap == 0)
		return MB200_EINVAL;
	ctx->nnz_per_row_cap = cap;
	return MB200_OK;
	}

// ------------------------------------------------------------------------------------------
// store introspection
int mb200_store_npairs(const mb200_ctx *ctx, uint32_t *npairs)
	{
	if (!ctx || !npairs)
		return MB200_EINVAL;
	*npairs = ctx->store.present ? (uint32_t) ctx->h_px.size() : 0;
	return MB200_OK;
	}

int mb200_store_nnz(mb200_ctx *ctx, uint32_t *nnz_out, uint64_t *total_nnz)
	{
	if (!ctx)
		return MB200_EINVAL;
	cudaSetDevice(ctx->device);
	const int rc = mb_store_require(ctx, "mb200_store_nnz", NEED_INDEX);
	if (rc != MB200_OK)
		return rc;
	uint64_t tot = 0;
	for (size_t k = 0; k < ctx->h_nnz.size(); ++k)
		{
		if (nnz_out)
			nnz_out[k] = ctx->h_nnz[k];
		tot += ctx->h_nnz[k];
		}
	if (total_nnz)
		*total_nnz = tot;
	return MB200_OK;
	}

int mb200_export_pair(mb200_ctx *ctx, uint32_t pair, uint32_t *offsets, mb200_entry *entries)
	{
	if (!ctx || !offsets)
		return mb_fail(ctx, MB200_EINVAL, "mb200_export_pair: bad argument");
	cudaSetDevice(ctx->device);
	// the host index is re-read only when the store changed: at C3 it is 6 MB, and callers export
	// pairs one at a time
	int rc = mb_store_require(ctx, "mb200_export_pair", NEED_INDEX);
	if (rc != MB200_OK)
		return rc;
	if (pair >= ctx->h_px.size())
		return mb_fail(ctx, MB200_EINVAL, "pair %u out of range", pair);
	const uint32_t LX = ctx->h_len[ctx->h_px[pair]];
	CU(cudaMemcpy(offsets, (const uint32_t *) ctx->d_rowoff.p + ctx->h_rowbase[pair], (LX + 1)*sizeof(uint32_t),
	  cudaMemcpyDeviceToHost));
	if (entries && ctx->h_nnz[pair] > 0)
		CU(cudaMemcpy(entries, (const mb200_entry *) ctx->d_entries.p + ctx->h_entbase[pair],
		  (size_t) ctx->h_nnz[pair]*sizeof(mb200_entry), cudaMemcpyDeviceToHost));
	return MB200_OK;
	}

} // extern "C"
