// post_kernel_sm.cuh -- k_posterior_sm: the fused Forward -> total -> Backward+posterior -> sparsify
// -> EA kernel.
//
// Replaces, per sequence pair, CalcFwdFlat (fwdflat3.cpp:12-153), CalcTotalProbFlat
// (totalprobflat.cpp:3-16), CalcBwdFlat (bwdflat3.cpp:10-184), CalcPostFlat
// (calcposteriorflat.cpp:4-27), MySparseMx::FromPost (mysparsemx.cpp:115-152) and CalcAlnScoreFlat
// (calcalnscoreflat.cpp:4-32) of the reference.
//
// Mapping.  One warp owns one chain of pairs that share Y at a time (persistent warps pull chains,
// longest first, from an atomic cursor; the wavefront fills and drains once per chain, see Forward
// and Backward below).  Lane l owns C consecutive DP columns of Y (C = ceil(LY/32) capped at the size
// class CM, a compile-time parameter); a warp therefore covers a strip of 32*C columns and longer Y
// are processed strip after strip with the strip-edge column handed over through a small per-warp
// buffer.  Rows of X are swept in anti-diagonal (wavefront) order: at step t lane l works on row t-l,
// the cell to the left lives in lane l-1 and was produced one step earlier, so the recurrence
// dependency is a few warp shuffles per step.  The per-column wavefront state lives in SHARED MEMORY,
// one record per (column, lane) stored [c][lane] (lane-contiguous: conflict free): {S, M, IX, JX} as
// one float4 and {class of Y, insert emission of Y} as one 64-bit word, so that a column costs one
// 128-bit load and store of state, one 64-bit load of its Y data and pointers that move by constants.
// The loop over the lane's columns is rolled: the hot loops are short and stay in the instruction
// cache (a register-resident, fully unrolled variant stalls on instruction fetch).  Only the
// Forward M-state is spilled (4 B/cell), in [step][c][lane] order so that both the Forward write
// and the Backward read are full 128-byte lines.  Backward walks the same anti-diagonals in
// reverse, fuses the Fwd (*) Bwd posterior score, thresholds it at log(0.01) and appends the scores of
// survivors to a per-row candidate list; the warp then turns the scores into probabilities 32 at a time,
// compacts the rows into MySparseMx order and runs the expected-accuracy max-sum DP from the candidates
// through a prefix-max tree over the columns (see mb_compact_ea for why that is exactly the reference's
// max3 recurrence).
//
// Border handling without special code paths: LOG_ZERO is absorbing under the branch-free LogAdd,
// so the reference's border formulas (first row/column of Forward, fwdflat3.cpp:35-93; last
// row/column of Backward, bwdflat3.cpp:132-176) fall out of the general cell update when the
// out-of-range neighbours are LOG_ZERO.  The only injected values are the start scores at Forward
// (0,0) and the end scores at Backward (LX,LY) (bwdflat3.cpp:53-61).  Columns past LY (the tail of
// the lane that holds column LY in the last strip) are never computed: Forward never flows back from
// them, and in Backward they would stay exactly LOG_ZERO, the value they are initialised to.  So the
// cell (LX,LY) is the last cell of its lane's row in Forward (read out after the loop) and the first
// in Backward (set before the loop), and the hot loops carry no test for either.
//
// Emissions.  Plain mode: residue classes index a K x K match table and a K-entry insert table
// (PairHMM::m_MatchScore / m_InsScore, pairhmm.h:26-29).  MEGA mode (Muscle-3D feature profiles,
// Mega::CalcFwdFlat_mega / CalcBwdFlat_mega, fwdflat_mega.cpp:14, bwdflat_mega.cpp): a position is a
// vector of <= 8 feature letters; the match emission of a cell is the sum over features of
// LogProbMx_f[a_f][b_f]*w_f accumulated from 0 in feature order (Mega::GetMatchScore,
// mega.cpp:340-359) -- the products are formed once on the host (same fp32 multiply), the kernel adds
// them in order -- and the insert emission is a per-position value precomputed the same way
// (Mega::GetInsScore, mega.cpp:273-286).  Same recurrences, same kernel, one template flag.
//
// DUMP: the instantiation used by mb200_calc_post_dense_pair runs the whole pair list with the same
// chains and also writes the dense Forward-M, Backward-M, posterior and total of store pair
// P.dbg_pair, wherever it sits in its chain; production launches carry no dump code.
#pragma once
#include "common.cuh"

// resident CTAs/SM the plain-mode register budget is tuned for (64K registers: <= 102 per thread at 5,
// 128 at 4).  The row-pair passes need about 96 registers; at 5 words per (column, lane) five CTAs of the
// classes up to 14 fit in an SM's shared memory, and four of class 16, which therefore gets 128.
#define MB_SM_BLOCKS 5

// sum over features of the pre-multiplied pair tables, in feature order starting from 0
// (mega.cpp:350-357); xb[f] = offset of row a_f of feature f's table, y0/y1 = packed letters of the column
__device__ __forceinline__ float mb_mega_emit(const float *T, const uint32_t (&xb)[8], uint32_t y0, uint32_t y1, int nf)
	{
	float e = ADD(0.0f, T[xb[0] + (y0 & 255u)]);
	if (nf > 1) e = ADD(e, T[xb[1] + ((y0 >> 8) & 255u)]);
	if (nf > 2) e = ADD(e, T[xb[2] + ((y0 >> 16) & 255u)]);
	if (nf > 3) e = ADD(e, T[xb[3] + (y0 >> 24)]);
	if (nf > 4) e = ADD(e, T[xb[4] + (y1 & 255u)]);
	if (nf > 5) e = ADD(e, T[xb[5] + ((y1 >> 8) & 255u)]);
	if (nf > 6) e = ADD(e, T[xb[6] + ((y1 >> 16) & 255u)]);
	if (nf > 7) e = ADD(e, T[xb[7] + (y1 >> 24)]);
	return e;
	}


// a sequence as the kernel reads it: residue classes (plain), or 8 letter bytes and the insert emission
// of every position (MEGA)
struct MbSeq
	{
	int len;
	const uint8_t *code;
	const uint2 *letters;
	const float *ins;
	};

__device__ __forceinline__ MbSeq mb_seq(const PostParams &P, uint32_t s)
	{
	const uint64_t o = P.seqoff[s];
	return { (int) P.seqlen[s], P.codes + o, reinterpret_cast<const uint2 *>(P.codes) + o, P.insT + o };
	}

// MEGA mode: position i of X as a row of the DP needs it (letters and insert emission); zeros when !in.
// Loaded one step ahead of its use.
struct MbXRow { uint2 letters; float ins; };

__device__ __forceinline__ MbXRow mb_x_row(const MbSeq &X, bool in, int i)
	{
	MbXRow r;
	r.letters = in ? X.letters[i] : make_uint2(0u, 0u);
	r.ins = in ? X.ins[i] : 0.0f;
	return r;
	}

// MEGA mode: X's side of the emissions of a row: its insert emission, and xb of mb_mega_emit for its letters
struct MbXEmit { float ins; uint32_t xb[8]; };

__device__ __forceinline__ MbXEmit mb_x_emit(const PostParams &P, const MbXRow &x)
	{
	MbXEmit e;
	e.ins = x.ins;
#pragma unroll
	for (int f = 0; f < 8; ++f)
		e.xb[f] = P.mega_base[f]
		  + ((f < 4 ? (x.letters.x >> (8*f)) : (x.letters.y >> (8*(f - 4)))) & 255u)*P.mega_alpha[f];
	return e;
	}

// MEGA mode: {match emission, insert emission of Y} of a column whose staged Y data is at yp / y2p, in a
// row with X's side xe
__device__ __forceinline__ float2 mb_col_emit(const float *matchT, const MbXEmit &xe, int nf, const uint2 *yp,
  const uint32_t *y2p)
	{
	const uint2 y = *yp;
	return make_float2(mb_mega_emit(matchT, xe.xb, y.x, *y2p, nf), __uint_as_float(y.y));
	}

// the values of a Forward cell (fwdflat3.cpp:110-140) and s, the LOG_ADD of its five states with their
// transitions to M, which the cell down-right takes as its diagonal.  diag: s of the cell up-left; uM,
// uIX, uJX: the cell above; lm: M of the cell to the left, laiy / lajy: its IY / JY plus tII / tJJ
struct MbFwdCell { float s, m, ix, jx, iy, jy; };

__device__ __forceinline__ MbFwdCell mb_fwd_cell(const MbHmm &h, const LogAdd &la, float diag, float em, float uM,
  float uIX, float uJX, float laiy, float lajy, float lm, float ex, float eyc)
	{
	MbFwdCell r;
	r.m = ADD(diag, em);
	r.ix = ADD(la(ADD(uIX, h.tII), ADD(uM, h.tMI)), ex);
	r.jx = ADD(la(ADD(uJX, h.tJJ), ADD(uM, h.tMJ)), ex);
	r.iy = ADD(la(laiy, ADD(lm, h.tMI)), eyc);
	r.jy = ADD(la(lajy, ADD(lm, h.tMJ)), eyc);
	r.s = la(ADD(r.m, h.tMM), la(ADD(r.ix, h.tIM), la(ADD(r.jx, h.tJM),
	  la(ADD(r.iy, h.tIM), ADD(r.jy, h.tJM)))));
	return r;
	}

// the five values of a Backward cell (bwdflat3.cpp:95-125) from the row below ({M, IX, JX} of this column
// and M of the next one) and the IY / JY of the cell to the right
struct MbBwdCell { float m, ix, jx, iy, jy; };

__device__ __forceinline__ MbBwdCell mb_bwd_cell(const MbHmm &h, const LogAdd &la, float mdiag, float vIX, float vJX,
  float riy, float rjy, float em, float eyc, float ex)
	{
	const float nM = ADD(mdiag, em);
	const float nIX = ADD(vIX, ex);
	const float nJX = ADD(vJX, ex);
	const float nIY = ADD(riy, eyc);
	const float nJY = ADD(rjy, eyc);
	MbBwdCell r;
	r.m = la(ADD(h.tMM, nM), la(ADD(h.tMI, nIX), la(ADD(h.tMJ, nJX),
	  la(ADD(h.tMI, nIY), ADD(h.tMJ, nJY)))));
	r.ix = la(ADD(h.tII, nIX), ADD(h.tIM, nM));
	r.jx = la(ADD(h.tJJ, nJX), ADD(h.tJM, nM));
	r.iy = la(ADD(h.tII, nIY), ADD(h.tIM, nM));
	r.jy = la(ADD(h.tJJ, nJY), ADD(h.tJM, nM));
	return r;
	}

// posterior score of cell (i, col) (calcposteriorflat.cpp:14-22) from its Forward and Backward M; when
// dump, the cell's Backward M and probability go to the dense dump (row 0 is not a cell of it)
__device__ __forceinline__ float mb_post_score(const PostParams &P, bool dump, int i, int LY, int col, float fmv,
  float m, float total)
	{
	const float score = __fsub_rn(ADD(fmv, m), total);
	if (dump && i >= 1)
		{
		P.dbg_bwd[(size_t)(i - 1)*LY + col] = m;
		P.dbg_post[(size_t)(i - 1)*LY + col] = score < P.h.minScore ? 0.0f : mb_post_prob(score);
		}
	return score;
	}

// one strip of a chain: j0, the position in Y of its first column; nl, the lanes that hold columns of it;
// cn, the lane's columns up to LY
struct MbStrip { int j0, nl, cn; bool last; };

// a chain's Y cut into n strips of W = 32*C columns, lane l holding local columns l*C .. l*C+C-1 of each;
// DP column LY is local column clast of lane lcl in the last strip
struct MbStrips
	{
	int C, W, n, lcl, clast;
	__device__ __forceinline__ MbStrip at(int s, int lane) const
		{
		const bool last = s == n - 1;
		return { s*W, last ? lcl + 1 : 32, (last && lane == lcl) ? clast + 1 : C, last };
		}
	};

__device__ __forceinline__ MbStrips mb_strips(int LY, int C)
	{
	const int W = 32*C, n = (LY + W - 1)/W;
	const int q = LY - 1 - (n - 1)*W;
	return { C, W, n, q/C, q - q/C*C };
	}

// strip s's edge buffers: strips alternate between the two halves
struct MbEdges { const float4 *in; float4 *out; };

__device__ __forceinline__ MbEdges mb_strip_edges(float4 *edge0, float4 *edge1, int s)
	{
	return { (s & 1) ? edge0 : edge1, (s & 1) ? edge1 : edge0 };
	}

// the lane's C state records to LOG_ZERO: the border a pair starts from
__device__ __forceinline__ void mb_clear_state(float4 *st, int C, int lane)
	{
#pragma unroll 1
	for (int c = 0; c < C; ++c)
		st[c*32 + lane] = make_float4(MB_LOG_ZERO, MB_LOG_ZERO, MB_LOG_ZERO, MB_LOG_ZERO);
	}

// stages Y for the lane's C columns of a strip, from position j of Y on (Backward reads the emissions of
// the column to its right, so it passes j one higher), and clears their state records.  Positions past
// LY get the padding class (plain) or zero letters and emission (MEGA).
template <bool MEGA>
__device__ __forceinline__ void mb_stage_y(const MbSeq &Y, int j, int C, int lane, int pad, float4 *st, uint2 *ye,
  uint32_t *y2)
	{
	for (int c = 0; c < C; ++c, ++j)
		{
		const bool in = j < Y.len;
		if (MEGA)
			{
			const uint2 yl = in ? Y.letters[j] : make_uint2(0u, 0u);
			ye[c*32 + lane] = make_uint2(yl.x, __float_as_uint(in ? Y.ins[j] : 0.0f));
			y2[c*32 + lane] = yl.y;
			}
		else
			y2[c*32 + lane] = in ? (uint32_t) Y.code[j] : (uint32_t) pad;
		}
	mb_clear_state(st, C, lane);
	}

// Compaction and expected accuracy of one pair of a chain, once Backward has left its candidate rows (scores,
// columns descending) at prow / pcnt: the warp turns the scores into probabilities 32 at a time, writes the
// entries >= 0.01 in MySparseMx order with their row offsets, and runs the expected-accuracy max-sum DP of
// CalcAlnScoreFlat (calcalnscoreflat.cpp:4-32).  kept: the lane's kept candidates of the pair.
//
// One strip (g.n == 1): from the candidates alone.  A cell without a candidate has P = 0 and fl(x + 0) = x,
// and rounding is monotone, so fl(max(a, b) + P) = max(fl(a + P), fl(b + P)); the reference's DP therefore
// computes, for each candidate (i, j), V = fl(P + Q) with Q the max of V over the candidates (i' < i, j' < j)
// (0 if none), and returns the max of all V (0 if none): bit for bit the same values, with the one addition
// B = Prevj1 + P it performs.  Q comes from a prefix-max Fenwick tree over the columns in the warp's state
// area (LY + 1 <= 32*CM words), queried by every candidate of row i before any of row i updates it.
// Several strips: a warp-wide prefix-max over every column of the row (new[j] = max_{k<=j} max(old[k],
// old[k-1]+P[k])), strip by strip through the edge buffers eIn / eOut.
template <bool MEGA, int CM>
__device__ void mb_compact_ea(const PostParams &P, uint32_t pair, int LX, int LY, uint32_t kept,
  const mb200_entry *prow, const uint8_t *pcnt, const MbStrips &g, float *wbase, float *eIn, float *eOut)
	{
	static_assert(32*CM + 32 + 2*MB_CAP <= MB_SM_ARRAYS*CM*32, "the EA tree and a row's updates fit the state area");
	const int lane = threadIdx.x & 31;
	const int C = g.C, W = g.W;
	for (int o = 16; o > 0; o >>= 1)
		kept += __shfl_xor_sync(MB_FULL, kept, o);
	unsigned long long base = 0;
	if (lane == 0)
		base = atomicAdd(P.ent_cursor, (unsigned long long) kept);
	base = __shfl_sync(MB_FULL, base, 0);
	const bool fits = (base + kept <= P.ent_cap);
	if (lane == 0)
		{
		if (!fits)
			atomicCAS(P.err, 0, MB200_ENOMEM);
		P.entbase[pair] = base;
		P.nnz[pair] = kept;
		}
	uint32_t *rowoff = P.rowoff + P.rowbase[pair];
	mb200_entry *out = P.entries + base;

	float eaScore = 0.0f;
	uint32_t written = 0;
	if (g.n == 1)
		{
		// node k of the tree (1..LY) holds the max of V over columns k - (k & -k) .. k-1 of the rows done.  The
		// values are >= +0, so their bits order as integers and an integer max on them is a float max.
		// Rows are packed: a pack is the next rows whose candidates add up to at most 32 (C3 rows average ~7),
		// lane k holding row i+k's count and lane l candidate l of the pack, so that the loads, expf and the
		// compaction run once per pack instead of once per row; only the tree's queries and updates go row by
		// row.  A row of more than 32 candidates runs alone, batch by batch, its updates held in pend until
		// all its batches have queried.  The batch code is not shared with the strip path below: that cost the
		// plain CM = 14 / 16 and the MEGA Backward loops 1 and 3 instructions.
		float *tree = wbase;
		uint2 *pend = reinterpret_cast<uint2 *>(wbase + 32*CM + 32);     // a long row's updates: {bits of V, column + 1}
		for (int k = lane; k <= LY; k += 32)
			tree[k] = 0.0f;
		uint32_t vmax = 0;
		__syncwarp();
		for (int i = 1; i <= LX; )
			{
			const uint32_t rc = i + lane <= LX ? pcnt[i - 1 + lane] : 0u;
			uint32_t incl = rc;
#pragma unroll
			for (int o = 1; o < 32; o <<= 1)
				{
				const uint32_t n = __shfl_up_sync(MB_FULL, incl, o);
				if (lane >= o)
					incl += n;
				}
			const uint32_t excl = incl - rc;
			const int m = max(1, __popc(__ballot_sync(MB_FULL, incl <= 32u && i + lane <= LX)));
			const uint32_t cnt0 = __shfl_sync(MB_FULL, rc, 0);
			if (cnt0 > 32u)
				{
				// a row of more than 32 candidates on its own, batch by batch
				const mb200_entry *row = prow + (size_t)(i - 1)*MB_CAP;
				if (lane == 0)
					rowoff[i - 1] = written;
				for (uint32_t e0 = 0; e0 < cnt0; e0 += 32)
					{
					const int idx = (int) cnt0 - 1 - (int)(e0 + lane);
					mb200_entry ent; ent.p = 0.0f; ent.col = 0;
					if (idx >= 0)
						{
						ent = row[idx];             // {score, column}: the probability (calcposteriorflat.cpp:20)
						ent.p = mb_post_prob(ent.p);
						}
					const bool keep = idx >= 0 && ent.p >= 0.01f;          // mysparsemx.cpp:139-141
					const uint32_t b = __ballot_sync(MB_FULL, keep);
					if (keep && fits)
						out[written + __popc(b & ((1u << lane) - 1u))] = ent;
					written += __popc(b);
					if (idx >= 0)
						{
						float q = 0.0f;
						for (uint32_t k = ent.col; k > 0; k &= k - 1)
							q = fmaxf(q, tree[k]);
						const uint32_t v = __float_as_uint(ADD(ent.p, q));
						vmax = max(vmax, v);
						pend[e0 + lane] = make_uint2(v, ent.col + 1);
						}
					}
				__syncwarp();
				for (uint32_t e = lane; e < cnt0; e += 32)
					{
					const uint2 u = pend[e];
					for (uint32_t k = u.y; k <= (uint32_t) LY; k += k & (0u - k))
						atomicMax(reinterpret_cast<int *>(tree) + k, (int) u.x);
					}
				__syncwarp();
				++i;
				continue;
				}
			// the pack's row r of lane l: the number of rows k < m with incl[k] <= l; candidate l - excl[r] of it
			// in ascending column order
			int r = 0;
#pragma unroll
			for (int o = 16; o > 0; o >>= 1)
				{
				const uint32_t t = __shfl_sync(MB_FULL, incl, min(r + o - 1, 31));
				if (r + o <= m && t <= (uint32_t) lane)
					r += o;
				}
			const uint32_t total = __shfl_sync(MB_FULL, incl, m - 1);
			const bool has = (uint32_t) lane < total;
			const uint32_t rcnt = __shfl_sync(MB_FULL, rc, r), rex = __shfl_sync(MB_FULL, excl, r);
			mb200_entry ent; ent.p = 0.0f; ent.col = 0;
			if (has)
				{
				ent = prow[(size_t)(i - 1 + r)*MB_CAP + rcnt - 1 - (lane - rex)];
				ent.p = mb_post_prob(ent.p);
				}
			const bool keep = has && ent.p >= 0.01f;
			const uint32_t b = __ballot_sync(MB_FULL, keep);
			if (keep && fits)
				out[written + __popc(b & ((1u << lane) - 1u))] = ent;
			if (lane < m)
				rowoff[i - 1 + lane] = written + __popc(excl < 32u ? b & ((1u << excl) - 1u) : b);
			written += __popc(b);
			// the tree row by row: a row's queries see the rows before it only
			for (int k = 0; k < m; ++k)
				{
				const bool mine = has && r == k;
				uint32_t v = 0;
				if (mine)
					{
					float q = 0.0f;
					for (uint32_t t = ent.col; t > 0; t &= t - 1)
						q = fmaxf(q, tree[t]);
					v = __float_as_uint(ADD(ent.p, q));
					vmax = max(vmax, v);
					}
				__syncwarp();
				if (mine)
					for (uint32_t t = ent.col + 1; t <= (uint32_t) LY; t += t & (0u - t))
						atomicMax(reinterpret_cast<int *>(tree) + t, (int) v);
				__syncwarp();
				}
			i += m;
			}
		if (lane == 0)
			rowoff[LX] = written;
		eaScore = __uint_as_float(__reduce_max_sync(MB_FULL, vmax));
		}
	else
		{
		// the warp's state area, reused as three plain float arrays of CM*32
		float *old = wbase;                 // [c][lane]
		float *rowbuf = wbase + CM*32;      // column-linear: [lane*C + c]
		float *pre = wbase + 2*CM*32;       // [c][lane]
		for (int strip = 0; strip < g.n; ++strip)
			{
			const auto [j0, nl, cn, last] = g.at(strip, lane);
			for (int c = 0; c < C; ++c)
				{
				old[c*32 + lane] = 0.0f;
				rowbuf[c*32 + lane] = 0.0f;
				}
			__syncwarp();
			for (int i = 1; i <= LX; ++i)
				{
				const uint32_t cnt = pcnt[i - 1];
				const mb200_entry *row = prow + (size_t)(i - 1)*MB_CAP;
				if (strip == 0 && lane == 0)
					rowoff[i - 1] = written;
				for (uint32_t e0 = 0; e0 < cnt; e0 += 32)
					{
					const int idx = (int) cnt - 1 - (int)(e0 + lane);
					mb200_entry ent; ent.p = 0.0f; ent.col = 0;
					if (idx >= 0)
						{
						ent = row[idx];             // {score, column}: the probability (calcposteriorflat.cpp:20)
						ent.p = mb_post_prob(ent.p);
						}
					const int lc = (int) ent.col - j0;
					if (idx >= 0 && lc >= 0 && lc < W)
						rowbuf[lc] = ent.p;
					if (strip == 0)
						{
						const bool keep = idx >= 0 && ent.p >= 0.01f;          // mysparsemx.cpp:139-141
						const uint32_t b = __ballot_sync(MB_FULL, keep);
						if (keep && fits)
							out[written + __popc(b & ((1u << lane) - 1u))] = ent;
						written += __popc(b);
						}
					}
				__syncwarp();
				// calcalnscoreflat.cpp:13-29 as a prefix-max over the row
				float leftOld = 0.0f, incoming = 0.0f;
				if (lane == 0)
					{
					leftOld = strip == 0 ? 0.0f : eIn[i - 1];
					incoming = strip == 0 ? 0.0f : eIn[i];
					}
				else
					leftOld = old[(C - 1)*32 + lane - 1];
				float run = 0.0f, prevOld = leftOld;
				for (int c = 0; c < C; ++c)
					{
					const float o = old[c*32 + lane];
					const float b = ADD(prevOld, rowbuf[lane*C + c]);
					float v = fmaxf(o, b);
					v = c == 0 ? v : fmaxf(v, run);
					run = v;
					pre[c*32 + lane] = v;
					prevOld = o;
					}
				__syncwarp();
				float scan = run;
#pragma unroll
				for (int o = 1; o < 32; o <<= 1)
					{
					const float n = __shfl_up_sync(MB_FULL, scan, o);
					if (lane >= o)
						scan = fmaxf(scan, n);
					}
				float excl = __shfl_up_sync(MB_FULL, scan, 1);
				const float inc0 = __shfl_sync(MB_FULL, incoming, 0);
				excl = lane == 0 ? inc0 : fmaxf(excl, inc0);
				float lastNew = 0.0f;
				for (int c = 0; c < C; ++c)
					{
					lastNew = fmaxf(pre[c*32 + lane], excl);
					old[c*32 + lane] = lastNew;
					}
				if (lane == 31 && !last)
					eOut[i] = lastNew;
				__syncwarp();
				for (uint32_t e0 = 0; e0 < cnt; e0 += 32)
					{
					const int idx = (int) cnt - 1 - (int)(e0 + lane);
					if (idx >= 0)
						{
						const int lc = (int) row[idx].col - j0;
						if (lc >= 0 && lc < W)
							rowbuf[lc] = 0.0f;
						}
					}
				__syncwarp();
				}
			if (strip == 0 && lane == 0)
				rowoff[LX] = written;
			if (lane == 31 && !last)
				eOut[0] = 0.0f;
			if (last)
				{
				// cell (LX,LY), local column g.clast of lane g.lcl.  Which form ptxas compiles best differs by mode:
				// reading g.clast keeps it live through Backward and costs the plain CM = 14 and 16 kernels a
				// register and 2 instructions per Backward column; forming the cell from LY instead costs the
				// MEGA kernels 2 instructions per Backward column.
				const int q = LY - 1 - j0;
				eaScore = MEGA ? old[g.clast*32 + g.lcl] : old[(q % C)*32 + q/C];
				}
			__syncwarp();
			float *tmp = eIn; eIn = eOut; eOut = tmp;
			}
		}
	if (lane == 0)
		P.ea[pair] = __fdiv_rn(eaScore, (float) min(LX, LY));     // calcposteriorflat.cpp:89
	__syncwarp();
	}

// CM: size class (columns per lane the shared memory is sized for; P.cmax <= CM caps C at run time)
template <bool MEGA, int CM, bool DUMP>
__global__ void __launch_bounds__(32*MB_WARPS_PER_BLOCK, (MEGA || CM > 14) ? 4 : MB_SM_BLOCKS)
k_posterior_sm(const PostParams P)
	{
	constexpr int NARR = MEGA ? MB_SM_ARRAYS_MEGA : MB_SM_ARRAYS;
	constexpr int R = mb_post_rows(MEGA);
	extern __shared__ __align__(16) unsigned char smem_raw[];
	PostSmemHdr &sm = *reinterpret_cast<PostSmemHdr *>(smem_raw);
	const MbHmm h = P.h;
	const int lane = threadIdx.x & 31;
	const int wib = threadIdx.x >> 5;
	const int gwarp = blockIdx.x*MB_WARPS_PER_BLOCK + wib;
	// plain mode: {match[x][y], ins[y]} pairs in rows of KS, so that one 64-bit load gives both emissions of
	// a column and the per-column record holds only the class of Y; MEGA: the feature tables
	float *matchT = reinterpret_cast<float *>(smem_raw + sizeof(PostSmemHdr));
	float2 *meT = reinterpret_cast<float2 *>(matchT);
	const int tsize = MEGA ? (int) P.mega_tsize : 2*h.K*h.KS;          // floats
	float *wbase = matchT + ((tsize + 3) & ~3) + (size_t) wib*NARR*CM*32;
	float4   *st = reinterpret_cast<float4 *>(wbase);                  // Forward {S, M, IX, JX}; Backward {M, IX, JX, posterior score}
	uint2    *ye = reinterpret_cast<uint2 *>(wbase + 4*CM*32);         // MEGA only: {letters 0..3, bits of eY}
	uint32_t *y2 = reinterpret_cast<uint32_t *>(wbase + (MEGA ? 6 : 4)*CM*32);   // MEGA: letters 4..7; plain: class of Y

	mb_logadd_fill(sm.coef, &sm.labase);
	if (!MEGA)
		{
		for (int k = threadIdx.x; k < h.K; k += blockDim.x)
			sm.insT[k] = P.insT[k];
		for (int k = threadIdx.x; k < h.K*h.KS; k += blockDim.x)
			{
			const int b = k % h.KS;                   // columns K..KS-1 pad the row and are never read
			meT[k] = make_float2(P.matchT[k], b < h.K ? P.insT[b] : 0.0f);
			}
		}
	else
		for (int k = threadIdx.x; k < tsize; k += blockDim.x)
			matchT[k] = P.matchT[k];
	const int nf = (int) P.mega_nf;
	__syncthreads();

	const LogAdd la = mb_logadd_make(&sm.labase);
	const float Z = MB_LOG_ZERO;

	float       *fm     = P.fm + (size_t) gwarp*P.fm_stride;
	float4      *edge0  = P.edge + (size_t) gwarp*P.edge_stride;
	float4      *edge1  = edge0 + (P.lxmax + 2);
	mb200_entry *rows   = P.rows + (size_t) gwarp*P.rows_stride;
	uint8_t     *rowcnt = P.rowcnt + (size_t) gwarp*P.rowcnt_stride;
	uint32_t    *ckept  = P.chainbuf + (size_t) gwarp*MB_CHAIN_BUF;      // [pair of the chain][lane]
	float       *ctotal = reinterpret_cast<float *>(ckept + MB_CHAIN_MAX*32);   // [pair of the chain]
	float       *cfin   = ctotal + MB_CHAIN_MAX;                               // [pair of the chain][5]: cell (LX,LY)

	for (;;)
		{
		uint32_t w = 0;
		if (lane == 0)
			w = atomicAdd(P.counter, 1u);
		w = __shfl_sync(MB_FULL, w, 0);
		if (w >= P.nwork)
			break;
		// the work unit is a chain: P.order[chain[w] .. chain[w+1]) are pairs with the same Y, in store order
		const uint32_t *cpairs = P.order + P.chain[w];
		const int nch = (int)(P.chain[w + 1] - P.chain[w]);
		const MbSeq Y = mb_seq(P, P.py[cpairs[0]]);
		const int LY = Y.len;
		const int sumLX = __reduce_add_sync(MB_FULL, lane < nch ? P.seqlen[P.px[cpairs[lane]]] : 0u);
		const int sumFS = R == 1 ? 0 : __reduce_add_sync(MB_FULL, lane < nch ? mb_fwd_steps(P.seqlen[P.px[cpairs[lane]]], R) : 0u);
		const int C = min(min(CM, (int) P.cmax), (LY + 31) >> 5);   // columns per lane for this chain
		const MbStrips g = mb_strips(LY, C);               // more than one strip only for a chain of one pair
		const int W = g.W;

		for (int k = 0; k < nch; ++k)
			ckept[k*32 + lane] = 0;

		// ============================ Forward ============================
		// Lane l steps through the chain's pairs one after the other: rows 0..LX of a pair, then one
		// separator step that resets the lane's state records to LOG_ZERO and passes LOG_ZERO on, so
		// that row 0 of the next pair sees exactly the border of a fresh pair.  Pair k starts at chain
		// step Fk + l, Fk = sum over earlier pairs of (LX + 2).  MEGA mode: one row per lane per step.
		if constexpr (MEGA)
			for (int strip = 0; strip < g.n; ++strip)
				{
				const auto [j0, nl, cn, last] = g.at(strip, lane);
				const auto [edgeIn, edgeOut] = mb_strip_edges(edge0, edge1, strip);
				float *fms = fm + (size_t) strip*P.fm_rows*W;

				mb_stage_y<true>(Y, j0 + lane*C, C, lane, h.pad, st, ye, y2);
				float outM = Z, outAIY = Z, outAJY = Z, outS = Z;
				float dprev = Z;
				float bIX = Z, bJX = Z;
				const int nsteps = sumLX + 2*nch - 2 + nl;
				int kp = 0, r0 = lane;                // the lane's pair and the step of its row 0
				MbSeq X = mb_seq(P, P.px[cpairs[0]]);
				MbXRow xPref = mb_x_row(X, false, 0);
				for (int t = 0; t < nsteps; ++t)
					{
					const int i = t - r0;
					const MbXRow x = xPref;
					xPref = mb_x_row(X, i >= 0 && i < X.len, i);
					float Lm = __shfl_up_sync(MB_FULL, outM, 1);
					float Laiy = __shfl_up_sync(MB_FULL, outAIY, 1);
					float Lajy = __shfl_up_sync(MB_FULL, outAJY, 1);
					float Ls = __shfl_up_sync(MB_FULL, outS, 1);
					if (i >= 0 && i <= X.len && lane < nl)
						{
						const MbXEmit xe = mb_x_emit(P, x);
						const float ex = xe.ins;
						if (lane == 0)
							{
							if (strip == 0)
								{
								Lm = Z;
								if (i == 0)
									{
									Laiy = h.tSI; Lajy = h.tSJ; Ls = h.tSM;
									}
								else
									{
									if (i == 1)
										{
										bIX = ADD(h.tSI, ex); bJX = ADD(h.tSJ, ex);
										}
									else
										{
										bIX = ADD(ADD(bIX, h.tII), ex); bJX = ADD(ADD(bJX, h.tJJ), ex);
										}
									Laiy = Z; Lajy = Z;
									Ls = la(ADD(bIX, h.tIM), ADD(bJX, h.tJM));
									}
								}
							else
								{
								const float4 e = edgeIn[i];
								Lm = e.x; Laiy = e.y; Lajy = e.z; Ls = e.w;
								}
							}
						float diag = dprev;
						dprev = Ls;
						float lm = Lm, laiy = Laiy, lajy = Lajy, sLast = Z;
						float ix = Z, jx = Z, iy = Z, jy = Z;
						float4 *sp = st + lane;
						const uint2 *yp = ye + lane;
						const uint32_t *y2p = y2 + lane;
						float *dst = fms + (size_t) t*W + lane;
						const bool dump = DUMP && i >= 1 && cpairs[kp] == P.dbg_pair;
#pragma unroll 1
						for (int c = 0; c < cn; ++c, sp += 32, yp += 32, y2p += 32, dst += 32)
							{
							const float4 v = *sp;                      // {S, M, IX, JX} of row i-1
							const auto [em, eyc] = mb_col_emit(matchT, xe, nf, yp, y2p);
							const MbFwdCell f = mb_fwd_cell(h, la, diag, em, v.y, v.z, v.w, laiy, lajy, lm, ex, eyc);
							ix = f.ix; jx = f.jx; iy = f.iy; jy = f.jy;
							diag = v.x;
							*sp = make_float4(f.s, f.m, f.ix, f.jx);
							lm = f.m;
							laiy = ADD(f.iy, h.tII);
							lajy = ADD(f.jy, h.tJJ);
							sLast = f.s;
							*dst = f.m;
							if (dump)
								P.dbg_fwd[(size_t)(i - 1)*LY + j0 + lane*C + c] = f.m;
							}
						if (last && i == X.len && lane == g.lcl)    // cell (LX,LY) is the lane's last
							{
							float *f = cfin + 5*kp;
							f[0] = lm; f[1] = ix; f[2] = iy; f[3] = jx; f[4] = jy;
							}
						outM = lm; outAIY = laiy; outAJY = lajy; outS = sLast;
						if (lane == 31 && !last)
							edgeOut[i] = make_float4(outM, outAIY, outAJY, outS);
						}
					else if (i == X.len + 1 && lane < nl)        // separator, then the next pair of the chain
						{
						mb_clear_state(st, C, lane);
						outM = Z; outAIY = Z; outAJY = Z; outS = Z;
						dprev = Z;
						if (++kp < nch)
							{
							X = mb_seq(P, P.px[cpairs[kp]]);
							r0 = t + 1;
							}
						else
							r0 = 1 << 30;                 // done: idle for the rest of the strip
						}
					}
				__syncwarp();
				}
		else
			{
			// Plain mode, two rows per lane per step.  Lane l steps through the pair's rows two at a time, row a
			// and row b = a+1: row b takes row a's {S, M, IX, JX} of each column from registers, and only row
			// b's record goes to shared memory.  A pair of even LX starts with row -1, which is all LOG_ZERO
			// (every input is, and LOG_ZERO is absorbing), so the steps hold rows (LX-1, LX), (LX-3, LX-2), ...
			// and Backward pairs its rows on the same Forward steps.  After row LX comes one separator step, as
			// above; pair k starts at chain step Fk + l, Fk = sum over earlier pairs of mb_fwd_steps(LX, 2).
			for (int strip = 0; strip < g.n; ++strip)
				{
				const auto [j0, nl, cn, last] = g.at(strip, lane);
				const auto [edgeIn, edgeOut] = mb_strip_edges(edge0, edge1, strip);
				float2 *fms = reinterpret_cast<float2 *>(fm) + (size_t) strip*P.fm_rows*W;   // [step][c][lane] {row a, row b}

				mb_stage_y<false>(Y, j0 + lane*C, C, lane, h.pad, st, ye, y2);
				float oMa = Z, oIa = Z, oJa = Z, oSa = Z, oMb = Z, oIb = Z, oJb = Z, oSb = Z;
				float dprev = Z;
				float bIX = Z, bJX = Z;
				const int nsteps = sumFS - 2 + nl;
				int kp = 0, r0 = lane;                // the lane's pair and the step of its first rows
				MbSeq X = mb_seq(P, P.px[cpairs[0]]);
				int pad = ~X.len & 1, nq = X.len/2 + 1;   // row -1 or not; the pair's row steps
				auto xcode = [&](int i) { return i >= 1 && i <= X.len ? (int) X.code[i - 1] : h.pad; };
				int xa = h.pad, xb = xcode(1 - pad);     // classes of the next step's rows
				// the left border of row i in lane 0 of strip 0: the start scores at (0,0), the bIX / bJX chain.
				// It stays apart from the MEGA pass's: each form tried for both changed one mode's SASS.
				auto border = [&](int i, float ex, float &Lm, float &Laiy, float &Lajy, float &Ls)
					{
					Lm = Z;
					if (i <= 0)
						{
						Laiy = i == 0 ? h.tSI : Z; Lajy = i == 0 ? h.tSJ : Z; Ls = i == 0 ? h.tSM : Z;
						}
					else
						{
						if (i == 1)
							{
							bIX = ADD(h.tSI, ex); bJX = ADD(h.tSJ, ex);
							}
						else
							{
							bIX = ADD(ADD(bIX, h.tII), ex); bJX = ADD(ADD(bJX, h.tJJ), ex);
							}
						Laiy = Z; Lajy = Z;
						Ls = la(ADD(bIX, h.tIM), ADD(bJX, h.tJM));
						}
					};
				for (int t = 0; t < nsteps; ++t)
					{
					const int q = t - r0;
					const int ia = 2*q - pad;             // rows ia and ia+1 of pair kp
					const int xca = xa, xcb = xb;
					xa = xcode(ia + 2); xb = xcode(ia + 3);
					float Lma = __shfl_up_sync(MB_FULL, oMa, 1);
					float Laiya = __shfl_up_sync(MB_FULL, oIa, 1);
					float Lajya = __shfl_up_sync(MB_FULL, oJa, 1);
					float Lsa = __shfl_up_sync(MB_FULL, oSa, 1);
					float Lmb = __shfl_up_sync(MB_FULL, oMb, 1);
					float Laiyb = __shfl_up_sync(MB_FULL, oIb, 1);
					float Lajyb = __shfl_up_sync(MB_FULL, oJb, 1);
					float Lsb = __shfl_up_sync(MB_FULL, oSb, 1);
					if (q >= 0 && q < nq && lane < nl)
						{
						const float2 *mea = meT + xca*h.KS, *meb = meT + xcb*h.KS;
						const float exa = sm.insT[xca], exb = sm.insT[xcb];
						if (lane == 0)
							{
							if (strip == 0)
								{
								border(ia, exa, Lma, Laiya, Lajya, Lsa);
								border(ia + 1, exb, Lmb, Laiyb, Lajyb, Lsb);
								}
							else
								{
								const float4 ea = edgeIn[ia + 1], eb = edgeIn[ia + 2];    // row i at i+1: row -1 too
								Lma = ea.x; Laiya = ea.y; Lajya = ea.z; Lsa = ea.w;
								Lmb = eb.x; Laiyb = eb.y; Lajyb = eb.z; Lsb = eb.w;
								}
							}
						float diaga = dprev, diagb = Lsa;
						dprev = Lsb;
						float lma = Lma, laiya = Laiya, lajya = Lajya, sLasta = Z;
						float lmb = Lmb, laiyb = Laiyb, lajyb = Lajyb, sLastb = Z;
						float ixb = Z, jxb = Z, iyb = Z, jyb = Z;
						float4 *sp = st + lane;
						const uint32_t *y2p = y2 + lane;
						float2 *dst = fms + (size_t) t*W + lane;
						const bool dump = DUMP && cpairs[kp] == P.dbg_pair;
#pragma unroll 1
						for (int c = 0; c < cn; ++c, sp += 32, y2p += 32, dst += 32)
							{
							const float4 v = *sp;                      // {S, M, IX, JX} of row a-1
							const uint32_t yc = *y2p;
							const float2 ea = mea[yc];                 // {match of row a, insert of Y}
							const float emb = reinterpret_cast<const float *>(meb + yc)[0];
							const MbFwdCell a = mb_fwd_cell(h, la, diaga, ea.x, v.y, v.z, v.w, laiya, lajya, lma, exa, ea.y);
							const MbFwdCell b = mb_fwd_cell(h, la, diagb, emb, a.m, a.ix, a.jx, laiyb, lajyb, lmb, exb, ea.y);
							ixb = b.ix; jxb = b.jx; iyb = b.iy; jyb = b.jy;
							diaga = v.x;
							diagb = a.s;
							*sp = make_float4(b.s, b.m, b.ix, b.jx);
							lma = a.m; laiya = ADD(a.iy, h.tII); lajya = ADD(a.jy, h.tJJ); sLasta = a.s;
							lmb = b.m; laiyb = ADD(b.iy, h.tII); lajyb = ADD(b.jy, h.tJJ); sLastb = b.s;
							*dst = make_float2(a.m, b.m);
							if (dump)
								{
								if (ia >= 1)
									P.dbg_fwd[(size_t)(ia - 1)*LY + j0 + lane*C + c] = a.m;
								if (ia >= 0)
									P.dbg_fwd[(size_t) ia*LY + j0 + lane*C + c] = b.m;
								}
							}
						if (last && ia + 1 == X.len && lane == g.lcl)    // cell (LX,LY): row b, the lane's last
							{
							float *f = cfin + 5*kp;
							f[0] = lmb; f[1] = ixb; f[2] = iyb; f[3] = jxb; f[4] = jyb;
							}
						oMa = lma; oIa = laiya; oJa = lajya; oSa = sLasta;
						oMb = lmb; oIb = laiyb; oJb = lajyb; oSb = sLastb;
						if (lane == 31 && !last)
							{
							edgeOut[ia + 1] = make_float4(oMa, oIa, oJa, oSa);
							edgeOut[ia + 2] = make_float4(oMb, oIb, oJb, oSb);
							}
						}
					else if (q == nq && lane < nl)        // separator, then the next pair of the chain
						{
						mb_clear_state(st, C, lane);
						oMa = Z; oIa = Z; oJa = Z; oSa = Z; oMb = Z; oIb = Z; oJb = Z; oSb = Z;
						dprev = Z;
						if (++kp < nch)
							{
							X = mb_seq(P, P.px[cpairs[kp]]);
							pad = ~X.len & 1; nq = X.len/2 + 1;
							r0 = t + 1;
							xa = h.pad; xb = xcode(1 - pad);
							}
						else
							r0 = 1 << 29;                 // done: idle for the rest of the strip
						}
					}
				__syncwarp();
				}
			}

		// ============================ total probability, lane k for pair k ============================
		if (lane < nch)
			{
			const float *f = cfin + 5*lane;
			float total = Z;
			total = la(total, ADD(f[0], h.tSM));
			total = la(total, ADD(f[1], h.tSI));
			total = la(total, ADD(f[2], h.tSI));
			total = la(total, ADD(f[3], h.tSJ));
			total = la(total, ADD(f[4], h.tSJ));
			ctotal[lane] = total;
			if (DUMP && cpairs[lane] == P.dbg_pair)
				*P.dbg_total = total;
			}
		__syncwarp();

		// ============================ Backward + posterior ============================
		// The chain's pairs last to first, rows LX..1 of a pair and then a separator step; pair k starts
		// at chain step (sum over later pairs of (LX + 1)) + nl-1-l.  ckept[k][l] counts the lane's
		// kept entries up to the end of pair k, so that each pair's count is a difference.
		// The column loop only tests the score: it keeps the score in the spare .w of the state record and
		// sets bit c of a per-lane mask.  After the loop each lane appends its survivors {score, column},
		// so the warp runs that code as often as the most survivors in one lane, not once per column in
		// which any lane has one (under SIMT a branch costs the whole warp when one lane takes it).  The
		// list holds scores, not probabilities: expf is a long FP64 chain, and the compaction forms p
		// from 32 converged lanes instead.  A candidate is kept when p >= 0.01f (mysparsemx.cpp:139-141),
		// which is a compare of the score with mb_keep_score (tests/test_logadd_expf_gpu.py checks the two
		// decisions agree on every score).  Row i's entry count travels with the wavefront like the state:
		// lane l+1 finished its columns of row i, which lie to the right, one step before lane l, so the
		// list stays in descending column order; across strips the count rides in the spare .w of the edge
		// record, and lane 0 of strip 0, the last to touch the row, stores it in rowcnt.  The threshold is
		// mb_keep_score's expression written out: called through the helper, ptxas assigns two registers
		// of the plain kernels differently.
		const float keepScore = fmaxf(h.minScore, __uint_as_float(0xc0935d8eu));
		uint32_t kept = 0;
		bool overflow = false;
		// MEGA mode: one row per lane per step.
		if constexpr (MEGA)
			for (int strip = g.n - 1; strip >= 0; --strip)
				{
				const auto [j0, nl, cn, last] = g.at(strip, lane);
				const auto [edgeIn, edgeOut] = mb_strip_edges(edge0, edge1, strip);
				const float *fms = fm + (size_t) strip*P.fm_rows*W;

				mb_stage_y<true>(Y, j0 + lane*C + 1, C, lane, h.pad, st, ye, y2);
				float outM = Z, outIY = Z, outJY = Z;
				uint32_t outCnt = 0;
				float dprev = Z;
				const int nsteps = sumLX + nch - 2 + nl;
				int kp = nch - 1, u0 = nl - 1 - lane;   // the lane's pair and the step of its row LX
				MbSeq X = mb_seq(P, P.px[cpairs[nch - 1]]);
				MbXRow xPref = mb_x_row(X, false, 0);
				int fk = sumLX - X.len + 2*(nch - 1);   // chain Forward step of the pair's row 0, less the lane
				int rk = sumLX - X.len;               // chain row of the pair's row 1 in rows / rowcnt
				float total = ctotal[nch - 1];
				for (int u = 0; u < nsteps; ++u)
					{
					const int i = X.len - u + u0;
					const MbXRow x = xPref;
					xPref = mb_x_row(X, i >= 2 && i <= X.len, i - 1);
					float Rm = __shfl_down_sync(MB_FULL, outM, 1);
					float Riy = __shfl_down_sync(MB_FULL, outIY, 1);
					float Rjy = __shfl_down_sync(MB_FULL, outJY, 1);
					uint32_t cnt = __shfl_down_sync(MB_FULL, outCnt, 1);    // entries already in the row
					if (i >= 1 && i <= X.len && lane < nl)
						{
						if (lane == nl - 1)
							{
							if (last)
								{
								Rm = Z; Riy = Z; Rjy = Z; cnt = 0;
								}
							else
								{
								const float4 e = edgeIn[i];
								Rm = e.x; Riy = e.y; Rjy = e.z; cnt = __float_as_uint(e.w);
								}
							}
						const MbXEmit xe = mb_x_emit(P, x);
						const float ex = xe.ins;
						const int t = fk + i + lane;
						const int col0 = j0 + lane*C;
						float mdiag = dprev;
						dprev = Rm;
						float riy = Riy, rjy = Rjy, mFirst = Z;
						// the posterior scores' threshold: columns arrive descending, so bit c of hits ends up on column c
						uint32_t hits = 0;
						const bool dump = DUMP && cpairs[kp] == P.dbg_pair;
						float4 *sp = st + lane;
						const uint2 *yp = ye + lane;
						const uint32_t *y2p = y2 + lane;
						const float *src = fms + (size_t) t*W + lane;     // Forward M of the lane's column 0
						int c = cn - 1;
						sp += c*32; yp += c*32; y2p += c*32; src += c*32;
						if (last && i == X.len && lane == g.lcl)
							{
							// cell (LX,LY), the lane's first: the end scores (bwdflat3.cpp:53-61)
							mdiag = sp->x;
							const float s = mb_post_score(P, dump, i, LY, col0 + c, *src, h.tSM, total);
							hits = s >= h.minScore ? 1u : 0u;
							*sp = make_float4(h.tSM, h.tSI, h.tSJ, s);
							riy = h.tSI; rjy = h.tSJ; mFirst = h.tSM;
							--c; sp -= 32; yp -= 32; y2p -= 32; src -= 32;
							}
						// Forward M is loaded two columns ahead.  ptxas places the load where register pressure lets
						// it, mid-loop here; one column ahead that left less than an iteration to cover an HBM miss and
						// cost C4 6 % (the CM = 16 class runs 4 warps per scheduler).  The loads stay within this step's
						// columns, except *src when the cell (LX,LY) was the lane's only column (c = -1): that is
						// step t-1's column C-1 (t is the same in every lane), inside this warp's spill since t >= 1
						float fmNext = *src;                       // column c
						float fmNext2 = c >= 1 ? src[-32] : 0.0f;  // column c-1
#pragma unroll 1
						for (; c >= 0; --c, sp -= 32, yp -= 32, y2p -= 32)
							{
							const float fmv = fmNext;
							fmNext = fmNext2;
							src -= 32;
							if (c >= 2)
								fmNext2 = src[-32];                // column c-2
							const float4 v = *sp;                      // {M, IX, JX, score} of row i+1
							const auto [em, eyc] = mb_col_emit(matchT, xe, nf, yp, y2p);
							const MbBwdCell b = mb_bwd_cell(h, la, mdiag, v.y, v.z, riy, rjy, em, eyc, ex);
							const float s = mb_post_score(P, dump, i, LY, col0 + c, fmv, b.m, total);
							hits = 2u*hits + (s >= h.minScore ? 1u : 0u);
							mdiag = v.x;
							*sp = make_float4(b.m, b.ix, b.jx, s);
							riy = b.iy; rjy = b.jy;
							mFirst = b.m;
							}
						// the survivors, highest column first (the row's order): the warp runs this loop as often as
						// the most survivors in one lane, not once per column in which any lane has one
						mb200_entry *row = rows + (size_t)(rk + i - 1)*MB_CAP;
						while (hits)
							{
							const int hc = 31 - __clz(hits);
							hits ^= 1u << hc;
							const float score = st[hc*32 + lane].w;
							if (cnt < MB_CAP)
								*reinterpret_cast<uint2 *>(row + cnt) = make_uint2(__float_as_uint(score), (uint32_t)(col0 + hc));
							else
								overflow = true;
							++cnt;
							kept += score >= keepScore ? 1u : 0u;
							}
						outM = mFirst; outIY = riy; outJY = rjy;
						outCnt = cnt;
						if (lane == 0)
							{
							if (strip > 0)
								edgeOut[i] = make_float4(outM, outIY, outJY, __uint_as_float(cnt));
							else
								rowcnt[rk + i - 1] = (uint8_t) min(cnt, (uint32_t) MB_CAP);
							}
						}
					else if (i == 0 && lane < nl)         // separator, then the previous pair of the chain
						{
						mb_clear_state(st, C, lane);
						outM = Z; outIY = Z; outJY = Z;
						outCnt = 0;
						dprev = Z;
						ckept[kp*32 + lane] = kept;
						if (kp > 0)
							{
							X = mb_seq(P, P.px[cpairs[--kp]]);
							u0 = u + 1;
							fk -= X.len + 2;
							rk -= X.len;
							total = ctotal[kp];
							}
						else
							u0 = -(1 << 30);              // done: idle for the rest of the strip
						}
					__syncwarp();
					}
				}
		else
			{
			// Plain mode, two rows per lane per step: row a and row b = a-1, paired on the Forward steps (row a
			// is a Forward row b), from row LX down, so that the end scores at (LX,LY) are always row a's.  Row b
			// takes row a's {M, IX, JX} of each column from registers; the record stores row b's and, in the
			// spare .w, row a's score; a survivor of row b gets its score formed again after the loop from the
			// stored M and the Forward-M line.  The hits of both rows share one mask (row a in bits 0-15, row b
			// in 16-31) and their counts one shuffled word.  A pair takes mb_fwd_steps(LX, 2) - 1 steps; when LX
			// is odd, its last row b is row 0, computed and dropped: the separator ends that step.
			for (int strip = g.n - 1; strip >= 0; --strip)
				{
				const auto [j0, nl, cn, last] = g.at(strip, lane);
				const auto [edgeIn, edgeOut] = mb_strip_edges(edge0, edge1, strip);
				const float2 *fms = reinterpret_cast<const float2 *>(fm) + (size_t) strip*P.fm_rows*W;

				mb_stage_y<false>(Y, j0 + lane*C + 1, C, lane, h.pad, st, ye, y2);
				float oMa = Z, oIa = Z, oJa = Z, oMb = Z, oIb = Z, oJb = Z;
				uint32_t oCnt = 0;                    // entries already in row a (bits 0-15) and row b (16-31)
				float dprev = Z;
				const int nsteps = sumFS - nch - 1 + nl;
				int kp = nch - 1, u0 = nl - 1 - lane;   // the lane's pair and the step of its row LX
				MbSeq X = mb_seq(P, P.px[cpairs[nch - 1]]);
				int pad = ~X.len & 1;
				int fk = sumFS - (int) mb_fwd_steps(X.len, 2);   // chain Forward step of the pair's first rows, less the lane
				int rk = sumLX - X.len;               // chain row of the pair's row 1 in rows / rowcnt
				float total = ctotal[nch - 1];
				auto xcode = [&](int i) { return i >= 1 && i < X.len ? (int) X.code[i] : h.pad; };   // row i reads residue i+1
				int xa = h.pad, xb = xcode(X.len - 1);   // classes of the next step's rows
				// then the previous pair of the chain.  The step's outputs stay: when row b is row 0, lane l-1 still
				// reads row a's next step (a whole separator step ignores them)
				auto separator = [&](int u)
					{
					mb_clear_state(st, C, lane);
					dprev = Z;
					ckept[kp*32 + lane] = kept;
					if (kp > 0)
						{
						X = mb_seq(P, P.px[cpairs[--kp]]);
						u0 = u + 1;
						pad = ~X.len & 1;
						fk -= mb_fwd_steps(X.len, 2);
						rk -= X.len;
						total = ctotal[kp];
						xa = h.pad; xb = xcode(X.len - 1);
						}
					else
						u0 = -(1 << 29);              // done: idle for the rest of the strip
					};
				for (int u = 0; u < nsteps; ++u)
					{
					const int ia = X.len - 2*(u - u0);   // rows ia and ia-1 of pair kp
					const int xca = xa, xcb = xb;
					xa = xcode(ia - 2); xb = xcode(ia - 3);
					float Rma = __shfl_down_sync(MB_FULL, oMa, 1);
					float Riya = __shfl_down_sync(MB_FULL, oIa, 1);
					float Rjya = __shfl_down_sync(MB_FULL, oJa, 1);
					float Rmb = __shfl_down_sync(MB_FULL, oMb, 1);
					float Riyb = __shfl_down_sync(MB_FULL, oIb, 1);
					float Rjyb = __shfl_down_sync(MB_FULL, oJb, 1);
					uint32_t cnt = __shfl_down_sync(MB_FULL, oCnt, 1);
					if (ia >= 1 && ia <= X.len && lane < nl)
						{
						if (lane == nl - 1)
							{
							if (last)
								{
								Rma = Z; Riya = Z; Rjya = Z; Rmb = Z; Riyb = Z; Rjyb = Z; cnt = 0;
								}
							else
								{
								const float4 ea = edgeIn[ia], eb = edgeIn[ia - 1];
								Rma = ea.x; Riya = ea.y; Rjya = ea.z;
								Rmb = eb.x; Riyb = eb.y; Rjyb = eb.z;
								cnt = __float_as_uint(ea.w) | __float_as_uint(eb.w) << 16;
								}
							}
						const float2 *mea = meT + xca*h.KS, *meb = meT + xcb*h.KS;
						const float exa = sm.insT[xca], exb = sm.insT[xcb];
						const int t = fk + (ia + pad - 1)/2 + lane;   // the Forward step of rows ia-1, ia
						const int col0 = j0 + lane*C;
						float mdiaga = dprev, mdiagb = Rma;
						dprev = Rmb;
						float riya = Riya, rjya = Rjya, riyb = Riyb, rjyb = Rjyb, mFirsta = Z, mFirstb = Z;
						// the posterior scores' threshold: columns arrive descending, so bit c of hits ends up on row a's
						// column c and bit 16+c on row b's
						uint32_t hits = 0;
						const bool dump = DUMP && cpairs[kp] == P.dbg_pair;
						float4 *sp = st + lane;
						const uint32_t *y2p = y2 + lane;
						const float2 *fmc = fms + (size_t) t*W + lane;   // Forward M {row ia-1, row ia} of the lane's column 0
						const float2 *src = fmc;
						int c = cn - 1;
						sp += c*32; y2p += c*32; src += c*32;
						if (last && ia == X.len && lane == g.lcl)
							{
							// cell (LX,LY), row a's first: the end scores (bwdflat3.cpp:53-61); row b's cell below it
							const float2 f = *src;
							const uint32_t yc = *y2p;
							const float2 e = meb[yc];
							const float sa = mb_post_score(P, dump, ia, LY, col0 + c, f.y, h.tSM, total);
							const MbBwdCell b = mb_bwd_cell(h, la, mdiagb, h.tSI, h.tSJ, riyb, rjyb, e.x, e.y, exb);
							const float sb = mb_post_score(P, dump, ia - 1, LY, col0 + c, f.x, b.m, total);
							hits = (sa >= h.minScore ? 1u : 0u) + (sb >= h.minScore ? 0x10000u : 0u);
							mdiaga = sp->x;
							mdiagb = h.tSM;
							*sp = make_float4(b.m, b.ix, b.jx, sa);
							riya = h.tSI; rjya = h.tSJ; mFirsta = h.tSM;
							riyb = b.iy; rjyb = b.jy; mFirstb = b.m;
							--c; sp -= 32; y2p -= 32; src -= 32;
							}
						// Forward M is loaded two columns ahead, as in the single-row loop, and never outside this
						// step's columns
						float2 fmNext = c >= 0 ? src[0] : make_float2(0.0f, 0.0f);      // column c
						float2 fmNext2 = c >= 1 ? src[-32] : make_float2(0.0f, 0.0f);   // column c-1
#pragma unroll 1
						for (; c >= 0; --c, sp -= 32, y2p -= 32)
							{
							const float2 f = fmNext;
							fmNext = fmNext2;
							src -= 32;
							if (c >= 2)
								fmNext2 = src[-32];                // column c-2
							const float4 v = *sp;                      // {M, IX, JX, -} of row ia+1
							const uint32_t yc = *y2p;
							const float2 e = mea[yc];                  // {match of row a, insert of Y}
							const float emb = reinterpret_cast<const float *>(meb + yc)[0];
							const MbBwdCell a = mb_bwd_cell(h, la, mdiaga, v.y, v.z, riya, rjya, e.x, e.y, exa);
							const float sa = mb_post_score(P, dump, ia, LY, col0 + c, f.y, a.m, total);
							const MbBwdCell b = mb_bwd_cell(h, la, mdiagb, a.ix, a.jx, riyb, rjyb, emb, e.y, exb);
							const float sb = mb_post_score(P, dump, ia - 1, LY, col0 + c, f.x, b.m, total);
							hits = 2u*hits + (sa >= h.minScore ? 1u : 0u) + (sb >= h.minScore ? 0x10000u : 0u);
							mdiaga = v.x;
							mdiagb = a.m;
							*sp = make_float4(b.m, b.ix, b.jx, sa);
							riya = a.iy; rjya = a.jy; mFirsta = a.m;
							riyb = b.iy; rjyb = b.jy; mFirstb = b.m;
							}
						// the survivors, row b's then row a's, highest column first (each row's order)
						if (ia == 1)
							hits &= 0xffffu;                   // row b is row 0, the separator
						uint32_t cnta = cnt & 0xffffu, cntb = cnt >> 16;
						mb200_entry *rowa = rows + (size_t)(rk + ia - 1)*MB_CAP;
						while (hits)
							{
							const int hb = 31 - __clz(hits);
							hits ^= 1u << hb;
							const bool inb = hb >= 16;
							const int hc = hb & 15;
							const float4 r = st[hc*32 + lane];
							const float score = inb ? __fsub_rn(ADD(fmc[hc*32].x, r.x), total) : r.w;
							const uint32_t n = inb ? cntb : cnta;
							if (n < MB_CAP)
								*reinterpret_cast<uint2 *>(rowa - (inb ? MB_CAP : 0) + n) =
								  make_uint2(__float_as_uint(score), (uint32_t)(col0 + hc));
							else
								overflow = true;
							if (inb)
								++cntb;
							else
								++cnta;
							kept += score >= keepScore ? 1u : 0u;
							}
						cnta = min(cnta, (uint32_t) MB_CAP);
						cntb = min(cntb, (uint32_t) MB_CAP);
						oMa = mFirsta; oIa = riya; oJa = rjya;
						oMb = mFirstb; oIb = riyb; oJb = rjyb;
						oCnt = cnta | cntb << 16;
						if (lane == 0)
							{
							if (strip > 0)
								{
								edgeOut[ia] = make_float4(oMa, oIa, oJa, __uint_as_float(cnta));
								edgeOut[ia - 1] = make_float4(oMb, oIb, oJb, __uint_as_float(cntb));
								}
							else
								{
								rowcnt[rk + ia - 1] = (uint8_t) cnta;
								if (ia > 1)
									rowcnt[rk + ia - 2] = (uint8_t) cntb;
								}
							}
						if (ia == 1)
							separator(u);
						}
					else if (ia == 0 && lane < nl)
						separator(u);
					__syncwarp();
					}
				}
			}
		ckept[lane] = kept;                       // the end of pair 0 (its separator may lie past the last step)
		overflow = __any_sync(MB_FULL, overflow);
		if (lane == 0 && overflow)
			atomicCAS(P.err, 0, MB200_EOVERFLOW);
		__syncwarp();

		// ============================ compaction + expected accuracy, pair by pair ============================
		int rk = 0;
		for (int k = 0; k < nch; ++k)
			{
			const uint32_t pair = cpairs[k];
			const int LX = (int) P.seqlen[P.px[pair]];
			mb_compact_ea<MEGA, CM>(P, pair, LX, LY, ckept[k*32 + lane] - (k + 1 < nch ? ckept[(k + 1)*32 + lane] : 0u),
			  rows + (size_t) rk*MB_CAP, rowcnt + rk, g, wbase, reinterpret_cast<float *>(edge0),
			  reinterpret_cast<float *>(edge1));
			rk += LX;
			}
		}
	}
