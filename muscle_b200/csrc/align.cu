// align.cu -- posterior decoding on the device: the max-sum DP with traceback (CalcAlnFlat) for
// batches of stored pairs, the column-posterior matrix of a progressive-alignment join (BuildPost),
// and the device-resident multiple alignments that progressive alignment and refinement work on.
//
// Replaces CalcAlnFlat (calcalnflat.cpp:6-46) + Best3 (best3.h:5-28) + TraceBackFlat
// (tracebackflat.cpp:3-37), MPCFlat::BuildPost (buildpostflat.cpp:18-105), MPCFlat::AlignAlns
// (alnalnsflat.cpp:7-52) including Sequence::AddGapsPath (sequence.cpp:115-140) and
// MultiSequence::Project (project.cpp:16-69) on position->column maps, i.e. the data path of
// MPCFlat::ProgAln (progalnflat.cpp:41-71) and MPCFlat::RefineIter (refineflat.cpp:4-31).
//
// Decoding DP (k_aln_wave).  One warp per 128-column strip (up to 16 strips per CTA, several CTAs per
// problem when it is wider); lane l owns 4
// consecutive columns and the rows are swept as an anti-diagonal wavefront (lane l is on row t-l at
// step t, the left neighbour's value arrives by one shuffle, the left strip's through a shared-memory
// ring), exactly the reference's recurrence
//      new[j] = max3(old[j-1] + P[i][j], old[j], new[j-1])
// evaluated with the same fp32 add and the same operands, so scores are bit-identical; the
// traceback letter follows Best3's tie rule (B if B>=X and B>=Y; else Y if B>=X; else X if X>=Y else
// Y) and is stored as 2 bits per cell (shared memory when it fits, else global), then walked by
// warp 0 (an 8-row x 16-column tile of traceback bytes cached across the lanes) and reversed.  Round 1 used one CTA
// with 4+ barriers per row and a serial traceback through global memory.
//
// BuildPost.  Every cell is a sum over (s,t) in the reference's s-major/t-minor order with at most
// one term per (s,t); the order is kept per cell, everything else is parallel.  Phase 1 (k_bp_gather,
// one thread per (residue of A's members, t)) does the random gathers into the store and writes each
// needed sparse row, mapped to columns of B, into a 16-entry staging slot; phase 2 (k_bp_apply, one warp per row,
// accumulator row in shared memory) streams the slots through a cp.async ring and applies
// them strictly in order, the entries of one sparse row in parallel.  Large joins take another route
// (k_bpc_*, further down): the terms are bucketed by output cell and every cell is summed front to back.
#include "engine.h"
#include <cuda_pipeline.h>
#include <cub/cub.cuh>
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>

// MB200_TRACE=1: wall-time split of the join path, printed at process exit
static bool g_trace = false;
static int g_trace_level = 0;          // 2: one line per join of >= 64 sequences
static double g_t[6] = { 0, 0, 0, 0, 0, 0 };
static double g_ts[5] = { 0, 0, 0, 0, 0 };   // sorted BuildPost path: count+order, emit, sort, runs, sum
static unsigned g_calls = 0;
static double now_s()
	{
	return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
	}
static void trace_report()
	{
	fprintf(stderr, "[mb200 trace] joins x%u: maps %.2f s, BuildPost gather %.2f s, apply %.2f s, decode DP %.2f s, "
	  "map update %.2f s, host %.2f s\n", g_calls, g_t[0], g_t[1], g_t[2], g_t[3], g_t[4], g_t[5]);
	if (g_ts[0] > 0)
		fprintf(stderr, "[mb200 trace] BuildPost by cell: count+order %.2f s, emit %.2f s, sort %.2f s, runs %.2f s, sum %.2f s\n",
		  g_ts[0], g_ts[1], g_ts[2], g_ts[3], g_ts[4]);
	}
static void trace_init()
	{
	static bool done = false;
	if (done)
		return;
	done = true;
	g_trace = getenv("MB200_TRACE") != nullptr;
	if (g_trace)
		{
		g_trace_level = atoi(getenv("MB200_TRACE"));
		atexit(trace_report);
		}
	}
// The running marks of one join: mark(k) adds the time since the previous mark to g_t[k], sub(k) the
// time since the previous sub to g_ts[k].  Both synchronise the stream, and only when tracing.
struct JoinTimer
	{
	cudaStream_t st;
	double tmark, tsub = 0;
	explicit JoinTimer(cudaStream_t s) : st(s) { trace_init(); tmark = now_s(); ++g_calls; }
	void mark(int k) { if (g_trace) { cudaStreamSynchronize(st); const double n = now_s(); g_t[k] += n - tmark; tmark = n; } }
	void sub(int k) { if (g_trace) { cudaStreamSynchronize(st); const double n = now_s(); g_ts[k] += n - tsub; tsub = n; } }
	};

// =============================================================================================
// decoding DP
#define AW_C 4                       // columns per lane (a single warp is bound by instruction latency: narrow
                                     // lanes put more warps on a row)
#define AW_W (32*AW_C)               // strip width
struct AlnProblem
	{
	uint32_t LX, LY, ld;             // ld: row pitch of dense (multiple of AW_C, padding zero)
	const float *dense;              // LX rows x ld, preceded by one row of zeros and followed by AW_PAD_BOT readable rows
	uint8_t *tb;                     // traceback bytes [LX][nstrips*32] (global), unused when the launch keeps it in smem
	uint2 *edge;                     // [npass-1][LX+1] {value, row tag}: hand-over between the CTAs of one problem (zeroed by the host)
	uint32_t *done;                  // CTAs of the problem that have finished (zeroed by the host)
	char *path;                      // LX+LY+1
	float *score;
	uint32_t *plen;                  // may be nullptr
	};

#define AW_MAXW 16                   // warps per CTA = strips in flight
#define AW_RING 64                   // rows of slack between neighbouring strips
#ifndef AW_PF
#define AW_PF 6                      // rows of the dense matrix in flight per lane
#endif
#define AW_PAD_BOT (AW_PF + 31)       // readable rows below row LX of a dense matrix (loads are not predicated)

// One warp per strip of 32*AW_C columns, AW_MAXW strips per CTA, and as many CTAs per problem
// (blockIdx.y) as the width needs.  Inside a warp the rows are an anti-diagonal wavefront over the
// lanes; between warps the same wavefront continues: strip w+1 consumes, row by row, the last column of
// strip w through a shared-memory ring whose entries carry {value, row} in ONE 64-bit word (no fence),
// and between CTAs through a global array of the same entries (the CTAs of a problem are dispatched in
// blockIdx.y order, so a consumer never waits for a producer that cannot start).  A 4349 x 4636 join
// therefore takes ~LX + 32*strips steps instead of LX*strips.
__device__ __forceinline__ void ring_put(uint2 *slot, float v, int row)
	{
	asm volatile("st.volatile.shared.v2.u32 [%0], {%1, %2};" :: "r"((uint32_t) __cvta_generic_to_shared(slot)),
	  "r"(__float_as_uint(v)), "r"((uint32_t) row) : "memory");
	}
__device__ __forceinline__ uint2 ring_get(const uint2 *slot)
	{
	uint2 e;
	asm volatile("ld.volatile.shared.v2.u32 {%0, %1}, [%2];" : "=r"(e.x), "=r"(e.y)
	  : "r"((uint32_t) __cvta_generic_to_shared(slot)) : "memory");
	return e;
	}
__device__ __forceinline__ void chan_put(uint2 *slot, float v, int row)
	{
	asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" :: "l"(slot), "r"(__float_as_uint(v)), "r"((uint32_t) row) : "memory");
	}
__device__ __forceinline__ uint2 chan_get(const uint2 *slot)
	{
	uint2 e;
	asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(e.x), "=r"(e.y) : "l"(slot) : "memory");
	return e;
	}

__device__ __forceinline__ uint2 lds_v2_volatile(uint32_t addr)
	{
	uint2 e;
	asm volatile("ld.volatile.shared.v2.u32 {%0, %1}, [%2];" : "=r"(e.x), "=r"(e.y) : "r"(addr) : "memory");
	return e;
	}
__device__ __forceinline__ void sts_v2_volatile(uint32_t addr, float v, int row)
	{
	asm volatile("st.volatile.shared.v2.u32 [%0], {%1, %2};" :: "r"(addr), "r"(__float_as_uint(v)), "r"((uint32_t) row) : "memory");
	}
__device__ __forceinline__ int lds_volatile(uint32_t addr)
	{
	int v;
	asm volatile("ld.volatile.shared.s32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
	return v;
	}

// The strip loop is written for a warp that is ALONE on its scheduler: what matters is the length of
// the dependent chain and the number of issue slots of one step, not occupancy.  A lane-0 spin loop
// would leave the warp split in two for the whole step, addresses recomputed from (i, strip, lane) in
// 64-bit arithmetic and predicated row loads would force register copies.  Here: every lane polls the same ring slot, so the wait loop is warp-uniform and nothing diverges; cells
// are computed unconditionally and only the traceback store is predicated; the dense matrix has one zero
// row above row 1 and AW_PAD_BOT readable rows below row LX, so the row loads need no predicate either
// (rows < 1 read the zero row and keep the wavefront at 0, rows > LX compute values nobody reads); all
// addresses advance by constants; the hand-over mode of a strip (none / shared ring / global channel on
// either side) is a template parameter.
struct AwLinks
	{
	uint32_t ringInBase, ringOutBase, consSelf, consNext;    // shared-memory addresses
	const uint2 *chanIn; uint2 *chanOut;
	};

template <bool TB_SMEM, int IN, int OUT>                     // 0: none, 1: shared-memory ring, 2: global channel
__device__ __forceinline__ void aw_strip(const AlnProblem &pr, const AwLinks &K, uint32_t tb_sm_base, int strip, int nstrips, int lane)
	{
	const int LX = (int) pr.LX, LY = (int) pr.LY;
	const int j0 = strip*AW_W;
	const int ncol = min(AW_W, LY - j0);
	const int nl = (ncol + AW_C - 1)/AW_C;
	const bool laneOn = lane < nl;
	float old[AW_C];
#pragma unroll
	for (int c = 0; c < AW_C; ++c)
		old[c] = 0.0f;                                       // row 0 (calcalnflat.cpp:15-19)
	float outNew = 0.0f, prevRecv = 0.0f;
	// rows are fetched AW_PF steps ahead: before step t the queue holds rows i .. i+AW_PF-1 of this lane,
	// one register set per step of the unrolled loop.  Row index -1 is the zero row.
	const long long ldb = (long long) pr.ld*(long long) sizeof(float);
	const long long base = (long long)(size_t)(pr.dense + j0 + (laneOn ? lane : 0)*AW_C);
	float4 q[AW_PF];
	int i = 1 - lane;                                        // 1-based row of this lane at step t
#pragma unroll
	for (int u = 0; u < AW_PF; ++u)
		q[u] = *reinterpret_cast<const float4 *>((size_t)(base + (long long) max(i + u - 1, -1)*ldb));
	long long nxt = base + (long long) max(i + AW_PF - 1, -1)*ldb;      // row i+AW_PF of this lane
	const int tbstep = nstrips*32;
	// traceback byte of (row i, this lane's column group); advanced every step, used only for rows 1..LX
	long long tbg = (long long)(size_t) pr.tb + ((long long)(i - 1)*nstrips + strip)*32 + lane;
	uint32_t tbs = tb_sm_base + (uint32_t)(((i - 1)*nstrips + strip)*32 + lane);
	const int nsteps = LX + nl - 1;
	auto step = [&](const int t, float4 &q)
		{
		float recv = __shfl_up_sync(MB_FULL, outNew, 1);
		float in = 0.0f;
		if (IN != 0)
			{
			const int i0 = t + 1;                            // row of lane 0 (warp-uniform)
			if (i0 <= LX)
				{
				uint2 e;
				if (IN == 1)
					{
					const uint32_t slot = K.ringInBase + ((uint32_t)(i0 & (AW_RING - 1)) << 3);
					do
						e = lds_v2_volatile(slot);           // all lanes read the same word: the loop is uniform
					while ((int) e.y != i0);                 // strip on the left has not produced row i0 yet
					if (lane == 0)
						asm volatile("st.volatile.shared.s32 [%0], %1;" :: "r"(K.consSelf), "r"(i0) : "memory");
					}
				else
					{
					do
						e = chan_get(K.chanIn + i0);
					while ((int) e.y != i0);
					}
				in = __uint_as_float(e.x);
				}
			}
		if (lane == 0)
			recv = in;
		const float4 pv = q;
		float Bv[AW_C];
		Bv[0] = __fadd_rn(prevRecv, pv.x);                   // calcalnflat.cpp:31-37: old[j-1] + P[i][j]
		Bv[1] = __fadd_rn(old[0], pv.y);
		Bv[2] = __fadd_rn(old[1], pv.z);
		Bv[3] = __fadd_rn(old[2], pv.w);
		q = *reinterpret_cast<const float4 *>((size_t) nxt);
		if (i >= -AW_PF)
			nxt += ldb;
		float Y = recv;                                      // new[i][first col - 1]
		uint32_t word = 0;
#pragma unroll
		for (int c = 0; c < AW_C; ++c)
			{
			const float B = Bv[c];
			const float X = old[c];
			const float M = fmaxf(B, X);
			const uint32_t mcode = (B >= X) ? 0u : 1u;       // best3.h:5-28: B if B>=X and B>=Y; X if X>B and X>=Y; else Y
			const uint32_t code = (M >= Y) ? mcode : 2u;
			const float nw = fmaxf(M, Y);
			word |= code << (2*c);
			old[c] = nw;
			Y = nw;
			}
		outNew = Y;
		if (laneOn && (unsigned)(i - 1) < (unsigned) LX)
			{
			if (TB_SMEM)
				asm volatile("st.shared.u8 [%0], %1;" :: "r"(tbs), "r"(word) : "memory");
			else
				*reinterpret_cast<uint8_t *>((size_t) tbg) = (uint8_t) word;
			}
		tbs += (uint32_t) tbstep;
		tbg += tbstep;
		if (OUT != 0)
			{
			const int i31 = t - 30;                          // row of lane 31 (warp-uniform)
			if (i31 >= 1 && i31 <= LX)
				{
				if (OUT == 1)
					{
					while (lds_volatile(K.consNext) < i31 - AW_RING)
						;                                     // the slot still holds an unconsumed row
					if (lane == 31)
						sts_v2_volatile(K.ringOutBase + ((uint32_t)(i31 & (AW_RING - 1)) << 3), outNew, i31);
					}
				else if (lane == 31)
					chan_put(K.chanOut + i31, outNew, i31);
				}
			}
		prevRecv = recv;
		++i;
		};
	int t = 0;
	for (; t + AW_PF <= nsteps; t += AW_PF)
		{
#pragma unroll
		for (int u = 0; u < AW_PF; ++u)
			step(t + u, q[u]);
		}
#pragma unroll
	for (int u = 0; u < AW_PF; ++u)
		if (t + u < nsteps)
			step(t + u, q[u]);
	if (strip == nstrips - 1 && lane == nl - 1)
		{
		// the lane that owns DP column LY finished row LX in the last step
		const int lastC = (LY - 1 - j0) % AW_C;
		float v = old[0];
#pragma unroll
		for (int c = 1; c < AW_C; ++c)
			if (c == lastC)
				v = old[c];
		*pr.score = v;
		}
	}

template <bool TB_SMEM>
__global__ void __launch_bounds__(32*AW_MAXW)
k_aln_wave(const AlnProblem *probs)
	{
	extern __shared__ uint8_t tb_sm[];
	__shared__ uint2 ring[AW_MAXW][AW_RING];          // {bits of the value, row it belongs to}: one 8-byte store
	__shared__ int cons[AW_MAXW];
	const AlnProblem pr = probs[blockIdx.x];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const int NW = blockDim.x >> 5;
	const int LX = (int) pr.LX, LY = (int) pr.LY;
	const int nstrips = (LY + AW_W - 1)/AW_W;
	const int pass = blockIdx.y;                             // which group of AW_MAXW strips this CTA owns
	if (pass*NW >= nstrips)
		return;                                              // narrower problem of a batch
	if (lane == 0)
		cons[wid] = 0;
	for (int k = lane; k < AW_RING; k += 32)
		ring[wid][k] = make_uint2(0u, 0u);                   // row tags start at 1
	__syncthreads();
	const int strip = pass*NW + wid;
	if (strip < nstrips)
		{
		const bool hasIn = strip > 0, hasOut = strip + 1 < nstrips;
		const int inMode = !hasIn ? 0 : (wid > 0 ? 1 : 2);      // the CTA on the left hands over through global memory
		const int outMode = !hasOut ? 0 : (wid + 1 < NW ? 1 : 2);
		AwLinks K;
		K.chanIn = pr.edge + (size_t)(pass > 0 ? pass - 1 : 0)*(LX + 1);
		K.chanOut = pr.edge + (size_t) pass*(LX + 1);
		K.ringInBase = (uint32_t) __cvta_generic_to_shared(&ring[wid > 0 ? wid - 1 : 0][0]);
		K.ringOutBase = (uint32_t) __cvta_generic_to_shared(&ring[wid][0]);
		K.consSelf = (uint32_t) __cvta_generic_to_shared(&cons[wid]);
		K.consNext = (uint32_t) __cvta_generic_to_shared(&cons[wid + 1 < AW_MAXW ? wid + 1 : wid]);
		const uint32_t tbb = (uint32_t) __cvta_generic_to_shared(tb_sm);
		if (TB_SMEM)
			{
			// one CTA per problem: no global channel
			if (inMode == 0 && outMode == 0)      aw_strip<TB_SMEM, 0, 0>(pr, K, tbb, strip, nstrips, lane);
			else if (inMode == 0)                 aw_strip<TB_SMEM, 0, 1>(pr, K, tbb, strip, nstrips, lane);
			else if (outMode == 0)                aw_strip<TB_SMEM, 1, 0>(pr, K, tbb, strip, nstrips, lane);
			else                                  aw_strip<TB_SMEM, 1, 1>(pr, K, tbb, strip, nstrips, lane);
			}
		else
			{
			switch (inMode*3 + outMode)
				{
				case 0: aw_strip<false, 0, 0>(pr, K, tbb, strip, nstrips, lane); break;
				case 1: aw_strip<false, 0, 1>(pr, K, tbb, strip, nstrips, lane); break;
				case 2: aw_strip<false, 0, 2>(pr, K, tbb, strip, nstrips, lane); break;
				case 3: aw_strip<false, 1, 0>(pr, K, tbb, strip, nstrips, lane); break;
				case 4: aw_strip<false, 1, 1>(pr, K, tbb, strip, nstrips, lane); break;
				case 5: aw_strip<false, 1, 2>(pr, K, tbb, strip, nstrips, lane); break;
				case 6: aw_strip<false, 2, 0>(pr, K, tbb, strip, nstrips, lane); break;
				case 7: aw_strip<false, 2, 1>(pr, K, tbb, strip, nstrips, lane); break;
				default: aw_strip<false, 2, 2>(pr, K, tbb, strip, nstrips, lane); break;
				}
			}
		}
	__syncthreads();
	// traceback (tracebackflat.cpp:3-37): TB(0,j) = 'Y', TB(i,0) = 'X'.  Done by warp 0 of the CTA that
	// finishes last (the one owning the last strip), all lanes in lockstep on the same (i,j); the lanes
	// cache the traceback bytes of an 8-row x 4-group (16-column) tile whose corner is the current cell, so
	// that a dependent load is needed about every 8 steps of a diagonal path.
	const int npass = (nstrips + NW - 1)/NW;
	if ((pass + 1)*NW < nstrips)
		{
		// not the last CTA of the problem: publish the traceback bytes and leave
		if (threadIdx.x == 0)
			{
			__threadfence();
			atomicAdd(pr.done, 1u);
			}
		return;
		}
	if (wid != 0)
		return;
	if (npass > 1)
		{
		if (lane == 0)
			while (atomicAdd(pr.done, 0u) < (uint32_t)(npass - 1))
				;
		__syncwarp();
		__threadfence();
		}
	uint32_t n = 0;
		{
		const uint8_t *tbb = TB_SMEM ? tb_sm : pr.tb;
		const int rowpitch = nstrips*32;
		int i = LX, j = LY;
		int cbase = -1, cidx = -1;
		uint32_t cw = 0;
		const int lr = lane >> 2, lg = lane & 3;
		while (i > 0 && j > 0)
			{
			const int jj = j - 1;
			const int idx = jj >> 2;                         // column group (AW_C = 4; 32 groups per strip, numbered across strips)
			const int dr = cbase - i, dg = cidx - idx;
			if ((unsigned) dr >= 8u || (unsigned) dg >= 4u)
				{
				cbase = i; cidx = idx;
				const int r = i - lr, g = idx - lg;
				cw = 0u;
				if (r >= 1 && g >= 0)
					cw = TB_SMEM ? (uint32_t) tbb[(size_t)(r - 1)*rowpitch + g]
					             : (uint32_t) __ldcv(tbb + (size_t)(r - 1)*rowpitch + g);    // other CTAs wrote it
				}
			const uint32_t w = __shfl_sync(MB_FULL, cw, ((cbase - i) << 2) + (cidx - idx));
			const uint32_t code = (w >> (2*(jj & 3))) & 3u;      // 0: B, 1: X, 2: Y
			if (lane == 0)
				pr.path[n] = code == 0 ? 'B' : (code == 1 ? 'X' : 'Y');
			++n;
			i -= (code != 2u);
			j -= (code != 1u);
			}
		// first row / first column: only gaps are left
		const char fill = i == 0 ? 'Y' : 'X';
		const uint32_t rest = (uint32_t)(i + j);
		for (uint32_t a = lane; a < rest; a += 32)
			pr.path[n + a] = fill;
		n += rest;
		if (lane == 0)
			{
			pr.path[n] = 0;
			if (pr.plen)
				*pr.plen = n;
			}
		}
	__syncwarp();
	for (uint32_t a = lane; a < n/2; a += 32)
		{
		const char x = pr.path[a], y = pr.path[n - 1 - a];
		pr.path[a] = y; pr.path[n - 1 - a] = x;
		}
	}

// dense copy of stored sparse pairs for the batched pair decoder: one warp per (problem,row)
struct DensifyJob { const uint32_t *rowoff; const mb200_entry *entries; float *dense; uint32_t LX, ld; };
__global__ void k_densify(const DensifyJob *jobs, uint32_t njobs, uint32_t maxrows)
	{
	const uint32_t warp = (blockIdx.x*blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
	const uint32_t job = warp/maxrows, row = warp % maxrows;
	if (job >= njobs)
		return;
	const DensifyJob J = jobs[job];
	if (row >= J.LX)
		return;
	float *dst = J.dense + (size_t) row*J.ld;
	for (uint32_t e = J.rowoff[row] + lane; e < J.rowoff[row + 1]; e += 32)
		dst[J.entries[e].col] = J.entries[e].p;
	}

// =============================================================================================
// BuildPost
struct BuildPostParams
	{
	uint32_t n;                                   // sequences in the store
	uint32_t na, nb, cols_a, cols_b, ld;          // ld: row pitch of post
	const uint32_t *ids_a, *ids_b;
	const int32_t *col2pos_a;                     // [na][cols_a], -1 = gap
	const uint32_t *p2c_b;                        // concatenated pos->col maps of B
	const uint64_t *p2c_b_off;                    // [nb]
	const uint64_t *rowbase;  const uint32_t *rowoff;  const mb200_entry *entries;
	const uint64_t *trbase;   const uint32_t *troff;   const mb200_entry *trentries;
	const uint64_t *entbase;
	float *post;                                  // cols_a x ld, zeroed
	};

#define BP_WARPS 4
#define BP_W 16           // staged entries per sparse row (rows are 7.2 +- 3 long: ~0.1 % exceed 16)
#define BP_G 16           // (s,t) steps per staged group

#define BP_END  0xffffffffu       // column value of an unused slot entry
#define BP_LONG 0xfffffffeu       // first entry of a slot whose sparse row is longer than BP_W (applied by direct gather)
struct BpStage
	{
	uint2   *slots;      // [residue of the batch][t][BP_W]  (column of B, bits of P), unused entries = BP_END
	uint32_t s_lo, s_n;  // batch of sequences of A
	const uint32_t *rb;  // [na+1] residues of A's members before member s (slots exist for residues only:
	                     // indexing by (column, s) would stage mostly gaps -- a 1000-row MSA of 350-residue
	                     // proteins has 7000+ columns)
	};

__device__ __forceinline__ void bp_operand(const BuildPostParams &P, uint32_t a, uint32_t b, const uint32_t *&ro,
  const mb200_entry *&en)
	{
	if (a < b)
		{
		const uint32_t q = mb_pair_index(P.n, a, b);
		ro = P.rowoff + P.rowbase[q]; en = P.entries + P.entbase[q];
		}
	else
		{
		const uint32_t q = mb_pair_index(P.n, b, a);
		ro = P.troff + P.trbase[q]; en = P.trentries + P.entbase[q];
		}
	}

__global__ void __launch_bounds__(256)
k_bp_gather(const BuildPostParams P, const BpStage G)
	{
	const uint32_t r0 = G.rb[G.s_lo];
	const uint64_t total = (uint64_t)(G.rb[G.s_lo + G.s_n] - r0)*P.nb;
	for (uint64_t idx = blockIdx.x*(uint64_t) blockDim.x + threadIdx.x; idx < total; idx += (uint64_t) gridDim.x*blockDim.x)
		{
		const uint32_t t = (uint32_t)(idx % P.nb);
		const uint32_t r = r0 + (uint32_t)(idx/P.nb);
		// member of A that owns residue r: largest s with rb[s] <= r
		uint32_t lo = G.s_lo, hi = G.s_lo + G.s_n;
		while (hi - lo > 1)
			{
			const uint32_t mid = (lo + hi) >> 1;
			if (G.rb[mid] <= r) lo = mid; else hi = mid;
			}
		const uint32_t s = lo;
		const uint32_t pos = r - G.rb[s];
		const uint32_t *ro;
		const mb200_entry *en;
		bp_operand(P, P.ids_a[s], P.ids_b[t], ro, en);
		const uint32_t e0 = ro[pos];
		const uint32_t n = ro[pos + 1] - e0;
		uint2 *dst = G.slots + idx*BP_W;
		if (n <= BP_W)
			{
			const uint32_t *p2c = P.p2c_b + P.p2c_b_off[t];
			for (uint32_t k = 0; k < n; ++k)
				{
				const mb200_entry v = en[e0 + k];
				dst[k] = make_uint2(p2c[v.col], __float_as_uint(v.p));
				}
			for (uint32_t k = n; k < BP_W; ++k)
				dst[k] = make_uint2(BP_END, 0u);
			}
		else
			{
			dst[0] = make_uint2(BP_LONG, 0u);
			for (uint32_t k = 1; k < BP_W; ++k)
				dst[k] = make_uint2(BP_END, 0u);
			}
		}
	}

// rows (columns of A) by descending number of members that have a residue there: the per-row chain of
// (s,t) steps is strictly serial, so a join lasts at least as long as its heaviest row (a conserved
// column: |A| x |B| steps); heavy rows must start first and light rows fill in behind them.
__global__ void k_bp_weight(const BuildPostParams P, uint32_t *__restrict__ weight, uint32_t *__restrict__ rowid)
	{
	const uint32_t row = blockIdx.x*blockDim.x + threadIdx.x;
	if (row >= P.cols_a)
		return;
	uint32_t w = 0;
	for (uint32_t s = 0; s < P.na; ++s)
		w += P.col2pos_a[(size_t) s*P.cols_a + row] >= 0 ? 1u : 0u;
	weight[row] = w;
	rowid[row] = row;
	}

#define BP_NBUF 3
// explicit 32-bit shared-memory accesses: with plain pointers the compiler re-derives the shared window
// base (S2UR SR_CgaCtaId + ULEA) inside the serial step loop, on the critical path of every step
__device__ __forceinline__ float lds_f32(uint32_t a)
	{
	float v;
	asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
	return v;
	}
__device__ __forceinline__ void sts_f32(uint32_t a, float v)
	{
	asm volatile("st.shared.f32 [%0], %1;" :: "r"(a), "f"(v) : "memory");
	}
__device__ __forceinline__ uint2 lds_u2(uint32_t a)
	{
	uint2 v;
	asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a) : "memory");
	return v;
	}

struct BpSched
	{
	const uint32_t *order;    // rows, heaviest first
	uint32_t *cursor;         // work cursor of this launch (zeroed by the host)
	};

// Persistent warps, one row (column of alignment A) at a time, heaviest rows first.  The (s,t)
// steps of one s are consumed in groups of BP_G: while group g is applied, the slots of groups g+1
// and g+2 are already on their way into a shared-memory ring (cp.async), so the ordered accumulation
// never waits on HBM; inside a step the <= 16 entries of the sparse row go to distinct columns and
// are added by one lane each.
__global__ void __launch_bounds__(32*BP_WARPS)
k_bp_apply(const BuildPostParams P, const BpStage G, const BpSched S)
	{
	extern __shared__ __align__(16) unsigned char bp_smem[];
	const uint32_t wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const size_t acc_bytes = ((size_t) BP_WARPS*P.cols_b*sizeof(float) + 15) & ~(size_t) 15;
	float *acc = reinterpret_cast<float *>(bp_smem) + (size_t) wib*P.cols_b;
	uint2 *stage = reinterpret_cast<uint2 *>(bp_smem + acc_bytes) + (size_t) wib*BP_NBUF*BP_G*BP_W;
	const uint32_t ngroups = (P.nb + BP_G - 1)/BP_G;
	const uint32_t rb0 = G.rb[G.s_lo];
	const uint32_t accA = (uint32_t) __cvta_generic_to_shared(acc);
	const uint32_t stageA = (uint32_t) __cvta_generic_to_shared(stage);
	for (;;)
		{
		uint32_t k = 0;
		if (lane == 0)
			k = atomicAdd(S.cursor, 1u);
		k = __shfl_sync(MB_FULL, k, 0);
		if (k >= P.cols_a)
			break;
		const uint32_t row = S.order[k];
		float *prow = P.post + (size_t) row*P.ld;
		for (uint32_t c = lane; c < P.cols_b; c += 32)
			acc[c] = prow[c];
		__syncwarp();
		for (uint32_t sl0 = 0; sl0 < G.s_n; sl0 += 32)
			{
			// which of the next 32 members have a residue in this column
			int32_t myPos = -1;
			if (sl0 + lane < G.s_n)
				myPos = P.col2pos_a[(size_t)(G.s_lo + sl0 + lane)*P.cols_a + row];
			uint32_t members = __ballot_sync(MB_FULL, myPos >= 0);
			while (members)
				{
				const uint32_t u = (uint32_t) __ffs(members) - 1;
				members &= members - 1;
				const int32_t pos = __shfl_sync(MB_FULL, myPos, u);
				const uint32_t s = G.s_lo + sl0 + u;
				const uint64_t base = (uint64_t)(G.rb[s] - rb0 + (uint32_t) pos)*P.nb;
				// issue the copy of group g into ring slot g % BP_NBUF
				auto issue = [&](uint32_t g)
					{
					if (g < ngroups)
						{
						const uint32_t t1 = g*BP_G;
						const uint32_t nt1 = min((uint32_t) BP_G, P.nb - t1);
						const uint4 *src = reinterpret_cast<const uint4 *>(G.slots + (base + t1)*BP_W);
						uint4 *dst = reinterpret_cast<uint4 *>(stage + (size_t)(g % BP_NBUF)*BP_G*BP_W);
						for (uint32_t q = lane; q < nt1*(BP_W/2); q += 32)
							__pipeline_memcpy_async(dst + q, src + q, 16);
						}
					__pipeline_commit();
					};
				issue(0);
				issue(1);
				for (uint32_t g = 0; g < ngroups; ++g)
					{
					const uint32_t t0 = g*BP_G;
					const uint32_t nt = min((uint32_t) BP_G, P.nb - t0);
					issue(g + 2);
					__pipeline_wait_prior(2);                          // group g has landed
					__syncwarp();
					const uint32_t curA = stageA + (g % BP_NBUF)*(BP_G*BP_W*8);
					// which steps of the group have entries at all (first entry of every slot)
					uint32_t rest = __ballot_sync(MB_FULL, lane < nt && lds_u2(curA + lane*(BP_W*8)).x != BP_END);
					// 1-deep software pipeline over the steps of the group: the next step's entry is fetched
					// from the stage before the current one is added
					uint2 v = make_uint2(BP_END, 0u);
					uint32_t l = 0;
					if (rest)
						{
						l = (uint32_t) __ffs(rest) - 1;
						if (lane < BP_W)
							v = lds_u2(curA + (l*BP_W + lane)*8);
						}
					while (rest)
						{
						rest &= rest - 1;
						uint2 v2 = make_uint2(BP_END, 0u);
						uint32_t l2 = 0;
						if (rest)
							{
							l2 = (uint32_t) __ffs(rest) - 1;
							if (lane < BP_W)
								v2 = lds_u2(curA + (l2*BP_W + lane)*8);
							}
						const bool isLong = __shfl_sync(MB_FULL, v.x, 0) == BP_LONG;
						if (!isLong)
							{
							if (v.x != BP_END)
								{
								const uint32_t a = accA + v.x*4;
								sts_f32(a, __fadd_rn(lds_f32(a), __uint_as_float(v.y)));        // += w1*w2*P, unit weights
								}
							}
						else if (lane == 0)
							{
							// rare: more than BP_W entries in the sparse row -> gather directly, still in order
							const uint32_t *ro;
							const mb200_entry *en;
							bp_operand(P, P.ids_a[s], P.ids_b[t0 + l], ro, en);
							const uint32_t *p2c = P.p2c_b + P.p2c_b_off[t0 + l];
							for (uint32_t e = ro[pos]; e < ro[pos + 1]; ++e)
								{
								const uint32_t a = accA + p2c[en[e].col]*4;
								sts_f32(a, __fadd_rn(lds_f32(a), en[e].p));
								}
							}
						__syncwarp();
						l = l2; v = v2;
						}
					__syncwarp();
					}
				__pipeline_wait_prior(0);
				}
			}
		for (uint32_t c = lane; c < P.cols_b; c += 32)
			prow[c] = acc[c];
		__syncwarp();
		}
	}

// =============================================================================================
// device-resident MSAs: position -> column maps
struct MsaJob
	{
	uint32_t na, nb;                         // members: ids[0..na) = A, ids[na..na+nb) = B
	const uint32_t *ids;
	const uint64_t *seqoff;                  // residue offset of every sequence (layout of p2c)
	const uint32_t *seqlen;
	uint32_t *p2c;                           // all sequences
	uint32_t *mark;                          // [2][cap]: column occupancy of A / B, then remap
	uint32_t cap;                            // >= old column counts
	uint32_t old_cols_a, old_cols_b;
	uint32_t *dims;                          // [0] cols_a, [1] cols_b after projection
	// filled for the maps kernel
	int32_t *c2p_a; uint32_t cols_a;         // [na][cols_a]
	uint32_t *p2c_b; const uint64_t *boff;   // concatenated
	// update
	const char *path; const uint32_t *plen;
	uint32_t *map;                           // [2][cap]: projected column -> column of the joined MSA
	};

__global__ void k_msa_identity(uint64_t total, const uint64_t *__restrict__ seqoff, uint32_t nseq, uint32_t *__restrict__ p2c)
	{
	// p2c[off[s] + i] = i : find s by binary search over the offsets
	for (uint64_t r = blockIdx.x*(uint64_t) blockDim.x + threadIdx.x; r < total; r += (uint64_t) gridDim.x*blockDim.x)
		{
		uint32_t lo = 0, hi = nseq;
		while (hi - lo > 1)
			{
			const uint32_t mid = (lo + hi) >> 1;
			if (seqoff[mid] <= r) lo = mid; else hi = mid;
			}
		p2c[r] = (uint32_t)(r - seqoff[lo]);
		}
	}

// grid (ceil(Lmax/256), na+nb)
__global__ void k_msa_mark(const MsaJob J)
	{
	const uint32_t m = blockIdx.y;
	const uint32_t s = J.ids[m];
	const uint32_t L = J.seqlen[s];
	uint32_t *mark = J.mark + (m < J.na ? 0 : J.cap);
	const uint32_t *p = J.p2c + J.seqoff[s];
	for (uint32_t i = blockIdx.x*blockDim.x + threadIdx.x; i < L; i += gridDim.x*blockDim.x)
		mark[p[i]] = 1u;
	}

// grid 2 (A, B), 1024 threads: exclusive scan of the occupancy marks -> projected column index
// (MultiSequence::Project drops all-gap columns, project.cpp:41-66)
__global__ void __launch_bounds__(1024)
k_msa_remap(const MsaJob J)
	{
	__shared__ uint32_t wsum[32];
	__shared__ uint32_t carry_s;
	const uint32_t which = blockIdx.x;
	uint32_t *mark = J.mark + which*J.cap;
	const uint32_t ncol = which == 0 ? J.old_cols_a : J.old_cols_b;
	const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	if (threadIdx.x == 0)
		carry_s = 0;
	__syncthreads();
	for (uint32_t c0 = 0; c0 < ncol; c0 += 1024)
		{
		const uint32_t c = c0 + threadIdx.x;
		const uint32_t f = c < ncol ? mark[c] : 0u;
		uint32_t v = f;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1)
			{
			const uint32_t t = __shfl_up_sync(MB_FULL, v, o);
			if (lane >= (uint32_t) o)
				v += t;
			}
		if (lane == 31)
			wsum[wid] = v;
		__syncthreads();
		uint32_t pre = carry_s;
		for (uint32_t w = 0; w < wid; ++w)
			pre += wsum[w];
		if (c < ncol)
			mark[c] = pre + v - f;                    // exclusive
		__syncthreads();
		if (threadIdx.x == 1023)
			carry_s = pre + v;
		__syncthreads();
		}
	if (threadIdx.x == 0)
		J.dims[which] = carry_s;
	}

// grid (ceil(Lmax/256), na+nb): col->pos of the projected A, pos->col of the projected B
__global__ void k_msa_maps(const MsaJob J)
	{
	const uint32_t m = blockIdx.y;
	const uint32_t s = J.ids[m];
	const uint32_t L = J.seqlen[s];
	const uint32_t *p = J.p2c + J.seqoff[s];
	if (m < J.na)
		{
		const uint32_t *remap = J.mark;
		int32_t *c2p = J.c2p_a + (size_t) m*J.cols_a;
		for (uint32_t i = blockIdx.x*blockDim.x + threadIdx.x; i < L; i += gridDim.x*blockDim.x)
			c2p[remap[p[i]]] = (int32_t) i;
		}
	else
		{
		const uint32_t *remap = J.mark + J.cap;
		uint32_t *dst = J.p2c_b + J.boff[m - J.na];
		for (uint32_t i = blockIdx.x*blockDim.x + threadIdx.x; i < L; i += gridDim.x*blockDim.x)
			dst[i] = remap[p[i]];
		}
	}

// one block: column of the joined MSA for every projected column of A ('B' or 'X' letters of the
// path, in order) and of B ('B' or 'Y') -- what Sequence::AddGapsPath does to a row (sequence.cpp:115-140)
__global__ void __launch_bounds__(1024)
k_msa_pathmap(const MsaJob J)
	{
	__shared__ uint32_t wsumA[32], wsumB[32];
	__shared__ uint32_t carryA, carryB;
	const uint32_t n = *J.plen;
	const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	if (threadIdx.x == 0)
		{
		carryA = 0; carryB = 0;
		}
	__syncthreads();
	for (uint32_t q0 = 0; q0 < n; q0 += 1024)
		{
		const uint32_t q = q0 + threadIdx.x;
		const char t = q < n ? J.path[q] : 0;
		const uint32_t fa = (t == 'B' || t == 'X') ? 1u : 0u;
		const uint32_t fb = (t == 'B' || t == 'Y') ? 1u : 0u;
		uint32_t va = fa, vb = fb;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1)
			{
			const uint32_t ta = __shfl_up_sync(MB_FULL, va, o);
			const uint32_t tb = __shfl_up_sync(MB_FULL, vb, o);
			if (lane >= (uint32_t) o)
				{
				va += ta; vb += tb;
				}
			}
		if (lane == 31)
			{
			wsumA[wid] = va; wsumB[wid] = vb;
			}
		__syncthreads();
		uint32_t pa = carryA, pb = carryB;
		for (uint32_t w = 0; w < wid; ++w)
			{
			pa += wsumA[w]; pb += wsumB[w];
			}
		if (fa)
			J.map[pa + va - 1] = q;
		if (fb)
			J.map[J.cap + pb + vb - 1] = q;
		__syncthreads();
		if (threadIdx.x == 1023)
			{
			carryA = pa + va; carryB = pb + vb;
			}
		__syncthreads();
		}
	}

// grid (ceil(Lmax/256), na+nb): p2c[s][i] = map[remap[p2c[s][i]]]
__global__ void k_msa_update(const MsaJob J)
	{
	const uint32_t m = blockIdx.y;
	const uint32_t s = J.ids[m];
	const uint32_t L = J.seqlen[s];
	uint32_t *p = J.p2c + J.seqoff[s];
	const uint32_t off = m < J.na ? 0 : J.cap;
	for (uint32_t i = blockIdx.x*blockDim.x + threadIdx.x; i < L; i += gridDim.x*blockDim.x)
		p[i] = J.map[off + J.mark[off + p[i]]];
	}

// ---------------------------------------------------------------------------------------------
// BuildPost for large joins: contributions bucketed by output cell.
//
// k_bp_apply keeps the reference's summation order by walking the (s,t) steps of an output row one
// after the other: a conserved column is a chain of |A| x |B| dependent steps at ~400 cycles each
// (one warp, ~30 instructions per step), most of a refinement join at 1000 sequences.  The
// order only matters PER CELL, so for large joins the contributions are written as (cell, value) pairs
// in (s, residue, t) order -- which is (s,t) order for every cell, a sequence has one residue per
// column -- bucketed by cell, and every run is summed front to back by one warp (coalesced loads, the
// ordered adds by shuffle: ~5 cycles per term instead of ~400).  Bucketing costs two radix passes, not
// four: the terms of a residue go to a position computed from a prefix sum over the residues ordered by
// (row, s), so the stream is already in (row, s, t) order when it is written; a STABLE sort on the column
// bits alone then leaves it in (col, row, s, t) order, i.e. every cell contiguous and in (s,t) order.
struct BpCells
	{
	uint32_t s_lo, s_n;          // batch of sequences of A
	const uint32_t *rb;          // [na+1] residues of A's members before member s
	const uint32_t *rowof;       // [residues of A] column of A's alignment = row of post
	const uint32_t *seqof;       // [residues of A] member of A that owns the residue
	uint32_t *cnt;               // [(residue of the batch) x nb] terms of the pair's sparse row
	uint64_t *eptr;              // [same] first entry of that sparse row: index into entries, bit 63 = transposed store
	const uint32_t *off;         // exclusive scan of cnt (one more entry than cnt)
	const uint32_t *base;        // [residue of the batch] first term of the residue in (row, s) order
	uint32_t colbits;            // key = row << colbits | col
	uint32_t *keys; float *vals; // [terms]
	};

__global__ void k_bp_rowof(const BuildPostParams P, const uint32_t *__restrict__ rb, uint32_t *__restrict__ rowof,
  uint32_t *__restrict__ seqof)
	{
	const uint32_t s = blockIdx.y;
	for (uint32_t c = blockIdx.x*blockDim.x + threadIdx.x; c < P.cols_a; c += gridDim.x*blockDim.x)
		{
		const int32_t pos = P.col2pos_a[(size_t) s*P.cols_a + c];
		if (pos >= 0)
			{
			rowof[rb[s] + (uint32_t) pos] = c;
			seqof[rb[s] + (uint32_t) pos] = s;
			}
		}
	}

// pass 1, one thread per (residue of the batch, member t of B): where the sparse row starts and how long it is
__global__ void k_bpc_count(const BuildPostParams P, const BpCells G)
	{
	const uint32_t r0 = G.rb[G.s_lo];
	const uint64_t total = (uint64_t)(G.rb[G.s_lo + G.s_n] - r0)*P.nb;
	for (uint64_t idx = blockIdx.x*(uint64_t) blockDim.x + threadIdx.x; idx < total; idx += (uint64_t) gridDim.x*blockDim.x)
		{
		const uint32_t t = (uint32_t)(idx % P.nb);
		const uint32_t r = r0 + (uint32_t)(idx/P.nb);
		const uint32_t s = G.seqof[r];
		const uint32_t pos = r - G.rb[s];
		const uint32_t a = P.ids_a[s], b = P.ids_b[t];
		uint32_t e0, e1;
		uint64_t ep;
		if (a < b)
			{
			const uint32_t q = mb_pair_index(P.n, a, b);
			const uint32_t *ro = P.rowoff + P.rowbase[q];
			e0 = ro[pos]; e1 = ro[pos + 1];
			ep = P.entbase[q] + e0;
			}
		else
			{
			const uint32_t q = mb_pair_index(P.n, b, a);
			const uint32_t *ro = P.troff + P.trbase[q];
			e0 = ro[pos]; e1 = ro[pos + 1];
			ep = (P.entbase[q] + e0) | (1ull << 63);
			}
		G.cnt[idx] = e1 - e0;
		G.eptr[idx] = ep;
		}
	}

// pass 2, eight lanes per (residue, t): the terms of the sparse row, one lane each
__global__ void k_bpc_emit(const BuildPostParams P, const BpCells G)
	{
	const uint32_t r0 = G.rb[G.s_lo];
	const uint64_t total = (uint64_t)(G.rb[G.s_lo + G.s_n] - r0)*P.nb;
	const uint32_t sub = threadIdx.x & 7;
	const uint64_t ngroups = ((uint64_t) gridDim.x*blockDim.x) >> 3;
	for (uint64_t idx = (blockIdx.x*(uint64_t) blockDim.x + threadIdx.x) >> 3; idx < total; idx += ngroups)
		{
		const uint32_t n = G.cnt[idx];
		if (n == 0)
			continue;
		const uint32_t t = (uint32_t)(idx % P.nb);
		const uint32_t rl = (uint32_t)(idx/P.nb);
		const uint64_t ep = G.eptr[idx];
		const mb200_entry *en = ((ep >> 63) ? P.trentries : P.entries) + (ep & ~(1ull << 63));
		const uint32_t *p2c = P.p2c_b + P.p2c_b_off[t];
		const uint32_t kbase = G.rowof[r0 + rl] << G.colbits;
		const uint32_t o = G.base[rl] + (G.off[idx] - G.off[(uint64_t) rl*P.nb]);
		for (uint32_t k = sub; k < n; k += 8)
			{
			const mb200_entry v = en[k];
			G.keys[o + k] = kbase | p2c[v.col];
			G.vals[o + k] = v.p;                               // w1*w2*P with unit weights (buildpostflat.cpp:60-70)
			}
		}
	}

// residues of the batch -> (row, local index), to be ordered by row
__global__ void k_bpc_reskeys(uint32_t nres, const uint32_t *__restrict__ rowof, uint32_t *__restrict__ keys, uint32_t *__restrict__ idx)
	{
	const uint32_t j = blockIdx.x*blockDim.x + threadIdx.x;
	if (j < nres)
		{ keys[j] = rowof[j]; idx[j] = j; }
	}
// terms of the residues in (row, s) order
__global__ void k_bpc_resterms(uint32_t nres, uint32_t nb, const uint32_t *__restrict__ perm, const uint32_t *__restrict__ off,
  uint32_t *__restrict__ nterms)
	{
	const uint32_t j = blockIdx.x*blockDim.x + threadIdx.x;
	if (j < nres)
		{
		const uint64_t r = perm[j];
		nterms[j] = off[(r + 1)*nb] - off[r*nb];
		}
	}
__global__ void k_bpc_resbase(uint32_t nres, const uint32_t *__restrict__ perm, const uint32_t *__restrict__ start, uint32_t *__restrict__ base)
	{
	const uint32_t j = blockIdx.x*blockDim.x + threadIdx.x;
	if (j < nres)
		base[perm[j]] = start[j];
	}

// post[cell] += the terms of the cell's run, front to back.  The adds of one cell are a dependent chain
// (4 cycles each); everything else must stay off that chain.  Runs are handed out longest first.
//  * long runs (>= BPC_LONG terms): one warp per run streams the terms through a shared-memory double buffer
//    with cp.async (the next BPC_CHUNK terms are in flight while lane 0 adds the current ones, four per
//    LDS.128) -- ~5 cycles per term.  Every lane adding shuffled terms is limited by one shuffle per cycle
//    per SM with a load exposed per 32 terms; one thread per run with 8 loads in flight pays an L2 round
//    trip per 8 terms on the longest runs (tens of thousands of terms).
//  * short runs: one thread per run; the lanes of a warp get runs of about the same length.
#define BPC_LONG 64
#define BPC_CHUNK 512
#define BPC_LWARPS 4
__global__ void __launch_bounds__(32*BPC_LWARPS)
k_bpc_sum_long(const uint32_t *__restrict__ perm, const uint32_t *__restrict__ ukeys, const uint32_t *__restrict__ ucnt,
  const uint32_t *__restrict__ uoff, uint32_t nlong, const float *__restrict__ vals, float *__restrict__ post, uint32_t colbits, uint32_t ld)
	{
	__shared__ __align__(16) float buf[BPC_LWARPS][2][BPC_CHUNK];
	const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
	const uint32_t j = blockIdx.x*BPC_LWARPS + wib;
	if (j >= nlong)
		return;
	const uint32_t r = perm[j];
	const uint32_t key = ukeys[r], n = ucnt[r];
	const float *v = vals + uoff[r];
	float *cell = post + (size_t)(key >> colbits)*ld + (key & ((1u << colbits) - 1u));
	float acc = *cell;
	const uint32_t nchunks = (n + BPC_CHUNK - 1)/BPC_CHUNK;
	auto issue = [&](uint32_t c)
		{
		if (c < nchunks)
			{
			const uint32_t b0 = c*BPC_CHUNK;
			float *dst = buf[wib][c & 1];
#pragma unroll
			for (uint32_t q = 0; q < BPC_CHUNK/32; ++q)
				{
				const uint32_t e = q*32 + lane;
				if (b0 + e < n)
					__pipeline_memcpy_async(dst + e, v + b0 + e, 4);
				}
			}
		__pipeline_commit();
		};
	issue(0);
	for (uint32_t c = 0; c < nchunks; ++c)
		{
		issue(c + 1);
		__pipeline_wait_prior(1);
		__syncwarp();
		if (lane == 0)
			{
			const uint32_t m = min((uint32_t) BPC_CHUNK, n - c*BPC_CHUNK);
			const float *src = buf[wib][c & 1];
			uint32_t i = 0;
			for (; i + 4 <= m; i += 4)
				{
				const float4 x = *reinterpret_cast<const float4 *>(src + i);
				acc = __fadd_rn(acc, x.x); acc = __fadd_rn(acc, x.y); acc = __fadd_rn(acc, x.z); acc = __fadd_rn(acc, x.w);
				}
			for (; i < m; ++i)
				acc = __fadd_rn(acc, src[i]);
			}
		__syncwarp();
		}
	if (lane == 0)
		*cell = acc;
	}

__global__ void __launch_bounds__(128)
k_bpc_sum_short(const uint32_t *__restrict__ perm, const uint32_t *__restrict__ ukeys, const uint32_t *__restrict__ ucnt,
  const uint32_t *__restrict__ uoff, uint32_t first, uint32_t nruns, const float *__restrict__ vals, float *__restrict__ post,
  uint32_t colbits, uint32_t ld)
	{
	const uint32_t j = first + blockIdx.x*blockDim.x + threadIdx.x;
	if (j >= nruns)
		return;
	const uint32_t r = perm[j];
	const uint32_t key = ukeys[r], n = ucnt[r];
	const float *v = vals + uoff[r];
	float *cell = post + (size_t)(key >> colbits)*ld + (key & ((1u << colbits) - 1u));
	float acc = *cell;
	uint32_t i = 0;
	for (; i + 8 <= n; i += 8)
		{
		float x[8];
#pragma unroll
		for (int u = 0; u < 8; ++u)
			x[u] = v[i + u];
#pragma unroll
		for (int u = 0; u < 8; ++u)
			acc = __fadd_rn(acc, x[u]);
		}
	for (; i < n; ++i)
		acc = __fadd_rn(acc, v[i]);
	*cell = acc;
	}
// number of leading elements >= bound in a descending array
__global__ void k_count_ge(const uint32_t *__restrict__ desc, uint32_t n, uint32_t bound, uint32_t *__restrict__ out)
	{
	uint32_t lo = 0, hi = n;                      // first index with desc[i] < bound
	while (lo < hi)
		{
		const uint32_t mid = (lo + hi) >> 1;
		if (desc[mid] >= bound) lo = mid + 1; else hi = mid;
		}
	*out = lo;
	}
__global__ void k_iota(uint32_t n, uint32_t *__restrict__ out)
	{
	const uint32_t j = blockIdx.x*blockDim.x + threadIdx.x;
	if (j < n)
		out[j] = j;
	}

// =============================================================================================
// host side
static inline size_t al256(size_t b) { return (b + 255)/256*256; }

// Geometry of one k_aln_wave problem (LX rows, LY columns) and the bytes of its pieces.  Every size is
// non-decreasing in LX and LY, and tb_smem can only turn on as they shrink.
struct AlnLayout
	{
	uint32_t LX, LY, ld, nstrips, nwarps, npass;
	bool tb_smem;                    // one CTA keeps the traceback in shared memory (tb_bytes of it)
	size_t dense_bytes;              // the matrix with its zero row above and AW_PAD_BOT rows below
	size_t tb_bytes;                 // traceback [LX][nstrips*32]
	size_t chan_bytes;               // hand-over channel [npass][LX+1], the done word in its last 256 bytes
	size_t path_bytes;
	size_t tb_carve() const { return tb_smem ? 256 : al256(tb_bytes); }
	// one problem as join_core carves it: dense | tb | channel | path | score | plen | the AlnProblem
	size_t bytes() const { return al256(dense_bytes) + tb_carve() + chan_bytes + al256(path_bytes) + 3*256; }
	};
static AlnLayout aln_layout(uint32_t LX, uint32_t LY, bool smem_ok)
	{
	AlnLayout L;
	L.LX = LX; L.LY = LY;
	L.ld = (LY + AW_C - 1)/AW_C*AW_C;
	L.nstrips = (LY + AW_W - 1)/AW_W;
	L.nwarps = std::min<uint32_t>(AW_MAXW, L.nstrips);
	L.npass = (L.nstrips + L.nwarps - 1)/L.nwarps;
	L.tb_bytes = (size_t) LX*L.nstrips*32;
	L.tb_smem = smem_ok && L.npass == 1 && L.tb_bytes <= 192*1024;
	L.dense_bytes = ((size_t) LX + 1 + AW_PAD_BOT)*L.ld*sizeof(float);
	L.chan_bytes = al256((size_t) L.npass*((size_t) LX + 1)*sizeof(uint2) + 256);
	L.path_bytes = (size_t) LX + LY + 16;
	return L;
	}
static void aln_place(const AlnLayout &L, char *dense, char *tb, char *chan, char *path, AlnProblem &q)
	{
	q.LX = L.LX; q.LY = L.LY; q.ld = L.ld;
	q.dense = (const float *) dense + L.ld;
	q.tb = (uint8_t *) tb;
	q.edge = (uint2 *) chan;
	q.done = (uint32_t *)(chan + L.chan_bytes - 256);
	q.path = path;
	}
// A join's members, A then B, and their copies at the front of ctx->d_join: ids, rb [na+1] (A's residues before
// member s), boff [nb] (B's member t in the concatenated pos->col maps), c2p [na][c2p cols], p2cb [btot]
struct JoinMembers
	{
	uint32_t na = 0, nb = 0, lmax = 0;
	uint64_t btot = 0;
	std::vector<uint32_t> ids, h_rb;
	std::vector<uint64_t> boff;
	uint32_t *d_ids = nullptr, *d_rb = nullptr, *d_p2cb = nullptr;
	uint64_t *d_boff = nullptr;
	int32_t *d_c2p = nullptr;
	};
// Checks the store and that every id is in range and listed once (A and B disjoint); builds the host maps
static int join_members(mb200_ctx *ctx, const char *who, uint32_t na, const uint32_t *ids_a, uint32_t nb, const uint32_t *ids_b,
  JoinMembers &M)
	{
	const int rc = mb_store_require(ctx, who, NEED_ALLPAIRS | FORM_TRANSPOSED);
	if (rc != MB200_OK)
		return rc;
	M.na = na; M.nb = nb;
	M.ids.resize(na + nb);
	M.h_rb.assign(na + 1, 0);
	M.boff.resize(nb);
	std::vector<uint8_t> member(ctx->nseq, 0);
	for (uint32_t m = 0; m < na + nb; ++m)
		{
		const uint32_t s = m < na ? ids_a[m] : ids_b[m - na];
		if (s >= ctx->nseq || member[s])
			return mb_fail(ctx, MB200_EINVAL, "%s: sequence id %u out of range, listed twice, or in both groups "
			  "(the reference asserts SMI_1 != SMI_2, buildpostflat.cpp:49)", who, s);
		member[s] = 1;
		M.ids[m] = s;
		M.lmax = std::max(M.lmax, ctx->h_len[s]);
		if (m < na)
			M.h_rb[m + 1] = M.h_rb[m] + ctx->h_len[s];
		else
			{
			M.boff[m - na] = M.btot;
			M.btot += ctx->h_len[s];
			}
		}
	return MB200_OK;
	}
// Carves the copies out of ctx->d_join, followed by `extra` bytes from `rest` on; uploads ids, boff and rb
static int upload_members(mb200_ctx *ctx, JoinMembers &M, uint32_t c2p_cols, size_t extra, JoinTimer &T, char *&rest)
	{
	const size_t na = M.na, nb = M.nb;
	ENSURE(ctx->d_join, al256((na + nb)*4) + al256((na + 1)*4) + al256(nb*8) + al256(na*c2p_cols*4) + al256(M.btot*4) + extra);
	char *p = (char *) ctx->d_join.p;
	M.d_ids = (uint32_t *) p;            p += al256((na + nb)*4);
	M.d_rb = (uint32_t *) p;             p += al256((na + 1)*4);
	M.d_boff = (uint64_t *) p;           p += al256(nb*8);
	M.d_c2p = (int32_t *) p;             p += al256(na*c2p_cols*4);
	M.d_p2cb = (uint32_t *) p;           p += al256(M.btot*4);
	rest = p;
	T.mark(5);
	CU(cudaMemcpyAsync(M.d_ids, M.ids.data(), (na + nb)*4, cudaMemcpyHostToDevice, ctx->stream));
	CU(cudaMemcpyAsync(M.d_boff, M.boff.data(), nb*8, cudaMemcpyHostToDevice, ctx->stream));
	CU(cudaMemcpyAsync(M.d_rb, M.h_rb.data(), (na + 1)*4, cudaMemcpyHostToDevice, ctx->stream));
	ctx->stats.h2d_bytes += (na + nb)*4 + nb*8;
	return MB200_OK;
	}
// A's members cut into batches of at most `budget` (residue of A, member of B) rows, at least one
// member each: batch b is members cuts[b] .. cuts[b+1]-1
struct MemberBatches
	{
	std::vector<uint32_t> cuts;
	uint64_t max_rows = 0;           // rows and residues of the largest batch
	uint32_t max_res = 0;
	};
static MemberBatches member_batches(const std::vector<uint32_t> &h_rb, uint32_t nb, uint64_t budget)
	{
	MemberBatches bt;
	bt.cuts.push_back(0);
	const uint32_t na = (uint32_t) h_rb.size() - 1;
	for (uint32_t s = 0; s < na; )
		{
		uint32_t e = s + 1;
		while (e < na && (uint64_t)(h_rb[e + 1] - h_rb[s])*nb <= budget)
			++e;
		bt.max_rows = std::max<uint64_t>(bt.max_rows, (uint64_t)(h_rb[e] - h_rb[s])*nb);
		bt.max_res = std::max(bt.max_res, h_rb[e] - h_rb[s]);
		bt.cuts.push_back(e);
		s = e;
		}
	return bt;
	}
// BuildPost with the terms bucketed by output cell (k_bpc_*).  Scratch: d_tmp (per residue and row of a batch),
// d_stage (per term), d_tmp2 (per run).  Reads back through ctx->h_pinned[4] (terms, then runs) and [5] (long runs).
static int buildpost_by_cell(mb200_ctx *ctx, const BuildPostParams &P, const uint32_t *d_rb, const std::vector<uint32_t> &h_rb,
  const MemberBatches &bt, uint32_t colbits, uint32_t rowbits, JoinTimer &T)
	{
	cudaStream_t st = ctx->stream;
	if (bt.max_rows >= 0x7ffffff0ull)
		return mb_fail(ctx, MB200_EOVERFLOW, "BuildPost batch of %llu rows", (unsigned long long) bt.max_rows);
	// d_tmp: rowof, seqof [residues] | cnt [max_rows+1] | off [max_rows+1] | eptr [max_rows] | 5 x [max_res] | nruns | cub scratch
	const size_t rowof_b = al256((size_t) h_rb[P.na]*4), rt_b = al256((size_t)(bt.max_rows + 1)*4), res_b = al256((size_t) bt.max_res*4);
	size_t scan_tb = 0, rsort_tb = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, scan_tb, (const uint32_t *) nullptr, (uint32_t *) nullptr, (int)(bt.max_rows + 1), st);
	cub::DeviceRadixSort::SortPairs(nullptr, rsort_tb, (const uint32_t *) nullptr, (uint32_t *) nullptr,
	  (const uint32_t *) nullptr, (uint32_t *) nullptr, (int) bt.max_res, 0, (int) rowbits, st);
	const size_t tb1 = al256(std::max(scan_tb, rsort_tb));
	ENSURE(ctx->d_tmp, 2*rowof_b + 4*rt_b + 5*res_b + 256 + tb1);
	char *tp = (char *) ctx->d_tmp.p;
	uint32_t *d_rowof = (uint32_t *) tp;             tp += rowof_b;
	uint32_t *d_seqof = (uint32_t *) tp;             tp += rowof_b;
	uint64_t *d_eptr = (uint64_t *) tp;              tp += 2*rt_b;
	uint32_t *d_cnt = (uint32_t *) tp;               tp += rt_b;
	uint32_t *d_off = (uint32_t *) tp;               tp += rt_b;
	uint32_t *d_rk = (uint32_t *) tp;                tp += res_b;      // row of the residue / sorted
	uint32_t *d_ri = (uint32_t *) tp;                tp += res_b;      // local index
	uint32_t *d_rk2 = (uint32_t *) tp;               tp += res_b;
	uint32_t *d_perm = (uint32_t *) tp;              tp += res_b;      // residues in (row, s) order
	uint32_t *d_base = (uint32_t *) tp;              tp += res_b;
	uint32_t *d_nruns = (uint32_t *) tp;             tp += 256;
	void *d_scratch1 = tp;
	k_bp_rowof<<<dim3((P.cols_a + 255)/256, P.na), 256, 0, st>>>(P, d_rb, d_rowof, d_seqof);
	CU(cudaGetLastError());
	const int sms = ctx->prop.multiProcessorCount;
	for (size_t b = 0; b + 1 < bt.cuts.size(); ++b)
		{
		T.tsub = now_s();
		BpCells C;
		C.s_lo = bt.cuts[b]; C.s_n = bt.cuts[b + 1] - bt.cuts[b];
		C.rb = d_rb; C.rowof = d_rowof; C.seqof = d_seqof; C.cnt = d_cnt; C.eptr = d_eptr; C.off = d_off; C.base = d_base;
		C.colbits = colbits;
		C.keys = nullptr; C.vals = nullptr;
		const uint32_t nres = h_rb[bt.cuts[b + 1]] - h_rb[bt.cuts[b]];
		const uint64_t rt = (uint64_t) nres*P.nb;
		const uint32_t gblocks = (uint32_t) std::min<uint64_t>((rt + 255)/256, (uint64_t) sms*32);
		const uint32_t rblocks = (nres + 255)/256;
		k_bpc_count<<<gblocks, 256, 0, st>>>(P, C);
		CU(cudaMemsetAsync(d_cnt + rt, 0, 4, st));
		size_t t0 = tb1;
		cub::DeviceScan::ExclusiveSum(d_scratch1, t0, (const uint32_t *) d_cnt, d_off, (int)(rt + 1), st);
		CU(cudaGetLastError());
		CU(cudaMemcpyAsync(ctx->h_pinned + 4, d_off + rt, 4, cudaMemcpyDeviceToHost, st));
		// residues ordered by (row, s): the input order is s-major, the sort is stable
		k_bpc_reskeys<<<rblocks, 256, 0, st>>>(nres, d_rowof + h_rb[bt.cuts[b]], d_rk, d_ri);
		t0 = tb1;
		cub::DeviceRadixSort::SortPairs(d_scratch1, t0, (const uint32_t *) d_rk, d_rk2, (const uint32_t *) d_ri, d_perm,
		  (int) nres, 0, (int) rowbits, st);
		k_bpc_resterms<<<rblocks, 256, 0, st>>>(nres, P.nb, d_perm, d_off, d_rk);           // d_rk: terms per residue, sorted order
		t0 = tb1;
		cub::DeviceScan::ExclusiveSum(d_scratch1, t0, (const uint32_t *) d_rk, d_rk2, (int) nres, st);
		k_bpc_resbase<<<rblocks, 256, 0, st>>>(nres, d_perm, d_rk2, d_base);
		CU(cudaGetLastError());
		CU(cudaStreamSynchronize(st));
		const uint64_t M = ctx->h_pinned[4];
		if (M >= 0x7fffffffull)
			return mb_fail(ctx, MB200_EOVERFLOW, "BuildPost batch of %llu terms", (unsigned long long) M);
		if (M == 0)
			continue;
		// d_stage: keys_in | vals_in | keys_out | vals_out | run offsets | cub scratch
		const size_t mb = al256((size_t) M*4);
		size_t sort_tb = 0, rle_tb = 0, scan2_tb = 0;
		cub::DeviceRadixSort::SortPairs(nullptr, sort_tb, (const uint32_t *) nullptr, (uint32_t *) nullptr,
		  (const float *) nullptr, (float *) nullptr, (int) M, 0, (int) colbits, st);
		cub::DeviceRunLengthEncode::Encode(nullptr, rle_tb, (const uint32_t *) nullptr, (uint32_t *) nullptr, (uint32_t *) nullptr,
		  (uint32_t *) nullptr, (int) M, st);
		cub::DeviceScan::ExclusiveSum(nullptr, scan2_tb, (const uint32_t *) nullptr, (uint32_t *) nullptr, (int) M, st);
		const size_t tb = std::max(sort_tb, std::max(rle_tb, scan2_tb));
		ENSURE(ctx->d_stage, 5*mb + al256(tb) + 256);
		char *sp = (char *) ctx->d_stage.p;
		uint32_t *keys_in = (uint32_t *) sp;              float *vals_in = (float *)(sp + mb);
		uint32_t *keys_out = (uint32_t *)(sp + 2*mb);     float *vals_out = (float *)(sp + 3*mb);
		uint32_t *uoff = (uint32_t *)(sp + 4*mb);
		void *scratch2 = sp + 5*mb;
		C.keys = keys_in; C.vals = vals_in;
		T.sub(0);
		k_bpc_emit<<<(uint32_t) std::min<uint64_t>((rt*8 + 255)/256, (uint64_t) sms*32), 256, 0, st>>>(P, C);
		CU(cudaGetLastError());
		T.sub(1);
		T.mark(1);
		// stable sort on the column bits only: (row, s, t) order survives inside every column
		size_t t1 = sort_tb;
		cub::DeviceRadixSort::SortPairs(scratch2, t1, (const uint32_t *) keys_in, keys_out, (const float *) vals_in, vals_out,
		  (int) M, 0, (int) colbits, st);
		T.sub(2);
		// runs of equal cells: unique keys and lengths reuse the input buffers
		uint32_t *ukeys = keys_in, *ucnt = (uint32_t *) vals_in;
		size_t t2 = rle_tb;
		cub::DeviceRunLengthEncode::Encode(scratch2, t2, (const uint32_t *) keys_out, ukeys, ucnt, d_nruns, (int) M, st);
		CU(cudaGetLastError());
		CU(cudaMemcpyAsync(ctx->h_pinned + 4, d_nruns, 4, cudaMemcpyDeviceToHost, st));
		CU(cudaStreamSynchronize(st));
		const uint32_t nruns = ctx->h_pinned[4];
		size_t t3 = scan2_tb;
		cub::DeviceScan::ExclusiveSum(scratch2, t3, (const uint32_t *) ucnt, uoff, (int) nruns, st);
		// runs by descending length (d_tmp2: counts out | index in | index out | cub scratch)
		size_t lsort_tb = 0;
		cub::DeviceRadixSort::SortPairsDescending(nullptr, lsort_tb, (const uint32_t *) nullptr, (uint32_t *) nullptr,
		  (const uint32_t *) nullptr, (uint32_t *) nullptr, (int) nruns, 0, 32, st);
		const size_t nrb = al256((size_t) nruns*4);
		ENSURE(ctx->d_tmp2, 3*nrb + al256(lsort_tb));
		uint32_t *d_lc = (uint32_t *) ctx->d_tmp2.p;
		uint32_t *d_li = (uint32_t *)((char *) ctx->d_tmp2.p + nrb);
		uint32_t *d_lperm = (uint32_t *)((char *) ctx->d_tmp2.p + 2*nrb);
		void *d_lscratch = (char *) ctx->d_tmp2.p + 3*nrb;
		k_iota<<<(nruns + 255)/256, 256, 0, st>>>(nruns, d_li);
		cub::DeviceRadixSort::SortPairsDescending(d_lscratch, lsort_tb, (const uint32_t *) ucnt, d_lc, (const uint32_t *) d_li, d_lperm,
		  (int) nruns, 0, 32, st);
		k_count_ge<<<1, 1, 0, st>>>(d_lc, nruns, BPC_LONG, d_nruns + 1);
		CU(cudaMemcpyAsync(ctx->h_pinned + 5, d_nruns + 1, 4, cudaMemcpyDeviceToHost, st));
		CU(cudaStreamSynchronize(st));
		const uint32_t nlong = ctx->h_pinned[5];
		T.sub(3);
		if (nlong > 0)
			k_bpc_sum_long<<<(nlong + BPC_LWARPS - 1)/BPC_LWARPS, 32*BPC_LWARPS, 0, st>>>(d_lperm, ukeys, ucnt, uoff, nlong, vals_out,
			  P.post, colbits, P.ld);
		if (nruns > nlong)
			k_bpc_sum_short<<<(nruns - nlong + 127)/128, 128, 0, st>>>(d_lperm, ukeys, ucnt, uoff, nlong, nruns, vals_out, P.post, colbits, P.ld);
		CU(cudaGetLastError());
		T.sub(4);
		T.mark(2);
		ctx->stats.kernel_launches += 14;
		}
	return MB200_OK;
	}
// Shared memory of one k_bp_apply block: the accumulator rows of BP_WARPS warps + their cp.async buffers.
// The ordered row walk runs only where this fits (cols_b <= 12544).
#define BP_SMEM_MAX (220*1024)
static size_t bp_row_smem(uint32_t cols_b)
	{
	return (((size_t) BP_WARPS*cols_b*sizeof(float) + 15) & ~(size_t) 15) + (size_t) BP_WARPS*BP_NBUF*BP_G*BP_W*sizeof(uint2);
	}
// BuildPost as an ordered walk over the rows (k_bp_gather / k_bp_apply).  Scratch: d_stage, d_tmp2.  No read-backs.
static int buildpost_by_row(mb200_ctx *ctx, const BuildPostParams &P, const uint32_t *d_rb, const std::vector<uint32_t> &h_rb,
  const MemberBatches &bt, JoinTimer &T)
	{
	cudaStream_t st = ctx->stream;
	const uint32_t cols_a = P.cols_a;
	const size_t acc_smem = bp_row_smem(P.cols_b);
	if (acc_smem > BP_SMEM_MAX)
		return mb_fail(ctx, MB200_EOVERFLOW, "alignment with %u columns too wide for the BuildPost kernel", P.cols_b);
	ENSURE(ctx->d_stage, bt.max_rows*BP_W*sizeof(uint2) + 256);
	BpStage G;
	G.slots = (uint2 *) ctx->d_stage.p;
	G.rb = d_rb;
	// row order: heaviest first (weights and the sorted ids live in d_tmp2 next to the cub scratch)
	size_t sort_tb = 0;
	cub::DeviceRadixSort::SortPairsDescending(nullptr, sort_tb, (const uint32_t *) nullptr, (uint32_t *) nullptr,
	  (const uint32_t *) nullptr, (uint32_t *) nullptr, (int) cols_a, 0, 32, st);
	const size_t wbytes = al256((size_t) cols_a*4);
	ENSURE(ctx->d_tmp2, 4*wbytes + 256 + sort_tb);
	uint32_t *d_w = (uint32_t *) ctx->d_tmp2.p;
	uint32_t *d_id = (uint32_t *)((char *) ctx->d_tmp2.p + wbytes);
	uint32_t *d_w2 = (uint32_t *)((char *) ctx->d_tmp2.p + 2*wbytes);
	uint32_t *d_order = (uint32_t *)((char *) ctx->d_tmp2.p + 3*wbytes);
	uint32_t *d_cursor = (uint32_t *)((char *) ctx->d_tmp2.p + 4*wbytes);
	void *d_sortscratch = (char *) ctx->d_tmp2.p + 4*wbytes + 256;
	k_bp_weight<<<(cols_a + 255)/256, 256, 0, st>>>(P, d_w, d_id);
	cub::DeviceRadixSort::SortPairsDescending(d_sortscratch, sort_tb, d_w, d_w2, d_id, d_order, (int) cols_a, 0, 32, st);
	CU(cudaGetLastError());
	BpSched S;
	S.order = d_order;
	S.cursor = d_cursor;
	CU(cudaFuncSetAttribute(k_bp_apply, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) acc_smem));
	int occ = 0;
	CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_bp_apply, 32*BP_WARPS, acc_smem));
	const uint32_t ablocks = std::max<uint32_t>(1, std::min<uint32_t>((cols_a + BP_WARPS - 1)/BP_WARPS,
	  (uint32_t) std::max(occ, 1)*ctx->prop.multiProcessorCount));
	for (size_t b = 0; b + 1 < bt.cuts.size(); ++b)
		{
		G.s_lo = bt.cuts[b];
		G.s_n = bt.cuts[b + 1] - bt.cuts[b];
		const uint64_t total = (uint64_t)(h_rb[bt.cuts[b + 1]] - h_rb[bt.cuts[b]])*P.nb;
		const uint32_t gblocks = (uint32_t) std::min<uint64_t>((total + 255)/256, (uint64_t) ctx->prop.multiProcessorCount*32);
		k_bp_gather<<<gblocks, 256, 0, st>>>(P, G);
		T.mark(1);
		CU(cudaMemsetAsync(d_cursor, 0, 4, st));
		k_bp_apply<<<ablocks, 32*BP_WARPS, acc_smem, st>>>(P, G, S);
		T.mark(2);
		ctx->stats.kernel_launches += 2;
		}
	ctx->stats.kernel_launches += 2;
	CU(cudaGetLastError());
	return MB200_OK;
	}

// BuildPost + decoding DP of a join whose members and maps are on the device.  Fills pr (the matrix,
// path, score and plen stay on the device) and does NOT synchronise.
static int join_core(mb200_ctx *ctx, const JoinMembers &M, uint32_t cols_a, uint32_t cols_b, char *scratch, size_t scratch_bytes,
  AlnProblem &pr, JoinTimer &T)
	{
	cudaStream_t st = ctx->stream;
	const uint32_t na = M.na, nb = M.nb;
	const AlnLayout L = aln_layout(cols_a, cols_b, true);
	if (L.bytes() > scratch_bytes)
		return mb_fail(ctx, MB200_EINVAL, "join scratch too small");
	char *tb = scratch + al256(L.dense_bytes), *chan = tb + L.tb_carve(), *path = chan + L.chan_bytes;
	char *tail = path + al256(L.path_bytes);                       // score | plen | the AlnProblem
	aln_place(L, scratch, tb, chan, path, pr);
	pr.score = (float *) tail; pr.plen = (uint32_t *)(tail + 256);
	AlnProblem *d_prob = (AlnProblem *)(tail + 512);
	CU(cudaMemsetAsync(scratch, 0, L.dense_bytes, st));

	BuildPostParams P;
	P.n = ctx->nseq; P.na = na; P.nb = nb; P.cols_a = cols_a; P.cols_b = cols_b; P.ld = L.ld;
	P.ids_a = M.d_ids; P.ids_b = M.d_ids + na; P.col2pos_a = M.d_c2p; P.p2c_b = M.d_p2cb; P.p2c_b_off = M.d_boff;
	P.rowbase = (const uint64_t *) ctx->d_rowbase.p; P.rowoff = (const uint32_t *) ctx->d_rowoff.p;
	P.entries = (const mb200_entry *) ctx->d_entries.p;
	P.trbase = (const uint64_t *) ctx->d_tr_rowbase.p; P.troff = (const uint32_t *) ctx->d_tr_rowoff.p;
	P.trentries = (const mb200_entry *) ctx->d_tr_entries.p;
	P.entbase = (const uint64_t *) ctx->d_entbase.p;
	P.post = (float *) pr.dense;
	// large joins: bucket the contributions by cell (see k_bpc_*); small ones: ordered row walk (k_bp_apply)
	const char *ev_sort = getenv("MB200_BP_SORT_MIN");             // tuning hook: (residues of A) x |B| from which to sort
	const long long sort_min = ev_sort ? atoll(ev_sort) : 1000000ll;
	uint32_t colbits = 1, rowbits = 1;
	while ((1u << colbits) < cols_b)
		++colbits;
	while ((1u << rowbits) < cols_a)
		++rowbits;
	// a join too wide for the row walk's shared-memory accumulator takes the by-cell route whatever its size
	const bool by_cell = ((uint64_t) M.h_rb[na]*nb >= (uint64_t) sort_min || bp_row_smem(cols_b) > BP_SMEM_MAX)
	  && colbits + rowbits <= 32 && na <= 65535;
	// batches of A's members: by cell at most ~16M (residue, t) rows; by row, the staging area (one slot
	// per residue of the batch and member of B) stays below ~2 GB
	const MemberBatches bt = member_batches(M.h_rb, nb, by_cell ? 16ull << 20 : (2048ull << 20)/(BP_W*sizeof(uint2)));
	const int rc = by_cell ? buildpost_by_cell(ctx, P, M.d_rb, M.h_rb, bt, colbits, rowbits, T)
	  : buildpost_by_row(ctx, P, M.d_rb, M.h_rb, bt, T);
	if (rc != MB200_OK)
		return rc;

	if (L.npass > 1)
		CU(cudaMemsetAsync(chan, 0, L.chan_bytes, st));
	CU(cudaMemcpyAsync(d_prob, &pr, sizeof pr, cudaMemcpyHostToDevice, st));
	if (L.tb_smem)
		{
		CU(cudaFuncSetAttribute(k_aln_wave<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(L.tb_bytes, 16)));
		k_aln_wave<true><<<1, 32*L.nwarps, L.tb_bytes, st>>>(d_prob);
		}
	else
		k_aln_wave<false><<<dim3(1, L.npass), 32*L.nwarps, 0, st>>>(d_prob);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches++;
	const double g1 = g_t[1], g2 = g_t[2], g3 = g_t[3];
	T.mark(3);
	if (g_trace_level >= 2 && na + nb >= 64)
		fprintf(stderr, "[mb200 join] %u x %u seqs, %u x %u cols, %zu batch(es): DP %.2f ms (BuildPost totals so far: gather %.1f ms apply %.1f ms)\n",
		  na, nb, cols_a, cols_b, bt.cuts.size() - 1, 1e3*(g_t[3] - g3), 1e3*g1, 1e3*g2);
	return MB200_OK;
	}

extern "C" {

int mb200_align_pairs(mb200_ctx *ctx, uint32_t n, const uint32_t *store_pairs, char *paths_out,
  const uint64_t *path_off, float *scores_out)
	{
	if (!ctx || n == 0 || !store_pairs || !paths_out || !path_off || !scores_out)
		return mb_fail(ctx, MB200_EINVAL, "mb200_align_pairs: bad argument");
	int rc = mb_store_require(ctx, "mb200_align_pairs", FORM_PACKED);
	if (rc != MB200_OK)
		return rc;
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	const uint32_t np = (uint32_t) ctx->h_px.size();
	std::vector<AlnProblem> probs(n);
	std::vector<DensifyJob> jobs(n);
	std::vector<AlnLayout> lay(n);
	uint64_t dense_total = 0, tb_total = 0, edge_total = 0;
	const uint64_t path_total = path_off[n];
	uint32_t lxmax = 0, maxstrips = 1;
	for (uint32_t k = 0; k < n; ++k)
		{
		const uint32_t sp = store_pairs[k];
		if (sp >= np)
			return mb_fail(ctx, MB200_EINVAL, "store pair %u out of range", sp);
		const uint32_t LX = ctx->h_len[ctx->h_px[sp]], LY = ctx->h_len[ctx->h_py[sp]];
		if (path_off[k + 1] < path_off[k] + LX + LY + 1)
			return mb_fail(ctx, MB200_EINVAL, "path_off[%u..%u] leaves less than LX+LY+1 bytes", k, k + 1);
		// the batch launch below keeps every traceback in global memory; with nwarps = min(AW_MAXW, nstrips)
		// each problem's npass is the one k_aln_wave derives from the launch's min(AW_MAXW, maxstrips) warps
		lay[k] = aln_layout(LX, LY, false);
		dense_total += al256(lay[k].dense_bytes);
		tb_total += lay[k].tb_carve();
		edge_total += lay[k].chan_bytes;
		lxmax = std::max(lxmax, LX);
		maxstrips = std::max(maxstrips, lay[k].nstrips);
		}
	const size_t need = dense_total + tb_total + edge_total + al256(path_total + 16) + al256(n*sizeof(float))
	  + al256(n*sizeof(AlnProblem)) + al256(n*sizeof(DensifyJob));
	ENSURE(ctx->d_join, need);
	char *p = (char *) ctx->d_join.p;
	char *d_dense = p;               p += dense_total;
	char *d_tb = p;                  p += tb_total;
	char *d_edge = p;                p += edge_total;
	char *d_paths = p;               p += al256(path_total + 16);
	float *d_scores = (float *) p;   p += al256(n*sizeof(float));
	AlnProblem *d_probs = (AlnProblem *) p;   p += al256(n*sizeof(AlnProblem));
	DensifyJob *d_jobs = (DensifyJob *) p;
	uint64_t od = 0, ot = 0, oe = 0;
	for (uint32_t k = 0; k < n; ++k)
		{
		const uint32_t sp = store_pairs[k];
		const AlnLayout &L = lay[k];
		AlnProblem &q = probs[k];
		aln_place(L, d_dense + od, d_tb + ot, d_edge + oe, d_paths + path_off[k], q);
		q.score = d_scores + k;
		q.plen = nullptr;
		DensifyJob &j = jobs[k];
		j.rowoff = (const uint32_t *) ctx->d_rowoff.p + ctx->h_rowbase[sp];
		uint64_t e_lo = 0, e_hi = 0;
		mb_store_entry_range(ctx, sp, sp + 1, &e_lo, &e_hi);
		j.entries = (const mb200_entry *) ctx->d_entries.p + e_lo;
		j.dense = (float *) q.dense;
		j.LX = L.LX; j.ld = L.ld;
		od += al256(L.dense_bytes);
		ot += L.tb_carve();
		oe += L.chan_bytes;
		}
	CU(cudaMemsetAsync(d_dense, 0, dense_total, st));
	CU(cudaMemcpyAsync(d_probs, probs.data(), n*sizeof(AlnProblem), cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(d_jobs, jobs.data(), n*sizeof(DensifyJob), cudaMemcpyHostToDevice, st));
	const uint64_t warps = (uint64_t) n*lxmax;
	k_densify<<<(uint32_t)((warps*32 + 255)/256), 256, 0, st>>>(d_jobs, n, lxmax);
	CU(cudaGetLastError());
	{
	const uint32_t bw = std::min<uint32_t>(AW_MAXW, maxstrips);
	CU(cudaMemsetAsync(d_edge, 0, edge_total, st));
	k_aln_wave<false><<<dim3(n, (maxstrips + bw - 1)/bw), 32*bw, 0, st>>>(d_probs);
	}
	CU(cudaGetLastError());
	ctx->stats.kernel_launches += 2;
	CU(cudaMemcpyAsync(paths_out, d_paths, path_total, cudaMemcpyDeviceToHost, st));
	CU(cudaMemcpyAsync(scores_out, d_scores, n*sizeof(float), cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));
	ctx->stats.d2h_bytes += path_total + n*sizeof(float);
	return MB200_OK;
	}

int mb200_align_groups(mb200_ctx *ctx, uint32_t na, const uint32_t *ids_a, const uint32_t *pos2col_a, uint32_t cols_a,
  uint32_t nb, const uint32_t *ids_b, const uint32_t *pos2col_b, uint32_t cols_b,
  char *path_out, float *score_out, float *post_out)
	{
	if (!ctx || na == 0 || nb == 0 || !ids_a || !ids_b || !pos2col_a || !pos2col_b || !path_out || cols_a == 0 || cols_b == 0)
		return mb_fail(ctx, MB200_EINVAL, "mb200_align_groups: bad argument");
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	JoinMembers M;
	int rc = join_members(ctx, "mb200_align_groups", na, ids_a, nb, ids_b, M);
	if (rc != MB200_OK)
		return rc;
	JoinTimer T(st);
	// host-side index maps (tiny): col->pos for A, concatenated pos->col for B; validated here
	std::vector<int32_t> c2p((size_t) na*cols_a, -1);
	for (uint32_t s = 0; s < na; ++s)
		for (uint32_t i = 0; i < M.h_rb[s + 1] - M.h_rb[s]; ++i)
			{
			const uint32_t c = pos2col_a[M.h_rb[s] + i];
			if (c >= cols_a)
				return mb_fail(ctx, MB200_EINVAL, "mb200_align_groups: group A pos2col out of range");
			c2p[(size_t) s*cols_a + c] = (int32_t) i;
			}
	for (uint64_t i = 0; i < M.btot; ++i)
		if (pos2col_b[i] >= cols_b)
			return mb_fail(ctx, MB200_EINVAL, "mb200_align_groups: group B pos2col out of range");
	const size_t jsz = aln_layout(cols_a, cols_b, true).bytes();
	char *scratch = nullptr;
	rc = upload_members(ctx, M, cols_a, jsz, T, scratch);
	if (rc != MB200_OK)
		return rc;
	CU(cudaMemcpyAsync(M.d_c2p, c2p.data(), c2p.size()*4, cudaMemcpyHostToDevice, st));
	CU(cudaMemcpyAsync(M.d_p2cb, pos2col_b, M.btot*4, cudaMemcpyHostToDevice, st));
	ctx->stats.h2d_bytes += c2p.size()*4 + M.btot*4;
	T.mark(0);
	AlnProblem pr;
	rc = join_core(ctx, M, cols_a, cols_b, scratch, jsz, pr, T);
	if (rc != MB200_OK)
		return rc;
	CU(cudaMemcpyAsync(path_out, pr.path, cols_a + cols_b + 1, cudaMemcpyDeviceToHost, st));
	if (score_out)
		CU(cudaMemcpyAsync(score_out, pr.score, sizeof(float), cudaMemcpyDeviceToHost, st));
	if (post_out)
		CU(cudaMemcpy2DAsync(post_out, (size_t) cols_b*sizeof(float), pr.dense, (size_t) pr.ld*sizeof(float),
		  (size_t) cols_b*sizeof(float), cols_a, cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));
	T.mark(5);
	ctx->stats.d2h_bytes += cols_a + cols_b + 1 + 4 + (post_out ? (size_t) cols_a*cols_b*4 : 0);
	return MB200_OK;
	}

// ---------------------------------------------------------------------------------------------
// device-resident MSAs
int mb200_msa_reset(mb200_ctx *ctx)
	{
	if (!ctx || ctx->nseq == 0)
		return mb_fail(ctx, MB200_EINVAL, "mb200_msa_reset: call mb200_set_seqs first");
	cudaSetDevice(ctx->device);
	const uint64_t total = ctx->h_off[ctx->nseq];
	ENSURE(ctx->d_p2c, total*sizeof(uint32_t) + 16);
	k_msa_identity<<<ctx->prop.multiProcessorCount*4, 256, 0, ctx->stream>>>(total, (const uint64_t *) ctx->d_seqoff.p,
	  ctx->nseq, (uint32_t *) ctx->d_p2c.p);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches++;
	CU(cudaStreamSynchronize(ctx->stream));
	ctx->h_msa_cols.assign(ctx->h_len.begin(), ctx->h_len.end());     // every sequence alone (progalnflat.cpp:79-85)
	ctx->msa_valid = true;
	return MB200_OK;
	}

// ctx->h_pinned: words 0-1 projected column counts, 2 path length, 3 score (4-5: buildpost_by_cell)
int mb200_msa_join(mb200_ctx *ctx, uint32_t na, const uint32_t *ids_a, uint32_t nb, const uint32_t *ids_b,
  uint32_t *cols_out, float *score_out, char *path_out, uint32_t path_cap)
	{
	if (!ctx || na == 0 || nb == 0 || !ids_a || !ids_b)
		return mb_fail(ctx, MB200_EINVAL, "mb200_msa_join: bad argument");
	if (!ctx->msa_valid)
		return mb_fail(ctx, MB200_EINVAL, "mb200_msa_join: call mb200_msa_reset first");
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	// members: every id once; all of A in one MSA (same column count), all of B in one MSA
	JoinMembers M;
	int rc = join_members(ctx, "mb200_msa_join", na, ids_a, nb, ids_b, M);
	if (rc != MB200_OK)
		return rc;
	JoinTimer T(st);
	const uint32_t old_a = ctx->h_msa_cols[ids_a[0]], old_b = ctx->h_msa_cols[ids_b[0]];
	for (uint32_t m = 0; m < na + nb; ++m)
		if (ctx->h_msa_cols[M.ids[m]] != (m < na ? old_a : old_b))
			return mb_fail(ctx, MB200_EINVAL, "mb200_msa_join: group %c members are not in one MSA", m < na ? 'A' : 'B');
	const uint32_t cap = std::max(old_a, old_b);
	// after the members: mark/remap [2][cap], map [2][cap], dims, join scratch.  c2p and the join scratch are sized
	// for the old column counts: the projected ones are no larger, and no size grows as they shrink
	const size_t jsz = aln_layout(old_a, old_b, true).bytes();
	char *p = nullptr;
	rc = upload_members(ctx, M, old_a, 2*al256(2*(size_t) cap*4) + 256 + jsz, T, p);
	if (rc != MB200_OK)
		return rc;
	uint32_t *d_mark = (uint32_t *) p;               p += al256(2*(size_t) cap*4);
	uint32_t *d_map = (uint32_t *) p;                p += al256(2*(size_t) cap*4);
	uint32_t *d_dims = (uint32_t *) p;               p += 256;
	CU(cudaMemsetAsync(d_mark, 0, 2*(size_t) cap*4, st));
	MsaJob J;
	memset(&J, 0, sizeof J);
	J.na = na; J.nb = nb; J.ids = M.d_ids;
	J.seqoff = (const uint64_t *) ctx->d_seqoff.p; J.seqlen = (const uint32_t *) ctx->d_seqlen.p;
	J.p2c = (uint32_t *) ctx->d_p2c.p;
	J.mark = d_mark; J.cap = cap; J.old_cols_a = old_a; J.old_cols_b = old_b; J.dims = d_dims;
	J.map = d_map;
	const dim3 mgrid((M.lmax + 255)/256, na + nb);
	k_msa_mark<<<mgrid, 256, 0, st>>>(J);
	k_msa_remap<<<2, 1024, 0, st>>>(J);
	CU(cudaGetLastError());
	CU(cudaMemcpyAsync(ctx->h_pinned, d_dims, 8, cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));
	const uint32_t cols_a = ctx->h_pinned[0], cols_b = ctx->h_pinned[1];
	if (cols_a == 0 || cols_b == 0 || cols_a > old_a || cols_b > old_b)
		return mb_fail(ctx, MB200_EINVAL, "mb200_msa_join: projection gave %u x %u columns", cols_a, cols_b);
	J.c2p_a = M.d_c2p; J.cols_a = cols_a; J.p2c_b = M.d_p2cb; J.boff = M.d_boff;
	CU(cudaMemsetAsync(M.d_c2p, 0xff, (size_t) na*cols_a*4, st));
	k_msa_maps<<<mgrid, 256, 0, st>>>(J);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches += 3;
	T.mark(0);
	AlnProblem pr;
	rc = join_core(ctx, M, cols_a, cols_b, p, jsz, pr, T);
	if (rc != MB200_OK)
		return rc;
	J.path = pr.path; J.plen = pr.plen;
	k_msa_pathmap<<<1, 1024, 0, st>>>(J);
	k_msa_update<<<mgrid, 256, 0, st>>>(J);
	CU(cudaGetLastError());
	ctx->stats.kernel_launches += 2;
	CU(cudaMemcpyAsync(ctx->h_pinned + 2, pr.plen, 4, cudaMemcpyDeviceToHost, st));
	CU(cudaMemcpyAsync(ctx->h_pinned + 3, pr.score, 4, cudaMemcpyDeviceToHost, st));
	if (path_out)
		{
		if (path_cap < cols_a + cols_b + 1)
			return mb_fail(ctx, MB200_EINVAL, "mb200_msa_join: path buffer of %u bytes, need %u", path_cap, cols_a + cols_b + 1);
		CU(cudaMemcpyAsync(path_out, pr.path, cols_a + cols_b + 1, cudaMemcpyDeviceToHost, st));
		}
	CU(cudaStreamSynchronize(st));
	T.mark(4);
	const uint32_t newcols = ctx->h_pinned[2];
	for (uint32_t m = 0; m < na + nb; ++m)
		ctx->h_msa_cols[M.ids[m]] = newcols;
	if (cols_out)
		*cols_out = newcols;
	if (score_out)
		memcpy(score_out, ctx->h_pinned + 3, 4);
	ctx->stats.d2h_bytes += 16 + (path_out ? cols_a + cols_b + 1 : 0);
	return MB200_OK;
	}

int mb200_msa_export(mb200_ctx *ctx, uint32_t n, const uint32_t *ids, uint32_t *pos2col_out, uint32_t *cols_out)
	{
	if (!ctx || n == 0 || !ids || !pos2col_out)
		return mb_fail(ctx, MB200_EINVAL, "mb200_msa_export: bad argument");
	if (!ctx->msa_valid)
		return mb_fail(ctx, MB200_EINVAL, "mb200_msa_export: call mb200_msa_reset first");
	cudaSetDevice(ctx->device);
	uint64_t off = 0;
	for (uint32_t k = 0; k < n; ++k)
		{
		const uint32_t s = ids[k];
		if (s >= ctx->nseq)
			return mb_fail(ctx, MB200_EINVAL, "mb200_msa_export: sequence id out of range");
		CU(cudaMemcpyAsync(pos2col_out + off, (const uint32_t *) ctx->d_p2c.p + ctx->h_off[s], ctx->h_len[s]*sizeof(uint32_t),
		  cudaMemcpyDeviceToHost, ctx->stream));
		off += ctx->h_len[s];
		if (cols_out)
			cols_out[k] = ctx->h_msa_cols[s];
		}
	CU(cudaStreamSynchronize(ctx->stream));
	ctx->stats.d2h_bytes += off*4;
	return MB200_OK;
	}

} // extern "C"
