// common.cuh -- shared device helpers and parameter blocks for libmuscle_b200 (sm_90a).
//
// Arithmetic contract (SURVEY.md section 7 hard part 1, Appendix A): every fp32 operation on the
// pair-HMM path is an explicit round-to-nearest add/mul (__fadd_rn/__fmul_rn are never fused into
// FMA) in the reference's association order, so Forward/Backward/total are bit-identical to the
// reference built with -ffp-contract=off.  The file is also compiled with -fmad=false.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/muscle_b200.h"

#define MB_FULL 0xffffffffu
#define MB_LOG_ZERO (-2e20f)          // scoretype.h:89
#define MB_MAX_K 64                    // residue classes the smem tables can hold
#define MB_CAP MB200_MAX_ROW_NNZ       // candidate entries per posterior row
#define MB_WARPS_PER_BLOCK 4            // posterior kernel: warps (chains in flight) per CTA
#define MB_SM_ARRAYS 5                  // posterior kernel: shared words per (column, lane): float4 state + class of Y
#define MB_SM_ARRAYS_MEGA 7             // MEGA: float4 state + {letters 0..3, eY} + letters 4..7
#define MB_CHAIN_MAX 32                 // posterior kernel: pairs in one chain (one per lane when the chain is read)
#define MB_CHAIN_BUF (MB_CHAIN_MAX*38)  // words of per-warp chain scratch: kept counts [pair][lane], totals [pair], final cells [pair][5]

// rows per lane per step of the posterior kernel's Forward and Backward passes: two in plain mode, one in
// MEGA mode
__host__ __device__ constexpr int mb_post_rows(bool mega)
	{
	return mega ? 1 : 2;
	}

// Forward steps one lane spends on a pair of LX rows at R rows per step: rows 0..LX, then one separator
// step.  At R = 2 a pair of even LX starts with one all-LOG_ZERO row (-1), so that its rows pair up as
// (LX-1, LX), (LX-3, LX-2), ... in Forward and Backward alike.
__host__ __device__ __forceinline__ uint32_t mb_fwd_steps(uint32_t LX, int R)
	{
	return R == 1 ? LX + 2 : LX/2 + 2;
	}

// index of pair (a,b), a < b, in the row-major all-pairs order of the store (mpcflat.cpp:139-159)
__host__ __device__ __forceinline__ uint32_t mb_pair_index(uint32_t n, uint32_t a, uint32_t b)
	{
	return (uint32_t)((uint64_t) a*n - (uint64_t) a*(a + 1)/2 + (b - a - 1));
	}

// Device view of an all-pairs store (mb_store_view).  Pair (a,b), a < b, is kept once, at mb_pair_index(n, a, b),
// in two orientations that share entbase: the forward one (rows = positions of a) and the transposed one
// (rows = positions of b).  Row i of pair q in one orientation has the entries rowoff[rowbase[q] + i] ..
// rowoff[rowbase[q] + i + 1] - 1 of entries + entbase[q] and, once the column masks are built, the header
// hdr[rowbase[q] + i] into words.
struct StoreSide
	{
	const uint64_t *rowbase;
	const uint32_t *rowoff;
	const mb200_entry *entries;
	const uint2 *hdr, *words;          // null unless the view was asked for FORM_MASKED
	};
struct StoreView
	{
	uint32_t n;                        // sequences
	const uint64_t *entbase;
	StoreSide fwd, tr;                 // tr is null unless the view was asked for FORM_TRANSPOSED or more
	};
// one pair's posteriors with rows = positions of sequence a and columns = positions of sequence b
struct StoreOperand
	{
	const uint32_t *ro;                // row offsets into en
	const mb200_entry *en;
	const uint2 *hdr, *words;          // column masks of the rows (not to be read from a view without masks)
	bool transposed;                   // read from the transposed orientation
	};
// a < b: the forward orientation of pair (a,b); a > b: the transposed orientation of pair (b,a).  Each branch
// assigns the fields itself: through a helper that returns the record, nvcc no longer sees that the pointers
// are global and the kernels read through them with generic loads.
__device__ __forceinline__ StoreOperand mb_store_operand(const StoreView &V, uint32_t a, uint32_t b)
	{
	StoreOperand o;
	if (a < b)
		{
		const uint32_t q = mb_pair_index(V.n, a, b);
		const uint64_t rb = V.fwd.rowbase[q];
		o.ro = V.fwd.rowoff + rb; o.en = V.fwd.entries + V.entbase[q]; o.hdr = V.fwd.hdr + rb; o.words = V.fwd.words;
		o.transposed = false;
		}
	else
		{
		const uint32_t q = mb_pair_index(V.n, b, a);
		const uint64_t rb = V.tr.rowbase[q];
		o.ro = V.tr.rowoff + rb; o.en = V.tr.entries + V.entbase[q]; o.hdr = V.tr.hdr + rb; o.words = V.tr.words;
		o.transposed = true;
		}
	return o;
	}

struct MbHmm
	{
	float tSM, tSI, tSJ, tMM, tMI, tMJ, tII, tIM, tJJ, tJM;   // hmmscores.h:1-13
	float minScore;                                            // logf(0.01f) from the host
	int   K, KS;                                               // classes, row stride of matchT
	int   pad;                                                 // class used for out-of-range residues
	};

// LOGEXP1 pieces (scoretype.h:95-105), {c3,c2,c1,c0} for x<=1, <=2.5, <=4.5, else.
__constant__ float4 c_logexp1[4] =
	{
	{ -0.009350833524763f, 0.130659527668286f, 0.498799810682272f, 0.693203116424741f },
	{ -0.014532321752540f, 0.139942324101744f, 0.495635523139337f, 0.692140569840976f },
	{ -0.004605031767994f, 0.063427417320019f, 0.695956496475118f, 0.514272634594009f },
	{ -0.000458661602210f, 0.009695946122598f, 0.930734667215156f, 0.168037164329057f },
	};

#define ADD(a, b) __fadd_rn((a), (b))
#define MUL(a, b) __fmul_rn((a), (b))

// LOG_ADD (scoretype.h:107-124), branch-free and bit-identical:
//  * |x-y| == (larger - smaller) exactly (round-to-nearest is sign symmetric);
//  * the reference's `smaller == LOG_ZERO` test is subsumed: if only the smaller is LOG_ZERO the gap
//    is ~2e20 >= 7.5 and the larger is returned; if both are LOG_ZERO the gap is 0 and
//    LOGEXP1(0)+LOG_ZERO rounds back to LOG_ZERO, the value the reference returns;
//  * the LOGEXP1 piece (cut points 1, 2.5, 4.5: all multiples of 1/2, intervals closed on the right)
//    is found WITHOUT compares: k = ceil(2d) is formed in the mantissa of 2d + 1.5*2^23 by one
//    FFMA with round-up, and k*16 added to a pre-biased base is the shared-memory address of a
//    17-entry {c3,c2,c1,c0} table (k = 0..2 -> piece 0, 3..5 -> 1, 6..9 -> 2, 10..16 -> 3).  The gap is
//    clamped to 4.75 before the index is formed: every d > 4.5 then reads entry 10 (piece 3, as before;
//    for d >= 7.5 the polynomial result is discarded by the final select).  The 32 lanes of a load so
//    touch at most 11 entries, not 17; entries k and k+8 share banks, and the kernels that use this are
//    bound by shared-memory wavefronts as much as by issue (clamping at 7.75 measured 1.5 % slower in
//    k_posterior_sm, H100 80GB HBM3 at 400 W).  A form with two compare/select pairs for
//    the piece takes 17 instructions per LOG_ADD, 8 of them on the half-rate ALU pipe; this form is
//    14 instructions with 4 on the ALU pipe.
//  The arithmetic (sub, three mul/add Horner steps with separate roundings, final add) is written
//  as explicit .rn PTX so that it can never be contracted into FMA.
#define MB_LA_MAGIC_BITS 0x4B400000u        // bits of 12582912.0f = 1.5 * 2^23
struct LogAdd
	{
	uint32_t tab;       // shared-memory byte address of the table - (MB_LA_MAGIC_BITS << 4), kept opaque in a register
	__device__ __forceinline__ float operator()(float x, float y) const
		{
		const float d = fabsf(__fsub_rn(x, y));
		const float lo = fminf(x, y);
		const float hi = fmaxf(x, y);
		// the address stays inside the 17-entry table for any gap (entries 11..16 are no longer read)
		const float t = __fmaf_ru(fminf(d, 4.75f), 2.0f, 12582912.0f);
		const uint32_t addr = tab + (__float_as_uint(t) << 4);
		float4 c;
		asm("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(c.x), "=f"(c.y), "=f"(c.z), "=f"(c.w) : "r"(addr));
		float q = ADD(MUL(c.x, d), c.y);
		q = ADD(MUL(q, d), c.z);
		q = ADD(MUL(q, d), c.w);
		const float r = d >= 7.5f ? hi : ADD(q, lo);
		return r;
		}
	};

// builds the 17-entry table in shared memory and stores its biased base next to it (call with >= 17
// threads, then __syncthreads)
__device__ __forceinline__ void mb_logadd_fill(float4 *tab16, uint32_t *biased)
	{
	if (threadIdx.x < 17)
		{
		const int k = threadIdx.x;
		tab16[k] = c_logexp1[k <= 2 ? 0 : (k <= 5 ? 1 : (k <= 9 ? 2 : 3))];
		}
	if (threadIdx.x == 0)
		*biased = (uint32_t) __cvta_generic_to_shared(tab16) - (MB_LA_MAGIC_BITS << 4);
	}
// The biased base is READ BACK from shared memory: a value the compiler cannot see as "table address +
// constant" stays in one register, and every LOG_ADD forms its address with one LEA.  (Computed in
// registers, ptxas splits the bias off again and spends an IMAD plus an add per LOG_ADD.)
__device__ __forceinline__ LogAdd mb_logadd_make(const uint32_t *biased)
	{
	uint32_t base;
	asm volatile("ld.shared.u32 %0, [%1];" : "=r"(base) : "r"((uint32_t) __cvta_generic_to_shared(biased)));
	LogAdd la = { base };
	return la;
	}

// ---------------------------------------------------------------------------------------------
// expf with glibc's result.  The reference computes the posterior with the host libm's expf
// (calcposteriorflat.cpp:20); glibc >= 2.27 uses the table-driven double-precision algorithm of the
// ARM optimized routines (sysdeps/ieee754/flt-32/e_expf.c: N=32 table of 2^(i/32), cubic in r,
// result rounded once to float).  The restatement below was checked here against glibc's expf on
// EVERY float in [-4.7, -0] (1 083 598 439 values, the whole range a posterior score can take:
// logf(0.01) <= score < 0) with zero mismatches, with and without FMA contraction of the cubic.
// Using it instead of CUDA's expf (<= 2 ulp) makes the posteriors, the sparse store and the EA
// scores bit-identical to the reference.  Table: asuint64(2^(i/32)) - (i << 47).
__constant__ unsigned long long c_exp2f_tab[32] =
	{
	0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull,
	0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull,
	0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
	0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull,
	0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,
	0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
	0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull,
	0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull,
	};

__device__ __forceinline__ float mb_expf_glibc(float x)
	{
	const double InvLn2N = 0x1.71547652b82fep+0*32.0;
	const double Shift = 0x1.8p+52;
	const double C0 = 0x1.c6af84b912394p-5/32.0/32.0/32.0;
	const double C1 = 0x1.ebfce50fac4f3p-3/32.0/32.0;
	const double C2 = 0x1.62e42ff0c52d6p-1/32.0;
	const double z = __dmul_rn(InvLn2N, (double) x);
	double kd = __dadd_rn(z, Shift);
	const unsigned long long ki = (unsigned long long) __double_as_longlong(kd);
	kd = __dsub_rn(kd, Shift);
	const double r = __dsub_rn(z, kd);
	const unsigned long long t = c_exp2f_tab[ki & 31ull] + (ki << 47);
	const double s = __longlong_as_double((long long) t);
	const double zz = __dadd_rn(__dmul_rn(C0, r), C1);
	const double r2 = __dmul_rn(r, r);
	double y = __dadd_rn(__dmul_rn(C2, r), 1.0);
	y = __dadd_rn(__dmul_rn(zz, r2), y);
	y = __dmul_rn(y, s);
	return __double2float_rn(y);
	}

// probability of a candidate posterior score, score >= minScore (calcposteriorflat.cpp:19-20)
__device__ __forceinline__ float mb_post_prob(float score)
	{
	return score >= 0.0f ? 1.0f : mb_expf_glibc(score);
	}

// least posterior score whose cell is kept in the sparse store.  A cell is kept when its probability is
// >= 0.01f (mysparsemx.cpp:139-141), and for every float s in [-10, 0] glibc's expf(s) >= 0.01f exactly
// when s >= -4.60517025f (0xc0935d8e, itself logf(0.01f)), so the kept decision is a compare of the score
// with this; a larger minScore cuts first.
__device__ __forceinline__ float mb_keep_score(const MbHmm &h)
	{
	return fmaxf(h.minScore, __uint_as_float(0xc0935d8eu));
	}

// head of k_posterior_sm's dynamic shared memory; the emission tables and the warps' state follow it
struct PostSmemHdr
	{
	float4   coef[17];    // LOGEXP1 pieces indexed by ceil(2*gap), see LogAdd
	float    insT[MB_MAX_K];
	uint32_t labase;      // biased shared address of coef (mb_logadd_make)
	};

struct PostParams
	{
	MbHmm h;
	const float   *matchT;          // K*KS                       | MEGA: concatenated pre-multiplied feature pair tables
	const float   *insT;            // K                          | MEGA: insert emission of every position
	const uint8_t *codes;           // residue classes, all sequences back to back | MEGA: 8 feature letters per position
	uint32_t mega_nf, mega_tsize;   // MEGA: features (<= 8), floats in the table
	uint32_t mega_base[8], mega_alpha[8];   // MEGA: offset and alphabet size of each feature's table
	const uint64_t *seqoff;
	const uint32_t *seqlen;
	const uint32_t *px, *py;        // store pair -> sequence ids
	const uint32_t *order;          // store pair ids, chain after chain
	const uint32_t *chain;          // work list: chain w is order[chain[w] .. chain[w+1]), longest first
	uint32_t nwork;                 // chains
	uint32_t *counter;              // work-stealing cursor for this launch
	// per-warp scratch
	float       *fm;      size_t fm_stride;      // floats
	float4      *edge;    size_t edge_stride;    // float4, two ping-pong halves
	mb200_entry *rows;    size_t rows_stride;    // entries
	uint8_t     *rowcnt;  size_t rowcnt_stride;  // bytes
	uint32_t    *chainbuf;                       // MB_CHAIN_BUF words per warp
	uint32_t     lxmax;                          // rows of one pair the scratch was sized for
	uint32_t     fm_rows;                        // mb_fwd_steps(lxmax, R) + 31: steps per strip slot in fm (R*W floats each)
	uint32_t     cmax;                           // k_posterior_sm: cap on the columns per lane (<= the size class)
	// outputs
	uint32_t       *rowoff;         // concatenated, pair k at rowbase[k], LX+1 entries
	const uint64_t *rowbase;
	mb200_entry    *entries;        // bump-allocated
	uint64_t        ent_cap;
	unsigned long long *ent_cursor;
	uint64_t       *entbase;        // per store pair
	uint32_t       *nnz;            // per store pair
	float          *ea;             // per store pair
	int            *err;            // sticky error code
	// optional dense dumps for one pair (parity surface, mb200_calc_post_dense_pair)
	float *dbg_fwd, *dbg_bwd, *dbg_post, *dbg_total;
	uint32_t dbg_pair;              // the store pair they are written for
	};
