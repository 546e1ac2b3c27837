/* oracle/muscle_oracle.h -- TEST INFRASTRUCTURE ONLY (CPU restatement of the MPCFlat hot path).
 *
 * Plain-C restatement of the reference algorithm (rcedgar/muscle @ 6c69a9b) used as the parity
 * checker for the CUDA library.  Nothing in muscle_b200/ (the product) may include, link or call
 * this; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
 *
 * Pinning status: PINNED.  tests/test_oracle_vs_ref.py checks every function below bit-for-bit
 * against the compiled reference (oracle/_ref/libmuscle_ref.so, strict-IEEE build) and
 * tests/test_oracle_golden.py checks it against committed golden vectors that the compiled
 * reference produced (tests/golden/make_golden.py).
 */
#ifndef MUSCLE_ORACLE_H
#define MUSCLE_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MO_LOG_ZERO (-2e20f)
enum { MO_M = 0, MO_IX = 1, MO_IY = 2, MO_JX = 3, MO_JY = 4, MO_NSTATE = 5 };

/* PairHMM score tables exactly as the reference host computes them (pairhmm.h:26-29). */
typedef struct
	{
	float start[5];        /* m_StartScore */
	float trans[25];       /* m_TransScore[from][to] */
	float ins[256];        /* m_InsScore */
	float match[65536];    /* m_MatchScore[a][b] */
	float min_sparse_score;/* logf(0.01f) as evaluated by the host libm (mysparsemx.h:4) */
	} mo_hmm;

typedef struct { float p; uint32_t col; } mo_entry;   /* MySparseMx wire format, 8 bytes */

float mo_logexp1(float x);
float mo_log_add(float x, float y);
/* batch forms (OpenMP): out[k] = mo_log_add(a[k], b[k]); out[k] = the probability CalcPostFlat writes for
 * score s[k] (calcposteriorflat.cpp:15-20, libm expf).  Range forms: a[k] / s[k] is the float whose bits are
 * first_bits + k; swap: out[k] = mo_log_add(b, a[k]). */
void  mo_log_add_n(uint64_t n, const float *a, const float *b, float *out);
void  mo_log_add_range(uint64_t n, uint32_t a_first_bits, float b, int swap, float *out);
void  mo_post_prob_n(uint64_t n, const float *s, float min_score, float *out);
void  mo_post_prob_range(uint64_t n, uint32_t s_first_bits, float min_score, float *out);

/* flat layout: flat[5*(i*(LY+1)+j)+s], 0<=i<=LX, 0<=j<=LY (flatmx.h:11-15) */
void  mo_fwd(const mo_hmm *h, const uint8_t *X, uint32_t LX, const uint8_t *Y, uint32_t LY, float *flat);
void  mo_bwd(const mo_hmm *h, const uint8_t *X, uint32_t LX, const uint8_t *Y, uint32_t LY, float *flat);
float mo_total(const float *fwd, const float *bwd, uint32_t LX, uint32_t LY);
void  mo_post(const mo_hmm *h, const float *fwd, const float *bwd, uint32_t LX, uint32_t LY, float *post);
/* fwd+bwd+post with internal scratch; post is LX*LY */
void  mo_calcpost(const mo_hmm *h, const uint8_t *X, uint32_t LX, const uint8_t *Y, uint32_t LY, float *post);

/* returns nnz; offsets[LX+1]; entries may be NULL to count only */
uint32_t mo_sparse_from_post(const float *post, uint32_t LX, uint32_t LY, uint32_t *offsets, mo_entry *entries);
float mo_alnscore(const float *post, uint32_t LX, uint32_t LY);
/* path gets LX+LY+1 bytes (NUL terminated, letters B/X/Y); returns DP score */
float mo_calcaln(const float *post, uint32_t LX, uint32_t LY, char *path);

/* All-pairs stage for N sequences (pair p=(i<j) row-major).  Outputs: per-pair CSR packed back to
 * back (pair_off[p] = first entry of pair p, row_off[rowbase[p] + r]), EA matrix N*N.
 * Pass entries==NULL to only count.  Runs pairs [p_lo,p_hi) with `threads` OpenMP threads and
 * returns DP cells processed. */
typedef struct
	{
	uint32_t  n;
	const uint8_t *const *seq;
	const uint32_t *len;
	} mo_seqset;

uint64_t mo_all_pairs(const mo_hmm *h, const mo_seqset *S, uint32_t p_lo, uint32_t p_hi, int threads,
  uint64_t *pair_nnz, uint32_t **row_off_out, mo_entry **entries_out, float *ea_out);
void mo_free(void *p);

/* One Jacobi consistency update of pair (x<y) (conspairflat.cpp:10-110): sparse store given as
 * per-pair arrays indexed by pair index p(i,j)= i*n - i*(i+1)/2 + (j-i-1). */
void mo_conspair(uint32_t n, const uint32_t *len, uint32_t x, uint32_t y,
  const uint32_t *const *row_off, const mo_entry *const *entries, mo_entry *out_entries);

/* BuildPost (buildpostflat.cpp:18-105) for two groups of gapped rows.
 * pos2col_a[s] maps residue position -> column for sequence ids_a[s]. */
void mo_buildpost(uint32_t n, const uint32_t *len,
  uint32_t na, const uint32_t *ids_a, const uint32_t *const *pos2col_a, uint32_t cols_a,
  uint32_t nb, const uint32_t *ids_b, const uint32_t *const *pos2col_b, uint32_t cols_b,
  const uint32_t *const *row_off, const mo_entry *const *entries, float *post);

/* guide tree: UPGMA5::FixEADistMx + UPGMA5::Run (upgma5.cpp:504-519,87-330); returns -1 if an EA is outside [0,1] */
int mo_upgma(uint32_t n, const float *ea, int linkage, uint32_t *left, uint32_t *right, float *llen, float *rlen);

#ifdef __cplusplus
}
#endif
#endif
