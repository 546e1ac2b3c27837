/* oracle/muscle_oracle.c -- TEST INFRASTRUCTURE ONLY.  See muscle_oracle.h for the rules.
 *
 * CPU restatement of MUSCLE5's MPCFlat hot path.  Every function names the reference lines it
 * follows (paths relative to /root/reference/src).  Build with -ffp-contract=off: the reference's
 * parity build has no FMA contraction and every fp32 operation below is written in the
 * reference's association order, so results are bit-identical (checked by tests/).
 */
#include "muscle_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ------------------------------------------------------------------ log-space helpers
 * scoretype.h:95-105  LOGEXP1: piecewise cubic for log(exp(x)+1), 0<=x<=7.5, Horner form.   */
float mo_logexp1(float x)
	{
	if (x <= 1.00f)
		return ((-0.009350833524763f*x + 0.130659527668286f)*x + 0.498799810682272f)*x + 0.693203116424741f;
	if (x <= 2.50f)
		return ((-0.014532321752540f*x + 0.139942324101744f)*x + 0.495635523139337f)*x + 0.692140569840976f;
	if (x <= 4.50f)
		return ((-0.004605031767994f*x + 0.063427417320019f)*x + 0.695956496475118f)*x + 0.514272634594009f;
	return ((-0.000458661602210f*x + 0.009695946122598f)*x + 0.930734667215156f)*x + 0.168037164329057f;
	}

/* scoretype.h:107-124  LOG_ADD / LOG_PLUS_EQUALS (identical branch structure). */
float mo_log_add(float x, float y)
	{
	if (x < y)
		return (x == MO_LOG_ZERO || y - x >= 7.5f) ? y : mo_logexp1(y - x) + x;
	return (y == MO_LOG_ZERO || x - y >= 7.5f) ? x : mo_logexp1(x - y) + y;
	}

/* scoretype.h:136-139: n-ary LOG_ADD is a right fold */
static float log_add5(float a, float b, float c, float d, float e)
	{
	return mo_log_add(a, mo_log_add(b, mo_log_add(c, mo_log_add(d, e))));
	}

#define CELL(flat, i, j, LY1) ((flat) + 5*((size_t)(i)*(LY1) + (j)))

/* ------------------------------------------------------------------ Forward
 * fwdflat3.cpp:12-153.  State order M,IX,IY,JX,JY (pairhmm.h:11-19). */
void mo_fwd(const mo_hmm *h, const uint8_t *X, uint32_t LX, const uint8_t *Y, uint32_t LY, float *flat)
	{
	const float tSM = h->start[MO_M], tSI = h->start[MO_IX], tSJ = h->start[MO_JX];
	const float tMM = h->trans[MO_M*5 + MO_M], tMI = h->trans[MO_M*5 + MO_IX], tMJ = h->trans[MO_M*5 + MO_JX];
	const float tII = h->trans[MO_IX*5 + MO_IX], tIM = h->trans[MO_IX*5 + MO_M];
	const float tJJ = h->trans[MO_JX*5 + MO_JX], tJM = h->trans[MO_JX*5 + MO_M];
	const uint32_t LY1 = LY + 1;
	const float Z = MO_LOG_ZERO;

	/* origin (fwdflat3.cpp:35-39) */
	float *c = CELL(flat, 0, 0, LY1);
	c[MO_M] = c[MO_IX] = c[MO_IY] = c[MO_JX] = c[MO_JY] = Z;

	/* column j=0: only X-insert chains are alive (fwdflat3.cpp:42-43,47-55,67-79) */
	for (uint32_t i = 1; i <= LX; ++i)
		{
		float *cur = CELL(flat, i, 0, LY1);
		const float e = h->ins[X[i - 1]];
		cur[MO_M] = cur[MO_IY] = cur[MO_JY] = Z;
		if (i == 1)
			{
			cur[MO_IX] = tSI + e;
			cur[MO_JX] = tSJ + e;
			}
		else
			{
			const float *up = CELL(flat, i - 1, 0, LY1);
			cur[MO_IX] = up[MO_IX] + tII + e;
			cur[MO_JX] = up[MO_JX] + tJJ + e;
			}
		}
	/* row i=0: only Y-insert chains (fwdflat3.cpp:44-45,57-65,81-93) */
	for (uint32_t j = 1; j <= LY; ++j)
		{
		float *cur = CELL(flat, 0, j, LY1);
		const float e = h->ins[Y[j - 1]];
		cur[MO_M] = cur[MO_IX] = cur[MO_JX] = Z;
		if (j == 1)
			{
			cur[MO_IY] = tSI + e;
			cur[MO_JY] = tSJ + e;
			}
		else
			{
			const float *lf = CELL(flat, 0, j - 1, LY1);
			cur[MO_IY] = lf[MO_IY] + tII + e;
			cur[MO_JY] = lf[MO_JY] + tJJ + e;
			}
		}
	/* interior (fwdflat3.cpp:100-152) */
	for (uint32_t i = 1; i <= LX; ++i)
		{
		const uint8_t x = X[i - 1];
		const float ex = h->ins[x];
		const float *mrow = h->match + 256*(size_t) x;
		for (uint32_t j = 1; j <= LY; ++j)
			{
			const uint8_t y = Y[j - 1];
			const float ey = h->ins[y];
			float *cur = CELL(flat, i, j, LY1);
			const float *dg = CELL(flat, i - 1, j - 1, LY1);
			const float *up = CELL(flat, i - 1, j, LY1);
			const float *lf = CELL(flat, i, j - 1, LY1);
			if (i == 1 && j == 1)
				cur[MO_M] = tSM + mrow[y];
			else
				cur[MO_M] = log_add5(dg[MO_M] + tMM, dg[MO_IX] + tIM, dg[MO_JX] + tJM,
				  dg[MO_IY] + tIM, dg[MO_JY] + tJM) + mrow[y];
			cur[MO_IX] = mo_log_add(up[MO_IX] + tII, up[MO_M] + tMI) + ex;
			cur[MO_JX] = mo_log_add(up[MO_JX] + tJJ, up[MO_M] + tMJ) + ex;
			cur[MO_IY] = mo_log_add(lf[MO_IY] + tII, lf[MO_M] + tMI) + ey;
			cur[MO_JY] = mo_log_add(lf[MO_JY] + tJJ, lf[MO_M] + tMJ) + ey;
			}
		}
	}

/* ------------------------------------------------------------------ Backward
 * bwdflat3.cpp:10-184.  Cell (i,j) = i letters of X and j of Y already consumed. */
void mo_bwd(const mo_hmm *h, const uint8_t *X, uint32_t LX, const uint8_t *Y, uint32_t LY, float *flat)
	{
	const float tSM = h->start[MO_M], tSI = h->start[MO_IX], tSJ = h->start[MO_JX];
	const float tMM = h->trans[MO_M*5 + MO_M], tMI = h->trans[MO_M*5 + MO_IX], tMJ = h->trans[MO_M*5 + MO_JX];
	const float tII = h->trans[MO_IX*5 + MO_IX], tIM = h->trans[MO_IX*5 + MO_M];
	const float tJJ = h->trans[MO_JX*5 + MO_JX], tJM = h->trans[MO_JX*5 + MO_M];
	const uint32_t LY1 = LY + 1;
	const float Z = MO_LOG_ZERO;

	for (int64_t i = LX; i >= 0; --i)
		{
		for (int64_t j = LY; j >= 0; --j)
			{
			float *cur = CELL(flat, i, j, LY1);
			if (i == (int64_t) LX && j == (int64_t) LY)
				{
				/* end of alignment re-uses the start probabilities (bwdflat3.cpp:53-61) */
				cur[MO_M] = tSM;
				cur[MO_IX] = cur[MO_IY] = tSI;
				cur[MO_JX] = cur[MO_JY] = tSJ;
				continue;
				}
			float nM = 0, nIX = 0, nJX = 0, nIY = 0, nJY = 0;
			if (i < (int64_t) LX)
				{
				const float ex = h->ins[X[i]];
				const float *dn = CELL(flat, i + 1, j, LY1);
				nIX = dn[MO_IX] + ex;
				nJX = dn[MO_JX] + ex;
				}
			if (j < (int64_t) LY)
				{
				const float ey = h->ins[Y[j]];
				const float *rt = CELL(flat, i, j + 1, LY1);
				nIY = rt[MO_IY] + ey;
				nJY = rt[MO_JY] + ey;
				}
			if (i < (int64_t) LX && j < (int64_t) LY)
				{
				/* bwdflat3.cpp:73-130 */
				nM = CELL(flat, i + 1, j + 1, LY1)[MO_M] + h->match[256*(size_t) X[i] + Y[j]];
				cur[MO_M] = (i > 0 && j > 0) ?
				  log_add5(tMM + nM, tMI + nIX, tMJ + nJX, tMI + nIY, tMJ + nJY) : Z;
				if (i > 0)
					{
					cur[MO_IX] = mo_log_add(tII + nIX, tIM + nM);
					cur[MO_JX] = mo_log_add(tJJ + nJX, tJM + nM);
					}
				else
					cur[MO_IX] = cur[MO_JX] = Z;
				if (j > 0)
					{
					cur[MO_IY] = mo_log_add(tII + nIY, tIM + nM);
					cur[MO_JY] = mo_log_add(tJJ + nJY, tJM + nM);
					}
				else
					cur[MO_IY] = cur[MO_JY] = Z;
				}
			else if (i < (int64_t) LX)
				{
				/* last column j==LY (bwdflat3.cpp:25-31,132-153): only X inserts can follow */
				cur[MO_IY] = cur[MO_JY] = Z;
				if (i > 0)
					{
					cur[MO_M] = mo_log_add(tMI + nIX, tMJ + nJX);
					cur[MO_IX] = tII + nIX;
					cur[MO_JX] = tJJ + nJX;
					}
				else
					cur[MO_M] = cur[MO_IX] = cur[MO_JX] = Z;
				}
			else
				{
				/* last row i==LX (bwdflat3.cpp:33-39,155-176): only Y inserts can follow */
				cur[MO_IX] = cur[MO_JX] = Z;
				if (j > 0)
					{
					cur[MO_M] = mo_log_add(tMI + nIY, tMJ + nJY);
					cur[MO_IY] = tII + nIY;
					cur[MO_JY] = tJJ + nJY;
					}
				else
					cur[MO_M] = cur[MO_IY] = cur[MO_JY] = Z;
				}
			}
		}
	}

/* totalprobflat.cpp:3-16 */
float mo_total(const float *fwd, const float *bwd, uint32_t LX, uint32_t LY)
	{
	const float *f = CELL(fwd, LX, LY, LY + 1);
	const float *b = CELL(bwd, LX, LY, LY + 1);
	float sum = MO_LOG_ZERO;
	for (int s = 0; s < 5; ++s)
		sum = mo_log_add(sum, f[s] + b[s]);
	return sum;
	}

/* calcposteriorflat.cpp:15-20: the probability CalcPostFlat writes for one posterior score */
static float post_prob(float score, float min_score)
	{
	if (score < min_score)
		return 0.0f;
	return (score >= 0.0f) ? 1.0f : expf(score);
	}

/* calcposteriorflat.cpp:4-27 */
void mo_post(const mo_hmm *h, const float *fwd, const float *bwd, uint32_t LX, uint32_t LY, float *post)
	{
	const float total = mo_total(fwd, bwd, LX, LY);
	for (uint32_t i = 1; i <= LX; ++i)
		for (uint32_t j = 1; j <= LY; ++j)
			{
			const float score = CELL(fwd, i, j, LY + 1)[MO_M] + CELL(bwd, i, j, LY + 1)[MO_M] - total;
			post[(size_t)(i - 1)*LY + (j - 1)] = post_prob(score, h->min_sparse_score);
			}
	}

/* batch and bit-range forms of mo_log_add and post_prob for the arithmetic sweeps of the tests */
static float bits_float(uint32_t u)
	{
	float f;
	memcpy(&f, &u, 4);
	return f;
	}

void mo_log_add_n(uint64_t n, const float *a, const float *b, float *out)
	{
#pragma omp parallel for schedule(static)
	for (int64_t k = 0; k < (int64_t) n; ++k)
		out[k] = mo_log_add(a[k], b[k]);
	}

void mo_log_add_range(uint64_t n, uint32_t a_first_bits, float b, int swap, float *out)
	{
#pragma omp parallel for schedule(static)
	for (int64_t k = 0; k < (int64_t) n; ++k)
		{
		const float a = bits_float(a_first_bits + (uint32_t) k);
		out[k] = swap ? mo_log_add(b, a) : mo_log_add(a, b);
		}
	}

void mo_post_prob_n(uint64_t n, const float *s, float min_score, float *out)
	{
#pragma omp parallel for schedule(static)
	for (int64_t k = 0; k < (int64_t) n; ++k)
		out[k] = post_prob(s[k], min_score);
	}

void mo_post_prob_range(uint64_t n, uint32_t s_first_bits, float min_score, float *out)
	{
#pragma omp parallel for schedule(static)
	for (int64_t k = 0; k < (int64_t) n; ++k)
		out[k] = post_prob(bits_float(s_first_bits + (uint32_t) k), min_score);
	}

/* calcpost.cpp:4-36 minus the label registry */
void mo_calcpost(const mo_hmm *h, const uint8_t *X, uint32_t LX, const uint8_t *Y, uint32_t LY, float *post)
	{
	const size_t n = 5*(size_t)(LX + 1)*(LY + 1);
	float *fwd = (float *) malloc(n*sizeof(float));
	float *bwd = (float *) malloc(n*sizeof(float));
	mo_fwd(h, X, LX, Y, LY, fwd);
	mo_bwd(h, X, LX, Y, LY, bwd);
	mo_post(h, fwd, bwd, LX, LY, post);
	free(fwd);
	free(bwd);
	}

/* mysparsemx.cpp:115-152  keep P >= 0.01f, row major, columns ascending */
uint32_t mo_sparse_from_post(const float *post, uint32_t LX, uint32_t LY, uint32_t *offsets, mo_entry *entries)
	{
	uint32_t n = 0;
	for (uint32_t i = 0; i < LX; ++i)
		{
		offsets[i] = n;
		for (uint32_t j = 0; j < LY; ++j)
			{
			const float p = post[(size_t) i*LY + j];
			if (p >= 0.01f)
				{
				if (entries)
					{
					entries[n].p = p;
					entries[n].col = j;
					}
				++n;
				}
			}
		}
	offsets[LX] = n;
	return n;
	}

/* best3.h:31-49 (value only; ties cannot change the value) */
static float max3(float b, float x, float y)
	{
	if (b >= x)
		return b >= y ? b : y;
	return x >= y ? x : y;
	}

/* calcalnscoreflat.cpp:4-32 */
float mo_alnscore(const float *post, uint32_t LX, uint32_t LY)
	{
	float *row = (float *) calloc(LY + 1, sizeof(float));
	for (uint32_t i = 1; i <= LX; ++i)
		{
		float diag = row[0];
		float left = 0.0f;
		row[0] = 0.0f;
		for (uint32_t j = 1; j <= LY; ++j)
			{
			const float up = row[j];
			const float v = max3(diag + post[(size_t)(i - 1)*LY + (j - 1)], up, left);
			diag = up;
			left = v;
			row[j] = v;
			}
		}
	const float s = row[LY];
	free(row);
	return s;
	}

/* calcalnflat.cpp:6-46 + best3.h:5-28 (tie order B, then X>=Y) + tracebackflat.cpp:3-37 */
float mo_calcaln(const float *post, uint32_t LX, uint32_t LY, char *path)
	{
	const size_t LY1 = (size_t) LY + 1;
	char *tb = (char *) malloc((size_t)(LX + 1)*LY1);
	float *prev = (float *) calloc(LY1, sizeof(float));
	float *cur = (float *) calloc(LY1, sizeof(float));
	for (uint32_t j = 0; j <= LY; ++j)
		tb[j] = 'Y';
	for (uint32_t i = 1; i <= LX; ++i)
		{
		tb[i*LY1] = 'X';
		cur[0] = 0.0f;
		for (uint32_t j = 1; j <= LY; ++j)
			{
			const float b = prev[j - 1] + post[(size_t)(i - 1)*LY + (j - 1)];
			const float x = prev[j];
			const float y = cur[j - 1];
			float best;
			char t;
			if (b >= x)
				{
				if (b >= y) { best = b; t = 'B'; }
				else        { best = y; t = 'Y'; }
				}
			else if (x >= y) { best = x; t = 'X'; }
			else             { best = y; t = 'Y'; }
			cur[j] = best;
			tb[i*LY1 + j] = t;
			}
		float *tmp = prev; prev = cur; cur = tmp;
		}
	const float score = prev[LY];
	/* walk back from (LX,LY) */
	size_t n = 0;
	int64_t i = LX, j = LY;
	while (i != 0 || j != 0)
		{
		const char t = tb[(size_t) i*LY1 + (size_t) j];
		path[n++] = t;
		if (t == 'B') { --i; --j; }
		else if (t == 'X') --i;
		else --j;
		}
	for (size_t a = 0, b2 = n; a + 1 < b2; ++a, --b2)
		{
		char t = path[a]; path[a] = path[b2 - 1]; path[b2 - 1] = t;
		}
	path[n] = 0;
	free(tb);
	free(prev);
	free(cur);
	return score;
	}

/* ------------------------------------------------------------------ all-pairs stage
 * MPCFlat::CalcPosterior calcposteriorflat.cpp:45-92 per pair; pair order mpcflat.cpp:139-159. */
void mo_free(void *p) { free(p); }

uint64_t mo_all_pairs(const mo_hmm *h, const mo_seqset *S, uint32_t p_lo, uint32_t p_hi, int threads,
  uint64_t *pair_nnz, uint32_t **row_off_out, mo_entry **entries_out, float *ea_out)
	{
	const uint32_t n = S->n;
	const uint32_t npairs = n*(n - 1)/2;
	if (p_hi > npairs)
		p_hi = npairs;
	uint32_t *px = (uint32_t *) malloc(sizeof(uint32_t)*(npairs + 1));
	uint32_t *py = (uint32_t *) malloc(sizeof(uint32_t)*(npairs + 1));
	uint32_t p = 0;
	for (uint32_t i = 0; i < n; ++i)
		for (uint32_t j = i + 1; j < n; ++j, ++p)
			{
			px[p] = i;
			py[p] = j;
			}
	const uint32_t cnt = p_hi - p_lo;
	uint32_t **offs = (uint32_t **) calloc(cnt ? cnt : 1, sizeof(uint32_t *));
	mo_entry **ents = (mo_entry **) calloc(cnt ? cnt : 1, sizeof(mo_entry *));
	uint64_t cells = 0;
#ifdef _OPENMP
	if (threads <= 0)
		threads = omp_get_max_threads();
#pragma omp parallel for num_threads(threads) schedule(dynamic, 1) reduction(+:cells)
#endif
	for (int64_t q = 0; q < (int64_t) cnt; ++q)
		{
		const uint32_t pi = p_lo + (uint32_t) q;
		const uint32_t x = px[pi], y = py[pi];
		const uint32_t LX = S->len[x], LY = S->len[y];
		float *post = (float *) malloc(sizeof(float)*(size_t) LX*LY);
		mo_calcpost(h, S->seq[x], LX, S->seq[y], LY, post);
		offs[q] = (uint32_t *) malloc(sizeof(uint32_t)*(LX + 1));
		const uint32_t nnz = mo_sparse_from_post(post, LX, LY, offs[q], NULL);
		ents[q] = (mo_entry *) malloc(sizeof(mo_entry)*(nnz ? nnz : 1));
		mo_sparse_from_post(post, LX, LY, offs[q], ents[q]);
		pair_nnz[q] = nnz;
		if (ea_out)
			{
			const float ea = mo_alnscore(post, LX, LY)/(float)(LX < LY ? LX : LY);
			ea_out[(size_t) x*n + y] = ea;
			ea_out[(size_t) y*n + x] = ea;
			}
		free(post);
		cells += (uint64_t) LX*LY;
		}
	if (row_off_out && entries_out)
		{
		size_t tot_rows = 0, tot_nnz = 0;
		for (uint32_t q = 0; q < cnt; ++q)
			{
			tot_rows += S->len[px[p_lo + q]] + 1;
			tot_nnz += pair_nnz[q];
			}
		uint32_t *ro = (uint32_t *) malloc(sizeof(uint32_t)*(tot_rows ? tot_rows : 1));
		mo_entry *en = (mo_entry *) malloc(sizeof(mo_entry)*(tot_nnz ? tot_nnz : 1));
		size_t r = 0, e = 0;
		for (uint32_t q = 0; q < cnt; ++q)
			{
			const uint32_t LX = S->len[px[p_lo + q]];
			memcpy(ro + r, offs[q], sizeof(uint32_t)*(LX + 1));
			memcpy(en + e, ents[q], sizeof(mo_entry)*pair_nnz[q]);
			r += LX + 1;
			e += pair_nnz[q];
			}
		*row_off_out = ro;
		*entries_out = en;
		}
	for (uint32_t q = 0; q < cnt; ++q)
		{
		free(offs[q]);
		free(ents[q]);
		}
	free(offs);
	free(ents);
	free(px);
	free(py);
	return cells;
	}

/* ------------------------------------------------------------------ consistency
 * conspairflat.cpp:10-110 + relaxflat.cpp:4-94 + mysparsemx.cpp:87-113.
 * The reference picks one of three loop nests by index order because only i<j pairs are stored;
 * all three add, for a fixed output cell (i,j) and a fixed Z, the products P_XZ[i,k]*P_ZY[k,j] in
 * ascending k, and Z runs ascending.  Here both operands are brought to "rows of the first index"
 * form (transposing the stored matrix when needed), which keeps that order. */
static uint32_t pair_index(uint32_t n, uint32_t i, uint32_t j)
	{
	return i*n - i*(i + 1)/2 + (j - i - 1);
	}

typedef struct { uint32_t rows; uint32_t *off; mo_entry *ent; int owned; } csr_t;

static csr_t csr_view(uint32_t rows, const uint32_t *off, const mo_entry *ent)
	{
	csr_t c = { rows, (uint32_t *) off, (mo_entry *) ent, 0 };
	return c;
	}

static csr_t csr_transpose(uint32_t rows, uint32_t cols, const uint32_t *off, const mo_entry *ent)
	{
	csr_t t;
	t.rows = cols;
	t.owned = 1;
	t.off = (uint32_t *) calloc(cols + 2, sizeof(uint32_t));
	const uint32_t nnz = off[rows];
	t.ent = (mo_entry *) malloc(sizeof(mo_entry)*(nnz ? nnz : 1));
	for (uint32_t e = 0; e < nnz; ++e)
		t.off[ent[e].col + 2]++;
	for (uint32_t c = 0; c < cols; ++c)
		t.off[c + 2] += t.off[c + 1];
	for (uint32_t r = 0; r < rows; ++r)
		for (uint32_t e = off[r]; e < off[r + 1]; ++e)
			{
			const uint32_t dst = t.off[ent[e].col + 1]++;
			t.ent[dst].p = ent[e].p;
			t.ent[dst].col = r;
			}
	return t;
	}

static void csr_release(csr_t *c)
	{
	if (c->owned)
		{
		free(c->off);
		free(c->ent);
		}
	}

/* matrix with rows = positions of a, cols = positions of b */
static csr_t oriented(uint32_t n, const uint32_t *len, uint32_t a, uint32_t b,
  const uint32_t *const *row_off, const mo_entry *const *entries)
	{
	if (a < b)
		{
		const uint32_t p = pair_index(n, a, b);
		return csr_view(len[a], row_off[p], entries[p]);
		}
	const uint32_t p = pair_index(n, b, a);
	return csr_transpose(len[b], len[a], row_off[p], entries[p]);
	}

void mo_conspair(uint32_t n, const uint32_t *len, uint32_t x, uint32_t y,
  const uint32_t *const *row_off, const mo_entry *const *entries, mo_entry *out_entries)
	{
	const uint32_t LX = len[x], LY = len[y];
	const uint32_t pxy = pair_index(n, x, y);
	const uint32_t *off = row_off[pxy];
	const mo_entry *ent = entries[pxy];
	float *post = (float *) calloc((size_t) LX*LY, sizeof(float));
	/* Z=X and Z=Y contribute P_XY each: factor 2 (conspairflat.cpp:26-30) */
	for (uint32_t i = 0; i < LX; ++i)
		for (uint32_t e = off[i]; e < off[i + 1]; ++e)
			post[(size_t) i*LY + ent[e].col] = ent[e].p*2;
	for (uint32_t z = 0; z < n; ++z)
		{
		if (z == x || z == y)
			continue;
		csr_t A = oriented(n, len, x, z, row_off, entries);   /* rows X, cols Z */
		csr_t B = oriented(n, len, z, y, row_off, entries);   /* rows Z, cols Y */
		for (uint32_t i = 0; i < LX; ++i)
			for (uint32_t a = A.off[i]; a < A.off[i + 1]; ++a)
				{
				const float pa = 1.0f*A.ent[a].p;          /* weight forced to 1 (conspairflat.cpp:41-42) */
				const uint32_t k = A.ent[a].col;
				for (uint32_t b = B.off[k]; b < B.off[k + 1]; ++b)
					post[(size_t) i*LY + B.ent[b].col] += pa*B.ent[b].p;
				}
		csr_release(&A);
		csr_release(&B);
		}
	/* mysparsemx.cpp:87-113: pattern kept, value = Post/SeqCount */
	for (uint32_t i = 0; i < LX; ++i)
		for (uint32_t e = off[i]; e < off[i + 1]; ++e)
			{
			out_entries[e].col = ent[e].col;
			out_entries[e].p = post[(size_t) i*LY + ent[e].col]/(float) n;
			}
	free(post);
	}

/* ------------------------------------------------------------------ BuildPost
 * buildpostflat.cpp:18-105: s-major, t-minor; rows then entries ascending inside one sparse
 * matrix; when the stored pair is (t,s) the loop runs over t's rows.  Weights are all 1. */
void mo_buildpost(uint32_t n, const uint32_t *len,
  uint32_t na, const uint32_t *ids_a, const uint32_t *const *pos2col_a, uint32_t cols_a,
  uint32_t nb, const uint32_t *ids_b, const uint32_t *const *pos2col_b, uint32_t cols_b,
  const uint32_t *const *row_off, const mo_entry *const *entries, float *post)
	{
	(void) cols_a;
	memset(post, 0, sizeof(float)*(size_t) cols_a*cols_b);
	for (uint32_t s = 0; s < na; ++s)
		for (uint32_t t = 0; t < nb; ++t)
			{
			const uint32_t a = ids_a[s], b = ids_b[t];
			const float w = 1.0f*1.0f;
			if (a < b)
				{
				const uint32_t p = pair_index(n, a, b);
				for (uint32_t i = 0; i < len[a]; ++i)
					for (uint32_t e = row_off[p][i]; e < row_off[p][i + 1]; ++e)
						post[(size_t) pos2col_a[s][i]*cols_b + pos2col_b[t][entries[p][e].col]] += w*entries[p][e].p;
				}
			else
				{
				const uint32_t p = pair_index(n, b, a);
				for (uint32_t i = 0; i < len[b]; ++i)
					for (uint32_t e = row_off[p][i]; e < row_off[p][i + 1]; ++e)
						post[(size_t) pos2col_a[s][entries[p][e].col]*cols_b + pos2col_b[t][i]] += w*entries[p][e].p;
				}
			}
	}

/* ------------------------------------------------------------------ guide tree
 * UPGMA5::FixEADistMx (upgma5.cpp:504-519) + UPGMA5::Run (upgma5.cpp:87-330), sequential, as the
 * reference: triangle subscript (upgma5.h:63-72), nearest-neighbour bookkeeping incl. the "nasty
 * special case" (:248-259), strict `<` scans in ascending index order.  ea: N(N-1)/2 values, row-major
 * i<j.  linkage: 1 min, 2 max, 3 avg, 4 biased (types.h:11-15).  Outputs: N-1 entries each. */
static uint32_t tri(uint32_t a, uint32_t b) { return a >= b ? b + (a*(a - 1))/2 : a + (b*(b - 1))/2; }
static float avg2(float x, float y) { return (x + y)/2; }
int mo_upgma(uint32_t n, const float *ea, int linkage, uint32_t *left, uint32_t *right, float *llen, float *rlen)
	{
	const uint32_t NONE = 0xffffffffu;
	float *dist = (float *) malloc(sizeof(float)*((size_t) n*(n - 1)/2 + 1));
	float *mind = (float *) malloc(sizeof(float)*n), *height = (float *) malloc(sizeof(float)*n);
	uint32_t *nn = (uint32_t *) malloc(4*n), *node = (uint32_t *) malloc(4*n);
	for (uint32_t i = 0; i < n; ++i)
		{
		mind[i] = FLT_MAX; nn[i] = NONE; node[i] = i;
		}
	for (uint32_t i = 1; i < n; ++i)
		for (uint32_t j = 0; j < i; ++j)
			{
			const float e = ea[pair_index(n, j, i)];
			if (!(e >= 0 && e <= 1))
				return -1;
			float d = 1 - e;
			if (d < 0)
				d = 0;
			dist[tri(i, j)] = d;
			if (d < mind[i]) { mind[i] = d; nn[i] = j; }
			if (d < mind[j]) { mind[j] = d; nn[j] = i; }
			}
	for (uint32_t k = 0; k + 1 < n; ++k)
		{
		uint32_t lmin = NONE, rmin = NONE;
		float best = FLT_MAX;
		for (uint32_t j = 0; j < n; ++j)
			{
			if (node[j] == NONE)
				continue;
			if (mind[j] < best) { best = mind[j]; lmin = j; rmin = nn[j]; }
			}
		float newmin = FLT_MAX;
		uint32_t newnn = NONE;
		for (uint32_t j = 0; j < n; ++j)
			{
			if (j == lmin || j == rmin || node[j] == NONE)
				continue;
			const float dL = dist[tri(lmin, j)], dR = dist[tri(rmin, j)];
			float nd;
			if (linkage == 3) nd = avg2(dL, dR);
			else if (linkage == 1) nd = dL < dR ? dL : dR;
			else if (linkage == 2) nd = dL > dR ? dL : dR;
			else nd = 0.1f*avg2(dL, dR) + (1 - 0.1f)*(dR < dL ? dR : dL);
			if (nn[j] == rmin)
				nn[j] = lmin;
			dist[tri(lmin, j)] = nd;
			if (nd < newmin) { newmin = nd; newnn = j; }
			}
		const float h = dist[tri(lmin, rmin)]/2;
		const uint32_t uL = node[lmin], uR = node[rmin];
		left[k] = uL; right[k] = uR;
		llen[k] = h - (uL < n ? 0 : height[uL - n]);
		rlen[k] = h - (uR < n ? 0 : height[uR - n]);
		height[k] = h;
		node[lmin] = n + k; nn[lmin] = newnn; mind[lmin] = newmin; node[rmin] = NONE;
		}
	free(dist); free(mind); free(height); free(nn); free(node);
	return 0;
	}
