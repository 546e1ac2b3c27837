// oracle/ref_math_probe.cpp -- TEST INFRASTRUCTURE ONLY.
//
// Our own glue (no reference code is copied here), compiled against the unmodified reference header
// scoretype.h with the parity flags into oracle/_ref/libref_math.so (see oracle/Makefile).  It evaluates
// the reference's own LOG_ADD (scoretype.h:120-124) and CalcPostFlat's score-to-probability expression
// (calcposteriorflat.cpp:15-20, the host libm's expf) on n inputs, for the arithmetic sweeps of
// tests/test_logadd_expf_cpu.py.  A library of its own, so that it is built wherever the reference is,
// whatever state an existing libmuscle_ref.so is in.
// Range forms: a[k] / s[k] is the float whose bits are first_bits + k; swap: out[k] = LOG_ADD(b, a[k]).
#include <cassert>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include "scoretype.h"

namespace {
float PostProb(float Score, float MinScore)
	{
	if (Score < MinScore)
		return 0;
	return Score >= LOG_ONE ? 1.0f : expf(Score);
	}

float BitsFloat(uint32_t u)
	{
	float f;
	memcpy(&f, &u, 4);
	return f;
	}
}

extern "C" {

void ref_log_add_n(uint64_t n, const float *a, const float *b, float *out)
	{
#pragma omp parallel for schedule(static)
	for (int64_t k = 0; k < (int64_t) n; ++k)
		out[k] = LOG_ADD(a[k], b[k]);
	}

void ref_log_add_range(uint64_t n, uint32_t a_first_bits, float b, int swap, float *out)
	{
#pragma omp parallel for schedule(static)
	for (int64_t k = 0; k < (int64_t) n; ++k)
		{
		const float a = BitsFloat(a_first_bits + (uint32_t) k);
		out[k] = swap ? LOG_ADD(b, a) : LOG_ADD(a, b);
		}
	}

void ref_post_prob_n(uint64_t n, const float *s, float min_score, float *out)
	{
#pragma omp parallel for schedule(static)
	for (int64_t k = 0; k < (int64_t) n; ++k)
		out[k] = PostProb(s[k], min_score);
	}

void ref_post_prob_range(uint64_t n, uint32_t s_first_bits, float min_score, float *out)
	{
#pragma omp parallel for schedule(static)
	for (int64_t k = 0; k < (int64_t) n; ++k)
		out[k] = PostProb(BitsFloat(s_first_bits + (uint32_t) k), min_score);
	}

}
