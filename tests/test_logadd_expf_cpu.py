"""CPU: the oracle's LOG_ADD and posterior probability against the compiled reference's own (scoretype.h's
LOG_ADD, calcposteriorflat.cpp's expression with the host libm's expf), bit for bit on the sweeps of
tests/math_sweeps.py -- exhaustive where test_logadd_expf_gpu.py is, so that device = oracle = reference on
every input.  Also pins the host libm's expf to glibc 2.39's, the one the device restatement
mb_expf_glibc was checked against, and checks on every score the device compares with that the kept
decision k_posterior_sm takes on the score (>= logf(0.01f)) is the reference's (expf(score) >= 0.01f)."""
import ctypes
import ctypes.util
import os
import numpy as np
import pytest
import math_sweeps as M
from conftest import GOLDEN
from oracle.pyoracle import bit_mismatches


@pytest.fixture(scope="module")
def ref():
	"""the reference's own LOG_ADD and posterior probability; present where oracle/_ref was built"""
	from oracle.pyoracle import RefMath, REF_MATH_SO
	if not os.path.exists(REF_MATH_SO):
		pytest.skip("oracle/_ref/libref_math.so not built")
	return RefMath()


def _log_add(oracle, ref, cases, what):
	for case in cases:
		if case[0] == "range":
			_, first, n, b, swap = case
			msg = bit_mismatches(oracle.log_add_range(n, first, b, swap), ref.log_add_range(n, first, b, swap), first,
			  "%s, b = %r%s" % (what, float(b), " (b, a)" if swap else ""))
		else:
			_, a, b = case
			msg = bit_mismatches(oracle.log_add_n(a, b), ref.log_add_n(a, b), (a, b), what)
		assert msg is None, msg


def test_log_add_l1_pieces(oracle, ref):
	_log_add(oracle, ref, M.sweep_l1(), "L1")


def test_log_add_l2_to_l5(oracle, ref, tables):
	_log_add(oracle, ref, M.sweep_l2(), "L2")
	_log_add(oracle, ref, M.sweep_l3(), "L3")
	_log_add(oracle, ref, M.sweep_l4(tables), "L4")
	_log_add(oracle, ref, M.sweep_l5(), "L5")


def _post_prob(oracle, ref, first, last, min_score, what):
	for _, k, n, _, _ in M.ranges(first, last):
		msg = bit_mismatches(oracle.post_prob_range(n, k, min_score), ref.post_prob_range(n, k, min_score), k, what)
		assert msg is None, msg


def test_post_prob_e1_e2_e4(oracle, ref, tables):
	_post_prob(oracle, ref, *M.E1, tables["min_sparse_score"], "E1")
	for lo, hi in M.E2:
		_post_prob(oracle, ref, lo, hi, tables["min_sparse_score"], "E2")
	_post_prob(oracle, ref, *M.E3, M.libm_logf(0.001), "E4")


@pytest.mark.parametrize("min_score", ["default", "logf(0.001f)"])
def test_keep_is_a_compare_of_the_score(ref, tables, min_score):
	"""E3: for every score from 1024 floats below logf(0.01f) up to -0.0, the reference keeps the cell
	(p >= 0.01f) exactly when score >= logf(0.01f), the compare k_posterior_sm makes"""
	ms = tables["min_sparse_score"] if min_score == "default" else M.libm_logf(0.001)
	thr = M.f32(M.KEEP_BITS)
	for _, k, n, _, _ in M.ranges(*M.E3):
		kept = ref.post_prob_range(n, k, ms) >= np.float32(0.01)
		s = M.f32(np.arange(k, k + n, dtype=np.uint64).astype(np.uint32))
		msg = bit_mismatches((s >= thr).astype(np.float32), kept.astype(np.float32), k, "kept decision")
		assert msg is None, msg


def test_host_expf_is_glibc_2_39():
	"""the reference's probabilities are the host libm's expf; the golden holds glibc 2.39's bits on every
	4096th float in [-4.7, 0] and on the 4096 floats nearest logf(0.01f)"""
	z = np.load(os.path.join(GOLDEN, "expf_glibc.npz"))
	libm = ctypes.CDLL(ctypes.util.find_library("m"))
	libm.expf.restype = ctypes.c_float
	libm.expf.argtypes = [ctypes.c_float]
	x = z["x_bits"].view(np.float32)
	got = np.array([libm.expf(float(v)) for v in x], np.float32)
	msg = bit_mismatches(got, z["expf_bits"].view(np.float32), (x,), "host expf vs glibc 2.39")
	assert msg is None, ("this host's libm expf is not glibc 2.39's: the reference's own posteriors moved, and "
	  "mb_expf_glibc (checked against glibc 2.39) no longer matches them. " + msg)
