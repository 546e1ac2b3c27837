"""GPU: k_posterior_sm's LOG_ADD and posterior probability against the CPU oracle on every input of their
domain, bit for bit (mb200_debug_math runs the kernel's own device code).  The sweeps and the argument for
why they cover LOG_ADD are in tests/math_sweeps.py; test_logadd_expf_cpu.py pins the oracle to the compiled
reference on the same inputs.  GPU memory in use: one chunk buffer of the context (768 MB)."""
import numpy as np
import pytest
import math_sweeps as M
from conftest import load_tables
from oracle.pyoracle import bit_mismatches

pytestmark = pytest.mark.gpu


def _log_add(engine, oracle, cases, what):
	from muscle_b200.engine import MATH_LOG_ADD, MATH_LOG_ADD_BA
	for case in cases:
		if case[0] == "range":
			_, first, n, b, swap = case
			got = engine.debug_math(MATH_LOG_ADD_BA if swap else MATH_LOG_ADD, n, a_first_bits=first, b_scalar=b)
			want = oracle.log_add_range(n, first, b, swap)
			msg = bit_mismatches(got, want, first, "%s, b = %r%s" % (what, float(b), " (b, a)" if swap else ""))
		else:
			_, a, b = case
			got = engine.debug_math(MATH_LOG_ADD, a=a, b=b)
			msg = bit_mismatches(got, oracle.log_add_n(a, b), (a, b), what)
		assert msg is None, msg


def test_log_add_l1_pieces(engine, oracle):
	_log_add(engine, oracle, M.sweep_l1(), "L1")


def test_log_add_l2_cut_and_clamp(engine, oracle):
	_log_add(engine, oracle, M.sweep_l2(), "L2")


def test_log_add_l3_final_add(engine, oracle):
	_log_add(engine, oracle, M.sweep_l3(), "L3")


def test_log_add_l4_log_zero(engine, oracle, tables):
	_log_add(engine, oracle, M.sweep_l4(tables), "L4")


def test_log_add_l5_random(engine, oracle):
	_log_add(engine, oracle, M.sweep_l5(), "L5")


def _post_prob(engine, oracle, first, last, min_score, what):
	from muscle_b200.engine import MATH_POST_PROB
	for _, k, n, _, _ in M.ranges(first, last):
		got = engine.debug_math(MATH_POST_PROB, n, a_first_bits=k)
		msg = bit_mismatches(got, oracle.post_prob_range(n, k, min_score), k, what)
		assert msg is None, msg


def _keep(engine, oracle, first, last, min_score, what):
	"""the kernel's kept decision on the score == (the probability CalcPostFlat writes >= 0.01f)"""
	from muscle_b200.engine import MATH_KEEP
	for _, k, n, _, _ in M.ranges(first, last):
		got = engine.debug_math(MATH_KEEP, n, a_first_bits=k)
		want = (oracle.post_prob_range(n, k, min_score) >= np.float32(0.01)).astype(np.float32)
		msg = bit_mismatches(got, want, k, what)
		assert msg is None, msg


def test_post_prob_e1(engine, oracle, tables):
	_post_prob(engine, oracle, *M.E1, tables["min_sparse_score"], "E1")


def test_post_prob_e2_outside(engine, oracle, tables):
	for lo, hi in M.E2:
		_post_prob(engine, oracle, lo, hi, tables["min_sparse_score"], "E2")


def test_keep_e3(engine, oracle, tables):
	_keep(engine, oracle, *M.E3, tables["min_sparse_score"], "E3")


def test_post_prob_and_keep_e4_lower_min_score(oracle):
	"""min_sparse_score = logf(0.001f): POST_PROB follows it, the kept threshold stays at logf(0.01f)"""
	from muscle_b200.engine import Engine
	t = dict(load_tables())
	t["min_sparse_score"] = M.libm_logf(0.001)
	e = Engine(0)
	try:
		e.set_hmm(t)
		_post_prob(e, oracle, *M.E1, t["min_sparse_score"], "E4/E1")
		_keep(e, oracle, *M.E3, t["min_sparse_score"], "E4/E3")
	finally:
		e.close()


def test_debug_math_rejects_bad_calls(engine):
	from muscle_b200.engine import MB200Error, MATH_KEEP
	lib = engine.lib
	out = np.empty(4, np.float32)
	assert lib.mb200_debug_math(None, 0, 4, None, 0, None, 0.0, out.ctypes.data) == -1
	for op in (-1, MATH_KEEP + 1):
		with pytest.raises(MB200Error):
			engine.debug_math(op, 4)
	assert engine.debug_math(MATH_KEEP, 0).size == 0
