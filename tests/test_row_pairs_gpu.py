"""GPU: k_posterior_sm's plain-mode passes, which run two DP rows per lane per step, at the boundaries of
their row pairs.

A pair of even LX starts its Forward with an all-LOG_ZERO row -1, so that Forward and Backward pair the
rows (LX-1, LX), (LX-3, LX-2), ...; a pair of odd LX ends its Backward with row 0 as the second row of a
step.  The cases mix odd and even LX in one chain (LX = 1, 2 and 3 among them), put the cell (LX,LY) in
the only column of its lane, run multi-strip pairs of odd and even LX, fill a chain to its pair and row
limits, and force the widths 3, 4, 12, 14 and 16.  Every pair's sparse store and EA, and the dense
Forward-M, Backward-M, total and posterior of chosen pairs inside their chains, are compared with the CPU
oracle with tolerance 0; X are windows of a homolog of Y, so that rows keep several survivors.
"""
import numpy as np
import pytest
from test_chains_gpu import _homologs, _windows, check_dense, run_list

pytestmark = pytest.mark.gpu

MIXED_X = [1, 2, 3, 4, 5, 8, 31, 64, 65, 150, 151]


@pytest.fixture(scope="module")
def limits(engine):
	"""(most Forward rows, most pairs) of one chain, as the library reports them"""
	engine.set_seqs(["ACDEF", "GHIKL"])
	engine.posteriors([0], [1])
	p = engine.debug_plan()
	return p["chain_rows"], p["chain_pairs"]


def mixed_case(LY, seed):
	"""one Y of LY residues and a chain of MIXED_X windows of its homolog, odd and even LX alternating"""
	Y, H = _homologs(seed, LY, max(MIXED_X))
	X = _windows(H, LY, MIXED_X, np.random.default_rng(seed))
	return [Y] + X, list(range(1, len(X) + 1)), [0]*len(X)


def _dense_all(engine, oracle, seqs, px, py, which, force_c=0, tag=""):
	for k in which:
		check_dense(engine, oracle, seqs, px, py, k, force_c=force_c, tag=tag)


# LY = 33 at two columns per lane puts column LY alone in lane 16; 200 and 300 end mid-lane
@pytest.mark.parametrize("LY", [33, 200, 300])
def test_mixed_lx_chain(engine, oracle, LY):
	seqs, px, py = mixed_case(LY, 500 + LY)
	chains, _, _, _ = run_list(engine, oracle, seqs, px, py, tag="mixed LY=%d" % LY)
	assert [len(c) for c in chains] == [len(px)]
	# LX = 1, 2, 3 at the chain's start, and an even and an odd pair after them
	_dense_all(engine, oracle, seqs, px, py, [0, 1, 2, 7, 8], tag="mixed LY=%d" % LY)


@pytest.mark.parametrize("force_c", [3, 4, 12, 14, 16])
def test_forced_widths(engine, oracle, force_c):
	seqs, px, py = mixed_case(300, 800)
	run_list(engine, oracle, seqs, px, py, force_c=force_c, tag="forced C=%d" % force_c)
	_dense_all(engine, oracle, seqs, px, py, [0, 1, 2, 9, 10], force_c=force_c, tag="forced C=%d" % force_c)


def test_multi_strip(engine, oracle):
	"""Y of 1100 residues (three strips of 512 columns), X of odd and even length: chains of one pair"""
	Y, H = _homologs(900, 1100, 1100)
	lengths = [1, 2, 3, 150, 151, 1099]
	X = _windows(H, 1100, lengths, np.random.default_rng(9))
	seqs, px, py = [Y] + X, list(range(1, len(X) + 1)), [0]*len(X)
	chains, _, _, _ = run_list(engine, oracle, seqs, px, py, tag="multi-strip")
	assert all(len(c) == 1 for c in chains)
	_dense_all(engine, oracle, seqs, px, py, [0, 1, 2, 3, 4], tag="multi-strip")
	# the same with three columns per lane: more strips, and LY ends mid-lane
	run_list(engine, oracle, seqs, px, py, force_c=3, tag="multi-strip C=3")
	_dense_all(engine, oracle, seqs, px, py, [2, 4], force_c=3, tag="multi-strip C=3")


def test_full_chain(engine, oracle, limits):
	"""a chain of the most pairs whose Forward rows (sum of LX+2) are exactly the limit, odd and even LX
	mixed, so that the row -1 of every even pair adds to its steps; then one more pair on the same Y"""
	R, M = limits
	base = (R - 2*M)//M
	lengths = [base + d for d in (-2, -1, 1, 2)*(M//4)] + [base]*(M % 4)
	lengths[-1] += R - sum(L + 2 for L in lengths)
	lengths.append(7)
	Y, H = _homologs(1000, 300, max(lengths))
	X = _windows(H, 300, lengths, np.random.default_rng(10))
	seqs, px, py = [Y] + X, list(range(1, len(X) + 1)), [0]*len(X)
	lens = [len(s) for s in seqs]
	chains, _, _, _ = run_list(engine, oracle, seqs, px, py, tag="full chain")
	full = [c for c in chains if len(c) == M]
	assert len(full) == 1 and sum(lens[px[k]] + 2 for k in full[0]) == R
	assert {lens[px[k]] % 2 for k in full[0]} == {0, 1}
	_dense_all(engine, oracle, seqs, px, py, [0, 1, M - 1, M], tag="full chain")
