"""GPU: k_posterior_sm's expected accuracy and sparse store, with the EA of one-strip pairs computed from the
candidate entries through a prefix-max tree (tests/test_sparse_ea_cpu.py has the argument and a model of
it) and that of multi-strip pairs by the dense strip sweep.  Every case compares the row offsets, the entry
bytes and the EA of every pair with the CPU oracle (or the Mega goldens) at tolerance 0.

Cases: all pairs of part of C2; all pairs of a repeat family and the repeat pairs of tests/repeat_util.py,
whose rows keep more than 32 and 64 entries and so take several 32-entry batches; a cut so high that no pair has a candidate (EA 0, empty store); a chain
of as many pairs on one Y as a chain holds; every forced width 1-16 on a list with one-strip and
multi-strip pairs; a pair whose Y needs several strips at full width; a Mega model."""
import numpy as np
import pytest
import mega_util
import repeat_util as ru
from muscle_b200 import synth

pytestmark = pytest.mark.gpu

_cache = {}


def _want(oracle, X, Y):
	"""oracle (row offsets, entry bytes, EA as float32) of pair (X, Y)"""
	key = (id(oracle), X, Y)
	if key not in _cache:
		p = oracle.post(X, Y)
		off, ent = oracle.sparse(p)
		ea = np.float32(np.float32(oracle.alnscore(p))/np.float32(min(len(X), len(Y))))
		_cache[key] = (off, ent.tobytes(), ea)
	return _cache[key]


def check_list(engine, oracle, seqs, px, py, force_c=0, tag=""):
	"""posteriors of the pair list against the oracle; -> (EA, entries per pair)"""
	engine.set_seqs(seqs)
	ea = engine.posteriors(px, py, force_c=force_c)
	offs, ents = engine.export_all()
	for k, (x, y) in enumerate(zip(px, py)):
		off, ent, want_ea = _want(oracle, seqs[x], seqs[y])
		assert np.array_equal(offs[k], off), "%s pair %d (%d, %d): row offsets" % (tag, k, x, y)
		assert ents[k].tobytes() == ent, "%s pair %d (%d, %d): entries" % (tag, k, x, y)
		assert np.float32(ea[k]).tobytes() == want_ea.tobytes(), "%s pair %d: EA %r != %r" % (tag, k, ea[k], want_ea)
	return ea, [len(e) for e in ents]


def check_allpairs(engine, oracle, seqs):
	"""all pairs of seqs against the oracle's all_pairs; -> most entries in one row"""
	n = len(seqs)
	r = oracle.all_pairs(seqs, threads=0)
	engine.set_seqs(seqs)
	ea = engine.posteriors_allpairs()
	iu = np.triu_indices(n, 1)
	assert ea.tobytes() == r["ea"][iu].astype(np.float32).tobytes()
	offs, ents = engine.export_all()
	for k in range(len(offs)):
		assert np.array_equal(offs[k], r["row_off"][k]) and ents[k].tobytes() == r["entries"][k].tobytes(), k
	return max(int(np.diff(o.astype(np.int64)).max()) for o in offs)


def _homolog_windows(seed, LY, lengths):
	"""Y of LY residues and windows of a homolog of it, so that the pairs have candidates"""
	L = max(LY, max(lengths))
	Y, H = synth.make_family(2, L, 0, seed=seed, min_len=1)
	rng = np.random.default_rng(seed)
	X = []
	for n in lengths:
		a = int(rng.integers(0, max(0, len(H) - n) + 1))
		X.append(H[a:a + n])
	return Y[:LY], X


def test_c2_allpairs(engine, oracle):
	seqs = synth.make_config("C2")[:48]
	assert check_allpairs(engine, oracle, seqs) > 0


def test_repeat_family(engine, oracle):
	assert check_allpairs(engine, oracle, ru.repeat_family(12, ru.REPEAT_SEED)) > 32


def test_repeat_pairs(engine, oracle):
	"""the repeat pairs whose rows keep more than 64 entries, so hold at least as many candidates"""
	seqs = [s for xy in ru.DENSE_PAIRS for s in xy]
	px, py = list(range(0, len(seqs), 2)), list(range(1, len(seqs), 2))
	check_list(engine, oracle, seqs, px, py, tag="repeat pairs")
	offs, _ = engine.export_all()
	assert max(np.diff(o.astype(np.int64)).max() for o in offs) > 64


def test_no_candidates(engine, oracle, tables):
	"""a cut of p >= 0.95: no cell of these pairs reaches it, so the EA is 0 and the store is empty"""
	from oracle.pyoracle import Oracle
	t = dict(tables)
	t["min_sparse_score"] = np.float32(-0.05)
	rng = np.random.default_rng(8)
	seqs = ["".join(rng.choice(list(synth.AMINO), L)) for L in (40, 300, 120, 7, 500)]
	seqs += synth.make_family(2, 200, 20, seed=9)
	px, py = [0, 2, 3, 1, 5, 4], [1, 1, 4, 4, 6, 3]
	engine.set_hmm(t)
	try:
		ea, nnz = check_list(engine, Oracle(t), seqs, px, py, tag="no candidates")
	finally:
		engine.set_hmm(tables)
	assert not np.any(ea) and not any(nnz)


def test_full_chain(engine, oracle):
	"""as many pairs on one Y as a chain holds, the longest X that lets them all fit"""
	engine.set_seqs(["ACDEF", "GHIKL"])
	engine.posteriors([0], [1])
	p = engine.debug_plan()
	M, R = p["chain_pairs"], p["chain_rows"]
	LX = R//M - 2
	Y, X = _homolog_windows(31, 300, [1 + (k*13) % LX for k in range(M - 1)] + [LX])
	check_list(engine, oracle, [Y] + X, list(range(1, M + 1)), [0]*M, tag="full chain")
	p = engine.debug_plan()
	assert np.diff(p["chain"]).max() == M


def _width_list():
	"""Y of 40, 300 and 700 residues with X windows of their homologs"""
	seqs, px, py = [], [], []
	for s, LY in enumerate((40, 300, 700)):
		Y, X = _homolog_windows(40 + s, LY, [1, 30, 90, 200])
		y = len(seqs)
		seqs.append(Y)
		for x in X:
			px.append(len(seqs))
			py.append(y)
			seqs.append(x)
	return seqs, px, py


@pytest.mark.parametrize("force_c", range(1, 17))
def test_forced_widths(engine, oracle, force_c):
	seqs, px, py = _width_list()
	ea, nnz = check_list(engine, oracle, seqs, px, py, force_c, tag="C=%d" % force_c)
	assert np.count_nonzero(ea) == len(px) and all(nnz)


def test_multi_strip(engine, oracle):
	"""Y longer than the 32 lanes x 16 columns of the widest class: the strip path at full width"""
	Y, X = _homolog_windows(50, 1100, [60, 700])
	ea, nnz = check_list(engine, oracle, [Y] + X, [1, 2], [0, 0], tag="multi-strip")
	assert len(Y) > 32*16 and np.all(ea > 0) and all(nnz)


def test_mega(engine, oracle):
	model, profiles, posts = mega_util.load_model()
	px = [0, 1, 2, 0, 2, 1]
	py = [3]*len(px)
	engine.set_seqs_mega(model, profiles)
	ea = engine.posteriors(px, py)
	offs, ents = engine.export_all()
	for k, x in enumerate(px):
		want = posts[(x, 3)]
		o, e = oracle.sparse(want)
		assert np.array_equal(offs[k], o) and ents[k].tobytes() == e.tobytes(), (k, x)
		assert np.float32(ea[k]) == np.float32(np.float32(oracle.alnscore(want))/np.float32(min(want.shape))), (k, x)
