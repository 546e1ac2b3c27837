"""GPU: the posterior, consistency and BuildPost kernels on repeat-rich sequences (tests/repeat_util.py),
whose posterior rows hold up to 83 entries >= 0.01 instead of the ~7 of the other inputs.  Everything is
compared with the CPU oracle with tolerance 0.  tests/test_dense_rows_cpu.py checks that these inputs
reach the paths they are chosen for and pins the oracle to the compiled reference on them.

Paths reached: survivor lists longer than 32 and 64 per row in k_posterior_sm, row counts carried across
strips, compaction in several 32-entry groups, posteriors next to the 0.01 cut; k_relax with several entry
sweeps per pair, several z chunks and many common columns per mask word; BuildPost rows longer than the
16 staged entries."""
import numpy as np
import pytest
import repeat_util as ru
from test_msa_gpu import host_join, project, rows_from_device

pytestmark = pytest.mark.gpu

FORCED = [0, 1, 2, 3, 5, 8, 16]


def _pairs(n):
	return [(i, j) for i in range(n) for j in range(i + 1, n)]


_cache = {}


def _want(oracle, X, Y):
	"""oracle (posterior, row offsets, entry bytes, EA as float32) of pair (X, Y)"""
	key = (X, Y)
	if key not in _cache:
		p = oracle.post(X, Y)
		off, ent = oracle.sparse(p)
		ea = np.float32(np.float32(oracle.alnscore(p))/np.float32(min(len(X), len(Y))))
		_cache[key] = (p, off, ent.tobytes(), ea)
	return _cache[key]


def export_store(engine):
	"""export_all, once every pair's entry count is possible: a row holds at most 100 entries >= 0.01
	(they sum to at most 1), so a larger count is wrong and the store is not worth copying.  Every row's
	columns must then lie inside the pair and ascend: the consistency and BuildPost kernels, and the
	oracle, index by column, so a store that breaks this fails here before either reads it."""
	nnz, _ = engine.store_nnz()
	px, py = engine._pairs
	rows = engine.lens[px]
	bad = np.flatnonzero(nnz > 100*rows)
	assert len(bad) == 0, "pair %d: %d entries in %d rows" % (bad[0], nnz[bad[0]], rows[bad[0]])
	offs, ents = engine.export_all()
	for k in range(len(offs)):
		LX, LY = int(engine.lens[px[k]]), int(engine.lens[py[k]])
		col = ents[k]["col"].astype(np.int64)
		assert offs[k][-1] == len(col), "pair %d: the rows hold %d entries, the pair %d" % (k, offs[k][-1], len(col))
		key = np.repeat(np.arange(LX), np.diff(offs[k].astype(np.int64)))*LY + col
		assert (col < LY).all() and (np.diff(key) > 0).all(), "pair %d: columns out of order or out of range" % k
	return offs, ents


def check_store(engine, oracle, seqs, px, py, ea, tag=""):
	offs, ents = export_store(engine)
	for k, (x, y) in enumerate(zip(px, py)):
		_, off, ent, want_ea = _want(oracle, seqs[x], seqs[y])
		assert np.array_equal(offs[k], off), "%s pair %d (%d, %d): row offsets" % (tag, k, x, y)
		assert ents[k].tobytes() == ent, "%s pair %d (%d, %d): entries" % (tag, k, x, y)
		assert np.float32(ea[k]) == want_ea, "%s pair %d (%d, %d): EA %r != %r" % (tag, k, x, y, ea[k], want_ea)
	return offs, ents


def check_dense(engine, oracle, seqs, px, py, which, force_c=0, tag=""):
	"""Forward-M, Backward-M, total and dense posterior of store pair `which`, run inside its list"""
	X, Y = seqs[px[which]], seqs[py[which]]
	post, fwd, bwd, tot = engine.calc_post_dense_pair(px, py, which, force_c=force_c)
	f, b = oracle.fwd(X, Y), oracle.bwd(X, Y)
	tag = "%s pair %d (%d x %d)" % (tag, which, len(X), len(Y))
	assert fwd.tobytes() == np.ascontiguousarray(f[1:, 1:, 0]).tobytes(), tag + ": Forward M"
	assert bwd.tobytes() == np.ascontiguousarray(b[1:, 1:, 0]).tobytes(), tag + ": Backward M"
	assert np.float32(tot) == np.float32(oracle.total(f, b)), tag + ": total"
	assert post.tobytes() == _want(oracle, X, Y)[0].tobytes(), tag + ": dense posterior"


def dense_list():
	"""every DENSE_PAIRS pair as a pair list over one sequence set"""
	seqs = [s for xy in ru.DENSE_PAIRS for s in xy]
	return seqs, list(range(0, len(seqs), 2)), list(range(1, len(seqs), 2))


def to_dense(off, ent, LX, LY):
	dense = np.zeros((LX, LY), np.float32)
	rows = np.repeat(np.arange(LX), np.diff(off.astype(np.int64)))
	dense[rows, ent["col"]] = ent["p"]
	return dense


# ------------------------------------------------------------------------------------------------
# posterior kernel
@pytest.mark.parametrize("force_c", FORCED)
def test_dense_pairs_dumps(engine, oracle, force_c):
	seqs, px, py = dense_list()
	engine.set_seqs(seqs)
	for k in range(len(px)):
		check_dense(engine, oracle, seqs, [px[k]], [py[k]], 0, force_c, "C=%d" % force_c)


@pytest.mark.parametrize("force_c", FORCED)
def test_dense_pairs_store(engine, oracle, force_c):
	seqs, px, py = dense_list()
	engine.set_seqs(seqs)
	ea = engine.posteriors(px, py, force_c=force_c)
	offs, _ = check_store(engine, oracle, seqs, px, py, ea, "C=%d" % force_c)
	assert max(np.diff(o.astype(np.int64)).max() for o in offs) > 64


def test_dense_rows_in_chains(engine, oracle):
	"""several X on one repeat Y, so that dense pairs run at chain positions > 0"""
	Y = ru.tandem("QQQP", 500)
	rng = np.random.default_rng(4)
	X = [ru.mutate(rng, ru.tandem("QQQP", L, L % 4), 0.03) for L in (30, 60, 45, 90, 120, 75, 20, 100)]
	X += [ru.tandem("PPG", 80, 1), ru.DENSE_PAIRS[0][0]]
	seqs = [Y] + X
	px, py = list(range(1, len(seqs))), [0]*len(X)
	engine.set_seqs(seqs)
	ea = engine.posteriors(px, py)
	plan = engine.debug_plan()
	order, chain = plan["order"].tolist(), plan["chain"].tolist()
	chains = [order[chain[c]:chain[c + 1]] for c in range(len(chain) - 1)]
	assert sum(len(X[k]) + 2 for k in range(len(X))) <= plan["chain_rows"] and len(X) <= plan["chain_pairs"]
	assert chains == [list(range(len(X)))], "the pairs on one Y do not form one chain: %r" % chains
	offs, _ = check_store(engine, oracle, seqs, px, py, ea, "chain")
	assert max(np.diff(o.astype(np.int64)).max() for o in offs[1:]) > 32
	ch = chains[0]
	for q in sorted({1, len(ch)//2, len(ch) - 1}):
		check_dense(engine, oracle, seqs, px, py, ch[q], tag="chain position %d" % q)


def test_dense_entry_pool_retry(engine, oracle):
	seqs, px, py = dense_list()
	engine.set_seqs(seqs)                  # forget the entry count of the last run
	engine.set_nnz_per_row_cap(1)
	try:
		k0 = engine.stats()["kernel_launches"]
		ea = engine.posteriors(px, py)
		launches = engine.stats()["kernel_launches"] - k0
	finally:
		engine.set_nnz_per_row_cap(12)
	nbins = int((np.diff(engine.debug_plan()["bin_start"][1:]) > 0).sum())
	assert launches == 2*nbins, "the entry pool did not overflow (%d launches, %d bins)" % (launches, nbins)
	check_store(engine, oracle, seqs, px, py, ea, "retry")


# ------------------------------------------------------------------------------------------------
# consistency
@pytest.fixture(scope="module")
def family():
	return ru.repeat_family(12, ru.REPEAT_SEED)


def test_consistency_repeat_family(engine, oracle, family):
	seqs = family
	lens = [len(s) for s in seqs]
	pairs = _pairs(len(seqs))
	engine.set_seqs(seqs)
	engine.posteriors_allpairs()
	offs, ents = export_store(engine)
	assert sum(len(e) > 2048 for e in ents) > 0
	for it in range(2):
		want = oracle.conspair_many(lens, pairs, offs, ents)
		engine.consistency_iter()
		offs2, got = export_store(engine)
		for p in range(len(pairs)):
			assert np.array_equal(offs2[p], offs[p]), (it, p)
			assert got[p].tobytes() == want[p].tobytes(), "iter %d pair %d %r" % (it, p, pairs[p])
		ents = got


def test_consistency_split_ranges(engine, oracle, family):
	"""two half-range calls, as two ranks would make them, split between two pairs of > 1024 entries"""
	seqs = family
	lens = [len(s) for s in seqs]
	pairs = _pairs(len(seqs))
	npairs = len(pairs)
	engine.set_seqs(seqs)
	engine.posteriors_allpairs()
	offs, ents = export_store(engine)
	want = oracle.conspair_many(lens, pairs, offs, ents)
	nnz, _ = engine.store_nnz()
	base = np.concatenate([[0], np.cumsum(nnz.astype(np.int64))])
	cuts = [h for h in range(1, npairs) if nnz[h - 1] > 1024 and nnz[h] > 1024]
	assert len(cuts) >= 2
	for h in (cuts[0], cuts[len(cuts)//2]):
		engine.posteriors_allpairs()
		engine.consistency_iter(0, h)
		va = engine.store_values_torch()
		engine.posteriors_allpairs()
		engine.consistency_iter(h, npairs)
		engine.store_set_values_torch(va[:int(base[h])], 0)
		_, got = engine.export_all()
		for p in range(npairs):
			assert got[p].tobytes() == want[p].tobytes(), "split at %d: pair %d" % (h, p)


@pytest.mark.parametrize("n", [65, 130])
def test_consistency_z_chunks(engine, oracle, n):
	"""N past one and two 64-sequence z chunks of k_relax, on a subset of the pairs: every pair of 0, 63, 64
	or N-1, the pairs of two repeats, and seeded random pairs"""
	seqs = ru.mixed_family(n, 7)
	lens = [len(s) for s in seqs]
	pairs = _pairs(n)
	slots = ru.repeat_slots(n)
	edge = {0, 63, 64, n - 1}
	sel = {p for p, (x, y) in enumerate(pairs) if x in edge or y in edge or (x in slots and y in slots)}
	sel |= set(np.random.default_rng(n).choice(len(pairs), 150, replace=False).tolist())
	sel = sorted(sel)
	engine.set_seqs(seqs)
	engine.posteriors_allpairs()
	offs, ents = export_store(engine)
	assert max(len(ents[p]) for p in sel) > 1024
	for it in range(2):
		want = oracle.conspair_many(lens, [pairs[p] for p in sel], offs, ents)
		engine.consistency_iter()
		_, got = export_store(engine)
		for p, w in zip(sel, want):
			assert got[p].tobytes() == w.tobytes(), "N=%d iter %d pair %d %r" % (n, it, p, pairs[p])
		ents = got


# ------------------------------------------------------------------------------------------------
# BuildPost and decoding
@pytest.mark.parametrize("bp_sort_min", ["1000000000000", "0"])      # ordered row walk / contributions sorted by cell
def test_align_groups_dense(engine, oracle, family, monkeypatch, bp_sort_min):
	monkeypatch.setenv("MB200_BP_SORT_MIN", bp_sort_min)
	seqs = family
	lens = [len(s) for s in seqs]
	engine.set_seqs(seqs)
	engine.posteriors_allpairs()
	export_store(engine)
	engine.consistency_iter()
	offs, ents = export_store(engine)
	rows_a, p2c_a = ru.staggered_rows(seqs, ru.GROUP_A)
	rows_b, p2c_b = ru.staggered_rows(seqs, ru.GROUP_B)
	ca, cb = len(rows_a[0]), len(rows_b[0])
	for ids1, p1, c1, ids2, p2, c2 in ((ru.GROUP_A, p2c_a, ca, ru.GROUP_B, p2c_b, cb),
	  (ru.GROUP_B, p2c_b, cb, ru.GROUP_A, p2c_a, ca)):
		assert ru.operand_row_counts(lens, ids1, ids2, offs, ents).max() > 16
		want = oracle.buildpost(lens, ids1, p1, c1, ids2, p2, c2, offs, ents)
		score, path, post = engine.align_groups(ids1, p1, c1, ids2, p2, c2, want_post=True)
		assert post.tobytes() == want.tobytes(), ("BuildPost", ids1)
		s, pth = oracle.calcaln(want)
		assert np.float32(s) == np.float32(score) and pth == path, ("CalcAlnFlat", ids1)


@pytest.mark.parametrize("bp_sort_min", ["1000000000000", "0"])
def test_msa_join_dense(engine, family, monkeypatch, bp_sort_min):
	"""progressive joins and refinement on the device against the same joins on the host
	(tests/test_msa_gpu.py)"""
	monkeypatch.setenv("MB200_BP_SORT_MIN", bp_sort_min)
	seqs = family
	n = len(seqs)
	engine.set_seqs(seqs)
	engine.posteriors_allpairs()
	export_store(engine)
	engine.consistency_iter()
	export_store(engine)
	engine.msa_reset()
	rng = np.random.default_rng(12)
	host = {i: [(i, seqs[i])] for i in range(n)}
	nodes = list(range(n))
	nxt = n
	while len(nodes) > 1:
		a, b = (int(v) for v in rng.choice(nodes, 2, replace=False))
		joined, path, score = host_join(engine, host[a], host[b])
		cols, dscore, dpath = engine.msa_join([i for i, _ in host[a]], [i for i, _ in host[b]], want_path=True)
		assert dpath == path and np.float32(dscore) == np.float32(score)
		assert cols == len(joined[0][1])
		nodes = [x for x in nodes if x not in (a, b)] + [nxt]
		host[nxt] = joined
		nxt += 1
	msa = host[nodes[0]]
	assert rows_from_device(engine, seqs, [i for i, _ in msa]) == msa
	for it in range(6):
		pick = rng.random(len(msa)) < 0.5
		g1 = [x for x, f in zip(msa, pick) if f]
		g2 = [x for x, f in zip(msa, pick) if not f]
		if not g1 or not g2:
			continue
		m1 = [(i, r) for (i, _), r in zip(g1, project([r for _, r in g1]))]
		m2 = [(i, r) for (i, _), r in zip(g2, project([r for _, r in g2]))]
		msa, path, score = host_join(engine, m1, m2)
		cols, dscore, dpath = engine.msa_join([i for i, _ in m1], [i for i, _ in m2], want_path=True)
		assert dpath == path and np.float32(dscore) == np.float32(score), it
		assert rows_from_device(engine, seqs, [i for i, _ in msa]) == msa, it


def test_align_pairs_dense(engine, oracle, family):
	seqs = family
	engine.set_seqs(seqs)
	engine.posteriors_allpairs()
	offs, ents = export_store(engine)
	pairs = _pairs(len(seqs))
	scores, paths = engine.align_pairs(list(range(len(pairs))))
	for k, (x, y) in enumerate(pairs):
		s, path = oracle.calcaln(to_dense(offs[k], ents[k], len(seqs[x]), len(seqs[y])))
		assert np.float32(s) == scores[k] and path == paths[k], (k, x, y)
