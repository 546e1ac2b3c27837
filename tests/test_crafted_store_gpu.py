"""GPU: the kernels that read the posterior store, on hand-built stores (tests/crafted_store.py), bit for bit
against the oracle (pinned to the compiled reference on the same stores by tests/test_crafted_store_cpu.py).

1. The decoding DP (k_densify + k_aln_wave) through mb200_align_pairs, one problem per call, over a grid of
   shapes: LX around the prefetch depth and the warp width, LY around the strip width and up to 4 CTAs per
   problem, tall and wide; then the same problems mixed in one batch.
2. Exact non-zero ties in every Best3 branch and values up to 1e6 (DP sums past 2**24).
3. The consistency iteration (k_mask_fill + k_relax) on empty pairs, empty and full rows and rows spanning
   many 32-column mask words, whole and as a split-range update.
4. BuildPost (k_bp_* and k_bpc_*) + the join's DP through mb200_align_groups under both routes, on gapped
   groups, and a join whose DP runs 3 CTAs.
5. Joins wider than 12544 columns, which the ordered row walk cannot hold in shared memory, through
   mb200_align_groups and mb200_msa_join, on a crafted store and on real posteriors."""
import numpy as np
import pytest
import crafted_store as cs
from muscle_b200 import synth

pytestmark = pytest.mark.gpu

ROUTES = ["0", "1000000000000"]          # BuildPost by cell / ordered row walk (MB200_BP_SORT_MIN)
AW_W, AW_MAXW = 128, 16                  # columns per strip, strips per CTA (align.cu)

LX_SET = [1, 2, 5, 6, 7, 13, 31, 32, 33, 64, 65, 300]
LY_SET = [1, 2, 3, 4, 5, 127, 128, 129, 2048, 2049, 4096, 4097, 6200]
TALL = 5000


def npass(LY):
	"""CTAs of a decoding DP over LY columns"""
	nstrips = (LY + AW_W - 1)//AW_W
	nw = min(AW_MAXW, nstrips)
	return (nstrips + nw - 1)//nw


def same_score(a, b):
	return np.float32(a).tobytes() == np.float32(b).tobytes()


def _pairs(n):
	return cs.pair_list(n)


@pytest.fixture(scope="module")
def grid(oracle):
	"""Sequences A = LX_SET, B = LY_SET + [TALL], A2 = LX_SET + [129]: the stored pairs (A, B) are every
	LX x LY of the grid, (B, A2) the same shapes turned over, plus TALL x 5 and TALL x 129.
	-> (lens, store, problems [(pair, LX, LY)], oracle results {pair: (score, path)})"""
	lens = LX_SET + LY_SET + [TALL] + LX_SET + [129]
	na, nb = len(LX_SET), len(LY_SET) + 1
	store = cs.make_store(lens, "mixed", 101)
	n = len(lens)
	probs = []
	for x in range(na):
		for y in range(na, na + nb):
			probs.append((cs.pair_index(n, x, y), lens[x], lens[y]))
	for x in range(na, na + nb):
		for y in range(na + nb, n):
			probs.append((cs.pair_index(n, x, y), lens[x], lens[y]))
	offs, ents = store
	want = {k: oracle.calcaln(cs.to_dense(offs[k], ents[k], LX, LY)) for k, LX, LY in probs}
	return lens, store, probs, want


def test_grid_covers_the_edges(grid):
	_, _, probs, _ = grid
	shapes = {(LX, LY) for _, LX, LY in probs}
	for v in LX_SET:
		assert (v, 1) in shapes and (v, 6200) in shapes and (1, v) in shapes and (TALL, v) in shapes
	for v in LY_SET:
		assert (1, v) in shapes and (300, v) in shapes and (v, 1) in shapes and (v, 300) in shapes
	assert (TALL, 5) in shapes and (TALL, 129) in shapes
	assert {npass(LY) for _, _, LY in probs} == {1, 2, 3, 4}


def test_decoder_shape_grid(engine, grid):
	lens, store, probs, want = grid
	cs.load(engine, lens, store)
	bad = []
	for k, LX, LY in probs:
		scores, paths = engine.align_pairs([k])
		s, path = want[k]
		if not (same_score(s, scores[0]) and paths[0] == path):
			bad.append((LX, LY))
	assert not bad, "decoder differs from the oracle at LX x LY = %s" % bad


def test_decoder_mixed_batch(engine, grid):
	"""one launch over a shuffled list with duplicates: 1 to 4 CTAs per problem, tiny shapes included"""
	lens, store, probs, want = grid
	cs.load(engine, lens, store)
	rng = np.random.default_rng(7)
	wide = [k for k, _, LY in probs if npass(LY) >= 3]
	tiny = [k for k, LX, LY in probs if LX <= 7 or LY <= 5]
	mid = [k for k, _, LY in probs if npass(LY) <= 2]
	sel = list(rng.choice(wide, 12)) + list(rng.choice(tiny, 20)) + list(rng.choice(mid, 20))
	sel += sel[:6]                                                      # duplicates
	rng.shuffle(sel)
	sel = [int(k) for k in sel]
	assert {npass(LY) for k, _, LY in probs if k in sel} == {1, 2, 3, 4}
	scores, paths = engine.align_pairs(sel)
	for q, k in enumerate(sel):
		s1, p1 = engine.align_pairs([k])
		s, path = want[k]
		assert same_score(scores[q], s1[0]) and paths[q] == p1[0], (q, k)
		assert same_score(scores[q], s) and paths[q] == path, (q, k)


@pytest.mark.parametrize("pattern", ["ties", "heavy"])
def test_decoder_ties_and_heavy(engine, oracle, pattern):
	lens = [300, 300, 700, 4200]
	store = cs.make_store(lens, pattern, 31)
	cs.load(engine, lens, store)
	offs, ents = store
	pairs = _pairs(len(lens))
	sel = list(range(len(pairs)))
	batch_s, batch_p = engine.align_pairs(sel)
	for k, (x, y) in enumerate(pairs):
		s, path = oracle.calcaln(cs.to_dense(offs[k], ents[k], lens[x], lens[y]))
		s1, p1 = engine.align_pairs([k])
		assert same_score(s, s1[0]) and path == p1[0], (lens[x], lens[y])
		assert same_score(s, batch_s[k]) and path == batch_p[k], (lens[x], lens[y])
	if pattern == "heavy":
		assert max(float(s) for s in batch_s) > 2.0**24


RELAX_LENS = [1, 5, 31, 64, 129, 400, 33, 250, 2, 300, 100, 7]


def test_relax_two_iterations(engine, oracle):
	lens = RELAX_LENS
	offs, ents = cs.make_store(lens, "mixed", 41)
	cs.load(engine, lens, (offs, ents))
	pairs = _pairs(len(lens))
	for it in range(2):
		want = oracle.conspair_many(lens, pairs, offs, ents)
		engine.consistency_iter()
		offs2, got = engine.export_all()
		for p in range(len(pairs)):
			assert np.array_equal(offs2[p], offs[p]), (it, p)
			assert got[p].tobytes() == want[p].tobytes(), ("iter", it, "pair", pairs[p])
		ents = got


def test_relax_split_range(engine, oracle):
	"""two half-range updates on copies of the store, the first one's values brought back == one full update"""
	lens = RELAX_LENS
	store = cs.make_store(lens, "mixed", 43)
	offs, ents = store
	pairs = _pairs(len(lens))
	want = oracle.conspair_many(lens, pairs, offs, ents)
	npairs = len(pairs)
	half = npairs//2
	cs.load(engine, lens, store)
	nnz, _ = engine.store_nnz()
	base = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
	engine.consistency_iter(0, half)
	va = engine.store_values_torch()
	cs.load(engine, lens, store)
	engine.consistency_iter(half, npairs)
	if base[half] > 0:
		engine.store_set_values_torch(va[:base[half]], 0)
	_, got = engine.export_all()
	for p in range(npairs):
		assert got[p].tobytes() == want[p].tobytes(), pairs[p]


def _check_join(engine, oracle, lens, offs, ents, ga, pa, ca, gb, pb, cb):
	want = oracle.buildpost(lens, ga, pa, ca, gb, pb, cb, offs, ents)
	score, path, post = engine.align_groups(ga, pa, ca, gb, pb, cb, want_post=True)
	assert post.tobytes() == want.tobytes(), "BuildPost"
	s, pth = oracle.calcaln(want)
	assert same_score(s, score) and pth == path, "decoding DP"
	return want


@pytest.mark.parametrize("bp_sort_min", ROUTES)
@pytest.mark.parametrize("pattern", ["mixed", "heavy", "ties"])
def test_buildpost_gapped_groups(engine, oracle, monkeypatch, bp_sort_min, pattern):
	"""members with full rows, empty pairs and wide-span rows; both orientations of the join"""
	monkeypatch.setenv("MB200_BP_SORT_MIN", bp_sort_min)
	lens = RELAX_LENS
	offs, ents = cs.make_store(lens, pattern, 47)
	cs.load(engine, lens, (offs, ents))
	rng = np.random.default_rng(53)
	ga, gb = [0, 2, 4, 5, 9], [1, 3, 6, 7, 8, 10, 11]
	ca, cb = max(lens[i] for i in ga) + 37, max(lens[i] for i in gb) + 23
	pa = [cs.gapped_map(rng, lens[i], ca) for i in ga]
	pb = [cs.gapped_map(rng, lens[i], cb) for i in gb]
	_check_join(engine, oracle, lens, offs, ents, ga, pa, ca, gb, pb, cb)
	_check_join(engine, oracle, lens, offs, ents, gb, pb, cb, ga, pa, ca)


@pytest.mark.parametrize("bp_sort_min", ROUTES)
def test_buildpost_join_three_passes(engine, oracle, monkeypatch, bp_sort_min):
	"""B spread over 4300 columns: the join's DP runs 3 CTAs"""
	monkeypatch.setenv("MB200_BP_SORT_MIN", bp_sort_min)
	lens = RELAX_LENS
	offs, ents = cs.make_store(lens, "mixed", 59)
	cs.load(engine, lens, (offs, ents))
	rng = np.random.default_rng(61)
	ga, gb = [5, 0, 11, 3], [9, 7, 1, 2, 4, 6, 8, 10]
	ca, cb = 450, 4300
	assert npass(cb) == 3
	pa = [cs.gapped_map(rng, lens[i], ca) for i in ga]
	pb = [cs.gapped_map(rng, lens[i], cb) for i in gb]
	post = _check_join(engine, oracle, lens, offs, ents, ga, pa, ca, gb, pb, cb)
	assert (post[:, 4096:] > 0).any()


WIDE = [12544, 12545, 13000]            # 12544: the widest join the ordered row walk can hold
WIDE_ROUTES = [None] + ROUTES            # None: the library's own choice (a 300 x 1 join is small: row walk)


def _set_route(monkeypatch, bp_sort_min):
	if bp_sort_min is None:
		monkeypatch.delenv("MB200_BP_SORT_MIN", raising=False)
	else:
		monkeypatch.setenv("MB200_BP_SORT_MIN", bp_sort_min)


def _wide_joins(engine, oracle, lens, offs, ents):
	"""A = sequence 0 (~300 residues) joined with each sequence of length in WIDE, through align_groups
	and msa_join (one sequence per group: each MSA has exactly as many columns as residues)"""
	for cb in WIDE:
		b = lens.index(cb)
		ca = lens[0]
		pa, pb = [np.arange(ca, dtype=np.uint32)], [np.arange(cb, dtype=np.uint32)]
		want = _check_join(engine, oracle, lens, offs, ents, [0], pa, ca, [b], pb, cb)
		s, pth = oracle.calcaln(want)
		engine.msa_reset()
		cols, score, path = engine.msa_join([0], [b], want_path=True)
		assert cols == len(path) and same_score(s, score) and path == pth, cb


@pytest.mark.parametrize("bp_sort_min", WIDE_ROUTES)
def test_wide_join_crafted(engine, oracle, monkeypatch, bp_sort_min):
	_set_route(monkeypatch, bp_sort_min)
	lens = [300] + WIDE
	pats = ["span", "full_rows", "ties", "band", "band", "band"]
	offs, ents = cs.make_store(lens, pats, 67)
	cs.load(engine, lens, (offs, ents))
	_wide_joins(engine, oracle, lens, offs, ents)


@pytest.fixture(scope="module")
def wide_family():
	base = synth.make_family(4, 13100, 0, seed=71, uniform=(13050, 13150))
	want = [300] + WIDE
	return [base[k][:n] for k, n in enumerate(want)]


@pytest.mark.parametrize("bp_sort_min", WIDE_ROUTES)
def test_wide_join_real_posteriors(engine, oracle, monkeypatch, wide_family, bp_sort_min):
	_set_route(monkeypatch, bp_sort_min)
	seqs = wide_family
	lens = [len(s) for s in seqs]
	assert lens == [300] + WIDE
	engine.set_seqs(seqs)
	engine.posteriors_allpairs()
	offs, ents = engine.export_all()
	_wide_joins(engine, oracle, lens, offs, ents)
