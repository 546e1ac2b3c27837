"""CPU: the C oracle on hand-built posterior stores (tests/crafted_store.py).

The GPU tests of the decoding DP, BuildPost and the consistency iteration on these stores compare
against the oracle.  The oracle was pinned to the compiled reference on posterior-built stores only,
so here it is pinned again, with tolerance 0, on the crafted ones: exact non-zero ties, values up to
1e6, empty pairs and rows, full rows and rows spanning the whole width.  The first tests need no
reference: the helper's stores reach the shapes they are meant to, and CalcAlnFlat of the oracle
equals a literal float32 transcription of it."""
import numpy as np
import pytest
import crafted_store as cs

# sequence lengths of the consistency and BuildPost stores: 1..~400, with widths past 4 mask words
LENS = [1, 5, 31, 64, 129, 400, 33, 250, 2, 300, 100, 7]


@pytest.fixture(scope="module")
def store():
	return cs.make_store(LENS, "mixed", 11)


def _pairs(n):
	return cs.pair_list(n)


def test_store_reaches_its_shapes(store):
	offs, ents = store
	pairs = _pairs(len(LENS))
	counts = [np.diff(o.astype(np.int64)) for o in offs]
	assert any(len(e) == 0 for e in ents), "no empty pair"
	assert any(len(e) > 0 and (c == 0).any() for c, e in zip(counts, ents)), "no empty row inside a non-empty pair"
	full = [int(c.max()) for (x, y), c in zip(pairs, counts) if LENS[x] > 0 and len(c) and c.max() == LENS[y]]
	assert max(full) > 128, "no full row past MB200_MAX_ROW_NNZ = 128 entries"
	spans = 0
	for (x, y), o, e in zip(pairs, offs, ents):
		for i in range(LENS[x]):
			c = e["col"][o[i]:o[i + 1]]
			if len(c) and c[0] == 0 and c[-1] == LENS[y] - 1 and LENS[y] > 4*32:
				spans += 1
	assert spans > 50, "too few rows spanning 4 or more mask words from column 0 to column LY-1"
	vals = np.concatenate([e["p"] for e in ents])
	assert vals.max() > 1e5 and (vals == 0.5).sum() > 100


def _calcaln_f32(post):
	"""CalcAlnFlat (calcalnflat.cpp, best3.h) transcribed literally with float32 scalars"""
	LX, LY = post.shape
	f = np.float32
	prev = [f(0)]*(LY + 1)
	tb = [["Y"]*(LY + 1)] + [["X"] + [""]*LY for _ in range(LX)]
	for i in range(1, LX + 1):
		cur = [f(0)]*(LY + 1)
		for j in range(1, LY + 1):
			b, x, y = f(prev[j - 1] + post[i - 1, j - 1]), prev[j], cur[j - 1]
			if b >= x and b >= y:
				cur[j], tb[i][j] = b, "B"
			elif x > b and x >= y:
				cur[j], tb[i][j] = x, "X"
			else:
				cur[j], tb[i][j] = y, "Y"
		prev = cur
	path, i, j = [], LX, LY
	while i or j:
		t = tb[i][j]
		path.append(t)
		i -= t != "Y"
		j -= t != "X"
	return prev[LY], "".join(reversed(path))


def dense_cases():
	"""crafted CalcAlnFlat inputs: ties in every Best3 branch, heavy values, 1x1, 1xN, Nx1, all-zero"""
	rng = np.random.default_rng(5)
	out = [np.zeros((1, 1), np.float32), np.ones((1, 1), np.float32), np.zeros((6, 9), np.float32),
	  np.full((7, 7), 0.5, np.float32), np.full((1, 13), 0.25, np.float32), np.full((13, 1), 0.25, np.float32),
	  rng.uniform(0, 1, (1, 40)).astype(np.float32), rng.uniform(0, 1, (40, 1)).astype(np.float32)]
	for LX, LY, pat in [(23, 31, "ties"), (31, 23, "ties"), (40, 40, "heavy"), (17, 60, "full_rows"), (60, 17, "span"),
	  (25, 25, "scatter"), (30, 12, "empty")]:
		off, ent = cs.make_pair(rng, LX, LY, pat)
		out.append(cs.to_dense(off, ent, LX, LY))
	out.append(rng.choice(np.array([0, 0.25, 0.5, 1], np.float32), size=(20, 20)))
	out.append((10.0**rng.uniform(5, 7, (30, 30))).astype(np.float32))     # DP sums far past 2**24
	return out


def test_calcaln_oracle_vs_transcription(oracle):
	for k, post in enumerate(dense_cases()):
		s, path = oracle.calcaln(post)
		s2, path2 = _calcaln_f32(post)
		assert np.float32(s) == s2 and path == path2, k


def test_calcaln_oracle_vs_ref(oracle, ref):
	for k, post in enumerate(dense_cases()):
		s, path = oracle.calcaln(post)
		s2, path2 = ref.calcaln(post)
		assert np.float32(s) == np.float32(s2) and path == path2, k


def _ref_with_store(ref, lens, store):
	m = ref.mpc(cs.seqs_of(lens))
	offs, ents = store
	for p in range(len(offs)):
		m.import_(p, offs[p], ents[p])
	return m


def test_consistency_oracle_vs_ref(oracle, ref, store):
	"""two ConsIter of the reference on the imported store == conspair of the oracle iterated twice"""
	offs, ents = store
	pairs = _pairs(len(LENS))
	m = _ref_with_store(ref, LENS, store)
	try:
		for it in range(2):
			want = oracle.conspair_many(LENS, pairs, offs, ents)
			m.consiter()
			offs2, got = m.export_all()
			for p in range(len(pairs)):
				assert np.array_equal(offs2[p], offs[p]), (it, p)
				assert got[p].tobytes() == want[p].tobytes(), ("consistency", it, p)
			ents = got
	finally:
		m.close()


@pytest.mark.parametrize("pattern", ["mixed", "heavy", "ties"])
def test_buildpost_oracle_vs_ref(oracle, ref, pattern):
	"""MPCFlat::BuildPost + CalcAlnFlat of the reference on gapped groups == oracle.buildpost + calcaln"""
	st = cs.make_store(LENS, pattern, 13)
	offs, ents = st
	seqs = cs.seqs_of(LENS)
	rng = np.random.default_rng(17)
	ga, gb = [0, 2, 4, 5, 9], [1, 3, 6, 7, 8, 10, 11]
	ca, cb = max(LENS[i] for i in ga) + 37, max(LENS[i] for i in gb) + 23
	pa = [cs.gapped_map(rng, LENS[i], ca) for i in ga]
	pb = [cs.gapped_map(rng, LENS[i], cb) for i in gb]
	rows_a = [cs.gapped_row(seqs[i], p, ca) for i, p in zip(ga, pa)]
	rows_b = [cs.gapped_row(seqs[i], p, cb) for i, p in zip(gb, pb)]
	# interior gaps, not only shifts
	assert all(np.diff(p.astype(np.int64)).max() > 1 for p in pa + pb if len(p) > 4)
	m = _ref_with_store(ref, LENS, st)
	try:
		for (g1, r1, p1, c1), (g2, r2, p2, c2) in [((ga, rows_a, pa, ca), (gb, rows_b, pb, cb)), ((gb, rows_b, pb, cb), (ga, rows_a, pa, ca))]:
			s_ref, path_ref, post_ref = m.alignalns(g1, r1, g2, r2)
			post = oracle.buildpost(LENS, g1, p1, c1, g2, p2, c2, offs, ents)
			assert post.tobytes() == post_ref.tobytes(), "BuildPost"
			s, path = oracle.calcaln(post)
			assert np.float32(s) == np.float32(s_ref) and path == path_ref, "CalcAlnFlat"
	finally:
		m.close()
