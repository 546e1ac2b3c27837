"""GPU: k_posterior_sm's chains (pairs that share Y, run back to back by one warp) at their limits.

Every case checks, for every pair, the sparse store (row offsets and entry bytes) and the EA against
the CPU oracle (or the Mega goldens) with tolerance 0, and checks that the library's plan is the one
the chain rule of build_plan (muscle_b200/csrc/engine.cu) gives, chain for chain, so that the cases
keep reaching the boundaries they were built for.  The boundaries are taken from the limits the
library reports, not hard-coded.  X sequences are windows of a homolog of Y, so that even short
pairs keep posterior entries >= 0.01 and a wrong kernel cannot pass on empty results.
"""
import numpy as np
import pytest
import mega_util
from muscle_b200 import synth

pytestmark = pytest.mark.gpu

Y_SWEEP = [1, 2, 31, 32, 33, 128, 129, 384, 385, 448, 449, 512, 513, 1100]
SWEEP_X = [1, 7, 33, 64, 150, 260]
FORCED = [1, 2, 3, 5, 8, 13, 16]


# ------------------------------------------------------------------------------------------------
# the chain rule, restated
def _size_class(c):
	return (c + 3)//4*4 if c <= 12 else (14 if c <= 14 else 16)


def mirror_plan(lens, px, py, force_c, max_rows, max_pairs):
	"""-> (order, chain, bin_start) as build_plan builds them: pairs are binned by columns per lane;
	inside a bin, pairs with the same Y join the open chain of that Y in store order unless it would
	pass max_rows Forward rows (sum of LX+2) or max_pairs pairs, or the pair needs more than one strip;
	chains are ordered by cells, most first, ties in creation order"""
	bins = {C: [] for C in range(1, 17)}
	for k, y in enumerate(py):
		C = force_c if force_c > 0 else _size_class(min(16, (lens[y] + 31)//32))
		bins[C].append(k)
	order, chain, bin_start = [], [], [0]*18
	for C in range(1, 17):
		chains, frows, cost, open_ = [], [], [], {}
		for k in bins[C]:
			LX, LY = lens[px[k]], lens[py[k]]
			c = open_.get(py[k], -1)
			if c < 0 or LY > 32*C or frows[c] + LX + 2 > max_rows or len(chains[c]) == max_pairs:
				c = open_[py[k]] = len(chains)
				chains.append([])
				frows.append(0)
				cost.append(0)
			chains[c].append(k)
			frows[c] += LX + 2
			cost[c] += LX*LY
		bin_start[C] = len(chain)
		for c in sorted(range(len(chains)), key=lambda c: -cost[c]):
			chain.append(len(order))
			order.extend(chains[c])
	bin_start[17] = len(chain)
	chain.append(len(order))
	return order, chain, bin_start


def check_plan(engine, lens, px, py, force_c=0):
	"""the library's plan equals the mirror; -> list of chains (lists of store pairs, in run order)"""
	p = engine.debug_plan()
	order, chain, bin_start = mirror_plan(lens, list(px), list(py), force_c, p["chain_rows"], p["chain_pairs"])
	assert p["order"].tolist() == order, "pair order differs from the chain rule"
	assert p["chain"].tolist() == chain, "chain boundaries differ from the chain rule"
	assert p["bin_start"].tolist() == bin_start, "size-class bins differ from the chain rule"
	return [order[chain[c]:chain[c + 1]] for c in range(len(chain) - 1)]


@pytest.fixture(scope="module")
def limits(engine):
	"""(most Forward rows, most pairs) of one chain, as the library reports them"""
	engine.set_seqs(["ACDEF", "GHIKL"])
	engine.posteriors([0], [1])
	p = engine.debug_plan()
	assert p["chain_rows"] >= 80 and p["chain_pairs"] >= 2
	return p["chain_rows"], p["chain_pairs"]


# ------------------------------------------------------------------------------------------------
# inputs
def _homologs(seed, LY, lmax):
	"""Y of LY residues and a homolog of it of at least lmax residues to cut X windows from"""
	L = max(LY, lmax)
	a, b = synth.make_family(2, L, 0, seed=seed, min_len=1)
	return a[:LY], b


def _windows(H, LY, lengths, rng):
	out = []
	for L in lengths:
		hi = max(0, min(len(H), max(LY + 8, L)) - L)
		a = int(rng.integers(0, hi + 1))
		out.append(H[a:a + L])
	return out


def pair_cap_case(max_rows, max_pairs, reverse=False):
	"""one Y of 300 residues, max_pairs + 8 short X: the first max_pairs pairs fill one chain"""
	lmax = max_rows//max_pairs - 2
	assert lmax >= 2
	n = max_pairs + 8
	lengths = [1 + (k*37) % lmax for k in range(n)]
	Y, H = _homologs(101, 300, 300)
	X = _windows(H, 300, lengths, np.random.default_rng(1))
	seqs = [Y] + X
	px = list(range(1, n + 1))
	if reverse:
		px = px[::-1]
	return seqs, px, [0]*n


def row_cap_case(max_rows, extra):
	"""X lengths whose chain has exactly max_rows Forward rows (+ extra residues in its last pair), then
	X of max_rows-2 (one pair at the limit) and max_rows-1 among short X on the same Y"""
	n = 20
	lengths = [(max_rows - 2*n)//n + (k % 5) - 2 for k in range(n)]
	lengths[-1] += max_rows - sum(L + 2 for L in lengths) + extra
	lengths += [17, max_rows - 2, 9, max_rows - 1, 1, 23]
	Y, H = _homologs(202, 300, max_rows)
	X = _windows(H, 300, lengths, np.random.default_rng(2))
	return [Y] + X, list(range(1, len(X) + 1)), [0]*len(X)


def y_sweep_case():
	"""every Y length of Y_SWEEP with a chain of SWEEP_X windows"""
	seqs, px, py = [], [], []
	for s, LY in enumerate(Y_SWEEP):
		Y, H = _homologs(300 + s, LY, max(SWEEP_X))
		yi = len(seqs)
		seqs.append(Y)
		for X in _windows(H, LY, SWEEP_X, np.random.default_rng(s)):
			px.append(len(seqs))
			py.append(yi)
			seqs.append(X)
	return seqs, px, py


# ------------------------------------------------------------------------------------------------
# checks
_cache = {}


def _want(oracle, X, Y):
	"""oracle (row offsets, entry bytes, EA as float32) of pair (X, Y)"""
	key = (X, Y)
	if key not in _cache:
		p = oracle.post(X, Y)
		off, ent = oracle.sparse(p)
		ea = np.float32(np.float32(oracle.alnscore(p))/np.float32(min(len(X), len(Y))))
		_cache[key] = (off, ent.tobytes(), ea)
	return _cache[key]


def export_store(engine):
	"""export_all, once every pair's entry count is possible: a row holds at most 100 entries >= 0.01
	(they sum to at most 1), so a larger count is wrong and the store is not worth copying"""
	nnz, _ = engine.store_nnz()
	rows = engine.lens[engine._pairs[0]]
	bad = np.flatnonzero(nnz > 100*rows)
	assert len(bad) == 0, "pair %d: %d entries in %d rows" % (bad[0], nnz[bad[0]], rows[bad[0]])
	return engine.export_all()


def check_store(engine, oracle, seqs, px, py, ea, tag="", varied=True):
	"""store and EA of every pair against the oracle; the data must be informative"""
	offs, ents = export_store(engine)
	nz = 0
	for k, (x, y) in enumerate(zip(px, py)):
		off, ent, want_ea = _want(oracle, seqs[x], seqs[y])
		assert np.array_equal(offs[k], off), "%s pair %d (%d, %d): row offsets" % (tag, k, x, y)
		assert ents[k].tobytes() == ent, "%s pair %d (%d, %d): entries" % (tag, k, x, y)
		assert np.float32(ea[k]) == want_ea, "%s pair %d (%d, %d): EA %r != %r" % (tag, k, x, y, ea[k], want_ea)
		nz += len(ents[k]) > 0
	assert nz >= 0.75*len(px), "%s: only %d of %d pairs have entries" % (tag, nz, len(px))
	assert not varied or len(set(np.asarray(ea).tolist())) > len(px)//4, "%s: EA values barely differ" % tag
	return offs, ents


def run_list(engine, oracle, seqs, px, py, force_c=0, tag="", varied=True):
	engine.set_seqs(seqs)
	ea = engine.posteriors(px, py, force_c=force_c)
	chains = check_plan(engine, [len(s) for s in seqs], px, py, force_c)
	offs, ents = check_store(engine, oracle, seqs, px, py, ea, tag, varied)
	return chains, ea, offs, ents


def check_dense(engine, oracle, seqs, px, py, which, force_c=0, tag=""):
	"""Forward-M, Backward-M, total and dense posterior of store pair `which`, run inside its chain"""
	X, Y = seqs[px[which]], seqs[py[which]]
	post, fwd, bwd, tot = engine.calc_post_dense_pair(px, py, which, force_c=force_c)
	f, b = oracle.fwd(X, Y), oracle.bwd(X, Y)
	tag = "%s pair %d" % (tag, which)
	assert fwd.tobytes() == np.ascontiguousarray(f[1:, 1:, 0]).tobytes(), tag + ": Forward M"
	assert bwd.tobytes() == np.ascontiguousarray(b[1:, 1:, 0]).tobytes(), tag + ": Backward M"
	assert np.float32(tot) == np.float32(oracle.total(f, b)), tag + ": total"
	assert post.tobytes() == oracle.post(X, Y).tobytes(), tag + ": dense posterior"


def _positions(ch, max_pairs):
	"""store pairs at chain positions 0, 1, middle, last and max_pairs-1 of chain ch"""
	pos = {0, 1, len(ch)//2, len(ch) - 1, max_pairs - 1}
	return [ch[q] for q in sorted(pos) if q < len(ch)]


# ------------------------------------------------------------------------------------------------
# 1. pair cap
@pytest.mark.parametrize("reverse", [False, True])
def test_pair_cap(engine, oracle, limits, reverse):
	R, M = limits
	seqs, px, py = pair_cap_case(R, M, reverse)
	chains, _, _, _ = run_list(engine, oracle, seqs, px, py, tag="pair cap")
	assert sorted(map(sorted, chains)) == [list(range(M)), list(range(M, M + 8))]


# 2. row cap
@pytest.mark.parametrize("extra", [0, 1])
def test_row_cap(engine, oracle, limits, extra):
	R, M = limits
	seqs, px, py = row_cap_case(R, extra)
	chains, _, _, _ = run_list(engine, oracle, seqs, px, py, tag="row cap +%d" % extra)
	lens = [len(s) for s in seqs]
	rows = {tuple(c): sum(lens[px[k]] + 2 for k in c) for c in chains}
	if extra == 0:
		assert list(range(20)) in chains and rows[tuple(range(20))] == R
	else:
		assert list(range(19)) in chains and list(range(20)) not in chains
	# the pairs of R-2 and R-1 residues run alone: one at the limit, one past it
	assert [21] in chains and rows[(21,)] == R and [23] in chains and rows[(23,)] == R + 1


# 3. Y length sweep, 4. forced widths
@pytest.mark.parametrize("force_c", [0] + FORCED)
def test_y_sweep(engine, oracle, force_c):
	seqs, px, py = y_sweep_case()
	chains, _, _, _ = run_list(engine, oracle, seqs, px, py, force_c, tag="Y sweep C=%d" % force_c)
	lens = [len(s) for s in seqs]
	W = 32*(force_c or 16)
	multi = [c for c in chains if lens[py[c[0]]] > W]
	assert all(len(c) == 1 for c in multi)
	assert any(len(c) == len(SWEEP_X) for c in chains)
	if force_c == 0:
		assert len(multi) == 2*len(SWEEP_X)          # LY = 513 and 1100


# 5. list shapes
def test_list_shapes(engine, oracle):
	seqs = synth.make_family(8, 90, 40, seed=55, min_len=20)
	# the same Y non-contiguous and interleaved with other Y, sequences as both X and Y, x == y pairs
	px = [1, 2, 0, 3, 4, 5, 2, 6, 7, 0, 1, 3, 6, 4, 2, 5, 7, 3, 0, 1]
	py = [0, 0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 1, 2, 2, 2, 1, 0, 3, 0, 0]
	chains, ea, offs, ents = run_list(engine, oracle, seqs, px, py, tag="interleaved")
	assert any(len(c) >= 5 and len({px[k] for k in c}) < len(c) for c in chains)
	# the same list shuffled: every pair keeps its result
	perm = np.random.default_rng(3).permutation(len(px))
	ea2 = engine.posteriors(np.array(px)[perm], np.array(py)[perm])
	check_plan(engine, [len(s) for s in seqs], np.array(px)[perm], np.array(py)[perm])
	offs2, ents2 = export_store(engine)
	for q, k in enumerate(perm):
		assert np.array_equal(offs2[q], offs[k]) and ents2[q].tobytes() == ents[k].tobytes(), (q, k)
		assert np.float32(ea2[q]) == np.float32(ea[k]), (q, k)


def test_copies_of_one_pair(engine, oracle, limits):
	R, M = limits
	Y, H = _homologs(77, 120, 120)
	seqs = [Y, H[10:40]]
	n = M + 1
	chains, ea, offs, ents = run_list(engine, oracle, seqs, [1]*n, [0]*n, tag="copies", varied=False)
	assert sorted(map(len, chains)) == [1, M]
	assert all(e.tobytes() == ents[0].tobytes() for e in ents) and len(set(ea.tolist())) == 1


# 6. isolation and permutation
def test_isolation(engine, oracle, limits):
	R, M = limits
	for seqs, px, py in (pair_cap_case(R, M), row_cap_case(R, 0), y_sweep_case()):
		engine.set_seqs(seqs)
		ea = engine.posteriors(px, py)
		offs, ents = export_store(engine)
		sample = sorted(set(np.random.default_rng(len(px)).choice(len(px), 8, replace=False).tolist()) | {len(px) - 1})
		for k in sample:
			e1 = engine.posteriors([px[k]], [py[k]])
			o1, n1 = export_store(engine)
			assert np.array_equal(o1[0], offs[k]) and n1[0].tobytes() == ents[k].tobytes(), k
			assert np.float32(e1[0]) == np.float32(ea[k]), k
		perm = np.random.default_rng(7).permutation(len(px))
		ea2 = engine.posteriors(np.array(px)[perm], np.array(py)[perm])
		offs2, ents2 = export_store(engine)
		for q, k in enumerate(perm):
			assert np.array_equal(offs2[q], offs[k]) and ents2[q].tobytes() == ents[k].tobytes(), (q, k)
			assert np.float32(ea2[q]) == np.float32(ea[k]), (q, k)


# 7. all-pairs sub-ranges
def allpairs_seqs():
	s = synth.make_family(52, 29, 6, seed=66, min_len=20)
	s = [x[:38] for x in s[:48]]
	return s + synth.make_family(4, 300, 60, seed=67)


def _check_allpairs_plan(engine, seqs, p_lo, p_hi):
	n = len(seqs)
	px, py = np.triu_indices(n, 1)
	return check_plan(engine, [len(s) for s in seqs], px[p_lo:p_hi].tolist(), py[p_lo:p_hi].tolist())


def test_allpairs_subranges(engine, oracle, limits):
	R, M = limits
	seqs = allpairs_seqs()
	n = len(seqs)
	npairs = n*(n - 1)//2
	r = oracle.all_pairs(seqs, threads=0)
	engine.set_seqs(seqs)
	ea = engine.posteriors_allpairs()
	chains = _check_allpairs_plan(engine, seqs, 0, npairs)
	assert max(map(len, chains)) == M
	iu = np.triu_indices(n, 1)
	assert ea.tobytes() == r["ea"][iu].astype(np.float32).tobytes()
	offs, ents = export_store(engine)
	for k in range(npairs):
		assert np.array_equal(offs[k], r["row_off"][k]) and ents[k].tobytes() == r["entries"][k].tobytes(), k
	assert sum(len(e) > 0 for e in ents) >= 0.75*npairs and len(set(ea.tolist())) > npairs//4
	# ranges that start and end inside chains of the full run
	for p_lo, p_hi in ((37, 1000), (200, 701), (513, npairs - 7), (5, 1290)):
		inside = [sum(p_lo <= k < p_hi for k in c) for c in chains]
		assert sum(0 < m < len(c) for m, c in zip(inside, chains)) >= 2
		ea_r = engine.posteriors_allpairs(p_lo, p_hi)
		_check_allpairs_plan(engine, seqs, p_lo, p_hi)
		offs_r, ents_r = export_store(engine)
		for q in range(p_hi - p_lo):
			k = p_lo + q
			assert np.array_equal(offs_r[q], offs[k]) and ents_r[q].tobytes() == ents[k].tobytes(), (p_lo, p_hi, k)
		assert ea_r.tobytes() == ea[p_lo:p_hi].tobytes(), (p_lo, p_hi)


# 8. entry-pool retry
def test_entry_pool_retry(engine, oracle, limits):
	R, M = limits
	for seqs, px, py in (pair_cap_case(R, M), (allpairs_seqs(), None, None)):
		engine.set_seqs(seqs)
		ea = engine.posteriors(px, py) if px is not None else engine.posteriors_allpairs()
		offs, ents = export_store(engine)
		nbins = int((np.diff(engine.debug_plan()["bin_start"][1:]) > 0).sum())
		engine.set_seqs(seqs)                  # forget the entry count of the last run
		engine.set_nnz_per_row_cap(1)
		try:
			k0 = engine.stats()["kernel_launches"]
			ea2 = engine.posteriors(px, py) if px is not None else engine.posteriors_allpairs()
			launches = engine.stats()["kernel_launches"] - k0
		finally:
			engine.set_nnz_per_row_cap(12)
		assert launches == 2*nbins, "the entry pool did not overflow (%d launches, %d bins)" % (launches, nbins)
		offs2, ents2 = export_store(engine)
		assert ea2.tobytes() == ea.tobytes()
		for k in range(len(offs)):
			assert np.array_equal(offs2[k], offs[k]) and ents2[k].tobytes() == ents[k].tobytes(), k


# 9. dense inside a chain
def test_dense_in_chain(engine, oracle, limits):
	R, M = limits
	for seqs, px, py, force_c, tag in ((*pair_cap_case(R, M), 0, "pair cap"), (*row_cap_case(R, 0), 0, "row cap"),
	  (*y_sweep_case(), 0, "Y sweep"), (*y_sweep_case(), 3, "Y sweep C=3")):
		engine.set_seqs(seqs)
		engine.posteriors(px, py, force_c=force_c)
		chains = check_plan(engine, [len(s) for s in seqs], px, py, force_c)
		long_ = [c for c in chains if len(c) > 1]
		assert long_
		picks = []
		for c in long_[:2] if tag != "Y sweep" else long_[::3]:
			picks += _positions(c, M)
		for k in picks:
			check_dense(engine, oracle, seqs, px, py, k, force_c, tag)


# 10. Mega chains
@pytest.mark.parametrize("force_c", [0, 3, 4])
def test_mega_chains(engine, oracle, limits, force_c):
	R, M = limits
	model, profiles, posts = mega_util.load_model()
	rng = np.random.default_rng(10)
	lens = [len(p) for p in profiles]
	px, rows = [], 0
	while rows + lens[2] + 2 <= R + 2*(lens[2] + 2):          # two more pairs past one full chain
		x = int(rng.integers(0, 3))
		px.append(x)
		rows += lens[x] + 2
	py = [3]*len(px)
	engine.set_seqs_mega(model, profiles)
	ea = engine.posteriors(px, py, force_c=force_c)
	chains = check_plan(engine, lens, px, py, force_c)
	assert max(map(len, chains)) >= 12
	offs, ents = export_store(engine)
	for k, x in enumerate(px):
		want = posts[(x, 3)]
		o, e = oracle.sparse(want)
		assert np.array_equal(offs[k], o) and ents[k].tobytes() == e.tobytes(), (k, x)
		assert np.float32(ea[k]) == np.float32(np.float32(oracle.alnscore(want))/np.float32(min(want.shape))), (k, x)
	for k in [q for c in chains for q in c[1:]][::3]:
		post, _, _, _ = engine.calc_post_dense_pair(px, py, k, force_c=force_c)
		assert post.tobytes() == posts[(px[k], 3)].tobytes(), (k, px[k])
