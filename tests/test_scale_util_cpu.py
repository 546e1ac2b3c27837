"""CPU: the stores of tests/scale_util.py hold every pair an oracle call reads.

The scale tests call the oracle on stores that hold only the pairs touching a few sequences
(star_store) or the pairs of two groups (cross_store), with placeholders in every other slot.  Here,
on hand-built stores (tests/crafted_store.py, mixed patterns), conspair and buildpost on such a store
must equal the same calls on the full store byte for byte.  The placeholders are valid pairs with
values no posterior has, so a read of one would change the result; the last tests show that it does."""
import numpy as np
import pytest
import crafted_store as cs
import scale_util as su

N = 70


class ListEngine:
	"""the part of Engine that the helpers use, over a store held in lists"""

	def __init__(self, lens, store):
		self.lens = np.asarray(lens, np.int64)
		self.offs, self.ents = store
		self.nnz_calls = 0
		self.exported = []

	def store_nnz(self):
		self.nnz_calls += 1
		nnz = np.array([len(e) for e in self.ents], np.uint32)
		return nnz, int(nnz.sum())

	def export_pair(self, k, nnz=None):
		assert nnz is not None and nnz == len(self.ents[k]), "export_pair without the pair's entry count"
		self.exported.append(k)
		return self.offs[k].copy(), self.ents[k].copy()


@pytest.fixture(scope="module")
def crafted():
	lens = np.random.default_rng(3).integers(1, 48, size=N)
	lens[[5, 40]] = [90, 130]                         # rows wider than four mask words
	store = cs.make_store(lens, "mixed", 21)
	return [int(L) for L in lens], store


@pytest.fixture(scope="module")
def full(crafted):
	lens, (offs, ents) = crafted
	return su.PairStore.full(lens, offs, ents)


def _pairs_of(ids):
	ids = sorted(ids)
	return [(x, y) for i, x in enumerate(ids) for y in ids[i + 1:]]


def test_pair_sets():
	n = 9
	allp = cs.pair_list(n)
	assert su.star_pairs(n, {2, 7}).tolist() == [k for k, (x, y) in enumerate(allp) if {x, y} & {2, 7}]
	assert su.cross_pairs(n, [5, 0], [3, 8]).tolist() == sorted(cs.pair_index(n, min(a, b), max(a, b)) for a in (5, 0) for b in (3, 8))
	assert all(su.pair_index(n, x, y) == k for k, (x, y) in enumerate(allp))


@pytest.mark.parametrize("full_rows", [False, True])
def test_star_store_holds_the_star_only(crafted, full_rows):
	lens, (offs, ents) = crafted
	S = {0, 5, 33, N - 1}
	eng = ListEngine(lens, (offs, ents))
	st = su.star_store(eng, lens, S, full_rows=full_rows)
	assert eng.nnz_calls == 1
	star = su.star_pairs(N, S)
	assert sorted(eng.exported) == star.tolist() and st.real.sum() == len(star)
	for k, (x, y) in enumerate(cs.pair_list(N)):
		if st.real[k]:
			assert st.offs[k].tobytes() == offs[k].tobytes() and st.ents[k].tobytes() == ents[k].tobytes()
			continue
		# a placeholder: valid, of the slot's shape, never empty, with values no posterior has
		cs.check_pair(st.offs[k], st.ents[k], lens[x], lens[y])
		assert len(st.ents[k]) >= lens[x] and (st.ents[k]["p"] >= 2).all()
		assert st.ents[k].tobytes() != ents[k].tobytes()


@pytest.mark.parametrize("full_rows", [False, True])
def test_conspair_on_star_store(oracle, crafted, full, full_rows):
	lens, (offs, ents) = crafted
	S = [0, 1, 5, 40, 41, N - 2, N - 1]
	st = su.star_store(ListEngine(lens, (offs, ents)), lens, S, full_rows=full_rows)
	pairs = _pairs_of(S)
	want = oracle.conspair_many(lens, pairs, offs, ents)          # plain binding, whole store
	got_full = full.conspair_many(oracle, pairs)
	got = st.conspair_many(oracle, pairs, threads=4)
	for xy, w, f, g in zip(pairs, want, got_full, got):
		assert f.tobytes() == w.tobytes() and g.tobytes() == w.tobytes(), xy


@pytest.mark.parametrize("full_rows", [False, True])
def test_buildpost_on_cross_store(oracle, crafted, full, full_rows):
	lens, (offs, ents) = crafted
	rng = np.random.default_rng(8)
	perm = rng.permutation(N)
	ids_a, ids_b = perm[:9].tolist(), perm[9:20].tolist()
	ca, cb = max(lens[i] for i in ids_a) + 17, max(lens[i] for i in ids_b) + 11
	pa = [cs.gapped_map(rng, lens[i], ca) for i in ids_a]
	pb = [cs.gapped_map(rng, lens[i], cb) for i in ids_b]
	eng = ListEngine(lens, (offs, ents))
	st = su.cross_store(eng, lens, ids_a, ids_b, store=su.PairStore(lens, full_rows))
	assert eng.nnz_calls == 1 and sorted(eng.exported) == su.cross_pairs(N, ids_a, ids_b).tolist()
	want = oracle.buildpost(lens, ids_a, pa, ca, ids_b, pb, cb, offs, ents)
	for store in (full, st):
		assert store.buildpost(oracle, ids_a, pa, ca, ids_b, pb, cb).tobytes() == want.tobytes()
		assert st.join(oracle, ids_a, pa, ca, ids_b, pb, cb) == oracle.calcaln(want)
	# B then A, and a refill with other groups drops the first ones
	assert st.buildpost(oracle, ids_b, pb, cb, ids_a, pa, ca).tobytes() == \
	  oracle.buildpost(lens, ids_b, pb, cb, ids_a, pa, ca, offs, ents).tobytes()
	ids_c = perm[20:23].tolist()
	pc = [np.arange(lens[i], dtype=np.uint32) for i in ids_c]
	cc = max(lens[i] for i in ids_c)
	su.cross_store(eng, lens, ids_a, ids_c, store=st)
	assert st.real.sum() == len(ids_a)*len(ids_c)
	assert st.buildpost(oracle, ids_a, pa, ca, ids_c, pc, cc).tobytes() == \
	  oracle.buildpost(lens, ids_a, pa, ca, ids_c, pc, cc, offs, ents).tobytes()
	with pytest.raises(AssertionError, match="lacks pairs"):
		st.buildpost(oracle, ids_a, pa, ca, ids_b, pb, cb)


def test_a_placeholder_read_changes_the_result(oracle, crafted):
	"""the same calls through the plain binding, which reads whatever the slots hold: one pair short
	of what each call reads, the result differs"""
	lens, (offs, ents) = crafted
	S = [0, 5, 40]
	eng = ListEngine(lens, (offs, ents))
	changed = 0
	for full_rows in (False, True):
		st = su.star_store(eng, lens, S, full_rows=full_rows)
		for x, y in _pairs_of(S):
			want = oracle.conspair(lens, x, y, offs, ents)
			for z in (1, 20, N - 1):
				k = su.pair_index(N, min(x, z), max(x, z))
				if len(ents[k]) == 0:
					continue
				st.clear(k)
				changed += oracle.conspair(lens, x, y, st.offs, st.ents).tobytes() != want.tobytes()
				st.set(k, offs[k], ents[k])
	assert changed >= 6
	rng = np.random.default_rng(9)
	ids_a, ids_b = [2, 3, 4], [6, 7]
	pa = [np.arange(lens[i], dtype=np.uint32) for i in ids_a]
	pb = [np.arange(lens[i], dtype=np.uint32) for i in ids_b]
	ca, cb = max(lens[i] for i in ids_a), max(lens[i] for i in ids_b)
	want = oracle.buildpost(lens, ids_a, pa, ca, ids_b, pb, cb, offs, ents)
	st = su.cross_store(eng, lens, ids_a, ids_b)
	for k in rng.permutation(su.cross_pairs(N, ids_a, ids_b)).tolist():
		st.clear(k)
		assert oracle.buildpost(lens, ids_a, pa, ca, ids_b, pb, cb, st.offs, st.ents).tobytes() != want.tobytes(), k
		st.set(k, offs[k], ents[k])
