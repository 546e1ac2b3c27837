"""CPU: the repeat-rich inputs of tests/repeat_util.py.

1. They stay informative: each input of the dense-row GPU tests (tests/test_dense_rows_gpu.py) still reaches
   the path it was chosen for.  A generator change that loses one fails here and names it.
2. The CPU oracle stays pinned to the compiled reference on these rows, with tolerance 0: posteriors,
   sparse store and EA of every pair, two consistency iterations, and one BuildPost + CalcAlnFlat.
   tests/test_oracle_vs_ref.py pins it on ordinary families only, where rows hold ~7 entries."""
import numpy as np
import pytest
import repeat_util as ru

W1 = 32          # columns per strip at force_c = 1


def _pairs(n):
	return [(i, j) for i in range(n) for j in range(i + 1, n)]


@pytest.fixture(scope="module")
def dense_sparse(oracle):
	return [oracle.sparse(oracle.post(X, Y)) for X, Y in ru.DENSE_PAIRS]


@pytest.fixture(scope="module")
def family(oracle):
	seqs = ru.repeat_family(12, ru.REPEAT_SEED)
	return seqs, oracle.all_pairs(seqs, threads=0)


def _counts(off):
	return np.diff(np.asarray(off, np.int64))


# ------------------------------------------------------------------------------------------------
# 1. informativeness
def test_dense_pairs_reach_long_rows(dense_sparse):
	cnt = [_counts(off) for off, _ in dense_sparse]
	assert max(c.max() for c in cnt) > 64, "no DENSE_PAIRS row holds more than 64 entries (rowcnt, __shfl_down counts)"
	assert sum((c > 32).sum() for c in cnt) > 0, "no DENSE_PAIRS row holds more than 32 entries (compaction groups)"
	assert max(len(e) for _, e in dense_sparse) > 2048, "no DENSE_PAIRS pair holds more than 2048 entries"


def test_dense_pairs_cross_strips(dense_sparse):
	"""at force_c = 1 a strip is 32 columns: some row has entries on both sides of a strip edge, so its count
	travels across strips in the edge record"""
	for off, ent in dense_sparse:
		for i in range(len(off) - 1):
			strips = set((ent["col"][off[i]:off[i + 1]] // W1).tolist())
			if len(strips) >= 3:
				return
	assert False, "no DENSE_PAIRS row spans three strips of 32 columns"


def test_dense_pairs_near_threshold(oracle):
	"""the homopolymer pairs put many posteriors next to the 0.01 cut, where the kept count (a compare of
	the score) and the compaction (a compare of expf(score)) must agree"""
	near = 0
	for X, Y in ru.DENSE_PAIRS:
		p = oracle.post(X, Y)
		near += int(((p > 0.0095) & (p < 0.0105)).sum())
	assert near >= 100, "only %d posteriors within 5 %% of 0.01" % near


def test_repeat_family_is_dense(family):
	seqs, r = family
	cnt = np.concatenate([_counts(o) for o in r["row_off"]])
	assert (cnt > 32).sum() > 0, "no repeat_family row holds more than 32 entries"
	assert (r["nnz"] > 1024).sum() > 0, "no repeat_family pair holds more than 1024 entries (one k_relax sweep)"
	assert (r["nnz"] > 2048).sum() > 0, "no repeat_family pair holds more than 2048 entries (two k_relax sweeps)"


def test_buildpost_operands_past_staging(family):
	"""BuildPost stages 16 entries per operand row; longer rows take the direct gather"""
	seqs, r = family
	c = ru.operand_row_counts([len(s) for s in seqs], ru.GROUP_A, ru.GROUP_B, r["row_off"], r["entries"])
	assert (c == 16).any(), "no BuildPost operand row of exactly 16 entries"
	assert (c >= 17).any(), "no BuildPost operand row of 17 or more entries"
	c2 = ru.operand_row_counts([len(s) for s in seqs], ru.GROUP_B, ru.GROUP_A, r["row_off"], r["entries"])
	assert (c2 >= 17).any(), "no BuildPost operand row of 17 or more entries in the transposed join"


def test_mixed_family_reaches_z_chunks(oracle):
	"""mixed_family at N = 65 and 130: the sequences at 63, 64 and N-1 are repeats, so pairs across the
	64-sequence z chunks of k_relax are dense"""
	for n in (65, 130):
		seqs = ru.mixed_family(n, 7)
		assert len(seqs) == n
		slots = ru.repeat_slots(n)
		assert 63 in slots and 64 in slots and n - 1 in slots
		most = {}
		for a in slots:
			for b in slots:
				if a < b:
					off, ent = oracle.sparse(oracle.post(seqs[a], seqs[b]))
					most[(a, b)] = (_counts(off).max(), len(ent))
		assert sum(m > 16 for m, _ in most.values()) >= 2, (n, most)
		assert any(m > 16 and nnz > 1024 and (63 in ab or 64 in ab) for ab, (m, nnz) in most.items()), (n, most)


# ------------------------------------------------------------------------------------------------
# 2. oracle against the compiled reference
def test_conspair_many_equals_conspair(oracle):
	seqs = ru.repeat_family(5, 3, lmin=20, lmax=60)
	r = oracle.all_pairs(seqs, threads=0)
	lens = [len(s) for s in seqs]
	pairs = _pairs(len(seqs))
	many = oracle.conspair_many(lens, pairs[::-1], r["row_off"], r["entries"])
	for (x, y), got in zip(pairs[::-1], many):
		assert got.tobytes() == oracle.conspair(lens, x, y, r["row_off"], r["entries"]).tobytes(), (x, y)
	assert sum(len(g) for g in many) > 0


def test_pairs_oracle_vs_ref(oracle, ref, family):
	seqs, _ = family
	for x, y in _pairs(len(seqs)):
		X, Y = seqs[x], seqs[y]
		po, pr = oracle.post(X, Y), ref.post(X, Y)
		assert po.tobytes() == pr.tobytes(), ("posterior", x, y)
		(oo, eo), (orf, er) = oracle.sparse(po), ref.sparse(pr)
		assert np.array_equal(oo, orf) and eo.tobytes() == er.tobytes(), ("sparse", x, y)
		assert np.float32(oracle.alnscore(po)) == np.float32(ref.alnscore(pr)), ("EA", x, y)


def test_consistency_and_buildpost_oracle_vs_ref(oracle, ref, family):
	seqs, r = family
	lens = [len(s) for s in seqs]
	pairs = _pairs(len(seqs))
	m = ref.mpc(seqs)
	try:
		m.posteriors()
		offs, ents = m.export_all()
		for p in range(len(pairs)):
			assert np.array_equal(offs[p], r["row_off"][p]) and ents[p].tobytes() == r["entries"][p].tobytes(), p
		for it in range(2):
			want = oracle.conspair_many(lens, pairs, offs, ents)
			m.consiter()
			offs2, got = m.export_all()
			for p in range(len(pairs)):
				assert np.array_equal(offs2[p], offs[p]), (it, p)
				assert got[p].tobytes() == want[p].tobytes(), ("consistency", it, p)
			ents = got
		rows1, p2c1 = ru.staggered_rows(seqs, ru.GROUP_A)
		rows2, p2c2 = ru.staggered_rows(seqs, ru.GROUP_B)
		s_ref, path_ref, post_ref = m.alignalns(ru.GROUP_A, rows1, ru.GROUP_B, rows2)
		post = oracle.buildpost(lens, ru.GROUP_A, p2c1, len(rows1[0]), ru.GROUP_B, p2c2, len(rows2[0]), offs, ents)
		assert post.tobytes() == post_ref.tobytes(), "BuildPost"
		s, path = oracle.calcaln(post)
		assert np.float32(s) == np.float32(s_ref) and path == path_ref, "CalcAlnFlat"
	finally:
		m.close()
