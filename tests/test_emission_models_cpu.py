"""CPU: the emission tables of tests/emission_util.py.

* the library's host-side table compaction (mb200_residue_classes) finds exactly the K classes the
  plain tables are built with;
* the vocabulary mapping of Mega profiles reproduces the dense posteriors the COMPILED REFERENCE computed
  for every pair of BB11001.mega (tests/golden/mega_bb11001.npz) bit for bit;
* the oracle equals the compiled reference (PairHMM tables swapped in with ref_set_hmm) on pairs of every
  table set the GPU tests use, so that a GPU == oracle check there is a check against the reference."""
import ctypes as C
import os
import numpy as np
import pytest
import emission_util as eu
import mega_util
from conftest import GOLDEN, load_tables

PLAIN_SETS = ["K=%d" % K for K in eu.PLAIN_K] + ["K=21,pad"]


def _classes(t):
	from muscle_b200.engine import load_library
	lib = load_library()
	ins = np.ascontiguousarray(t["ins"], np.float32)
	match = np.ascontiguousarray(t["match"], np.float32).reshape(-1)
	b2c = np.zeros(256, np.uint8)
	n = C.c_int()
	rc = lib.mb200_residue_classes(C.c_void_p(ins.ctypes.data), C.c_void_p(match.ctypes.data),
	  C.c_void_p(b2c.ctypes.data), C.byref(n), None)
	assert rc == 0
	return n.value, b2c


@pytest.mark.parametrize("K", list(range(1, 66)))
def test_plain_tables_class_count(K):
	t, alphabet = eu.plain_tables(K, 1000 + K)
	n, b2c = _classes(t)
	assert n == K
	assert len(set(b2c[np.frombuffer(alphabet, np.uint8)].tolist())) == K
	assert all(b < 128 for b in alphabet) and 0 not in alphabet
	m = t["match"].reshape(256, 256)
	if K > 1:
		assert not np.array_equal(m, m.T)
	if K >= 2:
		tp, ap = eu.plain_tables(K, 1000 + K, pad_shares_letter=True)
		n, b2c = _classes(tp)
		assert n == K and ap == alphabet and b2c[0] == b2c[alphabet[0]]


def test_vocabulary_tables_reproduce_reference_goldens():
	"""each BB11001 pair's own letter vectors as the vocabulary, bytes 0..255"""
	from oracle.pyoracle import Oracle
	base = load_tables()
	model, profiles, posts = mega_util.load_model()
	for (i, j), want in posts.items():
		vecs = np.unique(np.concatenate([profiles[i], profiles[j]]), axis=0)
		assert len(vecs) <= 256
		index = {v.tobytes(): k for k, v in enumerate(vecs)}
		X = bytes(index[v.tobytes()] for v in profiles[i])
		Y = bytes(index[v.tobytes()] for v in profiles[j])
		got = Oracle(eu.vocabulary_tables(base, model, vecs, first=0)).post(X, Y)
		assert got.tobytes() == want.tobytes(), (i, j, float(np.abs(got - want).max()))


def _table_sets():
	for name in PLAIN_SETS:
		t, alphabet = eu.plain_set(name)
		yield name, t, eu.plain_family(alphabet, [1, 37, 90, 140], 11)
	for name in sorted(eu.MEGA_MODELS):
		_, vocab, t = eu.mega_set(name)
		yield name, t, eu.mega_family(vocab, [1, 37, 90, 140], 12)[1]
	z = np.load(os.path.join(GOLDEN, "hmm_nucleo.npz"))
	yield "nucleo", {k: z[k] for k in ("start", "trans", "ins", "match", "min_sparse_score")}, \
	  [b"A", b"acgUUNAGTCCA", b"GATTACAnnGATTaca"*5, b"GATuACAnGATTtACcaGATTAC"*6]


def test_oracle_equals_reference_on_synthetic_tables(ref):
	from oracle.pyoracle import Oracle, _p, f32p
	saved = ref.tables()

	def set_ref(t):
		arr = [np.ascontiguousarray(t[k], np.float32).reshape(-1) for k in ("start", "trans", "ins", "match")]
		ref.lib.ref_set_hmm(*[_p(a, f32p) for a in arr])

	try:
		for name, t, seqs in _table_sets():
			# the transitions are the reference's own; min_sparse_score is a constant of the reference
			assert np.float32(t["min_sparse_score"]) == np.float32(ref.lib.ref_min_sparse_score())
			set_ref(t)
			O = Oracle(t)
			for X, Y in ((seqs[0], seqs[2]), (seqs[2], seqs[0]), (seqs[1], seqs[3]), (seqs[3], seqs[1]), (seqs[2], seqs[3])):
				tag = "%s %d x %d" % (name, len(X), len(Y))
				f, b = ref.fwd(X, Y), ref.bwd(X, Y)
				assert O.fwd(X, Y).tobytes() == f.tobytes(), tag + ": Forward"
				assert O.bwd(X, Y).tobytes() == b.tobytes(), tag + ": Backward"
				assert np.float32(O.total(f, b)) == np.float32(ref.total(f, b)), tag + ": total"
				p = ref.post(X, Y)
				assert O.post(X, Y).tobytes() == p.tobytes(), tag + ": posterior"
				assert len(X) == 1 or len(Y) == 1 or (p >= 0.01).sum() > 0, tag + ": no posterior entries"
	finally:
		set_ref(saved)
	assert ref.tables()["match"].tobytes() == saved["match"].tobytes()
