"""GPU: k_posterior_sm under emission tables past the one protein table and the one Mega model.

Plain mode with K = 1..64 residue classes (asymmetric match tables, padding byte inside a letter class),
the nucleotide tables, and Mega models of 1..8 features (alphabets 1..110, a 0-weight feature, pair tables
of exactly 12 288 floats, asymmetric matrices) -- tests/emission_util.py builds them.  Every check
compares with the CPU oracle, which tests/test_emission_models_cpu.py pins to the compiled reference on
these tables, with tolerance 0.  The module runs its own context, so the session `engine` keeps the
protein tables."""
import os
import numpy as np
import pytest
import emission_util as eu
from conftest import GOLDEN, load_tables
from muscle_b200 import synth

pytestmark = pytest.mark.gpu

PLAIN_SETS = ["K=%d" % K for K in eu.PLAIN_K] + ["K=21,pad"]
MEGA_SETS = sorted(eu.MEGA_MODELS)
FORCED = [0, 1, 3, 8, 13, 16]
# (LX, LY) of the dense checks, each also run as (LY, LX); LY = 700 is two strips at C = 16
DENSE_SHAPES = [(1, 1), (37, 1), (1, 33), (70, 33), (129, 129), (300, 449), (120, 700), (700, 700)]
# all-pairs lengths: as Y they fill size classes 4, 8, 12, 14 and 16, and 513..1100 take several strips
ALLPAIRS_LENGTHS = [100, 1, 200, 300, 420, 513, 700, 1100, 60, 150]


@pytest.fixture(scope="module")
def eng():
	import torch
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")
	from muscle_b200.engine import Engine
	e = Engine(0)
	e.set_hmm(load_tables())
	yield e
	e.close()


def _oracle(t):
	from oracle.pyoracle import Oracle, build
	build(ref=False)
	return Oracle(t)


def nucleo_tables():
	z = np.load(os.path.join(GOLDEN, "hmm_nucleo.npz"))
	return {k: z[k] for k in ("start", "trans", "ins", "match", "min_sparse_score")}


def make_case(name, lengths, seed):
	"""-> (load(engine), oracle, sequences as the oracle reads them) of table set `name` and a homologous
	family of the given lengths"""
	if name == "protein":
		t = load_tables()
		seqs = eu.plain_family(synth.AMINO.encode(), lengths, seed)
	elif name == "nucleo":
		t = nucleo_tables()
		seqs = eu.plain_family(b"ACGTUNacgtun", lengths, seed)
	elif name.startswith("K="):
		t, alphabet = eu.plain_set(name)
		seqs = eu.plain_family(alphabet, lengths, seed)
	else:
		model, vocab, t = eu.mega_set(name)
		profiles, seqs = eu.mega_family(vocab, lengths, seed)

		def load(e):
			e.set_hmm(load_tables())          # the transitions
			e.set_seqs_mega(model, profiles)
		return load, _oracle(t), seqs

	def load(e):
		e.set_hmm(t)
		e.set_seqs(seqs)
	return load, _oracle(t), seqs


# ------------------------------------------------------------------------------------------------
# checks (the helpers of test_chains_gpu cache the oracle by sequence bytes alone; here the same bytes
# mean different things under each table set, so the caches are per case)
def check_dense(eng, O, seqs, px, py, which, force_c, cache, tag):
	"""Forward-M, Backward-M, total and dense posterior of store pair `which` of the list (px, py)"""
	x, y = px[which], py[which]
	key = (x, y)
	if key not in cache:
		X, Y = seqs[x], seqs[y]
		f, b = O.fwd(X, Y), O.bwd(X, Y)
		cache[key] = (np.ascontiguousarray(f[1:, 1:, 0]).tobytes(), np.ascontiguousarray(b[1:, 1:, 0]).tobytes(),
		  np.float32(O.total(f, b)), O.post(X, Y))
	fw, bw, tot_w, post_w = cache[key]
	post, fwd, bwd, tot = eng.calc_post_dense_pair(px, py, which, force_c=force_c)
	tag = "%s C=%d (%d, %d) %d x %d" % (tag, force_c, x, y, len(seqs[x]), len(seqs[y]))
	assert fwd.tobytes() == fw, tag + ": Forward M"
	assert bwd.tobytes() == bw, tag + ": Backward M"
	assert np.float32(tot) == tot_w, tag + ": total"
	assert post.tobytes() == post_w.tobytes(), tag + ": dense posterior"
	return post_w


def _want_pair(O, X, Y):
	p = O.post(X, Y)
	off, ent = O.sparse(p)
	return off, ent.tobytes(), np.float32(np.float32(O.alnscore(p))/np.float32(min(len(X), len(Y))))


def check_store(eng, O, seqs, px, py, ea, tag):
	"""row offsets, entry bytes and EA of every pair of the list against the oracle"""
	offs, ents = eng.export_all()
	for k, (x, y) in enumerate(zip(px, py)):
		off, ent, want_ea = _want_pair(O, seqs[x], seqs[y])
		assert np.array_equal(offs[k], off), "%s pair %d (%d, %d): row offsets" % (tag, k, x, y)
		assert ents[k].tobytes() == ent, "%s pair %d (%d, %d): entries" % (tag, k, x, y)
		assert np.float32(ea[k]) == want_ea, "%s pair %d (%d, %d): EA %r != %r" % (tag, k, x, y, ea[k], want_ea)
	assert sum(len(e) > 0 for e in ents) >= 0.75*len(px), tag + ": most pairs have no entries"
	return offs, ents


def check_allpairs(eng, O, seqs, tag):
	"""all pairs of seqs: store and EA against oracle.all_pairs -> (EA, plan)"""
	n = len(seqs)
	r = O.all_pairs(seqs, threads=0)
	ea = eng.posteriors_allpairs()
	iu = np.triu_indices(n, 1)
	assert ea.tobytes() == r["ea"][iu].astype(np.float32).tobytes(), tag + ": EA"
	offs, ents = eng.export_all()
	for k in range(len(offs)):
		assert np.array_equal(offs[k], r["row_off"][k]), "%s pair %d: row offsets" % (tag, k)
		assert ents[k].tobytes() == r["entries"][k].tobytes(), "%s pair %d: entries" % (tag, k)
	assert sum(len(e) > 0 for e in ents) >= 0.75*len(ents), tag + ": most pairs have no entries"
	return ea, eng.debug_plan()


def _bins(plan):
	bs = plan["bin_start"]
	return [C for C in range(1, 17) if bs[C + 1] > bs[C]]


# ------------------------------------------------------------------------------------------------
# dense Forward / Backward / posterior at every forced width, both orientations
def _dense_case(eng, name):
	lengths = [L for xy in DENSE_SHAPES for L in xy]
	load, O, seqs = make_case(name, lengths, 31)
	load(eng)
	cache = {}
	top = 0.0
	for force_c in FORCED:
		for k in range(len(DENSE_SHAPES)):
			for x, y in ((2*k, 2*k + 1), (2*k + 1, 2*k)):
				p = check_dense(eng, O, seqs, [x], [y], 0, force_c, cache, name)
				top = max(top, float(p.max()))
	assert top > 0.5, "%s: no informative posterior (max %g)" % (name, top)


@pytest.mark.parametrize("name", PLAIN_SETS)
def test_plain_dense(eng, name):
	_dense_case(eng, name)


@pytest.mark.parametrize("name", MEGA_SETS)
def test_mega_dense(eng, name):
	_dense_case(eng, name)


# ------------------------------------------------------------------------------------------------
# sparse store and EA through all pairs, every size class
@pytest.mark.parametrize("name", PLAIN_SETS + MEGA_SETS + ["nucleo"])
def test_allpairs_store_and_ea(eng, name):
	load, O, seqs = make_case(name, ALLPAIRS_LENGTHS, 41)
	load(eng)
	_, plan = check_allpairs(eng, O, seqs, name)
	bins = _bins(plan)
	assert {4, 8, 12, 14, 16} <= set(bins), "%s: size classes %r" % (name, bins)
	if name == "nf3_12288":
		print("\n%s bin_start %s" % (name, plan["bin_start"].tolist()))


# ------------------------------------------------------------------------------------------------
# chains of pairs that share Y
@pytest.mark.parametrize("name", ["K=64", "nf3_12288"])
def test_chains(eng, name):
	rng = np.random.default_rng(5)
	xl = [int(v) for v in rng.integers(15, 140, 30)]
	load, O, seqs = make_case(name, [300] + xl, 51)
	load(eng)
	px, py = list(range(1, len(seqs))), [0]*(len(seqs) - 1)
	ea = eng.posteriors(px, py)
	plan = eng.debug_plan()
	order, chain = plan["order"].tolist(), plan["chain"].tolist()
	chains = [order[chain[c]:chain[c + 1]] for c in range(len(chain) - 1)]
	assert len(chains) >= 2 and max(map(len, chains)) >= 4, "%s: chains %r" % (name, chains)
	check_store(eng, O, seqs, px, py, ea, name)
	cache = {}
	for c in chains:
		if len(c) >= 3:
			check_dense(eng, O, seqs, px, py, c[len(c)//2], 0, cache, name + " chain middle")


# ------------------------------------------------------------------------------------------------
# one context through several models
def test_switching_models(eng):
	lengths = [50, 140, 300, 450, 600]
	for step, name in enumerate(["protein", "K=64", "nf3_12288", "nf1_a110", "protein"]):
		load, O, seqs = make_case(name, lengths, 61 + step)
		load(eng)
		check_allpairs(eng, O, seqs, "step %d %s" % (step, name))


# ------------------------------------------------------------------------------------------------
# limits and rejection
def test_rejected_plain_table_keeps_previous(eng):
	from muscle_b200.engine import MB200Error
	load, O, seqs = make_case("K=5", [80, 150, 260, 33], 71)
	load(eng)
	want, _ = check_allpairs(eng, O, seqs, "K=5")
	t65, _ = eu.plain_tables(65, 65)
	t65["start"] = t65["start"] - np.float32(0.25)          # rejected values that would change every result
	t65["trans"] = t65["trans"]*np.float32(0.5)
	t65["min_sparse_score"] = np.float32(-3.0)
	with pytest.raises(MB200Error) as ei:
		eng.set_hmm(t65)
	assert ei.value.code == -6
	eng.set_seqs(seqs)                                       # recodes with the byte map in force
	ea, _ = check_allpairs(eng, O, seqs, "K=5 after a rejected 65-class table")
	assert ea.tobytes() == want.tobytes()


def _set_seqs_mega_raw(eng, nfeat, alpha, tsize_floats, letters, offsets):
	"""mb200_set_seqs_mega with any feature count (Engine.set_seqs_mega needs nfeat >= 1) -> return code"""
	import ctypes as C
	alpha = np.ascontiguousarray(alpha, np.uint32)
	w = np.ones(max(nfeat, 1), np.float32)
	lp = np.zeros(max(int(alpha.sum()), 1), np.float32)
	lpm = np.zeros(max(tsize_floats, 1), np.float32)
	let = np.ascontiguousarray(letters, np.uint8)
	off = np.ascontiguousarray(offsets, np.uint64)
	p = lambda a: C.c_void_p(a.ctypes.data)
	return eng.lib.mb200_set_seqs_mega(eng.h, C.c_uint32(len(off) - 1), p(let), p(off), C.c_uint32(nfeat), p(alpha),
	  p(w), p(lp), p(lpm))


def test_mega_limits_rejected(eng):
	load, O, seqs = make_case("nf3_12288", [90, 200, 450], 81)
	load(eng)
	ea0, _ = check_allpairs(eng, O, seqs, "12 288 floats")
	# 12 289 floats, no features, nine features
	for nfeat, alpha in ((4, [64, 64, 64, 1]), (0, [1]), (9, [2]*9)):
		tsize = int(sum(a*a for a in alpha[:nfeat]))
		letters = np.zeros((5, max(nfeat, 1)), np.uint8)
		rc = _set_seqs_mega_raw(eng, nfeat, alpha, tsize, letters, [0, 2, 5])
		assert rc == -6, (nfeat, alpha, rc)
		# the previous profiles and model are still in force
		ea = eng.posteriors_allpairs()
		assert ea.tobytes() == ea0.tobytes(), (nfeat, alpha)
	check_allpairs(eng, O, seqs, "12 288 floats after rejections")
