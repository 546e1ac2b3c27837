"""GPU: the shapes of a join's decoding DP (k_aln_wave) that decide its launch and scratch layout, and a
join large enough that BuildPost cuts group A into several batches, through mb200_align_groups and
mb200_msa_join under both BuildPost routes.  Posterior matrix, path and score are compared bit for bit
against the oracle's BuildPost + CalcAlnFlat."""
import numpy as np
import pytest
from muscle_b200 import synth

pytestmark = pytest.mark.gpu

ROUTES = ["0", "1000000000000"]          # terms bucketed by cell / ordered row walk
AW_W, AW_MAXW = 128, 16                  # columns per strip, strips per CTA (align.cu)
BATCH_ROWS = 16 << 20                    # (residue of A, member of B) rows per BuildPost batch, both routes

# (cols_a, cols_b): one CTA with the traceback in shared memory (700 x 8 strips x 32 B = 179 200 B),
# one CTA with it in global memory, exactly 16 strips, two CTAs per problem
SHAPES = [(700, 1000), (800, 1000), (600, 2048), (600, 2049)]


def layout(cols_a, cols_b):
	"""-> (CTAs per problem, traceback in shared memory) as join_core chooses them"""
	nstrips = (cols_b + AW_W - 1)//AW_W
	npass = (nstrips + AW_MAXW - 1)//AW_MAXW
	return npass, npass == 1 and cols_a*nstrips*32 <= 192*1024


def test_shapes_cover_the_layouts():
	assert [layout(a, b) for a, b in SHAPES] == [(1, True), (1, False), (1, False), (2, False)]
	assert (2048 + AW_W - 1)//AW_W == AW_MAXW


def check_against_oracle(engine, oracle, lens, offs, ents, ids_a, p2c_a, cols_a, ids_b, p2c_b, cols_b):
	want = oracle.buildpost(lens, ids_a, p2c_a, cols_a, ids_b, p2c_b, cols_b, offs, ents)
	score, path, post = engine.align_groups(ids_a, p2c_a, cols_a, ids_b, p2c_b, cols_b, want_post=True)
	assert post.tobytes() == want.tobytes()
	s, pth = oracle.calcaln(want)
	assert np.float32(s) == np.float32(score) and pth == path
	return score, path, post


def shifted_maps(rng, lens, ids, cols):
	"""ungapped pos->col maps at random offsets; the last member ends in the last column"""
	shifts = [int(rng.integers(0, cols - lens[i] + 1)) for i in ids[:-1]] + [cols - lens[ids[-1]]]
	return [np.arange(lens[i], dtype=np.uint32) + sh for i, sh in zip(ids, shifts)]


@pytest.fixture
def family(engine):
	seqs = synth.make_family(6, 500, 0, seed=41, uniform=(470, 530))
	engine.set_seqs(seqs)
	engine.posteriors_allpairs()
	engine.consistency_iter()
	offs, ents = engine.export_all()
	return [len(s) for s in seqs], offs, ents


@pytest.mark.parametrize("bp_sort_min", ROUTES)
@pytest.mark.parametrize("cols_a,cols_b", SHAPES)
def test_align_groups_layouts(engine, oracle, family, monkeypatch, bp_sort_min, cols_a, cols_b):
	monkeypatch.setenv("MB200_BP_SORT_MIN", bp_sort_min)
	lens, offs, ents = family
	rng = np.random.default_rng(cols_a*7 + cols_b)
	ids_a, ids_b = [0, 2, 4], [1, 3, 5]
	p2c_a, p2c_b = shifted_maps(rng, lens, ids_a, cols_a), shifted_maps(rng, lens, ids_b, cols_b)
	check_against_oracle(engine, oracle, lens, offs, ents, ids_a, p2c_a, cols_a, ids_b, p2c_b, cols_b)


@pytest.mark.parametrize("bp_sort_min", ROUTES)
def test_msa_join_layouts(engine, oracle, monkeypatch, bp_sort_min):
	"""one sequence per group, so that each MSA has exactly as many columns as residues (msa_join does
	not return the posterior matrix: path and score)"""
	monkeypatch.setenv("MB200_BP_SORT_MIN", bp_sort_min)
	base = synth.make_family(4, 2200, 0, seed=43, uniform=(2100, 2300))
	want_lens = sorted({n for shape in SHAPES for n in shape})
	seqs = [base[k % len(base)][:n] for k, n in enumerate(want_lens)]
	lens = [len(s) for s in seqs]
	assert lens == want_lens
	engine.set_seqs(seqs)
	engine.posteriors_allpairs()
	offs, ents = engine.export_all()
	for cols_a, cols_b in SHAPES:
		a, b = lens.index(cols_a), lens.index(cols_b)
		want = oracle.buildpost(lens, [a], [np.arange(cols_a, dtype=np.uint32)], cols_a, [b], [np.arange(cols_b, dtype=np.uint32)],
		  cols_b, offs, ents)
		s, pth = oracle.calcaln(want)
		engine.msa_reset()
		_, score, path = engine.msa_join([a], [b], want_path=True)
		assert np.float32(s) == np.float32(score) and pth == path, (cols_a, cols_b)


def test_join_past_the_batch_budget(engine, oracle, monkeypatch):
	"""530 x 530 sequences of ~66 residues: more than BATCH_ROWS (residue of A, member of B) rows, so that
	both routes cut A into at least two batches.  The routes must agree with each other and with the
	oracle (a wrong cut that both routes share would agree with itself)."""
	seqs = synth.make_family(1060, 66, 0, seed=45, uniform=(62, 70))
	lens = [len(s) for s in seqs]
	engine.set_seqs(seqs)
	engine.posteriors_allpairs()
	offs, ents = engine.export_all()
	ids_a, ids_b = list(range(0, 1060, 2)), list(range(1, 1060, 2))
	assert sum(lens[i] for i in ids_a)*len(ids_b) > BATCH_ROWS
	rng = np.random.default_rng(47)
	cols_a, cols_b = max(lens) + 9, max(lens) + 5
	p2c_a, p2c_b = shifted_maps(rng, lens, ids_a, cols_a), shifted_maps(rng, lens, ids_b, cols_b)
	got = []
	for bp_sort_min in ROUTES:
		monkeypatch.setenv("MB200_BP_SORT_MIN", bp_sort_min)
		got.append(check_against_oracle(engine, oracle, lens, offs, ents, ids_a, p2c_a, cols_a, ids_b, p2c_b, cols_b))
	(s0, path0, post0), (s1, path1, post1) = got
	assert post0.tobytes() == post1.tobytes() and path0 == path1 and np.float32(s0) == np.float32(s1)
	assert float(post0.max()) > 1.0
