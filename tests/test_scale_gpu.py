"""GPU: the stages after the posteriors at the full size of C4 (128 sequences of 1500-3000 residues)
and C3 (1000 sequences of about 350, the benchmark's workload), tolerance 0 against the C oracle
(itself pinned to the compiled reference, tests/test_oracle_vs_ref.py, test_crafted_store_cpu.py).

These sizes reach what the small tests never produce: a relax store past 4 GiB with pair indexes up to
499 499 and z past several 64-sequence chunks, joins that take the by-cell BuildPost route on their
own and cut group A into three or more batches, and decoding DPs of two or more CTAs.

C4 runs the whole pipeline with every step checked: two consistency iterations on sampled pairs, the
guide tree under all four linkages, all 127 joins of the tree and 10 refinement joins.  C3 checks two
consistency iterations on the 28 pairs of 8 sequences, the guide tree, every tree join of at most 4096
sequence pairs, and one refinement join of 400 x 400 rows, against the oracle on stores that hold only
the pairs each call reads (tests/scale_util.py).  The largest C3 joins are out of the oracle's reach;
there the two BuildPost routes are checked against each other and against msa_join.

Measured on one H100 80GB HBM3 (700 W): the file takes about 100 s, the C3 consistency iteration 16.7 s.
The device in use reached 74.5 GB after the C3 posterior stage (its entry pool and scratch) and stood at
70.0 GB after relax (torch.cuda.mem_get_info, whole device)."""
import os
import time
from concurrent.futures import ThreadPoolExecutor
import numpy as np
import pytest
from muscle_b200 import synth
import scale_util as su

pytestmark = pytest.mark.gpu

ROUTES = ["0", "1000000000000"]          # MB200_BP_SORT_MIN: terms bucketed by cell / ordered row walk
BY_CELL_MIN = 1000000                    # (residues of A) x |B| from which a join goes by cell (align.cu join_core)
BATCH_ROWS = 16 << 20                    # (residue of A, member of B) rows per by-cell batch (align.cu)
AW_W, AW_MAXW = 128, 16                  # decoding DP: columns per strip, strips per CTA (align.cu)
RELAX_SWEEP = 256*4                      # entries of one pair k_relax holds per sweep (RELAX_THREADS x RELAX_EPT)
SMALL_JOIN = 4096                        # C3 tree joins with at most this many sequence pairs go to the oracle
C3_ITERS = 2                             # consistency iterations at C3 (MPCFlat's default)


def log(msg):
	print("[scale] " + msg, flush=True)


def batches(lens, ids_a, nb, budget=BATCH_ROWS):
	"""the number of batches BuildPost cuts A into (align.cu member_batches)"""
	rb = np.concatenate([[0], np.cumsum([lens[i] for i in ids_a])])
	count, s = 0, 0
	while s < len(ids_a):
		e = s + 1
		while e < len(ids_a) and (rb[e + 1] - rb[s])*nb <= budget:
			e += 1
		count += 1
		s = e
	return count


def dp_ctas(cols_b):
	return ((cols_b + AW_W - 1)//AW_W + AW_MAXW - 1)//AW_MAXW


def tree_groups(n, left, right):
	"""(members of the left child, members of the right child) of every internal node, in node order"""
	members = []
	out = []
	for l, r in zip(left.tolist(), right.tolist()):
		a = [l] if l < n else members[l - n]
		b = [r] if r < n else members[r - n]
		out.append((a, b))
		members.append(a + b)
	return out


def project(maps):
	"""drop the columns no member uses (MultiSequence::Project) -> (maps, cols)"""
	used = np.unique(np.concatenate(maps))
	return [np.searchsorted(used, m).astype(np.uint32) for m in maps], len(used)


def group_maps(engine, ids):
	maps, cols = engine.msa_export(ids)
	assert len(set(cols.tolist())) == 1, "the group is not one MSA"
	return project(maps)


def device_join(engine, ids_a, ids_b):
	"""msa_join with the projected maps it starts from; checks the MSA it leaves against the path.
	-> (maps_a, cols_a, maps_b, cols_b, score, path)"""
	ma, ca = group_maps(engine, ids_a)
	mb, cb = group_maps(engine, ids_b)
	cols, score, path = engine.msa_join(ids_a, ids_b, want_path=True)
	p = np.frombuffer(path.encode(), np.uint8)
	assert cols == len(path) and (p != ord("Y")).sum() == ca and (p != ord("X")).sum() == cb
	new_a, new_b = np.flatnonzero(p != ord("Y")), np.flatnonzero(p != ord("X"))
	after, cols2 = engine.msa_export(ids_a + ids_b)
	assert (cols2 == cols).all()
	want = [new_a[m] for m in ma] + [new_b[m] for m in mb]
	assert all(np.array_equal(w, g) for w, g in zip(want, after)), "MSA after the join"
	return ma, ca, mb, cb, score, path


def same_tree(a, b):
	return all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def check_relax(engine, oracle, store, pairs, tag):
	"""one consistency iteration; the new entries of `pairs` against conspair on `store`"""
	n = len(engine.lens)
	want = store.conspair_many(oracle, pairs)
	t0 = time.time()
	engine.consistency_iter()
	log("%s consistency iteration: %.1f s (k_relax %.0f ms)" % (tag, time.time() - t0, engine.stats()["last_kernel_ms"]))
	nnz, _ = engine.store_nnz()
	for (x, y), w in zip(pairs, want):
		k = su.pair_index(n, x, y)
		_, got = engine.export_pair(k, int(nnz[k]))
		assert got.tobytes() == w.tobytes(), "%s pair (%d, %d)" % (tag, x, y)


def relax_shapes(store, pairs):
	"""(largest entry count of the pairs, rows of theirs that span more than one 32-column mask word)"""
	n = store.n
	most, wide = 0, 0
	for x, y in pairs:
		k = su.pair_index(n, x, y)
		off, ent = store.offs[k], store.ents[k]
		most = max(most, len(ent))
		nz = np.flatnonzero(np.diff(off.astype(np.int64)) > 0)
		first, last = ent["col"][off[nz]] >> 5, ent["col"][off[nz + 1] - 1] >> 5
		wide += int((last != first).sum())
	return most, wide


@pytest.fixture
def library_route(monkeypatch):
	monkeypatch.delenv("MB200_BP_SORT_MIN", raising=False)


# ------------------------------------------------------------------------------------------------
# C4: 128 x 1500-3000, every step
def test_c4_pipeline(engine, oracle, library_route):
	seqs = synth.make_config("C4")
	n = len(seqs)
	lens = [len(s) for s in seqs]
	t0 = time.time()
	engine.set_seqs(seqs)
	ea = engine.posteriors_allpairs()
	for link in (1, 2, 3, 4):
		assert same_tree(engine.guide_tree(None, link), oracle.upgma(n, ea, link)), ("guide tree", link)
	# relax: every pair among the 3 longest and 3 shortest, (0, 127), and random pairs
	order = np.argsort(lens, kind="stable")
	ends = sorted(order[:3].tolist() + order[-3:].tolist())
	pairs = {(x, y) for i, x in enumerate(ends) for y in ends[i + 1:]} | {(0, n - 1)}
	rng = np.random.default_rng(4)
	while len(pairs) < 200:
		x, y = sorted(rng.choice(n, 2, replace=False).tolist())
		pairs.add((x, y))
	pairs = sorted(pairs)
	for it in range(2):
		store = su.PairStore.full(lens, *engine.export_all())
		if it == 0:
			most, wide = relax_shapes(store, pairs)
			assert most > 2*RELAX_SWEEP and wide > 0, (most, wide)
		check_relax(engine, oracle, store, pairs, "C4 iteration %d" % it)
		del store
	store = su.PairStore.full(lens, *engine.export_all())
	# progressive alignment along the tree, then refinement joins of random bipartitions
	left, right, _, _ = engine.guide_tree()
	engine.msa_reset()
	checks, reached = [], {"ctas": 0, "by_cell": 0}
	with ThreadPoolExecutor(su.workers()) as pool:
		def join(ids_a, ids_b, tag):
			ma, ca, mb, cb, score, path = device_join(engine, ids_a, ids_b)
			reached["ctas"] = max(reached["ctas"], dp_ctas(cb))
			reached["by_cell"] += sum(lens[i] for i in ids_a)*len(ids_b) >= BY_CELL_MIN
			checks.append((tag, score, path, pool.submit(store.join, oracle, ids_a, ma, ca, ids_b, mb, cb)))
		for k, (a, b) in enumerate(tree_groups(n, left, right)):
			join(a, b, "tree join %d" % k)
		for it in range(10):
			pick = rng.random(n) < 0.5
			a, b = np.flatnonzero(pick).tolist(), np.flatnonzero(~pick).tolist()
			join(a, b, "refinement %d" % it)
		for tag, score, path, fut in checks:
			s, p = fut.result()
			assert p == path and np.float32(s) == np.float32(score), tag
	assert reached["ctas"] >= 2 and reached["by_cell"] > 0, reached
	log("C4: %d joins, DP up to %d CTAs, %d by cell; %.1f s" % (len(checks), reached["ctas"], reached["by_cell"], time.time() - t0))


# ------------------------------------------------------------------------------------------------
# C3: 1000 x ~350, the benchmark's workload
def relax_need(lens, tot):
	"""device bytes a consistency iteration holds (relax.cu, store.cu): three entry images (forward, the
	Jacobi copy, transposed) and the permutation; offsets, mask headers and scratch per row slot of each
	orientation; about 1.6 mask words per row (relax.cu), counted as 2"""
	L = np.asarray(lens, np.int64)
	n = len(L)
	rows = int(((L + 1)*(n - 1 - np.arange(n))).sum())       # forward slots: LX + 1 per pair
	trows = int(((L + 1)*np.arange(n)).sum())                # transposed slots: LY + 1 per pair
	return 28*tot + (4 + 8 + 16)*(rows + trows) + 12*max(rows, trows)


def device_used():
	import torch
	free, total = torch.cuda.mem_get_info()
	return total - free


@pytest.fixture(scope="module")
def c3(engine, oracle):
	"""posteriors and two consistency iterations (as -align runs them); the 28 pairs of 8 sequences before
	and after each"""
	import torch
	from muscle_b200.engine import MB200Error
	seqs = synth.make_config("C3")
	n = len(seqs)
	lens = [len(s) for s in seqs]
	engine.set_seqs(seqs)
	ea = engine.posteriors_allpairs()
	nnz, tot = engine.store_nnz()
	need = relax_need(lens, tot)
	free, total = torch.cuda.mem_get_info()
	# most of what is in use is this engine's store and posterior scratch, which relax reuses or frees: the need
	# is weighed against the card.  On a card shared with other work the iteration can still run out of memory.
	msg = "C3 relax needs about %.1f GB of device memory: %.1f GB free, %.1f GB in use" % (need/1e9, free/1e9, (total - free)/1e9)
	log(msg + " (%d entries)" % tot)
	if need > total:
		pytest.skip(msg)
	longest = int(np.argmax(lens))
	S = sorted({0, 1, 63, 64, 65, longest, 998, 999})
	pairs = [(x, y) for i, x in enumerate(S) for y in S[i + 1:]]
	want, got = [], []
	for it in range(C3_ITERS):
		t0 = time.time()
		store = su.star_store(engine, lens, S, nnz)
		t1 = time.time()
		want.append(store.conspair_many(oracle, pairs))
		log("C3 star store of %d sequences: %d pairs exported in %.1f s, conspair of %d pairs %.1f s" % (len(S),
		  int(store.real.sum()), t1 - t0, len(pairs), time.time() - t1))
		if it == 0:
			shapes = relax_shapes(store, pairs)
		del store
		t0 = time.time()
		try:
			engine.consistency_iter()
		except MB200Error as e:
			if e.code == -4:                     # MB200_ENOMEM: the card is shared and too full
				pytest.skip(msg + "; " + str(e))
			raise
		log("C3 consistency iteration %d: %.1f s (k_relax %.0f ms); device in use %.1f GB" % (it, time.time() - t0,
		  engine.stats()["last_kernel_ms"], device_used()/1e9))
		nnz, _ = engine.store_nnz()
		got.append([engine.export_pair(k, int(nnz[k]))[1] for k in (su.pair_index(n, x, y) for x, y in pairs)])
	return {"seqs": seqs, "lens": lens, "ea": ea, "S": S, "pairs": pairs, "want": want, "got": got, "shapes": shapes}


def test_c3_relax(c3):
	pairs, n = c3["pairs"], len(c3["lens"])
	assert len(pairs) == 28 and su.pair_index(n, 998, 999) == 499499 and (0, 1) in pairs and (0, 999) in pairs
	most, wide = c3["shapes"]
	assert most > RELAX_SWEEP and wide > 0, c3["shapes"]
	for it in range(C3_ITERS):
		for (x, y), w, g in zip(pairs, c3["want"][it], c3["got"][it]):
			assert g.tobytes() == w.tobytes(), "C3 iteration %d pair (%d, %d)" % (it, x, y)


def test_c3_guide_tree(engine, oracle, c3):
	n = len(c3["lens"])
	for link in (1, 2, 3, 4):
		assert same_tree(engine.guide_tree(None, link), oracle.upgma(n, c3["ea"], link)), ("guide tree", link)


@pytest.fixture(scope="module")
def c3_msa(engine, oracle, c3):
	"""all 999 joins of the C3 tree on the device, after the consistency iterations.  Joins of at most
	SMALL_JOIN sequence pairs are checked against the oracle; the three largest by both BuildPost routes of
	align_groups."""
	os.environ.pop("MB200_BP_SORT_MIN", None)               # msa_join takes the library's own route
	lens = c3["lens"]
	n = len(lens)
	nnz, _ = engine.store_nnz()
	left, right, _, _ = engine.guide_tree()
	groups = tree_groups(n, left, right)
	rows = [sum(lens[i] for i in a)*len(b) for a, b in groups]
	largest = set(np.argsort(rows)[-3:].tolist())
	engine.msa_reset()
	store = su.PairStore(lens)
	out = {"oracle": 0, "exported": 0, "routes": [], "rows": rows}
	t0 = time.time()
	for k, (a, b) in enumerate(groups):
		if k in largest:
			out["routes"].append(routes_vs_msa_join(engine, a, b, "tree join %d" % k))
		elif len(a)*len(b) <= SMALL_JOIN:
			su.cross_store(engine, lens, a, b, nnz, store)
			ma, ca, mb, cb, score, path = device_join(engine, a, b)
			s, p = store.join(oracle, a, ma, ca, b, mb, cb)
			assert p == path and np.float32(s) == np.float32(score), "tree join %d" % k
			out["oracle"] += 1
			out["exported"] += len(a)*len(b)
		else:
			engine.msa_join(a, b)
	store.clear_all()
	log("C3 tree: %d joins, %d against the oracle (%d pairs exported), largest %d rows; %.1f s" % (len(groups),
	  out["oracle"], out["exported"], max(rows), time.time() - t0))
	return out


def routes_vs_msa_join(engine, ids_a, ids_b, tag):
	"""align_groups under both BuildPost routes, then msa_join: same matrix, path and score -> batches"""
	lens = engine.lens
	ma, ca = group_maps(engine, ids_a)
	mb, cb = group_maps(engine, ids_b)
	got = []
	for r in ROUTES:
		os.environ["MB200_BP_SORT_MIN"] = r
		try:
			got.append(engine.align_groups(ids_a, ma, ca, ids_b, mb, cb, want_post=True))
		finally:
			del os.environ["MB200_BP_SORT_MIN"]
	(s0, p0, post0), (s1, p1, post1) = got
	assert post0.tobytes() == post1.tobytes() and p0 == p1 and np.float32(s0) == np.float32(s1), tag
	del got, post0, post1
	_, _, _, _, score, path = device_join(engine, ids_a, ids_b)
	assert path == p0 and np.float32(score) == np.float32(s0), tag
	return batches(lens, ids_a, len(ids_b))


def test_c3_progressive(c3_msa):
	assert c3_msa["oracle"] > 0
	assert len(c3_msa["routes"]) == 3 and max(c3_msa["rows"]) >= BY_CELL_MIN


def test_c3_join_of_random_halves(engine, c3, c3_msa):
	"""two random halves of the final MSA, projected: about 8.8e7 rows, 6 batches"""
	n = len(c3["lens"])
	perm = np.random.default_rng(33).permutation(n)
	nb = routes_vs_msa_join(engine, sorted(perm[:n//2].tolist()), sorted(perm[n//2:].tolist()), "halves")
	assert nb >= 5, nb


def test_c3_refinement_join_vs_oracle(engine, oracle, c3, c3_msa):
	"""two disjoint sets of 400 rows of the final MSA, projected, against the oracle: about 5.6e7 rows,
	which BuildPost cuts into 4 batches"""
	lens = c3["lens"]
	n = len(lens)
	perm = np.random.default_rng(34).permutation(n)
	a, b = sorted(perm[:400].tolist()), sorted(perm[400:800].tolist())
	nb = batches(lens, a, len(b))
	assert nb >= 3, nb
	nnz, _ = engine.store_nnz()
	ks = su.cross_pairs(n, a, b)
	host = int(8*nnz[ks].astype(np.int64).sum() + 4*sum((lens[min(x, y)] + 1) for x in a for y in b))
	avail = os.sysconf("SC_AVPHYS_PAGES")*os.sysconf("SC_PAGE_SIZE")
	if avail < host + (2 << 30):
		pytest.skip("the 400 x 400 join needs about %.1f GB of host memory for its pairs, %.1f GB available" % (host/1e9, avail/1e9))
	t0 = time.time()
	store = su.cross_store(engine, lens, a, b, nnz)
	t1 = time.time()
	ma, ca = group_maps(engine, a)
	mb, cb = group_maps(engine, b)
	want = store.buildpost(oracle, a, ma, ca, b, mb, cb)
	score, path, post = engine.align_groups(a, ma, ca, b, mb, cb, want_post=True)
	assert post.tobytes() == want.tobytes()
	s, p = oracle.calcaln(want)
	assert p == path and np.float32(s) == np.float32(score)
	del post, want
	_, _, _, _, score2, path2 = device_join(engine, a, b)
	assert path2 == path and np.float32(score2) == np.float32(score)
	log("C3 400 x 400 join: %d batches, %.1f GB of pairs exported in %.1f s, checked in %.1f s" % (nb, host/1e9, t1 - t0,
	  time.time() - t1))
