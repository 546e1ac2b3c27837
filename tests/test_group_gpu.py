"""GPU: the single-process multi-device group (mb200_group_*, group.cu) with several members on one device.

`muscle_b200 -align`, `-super5` and `-profalign` run their posterior stage through a group: the pairs are
split into cell-balanced ranges (shard_pairs), every member computes its range on its own host thread,
every packed image is copied to every member (exchange 1), and after each sharded consistency iteration
every member's updated entry range is copied to the others (exchange 2).  The serial stages then run on
member 0, on the store it adopted.  A member list may repeat a device: each member is its own context
with its own stream and buffers, and a same-device peer copy is an ordinary device-to-device copy.  So
Group([0, 0, 0]) runs all of that code on one GPU.

Every check here compares with tolerance 0: the EA vector and, on every member, the store after the
posterior stage and after each iteration against a fresh single Engine on the same inputs (and one case
against the CPU oracle directly); the serial stages on member 0 against the same calls on the single
engine; and the CLI's MSAs with three members on device 0 against the reference's goldens."""
import os
import random
import subprocess
import numpy as np
import pytest
import emission_util as eu
from conftest import GOLDEN
from muscle_b200 import synth
from repeat_util import mixed_family, repeat_family
from test_e2e_cli_gpu import CLI, E2E, read_afa
from test_msa_gpu import host_join, project, rows_from_device

pytestmark = pytest.mark.gpu

ROUTES = ["1000000000000", "0"]          # MB200_BP_SORT_MIN: ordered row walk / contributions sorted by cell
DEFAULT_NNZ_PER_ROW_CAP = 12             # engine.h


@pytest.fixture(scope="module")
def cuda():
	import torch
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")
	return torch.cuda.device_count()


def shard_pairs(lens, ndev):
	"""group.cu's shard_pairs restated: contiguous ranges of the row-major pair list with about equal
	cells (sum of LX*LY) per member, in the same double arithmetic -> [(lo, hi)] per member"""
	n = len(lens)
	total = 0.0
	for i in range(n):
		for j in range(i + 1, n):
			total += float(lens[i])*lens[j]
	lo, hi = [0]*ndev, [0]*ndev
	run, p, r = 0.0, 0, 0
	for i in range(n):
		for j in range(i + 1, n):
			while r + 1 < ndev and run >= total*(r + 1)/ndev:
				hi[r] = p
				r += 1
				lo[r] = p
			run += float(lens[i])*lens[j]
			p += 1
	hi[r] = p
	for q in range(r + 1, ndev):
		lo[q] = hi[q] = p
	return list(zip(lo, hi))


def dna(seqs):
	"""a protein family written in ACGT (related sequences stay related)"""
	tr = str.maketrans(synth.AMINO, "ACGT"*5)
	return [s.translate(tr) for s in seqs]


def nucleo_tables():
	z = np.load(os.path.join(GOLDEN, "hmm_nucleo.npz"))
	return {k: z[k] for k in ("start", "trans", "ins", "match", "min_sparse_score")}


def plain(tables, seqs):
	def load(x):
		x.set_hmm(tables)
		x.set_seqs(seqs)
	return load


def engine_run(load, iters=2):
	"""a fresh single Engine: posteriors of all pairs, then `iters` consistency iterations
	-> dict(ea, cells, nnz, tot, stores = [store after the posteriors, after iteration 1, ...])"""
	from muscle_b200.engine import Engine
	e = Engine(0)
	load(e)
	out = {"ea": e.posteriors_allpairs(), "cells": e.stats()["cells"]}
	out["nnz"], out["tot"] = e.store_nnz()
	out["stores"] = [e.export_all()]
	for _ in range(iters):
		e.consistency_iter()
		out["stores"].append(e.export_all())
	e.close()
	return out


def assert_store(got, want, what):
	offs, ents = got
	woffs, wents = want
	assert len(offs) == len(woffs), what
	for p in range(len(woffs)):
		assert np.array_equal(offs[p], woffs[p]), (what, "offsets", p)
		assert ents[p].tobytes() == wents[p].tobytes(), (what, "entries", p)


def assert_members(g, want, what):
	for r in range(g.size):
		assert_store(g.engine(r).export_all(), want, (what, "member %d" % r))


def group_run(g, want, iters=2):
	"""the group's posterior stage and `iters` iterations on its current inputs, every member checked
	after every step against a single-engine run (engine_run); also the group's byte counts"""
	n, lens = g.nseq, [int(x) for x in g.lens]
	ea = g.posteriors_allpairs()
	assert ea.tobytes() == want["ea"].tobytes()
	assert_members(g, want["stores"][0], "posteriors")
	st = g.stats()
	assert st["ndev"] == g.size
	assert st["cells"] == want["cells"]
	if g.size > 1:
		rows = sum((lens[i] + 1)*(n - 1 - i) for i in range(n))
		assert st["exchange1_bytes_per_dev"] == 4*rows + 8*want["tot"]
	for it in range(iters):
		g.consistency_iter()
		assert_members(g, want["stores"][it + 1], "iteration %d" % (it + 1))
		if g.size > 1 and n >= 3:
			assert g.stats()["exchange2_bytes_per_dev"] == 8*want["tot"]
	return ea


# ------------------------------------------------------------------------------------------------
# the group's own edges
def seqs_family30():
	return synth.make_family(30, 100, 25, seed=35)


def seqs_dominant():
	"""two 1500-residue sequences among short ones: their pair holds most of the cells, so the members
	after the one that takes it get empty ranges"""
	s = synth.make_family(9, 30, 6, seed=51)
	long_pair = synth.make_family(2, 1500, 10, seed=52)
	return s[:3] + long_pair + s[3:]


def seqs_repeat():
	"""repeats of one motif: every pair is dense, so the ranges of 3 and 5 members start and end between
	pairs of more than 1024 entries"""
	return repeat_family(12, 1, lmin=150, motifs=["QQQP"])


CASES = {
	"family30": seqs_family30,
	"n2": lambda: synth.make_family(2, 90, 20, seed=61),
	"n3": lambda: synth.make_family(3, 90, 20, seed=62),
	"dominant": seqs_dominant,
	"repeat": seqs_repeat,
	"mixed70": lambda: mixed_family(70, 4),       # N > 64: k_relax's z loop runs in more than one chunk
}


def check_shards(case, seqs, ranges, want):
	"""the configuration reaches the edge it is meant for"""
	nonempty = [r for r, (lo, hi) in enumerate(ranges) if hi > lo]
	npairs = len(seqs)*(len(seqs) - 1)//2
	assert ranges[0][0] == 0 and ranges[-1][1] == npairs
	assert all(ranges[r][1] == ranges[r + 1][0] for r in range(len(ranges) - 1))
	if case in ("n2", "n3"):
		assert len(ranges) > npairs and len(nonempty) <= npairs
	elif case == "dominant":
		middle = [r for r in range(nonempty[0] + 1, nonempty[-1]) if r not in nonempty]
		assert middle, ranges
		# the pair of the two long sequences is the last of its member's range
		big = int(np.argmax([len(seqs[i])*len(seqs[j]) for i in range(len(seqs)) for j in range(i + 1, len(seqs))]))
		assert any(hi == big + 1 for lo, hi in ranges), (big, ranges)
	elif case == "repeat":
		for r in nonempty[1:]:
			lo = ranges[r][0]
			assert want["nnz"][lo - 1] > 1024 and want["nnz"][lo] > 1024, (r, ranges)
	elif case == "mixed70":
		assert len(seqs) > 64


GROUP_CASES = [("family30", 2), ("family30", 3), ("family30", 5), ("family30", 8), ("n2", 3), ("n3", 8),
  ("dominant", 5), ("repeat", 3), ("repeat", 5), ("mixed70", 8), ("family30", "0,1,0,1")]


@pytest.mark.parametrize("case,members", GROUP_CASES, ids=["%s-%s" % c for c in GROUP_CASES])
def test_group_equals_engine(cuda, tables, case, members):
	from muscle_b200.engine import Group
	if isinstance(members, str):
		devices = [int(d) for d in members.split(",")]
		if cuda < 2:
			pytest.skip("a mixed member list needs 2 GPUs")
	else:
		devices = [0]*members
	seqs = CASES[case]()
	want = engine_run(plain(tables, seqs))
	ranges = shard_pairs([len(s) for s in seqs], len(devices))
	check_shards(case, seqs, ranges, want)
	g = Group(devices)
	assert g.size == len(devices)
	g.set_hmm(tables)
	g.set_seqs(seqs)
	group_run(g, want)
	g.close()


def test_group_vs_oracle(cuda, tables, oracle):
	"""one sharded case pinned to the oracle itself, so that a fault shared by the engine and the group
	cannot hide"""
	from muscle_b200.engine import Group
	seqs = synth.make_family(14, 80, 20, seed=71)
	n, lens = len(seqs), [len(s) for s in seqs]
	pairs = [(i, j) for i in range(n) for j in range(i + 1, n)]
	o = oracle.all_pairs(seqs)
	g = Group([0]*5)
	g.set_hmm(tables)
	g.set_seqs(seqs)
	ea = g.posteriors_allpairs()
	assert ea.tobytes() == o["ea"][np.triu_indices(n, 1)].tobytes()
	want = (o["row_off"], o["entries"])
	assert_members(g, want, "posteriors")
	for it in range(2):
		want = (want[0], oracle.conspair_many(lens, pairs, want[0], want[1]))
		g.consistency_iter()
		assert_members(g, want, "iteration %d" % (it + 1))
	g.close()


@pytest.mark.parametrize("case,members", [("family30", 5), ("dominant", 5), ("repeat", 3)])
def test_member_cells(cuda, tables, case, members):
	"""each non-empty member computed exactly its range of shard_pairs: its cells equal a single engine's
	for posteriors_allpairs(lo, hi), and they add up to the single engine's all-pairs cells"""
	from muscle_b200.engine import Engine, Group
	seqs = CASES[case]()
	ranges = shard_pairs([len(s) for s in seqs], members)
	e = Engine(0)
	e.set_hmm(tables)
	e.set_seqs(seqs)
	e.posteriors_allpairs()
	all_cells = e.stats()["cells"]
	g = Group([0]*members)
	g.set_hmm(tables)
	g.set_seqs(seqs)
	g.posteriors_allpairs()
	total = 0
	for r, (lo, hi) in enumerate(ranges):
		if hi == lo:
			continue
		e.posteriors_allpairs(lo, hi)
		assert g.engine(r).stats()["cells"] == e.stats()["cells"], (r, lo, hi)
		total += e.stats()["cells"]
	assert total == all_cells == g.stats()["cells"]
	assert g.stats()["ndev"] == members
	g.close()
	e.close()


# ------------------------------------------------------------------------------------------------
def test_group_reuse(cuda, tables):
	"""one group runs several sequence sets in turn (what -super5 does per cluster), switches to the
	nucleotide tables on the way, and repeats the posterior stage on unchanged sequences after consistency"""
	from muscle_b200.engine import Group
	g = Group([0]*5)
	g.set_hmm(tables)
	nuc = nucleo_tables()
	runs = [(tables, synth.make_family(30, 100, 25, seed=81)), (tables, synth.make_family(12, 150, 40, seed=82)),
	  (nuc, dna(synth.make_family(2, 200, 10, seed=83))), (nuc, dna(synth.make_family(41, 70, 30, seed=84)))]
	current = tables
	for t, seqs in runs:
		if t is not current:
			g.set_hmm(t)
			current = t
		g.set_seqs(seqs)
		want = engine_run(plain(t, seqs))
		group_run(g, want)
	# again on the same sequences, after two iterations changed every member's store
	group_run(g, want)
	g.close()


def serial_stages(e, seqs, ea, seed, monkeypatch):
	"""the serial stages as the CLI runs them on member 0 -> list of every result"""
	out = [[a.tobytes() for a in e.guide_tree(ea)]]
	n = len(seqs)
	rng = random.Random(seed)
	e.msa_reset()
	members = {i: [i] for i in range(n)}
	nodes, nxt = list(range(n)), n
	while len(nodes) > 1:                                     # a random join order
		a, b = rng.sample(nodes, 2)
		cols, score, path = e.msa_join(members[a], members[b], want_path=True)
		out.append((cols, np.float32(score).tobytes(), path))
		members[nxt] = members[a] + members[b]
		nodes = [x for x in nodes if x not in (a, b)] + [nxt]
		nxt += 1
	msa = rows_from_device(e, seqs, members[nodes[0]])
	out.append(msa)
	for it in range(5):                                       # refinement joins of projected bipartitions
		pick = [rng.random() < 0.5 for _ in msa]
		g1 = [x for x, f in zip(msa, pick) if f]
		g2 = [x for x, f in zip(msa, pick) if not f]
		if not g1 or not g2:
			continue
		m1 = list(zip([i for i, _ in g1], project([r for _, r in g1])))
		m2 = list(zip([i for i, _ in g2], project([r for _, r in g2])))
		for route in ROUTES:
			monkeypatch.setenv("MB200_BP_SORT_MIN", route)
			joined, path, score = host_join(e, m1, m2)                # align_groups of the gapped groups
			out.append((route, joined, path, np.float32(score).tobytes()))
		monkeypatch.delenv("MB200_BP_SORT_MIN")
		cols, score, path = e.msa_join([i for i, _ in m1], [i for i, _ in m2], want_path=True)
		assert path == out[-1][2]
		msa = rows_from_device(e, seqs, [i for i, _ in m1] + [i for i, _ in m2])
		out.append((cols, np.float32(score).tobytes(), path, msa))
	return out


def test_serial_stages_on_member0(cuda, tables, monkeypatch):
	"""after a sharded run, member 0's adopted store drives the guide tree, the progressive joins and the
	refinement exactly like a single engine's store; it carries no EA vector of its own"""
	from muscle_b200.engine import Engine, Group, MB200Error
	seqs = synth.make_family(16, 110, 30, seed=91)
	e = Engine(0)
	e.set_hmm(tables)
	e.set_seqs(seqs)
	ea = e.posteriors_allpairs()
	e.consistency_iter()
	e.consistency_iter()
	want = serial_stages(e, seqs, ea, 5, monkeypatch)
	g = Group([0]*3)
	g.set_hmm(tables)
	g.set_seqs(seqs)
	ea_g = g.posteriors_allpairs()
	assert ea_g.tobytes() == ea.tobytes()
	g.consistency_iter()
	g.consistency_iter()
	m0 = g.engine(0)
	with pytest.raises(MB200Error):
		m0.guide_tree()
	got = serial_stages(m0, seqs, ea_g, 5, monkeypatch)
	assert len(got) == len(want)
	for k, (a, b) in enumerate(zip(got, want)):
		assert a == b, k
	g.close()
	e.close()


def test_entry_pool_retry_in_one_member(cuda, tables):
	"""member 1 sizes its entry pool for one entry per row, so its posterior stage overflows and retries
	with the exact count; nothing may change"""
	from muscle_b200.engine import Group
	seqs = seqs_family30()
	want = engine_run(plain(tables, seqs))
	ranges = shard_pairs([len(s) for s in seqs], 3)
	assert ranges[1][1] > ranges[1][0]
	g = Group([0]*3)
	g.set_hmm(tables)
	g.set_seqs(seqs)
	g.engine(1).set_nnz_per_row_cap(1)
	try:
		group_run(g, want)
	finally:
		g.engine(1).set_nnz_per_row_cap(DEFAULT_NNZ_PER_ROW_CAP)
	group_run(g, want)
	g.close()


def test_group_mega(cuda, tables):
	"""a random Mega model and family through Group.set_seqs_mega with 3 members == a single engine in
	Mega mode"""
	from muscle_b200.engine import Group
	model = eu.mega_model([20, 16, 6, 11], [0.4, 0.2, 0.3, 0.1], 95)
	vocab = eu.vocabulary(model, 127, 95)
	lengths = [int(x) for x in np.random.default_rng(95).integers(40, 220, 11)]
	profiles, _ = eu.mega_family(vocab, lengths, 95)

	def load(x):
		x.set_hmm(tables)                 # the transitions
		x.set_seqs_mega(model, profiles)
	want = engine_run(load)
	g = Group([0]*3)
	load(g)
	assert g.nseq == len(profiles) and list(g.lens) == lengths
	group_run(g, want)
	g.close()


def test_second_context_on_the_device(cuda, tables):
	"""-super5 keeps a pair-list context next to the group: a standalone engine's pair-list posteriors and
	align_pairs, interleaved with the group's steps, change neither side's results"""
	from muscle_b200.engine import Engine, Group
	seqs = synth.make_family(20, 90, 25, seed=101)
	other = synth.make_family(9, 130, 30, seed=102)
	rng = np.random.default_rng(103)
	px = rng.integers(0, 9, 24)
	py = (px + rng.integers(1, 9, 24)) % 9
	sel = list(range(0, 24, 2))

	def side(e, k):
		"""pair-list step k of the standalone engine"""
		if k % 2 == 0:
			return [e.posteriors(px, py).tobytes()] + [a.tobytes() for a in e.export_all()[1]]
		scores, paths = e.align_pairs(sel)
		return [scores.tobytes()] + paths

	iso = Engine(0)
	iso.set_hmm(tables)
	iso.set_seqs(other)
	want_side = [side(iso, k) for k in range(4)]
	iso.close()
	want = engine_run(plain(tables, seqs))
	s = Engine(0)
	s.set_hmm(tables)
	s.set_seqs(other)
	g = Group([0]*3)
	g.set_hmm(tables)
	got_side = [side(s, 0)]
	g.set_seqs(seqs)
	ea = g.posteriors_allpairs()
	got_side.append(side(s, 1))
	assert ea.tobytes() == want["ea"].tobytes()
	assert_members(g, want["stores"][0], "posteriors")
	for it in range(2):
		g.consistency_iter()
		got_side.append(side(s, it + 2))
		assert_members(g, want["stores"][it + 1], "iteration %d" % (it + 1))
	assert got_side == want_side
	g.close()
	s.close()


def test_call_order_and_errors(cuda, tables):
	from muscle_b200.engine import Group, MB200Error
	seqs = synth.make_family(6, 60, 10, seed=111)
	g = Group([0, 0])
	with pytest.raises(MB200Error):
		g.consistency_iter()                       # fresh: no sequences, no store
	g.set_hmm(tables)
	g.set_seqs(seqs)
	with pytest.raises(MB200Error):
		g.consistency_iter()                       # no sharded posterior stage yet
	g.posteriors_allpairs()
	g.consistency_iter()
	g.set_seqs(seqs[:5])
	with pytest.raises(MB200Error):
		g.consistency_iter()                       # the sharded store belongs to the previous sequences
	g.set_seqs(seqs[:1])
	with pytest.raises(MB200Error):
		g.posteriors_allpairs()                    # one sequence has no pairs
	g.close()
	for devices in ([0, cuda], [0, 0, -1]):          # a device that does not exist: the members made are destroyed
		with pytest.raises(MB200Error):
			Group(devices)
	g = Group([0, 0])
	want = engine_run(plain(tables, seqs))
	g.set_hmm(tables)
	g.set_seqs(seqs)
	group_run(g, want)
	g.close()


def test_device_list_from_environment(cuda, tables, monkeypatch):
	"""MB200_DEVICE_LIST sets the members of a group whose caller passes no device list (what the CLI's
	binding does); an explicit list wins, and a malformed one is refused"""
	from muscle_b200.engine import Group, MB200Error
	seqs = synth.make_family(9, 70, 15, seed=121)
	want = engine_run(plain(tables, seqs))
	monkeypatch.setenv("MB200_DEVICE_LIST", "0,0,0")
	g = Group(None)
	assert g.size == 3
	g.set_hmm(tables)
	g.set_seqs(seqs)
	group_run(g, want)
	g.close()
	g = Group([0, 0])
	assert g.size == 2
	g.close()
	for bad in ("", "0,", "0;0", "0,,0", "x", "0,-1", "0,%d" % cuda):
		monkeypatch.setenv("MB200_DEVICE_LIST", bad)
		with pytest.raises(MB200Error):
			Group(None)
	monkeypatch.delenv("MB200_DEVICE_LIST")
	g = Group(None)
	assert g.size == cuda
	g.close()


# ------------------------------------------------------------------------------------------------
# the CLI through a sharded group: three members on device 0
def run_cli(args, tmp_path, out_name, timeout=900):
	if not os.path.exists(CLI):
		pytest.skip("integration/_build/muscle_b200 not built (needs oracle/_ref built from the reference sources)")
	out = tmp_path / out_name
	env = {k: v for k, v in os.environ.items() if k not in ("MB200_DEVICE", "MB200_DEVICES")}
	env["MB200_DEVICE_LIST"] = "0,0,0"
	env["MB200_TRACE"] = "1"                      # reports the group's member count at exit
	r = subprocess.run([CLI] + args + ["-output", str(out), "-quiet"], capture_output=True, text=True, timeout=timeout,
	  env=env)
	assert r.returncode == 0, r.stderr[-2000:]
	assert "[mb200 trace] 3 GPU(s)" in r.stderr, r.stderr[-2000:]
	return read_afa(out)


@pytest.mark.parametrize("name", ["fam12", "rep16"])
def test_cli_align_three_members(cuda, tmp_path, name):
	got = run_cli(["-align", os.path.join(E2E, name + ".fa")], tmp_path, name + ".afa")
	assert got == read_afa(os.path.join(E2E, name + ".ref.afa"))


def test_cli_align_c2_three_members(cuda, tmp_path):
	ref = os.path.join(E2E, "c2.ref.afa")
	if not os.path.exists(ref):
		pytest.skip("c2 golden not generated")
	fa = tmp_path / "c2.fa"
	with open(fa, "w") as f:
		for i, q in enumerate(synth.make_config("C2")):
			f.write(">s%d\n%s\n" % (i, q))
	assert run_cli(["-align", str(fa)], tmp_path, "c2.afa") == read_afa(ref)


def test_cli_align_mega_three_members(cuda, tmp_path):
	got = run_cli(["-align", os.path.join(E2E, "BB11001.mega")], tmp_path, "bb11001.afa")
	assert got == read_afa(os.path.join(E2E, "BB11001.mega.ref.afa"))


def test_cli_profalign_three_members(cuda, tmp_path):
	got = run_cli(["-profalign", os.path.join(E2E, "profalign_a.afa"), "-input2", os.path.join(E2E, "profalign_b.afa")],
	  tmp_path, "profalign.afa")
	assert got == read_afa(os.path.join(E2E, "profalign.ref.afa"))


def test_cli_super5_three_members(cuda, tmp_path):
	"""-super5 re-uses one group for the posterior stage of every cluster, at many different sizes"""
	got = run_cli(["-super5", os.path.join(E2E, "super5_150.fa"), "-threads", "1"], tmp_path, "super5.afa")
	assert got == read_afa(os.path.join(E2E, "super5_150.ref.afa"))
