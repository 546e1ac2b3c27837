"""GPU: the life cycle of the sparse posterior store, walked through one engine.

Every stage after the posterior stage reads the store, and each asks something of it: consistency and
the joins need all N(N-1)/2 pairs, the guide tree without an EA argument needs the EA vector of all
pairs computed on this device, mb200_store_set_values needs the packed layout.  This file writes down,
in one place, which calls a context accepts after each call that produces or drops a store:

  fresh context (tables, no sequences)   posteriors, consistency and joins refused
  posteriors(px, py)                     align_pairs, export_all; not consistency, guide_tree(), msa_join
  posteriors_allpairs(0, k), k < all     not consistency, not guide_tree()
  posteriors_allpairs()                  consistency, guide_tree(), msa_join
  set_hmm                                no store; the MSAs survive
  set_seqs                               no store, no MSAs until msa_reset
  store_load_allpairs / exchange commit  consistency and msa_join; guide_tree() only with an EA argument
  unpacked store                         store_set_values refused until store_pack
  failed posterior call                  no store

Where a call produces a store or an alignment, the result is compared bit for bit with a fresh
engine that made the same store directly."""
import numpy as np
import pytest
from muscle_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
	import torch
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")


def seqs_of(n, seed):
	return synth.make_family(n, 60, 20, seed=seed)


def fresh(tables, seqs):
	from muscle_b200.engine import Engine
	e = Engine(0)
	e.set_hmm(tables)
	e.set_seqs(seqs)
	return e


def refused(call, *args):
	from muscle_b200.engine import MB200Error
	with pytest.raises(MB200Error):
		call(*args)


def same_store(a, b):
	oa, ea = a.export_all()
	ob, eb = b.export_all()
	assert len(oa) == len(ob)
	for p in range(len(oa)):
		assert oa[p].tobytes() == ob[p].tobytes() and ea[p].tobytes() == eb[p].tobytes(), p


def same_tree(a, b):
	assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def reference_run(tables, seqs, iters=1):
	"""posteriors_allpairs, `iters` consistency iterations, one join of sequences 0 and 1 on a fresh engine
	-> (engine, EA, guide tree, join result)"""
	r = fresh(tables, seqs)
	ea = r.posteriors_allpairs()
	tree = r.guide_tree()
	for _ in range(iters):
		r.consistency_iter()
	r.msa_reset()
	return r, ea, tree, r.msa_join([0], [1], want_path=True)


def test_lifecycle(cuda, tables):
	from muscle_b200.engine import Engine
	seqs = seqs_of(7, 41)
	n = len(seqs)
	npairs = n*(n - 1)//2
	ref, ea_ref, tree_ref, join_ref = reference_run(tables, seqs)

	# fresh context with tables, no sequences
	e = Engine(0)
	e.set_hmm(tables)
	refused(e.posteriors, [0], [1])
	refused(e.posteriors_allpairs, 0, 1)
	refused(e.consistency_iter)
	refused(e.msa_join, [0], [1])

	# a pair-list store: decoding and export, nothing that needs all pairs
	e.set_seqs(seqs)
	px, py = [0, 1, 2, 4], [3, 5, 6, 6]
	e.posteriors(px, py)
	r = fresh(tables, seqs)
	r.posteriors(px, py)
	same_store(e, r)
	s_e, p_e = e.align_pairs([0, 2, 3])
	s_r, p_r = r.align_pairs([0, 2, 3])
	assert s_e.tobytes() == s_r.tobytes() and p_e == p_r
	r.close()
	refused(e.consistency_iter)
	refused(e.guide_tree)
	e.msa_reset()
	refused(e.msa_join, [0], [1])

	# part of the all-pairs range
	e.posteriors_allpairs(0, npairs - 4)
	refused(e.consistency_iter)
	refused(e.guide_tree)

	# the whole range
	ea = e.posteriors_allpairs()
	assert ea.tobytes() == ea_ref.tobytes()
	same_tree(e.guide_tree(), tree_ref)
	e.consistency_iter()
	same_store(e, ref)
	assert e.msa_join([0], [1], want_path=True) == join_ref

	# new tables: the store is gone, the MSAs stay
	e.set_hmm(tables)
	refused(e.store_nnz)
	refused(e.export_all)
	refused(e.consistency_iter)
	refused(e.guide_tree)
	refused(e.msa_join, [2], [3])
	e.posteriors_allpairs()
	ref.posteriors_allpairs()
	same_store(e, ref)
	assert e.msa_join([0, 1], [2], want_path=True) == ref.msa_join([0, 1], [2], want_path=True)

	# new sequences: no MSAs until msa_reset
	e.set_seqs(seqs)
	e.posteriors_allpairs()
	refused(e.msa_join, [0], [1])

	# an unpacked store refuses new values; a packed one takes them
	import torch
	v = torch.zeros(4, dtype=torch.float32, device="cuda")
	refused(e.store_set_values_torch, v, 0)
	values = e.store_values_torch()
	e.store_set_values_torch(values, 0)
	e.msa_reset()
	ref.msa_reset()
	assert e.msa_join([0], [1], want_path=True) == ref.msa_join([0], [1], want_path=True)
	e.consistency_iter()
	ref.consistency_iter()
	same_store(e, ref)

	# a failed posterior call leaves no store
	e.set_seqs(["A"*21000, "C"*21000, "ACD"])
	e.posteriors([0], [2])
	e.store_nnz()
	refused(e.posteriors, [0], [1])
	refused(e.store_nnz)
	e.close()
	ref.close()


@pytest.mark.parametrize("route", ["load", "exchange"])
def test_adopted_image(cuda, tables, route):
	"""an all-pairs image adopted through mb200_store_load_allpairs or the in-place exchange: consistency and
	joins work, the guide tree needs the EA vector passed in (the image carries none)"""
	import torch
	from muscle_b200 import dist as mdist
	seqs = seqs_of(6, 43)
	n = len(seqs)
	npairs = n*(n - 1)//2
	ref, ea_ref, tree_ref, join_ref = reference_run(tables, seqs)
	src = fresh(tables, seqs)
	src.posteriors_allpairs()
	po, no, pe, ne = src.store_pack_ptrs()
	dev = torch.device("cuda", 0)
	img_off = mdist.device_view(po, no*4, dev).view(torch.int32).clone()
	img_ent = mdist.device_view(pe, ne*8, dev).view(torch.int64).clone()
	src.close()
	e = fresh(tables, seqs)
	if route == "load":
		e.store_load_allpairs(0, npairs, img_off.data_ptr(), img_off.numel(), img_ent.data_ptr(), img_ent.numel())
	else:
		do, de = e.store_exchange_begin(img_off.numel(), img_ent.numel())
		mdist.device_view(do, img_off.numel()*4, dev).view(torch.int32).copy_(img_off)
		mdist.device_view(de, img_ent.numel()*8, dev).view(torch.int64).copy_(img_ent)
		torch.cuda.synchronize()
		e.store_exchange_commit()
	refused(e.guide_tree)
	same_tree(e.guide_tree(ea_ref), tree_ref)
	e.consistency_iter()
	same_store(e, ref)
	e.msa_reset()
	assert e.msa_join([0], [1], want_path=True) == join_ref
	e.close()
	ref.close()


def test_stale_transposed_values(cuda, tables):
	"""a second posterior stage after a consistency iteration: the next iteration and the join read the new
	store, not the transposed copy of the old one"""
	seqs = seqs_of(9, 47)
	ref, _, _, join_ref = reference_run(tables, seqs)
	e = fresh(tables, seqs)
	e.posteriors_allpairs()
	e.consistency_iter()
	e.posteriors_allpairs()
	e.consistency_iter()
	same_store(e, ref)
	e.msa_reset()
	assert e.msa_join([0], [1], want_path=True) == join_ref
	e.close()
	ref.close()
