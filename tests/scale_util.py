"""Oracle inputs at full problem size without exporting the whole store.

At C3 (1000 sequences of about 350 residues) the posterior store holds about 1.2e9 entries, and an
export_all image needs about 10 GB of host memory.  An oracle call reads far fewer pairs:

  conspair(x, y)   (x, z) and (z, y) for every z: the pairs that touch x or y
  buildpost(A, B)  the pairs of A x B

star_store and cross_store export only those, one engine.export_pair each with the pair's entry
count from one store_nnz() call, and leave a placeholder in every other slot.  A placeholder is a
valid pair of the slot's LX rows over its LY columns (row i holds column i mod LY, or every column),
with values in [2, 3), which no posterior reaches.  An oracle call that read one would stay in
bounds and return another result; tests/test_scale_util_cpu.py checks that none is read.

The oracle calls take pointer tables built once per store and run on a thread pool: ctypes releases
the GIL, so the C oracle runs on every core.
"""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor
import numpy as np

ENTRY = np.dtype([("p", "<f4"), ("col", "<u4")])


def workers():
	return os.cpu_count() or 1


def pair_index(n, x, y):
	return x*n - x*(x + 1)//2 + (y - x - 1)


def star_pairs(n, seqset):
	"""all-pairs indexes of the pairs that touch a member of seqset, ascending"""
	px, py = np.triu_indices(n, 1)
	s = np.zeros(n, bool)
	s[list(seqset)] = True
	return np.flatnonzero(s[px] | s[py])


def cross_pairs(n, ids_a, ids_b):
	"""all-pairs indexes of the pairs of A x B (A and B disjoint), ascending"""
	a = np.asarray(ids_a, np.int64)[:, None]
	b = np.asarray(ids_b, np.int64)[None, :]
	x, y = np.minimum(a, b).ravel(), np.maximum(a, b).ravel()
	return np.unique(x*n - x*(x + 1)//2 + (y - x - 1))


def _ptr(a):
	return a.__array_interface__["data"][0]


class PairStore:
	"""Offsets and entries of every pair (x < y, row-major), as the oracle takes them: real where set,
	a placeholder elsewhere.  full_rows: placeholders hold every column (small stores only; each slot
	gets its own arrays).  Otherwise row i holds column i mod LY, and the placeholders of one LY are
	views of one array, so a C3 store of placeholders costs a few MB."""

	def __init__(self, lens, full_rows=False):
		self.lens = np.ascontiguousarray(lens, np.uint32)
		n = self.n = len(self.lens)
		px, py = np.triu_indices(n, 1)
		self._px = px
		npairs = len(px)
		lx, ly = self.lens[px].astype(np.int64), self.lens[py].astype(np.int64)
		self.real = np.zeros(npairs, bool)
		self.off_ptr = np.empty(npairs, np.uintp)
		self.ent_ptr = np.empty(npairs, np.uintp)
		self._ph_off, self._ph_ent = [], []
		lmax = int(self.lens.max())
		if full_rows:
			for k in range(npairs):
				off = (np.arange(lx[k] + 1)*ly[k]).astype(np.uint32)
				ent = np.empty(int(lx[k]*ly[k]), ENTRY)
				ent["col"] = np.tile(np.arange(ly[k]), lx[k])
				ent["p"] = 2 + (np.arange(len(ent)) % 101)/np.float32(101)
				self._ph_off.append(off)
				self._ph_ent.append(ent)
		else:
			ar = np.arange(lmax + 1, dtype=np.uint32)
			by_ly = {}
			for L in np.unique(ly).tolist():
				ent = np.empty(lmax, ENTRY)
				i = np.arange(lmax)
				ent["col"] = i % L
				ent["p"] = 2 + ((i*37 + L) % 101)/np.float32(101)
				by_ly[L] = ent
			self._ph_off = [ar[:a + 1] for a in lx.tolist()]
			self._ph_ent = [by_ly[b][:a] for a, b in zip(lx.tolist(), ly.tolist())]
		self.offs = list(self._ph_off)
		self.ents = list(self._ph_ent)
		self.off_ptr[:] = [_ptr(a) for a in self.offs]
		self.ent_ptr[:] = [_ptr(a) for a in self.ents]

	@classmethod
	def full(cls, lens, offs, ents):
		st = cls(lens)
		for k, (o, e) in enumerate(zip(offs, ents)):
			st.set(k, o, e)
		return st

	def set(self, k, off, ent):
		off = np.ascontiguousarray(off, np.uint32)
		ent = np.ascontiguousarray(ent, ENTRY)
		assert len(off) == int(self.lens[self._px[k]]) + 1 and int(off[-1]) == len(ent), k
		self.offs[k], self.ents[k] = off, ent
		self.off_ptr[k], self.ent_ptr[k] = _ptr(off), _ptr(ent)
		self.real[k] = True

	def clear(self, k):
		self.offs[k], self.ents[k] = self._ph_off[k], self._ph_ent[k]
		self.off_ptr[k], self.ent_ptr[k] = _ptr(self.offs[k]), _ptr(self.ents[k])
		self.real[k] = False

	def clear_all(self):
		for k in np.flatnonzero(self.real).tolist():
			self.clear(k)

	def fill(self, engine, ks, nnz):
		"""export pairs ks from the engine's store; nnz: the store_nnz() vector"""
		for k in np.asarray(ks).tolist():
			self.set(k, *engine.export_pair(k, int(nnz[k])))

	def _require(self, ks):
		missing = np.asarray(ks)[~self.real[np.asarray(ks)]]
		assert len(missing) == 0, "the store lacks pairs %r" % missing[:8].tolist()

	def conspair(self, oracle, x, y):
		"""oracle.conspair of (x, y) -> new entries of the pair"""
		self._require(star_pairs(self.n, (x, y)))
		out = np.empty(len(self.ents[pair_index(self.n, x, y)]), ENTRY)
		oracle.lib.mo_conspair(self.n, C.c_void_p(_ptr(self.lens)), int(x), int(y), C.c_void_p(_ptr(self.off_ptr)),
		  C.c_void_p(_ptr(self.ent_ptr)), C.c_void_p(_ptr(out)))
		return out

	def conspair_many(self, oracle, pairs, threads=None):
		with ThreadPoolExecutor(threads or workers()) as ex:
			return list(ex.map(lambda xy: self.conspair(oracle, *xy), pairs))

	def buildpost(self, oracle, ids_a, p2c_a, cols_a, ids_b, p2c_b, cols_b):
		"""oracle.buildpost -> the cols_a x cols_b float32 column posterior"""
		self._require(cross_pairs(self.n, ids_a, ids_b))
		ia = np.ascontiguousarray(ids_a, np.uint32)
		ib = np.ascontiguousarray(ids_b, np.uint32)
		pa = [np.ascontiguousarray(a, np.uint32) for a in p2c_a]
		pb = [np.ascontiguousarray(a, np.uint32) for a in p2c_b]
		pap = np.array([_ptr(a) for a in pa], np.uintp)
		pbp = np.array([_ptr(a) for a in pb], np.uintp)
		post = np.empty((cols_a, cols_b), np.float32)
		oracle.lib.mo_buildpost(self.n, C.c_void_p(_ptr(self.lens)), len(ia), C.c_void_p(_ptr(ia)), C.c_void_p(_ptr(pap)),
		  int(cols_a), len(ib), C.c_void_p(_ptr(ib)), C.c_void_p(_ptr(pbp)), int(cols_b), C.c_void_p(_ptr(self.off_ptr)),
		  C.c_void_p(_ptr(self.ent_ptr)), C.c_void_p(_ptr(post)))
		return post

	def join(self, oracle, ids_a, p2c_a, cols_a, ids_b, p2c_b, cols_b):
		"""BuildPost + CalcAlnFlat of the oracle -> (score, path)"""
		return oracle.calcaln(self.buildpost(oracle, ids_a, p2c_a, cols_a, ids_b, p2c_b, cols_b))


def star_store(engine, lens, seqset, nnz=None, full_rows=False):
	"""the pairs that touch seqset, exported from the engine; placeholders elsewhere"""
	if nnz is None:
		nnz = engine.store_nnz()[0]
	st = PairStore(lens, full_rows)
	st.fill(engine, star_pairs(len(lens), seqset), nnz)
	return st


def cross_store(engine, lens, ids_a, ids_b, nnz=None, store=None):
	"""the pairs of A x B, exported from the engine; placeholders elsewhere.  store: a PairStore of
	these lengths to reuse (whatever it held is dropped first)"""
	if nnz is None:
		nnz = engine.store_nnz()[0]
	if store is None:
		store = PairStore(lens)
	store.clear_all()
	store.fill(engine, cross_pairs(len(lens), ids_a, ids_b), nnz)
	return store
