"""ctypes binding of libmuscle_b200.so (the C ABI declared in include/muscle_b200.h).

This is plumbing only: every method is a 1:1 call into the CUDA library.  There is no CPU path;
if the shared library or a CUDA device is missing the constructor raises.
"""
import ctypes as C
import os
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MB200_LIB", os.path.join(HERE, "libmuscle_b200.so"))   # MB200_LIB: tuning builds only

ENTRY = np.dtype([("p", "<f4"), ("col", "<u4")])

EXPORTS = [
	"mb200_create", "mb200_destroy", "mb200_last_error", "mb200_version", "mb200_set_hmm", "mb200_set_seqs",
	"mb200_posteriors", "mb200_posteriors_allpairs", "mb200_store_npairs", "mb200_store_nnz",
	"mb200_export_pair", "mb200_export_all", "mb200_store_pack", "mb200_store_load_allpairs",
	"mb200_store_values", "mb200_store_set_values", "mb200_consistency_iter", "mb200_align_pairs",
	"mb200_align_groups", "mb200_calc_post_dense", "mb200_get_stats", "mb200_residue_classes",
	"mb200_debug_force_c", "mb200_set_nnz_per_row_cap", "mb200_debug_plan", "mb200_calc_post_dense_pair",
	"mb200_store_exchange_begin", "mb200_store_exchange_commit", "mb200_store_entries_ptr", "mb200_store_values_changed",
	"mb200_group_create", "mb200_group_destroy", "mb200_group_last_error", "mb200_group_size", "mb200_group_ctx",
	"mb200_group_set_hmm", "mb200_group_set_seqs", "mb200_group_posteriors_allpairs", "mb200_group_consistency_iter",
	"mb200_group_get_stats", "mb200_msa_reset", "mb200_msa_join", "mb200_msa_export", "mb200_guide_tree", "mb200_set_seqs_mega",
	"mb200_group_set_seqs_mega",
]


class MB200Error(RuntimeError):
	def __init__(self, code, msg):
		super().__init__("libmuscle_b200 error %d: %s" % (code, msg))
		self.code = code


class Stats(C.Structure):
	_fields_ = [("kernel_launches", C.c_uint64), ("cells", C.c_uint64), ("last_kernel_ms", C.c_float),
	  ("last_total_ms", C.c_float), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64)]


class GroupStats(C.Structure):
	_fields_ = [("ndev", C.c_uint32), ("cells", C.c_uint64), ("posterior_ms", C.c_float), ("exchange1_ms", C.c_float),
	  ("exchange1_bytes_per_dev", C.c_uint64), ("relax_ms", C.c_float), ("relax_kernel_ms", C.c_float),
	  ("exchange2_ms", C.c_float), ("exchange2_bytes_per_dev", C.c_uint64)]


_lib = None


def load_library():
	"""dlopen the CUDA library; raises if it was not built (no fallback)."""
	global _lib
	if _lib is None:
		if not os.path.exists(LIB_PATH):
			raise FileNotFoundError("%s not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
			  "(make -C muscle_b200/csrc)" % LIB_PATH)
		L = C.CDLL(LIB_PATH)
		L.mb200_last_error.restype = C.c_char_p
		L.mb200_last_error.argtypes = [C.c_void_p]
		L.mb200_version.restype = C.c_char_p
		L.mb200_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
		L.mb200_destroy.argtypes = [C.c_void_p]
		L.mb200_destroy.restype = None
		L.mb200_group_last_error.restype = C.c_char_p
		L.mb200_group_last_error.argtypes = [C.c_void_p]
		L.mb200_group_ctx.restype = C.c_void_p
		L.mb200_group_ctx.argtypes = [C.c_void_p, C.c_int]
		L.mb200_group_destroy.argtypes = [C.c_void_p]
		L.mb200_group_destroy.restype = None
		L.mb200_group_size.argtypes = [C.c_void_p]
		_lib = L
	return _lib


def _ptr(a):
	return C.c_void_p(a.ctypes.data) if a is not None else None


class Engine:
	"""One context on one CUDA device (mb200_create .. mb200_destroy)."""

	def __init__(self, device=0, _borrowed=None):
		self.lib = load_library()
		self._owned = _borrowed is None
		if _borrowed is not None:
			self.h = C.c_void_p(_borrowed)       # a context owned by a Group
		else:
			h = C.c_void_p()
			rc = self.lib.mb200_create(int(device), C.byref(h))
			if rc != 0:
				raise MB200Error(rc, self.lib.mb200_last_error(None).decode())
			self.h = h
		self.lens = None
		self.nseq = 0

	def close(self):
		if getattr(self, "h", None):
			if self._owned:
				self.lib.mb200_destroy(self.h)
			self.h = None

	def __del__(self):
		try:
			self.close()
		except Exception:
			pass

	def _ck(self, rc):
		if rc != 0:
			raise MB200Error(rc, self.lib.mb200_last_error(self.h).decode())

	# ---- inputs
	def set_hmm(self, tables):
		s = np.ascontiguousarray(tables["start"], np.float32)
		t = np.ascontiguousarray(tables["trans"], np.float32).reshape(-1)
		i = np.ascontiguousarray(tables["ins"], np.float32)
		m = np.ascontiguousarray(tables["match"], np.float32).reshape(-1)
		assert s.size == 5 and t.size == 25 and i.size == 256 and m.size == 65536
		self._ck(self.lib.mb200_set_hmm(self.h, _ptr(s), _ptr(t), _ptr(i), _ptr(m),
		  C.c_float(float(np.float32(tables["min_sparse_score"])))))

	def set_seqs(self, seqs):
		bs = [s if isinstance(s, (bytes, bytearray)) else s.encode() for s in seqs]
		self.lens = np.array([len(b) for b in bs], np.int64)
		off = np.zeros(len(bs) + 1, np.uint64)
		off[1:] = np.cumsum(self.lens)
		buf = np.frombuffer(b"".join(bs), dtype=np.uint8)
		self.nseq = len(bs)
		self._ck(self.lib.mb200_set_seqs(self.h, C.c_uint32(len(bs)), _ptr(buf), _ptr(off)))

	def set_seqs_mega(self, model, profiles):
		"""Mega feature profiles: model = dict(alpha[F], weights[F], logprobs, logprobmx), profiles = list of
		uint8 arrays [L][F] (Mega::m_Profiles)"""
		F = len(model["alpha"])
		alpha = np.ascontiguousarray(model["alpha"], np.uint32)
		w = np.ascontiguousarray(model["weights"], np.float32)
		lp = np.ascontiguousarray(model["logprobs"], np.float32)
		lpm = np.ascontiguousarray(model["logprobmx"], np.float32)
		self.lens = np.array([len(p) for p in profiles], np.int64)
		off = np.zeros(len(profiles) + 1, np.uint64)
		off[1:] = np.cumsum(self.lens)
		let = np.ascontiguousarray(np.concatenate([np.asarray(p, np.uint8).reshape(-1, F) for p in profiles]), np.uint8)
		self.nseq = len(profiles)
		self._ck(self.lib.mb200_set_seqs_mega(self.h, C.c_uint32(self.nseq), _ptr(let), _ptr(off), C.c_uint32(F), _ptr(alpha),
		  _ptr(w), _ptr(lp), _ptr(lpm)))

	# ---- posterior stage
	def posteriors(self, pair_x, pair_y, want_ea=True, force_c=0):
		px = np.ascontiguousarray(pair_x, np.uint32)
		py = np.ascontiguousarray(pair_y, np.uint32)
		ea = np.empty(len(px), np.float32) if want_ea else None
		self._ck(self.lib.mb200_posteriors(self.h, C.c_uint32(len(px)), _ptr(px), _ptr(py),
		  C.c_uint32((force_c & 0xff) << 8), _ptr(ea)))
		self._pairs = (px, py)
		return ea

	def posteriors_allpairs(self, p_lo=0, p_hi=None, want_ea=True):
		n = self.nseq
		if p_hi is None:
			p_hi = n*(n - 1)//2
		ea = np.empty(p_hi - p_lo, np.float32) if want_ea else None
		self._ck(self.lib.mb200_posteriors_allpairs(self.h, C.c_uint32(p_lo), C.c_uint32(p_hi), _ptr(ea)))
		px, py = np.triu_indices(n, 1)
		self._pairs = (px[p_lo:p_hi].astype(np.uint32), py[p_lo:p_hi].astype(np.uint32))
		return ea

	def store_nnz(self):
		np_ = C.c_uint32()
		self._ck(self.lib.mb200_store_npairs(self.h, C.byref(np_)))
		nnz = np.empty(np_.value, np.uint32)
		tot = C.c_uint64()
		self._ck(self.lib.mb200_store_nnz(self.h, _ptr(nnz), C.byref(tot)))
		return nnz, tot.value

	def export_pair(self, k, nnz=None):
		if nnz is None:
			nnz = int(self.store_nnz()[0][k])
		LX = int(self.lens[self._pairs[0][k]])
		off = np.empty(LX + 1, np.uint32)
		ent = np.empty(nnz, ENTRY)
		self._ck(self.lib.mb200_export_pair(self.h, C.c_uint32(k), _ptr(off), _ptr(ent)))
		return off, ent

	def export_all(self):
		nnz, tot = self.store_nnz()
		rows = int(sum(int(self.lens[x]) + 1 for x in self._pairs[0]))
		off = np.empty(rows, np.uint32)
		ent = np.empty(tot, ENTRY)
		self._ck(self.lib.mb200_export_all(self.h, _ptr(off), _ptr(ent)))
		offs, ents = [], []
		r = e = 0
		for k, x in enumerate(self._pairs[0]):
			L = int(self.lens[x])
			offs.append(off[r:r + L + 1])
			ents.append(ent[e:e + int(nnz[k])])
			r += L + 1
			e += int(nnz[k])
		return offs, ents

	def calc_post_dense(self, x, y, force_c=0):
		return self.calc_post_dense_pair([x], [y], 0, force_c)

	def calc_post_dense_pair(self, pair_x, pair_y, which, force_c=0):
		"""dense (post, Forward-M, Backward-M, total) of store pair `which`, run inside the whole list"""
		px = np.ascontiguousarray(pair_x, np.uint32)
		py = np.ascontiguousarray(pair_y, np.uint32)
		LX, LY = int(self.lens[px[which]]), int(self.lens[py[which]])
		post = np.empty((LX, LY), np.float32)
		fwd = np.empty((LX, LY), np.float32)
		bwd = np.empty((LX, LY), np.float32)
		tot = C.c_float()
		self._ck(self.lib.mb200_debug_force_c(self.h, int(force_c)))
		try:
			self._ck(self.lib.mb200_calc_post_dense_pair(self.h, C.c_uint32(len(px)), _ptr(px), _ptr(py),
			  C.c_uint32(which), _ptr(post), _ptr(fwd), _ptr(bwd), C.byref(tot)))
		finally:
			self.lib.mb200_debug_force_c(self.h, 0)
		self._pairs = (px, py)
		return post, fwd, bwd, tot.value

	def debug_plan(self):
		"""the plan of the last posterior call: dict(order, chain, bin_start, chain_rows, chain_pairs)"""
		npairs, nchains = C.c_uint32(), C.c_uint32()
		self._ck(self.lib.mb200_debug_plan(self.h, C.byref(npairs), C.byref(nchains), None, None, None, None))
		order = np.empty(npairs.value, np.uint32)
		chain = np.empty(nchains.value + 1, np.uint32)
		bin_start = np.empty(18, np.uint32)
		limits = np.empty(2, np.uint32)
		self._ck(self.lib.mb200_debug_plan(self.h, C.byref(npairs), C.byref(nchains), _ptr(order), _ptr(chain),
		  _ptr(bin_start), _ptr(limits)))
		return {"order": order, "chain": chain, "bin_start": bin_start, "chain_rows": int(limits[0]),
		  "chain_pairs": int(limits[1])}

	def set_nnz_per_row_cap(self, cap):
		self._ck(self.lib.mb200_set_nnz_per_row_cap(self.h, C.c_uint32(cap)))

	# ---- consistency
	def consistency_iter(self, p_lo=0, p_hi=None):
		if p_hi is None:
			p_hi = self.nseq*(self.nseq - 1)//2
		self._ck(self.lib.mb200_consistency_iter(self.h, C.c_uint32(p_lo), C.c_uint32(p_hi)))

	def store_values_torch(self):
		"""values-only image of the packed store as a CUDA torch tensor (exchange between iterations)"""
		import torch
		_, tot = self.store_nnz()
		# packing may change the layout: ask for the packed image first
		self._ck(self.lib.mb200_store_pack(self.h, None, None, None, None))
		v = torch.empty(int(tot), dtype=torch.float32, device="cuda")
		self._ck(self.lib.mb200_store_values(self.h, C.c_void_p(v.data_ptr()), C.c_uint64(int(tot))))
		return v

	def store_set_values_torch(self, v, first_entry):
		self._ck(self.lib.mb200_store_set_values(self.h, C.c_void_p(v.data_ptr()), C.c_uint64(int(first_entry)),
		  C.c_uint64(int(v.numel()))))

	def store_pack_ptrs(self):
		"""(d_offsets ptr, n_offsets, d_entries ptr, n_entries) of the packed store"""
		po, pe = C.c_void_p(), C.c_void_p()
		no, ne = C.c_uint64(), C.c_uint64()
		self._ck(self.lib.mb200_store_pack(self.h, C.byref(po), C.byref(no), C.byref(pe), C.byref(ne)))
		return po.value, no.value, pe.value, ne.value

	def store_load_allpairs(self, p_lo, p_hi, d_offsets_ptr, n_offsets, d_entries_ptr, n_entries):
		self._ck(self.lib.mb200_store_load_allpairs(self.h, C.c_uint32(p_lo), C.c_uint32(p_hi),
		  C.c_void_p(d_offsets_ptr), C.c_uint64(n_offsets), C.c_void_p(d_entries_ptr), C.c_uint64(n_entries)))
		n = self.nseq
		px, py = np.triu_indices(n, 1)
		self._pairs = (px[p_lo:p_hi].astype(np.uint32), py[p_lo:p_hi].astype(np.uint32))

	# ---- in-place exchange (multi-GPU)
	def store_exchange_begin(self, n_offsets, n_entries):
		"""-> (device ptr of the offsets image, device ptr of the entries image), library-owned"""
		po, pe = C.c_void_p(), C.c_void_p()
		self._ck(self.lib.mb200_store_exchange_begin(self.h, C.c_uint64(int(n_offsets)), C.c_uint64(int(n_entries)),
		  C.byref(po), C.byref(pe)))
		return po.value, pe.value

	def store_exchange_commit(self):
		self._ck(self.lib.mb200_store_exchange_commit(self.h))
		n = self.nseq
		px, py = np.triu_indices(n, 1)
		self._pairs = (px.astype(np.uint32), py.astype(np.uint32))

	def store_entries_ptr(self):
		pe = C.c_void_p()
		ne = C.c_uint64()
		self._ck(self.lib.mb200_store_entries_ptr(self.h, C.byref(pe), C.byref(ne)))
		return pe.value, ne.value

	def store_values_changed(self):
		self._ck(self.lib.mb200_store_values_changed(self.h))

	# ---- posterior decoding
	def align_pairs(self, store_pairs):
		sp = np.ascontiguousarray(store_pairs, np.uint32)
		lens = [int(self.lens[self._pairs[0][k]]) + int(self.lens[self._pairs[1][k]]) + 1 for k in sp]
		off = np.zeros(len(sp) + 1, np.uint64)
		off[1:] = np.cumsum(lens)
		buf = np.zeros(int(off[-1]), np.uint8)
		scores = np.empty(len(sp), np.float32)
		self._ck(self.lib.mb200_align_pairs(self.h, C.c_uint32(len(sp)), _ptr(sp), _ptr(buf), _ptr(off), _ptr(scores)))
		paths = []
		for k in range(len(sp)):
			raw = buf[int(off[k]):int(off[k + 1])].tobytes()
			paths.append(raw.split(b"\0")[0].decode())
		return scores, paths

	def align_groups(self, ids_a, p2c_a, cols_a, ids_b, p2c_b, cols_b, want_post=False):
		ia = np.ascontiguousarray(ids_a, np.uint32)
		ib = np.ascontiguousarray(ids_b, np.uint32)
		pa = np.ascontiguousarray(np.concatenate([np.asarray(a, np.uint32) for a in p2c_a]), np.uint32)
		pb = np.ascontiguousarray(np.concatenate([np.asarray(a, np.uint32) for a in p2c_b]), np.uint32)
		path = C.create_string_buffer(cols_a + cols_b + 1)
		score = C.c_float()
		post = np.empty((cols_a, cols_b), np.float32) if want_post else None
		self._ck(self.lib.mb200_align_groups(self.h, C.c_uint32(len(ia)), _ptr(ia), _ptr(pa), C.c_uint32(cols_a),
		  C.c_uint32(len(ib)), _ptr(ib), _ptr(pb), C.c_uint32(cols_b), path, C.byref(score), _ptr(post)))
		return score.value, path.value.decode(), post

	# ---- device-resident MSAs
	def msa_reset(self):
		self._ck(self.lib.mb200_msa_reset(self.h))

	def msa_join(self, ids_a, ids_b, want_path=False):
		"""-> (columns of the joined MSA, DP score, path or None)"""
		ia = np.ascontiguousarray(ids_a, np.uint32)
		ib = np.ascontiguousarray(ids_b, np.uint32)
		cols = C.c_uint32()
		score = C.c_float()
		cap = int(sum(int(self.lens[i]) for i in list(ia) + list(ib))) + 2 if want_path else 0
		path = C.create_string_buffer(cap) if want_path else None
		self._ck(self.lib.mb200_msa_join(self.h, C.c_uint32(len(ia)), _ptr(ia), C.c_uint32(len(ib)), _ptr(ib),
		  C.byref(cols), C.byref(score), path, C.c_uint32(cap)))
		return cols.value, score.value, (path.value.decode() if want_path else None)

	def msa_export(self, ids):
		"""-> (list of pos->col arrays, list of column counts)"""
		ii = np.ascontiguousarray(ids, np.uint32)
		tot = int(sum(int(self.lens[i]) for i in ii))
		buf = np.empty(tot, np.uint32)
		cols = np.empty(len(ii), np.uint32)
		self._ck(self.lib.mb200_msa_export(self.h, C.c_uint32(len(ii)), _ptr(ii), _ptr(buf), _ptr(cols)))
		out, o = [], 0
		for i in ii:
			L = int(self.lens[i])
			out.append(buf[o:o + L].copy())
			o += L
		return out, cols

	# ---- guide tree
	def guide_tree(self, ea=None, linkage=4):
		"""UPGMA on the device; ea None = the EA vector of the all-pairs store.  -> (left, right, left_len, right_len)"""
		n = self.nseq
		L, R = np.empty(n - 1, np.uint32), np.empty(n - 1, np.uint32)
		LL, RL = np.empty(n - 1, np.float32), np.empty(n - 1, np.float32)
		e = None if ea is None else np.ascontiguousarray(ea, np.float32)
		self._ck(self.lib.mb200_guide_tree(self.h, _ptr(e), C.c_int(linkage), _ptr(L), _ptr(R), _ptr(LL), _ptr(RL)))
		return L, R, LL, RL

	def stats(self):
		s = Stats()
		self._ck(self.lib.mb200_get_stats(self.h, C.byref(s)))
		return {f: getattr(s, f) for f, _ in Stats._fields_}


class Group:
	"""Several GPUs driven by one process (mb200_group_*): what `muscle_b200 -align` uses."""

	def __init__(self, devices=None):
		self.lib = load_library()
		g = C.c_void_p()
		if devices is None:
			rc = self.lib.mb200_group_create(0, None, C.byref(g))
		else:
			arr = (C.c_int*len(devices))(*devices)
			rc = self.lib.mb200_group_create(len(devices), arr, C.byref(g))
		if rc != 0:
			raise MB200Error(rc, self.lib.mb200_group_last_error(None).decode())
		self.g = g
		self.size = int(self.lib.mb200_group_size(g))
		self.nseq = 0
		self.lens = None

	def close(self):
		if getattr(self, "g", None):
			self.lib.mb200_group_destroy(self.g)
			self.g = None

	def __del__(self):
		try:
			self.close()
		except Exception:
			pass

	def _ck(self, rc):
		if rc != 0:
			raise MB200Error(rc, self.lib.mb200_group_last_error(self.g).decode())

	def engine(self, rank=0):
		"""Engine view of one member context (borrowed; rank 0 runs the serial stages)"""
		e = Engine(_borrowed=self.lib.mb200_group_ctx(self.g, int(rank)))
		e.lens, e.nseq = self.lens, self.nseq
		n = self.nseq
		px, py = np.triu_indices(n, 1)
		e._pairs = (px.astype(np.uint32), py.astype(np.uint32))
		return e

	def set_hmm(self, tables):
		s = np.ascontiguousarray(tables["start"], np.float32)
		t = np.ascontiguousarray(tables["trans"], np.float32).reshape(-1)
		i = np.ascontiguousarray(tables["ins"], np.float32)
		m = np.ascontiguousarray(tables["match"], np.float32).reshape(-1)
		self._ck(self.lib.mb200_group_set_hmm(self.g, _ptr(s), _ptr(t), _ptr(i), _ptr(m),
		  C.c_float(float(np.float32(tables["min_sparse_score"])))))

	def set_seqs(self, seqs):
		bs = [s if isinstance(s, (bytes, bytearray)) else s.encode() for s in seqs]
		self.lens = np.array([len(b) for b in bs], np.int64)
		off = np.zeros(len(bs) + 1, np.uint64)
		off[1:] = np.cumsum(self.lens)
		buf = np.frombuffer(b"".join(bs), dtype=np.uint8)
		self.nseq = len(bs)
		self._ck(self.lib.mb200_group_set_seqs(self.g, C.c_uint32(len(bs)), _ptr(buf), _ptr(off)))

	def posteriors_allpairs(self, want_ea=True):
		n = self.nseq
		ea = np.empty(n*(n - 1)//2, np.float32) if want_ea else None
		self._ck(self.lib.mb200_group_posteriors_allpairs(self.g, _ptr(ea)))
		return ea

	def consistency_iter(self):
		self._ck(self.lib.mb200_group_consistency_iter(self.g))

	def stats(self):
		s = GroupStats()
		self._ck(self.lib.mb200_group_get_stats(self.g, C.byref(s)))
		return {f: getattr(s, f) for f, _ in GroupStats._fields_}
