"""oracle/pyoracle.py -- TEST INFRASTRUCTURE ONLY.

ctypes bindings for the two CPU checkers:
  * Oracle  : oracle/liboracle.so      (our C restatement, oracle/muscle_oracle.c)
  * Ref     : oracle/_ref/libmuscle_ref.so (the unmodified reference + oracle/ref_probe.cpp)
  * RefMath : oracle/_ref/libref_math.so   (the reference's LOG_ADD and posterior probability, many inputs)
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import
this module.  The product package muscle_b200/ never does.
"""
import ctypes as C
import os
import subprocess
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "liboracle.so")
REF_SO = os.path.join(HERE, "_ref", "libmuscle_ref.so")
REF_CLI = os.path.join(HERE, "_ref", "muscle")
REF_MATH_SO = os.path.join(HERE, "_ref", "libref_math.so")

ENTRY = np.dtype([("p", "<f4"), ("col", "<u4")])

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
f32p = C.POINTER(C.c_float)


def build(ref=True):
	"""make the checkers (oracle always; _ref only when /root/reference is present)."""
	subprocess.run(["make", "-s", "-C", HERE, "oracle"], check=True)
	if ref and os.path.isdir("/root/reference/src"):
		subprocess.run(["make", "-s", "-j8", "-C", HERE, "ref"], check=True)


def _p(a, t):
	return a.ctypes.data_as(t)


class HMM(C.Structure):
	_fields_ = [("start", C.c_float*5), ("trans", C.c_float*25), ("ins", C.c_float*256),
	  ("match", C.c_float*65536), ("min_sparse_score", C.c_float)]


class SeqSet(C.Structure):
	_fields_ = [("n", C.c_uint32), ("seq", C.POINTER(u8p)), ("len", u32p)]


def hmm_from_tables(t):
	"""t: dict with start[5], trans[25], ins[256], match[65536], min_sparse_score."""
	h = HMM()
	C.memmove(h.start, np.ascontiguousarray(t["start"], np.float32).ctypes.data, 20)
	C.memmove(h.trans, np.ascontiguousarray(t["trans"], np.float32).ctypes.data, 100)
	C.memmove(h.ins, np.ascontiguousarray(t["ins"], np.float32).ctypes.data, 1024)
	C.memmove(h.match, np.ascontiguousarray(t["match"], np.float32).ctypes.data, 262144)
	h.min_sparse_score = float(np.float32(t["min_sparse_score"]))
	return h


def _seq(s):
	if isinstance(s, str):
		s = s.encode()
	return np.frombuffer(bytes(s), dtype=np.uint8).copy()


def _bind_sweeps(L, prefix):
	for f, args in (("log_add_n", [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
	  ("log_add_range", [C.c_uint64, C.c_uint32, C.c_float, C.c_int, C.c_void_p]),
	  ("post_prob_n", [C.c_uint64, C.c_void_p, C.c_float, C.c_void_p]),
	  ("post_prob_range", [C.c_uint64, C.c_uint32, C.c_float, C.c_void_p])):
		fn = getattr(L, prefix + f)
		fn.argtypes = args
		fn.restype = None


class _Sweeps:
	"""LOG_ADD and the posterior probability of a score on many inputs (OpenMP): `_sw` is mo_ or ref_"""
	_sw = None

	def _f(self, name):
		return getattr(self.lib, self._sw + name)

	def log_add_n(self, a, b):
		a = np.ascontiguousarray(a, np.float32)
		b = np.ascontiguousarray(b, np.float32)
		assert a.shape == b.shape
		out = np.empty(a.size, np.float32)
		self._f("log_add_n")(a.size, a.ctypes.data, b.ctypes.data, out.ctypes.data)
		return out

	def log_add_range(self, n, first_bits, b, swap=False):
		"""LOG_ADD(a[k], b), or LOG_ADD(b, a[k]) when swap, for the floats a[k] of bits first_bits + k"""
		out = np.empty(n, np.float32)
		self._f("log_add_range")(n, first_bits & 0xffffffff, float(np.float32(b)), int(swap), out.ctypes.data)
		return out

	def post_prob_n(self, s, min_score):
		s = np.ascontiguousarray(s, np.float32)
		out = np.empty(s.size, np.float32)
		self._f("post_prob_n")(s.size, s.ctypes.data, float(np.float32(min_score)), out.ctypes.data)
		return out

	def post_prob_range(self, n, first_bits, min_score):
		out = np.empty(n, np.float32)
		self._f("post_prob_range")(n, first_bits & 0xffffffff, float(np.float32(min_score)), out.ctypes.data)
		return out


def bit_mismatches(got, want, inputs, what, limit=16):
	"""None when got and want hold the same float32 bits everywhere (never compared as floats: -0.0 == 0.0
	and NaN != NaN); else a message with the count and the first `limit` offending inputs in hex.  inputs: an
	int (element k came from the float of bits inputs + k) or a tuple of float32 arrays (the operands)."""
	g = np.ascontiguousarray(got, np.float32).view(np.uint32)
	w = np.ascontiguousarray(want, np.float32).view(np.uint32)
	assert g.shape == w.shape, (g.shape, w.shape)
	bad = np.flatnonzero(g != w)
	if bad.size == 0:
		return None
	rows = []
	for k in bad[:limit]:
		if isinstance(inputs, (int, np.integer)):
			ops = ["%08x" % ((int(inputs) + int(k)) & 0xffffffff)]
		else:
			ops = ["%08x" % int(np.asarray(x, np.float32).view(np.uint32)[k]) for x in inputs]
		rows.append("(%s) -> %08x, want %08x" % (", ".join(ops), int(g[k]), int(w[k])))
	return "%s: %d of %d differ; first: %s" % (what, bad.size, g.size, "; ".join(rows))


class Oracle(_Sweeps):
	_sw = "mo_"

	def __init__(self, tables):
		if not os.path.exists(ORACLE_SO):
			build(ref=False)
		self.lib = L = C.CDLL(ORACLE_SO)
		self.h = hmm_from_tables(tables)
		L.mo_log_add.restype = C.c_float
		L.mo_log_add.argtypes = [C.c_float, C.c_float]
		L.mo_logexp1.restype = C.c_float
		L.mo_logexp1.argtypes = [C.c_float]
		L.mo_total.restype = C.c_float
		L.mo_alnscore.restype = C.c_float
		L.mo_calcaln.restype = C.c_float
		L.mo_sparse_from_post.restype = C.c_uint32
		L.mo_all_pairs.restype = C.c_uint64
		L.mo_free.argtypes = [C.c_void_p]
		_bind_sweeps(L, "mo_")

	def log_add(self, x, y):
		return self.lib.mo_log_add(x, y)

	def fwd(self, X, Y):
		X, Y = _seq(X), _seq(Y)
		out = np.empty((len(X) + 1, len(Y) + 1, 5), np.float32)
		self.lib.mo_fwd(C.byref(self.h), _p(X, u8p), len(X), _p(Y, u8p), len(Y), _p(out, f32p))
		return out

	def bwd(self, X, Y):
		X, Y = _seq(X), _seq(Y)
		out = np.empty((len(X) + 1, len(Y) + 1, 5), np.float32)
		self.lib.mo_bwd(C.byref(self.h), _p(X, u8p), len(X), _p(Y, u8p), len(Y), _p(out, f32p))
		return out

	def total(self, fwd, bwd):
		LX, LY = fwd.shape[0] - 1, fwd.shape[1] - 1
		return float(self.lib.mo_total(_p(fwd, f32p), _p(bwd, f32p), LX, LY))

	def post(self, X, Y):
		X, Y = _seq(X), _seq(Y)
		out = np.empty((len(X), len(Y)), np.float32)
		self.lib.mo_calcpost(C.byref(self.h), _p(X, u8p), len(X), _p(Y, u8p), len(Y), _p(out, f32p))
		return out

	def sparse(self, post):
		post = np.ascontiguousarray(post, np.float32)
		LX, LY = post.shape
		off = np.empty(LX + 1, np.uint32)
		n = self.lib.mo_sparse_from_post(_p(post, f32p), LX, LY, _p(off, u32p), None)
		ent = np.empty(n, ENTRY)
		self.lib.mo_sparse_from_post(_p(post, f32p), LX, LY, _p(off, u32p), C.c_void_p(ent.ctypes.data))
		return off, ent

	def alnscore(self, post):
		post = np.ascontiguousarray(post, np.float32)
		return float(self.lib.mo_alnscore(_p(post, f32p), post.shape[0], post.shape[1]))

	def calcaln(self, post):
		post = np.ascontiguousarray(post, np.float32)
		LX, LY = post.shape
		buf = C.create_string_buffer(LX + LY + 1)
		s = self.lib.mo_calcaln(_p(post, f32p), LX, LY, buf)
		return float(s), buf.value.decode()

	def all_pairs(self, seqs, p_lo=0, p_hi=None, threads=0, want_sparse=True):
		"""-> dict(cells, nnz[pairs], row_off (list per pair), entries (list per pair), ea[N,N])"""
		arrs = [_seq(s) for s in seqs]
		n = len(arrs)
		npairs = n*(n - 1)//2
		if p_hi is None:
			p_hi = npairs
		ptrs = (u8p*n)(*[_p(a, u8p) for a in arrs])
		lens = np.array([len(a) for a in arrs], np.uint32)
		S = SeqSet(n, ptrs, _p(lens, u32p))
		cnt = p_hi - p_lo
		nnz = np.zeros(max(cnt, 1), np.uint64)
		ea = np.zeros((n, n), np.float32)
		ro = u32p()
		en = C.c_void_p()
		cells = self.lib.mo_all_pairs(C.byref(self.h), C.byref(S), p_lo, p_hi, threads,
		  nnz.ctypes.data_as(C.POINTER(C.c_uint64)),
		  C.byref(ro) if want_sparse else None, C.byref(en) if want_sparse else None, _p(ea, f32p))
		res = {"cells": int(cells), "nnz": nnz[:cnt].astype(np.int64), "ea": ea}
		if want_sparse:
			pairs = [(i, j) for i in range(n) for j in range(i + 1, n)][p_lo:p_hi]
			tot_rows = sum(int(lens[i]) + 1 for i, _ in pairs)
			tot_nnz = int(nnz[:cnt].sum())
			ro_np = np.ctypeslib.as_array(ro, shape=(max(tot_rows, 1),)).copy()
			en_np = np.frombuffer((C.c_char*(8*max(tot_nnz, 1))).from_address(en.value), dtype=ENTRY).copy()
			self.lib.mo_free(ro)
			self.lib.mo_free(en)
			offs, ents = [], []
			r = e = 0
			for q, (i, _) in enumerate(pairs):
				L = int(lens[i])
				offs.append(ro_np[r:r + L + 1])
				ents.append(en_np[e:e + int(nnz[q])])
				r += L + 1
				e += int(nnz[q])
			res["row_off"] = offs
			res["entries"] = ents
		return res

	def upgma(self, n, ea, linkage=4):
		"""-> (left[n-1], right[n-1], left_len, right_len); ea: N(N-1)/2 EA values, row-major i<j"""
		ea = np.ascontiguousarray(ea, np.float32)
		L, R = np.empty(n - 1, np.uint32), np.empty(n - 1, np.uint32)
		LL, RL = np.empty(n - 1, np.float32), np.empty(n - 1, np.float32)
		rc = self.lib.mo_upgma(n, _p(ea, f32p), linkage, _p(L, u32p), _p(R, u32p), _p(LL, f32p), _p(RL, f32p))
		assert rc == 0, "EA outside [0,1]"
		return L, R, LL, RL

	def conspair(self, lens, x, y, row_off, entries):
		"""row_off/entries: lists indexed by pair index (all pairs). -> updated entries of pair (x,y)"""
		n = len(lens)
		npairs = n*(n - 1)//2
		lens = np.ascontiguousarray(lens, np.uint32)
		ro = [np.ascontiguousarray(a, np.uint32) for a in row_off]
		en = [np.ascontiguousarray(a, ENTRY) for a in entries]
		rop = (u32p*npairs)(*[_p(a, u32p) for a in ro])
		enp = (C.c_void_p*npairs)(*[a.ctypes.data for a in en])
		p = x*n - x*(x + 1)//2 + (y - x - 1)
		out = np.empty(len(en[p]), ENTRY)
		self.lib.mo_conspair(n, _p(lens, u32p), x, y, rop, enp, C.c_void_p(out.ctypes.data))
		return out

	def conspair_many(self, lens, pairs, row_off, entries):
		"""conspair of every (x, y) in pairs, with the per-pair pointer arrays built once -> list of entries"""
		n = len(lens)
		npairs = n*(n - 1)//2
		lens = np.ascontiguousarray(lens, np.uint32)
		ro = [np.ascontiguousarray(a, np.uint32) for a in row_off]
		en = [np.ascontiguousarray(a, ENTRY) for a in entries]
		rop = (u32p*npairs)(*[_p(a, u32p) for a in ro])
		enp = (C.c_void_p*npairs)(*[a.ctypes.data for a in en])
		outs = []
		for x, y in pairs:
			p = x*n - x*(x + 1)//2 + (y - x - 1)
			out = np.empty(len(en[p]), ENTRY)
			self.lib.mo_conspair(n, _p(lens, u32p), x, y, rop, enp, C.c_void_p(out.ctypes.data))
			outs.append(out)
		return outs

	def buildpost(self, lens, ids_a, p2c_a, cols_a, ids_b, p2c_b, cols_b, row_off, entries):
		n = len(lens)
		npairs = n*(n - 1)//2
		lens = np.ascontiguousarray(lens, np.uint32)
		ro = [np.ascontiguousarray(a, np.uint32) for a in row_off]
		en = [np.ascontiguousarray(a, ENTRY) for a in entries]
		rop = (u32p*npairs)(*[_p(a, u32p) for a in ro])
		enp = (C.c_void_p*npairs)(*[a.ctypes.data for a in en])
		ia = np.ascontiguousarray(ids_a, np.uint32)
		ib = np.ascontiguousarray(ids_b, np.uint32)
		pa = [np.ascontiguousarray(a, np.uint32) for a in p2c_a]
		pb = [np.ascontiguousarray(a, np.uint32) for a in p2c_b]
		pap = (u32p*len(pa))(*[_p(a, u32p) for a in pa])
		pbp = (u32p*len(pb))(*[_p(a, u32p) for a in pb])
		post = np.empty((cols_a, cols_b), np.float32)
		self.lib.mo_buildpost(n, _p(lens, u32p), len(ia), _p(ia, u32p), pap, cols_a,
		  len(ib), _p(ib, u32p), pbp, cols_b, rop, enp, _p(post, f32p))
		return post


class Ref:
	"""The compiled, unmodified reference (strict-IEEE build)."""

	def __init__(self, nucleo=False, threads=0):
		if not os.path.exists(REF_SO):
			raise FileNotFoundError(REF_SO + " (run `make -C oracle ref` where /root/reference exists)")
		self.lib = L = C.CDLL(REF_SO)
		L.ref_init(int(nucleo), int(threads))
		L.ref_total.restype = C.c_float
		L.ref_alnscore.restype = C.c_float
		L.ref_calcaln.restype = C.c_float
		L.ref_min_sparse_score.restype = C.c_float
		L.ref_mpc_create.restype = C.c_void_p
		L.ref_mpc_posteriors.restype = C.c_double
		L.ref_mpc_posteriors_range.restype = C.c_double
		L.ref_mpc_consiter.restype = C.c_double
		L.ref_mpc_conspairs_range.restype = C.c_double
		L.ref_mpc_alignalns.restype = C.c_float
		for f in ("ref_mpc_destroy", "ref_mpc_paircount", "ref_mpc_posteriors", "ref_mpc_posteriors_range",
		  "ref_mpc_pair_nnz", "ref_mpc_export", "ref_mpc_import", "ref_mpc_get_distmx", "ref_mpc_set_distmx",
		  "ref_mpc_consiter", "ref_mpc_conspairs_range", "ref_mpc_finish", "ref_mpc_alignalns"):
			getattr(L, f).argtypes = None
		self.threads = L.ref_threads()

	def tables(self):
		t = {"start": np.empty(5, np.float32), "trans": np.empty(25, np.float32),
		  "ins": np.empty(256, np.float32), "match": np.empty(65536, np.float32)}
		self.lib.ref_get_hmm(_p(t["start"], f32p), _p(t["trans"], f32p), _p(t["ins"], f32p), _p(t["match"], f32p))
		t["min_sparse_score"] = np.float32(self.lib.ref_min_sparse_score())
		return t

	def fwd(self, X, Y):
		X, Y = _seq(X), _seq(Y)
		out = np.empty((len(X) + 1, len(Y) + 1, 5), np.float32)
		self.lib.ref_fwd(_p(X, u8p), len(X), _p(Y, u8p), len(Y), _p(out, f32p))
		return out

	def bwd(self, X, Y):
		X, Y = _seq(X), _seq(Y)
		out = np.empty((len(X) + 1, len(Y) + 1, 5), np.float32)
		self.lib.ref_bwd(_p(X, u8p), len(X), _p(Y, u8p), len(Y), _p(out, f32p))
		return out

	def total(self, fwd, bwd):
		return float(self.lib.ref_total(_p(fwd, f32p), _p(bwd, f32p), fwd.shape[0] - 1, fwd.shape[1] - 1))

	def post(self, X, Y):
		X, Y = _seq(X), _seq(Y)
		out = np.empty((len(X), len(Y)), np.float32)
		self.lib.ref_calcpost(_p(X, u8p), len(X), _p(Y, u8p), len(Y), _p(out, f32p))
		return out

	def sparse(self, post):
		post = np.ascontiguousarray(post, np.float32)
		LX, LY = post.shape
		off = np.empty(LX + 1, np.uint32)
		ent = np.empty(LX*LY, ENTRY)
		n = self.lib.ref_frompost(_p(post, f32p), LX, LY, _p(off, u32p), C.c_void_p(ent.ctypes.data), LX*LY)
		return off, ent[:n].copy()

	def alnscore(self, post):
		post = np.ascontiguousarray(post, np.float32)
		return float(self.lib.ref_alnscore(_p(post, f32p), post.shape[0], post.shape[1]))

	def calcaln(self, post):
		post = np.ascontiguousarray(post, np.float32)
		LX, LY = post.shape
		buf = C.create_string_buffer(LX + LY + 1)
		s = self.lib.ref_calcaln(_p(post, f32p), LX, LY, buf)
		return float(s), buf.value.decode()

	def upgma(self, n, ea, linkage=4):
		ea = np.ascontiguousarray(ea, np.float32)
		L, R = np.empty(n - 1, np.uint32), np.empty(n - 1, np.uint32)
		LL, RL = np.empty(n - 1, np.float32), np.empty(n - 1, np.float32)
		self.lib.ref_upgma(n, _p(ea, f32p), linkage, _p(L, u32p), _p(R, u32p), _p(LL, f32p), _p(RL, f32p))
		return L, R, LL, RL

	def mpc(self, seqs):
		return RefMPC(self, seqs)


class RefMath(_Sweeps):
	"""The reference's own LOG_ADD and posterior probability on many inputs (oracle/ref_math_probe.cpp)"""
	_sw = "ref_"

	def __init__(self):
		if not os.path.exists(REF_MATH_SO):
			raise FileNotFoundError(REF_MATH_SO + " (run `make -C oracle ref` where /root/reference exists)")
		self.lib = C.CDLL(REF_MATH_SO)
		_bind_sweeps(self.lib, "ref_")


class RefMPC:
	"""Handle on a reference MPCFlat object (state of mpcflat.h:19-49)."""

	def __init__(self, ref, seqs):
		self.ref = ref
		self.lib = ref.lib
		self.seqs = [s if isinstance(s, bytes) else s.encode() for s in seqs]
		self.n = len(seqs)
		self.lens = [len(s) for s in self.seqs]
		arr = (C.c_char_p*self.n)(*self.seqs)
		self.h = C.c_void_p(self.lib.ref_mpc_create(self.n, arr))
		self.pairs = [(i, j) for i in range(self.n) for j in range(i + 1, self.n)]

	def close(self):
		if self.h:
			self.lib.ref_mpc_destroy(self.h)
			self.h = None

	def posteriors(self, threads=0):
		return float(self.lib.ref_mpc_posteriors(self.h, threads))

	def posteriors_range(self, lo, hi, threads=0):
		return float(self.lib.ref_mpc_posteriors_range(self.h, lo, hi, threads))

	def export(self, p):
		LX = self.lens[self.pairs[p][0]]
		n = self.lib.ref_mpc_pair_nnz(self.h, p)
		off = np.empty(LX + 1, np.uint32)
		ent = np.empty(n, ENTRY)
		self.lib.ref_mpc_export(self.h, p, _p(off, u32p), C.c_void_p(ent.ctypes.data))
		return off, ent

	def export_all(self):
		offs, ents = [], []
		for p in range(len(self.pairs)):
			o, e = self.export(p)
			offs.append(o)
			ents.append(e)
		return offs, ents

	def import_(self, p, off, ent):
		off = np.ascontiguousarray(off, np.uint32)
		ent = np.ascontiguousarray(ent, ENTRY)
		self.lib.ref_mpc_import(self.h, p, _p(off, u32p), C.c_void_p(ent.ctypes.data))

	def distmx(self):
		out = np.empty((self.n, self.n), np.float32)
		self.lib.ref_mpc_get_distmx(self.h, _p(out, f32p))
		return out

	def set_distmx(self, m):
		m = np.ascontiguousarray(m, np.float32)
		self.lib.ref_mpc_set_distmx(self.h, _p(m, f32p))

	def consiter(self):
		return float(self.lib.ref_mpc_consiter(self.h))

	def conspairs_range(self, lo, hi, threads=0):
		return float(self.lib.ref_mpc_conspairs_range(self.h, lo, hi, threads))

	def finish(self, consiters=2, refineiters=100):
		cap = self.n*(sum(self.lens) + 8)
		rows = C.create_string_buffer(cap)
		idx = (C.c_int*self.n)()
		cols = self.lib.ref_mpc_finish(self.h, consiters, refineiters, idx, rows, cap)
		out = []
		for i in range(self.n):
			out.append((int(idx[i]), rows.raw[i*(cols + 1):i*(cols + 1) + cols].decode()))
		return out

	def alignalns(self, idx1, rows1, idx2, rows2):
		c1, c2 = len(rows1[0]), len(rows2[0])
		post = np.empty((c1, c2), np.float32)
		path = C.create_string_buffer(c1 + c2 + 1)
		a1 = (C.c_int*len(idx1))(*idx1)
		a2 = (C.c_int*len(idx2))(*idx2)
		r1 = (C.c_char_p*len(rows1))(*[r.encode() for r in rows1])
		r2 = (C.c_char_p*len(rows2))(*[r.encode() for r in rows2])
		s = self.lib.ref_mpc_alignalns(self.h, len(idx1), a1, r1, len(idx2), a2, r2, _p(post, f32p), path)
		return float(s), path.value.decode(), post
