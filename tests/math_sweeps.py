"""Input sweeps of k_posterior_sm's two arithmetic primitives, shared by test_logadd_expf_cpu.py (oracle vs
the compiled reference) and test_logadd_expf_gpu.py (device vs oracle).

LOG_ADD(x, y) (scoretype.h:120-124) and its device restatement LogAdd (muscle_b200/csrc/common.cuh):

  With d = larger - smaller (exact in either order under round-to-nearest), both return
  `d >= 7.5 ? larger : LOGEXP1(d) + smaller`, where LOGEXP1 picks one of four cubics by the cut points 1, 2.5
  and 4.5 (closed on the right) and evaluates it in Horner form with a rounding after every operation.
  The reference also returns the larger when the smaller is LOG_ZERO; for finite inputs that only matters
  when the gap is below 7.5, i.e. when both are LOG_ZERO to fp32 precision, where LOGEXP1(0) + LOG_ZERO
  rounds back to LOG_ZERO.

  L1 feeds every float d in [+0, 7.5] against 0 in both orders and both signs.  That evaluates the piece
  selection, the clamp and the Horner cubic on every gap the polynomial can see, and the 7.5 cut at its
  edge, with `+ smaller` adding 0 or -d.  So for finite inputs the device can differ from the reference
  only through the final `q + smaller` at other magnitudes of the smaller operand and through the two
  selects (which operand is the larger, the >= 7.5 cut on gaps above 7.5): L2 covers the gaps above 7.5 up
  to FLT_MAX and the neighbourhoods of every cut point, L3 the final add with the smaller operand in every
  binade from 2^-24 to LOG_ZERO's, L4 LOG_ZERO, signed zeros and the default transitions pairwise, L5
  random gaps at the scores a DP produces.  NaN and +-inf are outside the DP's domain and not compared.

The probability of a posterior score (calcposteriorflat.cpp:15-20, `Score >= 0 ? 1 : expf(Score)` above
MIN_SPARSE_SCORE) and the kept decision (mysparsemx.cpp:139-141, p >= 0.01f), which k_posterior_sm makes as
a compare of the score: E1 every score in [logf(0.01f), -0.0]; E2 every float in [+0, 1] and in
[-4.7, logf(0.01f)); E3 the E1 range and 1024 floats below it; E4 E1 and E3 under min_sparse_score =
logf(0.001f), below the kept threshold.

A sweep is a list of cases, each ("range", first_bits, n, b, swap) -- operand a the floats of bits
first_bits .. first_bits + n - 1, b a scalar, swap: LOG_ADD(b, a) -- or ("pairs", a, b).  Ranges come in
pieces of at most CHUNK floats; the large sweeps are generators.
"""
import ctypes
import ctypes.util
import numpy as np

CHUNK = 1 << 26
LOG_ZERO = np.float32(-2e20)
KEEP_BITS = 0xc0935d8e                        # logf(0.01f): the least score whose expf is >= 0.01f
FLT_MAX = np.finfo(np.float32).max


def f32(bits):
	return np.asarray(bits, np.uint32).view(np.float32)


def bits(x):
	return int(np.asarray(x, np.float32).view(np.uint32))


def ranges(first, last, b=0.0, swap=False):
	"""("range", ...) cases for every float of bits first .. last (inclusive)"""
	out = []
	for k in range(first, last + 1, CHUNK):
		out.append(("range", k, min(CHUNK, last + 1 - k), np.float32(b), swap))
	return out


def both_orders(a, b):
	a = np.asarray(a, np.float32)
	b = np.broadcast_to(np.asarray(b, np.float32), a.shape)
	return [("pairs", a, np.ascontiguousarray(b)), ("pairs", np.ascontiguousarray(b), a)]


def _ordered(x):
	"""float32 -> an integer key monotone in the float's value (-0.0 just below +0.0)"""
	u = np.asarray(x, np.float32).view(np.uint32).astype(np.int64)
	return np.where(u >= 0x80000000, 0x7fffffff - u, u)


def _unordered(k):
	k = np.asarray(k, np.int64)
	return np.where(k < 0, 0x7fffffff - k, k).astype(np.uint32).view(np.float32)


def floats_between(lo, hi, cap):
	"""the floats in [lo, hi], at an even stride when there are more than cap"""
	a, b = int(_ordered(np.float32(lo))), int(_ordered(np.float32(hi)))
	stride = max(1, -(-(b - a + 1)//cap))
	return _unordered(np.arange(a, b + 1, stride))


def transitions(tables):
	"""the finite default transition scores (start and transition tables, LOG_ZERO entries excluded)"""
	v = np.concatenate([np.asarray(tables["start"], np.float32).ravel(), np.asarray(tables["trans"], np.float32).ravel()])
	return np.unique(v[v > np.float32(-1e19)])


def sweep_l1():
	out = []
	for sign in (0, 0x80000000):
		for swap in (False, True):
			out += ranges(sign, sign + 0x40F00000, 0.0, swap)
	return out


def sweep_l2():
	cuts = [0.5, 1.0, 2.5, 4.5, 4.75, 7.5]
	v = [f32(np.arange(0x40F00000, 0x41800001, dtype=np.uint32))]          # every float in [7.5, 16]
	for c in cuts:
		k = bits(c)
		v.append(f32(np.arange(k - 256, k + 257, dtype=np.uint32)))
	v.append(np.array([2.0**e for e in range(-149, 128)] + [FLT_MAX], np.float32))
	v = np.concatenate(v)
	out = []
	for lo in (np.float32(0.0), np.float32(-3.0)):
		x = (v + lo).astype(np.float32)
		out += both_orders(x, lo)
	return out


def sweep_l3(seed=7, cap=1 << 22):
	rng = np.random.default_rng(seed)
	los = [np.float32(-(1.0 + rng.random())*2.0**e) for e in range(-24, 68)] + [LOG_ZERO]
	for lo in los:
		y = floats_between(np.float32(lo - np.float32(8)), np.float32(lo + np.float32(8)), cap)
		yield from both_orders(y, lo)
	z = np.array([0.0, -0.0], np.float32)
	lo = np.array(los, np.float32)
	a = np.concatenate([np.repeat(z, 2), np.repeat(z, lo.size)])
	b = np.concatenate([np.tile(z, 2), np.tile(lo, 2)])
	yield from both_orders(a, b)


def sweep_l4(tables):
	t = transitions(tables)
	s = np.concatenate([np.array([LOG_ZERO, 2*LOG_ZERO, -FLT_MAX, -1e4, -7.5, -1.0, -0.0, 0.0], np.float32),
	  (LOG_ZERO + t).astype(np.float32), t])
	a, b = np.meshgrid(s, s, indexing="ij")
	return [("pairs", np.ascontiguousarray(a.ravel()), np.ascontiguousarray(b.ravel()))]


def sweep_l5(seed=11, n=1 << 28, piece=1 << 24):
	for k in range(n//piece):
		rng = np.random.default_rng([seed, k])
		x = rng.uniform(-5000.0, 0.0, piece).astype(np.float32)
		h = piece//2
		gap = np.concatenate([rng.uniform(0.0, 8.0, h), np.exp(rng.uniform(np.log(1e-6), np.log(1e6), piece - h))])
		y = (x + gap.astype(np.float32)).astype(np.float32)
		yield ("pairs", x, y) if k % 2 == 0 else ("pairs", y, x)


def libm_logf(x):
	libm = ctypes.CDLL(ctypes.util.find_library("m"))
	libm.logf.restype = ctypes.c_float
	libm.logf.argtypes = [ctypes.c_float]
	return np.float32(libm.logf(ctypes.c_float(x)))


E1 = (0x80000000, KEEP_BITS)                          # [logf(0.01f), -0.0]
E2 = ((0x00000000, 0x3f800000), (KEEP_BITS + 1, bits(np.float32(-4.7))))   # [+0, 1], [-4.7, logf(0.01f))
E3 = (0x80000000, KEEP_BITS + 1024)
