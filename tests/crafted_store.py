"""Hand-built posterior stores for the kernels that read the store: the decoding DP (k_densify +
k_aln_wave), BuildPost (k_bp_* and k_bpc_*), the transposed store and the consistency iteration
(k_mask_fill + k_relax).

Posterior-built stores all look alike (about 7 entries per row within about 55 columns, values in
[0.01, 1], no exact ties).  The patterns here reach the shapes those never have:

  band       diagonal band of random width, random values
  scatter    k random columns per row
  span       few entries per row, far apart, always including column 0 and column LY-1
  full_rows  a band, plus some rows that hold every column
  empty      about half the pairs hold no entry at all; in the others empty rows are interleaved
  ties       a band plus scattered entries, values from {0.25, 0.5, 1} or one constant
  heavy      a band with values up to about 1e6 (BuildPost magnitudes: DP sums pass 2**24)

A store is a list of (offsets, entries) per all-pairs index (x < y, row-major), in the MySparseMx
layout: offsets[LX+1] from 0, entries ENTRY with columns ascending inside each row.  Nothing here
computes a posterior; the sequences only give the lengths."""
import numpy as np

ENTRY = np.dtype([("p", "<f4"), ("col", "<u4")])
PATTERNS = ("band", "scatter", "span", "full_rows", "empty", "ties", "heavy")
AMINO = "ACDEFGHIKLMNPQRSTVWY"


def pair_list(n):
	return [(i, j) for i in range(n) for j in range(i + 1, n)]


def pair_index(n, x, y):
	return x*n - x*(x + 1)//2 + (y - x - 1)


def _band(rng, LX, LY):
	"""columns of a diagonal band of random half-width 0..5, one array per row"""
	half = int(rng.integers(0, 6))
	c = np.arange(LX)*LY//LX + rng.integers(-1, 2, size=LX)
	grid = c[:, None] + np.arange(-half, half + 1)[None, :]
	ok = (grid >= 0) & (grid < LY)
	return [g[m] for g, m in zip(grid, ok)]


def _rows(rng, LX, LY, pattern):
	"""-> list of LX column arrays (ascending, unique, < LY)"""
	if pattern in ("band", "heavy", "full_rows", "empty"):
		rows = _band(rng, LX, LY)
	elif pattern == "scatter":
		rows = [np.sort(rng.choice(LY, size=int(rng.integers(0, min(LY, 20) + 1)), replace=False)) for _ in range(LX)]
	elif pattern == "span":
		rows = [np.unique(np.concatenate([[0, LY - 1], rng.integers(0, LY, size=int(rng.integers(0, 4)))])) for _ in range(LX)]
	elif pattern == "ties":
		rows = [np.unique(np.concatenate([b, rng.integers(0, LY, size=int(rng.integers(0, 4)))])) for b in _band(rng, LX, LY)]
	else:
		raise ValueError(pattern)
	rows = [np.asarray(r, np.int64) for r in rows]
	if pattern == "full_rows":
		# a quarter of the rows, at most ~40 000 entries in full rows per pair
		for i in rng.choice(LX, size=max(1, min(LX//4, 40000//LY)), replace=False):
			rows[i] = np.arange(LY)
	if pattern == "empty":
		if rng.random() < 0.5:
			rows = [np.zeros(0, np.int64) for _ in range(LX)]
		else:
			run = int(rng.integers(1, 5))
			rows = [r if (i//run) % 2 else np.zeros(0, np.int64) for i, r in enumerate(rows)]
	return rows


def _values(rng, n, pattern):
	if pattern == "ties":
		if rng.random() < 0.5:
			return np.float32(rng.choice([0.25, 0.5, 1.0])) + np.zeros(n, np.float32)
		return rng.choice(np.array([0.25, 0.5, 1.0], np.float32), size=n)
	if pattern == "heavy":
		return (10.0**rng.uniform(-2.0, 6.0, size=n)).astype(np.float32)
	return rng.uniform(0.01, 1.0, size=n).astype(np.float32)


def make_pair(rng, LX, LY, pattern):
	"""one stored pair of LX rows over LY columns -> (offsets, entries)"""
	rows = _rows(rng, LX, LY, pattern)
	off = np.zeros(LX + 1, np.uint32)
	off[1:] = np.cumsum([len(r) for r in rows])
	ent = np.empty(int(off[-1]), ENTRY)
	ent["col"] = np.concatenate(rows) if LX > 0 and off[-1] > 0 else np.zeros(0, np.uint32)
	ent["p"] = _values(rng, len(ent), pattern)
	check_pair(off, ent, LX, LY)
	return off, ent


def check_pair(off, ent, LX, LY):
	"""the MySparseMx invariants every consumer relies on"""
	assert len(off) == LX + 1 and off[0] == 0 and off[-1] == len(ent)
	assert (np.diff(off.astype(np.int64)) >= 0).all()
	cols = ent["col"].astype(np.int64)
	assert (cols < LY).all()
	row = np.repeat(np.arange(LX), np.diff(off.astype(np.int64)))
	same = row[1:] == row[:-1]
	assert (np.diff(cols)[same] > 0).all(), "columns must ascend within each row"


def make_store(lens, pattern, seed):
	"""-> (offsets list, entries list) over all pairs of the lengths.  pattern: one name for every pair,
	a list with one name per pair, or "mixed" (every pair draws its own)"""
	rng = np.random.default_rng(seed)
	pairs = pair_list(len(lens))
	if isinstance(pattern, str):
		pats = [PATTERNS[int(rng.integers(0, len(PATTERNS)))] if pattern == "mixed" else pattern for _ in pairs]
	else:
		pats = list(pattern)
	assert len(pats) == len(pairs)
	offs, ents = [], []
	for (x, y), pat in zip(pairs, pats):
		o, e = make_pair(rng, int(lens[x]), int(lens[y]), pat)
		offs.append(o)
		ents.append(e)
	return offs, ents


def seqs_of(lens, seed=0):
	"""protein strings of the given lengths (their content does not matter to a loaded store)"""
	rng = np.random.default_rng(seed)
	return ["".join(rng.choice(list(AMINO), size=int(L))) for L in lens]


def load(engine, lens, store):
	"""set_seqs with strings of the given lengths, then store_load_allpairs of the packed all-pairs image"""
	import torch
	offs, ents = store
	engine.set_seqs(seqs_of(lens))
	npairs = len(offs)
	assert npairs == len(lens)*(len(lens) - 1)//2
	off = np.concatenate([np.asarray(o, np.uint32) for o in offs])
	ent = np.concatenate([np.asarray(e, ENTRY) for e in ents])
	d_off = torch.from_numpy(off.view(np.int32).copy()).cuda()
	n_ent = len(ent)
	raw = ent.view(np.int64) if n_ent else np.zeros(1, np.int64)     # a 1-entry dummy when the store is empty
	d_ent = torch.from_numpy(raw.copy()).cuda()
	engine.store_load_allpairs(0, npairs, d_off.data_ptr(), d_off.numel(), d_ent.data_ptr(), n_ent)
	torch.cuda.synchronize()


def to_dense(off, ent, LX, LY):
	d = np.zeros((LX, LY), np.float32)
	rows = np.repeat(np.arange(LX), np.diff(np.asarray(off, np.int64)))
	d[rows, ent["col"].astype(np.int64)] = ent["p"]
	return d


def gapped_map(rng, L, cols):
	"""pos -> col map of an L-residue member in a `cols`-column MSA with gaps at random interior columns"""
	assert 0 < L <= cols
	return np.sort(rng.choice(cols, size=L, replace=False)).astype(np.uint32)


def gapped_row(seq, p2c, cols):
	row = ["-"]*cols
	for ch, c in zip(seq, p2c):
		row[int(c)] = ch
	return "".join(row)
