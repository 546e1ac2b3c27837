"""Test helper: repeat-rich protein sequences, whose posterior rows are dense.

Tandem repeats and low-complexity regions (polyQ, collagen PPG, SG repeats, Ala runs) align to themselves
at many shifts, so a posterior row of a repeat pair holds up to 83 entries >= 0.01 instead of the ~7 of a
synth.make_family pair.  These inputs reach the code paths that only dense rows or many dense pairs take:
survivor lists longer than 32 in k_posterior_sm, more than one 32-entry group per row in its compaction,
more than one entry sweep in k_relax and BuildPost rows longer than the staged 16.  Plain Python and NumPy,
deterministic in the seed."""
import numpy as np
from muscle_b200 import synth

MOTIFS = ["QQQP", "PPG", "SG", "QQQQQQQP", "AAAAAG"]


def tandem(motif, length, phase=0):
	"""length residues of motif repeated, starting at offset phase into the motif"""
	k = (length + phase)//len(motif) + 1
	return (motif*k)[phase:phase + length]


def mutate(rng, s, rate):
	"""substitute each residue with probability rate by a uniform amino acid"""
	a = np.frombuffer(s.encode(), np.uint8).copy()
	hit = rng.random(len(a)) < rate
	a[hit] = np.frombuffer(synth.AMINO.encode(), np.uint8)[rng.integers(0, 20, int(hit.sum()))]
	return a.tobytes().decode()


# (X, Y): period-shifted repeats of one motif, and Ala homopolymers whose posteriors sit near 0.01
DENSE_PAIRS = [
	(tandem("QQQP", 60, 1), tandem("QQQP", 400)),
	(tandem("QQQQQQQP", 40, 3), tandem("QQQQQQQP", 700)),
	(tandem("SG", 80, 1), tandem("SG", 270)),
	(tandem("PPG", 80, 1), tandem("PPG", 270)),
	(tandem("QQQP", 120, 2), tandem("QQQP", 500)),
	(tandem("AG", 80, 1), tandem("AG", 240)),
	("A"*100, "A"*220),
]


def repeat_family(n, seed, lmin=30, lmax=420, rate=0.03, motifs=MOTIFS):
	"""n mutated tandem repeats: the motifs in turn, lengths in [lmin, lmax], random phase, a substitution
	rate of `rate`"""
	rng = np.random.default_rng(seed)
	out = []
	for k in range(n):
		motif = motifs[k % len(motifs)]
		L = int(rng.integers(lmin, lmax + 1))
		out.append(mutate(rng, tandem(motif, L, int(rng.integers(0, len(motif)))), rate))
	return out


REPEAT_SEED = 1
# two groups of repeat_family(12, REPEAT_SEED) for BuildPost, each member shifted right by (3k) % 7 columns
GROUP_A, GROUP_B = [0, 2, 4, 6, 8, 10], [1, 3, 5, 7, 9, 11]


def staggered_rows(seqs, ids):
	"""ungapped rows of the members ids, shifted right by (3k) % 7 and padded to one width -> (rows, p2c)"""
	shift = [(3*k) % 7 for k in range(len(ids))]
	cols = max(len(seqs[i]) + s for i, s in zip(ids, shift))
	rows = ["-"*s + seqs[i] + "-"*(cols - s - len(seqs[i])) for i, s in zip(ids, shift)]
	return rows, [np.arange(len(seqs[i]), dtype=np.uint32) + s for i, s in zip(ids, shift)]


def operand_row_counts(lens, ids_a, ids_b, row_off, entries):
	"""entries per row of every BuildPost operand S[s->t] (s in ids_a, t in ids_b) of an all-pairs store;
	when s > t the operand is the stored pair (t, s) transposed, and its row counts are column counts"""
	n = len(lens)
	out = []
	for s in ids_a:
		for t in ids_b:
			a, b = min(s, t), max(s, t)
			p = a*n - a*(a + 1)//2 + (b - a - 1)
			if s < t:
				out.append(np.diff(np.asarray(row_off[p], np.int64)))
			else:
				out.append(np.bincount(entries[p]["col"].astype(np.int64), minlength=lens[s]))
	return np.concatenate(out)


def repeat_slots(n):
	"""indexes of mixed_family(n) that hold repeat sequences"""
	return sorted({5, 63, 64, n - 1} & set(range(n)))


def mixed_family(n, seed):
	"""n sequences: short synth.make_family proteins, with mutated QQQP repeats of 40, 60, 200 and 260
	residues at repeat_slots(n) (either side of the 64-sequence boundary and the last index); a short
	repeat slides along a long one, so their pair is dense"""
	seqs = synth.make_family(n, 40, 10, seed=seed, min_len=12)
	rng = np.random.default_rng(seed + 1)
	for k, s in enumerate(repeat_slots(n)):
		seqs[s] = mutate(rng, tandem("QQQP", (40, 60, 200, 260)[k], k), 0.03)
	return seqs
