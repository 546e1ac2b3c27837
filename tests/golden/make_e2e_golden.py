"""End-to-end golden MSAs: run the COMPILED, UNMODIFIED reference CLI (oracle/_ref/muscle, strict-IEEE
build) on seeded synthetic FASTA inputs and commit input + output under tests/golden/e2e/.
    python tests/golden/make_e2e_golden.py
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from muscle_b200 import synth   # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "e2e")
CLI = os.path.join(ROOT, "oracle", "_ref", "muscle")

SETS = {
	"fam12": dict(n=12, mean=80, sd=12, seed=101),
	"fam30": dict(n=30, mean=120, sd=25, seed=102, dupes=[(3, 17)]),
	"fam6_long": dict(n=6, mean=600, sd=60, seed=103),
}


def main():
	os.makedirs(OUT, exist_ok=True)
	for name, cfg in SETS.items():
		seqs = synth.make_family(cfg["n"], cfg["mean"], cfg["sd"], cfg["seed"])
		for a, b in cfg.get("dupes", []):
			seqs[b] = seqs[a]                  # exercises Derep / InsertDupes (mpcflat.cpp:290-294,421)
		fa = os.path.join(OUT, name + ".fa")
		with open(fa, "w") as f:
			for i, s in enumerate(seqs):
				f.write(">s%d\n%s\n" % (i, s))
		out = os.path.join(OUT, name + ".ref.afa")
		subprocess.run([CLI, "-align", fa, "-output", out, "-quiet"], check=True)
		print(name, "->", out)


def super5():
	seqs = synth.make_family(150, 90, 15, seed=104, n_sub=12)
	fa = os.path.join(OUT, "super5_150.fa")
	with open(fa, "w") as f:
		for i, s in enumerate(seqs):
			f.write(">s%d\n%s\n" % (i, s))
	# -threads 1: the reference's own -super5 is NOT reproducible with several threads (two runs of the
	# unmodified binary share only ~60 % of their aligned residue pairs: OpenMP-order dependent
	# decisions in EACluster/CalcEADistMx); single-threaded it is deterministic.
	subprocess.run([CLI, "-super5", fa, "-output", os.path.join(OUT, "super5_150.ref.afa"), "-quiet", "-threads", "1"], check=True)


def profalign():
	"""-profalign golden: the two halves of fam12's reference MSA (projected), re-joined by the reference"""
	def read(path):
		rows, name = [], None
		for line in open(path):
			line = line.strip()
			if line.startswith(">"):
				name = line[1:]
				rows.append([name, ""])
			elif name is not None:
				rows[-1][1] += line
		return rows

	def proj(rs):
		cols = len(rs[0][1])
		keep = [c for c in range(cols) if any(r[1][c] != "-" for r in rs)]
		return [(n, "".join(q[c] for c in keep)) for n, q in rs]
	rows = read(os.path.join(OUT, "fam12.ref.afa"))
	for nm, rs in (("profalign_a.afa", proj(rows[:5])), ("profalign_b.afa", proj(rows[5:]))):
		with open(os.path.join(OUT, nm), "w") as f:
			for n, q in rs:
				f.write(">%s\n%s\n" % (n, q))
	subprocess.run([CLI, "-profalign", os.path.join(OUT, "profalign_a.afa"), "-input2", os.path.join(OUT, "profalign_b.afa"),
	  "-output", os.path.join(OUT, "profalign.ref.afa"), "-quiet"], check=True)


def repeats():
	"""rep16: 16 proteins of one family, each with a tandem-repeat region (QQQP, PPG or SG, 20-86 residues,
	3 % substitutions) in its middle, whose posterior rows hold up to 42 entries >= 0.01"""
	sys.path.insert(0, os.path.join(ROOT, "tests"))
	import numpy as np
	import repeat_util as ru
	seqs = synth.make_family(16, 150, 20, seed=105)
	rng = np.random.default_rng(105)
	for k, s in enumerate(seqs):
		rep = ru.mutate(rng, ru.tandem(ru.MOTIFS[k % 3], 20 + (11*k) % 67, k % 4), 0.03)
		seqs[k] = s[:len(s)//2] + rep + s[len(s)//2:]
	fa = os.path.join(OUT, "rep16.fa")
	with open(fa, "w") as f:
		for i, s in enumerate(seqs):
			f.write(">s%d\n%s\n" % (i, s))
	subprocess.run([CLI, "-align", fa, "-output", os.path.join(OUT, "rep16.ref.afa"), "-quiet"], check=True)


if __name__ == "__main__":
	if sys.argv[1:] == ["repeats"]:
		repeats()
		sys.exit()
	super5()
	main()
	profalign()
	repeats()
