"""GPU, end to end: the reference's own `muscle -align` control flow with libmuscle_b200 as its pair
engine (integration/_build/muscle_b200, built from integration/mpcflat_b200_shim.cpp) against the
MSAs the unmodified CPU reference produced for the same FASTA (tests/golden/e2e/*.ref.afa).

Bar: the identical MSA, row for row.  Every stage of the device path is bit-exact (including expf at the
0.01 cut), so there is no tolerance on aligned pairs any more; on a mismatch the fraction of shared
aligned residue pairs is reported to help debugging."""
import os
import subprocess
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "integration", "_build", "muscle_b200")
E2E = os.path.join(ROOT, "tests", "golden", "e2e")


def read_afa(path):
	rows, name = {}, None
	for line in open(path):
		line = line.strip()
		if line.startswith(">"):
			name = line[1:]
			rows[name] = ""
		elif name is not None:
			rows[name] += line
	return rows


def pair_set(rows):
	"""set of aligned residue pairs ((seqA,posA),(seqB,posB)) -- the Q-score universe"""
	names = sorted(rows)
	cols = len(next(iter(rows.values())))
	pos = {n: -1 for n in names}
	out = set()
	for c in range(cols):
		here = []
		for n in names:
			if rows[n][c] != "-":
				pos[n] += 1
				here.append((n, pos[n]))
		for a in range(len(here)):
			for b in range(a + 1, len(here)):
				out.add((here[a], here[b]))
	return out


@pytest.mark.parametrize("name", ["fam12", "fam30", "fam6_long", "rep16"])
def test_align_cli_matches_reference_msa(name, tmp_path):
	if not os.path.exists(CLI):
		pytest.skip("integration/_build/muscle_b200 not built (needs oracle/_ref built from the reference sources)")
	out = tmp_path / (name + ".afa")
	r = subprocess.run([CLI, "-align", os.path.join(E2E, name + ".fa"), "-output", str(out), "-quiet"],
	  capture_output=True, text=True, timeout=600)
	assert r.returncode == 0, r.stderr[-2000:]
	got, want = read_afa(out), read_afa(os.path.join(E2E, name + ".ref.afa"))
	assert sorted(got) == sorted(want)
	for n in want:
		assert got[n].replace("-", "") == want[n].replace("-", "")
	if got == want:
		return
	a, b = pair_set(got), pair_set(want)
	q = len(a & b)/max(1, len(b))
	assert False, "MSA differs from the reference: shared aligned pairs %.4f" % q


def test_super5_cli_matches_reference_msa(tmp_path):
	"""`-super5` (UClust/EACluster -> AlignPairFlat, per-cluster MPCFlat, CalcEADistMx, PProg joins with
	GetPostPairsAlignedFlat) with every CalcPost caller bound to the GPU engine
	(integration/pairlist_b200_shim.cpp + mpcflat_b200_shim.cpp)."""
	if not os.path.exists(CLI):
		pytest.skip("integration/_build/muscle_b200 not built (needs oracle/_ref built from the reference sources)")
	name = "super5_150"
	out = tmp_path / (name + ".afa")
	# -threads 1 on both sides: the unmodified reference's -super5 is run-to-run non-deterministic
	# with several OpenMP threads (see tests/golden/make_e2e_golden.py)
	r = subprocess.run([CLI, "-super5", os.path.join(E2E, name + ".fa"), "-output", str(out), "-quiet", "-threads", "1"],
	  capture_output=True, text=True, timeout=900)
	assert r.returncode == 0, r.stderr[-2000:]
	got, want = read_afa(out), read_afa(os.path.join(E2E, name + ".ref.afa"))
	assert sorted(got) == sorted(want)
	for n in want:
		assert got[n].replace("-", "") == want[n].replace("-", "")
	if got == want:
		return
	a, b = pair_set(got), pair_set(want)
	q = len(a & b)/max(1, len(b))
	assert False, "super5 MSA differs from the reference: shared aligned pairs %.4f" % q


def test_profalign_cli_matches_reference_msa(tmp_path):
	"""`-profalign` never calls CalcPosteriors: it calls MPCFlat::CalcPosterior per cross pair and then
	AlignAlns (profalign.cpp:28-54).  The binding defers the per-pair calls and runs one device batch."""
	if not os.path.exists(CLI):
		pytest.skip("integration/_build/muscle_b200 not built (needs oracle/_ref built from the reference sources)")
	out = tmp_path / "profalign.afa"
	r = subprocess.run([CLI, "-profalign", os.path.join(E2E, "profalign_a.afa"), "-input2", os.path.join(E2E, "profalign_b.afa"),
	  "-output", str(out), "-quiet"], capture_output=True, text=True, timeout=600)
	assert r.returncode == 0, r.stderr[-2000:]
	assert read_afa(out) == read_afa(os.path.join(E2E, "profalign.ref.afa"))


def test_align_cli_c2_matches_reference_msa(tmp_path):
	"""BASELINE.json config 2 (256 proteins, mean length 250) end to end: posteriors, 2 consistency
	iterations, 255 device joins, 100 refinement joins -- byte-identical to the CPU reference's MSA
	(tests/golden/e2e/c2.ref.afa, ~35 CPU-minutes on 6 threads to produce)."""
	if not os.path.exists(CLI):
		pytest.skip("integration/_build/muscle_b200 not built (needs oracle/_ref built from the reference sources)")
	ref = os.path.join(E2E, "c2.ref.afa")
	if not os.path.exists(ref):
		pytest.skip("c2 golden not generated")
	from muscle_b200 import synth
	fa = tmp_path / "c2.fa"
	with open(fa, "w") as f:
		for i, q in enumerate(synth.make_config("C2")):
			f.write(">s%d\n%s\n" % (i, q))
	out = tmp_path / "c2.afa"
	r = subprocess.run([CLI, "-align", str(fa), "-output", str(out), "-quiet"], capture_output=True, text=True, timeout=900)
	assert r.returncode == 0, r.stderr[-2000:]
	got, want = read_afa(out), read_afa(ref)
	assert got == want


def test_align_cli_mega_matches_reference_msa(tmp_path):
	"""`-align x.mega` (Muscle-3D feature profiles, calcpost.cpp:14-22): the reference's own
	test_data/mega/BB11001.mega through the engine's Mega emission mode"""
	if not os.path.exists(CLI):
		pytest.skip("integration/_build/muscle_b200 not built (needs oracle/_ref built from the reference sources)")
	out = tmp_path / "bb11001.afa"
	r = subprocess.run([CLI, "-align", os.path.join(E2E, "BB11001.mega"), "-output", str(out), "-quiet"],
	  capture_output=True, text=True, timeout=600)
	assert r.returncode == 0, r.stderr[-2000:]
	assert read_afa(out) == read_afa(os.path.join(E2E, "BB11001.mega.ref.afa"))
