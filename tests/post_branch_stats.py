"""Analysis helper (not a test): how the posterior survivors of k_posterior_sm's Backward sweep fall on the
warp.  Dense posteriors of random pairs of a synthetic configuration come from the CPU oracle; a cell is a
survivor when its posterior score passes logf(0.01) (p > 0 in the oracle's dense posterior).  The cells are
mapped onto the kernel's Backward layout: C = min(CM, ceil(LY/32)) columns per lane, strips of 32*C
columns, and at step u lane l on row LX-u+nl-1-l, columns l*C .. l*C+C-1 of the strip, highest first.
Printed per warp step (steps with at least one active lane):
  * the share of column iterations in which at least one lane has a survivor: a branch on the survivor
    inside the column loop costs the whole warp in those iterations;
  * survivors per step;
  * the most survivors in one lane: a per-lane loop over the survivors after the column loop runs this
    many times per step.
    python tests/post_branch_stats.py [C3] [npairs] [seed]"""
import os
import sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from conftest import load_tables          # noqa: E402
from oracle import pyoracle               # noqa: E402
from muscle_b200 import synth             # noqa: E402

cfg = sys.argv[1] if len(sys.argv) > 1 else "C3"
npairs = int(sys.argv[2]) if len(sys.argv) > 2 else 40
seed = int(sys.argv[3]) if len(sys.argv) > 3 else 0
CM = 16                                   # the largest size class

seqs = synth.make_config(cfg)
o = pyoracle.Oracle(load_tables())
rng = np.random.default_rng(seed)
iters = iters_hit = steps = 0
per_step, lane_max = [], []
cells = 0
for _ in range(npairs):
	x, y = rng.choice(len(seqs), 2, replace=False)
	H = o.post(seqs[x], seqs[y]) > 0.0
	LX, LY = H.shape
	cells += LX*LY
	C = min(CM, (LY + 31)//32)
	W = 32*C
	for j0 in range(0, LY, W):
		ncol = min(W, LY - j0)
		nl = (ncol + C - 1)//C
		sub = np.zeros((LX, nl*C), bool)
		sub[:, :ncol] = H[:, j0:j0 + ncol]
		sub = sub.reshape(LX, nl, C)
		lanes = np.arange(nl)
		for u in range(LX + nl - 1):
			rows = LX - u + nl - 1 - lanes
			act = (rows >= 1) & (rows <= LX)
			a = np.zeros((nl, C), bool)
			a[act] = sub[rows[act] - 1, lanes[act]]
			# columns past LY are not iterated: the lane that holds column LY stops there
			ncols = np.minimum(C, ncol - lanes*C)
			steps += 1
			iters += int(ncols[act].max())
			iters_hit += int(a.any(axis=0).sum())
			n = a.sum(axis=1)
			per_step.append(int(n.sum()))
			lane_max.append(int(n.max()))
print("config %s, %d random pairs (seed %d), %d cells, %d warp steps" % (cfg, npairs, seed, cells, steps))
print("column iterations with a survivor in some lane   %.1f %%" % (100.0*iters_hit/iters))
print("survivors per step                                %.2f" % np.mean(per_step))
print("most survivors in one lane, per step              %.2f" % np.mean(lane_max))
