"""CPU: the expected accuracy of k_posterior_sm's one-strip path, computed from the candidate entries alone.

CalcAlnScoreFlat (calcalnscoreflat.cpp:4-32) runs a max-sum DP over every cell of the dense posterior.
The kernel instead gives each candidate (i, j) the value V = fl(P + Q), Q being the max of V over the
candidates (i' < i, j' < j) or 0, read from a prefix-max Fenwick tree over the columns that row i queries
before it updates it, and returns the max of all V.  A cell without a candidate adds 0, which changes
nothing, and rounding is monotone, so both give the same float.  Here a numpy model of the kernel's
algorithm (same tree, same order of queries and updates) is compared bit for bit with
a literal float32 transcription of CalcAlnScoreFlat and with the C oracle's, on random sparse matrices
with ties, candidates in the first and last column, empty rows and matrices, and rows of 33-128
candidates."""
import numpy as np
import pytest

F = np.float32


def alnscore_literal(post):
	"""calcalnscoreflat.cpp:4-32 line for line, float32 throughout (Best3 from best3.h)"""
	LX, LY = post.shape
	row = [F(0)]*(LY + 1)
	for i in range(1, LX + 1):
		currj1 = F(0)
		prevj1 = row[0]
		row[0] = F(0)
		for j in range(1, LY + 1):
			prevj = row[j]
			B = F(prevj1 + post[i - 1, j - 1])
			X, Y = prevj, currj1
			prevj1 = row[j]
			if B >= X:
				currj1 = B if B >= Y else Y
			else:
				currj1 = X if X >= Y else Y
			row[j] = currj1
	return row[LY]


def alnscore_tree(post):
	"""the kernel's one-strip EA: row by row, every candidate queries the tree for columns < j, then the
	row's updates are applied; the score is the max of all V"""
	LX, LY = post.shape
	tree = np.zeros(LY + 1, np.float32)
	vmax = F(0)
	for i in range(LX):
		cols = np.flatnonzero(post[i] != 0)
		pend = []
		for e0 in range(0, len(cols), 32):
			for j in cols[e0:e0 + 32]:
				q, k = F(0), int(j)
				while k > 0:
					q = max(q, tree[k])
					k &= k - 1
				v = F(post[i, j] + q)
				vmax = max(vmax, v)
				pend.append((v, int(j) + 1))
		for v, k in pend:
			while k <= LY:
				tree[k] = max(tree[k], v)
				k += k & -k
	return vmax


def _sparse(rng, LX, LY, per_row, values):
	post = np.zeros((LX, LY), np.float32)
	for i in range(LX):
		n = min(LY, int(rng.integers(0, 2*per_row + 1)))
		post[i, rng.choice(LY, n, replace=False)] = rng.choice(values, n)
	return post


def cases():
	rng = np.random.default_rng(20)
	probs = np.float32(rng.random(4000))
	quantized = np.float32([0.01, 0.125, 0.25, 0.5, 1.0])           # sums that tie exactly
	yield "empty", np.zeros((7, 9), np.float32)
	yield "one row", np.float32([[0.0, 0.5, 0.0, 0.25]])
	yield "one column", np.float32([[0.3], [0.0], [0.6]])
	for s in range(12):
		LX, LY = int(rng.integers(1, 40)), int(rng.integers(1, 60))
		yield "random %d" % s, _sparse(rng, LX, LY, 3, probs)
		yield "ties %d" % s, _sparse(rng, LX, LY, 3, quantized)
	p = _sparse(rng, 30, 45, 4, quantized)
	p[:, 0] = 0.5
	p[:, -1] = 0.25
	p[::3] = 0.0                                                       # empty rows between full ones
	yield "first and last column", p
	p = np.zeros((24, 150), np.float32)
	for i, n in enumerate([33, 64, 65, 96, 97, 128, 0, 40] * 3):         # several batches of 32 per row
		p[i, rng.choice(150, n, replace=False)] = rng.choice(quantized if i % 2 else probs, n)
	yield "long rows", p
	yield "dense", np.float32(rng.random((20, 30)))


@pytest.mark.parametrize("name,post", list(cases()), ids=[n for n, _ in cases()])
def test_tree_equals_calcalnscoreflat(name, post):
	want = alnscore_literal(post)
	got = alnscore_tree(post)
	assert np.float32(got).tobytes() == np.float32(want).tobytes(), (name, got, want)


@pytest.mark.parametrize("name,post", list(cases()), ids=[n for n, _ in cases()])
def test_tree_equals_oracle(oracle, name, post):
	assert np.float32(alnscore_tree(post)) == np.float32(oracle.alnscore(post)), name
