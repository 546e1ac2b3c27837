"""Test helper: emission tables past the one protein table and the one Mega model (BB11001).

* plain_tables(K, seed): PairHMM tables with exactly K residue classes (K = 1..64 fit the device
  tables, 65 is the first count they must reject), asymmetric match tables, and the class alphabet to
  write sequences with.
* mega_model(alpha, weights, seed): random Mega feature models with asymmetric pair matrices.
* vocabulary profiles: every position of a set of Mega profiles is one of V <= 127 distinct letter
  vectors, so vocabulary_tables() can give vector v the byte v+1 of one PairHMM table whose ins/match
  entries are the Mega emissions of the vectors (mega_util.emissions).  The plain oracle then computes
  every pair of the set at any length, where mega_util.synthetic_tables stops at 128 positions.

Homologous families (substitutions plus indels) keep posteriors informative at every length.  Sequence
bytes stay below 128: the reference indexes its insert table with a signed char."""
import numpy as np
import mega_util
from conftest import load_tables

PRINTABLE = np.arange(33, 127, dtype=np.uint8)      # 94 bytes: up to 93 letter classes + the rest


def _log_probs(rng, K, asymmetric=True, enrich=8.0):
	"""-> (log q[K], log P[K,K]) float32: background frequencies and a joint pair distribution whose
	diagonal is enriched; off-diagonal pairs are drawn independently unless symmetric"""
	q = rng.dirichlet(np.full(K, 4.0))
	noise = np.exp(rng.normal(0.0, 0.7, (K, K)))
	if not asymmetric:
		noise = np.sqrt(noise*noise.T)
	P = np.outer(q, q)*noise
	P[np.diag_indices(K)] *= enrich
	P /= P.sum()
	return np.log(q).astype(np.float32), np.log(P).astype(np.float32)


def plain_tables(K, seed, asymmetric=True, pad_shares_letter=False):
	"""-> (tables, alphabet): PairHMM tables with exactly K residue classes and K bytes, alphabet[c] of class c.
	Start, transitions and min_sparse_score are the protein model's.  Classes 0..K-2 are single printable
	letters; every other byte, byte 0 included, forms class K-1 (alphabet[K-1] is a printable member of it).
	pad_shares_letter puts byte 0, which the reference reads past a sequence's end, into letter class 0."""
	assert 1 <= K <= len(PRINTABLE)
	assert not pad_shares_letter or K >= 2
	rng = np.random.default_rng(seed)
	alphabet = rng.permutation(PRINTABLE)[:K]
	ins_c, match_c = _log_probs(rng, K, asymmetric)
	cls = np.full(256, K - 1, np.int64)
	cls[alphabet[:K - 1]] = np.arange(K - 1)
	if pad_shares_letter:
		cls[0] = 0
	t = dict(load_tables())
	t["ins"] = np.ascontiguousarray(ins_c[cls])
	t["match"] = np.ascontiguousarray(match_c[cls[:, None], cls[None, :]].reshape(-1))
	return t, bytes(alphabet)


def _evolve(rng, root, V, p_sub, p_indel=0.03):
	out, i = [], 0
	while i < len(root):
		r = rng.random()
		if r < p_indel/2:                              # deletion
			i += int(rng.geometric(1/3))
			continue
		if r < p_indel:                                # insertion
			out.extend(rng.integers(0, V, int(rng.geometric(1/3))).tolist())
		out.append(int(root[i]) if rng.random() >= p_sub else int(rng.integers(0, V)))
		i += 1
	return out


def family_codes(V, lengths, seed, p_sub=0.3):
	"""-> list of int arrays over 0..V-1 of exactly the given lengths: homologs of one root (windows of
	mutated copies, extended by random symbols where a copy is too short)"""
	rng = np.random.default_rng(seed)
	root = rng.integers(0, V, max(lengths) + 16)
	out = []
	for L in lengths:
		s = _evolve(rng, root, V, p_sub)
		if len(s) >= L:
			a = int(rng.integers(0, len(s) - L + 1))
			s = s[a:a + L]
		else:
			s = s + rng.integers(0, V, L - len(s)).tolist()
		out.append(np.array(s, np.int64))
	return out


def plain_family(alphabet, lengths, seed, p_sub=0.3):
	"""-> byte strings over alphabet (one byte per class), homologs of one root"""
	a = np.frombuffer(bytes(alphabet), np.uint8)
	return [a[c].tobytes() for c in family_codes(len(a), lengths, seed, p_sub)]


# ------------------------------------------------------------------------------------------------
# Mega
def mega_model(alpha, weights, seed):
	"""-> Mega model dict(alpha, weights, logprobs, logprobmx): per feature a random log-frequency vector
	and an asymmetric log-probability pair matrix with an enriched diagonal"""
	rng = np.random.default_rng(seed)
	lp, lpm = [], []
	for a in alpha:
		q, P = _log_probs(rng, int(a))
		lp.append(q)
		lpm.append(P.reshape(-1))
	return {"alpha": np.array(alpha, np.uint32), "weights": np.array(weights, np.float32),
	  "logprobs": np.concatenate(lp).astype(np.float32), "logprobmx": np.concatenate(lpm).astype(np.float32)}


def vocabulary(model, V, seed):
	"""-> uint8 [V', nf]: V' = min(V, number of possible vectors) distinct letter vectors"""
	rng = np.random.default_rng(seed)
	alpha = [int(a) for a in model["alpha"]]
	V = int(min(V, np.prod(alpha, dtype=np.float64)))
	seen, out = set(), []
	while len(out) < V:
		v = tuple(int(rng.integers(0, a)) for a in alpha)
		if v not in seen:
			seen.add(v)
			out.append(v)
	return np.array(out, np.uint8).reshape(V, len(alpha))


def vocabulary_tables(base, model, vocab, first=1):
	"""PairHMM tables under which the plain oracle computes Mega pairs over vocab: vector v is byte v+first,
	its ins entry and the match entry of every vector pair are the Mega emissions (mega_util.emissions)"""
	V = len(vocab)
	assert first + V <= 256
	ins, _, match = mega_util.emissions(model, vocab, vocab)
	t = dict(base)
	i = np.zeros(256, np.float32)
	i[first:first + V] = ins
	m = np.zeros((256, 256), np.float32)
	m[first:first + V, first:first + V] = match
	t["ins"], t["match"] = i, m.reshape(-1)
	return t


def mega_family(vocab, lengths, seed, p_sub=0.3, first=1):
	"""-> (profiles as letter arrays [L][nf], the same as byte strings for vocabulary_tables)"""
	codes = family_codes(len(vocab), lengths, seed, p_sub)
	return [vocab[c] for c in codes], [(c + first).astype(np.uint8).tobytes() for c in codes]


# The table sets the GPU tests run: plain K values and Mega feature models (alpha, weights)
PLAIN_K = [1, 2, 5, 21, 32, 33, 63, 64]
MEGA_MODELS = {
	"nf1_a110": ([110], [1.0]),
	"nf2_a1": ([20, 1], [0.8, 0.35]),                                  # a feature with one letter
	"nf3_12288": ([64, 64, 64], [0.5, 0.3, 0.25]),                      # 3*64*64 = 12 288 table floats
	"nf4": ([5, 9, 3, 17], [0.3, 0.2, 0.35, 0.25]),
	"nf5_w0": ([20, 16, 6, 11, 4], [0.4, 0.2, 0.0, 0.3, 0.15]),        # a weight of exactly 0
	"nf6": ([4, 13, 16, 2, 8, 30], [0.1, 0.2, 0.15, 0.05, 0.2, 0.3]),
	"nf7": ([20, 16, 16, 16, 16, 16, 16], [0.4, 0.13, 0.2, 0.15, 0.09, 0.005, 0.02]),
	"nf8": ([20, 16, 16, 16, 16, 16, 16, 16], [0.4, 0.13, 0.2, 0.15, 0.09, 0.005, 0.018, 0.004]),
}


def plain_set(name):
	"""'K=<k>' or 'K=<k>,pad' -> (tables, alphabet)"""
	K = int(name.split(",")[0][2:])
	return plain_tables(K, 1000 + K, pad_shares_letter=name.endswith(",pad"))


def mega_set(name, V=127):
	"""-> (model, vocab, oracle tables)"""
	alpha, weights = MEGA_MODELS[name]
	seed = 2000 + sorted(MEGA_MODELS).index(name)
	model = mega_model(alpha, weights, seed)
	vocab = vocabulary(model, V, seed)
	return model, vocab, vocabulary_tables(load_tables(), model, vocab)
