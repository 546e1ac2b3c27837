/* muscle_b200.h -- C ABI of libmuscle_b200.so, the H100-native pair engine for MUSCLE5's MPCFlat stage.
 *
 * The reference (rcedgar/muscle @ 6c69a9b) has no plugin/FFI interface for this path: it is C++
 * free functions and the MPCFlat / PProg classes linked into one binary.  The boundary below is
 * therefore defined by the reference's call sites (SURVEY.md section 8b); every entry point names
 * the reference code it replaces (paths relative to /root/reference/src).  All functions are
 * extern "C", take plain pointers and sizes, return 0 on success or a negative MB200_E* code, and
 * leave a message retrievable with mb200_last_error() (the reference convention is Die() ->
 * exit(1), myutils.cpp:883; the C++ shim in INTEGRATION.md turns a non-zero return into Die()).
 *
 * Ownership: the library owns all device memory inside the context; every host buffer is
 * caller-allocated and never freed by the library.  A context is bound to one CUDA device and may
 * be used by one host thread at a time (the reference's OpenMP pair loops collapse into one batch
 * call issued by one thread; use one context per thread for UClust-style per-pair calls).
 *
 * There is NO CPU fallback: without a CUDA device every compute entry point fails with
 * MB200_ENODEV.
 */
#ifndef MUSCLE_B200_H
#define MUSCLE_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MB200_OK         0
#define MB200_EINVAL    -1   /* bad argument / call order                                  */
#define MB200_ENODEV    -2   /* no usable CUDA device                                      */
#define MB200_ECUDA     -3   /* CUDA runtime error (message has the cudaError string)      */
#define MB200_ENOMEM    -4   /* device allocation failed                                   */
#define MB200_EOVERFLOW -5   /* reference guard LX*LY*5+100 > INT_MAX (fwdflat3.cpp:17) or
                                more than MB200_MAX_ROW_NNZ candidate entries in one row   */
#define MB200_EALPHABET -6   /* more distinct residue classes than the device tables hold  */

#define MB200_MAX_ROW_NNZ 128  /* a posterior row holds <= 100 entries >= 0.01 (they sum to <= 1) */

typedef struct mb200_ctx mb200_ctx;

/* Sparse wire format = MySparseMx's own (mysparsemx.h:6-98): uint32 offsets[LX+1] and
 * nnz x {float P; uint32 col}, columns ascending, so host MySparseMx objects are filled by memcpy. */
typedef struct { float p; uint32_t col; } mb200_entry;

/* ---- lifetime ---------------------------------------------------------------------------- */
int         mb200_create(int device, mb200_ctx **out);
void        mb200_destroy(mb200_ctx *ctx);
const char *mb200_last_error(const mb200_ctx *ctx);   /* ctx may be NULL: last create() error */
/* library/ABI version and the sm target it was compiled for, e.g. "0.1.0 sm_90a" */
const char *mb200_version(void);

/* ---- inputs ------------------------------------------------------------------------------ */
/* Upload the PairHMM tables exactly as the host computed them: PairHMM::m_StartScore[5],
 * m_TransScore[5][5], m_InsScore[256], m_MatchScore[256][256] (pairhmm.h:26-29, filled by
 * HMMParams::ToPairHMM hmmparams.cpp:298-409), plus MIN_SPARSE_SCORE = logf(0.01f) as evaluated
 * by the host libm (mysparsemx.h:4).  Call again after every ToPairHMM (e.g. -perturb replicates). */
int mb200_set_hmm(mb200_ctx *ctx, const float start[5], const float trans[25],
                  const float ins[256], const float match[65536], float min_sparse_score);

/* Upload the sequences (raw bytes exactly as Sequence::GetBytePtr returns them, sequence.h:56-61).
 * offsets[nseq+1] index into bytes.  Replaces the label->sequence registry lookups of
 * CalcPost (calcpost.cpp:4-36, globalinputms.cpp:125-143): the library speaks indices.
 * Invalidates any stored posteriors. */
int mb200_set_seqs(mb200_ctx *ctx, uint32_t nseq, const uint8_t *bytes, const uint64_t *offsets);

/* Mega / Muscle-3D feature profiles (SURVEY.md section 8 f4) instead of residue bytes: the emission
 * side of Mega::CalcFwdFlat_mega / CalcBwdFlat_mega (fwdflat_mega.cpp:14, bwdflat_mega.cpp), i.e. what
 * CalcPost switches to when a .mega input is loaded (calcpost.cpp:14-22).  A position is a vector of
 * nfeat <= 8 feature letters (Mega::m_Profiles, mega.h:25): letters[(offsets[s]+i)*nfeat + f].
 * alpha[f] = alphabet size (Mega::m_AlphaSizes), weights[f] = Mega::m_Weights, logprobs = the vectors
 * Mega::m_LogProbsVec[f] back to back, logprobmx = the matrices Mega::m_LogProbMxVec[f] (row-major)
 * back to back.  Match emission = sum_f logprobmx_f[a_f][b_f]*w_f, insert emission = sum_f
 * logprobs_f[a_f]*w_f, both accumulated from 0 in feature order with separate fp32 multiply and add
 * (Mega::GetMatchScore / GetInsScore, mega.cpp:273-359).  Transitions and the sparsification cut still
 * come from mb200_set_hmm.  Replaces mb200_set_seqs (either call selects the emission mode). */
int mb200_set_seqs_mega(mb200_ctx *ctx, uint32_t nseq, const uint8_t *letters, const uint64_t *offsets,
                        uint32_t nfeat, const uint32_t *alpha, const float *weights,
                        const float *logprobs, const float *logprobmx);

/* ---- posterior stage --------------------------------------------------------------------- */
/* Replaces the OpenMP loop MPCFlat::CalcPosteriors (mpcflat.cpp:214-252) and, per pair,
 * MPCFlat::CalcPosterior (calcposteriorflat.cpp:45-92) = CalcPost (calcpost.cpp:4: CalcFwdFlat
 * fwdflat3.cpp:12, CalcBwdFlat bwdflat3.cpp:10, CalcPostFlat calcposteriorflat.cpp:4,
 * CalcTotalProbFlat totalprobflat.cpp:3) + MySparseMx::FromPost (mysparsemx.cpp:115) +
 * CalcAlnScoreFlat (calcalnscoreflat.cpp:4) + EA = Score/min(LX,LY).
 * Pair k is (pair_x[k], pair_y[k]); X indexes rows.  The sparse posteriors stay resident on the
 * device as "the store" (replacing m_SparsePosts1, mpcflat.h:46-49); ea_out[k] (host, may be
 * NULL) receives what the reference writes to m_DistMx[x][y].
 * Also serves PProg::GetPostPairsAlignedFlat (getpostpairsalignedflat.cpp:5), CalcEADistMx
 * (eadistmx.cpp:7) and AlignPairFlat_SparsePost (alignpairflat.cpp:3) with their pair lists. */
#define MB200_POST_DEFAULT 0u
int mb200_posteriors(mb200_ctx *ctx, uint32_t npairs, const uint32_t *pair_x, const uint32_t *pair_y,
                     uint32_t flags, float *ea_out);

/* Same, all-pairs convenience: pairs (i<j) in the reference's row-major order
 * (MPCFlat::InitPairs mpcflat.cpp:139-159), restricted to pair indexes [p_lo,p_hi) so that a
 * multi-GPU caller can shard; ea_out has p_hi-p_lo slots.  Store pair k <-> global pair p_lo+k. */
int mb200_posteriors_allpairs(mb200_ctx *ctx, uint32_t p_lo, uint32_t p_hi, float *ea_out);

/* Store introspection (host copies).  nnz_out[npairs]. */
int mb200_store_npairs(const mb200_ctx *ctx, uint32_t *npairs);
int mb200_store_nnz(mb200_ctx *ctx, uint32_t *nnz_out, uint64_t *total_nnz);
/* Copy one stored pair out in MySparseMx layout: offsets[LX+1], entries[nnz] (host buffers).
 * Replaces reading (*m_ptrSparsePosts)[PairIndex] (mpcflat.cpp:88-98). */
int mb200_export_pair(mb200_ctx *ctx, uint32_t pair, uint32_t *offsets, mb200_entry *entries);
/* Copy every stored pair out, packed back to back in store order: offsets_concat has
 * sum(LX_k+1) slots (each pair's offsets start at 0), entries_concat has total_nnz slots. */
int mb200_export_all(mb200_ctx *ctx, uint32_t *offsets_concat, mb200_entry *entries_concat);

/* ---- store exchange (multi-GPU, SURVEY.md section 8e) ------------------------------------- */
/* Device-side packed image of the store for NCCL all-gather: row offsets and entries of every
 * stored pair, in store order.  The pointers are device pointers owned by the context and stay
 * valid until the store changes.  n_offsets = sum(LX_k+1), n_entries = total nnz. */
int mb200_store_pack(mb200_ctx *ctx, const uint32_t **d_offsets, uint64_t *n_offsets,
                     const mb200_entry **d_entries, uint64_t *n_entries);
/* Replace the store with the concatenation of packed images of the all-pairs ranges
 * [p_lo,p_hi) (the gathered result); d_* are device pointers (caller-owned, copied). */
int mb200_store_load_allpairs(mb200_ctx *ctx, uint32_t p_lo, uint32_t p_hi,
                              const uint32_t *d_offsets, uint64_t n_offsets,
                              const mb200_entry *d_entries, uint64_t n_entries);
/* In-place variant for the NCCL all-gather-v (SURVEY.md section 8e): _begin returns library-owned
 * device buffers sized for the image of ALL N(N-1)/2 pairs (n_offsets = sum over pairs of LX+1,
 * n_entries = total nnz); the caller's collective receives every rank's packed image (its own
 * included, read from mb200_store_pack) directly at its final position, in pair order; _commit
 * adopts the buffers as the store.  The rank's own packed store stays readable until _commit. */
int mb200_store_exchange_begin(mb200_ctx *ctx, uint64_t n_offsets, uint64_t n_entries,
                               uint32_t **d_offsets, mb200_entry **d_entries);
int mb200_store_exchange_commit(mb200_ctx *ctx);
/* Device pointer of the packed entries (store order).  Between consistency iterations the ranks
 * all-gather their updated entry ranges in place through this pointer (the pattern is invariant,
 * mysparsemx.cpp:87-113) and then call mb200_store_values_changed. */
int mb200_store_entries_ptr(mb200_ctx *ctx, mb200_entry **d_entries, uint64_t *n_entries);
int mb200_store_values_changed(mb200_ctx *ctx);
/* values-only image (float per entry, store order) for the exchange between consistency
 * iterations: the pattern is invariant (mysparsemx.cpp:87-113). */
int mb200_store_values(mb200_ctx *ctx, float *d_values_out, uint64_t n_entries);
int mb200_store_set_values(mb200_ctx *ctx, const float *d_values, uint64_t first_entry, uint64_t n_entries);

/* ---- consistency (relax) ------------------------------------------------------------------ */
/* One Jacobi iteration over the all-pairs store: replaces MPCFlat::ConsIter (consflat.cpp:5-23)
 * = for every pair MPCFlat::ConsPair (conspairflat.cpp:10-110) with RelaxFlat_ZX_ZY / _XZ_ZY /
 * _XZ_YZ (relaxflat.cpp:4,33,62) and MySparseMx::UpdateFromPost (mysparsemx.cpp:87), followed by
 * the buffer swap.  Requires the store to hold all N(N-1)/2 pairs of the current sequences.
 * Only pairs with index in [p_lo,p_hi) are updated (multi-GPU sharding; pass 0,npairs for all);
 * the others keep their old values until mb200_store_set_values brings the peers' results. */
int mb200_consistency_iter(mb200_ctx *ctx, uint32_t p_lo, uint32_t p_hi);

/* ---- posterior decoding ------------------------------------------------------------------- */
/* Batched CalcAlnFlat (calcalnflat.cpp:6-46) + TraceBackFlat (tracebackflat.cpp:3-37) on the
 * stored pairs: for each listed store pair, densify its sparse posterior, run the max-sum DP with
 * Best3 tie order (best3.h:5-28) and trace back.  paths_out: concatenated, pair k's path starts
 * at path_off[k] and owns path_off[k+1]-path_off[k] >= LX_k+LY_k+1 bytes (path_off has n+1 entries,
 * path_off[n] = size of paths_out), NUL terminated, letters B/X/Y; scores_out[k] = DP score.  Serves AlignPairFlat (alignpairflat.cpp:23) and
 * PProg::GetPostPairsAlignedFlat (getpostpairsalignedflat.cpp:62-90). */
int mb200_align_pairs(mb200_ctx *ctx, uint32_t n, const uint32_t *store_pairs,
                      char *paths_out, const uint64_t *path_off, float *scores_out);

/* MPCFlat::AlignAlns (alnalnsflat.cpp:7-52) minus the gap insertion: BuildPost
 * (buildpostflat.cpp:18-105) of two groups of already-aligned sequences followed by CalcAlnFlat +
 * traceback.  ids_a[na]/ids_b[nb]: sequence indexes; pos2col_*: concatenated position->column maps
 * (Sequence::GetPosToCol sequence.cpp:144-154), sequence s of group a starting at
 * sum of lengths of the previous group members; cols_a/cols_b: column counts.
 * path_out needs cols_a+cols_b+1 bytes; post_out (cols_a*cols_b floats, host) may be NULL. */
int mb200_align_groups(mb200_ctx *ctx,
                       uint32_t na, const uint32_t *ids_a, const uint32_t *pos2col_a, uint32_t cols_a,
                       uint32_t nb, const uint32_t *ids_b, const uint32_t *pos2col_b, uint32_t cols_b,
                       char *path_out, float *score_out, float *post_out);

/* ---- device-resident multiple alignments (SURVEY.md section 8 f3) --------------------------- */
/* The data path of MPCFlat::ProgressiveAlign / ProgAln (progalnflat.cpp:41-100) and MPCFlat::RefineIter
 * (refineflat.cpp:4-31) without per-join host<->device traffic of column maps: the library keeps, for
 * every sequence, the position -> column map of the MSA it currently belongs to
 * (Sequence::GetPosToCol, sequence.cpp:144-154).
 *   mb200_msa_reset   every sequence becomes a one-row MSA (the leaves, progalnflat.cpp:79-85).
 *   mb200_msa_join    A and B are disjoint lists of sequence ids in MSA row order; all members of A
 *                     (resp. B) must currently share one MSA, of which A may be a subset.  Does, on
 *                     the device: MultiSequence::Project of each group (project.cpp:16-69: all-gap
 *                     columns dropped -- a no-op when the group is a whole MSA), MPCFlat::BuildPost
 *                     (buildpostflat.cpp:18-105), CalcAlnFlat + traceback (calcalnflat.cpp:6-46),
 *                     and Sequence::AddGapsPath (sequence.cpp:115-140) applied to the column maps of
 *                     every member ('X' for A, 'Y' for B, alnalnsflat.cpp:36-50).  Afterwards all
 *                     members share one MSA of *cols_out columns whose row order is A then B.
 *                     path_out (may be NULL; path_cap bytes >= cols_a+cols_b+1) receives the path.
 *   mb200_msa_export  concatenated position -> column maps of the listed sequences (what the host
 *                     needs to print the final MSA); cols_out[k] (may be NULL) = columns of its MSA. */
int mb200_msa_reset(mb200_ctx *ctx);
int mb200_msa_join(mb200_ctx *ctx, uint32_t na, const uint32_t *ids_a, uint32_t nb, const uint32_t *ids_b,
                   uint32_t *cols_out, float *score_out, char *path_out, uint32_t path_cap);
int mb200_msa_export(mb200_ctx *ctx, uint32_t n, const uint32_t *ids, uint32_t *pos2col_out, uint32_t *cols_out);

/* ---- guide tree (SURVEY.md section 8 f2) ------------------------------------------------------ */
/* UPGMA5::FixEADistMx (upgma5.cpp:504-519, distance = 1 - EA) + UPGMA5::Run (upgma5.cpp:87-330) as
 * MPCFlat::CalcGuideTree calls them (mpcflat.cpp:183-205) -- including the reference's nearest-
 * neighbour bookkeeping and tie order, which decide the topology.  ea: host vector of the N(N-1)/2 EA
 * values in all-pairs order (what mb200_posteriors_allpairs / mb200_group_posteriors_allpairs
 * returned), or NULL to use the EA vector the posterior stage left on this device.  Outputs are host
 * arrays of N-1 entries indexed by internal node (join order): children as node indexes (0..N-1
 * leaves, N+k internal node k) and branch lengths -- exactly the arguments of Tree::Create
 * (tree.cpp:1454).  Join order (guidetreejoinorder.cpp:103) is a traversal of that 2N-1 node tree
 * and stays on the host. */
#define MB200_LINKAGE_MIN    1      /* values of the reference's LINKAGE enum (types.h:11-15) */
#define MB200_LINKAGE_MAX    2
#define MB200_LINKAGE_AVG    3
#define MB200_LINKAGE_BIASED 4
int mb200_guide_tree(mb200_ctx *ctx, const float *ea, int linkage, uint32_t *left, uint32_t *right,
                     float *left_len, float *right_len);

/* ---- per-pair debug/parity surface -------------------------------------------------------- */
/* CalcPost (calcpost.cpp:4-36) for one pair with the dense result copied to the host:
 * post_out[LX*LY] thresholded posterior (CalcPostFlat), fwd_m_out / bwd_m_out (may be NULL)
 * the M-state planes [(LX)*(LY)] for rows/cols 1.., total_out the log total probability. */
int mb200_calc_post_dense(mb200_ctx *ctx, uint32_t x, uint32_t y, float *post_out,
                          float *fwd_m_out, float *bwd_m_out, float *total_out);

/* ---- test / tuning hooks (not needed by a binding) ------------------------------------------ */
/* Residue classes of a set of PairHMM tables: bytes with the same insert score and the same match
 * row and column share a class (21 for proteins: 20 letters, both cases, + one wildcard class).
 * Pure host code, works without a CUDA device.  rep_out (may be NULL) gets the first byte per class. */
int mb200_residue_classes(const float ins[256], const float match[65536], uint8_t byte2class[256],
                          int *nclass_out, int rep_out[256]);
/* force the columns-per-lane of mb200_calc_post_dense (0 = automatic): exercises the strip code */
int mb200_debug_force_c(mb200_ctx *ctx, int c);
/* expected entries per posterior row used to size the entry pool (default 12; the pool is re-sized
 * with the exact count and the stage re-run if it was too small) */
int mb200_set_nnz_per_row_cap(mb200_ctx *ctx, uint32_t cap);
/* The work plan of the last posterior call, as the kernel reads it.  A chain is a run of pairs that
 * share Y and that one warp computes back to back; chain c is order[chain[c] .. chain[c+1]) (store
 * pair ids).  *npairs and *nchains are always set; order[npairs], chain[nchains+1], bin_start[18]
 * (bin_start[C] = first chain of the pairs run at C columns per lane, C = 1..16; bin_start[17] =
 * nchains) and limits[2] (the most Forward rows, sum of LX+2, and the most pairs in one chain) are
 * filled when not NULL, so a first call with NULL arrays returns the counts. */
int mb200_debug_plan(mb200_ctx *ctx, uint32_t *npairs, uint32_t *nchains, uint32_t *order, uint32_t *chain,
                     uint32_t *bin_start, uint32_t *limits);
/* mb200_calc_post_dense for store pair `which` of a pair list: runs the whole list as
 * mb200_posteriors does (same chains, the store and EA are filled too) and copies out the dense
 * results of that one pair, at whatever position of its chain it runs.  Honours
 * mb200_debug_force_c.  mb200_calc_post_dense(x, y) is the one-pair case. */
int mb200_calc_post_dense_pair(mb200_ctx *ctx, uint32_t npairs, const uint32_t *pair_x, const uint32_t *pair_y,
                               uint32_t which, float *post_out, float *fwd_m_out, float *bwd_m_out,
                               float *total_out);

/* ---- several GPUs from one process (SURVEY.md section 8b: "mb200_create(ndev, ...)") -------- */
/* A group is ndev single-device contexts plus the two exchange steps of the path (section 8e).
 * It serves the single-process caller (`muscle_b200 -align`): mb200_group_posteriors_allpairs
 * replaces MPCFlat::CalcPosteriors (mpcflat.cpp:214-252) with the pair list sharded in contiguous
 * cell-balanced ranges and an all-gather-v of the packed store images over NVLink peer memory, so
 * that every device ends with the complete store; mb200_group_consistency_iter replaces
 * MPCFlat::ConsIter (consflat.cpp:5-23) with every device updating its own pair range followed by an
 * in-place exchange of the updated entries.  The serial stages (mb200_align_groups, mb200_msa_*)
 * run on mb200_group_ctx(g, 0).  devices == NULL or ndev <= 0: all visible devices. */
typedef struct mb200_group mb200_group;
int         mb200_group_create(int ndev, const int *devices, mb200_group **out);
void        mb200_group_destroy(mb200_group *g);
const char *mb200_group_last_error(const mb200_group *g);
int         mb200_group_size(const mb200_group *g);
mb200_ctx  *mb200_group_ctx(mb200_group *g, int rank);
int mb200_group_set_hmm(mb200_group *g, const float start[5], const float trans[25],
                        const float ins[256], const float match[65536], float min_sparse_score);
int mb200_group_set_seqs(mb200_group *g, uint32_t nseq, const uint8_t *bytes, const uint64_t *offsets);
int mb200_group_set_seqs_mega(mb200_group *g, uint32_t nseq, const uint8_t *letters, const uint64_t *offsets,
                              uint32_t nfeat, const uint32_t *alpha, const float *weights,
                              const float *logprobs, const float *logprobmx);
int mb200_group_posteriors_allpairs(mb200_group *g, float *ea_out);   /* ea_out[N(N-1)/2], may be NULL */
int mb200_group_consistency_iter(mb200_group *g);
typedef struct
	{
	uint32_t ndev;
	uint64_t cells;                    /* DP cells of the last posterior stage, all devices        */
	float    posterior_ms;             /* host wall, slowest device                                */
	float    exchange1_ms;             /* store all-gather-v                                       */
	uint64_t exchange1_bytes_per_dev;  /* bytes every device received                              */
	float    relax_ms;                 /* last consistency iteration, slowest device (host wall)   */
	float    relax_kernel_ms;          /* k_relax device time, slowest device                      */
	float    exchange2_ms;             /* in-place exchange of the updated entries                 */
	uint64_t exchange2_bytes_per_dev;
	} mb200_group_stats;
int mb200_group_get_stats(const mb200_group *g, mb200_group_stats *out);

/* ---- instrumentation ---------------------------------------------------------------------- */
typedef struct
	{
	uint64_t kernel_launches;    /* kernels launched by this context since creation         */
	uint64_t cells;              /* DP cells of the last posterior call                     */
	float    last_kernel_ms;     /* device time of the dominant kernel(s) of the last call  */
	float    last_total_ms;      /* device time of the whole last call (events)             */
	uint64_t h2d_bytes;          /* host->device bytes moved by the last call               */
	uint64_t d2h_bytes;          /* device->host bytes moved by the last call               */
	} mb200_stats;
int mb200_get_stats(const mb200_ctx *ctx, mb200_stats *out);

#ifdef __cplusplus
}
#endif
#endif
