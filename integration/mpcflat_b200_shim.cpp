// integration/mpcflat_b200_shim.cpp -- the reference-side binding a MUSCLE maintainer would add to
// make libmuscle_b200.so the pair engine of `muscle -align` (INTEGRATION.md).
//
// It is compiled against the UNMODIFIED reference headers and replaces, at link time, exactly the
// MPCFlat members that own the hot loops and the data path of the join/refine loop:
//   MPCFlat::CalcPosteriors   (mpcflat.cpp:214-252)    -> mb200_group_posteriors_allpairs (all visible GPUs)
//   MPCFlat::CalcPosterior    (calcposteriorflat.cpp:45-92, per-pair form used by -profalign/-profseq)
//                                                      -> deferred; the batch runs before the first AlignAlns
//   MPCFlat::CalcGuideTree    (mpcflat.cpp:183-205: UPGMA5::FixEADistMx + UPGMA5::Run, upgma5.cpp:504,87)
//                                                      -> mb200_guide_tree (+ the reference's Tree::Create / PermTree)
//   MPCFlat::ConsIter         (consflat.cpp:5-23)      -> mb200_group_consistency_iter
//   MPCFlat::AlignAlns        (alnalnsflat.cpp:7-52)   -> mb200_align_groups (+ the reference's own gap insertion)
//   MPCFlat::ProgressiveAlign (progalnflat.cpp:73-100) -> mb200_msa_reset + one mb200_msa_join per guide-tree join
//   MPCFlat::Refine           (mpcflat.cpp:255-265) / RefineIter (refineflat.cpp:4-31)
//                                                      -> one mb200_msa_join per bipartition (same rand() stream)
// Everything else (FASTA I/O, dereplication, Tree object and join order, sorting, MSA output) is the
// reference's own code, untouched.  Errors keep the reference convention: Die() -> message +
// exit(1) (myutils.cpp:883).  There is no CPU fallback.  A .mega input (Muscle-3D feature profiles)
// selects the engine's Mega emission mode for `-align`; the pair-list callers of -super7
// (pairlist_b200_shim.cpp) do not implement it and stop with a message instead of computing something else.
#include "muscle.h"
#include "mpcflat.h"
#include "pairhmm.h"
#include "mega.h"
#include "../include/muscle_b200.h"

#include <chrono>
static mb200_group *g_Group = 0;
static mb200_ctx *g_Ctx = 0;                       // device 0 of the group: the serial stages
static const MPCFlat *g_StoreOwner = 0;            // whose posteriors the device store holds
static const MPCFlat *volatile g_Deferred = 0;     // CalcPosterior() was called on this object: batch pending
static vector<uint> g_MSAOrder;                    // input-sequence index of every row of m_MSA

// MB200_TRACE=1: wall-time split of the replaced members, printed at exit
static double g_TPost = 0, g_TCons = 0, g_TProg = 0, g_TRefine = 0, g_TAlign = 0;
static uint g_NAlign = 0, g_NJoin = 0;
static double g_TCreate = 0, g_TUpload = 0, g_TPostCall = 0;      // parts of CalcPosteriors
static double Now()
	{
	return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
	}
static void TraceReport()
	{
	mb200_group_stats S;
	memset(&S, 0, sizeof S);
	if (g_Group != 0)
		mb200_group_get_stats(g_Group, &S);
	fprintf(stderr, "\n[mb200 trace] %u GPU(s): CalcPosteriors %.2f s (store exchange %.1f ms, %.2f GB/GPU), ConsIter %.2f s "
	  "(last: kernel %.1f ms, exchange %.1f ms), ProgressiveAlign %.2f s, Refine %.2f s (%u device joins), AlignAlns x%u %.2f s\n",
	  S.ndev, g_TPost, S.exchange1_ms, S.exchange1_bytes_per_dev/1e9, g_TCons, S.relax_kernel_ms, S.exchange2_ms,
	  g_TProg, g_TRefine, g_NJoin, g_NAlign, g_TAlign);
	fprintf(stderr, "[mb200 trace] CalcPosteriors: contexts %.2f s, tables+sequences %.2f s, posteriors call %.2f s (kernels %.0f ms)\n",
	  g_TCreate, g_TUpload, g_TPostCall, S.posterior_ms);
	}

static void Check(int rc, const char *What)
	{
	if (rc != MB200_OK)
		Die("libmuscle_b200 %s failed (%d): %s", What, rc, mb200_last_error(g_Ctx));
	}

static void CheckG(int rc, const char *What)
	{
	if (rc != MB200_OK)
		Die("libmuscle_b200 %s failed (%d): %s", What, rc, mb200_group_last_error(g_Group));
	}

static void EnsureGroup()
	{
	if (g_Group != 0)
		return;
	// MB200_DEVICES=n: use the first n visible GPUs (default: all); MB200_DEVICE=d: only device d.
	// Without MB200_DEVICE the library reads MB200_DEVICE_LIST=a,b,... itself (mb200_group_create).
	int rc;
	const char *one = getenv("MB200_DEVICE");
	const char *cnt = getenv("MB200_DEVICES");
	if (one != 0)
		{
		int Device = atoi(one);
		rc = mb200_group_create(1, &Device, &g_Group);
		}
	else
		rc = mb200_group_create(cnt != 0 ? atoi(cnt) : 0, 0, &g_Group);
	if (rc != MB200_OK)
		Die("libmuscle_b200 mb200_group_create failed (%d): %s", rc, mb200_group_last_error(0));
	g_Ctx = mb200_group_ctx(g_Group, 0);
	if (getenv("MB200_TRACE") != 0)
		atexit(TraceReport);
	}

// the whole posterior stage of one MPCFlat object on the device(s)
static void RunPosteriors(MPCFlat &M)
	{
	double TS = Now();
	EnsureGroup();
	g_TCreate += Now() - TS; TS = Now();
	const uint SeqCount = M.GetSeqCount();
	const uint PairCount = SIZE(M.m_Pairs);
	asserta(PairCount > 0);

// PairHMM tables are process-global statics rewritten between replicates (align.cpp:30-40):
// upload them every time, exactly as the host computed them.
	CheckG(mb200_group_set_hmm(g_Group, PairHMM::m_StartScore, &PairHMM::m_TransScore[0][0],
	  PairHMM::m_InsScore, &PairHMM::m_MatchScore[0][0], MIN_SPARSE_SCORE), "mb200_group_set_hmm");

	vector<byte> Bytes;
	vector<uint64_t> Offsets;
	Offsets.push_back(0);
	if (Mega::m_Loaded)
		{
		// calcpost.cpp:14-22: with a .mega input the emissions come from the feature profiles
		// (Mega::CalcFwdFlat_mega / CalcBwdFlat_mega); hand the model the host derived and the profiles
		// of this object's sequences (looked up by label, like CalcPost does) to the engine
		const uint F = Mega::GetFeatureCount();
		vector<uint> Alpha(F);
		vector<float> Weights(F), LogProbs, LogProbMx;
		for (uint f = 0; f < F; ++f)
			{
			const uint A = Mega::GetAlphaSize(f);
			Alpha[f] = A;
			Weights[f] = Mega::GetWeight(f);
			asserta(SIZE(Mega::m_LogProbsVec[f]) == A && SIZE(Mega::m_LogProbMxVec[f]) == A);
			LogProbs.insert(LogProbs.end(), Mega::m_LogProbsVec[f].begin(), Mega::m_LogProbsVec[f].end());
			for (uint x = 0; x < A; ++x)
				{
				asserta(SIZE(Mega::m_LogProbMxVec[f][x]) == A);
				LogProbMx.insert(LogProbMx.end(), Mega::m_LogProbMxVec[f][x].begin(), Mega::m_LogProbMxVec[f][x].end());
				}
			}
		uint64_t Pos = 0;
		for (uint i = 0; i < SeqCount; ++i)
			{
			const vector<vector<byte> > &Profile = *Mega::GetProfileByLabel(string(M.GetLabel(i)));
			const uint L = M.GetSeqLength(i);
			asserta(SIZE(Profile) == L);
			for (uint k = 0; k < L; ++k)
				{
				asserta(SIZE(Profile[k]) == F);
				Bytes.insert(Bytes.end(), Profile[k].begin(), Profile[k].end());
				}
			Pos += L;
			Offsets.push_back(Pos);
			}
		CheckG(mb200_group_set_seqs_mega(g_Group, SeqCount, Bytes.data(), Offsets.data(), F, Alpha.data(), Weights.data(),
		  LogProbs.data(), LogProbMx.data()), "mb200_group_set_seqs_mega");
		}
	else
		{
		for (uint i = 0; i < SeqCount; ++i)
			{
			const byte *Seq = M.GetBytePtr(i);
			const uint L = M.GetSeqLength(i);
			Bytes.insert(Bytes.end(), Seq, Seq + L);
			Offsets.push_back(Bytes.size());
			}
		CheckG(mb200_group_set_seqs(g_Group, SeqCount, Bytes.data(), Offsets.data()), "mb200_group_set_seqs");
		}

	g_TUpload += Now() - TS; TS = Now();
	vector<float> EAs(PairCount);
	CheckG(mb200_group_posteriors_allpairs(g_Group, EAs.data()), "mb200_group_posteriors_allpairs");
	g_TPostCall += Now() - TS;
	for (uint PairIndex = 0; PairIndex < PairCount; ++PairIndex)
		{
		const pair<uint, uint> &Pair = M.GetPair(PairIndex);
		const float EA = EAs[PairIndex];
		M.m_DistMx[Pair.first][Pair.second] = EA;			// calcposteriorflat.cpp:89-91
		M.m_DistMx[Pair.second][Pair.first] = EA;
		}
	g_StoreOwner = &M;
	g_Deferred = 0;
	}

// a caller is about to read the store of this object: run the deferred batch if there is one
static void NeedStore(MPCFlat &M)
	{
	if (g_Deferred == &M)
		RunPosteriors(M);
	if (g_StoreOwner != &M)
		Die("muscle_b200: posteriors of this MPCFlat object are not on the device "
		  "(AlignAlns / ProgressiveAlign called before CalcPosteriors)");
	}

void MPCFlat::CalcPosteriors()
	{
	const double T0 = Now();
	ProgressStep(0, 2, "Calc posteriors (GPU)");
	RunPosteriors(*this);
	ProgressStep(1, 2, "Calc posteriors (GPU)");
	g_TPost += Now() - T0;
	// The sparse posteriors stay resident in HBM for ConsIter / AlignAlns (the store replaces
	// m_SparsePosts1/2).  Set MB200_EXPORT_SPARSE=1 to also fill the host MySparseMx objects for
	// code that reads GetSparsePost() directly.
	if (getenv("MB200_EXPORT_SPARSE") != 0)
		{
		const uint PairCount = SIZE(m_Pairs);
		for (uint PairIndex = 0; PairIndex < PairCount; ++PairIndex)
			{
			const pair<uint, uint> &Pair = GetPair(PairIndex);
			const uint LX = GetSeqLength(Pair.first);
			const uint LY = GetSeqLength(Pair.second);
			MySparseMx &S = GetSparsePost(PairIndex);
			S.m_LX = LX;
			S.m_LY = LY;
			S.AllocLX(LX);
			Check(mb200_export_pair(g_Ctx, PairIndex, S.m_Offsets, 0), "mb200_export_pair");
			S.m_VecSize = S.m_Offsets[LX];
			S.AllocVec(S.m_VecSize);
			Check(mb200_export_pair(g_Ctx, PairIndex, S.m_Offsets, (mb200_entry *) S.m_ValueVec), "mb200_export_pair");
			S.m_X = GetBytePtr(Pair.first);
			S.m_Y = GetBytePtr(Pair.second);
			}
		}
	}

// -profalign / -profseq call this once per cross pair from an OpenMP loop (profalign.cpp:36-49,
// profseq.cpp:42) and then AlignAlns: the pairs are independent, so the work is deferred and done as
// ONE all-pairs batch on the device when AlignAlns needs the store (a superset of the cross pairs).
void MPCFlat::CalcPosterior(uint PairIndex)
	{
	(void) PairIndex;
	g_Deferred = this;
	}

// mpcflat.cpp:183-205.  The numeric part (distance = 1 - EA, biased-linkage UPGMA with the reference's
// nearest-neighbour bookkeeping) runs on the device; the Tree object, the optional permutation and
// the -guidetreeout exit are the reference's own code.
void MPCFlat::CalcGuideTree()
	{
	if (opt(randomchaintree))
		{
		CalcGuideTree_RandomChain();
		return;
		}
	NeedStore(*this);
	const uint SeqCount = GetSeqCount();
	asserta(SeqCount >= 2 && SIZE(m_Labels) == SeqCount);
	vector<float> EAs;
	EAs.reserve(SIZE(m_Pairs));
	for (uint i = 0; i < SeqCount; ++i)
		for (uint j = i + 1; j < SeqCount; ++j)
			EAs.push_back(m_DistMx[i][j]);
	vector<uint> Left(SeqCount - 1), Right(SeqCount - 1), Ids(SeqCount);
	vector<float> LeftLength(SeqCount - 1), RightLength(SeqCount - 1);
	Check(mb200_guide_tree(g_Ctx, EAs.data(), MB200_LINKAGE_BIASED, Left.data(), Right.data(),
	  LeftLength.data(), RightLength.data()), "mb200_guide_tree");
	vector<char *> Names(SeqCount);
	for (uint i = 0; i < SeqCount; ++i)
		{
		Ids[i] = i;
		Names[i] = mystrsave(m_Labels[i].c_str());
		}
	m_GuideTree.Create(SeqCount, SeqCount - 2, Left.data(), Right.data(), LeftLength.data(), RightLength.data(),
	  Ids.data(), Names.data());                       // as UPGMA5::Run does (upgma5.cpp:305-307)
	for (uint i = 0; i < SeqCount; ++i)
		myfree(Names[i]);
	PermTree(m_GuideTree, m_TreePerm);
	if (optset_guidetreeout)
		{
		const string &FN = opt(guidetreeout);
		Progress("Saving guide tree [%s] to %s\n", TREEPERMToStr(m_TreePerm), FN.c_str());
		m_GuideTree.ToFile(FN);
		Progress("Quitting.\n");
		exit(0);
		}
	}

void MPCFlat::ConsIter(uint Iter)
	{
	NeedStore(*this);
	const uint PairCount = SIZE(m_Pairs);
	asserta(PairCount > 0);
	ProgressStep(0, 2, "Consistency (%u/%u) (GPU)", Iter + 1, m_ConsistencyIterCount);
	const double T0 = Now();
	CheckG(mb200_group_consistency_iter(g_Group), "mb200_group_consistency_iter");
	g_TCons += Now() - T0;
	ProgressStep(1, 2, "Consistency (%u/%u) (GPU)", Iter + 1, m_ConsistencyIterCount);
	// the Jacobi buffer swap (consflat.cpp:22) happens inside the library
	}

MultiSequence *MPCFlat::AlignAlns(const MultiSequence &MSA1, const MultiSequence &MSA2, float *ptrScore)
	{
	NeedStore(*this);
	const double T0 = Now();
	++g_NAlign;
	const uint SeqCount1 = MSA1.GetSeqCount();
	const uint SeqCount2 = MSA2.GetSeqCount();
	const uint ColCount1 = MSA1.GetColCount();
	const uint ColCount2 = MSA2.GetColCount();

	vector<uint> Ids1, Ids2, P2C1, P2C2, PosToCol;
	for (uint i = 0; i < SeqCount1; ++i)
		{
		const Sequence *Seq = MSA1.GetSequence(i);
		Ids1.push_back(GetMyInputSeqIndex(Seq->m_Label));
		Seq->GetPosToCol(PosToCol);
		P2C1.insert(P2C1.end(), PosToCol.begin(), PosToCol.end());
		}
	for (uint i = 0; i < SeqCount2; ++i)
		{
		const Sequence *Seq = MSA2.GetSequence(i);
		Ids2.push_back(GetMyInputSeqIndex(Seq->m_Label));
		Seq->GetPosToCol(PosToCol);
		P2C2.insert(P2C2.end(), PosToCol.begin(), PosToCol.end());
		}

	vector<char> PathBuf(ColCount1 + ColCount2 + 1);
	float Score = 0;
	Check(mb200_align_groups(g_Ctx, SeqCount1, Ids1.data(), P2C1.data(), ColCount1,
	  SeqCount2, Ids2.data(), P2C2.data(), ColCount2, PathBuf.data(), &Score, 0), "mb200_align_groups");
	if (ptrScore != 0)
		*ptrScore = Score;
	const string Path(PathBuf.data());

// gap insertion exactly as alnalnsflat.cpp:36-50
	MultiSequence *result = new MultiSequence();
	for (uint SeqIndex1 = 0; SeqIndex1 < SeqCount1; ++SeqIndex1)
		{
		const Sequence *InputRow = MSA1.GetSequence(SeqIndex1);
		Sequence *AlignedRow = InputRow->AddGapsPath(Path, 'X');
		result->AddSequence(AlignedRow, true);
		}
	for (uint SeqIndex2 = 0; SeqIndex2 < SeqCount2; ++SeqIndex2)
		{
		const Sequence *InputRow = MSA2.GetSequence(SeqIndex2);
		Sequence *AlignedRow = InputRow->AddGapsPath(Path, 'Y');
		result->AddSequence(AlignedRow, true);
		}
	g_TAlign += Now() - T0;
	return result;
	}

// m_MSA from the device-resident column maps, rows in the given order of input-sequence indexes
static MultiSequence *MSAFromDevice(const MPCFlat &M, const vector<uint> &Order)
	{
	const uint N = SIZE(Order);
	uint64_t Total = 0;
	for (uint k = 0; k < N; ++k)
		Total += M.GetSeqLength(Order[k]);
	vector<uint> Maps(Total), Cols(N);
	Check(mb200_msa_export(g_Ctx, N, Order.data(), Maps.data(), Cols.data()), "mb200_msa_export");
	MultiSequence *MS = new MultiSequence;
	uint64_t Off = 0;
	for (uint k = 0; k < N; ++k)
		{
		const uint s = Order[k];
		const Sequence *In = M.m_MyInputSeqs->GetSequence(s);
		const uint L = M.GetSeqLength(s);
		asserta(Cols[k] == Cols[0]);
		Sequence *Row = NewSequence();
		Row->m_Label = In->m_Label;
		Row->m_CharVec.assign(Cols[k], '-');
		const byte *Letters = M.GetBytePtr(s);
		for (uint i = 0; i < L; ++i)
			Row->m_CharVec[Maps[Off + i]] = (char) Letters[i];
		Off += L;
		MS->AddSequence(Row, true);
		}
	return MS;
	}

// progalnflat.cpp:73-100 with ProgAln (:41-71) folded in: the N-1 joins of the guide tree run on the
// device-resident column maps; the host only keeps which sequences a node holds, in MSA row order
// (AlignAlns appends the rows of MSA2 to those of MSA1, alnalnsflat.cpp:36-50).
void MPCFlat::ProgressiveAlign()
	{
	NeedStore(*this);
	const double T0 = Now();
	const uint SeqCount = m_MyInputSeqs->GetSeqCount();
	const uint JoinCount = SeqCount - 1;
	asserta(SIZE(m_JoinIndexes1) == JoinCount);
	asserta(SIZE(m_JoinIndexes2) == JoinCount);
	ValidateJoinOrder(m_JoinIndexes1, m_JoinIndexes2);

	Check(mb200_msa_reset(g_Ctx), "mb200_msa_reset");
	vector<vector<uint> > Members(SeqCount);
	for (uint i = 0; i < SeqCount; ++i)
		Members[i].push_back(i);
	for (uint JoinIndex = 0; JoinIndex < JoinCount; ++JoinIndex)
		{
		const uint Index1 = m_JoinIndexes1[JoinIndex];
		const uint Index2 = m_JoinIndexes2[JoinIndex];
		asserta(Index1 < SIZE(Members) && Index2 < SIZE(Members));
		vector<uint> &A = Members[Index1];
		vector<uint> &B = Members[Index2];
		asserta(!A.empty() && !B.empty());
		Check(mb200_msa_join(g_Ctx, SIZE(A), A.data(), SIZE(B), B.data(), 0, 0, 0, 0), "mb200_msa_join");
		++g_NJoin;
		vector<uint> AB(A);
		AB.insert(AB.end(), B.begin(), B.end());
		A.clear();
		B.clear();
		Members.push_back(AB);
		}
	g_MSAOrder = Members.back();
	asserta(SIZE(g_MSAOrder) == SeqCount);
	m_MSA = MSAFromDevice(*this, g_MSAOrder);
	g_TProg += Now() - T0;
	}

// mpcflat.cpp:255-265 + refineflat.cpp:4-31.  The bipartition consumes the libc rand() stream exactly
// like the reference (one rand() per MSA row, in row order); MultiSequence::Project (all-gap columns
// dropped) and AlignAlns happen on the device maps.
void MPCFlat::Refine()
	{
	const uint SeqCount = GetSeqCount();
	if (SeqCount < 3)
		return;
	NeedStore(*this);
	asserta(m_MSA != 0);
	asserta(SIZE(g_MSAOrder) == SeqCount && m_MSA->GetSeqCount() == SeqCount);
	const double T0 = Now();
	for (uint Iter = 0; Iter < m_RefineIterCount; ++Iter)
		{
		ProgressStep(Iter, m_RefineIterCount, "Refining (GPU)");
		vector<uint> A, B;
		for (uint SeqIndex = 0; SeqIndex < SeqCount; SeqIndex++)
			if (rand()%2 == 0)
				A.push_back(g_MSAOrder[SeqIndex]);
			else
				B.push_back(g_MSAOrder[SeqIndex]);
		if (A.empty() || B.empty())
			continue;
		Check(mb200_msa_join(g_Ctx, SIZE(A), A.data(), SIZE(B), B.data(), 0, 0, 0, 0), "mb200_msa_join");
		++g_NJoin;
		g_MSAOrder = A;
		g_MSAOrder.insert(g_MSAOrder.end(), B.begin(), B.end());
		}
	delete m_MSA;
	m_MSA = MSAFromDevice(*this, g_MSAOrder);
	g_TRefine += Now() - T0;
	}
