// group.cu -- one host process driving several H100s: the multi-device form of the MPCFlat pair
// engine that `muscle_b200 -align` (a single process) uses (SURVEY.md section 8b/8e).
//
// A group is N single-device contexts plus the two exchange steps the path really has:
//   1. posterior stage: the N(N-1)/2 pairs are split into N contiguous, cell-balanced ranges of the
//      reference's row-major pair order (MPCFlat::InitPairs, mpcflat.cpp:139-159); every device
//      computes its range with no communication, then every packed store image is copied to its final
//      position on every peer (an all-gather-v over NVLink peer memory: cudaMemcpyPeerAsync on one
//      stream per source device, all sources concurrently through the NVSwitch) -- afterwards every
//      device holds the complete store, as the Jacobi iteration needs (consflat.cpp:5-23 reads
//      every XZ / ZY of the previous iteration);
//   2. after each sharded consistency iteration the devices exchange their updated entry ranges in
//      place (the pattern is invariant, mysparsemx.cpp:87-113).
// The serial stages (guide tree on the host, progressive alignment, refinement) run on device 0.
// The multi-process form of the same pipeline (one rank per GPU, NCCL) is muscle_b200/dist.py.
#include "engine.h"
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

struct mb200_group
	{
	int ndev = 0;
	std::vector<mb200_ctx *> ctx;
	std::vector<uint32_t> lo, hi;            // pair range per device
	std::vector<uint64_t> off_pos, ent_pos;  // position of each device's image in the gathered store
	bool sharded = false;
	mb200_group_stats stats = {};
	char err[512];
	};

static char g_group_create_error[512] = "";

static int gfail(mb200_group *g, int code, const char *fmt, ...)
	{
	char *dst = g ? g->err : g_group_create_error;
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(dst, 512, fmt, ap);
	va_end(ap);
	return code;
	}

static double now_ms()
	{
	return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
	}

// run f(rank) on one host thread per device; returns the first non-zero code
template <class F>
static int on_all(mb200_group *g, F f)
	{
	std::vector<int> rc(g->ndev, 0);
	if (g->ndev == 1)
		rc[0] = f(0);
	else
		{
		std::vector<std::thread> th;
		for (int r = 0; r < g->ndev; ++r)
			th.emplace_back([&, r] { rc[r] = f(r); });
		for (auto &t : th)
			t.join();
		}
	for (int r = 0; r < g->ndev; ++r)
		if (rc[r] != MB200_OK)
			return gfail(g, rc[r], "device %d: %s", g->ctx[r]->device, mb200_last_error(g->ctx[r]));
	return MB200_OK;
	}

// "a,b,..." -> device numbers; false unless the whole string is a non-empty comma-separated list
static bool parse_device_list(const char *s, std::vector<int> &out)
	{
	out.clear();
	for (const char *p = s;;)
		{
		char *end = nullptr;
		const long d = strtol(p, &end, 10);
		if (end == p || d < 0 || d > 4096)
			return false;
		out.push_back((int) d);
		if (*end == 0)
			return true;
		if (*end != ',')
			return false;
		p = end + 1;
		}
	}

extern "C" {

const char *mb200_group_last_error(const mb200_group *g) { return g ? g->err : g_group_create_error; }

int mb200_group_create(int ndev, const int *devices, mb200_group **out)
	{
	if (!out)
		return gfail(nullptr, MB200_EINVAL, "mb200_group_create: out is NULL");
	*out = nullptr;
	int have = 0;
	if (cudaGetDeviceCount(&have) != cudaSuccess || have == 0)
		{
		cudaGetLastError();
		return gfail(nullptr, MB200_ENODEV, "no CUDA device; libmuscle_b200 has no CPU path");
		}
	std::vector<int> devs;
	// MB200_DEVICE_LIST=a,b,...: the members of a group whose caller leaves the devices to the library,
	// one per listed device.  Repeats are allowed: every member is its own context, and a same-device peer
	// copy is a device-to-device copy, so a list like 0,0,0 runs the sharded path on one GPU.
	const char *list = devices == nullptr ? getenv("MB200_DEVICE_LIST") : nullptr;
	if (list != nullptr)
		{
		if (!parse_device_list(list, devs))
			return gfail(nullptr, MB200_EINVAL, "MB200_DEVICE_LIST=%s: expected comma-separated device numbers", list);
		}
	else if (ndev <= 0 || devices == nullptr)
		{
		const int n = ndev <= 0 ? have : std::min(ndev, have);
		for (int d = 0; d < n; ++d)
			devs.push_back(d);
		}
	else
		devs.assign(devices, devices + ndev);
	mb200_group *g = new mb200_group();
	g->err[0] = 0;
	// one thread per device: CUDA context creation is ~0.5 s per GPU and would otherwise be serial
	g->ctx.assign(devs.size(), nullptr);
	std::vector<int> rcs(devs.size(), MB200_OK);
		{
		std::vector<std::thread> th;
		for (size_t k = 0; k < devs.size(); ++k)
			th.emplace_back([&, k] { rcs[k] = mb200_create(devs[k], &g->ctx[k]); });
		for (auto &t : th)
			t.join();
		}
	for (size_t k = 0; k < devs.size(); ++k)
		if (rcs[k] != MB200_OK)
			{
			const int rc = rcs[k];
			gfail(nullptr, rc, "device %d: %s", devs[k], mb200_last_error(nullptr));
			for (mb200_ctx *o : g->ctx)
				if (o)
					mb200_destroy(o);
			delete g;
			return rc;
			}
	g->ndev = (int) g->ctx.size();
	// peer access between every pair of devices (NVLink / NVSwitch); without it the copies below
	// would be staged through the host
	// (one thread per source device: enabling a peer mapping takes ~0.1 s and there are ndev*(ndev-1) of them)
		{
		std::vector<std::thread> th;
		for (int a = 0; a < g->ndev; ++a)
			th.emplace_back([&, a]
				{
				cudaSetDevice(devs[a]);
				for (int b = 0; b < g->ndev; ++b)
					{
					if (a == b)
						continue;
					int can = 0;
					cudaDeviceCanAccessPeer(&can, devs[a], devs[b]);
					if (can && cudaDeviceEnablePeerAccess(devs[b], 0) != cudaSuccess)
						cudaGetLastError();          // already enabled is fine
					}
				});
		for (auto &t : th)
			t.join();
		}
	g->lo.assign(g->ndev, 0);
	g->hi.assign(g->ndev, 0);
	*out = g;
	return MB200_OK;
	}

void mb200_group_destroy(mb200_group *g)
	{
	if (!g)
		return;
	for (mb200_ctx *c : g->ctx)
		mb200_destroy(c);
	delete g;
	}

int mb200_group_size(const mb200_group *g) { return g ? g->ndev : 0; }

mb200_ctx *mb200_group_ctx(mb200_group *g, int rank)
	{
	return (g && rank >= 0 && rank < g->ndev) ? g->ctx[rank] : nullptr;
	}

int mb200_group_get_stats(const mb200_group *g, mb200_group_stats *out)
	{
	if (!g || !out)
		return MB200_EINVAL;
	*out = g->stats;
	return MB200_OK;
	}

int mb200_group_set_hmm(mb200_group *g, const float start[5], const float trans[25], const float ins[256],
  const float match[65536], float min_sparse_score)
	{
	if (!g)
		return MB200_EINVAL;
	return on_all(g, [&](int r) { return mb200_set_hmm(g->ctx[r], start, trans, ins, match, min_sparse_score); });
	}

int mb200_group_set_seqs(mb200_group *g, uint32_t nseq, const uint8_t *bytes, const uint64_t *offsets)
	{
	if (!g)
		return MB200_EINVAL;
	g->sharded = false;
	return on_all(g, [&](int r) { return mb200_set_seqs(g->ctx[r], nseq, bytes, offsets); });
	}

int mb200_group_set_seqs_mega(mb200_group *g, uint32_t nseq, const uint8_t *letters, const uint64_t *offsets,
  uint32_t nfeat, const uint32_t *alpha, const float *weights, const float *logprobs, const float *logprobmx)
	{
	if (!g)
		return MB200_EINVAL;
	g->sharded = false;
	return on_all(g, [&](int r)
		{ return mb200_set_seqs_mega(g->ctx[r], nseq, letters, offsets, nfeat, alpha, weights, logprobs, logprobmx); });
	}

// contiguous ranges of the row-major pair list with ~equal DP cells (sum of LX*LY) per device
static void shard_pairs(const std::vector<uint32_t> &len, int ndev, std::vector<uint32_t> &lo, std::vector<uint32_t> &hi)
	{
	const uint32_t n = (uint32_t) len.size();
	double total = 0;
	for (uint32_t i = 0; i < n; ++i)
		for (uint32_t j = i + 1; j < n; ++j)
			total += (double) len[i]*len[j];
	lo.assign(ndev, 0);
	hi.assign(ndev, 0);
	double run = 0;
	uint32_t p = 0;
	int r = 0;
	for (uint32_t i = 0; i < n; ++i)
		for (uint32_t j = i + 1; j < n; ++j, ++p)
			{
			// pair p belongs to the first rank whose quota is not yet filled
			while (r + 1 < ndev && run >= total*(r + 1)/ndev)
				{
				hi[r] = p;
				++r;
				lo[r] = p;
				}
			run += (double) len[i]*len[j];
			}
	hi[r] = p;
	for (int q = r + 1; q < ndev; ++q)
		lo[q] = hi[q] = p;
	}

int mb200_group_posteriors_allpairs(mb200_group *g, float *ea_out)
	{
	if (!g || g->ndev == 0)
		return MB200_EINVAL;
	mb200_ctx *c0 = g->ctx[0];
	const uint32_t n = c0->nseq;
	if (n < 2)
		return gfail(g, MB200_EINVAL, "mb200_group_posteriors_allpairs: need >= 2 sequences");
	const uint64_t all = (uint64_t) n*(n - 1)/2;
	g->stats = {};
	g->stats.ndev = (uint32_t) g->ndev;
	shard_pairs(c0->h_len, g->ndev, g->lo, g->hi);
	double t0 = now_ms();
	int rc = on_all(g, [&](int r)
		{
		if (g->hi[r] == g->lo[r])
			return (int) MB200_OK;
		return mb200_posteriors_allpairs(g->ctx[r], g->lo[r], g->hi[r], ea_out ? ea_out + g->lo[r] : nullptr);
		});
	if (rc != MB200_OK)
		return rc;
	g->stats.posterior_ms = (float)(now_ms() - t0);
	for (int r = 0; r < g->ndev; ++r)
		if (g->hi[r] > g->lo[r])
			g->stats.cells += g->ctx[r]->stats.cells;
	g->sharded = true;
	if (g->ndev == 1)
		return MB200_OK;

	// ---- exchange 1: all-gather-v of the packed store images over peer memory
	t0 = now_ms();
	std::vector<const uint32_t *> src_off(g->ndev, nullptr);
	std::vector<const mb200_entry *> src_ent(g->ndev, nullptr);
	std::vector<uint64_t> n_off(g->ndev, 0), n_ent(g->ndev, 0);
	rc = on_all(g, [&](int r)
		{
		if (g->hi[r] == g->lo[r])
			return (int) MB200_OK;
		return mb200_store_pack(g->ctx[r], &src_off[r], &n_off[r], &src_ent[r], &n_ent[r]);
		});
	if (rc != MB200_OK)
		return rc;
	g->off_pos.assign(g->ndev + 1, 0);
	g->ent_pos.assign(g->ndev + 1, 0);
	for (int r = 0; r < g->ndev; ++r)
		{
		g->off_pos[r + 1] = g->off_pos[r] + n_off[r];
		g->ent_pos[r + 1] = g->ent_pos[r] + n_ent[r];
		}
	std::vector<uint32_t *> dst_off(g->ndev, nullptr);
	std::vector<mb200_entry *> dst_ent(g->ndev, nullptr);
	// (in parallel: every device allocates buffers for the whole store here)
	rc = on_all(g, [&](int d)
		{ return mb200_store_exchange_begin(g->ctx[d], g->off_pos[g->ndev], g->ent_pos[g->ndev], &dst_off[d], &dst_ent[d]); });
	if (rc != MB200_OK)
		return rc;
	// one stream per SOURCE device carries its image to every destination (itself included)
	for (int r = 0; r < g->ndev; ++r)
		{
		if (n_off[r] == 0)
			continue;
		cudaSetDevice(g->ctx[r]->device);
		for (int k = 0; k < g->ndev; ++k)
			{
			const int d = (r + k) % g->ndev;          // stagger the destinations
			cudaMemcpyPeerAsync(dst_off[d] + g->off_pos[r], g->ctx[d]->device, src_off[r], g->ctx[r]->device,
			  n_off[r]*sizeof(uint32_t), g->ctx[r]->stream);
			if (n_ent[r])
				cudaMemcpyPeerAsync(dst_ent[d] + g->ent_pos[r], g->ctx[d]->device, src_ent[r], g->ctx[r]->device,
				  n_ent[r]*sizeof(mb200_entry), g->ctx[r]->stream);
			}
		}
	for (int r = 0; r < g->ndev; ++r)
		{
		cudaSetDevice(g->ctx[r]->device);
		const cudaError_t e = cudaStreamSynchronize(g->ctx[r]->stream);
		if (e != cudaSuccess)
			return gfail(g, MB200_ECUDA, "store exchange from device %d: %s", g->ctx[r]->device, cudaGetErrorString(e));
		}
	g->stats.exchange1_ms = (float)(now_ms() - t0);
	g->stats.exchange1_bytes_per_dev = (g->off_pos[g->ndev]*sizeof(uint32_t) + g->ent_pos[g->ndev]*sizeof(mb200_entry));
	rc = on_all(g, [&](int r) { return mb200_store_exchange_commit(g->ctx[r]); });
	if (rc != MB200_OK)
		return rc;
	(void) all;
	return MB200_OK;
	}

int mb200_group_consistency_iter(mb200_group *g)
	{
	if (!g || g->ndev == 0)
		return MB200_EINVAL;
	mb200_ctx *c0 = g->ctx[0];
	const uint32_t n = c0->nseq;
	const uint32_t np = (uint32_t)((uint64_t) n*(n - 1)/2);
	if (g->ndev == 1)
		{
		const double t0 = now_ms();
		const int rc = mb200_consistency_iter(c0, 0, np);
		if (rc != MB200_OK)
			return gfail(g, rc, "device %d: %s", c0->device, mb200_last_error(c0));
		g->stats.relax_ms = (float)(now_ms() - t0);
		g->stats.relax_kernel_ms = c0->stats.last_kernel_ms;
		return MB200_OK;
		}
	if (!g->sharded)
		return gfail(g, MB200_EINVAL, "mb200_group_consistency_iter: run mb200_group_posteriors_allpairs first");
	if (n < 3)
		return MB200_OK;
	double t0 = now_ms();
	int rc = on_all(g, [&](int r) { return mb200_consistency_iter(g->ctx[r], g->lo[r], g->hi[r]); });
	if (rc != MB200_OK)
		return rc;
	g->stats.relax_ms = (float)(now_ms() - t0);
	float km = 0;
	for (int r = 0; r < g->ndev; ++r)
		km = std::max(km, g->ctx[r]->stats.last_kernel_ms);
	g->stats.relax_kernel_ms = km;
	// ---- exchange 2: every device sends the entries of its pair range to all peers, in place
	t0 = now_ms();
	std::vector<mb200_entry *> ent(g->ndev, nullptr);
	for (int r = 0; r < g->ndev; ++r)
		{
		uint64_t ne = 0;
		rc = mb200_store_entries_ptr(g->ctx[r], &ent[r], &ne);
		if (rc != MB200_OK)
			return gfail(g, rc, "device %d: %s", g->ctx[r]->device, mb200_last_error(g->ctx[r]));
		}
	uint64_t bytes = 0;
	for (int r = 0; r < g->ndev; ++r)
		{
		if (g->hi[r] == g->lo[r])
			continue;
		mb200_ctx *c = g->ctx[r];
		uint64_t e_lo = 0, e_hi = 0;
		mb_store_entry_range(c, g->lo[r], g->hi[r], &e_lo, &e_hi);
		if (e_hi == e_lo)
			continue;
		bytes += (e_hi - e_lo)*sizeof(mb200_entry);
		cudaSetDevice(c->device);
		for (int k = 1; k < g->ndev; ++k)
			{
			const int d = (r + k) % g->ndev;
			cudaMemcpyPeerAsync(ent[d] + e_lo, g->ctx[d]->device, ent[r] + e_lo, c->device, (e_hi - e_lo)*sizeof(mb200_entry),
			  c->stream);
			}
		}
	for (int r = 0; r < g->ndev; ++r)
		{
		cudaSetDevice(g->ctx[r]->device);
		const cudaError_t e = cudaStreamSynchronize(g->ctx[r]->stream);
		if (e != cudaSuccess)
			return gfail(g, MB200_ECUDA, "values exchange from device %d: %s", g->ctx[r]->device, cudaGetErrorString(e));
		mb200_store_values_changed(g->ctx[r]);
		}
	g->stats.exchange2_ms = (float)(now_ms() - t0);
	g->stats.exchange2_bytes_per_dev = bytes;
	return MB200_OK;
	}

} // extern "C"
