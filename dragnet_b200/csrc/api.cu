/*
 * api.cu: the C ABI of libdragnet_gpu.so (include/dragnet_gpu.h), but for
 * compressed input (compressed.cu).
 *
 * Host-side plumbing only: device buffers, the H2D ring that keeps PCIe busy
 * while the previous chunk is being scanned, line carry between chunks
 * (lstream semantics, lib/format-json.js:32-33), kernel launches, result
 * download.  There is deliberately no host execution path for records: if no
 * CUDA device is usable, dng_scan_open() fails.
 */
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <map>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <cerrno>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/dragnet_gpu.h"
#include "plan.h"
#include "result.h"
#include "scan.h"
#include "scan_kernel.cuh"
#include "fast_kernel.cuh"
#include "jit.h"
#include "jit_cache.h"
#include "gen.cuh"
#include "direct_read.h"

using namespace dng;

namespace {

const size_t CARRY_ROOM = (size_t)DNG_MAXREC + 4096;	/* room before a chunk */
const size_t DNG_ARENA_MAX = (size_t)2 << 30;	/* largest DNG_ARENA_BYTES */

size_t env_size(const char *name, size_t dflt)
{
	const char *v = getenv(name);
	if (!v || !*v)
		return dflt;
	return (size_t)strtoull(v, nullptr, 0);
}

/*
 * Scan buffers (table, key arena, carry, H2D ring, pinned staging) have the
 * same few sizes for every scan, and cudaMalloc / cudaMallocHost / cudaFree
 * cost milliseconds each: destroyed scans park their buffers here and the
 * next scan on that device takes them back.  Bounded (DNG_CACHE_BYTES, default
 * 2 GiB per kind); dng_release_cached() empties it.
 */
struct BufCache {
	std::mutex mu;
	std::multimap<std::pair<int, size_t>, void *> idle;	/* (device|-1 host, bytes) */
	std::map<void *, std::pair<int, size_t>> live;
	size_t idle_dev = 0, idle_host = 0;
};

BufCache &buf_cache()
{
	static BufCache *c = new BufCache();	/* outlives static destructors */
	return *c;
}

cudaError_t cached_alloc(int device, void **p, size_t n)
{
	BufCache &c = buf_cache();
	{
		std::lock_guard<std::mutex> g(c.mu);
		auto it = c.idle.find(std::make_pair(device, n));
		if (it != c.idle.end()) {
			*p = it->second;
			c.idle.erase(it);
			(device < 0 ? c.idle_host : c.idle_dev) -= n;
			c.live[*p] = std::make_pair(device, n);
			return cudaSuccess;
		}
	}
	cudaError_t e = device < 0 ? cudaMallocHost(p, n) : cudaMalloc(p, n);
	if (e == cudaSuccess) {
		std::lock_guard<std::mutex> g(c.mu);
		c.live[*p] = std::make_pair(device, n);
	}
	return e;
}

void cached_free(void *p)
{
	if (!p)
		return;
	static const size_t limit = env_size("DNG_CACHE_BYTES", (size_t)2 << 30);
	BufCache &c = buf_cache();
	int device = 0;
	{
		std::lock_guard<std::mutex> g(c.mu);
		auto it = c.live.find(p);
		if (it == c.live.end())
			return;
		device = it->second.first;
		size_t n = it->second.second;
		c.live.erase(it);
		size_t &idle = device < 0 ? c.idle_host : c.idle_dev;
		if (idle + n <= limit) {
			idle += n;
			c.idle.insert(std::make_pair(std::make_pair(device, n), p));
			return;
		}
	}
	if (device < 0)
		cudaFreeHost(p);
	else
		cudaFree(p);
}

void set_err(char *err, size_t errlen, const char *fmt, const char *a = "")
{
	if (err && errlen)
		snprintf(err, errlen, fmt, a);
}

} /* namespace */

/* the same buffer cache for the library's other translation units (scan.h) */
cudaError_t dng_cached_alloc(int device, void **p, size_t n)
{
	return cached_alloc(device, p, n);
}

void dng_cached_free(void *p)
{
	cached_free(p);
}

cudaEvent_t get_event(dng_scan *s)
{
	if (!s->ev_pool.empty()) {
		cudaEvent_t e = s->ev_pool.back();
		s->ev_pool.pop_back();
		return e;
	}
	cudaEvent_t e;
	cudaEventCreate(&e);
	return e;
}

namespace {

/* shared memory set aside for the template trie when sizing the tally cache */
static constexpr size_t TMPL_RESERVE = 4096;

/* the record parser's view of one sample line per template candidate */
__global__ void resolve_pairs_kernel(const DevPlan *plan, const u8 *lines,
    const u32 *se, u32 n, TResolved *out)
{
	u32 i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n)
		return;
	RecState R;
	parse_record(lines + se[2 * i], se[2 * i + 1] - se[2 * i], *plan, R);
	out[i].flags = R.flags;
	out[i].set_mask = R.set_mask;
	for (int k = 0; k < MAX_SLOTS; k++)
		out[i].slots[k] = ((R.set_mask >> k) & 1) ? R.slots[k] : 0;
}

/*
 * A trie blob (tmpl_build, at most TMPL_RESERVE bytes) into a new device buffer
 * `*dst`, padded to 128 bytes, through half `half` of the pinned staging.  No
 * wait: the stream orders the copy before every launch that reads the blob.
 * A half is written again only after the stream has been waited for (the F
 * half by the next learn, the general half by the build after the next learn),
 * so the copy out of it has finished by then.
 */
int upload_blob(dng_scan *s, int half, std::vector<u8> &blob, u8 **dst)
{
	const size_t padded = (blob.size() + 127) & ~(size_t)127;
	blob.resize(padded, 0);
	if (!s->h_blobs)
		CK(s, HOST_ALLOC(&s->h_blobs, 2 * TMPL_RESERVE));
	u8 *stage = s->h_blobs + half * TMPL_RESERVE;
	memcpy(stage, blob.data(), padded);
	CK(s, DEV_ALLOC(s, dst, padded));
	CK(s, cudaMemcpyAsync(*dst, stage, padded, cudaMemcpyHostToDevice,
	    s->stream));
	return 0;
}

/*
 * Do the accepted templates' sample lines all have short group keys (fast.cuh
 * FKey)?  What the compiled kernel keeps in its record loop depends on it
 * (FPlan::short_keys); what it counts does not.
 */
static bool fsample_keys_short(const FPlan &F,
    const std::vector<TResolved> &fres, const std::vector<u8> &accepted)
{
	if (F.ncols > FK_COLS)
		return false;
	for (size_t i = 0; i < fres.size(); i++) {
		if (!accepted[i])
			continue;
		for (u32 j = 0; j < F.ncols; j++) {
			const Col &col = F.col[j];
			if (col.kind != COL_DISCRETE)
				continue;
			/* (undefined is 9 bytes) */
			if (col.src.kind != SRC_PATH ||
			    !((fres[i].set_mask >> col.src.idx) & 1))
				return false;
			const u64 v = fres[i].slots[col.src.idx];
			const u32 t = val_type(v);
			if ((t == T_STR || t == T_NUM) && val_len(v) > FK_W)
				return false;
		}
	}
	return true;
}

/*
 * The F path's templates (fast.h): the same candidates, their captures indexed
 * by path, compact literals.  `blob` keeps them for the compiled matcher, `t`
 * says what they cover of the sample.
 */
int learn_ftemplates(dng_scan *s, const std::vector<TCandidate> &cands,
    const std::vector<TResolved> &res, size_t sampled_lines,
    std::vector<u8> &blob, KcTemplates &t)
{
	std::vector<TResolved> fres(res.size());
	for (size_t i = 0; i < res.size(); i++)
		fplan_resolve(s->plan.dev, res[i], fres[i]);
	std::vector<u8> accepted;
	u32 nt = 0;
	tmpl_build(cands, fres, TMPL_RESERVE, blob, &nt, true, &accepted);
	s->fplan.short_keys = !blob.empty() &&
	    fsample_keys_short(s->fplan, fres, accepted);
	cached_free(s->d_ftmpl);
	s->d_ftmpl = nullptr;
	s->ftmpl_bytes = 0;
	s->nftemplates = 0;
	if (!blob.empty()) {
		const THdr *th = (const THdr *)blob.data();
		s->ftmpl_leaf_off = th->leaf_off;
		s->ftmpl_pool_off = th->pool_off;
	}
	t.learned = true;
	t.blob = !blob.empty();
	t.lines = sampled_lines;
	for (size_t i = 0; i < cands.size(); i++)
		if (accepted[i])
			t.covered += cands[i].count;
	if (!blob.empty()) {
		/* (the blob this replaces was freed above, after the resolve
		 * waited for the stream: no launch was reading it) */
		if (upload_blob(s, 0, blob, &s->d_ftmpl))
			return s->err_code;
		s->ftmpl_bytes = (u32)blob.size();
		s->nftemplates = nt;
	}
	return 0;
}

/*
 * The general kernels' blob from the learns since it was last built: the
 * latest learn whose candidates give one, as if every learn had built its own
 * and one that gives none had left the previous blob in place.
 */
void general_blob(const dng_scan *s, std::vector<u8> &blob, u32 *nt)
{
	blob.clear();
	*nt = 0;
	for (size_t i = s->tmpl_pending.size(); i-- > 0 && blob.empty();)
		tmpl_build(s->tmpl_pending[i].first, s->tmpl_pending[i].second,
		    TMPL_RESERVE, blob, nt);
}

/* d_tmpl for a general launch, if learns since the last build left any */
int build_general(dng_scan *s)
{
	if (s->tmpl_pending.empty())
		return 0;
	std::vector<u8> blob;
	u32 nt = 0;
	general_blob(s, blob, &nt);
	s->tmpl_pending.clear();
	if (blob.empty())
		return 0;
	/*
	 * Only general launches read d_tmpl, and every one since it was last
	 * built came before the learn that queued this build, which waited for
	 * the stream: the blob being replaced is not in use, even with F
	 * launches still running.
	 */
	cached_free(s->d_tmpl);
	s->d_tmpl = nullptr;
	s->tmpl_bytes = 0;
	if (upload_blob(s, 1, blob, &s->d_tmpl))
		return s->err_code;
	s->tmpl_bytes = (u32)blob.size();
	s->ntemplates = nt;
	return 0;
}

/*
 * Record templates from a sample (host memory): skeletons on the host
 * (lexical only), what their wildcards mean to the plan from the device's own
 * parser.  Failure to learn anything is not an error: the kernel then parses
 * every record itself.
 */
int build_templates(dng_scan *s, const u8 *head, size_t n,
    std::vector<u8> &fblob, KcTemplates &ft)
{
	std::vector<TCandidate> cands;
	size_t sampled_lines = 0;
	tmpl_candidates(head, n, TMPL_MAX_LEAVES, cands, &sampled_lines);
	if (cands.empty())
		return 0;
	std::vector<u8> lines;
	std::vector<u32> offs(1, 0);
	for (const TCandidate &c : cands) {
		lines.insert(lines.end(), c.sample.begin(), c.sample.end());
		lines.push_back('\n');
		offs.push_back((u32)lines.size());
	}
	u8 *d_lines = nullptr;
	u32 *d_offs = nullptr;
	TResolved *d_res = nullptr;
	std::vector<TResolved> res(cands.size());
	/* constant sizes, so that the buffer cache can hand them back */
	cudaError_t e = DEV_ALLOC(s, &d_lines,
	    (size_t)TMPL_MAX_LEAVES * (TMPL_MAX_LINE + 1) + 16);
	if (e == cudaSuccess)
		e = DEV_ALLOC(s, &d_offs, 2 * (TMPL_MAX_LEAVES + 1) * sizeof (u32));
	if (e == cudaSuccess)
		e = DEV_ALLOC(s, &d_res, TMPL_MAX_LEAVES * sizeof (TResolved));
	if (e == cudaSuccess)
		e = cudaMemcpyAsync(d_lines, lines.data(), lines.size(),
		    cudaMemcpyHostToDevice, s->stream);
	/* line i = [offs[i], offs[i + 1] - 1): keep starts and ends apart */
	std::vector<u32> se;
	for (size_t i = 0; i < cands.size(); i++) {
		se.push_back(offs[i]);
		se.push_back(offs[i + 1] - 1);
	}
	if (e == cudaSuccess)
		e = cudaMemcpyAsync(d_offs, se.data(), se.size() * sizeof (u32),
		    cudaMemcpyHostToDevice, s->stream);
	if (e == cudaSuccess) {
		s->aux_launches++;
		resolve_pairs_kernel<<<1, 32, 0, s->stream>>>(s->d_plan, d_lines,
		    d_offs, (u32)cands.size(), d_res);
		e = cudaGetLastError();
	}
	if (e == cudaSuccess)
		e = cudaMemcpyAsync(res.data(), d_res,
		    res.size() * sizeof (TResolved), cudaMemcpyDeviceToHost,
		    s->stream);
	if (e == cudaSuccess)
		e = cudaStreamSynchronize(s->stream);
	cached_free(d_lines);
	cached_free(d_offs);
	cached_free(d_res);
	if (e != cudaSuccess)
		return s->cuda(e, "template resolve");
	if (s->kc.f_ok && learn_ftemplates(s, cands, res, sampled_lines, fblob,
	    ft))
		return s->err_code;
	s->tmpl_pending.emplace_back(std::move(cands), std::move(res));
	return 0;
}

/*
 * Sample the head of data[start, nbytes) (device memory): its lines set the
 * kernel geometry, its records the templates.  `sample`: that head already
 * copied to host memory by the caller (with the stream waited for since), or
 * null.
 */
int learn_templates(dng_scan *s, const u8 *data, unsigned long long start,
    unsigned long long nbytes, const u8 *sample)
{
	s->tmpl_tried = true;
	if (!kc_wants_sample(s->kc, s->tmpl_enabled))
		return 0;
	size_t n = (size_t)std::min<unsigned long long>(nbytes - start,
	    TMPL_SAMPLE_BYTES);
	/* pinned (and cached) so that the copy is a plain DMA */
	u8 *hbuf = nullptr;
	struct Release {
		u8 *p;
		~Release() { cached_free(p); }
	} release{nullptr};
	if (!sample) {
		CK(s, HOST_ALLOC(&hbuf, TMPL_SAMPLE_BYTES));
		release.p = hbuf;
		CK(s, cudaMemcpyAsync(hbuf, data + start, n,
		    cudaMemcpyDeviceToHost, s->stream));
		CK(s, cudaStreamSynchronize(s->stream));
		sample = hbuf;
	}
	std::vector<u8> fblob;
	KcTemplates ft;
	if (s->tmpl_enabled && build_templates(s, sample, n, fblob, ft))
		return s->err_code;
	kc_sample(s->kc, sample, n, ft);
	if (ft.learned) {
		s->jit.reset();
		if (s->jit_mode && !fblob.empty())
			s->jit = jit_request(fblob.data(), fblob.size(),
			    &s->fplan, (int)s->kc.f_nsl, s->device,
			    (int)s->f_smem_max, s->jit_mode == 2);
	}
	return 0;
}

/* tier 2 of a tally cache: as many compact slots as fit in `room` (a power of
 * two) */
u32 tier2_slots(size_t room)
{
	u32 n = DNG_SSLOTS_MIN;
	while (n * 2 <= DNG_SSLOTS_MAX && (size_t)n * 2 * sizeof (SSlot) <= room)
		n *= 2;
	return n;
}

/* the F kernel for lane slices of nsl x 16 bytes */
const void *fkernel(u32 nsl)
{
	switch (nsl) {
	case 7:
		return (const void *)scan_kernel_f<7>;
	case 9:
		return (const void *)scan_kernel_f<9>;
	case 11:
		return (const void *)scan_kernel_f<11>;
	default:
		return (const void *)scan_kernel_f<13>;
	}
}

/* after a scan launch: its timing, the pinned copy of the counters the next
 * launch decides on, the counts */
void launched(dng_scan *s, cudaEvent_t e0, unsigned long long bytes)
{
	cudaEvent_t e1 = get_event(s);
	cudaEventRecord(e1, s->stream);
	if (!s->h_live && HOST_ALLOC(&s->h_live, NCTR * sizeof (unsigned long long))
	    == cudaSuccess)
		memset(s->h_live, 0, NCTR * sizeof (unsigned long long));
	if (s->h_live)
		cudaMemcpyAsync(s->h_live, s->d_counters,
		    NCTR * sizeof (unsigned long long), cudaMemcpyDeviceToHost,
		    s->stream);
	s->ev_pairs.emplace_back(e0, e1);
	s->launches++;
	s->kernel_bytes += bytes;
}

/*
 * The F path over data[start, nbytes): scan_kernel_f, then scan_miss_kernel
 * for what it did not take (it exits at once when the list is empty).
 */
int launch_fscan(dng_scan *s, const u8 *data, unsigned long long start,
    unsigned long long nbytes, bool final)
{
	if (!s->d_miss) {
		s->miss_cap = (u32)env_size("DNG_MISS_CAP", (size_t)4 << 20);
		CK(s, DEV_ALLOC(s, &s->d_miss, (size_t)s->miss_cap *
		    sizeof (MissEnt)));
		CK(s, DEV_ALLOC(s, &s->d_miss_n, 64));
		CK(s, cudaMemsetAsync(s->d_miss_n, 0, 64, s->stream));
	}
	/* the kernel wants the first valid byte inside the first 16 */
	const unsigned long long skip = start & ~15ull;
	data += skip;
	start -= skip;
	nbytes -= skip;
	FScanArgs a;
	a.data = data;
	a.start = start;
	a.nbytes = nbytes;
	a.fplan = s->d_fplan;
	a.plan = s->d_plan;
	a.tmpl = s->d_ftmpl;
	a.tmpl_bytes = s->ftmpl_bytes;
	a.leaf_off = s->ftmpl_leaf_off;
	a.pool_off = s->ftmpl_pool_off;
	a.counters = s->d_counters;
	a.tab = s->tab;
	a.final = final ? 1 : 0;
	a.nrows = s->fplan.nrows;
	a.miss = s->d_miss;
	a.miss_cap = s->miss_cap;
	a.miss_n = s->d_miss_n;
	const u32 nsl = s->kc.f_nsl;
	const unsigned long long chunk = 32ull * 16 * nsl;
	a.nchunks = (u32)((nbytes + chunk - 1) / chunk);
	const u32 nw = s->kc.f_nw;
	const u32 grid = std::min<u32>((a.nchunks + nw - 1) / nw,
	    (u32)s->sm_count);
	/* segments: long enough to amortise the pre-lap, short enough to keep
	 * every warp of the grid busy */
	const u32 nwarps = grid * nw;
	a.seg = std::max<u32>(1, std::min<u32>(DNG_F_SEG,
	    a.nchunks / (nwarps * 8)));
	/* the segment queue: [1] of the miss counter's allocation */
	a.seg_next = s->d_miss_n + 1;
	cudaMemsetAsync(s->d_miss_n, 0, 2 * sizeof (u32), s->stream);
	cudaEvent_t e0 = get_event(s);
	cudaEventRecord(e0, s->stream);
	/* the matcher compiled for these templates, once it is there */
	const bool jit = s->jit && s->jit->state.load() == 1 && s->ftmpl_bytes;
	a.wunits = fwindow_units(nsl, nw);
	const u32 warp_bytes = fwarp_bytes(a.wunits);
	const void *kern = fkernel(nsl);
	/* (the compiled matcher has the templates in its code: no trie in shared
	 * memory, more of it for the tally cache) */
	const u32 tmpl_room = jit ? 0 : (u32)TMPL_RESERVE;
	if (jit) {
		kern = (const void *)s->jit->kern;
		a.tmpl_bytes = 0;
		s->jit_launches++;
	}
	/* the tally cache takes what the buffers leave, its first tier up to
	 * three quarters of that */
	const size_t fixed = fkernel_smem(warp_bytes, tmpl_room, 0, 0, a.nrows, nw);
	const size_t room = s->f_smem_max > fixed ? s->f_smem_max - fixed : 0;
	a.s1slots = 32;
	while (a.s1slots < 1024 && (size_t)a.s1slots * 2 * sizeof (SSlot1) +
	    DNG_SSLOTS_MIN * sizeof (SSlot) <= room * 3 / 4)
		a.s1slots *= 2;
	a.sslots = tier2_slots(room - std::min(room,
	    (size_t)a.s1slots * sizeof (SSlot1)));
	void *args[] = { &a };
	cudaError_t le = cudaLaunchKernel(kern, dim3(grid), dim3(32 * nw), args,
	    fkernel_smem(warp_bytes, a.tmpl_bytes, a.s1slots, a.sslots, a.nrows,
	    nw), s->stream);
	if (le == cudaSuccess)
		le = cudaGetLastError();
	FMissArgs ma;
	ma.data = data;
	ma.start = start;
	ma.plan = s->d_plan;
	ma.plan_bytes = s->plan_bytes;
	ma.counters = s->d_counters;
	ma.tab = s->tab;
	ma.s1slots = 64;
	ma.sslots = 1024;
	ma.miss = s->d_miss;
	ma.miss_n = s->d_miss_n;
	ma.miss_cap = s->miss_cap;
	if (le == cudaSuccess) {
		scan_miss_kernel<<<s->sm_count * 2, DNG_MISS_NT, s->plan_bytes +
		    ma.s1slots * sizeof (SSlot1) + ma.sslots * sizeof (SSlot),
		    s->stream>>>(ma);
		le = cudaGetLastError();
	}
	launched(s, e0, nbytes - start);
	s->aux_launches++;
	return s->cuda(le, "scan_kernel_f launch");
}

/* launch the scan kernel over data[start, nbytes); `sample`: see
 * learn_templates */
int launch_scan(dng_scan *s, const u8 *data, unsigned long long start,
    unsigned long long nbytes, bool final, const u8 *sample = nullptr)
{
	if (nbytes <= start)
		return 0;
	if (!s->tmpl_tried) {
		if (learn_templates(s, data, start, nbytes, sample))
			return s->err_code;
	} else if (s->h_live) {
		const volatile unsigned long long *lv = s->h_live;
		const KcLive live = { lv[CTR_LINES], lv[CTR_LONG], lv[CTR_TMPL],
		    lv[CTR_AGGR], lv[CTR_OVER] };
		if (kc_counters(s->kc, live, s->tmpl_enabled)) {
			if (learn_templates(s, data, start, nbytes, nullptr))
				return s->err_code;
			/* the stream was waited for after the last launch (the
			 * blob uploads since touch no counter): the counters
			 * below are current */
			s->kc.learn_lines = lv[CTR_LINES];
			s->kc.learn_tmpl = lv[CTR_TMPL];
		}
	}
	const int kind = kc_pick(s->kc);
	if (kind == KK_F)
		return launch_fscan(s, data, start, nbytes, final);
	if (build_general(s))
		return s->err_code;
	ScanArgs a;
	a.data = data;
	a.start = start;
	a.nbytes = nbytes;
	a.plan = s->d_plan;
	a.counters = s->d_counters;
	a.tab = s->tab;
	a.final = final ? 1 : 0;
	a.plan_bytes = s->plan_bytes;
	a.tmpl = s->d_tmpl;
	a.tmpl_bytes = s->tmpl_bytes;
	a.wslice = DNG_W_SLICE_MAX;
	cudaEvent_t e0 = get_event(s);
	cudaEventRecord(e0, s->stream);
	if (kind == KK_WARP) {
		const unsigned long long chunk = 32ull * s->kc.wslice;
		a.wslice = s->kc.wslice;
		a.ntiles = (u32)((nbytes + chunk - 1) / chunk);
		a.sslots = s->w_sslots;
		a.s1slots = s->w_s1slots;
		u32 grid = std::min<u32>((a.ntiles + DNG_NW - 1) / DNG_NW,
		    (u32)s->sm_count);
		scan_kernel_w<<<grid, DNG_NT, SMEM_W_FIXED + s->plan_bytes +
		    s->tmpl_bytes + a.sslots * sizeof (SSlot) +
		    a.s1slots * sizeof (SSlot1), s->stream>>>(a);
	} else {
		a.ntiles = (u32)((nbytes + DNG_TILE - 1) / DNG_TILE);
		a.sslots = s->sslots;
		a.s1slots = s->s1slots;
		u32 grid = std::min<u32>(a.ntiles,
		    (u32)s->sm_count * DNG_CTAS_PER_SM);
		scan_kernel<<<grid, DNG_NT, SMEM_FIXED + s->plan_bytes +
		    s->tmpl_bytes + a.sslots * sizeof (SSlot) +
		    a.s1slots * sizeof (SSlot1), s->stream>>>(a);
	}
	launched(s, e0, nbytes - start);
	return s->cuda(cudaGetLastError(), "scan_kernel launch");
}

void drain_events(dng_scan *s)
{
	for (auto &p : s->ev_pairs) {
		float ms = 0;
		if (cudaEventElapsedTime(&ms, p.first, p.second) == cudaSuccess)
			s->kernel_ms += ms;
		s->ev_pool.push_back(p.first);
		s->ev_pool.push_back(p.second);
	}
	s->ev_pairs.clear();
}

/*
 * One piece of host input (<= ring_cap bytes) whose bytes up to `upto`
 * (exclusive; ends just after a newline) are complete lines.  The previous
 * carry is prepended on the device; bytes [upto, len) become the new carry.
 */
int feed_piece(dng_scan *s, const u8 *buf, size_t len, size_t upto, bool pinned)
{
	size_t slot = s->next_slot;
	s->next_slot = (slot + 1) % RING_SLOTS;
	if (s->slot_used[slot])
		CK(s, cudaEventSynchronize(s->ev_free[slot]));
	const u8 *src = buf;
	if (!pinned) {
		memcpy(s->h_stage[slot], buf, len);
		src = s->h_stage[slot];
	}
	u8 *dst = s->d_ring[slot] + CARRY_ROOM;
	CK(s, cudaMemcpyAsync(dst, src, len, cudaMemcpyHostToDevice,
	    s->copy_stream));
	CK(s, cudaEventRecord(s->ev_ready[slot], s->copy_stream));
	CK(s, cudaStreamWaitEvent(s->stream, s->ev_ready[slot], 0));
	if (upto > 0) {
		u8 *begin = dst - s->carry_len;
		if (s->carry_len)
			CK(s, cudaMemcpyAsync(begin, s->d_carry, s->carry_len,
			    cudaMemcpyDeviceToDevice, s->stream));
		u8 *base = (u8 *)((uintptr_t)begin & ~(uintptr_t)15);
		if (launch_scan(s, base, (unsigned long long)(begin - base),
		    (unsigned long long)(dst + upto - base), false))
			return s->err_code;
		s->carry_len = 0;
	}
	if (len > upto) {
		/* a line is refused once 16 MiB of it, before its newline, have
		 * to be carried (DESIGN.md section 4) */
		size_t tail = len - upto;
		if (s->carry_len + tail >= DNG_MAXREC)
			return s->fail(DNG_ELIMIT, "input line longer than 16 MiB");
		CK(s, cudaMemcpyAsync(s->d_carry + s->carry_len, dst + upto, tail,
		    cudaMemcpyDeviceToDevice, s->stream));
		s->carry_len += tail;
	}
	CK(s, cudaEventRecord(s->ev_free[slot], s->stream));
	s->slot_used[slot] = true;
	return 0;
}

int feed_host(dng_scan *s, const void *vbuf, size_t len, bool pinned)
{
	if (s->err_code)
		return s->err_code;
	if (s->finished)
		return s->fail(DNG_EINVAL, "scan already finished");
	const u8 *buf = (const u8 *)vbuf;
	s->bytes_fed += len;
	while (len > 0) {
		size_t n = std::min(len, s->ring_cap);
		/* complete lines end at the last '\n' of the piece */
		const void *nl = memrchr(buf, '\n', n);
		size_t upto = nl ? (size_t)((const u8 *)nl - buf) + 1 : 0;
		int rc = feed_piece(s, buf, n, upto, pinned);
		if (rc)
			return rc;
		buf += n;
		len -= n;
	}
	return 0;
}

} /* namespace */

const char *dng_version(void)
{
	return "dragnet-b200 0.1 (sm_90a)";
}

int dng_plan_create(const char *plan_json, dng_plan **out, char *err,
    size_t errlen)
{
	if (!plan_json || !out) {
		set_err(err, errlen, "null argument");
		return DNG_EINVAL;
	}
	dng_plan *p = new dng_plan();
	int rc = dng_plan_compile(plan_json, p, err, errlen);
	if (rc) {
		delete p;
		return rc;
	}
	*out = p;
	return DNG_OK;
}

void dng_plan_destroy(dng_plan *plan)
{
	delete plan;
}

int dng_device_count(void)
{
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess)
		return 0;
	return n;
}

int dng_scan_open(const dng_plan *plan, int device, dng_scan **out, char *err,
    size_t errlen)
{
	if (!plan || !out) {
		set_err(err, errlen, "null argument");
		return DNG_EINVAL;
	}
	int ndev = 0;
	cudaError_t e = cudaGetDeviceCount(&ndev);
	if (e != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
		set_err(err, errlen, "no usable CUDA device (%s); "
		    "libdragnet_gpu has no CPU fallback", e != cudaSuccess ?
		    cudaGetErrorString(e) : "device index out of range");
		return DNG_ENODEV;
	}
	dng_scan *s = new dng_scan();
	s->plan = *plan;
	s->device = device;
	int rc = 0;
	do {
		if ((rc = s->cuda(cudaSetDevice(device), "cudaSetDevice")))
			break;
		/* cudaGetDeviceProperties costs about a millisecond: once
		 * per device */
		static std::mutex prop_mu;
		static std::map<int, cudaDeviceProp> props;
		cudaDeviceProp prop;
		{
			std::lock_guard<std::mutex> g(prop_mu);
			auto it = props.find(device);
			if (it == props.end()) {
				if ((rc = s->cuda(cudaGetDeviceProperties(&prop,
				    device), "cudaGetDeviceProperties")))
					break;
				props[device] = prop;
			} else {
				prop = it->second;
			}
		}
		s->sm_count = prop.multiProcessorCount;
		if (const char *ev = getenv("DNG_TEMPLATES"))
			s->tmpl_enabled = atoi(ev) != 0;
		s->plan_bytes = devplan_smem_bytes(plan->dev);
		{
			/* the tally cache takes whatever shared memory is left
			 * when two CTAs share an SM (1 KB is reserved per CTA) */
			size_t per_cta = prop.sharedMemPerMultiprocessor /
			    DNG_CTAS_PER_SM - 1024 - 256;
			/* a single block may not exceed the opt-in limit, which
			 * also covers the kernel's static shared variables */
			per_cta = std::min(per_cta,
			    (size_t)prop.sharedMemPerBlockOptin - 1024 - 512);
			/* tier 1: 128 inline-key slots (64 when tight); tier 2:
			 * as many compact slots as still fit.  The per-warp
			 * kernel's fixed part differs: its own sizes */
			size_t used = SMEM_FIXED + s->plan_bytes + TMPL_RESERVE;
			size_t usedw = SMEM_W_FIXED + s->plan_bytes + TMPL_RESERVE;
			size_t room = per_cta > used ? per_cta - used : 0;
			size_t roomw = per_cta > usedw ? per_cta - usedw : 0;
			s->s1slots = room >= 24576 ? 256 : room >= 12288 ? 128 : 64;
			s->w_s1slots = roomw >= 24576 ? 256 : roomw >= 12288 ? 128 : 64;
			s->sslots = tier2_slots(room - std::min(room,
			    (size_t)s->s1slots * sizeof (SSlot1)));
			s->w_sslots = tier2_slots(roomw - std::min(roomw,
			    (size_t)s->w_s1slots * sizeof (SSlot1)));
		}
		/* the F path (fast.h), for the plans it models */
		fplan_build(plan->dev, s->fplan);
		if (const char *ev = getenv("DNG_JIT"))
			s->jit_mode = !strcmp(ev, "sync") || !strcmp(ev, "wait") ? 2 :
			    (!strcmp(ev, "0") || !strcmp(ev, "off")) ? 0 : 1;
		s->f_smem_max = (u32)prop.sharedMemPerBlockOptin - 1024;
		cudaError_t fe = cudaFuncSetAttribute(scan_miss_kernel,
		    cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s->f_smem_max);
		for (u32 nsl = 7; nsl <= 13 && fe == cudaSuccess; nsl += 2)
			fe = cudaFuncSetAttribute(fkernel(nsl),
			    cudaFuncAttributeMaxDynamicSharedMemorySize,
			    (int)s->f_smem_max);
		if ((rc = s->cuda(fe, "cudaFuncSetAttribute")))
			break;
		if ((rc = s->cuda(cudaFuncSetAttribute(scan_kernel,
		    cudaFuncAttributeMaxDynamicSharedMemorySize,
		    (int)prop.sharedMemPerBlockOptin - 1024),
		    "cudaFuncSetAttribute")))
			break;
		if ((rc = s->cuda(cudaFuncSetAttribute(scan_kernel_w,
		    cudaFuncAttributeMaxDynamicSharedMemorySize,
		    (int)prop.sharedMemPerBlockOptin - 1024),
		    "cudaFuncSetAttribute")))
			break;
		if (SMEM_FIXED + s->plan_bytes + TMPL_RESERVE +
		    s->sslots * sizeof (SSlot) + s->s1slots * sizeof (SSlot1) >
		    prop.sharedMemPerBlockOptin - 1024) {
			rc = s->fail(DNG_ELIMIT, "plan does not fit in shared "
			    "memory (fixed " + std::to_string(SMEM_FIXED) +
			    " + plan " + std::to_string(s->plan_bytes) +
			    " + tier2 " + std::to_string(s->sslots) + " + tier1 " +
			    std::to_string(s->s1slots) + " slots > " +
			    std::to_string(prop.sharedMemPerBlockOptin) + ")");
			break;
		}
		/* (a plan with many capture rows leaves the F kernel's buffers
		 * no room) */
		const u32 warp_bytes = fwarp_bytes(fwindow_units(13, DNG_F_NW));
		const bool f_fits = fkernel_smem(warp_bytes, TMPL_RESERVE, 32,
		    DNG_SSLOTS_MIN, s->fplan.nrows, DNG_F_NW) <= s->f_smem_max;
		const bool warp_fits = SMEM_W_FIXED + s->plan_bytes + TMPL_RESERVE +
		    s->w_sslots * sizeof (SSlot) + s->w_s1slots * sizeof (SSlot1) <=
		    prop.sharedMemPerBlockOptin - 1024;
		kc_open(s->kc, plan->dev.nmetrics > 1, s->fplan.ok != 0, f_fits,
		    warp_fits, getenv("DNG_KERNEL"), getenv("DNG_FAST"),
		    getenv("DNG_F_WARPS"));
		if ((rc = s->cuda(cudaStreamCreateWithFlags(&s->stream,
		    cudaStreamNonBlocking), "cudaStreamCreate")))
			break;
		s->own_stream = s->stream;
		if ((rc = s->cuda(cudaStreamCreateWithFlags(&s->copy_stream,
		    cudaStreamNonBlocking), "cudaStreamCreate")))
			break;
		if ((rc = s->cuda(DEV_ALLOC(s, &s->d_plan, sizeof (DevPlan) + 256),
		    "cudaMalloc plan")))
			break;
		if (s->kc.f_ok) {
			if ((rc = s->cuda(DEV_ALLOC(s, &s->d_fplan, FPLAN_SMEM),
			    "cudaMalloc fplan")))
				break;
			if ((rc = s->cuda(cudaMemcpyAsync(s->d_fplan, &s->fplan,
			    sizeof (FPlan), cudaMemcpyHostToDevice, s->stream),
			    "fplan upload")))
				break;
		}
		/* s->plan is this scan's own copy: safe to upload from */
		if ((rc = s->cuda(cudaMemcpyAsync(s->d_plan, &s->plan.dev,
		    sizeof (DevPlan), cudaMemcpyHostToDevice, s->stream),
		    "plan upload")))
			break;
		size_t cap = env_size("DNG_TABLE_CAP", (size_t)1 << 20);
		size_t c2 = 1024;
		while (c2 < cap)
			c2 <<= 1;
		s->table_cap = c2;
		size_t arena = env_size("DNG_ARENA_BYTES", (size_t)64 << 20);
		if (arena > DNG_ARENA_MAX) {
			/* key offsets and the bump offset are u32: refused, not
			 * truncated.  The offset passes the cap only by the keys
			 * claimed while the arena fills up (global_find: at most
			 * one per resident thread, 520 B each, < 160 MiB on an
			 * H100), which 2 GiB leaves room for whatever the table
			 * size */
			rc = s->fail(DNG_EINVAL, "DNG_ARENA_BYTES " +
			    std::to_string(arena) + " is larger than the key arena "
			    "can address (" + std::to_string(DNG_ARENA_MAX) + ")");
			break;
		}
		if ((rc = s->cuda(DEV_ALLOC(s, &s->tab.entries,
		    c2 * sizeof (GEntry)), "cudaMalloc table")))
			break;
		if ((rc = s->cuda(DEV_ALLOC(s, &s->tab.arena, arena),
		    "cudaMalloc arena")))
			break;
		if ((rc = s->cuda(DEV_ALLOC(s, &s->tab.misc, 16 * sizeof (u32)),
		    "cudaMalloc misc")))
			break;
		s->tab.mask = (u32)(c2 - 1);
		s->tab.arena_cap = (u32)arena;
		cudaMemsetAsync(s->tab.entries, 0, c2 * sizeof (GEntry), s->stream);
		cudaMemsetAsync(s->tab.misc, 0, 16 * sizeof (u32), s->stream);
		const size_t nctr = NCTR + (MAX_METRICS - 1) * MCTR_PER;
		if ((rc = s->cuda(DEV_ALLOC(s, &s->d_counters,
		    nctr * sizeof (unsigned long long)), "cudaMalloc counters")))
			break;
		cudaMemsetAsync(s->d_counters, 0,
		    nctr * sizeof (unsigned long long), s->stream);
		if ((rc = s->cuda(DEV_ALLOC(s, &s->d_nl,
		    2 * sizeof (unsigned long long)), "cudaMalloc nl")))
			break;
		if ((rc = s->cuda(DEV_ALLOC(s, &s->d_carry, CARRY_ROOM + 64),
		    "cudaMalloc carry")))
			break;
		s->ring_cap = env_size("DNG_RING_BYTES", (size_t)64 << 20);
		/* whichever stream the scan ends up on waits for this setup */
		if ((rc = s->cuda(cudaEventCreateWithFlags(&s->ev_init,
		    cudaEventDisableTiming), "cudaEventCreate")))
			break;
		rc = s->cuda(cudaEventRecord(s->ev_init, s->stream), "init");
	} while (0);
	if (rc) {
		set_err(err, errlen, "%s", s->err.c_str());
		dng_scan_destroy(s);
		return rc;
	}
	*out = s;
	set_err(err, errlen, "");
	return DNG_OK;
}

int dng_scan_open_devices(const dng_plan *plan, const int *devices, int n,
    dng_scan **out, char *err, size_t errlen)
{
	if (!plan || !devices || n <= 0 || !out) {
		set_err(err, errlen, "null argument or no devices");
		return DNG_EINVAL;
	}
	dng_scan *s = new dng_scan();
	s->plan = *plan;
	s->device = devices[0];
	s->multi = true;
	for (int k = 0; k < n; k++) {
		dng_scan *sh = nullptr;
		int rc = dng_scan_open(plan, devices[k], &sh, err, errlen);
		if (rc) {
			dng_scan_destroy(s);
			return rc;
		}
		s->shards.push_back(sh);
	}
	*out = s;
	return DNG_OK;
}

dng_scan *dng_scan_shard(const dng_scan *s, int i)
{
	if (!s || !s->multi || i < 0 || (size_t)i >= s->shards.size())
		return nullptr;
	return s->shards[i];
}

/* what a multi-device scan refuses: not sticky, the scan goes on */
int refuse_multi(dng_scan *s, const char *what)
{
	if (!s->err_code)
		s->err = std::string(what) + " on a scan over several devices "
		    "(it reads files only; per-shard state: dng_scan_shard)";
	return DNG_EINVAL;
}

int dng_scan_set_stream(dng_scan *s, void *cuda_stream)
{
	if (!s)
		return DNG_EINVAL;
	if (s->multi)
		return refuse_multi(s, "dng_scan_set_stream");
	if (s->launches || s->bytes_fed)
		return s->fail(DNG_EINVAL, "dng_scan_set_stream after a feed");
	s->stream = (cudaStream_t)cuda_stream;
	CK(s, cudaStreamWaitEvent(s->stream, s->ev_init, 0));
	return DNG_OK;
}

static int ensure_ring(dng_scan *s, bool need_stage)
{
	for (size_t i = 0; i < RING_SLOTS; i++) {
		if (!s->d_ring[i]) {
			CK(s, DEV_ALLOC(s, &s->d_ring[i], CARRY_ROOM +
			    s->ring_cap + 64));
			CK(s, cudaEventCreateWithFlags(&s->ev_ready[i],
			    cudaEventDisableTiming));
			CK(s, cudaEventCreateWithFlags(&s->ev_free[i],
			    cudaEventDisableTiming));
		}
		if (need_stage && !s->h_stage[i])
			CK(s, HOST_ALLOC(&s->h_stage[i], s->ring_cap));
	}
	return 0;
}

int dng_scan_feed(dng_scan *s, const void *buf, size_t len)
{
	if (!s || (!buf && len))
		return DNG_EINVAL;
	if (s->multi)
		return refuse_multi(s, "dng_scan_feed");
	cudaSetDevice(s->device);
	if (cz_flush(s) || ensure_ring(s, true))
		return s->err_code;
	return feed_host(s, buf, len, false);
}

int dng_scan_feed_pinned(dng_scan *s, const void *buf, size_t len)
{
	if (!s || (!buf && len))
		return DNG_EINVAL;
	if (s->multi)
		return refuse_multi(s, "dng_scan_feed_pinned");
	cudaSetDevice(s->device);
	if (cz_flush(s) || ensure_ring(s, false))
		return s->err_code;
	return feed_host(s, buf, len, true);
}

/*
 * Sequential fallback for inputs that cannot be pread (pipes, /dev/stdin):
 * read(2) into two pinned buffers, DMA from one while filling the other.
 */
static int feed_fd_sequential(dng_scan *s, int fd, const char *path)
{
	size_t cap = std::min(s->ring_cap, (size_t)16 << 20);
	u8 *bufs[2] = { nullptr, nullptr };
	cudaEvent_t done[2] = { nullptr, nullptr };
	bool inflight[2] = { false, false };
	int rc = 0;
	for (int i = 0; i < 2 && !rc; i++) {
		rc = s->cuda(cudaMallocHost(&bufs[i], cap), "cudaMallocHost");
		if (!rc)
			rc = s->cuda(cudaEventCreateWithFlags(&done[i],
			    cudaEventDisableTiming), "cudaEventCreate");
	}
	int which = 0;
	while (!rc) {
		if (inflight[which]) {
			rc = s->cuda(cudaEventSynchronize(done[which]),
			    "copy sync");
			if (rc)
				break;
		}
		ssize_t n = read(fd, bufs[which], cap);
		if (n < 0) {
			rc = s->fail(DNG_EIO, std::string("read ") + path + ": " +
			    strerror(errno));
			break;
		}
		if (n == 0)
			break;
		rc = feed_host(s, bufs[which], (size_t)n, true);
		if (!rc)
			rc = s->cuda(cudaEventRecord(done[which], s->copy_stream),
			    "cudaEventRecord");
		inflight[which] = true;
		which ^= 1;
	}
	cudaStreamSynchronize(s->copy_stream);
	for (int i = 0; i < 2; i++) {
		if (bufs[i])
			cudaFreeHost(bufs[i]);
		if (done[i])
			cudaEventDestroy(done[i]);
	}
	return rc;
}

/*
 * Regular files: a few reader threads read fixed-size blocks into a ring of
 * pinned buffers while this thread feeds completed blocks, in order, to the
 * H2D ring.  The reference reads with 2 concurrent 16 KB-request streams
 * (lib/datasource-file.js:262-266).  Reads bytes [off, off + size) of the
 * file; `exact`: a file that ends before that fails with DNG_EIO (else it is
 * read to where it ends now).
 *
 * A range mostly absent from the page cache is read with O_DIRECT, storage
 * straight into the pinned ring (direct_read.h); a cached one with pread,
 * whose page-cache memcpy is the slow part of reading, so it is spread over
 * the threads.
 */
static int feed_file_parallel(dng_scan *s, int fd, size_t off, size_t size,
    const char *path, bool exact, u8 *to_dev = nullptr)
{
	const size_t BLK = DR_BLK;
	const size_t NSLOT = 32;	/* 128 MiB of pinned ring */
	const size_t LAG = 6;		/* blocks kept back for in-flight DMA */
	const size_t GROUP = 4;		/* ready neighbours fed as one chunk */
	if (!s->file_buf) {
		CK(s, HOST_ALLOC(&s->file_buf, NSLOT * BLK));
		for (size_t i = 0; i < NSLOT; i++)
			CK(s, cudaEventCreateWithFlags(&s->file_done[i],
			    cudaEventDisableTiming));
	}
	DrRange r;
	r.fd = fd;
	r.exact = exact;
	size_t align = 1;
	if (dr_direct(dr_cached_fraction(fd, off, size))) {
		/* the same file, whatever happened to the path since */
		const std::string self = "/proc/self/fd/" + std::to_string(fd);
		align = dr_direct_align(dr_align(fd), s->file_buf);
		if (align)
			r.dfd = open(self.c_str(), O_RDONLY | O_DIRECT);
		if (r.dfd >= 0) {
			r.direct = true;
		} else {
			s->read_fallbacks++;
			align = 1;
		}
	}
	r.plan = dr_plan(off, size, align);
	const size_t nblocks = r.plan.nblocks;
	/* 16 readers by default: more threads contend in the page cache, and
	 * 16 direct reads in flight are the storage's queue depth */
	size_t nthreads = env_size("DNG_READ_THREADS", 16);
	nthreads = std::max<size_t>(1, std::min(nthreads, std::min(nblocks,
	    NSLOT - LAG)));
	std::mutex mu;
	std::condition_variable cv;
	size_t next_block = 0;		/* next block a reader takes */
	size_t released = NSLOT;	/* blocks < released may be (re)filled */
	std::vector<ssize_t> got(nblocks, -2);	/* fed bytes; -2 pending, -1 error */
	int read_errno = 0;
	bool abort_all = false;
	auto reader = [&]() {
		for (;;) {
			size_t b;
			{
				std::unique_lock<std::mutex> lk(mu);
				b = next_block++;
				if (b >= nblocks)
					return;
				cv.wait(lk, [&] { return b < released ||
				    abort_all; });
				if (abort_all)
					return;
			}
			size_t lo = 0, hi = 0;
			bool via_direct = false;
			int err = dr_fetch(pread, r, b,
			    s->file_buf + (b % NSLOT) * BLK, &lo, &hi, &via_direct);
			std::lock_guard<std::mutex> lk(mu);
			if (err) {
				read_errno = err;
				got[b] = -1;
			} else {
				got[b] = (ssize_t)(hi - lo);
				(via_direct ? s->direct_bytes : s->buffered_bytes) +=
				    hi - lo;
			}
			cv.notify_all();
		}
	};
	std::vector<std::thread> pool;
	for (size_t i = 0; i < nthreads; i++)
		pool.emplace_back(reader);
	int rc = 0;
	size_t b = 0;
	while (b < nblocks && !rc) {
		/* block b, plus ready full neighbours that are contiguous in
		 * the ring, go down as one chunk */
		size_t k = 0, bytes = 0;
		{
			std::unique_lock<std::mutex> lk(mu);
			cv.wait(lk, [&] { return got[b] != -2; });
			while (k < GROUP && b + k < nblocks &&
			    got[b + k] != -2 && (b + k) % NSLOT >= b % NSLOT) {
				if (got[b + k] < 0) {
					if (k == 0)
						rc = s->fail(DNG_EIO,
						    std::string("read ") + path +
						    ": " + (read_errno < 0 ?
						    "file is shorter than when "
						    "it was fed" :
						    strerror(read_errno)));
					break;
				}
				bytes += (size_t)got[b + k];
				k++;
				if (r.plan.lo(b + k - 1) + (size_t)got[b + k - 1]
				    != BLK)
					break;	/* short block: last one */
			}
		}
		if (rc)
			break;
		if (bytes && to_dev) {	/* (a compressed file: to its batch) */
			rc = s->cuda(cudaMemcpyAsync(to_dev, s->file_buf +
			    (b % NSLOT) * BLK + r.plan.lo(b), bytes,
			    cudaMemcpyHostToDevice, s->copy_stream),
			    "cudaMemcpyAsync");
			to_dev += bytes;
		} else if (bytes) {
			rc = feed_host(s, s->file_buf + (b % NSLOT) * BLK +
			    r.plan.lo(b), bytes, true);
		}
		for (size_t j = 0; j < k && !rc; j++)
			rc = s->cuda(cudaEventRecord(
			    s->file_done[(b + j) % NSLOT], s->copy_stream),
			    "cudaEventRecord");
		b += k;
		/* slots LAG blocks behind have certainly been DMA'd: hand them
		 * back to the readers */
		if (!rc && b > LAG) {
			size_t old = b - LAG - 1;
			rc = s->cuda(cudaEventSynchronize(
			    s->file_done[old % NSLOT]), "copy sync");
			std::lock_guard<std::mutex> lk(mu);
			released = old + NSLOT + 1;
			cv.notify_all();
		}
	}
	{
		std::lock_guard<std::mutex> lk(mu);
		abort_all = true;
		cv.notify_all();
	}
	for (auto &t : pool)
		t.join();
	if (r.dfd >= 0)
		close(r.dfd);
	s->direct_ranges += r.direct;	/* (not when it fell back) */
	s->read_fallbacks += r.fallbacks;
	/* the pinned ring is reused by the next file: drain its copies */
	cudaStreamSynchronize(s->copy_stream);
	return rc;
}

/* bytes [0, size) of the file at `path` to device memory at `dst`, through
 * the reader above (a compressed file, to its batch buffer); a file that is
 * now shorter fails with DNG_EIO */
int read_to_device(dng_scan *s, const char *path, size_t size, u8 *dst)
{
	int fd = open(path, O_RDONLY);
	if (fd < 0)
		return s->fail(DNG_EIO, std::string("open ") + path + ": " +
		    strerror(errno));
	const int rc = feed_file_parallel(s, fd, 0, size, path, true, dst);
	close(fd);
	return rc;
}

/* ---- scans over several devices (dng_scan_open_devices) -------------------
 *
 * The files fed are one logical stream of T bytes, as the reference
 * concatenates them (CatStreams, lib/datasource-file.js:252-288), so that a
 * file without a trailing newline joins its last line to the next file's
 * first.  Shard k of n owns the lines that START in [a_k, a_k+1), a_k =
 * floor(k T / n): it reads from its first line start to the first line start
 * at or after a_k+1 (T for the last shard), across file boundaries where its
 * last line spans them.  Every byte is read by exactly one shard.
 */

typedef std::pair<std::string, size_t> FedFile;	/* path, size when fed */

static size_t cut_point(size_t T, size_t k, size_t n)
{
	return (size_t)((unsigned __int128)T * k / n);
}

/* a fed file, open for reading, if it still has the size it was fed with */
static int open_fed(dng_scan *sh, const FedFile &f, int *fd)
{
	*fd = open(f.first.c_str(), O_RDONLY);
	if (*fd < 0)
		return sh->fail(DNG_EIO, "open " + f.first + ": " +
		    strerror(errno));
	struct stat st;
	if (fstat(*fd, &st) != 0 || (size_t)st.st_size != f.second) {
		close(*fd);
		*fd = -1;
		return sh->fail(DNG_EIO, "read " + f.first + ": file changed "
		    "size after it was fed");
	}
	return 0;
}

/* the first line start at or after stream position a: a itself when it is 0
 * or follows a '\n', else just past the next '\n', else T */
static int line_start(dng_scan *sh, const std::vector<FedFile> &files,
    size_t T, size_t a, size_t *out)
{
	*out = std::min(a, T);
	if (a == 0 || a >= T)
		return 0;
	const size_t pos = a - 1;	/* the byte that decides */
	std::vector<char> buf((size_t)64 << 10);
	size_t base = 0;
	for (const FedFile &f : files) {
		const size_t end = base + f.second;
		if (end > pos) {
			int fd;
			if (open_fed(sh, f, &fd))
				return sh->err_code;
			size_t o = pos > base ? pos - base : 0;
			while (o < f.second) {
				ssize_t n = pread(fd, buf.data(), std::min(buf.size(),
				    f.second - o), (off_t)o);
				if (n < 0 && errno == EINTR)
					continue;
				if (n <= 0) {
					const std::string why = n < 0 ?
					    strerror(errno) : "file is shorter "
					    "than when it was fed";
					close(fd);
					return sh->fail(DNG_EIO, "read " + f.first +
					    ": " + why);
				}
				const char *nl = (const char *)memchr(buf.data(),
				    '\n', (size_t)n);
				if (nl) {
					close(fd);
					*out = base + o + (size_t)(nl - buf.data()) + 1;
					return 0;
				}
				o += (size_t)n;
			}
			close(fd);
		}
		base = end;
	}
	*out = T;
	return 0;
}

/* shard k: its byte range of the stream fed to its scan, then its result */
static int run_shard(dng_scan *s, size_t k, size_t T, dng_result **res)
{
	dng_scan *sh = s->shards[k];
	const size_t n = s->shards.size();
	cudaSetDevice(sh->device);
	size_t begin, end;
	if (line_start(sh, s->files, T, cut_point(T, k, n), &begin) ||
	    line_start(sh, s->files, T, cut_point(T, k + 1, n), &end))
		return sh->err_code;
	size_t base = 0;
	for (const FedFile &f : s->files) {
		const size_t lo = std::max(begin, base);
		const size_t hi = std::min(end, base + f.second);
		if (lo < hi) {
			int fd;
			if (ensure_ring(sh, false) || open_fed(sh, f, &fd))
				return sh->err_code;
			int rc = feed_file_parallel(sh, fd, lo - base, hi - lo,
			    f.first.c_str(), true);
			close(fd);
			if (rc)
				return rc;
		}
		base += f.second;
	}
	return dng_scan_finish(sh, res);
}

/* sum values over identical tuples: the host merge of merge.cu */
static int merge_results(const std::vector<dng_result *> &res,
    dng_result **out)
{
	const size_t n = res.size();
	std::vector<const void *> bufs(n);
	std::vector<size_t> lens(n);
	for (size_t k = 0; k < n; k++)
		dng_result_dict(res[k], &bufs[k], &lens[k]);
	void *gdict = nullptr;
	size_t glen = 0;
	int rc = dng_dict_union(bufs.data(), lens.data(), n, &gdict, &glen);
	if (rc)
		return rc;
	const size_t G = dng_dict_count(gdict, glen);
	std::vector<uint64_t> sum(std::max<size_t>(G, 1), 0), one(sum.size());
	for (size_t k = 0; k < n && !rc; k++) {
		rc = dng_result_dense(res[k], gdict, glen, one.data(), G);
		for (size_t i = 0; i < G; i++)
			sum[i] += one[i];
	}
	if (!rc)
		rc = dng_result_from_dense(res[0], gdict, glen, sum.data(), G, out);
	dng_buf_free(gdict);
	return rc;
}

/* dng_scan_finish of a multi-device scan: one thread per shard */
static int finish_multi(dng_scan *s, dng_result **out)
{
	const size_t n = s->shards.size();
	size_t T = 0;
	for (const FedFile &f : s->files)
		T += f.second;
	std::vector<dng_result *> res(n, nullptr);
	std::vector<int> rc(n, 0);
	const bool again = s->finished;	/* (a second finish reads nothing) */
	std::vector<std::thread> th;
	for (size_t k = 0; k < n; k++)
		th.emplace_back([&, k] {
			rc[k] = again ? dng_scan_finish(s->shards[k], &res[k]) :
			    run_shard(s, k, T, &res[k]);
		});
	for (auto &t : th)
		t.join();
	s->finished = true;
	int r = 0;
	for (size_t k = 0; k < n && !r; k++)
		if (rc[k])
			r = s->fail(rc[k], "shard " + std::to_string(k) +
			    " (device " + std::to_string(s->shards[k]->device) +
			    "): " + s->shards[k]->err);
	if (!r)
		r = merge_results(res, out);
	for (dng_result *x : res)
		dng_result_destroy(x);
	return r ? s->fail(r, "merging the shards' results") : DNG_OK;
}

/* the counters of metric m: the shards' summed */
static int counters_multi(dng_scan *s, int m, dng_counters *out)
{
	memset(out, 0, sizeof (*out));
	for (dng_scan *sh : s->shards) {
		dng_counters c;
		int rc = dng_scan_counters_metric(sh, m, &c);
		if (rc)
			return s->fail(rc, sh->err);
		const uint64_t *a = (const uint64_t *)&c;
		uint64_t *o = (uint64_t *)out;
		for (size_t i = 0; i < sizeof (c) / sizeof (uint64_t); i++)
			o[i] += a[i];
	}
	return DNG_OK;
}

/* dng_scan_feed_file of a multi-device scan: the path and its size only */
static int record_file(dng_scan *s, const char *path)
{
	if (s->err_code)
		return s->err_code;
	if (s->finished)
		return s->fail(DNG_EINVAL, "scan already finished");
	int fd = open(path, O_RDONLY);
	if (fd < 0)
		return s->fail(DNG_EIO, std::string("open ") + path + ": " +
		    strerror(errno));
	struct stat st;
	const bool reg = fstat(fd, &st) == 0 && S_ISREG(st.st_mode);
	close(fd);
	if (!reg)
		return s->fail(DNG_EINVAL, std::string(path) + ": not a regular "
		    "file (a scan over several devices cuts its input by size)");
	s->files.emplace_back(path, (size_t)st.st_size);
	return DNG_OK;
}

int dng_scan_feed_file(dng_scan *s, const char *path)
{
	if (!s || !path)
		return DNG_EINVAL;
	if (s->multi)
		return record_file(s, path);
	cudaSetDevice(s->device);
	if (cz_flush(s) || ensure_ring(s, false))
		return s->err_code;
	int fd = open(path, O_RDONLY);
	if (fd < 0)
		return s->fail(DNG_EIO, std::string("open ") + path + ": " +
		    strerror(errno));
	struct stat st;
	int rc;
	if (fstat(fd, &st) == 0 && S_ISREG(st.st_mode) && st.st_size > 0)
		rc = feed_file_parallel(s, fd, 0, (size_t)st.st_size, path, false);
	else
		rc = feed_fd_sequential(s, fd, path);
	close(fd);
	return rc;
}

int dng_scan_feed_device(dng_scan *s, const void *devbuf, size_t len)
{
	if (!s || (!devbuf && len))
		return DNG_EINVAL;
	if (s->multi)
		return refuse_multi(s, "dng_scan_feed_device");
	cudaSetDevice(s->device);
	if (cz_flush(s))
		return s->err_code;
	return feed_device(s, devbuf, len);
}

/* dng_scan_feed_device of a single-device scan with no compressed files
 * queued */
int feed_device(dng_scan *s, const void *devbuf, size_t len)
{
	if (s->err_code)
		return s->err_code;
	if (s->finished)
		return s->fail(DNG_EINVAL, "scan already finished");
	if ((uintptr_t)devbuf & 15)
		return s->fail(DNG_EINVAL, "device buffer must be 16-byte "
		    "aligned");
	if (len == 0)
		return 0;
	/*
	 * A CTA's tally cache counts in 32 bits and is flushed once per launch.
	 * With weight-1 records that cannot wrap within a launch over any buffer
	 * HBM holds; with json-skinner weights (up to 255 take the cache) a
	 * launch is kept to 4 GiB: at most 33 MB per CTA on an H100's 132 SMs,
	 * under
	 * 2^32 / 255 records of even the shortest point line.
	 */
	const size_t LAUNCH_MAX = (size_t)4 << 30;
	if (s->plan.dev.format == FMT_SKINNER && len > LAUNCH_MAX) {
		for (size_t off = 0; off < len; off += LAUNCH_MAX) {
			int rc = feed_device(s, (const u8 *)devbuf + off,
			    std::min(LAUNCH_MAX, len - off));
			if (rc)
				return rc;
		}
		return 0;
	}
	cudaSetDevice(s->device);
	const u8 *d = (const u8 *)devbuf;
	s->bytes_fed += len;
	/*
	 * The first scan of this data starts at its first byte when nothing is
	 * carried: the head the scan learns its templates from is copied out
	 * along with the newline search, and arrives with it, in one wait.
	 */
	u8 *sample = nullptr;
	struct Release {
		u8 *p;
		~Release() { cached_free(p); }
	} release{nullptr};
	if (!s->tmpl_tried && !s->carry_len &&
	    kc_wants_sample(s->kc, s->tmpl_enabled)) {
		CK(s, HOST_ALLOC(&sample, TMPL_SAMPLE_BYTES));
		release.p = sample;
		CK(s, cudaMemcpyAsync(sample, d, std::min<size_t>(len,
		    TMPL_SAMPLE_BYTES), cudaMemcpyDeviceToHost, s->stream));
	}
	/* locate the first and last newline (windows first, then all) */
	unsigned long long init[2] = { ~0ull, 0 }, got[2];
	const unsigned long long W = 1 << 20;
	for (int attempt = 0; attempt < 2; attempt++) {
		CK(s, cudaMemcpyAsync(s->d_nl, init, sizeof (init),
		    cudaMemcpyHostToDevice, s->stream));
		if (attempt == 0) {
			s->aux_launches++;
			find_nl_kernel<<<64, 256, 0, s->stream>>>(d, 0,
			    std::min<unsigned long long>(len, W), s->d_nl,
			    s->d_nl + 1);
			if (len > W) {
				s->aux_launches++;
				find_nl_kernel<<<64, 256, 0, s->stream>>>(d,
				    len - W, len, s->d_nl, s->d_nl + 1);
			}
		} else {
			s->aux_launches++;
			find_nl_kernel<<<1024, 256, 0, s->stream>>>(d, 0, len,
			    s->d_nl, s->d_nl + 1);
		}
		CK(s, cudaMemcpyAsync(got, s->d_nl, sizeof (got),
		    cudaMemcpyDeviceToHost, s->stream));
		CK(s, cudaStreamSynchronize(s->stream));
		/* with windows: `first` is only trustworthy if it fell in the
		 * head window, `last` if it fell in the tail window */
		bool first_ok = got[0] != ~0ull && (len <= W || got[0] < W);
		bool last_ok = got[1] != 0 && (len <= W || got[1] > len - W);
		if ((first_ok && last_ok) || attempt == 1 || len <= W)
			break;
	}
	if (got[0] == ~0ull) {
		/* no newline at all: the whole chunk extends the carry */
		if (s->carry_len + len >= DNG_MAXREC)
			return s->fail(DNG_ELIMIT, "input line longer than 16 MiB");
		CK(s, cudaMemcpyAsync(s->d_carry + s->carry_len, d, len,
		    cudaMemcpyDeviceToDevice, s->stream));
		s->carry_len += len;
		return 0;
	}
	unsigned long long first = got[0], last = got[1];
	unsigned long long start = 0;
	if (s->carry_len) {
		/* finish the carried line in a side buffer (`head` counts its
		 * newline) */
		size_t head = (size_t)first + 1;
		if (s->carry_len + head > DNG_MAXREC)
			return s->fail(DNG_ELIMIT, "input line longer than 16 MiB");
		if (!s->d_side)
			CK(s, DEV_ALLOC(s, &s->d_side, CARRY_ROOM + 64));
		CK(s, cudaMemcpyAsync(s->d_side, s->d_carry, s->carry_len,
		    cudaMemcpyDeviceToDevice, s->stream));
		CK(s, cudaMemcpyAsync(s->d_side + s->carry_len, d, head,
		    cudaMemcpyDeviceToDevice, s->stream));
		if (launch_scan(s, s->d_side, 0, s->carry_len + head, false))
			return s->err_code;
		s->carry_len = 0;
		start = head;
	}
	if (launch_scan(s, d, start, last, false, start == 0 ? sample : nullptr))
		return s->err_code;
	if (last < len) {
		size_t tail = len - (size_t)last;
		if (tail >= DNG_MAXREC)
			return s->fail(DNG_ELIMIT, "input line longer than 16 MiB");
		CK(s, cudaMemcpyAsync(s->d_carry, d + last, tail,
		    cudaMemcpyDeviceToDevice, s->stream));
		s->carry_len = tail;
	}
	return 0;
}

int dng_scan_sync(dng_scan *s)
{
	if (!s)
		return DNG_EINVAL;
	if (s->multi)	/* (its shards run only inside dng_scan_finish) */
		return s->err_code;
	cudaSetDevice(s->device);
	cz_flush(s);
	CK(s, cudaStreamSynchronize(s->copy_stream));
	CK(s, cudaStreamSynchronize(s->stream));
	drain_events(s);
	return s->err_code;
}

static int flush_tail(dng_scan *s)
{
	if (s->finished)
		return 0;
	s->finished = true;
	if (s->carry_len) {
		/* lstream emits the final unterminated line */
		if (launch_scan(s, s->d_carry, 0, s->carry_len, true))
			return s->err_code;
		s->carry_len = 0;
	}
	return 0;
}

int dng_scan_counters(dng_scan *s, dng_counters *out)
{
	if (!s || !out)
		return DNG_EINVAL;
	if (s->multi)
		return counters_multi(s, 0, out);
	cudaSetDevice(s->device);
	if (dng_scan_sync(s))
		return s->err_code;
	unsigned long long c[NCTR];
	CK(s, cudaMemcpy(c, s->d_counters, sizeof (c), cudaMemcpyDeviceToHost));
	memset(out, 0, sizeof (*out));
	out->lines = c[CTR_LINES];
	out->invalid_json = c[CTR_INVALID_JSON];
	out->invalid_point = c[CTR_INVALID_POINT];
	out->ds_filtered = c[CTR_DS_FILTERED];
	out->ds_failedeval = c[CTR_DS_FAILED];
	out->user_filtered = c[CTR_USER_FILTERED];
	out->user_failedeval = c[CTR_USER_FAILED];
	out->synth_undef = c[CTR_SYNTH_UNDEF];
	out->synth_baddate = c[CTR_SYNTH_BADDATE];
	out->time_filtered = c[CTR_TIME_FILTERED];
	out->time_failedeval = c[CTR_TIME_FAILED];
	out->aggr_ninputs = c[CTR_AGGR];
	out->slowpath_records = c[CTR_SLOW];
	out->unsupported = c[CTR_UNSUPPORTED];
	out->long_records = c[CTR_LONG];
	out->bytes = s->bytes_fed;
	uint64_t n = out->lines - out->invalid_json - out->invalid_point;
	const DevPlan &P = s->plan.dev;
	if (P.ds_entry >= 0) {
		out->ds_ninputs = n;
		n -= out->ds_filtered + out->ds_failedeval;
	}
	if (P.metric[0].user_entry >= 0) {
		out->user_ninputs = n;
		n -= out->user_filtered + out->user_failedeval;
	}
	if (P.metric[0].nsyn) {
		out->synth_ninputs = n;
		n -= out->synth_undef + out->synth_baddate;
	}
	if (P.metric[0].time_entry >= 0)
		out->time_ninputs = n;
	return DNG_OK;
}

int dng_scan_counters_metric(dng_scan *s, int m, dng_counters *out)
{
	if (!s || !out || m < 0 || m >= s->plan.dev.nmetrics)
		return DNG_EINVAL;
	if (s->multi)
		return counters_multi(s, m, out);
	int rc = dng_scan_counters(s, out);
	if (rc || m == 0)
		return rc;
	unsigned long long c[MCTR_PER];
	CK(s, cudaMemcpy(c, s->d_counters + NCTR + (m - 1) * MCTR_PER,
	    sizeof (c), cudaMemcpyDeviceToHost));
	const Metric &M = s->plan.dev.metric[m];
	uint64_t n = out->lines - out->invalid_json - out->invalid_point -
	    out->ds_filtered - out->ds_failedeval;
	out->user_ninputs = out->synth_ninputs = out->time_ninputs = 0;
	out->user_filtered = c[0];
	out->user_failedeval = c[1];
	out->synth_undef = c[2];
	out->synth_baddate = c[3];
	out->time_filtered = c[4];
	out->time_failedeval = c[5];
	out->aggr_ninputs = c[6];
	if (M.user_entry >= 0) {
		out->user_ninputs = n;
		n -= c[0] + c[1];
	}
	if (M.nsyn) {
		out->synth_ninputs = n;
		n -= c[2] + c[3];
	}
	if (M.time_entry >= 0)
		out->time_ninputs = n;
	return DNG_OK;
}

int dng_scan_finish(dng_scan *s, dng_result **out)
{
	if (!s || !out)
		return DNG_EINVAL;
	if (s->err_code)
		return s->err_code;
	if (s->multi)
		return finish_multi(s, out);
	cudaSetDevice(s->device);
	if (cz_flush(s) || flush_tail(s))
		return s->err_code;
	if (dng_scan_sync(s))
		return s->err_code;
	u32 misc[4];
	CK(s, cudaMemcpy(misc, s->tab.misc, sizeof (misc),
	    cudaMemcpyDeviceToHost));
	if (misc[2] & ST_TABLE_FULL)
		return s->fail(DNG_ELIMIT, "too many distinct tuples for the "
		    "device table (raise DNG_TABLE_CAP)");
	if (misc[2] & ST_ARENA_FULL)
		return s->fail(DNG_ELIMIT, "group-key arena exhausted (raise "
		    "DNG_ARENA_BYTES)");
#ifdef DNG_PROFILE_PHASES
	{	/* tuning builds only: where a tile's cycles go (see scan_kernel) */
		unsigned long long pc[NCTR];
		CK(s, cudaMemcpy(pc, s->d_counters, sizeof (pc),
		    cudaMemcpyDeviceToHost));
		double nw = (double)pc[18] ? (double)pc[18] : 1;
		fprintf(stderr, "phases: per warp-tile cycles: load-wait %.0f "
		    "index %.0f records-busy %.0f records-phase %.0f total %.0f "
		    "(%llu warp-tiles)\n", pc[19] / nw, pc[20] / nw, pc[16] / nw,
		    pc[17] / nw, pc[21] / nw, pc[18]);
	}
#endif
	dng_counters c;
	if (dng_scan_counters(s, &c))
		return s->err_code;
	if (c.unsupported)
		return s->fail(DNG_EUNSUPPORTED, "input contains records the "
		    "device path cannot decide yet (" +
		    std::to_string(c.unsupported) + "): nesting deeper than 64, "
		    "a group key longer than 512 bytes, a line >= 16 MiB, an "
		    "array where an index/length lookup is needed, or a date "
		    "string outside the ISO format (V8's legacy Date.parse "
		    "forms are not restated)");
	u32 n = misc[1];
	dng_result *r = new dng_result();
	r->init_from_plan(&s->plan);
	if (n) {
		OutEntry *d_out = nullptr;
		u32 *d_n = nullptr;
		size_t cap_out = 4096;		/* few sizes: cache-friendly */
		while (cap_out < n)
			cap_out <<= 1;
		CK(s, DEV_ALLOC(s, &d_out, cap_out * sizeof (OutEntry)));
		CK(s, DEV_ALLOC(s, &d_n, 16));
		CK(s, cudaMemsetAsync(d_n, 0, sizeof (u32), s->stream));
		s->aux_launches++;
		compact_kernel<<<256, 256, 0, s->stream>>>(s->tab.entries,
		    s->tab.mask + 1, d_out, d_n);
		std::vector<OutEntry> ents(n);
		std::vector<u8> arena(misc[0]);
		CK(s, cudaMemcpyAsync(ents.data(), d_out,
		    (size_t)n * sizeof (OutEntry), cudaMemcpyDeviceToHost,
		    s->stream));
		if (misc[0])
			CK(s, cudaMemcpyAsync(arena.data(), s->tab.arena, misc[0],
			    cudaMemcpyDeviceToHost, s->stream));
		CK(s, cudaStreamSynchronize(s->stream));
		cached_free(d_out);
		cached_free(d_n);
		r->keys.reserve(n);
		r->values.reserve(n);
		for (u32 i = 0; i < n; i++) {
			r->keys.emplace_back((const char *)arena.data() +
			    ents[i].koff, ents[i].klen);
			r->values.push_back(ents[i].count);
		}
	}
	r->finalize();
	*out = r;
	return DNG_OK;
}

const char *dng_scan_error(const dng_scan *s)
{
	return s ? s->err.c_str() : "null scan";
}

int dng_scan_set_templates(dng_scan *s, int enable)
{
	if (!s)
		return DNG_EINVAL;
	if (s->multi) {
		if (s->finished)
			return s->fail(DNG_EINVAL, "templates are fixed once data "
			    "has been fed");
		for (dng_scan *sh : s->shards)
			dng_scan_set_templates(sh, enable);
		return DNG_OK;
	}
	if (s->tmpl_tried)
		return s->fail(DNG_EINVAL, "templates are fixed once data has "
		    "been fed");
	s->tmpl_enabled = enable != 0;
	return DNG_OK;
}

int dng_scan_template_stats(dng_scan *s, uint64_t *templates,
    uint64_t *templated_records)
{
	if (!s)
		return DNG_EINVAL;
	if (s->multi)
		return refuse_multi(s, "dng_scan_template_stats");
	cudaSetDevice(s->device);
	if (dng_scan_sync(s))
		return s->err_code;
	unsigned long long c = 0;
	CK(s, cudaMemcpy(&c, s->d_counters + CTR_TMPL, sizeof (c),
	    cudaMemcpyDeviceToHost));
	if (templates) {
		/* (what the general kernels' blob holds once it is built) */
		std::vector<u8> blob;
		u32 nt = 0;
		general_blob(s, blob, &nt);
		*templates = blob.empty() ? s->ntemplates : nt;
	}
	put(templated_records, c);
	return DNG_OK;
}

uint64_t dng_scan_launch_count(const dng_scan *s)
{
	if (s && s->multi) {
		uint64_t n = 0;
		for (const dng_scan *sh : s->shards)
			n += dng_scan_launch_count(sh);
		return n;
	}
	return s ? s->launches + s->aux_launches : 0;
}

int dng_scan_read_stats(dng_scan *s, uint64_t *direct_bytes,
    uint64_t *buffered_bytes, uint64_t *direct_ranges, uint64_t *fallbacks)
{
	if (!s)
		return DNG_EINVAL;
	uint64_t v[4] = { s->direct_bytes, s->buffered_bytes, s->direct_ranges,
	    s->read_fallbacks };
	for (dng_scan *sh : s->shards) {
		uint64_t one[4];
		dng_scan_read_stats(sh, &one[0], &one[1], &one[2], &one[3]);
		for (int i = 0; i < 4; i++)
			v[i] += one[i];
	}
	put(direct_bytes, v[0]);
	put(buffered_bytes, v[1]);
	put(direct_ranges, v[2]);
	put(fallbacks, v[3]);
	return DNG_OK;
}

int dng_scan_kernel_kind(const dng_scan *s)
{
	if (!s || s->multi)
		return DNG_EINVAL;
	return kc_pick(s->kc);
}

int dng_scan_jit_stats(dng_scan *s, int *state, uint64_t *launches,
    double *compile_ms, double *link_ms, char *err, size_t errlen)
{
	if (!s)
		return DNG_EINVAL;
	if (s->multi)
		return refuse_multi(s, "dng_scan_jit_stats");
	const int st = s->jit ? s->jit->state.load() : 0;
	put(state, st);
	put(launches, s->jit_launches);
	put(compile_ms, st ? s->jit->compile_ms : 0);
	put(link_ms, st ? s->jit->link_ms : 0);
	set_err(err, errlen, "%s", st == 2 ? s->jit->err.c_str() : "");
	return DNG_OK;
}

int dng_scan_kernel_stats(dng_scan *s, double *kernel_ms, uint64_t *launches,
    uint64_t *kernel_bytes)
{
	if (!s)
		return DNG_EINVAL;
	if (s->multi)
		return refuse_multi(s, "dng_scan_kernel_stats");
	cudaSetDevice(s->device);
	if (dng_scan_sync(s))
		return s->err_code;
	put(kernel_ms, s->kernel_ms);
	put(launches, s->launches);
	put(kernel_bytes, s->kernel_bytes);
	return DNG_OK;
}

int dng_scan_tally_stats(dng_scan *s, uint64_t *inline_overflow, int *f_warps)
{
	if (!s)
		return DNG_EINVAL;
	if (s->multi)
		return refuse_multi(s, "dng_scan_tally_stats");
	cudaSetDevice(s->device);
	if (dng_scan_sync(s))
		return s->err_code;
	unsigned long long c = 0;
	CK(s, cudaMemcpy(&c, s->d_counters + CTR_OVER, sizeof (c),
	    cudaMemcpyDeviceToHost));
	put(inline_overflow, c);
	put(f_warps, (int)s->kc.f_nw);
	return DNG_OK;
}

void dng_jit_finish(void)
{
	dng::jit_finish();
}

int dng_jit_cache_dir(const char *dir)
{
	dng::jit_cache_set_dir(dir);
	return DNG_OK;
}

int dng_jit_cache_stats(uint64_t *hits, uint64_t *misses, uint64_t *writes,
    uint64_t *evictions, uint64_t *errors)
{
	const dng::JitCacheStats st = dng::jit_cache_stats();
	put(hits, st.hits);
	put(misses, st.misses);
	put(writes, st.writes);
	put(evictions, st.evictions);
	put(errors, st.errors);
	return DNG_OK;
}

void dng_release_cached(void)
{
	BufCache &c = buf_cache();
	std::multimap<std::pair<int, size_t>, void *> idle;
	{
		std::lock_guard<std::mutex> g(c.mu);
		idle.swap(c.idle);
		c.idle_dev = c.idle_host = 0;
	}
	for (auto &kv : idle) {
		if (kv.first.first < 0) {
			cudaFreeHost(kv.second);
		} else {
			cudaSetDevice(kv.first.first);
			cudaFree(kv.second);
		}
	}
}

void dng_scan_destroy(dng_scan *s)
{
	if (!s)
		return;
	if (s->multi) {
		for (dng_scan *sh : s->shards)
			dng_scan_destroy(sh);
		delete s;
		return;
	}
	cudaSetDevice(s->device);
	if (s->stream)
		cudaStreamSynchronize(s->stream);
	if (s->own_stream && s->own_stream != s->stream)
		cudaStreamSynchronize(s->own_stream);
	if (s->copy_stream)
		cudaStreamSynchronize(s->copy_stream);
	drain_events(s);
	if (s->ev_init)
		cudaEventDestroy(s->ev_init);
	for (auto e : s->ev_pool)
		cudaEventDestroy(e);
	for (size_t i = 0; i < RING_SLOTS; i++) {
		if (s->d_ring[i]) {
			cached_free(s->d_ring[i]);
			cudaEventDestroy(s->ev_ready[i]);
			cudaEventDestroy(s->ev_free[i]);
		}
		if (s->h_stage[i])
			cached_free(s->h_stage[i]);
	}
	if (s->file_buf) {
		cached_free(s->file_buf);
		for (int i = 0; i < 32; i++)
			cudaEventDestroy(s->file_done[i]);
	}
	cached_free(s->h_live);
	cached_free(s->h_blobs);
	cached_free(s->d_plan);
	cached_free(s->d_tmpl);
	cached_free(s->d_fplan);
	cached_free(s->d_ftmpl);
	cached_free(s->d_miss);
	cached_free(s->d_miss_n);
	cached_free(s->tab.entries);
	cached_free(s->tab.arena);
	cached_free(s->tab.misc);
	cached_free(s->d_counters);
	cached_free(s->d_nl);
	cached_free(s->d_carry);
	cached_free(s->d_side);
	cz_free(s->cz);
	if (s->own_stream)
		cudaStreamDestroy(s->own_stream);
	if (s->copy_stream)
		cudaStreamDestroy(s->copy_stream);
	delete s;
}

void *dng_pinned_alloc(size_t len)
{
	void *p = nullptr;
	if (cudaMallocHost(&p, len) != cudaSuccess)
		return nullptr;
	return p;
}

void dng_pinned_free(void *p)
{
	if (p)
		cudaFreeHost(p);
}

/* ---- results ------------------------------------------------------------ */

size_t dng_result_count(const dng_result *r)
{
	return r ? r->keys.size() : 0;
}

size_t dng_result_ncols(const dng_result *r)
{
	size_t n = 0;
	for (int m = 0; r && m < r->nmetrics; m++)
		n = std::max(n, (size_t)r->ncols[m]);
	return n;		/* widest metric; == ncols for a plain scan */
}

size_t dng_result_nmetrics(const dng_result *r)
{
	return r ? (size_t)r->nmetrics : 0;
}

size_t dng_result_ncols_metric(const dng_result *r, int m)
{
	return r && m >= 0 && m < r->nmetrics ? (size_t)r->ncols[m] : 0;
}

int dng_result_metric(const dng_result *r, size_t i)
{
	return r && i < r->metric.size() ? r->metric[i] : -1;
}

int dng_result_get(const dng_result *r, size_t i, const char **strs,
    size_t *strlens, uint8_t *is_number, double *numvals, uint64_t *value)
{
	if (!r || i >= r->keys.size())
		return DNG_EINVAL;
	for (int j = 0; j < r->ncols[r->metric[i]]; j++) {
		const dng_result::Cell &c = r->cells[r->cell0[i] + j];
		if (is_number)
			is_number[j] = c.is_number;
		if (numvals)
			numvals[j] = c.num;
		if (strs)
			strs[j] = c.is_number ? nullptr :
			    r->keys[i].data() + c.off;
		if (strlens)
			strlens[j] = c.is_number ? 0 : c.len;
	}
	if (value)
		*value = r->values[i];
	return DNG_OK;
}

void dng_result_destroy(dng_result *r)
{
	delete r;
}

/* ---- synthetic input ------------------------------------------------------ */

void dng_gen_defaults(dng_gen_params *p)
{
	p->seed = 0xD5A60000ull;
	p->total_records = 1000;
	p->time_min_ms = 1401570000000ll;	/* 2014-05-31T21:00:00Z */
	p->time_max_ms = 1401580799000ll;	/* 2014-05-31T23:59:59Z */
	p->string_latency = 0;
}

int dng_gen_host(const dng_gen_params *p, uint64_t first, uint64_t count,
    void *buf, size_t cap, size_t *len)
{
	if (!p || !buf || !len)
		return DNG_EINVAL;
	char *o = (char *)buf;
	size_t n = 0;
	char tmp[GEN_MAXREC];
	for (uint64_t j = first; j < first + count; j++) {
		int k = gen_record(*p, j, tmp);
		if (n + (size_t)k > cap)
			return DNG_ELIMIT;
		memcpy(o + n, tmp, (size_t)k);
		n += (size_t)k;
	}
	*len = n;
	return DNG_OK;
}


namespace {

__global__ void gen_len_kernel(dng_gen_params p, uint64_t first, uint64_t count,
    unsigned long long *block_sums, u32 *lens)
{
	__shared__ u32 red[256 / 32];
	uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	char tmp[GEN_MAXREC];
	u32 k = 0;
	if (j < count) {
		k = (u32)gen_record(p, first + j, tmp);
		lens[j] = k;
	}
	u32 v = k;
	for (int d = 16; d > 0; d >>= 1)
		v += __shfl_xor_sync(0xffffffffu, v, d);
	if ((threadIdx.x & 31) == 0)
		red[threadIdx.x >> 5] = v;
	__syncthreads();
	if (threadIdx.x == 0) {
		u32 t = 0;
		for (int i = 0; i < 256 / 32; i++)
			t += red[i];
		block_sums[blockIdx.x] = t;
	}
}

__global__ void gen_write_kernel(dng_gen_params p, uint64_t first,
    uint64_t count, const unsigned long long *block_offs, const u32 *lens,
    char *out)
{
	__shared__ u32 soff[256];
	uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	u32 k = j < count ? lens[j] : 0;
	soff[threadIdx.x] = k;
	__syncthreads();
	/* exclusive scan within the block (serial by thread 0: 256 adds) */
	if (threadIdx.x == 0) {
		u32 acc = 0;
		for (int i = 0; i < 256; i++) {
			u32 t = soff[i];
			soff[i] = acc;
			acc += t;
		}
	}
	__syncthreads();
	if (j < count) {
		char tmp[GEN_MAXREC];
		int n = gen_record(p, first + j, tmp);
		char *dst = out + block_offs[blockIdx.x] + soff[threadIdx.x];
		for (int i = 0; i < n; i++)
			dst[i] = tmp[i];
	}
}

} /* namespace */

extern "C" int dng_gen_device(const dng_gen_params *p, int device,
    uint64_t first, uint64_t count, void *devbuf, size_t cap, size_t *len)
{
	if (!p || !devbuf || !len)
		return DNG_EINVAL;
	if (cudaSetDevice(device) != cudaSuccess)
		return DNG_ENODEV;
	if (count == 0) {
		*len = 0;
		return DNG_OK;
	}
	u32 nblocks = (u32)((count + 255) / 256);
	unsigned long long *d_sums = nullptr;
	u32 *d_lens = nullptr;
	int rc = DNG_OK;
	if (cudaMalloc(&d_sums, (size_t)nblocks * 8) != cudaSuccess ||
	    cudaMalloc(&d_lens, (size_t)count * 4) != cudaSuccess) {
		cudaFree(d_sums);
		cudaFree(d_lens);
		return DNG_ENOMEM;
	}
	gen_len_kernel<<<nblocks, 256>>>(*p, first, count, d_sums, d_lens);
	std::vector<unsigned long long> sums(nblocks);
	if (cudaMemcpy(sums.data(), d_sums, (size_t)nblocks * 8,
	    cudaMemcpyDeviceToHost) != cudaSuccess)
		rc = DNG_ECUDA;
	unsigned long long acc = 0;
	for (u32 i = 0; i < nblocks; i++) {
		unsigned long long t = sums[i];
		sums[i] = acc;
		acc += t;
	}
	if (!rc && acc > cap)
		rc = DNG_ELIMIT;
	if (!rc) {
		cudaMemcpy(d_sums, sums.data(), (size_t)nblocks * 8,
		    cudaMemcpyHostToDevice);
		gen_write_kernel<<<nblocks, 256>>>(*p, first, count, d_sums,
		    d_lens, (char *)devbuf);
		if (cudaDeviceSynchronize() != cudaSuccess)
			rc = DNG_ECUDA;
		*len = (size_t)acc;
	}
	cudaFree(d_sums);
	cudaFree(d_lens);
	return rc;
}
