/*
 * compressed.cu: compressed input of a scan.  dng_scan_feed_gzip and
 * dng_scan_feed_bzip2 queue files; cz_flush decodes each batch on the device
 * (inflate.cuh, inflate_split.cuh, bunzip.cuh) and feeds the decompressed
 * bytes to the scan as device buffers (feed_device, api.cu).
 */
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <cstring>
#include <list>
#include <numeric>
#include <string>
#include <vector>

#include "scan.h"
#include "inflate.cuh"
#include "inflate_policy.h"
#include "inflate_split.cuh"
#include "bunzip.cuh"
#include "bunzip_policy.h"

using namespace dng;

/* a device buffer from the scan's buffer cache, returned to it with the
 * state (the inflate jobs' staging is pinned host memory) */
struct DevBuf {
	u8 *p = nullptr;
	size_t cap = 0;
	DevBuf() = default;
	DevBuf(const DevBuf &) = delete;
	DevBuf &operator=(const DevBuf &) = delete;
	~DevBuf() { dng_cached_free(p); }
};

/* a queued file: its compressed size, the output room of a gzip file, the
 * first four bytes of a bzip2 file */
struct CzFile {
	std::string path;
	size_t size;
	uint64_t hint;
	uint32_t head;
};

struct CzState {
	/* files queued for the next batch, all of one format, and the batch's
	 * compressed bytes and output room */
	std::vector<CzFile> queue;
	bool bzip2 = false;		/* the queue's format */
	uint64_t queued_in = 0, queued_out = 0;
	DevBuf in;			/* the batch's compressed bytes */
	/* the gzip path: outputs, a file decoded again in more room, a run
	 * realigned; jobs, results and next (device and pinned) */
	DevBuf gz_out, gz_big, gz_join, gz_jobs, gz_jobs_host;
	uint64_t gz_files = 0, gz_members = 0, gz_in_bytes = 0, gz_out_bytes = 0;
	uint64_t gz_launches = 0;
	double gz_ms = 0;
	/* the split path (inflate_split.cuh): a batch's chunk state, symbols,
	 * outputs that missed their regions and checks; its stats */
	DevBuf gz_split, gz_sym, gz_sout, gz_check;
	uint64_t gz_split_files = 0, gz_chunks = 0, gz_false_starts = 0;
	uint64_t gz_fallbacks = 0, gz_split_launches = 0;
	uint32_t gz_split_blocks = 0;	/* CTAs of split_decode_kernel per SM */
	/* the bzip2 path (bunzip.cuh): candidates, BWT slots, transformation
	 * vectors, per-block records and output of a wave; its stats */
	DevBuf bz_find, bz_slot, bz_tt, bz_rec, bz_out;
	uint64_t bz_files = 0, bz_streams = 0, bz_blocks = 0;
	uint64_t bz_false_starts = 0, bz_in_bytes = 0, bz_out_bytes = 0;
	uint64_t bz_launches = 0;
	double bz_ms = 0;
	double bz_stage_ms[4] = {};	/* find, decode, invert, emit */
};

void cz_free(CzState *cz)
{
	delete cz;
}

static size_t align_up(size_t n, size_t a)
{
	return (n + a - 1) & ~(a - 1);
}

/* make `b` hold at least n bytes (powers of two from 1 MiB, so the buffer
 * cache takes them back); what the old buffer held is not kept */
static int grow(dng_scan *s, DevBuf &b, size_t n)
{
	if (b.p && b.cap >= n)
		return 0;
	size_t c = (size_t)1 << 20;
	while (c < n)
		c <<= 1;
	if (b.p) {
		/* scan kernels enqueued earlier may still read it */
		CK(s, cudaStreamSynchronize(s->stream));
		dng_cached_free(b.p);
		b.p = nullptr;
		b.cap = 0;
	}
	CK(s, DEV_ALLOC(s, &b.p, c));
	b.cap = c;
	return 0;
}

/* the device time of a stage of decoder kernels on the scan's stream: its
 * launches count in `*launches`, its time in `*ms` (and `*stage`) */
struct Timer {
	cudaEvent_t e0, e1;
	uint64_t *launches;
	double *ms, *stage;
};

static Timer timer_start(dng_scan *s, uint64_t &launches, double &ms,
    double *stage = nullptr)
{
	Timer t = { get_event(s), get_event(s), &launches, &ms, stage };
	cudaEventRecord(t.e0, s->stream);
	return t;
}

/* the stage's n kernels are launched: count them, close the timer */
static void timer_stop(dng_scan *s, Timer &t, uint32_t n)
{
	cudaEventRecord(t.e1, s->stream);
	*t.launches += n;
	s->aux_launches += n;
}

/* once the stream is idle (or failed): the stage's time, and its events back
 * to the pool (dng_scan_destroy waits for the stream before freeing them) */
static void timer_read(dng_scan *s, Timer &t)
{
	float ms = 0;
	if (cudaEventElapsedTime(&ms, t.e0, t.e1) == cudaSuccess) {
		*t.ms += ms;
		if (t.stage)
			*t.stage += ms;
	}
	s->ev_pool.push_back(t.e0);
	s->ev_pool.push_back(t.e1);
}

/* the stage's n kernels are launched; its one wait: `bytes` of results from
 * `src` on the device to `dst`, then its time.  An error of the launch or the
 * wait fails the scan in the name of `kernel`. */
static int wait_results(dng_scan *s, Timer &t, uint32_t n, const char *kernel,
    void *dst, const void *src, size_t bytes)
{
	timer_stop(s, t, n);
	cudaError_t e = cudaGetLastError();
	if (e == cudaSuccess)
		e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost,
		    s->stream);
	if (e == cudaSuccess)
		e = cudaStreamSynchronize(s->stream);
	timer_read(s, t);
	return s->cuda(e, kernel);
}

/* fail the scan on a damaged file: "corrupt <format> data: <kind>", or the
 * kind alone when `format` is null, and where */
static int damage(dng_scan *s, const std::string &path, const char *format,
    const char *kind, uint64_t bit)
{
	const std::string what = format ?
	    std::string("corrupt ") + format + " data: " + kind : kind;
	return s->fail(DNG_EIO, path + ": " + what + " (compressed byte " +
	    std::to_string(bit / 8) + ")");
}

/* ---- gzip files (dng_scan_feed_gzip) -------------------------------------
 *
 * Queued files are inflated in batches by inflate_kernel (inflate.cuh), one
 * warp per file, into output regions laid out back to back in one device
 * buffer, each as large as its file's ISIZE trailer says (exact for a single
 * member under 4 GiB).  When every file filled its region exactly, the batch
 * is fed as one device buffer (one newline search, one wait).  Otherwise
 * each run of files that filled their regions is fed as one buffer, each file
 * that did not on its own, and a file that ran out of room is decoded again,
 * alone, in twice the room until it fits (several members, trailing zeros, or
 * >= 4 GiB).
 *
 * A batch holds at most 2 GiB of output room, 512 MiB of compressed bytes
 * and 256 files; a larger file goes alone.  One warp decodes one file, except
 * the large files of a batch of few, which are split (below).  Its buffers
 * (2.5 GiB) live beside the scan's own (table, arena, H2D ring: about
 * 2.5 GiB at the defaults), far below an H100's 80 GB.  Every batch buffer is written on the
 * scan's stream, after the scan kernels that read it earlier: a region stays
 * valid until those kernels have finished, as dng_scan_feed_device needs.
 */
static const size_t GZ_BATCH_OUT = (size_t)2 << 30;
static const size_t GZ_BATCH_IN = (size_t)512 << 20;
static const size_t GZ_BATCH_FILES = 256;

/* one inflate launch over jobs[0, n) on the scan's stream, and its results:
 * the one wait of a batch */
static int gz_launch(dng_scan *s, const InfJob *jobs, u32 n, InfResult *out)
{
	CzState *cz = s->cz;
	const size_t jb = GZ_BATCH_FILES * sizeof (InfJob);
	const size_t rb = GZ_BATCH_FILES * sizeof (InfResult);
	if (!cz->gz_jobs.p) {
		CK(s, DEV_ALLOC(s, &cz->gz_jobs.p, jb + rb + 64));
		CK(s, HOST_ALLOC(&cz->gz_jobs_host.p, jb + rb));
	}
	u8 *const d = cz->gz_jobs.p, *const h = cz->gz_jobs_host.p;
	memcpy(h, jobs, n * sizeof (InfJob));
	CK(s, cudaMemcpyAsync(d, h, n * sizeof (InfJob), cudaMemcpyHostToDevice,
	    s->stream));
	u32 *d_next = (u32 *)(d + jb + rb);
	CK(s, cudaMemsetAsync(d_next, 0, sizeof (u32), s->stream));
	Timer t = timer_start(s, cz->gz_launches, cz->gz_ms);
	const u32 grid = std::min<u32>((n + INF_WARPS - 1) / INF_WARPS,
	    (u32)s->sm_count * 4);
	inflate_kernel<<<grid, 32 * INF_WARPS, 0, s->stream>>>(
	    (const InfJob *)d, (InfResult *)(d + jb), n, d_next);
	if (wait_results(s, t, 1, "inflate_kernel", h + jb, d + jb,
	    n * sizeof (InfResult)))
		return s->err_code;
	memcpy(out, h + jb, n * sizeof (InfResult));
	return 0;
}

/* ---- gzip files split into chunks (inflate_split.cuh) ----------------------
 *
 * A batch with fewer files than the device holds decode warps cuts its large
 * files into chunks (gz_split_plan, inflate_policy.h).  Before the batch's
 * one wait: split_find_kernel finds each chunk's candidate block start and
 * split_decode_kernel decodes every chunk into 16-bit symbols.  After it the
 * host chains each file's chunks; a chain that ends in a chunk out of room
 * decodes that chunk, and each later one that ran out, again in four times
 * the room and member slots.  Then split_tail_kernel and split_body_kernel
 * write each file's bytes, into its region when its length is the hint and
 * into gz_sout otherwise, and split_crc_kernel and split_member_kernel
 * check every member.  A file the split path cannot vouch for is decoded
 * again by inflate_kernel, whose answer stands.
 *
 * Scratch, from the buffer cache: 16-bit symbols for 1.25 times each split
 * file's hint plus 32 Ki symbols per chunk (2.5 times the batch's output
 * room, plus 64 KiB per chunk), and four times that for each chunk decoded
 * again; per chunk its candidate, job, result and four member slots; the
 * pieces and members of the checks.
 */
struct GzChunk {		/* host state of one chunk */
	SplitJob job;
	SplitRes res;
	std::vector<InfMember> mem;
};

struct GzSplitFile {
	size_t file;			/* in the batch */
	uint32_t first, n;		/* its chunks in the batch's list */
	int chain;
	std::vector<uint32_t> proven;
	SplitLayout lay;
	u8 *dst;
	bool ok;
};

static uint64_t gz_resident(dng_scan *s)
{
	CzState *cz = s->cz;
	if (!cz->gz_split_blocks) {
		int b = 0;
		cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b,
		    split_decode_kernel, 32 * SPLIT_WARPS, 0);
		cz->gz_split_blocks = b > 0 ? (uint32_t)b : 1;
	}
	return (uint64_t)cz->gz_split_blocks * SPLIT_WARPS * s->sm_count;
}

/* split_decode_kernel over the chunks `which` (their jobs set), on the
 * stream; device records at d_jobs / d_res */
static int gz_split_decode(dng_scan *s, std::vector<GzChunk> &ck,
    const std::vector<uint32_t> &which, u8 *d_jobs, u8 *d_res, u32 *d_next)
{
	const size_t n = which.size();
	std::vector<SplitJob> jobs(n);
	for (size_t i = 0; i < n; i++)
		jobs[i] = ck[which[i]].job;
	CK(s, cudaMemcpyAsync(d_jobs, jobs.data(), n * sizeof (SplitJob),
	    cudaMemcpyHostToDevice, s->stream));
	CK(s, cudaMemsetAsync(d_next, 0, sizeof (u32), s->stream));
	gz_resident(s);
	const u32 grid = std::min<u32>((u32)((n + SPLIT_WARPS - 1) / SPLIT_WARPS),
	    s->cz->gz_split_blocks * (u32)s->sm_count);
	split_decode_kernel<<<grid, 32 * SPLIT_WARPS, 0, s->stream>>>(
	    (const SplitJob *)d_jobs, (SplitRes *)d_res, (u32)n, d_next);
	CK(s, cudaGetLastError());
	return 0;
}

/* 1 and 2: enqueue the finder and the first decode of every chunk of the
 * split files (no wait) */
static int gz_split_start(dng_scan *s, const std::vector<CzFile> &q,
    const std::vector<size_t> &in_off, const std::vector<u32> &nch,
    std::vector<GzSplitFile> &sf, std::vector<GzChunk> &ck, Timer &t)
{
	CzState *cz = s->cz;
	uint32_t total = 0;
	uint64_t room = 0;
	for (size_t i = 0; i < q.size(); i++) {
		if (nch[i] < 2)
			continue;
		GzSplitFile f = {};
		f.file = i;
		f.first = total;
		f.n = nch[i];
		sf.push_back(f);
		total += nch[i];
		const CzFile &g = q[i];
		for (uint32_t k = 0; k < f.n; k++) {
			const uint64_t cb = split_cut(g.size, f.n, k + 1) -
			    split_cut(g.size, f.n, k);
			ck.emplace_back();
			SplitJob &j = ck.back().job;
			j = {};
			j.in = cz->in.p + in_off[f.file];
			j.in_len = g.size;
			j.cap = split_room(g.hint, g.size, cb);
			j.k = k;
			j.nchunks = f.n;
			j.mcap = SPLIT_MSLOTS;
			room += j.cap;
		}
	}
	/* candidates | find jobs | decode jobs | results | member slots | next */
	const size_t oc = 0, of = oc + total * sizeof (uint64_t),
	    oj = of + total * sizeof (SplitFind),
	    orr = oj + total * sizeof (SplitJob),
	    om = orr + total * sizeof (SplitRes),
	    on = om + (size_t)total * SPLIT_MSLOTS * sizeof (InfMember);
	if (grow(s, cz->gz_split, on + 16) || grow(s, cz->gz_sym, room * 2))
		return s->err_code;
	u8 *const d = cz->gz_split.p;
	uint64_t *d_cand = (uint64_t *)(d + oc);
	std::vector<SplitFind> finds;
	uint64_t sym = 0;
	for (const GzSplitFile &f : sf) {
		const CzFile &g = q[f.file];
		for (uint32_t k = 0; k < f.n; k++) {
			SplitJob &j = ck[f.first + k].job;
			j.cand = d_cand + f.first;
			j.out = (uint16_t *)cz->gz_sym.p + sym;
			j.mem = (InfMember *)(d + om) +
			    (size_t)(f.first + k) * SPLIT_MSLOTS;
			sym += j.cap;
			if (k)
				finds.push_back({ j.in, g.size,
				    split_cut(g.size, f.n, k) * 8,
				    split_cut(g.size, f.n, k + 1) * 8,
				    d_cand + f.first + k });
		}
	}
	CK(s, cudaMemcpyAsync(d + of, finds.data(),
	    finds.size() * sizeof (SplitFind), cudaMemcpyHostToDevice,
	    s->stream));
	t = timer_start(s, cz->gz_split_launches, cz->gz_ms);
	const u32 grid = std::min<u32>((u32)finds.size(), (u32)s->sm_count * 6);
	split_find_kernel<<<grid, 32, 0, s->stream>>>(
	    (const SplitFind *)(d + of), (u32)finds.size());
	CK(s, cudaGetLastError());
	std::vector<uint32_t> all(total);
	std::iota(all.begin(), all.end(), 0u);
	if (gz_split_decode(s, ck, all, d + oj, d + orr, (u32 *)(d + on)))
		return s->err_code;
	timer_stop(s, t, 2);
	return 0;
}

/* results of chunks `which`, decoded into d_res, and their member records
 * from the slots [d_mem, + nslots) their jobs point into */
static int gz_split_collect(dng_scan *s, std::vector<GzChunk> &ck,
    const std::vector<uint32_t> &which, const u8 *d_res,
    const InfMember *d_mem, size_t nslots)
{
	std::vector<SplitRes> r(which.size());
	std::vector<InfMember> m(nslots);
	CK(s, cudaMemcpyAsync(r.data(), d_res, r.size() * sizeof (SplitRes),
	    cudaMemcpyDeviceToHost, s->stream));
	CK(s, cudaMemcpyAsync(m.data(), d_mem, nslots * sizeof (InfMember),
	    cudaMemcpyDeviceToHost, s->stream));
	CK(s, cudaStreamSynchronize(s->stream));
	for (size_t i = 0; i < which.size(); i++) {
		GzChunk &c = ck[which[i]];
		c.res = r[i];
		const InfMember *h = m.data() + (c.job.mem - d_mem);
		c.mem.assign(h, h + c.res.members);
	}
	return 0;
}

/*
 * 3 to 5, after the batch's wait: chain, decode again what ran out of room,
 * resolve and check.  by_file[i] of a split file: DONE with its length and
 * members (alt[i]: where its bytes are when not in its region), or ROOM,
 * to be decoded whole (a fallback).
 */
static int gz_split_finish(dng_scan *s, const std::vector<CzFile> &q,
    const std::vector<size_t> &out_off, std::vector<GzSplitFile> &sf,
    std::vector<GzChunk> &ck, std::vector<InfResult> &by_file,
    std::vector<const u8 *> &alt)
{
	CzState *cz = s->cz;
	std::vector<uint32_t> all(ck.size());
	std::iota(all.begin(), all.end(), 0u);
	const size_t orr = ck.size() * (sizeof (uint64_t) + sizeof (SplitFind) +
	    sizeof (SplitJob)), om = orr + ck.size() * sizeof (SplitRes);
	if (gz_split_collect(s, ck, all, cz->gz_split.p + orr,
	    (const InfMember *)(cz->gz_split.p + om), ck.size() * SPLIT_MSLOTS))
		return s->err_code;
	std::list<DevBuf> extra;	/* rooms of chunks decoded again */
	for (;;) {
		std::vector<uint32_t> redo, r;
		for (GzSplitFile &f : sf) {
			std::vector<SplitRes> res(f.n);
			for (uint32_t k = 0; k < f.n; k++)
				res[k] = ck[f.first + k].res;
			f.chain = split_chain(res.data(), f.proven);
			if (f.chain != CHAIN_ROOM)
				continue;
			split_redo(res.data(), f.n, f.proven, r);
			for (const uint32_t k : r)
				redo.push_back(f.first + k);
		}
		if (redo.empty())
			break;
		uint64_t room = 0, slots = 0;
		for (const uint32_t c : redo) {
			room += ck[c].job.cap * 4;
			slots += ck[c].job.mcap * 4;
		}
		const size_t bj = redo.size() * sizeof (SplitJob),
		    br = redo.size() * sizeof (SplitRes),
		    bm = slots * sizeof (InfMember);
		extra.emplace_back();
		CK(s, DEV_ALLOC(s, &extra.back().p,
		    room * 2 + bj + br + bm + 16));
		u8 *const d = extra.back().p;
		uint64_t sym = 0, slot = 0;
		for (const uint32_t c : redo) {
			SplitJob &j = ck[c].job;
			j.cap *= 4;
			j.mcap *= 4;
			j.out = (uint16_t *)d + sym;
			j.mem = (InfMember *)(d + room * 2 + bj + br) + slot;
			sym += j.cap;
			slot += j.mcap;
		}
		Timer t = timer_start(s, cz->gz_split_launches, cz->gz_ms);
		if (gz_split_decode(s, ck, redo, d + room * 2, d + room * 2 + bj,
		    (u32 *)(d + room * 2 + bj + br + bm)))
			return s->err_code;
		timer_stop(s, t, 1);
		const int rc = gz_split_collect(s, ck, redo, d + room * 2 + bj,
		    (const InfMember *)(d + room * 2 + bj + br), slots);
		timer_read(s, t);
		if (rc)
			return rc;
	}
	/* lay out every file whose chain reached the end */
	size_t sout = 0;
	for (GzSplitFile &f : sf) {
		f.ok = f.chain == CHAIN_END;
		cz->gz_split_files++;
		cz->gz_chunks += f.n;
		if (!f.ok)
			continue;
		std::vector<SplitRes> res(f.n);
		std::vector<const InfMember *> mem(f.n);
		for (uint32_t k = 0; k < f.n; k++) {
			res[k] = ck[f.first + k].res;
			mem[k] = ck[f.first + k].mem.data();
		}
		cz->gz_false_starts += split_false_starts(res.data(), f.n,
		    f.proven);
		split_layout(res.data(), mem.data(), f.proven, f.lay);
		if (f.lay.len != q[f.file].hint)
			sout += align_up(f.lay.len, 16);
	}
	if (sout && grow(s, cz->gz_sout, sout))
		return s->err_code;
	/* resolve pieces | first | bad | CRC pieces | CRCs | members */
	std::vector<SplitPiece> pieces;
	std::vector<u32> first;
	std::vector<CrcPiece> cp;
	std::vector<CrcMember> cm;
	std::vector<GzSplitFile *> okf;
	sout = 0;
	for (GzSplitFile &f : sf) {
		if (!f.ok)
			continue;
		const u32 fi = (u32)okf.size();
		okf.push_back(&f);
		if (f.lay.len == q[f.file].hint) {
			f.dst = cz->gz_out.p + out_off[f.file];
		} else {
			f.dst = cz->gz_sout.p + sout;
			sout += align_up(f.lay.len, 16);
		}
		first.push_back((u32)pieces.size());
		for (size_t i = 0; i < f.proven.size(); i++) {
			const GzChunk &c = ck[f.first + f.proven[i]];
			pieces.push_back({ c.job.out, f.dst, f.lay.off[i],
			    c.res.out_len, f.lay.minidx[i], fi });
		}
		for (size_t m = 0; m < f.lay.mstart.size(); m++) {
			CrcMember x = { (u32)cp.size(), 0, f.lay.crc[m],
			    f.lay.isize[m], f.lay.mend[m] - f.lay.mstart[m], fi,
			    0 };
			for (uint64_t a = f.lay.mstart[m]; a < f.lay.mend[m];
			    a += SPLIT_CRC_PIECE)
				cp.push_back({ f.dst + a, std::min<uint64_t>(
				    SPLIT_CRC_PIECE, f.lay.mend[m] - a) });
			x.p1 = (u32)cp.size();
			cm.push_back(x);
		}
	}
	first.push_back((u32)pieces.size());
	const size_t nok = okf.size();
	std::vector<u32> bad(nok, 0);
	if (nok) {
		const size_t o1 = pieces.size() * sizeof (SplitPiece),
		    o2 = o1 + first.size() * sizeof (u32),
		    o3 = align_up(o2 + nok * sizeof (u32), 16),
		    o4 = o3 + cp.size() * sizeof (CrcPiece),
		    o5 = align_up(o4 + cp.size() * sizeof (u32), 16),
		    o6 = o5 + cm.size() * sizeof (CrcMember);
		if (grow(s, cz->gz_check, o6))
			return s->err_code;
		u8 *d = cz->gz_check.p;
		CK(s, cudaMemcpyAsync(d, pieces.data(), o1,
		    cudaMemcpyHostToDevice, s->stream));
		CK(s, cudaMemcpyAsync(d + o1, first.data(), o2 - o1,
		    cudaMemcpyHostToDevice, s->stream));
		CK(s, cudaMemsetAsync(d + o2, 0, nok * sizeof (u32), s->stream));
		if (!cp.empty())
			CK(s, cudaMemcpyAsync(d + o3, cp.data(), o4 - o3,
			    cudaMemcpyHostToDevice, s->stream));
		if (!cm.empty())
			CK(s, cudaMemcpyAsync(d + o5, cm.data(), o6 - o5,
			    cudaMemcpyHostToDevice, s->stream));
		u32 *d_bad = (u32 *)(d + o2);
		Timer t = timer_start(s, cz->gz_split_launches, cz->gz_ms);
		split_tail_kernel<<<(u32)nok, 1024, 0, s->stream>>>(
		    (const SplitPiece *)d, (const u32 *)(d + o1), d_bad);
		split_body_kernel<<<(u32)pieces.size(), 256, 0, s->stream>>>(
		    (const SplitPiece *)d, d_bad);
		if (!cp.empty()) {
			split_crc_kernel<<<(u32)((cp.size() + 255) / 256), 256, 0,
			    s->stream>>>((const CrcPiece *)(d + o3),
			    (u32 *)(d + o4), (u32)cp.size());
			split_member_kernel<<<(u32)((cm.size() + 3) / 4), 128, 0,
			    s->stream>>>((const CrcMember *)(d + o5),
			    (u32)cm.size(), (const CrcPiece *)(d + o3),
			    (const u32 *)(d + o4), d_bad);
		}
		if (wait_results(s, t, cp.empty() ? 2 : 4, "split check kernels",
		    bad.data(), d_bad, nok * sizeof (u32)))
			return s->err_code;
	}
	for (size_t fi = 0; fi < nok; fi++)
		okf[fi]->ok = !bad[fi];
	for (const GzSplitFile &f : sf) {
		InfResult &r = by_file[f.file];
		r = {};
		if (!f.ok) {
			r.status = INF_ROOM;	/* decoded whole */
			cz->gz_fallbacks++;
			continue;
		}
		r.status = INF_DONE;
		r.out_len = f.lay.len;
		r.members = (uint32_t)f.lay.mstart.size();
		if (f.dst != cz->gz_out.p + out_off[f.file])
			alt[f.file] = f.dst;
	}
	return 0;
}

/* inflate and feed a batch of gzip files, whose compressed bytes are in
 * the batch buffer at in_off, in the order they were fed */
static int gz_batch(dng_scan *s, const std::vector<CzFile> &q,
    const std::vector<size_t> &in_off)
{
	CzState *cz = s->cz;
	const size_t n = q.size();
	std::vector<size_t> out_off(n);
	size_t tout = 0;
	for (size_t i = 0; i < n; i++) {
		out_off[i] = tout;
		tout += q[i].hint;
	}
	if (grow(s, cz->gz_out, tout))
		return s->err_code;
	/* large files of a batch of few: split (inflate_policy.h) */
	std::vector<uint64_t> sizes(n);
	for (size_t i = 0; i < n; i++)
		sizes[i] = q[i].size;
	std::vector<u32> nch(n);
	gz_split_plan(sizes.data(), n, gz_resident(s), DNG_GZ_SPLIT_FLOOR,
	    nch.data());
	std::vector<GzSplitFile> sf;
	std::vector<GzChunk> ck;
	Timer st = {};
	for (size_t i = 0; i < n; i++)
		if (nch[i] > 1) {
			if (gz_split_start(s, q, in_off, nch, sf, ck, st))
				return s->err_code;
			break;
		}
	/* the rest one warp each, largest first, so that no big file is left
	 * running alone */
	std::vector<u32> order;
	for (size_t i = 0; i < n; i++)
		if (nch[i] < 2)
			order.push_back((u32)i);
	std::stable_sort(order.begin(), order.end(), [&](u32 a, u32 b) {
		return q[a].size > q[b].size;
	});
	auto whole = [&](const std::vector<u32> &files,
	    std::vector<InfResult> &by) {
		std::vector<InfJob> jobs(files.size());
		std::vector<InfResult> res(files.size());
		for (size_t k = 0; k < files.size(); k++) {
			const u32 i = files[k];
			jobs[k] = { cz->in.p + in_off[i], q[i].size,
			    cz->gz_out.p + out_off[i], q[i].hint };
		}
		if (gz_launch(s, jobs.data(), (u32)files.size(), res.data()))
			return s->err_code;
		for (size_t k = 0; k < files.size(); k++)
			by[files[k]] = res[k];
		return 0;
	};
	std::vector<InfResult> by_file(n);
	std::vector<const u8 *> alt(n, nullptr);
	if (!order.empty() && whole(order, by_file))
		return s->err_code;
	if (!sf.empty()) {
		if (order.empty())
			CK(s, cudaStreamSynchronize(s->stream));
		timer_read(s, st);
		if (gz_split_finish(s, q, out_off, sf, ck, by_file, alt))
			return s->err_code;
		/* what the split path could not vouch for, decoded whole */
		std::vector<u32> again;
		for (const GzSplitFile &f : sf)
			if (!f.ok)
				again.push_back((u32)f.file);
		if (!again.empty() && whole(again, by_file))
			return s->err_code;
	}
	for (size_t i = 0; i < n; i++) {
		if (by_file[i].status == INF_ERROR)
			return damage(s, q[i].path, "gzip",
			    inflate_error_name(by_file[i].kind), by_file[i].bit);
		cz->gz_in_bytes += q[i].size;
	}
	cz->gz_files += n;
	/* in file order: each run of files that filled their regions exactly
	 * is one feed (the whole batch when every hint held); a file that did
	 * not is fed on its own, decoded again in more room if it ran out */
	auto filled = [&](size_t i) {
		return by_file[i].status == INF_DONE &&
		    by_file[i].out_len == q[i].hint;
	};
	for (size_t i = 0, next; i < n; i = next) {
		const u8 *src = cz->gz_out.p + out_off[i];
		uint64_t len = 0;
		next = i + 1;
		if (filled(i)) {
			while (next < n && filled(next))
				next++;
			for (size_t k = i; k < next; k++) {
				cz->gz_members += by_file[k].members;
				len += by_file[k].out_len;
			}
		} else {
			InfResult r = by_file[i];
			if (alt[i])	/* split, and not the hint's length */
				src = alt[i];
			uint64_t cap = q[i].hint;
			while (r.status == INF_ROOM) {
				cap = std::max<uint64_t>(cap * 2,
				    (uint64_t)1 << 20);
				if (grow(s, cz->gz_big, cap))
					return s->err_code;
				const InfJob j = { cz->in.p + in_off[i],
				    q[i].size, cz->gz_big.p, cap };
				if (gz_launch(s, &j, 1, &r))
					return s->err_code;
				src = cz->gz_big.p;
			}
			if (r.status == INF_ERROR)
				return damage(s, q[i].path, "gzip",
				    inflate_error_name(r.kind), r.bit);
			cz->gz_members += r.members;
			len = r.out_len;
		}
		cz->gz_out_bytes += len;
		if (!len)
			continue;	/* (an empty file adds nothing) */
		if ((uintptr_t)src & 15) {
			/* regions start where the hints before them end: a run
			 * after a file that missed its hint is realigned */
			if (grow(s, cz->gz_join, len))
				return s->err_code;
			CK(s, cudaMemcpyAsync(cz->gz_join.p, src, len,
			    cudaMemcpyDeviceToDevice, s->stream));
			src = cz->gz_join.p;
		}
		if (feed_device(s, src, len))
			return s->err_code;
	}
	return 0;
}

/* ---- bzip2 files (dng_scan_feed_bzip2) -------------------------------------
 *
 * A batch (the queue's limits: 256 files, 512 MiB compressed) is decoded by
 * the stages of bunzip.cuh.  bz_find_kernel finds every candidate magic of
 * every file; after that wait the host sorts them per file and cuts the block
 * candidates into waves (bunzip_policy.h).  Per wave: bz_decode_kernel
 * decodes every candidate (one wait), the host advances each file's chain
 * through them, bz_ibwt_kernel inverts the chained blocks and sizes their
 * output (one wait), and bz_emit_kernel writes each group of blocks back to
 * back, files in feed order, with their CRCs (one wait per group).  A group
 * is fed as one device buffer once its CRCs hold.  Every buffer is written on
 * the scan's stream, after the scan kernels that read it earlier.
 */

/* every candidate magic of the batch, sorted by file and bit, and each
 * file's one past its last nonzero byte */
static int bz_find(dng_scan *s, const std::vector<CzFile> &q,
    const std::vector<size_t> &in_off, std::vector<BzCand> &cand,
    std::vector<unsigned long long> &nz)
{
	CzState *cz = s->cz;
	const size_t n = q.size();
	uint64_t tin = 0, maxlen = 0;
	std::vector<BzFile> files(n);
	for (size_t i = 0; i < n; i++) {
		files[i] = { cz->in.p + in_off[i], q[i].size };
		tin += q[i].size;
		maxlen = std::max<uint64_t>(maxlen, q[i].size);
	}
	/* files | each file's nz, then the candidate count, read back in one
	 * copy | candidates */
	const size_t o_nz = align_up(n * sizeof (BzFile), 256);
	const size_t o_cnt = o_nz + n * 8;
	const size_t o_cand = align_up(o_cnt + 8, 256);
	size_t cap = tin / 512 + 4096;
	uint32_t count = 0;
	nz.resize(n + 1);
	for (;;) {
		if (grow(s, cz->bz_find, o_cand + cap * sizeof (BzCand)))
			return s->err_code;
		u8 *const d = cz->bz_find.p;
		CK(s, cudaMemcpyAsync(d, files.data(), n * sizeof (BzFile),
		    cudaMemcpyHostToDevice, s->stream));
		CK(s, cudaMemsetAsync(d + o_nz, 0, o_cand - o_nz, s->stream));
		const uint64_t per = 256 * 16;	/* bytes per CTA and sweep */
		const dim3 grid((u32)std::min<uint64_t>(std::max<uint64_t>(
		    (maxlen + per - 1) / per, 1), 65535), (u32)n);
		Timer t = timer_start(s, cz->bz_launches, cz->bz_ms,
		    &cz->bz_stage_ms[0]);
		bz_find_kernel<<<grid, 256, 0, s->stream>>>(
		    (const BzFile *)d, (BzCand *)(d + o_cand), (u32)cap,
		    (u32 *)(d + o_cnt), (unsigned long long *)(d + o_nz));
		if (wait_results(s, t, 1, "bz_find_kernel", nz.data(), d + o_nz,
		    (n + 1) * 8))
			return s->err_code;
		count = (uint32_t)nz[n];
		if (count <= cap)
			break;
		cap = count;	/* more candidates than room: find again */
	}
	nz.pop_back();
	cand.resize(count);
	if (count) {
		CK(s, cudaMemcpyAsync(cand.data(), cz->bz_find.p + o_cand,
		    count * sizeof (BzCand), cudaMemcpyDeviceToHost, s->stream));
		CK(s, cudaStreamSynchronize(s->stream));
	}
	std::sort(cand.begin(), cand.end(), [](const BzCand &a,
	    const BzCand &b) {
		return a.file != b.file ? a.file < b.file : a.bit < b.bit;
	});
	return 0;
}

/* decode, chain, invert and emit a batch of bzip2 files (above) */
static int bz_batch(dng_scan *s, const std::vector<CzFile> &q,
    const std::vector<size_t> &in_off)
{
	CzState *cz = s->cz;
	const size_t n = q.size();
	std::vector<BzCand> cand;
	std::vector<unsigned long long> nz;
	if (bz_find(s, q, in_off, cand, nz))
		return s->err_code;
	/* each file's candidates, and the block candidates in order */
	std::vector<u32> fbeg(n + 1, 0), bidx, which(cand.size(), ~0u);
	for (const BzCand &c : cand)
		fbeg[c.file + 1]++;
	for (size_t i = 0; i < n; i++)
		fbeg[i + 1] += fbeg[i];
	for (u32 i = 0; i < cand.size(); i++)
		if (cand[i].kind == BZ_CAND_BLOCK) {
			which[i] = (u32)bidx.size();
			bidx.push_back(i);
		}
	std::vector<size_t> ends(bidx.size() + 1);
	const size_t nw = bz_waves(bidx.size(), DNG_BZ_WAVE_BLOCKS,
	    ends.data());
	std::vector<BzChain> ch(n);
	for (size_t i = 0; i < n; i++)
		bz_chain_init(ch[i], q[i].size, nz[i], q[i].head);
	std::vector<BzDecResult> res(bidx.size());
	size_t f = 0;	/* the first file whose chain is not done */
	for (size_t w = 0, lo = 0;; w++) {
		const size_t hi = w < nw ? ends[w] : lo, wn = hi - lo;
		size_t o = 0;
		auto at = [&](size_t bytes) {
			const size_t r = o;
			o += align_up(bytes, 256);
			return r;
		};
		const size_t o_dj = at(wn * sizeof (BzDecJob));
		const size_t o_dr = at(wn * sizeof (BzDecResult));
		const size_t o_hist = at(wn * 256 * 4), o_next = at(16);
		const size_t o_bj = at(wn * sizeof (BzBwtJob));
		const size_t o_br = at(wn * sizeof (BzBwtResult));
		const size_t o_ck = at(wn * BZ_CHUNKS * 8);
		const size_t o_ej = at(wn * sizeof (BzEmitJob));
		const size_t o_crc = at(wn * 4);
		u8 *rec = nullptr;
		if (wn) {
			/* decode the wave's candidates, one warp each */
			if (grow(s, cz->bz_rec, o) ||
			    grow(s, cz->bz_slot, wn * (size_t)BZ_SLOT))
				return s->err_code;
			rec = cz->bz_rec.p;
			std::vector<BzDecJob> dj(wn);
			for (size_t k = 0; k < wn; k++) {
				const BzCand &c = cand[bidx[lo + k]];
				dj[k] = { cz->in.p + in_off[c.file],
				    q[c.file].size, c.bit,
				    cz->bz_slot.p + k * (size_t)BZ_SLOT,
				    (uint32_t *)(rec + o_hist) + k * 256 };
			}
			CK(s, cudaMemcpyAsync(rec + o_dj, dj.data(),
			    wn * sizeof (BzDecJob), cudaMemcpyHostToDevice,
			    s->stream));
			CK(s, cudaMemsetAsync(rec + o_next, 0, 16, s->stream));
			const u32 grid = (u32)std::min<size_t>((wn + BZ_DEC_WARPS -
			    1) / BZ_DEC_WARPS, (size_t)s->sm_count * 8);
			Timer t = timer_start(s, cz->bz_launches, cz->bz_ms,
			    &cz->bz_stage_ms[1]);
			bz_decode_kernel<<<grid, 32 * BZ_DEC_WARPS, 0,
			    s->stream>>>((const BzDecJob *)(rec + o_dj),
			    (BzDecResult *)(rec + o_dr), (u32)wn,
			    (u32 *)(rec + o_next));
			if (wait_results(s, t, 1, "bz_decode_kernel",
			    res.data() + lo, rec + o_dr,
			    wn * sizeof (BzDecResult)))
				return s->err_code;
		}
		/* chain every file the decodes so far reach, in feed order; a
		 * damaged file stops it, and fails the scan once the blocks
		 * before the damage have passed their CRCs */
		std::vector<u32> took;
		bool early = false;
		size_t damaged = n;
		for (; f < n; f++) {
			BzChain &c = ch[f];
			const u32 b0 = fbeg[f];
			bz_chain_run(c, cand.data() + b0, fbeg[f + 1] - b0,
			    [&](u32 i) -> const BzDecResult * {
				const size_t k = which[b0 + i];
				return k < hi ? &res[k] : nullptr;
			    }, [&](u32 i) {
				early |= which[b0 + i] < lo;
				took.push_back(which[b0 + i]);
			    });
			if (c.kind) {
				damaged = f;
				break;
			}
			if (early)
				return s->fail(DNG_EIO, q[f].path + ": bzip2 "
				    "chain went back to an earlier wave");
			if (!c.done)
				break;
		}
		cz->bz_false_starts += wn - took.size();
		const size_t m = took.size();
		if (m) {
			/* invert the chained blocks, one CTA each */
			std::vector<size_t> tt_off(m);
			size_t tsum = 0;
			for (size_t k = 0; k < m; k++) {
				tt_off[k] = tsum;
				tsum += align_up((size_t)res[took[k]].nblock * 4,
				    16);
			}
			if (grow(s, cz->bz_tt, tsum))
				return s->err_code;
			std::vector<BzBwtJob> bj(m);
			for (size_t k = 0; k < m; k++) {
				const size_t c = took[k] - lo;
				const BzDecResult &r = res[took[k]];
				bj[k] = { cz->bz_slot.p + c * (size_t)BZ_SLOT,
				    (uint32_t *)(cz->bz_tt.p + tt_off[k]),
				    (const uint32_t *)(rec + o_hist) + c * 256,
				    (uint32_t *)(rec + o_ck) + k * BZ_CHUNKS * 2,
				    r.nblock, r.orig, r.rand, 0 };
			}
			CK(s, cudaMemcpyAsync(rec + o_bj, bj.data(),
			    m * sizeof (BzBwtJob), cudaMemcpyHostToDevice,
			    s->stream));
			std::vector<BzBwtResult> br(m);
			Timer t = timer_start(s, cz->bz_launches, cz->bz_ms,
			    &cz->bz_stage_ms[2]);
			bz_ibwt_kernel<<<(u32)m, BZ_THREADS, 0, s->stream>>>(
			    (const BzBwtJob *)(rec + o_bj),
			    (BzBwtResult *)(rec + o_br));
			if (wait_results(s, t, 1, "bz_ibwt_kernel", br.data(),
			    rec + o_br, m * sizeof (BzBwtResult)))
				return s->err_code;
			std::vector<uint64_t> lens(m);
			for (size_t k = 0; k < m; k++) {
				const BzCand &c = cand[bidx[took[k]]];
				if (!br[k].ok)	/* a run without its count */
					return damage(s, q[c.file].path,
					    "bzip2",
					    bunzip_error_name(BE_OVERFLOW),
					    c.bit);
				lens[k] = br[k].out_len;
			}
			/* emit in groups, each fed once its CRCs hold */
			std::vector<size_t> gend(m);
			const size_t ng = bz_emit_groups(lens.data(), m,
			    DNG_BZ_EMIT_OUT, gend.data());
			for (size_t g = 0, g0 = 0; g < ng; g0 = gend[g++]) {
				const size_t g1 = gend[g];
				uint64_t sum = 0;
				std::vector<BzEmitJob> ej(g1 - g0);
				for (size_t k = g0; k < g1; k++)
					sum += lens[k];
				if (grow(s, cz->bz_out, sum))
					return s->err_code;
				uint64_t off = 0;
				for (size_t k = g0; k < g1; k++) {
					ej[k - g0] = { bj[k].slot, bj[k].chunks,
					    cz->bz_out.p + off, bj[k].n, 0 };
					off += lens[k];
				}
				CK(s, cudaMemcpyAsync(rec + o_ej, ej.data(),
				    ej.size() * sizeof (BzEmitJob),
				    cudaMemcpyHostToDevice, s->stream));
				std::vector<uint32_t> crc(g1 - g0);
				Timer te = timer_start(s, cz->bz_launches,
				    cz->bz_ms, &cz->bz_stage_ms[3]);
				bz_emit_kernel<<<(u32)(g1 - g0), BZ_THREADS, 0,
				    s->stream>>>((const BzEmitJob *)(rec + o_ej),
				    (uint32_t *)(rec + o_crc));
				if (wait_results(s, te, 1, "bz_emit_kernel",
				    crc.data(), rec + o_crc, crc.size() * 4))
					return s->err_code;
				for (size_t k = g0; k < g1; k++)
					if (crc[k - g0] != res[took[k]].crc) {
						const BzCand &c =
						    cand[bidx[took[k]]];
						return damage(s,
						    q[c.file].path, "bzip2",
						    bunzip_error_name(
						    BE_BLOCK_CRC), c.bit);
					}
				cz->bz_out_bytes += sum;
				if (feed_device(s, cz->bz_out.p, sum))
					return s->err_code;
			}
		}
		if (damaged < n) {
			/* (trailing data is not corrupt bzip2 data) */
			const BzChain &c = ch[damaged];
			return damage(s, q[damaged].path, c.kind == BE_TRAILING ?
			    nullptr : "bzip2", bunzip_error_name(c.kind),
			    c.err_bit);
		}
		lo = hi;
		if (f == n) {
			/* candidates past every chain's end: never decoded */
			cz->bz_false_starts += bidx.size() - hi;
			break;
		}
		if (w >= nw)
			return s->fail(DNG_EIO, q[f].path + ": bzip2 chain "
			    "stopped before its end");
	}
	for (size_t i = 0; i < n; i++) {
		cz->bz_in_bytes += q[i].size;
		cz->bz_streams += ch[i].streams;
		cz->bz_blocks += ch[i].blocks;
	}
	cz->bz_files += n;
	return 0;
}

int cz_flush(dng_scan *s)
{
	CzState *cz = s->cz;
	if (!cz || cz->queue.empty())
		return s->err_code;
	std::vector<CzFile> q;
	q.swap(cz->queue);
	cz->queued_in = cz->queued_out = 0;
	if (s->err_code)
		return s->err_code;
	const size_t n = q.size();
	std::vector<size_t> in_off(n);
	size_t tin = 0;
	for (size_t i = 0; i < n; i++) {
		in_off[i] = tin;
		tin += align_up(q[i].size, 16);
	}
	if (grow(s, cz->in, tin))
		return s->err_code;
	/* compressed bytes through the file reader (direct_read.h's policy) */
	for (size_t i = 0; i < n; i++)
		if (read_to_device(s, q[i].path.c_str(), q[i].size,
		    cz->in.p + in_off[i]))
			return s->err_code;
	return cz->bzip2 ? bz_batch(s, q, in_off) : gz_batch(s, q, in_off);
}

/*
 * What dng_scan_feed_gzip and dng_scan_feed_bzip2 share: the scan's checks;
 * the file, which must be a regular file that `accept` takes by what it reads
 * of it (refused with `refusal` if not: not failed, the scan goes on); then
 * the queue, flushed first when it holds the other format or the file would
 * take it past a batch's limits.
 */
static int cz_feed(dng_scan *s, const char *path, const char *what,
    bool bzip2, const char *refusal,
    bool (*accept)(int fd, size_t size, CzFile &f))
{
	if (!s || !path)
		return DNG_EINVAL;
	if (s->multi)
		return refuse_multi(s, what);
	if (s->err_code)
		return s->err_code;
	if (s->finished)
		return s->fail(DNG_EINVAL, "scan already finished");
	cudaSetDevice(s->device);
	int fd = open(path, O_RDONLY);
	if (fd < 0)
		return s->fail(DNG_EIO, std::string("open ") + path + ": " +
		    strerror(errno));
	struct stat st;
	const bool reg = fstat(fd, &st) == 0 && S_ISREG(st.st_mode);
	CzFile f = { path, reg ? (size_t)st.st_size : 0, 0, 0 };
	const bool ok = reg && accept(fd, f.size, f);
	close(fd);
	if (!ok) {
		if (!s->err_code)
			s->err = std::string(path) + (reg ? refusal :
			    ": not a regular file");
		return DNG_EINVAL;
	}
	if (!s->cz) {
		s->cz = new CzState();
		/* the decoders' module loads here, not in a stage's timer */
		cudaFuncAttributes fa;
		cudaFuncGetAttributes(&fa, bz_find_kernel);
	}
	CzState *cz = s->cz;
	const size_t in = align_up(f.size, 16);
	if (!cz->queue.empty() && (cz->bzip2 != bzip2 ||
	    cz->queue.size() >= GZ_BATCH_FILES ||
	    cz->queued_in + in > GZ_BATCH_IN ||
	    cz->queued_out + f.hint > GZ_BATCH_OUT) && cz_flush(s))
		return s->err_code;
	cz->bzip2 = bzip2;
	cz->queued_in += in;
	cz->queued_out += f.hint;
	cz->queue.push_back(std::move(f));
	return DNG_OK;
}

/* the stats of a scan that never queued a compressed file */
static const CzState &stats(const dng_scan *s)
{
	static const CzState none;
	return s->cz ? *s->cz : none;
}

int dng_scan_feed_gzip(dng_scan *s, const char *path)
{
	return cz_feed(s, path, "dng_scan_feed_gzip", false,
	    ": not a gzip file (it does not start with 1f 8b 08)",
	    [](int fd, size_t size, CzFile &f) {
		u8 head[3], tail[4];
		if (size < 3 || pread(fd, head, 3, 0) != 3 ||
		    head[0] != 0x1f || head[1] != 0x8b || head[2] != 8)
			return false;
		if (size >= 4 && pread(fd, tail, 4, size - 4) == 4)
			f.hint = inflate_hint(tail, size);
		return true;
	    });
}

int dng_scan_gzip_stats(dng_scan *s, uint64_t *files, uint64_t *members,
    uint64_t *compressed_bytes, uint64_t *inflated_bytes, uint64_t *launches,
    double *inflate_ms)
{
	if (!s)
		return DNG_EINVAL;
	const CzState &cz = stats(s);
	put(files, cz.gz_files);
	put(members, cz.gz_members);
	put(compressed_bytes, cz.gz_in_bytes);
	put(inflated_bytes, cz.gz_out_bytes);
	put(launches, cz.gz_launches);
	put(inflate_ms, cz.gz_ms);
	return DNG_OK;
}

int dng_scan_gzip_split_stats(dng_scan *s, uint64_t *split_files,
    uint64_t *chunks, uint64_t *false_starts, uint64_t *fallbacks,
    uint64_t *launches)
{
	if (!s)
		return DNG_EINVAL;
	const CzState &cz = stats(s);
	put(split_files, cz.gz_split_files);
	put(chunks, cz.gz_chunks);
	put(false_starts, cz.gz_false_starts);
	put(fallbacks, cz.gz_fallbacks);
	put(launches, cz.gz_split_launches);
	return DNG_OK;
}

int dng_scan_feed_bzip2(dng_scan *s, const char *path)
{
	return cz_feed(s, path, "dng_scan_feed_bzip2", true,
	    ": not a bzip2 file (it does not start with BZh and a level 1-9)",
	    [](int fd, size_t size, CzFile &f) {
		u8 h[4];
		if (size < 4 || pread(fd, h, 4, 0) != 4)
			return false;
		f.head = (uint32_t)h[0] << 24 | (uint32_t)h[1] << 16 |
		    (uint32_t)h[2] << 8 | h[3];
		return bz_level_ok(f.head);
	    });
}

int dng_scan_bzip2_stats(dng_scan *s, uint64_t *files, uint64_t *streams,
    uint64_t *blocks, uint64_t *false_starts, uint64_t *compressed_bytes,
    uint64_t *decompressed_bytes, uint64_t *launches, double *bunzip_ms)
{
	if (!s)
		return DNG_EINVAL;
	const CzState &cz = stats(s);
	put(files, cz.bz_files);
	put(streams, cz.bz_streams);
	put(blocks, cz.bz_blocks);
	put(false_starts, cz.bz_false_starts);
	put(compressed_bytes, cz.bz_in_bytes);
	put(decompressed_bytes, cz.bz_out_bytes);
	put(launches, cz.bz_launches);
	put(bunzip_ms, cz.bz_ms);
	return DNG_OK;
}

int dng_scan_bzip2_stage_ms(dng_scan *s, double *find_ms, double *decode_ms,
    double *invert_ms, double *emit_ms)
{
	if (!s)
		return DNG_EINVAL;
	double *const out[4] = { find_ms, decode_ms, invert_ms, emit_ms };
	for (int i = 0; i < 4; i++)
		put(out[i], stats(s).bz_stage_ms[i]);
	return DNG_OK;
}
