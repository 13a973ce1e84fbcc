/*
 * scan.h: the state of one scan, for api.cu and compressed.cu.  Host headers
 * only: each kernel is compiled in the one file that launches it.
 */
#ifndef DNG_SCAN_H
#define DNG_SCAN_H

#include <cuda_runtime.h>

#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/dragnet_gpu.h"
#include "plan.h"
#include "jit.h"
#include "compressed.h"

namespace dng { struct MissEnt; }	/* fast_kernel.cuh */

const size_t RING_SLOTS = 3;

struct dng_scan {
	dng_plan plan;
	int device = 0;
	int sm_count = 0;
	dng::u32 plan_bytes = 0, sslots = 0, s1slots = 0;
	cudaStream_t stream = nullptr, copy_stream = nullptr;
	cudaStream_t own_stream = nullptr;
	dng::DevPlan *d_plan = nullptr;
	dng::GTable tab{};
	unsigned long long *d_counters = nullptr;
	unsigned long long *d_nl = nullptr;	/* find_nl scratch (2) */
	size_t table_cap = 0;
	/* H2D ring */
	size_t ring_cap = 0;
	dng::u8 *d_ring[RING_SLOTS] = {};
	dng::u8 *h_stage[RING_SLOTS] = {};
	cudaEvent_t ev_ready[RING_SLOTS] = {}, ev_free[RING_SLOTS] = {};
	bool slot_used[RING_SLOTS] = {};
	size_t next_slot = 0;
	/* carry: the unterminated tail of everything fed so far */
	dng::u8 *d_carry = nullptr;
	size_t carry_len = 0;
	dng::u8 *d_side = nullptr;		/* carry + head of a device chunk */
	/* pinned block ring of dng_scan_feed_file's reader threads */
	dng::u8 *file_buf = nullptr;
	cudaEvent_t file_done[32] = {};
	/* dng_scan_read_stats */
	uint64_t direct_bytes = 0, buffered_bytes = 0, direct_ranges = 0;
	uint64_t read_fallbacks = 0;
	/* dng_scan_feed_gzip and dng_scan_feed_bzip2: their queue, buffers and
	 * stats (compressed.cu), from the first compressed file fed */
	CzState *cz = nullptr;
	/* stats */
	std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_pairs;
	std::vector<cudaEvent_t> ev_pool;
	double kernel_ms = 0;
	uint64_t launches = 0, kernel_bytes = 0, bytes_fed = 0;
	uint64_t aux_launches = 0;	/* resolve / find_nl / compact kernels */
	cudaEvent_t ev_init = nullptr;	/* setup enqueued by dng_scan_open */
	bool finished = false;
	/* record templates (tmpl.h), learned from the head of the input */
	bool tmpl_enabled = true, tmpl_tried = false;
	dng::KernelChoice kc;		/* which kernel, at what geometry */
	dng::u32 w_sslots = 0, w_s1slots = 0;
	/* counters of finished launches, copied to pinned memory after every
	 * launch: lets the host notice that the input changed character */
	unsigned long long *h_live = nullptr;
	dng::u8 *d_tmpl = nullptr;
	dng::u32 tmpl_bytes = 0, ntemplates = 0;
	/* what learns since d_tmpl was last built resolved, oldest first: the
	 * first general launch builds d_tmpl from it (an F scan never does) */
	std::vector<std::pair<std::vector<dng::TCandidate>,
	    std::vector<dng::TResolved>>> tmpl_pending;
	dng::u8 *h_blobs = nullptr;		/* pinned staging of the blob uploads */
	/* the F path (fast.h): its plan, its templates, its miss list */
	dng::FPlan fplan;
	dng::FPlan *d_fplan = nullptr;
	dng::u8 *d_ftmpl = nullptr;
	dng::u32 ftmpl_bytes = 0, nftemplates = 0;
	dng::u32 ftmpl_leaf_off = 0, ftmpl_pool_off = 0;
	dng::u32 f_smem_max = 0;		/* dynamic shared memory a CTA may ask for */
	/* run-time compiled matcher (jit.h): 0 off, 1 in the background, 2 wait */
	int jit_mode = 1;
	std::shared_ptr<dng::JitKernels> jit;
	uint64_t jit_launches = 0;
	dng::MissEnt *d_miss = nullptr;
	dng::u32 *d_miss_n = nullptr;
	dng::u32 miss_cap = 0;
	unsigned long long seen_tmpl = 0;
	/* a scan over several devices (dng_scan_open_devices) holds no device
	 * state of its own: it records the files fed, with their sizes, and
	 * at finish cuts them into one byte range per shard */
	bool multi = false;
	std::vector<dng_scan *> shards;
	std::vector<std::pair<std::string, size_t>> files;
	std::string err;
	int err_code = 0;

	int fail(int code, const std::string &m) {
		if (!err_code) {
			err_code = code;
			err = m;
		}
		return code;
	}
	int cuda(cudaError_t e, const char *what) {
		if (e == cudaSuccess)
			return 0;
		return fail(DNG_ECUDA, std::string(what) + ": " +
		    cudaGetErrorString(e));
	}
};

#define CK(s, call) do { if ((s)->cuda((call), #call)) return (s)->err_code; } while (0)

/* the per-process buffer cache (api.cu): device `device`, or pinned host
 * memory for device -1 */
cudaError_t dng_cached_alloc(int device, void **p, size_t n);
void dng_cached_free(void *p);

#define DEV_ALLOC(s, p, n) dng_cached_alloc((s)->device, (void **)(p), (n))
#define HOST_ALLOC(p, n) dng_cached_alloc(-1, (void **)(p), (n))

/* an output of a stats call, where the caller asked for it */
template <class T, class V> void put(T *dst, V v)
{
	if (dst)
		*dst = v;
}

/* api.cu */
cudaEvent_t get_event(dng_scan *s);
int refuse_multi(dng_scan *s, const char *what);
int feed_device(dng_scan *s, const void *devbuf, size_t len);
int read_to_device(dng_scan *s, const char *path, size_t size, dng::u8 *dst);

#endif
