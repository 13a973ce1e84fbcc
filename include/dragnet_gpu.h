/*
 * dragnet_gpu.h: C ABI of libdragnet_gpu.so -- the H100-native replacement for
 * dragnet's raw-data scan path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  The reference has no
 * FFI of its own (it is pure JavaScript), so the entry points below are what a
 * thin N-API addon binds to implement a `Datasource` whose scan() replaces
 *
 *     DatasourceFile.scan()            lib/datasource-file.js:72-108
 *       -> parserFor(format)           lib/dragnet-impl.js:131-140
 *          JsonLineStream              lib/format-json.js:26-46
 *       -> [Datasource filter]         lib/datasource-file.js:154-163
 *       -> new StreamScan(...)         lib/stream-scan.js:40-94
 *            KrillSkinnerStream        lib/krill-skinner-stream.js:29-52
 *            SyntheticTransformer      lib/stream-synthetic.js:37-85
 *            time-bounds filter        lib/dragnet-impl.js:94-125
 *            skinner aggregator        lib/dragnet-impl.js:48-89
 *
 * i.e. bytes of newline-delimited JSON in, skinner points out.  See
 * INTEGRATION.md for the reference-side binding (datasource-gpu.js + addon).
 *
 * Conventions: every function returns 0 on success or a negative DNG_E* code;
 * functions taking (err, errlen) also write a NUL-terminated message.  Plain
 * pointers and sizes only.  A dng_scan is not thread-safe (serialise calls
 * externally); different scans may be driven from different threads.  There is
 * no CPU fallback: without a CUDA device dng_scan_open fails with DNG_ENODEV.
 */
#ifndef DRAGNET_GPU_H
#define DRAGNET_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DNG_OK            0
#define DNG_EINVAL       -1   /* bad argument / malformed plan               */
#define DNG_ENODEV       -2   /* no usable CUDA device                       */
#define DNG_ECUDA        -3   /* CUDA runtime error (see dng_scan_error)     */
#define DNG_ENOMEM       -4
#define DNG_EIO          -5   /* dng_scan_feed_file could not read           */
#define DNG_EUNSUPPORTED -6   /* input needed a path the device code lacks   */
#define DNG_ELIMIT       -7   /* a documented limit was exceeded             */
#define DNG_ENCCL        -8

typedef struct dng_plan dng_plan;
typedef struct dng_scan dng_scan;
typedef struct dng_result dng_result;
typedef struct dng_comm dng_comm;

/*
 * Per-stage counters, mirroring the vstream counters `dn scan --counters`
 * prints (bin/dn:911-916; goldens tests/dn/local/tst.scan_fileset.sh.out:2455-2660).
 * Stage ninputs/noutputs are derivable: e.g. json parser ninputs = lines,
 * noutputs = lines - invalid_json.
 */
typedef struct dng_counters {
	uint64_t lines;            /* json parser ninputs (every line, incl. empty) */
	uint64_t invalid_json;     /* json parser "invalid json"                    */
	uint64_t invalid_point;    /* json-skinner line that is not a point         */
	uint64_t ds_ninputs;       /* Datasource filter ninputs                     */
	uint64_t ds_filtered;      /* Datasource filter nfilteredout                */
	uint64_t ds_failedeval;    /* Datasource filter nfailedeval                 */
	uint64_t user_ninputs;     /* User filter ...                               */
	uint64_t user_filtered;
	uint64_t user_failedeval;
	uint64_t synth_ninputs;    /* Datetime parser ninputs                       */
	uint64_t synth_undef;      /* Datetime parser undef                         */
	uint64_t synth_baddate;    /* Datetime parser baddate                       */
	uint64_t time_ninputs;     /* Time filter ...                               */
	uint64_t time_filtered;
	uint64_t time_failedeval;
	uint64_t aggr_ninputs;     /* Aggregator ninputs (records aggregated)       */
	uint64_t slowpath_records; /* records that took a device slow path          */
	uint64_t long_records;     /* records longer than the in-tile window        */
	uint64_t unsupported;      /* records the device code could not decide      */
	uint64_t bytes;            /* input bytes consumed                          */
} dng_counters;

/* ---- plan ------------------------------------------------------------- */

/*
 * plan_json: the serialised QueryConfig + datasource properties
 * (lib/dragnet.js:28-77, lib/datasource-file.js:47-56):
 *   { "format": "json" | "json-skinner",
 *     "ds_filter": <krill predicate> | null,
 *     "filter":    <krill predicate> | null,
 *     "synthetic": [ { "name": s, "field": s }, ... ],   // qc_synthetic (+dn_ts)
 *     "time_bounds": { "field": "dn_ts", "ge": sec, "lt": sec } | null,
 *     "breakdowns": [ { "name": s, "field": s, ["date": true,]
 *                       ["aggr": "quantize" | "lquantize", "step": n] }, ... ] }
 * or, to scan several metrics in one pass over the data (dn build):
 *   { "format": ..., "ds_filter": ...,
 *     "metrics": [ { "filter", "synthetic", "time_bounds", "breakdowns" }, ... ] }
 */
int dng_plan_create(const char *plan_json, dng_plan **out,
    char *err, size_t errlen);
void dng_plan_destroy(dng_plan *plan);

/* ---- scan ------------------------------------------------------------- */

int dng_device_count(void);

int dng_scan_open(const dng_plan *plan, int device, dng_scan **out,
    char *err, size_t errlen);

/*
 * One scan over several devices, for files only.  The files fed are one
 * logical byte stream of T bytes (their sizes taken when fed), as the
 * reference concatenates them: a file without a trailing newline joins its
 * last line to the next file's first.  dng_scan_finish cuts that stream into
 * n shards, shard k owning the lines that start in [floor(k T/n),
 * floor((k+1) T/n)), and scans each with an ordinary scan of its own on
 * devices[k], from a thread of its own; the points and counters it returns
 * are exactly those of one scan of the same files (counters summed per
 * metric; the shards' `bytes` sum to T).
 *   - A device may be listed more than once; a bad index fails here with
 *     DNG_ENODEV, as dng_scan_open does, as does a machine without CUDA.
 *   - dng_scan_feed_file only records the path and its size: it must name a
 *     regular file, and one whose size has changed by the time it is read
 *     fails the scan with DNG_EIO.  The 16 MiB line limit holds across cuts.
 *   - dng_scan_feed, _pinned, _device and dng_scan_set_stream return
 *     DNG_EINVAL; set_templates applies to every shard.
 *   - Each shard holds what a single scan holds: its device buffers, a
 *     128 MiB pinned file ring and, while it reads, DNG_READ_THREADS
 *     reader threads (default 16) -- the knob is per shard, so n shards
 *     read with up to 16 n threads.
 */
int dng_scan_open_devices(const dng_plan *plan, const int *devices, int n,
    dng_scan **out, char *err, size_t errlen);
/*
 * Shard i of a scan from dng_scan_open_devices (NULL for any other scan or
 * index), owned by that scan: for the stats calls only (kernel_kind,
 * kernel_stats, tally_stats, template_stats, jit_stats, launch_count,
 * read_stats, and
 * counters after finish); never feed, finish or destroy it.  Shards learn
 * their templates from their own head and may pick different kernels;
 * results never depend on either.  Those stats calls on the multi-device scan
 * itself return DNG_EINVAL (dng_scan_launch_count and dng_scan_read_stats
 * sum the shards').
 */
dng_scan *dng_scan_shard(const dng_scan *scan, int i);

/* Run this scan's kernels on a caller-owned CUDA stream (a cudaStream_t) instead
 * of the scan's private one, e.g. to bracket them with the caller's events.
 * Call before the first feed. */
int dng_scan_set_stream(dng_scan *scan, void *cuda_stream);

/*
 * Feed arbitrary byte chunks (lstream semantics: lines split on '\n', partial
 * trailing line carried to the next feed; lib/format-json.js:32-33).
 * dng_scan_feed: any host memory; the bytes are consumed (copied to a pinned
 *   staging ring) before it returns.
 * dng_scan_feed_pinned: page-locked host memory (dng_pinned_alloc or
 *   cudaHostRegister'd); DMA'd directly; the buffer must stay valid and
 *   unmodified until the next dng_scan_sync()/dng_scan_finish().
 * dng_scan_feed_device: bytes already resident in this device's HBM
 *   (16-byte aligned); scanned in place, no copy.  The kernels that read the
 *   buffer are only ENQUEUED when this returns (on the scan's stream, or the
 *   caller's after dng_scan_set_stream): like a pinned buffer, it must stay
 *   valid and unmodified until the next dng_scan_sync()/dng_scan_finish().
 * dng_scan_feed_file: read the file into the pinned ring and feed it: with
 *   O_DIRECT (storage straight into pinned memory, the page cache bypassed)
 *   when little of it is in the page cache, else through the page cache
 *   (dng_scan_read_stats).  Pipes and devices are read(2) in sequence.
 */
int dng_scan_feed(dng_scan *scan, const void *buf, size_t len);
int dng_scan_feed_pinned(dng_scan *scan, const void *buf, size_t len);
int dng_scan_feed_device(dng_scan *scan, const void *devbuf, size_t len);
int dng_scan_feed_file(dng_scan *scan, const char *path);
int dng_scan_sync(dng_scan *scan);

/*
 * dng_scan_feed_gzip: a gzip file (RFC 1952: one or more members of DEFLATE
 *   data, zero bytes after a member ignored, as Python's gzip.decompress
 *   accepts), inflated on the device.  Its decompressed bytes join the scan's
 *   stream at this point, exactly as dng_scan_feed_file of the decompressed
 *   file would: `bytes` counts decompressed bytes, and a file without a
 *   trailing newline joins its last line to the next file's first.  A file
 *   that does not start with 1f 8b 08 fails here with DNG_EINVAL.  Files are
 *   queued and inflated in batches, read as dng_scan_feed_file reads; the
 *   queue is processed no later than the scan's next feed of any kind,
 *   dng_scan_sync or dng_scan_finish, and a corrupt file (bad header, codes or
 *   lengths, truncated, CRC-32 or ISIZE mismatch) fails the scan with DNG_EIO
 *   from that call, naming the file and the damage.  A scan over several
 *   devices refuses it (DNG_EINVAL).
 */
int dng_scan_feed_gzip(dng_scan *scan, const char *path);
/* Gzip files inflated so far, their members, compressed and decompressed
 * bytes, inflate kernel launches (one per batch that has a file decoded by
 * one warp, plus one per decode of a file again in more room, or whole after
 * the split path could not vouch for it) and the time of every inflate
 * kernel, the split path's included (CUDA events). */
int dng_scan_gzip_stats(dng_scan *scan, uint64_t *files, uint64_t *members,
    uint64_t *compressed_bytes, uint64_t *inflated_bytes, uint64_t *launches,
    double *inflate_ms);
/* The split path: a large file in a batch of fewer files than the device
 * holds decode warps is cut into chunks at block starts found on the device
 * and decoded by one warp per chunk.  Files split, their chunks, candidate
 * block starts nothing landed on (false starts), files decoded whole after
 * the split path could not vouch for them (fallbacks: damaged files only),
 * and the split kernels' launches (also in dng_scan_launch_count). */
int dng_scan_gzip_split_stats(dng_scan *scan, uint64_t *split_files,
    uint64_t *chunks, uint64_t *false_starts, uint64_t *fallbacks,
    uint64_t *launches);

/*
 * dng_scan_feed_bzip2: a bzip2 file (one or more complete streams, levels
 *   BZh1-BZh9 mixed, randomised blocks included, optionally followed by zero
 *   bytes), decoded on the device with all its blocks in parallel.  Its
 *   decompressed bytes join the scan's stream at this point, as for
 *   dng_scan_feed_gzip.  A file that does not start with "BZh" and a digit
 *   1-9 fails here with DNG_EINVAL.  It shares the gzip queue: a batch holds
 *   files of one format, and a feed of another kind processes the queue
 *   first.  Damage (bad stream or block header, bad selectors or code
 *   lengths, an invalid code, a block overflow, a block or stream CRC
 *   mismatch, truncation) fails the scan with DNG_EIO naming the file, the
 *   damage and the compressed byte; so does anything after the last stream
 *   that is not zero bytes, which Python's bz2.decompress would ignore.  A
 *   scan over several devices refuses it (DNG_EINVAL).
 */
int dng_scan_feed_bzip2(dng_scan *scan, const char *path);
/* Bzip2 files decoded so far, their streams and blocks, block candidates
 * the chain of blocks did not land on (false starts), compressed and
 * decompressed bytes, launches of the bzip2 kernels (also in
 * dng_scan_launch_count) and their time (CUDA events).  Any pointer may be
 * NULL. */
int dng_scan_bzip2_stats(dng_scan *scan, uint64_t *files, uint64_t *streams,
    uint64_t *blocks, uint64_t *false_starts, uint64_t *compressed_bytes,
    uint64_t *decompressed_bytes, uint64_t *launches, double *bunzip_ms);
/* bunzip_ms by stage: finding magics, decoding blocks, inverting them
 * (inverse BWT and run lengths), emitting them (final run-length stage and
 * CRCs). */
int dng_scan_bzip2_stage_ms(dng_scan *scan, double *find_ms,
    double *decode_ms, double *invert_ms, double *emit_ms);

/* End of input: flushes the final unterminated line, then emits the points. */
int dng_scan_finish(dng_scan *scan, dng_result **out);
int dng_scan_counters(dng_scan *scan, dng_counters *out);
/* counters of metric m's StreamScan (m = 0 is what dng_scan_counters gives) */
int dng_scan_counters_metric(dng_scan *scan, int metric, dng_counters *out);
const char *dng_scan_error(const dng_scan *scan);
void dng_scan_destroy(dng_scan *scan);
/* Destroyed scans keep their device and pinned buffers for the next scan of
 * this process (bounded by DNG_CACHE_BYTES per kind, default 2 GiB); this
 * returns them to the driver. */
void dng_release_cached(void);
/* Waits for the matchers being compiled in the background (DNG_JIT=async,
 * the default) and drops those still queued; later scans compile none in the
 * background.  Call it before the process exits: a compile still running when
 * exit() tears the compiler libraries down can crash the process.  The Python
 * package calls it from an atexit handler. */
void dng_jit_finish(void);
/*
 * Keeps the F path's run-time compiled kernels (dng_scan_jit_stats) in `dir`,
 * one file per kernel, so that a later process loads the kernel instead of
 * compiling and linking it, and runs it from its first launch in
 * DNG_JIT=async mode too.  NULL or "" turns the cache off for this process.
 * Overrides the environment's DNG_JIT_CACHE_DIR; call it before the first scan
 * is opened.  Off by default: then nothing is read or written.
 *
 * An entry is found by its full key: the scan's templates and plan, the lane
 * slice size, the shared-memory limit, the device's compute capability and a
 * build id of this library (a hash of the whole library file), so a kernel is
 * only ever loaded by the same library file that linked it.  A damaged,
 * truncated or foreign entry is a miss and the kernel is linked again; the
 * directory (created with mode 0700) is held under 512 MiB by deleting the
 * least recently used entries.  A directory that is not the calling user's,
 * or that group or others may write to, is not used (an error is counted):
 * whoever can write an entry chooses the code a scan runs.  No cache failure
 * fails a scan or changes its results: it is counted and the kernel is built
 * as without the cache.
 */
int dng_jit_cache_dir(const char *dir);
/* process-wide counters of that cache: entries loaded, looked up and not
 * found (or damaged), written, deleted to stay under the bound, and failures
 * (a directory that cannot be created or written, an entry the driver
 * refused); any pointer may be NULL */
int dng_jit_cache_stats(uint64_t *hits, uint64_t *misses, uint64_t *writes,
    uint64_t *evictions, uint64_t *errors);

/* Device time (ms, CUDA events on the scan stream) spent in scan kernels and
 * the number of kernel launches since open; for bench.py's roofline. */
int dng_scan_kernel_stats(dng_scan *scan, double *kernel_ms,
    uint64_t *launches, uint64_t *kernel_bytes);
/*
 * The F kernel's tally cache: *inline_overflow = records whose key its inline
 * tier had no slot for (they took the general tally path), *f_warps = warps
 * per CTA it launches with now (28 or 24; the scan drops to 24 when keys
 * overflow, environment DNG_F_WARPS=28|24 sets the start).  Read-only.
 */
int dng_scan_tally_stats(dng_scan *scan, uint64_t *inline_overflow,
    int *f_warps);

/*
 * Record templates: the scan learns the few shapes (key order + punctuation)
 * the input's records repeat from the head of the first data it is fed, and
 * matches records against them before falling back to its byte automaton;
 * results never depend on it.  On by default (environment DNG_TEMPLATES=0
 * turns it off); set_templates must precede the first feed.  The stats give
 * the number of templates in use and how many records they accepted.
 */
int dng_scan_set_templates(dng_scan *scan, int enable);
int dng_scan_template_stats(dng_scan *scan, uint64_t *templates,
    uint64_t *templated_records);

/*
 * Which kernel the scan runs (chosen from the plan and from a sample of the
 * first data fed; environment DNG_KERNEL=tile|warp|fast forces one): 0 = CTA-wide
 * tiles (any line length), 1 = per-warp chunks (short lines), 2 = the F path
 * (templated input, plans it models: scan_kernel_f + the miss kernel).
 */
int dng_scan_kernel_kind(const dng_scan *scan);
/*
 * The F path's run-time compiled matcher (NVRTC + nvJitLink, cached per
 * process; environment DNG_JIT=0|async|sync, default async: scans use the
 * interpreted matcher until the compiled one is there).  *state: 0 none / being
 * built, 1 in use, 2 failed (message in err); *launches = scan launches that
 * ran the compiled kernel; compile and link times in milliseconds.
 */
int dng_scan_jit_stats(dng_scan *scan, int *state, uint64_t *launches,
    double *compile_ms, double *link_ms, char *err, size_t errlen);
/* Bytes dng_scan_feed_file read with O_DIRECT (straight from storage into
 * pinned memory) and through the page cache, and the files or shard ranges
 * that were read direct.  Files mostly absent from the page cache are read
 * direct; results never depend on it.  *fallbacks counts the ranges chosen
 * for O_DIRECT that the filesystem refused (they are read through the page
 * cache).  Regular files only; on a multi-device scan, the shards' sums.
 * Any pointer may be NULL. */
int dng_scan_read_stats(dng_scan *scan, uint64_t *direct_bytes,
    uint64_t *buffered_bytes, uint64_t *direct_ranges, uint64_t *fallbacks);
/* Every kernel this scan has launched so far: scan kernels plus the small
 * ones around them (template resolution, newline search of device feeds,
 * result compaction). */
uint64_t dng_scan_launch_count(const dng_scan *scan);

void *dng_pinned_alloc(size_t len);
void dng_pinned_free(void *p);

/* ---- results: skinner points ---------------------------------------------
 * One point per observed tuple; with zero breakdowns exactly one point whose
 * value is the total (possibly 0); nothing for >=1 breakdown and no input
 * (tests/dn/local/tst.empty.sh.out).  Column j of point i is either a string
 * (discrete breakdown: the JS String(value), UTF-8, not NUL-terminated) or a
 * number (quantized breakdown: bucketMin(ordinal), may be NaN/Inf).
 * Points are sorted by encoded key bytes (deterministic; the reference's
 * emission order is unspecified).
 */
size_t dng_result_count(const dng_result *r);
size_t dng_result_ncols(const dng_result *r);
/* Fan-out plans ("metrics": [...], the reference's dn build / index-scan,
 * lib/datasource-file.js:386-432): every point belongs to one metric (the
 * reference tags it fields.__dn_metric) and has that metric's columns. */
size_t dng_result_nmetrics(const dng_result *r);
size_t dng_result_ncols_metric(const dng_result *r, int metric);
int dng_result_metric(const dng_result *r, size_t i);
int dng_result_get(const dng_result *r, size_t i, const char **strs,
    size_t *strlens, uint8_t *is_number, double *numvals, uint64_t *value);
void dng_result_destroy(dng_result *r);

/* ---- shard merge (the reference's Manta reduce phase,
 * lib/datasource-manta.js:202-219): sum values over identical tuples ------ */

/* Build a result by re-aggregating skinner points, as the reference's reduce
 * phase does (`dn scan --points` over json-skinner input,
 * lib/datasource-manta.js:212-219): string columns are taken as is, numeric
 * columns are bucket minima and are re-bucketized (idempotent).  Column j of
 * point i is strs[i*ncols+j] (strlens bytes) or numvals[i*ncols+j]. */
int dng_result_from_points(const dng_plan *plan, size_t npoints,
    const char *const *strs, const size_t *strlens, const double *numvals,
    const uint64_t *values, dng_result **out);

/* Serialised tuple dictionary of a result (keys only), for exchange. */
int dng_result_dict(const dng_result *r, const void **buf, size_t *len);
/* Union of n serialised dictionaries -> sorted global dictionary. */
int dng_dict_union(const void *const *bufs, const size_t *lens, size_t n,
    void **out, size_t *outlen);
void dng_buf_free(void *p);
size_t dng_dict_count(const void *dict, size_t len);
/* Scatter r's values into a dense vector indexed by the global dictionary. */
int dng_result_dense(const dng_result *r, const void *dict, size_t dictlen,
    uint64_t *vec, size_t n);
/* Rebuild a result from the global dictionary + summed dense vector. */
int dng_result_from_dense(const dng_result *like, const void *dict,
    size_t dictlen, const uint64_t *vec, size_t n, dng_result **out);

/* NCCL transport for the above: ncclAllGather of the dictionaries and ONE
 * ncclReduce(sum, uint64) of the dense tallies (+ counters) to `root`. */
int dng_comm_unique_id(void *id128);            /* rank 0; 128 bytes out */
int dng_comm_init(dng_comm **out, int nranks, int rank, const void *id128,
    int device, char *err, size_t errlen);
int dng_merge_nccl(dng_scan *scan, dng_comm *comm, int root,
    dng_result **out, dng_counters *counters);
void dng_comm_destroy(dng_comm *comm);

/* ---- synthetic input (tools/mktestdata shape, deterministic) ------------
 * Writes records [first, first+count) of stream `seed` as NDJSON.
 * dng_gen_host fills host memory; dng_gen_device runs the generator kernel
 * on `device`; both produce byte-identical output. Returns bytes written via
 * *len (or DNG_ELIMIT when cap is too small).
 */
typedef struct dng_gen_params {
	uint64_t seed;
	uint64_t total_records;   /* n in `time = round(j/n*(max-min)+min)`   */
	int64_t  time_min_ms;     /* default 2014-05-31T21:00:00Z             */
	int64_t  time_max_ms;     /* default 2014-05-31T23:59:59Z             */
	int      string_latency;  /* emit latency as a string (mktestdata)    */
} dng_gen_params;
void dng_gen_defaults(dng_gen_params *p);
int dng_gen_host(const dng_gen_params *p, uint64_t first, uint64_t count,
    void *buf, size_t cap, size_t *len);
int dng_gen_device(const dng_gen_params *p, int device, uint64_t first,
    uint64_t count, void *devbuf, size_t cap, size_t *len);

const char *dng_version(void);

#ifdef __cplusplus
}
#endif
#endif /* DRAGNET_GPU_H */
