"""ctypes binding of libdragnet_gpu.so (include/dragnet_gpu.h).

This is the Python stand-in for the N-API addon a Node deployment would use
(INTEGRATION.md): same entry points, same ownership rules.  Loading fails
loudly when the library has not been built; there is no fallback.
"""

import atexit
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# DNG_LIB: another build of the same library (kernel tuning experiments)
LIB_PATH = os.environ.get('DNG_LIB') or os.path.join(_HERE,
                                                    'libdragnet_gpu.so')

DNG_OK = 0
ERRORS = {-1: 'EINVAL', -2: 'ENODEV', -3: 'ECUDA', -4: 'ENOMEM', -5: 'EIO',
          -6: 'EUNSUPPORTED', -7: 'ELIMIT', -8: 'ENCCL'}

COUNTER_FIELDS = [
    'lines', 'invalid_json', 'invalid_point', 'ds_ninputs', 'ds_filtered',
    'ds_failedeval', 'user_ninputs', 'user_filtered', 'user_failedeval',
    'synth_ninputs', 'synth_undef', 'synth_baddate', 'time_ninputs',
    'time_filtered', 'time_failedeval', 'aggr_ninputs', 'slowpath_records',
    'long_records', 'unsupported', 'bytes']


class DngCounters(ctypes.Structure):
    _fields_ = [(n, ctypes.c_uint64) for n in COUNTER_FIELDS]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n in COUNTER_FIELDS}


class DngGenParams(ctypes.Structure):
    _fields_ = [('seed', ctypes.c_uint64), ('total_records', ctypes.c_uint64),
                ('time_min_ms', ctypes.c_int64),
                ('time_max_ms', ctypes.c_int64),
                ('string_latency', ctypes.c_int)]


class DngError(RuntimeError):
    def __init__(self, code, msg):
        RuntimeError.__init__(self, 'libdragnet_gpu: %s (%s)' %
                              (msg, ERRORS.get(code, code)))
        self.code = code


_lib = None

# every symbol include/dragnet_gpu.h declares: (name, restype, argtypes)
_P = ctypes.c_void_p
_SIGS = [
    ('dng_plan_create', ctypes.c_int, [ctypes.c_char_p, ctypes.POINTER(_P),
                                       ctypes.c_char_p, ctypes.c_size_t]),
    ('dng_plan_destroy', None, [_P]),
    ('dng_device_count', ctypes.c_int, []),
    ('dng_scan_open', ctypes.c_int, [_P, ctypes.c_int, ctypes.POINTER(_P),
                                     ctypes.c_char_p, ctypes.c_size_t]),
    ('dng_scan_open_devices', ctypes.c_int,
     [_P, ctypes.POINTER(ctypes.c_int), ctypes.c_int, ctypes.POINTER(_P),
      ctypes.c_char_p, ctypes.c_size_t]),
    ('dng_scan_shard', _P, [_P, ctypes.c_int]),
    ('dng_scan_set_stream', ctypes.c_int, [_P, _P]),
    ('dng_scan_feed', ctypes.c_int, [_P, _P, ctypes.c_size_t]),
    ('dng_scan_feed_pinned', ctypes.c_int, [_P, _P, ctypes.c_size_t]),
    ('dng_scan_feed_device', ctypes.c_int, [_P, _P, ctypes.c_size_t]),
    ('dng_scan_feed_file', ctypes.c_int, [_P, ctypes.c_char_p]),
    ('dng_scan_feed_gzip', ctypes.c_int, [_P, ctypes.c_char_p]),
    ('dng_scan_feed_bzip2', ctypes.c_int, [_P, ctypes.c_char_p]),
    ('dng_scan_sync', ctypes.c_int, [_P]),
    ('dng_scan_finish', ctypes.c_int, [_P, ctypes.POINTER(_P)]),
    ('dng_scan_counters', ctypes.c_int, [_P, ctypes.POINTER(DngCounters)]),
    ('dng_scan_counters_metric', ctypes.c_int,
     [_P, ctypes.c_int, ctypes.POINTER(DngCounters)]),
    ('dng_scan_error', ctypes.c_char_p, [_P]),
    ('dng_scan_destroy', None, [_P]),
    ('dng_release_cached', None, []),
    ('dng_jit_finish', None, []),
    ('dng_jit_cache_dir', ctypes.c_int, [ctypes.c_char_p]),
    ('dng_jit_cache_stats', ctypes.c_int,
     [ctypes.POINTER(ctypes.c_uint64)] * 5),
    ('dng_scan_kernel_stats', ctypes.c_int,
     [_P, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_uint64),
      ctypes.POINTER(ctypes.c_uint64)]),
    ('dng_scan_tally_stats', ctypes.c_int,
     [_P, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int)]),
    ('dng_scan_set_templates', ctypes.c_int, [_P, ctypes.c_int]),
    ('dng_scan_template_stats', ctypes.c_int,
     [_P, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64)]),
    ('dng_scan_kernel_kind', ctypes.c_int, [_P]),
    ('dng_scan_jit_stats', ctypes.c_int,
     [_P, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_uint64),
      ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double),
      ctypes.c_char_p, ctypes.c_size_t]),
    ('dng_scan_read_stats', ctypes.c_int,
     [_P] + [ctypes.POINTER(ctypes.c_uint64)] * 4),
    ('dng_scan_gzip_stats', ctypes.c_int,
     [_P] + [ctypes.POINTER(ctypes.c_uint64)] * 5 +
     [ctypes.POINTER(ctypes.c_double)]),
    ('dng_scan_gzip_split_stats', ctypes.c_int,
     [_P] + [ctypes.POINTER(ctypes.c_uint64)] * 5),
    ('dng_scan_bzip2_stats', ctypes.c_int,
     [_P] + [ctypes.POINTER(ctypes.c_uint64)] * 7 +
     [ctypes.POINTER(ctypes.c_double)]),
    ('dng_scan_bzip2_stage_ms', ctypes.c_int,
     [_P] + [ctypes.POINTER(ctypes.c_double)] * 4),
    ('dng_scan_launch_count', ctypes.c_uint64, [_P]),
    ('dng_pinned_alloc', _P, [ctypes.c_size_t]),
    ('dng_pinned_free', None, [_P]),
    ('dng_result_count', ctypes.c_size_t, [_P]),
    ('dng_result_ncols', ctypes.c_size_t, [_P]),
    ('dng_result_nmetrics', ctypes.c_size_t, [_P]),
    ('dng_result_ncols_metric', ctypes.c_size_t, [_P, ctypes.c_int]),
    ('dng_result_metric', ctypes.c_int, [_P, ctypes.c_size_t]),
    ('dng_result_get', ctypes.c_int,
     [_P, ctypes.c_size_t, ctypes.POINTER(ctypes.c_char_p),
      ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_uint8),
      ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_uint64)]),
    ('dng_result_destroy', None, [_P]),
    ('dng_result_from_points', ctypes.c_int,
     [_P, ctypes.c_size_t, ctypes.POINTER(ctypes.c_char_p),
      ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_double),
      ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(_P)]),
    ('dng_result_dict', ctypes.c_int, [_P, ctypes.POINTER(_P),
                                       ctypes.POINTER(ctypes.c_size_t)]),
    ('dng_dict_union', ctypes.c_int,
     [ctypes.POINTER(_P), ctypes.POINTER(ctypes.c_size_t), ctypes.c_size_t,
      ctypes.POINTER(_P), ctypes.POINTER(ctypes.c_size_t)]),
    ('dng_buf_free', None, [_P]),
    ('dng_dict_count', ctypes.c_size_t, [_P, ctypes.c_size_t]),
    ('dng_result_dense', ctypes.c_int,
     [_P, _P, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64),
      ctypes.c_size_t]),
    ('dng_result_from_dense', ctypes.c_int,
     [_P, _P, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64),
      ctypes.c_size_t, ctypes.POINTER(_P)]),
    ('dng_comm_unique_id', ctypes.c_int, [_P]),
    ('dng_comm_init', ctypes.c_int,
     [ctypes.POINTER(_P), ctypes.c_int, ctypes.c_int, _P, ctypes.c_int,
      ctypes.c_char_p, ctypes.c_size_t]),
    ('dng_merge_nccl', ctypes.c_int,
     [_P, _P, ctypes.c_int, ctypes.POINTER(_P),
      ctypes.POINTER(DngCounters)]),
    ('dng_comm_destroy', None, [_P]),
    ('dng_gen_defaults', None, [ctypes.POINTER(DngGenParams)]),
    ('dng_gen_host', ctypes.c_int,
     [ctypes.POINTER(DngGenParams), ctypes.c_uint64, ctypes.c_uint64, _P,
      ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]),
    ('dng_gen_device', ctypes.c_int,
     [ctypes.POINTER(DngGenParams), ctypes.c_int, ctypes.c_uint64,
      ctypes.c_uint64, _P, ctypes.c_size_t,
      ctypes.POINTER(ctypes.c_size_t)]),
    ('dng_version', ctypes.c_char_p, []),
]
SYMBOLS = [s[0] for s in _SIGS]


def lib():
    """Load (once) and return the shared library.  Raises if it is missing:
    the product path must fail loudly rather than run anything on the CPU."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                'libdragnet_gpu.so is not built (%s); run '
                '`python -c "import __graft_entry__ as g; g.build()"` or '
                '`make -C dragnet_b200/csrc`' % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, res, args in _SIGS:
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
        # before the interpreter's own teardown and the C exit handlers:
        # a background compile still running when the compiler libraries
        # tear themselves down at exit() can crash the process
        atexit.register(L.dng_jit_finish)
    return _lib


JIT_CACHE_STATS = ['hits', 'misses', 'writes', 'evictions', 'errors']
READ_STATS = ['direct_bytes', 'buffered_bytes', 'direct_ranges', 'fallbacks']
GZIP_STATS = ['gzip_files', 'gzip_members', 'gzip_compressed_bytes',
              'gzip_inflated_bytes', 'inflate_launches', 'inflate_ms']
GZIP_SPLIT_STATS = ['gzip_split_files', 'gzip_chunks', 'gzip_false_starts',
                    'gzip_fallbacks', 'gzip_split_launches']
BZIP2_STATS = ['bzip2_files', 'bzip2_streams', 'bzip2_blocks',
               'bzip2_false_starts', 'bzip2_compressed_bytes',
               'bzip2_decompressed_bytes', 'bunzip_launches', 'bunzip_ms']
BZIP2_STAGES = ['find', 'decode', 'invert', 'emit']


def set_jit_cache_dir(path):
    """Keep the run-time compiled kernels of this process's scans in
    directory `path` (None: no cache), so that later processes load them
    instead of building them (dng_jit_cache_dir; overrides the environment's
    DNG_JIT_CACHE_DIR).  Before the first scan is opened."""
    _check(lib().dng_jit_cache_dir(None if path is None
                                   else os.fsencode(path)))


def jit_cache_stats():
    """The process's counters of that cache: {hits, misses, writes,
    evictions, errors}."""
    v = [ctypes.c_uint64() for _ in JIT_CACHE_STATS]
    _check(lib().dng_jit_cache_stats(*[ctypes.byref(x) for x in v]))
    return {n: int(x.value) for n, x in zip(JIT_CACHE_STATS, v)}


def _check(rc, scan=None, msg=None):
    if rc != DNG_OK:
        if scan is not None:
            m = lib().dng_scan_error(scan)
            msg = m.decode('utf-8', 'replace') if m else msg
        raise DngError(rc, msg or 'call failed')


class Plan(object):
    def __init__(self, plan_json):
        if isinstance(plan_json, str):
            plan_json = plan_json.encode('utf-8')
        self.handle = _P()
        err = ctypes.create_string_buffer(512)
        rc = lib().dng_plan_create(plan_json, ctypes.byref(self.handle), err,
                                   len(err))
        if rc != DNG_OK:
            raise DngError(rc, err.value.decode('utf-8', 'replace'))

    def close(self):
        if self.handle:
            lib().dng_plan_destroy(self.handle)
            self.handle = _P()

    def __del__(self):
        # (at interpreter exit the module's globals may be gone already)
        try:
            self.close()
        except Exception:
            pass


class Result(object):
    """Owns a dng_result; .points() -> [([(bytes|float), ...], value)]."""

    def __init__(self, handle):
        self.handle = handle

    def points(self, with_metric=False):
        """[([col, ...], value)]; with_metric=True -> [(metric, cols, value)]
        for fan-out plans."""
        L = lib()
        n = L.dng_result_count(self.handle)
        nc = L.dng_result_ncols(self.handle)
        strs = (ctypes.c_char_p * max(nc, 1))()
        lens = (ctypes.c_size_t * max(nc, 1))()
        isnum = (ctypes.c_uint8 * max(nc, 1))()
        nums = (ctypes.c_double * max(nc, 1))()
        val = ctypes.c_uint64()
        ptrs = ctypes.cast(strs, ctypes.POINTER(ctypes.c_void_p))
        out = []
        for i in range(n):
            _check(L.dng_result_get(self.handle, i, strs, lens, isnum, nums,
                                    ctypes.byref(val)))
            cols = []
            m = L.dng_result_metric(self.handle, i)
            for j in range(L.dng_result_ncols_metric(self.handle, m)):
                if isnum[j]:
                    cols.append(float(nums[j]))
                else:
                    cols.append(ctypes.string_at(ptrs[j], lens[j])
                                if lens[j] else b'')
            if with_metric:
                out.append((m, cols, int(val.value)))
            else:
                out.append((cols, int(val.value)))
        return out

    def dict_bytes(self):
        buf = _P()
        n = ctypes.c_size_t()
        _check(lib().dng_result_dict(self.handle, ctypes.byref(buf),
                                     ctypes.byref(n)))
        return ctypes.string_at(buf, n.value)

    def dense(self, gdict):
        n = lib().dng_dict_count(gdict, len(gdict))
        vec = (ctypes.c_uint64 * max(n, 1))()
        _check(lib().dng_result_dense(self.handle, gdict, len(gdict), vec, n))
        return [int(vec[i]) for i in range(n)]

    def from_dense(self, gdict, values):
        n = len(values)
        vec = (ctypes.c_uint64 * max(n, 1))(*values)
        out = _P()
        _check(lib().dng_result_from_dense(self.handle, gdict, len(gdict),
                                           vec, n, ctypes.byref(out)))
        return Result(out)

    def close(self):
        if self.handle:
            lib().dng_result_destroy(self.handle)
            self.handle = _P()

    def __del__(self):
        # (at interpreter exit the module's globals may be gone already)
        try:
            self.close()
        except Exception:
            pass


def result_from_points(plan, points):
    """points: [([bytes|float, ...], value)] -> Result (re-aggregated)."""
    n = len(points)
    nc = len(points[0][0]) if n else 0
    m = max(n * nc, 1)
    strs = (ctypes.c_char_p * m)()
    lens = (ctypes.c_size_t * m)()
    nums = (ctypes.c_double * m)()
    vals = (ctypes.c_uint64 * max(n, 1))()
    for i, (cols, v) in enumerate(points):
        vals[i] = v
        for j, c in enumerate(cols):
            if isinstance(c, bytes):
                strs[i * nc + j] = c
                lens[i * nc + j] = len(c)
            else:
                nums[i * nc + j] = c
    out = _P()
    _check(lib().dng_result_from_points(plan.handle, n, strs, lens, nums,
                                        vals, ctypes.byref(out)))
    return Result(out)


def dict_union(dicts):
    n = len(dicts)
    bufs = (ctypes.c_void_p * n)()
    lens = (ctypes.c_size_t * n)()
    keep = []
    for i, d in enumerate(dicts):
        b = ctypes.create_string_buffer(d, len(d))
        keep.append(b)
        bufs[i] = ctypes.cast(b, ctypes.c_void_p)
        lens[i] = len(d)
    out = _P()
    outlen = ctypes.c_size_t()
    _check(lib().dng_dict_union(bufs, lens, n, ctypes.byref(out),
                                ctypes.byref(outlen)))
    try:
        return ctypes.string_at(out, outlen.value)
    finally:
        lib().dng_buf_free(out)


class _ScanStats(object):
    """The stats calls of a dng_scan (self.handle)."""

    def kernel_stats(self):
        ms = ctypes.c_double()
        n = ctypes.c_uint64()
        b = ctypes.c_uint64()
        _check(lib().dng_scan_kernel_stats(self.handle, ctypes.byref(ms),
                                           ctypes.byref(n), ctypes.byref(b)),
               self.handle)
        over = ctypes.c_uint64()
        fw = ctypes.c_int()
        _check(lib().dng_scan_tally_stats(self.handle, ctypes.byref(over),
                                          ctypes.byref(fw)), self.handle)
        return {'kernel_ms': ms.value, 'launches': int(n.value),
                'kernel_bytes': int(b.value),
                'all_launches': int(lib().dng_scan_launch_count(self.handle)),
                'inline_overflow': int(over.value), 'f_warps': int(fw.value)}

    def template_stats(self):
        t = ctypes.c_uint64()
        r = ctypes.c_uint64()
        _check(lib().dng_scan_template_stats(self.handle, ctypes.byref(t),
                                             ctypes.byref(r)), self.handle)
        st = ctypes.c_int()
        jl = ctypes.c_uint64()
        cms = ctypes.c_double()
        lms = ctypes.c_double()
        err = ctypes.create_string_buffer(512)
        _check(lib().dng_scan_jit_stats(self.handle, ctypes.byref(st),
                                        ctypes.byref(jl), ctypes.byref(cms),
                                        ctypes.byref(lms), err, len(err)),
               self.handle)
        kind = lib().dng_scan_kernel_kind(self.handle)
        return {'templates': int(t.value), 'templated_records': int(r.value),
                'kernel': {0: 'CTA tiles', 1: 'per-warp chunks',
                           2: 'F path'}.get(kind, str(kind)),
                'jit': {'state': int(st.value), 'launches': int(jl.value),
                        'compile_ms': cms.value, 'link_ms': lms.value,
                        'error': err.value.decode('utf-8', 'replace')}}


    def read_stats(self):
        """How dng_scan_feed_file read: bytes with O_DIRECT and through the
        page cache, ranges read direct, ranges the filesystem refused
        O_DIRECT for (read through the page cache).  A multi-device scan
        gives its shards' sums."""
        v = [ctypes.c_uint64() for _ in READ_STATS]
        _check(lib().dng_scan_read_stats(self.handle,
                                         *[ctypes.byref(x) for x in v]),
               self.handle)
        return dict(zip(READ_STATS, (int(x.value) for x in v)))

    def gzip_stats(self):
        """What dng_scan_feed_gzip inflated: files, gzip members,
        compressed and decompressed bytes, inflate kernel launches and
        milliseconds."""
        v = [ctypes.c_uint64() for _ in range(5)]
        ms = ctypes.c_double()
        _check(lib().dng_scan_gzip_stats(self.handle,
                                         *[ctypes.byref(x) for x in v],
                                         ctypes.byref(ms)), self.handle)
        return dict(zip(GZIP_STATS, [int(x.value) for x in v] + [ms.value]))

    def gzip_split_stats(self):
        """The split path of dng_scan_feed_gzip: files cut into chunks,
        chunks, false starts among their candidates, files decoded whole
        after the split path could not vouch for them, split kernel
        launches."""
        v = [ctypes.c_uint64() for _ in GZIP_SPLIT_STATS]
        _check(lib().dng_scan_gzip_split_stats(
            self.handle, *[ctypes.byref(x) for x in v]), self.handle)
        return dict(zip(GZIP_SPLIT_STATS, (int(x.value) for x in v)))

    def bzip2_stats(self):
        """What dng_scan_feed_bzip2 decoded: files, streams, blocks, block
        candidates the chain did not land on, compressed and decompressed
        bytes, bzip2 kernel launches and milliseconds."""
        v = [ctypes.c_uint64() for _ in range(7)]
        ms = ctypes.c_double()
        _check(lib().dng_scan_bzip2_stats(self.handle,
                                          *[ctypes.byref(x) for x in v],
                                          ctypes.byref(ms)), self.handle)
        return dict(zip(BZIP2_STATS, [int(x.value) for x in v] + [ms.value]))

    def bzip2_stage_ms(self):
        """bunzip_ms by stage: find, decode, invert, emit."""
        v = [ctypes.c_double() for _ in BZIP2_STAGES]
        _check(lib().dng_scan_bzip2_stage_ms(
            self.handle, *[ctypes.byref(x) for x in v]), self.handle)
        return dict(zip(BZIP2_STAGES, (x.value for x in v)))


class Scan(_ScanStats):
    def __init__(self, plan, device=0, devices=None):
        """devices: a list of device indices -> one scan over all of them,
        the files fed cut into one byte range per device
        (dng_scan_open_devices; files only)."""
        self.plan = plan
        self.handle = _P()
        err = ctypes.create_string_buffer(512)
        if devices is None:
            rc = lib().dng_scan_open(plan.handle, device,
                                     ctypes.byref(self.handle), err, len(err))
        else:
            devs = (ctypes.c_int * max(len(devices), 1))(*devices)
            rc = lib().dng_scan_open_devices(plan.handle, devs, len(devices),
                                             ctypes.byref(self.handle), err,
                                             len(err))
        if rc != DNG_OK:
            raise DngError(rc, err.value.decode('utf-8', 'replace'))

    def set_stream(self, cuda_stream):
        _check(lib().dng_scan_set_stream(self.handle, cuda_stream),
               self.handle)

    def feed(self, data):
        b = (ctypes.c_char * len(data)).from_buffer_copy(data) \
            if not isinstance(data, bytes) else data
        _check(lib().dng_scan_feed(self.handle, b, len(data)), self.handle)

    def feed_pinned(self, ptr, length):
        _check(lib().dng_scan_feed_pinned(self.handle, ptr, length),
               self.handle)

    def feed_device(self, ptr, length):
        _check(lib().dng_scan_feed_device(self.handle, ptr, length),
               self.handle)

    def feed_file(self, path):
        _check(lib().dng_scan_feed_file(self.handle, os.fsencode(path)),
               self.handle)

    def feed_gzip(self, path):
        """A gzip file, inflated on the device; queued, and processed no
        later than the next feed, sync or finish."""
        _check(lib().dng_scan_feed_gzip(self.handle, os.fsencode(path)),
               self.handle)

    def feed_bzip2(self, path):
        """A bzip2 file, decoded on the device with its blocks in
        parallel; queued with gzip files, and processed no later than the
        next feed of another kind, sync or finish."""
        _check(lib().dng_scan_feed_bzip2(self.handle, os.fsencode(path)),
               self.handle)

    def sync(self):
        _check(lib().dng_scan_sync(self.handle), self.handle)

    def finish(self):
        out = _P()
        _check(lib().dng_scan_finish(self.handle, ctypes.byref(out)),
               self.handle)
        return Result(out)

    def counters(self, metric=0):
        c = DngCounters()
        _check(lib().dng_scan_counters_metric(self.handle, metric,
                                              ctypes.byref(c)), self.handle)
        return c.as_dict()

    def set_templates(self, enable):
        """Record templates on/off (default on); before the first feed."""
        _check(lib().dng_scan_set_templates(self.handle, 1 if enable else 0),
               self.handle)

    def shards(self, n):
        """The n shards of a multi-device scan."""
        return [Shard(self, i) for i in range(n)]

    def close(self):
        if self.handle:
            lib().dng_scan_destroy(self.handle)
            self.handle = _P()

    def __del__(self):
        # (at interpreter exit the module's globals may be gone already)
        try:
            self.close()
        except Exception:
            pass


class Shard(_ScanStats):
    """Shard i of a multi-device Scan: its stats only (dng_scan_shard)."""

    def __init__(self, scan, i):
        self.scan = scan                # the owner outlives this view
        self.handle = lib().dng_scan_shard(scan.handle, i)
        if not self.handle:
            raise DngError(-1, 'no shard %d' % i)


def gen_params(seed=0xD5A60000, total_records=1000, string_latency=False,
               time_min_ms=None, time_max_ms=None):
    p = DngGenParams()
    lib().dng_gen_defaults(ctypes.byref(p))
    p.seed = seed
    p.total_records = total_records
    p.string_latency = 1 if string_latency else 0
    if time_min_ms is not None:
        p.time_min_ms = time_min_ms
    if time_max_ms is not None:
        p.time_max_ms = time_max_ms
    return p


def gen_host(params, first, count):
    cap = count * 320 + 64
    buf = ctypes.create_string_buffer(cap)
    n = ctypes.c_size_t()
    _check(lib().dng_gen_host(ctypes.byref(params), first, count, buf, cap,
                              ctypes.byref(n)), msg='dng_gen_host')
    return buf.raw[:n.value]
