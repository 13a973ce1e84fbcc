"""Times dng_scan_feed_file on a file that is not in the page cache: this
library, which reads such a file with O_DIRECT straight into the pinned ring,
against a build of the library from before O_DIRECT reads (--old-lib), which
reads every file through the page cache.  Alternates the two, one process per
sample, on the same generated NDJSON file:

  cold      made cold (fsync + POSIX_FADV_DONTNEED on the file) before each
  partial   made cold, then its first FRACTION read back, for each fraction
  hot       read whole before each: both libraries must read it buffered

Reports per library and condition the median and range of records/s, wall
seconds (feed_file to result), the process's CPU seconds per GB (getrusage,
all threads) and read_stats; checks every sample's points and counters
against the C++ oracle on the same bytes.  The first line names the GPU and
its power limit.  The file must be on a filesystem with a page cache and
O_DIRECT: the script refuses tmpfs.

    python tools/direct_read_leg.py --old-lib OLD.so [--dir DIR] [--gb 4]
        [--pairs 5] [--fractions 0.0625,0.125,0.25,0.5] [--out FILE]

The cache is dropped per file with posix_fadvise only, never system-wide.
"""

import argparse
import json
import os
import resource
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

PLAN = {'format': 'json', 'ds_filter': None,
        'filter': {'ne': ['req.method', 'HEAD']}, 'synthetic': [],
        'time_bounds': None,
        'breakdowns': [{'name': 'req.method', 'field': 'req.method'},
                       {'name': 'res.statusCode', 'field': 'res.statusCode'},
                       {'name': 'host', 'field': 'host'}]}
NAMES = [b['name'] for b in PLAN['breakdowns']]


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit',
                              '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out.split('\n')
    except (OSError, subprocess.SubprocessError):
        return []


def fs_type(path):
    path = os.path.realpath(path)
    best, typ = '', None
    with open('/proc/self/mountinfo') as f:
        for line in f:
            parts = line.split()
            mnt, fstype = parts[4], parts[parts.index('-') + 1]
            if (path == mnt or path.startswith(mnt.rstrip('/') + '/')) \
                    and len(mnt) >= len(best):
                best, typ = mnt, fstype
    return typ


def resident(path):
    """share of the file's pages in the page cache (mincore)"""
    import ctypes
    n = os.path.getsize(path)
    libc = ctypes.CDLL(None, use_errno=True)
    libc.mmap.restype = ctypes.c_void_p
    libc.mmap.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int,
                          ctypes.c_int, ctypes.c_int, ctypes.c_long]
    ps = os.sysconf('SC_PAGE_SIZE')
    vec = (ctypes.c_ubyte * ((n + ps - 1) // ps))()
    fd = os.open(path, os.O_RDONLY)
    try:
        addr = libc.mmap(None, n, 1, 1, fd, 0)
        libc.mincore(ctypes.c_void_p(addr), ctypes.c_size_t(n), vec)
        libc.munmap(ctypes.c_void_p(addr), ctypes.c_size_t(n))
    finally:
        os.close(fd)
    return sum(v & 1 for v in vec) / len(vec)


def make_cold(path):
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)
        os.posix_fadvise(fd, 0, 0, os.POSIX_FADV_DONTNEED)
    finally:
        os.close(fd)


def read_head(path, n):
    with open(path, 'rb') as f:
        while n > 0:
            b = f.read(min(n, 8 << 20))
            if not b:
                break
            n -= len(b)


def child(path):
    """one sample in this process, with the library DNG_LIB names"""
    import ctypes
    from dragnet_b200 import native
    have = ctypes.CDLL(native.LIB_PATH)
    # a library from before read_stats lacks it: bind what it has
    native._SIGS = [s for s in native._SIGS if hasattr(have, s[0])]
    p = native.Plan(json.dumps(PLAN))
    s = native.Scan(p)
    r0 = resource.getrusage(resource.RUSAGE_SELF)
    t0 = time.perf_counter()
    s.feed_file(path)
    res = s.finish()
    wall = time.perf_counter() - t0
    r1 = resource.getrusage(resource.RUSAGE_SELF)
    pts = [[[['s', c.decode('latin-1')] if isinstance(c, bytes) else
             ['n', c] for c in cols], v] for cols, v in res.points()]
    res.close()
    rs = s.read_stats() if hasattr(have, 'dng_scan_read_stats') else None
    out = {'wall_s': wall,
           'cpu_s': (r1.ru_utime - r0.ru_utime) + (r1.ru_stime - r0.ru_stime),
           'counters': s.counters(), 'points': sorted(pts, key=repr),
           'read_stats': rs}
    s.close()
    p.close()
    print(json.dumps(out))


def sample(lib, path, env):
    e = dict(env, DNG_LIB=lib)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), '--child',
                        path], capture_output=True, text=True, env=e,
                       timeout=1800)
    if r.returncode:
        raise SystemExit('sample failed (%s): %s' % (lib, r.stderr[-2000:]))
    return json.loads(r.stdout.strip().split('\n')[-1])


def write_file(path, gb):
    from dragnet_b200 import native
    target = int(gb * 1e9)
    params = native.gen_params(total_records=1 << 40)
    n, first = 0, 0
    with open(path, 'wb') as f:
        while n < target:
            b = native.gen_host(params, first, 400000)
            f.write(b)
            n += len(b)
            first += 400000
    return first


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--child')
    ap.add_argument('--old-lib')
    ap.add_argument('--dir')
    ap.add_argument('--gb', type=float, default=4.0)
    ap.add_argument('--pairs', type=int, default=5)
    ap.add_argument('--fractions', default='0.0625,0.125,0.25,0.5')
    ap.add_argument('--out')
    a = ap.parse_args()
    if a.child:
        child(a.child)
        return
    from dragnet_b200 import datasource_gpu, native
    from engines import canon_points, cpp_engine
    if not a.old_lib or not os.path.exists(a.old_lib):
        raise SystemExit('--old-lib: a library built before O_DIRECT reads')
    d = a.dir or tempfile.mkdtemp(prefix='dng-direct-leg-', dir=os.getcwd())
    os.makedirs(d, exist_ok=True)
    if fs_type(d) in (None, 'tmpfs', 'ramfs'):
        raise SystemExit('%s is on %s: every page of a file there is cached; '
                         'give --dir on a disk filesystem' % (d, fs_type(d)))
    out = open(a.out, 'w') if a.out else sys.stdout

    def emit(o):
        out.write(json.dumps(o) + '\n')
        out.flush()
    emit({'gpu': gpu_info(), 'dir': d, 'fs': fs_type(d),
          'cpus': os.cpu_count(),
          'read_threads': os.environ.get('DNG_READ_THREADS', '16')})
    path = os.path.join(d, 'leg.log')
    t = time.perf_counter()
    nrec = write_file(path, a.gb)
    size = os.path.getsize(path)
    exp_p, exp_c = cpp_engine(PLAN, [path], threads=os.cpu_count() or 1)
    exp = canon_points(exp_p)
    emit({'file_bytes': size, 'records': nrec,
          'setup_s': round(time.perf_counter() - t, 1)})
    env = dict(os.environ)
    env['DNG_JIT_CACHE_DIR'] = tempfile.mkdtemp(prefix='dng-jit-')
    libs = {'old': os.path.abspath(a.old_lib), 'new': native.LIB_PATH}
    for lib in libs.values():               # compile and cache the matcher
        sample(lib, path, env)

    def check(r):
        pts = [(list(zip(NAMES, [c.encode('latin-1') if t == 's' else c
                                 for t, c in cols])), v)
               for cols, v in r['points']]
        return canon_points(pts) == exp and datasource_gpu.stage_counters(
            PLAN, r['counters'], len(pts)) == exp_c

    conds = [('cold', 0.0)] + [('partial', float(f)) for f in
                               a.fractions.split(',') if f] + [('hot', 1.0)]
    for cond, frac in conds:
        rows = {k: [] for k in libs}
        for i in range(a.pairs):
            order = ['old', 'new'] if i % 2 == 0 else ['new', 'old']
            for k in order:
                make_cold(path)
                if cond == 'partial':
                    read_head(path, int(size * frac))
                elif cond == 'hot':
                    read_head(path, size)
                res_frac = resident(path)
                r = sample(libs[k], path, env)
                r['exact'] = check(r)
                r['resident'] = res_frac
                del r['points']
                rows[k].append(r)
        for k, rs in rows.items():
            rps = [nrec / r['wall_s'] for r in rs]
            cpu = [r['cpu_s'] / (size / 1e9) for r in rs]
            emit({'cond': cond, 'fraction': frac, 'lib': k,
                  'resident': [round(r['resident'], 4) for r in rs],
                  'records_per_s_median': statistics.median(rps),
                  'records_per_s_range': [min(rps), max(rps)],
                  'wall_s_median': statistics.median(r['wall_s'] for r in rs),
                  'gb_per_s_median': size / 1e9 / statistics.median(
                      r['wall_s'] for r in rs),
                  'cpu_s_per_gb_median': statistics.median(cpu),
                  'cpu_s_per_gb_range': [min(cpu), max(cpu)],
                  'read_stats': [r['read_stats'] for r in rs],
                  'exact': all(r['exact'] for r in rs)})
    os.unlink(path)
    shutil.rmtree(env['DNG_JIT_CACHE_DIR'], ignore_errors=True)
    if not a.dir:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == '__main__':
    main()
