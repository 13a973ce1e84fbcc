"""dng_scan_feed_file on files that are not in the page cache: read with
O_DIRECT straight into the pinned ring (direct_read.h), on the GPU.  Points
and counters equal the oracle's on the same files, read cold and hot, on one
device and cut over several, under the library's kernel choice and each
forced kernel; read_stats says how the bytes were read.

The files are made cold with fsync + POSIX_FADV_DONTNEED on each one; that
needs a directory on a filesystem with a page cache and O_DIRECT (not tmpfs).
Where there is none, the tests skip and say so."""

import ctypes
import json
import os
import shutil
import sys
import tempfile

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import canon_points, cpp_engine  # noqa: E402
from golden_harness import check_section  # noqa: E402
from test_gpu_framing import limit_input  # noqa: E402
from dragnet_b200 import datasource_gpu, native  # noqa: E402

pytestmark = pytest.mark.gpu

EIO, EUNSUPPORTED, ELIMIT = -5, -6, -7
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLAN = corpus.make_plan(['-b', 'req.method,res.statusCode,host', '-f',
                         '{"ne":["req.method","HEAD"]}'])


@pytest.fixture(params=['auto', 'tile', 'warp', 'fast'])
def kernel(request, monkeypatch):
    """The library's own choice, the general kernels' two geometries and the
    F path forced on, as the parity tests run them."""
    for v in ('DNG_KERNEL', 'DNG_JIT'):
        monkeypatch.delenv(v, raising=False)
    if request.param == 'fast':
        monkeypatch.setenv('DNG_JIT', '0')
    if request.param != 'auto':
        monkeypatch.setenv('DNG_KERNEL', request.param)
    return request.param


def fs_type(path):
    """The type of the filesystem path is on (/proc/self/mountinfo)."""
    path = os.path.realpath(path)
    best, typ = '', None
    with open('/proc/self/mountinfo') as f:
        for line in f:
            parts = line.split()
            mnt = parts[4]
            fstype = parts[parts.index('-') + 1]
            if (path == mnt or path.startswith(mnt.rstrip('/') + '/')) \
                    and len(mnt) >= len(best):
                best, typ = mnt, fstype
    return typ


def resident(path):
    """The share of path's pages in the page cache (mincore)."""
    n = os.path.getsize(path)
    if not n:
        return 0.0
    libc = ctypes.CDLL(None, use_errno=True)
    libc.mmap.restype = ctypes.c_void_p
    libc.mmap.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int,
                          ctypes.c_int, ctypes.c_int, ctypes.c_long]
    ps = os.sysconf('SC_PAGE_SIZE')
    pages = (n + ps - 1) // ps
    vec = (ctypes.c_ubyte * pages)()
    fd = os.open(path, os.O_RDONLY)
    try:
        addr = libc.mmap(None, n, 1, 1, fd, 0)     # PROT_READ, MAP_SHARED
        assert addr not in (None, ctypes.c_void_p(-1).value)
        try:
            assert libc.mincore(ctypes.c_void_p(addr), ctypes.c_size_t(n),
                                vec) == 0
        finally:
            libc.munmap(ctypes.c_void_p(addr), ctypes.c_size_t(n))
    finally:
        os.close(fd)
    return sum(v & 1 for v in vec) / pages


def make_cold(*paths):
    for p in paths:
        fd = os.open(p, os.O_RDONLY)
        try:
            os.fsync(fd)
            os.posix_fadvise(fd, 0, 0, os.POSIX_FADV_DONTNEED)
        finally:
            os.close(fd)


def make_hot(*paths):
    for p in paths:
        with open(p, 'rb') as f:
            while f.read(8 << 20):
                pass


def _usable(d):
    """d can hold a file the tests make cold and read with O_DIRECT"""
    if fs_type(d) in (None, 'tmpfs', 'ramfs', 'devtmpfs'):
        return False
    p = os.path.join(d, 'probe')
    try:
        with open(p, 'wb') as f:
            f.write(b'x' * (1 << 20))
        make_cold(p)
        fd = os.open(p, os.O_RDONLY | os.O_DIRECT)
        os.close(fd)
        return resident(p) < 0.05
    except OSError:
        return False
    finally:
        if os.path.exists(p):
            os.unlink(p)


@pytest.fixture(scope='module')
def cold_dir(tmp_path_factory):
    made = []
    cands = [str(tmp_path_factory.mktemp('direct'))]
    for parent in (os.path.expanduser('~'), ROOT):
        try:
            made.append(tempfile.mkdtemp(prefix='dng-direct-', dir=parent))
            cands.append(made[-1])
        except OSError:
            pass
    found = next((d for d in cands if _usable(d)), None)
    try:
        if found is None:
            pytest.skip('no directory on a filesystem with a page cache that '
                        'supports O_DIRECT (tried %s)' % ', '.join(
                            '%s: %s' % (d, fs_type(d)) for d in cands))
        print('cold files on %s (%s)' % (found, fs_type(found)))
        yield found
    finally:
        for d in made:
            shutil.rmtree(d, ignore_errors=True)


def read_stats_of(plan, files, devices=None):
    """(points, counters, flat counters, read stats, per-shard read stats)
    of one scan of files"""
    p = native.Plan(json.dumps(plan))
    s = native.Scan(p, devices=devices) if devices else native.Scan(p)
    try:
        for f in files:
            s.feed_file(f)
        r = s.finish()
        names = [b['name'] for b in plan['breakdowns']]
        pts = [(list(zip(names, c)), v) for c, v in r.points()]
        r.close()
        flat = s.counters()
        per = [sh.read_stats() for sh in s.shards(len(devices))] \
            if devices else []
        return pts, flat, s.read_stats(), per
    finally:
        s.close()
        p.close()


def _records(n, first=0, total=2000000):
    return native.gen_host(native.gen_params(total_records=total), first, n)


def _write(path, data):
    with open(path, 'wb') as f:
        f.write(data)


# -- the golden data, cold ----------------------------------------------------

@pytest.mark.parametrize('suite', ['scan_file', 'scan_fileset'])
def test_goldens_cold(suite, kernel, goldens, datadir, cold_dir):
    """Every scan case of the golden file and fileset, each file made cold
    before the scan: the goldens, every byte read direct."""
    d = os.path.join(cold_dir, 'golden-' + suite)
    if not os.path.isdir(d):
        shutil.copytree(datadir, d)

    def engine(plan, files):
        make_cold(*files)
        r = datasource_gpu.run_plan(plan, files=files)
        total = sum(os.path.getsize(f) for f in files)
        assert r.stats['direct_bytes'] == total, r.stats
        assert r.stats['buffered_bytes'] == 0
        assert r.stats['direct_ranges'] == sum(
            1 for f in files if os.path.getsize(f))
        assert r.stats['fallbacks'] == 0
        return r.points, r.counters
    n = 0
    for i, sec in enumerate(goldens['suites'][suite]):
        if sec['cmd'] == 'scan':
            check_section(engine, suite, i, sec, d)
            n += 1
    assert n >= 8


def test_cold_fileset_edges(kernel, datadir, cold_dir):
    """Golden logs with an empty file, files under 4096 bytes, and a file
    without its trailing newline whose last record ends in the next file,
    both read direct: the oracle's points and counters."""
    d = os.path.join(cold_dir, 'edges')
    os.makedirs(d, exist_ok=True)
    logs = sorted(os.path.join(r, f) for r, _, fs in os.walk(datadir)
                  for f in fs)
    with open(logs[0], 'rb') as f:
        a = f.read()
    with open(logs[1], 'rb') as f:
        b = f.read()
    cut = a.rfind(b'\n', 0, len(a) - 1) + 30      # inside a's last record
    parts = [a[:cut], a[cut:] + b[:3000], b'', b[3000:4000], b[4000:]]
    files = []
    for i, data in enumerate(parts):
        p = os.path.join(d, 'part%d.log' % i)
        _write(p, data)
        files.append(p)
    assert not parts[0].endswith(b'\n') and len(parts[1]) < 4096
    exp_p, exp_c = cpp_engine(PLAN, files)
    make_cold(*files)
    r = datasource_gpu.run_plan(PLAN, files=files)
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    assert r.stats['direct_bytes'] > 0
    assert r.stats['direct_bytes'] + r.stats['buffered_bytes'] == \
        sum(map(len, parts))
    assert r.stats['direct_ranges'] == 4


# -- one large generated file, cold and hot -----------------------------------

@pytest.fixture(scope='module')
def big(cold_dir):
    """~300 MB: many 4 MiB blocks, every slot of the pinned ring several
    times over, GROUP boundaries; with the oracle's answer"""
    p = os.path.join(cold_dir, 'big.log')
    n = 1200000
    with open(p, 'wb') as f:
        for first in range(0, n, 400000):
            f.write(_records(min(400000, n - first), first))
        f.write(b'{"req":{"method":"GET"},"res":{"statusCode":200}')  # no \n
    exp = cpp_engine(PLAN, [p], threads=os.cpu_count() or 1)
    return p, exp


def test_large_file_cold(kernel, big):
    p, (exp_p, exp_c) = big
    make_cold(p)
    r = datasource_gpu.run_plan(PLAN, files=[p])
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    assert r.flat_counters['bytes'] == os.path.getsize(p)
    assert r.stats['direct_bytes'] == os.path.getsize(p), r.stats
    assert r.stats['buffered_bytes'] == 0 and r.stats['direct_ranges'] == 1


def test_large_file_hot(kernel, big):
    p, (exp_p, exp_c) = big
    make_hot(p)
    if resident(p) < 0.99:
        pytest.skip('the page cache does not hold the whole file here')
    r = datasource_gpu.run_plan(PLAN, files=[p])
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    assert r.stats['direct_bytes'] == 0 and r.stats['direct_ranges'] == 0
    assert r.stats['buffered_bytes'] == os.path.getsize(p)


# -- several devices: shard ranges that start and end unaligned ---------------

def _filler(n):
    head, tail = b'{"req":{"method":"PAD"},"pad":"', b'"}\n'
    return head + b'x' * (n - len(head) - len(tail)) + tail


def cut_files(d):
    """Two files (the first not a multiple of 4096 bytes) padded so that two
    shards cut the stream just before, on and just after a newline in the
    middle of the first file"""
    A = _records(150000) + b'{"req":{"method":"SPLIT"'    # ends mid-record
    B = b'},"res":{"statusCode":201}}\n' + _records(90000, 150000)
    assert len(A) % 4096
    T0 = len(A) + len(B)
    nl = A.index(b'\n', T0 // 2 + 1000)
    out = {}
    for name, c in (('before', nl - 1), ('on', nl), ('after', nl + 1)):
        paths = []
        for i, data in enumerate((A, B + _filler(2 * c - T0))):
            p = os.path.join(d, 'cut-%s.%d.log' % (name, i))
            _write(p, data)
            paths.append(p)
        assert sum(map(os.path.getsize, paths)) // 2 == c
        out[name] = paths
    return out


@pytest.fixture(scope='module')
def cuts(cold_dir):
    out = {}
    for name, paths in cut_files(cold_dir).items():
        out[name] = (paths, cpp_engine(PLAN, paths))
    return out


@pytest.mark.parametrize('case', ['before', 'on', 'after'])
def test_shards_cold(case, kernel, cuts):
    """devices = [0, 0] (plus [0, 0, 0], and [0, 1] where there are two
    GPUs) over cold files: the oracle's points and counters, the shards'
    read_stats sum to the scan's, every byte read once."""
    import torch
    paths, (exp_p, exp_c) = cuts[case]
    T = sum(map(os.path.getsize, paths))
    configs = [[0, 0], [0, 0, 0]]
    if torch.cuda.device_count() > 1:
        configs.append([0, 1])
    for devices in configs:
        make_cold(*paths)
        pts, flat, rs, per = read_stats_of(PLAN, paths, devices)
        assert canon_points(pts) == canon_points(exp_p), devices
        assert flat['bytes'] == T
        assert len(per) == len(devices)
        for k in rs:
            assert rs[k] == sum(p[k] for p in per), (k, rs, per)
        assert rs['direct_bytes'] + rs['buffered_bytes'] == T
        assert rs['direct_bytes'] > 0, rs
        make_cold(*paths)
        r = datasource_gpu.run_plan(PLAN, files=paths, devices=devices)
        assert r.counters == exp_c, devices
        assert [sh['direct_bytes'] + sh['buffered_bytes']
                for sh in r.stats['shards']] == [
                    p['direct_bytes'] + p['buffered_bytes'] for p in per]


# -- errors -------------------------------------------------------------------

@pytest.fixture(scope='module')
def long_lines(cold_dir):
    out = {}
    for n in ((1 << 24) - 1, 1 << 24):
        term, _, _ = limit_input(n)
        p = os.path.join(cold_dir, 'long%d.log' % n)
        _write(p, term)
        out[n] = p
    return out


def test_longest_line_cold(kernel, long_lines):
    """A line of 2^24 - 1 bytes over several blocks of a cold file scans as
    the oracle says; one of 2^24 bytes fails as on the page-cache path."""
    plan = corpus.make_plan(['-b', 'req.method'])
    p = long_lines[(1 << 24) - 1]
    exp_p, exp_c = cpp_engine(plan, [p])
    make_cold(p)
    r = datasource_gpu.run_plan(plan, files=[p])
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    assert r.stats['direct_bytes'] == os.path.getsize(p)
    make_cold(long_lines[1 << 24])
    with pytest.raises(native.DngError) as ei:
        datasource_gpu.run_plan(plan, files=[long_lines[1 << 24]])
    assert ei.value.code in (ELIMIT, EUNSUPPORTED), ei.value


def test_truncated_after_feed_is_eio(kernel, cold_dir):
    """A cold file truncated between feed_file and finish of a multi-device
    scan fails with DNG_EIO.  The shards find the size changed when they open
    the file, before any read: the direct reader's own rule for a file that
    ends early (DR_SHORT) is tested on the CPU, in
    test_direct_read_host.py."""
    data = _records(200000)
    p = os.path.join(cold_dir, 'trunc.log')
    pl = native.Plan(json.dumps(PLAN))
    try:
        _write(p, data)
        make_cold(p)
        s = native.Scan(pl, devices=[0, 0])
        s.feed_file(p)
        os.truncate(p, len(data) // 3)
        make_cold(p)
        with pytest.raises(native.DngError) as ei:
            s.finish()
        assert ei.value.code == EIO
        s.close()
    finally:
        pl.close()
