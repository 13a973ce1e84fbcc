"""How dng_scan_feed_file reads a byte range of a regular file
(dragnet_b200/csrc/direct_read.h), on the CPU: the O_DIRECT alignment plan
read through with real O_DIRECT reads and compared byte for byte with a
buffered read of the same range, the page-cache residency probe on cold,
hot and half-read files and through an overlayfs mount, a file that shrinks
after the plan, and a filesystem that refuses O_DIRECT.  Driven through
tests/hostcheck/direct_read_check.cpp."""

import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')
DRIVER = os.path.join(ROOT, 'tests', 'hostcheck', 'direct_read_check.cpp')


def _kv(line):
    return {k: (int(v) if v.lstrip('-').isdigit() else
                float(v) if v.replace('.', '', 1).lstrip('-').isdigit() else v)
            for k, v in (kv.split('=') for kv in line.split())}


@pytest.fixture(scope='module')
def drc(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp('drc') / 'direct_read_check')
    subprocess.check_call(['g++', '-std=c++17', '-O1', '-Wall', '-Wextra',
                           '-Werror', '-I', CSRC, '-o', exe, DRIVER])

    def run(*cmds):
        r = subprocess.run([exe], input='\n'.join(cmds) + '\n',
                           capture_output=True, text=True, check=True)
        return [_kv(line) for line in r.stdout.splitlines()]
    run.exe = exe
    return run


@pytest.fixture(scope='module')
def C(drc):
    return drc('const')[0]


def _write(path, data):
    with open(path, 'wb') as f:
        f.write(data)
        f.flush()
        os.fsync(f.fileno())


def _cold(path):
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)
        os.posix_fadvise(fd, 0, 0, os.POSIX_FADV_DONTNEED)
    finally:
        os.close(fd)


def _hot(path):
    with open(path, 'rb') as f:
        while f.read(1 << 20):
            pass


@pytest.fixture(scope='module')
def direct_dir(tmp_path_factory, drc):
    d = tmp_path_factory.mktemp('direct')
    p = str(d / 'probe')
    _write(p, b'x' * 8192)
    a = drc('align ' + p)[0]
    r = drc('read %s 0 8192 1 - %s' % (p, d / 'probe.out'))[0]
    if not a['ok'] or r['rc'] == 'nodirect':
        pytest.skip('%s does not support O_DIRECT' % d)
    return d


def _pattern(n, seed):
    import random
    rng = random.Random(seed)
    return bytes(rng.getrandbits(8) for _ in range(n % 4096)) + \
        rng.randbytes(n - n % 4096)


def _cases(fsize, align, blk):
    offs = [0, 1, align - 1, align, align + 1, blk - 1, blk, blk + 1,
            fsize - 1]
    out = set()
    for off in offs:
        if not 0 <= off < fsize:
            continue
        for size in (fsize - off, 1, align - 1, align + 1, blk - 1, blk + 1,
                     4095, 5000, fsize - off - 1):
            if 0 < size <= fsize - off:
                out.add((off, size))
    return sorted(out)


@pytest.mark.parametrize('fsize', [1, 100, 4095, 4097, 3 << 20,
                                   (2 << 22) + 777])
def test_plan_feeds_the_range_byte_for_byte(drc, C, direct_dir, fsize):
    """Every offset and size of the sweep (0, 1, the alignment +- 1, the block
    size +- 1, ranges ending at EOF and before it) read cold through the
    plan with O_DIRECT feeds exactly the bytes a buffered pread of the range
    gives, all of them read direct."""
    blk = C['blk']
    p = str(direct_dir / ('f%d' % fsize))
    data = _pattern(fsize, fsize)
    _write(p, data)
    _cold(p)
    align = drc('align ' + p)[0]['plan']
    cases = _cases(fsize, align, blk)
    cmds, outs = [], []
    for i, (off, size) in enumerate(cases):
        o = str(direct_dir / ('f%d.%d.out' % (fsize, i)))
        if os.path.exists(o):
            os.unlink(o)
        outs.append(o)
        cmds.append('read %s %d %d 1 - %s' % (p, off, size, o))
    res = drc(*cmds)
    for (off, size), o, r in zip(cases, outs, res):
        assert r['rc'] == 0, (off, size, r)
        assert r['base'] == off // align * align
        assert r['nblocks'] == -(-(off + size - r['base']) // blk)
        with open(o, 'rb') as f:
            got = f.read()
        assert got == data[off:off + size], (off, size)
        assert r['direct_bytes'] == size and r['buffered_bytes'] == 0
        assert r['fallbacks'] == 0


def test_residency_probe_cold_and_hot(drc, C, direct_dir):
    """Near 0 after fsync + POSIX_FADV_DONTNEED, near 1 after a full read,
    and on a half-read file what cachestat(2) counts over the whole range
    (where the kernel has it); the policy reads the cold range direct and the
    hot one buffered."""
    p = str(direct_dir / 'resident')
    n = (8 << 20) + 123
    _write(p, _pattern(n, 7))
    _cold(p)
    cold = drc('cached %s 0 %d' % (p, n), 'cached %s 4097 %d' % (p, n - 5000))
    for r in cold:
        assert 0 <= r['fraction'] <= 0.02, r
        assert r['direct'] == 1
    _hot(p)
    hot = drc('cached %s 0 %d' % (p, n), 'cached %s 4097 %d' % (p, n - 5000))
    for r in hot:
        assert r['fraction'] >= 0.98, r
        assert r['direct'] == 0
    # half of it, without readahead (pages still being read count for
    # cachestat, not for mincore): the probe samples 64 windows of the range,
    # cachestat counts every page; they agree to within the windows'
    # resolution
    _cold(p)
    with open(p, 'rb') as f:
        os.posix_fadvise(f.fileno(), 0, 0, os.POSIX_FADV_RANDOM)
        f.read(n // 2)
    for r in drc('cached %s 0 %d' % (p, n), 'cached %s %d %d' % (p, n // 4,
                                                                 n // 2)):
        assert 0.2 < r['fraction'] <= 1.0, r
        if r['cachestat'] >= 0:
            assert abs(r['cachestat'] - r['fraction']) < 0.05, r
        assert r['direct'] == int(r['fraction'] < C['direct_below'])


def test_residency_probe_through_overlayfs(drc, direct_dir):
    """A file read through an overlayfs mount (a container's root
    filesystem), whose pages live on the backing file: hot, it is read
    buffered, though cachestat on the overlay descriptor sees no page; cold,
    it is read direct.  Mounted in a user namespace; skipped where the host
    allows none."""
    import shutil
    if not shutil.which('unshare'):
        pytest.skip('no unshare(1)')
    d = direct_dir / 'ovl'
    for sub in ('lower', 'upper', 'work', 'merged'):
        (d / sub).mkdir(parents=True, exist_ok=True)
    n = 8000000
    _write(str(d / 'lower' / 'f'), _pattern(n, 11))
    def probe():
        script = ('mount -t overlay overlay -o lowerdir={0}/lower,upperdir='
                  '{0}/upper,workdir={0}/work {0}/merged && '
                  'printf "cached {0}/merged/f 0 %d\n" | "$DRC"' % n
                  ).format(d)
        r = subprocess.run(['unshare', '-rm', 'sh', '-c', script],
                           capture_output=True, text=True,
                           env=dict(os.environ, DRC=drc.exe))
        if r.returncode:
            pytest.skip('no overlayfs mount in a user namespace here: %s'
                        % r.stderr.strip()[-200:])
        return _kv(r.stdout.strip())
    _hot(str(d / 'lower' / 'f'))
    hot = probe()
    assert hot['fraction'] >= 0.98 and hot['direct'] == 0, hot
    _cold(str(d / 'lower' / 'f'))
    cold = probe()
    assert cold['fraction'] <= 0.02 and cold['direct'] == 1, cold


@pytest.mark.parametrize('exact', [1, 0])
def test_file_shrinks_after_the_plan(drc, direct_dir, exact):
    """Truncated between planning and reading: an exact range fails with the
    short-read code (DNG_EIO in the library); otherwise the range is fed to
    where the file ends now."""
    p = str(direct_dir / ('shrink%d' % exact))
    n = (3 << 22) + 99
    data = _pattern(n, 3)
    _write(p, data)
    _cold(p)
    o = str(direct_dir / ('shrink%d.out' % exact))
    cut = (5 << 20) + 17
    r = drc('read %s 1 %d %d shrink:%d %s' % (p, n - 1, exact, cut, o))[0]
    if exact:
        assert r['rc'] == -1, r
    else:
        assert r['rc'] == 0, r
        with open(o, 'rb') as f:
            assert f.read() == data[1:cut]


def test_einval_falls_back_to_buffered(drc, direct_dir):
    """O_DIRECT refused with EINVAL: the range is read through the page
    cache, the same bytes, and the fallback is counted once."""
    p = str(direct_dir / 'einval')
    n = (9 << 20) + 5
    data = _pattern(n, 5)
    _write(p, data)
    _cold(p)
    o = str(direct_dir / 'einval.out')
    r = drc('read %s 4097 %d 1 einval %s' % (p, n - 4097, o))[0]
    assert r['rc'] == 0 and r['fallbacks'] == 1, r
    assert r['direct_bytes'] == 0 and r['buffered_bytes'] == n - 4097
    with open(o, 'rb') as f:
        assert f.read() == data[4097:]
