"""dng_scan_feed_gzip on the GPU: gzip files inflated by inflate_kernel and
scanned in place.  A gzip file's points and counters equal those of the same
scan over its decompressed bytes, read as a plain file, under the library's
kernel choice and each forced kernel: the reference goldens and index
goldens through gzip, generated data against the plain files and the C++
oracle, joins between plain and gzip files, batches of many files, files
whose ISIZE understates their size, and the errors."""

import gzip
import json
import os
import shutil
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
import gzcorpus  # noqa: E402
from engines import canon_points, cpp_engine  # noqa: E402
from golden_harness import check_section  # noqa: E402
from hostmirror import dn_index  # noqa: E402
from hostmirror import find as mod_find  # noqa: E402
from dragnet_b200 import datasource_gpu, native  # noqa: E402

pytestmark = pytest.mark.gpu

EINVAL, EIO = -1, -5
PLAN = corpus.make_plan(['-b', 'req.method,res.statusCode,host', '-f',
                         '{"ne":["req.method","HEAD"]}'])


@pytest.fixture(params=['auto', 'tile', 'warp', 'fast', 'jit'])
def kernel(request, monkeypatch):
    """The library's own choice, the general kernels' two geometries, the F
    path with the interpreted matcher and with the compiled one."""
    for v in ('DNG_KERNEL', 'DNG_JIT'):
        monkeypatch.delenv(v, raising=False)
    if request.param == 'fast':
        monkeypatch.setenv('DNG_JIT', '0')
    if request.param == 'jit':
        monkeypatch.setenv('DNG_JIT', 'sync')
    if request.param != 'auto':
        monkeypatch.setenv('DNG_KERNEL', 'fast' if request.param == 'jit'
                           else request.param)
    return request.param


def _write(path, data):
    with open(path, 'wb') as f:
        f.write(data)
    return str(path)


def _records(n, first=0, total=2000000):
    return native.gen_host(native.gen_params(total_records=total), first, n)


def _gz_tree(src, dst):
    """src copied to dst with every file gzipped in place (same names)"""
    shutil.copytree(src, dst)
    for r, _, fs in os.walk(dst):
        for f in fs:
            p = os.path.join(r, f)
            with open(p, 'rb') as fh:
                data = fh.read()
            _write(p, gzip.compress(data, 6))


def scan(plan, files, compression='gzip'):
    return datasource_gpu.run_plan(plan, files=files, compression=compression)


# -- the reference goldens, gzipped --------------------------------------------

@pytest.fixture(scope='module')
def gz_datadir(datadir, tmp_path_factory):
    d = tmp_path_factory.mktemp('gz') / 'tests' / 'data'
    _gz_tree(datadir, str(d))
    return str(d)


@pytest.mark.parametrize('suite', ['scan_file', 'scan_fileset'])
def test_goldens_through_gzip(suite, kernel, goldens, gz_datadir):
    """Every scan case of the golden file and fileset over gzipped data
    prints exactly its golden output."""
    def engine(plan, files):
        r = scan(plan, files)
        assert r.stats['gzip_files'] == len(files), r.stats
        return r.points, r.counters
    n = 0
    for i, sec in enumerate(goldens['suites'][suite]):
        if sec['cmd'] == 'scan':
            check_section(engine, suite, i, sec, gz_datadir)
            n += 1
    assert n >= 8


@pytest.mark.parametrize('suite', ['index_file', 'index_fileset'])
def test_index_goldens_through_gzip(suite, kernel, gz_datadir, tmp_path):
    """`dn build` over gzipped data with compression "gzip", then `dn
    query`: both index goldens."""
    if kernel in ('fast', 'jit'):
        pytest.skip('a fan-out plan never takes the F path')
    with open(os.path.join(os.path.dirname(__file__), 'golden',
                           'index_goldens.json')) as f:
        goldens = json.load(f)

    def builder(ds, metrics, interval):
        ds = dict(ds, compression='gzip')
        d = datasource_gpu.createDatasource(
            {'dsconfig': ds, 'findFiles': mod_find.find_files})
        res = d.build({'metrics': metrics, 'interval': interval,
                       'dryRun': False})
        assert not isinstance(res, Exception), res
    n = 0
    for header, act, exp in dn_index.replay(suite, goldens, gz_datadir,
                                            str(tmp_path), builder):
        assert act == exp, header
        n += header != 'find'
    assert n == len(goldens['suites'][suite])


# -- generated data: gzip against plain files and the oracle -------------------

@pytest.fixture(scope='module')
def generated(tmp_path_factory):
    """~150k records in 5 files, plain and gzipped at levels 1, 6 and 9, the
    last without its trailing newline; with the oracle's answer"""
    d = tmp_path_factory.mktemp('gen')
    plain, gz = [], []
    for k in range(5):
        data = _records(30000, 30000 * k)
        if k == 4:
            data = data.rstrip(b'\n')
        plain.append(_write(d / ('p%d.log' % k), data))
        gz.append(_write(d / ('p%d.log.gz' % k),
                         gzip.compress(data, (1, 6, 9)[k % 3])))
    for p, g in zip(plain, gz):
        with open(p, 'rb') as a, open(g, 'rb') as b:
            assert gzcorpus.oracle(b.read()) == a.read()
    return plain, gz, cpp_engine(PLAN, plain)


def test_generated_equals_plain(kernel, generated):
    plain, gz, (exp_p, exp_c) = generated
    rp = scan(PLAN, plain, None)
    rg = scan(PLAN, gz)
    assert canon_points(rg.points) == canon_points(rp.points) == \
        canon_points(exp_p)
    assert rg.counters == rp.counters == exp_c
    assert rg.flat_counters == rp.flat_counters
    st = rg.stats
    assert st['gzip_files'] == 5 and st['gzip_members'] == 5
    assert st['gzip_inflated_bytes'] == sum(map(os.path.getsize, plain))
    assert st['gzip_compressed_bytes'] == sum(map(os.path.getsize, gz))
    assert st['inflate_ms'] > 0


def test_kernel_choice_on_decompressed_head(generated, monkeypatch):
    """Templated data through gzip: the F kernel, templates learned from the
    decompressed head, as over the plain files."""
    for v in ('DNG_KERNEL', 'DNG_JIT'):
        monkeypatch.delenv(v, raising=False)
    plain, gz, _ = generated
    rp = scan(PLAN, plain, None)
    rg = scan(PLAN, gz)
    assert rg.stats['kernel'] == rp.stats['kernel'] == 'F path'
    assert rg.stats['templates'] == rp.stats['templates'] > 0
    assert rg.stats['templated_records'] == rp.stats['templated_records'] > 0


# -- joins between files ---------------------------------------------------------

def test_joins_between_files(kernel, tmp_path):
    """Plain and gzip files mixed; files that end without a newline; one line
    spread over three .gz files; empty .gz files and .gz files holding only
    part of a line."""
    data = _records(3000)
    rec = data.split(b'\n')
    long_line = rec[5]
    a, b = long_line[:40], long_line[40:90]
    pieces = [
        (b'\n'.join(rec[:100]) + b'\n' + rec[100][:20], 'gz'),
        (rec[100][20:] + b'\n' + b'\n'.join(rec[101:200]), 'plain'),
        (b'\n', 'gz'),
        (b'', 'gz'),
        (a, 'gz'),
        (b, 'gz'),
        (long_line[90:] + b'\n', 'gz'),
        (b'', 'plain'),
        (b'\n'.join(rec[200:1500]) + b'\n', 'gz'),
        (rec[1500][:10], 'plain'),
        (rec[1500][10:] + b'\n', 'gz'),
        (b'', 'gz'),
        (b'\n'.join(rec[1501:2999]), 'gz'),
    ]
    files, plain = [], []
    for i, (chunk, kind) in enumerate(pieces):
        p = _write(tmp_path / ('f%02d.log' % i), chunk)
        plain.append(p)
        files.append(p if kind == 'plain' else _write(
            tmp_path / ('f%02d.log.gz' % i), gzip.compress(chunk)))
    exp_p, exp_c = cpp_engine(PLAN, plain)
    r = scan(PLAN, files)
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    assert r.flat_counters['bytes'] == sum(map(os.path.getsize, plain))
    assert r.stats['gzip_files'] == sum(k == 'gz' for _, k in pieces)


# -- many streams, one large one, wrong size hints ----------------------------

def test_many_streams_and_wrong_hints(kernel, tmp_path):
    """600 small .gz files (several batches), one far larger than the rest
    in the same batch, and multi-member files whose ISIZE names their last
    member only (decoded again in more room)."""
    files, plain = [], []
    first = 0
    for i in range(620):
        n = 4 + (i * 7) % 50
        if i == 300:
            n = 120000
        data = _records(n, first)
        first += n
        p = _write(tmp_path / ('m%03d.log' % i), data)
        plain.append(p)
        if i % 97 == 5:       # several members, and zeros after the last
            cut = data.find(b'\n', len(data) // 3) + 1
            z = gzip.compress(data[:cut]) + gzip.compress(data[cut:], 1) + \
                b'\x00' * 7
        else:
            z = gzip.compress(data)
        files.append(_write(tmp_path / ('m%03d.log.gz' % i), z))
    exp_p, exp_c = cpp_engine(PLAN, plain)
    r = scan(PLAN, files)
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    nmulti = sum(1 for i in range(620) if i % 97 == 5)
    assert r.stats['gzip_files'] == 620
    assert r.stats['gzip_members'] == 620 + nmulti
    assert r.stats['gzip_inflated_bytes'] == sum(map(os.path.getsize, plain))
    # 256 files per batch: three batches, plus one decode again in more room
    # per multi-member file (its ISIZE names only its last member, here 0)
    assert nmulti == 7
    assert r.stats['inflate_launches'] == 3 + nmulti


def test_empty_files_beside_wrong_hints(kernel, tmp_path):
    """Empty .gz files after files of odd sizes, between and after
    multi-member files, in one batch: the runs of files that filled their
    regions start off 16-byte boundaries, and an empty file may be a run of
    its own."""
    data = _records(400)
    cut = [0, 1001, 2778, 2790, 5000, 9003, 12000]
    chunk = [data[cut[k]:cut[k + 1]] for k in range(len(cut) - 1)]
    gz = gzip.compress

    def multi(d):
        h = d.find(b'\n', len(d) // 2) + 1
        return gz(d[:h]) + gz(d[h:], 1)
    pieces = [
        (chunk[0], gz(chunk[0])),                 # 1001 bytes
        (chunk[1], multi(chunk[1])),              # runs out of room
        (b'', gz(b'')),                           # an empty run
        (chunk[2], multi(chunk[2]) + b'\x00' * 3),
        (b'', gz(b'') + b'\x00' * 4),
        (chunk[3], gz(chunk[3])),                 # 2210 bytes, off 16
        (b'', gz(b'') + gz(b'')),
        (chunk[4], gz(chunk[4])),
        (chunk[5], multi(chunk[5])),
        (b'', gz(b'')),                           # last in the batch
    ]
    files, plain = [], []
    for i, (raw, z) in enumerate(pieces):
        plain.append(_write(tmp_path / ('e%02d.log' % i), raw))
        files.append(_write(tmp_path / ('e%02d.log.gz' % i), z))
        assert gzcorpus.oracle(z) == raw
    exp_p, exp_c = cpp_engine(PLAN, plain)
    r = scan(PLAN, files)
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    assert r.flat_counters['bytes'] == cut[-1]
    assert r.stats['gzip_files'] == len(pieces)
    assert r.stats['gzip_members'] == len(pieces) + 4
    assert r.stats['inflate_launches'] == 1 + 3


# -- errors ------------------------------------------------------------------------

def _feed_one(path, plan=PLAN):
    p = native.Plan(json.dumps(plan))
    s = native.Scan(p)
    try:
        s.feed_gzip(path)
        s.finish().close()
    finally:
        s.close()
        p.close()


def test_errors(tmp_path, monkeypatch):
    """A truncated file and one with a flipped byte fail with DNG_EIO naming
    the file; a plain file is refused with DNG_EINVAL; a scan over several
    devices refuses feed_gzip; a following scan succeeds."""
    for v in ('DNG_KERNEL', 'DNG_JIT'):
        monkeypatch.delenv(v, raising=False)
    data = _records(2000)
    z = gzip.compress(data)
    trunc = _write(tmp_path / 'trunc.log.gz', z[:len(z) * 2 // 3])
    with pytest.raises(native.DngError) as e:
        _feed_one(trunc)
    assert e.value.code == EIO and 'trunc.log.gz' in str(e.value)
    assert 'truncated' in str(e.value)
    pos = len(z) // 2
    while True:
        b = bytearray(z)
        b[pos] ^= 0x20
        if gzcorpus.oracle(bytes(b)) is None:
            break
        pos += 1
    flip = _write(tmp_path / 'flip.log.gz', bytes(b))
    with pytest.raises(native.DngError) as e:
        _feed_one(flip)
    assert e.value.code == EIO and 'flip.log.gz' in str(e.value)
    plain = _write(tmp_path / 'plain.log', data)
    with pytest.raises(native.DngError) as e:
        _feed_one(plain)
    assert e.value.code == EINVAL and 'not a gzip file' in str(e.value)
    good = _write(tmp_path / 'good.log.gz', z)
    p = native.Plan(json.dumps(PLAN))
    s = native.Scan(p, devices=[0, 0])
    try:
        with pytest.raises(native.DngError) as e:
            s.feed_gzip(good)
        assert e.value.code == EINVAL
    finally:
        s.close()
        p.close()
    with pytest.raises(datasource_gpu.DsError):
        datasource_gpu.run_plan(PLAN, files=[good], devices=[0, 0],
                                compression='gzip')
    exp_p, exp_c = cpp_engine(PLAN, [plain])
    r = scan(PLAN, [good])
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
