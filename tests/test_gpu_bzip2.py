"""dng_scan_feed_bzip2 on the GPU: bzip2 files decoded with all their blocks
in parallel and scanned in place.  A bzip2 file's points and counters equal
those of the same scan over its decompressed bytes read as a plain file,
under each kernel choice: the reference goldens and index goldens through
bzip2, generated data against the plain files and the C++ oracle, files
that span several waves of blocks, many small files, joins between plain,
gzip and bzip2 files, hand-built streams (one with a false start), and the
errors."""

import bz2
import gzip
import json
import os
import shutil
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import bzcorpus  # noqa: E402
import corpus  # noqa: E402
from engines import canon_points, cpp_engine  # noqa: E402
from golden_harness import check_section  # noqa: E402
from hostmirror import dn_index  # noqa: E402
from hostmirror import find as mod_find  # noqa: E402
from dragnet_b200 import datasource_gpu, native  # noqa: E402

pytestmark = pytest.mark.gpu

EINVAL, EIO = -1, -5
PLAN = corpus.make_plan(['-b', 'req.method,res.statusCode,host', '-f',
                         '{"ne":["req.method","HEAD"]}'])
WAVE_BLOCKS = 1024      # DNG_BZ_WAVE_BLOCKS


@pytest.fixture(params=['tile', 'warp', 'fast'])
def kernel(request, monkeypatch):
    """The general kernels' two geometries and the F path."""
    monkeypatch.delenv('DNG_JIT', raising=False)
    monkeypatch.setenv('DNG_KERNEL', request.param)
    if request.param == 'fast':
        monkeypatch.setenv('DNG_JIT', '0')
    return request.param


def _write(path, data):
    with open(path, 'wb') as f:
        f.write(data)
    return str(path)


def _records(n, first=0, total=2000000):
    return native.gen_host(native.gen_params(total_records=total), first, n)


def scan(plan, files, compression='bzip2'):
    return datasource_gpu.run_plan(plan, files=files, compression=compression)


def _same(r, plain):
    exp_p, exp_c = cpp_engine(PLAN, plain)
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    assert r.flat_counters['bytes'] == sum(map(os.path.getsize, plain))
    assert r.stats['bzip2_decompressed_bytes'] == r.flat_counters['bytes'] \
        or r.stats['bzip2_files'] < len(plain)


# -- the reference goldens, bzip2 ----------------------------------------------

@pytest.fixture(scope='module')
def bz_datadir(datadir, tmp_path_factory):
    d = str(tmp_path_factory.mktemp('bz') / 'tests' / 'data')
    shutil.copytree(datadir, d)
    for r, _, fs in os.walk(d):
        for f in fs:
            p = os.path.join(r, f)
            with open(p, 'rb') as fh:
                data = fh.read()
            _write(p, bz2.compress(data, 9))
    return d


@pytest.mark.parametrize('suite', ['scan_file', 'scan_fileset'])
def test_goldens_through_bzip2(suite, kernel, goldens, bz_datadir):
    def engine(plan, files):
        r = scan(plan, files)
        assert r.stats['bzip2_files'] == len(files), r.stats
        return r.points, r.counters
    n = 0
    for i, sec in enumerate(goldens['suites'][suite]):
        if sec['cmd'] == 'scan':
            check_section(engine, suite, i, sec, bz_datadir)
            n += 1
    assert n >= 8


@pytest.mark.parametrize('suite', ['index_file', 'index_fileset'])
def test_index_goldens_through_bzip2(suite, kernel, bz_datadir, tmp_path):
    if kernel == 'fast':
        pytest.skip('a fan-out plan never takes the F path')
    with open(os.path.join(os.path.dirname(__file__), 'golden',
                           'index_goldens.json')) as f:
        goldens = json.load(f)

    def builder(ds, metrics, interval):
        ds = dict(ds, compression='bzip2')
        d = datasource_gpu.createDatasource(
            {'dsconfig': ds, 'findFiles': mod_find.find_files})
        res = d.build({'metrics': metrics, 'interval': interval,
                       'dryRun': False})
        assert not isinstance(res, Exception), res
    n = 0
    for header, act, exp in dn_index.replay(suite, goldens, bz_datadir,
                                            str(tmp_path), builder):
        assert act == exp, header
        n += header != 'find'
    assert n == len(goldens['suites'][suite])


# -- large files: hundreds of blocks, several waves ------------------------------

@pytest.fixture(scope='module')
def large(tmp_path_factory):
    """500k records at level 1 (over 1024 blocks: two waves) and 400k at
    level 9, with their plain files"""
    d = tmp_path_factory.mktemp('large')
    out = {}
    for lv, n in ((1, 500000), (9, 400000)):
        data = _records(n)
        plain = _write(d / ('l%d.log' % lv), data)
        out[lv] = (plain, _write(d / ('l%d.log.bz2' % lv),
                                 bz2.compress(data, lv)))
    return out


@pytest.mark.parametrize('level', [1, 9])
def test_large_file(kernel, large, level):
    plain, bz = large[level]
    r = scan(PLAN, [bz])
    _same(r, [plain])
    st = r.stats
    assert st['bzip2_files'] == 1 and st['bzip2_streams'] == 1
    assert st['bzip2_blocks'] >= 100
    if level == 1:
        assert st['bzip2_blocks'] > WAVE_BLOCKS     # spans two waves
    assert st['bzip2_compressed_bytes'] == os.path.getsize(bz)
    assert st['bzip2_decompressed_bytes'] == os.path.getsize(plain)
    assert st['bunzip_ms'] > 0 and st['bunzip_launches'] >= 4


def test_many_small_files(kernel, tmp_path):
    """620 files: three batches of at most 256; some multi-stream, some with
    zeros after the last stream, some empty."""
    files, plain, streams = [], [], 0
    first = 0
    for i in range(620):
        n = (i * 7) % 40
        data = _records(n, first)
        first += n
        plain.append(_write(tmp_path / ('m%03d.log' % i), data))
        if i % 50 == 3:
            cut = data.find(b'\n', len(data) // 3) + 1
            z = bz2.compress(data[:cut], 2) + bz2.compress(data[cut:], 8)
            streams += 2
        else:
            z = bz2.compress(data, 1 + i % 9) + b'\0' * (i % 3)
            streams += 1
        files.append(_write(tmp_path / ('m%03d.log.bz2' % i), z))
    r = scan(PLAN, files)
    _same(r, plain)
    assert r.stats['bzip2_files'] == 620
    assert r.stats['bzip2_streams'] == streams
    assert r.stats['bzip2_false_starts'] == 0


def test_joins_plain_gzip_bzip2(kernel, tmp_path):
    """Plain, gzip and bzip2 files interleaved in one scan: unterminated
    last lines at every kind of join, empty and multi-stream files."""
    data = _records(3000)
    rec = data.split(b'\n')
    ln = rec[7]
    pieces = [
        (b'\n'.join(rec[:100]) + b'\n' + rec[100][:20], 'bz'),
        (rec[100][20:] + b'\n' + b'\n'.join(rec[101:200]), 'gz'),
        (b'\n' + rec[200][:5], 'bz'),
        (rec[200][5:] + b'\n' + rec[201][:9], 'plain'),
        (rec[201][9:] + b'\n' + rec[202][:3], 'bz'),
        (rec[202][3:] + b'\n', 'gz'),
        (b'', 'bz'),
        (ln[:30], 'bz'),
        (ln[30:60], 'gz'),
        (ln[60:] + b'\n', 'bz2streams'),
        (b'\n'.join(rec[203:1500]) + b'\n', 'bz2streams'),
        (b'', 'plain'),
        (b'\n'.join(rec[1500:2999]), 'bz'),
    ]
    files, plain = [], []
    for i, (chunk, kind) in enumerate(pieces):
        p = _write(tmp_path / ('f%02d.log' % i), chunk)
        plain.append(p)
        if kind == 'plain':
            files.append(p)
        elif kind == 'gz':
            files.append(_write(tmp_path / ('f%02d.gz' % i),
                                gzip.compress(chunk)))
        else:
            z = bz2.compress(chunk)
            if kind == 'bz2streams':
                h = len(chunk) // 2
                z = bz2.compress(chunk[:h], 3) + bz2.compress(b'') + \
                    bz2.compress(chunk[h:], 9)
            files.append(_write(tmp_path / ('f%02d.bz2' % i), z))
    exp_p, exp_c = cpp_engine(PLAN, plain)
    p = native.Plan(json.dumps(PLAN))
    s = native.Scan(p)
    try:
        for f, (_, kind) in zip(files, pieces):
            if kind == 'plain':
                s.feed_file(f)
            elif kind == 'gz':
                s.feed_gzip(f)
            else:
                s.feed_bzip2(f)
        res = s.finish()
        pts = [(list(zip(['req.method', 'res.statusCode', 'host'], c)), v)
               for c, v in res.points()]
        res.close()
        flat = s.counters()
        st = s.bzip2_stats()
    finally:
        s.close()
        p.close()
    assert canon_points(pts) == canon_points(exp_p)
    assert flat['bytes'] == sum(map(os.path.getsize, plain))
    nbz = sum(k.startswith('bz') for _, k in pieces)
    assert st['bzip2_files'] == nbz
    assert st['bzip2_streams'] == nbz + 2 * 2
    r = datasource_gpu.run_plan(PLAN, files=files, compression='bzip2')
    assert r.stats['bzip2_files'] == nbz


def test_hand_built_streams(kernel, tmp_path):
    """Streams Python's bz2 does not write: randomised blocks, 2 and 6
    groups, 20-bit codes, 20,000 selectors, origPtr at either end, a full
    level-1 block, and a block whose coded symbols hold the block magic (a
    false start the chain drops)."""
    files, plain = [], []
    for name, z in bzcorpus.hand_built():
        raw = bzcorpus.oracle(z)
        assert raw is not None, name
        # a newline after each, so that each is a record of its own
        plain.append(_write(tmp_path / (name + '.log'), raw))
        plain.append(_write(tmp_path / (name + '.nl'), b'\n'))
        files.append(_write(tmp_path / (name + '.bz2'), z))
        files.append(_write(tmp_path / (name + '.nl.bz2'),
                            bz2.compress(b'\n')))
    r = scan(PLAN, files)
    _same(r, plain)
    assert r.stats['bzip2_false_starts'] >= 1
    assert r.stats['bzip2_blocks'] == len(files)


def test_kernel_choice_on_decompressed_head(large, monkeypatch):
    """Templated data through bzip2: the F kernel, with templates learned
    from the decompressed head, as over the plain file."""
    for v in ('DNG_KERNEL', 'DNG_JIT'):
        monkeypatch.delenv(v, raising=False)
    plain, bz = large[9]
    rp = scan(PLAN, [plain], None)
    rb = scan(PLAN, [bz])
    assert rb.stats['kernel'] == rp.stats['kernel'] == 'F path'
    assert rb.stats['templates'] == rp.stats['templates'] > 0


# -- errors ------------------------------------------------------------------------

def _feed_one(path):
    p = native.Plan(json.dumps(PLAN))
    s = native.Scan(p)
    try:
        s.feed_bzip2(path)
        s.finish().close()
    finally:
        s.close()
        p.close()


def test_errors(tmp_path, monkeypatch):
    """Damage fails with DNG_EIO naming the file and the kind; trailing data
    fails; a plain file is refused with DNG_EINVAL; a scan over several
    devices refuses feed_bzip2; a following scan succeeds."""
    for v in ('DNG_KERNEL', 'DNG_JIT'):
        monkeypatch.delenv(v, raising=False)
    data = _records(20000)
    z = bz2.compress(data, 1)
    cases = dict(bzcorpus.damaged_corpus())
    for name, want in (('trunc', 'truncated'),
                       ('crc', 'block CRC mismatch'),
                       ('scrc', 'stream CRC mismatch'),
                       ('header', 'bad block header'),
                       ('trailing', 'trailing data after the last bzip2 '
                        'stream')):
        if name == 'trunc':
            b = z[:len(z) * 2 // 3]
        elif name == 'crc':
            b = cases['bad-block-crc']
        elif name == 'scrc':
            b = cases['bad-stream-crc']
        elif name == 'header':
            b = cases['flip32']
        else:
            b = z + b'junk'
        assert bzcorpus.oracle(b) is None
        f = _write(tmp_path / ('%s.log.bz2' % name), b)
        with pytest.raises(native.DngError) as e:
            _feed_one(f)
        assert e.value.code == EIO, name
        assert '%s.log.bz2' % name in str(e.value), str(e.value)
        assert want in str(e.value), str(e.value)
        assert 'compressed byte' in str(e.value)
    plain = _write(tmp_path / 'plain.log', data)
    with pytest.raises(native.DngError) as e:
        _feed_one(plain)
    assert e.value.code == EINVAL and 'not a bzip2 file' in str(e.value)
    good = _write(tmp_path / 'good.log.bz2', z)
    p = native.Plan(json.dumps(PLAN))
    s = native.Scan(p, devices=[0, 0])
    try:
        with pytest.raises(native.DngError) as e:
            s.feed_bzip2(good)
        assert e.value.code == EINVAL
    finally:
        s.close()
        p.close()
    with pytest.raises(datasource_gpu.DsError):
        datasource_gpu.run_plan(PLAN, files=[good], devices=[0, 0],
                                compression='bzip2')
    r = scan(PLAN, [good])
    _same(r, [plain])
