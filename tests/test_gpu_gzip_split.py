"""dng_scan_feed_gzip's split path on the GPU: a large gzip file in a batch
of few is cut into chunks at block starts found on the device and decoded by
many warps (inflate_split.cuh).  Every case compares its points and counters
with the same scan over the plain files and with the C++ oracle; the split
counters show which path ran, and that valid files never fall back to the
one-warp decoder.  Damaged files fail exactly as that decoder, run on the
host, says they do."""

import gzip
import json
import os
import random
import struct
import subprocess
import sys
import zlib

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
import gzcorpus  # noqa: E402
from engines import canon_points, cpp_engine  # noqa: E402
from dragnet_b200 import datasource_gpu, native  # noqa: E402

pytestmark = pytest.mark.gpu

EIO = -5
PLAN = corpus.make_plan(['-b', 'req.method,res.statusCode,host', '-f',
                         '{"ne":["req.method","HEAD"]}'])
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ['none', 'bad gzip header', 'truncated stream', 'invalid block type',
         'invalid stored block lengths', 'invalid Huffman code set',
         'invalid code', 'distance too far back', 'CRC-32 mismatch',
         'ISIZE mismatch']


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


@pytest.fixture
def auto(monkeypatch):
    for v in ('DNG_KERNEL', 'DNG_JIT'):
        monkeypatch.delenv(v, raising=False)


def _write(path, data):
    with open(path, 'wb') as f:
        f.write(data)
    return str(path)


def _records(n, first=0, total=4000000):
    return native.gen_host(native.gen_params(total_records=total), first, n)


def compare(plain, gz):
    """the scan of gz equals the scan of plain and the oracle's; its stats"""
    exp_p, exp_c = cpp_engine(PLAN, plain)
    rp = datasource_gpu.run_plan(PLAN, files=plain)
    rg = datasource_gpu.run_plan(PLAN, files=gz, compression='gzip')
    assert canon_points(rg.points) == canon_points(rp.points) == \
        canon_points(exp_p)
    assert rg.counters == rp.counters == exp_c
    st = rg.stats
    assert st['gzip_inflated_bytes'] == sum(
        os.path.getsize(p) for p, g in zip(plain, gz) if g.endswith('.gz'))
    assert st['gzip_fallbacks'] == 0
    assert st['inflate_ms'] > 0
    return st


def pair(d, name, data, z):
    return _write(d / name, data), _write(d / (name + '.gz'), z)


# -- one large file ------------------------------------------------------------------

@pytest.fixture(scope='module')
def big_data():
    return _records(400000)


@pytest.fixture(scope='module')
def big(big_data, tmp_path_factory):
    """400k records, gzipped at levels 1, 6, 9 and with Z_HUFFMAN_ONLY"""
    d = tmp_path_factory.mktemp('big')
    out = {}
    for name, z in (('1', gzip.compress(big_data, 1)),
                    ('6', gzip.compress(big_data, 6)),
                    ('9', gzip.compress(big_data, 9)),
                    ('huffman', gzcorpus.gz(big_data, 6,
                                            strategy=zlib.Z_HUFFMAN_ONLY))):
        out[name] = pair(d, 'big%s.log' % name, big_data, z)
    return out


def _one_split(st, min_chunks=32):
    assert st['gzip_files'] == 1 and st['gzip_split_files'] == 1, st
    assert st['gzip_chunks'] >= min_chunks, st
    assert st['gzip_members'] == 1
    assert st['gzip_split_launches'] >= 4
    assert st['inflate_launches'] == 0


def test_large_file_every_kernel(kernel, big):
    p, g = big['6']
    _one_split(compare([p], [g]))


@pytest.mark.parametrize('level', ['1', '9', 'huffman'])
def test_large_file_levels(auto, big, level):
    p, g = big[level]
    _one_split(compare([p], [g]))


# -- streams that are hard to split ---------------------------------------------------

def far_repeats(seed=3):
    """records text repeated at a period of 32,500 bytes with a digit
    changed every ~60 bytes: matches reaching ~32 KiB back across every
    chunk start"""
    rng = random.Random(seed)
    block = bytearray(_records(150, 7)[:32500])
    out = bytearray()
    for _ in range(600):
        for i in range(rng.randrange(60), len(block), 61):
            if 48 <= block[i] <= 57:
                block[i] = 48 + rng.randrange(10)
        out += block
    return bytes(out)


def stored_payload():
    """dynamic blocks, stored blocks holding raw deflate streams, dynamic
    blocks: the stored bytes hold block headers that are no block starts"""
    a_txt, c_txt = _records(90000, 0), _records(90000, 90000)
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    a = c.compress(a_txt) + c.flush(zlib.Z_FULL_FLUSH)
    payload = b''.join(gzcorpus.raw_deflate(_records(4000, 200000 + 4000 * s),
                                            9) for s in range(8))
    body = a + gzcorpus.stored(payload, final=False) + \
        gzcorpus.raw_deflate(c_txt, 6)
    data = a_txt + payload + c_txt
    return data, gzcorpus.member(body, data)


def test_far_repeats(auto, tmp_path):
    data = far_repeats()
    p, g = pair(tmp_path, 'far.log', data, gzip.compress(data, 9))
    _one_split(compare([p], [g]), 2)


def test_stored_payload(auto, tmp_path):
    data, z = stored_payload()
    assert gzip.decompress(z) == data
    p, g = pair(tmp_path, 'stored.log', data, z)
    st = compare([p], [g])
    _one_split(st)
    assert st['gzip_false_starts'] >= 1


def test_compressibility_swing(auto, tmp_path):
    """records, then ~100 MB of records padded with 8 KB of spaces (about
    1000 times more compressible), then records"""
    pad = b'{"pad":"' + b' ' * 8192 + b'"}\n'
    data = _records(100000) + pad * 12000 + _records(50000, 100000)
    p, g = pair(tmp_path, 'swing.log', data, gzip.compress(data, 6))
    _one_split(compare([p], [g]), 16)


def test_members_and_zeros(auto, tmp_path):
    """two large members and zeros after them: ISIZE names the last member
    only, the chain gives the length"""
    a, b = _records(100000), _records(100000, 100000)
    z = gzip.compress(a, 6) + gzip.compress(b, 1) + b'\x00' * 100
    assert struct.unpack('<I', z[-104:-100])[0] == len(b)
    p, g = pair(tmp_path, 'members.log', a + b, z)
    st = compare([p], [g])
    assert st['gzip_split_files'] == 1 and st['gzip_members'] == 2
    assert st['gzip_chunks'] >= 32 and st['inflate_launches'] == 0


def test_large_among_small(auto, tmp_path):
    """one large file without its trailing newline in a batch with small
    gzip files, between plain files; lines join across every file"""
    data = _records(160000)
    cuts = [0, 900, 2500, data.find(b'\n', 2000000) + 30, None]
    cuts[-1] = cuts[3] + 5000
    pieces = [data[cuts[k]:cuts[k + 1]] for k in range(4)]
    pieces.append(data[cuts[4]:])
    kinds = ['plain', 'gz', 'gz', 'gz', 'plain']
    plain, files = [], []
    for i, (piece, kind) in enumerate(zip(pieces, kinds)):
        pp, gg = pair(tmp_path, 'm%d.log' % i, piece, gzip.compress(piece))
        plain.append(pp)
        files.append(pp if kind == 'plain' else gg)
    assert not pieces[2].endswith(b'\n')
    st = compare(plain, files)
    assert st['gzip_files'] == 3 and st['gzip_split_files'] == 1
    assert st['inflate_launches'] == 1


def test_many_small_files(auto, tmp_path):
    plain, files = [], []
    for i in range(64):
        data = _records(3000, 3000 * i)
        pp, gg = pair(tmp_path, 's%02d.log' % i, data, gzip.compress(data))
        plain.append(pp)
        files.append(gg)
    st = compare(plain, files)
    assert st['gzip_split_files'] == 0 and st['gzip_chunks'] == 0
    assert st['inflate_launches'] == 1


# -- damage ---------------------------------------------------------------------------

@pytest.fixture(scope='module')
def whole(tmp_path_factory):
    """the one-lane decoder built for the host"""
    exe = str(tmp_path_factory.mktemp('ic') / 'inflate_check')
    subprocess.check_call(['g++', '-std=c++17', '-O2', '-I',
                           os.path.join(ROOT, 'dragnet_b200', 'csrc'), '-o',
                           exe, os.path.join(ROOT, 'tests', 'hostcheck',
                                             'inflate_check.cpp')])
    return exe


def host_error(exe, z, tmp_path):
    src, dst = tmp_path / 'c.bin', tmp_path / 'r.bin'
    src.write_bytes(struct.pack('<IQ', 1, len(z)) + z)
    subprocess.check_call([exe, str(src), str(dst)])
    status, kind, bit = struct.unpack_from('<IIQ', dst.read_bytes())
    assert status == 2
    return '%s (compressed byte %d)' % (KINDS[kind], bit // 8)


def _feed_one(path):
    p = native.Plan(json.dumps(PLAN))
    s = native.Scan(p)
    try:
        s.feed_gzip(path)
        s.finish().close()
    finally:
        s.close()
        p.close()


def _failing_flip(z, pos):
    while True:
        b = bytearray(z)
        b[pos] ^= 0x20
        if gzcorpus.oracle(bytes(b)) is None:
            return bytes(b)
        pos += 1


def test_damage(auto, whole, tmp_path):
    data = _records(100000)
    z = gzip.compress(data, 6)
    assert len(z) > 40 * (64 << 10) // 2
    cases = {'trunc': z[:len(z) * 2 // 3],
             'first': _failing_flip(z, 2000),
             'middle': _failing_flip(z, len(z) // 2),
             'last': _failing_flip(z, len(z) - 3000)}
    crc = bytearray(z)
    crc[-8] ^= 1
    isz = bytearray(z)
    isz[-4] ^= 1
    cases['crc'], cases['isize'] = bytes(crc), bytes(isz)
    for name, bad in sorted(cases.items()):
        path = _write(tmp_path / ('%s.log.gz' % name), bad)
        want = host_error(whole, bad, tmp_path)
        with pytest.raises(native.DngError) as e:
            _feed_one(path)
        assert e.value.code == EIO, name
        assert path + ': corrupt gzip data: ' + want + ' (EIO)' in \
            str(e.value), (name, str(e.value), want)
    p, g = pair(tmp_path, 'good.log', data, z)
    _one_split(compare([p], [g]))
