"""The bytes the GPU gzip and bzip2 decoders feed the scan, byte for byte
against zlib and bz2 (gzcorpus.oracle, bzcorpus.oracle).

tests/gpucheck/cz_capture.cu links the library's own compressed-input object
(compressed.o) with stubs for the six functions it takes from api.cu, and
keeps every buffer compressed.cu feeds, copied out on the scan's stream when
the scan's kernels would read it.  Every buffer the decoders allocate starts
filled with a poison byte, so bytes a decoder never wrote differ between
poisons.  A second build of compressed.cu with tiny policy limits makes
ordinary files span bzip2 waves, emit in many groups and split into many
gzip chunks.  Errors are checked against the host one-lane drivers
(tests/hostcheck/inflate_check.cpp, bunzip_check.cpp); counts against them
too.  Last, one scan through the real library feeds plain, gzip and bzip2
pieces of one stream and must find every line exactly once."""

import bz2
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
import bzcorpus  # noqa: E402
import corpus  # noqa: E402
import gzcorpus  # noqa: E402
from engines import cpp_engine  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')
HARNESS = os.path.join(ROOT, 'tests', 'gpucheck', 'cz_capture.cu')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
EINVAL, EIO = -1, -5
# the policy variant: bzip2 waves of 3 block candidates, emit groups of
# 64 KiB, gzip chunks down to 32 KiB
VARIANT = ['-DDNG_BZ_WAVE_BLOCKS=3', '-DDNG_BZ_EMIT_OUT=65536',
           '-DDNG_GZ_SPLIT_FLOOR=32768']
WAVE = {'lib': 1024, 'variant': 3}     # DNG_BZ_WAVE_BLOCKS of each build
GZ_KINDS = ['none', 'bad gzip header', 'truncated stream',
            'invalid block type', 'invalid stored block lengths',
            'invalid Huffman code set', 'invalid code',
            'distance too far back', 'CRC-32 mismatch', 'ISIZE mismatch']
BZ_KINDS = ['none', 'bad stream header', 'bad block header',
            'bad selector or code lengths', 'invalid code', 'block overflow',
            'block CRC mismatch', 'stream CRC mismatch', 'truncated',
            'trailing data after the last bzip2 stream']
BZ_TRAILING = 9


# -- building ---------------------------------------------------------------------

def nvflags():
    """the Makefile's NVFLAGS"""
    out = subprocess.check_output(
        ['make', '-s', '--no-print-directory', '-C', CSRC, '--eval',
         'print-nvflags: ; @echo $(NVFLAGS)', 'print-nvflags'])
    return out.decode().split()


def compile_object(dest, defines=()):
    subprocess.check_call([NVCC] + nvflags() + list(defines) +
                          ['-c', '-o', dest,
                           os.path.join(CSRC, 'compressed.cu')])
    return dest


def link_harness(obj, dest):
    subprocess.check_call([NVCC, '-O2', '-std=c++17', '-gencode',
                           'arch=compute_90a,code=sm_90a', '-Xcompiler',
                           '-Wall', '-I', CSRC, '-o', dest, HARNESS, obj])
    return dest


@pytest.fixture(scope='module')
def exes(tmp_path_factory):
    """the harness on the library's object and on the policy variant"""
    d = tmp_path_factory.mktemp('cz')
    obj = os.path.join(CSRC, 'build', 'compressed.o')
    if not os.path.exists(obj):
        obj = compile_object(str(d / 'compressed.o'))
    var = compile_object(str(d / 'variant.o'), VARIANT)
    return {'lib': link_harness(obj, str(d / 'cz_lib')),
            'variant': link_harness(var, str(d / 'cz_variant'))}


def _host_tool(tmp_path_factory, name):
    exe = str(tmp_path_factory.mktemp(name) / name)
    subprocess.check_call(['g++', '-std=c++17', '-O2', '-I', CSRC, '-o', exe,
                           os.path.join(ROOT, 'tests', 'hostcheck',
                                        name + '.cpp')])
    return exe


@pytest.fixture(scope='module')
def inflate_check(tmp_path_factory):
    return _host_tool(tmp_path_factory, 'inflate_check')


@pytest.fixture(scope='module')
def bunzip_check(tmp_path_factory):
    return _host_tool(tmp_path_factory, 'bunzip_check')


def host_inflate(exe, cases, tmp_path):
    """per case (status, kind, bit, members) of the one-lane gzip decoder"""
    src, dst = tmp_path / 'ic.in', tmp_path / 'ic.out'
    src.write_bytes(struct.pack('<I', len(cases)) + b''.join(
        struct.pack('<Q', len(z)) + z for z in cases))
    subprocess.check_call([exe, str(src), str(dst)])
    raw, off, out = dst.read_bytes(), 0, []
    for _ in cases:
        status, kind, bit, members, _, n = struct.unpack_from('<IIQIIQ', raw,
                                                              off)
        off += 32 + n
        out.append((status, kind, bit, members))
    return out


def host_bunzip(exe, cases, wave, tmp_path):
    """per case (kind, bit, streams, blocks, false_starts) of the one-lane
    bzip2 decoder at `wave` block candidates per wave"""
    src, dst = tmp_path / 'bc.in', tmp_path / 'bc.out'
    src.write_bytes(bzcorpus.pack_cases([(z, []) for z in cases]))
    subprocess.check_call([exe, str(src), str(dst), str(wave)])
    raw, off, out = dst.read_bytes(), 0, []
    for _ in cases:
        kind, bit, st, bl, fs, n = struct.unpack_from('<IQIIIQ', raw, off)
        off += 32 + n
        out.append((kind, bit, st, bl, fs))
    return out


# -- running the harness ----------------------------------------------------------

def _write(path, data):
    with open(path, 'wb') as f:
        f.write(data)
    return str(path)


def capture(exe, scans, tmp_path, timeout=300):
    """Run `scans` (each a dict: name, files [(kind 'gz'|'bz', path)], sm,
    poison, cap) in one harness process; per scan its result line with its
    captured bytes under 'bytes'."""
    out = tmp_path / 'out'
    out.mkdir(exist_ok=True)
    lines = []
    for sc in scans:
        lines.append('scan %s %d %d %d' % (sc['name'], sc.get('sm', 0),
                                           sc.get('poison', 0), sc['cap']))
        lines += ['%s %s' % f for f in sc['files']]
        lines.append('end')
    man = tmp_path / 'manifest'
    man.write_text('\n'.join(lines) + '\n')
    try:
        r = subprocess.run([exe, str(man), str(out)], capture_output=True,
                           timeout=timeout)
        said = r.stdout.decode()
    except subprocess.TimeoutExpired as e:
        said = (e.stdout or b'').decode()
        raise AssertionError('hung in ' + (said.strip().split('\n') or
                                           ['?'])[-1])
    assert r.returncode == 0, (r.returncode, said[-500:],
                               r.stderr.decode()[-2000:])
    res = [json.loads(ln) for ln in (out / 'results').read_text().split('\n')
           if ln]
    assert len(res) == len(scans)
    for k, x in enumerate(res):
        x['bytes'] = (out / ('%d.bin' % k)).read_bytes()
        assert not x['overflow'], x['name']
    return res


def clean(x):
    """every feed aligned, no buffer freed while the stream was busy"""
    assert all(a for _, a in x['feeds']), (x['name'], x['feeds'])
    assert x['busy_frees'] == 0, x['name']


def decoded(x, want):
    """a scan that decoded: no error, the oracle's bytes, counted"""
    clean(x)
    assert x['rcs'] == [0] * len(x['rcs']) and x['err_code'] == 0, \
        (x['name'], x['rcs'], x['err'])
    got = x['bytes']
    if got != want:
        at = next((i for i, (a, b) in enumerate(zip(got, want)) if a != b),
                  min(len(got), len(want)))
        raise AssertionError('%s: %d bytes, the oracle %d; first difference '
                             'at byte %d' % (x['name'], len(got), len(want),
                                             at))
    assert sum(n for n, _ in x['feeds']) == len(want)


def cap_of(*lens):
    return max(sum(lens), 1)


# -- inputs ---------------------------------------------------------------------------

def tiny_streams():
    """6,000 bzip2 streams of one short line each"""
    lines = [b'{"n":%d}\n' % i for i in range(6000)]
    return b''.join(bz2.compress(ln, 1 + i % 9) for i, ln in enumerate(lines))


def big_text():
    return gzcorpus.ndjson(110000, 9)     # about 15 MB


def far_repeats(seed=3):
    """text repeated at a period of 32,500 bytes with a digit changed every
    ~60 bytes: matches reaching ~32 KiB back across every chunk start"""
    rng = random.Random(seed)
    block = bytearray(gzcorpus.ndjson(200, 7)[:32500])
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
    a_txt, c_txt = gzcorpus.ndjson(20000, 11), gzcorpus.ndjson(20000, 12)
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    a = c.compress(a_txt) + c.flush(zlib.Z_FULL_FLUSH)
    payload = b''.join(gzcorpus.raw_deflate(gzcorpus.ndjson(1000, 20 + s), 9)
                       for s in range(8))
    body = a + gzcorpus.stored(payload, final=False) + \
        gzcorpus.raw_deflate(c_txt, 6)
    return gzcorpus.member(body, a_txt + payload + c_txt)


def many_members():
    """at least 4 MB in 3,200 members, a few of them empty: more members
    than a split chunk has slots for"""
    text = gzcorpus.ndjson(170000, 13)
    cuts = sorted(random.Random(4).sample(range(1, len(text)), 3199))
    parts = [text[a:b] for a, b in zip([0] + cuts, cuts + [len(text)])]
    parts[100] = parts[2000] = b''
    z = b''.join(gzip.compress(p, 1 + i % 9) for i, p in enumerate(parts))
    assert len(z) >= 4 << 20
    return z


@pytest.fixture(scope='module')
def gz_large(tmp_path_factory):
    """(name, path, oracle bytes) of the large gzip files"""
    d = tmp_path_factory.mktemp('gzl')
    text = big_text()
    out = []
    for name, z in (('l1', gzip.compress(text, 1)),
                    ('l6', gzip.compress(text, 6)),
                    ('l9', gzip.compress(text, 9)),
                    ('huffman', gzcorpus.gz(text, 6,
                                            strategy=zlib.Z_HUFFMAN_ONLY)),
                    ('far', gzip.compress(far_repeats(), 9)),
                    ('stored', stored_payload()),
                    ('members3200', many_members())):
        out.append((name, _write(d / (name + '.gz'), z), gzcorpus.oracle(z)))
    return out


def bz_valid():
    return bzcorpus.valid_corpus() + bzcorpus.hand_built() + \
        [('tiny6000', tiny_streams())]


def gz_valid():
    return gzcorpus.valid_corpus()


# -- valid input, one file per scan -----------------------------------------------

@pytest.mark.parametrize('build', ['lib', 'variant'])
def test_bzip2_bytes(build, exes, bunzip_check, tmp_path):
    """every valid bzip2 file alone, under two poisons: bz2's bytes, and the
    one-lane decoder's streams, blocks and false starts at the same wave"""
    cases = bz_valid()
    paths = [_write(tmp_path / ('%s.bz2' % n), z) for n, z in cases]
    want = [bzcorpus.oracle(z) for _, z in cases]
    host = host_bunzip(bunzip_check, [z for _, z in cases], WAVE[build],
                       tmp_path)
    scans = [dict(name='%s-%02x' % (n, p), files=[('bz', f)], poison=p,
                  cap=cap_of(len(w)))
             for p in (0x00, 0xff)
             for (n, _), f, w in zip(cases, paths, want)]
    res = capture(exes[build], scans, tmp_path)
    for k, x in enumerate(res):
        i = k % len(cases)
        decoded(x, want[i])
        files, streams, blocks, fs = x['bzip2'][:4]
        assert files == 1
        assert (streams, blocks, fs) == host[i][2:], (x['name'], host[i])
    byname = {x['name']: x for x in res}
    tiny = byname['tiny6000-00']['bzip2']
    assert tiny[1] == 6000
    # 12,000 candidate magics are more than bz_find's first room (a
    # 512th of the input plus 4,096): it finds twice, then decodes,
    # inverts and emits one group per wave
    waves = -(-6000 // WAVE[build])
    assert tiny[6] == 2 + 3 * waves, tiny
    if build == 'variant':
        # 6,000 blocks span waves of 3 and emit in groups of 64 KiB
        assert len(byname['tiny6000-00']['feeds']) > 3


@pytest.mark.parametrize('build', ['lib', 'variant'])
def test_gzip_bytes(build, exes, inflate_check, gz_large, tmp_path):
    """every valid gzip file alone, under two poisons (the large ones at one
    SM, five and the device's): zlib's bytes and members, no fallback"""
    cases = [(n, _write(tmp_path / ('%s.gz' % n), z), gzcorpus.oracle(z), z)
             for n, z in gz_valid()]
    cases += [(n, p, w, open(p, 'rb').read()) for n, p, w in gz_large]
    host = host_inflate(inflate_check, [c[3] for c in cases], tmp_path)
    large = {n for n, _, _ in gz_large}
    scans, expect = [], []
    for (n, p, w, z), h in zip(cases, host):
        for poison in (0x00, 0xff):
            for sm in ((1, 5, 0) if n in large else (0,)):
                scans.append(dict(name='%s-%02x-sm%d' % (n, poison, sm),
                                  files=[('gz', p)], sm=sm, poison=poison,
                                  cap=cap_of(len(w or b''))))
                expect.append((n, w, h, len(z)))
    res = capture(exes[build], scans, tmp_path)
    for x, (n, w, h, size) in zip(res, expect):
        if n == 'nothing':
            # no gzip magic: refused at the feed, nothing decoded
            assert x['rcs'] == [EINVAL] and x['feeds'] == [], x
            assert x['gzip'][0] == 0
            continue
        decoded(x, w)
        files, members, cin, cout = x['gzip'][:4]
        assert (files, cin, cout) == (1, size, len(w)), x['name']
        assert members == h[3], (x['name'], members, h)
        assert x['split'][3] == 0, (x['name'], 'fell back', x['split'])
        if n in large:
            # split at every SM count
            assert x['split'][0] == 1, (x['name'], x['split'])
        if n == 'members3200':
            # chunks out of member slots are decoded again: more than the
            # finder, the first decode and the four checks
            assert x['split'][4] > 6, (x['name'], x['split'])


# -- batches ------------------------------------------------------------------------

def _small_gz(tmp_path):
    """the valid small gzip files, some of which miss their ISIZE hint"""
    out = []
    for n, z in gz_valid():
        if n == 'nothing':
            continue
        out.append((_write(tmp_path / ('b-%s.gz' % n), z), gzcorpus.oracle(z)))
    return out


def gz_feeds(files):
    """(lengths, realigned) of the feeds of one gzip batch of `files`
    [(compressed, decoded)]: each run of files that fill their ISIZE hint is
    one feed, each file that misses it one of its own; `realigned` counts
    the runs whose region does not start 16-byte aligned"""
    lens, realigned, at, run, start = [], 0, 0, None, 0
    for z, out in files:
        hint = 0 if len(z) < 4 else min(struct.unpack('<I', z[-4:])[0],
                                         len(z) * 1032 + 64)
        if len(out) == hint:
            if run is None:
                run, start = 0, at
            run += hint
        else:
            if run:
                lens.append(run)
                realigned += start % 16 != 0
            run = None
            if out:
                lens.append(len(out))
        at += hint
    if run:
        lens.append(run)
        realigned += start % 16 != 0
    return lens, realigned


def test_batches(exes, tmp_path):
    """many files in one scan: the oracles' bytes in feed order"""
    gz_files = _small_gz(tmp_path)
    small_feeds, realigned = gz_feeds([(open(p, 'rb').read(), w)
                                       for p, w in gz_files])
    assert realigned and len(small_feeds) > 1
    bz_files = [(_write(tmp_path / ('b-%s.bz2' % n), z), bzcorpus.oracle(z))
                for n, z in bz_valid() if len(z) < (1 << 20)]
    # every hint holds: one feed per batch
    exact = []
    for i in range(40):
        data = gzcorpus.ndjson(50 + i, 100 + i)
        exact.append((_write(tmp_path / ('e%02d.gz' % i),
                             gzip.compress(data, 1 + i % 9)), data))
    # 300 files: two batches of at most 256
    many = []
    for i in range(300):
        data = b'{"i":%d}\n' % i
        many.append((_write(tmp_path / ('m%03d.gz' % i),
                            gzip.compress(data)), data))
    # alternating formats: a flush at each change
    alt = []
    for i in range(12):
        data = gzcorpus.ndjson(20 + i, 300 + i)
        if i % 2:
            alt.append(('bz', _write(tmp_path / ('a%02d.bz2' % i),
                                     bz2.compress(data)), data))
        else:
            alt.append(('gz', _write(tmp_path / ('a%02d.gz' % i),
                                     gzip.compress(data)), data))

    def scan(name, kind, files, poison=0):
        return dict(name=name, files=[(kind, p) for p, _ in files],
                    poison=poison,
                    cap=cap_of(*(len(w) for _, w in files)))
    scans = [scan('gz-small', 'gz', gz_files, poison) for poison in (0, 255)]
    scans += [scan('bz-small', 'bz', bz_files, poison)
              for poison in (0, 255)]
    scans += [scan('exact', 'gz', exact), scan('many300', 'gz', many),
              dict(name='alternating', files=[(k, p) for k, p, _ in alt],
                   cap=cap_of(*(len(d) for _, _, d in alt)))]
    for build in ('lib', 'variant'):
        (tmp_path / build).mkdir()
        res = capture(exes[build], scans, tmp_path / build)
        for x in res[:2]:
            decoded(x, b''.join(w for _, w in gz_files))
            assert x['gzip'][0] == len(gz_files)
            # runs around the files that miss their hint, realigned
            assert [n for n, _ in x['feeds']] == small_feeds
        for x in res[2:4]:
            decoded(x, b''.join(w for _, w in bz_files))
            assert x['bzip2'][0] == len(bz_files)
        x = res[4]
        decoded(x, b''.join(w for _, w in exact))
        assert len(x['feeds']) == 1
        x = res[5]
        decoded(x, b''.join(w for _, w in many))
        assert x['gzip'][0] == 300
        assert [n for n, _ in x['feeds']] == [
            sum(len(w) for _, w in many[:256]),
            sum(len(w) for _, w in many[256:])]
        x = res[6]
        decoded(x, b''.join(d for _, _, d in alt))
        assert len(x['feeds']) == len(alt)
        assert x['gzip'][0] == x['bzip2'][0] == len(alt) // 2


# -- damage ------------------------------------------------------------------------

def _gz_magic(z):
    return len(z) >= 3 and z[:3] == b'\x1f\x8b\x08'


def _bz_magic(z):
    return len(z) >= 4 and z[:3] == b'BZh' and 0x31 <= z[3] <= 0x39


def check_damage(res, paths, cases, host, fmt):
    """each damaged case: refused at the feed without the magic, else failed
    with EIO naming the host decoder's kind and byte, or the oracle's bytes
    where it decodes"""
    magic = _gz_magic if fmt == 'gzip' else _bz_magic
    oracle = gzcorpus.oracle if fmt == 'gzip' else bzcorpus.oracle
    for x, p, (name, z), h in zip(res, paths, cases, host):
        clean(x)
        if not magic(z):
            assert x['rcs'] == [EINVAL] and x['feeds'] == [], (name, x)
            continue
        assert x['rcs'] == [0], (name, x['rcs'], x['err'])
        want = oracle(z)
        if want is not None:
            decoded(x, want)
            continue
        assert x['err_code'] == EIO, (name, x['err_code'], x['err'])
        if fmt == 'gzip':
            status, kind, bit, _ = h
            assert status == 2, (name, h)
            what = 'corrupt gzip data: ' + GZ_KINDS[kind]
        else:
            kind, bit = h[:2]
            what = BZ_KINDS[kind] if kind == BZ_TRAILING else \
                'corrupt bzip2 data: ' + BZ_KINDS[kind]
        assert x['err'] == '%s: %s (compressed byte %d)' % (p, what,
                                                              bit // 8), \
            (name, x['err'])


def test_bzip2_damage(exes, bunzip_check, tmp_path):
    cases = bzcorpus.damaged_corpus()
    paths = [_write(tmp_path / ('%s.bz2' % n), z) for n, z in cases]
    host = host_bunzip(bunzip_check, [z for _, z in cases], WAVE['lib'],
                       tmp_path)
    res = capture(exes['lib'], [dict(name=n, files=[('bz', p)], cap=1 << 20)
                                for (n, _), p in zip(cases, paths)], tmp_path)
    check_damage(res, paths, cases, host, 'bzip2')


def test_gzip_damage(exes, inflate_check, tmp_path):
    """the damaged corpus, its ~3,000 byte flips and sets sampled with a
    fixed seed; and damage to a 4 MB member on the split path"""
    cases = gzcorpus.damaged_corpus()
    rng = random.Random(7)
    cases = [c for c in cases
             if not c[0].startswith(('flip', 'set')) or rng.random() < 0.2]
    text = big_text()[:5 << 20]
    z = gzip.compress(text, 6)
    rng = random.Random(8)
    for k in range(10):
        cases.append(('split-trunc%d' % k,
                      z[:rng.randrange(len(z) // 10, len(z))]))
    for k in range(10):
        b = bytearray(z)
        b[rng.randrange(20, len(z) - 8)] ^= 1 << rng.randrange(8)
        cases.append(('split-flip%d' % k, bytes(b)))
    paths = [_write(tmp_path / ('%s.gz' % n), c) for n, c in cases]
    host = host_inflate(inflate_check, [c for _, c in cases], tmp_path)
    scans = []
    for (n, c), p in zip(cases, paths):
        for sm in ((0, 5) if n.startswith('split') else (0,)):
            scans.append(dict(name='%s-sm%d' % (n, sm), files=[('gz', p)],
                              sm=sm, cap=max(len(text), 1 << 20)))
    res = capture(exes['lib'], scans, tmp_path)
    it = iter(res)
    for (n, c), p, h in zip(cases, paths, host):
        for sm in ((0, 5) if n.startswith('split') else (0,)):
            check_damage([next(it)], [p], [(n, c)], [h], 'gzip')


# -- end to end, through the library --------------------------------------------

def e2e_lines(n=150000, seed=21):
    rng = random.Random(seed)
    alphabet = [chr(c) for c in range(32, 127) if chr(c) not in '"\\']
    out = []
    for i in range(n):
        r = rng.random()
        if r < 0.3 and out:
            body = out[rng.randrange(len(out))].split(' ', 1)[1]
        elif r < 0.6:
            body = rng.choice(alphabet) * rng.randrange(1, 301)
        else:
            body = ''.join(rng.choice(alphabet)
                           for _ in range(rng.randrange(0, 400)))
        out.append('%07d %s' % (i, body[:400]))
    return out


@pytest.mark.parametrize('kernel', ['auto', 'tile'])
def test_end_to_end(kernel, tmp_path, monkeypatch):
    """one stream of 150k lines cut at arbitrary bytes into plain, gzip and
    bzip2 pieces, fed interleaved: every line exactly once"""
    from dragnet_b200 import datasource_gpu, native
    for v in ('DNG_KERNEL', 'DNG_JIT'):
        monkeypatch.delenv(v, raising=False)
    if kernel == 'tile':
        monkeypatch.setenv('DNG_KERNEL', 'tile')
    lines = e2e_lines()
    stream = ''.join('{"l":"%s"}\n' % ln for ln in lines).encode()
    rng = random.Random(22)
    big_at = len(stream) // 4
    cuts = sorted(set(rng.sample(range(1, len(stream)), 40) +
                      [big_at, big_at + (17 << 20)]))
    cuts = [c for c in cuts if not big_at < c < big_at + (17 << 20)]
    bounds = [0] + cuts + [len(stream)]
    plain, feeds = [], []
    for k in range(len(bounds) - 1):
        piece = stream[bounds[k]:bounds[k + 1]]
        p = _write(tmp_path / ('p%02d.log' % k), piece)
        plain.append(p)
        if bounds[k] == big_at:
            kind = 'gz'
        else:
            kind = ('gz', 'bz', 'plain')[k % 3]
        if kind == 'gz':
            h = len(piece) // 2
            z = gzip.compress(piece, 1 + k % 9) if k % 2 or \
                bounds[k] == big_at else \
                gzip.compress(piece[:h]) + gzip.compress(piece[h:], 1)
            feeds.append(('gz', _write(tmp_path / ('p%02d.gz' % k), z)))
        elif kind == 'bz':
            h = len(piece) // 3
            z = bz2.compress(piece, 1 + k % 9) if k % 2 else \
                bz2.compress(piece[:h], 2) + bz2.compress(piece[h:], 7)
            feeds.append(('bz', _write(tmp_path / ('p%02d.bz2' % k), z)))
        else:
            feeds.append(('plain', p))
    plan = corpus.make_plan(['-b', 'l,'])
    p = native.Plan(json.dumps(plan))
    s = native.Scan(p)
    try:
        for kind, f in feeds:
            {'gz': s.feed_gzip, 'bz': s.feed_bzip2,
             'plain': s.feed_file}[kind](f)
        res = s.finish()
        pts = res.points()
        res.close()
        flat = s.counters()
        gst = s.gzip_split_stats()
    finally:
        s.close()
        p.close()
    assert gst['gzip_split_files'] >= 1 and gst['gzip_fallbacks'] == 0
    got = sorted((c[0], v) for c, v in pts)
    assert got == sorted((ln.encode(), 1) for ln in lines)
    assert flat['bytes'] == len(stream)
    _, exp_c = cpp_engine(plan, plain)
    assert datasource_gpu.stage_counters(plan, flat, len(pts)) == exp_c
