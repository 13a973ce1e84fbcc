"""The split gzip decoder (dragnet_b200/csrc/inflate_split.cuh) built for the
host and run as one lane through every stage the library runs
(tests/hostcheck/inflate_split_check.cpp), at chunk sizes far below the
library's floor so that small inputs are cut into many chunks: it must give
gzip.decompress's bytes without falling back on every valid input, and
exactly the one-lane decoder's answer on every damaged one.  Also the
finder's guarantee that it never passes a true dynamic-block start, and the
split policy (inflate_policy.h)."""

import gzip
import os
import random
import struct
import subprocess
import sys
import zlib

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gzcorpus  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')
HOSTCHECK = os.path.join(ROOT, 'tests', 'hostcheck')

DONE, ROOM, ERROR = 0, 1, 2
NOSTART = (1 << 64) - 1
KIB = 1024


def _build(tmp_path_factory, name, src, flags):
    exe = str(tmp_path_factory.mktemp(name) / name)
    subprocess.check_call(['g++', '-std=c++17', '-Wall', '-Wextra', '-Werror',
                           '-I', CSRC] + flags +
                          ['-o', exe, os.path.join(HOSTCHECK, src)])
    return exe


ASAN = ['-O1', '-g', '-fsanitize=address,undefined',
        '-fno-sanitize-recover=all', '-fno-omit-frame-pointer']


@pytest.fixture(scope='module')
def split(tmp_path_factory):
    return _build(tmp_path_factory, 'inflate_split_check',
                  'inflate_split_check.cpp', ['-O2'])


@pytest.fixture(scope='module')
def split_asan(tmp_path_factory):
    return _build(tmp_path_factory, 'inflate_split_check',
                  'inflate_split_check.cpp', ASAN)


@pytest.fixture(scope='module')
def whole(tmp_path_factory):
    return _build(tmp_path_factory, 'inflate_check', 'inflate_check.cpp',
                  ['-O2'])


def _write_cases(path, cases):
    path.write_bytes(struct.pack('<I', len(cases)) + b''.join(
        struct.pack('<Q', len(c)) + c for c in cases))


def run_split(exe, cases, chunk, tmp_path):
    """per case: dict(status, kind, bit, members, fallbacks, chunks,
    false_starts, passes, data, cuts=[(first bit, candidate)], starts)"""
    src, dst = tmp_path / 'in.bin', tmp_path / 'out.bin'
    _write_cases(src, cases)
    r = subprocess.run([exe, str(chunk), str(src), str(dst)],
                       capture_output=True,
                       env=dict(os.environ, ASAN_OPTIONS='detect_leaks=0'))
    assert r.returncode == 0 and not r.stderr, r.stderr.decode()[-3000:]
    out, raw, off = [], dst.read_bytes(), 0
    for _ in cases:
        v = struct.unpack_from('<IIQIIIIIQ', raw, off)
        off += 44
        d = dict(zip(('status', 'kind', 'bit', 'members', 'fallbacks',
                      'chunks', 'false_starts', 'passes'), v[:8]))
        d['data'] = raw[off:off + v[8]]
        off += v[8]
        (n,) = struct.unpack_from('<I', raw, off)
        off += 4
        cuts = struct.unpack_from('<%dQ' % (2 * n), raw, off)
        off += 16 * n
        d['cuts'] = list(zip(cuts[0::2], cuts[1::2]))
        (ns,) = struct.unpack_from('<I', raw, off)
        off += 4
        d['starts'] = list(struct.unpack_from('<%dQ' % ns, raw, off))
        off += 8 * ns
        out.append(d)
    assert off == len(raw)
    return out


def run_whole(exe, cases, tmp_path):
    """per case: (status, kind, bit, members) of the one-lane decoder"""
    src, dst = tmp_path / 'win.bin', tmp_path / 'wout.bin'
    _write_cases(src, cases)
    subprocess.check_call([exe, str(src), str(dst)])
    out, raw, off = [], dst.read_bytes(), 0
    for _ in cases:
        status, kind, bit, members, _, n = struct.unpack_from(
            '<IIQIIQ', raw, off)
        off += 32 + n
        out.append((status, kind, bit, members))
    return out


def check_finder(name, d, size):
    """each chunk's candidate is at or before the first true dynamic-block
    start at or after its first bit, and within the chunk"""
    cuts = d['cuts']
    for k in range(1, len(cuts)):
        lo, cand = cuts[k]
        hi = cuts[k + 1][0] if k + 1 < len(cuts) else 8 * size
        true = [b for b in d['starts'] if b >= lo]
        first = true[0] if true else None
        if cand == NOSTART:
            assert first is None or first >= hi, (name, k, lo, first)
        else:
            assert lo <= cand < hi, (name, k)
            assert first is None or cand <= first, (name, k, cand, first)


def check_valid(cases, res, want_members):
    for (name, data), d, m in zip(cases, res, want_members):
        assert d['status'] == DONE, (name, d['kind'], d['bit'])
        assert d['data'] == gzip.decompress(data), name
        assert d['fallbacks'] == 0, name
        assert d['members'] == m, name
        check_finder(name, d, len(data))


# -- hand-built inputs -----------------------------------------------------------

def stored_payload():
    """one member: dynamic blocks, then stored blocks whose bytes are raw
    deflate streams (full of parseable block headers that are not block
    starts of this stream), then dynamic blocks again"""
    text = gzcorpus.ndjson(6000, 11)
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    a = c.compress(text[:300000]) + c.flush(zlib.Z_FULL_FLUSH)
    payload = b''.join(gzcorpus.raw_deflate(gzcorpus.ndjson(800, s), lvl)
                       for s, lvl in ((21, 9), (22, 6), (23, 1), (24, 9)))
    mid = gzcorpus.stored(payload, final=False)
    z = text[300000:]
    tail = gzcorpus.raw_deflate(z, 6)
    data = text[:300000] + payload + z
    return gzcorpus.member(a + mid + tail, data)


def far_repeats():
    """a random block repeated at a period just inside zlib's reach, so that
    every chunk's matches reach back across its start"""
    rng = random.Random(5)
    block = bytes(rng.randrange(256) for _ in range(32500))
    data = bytearray(block * 24)
    for i in range(0, len(data), 4099):
        data[i] ^= 0x5a
    return gzcorpus.gz(bytes(data), 9)


def swing():
    """compressibility that swings about 1000x between halves"""
    text = gzcorpus.ndjson(2000, 12)
    return gzcorpus.gz(text + b'\x00' * (4 << 20) + text, 6)


def hand_built():
    text = gzcorpus.ndjson(8000, 13)
    m1, m2 = gzcorpus.gz(text[:900000], 6), gzcorpus.gz(text[900000:], 1)
    return [
        ('stored-payload', stored_payload()),
        ('far-repeats', far_repeats()),
        ('fixed', gzcorpus.gz(text, 6, strategy=zlib.Z_FIXED)),
        ('huffman-only', gzcorpus.gz(text, 6, strategy=zlib.Z_HUFFMAN_ONLY)),
        ('level0', gzcorpus.gz(text[:500000], 0)),
        ('members-zeros', m1 + m2 + gzcorpus.gz(b'') + b'\x00' * 40),
        ('members-zeros-between', m1 + b'\x00' * 9 + m2 + b'\x00' * 3),
        ('swing', swing()),
    ]


@pytest.fixture(scope='module')
def hand(whole, tmp_path_factory):
    cases = hand_built()
    members = [w[3] for w in run_whole(whole, [c for _, c in cases],
                                       tmp_path_factory.mktemp('hm'))]
    return cases, members


# -- tests -------------------------------------------------------------------------

@pytest.mark.parametrize('chunk', [1 * KIB, 4 * KIB, 33 * KIB, 64 * KIB])
def test_valid_corpus(split, whole, chunk, tmp_path):
    cases = gzcorpus.valid_corpus()
    blobs = [c for _, c in cases]
    members = [w[3] for w in run_whole(whole, blobs, tmp_path)]
    res = run_split(split, blobs, chunk, tmp_path)
    check_valid(cases, res, members)
    # the corpus is cut into many chunks at the small sizes
    if chunk == 1 * KIB:
        byname = {n: d for (n, _), d in zip(cases, res)}
        assert byname['ndjson']['chunks'] > 100


@pytest.mark.parametrize('chunk', [4 * KIB, 33 * KIB])
def test_hand_built(split, hand, chunk, tmp_path):
    cases, members = hand
    res = run_split(split, [c for _, c in cases], chunk, tmp_path)
    check_valid(cases, res, members)
    byname = {n: d for (n, _), d in zip(cases, res)}
    # the stored deflate streams hold candidates nothing lands on
    assert byname['stored-payload']['false_starts'] > 0
    # Z_FIXED writes no dynamic block: nothing to cut at
    assert all(c == NOSTART for _, c in byname['fixed']['cuts'][1:])
    # the output estimate is far off for the zeros: decoded again in more
    # room, without falling back
    assert byname['swing']['passes'] > 0
    assert byname['members-zeros']['members'] == 3
    for name in ('far-repeats', 'huffman-only', 'swing', 'members-zeros'):
        d = byname[name]
        assert d['false_starts'] < d['chunks'], name
        assert d['chunks'] >= 2 or chunk > 4 * KIB, name


def _damaged_agree(split_exe, whole_exe, cases, chunk, tmp_path):
    blobs = [c for _, c in cases]
    res = run_split(split_exe, blobs, chunk, tmp_path)
    ref = run_whole(whole_exe, blobs, tmp_path)
    bad = []
    for (name, data), d, w in zip(cases, res, ref):
        if (d['status'], d['kind'], d['bit']) != w[:3]:
            bad.append((name, (d['status'], d['kind'], d['bit']), w[:3]))
        elif d['status'] == DONE and d['data'] != gzcorpus.oracle(data):
            bad.append((name, 'bytes'))
        if d['status'] == DONE and gzcorpus.oracle(data) is None:
            bad.append((name, 'split decoded what gzip refuses'))
    assert not bad, bad[:20]
    return res


@pytest.mark.parametrize('chunk', [256, 1 * KIB])
def test_damaged_corpus(split, whole, chunk, tmp_path):
    _damaged_agree(split, whole, gzcorpus.damaged_corpus(), chunk, tmp_path)


def test_damaged_large(split, whole, tmp_path):
    """truncations and flips in the first, a middle and the last chunk of a
    file cut into many chunks, in its CRC and in its ISIZE"""
    z = gzcorpus.gz(gzcorpus.ndjson(3000, 17), 6)
    rng = random.Random(8)
    cases = [('trunc%d' % i, z[:i]) for i in (len(z) // 3, len(z) - 9,
                                                len(z) - 1)]
    for where in (40, len(z) // 2, len(z) - 400, len(z) - 8, len(z) - 3):
        for _ in range(4):
            b = bytearray(z)
            b[where + rng.randrange(16) if where < len(z) - 20 else where] \
                ^= 1 << rng.randrange(8)
            cases.append(('flip%d' % where, bytes(b)))
    res = _damaged_agree(split, whole, cases, 1 * KIB, tmp_path)
    assert all(d['chunks'] > 10 for d in res)


def test_sanitized(split_asan, whole, hand, tmp_path):
    cases = gzcorpus.damaged_corpus(seed=3)
    _damaged_agree(split_asan, whole, cases, 512, tmp_path)
    hcases, members = hand
    keep = [i for i, (n, _) in enumerate(hcases) if n != 'swing']
    res = run_split(split_asan, [hcases[i][1] for i in keep], 8 * KIB,
                    tmp_path)
    check_valid([hcases[i] for i in keep], res, [members[i] for i in keep])


# -- the policy ----------------------------------------------------------------------

def policy(split, floor, resident, sizes):
    r = subprocess.run([split, 'policy', str(floor), str(resident)] +
                       [str(s) for s in sizes], capture_output=True,
                       text=True, check=True)
    return [int(x) for x in r.stdout.split()]


FLOOR = 64 * KIB


def test_policy(split):
    # all small files: nothing is split
    assert policy(split, FLOOR, 2000, [1000] * 50 + [FLOOR]) == [1] * 51
    # one file: cut to the resident warps, never below the floor
    assert policy(split, FLOOR, 2000, [2000 * FLOOR * 3]) == [2000]
    assert policy(split, FLOOR, 2000, [100 * FLOOR]) == [100]
    assert policy(split, FLOOR, 2000, [100 * FLOOR + FLOOR - 1]) == [100]
    # just under and just over twice the floor
    assert policy(split, FLOOR, 2000, [2 * FLOOR - 1]) == [1]
    assert policy(split, FLOOR, 2000, [2 * FLOOR]) == [2]
    assert policy(split, FLOOR, 2000, [2 * FLOOR + 1]) == [2]
    # as many files as resident warps, or more: nothing is split
    assert policy(split, FLOOR, 4, [10 * FLOOR] * 4) == [1] * 4
    assert policy(split, FLOOR, 4, [10 * FLOOR] * 5) == [1] * 5
    assert policy(split, FLOOR, 5, [10 * FLOOR] * 4) == [2] * 4
    # zero-byte files, beside one that is split
    assert policy(split, FLOOR, 100, [0, 0, 40 * FLOOR, 0]) == [1, 1, 40, 1]
    assert policy(split, FLOOR, 100, [0, 0]) == [1, 1]
    # the largest files are cut until no work item exceeds the target
    sizes = [400 * FLOOR, 50 * FLOOR, 3 * FLOOR, 1000]
    got = policy(split, FLOOR, 100, sizes)
    target = max(FLOOR, sum(sizes) // 100)
    assert got[3] == 1
    for s, c in zip(sizes, got):
        assert c == 1 or (s // c >= FLOOR and -(-s // c) <= target + 1)
        assert c > 1 or s <= target or s < 2 * FLOOR
