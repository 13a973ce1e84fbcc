"""The F kernel's short group keys (dragnet_b200/csrc/fast.cuh FKey) on the
GPU: keys of at most four columns whose discrete pieces are at most 8 bytes are
tallied from registers in the CTA's inline tier and unpacked into record.cuh's
encoding when the kernel flushes it.  Every scan is compared, points and
counters, with the C++ oracle, under the library's own kernel choice, the F
kernel forced on, and the F kernel with its compiled matcher."""

import os
import random
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import cpp_engine  # noqa: E402
from test_fkey_short_host import _corpus as short_corpus, _plan  # noqa: E402
from dragnet_b200 import datasource_gpu  # noqa: E402

pytestmark = pytest.mark.gpu

M32 = 0xffffffff


@pytest.fixture(params=['auto', 'fast', 'jit'])
def mode(request, monkeypatch):
    for v in ('DNG_KERNEL', 'DNG_JIT', 'DNG_F_WARPS'):
        monkeypatch.delenv(v, raising=False)
    if request.param == 'fast':
        monkeypatch.setenv('DNG_KERNEL', 'fast')
        monkeypatch.setenv('DNG_JIT', '0')
    elif request.param == 'jit':
        monkeypatch.setenv('DNG_KERNEL', 'fast')
        monkeypatch.setenv('DNG_JIT', 'sync')
    return request.param


# fast.cuh fmix / fkey_short_hash, restated
def fmix(h, w):
    h = ((h ^ w) * 0x9E3779B1) & M32
    return h ^ (h >> 15)


def _unfmix(h, out):
    """the w with fmix(h, w) == out"""
    x = out ^ (out >> 15)
    x ^= x >> 30
    x = (x * pow(0x9E3779B1, -1, 1 << 32)) & M32
    return x ^ h


def _pre(key):
    """fkey_short_hash of a one-column discrete key up to its last word"""
    b = key.ljust(8, b'\0')
    h = fmix(0x2545F491, 0x80000000 | 1 << 16 | len(key))
    return fmix(h, int.from_bytes(b[:4], 'little')), \
        int.from_bytes(b[4:], 'little')


def short_hash(key):
    h, hi = _pre(key)
    h = fmix(h, hi)
    h ^= h >> 16
    h = (h * 0x85ebca6b) & M32
    return h ^ (h >> 13)


def _unfinal(h):
    """the chain value whose finaliser gives h"""
    h ^= h >> 13
    h ^= h >> 26
    h = (h * pow(0x85ebca6b, -1, 1 << 32)) & M32
    return h ^ (h >> 16)


OK = bytes(c for c in range(0x21, 0x7f) if c not in b'"\\')


def full_collisions(count, seed):
    """count 8-byte keys with one short hash: the last word solved for"""
    rnd = random.Random(seed)
    target = _unfinal(rnd.getrandbits(32))
    out = set()
    while len(out) < count:
        lo = bytes(rnd.choice(OK) for _ in range(4))
        h, _ = _pre(lo + b'aaaa')
        hi = _unfmix(h, target).to_bytes(4, 'little')
        if all(c in OK for c in hi):
            out.add(lo + hi)
    keys = sorted(out)
    assert len({short_hash(k) for k in keys}) == 1
    return keys


def index_collisions(count, seed):
    """count keys of 1..8 bytes whose short hashes share bits 7..16: one
    tier-1 slot for every table of up to 1024 slots"""
    rnd = random.Random(seed)
    want, out = None, set()
    while len(out) < count:
        k = bytes(rnd.choice(OK) for _ in range(rnd.randint(1, 8)))
        b = (short_hash(k) >> 7) & 1023
        if want is None:
            want = b
        if b == want:
            out.add(k)
    return sorted(out)


def _write(tmp_path, name, lines):
    p = str(tmp_path / (name + '.log'))
    with open(p, 'wb') as f:
        f.write(b'\n'.join(lines) + b'\n')
    return p


def check(plan, path):
    exp_p, exp_c = cpp_engine(plan, [path], threads=8)
    r = datasource_gpu.run_plan(plan, files=[path])

    def canon(pts):
        return sorted((tuple(('nan',) if v != v else v for _, v in f), c)
                      for f, c in pts)
    assert canon(r.points) == canon(exp_p)
    assert r.counters == exp_c
    return r


def _ran_f(r, mode):
    if mode != 'auto':
        assert r.stats['kernel'] == 'F path', r.stats
    if mode == 'jit':
        assert r.stats['jit']['state'] == 1, r.stats


@pytest.mark.parametrize('ncols,bucket_col', [(1, None), (2, None),
                                              (4, None), (5, None), (4, 3)])
def test_short_key_corpus(mode, ncols, bucket_col, tmp_path):
    """the host test's corpus (piece lengths 0..9 in every position, integers,
    null / true / false / undefined, ordinals with NaN, +-Infinity, -0),
    repeated so that every CTA meets its keys many times"""
    lines = short_corpus(ncols, bucket_col).splitlines() * 300
    random.Random(ncols).shuffle(lines)
    r = check(_plan(ncols, bucket_col), _write(tmp_path, 'short', lines))
    # (the wider corpora have more record shapes than the F templates hold:
    # the library scans them on the general kernels, even when asked for F)
    if ncols <= 2:
        _ran_f(r, mode)


def test_colliding_short_keys(mode, tmp_path):
    """40 keys with one short hash and 40 with one tier-1 slot, interleaved:
    equality is decided on the words alone, and probe chains run out (the
    keys that find no room take the general path and are counted as inline
    overflow)"""
    keys = full_collisions(40, 1) + index_collisions(40, 2)
    lines = [b'{"key":"%s","n":%d}' % (k, i) for i in range(60)
             for k in keys]
    r = check(corpus.make_plan(['-b', 'key']), _write(tmp_path, 'coll', lines))
    _ran_f(r, mode)
    if mode != 'auto':
        assert r.stats['inline_overflow'] > 0, r.stats


def test_keys_on_both_sides_of_the_width(mode, tmp_path):
    """8- and 9-byte values with one prefix, and keys that differ only past
    the 8th byte, in every window: short and long keys in one CTA"""
    vals = [b'abcdefgh', b'abcdefghi', b'abcdefghj', b'abcdefg', b'',
            b'12345678', b'123456789']
    lines = []
    for i in range(40000):
        v = vals[i % len(vals)]
        lines.append(b'{"key":"%s","tag":"%s"}' % (v, vals[(i // 7) % 3]))
    r = check(corpus.make_plan(['-b', 'key,tag']),
              _write(tmp_path, 'width', lines))
    _ran_f(r, mode)
