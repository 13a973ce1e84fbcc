"""The F path's short group key (dragnet_b200/csrc/fast.cuh FKey) on the host:
a key of at most four columns whose discrete pieces are at most 8 bytes is
packed into registers, hashed, compared and stored as words, and unpacked into
record.cuh's encoding when the F kernel flushes its tally cache.  A host build
(tests/hostcheck/fkey_check.cpp) must unpack every short key to fkey_write's
bytes, take the short form exactly for the keys that fit, give equal keys one
short form, and tally what the Python oracle tallies."""

import json
import os
import struct
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import canon_points, py_engine  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')
DRIVER = os.path.join(ROOT, 'tests', 'hostcheck', 'fkey_check.cpp')
W = 8           # fast.cuh FK_W
COLS = 4        # fast.cuh FK_COLS


def _build(tmp_path_factory, name, flags):
    exe = str(tmp_path_factory.mktemp(name) / 'fkey_check')
    subprocess.check_call(
        ['g++', '-std=c++17', '-w', '-I', CSRC] + flags +
        ['-o', exe, DRIVER] +
        [os.path.join(CSRC, n) for n in ('plan.cpp', 'result.cpp', 'tmpl.cpp',
                                         'fast.cpp')])
    return exe


@pytest.fixture(scope='module')
def check(tmp_path_factory):
    return _build(tmp_path_factory, 'fkey', ['-O1'])


@pytest.fixture(scope='module')
def check_asan(tmp_path_factory):
    return _build(tmp_path_factory, 'fkey_asan',
                  ['-O1', '-g', '-fsanitize=address,undefined',
                   '-fno-sanitize-recover=all', '-fno-omit-frame-pointer'])


# values of every form the F path keys on, as JSON text, and String(value)
# (None: undefined, the field is absent)
def _values():
    out = []
    for n in range(W + 2):              # strings of 0..W+1 bytes
        s = ''.join(chr(ord('a') + (i + n) % 26) for i in range(n))
        out.append((json.dumps(s), s))
    for v in ('0', '-1', '7', '12345678', '-1234567', '123456789'):
        out.append((v, v))              # simple integers, up to W+1 digits
    for v in ('null', 'true', 'false'):
        out.append((v, v))
    out.append(('"null"', 'null'))      # one group with null
    out.append((None, 'undefined'))     # 9 bytes: never a short key
    return out


VALUES = _values()
ORDS = ['0', '-0', '3', '-7', '1e308', '-1e308', '"NaN"', '"x"', 'null',
        '"Infinity"', '"-Infinity"', '1.5']


def _corpus(ncols, bucket_col=None):
    """Every value in every column position (the other columns cycling), and
    ordinals when bucket_col is set."""
    lines = []
    nv = len(VALUES)
    for pos in range(ncols):
        for i in range(nv):
            for shift in (0, 3):
                parts = []
                for c in range(ncols):
                    if c == bucket_col:
                        txt = ORDS[(i + shift + c) % len(ORDS)]
                    else:
                        txt = VALUES[i if c == pos else
                                     (i + shift + 5 * c) % nv][0]
                    if txt is not None:
                        parts.append('"c%d":%s' % (c, txt))
                lines.append('{' + ','.join(parts) + '}')
    return ('\n'.join(lines) + '\n').encode()


def _plan(ncols, bucket_col=None):
    cols = ','.join('c%d' % c + ('[aggr=lquantize,step=10]'
                                 if c == bucket_col else '')
                    for c in range(ncols))
    return corpus.make_plan(['-b', cols])


def _decode(plan, key):
    fields, o = [], 0
    for b in plan['breakdowns']:
        n = key[o] | key[o + 1] << 8
        if n == 0xffff:
            # (the ordinal of lquantize, step=10: its bucket is 10 x it)
            fields.append((b['name'], 10 * struct.unpack(
                '<d', key[o + 2:o + 10])[0]))
            o += 10
        else:
            fields.append((b['name'], bytes(key[o + 2:o + 2 + n])))
            o += 2 + n
    assert o == len(key)
    return fields


def _fits(plan, key):
    if len(plan['breakdowns']) > COLS:
        return False
    o = 0
    for _ in plan['breakdowns']:
        n = key[o] | key[o + 1] << 8
        if n == 0xffff:
            o += 10
            continue
        if n > W:
            return False
        o += 2 + n
    return True


def _run(exe, plan, data, tmp_path):
    pf, df = tmp_path / 'plan.json', tmp_path / 'data.log'
    pf.write_text(json.dumps(plan))
    df.write_bytes(data)
    r = subprocess.run([exe, str(pf), str(df)], capture_output=True,
                       env=dict(os.environ, ASAN_OPTIONS='detect_leaks=0'))
    assert r.returncode == 0 and not r.stderr, r.stderr.decode()[-3000:]
    return r.stdout.decode().splitlines(), str(df)


CASES = [(n, None) for n in range(1, COLS + 2)] + [(3, 1), (1, 0), (4, 3)]


def _check(exe, ncols, bucket_col, tmp_path):
    plan = _plan(ncols, bucket_col)
    data = _corpus(ncols, bucket_col)
    out, df = _run(exe, plan, data, tmp_path)
    assert len(out) == data.count(b'\n')
    tally, short_of, nshort, nlong = {}, {}, 0, 0
    # (records of shapes beyond the templates' room go to the general code)
    taken = [r for r, line in zip(data.splitlines(True), out) if line != 'M']
    assert len(taken) * 2 > len(out)
    for line in out:
        f = line.split()
        assert f[0] in 'PLM', line
        if f[0] == 'M':
            continue
        key = bytes.fromhex(f[-1]) if len(f) > 1 else b''
        # the short form exactly for the keys that fit
        assert (f[0] == 'P') == _fits(plan, key), line
        if f[0] == 'P':
            nshort += 1
            # one short form (header and hash) per key, one key per form
            form = (f[1], f[2])
            assert short_of.setdefault(key, form) == form, line
        else:
            nlong += 1
        tally[key] = tally.get(key, 0) + 1
    forms = list(short_of.values())
    assert len(set(forms)) == len(forms)
    # (9-byte strings and undefined in every discrete column: long keys)
    assert (nshort > 0) == (ncols <= COLS)
    assert (nlong > 0) == (bucket_col is None or ncols > 1)
    points = [(_decode(plan, k), v) for k, v in tally.items()]
    with open(df, 'wb') as f:
        f.write(b''.join(taken))
    exp, _ = py_engine(plan, [df])
    assert canon_points(points) == canon_points(exp)


@pytest.mark.parametrize('ncols,bucket_col', CASES)
def test_short_keys_unpack_to_the_encoding_and_match_the_oracle(
        check, ncols, bucket_col, tmp_path):
    _check(check, ncols, bucket_col, tmp_path)


@pytest.mark.parametrize('ncols,bucket_col', [(2, None), (4, 3), (5, None)])
def test_short_keys_under_sanitizers(check_asan, ncols, bucket_col, tmp_path):
    _check(check_asan, ncols, bucket_col, tmp_path)


def test_null_and_the_string_null_are_one_short_key(check, tmp_path):
    plan = _plan(2)
    data = b'{"c0":null,"c1":1}\n{"c0":"null","c1":1}\n'
    out, _ = _run(check, plan, data, tmp_path)
    assert len(out) == 2 and out[0] == out[1] and out[0].startswith('P '), out
