"""The gzip decoder (dragnet_b200/csrc/inflate.cuh) built for the host, one
lane per file (tests/hostcheck/inflate_check.cpp), against Python's
gzip.decompress: for every input it must fail exactly when that fails, and
return the same bytes otherwise.  The damaged corpus also runs under
AddressSanitizer and UBSan, so no malformed input reads out of bounds."""

import os
import struct
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gzcorpus  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')
DRIVER = os.path.join(ROOT, 'tests', 'hostcheck', 'inflate_check.cpp')

DONE, ROOM, ERROR = 0, 1, 2


def _build(tmp_path_factory, name, flags):
    exe = str(tmp_path_factory.mktemp(name) / 'inflate_check')
    subprocess.check_call(['g++', '-std=c++17', '-Wall', '-Wextra', '-Werror',
                           '-I', CSRC] + flags + ['-o', exe, DRIVER])
    return exe


@pytest.fixture(scope='module')
def check(tmp_path_factory):
    return _build(tmp_path_factory, 'inflate', ['-O2'])


@pytest.fixture(scope='module')
def check_asan(tmp_path_factory):
    return _build(tmp_path_factory, 'inflate_asan',
                  ['-O1', '-g', '-fsanitize=address,undefined',
                   '-fno-sanitize-recover=all', '-fno-omit-frame-pointer'])


def run(exe, cases, tmp_path):
    """[(status, kind, bit, members, redecodes, bytes)] per case"""
    src, dst = tmp_path / 'in.bin', tmp_path / 'out.bin'
    src.write_bytes(struct.pack('<I', len(cases)) + b''.join(
        struct.pack('<Q', len(c)) + c for c in cases))
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True,
                       env=dict(os.environ, ASAN_OPTIONS='detect_leaks=0'))
    assert r.returncode == 0 and not r.stderr, r.stderr.decode()[-3000:]
    out, raw, off = [], dst.read_bytes(), 0
    for _ in cases:
        status, kind, bit, members, redo, n = struct.unpack_from(
            '<IIQIIQ', raw, off)
        off += 32
        out.append((status, kind, bit, members, redo, raw[off:off + n]))
        off += n
    assert off == len(raw)
    return out


def agree(cases, results):
    bad = []
    for (name, data), (status, kind, bit, _, _, got) in zip(cases, results):
        want = gzcorpus.oracle(data)
        assert status != ROOM, name
        if want is None:
            if status != ERROR:
                bad.append('%s: decoded, gzip fails' % name)
            elif bit > 8 * len(data):
                bad.append('%s: error bit %d past the input' % (name, bit))
        elif status != DONE:
            bad.append('%s: error kind %d at bit %d, gzip decodes' %
                       (name, kind, bit))
        elif got != want:
            bad.append('%s: %d bytes differ from gzip\'s %d' %
                       (name, len(got), len(want)))
    assert not bad, bad[:20]


def test_valid_corpus(check, tmp_path):
    cases = gzcorpus.valid_corpus()
    res = run(check, [c for _, c in cases], tmp_path)
    agree(cases, res)
    byname = {n: r for (n, _), r in zip(cases, res)}
    # several members: ISIZE names the last one only, so the output is
    # decoded again in more room
    assert byname['members'][3] == 3 and byname['members'][4] > 0
    assert byname['members-zeros'][3] == 2
    assert byname['nothing'][3] == 0
    for name in ('level6', 'ndjson', 'wbits9', 'dist32768-len258'):
        assert byname[name][4] == 0, name


def test_damaged_corpus(check, tmp_path):
    cases = gzcorpus.damaged_corpus()
    agree(cases, run(check, [c for _, c in cases], tmp_path))


def test_error_kinds(check, tmp_path):
    """The kind of damage each hand-built input reports."""
    cases = dict(gzcorpus.damaged_corpus())
    kinds = {'bad-crc': 8, 'bad-isize': 9, 'bad-magic': 1, 'bad-method': 1,
             'trailing-garbage': 1, 'btype3': 3, 'lit286': 6, 'dist30': 6,
             'too-far': 7, 'too-far-first': 7, 'dyn-over': 5,
             'dyn-incomplete': 5, 'dyn-too-many': 5, 'dyn-no-eob': 5,
             'trunc30': 2}
    names = sorted(kinds)
    res = run(check, [cases[n] for n in names], tmp_path)
    got = {n: r[1] for n, r in zip(names, res)}
    assert got == kinds


def test_damaged_corpus_sanitized(check_asan, tmp_path):
    cases = gzcorpus.damaged_corpus(seed=3) + [
        (n, c) for n, c in gzcorpus.valid_corpus()
        if n in ('members', 'dist32768-len258', 'stored65535', 'flags31')]
    agree(cases, run(check_asan, [c for _, c in cases], tmp_path))
