"""The bzip2 decoder (dragnet_b200/csrc/bunzip.cuh) built for the host with
every stage one lane (tests/hostcheck/bunzip_check.cpp), against Python's
bz2 module stream by stream, with zero bytes and nothing else allowed after
the last stream (bzcorpus.oracle): for every input it must fail exactly when
that fails, and return the same bytes otherwise.  Waves are kept small so
that files span them.  The damaged corpus also runs under AddressSanitizer
and UBSan, so no malformed input reads out of bounds.  Also: the
randomisation table, the wave policy, and the datasource's bzip2 key."""

import os
import re
import struct
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import bzcorpus  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')
DRIVER = os.path.join(ROOT, 'tests', 'hostcheck', 'bunzip_check.cpp')

(NONE, STREAM_HEADER, BLOCK_HEADER, TABLES, CODE, OVERFLOW, BLOCK_CRC,
 STREAM_CRC, TRUNCATED, TRAILING) = range(10)


def _build(tmp_path_factory, name, src, flags):
    exe = str(tmp_path_factory.mktemp(name) / name)
    subprocess.check_call(['g++', '-std=c++17', '-Wall', '-Wextra', '-Werror',
                           '-I', CSRC] + flags + ['-o', exe, src])
    return exe


@pytest.fixture(scope='module')
def check(tmp_path_factory):
    return _build(tmp_path_factory, 'bunzip_check', DRIVER, ['-O2'])


@pytest.fixture(scope='module')
def check_asan(tmp_path_factory):
    return _build(tmp_path_factory, 'bunzip_asan', DRIVER,
                  ['-O1', '-g', '-fsanitize=address,undefined',
                   '-fno-sanitize-recover=all', '-fno-omit-frame-pointer'])


def run(exe, cases, tmp_path, wave=3):
    """[(kind, bit, streams, blocks, false_starts, bytes)] per case; cases
    are bytes or (bytes, extra candidate bits)"""
    cases = [c if isinstance(c, tuple) else (c, []) for c in cases]
    src, dst = tmp_path / 'in.bin', tmp_path / 'out.bin'
    src.write_bytes(bzcorpus.pack_cases(cases))
    r = subprocess.run([exe, str(src), str(dst), str(wave)],
                       capture_output=True,
                       env=dict(os.environ, ASAN_OPTIONS='detect_leaks=0'))
    assert r.returncode == 0 and not r.stderr, r.stderr.decode()[-3000:]
    out, raw, off = [], dst.read_bytes(), 0
    for _ in cases:
        kind, bit, st, bl, fs, n = struct.unpack_from('<IQIIIQ', raw, off)
        off += 32
        out.append((kind, bit, st, bl, fs, raw[off:off + n]))
        off += n
    assert off == len(raw)
    return out


def agree(cases, results):
    bad = []
    for (name, data), (kind, bit, _, _, _, got) in zip(cases, results):
        want = bzcorpus.oracle(data)
        if want is None:
            if kind == NONE:
                bad.append('%s: decoded, bz2 fails' % name)
            elif bit > 8 * len(data):
                bad.append('%s: error bit %d past the input' % (name, bit))
        elif kind != NONE:
            bad.append('%s: error kind %d at bit %d, bz2 decodes' %
                       (name, kind, bit))
        elif got != want:
            bad.append('%s: %d bytes differ from bz2\'s %d' %
                       (name, len(got), len(want)))
    assert not bad, bad[:20]


def test_valid_corpus(check, tmp_path):
    cases = bzcorpus.valid_corpus()
    res = run(check, [c for _, c in cases], tmp_path)
    agree(cases, res)
    byname = {n: r for (n, _), r in zip(cases, res)}
    assert byname['empty'][2:4] == (1, 0)
    assert byname['multi-levels'][2] == 4
    assert byname['lines'][3] >= 2
    assert all(r[4] == 0 for r in res)


def test_hand_built(check, tmp_path):
    cases = bzcorpus.hand_built()
    res = run(check, [c for _, c in cases], tmp_path)
    agree(cases, res)
    byname = {n: r for (n, _), r in zip(cases, res)}
    assert byname['false-start'][4] >= 1
    for name, r in byname.items():
        if name != 'false-start':
            assert r[4] == 0, name
        assert r[3] == 1, name


def test_wave_sizes(check, tmp_path):
    """One wave per candidate, and one wave for all: the same bytes."""
    cases = [c for c in bzcorpus.valid_corpus()
             if c[0] in ('multi-levels', 'lines', 'level1')]
    for wave in (1, 2, 1000):
        agree(cases, run(check, [c for _, c in cases], tmp_path, wave))


def test_extra_candidates(check, tmp_path):
    """Block candidates at arbitrary bits are decoded beside the true ones
    and dropped by the chain: the output never changes."""
    import random
    rnd = random.Random(11)
    cases = [c for c in bzcorpus.valid_corpus()
             if c[0] in ('multi-levels', 'lines', 'run260')]
    cases += [c for c in bzcorpus.hand_built()
              if c[0] in ('randomised', 'groups6')]
    runs = []
    for _, data in cases:
        extra = sorted(rnd.sample(range(8 * len(data)), 40))
        runs.append((data, extra))
    res = run(check, runs, tmp_path)
    agree(cases, res)
    assert all(r[4] >= 30 for r in res)


def test_damaged_corpus(check, tmp_path):
    cases = bzcorpus.damaged_corpus()
    agree(cases, run(check, [c for _, c in cases], tmp_path))


def test_error_kinds(check, tmp_path):
    """The kind of damage each hand-picked input reports."""
    cases = dict(bzcorpus.damaged_corpus())
    kinds = {'bad-block-crc': BLOCK_CRC, 'bad-stream-crc': STREAM_CRC,
             'level-0': STREAM_HEADER, 'level-a': STREAM_HEADER,
             'trunc100': TRUNCATED, 'trunc13': TRUNCATED,
             'trailing-junk': TRAILING, 'trailing-zeros-junk': TRAILING,
             'trailing-bzh': TRUNCATED, 'bad-second-header': TRAILING,
             'flip32': BLOCK_HEADER, 'no-eos': TRUNCATED}
    names = sorted(kinds)
    res = run(check, [cases[n] for n in names], tmp_path)
    got = {n: r[0] for n, r in zip(names, res)}
    assert got == kinds
    # a block longer than its stream's level: a level-9 block relabelled 1
    big = bzcorpus.bz2.compress(bzcorpus.log_lines(2000), 9)
    assert run(check, [big[:3] + b'1' + big[4:]], tmp_path)[0][0] == OVERFLOW


def test_damaged_corpus_sanitized(check_asan, tmp_path):
    cases = bzcorpus.damaged_corpus(seed=3) + [
        c for c in bzcorpus.valid_corpus()
        if c[0] in ('multi-levels', 'run260', 'zeros-after', 'bytes256')] + [
        c for c in bzcorpus.hand_built()
        if c[0] in ('randomised', 'len20', 'false-start')]
    agree(cases, run(check_asan, [c for _, c in cases], tmp_path))


def test_randomisation_table():
    src = open(os.path.join(CSRC, 'bunzip.cuh')).read()
    body = src[src.index('#define BZ_RNUMS'):]
    body = body[:body.index('#ifdef')]
    ours = [int(x) for x in re.findall(r'\d+', body.split('\\', 1)[1])]
    assert ours == bzcorpus.rnums()


POLICY = r'''
#include <stdio.h>
#include "bunzip_policy.h"
using namespace dng;
int main()
{
	size_t ends[64];
	const size_t cases[][2] = { {0, 4}, {1, 4}, {4, 4}, {5, 4}, {8, 4},
	    {9, 1}, {3, 1000} };
	for (auto &c : cases) {
		size_t w = bz_waves(c[0], c[1], ends);
		printf("W %zu", w);
		for (size_t i = 0; i < w; i++)
			printf(" %zu", ends[i]);
		printf("\n");
	}
	const uint64_t lens[] = { 5, 5, 10, 1, 30, 2, 2 };
	const uint64_t caps[] = { 10, 11, 1, 100 };
	for (uint64_t cap : caps) {
		size_t g = bz_emit_groups(lens, 7, cap, ends);
		printf("G %zu", g);
		for (size_t i = 0; i < g; i++)
			printf(" %zu", ends[i]);
		printf("\n");
	}
	printf("G %zu\n", bz_emit_groups(lens, 0, 10, ends));
	return 0;
}
'''


def test_wave_policy(tmp_path):
    src = tmp_path / 'policy.cpp'
    src.write_text(POLICY)
    exe = str(tmp_path / 'policy')
    subprocess.check_call(['g++', '-std=c++17', '-Wall', '-Wextra', '-Werror',
                           '-I', CSRC, '-o', exe, str(src)])
    got = subprocess.check_output([exe]).decode().split('\n')
    assert got[:12] == [
        'W 0', 'W 1 1', 'W 1 4', 'W 2 4 5', 'W 2 4 8',
        'W 9 1 2 3 4 5 6 7 8 9', 'W 1 3',
        'G 5 2 3 4 5 7',        # 5+5 | 10 | 1 | 30 | 2+2: none over 10
        'G 4 2 4 5 7',
        'G 7 1 2 3 4 5 6 7',    # each alone when none fits
        'G 1 7', 'G 0']


def test_datasource_bzip2(tmp_path):
    sys.path.insert(0, ROOT)
    from dragnet_b200 import datasource_gpu as dg
    assert 'bzip2' in dg.COMPRESSIONS
    ok = tmp_path / 'a.bz2'
    ok.write_bytes(bzcorpus.bz2.compress(b'x\n'))
    for name, data, want in (('a.bz2', None, True),
                             ('b', b'BZh0....', False),
                             ('c', b'BZh', False), ('d', b'', False),
                             ('e', b'\x1f\x8b\x08\x00', False),
                             ('f', b'BZh1', True)):
        p = tmp_path / name
        if data is not None:
            p.write_bytes(data)
        assert dg.is_bzip2(str(p)) is want, name
    ds = dg.DatasourceGpu({'dsconfig': {
        'backend_config': {'path': str(tmp_path), 'compression': 'bzip2'},
        'devices': [0, 1]}})
    err = ds._run({}, [str(ok)])
    assert isinstance(err, dg.DsError)
    assert 'compression "bzip2" is not supported on a scan over several ' \
        'devices' in str(err)
    with pytest.raises(dg.DsError, match='"bzip2" is not supported'):
        dg.run_plan({}, files=[str(ok)], devices=[0, 1],
                    compression='bzip2')
