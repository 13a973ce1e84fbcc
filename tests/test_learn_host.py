"""What a scan computes on the host before its first launch (csrc/tmpl.cpp
tmpl_candidates, csrc/jit.cpp jit_key), on the CPU with a small driver
(tests/hostcheck/learn_check.cpp): the candidate pass groups lines exactly as a
plain grouping by tmpl_skeletonize() does, and the run-time compiled kernel
cache tells apart every input the generated matcher is made from."""

import os
import random
import subprocess
import sys
import tarfile

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
import framing  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')
DRIVER = os.path.join(ROOT, 'tests', 'hostcheck', 'learn_check.cpp')


@pytest.fixture(scope='module')
def learn_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp('lc') / 'learn_check')
    # jit.cpp links the relocatable kernel and fscan.cuh as data
    subprocess.check_call(['make', '-s', '-C', CSRC, 'build/jit_blob.o'])
    subprocess.check_call(
        ['g++', '-std=c++17', '-O1', '-I/usr/local/cuda/include', '-o', exe,
         DRIVER] + [os.path.join(CSRC, f) for f in
                    ('plan.cpp', 'result.cpp', 'tmpl.cpp', 'fast.cpp',
                     'jit.cpp')] +
        [os.path.join(CSRC, 'build', 'jit_blob.o'), '-ldl'])
    return exe


def candidates(exe, data, tmp_path, maxk=256):
    import json
    p = tmp_path / 'in.log'
    p.write_bytes(data)
    r = subprocess.run([exe, 'cands', str(p), str(maxk)], capture_output=True,
                       check=True)
    return json.loads(r.stdout)


def check_same(exe, data, tmp_path):
    """the candidates, their order, counts, segments and samples, and the
    lines looked at, with every shape kept and with the scan's own limit"""
    for maxk in (256, 24):
        d = candidates(exe, data, tmp_path, maxk)
        assert d['fast'] == d['plain'], maxk


def pieces(data, nlines=150):
    """pieces of at most nlines lines: every shape of a piece is kept (one line
    is more than 0.5 % of it), so its candidates are the whole grouping"""
    lines = data.split(b'\n')
    return [b'\n'.join(lines[i:i + nlines]) + b'\n'
            for i in range(0, len(lines), nlines)]


def test_edge_corpus(learn_check, tmp_path):
    data = b'\n'.join(corpus.EDGE_LINES + corpus.SKINNER_LINES) + b'\n'
    for p in pieces(data):
        check_same(learn_check, p, tmp_path)
    # every edge line next to copies of itself with other scalar values
    for line in corpus.EDGE_LINES:
        check_same(learn_check, (line + b'\n') * 3 + line, tmp_path)


@pytest.mark.parametrize('seed', range(6))
def test_seeded_json(learn_check, tmp_path, seed):
    data = b'\n'.join(corpus.random_lines(seed, 600)) + b'\n'
    for p in pieces(data):
        check_same(learn_check, p, tmp_path)
    check_same(learn_check, data, tmp_path)


def test_shapes_that_differ_late_and_in_values(learn_check, tmp_path):
    """shapes sharing long prefixes, strings with escapes and quotes,
    scalars next to every delimiter: the pass resumes a failed shape's common
    segments on the next one"""
    rng = random.Random(5)
    strs = [b'', b'a', b'\\"', b'x\\\\', b'\\\\\\"q', b'{[,:]}', b'\\u0041 b']
    bares = [b'0', b'-1.5e3', b'true', b'null', b'false', b'12x']
    lines = []
    for _ in range(2000):
        parts = [b'"k%d":' % rng.randrange(3) + rng.choice(
            [b'"' + rng.choice(strs) + b'"', rng.choice(bares),
             b'[' + rng.choice(bares) + b' ,' + rng.choice(bares) + b']',
             b'{"z" : ' + rng.choice(bares) + b'}'])
            for _ in range(rng.randrange(1, 5))]
        sep = rng.choice([b',', b', ', b' ,\t'])
        line = b'{' + sep.join(parts) + b'}'
        if rng.random() < 0.05:
            line = line[:rng.randrange(len(line))]     # not a JSON text
        lines.append(line)
    data = b'\n'.join(lines) + b'\n'
    for p in pieces(data):
        check_same(learn_check, p, tmp_path)
    check_same(learn_check, data, tmp_path)


def test_framing_layouts(learn_check, tmp_path):
    data, _ = framing.f_block(seed=1, rounds=1)
    head = data[:framing.SAMPLE]
    check_same(learn_check, head, tmp_path)
    for p in pieces(head)[:40]:
        check_same(learn_check, p, tmp_path)
    check_same(learn_check, framing.long_line(5000) + b'\n' +
               framing.long_line(300) + b'\n', tmp_path)


def test_golden_data(learn_check, tmp_path):
    with tarfile.open(os.path.join(ROOT, 'tests', 'golden',
                                   'data.tar.gz')) as tf:
        for m in tf.getmembers():
            if not m.isfile():
                continue
            data = tf.extractfile(m).read()
            check_same(learn_check, data[:framing.SAMPLE], tmp_path)
            for p in pieces(data)[:5]:
                check_same(learn_check, p, tmp_path)


def test_bench_sample_and_limits(learn_check, tmp_path):
    """the head the bench's scans learn from; over 8192 lines; more than 256
    shapes; lines over TMPL_MAX_LINE and empty lines"""
    from dragnet_b200 import native
    n = 3000
    data = native.gen_host(native.gen_params(seed=0xD5A60000,
                                             total_records=100000000), 0, n)
    d = candidates(learn_check, data[:framing.SAMPLE], tmp_path, 24)
    assert d['fast'] == d['plain']
    assert len(d['fast']['cands']) == 3
    many = b''.join(b'{"a%d":%d}\n' % (i % 300, i) for i in range(9000))
    d = candidates(learn_check, many, tmp_path)
    assert d['fast'] == d['plain'] and d['fast']['lines'] == 8192
    odd = b'\n'.join([b'{"x":1}', b'', b'{"x":"' + b'y' * 5000 + b'"}',
                      b'{"x":2}', b'[' * 70 + b']' * 70, b'{"x":3}']) + b'\n'
    check_same(learn_check, odd, tmp_path)


def test_jit_cache_key(learn_check):
    r = subprocess.run([learn_check, 'jitkey'], capture_output=True,
                       text=True, check=True)
    got = dict(line.split() for line in r.stdout.splitlines())
    assert got.pop('identical') == 'same'
    # DNG_JIT_SHARED=0 on a one-column plan: the choice it already had
    assert got.pop('shared_off') == 'same'
    assert got and all(v == 'differs' for v in got.values()), got
