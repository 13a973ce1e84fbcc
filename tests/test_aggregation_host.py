"""The group-by corpora of tests/corpus.py on the CPU: the oracles and the host
build of the device's per-record code agree on them (so that the GPU tests
may compare against the threaded C++ oracle at full size), the key-length
limit sits where the device puts it, and the colliding key groups really
collide in the hashes the device computes."""

import json
import os
import subprocess
import sys
import tempfile

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import (build_hostcheck, canon_points, cpp_engine,  # noqa: E402
                     hostcheck_engine, py_engine)


def _write(tmp_path, name, lines):
    p = tmp_path / name
    p.write_bytes(b'\n'.join(lines) + b'\n')
    return str(p)


def _collision_lines(n=6000):
    keys = [k for g in corpus.collision_groups().values() for k in g]
    return corpus.kv_lines(keys, n, seed=3)


CORPORA = {
    'sweep': (lambda: corpus.sweep_lines(1500, 20000), [['-b', 'key']]),
    'skew': (lambda: corpus.skew_lines(20000, tail=5000), [['-b', 'key']]),
    'lengths': (lambda: corpus.key_length_lines(reps=3), [['-b', 'key']]),
    'lengths2': (lambda: corpus.key_length_lines(True, reps=3),
                 [['-b', 'key,key2'], ['-b', 'key2']]),
    'merge_apart': (lambda: corpus.merge_apart_lines(reps=3),
                    [['-b', 'key,key2'], ['-b', 'key']]),
    'buckets': (lambda: corpus.BUCKET_LINES,
                [['-b', 'num[aggr=quantize]'], ['-b', 'num'],
                 ['-b', 'num[aggr=lquantize,step=2]']]),
    'collisions': (_collision_lines, [['-b', 'key']]),
}


@pytest.mark.parametrize('hostf', [False, True])
@pytest.mark.parametrize('name', sorted(CORPORA))
def test_engines_agree_on_group_by_corpora(name, hostf, tmp_path,
                                           monkeypatch):
    """py oracle == C++ oracle == host build of the device code (with the F
    path's templates, piece-wise hash and key compare in front, or not)."""
    make, queries = CORPORA[name]
    path = _write(tmp_path, name + '.log', make())
    monkeypatch.delenv('DNG_HOSTCHECK_F', raising=False)
    if hostf:
        monkeypatch.setenv('DNG_HOSTCHECK_F', '1')
    for argv in queries:
        plan = corpus.make_plan(argv)
        exp_p, exp_c = py_engine(plan, [path])
        cp, cc = cpp_engine(plan, [path], threads=2)
        hp, hc = hostcheck_engine(plan, [path])
        assert canon_points(cp) == canon_points(exp_p), argv
        assert cc == exp_c, argv
        assert canon_points(hp) == canon_points(exp_p), argv
        assert hc == exp_c, argv


def test_engines_agree_on_weights(tmp_path):
    """The weights corpus the GPU test uses, whole: both oracles and the host
    build agree, and equal the Python integer sums, all below 2^63 (the C++
    oracle and the device sum in u64; past 2^64 they would agree on a
    wrapped value)."""
    lines = corpus.weight_lines()
    path = _write(tmp_path, 'w.log', lines)
    plan = corpus.make_plan(['-b', 'key'], {'dataFormat': 'json-skinner'})
    exp_p, exp_c = py_engine(plan, [path])
    cp, cc = cpp_engine(plan, [path], threads=4)
    hp, hc = hostcheck_engine(plan, [path])
    assert canon_points(cp) == canon_points(exp_p)
    assert canon_points(hp) == canon_points(exp_p)
    assert cc == exp_c == hc
    sums = corpus.weight_sums(lines)
    assert {f[0][1]: v for f, v in exp_p} == sums
    assert max(sums.values()) < 1 << 63
    assert min(v for k, v in sums.items() if k.startswith(b'shared')) > \
        1 << 56
    assert [sums[b'zero%d' % i] for i in range(7)] == [0] * 7
    # 9007199254740994 (2^53 + 2) is not a safe integer: an invalid point;
    # 9007199254740993 rounds to 2^53 and counts
    bad = sum(1 for ln in lines if ln.endswith(b':9007199254740994}'))
    assert bad > 0
    assert exp_c['json parser']['invalid point'] == bad


def _hostcheck_doc(plan, path, env=None):
    exe = build_hostcheck()
    with tempfile.NamedTemporaryFile('w', suffix='.json', delete=False) as f:
        json.dump(plan, f)
        pf = f.name
    try:
        out = subprocess.run([exe, pf, path], capture_output=True, check=True,
                             env=dict(os.environ, **(env or {}))).stdout
    finally:
        os.unlink(pf)
    return json.loads(out)


@pytest.mark.parametrize('cols,ok', [
    ((510,), True), ((511,), False),            # one column: klen 512 / 513
    ((500, 8), True), ((500, 9), False),        # two: klen 512 / 513
    ((501, 0), False),                          # klen 505, but the second
                                                # column starts past 502
    ((250, 254), True)])
def test_longest_group_key(cols, ok, tmp_path):
    """KEY_MAX: the longest key the device tallies is 512 bytes, and a
    second column is refused once fewer than 10 bytes are left for it
    (process_metric); anything longer is counted as unsupported."""
    vals = [b'v' * n for n in cols]
    names = ['key', 'key2'][:len(cols)]
    line = b'{' + b','.join(b'"%s":"%s"' % (n.encode(), v)
                            for n, v in zip(names, vals)) + b'}'
    path = _write(tmp_path, 'long.log', [line] * 3)
    doc = _hostcheck_doc(corpus.make_plan(['-b', ','.join(names)]), path)
    assert doc['counters']['unsupported'] == (0 if ok else 3), doc
    assert len(doc['points']) == (1 if ok else 0)
    if ok:
        assert len(corpus.encode_key(*vals)) <= corpus.KEY_MAX


def _key_dump(tmp_path, lines, argv=('-b', 'key')):
    path = _write(tmp_path, 'keys.log', lines)
    dump = str(tmp_path / 'keys.txt')
    doc = _hostcheck_doc(corpus.make_plan(list(argv)), path,
                         {'DNG_HOSTCHECK_F': '1', 'DNG_HOSTCHECK_KEYS': dump})
    keys = {}
    with open(dump) as f:
        for ln in f:
            k, fh, gh = ln.split()
            keys[bytes.fromhex(k)] = (None if fh == '-' else int(fh, 16),
                                      int(gh, 16))
    return doc, keys


def test_key_dump_shows_the_collisions(tmp_path):
    """Every group of corpus.collision_groups meets where it claims to, in
    the hashes the device code computes (hostcheck's dump), and the Python
    restatement of both hashes matches them key for key."""
    groups = corpus.collision_groups()
    doc, keys = _key_dump(tmp_path, _collision_lines())
    assert doc['nfmatch'] > 0.99 * doc['counters']['lines'], doc
    for name, strs in groups.items():
        got = [keys[corpus.encode_key(s)] for s in strs]
        fh = [f for f, _ in got]
        gh = [g for _, g in got]
        assert None not in fh, (name, 'not through the F path')
        assert fh == [corpus.fkey_hash(s) for s in strs], name
        assert gh == [corpus.gkey_hash(s) for s in strs], name
        assert len(strs) >= 32, name
        if name == 'f_full':
            assert len(set(fh)) == 1, name
            assert len(corpus.encode_key(strs[0])) <= corpus.SKEY
        elif name == 'f_index':
            assert len({(h >> 7) & 1023 for h in fh}) == 1, name
            assert len(set(fh)) == len(fh), name
            assert len(corpus.encode_key(strs[0])) <= corpus.SKEY
        elif name in ('g1_full', 'g2_full'):
            assert len(set(gh)) == 1, name
        else:
            shift, bits = {'g1_index': (40, 10), 'g2_index': (28, 12),
                           'global_index': (17, 10)}[name]
            slots = {(h >> shift) & ((1 << bits) - 1) for h in gh}
            assert len(slots) == 1, name
            if name == 'global_index':
                # near the end of a 1024-entry table: the chain wraps
                assert slots == {corpus.GLOBAL_SLOT}
                assert corpus.GLOBAL_SLOT + len(strs) > 1024
            assert len(set(gh)) == len(gh), name
        klen = len(corpus.encode_key(strs[0]))
        if name.startswith('g1'):
            assert klen <= corpus.SKEY, name
        if name.startswith('g2'):
            assert klen > corpus.SKEY, name
