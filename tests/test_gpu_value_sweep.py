"""The value sweep (corpus.value_sweep_lines) through the CUDA scan under every
kernel: the F path's own conversions (fsimple_int, fnumber, feval_leaf,
fdate, fprep) and the general tiers' on numbers at binary64 and
simple-integer edges, numeric strings, strings at UTF-8/UTF-16 edges and
dates over years 0000-9999.  Points and counters are compared with the C++
oracle, and for the numeric columns and the filters also with a second
reference derived from the generated values (corpus.sweep_reference)."""

import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import canon_points, cpp_engine  # noqa: E402
from dragnet_b200 import datasource_gpu, native  # noqa: E402

pytestmark = pytest.mark.gpu

SEEDS = (0, 1)
N = 100000
QNAMES = sorted(corpus.sweep_queries(corpus.value_sweep_records(0, 50)))


@pytest.fixture(params=['auto', 'tile', 'warp', 'fast', 'jit'])
def kernel(request, monkeypatch):
    monkeypatch.delenv('DNG_KERNEL', raising=False)
    monkeypatch.delenv('DNG_JIT', raising=False)
    k = request.param
    if k in ('fast', 'jit'):
        monkeypatch.setenv('DNG_KERNEL', 'fast')
        monkeypatch.setenv('DNG_JIT', 'sync' if k == 'jit' else '0')
    elif k != 'auto':
        monkeypatch.setenv('DNG_KERNEL', k)
    return k


_CORPORA = {}
_ORACLE = {}


def sweep(seed, tmp_path_factory):
    if seed not in _CORPORA:
        recs = corpus.value_sweep_records(seed, N)
        data = b'\n'.join(corpus.value_sweep_line(r) for r in recs) + b'\n'
        p = tmp_path_factory.mktemp('sweep') / ('sweep%d.log' % seed)
        p.write_bytes(data)
        _CORPORA[seed] = (recs, data, str(p), corpus.sweep_queries(recs))
    return _CORPORA[seed]


def oracle(seed, name, plan, path, recs, kind, arg):
    """(canon points, counters, second reference) of the C++ oracle, once per
    module."""
    if (seed, name) not in _ORACLE:
        p, c = cpp_engine(plan, [path], threads=8)
        ref = corpus.sweep_reference(recs, kind, arg) if kind else None
        _ORACLE[seed, name] = (canon_points(p), c, ref)
    return _ORACLE[seed, name]


def _odd_chunks(data, seed):
    """data cut at odd sizes, mid-line and mid-character."""
    out, i, k = [], 0, 0
    sizes = (1 << 20) + 7, 65521, 3 << 20, 999983
    while i < len(data):
        n = sizes[(k + seed) % len(sizes)]
        out.append(data[i:i + n])
        i, k = i + n, k + 1
    return out


@pytest.mark.parametrize('name', QNAMES)
@pytest.mark.parametrize('seed', SEEDS)
def test_value_sweep(seed, name, kernel, tmp_path_factory):
    recs, data, path, queries = sweep(seed, tmp_path_factory)
    argv, ds, kind, arg = queries[name]
    plan = corpus.make_plan(argv, ds)
    exp_p, exp_c, ref = oracle(seed, name, plan, path, recs, kind, arg)
    for feed in ('file', 'chunks'):
        if feed == 'file':
            r = datasource_gpu.run_plan(plan, files=[path])
        else:
            r = datasource_gpu.run_plan(plan, chunks=_odd_chunks(data, seed))
        assert canon_points(r.points) == exp_p, (name, feed)
        assert r.counters == exp_c, (name, feed)
        if kind:
            assert corpus.sweep_points(r.points, kind, arg) == ref, \
                (name, feed)
        st = r.stats
        if kernel in ('fast', 'jit'):
            # under the F kernel, templated_records counts exactly the
            # records it decided (the miss kernel adds none)
            need = corpus.sweep_f_decided(recs, argv)
            assert st['templated_records'] >= need, (name, feed, need, st)
        elif kernel in ('tile', 'warp'):
            assert st['templated_records'] >= 0.9 * N, (name, feed, st)
        if kernel == 'jit':
            assert st['jit']['state'] == 1, st
            assert st['jit']['launches'] >= 1, st


LEGACY = [b'Thu, 01 May 2014 00:00:00 GMT', b'2014-05-01 12:00:00']


@pytest.mark.parametrize('bad', LEGACY)
def test_legacy_date_string_fails_the_scan(bad, kernel, tmp_path):
    """A date string V8's legacy Date.parse might read, among sweep records:
    the scan fails with DNG_EUNSUPPORTED (it is neither parsed nor called
    NaN).  On the F path such a record is a miss, so the miss kernel decides
    it."""
    lines = corpus.value_sweep_lines(3, 20000)
    lines.insert(12345, b'{"num":1,"nstr":"2","str":"s","ts":"%s","pad":"%s"}'
                 % (bad, b'p' * 100))
    p = tmp_path / 'legacy.log'
    p.write_bytes(b'\n'.join(lines) + b'\n')
    plan = corpus.make_plan(['-b', 'ts[date,field=ts,aggr=lquantize,'
                             'step=86400]'])
    with pytest.raises(native.DngError) as ei:
        datasource_gpu.run_plan(plan, files=[str(p)])
    assert ei.value.code == -6, ei.value
