"""krill filters (corpus.filter_lines) through the CUDA scan under every
kernel: the comparison matrix of `v` in every value form against every
constant, random predicate trees of 1-48 leaves and datasource + user +
time-bound programs in one plan.  The general tiers evaluate them with
record.cuh eval_program, the F kernel with fast.cuh feval, and its run-time
linked form (DNG_JIT=sync) with feval unrolled over a constant plan, which
only a GPU run reaches.  Points and counters are compared with the C++
oracle, tallies and the filter stages' counters with the second reference
(corpus.krill_reference).  Also the kernel each kind of plan runs on, and
the plan limits at plan creation."""

import json
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import canon_points, cpp_engine  # noqa: E402
from dragnet_b200 import datasource_gpu, native  # noqa: E402

pytestmark = pytest.mark.gpu

SEED = 0
N = 30000
QUERIES = corpus.filter_queries()
QNAMES = sorted(QUERIES)
JIT_NAMES = corpus.filter_jit_names(QNAMES)


@pytest.fixture(scope='module')
def filters(tmp_path_factory):
    recs = corpus.filter_records(SEED, N)
    data = b'\n'.join(corpus.filter_line(r) for r in recs) + b'\n'
    p = tmp_path_factory.mktemp('filters') / 'filters.log'
    p.write_bytes(data)
    return recs, data, str(p)


def _set_kernel(monkeypatch, k):
    monkeypatch.delenv('DNG_KERNEL', raising=False)
    monkeypatch.delenv('DNG_JIT', raising=False)
    if k in ('fast', 'jit'):
        monkeypatch.setenv('DNG_KERNEL', 'fast')
        monkeypatch.setenv('DNG_JIT', 'sync' if k == 'jit' else '0')
    elif k != 'auto':
        monkeypatch.setenv('DNG_KERNEL', k)


@pytest.fixture(params=['auto', 'tile', 'warp', 'fast'])
def kernel(request, monkeypatch):
    _set_kernel(monkeypatch, request.param)
    return request.param


_ORACLE = {}


def oracle(key, plan, path):
    """(canon points, counters) of the C++ oracle, once per module."""
    if key not in _ORACLE:
        p, c = cpp_engine(plan, [path], threads=8)
        _ORACLE[key] = (canon_points(p), c)
    return _ORACLE[key]


def _odd_chunks(data, seed):
    """data cut at odd sizes, mid-line and mid-character."""
    out, i, k = [], 0, 0
    sizes = (1 << 20) + 7, 65521, 3 << 20, 999983
    while i < len(data):
        n = sizes[(k + seed) % len(sizes)]
        out.append(data[i:i + n])
        i, k = i + n, k + 1
    return out


def scan_both_feeds(key, argv, ds, filters):
    """The plan over the corpus as a file and as odd chunks; each result
    checked against the C++ oracle.  Returns the two results."""
    recs, data, path = filters
    plan = corpus.make_plan(argv, ds)
    exp_p, exp_c = oracle(key, plan, path)
    out = []
    for feed in ('file', 'chunks'):
        if feed == 'file':
            r = datasource_gpu.run_plan(plan, files=[path])
        else:
            r = datasource_gpu.run_plan(plan, chunks=_odd_chunks(data, SEED))
        assert canon_points(r.points) == exp_p, (key, feed)
        assert r.counters == exp_c, (key, feed)
        out.append(r)
    return out


def check_query(name, kernel, filters):
    recs = filters[0]
    q = QUERIES[name]
    argv, ds, pred, dsp, bounds = q
    tally, split = corpus.krill_reference(recs, pred, dsp, bounds)
    for r in scan_both_feeds(name, argv, ds, filters):
        assert corpus.tag_points(r.points) == tally, name
        for stage, want in split.items():
            assert corpus.filter_split(r.counters, stage) == want, \
                (name, stage)
        st = r.stats
        if kernel in ('fast', 'jit') and corpus.query_leaves(q) <= 16 and \
                corpus.query_capture_rows(q) <= 3:
            # forced F kernel, and a plan the F path models whose capture
            # rows fit in shared memory beside the widest lane slice
            assert st['kernel'] == 'F path', (name, st)
        if st['kernel'] == 'F path':
            assert st['templated_records'] > 0, (name, st)
            if kernel == 'jit':
                assert st['jit']['state'] == 1, (name, st)
                assert st['jit']['launches'] >= 1, (name, st)


@pytest.mark.parametrize('name', QNAMES)
def test_filter(name, kernel, filters):
    """Every filter query under auto, tile, warp and the forced F kernel.
    Under the F kernel the plans it must take (at most 16 leaves, at most 3
    capture rows) are asserted to run on it, so that its evaluator, not the
    miss kernel's, is what the comparison checks."""
    check_query(name, kernel, filters)


@pytest.mark.parametrize('name', JIT_NAMES)
def test_filter_jit(name, filters, monkeypatch):
    """The run-time linked F kernel (DNG_KERNEL=fast DNG_JIT=sync), whose
    feval is unrolled over the plan's leaves as constants and relies on
    jumps going forward only.  Where the plan is the F path's, the linked
    kernel must have been built and launched."""
    _set_kernel(monkeypatch, 'jit')
    check_query(name, 'jit', filters)


# (argv, rows) of the fit boundary: capture rows are one per path plus two
# per bucketized column
FIT = {'rows3': (['-b', 'n[aggr=lquantize,step=10]'], 3),
       'rows4': (['-b', 'n[aggr=lquantize,step=10],s,'], 4)}


@pytest.mark.parametrize('case', sorted(FIT))
def test_f_kernel_capture_row_fit(case, filters, monkeypatch):
    """The F kernel's shared memory is sized for 28 warps and the widest
    lane slice (api.cu dng_scan_open): on an H100 (227 KB a block) that
    leaves room for 3 capture rows of 3,584 bytes.  A plan of 4 rows runs
    on the general kernels even under DNG_KERNEL=fast, with the same
    results; this pins where the boundary is today."""
    _set_kernel(monkeypatch, 'fast')
    argv, rows = FIT[case]
    for r in scan_both_feeds('fit_' + case, argv, None, filters):
        if rows <= 3:
            assert r.stats['kernel'] == 'F path', r.stats
            assert r.stats['templated_records'] > 0, r.stats
        else:
            assert r.stats['kernel'] != 'F path', r.stats


@pytest.mark.parametrize('limit', sorted(corpus.F_LIMITS))
def test_f_plan_limit(limit, filters, monkeypatch):
    """Each limit of the F plan under DNG_KERNEL=fast, at the limit and one
    past it: results equal the oracle's both ways.  The leaf and pool cases
    need two capture rows, so the F kernel's fit decides nothing there: at
    the limit the plan must run on the F kernel, one past it must not.  The
    path, column and synthetic-field cases need 5 or more capture rows even
    at the limit, which no plan gets on the F kernel of an H100 today
    (test_f_kernel_capture_row_fit), so on the GPU they only compare
    results; test_filters_host.py's F mode, which has no shared-memory fit,
    is what pins those three limits."""
    _set_kernel(monkeypatch, 'fast')
    at, over = corpus.F_LIMITS[limit]
    r_at = scan_both_feeds('f_' + limit, at, None, filters)
    r_over = scan_both_feeds('f_over_' + limit, over, None, filters)
    for r in r_at:
        if limit in ('leaves_16', 'pool_484'):
            assert r.stats['kernel'] == 'F path', r.stats
        if r.stats['kernel'] == 'F path':
            assert r.stats['templated_records'] > 0, r.stats
    for r in r_over:
        if limit in ('leaves_16', 'pool_484'):
            assert r.stats['kernel'] != 'F path', r.stats


@pytest.mark.parametrize('limit', sorted(corpus.PLAN_LIMITS))
def test_plan_limit(limit, filters, monkeypatch):
    """A plan at each compiler limit scans as the oracle does; one past it,
    plan creation fails with DNG_ELIMIT.  The scans run in the default
    mode, where the matcher is compiled on a worker thread: they are short,
    so the module may end with such a compile still in flight, and the
    process must still exit cleanly (jit.cpp jit_prepare)."""
    _set_kernel(monkeypatch, 'auto')
    at, over, msg = corpus.PLAN_LIMITS[limit]
    scan_both_feeds('limit_' + limit, at, None, filters)
    with pytest.raises(native.DngError) as ei:
        native.Plan(json.dumps(corpus.make_plan(over)))
    assert ei.value.code == -7, ei.value
    assert msg in str(ei.value)
