"""Scans over several devices (dng_scan_open_devices) on the GPU: the files cut
by bytes into one range per shard, the shards' tallies merged exactly.  One
H100 is enough: a device listed k times runs k shards on it."""

import ctypes
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import canon_points, cpp_engine  # noqa: E402
from golden_harness import check_section  # noqa: E402
from hostmirror import dn_index  # noqa: E402
from hostmirror import find as mod_find  # noqa: E402
from test_multi_device_host import even_cuts, shard_ranges  # noqa: E402
from dragnet_b200 import datasource_gpu, native  # noqa: E402

pytestmark = pytest.mark.gpu

EINVAL, EIO, EUNSUPPORTED, ELIMIT = -1, -5, -6, -7


@pytest.fixture(params=['auto', 'tile', 'warp', 'fast'])
def kernel(request, monkeypatch):
    """The library's own choice, the general kernels' two geometries and the
    F path forced on, as the parity tests run them."""
    for v in ('DNG_KERNEL', 'DNG_JIT'):
        monkeypatch.delenv(v, raising=False)
    if request.param == 'fast':
        monkeypatch.setenv('DNG_JIT', '0')
    if request.param != 'auto':
        monkeypatch.setenv('DNG_KERNEL', request.param)
    return request.param


def shard_counters(scan, n):
    out = []
    for sh in scan.shards(n):
        c = native.DngCounters()
        assert native.lib().dng_scan_counters(sh.handle, ctypes.byref(c)) == 0
        out.append(c.as_dict())
    return out


def multi_scan(plan, files, devices):
    """-> (points, flat counters, per-shard flat counters)"""
    import json
    p = native.Plan(json.dumps(plan))
    s = native.Scan(p, devices=devices)
    try:
        for f in files:
            s.feed_file(f)
        r = s.finish()
        pts = r.points()
        r.close()
        return pts, s.counters(), shard_counters(s, len(devices))
    finally:
        s.close()
        p.close()


# -- goldens ------------------------------------------------------------------

@pytest.mark.parametrize('k', [1, 2, 3, 4])
@pytest.mark.parametrize('suite', ['scan_file', 'scan_fileset'])
def test_goldens_split_over_shards(suite, k, goldens, datadir):
    """Every scan case of the golden file and fileset through the datasource's
    scan driver with devices = [0] * k: the goldens, and exactly what one
    scan on one device gives."""
    _goldens_on(suite, [0] * k, goldens, datadir)


def _goldens_on(suite, devices, goldens, datadir):
    def engine(plan, files):
        one = datasource_gpu.run_plan(plan, files=files)
        r = datasource_gpu.run_plan(plan, files=files, devices=devices)
        assert canon_points(r.points) == canon_points(one.points)
        assert r.counters == one.counters
        assert r.flat_counters['bytes'] == sum(os.path.getsize(f)
                                               for f in files)
        if len(devices) > 1:
            assert len(r.stats['shards']) == len(devices)
        return r.points, r.counters
    n = 0
    for i, sec in enumerate(goldens['suites'][suite]):
        if sec['cmd'] != 'scan':
            continue
        check_section(engine, suite, i, sec, datadir)
        n += 1
    assert n >= 8


def test_datasource_scan_uses_every_device(datadir):
    ds = datasource_gpu.createDatasource({
        'dsconfig': {'path': datadir, 'timeFormat': '%Y/%m-%d',
                     'timeField': 'time', 'devices': [0, 0, 0]},
        'findFiles': mod_find.find_files})
    from hostmirror import dn as mod_dn
    q = mod_dn.dnQueryConfig(mod_dn.dnParseArgs(
        ['-b', 'req.method,res.statusCode']))['query']
    r = ds.scan({'query': q, 'dryRun': False})
    assert r.stats['devices'] == [0, 0, 0]
    assert len(r.stats['shards']) == 3
    one = datasource_gpu.createDatasource({
        'dsconfig': {'path': datadir, 'timeFormat': '%Y/%m-%d',
                     'timeField': 'time'},
        'findFiles': mod_find.find_files}).scan({'query': q, 'dryRun': False})
    assert canon_points(r.points) == canon_points(one.points)
    assert r.counters == one.counters
    dry = ds.scan({'query': q, 'dryRun': True})
    assert dry.points == [] and dry.files == one.files


@pytest.mark.parametrize('suite', ['scan_file', 'scan_fileset'])
def test_goldens_on_two_gpus(suite, goldens, datadir):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('one GPU')
    _goldens_on(suite, [0, 1], goldens, datadir)


# -- where the cut lands ------------------------------------------------------

def _records(n, first=0):
    return native.gen_host(native.gen_params(total_records=200000), first, n)


def _filler(n, terminated=True):
    """One record of exactly n bytes."""
    head, tail = b'{"req":{"method":"PAD"},"pad":"', b'"}'
    body = n - len(head) - len(tail) - (1 if terminated else 0)
    assert body >= 0
    return head + b'x' * body + tail + (b'\n' if terminated else b'')


def _halve_at(files, c, terminated=True):
    """files + a trailing filler record so that T = 2c: two shards cut the
    stream at c exactly."""
    T0 = sum(map(len, files))
    files = files + [_filler(2 * c - T0, terminated)]
    T = sum(map(len, files))
    assert T // 2 == c
    return files


def cut_cases():
    R = _records(3000)
    nl = len(R) - 1                                 # R's last newline
    R2 = _records(100, 3000)
    out = {
        'on_newline': _halve_at([R, R2], nl),
        'before_newline': _halve_at([R, R2], nl - 1),
        'after_newline': _halve_at([R, R2], nl + 1),
        'empty_line': _halve_at([R + b'\n\n' + R2], len(R)),
        'second_empty_line': _halve_at([R + b'\n\n' + R2], len(R) + 1),
        'file_boundary_in_line': _halve_at(
            [R + b'{"req":{"meth', b'od":"GET"}}\n' + R2], len(R) + 13),
        'three_file_line_first': _halve_at(
            [R + b'{"req":', b'{"method":', b'"PUT"}}\n' + R2], len(R) + 7),
        'three_file_line_second': _halve_at(
            [R + b'{"req":', b'{"method":', b'"PUT"}}\n' + R2], len(R) + 17),
        'empty_file_at_cut': _halve_at([R, b'', R2], len(R)),
        'crlf': _halve_at([R.replace(b'\n', b'\r\n')],
                          len(R.replace(b'\n', b'\r\n')) - 1),
    }
    # the unterminated tail: a cut at its first byte and one inside it
    T0 = len(R)
    out['tail_start'] = [R, _filler(T0, False)]
    out['tail_inside'] = [R, _filler(T0 + 40, False)]
    return out


@pytest.fixture(scope='module')
def cut_files(tmp_path_factory):
    d = tmp_path_factory.mktemp('cuts')
    out = {}
    cases = cut_cases()
    assert sorted(cases) == sorted(CUTS)
    for name, files in cases.items():
        paths = []
        for i, f in enumerate(files):
            p = d / ('%s.%d.log' % (name, i))
            p.write_bytes(f)
            paths.append(str(p))
        out[name] = (paths, b''.join(files))
    return out


CUTS = ['on_newline', 'before_newline', 'after_newline', 'empty_line',
        'second_empty_line', 'file_boundary_in_line', 'three_file_line_first',
        'three_file_line_second', 'empty_file_at_cut', 'crlf', 'tail_start',
        'tail_inside']


@pytest.mark.parametrize('case', CUTS)
def test_cut_placement(case, kernel, cut_files):
    """Two shards cut the stream exactly at the named place (three cut it
    elsewhere): points and counters are the single scan's, each shard reads
    the bytes and lines the cut rule gives it, and the shards' bytes sum to
    T."""
    paths, stream = cut_files[case]
    T = len(stream)
    plan = corpus.make_plan(['-b', 'req.method,res.statusCode'])
    one = datasource_gpu.run_plan(plan, files=paths)
    for n in (2, 3):
        pts, flat, per = multi_scan(plan, paths, [0] * n)
        assert canon_points([(list(zip(['req.method', 'res.statusCode'], c)),
                              v) for c, v in pts]) == \
            canon_points(one.points), (case, n)
        assert flat == one.flat_counters, (case, n)
        assert flat['bytes'] == T
        ranges = shard_ranges(stream, even_cuts(T, n))
        assert [c['bytes'] for c in per] == [e - b for b, e in ranges]
        assert [c['lines'] for c in per] == [
            len([1 for _ in _lstream(stream[b:e])]) for b, e in ranges]


def _lstream(data):
    p = 0
    while p < len(data):
        j = data.find(b'\n', p)
        yield data[p:(len(data) if j < 0 else j)]
        p = len(data) if j < 0 else j + 1


def test_fanout_plan_merges_per_metric(cut_files):
    """A fan-out plan's points ([0xFD, metric] keys) and its counters of
    every metric, merged over shards."""
    paths, _ = cut_files['file_boundary_in_line']
    plan = {'format': 'json', 'ds_filter': None, 'metrics': [
        {'filter': None, 'synthetic': [], 'time_bounds': None,
         'breakdowns': [{'name': 'm', 'field': 'req.method'}]},
        {'filter': {'eq': ['res.statusCode', 200]}, 'synthetic': [],
         'time_bounds': None, 'breakdowns': []},
        {'filter': None, 'synthetic': [], 'time_bounds': None,
         'breakdowns': [{'name': 'h', 'field': 'host'},
                        {'name': 'l', 'field': 'latency',
                         'aggr': 'quantize'}]}]}
    one = datasource_gpu.run_plan(plan, files=paths)
    for k in (2, 4):
        r = datasource_gpu.run_plan(plan, files=paths, devices=[0] * k)
        assert canon_points(r.points) == canon_points(one.points), k
        assert r.flat_counters == one.flat_counters, k
        assert r.counters == one.counters, k


# -- a large file over 2, 3 and 4 shards --------------------------------------

def test_large_file_spread(tmp_path):
    n = 1500000
    p = tmp_path / 'gen.log'
    params = native.gen_params(total_records=n)
    with open(p, 'wb') as f:
        for first in range(0, n, 500000):
            f.write(native.gen_host(params, first, min(500000, n - first)))
    plan = corpus.make_plan(['-b', 'req.method,res.statusCode,host', '-f',
                             '{"ne":["req.method","HEAD"]}'])
    exp_p, exp_c = cpp_engine(plan, [str(p)], threads=os.cpu_count() or 1)
    for k in (2, 3, 4):
        r = datasource_gpu.run_plan(plan, files=[str(p)], devices=[0] * k)
        assert canon_points(r.points) == canon_points(exp_p), k
        assert r.counters == exp_c, k
        assert r.flat_counters['lines'] == n
        assert r.flat_counters['bytes'] == os.path.getsize(p)


# -- dn build -----------------------------------------------------------------

@pytest.mark.parametrize('suite', ['index_file', 'index_fileset'])
def test_build_over_three_shards(suite, datadir, tmp_path):
    """build with devices=[0, 0, 0] writes the rows a single-device build
    writes, and the reference's index goldens replay against it."""
    from test_gpu_index import table_rows
    import json
    with open(os.path.join(os.path.dirname(__file__), 'golden',
                           'index_goldens.json')) as f:
        index_goldens = json.load(f)
    nb = []

    def build(ds, metrics, interval):
        d = datasource_gpu.createDatasource({'dsconfig': ds,
                                             'findFiles': mod_find.find_files})
        res = d.build({'metrics': metrics, 'interval': interval,
                       'dryRun': False})
        assert not isinstance(res, Exception), res
        return res

    def builder(ds, metrics, interval):
        res = build(dict(ds, devices=[0, 0, 0]), metrics, interval)
        st = res.stats if isinstance(res.stats, list) else [res.stats]
        assert all(len(s['shards']) == 3 for s in st)
        root = str(tmp_path / 'one' / str(len(nb)))
        nb.append(1)
        one = build(dict(ds, indexPath=root), metrics, interval)
        assert [os.path.relpath(f, ds['indexPath'])
                for f in res.index_files] == \
            [os.path.relpath(f, root) for f in one.index_files]
        for g, c in zip(res.index_files, one.index_files):
            assert table_rows(g) == table_rows(c), g

    n = 0
    for header, act, exp in dn_index.replay(suite, index_goldens, datadir,
                                            str(tmp_path), builder):
        assert act == exp, header
        n += header != 'find'
    assert n == len(index_goldens['suites'][suite])


# -- errors -------------------------------------------------------------------

def test_long_line_across_a_cut(tmp_path):
    """A line of 2^24 bytes that crosses the cut fails with the code a single
    scan of the same file gives (which of the two the 16 MiB rule gives
    depends on how the reads fall; either way no result)."""
    pre = _records(20000)
    line = b'{"x":"' + b'y' * ((1 << 24) - 8) + b'"}'
    assert len(line) == 1 << 24
    p = tmp_path / 'long.log'
    p.write_bytes(pre + line + b'\n' + _records(1000, 20000))
    T = os.path.getsize(p)
    assert len(pre) < T // 2 < len(pre) + len(line)
    plan = corpus.make_plan(['-b', 'req.method'])
    with pytest.raises(native.DngError) as one:
        datasource_gpu.run_plan(plan, files=[str(p)])
    assert one.value.code in (ELIMIT, EUNSUPPORTED)
    for k in (2, 3):
        with pytest.raises(native.DngError) as ei:
            datasource_gpu.run_plan(plan, files=[str(p)], devices=[0] * k)
        assert ei.value.code in (ELIMIT, EUNSUPPORTED), ei.value


def test_file_changed_after_feed_is_eio(tmp_path):
    import json
    data = _records(5000)
    plan = json.dumps(corpus.make_plan(['-b', 'req.method']))
    for change in (data[:len(data) // 2], data + data[:100]):
        p = tmp_path / 'a.log'
        p.write_bytes(data)
        pl = native.Plan(plan)
        s = native.Scan(pl, devices=[0, 0])
        s.feed_file(str(p))
        p.write_bytes(change)                   # truncated, or grown
        with pytest.raises(native.DngError) as ei:
            s.finish()
        assert ei.value.code == EIO
        assert 'size' in str(ei.value) or 'shorter' in str(ei.value)
        s.close()
        pl.close()


def test_host_feeds_are_refused(tmp_path):
    import json
    import torch
    p = tmp_path / 'a.log'
    data = _records(1000)
    p.write_bytes(data)
    plan = corpus.make_plan(['-b', 'req.method'])
    pl = native.Plan(json.dumps(plan))
    s = native.Scan(pl, devices=[0, 0])
    buf = torch.empty(64, dtype=torch.uint8, device='cuda:0')
    for call in (lambda: s.feed(b'{"req":{"method":"GET"}}\n'),
                 lambda: s.feed_device(buf.data_ptr(), 16),
                 lambda: s.feed_pinned(buf.data_ptr(), 16),
                 lambda: s.set_stream(torch.cuda.current_stream().cuda_stream),
                 lambda: s.kernel_stats()):
        with pytest.raises(native.DngError) as ei:
            call()
        assert ei.value.code == EINVAL
    # not sticky: the scan still reads files
    s.feed_file(str(p))
    r = s.finish()
    one = datasource_gpu.run_plan(plan, files=[str(p)])
    assert sum(v for _, v in r.points()) == sum(v for _, v in one.points)
    assert s.counters()['lines'] == 1000
    with pytest.raises(native.DngError) as ei:
        native.Scan(pl, devices=[0, native.lib().dng_device_count()])
    assert ei.value.code == -2
    r.close()
    s.close()
    pl.close()
