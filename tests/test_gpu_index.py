"""`dn build` on the GPU: index files written by DatasourceGpu.build from the
fan-out scan, replayed against the reference's index goldens
(tests/dn/local/tst.index_file.sh.out, tst.index_fileset.sh.out) and compared
row for row with index files built from the CPU oracle's points."""

import os
import sqlite3
import sys
import time

import pytest

sys.path.insert(0, os.path.dirname(__file__))
from engines import canon_points, cpp_engine  # noqa: E402
from hostmirror import dn_index  # noqa: E402
from hostmirror import find as mod_find  # noqa: E402
from test_index_host import NINE, cpu_points  # noqa: E402
from dragnet_b200 import datasource_gpu  # noqa: E402
from dragnet_b200 import index as mod_index  # noqa: E402
from dragnet_b200 import query as mod_query  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def index_goldens():
    import json
    with open(os.path.join(os.path.dirname(__file__), 'golden',
                           'index_goldens.json')) as f:
        return json.load(f)


@pytest.fixture(params=['auto', 'tile', 'warp'])
def kernel(request, monkeypatch):
    """The library's own choice and the general kernels' two geometries (a
    fan-out plan never takes the F path)."""
    for v in ('DNG_KERNEL', 'DNG_JIT', 'DNG_F_WARPS', 'DNG_TABLE_CAP'):
        monkeypatch.delenv(v, raising=False)
    if request.param != 'auto':
        monkeypatch.setenv('DNG_KERNEL', request.param)
    return request.param


def gpu_build(ds, metrics, interval):
    d = datasource_gpu.createDatasource({'dsconfig': ds,
                                         'findFiles': mod_find.find_files})
    res = d.build({'metrics': metrics, 'interval': interval,
                   'dryRun': False})
    assert not isinstance(res, Exception), res
    return res


def table_rows(path):
    """Every table of an index file, rows in a fixed order."""
    db = sqlite3.connect(path)
    try:
        out = {}
        for (t,) in db.execute("SELECT name FROM sqlite_master WHERE "
                               "type = 'table' ORDER BY name"):
            out[t] = db.execute('SELECT * FROM %s ORDER BY %s' % (
                t, ','.join(str(i + 1) for i in range(len(
                    db.execute('SELECT * FROM %s' % t).description))))
            ).fetchall()
        return out
    finally:
        db.close()


@pytest.mark.parametrize('suite', ['index_file', 'index_fileset'])
def test_index_goldens_replay_gpu_built(suite, kernel, index_goldens,
                                        datadir, tmp_path):
    nbuilds = []

    def builder(ds, metrics, interval):
        res = gpu_build(ds, metrics, interval)
        assert res.stats['kernel'] != 'F path'
        root = str(tmp_path / 'cpu' / str(len(nbuilds)))
        nbuilds.append(1)
        cpu = mod_index.write_index(root, metrics, interval,
                                    cpu_points(ds, metrics, interval))
        assert [os.path.relpath(f, ds['indexPath'])
                for f in res.index_files] == \
            [os.path.relpath(f, root) for f in cpu]
        for g, c in zip(res.index_files, cpu):
            assert table_rows(g) == table_rows(c), g

    n = 0
    for header, act, exp in dn_index.replay(suite, index_goldens, datadir,
                                            str(tmp_path), builder):
        assert act == exp, header
        n += header != 'find'
    assert n == len(index_goldens['suites'][suite])
    if suite == 'index_fileset':
        assert not dn_index.empty_build(gpu_build, str(tmp_path))


def test_nine_metrics_take_two_passes(datadir, tmp_path):
    ds = {'path': datadir, 'timeField': 'time',
          'indexPath': str(tmp_path / 'idx'),
          'filter': {'ne': ['req.method', 'HEAD']}}
    res = gpu_build(ds, NINE, 'hour')
    assert isinstance(res.stats, list) and len(res.stats) == 2
    assert len(res.counters) == 9
    for i, m in enumerate(NINE):
        got = [(f[:-1], v) for f, v in res.points if f[-1] == ('__dn_metric',
                                                               i)]
        exp = [(f[:-1], v) for f, v in cpu_points(ds, [m], 'hour')]
        assert got and canon_points(got) == canon_points(exp), i
    cpu = mod_index.write_index(str(tmp_path / 'cpu'), NINE, 'hour',
                                cpu_points(ds, NINE, 'hour'))
    assert [os.path.basename(f) for f in res.index_files] == \
        [os.path.basename(f) for f in cpu]
    for g, c in zip(res.index_files, cpu):
        rows = table_rows(g)
        assert len([t for t in rows if t.startswith('dragnet_index_')]) == 9
        assert rows == table_rows(c), g


GEN_METRICS = [
    {'name': 'bymethod', 'filter': None,
     'breakdowns': [{'name': 'req.method', 'field': 'req.method'},
                    {'name': 'host', 'field': 'host'}]},
    {'name': 'latency', 'filter': {'eq': ['res.statusCode', 200]},
     'breakdowns': [{'name': 'operation', 'field': 'operation'},
                    {'name': 'latency', 'field': 'latency',
                     'aggr': 'quantize'}]},
]


def _row(fields, value):
    row = []
    for _, v in fields:
        if isinstance(v, bytes):
            row.append(v.decode('utf-8'))
        elif v != v:
            row.append(None)
        else:
            row.append(int(v) if v == int(v) else v)
    return tuple(row) + (value,)


def test_hourly_build_of_generated_rows(tmp_path):
    """A few million generated records over three hours: every hour file
    holds exactly the oracle's points for that hour."""
    from dragnet_b200 import native
    n = 3000000
    p = tmp_path / 'gen.log'
    with open(p, 'wb') as f:
        step = 500000
        params = native.gen_params(total_records=n)
        for first in range(0, n, step):
            f.write(native.gen_host(params, first, min(step, n - first)))
    ds = {'path': str(p), 'timeField': 'time',
          'indexPath': str(tmp_path / 'idx')}
    res = gpu_build(ds, GEN_METRICS, 'hour')
    labels = [os.path.basename(f) for f in res.index_files]
    assert len(labels) >= 3
    for i, m in enumerate(GEN_METRICS):
        q = mod_query.metricQuery(m, None, None, 'hour', 'time')
        plan = mod_query.scan_plan(q, time_field='time')
        pts, _ = cpp_engine(plan, [str(p)], threads=os.cpu_count() or 1)
        byhour = {}
        for fields, value in pts:
            assert fields[0][0] == '__dn_ts'
            label = time.strftime('%Y-%m-%d-%H.sqlite',
                                  time.gmtime(fields[0][1]))
            byhour.setdefault(label, []).append(_row(fields[1:], value))
        assert sorted(byhour) == labels, i
        for f in res.index_files:
            db = sqlite3.connect(f)
            got = db.execute('SELECT * FROM dragnet_index_%d' % i).fetchall()
            db.close()
            assert sorted(got, key=repr) == \
                sorted(byhour[os.path.basename(f)], key=repr), (i, f)
