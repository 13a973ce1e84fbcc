"""`dn build` + `dn query` without a GPU: index files written by
dragnet_b200.index from points the CPU oracle computes, queried through the
GPU datasource's query() (which reads no raw data), checked against the
reference's index goldens (tests/dn/local/tst.index_file.sh.out,
tst.index_fileset.sh.out) and against lib/index-sink.js / index-query.js."""

import json
import os
import sqlite3
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
from engines import canon_points, py_engine  # noqa: E402
from hostmirror import dn_index  # noqa: E402
from hostmirror import find as mod_find  # noqa: E402
from dragnet_b200 import datasource_gpu  # noqa: E402
from dragnet_b200 import index as mod_index  # noqa: E402
from dragnet_b200 import query as mod_query  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')


@pytest.fixture(scope='module')
def index_goldens():
    with open(os.path.join(GOLDEN, 'index_goldens.json')) as f:
        return json.load(f)


def cpu_points(ds, metrics, interval):
    """The tagged points of `dn build`, one oracle scan per metric."""
    files = mod_find.find_files(ds['path'])
    pts = []
    for i, m in enumerate(metrics):
        q = mod_query.metricQuery(m, None, None, interval,
                                  ds.get('timeField'))
        plan = mod_query.scan_plan(q, ds_filter=ds.get('filter'),
                                   time_field=ds.get('timeField'))
        p, _ = py_engine(plan, files)
        pts += [(f + [('__dn_metric', i)], v) for f, v in p]
    return pts


def cpu_builder(ds, metrics, interval):
    return mod_index.write_index(ds['indexPath'], metrics, interval,
                                 cpu_points(ds, metrics, interval))


@pytest.mark.parametrize('suite', ['index_file', 'index_fileset'])
def test_index_goldens_replay(suite, index_goldens, datadir, tmp_path):
    n = 0
    for header, act, exp in dn_index.replay(suite, index_goldens, datadir,
                                            str(tmp_path), cpu_builder):
        assert act == exp, header
        n += header != 'find'
    assert n == len(index_goldens['suites'][suite])


def test_index_golden_section_count(index_goldens):
    assert sum(len(v) for v in index_goldens['suites'].values()) == 35
    assert len(index_goldens['find']['index_fileset']) == 120


def test_empty_input_creates_no_directory(tmp_path):
    assert not dn_index.empty_build(cpu_builder, str(tmp_path))
    assert mod_index.write_index(str(tmp_path / 'x'), [], 'hour', []) == []
    assert not (tmp_path / 'x').exists()


# ---------------------------------------------------------------------------
# the index file itself (lib/index-sink.js)
# ---------------------------------------------------------------------------

METRICS = [
    {'name': 'big', 'filter': None,
     'breakdowns': [{'name': 'host', 'field': 'host'},
                    {'name': 'req.method', 'field': 'req.method'},
                    {'name': 'latency', 'field': 'latency',
                     'aggr': 'quantize'}]},
    {'name': 'daily', 'filter': {'eq': ['req.method', 'GET']},
     'breakdowns': [{'name': 'timestamp', 'field': 'time', 'date': '',
                     'aggr': 'lquantize', 'step': 86400}]},
]


def _dump(path, sql):
    db = sqlite3.connect(path)
    try:
        return db.execute(sql).fetchall()
    finally:
        db.close()


def test_schema_matches_index_sink(tmp_path):
    pts = [([('host', b'ralph'), ('req.method', b'GET'), ('latency', 16.0),
             ('__dn_metric', 0)], 3),
           ([('timestamp', 1398902400.0), ('__dn_metric', 1)], 5)]
    files = mod_index.write_index(str(tmp_path), METRICS, 'all', pts)
    assert files == [str(tmp_path / 'all')]
    sql = dict(_dump(files[0], "SELECT name, sql FROM sqlite_master "
                               "WHERE type = 'table'"))
    assert sql == {
        'dragnet_config': 'CREATE TABLE dragnet_config(\n'
                          '    key varchar(128) primary key,\n'
                          '    value varchar(128)\n)',
        'dragnet_metrics': 'CREATE TABLE dragnet_metrics(\n'
                           '    id integer,\n    label varchar(64),\n'
                           '    filter varchar(1024),\n'
                           '    params varchar(1024)\n)',
        'dragnet_index_0': 'CREATE TABLE dragnet_index_0(\n'
                           '    host varchar(128),\n'
                           '    req_method varchar(128),\n'
                           '    latency integer,\n    value integer\n)',
        'dragnet_index_1': 'CREATE TABLE dragnet_index_1(\n'
                           '    timestamp integer,\n    value integer\n)',
    }
    assert _dump(files[0], 'SELECT * FROM dragnet_config') == \
        [('version', '2.0.0')]
    assert _dump(files[0], 'SELECT * FROM dragnet_metrics') == [
        (0, 'big', 'null',
         '[{"name":"host","field":"host"},'
         '{"name":"req.method","field":"req.method"},'
         '{"name":"latency","field":"latency","aggr":"quantize"}]'),
        (1, 'daily', '{"eq":["req.method","GET"]}',
         '[{"name":"timestamp","field":"time","date":"",'
         '"aggr":"lquantize","step":86400}]')]
    rows = _dump(files[0], 'SELECT *, typeof(host), typeof(latency) '
                           'FROM dragnet_index_0')
    assert rows == [('ralph', 'GET', 16, 3, 'text', 'integer')]
    assert _dump(files[0], 'SELECT * FROM dragnet_index_1') == \
        [(1398902400, 5)]


def test_interval_files_and_dn_start(tmp_path):
    def pt(ts, v):
        return ([('__dn_ts', ts), ('host', b'h'), ('req.method', b'GET'),
                 ('latency', 1.0), ('__dn_metric', 0)], v)
    pts = [pt(1398902400.0, 1), pt(1398906000.0, 2), pt(1398988800.0, 4)]
    hour = mod_index.write_index(str(tmp_path), METRICS, 'hour', pts)
    assert [os.path.relpath(f, str(tmp_path)) for f in hour] == [
        'by_hour/2014-05-01-00.sqlite', 'by_hour/2014-05-01-01.sqlite',
        'by_hour/2014-05-02-00.sqlite']
    assert _dump(hour[1], 'SELECT * FROM dragnet_config') == \
        [('version', '2.0.0'), ('dn_start', '1398906000')]
    day = mod_index.write_index(str(tmp_path), METRICS, 'day', pts)
    assert [os.path.relpath(f, str(tmp_path)) for f in day] == [
        'by_day/2014-05-01.sqlite', 'by_day/2014-05-02.sqlite']
    assert _dump(day[0], 'SELECT value FROM dragnet_index_0') == [(1,), (2,)]
    assert isinstance(mod_index.write_index(str(tmp_path), METRICS, 'week',
                                            pts), Exception)


def test_written_under_a_temporary_name_then_renamed(tmp_path):
    target = str(tmp_path / 'sub' / 'all')
    sink = mod_index.IndexSink(METRICS, target)
    tmpname = '%s.%d' % (target, os.getpid())
    assert os.path.exists(tmpname) and not os.path.exists(target)
    # (a setting of the writing connection, not of the file)
    assert sink.is_db.execute('PRAGMA synchronous').fetchall() == [(0,)]
    sink.write([([('timestamp', 0.0), ('__dn_metric', 1)], 1)])
    assert sink.close() == target
    assert os.path.exists(target) and not os.path.exists(tmpname)
    assert _dump(target, 'SELECT * FROM dragnet_index_1') == [(0, 1)]


# ---------------------------------------------------------------------------
# the querier (lib/index-query.js)
# ---------------------------------------------------------------------------

def _query(breakdowns=(), filt=None, after=None, before=None):
    q = {'breakdowns': [dict(b) for b in breakdowns]}
    if filt is not None:
        q['filter'] = filt
    if after is not None:
        q['timeAfter'], q['timeBefore'] = after, before
    return mod_query.queryLoad({'query': q})


@pytest.fixture
def querier(tmp_path):
    path = mod_index.write_index(str(tmp_path), METRICS, 'all', [])[0]
    qi = mod_index.IndexQuerier(path)
    assert qi.error is None
    yield qi
    qi.close()


def test_find_metric(querier):
    fm = querier.findMetric
    assert fm(_query([{'name': 'host'}]))['table'] == 'dragnet_index_0'
    # the filtered metric serves only its own filter, compared as text
    assert fm(_query(filt={'eq': ['req.method', 'GET']})) == {
        'datefield': None, 'table': 'dragnet_index_0',
        'ignore_filter': False}
    # time bounds need a date column: only metric 1 has one
    r = fm(_query(filt={'eq': ['req.method', 'GET']}, after='2014-05-01',
                  before='2014-05-02'))
    assert r == {'datefield': 'timestamp', 'table': 'dragnet_index_1',
                 'ignore_filter': True}
    for q in [_query([{'name': 'operation'}]),
              _query(filt={'eq': ['operation', 'x']}),
              _query([{'name': 'host'}], after='2014-05-01',
                     before='2014-05-02'),
              _query([{'name': 'timestamp'}],
                     filt={'eq': ['req.method', 'PUT']}),
              _query(filt={'eq': ['req.method', 'PUT']}, after='2014-05-01',
                     before='2014-05-02')]:
        r = fm(q)
        assert isinstance(r, Exception)
        assert str(r) == 'no metrics available to serve query'


def test_sql(querier):
    assert querier.sql(_query([{'name': 'host'}, {'name': 'req.method'}])) \
        == ('SELECT host,req_method,SUM(value) as value from '
            'dragnet_index_0 WHERE 1 GROUP BY host,req_method')
    assert querier.sql(_query()) == \
        'SELECT SUM(value) as value from dragnet_index_0 WHERE 1 '
    r = querier.sql(_query(
        [{'name': 'timestamp', 'aggr': 'lquantize', 'step': 3600}],
        filt={'eq': ['req.method', 'GET']}, after='2014-05-02T04:05:06.123',
        before='2014-05-02T04:15:10'))
    assert r == ('SELECT timestamp,SUM(value) as value from dragnet_index_1 '
                 'WHERE (timestamp >= 1399003507) AND (timestamp < '
                 '1399004110) GROUP BY timestamp')
    r = querier.sql(_query([{'name': 'host'}], filt={'or': [
        {'eq': ['req.method', 'GET']},
        {'and': [{'ge': ['latency', 10]}, {'ne': ['host', 'a"b']}]}]}))
    assert r == ('SELECT host,SUM(value) as value from dragnet_index_0 '
                 'WHERE (req_method == "GET") OR ((latency >= 10) AND '
                 '(host != "a""b")) GROUP BY host')
    # a date breakdown computed from another field has no column to group
    r = querier.sql(_query([{'name': 'timestamp', 'field': 'time',
                             'date': ''}], filt={'eq': ['req.method',
                                                        'GET']}))
    assert r == ('SELECT SUM(value) as value from dragnet_index_1 '
                 'WHERE 1 ')


@pytest.mark.parametrize('op,c,sql', [
    ('eq', 'GET', 'f == "GET"'), ('ne', 'GET', 'f != "GET"'),
    ('lt', 'GET', 'f < "GET"'), ('le', 'GET', 'f <= "GET"'),
    ('gt', 'GET', 'f > "GET"'), ('ge', 'GET', 'f >= "GET"'),
    ('eq', 200, 'f == 200'), ('ne', 200, 'f != 200'),
    ('lt', 1.5, 'f < 1.5'), ('le', -3, 'f <= -3'), ('gt', 2.0, 'f > 2'),
    ('ge', 0, 'f >= 0'), ('eq', True, 'f == true')])
def test_sql_leaf(op, c, sql):
    assert mod_index.toSqlString({op: ['f', c]}) == sql


def test_sql_leaf_semantics_in_sqlite():
    """What the rendered leaves mean to this sqlite: a double-quoted word is
    a string, and a number matches a text column through type affinity."""
    assert mod_index._double_quoted_strings()
    db = sqlite3.connect(':memory:')
    db.execute('CREATE TABLE t(f varchar(128), n integer, value integer)')
    db.executemany('INSERT INTO t VALUES (?, ?, ?)',
                   [('200', 1, 1), ('GET', 2, 2), ('PUT', 3, 4)])
    for filt, want in [({'eq': ['f', 200]}, 1), ({'eq': ['f', 'GET']}, 2),
                       ({'ne': ['f', 'GET']}, 5), ({'gt': ['f', 'GET']}, 4),
                       ({'ge': ['n', 2]}, 6), ({'lt': ['n', 2.5]}, 3),
                       ({'or': [{'eq': ['f', 'GET']}, {'eq': ['n', 3]}]}, 6),
                       ({}, 7)]:
        got = db.execute('SELECT SUM(value) FROM t WHERE ' +
                         mod_index.toSqlString(filt)).fetchone()[0]
        assert got == want, filt


def test_query_errors(tmp_path):
    ds = datasource_gpu.createDatasource(
        {'dsconfig': {'path': '/dev/null'}, 'findFiles': mod_find.find_files})
    r = ds.query({'query': _query(), 'dryRun': False})
    assert str(r) == 'datasource is missing "indexpath"'
    r = ds.build({'metrics': [], 'interval': 'hour', 'dryRun': False})
    assert str(r) == 'datasource is missing "indexpath"'
    ds = datasource_gpu.createDatasource(
        {'dsconfig': {'path': '/dev/null', 'indexPath': str(tmp_path)},
         'findFiles': mod_find.find_files})
    r = ds.build({'metrics': [], 'interval': 'hour', 'dryRun': False})
    assert str(r) == 'datasource is missing "timefield"'
    r = ds.build({'metrics': [], 'interval': 'all', 'dryRun': False,
                  'timeAfter': 1})
    assert str(r) == 'cannot specify --after without --before'
    r = ds.build({'metrics': [], 'interval': 'all', 'dryRun': False,
                  'timeBefore': 1})
    assert str(r) == 'cannot specify --before without --after'
    ds = datasource_gpu.createDatasource(
        {'dsconfig': {'path': '/dev/null', 'indexPath': str(tmp_path),
                      'timeField': 'time'},
         'findFiles': mod_find.find_files})
    r = ds.build({'metrics': [], 'interval': 'week', 'dryRun': False})
    assert str(r) == 'unsupported interval: "week"'
    r = ds.query({'query': _query(), 'dryRun': False, 'interval': 'week'})
    assert str(r) == 'unsupported interval: "week"'


def test_index_read(tmp_path):
    """indexRead stores tagged json-skinner points as they are."""
    ds = datasource_gpu.createDatasource(
        {'dsconfig': {'path': '/dev/null', 'indexPath': str(tmp_path)},
         'findFiles': mod_find.find_files})
    lines = [json.dumps({'fields': {'__dn_ts': 1398902400, 'timestamp':
                                    1398902460, '__dn_metric': 1},
                         'value': 2}),
             'not json',
             json.dumps({'fields': {'__dn_ts': 1398902400, 'timestamp':
                                    1398902460, '__dn_metric': 1},
                         'value': 3})]
    files = ds.indexRead({'metrics': METRICS, 'interval': 'hour',
                          'input': '\n'.join(lines).encode()})
    assert [os.path.basename(f) for f in files] == ['2014-05-01-00.sqlite']
    assert _dump(files[0], 'SELECT * FROM dragnet_index_1') == \
        [(1398902460, 2), (1398902460, 3)]


# ---------------------------------------------------------------------------
# more metrics than one fan-out plan holds
# ---------------------------------------------------------------------------

NINE = [{'name': 'm%d' % i, 'filter': f, 'breakdowns': b} for i, (f, b) in
        enumerate([
            (None, []),
            (None, [{'name': 'host', 'field': 'host'}]),
            ({'eq': ['req.method', 'GET']},
             [{'name': 'operation', 'field': 'operation'}]),
            (None, [{'name': 'latency', 'field': 'latency',
                     'aggr': 'quantize'}]),
            (None, [{'name': 'req.caller', 'field': 'req.caller'}]),
            ({'ne': ['host', 'ralph']},
             [{'name': 'res.statusCode', 'field': 'res.statusCode'}]),
            (None, [{'name': 'latency', 'field': 'latency',
                     'aggr': 'lquantize', 'step': 100}]),
            (None, [{'name': 'req.method', 'field': 'req.method'},
                    {'name': 'host', 'field': 'host'}]),
            ({'eq': ['operation', 'getstorage']},
             [{'name': 'timestamp', 'field': 'time', 'date': '',
               'aggr': 'lquantize', 'step': 3600}])])]


def test_nine_metrics_in_passes_equal_one_at_a_time(datadir, monkeypatch):
    """build/indexScan split more than MAX_METRICS metrics into passes and
    renumber __dn_metric; checked here with each pass run through the host
    build of the device code."""
    from engines import hostcheck_multi
    calls = []

    def fake_run_plan(plan, files=(), device=0, **_):
        calls.append(len(plan['metrics']))
        per, _ = hostcheck_multi(plan, files)
        pts = []
        for m in sorted(per):
            pts += [(f + [('__dn_metric', m)], v) for f, v in per[m]]
        return datasource_gpu.ScanResult(pts, [{}] * len(plan['metrics']),
                                         files, [{}] * len(plan['metrics']))
    monkeypatch.setattr(datasource_gpu, 'run_plan', fake_run_plan)
    ds = datasource_gpu.createDatasource(
        {'dsconfig': {'path': datadir, 'timeField': 'time',
                      'filter': {'ne': ['req.method', 'HEAD']}},
         'findFiles': mod_find.find_files})
    res = ds.indexScan({'metrics': NINE, 'interval': 'hour',
                        'dryRun': False})
    assert calls == [8, 1]
    files = mod_find.find_files(datadir)
    for i, m in enumerate(NINE):
        got = [(f[:-1], v) for f, v in res.points if f[-1] == ('__dn_metric',
                                                               i)]
        exp = cpu_points({'path': datadir, 'timeField': 'time',
                          'filter': {'ne': ['req.method', 'HEAD']}},
                         [m], 'hour')
        assert got, i
        assert canon_points(got) == canon_points(
            [(f[:-1], v) for f, v in exp]), i
