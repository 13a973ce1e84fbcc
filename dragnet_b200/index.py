"""Dragnet indexes: the sqlite files `dn build` writes and `dn query` reads.

Host-side restatement of the reference's index writer and reader:
  lib/index-sink.js:44-361      IndexSink (one sqlite file)
  lib/datasource-file.js:444-547 indexSink (the "all" file, or one file per
                                hour or day chosen from fields.__dn_ts)
  lib/index-query.js:31-459     IndexQuerier (findMetric, SQL, row decoding)
  lib/dragnet-impl.js:194-270   indexFindParams, metricSerialize

None of this touches record data.  `dn build` reads the raw data once, on the
GPU, as a fan-out scan (one point set per metric, datasource_gpu.run_plan);
what arrives here is the aggregated points, O(#tuples), and what leaves is
the rows of a few sqlite tables.  Query results are re-aggregated through the
library's own reduce (native.result_from_points), as the reference runs its
skinner aggregator over index rows.

Metrics are in their configuration form: {'name', 'filter', 'breakdowns':
[{'name', 'field'[, 'date'][, 'aggr'][, 'step']}]}.  Errors are returned as
Exception instances, following the rest of the package.
"""

import copy
import json
import math
import os
import re
import sqlite3

from . import jsdate
from . import krill
from . import query as mod_query
from .query import DnError

INDEX_VERSION = '2.0.0'


def sqlite3Escape(s):
    """lib/index-sink.js:232-235: '.' and '-' cannot appear in a column."""
    return re.sub(r'[.-]', '_', s)


def _js_value(v):
    if isinstance(v, float) and v == v and not math.isinf(v) and \
            v == int(v) and abs(v) < 1e21:
        return int(v)
    if isinstance(v, dict):
        return {k: _js_value(x) for k, x in v.items()}
    if isinstance(v, list):
        return [_js_value(x) for x in v]
    return v


def js_stringify(v):
    """JSON.stringify for the JSON-parsed values filters and metrics hold:
    compact, key order kept, integral numbers without a fraction."""
    return json.dumps(_js_value(v), separators=(',', ':'), ensure_ascii=False)


def metricSerialize(metric):
    """lib/dragnet-impl.js:243-265 with skipdatasource: the breakdowns as
    stored in dragnet_metrics.params (keys in this order)."""
    out = []
    for b in metric.get('breakdowns') or []:
        e = {'name': b['name'], 'field': b.get('field', b['name'])}
        for k in ('date', 'aggr', 'step'):
            if k in b:
                e[k] = b[k]
        out.append(e)
    return out


# ---------------------------------------------------------------------------
# writing
# ---------------------------------------------------------------------------

def _sql_value(v):
    # The GPU hands discrete values over as UTF-8 bytes (the JS String of the
    # value); sqlite must see them as text, not as blobs.
    if isinstance(v, bytes):
        return v.decode('utf-8', 'replace')
    return v


class IndexSink(object):
    """lib/index-sink.js: one sqlite index file.  The database is written
    under `<filename>.<pid>` and renamed into place by close(), so a reader
    never sees a half-written index."""

    def __init__(self, metrics, filename, config=None):
        self.is_metrics = metrics
        self.is_dbfilename = filename
        self.is_dbtmpfilename = '%s.%d' % (filename, os.getpid())
        os.makedirs(os.path.dirname(filename) or '.', exist_ok=True)
        if os.path.exists(self.is_dbtmpfilename):
            os.unlink(self.is_dbtmpfilename)
        self.is_db = sqlite3.connect(self.is_dbtmpfilename,
                                     isolation_level=None)
        self._init_db(dict(config or {}))

    def _init_db(self, config):
        """lib/index-sink.js:116-230."""
        tables = [
            ('dragnet_config', [('key', 'varchar(128) primary key'),
                                ('value', 'varchar(128)')]),
            ('dragnet_metrics', [('id', 'integer'), ('label', 'varchar(64)'),
                                 ('filter', 'varchar(1024)'),
                                 ('params', 'varchar(1024)')]),
        ]
        configpairs = [('version', INDEX_VERSION)]
        for k, v in config.items():
            assert k != 'version'
            configpairs.append((k, v))
        metricrows = []
        for i, m in enumerate(self.is_metrics):
            metricrows.append((i, m.get('name'),
                               js_stringify(m.get('filter')),
                               js_stringify(metricSerialize(m))))
            cols = {}
            for b in m.get('breakdowns') or []:
                cols[sqlite3Escape(b['name'])] = \
                    'integer' if 'aggr' in b else 'varchar(128)'
            cols['value'] = 'integer'
            tables.append(('dragnet_index_%d' % i, list(cols.items())))

        db = self.is_db
        # The caller syncs the file if it cares (lib/index-sink.js:165-168).
        db.execute('pragma synchronous = off;')
        db.execute('BEGIN')
        for name, cols in tables:
            db.execute('CREATE TABLE %s(\n%s\n);' % (name, ',\n'.join(
                '    %s %s' % c for c in cols)))
        db.executemany('INSERT INTO dragnet_config VALUES (?, ?)',
                       configpairs)
        db.executemany('INSERT INTO dragnet_metrics VALUES (?, ?, ?, ?)',
                       metricrows)

    def write(self, points):
        """Store points, each (fields, value) with fields a dict or a list of
        (name, value) pairs holding every breakdown of metric
        fields['__dn_metric'] (lib/index-sink.js:237-262).  All the rows go
        into the transaction close() commits."""
        rows = [[] for _ in self.is_metrics]
        for fields, value in points:
            f = fields if isinstance(fields, dict) else dict(fields)
            mi = f['__dn_metric']
            assert 0 <= mi < len(self.is_metrics), mi
            row = []
            for b in self.is_metrics[mi].get('breakdowns') or []:
                row.append(_sql_value(f[b['name']]))
            row.append(value)
            rows[mi].append(row)
        for mi, rs in enumerate(rows):
            if rs:
                self.is_db.executemany(
                    'INSERT INTO dragnet_index_%d VALUES (%s)' % (
                        mi, ', '.join('?' * len(rs[0]))), rs)

    def close(self):
        self.is_db.execute('COMMIT')
        self.is_db.close()
        os.rename(self.is_dbtmpfilename, self.is_dbfilename)
        return self.is_dbfilename


INTERVALS = {
    # interval: (length of the ISO-string prefix naming a bucket, what
    # completes that prefix to the bucket's start), lib/datasource-file.js:463
    'hour': (len('2014-07-02T00'), ':00:00Z'),
    'day': (len('2014-07-02'), 'T00:00:00Z'),
}


def interval_bucket(dnts, interval):
    """fields.__dn_ts (seconds) -> (file label, bucket start in seconds),
    lib/datasource-file.js:498-514."""
    prefixlen, suffix = INTERVALS[interval]
    assert isinstance(dnts, (int, float)) and dnts == dnts, dnts
    name = jsdate.to_iso_string(dnts * 1000)[:prefixlen]
    start = jsdate.date_parse_ms(name + suffix) // 1000
    return name.replace('T', '-', 1), start


def index_files_for(indexpath, interval, points):
    """The files write_index creates, as ({path: [points]} in path order,
    {path: dn_start or None}), or an Exception for an unknown interval."""
    if interval == 'all':
        path = os.path.join(indexpath, 'all')
        return {path: list(points)}, {path: None}
    if interval not in INTERVALS:
        return DnError('unsupported interval: "%s"' % interval)
    root = os.path.join(indexpath, 'by_' + interval)
    out = {}
    starts = {}
    for p in points:
        fields = p[0] if isinstance(p[0], dict) else dict(p[0])
        label, start = interval_bucket(fields['__dn_ts'], interval)
        path = os.path.join(root, label + '.sqlite')
        out.setdefault(path, []).append(p)
        starts[path] = start
    return {k: out[k] for k in sorted(out)}, starts


def write_index(indexpath, metrics, interval, points):
    """The index sink of `dn build` (lib/datasource-file.js:444-547): for
    interval 'all', one file `<indexpath>/all`; for 'hour' and 'day', one
    file `by_hour/YYYY-MM-DD-HH.sqlite` or `by_day/YYYY-MM-DD.sqlite` per
    bucket of fields.__dn_ts that holds a point, with `dn_start` (the
    bucket's start, seconds) in its config.  No point, no file: an empty
    input leaves no directory behind.  Returns the files written."""
    r = index_files_for(indexpath, interval, points)
    if isinstance(r, Exception):
        return r
    byfile, starts = r
    written = []
    for path, pts in byfile.items():
        sink = IndexSink(metrics, path, None if starts[path] is None else
                         {'dn_start': starts[path]})
        sink.write(pts)
        written.append(sink.close())
    return written


# ---------------------------------------------------------------------------
# reading
# ---------------------------------------------------------------------------

def indexFindParams(interval, indexpath, after, before):
    """lib/dragnet-impl.js:194-236: where the index files of an interval
    are, and the strftime pattern that prunes them by time."""
    if interval == 'day':
        return {'root': os.path.join(indexpath, 'by_day'),
                'timeformat': '%Y-%m-%d.sqlite', 'after': after,
                'before': before}
    if interval == 'hour':
        return {'root': os.path.join(indexpath, 'by_hour'),
                'timeformat': '%Y-%m-%d-%H.sqlite', 'after': after,
                'before': before}
    if interval == 'all':
        return {'root': os.path.join(indexpath, 'all'), 'timeformat': None,
                'after': None, 'before': None}
    return DnError('unsupported interval: "%s"' % interval)


_DQS = None


def _double_quoted_strings():
    """Whether this sqlite reads "x" as a string when no column is named x.
    The reference's SQL (krill's C-style predicates) relies on that legacy
    behaviour, which sqlite builds may compile out (SQLITE_DQS=0)."""
    global _DQS
    if _DQS is None:
        try:
            sqlite3.connect(':memory:').execute('SELECT "x"').fetchall()
            _DQS = True
        except sqlite3.OperationalError:
            _DQS = False
    return _DQS


C_OPS = {'eq': '==', 'ne': '!=', 'lt': '<', 'le': '<=', 'gt': '>',
         'ge': '>='}


def sql_constant(c):
    """A krill constant as krill's toCStyleString writes it: strings in
    double quotes, numbers and booleans as JavaScript prints them.  Krill is
    not vendored here, so this restates it.  sqlite reads a double-quoted
    word as a string only when no column has that name, and only if built
    to accept double-quoted strings at all; where it is not, strings are
    written in single quotes, which mean the same to sqlite.  A string
    compared with a text column also matches a number: `eq res.statusCode
    200` against a varchar column finds "200" through sqlite's type
    affinity, as it does for the reference."""
    if isinstance(c, bool):
        return 'true' if c else 'false'
    if isinstance(c, (int, float)):
        return mod_query._js_num_str(c)
    if _double_quoted_strings():
        return '"%s"' % c.replace('"', '""')
    return "'%s'" % c.replace("'", "''")


def escapeFilter(filt):
    """lib/index-query.js:414-431: escape every field name, in place."""
    if not filt:
        return
    if 'and' in filt:
        for f in filt['and']:
            escapeFilter(f)
        return
    if 'or' in filt:
        for f in filt['or']:
            escapeFilter(f)
        return
    key = next(iter(filt))
    filt[key][0] = sqlite3Escape(filt[key][0])


def toSqlString(filt):
    """lib/index-query.js:434-454."""
    if not filt:
        return '1'
    if 'and' in filt:
        return ' AND '.join('(%s)' % toSqlString(c) for c in filt['and'])
    if 'or' in filt:
        return ' OR '.join('(%s)' % toSqlString(c) for c in filt['or'])
    key = next(iter(filt))
    field, const = filt[key]
    return '%s %s %s' % (field, C_OPS[key], sql_constant(const))


def _semver_tilde2(v):
    """semver.satisfies(v, '~2'): 2.x.y."""
    m = re.match(r'^v?(\d+)\.(\d+)\.(\d+)$', str(v).strip())
    return bool(m) and int(m.group(1)) == 2


class IndexQuerier(object):
    """lib/index-query.js: runs one query against one index file.  The
    constructor loads the config and metrics (:61-143); check .error."""

    def __init__(self, filename):
        self.qi_dbfilename = filename
        self.qi_config = None
        self.qi_metrics = None
        self.error = None
        try:
            self.qi_db = sqlite3.connect(
                'file:%s?mode=ro' % _uri_path(filename), uri=True)
            self._load()
        except sqlite3.Error as ex:
            self.error = DnError('database error: %s' % ex)

    def _load(self):
        db = self.qi_db
        self.qi_config = {k: v for k, v in
                          db.execute('SELECT * FROM dragnet_config')}
        if 'version' not in self.qi_config:
            self.error = DnError('index missing dragnet "version"')
            return
        if not _semver_tilde2(self.qi_config['version']):
            self.error = DnError('unsupported index version: "%s"' %
                                     self.qi_config['version'])
            return
        self.qi_metrics = []
        for mid, label, filt, params in db.execute(
                'SELECT id, label, filter, params FROM dragnet_metrics'):
            try:
                f = None if filt is None else json.loads(filt)
            except ValueError as ex:
                self.error = DnError('failed to parse filter for metric '
                                         '"%s": %s' % (label, ex))
                return
            try:
                p = {} if params is None else json.loads(params)
            except ValueError as ex:
                self.error = DnError('failed to parse params for metric '
                                         '"%s": %s' % (label, ex))
                return
            self.qi_metrics.append({'qm_id': mid, 'qm_label': label,
                                    'qm_filter': f, 'qm_params': p,
                                    'qm_filter_raw': filt})

    def close(self):
        if getattr(self, 'qi_db', None) is not None:
            self.qi_db.close()
            self.qi_db = None

    def findMetric(self, query):
        """lib/index-query.js:154-263: the first metric that can serve the
        query, as {'datefield', 'table', 'ignore_filter'}, or an error."""
        filter_raw = None
        if query.qc_filter is not None:
            filter_raw = js_stringify(query.qc_filter)
        for met in self.qi_metrics:
            if met['qm_filter'] is not None:
                # A filtered metric holds a subset of the data: it serves
                # only a query with the very same filter.
                if query.qc_filter is None:
                    continue
                if met['qm_filter_raw'] != filter_raw:
                    continue
            datefield = None
            if query.qc_before is not None or query.qc_after is not None:
                dated = [b for b in met['qm_params'] if 'date' in b]
                if not dated:
                    continue
                datefield = dated[0]['name']
            needed = []
            if query.qc_filter is not None and met['qm_filter'] is None:
                needed += krill.createPredicate(query.qc_filter).fields()
            needed += [b['name'] for b in query.qc_breakdowns]
            have = set(b['name'] for b in met['qm_params'])
            if all(f in have for f in needed):
                return {'datefield': datefield,
                        'table': 'dragnet_index_%d' % met['qm_id'],
                        'ignore_filter': met['qm_filter'] is not None}
        return DnError('no metrics available to serve query')

    def sql(self, query):
        """lib/index-query.js:269-338: the SELECT that serves the query."""
        table = self.findMetric(query)
        if isinstance(table, Exception):
            return table
        whenfilter = None
        if table['datefield'] is not None:
            whenfilter = mod_query.queryTimeBoundsFilter(query,
                                                         table['datefield'])
        qfilter = None if table['ignore_filter'] else query.qc_filter
        if qfilter is not None and whenfilter is not None:
            filt = {'and': [copy.deepcopy(qfilter), whenfilter]}
        elif whenfilter is not None:
            filt = whenfilter
        elif qfilter is not None:
            filt = copy.deepcopy(qfilter)
        else:
            filt = {}
        escapeFilter(filt)
        # A date breakdown whose field differs from its name is computed from
        # the raw field during a scan; the index has no such column.
        groupby = [sqlite3Escape(b['name']) for b in query.qc_breakdowns
                   if 'date' not in b or b['field'] == b['name']]
        columns = groupby + ['SUM(value) as value']
        sql = 'SELECT %s from %s WHERE %s ' % (','.join(columns),
                                               table['table'],
                                               toSqlString(filt))
        if groupby:
            sql += 'GROUP BY ' + ','.join(groupby)
        return sql

    def run(self, query):
        """Rows of the query as [([col, ...], value)], one column per query
        breakdown, ready for native.result_from_points: discrete columns
        as UTF-8 bytes, quantized ones as numbers (lib/index-query.js:382-405
        deserializeRow)."""
        sql = self.sql(query)
        if isinstance(sql, Exception):
            return sql
        try:
            cur = self.qi_db.execute(sql)
            names = [d[0] for d in cur.description]
            rows = cur.fetchall()
        except sqlite3.Error as ex:
            return DnError('executing query "%s": %s' % (sql, ex))
        out = []
        for r in rows:
            row = dict(zip(names, r))
            value = row['value']
            if value is None:       # SUM() over no rows is NULL
                value = 0
            cols = []
            for b in query.qc_breakdowns:
                col = sqlite3Escape(b['field'])
                cols.append(_point_col(row[col] if col in row else _MISSING,
                                       'aggr' in b))
            out.append((cols, int(value)))
        return out


def query_indexes(files, query):
    """Run the query against every index file and aggregate the rows of all
    of them (lib/datasource-file.js:573-691).  Each file's rows are first
    aggregated on their own, as the reference's per-file "Index Aggregator"
    does: its rows hold one entry per bucket of the index, which the query
    may bucket more coarsely (minutes into days, say).  Both steps are the
    library's reduce, which takes string columns as they are and
    re-bucketizes numeric ones.  Returns (points, counters) or an error."""
    from . import native
    # (the reduce needs only the columns: which are bucketized, and how)
    plan = native.Plan(mod_query.scan_plan_json(
        mod_query.QueryConfig(breakdowns=query.qc_breakdowns)))
    try:
        listed = []
        for f in files:
            qi = IndexQuerier(f)
            try:
                if qi.error is not None:
                    return DnError('index "%s"' % f, qi.error)
                rows = qi.run(query)
            finally:
                qi.close()
            if isinstance(rows, Exception):
                return DnError('index "%s" query' % f, rows)
            res = native.result_from_points(plan, rows)
            try:
                listed += res.points()
            finally:
                res.close()
        res = native.result_from_points(plan, listed)
        try:
            out = res.points()
        finally:
            res.close()
    finally:
        plan.close()
    names = [b['name'] for b in query.qc_breakdowns]
    points = [(list(zip(names, cols)), value) for cols, value in out]
    n = len(listed)
    counters = {}
    if n:
        counters['Index List'] = {'ninputs': n, 'noutputs': n}
        counters['Index Result Aggregator'] = {'ninputs': n}
    if points:
        counters.setdefault('Index Result Aggregator', {})['noutputs'] = \
            len(points)
    return points, counters


_MISSING = object()


def _point_col(v, numeric):
    """One index cell as a point column.  A quantized cell is a bucket
    minimum; sqlite stores a NaN one as NULL, which becomes NaN again.  A
    discrete cell is what JavaScript's String() makes of it."""
    if numeric:
        if isinstance(v, (int, float)) and not isinstance(v, bool):
            return float(v)
        try:
            return float(v)
        except (TypeError, ValueError):
            return float('nan')
    if v is _MISSING:
        return b'undefined'
    if v is None:
        return b'null'
    if isinstance(v, (int, float)):
        return mod_query._js_num_str(v).encode()
    if isinstance(v, bytes):
        return v
    return v.encode('utf-8')


def _uri_path(path):
    from urllib.parse import quote
    return quote(os.path.abspath(path))
