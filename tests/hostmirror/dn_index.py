"""`dn build` followed by `dn query`, as the reference's index tests run them
(tests/dn/local/tst.index_file.sh, tst.index_fileset.sh), over the GPU
datasource (dragnet_b200.datasource_gpu).

Host-side mirror of the index-related parts of the reference CLI:
  bin/dn:184-186  --interval, default "day" (build and query alike)
  bin/dn:520-545  metric-add (a metric is its name, filter and breakdowns)
  bin/dn:640-694  build
  bin/dn:837-864  query (printed like scan, bin/dn:924-967)
  bin/dn:911-916  --counters

Like hostmirror/dn.py this is TEST INFRASTRUCTURE: it never touches record
data, only index files and the points a query returns.  How an index is built
is the caller's choice (``builder``): the GPU datasource's own build(), or
points computed on the CPU and written with dragnet_b200.index.write_index.
"""

import os
import shutil

from dragnet_b200 import datasource_gpu
from . import dn as mod_dn
from . import find as mod_find

FOREIGN_STAGES = ('FindStart ', 'FindStatter ', 'FindTraverser ',
                  'FindFeedback ', 'PathEnumerator ')

# the stages `dn query --counters` prints, in pipeline order
QUERY_STAGES = ['Index List', 'Index Result Aggregator']

# scan_testcases.sh: the 13 queries both index tests replay first
N_SCAN_TESTCASES = 13


def parse_args(argv):
    """dnParseArgs plus `--interval` / `-i` (default "day")."""
    rest = []
    interval = 'day'
    i = 0
    while i < len(argv):
        a = argv[i]
        if a.startswith('--interval='):
            interval = a.split('=', 1)[1]
        elif a in ('--interval', '-i'):
            i += 1
            interval = argv[i]
        else:
            rest.append(a)
        i += 1
    opts = mod_dn.dnParseArgs(rest)
    opts['interval'] = interval
    return opts


def metric_add(name, argv):
    """`dn metric-add DS NAME [-f FILTER] [-b BREAKDOWNS]` -> the metric."""
    opts = mod_dn.dnParseArgs(argv)
    return {'name': name, 'filter': opts.get('filter') or None,
            'breakdowns': opts['breakdowns']}


def format_counters(counters, flattened):
    """vstream vsDumpCounters for the stages of a query: the same layout as
    hostmirror/dn.py's format_counters."""
    lines = []
    cs = dict(counters)
    stages = list(QUERY_STAGES)
    if flattened and 'Index Result Aggregator' in cs:
        cs['Flattener'] = {
            'ninputs': cs['Index Result Aggregator'].get('noutputs', 0),
            'noutputs': 1}
        stages.append('Flattener')
    for st in stages:
        for name in sorted(cs.get(st, {})):
            if cs[st][name]:
                lines.append('%-18s %-14s %6d' % (st, name + ':',
                                                  cs[st][name]))
    return ''.join(l + '\n' for l in lines)


def dn_query(dsconfig, argv, title='input', interval=None):
    """What `dn query [argv] DS` prints (stdout, then stderr as `2>&1`
    leaves it in the goldens)."""
    options = parse_args(argv)
    if interval is not None:
        options['interval'] = interval
    ds = datasource_gpu.datasourceForConfig(
        {'dsconfig': dsconfig, 'findFiles': mod_find.find_files})
    assert not isinstance(ds, Exception), ds
    qargs = mod_dn.dnQueryConfig(options)
    qargs['interval'] = options['interval']
    res = ds.query(qargs)
    if isinstance(res, Exception):
        raise mod_dn.FatalError(str(res))
    out = mod_dn.render_scan(qargs['query'], options, res.points, title)
    if options.get('counters'):
        out += format_counters(res.counters, not options.get('points'))
    return out


def expected_text(section):
    """A golden section without the counters of the file finder and path
    enumerator, which sit outside the query (golden_harness.py drops them
    the same way)."""
    return '\n'.join(l for l in section['text'].split('\n')
                     if not l.startswith(FOREIGN_STAGES)).rstrip('\n')


def index_file_steps(datadir, indexpath):
    """tst.index_file.sh: (dsconfig, metrics, build interval, number of
    sections queried against that build)."""
    path = os.path.join(datadir, '2014/05-01/one.log')
    ds = {'path': path, 'indexPath': indexpath, 'timeField': 'time'}
    dsf = dict(ds, filter={'eq': ['req.method', 'GET']})
    return [
        (ds, [metric_add('big_metric', [
            '-b', 'host,operation,req.caller,req.method,'
            'latency[aggr=quantize]'])], 'day', N_SCAN_TESTCASES),
        (ds, [metric_add('filtered_metric', [
            '-f', '{ "eq": [ "req.method", "GET" ] }'])], 'day', 1),
        (dsf, [metric_add('bycode', ['-b', 'res.statusCode'])], 'day', 2),
    ]


def index_fileset_steps(datadir, indexpath):
    """tst.index_fileset.sh, as index_file_steps; every query there asks
    for --interval=hour."""
    ds = {'path': datadir, 'indexPath': indexpath, 'timeField': 'time'}
    day = 'timestamp[date,field=time,aggr=lquantize,step=86400]'
    return [
        (ds, [metric_add('myindex', [
            '-b', day + ',host,operation',
            '-b', 'req.caller,req.method,latency[aggr=quantize]'])],
         'hour', N_SCAN_TESTCASES + 2),
        (ds, [metric_add('myindex', [
            '--filter={ "eq": [ "req.method", "GET" ] }', '-b', day])],
         'hour', 1),
        (ds, [metric_add('myindex', [
            '-b', 'timestamp[date,field=time,aggr=lquantize,step=60]'])],
         'hour', 3),
    ]


SUITES = {
    'index_file': (index_file_steps, None, False),
    'index_fileset': (index_fileset_steps, 'hour', True),
}


def replay(suite, goldens, datadir, workdir, builder):
    """Run a suite's builds and queries.  builder(dsconfig, metrics,
    interval) builds the index.  Yields, in order, ('find', actual listing,
    expected listing) after a build whose listing the golden shows, then
    (header, actual, expected) for every query section."""
    steps_fn, query_interval, fresh = SUITES[suite]
    indexpath = os.path.join(workdir, suite)
    sections = goldens['suites'][suite]
    si = 0
    for bi, (ds, metrics, interval, nq) in enumerate(
            steps_fn(datadir, indexpath)):
        if fresh and os.path.exists(indexpath):
            shutil.rmtree(indexpath)        # `rm -rf "$tmpdir"`
        builder(ds, metrics, interval)
        if bi == 0 and goldens['find'][suite]:
            yield ('find', list_index(indexpath), goldens['find'][suite])
        for sec in sections[si:si + nq]:
            act = dn_query(ds, sec['argv'], interval=query_interval)
            yield sec['header'], act.rstrip('\n'), expected_text(sec)
        si += nq
    assert si == len(sections), (si, len(sections))


def list_index(indexpath):
    """`(cd "$tmpdir" && find . -type f | sort -n)`."""
    out = []
    for dp, _, fn in os.walk(indexpath):
        for n in fn:
            out.append('./' + os.path.relpath(os.path.join(dp, n), indexpath))
    return sorted(out)


def empty_build(builder, workdir):
    """The end of tst.index_fileset.sh: a build over /dev/null must leave
    no index directory.  Returns whether the directory exists."""
    indexpath = os.path.join(workdir, 'empty_index')
    ds = {'path': '/dev/null', 'indexPath': indexpath, 'timeField': 'time'}
    builder(ds, [metric_add('myindex', ['-b', 'timestamp[date,field=time]'])],
            'day')
    return os.path.exists(indexpath)
