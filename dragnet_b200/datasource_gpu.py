"""The GPU datasource: what `datasourceForConfig` returns for backend "gpu"
(and, as a drop-in, for "file").

Host-side mirror of the reference's Datasource interface for the scan path:
  lib/dragnet.js:288-304        datasourceForConfig (backend dispatch)
  lib/datasource-file.js:31-56  createDatasource / DatasourceFile fields
  lib/datasource-file.js:72-108 scan({query, dryRun})
  lib/datasource-file.js:124-192 scanInit (timeField check, dry run)
  lib/datasource-file.js:307-433 build / indexScanImpl (fan-out scan)
  lib/datasource-file.js:549-566 checkTimeArgs / checkIndexArgs
  lib/datasource-file.js:573-618 query (index files -> points)
  lib/datasource-file.js:729-746 indexRead
The reference returns an object-mode stream of skinner points; here scan()
returns a ScanResult holding the points, the per-stage counters and the list of
files.  build() reads the raw data on the GPU and writes the sqlite indexes
(index.py); query() and indexRead() never read raw data.
"""

import json
import time

from . import index as mod_index
from . import native
from . import query as mod_query

# Metrics one fan-out plan may hold (csrc/plan.h MAX_METRICS).
MAX_METRICS = 8


class DsError(Exception):
    pass


class ScanResult(object):
    def __init__(self, points, counters, files, flat=None, stats=None):
        self.points = points        # [([(name, bytes|float)...], value)]
        self.counters = counters    # {stage: {counter: n}} vstream style
        self.files = files
        self.flat_counters = flat   # dng_counters as a dict
        self.stats = stats
        self.index_files = None     # build(): the index files written
        self.timing = None          # build(): {'scan_s', 'index_s'}


def stage_counters(plan, c, npoints):
    """dng_counters -> vstream-style per-stage counters (bin/dn:911-916)."""
    out = {}

    def put(stage, name, n):
        if n:
            out.setdefault(stage, {})[name] = n

    n = c['lines']
    put('json parser', 'ninputs', n)
    put('json parser', 'invalid json', c['invalid_json'])
    n -= c['invalid_json']
    put('json parser', 'noutputs', n)
    if plan.get('format', 'json') == 'json':
        put('SkinnerAdapterStream', 'ninputs', n)
        put('SkinnerAdapterStream', 'noutputs', n)
    else:
        put('json parser', 'invalid point', c.get('invalid_point', 0))
        n -= c.get('invalid_point', 0)

    def filt(stage, present, kf, ke):
        nonlocal n
        if not present:
            return
        put(stage, 'ninputs', n)
        put(stage, 'nfilteredout', c[kf])
        put(stage, 'nfailedeval', c[ke])
        n -= c[kf] + c[ke]
        put(stage, 'noutputs', n)

    filt('Datasource filter', plan.get('ds_filter'), 'ds_filtered',
         'ds_failedeval')
    filt('User filter', plan.get('filter'), 'user_filtered',
         'user_failedeval')
    if plan.get('synthetic'):
        put('Datetime parser', 'ninputs', n)
        put('Datetime parser', 'undef', c['synth_undef'])
        put('Datetime parser', 'baddate', c['synth_baddate'])
        n -= c['synth_undef'] + c['synth_baddate']
        put('Datetime parser', 'noutputs', n)
    filt('Time filter', plan.get('time_bounds'), 'time_filtered',
         'time_failedeval')
    # (what is left must be what the aggregator counted)
    naggr = c.get('aggr_ninputs', c.get('aggr'))
    if naggr is not None and n != naggr:
        raise DsError('stage counters do not add up: %r' % (c,))
    put('Aggregator', 'ninputs', n)
    put('Aggregator', 'noutputs', npoints)
    return out


GZIP_MAGIC = b'\x1f\x8b\x08'
COMPRESSIONS = (None, 'none', 'gzip', 'bzip2')


def is_gzip(path):
    """Whether the file starts as a gzip member of DEFLATE data does."""
    with open(path, 'rb') as f:
        return f.read(3) == GZIP_MAGIC


def is_bzip2(path):
    """Whether the file starts as a bzip2 stream does: BZh and a level
    digit 1-9."""
    with open(path, 'rb') as f:
        head = f.read(4)
    return len(head) == 4 and head[:3] == b'BZh' and 0x31 <= head[3] <= 0x39


def run_plan(plan, files=(), chunks=None, device=0, device_buffers=None,
             templates=None, devices=None, compression=None):
    """Drive one scan through the C ABI.  Input is any of: files (read by the
    library), host byte chunks, or (ptr, len) device buffers.  devices: more
    than one device index -> one scan over all of them, the files cut into a
    byte range per device (files only); its stats are per shard.
    compression 'gzip': files that start with 1f 8b 08 are inflated on the
    device (dng_scan_feed_gzip), others read as they are; 'bzip2': files
    that start with BZh and a level 1-9 are decoded on the device
    (dng_scan_feed_bzip2), others read as they are; one device only."""
    import json
    multi = devices is not None and len(devices) > 1
    gzip = compression == 'gzip'
    bzip2 = compression == 'bzip2'
    if (gzip or bzip2) and multi:
        raise DsError('compression "%s" is not supported on a scan over '
                      'several devices' % compression)
    p = native.Plan(json.dumps(plan, separators=(',', ':')))
    if devices and not multi:
        device = devices[0]
    s = native.Scan(p, devices=list(devices)) if multi else \
        native.Scan(p, device)
    try:
        if templates is not None:
            s.set_templates(templates)
        for f in files:
            if gzip and is_gzip(f):
                s.feed_gzip(f)
            elif bzip2 and is_bzip2(f):
                s.feed_bzip2(f)
            else:
                s.feed_file(f)
        for c in (chunks or ()):
            s.feed(c)
        for ptr, n in (device_buffers or ()):
            s.feed_device(ptr, n)
        res = s.finish()
        flat = s.counters()
        if multi:
            stats = {'devices': list(devices), 'shards': []}
            for sh in s.shards(len(devices)):
                one = sh.kernel_stats()
                one.update(sh.template_stats())
                one.update(sh.read_stats())
                stats['shards'].append(one)
        else:
            stats = s.kernel_stats()
            stats.update(s.template_stats())
            stats.update(s.read_stats())
            if gzip:
                stats.update(s.gzip_stats())
                stats.update(s.gzip_split_stats())
            if bzip2:
                stats.update(s.bzip2_stats())
        pts = []
        if 'metrics' in plan:
            # fan-out: points are tagged like the reference tags them
            # (fields.__dn_metric = qi, lib/datasource-file.js:412-419)
            mflat = [s.counters(m) for m in range(len(plan['metrics']))]
            for m, cols, value in res.points(with_metric=True):
                names = [b['name'] for b in plan['metrics'][m]['breakdowns']]
                pts.append((list(zip(names, cols)) + [('__dn_metric', m)],
                            value))
            res.close()
            counters = []
            for m, mp in enumerate(plan['metrics']):
                one = dict(mp, format=plan.get('format', 'json'),
                           ds_filter=plan.get('ds_filter'))
                npts = sum(1 for f, _ in pts if f[-1][1] == m)
                counters.append(stage_counters(one, mflat[m], npts))
            return ScanResult(pts, counters, list(files), mflat, stats)
        names = [b['name'] for b in plan['breakdowns']]
        for cols, value in res.points():
            pts.append((list(zip(names, cols)), value))
        res.close()
        return ScanResult(pts, stage_counters(plan, flat, len(pts)),
                          list(files), flat, stats)
    finally:
        s.close()
        p.close()


class DatasourceGpu(object):
    def __init__(self, args):
        dsconfig = args['dsconfig']
        bc = dsconfig.get('backend_config') or dsconfig
        self.ds_format = dsconfig.get('dataFormat') or \
            dsconfig.get('ds_format') or 'json'
        self.ds_timeformat = bc.get('timeFormat') or None
        self.ds_timefield = bc.get('timeField') or None
        self.ds_datapath = bc.get('path')
        self.ds_indexpath = bc.get('indexPath') or None
        self.ds_filter = dsconfig.get('filter') or None
        self.ds_device = dsconfig.get('device', 0)
        # a list of device indices, or "all": one scan over all of them
        # (files cut by bytes, tallies merged exactly), else ds_device alone
        self.ds_devices = dsconfig.get('devices')
        # "gzip" / "bzip2": files of that format among the input are
        # decoded on the device
        self.ds_compression = bc.get('compression')
        if self.ds_compression == 'none':
            self.ds_compression = None
        # (root, timeFormat, after_ms, before_ms) -> [paths]: the reference's
        # own enumeration (lib/datasource-file.js:218-246 findStream), which
        # the real integration keeps; the tests pass their mirror of it
        self.ds_find = args.get('findFiles')

    def close(self):
        pass

    def _devices(self):
        if self.ds_devices == 'all':
            return list(range(native.lib().dng_device_count()))
        return self.ds_devices

    def _run(self, plan, files):
        devices = self._devices()
        if self.ds_compression in ('gzip', 'bzip2') and devices and \
                len(devices) > 1:
            return DsError('compression "%s" is not supported on a scan '
                           'over several devices' % self.ds_compression)
        return run_plan(plan, files=files, device=self.ds_device,
                        devices=devices, compression=self.ds_compression)

    def scan(self, args):
        """lib/datasource-file.js:72-108.  Returns ScanResult or an Error."""
        query = args['query']
        dry = args['dryRun']
        assert isinstance(dry, bool)
        if self.ds_timefield is None and (query.qc_before is not None or
                                          query.qc_after is not None):
            return DsError('datasource is missing "timefield" for "before" '
                           'and "after" constraints')
        if self.ds_format not in ('json', 'json-skinner'):
            return DsError('unsupported format: "%s"' % self.ds_format)
        if self.ds_find is None:
            return DsError('no file enumerator ("findFiles")')
        files = self.ds_find(self.ds_datapath, self.ds_timeformat,
                             query.qc_after, query.qc_before)
        if dry:
            return ScanResult([], {}, files)
        plan = mod_query.scan_plan(query, ds_filter=self.ds_filter,
                                   time_field=self.ds_timefield,
                                   data_format=self.ds_format)
        return self._run(plan, files)

    def checkTimeArgs(self, args):
        """lib/datasource-file.js:549-556."""
        after, before = args.get('timeAfter'), args.get('timeBefore')
        if after is not None and before is None:
            return DsError('cannot specify --after without --before')
        if before is not None and after is None:
            return DsError('cannot specify --before without --after')
        return None

    def checkIndexArgs(self, args, needsindex, needstime):
        """lib/datasource-file.js:558-566."""
        if needsindex and self.ds_indexpath is None:
            return DsError('datasource is missing "indexpath"')
        if needstime and args['interval'] != 'all' and \
                self.ds_timefield is None:
            return DsError('datasource is missing "timefield"')
        return None

    def _fanout(self, metrics, interval, after, before, files):
        """Every metric over the raw data, each point tagged ('__dn_metric',
        i).  A plan holds at most MAX_METRICS metrics, so more are computed in
        passes of that many, and each pass reads the input again."""
        queries = [mod_query.metricQuery(m, after, before, interval,
                                         self.ds_timefield)
                   for m in metrics]
        pts, counters, flats, stats = [], [], [], []
        for base in range(0, len(queries), MAX_METRICS):
            plan = mod_query.scan_plan_multi(
                queries[base:base + MAX_METRICS], ds_filter=self.ds_filter,
                time_field=self.ds_timefield, data_format=self.ds_format)
            r = self._run(plan, files)
            if isinstance(r, DsError):
                return r
            for fields, value in r.points:
                fields[-1] = ('__dn_metric', base + fields[-1][1])
                pts.append((fields, value))
            counters += r.counters
            flats += r.flat_counters
            stats.append(r.stats)
        return ScanResult(pts, counters, list(files), flats,
                          stats[0] if len(stats) == 1 else stats)

    def indexScan(self, args):
        """The scan half of build/index-scan (lib/datasource-file.js:321-433):
        one pass over the raw data computing every metric (one pass per
        MAX_METRICS metrics); returns the points an IndexSink would store,
        each tagged ('__dn_metric', i).  args: metrics [{'filter',
        'breakdowns'}], interval, dryRun, timeAfter, timeBefore (ms)."""
        after, before = args.get('timeAfter'), args.get('timeBefore')
        if self.ds_timefield is None and (args['interval'] != 'all' or
                                          after or before):
            return DsError('datasource is missing "timefield"')
        if self.ds_find is None:
            return DsError('no file enumerator ("findFiles")')
        files = self.ds_find(self.ds_datapath, self.ds_timeformat,
                             after, before)
        if args.get('dryRun'):
            return ScanResult([], {}, files)
        return self._fanout(args['metrics'], args['interval'], after, before,
                            files)

    def build(self, args):
        """`dn build` (lib/datasource-file.js:307-433): the fan-out scan of
        every metric on the GPU, with the datasource filter applied, then
        the points into the index files of args['interval'] under the
        datasource's indexPath.  args: metrics (configuration form, each with
        a 'name'), interval ('all', 'hour' or 'day'), dryRun, timeAfter,
        timeBefore (ms).  A dry run only lists the input files.  Returns a
        ScanResult whose .index_files are the files written and whose
        .timing splits the wall time into the scan and the sqlite writes."""
        after, before = args.get('timeAfter'), args.get('timeBefore')
        err = self.checkTimeArgs(args) or \
            self.checkIndexArgs(args, True, True)
        if err is not None:
            return err
        if args['interval'] not in ('all',) + tuple(mod_index.INTERVALS):
            return DsError('unsupported interval: "%s"' % args['interval'])
        if self.ds_format not in ('json', 'json-skinner'):
            return DsError('unsupported format: "%s"' % self.ds_format)
        if self.ds_find is None:
            return DsError('no file enumerator ("findFiles")')
        files = self.ds_find(self.ds_datapath, self.ds_timeformat,
                             after, before)
        if args.get('dryRun'):
            return ScanResult([], {}, files)
        t0 = time.perf_counter()
        res = self._fanout(args['metrics'], args['interval'], after, before,
                           files)
        if isinstance(res, DsError):
            return res
        t1 = time.perf_counter()
        written = mod_index.write_index(self.ds_indexpath, args['metrics'],
                                        args['interval'], res.points)
        if isinstance(written, Exception):
            return DsError(str(written))
        res.index_files = written
        res.timing = {'scan_s': t1 - t0,
                      'index_s': time.perf_counter() - t1}
        return res

    def query(self, args):
        """`dn query` (lib/datasource-file.js:573-618): the index files of
        args['interval'] (default 'all') that the query's time bounds
        select, the query run against each, and the rows of all of them
        aggregated as the query asks.  The counters are the reference's
        'Index List' and 'Index Result Aggregator' stage counters."""
        query = args['query']
        err = self.checkTimeArgs(args) or \
            self.checkIndexArgs(args, True, False)
        if err is not None:
            return err
        fp = mod_index.indexFindParams(args.get('interval') or 'all',
                                       self.ds_indexpath, query.qc_after,
                                       query.qc_before)
        if isinstance(fp, Exception):
            return DsError(str(fp))
        if self.ds_find is None:
            return DsError('no file enumerator ("findFiles")')
        files = self.ds_find(fp['root'], fp['timeformat'], fp['after'],
                             fp['before'])
        if args['dryRun']:
            return ScanResult([], {}, files)
        r = mod_index.query_indexes(files, query)
        if isinstance(r, Exception):
            return DsError(str(r))
        points, counters = r
        return ScanResult(points, counters, files)

    def indexRead(self, args):
        """`dn index-read` (lib/datasource-file.js:729-746): json-skinner
        points that already carry fields.__dn_metric (args['input']: bytes,
        or an iterable of lines) into the index files of args['interval'],
        stored as they are, without aggregating them again.  Lines that are
        not JSON are skipped, as the reference's json-skinner parser drops
        them.  Returns the files written."""
        if args['interval'] not in ('all',) + tuple(mod_index.INTERVALS):
            return DsError('unsupported interval: "%s"' % args['interval'])
        err = self.checkIndexArgs(args, True, False)
        if err is not None:
            return err
        data = args['input']
        lines = data.split(b'\n') if isinstance(data, bytes) else data
        points = []
        nmetrics = len(args['metrics'])
        for line in lines:
            if isinstance(line, bytes):
                line = line.decode('utf-8', 'replace')
            if not line.strip():
                continue
            try:
                p = json.loads(line)
            except ValueError:
                continue
            if not isinstance(p, dict) or \
                    not isinstance(p.get('fields'), dict):
                continue
            mi = p['fields'].get('__dn_metric')
            if not isinstance(mi, int) or isinstance(mi, bool) or \
                    not 0 <= mi < nmetrics:
                return DsError('point without a valid "__dn_metric": %s'
                               % line.strip())
            points.append((p['fields'], p.get('value')))
        written = mod_index.write_index(self.ds_indexpath, args['metrics'],
                                        args['interval'], points)
        if isinstance(written, Exception):
            return DsError(str(written))
        return written


def createDatasource(args):
    dsconfig = args['dsconfig']
    bc = dsconfig.get('backend_config') or dsconfig
    if not isinstance(bc.get('path'), str):
        return DsError('expected datasource "path" to be a string')
    devs = dsconfig.get('devices')
    if devs is not None and devs != 'all' and (
            not isinstance(devs, (list, tuple)) or not devs or
            not all(isinstance(d, int) and not isinstance(d, bool) and d >= 0
                    for d in devs)):
        return DsError('expected datasource "devices" to be "all" or a '
                       'non-empty list of device indices')
    comp = bc.get('compression')
    if comp not in COMPRESSIONS:
        return DsError('unsupported compression: "%s"' % (comp,))
    return DatasourceGpu(args)


def datasourceForConfig(args):
    """lib/dragnet.js:288-304 with the one added branch INTEGRATION.md shows."""
    bename = args['dsconfig'].get('backend', 'gpu')
    if bename in ('gpu', 'file'):
        return createDatasource(args)
    return DsError('unknown datasource backend: "%s"' % bename)
