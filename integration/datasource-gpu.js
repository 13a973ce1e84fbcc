/*
 * lib/datasource-gpu.js: Datasource backend that runs `scan` on an H100 through
 * libdragnet_gpu.so (via the dragnet_gpu N-API addon, integration/addon.cc).
 *
 * NOT EXECUTED IN THIS REPOSITORY: node is not installed in the build image.
 * It is the reference-side half of the drop-in boundary and mirrors
 * lib/datasource-file.js:31-108 and :307-433 of the reference: scan(), and
 * the raw-data pass of build() and indexScan(), run on the GPU; query() and
 * indexRead(), which read only index files and points, stay on the file
 * backend.  Add to lib/dragnet.js:datasourceForConfig:
 *
 *     if (bename == 'gpu')
 *             return (mod_datasource_gpu.createDatasource(args));
 *
 * A host that keeps a directory for compiled scan kernels passes it as
 * args.jitCacheDir, next to log and dsconfig: later `dn` processes then load
 * the kernels instead of compiling them (dng_jit_cache_dir).  It is a setting
 * of the process, not of a datasource, so the first datasource created sets
 * it; without it the environment's DNG_JIT_CACHE_DIR applies.
 */

var mod_assertplus = require('assert-plus');
var mod_fs = require('fs');
var mod_stream = require('stream');
var mod_vasync = require('vasync');
var mod_vstream = require('vstream');
var VError = require('verror');

var mod_datasource_file = require('./datasource-file');
var mod_dragnet_impl = require('./dragnet-impl');
var dragnet_gpu = require('dragnet_gpu');	/* the N-API addon */
var jitCacheDirSet = false;

exports.createDatasource = function createDatasource(args)
{
	var filecfg, fileds, comp;

	mod_assertplus.object(args.dsconfig);
	mod_assertplus.optionalString(args.jitCacheDir, 'args.jitCacheDir');
	if (typeof (args.dsconfig.ds_backend_config.path) != 'string')
		return (new VError('expected datasource "path" to be a string'));
	comp = args.dsconfig.ds_backend_config.compression;
	if (comp !== undefined && comp !== 'none' && comp !== 'gzip' &&
	    comp !== 'bzip2')
		return (new VError('unsupported compression: "%s"', comp));
	/*
	 * "all" on a host with one GPU is a scan on that GPU and reads
	 * compressed files, as in DatasourceGpu in Python; on several GPUs the
	 * scan over all of them refuses feedGzip and feedBzip2 with DNG_EINVAL.
	 */
	if ((comp === 'gzip' || comp === 'bzip2') &&
	    Array.isArray(args.dsconfig.ds_backend_config.devices) &&
	    args.dsconfig.ds_backend_config.devices.length > 1)
		return (new VError('compression "%s" is not supported on a ' +
		    'scan over several devices', comp));

	/* (before the first scan is opened) */
	if (args.jitCacheDir !== undefined && !jitCacheDirSet) {
		dragnet_gpu.jitCacheDir(args.jitCacheDir);
		jitCacheDirSet = true;
	}

	/* query/indexRead and the index files stay on the file backend */
	filecfg = Object.create(args.dsconfig);
	filecfg.ds_backend = 'file';
	fileds = mod_datasource_file.createDatasource(
	    { 'dsconfig': filecfg, 'log': args.log });
	if (fileds instanceof Error)
		return (fileds);
	return (new DatasourceGpu(args, fileds));
};

function DatasourceGpu(args, fileds)
{
	this.ds_file = fileds;
	this.ds_format = args.dsconfig.ds_format;
	this.ds_timefield = args.dsconfig.ds_backend_config.timeField || null;
	this.ds_filter = args.dsconfig.ds_filter || null;
	this.ds_device = args.dsconfig.ds_backend_config.device || 0;
	/*
	 * "devices": an array of device indices or "all": one scan over all of
	 * them, the files cut into one byte range per device and the tallies
	 * merged exactly (dng_scan_open_devices); without it, "device" alone.
	 */
	if (args.dsconfig.ds_backend_config.devices !== undefined)
		this.ds_device = args.dsconfig.ds_backend_config.devices;
	/*
	 * "compression": "gzip": files that start with 1f 8b 08 (rotated logs)
	 * are inflated on the GPU (dng_scan_feed_gzip); "bzip2": files that
	 * start with BZh and a level 1-9 are decoded on the GPU
	 * (dng_scan_feed_bzip2).  Any other file (the live log beside them) is
	 * read as it is.
	 */
	this.ds_compression = args.dsconfig.ds_backend_config.compression;
	if (this.ds_compression !== 'gzip' && this.ds_compression !== 'bzip2')
		this.ds_compression = null;
	this.ds_log = args.log;
}

/*
 * Feed one file to a scan: feedGzip() or feedBzip2() for a file of the
 * datasource's compression, else feedFile().  All are N-API async work
 * items.
 */
DatasourceGpu.prototype.feedPath = function (scan, path, callback)
{
	var comp = this.ds_compression;

	if (comp === null) {
		scan.feedFile(path, callback);
		return;
	}
	mod_fs.open(path, 'r', function (err, fd) {
		if (err) {
			callback(err);
			return;
		}
		var head = Buffer.alloc(4);
		mod_fs.read(fd, head, 0, 4, 0, function (rerr, n) {
			mod_fs.close(fd, function () {});
			if (rerr) {
				callback(rerr);
				return;
			}
			if (comp === 'gzip' && n >= 3 && head[0] == 0x1f &&
			    head[1] == 0x8b && head[2] == 0x08)
				scan.feedGzip(path, callback);
			else if (comp === 'bzip2' && n == 4 && head[0] == 0x42 &&
			    head[1] == 0x5a && head[2] == 0x68 &&
			    head[3] >= 0x31 && head[3] <= 0x39)
				scan.feedBzip2(path, callback);
			else
				scan.feedFile(path, callback);
		});
	});
};

/* metrics one fan-out plan may hold (MAX_METRICS, csrc/plan.h) */
var MAX_METRICS = 8;

[ 'close', 'query', 'indexRead' ].forEach(function (m) {
	DatasourceGpu.prototype[m] = function () {
		return (this.ds_file[m].apply(this.ds_file, arguments));
	};
});

/*
 * scan(): same contract as DatasourceFile.scan (lib/datasource-file.js:72-108):
 * returns an object-mode Readable of skinner points, then 'end'.
 */
DatasourceGpu.prototype.scan = function (args)
{
	var self = this;
	var query = args.query;
	var scanctx, plan, scan, out;

	/* file enumeration, --dry-run and the timeField check are unchanged */
	scanctx = this.ds_file.scanInit({
	    'filter': null, 'dryRun': args.dryRun,
	    'timeBefore': query.qc_before, 'timeAfter': query.qc_after
	});
	if (scanctx instanceof Error)
		return (mod_dragnet_impl.asyncError(scanctx));
	if (args.dryRun)
		return (scanctx.outstream);

	/* the plan JSON is just the QueryConfig + datasource properties */
	plan = queryPlan(query, this.ds_timefield);
	plan.format = this.ds_format;
	plan.ds_filter = this.ds_filter;
	plan = JSON.stringify(plan);

	out = mod_vstream.wrapStream(new mod_stream.PassThrough(
	    { 'objectMode': true, 'highWaterMark': 0 }), 'Aggregator');
	/* throws on error; the names label the point fields, in order */
	scan = dragnet_gpu.scanOpen(plan, this.ds_device,
	    query.qc_breakdowns.map(function (b) { return (b.name); }));

	/*
	 * Feed files as they are found.  feedFile() is an N-API async work item:
	 * read(2) into pinned buffers + cudaMemcpyAsync run on a worker thread,
	 * the event loop is never blocked.
	 */
	scanctx.findstream.on('data', function (fileinfo) {
		if (fileinfo.error)
			return;
		scanctx.findstream.pause();
		self.feedPath(scan, fileinfo.path, function (err) {
			if (err)
				out.emit('error', err);
			else
				scanctx.findstream.resume();
		});
	});
	scanctx.findstream.on('end', function () {
		scan.finish(function (err, points, counters) {
			if (err) {
				out.emit('error', err);
				return;
			}
			/* counters mirror the vstream per-stage counters */
			self.ds_counters = counters;
			points.forEach(function (p) { out.write(p); });
			out.end();
			scan.close();
		});
	});
	return (out);
};

/*
 * What a scan of one query computes: its filter, synthetic date fields, time
 * bounds and breakdowns, as the plan JSON names them.
 */
function queryPlan(query, timefield)
{
	var synthetic, bounds, tf;

	synthetic = query.qc_synthetic.map(function (s) {
		return ({ 'name': s.name, 'field': s.field });
	});
	bounds = null;
	/* (as lib/stream-scan.js:62: either bound asks for the time filter) */
	if (query.qc_before !== null || query.qc_after !== null) {
		synthetic.push({ 'name': 'dn_ts', 'field': timefield });
		tf = mod_dragnet_impl.queryTimeBoundsFilter(query, 'dn_ts');
		bounds = { 'field': 'dn_ts',
		    'ge': tf.and[0].ge[1], 'lt': tf.and[1].lt[1] };
	}
	return ({
	    'filter': query.qc_filter,
	    'synthetic': synthetic,
	    'time_bounds': bounds,
	    'breakdowns': query.qc_breakdowns
	});
}

/*
 * build(): same contract as DatasourceFile.build (lib/datasource-file.js:
 * 307-320): the datasource filter applies, the points go into the file
 * backend's own index sink.
 */
DatasourceGpu.prototype.build = function (args, callback)
{
	var scanargs, key;

	mod_assertplus.ok(!args.hasOwnProperty('sink'));
	mod_assertplus.ok(!args.hasOwnProperty('filter'));
	scanargs = {};
	for (key in args)
		scanargs[key] = args[key];
	scanargs.filter = this.ds_filter;
	return (this.indexScanImpl(scanargs, callback));
};

/*
 * indexScan(): same contract as DatasourceFile.indexScan (:698-723): the
 * tagged points, into a PassThrough instead of index files.
 */
DatasourceGpu.prototype.indexScan = function (args)
{
	var sink = new mod_stream.PassThrough({
	    'objectMode': true,
	    'highWaterMark': 128
	});

	this.indexScanImpl({
	    'dryRun': false,
	    'filter': args.filter,
	    'interval': args.interval,
	    'metrics': args.metrics,
	    'sink': sink,
	    'timeAfter': args.timeAfter,
	    'timeBefore': args.timeBefore
	}, function (err) {
		if (err)
			sink.emit('error', err);
	});
	return (sink);
};

/*
 * The raw-data pass of build and indexScan (lib/datasource-file.js:322-433):
 * one fan-out scan computes every metric, and each point is written to the
 * sink tagged fields.__dn_metric.  A plan holds at most MAX_METRICS metrics,
 * so more are computed in passes of that many; each pass reads the input
 * files again.
 */
DatasourceGpu.prototype.indexScanImpl = function (args, callback)
{
	var self = this;
	var fileds = this.ds_file;
	var error, scanctx, sink, queries, passes, paths, i;

	mod_assertplus.arrayOfObject(args.metrics, 'args.metrics');
	mod_assertplus.bool(args.dryRun, 'args.dryRun');
	mod_assertplus.string(args.interval, 'args.interval');

	error = fileds.checkTimeArgs(args);
	if (error === null)
		error = fileds.checkIndexArgs(args, args.sink === undefined, true);
	if (error === null) {
		/* (the datasource filter goes into the plan) */
		scanctx = fileds.scanInit({
		    'filter': null,
		    'dryRun': args.dryRun,
		    'timeAfter': args.timeAfter,
		    'timeBefore': args.timeBefore
		});
		if (scanctx instanceof Error)
			error = scanctx;
	}
	if (error !== null) {
		setImmediate(callback, error);
		return (null);
	}
	if (args.dryRun) {
		scanctx.outstream.on('end', callback);
		scanctx.outstream.on('data', function () {});
		return (scanctx.outstream);
	}

	sink = args.sink || fileds.indexSink({
	    'metrics': args.metrics,
	    'interval': args.interval
	});
	if (sink instanceof Error) {
		setImmediate(callback, sink);
		return (null);
	}

	queries = args.metrics.map(function (m) {
		return (mod_dragnet_impl.metricQuery(m, args.timeAfter,
		    args.timeBefore, args.interval, self.ds_timefield));
	});
	passes = [];
	for (i = 0; i < queries.length; i += MAX_METRICS)
		passes.push(i);

	paths = [];
	scanctx.findstream.on('data', function (fileinfo) {
		if (!fileinfo.error)
			paths.push(fileinfo.path);
	});
	scanctx.findstream.on('end', function () {
		mod_vasync.forEachPipeline({
		    'inputs': passes,
		    'func': function (base, passcb) {
			self.fanoutPass(queries.slice(base, base + MAX_METRICS),
			    base, args.filter || null, paths, sink, passcb);
		    }
		}, function (err) {
			if (err) {
				callback(err);
				return;
			}
			if (args.sink) {
				sink.end();
				callback();
				return;
			}
			sink.on('flushed', callback);
			sink.end();
		});
	});
	return (sink);
};

/*
 * One fan-out scan of up to MAX_METRICS queries over the files; its points
 * are written to the sink with __dn_metric renumbered from "base".
 */
DatasourceGpu.prototype.fanoutPass = function (queries, base, dsfilter, paths,
    sink, callback)
{
	var self = this;
	var names, plan, scan;

	names = [];
	queries.forEach(function (q) {
		q.qc_breakdowns.forEach(function (b) { names.push(b.name); });
	});
	plan = JSON.stringify({
	    'format': this.ds_format,
	    'ds_filter': dsfilter,
	    'metrics': queries.map(
		function (q) { return (queryPlan(q, this.ds_timefield)); },
		this)
	});

	try {
		scan = dragnet_gpu.scanOpen(plan, this.ds_device, names, 1);
	} catch (ex) {
		setImmediate(callback, ex);
		return;
	}
	mod_vasync.forEachPipeline({
	    'inputs': paths,
	    'func': function (path, feedcb) {
		self.feedPath(scan, path, feedcb);
	    }
	}, function (err) {
		if (err) {
			scan.close();
			callback(err);
			return;
		}
		scan.finish(function (ferr, points) {
			scan.close();
			if (ferr) {
				callback(ferr);
				return;
			}
			points.forEach(function (p) {
				p.fields.__dn_metric += base;
				sink.write(p);
			});
			callback();
		});
	});
};
