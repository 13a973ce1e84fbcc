/*
 * dragnet_gpu N-API addon: a thin binding of libdragnet_gpu.so
 * (include/dragnet_gpu.h) for integration/datasource-gpu.js, which replaces
 * the scan() of the reference's file datasource (lib/datasource-file.js:72-108;
 * backend dispatch lib/dragnet.js:296-303).
 *
 *   scanOpen(planJson, device, breakdownNames[, tagMetric])
 *                               -> scan object (throws Error on DNG_E*)
 *                                  device: an index, an array of them or
 *                                  "all" (every device): with more than
 *                                  one, one scan over all of them
 *                                  (dng_scan_open_devices), fed files only
 *                                  For a fan-out plan ("metrics": [...], the
 *                                  scan of `dn build`), breakdownNames holds
 *                                  every metric's names one metric after the
 *                                  other, and a true tagMetric adds
 *                                  fields.__dn_metric to each point.
 *   scan.feed(buffer, cb)          dng_scan_feed      (bytes are consumed)
 *   scan.feedFile(path, cb)        dng_scan_feed_file
 *   scan.feedGzip(path, cb)        dng_scan_feed_gzip (inflated on the GPU)
 *   scan.feedBzip2(path, cb)       dng_scan_feed_bzip2 (decoded on the GPU)
 *   scan.finish(cb)             -> cb(err, points, counters)
 *                                  points   = [{fields: {name: string|number},
 *                                              value: N}, ...]
 *                                  (counters: of the plan's first metric)
 *                                  counters = {lines, invalid_json, ...}
 *   scan.close()                   dng_scan_destroy + dng_plan_destroy
 *   jitCacheDir(dir)               dng_jit_cache_dir: keep the compiled scan
 *                                  kernels in directory `dir` (null: none)
 *                                  for later processes; before scanOpen
 *
 * Every call that can block (reads, H2D copies, waiting for kernels) runs as
 * napi async work on the libuv pool: the event loop is never blocked, as the
 * reference's streams never block it (lib/krill-skinner-stream.js:51).
 *
 * Node is not installed in this image: tests/test_integration_addon.py only
 * COMPILES this file, against tests/node_api_stub/node_api.h (declarations of
 * the N-API calls used here).  Build for real with node-gyp, linking
 * libdragnet_gpu.so (INTEGRATION.md).
 */
#include <node_api.h>

#include <string.h>

#include <string>
#include <vector>

#include "dragnet_gpu.h"

namespace {

struct ScanWrap {
	dng_plan *plan = nullptr;
	dng_scan *scan = nullptr;
	std::vector<std::string> names;		/* breakdown names, in order */
	bool tag = false;		/* fan-out: set fields.__dn_metric */
};

void Throw(napi_env env, const char *msg)
{
	napi_throw_error(env, nullptr, msg);
}

ScanWrap *Unwrap(napi_env env, napi_callback_info info, size_t *argc,
    napi_value *argv)
{
	napi_value self;
	void *p = nullptr;
	if (napi_get_cb_info(env, info, argc, argv, &self, nullptr) != napi_ok ||
	    napi_unwrap(env, self, &p) != napi_ok || !p ||
	    !((ScanWrap *)p)->scan) {
		Throw(env, "dragnet_gpu: not an open scan");
		return nullptr;
	}
	return (ScanWrap *)p;
}

std::string GetString(napi_env env, napi_value v)
{
	size_t n = 0;
	napi_get_value_string_utf8(env, v, nullptr, 0, &n);
	std::string s(n, '\0');
	napi_get_value_string_utf8(env, v, &s[0], n + 1, &n);
	return s;
}

/* ---- one asynchronous operation on a scan -------------------------------- */

struct Work {
	napi_async_work work = nullptr;
	napi_ref cb = nullptr, keep = nullptr;	/* callback; Buffer being fed */
	ScanWrap *w = nullptr;
	enum { FEED, FEED_FILE, FEED_GZIP, FEED_BZIP2, FINISH } op = FEED;
	std::string path;
	const void *buf = nullptr;
	size_t len = 0;
	int rc = 0;
	dng_result *res = nullptr;
	dng_counters ctr;
};

void Exec(napi_env, void *d)
{
	Work *k = (Work *)d;
	switch (k->op) {
	case Work::FEED:
		k->rc = dng_scan_feed(k->w->scan, k->buf, k->len);
		break;
	case Work::FEED_FILE:
		k->rc = dng_scan_feed_file(k->w->scan, k->path.c_str());
		break;
	case Work::FEED_GZIP:
		k->rc = dng_scan_feed_gzip(k->w->scan, k->path.c_str());
		break;
	case Work::FEED_BZIP2:
		k->rc = dng_scan_feed_bzip2(k->w->scan, k->path.c_str());
		break;
	case Work::FINISH:
		k->rc = dng_scan_finish(k->w->scan, &k->res);
		if (k->rc == 0)
			k->rc = dng_scan_counters(k->w->scan, &k->ctr);
		break;
	}
}

napi_value Points(napi_env env, Work *k)
{
	const size_t n = dng_result_count(k->res);
	const size_t nc = dng_result_ncols(k->res);
	/* metric m's names start at first[m] in the names given to scanOpen */
	const size_t nm = dng_result_nmetrics(k->res);
	std::vector<size_t> first(nm + 1, 0), ncm(nm, 0);
	for (size_t m = 0; m < nm; m++) {
		ncm[m] = dng_result_ncols_metric(k->res, (int)m);
		first[m + 1] = first[m] + ncm[m];
	}
	napi_value arr;
	napi_create_array_with_length(env, n, &arr);
	std::vector<const char *> strs(nc);
	std::vector<size_t> lens(nc);
	std::vector<uint8_t> isnum(nc);
	std::vector<double> nums(nc);
	for (size_t i = 0; i < n; i++) {
		uint64_t value = 0;
		dng_result_get(k->res, i, strs.data(), lens.data(), isnum.data(),
		    nums.data(), &value);
		const int m = dng_result_metric(k->res, i);
		const size_t base = m >= 0 && (size_t)m < nm ? first[m] : 0;
		const size_t ncols = m >= 0 && (size_t)m < nm ? ncm[m] : nc;
		napi_value pt, fields, v;
		napi_create_object(env, &pt);
		napi_create_object(env, &fields);
		for (size_t j = 0; j < ncols && base + j < k->w->names.size();
		    j++) {
			/* discrete values are strings, bucketized ones the
			 * bucket minimum as a number (tst.scan_file.sh.out:86) */
			if (isnum[j])
				napi_create_double(env, nums[j], &v);
			else
				napi_create_string_utf8(env, strs[j], lens[j], &v);
			napi_set_named_property(env, fields,
			    k->w->names[base + j].c_str(), v);
		}
		if (k->w->tag) {
			/* lib/datasource-file.js:412-419 */
			napi_create_double(env, (double)m, &v);
			napi_set_named_property(env, fields, "__dn_metric", v);
		}
		napi_set_named_property(env, pt, "fields", fields);
		napi_create_double(env, (double)value, &v);
		napi_set_named_property(env, pt, "value", v);
		napi_set_element(env, arr, (uint32_t)i, pt);
	}
	return arr;
}

napi_value Counters(napi_env env, const dng_counters &c)
{
	napi_value o, v;
	napi_create_object(env, &o);
#define PUT(name) napi_create_double(env, (double)c.name, &v); \
	napi_set_named_property(env, o, #name, v)
	PUT(lines); PUT(invalid_json); PUT(invalid_point); PUT(ds_filtered);
	PUT(ds_failedeval); PUT(user_filtered); PUT(user_failedeval);
	PUT(synth_undef); PUT(synth_baddate); PUT(time_filtered);
	PUT(time_failedeval); PUT(aggr_ninputs); PUT(slowpath_records);
#undef PUT
	return o;
}

void Done(napi_env env, napi_status, void *d)
{
	Work *k = (Work *)d;
	napi_value cb, undef, argv[3];
	size_t argc = 1;
	napi_get_reference_value(env, k->cb, &cb);
	napi_get_undefined(env, &undef);
	argv[0] = undef;
	if (k->rc != 0) {
		napi_value msg;
		napi_create_string_utf8(env, dng_scan_error(k->w->scan),
		    NAPI_AUTO_LENGTH, &msg);
		napi_create_error(env, nullptr, msg, &argv[0]);
	} else if (k->op == Work::FINISH) {
		argv[1] = Points(env, k);
		argv[2] = Counters(env, k->ctr);
		argc = 3;
	}
	if (k->res)
		dng_result_destroy(k->res);
	napi_call_function(env, undef, cb, argc, argv, nullptr);
	napi_delete_reference(env, k->cb);
	if (k->keep)
		napi_delete_reference(env, k->keep);
	napi_delete_async_work(env, k->work);
	delete k;
}

napi_value Queue(napi_env env, Work *k, napi_value cb, const char *what)
{
	napi_value name, undef;
	napi_get_undefined(env, &undef);
	napi_create_reference(env, cb, 1, &k->cb);
	napi_create_string_utf8(env, what, NAPI_AUTO_LENGTH, &name);
	napi_create_async_work(env, nullptr, name, Exec, Done, k, &k->work);
	napi_queue_async_work(env, k->work);
	return undef;
}

/* scan.feed(buffer, cb): the Buffer is referenced until the bytes are taken */
napi_value Feed(napi_env env, napi_callback_info info)
{
	size_t argc = 2;
	napi_value argv[2];
	ScanWrap *w = Unwrap(env, info, &argc, argv);
	if (!w)
		return nullptr;
	Work *k = new Work();
	k->w = w;
	k->op = Work::FEED;
	void *p = nullptr;
	if (argc < 2 ||
	    napi_get_buffer_info(env, argv[0], &p, &k->len) != napi_ok) {
		delete k;
		Throw(env, "feed(buffer, callback)");
		return nullptr;
	}
	k->buf = p;
	napi_create_reference(env, argv[0], 1, &k->keep);
	return Queue(env, k, argv[1], "dragnet_gpu.feed");
}

/* scan.feedFile(path, cb) */
napi_value FeedFile(napi_env env, napi_callback_info info)
{
	size_t argc = 2;
	napi_value argv[2];
	ScanWrap *w = Unwrap(env, info, &argc, argv);
	if (!w)
		return nullptr;
	if (argc < 2) {
		Throw(env, "feedFile(path, callback)");
		return nullptr;
	}
	Work *k = new Work();
	k->w = w;
	k->op = Work::FEED_FILE;
	k->path = GetString(env, argv[0]);
	return Queue(env, k, argv[1], "dragnet_gpu.feedFile");
}

/* scan.feedGzip(path, cb) */
napi_value FeedGzip(napi_env env, napi_callback_info info)
{
	size_t argc = 2;
	napi_value argv[2];
	ScanWrap *w = Unwrap(env, info, &argc, argv);
	if (!w)
		return nullptr;
	if (argc < 2) {
		Throw(env, "feedGzip(path, callback)");
		return nullptr;
	}
	Work *k = new Work();
	k->w = w;
	k->op = Work::FEED_GZIP;
	k->path = GetString(env, argv[0]);
	return Queue(env, k, argv[1], "dragnet_gpu.feedGzip");
}

/* scan.feedBzip2(path, cb) */
napi_value FeedBzip2(napi_env env, napi_callback_info info)
{
	size_t argc = 2;
	napi_value argv[2];
	ScanWrap *w = Unwrap(env, info, &argc, argv);
	if (!w)
		return nullptr;
	if (argc < 2) {
		Throw(env, "feedBzip2(path, callback)");
		return nullptr;
	}
	Work *k = new Work();
	k->w = w;
	k->op = Work::FEED_BZIP2;
	k->path = GetString(env, argv[0]);
	return Queue(env, k, argv[1], "dragnet_gpu.feedBzip2");
}

/* scan.finish(cb) */
napi_value Finish(napi_env env, napi_callback_info info)
{
	size_t argc = 1;
	napi_value argv[1];
	ScanWrap *w = Unwrap(env, info, &argc, argv);
	if (!w)
		return nullptr;
	if (argc < 1) {
		Throw(env, "finish(callback)");
		return nullptr;
	}
	Work *k = new Work();
	k->w = w;
	k->op = Work::FINISH;
	return Queue(env, k, argv[0], "dragnet_gpu.finish");
}

void Release(ScanWrap *w)
{
	if (w->scan)
		dng_scan_destroy(w->scan);
	if (w->plan)
		dng_plan_destroy(w->plan);
	w->scan = nullptr;
	w->plan = nullptr;
}

/* scan.close(): also run when the object is collected */
napi_value Close(napi_env env, napi_callback_info info)
{
	napi_value self, undef;
	void *p = nullptr;
	size_t argc = 0;
	napi_get_undefined(env, &undef);
	if (napi_get_cb_info(env, info, &argc, nullptr, &self, nullptr) ==
	    napi_ok && napi_unwrap(env, self, &p) == napi_ok && p)
		Release((ScanWrap *)p);
	return undef;
}

void Finalize(napi_env, void *data, void *)
{
	ScanWrap *w = (ScanWrap *)data;
	Release(w);
	delete w;
}

/* scanOpen(planJson, device, breakdownNames[, tagMetric]) */
napi_value ScanOpen(napi_env env, napi_callback_info info)
{
	size_t argc = 4;
	napi_value argv[4], obj, fn;
	if (napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr) !=
	    napi_ok || argc < 3) {
		Throw(env, "scanOpen(planJson, device, breakdownNames)");
		return nullptr;
	}
	const std::string plan = GetString(env, argv[0]);
	int32_t device = 0;
	std::vector<int> devices;
	uint32_t ndev = 0;
	char all[4] = "";
	size_t alllen = 0;
	const bool listed = napi_get_array_length(env, argv[1], &ndev) ==
	    napi_ok;
	if (listed) {
		for (uint32_t i = 0; i < ndev; i++) {
			napi_value e;
			int32_t d = -1;
			napi_get_element(env, argv[1], i, &e);
			napi_get_value_int32(env, e, &d);
			devices.push_back(d);
		}
	} else if (napi_get_value_string_utf8(env, argv[1], all, sizeof (all),
	    &alllen) == napi_ok && strcmp(all, "all") == 0) {
		for (int d = 0; d < dng_device_count(); d++)
			devices.push_back(d);
	} else {
		napi_get_value_int32(env, argv[1], &device);
	}
	if (devices.size() == 1)
		device = devices[0];
	ScanWrap *w = new ScanWrap();
	uint32_t nnames = 0;
	napi_get_array_length(env, argv[2], &nnames);
	for (uint32_t i = 0; i < nnames; i++) {
		napi_value e;
		napi_get_element(env, argv[2], i, &e);
		w->names.push_back(GetString(env, e));
	}
	int32_t tag = 0;
	if (argc >= 4)
		napi_get_value_int32(env, argv[3], &tag);
	w->tag = tag != 0;
	char err[512];
	err[0] = '\0';
	int rc = dng_plan_create(plan.c_str(), &w->plan, err, sizeof (err));
	/* (an empty list is refused there; "all" without devices fails as
	 * dng_scan_open does) */
	if (rc == 0 && (devices.size() > 1 || (listed && devices.empty())))
		rc = dng_scan_open_devices(w->plan, devices.data(),
		    (int)devices.size(), &w->scan, err, sizeof (err));
	else if (rc == 0)
		rc = dng_scan_open(w->plan, device, &w->scan, err, sizeof (err));
	if (rc != 0) {
		Release(w);
		delete w;
		Throw(env, err[0] ? err : "dragnet_gpu: cannot open scan");
		return nullptr;
	}
	napi_create_object(env, &obj);
	napi_wrap(env, obj, w, Finalize, nullptr, nullptr);
	const struct { const char *name; napi_callback fn; } methods[] = {
	    { "feed", Feed }, { "feedFile", FeedFile },
	    { "feedGzip", FeedGzip },
	    { "feedBzip2", FeedBzip2 }, { "finish", Finish },
	    { "close", Close } };
	for (const auto &m : methods) {
		napi_create_function(env, m.name, NAPI_AUTO_LENGTH, m.fn, nullptr,
		    &fn);
		napi_set_named_property(env, obj, m.name, fn);
	}
	return obj;
}

/* jitCacheDir(dir): a string, or null / undefined for none */
napi_value JitCacheDir(napi_env env, napi_callback_info info)
{
	size_t argc = 1;
	napi_value argv[1], undef;
	napi_get_undefined(env, &undef);
	if (napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr) !=
	    napi_ok) {
		Throw(env, "jitCacheDir(dir)");
		return nullptr;
	}
	size_t n = 0;
	const bool named = argc >= 1 && napi_get_value_string_utf8(env, argv[0],
	    nullptr, 0, &n) == napi_ok;
	const std::string dir = named ? GetString(env, argv[0]) : std::string();
	if (dng_jit_cache_dir(named ? dir.c_str() : nullptr) != 0) {
		Throw(env, "dragnet_gpu: jitCacheDir failed");
		return nullptr;
	}
	return undef;
}

} /* namespace */

NAPI_MODULE_INIT()
{
	napi_value fn;
	napi_create_function(env, "scanOpen", NAPI_AUTO_LENGTH, ScanOpen, nullptr,
	    &fn);
	napi_set_named_property(env, exports, "scanOpen", fn);
	napi_create_function(env, "jitCacheDir", NAPI_AUTO_LENGTH, JitCacheDir,
	    nullptr, &fn);
	napi_set_named_property(env, exports, "jitCacheDir", fn);
	return exports;
}
