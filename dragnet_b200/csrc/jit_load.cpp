/*
 * jit_load.cpp: the per-process cache of run-time compiled kernels (jit.h),
 * the kernels kept on disk (jit_cache.h), their compilation off the caller's
 * thread and their loading into the CUDA runtime.
 */
#include <stdlib.h>

#include <condition_variable>
#include <map>
#include <mutex>
#include <thread>
#include <vector>

#include "jit.h"
#include "jit_cache.h"

namespace dng {

namespace {

std::mutex g_mu;
std::condition_variable g_cv;
std::map<std::string, std::shared_ptr<JitKernels>> g_cache;	/* by jit_key */

/*
 * Compiler threads must be joined before the compiler libraries tear
 * themselves down at exit (a compile in flight while they do segfaults or
 * hangs): by dng_jit_finish(), which the host calls before it exits (the
 * Python package from atexit); failing that, by an atexit() handler
 * registered after jit_prepare() -- which loads the libraries and runs them
 * once, so that most of the exit handlers they register come before it and
 * run after it (not all: libnvJitLink registers some only in its first real
 * link) -- and, for good measure, when this library's statics go.
 */
struct Workers {
	std::vector<std::thread> th;
	void join_all() {
		std::vector<std::thread> mine;
		{
			std::lock_guard<std::mutex> g(g_mu);
			mine.swap(th);
		}
		for (auto &t : mine)
			if (t.joinable())
				t.join();
	}
	~Workers() { join_all(); }
} g_workers;

bool g_exiting = false;

void join_workers_at_exit()
{
	{
		std::lock_guard<std::mutex> g(g_mu);
		g_exiting = true;
	}
	g_workers.join_all();
}

/* the linked kernel in `cubin` loaded for device `dev` (current on this
 * thread then) */
bool load_into(JitKernels &k, const std::string &cubin, int dev, int smem_max,
    std::string &err)
{
	cudaSetDevice(dev);
	/* (an error some earlier call left for its caller's check stays) */
	const bool clean = cudaPeekAtLastError() == cudaSuccess;
	cudaError_t e = cudaLibraryLoadData(&k.lib, cubin.data(), nullptr,
	    nullptr, 0, nullptr, nullptr, 0);
	if (e == cudaSuccess)
		e = cudaLibraryGetKernel(&k.kern, k.lib, "dng_scan_kernel_j");
	if (e == cudaSuccess)
		e = cudaFuncSetAttribute((const void *)k.kern,
		    cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
	if (e != cudaSuccess) {
		/* (ours is not left for the scan's next error check to find) */
		if (clean)
			cudaGetLastError();
		if (k.lib)
			cudaLibraryUnload(k.lib);
		k.lib = nullptr;
		k.kern = nullptr;
		err = std::string("loading the linked kernel: ") +
		    cudaGetErrorString(e);
		return false;
	}
	return true;
}

/* where a kernel goes on disk: the cache directory ("" none), the entry's key
 * and its file name */
struct DiskEntry {
	std::string dir, key, name;
};

/*
 * The key of a kernel on disk: jit_key() with the device's compute capability
 * in place of its index (an index means nothing to another process), after
 * the build id of this library file; "" (no cache) if that cannot be read.
 */
std::string disk_key(const u8 *blob, size_t bytes, const FPlan *plan, int nsl,
    int dev, int smem_max)
{
	static const std::string build = jit_cache_build_id(nullptr);
	if (build.empty())
		return "";
	int major = 0, minor = 0;
	cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
	cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
	return build + jit_key(blob, bytes, plan, nsl, major * 10 + minor,
	    smem_max);
}

void build_into(std::shared_ptr<JitKernels> k, std::string source, int nsl,
    int dev, int smem_max, std::string key, DiskEntry disk, bool on_caller)
{
	/* one build at a time; by the time it is this one's turn the scan that
	 * asked may be gone (short scans, test suites), or the process on its
	 * way out: then there is nothing to build (and the next request for
	 * this source starts afresh) */
	static std::mutex turn;
	std::lock_guard<std::mutex> my_turn(turn);
	{
		std::lock_guard<std::mutex> g(g_mu);
		/* (the cache, this thread, the scan) */
		if (g_exiting || k.use_count() <= 2) {
			auto it = g_cache.find(key);
			if (it != g_cache.end() && it->second == k)
				g_cache.erase(it);
			k->err = "abandoned";
			k->state.store(2);
			g_cv.notify_all();
			return;
		}
	}
	std::string cubin, err;
	bool ok = jit_build(source, nsl, cubin, err, &k->compile_ms, &k->link_ms);
	if (ok)
		ok = load_into(*k, cubin, dev, smem_max, err);
	{
		std::lock_guard<std::mutex> g(g_mu);
		k->err = err;
		k->ok = ok;
		k->state.store(ok ? 1 : 2);
	}
	g_cv.notify_all();
	/* written after the scan has its kernel, and never on the scan's
	 * thread: a build that ran there (sync mode) hands the write to a
	 * thread of its own, joined with the compiler threads */
	if (!ok || disk.dir.empty())
		return;
	if (!on_caller) {
		jit_cache_put(disk.dir, disk.name, disk.key, cubin,
		    JIT_CACHE_BOUND);
		return;
	}
	std::lock_guard<std::mutex> g(g_mu);
	if (!g_exiting)
		g_workers.th.emplace_back(jit_cache_put, disk.dir, disk.name,
		    disk.key, std::move(cubin), JIT_CACHE_BOUND);
}

} /* namespace */

void jit_finish()
{
	join_workers_at_exit();
}

std::shared_ptr<JitKernels> jit_request(const u8 *blob, size_t bytes,
    const FPlan *plan, int nsl, int dev, int smem_max, bool wait)
{
	std::string key = jit_key(blob, bytes, plan, nsl, dev, smem_max);
	std::unique_lock<std::mutex> g(g_mu);
	std::shared_ptr<JitKernels> k;
	auto it = g_cache.find(key);
	if (it != g_cache.end()) {
		k = it->second;
	} else {
		/* (failures are cached too: not tried again for every scan) */
		k = std::make_shared<JitKernels>();
		g_cache[key] = k;
		/* a kernel on disk is loaded here, on the caller's thread, in
		 * either mode: the scan's first launch runs it, and neither
		 * compiler library is loaded.  Requests for it meanwhile
		 * (the shards of a multi-device scan) wait for the answer */
		DiskEntry disk;
		disk.dir = jit_cache_dir();
		k->disk_pending = !disk.dir.empty();
		g.unlock();
		if (!disk.dir.empty()) {
			disk.key = disk_key(blob, bytes, plan, nsl, dev, smem_max);
			disk.name = jit_cache_name(disk.key);
			std::string cubin, err;
			if (disk.key.empty()) {
				/* (no build id: nothing read or written) */
				jit_cache_count_error();
				disk.dir.clear();
			} else if (jit_cache_get(disk.dir, disk.name, disk.key,
			    cubin)) {
				int cur = dev;
				cudaGetDevice(&cur);
				const bool ok = load_into(*k, cubin, dev, smem_max,
				    err);
				cudaSetDevice(cur);
				if (ok) {
					g.lock();
					k->ok = true;
					k->state.store(1);
					k->disk_pending = false;
					g_cv.notify_all();
					return k;
				}
				/* (a cubin the driver refuses: built anew) */
				jit_cache_count_error();
			}
			g.lock();
			k->disk_pending = false;
			g_cv.notify_all();
			g.unlock();
		}
		const std::string source = jit_source(blob, bytes, plan);
		if (wait) {
			build_into(k, source, nsl, dev, smem_max, key, disk,
			    true);
			g.lock();
		} else {
			/* (the libraries loaded and run once, here, and then
			 * the handler that waits for the thread: see Workers) */
			jit_prepare();
			static std::once_flag once;
			std::call_once(once, [] { atexit(join_workers_at_exit); });
			g.lock();
			g_workers.th.emplace_back(build_into, k, source, nsl, dev,
			    smem_max, key, disk, false);
		}
	}
	if (wait)
		g_cv.wait(g, [&] { return k->state.load() != 0; });
	else
		g_cv.wait(g, [&] { return !k->disk_pending; });
	return k;
}

} /* namespace dng */
