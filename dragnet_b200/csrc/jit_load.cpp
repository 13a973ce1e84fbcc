/*
 * jit_load.cpp: the per-process cache of run-time compiled kernels (jit.h),
 * their compilation off the caller's thread and their loading into the CUDA
 * runtime.
 */
#include <stdlib.h>

#include <condition_variable>
#include <map>
#include <mutex>
#include <thread>
#include <vector>

#include "jit.h"

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

void build_into(std::shared_ptr<JitKernels> k, std::string source, int nsl,
    int dev, int smem_max, std::string key)
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
	if (ok) {
		cudaSetDevice(dev);
		cudaError_t e = cudaLibraryLoadData(&k->lib, cubin.data(), nullptr,
		    nullptr, 0, nullptr, nullptr, 0);
		if (e == cudaSuccess)
			e = cudaLibraryGetKernel(&k->kern, k->lib, "dng_scan_kernel_j");
		if (e == cudaSuccess)
			e = cudaFuncSetAttribute((const void *)k->kern,
			    cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
		if (e != cudaSuccess) {
			ok = false;
			err = std::string("loading the linked kernel: ") +
			    cudaGetErrorString(e);
		}
	}
	{
		std::lock_guard<std::mutex> g(g_mu);
		k->err = err;
		k->ok = ok;
		k->state.store(ok ? 1 : 2);
	}
	g_cv.notify_all();
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
		g.unlock();
		const std::string source = jit_source(blob, bytes, plan);
		if (wait) {
			build_into(k, source, nsl, dev, smem_max, key);
			g.lock();
		} else {
			/* (the libraries loaded and run once, here, and then
			 * the handler that waits for the thread: see Workers) */
			jit_prepare();
			static std::once_flag once;
			std::call_once(once, [] { atexit(join_workers_at_exit); });
			g.lock();
			g_workers.th.emplace_back(build_into, k, source, nsl, dev,
			    smem_max, key);
		}
	}
	if (wait)
		g_cv.wait(g, [&] { return k->state.load() != 0; });
	return k;
}

} /* namespace dng */
