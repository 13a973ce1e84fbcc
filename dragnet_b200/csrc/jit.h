/*
 * jit.h: run-time compilation of a scan's record templates (tmpl.h / fast.h)
 * into the matcher of scan_kernel_j -- the F kernel with its interpreted trie
 * walk replaced by straight-line code with the literals as immediates.
 *
 * What is generated at run time is ONLY the matcher, dng_jmatch(): a few
 * hundred lines from the trie blob plus the wildcard scanners of fscan.cuh
 * (embedded as text).  NVRTC turns it into LTO-IR and nvJitLink optimises it
 * together with the LTO-IR build of the kernel that ships inside the library
 * (fast_jit.cu): the matcher is inlined into the record loop and registers are
 * allocated across it.  Everything else -- chunk pipeline, newline index,
 * stages, tally, miss handling -- is the code of scan_kernel_f; its rare paths
 * (fast_jit_cold.cu) are compiled ahead of time and only linked.  Results cannot depend on this choice: the generated
 * matcher accepts exactly what fmatch() accepts (same trie, same scanners) and
 * everything it rejects is parsed by the general code.
 *
 * Kernels are cached per process by what the generated source and its build
 * are made from (jit_key), so a scan whose kernel is cached generates no
 * source; with a cache directory also on disk (jit_cache.h), so that a new
 * process loads the kernel an earlier one linked.  Both libraries are
 * dlopen()ed; without them (or with DNG_JIT=0) scans use the interpreted
 * matcher.
 */
#ifndef DNG_JIT_H
#define DNG_JIT_H

#include <cuda_runtime.h>

#include <atomic>
#include <memory>
#include <string>

#include "fast.h"

namespace dng {

struct JitKernels {
	cudaLibrary_t lib = nullptr;
	cudaKernel_t kern = nullptr;	/* dng_scan_kernel_j for one slice size */
	std::atomic<int> state{0};	/* 0 being built, 1 ready, 2 failed */
	bool disk_pending = false;	/* being looked up on disk (jit_cache.h) */
	bool ok = false;
	std::string err;
	double compile_ms = 0, link_ms = 0;
};

/* the CUDA source of dng_jmatch() for an F trie blob (tmpl_build, compact)
 * and of the plan constant the kernel is specialised to (null: left out);
 * `prelude` replaces the device definitions the generated code builds on
 * (tests/hostcheck compiles the same code for the host with its own).
 * A pure function of the blob's bytes, the plan's bytes, jit_shared(plan) and
 * the prelude: the rest it writes out is constant text of this library. */
std::string jit_source(const u8 *blob, size_t bytes, const FPlan *plan,
    const char *prelude = nullptr);

/* whether the generated matcher calls one shared copy of each wildcard
 * scanner instead of inlining them (DNG_JIT_SHARED=0|1 forces) */
bool jit_shared(const FPlan *plan);

/* the cache key of the kernels for an F blob and plan at lane slices of nsl x
 * 16 bytes on device `dev`: every input of jit_source() and of the build, byte
 * for byte (no hash, so that different inputs never share a kernel) */
std::string jit_key(const u8 *blob, size_t bytes, const FPlan *plan, int nsl,
    int dev, int smem_max);

/*
 * The kernels for this blob and plan on device `dev`, from the cache, else
 * from the cache directory (loaded on the caller's thread: state 1 on return,
 * in either mode), or built now from jit_source(blob, bytes, plan): on the
 * caller's thread if `wait` (then state is 1 or 2 on return), else on a
 * worker thread (state 0 until it is done: the caller keeps using the
 * interpreted matcher meanwhile).  A build is written to the cache directory
 * after the kernel is ready, never on the caller's thread: by the worker that
 * built it, or (wait) by a thread of its own, joined like the workers.
 * smem_max = dynamic shared memory the kernels may be launched with.
 */
std::shared_ptr<JitKernels> jit_request(const u8 *blob, size_t bytes,
    const FPlan *plan, int nsl, int dev, int smem_max, bool wait);

/* load the two compiler libraries now, on this thread (they are dlopen()ed
 * once per process), and compile and link an empty kernel with them once, so
 * that the exit handlers they register on first use are registered before any
 * the caller registers next; false if they are not there */
bool jit_prepare();

/* dng_jit_finish(): join the compiler threads, drop queued builds */
void jit_finish();

/* only compile + link, to `cubin` (no device needed: tests); nsl = 16-byte
 * units per lane slice: 7, 9, 11 or 13 */
bool jit_build(const std::string &source, int nsl, std::string &cubin,
    std::string &err, double *compile_ms, double *link_ms);

} /* namespace dng */

#endif
