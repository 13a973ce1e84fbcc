/*
 * jit_cache.h: run-time compiled kernels kept on disk (jit.h), so that a new
 * process finds the kernel a process before it linked instead of linking it
 * again.  Host code only, no CUDA: the file format and the policy.
 *
 * Off unless a directory is given (dng_jit_cache_dir() or the environment's
 * DNG_JIT_CACHE_DIR); off, nothing is read or written.  One file per kernel,
 * named by a 64-bit hash of its key:
 *
 *     magic "DNGJITK\0" | u32 format version | u32 0 | u64 key length | key |
 *     u64 cubin length | cubin | u64 checksum of everything before it
 *
 * A read compares the stored key byte for byte: another key under the same
 * name, a short file, a flipped byte, another format version or another
 * build's key is a miss, decided here before anything reaches the driver.
 * Writes go to a temporary file in the directory and are renamed into place
 * (readers never see part of an entry; of two writers of one key the last
 * wins); after a write the least recently used entries are deleted while the
 * directory holds more than a bound.  A directory that is not this user's,
 * or that others may write to, is not used: anyone who can write an entry
 * chooses the code the scan runs.  No failure here fails a scan: it is
 * counted (stats().errors) and the kernel is built as without the cache.
 */
#ifndef DNG_JIT_CACHE_H
#define DNG_JIT_CACHE_H

#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <string>

namespace dng {

/* bytes of entries a directory may hold after a write */
const uint64_t JIT_CACHE_BOUND = 512ull << 20;

const uint32_t JIT_CACHE_FORMAT = 1;

struct JitCacheStats {
	uint64_t hits, misses, writes, evictions, errors;
};

/* 64-bit hash of `n` bytes (not cryptographic: names and checksums).  One
 * multiply per word, and every step is invertible in the state, so inputs
 * that differ in one word never hash alike. */
inline uint64_t jit_cache_hash(const void *p, size_t n, uint64_t seed)
{
	const unsigned char *b = (const unsigned char *)p;
	uint64_t h = seed ^ ((uint64_t)n * 0x9e3779b97f4a7c15ull);
	auto mix = [](uint64_t h, uint64_t w) {
		h ^= w;
		h *= 0xff51afd7ed558ccdull;
		return h ^ (h >> 32);
	};
	size_t i = 0;
	for (; i + 8 <= n; i += 8) {
		uint64_t w;
		memcpy(&w, b + i, 8);
		h = mix(h, w);
	}
	if (i < n) {
		uint64_t w = 0;
		memcpy(&w, b + i, n - i);
		h = mix(h, w);
	}
	h ^= h >> 29;
	h *= 0xbf58476d1ce4e5b9ull;
	return h ^ (h >> 32);
}

/* the directory for this process (null or "": off; overrides the
 * environment), and the one in force: the one set, else DNG_JIT_CACHE_DIR,
 * else "" (off) */
void jit_cache_set_dir(const char *dir);
std::string jit_cache_dir();

/*
 * The build id every key on disk starts with: a hash and the size of the
 * whole library file `path` (null: the file this code was loaded from), so
 * that any change to the library -- the matcher generator, the compiler
 * options, the embedded kernel builds -- gives its kernels other keys.  ""
 * when the file cannot be read.  32 characters.
 */
std::string jit_cache_build_id(const char *path);

/* the file name of the entry for `key` */
std::string jit_cache_name(const std::string &key);

/* the bytes of an entry file in format version `format` */
std::string jit_cache_entry(const std::string &key, const std::string &cubin,
    uint32_t format);

/* the cubin stored under `name` in `dir` for exactly `key`: true on a hit
 * (whose mtime is then refreshed); anything else is a miss */
bool jit_cache_get(const std::string &dir, const std::string &name,
    const std::string &key, std::string &cubin);

/* store `cubin` for `key` under `name` (creating `dir`, mode 0700), then
 * delete least recently used entries while the directory holds more than
 * `bound` bytes of them; false (and an error counted) if it could not */
bool jit_cache_put(const std::string &dir, const std::string &name,
    const std::string &key, const std::string &cubin, uint64_t bound);

/* a failure outside this module that the cache caused (a cubin the driver
 * refused) */
void jit_cache_count_error();

JitCacheStats jit_cache_stats();

} /* namespace dng */

#endif
