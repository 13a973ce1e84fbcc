/*
 * jit_cache.cpp: see jit_cache.h.  POSIX host code only.
 */
#include <dirent.h>
#include <dlfcn.h>
#include <errno.h>
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <vector>

#include "jit_cache.h"

namespace dng {

namespace {

const char MAGIC[8] = { 'D', 'N', 'G', 'J', 'I', 'T', 'K', '\0' };
const char SUFFIX[] = ".jitk";
const uint64_t SEED_NAME = 0x6a69742d6e616d65ull;
const uint64_t SEED_SUM = 0x6a69742d73756d73ull;
const uint64_t SEED_BUILD = 0x6a69742d6275696cull;
/* no entry is this large: a length field beyond it is damage */
const uint64_t MAX_ENTRY = 1ull << 30;
/* a temporary file this old belongs to a writer that died */
const time_t STRAY_SECONDS = 60;

std::atomic<uint64_t> g_hits{0}, g_misses{0}, g_writes{0}, g_evictions{0},
    g_errors{0};

std::mutex g_dir_mu;
bool g_dir_set = false;
std::string g_dir;

bool ends_with(const char *s, const char *suffix)
{
	const size_t n = strlen(s), m = strlen(suffix);
	return n >= m && memcmp(s + n - m, suffix, m) == 0;
}

void put64(std::string &s, uint64_t v)
{
	s.append((const char *)&v, 8);
}

uint64_t get64(const std::string &s, size_t at)
{
	uint64_t v;
	memcpy(&v, s.data() + at, 8);
	return v;
}

/* a directory this user owns and nobody else may write to */
bool dir_private(const struct stat &st)
{
	return S_ISDIR(st.st_mode) && st.st_uid == geteuid() &&
	    (st.st_mode & (S_IWGRP | S_IWOTH)) == 0;
}

/* mkdir -p, each level created with mode 0700; then the directory must be
 * private */
bool make_dir(const std::string &dir)
{
	for (size_t i = 1; i <= dir.size(); i++) {
		if (i < dir.size() && dir[i] != '/')
			continue;
		const std::string d = dir.substr(0, i);
		if (mkdir(d.c_str(), 0700) != 0 && errno != EEXIST)
			return false;
	}
	struct stat st;
	return stat(dir.c_str(), &st) == 0 && dir_private(st);
}

bool write_all(int fd, const std::string &s)
{
	size_t off = 0;
	while (off < s.size()) {
		const ssize_t n = write(fd, s.data() + off, s.size() - off);
		if (n < 0 && errno == EINTR)
			continue;
		if (n <= 0)
			return false;
		off += (size_t)n;
	}
	return true;
}

bool read_all(int fd, std::string &s, size_t n)
{
	s.resize(n);
	size_t off = 0;
	while (off < n) {
		const ssize_t r = pread(fd, &s[off], n - off, (off_t)off);
		if (r < 0 && errno == EINTR)
			continue;
		if (r <= 0)
			return false;
		off += (size_t)r;
	}
	return true;
}

/* the cubin of a whole entry file for exactly `key`, or false */
bool parse(const std::string &f, const std::string &key, std::string &cubin)
{
	const size_t head = sizeof (MAGIC) + 8;
	if (f.size() < head + 8 || memcmp(f.data(), MAGIC, sizeof (MAGIC)) != 0)
		return false;
	uint32_t ver, zero;
	memcpy(&ver, f.data() + 8, 4);
	memcpy(&zero, f.data() + 12, 4);
	if (ver != JIT_CACHE_FORMAT || zero != 0)
		return false;
	const uint64_t klen = get64(f, head);
	size_t at = head + 8;
	if (klen != key.size() || f.size() - at < klen + 8 ||
	    memcmp(f.data() + at, key.data(), klen) != 0)
		return false;
	at += klen;
	const uint64_t clen = get64(f, at);
	at += 8;
	if (f.size() - at < 8 || clen != f.size() - at - 8)
		return false;
	if (get64(f, at + clen) != jit_cache_hash(f.data(), at + clen, SEED_SUM))
		return false;
	cubin.assign(f.data() + at, clen);
	return true;
}

struct Entry {
	struct timespec mtime;
	uint64_t bytes;
	std::string name;
};

/* delete the least recently used entries while more than `bound` bytes of
 * them are left, and temporary files that writers left behind */
void sweep(const std::string &dir, uint64_t bound)
{
	DIR *d = opendir(dir.c_str());
	if (!d) {
		g_errors++;
		return;
	}
	const int dfd = dirfd(d);
	const time_t now = time(nullptr);
	std::vector<Entry> ents;
	uint64_t total = 0;
	while (struct dirent *e = readdir(d)) {
		const bool tmp = e->d_name[0] == '.' && ends_with(e->d_name, ".tmp");
		if (!tmp && !ends_with(e->d_name, SUFFIX))
			continue;
		struct stat st;
		if (fstatat(dfd, e->d_name, &st, AT_SYMLINK_NOFOLLOW) != 0 ||
		    !S_ISREG(st.st_mode))
			continue;
		if (tmp) {
			if (now - st.st_mtime > STRAY_SECONDS)
				unlinkat(dfd, e->d_name, 0);
			continue;
		}
		ents.push_back(Entry{ st.st_mtim, (uint64_t)st.st_size,
		    e->d_name });
		total += (uint64_t)st.st_size;
	}
	std::sort(ents.begin(), ents.end(), [](const Entry &a, const Entry &b) {
		return a.mtime.tv_sec != b.mtime.tv_sec ?
		    a.mtime.tv_sec < b.mtime.tv_sec :
		    a.mtime.tv_nsec < b.mtime.tv_nsec;
	});
	for (size_t i = 0; i < ents.size() && total > bound; i++) {
		/* (another process may have taken it already) */
		if (unlinkat(dfd, ents[i].name.c_str(), 0) == 0)
			g_evictions++;
		else if (errno != ENOENT)
			continue;
		total -= ents[i].bytes;
	}
	closedir(d);
}

} /* namespace */

void jit_cache_set_dir(const char *dir)
{
	std::lock_guard<std::mutex> g(g_dir_mu);
	g_dir_set = true;
	g_dir = dir ? dir : "";
}

std::string jit_cache_dir()
{
	std::lock_guard<std::mutex> g(g_dir_mu);
	if (g_dir_set)
		return g_dir;
	const char *ev = getenv("DNG_JIT_CACHE_DIR");
	return ev ? ev : "";
}

std::string jit_cache_build_id(const char *path)
{
	Dl_info info;
	if (!path) {
		if (!dladdr((const void *)&jit_cache_build_id, &info) ||
		    !info.dli_fname || !info.dli_fname[0])
			return "";
		path = info.dli_fname;
	}
	const int fd = open(path, O_RDONLY | O_CLOEXEC);
	if (fd < 0)
		return "";
	struct stat st;
	void *m = MAP_FAILED;
	if (fstat(fd, &st) == 0 && S_ISREG(st.st_mode) && st.st_size > 0)
		m = mmap(nullptr, (size_t)st.st_size, PROT_READ,
		    MAP_PRIVATE | MAP_POPULATE, fd, 0);
	close(fd);
	if (m == MAP_FAILED)
		return "";
	/*
	 * (this is host time before a warm process's first launch: the file is
	 * mapped, not copied, and hashed in four independent chains, which the
	 * core runs side by side; each is invertible in its state, so a change
	 * to any one word changes the id, like jit_cache_hash)
	 */
	const unsigned char *b = (const unsigned char *)m;
	const size_t n = (size_t)st.st_size;
	uint64_t h[5] = { SEED_BUILD, SEED_BUILD + 1, SEED_BUILD + 2,
	    SEED_BUILD + 3, 0 };
	size_t i = 0;
	for (; i + 32 <= n; i += 32)
		for (int j = 0; j < 4; j++) {
			uint64_t w;
			memcpy(&w, b + i + 8 * j, 8);
			h[j] ^= w;
			h[j] *= 0xff51afd7ed558ccdull;
			h[j] ^= h[j] >> 32;
		}
	h[4] = jit_cache_hash(b + i, n - i, SEED_BUILD);
	munmap(m, n);
	char buf[40];
	snprintf(buf, sizeof (buf), "%016llx%016llx", (unsigned long long)
	    jit_cache_hash(h, sizeof (h), SEED_BUILD), (unsigned long long)n);
	return buf;
}

std::string jit_cache_name(const std::string &key)
{
	char buf[32];
	snprintf(buf, sizeof (buf), "%016llx%s", (unsigned long long)
	    jit_cache_hash(key.data(), key.size(), SEED_NAME), SUFFIX);
	return buf;
}

std::string jit_cache_entry(const std::string &key, const std::string &cubin,
    uint32_t format)
{
	std::string s(MAGIC, sizeof (MAGIC));
	const uint32_t ver[2] = { format, 0 };
	s.append((const char *)ver, sizeof (ver));
	put64(s, key.size());
	s += key;
	put64(s, cubin.size());
	s += cubin;
	put64(s, jit_cache_hash(s.data(), s.size(), SEED_SUM));
	return s;
}

bool jit_cache_get(const std::string &dir, const std::string &name,
    const std::string &key, std::string &cubin)
{
	struct stat ds;
	const bool there = stat(dir.c_str(), &ds) == 0;
	if (!there || !dir_private(ds)) {
		/* (a directory not there yet is no error: the first build
		 * makes it) */
		if (there || (errno != ENOENT && errno != ENOTDIR))
			g_errors++;
		g_misses++;
		return false;
	}
	const std::string path = dir + "/" + name;
	const int fd = open(path.c_str(), O_RDONLY | O_CLOEXEC);
	if (fd < 0) {
		if (errno != ENOENT)
			g_errors++;
		g_misses++;
		return false;
	}
	struct stat st;
	std::string f;
	bool hit = false;
	if (fstat(fd, &st) != 0) {
		g_errors++;
	} else if (S_ISREG(st.st_mode) && (uint64_t)st.st_size <= MAX_ENTRY) {
		if (!read_all(fd, f, (size_t)st.st_size))
			g_errors++;
		else
			hit = parse(f, key, cubin);
	}
	/* used now: the last to be evicted (failing that, it is only evicted
	 * sooner) */
	if (hit)
		futimens(fd, nullptr);
	close(fd);
	(hit ? g_hits : g_misses)++;
	return hit;
}

bool jit_cache_put(const std::string &dir, const std::string &name,
    const std::string &key, const std::string &cubin, uint64_t bound)
{
	if (!make_dir(dir)) {
		g_errors++;
		return false;
	}
	static std::atomic<unsigned> seq{0};
	char tmp[96];
	snprintf(tmp, sizeof (tmp), "/.%s.%ld.%u.tmp", name.c_str(),
	    (long)getpid(), seq++);
	const std::string tpath = dir + tmp, path = dir + "/" + name;
	const int fd = open(tpath.c_str(), O_WRONLY | O_CREAT | O_EXCL | O_CLOEXEC,
	    0600);
	if (fd < 0) {
		g_errors++;
		return false;
	}
	bool ok = write_all(fd, jit_cache_entry(key, cubin, JIT_CACHE_FORMAT));
	ok = close(fd) == 0 && ok;
	ok = ok && rename(tpath.c_str(), path.c_str()) == 0;
	if (!ok) {
		unlink(tpath.c_str());
		g_errors++;
		return false;
	}
	g_writes++;
	sweep(dir, bound);
	return true;
}

void jit_cache_count_error()
{
	g_errors++;
}

JitCacheStats jit_cache_stats()
{
	return JitCacheStats{ g_hits.load(), g_misses.load(), g_writes.load(),
	    g_evictions.load(), g_errors.load() };
}

} /* namespace dng */
