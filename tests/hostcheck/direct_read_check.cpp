/*
 * direct_read_check: drives the file reader's host pieces
 * (dragnet_b200/csrc/direct_read.h) from commands on stdin, one per line, and
 * prints one line of results per command (TEST ONLY;
 * tests/test_direct_read_host.py).
 *
 *   const                          DR_BLK and the policy's threshold
 *   align PATH                     the file's O_DIRECT alignment
 *   cached PATH OFF SIZE           the residency probe (sampled mincore),
 *                                  cachestat(2) over the whole range as a
 *                                  reference (-1 where the kernel lacks it),
 *                                  and the policy's answer
 *   read PATH OFF SIZE EXACT FAULT OUT
 *       reads [OFF, OFF + SIZE) of PATH through the plan, block by block, with
 *       O_DIRECT, into one DR_BLK buffer, and appends the bytes it feeds to
 *       OUT.  FAULT: "-" none, "einval" (every O_DIRECT read fails with
 *       EINVAL, as on a filesystem that refuses it), "shrink:N" (the file is
 *       truncated to N bytes after the plan is made)
 */
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <string>

#include "direct_read.h"

using namespace dng;

/* the share of [off, off + size) cached by cachestat(2) (Linux >= 6.5), whole
 * range in one call: what the sampled probe is checked against */
static double cachestat(int fd, uint64_t off, uint64_t size)
{
	const uint64_t ps = (uint64_t)sysconf(_SC_PAGESIZE);
	const uint64_t start = off / ps * ps;
	const uint64_t pages = (off + size + ps - 1) / ps - off / ps;
	struct { uint64_t off, len; } range = { start, off + size - start };
	struct { uint64_t nr_cache, nr_dirty, nr_writeback, nr_evicted,
	    nr_recently_evicted; } cs = {};
	if (!pages || syscall(451 /* cachestat */, fd, &range, &cs, 0) != 0)
		return -1;
	return std::min(1.0, (double)cs.nr_cache / (double)pages);
}

int main()
{
	char cmd[32];
	uint8_t *buf = (uint8_t *)aligned_alloc(4096, DR_BLK);
	while (scanf("%31s", cmd) == 1) {
		if (!strcmp(cmd, "const")) {
			printf("blk=%zu direct_below=%.6f\n", DR_BLK,
			    DR_DIRECT_BELOW);
			continue;
		}
		char path[4096], fault[64], out[4096];
		unsigned long long off = 0, size = 0;
		int exact = 0;
		if (scanf("%4095s", path) != 1)
			return 2;
		int fd = open(path, O_RDONLY);
		if (fd < 0)
			return 3;
		if (!strcmp(cmd, "align")) {
			DioAlign a = dr_align(fd);
			printf("mem=%zu off=%zu ok=%d plan=%zu\n", a.mem, a.off,
			    (int)a.ok, dr_direct_align(a, buf));
		} else if (!strcmp(cmd, "cached")) {
			if (scanf("%llu %llu", &off, &size) != 2)
				return 2;
			double f = dr_cached_fraction(fd, off, size);
			printf("cachestat=%.6f fraction=%.6f direct=%d\n",
			    cachestat(fd, off, size), f, (int)dr_direct(f));
		} else if (!strcmp(cmd, "read")) {
			if (scanf("%llu %llu %d %63s %4095s", &off, &size, &exact,
			    fault, out) != 5)
				return 2;
			DrRange r;
			r.fd = fd;
			r.exact = exact != 0;
			size_t align = dr_direct_align(dr_align(fd), buf);
			r.dfd = open(path, O_RDONLY | O_DIRECT);
			if (!align || r.dfd < 0) {
				printf("rc=nodirect\n");
				fflush(stdout);
				close(fd);
				continue;
			}
			r.direct = true;
			r.plan = dr_plan(off, size, align);
			const bool einval = !strcmp(fault, "einval");
			if (!strncmp(fault, "shrink:", 7) &&
			    truncate(path, atoll(fault + 7)) != 0)
				return 4;
			auto rd = [&](int f, void *dst, size_t n, off_t at) {
				if (einval && f == r.dfd) {
					errno = EINVAL;
					return (ssize_t)-1;
				}
				return pread(f, dst, n, at);
			};
			FILE *o = fopen(out, "ab");
			uint64_t dbytes = 0, bbytes = 0;
			int rc = 0;
			for (size_t b = 0; b < r.plan.nblocks && !rc; b++) {
				size_t lo = 0, hi = 0;
				bool via = false;
				rc = dr_fetch(rd, r, b, buf, &lo, &hi, &via);
				if (!rc) {
					fwrite(buf + lo, 1, hi - lo, o);
					(via ? dbytes : bbytes) += hi - lo;
				}
			}
			fclose(o);
			close(r.dfd);
			printf("rc=%d nblocks=%zu align=%zu base=%llu direct_bytes=%llu "
			    "buffered_bytes=%llu fallbacks=%llu\n", rc,
			    r.plan.nblocks, align, (unsigned long long)r.plan.base,
			    (unsigned long long)dbytes,
			    (unsigned long long)bbytes,
			    (unsigned long long)r.fallbacks.load());
		} else {
			return 2;
		}
		fflush(stdout);
		close(fd);
	}
	free(buf);
	return 0;
}
