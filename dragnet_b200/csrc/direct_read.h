/*
 * direct_read.h: how dng_scan_feed_file reads a byte range of a regular file
 * (feed_file_parallel in api.cu), in host code only so that the CPU tests
 * compile it (tests/hostcheck/direct_read_check.cpp).
 *
 * A range mostly absent from the page cache is read with O_DIRECT: the storage
 * device DMAs it into the pinned block ring, with no CPU copy and without
 * filling the page cache with a log that is read once.  A cached range is read
 * through the page cache (pread), as it always was.  Which one is decided per
 * range from what the page cache holds of it (dr_cached_fraction, dr_direct);
 * results never depend on it.
 *
 * O_DIRECT reads whole aligned units at aligned offsets into aligned memory.
 * The range [off, off + size) is read in blocks of DR_BLK bytes from `base`,
 * off rounded down to the file's offset alignment: block b covers file bytes
 * [base + b DR_BLK, base + (b + 1) DR_BLK) and feeds the part of them inside
 * the range.  Blocks are read at their aligned length, so the last one may
 * ask past the end of the file (the read comes back short there) or past the
 * end of the range (the extra bytes are not fed).  With an alignment of 1 the
 * plan is the buffered reader's: blocks from off itself, read at the length
 * fed.
 */
#pragma once

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cerrno>
#include <cstddef>
#include <cstdint>

namespace dng {

const size_t DR_BLK = (size_t)4 << 20;	/* one slot of the pinned ring */
const size_t DR_ALIGN_DEFAULT = 4096;	/* when statx does not report it */
/* a range is read direct when less than this share of its pages is cached:
 * a starting point, not yet measured against storage (DESIGN.md section 6) */
const double DR_DIRECT_BELOW = 0.125;
const int DR_SHORT = -1;		/* dr_read_block: the file ended early */

struct DioAlign {
	size_t mem = DR_ALIGN_DEFAULT;	/* buffer address and length */
	size_t off = DR_ALIGN_DEFAULT;	/* file offset */
	bool ok = true;			/* false: the file refuses O_DIRECT */
};

/* the kernel's struct statx (glibc's lacks the direct I/O fields) */
struct DrStatx {
	uint32_t mask, blksize;
	uint64_t attributes;
	uint32_t nlink, uid, gid;
	uint16_t mode, spare0;
	uint64_t ino, size, blocks, attributes_mask;
	uint64_t ts[8];			/* atime, btime, ctime, mtime */
	uint32_t rdev_major, rdev_minor, dev_major, dev_minor;
	uint64_t mnt_id;
	uint32_t dio_mem_align, dio_offset_align;
	uint64_t spare[12];
};
static_assert(offsetof(DrStatx, dio_mem_align) == 0x98 &&
    sizeof (DrStatx) == 0x100, "struct statx layout");

/* the O_DIRECT alignment of an open file: statx(STATX_DIOALIGN), Linux >= 6.1;
 * DR_ALIGN_DEFAULT where the kernel or the filesystem does not report it */
inline DioAlign dr_align(int fd)
{
	const unsigned DR_STATX_DIOALIGN = 0x2000;
	DioAlign a;
	DrStatx st = {};
	if (syscall(SYS_statx, fd, "", AT_EMPTY_PATH, DR_STATX_DIOALIGN,
	    &st) != 0 || !(st.mask & DR_STATX_DIOALIGN))
		return a;
	if (!st.dio_mem_align || !st.dio_offset_align) {
		a.ok = false;	/* reported: no direct I/O on this file */
		return a;
	}
	a.mem = st.dio_mem_align;
	a.off = st.dio_offset_align;
	return a;
}

/* [off, off + size) of a file, in blocks of DR_BLK from base */
struct DrPlan {
	uint64_t off = 0, size = 0, base = 0;
	size_t align = 1, nblocks = 0;

	/* slot bytes [lo, hi) of block b are the range's */
	size_t lo(size_t b) const { return b ? 0 : (size_t)(off - base); }
	size_t hi(size_t b) const {
		return (size_t)std::min<uint64_t>(DR_BLK,
		    off + size - (base + b * DR_BLK));
	}
	uint64_t at(size_t b) const { return base + b * DR_BLK; }
	/* bytes block b reads: hi rounded up to the alignment */
	size_t len(size_t b) const {
		return (hi(b) + align - 1) / align * align;
	}
};

/* align: 1 (buffered) or the O_DIRECT offset and length alignment, a power of
 * two that divides DR_BLK */
inline DrPlan dr_plan(uint64_t off, uint64_t size, size_t align)
{
	DrPlan p;
	p.off = off;
	p.size = size;
	p.align = align;
	p.base = off / align * align;
	p.nblocks = size ? (size_t)((off + size - p.base + DR_BLK - 1) / DR_BLK)
	    : 0;
	return p;
}

/* the alignment dr_plan needs for O_DIRECT reads into `mem`, whose slots
 * start DR_BLK apart; 0 when they cannot be read direct */
inline size_t dr_direct_align(const DioAlign &a, const void *mem)
{
	const size_t al = std::max(a.mem, a.off);
	if (!a.ok || al > DR_BLK || (al & (al - 1)) ||
	    (uintptr_t)mem % a.mem)
		return 0;
	return al;
}

/*
 * Reads block b of p from fd into dst (a slot of DR_BLK bytes) with rd, a
 * pread(2).  Returns 0 with the slot bytes to feed in [*lo, *hi), an errno,
 * or DR_SHORT when the file ends inside the range and `exact` (else the block
 * feeds what is there).  A direct read comes back short only at the end of
 * the file: the next read would start unaligned, so a short read ends it.
 */
template <class Pread>
int dr_read_block(Pread &&rd, int fd, const DrPlan &p, size_t b, uint8_t *dst,
    bool exact, size_t *lo, size_t *hi)
{
	const size_t want = p.len(b), need = p.hi(b);
	size_t have = 0;
	while (have < need) {
		ssize_t n = rd(fd, dst + have, want - have,
		    (off_t)(p.at(b) + have));
		if (n < 0) {
			if (errno == EINTR)
				continue;
			return errno;
		}
		if (n == 0)
			break;
		have += (size_t)n;
		if (have % p.align)
			break;
	}
	if (have < need && exact)
		return DR_SHORT;
	*lo = p.lo(b);
	*hi = std::max(*lo, std::min(have, need));
	return 0;
}

/*
 * One range's read, shared by the reader threads: block b from the O_DIRECT
 * descriptor dfd while `direct` holds, else from the buffered one.  A
 * filesystem that refuses O_DIRECT (EINVAL) makes the range buffered from
 * there on: the block is read again through fd, and the fallback is counted
 * once.  *via_direct: which descriptor the block came from.
 */
struct DrRange {
	int fd = -1, dfd = -1;
	DrPlan plan;
	bool exact = false;
	std::atomic<bool> direct{false};
	std::atomic<uint64_t> fallbacks{0};
};

template <class Pread>
int dr_fetch(Pread &&rd, DrRange &r, size_t b, uint8_t *dst, size_t *lo,
    size_t *hi, bool *via_direct)
{
	if (r.direct.load()) {
		int err = dr_read_block(rd, r.dfd, r.plan, b, dst, r.exact, lo,
		    hi);
		if (err != EINVAL) {
			*via_direct = true;
			return err;
		}
		if (r.direct.exchange(false))
			r.fallbacks++;
	}
	*via_direct = false;
	return dr_read_block(rd, r.fd, r.plan, b, dst, r.exact, lo, hi);
}

/*
 * The share of the pages of [off, off + size) in the page cache, from
 * count(page-aligned offset, length) -> cached pages of it (or -1), asked of
 * at most DR_PROBE_WINDOWS windows of DR_PROBE_PAGES pages spread evenly over
 * the range (all of a short one): it costs the same for a file of any size.
 */
const size_t DR_PROBE_WINDOWS = 64, DR_PROBE_PAGES = 16;

template <class Count>
double dr_sampled(uint64_t off, uint64_t size, Count &&count)
{
	const uint64_t ps = (uint64_t)sysconf(_SC_PAGESIZE);
	const uint64_t first = off / ps;
	const size_t pages = (size_t)((off + size + ps - 1) / ps - first);
	if (!size || !pages)
		return 0;
	const size_t nwin = std::min(DR_PROBE_WINDOWS,
	    (pages + DR_PROBE_PAGES - 1) / DR_PROBE_PAGES);
	size_t seen = 0, cached = 0;
	for (size_t i = 0; i < nwin; i++) {
		const size_t p = pages * i / nwin;
		const size_t n = std::min(DR_PROBE_PAGES, pages * (i + 1) / nwin - p);
		const long c = count((first + p) * ps, n * ps);
		if (c < 0)
			return -1;
		cached += (size_t)c;
		seen += n;
	}
	return std::min(1.0, (double)cached / (double)seen);
}

/*
 * The share of the range's pages in the page cache: mincore(2) over read-only
 * mappings of sampled windows; -1 when it cannot be told (a file that cannot
 * be mapped).  A mapping reaches the pages that back the file where the
 * descriptor's own page cache may hold none: cachestat(2) on an overlayfs
 * file (the root filesystem of a container) reports a hot file as cold.  One
 * mapping of a whole large file, and its page vector, would cost more than
 * the scan of a cached file can spare.
 */
inline double dr_cached_fraction(int fd, uint64_t off, uint64_t size)
{
	const size_t ps = (size_t)sysconf(_SC_PAGESIZE);
	return dr_sampled(off, size, [fd, ps](uint64_t at, uint64_t len) -> long {
		void *m = mmap(nullptr, (size_t)len, PROT_READ, MAP_SHARED, fd,
		    (off_t)at);
		if (m == MAP_FAILED)
			return -1;
		unsigned char vec[DR_PROBE_PAGES];
		int rc = mincore(m, (size_t)len, vec);
		munmap(m, (size_t)len);
		if (rc != 0)
			return -1;
		long n = 0;
		for (size_t i = 0; i < len / ps; i++)
			n += vec[i] & 1;
		return n;
	});
}

/* read direct: little of the range is cached (unknown counts as cached) */
inline bool dr_direct(double cached)
{
	return cached >= 0 && cached < DR_DIRECT_BELOW;
}

} /* namespace dng */
