/*
 * inflate_policy.h: which gzip files of an inflate batch are split and
 * decoded by many warps (inflate_split.cuh), and into how many chunks.  The
 * rest go one warp per file (inflate_kernel).
 *
 * The aim is about as many work items as the device holds decode warps at
 * once (the split decode kernel's occupancy times the SM count): a batch of
 * that many files is already spread over the device, and a large file
 * decoded by one warp leaves the rest of it idle.  A chunk smaller than the
 * floor would spend more on finding its start and on the 32 KiB its decode
 * reaches back than on decoding, so none is cut smaller.
 *
 * Host-only and free of CUDA; tests/test_inflate_split_host.py drives it on
 * the CPU.  Building with -DDNG_NO_GZIP_SPLIT splits nothing (the measured
 * comparison in DESIGN.md §7.A).
 */
#ifndef DNG_INFLATE_POLICY_H
#define DNG_INFLATE_POLICY_H

#include <stddef.h>
#include <stdint.h>

/* the smallest chunk, in compressed bytes */
#ifndef DNG_GZ_SPLIT_FLOOR
#define DNG_GZ_SPLIT_FLOOR ((uint64_t)64 << 10)
#endif

/* a chunk's decode must cover more than the window it reaches back over */
static_assert(DNG_GZ_SPLIT_FLOOR >= 32768, "split floor below the window");

namespace dng {

/*
 * chunks[i] for each of n files of sizes[i] compressed bytes: 1 (one warp)
 * or the number of chunks to cut it into.  A file under twice the floor is
 * never split, nor is any when the batch holds at least `resident` files.
 * Otherwise each file larger than max(floor, total / resident) is cut into
 * equal chunks no larger than that, none smaller than the floor.
 */
inline void gz_split_plan(const uint64_t *sizes, size_t n, uint64_t resident,
    uint64_t floor, uint32_t *chunks)
{
	uint64_t total = 0;
	for (size_t i = 0; i < n; i++) {
		chunks[i] = 1;
		total += sizes[i];
	}
#ifdef DNG_NO_GZIP_SPLIT
	return;
#endif
	if (!resident || n >= resident)
		return;
	const uint64_t target = total / resident > floor ? total / resident :
	    floor;
	for (size_t i = 0; i < n; i++) {
		const uint64_t s = sizes[i];
		if (s < 2 * floor || s <= target)
			continue;
		uint64_t c = (s + target - 1) / target;
		if (c > s / floor)
			c = s / floor;
		chunks[i] = (uint32_t)c;
	}
}

} /* namespace dng */

#endif /* DNG_INFLATE_POLICY_H */
