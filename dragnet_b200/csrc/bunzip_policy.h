/*
 * bunzip_policy.h: how a batch of bzip2 files (bunzip.cuh) is cut so that
 * its device memory stays bounded.
 *
 * A batch's block candidates, in file order, go in waves of at most
 * DNG_BZ_WAVE_BLOCKS: a wave holds one BWT slot per candidate (BZ_SLOT
 * bytes) and one transformation vector per chained block (4 bytes per block
 * byte).  A file may span waves; the chain picks up where the last wave left
 * it.  A wave's chained blocks are emitted in groups of at most
 * DNG_BZ_EMIT_OUT output bytes (a block is at most about 46 MB), and each
 * group is fed before the next is written.
 *
 * Host-only and free of CUDA; tests/test_bunzip_host.py drives it on the CPU.
 */
#ifndef DNG_BUNZIP_POLICY_H
#define DNG_BUNZIP_POLICY_H

#include <stddef.h>
#include <stdint.h>

#ifndef DNG_BZ_WAVE_BLOCKS
#define DNG_BZ_WAVE_BLOCKS ((size_t)1024)
#endif
#ifndef DNG_BZ_EMIT_OUT
#define DNG_BZ_EMIT_OUT ((uint64_t)2 << 30)
#endif

namespace dng {

/* the waves of n block candidates, at most `per` each: ends[w] is one past
 * wave w's last; the number of waves */
inline size_t bz_waves(size_t n, size_t per, size_t *ends)
{
	size_t w = 0;
	for (size_t at = 0; at < n; w++) {
		at = n - at > per ? at + per : n;
		ends[w] = at;
	}
	return w;
}

/* consecutive blocks of lens[0, n) in groups of at most `cap` output bytes
 * (a block larger than cap alone): ends[g] one past group g's last; the
 * number of groups */
inline size_t bz_emit_groups(const uint64_t *lens, size_t n, uint64_t cap,
    size_t *ends)
{
	size_t g = 0;
	uint64_t sum = 0;
	for (size_t i = 0; i < n; i++) {
		if (i && sum + lens[i] > cap) {
			ends[g++] = i;
			sum = 0;
		}
		sum += lens[i];
	}
	if (n)
		ends[g++] = n;
	return g;
}

} /* namespace dng */

#endif /* DNG_BUNZIP_POLICY_H */
