/*
 * fast_jit_cold.cu: the rare paths of the run-time linked F kernel
 * (fast_jit.cu), compiled ahead of time as relocatable SASS: a key the inline
 * tally tier has no room for, a record the miss list has no room for (the
 * general parser, from HBM), the end-of-launch flush of the tally cache.
 */
#define DNG_NO_GENERAL_KERNELS
#include "fast_kernel.cuh"

using namespace dng;

extern "C" __device__ void dng_cold_slow_add(FSmem m, const FPlan *F,
    u32 defmask, u32 klen, STab stab, const GTable *gt)
{
	fslow_add(m, F, defmask, klen, stab, gt);
}

extern "C" __device__ void dng_cold_miss(const u8 *data,
    unsigned long long start, unsigned long long beg, unsigned long long end,
    const DevPlan *plan, STab stab, const GTable *gt,
    unsigned long long *counters)
{
	fmiss_inline(data, start, beg, end, plan, stab, gt, counters);
}

extern "C" __device__ void dng_cold_flush(STab stab, u32 s1slots, u32 sslots,
    const GTable *tab)
{
	fflush_tally(stab, s1slots, sslots, *tab);
}

extern "C" __device__ bool dng_cold_long_tally(FSmem m, const FPlan *F,
    u32 defmask, STab stab, const GTable *gt, u32 over_sa)
{
	return flong_tally(m, *F, F, defmask, stab, *gt, over_sa);
}
