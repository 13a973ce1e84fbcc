/*
 * fast_kernel.cuh: scan_kernel_f, the F path's kernel (fast.h), and
 * scan_miss_kernel, which hands the records it did not take to the general
 * per-record code.
 *
 * Geometry: one persistent 896-thread CTA per SM; every WARP is its own
 * pipeline, as in scan_kernel_w, over SEGMENTS of consecutive chunks:
 *
 *   - a chunk is 32 x NSL x 16 bytes (the host picks NSL so that a chunk
 *     holds just under 32 average records); a segment owns the records whose
 *     newline lies in its chunks;
 *   - the warp walks its segment in WINDOWS of 32 lane slices of `wunits` x
 *     16 bytes, each staged by one TMA bulk copy into its private buffer.  The
 *     first stages the 512-byte pre-lap before the segment with it, to find
 *     where the open record starts; every later one starts at the first
 *     record not yet taken (16-byte aligned), so it holds 32 complete records
 *     where the lines allow and every lane of the record pass has one.  The
 *     bytes after the 32nd come again with the next window, from L2;
 *   - newline index: every lane tests its slice 16 bytes at a time with one
 *     "any byte == '\n'" SWAR test per word (exact analysis only where it
 *     fires), a shuffle scan orders the hits, lanes write their positions;
 *     record r of the window goes to lane r;
 *   - fmatch() -> fstage() -> fkey_hash() / tally (fast.cuh): captures are one
 *     word per path in shared memory ([path][thread]: conflict free), the key
 *     is hashed and compared in place against the CTA's tally cache;
 *   - a record the F path does not decide is appended to the miss list
 *     (absolute offsets) and parsed by scan_miss_kernel right after this
 *     kernel; if the list is full it is parsed here, out of line, from HBM.
 *
 * Bound: HBM read of the input, once (+ 512 bytes per segment); the windows
 * read it from L2 once more per 32 records, in part.
 */
#ifndef DNG_FAST_KERNEL_CUH
#define DNG_FAST_KERNEL_CUH

#include <stddef.h>

#include "scan_kernel.cuh"
#include "fast.cuh"

namespace dng {

#define DNG_F_NT F_NT			/* threads per CTA */
#define DNG_F_PRE 512			/* pre-lap bytes = longest straddling head */
#define DNG_F_SLACK 64
#define DNG_F_MAXLINE DNG_F_PRE		/* host: sampled lines must be shorter */
#define DNG_F_SEG 16			/* chunks per segment (at most) */

struct MissEnt {
	unsigned long long beg;		/* ~0: unknown, before `end` */
	unsigned long long end;		/* the record's newline (or end of input) */
};

struct FScanArgs {
	const u8 *data;			/* 16-byte aligned */
	unsigned long long start;	/* first valid byte (< 16) */
	unsigned long long nbytes;	/* end of valid bytes */
	const FPlan *fplan;
	const DevPlan *plan;		/* the full plan (global): overflow path */
	const u8 *tmpl;			/* F trie blob or null */
	u32 tmpl_bytes;
	u32 leaf_off, pool_off;		/* its THdr's, for the kernel's convenience */
	unsigned long long *counters;
	GTable tab;
	u32 nchunks, seg;		/* chunks, chunks per segment */
	u32 wunits;			/* window: lane slices of NSL + 1 or
					 * NSL + 2 16-byte units (fwindow_units) */
	u32 final;
	u32 s1slots, sslots;
	u32 nrows;			/* capture rows (FPlan::nrows) */
	MissEnt *miss;
	u32 miss_cap;
	u32 *miss_n;
	u32 *seg_next;			/* segment queue: zero at launch */
};

/*
 * The window's lane slices, in 16-byte units, for chunks of nsl-unit slices
 * and nw warps per CTA.  A chunk holds just under 32 average records, and so
 * does pre-lap + chunk (nsl + 1 units) once a window starts up to 15 bytes
 * before its first record: too often for a segment to take fewer passes than
 * it has chunks (tools/f_passes.py).  512 bytes more (nsl + 2, odd like nsl:
 * the lanes' 16-byte loads are free of bank conflicts) hold 32; fewer warps
 * than DNG_F_NW leave the room for them, DNG_F_NW do not.
 */
static inline u32 fwindow_units(u32 nsl, u32 nw)
{
	return nw < DNG_F_NW ? nsl + 2 : nsl + 1;
}

/* per-warp shared memory: window, the quotes behind it, newline positions,
 * mbarrier */
__host__ __device__ __forceinline__ u32 fwarp_bytes(u32 wunits)
{
	return (32 * 16 * wunits + DNG_F_SLACK + 2 * DNG_F_NLCAP + 16 + 127) &
	    ~127u;
}

static constexpr u32 FPLAN_SMEM = (sizeof (FPlan) + 127) & ~127u;

/* (warp_bytes = fwarp_bytes(wunits); nw = warps of the launch: DNG_F_NW,
 * or fewer -- the capture rows keep their stride -- when the tally cache
 * needs the room) */
static inline size_t fkernel_smem(u32 warp_bytes, u32 tmpl_bytes, u32 s1slots,
    u32 sslots, u32 nrows, u32 nw)
{
	return FPLAN_SMEM + tmpl_bytes + (size_t)s1slots * sizeof (SSlot1) +
	    (size_t)sslots * sizeof (SSlot) + (size_t)nrows * DNG_F_NT * 4 +
	    (size_t)nw * warp_bytes;
}

/* mbarrier / TMA helpers on 32-bit shared addresses (no generic pointers to
 * keep alive across the record loop) */
__device__ __forceinline__ void mbar_init_sa(u32 bar, u32 count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;"
	    :: "r"(bar), "r"(count) : "memory");
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx_sa(u32 bar, u32 bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
	    :: "r"(bar), "r"(bytes) : "memory");
}

__device__ __forceinline__ void tma_load_1d_sa(u32 dst, const void *src,
    u32 bytes, u32 bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::"
	    "complete_tx::bytes [%0], [%1], %2, [%3];"
	    :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

__device__ __forceinline__ void mbar_wait_sa(u32 bar, u32 parity)
{
	asm volatile(
	    "{\n"
	    ".reg .pred p;\n"
	    "WAIT_%=:\n"
	    "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
	    "@p bra DONE_%=;\n"
	    "bra WAIT_%=;\n"
	    "DONE_%=:\n"
	    "}\n"
	    :: "r"(bar), "r"(parity) : "memory");
}

__device__ __forceinline__ void sts8(u32 addr, u32 v)
{
	asm volatile("st.shared.u8 [%0], %1;" :: "r"(addr), "r"(v) : "memory");
}

__device__ __forceinline__ void sts16(u32 addr, u32 v)
{
	asm volatile("st.shared.u16 [%0], %1;" :: "r"(addr), "r"(v) : "memory");
}

__device__ __forceinline__ void sts128(u32 addr, uint4 v)
{
	asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};"
	    :: "r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

__device__ __forceinline__ void sts32(u32 addr, u32 v)
{
	asm volatile("st.shared.u32 [%0], %1;" :: "r"(addr), "r"(v) : "memory");
}

__device__ __forceinline__ void sts64(u32 addr, unsigned long long v)
{
	asm volatile("st.shared.u64 [%0], %1;" :: "r"(addr), "l"(v) : "memory");
}

__device__ __forceinline__ unsigned long long lds64(u32 addr)
{
	unsigned long long v;
	asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
	return v;
}

/* shared-memory access for fmatch()/fstage()/fkey_*() */
struct FSmem {
	u32 ra;			/* record start (shared address) */
	u32 nodes, leaves, pool;
	u32 caps;		/* this thread's capture column */

	typedef TmplSmem::Cur Cur;
	__device__ __forceinline__ Cur cursor(u32 off) const
	{
		Cur c;
		const u32 a = ra + off;
		c.sh = (a & 3) * 8;
		c.wa = (a & ~3u) + 4;
		c.w0 = lds32(c.wa - 4);
		c.w1 = lds32(c.wa);
		return c;
	}
	/* aligned words (fscan.cuh) */
	struct ACur {
		u32 wa, k;
		__device__ __forceinline__ u32 next()
		{
			const u32 v = lds32(wa);
			wa += 4;
			return v;
		}
	};
	__device__ __forceinline__ ACur acursor(u32 off) const
	{
		ACur c;
		const u32 a = ra + off;
		c.k = a & 3;
		c.wa = a & ~3u;
		return c;
	}
	__device__ __forceinline__ u32 apos(const ACur &c) const
	{
		return c.wa - 4 - ra;
	}
	__device__ __forceinline__ u32 byte(u32 off) const { return lds8(ra + off); }
	/* the 8 bytes from off: the two aligned 8-byte words around them (the
	 * window is 8-byte aligned, and its slack follows it) */
	__device__ __forceinline__ void words2(u32 off, u32 &lo, u32 &hi) const
	{
		const u32 a = ra + off;
		const unsigned long long q0 = lds64(a & ~7u);
		const unsigned long long q1 = lds64((a & ~7u) + 8);
		const u32 sh = (a & 7) * 8;
		const unsigned long long v = sh ? (q0 >> sh) | (q1 << (64 - sh)) :
		    q0;
		lo = (u32)v;
		hi = (u32)(v >> 32);
	}
	__device__ __forceinline__ u32 word(u32 off) const
	{
		Cur c = cursor(off);
		return c.next();
	}
	__device__ __forceinline__ const u8 *ptr(u32 off) const
	{
		return (const u8 *)__cvta_shared_to_generic(ra + off);
	}
	__device__ __forceinline__ TQuad node(u32 i) const
	{
		const uint4 v = lds128(nodes + i * 16);
		TQuad q;
		q.x = v.x; q.y = v.y; q.z = v.z; q.w = v.w;
		return q;
	}
	__device__ __forceinline__ u32 litw(u32 off) const { return lds32(pool + off); }
	__device__ __forceinline__ u32 leaf(u32 i) const { return lds32(leaves + 4 * i); }
	__device__ __forceinline__ u32 pool32(u32 off) const { return lds32(pool + off); }
	__device__ __forceinline__ void setcap(u32 p, u32 v) const
	{
		sts32(caps + p * (DNG_F_NT * 4), v);
	}
	__device__ __forceinline__ u32 getcap(u32 p) const
	{
		return lds32(caps + p * (DNG_F_NT * 4));
	}
};

/* a tally slot's inline key, any alignment */
struct FKeySmem {
	u32 ka;
	typedef TmplSmem::Cur Cur;
	__device__ __forceinline__ Cur cursor(u32 off) const
	{
		Cur c;
		const u32 a = ka + off;
		c.sh = (a & 3) * 8;
		c.wa = (a & ~3u) + 4;
		c.w0 = lds32(c.wa - 4);
		c.w1 = lds32(c.wa);
		return c;
	}
};

#ifdef DNG_JIT_HOT
/*
 * The link-time-optimised build of the kernel (fast_jit.cu) keeps its rare,
 * large paths out of the optimiser's way: they are compiled ahead of time
 * (fast_jit_cold.cu) and only linked in.
 */
extern "C" __device__ void dng_cold_slow_add(FSmem m, const FPlan *F,
    u32 defmask, u32 klen, STab stab, const GTable *gt);
extern "C" __device__ void dng_cold_miss(const u8 *data,
    unsigned long long start, unsigned long long beg, unsigned long long end,
    const DevPlan *plan, STab stab, const GTable *gt,
    unsigned long long *counters);
extern "C" __device__ void dng_cold_flush(STab stab, u32 s1slots, u32 sslots,
    const GTable *tab);
extern "C" __device__ bool dng_cold_long_tally(FSmem m, const FPlan *F,
    u32 defmask, STab stab, const GTable *gt, u32 over_sa);
/*
 * The scan's plan as a CONSTANT of the generated code (jit.cpp writes it out
 * with its initialiser): after link-time optimisation the stage and key code
 * below is specialised to it -- column loops unrolled, kinds and entry points
 * folded, absent filters gone.  (The copy in shared memory is still what the
 * rare paths are handed.)
 */
extern "C" __constant__ const FPlan dng_jplan;
#define fslow_add dng_cold_slow_add
#define fmiss_inline dng_cold_miss
#else
/* first sighting of a key in this CTA, or a key the inline tier has no room
 * for: materialise it and take the general tally path */
__device__ __noinline__ void fslow_add(FSmem m, const FPlan *F, u32 defmask,
    u32 klen, STab stab, const GTable *gt)
{
	__align__(8) u8 kbuf[F_MAXKEY + 16];
	fkey_write(m, *F, defmask, kbuf);
	const unsigned long long *kw = (const unsigned long long *)kbuf;
	shared_add(stab, *gt, key_hash_words(kw, klen), kw, klen, 1);
}

#endif /* DNG_JIT_HOT */

__device__ __forceinline__ unsigned long long lds64_acquire(u32 addr)
{
	unsigned long long v;
	asm volatile("ld.acquire.cta.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr)
	    : "memory");
	return v;
}

__device__ __forceinline__ void sts64_release(u32 addr, unsigned long long v)
{
	asm volatile("st.release.cta.shared.u64 [%0], %1;" :: "r"(addr), "l"(v)
	    : "memory");
}

/* a key the inline tier has no room for (counted: the host gives the cache
 * more room if this is common) */
__device__ __forceinline__ void fover(FSmem &m, const FPlan *Fcold,
    u32 defmask, u32 klen, const STab &stab, const GTable &gt, u32 over_sa)
{
	asm volatile("red.shared.add.u32 [%0], 1;" :: "r"(over_sa) : "memory");
	fslow_add(m, Fcold, defmask, klen, stab, &gt);
}

/*
 * Count the record's key: the CTA's inline tier, probed with the F hash.  A
 * slot's tag is published with release semantics once its key is written and
 * read with acquire semantics (plain shared loads and stores in SASS: no
 * fence on the path every record takes).
 */
__device__ __forceinline__ void ftally(FSmem &m, const FPlan &F,
    const FPlan *Fcold, u32 defmask, u32 h, u32 klen, const STab &stab,
    const GTable &gt, u32 over_sa)
{
	if (klen <= DNG_SKEY) {
		const unsigned long long claim = (unsigned long long)(h | 1u);
		u32 idx = (h >> 7) & stab.mask1;
		for (u32 probe = 0; probe < 8; probe++) {
			SSlot1 *s = &stab.s1[idx];
			const u32 sa = smem_u32(s);
			unsigned long long tag = lds64_acquire(sa);
			if (tag == 0) {
				const unsigned long long old =
				    atomicCAS(&s->tag, 0ull, claim);
				if (old == 0) {
					s->klen = klen;
					fkey_write(m, F, defmask, (u8 *)s->key);
					atomicAdd(&s->count, 1u);
					sts64_release(sa, claim | DNG_READY);
					return;
				}
				tag = old;
			}
			if ((tag & ~DNG_READY) == claim) {
				while (!(tag & DNG_READY))
					tag = lds64_acquire(sa);
				if (lds32(sa + (u32)offsetof(SSlot1, klen)) == klen) {
					FKeySmem k;
					k.ka = sa + (u32)offsetof(SSlot1, key);
					if (fkey_equal(m, F, defmask, k)) {
						atomicAdd(&s->count, 1u);
						return;
					}
				}
			}
			idx = (idx + 1) & stab.mask1;
		}
	}
	fover(m, Fcold, defmask, klen, stab, gt, over_sa);
}

/*
 * Count a short key (fast.cuh FKey): the same inline tier, probed with the
 * short key's hash; the slot holds k.hdr for klen and k.w as its key, read
 * and written 8 bytes at a time at their fixed places.  A key the tier has no
 * room for takes the general path in record.cuh's encoding.
 */
__device__ __forceinline__ void ftally_short(FSmem &m, const FPlan &F,
    const FPlan *Fcold, u32 defmask, const FKey &k, const STab &stab,
    const GTable &gt, u32 over_sa)
{
	const u32 h = fkey_short_hash(k, F.ncols);
	const unsigned long long claim = (unsigned long long)(h | 1u);
	u32 idx = (h >> 7) & stab.mask1;
	for (u32 probe = 0; probe < 8; probe++) {
		SSlot1 *s = &stab.s1[idx];
		const u32 sa = smem_u32(s);
		const u32 ka = sa + (u32)offsetof(SSlot1, key);
		unsigned long long tag = lds64_acquire(sa);
		if (tag == 0) {
			const unsigned long long old = atomicCAS(&s->tag, 0ull,
			    claim);
			if (old == 0) {
				sts32(sa + (u32)offsetof(SSlot1, klen), k.hdr);
#pragma unroll
				for (u32 j = 0; j < FK_COLS; j++)
					if (j < F.ncols)
						sts64(ka + 8 * j, k.w[2 * j] |
						    (unsigned long long)
						    k.w[2 * j + 1] << 32);
				atomicAdd(&s->count, 1u);
				sts64_release(sa, claim | DNG_READY);
				return;
			}
			tag = old;
		}
		if ((tag & ~DNG_READY) == claim) {
			while (!(tag & DNG_READY))
				tag = lds64_acquire(sa);
			unsigned long long diff = lds32(sa +
			    (u32)offsetof(SSlot1, klen)) ^ k.hdr;
#pragma unroll
			for (u32 j = 0; j < FK_COLS; j++)
				if (j < F.ncols)
					diff |= lds64(ka + 8 * j) ^ (k.w[2 * j] |
					    (unsigned long long)k.w[2 * j + 1] << 32);
			if (diff == 0) {
				atomicAdd(&s->count, 1u);
				return;
			}
		}
		idx = (idx + 1) & stab.mask1;
	}
	/* (the key's length in record.cuh's encoding) */
	u32 klen = 0;
#pragma unroll
	for (u32 j = 0; j < FK_COLS; j++) {
		const u32 n = (k.hdr >> (4 * j)) & 0xf;
		if (j < F.ncols)
			klen += n == FK_ORD ? 10 : 2 + n;
	}
	fover(m, Fcold, defmask, klen, stab, gt, over_sa);
}

/* the F kernel's end: its short keys in record.cuh's encoding, then the
 * common flush (flush_tally) */
__device__ __forceinline__ void fflush_tally(const STab &stab, u32 s1slots,
    u32 sslots, const GTable &tab)
{
	__syncthreads();
	for (u32 i = threadIdx.x; i < s1slots; i += blockDim.x) {
		SSlot1 *s = &stab.s1[i];
		if (s->tag == 0 || !(s->klen & FK_PACKED))
			continue;
		FKey k;
		k.hdr = s->klen;
#pragma unroll
		for (u32 j = 0; j < FK_COLS; j++) {
			k.w[2 * j] = (u32)s->key[j];
			k.w[2 * j + 1] = (u32)(s->key[j] >> 32);
		}
		s->klen = fkey_unpack(k, (u8 *)s->key);
	}
	flush_tally(stab, s1slots, sslots, tab);
}

/*
 * A key that is not a short key: hashed, compared and tallied piece by piece
 * (false: longer than the F path carries).  Where the templates' samples have
 * only short keys (FPlan::short_keys) the link-time optimised kernel calls it
 * out of line (dng_cold_long_tally): the H100's instruction cache does not
 * hold its code in the record loop as well as the short key's.
 */
__device__ __forceinline__ bool flong_tally(FSmem &m, const FPlan &F,
    const FPlan *Fcold, u32 defmask, const STab &stab, const GTable &gt,
    u32 over_sa)
{
	u32 h, klen;
	if (!fkey_hash(m, F, defmask, h, klen))
		return false;
	ftally(m, F, Fcold, defmask, h, klen, stab, gt, over_sa);
	return true;
}

#ifndef DNG_JIT_HOT
/*
 * A record the miss list had no room for: the general parser, from HBM, right
 * here.  Entirely out of line, with its own counters (added to the global
 * ones directly), so that the kernel's per-thread state stays in registers.
 */
__device__ __noinline__ void fmiss_inline(const u8 *data,
    unsigned long long start, unsigned long long beg, unsigned long long end,
    const DevPlan *plan, STab stab, const GTable *gt,
    unsigned long long *counters)
{
	u32 mctr[(MAX_METRICS - 1) * MCTR_PER];
	for (int k = 0; k < (MAX_METRICS - 1) * MCTR_PER; k++)
		mctr[k] = 0;
	LocalCounters C;
	C.lines = C.invalid_json = C.invalid_point = 0;
	C.ds_filtered = C.ds_failedeval = C.user_filtered = 0;
	C.user_failedeval = C.synth_undef = C.synth_baddate = 0;
	C.time_filtered = C.time_failedeval = C.aggr = C.slow = 0;
	C.unsupported = 0;
	unsigned long long q = beg;
	u32 nlong = 0;
	if (q == ~0ull) {
		q = end;
		while (q > start && data[q - 1] != '\n')
			q--;
		nlong = 1;
	}
	scan_one_global(data + q, (u32)min((unsigned long long)DNG_MAXREC,
	    end - q), *plan, stab, *gt, C, mctr);
	const u32 vals[CTR_TMPL] = { C.lines, C.invalid_json, C.invalid_point,
	    C.ds_filtered, C.ds_failedeval, C.user_filtered, C.user_failedeval,
	    C.synth_undef, C.synth_baddate, C.time_filtered, C.time_failedeval,
	    C.aggr, C.slow, C.unsupported, nlong };
	for (int k = 0; k < CTR_TMPL; k++)
		if (vals[k])
			atomicAdd(&counters[k], (unsigned long long)vals[k]);
}

#endif /* DNG_JIT_HOT */

/* append to the miss list, or parse here when it is full */
__device__ __forceinline__ void fmiss_put(const FScanArgs &a, const STab &stab,
    u32 at, unsigned long long beg, unsigned long long end)
{
	if (at < a.miss_cap) {
		MissEnt e;
		e.beg = beg;
		e.end = end;
		a.miss[at] = e;
	} else {
		fmiss_inline(a.data, a.start, beg, end, a.plan, stab, &a.tab,
		    a.counters);
	}
}

/*
 * The matcher the run-time compiler generates for one scan's templates
 * (jit.cpp): fmatch() with the trie turned into straight-line code, literals as
 * immediates.  Returns 0, or 1 | defmask << 1.  Only the relocatable build of
 * this file (fast_jit.cu) calls it; it is resolved when that build is linked
 * with the generated code.
 */
extern "C" __device__ unsigned dng_jmatch(unsigned ra, unsigned len,
    unsigned active, unsigned caps);

template <int NSL, bool JIT>
__device__ __forceinline__ void fscan_body(const FScanArgs &a)
{
	constexpr u32 CHUNK = 32 * 16 * NSL, D0 = DNG_F_PRE;
	const u32 SLICE = 16 * a.wunits, W = 32 * SLICE;
	extern __shared__ __align__(128) u8 smem[];
#ifdef DNG_JIT_HOT
	const FPlan &F = dng_jplan;
#else
	const FPlan &F = *(const FPlan *)smem;
#endif
	u8 *sp = smem + FPLAN_SMEM;
	const u32 tmpl_sa = smem_u32(sp);
	sp += a.tmpl_bytes;
	STab stab;
	stab.s1 = (SSlot1 *)sp;
	sp += a.s1slots * sizeof (SSlot1);
	stab.s = (SSlot *)sp;
	sp += a.sslots * sizeof (SSlot);
	stab.mask1 = a.s1slots - 1;
	stab.mask = a.sslots - 1;
	const u32 caps_sa = smem_u32(sp);
	sp += a.nrows * DNG_F_NT * 4;

	const u32 tid = threadIdx.x;
	const u32 lane = tid & 31, wid = tid >> 5;
	/* this warp's window, newline positions (u16) and mbarrier: shared
	 * addresses */
	const u32 sb = smem_u32(sp) + wid * fwarp_bytes(a.wunits);
	const u32 nlpos = sb + W + DNG_F_SLACK;
	const u32 mbar = nlpos + 2 * DNG_F_NLCAP;

	{	/* plan, templates -> shared; clear the tally cache */
		const uint4 *src = (const uint4 *)a.fplan;
		uint4 *dst = (uint4 *)smem;
		for (u32 i = tid; i < FPLAN_SMEM / 16; i += blockDim.x)
			dst[i] = src[i];
		const uint4 *tsrc = (const uint4 *)a.tmpl;
		uint4 *tdst = (uint4 *)(smem + FPLAN_SMEM);
		for (u32 i = tid; i < a.tmpl_bytes / 16; i += blockDim.x)
			tdst[i] = tsrc[i];
		const uint4 z = make_uint4(0, 0, 0, 0);
		uint4 *tz = (uint4 *)stab.s1;
		const u32 tab_bytes = a.s1slots * (u32)sizeof (SSlot1) +
		    a.sslots * (u32)sizeof (SSlot);
		for (u32 i = tid; i < tab_bytes / 16; i += blockDim.x)
			tz[i] = z;
		if (lane == 0)
			mbar_init_sa(mbar, 1);
		/* the quotes after the buffer that end a runaway string scan
		 * (fscan.cuh) */
		if (lane < DNG_F_SLACK / 4)
			sts32(sb + W + 4 * lane, 0x22222222u);
	}
	__syncthreads();

	const bool use_tmpl = a.tmpl_bytes != 0;
	FSmem m;
	m.ra = 0;
	m.nodes = tmpl_sa + (u32)sizeof (THdr);
	m.leaves = tmpl_sa + a.leaf_off;
	m.pool = tmpl_sa + a.pool_off;
	m.caps = caps_sa + tid * 4;

	/* counters: records taken and aggregated per warp (the same value in
	 * every lane); the drop counters and `slow` in shared memory */
	__shared__ u32 s_drop[16];
	if (tid < 16)
		s_drop[tid] = 0;
	u32 ntmpl = 0, naggr = 0, parity = 0;
	const u32 ltmask = (1u << lane) - 1;

	/*
	 * Segments are handed out through a counter: a warp that finishes
	 * early takes the next one, so that the launch ends within a segment's
	 * time of its last warp (static shares left warps parked at the final
	 * barrier).  The first round is implicit -- warp gw takes
	 * segment gw, spread over the SMs -- the counter hands out the rest.
	 */
	const u32 nwarps = gridDim.x * (blockDim.x >> 5);
	const u32 gw = wid * gridDim.x + blockIdx.x;
	const u32 nseg = (a.nchunks + a.seg - 1) / a.seg;

	for (u32 seg = gw; seg < nseg; ) {
		/* the segment's bytes: [g0, g1) */
		const unsigned long long g0 = (unsigned long long)seg * a.seg *
		    CHUNK;
		const unsigned long long g1 = min(g0 + (unsigned long long)a.seg *
		    CHUNK, a.nbytes);
		/* the window [base, base + W); `next`: the first byte no pass
		 * has looked at; the open record's start, if it is known */
		unsigned long long base = g0 ? g0 - D0 : 0;
		unsigned long long next = g0 ? g0 : a.start;
		unsigned long long open_abs = a.start;
		for (bool first = true;; first = false) {
			const u32 dlen = (u32)min((unsigned long long)W,
			    a.nbytes - base);
			const u32 bulk = dlen & ~15u;

			__syncwarp();
			if (lane == 0) {
				asm volatile("fence.proxy.async.shared::cta;"
				    ::: "memory");
				if (bulk) {
					mbar_expect_tx_sa(mbar, bulk);
					tma_load_1d_sa(sb, a.data + base, bulk,
					    mbar);
				}
			}
			for (u32 i = bulk + lane; i < dlen; i += 32)
				sts8(sb + i, a.data[base + i]);
			/* (a short last window: the sentinel right behind it) */
			if (dlen < W && lane < 16)
				sts8(sb + dlen + lane, '"');
			if (bulk) {
				mbar_wait_sa(mbar, parity);
				parity ^= 1;
			}
			__syncwarp();

			/* the bytes whose newlines this pass takes: [lo, hi) of
			 * the window (those after the segment are the next
			 * one's) */
			const u32 lo = (u32)(next - base);
			const u32 hi = (u32)(min(base + dlen, g1) - base);
			if (first && g0) {
				/* where the open record starts: after the last
				 * newline of the pre-lap, which the lanes search
				 * together (16 bytes each) */
				const uint4 v = lds128(sb + D0 - 16 * (lane + 1));
				const u32 wd[4] = { v.x, v.y, v.z, v.w };
				u32 mine = 0;
#pragma unroll
				for (int j = 3; j >= 0; j--) {
					const u32 mk = nl_mask(wd[j]);
					if (mk && !mine)
						mine = D0 - 16 * (lane + 1) +
						    4 * j + ((31 - __clz(mk)) >> 3) + 1;
				}
				const u32 best = __reduce_max_sync(0xffffffffu, mine);
				open_abs = best ? base + best : ~0ull;
			}
			/* ... and in the window (-1: before it, or unknown) */
			const int beg0 = open_abs != ~0ull && open_abs >= base ?
			    (int)(open_abs - base) : -1;

			/* ---- newline index ---- */
			/*
			 * Bit j of hot: 16-byte unit j of the lane's slice holds a
			 * newline (a SWAR test with no false negatives); the units
			 * it flags are then looked at exactly, twice: to count, and
			 * -- once a shuffle scan has ordered the lanes -- to write
			 * the positions.
			 */
			const u32 c0 = lane * SLICE;
			u32 hot = 0, cnt = 0, one = 0;
#pragma unroll
			for (u32 j = 0; j < (u32)NSL + 2; j++) {
				/* (slices of NSL + 1 or NSL + 2 units) */
				if (j == NSL + 1 && a.wunits == NSL + 1)
					break;
				/* any byte <= '\n' in these 16?  (b - 0x0b borrows
				 * exactly for those; a borrow into the next byte can
				 * only add a flag) */
				const uint4 v = lds128(sb + c0 + 16 * j);
				u32 t = (v.x - 0x0b0b0b0bu) & ~v.x;
				t |= (v.y - 0x0b0b0b0bu) & ~v.y;
				t |= (v.z - 0x0b0b0b0bu) & ~v.z;
				t |= (v.w - 0x0b0b0b0bu) & ~v.w;
				if (t & 0x80808080u)
					hot |= 1u << j;
			}
#pragma unroll 1
			for (u32 hm = hot; hm; hm &= hm - 1) {
				const u32 p = c0 + 16 * (__ffs(hm) - 1);
				const uint4 v = lds128(sb + p);
				u32 m0 = nl_mask(v.x), m1 = nl_mask(v.y);
				u32 m2 = nl_mask(v.z), m3 = nl_mask(v.w);
				if (p < lo || p + 16 > hi) {
					/* the ends of the pass */
					m0 &= byte_range_mask(p, lo, hi);
					m1 &= byte_range_mask(p + 4, lo, hi);
					m2 &= byte_range_mask(p + 8, lo, hi);
					m3 &= byte_range_mask(p + 12, lo, hi);
				}
				const u32 k = __popc(m0) + __popc(m1) + __popc(m2) +
				    __popc(m3);
				/* (the usual case, one newline per lane: its
				 * position right away) */
				if (k == 1)
					one = p + (m0 ? 0 : m1 ? 4 : m2 ? 8 : 12) +
					    ((__ffs(m0 | m1 | m2 | m3) - 1) >> 3);
				cnt += k;
			}

			u32 incl = cnt;
#pragma unroll
			for (int d = 1; d < 32; d <<= 1) {
				const u32 y = __shfl_up_sync(0xffffffffu, incl, d);
				if (lane >= (u32)d)
					incl += y;
			}
			const u32 mybase = incl - cnt;
			const u32 total = __shfl_sync(0xffffffffu, incl, 31);
			const bool dense = total > DNG_F_NLCAP;
			if (dense) {
				/*
				 * Degenerate input (lines of a few bytes): one lane
				 * walks the window and hands every record to the
				 * general parser.
				 */
				if (lane == 0) {
					unsigned long long b = open_abs;
					for (u32 p = lo; p < hi; p++) {
						if (lds8(sb + p) != '\n')
							continue;
						const unsigned long long e = base + p;
						fmiss_put(a, stab, atomicAdd(a.miss_n, 1u),
						    b, e);
						b = e + 1;
					}
					open_abs = b;
				}
				open_abs = __shfl_sync(0xffffffffu, open_abs, 0);
				next = open_abs;
			} else if (total) {
				/* (cnt == 1: from a unit of one newline) */
				if (cnt == 1) {
					sts16(nlpos + 2 * mybase, one);
				} else if (cnt) {
					u32 idx = mybase;
#pragma unroll 1
					for (u32 hm = hot; hm; hm &= hm - 1) {
						const u32 p = c0 + 16 * (__ffs(hm) - 1);
#pragma unroll 1
						for (u32 q = 0; q < 4; q++) {
							u32 mk = nl_mask(lds32(sb + p + 4 * q));
#pragma unroll 1
							for (; mk; mk &= mk - 1) {
								const u32 pos = p + 4 * q +
								    ((__ffs(mk) - 1) >> 3);
								if (pos >= lo && pos < hi)
									sts16(nlpos + 2 * idx++,
									    pos);
							}
						}
					}
				}
				__syncwarp();
				/* the first 32 records, one per lane */
				const u32 take = min(total, 32u);
				if (lane == 0 && total > 32) {
					/* what the next window adds to this
					 * one: into L2 while the records are
					 * matched */
					const unsigned long long nb = (base +
					    lds16(nlpos + 2 * 31) + 1) & ~15ull;
					if (nb + W <= a.nbytes)
						asm volatile("cp.async.bulk."
						    "prefetch.L2.global [%0], %1;"
						    :: "l"(a.data + base + W),
						    "r"((u32)(nb - base)) : "memory");
				}

				const u32 r = lane;
				const bool have = r < take;
				int beg = 0;
				u32 end = 0;
				if (have) {
					end = lds16(nlpos + 2 * r);
					beg = r ? (int)lds16(nlpos + 2 * r - 2) +
					    1 : beg0;
				}
				/* (captures carry 12-bit offsets and lengths) */
				const bool inbuf = have && beg >= 0 &&
				    end - (u32)beg <= F_MAXLINE;
				const u32 len = inbuf ? end - (u32)beg : 0;
				m.ra = sb + (inbuf ? (u32)beg : 0);
				u32 defmask = 0;
				u32 fo = FO_MISS;
				bool matched;
				if (JIT) {
					const u32 r_ = dng_jmatch(m.ra, len, inbuf,
					    m.caps);
					matched = r_ & 1;
					defmask = r_ >> 1;
				} else {
					matched = use_tmpl &&
					    fmatch(m, len, inbuf, defmask);
				}
				if (matched) {
					double s0, s1;
					fo = fstage(m, F, defmask, s0, s1);
					u32 slow = 0;
					FKey k;
					if (fo == FO_AGGR && !fprep(m, F, defmask, s0,
					    s1, slow, k))
						fo = FO_MISS;
					if (fo == FO_AGGR) {
						if (k.hdr)
							ftally_short(m, F,
							    (const FPlan *)smem,
							    defmask, k, stab, a.tab,
							    smem_u32(&s_drop[15]));
						else if (!(
#ifdef DNG_JIT_HOT
						    F.short_keys ?
						    dng_cold_long_tally(m,
						    (const FPlan *)smem, defmask,
						    stab, &a.tab,
						    smem_u32(&s_drop[15])) :
#endif
						    flong_tally(m, F, (const FPlan *)
						    smem, defmask, stab, a.tab,
						    smem_u32(&s_drop[15]))))
							fo = FO_MISS;
						if (fo == FO_AGGR && slow)
							atomicAdd(&s_drop[1], 1u);
					}
				}
				const bool done = fo != FO_MISS;
				ntmpl += __popc(__ballot_sync(0xffffffffu, done));
				naggr += __popc(__ballot_sync(0xffffffffu,
				    fo == FO_AGGR));
				{
					/* dropped records: one shared atomic per
					 * outcome present in the warp */
					u32 dm = __ballot_sync(0xffffffffu,
					    fo >= FO_DS_FILTERED);
					while (dm) {
						const u32 f0 = __shfl_sync(0xffffffffu,
						    fo, __ffs(dm) - 1);
						const u32 same = __ballot_sync(
						    0xffffffffu, fo == f0);
						if (lane == 0)
							atomicAdd(&s_drop[f0],
							    (u32)__popc(same));
						dm &= ~same;
					}
				}
				/* what the F path did not take */
				const bool miss = have && !done;
				const u32 mm = __ballot_sync(0xffffffffu, miss);
				if (mm) {
					u32 mb = 0;
					if (lane == 0)
						mb = atomicAdd(a.miss_n,
						    (u32)__popc(mm));
					mb = __shfl_sync(0xffffffffu, mb, 0);
					if (miss)
						fmiss_put(a, stab, mb +
						    __popc(mm & ltmask), r ? base +
						    (u32)beg : open_abs, base + end);
				}
				__syncwarp();
				/* the cursor: past the last record taken */
				open_abs = next = base +
				    lds16(nlpos + 2 * (take - 1)) + 1;
			} else {
				/* no newline: the open record goes on past the
				 * window */
				next = base + dlen;
			}
			/* every newline of the segment taken? */
			if ((dense || total <= 32) && base + dlen >= g1)
				break;
			base = next & ~15ull;
		}
		/* an unterminated final line ends at a virtual newline: it is
		 * never templated (nothing terminates its scans) */
		if (g1 == a.nbytes && a.final && lane == 0 &&
		    lds8(sb + (u32)(a.nbytes - 1 - base)) != '\n') {
			/* the tail [open, end of input) */
			fmiss_put(a, stab, atomicAdd(a.miss_n, 1u), open_abs,
			    a.nbytes);
		}
		/* the next segment nobody has taken yet */
		if (lane == 0)
			seg = nwarps + atomicAdd(a.seg_next, 1u);
		seg = __shfl_sync(0xffffffffu, seg, 0);
	}

#ifdef DNG_JIT_HOT
	__syncthreads();
	dng_cold_flush(stab, a.s1slots, a.sslots, &a.tab);
#else
	fflush_tally(stab, a.s1slots, a.sslots, a.tab);
#endif
	if (lane == 0) {
		if (ntmpl) {
			atomicAdd(&a.counters[CTR_LINES], (unsigned long long)ntmpl);
			atomicAdd(&a.counters[CTR_TMPL], (unsigned long long)ntmpl);
		}
		if (naggr)
			atomicAdd(&a.counters[CTR_AGGR], (unsigned long long)naggr);
	}
	if (tid == 15 && s_drop[15])
		atomicAdd(&a.counters[CTR_OVER], (unsigned long long)s_drop[15]);
	if (tid < 15 && s_drop[tid]) {
		/* FO_* -> CTR_*; s_drop[1] = records that took a slow conversion */
		const int ctr = tid == 1 ? (int)CTR_SLOW :
		    tid == FO_DS_FILTERED ? (int)CTR_DS_FILTERED :
		    tid == FO_DS_FAILED ? (int)CTR_DS_FAILED :
		    tid == FO_USER_FILTERED ? (int)CTR_USER_FILTERED :
		    tid == FO_USER_FAILED ? (int)CTR_USER_FAILED :
		    tid == FO_SYNTH_UNDEF ? (int)CTR_SYNTH_UNDEF :
		    tid == FO_SYNTH_BADDATE ? (int)CTR_SYNTH_BADDATE :
		    tid == FO_TIME_FILTERED ? (int)CTR_TIME_FILTERED :
		    tid == FO_TIME_FAILED ? (int)CTR_TIME_FAILED : -1;
		if (ctr >= 0)
			atomicAdd(&a.counters[ctr], (unsigned long long)s_drop[tid]);
	}
}

#ifndef DNG_JIT_HOT
template <int NSL>
__global__ void __launch_bounds__(DNG_F_NT, 1)
scan_kernel_f(const FScanArgs a)
{
	fscan_body<NSL, false>(a);
}
#endif

#ifndef DNG_JIT_HOT
/* ---- the records the F path did not take ------------------------------------ */

struct FMissArgs {
	const u8 *data;
	unsigned long long start;
	const DevPlan *plan;
	u32 plan_bytes;
	unsigned long long *counters;
	GTable tab;
	u32 s1slots, sslots;
	const MissEnt *miss;
	const u32 *miss_n;
	u32 miss_cap;
};

#define DNG_MISS_NT 256

__global__ void __launch_bounds__(DNG_MISS_NT)
scan_miss_kernel(const FMissArgs a)
{
	const u32 n = min(*a.miss_n, a.miss_cap);
	if (blockIdx.x * DNG_MISS_NT >= n)
		return;
	extern __shared__ __align__(128) u8 smem[];
	DevPlan *sp = (DevPlan *)smem;
	STab stab;
	stab.s1 = (SSlot1 *)(smem + a.plan_bytes);
	stab.s = (SSlot *)(smem + a.plan_bytes + a.s1slots * sizeof (SSlot1));
	stab.mask1 = a.s1slots - 1;
	stab.mask = a.sslots - 1;
	const u32 tid = threadIdx.x;
	{
		const uint4 *src = (const uint4 *)a.plan;
		uint4 *dst = (uint4 *)sp;
		for (u32 i = tid; i < a.plan_bytes / 16; i += DNG_MISS_NT)
			dst[i] = src[i];
		const uint4 z = make_uint4(0, 0, 0, 0);
		uint4 *tz = (uint4 *)stab.s1;
		const u32 tab_bytes = a.s1slots * (u32)sizeof (SSlot1) +
		    a.sslots * (u32)sizeof (SSlot);
		for (u32 i = tid; i < tab_bytes / 16; i += DNG_MISS_NT)
			tz[i] = z;
	}
	__syncthreads();
	const DevPlan &P = *sp;
	LocalCounters C;
	C.lines = C.invalid_json = C.invalid_point = 0;
	C.ds_filtered = C.ds_failedeval = C.user_filtered = 0;
	C.user_failedeval = C.synth_undef = C.synth_baddate = 0;
	C.time_filtered = C.time_failedeval = C.aggr = C.slow = 0;
	C.unsupported = 0;
	u32 nlong = 0;
	u32 mctr[(MAX_METRICS - 1) * MCTR_PER];
	for (int k = 0; k < (MAX_METRICS - 1) * MCTR_PER; k++)
		mctr[k] = 0;
	for (u32 i = blockIdx.x * DNG_MISS_NT + tid; i < n;
	    i += gridDim.x * DNG_MISS_NT) {
		const MissEnt e = a.miss[i];
		unsigned long long q = e.beg;
		if (q == ~0ull) {
			q = e.end;
			while (q > a.start && a.data[q - 1] != '\n')
				q--;
			nlong++;
		}
		scan_one_global(a.data + q, (u32)min((unsigned long long)
		    DNG_MAXREC, e.end - q), P, stab, a.tab, C, mctr);
	}
	flush_tally(stab, a.s1slots, a.sslots, a.tab);
	flush_counters(a.counters, C, nlong, 0);
}

#endif /* DNG_JIT_HOT */

} /* namespace dng */
#endif
