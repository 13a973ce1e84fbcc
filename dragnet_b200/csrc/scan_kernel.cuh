/*
 * scan_kernel.cuh: the fused sm_90a scan kernels.
 *
 * One launch = one pass of dragnet's raw-scan pipeline over a byte range that
 * is resident in HBM:
 *
 *   lstream line split      (lib/format-json.js:32-33)   newline index
 *   JSON.parse + adapter    (lib/format-json.js:34-46)   tmpl_match() ->
 *                                                        fast_step() ->
 *                                                        parse_record()
 *   krill filters, dates,   (lib/stream-scan.js:56-86)   prepare_record(),
 *   time bounds                                          process_metric()
 *   skinner aggregator      (lib/dragnet-impl.js:48-51)  shared-memory tally
 *                                                        cache -> global table
 *
 * Two geometries over the same per-record code (scan_record, scan_tail,
 * scan_epilogue), one persistent 768-thread CTA per SM either way:
 *
 *   scan_kernel_w  every warp stages its own small chunk (TMA bulk copy into
 *                  a private slice of shared memory, its own mbarrier), indexes
 *                  it with shuffles and walks its records: no CTA barrier in
 *                  the loop.  For input with short lines.
 *   scan_kernel    the CTA stages a 156 KB tile, indexes it with a block scan
 *                  and its threads take one record each.  Any line length.
 *
 * A tile / chunk owns the records that END in it and stages a pre-lap before
 * itself for the record that straddles its start.  Group keys are counted in a
 * per-CTA shared-memory tally cache (exact: key bytes are compared, hashes
 * only pick the slot) that is flushed once per launch into the global table
 * with 64-bit atomics.  Input is read from HBM once (+ the pre-laps); no
 * intermediate columns are written.
 */
#ifndef DNG_SCAN_KERNEL_CUH
#define DNG_SCAN_KERNEL_CUH

#include <cuda_runtime.h>
#include "record.cuh"
#include "tmpl.cuh"
#include "kernel_choice.h"

namespace dng {

#ifndef DNG_NT
#define DNG_NT 768			/* threads per CTA */
#endif
#ifndef DNG_TILE
/* bytes of input a tile owns: DNG_NT slices of 13 x 16 bytes -- an odd number
 * of 16-byte units per lane keeps the per-lane uint4 reads of the newline
 * index free of shared-memory bank conflicts */
#define DNG_TILE (DNG_NT * 208)
#endif
#ifndef DNG_PRELAP
#define DNG_PRELAP 4096			/* bytes staged before the tile */
#endif
#ifndef DNG_CTAS_PER_SM
#define DNG_CTAS_PER_SM 1
#endif
#ifndef DNG_NLCAP
#define DNG_NLCAP 2048			/* newline positions per pass */
#endif
#define DNG_SSLOTS_MIN 64		/* shared tally slots: as many as fit (pow2) */
#define DNG_SSLOTS_MAX 4096
#define DNG_FASTMAX 16384		/* longest line the lock-step automaton takes */
#define DNG_SLACK 1024			/* readable bytes past the staged window */
#define DNG_MAXREC (1u << 24)		/* longest line handled */
#define DNG_NW (DNG_NT / 32)		/* warps per CTA */

enum { NCTR = 24, MCTR_PER = 8 };	/* + (MAX_METRICS-1) x MCTR_PER for fan-out */
enum {
	CTR_LINES = 0, CTR_INVALID_JSON, CTR_INVALID_POINT,
	CTR_DS_FILTERED, CTR_DS_FAILED, CTR_USER_FILTERED, CTR_USER_FAILED,
	CTR_SYNTH_UNDEF, CTR_SYNTH_BADDATE, CTR_TIME_FILTERED, CTR_TIME_FAILED,
	CTR_AGGR, CTR_SLOW, CTR_UNSUPPORTED, CTR_LONG, CTR_TMPL,
	CTR_OVER	/* F kernel: keys its inline tally tier had no room for */
};

enum { ST_TABLE_FULL = 1, ST_ARENA_FULL = 2 };

/*
 * Per-CTA tally cache, two tiers (hashes pick the slot, key BYTES decide):
 *   tier 1: a few 64-byte slots with the key inline -- the common
 *           low-cardinality case is decided entirely in shared memory;
 *   tier 2: many 16-byte slots holding only the global entry index; a hit is
 *           verified against the key bytes in the global arena (L2), so
 *           hundreds to thousands of tuples still avoid global atomics.
 * Whatever fits in neither goes to the global table directly.
 */
#define DNG_SKEY 40			/* inline key bytes per tier-1 slot */
struct SSlot1 {
	unsigned long long tag;		/* 0 empty; (hash|1) & ~READY; READY set
					 * once klen/key are written */
	u32 count;			/* records this launch (weights <= 255) */
	u32 klen;
	u32 gidx1;			/* global entry index + 1, set at flush */
	u32 pad;
	unsigned long long key[DNG_SKEY / 8];	/* zero padded */
};
struct SSlot {
	unsigned long long tag;		/* 0 empty; (hash|1) & ~READY */
	u32 count;
	u32 gidx1;			/* global entry index + 1; 0 = unpublished */
};

struct ScanArgs {
	const u8 *data;			/* 16-byte aligned */
	unsigned long long start;	/* first valid byte */
	unsigned long long nbytes;	/* end of valid bytes */
	const DevPlan *plan;
	unsigned long long *counters;
	GTable tab;
	u32 ntiles;
	u32 final;			/* treat an unterminated tail as a line */
	u32 plan_bytes;			/* devplan_smem_bytes(plan) */
	u32 sslots;			/* tier-2 slots (power of two) */
	u32 s1slots;			/* tier-1 slots (power of two) */
	u32 wslice;			/* per-warp kernel: bytes per lane (16 x odd) */
	const u8 *tmpl;			/* record templates (tmpl.h blob) or null */
	u32 tmpl_bytes;			/* multiple of 128, 0 = no templates */
};

#define DNG_READY 0x8000000000000000ull

/* the hot-plan copy is as large as the plan needs (devplan_smem_bytes) */
static constexpr size_t SMEM_NL = sizeof (u32) * DNG_NLCAP;
/* the slack lets lanes of a warp keep stepping (in an absorbing state) past
 * the end of their own short record while a neighbour finishes a longer one */
static constexpr size_t SMEM_DATA = DNG_PRELAP + DNG_TILE + DNG_SLACK + 128;
/* records the templates did not take, per pass (u16 indexes) */
static constexpr size_t SMEM_FQ = sizeof (u16) * DNG_NLCAP;
static constexpr size_t SMEM_FIXED = SMEM_NL + SMEM_FQ + SMEM_DATA;	/* + hot plan + slots */

/* ---- global table ------------------------------------------------------- */

/* find or insert key in the global table; returns the entry index, or
 * 0xffffffff when the table or the arena is exhausted (status is flagged) */
__device__ __forceinline__ u32 global_find(const GTable &t, u64 h,
    const u8 *key, u32 klen)
{
	unsigned long long claim = h | 1ull;
	u32 idx = (u32)(h >> 17) & t.mask;
	for (u32 probe = 0; probe <= t.mask; probe++) {
		GEntry *e = &t.entries[idx];
		unsigned long long tag =
		    *(volatile unsigned long long *)&e->tag;
		if (tag == 0) {
			unsigned long long old = atomicCAS(&e->tag, 0ull, claim);
			if (old == 0) {
				u32 need = (klen + 7) & ~7u;
				/* once the arena is full the offset stops growing
				 * (only keys claimed at that moment push it past
				 * the cap), so it cannot wrap around 2^32 */
				u32 off = *(volatile u32 *)&t.misc[0];
				if (off + need <= t.arena_cap)
					off = atomicAdd(&t.misc[0], need);
				if (off + need > t.arena_cap) {
					atomicOr(&t.misc[2], ST_ARENA_FULL);
					off = 0;
					klen = 0;
				} else {
					for (u32 k = 0; k < klen; k++)
						t.arena[off + k] = key[k];
				}
				e->klen = klen;
				__threadfence();
				atomicExch(&e->koff, off + 1);
				atomicAdd(&t.misc[1], 1u);
				return idx;
			}
			tag = old;
		}
		if (tag == claim) {
			u32 koff;
			while ((koff = *(volatile u32 *)&e->koff) == 0)
				;
			__threadfence();
			if (*(volatile u32 *)&e->klen == klen) {
				const u8 *s = t.arena + (koff - 1);
				u32 k = 0;
				while (k < klen && s[k] == key[k])
					k++;
				if (k == klen)
					return idx;
			}
		}
		idx = (idx + 1) & t.mask;
	}
	atomicOr(&t.misc[2], ST_TABLE_FULL);
	return 0xffffffffu;
}

__device__ __forceinline__ void global_add(const GTable &t, u64 h,
    const u8 *key, u32 klen, unsigned long long w)
{
	u32 idx = global_find(t, h, key, klen);
	if (idx != 0xffffffffu)
		atomicAdd(&t.entries[idx].count, w);
}

/* ---- shared tally cache ------------------------------------------------------ */

/*
 * Does global entry gi hold exactly this key?  Entries and arena bytes are
 * written by other SMs, and L1 is not coherent, so they are read with
 * ld.global.cg (L2); the handful of hot keys stays L2-resident.
 */
__device__ __forceinline__ bool entry_is(const GTable &gt, u32 gi,
    const unsigned long long *key, u32 klen)
{
	const GEntry *e = &gt.entries[gi];
	if (__ldcg(&e->klen) != klen)
		return false;
	const unsigned long long *s = (const unsigned long long *)
	    (gt.arena + (__ldcg(&e->koff) - 1));	/* 8-byte aligned */
	u32 nw = (klen + 7) >> 3;
	for (u32 k = 0; k < nw; k++) {
		unsigned long long a = __ldcg(&s[k]), b = key[k];
		if (k == nw - 1 && (klen & 7)) {
			unsigned long long m = (1ull << (8 * (klen & 7))) - 1;
			a &= m;
			b &= m;
		}
		if (a != b)
			return false;
	}
	return true;
}

struct STab {
	SSlot1 *s1;
	SSlot *s;
	u32 mask1, mask;		/* slots - 1 */
};

/* key: klen bytes, zero padded to a multiple of 8, 8-byte aligned */
__device__ __forceinline__ void shared_add(const STab &st, const GTable &gt,
    u64 h, const unsigned long long *key, u32 klen, unsigned long long w)
{
	const u32 nw = (klen + 7) >> 3;
	if (w <= 255) {
		const unsigned long long claim = (h | 1ull) & ~DNG_READY;
		/* tier 1: inline keys */
		if (klen <= DNG_SKEY) {
			u32 idx = (u32)(h >> 40) & st.mask1;
			for (u32 probe = 0; probe < 8; probe++) {
				SSlot1 *s = &st.s1[idx];
				unsigned long long tag =
				    *(volatile unsigned long long *)&s->tag;
				if (tag == 0) {
					unsigned long long old =
					    atomicCAS(&s->tag, 0ull, claim);
					if (old == 0) {
						s->klen = klen;
						for (u32 k = 0; k < nw; k++)
							s->key[k] = key[k];
						atomicAdd(&s->count, (u32)w);
						__threadfence_block();
						*(volatile unsigned long long *)
						    &s->tag = claim | DNG_READY;
						return;
					}
					tag = old;
				}
				if ((tag & ~DNG_READY) == claim) {
					while (!(tag & DNG_READY))
						tag = *(volatile unsigned long
						    long *)&s->tag;
					__threadfence_block();
					if (*(volatile u32 *)&s->klen == klen) {
						const volatile unsigned long
						    long *sk = s->key;
						u32 k = 0;
						while (k < nw && sk[k] == key[k])
							k++;
						if (k == nw) {
							atomicAdd(&s->count,
							    (u32)w);
							return;
						}
					}
				}
				idx = (idx + 1) & st.mask1;
			}
		}
		/* tier 2: compact slots, bytes verified in the arena */
		u32 idx = (u32)(h >> 28) & st.mask;
		for (u32 probe = 0; probe < 24; probe++) {
			SSlot *s = &st.s[idx];
			unsigned long long tag =
			    *(volatile unsigned long long *)&s->tag;
			if (tag == 0) {
				unsigned long long old =
				    atomicCAS(&s->tag, 0ull, claim);
				if (old == 0) {
					u32 gi = global_find(gt, h,
					    (const u8 *)key, klen);
					if (gi == 0xffffffffu) {
						*(volatile u32 *)&s->gidx1 =
						    0xffffffffu;
						return;	/* status is flagged */
					}
					atomicAdd(&s->count, (u32)w);
					__threadfence_block();
					*(volatile u32 *)&s->gidx1 = gi + 1;
					return;
				}
				tag = old;
			}
			if (tag == claim) {
				u32 g1;
				while ((g1 = *(volatile u32 *)&s->gidx1) == 0)
					;
				if (g1 != 0xffffffffu &&
				    entry_is(gt, g1 - 1, key, klen)) {
					atomicAdd(&s->count, (u32)w);
					return;
				}
			}
			idx = (idx + 1) & st.mask;
		}
	}
	global_add(gt, h, (const u8 *)key, klen, w);
}

/* ---- TMA / mbarrier helpers ----------------------------------------------- */

__device__ __forceinline__ u32 smem_u32(const void *p)
{
	return (u32)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ void mbar_init(u64 *bar, u32 count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;"
	    :: "r"(smem_u32(bar)), "r"(count) : "memory");
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(u64 *bar, u32 bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
	    :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void tma_load_1d(void *dst, const void *src,
    u32 bytes, u64 *bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::"
	    "complete_tx::bytes [%0], [%1], %2, [%3];"
	    :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
	    : "memory");
}

__device__ __forceinline__ void mbar_wait(u64 *bar, u32 parity)
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
	    :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}

__device__ __forceinline__ u32 lds32(u32 addr)
{
	u32 v;
	asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
	return v;
}

__device__ __forceinline__ u32 lds8(u32 addr)
{
	u32 v;
	asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
	return v;
}

__device__ __forceinline__ u32 lds16(u32 addr)
{
	u32 v;
	asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr));
	return v;
}

__device__ __forceinline__ uint4 lds128(u32 addr)
{
	uint4 v;
	asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
	    : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
	return v;
}

/*
 * Shared-memory access for tmpl_match(): the record in the staged tile (any
 * byte alignment: aligned 32-bit loads + a funnel shift) and the trie blob.
 */
struct TmplSmem {
	u32 ra;			/* record start */
	u32 nodes, leaves, pool;

	/* successive unaligned words; the aligned word after the one being
	 * consumed is always already in flight, so a scan loop does not wait
	 * for shared memory between its iterations */
	struct Cur {
		u32 wa, w0, w1, sh;
		__device__ __forceinline__ u32 next()
		{
			const u32 d = __funnelshift_r(w0, w1, sh);
			w0 = w1;
			wa += 4;
			w1 = lds32(wa);
			return d;
		}
	};
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
	__device__ __forceinline__ u32 byte(u32 off) const
	{
		return lds8(ra + off);
	}
	__device__ __forceinline__ u32 word(u32 off) const
	{
		Cur c = cursor(off);
		return c.next();
	}
	__device__ __forceinline__ TQuad node(u32 i) const
	{
		const uint4 v = lds128(nodes + i * 16);
		TQuad q;
		q.x = v.x; q.y = v.y; q.z = v.z; q.w = v.w;
		return q;
	}
	__device__ __forceinline__ TQuad lit2(u32 off) const
	{
		const uint4 v = lds128(pool + off);
		TQuad q;
		q.x = v.x; q.y = v.y; q.z = v.z; q.w = v.w;
		return q;
	}
	__device__ __forceinline__ u32 leaf(u32 i) const
	{
		return lds32(leaves + 4 * i);
	}
	__device__ __forceinline__ u32 pool32(u32 off) const
	{
		return lds32(pool + off);
	}

};

/* one automaton step on a class code (see record.cuh fast_step) */
#define FAST_STEP(cc, pos) do {						\
	u32 e_ = lds16(trb + (fs.state * stride + (cc)) * 2);		\
	fs.state = e_ & 0xff;						\
	if ((e_ >> 8) & fs.arm)						\
		fast_event(fs, H, R.slots, e_ >> 8, (pos));		\
} while (0)

/* exact per-byte equality mask: 0x80 in every byte of w equal to 0x0a */
__device__ __forceinline__ u32 nl_mask(u32 w)
{
	u32 x = w ^ 0x0a0a0a0au;
	u32 t = ((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x;
	return ~(t | 0x7f7f7f7fu);
}

/* 0x80 in byte k of the result iff lo <= p + k < hi (p = address of byte 0) */
__device__ __forceinline__ u32 byte_range_mask(u32 p, u32 lo, u32 hi)
{
	u32 m = 0;
#pragma unroll
	for (u32 k = 0; k < 4; k++)
		if (p + k >= lo && p + k < hi)
			m |= 0x80u << (8 * k);
	return m;
}

#ifndef DNG_JIT_HOT	/* (the LTO build of the F kernel: none of the general path) */
/* ---- one record ----------------------------------------------------------- */

/*
 * Fan-out (dn build / index-scan): the further metrics of an already parsed
 * and prepared record.  Out of line so that the single-metric path stays lean;
 * stage counters of metrics >= 1 are per-thread tallies in local memory.
 */
__device__ __noinline__ void scan_tail_fanout(const u8 *rec, const DevPlan &P,
    RecState &R, STab stab, const GTable &gt, LocalCounters &C, u32 *mctr,
    u64 w)
{
	__align__(8) u8 kbuf[KEY_MAX + 16];
	const unsigned long long *kw = (const unsigned long long *)kbuf;
	u32 klen;
	for (u32 mi = 1; mi < P.nmetrics; mi++) {
		LocalCounters T;
		T.user_filtered = T.user_failedeval = T.synth_undef = 0;
		T.synth_baddate = T.time_filtered = T.time_failedeval = 0;
		T.aggr = T.slow = T.unsupported = 0;
		if (process_metric(rec, P, mi, R, T, kbuf, klen))
			shared_add(stab, gt, key_hash_words(kw, klen), kw,
			    klen, w);
		/* per-thread tallies (local memory), reduced once per launch */
		u32 *mc = mctr + (mi - 1) * MCTR_PER;
		mc[0] += T.user_filtered;
		mc[1] += T.user_failedeval;
		mc[2] += T.synth_undef;
		mc[3] += T.synth_baddate;
		mc[4] += T.time_filtered;
		mc[5] += T.time_failedeval;
		mc[6] += T.aggr;
		C.slow += T.slow;
		C.unsupported += T.unsupported;
	}
}

/* stages after JSON decode + aggregation, for a parsed record */
__device__ __forceinline__ void scan_tail(const u8 *rec, u32 len,
    const DevPlan &P, RecState &R, STab stab, const GTable &gt,
    LocalCounters &C, u32 *mctr)
{
	(void)len;
	__align__(8) u8 kbuf[KEY_MAX + 16];
	u32 klen;
	u64 w;
	if (!prepare_record(rec, P, R, C, kbuf, w))
		return;
	const unsigned long long *kw = (const unsigned long long *)kbuf;
	if (process_metric(rec, P, 0, R, C, kbuf, klen))
		shared_add(stab, gt, key_hash_words(kw, klen), kw, klen,
		    w);
	if (P.nmetrics > 1)
		scan_tail_fanout(rec, P, R, stab, gt, C, mctr, w);
}

/* general (branchy, exact for everything) path */
__device__ __forceinline__ void scan_one(const u8 *rec, u32 len,
    const DevPlan &P, STab stab, const GTable &gt, LocalCounters &C,
    u32 *mctr)
{
	RecState R;
	C.lines++;
	if (len >= DNG_MAXREC) {
		C.unsupported++;
		return;
	}
	parse_record(rec, len, P, R);
	if (R.flags & RF_UNSUPPORTED)
		C.unsupported++;
	if (R.flags & RF_INVALID) {
		C.invalid_json++;
		return;
	}
	scan_tail(rec, len, P, R, stab, gt, C, mctr);
}

__device__ __noinline__ void scan_one_shared(const u8 *rec, u32 len,
    const DevPlan &P, STab stab, const GTable &gt, LocalCounters &C,
    u32 *mctr)
{
	scan_one(rec, len, P, stab, gt, C, mctr);
}

/* out-of-line copy for lines that begin before the staged window (rare):
 * keeps the hot shared-memory instantiation of the parser small */
__device__ __noinline__ void scan_one_global(const u8 *rec, u32 len,
    const DevPlan &P, STab stab, const GTable &gt, LocalCounters &C,
    u32 *mctr)
{
	scan_one(rec, len, P, stab, gt, C, mctr);
}

/*
 * What both kernels know while they walk the records of one staged window
 * (a tile of the CTA-wide kernel, a chunk of the per-warp kernel).
 */
struct WinCtx {
	const ScanArgs &a;
	const DevPlan &P;
	STab stab;
	TmplSmem tm;
	LocalCounters &C;
	u32 *mctr;
	u32 &ntmpl, &nlong;
	const u8 *sdata;		/* the window, in shared memory */
	unsigned long long ws;		/* its offset in the input */
	u32 wlen, lower;		/* valid bytes: [lower, wlen) */
	u32 wlim;			/* last shared address a lane may read */
	__device__ WinCtx(const ScanArgs &a_, const DevPlan &P_, STab st,
	    const TmplSmem &tm_, LocalCounters &C_, u32 *mc, u32 &nt, u32 &nl)
	    : a(a_), P(P_), stab(st), tm(tm_), C(C_), mctr(mc), ntmpl(nt),
	    nlong(nl), sdata(nullptr), ws(0), wlen(0), lower(0), wlim(0) {}
};

/*
 * One record per lane, the window's bytes [beg, end) (`end` is its newline).
 * Phase 0 tries the template trie and returns true for a record it did not
 * take (the caller queues it); phase 1 runs the lock-step byte automaton and
 * its fallbacks.  Every lane of the warp must call this (have = false for
 * lanes without a record): both matchers keep the warp in lock step.
 */
__device__ __forceinline__ bool scan_record(WinCtx &w, u32 phase, bool have,
    bool islong, u32 beg, u32 end)
{
	const DevPlan &P = w.P;
	const HotPlan &H = P.hot;
	const u8 *sdata = w.sdata;
	const u32 wlen = w.wlen;
	LocalCounters &C = w.C;
	const u32 len = end - beg;
	RecState R;
	bool parsed = false, failed = false;
	const u8 *rec = sdata;
	if (phase == 0) {
		/* newline-terminated lines inside the window */
		const bool elig = have && !islong && end < wlen &&
		    len <= TMPL_MAX_LINE;
		rec = sdata + beg;
		w.tm.ra = smem_u32(rec);
		parsed = tmpl_match(w.tm, len, R, elig);
		if (parsed) {
			C.lines++;
			w.ntmpl++;
		} else {
			failed = have;
		}
	} else {
		/*
		 * Lock-step fast path: every lane steps the plan's byte
		 * automaton over its own record; lanes without a (short,
		 * newline-terminated) record idle in the absorbing FIN state.
		 */
		const bool fast = have && !islong && H.fast.ok &&
		    len <= DNG_FASTMAX && end < wlen;
		FastState fs;
		fast_init(fs);
		if (!fast)
			fs.state = FS_FIN;
		rec = sdata + (fast ? beg : 0);
		u32 trip = __reduce_max_sync(0xffffffffu, fast ? len + 1 : 0);
		/*
		 * Four bytes per round: one aligned 32-bit shared load (+
		 * funnel shift for the record's byte alignment) and four
		 * independent class lookups are issued up front; only the
		 * state transition itself is a dependent chain.
		 */
		{
			const u32 ra = smem_u32(rec);
			const u32 sh = (ra & 3) * 8;
			u32 wa = ra & ~3u;
			/* lanes idling past their own line while a neighbour
			 * finishes a longer one must not run off the staged
			 * window */
			const u32 wlim = w.wlim;
			u32 w0 = lds32(wa);
			const u32 clsb = smem_u32(H.fast.cls);
			const u32 trb = smem_u32(H.trans);
			const u32 stride = H.fast.stride;
			for (u32 i = 0; i < trip; i += 4) {
				wa = min(wa + 4, wlim);
				u32 w1 = lds32(wa);
				u32 wd = __funnelshift_r(w0, w1, sh);
				w0 = w1;
				u32 c0 = lds8(clsb + (wd & 0xff));
				u32 c1 = lds8(clsb + ((wd >> 8) & 0xff));
				u32 c2 = lds8(clsb + ((wd >> 16) & 0xff));
				u32 c3 = lds8(clsb + (wd >> 24));
				FAST_STEP(c0, i);
				FAST_STEP(c1, i + 1);
				FAST_STEP(c2, i + 2);
				FAST_STEP(c3, i + 3);
			}
		}
		if (fast && fs.state == FS_FIN) {
			C.lines++;
			fast_finish(rec, fs, R);
			parsed = true;
		} else if (fast && fs.state == FS_ERR) {
			C.lines++;
			C.invalid_json++;
		} else if (have && !islong) {
			scan_one_shared(sdata + beg, len, P, w.stab, w.a.tab, C,
			    w.mctr);
		} else if (have) {
			/* the line began before the staged window: find its
			 * start in HBM and parse it from there */
			unsigned long long q = w.ws + w.lower;
			while (q > w.a.start && w.a.data[q - 1] != '\n')
				q--;
			w.nlong++;
			scan_one_global(w.a.data + q,
			    (u32)min((unsigned long long)DNG_MAXREC,
			    w.ws + end - q), P, w.stab, w.a.tab, C, w.mctr);
		}
	}
	if (parsed)
		scan_tail(rec, len, P, R, w.stab, w.a.tab, C, w.mctr);
	return failed;
}

#endif /* DNG_JIT_HOT */

/* end of a kernel, part 1: the CTA's tally cache -> the global table */
__device__ __forceinline__ void flush_tally(const STab &stab, u32 s1slots,
    u32 sslots, const GTable &tab)
{
	const u32 tid = threadIdx.x;
	__syncthreads();
	for (u32 i = tid; i < s1slots; i += blockDim.x) {
		const SSlot1 *s = &stab.s1[i];
		/* (a count of 0 is a key all of whose points weighed 0: it is
		 * still a point of the result, with value 0) */
		if (s->tag != 0)
			global_add(tab, key_hash_words(s->key, s->klen),
			    (const u8 *)s->key, s->klen,
			    (unsigned long long)s->count);
	}
	for (u32 i = tid; i < sslots; i += blockDim.x) {
		const SSlot *s = &stab.s[i];
		if (s->tag != 0 && s->gidx1 != 0 && s->gidx1 != 0xffffffffu &&
		    s->count)
			atomicAdd(&tab.entries[s->gidx1 - 1].count,
			    (unsigned long long)s->count);
	}
}

/* part 2: per-thread counters: warp reduce, one atomic per warp per counter */
__device__ __forceinline__ void flush_counters(unsigned long long *counters,
    const LocalCounters &C, u32 nlong, u32 ntmpl)
{
	const u32 lane = threadIdx.x & 31;
	u32 vals[NCTR];
	for (int k = 0; k < NCTR; k++)
		vals[k] = 0;
	vals[CTR_LINES] = C.lines;
	vals[CTR_INVALID_JSON] = C.invalid_json;
	vals[CTR_INVALID_POINT] = C.invalid_point;
	vals[CTR_DS_FILTERED] = C.ds_filtered;
	vals[CTR_DS_FAILED] = C.ds_failedeval;
	vals[CTR_USER_FILTERED] = C.user_filtered;
	vals[CTR_USER_FAILED] = C.user_failedeval;
	vals[CTR_SYNTH_UNDEF] = C.synth_undef;
	vals[CTR_SYNTH_BADDATE] = C.synth_baddate;
	vals[CTR_TIME_FILTERED] = C.time_filtered;
	vals[CTR_TIME_FAILED] = C.time_failedeval;
	vals[CTR_AGGR] = C.aggr;
	vals[CTR_SLOW] = C.slow;
	vals[CTR_UNSUPPORTED] = C.unsupported;
	vals[CTR_LONG] = nlong;
	vals[CTR_TMPL] = ntmpl;
#pragma unroll
	for (int k = 0; k <= CTR_TMPL; k++) {
		u32 v = vals[k];
		for (int d = 16; d > 0; d >>= 1)
			v += __shfl_xor_sync(0xffffffffu, v, d);
		if (lane == 0 && v)
			atomicAdd(&counters[k], (unsigned long long)v);
	}
}

#ifndef DNG_JIT_HOT
/* end of a kernel: shared tally cache -> global table, counters -> global */
__device__ __forceinline__ void scan_epilogue(const ScanArgs &a,
    const DevPlan &P, const STab &stab, const LocalCounters &C,
    const u32 *s_mctr, u32 nlong, u32 ntmpl)
{
	const u32 lane = threadIdx.x & 31;
	flush_tally(stab, a.s1slots, a.sslots, a.tab);

	if (P.nmetrics > 1) {
		for (u32 k = 0; k < (u32)(P.nmetrics - 1) * MCTR_PER; k++) {
			u32 v = s_mctr[k];
			for (int d = 16; d > 0; d >>= 1)
				v += __shfl_xor_sync(0xffffffffu, v, d);
			if (lane == 0 && v)
				atomicAdd(&a.counters[NCTR + k],
				    (unsigned long long)v);
		}
	}
	flush_counters(a.counters, C, nlong, ntmpl);
}

/*
 * Newlines in a lane's slice [c0, c1) of the window at shared address sbase
 * (bytes before `lower` do not count): their number, and << 16 the mask of the
 * 16-byte words that hold one.  Out of line on purpose: inlined into the
 * kernel, the loop's handful of live values were spilled to local memory and
 * reloaded on every iteration.
 */
__device__ __noinline__ u32 slice_newlines(u32 sbase, u32 c0, u32 c1, u32 lower)
{
	u32 cnt = 0, hot = 0;
	for (u32 p = c0; p < c1; p += 16) {
		const uint4 v = lds128(sbase + p);
		u32 m0 = nl_mask(v.x), m1 = nl_mask(v.y);
		u32 m2 = nl_mask(v.z), m3 = nl_mask(v.w);
		if (p + 16 > c1 || p < lower) {
			/* partial word: keep only bytes in [lower, c1) */
			m0 &= byte_range_mask(p, lower, c1);
			m1 &= byte_range_mask(p + 4, lower, c1);
			m2 &= byte_range_mask(p + 8, lower, c1);
			m3 &= byte_range_mask(p + 12, lower, c1);
		}
		const u32 k = __popc(m0) + __popc(m1) + __popc(m2) + __popc(m3);
		cnt += k;
		if (k)
			hot |= 1u << ((p - c0) >> 4);
	}
	return cnt | (hot << 16);
}

#endif /* DNG_JIT_HOT */

#ifndef DNG_NO_GENERAL_KERNELS	/* (fast_jit.cu only wants the shared parts) */
/* ---- the kernel ------------------------------------------------------------ */

__global__ void __launch_bounds__(DNG_NT, DNG_CTAS_PER_SM)
scan_kernel(const ScanArgs a)
{
	extern __shared__ __align__(128) u8 smem[];
	DevPlan *sp = (DevPlan *)smem;
	const u32 tab1_bytes = a.s1slots * (u32)sizeof (SSlot1);
	const u32 tab_bytes = tab1_bytes + a.sslots * (u32)sizeof (SSlot);
	STab stab;
	const u32 fixed_bytes = a.plan_bytes + a.tmpl_bytes;
	stab.s1 = (SSlot1 *)(smem + fixed_bytes);
	stab.s = (SSlot *)(smem + fixed_bytes + tab1_bytes);
	stab.mask1 = a.s1slots - 1;
	stab.mask = a.sslots - 1;
	u32 *nlpos = (u32 *)(smem + fixed_bytes + tab_bytes);
	u16 *failq = (u16 *)(smem + fixed_bytes + tab_bytes + SMEM_NL);
	u8 *sdata = smem + fixed_bytes + tab_bytes + SMEM_NL + SMEM_FQ;
	__shared__ __align__(8) u64 mbar;
	__shared__ u32 wsum[DNG_NT / 32];
	__shared__ u32 s_total;
	__shared__ u32 s_prev;		/* newline before the current pass */
	__shared__ u32 s_nfail;		/* records the templates did not take */
	u32 s_mctr[(MAX_METRICS - 1) * MCTR_PER];	/* thread-local */
	for (int k = 0; k < (MAX_METRICS - 1) * MCTR_PER; k++)
		s_mctr[k] = 0;

	const u32 tid = threadIdx.x;
	const u32 lane = tid & 31, wid = tid >> 5;

	{	/* plan -> shared, clear the table */
		const uint4 *src = (const uint4 *)a.plan;
		uint4 *dst = (uint4 *)sp;
		for (u32 i = tid; i < a.plan_bytes / 16; i += DNG_NT)
			dst[i] = src[i];
		const uint4 *tsrc = (const uint4 *)a.tmpl;
		uint4 *tdst = (uint4 *)(smem + a.plan_bytes);
		for (u32 i = tid; i < a.tmpl_bytes / 16; i += DNG_NT)
			tdst[i] = tsrc[i];
		uint4 z = make_uint4(0, 0, 0, 0);
		uint4 *tz = (uint4 *)stab.s1;
		for (u32 i = tid; i < tab_bytes / 16; i += DNG_NT)
			tz[i] = z;
		if (tid == 0)
			mbar_init(&mbar, 1);
	}
	__syncthreads();
	const DevPlan &P = *sp;		/* the plan, in shared memory */

	/* record templates, if the host learned any for this input */
	const bool use_tmpl = a.tmpl_bytes != 0;
	TmplSmem tm;
	tm.ra = 0;
	tm.nodes = smem_u32(smem + a.plan_bytes) + (u32)sizeof (THdr);
	tm.leaves = tm.pool = 0;
	if (use_tmpl) {
		const THdr *th = (const THdr *)(smem + a.plan_bytes);
		tm.leaves = smem_u32(smem + a.plan_bytes) + th->leaf_off;
		tm.pool = smem_u32(smem + a.plan_bytes) + th->pool_off;
	}
	u32 ntmpl = 0;

	LocalCounters C;
	C.lines = C.invalid_json = C.invalid_point = 0;
	C.ds_filtered = C.ds_failedeval = C.user_filtered = 0;
	C.user_failedeval = C.synth_undef = C.synth_baddate = 0;
	C.time_filtered = C.time_failedeval = C.aggr = C.slow = 0;
	C.unsupported = 0;
	u32 nlong = 0;
	u32 parity = 0;
	WinCtx w(a, P, stab, tm, C, s_mctr, ntmpl, nlong);
	w.sdata = sdata;
	w.wlim = smem_u32(sdata) + DNG_PRELAP + DNG_TILE + DNG_SLACK;

#ifdef DNG_PROFILE_PHASES
	long long pf_load = 0, pf_index = 0, pf_busy = 0, pf_phase = 0;
	long long pf_total = 0, pf_n = 0;
#define PF_CLK() clock64()
#endif
	for (u32 tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
#ifdef DNG_PROFILE_PHASES
		const long long pf_t0 = PF_CLK();
#endif
		const unsigned long long g0 = (unsigned long long)tile * DNG_TILE;
		const unsigned long long ws = g0 >= DNG_PRELAP ?
		    g0 - DNG_PRELAP : 0;
		unsigned long long we = g0 + DNG_TILE;
		if (we > a.nbytes)
			we = a.nbytes;
		const u32 wlen = (u32)(we - ws);
		const u32 bulk = wlen & ~15u;
		const u32 off0 = (u32)(g0 - ws);	/* tile start in window */

		if (tid == 0 && bulk) {
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
			mbar_expect_tx(&mbar, bulk);
			tma_load_1d(sdata, a.data + ws, bulk, &mbar);
			/* start pulling this CTA's next tile into L2 */
			unsigned long long nx = g0 +
			    (unsigned long long)gridDim.x * DNG_TILE;
			if (nx + DNG_TILE <= a.nbytes)
				asm volatile("cp.async.bulk.prefetch.L2.global "
				    "[%0], %1;" :: "l"(a.data + nx),
				    "r"((u32)DNG_TILE) : "memory");
		}
		for (u32 i = bulk + tid; i < wlen; i += DNG_NT)
			sdata[i] = a.data[ws + i];
		if (bulk) {
			mbar_wait(&mbar, parity);
			parity ^= 1;
		}
		__syncthreads();
#ifdef DNG_PROFILE_PHASES
		const long long pf_t1 = PF_CLK();
		pf_load += pf_t1 - pf_t0;
		long long pf_rec = 0;
#endif

		/* lowest window offset that holds valid input */
		const u32 lower = a.start > ws ? (u32)(a.start - ws) : 0;
		w.ws = ws;
		w.wlen = wlen;
		w.lower = lower;
		/* this thread's slice of the tile, 16-byte words */
		const u32 CH = DNG_TILE / DNG_NT;
		u32 c0 = off0 + tid * CH, c1 = c0 + CH;
		if (c1 > wlen)
			c1 = wlen;
		/* bit j of hot: 16-byte word j of the slice holds a newline */
		const u32 sn = slice_newlines(smem_u32(sdata), c0, c1, lower);
		u32 cnt = sn & 0xffff;
		const u32 hot = sn >> 16;
		/* an unterminated final line ends at a virtual newline */
		const bool vnl = a.final && we == a.nbytes && tid == DNG_NT - 1 &&
		    a.nbytes > a.start && wlen > 0 && wlen > lower &&
		    sdata[wlen - 1] != '\n';
		if (vnl)
			cnt++;

		/* block exclusive scan of cnt */
		u32 incl = cnt;
		for (int d = 1; d < 32; d <<= 1) {
			u32 y = __shfl_up_sync(0xffffffffu, incl, d);
			if (lane >= (u32)d)
				incl += y;
		}
		if (lane == 31)
			wsum[wid] = incl;
		__syncthreads();
		if (wid == 0) {
			u32 s = lane < DNG_NT / 32 ? wsum[lane] : 0;
			u32 si = s;
			for (int d = 1; d < 32; d <<= 1) {
				u32 y = __shfl_up_sync(0xffffffffu, si, d);
				if (lane >= (u32)d)
					si += y;
			}
			if (lane < DNG_NT / 32)
				wsum[lane] = si - s;
			if (lane == DNG_NT / 32 - 1)
				s_total = si;
		}
		__syncthreads();
		const u32 mybase = wsum[wid] + incl - cnt;
		const u32 total = s_total;

		for (u32 pass = 0; pass < total; pass += DNG_NLCAP) {
			/* write this pass's newline positions, in order */
			u32 idx = mybase;
			if (idx < pass + DNG_NLCAP && idx + cnt > pass) {
				for (u32 hm = hot; hm; hm &= hm - 1) {
					const u32 p = c0 + ((__ffs(hm) - 1) << 4);
					uint4 v = *(const uint4 *)(sdata + p);
					u32 mm[4] = { nl_mask(v.x), nl_mask(v.y),
					    nl_mask(v.z), nl_mask(v.w) };
					const bool partial = p + 16 > c1 || p < lower;
#pragma unroll
					for (u32 q = 0; q < 4; q++) {
						u32 m = mm[q];
						if (partial)
							m &= byte_range_mask(p + 4 * q,
							    lower, c1);
						while (m) {
							u32 b = (__ffs(m) - 1) >> 3;
							m &= m - 1;
							if (idx >= pass &&
							    idx < pass + DNG_NLCAP)
								nlpos[idx - pass] =
								    p + 4 * q + b;
							idx++;
						}
					}
				}
				if (vnl && idx >= pass && idx < pass + DNG_NLCAP)
					nlpos[idx - pass] = wlen;
			}
			__syncthreads();
			u32 n = total - pass;
			if (n > DNG_NLCAP)
				n = DNG_NLCAP;
			if (tid == 0)
				s_nfail = 0;
			__syncthreads();
			/*
			 * Phase 0 (only with templates): every record is tried
			 * against the template trie; what does not match is
			 * queued.  Phase 1: the queued records (or, without
			 * templates, all records) go through the byte automaton
			 * and its fallbacks, densely packed into warps again.
			 */
#ifdef DNG_PROFILE_PHASES
			const long long pf_t2 = PF_CLK();
#endif
			for (u32 phase = use_tmpl ? 0 : 1; phase < 2; phase++) {
			const u32 nn = (phase == 1 && use_tmpl) ? s_nfail : n;
			for (u32 rb = 0; rb < nn; rb += DNG_NT) {
				const bool have = rb + tid < nn;
				u32 r = rb + tid;
				if (have && phase == 1 && use_tmpl)
					r = failq[r];
				u32 end = 0, beg = 0;
				bool islong = false;
				if (have) {
					end = nlpos[r];
					if (r > 0) {
						beg = nlpos[r - 1] + 1;
					} else if (pass > 0) {
						beg = s_prev + 1;
					} else {
						u32 p = off0 < lower ? lower : off0;
						if (p > end)
							p = end;
						while (p > lower &&
						    sdata[p - 1] != '\n')
							p--;
						beg = p;
						if (p == lower && ws + lower > a.start &&
						    (p == 0 || sdata[p - 1] != '\n'))
							islong = true;
					}
				}
				const bool failed = scan_record(w, phase, have, islong,
				    beg, end);
				if (failed)
					failq[atomicAdd(&s_nfail, 1u)] = (u16)r;
			}
#ifdef DNG_PROFILE_PHASES
			if (phase == 0)
				pf_busy += PF_CLK() - pf_t2;
#endif
			__syncthreads();
			}
#ifdef DNG_PROFILE_PHASES
			pf_phase += PF_CLK() - pf_t2;
			pf_rec += PF_CLK() - pf_t2;
#endif
			__syncthreads();
			if (tid == 0)
				s_prev = nlpos[n - 1];
			__syncthreads();
		}
		__syncthreads();
#ifdef DNG_PROFILE_PHASES
		pf_total += PF_CLK() - pf_t0;
		pf_index += PF_CLK() - pf_t1 - pf_rec;
		pf_n++;
#endif
	}
#ifdef DNG_PROFILE_PHASES
	if (lane == 0) {
		atomicAdd(&a.counters[16], (unsigned long long)pf_busy);
		atomicAdd(&a.counters[17], (unsigned long long)pf_phase);
		atomicAdd(&a.counters[18], (unsigned long long)pf_n);
		atomicAdd(&a.counters[19], (unsigned long long)pf_load);
		atomicAdd(&a.counters[20], (unsigned long long)pf_index);
		atomicAdd(&a.counters[21], (unsigned long long)pf_total);
	}
#endif

	scan_epilogue(a, P, stab, C, s_mctr, nlong, ntmpl);
}

/* ---- the per-warp kernel ---------------------------------------------------- */

/*
 * Same algorithm, different geometry: every WARP stages its own small chunk of
 * the input (TMA into a private slice of shared memory, its own mbarrier),
 * finds the newlines in it with warp shuffles and walks its ~30 records, with
 * no CTA-wide barrier anywhere in the loop.  In the CTA-wide kernel above a
 * tile is one batch of records per warp between barriers, so half the warps of
 * an SM are parked at a barrier at any time; here all of them always have
 * work, which is what hides the latencies of the record matchers.
 *
 * A chunk owns the records that END in it and stages DNG_W_PRELAP bytes before
 * itself for the record that straddles its start; lines longer than that take
 * the HBM path, so the host picks this kernel only for input whose (sampled)
 * lines are short (DNG_W_MAXLINE) and the CTA-wide kernel otherwise.
 */
/* a chunk is 32 lane slices of a.wslice bytes (16 x an odd number, so that the
 * lanes' uint4 reads do not collide on banks); the host picks the slice that
 * puts just under 32 (or 64, ...) average records in a chunk (kernel_choice.h) */
#define DNG_W_CHUNK (32 * DNG_W_SLICE_MAX)	/* largest chunk: 6656 bytes */
#define DNG_W_PRELAP 768
#define DNG_W_SLACK 64
#define DNG_W_NLCAP 32				/* newline positions per pass */

static constexpr size_t SMEM_W_BUF = DNG_W_PRELAP + DNG_W_CHUNK + DNG_W_SLACK;
/* per warp: window, newline positions, fallback queue, mbarrier */
static constexpr size_t SMEM_W_WARP = SMEM_W_BUF + 4 * DNG_W_NLCAP +
    DNG_W_NLCAP + 16;
static constexpr size_t SMEM_W_FIXED = DNG_NW * SMEM_W_WARP + 128;

__global__ void __launch_bounds__(DNG_NT, 1)
scan_kernel_w(const ScanArgs a)
{
	extern __shared__ __align__(128) u8 smem[];
	DevPlan *sp = (DevPlan *)smem;
	const u32 tab1_bytes = a.s1slots * (u32)sizeof (SSlot1);
	const u32 tab_bytes = tab1_bytes + a.sslots * (u32)sizeof (SSlot);
	STab stab;
	const u32 fixed_bytes = a.plan_bytes + a.tmpl_bytes;
	stab.s1 = (SSlot1 *)(smem + fixed_bytes);
	stab.s = (SSlot *)(smem + fixed_bytes + tab1_bytes);
	stab.mask1 = a.s1slots - 1;
	stab.mask = a.sslots - 1;
	u32 s_mctr[(MAX_METRICS - 1) * MCTR_PER];	/* thread-local */
	for (int k = 0; k < (MAX_METRICS - 1) * MCTR_PER; k++)
		s_mctr[k] = 0;

	const u32 tid = threadIdx.x;
	const u32 lane = tid & 31, wid = tid >> 5;
	/* this warp's private slice */
	u8 *sdata = smem + fixed_bytes + tab_bytes + wid * SMEM_W_WARP;
	u32 *nlpos = (u32 *)(sdata + SMEM_W_BUF);
	u8 *failq = (u8 *)(nlpos + DNG_W_NLCAP);
	u64 *mbar = (u64 *)(failq + DNG_W_NLCAP);

	{	/* plan -> shared, clear the table */
		const uint4 *src = (const uint4 *)a.plan;
		uint4 *dst = (uint4 *)sp;
		for (u32 i = tid; i < a.plan_bytes / 16; i += DNG_NT)
			dst[i] = src[i];
		const uint4 *tsrc = (const uint4 *)a.tmpl;
		uint4 *tdst = (uint4 *)(smem + a.plan_bytes);
		for (u32 i = tid; i < a.tmpl_bytes / 16; i += DNG_NT)
			tdst[i] = tsrc[i];
		uint4 z = make_uint4(0, 0, 0, 0);
		uint4 *tz = (uint4 *)stab.s1;
		for (u32 i = tid; i < tab_bytes / 16; i += DNG_NT)
			tz[i] = z;
		if (lane == 0)
			mbar_init(mbar, 1);
	}
	__syncthreads();
	const DevPlan &P = *sp;

	const bool use_tmpl = a.tmpl_bytes != 0;
	TmplSmem tm;
	tm.ra = 0;
	tm.nodes = smem_u32(smem + a.plan_bytes) + (u32)sizeof (THdr);
	tm.leaves = tm.pool = 0;
	if (use_tmpl) {
		const THdr *th = (const THdr *)(smem + a.plan_bytes);
		tm.leaves = smem_u32(smem + a.plan_bytes) + th->leaf_off;
		tm.pool = smem_u32(smem + a.plan_bytes) + th->pool_off;
	}
	u32 ntmpl = 0;

	LocalCounters C;
	C.lines = C.invalid_json = C.invalid_point = 0;
	C.ds_filtered = C.ds_failedeval = C.user_filtered = 0;
	C.user_failedeval = C.synth_undef = C.synth_baddate = 0;
	C.time_filtered = C.time_failedeval = C.aggr = C.slow = 0;
	C.unsupported = 0;
	u32 nlong = 0;
	u32 parity = 0;
	WinCtx w(a, P, stab, tm, C, s_mctr, ntmpl, nlong);
	w.sdata = sdata;
	w.wlim = smem_u32(sdata) + (u32)SMEM_W_BUF;
	const u32 ltmask = (1u << lane) - 1;

	const u32 nwarps = gridDim.x * DNG_NW;
	const u32 chunk = 32 * a.wslice;
	for (u32 ch = blockIdx.x * DNG_NW + wid; ch < a.ntiles; ch += nwarps) {
		const unsigned long long g0 = (unsigned long long)ch * chunk;
		const unsigned long long ws = g0 >= DNG_W_PRELAP ?
		    g0 - DNG_W_PRELAP : 0;
		unsigned long long we = g0 + chunk;
		if (we > a.nbytes)
			we = a.nbytes;
		const u32 wlen = (u32)(we - ws);
		const u32 bulk = wlen & ~15u;
		const u32 off0 = (u32)(g0 - ws);	/* chunk start in window */

		__syncwarp();		/* the previous chunk is done with */
		if (lane == 0 && bulk) {
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
			mbar_expect_tx(mbar, bulk);
			tma_load_1d(sdata, a.data + ws, bulk, mbar);
			/* start pulling this warp's next chunk into L2 */
			unsigned long long nx = g0 +
			    (unsigned long long)nwarps * chunk;
			if (nx + chunk <= a.nbytes)
				asm volatile("cp.async.bulk.prefetch.L2.global "
				    "[%0], %1;" :: "l"(a.data + nx),
				    "r"(chunk) : "memory");
		}
		for (u32 i = bulk + lane; i < wlen; i += 32)
			sdata[i] = a.data[ws + i];
		if (bulk) {
			mbar_wait(mbar, parity);
			parity ^= 1;
		}
		__syncwarp();

		/* lowest window offset that holds valid input */
		const u32 lower = a.start > ws ? (u32)(a.start - ws) : 0;
		w.ws = ws;
		w.wlen = wlen;
		w.lower = lower;
		/* this lane's slice of the chunk, 16-byte words */
		u32 c0 = off0 + lane * a.wslice, c1 = c0 + a.wslice;
		if (c1 > wlen)
			c1 = wlen;
		/* bit j of hot: 16-byte word j of the slice holds a newline */
		const u32 sn = slice_newlines(smem_u32(sdata), c0, c1, lower);
		u32 cnt = sn & 0xffff;
		const u32 hot = sn >> 16;
		/* an unterminated final line ends at a virtual newline */
		const bool vnl = a.final && we == a.nbytes && lane == 31 &&
		    a.nbytes > a.start && wlen > 0 && wlen > lower &&
		    sdata[wlen - 1] != '\n';
		if (vnl)
			cnt++;

		/* warp exclusive scan of cnt */
		u32 incl = cnt;
		for (int d = 1; d < 32; d <<= 1) {
			u32 y = __shfl_up_sync(0xffffffffu, incl, d);
			if (lane >= (u32)d)
				incl += y;
		}
		const u32 mybase = incl - cnt;
		const u32 total = __shfl_sync(0xffffffffu, incl, 31);
		if (total == 0)
			continue;

		/*
		 * Where the first record starts: after the last newline of the
		 * pre-lap [lower, start0), which the lanes search together (32
		 * bytes each, nearest the chunk first).
		 */
		u32 beg0 = lower;
		bool islong0 = false;
		{
			u32 mine = 0;		/* 1 + position of a newline */
			if (off0 > lower && off0 >= 32 * (lane + 1)) {
				const u32 lo = off0 - 32 * (lane + 1);
				const uint4 v0 = *(const uint4 *)(sdata + lo);
				const uint4 v1 = *(const uint4 *)(sdata + lo + 16);
				const u32 wd[8] = { v0.x, v0.y, v0.z, v0.w,
				    v1.x, v1.y, v1.z, v1.w };
#pragma unroll
				for (int j = 7; j >= 0; j--) {
					u32 m = nl_mask(wd[j]);
					if (lo < lower)
						m &= byte_range_mask(lo + 4 * j,
						    lower, off0);
					if (m && !mine)
						mine = lo + 4 * j +
						    ((31 - __clz(m)) >> 3) + 1;
				}
			}
			const u32 best = __reduce_max_sync(0xffffffffu, mine);
			if (best)
				beg0 = best;
			else
				islong0 = ws + lower > a.start &&
				    (lower == 0 || sdata[lower - 1] != '\n');
		}

		u32 prev_end = 0;	/* newline that closed the previous pass */
		for (u32 pass = 0; pass < total; pass += DNG_W_NLCAP) {
			/* write this pass's newline positions, in order */
			u32 idx = mybase;
			if (idx < pass + DNG_W_NLCAP && idx + cnt > pass) {
				for (u32 hm = hot; hm; hm &= hm - 1) {
					const u32 p = c0 + ((__ffs(hm) - 1) << 4);
					uint4 v = *(const uint4 *)(sdata + p);
					u32 mm[4] = { nl_mask(v.x), nl_mask(v.y),
					    nl_mask(v.z), nl_mask(v.w) };
					const bool partial = p + 16 > c1 || p < lower;
#pragma unroll
					for (u32 q = 0; q < 4; q++) {
						u32 m = mm[q];
						if (partial)
							m &= byte_range_mask(p + 4 * q,
							    lower, c1);
						while (m) {
							u32 b = (__ffs(m) - 1) >> 3;
							m &= m - 1;
							if (idx >= pass &&
							    idx < pass + DNG_W_NLCAP)
								nlpos[idx - pass] =
								    p + 4 * q + b;
							idx++;
						}
					}
				}
				if (vnl && idx >= pass && idx < pass + DNG_W_NLCAP)
					nlpos[idx - pass] = wlen;
			}
			__syncwarp();
			u32 n = total - pass;
			if (n > DNG_W_NLCAP)
				n = DNG_W_NLCAP;
			u32 nfail = 0;
			/* phase 0: templates; phase 1: what they did not take
			 * (or, without templates, everything) */
			for (u32 phase = use_tmpl ? 0 : 1; phase < 2; phase++) {
				const u32 nn = (phase == 1 && use_tmpl) ? nfail : n;
				for (u32 rb = 0; rb < nn; rb += 32) {
					const bool have = rb + lane < nn;
					u32 r = rb + lane;
					if (have && phase == 1 && use_tmpl)
						r = failq[r];
					u32 end = 0, beg = 0;
					bool islong = false;
					if (have) {
						end = nlpos[r];
						if (r > 0) {
							beg = nlpos[r - 1] + 1;
						} else if (pass > 0) {
							beg = prev_end + 1;
						} else {
							beg = beg0 < end ? beg0 : end;
							islong = islong0;
						}
					}
					const bool failed = scan_record(w, phase, have,
					    islong, beg, end);
					const u32 fm = __ballot_sync(0xffffffffu, failed);
					if (failed)
						failq[nfail + __popc(fm & ltmask)] = (u8)r;
					nfail += __popc(fm);
				}
				__syncwarp();
			}
			prev_end = nlpos[n - 1];
			__syncwarp();
		}
	}

	scan_epilogue(a, P, stab, C, s_mctr, nlong, ntmpl);
}

/* gather occupied entries: out[i] = {koff-1, klen, count} */
struct OutEntry {
	unsigned long long count;
	u32 koff, klen;
};

__global__ void compact_kernel(const GEntry *entries, u32 cap, OutEntry *out,
    u32 *nout)
{
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < cap;
	    i += gridDim.x * blockDim.x) {
		if (entries[i].tag != 0) {
			u32 p = atomicAdd(nout, 1u);
			out[p].count = entries[i].count;
			out[p].koff = entries[i].koff - 1;
			out[p].klen = entries[i].klen;
		}
	}
}

/* first and last '\n' in data[lo, hi): *first = min pos, *last = max pos + 1 */
__global__ void find_nl_kernel(const u8 *data, unsigned long long lo,
    unsigned long long hi, unsigned long long *first, unsigned long long *last)
{
	for (unsigned long long i = lo + blockIdx.x * (unsigned long long)
	    blockDim.x + threadIdx.x; i < hi;
	    i += (unsigned long long)gridDim.x * blockDim.x) {
		if (data[i] == '\n') {
			atomicMin(first, i);
			atomicMax(last, i + 1);
		}
	}
}

#endif /* DNG_NO_GENERAL_KERNELS */

} /* namespace dng */
#endif
