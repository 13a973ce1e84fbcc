/*
 * kernel_choice.h: which kernel a scan launches -- CTA tiles (scan_kernel),
 * per-warp chunks (scan_kernel_w) or the F path (scan_kernel_f, then
 * scan_miss_kernel) -- and with how many warps the F kernel runs.  Results never
 * depend on the choice, only the speed does.
 *
 * Host-only and free of CUDA: api.cu takes the sample and the counters of
 * finished launches from the device and hands them to these functions, which
 * hold the whole policy.  tests/test_kernel_choice_host.py drives them on the
 * CPU.  The kernels share the geometry constants below.
 */
#ifndef DNG_KERNEL_CHOICE_H
#define DNG_KERNEL_CHOICE_H

#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* per-warp kernel: lines longer than its pre-lap take the HBM path, so it is
 * chosen for input whose sampled lines are at most this long */
#define DNG_W_MAXLINE 512
#define DNG_W_SLICE_MAX 208		/* largest lane slice: 13 x 16 bytes */
#define DNG_F_NLCAP 128			/* F kernel: newline positions per chunk */
#define DNG_F_NW 28			/* F kernel: most warps per CTA */
#define DNG_F_NW_START 24		/* ... and what a scan starts with */

namespace dng {

enum KernelMode { KC_AUTO, KC_TILE, KC_WARP, KC_FAST };
enum KernelKind { KK_TILE = 0, KK_WARP = 1, KK_F = 2 };	/* dng_scan_kernel_kind */

struct KernelChoice {
	int mode = KC_AUTO;
	bool f_ok = false;		/* the F path models the plan, DNG_FAST != 0 */
	bool f_fits = false;		/* its buffers fit at DNG_F_NW warps */
	bool warp = false;		/* per-warp chunks, not CTA tiles */
	bool f = false;			/* the F kernel */
	uint32_t f_nw = DNG_F_NW_START;	/* warps per CTA of the F kernel */
	uint32_t wslice = DNG_W_SLICE_MAX;	/* bytes per lane of a warp's chunk */
	uint32_t f_nsl = 13;		/* 16-byte units per F lane slice */
	double mean_line = 224;		/* of the last sample */
	bool sampled = false;
	int relearns = 0;
	/* counters of finished launches at the last learn, at the last look */
	unsigned long long learn_lines = 0, learn_tmpl = 0;
	unsigned long long seen_lines = 0, seen_long = 0;
	unsigned long long seen_over = 0, seen_aggr = 0;
};

/*
 * At open: what the plan allows and the settings DNG_KERNEL, DNG_FAST and
 * DNG_F_WARPS (null when unset).
 */
inline void kc_open(KernelChoice &c, bool fanout, bool f_modelled, bool f_fits,
    bool warp_fits, const char *kernel, const char *fast, const char *fwarps)
{
	/* a fan-out plan runs a long stage list per record and tallies many
	 * tuples: it ran faster on CTA tiles (whose warps move through the
	 * stages together and whose tally cache is larger) than on per-warp
	 * chunks */
	c.mode = fanout ? KC_TILE : KC_AUTO;
	if (kernel)	/* tuning/testing: force one kernel geometry */
		c.mode = !strcmp(kernel, "tile") ? KC_TILE :
		    !strcmp(kernel, "warp") ? KC_WARP :
		    !strcmp(kernel, "fast") ? KC_FAST : KC_AUTO;
	c.f_ok = f_modelled && !(fast && atoi(fast) == 0);
	c.f_fits = f_fits;
	/* forced F: every eligible plan takes it, whatever the templates
	 * cover; others choose as usual */
	if (c.mode == KC_FAST && !c.f_ok)
		c.mode = fanout ? KC_TILE : KC_AUTO;
	if (!warp_fits && c.mode != KC_FAST)
		c.mode = KC_TILE;
	c.warp = c.mode == KC_WARP;
	c.f = c.mode == KC_FAST && c.f_fits;
	/* 24 warps leave the F kernel's tally cache 30 KB more than 28 */
	c.f_nw = fwarps && atoi(fwarps) >= DNG_F_NW ? DNG_F_NW : DNG_F_NW_START;
}

/* a forced geometry needs nothing from a sample but its templates */
inline bool kc_wants_sample(const KernelChoice &c, bool templates)
{
	return templates || c.mode == KC_AUTO;
}

/*
 * The lane slice (16 x odd bytes) whose chunk holds the most records per
 * 32-lane pass, given the mean line, among those whose chunk holds at most
 * `cap` records with a quarter to spare.
 */
inline uint32_t kc_lane_slice(double mean, double cap)
{
	double best = -1;
	uint32_t pick = 112;
	for (uint32_t sl = 112; sl <= DNG_W_SLICE_MAX; sl += 32) {
		double recs = 32.0 * sl / mean;
		double passes = ceil((recs + 1.5) / 32.0);
		double util = recs / (32.0 * passes);
		if (recs * 1.25 <= cap && util >= best) {
			best = util;
			pick = sl;
		}
	}
	return pick;
}

/* the F templates learned from a sample (learned: none were built) */
struct KcTemplates {
	bool learned = false;
	bool blob = false;		/* not empty */
	size_t covered = 0;		/* sampled records they match */
	size_t lines = 0;		/* lines sampled */
};

/*
 * On a sample of the input: the head of the first data, or of the data about
 * to be launched when templates are learned again.
 */
inline void kc_sample(KernelChoice &c, const uint8_t *p, size_t n,
    const KcTemplates &t)
{
	size_t longest = 0, nl = 0, pos = 0;
	while (pos < n) {
		const void *q = memchr(p + pos, '\n', n - pos);
		const size_t end = q ? (size_t)((const uint8_t *)q - p) : n;
		longest = longest > end - pos ? longest : end - pos;
		if (!q)
			break;
		nl++;
		pos = end + 1;
	}
	const bool short_lines = longest <= DNG_W_MAXLINE;
	c.mean_line = nl ? (double)n / (double)nl : 224.0;
	c.wslice = kc_lane_slice(c.mean_line, HUGE_VAL);
	c.f_nsl = kc_lane_slice(c.mean_line, DNG_F_NLCAP) / 16;
	if (c.mode == KC_AUTO) {
		/* short lines: every warp stages its own chunk; otherwise CTA
		 * tiles, whose window holds long lines.  Once long lines were
		 * seen the tiles stay */
		c.warp = short_lines && (!c.sampled || c.warp);
		/* the F path pays when its templates take nearly every record
		 * and a chunk holds enough of them */
		if (t.learned)
			c.f = c.f_fits && short_lines && t.blob &&
			    t.covered * 10 >= t.lines * 9 &&
			    c.mean_line * DNG_F_NLCAP >= 32.0 * 16 * c.f_nsl * 1.5;
	}
	c.sampled = true;
}

/* counters of the launches that finished so far */
struct KcLive {
	unsigned long long lines, long_lines, templated, aggregated, overflowed;
};

/*
 * Before a launch: input that changes character mid-stream (another file,
 * another producer).  Returns whether to learn templates again from the data
 * about to be launched (a few times at most: each costs a stream
 * synchronisation); the caller then samples it and sets learn_lines and
 * learn_tmpl from the counters once the stream is idle.
 */
inline bool kc_counters(KernelChoice &c, const KcLive &v, bool templates)
{
	/* many lines longer than a warp's pre-lap: the tile kernel from here on */
	if (v.lines - c.seen_lines >= 64) {
		if (c.warp && c.mode == KC_AUTO &&
		    (v.long_lines - c.seen_long) * 16 > v.lines - c.seen_lines)
			c.warp = false;
		c.seen_lines = v.lines;
		c.seen_long = v.long_lines;
	}
	/* keys the F kernel's inline tally tier had no room for: fewer warps
	 * leave it more */
	if (c.f_nw > DNG_F_NW_START && v.aggregated - c.seen_aggr >= 4096) {
		if ((v.overflowed - c.seen_over) * 64 > v.aggregated - c.seen_aggr)
			c.f_nw = DNG_F_NW_START;
		c.seen_over = v.overflowed;
		c.seen_aggr = v.aggregated;
	}
	/* the F path only pays while it takes nearly every record: with more
	 * than a few percent going through the miss list, learn again; if that
	 * was already done, leave it to the general kernels (whose second tier
	 * runs from shared memory) */
	const unsigned long long dl = v.lines - c.learn_lines;
	const unsigned long long dt = v.templated - c.learn_tmpl;
	const bool fmiss = c.mode == KC_AUTO && (dl - dt) * 16 > dl;
	if (c.f && fmiss && dl > 200000 && c.relearns >= 1)
		c.f = false;
	if (!templates || c.relearns >= 3 || dl <= 200000 ||
	    !(dt * 2 < dl || (c.f && fmiss)))
		return false;
	c.relearns++;
	return true;
}

inline int kc_pick(const KernelChoice &c)
{
	return c.f ? KK_F : c.warp ? KK_WARP : KK_TILE;
}

} /* namespace dng */

#endif
