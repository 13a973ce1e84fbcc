/*
 * plan.h: the flat, device-resident form of one scan.
 *
 * A dng_plan is the reference's QueryConfig (lib/dragnet.js:28-77) plus the
 * datasource properties StreamScan needs (lib/stream-scan.js:40-94), compiled
 * once on the host into plain arrays the scan kernel copies to shared memory:
 *
 *   - a trie of "contexts" for jsprim.pluck-style dotted lookups
 *     (whole-key-first, then split at the first dot; lib/stream-synthetic.js:47),
 *   - krill predicates as short-circuit jump code
 *     (lib/krill-skinner-stream.js:29-52),
 *   - synthetic date fields (lib/stream-synthetic.js:37-85),
 *   - breakdown columns with their bucketizers (lib/dragnet.js:52-71).
 */
#ifndef DNG_PLAN_H
#define DNG_PLAN_H

#include <stdint.h>

namespace dng {

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

enum ValType : u8 {
	T_UNDEF = 0, T_NULL = 1, T_FALSE = 2, T_TRUE = 3,
	T_NUM = 4, T_STR = 5, T_OBJ = 6, T_ARR = 7
};

/* value flags */
enum : u8 {
	VF_ESCAPED = 1,		/* string contains a backslash escape */
	VF_SIMPLEINT = 2,	/* number is [-]digits, <= 15 digits, not "-0" */
	/* 4 = VF_BINARY (record.cuh): number held as a double */
	VF_INLINE = 8,		/* number is the value's `off` field itself */
};

enum : int {
	MAX_SLOTS = 32, MAX_CTX = 24, MAX_CANDS = 64, MAX_PATHS = 24,
	MAX_LEVELS = 8, MAX_CODE = 48, MAX_SYN = 12, MAX_COLS = 16,
	MAX_METRICS = 8,
	POOL_BYTES = 2048, KEY_MAX = 512
};

/* record flags produced by the parser */
enum : u32 {
	RF_INVALID = 1,		/* not valid JSON */
	RF_SLOW = 2,		/* took a slow path (escaped key compare, ...) */
	RF_UNSUPPORTED = 4,	/* device code cannot decide this record */
};

struct Cand {			/* a key that matters inside one context */
	u32 hash;		/* FNV-1a of the raw key bytes */
	u16 off, len;		/* key bytes in pool */
	int8_t term_slot;	/* slot receiving the value, or -1 */
	int8_t child_ctx;	/* context entered if the value is an object, or -1 */
	u16 pad;
};

struct Ctx {
	u64 bloom;		/* bit (hash & 63) for every candidate */
	u32 subtree_mask;	/* slots at or below this context */
	u16 cand_begin, cand_end;
	int8_t parent;
	u8 depth;		/* container depth at which this context lives */
	u16 arraylike;		/* a candidate is "length" or an array index:
				 * an ARRAY here would need index semantics */
};

struct PathInfo {
	u8 slot0;		/* level l of this path uses slot slot0 + l */
	u8 nlevels;		/* levels that may supply the value */
	u16 pad;
};

enum SrcKind : u8 { SRC_UNDEF = 0, SRC_PATH = 1, SRC_SYNTH = 2 };
struct Src { u8 kind; u8 idx; };

enum Op : u8 { OP_EQ = 0, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_TRUE };

struct Leaf {
	double cnum;		/* ToNumber(constant) */
	u16 coff, clen;		/* constant bytes in pool when cstr */
	int16_t jt, jf;		/* next leaf if true/false; -1 accept, -2 reject */
	u8 op;
	u8 cstr;		/* constant is a string */
	Src src;
	u32 pad;
};

struct Col {
	double step;
	Src src;
	u8 kind;		/* 0 discrete, 1 power-of-two, 2 linear */
	u8 pad[5];
};

enum : u8 { COL_DISCRETE = 0, COL_P2 = 1, COL_LINEAR = 2 };
enum : u8 { FMT_JSON = 0, FMT_SKINNER = 1 };

/*
 * Fast path: a per-plan byte automaton (record.cuh fast_step).  Every lane of
 * a warp feeds one byte of its own record per iteration through
 *     cls = fast.cls[byte];  e = fast.trans[state * FAST_NCLS + cls]
 * (low byte = next state, high byte = event flags), so the warp stays in
 * lock step; the plan's candidate keys are folded into the automaton as a
 * trie, so "is this key one we need" costs nothing per byte.  Only flagged
 * bytes (container open/close, a candidate key, the value after one) run
 * divergent code.  Anything the automaton does not model exactly (escapes in
 * keys, nesting > 31, a top-level scalar) ends in FS_FB and the record is
 * re-parsed by the general parser (parse_record).
 */
enum : int { FAST_NCLS = 64, FAST_MAXSTATES = 200, FAST_MAXKEYS = 48,
	FAST_MAXCTX = 12 };
enum : u8 {			/* event flags (high byte of a transition) */
	FE_PUSH = 1, FE_POP = 2, FE_OBJ = 4, FE_KEYHIT = 8,
	FE_VALSTART = 16, FE_VALEND_INCL = 32, FE_VALEND_EXCL = 64
};
enum : u8 {			/* fixed state numbers */
	FS_ERR = 0, FS_FIN = 1, FS_FB = 2, FS_START = 3, FS_DONE = 4,
	FS_AFTER_O = 5, FS_AFTER_A = 6, FS_OF = 7, FS_AF = 8, FS_KC = 9
};

struct FastTab {
	u8 cls[256];
	u8 candmap[FAST_MAXCTX * FAST_MAXKEYS][2];	/* [ctx][key] -> term, child */
	u8 ok;			/* tables are valid for this plan */
	u8 nstates, nkeys;
	u8 kc_base;		/* state kc_base + g = "key g just closed" */
	u8 stride;		/* classes per row of trans[] (<= FAST_NCLS) */
	u8 pad[3];
};

/*
 * One metric = one StreamScan of the reference (lib/stream-scan.js:40-94): user
 * filter, its synthetic date fields, time bounds, breakdown columns.  A plain
 * `dn scan` has one; `dn build` / index-scan fans one parsed record out to
 * several (lib/datasource-file.js:386-432).
 */
struct Metric {
	int16_t user_entry, time_entry;		/* -1 none */
	u8 syn0, nsyn;				/* range in DevPlan::syn */
	u8 col0, ncols;				/* range in DevPlan::col */
};

/*
 * The part of a plan the lock-step loop touches on every byte / event.  It is
 * the tail of DevPlan so that CTAs can copy a plan prefix that ends with just
 * the used rows of the transition table.
 */
struct alignas(16) HotPlan {
	Ctx ctx[MAX_CTX];
	FastTab fast;
	u8 nctx;
	u8 pad[7];
	/* LAST: only the first fast.nstates rows of fast.stride entries are
	 * meaningful and copied */
	u16 trans[FAST_MAXSTATES * FAST_NCLS];
};

struct DevPlan {
	Leaf code[MAX_CODE];
	Col col[MAX_COLS];
	Cand cand[MAX_CANDS];
	PathInfo path[MAX_PATHS];
	Src syn[MAX_SYN];
	Metric metric[MAX_METRICS];
	int16_t ds_entry;		/* datasource filter, -1 none */
	u8 format;
	u8 nmetrics;
	u8 ncand, npaths, nslots, ncode;
	int8_t root_ctx;	/* context of the record's fields object */
	int8_t sk_fields_slot, sk_value_slot;	/* json-skinner envelope */
	u8 pad[3];
	char pool[POOL_BYTES];
	HotPlan hot;		/* LAST */
};

/* bytes of a DevPlan a CTA copies into shared memory: everything up to and
 * including the used rows of the transition table (which is last) */
static inline u32 devplan_smem_bytes(const DevPlan &p)
{
	u32 rows = p.hot.fast.ok ? p.hot.fast.nstates : 0;
	u32 n = (u32)((const char *)p.hot.trans - (const char *)&p) +
	    rows * p.hot.fast.stride * 2u;
	return (n + 127u) & ~127u;
}

/* the global tally table of a scan: the host allocates it, the scan kernels
 * (scan_kernel.cuh) count into it */
struct GEntry {
	unsigned long long tag;		/* 0 empty, else hash | 1 */
	unsigned long long count;
	u32 koff;			/* key offset in arena + 1; 0 = unpublished */
	u32 klen;
};

struct GTable {
	GEntry *entries;
	u8 *arena;
	u32 *misc;			/* [0] arena cursor [1] nentries [2] status */
	u32 mask;			/* capacity - 1 */
	u32 arena_cap;
};

} /* namespace dng */

struct dng_plan {
	dng::DevPlan dev;
	/* host copies for result rendering, per metric */
	int nmetrics;
	int ncols[dng::MAX_METRICS];
	dng::u8 col_kind[dng::MAX_METRICS][dng::MAX_COLS];
	double col_step[dng::MAX_METRICS][dng::MAX_COLS];
};

/* host-only: compile plan JSON. Returns 0 or DNG_E*, message in err. */
int dng_plan_compile(const char *json, dng_plan *out, char *err,
    unsigned long errlen);

#endif
