/*
 * inflate_split.cuh: one gzip file decoded by many warps at once, its
 * DEFLATE stream cut into chunks at block starts found on the device
 * (speculative block-parallel decoding, as pugz and rapidgzip do it on CPUs).
 * The same source runs as one lane on the host
 * (tests/hostcheck/inflate_split_check.cpp).
 *
 *   1. split_find: for each chunk after the first, the first bit in it where
 *      a dynamic-Huffman block header parses under the decoder's own rules
 *      (InflaterT::build_dynamic), its candidate.  A true block start always
 *      passes; a false one may too.
 *   2. split_decode: each chunk decoded from its candidate (chunk 0 from bit
 *      0) into 16-bit symbols, a marker 256 + i standing for byte i of the
 *      32 KiB before the chunk, until a block starts exactly at a later
 *      chunk's candidate (it "lands" there), the stream ends, an error, or it
 *      runs out of room.  Member ends are recorded with their CRC-32 and
 *      ISIZE.
 *   3. split_chain (host): chunk 0 is proven; a chunk a proven chunk landed
 *      on is proven.  A proven decode lands only on true block starts, so
 *      the chunks nothing landed on were false starts and are dropped.
 *   4. split_resolve: each proven chunk's markers read the resolved bytes
 *      before it: the last 32 KiB of every chunk in chain order, then the
 *      rest of every chunk at once.
 *   5. split_member_ok: each member's CRC-32 over pieces, joined; ISIZE.
 *
 * The split path never reports damage: anything it cannot vouch for (an
 * error in a proven chunk, a marker before its member's start, a CRC or
 * ISIZE mismatch) sends the file back to inflate_one, whose answer stands.
 */
#ifndef DNG_INFLATE_SPLIT_CUH
#define DNG_INFLATE_SPLIT_CUH

#include <stdint.h>

#include <vector>

#include "inflate.cuh"

namespace dng {

/* the finder's tables, one set per lane: no fast tables (every symbol is
 * decoded bit by bit), so that 32 sets fit in a warp's shared memory */
struct InfHeadTables {
	enum { LBITS = 0, DBITS = 0 };
	uint16_t lcount[16], loffs[16], lfirst[16];
	uint16_t dcount[16], doffs[16], dfirst[16];
	uint16_t lsym[288], dsym[32];
	uint16_t lfast[1];
	uint16_t dfast[1];
	uint8_t lens[288 + 32];
	uint32_t fixed;
};

/* ---- 1. candidate block starts --------------------------------------------- */

/* whether a dynamic-Huffman block header (either BFINAL) parses at `bit` */
DNG_HDI bool split_header_at(const uint8_t *in, uint64_t n, uint64_t bit,
    InfHeadTables *T)
{
	const uint64_t i = bit >> 3;
	if (i + 3 > n)	/* (a real one is followed by codes and a trailer) */
		return false;
	/* BTYPE 10, HLIT <= 29, HDIST <= 29: the first 17 bits */
	uint32_t v = (uint32_t)in[i] | (uint32_t)in[i + 1] << 8 |
	    (uint32_t)in[i + 2] << 16 | (i + 3 < n ? (uint32_t)in[i + 3] << 24 :
	    0u);
	v >>= bit & 7;
	if (((v >> 1) & 3) != 2 || ((v >> 3) & 31) > 29 || ((v >> 8) & 31) > 29)
		return false;
	InflaterT<uint8_t, InfOneLane, InfHeadTables> f;
	f.reset();
	f.in = in;
	f.n = n;
	f.out = nullptr;
	f.cap = 0;
	f.T = T;
	f.seek(bit);
	uint32_t last, type;
	return f.bits(1, last) && f.bits(2, type) && f.build_dynamic();
}

struct SplitFind {
	const uint8_t *in;
	uint64_t in_len;
	uint64_t lo, hi;	/* the chunk's bits */
	uint64_t *cand;		/* out: the first candidate, or INF_NOSTART */
};

/* lanes test neighbouring bits; T: one table set per lane */
template <class Lanes>
DNG_HDI void split_find(const SplitFind &j, InfHeadTables *T, Lanes L)
{
	uint64_t found = INF_NOSTART;
	for (uint64_t b0 = j.lo; b0 < j.hi; b0 += L.n()) {
		const uint64_t b = b0 + L.lane();
		const uint32_t m = L.ballot(b < j.hi &&
		    split_header_at(j.in, j.in_len, b, T + L.lane()));
		if (m) {
#ifdef __CUDA_ARCH__
			found = b0 + __ffs(m) - 1;
#else
			found = b0 + __builtin_ctz(m);
#endif
			break;
		}
	}
	if (L.lane() == 0)
		*j.cand = found;
}

/* ---- 2. speculative decode -------------------------------------------------- */

struct SplitJob {
	const uint8_t *in;
	uint64_t in_len;
	const uint64_t *cand;	/* the file's candidates (cand[0] unused) */
	uint16_t *out;
	uint64_t cap;		/* symbols */
	InfMember *mem;
	uint32_t k, nchunks;	/* this chunk of the file's */
	uint32_t mcap, pad;	/* member slots in mem */
};

struct SplitRes {
	uint64_t start, end;	/* input bits */
	uint64_t out_len;	/* symbols */
	uint64_t bit;		/* of an error */
	uint32_t status;	/* INF_*, or SPLIT_NOSTART */
	uint32_t kind;
	uint32_t land;		/* the chunk it landed on, or INF_NOLAND */
	uint32_t members;	/* member ends in mem */
};

enum { SPLIT_NOSTART = 3 };	/* a chunk without a candidate */

template <class Lanes>
DNG_HDI void split_decode(const SplitJob &j, InfTables *T, Lanes L,
    SplitRes &r)
{
	const uint64_t start = j.k ? j.cand[j.k] : 0;
	r.start = start;
	r.end = start;
	r.out_len = 0;
	r.bit = 0;
	r.kind = 0;
	r.land = INF_NOLAND;
	r.members = 0;
	if (start == INF_NOSTART) {
		r.status = SPLIT_NOSTART;
		return;
	}
	InflaterT<uint16_t, Lanes, InfTables> f;
	f.reset();
	f.in = j.in;
	f.n = j.in_len;
	f.out = j.out;
	f.cap = j.cap;
	f.T = T;
	f.L = L;
	if (j.k) {
		f.seek(start);
		f.window = true;
	}
	f.cand = j.cand + j.k + 1;
	f.ncand = j.nchunks - j.k - 1;
	f.mem = j.mem;
	f.mcap = j.mcap;
	InfResult ir;
	f.run(ir);
	r.end = f.bitpos();
	r.out_len = ir.out_len;
	r.bit = ir.bit;
	r.status = ir.status;
	r.kind = ir.kind;
	r.members = ir.members;
	if (f.land != INF_NOLAND)
		r.land = j.k + 1 + f.land;
}

/* the room a chunk of `cbytes` of a file's `size` compressed bytes gets
 * first, in symbols: its share of the file's output hint, with a margin */
inline uint64_t split_room(uint64_t hint, uint64_t size, uint64_t cbytes)
{
	const double share = size ? (double)hint * cbytes / size : 0;
	return ((uint64_t)(share * 1.25) + 32768 + 7) & ~(uint64_t)7;
}

enum { SPLIT_MSLOTS = 4 };	/* member slots a chunk gets first */

/* chunk k of n of a file of `size` bytes: [split_cut(k), split_cut(k + 1)) */
DNG_HDI uint64_t split_cut(uint64_t size, uint32_t n, uint32_t k)
{
	return size / n * k + size % n * k / n;
}

/* ---- 3. the chain (host) ----------------------------------------------------- */

enum { CHAIN_END = 0, CHAIN_ROOM = 1, CHAIN_FAIL = 2 };

/*
 * The proven chunks of a file, in order: chunk 0, then each chunk the last
 * one landed on.  CHAIN_END: the last decoded to the end of the stream;
 * CHAIN_ROOM: it ran out of room (decode it again in more); CHAIN_FAIL: it
 * failed.
 */
inline int split_chain(const SplitRes *r, std::vector<uint32_t> &proven)
{
	proven.clear();
	for (uint32_t k = 0;;) {
		proven.push_back(k);
		if (r[k].status == INF_ROOM)
			return CHAIN_ROOM;
		if (r[k].status != INF_DONE)
			return CHAIN_FAIL;
		if (r[k].land == INF_NOLAND)
			return CHAIN_END;
		k = r[k].land;
	}
}

/* after CHAIN_ROOM: the chunks to decode again in more room, the chain's
 * last and each later one that ran out (earlier ones are settled) */
inline void split_redo(const SplitRes *r, uint32_t nchunks,
    const std::vector<uint32_t> &proven, std::vector<uint32_t> &redo)
{
	redo.clear();
	const uint32_t at = proven.back();
	redo.push_back(at);
	for (uint32_t k = at + 1; k < nchunks; k++)
		if (r[k].status == INF_ROOM)
			redo.push_back(k);
}

/* the candidates nothing landed on */
inline uint32_t split_false_starts(const SplitRes *r, uint32_t nchunks,
    const std::vector<uint32_t> &proven)
{
	uint32_t n = 0;
	for (uint32_t k = 1, i = 1; k < nchunks; k++) {
		while (i < proven.size() && proven[i] < k)
			i++;
		if (r[k].status != SPLIT_NOSTART &&
		    !(i < proven.size() && proven[i] == k))
			n++;
	}
	return n;
}

/* a file's output laid out from a CHAIN_END chain */
struct SplitLayout {
	uint64_t len = 0;			/* bytes */
	std::vector<uint64_t> off;		/* per proven chunk */
	std::vector<uint32_t> minidx;		/* per proven chunk */
	std::vector<uint64_t> mstart, mend;	/* per member */
	std::vector<uint32_t> crc, isize;
};

/*
 * mem[k]: chunk k's member records.  A chunk's markers must not reach before
 * the member it starts in: those below minidx are refused (a valid stream
 * has none).
 */
inline void split_layout(const SplitRes *r, const InfMember *const *mem,
    const std::vector<uint32_t> &proven, SplitLayout &o)
{
	o = SplitLayout();
	uint64_t off = 0, s = 0;	/* s: where the current member began */
	for (const uint32_t k : proven) {
		const uint64_t d = off - s;
		o.off.push_back(off);
		o.minidx.push_back(d >= 32768 ? 0 : (uint32_t)(32768 - d));
		for (uint32_t m = 0; m < r[k].members; m++) {
			const uint64_t e = off + mem[k][m].end;
			o.mstart.push_back(s);
			o.mend.push_back(e);
			o.crc.push_back(mem[k][m].crc);
			o.isize.push_back(mem[k][m].isize);
			s = e;
		}
		off += r[k].out_len;
	}
	o.len = off;
}

/* ---- 4. resolve ---------------------------------------------------------------- */

struct SplitPiece {		/* a proven chunk, as the resolve kernels see it */
	const uint16_t *sym;
	uint8_t *dst;		/* the file's output */
	uint64_t off, len;	/* its place there; its symbols */
	uint32_t minidx;
	uint32_t file;		/* its file's flag */
};

/* where split_resolve's first pass starts: the chunk's last 32 KiB */
DNG_HDI uint64_t split_tail(const SplitPiece &p)
{
	return p.len > 32768 ? p.len - 32768 : 0;
}

/* symbols [lo, hi) of a chunk to bytes, thread t of nt; false: a marker
 * before its member */
DNG_HDI bool split_resolve(const SplitPiece &p, uint64_t lo, uint64_t hi,
    uint32_t t, uint32_t nt)
{
	bool ok = true;
	uint8_t *d = p.dst + p.off;
	for (uint64_t i = lo + t; i < hi; i += nt) {
		const uint32_t s = p.sym[i];
		if (s < 256) {
			d[i] = (uint8_t)s;
		} else if (s - 256 < p.minidx) {
			ok = false;
		} else {
			d[i] = d[(int64_t)(s - 256) - 32768];
		}
	}
	return ok;
}

/* ---- 5. member checks ------------------------------------------------------------ */

enum { SPLIT_CRC_PIECE = 32768 };

struct CrcPiece {
	const uint8_t *p;
	uint64_t len;
};

struct CrcMember {
	uint32_t p0, p1;	/* its pieces */
	uint32_t crc, isize;	/* from its trailer */
	uint64_t len;
	uint32_t file, pad;
};

/* a member's pieces' CRCs joined in order, then checked; lanes take runs */
template <class Lanes>
DNG_HDI bool split_member_ok(const CrcMember &m, const CrcPiece *pieces,
    const uint32_t *crcs, Lanes L)
{
	const uint32_t np = m.p1 - m.p0;
	const uint32_t per = (np + L.n() - 1) / L.n();
	const uint32_t a = m.p0 + (per * L.lane() < np ? per * L.lane() : np);
	const uint32_t b = m.p0 + (per * (L.lane() + 1) < np ?
	    per * (L.lane() + 1) : np);
	uint32_t mine = 0, op = 0;
	uint64_t mlen = 0, oplen = ~0ull;
	for (uint32_t i = a; i < b; i++) {
		if (pieces[i].len != oplen) {
			oplen = pieces[i].len;
			op = crc32_shift(oplen);
		}
		mine = crc32_mulmod(op, mine) ^ crcs[i];
		mlen += pieces[i].len;
	}
	uint32_t crc = 0;
	for (uint32_t l = 0; l < L.n(); l++) {
		const uint32_t c = L.bcast(mine, l);
		const uint64_t n = (uint64_t)L.bcast((uint32_t)mlen, l) |
		    (uint64_t)L.bcast((uint32_t)(mlen >> 32), l) << 32;
		crc = crc32_combine(crc, c, n);
	}
	return crc == m.crc && m.isize == (uint32_t)m.len;
}

/* ---- the kernels --------------------------------------------------------------- */

#ifdef __CUDACC__
enum { SPLIT_WARPS = 4 };	/* warps per CTA of split_decode_kernel */

/* one warp per chunk (after each file's first) */
__global__ void __launch_bounds__(32)
split_find_kernel(const SplitFind *jobs, uint32_t njobs)
{
	__shared__ InfHeadTables tabs[32];
	for (uint32_t j = blockIdx.x; j < njobs; j += gridDim.x)
		split_find(jobs[j], tabs, InfLanes());
}

/* one warp per chunk, taken from *next in the order of `jobs` */
__global__ void __launch_bounds__(32 * SPLIT_WARPS)
split_decode_kernel(const SplitJob *jobs, SplitRes *res, uint32_t njobs,
    uint32_t *next)
{
	__shared__ InfTables tabs[SPLIT_WARPS];
	const uint32_t lane = threadIdx.x & 31;
	InfTables *T = &tabs[threadIdx.x >> 5];
	for (;;) {
		uint32_t j = 0;
		if (lane == 0)
			j = atomicAdd(next, 1u);
		j = __shfl_sync(0xffffffffu, j, 0);
		if (j >= njobs)
			return;
		SplitRes r;
		split_decode(jobs[j], T, InfLanes(), r);
		if (lane == 0)
			res[j] = r;
		__syncwarp();
	}
}

/* one CTA per file: the last 32 KiB of each of its chunks, in chain order
 * (pieces[first[f], first[f + 1])) */
__global__ void split_tail_kernel(const SplitPiece *pieces,
    const uint32_t *first, uint32_t *bad)
{
	const uint32_t f = blockIdx.x;
	bool ok = true;
	for (uint32_t k = first[f]; k < first[f + 1]; k++) {
		const SplitPiece p = pieces[k];
		ok &= split_resolve(p, split_tail(p), p.len, threadIdx.x,
		    blockDim.x);
		__syncthreads();
	}
	if (!ok)
		bad[f] = 1;
}

/* every chunk's symbols before its tail, one CTA per chunk */
__global__ void split_body_kernel(const SplitPiece *pieces, uint32_t *bad)
{
	const SplitPiece p = pieces[blockIdx.x];
	if (!split_resolve(p, 0, split_tail(p), threadIdx.x, blockDim.x))
		bad[p.file] = 1;
}

__global__ void split_crc_kernel(const CrcPiece *pieces, uint32_t *crcs,
    uint32_t n)
{
	__shared__ uint32_t crct[256];
	crc32_table(crct, threadIdx.x, blockDim.x);
	__syncthreads();
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n)
		crcs[i] = crc32_run(crct, pieces[i].p, pieces[i].len);
}

/* one warp per member */
__global__ void split_member_kernel(const CrcMember *members, uint32_t n,
    const CrcPiece *pieces, const uint32_t *crcs, uint32_t *bad)
{
	const uint32_t m = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
	if (m >= n)
		return;
	if (!split_member_ok(members[m], pieces, crcs, InfLanes()) &&
	    (threadIdx.x & 31) == 0)
		bad[members[m].file] = 1;
}
#endif

} /* namespace dng */

#endif /* DNG_INFLATE_SPLIT_CUH */
