/*
 * inflate.cuh: gzip (RFC 1952) over DEFLATE (RFC 1951), one warp per file on
 * the device (inflate_kernel, below), one thread per file on the host
 * (tests/hostcheck/inflate_check.cpp).
 *
 * Acceptance is Python's gzip.decompress: members are decoded in sequence,
 * zero bytes between and after members are skipped, the header flags are
 * skipped (the header CRC is not checked), and anything else fails: a bad
 * magic or method, a bad block type, a stored block whose NLEN is not ~LEN, a
 * Huffman code that is over-subscribed or incomplete where zlib's
 * inflate_table refuses it, an invalid code, a distance before the start of
 * the member's output, a truncated stream, a CRC-32 or ISIZE mismatch.
 *
 * The warp runs in lockstep: every lane keeps the same bit reader and decodes
 * every symbol (its loads and table lookups are broadcasts), lane 0 stores
 * the literals, and a match is copied by all 32 lanes at once.  Decode tables
 * are built per block in the warp's shared memory; a member's CRC-32 is taken
 * over 32 pieces and combined (multiplication by x^(8n) modulo the CRC
 * polynomial, as zlib's crc32_combine).
 */
#ifndef DNG_INFLATE_CUH
#define DNG_INFLATE_CUH

#include <stdint.h>

#include "jsnum.cuh"

namespace dng {

/* what one file ended with */
enum {
	INF_DONE = 0,		/* out_len bytes */
	INF_ROOM = 1,		/* the output did not fit its capacity */
	INF_ERROR = 2,		/* `kind` at input bit `bit` */
};

enum {
	IE_NONE = 0,
	IE_HEADER,		/* not a gzip member, or not deflate */
	IE_TRUNCATED,
	IE_BLOCK_TYPE,
	IE_STORED_LEN,
	IE_TABLE,		/* a code set zlib refuses */
	IE_CODE,		/* an invalid literal/length or distance code */
	IE_DISTANCE,		/* reaches before the member's output */
	IE_CRC,
	IE_ISIZE,
	IE_NKINDS
};

inline const char *inflate_error_name(uint32_t kind)
{
	static const char *const names[IE_NKINDS] = {
		"none", "bad gzip header", "truncated stream",
		"invalid block type", "invalid stored block lengths",
		"invalid Huffman code set", "invalid code",
		"distance too far back", "CRC-32 mismatch", "ISIZE mismatch",
	};
	return kind < IE_NKINDS ? names[kind] : "unknown";
}

struct InfJob {
	const uint8_t *in;
	uint64_t in_len;
	uint8_t *out;
	uint64_t cap;
};

struct InfResult {
	uint64_t out_len;
	uint64_t bit;		/* input bit offset of an error */
	uint32_t status;
	uint32_t kind;
	uint32_t members;
	uint32_t pad;
};

enum { INF_LBITS = 10, INF_DBITS = 8 };

/*
 * The output room to try first for a file of `in_len` compressed bytes whose
 * last four are `tail` (the last member's ISIZE: exact for one member under
 * 4 GiB).  Bounded by what DEFLATE can expand to (258 bytes from 2 bits, so
 * under 1032 times its input), which a damaged trailer cannot raise.
 */
inline uint64_t inflate_hint(const uint8_t *tail, uint64_t in_len)
{
	if (in_len < 4)
		return 0;
	const uint64_t isize = (uint64_t)tail[0] | (uint64_t)tail[1] << 8 |
	    (uint64_t)tail[2] << 16 | (uint64_t)tail[3] << 24;
	const uint64_t most = in_len * 1032 + 64;
	return isize < most ? isize : most;
}

/* decode tables of one block, in the warp's shared memory; an entry of a fast
 * table is (symbol << 4) | length, 0 for "not a code of <= its bits" */
struct InfTables {
	enum { LBITS = INF_LBITS, DBITS = INF_DBITS };
	uint16_t lcount[16], loffs[16], lfirst[16];
	uint16_t dcount[16], doffs[16], dfirst[16];
	uint16_t lsym[288], dsym[32];
	uint16_t lfast[1 << INF_LBITS];
	uint16_t dfast[1 << INF_DBITS];
	uint8_t lens[288 + 32];
	uint32_t fixed;		/* the fixed code is built */
};

/* the lanes of a warp on the device, one lane on the host */
struct InfLanes {
#ifdef __CUDA_ARCH__
	__device__ uint32_t lane() const { return threadIdx.x & 31; }
	__device__ uint32_t n() const { return 32; }
	__device__ void sync() const { __syncwarp(); }
	__device__ uint32_t bcast(uint32_t v, uint32_t src) const
	{
		return __shfl_sync(0xffffffffu, v, src);
	}
	__device__ uint32_t ballot(bool v) const
	{
		return __ballot_sync(0xffffffffu, v);
	}
#else
	uint32_t lane() const { return 0; }
	uint32_t n() const { return 1; }
	void sync() const {}
	uint32_t bcast(uint32_t v, uint32_t) const { return v; }
	uint32_t ballot(bool v) const { return v; }
#endif
};

/* one thread on its own, on the device as on the host */
struct InfOneLane {
	DNG_HDI uint32_t lane() const { return 0; }
	DNG_HDI uint32_t n() const { return 1; }
	DNG_HDI void sync() const {}
	DNG_HDI uint32_t bcast(uint32_t v, uint32_t) const { return v; }
	DNG_HDI uint32_t ballot(bool v) const { return v; }
};

/* a split decode (inflate_split.cuh): a member's end, CRC-32 and ISIZE,
 * checked once the pieces are joined */
struct InfMember {
	uint64_t end;		/* output offset of the member's end */
	uint32_t crc, isize;
};

static const uint64_t INF_NOSTART = ~0ull;	/* a chunk without a candidate */
static const uint32_t INF_NOLAND = ~0u;

/* ---- CRC-32 (reflected, polynomial 0xedb88320) ------------------------- */

DNG_HDI void crc32_table(uint32_t *t, uint32_t lane, uint32_t nl)
{
	for (uint32_t i = lane; i < 256; i += nl) {
		uint32_t c = i;
		for (int k = 0; k < 8; k++)
			c = c & 1 ? (c >> 1) ^ 0xedb88320u : c >> 1;
		t[i] = c;
	}
}

DNG_HDI uint32_t crc32_run(const uint32_t *t, const uint8_t *p, uint64_t n)
{
	uint32_t c = 0xffffffffu;
	for (uint64_t i = 0; i < n; i++)
		c = t[(c ^ p[i]) & 0xff] ^ (c >> 8);
	return c ^ 0xffffffffu;
}

/* a * b modulo the polynomial, bit-reflected (x^0 is bit 31) */
DNG_HDI uint32_t crc32_mulmod(uint32_t a, uint32_t b)
{
	uint32_t p = 0;
	for (uint32_t m = 1u << 31; m; m >>= 1) {
		if (a & m)
			p ^= b;
		b = b & 1 ? (b >> 1) ^ 0xedb88320u : b >> 1;
	}
	return p;
}

/* x^(8 nb) modulo the polynomial: what appending nb bytes multiplies by */
DNG_HDI uint32_t crc32_shift(uint64_t nb)
{
	uint32_t x = 1u << 30;		/* x^1: x^(2^k) as k steps */
	uint32_t p = 1u << 31;		/* x^0 */
	uint64_t n = nb * 8;
	while (n) {
		if (n & 1)
			p = crc32_mulmod(x, p);
		x = crc32_mulmod(x, x);
		n >>= 1;
	}
	return p;
}

/* crc32(A || B) from crc32(A), crc32(B) and |B| */
DNG_HDI uint32_t crc32_combine(uint32_t ca, uint32_t cb, uint64_t nb)
{
	return crc32_mulmod(crc32_shift(nb), ca) ^ cb;
}

/* ---- the decoder -----------------------------------------------------------
 *
 * Sym is the output symbol: bytes (inflate_one), or 16-bit symbols for a
 * decode that starts at a block inside a member (inflate_split.cuh), where a
 * distance reaching before the start gives a marker, 256 + i for byte i of
 * the 32 KiB before it.  Lanes: a warp, or one thread.  Tab: the decode
 * tables; Tab::LBITS and Tab::DBITS size their fast tables (0: none).
 */
template <class Sym, class Lanes, class Tab>
struct InflaterT {
	const uint8_t *in;
	uint64_t n;		/* compressed bytes */
	uint64_t next;		/* next byte to load into bb */
	uint64_t bb;		/* bit buffer, low bits first */
	uint32_t bc;		/* bits in bb */
	Sym *out;
	uint64_t cap, pos;
	uint64_t mstart;	/* output offset of the current member */
	uint32_t kind;
	Tab *T;
	const uint32_t *crct;
	Lanes L;
	/* a split decode: the member began before the output's start (markers);
	 * the later chunks' candidate bits, where a block start ends the decode
	 * (`land`: which one); the member ends, recorded instead of checked */
	bool window;
	const uint64_t *cand;
	uint32_t ncand, ci, land;
	InfMember *mem;
	uint32_t mcap;

	/* every field but the input, output and tables: a decode from bit 0 */
	DNG_HDI void reset()
	{
		next = 0;
		bb = 0;
		bc = 0;
		pos = 0;
		mstart = 0;
		kind = 0;
		crct = nullptr;
		window = false;
		cand = nullptr;
		ncand = ci = 0;
		land = INF_NOLAND;
		mem = nullptr;
		mcap = 0;
	}

	DNG_HDI uint64_t bitpos() const { return next * 8 - bc; }

	/* start reading at input bit `bit` (< 8 n) */
	DNG_HDI void seek(uint64_t bit)
	{
		next = bit >> 3;
		bb = 0;
		bc = 0;
		refill();
		bb >>= bit & 7;
		bc -= bit & 7;
	}

	/* a block starts here: is it a later chunk's candidate? */
	DNG_HDI bool landed()
	{
		if (!cand)
			return false;
		const uint64_t b = bitpos();
		while (ci < ncand && (cand[ci] < b || cand[ci] == INF_NOSTART))
			ci++;
		if (ci < ncand && cand[ci] == b) {
			land = ci;
			return true;
		}
		return false;
	}

	DNG_HDI void refill()
	{
		while (bc <= 56 && next < n) {
			bb |= (uint64_t)in[next++] << bc;
			bc += 8;
		}
	}

	/* k <= 32 bits; false: the input ended */
	DNG_HDI bool bits(uint32_t k, uint32_t &v)
	{
		if (bc < k)
			refill();
		if (bc < k)
			return fail(IE_TRUNCATED);
		v = (uint32_t)(bb & ((1ull << k) - 1));
		bb >>= k;
		bc -= k;
		return true;
	}

	DNG_HDI bool fail(uint32_t k)
	{
		if (!kind)
			kind = k;
		return false;
	}

	/* drop to a byte boundary and hand the whole bytes back to the input */
	DNG_HDI void align()
	{
		bb >>= bc & 7;
		bc -= bc & 7;
		next -= bc / 8;
		bb = 0;
		bc = 0;
	}

	DNG_HDI bool byte(uint32_t &v)
	{
		if (next >= n)
			return fail(IE_TRUNCATED);
		v = in[next++];
		return true;
	}

	/*
	 * Build the canonical code of lens[0, nsym) into count/offs/first/sym and
	 * its fast table.  `codes`: the code-lengths code (an incomplete set is
	 * refused even with one code); else an incomplete set is allowed only as
	 * one code of length 1, or none (inflate_table's rules).
	 */
	DNG_HDI bool build(const uint8_t *lens, uint32_t nsym, uint16_t *count,
	    uint16_t *offs, uint16_t *first, uint16_t *sym, uint16_t *fast,
	    uint32_t fbits, bool codes)
	{
		int bad = 0;
		if (L.lane() == 0) {
			for (int i = 0; i < 16; i++)
				count[i] = 0;
			for (uint32_t s = 0; s < nsym; s++)
				count[lens[s]]++;
			int max = 15;
			while (max >= 1 && !count[max])
				max--;
			int left = 1;
			for (int l = 1; l <= 15; l++) {
				left <<= 1;
				left -= count[l];
				if (left < 0)
					break;
			}
			if (left < 0)
				bad = 1;
			else if (max > 0 && left > 0 && (codes || max != 1))
				bad = 1;
			offs[1] = 0;
			first[1] = 0;
			for (int l = 1; l < 15; l++) {
				offs[l + 1] = offs[l] + count[l];
				first[l + 1] = (uint16_t)((first[l] + count[l]) << 1);
			}
			uint16_t o[16];
			for (int l = 1; l < 16; l++)
				o[l] = offs[l];
			for (uint32_t s = 0; s < nsym; s++)
				if (lens[s])
					sym[o[lens[s]]++] = (uint16_t)s;
		}
		L.sync();
		bad = (int)L.bcast((uint32_t)bad, 0);
		if (bad)
			return fail(IE_TABLE);
		const uint32_t nf = 1u << fbits;
		for (uint32_t j = L.lane(); j < nf; j += L.n())
			fast[j] = 0;
		L.sync();
		const uint32_t ncoded = offs[15] + count[15];
		for (uint32_t i = L.lane(); i < ncoded; i += L.n()) {
			const uint32_t s = sym[i], l = lens[s];
			if (l > fbits)
				continue;
			const uint32_t code = first[l] + (i - offs[l]);
			uint32_t rev = 0;
			for (uint32_t b = 0; b < l; b++)
				rev |= ((code >> b) & 1) << (l - 1 - b);
			const uint16_t e = (uint16_t)((s << 4) | l);
			for (uint32_t j = rev; j < nf; j += 1u << l)
				fast[j] = e;
		}
		L.sync();
		return true;
	}

	/* one symbol of a code; false: invalid or truncated */
	DNG_HDI bool decode(const uint16_t *count, const uint16_t *sym,
	    const uint16_t *fast, uint32_t fbits, uint32_t &s)
	{
		if (bc < 15)
			refill();
		const uint32_t e = fast[bb & ((1u << fbits) - 1)];
		if (e) {
			const uint32_t l = e & 15;
			if (l > bc)
				return fail(IE_TRUNCATED);
			bb >>= l;
			bc -= l;
			s = e >> 4;
			return true;
		}
		/* a longer code, or none: canonical decode bit by bit */
		int code = 0, first = 0, index = 0;
		for (uint32_t l = 1; l <= 15; l++) {
			if (l > bc)
				return fail(IE_TRUNCATED);
			code |= (int)((bb >> (l - 1)) & 1);
			const int c = count[l];
			if (code - c < first) {
				s = sym[index + (code - first)];
				bb >>= l;
				bc -= l;
				return true;
			}
			index += c;
			first = (first + c) << 1;
			code <<= 1;
		}
		return fail(IE_CODE);
	}

	DNG_HDI bool build_fixed()
	{
		if (T->fixed)
			return true;
		for (uint32_t i = L.lane(); i < 288 + 32; i += L.n())
			T->lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 :
			    i < 288 ? 8 : 5;
		L.sync();
		if (!build(T->lens, 288, T->lcount, T->loffs, T->lfirst, T->lsym,
		    T->lfast, Tab::LBITS, false) ||
		    !build(T->lens + 288, 32, T->dcount, T->doffs, T->dfirst,
		    T->dsym, T->dfast, Tab::DBITS, false))
			return false;
		T->fixed = 1;	/* (every lane stores the same value) */
		return true;
	}

	DNG_HDI bool build_dynamic()
	{
		uint32_t nlen, ndist, ncode;
		if (!bits(5, nlen) || !bits(5, ndist) || !bits(4, ncode))
			return false;
		nlen += 257;
		ndist += 1;
		ncode += 4;
		if (nlen > 286 || ndist > 30)
			return fail(IE_TABLE);
		T->fixed = 0;
		L.sync();
		static const uint8_t order[19] = { 16, 17, 18, 0, 8, 7, 9, 6,
		    10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15 };
		uint8_t cl[19];
		for (int i = 0; i < 19; i++)
			cl[i] = 0;
		for (uint32_t i = 0; i < ncode; i++) {
			uint32_t v;
			if (!bits(3, v))
				return false;
			cl[order[i]] = (uint8_t)v;
		}
		/* the code-lengths code lives in the distance tables for now */
		if (L.lane() == 0)
			for (int i = 0; i < 19; i++)
				T->lens[288 + i] = cl[i];
		L.sync();
		if (!build(T->lens + 288, 19, T->dcount, T->doffs, T->dfirst,
		    T->dsym, T->dfast, Tab::DBITS, true))
			return false;
		const uint32_t total = nlen + ndist;
		uint32_t have = 0, prev = 0;
		uint8_t *lens = T->lens;
		L.sync();
		while (have < total) {
			uint32_t s, rep, v = 0;
			if (!decode(T->dcount, T->dsym, T->dfast, Tab::DBITS, s))
				return false;
			if (s < 16) {
				if (L.lane() == 0)
					lens[have] = (uint8_t)s;
				prev = s;
				have++;
				continue;
			}
			if (s == 16) {
				if (!have)
					return fail(IE_TABLE);
				if (!bits(2, rep))
					return false;
				rep += 3;
				v = prev;
			} else if (s == 17) {
				if (!bits(3, rep))
					return false;
				rep += 3;
			} else {
				if (!bits(7, rep))
					return false;
				rep += 11;
			}
			if (have + rep > total)
				return fail(IE_TABLE);
			for (uint32_t i = L.lane(); i < rep; i += L.n())
				lens[have + i] = (uint8_t)v;
			prev = v;
			have += rep;
		}
		L.sync();
		if (!lens[256])
			return fail(IE_TABLE);
		/* the distance lengths move up to their own slot: copy through
		 * registers so no lane reads a byte another lane overwrote */
		uint8_t dl[30];
		for (uint32_t i = 0; i < 30; i++)
			dl[i] = i < ndist ? lens[nlen + i] : 0;
		L.sync();
		for (uint32_t i = nlen + L.lane(); i < 288; i += L.n())
			lens[i] = 0;
		for (uint32_t i = L.lane(); i < 32; i += L.n())
			lens[288 + i] = i < 30 ? dl[i] : 0;
		L.sync();
		return build(lens, nlen, T->lcount, T->loffs, T->lfirst, T->lsym,
		    T->lfast, Tab::LBITS, false) &&
		    build(lens + 288, ndist, T->dcount, T->doffs, T->dfirst,
		    T->dsym, T->dfast, Tab::DBITS, false);
	}

	/* 0: block ok, 1: out of room, else false via fail() */
	DNG_HDI int codes()
	{
		static const uint16_t lbase[29] = { 3, 4, 5, 6, 7, 8, 9, 10, 11,
		    13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
		    131, 163, 195, 227, 258 };
		static const uint8_t lext[29] = { 0, 0, 0, 0, 0, 0, 0, 0, 1, 1,
		    1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0 };
		static const uint16_t dbase[30] = { 1, 2, 3, 4, 5, 7, 9, 13, 17,
		    25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
		    2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577 };
		static const uint8_t dext[30] = { 0, 0, 0, 0, 1, 1, 2, 2, 3, 3,
		    4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12,
		    13, 13 };
		for (;;) {
			uint32_t s;
			if (!decode(T->lcount, T->lsym, T->lfast, Tab::LBITS, s))
				return -1;
			if (s < 256) {
				if (pos >= cap)
					return 1;
				if (L.lane() == 0)
					out[pos] = (Sym)s;
				pos++;
				continue;
			}
			if (s == 256)
				return 0;
			s -= 257;
			if (s >= 29)
				return fail(IE_CODE) ? 0 : -1;
			uint32_t e, len, ds, dist;
			if (!bits(lext[s], e))
				return -1;
			len = lbase[s] + e;
			if (!decode(T->dcount, T->dsym, T->dfast, Tab::DBITS, ds))
				return -1;
			if (ds >= 30)
				return fail(IE_CODE) ? 0 : -1;
			if (!bits(dext[ds], e))
				return -1;
			dist = dbase[ds] + e;
			if (dist > pos - mstart && !window)
				return fail(IE_DISTANCE) ? 0 : -1;
			if (pos + len > cap)
				return 1;
			L.sync();	/* lane 0's literals, seen by every lane */
			Sym *dst = out + pos;
			if (dist > pos) {
				/* (only with a window) markers for what lies before */
				const int64_t from = (int64_t)pos - dist;
				for (uint32_t i = L.lane(); i < len; i += L.n()) {
					const int64_t k = from + i % dist;
					dst[i] = k >= 0 ? out[k] : (Sym)(256 + 32768 + k);
				}
				pos += len;
				continue;
			}
			const Sym *src = out + pos - dist;
			if (dist >= len) {
				for (uint32_t i = L.lane(); i < len; i += L.n())
					dst[i] = src[i];
			} else {
				for (uint32_t i = L.lane(); i < len; i += L.n())
					dst[i] = src[i % dist];
			}
			pos += len;
		}
	}

	DNG_HDI int stored()
	{
		align();
		uint32_t b[4];
		for (int i = 0; i < 4; i++)
			if (!byte(b[i]))
				return -1;
		const uint32_t len = b[0] | b[1] << 8, nlen = b[2] | b[3] << 8;
		if (len != (~nlen & 0xffff))
			return fail(IE_STORED_LEN) ? 0 : -1;
		if (n - next < len) {
			next = n;
			return fail(IE_TRUNCATED) ? 0 : -1;
		}
		if (pos + len > cap)
			return 1;
		L.sync();
		for (uint32_t i = L.lane(); i < len; i += L.n())
			out[pos + i] = in[next + i];
		next += len;
		pos += len;
		return 0;
	}

	/* one member's header; false: error */
	DNG_HDI bool header()
	{
		uint32_t h[10];
		static const uint8_t magic[3] = { 0x1f, 0x8b, 8 };
		for (int i = 0; i < 10; i++) {
			if (i < 3 && next < n && in[next] != magic[i])
				return fail(IE_HEADER);
			if (!byte(h[i]))
				return false;
		}
		const uint32_t flg = h[3];
		uint32_t a, b;
		if (flg & 4) {	/* FEXTRA */
			if (!byte(a) || !byte(b))
				return false;
			const uint32_t xlen = a | b << 8;
			if (n - next < xlen) {
				next = n;
				return fail(IE_TRUNCATED);
			}
			next += xlen;
		}
		for (uint32_t f = 8; f <= 16; f <<= 1)	/* FNAME, FCOMMENT */
			if (flg & f)
				while (next < n && in[next++] != 0)
					;
		if (flg & 2)	/* FHCRC */
			if (!byte(a) || !byte(b))
				return false;
		return true;
	}

	/* one member's trailer; its output is [mstart, pos), or, in a split
	 * decode, ends at pos and is recorded as member m */
	DNG_HDI bool trailer(uint32_t m)
	{
		align();
		uint32_t t[8];
		for (int i = 0; i < 8; i++)
			if (!byte(t[i]))
				return false;
		const uint32_t want = t[0] | t[1] << 8 | t[2] << 16 | t[3] << 24;
		const uint32_t isize = t[4] | t[5] << 8 | t[6] << 16 | t[7] << 24;
		if (mem) {
			if (L.lane() == 0)
				mem[m] = { pos, want, isize };
			return true;
		}
		/* each lane a piece of at least 4 KiB, combined in order */
		L.sync();
		const uint64_t total = pos - mstart;
		uint64_t piece = (total + L.n() - 1) / L.n();
		if (piece < 4096)
			piece = 4096;
		const uint64_t lo = mstart + piece * L.lane();
		const uint64_t hi = lo + piece < pos ? lo + piece : pos;
		const uint32_t mine = lo < hi ?
		    crc32_run(crct, (const uint8_t *)(out + lo), hi - lo) : 0;
		uint32_t crc = 0;
		for (uint32_t i = 0; i < L.n(); i++) {
			const uint32_t c = L.bcast(mine, i);
			const uint64_t plo = mstart + piece * i;
			const uint64_t phi = plo + piece < pos ? plo + piece : pos;
			if (plo < phi)
				crc = crc32_combine(crc, c, phi - plo);
		}
		if (crc != want)
			return fail(IE_CRC);
		if (isize != (uint32_t)total)
			return fail(IE_ISIZE);
		return true;
	}

	/* the whole file; or, with a window, from a block inside a member to
	 * the end, or to a block start that landed() */
	DNG_HDI void run(InfResult &r)
	{
		r.status = INF_DONE;
		r.kind = IE_NONE;
		r.members = 0;
		r.bit = 0;
		T->fixed = 0;
		L.sync();
		for (bool inside = window;; inside = false) {
			if (!inside) {
				while (r.members && next < n && in[next] == 0)
					next++;
				if (next >= n)
					break;
				if (!header())
					goto error;
				mstart = pos;
				window = false;
			}
			for (;;) {
				if (landed()) {
					r.out_len = pos;
					return;
				}
				uint32_t last, type;
				if (!bits(1, last) || !bits(2, type))
					goto error;
				int rc;
				if (type == 0)
					rc = stored();
				else if (type == 1)
					rc = build_fixed() ? codes() : -1;
				else if (type == 2)
					rc = build_dynamic() ? codes() : -1;
				else
					rc = fail(IE_BLOCK_TYPE) ? 0 : -1;
				if (rc < 0)
					goto error;
				if (rc > 0)
					goto room;
				if (last)
					break;
			}
			if (mem && r.members >= mcap)
				goto room;	/* (no slot for the member) */
			if (!trailer(r.members))
				goto error;
			r.members++;
		}
		r.out_len = pos;
		return;
	room:
		r.status = INF_ROOM;
		r.out_len = pos;
		return;
	error:
		r.status = INF_ERROR;
		r.kind = kind ? kind : (uint32_t)IE_TRUNCATED;
		r.bit = bitpos();
		r.out_len = pos;
	}
};

typedef InflaterT<uint8_t, InfLanes, InfTables> Inflater;

/* decode in[0, in_len) into out[0, cap): the host's entry (one lane) and the
 * body of each warp of inflate_kernel */
DNG_HDI void inflate_one(const InfJob &j, InfTables *T, const uint32_t *crct,
    InfResult &r)
{
	Inflater f;
	f.reset();
	f.in = j.in;
	f.n = j.in_len;
	f.out = j.out;
	f.cap = j.cap;
	f.T = T;
	f.crct = crct;
	f.run(r);
}

#ifdef __CUDACC__
enum { INF_WARPS = 4 };	/* warps per CTA of inflate_kernel */

/* one warp per file: files taken from *next, in the order of `jobs` (the
 * caller puts the largest first so that none is left running alone) */
__global__ void __launch_bounds__(32 * INF_WARPS)
inflate_kernel(const InfJob *jobs, InfResult *res, uint32_t njobs,
    uint32_t *next)
{
	__shared__ InfTables tabs[INF_WARPS];
	__shared__ uint32_t crct[256];
	crc32_table(crct, threadIdx.x, blockDim.x);
	__syncthreads();
	const uint32_t lane = threadIdx.x & 31;
	InfTables *T = &tabs[threadIdx.x >> 5];
	for (;;) {
		uint32_t j = 0;
		if (lane == 0)
			j = atomicAdd(next, 1u);
		j = __shfl_sync(0xffffffffu, j, 0);
		if (j >= njobs)
			return;
		InfResult r;
		inflate_one(jobs[j], T, crct, r);
		if (lane == 0)
			res[j] = r;
		__syncwarp();
	}
}
#endif

} /* namespace dng */

#endif /* DNG_INFLATE_CUH */
