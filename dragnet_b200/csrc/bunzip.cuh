/*
 * bunzip.cuh: bzip2 decoded with all its blocks in parallel: every stage runs
 * on the device (the kernels at the bottom) and as one lane on the host
 * (tests/hostcheck/bunzip_check.cpp).
 *
 * A bzip2 file is one or more streams ("BZh" and a level digit 1-9, blocks,
 * an end-of-stream mark and the stream CRC, padded to a byte).  Each block
 * starts with the 48-bit magic 0x314159265359 at any bit offset, holds at
 * most level x 100,000 bytes of a Burrows-Wheeler transformed block, and
 * refers to no other block.  The stages of one batch:
 *
 *   find    every bit offset of either magic in every file (bz_find_kernel);
 *   decode  each block candidate, one warp each (bz_decode_kernel): header,
 *           selectors, code lengths, Huffman symbols, RUNA/RUNB and
 *           move-to-front, into the candidate's BWT slot;
 *   chain   on the host: from bit 32 of the first stream, each block ends
 *           where the next candidate begins; candidates the chain does not
 *           land on are false starts and are dropped;
 *   invert  one CTA per chained block (bz_ibwt_kernel): the transformation
 *           vector by a stable counting sort, then the walk from origPtr by
 *           many walkers (segments between sampled positions, linked from
 *           origPtr), the randomisation of old encoders, and the length of
 *           each chunk after the final run-length stage, composed over the
 *           block's run states;
 *   emit    one CTA per block (bz_emit_kernel): the final run-length stage
 *           into the block's place in the output, with its CRC taken over
 *           pieces and joined.
 *
 * Acceptance follows libbz2 1.0.8 (what Python's bz2 links): its canonical
 * limit/base/perm Huffman tables, selectors past 18,002 read and ignored,
 * a run of four equal bytes that ends a block without its count is damage.
 */
#ifndef DNG_BUNZIP_CUH
#define DNG_BUNZIP_CUH

#include <stdint.h>
#include <string.h>

#include "inflate.cuh"

namespace dng {

enum {
	BZ_MAX_BLOCK = 900000,	/* bytes of a level-9 block */
	BZ_MAX_SEL = 18002,	/* selectors libbz2 keeps */
	BZ_SEL_ROOM = 18016,
	BZ_SLOT = BZ_MAX_BLOCK + BZ_SEL_ROOM,	/* a candidate's BWT slot */
	BZ_MAX_GROUPS = 6,
	BZ_MAX_ALPHA = 258,
	BZ_CODE_LEN = 23,
	BZ_CHUNKS = 512,	/* run-length chunks of a block = CTA threads */
	BZ_THREADS = 512,	/* threads of bz_ibwt_kernel, bz_emit_kernel */
};

/* walkers of one block's inverse BWT: sampled start positions (DESIGN.md
 * §7.B: chosen from tools/bzip2_leg.py) */
#ifndef BZ_WALKERS
#define BZ_WALKERS 2048
#endif
static_assert(BZ_WALKERS <= 4096 && BZ_WALKERS >= BZ_THREADS,
    "walker count");

static const uint64_t BZ_BLOCK_MAGIC = 0x314159265359ull;
static const uint64_t BZ_EOS_MAGIC = 0x177245385090ull;

/* the damage a file fails with */
enum {
	BE_NONE = 0,
	BE_STREAM_HEADER,
	BE_BLOCK_HEADER,
	BE_TABLES,		/* selectors or code lengths */
	BE_CODE,
	BE_OVERFLOW,		/* block too long, origPtr outside it */
	BE_BLOCK_CRC,
	BE_STREAM_CRC,
	BE_TRUNCATED,
	BE_TRAILING,		/* data after the last stream, not zeros */
	BE_NKINDS
};

inline const char *bunzip_error_name(uint32_t kind)
{
	static const char *const names[BE_NKINDS] = {
		"none", "bad stream header", "bad block header",
		"bad selector or code lengths", "invalid code",
		"block overflow", "block CRC mismatch", "stream CRC mismatch",
		"truncated", "trailing data after the last bzip2 stream",
	};
	return kind < BE_NKINDS ? names[kind] : "unknown";
}

/* the randomisation table of the bzip2 format (BZ2_rNums in libbz2):
 * tests/test_bunzip_host.py compares it with the library's */
#define BZ_RNUMS \
	619, 720, 127, 481, 931, 816, 813, 233, 566, 247, 985, 724, 205, 454, \
	863, 491, 741, 242, 949, 214, 733, 859, 335, 708, 621, 574, 73, 654, \
	730, 472, 419, 436, 278, 496, 867, 210, 399, 680, 480, 51, 878, 465, \
	811, 169, 869, 675, 611, 697, 867, 561, 862, 687, 507, 283, 482, 129, \
	807, 591, 733, 623, 150, 238, 59, 379, 684, 877, 625, 169, 643, 105, \
	170, 607, 520, 932, 727, 476, 693, 425, 174, 647, 73, 122, 335, 530, \
	442, 853, 695, 249, 445, 515, 909, 545, 703, 919, 874, 474, 882, 500, \
	594, 612, 641, 801, 220, 162, 819, 984, 589, 513, 495, 799, 161, 604, \
	958, 533, 221, 400, 386, 867, 600, 782, 382, 596, 414, 171, 516, 375, \
	682, 485, 911, 276, 98, 553, 163, 354, 666, 933, 424, 341, 533, 870, \
	227, 730, 475, 186, 263, 647, 537, 686, 600, 224, 469, 68, 770, 919, \
	190, 373, 294, 822, 808, 206, 184, 943, 795, 384, 383, 461, 404, 758, \
	839, 887, 715, 67, 618, 276, 204, 918, 873, 777, 604, 560, 951, 160, \
	578, 722, 79, 804, 96, 409, 713, 940, 652, 934, 970, 447, 318, 353, \
	859, 672, 112, 785, 645, 863, 803, 350, 139, 93, 354, 99, 820, 908, \
	609, 772, 154, 274, 580, 184, 79, 626, 630, 742, 653, 282, 762, 623, \
	680, 81, 927, 626, 789, 125, 411, 521, 938, 300, 821, 78, 343, 175, \
	128, 250, 170, 774, 972, 275, 999, 639, 495, 78, 352, 126, 857, 956, \
	358, 619, 580, 124, 737, 594, 701, 612, 669, 112, 134, 694, 363, 992, \
	809, 743, 168, 974, 944, 375, 748, 52, 600, 747, 642, 182, 862, 81, \
	344, 805, 988, 739, 511, 655, 814, 334, 249, 515, 897, 955, 664, 981, \
	649, 113, 974, 459, 893, 228, 433, 837, 553, 268, 926, 240, 102, 654, \
	459, 51, 686, 754, 806, 760, 493, 403, 415, 394, 687, 700, 946, 670, \
	656, 610, 738, 392, 760, 799, 887, 653, 978, 321, 576, 617, 626, 502, \
	894, 679, 243, 440, 680, 879, 194, 572, 640, 724, 926, 56, 204, 700, \
	707, 151, 457, 449, 797, 195, 791, 558, 945, 679, 297, 59, 87, 824, \
	713, 663, 412, 693, 342, 606, 134, 108, 571, 364, 631, 212, 174, 643, \
	304, 329, 343, 97, 430, 751, 497, 314, 983, 374, 822, 928, 140, 206, \
	73, 263, 980, 736, 876, 478, 430, 305, 170, 514, 364, 692, 829, 82, \
	855, 953, 676, 246, 369, 970, 294, 750, 807, 827, 150, 790, 288, 923, \
	804, 378, 215, 828, 592, 281, 565, 555, 710, 82, 896, 831, 547, 261, \
	524, 462, 293, 465, 502, 56, 661, 821, 976, 991, 658, 869, 905, 758, \
	745, 193, 768, 550, 608, 933, 378, 286, 215, 979, 792, 961, 61, 688, \
	793, 644, 986, 403, 106, 366, 905, 644, 372, 567, 466, 434, 645, 210, \
	389, 550, 919, 135, 780, 773, 635, 389, 707, 100, 626, 958, 165, 504, \
	920, 176, 193, 713, 857, 265, 203, 50, 668, 108, 645, 990, 626, 197, \
	510, 357, 358, 850, 858, 364, 936, 638
#ifdef __CUDACC__
__constant__ uint16_t bz_rnums_dev[512] = { BZ_RNUMS };
#endif
static const uint16_t bz_rnums_host[512] = { BZ_RNUMS };

DNG_HDI uint32_t bz_rnum(uint32_t i)
{
#ifdef __CUDA_ARCH__
	return bz_rnums_dev[i];
#else
	return bz_rnums_host[i];
#endif
}

/* ---- find ----------------------------------------------------------------*/

enum { BZ_CAND_BLOCK = 1, BZ_CAND_EOS = 2 };

struct BzFile {			/* a file of the batch, for bz_find_kernel */
	const uint8_t *in;
	uint64_t len;
};

struct BzCand {
	uint64_t bit;		/* of the magic's first bit */
	uint32_t file, kind;
	uint32_t crc;		/* BZ_CAND_EOS: the 32 bits after the magic */
	uint32_t next;		/* ... and the 4 bytes after them, padded */
};

/* the 56 bits from byte i on (bytes past the end read as 0) */
DNG_HDI uint64_t bz_load56(const uint8_t *in, uint64_t len, uint64_t i)
{
	uint64_t v = 0;
	for (int k = 0; k < 7; k++)
		v = v << 8 | (i + k < len ? in[i + k] : 0);
	return v;
}

/* 32 bits from bit b on */
DNG_HDI uint32_t bz_load32(const uint8_t *in, uint64_t len, uint64_t b)
{
	const uint64_t v = bz_load56(in, len, b >> 3);
	return (uint32_t)(v >> (24 - (b & 7)));
}

/* the magics that begin in byte i: bit k for a block magic at bit 8 i + k,
 * bit 8 + k for an end-of-stream magic there */
DNG_HDI uint32_t bz_find_at(const uint8_t *in, uint64_t len, uint64_t i)
{
	const uint64_t v = bz_load56(in, len, i);
	uint32_t m = 0;
	for (uint32_t k = 0; k < 8; k++) {
		const uint64_t w = (v >> (8 - k)) & 0xffffffffffffull;
		if ((i * 8 + k) + 48 > len * 8)
			break;
		if (w == BZ_BLOCK_MAGIC)
			m |= 1u << k;
		else if (w == BZ_EOS_MAGIC)
			m |= 1u << (8 + k);
	}
	return m;
}

/* what follows an end-of-stream mark at `bit`: its stream CRC, and the four
 * bytes after it once aligned to a byte (zeros past the end) */
DNG_HDI void bz_eos_tail(const uint8_t *in, uint64_t len, BzCand &c)
{
	c.crc = bz_load32(in, len, c.bit + 48);
	const uint64_t a = (c.bit + 80 + 7) >> 3;
	c.next = bz_load32(in, len, a * 8);
}

/* ---- decode: one block candidate -----------------------------------------*/

struct BzDecJob {
	const uint8_t *in;	/* the file */
	uint64_t len;
	uint64_t bit;		/* of the block magic */
	uint8_t *slot;		/* BZ_SLOT bytes: the block, then selectors */
	uint32_t *hist;		/* 256 counts */
};

struct BzDecResult {
	uint64_t end_bit;	/* where the next magic must begin */
	uint64_t err_bit;
	uint32_t nblock, orig, crc, rand;
	uint32_t kind, pad;
};

struct BzDecShared {		/* one warp's tables */
	int32_t limit[BZ_MAX_GROUPS][BZ_CODE_LEN];
	int32_t base[BZ_MAX_GROUPS][BZ_CODE_LEN];
	uint16_t perm[BZ_MAX_GROUPS][BZ_MAX_ALPHA];
	uint8_t lens[BZ_MAX_GROUPS][BZ_MAX_ALPHA];
	uint8_t minlen[BZ_MAX_GROUPS];
	uint8_t mtf[256];
	uint8_t unseq[256];
	uint32_t hist[256];
};

/* MSB-first bit reader; reads past the end give zeros and mark truncation */
struct BzBits {
	const uint8_t *in;
	uint64_t len, next, pos, nbits;
	uint64_t bb;
	uint32_t bc;

	DNG_HDI void start(const uint8_t *p, uint64_t n, uint64_t bit)
	{
		in = p;
		len = n;
		nbits = n * 8;
		next = bit >> 3;
		bb = 0;
		bc = 0;
		pos = bit & ~7ull;
		get(bit & 7);
	}
	DNG_HDI void fill()
	{
		while (bc <= 56) {
			const uint64_t b = next < len ? in[next] : 0;
			next++;
			bb |= b << (56 - bc);
			bc += 8;
		}
	}
	/* the next n <= 32 bits, not consumed */
	DNG_HDI uint32_t peek(uint32_t n)
	{
		fill();
		return n ? (uint32_t)(bb >> (64 - n)) : 0;
	}
	DNG_HDI void skip(uint32_t n)
	{
		bb <<= n;
		bc -= n;
		pos += n;
	}
	DNG_HDI uint32_t get(uint32_t n)
	{
		const uint32_t v = peek(n);
		skip(n);
		return v;
	}
	DNG_HDI bool truncated() const { return pos > nbits; }
};

/* libbz2's hbCreateDecodeTables, for group t */
DNG_HDI void bz_tables(BzDecShared *S, uint32_t t, uint32_t alpha)
{
	const uint8_t *len = S->lens[t];
	int32_t *limit = S->limit[t], *base = S->base[t];
	uint16_t *perm = S->perm[t];
	int32_t minl = 32, maxl = 0;
	for (uint32_t i = 0; i < alpha; i++) {
		if (len[i] > maxl)
			maxl = len[i];
		if (len[i] < minl)
			minl = len[i];
	}
	int32_t pp = 0;
	for (int32_t i = minl; i <= maxl; i++)
		for (uint32_t j = 0; j < alpha; j++)
			if (len[j] == i)
				perm[pp++] = (uint16_t)j;
	for (int32_t i = pp; i < BZ_MAX_ALPHA; i++)
		perm[i] = 0;
	for (int i = 0; i < BZ_CODE_LEN; i++)
		base[i] = limit[i] = 0;
	for (uint32_t i = 0; i < alpha; i++)
		base[len[i] + 1]++;
	for (int i = 1; i < BZ_CODE_LEN; i++)
		base[i] += base[i - 1];
	int32_t vec = 0;
	for (int32_t i = minl; i <= maxl; i++) {
		vec += base[i + 1] - base[i];
		limit[i] = vec - 1;
		vec <<= 1;
	}
	for (int32_t i = minl + 1; i <= maxl; i++)
		base[i] = ((limit[i - 1] + 1) << 1) - base[i];
	S->minlen[t] = (uint8_t)minl;
}

/*
 * Decode the block whose magic is at j.bit: its BWT block into j.slot, its
 * byte counts into j.hist.  Lanes: a warp (in lockstep: every lane reads the
 * same bits; lane 0 stores single bytes, all lanes store a run and shift the
 * move-to-front list together) or one thread.
 */
template <class Lanes>
DNG_HDI void bz_decode_one(const BzDecJob &j, BzDecShared *S, Lanes L,
    BzDecResult &r)
{
	const uint32_t lane = L.lane(), nl = L.n();
	BzBits b;
	b.start(j.in, j.len, j.bit);
	r.end_bit = r.err_bit = 0;
	r.nblock = r.orig = r.crc = r.rand = 0;
	r.kind = BE_NONE;
	r.pad = 0;
	uint32_t kind = BE_NONE;
	uint32_t nblock = 0, nsel = 0, ngroups = 0, ninuse = 0;
	uint8_t *sel = j.slot + BZ_MAX_BLOCK;
	for (uint32_t i = lane; i < 256; i += nl) {
		S->hist[i] = 0;
		S->mtf[i] = (uint8_t)i;
	}
	L.sync();
	{
		const uint64_t m = (uint64_t)b.get(24) << 24 | b.get(24);
		r.crc = b.get(32);
		r.rand = b.get(1);
		r.orig = b.get(24);
		if (m != BZ_BLOCK_MAGIC) {
			kind = BE_BLOCK_HEADER;
			goto out;
		}
	}
	{
		const uint32_t used = b.get(16);
		for (uint32_t i = 0; i < 16; i++)
			if (used >> (15 - i) & 1) {
				const uint32_t w = b.get(16);
				for (uint32_t k = 0; k < 16; k++)
					if (w >> (15 - k) & 1) {
						if (lane == 0)
							S->unseq[ninuse] =
							    (uint8_t)(i * 16 + k);
						ninuse++;
					}
			}
		if (ninuse == 0) {
			kind = BE_BLOCK_HEADER;
			goto out;
		}
	}
	ngroups = b.get(3);
	nsel = b.get(15);
	if (ngroups < 2 || ngroups > BZ_MAX_GROUPS || nsel < 1) {
		kind = BE_TABLES;
		goto out;
	}
	{
		/* selectors, move-to-front coded in unary */
		uint8_t pos[BZ_MAX_GROUPS] = { 0, 1, 2, 3, 4, 5 };
		for (uint32_t i = 0; i < nsel; i++) {
			uint32_t v = 0;
			while (b.get(1)) {
				if (++v >= ngroups) {
					kind = BE_TABLES;
					goto out;
				}
				if (b.truncated())
					goto out;
			}
			const uint8_t g = pos[v];
			for (; v > 0; v--)
				pos[v] = pos[v - 1];
			pos[0] = g;
			if (i < BZ_MAX_SEL && lane == 0)
				sel[i] = g;
		}
		if (nsel > BZ_MAX_SEL)
			nsel = BZ_MAX_SEL;
	}
	{
		const uint32_t alpha = ninuse + 2;
		for (uint32_t t = 0; t < ngroups; t++) {
			int32_t curr = (int32_t)b.get(5);
			for (uint32_t i = 0; i < alpha; i++) {
				for (;;) {
					if (curr < 1 || curr > 20) {
						kind = BE_TABLES;
						goto out;
					}
					if (!b.get(1))
						break;
					curr += b.get(1) ? -1 : 1;
				}
				if (lane == 0)
					S->lens[t][i] = (uint8_t)curr;
			}
			if (b.truncated())
				goto out;
		}
		L.sync();
		for (uint32_t t = lane; t < ngroups; t += nl)
			bz_tables(S, t, alpha);
		L.sync();
	}
	{
		/* symbols: RUNA/RUNB runs of the front byte, or a move-to-front
		 * index + 1, until EOB */
		const uint32_t eob = ninuse + 1;
		uint32_t gno = 0, gpos = 0, g = 0;
		uint32_t es = 0, nrun = 1;
		bool inrun = false;
		for (;;) {
			if (gpos == 0) {
				if (gno >= nsel) {
					kind = BE_CODE;
					goto out;
				}
				g = sel[gno++];
				gpos = 50;
			}
			gpos--;
			const uint32_t v = b.peek(20);
			int32_t zn = S->minlen[g];
			int32_t zvec = (int32_t)(v >> (20 - zn));
			while (zvec > S->limit[g][zn]) {
				if (++zn > 20) {
					kind = BE_CODE;
					goto out;
				}
				zvec = (int32_t)(v >> (20 - zn));
			}
			b.skip((uint32_t)zn);
			const int32_t k = zvec - S->base[g][zn];
			if (k < 0 || k >= BZ_MAX_ALPHA) {
				kind = BE_CODE;
				goto out;
			}
			if (b.truncated())
				goto out;
			const uint32_t sym = S->perm[g][k];
			if (sym <= 1) {
				if (nrun >= 2 * 1024 * 1024) {
					kind = BE_CODE;
					goto out;
				}
				es += (sym + 1) * nrun;
				nrun <<= 1;
				inrun = true;
				continue;
			}
			if (inrun) {
				/* the run ends: es copies of the front byte */
				const uint8_t uc = S->unseq[S->mtf[0]];
				if (es > BZ_MAX_BLOCK - nblock) {
					kind = BE_OVERFLOW;
					goto out;
				}
				for (uint32_t i = lane; i < es; i += nl)
					j.slot[nblock + i] = uc;
				if (lane == 0)
					S->hist[uc] += es;
				nblock += es;
				es = 0;
				nrun = 1;
				inrun = false;
			}
			if (sym == eob)
				break;
			if (nblock >= BZ_MAX_BLOCK) {
				kind = BE_OVERFLOW;
				goto out;
			}
			const uint32_t nn = sym - 1;
			const uint8_t m = S->mtf[nn];
			for (int32_t top = (int32_t)nn; top > 0; top -= (int32_t)nl) {
				const int32_t at = top - (int32_t)lane;
				uint8_t x = 0;
				if (at >= 1)
					x = S->mtf[at - 1];
				L.sync();
				if (at >= 1)
					S->mtf[at] = x;
				L.sync();
			}
			const uint8_t uc = S->unseq[m];
			if (lane == 0) {
				S->mtf[0] = m;
				j.slot[nblock] = uc;
				S->hist[uc]++;
			}
			L.sync();
			nblock++;
		}
	}
	if (r.orig >= nblock) {
		kind = BE_OVERFLOW;
		goto out;
	}
	r.nblock = nblock;
	r.end_bit = b.pos;
	L.sync();
	for (uint32_t i = lane; i < 256; i += nl)
		j.hist[i] = S->hist[i];
	return;
out:
	/* reading past the end is truncation, whatever it decoded to */
	r.kind = b.truncated() ? (uint32_t)BE_TRUNCATED : kind ? kind :
	    (uint32_t)BE_TRUNCATED;
	r.err_bit = b.pos < b.nbits ? b.pos : b.nbits;
	L.sync();
}

/* ---- chain (host) ------------------------------------------------------*/

/*
 * One file's chain through its sorted candidates, advanced as the
 * candidates' decodes arrive.  `step` is called with the index of the block
 * candidate the chain needs next; it answers whether that decode is known.
 */
struct BzChain {
	uint64_t len;		/* compressed bytes */
	uint64_t nz_end;	/* one past the last nonzero byte */
	uint32_t head;		/* the file's first four bytes, big-endian */
	uint64_t bit;		/* where the chain stands: a magic must begin */
	uint32_t level;		/* the current stream's, 0 between streams */
	uint32_t scrc;		/* the stream CRC folded so far */
	uint32_t streams, blocks;
	uint32_t kind;		/* BE_* once failed */
	uint64_t err_bit;
	bool done;
};

inline bool bz_level_ok(uint32_t head4)
{
	return (head4 >> 8) == 0x425a68u && (head4 & 0xff) >= '1' &&
	    (head4 & 0xff) <= '9';
}

inline void bz_chain_init(BzChain &c, uint64_t len, uint64_t nz_end,
    uint32_t head)
{
	memset(&c, 0, sizeof c);
	c.len = len;
	c.nz_end = nz_end;
	c.head = head;
	if (!bz_level_ok(head)) {
		c.kind = len < 4 ? BE_TRUNCATED : BE_STREAM_HEADER;
		c.done = true;
		return;
	}
	c.level = (head & 0xff) - '0';
	c.bit = 32;
	c.streams = 1;
}

inline void bz_chain_fail(BzChain &c, uint32_t kind, uint64_t bit)
{
	c.kind = kind;
	c.err_bit = bit;
	c.done = true;
}

/*
 * Advance the chain over candidates cand[0, n) of this file (sorted by bit).
 * dec(i) gives the decode of block candidate i, or nullptr if it is not known
 * yet (the chain then stops there).  take(i) is called for each block the
 * chain lands on, in order.
 */
template <class Dec, class Take>
inline void bz_chain_run(BzChain &c, const BzCand *cand, uint32_t n, Dec dec,
    Take take)
{
	while (!c.done) {
		/* the candidate at c.bit */
		uint32_t lo = 0, hi = n;
		while (lo < hi) {
			const uint32_t m = (lo + hi) / 2;
			if (cand[m].bit < c.bit)
				lo = m + 1;
			else
				hi = m;
		}
		if (lo == n || cand[lo].bit != c.bit) {
			bz_chain_fail(c, c.bit + 48 > c.len * 8 ? BE_TRUNCATED :
			    BE_BLOCK_HEADER, c.bit);
			return;
		}
		const BzCand &k = cand[lo];
		if (k.kind == BZ_CAND_BLOCK) {
			const BzDecResult *r = dec(lo);
			if (!r)
				return;
			if (r->kind) {
				bz_chain_fail(c, r->kind, r->err_bit);
				return;
			}
			if (r->nblock > c.level * 100000u) {
				bz_chain_fail(c, BE_OVERFLOW, c.bit);
				return;
			}
			c.scrc = (c.scrc << 1 | c.scrc >> 31) ^ r->crc;
			c.blocks++;
			take(lo);
			c.bit = r->end_bit;
			continue;
		}
		/* end of stream: its CRC, then another stream, zeros or the end */
		if (k.bit + 80 > c.len * 8) {
			bz_chain_fail(c, BE_TRUNCATED, c.len * 8);
			return;
		}
		if (k.crc != c.scrc) {
			bz_chain_fail(c, BE_STREAM_CRC, k.bit + 48);
			return;
		}
		const uint64_t a = (k.bit + 80 + 7) >> 3;
		if (a >= c.nz_end) {
			c.done = true;		/* the end, or zeros to it */
			return;
		}
		if (!bz_level_ok(k.next)) {
			bz_chain_fail(c, BE_TRAILING, a * 8);
			return;
		}
		c.level = (k.next & 0xff) - '0';
		c.scrc = 0;
		c.streams++;
		c.bit = a * 8 + 32;
	}
}

/* ---- invert: transformation vector, walk, run lengths ------------------- */

struct BzBwtJob {
	uint8_t *slot;		/* the block in; the walked bytes out */
	uint32_t *tt;		/* 4 bytes per block byte */
	const uint32_t *hist;
	uint32_t *chunks;	/* BZ_CHUNKS x (offset, incoming state) */
	uint32_t n, orig, rand, pad;
};

struct BzBwtResult {
	uint64_t out_len;
	uint32_t ok;		/* 0: a run of four without its count */
	uint32_t pad;
};

enum { BZ_TMASK = 0xfffff, BZ_MARK = 0x80000000u };

/* the sort's per-warp counts (then the run states), the walkers' segments */
struct BzBwtShared {
	union {
		uint32_t cnt[BZ_THREADS / 32][256];
		struct {
			uint32_t run_len[BZ_CHUNKS][5];
			uint8_t run_out[BZ_CHUNKS][5];
		};
	};
	uint32_t seg_len[BZ_WALKERS];
	uint32_t seg_off[BZ_WALKERS];
	uint16_t seg_next[BZ_WALKERS];
	uint32_t head, fallback;
};

/* threads of a CTA, or one thread on the host */
struct BzCta {
#ifdef __CUDA_ARCH__
	__device__ uint32_t t() const { return threadIdx.x; }
	__device__ uint32_t n() const { return blockDim.x; }
	__device__ void sync() const { __syncthreads(); }
#else
	uint32_t t() const { return 0; }
	uint32_t n() const { return 1; }
	void sync() const {}
#endif
};

/* the run-length stage over bytes p[a, b) entered in run state st (0: none;
 * 1-3: that many equal bytes ending at p[a - 1]; 4: a count is next):
 * bytes out, state after */
DNG_HDI uint32_t bz_run_sim(const uint8_t *p, uint32_t a, uint32_t b,
    uint32_t st, uint32_t *out_state)
{
	uint32_t len = 0;
	uint32_t prev = a ? p[a - 1] : 256;
	for (uint32_t i = a; i < b; i++) {
		const uint32_t c = p[i];
		if (st == 4) {
			len += c;
			st = 0;
			continue;
		}
		len++;
		st = st && c == prev ? st + 1 : 1;
		prev = c;
	}
	*out_state = st;
	return len;
}

/* the stable counting sort's scatter of warp w's segment [lo, hi) */
DNG_HDI void bz_scatter(const uint8_t *ll, uint32_t *tt, uint32_t *off,
    uint32_t lo, uint32_t hi)
{
#ifdef __CUDA_ARCH__
	const uint32_t lane = threadIdx.x & 31;
	for (uint32_t base = lo; base < hi; base += 32) {
		const uint32_t i = base + lane;
		const uint32_t c = i < hi ? ll[i] : 256 + lane;
		const uint32_t peers = __match_any_sync(0xffffffffu, c);
		if (i < hi) {
			const uint32_t rank = __popc(peers & ((1u << lane) - 1));
			const uint32_t at = off[c] + rank;
			tt[at] |= i << 8;
		}
		__syncwarp();
		if (i < hi && (peers & ((1u << lane) - 1)) == 0)
			off[c] += __popc(peers);
		__syncwarp();
	}
#else
	for (uint32_t i = lo; i < hi; i++)
		tt[off[ll[i]]++] |= i << 8;
#endif
}

/*
 * Invert one block: j.slot holds its n BWT bytes; afterwards it holds the n
 * bytes of the inverse transform (randomisation undone), and j.chunks each
 * chunk's output offset and run state for bz_emit_one.
 */
DNG_HDI void bz_ibwt_one(const BzBwtJob &j, BzBwtShared *S, BzCta C,
    BzBwtResult &r)
{
	const uint32_t t = C.t(), nt = C.n(), n = j.n;
	const uint32_t nw = nt >= 32 ? nt / 32 : 1;
	const uint32_t w = t / 32 < nw ? t / 32 : 0;
	uint8_t *ll = j.slot;
	uint32_t *tt = j.tt;
	/* 1. counts per warp over equal segments, and the low bytes */
	const uint32_t seg = (n + nw - 1) / nw;
	const uint32_t lo = w * seg < n ? w * seg : n;
	const uint32_t hi = lo + seg < n ? lo + seg : n;
	for (uint32_t i = t; i < 256 * nw; i += nt)
		S->cnt[i / 256][i % 256] = 0;
	C.sync();
	for (uint32_t i = t; i < n; i += nt)
		tt[i] = ll[i];
	for (uint32_t i = lo + (nt >= 32 ? t % 32 : 0); i < hi;
	    i += (nt >= 32 ? 32 : 1)) {
#ifdef __CUDA_ARCH__
		atomicAdd(&S->cnt[w][ll[i]], 1u);
#else
		S->cnt[w][ll[i]]++;
#endif
	}
	C.sync();
	/* 2. each warp's first place for each byte value */
	if (t == 0) {
		uint32_t at = 0;
		for (uint32_t c = 0; c < 256; c++) {
			for (uint32_t v = 0; v < nw; v++) {
				const uint32_t k = S->cnt[v][c];
				S->cnt[v][c] = at;
				at += k;
			}
		}
	}
	C.sync();
	/* 3. the stable scatter: tt[k] high bits = the position sorted to k */
	if (t / 32 < nw || nt < 32)
		bz_scatter(ll, tt, S->cnt[w], lo, hi);
	C.sync();
	/* 4. walkers: sampled positions marked, each runs to the next mark */
	const uint32_t stride = (n + BZ_WALKERS - 1) / BZ_WALKERS;
	const uint32_t ns = (n + stride - 1) / stride;
	for (uint32_t k = t; k < ns; k += nt)
		tt[k * stride] |= BZ_MARK;
	C.sync();
	for (uint32_t k = t; k < ns; k += nt) {
		uint32_t e = tt[k * stride], len = 0, p;
		do {
			len++;
			p = (e >> 8) & BZ_TMASK;
			e = tt[p];
		} while (!(e & BZ_MARK) && len < n);
		S->seg_len[k] = len;
		S->seg_next[k] = (uint16_t)(p / stride);
		S->seg_off[k] = ~0u;
	}
	C.sync();
	/* 5. link the segments from origPtr (a walk that returns to itself
	 * before n bytes, which no encoder writes, is walked by one thread) */
	if (t == 0) {
		uint32_t p = (tt[j.orig] >> 8) & BZ_TMASK, h = 0;
		while (h < n && !(tt[p] & BZ_MARK)) {
			h++;
			p = (tt[p] >> 8) & BZ_TMASK;
		}
		uint32_t fb = h >= n;
		if (!fb) {
			uint32_t k = p / stride, off = h;
			while (off < n) {
				if (S->seg_off[k] != ~0u) {
					fb = 1;
					break;
				}
				S->seg_off[k] = off;
				off += S->seg_len[k];
				k = S->seg_next[k];
			}
		}
		S->head = fb ? n : h;
		S->fallback = fb;
	}
	C.sync();
	/* 6. walk again and write */
	if (t == 0) {
		uint32_t p = (tt[j.orig] >> 8) & BZ_TMASK;
		for (uint32_t i = 0; i < S->head; i++) {
			const uint32_t e = tt[p];
			ll[i] = (uint8_t)e;
			p = (e >> 8) & BZ_TMASK;
		}
	}
	if (!S->fallback)
		for (uint32_t k = t; k < ns; k += nt) {
			const uint32_t off = S->seg_off[k];
			if (off == ~0u)
				continue;
			uint32_t p = k * stride;
			const uint32_t end = off + S->seg_len[k] < n ?
			    off + S->seg_len[k] : n;
			for (uint32_t i = off; i < end; i++) {
				const uint32_t e = tt[p];
				ll[i] = (uint8_t)e;
				p = (e >> 8) & BZ_TMASK;
			}
		}
	C.sync();
	/* 7. randomised blocks: byte (r0 + ... + rk) - 2 has its low bit
	 * flipped, the table taken round */
	if (j.rand && t == 0) {
		uint64_t at = 0;
		for (uint32_t k = 0;; k++) {
			at += bz_rnum(k & 511);
			if (at - 2 >= n)
				break;
			ll[at - 2] ^= 1;
		}
	}
	C.sync();
	/* 8. run lengths per chunk from every incoming state, composed */
	const uint32_t cs = (n + BZ_CHUNKS - 1) / BZ_CHUNKS;
	for (uint32_t c = t; c < BZ_CHUNKS; c += nt) {
		const uint32_t a = c * cs < n ? c * cs : n;
		const uint32_t b = a + cs < n ? a + cs : n;
		for (uint32_t st = 0; st < 5; st++) {
			uint32_t o;
			S->run_len[c][st] = bz_run_sim(ll, a, b, st, &o);
			S->run_out[c][st] = (uint8_t)o;
		}
	}
	C.sync();
	if (t == 0) {
		uint64_t off = 0;
		uint32_t st = 0;
		for (uint32_t c = 0; c < BZ_CHUNKS; c++) {
			j.chunks[2 * c] = (uint32_t)off;
			j.chunks[2 * c + 1] = st;
			off += S->run_len[c][st];
			st = S->run_out[c][st];
		}
		r.out_len = off;
		r.ok = st != 4;
		r.pad = 0;
	}
	C.sync();
}

/* ---- emit: the final run-length stage, and the block CRC ----------------*/

struct BzEmitJob {
	const uint8_t *slot;	/* the inverse transform */
	const uint32_t *chunks;
	uint8_t *out;
	uint32_t n, pad;
};

/* CRC-32 MSB first, polynomial 0x04c11db7 (bzip2's) */
DNG_HDI void bz_crc_table(uint32_t *t, uint32_t lane, uint32_t nl)
{
	for (uint32_t i = lane; i < 256; i += nl) {
		uint32_t c = i << 24;
		for (int k = 0; k < 8; k++)
			c = c & 0x80000000u ? (c << 1) ^ 0x04c11db7u : c << 1;
		t[i] = c;
	}
}

/* a * b modulo the polynomial (bit i is x^i) */
DNG_HDI uint32_t bz_mulmod(uint32_t a, uint32_t b)
{
	uint32_t p = 0;
	for (int i = 31; i >= 0; i--) {
		p = p & 0x80000000u ? (p << 1) ^ 0x04c11db7u : p << 1;
		if (a >> i & 1)
			p ^= b;
	}
	return p;
}

/* x^(8 nb) modulo the polynomial */
DNG_HDI uint32_t bz_crc_shift(uint64_t nb)
{
	uint32_t x = 2, p = 1;
	uint64_t k = nb * 8;
	while (k) {
		if (k & 1)
			p = bz_mulmod(x, p);
		x = bz_mulmod(x, x);
		k >>= 1;
	}
	return p;
}

/* one chunk's output and CRC (init ~0, final ~) */
DNG_HDI uint32_t bz_emit_chunk(const BzEmitJob &j, const uint32_t *crct,
    uint32_t c, uint64_t *len)
{
	const uint32_t n = j.n, cs = (n + BZ_CHUNKS - 1) / BZ_CHUNKS;
	const uint32_t a = c * cs < n ? c * cs : n;
	const uint32_t b = a + cs < n ? a + cs : n;
	uint8_t *o = j.out + j.chunks[2 * c];
	uint32_t st = j.chunks[2 * c + 1];
	uint32_t prev = a ? j.slot[a - 1] : 256;
	uint32_t crc = 0xffffffffu;
	uint64_t k = 0;
	for (uint32_t i = a; i < b; i++) {
		const uint32_t v = j.slot[i];
		if (st == 4) {
			for (uint32_t m = 0; m < v; m++) {
				o[k++] = (uint8_t)prev;
				crc = (crc << 8) ^ crct[(crc >> 24) ^ prev];
			}
			st = 0;
			continue;
		}
		o[k++] = (uint8_t)v;
		crc = (crc << 8) ^ crct[(crc >> 24) ^ v];
		st = st && v == prev ? st + 1 : 1;
		prev = v;
	}
	*len = k;
	return ~crc;
}

#ifdef __CUDACC__
enum { BZ_DEC_WARPS = 4 };	/* warps per CTA of bz_decode_kernel */

/* bytes i of file blockIdx.y, a grid-stride over the file */
__global__ void __launch_bounds__(256)
bz_find_kernel(const BzFile *files, BzCand *out, uint32_t cap,
    uint32_t *count, unsigned long long *nz_end)
{
	const uint32_t f = blockIdx.y;
	const uint8_t *in = files[f].in;
	const uint64_t len = files[f].len;
	unsigned long long nz = 0;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	    i < len; i += (uint64_t)gridDim.x * blockDim.x) {
		if (in[i])
			nz = i + 1;
		uint32_t m = bz_find_at(in, len, i);
		while (m) {
			const uint32_t b = __ffs(m) - 1;
			m &= m - 1;
			const uint32_t at = atomicAdd(count, 1u);
			if (at >= cap)
				continue;
			BzCand c;
			c.bit = i * 8 + (b & 7);
			c.file = f;
			c.kind = b < 8 ? BZ_CAND_BLOCK : BZ_CAND_EOS;
			c.crc = c.next = 0;
			if (c.kind == BZ_CAND_EOS)
				bz_eos_tail(in, len, c);
			out[at] = c;
		}
	}
	if (nz)
		atomicMax(&nz_end[f], nz);
}

/* one warp per block candidate, taken from *next */
__global__ void __launch_bounds__(32 * BZ_DEC_WARPS)
bz_decode_kernel(const BzDecJob *jobs, BzDecResult *res, uint32_t njobs,
    uint32_t *next)
{
	__shared__ BzDecShared sh[BZ_DEC_WARPS];
	const uint32_t lane = threadIdx.x & 31;
	BzDecShared *S = &sh[threadIdx.x >> 5];
	for (;;) {
		uint32_t j = 0;
		if (lane == 0)
			j = atomicAdd(next, 1u);
		j = __shfl_sync(0xffffffffu, j, 0);
		if (j >= njobs)
			return;
		BzDecResult r;
		bz_decode_one(jobs[j], S, InfLanes(), r);
		if (lane == 0)
			res[j] = r;
		__syncwarp();
	}
}

/* one CTA per chained block */
__global__ void __launch_bounds__(BZ_THREADS)
bz_ibwt_kernel(const BzBwtJob *jobs, BzBwtResult *res)
{
	__shared__ BzBwtShared sh;
	BzBwtResult r;
	bz_ibwt_one(jobs[blockIdx.x], &sh, BzCta(), r);
	if (threadIdx.x == 0)
		res[blockIdx.x] = r;
}

/* one CTA per block: one thread per chunk, CRC pieces joined by thread 0 */
__global__ void __launch_bounds__(BZ_THREADS)
bz_emit_kernel(const BzEmitJob *jobs, uint32_t *crcs)
{
	__shared__ uint32_t crct[256];
	__shared__ uint32_t piece[BZ_CHUNKS], shift[BZ_CHUNKS];
	bz_crc_table(crct, threadIdx.x, blockDim.x);
	__syncthreads();
	const BzEmitJob &j = jobs[blockIdx.x];
	for (uint32_t c = threadIdx.x; c < BZ_CHUNKS; c += blockDim.x) {
		uint64_t len;
		piece[c] = bz_emit_chunk(j, crct, c, &len);
		shift[c] = bz_crc_shift(len);
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		uint32_t crc = 0;
		for (uint32_t c = 0; c < BZ_CHUNKS; c++)
			crc = bz_mulmod(shift[c], crc) ^ piece[c];
		crcs[blockIdx.x] = crc;
	}
}
#endif

} /* namespace dng */

#endif /* DNG_BUNZIP_CUH */
