/*
 * bunzip_check: the bzip2 decoder (dragnet_b200/csrc/bunzip.cuh) built for
 * the host, every stage one lane, in the library's order: find, waves of
 * block candidates decoded, the chain, inverse BWT, run lengths, emit and
 * CRCs (TEST ONLY; tests/test_bunzip_host.py).
 *
 *   bunzip_check IN OUT WAVE
 *
 * IN holds the cases: a u32 count, then per case a u64 length, the bytes, a
 * u32 count of extra candidates and their u64 bit offsets (decoded as block
 * candidates beside the ones found, which must never change the result).
 * WAVE is the number of block candidates per wave.  OUT gets per case: u32
 * error kind (BE_*), u64 error bit, u32 streams, u32 blocks, u32 false
 * starts, u64 length and the decoded bytes (none on error).  Every buffer is
 * exactly as long as its content, so a read or write past either end is
 * caught by -fsanitize=address.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "bunzip.cuh"
#include "bunzip_policy.h"

using namespace dng;

static bool get(FILE *f, void *p, size_t n)
{
	return fread(p, 1, n, f) == n;
}

struct Out {
	uint32_t kind = BE_NONE;
	uint64_t bit = 0;
	uint32_t streams = 0, blocks = 0, false_starts = 0;
	std::vector<uint8_t> bytes;
};

static void decode_file(const uint8_t *in, uint64_t len,
    const std::vector<uint64_t> &extra, size_t wave, Out &o)
{
	/* find */
	std::vector<BzCand> cand;
	uint64_t nz_end = 0;
	for (uint64_t i = 0; i < len; i++) {
		if (in[i])
			nz_end = i + 1;
		uint32_t m = bz_find_at(in, len, i);
		for (uint32_t b = 0; b < 16; b++) {
			if (!(m >> b & 1))
				continue;
			BzCand c = {};
			c.bit = i * 8 + (b & 7);
			c.kind = b < 8 ? BZ_CAND_BLOCK : BZ_CAND_EOS;
			if (c.kind == BZ_CAND_EOS)
				bz_eos_tail(in, len, c);
			cand.push_back(c);
		}
	}
	for (uint64_t bit : extra) {
		bool dup = false;
		for (const BzCand &c : cand)
			dup |= c.bit == bit;
		if (!dup && bit < len * 8) {
			BzCand c = {};
			c.bit = bit;
			c.kind = BZ_CAND_BLOCK;
			cand.push_back(c);
		}
	}
	std::sort(cand.begin(), cand.end(), [](const BzCand &a,
	    const BzCand &b) { return a.bit < b.bit; });
	std::vector<uint32_t> bidx, which(cand.size(), ~0u);
	for (uint32_t i = 0; i < cand.size(); i++)
		if (cand[i].kind == BZ_CAND_BLOCK) {
			which[i] = (uint32_t)bidx.size();
			bidx.push_back(i);
		}
	std::vector<size_t> ends(bidx.size() + 1);
	const size_t nw = bz_waves(bidx.size(), wave, ends.data());

	BzChain ch;
	const uint32_t head = len >= 4 ? (uint32_t)in[0] << 24 |
	    (uint32_t)in[1] << 16 | (uint32_t)in[2] << 8 | in[3] : 0;
	bz_chain_init(ch, len, nz_end, head);
	BzDecShared *DS = new BzDecShared();
	BzBwtShared *BS = new BzBwtShared();
	uint32_t crct[256];
	bz_crc_table(crct, 0, 1);
	std::vector<BzDecResult> res(bidx.size());
	std::vector<uint8_t *> slots(bidx.size(), nullptr);
	std::vector<uint32_t *> hists(bidx.size(), nullptr);
	size_t w = 0, lo = 0;
	for (;;) {
		const size_t hi = w < nw ? ends[w] : lo;
		for (size_t k = lo; k < hi; k++) {
			slots[k] = (uint8_t *)malloc(BZ_SLOT);
			hists[k] = (uint32_t *)malloc(256 * 4);
			BzDecJob j = { in, len, cand[bidx[k]].bit, slots[k],
			    hists[k] };
			bz_decode_one(j, DS, InfOneLane(), res[k]);
		}
		std::vector<size_t> took;
		bz_chain_run(ch, cand.data(), (uint32_t)cand.size(),
		    [&](uint32_t i) -> const BzDecResult * {
			const size_t k = which[i];
			return k < hi ? &res[k] : nullptr;
		    }, [&](uint32_t i) { took.push_back(which[i]); });
		o.false_starts += (uint32_t)(hi - lo - took.size());
		/* blocks before a damaged place are checked first: their CRC
		 * mismatch is the earlier damage */
		for (size_t k : took) {
			if (!o.kind) {
				const BzDecResult &r = res[k];
				uint32_t *tt = (uint32_t *)malloc(
				    (size_t)r.nblock * 4);
				uint32_t *chunks = (uint32_t *)malloc(
				    BZ_CHUNKS * 8);
				BzBwtJob bj = { slots[k], tt, hists[k], chunks,
				    r.nblock, r.orig, r.rand, 0 };
				BzBwtResult br;
				bz_ibwt_one(bj, BS, BzCta(), br);
				free(tt);
				if (!br.ok) {
					o.kind = BE_OVERFLOW;
					o.bit = cand[bidx[k]].bit;
				} else {
					uint8_t *out = (uint8_t *)malloc(
					    br.out_len ? br.out_len : 1);
					BzEmitJob ej = { slots[k], chunks, out,
					    r.nblock, 0 };
					uint32_t crc = 0;
					uint64_t sum = 0;
					for (uint32_t c = 0; c < BZ_CHUNKS;
					    c++) {
						uint64_t n;
						const uint32_t p =
						    bz_emit_chunk(ej, crct, c,
						    &n);
						crc = bz_mulmod(bz_crc_shift(n),
						    crc) ^ p;
						sum += n;
					}
					if (sum != br.out_len)
						abort();
					if (crc != r.crc) {
						o.kind = BE_BLOCK_CRC;
						o.bit = cand[bidx[k]].bit;
					}
					o.bytes.insert(o.bytes.end(), out,
					    out + br.out_len);
					free(out);
				}
				free(chunks);
			}
		}
		for (size_t k = lo; k < hi; k++) {
			free(slots[k]);
			free(hists[k]);
		}
		lo = hi;
		w++;
		if (ch.done || o.kind || w > nw)
			break;
	}
	/* candidates past the chain's end are never decoded: false starts */
	if (ch.done && !ch.kind)
		o.false_starts += (uint32_t)(bidx.size() - lo);
	if (!ch.done && !ch.kind && !o.kind)
		abort();	/* the chain waits on a wave that never comes */
	if (ch.kind && !o.kind) {
		o.kind = ch.kind;
		o.bit = ch.err_bit;
	}
	o.streams = ch.streams;
	o.blocks = ch.blocks;
	if (o.kind)
		o.bytes.clear();
	delete DS;
	delete BS;
}

int main(int argc, char **argv)
{
	if (argc != 4) {
		fprintf(stderr, "usage: bunzip_check IN OUT WAVE\n");
		return 2;
	}
	FILE *in = fopen(argv[1], "rb"), *out = fopen(argv[2], "wb");
	const size_t wave = strtoul(argv[3], nullptr, 0);
	if (!in || !out || !wave) {
		perror("open");
		return 2;
	}
	uint32_t count = 0;
	if (!get(in, &count, 4))
		return 2;
	for (uint32_t c = 0; c < count; c++) {
		uint64_t len = 0;
		uint32_t nx = 0;
		if (!get(in, &len, 8))
			return 2;
		/* a heap block of exactly `len` bytes, so ASan sees overreads */
		uint8_t *src = (uint8_t *)malloc(len ? len : 1);
		if (len && !get(in, src, len))
			return 2;
		if (!get(in, &nx, 4))
			return 2;
		std::vector<uint64_t> extra(nx);
		if (nx && !get(in, extra.data(), 8 * nx))
			return 2;
		Out o;
		decode_file(src, len, extra, wave, o);
		const uint64_t n = o.bytes.size();
		fwrite(&o.kind, 4, 1, out);
		fwrite(&o.bit, 8, 1, out);
		fwrite(&o.streams, 4, 1, out);
		fwrite(&o.blocks, 4, 1, out);
		fwrite(&o.false_starts, 4, 1, out);
		fwrite(&n, 8, 1, out);
		if (n)
			fwrite(o.bytes.data(), 1, n, out);
		free(src);
	}
	fclose(out);
	return 0;
}
