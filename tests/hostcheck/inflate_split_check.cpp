/*
 * inflate_split_check: the split gzip decoder (dragnet_b200/csrc/
 * inflate_split.cuh) built for the host and run as one lane, every stage in
 * the order the library runs them; and the split policy (inflate_policy.h)
 * (TEST ONLY; tests/test_inflate_split_host.py).
 *
 *   inflate_split_check CHUNK IN OUT
 *
 * IN holds the cases: a u32 count, then per case a u64 length and the bytes.
 * Each case is cut into chunks of about CHUNK compressed bytes, and its
 * candidates found, chunks decoded (again in four times the room while the
 * chain ends in one that ran out), chained, resolved and checked; where the
 * split path cannot vouch for the result, the file is decoded whole by
 * inflate_one, as the library does.  OUT gets per case: u32 status, u32 kind,
 * u64 bit, u32 members, u32 fallbacks, u32 chunks, u32 false starts, u32 room
 * passes, u64 length and the bytes (none on error); then u32 chunks and per
 * chunk its first bit and candidate (u64 each); then u32 count and the bits
 * of the dynamic-block starts a sequential decode crosses (u64 each).
 *
 *   inflate_split_check policy FLOOR RESIDENT SIZE...
 *
 * prints the chunks of each file, space separated.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "inflate_policy.h"
#include "inflate_split.cuh"

using namespace dng;

static bool get(FILE *f, void *p, size_t n)
{
	return fread(p, 1, n, f) == n;
}

struct Chunk {
	std::vector<uint16_t> sym;
	std::vector<InfMember> mem;
	SplitJob job;
};

static void decode(const uint8_t *src, uint64_t len, const uint64_t *cand,
    uint32_t n, uint32_t k, uint64_t room, uint32_t mcap, Chunk &c,
    InfTables *T, SplitRes &r)
{
	c.sym.assign(room, 0);
	c.mem.assign(mcap, InfMember());
	c.job = { src, len, cand, c.sym.data(), room, c.mem.data(), k, n, mcap,
	    0 };
	split_decode(c.job, T, InfLanes(), r);
}

/* the whole file by inflate_one, in more room while it runs out */
static void whole(const uint8_t *src, uint64_t len, InfTables *T,
    const uint32_t *crct, InfResult &r, std::vector<uint8_t> &out)
{
	uint64_t cap = len >= 4 ? inflate_hint(src + len - 4, len) : 0;
	for (;;) {
		out.assign(cap ? cap : 1, 0);
		InfJob j = { src, len, out.data(), cap };
		inflate_one(j, T, crct, r);
		if (r.status != INF_ROOM)
			break;
		cap = cap < 32 ? 64 : cap * 2;
	}
	out.resize(r.status == INF_DONE ? r.out_len : 0);
}

/* the dynamic-block starts of a sequential decode: each decode lands on the
 * next block start (every bit is a candidate) and the next resumes there */
static std::vector<uint64_t> block_starts(const uint8_t *src, uint64_t len,
    InfTables *T)
{
	std::vector<uint64_t> all(len * 8 + 1), out;
	for (uint64_t i = 0; i < all.size(); i++)
		all[i] = i;
	uint64_t b = 0;
	uint64_t room = 1 << 16;
	Chunk c;
	for (;;) {
		SplitRes r;
		decode(src, len, all.data(), (uint32_t)all.size(), (uint32_t)b,
		    room, 1, c, T, r);
		if (r.status == INF_ROOM) {
			room *= 4;
			continue;
		}
		if (r.status != INF_DONE || r.land == INF_NOLAND)
			break;
		b = r.land;
		const uint64_t i = b >> 3;
		if (i >= len)
			break;
		const uint32_t v = (src[i] | (i + 1 < len ? src[i + 1] << 8 : 0)) >>
		    (b & 7);
		if (((v >> 1) & 3) == 2)
			out.push_back(b);
	}
	return out;
}

static int policy(int argc, char **argv)
{
	const uint64_t floor = strtoull(argv[2], nullptr, 10);
	const uint64_t resident = strtoull(argv[3], nullptr, 10);
	std::vector<uint64_t> sizes;
	for (int i = 4; i < argc; i++)
		sizes.push_back(strtoull(argv[i], nullptr, 10));
	std::vector<uint32_t> chunks(sizes.size());
	gz_split_plan(sizes.data(), sizes.size(), resident, floor,
	    chunks.data());
	for (size_t i = 0; i < chunks.size(); i++)
		printf("%s%u", i ? " " : "", chunks[i]);
	printf("\n");
	return 0;
}

int main(int argc, char **argv)
{
	if (argc >= 4 && !strcmp(argv[1], "policy"))
		return policy(argc, argv);
	if (argc != 4) {
		fprintf(stderr, "usage: inflate_split_check CHUNK IN OUT\n");
		return 2;
	}
	const uint64_t cs = strtoull(argv[1], nullptr, 10);
	FILE *in = fopen(argv[2], "rb"), *out = fopen(argv[3], "wb");
	if (!in || !out || !cs) {
		perror("open");
		return 2;
	}
	uint32_t count = 0;
	if (!get(in, &count, 4))
		return 2;
	uint32_t crct[256];
	crc32_table(crct, 0, 1);
	InfTables *T = new InfTables();
	InfHeadTables *H = new InfHeadTables();
	for (uint32_t c = 0; c < count; c++) {
		uint64_t len = 0;
		if (!get(in, &len, 8))
			return 2;
		/* a heap block of exactly `len` bytes, so ASan sees overreads */
		uint8_t *src = (uint8_t *)malloc(len ? len : 1);
		if (len && !get(in, src, len))
			return 2;
		const uint64_t hint = len >= 4 ? inflate_hint(src + len - 4, len) :
		    0;
		const uint32_t n = len / cs > 1 ? (uint32_t)(len / cs) : 1;
		/* 1. candidates */
		std::vector<uint64_t> cand(n, 0), lo(n, 0);
		for (uint32_t k = 1; k < n; k++) {
			lo[k] = split_cut(len, n, k) * 8;
			const SplitFind f = { src, len, lo[k],
			    split_cut(len, n, k + 1) * 8, &cand[k] };
			split_find(f, H, InfLanes());
		}
		/* 2. speculative decode, 3. chain, in more room while needed */
		std::vector<Chunk> ch(n);
		std::vector<SplitRes> res(n);
		std::vector<uint64_t> room(n);
		std::vector<uint32_t> mcap(n, SPLIT_MSLOTS);
		for (uint32_t k = 0; k < n; k++) {
			room[k] = split_room(hint, len, split_cut(len, n, k + 1) -
			    split_cut(len, n, k));
			decode(src, len, cand.data(), n, k, room[k], mcap[k], ch[k],
			    T, res[k]);
		}
		std::vector<uint32_t> proven, redo;
		uint32_t passes = 0;
		int chain;
		while ((chain = split_chain(res.data(), proven)) == CHAIN_ROOM) {
			split_redo(res.data(), n, proven, redo);
			for (const uint32_t k : redo) {
				room[k] *= 4;
				mcap[k] *= 4;
				decode(src, len, cand.data(), n, k, room[k],
				    mcap[k], ch[k], T, res[k]);
			}
			passes++;
		}
		uint32_t fallbacks = 0, members = 0, false_starts = 0;
		std::vector<uint8_t> bytes;
		InfResult r = {};
		bool ok = chain == CHAIN_END;
		if (ok) {
			false_starts = split_false_starts(res.data(), n, proven);
			std::vector<const InfMember *> mem(n);
			for (uint32_t k = 0; k < n; k++)
				mem[k] = ch[k].mem.data();
			SplitLayout lay;
			split_layout(res.data(), mem.data(), proven, lay);
			/* 4. resolve: tails in chain order, then the bodies */
			bytes.assign(lay.len ? lay.len : 1, 0);
			std::vector<SplitPiece> pieces;
			for (size_t i = 0; i < proven.size(); i++) {
				const uint32_t k = proven[i];
				pieces.push_back({ ch[k].sym.data(), bytes.data(),
				    lay.off[i], res[k].out_len, lay.minidx[i], 0 });
			}
			for (const SplitPiece &p : pieces)
				ok &= split_resolve(p, split_tail(p), p.len, 0, 1);
			for (const SplitPiece &p : pieces)
				ok &= split_resolve(p, 0, split_tail(p), 0, 1);
			/* 5. every member's CRC-32 over pieces, and ISIZE */
			std::vector<CrcPiece> cp;
			std::vector<uint32_t> crcs;
			for (size_t m = 0; ok && m < lay.mstart.size(); m++) {
				CrcMember cm = { (uint32_t)cp.size(), 0, lay.crc[m],
				    lay.isize[m], lay.mend[m] - lay.mstart[m], 0,
				    0 };
				for (uint64_t a = lay.mstart[m]; a < lay.mend[m];
				    a += SPLIT_CRC_PIECE) {
					const uint64_t b = a + SPLIT_CRC_PIECE <
					    lay.mend[m] ? a + SPLIT_CRC_PIECE :
					    lay.mend[m];
					cp.push_back({ bytes.data() + a, b - a });
					crcs.push_back(crc32_run(crct, bytes.data() + a,
					    b - a));
				}
				cm.p1 = (uint32_t)cp.size();
				ok &= split_member_ok(cm, cp.data(), crcs.data(),
				    InfLanes());
			}
			members = (uint32_t)lay.mstart.size();
			bytes.resize(lay.len);
		}
		if (ok) {
			r.status = INF_DONE;
		} else {
			fallbacks = 1;
			whole(src, len, T, crct, r, bytes);
			members = r.members;
		}
		const uint64_t olen = r.status == INF_DONE ? bytes.size() : 0;
		fwrite(&r.status, 4, 1, out);
		fwrite(&r.kind, 4, 1, out);
		fwrite(&r.bit, 8, 1, out);
		fwrite(&members, 4, 1, out);
		fwrite(&fallbacks, 4, 1, out);
		fwrite(&n, 4, 1, out);
		fwrite(&false_starts, 4, 1, out);
		fwrite(&passes, 4, 1, out);
		fwrite(&olen, 8, 1, out);
		if (olen)
			fwrite(bytes.data(), 1, olen, out);
		fwrite(&n, 4, 1, out);
		for (uint32_t k = 0; k < n; k++) {
			fwrite(&lo[k], 8, 1, out);
			fwrite(&cand[k], 8, 1, out);
		}
		const std::vector<uint64_t> starts = block_starts(src, len, T);
		const uint32_t ns = (uint32_t)starts.size();
		fwrite(&ns, 4, 1, out);
		if (ns)
			fwrite(starts.data(), 8, ns, out);
		free(src);
	}
	delete T;
	delete H;
	fclose(out);
	return 0;
}
