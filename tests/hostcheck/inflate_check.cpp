/*
 * inflate_check: the gzip decoder (dragnet_b200/csrc/inflate.cuh) built for
 * the host, one lane per file (TEST ONLY; tests/test_inflate_host.py).
 *
 *   inflate_check IN OUT
 *
 * IN holds the cases: a u32 count, then per case a u64 length and the bytes.
 * Each case is decoded as the library decodes a file: into the room its
 * trailer hints (inflate_hint), redecoded with twice the room while it runs
 * out.  OUT gets per case: u32 status, u32 error kind, u64 error bit, u32
 * members, u32 redecodes, u64 length and the decoded bytes (none on error).
 * Every buffer is exactly as long as its content, so a read or write past
 * either end is caught by -fsanitize=address.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "inflate.cuh"

using namespace dng;

static bool get(FILE *f, void *p, size_t n)
{
	return fread(p, 1, n, f) == n;
}

int main(int argc, char **argv)
{
	if (argc != 3) {
		fprintf(stderr, "usage: inflate_check IN OUT\n");
		return 2;
	}
	FILE *in = fopen(argv[1], "rb"), *out = fopen(argv[2], "wb");
	if (!in || !out) {
		perror("open");
		return 2;
	}
	uint32_t count = 0;
	if (!get(in, &count, 4))
		return 2;
	uint32_t crct[256];
	crc32_table(crct, 0, 1);
	InfTables *T = new InfTables();
	for (uint32_t c = 0; c < count; c++) {
		uint64_t len = 0;
		if (!get(in, &len, 8))
			return 2;
		/* a heap block of exactly `len` bytes, so ASan sees overreads */
		uint8_t *src = (uint8_t *)malloc(len ? len : 1);
		if (len && !get(in, src, len))
			return 2;
		uint64_t cap = len >= 4 ? inflate_hint(src + len - 4, len) : 0;
		uint32_t redecodes = 0;
		InfResult r;
		uint8_t *dst = nullptr;
		for (;;) {
			dst = (uint8_t *)malloc(cap ? cap : 1);
			InfJob j = { src, len, dst, cap };
			inflate_one(j, T, crct, r);
			if (r.status != INF_ROOM)
				break;
			free(dst);
			cap = cap < 32 ? 64 : cap * 2;
			redecodes++;
		}
		const uint64_t olen = r.status == INF_DONE ? r.out_len : 0;
		fwrite(&r.status, 4, 1, out);
		fwrite(&r.kind, 4, 1, out);
		fwrite(&r.bit, 8, 1, out);
		fwrite(&r.members, 4, 1, out);
		fwrite(&redecodes, 4, 1, out);
		fwrite(&olen, 8, 1, out);
		if (olen)
			fwrite(dst, 1, olen, out);
		free(dst);
		free(src);
	}
	delete T;
	fclose(out);
	return 0;
}
