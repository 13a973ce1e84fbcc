/*
 * fkey_check: TEST-ONLY host build of the F path's short group key
 * (dragnet_b200/csrc/fast.cuh FKey: fprep, fkey_short_hash, fkey_unpack).
 *
 *   fkey_check PLAN.json FILE   -> one line per record on stdout:
 *     "P HDR HASH KEY"  the record's key is a short key: its header and hash
 *                       (hex), and its bytes as fkey_unpack writes them
 *     "L KEY"           the key does not fit a short key: fkey_write's bytes
 *     "D"               the stages dropped the record
 *     "M"               the F path does not take the record
 *   (KEY in hex).  Exits 3 when fkey_unpack's bytes are not fkey_write's.
 */
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "../../dragnet_b200/csrc/record.cuh"
#include "../../dragnet_b200/csrc/tmpl.cuh"
#include "../../dragnet_b200/csrc/fast.cuh"
#include "../../dragnet_b200/csrc/result.h"
#include "../../include/dragnet_gpu.h"

using namespace dng;

static std::string slurp(const char *path)
{
	std::ifstream f(path, std::ios::binary);
	std::stringstream ss;
	ss << f.rdbuf();
	return ss.str();
}

static void hex(const u8 *p, u32 n)
{
	for (u32 i = 0; i < n; i++)
		printf("%02x", p[i]);
}

int main(int argc, char **argv)
{
	if (argc != 3) {
		fprintf(stderr, "usage: fkey_check PLAN.json FILE\n");
		return 2;
	}
	const std::string pj = slurp(argv[1]), data = slurp(argv[2]);
	static dng_plan plan;
	char err[256];
	if (dng_plan_compile(pj.c_str(), &plan, err, sizeof (err)) != 0) {
		fprintf(stderr, "plan: %s\n", err);
		return 1;
	}
	static FPlan FP;
	fplan_build(plan.dev, FP);
	if (!FP.ok) {
		fprintf(stderr, "plan: not an F plan\n");
		return 1;
	}
	/* the F templates, learnt from the head of the input as api.cu does */
	std::vector<TCandidate> cands;
	tmpl_candidates((const u8 *)data.data(), std::min<size_t>(data.size(),
	    TMPL_SAMPLE_BYTES), TMPL_MAX_LEAVES, cands);
	std::vector<TResolved> res(cands.size());
	for (size_t i = 0; i < cands.size(); i++) {
		static RecState TR;
		TResolved r0;
		parse_record((const u8 *)cands[i].sample.data(),
		    (u32)cands[i].sample.size(), plan.dev, TR);
		r0.flags = TR.flags;
		r0.set_mask = TR.set_mask;
		memcpy(r0.slots, TR.slots, sizeof (TR.slots));
		fplan_resolve(plan.dev, r0, res[i]);
	}
	std::vector<u8> fblob;
	tmpl_build(cands, res, 60000, fblob, nullptr, true);
	if (fblob.empty()) {
		fprintf(stderr, "no F templates\n");
		return 1;
	}

	static u8 kbuf[F_MAXKEY + 16], ubuf[8 * FK_COLS + 8];
	size_t pos = 0;
	while (pos < data.size()) {
		size_t nl = data.find('\n', pos);
		if (nl == std::string::npos)
			break;
		const u32 len = (u32)(nl - pos);
		FastHostMem fm;
		fm.rec = (const u8 *)data.data() + pos;
		fm.len = len;
		fm.blob = fblob.data();
		pos = nl + 1;
		u32 defmask = 0, slow = 0, h = 0, klen = 0;
		double s0 = 0, s1 = 0;
		FKey k;
		if (len > F_MAXLINE || !fmatch(fm, len, true, defmask)) {
			printf("M\n");
			continue;
		}
		const u32 fo = fstage(fm, FP, defmask, s0, s1);
		if (fo != FO_AGGR) {
			printf(fo == FO_MISS ? "M\n" : "D\n");
			continue;
		}
		if (!fprep(fm, FP, defmask, s0, s1, slow, k) ||
		    !fkey_hash(fm, FP, defmask, h, klen)) {
			printf("M\n");
			continue;
		}
		memset(kbuf, 0xee, sizeof (kbuf));
		fkey_write(fm, FP, defmask, kbuf);
		if (!k.hdr) {
			printf("L ");
			hex(kbuf, klen);
			printf("\n");
			continue;
		}
		memset(ubuf, 0xee, sizeof (ubuf));
		const u32 ulen = fkey_unpack(k, ubuf);
		if (ulen != klen || memcmp(ubuf, kbuf, (klen + 7) & ~7u) != 0) {
			fprintf(stderr, "fkey_unpack: not fkey_write's bytes\n");
			return 3;
		}
		printf("P %08x %08x ", k.hdr, fkey_short_hash(k, FP.ncols));
		hex(ubuf, ulen);
		printf("\n");
	}
	return 0;
}
