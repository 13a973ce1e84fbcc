/*
 * hostcheck: TEST-ONLY host build of the per-record device logic
 * (dragnet_b200/csrc/record.cuh) so that it can be checked against oracle/
 * in this GPU-less container before a gpurun.  It is NOT part of
 * libdragnet_gpu.so, is never installed and is not a CPU fallback: the
 * product has no host execution path.
 *
 *   hostcheck PLAN.json FILE...   -> one JSON document on stdout
 */
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <fstream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../../dragnet_b200/csrc/record.cuh"
#include "../../dragnet_b200/csrc/tmpl.cuh"
#include "../../dragnet_b200/csrc/fast.cuh"
#include "../../dragnet_b200/csrc/jit.h"
#include <dlfcn.h>
#include <unistd.h>
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

/*
 * DNG_HOSTCHECK_JIT: the matcher the run-time compiler generates for the F
 * templates (jit.cpp), two ways: (1) the real thing -- NVRTC + nvJitLink against
 * the relocatable kernel embedded in the library -- must build (no GPU needed
 * for that); (2) the same generated code compiled for the HOST with a prelude
 * that maps its shared-memory accessors onto a byte array, and used below in
 * place of fmatch(), so that its control flow and immediates are checked
 * against the oracle like everything else.
 */
static const char *HOST_PRELUDE =
"#include <stdint.h>\n#include <string.h>\n"
"typedef uint8_t u8; typedef uint32_t u32; typedef uint64_t u64;\n"
"#define DNG_HD static inline\n#define __device__\n#define __syncwarp()\n"
"enum { T_UNDEF = 0, T_NULL = 1, T_FALSE = 2, T_TRUE = 3, T_NUM = 4, T_STR = 5 };\n"
"#define DNG_FCAP(type, off, len, flag) \\\n"
"	((u32)(off) | ((u32)(len) << 12) | ((u32)(type) << 24) | ((u32)(flag) << 27))\n"
"DNG_HD bool is_hex(u32 c) { return (c >= '0' && c <= '9') || ((c | 0x20) >= 'a' && (c | 0x20) <= 'f'); }\n"
"DNG_HD u32 tm_isdigit(u32 c) { return c - '0' <= 9u; }\n"
"DNG_HD u32 nondigit_mask(u32 w) { const u32 x = w ^ 0x30303030u; return (((x & 0x7f7f7f7fu) + 0x76767676u) | x) & 0x80808080u; }\n"
"DNG_HD u32 low_flag_byte(u32 m) { u32 k = 0; while (!((m >> (8 * k + 7)) & 1)) k++; return k; }\n"
"extern \"C\" unsigned char *dng_jit_host_mem;\nunsigned char *dng_jit_host_mem;\n"
"DNG_HD u32 jlds32(u32 a) { u32 v; memcpy(&v, dng_jit_host_mem + a, 4); return v; }\n"
"DNG_HD u32 jlds8(u32 a) { return dng_jit_host_mem[a]; }\n"
"DNG_HD void jsts32(u32 a, u32 v) { memcpy(dng_jit_host_mem + a, &v, 4); }\n"
"DNG_HD u32 __funnelshift_r(u32 lo, u32 hi, u32 sh) { return sh ? (lo >> sh) | (hi << (32 - sh)) : lo; }\n"
"struct JMem {\n	u32 ra;\n	struct Cur { u32 wa, w0, w1, sh;\n"
"		u32 next() { const u32 d = __funnelshift_r(w0, w1, sh); w0 = w1; wa += 4; w1 = jlds32(wa); return d; } };\n"
"	Cur cursor(u32 off) const { Cur c; const u32 a = ra + off; c.sh = (a & 3) * 8; c.wa = (a & ~3u) + 4;\n"
"		c.w0 = jlds32(c.wa - 4); c.w1 = jlds32(c.wa); return c; }\n"
"	struct ACur { u32 wa, k; u32 next() { const u32 v = jlds32(wa); wa += 4; return v; } };\n"
"	ACur acursor(u32 off) const { ACur c; const u32 a = ra + off; c.k = a & 3; c.wa = a & ~3u; return c; }\n"
"	u32 apos(const ACur &c) const { return c.wa - 4 - ra; }\n"
"	u32 byte(u32 off) const { return jlds8(ra + off); }\n"
"	u32 word(u32 off) const { Cur c = cursor(off); return c.next(); }\n};\n";

typedef unsigned (*jmatch_fn)(unsigned, unsigned, unsigned, unsigned);

static jmatch_fn host_jit(const std::vector<u8> &fblob, const FPlan *fplan,
    unsigned char ***mem)
{
	std::string dev = jit_source(fblob.data(), fblob.size(), fplan);
	std::string cubin, err;
	double cms = 0, lms = 0;
	/* DNG_HOSTCHECK_JIT=2: the device build too (a second or two) */
	if (atoi(getenv("DNG_HOSTCHECK_JIT")) >= 2) {
		if (!jit_build(dev, 13, cubin, err, &cms, &lms)) {
			fprintf(stderr, "jit_build: %s\n", err.c_str());
			exit(4);
		}
		fprintf(stderr, "jit: %zu bytes of source, nvrtc %.0f ms, link "
		    "%.0f ms, cubin %zu bytes\n", dev.size(), cms, lms,
		    cubin.size());
	}
	if (const char *dump = getenv("DNG_HOSTCHECK_JIT_DUMP")) {
		FILE *d1 = fopen((std::string(dump) + ".cu").c_str(), "w");
		fwrite(dev.data(), 1, dev.size(), d1);
		fclose(d1);
		FILE *d2 = fopen((std::string(dump) + ".cubin").c_str(), "w");
		fwrite(cubin.data(), 1, cubin.size(), d2);
		fclose(d2);
	}
	std::string host = jit_source(fblob.data(), fblob.size(), nullptr,
	    HOST_PRELUDE);
	char dir[] = "/tmp/dng_jit_XXXXXX";
	if (!mkdtemp(dir))
		exit(4);
	std::string src = std::string(dir) + "/jm.cpp", so = std::string(dir) +
	    "/jm.so";
	FILE *f = fopen(src.c_str(), "w");
	fwrite(host.data(), 1, host.size(), f);
	fclose(f);
	std::string cmd = "g++ -std=c++17 -O1 -w -shared -fPIC -o " + so + " " + src;
	if (system(cmd.c_str()) != 0) {
		fprintf(stderr, "host build of the generated matcher failed: %s\n",
		    src.c_str());
		exit(4);
	}
	void *h = dlopen(so.c_str(), RTLD_NOW);
	if (!h) {
		fprintf(stderr, "dlopen: %s\n", dlerror());
		exit(4);
	}
	*mem = (unsigned char **)dlsym(h, "dng_jit_host_mem");
	jmatch_fn fn = (jmatch_fn)dlsym(h, "dng_jmatch");
	unlink(src.c_str());
	unlink(so.c_str());
	rmdir(dir);
	if (!fn || !*mem)
		exit(4);
	return fn;
}

int main(int argc, char **argv)
{
	if (argc < 2) {
		fprintf(stderr, "usage: hostcheck PLAN.json FILE...\n");
		return 2;
	}
	std::string pj = slurp(argv[1]);
	static dng_plan plan;
	char err[256];
	int rc = dng_plan_compile(pj.c_str(), &plan, err, sizeof (err));
	if (rc != 0) {
		fprintf(stderr, "plan: %s\n", err);
		return 1;
	}
	std::string data;
	for (int i = 2; i < argc; i++)
		data += slurp(argv[i]);

	LocalCounters C;
	memset(&C, 0, sizeof (C));
	bool use_fast = getenv("DNG_HOSTCHECK_FAST") != nullptr;
	unsigned long nfast = 0, ntmpl = 0;
	/* DNG_HOSTCHECK_TMPL: learn record templates from the head of the input
	 * (as api.cu does, with the parser run on the host instead of by
	 * resolve_kernel) and try them before the other parsers */
	std::vector<u8> blob;
	if (getenv("DNG_HOSTCHECK_TMPL") != nullptr) {
		std::vector<TCandidate> cands;
		tmpl_candidates((const u8 *)data.data(),
		    std::min<size_t>(data.size(), TMPL_SAMPLE_BYTES),
		    TMPL_MAX_LEAVES, cands);
		std::vector<TResolved> res(cands.size());
		for (size_t i = 0; i < cands.size(); i++) {
			static RecState TR;
			parse_record((const u8 *)cands[i].sample.data(),
			    (u32)cands[i].sample.size(), plan.dev, TR);
			res[i].flags = TR.flags;
			res[i].set_mask = TR.set_mask;
			memcpy(res[i].slots, TR.slots, sizeof (TR.slots));
		}
		tmpl_build(cands, res, 60000, blob, nullptr);
		if (getenv("DNG_HOSTCHECK_TMPL_DEBUG"))
			fprintf(stderr, "tmpl: %zu candidates, blob %zu bytes, "
			    "%u nodes, %u leaves\n", cands.size(), blob.size(),
			    blob.empty() ? 0 : ((THdr *)blob.data())->nnodes,
			    blob.empty() ? 0 : ((THdr *)blob.data())->nleaves);
	}
	/* DNG_HOSTCHECK_F: the F path (fast.cuh) in front of everything else:
	 * its own (path indexed, compact) templates, its stages and its
	 * piece-wise key functions; misses fall through to the code below */
	static FPlan FP;
	std::vector<u8> fblob;
	unsigned long nf_match = 0, nf_miss = 0;
	std::map<std::string, u32> fhashes;
	if (getenv("DNG_HOSTCHECK_F") != nullptr) {
		fplan_build(plan.dev, FP);
		if (FP.ok) {
			std::vector<TCandidate> cands;
			tmpl_candidates((const u8 *)data.data(),
			    std::min<size_t>(data.size(), TMPL_SAMPLE_BYTES),
			    TMPL_MAX_LEAVES, cands);
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
			tmpl_build(cands, res, 60000, fblob, nullptr, true);
		}
	}
	jmatch_fn jm = nullptr;
	unsigned char **jmem = nullptr;
	static unsigned char jbuf[65536];
	if (getenv("DNG_HOSTCHECK_JIT") != nullptr && !fblob.empty()) {
		jm = host_jit(fblob, &FP, &jmem);
		*jmem = jbuf;
	}
	/* DNG_HOSTCHECK_KEYS=PATH: one line per tallied record, "KEY FHASH GHASH"
	 * (key bytes in hex; the F path's 32-bit hash, "-" when the F path did
	 * not take the record; the general 64-bit hash), so that tests can pick
	 * keys that collide in the device's tally tables.  Skips the all-pairs
	 * fkey_equal check, which is quadratic in the keys. */
	FILE *keys_out = nullptr;
	if (const char *kp = getenv("DNG_HOSTCHECK_KEYS")) {
		keys_out = fopen(kp, "w");
		if (!keys_out) {
			fprintf(stderr, "cannot write %s\n", kp);
			return 2;
		}
	}
	auto dump_key = [&](const u8 *k, u32 klen, const char *fh) {
		static u8 padded[KEY_MAX + 64];
		memset(padded, 0, sizeof (padded));
		memcpy(padded, k, klen);
		for (u32 i = 0; i < klen; i++)
			fprintf(keys_out, "%02x", k[i]);
		fprintf(keys_out, " %s %016llx\n", fh,
		    (unsigned long long)key_hash(padded, klen));
	};
	static LocalCounters MCs[MAX_METRICS];
	memset(MCs, 0, sizeof (MCs));
	std::map<std::string, uint64_t> table;
	static RecState R;
	static u8 kbuf[KEY_MAX + 64];
	size_t pos = 0;
	while (pos < data.size()) {
		size_t nl = data.find('\n', pos);
		size_t end = nl == std::string::npos ? data.size() : nl;
		u32 len = (u32)(end - pos);
		const u8 *rec = (const u8 *)data.data() + pos;
		C.lines++;
		bool done = false;
		if (!fblob.empty() && nl != std::string::npos && len <= 4095) {
			FastHostMem fm;
			fm.rec = rec;
			fm.len = len;
			fm.blob = fblob.data();
			u32 defmask = 0;
			double s0 = 0, s1 = 0;
			u32 fo = FO_MISS, h = 0, klen = 0, slow = 0;
			bool matched;
			if (jm) {
				/* the record at an odd address of the fake shared
				 * memory, '\n' and the sentinel quotes after it,
				 * captures in rows of F_NT */
				const u32 ra = 1027, caps = 32768;
				memcpy(jbuf + ra, rec, len);
				jbuf[ra + len] = '\n';
				memset(jbuf + ra + len + 1, '"', 64);
				const unsigned r = jm(ra, len, 1, caps);
				matched = r & 1;
				defmask = r >> 1;
				for (u32 k = 0; k < F_MAXPATHS; k++)
					memcpy(&fm.caps[k], jbuf + caps + k * F_NT * 4, 4);
			} else {
				matched = fmatch(fm, len, true, defmask);
			}
			if (matched)
				fo = fstage(fm, FP, defmask, s0, s1);
			if (fo == FO_AGGR &&
			    (!fprep(fm, FP, defmask, s0, s1, slow) ||
			    !fkey_hash(fm, FP, defmask, h, klen)))
				fo = FO_MISS;
			if (fo != FO_MISS) {
				nf_match++;
				switch (fo) {
				case FO_DS_FILTERED: C.ds_filtered++; break;
				case FO_DS_FAILED: C.ds_failedeval++; break;
				case FO_USER_FILTERED: C.user_filtered++; break;
				case FO_USER_FAILED: C.user_failedeval++; break;
				case FO_SYNTH_UNDEF: C.synth_undef++; break;
				case FO_SYNTH_BADDATE: C.synth_baddate++; break;
				case FO_TIME_FILTERED: C.time_filtered++; break;
				case FO_TIME_FAILED: C.time_failedeval++; break;
				default: {
					memset(kbuf, 0xee, F_MAXKEY + 8);
					fkey_write(fm, FP, defmask, kbuf);
					std::string key((char *)kbuf, klen);
					/* the piece-wise functions agree with the
					 * key they describe */
					FastHostKey hk;
					hk.key = kbuf;
					hk.len = klen;
					if (!fkey_equal(fm, FP, defmask, hk)) {
						fprintf(stderr, "fkey_equal: own key\n");
						return 3;
					}
					auto it = fhashes.find(key);
					if (it != fhashes.end() && it->second != h) {
						fprintf(stderr, "fkey_hash: unstable\n");
						return 3;
					}
					if (keys_out) {
						char fh[16];
						snprintf(fh, sizeof (fh), "%08x", h);
						dump_key(kbuf, klen, fh);
					}
					for (auto &kv : fhashes) {
						if (keys_out)
							break;
						if (kv.first == key ||
						    kv.first.size() != key.size())
							continue;
						FastHostKey ok_;
						ok_.key = (const u8 *)kv.first.data();
						ok_.len = (u32)kv.first.size();
						if (fkey_equal(fm, FP, defmask, ok_)) {
							fprintf(stderr, "fkey_equal: "
							    "other key\n");
							return 3;
						}
					}
					fhashes[key] = h;
					table[key] += 1;
					C.aggr++;
					if (slow)
						C.slow++;
				}
				}
				pos = end + 1;
				continue;
			}
			nf_miss++;
		}
		if (!blob.empty() && nl != std::string::npos) {
			TmplHostMem m;
			m.rec = rec;
			m.len = len;
			m.blob = blob.data();
			if (tmpl_match(m, len, R, true)) {
				done = true;
				ntmpl++;
			}
		}
		if (!done && use_fast && plan.dev.hot.fast.ok && len <= 2048) {
			FastState fs;
			fast_init(fs);
			for (u32 i = 0; i <= len; i++)
				fast_step(fs, plan.dev.hot, R.slots,
				    i < len ? rec[i] : (u8)'\n', i);
			/* keep stepping on garbage like neighbouring lanes do */
			for (u32 i = 0; i < 64; i++)
				fast_step(fs, plan.dev.hot, R.slots,
				    (u8)("{\"x\":[1,\"\\\n}]"[i % 12]), len + 1 + i);
			if (fs.state == FS_FIN) {
				fast_finish(rec, fs, R);
				done = true;
				nfast++;
			} else if (fs.state == FS_ERR) {
				R.flags = RF_INVALID;
				R.set_mask = 0;
				done = true;
				nfast++;
			}
		}
		if (!done)
			parse_record(rec, len, plan.dev, R);
		if (R.flags & RF_UNSUPPORTED)
			C.unsupported++;
		if (R.flags & RF_INVALID) {
			C.invalid_json++;
		} else {
			u32 klen;
			u64 w;
			if (prepare_record(rec, plan.dev, R, C, kbuf, w)) {
				for (u32 mi = 0; mi < plan.dev.nmetrics; mi++) {
					LocalCounters &MC = mi ? MCs[mi] : C;
					if (process_metric(rec, plan.dev, mi, R, MC,
					    kbuf, klen)) {
						if (keys_out)
							dump_key(kbuf, klen, "-");
						table[std::string((char *)kbuf,
						    klen)] += w;
					}
				}
			}
		}
		pos = end + 1;
	}
	if (keys_out)
		fclose(keys_out);
	dng_result res;
	res.init_from_plan(&plan);
	for (auto &kv : table) {
		res.keys.push_back(kv.first);
		res.values.push_back(kv.second);
	}
	res.finalize();
	printf("{\"points\":[");
	for (size_t i = 0; i < res.keys.size(); i++) {
		printf("%s{\"metric\":%d,\"cols\":[", i ? "," : "", res.metric[i]);
		for (int j = 0; j < res.ncols[res.metric[i]]; j++) {
			const dng_result::Cell &c = res.cells[res.cell0[i] + j];
			if (j)
				printf(",");
			if (c.is_number) {
				uint64_t b;
				memcpy(&b, &c.num, 8);
				printf("{\"n\":\"%016llx\"}",
				    (unsigned long long)b);
			} else {
				printf("{\"s\":\"");
				for (size_t x = 0; x < c.len; x++)
					printf("%02x", (unsigned char)
					    res.keys[i][c.off + x]);
				printf("\"}");
			}
		}
		printf("],\"value\":%llu}", (unsigned long long)res.values[i]);
	}
	printf("],\"counters\":{");
#define CTR(n) printf("\"" #n "\":%u,", C.n)
	CTR(lines); CTR(invalid_json); CTR(invalid_point); CTR(ds_filtered);
	CTR(ds_failedeval); CTR(user_filtered); CTR(user_failedeval);
	CTR(synth_undef); CTR(synth_baddate); CTR(time_filtered);
	CTR(time_failedeval); CTR(aggr); CTR(slow);
	printf("\"unsupported\":%u},\"mcounters\":[", C.unsupported);
	for (u32 mi = 1; mi < plan.dev.nmetrics; mi++) {
		const LocalCounters &M = MCs[mi];
		printf("%s{\"user_filtered\":%u,\"user_failedeval\":%u,"
		    "\"synth_undef\":%u,\"synth_baddate\":%u,"
		    "\"time_filtered\":%u,\"time_failedeval\":%u,\"aggr\":%u}",
		    mi > 1 ? "," : "", M.user_filtered, M.user_failedeval,
		    M.synth_undef, M.synth_baddate, M.time_filtered,
		    M.time_failedeval, M.aggr);
		C.unsupported += M.unsupported;
	}
	printf("],\"nfast\":%lu,\"ntmpl\":%lu,\"nfmatch\":%lu,\"nfmiss\":%lu}\n",
	    nfast, ntmpl, nf_match, nf_miss);
	return 0;
}
