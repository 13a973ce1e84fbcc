/*
 * learn_check: TEST-ONLY host driver of what a scan does on the host before
 * its first launch (api.cu learn_templates): the template candidates, the
 * sample's line statistics, the two trie blobs and the generated matcher
 * source, with the record parser run on the host instead of by
 * resolve_pairs_kernel.  Not part of libdragnet_gpu.so.
 *
 *   learn_check cands FILE MAXK   candidates of FILE's bytes, and those of a
 *                                 plain grouping of its lines by
 *                                 tmpl_skeletonize(), as JSON
 *   learn_check jitkey            which input changes change the JIT cache
 *                                 key, one "name same|differs" per line
 *   learn_check cost PLAN FILE N  each host step of learning from the head
 *                                 of FILE, the fastest of N runs, as JSON
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <fstream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../../dragnet_b200/csrc/record.cuh"
#include "../../dragnet_b200/csrc/kernel_choice.h"
#include "../../dragnet_b200/csrc/jit.h"

using namespace dng;

static std::string slurp(const char *path)
{
	std::ifstream f(path, std::ios::binary);
	std::stringstream ss;
	ss << f.rdbuf();
	return ss.str();
}

static std::string hex(const std::string &s)
{
	static const char d[] = "0123456789abcdef";
	std::string h;
	for (unsigned char c : s) {
		h += d[c >> 4];
		h += d[c & 15];
	}
	return h;
}

/* the definition tmpl_candidates() must agree with: lines grouped by their
 * tmpl_skeletonize() literals and wildcard kinds, first seen first */
static void plain_candidates(const u8 *data, size_t len, size_t maxk,
    std::vector<TCandidate> &out, size_t *nlines_out)
{
	out.clear();
	std::map<std::string, size_t> seen;
	size_t pos = 0, nlines = 0;
	std::vector<TSeg> segs;
	while (pos < len && nlines < 8192) {
		const u8 *nl = (const u8 *)memchr(data + pos, '\n', len - pos);
		if (!nl)
			break;
		size_t n = (size_t)(nl - (data + pos));
		const u8 *line = data + pos;
		pos += n + 1;
		nlines++;
		if (n == 0 || n > TMPL_MAX_LINE ||
		    !tmpl_skeletonize(line, (u32)n, segs))
			continue;
		std::string key;
		for (const TSeg &g : segs) {
			key += std::to_string(g.lit.size()) + ":" + g.lit;
			key += (char)('0' + g.kind);
		}
		auto it = seen.find(key);
		if (it != seen.end()) {
			out[it->second].count++;
			continue;
		}
		if (seen.size() >= 256)
			continue;
		seen[key] = out.size();
		TCandidate c;
		c.sample.assign((const char *)line, n);
		c.segs = segs;
		c.count = 1;
		out.push_back(c);
	}
	std::stable_sort(out.begin(), out.end(),
	    [](const TCandidate &a, const TCandidate &b) {
		    return a.count > b.count;
	    });
	*nlines_out = nlines;
	size_t keep = 0;
	while (keep < out.size() && keep < maxk &&
	    (size_t)out[keep].count * 200 >= nlines)
		keep++;
	out.resize(keep);
}

static void print_cands(const char *name, const std::vector<TCandidate> &cs,
    size_t nlines)
{
	printf("\"%s\": {\"lines\": %zu, \"cands\": [", name, nlines);
	for (size_t i = 0; i < cs.size(); i++) {
		printf("%s{\"count\": %u, \"sample\": \"%s\", \"segs\": [",
		    i ? ", " : "", cs[i].count, hex(cs[i].sample).c_str());
		for (size_t k = 0; k < cs[i].segs.size(); k++) {
			const TSeg &g = cs[i].segs[k];
			printf("%s[\"%s\", %u, %u, %u]", k ? ", " : "",
			    hex(g.lit).c_str(), g.kind, g.woff, g.wlen);
		}
		printf("]}");
	}
	printf("]}");
}

static int cmd_cands(const char *path, size_t maxk)
{
	std::string d = slurp(path);
	std::vector<TCandidate> a, b;
	size_t na = 0, nb = 0;
	tmpl_candidates((const u8 *)d.data(), d.size(), maxk, a, &na);
	plain_candidates((const u8 *)d.data(), d.size(), maxk, b, &nb);
	printf("{");
	print_cands("fast", a, na);
	printf(", ");
	print_cands("plain", b, nb);
	printf("}\n");
	return 0;
}

static int cmd_jitkey()
{
	static FPlan P;
	memset(&P, 0, sizeof (P));
	P.ncols = 1;
	std::vector<u8> blob(256);
	for (size_t i = 0; i < blob.size(); i++)
		blob[i] = (u8)(i * 7);
	unsetenv("DNG_JIT_SHARED");
	const std::string base = jit_key(blob.data(), blob.size(), &P, 13, 0,
	    200000);
	auto report = [&](const char *name, const std::string &k) {
		printf("%s %s\n", name, k == base ? "same" : "differs");
	};
	report("identical", jit_key(blob.data(), blob.size(), &P, 13, 0, 200000));
	std::vector<u8> b2 = blob;
	b2[200] ^= 1;
	report("blob_byte", jit_key(b2.data(), b2.size(), &P, 13, 0, 200000));
	b2 = blob;
	b2.push_back(0);
	report("blob_length", jit_key(b2.data(), b2.size(), &P, 13, 0, 200000));
	static FPlan P2;
	P2 = P;
	P2.pool[100] = 1;
	report("plan_byte", jit_key(blob.data(), blob.size(), &P2, 13, 0, 200000));
	report("no_plan", jit_key(blob.data(), blob.size(), nullptr, 13, 0,
	    200000));
	report("nsl", jit_key(blob.data(), blob.size(), &P, 11, 0, 200000));
	report("device", jit_key(blob.data(), blob.size(), &P, 13, 1, 200000));
	report("smem_max", jit_key(blob.data(), blob.size(), &P, 13, 0, 100000));
	setenv("DNG_JIT_SHARED", "1", 1);
	report("shared_forced", jit_key(blob.data(), blob.size(), &P, 13, 0,
	    200000));
	setenv("DNG_JIT_SHARED", "0", 1);
	report("shared_off", jit_key(blob.data(), blob.size(), &P, 13, 0,
	    200000));
	return 0;
}

static double now_ms()
{
	return std::chrono::duration<double, std::milli>(
	    std::chrono::steady_clock::now().time_since_epoch()).count();
}

/* the fastest of n runs of f, in ms */
template <class F>
static double best_of(int n, F f)
{
	double best = 1e30;
	for (int i = 0; i < n; i++) {
		const double t0 = now_ms();
		f();
		best = std::min(best, now_ms() - t0);
	}
	return best;
}

static int cmd_cost(const char *plan_path, const char *path, int reps)
{
	std::string pj = slurp(plan_path);
	static dng_plan plan;
	char err[256];
	if (dng_plan_compile(pj.c_str(), &plan, err, sizeof (err)) != 0) {
		fprintf(stderr, "plan: %s\n", err);
		return 1;
	}
	std::string d = slurp(path);
	const size_t n = std::min<size_t>(d.size(), TMPL_SAMPLE_BYTES);
	const u8 *p = (const u8 *)d.data();
	std::vector<TCandidate> cands;
	size_t lines = 0;
	const double t_cands = best_of(reps, [&] {
		tmpl_candidates(p, n, TMPL_MAX_LEAVES, cands, &lines);
	});
	/* what resolve_pairs_kernel reports for each candidate's sample */
	std::vector<TResolved> res(cands.size()), fres(cands.size());
	for (size_t i = 0; i < cands.size(); i++) {
		static RecState R;
		parse_record((const u8 *)cands[i].sample.data(),
		    (u32)cands[i].sample.size(), plan.dev, R);
		res[i].flags = R.flags;
		res[i].set_mask = R.set_mask;
		for (int k = 0; k < MAX_SLOTS; k++)
			res[i].slots[k] = ((R.set_mask >> k) & 1) ? R.slots[k] : 0;
	}
	static FPlan F;
	fplan_build(plan.dev, F);
	std::vector<u8> fblob, blob;
	const double t_fblob = best_of(reps, [&] {
		for (size_t i = 0; i < res.size(); i++)
			fplan_resolve(plan.dev, res[i], fres[i]);
		tmpl_build(cands, fres, 4096, fblob, nullptr, true);
	});
	const double t_blob = best_of(reps, [&] {
		tmpl_build(cands, res, 4096, blob, nullptr);
	});
	/* as api.cu uploads (and generates from) it */
	fblob.resize((fblob.size() + 127) & ~(size_t)127, 0);
	KernelChoice kc;
	KcTemplates ft;
	const double t_kc = best_of(reps, [&] { kc_sample(kc, p, n, ft); });
	std::string src;
	const double t_src = best_of(reps, [&] {
		src = jit_source(fblob.data(), fblob.size(), &F);
	});
	std::string key;
	const double t_key = best_of(reps, [&] {
		key = jit_key(fblob.data(), fblob.size(), &F, (int)kc.f_nsl, 0,
		    0);
	});
	unsigned long long h = 1469598103934665603ull;
	for (unsigned char c : src)
		h = (h ^ c) * 1099511628211ull;
	printf("{\"sample_bytes\": %zu, \"lines\": %zu, \"candidates\": %zu, "
	    "\"fblob_bytes\": %zu, \"blob_bytes\": %zu, \"source_bytes\": %zu, "
	    "\"source_fnv1a\": \"%016llx\", \"ms\": {\"tmpl_candidates\": %.4f, "
	    "\"kc_sample\": %.4f, \"f_blob\": %.4f, \"general_blob\": %.4f, "
	    "\"jit_source\": %.4f, \"jit_key\": %.4f}}\n", n, lines,
	    cands.size(), fblob.size(), blob.size(), src.size(), h, t_cands,
	    t_kc, t_fblob, t_blob, t_src, t_key);
	return 0;
}

int main(int argc, char **argv)
{
	if (argc >= 4 && !strcmp(argv[1], "cands"))
		return cmd_cands(argv[2], (size_t)atoi(argv[3]));
	if (argc >= 2 && !strcmp(argv[1], "jitkey"))
		return cmd_jitkey();
	if (argc >= 5 && !strcmp(argv[1], "cost"))
		return cmd_cost(argv[2], argv[3], atoi(argv[4]));
	fprintf(stderr, "usage: learn_check cands FILE MAXK | jitkey | "
	    "cost PLAN FILE N\n");
	return 2;
}
