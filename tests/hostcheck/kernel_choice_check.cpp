/*
 * kernel_choice_check: drives the kernel-choice policy
 * (dragnet_b200/csrc/kernel_choice.h) from commands on stdin, one per line,
 * and prints the state after each (TEST ONLY; tests/test_kernel_choice_host.py).
 *
 *   const                                    the policy's constants
 *   open FANOUT MODELLED F_FITS W_FITS KERNEL FAST F_WARPS   ("-": unset)
 *   sample COUNT LEN LONG LEARNED BLOB COVERED LINES
 *       COUNT lines of LEN bytes, then one of LONG bytes when LONG > 0, with
 *       the F templates' facts
 *   live LINES LONG TEMPLATED AGGREGATED OVERFLOWED TEMPLATES
 *   rebase LINES TEMPLATED                   counters after a relearn
 */
#include <stdio.h>
#include <string.h>

#include <string>

#include "kernel_choice.h"

using namespace dng;

static const char *opt(const char *s)
{
	return strcmp(s, "-") ? s : nullptr;
}

int main()
{
	static const char *modes[] = { "auto", "tile", "warp", "fast" };
	static const char *kinds[] = { "tile", "warp", "f" };
	KernelChoice c;
	char cmd[32];
	int relearn = 0;
	while (scanf("%31s", cmd) == 1) {
		if (!strcmp(cmd, "const")) {
			printf("w_maxline=%d w_slice_max=%d f_nlcap=%d f_nw=%d "
			    "f_nw_start=%d\n", DNG_W_MAXLINE, DNG_W_SLICE_MAX,
			    DNG_F_NLCAP, DNG_F_NW, DNG_F_NW_START);
			continue;
		}
		relearn = 0;
		if (!strcmp(cmd, "open")) {
			int fan, mod, ffit, wfit;
			char k[32], f[32], w[32];
			if (scanf("%d %d %d %d %31s %31s %31s", &fan, &mod, &ffit,
			    &wfit, k, f, w) != 7)
				return 2;
			c = KernelChoice();
			kc_open(c, fan, mod, ffit, wfit, opt(k), opt(f), opt(w));
		} else if (!strcmp(cmd, "sample")) {
			size_t count, len, lng, covered, lines;
			int learned, blob;
			if (scanf("%zu %zu %zu %d %d %zu %zu", &count, &len, &lng,
			    &learned, &blob, &covered, &lines) != 7)
				return 2;
			std::string s;
			for (size_t i = 0; i < count; i++)
				s.append(len, 'x').push_back('\n');
			if (lng)
				s.append(lng, 'y').push_back('\n');
			KcTemplates t;
			t.learned = learned;
			t.blob = blob;
			t.covered = covered;
			t.lines = lines;
			kc_sample(c, (const uint8_t *)s.data(), s.size(), t);
		} else if (!strcmp(cmd, "live")) {
			KcLive v;
			int templates;
			if (scanf("%llu %llu %llu %llu %llu %d", &v.lines,
			    &v.long_lines, &v.templated, &v.aggregated,
			    &v.overflowed, &templates) != 6)
				return 2;
			relearn = kc_counters(c, v, templates);
		} else if (!strcmp(cmd, "rebase")) {
			if (scanf("%llu %llu", &c.learn_lines, &c.learn_tmpl) != 2)
				return 2;
		} else {
			return 2;
		}
		printf("mode=%s warp=%d f=%d f_nw=%u wslice=%u f_nsl=%u pick=%s "
		    "relearn=%d relearns=%d sample_tmpl=%d sample_notmpl=%d\n",
		    modes[c.mode], c.warp, c.f, c.f_nw, c.wslice, c.f_nsl,
		    kinds[kc_pick(c)], relearn, c.relearns,
		    kc_wants_sample(c, true), kc_wants_sample(c, false));
	}
	return 0;
}
