/*
 * tmpl.cpp: host side of record templates (tmpl.h): lexical skeletons of a
 * sample of the input, and the trie blob the kernel matches against.  Nothing
 * here parses records for their values: what a template's wildcards mean to
 * the plan is resolved by running the device's own record parser on one sample
 * line per template (api.cu resolve_kernel).
 */
#include <string.h>

#include <algorithm>

#include "tmpl.h"

namespace dng {

static inline bool is_ws(u8 c)
{
	return c == ' ' || c == '\t' || c == '\r' || c == '\n';
}

/*
 * The lexical walk, reporting literal runs and wildcards to a sink:
 *   sink.lit(ptr, len)              a literal run
 *   sink.wild(kind, off, len)       the wildcard that follows it
 */
template <class Sink>
static bool skeleton_walk(const u8 *s, u32 n, Sink &sink)
{
	char stack[64];			/* '{' or '[' per open container */
	u32 depth = 0;
	bool expect_key = false;
	u32 i = 0, lit_start = 0;
	while (i < n) {
		u8 c = s[i];
		if (c == '"') {
			u32 j = i + 1;
			while (j < n && s[j] != '"') {
				if (s[j] == '\\')
					j++;
				j++;
			}
			if (j >= n)
				return false;
			if (depth && stack[depth - 1] == '{' && expect_key) {
				expect_key = false;
				i = j + 1;
				continue;
			}
			sink.lit(s + lit_start, i + 1 - lit_start);
			sink.wild(TK_STR, i + 1, j - (i + 1));
			lit_start = j;
			i = j + 1;
		} else if (c == '{' || c == '[') {
			if (depth >= sizeof (stack))
				return false;
			stack[depth++] = (char)c;
			expect_key = c == '{';
			i++;
		} else if (c == '}' || c == ']') {
			if (!depth || stack[depth - 1] != (c == '}' ? '{' : '['))
				return false;
			depth--;
			expect_key = false;
			i++;
		} else if (c == ',') {
			expect_key = depth && stack[depth - 1] == '{';
			i++;
		} else if (c == ':' || is_ws(c)) {
			i++;
		} else {
			u32 j = i;
			while (j < n && s[j] != ',' && s[j] != ']' && s[j] != '}' &&
			    s[j] != ':' && s[j] != '"' && !is_ws(s[j]))
				j++;
			sink.lit(s + lit_start, i - lit_start);
			sink.wild(TK_BARE, i, j - i);
			lit_start = j;
			i = j;
		}
	}
	if (depth)
		return false;
	sink.lit(s + lit_start, n - lit_start);
	sink.wild(TK_NONE, n, 0);
	return true;
}

namespace {
struct SegSink {
	std::vector<TSeg> &out;
	TSeg cur;
	void lit(const u8 *p, u32 n) { cur.lit.assign((const char *)p, n); }
	void wild(u8 kind, u32 off, u32 len) {
		cur.kind = kind;
		cur.woff = off;
		cur.wlen = len;
		out.push_back(cur);
	}
};
/* bytes that end a bare scalar in skeleton_walk */
struct BareEnd {
	bool t[256];
	BareEnd() {
		for (int c = 0; c < 256; c++)
			t[c] = c == ',' || c == ']' || c == '}' || c == ':' ||
			    c == '"' || is_ws((u8)c);
	}
};
const BareEnd bare_end;

/*
 * Does line s[0, n) have the skeleton `segs`?  The walk's state (open
 * containers, key expected) at any byte depends only on the bytes before it
 * outside wildcards, so a line whose literal runs are those of `segs`, whose
 * wildcards start where the walk would start one and end where the walk would
 * end it, is walked exactly as the line the segments came from: same literal
 * runs, same wildcard kinds, and it is a JSON text exactly when that one was.
 *
 * Starts at segment `k`, whose literal begins at at[k]; records where each
 * later one begins in at[].  Returns segs.size() if the line matches, else the
 * segment that does not (the ones before it do).
 */
size_t skeleton_match(const u8 *s, size_t n, const std::vector<TSeg> &segs,
    size_t k, size_t *at)
{
	size_t i = at[k];
	for (; k < segs.size(); k++) {
		const TSeg &g = segs[k];
		at[k] = i;
		const size_t L = g.lit.size();
		if (n - i < L || memcmp(s + i, g.lit.data(), L) != 0)
			return k;
		i += L;
		if (g.kind == TK_STR) {
			/* after the opening quote (the literal's last byte): the
			 * closing one, escapes skipped as the walk does */
			for (;;) {
				const u8 *q = (const u8 *)memchr(s + i, '"',
				    n - i);
				if (!q)
					return k;
				const u8 *b = (const u8 *)memchr(s + i, '\\',
				    (size_t)(q - (s + i)));
				if (!b) {
					i = (size_t)(q - s);
					break;
				}
				i = (size_t)(b - s) + 2;
				if (i >= n)
					return k;
			}
		} else if (g.kind == TK_BARE) {
			/* the walk takes a bare scalar from any other byte */
			if (i >= n || bare_end.t[s[i]] || s[i] == '{' ||
			    s[i] == '[')
				return k;
			while (i < n && !bare_end.t[s[i]])
				i++;
		} else {
			return i == n ? segs.size() : k;
		}
	}
	return k;
}

/* how many leading segments two skeletons have in common */
size_t common_segs(const std::vector<TSeg> &a, const std::vector<TSeg> &b)
{
	size_t k = 0;
	while (k < a.size() && k < b.size() && a[k].kind == b[k].kind &&
	    a[k].lit == b[k].lit)
		k++;
	return k;
}

}

bool tmpl_skeletonize(const u8 *s, u32 n, std::vector<TSeg> &out)
{
	out.clear();
	SegSink sink{out, TSeg()};
	return skeleton_walk(s, n, sink);
}

void tmpl_candidates(const u8 *data, size_t len, size_t maxk,
    std::vector<TCandidate> &out, size_t *nlines_out)
{
	out.clear();
	if (nlines_out)
		*nlines_out = 0;
	/*
	 * Count lines by skeleton: a line is tried against the shapes already
	 * seen (the last one matched first), and only a line that has none of
	 * them is walked.  Where a shape fails at segment k, the next one goes
	 * on from the segments it shares with that one (up to k), and is passed
	 * over if it shares segment k as well.
	 */
	size_t pos = 0, nlines = 0, last = 0;
	std::vector<TSeg> segs;
	std::vector<std::vector<size_t>> common;	/* common_segs per pair */
	std::vector<size_t> at(TMPL_MAX_LINE + 2);
	while (pos < len && nlines < 8192) {
		const u8 *nl = (const u8 *)memchr(data + pos, '\n', len - pos);
		if (!nl)
			break;
		size_t n = (size_t)(nl - (data + pos));
		const u8 *line = data + pos;
		pos += n + 1;
		nlines++;
		if (n == 0 || n > TMPL_MAX_LINE)
			continue;
		size_t hit = out.size();
		if (!out.empty()) {
			/* the shape tried last, where it failed (at[] holds
			 * where its segments up to that one begin) */
			size_t prev = last;
			at[0] = 0;
			size_t fail = skeleton_match(line, n, out[last].segs, 0,
			    at.data());
			if (fail == out[last].segs.size())
				hit = last;
			for (size_t k = 0; hit == out.size() && k < out.size();
			    k++) {
				const size_t c = common[prev][k];
				if (k == last || c > fail)
					continue;
				fail = skeleton_match(line, n, out[k].segs, c,
				    at.data());
				prev = k;
				if (fail == out[k].segs.size())
					hit = k;
			}
		}
		if (hit < out.size()) {
			out[hit].count++;
			last = hit;
			continue;
		}
		if (out.size() >= 256 || !tmpl_skeletonize(line, (u32)n, segs))
			continue;
		TCandidate c;
		c.sample.assign((const char *)line, n);
		c.segs = segs;
		c.count = 1;
		last = out.size();
		common.emplace_back();
		for (size_t k = 0; k < out.size(); k++) {
			const size_t m = common_segs(out[k].segs, segs);
			common[k].push_back(m);
			common.back().push_back(m);
		}
		common.back().push_back(segs.size());
		out.push_back(c);
	}
	std::stable_sort(out.begin(), out.end(),
	    [](const TCandidate &a, const TCandidate &b) {
		    return a.count > b.count;
	    });
	if (nlines_out)
		*nlines_out = nlines;
	/* shapes seen in under 0.5% of the lines are not worth a trie branch */
	size_t keep = 0;
	while (keep < out.size() && keep < maxk &&
	    (size_t)out[keep].count * 200 >= nlines)
		keep++;
	out.resize(keep);
}

namespace {

struct PSeg {			/* a template segment with its captures */
	std::string lit;
	u8 kind, cap, poscap;
	u16 posoff;
};

struct PTmpl {
	std::vector<PSeg> segs;
	u32 set_mask;
	int want[MAX_SLOTS];	/* segment that must supply each set slot */
};

/* attach the parser's slot values to the candidate's wildcards */
bool plan_template(const TCandidate &c, const TResolved &r, PTmpl &t)
{
	if (r.flags != 0)
		return false;
	t.segs.clear();
	std::vector<u32> start;		/* offset of each literal in the sample */
	u32 pos = 0;
	for (const TSeg &g : c.segs) {
		PSeg p;
		p.lit = g.lit;
		p.kind = g.kind;
		p.cap = p.poscap = 0;
		p.posoff = 0;
		t.segs.push_back(p);
		start.push_back(pos);
		pos = g.woff + g.wlen;
	}
	t.set_mask = r.set_mask;
	for (int s = 0; s < MAX_SLOTS; s++)
		t.want[s] = -1;
	/*
	 * Captured containers: a literal remembers one (at an offset); a second
	 * one in the same literal cuts it, so that it opens a literal of its
	 * own.  In increasing offset order, so that cuts stay behind the
	 * offsets already recorded.
	 */
	std::vector<std::pair<u32, u32>> conts;		/* (offset, slot) */
	for (u32 s = 0; s < MAX_SLOTS; s++) {
		if (!((r.set_mask >> s) & 1))
			continue;
		u64 v = r.slots[s];
		u32 type = (u32)(v >> 56) & 0xf;
		if (type == T_OBJ || type == T_ARR)
			conts.push_back(std::make_pair((u32)v, s));
	}
	std::sort(conts.begin(), conts.end());
	for (auto &c2 : conts) {
		const u32 off = c2.first, slot = c2.second;
		bool found = false;
		for (size_t i = 0; i < t.segs.size() && !found; i++) {
			if (off < start[i] || off >= start[i] + t.segs[i].lit.size())
				continue;
			if (t.segs[i].poscap) {
				u32 d = off - start[i];
				if (d == 0 || d <= t.segs[i].posoff)
					return false;
				PSeg head;
				head.lit = t.segs[i].lit.substr(0, d);
				head.kind = TK_NONE;
				head.cap = 0;
				head.poscap = t.segs[i].poscap;
				head.posoff = t.segs[i].posoff;
				t.segs[i].lit.erase(0, d);
				t.segs[i].poscap = 0;
				t.segs.insert(t.segs.begin() + i, head);
				start.insert(start.begin() + i + 1, off);
				i++;
			}
			char open = t.segs[i].lit[off - start[i]];
			u32 type = (u32)(r.slots[slot] >> 56) & 0xf;
			if (open != (type == T_OBJ ? '{' : '['))
				return false;
			t.segs[i].poscap = (u8)(slot + 1);
			t.segs[i].posoff = (u16)(off - start[i]);
			t.want[slot] = 1;	/* fixed up below */
			found = true;
		}
		if (!found)
			return false;
	}
	for (u32 s = 0; s < MAX_SLOTS; s++) {
		if (!((r.set_mask >> s) & 1))
			continue;
		u64 v = r.slots[s];
		u32 type = (u32)(v >> 56) & 0xf, flags = (u32)(v >> 60) & 0xf;
		u32 off = (u32)v;
		if (flags & VF_INLINE)
			return false;
		if (type == T_OBJ || type == T_ARR)
			continue;		/* placed above */
		bool found = false;
		for (size_t i = 0; i < t.segs.size() && !found; i++) {
			PSeg &g = t.segs[i];
			if (g.kind != (type == T_STR ? TK_STR : TK_BARE) ||
			    start[i] + g.lit.size() != off)
				continue;
			if (g.cap)
				return false;
			g.cap = (u8)(s + 1);
			found = true;
		}
		if (!found)
			return false;
	}
	/* which segment supplies each slot (cuts above moved indexes) */
	for (size_t i = 0; i < t.segs.size(); i++) {
		if (t.segs[i].poscap)
			t.want[t.segs[i].poscap - 1] = (int)i;
		if (t.segs[i].cap)
			t.want[t.segs[i].cap - 1] = (int)i;
	}
	return true;
}

struct BNode {
	std::string lit;
	u8 kind, cap, poscap;
	u16 posoff;
	std::vector<int> kids;
	int leaf;
};

struct Trie {
	std::vector<BNode> nodes;	/* nodes[0] = virtual root */
	std::vector<u32> leaf_mask;
	size_t pool;
	bool compact;		/* literals as plain words (the F path) */

	explicit Trie(bool compact_ = false) : pool(0), compact(compact_) {
		BNode r;
		r.kind = r.cap = r.poscap = 0;
		r.posoff = 0;
		r.leaf = -1;
		nodes.push_back(r);
	}

	bool insert(const PTmpl &t) {
		int cur = 0;
		for (size_t i = 0; i < t.segs.size(); i++) {
			const PSeg &g = t.segs[i];
			int hit = -1;
			for (int k : nodes[cur].kids)
				if (nodes[k].lit == g.lit && nodes[k].kind == g.kind)
					hit = k;
			if (hit < 0) {
				BNode b;
				b.lit = g.lit;
				b.kind = g.kind;
				b.cap = g.cap;
				b.poscap = g.poscap;
				b.posoff = g.posoff;
				b.leaf = -1;
				hit = (int)nodes.size();
				nodes.push_back(b);
				nodes[cur].kids.push_back(hit);
				pool += compact ? (g.lit.size() + 3) / 4 * 4 + 12 :
				    (g.lit.size() + 7) / 8 * 16;
			} else {
				BNode &b = nodes[hit];
				if (g.cap) {
					if (b.cap && b.cap != g.cap)
						return false;
					b.cap = g.cap;
				}
				if (g.poscap) {
					if (b.poscap && (b.poscap != g.poscap ||
					    b.posoff != g.posoff))
						return false;
					b.poscap = g.poscap;
					b.posoff = g.posoff;
				}
			}
			cur = hit;
		}
		if (nodes[cur].leaf >= 0 || !nodes[cur].kids.empty())
			return false;
		nodes[cur].leaf = (int)leaf_mask.size();
		leaf_mask.push_back(t.set_mask);
		/* an interior node may not also end another template */
		for (const BNode &b : nodes)
			if (b.leaf >= 0 && !b.kids.empty())
				return false;
		return true;
	}

	/*
	 * The byte offset at which a sibling group is dispatched: all literals
	 * reach it and it tells the most siblings apart (-1: no dispatch).
	 */
	int disc_offset(const std::vector<int> &kids) const {
		if (kids.size() < 2)
			return -1;
		size_t minl = (size_t)-1;
		for (int k : kids)
			minl = std::min(minl, nodes[k].lit.size());
		int best = -1;
		size_t bestn = 1;
		for (size_t o = 0; o < minl && o < 0xffff; o++) {
			bool seen[256] = { false };
			size_t n = 0;
			for (int k : kids) {
				u8 b = (u8)nodes[k].lit[o];
				if (!seen[b]) {
					seen[b] = true;
					n++;
				}
			}
			if (n > bestn) {
				bestn = n;
				best = (int)o;
			}
		}
		return best;
	}

	/* the siblings the matcher tries, in its order, for a record whose
	 * literal at this place is `lit` */
	std::vector<int> tried(const std::vector<int> &kids,
	    const std::string &lit) const {
		int o = disc_offset(kids);
		if (o < 0)
			return kids;
		std::vector<int> out;
		for (int k : kids)
			if ((size_t)o < lit.size() && nodes[k].lit[o] == lit[o])
				out.push_back(k);
		return out;
	}

	/* does matching t's own shape leave every set slot filled from the
	 * segment the parser took it from? */
	bool verify(const PTmpl &t) const {
		int last[MAX_SLOTS];
		for (int s = 0; s < MAX_SLOTS; s++)
			last[s] = -1;
		int cur = 0;
		for (size_t i = 0; i < t.segs.size(); i++) {
			const PSeg &g = t.segs[i];
			int hit = -1;
			for (int k : tried(nodes[cur].kids, g.lit)) {
				if (nodes[k].lit == g.lit && nodes[k].kind == g.kind) {
					hit = k;
					break;
				}
				/* an earlier wildcard-less sibling whose literal
				 * is a prefix of ours would be taken instead
				 * (the matcher does not backtrack) */
				if (nodes[k].kind == TK_NONE &&
				    nodes[k].lit.size() <= g.lit.size() &&
				    g.lit.compare(0, nodes[k].lit.size(),
				    nodes[k].lit) == 0)
					return false;
			}
			if (hit < 0)
				return false;
			const BNode &b = nodes[hit];
			if (b.poscap)
				last[b.poscap - 1] = (int)i;
			if (b.cap)
				last[b.cap - 1] = (int)i;
			cur = hit;
		}
		if (nodes[cur].leaf < 0 ||
		    leaf_mask[nodes[cur].leaf] != t.set_mask)
			return false;
		for (int s = 0; s < MAX_SLOTS; s++)
			if (((t.set_mask >> s) & 1) && last[s] != t.want[s])
				return false;
		return true;
	}
};

size_t disp_bytes(const Trie &tr)
{
	size_t n = 0;
	for (const BNode &b : tr.nodes)
		if (tr.disc_offset(b.kids) >= 0)
			n += (4 + 4 * b.kids.size() + 15) & ~(size_t)15;
	return n;
}

size_t blob_bytes(const Trie &tr)
{
	size_t nn = tr.nodes.size() - 1 + (tr.nodes[0].kids.size() > 1 ? 1 : 0);
	size_t n = sizeof (THdr) + nn * sizeof (TNode) + 4 * tr.leaf_mask.size();
	n = (n + 15) & ~(size_t)15;
	return ((n + tr.pool + disp_bytes(tr) + 15) & ~(size_t)15);
}

bool build_trie(const std::vector<PTmpl> &ts, Trie &tr, size_t max_bytes)
{
	for (const PTmpl &t : ts)
		if (!tr.insert(t))
			return false;
	for (const PTmpl &t : ts)
		if (!tr.verify(t))
			return false;
	return tr.nodes.size() - 1 <= TMPL_MAX_NODES &&
	    tr.pool + disp_bytes(tr) <= TMPL_MAX_POOL &&
	    tr.leaf_mask.size() <= TMPL_MAX_LEAVES &&
	    blob_bytes(tr) <= max_bytes;
}

} /* namespace */

void tmpl_build(const std::vector<TCandidate> &cands,
    const std::vector<TResolved> &res, size_t max_bytes, std::vector<u8> &blob,
    u32 *ntemplates, bool compact, std::vector<u8> *accepted)
{
	blob.clear();
	if (ntemplates)
		*ntemplates = 0;
	if (accepted)
		accepted->assign(cands.size(), 0);
	std::vector<PTmpl> acc;
	std::vector<size_t> acc_idx;
	for (size_t i = 0; i < cands.size() && i < res.size(); i++) {
		PTmpl t;
		if (!plan_template(cands[i], res[i], t))
			continue;
		acc.push_back(t);
		acc_idx.push_back(i);
		Trie probe(compact);
		if (!build_trie(acc, probe, max_bytes)) {
			acc.pop_back();
			acc_idx.pop_back();
		}
	}
	if (acc.empty())
		return;
	Trie tr(compact);
	if (!build_trie(acc, tr, max_bytes))
		return;
	if (ntemplates)
		*ntemplates = (u32)acc.size();
	if (accepted)
		for (size_t i : acc_idx)
			(*accepted)[i] = 1;

	/* number the nodes: the children of one node are consecutive and
	 * chained through `alt`; the root's first child is node 0 */
	const bool synth_root = tr.nodes[0].kids.size() > 1;
	size_t nn = tr.nodes.size() - 1 + (synth_root ? 1 : 0);
	std::vector<int> index(tr.nodes.size(), -1);
	std::vector<int> order;
	std::vector<int> queue(1, 0);
	if (synth_root) {
		index[0] = 0;		/* the empty node the top-level shapes hang off */
		order.push_back(0);
	}
	for (size_t q = 0; q < queue.size(); q++) {
		for (int k : tr.nodes[queue[q]].kids) {
			index[k] = (int)order.size();
			order.push_back(k);
			queue.push_back(k);
		}
	}
	std::vector<TNode> out(nn);
	if (synth_root) {
		out[0].alt = (u16)TN_NOALT;
		out[0].disp = TN_NODISP;
		out[0].next = (u16)index[tr.nodes[0].kids[0]];
	}
	std::string pool;
	for (size_t q = 0; q < queue.size(); q++) {
		const std::vector<int> &kids = tr.nodes[queue[q]].kids;
		/* dispatch table of this sibling group */
		const int disc = tr.disc_offset(kids);
		u16 disp = TN_NODISP;
		if (disc >= 0) {
			std::vector<u32> ents;
			bool seen[256] = { false };
			for (int k : kids) {
				u8 b = (u8)tr.nodes[k].lit[disc];
				if (!seen[b]) {
					seen[b] = true;
					ents.push_back((u32)b | ((u32)index[k] << 16));
				}
			}
			disp = (u16)(pool.size() / 4);
			u32 head = (u32)disc | ((u32)ents.size() << 16);
			pool.append((const char *)&head, 4);
			pool.append((const char *)ents.data(), 4 * ents.size());
			pool.append((16 - pool.size() % 16) % 16, '\0');
		}
		if (index[queue[q]] >= 0)
			out[index[queue[q]]].disp = disp;
		for (size_t j = 0; j < kids.size(); j++) {
			const BNode &b = tr.nodes[kids[j]];
			TNode &o = out[index[kids[j]]];
			o.lit = (u16)pool.size();
			o.len = (u16)b.lit.size();
			for (size_t k = 0; k < b.lit.size(); k += 4) {
				u32 v = 0, mk = 0;
				for (size_t x = 0; x < 4 && k + x < b.lit.size(); x++) {
					v |= (u32)(u8)b.lit[k + x] << (8 * x);
					mk |= 0xffu << (8 * x);
				}
				pool.append((const char *)&v, 4);
				if (!compact)
					pool.append((const char *)&mk, 4);
			}
			pool.append((16 - pool.size() % 16) % 16, '\0');
			o.kind = b.kind;
			o.cap = b.cap;
			o.poscap = b.poscap;
			o.posoff = b.posoff;
			o.disp = TN_NODISP;	/* filled in when its children are emitted */
			/* next sibling the matcher may try after this one:
			 * with a dispatch table, only one with the same byte */
			o.alt = (u16)TN_NOALT;
			for (size_t x = j + 1; x < kids.size(); x++) {
				if (disc >= 0 && tr.nodes[kids[x]].lit[disc] !=
				    b.lit[disc])
					continue;
				o.alt = (u16)index[kids[x]];
				break;
			}
			o.next = b.leaf >= 0 ? (u16)(TN_LEAF | b.leaf) :
			    (u16)index[b.kids[0]];
		}
	}
	THdr h;
	memset(&h, 0, sizeof (h));
	h.nnodes = (u16)nn;
	h.nleaves = (u16)tr.leaf_mask.size();
	h.leaf_off = (u16)(sizeof (THdr) + nn * sizeof (TNode));
	h.pool_off = (u16)((h.leaf_off + 4 * h.nleaves + 15) & ~15u);
	h.bytes = (u32)((h.pool_off + pool.size() + 15) & ~(size_t)15);
	blob.assign(h.bytes, 0);
	memcpy(blob.data(), &h, sizeof (h));
	memcpy(blob.data() + sizeof (THdr), out.data(), nn * sizeof (TNode));
	memcpy(blob.data() + h.leaf_off, tr.leaf_mask.data(), 4 * h.nleaves);
	memcpy(blob.data() + h.pool_off, pool.data(), pool.size());
}

} /* namespace dng */
