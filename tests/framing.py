"""Record framing at the staging boundaries of the scan kernels: their
geometry restated from the headers, and inputs whose newlines sit at chosen
offsets from those boundaries.

Every kernel stages its input in units and frames records across them:

  F kernel     chunks of 512 x nsl bytes behind a DNG_F_PRE pre-lap, at most
               DNG_F_NLCAP newline positions per chunk, segments of up to
               DNG_F_SEG chunks (fast_kernel.cuh, api.cu launch_fscan)
  per-warp     chunks of 32 x wslice bytes behind a DNG_W_PRELAP pre-lap,
               DNG_W_NLCAP newline positions per pass (scan_kernel_w)
  CTA tiles    DNG_TILE bytes behind a DNG_PRELAP pre-lap, DNG_NLCAP newline
               positions per pass (scan_kernel)

A launch over a 16-byte aligned device buffer with no carry starts its unit k
at byte k x U of the buffer, so a layout built for U puts its cases exactly on
the boundaries the kernel sees.  Tests: test_framing_host.py (no GPU),
test_gpu_framing.py."""

import math
import os
import random
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')

_HEADERS = ('scan_kernel.cuh', 'kernel_choice.h', 'fast_kernel.cuh', 'fast.h',
            'tmpl.h')
NAMES = ('DNG_NT', 'DNG_TILE', 'DNG_PRELAP', 'DNG_NLCAP', 'DNG_MAXREC',
         'DNG_W_PRELAP', 'DNG_W_NLCAP', 'DNG_W_SLICE_MAX', 'DNG_F_NLCAP',
         'DNG_F_NW_START', 'DNG_F_PRE', 'DNG_F_SEG', 'F_MAXLINE',
         'TMPL_SAMPLE_BYTES')


def header_constants():
    """The framing constants as the headers define them (#define NAME expr,
    or NAME = expr in an enum), expressions evaluated in terms of each
    other."""
    raw = {}
    for h in _HEADERS:
        with open(os.path.join(CSRC, h)) as f:
            text = re.sub(r'/\*.*?\*/', ' ', f.read(), flags=re.S)
        for name in NAMES:
            m = re.search(r'^\s*#define\s+%s\s+(.+?)\s*$' % name, text, re.M) \
                or re.search(r'\b%s\s*=\s*([^,}\n]+)' % name, text)
            if m and name not in raw:
                raw[name] = re.sub(r'\b(\d+)u\b', r'\1', m.group(1)).strip()
    missing = [n for n in NAMES if n not in raw]
    if missing:
        raise KeyError('constants not found in %s: %s' % (_HEADERS, missing))
    out = {}
    while len(out) < len(raw):
        for name, expr in raw.items():
            if name in out:
                continue
            try:
                out[name] = int(eval(expr, {'__builtins__': {}}, dict(out)))
            except NameError:
                pass
    return out


C = header_constants()
F_PRE, W_PRELAP, PRELAP = C['DNG_F_PRE'], C['DNG_W_PRELAP'], C['DNG_PRELAP']
F_NLCAP, W_NLCAP, NLCAP = C['DNG_F_NLCAP'], C['DNG_W_NLCAP'], C['DNG_NLCAP']
F_MAXLINE, MAXREC, F_SEG = C['F_MAXLINE'], C['DNG_MAXREC'], C['DNG_F_SEG']
SAMPLE = C['TMPL_SAMPLE_BYTES']
TILE = C['DNG_TILE']
F_WARPS = C['DNG_F_NW_START']           # warps per CTA a scan launches with


# -- geometry ------------------------------------------------------------------

def lane_slice(mean, cap):
    """kernel_choice.h kc_lane_slice: bytes per lane slice for lines of this
    mean length, at most `cap` records per chunk with a quarter to spare."""
    best, pick = -1.0, 112
    for sl in range(112, C['DNG_W_SLICE_MAX'] + 1, 32):
        recs = 32.0 * sl / mean
        passes = math.ceil((recs + 1.5) / 32.0)
        util = recs / (32.0 * passes)
        if recs * 1.25 <= cap and util >= best:
            best, pick = util, sl
    return pick


def sample_mean(launch):
    """kc_sample's mean line over the head of a launch's bytes (from its
    first valid byte): TMPL_SAMPLE_BYTES at most, 224 without a newline."""
    head = launch[:SAMPLE]
    nl = head.count(b'\n')
    return len(head) / nl if nl else 224.0


def geometry(mean):
    """{'wslice', 'f_nsl', 'f_chunk', 'w_chunk', 'tile'} for a sample mean."""
    wslice = lane_slice(mean, math.inf)
    nsl = lane_slice(mean, F_NLCAP) // 16
    return {'wslice': wslice, 'f_nsl': nsl, 'f_chunk': 32 * 16 * nsl,
            'w_chunk': 32 * wslice, 'tile': TILE}


def f_segment(nbytes, f_chunk, sm_count, warps=F_WARPS):
    """api.cu launch_fscan: chunks per segment of a launch over nbytes (from
    its 16-byte aligned base)."""
    nchunks = -(-nbytes // f_chunk)
    grid = min(-(-nchunks // warps), sm_count)
    return max(1, min(F_SEG, nchunks // (grid * warps * 8)))


def f_bytes_for_segment(seg, f_chunk, sm_count, warps=F_WARPS):
    """The fewest bytes whose launch runs segments of `seg` chunks (seg > 1:
    the grid is full, so the chunk count alone decides)."""
    return seg * sm_count * warps * 8 * f_chunk


KERNEL_UNIT = {'fast': ('f_chunk', F_PRE, F_NLCAP),
               'warp': ('w_chunk', W_PRELAP, W_NLCAP),
               'tile': ('tile', PRELAP, NLCAP)}


# -- records -------------------------------------------------------------------

WORDS = [b'alpha', b'b', b'gamma', b'de', b'epsilon-zeta']
MINREC = 48             # a filler record no shorter (ids below 10^7)


def _pad(rng, n, utf8=True):
    """n bytes of string content, valid UTF-8 with some multi-byte
    characters (their lead bytes are >= 0xc2: never a newline, but some sit
    next to the SWAR test's borrow)."""
    out = bytearray()
    while len(out) < n:
        left = n - len(out)
        r = rng.random()
        if utf8 and r < 0.04 and left >= 3:
            out += '€'.encode()
        elif utf8 and r < 0.08 and left >= 2:
            out += 'é'.encode()
        else:
            out.append(rng.choice(b'abcdefghijklmnopqrstuvwxyz0123456789 '))
    return bytes(out)


def _head(i):
    return b'{"id":%d,"g":%d,"k":"%s","p":"' % (i, i % 997, WORDS[i % 5])


class Layout(object):
    """An input built record by record.  Every record carries `id` (and `g` =
    id % 997) so that a result grouped by them names a lost or doubled
    record.  `cases` lists (kind, boundary, detail) of what was placed."""

    def __init__(self, seed, first_id=0):
        self.rng = random.Random(seed)
        self.buf = bytearray()
        self.id = first_id
        self.cases = []

    def _next(self):
        self.id += 1
        return self.id

    def record(self, length, pad=None, tail=b''):
        """One templated record of exactly `length` bytes with its
        newline."""
        i = self._next()
        h = _head(i)
        n = length - 1 - len(h) - 2 - len(tail)
        if n < 0:
            raise ValueError('record of %d bytes is too short' % length)
        body = pad(n) if pad else _pad(self.rng, n)
        line = h + body + b'"}' + tail + b'\n'
        assert len(line) == length
        self.buf += line

    def filler(self):
        self.record(self.rng.randint(MINREC, MINREC + 40))

    def fill_to(self, t):
        """Records up to byte t: the last one's newline at t - 1."""
        d = t - len(self.buf)
        if d == 0:
            return
        if d < MINREC:
            raise ValueError('no room for a record before %d' % t)
        while d > 2 * (MINREC + 40):
            self.filler()
            d = t - len(self.buf)
        if d > MINREC + 80:
            self.record(d // 2)
            d = t - len(self.buf)
        self.record(d)

    def special_at(self, t, kind):
        """A record with a byte the SWAR newline test may flag at byte t:
        'tab' / 'cr' (JSON whitespace after the object: valid), 'ctl' (a raw
        0x00-0x09 inside a string: invalid JSON), 'utf8' (a multi-byte
        character starting there)."""
        if kind in ('tab', 'cr'):
            # the whitespace run starts at t: body ends at t - 1
            ws = b'\t \r' if kind == 'tab' else b'\r'
            i = len(self.buf)
            self.record(t - i + len(ws) + 1, tail=ws)
            return
        i = len(self.buf)
        a = t - i - len(_head(self.id + 1))
        assert a >= 0
        ch = {'ctl': bytes([self.rng.choice([0, 1, 8, 9])]),
              'utf8': self.rng.choice(['é', '€',
                                       '\U0001f600']).encode()}[kind]
        extra = self.rng.randint(4, 30)
        self.record(len(_head(self.id + 1)) + a + len(ch) + extra + 3,
                    pad=lambda n: b'q' * a + ch + b'r' * (n - a - len(ch)))

    def tiny(self, n):
        """n lines of 1-3 bytes: empty, `{}`, ` `."""
        for _ in range(n):
            self.buf += self.rng.choice([b'\n', b'{}\n', b' \n'])

    def lines_in(self, start, end, n):
        """Exactly n records from byte start to byte end (the last newline at
        end - 1), as even as MINREC allows: the rest as tiny lines."""
        assert len(self.buf) == start
        u = end - start
        t = 0
        if u < n * MINREC:
            t = -(-(n * MINREC - u) // (MINREC - 3))
            if t > n - 1:
                t = n - 1
        full = n - t
        # tiny lines are 1-3 bytes: place them first, then share the rest
        self.tiny(t)
        rest = end - len(self.buf)
        for k in range(full):
            left = full - k
            ln = rest // left
            self.record(ln)
            rest -= ln
        assert len(self.buf) == end, (len(self.buf), end)

    def data(self):
        return bytes(self.buf)


def _cases(U, P, K):
    """(name, lead, fn(layout, b)) for boundary b: lead = how far before b
    the case's first record may end."""
    cs = []
    for d in (-1, 0, 1):
        cs.append(('nl%+d' % d, 1,
                   lambda L, b, d=d: L.fill_to(b + d + 1)))
    for h in (P - 1, P, P + 1, 1, 15, 16, 17):
        def head(L, b, h=h):
            L.fill_to(b - h)
            L.record(h + L.rng.randint(MINREC, 300))
        cs.append(('head%d' % h, h, head))
    for n in (767, 768, 769, 4095, 4096, 4097):
        # a line of n bytes before its newline, its start and end near b
        for where in ('ends', 'starts'):
            def longline(L, b, n=n, where=where):
                if where == 'ends':
                    L.fill_to(b - n + L.rng.choice([0, 1, 2, 37]) - 1)
                else:
                    L.fill_to(b - L.rng.choice([0, 1, 17, 511]))
                L.record(n + 1)
            cs.append(('len%d%s' % (n, where), n + 512, longline))
    for k in (2, 3):
        def span(L, b, k=k):
            L.fill_to(b - L.rng.randint(1, 200))
            L.record(k * U + 200 + L.rng.randint(1, 300))
        cs.append(('span%d' % k, 200, span))
    for n in (K, K + 1):
        for first in (0, 1):
            # n newlines in [b, b + U); first=1: one of them at b
            def dense(L, b, n=n, first=first):
                L.fill_to(b + first)
                L.lines_in(b + first, b + U, n - first)
            cs.append(('nl%d_%s' % (n, 'at_b' if first else 'after'), 0,
                       dense))
    for kind in ('tab', 'cr', 'ctl', 'utf8'):
        for d in (-1, 0, 1):
            def sp(L, b, kind=kind, d=d):
                L.fill_to(b + d - 70)
                L.special_at(b + d, kind)
            cs.append(('%s%+d' % (kind, d), 71, sp))
    return cs


def build_layout(U, P, K, seed=0, rounds=1, first_id=0, unterminated=True):
    """A layout for units of U bytes, pre-lap P and newline cap K: each case
    of _cases on its own unit boundary (some units are left between cases to
    cool down), `rounds` times, then filler to the next boundary and, if
    asked, an unterminated final line."""
    L = Layout(seed, first_id)
    cs = _cases(U, P, K)
    b = U
    for _ in range(rounds):
        order = list(cs)
        L.rng.shuffle(order)
        for name, lead, fn in order:
            while len(L.buf) + MINREC > b - lead:
                b += U
            fn(L, b)
            L.cases.append((name, b))
            b += U
    L.fill_to(b + L.rng.randint(MINREC, 200))
    if unterminated:
        L.buf += _head(L._next()) + b'end"}'
    return L


def fixed_layout(kernel, seed=0, rounds=1, unterminated=True):
    """The layout whose units are exactly the kernel's: for the F and
    per-warp kernels the unit depends on the mean line of the head of the
    launch, which depends on the layout, so it is built until the two agree.
    Returns (layout, geometry, unit)."""
    key, P, K = KERNEL_UNIT[kernel]
    U = TILE if kernel == 'tile' else 32 * 16 * 7
    for _ in range(6):
        L = build_layout(U, P, K, seed=seed, rounds=rounds,
                         unterminated=unterminated)
        data = L.data()
        last = data.rfind(b'\n') + 1
        g = geometry(sample_mean(data[:last]))
        if g[key] == U:
            return L, g, U
        U = g[key]
    raise RuntimeError('no fixed point for the %s layout' % kernel)


# -- what the kernels count as long --------------------------------------------

def records(data):
    """(begin, end) of every terminated record: end = its newline."""
    a = np.frombuffer(data, dtype=np.uint8)
    nl = np.flatnonzero(a == 10).astype(np.int64)
    beg = np.concatenate(([0], nl[:-1] + 1)) if len(nl) else nl
    return beg, nl


def long_records(beg, end, unit, pre, seg=1, base=0):
    """Records a kernel reaches only from HBM (CTR_LONG): those whose first
    newline-holding segment starts at g0 > 0 while they begin at or before
    g0 - pre.  Positions are relative to the launch's base; seg = units per
    segment (the F kernel's; 1 for the others)."""
    beg = np.asarray(beg, dtype=np.int64) - base
    end = np.asarray(end, dtype=np.int64) - base
    g0 = (end // unit) // seg * seg * unit
    return int(np.count_nonzero((g0 > 0) & (beg <= g0 - pre)))


def host_pieces_long(beg, end, nbytes, unit, pre, ring):
    """long_records of the F kernel when input of nbytes bytes whose records
    are (beg, end) is fed as host pieces of `ring` bytes (api.cu feed_host,
    feed_piece): each piece's complete lines are one launch from the 16-byte
    aligned base before its carried line, with one-chunk segments (a ring
    slot holds far fewer chunks than a segment of two needs)."""
    total, carry_from, off = 0, 0, 0
    while off < nbytes:
        n = min(ring, nbytes - off)
        k = int(np.searchsorted(end, off + n)) - 1
        if k >= 0 and end[k] >= off:
            upto = int(end[k]) + 1
            base = carry_from - (-(off - carry_from) % 16)
            i0 = int(np.searchsorted(end, carry_from))
            total += long_records(beg[i0:k + 1], end[i0:k + 1], unit, pre, 1,
                                  base)
            carry_from = upto
        off += n
    return total


def replicate(beg, end, length, reps):
    """Records of `reps` copies of an input of `length` bytes in a row."""
    offs = np.arange(reps, dtype=np.int64)[:, None] * length
    return (beg[None, :] + offs).ravel(), (end[None, :] + offs).ravel()


def f_block(seed=0, rounds=8):
    """A few MB of F-chunk boundary cases, newline-terminated, its length odd
    mod 16 and not a multiple of the chunk: replicated, every copy meets the
    chunk grid at another phase.  Returns (bytes, geometry)."""
    L, g, U = fixed_layout('fast', seed=seed, rounds=rounds,
                           unterminated=False)
    while len(L.buf) % 2 == 0 or len(L.buf) % U == 0:
        L.record(L.rng.randint(MINREC, MINREC + 40))
    return L.data(), g


def long_line(n, i=1):
    """A templated record of exactly n bytes before its newline."""
    h = _head(i)
    return h + b'L' * (n - len(h) - 2) + b'"}'
