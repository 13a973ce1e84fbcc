"""Record passes of the F kernel per segment, counted on the CPU with the
kernel's framing rule (fast_kernel.cuh) over the head of the bench's input
(oracle/gen_ndjson, the bench's seed, 100 M rows): one window per pass, each
from the first record not yet taken, 32 records at most.  Prints, as JSON, the
lane slice the sample picks and, for windows of nsl + 1 units (28 warps) and
nsl + 2 units (24 warps, the default), the passes per full segment and the
lanes with a record per pass, next to one pass per chunk (the old rule).

    python tools/f_passes.py [ROWS] [SEG]
"""
import collections
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(R, 'tests'))
import framing  # noqa: E402

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 2000000
seg = int(sys.argv[2]) if len(sys.argv) > 2 else framing.F_SEG


def window_passes(nl, nbytes, g0, g1, W):
    """Records of each pass over the segment [g0, g1) (a dense window, more
    than F_NLCAP newlines, is one pass of 0)."""
    base = g0 - framing.F_PRE if g0 else 0
    nxt = g0
    out = []
    while True:
        dlen = min(W, nbytes - base)
        hi = min(base + dlen, g1)
        i, j = np.searchsorted(nl, [nxt, hi])
        total = int(j - i)
        if total > framing.F_NLCAP:
            out.append(0)
            nxt = int(nl[j - 1]) + 1
        elif total:
            take = min(total, 32)
            out.append(take)
            nxt = int(nl[i + take - 1]) + 1
        else:
            nxt = base + dlen
        if (total > framing.F_NLCAP or total <= 32) and base + dlen >= g1:
            return out
        base = nxt & ~15


with tempfile.TemporaryDirectory() as d:
    subprocess.check_call(['make', '-s', '-C', os.path.join(R, 'oracle'),
                           'gen_ndjson'])
    path = os.path.join(d, 'head.log')
    subprocess.check_call([os.path.join(R, 'oracle', 'gen_ndjson'), path,
                           str(0xD5A60000), '100000000', '0', str(rows)])
    data = np.fromfile(path, dtype=np.uint8)
nl = np.flatnonzero(data == 10).astype(np.int64)
nbytes = len(data)
lengths = np.diff(np.concatenate(([-1], nl)))      # with the newline
mean = framing.sample_mean(data[:framing.SAMPLE].tobytes())
g = framing.geometry(mean)
nsl, chunk = g['f_nsl'], g['f_chunk']
nseg = nbytes // (seg * chunk)         # full segments only

per_chunk = np.bincount(nl // chunk)
old = -(-per_chunk[:nseg * seg] // 32)
res = {'rows': rows, 'bytes': nbytes, 'mean_line': float(lengths.mean()),
       'line_min': int(lengths.min()), 'line_max': int(lengths.max()),
       'nsl': nsl, 'chunk': chunk, 'seg_chunks': seg, 'segments': nseg,
       'chunk_records': dict(sorted(collections.Counter(
           per_chunk[:nseg * seg].tolist()).items())),
       'one_pass_per_chunk': {
           'passes_per_segment': dict(collections.Counter(
               old.reshape(nseg, seg).sum(axis=1).tolist())),
           'records_per_pass': float(per_chunk[:nseg * seg].sum() /
                                     old.sum())}}
for units in (nsl + 1, nsl + 2):
    W = 512 * units
    hist, recs, passes = collections.Counter(), 0, 0
    for s in range(nseg):
        p = window_passes(nl, nbytes, s * seg * chunk, (s + 1) * seg * chunk,
                          W)
        hist[len(p)] += 1
        recs += sum(p)
        passes += len(p)
    res['window_%d' % W] = {'units_per_lane': units,
                            'passes_per_segment': dict(sorted(hist.items())),
                            'records_per_pass': recs / passes}
print(json.dumps(res, indent=1))
