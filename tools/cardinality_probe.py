"""F kernel tally-cache adaptivity: a query with many keys (-b req.url,host) and
one with few, with the CTA's warps forced (DNG_F_WARPS=28|24) or chosen by the
library.  One device buffer per scan."""
import ctypes, os, sys, time
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, 'tests'))
import torch
from dragnet_b200 import native, datasource_gpu
import corpus
os.environ.setdefault('DNG_JIT', 'sync')
n = int(sys.argv[1]) if len(sys.argv) > 1 else 8000000
params = native.gen_params(total_records=n)
cap = n * 232
buf = torch.empty(cap, dtype=torch.uint8, device='cuda:0')
ln = ctypes.c_size_t()
native.lib().dng_gen_device(ctypes.byref(params), 0, 0, n, buf.data_ptr(), cap, ctypes.byref(ln))
torch.cuda.synchronize()
for argv in (['-b', 'req.method'], ['-b', 'req.url,host'], ['-b', 'operation,req.method,host']):
    plan = corpus.make_plan(argv)
    ref = None
    for warps in ('28', '24', None):
        if warps: os.environ['DNG_F_WARPS'] = warps
        else: os.environ.pop('DNG_F_WARPS', None)
        for rep in range(2):
            r = datasource_gpu.run_plan(plan, device_buffers=[(buf.data_ptr(), ln.value)])
        pts = sorted((tuple(v for _, v in f), c) for f, c in r.points)
        if ref is None: ref = pts
        assert pts == ref
        print('%-28s warps=%-5s kernel %.2f ms  %.2f Grec/s  points %d launches %d' % (' '.join(argv), warps, r.stats['kernel_ms'], n / r.stats['kernel_ms'] / 1e6, len(pts), r.stats['launches']), flush=True)
