"""Times gzip scans with the split path (inflate_split.cuh: a large file in
a batch of few decoded by many warps) against a build without it.

Generates RECORDS records (dng_gen_host) as K gzip files (zlib level 6) for
each K in --ks.  Builds the library again with -DDNG_NO_GZIP_SPLIT
(tools/build_variant.sh nosplit), then, one fresh process per sample,
alternating the default build and that one, scans each set and checks its
points and counters against the C++ oracle on the plain files.  Reports per
set and build the median and range of records/s (open to result), inflate
GB/s of decompressed output from inflate_ms (every inflate kernel, the split
path's included), and the split counters (chunks, false starts, fallbacks).
The first line names the GPU and its power limit.

    python tools/gzip_split_leg.py [--records 8000000] [--ks 1,8,256,4096]
        [--samples 5] [--dir DIR] [--out FILE] [--reuse-variant]
"""

import argparse
import gzip
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, HERE)

import gzip_leg  # noqa: E402

VARIANT = os.path.join(ROOT, 'dragnet_b200', 'libdragnet_gpu_nosplit.so')
SPLIT_KEYS = ('gzip_files', 'gzip_members', 'gzip_split_files', 'gzip_chunks',
              'gzip_false_starts', 'gzip_fallbacks', 'gzip_split_launches',
              'inflate_launches')


def write_sets(d, records, k):
    """K files of RECORDS records in all, plain and gzipped (level 6), as
    even as whole records allow"""
    from dragnet_b200 import native
    params = native.gen_params(total_records=records)
    plain, gz = [], []
    raw = comp = 0
    for i in range(k):
        first = i * records // k
        data = native.gen_host(params, first, (i + 1) * records // k - first)
        p = os.path.join(d, 'k%d-%04d.log' % (k, i))
        with open(p, 'wb') as f:
            f.write(data)
        z = gzip.compress(data, 6)
        with open(p + '.gz', 'wb') as f:
            f.write(z)
        plain.append(p)
        gz.append(p + '.gz')
        raw += len(data)
        comp += len(z)
    return plain, gz, raw, comp


def main():
    if len(sys.argv) > 1 and sys.argv[1] == '--child':
        return gzip_leg.child(sys.argv[2:])
    ap = argparse.ArgumentParser()
    ap.add_argument('--records', type=int, default=8000000)
    ap.add_argument('--ks', default='1,8,256,4096')
    ap.add_argument('--samples', type=int, default=5)
    ap.add_argument('--dir', default=None)
    ap.add_argument('--out', default=None)
    ap.add_argument('--reuse-variant', action='store_true',
                    help='use the nosplit build already made')
    a = ap.parse_args()
    from engines import canon_points, cpp_engine
    info = gzip_leg.gpu_info()
    if not info:
        sys.exit('no GPU (nvidia-smi): nothing is measured')
    print('gpu: %s' % info, flush=True)
    if not (a.reuse_variant and os.path.exists(VARIANT)):
        subprocess.check_call([os.path.join(HERE, 'build_variant.sh'),
                               'nosplit', '-DDNG_NO_GZIP_SPLIT'],
                              stdout=subprocess.DEVNULL)
    builds = (('split', None), ('nosplit', VARIANT))
    d = tempfile.mkdtemp(prefix='dng-gzsplit-', dir=a.dir)
    rows = []
    try:
        for k in [int(x) for x in a.ks.split(',')]:
            plain, gz, raw, comp = write_sets(d, a.records, k)
            exp_p, exp_c = cpp_engine(gzip_leg.PLAN, plain,
                                      threads=os.cpu_count() or 1)
            exp_p = repr(canon_points(exp_p))
            lst = os.path.join(d, 'gzip-%d.json' % k)
            with open(lst, 'w') as f:
                json.dump(gz, f)
            got = {b: [] for b, _ in builds}
            for _ in range(a.samples):
                for b, lib in builds:
                    out = os.path.join(d, 'out.json')
                    env = dict(os.environ)
                    if lib:
                        env['DNG_LIB'] = lib
                    subprocess.check_call([sys.executable, __file__,
                                           '--child', 'gzip', lst, out],
                                          env=env)
                    with open(out) as f:
                        r = json.load(f)
                    if r['points'] != exp_p or r['counters'] != exp_c:
                        sys.exit('%s K=%d: result differs from the oracle'
                                 % (b, k))
                    got[b].append(r)
            for b, _ in builds:
                rs = sorted(a.records / r['s'] for r in got[b])
                gbs = sorted(raw / (r['stats']['inflate_ms'] * 1e6)
                             for r in got[b])
                row = {'k': k, 'build': b, 'records': a.records,
                       'raw_bytes': raw, 'gz_bytes': comp,
                       'mrec_s_median': round(statistics.median(rs) / 1e6, 2),
                       'mrec_s_range': [round(rs[0] / 1e6, 2),
                                        round(rs[-1] / 1e6, 2)],
                       'inflate_gb_s_median': round(statistics.median(gbs), 2),
                       'inflate_gb_s_range': [round(gbs[0], 2),
                                              round(gbs[-1], 2)],
                       'stats': {x: got[b][-1]['stats'].get(x)
                                 for x in SPLIT_KEYS}}
                rows.append(row)
                print(json.dumps(row), flush=True)
            for p in plain + gz:
                os.unlink(p)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump({'gpu': info, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
