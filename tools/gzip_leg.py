"""Times scans of gzip files (dng_scan_feed_gzip, inflated on the device)
against scans of the same records as plain files (dng_scan_feed_file).

Generates RECORDS records with dng_gen_host and writes them twice for each K
in --ks: as K gzip files (zlib level 6) and as K plain files.  Then, one fresh
process per sample, alternating plain and gzip, scans each set and checks its
points and counters against the C++ oracle on the plain files.  Reports per
set the median and range of records/s (open to result), and for the gzip sets
the inflate kernel's decompressed GB/s (from inflate_ms: all streams of a
batch at once; K = 1 is one stream, one warp), the compression ratio and the
gzip stats.  The first line names the GPU and its power limit.

    python tools/gzip_leg.py [--records 8000000] [--ks 1,8,256] [--pairs 3]
        [--dir DIR] [--out FILE]
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
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

PLAN = {'format': 'json', 'ds_filter': None,
        'filter': {'ne': ['req.method', 'HEAD']}, 'synthetic': [],
        'time_bounds': None,
        'breakdowns': [{'name': 'req.method', 'field': 'req.method'},
                       {'name': 'res.statusCode', 'field': 'res.statusCode'},
                       {'name': 'host', 'field': 'host'}]}


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit',
                               '--format=csv,noheader'], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ''


def sample(kind, files):
    """one scan in this process: (seconds, points, counters, stats)"""
    from dragnet_b200 import datasource_gpu
    t0 = time.perf_counter()
    r = datasource_gpu.run_plan(PLAN, files=files,
                                compression='gzip' if kind == 'gzip' else None)
    dt = time.perf_counter() - t0
    return dt, r.points, r.counters, r.stats


def child(args):
    kind, listfile, out = args
    with open(listfile) as f:
        files = json.load(f)
    dt, pts, ctr, st = sample(kind, files)
    from engines import canon_points
    with open(out, 'w') as f:
        json.dump({'s': dt, 'points': repr(canon_points(pts)),
                   'counters': ctr, 'stats': st}, f)


def write_sets(d, records, k):
    from dragnet_b200 import native
    params = native.gen_params(total_records=records)
    plain, gz = [], []
    per = (records + k - 1) // k
    raw = comp = 0
    for i in range(k):
        first = i * per
        n = min(per, records - first)
        data = native.gen_host(params, first, n)
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
        return child(sys.argv[2:])
    ap = argparse.ArgumentParser()
    ap.add_argument('--records', type=int, default=8000000)
    ap.add_argument('--ks', default='1,8,256')
    ap.add_argument('--pairs', type=int, default=3)
    ap.add_argument('--dir', default=None)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from engines import canon_points, cpp_engine
    info = gpu_info()
    if not info:
        sys.exit('no GPU (nvidia-smi): nothing is measured')
    print('gpu: %s' % info)
    d = tempfile.mkdtemp(prefix='dng-gzip-', dir=a.dir)
    rows = []
    try:
        for k in [int(x) for x in a.ks.split(',')]:
            plain, gz, raw, comp = write_sets(d, a.records, k)
            exp_p, exp_c = cpp_engine(PLAN, plain,
                                      threads=os.cpu_count() or 1)
            exp_p = repr(canon_points(exp_p))
            lists = {}
            for kind, files in (('plain', plain), ('gzip', gz)):
                lists[kind] = os.path.join(d, '%s-%d.json' % (kind, k))
                with open(lists[kind], 'w') as f:
                    json.dump(files, f)
            got = {'plain': [], 'gzip': []}
            for _ in range(a.pairs):
                for kind in ('plain', 'gzip'):
                    out = os.path.join(d, 'out.json')
                    subprocess.check_call([sys.executable, __file__,
                                           '--child', kind, lists[kind],
                                           out])
                    with open(out) as f:
                        r = json.load(f)
                    if r['points'] != exp_p or r['counters'] != exp_c:
                        sys.exit('%s K=%d: result differs from the oracle'
                                 % (kind, k))
                    got[kind].append(r)
            for kind in ('plain', 'gzip'):
                rs = sorted(a.records / r['s'] for r in got[kind])
                row = {'k': k, 'set': kind, 'records': a.records,
                       'raw_bytes': raw, 'gz_bytes': comp,
                       'ratio': round(raw / comp, 2),
                       'mrec_s_median': round(statistics.median(rs) / 1e6, 1),
                       'mrec_s_range': [round(rs[0] / 1e6, 1),
                                        round(rs[-1] / 1e6, 1)]}
                if kind == 'gzip':
                    ms = sorted(r['stats']['inflate_ms'] for r in got[kind])
                    row['inflate_ms_median'] = round(statistics.median(ms), 1)
                    row['inflate_gb_s'] = round(
                        raw / (statistics.median(ms) * 1e6), 2)
                    row['gzip_stats'] = {x: got[kind][-1]['stats'][x] for x in
                                         ('gzip_files', 'gzip_members',
                                          'gzip_compressed_bytes',
                                          'gzip_inflated_bytes')}
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
