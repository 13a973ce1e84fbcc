"""Times scans of bzip2 files (dng_scan_feed_bzip2, decoded on the device)
against scans of the same records as plain files and as gzip files.

Generates RECORDS records with dng_gen_host and writes them for each K in
--ks as K plain files, K gzip files (level 6) and K bzip2 files (level 9).
Then, one fresh process per sample, the three kinds alternating, scans each
set and checks its points and counters against the C++ oracle on the plain
files.  Reports per set the median and range of records/s (open to result);
for the bzip2 sets also the decompressed GB/s (decompressed bytes over
bunzip_ms), the milliseconds of each stage's kernels, blocks and false
starts.  The first line names the GPU and its power limit; the last, for
context, bz2.decompress on one core of this host (a host figure).

    python tools/bzip2_leg.py [--records 8000000] [--ks 1,8,256]
        [--samples 5] [--dir DIR] [--out FILE]
"""

import argparse
import bz2
import gzip
import json
import multiprocessing
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
KINDS = ('plain', 'gzip', 'bzip2')


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit',
                               '--format=csv,noheader'], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ''


def child(args):
    kind, listfile, out = args
    with open(listfile) as f:
        files = json.load(f)
    from dragnet_b200 import datasource_gpu, native
    from engines import canon_points
    t0 = time.perf_counter()
    comp = None if kind == 'plain' else kind
    p = native.Plan(json.dumps(PLAN))
    s = native.Scan(p)
    stages = {}
    try:
        for fn in files:
            if kind == 'gzip':
                s.feed_gzip(fn)
            elif kind == 'bzip2':
                s.feed_bzip2(fn)
            else:
                s.feed_file(fn)
        res = s.finish()
        names = [b['name'] for b in PLAN['breakdowns']]
        pts = [(list(zip(names, c)), v) for c, v in res.points()]
        res.close()
        dt = time.perf_counter() - t0
        ctr = datasource_gpu.stage_counters(PLAN, s.counters(), len(pts))
        st = s.bzip2_stats() if comp == 'bzip2' else {}
        if comp == 'bzip2':
            stages = s.bzip2_stage_ms()
    finally:
        s.close()
        p.close()
    with open(out, 'w') as f:
        json.dump({'s': dt, 'points': repr(canon_points(pts)),
                   'counters': ctr, 'stats': st, 'stages': stages}, f)


def _compress(job):
    path, kind = job
    with open(path, 'rb') as f:
        data = f.read()
    if kind == 'gzip':
        z, out = gzip.compress(data, 6), path + '.gz'
    else:
        z, out = bz2.compress(data, 9), path + '.bz2'
    with open(out, 'wb') as f:
        f.write(z)
    return out, len(z)


def write_sets(d, records, k):
    from dragnet_b200 import native
    params = native.gen_params(total_records=records)
    plain = []
    per = (records + k - 1) // k
    raw = 0
    for i in range(k):
        first = i * per
        n = min(per, records - first)
        data = native.gen_host(params, first, n)
        p = os.path.join(d, 'k%d-%04d.log' % (k, i))
        with open(p, 'wb') as f:
            f.write(data)
        plain.append(p)
        raw += len(data)
    jobs = [(p, kind) for kind in ('gzip', 'bzip2') for p in plain]
    with multiprocessing.Pool(os.cpu_count() or 1) as pool:
        done = pool.map(_compress, jobs)
    sets = {'plain': plain, 'gzip': [o for o, _ in done[:k]],
            'bzip2': [o for o, _ in done[k:]]}
    size = {'gzip': sum(n for _, n in done[:k]),
            'bzip2': sum(n for _, n in done[k:]), 'plain': raw}
    return sets, raw, size


def host_bz2_rate(path):
    """bz2.decompress of one file on one core of this host: MB/s"""
    with open(path, 'rb') as f:
        z = f.read()
    t0 = time.perf_counter()
    n = len(bz2.decompress(z))
    return n / (time.perf_counter() - t0) / 1e6


def main():
    if len(sys.argv) > 1 and sys.argv[1] == '--child':
        return child(sys.argv[2:])
    ap = argparse.ArgumentParser()
    ap.add_argument('--records', type=int, default=8000000)
    ap.add_argument('--ks', default='1,8,256')
    ap.add_argument('--samples', type=int, default=5)
    ap.add_argument('--dir', default=None)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from engines import canon_points, cpp_engine
    info = gpu_info()
    if not info:
        sys.exit('no GPU (nvidia-smi): nothing is measured')
    print('gpu: %s' % info, flush=True)
    d = tempfile.mkdtemp(prefix='dng-bzip2-', dir=a.dir)
    rows, host = [], None
    try:
        for k in [int(x) for x in a.ks.split(',')]:
            sets, raw, size = write_sets(d, a.records, k)
            exp_p, exp_c = cpp_engine(PLAN, sets['plain'],
                                      threads=os.cpu_count() or 1)
            exp_p = repr(canon_points(exp_p))
            lists = {}
            for kind in KINDS:
                lists[kind] = os.path.join(d, '%s-%d.json' % (kind, k))
                with open(lists[kind], 'w') as f:
                    json.dump(sets[kind], f)
            got = {kind: [] for kind in KINDS}
            for _ in range(a.samples):
                for kind in KINDS:
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
            for kind in KINDS:
                rs = sorted(a.records / r['s'] for r in got[kind])
                row = {'k': k, 'set': kind, 'records': a.records,
                       'raw_bytes': raw, 'bytes': size[kind],
                       'ratio': round(raw / size[kind], 2),
                       'mrec_s_median': round(statistics.median(rs) / 1e6, 2),
                       'mrec_s_range': [round(rs[0] / 1e6, 2),
                                        round(rs[-1] / 1e6, 2)]}
                if kind == 'bzip2':
                    ms = sorted(r['stats']['bunzip_ms'] for r in got[kind])
                    row['bunzip_ms_median'] = round(statistics.median(ms), 1)
                    row['decompress_gb_s'] = round(
                        raw / (statistics.median(ms) * 1e6), 2)
                    row['stage_ms_median'] = {
                        s: round(statistics.median(r['stages'][s]
                                                   for r in got[kind]), 1)
                        for s in ('find', 'decode', 'invert', 'emit')}
                    last = got[kind][-1]['stats']
                    row['blocks'] = last['bzip2_blocks']
                    row['false_starts'] = last['bzip2_false_starts']
                rows.append(row)
                print(json.dumps(row), flush=True)
            if host is None:
                host = host_bz2_rate(sets['bzip2'][0])
            for kind in KINDS:
                for p in sets[kind]:
                    os.unlink(p)
        print(json.dumps({'host_bz2_decompress_mb_s_one_core':
                          round(host, 1)}), flush=True)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump({'gpu': info, 'rows': rows,
                       'host_bz2_decompress_mb_s_one_core': host}, f,
                      indent=1)


if __name__ == '__main__':
    main()
