"""Times the file leg of a scan spread over several devices
(dng_scan_open_devices): one generated NDJSON file on tmpfs, scanned with
devices = [0] * k for each k asked for and, when the machine has more than one
GPU, with distinct devices.  Prints one JSON line per configuration: wall
time from the first feed to the merged result (open excluded), records/s,
GB/s, and parity with a single-device scan of the same file (points and
counters exact).  The first line names the GPU, its power limit and the
reader-thread setting, which are part of the numbers.

    python tools/multi_device_file_leg.py [--records N] [--shards 1,2,3,4]
        [--repeat R] [--total-threads N] [--out FILE]

DNG_READ_THREADS is per shard; --total-threads N sets it to N // k for a scan
of k shards instead (N for the single-device scan), to compare a fixed total
of reader threads with one that grows with the shards.
"""

import argparse
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
from dragnet_b200 import native  # noqa: E402

PLAN = {'format': 'json', 'ds_filter': None,
        'filter': {'ne': ['req.method', 'HEAD']}, 'synthetic': [],
        'time_bounds': None,
        'breakdowns': [{'name': 'req.method', 'field': 'req.method'},
                       {'name': 'res.statusCode', 'field': 'res.statusCode'},
                       {'name': 'host', 'field': 'host'}]}


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit',
                              '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out.split('\n')
    except (OSError, subprocess.SubprocessError):
        return []


def scan(plan, path, devices):
    """-> (seconds from first feed to result, points, counters)"""
    s = native.Scan(plan, devices=devices) if len(devices) > 1 else \
        native.Scan(plan, devices[0])
    try:
        t0 = time.perf_counter()
        s.feed_file(path)
        r = s.finish()
        dt = time.perf_counter() - t0
        pts = sorted(r.points(), key=repr)
        r.close()
        return dt, pts, s.counters()
    finally:
        s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--records', type=int, default=8000000)
    ap.add_argument('--shards', default='1,2,3,4')
    ap.add_argument('--repeat', type=int, default=3)
    ap.add_argument('--total-threads', type=int, default=0)
    ap.add_argument('--out', default=None, help='also append the lines here')
    args = ap.parse_args()
    ndev = native.lib().dng_device_count()
    if ndev < 1:
        sys.exit('no CUDA device: nothing to measure')
    d = tempfile.mkdtemp(dir='/dev/shm' if os.path.isdir('/dev/shm')
                         else None)
    lines = []

    def emit(doc):
        line = json.dumps(doc, sort_keys=True)
        print(line, flush=True)
        lines.append(line)
    try:
        path = os.path.join(d, 'gen.log')
        params = native.gen_params(total_records=args.records)
        step = 500000
        with open(path, 'wb') as f:
            for first in range(0, args.records, step):
                f.write(native.gen_host(params, first,
                                        min(step, args.records - first)))
        size = os.path.getsize(path)
        emit({'gpus': gpu_info(), 'device_count': ndev,
              'DNG_READ_THREADS': os.environ.get('DNG_READ_THREADS',
                                                 '16 (default)'),
              'cpus': len(os.sched_getaffinity(0)), 'records': args.records,
              'file_bytes': size, 'file_dir': d})
        plan = native.Plan(json.dumps(PLAN))
        scan(plan, path, [0])                   # warm-up: contexts, caches
        _, ref_p, ref_c = scan(plan, path, [0])
        configs = [[0] * int(k) for k in args.shards.split(',')]
        if ndev > 1:
            configs += [list(range(n)) for n in range(2, ndev + 1)]
        for devs in configs:
            if args.total_threads:
                os.environ['DNG_READ_THREADS'] = str(
                    max(1, args.total_threads // len(devs)))
            scan(plan, path, devs)              # warm-up of this shape
            ts, ok = [], True
            for _ in range(args.repeat):
                dt, p, c = scan(plan, path, devs)
                ts.append(dt)
                ok = ok and p == ref_p and c == ref_c
            med = statistics.median(ts)
            emit({'devices': devs, 'seconds_median': med,
                  'read_threads_per_shard': int(os.environ.get(
                      'DNG_READ_THREADS', 16)),
                  'seconds_min': min(ts), 'records_per_s': args.records / med,
                  'gb_per_s': size / 1e9 / med,
                  'parity': 'exact' if ok else 'MISMATCH'})
        plan.close()
    finally:
        shutil.rmtree(d, ignore_errors=True)
        if args.out:
            with open(args.out, 'a') as f:
                f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
