#!/usr/bin/env python
"""Time `dn build --interval=hour` on the GPU: DatasourceGpu.build over
generated records, split into the fan-out scan (raw data -> points, on the
GPU) and the sqlite writes (points -> one index file per hour, on the host).

The records come from the library's seeded generator (native.gen_host), spread
evenly over --hours hours, and sit in a tmpfs file (/dev/shm when there is
one) so that the disk is not what is timed.  Each timed build writes a fresh
index directory.  Prints one JSON line; the card's name and power limit are
read in the same run.

  python tools/bench_build.py --rows 10000000 --hours 24 --steps 5 --warmup 1
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

from dragnet_b200 import datasource_gpu, native  # noqa: E402

T0_MS = 1401580800000       # 2014-06-01T00:00:00Z

# an index like the reference's own (tests/dn/local/tst.index_fileset.sh):
# per-minute counts, and a wide breakdown with a latency histogram
METRICS = [
    {'name': 'byminute', 'filter': None,
     'breakdowns': [{'name': 'timestamp', 'field': 'time', 'date': '',
                     'aggr': 'lquantize', 'step': 60}]},
    {'name': 'wide', 'filter': None,
     'breakdowns': [{'name': 'host', 'field': 'host'},
                    {'name': 'operation', 'field': 'operation'},
                    {'name': 'req.method', 'field': 'req.method'},
                    {'name': 'latency', 'field': 'latency',
                     'aggr': 'quantize'}]},
    {'name': 'errors', 'filter': {'ge': ['res.statusCode', 500]},
     'breakdowns': [{'name': 'operation', 'field': 'operation'},
                    {'name': 'host', 'field': 'host'}]},
]


def card():
    out = subprocess.run(
        ['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader',
         '-i', '0'], capture_output=True, text=True, check=True).stdout
    name, power = [x.strip() for x in out.strip().split('\n')[0].split(',')]
    return {'gpu': name, 'power_limit': power}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--rows', type=int, default=10000000)
    ap.add_argument('--hours', type=int, default=24)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()

    base = '/dev/shm' if os.path.isdir('/dev/shm') else None
    work = tempfile.mkdtemp(prefix='dng_bench_build_', dir=base)
    try:
        data = os.path.join(work, 'input.log')
        params = native.gen_params(
            total_records=args.rows, time_min_ms=T0_MS,
            time_max_ms=T0_MS + args.hours * 3600000 - 1)
        step = 1000000
        with open(data, 'wb') as f:
            for first in range(0, args.rows, step):
                f.write(native.gen_host(params, first,
                                        min(step, args.rows - first)))
        nbytes = os.path.getsize(data)

        runs = []
        for i in range(args.warmup + args.steps):
            idx = os.path.join(work, 'index')
            shutil.rmtree(idx, ignore_errors=True)
            ds = datasource_gpu.createDatasource({
                'dsconfig': {'path': data, 'timeField': 'time',
                             'indexPath': idx},
                'findFiles': lambda root, *_: [root]})
            t = time.perf_counter()
            res = ds.build({'metrics': METRICS, 'interval': 'hour',
                            'dryRun': False})
            wall = time.perf_counter() - t
            if isinstance(res, Exception):
                raise res
            if i >= args.warmup:
                runs.append({'wall_s': wall, 'scan_s': res.timing['scan_s'],
                             'index_s': res.timing['index_s'],
                             'files': len(res.index_files),
                             'points': len(res.points)})

        def med(k):
            return statistics.median(r[k] for r in runs)
        out = dict(card(), rows=args.rows, input_bytes=nbytes,
                   hours=args.hours, metrics=len(METRICS),
                   steps=args.steps, warmup=args.warmup,
                   files=runs[-1]['files'], points=runs[-1]['points'],
                   wall_s_median=med('wall_s'), scan_s_median=med('scan_s'),
                   index_s_median=med('index_s'),
                   scan_s_min=min(r['scan_s'] for r in runs),
                   index_s_min=min(r['index_s'] for r in runs),
                   index_share_median=statistics.median(
                       r['index_s'] / r['wall_s'] for r in runs))
        print(json.dumps(out, sort_keys=True))
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == '__main__':
    sys.exit(main())
