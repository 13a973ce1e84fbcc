"""Cold start of a scan process with the on-disk kernel cache (dng_jit_cache_dir)
off, cold (an empty directory) and warm (the directory the cold process left),
alternated, one fresh Python process per sample, on the bench's headline query
(-b req.method,res.statusCode -f eq GET) over

  small   the reference's test inputs (tests/golden, ~2 250 records in 9
          files): what one `dn scan` of a small datasource pays;
  file    ~2 GB generated with dng_gen_host into a file (tmpfs when there is
          one), fed with dng_scan_feed_file;
  device  the same bytes generated on the device (dng_gen_device) and fed
          from device memory.

For each process: wall time from spawn to exit, open -> result, open -> the
scan's first kernel launch (seen by a thread polling dng_scan_launch_count,
~0.2 ms resolution), scan launches and how many ran the compiled F kernel,
the cache's counters, and whether libnvrtc / libnvJitLink were mapped.  Every
process's points and counters are checked against the C++ oracle.  One JSON
line per process, then one summary line (medians, min and max per input and
condition) with the card's name and power limit.

    python tools/jit_cold_start.py [--reps 3] [--gb 2] [--jit async]
"""
import argparse
import ctypes
import hashlib
import json
import os
import shutil
import statistics
import subprocess
import sys
import tarfile
import tempfile
import threading
import time

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
sys.path.insert(0, os.path.join(R, 'tests'))

HEADLINE = ['-b', 'req.method,res.statusCode', '-f',
            '{"eq":["req.method","GET"]}']
CONDITIONS = ('off', 'cold', 'warm')


def digest(points, counters):
    from engines import canon_points
    return hashlib.sha256(repr((sorted(canon_points(points)), json.dumps(
        counters, sort_keys=True))).encode()).hexdigest()


def cudart():
    for p in (os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'),
                           'lib64', 'libcudart.so.12'), 'libcudart.so.12'):
        try:
            return ctypes.CDLL(p)
        except OSError:
            pass
    raise RuntimeError('libcudart.so.12 not found')


def child(a):
    """One scan in this process -> one JSON line."""
    from dragnet_b200 import datasource_gpu, native
    import corpus
    plan = corpus.make_plan(HEADLINE)
    L = native.lib()
    dev = None
    if a['input'] == 'device':
        rt = cudart()
        g = native.gen_params(total_records=a['records'])
        cap = a['records'] * 320 + 64
        dev = ctypes.c_void_p()
        assert rt.cudaMalloc(ctypes.byref(dev), ctypes.c_size_t(cap)) == 0
        n = ctypes.c_size_t()
        native._check(L.dng_gen_device(ctypes.byref(g), 0, 0, a['records'],
                                       dev, cap, ctypes.byref(n)))
        assert rt.cudaDeviceSynchronize() == 0
        dev_len = n.value
    t_open = time.perf_counter()
    p = native.Plan(json.dumps(plan, separators=(',', ':')))
    s = native.Scan(p, 0)
    first = []
    done = threading.Event()

    def poll():
        while not done.is_set():
            if L.dng_scan_launch_count(s.handle) > 0:
                first.append(time.perf_counter())
                return
            time.sleep(0.0002)
    th = threading.Thread(target=poll)
    th.start()
    try:
        for f in a.get('files', ()):
            s.feed_file(f)
        if dev is not None:
            s.feed_device(dev.value, dev_len)
        res = s.finish()
        raw = res.points()
        t_res = time.perf_counter()
    finally:
        done.set()
        th.join()
    counters = s.counters()
    st = s.kernel_stats()
    st.update(s.template_stats())
    res.close()
    s.close()
    p.close()
    names = [b['name'] for b in plan['breakdowns']]
    points = [(list(zip(names, cols)), v) for cols, v in raw]
    maps = open('/proc/self/maps').read()
    # (joins the threads that write entries, as exit would: their counts)
    L.dng_jit_finish()
    print(json.dumps({
        'open_to_result_ms': (t_res - t_open) * 1e3,
        'first_launch_ms': (first[0] - t_open) * 1e3 if first else None,
        'kernel': st['kernel'], 'launches': st['launches'],
        'jit_launches': st['jit']['launches'], 'jit_state': st['jit']['state'],
        'compile_ms': st['jit']['compile_ms'], 'link_ms': st['jit']['link_ms'],
        'cache': native.jit_cache_stats(),
        'nvrtc_mapped': 'libnvrtc' in maps,
        'nvjitlink_mapped': 'libnvJitLink' in maps,
        'digest': digest(points, datasource_gpu.stage_counters(
            plan, counters, len(points)))}))
    if dev is not None:
        cudart().cudaFree(dev)


def gpu_identity():
    try:
        out = subprocess.run(
            ['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit',
             '--format=csv,noheader'], capture_output=True, text=True,
            timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(',')[:2]]
        return {'name': name, 'power_limit': power}
    except Exception as e:      # (the numbers still stand, unlabelled)
        return {'error': str(e)}


def expected(files):
    """The C++ oracle's points and counters, as the children digest
    theirs."""
    from engines import cpp_engine
    import corpus
    plan = corpus.make_plan(HEADLINE)
    return digest(*cpp_engine(plan, files, threads=os.cpu_count() or 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--gb', type=float, default=2.0)
    ap.add_argument('--jit', default='async', choices=['async', 'sync'])
    ap.add_argument('--inputs', default='small,file,device')
    ap.add_argument('--child')
    a = ap.parse_args()
    if a.child:
        child(json.loads(a.child))
        return
    from dragnet_b200 import native
    inputs = a.inputs.split(',')
    base = '/dev/shm' if os.path.isdir('/dev/shm') else None
    work = tempfile.mkdtemp(prefix='dng_cold_', dir=base)
    try:
        runs = {}
        small = os.path.join(work, 'small')
        os.makedirs(small)
        with tarfile.open(os.path.join(R, 'tests', 'golden',
                                       'data.tar.gz')) as tf:
            tf.extractall(small, filter='data')
        sfiles = sorted(os.path.join(d, f) for d, _, fs in os.walk(small)
                        for f in fs)
        runs['small'] = {'files': sfiles}
        records = int(a.gb * 1e9 / 225)
        if 'file' in inputs or 'device' in inputs:
            big = os.path.join(work, 'big.log')
            g = native.gen_params(total_records=records)
            with open(big, 'wb') as f:
                step = 1 << 20
                for first in range(0, records, step):
                    f.write(native.gen_host(g, first,
                                            min(step, records - first)))
            if 'file' in inputs:
                runs['file'] = {'files': [big]}
            if 'device' in inputs:
                runs['device'] = {'records': records}
        oracle = {}
        for name in inputs:
            oracle[name] = expected(runs[name].get('files') or [big])
        ident = gpu_identity()
        print(json.dumps({'gpu': ident, 'jit': a.jit, 'reps': a.reps,
                          'big_bytes': os.path.getsize(big)
                          if 'file' in inputs or 'device' in inputs
                          else None}), flush=True)
        samples = []
        for rep in range(a.reps):
            for name in inputs:
                cache = os.path.join(work, 'cache_%s_%d' % (name, rep))
                for cond in CONDITIONS:
                    env = dict(os.environ, DNG_JIT=a.jit,
                               PYTHONPATH=os.pathsep.join(
                                   [R, os.path.join(R, 'tests')]))
                    env.pop('DNG_JIT_CACHE_DIR', None)
                    if cond != 'off':
                        env['DNG_JIT_CACHE_DIR'] = cache
                    arg = dict(runs[name], input=name)
                    t0 = time.perf_counter()
                    r = subprocess.run([sys.executable, __file__, '--child',
                                        json.dumps(arg)], env=env, cwd=R,
                                       capture_output=True, text=True)
                    wall = (time.perf_counter() - t0) * 1e3
                    if r.returncode != 0:
                        raise SystemExit(r.stderr[-4000:])
                    doc = json.loads(r.stdout.strip().splitlines()[-1])
                    doc.update(input=name, condition=cond, rep=rep,
                               wall_ms=wall,
                               parity=doc.pop('digest') == oracle[name])
                    print(json.dumps(doc), flush=True)
                    if not doc['parity']:
                        raise SystemExit('results differ from the oracle')
                    samples.append(doc)
        summary = {}
        for name in inputs:
            for cond in CONDITIONS:
                ss = [d for d in samples if d['input'] == name and
                      d['condition'] == cond]
                row = {}
                for k in ('wall_ms', 'open_to_result_ms', 'first_launch_ms'):
                    v = [d[k] for d in ss if d[k] is not None]
                    if v:
                        row[k] = {'median': statistics.median(v),
                                  'min': min(v), 'max': max(v)}
                row['jit_launches/launches'] = ['%d/%d' % (
                    d['jit_launches'], d['launches']) for d in ss]
                row['compilers_mapped'] = [d['nvrtc_mapped'] or
                                           d['nvjitlink_mapped'] for d in ss]
                row['cache_hits'] = [d['cache']['hits'] for d in ss]
                summary['%s/%s' % (name, cond)] = row
        print(json.dumps({'summary': summary, 'gpu': ident,
                          'parity': all(d['parity'] for d in samples)}))
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == '__main__':
    main()
