"""Scan engines the parity tests can drive with the golden harness.

  py_engine         oracle/dn_oracle.py
  hostcheck_engine  tests/hostcheck/hostcheck: the device per-record code
                    (dragnet_b200/csrc/record.cuh) compiled for the host,
                    TEST ONLY
"""

import json
import math
import os
import struct
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import dn_oracle  # noqa: E402

HOSTCHECK_DIR = os.path.join(ROOT, 'tests', 'hostcheck')
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')


def py_engine(plan, files):
    def chunks():
        for p in files:
            with open(p, 'rb') as f:
                while True:
                    b = f.read(16834)   # lib/datasource-file.js:264
                    if not b:
                        break
                    yield b
    return dn_oracle.scan(plan, chunks())


def build_hostcheck():
    exe = os.path.join(HOSTCHECK_DIR, 'hostcheck')
    srcs = [os.path.join(HOSTCHECK_DIR, 'hostcheck.cpp'),
            os.path.join(CSRC, 'plan.cpp'), os.path.join(CSRC, 'result.cpp'),
            os.path.join(CSRC, 'tmpl.cpp'), os.path.join(CSRC, 'fast.cpp')]
    deps = srcs + [os.path.join(CSRC, n) for n in
                   ('record.cuh', 'jsnum.cuh', 'jsdate.cuh', 'plan.h',
                    'result.h', 'tmpl.h', 'tmpl.cuh', 'fast.h', 'fast.cuh',
                    'kernel_choice.h',
                    'fscan.cuh')]
    srcs.append(os.path.join(CSRC, 'jit.cpp'))
    deps += [os.path.join(CSRC, 'jit.cpp'), os.path.join(CSRC, 'jit.h'),
             os.path.join(CSRC, 'fast_kernel.cuh'),
             os.path.join(CSRC, 'fast_jit.cu')]
    def stale():
        return not os.path.exists(exe) or \
            os.path.getmtime(exe) < max(os.path.getmtime(d) for d in deps)
    if stale():
        # (pytest-xdist workers all come here at once: one of them builds)
        import fcntl
        with open(exe + '.lock', 'w') as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            if stale():
                # the relocatable kernel + fscan.cuh as data (jit.cpp links
                # them in)
                subprocess.check_call(['make', '-s', '-C', CSRC,
                                       'build/jit_blob.o'])
                subprocess.check_call(['g++', '-std=c++17', '-O1', '-g',
                                       '-I/usr/local/cuda/include', '-o',
                                       exe + '.new'] + srcs +
                                      [os.path.join(CSRC, 'build',
                                                    'jit_blob.o'), '-ldl'])
                os.replace(exe + '.new', exe)
    return exe


# flat drop counters (dng_counters) -> vstream-style per-stage counters: the
# product's own shaping (the oracles count per stage on their own, so the
# comparison with them checks it)
from dragnet_b200.datasource_gpu import stage_counters as staged_counters  # noqa: E402


def hostcheck_engine(plan, files):
    exe = build_hostcheck()
    with tempfile.NamedTemporaryFile('w', suffix='.json', delete=False) as f:
        json.dump(plan, f)
        pf = f.name
    try:
        out = subprocess.run([exe, pf] + list(files), capture_output=True,
                             check=True).stdout
    finally:
        os.unlink(pf)
    doc = json.loads(out)
    assert doc['counters']['unsupported'] == 0, doc['counters']
    points = []
    for p in doc['points']:
        fields = []
        for b, col in zip(plan['breakdowns'], p['cols']):
            if 's' in col:
                fields.append((b['name'], bytes.fromhex(col['s'])))
            else:
                fields.append((b['name'], struct.unpack(
                    '<d', struct.pack('<Q', int(col['n'], 16)))[0]))
        points.append((fields, p['value']))
    return points, staged_counters(plan, doc['counters'], len(points))


def hostcheck_multi(plan, files, fast=False):
    """Fan-out plan through the host build of the device logic ->
    ({metric: canon points}, [flat drop counters per metric])."""
    exe = build_hostcheck()
    with tempfile.NamedTemporaryFile('w', suffix='.json', delete=False) as f:
        json.dump(plan, f)
        pf = f.name
    env = dict(os.environ)
    env.pop('DNG_HOSTCHECK_FAST', None)
    if fast:
        env['DNG_HOSTCHECK_FAST'] = '1'
    try:
        out = subprocess.run([exe, pf] + list(files), capture_output=True,
                             check=True, env=env).stdout
    finally:
        os.unlink(pf)
    doc = json.loads(out)
    assert doc['counters']['unsupported'] == 0
    per = {}
    for p in doc['points']:
        m = p['metric']
        bds = plan['metrics'][m]['breakdowns']
        fields = []
        for b, col in zip(bds, p['cols']):
            if 's' in col:
                fields.append((b['name'], bytes.fromhex(col['s'])))
            else:
                fields.append((b['name'], struct.unpack(
                    '<d', struct.pack('<Q', int(col['n'], 16)))[0]))
        per.setdefault(m, []).append((fields, p['value']))
    flats = [doc['counters']] + doc['mcounters']
    return per, flats


def build_cpp_oracle():
    subprocess.check_call(['make', '-s', '-C', os.path.join(ROOT, 'oracle')])
    return os.path.join(ROOT, 'oracle', 'dn_oracle_cpp')


def _decode_doc(plan, doc):
    points = []
    for p in doc['points']:
        fields = []
        for b, col in zip(plan['breakdowns'], p['cols']):
            if 's' in col:
                fields.append((b['name'], bytes.fromhex(col['s'])))
            else:
                fields.append((b['name'], struct.unpack(
                    '<d', struct.pack('<Q', int(col['n'], 16)))[0]))
        points.append((fields, p['value']))
    return points, staged_counters(plan, doc['counters'], len(points))


def cpp_engine(plan, files, threads=1):
    """oracle/dn_oracle.cpp (DOM-based C++ restatement; also the CPU
    baseline bench.py times)."""
    exe = build_cpp_oracle()
    with tempfile.NamedTemporaryFile('w', suffix='.json', delete=False) as f:
        json.dump(plan, f)
        pf = f.name
    try:
        out = subprocess.run([exe, pf, '--threads', str(threads)] +
                             list(files), capture_output=True,
                             check=True).stdout
    finally:
        os.unlink(pf)
    return _decode_doc(plan, json.loads(out))


def canon_points(points):
    """Order-independent, NaN-safe form for comparing two engines."""
    out = []
    for fields, value in points:
        key = []
        for name, v in fields:
            if isinstance(v, bytes):
                key.append(('s', v))
            elif v != v:
                key.append(('n', 'nan'))
            else:
                key.append(('n', float(v) + 0.0))
        out.append((tuple(key), value))
    return sorted(out, key=repr)
