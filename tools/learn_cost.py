"""Host cost of learning templates before a scan's first launch, no GPU needed:
writes the head of the bench's input (oracle/gen_ndjson, the bench's seed),
builds tests/hostcheck/learn_check.cpp and prints, as JSON, the fastest of N
runs of each step (tmpl_candidates, kc_sample, the F and general blobs,
jit_source, jit_key) and a hash of the generated matcher source.

    python tools/learn_cost.py [N]
"""
import json
import os
import subprocess
import sys
import tempfile

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
sys.path.insert(0, os.path.join(R, 'tests'))
import corpus  # noqa: E402

CSRC = os.path.join(R, 'dragnet_b200', 'csrc')
reps = sys.argv[1] if len(sys.argv) > 1 else '200'
with tempfile.TemporaryDirectory() as d:
    subprocess.check_call(['make', '-s', '-C', os.path.join(R, 'oracle'),
                           'gen_ndjson'])
    subprocess.check_call(['make', '-s', '-C', CSRC, 'build/jit_blob.o'])
    exe = os.path.join(d, 'learn_check')
    subprocess.check_call(
        ['g++', '-std=c++17', '-O2', '-I/usr/local/cuda/include', '-o', exe,
         os.path.join(R, 'tests', 'hostcheck', 'learn_check.cpp')] +
        [os.path.join(CSRC, f) for f in ('plan.cpp', 'result.cpp', 'tmpl.cpp',
                                         'fast.cpp', 'jit.cpp')] +
        [os.path.join(CSRC, 'build', 'jit_blob.o'), '-ldl'])
    sample = os.path.join(d, 'sample.log')
    # bench.py: seed 0xD5A60000, 100 M rows; the sample is its first 256 KB
    subprocess.check_call([os.path.join(R, 'oracle', 'gen_ndjson'), sample,
                           str(0xD5A60000), '100000000', '0', '2000'])
    plan = os.path.join(d, 'plan.json')
    with open(plan, 'w') as f:
        json.dump(corpus.make_plan(['-b', 'req.method,res.statusCode', '-f',
                                    '{"eq":["req.method","GET"]}']), f)
    sys.stdout.write(subprocess.check_output([exe, 'cost', plan, sample,
                                              reps]).decode())
