"""The on-disk cache of run-time compiled kernels (dng_jit_cache_dir,
DNG_JIT_CACHE_DIR) on the GPU.  Every step is a new process, waited for, so
that the per-process map of kernels cannot answer for the disk: a process that
finds its kernel on disk must run it from its first launch, in async mode too,
without loading either compiler library, and every result must be the
oracle's."""

import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import canon_points, py_engine  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# one scan in a fresh process -> one JSON line
WORKER = r'''
import json, sys
args = json.loads(sys.argv[1])
from dragnet_b200 import datasource_gpu, native
from engines import canon_points
if 'api_dir' in args:
    native.set_jit_cache_dir(args['api_dir'])
r = datasource_gpu.run_plan(args['plan'], files=args['files'],
                            devices=args.get('devices'))
maps = open('/proc/self/maps').read()
# (the threads that write entries are joined here, as at exit)
native.lib().dng_jit_finish()
shards = r.stats['shards'] if 'shards' in r.stats else [r.stats]
print(json.dumps({
    'points': repr(sorted(canon_points(r.points))),
    'counters': r.counters,
    'shards': [{'kernel': s['kernel'], 'launches': s['launches'],
                'jit': s['jit']} for s in shards],
    'cache': native.jit_cache_stats(),
    'nvrtc': 'libnvrtc' in maps, 'nvjitlink': 'libnvJitLink' in maps}))
'''

HEADLINE = ['-b', 'req.method,res.statusCode', '-f',
            '{"eq":["req.method","GET"]}']


def run(tmp_path, plan, files, mode, cache=None, devices=None, api_dir=None):
    home = tmp_path / 'home'
    home.mkdir(exist_ok=True)
    env = dict(os.environ, DNG_JIT=mode, HOME=str(home),
               XDG_CACHE_HOME=str(home / '.cache'),
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, 'tests')]))
    for v in ('DNG_JIT_CACHE_DIR', 'DNG_KERNEL', 'DNG_TEMPLATES'):
        env.pop(v, None)
    if cache is not None:
        env['DNG_JIT_CACHE_DIR'] = str(cache)
    args = {'plan': plan, 'files': [str(f) for f in files]}
    if devices:
        args['devices'] = devices
    if api_dir is not None:
        args['api_dir'] = str(api_dir)
    r = subprocess.run([sys.executable, '-c', WORKER, json.dumps(args)],
                       capture_output=True, text=True, env=env, cwd=ROOT,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def expect(plan, files):
    pts, counters = py_engine(plan, [str(f) for f in files])
    return repr(sorted(canon_points(pts))), counters


def entries(d):
    return sorted(f for f in os.listdir(d) if f.endswith('.jitk')) \
        if os.path.isdir(d) else []


def all_compiled(doc):
    """Every scan launch of every shard ran the compiled F kernel."""
    return all(s['kernel'] == 'F path' and s['jit']['state'] == 1 and
               s['jit']['launches'] == s['launches'] > 0
               for s in doc['shards'])


@pytest.fixture(scope='module')
def data(tmp_path_factory):
    from dragnet_b200 import native
    d = tmp_path_factory.mktemp('jc_data')
    n = 40000
    a = d / 'syn.log'
    a.write_bytes(native.gen_host(native.gen_params(total_records=n), 0, n))
    # other record templates: latency as a string
    b = d / 'syn_str.log'
    b.write_bytes(native.gen_host(native.gen_params(
        seed=7, total_records=n, string_latency=True), 0, n))
    return a, b


def test_cache_off_writes_nothing(tmp_path, data):
    plan = corpus.make_plan(HEADLINE)
    pts, counters = expect(plan, [data[0]])
    doc = run(tmp_path, plan, [data[0]], 'sync')
    assert doc['points'] == pts and doc['counters'] == counters
    assert doc['cache'] == dict.fromkeys(doc['cache'], 0)
    # the kernel is built as it always was
    assert all_compiled(doc)
    jit = doc['shards'][0]['jit']
    assert jit['compile_ms'] > 0 and jit['link_ms'] > 0
    # (the CUDA driver keeps its own compute cache under ~/.nv)
    home = tmp_path / 'home'
    assert [p for p in home.rglob('*')
            if p.relative_to(home).parts[0] != '.nv'] == []


def test_cold_then_warm_then_damaged(tmp_path, data):
    plan = corpus.make_plan(HEADLINE)
    pts, counters = expect(plan, [data[0]])
    cache = tmp_path / 'cache'
    # cold: built, one entry written
    cold = run(tmp_path, plan, [data[0]], 'sync', cache=cache)
    assert cold['points'] == pts and cold['counters'] == counters
    assert cold['cache']['writes'] == 1 and cold['cache']['hits'] == 0
    assert cold['cache']['misses'] == 1 and cold['cache']['errors'] == 0
    assert all_compiled(cold)
    assert len(entries(cache)) == 1
    assert os.stat(cache).st_mode & 0o777 == 0o700
    # its key: the library file's build id (a hash, then the file's size),
    # then jit_key() with the compute capability in place of the device
    import struct
    import torch
    f = (cache / entries(cache)[0]).read_bytes()
    klen = struct.unpack_from('<Q', f, 16)[0]
    key = f[24:24 + klen]
    lib = os.path.join(ROOT, 'dragnet_b200', 'libdragnet_gpu.so')
    assert int(key[16:32], 16) == os.path.getsize(lib)
    major, minor = torch.cuda.get_device_capability(0)
    assert struct.unpack_from('<i', key, 32)[0] == major * 10 + minor
    # warm, async: the compiled kernel from the first launch, no compiler
    warm = run(tmp_path, plan, [data[0]], 'async', cache=cache)
    assert warm['points'] == pts and warm['counters'] == counters
    assert warm['cache'] == {'hits': 1, 'misses': 0, 'writes': 0,
                             'evictions': 0, 'errors': 0}
    jit = warm['shards'][0]['jit']
    assert jit['compile_ms'] == 0 and jit['link_ms'] == 0
    assert all_compiled(warm)
    assert not warm['nvrtc'] and not warm['nvjitlink']
    # the same through dng_jit_cache_dir(), which overrides the environment
    api = run(tmp_path, plan, [data[0]], 'async', cache=tmp_path / 'unused',
              api_dir=cache)
    assert api['points'] == pts and api['cache']['hits'] == 1
    assert all_compiled(api) and not (tmp_path / 'unused').exists()
    # damaged on disk: a miss, rebuilt without an error, results exact
    p = cache / entries(cache)[0]
    b = bytearray(p.read_bytes())
    b[len(b) // 2] ^= 0x40
    p.write_bytes(bytes(b))
    fixed = run(tmp_path, plan, [data[0]], 'sync', cache=cache)
    assert fixed['points'] == pts and fixed['counters'] == counters
    assert fixed['cache'] == {'hits': 0, 'misses': 1, 'writes': 1,
                              'evictions': 0, 'errors': 0}
    assert all_compiled(fixed) and fixed['shards'][0]['jit']['link_ms'] > 0
    # and the rewritten entry is good again
    again = run(tmp_path, plan, [data[0]], 'async', cache=cache)
    assert again['points'] == pts and again['cache']['hits'] == 1
    assert all_compiled(again)


def test_two_shards_start_on_the_cached_kernel(tmp_path, data):
    plan = corpus.make_plan(HEADLINE)
    pts, counters = expect(plan, [data[0]])
    cache = tmp_path / 'cache'
    cold = run(tmp_path, plan, [data[0]], 'sync', cache=cache, devices=[0, 0])
    assert cold['points'] == pts and cold['counters'] == counters
    assert cold['cache']['writes'] >= 1
    warm = run(tmp_path, plan, [data[0]], 'async', cache=cache,
               devices=[0, 0])
    assert warm['points'] == pts and warm['counters'] == counters
    assert len(warm['shards']) == 2 and all_compiled(warm)
    assert warm['cache']['misses'] == 0 and warm['cache']['hits'] >= 1
    assert warm['cache']['errors'] == 0
    assert not warm['nvrtc'] and not warm['nvjitlink']


def test_other_templates_get_their_own_entry(tmp_path, data):
    plan = corpus.make_plan(HEADLINE)
    cache = tmp_path / 'cache'
    run(tmp_path, plan, [data[0]], 'sync', cache=cache)
    first = entries(cache)
    assert len(first) == 1
    other = corpus.make_plan(['-b', 'host,req.method'])
    pts, counters = expect(other, [data[1]])
    doc = run(tmp_path, other, [data[1]], 'sync', cache=cache)
    assert doc['points'] == pts and doc['counters'] == counters
    # not the first entry's kernel: a miss, a build and a second entry
    assert doc['cache'] == {'hits': 0, 'misses': 1, 'writes': 1,
                            'evictions': 0, 'errors': 0}
    assert all_compiled(doc)
    assert len(entries(cache)) == 2 and set(first) <= set(entries(cache))
    # and each finds its own from now on
    for plan_, f, p_ in ((plan, data[0], expect(plan, [data[0]])[0]),
                         (other, data[1], pts)):
        doc = run(tmp_path, plan_, [f], 'async', cache=cache)
        assert doc['points'] == p_ and doc['cache']['hits'] == 1
        assert all_compiled(doc)
