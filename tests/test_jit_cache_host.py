"""The on-disk cache of run-time compiled kernels (dragnet_b200/csrc/
jit_cache.h) without a GPU: its file format and policy compiled with a small
driver (tests/hostcheck/jit_cache_check.cpp) and stepped through stores,
lookups, damaged entries, concurrent writers and eviction; and one real linked
kernel (jit_build(), through tests/hostcheck) stored and read back."""

import json
import os
import struct
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import build_hostcheck  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')
DRIVER = os.path.join(ROOT, 'tests', 'hostcheck', 'jit_cache_check.cpp')
BIG = 1 << 30
HEAD = 24       # magic, format version, 0, key length


@pytest.fixture(scope='module')
def jc(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp('jc') / 'jit_cache_check')
    subprocess.check_call(['g++', '-std=c++17', '-O1', '-Wall', '-Wextra',
                           '-Werror', '-I', CSRC, '-o', exe, DRIVER,
                           os.path.join(CSRC, 'jit_cache.cpp')])

    def run(*cmds):
        r = subprocess.run([exe], input='\n'.join(cmds) + '\n',
                           capture_output=True, text=True, check=True)
        return [{k: int(v) if v.isdigit() else v
                 for k, v in (kv.split('=') for kv in line.split())}
                for line in r.stdout.splitlines()]
    return run


def name(jc, key):
    return jc('name ' + key)[0]['name']


def entries(d):
    return sorted(f for f in os.listdir(d) if f.endswith('.jitk'))


def test_round_trip(jc, tmp_path):
    d = str(tmp_path / 'c')
    put, get, st = jc('put %s k1 5000 %d -' % (d, BIG), 'get %s k1 -' % d,
                      'stats')
    assert put['ok'] == 1
    assert get == {'hit': 1, 'bytes': 5000, 'same': 1}
    assert st == {'hits': 1, 'misses': 0, 'writes': 1, 'evictions': 0,
                  'errors': 0}
    assert entries(d) == [name(jc, 'k1')]
    # the directory is created private, and nothing else is left in it
    assert os.stat(d).st_mode & 0o777 == 0o700
    assert os.listdir(d) == [name(jc, 'k1')]
    # a key never stored: a miss, nothing counted as an error
    assert jc('get %s k2 -' % d, 'stats') == [
        {'hit': 0, 'bytes': 0, 'same': 0},
        {'hits': 0, 'misses': 1, 'writes': 0, 'evictions': 0, 'errors': 0}]


def test_other_key_under_the_same_name_is_a_miss(jc, tmp_path):
    d = str(tmp_path / 'c')
    r = jc('put %s keyA 3000 %d forced.jitk' % (d, BIG),
           'get %s keyB forced.jitk' % d,
           # (a key that is a prefix of the stored one, and one longer)
           'get %s key forced.jitk' % d, 'get %s keyAA forced.jitk' % d,
           'get %s keyA forced.jitk' % d, 'stats')
    assert [x.get('hit') for x in r[1:5]] == [0, 0, 0, 1]
    assert r[-1]['misses'] == 3 and r[-1]['errors'] == 0


def test_build_id_covers_every_byte_of_the_library(jc, tmp_path):
    """Keys on disk start with the build id of the library file: a hash of
    all of it, so that a library whose matcher generator, compiler options or
    embedded kernel builds differ never finds another build's kernels."""
    import __graft_entry__
    __graft_entry__.build()
    lib = open(os.path.join(ROOT, 'dragnet_b200', 'libdragnet_gpu.so'),
               'rb').read()
    # what the generated source and its build are made from, as the library
    # holds it: the NVRTC and nvJitLink options, the prelude of the
    # generated matcher, the scanners' text
    edits = {}
    for what, marker in (('options', b'-maxrregcount=72'),
                         ('prelude', b'struct JMem {'),
                         ('scanners', b'fscan_str')):
        at = lib.find(marker)
        assert at > 0, what
        edits[what] = at + len(marker) - 1
    edits['one byte anywhere'] = len(lib) // 3
    ids = {}
    for what, at in [('as built', None)] + sorted(edits.items()):
        b = bytearray(lib)
        if at is not None:
            b[at] ^= 0x01
        p = tmp_path / ('lib_%d.so' % len(ids))
        p.write_bytes(bytes(b))
        ids[what] = jc('buildid %s' % p)[0]['id']
    assert len(set(ids.values())) == len(ids), ids
    assert all(len(i) == 32 for i in ids.values())
    # the same bytes under another name: the same id
    (tmp_path / 'copy.so').write_bytes(lib)
    assert jc('buildid %s' % (tmp_path / 'copy.so'))[0]['id'] == \
        ids['as built']
    assert jc('buildid %s' % (tmp_path / 'none.so'))[0]['id'] == '-'


def test_directory_others_may_write_to_is_not_used(jc, tmp_path):
    """Whoever can write an entry chooses the code a scan runs: a directory
    that group or others may write to is neither read nor written."""
    d = tmp_path / 'shared'
    d.mkdir()
    assert jc('put %s k 1000 %d -' % (d, BIG))[0]['ok'] == 1
    for mode in (0o770, 0o777, 0o1777):
        os.chmod(d, mode)
        put, get, st = jc('put %s k2 1000 %d -' % (d, BIG),
                          'get %s k -' % d, 'stats')
        assert put['ok'] == 0 and get['hit'] == 0, mode
        assert st['errors'] == 2 and st['misses'] == 1, (mode, st)
    os.chmod(d, 0o755)
    assert jc('get %s k -' % d)[0]['hit'] == 1
    assert entries(d) == [name(jc, 'k')]


def damage_cases(f, klen):
    n = len(f)
    cub = HEAD + klen + 8
    flip = lambda b, i: b[:i] + bytes([b[i] ^ 0x10]) + b[i + 1:]  # noqa
    return {
        'truncated': f[:-1],
        'truncated_to_head': f[:HEAD + 4],
        'empty': b'',
        'longer': f + b'\0',
        'magic': flip(f, 0),
        'key_length': flip(f, 16),
        'key_byte': flip(f, HEAD + klen // 2),
        'cubin_length': flip(f, HEAD + klen),
        'cubin_first': flip(f, cub),
        'cubin_middle': flip(f, cub + (n - 8 - cub) // 2),
        'cubin_last': flip(f, n - 9),
        'checksum': flip(f, n - 3),
    }


@pytest.mark.parametrize('case', sorted(damage_cases(b'\0' * 100, 10)))
def test_damaged_entry_is_a_miss(jc, tmp_path, case):
    d = str(tmp_path / 'c')
    key = 'some-kernel-key'
    assert jc('put %s %s 4000 %d -' % (d, key, BIG))[0]['ok'] == 1
    p = os.path.join(d, name(jc, key))
    f = open(p, 'rb').read()
    assert struct.unpack_from('<Q', f, 16)[0] == len(key)
    open(p, 'wb').write(damage_cases(f, len(key))[case])
    get, st = jc('get %s %s -' % (d, key), 'stats')
    assert get['hit'] == 0
    assert st['misses'] == 1 and st['hits'] == 0
    # and a new build replaces it
    get = jc('put %s %s 4000 %d -' % (d, key, BIG), 'get %s %s -' % (d, key))
    assert get[1] == {'hit': 1, 'bytes': 4000, 'same': 1}


def test_wrong_format_version_is_a_miss(jc, tmp_path):
    d = str(tmp_path)
    r = jc('forge %s k 2000 - 2' % d, 'get %s k -' % d,
           'forge %s k 2000 - 1' % d, 'get %s k -' % d)
    # (the entry is whole, checksum and all: only its version differs)
    assert [r[1]['hit'], r[3]['hit']] == [0, 1]


def test_concurrent_writers_leave_one_valid_entry(jc, tmp_path):
    d = str(tmp_path / 'c')
    key = 'one-key-eight-writers'
    r = jc('fork 8 %s %s 300000 %d' % (d, key, BIG), 'get %s %s -' % (d, key))
    assert r[0]['failed'] == 0
    assert r[1] == {'hit': 1, 'bytes': 300000, 'same': 1}
    assert os.listdir(d) == [name(jc, key)]


def test_eviction_keeps_the_bound_and_drops_least_recently_hit(jc, tmp_path):
    d = str(tmp_path / 'c')
    size = 10000
    bound = 3 * (size + 200)        # three entries fit, four do not
    r = jc(*['put %s k%d %d %d -' % (d, i, size, bound) for i in range(3)])
    assert all(x['ok'] for x in r)
    names = {i: name(jc, 'k%d' % i) for i in range(5)}
    # k0 oldest, then k1, then k2; then k0 is hit and is the newest
    r = jc('age %s %s 300' % (d, names[0]), 'age %s %s 200' % (d, names[1]),
           'age %s %s 100' % (d, names[2]), 'get %s k0 -' % d,
           'put %s k3 %d %d -' % (d, size, bound), 'stats')
    assert r[3]['hit'] == 1 and r[4]['ok'] == 1
    assert r[-1]['evictions'] == 1
    assert entries(d) == sorted([names[0], names[2], names[3]])
    total = sum(os.path.getsize(os.path.join(d, f)) for f in entries(d))
    assert total <= bound
    # the next write drops k2, the least recently used left
    jc('put %s k4 %d %d -' % (d, size, bound))
    assert entries(d) == sorted([names[0], names[3], names[4]])


def test_stray_temporary_files_are_swept_after_a_minute(jc, tmp_path):
    d = tmp_path / 'c'
    d.mkdir()
    old = d / '.abc.jitk.1234.0.tmp'
    new = d / '.def.jitk.1234.1.tmp'
    old.write_bytes(b'x' * 100)
    new.write_bytes(b'x' * 100)
    r = jc('age %s %s 61' % (d, old.name), 'put %s k 100 %d -' % (d, BIG))
    assert r[1]['ok'] == 1
    assert not old.exists() and new.exists()


def test_unwritable_directory_counts_an_error_and_misses(jc, tmp_path):
    f = tmp_path / 'file'
    f.write_bytes(b'')
    d = str(f / 'cache')            # (under a regular file: never creatable)
    put, get, st = jc('put %s k 1000 %d -' % (d, BIG), 'get %s k -' % d,
                      'stats')
    assert put['ok'] == 0 and get['hit'] == 0
    assert st == {'hits': 0, 'misses': 1, 'writes': 0, 'evictions': 0,
                  'errors': 1}


def test_real_linked_kernel_round_trips(jc, tmp_path):
    """A kernel jit_build() really linked for a scan's templates, stored and
    read back byte for byte."""
    from dragnet_b200 import native
    n = 2000
    data = native.gen_host(native.gen_params(total_records=n), 0, n)
    p = tmp_path / 'syn.log'
    p.write_bytes(data)
    plan = corpus.make_plan(['-b', 'req.method,res.statusCode'])
    pf = tmp_path / 'plan.json'
    pf.write_text(json.dumps(plan))
    dump = str(tmp_path / 'jm')
    env = dict(os.environ, DNG_HOSTCHECK_F='1', DNG_HOSTCHECK_JIT='2',
               DNG_HOSTCHECK_JIT_DUMP=dump)
    r = subprocess.run([build_hostcheck(), str(pf), str(p)],
                       capture_output=True, env=env)
    assert r.returncode == 0, r.stderr.decode()
    cubin = open(dump + '.cubin', 'rb').read()
    assert cubin[:4] == b'\x7fELF' and len(cubin) > 10000
    d = str(tmp_path / 'c')
    out = str(tmp_path / 'back.cubin')
    r = jc('put %s real-key @%s.cubin %d -' % (d, dump, BIG),
           'get %s real-key - %s' % (d, out))
    assert r[0]['ok'] == 1 and r[1]['hit'] == 1
    assert open(out, 'rb').read() == cubin


def test_library_exports_the_cache_entry_points():
    import __graft_entry__
    __graft_entry__.build()
    from dragnet_b200 import native
    L = native.lib()
    for sym in ('dng_jit_cache_dir', 'dng_jit_cache_stats'):
        assert hasattr(L, sym) and sym in native.SYMBOLS
    # pure host calls, they work without a GPU; in a process of their own,
    # since the directory set is the process's for good
    code = (
        'from dragnet_b200 import native\n'
        'st = native.jit_cache_stats()\n'
        'assert sorted(st) == sorted(native.JIT_CACHE_STATS), st\n'
        'assert all(v == 0 for v in st.values()), st\n'
        'native.set_jit_cache_dir("/nonexistent/dir")\n'
        'native.set_jit_cache_dir(None)\n')
    env = dict(os.environ, PYTHONPATH=ROOT)
    env.pop('DNG_JIT_CACHE_DIR', None)
    subprocess.run([sys.executable, '-c', code], check=True, cwd=ROOT,
                   env=env)
