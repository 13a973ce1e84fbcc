"""Parity of the CUDA path (through the C ABI) with the oracle.  These need a
CUDA device (`-m gpu`) and read only files of this repository."""

import ctypes
import hashlib
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import canon_points, cpp_engine, py_engine  # noqa: E402
from golden_harness import check_section  # noqa: E402

pytestmark = pytest.mark.gpu


# under 'jit' every distinct template set costs a second or two of compilation:
# the cases that exercise the matcher, not all of them
JIT_TESTS = {'test_reference_goldens_through_c_abi', 'test_edge_lines',
             'test_synthetic_matches_oracle',
             'test_scalar_forms_behind_one_template',
             'test_optional_fields_make_a_branching_trie',
             'test_template_fuzz', 'test_chunk_boundaries_do_not_matter'}


@pytest.fixture(params=['auto', 'tile', 'warp', 'fast', 'jit'], autouse=True)
def kernel_geometry(request, monkeypatch):
    """Every case under the general kernels' two geometries (CTA-wide tiles,
    per-warp chunks), under the F path forced on (scan_kernel_f + the miss
    kernel, whatever the templates cover) and under the library's own choice
    between them."""
    monkeypatch.delenv('DNG_KERNEL', raising=False)
    monkeypatch.delenv('DNG_JIT', raising=False)
    if request.param == 'jit':
        # the F path with the matcher compiled at run time for the templates
        # (jit.cpp), waited for; 'fast' = the same with the interpreted one
        if request.node.originalname not in JIT_TESTS:
            pytest.skip('not a matcher test')
        monkeypatch.setenv('DNG_KERNEL', 'fast')
        monkeypatch.setenv('DNG_JIT', 'sync')
    elif request.param == 'fast':
        monkeypatch.setenv('DNG_KERNEL', 'fast')
        monkeypatch.setenv('DNG_JIT', '0')
    elif request.param != 'auto':
        monkeypatch.setenv('DNG_KERNEL', request.param)


def gpu_engine(plan, files):
    from dragnet_b200 import datasource_gpu
    r = datasource_gpu.run_plan(plan, files=files)
    return r.points, r.counters


def gpu_engine_chunks(plan, data, chunk):
    from dragnet_b200 import datasource_gpu
    chunks = [data[i:i + chunk] for i in range(0, len(data), chunk)]
    r = datasource_gpu.run_plan(plan, chunks=chunks)
    return r.points, r.counters


@pytest.mark.parametrize('suite', ['scan_file', 'scan_fileset', 'empty',
                                   'scan_manta'])
def test_reference_goldens_through_c_abi(suite, goldens, datadir):
    n = 0
    for i, sec in enumerate(goldens['suites'][suite]):
        if sec['cmd'] != 'scan':
            continue
        if suite == 'scan_manta' and ('--counters' in sec['argv'] or
                                      '--dry-run' in sec['argv'] or
                                      '-n' in sec['argv']):
            continue
        check_section(gpu_engine, suite, i, sec, datadir)
        n += 1
    assert n >= 8


def _write(tmp_path, name, lines, final_newline=True):
    p = tmp_path / name
    p.write_bytes(b'\n'.join(lines) + (b'\n' if final_newline else b''))
    return str(p)


@pytest.mark.parametrize('qi', range(len(corpus.EDGE_QUERIES)))
def test_edge_lines(qi, tmp_path):
    argv, ds = corpus.EDGE_QUERIES[qi]
    plan = corpus.make_plan(argv, ds)
    path = _write(tmp_path, 'edge.log', corpus.EDGE_LINES)
    exp_p, exp_c = py_engine(plan, [path])
    act_p, act_c = gpu_engine(plan, [path])
    assert canon_points(act_p) == canon_points(exp_p)
    assert act_c == exp_c


@pytest.mark.parametrize('qi', range(len(corpus.SKINNER_QUERIES)))
def test_skinner_lines(qi, tmp_path):
    argv, ds = corpus.SKINNER_QUERIES[qi]
    plan = corpus.make_plan(argv, ds)
    path = _write(tmp_path, 'sk.log', corpus.SKINNER_LINES)
    exp_p, exp_c = py_engine(plan, [path])
    act_p, act_c = gpu_engine(plan, [path])
    assert canon_points(act_p) == canon_points(exp_p)
    assert act_c == exp_c


@pytest.mark.parametrize('seed', range(4))
def test_random_lines(seed, tmp_path):
    path = _write(tmp_path, 'rand.log', corpus.random_lines(seed, 3000),
                  final_newline=(seed % 2 == 0))
    for argv, ds in corpus.EDGE_QUERIES[::4]:
        plan = corpus.make_plan(argv, ds)
        exp_p, exp_c = py_engine(plan, [path])
        act_p, act_c = gpu_engine(plan, [path])
        assert canon_points(act_p) == canon_points(exp_p), argv
        assert act_c == exp_c, argv


def test_chunk_boundaries_do_not_matter(tmp_path):
    """lstream carries partial lines across arbitrary chunk boundaries."""
    from dragnet_b200 import native
    data = native.gen_host(native.gen_params(total_records=3000), 0, 3000)
    data += b'{"req":{"method":"TAIL"}}'          # unterminated last line
    plan = corpus.make_plan(['-b', 'req.method,res.statusCode'])
    ref = None
    for chunk in (len(data), 1 << 16, 4099, 257, 31):
        pts, ctr = gpu_engine_chunks(plan, data, chunk)
        if ref is None:
            ref = (canon_points(pts), ctr)
            assert ctr['json parser']['ninputs'] == 3001
        assert (canon_points(pts), ctr) == ref, chunk


@pytest.mark.parametrize('name', sorted(corpus.BASELINE_QUERIES))
def test_synthetic_matches_oracle(name, tmp_path):
    """BASELINE.json query shapes on mktestdata-shaped input, vs the oracle."""
    from dragnet_b200 import native
    n = 20000
    data = native.gen_host(native.gen_params(total_records=n), 0, n)
    p = tmp_path / 'syn.log'
    p.write_bytes(data)
    argv, ds = corpus.BASELINE_QUERIES[name]
    plan = corpus.make_plan(argv, ds)
    exp_p, exp_c = py_engine(plan, [str(p)])
    act_p, act_c = gpu_engine(plan, [str(p)])
    assert canon_points(act_p) == canon_points(exp_p)
    assert act_c == exp_c


def test_device_generator_is_byte_identical_and_feed_device_matches():
    import torch
    from dragnet_b200 import datasource_gpu, native
    n = 200000
    params = native.gen_params(total_records=n)
    host = native.gen_host(params, 0, n)
    cap = n * 320
    buf = torch.empty(cap, dtype=torch.uint8, device='cuda:0')
    ln = ctypes.c_size_t()
    rc = native.lib().dng_gen_device(ctypes.byref(params), 0, 0, n,
                                     buf.data_ptr(), cap, ctypes.byref(ln))
    assert rc == 0
    assert ln.value == len(host)
    dev = bytes(buf[:ln.value].cpu().numpy().tobytes())
    assert hashlib.sha256(dev).digest() == hashlib.sha256(host).digest()
    plan = corpus.make_plan(['-b', 'operation,req.method,host'])
    a = datasource_gpu.run_plan(plan, device_buffers=[(buf.data_ptr(),
                                                       ln.value)])
    b = datasource_gpu.run_plan(plan, chunks=[host])
    assert canon_points(a.points) == canon_points(b.points)
    assert a.flat_counters['lines'] == n
    # split device feed at an arbitrary (unaligned-to-line) 16-byte boundary
    cut = (ln.value // 3) & ~15
    c = datasource_gpu.run_plan(plan, device_buffers=[
        (buf.data_ptr(), cut), (buf.data_ptr() + cut, ln.value - cut)])
    assert canon_points(c.points) == canon_points(b.points)
    assert c.flat_counters['lines'] == n


def test_feed_file_reader_threads_match_feed(tmp_path):
    """dng_scan_feed_file (pread by several threads into a pinned ring, fed in
    order) must equal feeding the same bytes directly; two files in a row
    exercise ring reuse and the carry across files."""
    from dragnet_b200 import datasource_gpu, native
    n = 330000                                   # ~74 MB: 18 blocks of 4 MiB
    data = native.gen_host(native.gen_params(total_records=n), 0, n)
    cut = len(data) // 2 + 1234                  # mid-line split across files
    (tmp_path / 'a.log').write_bytes(data[:cut])
    (tmp_path / 'b.log').write_bytes(data[cut:])
    plan = corpus.make_plan(['-b', 'req.method,res.statusCode,host'])
    a = datasource_gpu.run_plan(plan, files=[str(tmp_path / 'a.log'),
                                             str(tmp_path / 'b.log')])
    b = datasource_gpu.run_plan(plan, chunks=[data])
    assert canon_points(a.points) == canon_points(b.points)
    assert a.flat_counters['lines'] == n == b.flat_counters['lines']
    assert a.flat_counters['invalid_json'] == 0


def test_medium_lines_take_the_lock_step_path(tmp_path):
    """1-16 KB lines mixed with short ones: warps whose lanes hold lines of
    very different lengths (the automaton idles in an absorbing state)."""
    import random
    rng = random.Random(7)
    lines = []
    for i in range(4000):
        pad = rng.choice([0, 0, 0, 50, 900, 1500, 3000, 6000, 12000])
        lines.append(b'{"a":"k%d","pad":"' % (i % 7) + b'x' * pad +
                     b'","n":{"b":[1,{"c":"\\\\"}]},"z":%d}' % i)
    lines[100] = lines[100][:-1]                    # invalid
    lines[200] = b'{"a":"esc\\u0041","pad":"' + b'y' * 5000 + b'"}'
    path = _write(tmp_path, 'medium.log', lines)
    for argv in (['-b', 'a,'], ['-b', 'n.b.length'], []):
        plan = corpus.make_plan(argv)
        exp_p, exp_c = py_engine(plan, [path])
        act_p, act_c = gpu_engine(plan, [path])
        assert canon_points(act_p) == canon_points(exp_p), argv
        assert act_c == exp_c, argv


def test_long_lines_and_large_counts(tmp_path):
    """Lines longer than the staged window take the HBM path; many small
    lines exercise the multi-pass newline index."""
    lines = [b'{"a":"s","pad":"' + b'p' * 70000 + b'"}',
             b'{"pad":"' + b'q' * 200000 + b'","a":"t"}'] + [b'{"a":1}'] * 50000
    lines += [b''] * 30000 + [b'{"a":"s"}']
    path = _write(tmp_path, 'long.log', lines)
    plan = corpus.make_plan(['-b', 'a,'])
    exp_p, exp_c = py_engine(plan, [path])
    act_p, act_c = gpu_engine(plan, [path])
    assert canon_points(act_p) == canon_points(exp_p)
    assert act_c == exp_c


def test_record_templates_do_not_change_results():
    """Record templates (tmpl.h): on mktestdata-shaped input nearly every
    record is taken by a learned template; the points and every counter must
    equal the run with templates switched off."""
    from dragnet_b200 import datasource_gpu, native
    n = 300000
    data = native.gen_host(native.gen_params(total_records=n), 0, n)
    for name in sorted(corpus.BASELINE_QUERIES):
        argv, ds = corpus.BASELINE_QUERIES[name]
        plan = corpus.make_plan(argv, ds)
        on = datasource_gpu.run_plan(plan, chunks=[data], templates=True)
        off = datasource_gpu.run_plan(plan, chunks=[data], templates=False)
        assert canon_points(on.points) == canon_points(off.points), name
        assert on.flat_counters == off.flat_counters, name
        assert off.stats['templated_records'] == 0
        assert on.stats['templates'] >= 3, on.stats
        assert on.stats['templated_records'] >= 0.99 * n, on.stats


@pytest.mark.parametrize('rot', [0, 24, 48, 72, 96, 120, 144])
def test_edge_lines_with_templates_learned_from_different_heads(rot, tmp_path):
    """Templates are learned from the first lines of the input: rotate the
    edge corpus so that every odd shape gets to be a template once."""
    lines = corpus.EDGE_LINES[rot:] + corpus.EDGE_LINES[:rot]
    path = _write(tmp_path, 'edge.log', lines)
    for argv, ds in corpus.EDGE_QUERIES[::4]:
        plan = corpus.make_plan(argv, ds)
        exp_p, exp_c = py_engine(plan, [path])
        act_p, act_c = gpu_engine(plan, [path])
        assert canon_points(act_p) == canon_points(exp_p), (rot, argv)
        assert act_c == exp_c, (rot, argv)


def test_templates_with_unmatched_records_in_the_same_tile(tmp_path):
    """Templated records interleaved with records of other shapes, invalid
    lines, escapes in captured strings and non-integer numbers: the matcher
    must hand exactly those to the automaton."""
    from dragnet_b200 import native
    n = 60000
    data = native.gen_host(native.gen_params(total_records=n), 0, n)
    recs = data.split(b'\n')[:-1]
    odd = [b'{"req":{"method":"PATCH"},"latency":3}',
           b'{"time":"x","req":{"method":"G\\u0045T"},"latency":1.5e1}',
           b'{"req":{"method":"GET"}', b'', b'[1,2]',
           recs[5].replace(b'"GET"', b'"G\\tT"').replace(b'"PUT"', b'"P\\\\T"'),
           recs[6].replace(b'"latency":', b'"latency":-0.0e+0,"latency":'),
           recs[7].replace(b'}}', b'} }'), recs[8] + b' ', recs[9][:-1]]
    out = []
    for i, r in enumerate(recs):
        out.append(r)
        if i % 97 == 0:
            out.append(odd[(i // 97) % len(odd)])
    path = _write(tmp_path, 'mixed.log', out)
    for argv in (['-b', 'req.method'], ['-b', 'latency[aggr=quantize]'],
                 ['-b', 'req.method,latency', '-f',
                  '{"ne":["req.method","HEAD"]}']):
        plan = corpus.make_plan(argv)
        exp_p, exp_c = py_engine(plan, [path])
        act_p, act_c = gpu_engine(plan, [path])
        assert canon_points(act_p) == canon_points(exp_p), argv
        assert act_c == exp_c, argv


@pytest.mark.parametrize('pad', [b'', b'"host":"padding-padding-padding-x",'])
def test_scalar_forms_behind_one_template(pad, tmp_path):
    """Every number / literal / string-body form in one record shape, so that
    the template's wildcard scans see them all (see tests/corpus.py).  The
    padded variant makes the lines long enough for the F kernel's chunks
    (more than 128 lines per chunk go to the general parser as they are)."""
    from dragnet_b200 import datasource_gpu
    lines = [b'{"a":7,"s":"k0"}'] * 3 + corpus.scalar_lines()
    lines = [b'{' + pad + ln[1:] for ln in lines]
    if os.environ.get('DNG_KERNEL') == 'fast' and not pad:
        pytest.skip('lines of 16 bytes: the F kernel hands them all over')
    jit_expected = os.environ.get('DNG_JIT') == 'sync'
    path = _write(tmp_path, 'scalars.log', lines)
    for argv in (['-b', 'a,'], ['-b', 's,'], ['-b', 'a[aggr=quantize]'],
                 ['-b', 'a,s,', '-f', '{"ge":["a",1]}']):
        plan = corpus.make_plan(argv)
        exp_p, exp_c = py_engine(plan, [path])
        r = datasource_gpu.run_plan(plan, files=[path])
        assert canon_points(r.points) == canon_points(exp_p), argv
        assert r.counters == exp_c, argv
        assert r.stats['templated_records'] > 20, r.stats
        if jit_expected:
            assert r.stats['jit']['state'] == 1, r.stats
            assert r.stats['jit']['launches'] >= 1, r.stats


@pytest.mark.parametrize('pad', [0, 40, 90, 140, 260, 380, 700])
def test_line_lengths_pick_different_chunk_geometries(pad, tmp_path):
    """The per-warp kernel sizes its chunks from the sampled mean line length
    (and gives way to the tile kernel for long lines): same answers at every
    size."""
    import random
    rng = random.Random(pad)
    lines = []
    for i in range(30000):
        extra = b'y' * rng.randrange(0, 9)
        lines.append(b'{"a":"k%d","n":%d,"pad":"' % (i % 11, i % 97) +
                     b'x' * pad + extra + b'","b":{"c":%s}}' %
                     (b'null' if i % 5 == 0 else b'"v%d"' % (i % 3)))
    lines[777] = lines[777][:-1]                    # invalid
    path = _write(tmp_path, 'len.log', lines)
    for argv in (['-b', 'a,b.c'], ['-b', 'n[aggr=lquantize,step=10]']):
        plan = corpus.make_plan(argv)
        exp_p, exp_c = py_engine(plan, [path])
        act_p, act_c = gpu_engine(plan, [path])
        assert canon_points(act_p) == canon_points(exp_p), (pad, argv)
        assert act_c == exp_c, (pad, argv)


def _chunks(data, n):
    return [data[i:i + n] for i in range(0, len(data), n)]


def test_stream_that_changes_shape_is_relearned(tmp_path):
    """Templates come from the head of the first data; when later input has
    another shape the scan notices (most records miss) and learns again."""
    from dragnet_b200 import datasource_gpu
    a = b''.join(b'{"a":"x%d","n":%d}\n' % (i % 5, i % 13)
                 for i in range(300000))
    b = b''.join(b'{"kind":"b","a":"y%d","m":{"z":%d},"n":%d}\n' %
                 (i % 7, i % 3, i % 17) for i in range(1200000))
    path = tmp_path / 'two.log'
    path.write_bytes(a + b)
    plan = corpus.make_plan(['-b', 'a,n,'])
    exp_p, exp_c = cpp_engine(plan, [str(path)], threads=8)
    r = datasource_gpu.run_plan(plan, chunks=_chunks(a + b, 4 << 20))
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    if os.environ.get('DNG_KERNEL') != 'tile':
        # the later shape got its own template for most of its records
        assert r.stats['templated_records'] > 0.6 * 1500000, r.stats


def test_stream_that_turns_to_long_lines_switches_kernel(tmp_path):
    """Short lines first (per-warp chunks are chosen), then 3 KB lines: they
    straddle the warps' pre-lap, the scan falls back to CTA-wide tiles."""
    from dragnet_b200 import datasource_gpu
    a = b''.join(b'{"a":"x%d","n":%d}\n' % (i % 5, i % 13)
                 for i in range(300000))
    b = b''.join(b'{"a":"L%d","pad":"' % (i % 3) + b'p' * 3000 +
                 b'","n":%d}\n' % (i % 7) for i in range(12000))
    path = tmp_path / 'long.log'
    path.write_bytes(a + b)
    plan = corpus.make_plan(['-b', 'a,n,'])
    exp_p, exp_c = cpp_engine(plan, [str(path)], threads=8)
    r = datasource_gpu.run_plan(plan, chunks=_chunks(a + b, 4 << 20))
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    if 'DNG_KERNEL' not in os.environ:
        assert r.stats['kernel'] == 'CTA tiles', r.stats


def test_optional_fields_make_a_branching_trie(tmp_path):
    """Four optional fields -> sixteen record shapes sharing prefixes (sibling
    dispatch + alt chains in the template trie): all templated, answers equal
    the oracle's."""
    import random
    from dragnet_b200 import datasource_gpu
    rng = random.Random(11)
    lines = []
    for i in range(40000):
        parts = [b'"id":%d' % i]
        if rng.random() < 0.5:
            parts.append(b'"a":"x%d"' % (i % 3))
        if rng.random() < 0.5:
            parts.append(b'"b":{"c":%d}' % (i % 4))
        if rng.random() < 0.5:
            parts.append(b'"d":null')
        if rng.random() < 0.5:
            parts.append(b'"e":[%d,"s"]' % (i % 2))
        parts.append(b'"z":"end"')
        lines.append(b'{' + b','.join(parts) + b'}')
    path = _write(tmp_path, 'opt.log', lines)
    plan = corpus.make_plan(['-b', 'a,b.c,d,'])
    exp_p, exp_c = cpp_engine(plan, [path], threads=4)
    r = datasource_gpu.run_plan(plan, files=[path])
    assert canon_points(r.points) == canon_points(exp_p)
    assert r.counters == exp_c
    assert r.stats['templates'] == 16, r.stats
    assert r.stats['templated_records'] == len(lines), r.stats


@pytest.mark.parametrize('seed', range(3))
def test_template_fuzz(seed, tmp_path):
    """corpus.template_fuzz_lines through the GPU: shapes with re-rolled scalar
    values and a little damage."""
    path = _write(tmp_path, 'fz.log', corpus.template_fuzz_lines(100 + seed, 3000))
    for argv, ds in corpus.EDGE_QUERIES[:30:5]:
        plan = corpus.make_plan(argv, ds)
        exp_p, exp_c = py_engine(plan, [path])
        act_p, act_c = gpu_engine(plan, [path])
        assert canon_points(act_p) == canon_points(exp_p), (seed, argv)
        assert act_c == exp_c, (seed, argv)
