"""Record framing at every staging boundary of the scan kernels (`-m gpu`).

Layouts (framing.py) put newlines, long-record heads, dense units and bytes
the SWAR newline test flags at chosen offsets from the units of one kernel.
Fed as one 16-byte aligned device buffer, unit k of the launch starts at
byte k x U of the buffer, so each case sits exactly where it was built.  Each
scan is compared with the C++ oracle (and, for the small layouts, the oracle
with the Python one); the device feed's long_records counter, which counts
the records a kernel had to reach from HBM, is predicted from the layout, so
that it also checks the geometry the kernel ran with.

  test_exact_placement       each layout under tile, warp, fast and auto
                             (jit for the F layout), fed to the device, as
                             odd host chunks and as a file
  test_f_multi_chunk_segments  a block replicated on the device until the F
                             kernel's segments hold 2, 6 and 16 chunks: the
                             path only inputs of hundreds of MB reach
  test_device_feed_framing   dng_scan_feed_device's newline search and carry
  test_line_limit            lines of 2^24 - 1, 2^24 and 2^24 + 1 bytes

Scans run with DNG_JIT=0 except under jit, so that no background compile is
left running when the module ends."""

import json
import os
import random
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
import framing  # noqa: E402
from engines import canon_points, cpp_engine, py_engine  # noqa: E402
from dragnet_b200 import datasource_gpu, native  # noqa: E402

pytestmark = pytest.mark.gpu

KIND = {'tile': 'CTA tiles', 'warp': 'per-warp chunks', 'fast': 'F path',
        'jit': 'F path'}
UNIT = {'CTA tiles': ('tile', framing.PRELAP),
        'per-warp chunks': ('w_chunk', framing.W_PRELAP),
        'F path': ('f_chunk', framing.F_PRE)}
RING = 64 << 20         # api.cu: DNG_RING_BYTES default
ELIMIT, EUNSUPPORTED = -7, -6


def _set_kernel(monkeypatch, k):
    monkeypatch.delenv('DNG_KERNEL', raising=False)
    monkeypatch.setenv('DNG_JIT', 'sync' if k == 'jit' else '0')
    if k in ('fast', 'jit'):
        monkeypatch.setenv('DNG_KERNEL', 'fast')
    elif k != 'auto':
        monkeypatch.setenv('DNG_KERNEL', k)


def _device(data, pad=0):
    """data in a fresh device buffer (256-byte aligned by the allocator)."""
    import torch
    buf = torch.empty(len(data) + pad + 16, dtype=torch.uint8,
                      device='cuda:0')
    buf[:len(data)].copy_(torch.frombuffer(bytearray(data),
                                           dtype=torch.uint8))
    return buf


def _odd_chunks(data, seed):
    rng = random.Random(seed)
    out, i = [], 0
    while i < len(data):
        n = rng.choice([1, 15, 16, 17, 511, 4097, 65521, 300007])
        out.append(data[i:i + n])
        i += n
    return out


_ORACLE = {}


def oracle(key, plan, path, python=False):
    """(canon points, counters) of the C++ oracle, once per module; with
    python=True the Python oracle must agree."""
    if key not in _ORACLE:
        p, c = cpp_engine(plan, [path], threads=8)
        if python:
            pp, pc = py_engine(plan, [path])
            assert canon_points(pp) == canon_points(p), key
            assert pc == c, key
        _ORACLE[key] = (canon_points(p), c)
    return _ORACLE[key]


def scan(plan, **feed):
    r = datasource_gpu.run_plan(plan, **feed)
    return canon_points(r.points), r.counters, r.flat_counters, r.stats


# -- 1. exact placement --------------------------------------------------------

_LAYOUTS = {}


def layout(name, tmp_path_factory):
    if name not in _LAYOUTS:
        L, g, U = framing.fixed_layout(name, seed=11)
        data = L.data()
        p = tmp_path_factory.mktemp('framing') / ('%s.log' % name)
        p.write_bytes(data)
        _LAYOUTS[name] = (data, g, U, str(p))
    return _LAYOUTS[name]


QUERIES = {'g': ['-b', 'g,k,'], 'id': ['-b', 'id,']}


@pytest.mark.parametrize('kernel', ['tile', 'warp', 'fast', 'auto', 'jit'])
@pytest.mark.parametrize('name', ['fast', 'warp', 'tile'])
def test_exact_placement(name, kernel, tmp_path_factory, monkeypatch):
    """Each kernel's layout under every kernel: results equal the oracle's
    for every feed, and the device feed's long_records equals the count the
    layout predicts for the kernel that ran."""
    if kernel == 'jit' and name != 'fast':
        pytest.skip('the run-time compiled matcher: the F layout only')
    _set_kernel(monkeypatch, kernel)
    data, g, U, path = layout(name, tmp_path_factory)
    small = name != 'tile'
    last = data.rfind(b'\n') + 1
    beg, end = framing.records(data[:last])
    buf = _device(data)
    for q in (['g', 'id'] if small else ['g']):
        plan = corpus.make_plan(QUERIES[q])
        exp_p, exp_c = oracle((name, q), plan, path, python=small)
        feeds = {'device': dict(device_buffers=[(buf.data_ptr(),
                                                 len(data))]),
                 'chunks': dict(chunks=_odd_chunks(data, len(data))),
                 'file': dict(files=[path])}
        for feed, kw in feeds.items():
            pts, ctr, flat, st = scan(plan, **kw)
            assert pts == exp_p, (name, kernel, q, feed)
            assert ctr == exp_c, (name, kernel, q, feed)
            if kernel != 'auto':
                assert st['kernel'] == KIND[kernel], (feed, st)
            if feed == 'device' and kernel != 'auto':
                key, pre = UNIT[st['kernel']]
                seg = 1
                if st['kernel'] == 'F path':
                    seg = framing.f_segment(last, g['f_chunk'], _sms())
                    assert seg == 1
                want = framing.long_records(beg, end, g[key], pre, seg)
                assert flat['long_records'] == want, (name, kernel, q)
    del buf


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# -- 2. multi-chunk F segments -------------------------------------------------

_BLOCK = {}


def f_block(tmp_path_factory):
    if not _BLOCK:
        data, g = framing.f_block(seed=5)
        p = tmp_path_factory.mktemp('fblock') / 'block.log'
        p.write_bytes(data)
        _BLOCK.update(data=data, g=g, path=str(p))
    return _BLOCK


def _scaled(counters, reps):
    """Stage counters of `reps` copies of an input: every count times reps,
    but the aggregator's points once."""
    out = {}
    for stage, cs in counters.items():
        out[stage] = {k: v if (stage, k) == ('Aggregator', 'noutputs')
                      else v * reps for k, v in cs.items()}
    return out


SEGMENTS = [2, 6, 16]


@pytest.mark.parametrize('kernel', ['fast', 'jit'])
@pytest.mark.parametrize('seg', SEGMENTS)
def test_f_multi_chunk_segments(seg, kernel, tmp_path_factory, monkeypatch):
    """The F kernel's segments of several chunks: the tail of one chunk is
    the next one's pre-lap (shared -> shared), the open record and its start
    carry over, dense and newline-free chunks come mid-segment.  A launch
    gets segments of two chunks only from about 50,000 chunks on, so the
    block is replicated on the device to the size the launch formula needs.
    The result must be reps x the oracle's for the block, and long_records
    (records straddling a segment start g0 > 0 that begin at or before
    g0 - DNG_F_PRE) exactly as predicted.  Under fast the same bytes then go
    through the host feed, whose 64 MiB launches run one-chunk segments: the
    larger count it must give proves the segments above really held several
    chunks."""
    import torch
    _set_kernel(monkeypatch, kernel)
    B = f_block(tmp_path_factory)
    data, g = B['data'], B['g']
    chunk, sms = g['f_chunk'], _sms()
    reps = -(-framing.f_bytes_for_segment(seg, chunk, sms) // len(data))
    total = reps * len(data)
    assert framing.f_segment(total, chunk, sms) == seg
    plan = corpus.make_plan(QUERIES['g'])
    exp_p, exp_c = oracle(('block', 'g'), plan, B['path'])
    exp_p = [(k, v * reps) for k, v in exp_p]
    exp_c = _scaled(exp_c, reps)

    b0, e0 = framing.records(data)
    far = (e0 - b0) >= framing.F_PRE    # only these can be long
    beg, end = framing.replicate(b0[far], e0[far], len(data), reps)
    want_dev = framing.long_records(beg, end, chunk, framing.F_PRE, seg)

    host = torch.frombuffer(bytearray(data), dtype=torch.uint8)
    dev = host.to('cuda:0').repeat(reps)
    pts, ctr, flat, st = scan(plan, device_buffers=[(dev.data_ptr(), total)])
    assert st['kernel'] == 'F path', st
    assert pts == exp_p
    assert ctr == exp_c
    assert flat['long_records'] == want_dev, (seg, total)
    print('segment %d (%s): %d bytes, %d chunks, long_records predicted %d '
          'observed %d' % (seg, kernel, total, -(-total // chunk), want_dev,
                           flat['long_records']))
    del dev
    if kernel != 'fast':
        torch.cuda.empty_cache()
        return
    # the same bytes from the host: 64 MiB launches, one-chunk segments
    assert framing.f_segment(RING + 2 * framing.MAXREC, chunk, sms) == 1
    b1, e1 = framing.replicate(b0, e0, len(data), reps)
    want_host = framing.host_pieces_long(b1, e1, total, chunk, framing.F_PRE,
                                         RING)
    assert want_host > want_dev
    whole = host.repeat(reps)
    p = native.Plan(json.dumps(plan))
    s = native.Scan(p, 0)
    try:
        native._check(native.lib().dng_scan_feed(s.handle, whole.data_ptr(),
                                                 total), s.handle)
        res = s.finish()
        flat = s.counters()
        st = s.template_stats()
        names = [b['name'] for b in plan['breakdowns']]
        hp = canon_points([(list(zip(names, c)), v) for c, v in res.points()])
        res.close()
    finally:
        s.close()
        p.close()
    del whole
    assert st['kernel'] == 'F path', st
    assert hp == exp_p
    assert datasource_gpu.stage_counters(plan, flat, len(hp)) == exp_c
    assert flat['long_records'] == want_host
    print('segment %d host feed: long_records predicted %d observed %d' %
          (seg, want_host, flat['long_records']))
    torch.cuda.empty_cache()


# -- 3. device-feed framing ----------------------------------------------------

MiB = 1 << 20


def _records_to(L, n):
    """Filler records until the layout holds at least n bytes."""
    while len(L.buf) < n:
        L.filler()


def device_cases():
    """name -> (bytes, [buffer lengths]): every cut 16-byte aligned."""
    out = {}
    L = framing.Layout(21)
    _records_to(L, int(1.5 * MiB))
    a = len(L.buf)                      # a 2.3 MiB line starts here
    L.buf += framing.long_line(int(2.3 * MiB), L._next()) + b'\n'
    nl = len(L.buf) - 1
    _records_to(L, len(L.buf) + 200000)
    data = L.data()

    def rest(*lens):
        return list(lens) + [len(data) - sum(lens)]
    # the carried line ends 1.5 MiB into the next buffer: its first newline
    # is outside the head window
    cut = (nl - int(1.5 * MiB)) & ~15
    out['carried_1.5MiB'] = (data, rest(cut))
    # the first buffer's last newline lies 1.2 MiB before its end, outside
    # both windows; then a buffer without a newline, then the line's end
    c1 = (a + int(1.2 * MiB)) & ~15
    c2 = ((nl - MiB // 2) & ~15) - c1
    out['last_nl_1.2MiB_before_end'] = (data, rest(c1, c2))
    # three buffers without a newline between the line's start and end
    out['three_without_newline'] = (data, rest((a + 4096) & ~15, MiB,
                                               MiB - 48, 4096))
    # a buffer of 18 MiB whose newlines all lie between its 1 MiB windows:
    # taken for one without a newline, it would be carried and refused
    L3 = framing.Layout(22)
    _records_to(L3, 300000)
    a3 = len(L3.buf)
    L3.buf += framing.long_line(int(2.3 * MiB), L3._next()) + b'\n'
    _records_to(L3, len(L3.buf) + 15 * MiB)
    b3 = len(L3.buf)
    L3.buf += framing.long_line(2 * MiB, L3._next()) + b'\n'
    _records_to(L3, len(L3.buf) + 200000)
    d3 = L3.data()
    c0 = (a3 + MiB // 2) & ~15
    c1 = ((b3 + int(1.5 * MiB)) & ~15) - c0
    out['newlines_only_between_windows'] = (d3, [c0, c1, len(d3) - c0 - c1])
    # many cuts, some of them tiny
    L2, _, _ = framing.fixed_layout('fast', seed=23)
    d2 = L2.data()
    rng = random.Random(3)
    offs = sorted(set([rng.randrange(0, len(d2)) & ~15 for _ in range(40)] +
                      [16, 32, 48, 4608, 4624]))
    offs = [o for o in offs if 0 < o < len(d2)]
    lens = [y - x for x, y in zip([0] + offs, offs + [len(d2)])]
    out['many_cuts'] = (d2, lens)
    return out


DEVICE_CASES = device_cases()


@pytest.mark.parametrize('kernel', ['tile', 'fast'])
@pytest.mark.parametrize('name', sorted(DEVICE_CASES))
def test_device_feed_framing(name, kernel, monkeypatch):
    """dng_scan_feed_device looks for the first and last newline in 1 MiB
    windows at the ends of a buffer, and searches all of it when either is
    not in its window; the carried line is finished in a side buffer.  Each
    split must give what the host feed of the same bytes gives."""
    _set_kernel(monkeypatch, kernel)
    data, lens = DEVICE_CASES[name]
    assert sum(lens) == len(data)
    plan = corpus.make_plan(QUERIES['g'])
    buf = _device(data)
    bufs, off = [], 0
    for n in lens:
        assert off % 16 == 0
        bufs.append((buf.data_ptr() + off, n))
        off += n
    want = scan(plan, chunks=[data])
    got = scan(plan, device_buffers=bufs)
    assert got[0] == want[0], name
    assert got[1] == want[1], name
    assert got[2]['lines'] == data.count(b'\n') + (data[-1:] != b'\n')
    del buf


# -- 4. the 16 MiB line limit --------------------------------------------------

LINE_LENGTHS = [framing.MAXREC - 1, framing.MAXREC, framing.MAXREC + 1]


def limit_input(n):
    """(terminated, unterminated, pre): records, one line of n bytes before
    its newline, records; the line's newline 16-byte aligned."""
    L = framing.Layout(31)
    _records_to(L, 100000)
    L.fill_to(len(L.buf) + framing.MINREC + (-(len(L.buf) +
              framing.MINREC + n) % 16))
    pre = L.data()
    line = framing.long_line(n, L._next())
    assert len(line) == n and (len(pre) + n) % 16 == 0
    L2 = framing.Layout(32, first_id=L.id)
    _records_to(L2, 60000)
    return pre + line + b'\n' + L2.data(), pre + line, len(pre)


@pytest.fixture(scope='module')
def limit_files(tmp_path_factory):
    out = {}
    d = tmp_path_factory.mktemp('limit')
    for n in LINE_LENGTHS:
        term, unterm, pre = limit_input(n)
        pt, pu = d / ('t%d.log' % n), d / ('u%d.log' % n)
        pt.write_bytes(term)
        pu.write_bytes(unterm)
        out[n] = (term, unterm, pre, str(pt), str(pu))
    return out


# feed -> the error a line of 2^24 bytes or more must give: ELIMIT where a
# feed has to carry 2^24 bytes of it, EUNSUPPORTED where a kernel sees it
# whole, either where the cuts decide
LIMIT_FEEDS = {'host_whole': [EUNSUPPORTED], 'host_cut': [ELIMIT, EUNSUPPORTED],
               'host_carry': [ELIMIT], 'host_final': [ELIMIT],
               'file': [ELIMIT, EUNSUPPORTED], 'device_whole': [EUNSUPPORTED],
               'device_split': [ELIMIT], 'device_carry': [ELIMIT],
               'device_final': [ELIMIT]}


@pytest.mark.parametrize('kernel', ['tile', 'fast'])
@pytest.mark.parametrize('n', LINE_LENGTHS)
def test_line_limit(n, kernel, limit_files, monkeypatch):
    """A line of 2^24 - 1 bytes (before its newline) scans as the oracle
    says through every feed, also as the unterminated final line; a line of
    2^24 or 2^24 + 1 bytes fails every feed with the error DESIGN.md section
    4 names, and never returns a result."""
    _set_kernel(monkeypatch, kernel)
    term, unterm, pre, pt, pu = limit_files[n]
    nl = pre + n                        # the line's newline: 16-aligned
    plan = corpus.make_plan(QUERIES['g'])
    buf = _device(term)
    p0 = buf.data_ptr()
    mid = (pre + n // 2) & ~15
    feeds = {
        'host_whole': dict(chunks=[term]),
        'host_cut': dict(chunks=[term[i:i + 5 * MiB + 7]
                                 for i in range(0, len(term), 5 * MiB + 7)]),
        'host_carry': dict(chunks=[term[:nl], term[nl:]]),
        'host_final': dict(chunks=[unterm]),
        'file': dict(files=[pt]),
        'device_whole': dict(device_buffers=[(p0, len(term))]),
        'device_split': dict(device_buffers=[(p0, mid),
                                             (p0 + mid, len(term) - mid)]),
        'device_carry': dict(device_buffers=[(p0, nl),
                                             (p0 + nl, len(term) - nl)]),
        'device_final': dict(device_buffers=[(p0, len(unterm))]),
    }
    for feed, kw in feeds.items():
        final = feed.endswith('_final')
        if n < framing.MAXREC:
            exp_p, exp_c = oracle(('limit', n, final), plan,
                                  pu if final else pt)
            pts, ctr, flat, st = scan(plan, **kw)
            assert pts == exp_p, (feed, n)
            assert ctr == exp_c, (feed, n)
            if kernel == 'fast':
                assert st['kernel'] == 'F path', st
        else:
            with pytest.raises(native.DngError) as ei:
                scan(plan, **kw)
            assert ei.value.code in LIMIT_FEEDS[feed], (feed, n, ei.value)
    del buf
