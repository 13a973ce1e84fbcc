"""Group-by aggregation on the GPU where it can go wrong: many distinct keys,
keys whose hashes collide on purpose (tests/corpus.py; test_aggregation_host.py
shows that they collide in the device's hashes), key lengths at the tally
tiers' edges, weights above 255, and the table, arena and miss-list limits.
Every result is compared, points and counters, with the threaded C++ oracle,
which test_aggregation_host.py checks against the Python one."""

import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import cpp_engine  # noqa: E402
from dragnet_b200 import datasource_gpu, native, query as mod_query  # noqa: E402

pytestmark = pytest.mark.gpu

# the F kernel's cases also run with the run-time compiled matcher (each
# template set costs a second or two to link)
JIT_TESTS = {'test_sweep', 'test_skew', 'test_key_lengths',
             'test_merge_and_apart', 'test_colliding_keys',
             'test_miss_list_overflow'}


@pytest.fixture(params=['auto', 'tile', 'warp', 'fast', 'fast28', 'jit'])
def geometry(request, monkeypatch):
    """The library's own choice, the general kernels' two geometries, the F
    path forced on (24 warps, and 28 until keys overflow its inline tier) and
    the F path with its compiled matcher."""
    for v in ('DNG_KERNEL', 'DNG_JIT', 'DNG_F_WARPS', 'DNG_TABLE_CAP',
              'DNG_ARENA_BYTES', 'DNG_MISS_CAP'):
        monkeypatch.delenv(v, raising=False)
    g = request.param
    if g == 'jit':
        if request.node.originalname not in JIT_TESTS:
            pytest.skip('not an F path test')
        monkeypatch.setenv('DNG_KERNEL', 'fast')
        monkeypatch.setenv('DNG_JIT', 'sync')
    elif g in ('fast', 'fast28'):
        monkeypatch.setenv('DNG_KERNEL', 'fast')
        monkeypatch.setenv('DNG_JIT', '0')
        if g == 'fast28':
            monkeypatch.setenv('DNG_F_WARPS', '28')
    elif g != 'auto':
        monkeypatch.setenv('DNG_KERNEL', g)
    return g


def _key(fields):
    return tuple(('nan',) if v != v else v for _, v in fields)


def as_dict(points):
    """points -> {key tuple: value}; keys must be unique."""
    d = {}
    for f, v in points:
        k = _key(f)
        assert k not in d, ('key reported twice', k)
        d[k] = v
    return d


_ORACLE = {}


class Corpus(object):
    def __init__(self, name, lines, tmpdir):
        self.name = name
        self.data = b'\n'.join(lines) + b'\n'
        self.path = os.path.join(tmpdir, name + '.log')
        with open(self.path, 'wb') as f:
            f.write(self.data)

    def oracle(self, plan):
        """(points as a dict, counters) of the C++ oracle, once per module."""
        k = (self.name, repr(plan))
        if k not in _ORACLE:
            p, c = cpp_engine(plan, [self.path], threads=8)
            _ORACLE[k] = (as_dict(p), c)
        return _ORACLE[k]


_CORPORA = {}


def _corpus(name, make, tmp_path_factory):
    if name not in _CORPORA:
        d = str(tmp_path_factory.mktemp('agg'))
        _CORPORA[name] = Corpus(name, make(), d)
    return _CORPORA[name]


def run(plan, c, feed):
    """One scan of corpus c: 'device' = the whole corpus as one device
    buffer (one launch), 'chunks' = host chunks of 1 MiB (a launch and a
    flush each), 'file' = read by the library."""
    if feed == 'device':
        import torch
        buf = torch.frombuffer(bytearray(c.data), dtype=torch.uint8).cuda()
        r = datasource_gpu.run_plan(plan, device_buffers=[(buf.data_ptr(),
                                                          len(c.data))])
        del buf
        return r
    if feed == 'chunks':
        step = 1 << 20
        return datasource_gpu.run_plan(plan, chunks=[
            c.data[i:i + step] for i in range(0, len(c.data), step)])
    return datasource_gpu.run_plan(plan, files=[c.path])


def check(plan, c, feed):
    exp_p, exp_c = c.oracle(plan)
    r = run(plan, c, feed)
    got = as_dict(r.points)
    if got != exp_p:
        miss = [k for k in exp_p if got.get(k) != exp_p[k]][:5]
        extra = [k for k in got if k not in exp_p][:5]
        pytest.fail('%s/%s: %d points, expected %d; wrong or missing %r, '
                    'unexpected %r' % (c.name, feed, len(got), len(exp_p),
                                       [(k, got.get(k), exp_p[k])
                                        for k in miss], extra))
    assert r.counters == exp_c, (c.name, feed)
    return r


def _ran_f(r, geometry):
    if geometry in ('fast', 'fast28', 'jit'):
        assert r.stats['kernel'] == 'F path', r.stats
        if geometry == 'jit':
            assert r.stats['jit']['state'] == 1, r.stats
    elif geometry in ('tile', 'warp'):
        assert r.stats['kernel'] == {'tile': 'CTA tiles',
                                     'warp': 'per-warp chunks'}[geometry]


FEEDS = ['device', 'chunks', 'file']
SWEEP_N = 1000000


@pytest.mark.parametrize('k', [200, 1500, 6000, 50000, 400000])
def test_sweep(k, geometry, tmp_path_factory):
    """k distinct keys over 10^6 records: from everything in every CTA's
    tier 1 to nearly every record a key of its own (tier 2 full, the direct
    global path, long probe chains)."""
    c = _corpus('sweep%d' % k, lambda: corpus.sweep_lines(k, SWEEP_N, seed=k),
                tmp_path_factory)
    plan = corpus.make_plan(['-b', 'key'])
    for feed in FEEDS:
        r = check(plan, c, feed)
        _ran_f(r, geometry)
    if geometry in ('fast', 'fast28', 'jit') and k >= 50000:
        # keys the F kernel's inline tier had no room for took the general
        # tally path (and had to meet the inline ones at flush)
        assert r.stats['inline_overflow'] > 0, r.stats


def test_skew(geometry, tmp_path_factory):
    c = _corpus('skew', lambda: corpus.skew_lines(SWEEP_N), tmp_path_factory)
    plan = corpus.make_plan(['-b', 'key'])
    for feed in FEEDS:
        r = check(plan, c, feed)
        _ran_f(r, geometry)
    if geometry in ('fast', 'fast28', 'jit'):
        assert r.stats['inline_overflow'] > 0, r.stats


def test_data_size_fills_most_of_the_table(geometry, tmp_path_factory):
    """-b dataSize over 10^6 generator records: about 95 % of the default
    2^20-entry table."""
    n = 1000000
    c = _corpus('gen', lambda: native.gen_host(
        native.gen_params(total_records=n), 0, n).split(b'\n')[:-1],
        tmp_path_factory)
    plan = corpus.make_plan(['-b', 'dataSize'])
    exp_p, _ = c.oracle(plan)
    assert len(exp_p) > 0.9 * (1 << 20), len(exp_p)
    check(plan, c, 'device')


@pytest.mark.parametrize('two', [False, True])
def test_key_lengths(two, geometry, tmp_path_factory):
    """Keys of 38-42, 47-49, 254-258, 511 and 512 bytes, in one column and
    split over two."""
    c = _corpus('len%d' % two, lambda: corpus.key_length_lines(
        two, reps=400), tmp_path_factory)
    plan = corpus.make_plan(['-b', 'key,key2' if two else 'key'])
    for feed in FEEDS:
        check(plan, c, feed)


def test_merge_and_apart(geometry, tmp_path_factory):
    c = _corpus('merge', lambda: corpus.merge_apart_lines(reps=2000),
                tmp_path_factory)
    for argv in (['-b', 'key,key2'], ['-b', 'key']):
        plan = corpus.make_plan(argv)
        for feed in FEEDS:
            check(plan, c, feed)
    b = _corpus('buckets', lambda: corpus.BUCKET_LINES * 200,
                tmp_path_factory)
    for argv in (['-b', 'num[aggr=quantize]'], ['-b', 'num'],
                 ['-b', 'num[aggr=lquantize,step=2]']):
        for feed in FEEDS:
            check(corpus.make_plan(argv), b, feed)


def _collision_corpus(tmp_path_factory):
    def make():
        keys = [k for g in corpus.collision_groups().values() for k in g]
        return corpus.kv_lines(keys, 300000, seed=5)
    return _corpus('collide', make, tmp_path_factory)


def test_colliding_keys(geometry, tmp_path_factory):
    """Groups of 40 keys that share an F-hash slot or the whole F hash, a
    general tier-1 or tier-2 slot or the whole 64-bit hash, or a slot of a
    1024-entry table, interleaved so that they meet in every CTA: probe
    chains run out and equality is decided on the key bytes alone."""
    c = _collision_corpus(tmp_path_factory)
    plan = corpus.make_plan(['-b', 'key'])
    for feed in FEEDS:
        r = check(plan, c, feed)
        _ran_f(r, geometry)
    if geometry in ('fast', 'fast28', 'jit'):
        assert r.stats['inline_overflow'] > 0, r.stats


def test_colliding_keys_in_a_small_table(geometry, monkeypatch,
                                         tmp_path_factory):
    """The same with DNG_TABLE_CAP=1024 (280 keys): the 40 keys of one
    global slot start at slot 1020, so their probe chain wraps around the
    table's end."""
    monkeypatch.setenv('DNG_TABLE_CAP', '1024')
    c = _collision_corpus(tmp_path_factory)
    for feed in FEEDS:
        check(corpus.make_plan(['-b', 'key']), c, feed)


def test_weights(geometry, tmp_path_factory):
    """json-skinner weights 0 .. 2^53 (<= 255 through the tally cache, above
    it straight to the table) on shared keys and over 20 000 keys, and keys
    all of whose points weigh 0.  The expected values are also the Python
    integer sums of the corpus, all below 2^63, so that the u64 sums of the
    device and of the C++ oracle cannot agree on a wrapped value."""
    lines = corpus.weight_lines()
    c = _corpus('weights', lambda: lines, tmp_path_factory)
    plan = corpus.make_plan(['-b', 'key'], {'dataFormat': 'json-skinner'})
    sums = corpus.weight_sums(lines)
    assert max(sums.values()) < 1 << 63
    assert c.oracle(plan)[0] == {(k,): v for k, v in sums.items()}
    for feed in FEEDS:
        r = check(plan, c, feed)
    got = {f[0][1]: v for f, v in r.points}
    assert min(got[b'shared%d' % i] for i in range(3)) > 1 << 56
    assert [got[b'zero%d' % i] for i in range(7)] == [0] * 7


def _distinct_lines(n, tag=b''):
    return [b'{"key":"%sd%d","pad":"%s"}' % (tag, i, b'z' * 40)
            for i in range(n)] * 20


def test_table_capacity(geometry, monkeypatch, tmp_path_factory):
    """DNG_TABLE_CAP=1024 holds 1024 distinct keys exactly; one more fails
    loudly, naming the setting; the next scan of the process is exact."""
    monkeypatch.setenv('DNG_TABLE_CAP', '1024')
    plan = corpus.make_plan(['-b', 'key'])
    full = _corpus('cap1024', lambda: _distinct_lines(1024), tmp_path_factory)
    check(plan, full, 'chunks')
    over = _corpus('cap1025', lambda: _distinct_lines(1025), tmp_path_factory)
    with pytest.raises(native.DngError) as ei:
        run(plan, over, 'chunks')
    assert ei.value.code == -7 and 'DNG_TABLE_CAP' in str(ei.value)
    monkeypatch.delenv('DNG_TABLE_CAP')
    check(plan, over, 'chunks')


def test_arena_capacity(geometry, monkeypatch, tmp_path_factory):
    """One arena allocation per distinct key (round8(klen) bytes): an arena
    of exactly their sum is enough, one word less fails naming the arena."""
    c = _corpus('arena', lambda: corpus.key_length_lines(reps=30),
                tmp_path_factory)
    plan = corpus.make_plan(['-b', 'key'])
    exp_p, _ = c.oracle(plan)
    need = sum((len(corpus.encode_key(k[0])) + 7) & ~7 for k in exp_p)
    monkeypatch.setenv('DNG_ARENA_BYTES', str(need))
    check(plan, c, 'chunks')
    monkeypatch.setenv('DNG_ARENA_BYTES', str(need - 8))
    with pytest.raises(native.DngError) as ei:
        run(plan, c, 'chunks')
    assert ei.value.code == -7 and 'DNG_ARENA_BYTES' in str(ei.value)
    monkeypatch.delenv('DNG_ARENA_BYTES')
    check(plan, c, 'chunks')


def test_key_one_byte_too_long(geometry, tmp_path_factory):
    """A 513-byte key among 512-byte ones: DNG_EUNSUPPORTED, not a wrong
    tally; the next scan is exact."""
    ok = [b'{"key":"%s","pad":"x"}' % (b'%03d' % i + b'v' * 507)
          for i in range(200)] * 10
    plan = corpus.make_plan(['-b', 'key'])
    good = _corpus('klen512', lambda: ok, tmp_path_factory)
    check(plan, good, 'chunks')
    bad = _corpus('klen513', lambda: ok + [b'{"key":"%s"}' % (b'w' * 511)],
                  tmp_path_factory)
    with pytest.raises(native.DngError) as ei:
        run(plan, bad, 'chunks')
    assert ei.value.code == -6, ei.value
    check(plan, good, 'file')


def test_arena_larger_than_offsets_address_is_refused(monkeypatch):
    """Key offsets are 32-bit: DNG_ARENA_BYTES above 2 GiB is refused when
    the scan opens (it used to be truncated: 4 GiB + 4 KiB gave a 4 KiB
    arena)."""
    monkeypatch.setenv('DNG_ARENA_BYTES', str((4 << 30) + 4096))
    p = native.Plan('{"format":"json","breakdowns":[]}')
    with pytest.raises(native.DngError) as ei:
        native.Scan(p)
    assert ei.value.code == -1 and 'DNG_ARENA_BYTES' in str(ei.value)
    monkeypatch.setenv('DNG_ARENA_BYTES', str(2 << 30))
    s = native.Scan(p)
    s.close()
    p.close()


def _miss_lines():
    """Generator records with about one in ten of another shape, invalid,
    escaped or with a key over the F path's 256 bytes."""
    n = 60000
    data = native.gen_host(native.gen_params(total_records=n), 0, n)
    recs = data.split(b'\n')[:-1]
    odd = [b'{"req":{"method":"PATCH"},"latency":3}',
           b'{"time":"x","req":{"method":"G\\u0045T"},"latency":1.5e1}',
           b'{"req":{"method":"GET"}', b'', b'[1,2]',
           recs[5].replace(b'"GET"', b'"G\\tT"').replace(b'"PUT"', b'"P\\\\T"'),
           recs[6].replace(b'"latency":', b'"latency":-0.0e+0,"latency":'),
           recs[7].replace(b'}}', b'} }'), recs[8] + b' ', recs[9][:-1],
           recs[10].replace(b'"GET"', b'"' + b'L' * 300 + b'"'),
           recs[11].replace(b'"PUT"', b'"' + b'M' * 400 + b'"')]
    out = []
    for i, r in enumerate(recs):
        out.append(r)
        if i % 9 == 0:
            out.append(odd[(i // 9) % len(odd)])
    return out


@pytest.mark.parametrize('cap', [1, 64])
def test_miss_list_overflow(cap, geometry, monkeypatch, tmp_path_factory):
    """DNG_MISS_CAP far below the ~6 700 records the F kernel hands over per
    launch: the rest are parsed in place (fmiss_inline) and every count
    still adds up."""
    if geometry not in ('fast', 'jit'):
        pytest.skip('the miss list is the F path\'s')
    monkeypatch.setenv('DNG_MISS_CAP', str(cap))
    c = _corpus('miss', _miss_lines, tmp_path_factory)
    for argv in (['-b', 'req.method'], ['-b', 'latency[aggr=quantize]'],
                 ['-b', 'req.method,latency', '-f',
                  '{"ne":["req.method","HEAD"]}']):
        plan = corpus.make_plan(argv)
        for feed in ('device', 'chunks'):
            r = check(plan, c, feed)
            _ran_f(r, geometry)


def test_forced_warps_switch_and_are_not_remembered(geometry, monkeypatch,
                                                    tmp_path_factory):
    """DNG_F_WARPS=28 over 400 000 keys fed in chunks: the scan drops to 24
    warps when keys overflow the inline tier and stays exact.  A forced
    scan that kept its 28 warps must not leave them behind for the unforced
    scans of the same plan."""
    if geometry != 'fast':
        pytest.skip('one geometry: the F path')
    plan = corpus.make_plan(['-b', 'key'])
    big = _corpus('sweep400000', lambda: corpus.sweep_lines(
        400000, SWEEP_N, seed=400000), tmp_path_factory)
    monkeypatch.setenv('DNG_F_WARPS', '28')
    r = check(plan, big, 'chunks')
    assert r.stats['inline_overflow'] > 0 and r.stats['f_warps'] == 24, \
        r.stats
    # (20 keys: room for all of them in the 28-warp inline tier)
    small = _corpus('sweep20', lambda: corpus.sweep_lines(20, 300000),
                    tmp_path_factory)
    r = check(plan, small, 'chunks')
    assert r.stats['f_warps'] == 28, r.stats
    monkeypatch.delenv('DNG_F_WARPS')
    r = check(plan, small, 'chunks')
    assert r.stats['f_warps'] == 24, r.stats


def test_fanout_of_two_high_cardinality_metrics(geometry, tmp_path_factory):
    """Two metrics of 50 000 and 30 000 keys in one pass (keys prefixed
    0xFD, metric) equal two single-metric scans."""
    def make():
        import random
        rng = random.Random(9)
        return [b'{"key":"a%d","key2":"b%d","pad":"%s"}' %
                (rng.randrange(50000), rng.randrange(30000), b'f' * 30)
                for _ in range(400000)]
    c = _corpus('fanout', make, tmp_path_factory)
    metrics = [{'filter': None, 'breakdowns': [{'name': 'key',
                                                'field': 'key'}]},
               {'filter': {'ne': ['key', 'a7']},
                'breakdowns': [{'name': 'key2', 'field': 'key2'},
                               {'name': 'key', 'field': 'key'}]}]
    queries = [mod_query.metricQuery(m, None, None, 'all', None)
               for m in metrics]
    multi = mod_query.scan_plan_multi(queries)
    singles = [mod_query.scan_plan(q) for q in queries]
    r = run(multi, c, 'chunks')
    for m, single in enumerate(singles):
        exp_p, exp_c = c.oracle(single)
        got = as_dict([(f[:-1], v) for f, v in r.points
                       if f[-1] == ('__dn_metric', m)])
        assert got == exp_p, m
        assert r.counters[m] == exp_c, m
