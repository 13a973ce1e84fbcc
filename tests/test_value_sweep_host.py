"""The value sweep (corpus.value_sweep_lines: numbers at binary64 and
simple-integer edges, numeric strings, strings at UTF-8/UTF-16 edges, dates
over years 0000-9999) through the device per-record logic compiled for the
host (TEST ONLY), in every parser mode, against the Python oracle; the oracle
itself against the C++ one and against a second reference derived from the
generated values (corpus.sweep_reference)."""

import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import (_decode_doc, build_hostcheck, canon_points,  # noqa: E402
                     cpp_engine, py_engine)

SEEDS = (0, 1)
N = 3000
MODES = {'general': {}, 'fast': {'DNG_HOSTCHECK_FAST': '1'},
         'tmpl': {'DNG_HOSTCHECK_FAST': '1', 'DNG_HOSTCHECK_TMPL': '1'},
         'fpath': {'DNG_HOSTCHECK_F': '1'},
         'jit': {'DNG_HOSTCHECK_F': '1', 'DNG_HOSTCHECK_JIT': '1'}}
_ENV = ('DNG_HOSTCHECK_FAST', 'DNG_HOSTCHECK_TMPL', 'DNG_HOSTCHECK_F',
        'DNG_HOSTCHECK_JIT')

_CORPORA = {}
_ORACLE = {}


def sweep(seed, tmp_path_factory):
    if seed not in _CORPORA:
        recs = corpus.value_sweep_records(seed, N)
        p = tmp_path_factory.mktemp('sweep') / ('sweep%d.log' % seed)
        p.write_bytes(b'\n'.join(corpus.value_sweep_line(r) for r in recs) +
                      b'\n')
        _CORPORA[seed] = (recs, str(p), corpus.sweep_queries(recs))
    return _CORPORA[seed]


def oracle(seed, name, plan, path):
    if (seed, name) not in _ORACLE:
        _ORACLE[seed, name] = py_engine(plan, [path])
    return _ORACLE[seed, name]


def hostcheck(plan, path, env):
    pf = path + '.plan.json'
    with open(pf, 'w') as f:
        json.dump(plan, f)
    full = {k: v for k, v in os.environ.items() if k not in _ENV}
    full.update(env)
    out = subprocess.run([build_hostcheck(), pf, path], capture_output=True,
                         check=True, env=full).stdout
    return json.loads(out)


QNAMES = sorted(corpus.sweep_queries(corpus.value_sweep_records(0, 50)))


@pytest.mark.parametrize('seed', SEEDS)
@pytest.mark.parametrize('mode', sorted(MODES))
def test_value_sweep_in_every_parser_mode(mode, seed, tmp_path_factory):
    recs, path, queries = sweep(seed, tmp_path_factory)
    for name in QNAMES:
        argv, ds, _, _ = queries[name]
        plan = corpus.make_plan(argv, ds)
        exp_p, exp_c = oracle(seed, name, plan, path)
        doc = hostcheck(plan, path, MODES[mode])
        assert doc['counters']['unsupported'] == 0, (name, doc['counters'])
        act_p, act_c = _decode_doc(plan, doc)
        assert canon_points(act_p) == canon_points(exp_p), (mode, name)
        assert act_c == exp_c, (mode, name)
        if mode in ('fpath', 'jit'):
            # the F path decides every record but those it hands over by
            # design: escaped strings it reads, non-integer discrete keys
            need = corpus.sweep_f_decided(recs, argv)
            assert doc['nfmatch'] >= need, (name, doc['nfmatch'], need)


@pytest.mark.parametrize('seed', SEEDS)
def test_oracles_agree_with_each_other_and_the_second_reference(
        seed, tmp_path_factory):
    recs, path, queries = sweep(seed, tmp_path_factory)
    for name in QNAMES:
        argv, ds, kind, arg = queries[name]
        plan = corpus.make_plan(argv, ds)
        exp_p, exp_c = oracle(seed, name, plan, path)
        cpp_p, cpp_c = cpp_engine(plan, [path])
        assert canon_points(cpp_p) == canon_points(exp_p), name
        assert cpp_c == exp_c, name
        if kind:
            assert corpus.sweep_points(exp_p, kind, arg) == \
                corpus.sweep_reference(recs, kind, arg), name


def test_sweep_reaches_its_edges():
    """What the sweep is for is in it: 16-digit integers above 2^53, day 29-31
    carries, 23:59:59.999, escaped and raw strings on both sides of the
    surrogate range, numeric constants and their neighbours."""
    recs = corpus.value_sweep_records(0, 200000)
    nums = [r['num'] for r in recs]
    big16 = [t for t in nums if len(t) == 16 and t.isdigit() and
             int(t) > corpus.TWO53 and float(t) != int(t)]
    assert len(big16) > 1000
    assert {'-0', '0.0', '-0.0', '1e309', '5e-324'} <= set(nums)
    c = corpus.SWEEP_CONST
    import math
    for x in (c, math.nextafter(c, 0), math.nextafter(c, math.inf)):
        assert repr(x) in nums
    dates = [r['date'] for r in recs if r['date']]
    assert any(d[2] == 31 and d[1] in (4, 6, 9, 11) for d in dates)
    assert any(d[2] in (29, 30, 31) and d[1] == 2 for d in dates)
    assert any(d[3:7] == (23, 59, 59, 999) for d in dates)
    assert any(d[0] == 0 for d in dates) and any(d[0] == 9999 for d in dates)
    strs = ''.join(corpus._str_value(r) for r in recs)
    assert {'｡', '\U0001f600', '\U0010ffff', ''} <= set(strs)
    assert sum(r['str_esc'] for r in recs) > 1000
    lens = [len(corpus.value_sweep_line(r)) for r in recs[:5000]]
    assert 120 <= min(lens) and max(lens) <= 210


def test_reference_quirk_of_one_character_breakdowns():
    """dn drops a trailing bare breakdown of one character (the reference's
    attrsParse); make_plan refuses such a query unless told the drop is
    meant, and a trailing comma keeps the name."""
    assert corpus.make_plan(['-b', 'a'], allow_dropped=True)['breakdowns'] == []
    with pytest.raises(corpus.DroppedBreakdown):
        corpus.make_plan(['-b', 'a'])
    with pytest.raises(corpus.DroppedBreakdown):
        corpus.make_plan(['-b', 'ts[date,field=t],a'])
    assert [b['name'] for b in corpus.make_plan(['-b', 'a,'])['breakdowns']] \
        == ['a']
    assert [b['name'] for b in corpus.make_plan(
        ['-b', 'b[aggr=lquantize,step=7],a,'])['breakdowns']] == ['b', 'a']
    assert [b['name'] for b in corpus.make_plan(
        ['-b', 'ab', '-b', 'a.b[aggr=quantize]'])['breakdowns']] == \
        ['ab', 'a.b']
