"""krill filters (corpus.filter_lines: a field `v` in every value form, the
comparison matrix, random predicate trees, datasource + user + time-bound
programs in one plan) through the device per-record logic compiled for the
host (TEST ONLY), in every parser mode, against the Python oracle; the
oracle itself against the C++ one and against a second reference written
from ECMA-262 (corpus.krill_reference).  Also every limit of the plan
compiler, of the F plan and of the key automaton, at the limit and one past
it."""

import json
import os
import random
import subprocess
import sys
from collections import Counter

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import (_decode_doc, build_hostcheck, canon_points,  # noqa: E402
                     cpp_engine, py_engine)
from dragnet_b200 import native  # noqa: E402

SEED = 0
N = 3000
MODES = {'general': {}, 'fast': {'DNG_HOSTCHECK_FAST': '1'},
         'tmpl': {'DNG_HOSTCHECK_FAST': '1', 'DNG_HOSTCHECK_TMPL': '1'},
         'fpath': {'DNG_HOSTCHECK_F': '1'},
         'jit': {'DNG_HOSTCHECK_F': '1', 'DNG_HOSTCHECK_JIT': '1'}}
_ENV = ('DNG_HOSTCHECK_FAST', 'DNG_HOSTCHECK_TMPL', 'DNG_HOSTCHECK_F',
        'DNG_HOSTCHECK_JIT')

QUERIES = corpus.filter_queries()
QNAMES = sorted(QUERIES)
_ORACLE = {}


@pytest.fixture(scope='module')
def filters(tmp_path_factory):
    recs = corpus.filter_records(SEED, N)
    p = tmp_path_factory.mktemp('filters') / 'filters.log'
    p.write_bytes(b'\n'.join(corpus.filter_line(r) for r in recs) + b'\n')
    return recs, str(p)


def oracle(plan, path):
    """The Python oracle's (points, counters), once per plan and input."""
    key = (json.dumps(plan, sort_keys=True), path)
    if key not in _ORACLE:
        _ORACLE[key] = py_engine(plan, [path])
    return _ORACLE[key]


def hostcheck(plan, path, env):
    pf = path + '.plan.json'
    with open(pf, 'w') as f:
        json.dump(plan, f)
    full = {k: v for k, v in os.environ.items() if k not in _ENV}
    full.update(env)
    out = subprocess.run([build_hostcheck(), pf, path], capture_output=True,
                         check=True, env=full).stdout
    return json.loads(out)


def check_mode(name, argv, ds, path, mode):
    plan = corpus.make_plan(argv, ds)
    exp_p, exp_c = oracle(plan, path)
    doc = hostcheck(plan, path, MODES[mode])
    assert doc['counters']['unsupported'] == 0, (name, doc['counters'])
    act_p, act_c = _decode_doc(plan, doc)
    assert canon_points(act_p) == canon_points(exp_p), (mode, name)
    assert act_c == exp_c, (mode, name)
    return doc


@pytest.mark.parametrize('mode', sorted(MODES))
def test_filters_in_every_parser_mode(mode, filters):
    recs, path = filters
    for name in QNAMES:
        argv, ds, _, _, _ = QUERIES[name]
        doc = check_mode(name, argv, ds, path, mode)
        if mode in ('fpath', 'jit') and corpus.query_leaves(
                QUERIES[name]) <= 16:
            # a plan of at most 16 leaves is the F path's: it decides
            # records itself (all but escaped strings and containers it
            # reaches)
            assert doc['nfmatch'] > 0, (name, doc['nfmatch'])


def test_oracles_agree_with_each_other_and_the_second_reference(
        filters):
    recs, path = filters
    for name in QNAMES:
        argv, ds, pred, dsp, bounds = QUERIES[name]
        plan = corpus.make_plan(argv, ds)
        exp_p, exp_c = oracle(plan, path)
        cpp_p, cpp_c = cpp_engine(plan, [path])
        assert canon_points(cpp_p) == canon_points(exp_p), name
        assert cpp_c == exp_c, name
        tally, split = corpus.krill_reference(recs, pred, dsp, bounds)
        assert corpus.tag_points(exp_p) == tally, name
        for stage, want in split.items():
            assert corpus.filter_split(exp_c, stage) == want, (name, stage)
        assert exp_c['json parser'].get('invalid json', 0) == \
            sum(1 for r in recs if r['damage']), name


def test_combined_programs_share_one_code_array():
    """The datasource filter, the user filter and the two time-bound leaves
    are compiled into one code[]: 16 and 17 leaves in all, on either side of
    the F path's 16."""
    for name, total in (('comb16', 16), ('comb17', 17)):
        assert corpus.query_leaves(QUERIES[name]) == total
        plan = corpus.make_plan(*QUERIES[name][:2])
        assert plan['ds_filter'] and plan['filter'] and plan['time_bounds']


def _plan_error(argv):
    with pytest.raises(native.DngError) as ei:
        native.Plan(json.dumps(corpus.make_plan(argv)))
    return ei.value


@pytest.mark.parametrize('limit', sorted(corpus.PLAN_LIMITS))
def test_plan_limit(limit, filters):
    """At the limit the plan compiles and scans as the oracle does; one past
    it, plan creation fails with DNG_ELIMIT and plan.cpp's message."""
    at, over, msg = corpus.PLAN_LIMITS[limit]
    recs, path = filters
    native.Plan(json.dumps(corpus.make_plan(at)))
    check_mode('limit_' + limit, at, None, path, 'general')
    e = _plan_error(over)
    assert e.code == -7, e
    assert str(e) == 'libdragnet_gpu: %s (ELIMIT)' % msg, e


def test_plan_limit_leaves_count_every_program():
    """The 48 leaves are shared by the datasource filter, the user filter
    and the time bounds: 46 + 2 compile, 47 + 2 do not."""
    for n, ok in ((46, True), (47, False)):
        pred = corpus.random_predicate(random.Random(n), n, ('v',))
        argv = ['-f', json.dumps(pred),
                '-b', 'tag,', '--after', corpus.FILTER_AFTER, '--before',
                corpus.FILTER_BEFORE]
        plan = corpus.make_plan(argv, {'timeField': 't'})
        if ok:
            native.Plan(json.dumps(plan))
        else:
            with pytest.raises(native.DngError) as ei:
                native.Plan(json.dumps(plan))
            assert 'filter too large' in str(ei.value)


@pytest.mark.parametrize('limit', sorted(corpus.F_LIMITS))
def test_f_plan_limit(limit, filters):
    """At each limit of fplan_build the F path takes the plan and decides
    records; one past it the plan is not the F path's, and every record
    goes to the general code.  Results equal the oracle's both ways."""
    at, over = corpus.F_LIMITS[limit]
    recs, path = filters
    doc = check_mode('f_' + limit, at, None, path, 'fpath')
    assert doc['nfmatch'] > 0, (limit, doc)
    doc = check_mode('f_over_' + limit, over, None, path, 'fpath')
    assert doc['nfmatch'] == 0, (limit, doc)


def test_f_plan_limit_pool_bytes():
    """The pool case sits where it says: constants padded to 4-byte words
    fill 484 of the 512 bytes after the 28-byte header, then 488."""
    for argv, want in zip(corpus.F_LIMITS['pool_484'], (484, 488)):
        cs = [leaf['eq'][1] for leaf in json.loads(argv[1])['or']]
        assert len(cs) == 16
        assert sum((len(c) + 3) & ~3 for c in cs) == want


@pytest.mark.parametrize('limit', sorted(corpus.AUTOMATON_LIMITS))
def test_automaton_limit(limit, filters):
    """Plans the key automaton cannot express are parsed by the general
    parser alone, with the oracle's results."""
    recs, path = filters
    doc = check_mode('auto_' + limit, corpus.AUTOMATON_LIMITS[limit], None,
                     path, 'fast')
    assert doc['nfast'] == 0, (limit, doc['nfast'])
    # (a small plan over the same fields does take the automaton)
    doc = check_mode('eq_26', ['-f', '{"eq":["v",26]}', '-b', 'tag,'], None,
                     path, 'fast')
    assert doc['nfast'] > 0


def test_filter_corpus_reaches_its_forms():
    """Every form of v in at least 1 % of records, opt in two shapes of four,
    a.b both nested and as a literal key, about 1 % damaged lines, and
    undamaged lines of 120-220 bytes."""
    recs = corpus.filter_records(SEED, 30000)
    forms = Counter(r['tag'] for r in recs)
    assert set(forms) == {t for t, _, _ in corpus.V_FORMS}
    assert min(forms.values()) >= 300, forms
    assert {r['shape'] for r in recs if r['opt'] is corpus.MISSING} == {1, 3}
    assert any(b'"a.b":' in corpus.filter_line(r) for r in recs[:50])
    assert 150 <= sum(1 for r in recs if r['damage']) <= 450
    lens = [len(corpus.filter_line(r)) for r in recs if not r['damage']]
    assert 120 <= min(lens) and max(lens) <= 220
    assert {n.split('_', 1)[0] for n in QNAMES} >= set(corpus.OPS)
    sizes = [int(n.rsplit('_', 1)[1]) for n in QNAMES if n.startswith('tree')]
    assert len(sizes) >= 55 and min(sizes) == 1 and max(sizes) == 48
    assert sum(1 for s in sizes if 14 <= s <= 18) >= 20


def test_second_reference_on_known_cases():
    """krill_reference's comparisons on cases whose JavaScript answer is
    known (ECMA-262 7.2.13, 7.2.14)."""
    eq, cmp = corpus.loose_equals, corpus.js_compare
    assert eq('0x1a', 26.0) and eq(' 26 ', 26.0) and not eq('26', ' 26 ')
    assert eq([], 0.0) and eq([], '') and eq([], False) and not eq({}, 0.0)
    assert eq({}, '[object Object]') and eq([1.0, 2.0], '1,2')
    assert eq(True, '1') and eq(True, 1.0) and not eq(True, 'true')
    assert not eq(None, 0.0) and not eq(None, False) and not eq(None, '')
    assert eq(-0.0, 0.0) and eq('', 0.0) and eq('', False)
    assert eq(float(corpus.TWO53), float(corpus.TWO53 + 1))
    assert cmp('ge', None, 0.0) and cmp('le', None, 0.0)
    assert not cmp('lt', None, 'abc') and not cmp('ge', None, 'abc')
    assert cmp('lt', '\U0001f600', 'ｶﾀ')        # UTF-16: D83D < FF76
    assert cmp('gt', 'é', 'z') and cmp('lt', '', 'A')
    assert cmp('lt', [], 'A') and cmp('gt', {}, '[')
    assert not cmp('lt', 'abc', 1.0) and not cmp('ge', 'abc', 1.0)
    assert cmp('le', '26', 26.0) and cmp('lt', False, True)
