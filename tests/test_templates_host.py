"""Record templates (csrc/tmpl.*), host side: the lexical skeletons, the trie
builder and the matcher compiled for the host by tests/hostcheck (TEST ONLY).
What they produce is compared with the oracle in test_hostcheck_*.py; here the
point is coverage: that the shapes one expects to be templated are."""

import json
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import build_hostcheck  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run_tmpl(plan, path, tmp_path):
    exe = build_hostcheck()
    pf = tmp_path / 'plan.json'
    pf.write_text(json.dumps(plan))
    env = dict(os.environ, DNG_HOSTCHECK_TMPL='1', DNG_HOSTCHECK_FAST='1',
               DNG_HOSTCHECK_TMPL_DEBUG='1')
    r = subprocess.run([exe, str(pf), path], capture_output=True, env=env,
                       check=True)
    return json.loads(r.stdout), r.stderr.decode()


@pytest.mark.parametrize('name', sorted(corpus.BASELINE_QUERIES))
def test_generated_workload_is_fully_templated(name, tmp_path):
    """mktestdata-shaped records have three shapes (caller string / null /
    absent): every record must be taken by a template, whatever the query."""
    from dragnet_b200 import native
    n = 5000
    p = tmp_path / 'gen.log'
    p.write_bytes(native.gen_host(native.gen_params(total_records=n), 0, n))
    argv, ds = corpus.BASELINE_QUERIES[name]
    doc, dbg = run_tmpl(corpus.make_plan(argv, ds), str(p), tmp_path)
    assert doc['counters']['lines'] == n
    assert doc['ntmpl'] == n, dbg
    assert '3 leaves' in dbg, dbg


def test_shapes_that_cannot_be_templates_fall_through(tmp_path):
    """A plan slot that is an array length (an inline constant) or an invalid
    sample line yields no template; escapes and odd numbers in VALUES do not
    stop a record from matching one."""
    lines = [b'{"a":[1,2,3],"s":"x"}'] * 40 + \
            [b'{"a":"v\\u0041","n":1.5e3}', b'{"a":"w\\\\\\"","n":-0}'] * 20 + \
            [b'{"a":"v","n":}'] * 5
    p = tmp_path / 'mix.log'
    p.write_bytes(b'\n'.join(lines) + b'\n')
    doc, dbg = run_tmpl(corpus.make_plan(['-b', 'a.length']), str(p), tmp_path)
    # the array shape needs index semantics: never templated
    assert doc['ntmpl'] == 40, (doc['ntmpl'], dbg)
    assert doc['counters']['invalid_json'] == 5
    doc, dbg = run_tmpl(corpus.make_plan(['-b', 'a,n,']), str(p), tmp_path)
    assert doc['ntmpl'] == 80, (doc['ntmpl'], dbg)


def test_optional_fields_make_a_branching_trie(tmp_path):
    """Four optional fields -> sixteen shapes sharing prefixes: all of them are
    templated (sibling dispatch + alt chains), and the answers are the
    oracle's."""
    import random
    from engines import canon_points, hostcheck_engine, py_engine
    rng = random.Random(11)
    lines = []
    for i in range(4000):
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
    p = tmp_path / 'opt.log'
    p.write_bytes(b'\n'.join(lines) + b'\n')
    plan = corpus.make_plan(['-b', 'a,b.c,d,'])
    doc, dbg = run_tmpl(plan, str(p), tmp_path)
    assert doc['ntmpl'] == len(lines), (doc['ntmpl'], dbg)
    assert '16 leaves' in dbg, dbg
    os.environ['DNG_HOSTCHECK_TMPL'] = '1'
    try:
        act_p, act_c = hostcheck_engine(plan, [str(p)])
    finally:
        del os.environ['DNG_HOSTCHECK_TMPL']
    exp_p, exp_c = py_engine(plan, [str(p)])
    assert canon_points(act_p) == canon_points(exp_p)
    assert act_c == exp_c
