"""Device per-record logic (host-compiled, TEST ONLY) vs the Python oracle on
edge-case and randomized inputs: JSON grammar corners, escapes, duplicate
keys, pluck precedence, JS number/string coercions, dates, json-skinner."""

import os
import sys

import pytest


@pytest.fixture(params=['general', 'fast', 'tmpl', 'fpath', 'jit'], autouse=True)
def parser_mode(request, monkeypatch):
    """Run every case with the general parser only, with the lock-step fast
    automaton (+ fallback), and with record templates learned from the input
    in front of both -- the three tiers the general kernels use -- and with the
    F path (fast.cuh: path-indexed templates, lean stages, piece-wise keys) in
    front of all of them, as scan_kernel_f does."""
    monkeypatch.delenv('DNG_HOSTCHECK_FAST', raising=False)
    monkeypatch.delenv('DNG_HOSTCHECK_TMPL', raising=False)
    monkeypatch.delenv('DNG_HOSTCHECK_F', raising=False)
    monkeypatch.delenv('DNG_HOSTCHECK_JIT', raising=False)
    if request.param in ('fpath', 'jit'):
        monkeypatch.setenv('DNG_HOSTCHECK_F', '1')
    if request.param == 'jit':
        # + the matcher jit.cpp generates for the templates: built for the
        # device (NVRTC + nvJitLink, no GPU needed) and run on the host
        monkeypatch.setenv('DNG_HOSTCHECK_JIT', '1')
    if request.param in ('fast', 'tmpl'):
        monkeypatch.setenv('DNG_HOSTCHECK_FAST', '1')
    if request.param == 'tmpl':
        monkeypatch.setenv('DNG_HOSTCHECK_TMPL', '1')

sys.path.insert(0, os.path.dirname(__file__))
import corpus  # noqa: E402
from engines import canon_points, hostcheck_engine, py_engine  # noqa: E402


def _write(tmp_path, name, lines):
    p = tmp_path / name
    p.write_bytes(b'\n'.join(lines) + b'\n')
    return str(p)


def _compare(plan, path):
    exp_p, exp_c = py_engine(plan, [path])
    act_p, act_c = hostcheck_engine(plan, [path])
    assert canon_points(act_p) == canon_points(exp_p), plan
    assert act_c == exp_c, plan


@pytest.mark.parametrize('qi', range(len(corpus.EDGE_QUERIES)))
def test_edge_lines(qi, tmp_path):
    argv, ds = corpus.EDGE_QUERIES[qi]
    path = _write(tmp_path, 'edge.log', corpus.EDGE_LINES)
    _compare(corpus.make_plan(argv, ds), path)


@pytest.mark.parametrize('qi', range(len(corpus.SKINNER_QUERIES)))
def test_skinner_lines(qi, tmp_path):
    argv, ds = corpus.SKINNER_QUERIES[qi]
    path = _write(tmp_path, 'sk.log', corpus.SKINNER_LINES)
    _compare(corpus.make_plan(argv, ds), path)


@pytest.mark.parametrize('seed', range(6))
def test_random_lines(seed, tmp_path):
    path = _write(tmp_path, 'rand.log', corpus.random_lines(seed, 400))
    for argv, ds in corpus.EDGE_QUERIES[:24:3]:
        _compare(corpus.make_plan(argv, ds), path)


@pytest.mark.parametrize('rot', [24, 48, 72, 96, 120, 144])
def test_edge_lines_rotated(rot, tmp_path):
    """Templates are learned from the head of the input: rotate the corpus so
    that every odd shape gets to be a template once."""
    lines = corpus.EDGE_LINES[rot:] + corpus.EDGE_LINES[:rot]
    path = _write(tmp_path, 'edge.log', lines)
    for argv, ds in corpus.EDGE_QUERIES[::3]:
        _compare(corpus.make_plan(argv, ds), path)


def test_scalar_forms_behind_one_template(tmp_path):
    """Every number / literal / string-body form in the same record shape: in
    template mode the first lines make the template and all others meet its
    wildcard scans."""
    lines = [b'{"a":7,"s":"k0"}'] * 3 + corpus.scalar_lines()
    path = _write(tmp_path, 'scalars.log', lines)
    for argv in (['-b', 'a,'], ['-b', 's,'], ['-b', 'a[aggr=quantize]'],
                 ['-b', 'a,s,', '-f', '{"ge":["a",1]}']):
        _compare(corpus.make_plan(argv), path)


@pytest.mark.parametrize('seed', range(8))
def test_template_fuzz(seed, tmp_path):
    """A few shapes, re-rolled scalars, some damage (corpus.template_fuzz_lines):
    in template mode most lines meet a learned template."""
    path = _write(tmp_path, 'fz.log', corpus.template_fuzz_lines(seed, 800))
    for argv, ds in corpus.EDGE_QUERIES[:30:4]:
        _compare(corpus.make_plan(argv, ds), path)


def test_legacy_date_strings_are_refused_not_dropped(tmp_path):
    """A date string outside the ES5 format that V8's legacy Date.parse might
    accept is neither parsed nor called NaN: the device code flags the record
    unsupported (the scan then fails with DNG_EUNSUPPORTED) and the oracle
    raises; anything that does not even look like such a form is NaN
    (`baddate`) in both."""
    import json
    import subprocess
    import dn_oracle
    from engines import build_hostcheck
    lines = [b'{"time":"2014-05-01T00:00:00Z","a":1}',
             b'{"time":"nonsense","a":1}', b'{"time":" 12 ,x"}',
             b'{"time":"gurble 7"}']
    plan = corpus.make_plan(
        ['-b', 'ts[date,field=time,aggr=lquantize,step=86400]'])
    p = tmp_path / 'ok.log'
    p.write_bytes(b'\n'.join(lines) + b'\n')
    _compare(plan, str(p))
    for bad in (b'Thu, 01 May 2014 00:00:00 GMT', b'2014-05-01 12:00:00',
                b'May 1, 2014', b'2014-13-45'):
        q = tmp_path / 'bad.log'
        q.write_bytes(b'\n'.join(lines + [b'{"time":"' + bad + b'"}']) + b'\n')
        with pytest.raises(dn_oracle.Unsupported):
            py_engine(plan, [str(q)])
        pf = tmp_path / 'plan.json'
        pf.write_text(json.dumps(plan))
        out = subprocess.run([build_hostcheck(), str(pf), str(q)],
                             capture_output=True, env=dict(os.environ),
                             check=True).stdout
        assert json.loads(out)['counters']['unsupported'] == 1, bad
    # day 30 of February carries over (V8), it is not NaN
    r = tmp_path / 'feb.log'
    r.write_bytes(b'{"time":"2014-02-30T00:00:00Z"}\n'
                  b'{"time":"2014-03-02T00:00:00Z"}\n')
    exp_p, _ = py_engine(plan, [str(r)])
    assert [v for _, v in exp_p] == [2]
    _compare(plan, str(r))
