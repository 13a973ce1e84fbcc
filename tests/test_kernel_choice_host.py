"""Which kernel a scan launches (dragnet_b200/csrc/kernel_choice.h), on the
CPU: the policy compiled with a small driver (tests/hostcheck/
kernel_choice_check.cpp) and stepped through opens, samples and counter
snapshots.  The limits come from the header itself."""

import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'dragnet_b200', 'csrc')
DRIVER = os.path.join(ROOT, 'tests', 'hostcheck', 'kernel_choice_check.cpp')


@pytest.fixture(scope='module')
def kc(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp('kc') / 'kernel_choice_check')
    subprocess.check_call(['g++', '-std=c++17', '-O1', '-Wall', '-Werror',
                           '-I', CSRC, '-o', exe, DRIVER])

    def run(*cmds):
        r = subprocess.run([exe], input='\n'.join(cmds) + '\n',
                           capture_output=True, text=True, check=True)
        return [{k: int(v) if v.isdigit() else v
                 for k, v in (kv.split('=') for kv in line.split())}
                for line in r.stdout.splitlines()]
    return run


@pytest.fixture(scope='module')
def C(kc):
    return kc('const')[0]


def op(fanout=0, modelled=1, f_fits=1, w_fits=1, kernel='-', fast='-',
       f_warps='-'):
    return 'open %d %d %d %d %s %s %s' % (fanout, modelled, f_fits, w_fits,
                                          kernel, fast, f_warps)


def smp(length, count=400, long=0, learned=1, blob=1, covered=None,
        lines=None):
    n = count + (1 if long else 0)
    return 'sample %d %d %d %d %d %d %d' % (
        count, length, long, learned, blob, n if covered is None else covered,
        n if lines is None else lines)


def live(lines, long=0, tmpl=0, aggr=0, over=0, templates=1):
    return 'live %d %d %d %d %d %d' % (lines, long, tmpl, aggr, over,
                                       templates)


def f_edge(C):
    """The shortest line (without its newline) that lets the F path in: a
    chunk of the narrowest lane slice must hold the records its newline index
    was sized for, with half again to spare."""
    nsl = 112 // 16
    return int(32 * 16 * nsl * 1.5 / C['f_nlcap']) - 1


# -- at open ------------------------------------------------------------------

@pytest.mark.parametrize('fanout,kernel,mode', [
    (0, '-', 'auto'), (1, '-', 'tile'),
    (0, 'tile', 'tile'), (0, 'warp', 'warp'), (0, 'fast', 'fast'),
    (1, 'warp', 'warp'), (1, 'fast', 'fast'),
    # any other value is auto, even for a fan-out plan
    (1, 'auto', 'auto'), (0, 'bogus', 'auto'),
])
def test_open_mode(kc, fanout, kernel, mode):
    s = kc(op(fanout=fanout, kernel=kernel))[0]
    assert s['mode'] == mode
    assert s['warp'] == (mode == 'warp')
    assert s['f'] == (mode == 'fast')
    assert s['pick'] == {'fast': 'f', 'warp': 'warp'}.get(mode, 'tile')


@pytest.mark.parametrize('fanout', [0, 1])
@pytest.mark.parametrize('modelled,fast', [(0, '-'), (1, '0'), (0, '1'),
                                           (1, 'no')])
def test_fast_forced_but_not_eligible(kc, fanout, modelled, fast):
    s = kc(op(fanout=fanout, modelled=modelled, kernel='fast', fast=fast))[0]
    assert s['mode'] == ('tile' if fanout else 'auto')
    assert s['f'] == 0 and s['pick'] == 'tile'


def test_fast_setting_other_than_zero_keeps_the_f_path(kc):
    s = kc(op(kernel='fast', fast='1'))[0]
    assert s['mode'] == 'fast' and s['pick'] == 'f'


@pytest.mark.parametrize('kernel,mode,pick', [
    ('-', 'tile', 'tile'), ('warp', 'tile', 'tile'), ('tile', 'tile', 'tile'),
    ('fast', 'fast', 'f')])
def test_warp_geometry_does_not_fit(kc, C, kernel, mode, pick):
    s = kc(op(w_fits=0, kernel=kernel), smp(100))
    assert [x['mode'] for x in s] == [mode, mode]
    assert [x['pick'] for x in s] == [pick, pick]


def test_fast_forced_but_f_buffers_do_not_fit(kc):
    s = kc(op(kernel='fast', f_fits=0), smp(100))
    # the tile kernel, not auto: short lines do not bring the warp kernel
    assert [x['mode'] for x in s] == ['fast', 'fast']
    assert [x['pick'] for x in s] == ['tile', 'tile']


def test_auto_f_buffers_do_not_fit(kc, C):
    s = kc(op(f_fits=0), smp(100))[-1]
    assert s['warp'] == 1 and s['f'] == 0 and s['pick'] == 'warp'


@pytest.mark.parametrize('f_warps,nw', [(None, 'f_nw_start'),
                                        ('28', 'f_nw'), ('32', 'f_nw'),
                                        ('27', 'f_nw_start'),
                                        ('24', 'f_nw_start')])
def test_open_f_warps(kc, C, f_warps, nw):
    assert kc(op(f_warps=f_warps or '-'))[0]['f_nw'] == C[nw]


# -- samples ------------------------------------------------------------------

@pytest.mark.parametrize('kernel', ['tile', 'warp', 'fast'])
def test_forced_modes_with_templates_off_take_no_sample(kc, C, kernel):
    s = kc(op(kernel=kernel))[0]
    assert s['sample_notmpl'] == 0 and s['sample_tmpl'] == 1
    # nothing is learned: the geometry keeps its defaults
    assert s['wslice'] == C['w_slice_max']
    assert s['f_nsl'] == C['w_slice_max'] // 16


def test_auto_takes_a_sample_with_templates_off(kc):
    s = kc(op())[0]
    assert s['sample_notmpl'] == 1 and s['sample_tmpl'] == 1


@pytest.mark.parametrize('kernel,pick', [('tile', 'tile'), ('warp', 'warp')])
def test_forced_mode_learns_slices_not_the_kernel(kc, C, kernel, pick):
    s = kc(op(kernel=kernel), smp(C['w_maxline'] + 1), smp(20))
    assert [x['pick'] for x in s] == [pick] * 3
    assert s[2]['f_nsl'] == 112 // 16


@pytest.mark.parametrize('extra,warp', [(0, 1), (1, 0)])
def test_sample_longest_line(kc, C, extra, warp):
    s = kc(op(), smp(100, long=C['w_maxline'] + extra, learned=0))[-1]
    assert s['warp'] == warp and s['pick'] == ('warp' if warp else 'tile')


def test_short_then_long_then_short_lines(kc, C):
    """Warp goes off on a sample with long lines and stays off."""
    s = kc(op(), smp(100), 'rebase 0 0',
           smp(100, long=C['w_maxline'] + 1), 'rebase 0 0', smp(100))
    assert [x['warp'] for x in s] == [0, 1, 1, 0, 0, 0]


def test_lane_slices(kc, C):
    # long lines: the widest slice; F: at most f_nlcap records a chunk
    s = kc(op(), smp(2000, count=8, learned=0))[-1]
    assert s['wslice'] == C['w_slice_max']
    assert s['f_nsl'] == C['w_slice_max'] // 16
    s = kc(op(), smp(20, learned=0))[-1]
    assert s['f_nsl'] == 112 // 16
    # every slice is 16 x an odd number
    for n in (20, 60, 100, 300):
        s = kc(op(), smp(n, learned=0))[-1]
        assert s['wslice'] % 32 == 16 and s['f_nsl'] % 2 == 1
        assert s['f_nsl'] * 16 <= s['wslice']


def test_f_from_sample(kc, C):
    assert kc(op(), smp(100))[-1]['pick'] == 'f'
    # no blob, or coverage under 90 %
    assert kc(op(), smp(100, blob=0))[-1]['pick'] == 'warp'
    assert kc(op(), smp(100, covered=90, lines=100))[-1]['pick'] == 'f'
    assert kc(op(), smp(100, covered=89, lines=100))[-1]['pick'] == 'warp'
    assert kc(op(), smp(100, covered=899, lines=1000))[-1]['pick'] == 'warp'
    # long lines
    s = kc(op(), smp(100, long=C['w_maxline'] + 1))[-1]
    assert s['f'] == 0 and s['pick'] == 'tile'
    s = kc(op(), smp(100, long=C['w_maxline']))[-1]
    assert s['pick'] == 'f'


def test_f_needs_lines_long_enough(kc, C):
    e = f_edge(C)
    s = kc(op(), smp(e))[-1]
    assert s['f_nsl'] == 112 // 16 and s['pick'] == 'f'
    s = kc(op(), smp(e - 1))[-1]
    assert s['f_nsl'] == 112 // 16 and s['pick'] == 'warp'


@pytest.mark.parametrize('kernel', ['tile', 'warp'])
def test_forced_modes_never_take_f_from_a_sample(kc, kernel):
    assert kc(op(kernel=kernel), smp(100))[-1]['f'] == 0


def test_sample_without_candidates_leaves_f(kc):
    s = kc(op(), smp(100), smp(100, learned=0, blob=0, covered=0))
    assert [x['f'] for x in s] == [0, 1, 1]
    s = kc(op(), smp(100, blob=0), smp(100, learned=0))
    assert [x['f'] for x in s] == [0, 0, 0]


def test_relearn_after_warp_off_brings_f_back(kc, C):
    """A relearn's own line test decides F even when warp is already off."""
    s = kc(op(), smp(100, long=C['w_maxline'] + 1), live(200001),
           smp(100), 'rebase 200001 0')
    assert [x['pick'] for x in s] == ['tile', 'tile', 'tile', 'f', 'f']
    assert s[-1]['warp'] == 0 and s[2]['relearn'] == 1


# -- counters of finished launches --------------------------------------------

@pytest.mark.parametrize('lines,long,warp', [
    (64, 5, 0), (64, 4, 1), (63, 63, 1), (1008, 63, 1), (1007, 63, 0)])
def test_long_lines_turn_warp_off(kc, lines, long, warp):
    s = kc(op(), smp(100, blob=0), live(lines, long=long))[-1]
    assert s['warp'] == warp


def test_warp_off_is_sticky_and_counted_since_last_look(kc):
    s = kc(op(), smp(100, blob=0), live(64, long=4), live(128, long=9),
           live(1000, long=9), live(2000, long=9))
    assert [x['warp'] for x in s[2:]] == [1, 0, 0, 0]
    # new lines only: 60 long in the first look do not count again
    s = kc(op(), smp(100, blob=0), live(1000, long=60), live(1064, long=60))
    assert [x['warp'] for x in s[2:]] == [1, 1]


@pytest.mark.parametrize('kernel', ['warp'])
def test_forced_warp_is_kept_on_long_lines(kc, kernel):
    s = kc(op(kernel=kernel), live(1000, long=1000))[-1]
    assert s['warp'] == 1 and s['pick'] == 'warp'


def test_f_warps_drop_on_overflow(kc, C):
    s = kc(op(f_warps='28'), live(10, aggr=4096, over=65))[-1]
    assert s['f_nw'] == C['f_nw_start']
    s = kc(op(f_warps='28'), live(10, aggr=4096, over=64))[-1]
    assert s['f_nw'] == C['f_nw']
    s = kc(op(f_warps='28'), live(10, aggr=4095, over=4095))[-1]
    assert s['f_nw'] == C['f_nw']
    # over the launches since the last look only
    s = kc(op(f_warps='28'), live(10, aggr=4096, over=64),
           live(10, aggr=8192, over=128), live(10, aggr=12288, over=193))
    assert [x['f_nw'] for x in s[1:]] == [C['f_nw'], C['f_nw'],
                                          C['f_nw_start']]


def test_f_gives_up_then_comes_back(kc, C):
    d = 200001
    s = kc(op(), smp(100),
           # many records miss the F templates: learn again first
           live(d, tmpl=d * 9 // 10), smp(100), 'rebase %d %d' % (d, d * 9 // 10),
           # and again: now the F path gives up, nothing more to learn
           live(2 * d, tmpl=d * 9 // 10 + d * 9 // 10),
           # most records untemplated: a relearn may turn it on again
           live(3 * d + 1, tmpl=d * 9 // 10 * 2), smp(100))
    assert [x['relearn'] for x in s] == [0, 0, 1, 0, 0, 0, 1, 0]
    assert [x['pick'] for x in s] == ['tile', 'f', 'f', 'f', 'f', 'warp',
                                      'warp', 'f']


def test_f_gives_up_only_after_a_relearn(kc):
    d = 200001
    s = kc(op(), smp(100), live(d, tmpl=d * 9 // 10))[-1]
    assert s['f'] == 1 and s['relearn'] == 1
    s = kc(op(), smp(100), live(d, tmpl=d * 9 // 10), 'rebase 0 0',
           live(d, tmpl=d * 9 // 10))[-1]
    assert s['f'] == 0 and s['relearn'] == 0
    # not when few records miss
    s = kc(op(), smp(100), live(d, tmpl=d * 9 // 10), 'rebase 0 0',
           live(d, tmpl=d - d // 16))[-1]
    assert s['f'] == 1 and s['relearn'] == 0
    # nor within 200 000 lines of the last learn
    s = kc(op(), smp(100), live(d, tmpl=d * 9 // 10), 'rebase 1 0',
           live(d, tmpl=d * 9 // 10))[-1]
    assert s['f'] == 1 and s['relearn'] == 0


def test_forced_fast_never_gives_up(kc):
    d = 200001
    s = kc(op(kernel='fast'), live(d), 'rebase 0 0', live(d), live(d * 3))
    assert [x['pick'] for x in s] == ['f'] * 5
    assert [x['relearn'] for x in s] == [0, 1, 0, 1, 1]


@pytest.mark.parametrize('lines,tmpl,templates,relearn', [
    (200001, 0, 1, 1), (200000, 0, 1, 0), (200001, 100000, 1, 1),
    (200001, 100001, 1, 0), (200002, 100001, 1, 0), (200001, 0, 0, 0)])
def test_relearn_condition(kc, lines, tmpl, templates, relearn):
    s = kc(op(), smp(100, blob=0), live(lines, tmpl=tmpl,
                                        templates=templates))[-1]
    assert s['relearn'] == relearn and s['relearns'] == relearn


def test_relearn_when_f_is_weak(kc):
    """F on and more than 1/16 of records missing: learn again even though
    most records are templated."""
    d = 200001
    assert kc(op(), smp(100), live(d, tmpl=d - d // 16 + 1))[-1]['relearn'] == 0
    assert kc(op(), smp(100), live(d, tmpl=d - d // 15))[-1]['relearn'] == 1
    # exactly 1/16 missing is not weak
    d = 200016
    assert kc(op(), smp(100), live(d, tmpl=d - d // 16))[-1]['relearn'] == 0
    assert kc(op(), smp(100, blob=0),
              live(d, tmpl=d - d // 15))[-1]['relearn'] == 0


def test_relearns_at_most_three(kc):
    d = 200001
    cmds = [op(kernel='tile')]
    for i in range(1, 6):
        cmds += [live(d * i), 'rebase %d 0' % (d * i)]
    s = kc(*cmds)
    assert [x['relearn'] for x in s[1::2]] == [1, 1, 1, 0, 0]
    assert s[-1]['relearns'] == 3
