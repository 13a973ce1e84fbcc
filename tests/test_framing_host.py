"""The framing geometry test_gpu_framing.py relies on, on the CPU: the lane
slice restated in framing.py against kernel_choice.h itself (compiled with
tests/hostcheck/kernel_choice_check.cpp), the constants read from the
headers, and the layouts holding the cases they claim."""

import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
import framing  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(ROOT, 'tests', 'hostcheck', 'kernel_choice_check.cpp')


@pytest.fixture(scope='module')
def kc(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp('kc') / 'kernel_choice_check')
    subprocess.check_call(['g++', '-std=c++17', '-O1', '-Wall', '-Werror',
                           '-I', framing.CSRC, '-o', exe, DRIVER])

    def run(cmds):
        r = subprocess.run([exe], input='\n'.join(cmds) + '\n',
                           capture_output=True, text=True, check=True)
        return [dict(kv.split('=') for kv in line.split())
                for line in r.stdout.splitlines()]
    return run


def test_constants_from_the_headers(kc):
    C = framing.C
    k = kc(['const'])[0]
    assert int(k['w_slice_max']) == C['DNG_W_SLICE_MAX']
    assert int(k['f_nlcap']) == C['DNG_F_NLCAP']
    assert int(k['f_nw_start']) == C['DNG_F_NW_START']
    assert C['DNG_TILE'] == C['DNG_NT'] * 208
    assert C['DNG_MAXREC'] == 1 << 24
    # the pre-laps the layouts straddle, and the longest F line (4095) is one
    # byte short of the tile pre-lap
    assert C['F_MAXLINE'] + 1 == C['DNG_PRELAP']
    assert C['DNG_F_PRE'] < C['DNG_W_PRELAP'] < C['DNG_PRELAP']


# (count, len, long): the sample kernel_choice_check builds -- count lines of
# len bytes, then one of long bytes -- whose mean line is computed below
SAMPLES = [(400, n, 0) for n in range(8, 700, 3)] + \
          [(c, n, lng) for c in (3, 50, 333) for n in (20, 63, 90, 200)
           for lng in (1, 511, 4000)]


def test_lane_slice_matches_kernel_choice(kc):
    cmds = ['open 0 1 1 1 auto - -']
    for c, n, lng in SAMPLES:
        cmds.append('sample %d %d %d 1 1 %d %d' % (c, n, lng, c + 1, c + 1))
    out = kc(cmds)[1:]
    for (c, n, lng), o in zip(SAMPLES, out):
        nbytes = c * (n + 1) + (lng + 1 if lng else 0)
        nl = c + (1 if lng else 0)
        g = framing.geometry(nbytes / nl)
        assert int(o['wslice']) == g['wslice'], (c, n, lng)
        assert int(o['f_nsl']) == g['f_nsl'], (c, n, lng)
        assert g['f_chunk'] == 512 * g['f_nsl']
        assert g['w_chunk'] == 32 * g['wslice']


def test_sample_mean_is_the_head_of_the_launch():
    line = b'x' * 99 + b'\n'
    data = line * (framing.SAMPLE // 100 + 50) + b'y' * 10
    assert framing.sample_mean(data) == framing.SAMPLE / (framing.SAMPLE //
                                                          100)
    assert framing.sample_mean(b'no newline') == 224.0


def test_f_segment_formula():
    chunk, sms = 4608, 132
    for seg in (2, 6, 16):
        n = framing.f_bytes_for_segment(seg, chunk, sms)
        assert framing.f_segment(n, chunk, sms) == seg
        assert framing.f_segment(n - chunk, chunk, sms) == seg - 1
    # a 64 MiB ring slot (plus a carried line) never gets two
    assert framing.f_segment((64 << 20) + (16 << 20), 3584, sms) == 1
    assert framing.f_segment(10 ** 12, chunk, sms) == framing.F_SEG


@pytest.mark.parametrize('kernel', ['fast', 'warp', 'tile'])
def test_layout_holds_its_cases(kernel):
    """Every case sits where it was placed, relative to the unit the layout's
    own head gives the kernel."""
    L, g, U = framing.fixed_layout(kernel, seed=11)
    data = L.data()
    key, P, K = framing.KERNEL_UNIT[kernel]
    assert g[key] == U
    if kernel != 'tile':
        assert U % 16 == 0 and U < framing.SAMPLE
    names = set()
    for name, b in L.cases:
        names.add(name)
        assert b % U == 0 and b > 0
        if name in ('nl-1', 'nl+0', 'nl+1'):
            assert data[b + int(name[2:])] == 10, name
        elif name.startswith('head'):
            h = int(name[4:])
            assert data[b - h - 1] == 10 and b'\n' not in data[b - h:b], name
        elif name.startswith('span'):
            k = int(name[4])
            assert b'\n' not in data[b:b + k * U], name
        elif name.startswith('nl') and '_' in name:
            n = int(name[2:name.index('_')])
            assert data.count(b'\n', b, b + U) == n, name
            assert (data[b] == 10) == name.endswith('at_b'), name
        elif name.startswith('len'):
            n = int(name[3:].rstrip('ensdtar'))
            lens = [len(x) for x in data[b - n - 600:b + n + 600].split(b'\n')]
            assert n in lens, name
        else:
            kind, d = name[:-2], int(name[-2:])
            c = data[b + d]
            assert {'tab': c == 9, 'cr': c == 13, 'ctl': c <= 9 and c != 10,
                    'utf8': c >= 0xc2}[kind], name
    assert len(names) == len(L.cases) == 40
    assert {'nl%d_after' % K, 'nl%d_at_b' % (K + 1), 'head%d' % P,
            'head%d' % (P + 1), 'head%d' % (P - 1)} <= names
    assert data[-1:] != b'\n'


def test_long_record_prediction():
    # records [0,99], [100,1099], [1100,1199]; units of 512 bytes
    beg, end = [0, 100, 1100], [99, 1099, 1199]
    # record 1 ends in unit 2 (g0 = 1024) and began at 100 <= 1024 - 512
    assert framing.long_records(beg, end, 512, 512) == 1
    # a pre-lap of 1000 holds its start
    assert framing.long_records(beg, end, 512, 1000) == 0
    # units 2 and 3 make segment 1: the same g0
    assert framing.long_records(beg, end, 512, 512, seg=2) == 1
    # units 0-3 make segment 0: nothing straddles a segment start
    assert framing.long_records(beg, end, 512, 512, seg=4) == 0
    # from a base 100 bytes later, record 1 ends in unit 1 and began
    # 512 bytes before its start
    assert framing.long_records(beg, end, 512, 512, base=100) == 1
