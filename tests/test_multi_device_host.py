"""Scans over several devices (dng_scan_open_devices), the parts that need no
GPU: the entry points are exported and refuse what they must, and the rule
that cuts the fed files into one byte range per shard -- restated here in
Python -- owns every line of the logical stream exactly once, wherever the
cuts fall."""

import ctypes
import itertools
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))


# -- the cut rule -------------------------------------------------------------
#
# The ordered files are one stream of T bytes.  Shard k of n owns the lines
# that start in [a_k, a_k+1), a_k = floor(k T / n); a line starts at p < T when
# p == 0 or byte p - 1 is '\n'.  Shard k reads from its first line start to
# the first line start at or after a_k+1 (T for the last shard).

def line_start(stream, a):
    """The first line start at or after a (len(stream) if there is none)."""
    T = len(stream)
    if a == 0 or a >= T:
        return min(a, T)
    j = stream.find(b'\n', a - 1)
    return T if j < 0 else j + 1


def shard_ranges(stream, cuts):
    """cuts: a_0 = 0 <= a_1 <= ... <= a_n = T -> [(begin, end)] per shard."""
    starts = [line_start(stream, a) for a in cuts]
    return list(zip(starts[:-1], starts[1:]))


def even_cuts(T, n):
    return [T * k // n for k in range(n + 1)]


def segments(sizes, begin, end):
    """(file index, offset, length) a shard reads for stream bytes [begin,
    end): what the library feeds its scan, file by file."""
    out, base = [], 0
    for i, size in enumerate(sizes):
        lo, hi = max(begin, base), min(end, base + size)
        if lo < hi:
            out.append((i, lo - base, hi - lo))
        base += size
    return out


def lines_of(data):
    """lstream: split on '\\n'; the unterminated tail is a line, nothing
    after a final '\\n' is.  -> [(start, bytes)]"""
    out, p = [], 0
    while p < len(data):
        j = data.find(b'\n', p)
        end = len(data) if j < 0 else j
        out.append((p, data[p:end]))
        p = end + 1
    return out


def check_cuts(files, cuts):
    stream = b''.join(files)
    T = len(stream)
    ranges = shard_ranges(stream, cuts)
    whole = lines_of(stream)
    owned = []
    for k, (b, e) in enumerate(ranges):
        # every line the shard reads starts in its range, and it reads
        # every line that does, whole
        mine = [(b + p, ln) for p, ln in lines_of(stream[b:e])]
        assert all(cuts[k] <= p < cuts[k + 1] for p, _ in mine), (k, cuts)
        assert mine == [(p, ln) for p, ln in whole
                        if cuts[k] <= p < cuts[k + 1]], (k, cuts)
        # the file segments it is fed are exactly those bytes
        got = b''.join(files[i][o:o + n]
                       for i, o, n in segments([len(f) for f in files], b, e))
        assert got == stream[b:e]
        owned += mine
    assert owned == whole
    assert sum(e - b for b, e in ranges) == T
    return ranges


STREAMS = {
    'empty_lines': [b'{"a":1}\n\n\n{"a":2}\n\n'],
    'crlf': [b'{"a":1}\r\n{"a":2}\r\n\r\n{"a":3}\r\n'],
    'empty_files': [b'', b'{"a":1}\n', b'', b'', b'{"a":2}\n', b''],
    'no_trailing_newline': [b'{"a":1}\n{"a"', b':2}\n{"a":3}', b'\n{"a":4}\n'],
    'line_over_three_files': [b'{"a":1}\n{"b":', b'"xy', b'z"}\n{"a":2}\n'],
    'unterminated_final_line': [b'{"a":1}\n\n{"a":2}\n{"tail":tr', b'ue}'],
    'only_newlines': [b'\n', b'\n\n'],
    'one_unterminated_line': [b'abc', b'def'],
}


@pytest.mark.parametrize('name', sorted(STREAMS))
def test_every_line_owned_once_for_every_cut(name):
    files = STREAMS[name]
    T = sum(len(f) for f in files)
    for c in range(T + 1):                      # two shards, one cut
        check_cuts(files, [0, c, T])
    for c1, c2 in itertools.combinations_with_replacement(range(T + 1), 2):
        check_cuts(files, [0, c1, c2, T])       # three shards
    for n in range(1, 9):                       # the library's even cuts
        check_cuts(files, even_cuts(T, n))


def test_cuts_at_the_edges_of_a_line():
    """On a newline, a byte either side of it, on an empty line: the shard
    whose range holds the line's first byte reads the line."""
    s = [b'{"a":1}\n\n{"a":2}\n']
    nl = s[0].index(b'\n')
    assert check_cuts(s, [0, nl, len(s[0])])[1][0] == nl + 1
    assert check_cuts(s, [0, nl - 1, len(s[0])])[1][0] == nl + 1
    assert check_cuts(s, [0, nl + 1, len(s[0])])[1][0] == nl + 1   # empty line
    assert check_cuts(s, [0, nl + 2, len(s[0])])[1][0] == nl + 2
    # a cut inside a line that spans three files: the next shard starts after
    # the line, in the third file
    f = STREAMS['line_over_three_files']
    T = sum(map(len, f))
    b = check_cuts(f, [0, len(f[0]) + 1, T])[1][0]
    assert b == len(f[0]) + len(f[1]) + f[2].index(b'\n') + 1
    # the unterminated tail belongs to the shard it starts in
    u = STREAMS['unterminated_final_line']
    T = sum(map(len, u))
    assert check_cuts(u, [0, T - 2, T])[1] == (T, T)


# -- the C ABI without a GPU --------------------------------------------------

@pytest.fixture(scope='module')
def native():
    import __graft_entry__
    __graft_entry__.build()
    from dragnet_b200 import native as n
    return n


def test_new_symbols_are_exported(native):
    for name in ('dng_scan_open_devices', 'dng_scan_shard'):
        assert name in native.SYMBOLS
        assert hasattr(native.lib(), name)


def test_open_devices_refuses_no_devices(native):
    L = native.lib()
    p = native.Plan('{"breakdowns":[]}')
    out = ctypes.c_void_p()
    err = ctypes.create_string_buffer(256)
    devs = (ctypes.c_int * 1)(0)
    assert L.dng_scan_open_devices(p.handle, None, 2, ctypes.byref(out), err,
                                   len(err)) == -1
    for n in (0, -1):
        assert L.dng_scan_open_devices(p.handle, devs, n, ctypes.byref(out),
                                       err, len(err)) == -1
    assert not out.value
    assert L.dng_scan_shard(None, 0) is None
    with pytest.raises(native.DngError) as ei:
        native.Scan(p, devices=[])
    assert ei.value.code == -1


def test_open_devices_without_cuda_is_enodev(native):
    if native.lib().dng_device_count() > 0:
        pytest.skip('a GPU is present')
    p = native.Plan('{"breakdowns":[]}')
    for devs in ([0], [0, 0, 0], [0, 1]):
        with pytest.raises(native.DngError) as ei:
            native.Scan(p, devices=devs)
        assert ei.value.code == -2


def test_datasource_checks_devices():
    from dragnet_b200 import datasource_gpu
    for bad in ([], 'some', [0, -1], [0, '1'], [True], 3):
        r = datasource_gpu.createDatasource({'dsconfig': {
            'path': '/x', 'devices': bad}})
        assert isinstance(r, datasource_gpu.DsError), bad
        assert '"devices"' in str(r)
    for good in ([0], [0, 0, 0], 'all'):
        r = datasource_gpu.createDatasource({'dsconfig': {
            'path': '/x', 'devices': good}})
        assert isinstance(r, datasource_gpu.DatasourceGpu), good
