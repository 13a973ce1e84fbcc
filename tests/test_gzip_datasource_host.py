"""The datasource's `compression` key, on the CPU: the values it takes, the
values and device lists it refuses, and which files it would inflate."""

import gzip
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))
from dragnet_b200 import datasource_gpu  # noqa: E402


def _ds(**cfg):
    return datasource_gpu.createDatasource(
        {'dsconfig': dict({'path': '/nonexistent'}, **cfg)})


def test_values():
    for v in (None, 'none', 'gzip'):
        cfg = {} if v is None else {'compression': v}
        d = _ds(**cfg)
        assert isinstance(d, datasource_gpu.DatasourceGpu), d
        assert d.ds_compression == ('gzip' if v == 'gzip' else None)
    for v in ('zstd', 'GZIP', '', 1):
        e = _ds(compression=v)
        assert isinstance(e, datasource_gpu.DsError)
        assert str(e) == 'unsupported compression: "%s"' % (v,)


def test_several_devices_refused():
    d = _ds(compression='gzip', devices=[0, 1])
    e = d._run({}, [])
    assert isinstance(e, datasource_gpu.DsError)
    assert 'several devices' in str(e)
    with pytest.raises(datasource_gpu.DsError):
        datasource_gpu.run_plan({}, files=[], devices=[0, 1],
                                compression='gzip')


def test_which_files_are_gzip(tmp_path):
    cases = {'a.gz': gzip.compress(b'x\n'), 'b.log': b'{"a":1}\n',
             'c.gz': b'\x1f\x8b', 'd': b'', 'e.gz': b'\x1f\x8b\x07abc'}
    got = {}
    for name, data in cases.items():
        p = tmp_path / name
        p.write_bytes(data)
        got[name] = datasource_gpu.is_gzip(str(p))
    assert got == {'a.gz': True, 'b.log': False, 'c.gz': False, 'd': False,
                   'e.gz': False}
