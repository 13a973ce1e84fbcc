"""The compressed-input object links on its own: tests/gpucheck/cz_capture.cu
builds with nvcc against compressed.cu compiled with the policy variant of
tests/test_gpu_decode_bytes.py, with nothing of api.cu but its six stubs.  A
seventh dependency between compressed.cu and api.cu breaks this CPU test
instead of the GPU run; a policy macro that lost its #ifndef guard breaks
the variant's compile."""

import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(__file__))

NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')


@pytest.mark.skipif(not os.path.exists(NVCC), reason='needs nvcc')
def test_harness_links_against_variant(tmp_path):
    import test_gpu_decode_bytes as t
    obj = t.compile_object(str(tmp_path / 'variant.o'), t.VARIANT)
    exe = t.link_harness(obj, str(tmp_path / 'cz_capture'))
    assert os.path.getsize(exe) > 0
    # the six symbols compressed.o takes from the rest of the library
    undef = subprocess.check_output(['nm', '-uC', obj]).decode()
    got = sorted(ln.split(' U ', 1)[1].split('(')[0].strip()
                 for ln in undef.splitlines()
                 if '(dng_scan' in ln or 'dng_cached' in ln)
    assert got == ['dng_cached_alloc', 'dng_cached_free', 'feed_device',
                   'get_event', 'read_to_device', 'refuse_multi']
