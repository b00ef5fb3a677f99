"""The width selector of bound calls with a width ladder (csrc/pwpp_ladder.cuh, k_ladder_select) on the CPU and on the H100,
from one case list: the cases of test_simt_bound_ladder.py, the width and the SWITCH value compared with the same numpy statement
of the width rule on both backends.

The "simt" backend runs the kernel through the SIMT stand-in (tests/simt/simt_bound_ladder.cpp), whose cudaGraphSetConditional
records the value. The "device" backend runs it as compiled for sm_90a inside a real CUDA graph (tests/gpu_bound_ladder_probe.cu,
built by patchwork-plusplus_b200/build.py): a SWITCH node behind the selector whose body i is a memset node writing i, so the
test reads the body the device API actually launched."""
import ctypes as C
import os

import pytest

import test_simt_bound_ladder as S

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
PROBE = os.path.join(REPO, "patchwork-plusplus_b200", "lib", "libpwpp_bound_ladder_probe.so")


@pytest.fixture(scope="module")
def simt():
    return S.build_lib()


@pytest.fixture(scope="module")
def device():
    assert os.path.exists(PROBE), "lib/libpwpp_bound_ladder_probe.so was not built (patchwork-plusplus_b200/build.py)"
    return S.declare(C.CDLL(PROBE), "probe_ladder_select")


@pytest.mark.parametrize("group", list(S.GROUPS))
def test_bound_ladder_simt(simt, group):
    S.run_group(simt, group)


@pytest.mark.gpu
@pytest.mark.parametrize("group", list(S.GROUPS))
def test_bound_ladder_device(device, group):
    S.run_group(device, group)
