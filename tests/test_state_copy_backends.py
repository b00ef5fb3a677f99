"""The cases of tests/test_simt_state_copy.py on the H100: the device state copies (csrc/pwpp_state_copy.cuh) as compiled for sm_90a
(tests/gpu_state_copy_probe.cu, built by build.py), against the same numpy rows and states."""
import os

import pytest

from test_simt_state_copy import *  # noqa: F401,F403 (the cases and their model)
from test_simt_state_copy import Backend

PROBE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "patchwork-plusplus_b200", "lib", "libpwpp_state_copy_probe.so")

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def backend():
    assert os.path.exists(PROBE), "lib/libpwpp_state_copy_probe.so was not built (patchwork-plusplus_b200/build.py)"
    return Backend(PROBE, "probe")
