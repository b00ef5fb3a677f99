"""The kernels of bound calls with a stream table (csrc/pwpp_records.cuh, k_bound_table_streams, k_bound_table_rings_streams,
k_bound_table_packed_streams, k_bound_reset; csrc/pwpp_getters.cuh, k_bound_states_streams) on the CPU and on the H100, from one
case list: the cases of test_simt_bound_streams.py, every output word, the claim table, the action and slot copies, the run's
record table, every state and every state row compared with the same numpy statement of the rules on both backends, so the two
agree bit for bit. The duplicate check's global atomics, barriers and re-read of the claims run here as compiled for sm_90a.

The "simt" backend runs the kernels through the SIMT stand-in (tests/simt/simt_bound_streams.cpp); the "device" backend runs
them as compiled for sm_90a (tests/gpu_bound_streams_probe.cu, built by patchwork-plusplus_b200/build.py), every array copied to
the device before a launch and back after it."""
import ctypes as C
import os

import pytest

import test_simt_bound_streams as S

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
PROBE = os.path.join(REPO, "patchwork-plusplus_b200", "lib", "libpwpp_bound_streams_probe.so")
CASES = ([("schedules", kind, acts, shape) for kind in S.KINDS for acts in (False, True) for shape in S.SHAPES] +
         [("every_action", kind, None, None) for kind in S.KINDS] + [("first_skipped", None, None, None), ("identity", None, None, None),
                                                                      ("all_holes", None, None, None)])
IDS = ["-".join(str(x) for x in c if x is not None) for c in CASES]


@pytest.fixture(scope="module")
def simt():
    return S.Backend(S.build_lib(), "simt_")


@pytest.fixture(scope="module")
def device():
    import torch
    assert os.path.exists(PROBE), "lib/libpwpp_bound_streams_probe.so was not built (patchwork-plusplus_b200/build.py)"

    def back(a, d):
        a[...] = d.cpu().numpy()
    return S.Backend(S.declare(C.CDLL(PROBE), "probe_"), "probe_", to_device=lambda a: torch.from_numpy(a).cuda(), back=back)


def run(lib, case):
    name, kind, acts, shape = case
    if name == "schedules":
        S.schedules(lib, kind, acts, shape)
    elif name == "every_action":
        S.test_every_action_with_every_stream_case(lib, kind)
    elif name == "first_skipped":
        S.test_duplicates_first_occurrence_skipped_by_action(lib)
    elif name == "identity":
        S.test_identity_matches_bound_streams(lib)
    else:
        S.test_all_holes(lib)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_bound_streams_simt(simt, case):
    run(simt, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_bound_streams_device(device, case):
    run(device, case)
