"""The record gather kernel (csrc/pwpp_records.cuh, k_gather_records) on the CPU and on the H100, from one case list.

The cases are tests/test_simt_records_gather.py's CASES: steps 12 to 1024 over several tiles, every source alignment 0-15,
ground + non-ground counts at and around tile boundaries with and without dropped points, empty, all-dropped, all-ground and
all-non-ground frames, and a mixed-layout launch that includes steps below 4. Every case checks each frame's region byte for
byte against numpy's records[lists] and that no byte of a sentinel-filled dst outside the regions' records was written.
The "device" backend runs the kernel as compiled for sm_90a (tests/gpu_records_gather_probe.cu, built by
patchwork-plusplus_b200/build.py); each frame is copied to the device at the same distance from a 16-byte boundary as its
host array."""
import ctypes as C
import os

import numpy as np
import pytest

import test_simt_records_gather as G

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
PROBE = os.path.join(REPO, "patchwork-plusplus_b200", "lib", "libpwpp_records_gather_probe.so")


def device_launch(probe):
    def launch(nf, ptrs, n, step, idx, nd, dst, off):
        import torch
        keep, d_ptrs = [], []
        for f in range(nf):
            nbytes = int(n[f]) * int(step[f])
            mis = ptrs[f] % 16 if nbytes else 0
            t = torch.zeros(64 + mis + nbytes + 64, dtype=torch.uint8, device="cuda")   # (base: 512-byte aligned)
            if nbytes:
                t[64 + mis:64 + mis + nbytes] = torch.frombuffer(bytearray(C.string_at(ptrs[f], nbytes)), dtype=torch.uint8)
            keep.append(t)
            d_ptrs.append(t.data_ptr() + 64 + mis)
        d_dst = torch.from_numpy(dst.copy()).cuda()   # (a fresh allocation: 16-byte aligned like dst)
        torch.cuda.synchronize()
        rc = probe.probe_gather_records(nf, (C.c_void_p * nf)(*d_ptrs), n.ctypes.data, step.ctypes.data, idx.ctypes.data, nd.ctypes.data,
                                        d_dst.data_ptr(), off.ctypes.data)   # (synchronous)
        dst[:] = d_dst.cpu().numpy()
        return rc
    return launch


@pytest.fixture(scope="module")
def probe():
    assert os.path.exists(PROBE), "lib/libpwpp_records_gather_probe.so was not built (patchwork-plusplus_b200/build.py)"
    L = C.CDLL(PROBE)
    L.probe_gather_records.argtypes = G.ARGS
    L.probe_gather_records.restype = C.c_int
    return L


@pytest.fixture(params=["simt", pytest.param("device", marks=pytest.mark.gpu)])
def launch(request):
    if request.param == "simt":
        return G.simt_launch(request.getfixturevalue("lib"))
    return device_launch(request.getfixturevalue("probe"))


lib = G.lib   # the SIMT library fixture


@pytest.mark.parametrize("name", list(G.CASES))
def test_gather_case(launch, name):
    G.run_case(launch, name)
