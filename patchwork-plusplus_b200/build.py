"""Builds the product's native code IN-TREE (the .so files travel to the GPU box with the snapshot).

  lib/libpwpp_b200.so    CUDA kernels + C-ABI (csrc/pwpp_capi.cu), sm_90a (H100) only
  lib/pypatchworkpp*.so  pybind11 module mirroring the reference binding (python/pybinding.cpp)

No torch, no JIT cache: plain nvcc / g++ invocations.
"""
import glob
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "lib")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def build_core(force=False, verbose=False):
    os.makedirs(LIB, exist_ok=True)
    src = os.path.join(HERE, "csrc", "pwpp_capi.cu")
    deps = glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]
    out = os.path.join(LIB, "libpwpp_b200.so")
    if force or _newer(out, deps):
        cmd = [NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out, src]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        cmd[1:1] = os.environ.get("PWPP_EXTRA_NVCC_FLAGS", "").split()
        subprocess.check_call(cmd)
    return out


def build_pybind(force=False):
    import pybind11
    os.makedirs(LIB, exist_ok=True)
    src = os.path.join(HERE, "python", "pybinding.cpp")
    hdr = os.path.join(REPO, "include", "patchwork", "patchworkpp.h")
    ext = sysconfig.get_config_var("EXT_SUFFIX")
    out = os.path.join(LIB, "pypatchworkpp" + ext)
    core = build_core()
    if force or _newer(out, [src, hdr, core]):
        cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden",
               "-I" + pybind11.get_include(), "-I" + sysconfig.get_paths()["include"],
               "-I" + os.path.join(REPO, "include"), src, "-o", out,
               "-L" + LIB, "-lpwpp_b200", "-Wl,-rpath,$ORIGIN"]
        subprocess.check_call(cmd)
    return out


def build_examples(force=False):
    """examples/pwpp_sequence.cpp -> lib/pwpp_sequence (the demo_sequential equivalent: directory of KITTI scans, one stream)."""
    src = os.path.join(REPO, "examples", "pwpp_sequence.cpp")
    hdr = os.path.join(REPO, "include", "patchwork", "patchworkpp.h")
    out = os.path.join(LIB, "pwpp_sequence")
    core = build_core()
    if force or _newer(out, [src, hdr, core]):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(REPO, "include"), src, "-o", out,
                               "-L" + LIB, "-lpwpp_b200", "-Wl,-rpath,$ORIGIN", "-lpthread"])
    src2 = os.path.join(REPO, "examples", "pwpp_latency.cpp")
    out2 = os.path.join(LIB, "pwpp_latency")
    if force or _newer(out2, [src2, hdr, core]):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(REPO, "include"), src2, "-o", out2,
                               "-L" + LIB, "-lpwpp_b200", "-Wl,-rpath,$ORIGIN", "-lpthread"])
    src3 = os.path.join(REPO, "tests", "pc2_driver.cpp")   # the PointCloud2 front end against the real engine (GPU test)
    out3 = os.path.join(LIB, "pc2_driver")
    if force or _newer(out3, [src3, hdr, os.path.join(REPO, "include", "patchwork", "pointcloud2.hpp"), core]):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(REPO, "include"), src3, "-o", out3,
                               "-L" + LIB, "-lpwpp_b200", "-Wl,-rpath,$ORIGIN"])
    src4 = os.path.join(REPO, "tests", "pc2_records_driver.cpp")   # the records path of pointcloud2.hpp against the real engine (GPU test)
    out4 = os.path.join(LIB, "pc2_records_driver")
    if force or _newer(out4, [src4, hdr, os.path.join(REPO, "include", "patchwork", "pointcloud2.hpp"), core]):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(REPO, "include"), src4, "-o", out4,
                               "-L" + LIB, "-lpwpp_b200", "-Wl,-rpath,$ORIGIN"])
    src7 = os.path.join(REPO, "tests", "pc2_records_out_driver.cpp")   # makeRecordsPayload against the real engine (GPU test)
    out7 = os.path.join(LIB, "pc2_records_out_driver")
    if force or _newer(out7, [src7, hdr, os.path.join(REPO, "include", "patchwork", "pointcloud2.hpp"), core]):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(REPO, "include"), src7, "-o", out7,
                               "-L" + LIB, "-lpwpp_b200", "-Wl,-rpath,$ORIGIN"])
    # the record unpack kernel alone, compiled for sm_90a like the core (GPU cases of tests/test_simt_records.py)
    src5 = os.path.join(REPO, "tests", "gpu_records_probe.cu")
    out5 = os.path.join(LIB, "libpwpp_records_probe.so")
    if force or _newer(out5, [src5] + glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out5, src5])
    # the record gather kernel alone, the same way (GPU cases of tests/test_records_gather_backends.py)
    src6 = os.path.join(REPO, "tests", "gpu_records_gather_probe.cu")
    out6 = os.path.join(LIB, "libpwpp_records_gather_probe.so")
    if force or _newer(out6, [src6] + glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out6, src6])
    # the record gather of a bound call's record results, the same way (GPU cases of tests/test_records_parts_backends.py)
    src8 = os.path.join(REPO, "tests", "gpu_records_parts_probe.cu")
    out8 = os.path.join(LIB, "libpwpp_records_parts_probe.so")
    if force or _newer(out8, [src8] + glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out8, src8])
    # the kernels of a bound call's getter results, the same way (GPU cases of tests/test_bound_getters_backends.py)
    src9 = os.path.join(REPO, "tests", "gpu_bound_getters_probe.cu")
    out9 = os.path.join(LIB, "libpwpp_bound_getters_probe.so")
    if force or _newer(out9, [src9] + glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out9, src9])
    # the kernels of a bound call's packed xyz results, the same way (GPU cases of tests/test_bound_packed_xyz_backends.py)
    src10 = os.path.join(REPO, "tests", "gpu_bound_packed_probe.cu")
    out10 = os.path.join(LIB, "libpwpp_bound_packed_probe.so")
    if force or _newer(out10, [src10] + glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out10, src10])
    # the kernels of a bound call's packed records, the same way (GPU cases of tests/test_records_packed_backends.py)
    src11 = os.path.join(REPO, "tests", "gpu_records_packed_probe.cu")
    out11 = os.path.join(LIB, "libpwpp_records_packed_probe.so")
    if force or _newer(out11, [src11] + glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out11, src11])
    # the reference-order sort and its libstdc++ tie fix-up alone, the same way (GPU cases of tests/test_order_exact_backends.py)
    src12 = os.path.join(REPO, "tests", "gpu_order_exact_probe.cu")
    out12 = os.path.join(LIB, "libpwpp_order_exact_probe.so")
    if force or _newer(out12, [src12] + glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out12, src12])
    # the device state copies alone, the same way (GPU cases of tests/test_state_copy_backends.py)
    src13 = os.path.join(REPO, "tests", "gpu_state_copy_probe.cu")
    out13 = os.path.join(LIB, "libpwpp_state_copy_probe.so")
    if force or _newer(out13, [src13] + glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out13, src13])
    # the kernels of bound calls with a stream table, the same way (GPU cases of tests/test_bound_streams_backends.py)
    src15 = os.path.join(REPO, "tests", "gpu_bound_streams_probe.cu")
    out15 = os.path.join(LIB, "libpwpp_bound_streams_probe.so")
    if force or _newer(out15, [src15] + glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out15, src15])
    # the width selector of bound calls with a width ladder, inside a real graph (GPU cases of tests/test_bound_ladder_backends.py)
    src16 = os.path.join(REPO, "tests", "gpu_bound_ladder_probe.cu")
    out16 = os.path.join(LIB, "libpwpp_bound_ladder_probe.so")
    if force or _newer(out16, [src16] + glob.glob(os.path.join(HERE, "csrc", "*")) + [os.path.join(REPO, "include", "pwpp.h")]):
        subprocess.check_call([NVCC, "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared",
                               "-I" + os.path.join(REPO, "include"), "-I" + os.path.join(HERE, "csrc"), "-cudart", "static", "-o", out16, src16])
    src14 = os.path.join(REPO, "tests", "pwpp_copy_driver.cpp")   # copies of the drop-in class against the real engine (GPU test)
    out14 = os.path.join(LIB, "pwpp_copy_driver")
    if force or _newer(out14, [src14, hdr, core]):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(REPO, "include"), src14, "-o", out14,
                               "-L" + LIB, "-lpwpp_b200", "-Wl,-rpath,$ORIGIN"])
    return out


def build_all(force=False):
    build_core(force)
    build_pybind(force)
    build_examples(force)


if __name__ == "__main__":
    build_core(force="--force" in sys.argv, verbose="-v" in sys.argv)
    if "--core-only" not in sys.argv:
        build_pybind(force="--force" in sys.argv)
