"""Thin ctypes front-end of the C-ABI in include/pwpp.h (lib/libpwpp_b200.so).

Used by tests/ and bench.py to call the product exactly as a foreign-language host would: plain
pointers and sizes, no torch types. The CUDA library is REQUIRED: loading fails loudly when it is
missing and creating an Engine fails loudly without a CUDA device — there is no CPU fallback.
"""
import ctypes as C
import os

import numpy as np

from pwpp_ctypes import PwppBinResult, PwppParams, PwppPointLayout, PwppState, default_params  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PWPP_LIB") or os.path.join(_HERE, "lib", "libpwpp_b200.so")   # PWPP_LIB: a diagnostic build of the same library

_lib = None


def load_library():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: build it with `python patchwork-plusplus_b200/build.py` "
                           "(nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
    lib.pwpp_params_default.argtypes = [C.POINTER(PwppParams)]; lib.pwpp_params_default.restype = None
    lib.pwpp_create.argtypes = [C.POINTER(PwppParams), i32, i32, i64, C.POINTER(vp)]; lib.pwpp_create.restype = i32
    lib.pwpp_destroy.argtypes = [vp]; lib.pwpp_destroy.restype = None
    lib.pwpp_last_error.argtypes = []; lib.pwpp_last_error.restype = C.c_char_p
    lib.pwpp_abi_version.argtypes = []; lib.pwpp_abi_version.restype = i32
    lib.pwpp_num_bins.argtypes = [vp]; lib.pwpp_num_bins.restype = i32
    lib.pwpp_create_sets.argtypes = [C.POINTER(PwppParams), i32, vp, i32, i32, i64, C.POINTER(vp)]; lib.pwpp_create_sets.restype = i32
    lib.pwpp_stream_num_bins.argtypes = [vp, i32]; lib.pwpp_stream_num_bins.restype = i32
    lib.pwpp_stream_set.argtypes = [vp, i32]; lib.pwpp_stream_set.restype = i32
    lib.pwpp_stream_state_blob_size.argtypes = [vp, i32]; lib.pwpp_stream_state_blob_size.restype = C.c_size_t
    lib.pwpp_estimate_host.argtypes = [vp, i32, C.POINTER(vp), C.POINTER(i64), i32, i64, i64]; lib.pwpp_estimate_host.restype = i32
    lib.pwpp_estimate_device.argtypes = [vp, i32, vp, C.POINTER(i64), i32, vp]; lib.pwpp_estimate_device.restype = i32
    lib.pwpp_estimate_host_streams.argtypes = [vp, i32, vp, C.POINTER(vp), C.POINTER(i64), i32, i64, i64]
    lib.pwpp_estimate_host_streams.restype = i32
    lib.pwpp_estimate_device_streams.argtypes = [vp, i32, vp, vp, C.POINTER(i64), i32, vp]; lib.pwpp_estimate_device_streams.restype = i32
    lib.pwpp_estimate_host_records.argtypes = [vp, i32, vp, vp, vp, vp]; lib.pwpp_estimate_host_records.restype = i32
    lib.pwpp_estimate_device_records.argtypes = [vp, i32, vp, vp, vp, vp, vp]; lib.pwpp_estimate_device_records.restype = i32
    lib.pwpp_synchronize.argtypes = [vp]; lib.pwpp_synchronize.restype = i32
    lib.pwpp_device_record_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]; lib.pwpp_device_record_results.restype = i32
    lib.pwpp_host_record_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]; lib.pwpp_host_record_results.restype = i32
    for n in ("pwpp_copy_ground_records", "pwpp_copy_nonground_records"):
        getattr(lib, n).argtypes = [vp, i32, vp]; getattr(lib, n).restype = i32
    for n in ("pwpp_num_ground", "pwpp_num_nonground"):
        getattr(lib, n).argtypes = [vp, i32]; getattr(lib, n).restype = i64
    for n in ("pwpp_copy_ground_indices", "pwpp_copy_nonground_indices", "pwpp_copy_ground_xyz", "pwpp_copy_nonground_xyz",
              "pwpp_copy_centers", "pwpp_copy_normals", "pwpp_copy_bin_results", "pwpp_copy_bin_ids"):
        getattr(lib, n).argtypes = [vp, i32, vp]; getattr(lib, n).restype = i32
    lib.pwpp_num_patches.argtypes = [vp, i32]; lib.pwpp_num_patches.restype = i32
    lib.pwpp_height.argtypes = [vp, i32]; lib.pwpp_height.restype = C.c_double
    lib.pwpp_time_us.argtypes = [vp]; lib.pwpp_time_us.restype = C.c_double
    lib.pwpp_call_times_us.argtypes = [vp, C.POINTER(C.c_float)]; lib.pwpp_call_times_us.restype = i32
    lib.pwpp_device_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]; lib.pwpp_device_results.restype = i32
    lib.pwpp_get_state.argtypes = [vp, i32, C.POINTER(PwppState)]; lib.pwpp_get_state.restype = i32
    lib.pwpp_copy_history.argtypes = [vp, i32, i32, i32, vp]; lib.pwpp_copy_history.restype = i32
    lib.pwpp_state_blob_size.argtypes = [vp]; lib.pwpp_state_blob_size.restype = C.c_size_t
    lib.pwpp_export_state.argtypes = [vp, i32, vp]; lib.pwpp_export_state.restype = i32
    lib.pwpp_import_state.argtypes = [vp, i32, vp, C.c_size_t]; lib.pwpp_import_state.restype = i32
    lib.pwpp_reset_stream.argtypes = [vp, i32]; lib.pwpp_reset_stream.restype = i32
    lib.pwpp_reset_all.argtypes = [vp]; lib.pwpp_reset_all.restype = i32
    lib.pwpp_host_alloc.argtypes = [C.c_size_t]; lib.pwpp_host_alloc.restype = vp
    lib.pwpp_host_free.argtypes = [vp]; lib.pwpp_host_free.restype = None
    lib.pwpp_set_profiling.argtypes = [vp, i32]; lib.pwpp_set_profiling.restype = i32
    lib.pwpp_stage_times_ms.argtypes = [vp, C.POINTER(C.c_float)]; lib.pwpp_stage_times_ms.restype = i32
    lib.pwpp_stage_name.argtypes = [i32]; lib.pwpp_stage_name.restype = C.c_char_p
    lib.pwpp_launch_count.argtypes = [vp]; lib.pwpp_launch_count.restype = i64
    lib.pwpp_set_output_order.argtypes = [vp, i32]; lib.pwpp_set_output_order.restype = i32
    lib.pwpp_host_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]; lib.pwpp_host_results.restype = i32
    lib.pwpp_bind_host_to_device.argtypes = [i32]; lib.pwpp_bind_host_to_device.restype = i32
    _lib = lib
    return lib


def bind_host_to_device(device: int) -> int:
    """pwpp_bind_host_to_device: pin the calling thread to the CPUs of the GPU's NUMA node (returns the node or -1)."""
    return int(load_library().pwpp_bind_host_to_device(device))


class PwppError(RuntimeError):
    pass


# sensor_msgs/PointField datatype codes (PWPP_FIELD_* of include/pwpp.h) of the numpy scalar types
FIELD_CODES = {np.dtype(np.int8): 1, np.dtype(np.uint8): 2, np.dtype(np.int16): 3, np.dtype(np.uint16): 4, np.dtype(np.int32): 5,
               np.dtype(np.uint32): 6, np.dtype(np.float32): 7, np.dtype(np.float64): 8}


def layout_from_dtype(dtype) -> PwppPointLayout:
    """The record layout of a numpy structured dtype: fields `x`, `y`, `z` and optionally `intensity` (the names the reference's
    PointCloud2 iterators use), their offsets and datatypes, and the itemsize as point_step. Fields must be scalars of native
    (little-endian) byte order."""
    dtype = np.dtype(dtype)
    if dtype.fields is None:
        raise PwppError(f"not a structured dtype: {dtype}")
    lay = PwppPointLayout()
    lay.point_step = dtype.itemsize
    for c, name in enumerate(("x", "y", "z", "intensity")):
        if name not in dtype.fields:
            if c < 3:
                raise PwppError(f"record dtype has no field {name!r}")
            lay.offset[3], lay.datatype[3] = -1, 0
            continue
        ft, off = dtype.fields[name][:2]
        if ft.subdtype is not None:
            raise PwppError(f"field {name!r} has count > 1 ({ft})")
        if not ft.isnative:
            raise PwppError(f"field {name!r} is not in native byte order ({ft.str}); records are little-endian")
        code = FIELD_CODES.get(ft)
        if code is None:
            raise PwppError(f"field {name!r} has a datatype PointCloud2 does not define ({ft})")
        lay.offset[c], lay.datatype[c] = off, code
    return lay


def _check(rc):
    if rc != 0:
        raise PwppError(f"pwpp error {rc}: {load_library().pwpp_last_error().decode()}")


class Engine:
    """One `pwpp_ctx`: `num_streams` independent sensor streams on one CUDA device.

    `params` is one PwppParams (every stream runs with it), or a list of up to 8 parameter sets together with `stream_set`,
    the set of every stream (pwpp_create_sets): stream s then runs with params[stream_set[s]] for its whole life."""

    def __init__(self, params=None, device: int = 0, num_streams: int = 1, max_points_per_frame: int = 0, stream_set=None):
        self.lib = load_library()
        h = C.c_void_p()
        if isinstance(params, (list, tuple)):
            if stream_set is None:
                raise PwppError("a list of parameter sets needs stream_set, the set of every stream")
            sets = (PwppParams * max(len(params), 1))(*params)
            ids = np.ascontiguousarray(stream_set, dtype=np.int32)
            if ids.shape != (num_streams,):
                raise PwppError(f"stream_set must name one set per stream ({num_streams}), got shape {ids.shape}")
            _check(self.lib.pwpp_create_sets(sets, len(params), ids.ctypes.data, device, num_streams, max_points_per_frame, C.byref(h)))
            self.params = list(params)
            self.stream_set = ids.tolist()
        else:
            if stream_set is not None and any(int(k) != 0 for k in stream_set):
                raise PwppError("stream_set names sets other than 0, but only one parameter set was given")
            self.params = params if params is not None else default_params()
            _check(self.lib.pwpp_create(C.byref(self.params), device, num_streams, max_points_per_frame, C.byref(h)))
            self.stream_set = [0] * num_streams
        self._h = h
        self.num_streams = num_streams
        self.nbins = self.lib.pwpp_num_bins(h)   # with several sets: the largest bin count of the sets
        self._n = []
        self._streams = []   # stream of every frame of the last call
        self._rec_dtypes = []   # record dtype of every frame of the last records call (uint8 rows of point_step for (buffer, layout) frames)

    def close(self):
        if getattr(self, "_h", None):
            self.lib.pwpp_destroy(self._h)
            self._h = None

    def __del__(self):
        # at interpreter shutdown the CUDA runtime may already be torn down: only release explicitly-open handles
        # while the library is still importable
        try:
            import sys
            if sys is not None and not sys.is_finalizing():
                self.close()
        except Exception:
            pass

    # ---- hot path ----
    @staticmethod
    def _stream_table(streams, nf):
        ids = np.ascontiguousarray(streams, dtype=np.int32)
        if ids.shape != (nf,):
            raise PwppError(f"streams must name one stream per frame ({nf}), got shape {ids.shape}")
        return ids

    def estimate_host(self, frames, streams=None):
        """frames: list of C-contiguous float32 arrays (n_f, 3|4). Without `streams` frame f goes to stream f; with it, to
        stream streams[f] (any subset, any order, repeats run in call order). Results are indexed by the frame's position
        in the call, state by stream id."""
        frames = [np.ascontiguousarray(f, dtype=np.float32) for f in frames]
        cols = frames[0].shape[1]
        assert all(f.ndim == 2 and f.shape[1] == cols for f in frames)
        nf = len(frames)
        ptrs = (C.c_void_p * nf)(*[f.ctypes.data for f in frames])
        ns = (C.c_int64 * nf)(*[f.shape[0] for f in frames])
        if streams is None:
            _check(self.lib.pwpp_estimate_host(self._h, nf, ptrs, ns, cols, cols, 1))
        else:
            ids = self._stream_table(streams, nf)
            _check(self.lib.pwpp_estimate_host_streams(self._h, nf, ids.ctypes.data, ptrs, ns, cols, cols, 1))
        self._n = [f.shape[0] for f in frames]
        self._streams = list(range(nf)) if streams is None else [int(s) for s in streams]
        self._rec_dtypes = []

    def estimate_host_strided(self, ptrs, ns, cols, row_stride, col_stride):
        nf = len(ptrs)
        p = (C.c_void_p * nf)(*ptrs)
        n = (C.c_int64 * nf)(*ns)
        self._n = list(ns)
        self._streams = list(range(nf))
        self._rec_dtypes = []
        _check(self.lib.pwpp_estimate_host(self._h, nf, p, n, cols, row_stride, col_stride))

    def estimate_device(self, d_ptr: int, offsets, has_intensity: bool = True, stream: int = 0, streams=None):
        """Packed float4 points on the device, frame f at [offsets[f], offsets[f + 1]); `streams` as for estimate_host."""
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        nf = len(offsets) - 1
        offs = offsets.ctypes.data_as(C.POINTER(C.c_int64))
        if streams is None:
            _check(self.lib.pwpp_estimate_device(self._h, nf, C.c_void_p(d_ptr), offs, 1 if has_intensity else 0, C.c_void_p(stream)))
        else:
            ids = self._stream_table(streams, nf)
            _check(self.lib.pwpp_estimate_device_streams(self._h, nf, ids.ctypes.data, C.c_void_p(d_ptr), offs, 1 if has_intensity else 0,
                                                         C.c_void_p(stream)))
        self._n = np.diff(offsets).tolist()
        self._streams = list(range(nf)) if streams is None else [int(s) for s in streams]
        self._rec_dtypes = []

    def _records_call(self, fn, nf, streams, ptrs, ns, layouts, *extra, dtypes=None):
        ids = np.arange(nf, dtype=np.int32) if streams is None else self._stream_table(streams, nf)
        p = (C.c_void_p * max(nf, 1))(*ptrs)
        n = (C.c_int64 * max(nf, 1))(*ns)
        lays = (PwppPointLayout * max(nf, 1))(*layouts)
        self._rec_dtypes = []
        _check(fn(self._h, nf, ids.ctypes.data, p, n, lays, *extra))
        self._n = [int(k) for k in ns]
        self._streams = ids.tolist()
        self._rec_dtypes = [dt if dt is not None else np.dtype((np.uint8, (lay.point_step,)))
                            for dt, lay in zip(dtypes or [None] * nf, layouts)]

    def estimate_host_records(self, frames, streams=None):
        """Sensor records of any layout from host memory (pwpp_estimate_host_records). Every frame is a 1-D structured array
        (layout_from_dtype) or a pair (uint8 buffer, PwppPointLayout) holding len(buffer) // point_step records. `streams` as for
        estimate_host (None: frame f on stream f)."""
        ptrs, ns, layouts, keep, dtypes = [], [], [], [], []
        for fr in frames:
            if isinstance(fr, tuple):
                buf, lay = fr
                buf = np.asarray(buf)
                if buf.dtype != np.uint8 or not buf.flags.c_contiguous:
                    raise PwppError("a (buffer, layout) frame needs a C-contiguous uint8 buffer")
                n = buf.nbytes // lay.point_step if lay.point_step > 0 else 0
                dtypes.append(None)
            else:
                buf = np.asarray(fr)
                if buf.ndim != 1 or buf.strides[0] != buf.dtype.itemsize:
                    raise PwppError("a structured frame must be a contiguous 1-D array of records")
                lay, n = layout_from_dtype(buf.dtype), len(buf)
                dtypes.append(buf.dtype)
            keep.append(buf)
            ptrs.append(buf.ctypes.data)
            ns.append(n)
            layouts.append(lay)
        self._records_call(self.lib.pwpp_estimate_host_records, len(frames), streams, ptrs, ns, layouts, dtypes=dtypes)

    def estimate_device_records(self, ptrs, ns, layouts, streams=None, stream: int = 0, dtypes=None):
        """Sensor records resident on the device (pwpp_estimate_device_records): frame f is ns[f] records of layouts[f] at device
        address ptrs[f] (any alignment), unpacked on CUDA stream `stream` (0: the ctx's own stream). `dtypes`: optional record dtype
        of every frame, the dtype ground_records / nonground_records return (default: uint8 rows of point_step). The buffers must
        stay untouched until the record results are fetched, when they are wanted."""
        self._records_call(self.lib.pwpp_estimate_device_records, len(ptrs), streams, [int(p) for p in ptrs], ns, layouts, C.c_void_p(stream),
                           dtypes=dtypes)

    def synchronize(self):
        _check(self.lib.pwpp_synchronize(self._h))

    # ---- results ----
    def num_ground(self, f=0): return int(self.lib.pwpp_num_ground(self._h, f))
    def num_nonground(self, f=0): return int(self.lib.pwpp_num_nonground(self._h, f))

    def _get(self, fn, f, n, dtype, shape):
        out = np.empty(shape, dtype=dtype)
        if n > 0:
            _check(fn(self._h, f, out.ctypes.data))
        return out

    def ground_indices(self, f=0):
        n = self.num_ground(f); return self._get(self.lib.pwpp_copy_ground_indices, f, n, np.int32, (n,))

    def nonground_indices(self, f=0):
        n = self.num_nonground(f); return self._get(self.lib.pwpp_copy_nonground_indices, f, n, np.int32, (n,))

    def ground_xyz(self, f=0):
        n = self.num_ground(f); return self._get(self.lib.pwpp_copy_ground_xyz, f, n, np.float32, (n, 3))

    def nonground_xyz(self, f=0):
        n = self.num_nonground(f); return self._get(self.lib.pwpp_copy_nonground_xyz, f, n, np.float32, (n, 3))

    def _records(self, fn, f, n):
        if not 0 <= f < len(self._rec_dtypes):   # (no records call, or a bad f: the C-ABI reports it)
            _check(fn(self._h, f, None))
        dt = self._rec_dtypes[f]
        out = np.empty(n, dtype=dt)
        if n > 0:
            _check(fn(self._h, f, out.ctypes.data))
        return out

    def ground_records(self, f=0):
        """Ground points of frame f of the last records call as whole input records, byte for byte (every field the sensor sent):
        an array of the frame's structured dtype, or (count, point_step) uint8 for a (buffer, layout) frame."""
        return self._records(self.lib.pwpp_copy_ground_records, f, self.num_ground(f))

    def nonground_records(self, f=0):
        return self._records(self.lib.pwpp_copy_nonground_records, f, self.num_nonground(f))

    def device_record_lists(self):
        """Zero-copy view of the last records call's record results on the device: (records, offsets) with records a torch uint8
        CUDA tensor and offsets int64[nframes + 1] (numpy). Frame f's region starts at byte offsets[f]: num_ground(f) ground
        records, then num_nonground(f) non-ground records of its point_step. The gather is enqueued on the call's stream: the
        caller synchronizes with it (or Engine.synchronize()). Valid until the next estimate call."""
        import torch
        a, b = C.c_void_p(), C.c_void_p()
        _check(self.lib.pwpp_device_record_results(self._h, C.byref(a), C.byref(b)))
        nf = len(self._n)
        off = np.ctypeslib.as_array((C.c_int64 * (nf + 1)).from_address(b.value)).copy()
        total = int(off[-1])

        class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
            def __init__(self, ptr, n):
                self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None}
        rec = torch.as_tensor(_View(a.value, total), device="cuda") if total > 0 else torch.empty(0, dtype=torch.uint8, device="cuda")
        return rec, off

    def host_record_lists(self):
        """The same in the page-locked host view (one device->host copy): (records uint8[total] numpy view, offsets int64[nframes + 1])."""
        a, b = C.c_void_p(), C.c_void_p()
        _check(self.lib.pwpp_host_record_results(self._h, C.byref(a), C.byref(b)))
        nf = len(self._n)
        off = np.ctypeslib.as_array((C.c_int64 * (nf + 1)).from_address(b.value)).copy()
        rec = np.ctypeslib.as_array((C.c_uint8 * max(int(off[-1]), 1)).from_address(a.value))[:int(off[-1])]
        return rec, off

    def num_patches(self, f=0): return int(self.lib.pwpp_num_patches(self._h, f))

    def centers(self, f=0):
        n = self.num_patches(f); return self._get(self.lib.pwpp_copy_centers, f, n, np.float32, (n, 3))

    def normals(self, f=0):
        n = self.num_patches(f); return self._get(self.lib.pwpp_copy_normals, f, n, np.float32, (n, 3))

    def height(self, f=0): return float(self.lib.pwpp_height(self._h, f))
    def time_us(self): return float(self.lib.pwpp_time_us(self._h))

    def call_times_us(self):
        """{h2d, kernels, d2h, device_total} of the last single-chunk estimate_host call, microseconds (CUDA events)."""
        arr = (C.c_float * 4)()
        _check(self.lib.pwpp_call_times_us(self._h, arr))
        return dict(zip(("h2d", "kernels", "d2h", "device_total"), (float(v) for v in arr)))

    def stream_num_bins(self, s: int) -> int:
        """Bin count of stream s's parameter set."""
        n = int(self.lib.pwpp_stream_num_bins(self._h, s))
        if n < 0:
            _check(n)
        return n

    def bin_results(self, f=0):
        """Patch records of frame f of the last call: the bins of the frame's parameter set."""
        nb = self.stream_num_bins(self._streams[f]) if 0 <= f < len(self._streams) else self.nbins   # (a bad f: the C-ABI reports it)
        arr = (PwppBinResult * nb)()
        _check(self.lib.pwpp_copy_bin_results(self._h, f, C.byref(arr)))
        return arr

    def bin_ids(self, f=0):
        out = np.empty(self._n[f], dtype=np.uint16)
        if self._n[f] > 0:
            _check(self.lib.pwpp_copy_bin_ids(self._h, f, out.ctypes.data))
        return out

    def state(self, f=0) -> PwppState:
        st = PwppState()
        _check(self.lib.pwpp_get_state(self._h, f, C.byref(st)))
        return st

    def history(self, f, ring, which):
        st = self.state(f)
        n = (st.n_flatness if which else st.n_elevation)[ring]
        out = np.empty(n, dtype=np.float64)
        _check(self.lib.pwpp_copy_history(self._h, f, ring, which, out.ctypes.data))
        return out

    def export_state(self, f=0) -> bytes:
        """Complete temporal state of stream f as an opaque blob (checkpoint / migration to another ctx or GPU)."""
        buf = C.create_string_buffer(self.lib.pwpp_stream_state_blob_size(self._h, f))
        _check(self.lib.pwpp_export_state(self._h, f, buf))
        return buf.raw

    def import_state(self, f, blob: bytes):
        _check(self.lib.pwpp_import_state(self._h, f, blob, len(blob)))

    def device_index_lists(self):
        """Zero-copy view of the last call's results on the device: (indices, num_ground) as torch int32 CUDA tensors.
        indices is laid out like the input (frame f's region starts at its point offset): ground list, then non-ground
        list. Valid until the next estimate call; the caller synchronizes with its stream (or Engine.synchronize())."""
        import torch
        d_idx, d_ng = self.device_results()
        total, nf = int(sum(self._n)), len(self._n)

        class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
            def __init__(self, ptr, n):
                self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3, "strides": None}
        idx = torch.as_tensor(_View(d_idx, total), device="cuda") if total > 0 else torch.empty(0, dtype=torch.int32, device="cuda")
        ng = torch.as_tensor(_View(d_ng, nf), device="cuda")
        return idx, ng

    def host_index_lists(self):
        """Zero-copy numpy views of the last call's results in the page-locked result buffer: (indices int32[total],
        num_ground int32[nframes], offsets int64[nframes + 1]). Frame f: ground = indices[off[f] : off[f] + ng[f]], non-ground
        follows up to off[f + 1] (minus dropped points). Valid until the next estimate call."""
        a, b, c = C.c_void_p(), C.c_void_p(), C.c_void_p()
        _check(self.lib.pwpp_host_results(self._h, C.byref(a), C.byref(b), C.byref(c)))
        total, nf = int(sum(self._n)), len(self._n)
        idx = np.ctypeslib.as_array((C.c_int32 * max(total, 1)).from_address(a.value))[:total]
        ng = np.ctypeslib.as_array((C.c_int32 * nf).from_address(b.value))
        off = np.ctypeslib.as_array((C.c_int64 * (nf + 1)).from_address(c.value))
        return idx, ng, off

    def device_results(self):
        a, b = C.c_void_p(), C.c_void_p()
        _check(self.lib.pwpp_device_results(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    ORDER_BIN, ORDER_REFERENCE = 0, 1

    def set_output_order(self, order: int):
        """ORDER_BIN (default): ascending point index inside a bin; ORDER_REFERENCE: the reference's z order (pwpp.h)."""
        _check(self.lib.pwpp_set_output_order(self._h, order))

    NUM_STAGES = 11

    def set_profiling(self, on: bool):
        _check(self.lib.pwpp_set_profiling(self._h, 1 if on else 0))

    def stage_times_ms(self):
        arr = (C.c_float * self.NUM_STAGES)()
        _check(self.lib.pwpp_stage_times_ms(self._h, arr))
        return {self.lib.pwpp_stage_name(i).decode(): float(arr[i]) for i in range(self.NUM_STAGES)}

    def launch_count(self) -> int:
        return int(self.lib.pwpp_launch_count(self._h))

    def reset(self, f=None):
        _check(self.lib.pwpp_reset_all(self._h) if f is None else self.lib.pwpp_reset_stream(self._h, f))
