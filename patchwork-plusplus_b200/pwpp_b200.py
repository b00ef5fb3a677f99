"""Thin ctypes front-end of the C-ABI in include/pwpp.h (lib/libpwpp_b200.so).

Used by tests/ and bench.py to call the product exactly as a foreign-language host would: plain
pointers and sizes, no torch types. The CUDA library is REQUIRED: loading fails loudly when it is
missing and creating an Engine fails loudly without a CUDA device — there is no CPU fallback.
"""
import ctypes as C
import os

import numpy as np

from pwpp_ctypes import PwppBinResult, PwppBoundGetters, PwppParams, PwppPointLayout, PwppScanRing, PwppState, default_params  # noqa: F401

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
    lib.pwpp_set_arithmetic.argtypes = [vp, i32]; lib.pwpp_set_arithmetic.restype = i32
    lib.pwpp_arithmetic.argtypes = [vp]; lib.pwpp_arithmetic.restype = i32
    lib.pwpp_order_exact_counts.argtypes = [vp, vp, i32]; lib.pwpp_order_exact_counts.restype = i32
    lib.pwpp_host_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]; lib.pwpp_host_results.restype = i32
    lib.pwpp_bind_host_to_device.argtypes = [i32]; lib.pwpp_bind_host_to_device.restype = i32
    lib.pwpp_bind_call.argtypes = [vp, i32, vp, vp, vp, vp, vp]; lib.pwpp_bind_call.restype = i32
    lib.pwpp_bind_call_actions.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp]; lib.pwpp_bind_call_actions.restype = i32
    lib.pwpp_bind_call_rings.argtypes = [vp, i32, vp, C.POINTER(PwppScanRing), vp, vp, vp, vp]; lib.pwpp_bind_call_rings.restype = i32
    lib.pwpp_bound_call_slots.argtypes = [vp, C.POINTER(vp)]; lib.pwpp_bound_call_slots.restype = i32
    lib.pwpp_bind_call_packed.argtypes = [vp, i32, vp, vp, C.POINTER(PwppPointLayout), i64, vp, vp, vp]; lib.pwpp_bind_call_packed.restype = i32
    lib.pwpp_bind_stream_table.argtypes = [vp, vp]; lib.pwpp_bind_stream_table.restype = i32
    lib.pwpp_bound_call_streams.argtypes = [vp, C.POINTER(vp)]; lib.pwpp_bound_call_streams.restype = i32
    lib.pwpp_bind_packed_xyz.argtypes = [vp, i32]; lib.pwpp_bind_packed_xyz.restype = i32
    lib.pwpp_bound_packed_xyz.argtypes = [vp] + [C.POINTER(vp)] * 4; lib.pwpp_bound_packed_xyz.restype = i32
    lib.pwpp_bind_packed_records.argtypes = [vp, i32]; lib.pwpp_bind_packed_records.restype = i32
    lib.pwpp_bound_packed_records.argtypes = [vp] + [C.POINTER(vp)] * 4 + [C.POINTER(i32)]; lib.pwpp_bound_packed_records.restype = i32
    lib.pwpp_run_bound_call.argtypes = [vp, vp]; lib.pwpp_run_bound_call.restype = i32
    lib.pwpp_bound_call_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]; lib.pwpp_bound_call_results.restype = i32
    lib.pwpp_unbind_call.argtypes = [vp]; lib.pwpp_unbind_call.restype = i32
    lib.pwpp_select_bound_call.argtypes = [vp, i32]; lib.pwpp_select_bound_call.restype = i32
    lib.pwpp_selected_bound_call.argtypes = [vp]; lib.pwpp_selected_bound_call.restype = i32
    lib.pwpp_bind_width_ladder.argtypes = [vp, i32, vp]; lib.pwpp_bind_width_ladder.restype = i32
    lib.pwpp_bound_call_width.argtypes = [vp, C.POINTER(vp)]; lib.pwpp_bound_call_width.restype = i32
    lib.pwpp_bind_record_results.argtypes = [vp, i32]; lib.pwpp_bind_record_results.restype = i32
    lib.pwpp_bound_record_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    lib.pwpp_bound_record_results.restype = i32
    lib.pwpp_bind_getter_results.argtypes = [vp, i32]; lib.pwpp_bind_getter_results.restype = i32
    lib.pwpp_bound_getter_results.argtypes = [vp, C.POINTER(PwppBoundGetters)]; lib.pwpp_bound_getter_results.restype = i32
    lib.pwpp_export_states_device.argtypes = [vp, i32, vp, vp, i64, vp, vp]; lib.pwpp_export_states_device.restype = i32
    lib.pwpp_import_states_device.argtypes = [vp, i32, vp, vp, i64, vp, vp]; lib.pwpp_import_states_device.restype = i32
    lib.pwpp_clone.argtypes = [vp, i32, C.POINTER(vp)]; lib.pwpp_clone.restype = i32
    _lib = lib
    return lib


def bind_host_to_device(device: int) -> int:
    """pwpp_bind_host_to_device: pin the calling thread to the CPUs of the GPU's NUMA node (returns the node or -1)."""
    return int(load_library().pwpp_bind_host_to_device(device))


class PwppError(RuntimeError):
    pass


# per-frame actions of a bound call and the status values they leave (PWPP_FRAME_* / PWPP_ACTION_INVALID of include/pwpp.h)
FRAME_RUN, FRAME_SKIP, FRAME_RESET = 0, 1, 2
FRAME_SKIPPED, ACTION_INVALID = 2, 3
SLOT_OUT_OF_RANGE = 4   # status of a ring-bound frame whose slot is outside its ring (PWPP_SLOT_OUT_OF_RANGE)
STREAM_OUT_OF_RANGE, STREAM_DUPLICATE = 6, 7   # statuses of a stream table's rejected frames (PWPP_STREAM_*)


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


MAX_BOUND_CALLS = 32   # PWPP_MAX_BOUND_CALLS
MAX_LADDER_WIDTHS = 8  # PWPP_MAX_LADDER_WIDTHS


class _BoundCall:
    """What the Engine keeps of one bound call of the ctx (pwpp_select_bound_call)."""

    def __init__(self):
        self.call = None            # (frames, counts, streams, sum of max_n) of the bind
        self.actions = None         # its actions tensor (bind_call(actions=...)), kept alive while bound
        self.rings = None           # its ring tensors and slots (bind_call_rings), kept alive while bound
        self.streams = None         # its stream table (bind_stream_table), kept alive while bound
        self.table_streams = None   # Engine._streams while its last run is the last call and it has a stream table


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
        self.device = device
        self.num_streams = num_streams
        self.nbins = self.lib.pwpp_num_bins(h)   # with several sets: the largest bin count of the sets
        self._n = []
        self._streams = []   # stream of every frame of the last call
        self._rec_dtypes = []   # record dtype of every frame of the last records call (uint8 rows of point_step for (buffer, layout) frames)
        self._calls = [_BoundCall() for _ in range(MAX_BOUND_CALLS)]
        self._sel = 0       # the selected bound call (select_bound_call)
        self._last = None   # the _BoundCall that ran last (run_bound_call / bound_call_results)

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

    # ---- bound call: frame sizes read on the GPU, capturable into a CUDA graph ----
    def bind_call(self, frames, max_n, layouts, counts, streams=None, actions=None):
        """Binds a call whose frame sizes live on the device (pwpp_bind_call). Frame f is up to max_n[f] records of layouts[f] at
        `frames[f]` (a device address or a CUDA tensor, any alignment), its size counts[f] of `counts`, an int64 CUDA tensor of
        nframes entries read by the GPU at every run. `streams` as for estimate_host (None: frame f on stream f). `actions`: an
        optional int32 CUDA tensor of nframes per-frame actions read by the GPU at every run (pwpp_bind_call_actions):
        FRAME_RUN, FRAME_SKIP (the frame is left out, its stream keeps its state) or FRAME_RESET (reset the stream, then run the
        frame). The tensors are kept alive while the call is bound; their contents may change between runs."""
        import torch
        nf = len(frames)
        if not (isinstance(counts, torch.Tensor) and counts.is_cuda and counts.dtype == torch.int64 and counts.is_contiguous()
                and counts.numel() == nf):
            raise PwppError(f"counts must be a contiguous int64 CUDA tensor of {nf} entries")
        if actions is not None and not (isinstance(actions, torch.Tensor) and actions.is_cuda and actions.dtype == torch.int32
                                        and actions.is_contiguous() and actions.numel() == nf):
            raise PwppError(f"actions must be a contiguous int32 CUDA tensor of {nf} entries")
        ids = np.arange(nf, dtype=np.int32) if streams is None else self._stream_table(streams, nf)
        ptrs = [int(fr.data_ptr()) if isinstance(fr, torch.Tensor) else int(fr) for fr in frames]
        p = (C.c_void_p * max(nf, 1))(*ptrs)
        n = (C.c_int64 * max(nf, 1))(*[int(k) for k in max_n])
        lays = (PwppPointLayout * max(nf, 1))(*layouts)
        if actions is None:
            _check(self.lib.pwpp_bind_call(self._h, nf, ids.ctypes.data, p, n, lays, C.c_void_p(counts.data_ptr())))
        else:
            _check(self.lib.pwpp_bind_call_actions(self._h, nf, ids.ctypes.data, p, n, lays, C.c_void_p(counts.data_ptr()),
                                                   C.c_void_p(actions.data_ptr())))
        self._call.call = (list(frames), counts, ids.tolist(), sum(int(k) for k in max_n))
        self._call.actions = actions

    def bind_call_rings(self, rings, max_n, layouts, slots, streams=None, actions=None):
        """Binds a call whose frames live in scan rings (pwpp_bind_call_rings): at every run or replay frame f reads slot
        slots[f] of rings[f] and segments the records written there. A ring is (buffer, counts) or (buffer, counts, slot_stride):
        buffer a contiguous CUDA tensor holding the slots (without slot_stride: its first dimension is the slot, e.g. uint8
        (num_slots, slot_stride)), counts a contiguous int64 CUDA tensor of num_slots record counts read by the GPU, slot_stride
        the bytes from one slot to the next. Frame f holds up to max_n[f] records of layouts[f]. `slots`: a contiguous int32 CUDA
        tensor of nframes slot numbers read by the GPU at every run. `streams` and `actions` as for bind_call. The tensors are
        kept alive while the call is bound; the slots, the counts and the slots' contents may change between runs."""
        import torch
        nf = len(rings)

        def cuda_vec(t, dtype, n, what):
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous() and (n is None or t.numel() == n)):
                raise PwppError(f"{what} must be a contiguous {str(dtype).replace('torch.', '')} CUDA tensor" + (f" of {n} entries" if n else ""))
        cuda_vec(slots, torch.int32, nf, "slots")
        if actions is not None:
            cuda_vec(actions, torch.int32, nf, "actions")
        if len(max_n) != nf or len(layouts) != nf:
            raise PwppError(f"max_n and layouts must name one entry per ring ({nf})")
        descs = (PwppScanRing * max(nf, 1))()
        for f, ring in enumerate(rings):
            if not isinstance(ring, tuple) or len(ring) not in (2, 3):
                raise PwppError(f"ring {f}: a ring is (buffer, counts) or (buffer, counts, slot_stride)")
            buf, counts = ring[:2]
            if not (isinstance(buf, torch.Tensor) and buf.is_cuda and buf.is_contiguous()):
                raise PwppError(f"ring {f}: buffer must be a contiguous CUDA tensor")
            cuda_vec(counts, torch.int64, None, f"ring {f}: counts")
            num_slots = counts.numel()
            nbytes = buf.numel() * buf.element_size()
            if len(ring) == 3:
                stride = int(ring[2])
            else:
                if buf.dim() < 1 or buf.shape[0] != num_slots:
                    raise PwppError(f"ring {f}: buffer's first dimension must be the {num_slots} slots of counts")
                stride = nbytes // num_slots if num_slots else 0
            need = (num_slots - 1) * stride + int(max_n[f]) * layouts[f].point_step
            if num_slots >= 1 and int(max_n[f]) > 0 and need > nbytes:
                raise PwppError(f"ring {f}: {num_slots} slots of stride {stride} with max_n {int(max_n[f])} reach {need} bytes, "
                                f"past the buffer's {nbytes}")
            descs[f].base, descs[f].slot_stride = buf.data_ptr(), stride
            descs[f].d_counts, descs[f].num_slots = counts.data_ptr(), num_slots
        ids = np.arange(nf, dtype=np.int32) if streams is None else self._stream_table(streams, nf)
        n = (C.c_int64 * max(nf, 1))(*[int(k) for k in max_n])
        lays = (PwppPointLayout * max(nf, 1))(*layouts)
        _check(self.lib.pwpp_bind_call_rings(self._h, nf, ids.ctypes.data, descs, n, lays, C.c_void_p(slots.data_ptr()),
                                             C.c_void_p(actions.data_ptr() if actions is not None else None)))
        self._call.call = ([r[0] for r in rings], None, ids.tolist(), sum(int(k) for k in max_n))
        self._call.actions = actions
        self._call.rings = (list(rings), slots)

    def bind_call_packed(self, points, offsets, max_n, layout=None, streams=None, actions=None):
        """Binds a call over one packed batch (pwpp_bind_call_packed): at every run or replay frame f is records
        [offsets[f], offsets[f + 1]) of `points`, read by the GPU. `points` is a contiguous CUDA tensor; a float32 (N, 4) or (N, 3)
        tensor gives its layout (x, y, z[, intensity]), any other needs `layout` (a PwppPointLayout), and the buffer holds
        nbytes // point_step records. `offsets`: a contiguous int64 CUDA tensor of nframes + 1 entries. Frame f holds up to
        max_n[f] records. `streams` and `actions` as for bind_call. The tensors are kept alive while the call is bound; the
        offsets and the records may change between runs."""
        import torch
        nf = len(max_n)
        if not (isinstance(points, torch.Tensor) and points.is_cuda and points.is_contiguous()):
            raise PwppError("points must be a contiguous CUDA tensor")
        if not (isinstance(offsets, torch.Tensor) and offsets.is_cuda and offsets.dtype == torch.int64 and offsets.is_contiguous()
                and offsets.numel() == nf + 1):
            raise PwppError(f"offsets must be a contiguous int64 CUDA tensor of {nf + 1} entries")
        if actions is not None and not (isinstance(actions, torch.Tensor) and actions.is_cuda and actions.dtype == torch.int32
                                        and actions.is_contiguous() and actions.numel() == nf):
            raise PwppError(f"actions must be a contiguous int32 CUDA tensor of {nf} entries")
        if layout is None:
            if points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] not in (3, 4):
                raise PwppError("points needs a layout unless it is a float32 (N, 4) or (N, 3) tensor")
            cols = int(points.shape[1])
            layout = layout_from_dtype(np.dtype({"names": ["x", "y", "z", "intensity"][:cols], "formats": ["<f4"] * cols,
                                                 "offsets": [0, 4, 8, 12][:cols], "itemsize": 4 * cols}))
        capacity = points.numel() * points.element_size() // layout.point_step if layout.point_step > 0 else 0
        ids = np.arange(nf, dtype=np.int32) if streams is None else self._stream_table(streams, nf)
        n = (C.c_int64 * max(nf, 1))(*[int(k) for k in max_n])
        _check(self.lib.pwpp_bind_call_packed(self._h, nf, ids.ctypes.data, C.c_void_p(points.data_ptr()), C.byref(layout), capacity, n,
                                              C.c_void_p(offsets.data_ptr()), C.c_void_p(actions.data_ptr() if actions is not None else None)))
        self._call.call = ([points] * nf, offsets, ids.tolist(), sum(int(k) for k in max_n))
        self._call.actions = actions

    def bind_packed_xyz(self, ground: bool = True, nonground: bool = True):
        """Enables packed xyz results for the bound call (pwpp_bind_packed_xyz): every later run_bound_call, and every graph
        captured after this, also writes each part's xyz rows of all frames back to back and their device offsets. Host work
        that synchronizes: call it before a capture."""
        _check(self.lib.pwpp_bind_packed_xyz(self._h, (1 if ground else 0) | (2 if nonground else 0)))

    def bound_packed_xyz(self):
        """Zero-copy views of the packed xyz results (pwpp_bound_packed_xyz), as a dict: ground / nonground float32 CUDA tensors
        (sum(max_n), 3) and ground_offsets / nonground_offsets int64 CUDA tensors (nframes + 1,), None for a part that is not
        enabled. After a run or replay frame f's non-ground cloud is nonground[nonground_offsets[f]:nonground_offsets[f + 1]].
        Fixed addresses while the call is bound."""
        import torch
        ptrs = [C.c_void_p() for _ in range(4)]
        _check(self.lib.pwpp_bound_packed_xyz(self._h, *[C.byref(p) for p in ptrs]))
        nf, rows = len(self._call.call[0]), self._call.call[3]

        class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
            def __init__(self, ptr, shape, typestr):
                self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}

        def view(ptr, shape, typestr):
            if not ptr:
                return None
            if 0 in shape:
                return torch.empty(shape, dtype=torch.float32, device="cuda")
            return torch.as_tensor(_View(ptr, shape, typestr), device="cuda")
        g, n, go, no = (p.value for p in ptrs)
        return {"ground": view(g, (rows, 3), "<f4"), "nonground": view(n, (rows, 3), "<f4"),
                "ground_offsets": view(go, (nf + 1,), "<i8"), "nonground_offsets": view(no, (nf + 1,), "<i8")}

    def bind_packed_records(self, ground: bool = True, nonground: bool = True):
        """Enables packed records for the bound call (pwpp_bind_packed_records): every later run_bound_call, and every graph
        captured after this, also writes each part's records of all frames back to back, in the sensor's own layout, and their
        device offsets. Every frame of the call must have the same point_step. Host work that synchronizes: call it before a
        capture."""
        _check(self.lib.pwpp_bind_packed_records(self._h, (1 if ground else 0) | (2 if nonground else 0)))

    def bound_packed_records(self):
        """Zero-copy views of the packed records (pwpp_bound_packed_records), as a dict: ground / nonground uint8 CUDA tensors
        (sum(max_n), point_step) and ground_offsets / nonground_offsets int64 CUDA tensors (nframes + 1,), None for a part that
        is not enabled, and point_step. After a run or replay frame f's non-ground records are
        nonground[nonground_offsets[f]:nonground_offsets[f + 1]]. For a 16-byte float32 layout (x, y, z, intensity),
        nonground.view(torch.float32) is the (sum(max_n), 4) xyzi batch and nonground_offsets its batch offsets. The offsets are
        those of bound_packed_xyz when both are enabled. Fixed addresses while the call is bound."""
        import torch
        ptrs = [C.c_void_p() for _ in range(4)]
        step = C.c_int32()
        _check(self.lib.pwpp_bound_packed_records(self._h, *[C.byref(p) for p in ptrs], C.byref(step)))
        nf, rows, step = len(self._call.call[0]), self._call.call[3], step.value

        class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
            def __init__(self, ptr, shape, typestr):
                self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}

        def view(ptr, shape, typestr, dtype):
            if not ptr:
                return None
            if 0 in shape:
                return torch.empty(shape, dtype=dtype, device="cuda")
            return torch.as_tensor(_View(ptr, shape, typestr), device="cuda")
        g, n, go, no = (p.value for p in ptrs)
        return {"ground": view(g, (rows, step), "|u1", torch.uint8), "nonground": view(n, (rows, step), "|u1", torch.uint8),
                "ground_offsets": view(go, (nf + 1,), "<i8", torch.int64), "nonground_offsets": view(no, (nf + 1,), "<i8", torch.int64),
                "point_step": step}

    def bound_call_slots(self):
        """Torch view (int32 [nframes]) of the slots the last run read (pwpp_bound_call_slots): the run's own copy, -1 where the
        action skipped the frame. Fixed address while the call is bound."""
        import torch
        a = C.c_void_p()
        _check(self.lib.pwpp_bound_call_slots(self._h, C.byref(a)))
        nf = len(self._call.call[0])

        class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
            def __init__(self, ptr, n):
                self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3, "strides": None}
        return torch.as_tensor(_View(a.value, nf), device="cuda")

    def bind_stream_table(self, streams):
        """Reads every frame's stream of the bound call from `streams`, a contiguous int32 CUDA tensor of nframes entries, at every
        run or replay (pwpp_bind_stream_table): -1 leaves the frame out, an id >= num_streams or a second frame of one run on the
        same stream is skipped with STREAM_OUT_OF_RANGE / STREAM_DUPLICATE. The runs stay those of the bound streams. Call it
        before the bound call's first run; the tensor is kept alive while bound and its contents may change between runs."""
        import torch
        if self._call.call is None:
            raise PwppError("no call is bound")
        nf = len(self._call.call[2])
        if not (isinstance(streams, torch.Tensor) and streams.is_cuda and streams.dtype == torch.int32 and streams.is_contiguous()
                and streams.numel() == nf):
            raise PwppError(f"streams must be a contiguous int32 CUDA tensor of {nf} entries")
        _check(self.lib.pwpp_bind_stream_table(self._h, C.c_void_p(streams.data_ptr())))
        self._call.streams = streams

    def bound_call_streams(self):
        """Torch view (int32 [nframes]) of the streams the last run read (pwpp_bound_call_streams): the run's own copy, invalid ids
        included, -1 before the first run. Fixed address while the call is bound."""
        import torch
        a = C.c_void_p()
        _check(self.lib.pwpp_bound_call_streams(self._h, C.byref(a)))
        nf = len(self._call.call[2])

        class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
            def __init__(self, ptr, n):
                self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3, "strides": None}
        return torch.as_tensor(_View(a.value, nf), device="cuda")

    def bind_width_ladder(self, widths):
        """Lets the GPU pick, at every run or replay, how many positions the bound call launches (pwpp_bind_width_ladder): the
        narrowest of `widths` (strictly increasing, each in [1, nframes); nframes is always the last width) that holds every
        position its table kernel did not reject. Results are bit for bit those of the call without a ladder. The call needs
        actions or a stream table; enable result buffers and the stream table first. Host work that synchronizes."""
        if self._call.call is None:
            raise PwppError("no call is bound")
        w = np.ascontiguousarray(widths, dtype=np.int32)
        _check(self.lib.pwpp_bind_width_ladder(self._h, len(w), w.ctypes.data))

    def bound_call_width(self):
        """Torch view (int32 [1]) of the width the last run launched (pwpp_bound_call_width): nframes without a ladder, 0 after
        the ladder's enable until its first run. Fixed address while the call is bound."""
        import torch
        a = C.c_void_p()
        _check(self.lib.pwpp_bound_call_width(self._h, C.byref(a)))

        class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
            def __init__(self, ptr):
                self.__cuda_array_interface__ = {"shape": (1,), "typestr": "<i4", "data": (ptr, False), "version": 3, "strides": None}
        return torch.as_tensor(_View(a.value), device="cuda")

    def run_bound_call(self, stream: int = 0):
        """Enqueues the bound call on CUDA stream `stream` (0: the ctx's own stream; inside torch.cuda.graph pass
        torch.cuda.current_stream().cuda_stream). No host synchronisation: it may be captured and replayed."""
        _check(self.lib.pwpp_run_bound_call(self._h, C.c_void_p(stream)))
        self._use_bound()

    def bound_call_results(self):
        """Torch views of the bound call's device results (pwpp_bound_call_results): (indices int32[sum(max_n)], offsets
        int64[nframes + 1], num_ground int32[nframes], status int32[nframes]). Frame f's lists start at offsets[f]: ground,
        then non-ground. Fixed addresses while the call is bound. Also makes the bound call the last call of the host getters."""
        import torch
        a, b, c, d = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        _check(self.lib.pwpp_bound_call_results(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        self._use_bound()
        frames, _, _, cap = self._call.call
        nf = len(frames)

        class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
            def __init__(self, ptr, n, typestr):
                self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}
        idx = torch.as_tensor(_View(a.value, cap, "<i4"), device="cuda") if cap > 0 else torch.empty(0, dtype=torch.int32, device="cuda")
        return (idx, torch.as_tensor(_View(b.value, nf + 1, "<i8"), device="cuda"), torch.as_tensor(_View(c.value, nf, "<i4"), device="cuda"),
                torch.as_tensor(_View(d.value, nf, "<i4"), device="cuda"))

    def bind_record_results(self, ground: bool = True, nonground: bool = True):
        """Enables the bound call's record results (pwpp_bind_record_results): every later run_bound_call, and every graph captured
        after this, also gathers the ground and / or non-ground records of every frame into fixed device buffers. Host work
        that synchronizes: call it before a capture, not inside one."""
        parts = (1 if ground else 0) | (2 if nonground else 0)
        _check(self.lib.pwpp_bind_record_results(self._h, parts))

    def bound_record_results(self):
        """(ground, nonground, offsets, counts) of the bound call's record results (pwpp_bound_record_results): ground and
        nonground are zero-copy uint8 CUDA tensors of offsets[-1] bytes (None for a part that is not enabled), offsets int64
        numpy [nframes + 1] (frame f's region of each starts at offsets[f]), counts an int32 CUDA tensor view (nframes, 2) of
        every frame's ground and non-ground record counts. Frame f's non-ground cloud after a run or replay is
        nonground[offsets[f]: offsets[f] + counts[f, 1] * point_step]. Fixed addresses while the call is bound."""
        import torch
        a, b, c, d = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        _check(self.lib.pwpp_bound_record_results(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        nf = len(self._call.call[0])
        off = np.ctypeslib.as_array((C.c_int64 * (nf + 1)).from_address(c.value)).copy()
        total = int(off[-1])

        class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
            def __init__(self, ptr, shape, typestr):
                self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}

        def part(ptr):
            if not ptr:
                return None
            return torch.as_tensor(_View(ptr, (total,), "|u1"), device="cuda") if total > 0 else torch.empty(0, dtype=torch.uint8, device="cuda")
        return part(a.value), part(b.value), off, torch.as_tensor(_View(d.value, (nf, 2), "<i4"), device="cuda")

    def bind_getter_results(self, ground_xyz: bool = True, nonground_xyz: bool = True, state: bool = True):
        """Enables the bound call's getter results (pwpp_bind_getter_results): every later run_bound_call, and every graph
        captured after this, also writes the ground and / or non-ground xyz of every frame and / or the state of every frame's
        stream right after the frame into fixed device buffers. Host work that synchronizes: call it before a capture."""
        what = (1 if ground_xyz else 0) | (2 if nonground_xyz else 0) | (4 if state else 0)
        _check(self.lib.pwpp_bind_getter_results(self._h, what))

    def bound_getter_results(self):
        """Zero-copy views of the bound call's getter results (pwpp_bound_getter_results), as a dict. Fixed addresses while the
        call is bound; valid after a run or replay until the next one.
          ground_xyz, nonground_xyz: float32 CUDA tensors (sum(max_n), 3), None for a part that is not enabled;
          row_off: int64 numpy [nframes + 1], frame f's rows start at row_off[f];
          xyz_counts: int32 CUDA tensor (nframes, 2), ground and non-ground rows of every frame (None without an xyz part),
            so frame f's non-ground cloud is nonground_xyz[row_off[f]:][:xyz_counts[f, 1]];
          centers, normals: float32 CUDA tensors (nframes, patch_row_stride, 3), num_patches int32 [nframes]: frame f's patches
            are centers[f, :num_patches[f]];
          height (nframes,), elevation_thr, flatness_thr (nframes, 4) float64 and n_elevation, n_flatness (nframes, 4) int32:
            strided CUDA views of the state rows (None when the state is not enabled), row f the state of frame f's stream
            right after frame f."""
        import torch
        g = PwppBoundGetters()
        _check(self.lib.pwpp_bound_getter_results(self._h, C.byref(g)))
        nf = len(self._call.call[0])
        row_off = np.ctypeslib.as_array((C.c_int64 * (nf + 1)).from_address(g.h_row_off)).copy()
        rows, stride = int(row_off[-1]), int(g.patch_row_stride)

        class _View:   # __cuda_array_interface__ v3: torch.as_tensor wraps the memory without copying
            def __init__(self, ptr, shape, typestr, strides=None):
                self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3, "strides": strides}

        def view(ptr, shape, typestr, strides=None):
            if not ptr:
                return None
            if 0 in shape:
                return torch.empty(shape, dtype={"<f4": torch.float32, "<f8": torch.float64, "<i4": torch.int32}[typestr], device="cuda")
            return torch.as_tensor(_View(ptr, shape, typestr, strides), device="cuda")
        st = C.sizeof(PwppState)
        s = g.states
        return {"ground_xyz": view(g.ground_xyz, (rows, 3), "<f4"), "nonground_xyz": view(g.nonground_xyz, (rows, 3), "<f4"),
                "row_off": row_off, "xyz_counts": view(g.xyz_counts, (nf, 2), "<i4"),
                "centers": view(g.centers, (nf, stride, 3), "<f4"), "normals": view(g.normals, (nf, stride, 3), "<f4"),
                "num_patches": view(g.num_patches, (nf,), "<i4"),
                "height": view(s, (nf,), "<f8", (st,)),
                "elevation_thr": view(s and s + PwppState.elevation_thr.offset, (nf, 4), "<f8", (st, 8)),
                "flatness_thr": view(s and s + PwppState.flatness_thr.offset, (nf, 4), "<f8", (st, 8)),
                "n_elevation": view(s and s + PwppState.n_elevation.offset, (nf, 4), "<i4", (st, 4)),
                "n_flatness": view(s and s + PwppState.n_flatness.offset, (nf, 4), "<i4", (st, 4))}

    def unbind_call(self):
        """Releases the selected bound call (pwpp_unbind_call). When it ran last, the host getters keep serving its results."""
        if self._streams is self._call.table_streams:
            # the last call keeps its host getters after the unbind: name the streams its frames read (an invalid id: the bound
            # stream, whose set the frame ran with), so bin_results sizes the records of each frame's set without the table
            self.synchronize()
            read = self.bound_call_streams().cpu().tolist()
            self._streams = [s if 0 <= s < self.num_streams else b for s, b in zip(read, self._call.call[2])]
        _check(self.lib.pwpp_unbind_call(self._h))
        self._calls[self._sel] = _BoundCall()

    def select_bound_call(self, k: int):
        """Selects bound call k of the ctx, 0 <= k < MAX_BOUND_CALLS (pwpp_select_bound_call): the bind, run, result and unbind
        methods act on it. Host-only. Call 0 is selected at creation. A graph captured from run_bound_call holds the call that was
        selected at capture. The calls share the streams, the scratch slots and the work buffers (include/pwpp.h)."""
        _check(self.lib.pwpp_select_bound_call(self._h, int(k)))
        self._sel = int(k)

    @property
    def selected_bound_call(self) -> int:
        return self._sel

    @property
    def _call(self):
        return self._calls[self._sel]

    def _use_bound(self):
        """The host getters now serve the selected bound call: its frame sizes are fetched from the device when first needed."""
        self._n = None
        self._streams = list(self._call.call[2])
        self._rec_dtypes = []
        self._call.table_streams = self._streams if self._call.streams is not None else None   # bin_results: sets read on the device
        self._last = self._call

    def _last_call_streams(self):
        """bound_call_streams of the call that ran last, whichever call is selected."""
        sel = self._sel
        self.select_bound_call(self._calls.index(self._last))
        try:
            return self.bound_call_streams()
        finally:
            self.select_bound_call(sel)

    def _sizes(self):
        """Point count of every frame of the last call (after a bound call: from its device offsets, one device->host copy)."""
        if self._n is None:
            a, b, c = C.c_void_p(), C.c_void_p(), C.c_void_p()
            _check(self.lib.pwpp_host_results(self._h, C.byref(a), C.byref(b), C.byref(c)))
            nf = len(self._streams)
            self._n = np.diff(np.ctypeslib.as_array((C.c_int64 * (nf + 1)).from_address(c.value))).tolist()
        return self._n

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
        if self._last is not None and self._streams is self._last.table_streams:
            # a stream table: the C-ABI writes the bins of the set the frame ran with; the stream it read names that set (an
            # invalid id: its bound stream's)
            arr = (PwppBinResult * self.nbins)()
            _check(self.lib.pwpp_copy_bin_results(self._h, f, C.byref(arr)))
            s = int(self._last_call_streams()[f])
            nb = self.stream_num_bins(s if 0 <= s < self.num_streams else self._streams[f])
            return (PwppBinResult * nb).from_buffer(arr)
        nb = self.stream_num_bins(self._streams[f]) if 0 <= f < len(self._streams) else self.nbins   # (a bad f: the C-ABI reports it)
        arr = (PwppBinResult * nb)()
        _check(self.lib.pwpp_copy_bin_results(self._h, f, C.byref(arr)))
        return arr

    def bin_ids(self, f=0):
        n = self._sizes()[f]
        out = np.empty(n, dtype=np.uint16)
        if n > 0:
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

    # ---- stream state on the GPU (pwpp_export_states_device / pwpp_import_states_device / pwpp_clone) ----
    STATE_OK, STATE_SKIPPED, STATE_OUT_OF_RANGE, STATE_BLOB_MISMATCH, STATE_DUPLICATE = 0, 1, 2, 3, 4

    def state_blob_size(self) -> int:
        """pwpp_state_blob_size: the largest stream blob of the ctx (a row of export_states holds any stream's)."""
        return int(self.lib.pwpp_state_blob_size(self._h))

    def _state_list(self, streams):
        """The stream list as a device int32 tensor: a device tensor is used as it is (a graph may rewrite it between replays),
        anything else is copied to the ctx's device (not capturable)."""
        import torch
        if isinstance(streams, torch.Tensor) and streams.is_cuda:
            if streams.dtype != torch.int32 or streams.dim() != 1 or not streams.is_contiguous():
                raise PwppError("a device stream list must be a contiguous 1-D int32 tensor")
            return streams
        return torch.as_tensor(np.ascontiguousarray(streams, dtype=np.int32).reshape(-1), device=torch.device("cuda", self.device))

    def _torch_stream(self, stream):
        """`stream`, or for 0 torch's current stream on the ctx's device (its legacy default stream as cudaStreamLegacy), so that
        the lists and rows torch wrote and the status tensors returned are ordered with torch's own work."""
        import torch
        if stream:
            return stream
        return torch.cuda.current_stream(self.device).cuda_stream or 1

    @staticmethod
    def _blob_rows(t, what):
        import torch
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.uint8 and t.dim() == 2 and t.stride(1) == 1):
            raise PwppError(f"{what} must be a CUDA uint8 tensor [n, row_bytes] with contiguous rows")
        return t.stride(0)

    def export_states(self, streams, out=None, stream: int = 0):
        """The complete state of stream streams[i] into row i of a device uint8 tensor [n, stride] (stride: the state blob size
        rounded up to 16 bytes, or out's row stride), each row byte for byte export_state's blob. Returns (rows, status int32[n]):
        STATE_OK, or STATE_SKIPPED (id < 0) / STATE_OUT_OF_RANGE, whose rows are not written. Enqueued on CUDA stream `stream`
        (0: torch's current stream) with no host synchronisation, so it may be captured into a CUDA graph. The ctx's own calls
        are ordered by the caller (estimate_host has finished when it returns)."""
        import torch
        ids = self._state_list(streams)
        n = ids.numel()
        if out is None:
            out = torch.empty((n, (self.state_blob_size() + 15) // 16 * 16), dtype=torch.uint8, device=ids.device)
        stride = self._blob_rows(out, "out")
        if out.shape[0] < n:
            raise PwppError(f"out holds {out.shape[0]} rows, the list {n}")
        status = torch.empty(n, dtype=torch.int32, device=ids.device)
        _check(self.lib.pwpp_export_states_device(self._h, n, ids.data_ptr(), out.data_ptr(), stride, status.data_ptr(),
                                                  C.c_void_p(self._torch_stream(stream))))
        return out, status

    def import_states(self, blobs, streams, stream: int = 0):
        """Row i of the device uint8 tensor `blobs` into stream streams[i], checked on the GPU as import_state checks a blob.
        Returns the status int32[n]: STATE_OK, STATE_SKIPPED (id < 0: nothing read or written), STATE_OUT_OF_RANGE,
        STATE_BLOB_MISMATCH (stream untouched) or STATE_DUPLICATE (an earlier entry names the stream). Capturable; `stream` as
        for export_states. The host getters see the import once that stream has been synchronized."""
        import torch
        ids = self._state_list(streams)
        n = ids.numel()
        stride = self._blob_rows(blobs, "blobs")
        if blobs.shape[0] < n:
            raise PwppError(f"blobs holds {blobs.shape[0]} rows, the list {n}")
        status = torch.empty(n, dtype=torch.int32, device=ids.device)
        _check(self.lib.pwpp_import_states_device(self._h, n, ids.data_ptr(), blobs.data_ptr(), stride, status.data_ptr(),
                                                  C.c_void_p(self._torch_stream(stream))))
        return status

    def clone(self, device=None):
        """pwpp_clone: a new Engine on `device` (None: this one's) with this one's parameter sets, stream states and last call's
        results; both continue identically. Refused while a call is bound."""
        h = C.c_void_p()
        _check(self.lib.pwpp_clone(self._h, -1 if device is None else int(device), C.byref(h)))
        e = Engine.__new__(Engine)
        e.__dict__.update(self.__dict__)
        e._h, e.device = h, self.device if device is None else int(device)
        e.params = list(self.params) if isinstance(self.params, list) else self.params
        e._n, e._streams, e._rec_dtypes = None if self._n is None else list(self._n), list(self._streams), []
        e._calls, e._sel, e._last = [_BoundCall() for _ in range(MAX_BOUND_CALLS)], 0, None   # a clone holds no bound call
        return e

    def device_index_lists(self):
        """Zero-copy view of the last call's results on the device: (indices, num_ground) as torch int32 CUDA tensors.
        indices is laid out like the input (frame f's region starts at its point offset): ground list, then non-ground
        list. Valid until the next estimate call; the caller synchronizes with its stream (or Engine.synchronize())."""
        import torch
        d_idx, d_ng = self.device_results()
        total, nf = int(sum(self._sizes())), len(self._sizes())

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
        total, nf = int(sum(self._sizes())), len(self._sizes())
        idx = np.ctypeslib.as_array((C.c_int32 * max(total, 1)).from_address(a.value))[:total]
        ng = np.ctypeslib.as_array((C.c_int32 * nf).from_address(b.value))
        off = np.ctypeslib.as_array((C.c_int64 * (nf + 1)).from_address(c.value))
        return idx, ng, off

    def device_results(self):
        a, b = C.c_void_p(), C.c_void_p()
        _check(self.lib.pwpp_device_results(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    ORDER_BIN, ORDER_REFERENCE, ORDER_REFERENCE_EXACT = 0, 1, 2

    def set_output_order(self, order: int):
        """ORDER_BIN (default): ascending point index inside a bin; ORDER_REFERENCE: the reference's z order, equal z in ascending
        point index; ORDER_REFERENCE_EXACT: the reference's z order with equal z as libstdc++'s std::sort leaves them (pwpp.h)."""
        _check(self.lib.pwpp_set_output_order(self._h, order))

    ARITH_DOUBLE, ARITH_REFERENCE = 0, 1

    def set_arithmetic(self, mode: int):
        """ARITH_DOUBLE (default): order-free double sums; ARITH_REFERENCE: the reference's fp32 arithmetic, every result bit for
        bit the reference build's (pwpp.h). Refused while a call is bound."""
        _check(self.lib.pwpp_set_arithmetic(self._h, mode))

    def arithmetic(self) -> int:
        return self.lib.pwpp_arithmetic(self._h)

    def order_exact_counts(self, reset: bool = False):
        """Counters of the ORDER_REFERENCE_EXACT fix-up: (patches simulated, heap fall-backs, NaN bins); synchronises the device."""
        out = np.zeros(3, np.uint64)
        _check(self.lib.pwpp_order_exact_counts(self._h, out.ctypes.data, 1 if reset else 0))
        return tuple(int(v) for v in out)

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
