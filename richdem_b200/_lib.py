"""ctypes binding of librichdem_b200.so (the C ABI in include/richdem_b200.h).

This is the only way the Python layer reaches the compute path.  There is no CPU fallback: if the
shared library is missing, or no H100 is visible, every call raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RICHDEM_B200_LIB") or os.path.join(_HERE, "librichdem_b200.so")

_lib = None


class RichdemB200Error(RuntimeError):
    """Raised for any non-zero status from the C ABI (mirrors the std::runtime_error ->
    RuntimeError translation pybind11 does for the reference, pywrapper.hpp:109-123)."""


class Stats(C.Structure):
    _fields_ = [
        ("cells", C.c_int64), ("kernel_launches", C.c_int64), ("fill_rounds", C.c_int64),
        ("fill_tile_visits", C.c_int64), ("fill_tile_cells", C.c_int64), ("fill_tile_iters", C.c_int64),
        ("accum_rounds", C.c_int64), ("flat_bfs_levels", C.c_int64), ("flat_cells_raised", C.c_int64),
        ("ms_total", C.c_double), ("ms_main_kernel", C.c_double), ("ms_h2d", C.c_double),
        ("ms_d2h", C.c_double),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


# every symbol include/richdem_b200.h declares: name -> argtypes (restype is int unless noted)
_i32, _f32, _f64, _vp = C.c_int32, C.c_float, C.c_double, C.c_void_p
SIGNATURES = {
    "rdb200_init": [C.c_int],
    "rdb200_set_stream": [C.c_void_p],
    "rdb200_get_stats": [C.POINTER(Stats)],
    "rdb200_set_param": [C.c_char_p, C.c_int64],
    "rdb200_fill_depressions_d8_f32": [_vp, _i32, _i32],
    "rdb200_fill_depressions_d4_f32": [_vp, _i32, _i32],
    "rdb200_dev_fill_depressions_d4_f32": [_vp, _i32, _i32],
    "rdb200_fill_depressions_epsilon_d8_f32": [_vp, _i32, _i32, _f32],
    "rdb200_fill_depressions_epsilon_d4_f32": [_vp, _i32, _i32, _f32],
    "rdb200_dev_fill_depressions_epsilon_d8_f32": [_vp, _i32, _i32, _f32],
    "rdb200_dev_fill_depressions_epsilon_d4_f32": [_vp, _i32, _i32, _f32],
    "rdb200_pit_mask_d8_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_pit_mask_d4_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_has_depressions_d8_f32": [_vp, _i32, _i32, C.POINTER(_i32)],
    "rdb200_has_depressions_d4_f32": [_vp, _i32, _i32, C.POINTER(_i32)],
    "rdb200_dev_pit_mask_d8_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_dev_pit_mask_d4_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_dev_has_depressions_d8_f32": [_vp, _i32, _i32, C.POINTER(_i32)],
    "rdb200_dev_has_depressions_d4_f32": [_vp, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_pit_mask_d8_f32": [_vp, _vp, _vp, _i32, _i32, _f32, _i32, _i32, _i32, _i32],
    "rdb200_mgpu_pit_mask_d4_f32": [_vp, _vp, _vp, _i32, _i32, _f32, _i32, _i32, _i32, _i32],
    "rdb200_mgpu_has_depressions_d8_f32": [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_has_depressions_d4_f32": [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_resolve_flats_epsilon_f32": [_vp, _i32, _i32, _f32],
    "rdb200_get_flat_mask_f32": [_vp, _vp, _vp, _i32, _i32, _f32],
    "rdb200_d8_flow_directions_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_d8_flow_directions_flats_f32": [_vp, _vp, _i32, _i32, _f32, _i32],
    "rdb200_dev_d8_flow_directions_flats_f32": [_vp, _vp, _i32, _i32, _f32, _i32],
    "rdb200_d8_flow_accum_u8_i32": [_vp, _vp, _i32, _i32],
    "rdb200_fm_d8_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_fm_tarboton_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_fm_d4_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_fm_quinn_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_fm_holmgren_f32": [_vp, _vp, _i32, _i32, _f32, C.c_double],
    "rdb200_fm_freeman_f32": [_vp, _vp, _i32, _i32, _f32, C.c_double],
    "rdb200_terrain_attribute_f32": [_i32, _vp, _vp, _i32, _i32, _f32, _f32, _f32, C.c_double, C.c_double],
    "rdb200_dev_terrain_attribute_f32": [_i32, _vp, _vp, _i32, _i32, _f32, _f32, _f32, C.c_double, C.c_double],
    "rdb200_fa_d4_f32_f64": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_fa_quinn_f32_f64": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_fa_holmgren_f32_f64": [_vp, _vp, _i32, _i32, _f32, C.c_double],
    "rdb200_fa_freeman_f32_f64": [_vp, _vp, _i32, _i32, _f32, C.c_double],
    "rdb200_dev_fm_method_f32": [_i32, _vp, _vp, _i32, _i32, _f32, C.c_double],
    "rdb200_dev_fa_method_f32_f64": [_i32, _vp, _vp, _i32, _i32, _f32, C.c_double],
    "rdb200_flow_accumulation_props_f64": [_vp, _vp, _i32, _i32],
    "rdb200_fa_d8_f32_f64": [_vp, _vp, _i32, _i32, _f32, _i32],
    "rdb200_fa_tarboton_f32_f64": [_vp, _vp, _i32, _i32, _f32, _i32],
    "rdb200_dev_fill_depressions_d8_f32": [_vp, _i32, _i32],
    "rdb200_dev_resolve_flats_epsilon_f32": [_vp, _i32, _i32, _f32],
    "rdb200_dev_d8_flow_directions_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_dev_d8_flow_accum_u8_i32": [_vp, _vp, _i32, _i32],
    "rdb200_dev_fm_d8_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_dev_fm_tarboton_f32": [_vp, _vp, _i32, _i32, _f32],
    "rdb200_dev_flow_accumulation_props_f64": [_vp, _vp, _i32, _i32],
    "rdb200_dev_fa_d8_f32_f64": [_vp, _vp, _i32, _i32, _f32, _i32],
    "rdb200_dev_fa_tarboton_f32_f64": [_vp, _vp, _i32, _i32, _f32, _i32],
    "rdb200_fill_depressions_d8_f64": [_vp, _i32, _i32],
    "rdb200_fill_depressions_d4_f64": [_vp, _i32, _i32],
    "rdb200_pit_mask_d8_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_pit_mask_d4_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_has_depressions_d8_f64": [_vp, _i32, _i32, C.POINTER(_i32)],
    "rdb200_has_depressions_d4_f64": [_vp, _i32, _i32, C.POINTER(_i32)],
    "rdb200_resolve_flats_epsilon_f64": [_vp, _i32, _i32, _f64],
    "rdb200_d8_flow_directions_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_get_flat_mask_f64": [_vp, _vp, _vp, _i32, _i32, _f64],
    "rdb200_d8_flow_directions_flats_f64": [_vp, _vp, _i32, _i32, _f64, _i32],
    "rdb200_dev_d8_flow_directions_flats_f64": [_vp, _vp, _i32, _i32, _f64, _i32],
    "rdb200_fa_d8_f64_f64": [_vp, _vp, _i32, _i32, _f64, _i32],
    "rdb200_fa_d4_f64_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_f64_order_keys": [_vp, _vp, _i32, _i32, _f64, C.POINTER(_f32), C.POINTER(_i32)],
    "rdb200_dev_fill_depressions_d8_f64": [_vp, _i32, _i32],
    "rdb200_dev_fill_depressions_d4_f64": [_vp, _i32, _i32],
    "rdb200_dev_pit_mask_d8_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_dev_pit_mask_d4_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_dev_has_depressions_d8_f64": [_vp, _i32, _i32, C.POINTER(_i32)],
    "rdb200_dev_has_depressions_d4_f64": [_vp, _i32, _i32, C.POINTER(_i32)],
    "rdb200_dev_resolve_flats_epsilon_f64": [_vp, _i32, _i32, _f64],
    "rdb200_dev_d8_flow_directions_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_dev_fa_d8_f64_f64": [_vp, _vp, _i32, _i32, _f64, _i32],
    "rdb200_dev_fa_d4_f64_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_dev_f64_order_keys": [_vp, _vp, _i32, _i32, _f64, C.POINTER(_f32), C.POINTER(_i32)],
    "rdb200_fm_d8_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_fm_tarboton_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_fm_d4_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_fm_quinn_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_fm_holmgren_f64": [_vp, _vp, _i32, _i32, _f64, _f64],
    "rdb200_fm_freeman_f64": [_vp, _vp, _i32, _i32, _f64, _f64],
    "rdb200_fa_tarboton_f64_f64": [_vp, _vp, _i32, _i32, _f64, _i32],
    "rdb200_fa_quinn_f64_f64": [_vp, _vp, _i32, _i32, _f64],
    "rdb200_fa_holmgren_f64_f64": [_vp, _vp, _i32, _i32, _f64, _f64],
    "rdb200_fa_freeman_f64_f64": [_vp, _vp, _i32, _i32, _f64, _f64],
    "rdb200_terrain_attribute_f64": [_i32, _vp, _vp, _i32, _i32, _f64, _f32, _f32, _f64, _f64],
    "rdb200_dev_fm_method_f64": [_i32, _vp, _vp, _i32, _i32, _f64, _f64],
    "rdb200_dev_fa_method_f64_f64": [_i32, _vp, _vp, _i32, _i32, _f64, _f64],
    "rdb200_dev_fa_tarboton_f64_f64": [_vp, _vp, _i32, _i32, _f64, _i32],
    "rdb200_dev_terrain_attribute_f64": [_i32, _vp, _vp, _i32, _i32, _f64, _f32, _f32, _f64, _f64],
    "rdb200_dev_generate_fbm_f32": [_vp, _i32, _i32, _i32, C.c_uint32, _i32, _f32],
    "rdb200_nccl_unique_id": [_vp],
    "rdb200_comm_create_nccl": [C.POINTER(_vp), _i32, _i32, _vp],
    "rdb200_comm_create_callbacks": [C.POINTER(_vp), _i32, _i32, _vp, _vp, _vp],
    "rdb200_comm_destroy": [_vp],
    "rdb200_mgpu_fill_depressions_d8_f32": [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_fill_depressions_d4_f32": [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_fa_f32_f64": [_vp, _vp, _vp, _i32, _i32, _f32, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_fa_method_f32_f64": [_vp, _vp, _vp, _i32, _i32, _f32, _i32, _i32, _i32, C.c_double, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_resolve_flats_epsilon_f32": [_vp, _vp, _i32, _i32, _f32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_d8_flow_directions_flats_f32": [_vp, _vp, _vp, _i32, _i32, _f32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_d8_flow_accum_u8_i32": [_vp, _vp, _vp, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_fm_method_f32": [_vp, _i32, _vp, _vp, _i32, _i32, _f32, _i32, _i32, C.c_double],
    "rdb200_mgpu_terrain_attribute_f32": [_vp, _i32, _vp, _vp, _i32, _i32, _f32, _f32, _f32, C.c_double, C.c_double, _i32, _i32],
    "rdb200_mgpu_flow_accumulation_props_f64": [_vp, _vp, _vp, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_fill_depressions_d8_f64": [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_fill_depressions_d4_f64": [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_pit_mask_d8_f64": [_vp, _vp, _vp, _i32, _i32, _f64, _i32, _i32, _i32, _i32],
    "rdb200_mgpu_pit_mask_d4_f64": [_vp, _vp, _vp, _i32, _i32, _f64, _i32, _i32, _i32, _i32],
    "rdb200_mgpu_has_depressions_d8_f64": [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_has_depressions_d4_f64": [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_resolve_flats_epsilon_f64": [_vp, _vp, _i32, _i32, _f64, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_d8_flow_directions_flats_f64": [_vp, _vp, _vp, _i32, _i32, _f64, _i32, _i32, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_fm_method_f64": [_vp, _i32, _vp, _vp, _i32, _i32, _f64, _i32, _i32, _f64],
    "rdb200_mgpu_terrain_attribute_f64": [_vp, _i32, _vp, _vp, _i32, _i32, _f64, _f32, _f32, _f64, _f64, _i32, _i32],
    "rdb200_mgpu_fa_method_f64_f64": [_vp, _vp, _vp, _i32, _i32, _f64, _i32, _i32, _i32, _f64, _i32, C.POINTER(_i32)],
    "rdb200_mgpu_f64_order_keys": [_vp, _vp, _vp, _i32, _i32, _f64, _i32, _i32, C.POINTER(_f32), C.POINTER(_i32)],
    "rdb200_dev_fill_begin": [C.POINTER(_vp), _vp, _i32, _i32],
    "rdb200_dev_fill_begin_lifted": [C.POINTER(_vp), _vp, _i32, _i32, _vp, _i32, _i32, _i32],
    "rdb200_dev_maxpool_rows_f32": [_vp, _i32, _i32, _i32, _i32, _vp, _i32, _i32],
    "rdb200_dev_fill_blockmax": [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32],
    "rdb200_dev_fill_relax_from_f32": [_vp, _vp, _i32, _i32],
    "rdb200_dev_fill_prolong": [_vp, _vp, _i32, _i32, _i32, C.POINTER(C.c_int32)],
    "rdb200_dev_fill_run": [_vp, C.POINTER(_i32)],
    "rdb200_dev_fill_read_row": [_vp, _i32, _vp],
    "rdb200_dev_fill_update_row": [_vp, _i32, _vp],
    "rdb200_dev_fill_finish": [_vp, _vp],
    "rdb200_dev_facc_begin": [C.POINTER(_vp), _vp, _vp, _i32, _i32, _f32, _i32, _i32, _i32, _i32],
    "rdb200_dev_facc_begin_method": [C.POINTER(_vp), _vp, _vp, _i32, _i32, _f32, _i32, _i32, _i32, C.c_double, _i32],
    "rdb200_dev_facc_get_edge_codes": [_vp, _i32, _vp, _vp],
    "rdb200_dev_facc_set_ghost_codes": [_vp, _i32, _vp, _vp],
    "rdb200_dev_facc_run": [_vp, C.POINTER(_i32), C.POINTER(_i32)],
    "rdb200_dev_facc_take_outflow": [_vp, _i32, _vp, _vp],
    "rdb200_dev_facc_apply_inflow": [_vp, _i32, _vp, _vp],
    "rdb200_dev_facc_finish": [_vp],
    "rdb200_dev_flats_begin": [C.POINTER(_vp), _vp, _i32, _i32, _f32, _i32, _i32],
    "rdb200_dev_flats_arrays": [_vp, C.POINTER(C.c_uint64)],
    "rdb200_dev_flats_edges": [_vp],
    "rdb200_dev_flats_components": [_vp],
    "rdb200_dev_flats_labels": [_vp],
    "rdb200_dev_flats_gradient_begin": [_vp, _i32, C.POINTER(_vp)],
    "rdb200_dev_flats_gradient_end": [_vp, _i32, _vp],
    "rdb200_dev_flats_apply": [_vp],
    "rdb200_dev_flats_finish": [_vp],
}
OTHER_SYMBOLS = ["rdb200_shutdown", "rdb200_last_error", "rdb200_version"]


def lib():
    """Load (once) and return the shared library; raises loudly when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RichdemB200Error(
                f"{LIB_PATH} not found: build it with `python -m richdem_b200.build` "
                "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        if hasattr(L, "rdb200_emulated"):
            # tests/emu builds the kernel sources for a CPU fiber model to check their logic; it is
            # test infrastructure, never a compute path
            raise RichdemB200Error(
                f"{LIB_PATH} is the CPU kernel-emulation test build, not librichdem_b200 "
                "(there is no CPU fallback)")
        for name, argtypes in SIGNATURES.items():
            f = getattr(L, name)
            f.argtypes = argtypes
            f.restype = C.c_int
        L.rdb200_last_error.restype = C.c_char_p
        L.rdb200_last_error.argtypes = []
        L.rdb200_version.restype = C.c_int
        L.rdb200_shutdown.restype = None
        _lib = L
        # experiment hook: RDB200_PARAMS="fill_multigrid=8,accum_fused_prep=1" presets rdb200_set_param switches for
        # this process (tools, bench.py and the GPU tests can then run unchanged under candidate defaults)
        for kv in filter(None, os.environ.get("RDB200_PARAMS", "").split(",")):
            k, _, v = kv.partition("=")
            if L.rdb200_set_param(k.strip().encode(), int(v)):
                msg = L.rdb200_last_error()
                raise RichdemB200Error(f"RDB200_PARAMS: {msg.decode('utf-8', 'replace') if msg else kv}")
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        msg = lib().rdb200_last_error()
        raise RichdemB200Error(msg.decode("utf-8", "replace") if msg else f"librichdem_b200 error {rc}")


def ptr(a: np.ndarray) -> int:
    return a.ctypes.data


def stats() -> dict:
    s = Stats()
    check(lib().rdb200_get_stats(C.byref(s)))
    return s.as_dict()


_param_values: dict = {}  # what this process set through set_param (the C ABI has no getter)


def set_param(name: str, value: int) -> None:
    check(lib().rdb200_set_param(name.encode(), int(value)))
    if name == "reset_defaults":
        _param_values.clear()
    elif name != "trim_workspace":
        _param_values[name] = int(value)


def reset_params() -> None:
    """Every rdb200_set_param switch back to its shipped default."""
    set_param("reset_defaults", 1)


class scoped_param:
    """`with scoped_param("fill_band_rounds", 64): ...` -- a switch for the duration of a block, then back to what this
    process had set before (or to `default`, the library's own default, if it never set it)."""

    def __init__(self, name: str, value: int, default: int = 0):
        self.name, self.value, self.default = name, int(value), int(default)

    def __enter__(self):
        self.previous = _param_values.get(self.name)
        set_param(self.name, self.value)
        return self

    def __exit__(self, *exc):
        if self.previous is None:
            set_param(self.name, self.default)
            _param_values.pop(self.name, None)
        else:
            set_param(self.name, self.previous)
        return False


def init(device: int = 0) -> None:
    check(lib().rdb200_init(int(device)))


def set_stream(cuda_stream) -> None:
    """Run subsequent work on `cuda_stream` (int handle, e.g. torch.cuda.current_stream().cuda_stream).
    None restores the library's own stream; 0 (torch's default stream) selects CUDA's legacy default
    stream explicitly (cudaStreamLegacy)."""
    if cuda_stream is None:
        check(lib().rdb200_set_stream(C.c_void_p(None)))
    else:
        h = int(cuda_stream)
        check(lib().rdb200_set_stream(C.c_void_p(h if h != 0 else 1)))


def use_torch_stream() -> None:
    """Order the library's work with torch's: run on torch's current CUDA stream."""
    import torch
    set_stream(torch.cuda.current_stream().cuda_stream)


def shutdown() -> None:
    lib().rdb200_shutdown()
