"""TEST INFRASTRUCTURE ONLY -- the reference of the direction-grid pipeline for float64 (and float32) DEMs.

:func:`ref` loads ``oracle/_ref/libref_f64_flowdirs.so``: the UNMODIFIED reference barnes_flat_resolution_d8 (both
``alter`` modes), GetFlatMask and d8_flow_accum (oracle/f64_flowdirs_shim.cpp), only where the reference tree exists.
The dtype of the DEM picks the instantiation.  :func:`float_steps` restates the float steps with which the reference
alters a double (flats/flat_resolution.hpp:565-568: ``nextafterf``).  Only tests and tools import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import _HERE
from .f64 import REF

_REF_PATH = os.path.join(_HERE, "_ref", "libref_f64_flowdirs.so")


def build(force: bool = False) -> None:
    shim = os.path.join(_HERE, "f64_flowdirs_shim.cpp")
    stale = not os.path.exists(_REF_PATH) or os.path.getmtime(_REF_PATH) < os.path.getmtime(shim)
    if os.path.isdir(os.path.join(REF, "include", "richdem")) and (force or stale):
        os.makedirs(os.path.dirname(_REF_PATH), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-DNDEBUG", "-DRICHDEM_NO_PROGRESS", "-fPIC", "-shared",
                               "-I" + os.path.join(REF, "include"), shim, "-o", _REF_PATH])


def have_ref() -> bool:
    return os.path.exists(_REF_PATH)


def float_steps(z, m) -> np.ndarray:
    """m successive nextafterf(z, +inf) of each double z, starting from z rounded to float32; m <= 0 keeps z."""
    z = np.array(z, np.float64)
    m = np.broadcast_to(np.asarray(m, np.int64), z.shape)
    out = z.copy()
    inf32 = np.float32(np.inf)
    with np.errstate(over="ignore"):
        for idx in zip(*np.nonzero(m > 0)):
            f = np.float32(z[idx])
            for _ in range(int(m[idx])):
                f = np.nextafter(f, inf32)
            out[idx] = np.float64(f)
    return out


class _Ref:
    def __init__(self, path: str):
        L = C.CDLL(path)
        self.lib = L
        u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
        i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
        for s, T, ct in (("f64", np.float64, C.c_double), ("f32", np.float32, C.c_float)):
            p = np.ctypeslib.ndpointer(T, flags="C_CONTIGUOUS")
            f = getattr(L, f"ref_flowdirs_flats_{s}")
            f.argtypes, f.restype = [p, C.c_int, C.c_int, ct, C.c_int, u8p], None
            f = getattr(L, f"ref_flat_mask_{s}")
            f.argtypes, f.restype = [p, C.c_int, C.c_int, ct, i32p, i32p], None
        L.ref_d8_flow_accum.argtypes, L.ref_d8_flow_accum.restype = [u8p, C.c_int, C.c_int, i32p], None

    @staticmethod
    def _sfx(a):
        assert a.ndim == 2 and a.dtype in (np.float32, np.float64)
        return "f64" if a.dtype == np.float64 else "f32"

    def flowdirs_flats(self, dem, nodata, alter=False):
        """barnes_flat_resolution_d8 -> (uint8 directions, the DEM after the call: altered when ``alter``)."""
        a = np.array(dem, copy=True, order="C")
        out = np.empty(a.shape, np.uint8)
        getattr(self.lib, f"ref_flowdirs_flats_{self._sfx(a)}")(a, a.shape[1], a.shape[0], nodata, int(bool(alter)), out)
        return out, a

    def flat_mask(self, dem, nodata):
        """GetFlatMask -> (int32 mask, int32 labels)."""
        a = np.ascontiguousarray(dem)
        m = np.empty(a.shape, np.int32)
        lab = np.empty(a.shape, np.int32)
        getattr(self.lib, f"ref_flat_mask_{self._sfx(a)}")(a, a.shape[1], a.shape[0], nodata, m, lab)
        return m, lab

    def d8_flow_accum(self, dirs):
        d = np.ascontiguousarray(dirs, np.uint8)
        area = np.empty(d.shape, np.int32)
        self.lib.ref_d8_flow_accum(d, d.shape[1], d.shape[0], area)
        return area


_REF = None


def ref() -> _Ref:
    global _REF
    if _REF is None:
        _REF = _Ref(_REF_PATH)
    return _REF
