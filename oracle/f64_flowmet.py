"""TEST INFRASTRUCTURE ONLY -- the reference of the float64 flow metrics, accumulations and terrain attributes.

:func:`ref` loads ``oracle/_ref/libref_f64_flowmet.so``: the UNMODIFIED reference FM_*, FA_* and TA_* templates with
E / T = double and = float (oracle/f64_flowmet_shim.cpp), only where the reference tree exists.  The dtype of the DEM
picks the instantiation.  Methods are numbered as in the C ABI (0 D8, 1 Tarboton, 2 D4, 3 Holmgren / Quinn at exponent
1, 4 Freeman), attributes as RDB200_TA_*.  Only tests and tools import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import _HERE
from .f64 import REF

_REF_PATH = os.path.join(_HERE, "_ref", "libref_f64_flowmet.so")


def build(force: bool = False) -> None:
    shim = os.path.join(_HERE, "f64_flowmet_shim.cpp")
    stale = not os.path.exists(_REF_PATH) or os.path.getmtime(_REF_PATH) < os.path.getmtime(shim)
    if os.path.isdir(os.path.join(REF, "include", "richdem")) and (force or stale):
        os.makedirs(os.path.dirname(_REF_PATH), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-DNDEBUG", "-DRICHDEM_NO_PROGRESS", "-fPIC", "-shared",
                               "-I" + os.path.join(REF, "include"), shim, "-o", _REF_PATH])


def have_ref() -> bool:
    return os.path.exists(_REF_PATH)


class _Ref:
    def __init__(self, path: str):
        L = C.CDLL(path)
        self.lib = L
        f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
        f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
        for s, T, ct in (("f64", np.float64, C.c_double), ("f32", np.float32, C.c_float)):
            p = np.ctypeslib.ndpointer(T, flags="C_CONTIGUOUS")
            sigs = {"fm": [C.c_int, p, C.c_int, C.c_int, ct, C.c_double, f32p],
                    "fa": [C.c_int, p, C.c_int, C.c_int, ct, C.c_double, f64p],
                    "ta": [C.c_int, p, C.c_int, C.c_int, ct, C.c_float, C.c_float, C.c_double, C.c_double, f32p]}
            for name, args in sigs.items():
                f = getattr(L, f"ref_{name}_{s}")
                f.argtypes, f.restype = args, None

    def _call(self, name, dem):
        a = np.array(dem, copy=True, order="C")
        assert a.ndim == 2 and a.dtype in (np.float32, np.float64)
        return a, getattr(self.lib, f"ref_{name}_{'f64' if a.dtype == np.float64 else 'f32'}")

    def fm(self, dem, nodata, method, exponent=1.0):
        """FM_x -> (H, W, 9) float32."""
        a, f = self._call("fm", dem)
        props = np.empty(a.shape + (9,), np.float32)
        f(method, a, a.shape[1], a.shape[0], nodata, float(exponent), props)
        return props

    def fa(self, dem, nodata, method, exponent=1.0, weights=None):
        """FA_x with the caller's weights (unit weights when None)."""
        a, f = self._call("fa", dem)
        acc = np.ones(a.shape, np.float64) if weights is None else np.array(weights, np.float64, order="C")
        f(method, a, a.shape[1], a.shape[0], nodata, float(exponent), acc)
        return acc

    def ta(self, dem, attrib, nodata, zscale=1.0, cell=(1.0, 1.0), nodata_out=-9999.0):
        """TA_x -> float32."""
        a, f = self._call("ta", dem)
        out = np.empty(a.shape, np.float32)
        f(attrib, a, a.shape[1], a.shape[0], nodata, nodata_out, zscale, cell[0], cell[1], out)
        return out


_ref = None


def ref() -> _Ref:
    """The reference templates (raises where oracle/_ref was never built)."""
    global _ref
    if _ref is None:
        if not have_ref():
            build()
        if not have_ref():
            raise RuntimeError("oracle/_ref/libref_f64_flowmet.so absent (reference tree not available)")
        _ref = _Ref(_REF_PATH)
    return _ref
