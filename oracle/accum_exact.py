"""TEST INFRASTRUCTURE ONLY -- flow accumulation from given proportions in extended precision, with the per-cell error
budget of the library's double engines and of its packed fixed-point D-infinity walk (``oracle/accum_exact.c``, a plain
C statement of flow_accumulation_generic's recursion; see there for the bounds).  Only tests and tools import this
module."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import _HERE

_SRC = os.path.join(_HERE, "accum_exact.c")
_PATH = os.path.join(_HERE, "libaccum_exact.so")
_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_lib = None


def build(force: bool = False) -> None:
    if force or not os.path.exists(_PATH) or os.path.getmtime(_PATH) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", _PATH, _SRC, "-lm"])


def _load():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_PATH)
        f = L.ae_accumulate
        f.argtypes = [_f32p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, _f64p, _f64p, _f64p, C.c_void_p, C.c_void_p,
                      _i32p]
        f.restype = C.c_int
        _lib = L
    return _lib


@dataclass
class Exact:
    ref: np.ndarray                   # the accumulation in extended precision, rounded to double (-1 at NoData)
    budget: np.ndarray                # the engine's error budget per cell (0 at NoData)
    err: Optional[np.ndarray]         # |got - ref| in extended precision (NoData: 0 if got is -1, else inf)
    shares: np.ndarray                # shares received (mode "double") / rounded shares received (mode "packed")
    packed: Optional[np.ndarray]      # mode "packed": the packed walk's bits, product and half rounded separately ...
    packed_fma: Optional[np.ndarray]  # ... and rounded once (fused multiply-add)

    def excess(self) -> np.ndarray:
        """err / budget (<= 1 passes); cells whose reference is not finite are 0 (checked separately)."""
        with np.errstate(divide="ignore", invalid="ignore"):
            q = np.where(self.err == 0, 0.0, self.err / self.budget)
        return np.where(np.isfinite(self.ref), q, 0.0)


def accumulate(props, weights=None, mode: str = "double", got=None) -> Exact:
    """A(c) = w(c) + sum p(d, c) A(d) over float32 (H, W, 9) proportions; ``weights`` None means ones.  ``mode``:
    "double" (the budget of the double engines) or "packed" (the fixed-point D-infinity walk, unit weights only)."""
    L = _load()
    p = np.ascontiguousarray(props, np.float32)
    h, w = p.shape[0:2]
    assert p.shape == (h, w, 9)
    m = {"double": 0, "packed": 1}[mode]
    assert m == 0 or weights is None
    wt = None if weights is None else np.ascontiguousarray(weights, np.float64)
    g = None if got is None else np.ascontiguousarray(got, np.float64)
    ref, budget, err = (np.empty((h, w), np.float64) for _ in range(3))
    shares = np.zeros((h, w), np.int32)
    pk = np.empty((h, w), np.float64) if m == 1 else None
    pf = np.empty((h, w), np.float64) if m == 1 else None
    left = L.ae_accumulate(p.reshape(-1), None if wt is None else wt.ctypes.data, w, h, m,
                           None if g is None else g.ctypes.data, ref, budget, err,
                           None if pk is None else pk.ctypes.data, None if pf is None else pf.ctypes.data, shares)
    if left != 0:
        raise RuntimeError(f"accum_exact: {left} cells were never completed (a cycle in the proportions?)")
    return Exact(ref, budget, err if g is not None else None, shares, pk, pf)
