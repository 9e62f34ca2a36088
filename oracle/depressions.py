"""TEST INFRASTRUCTURE ONLY -- CPU oracles of pit_mask<topo> and HasDepressions<topo> (reference
include/richdem/depressions/Barnes2014.hpp:593-676, :43-104), with the two back ends of :mod:`oracle`:

* ``port`` -- ``oracle/libdepressions_oracle.so``: the C restatement in ``oracle/depressions.c`` (the fill of
  ``oracle/oracle.c`` and one compare; always buildable).
* ``ref``  -- ``oracle/_ref/libref_depressions.so``: the UNMODIFIED reference templates compiled from
  ``oracle/depressions_shim.cpp`` (only where the reference tree exists).

``topology`` is ``"D8"`` or ``"D4"``.  Only tests and tools import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import _HERE
from . import build as _build_oracle

REF = "/root/reference"
_PORT_PATH = os.path.join(_HERE, "libdepressions_oracle.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libref_depressions.so")
_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")


def _stale(out: str, src: str) -> bool:
    return not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(src)


def build(force: bool = False) -> None:
    """Compile the C restatement (and the reference shim when the reference tree exists)."""
    _build_oracle()  # liboracle.so: the fill the restatement links against
    src = os.path.join(_HERE, "depressions.c")
    if force or _stale(_PORT_PATH, src) or _stale(_PORT_PATH, os.path.join(_HERE, "liboracle.so")):
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", _PORT_PATH, src,
                               "-L" + _HERE, "-l:liboracle.so", "-Wl,-rpath,$ORIGIN"])
    shim = os.path.join(_HERE, "depressions_shim.cpp")
    if os.path.isdir(os.path.join(REF, "include", "richdem")) and (force or _stale(_REF_PATH, shim)):
        os.makedirs(os.path.dirname(_REF_PATH), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O3", "-DNDEBUG", "-DRICHDEM_NO_PROGRESS", "-fPIC", "-shared",
                               "-I" + os.path.join(REF, "include"), shim, "-o", _REF_PATH], stderr=subprocess.DEVNULL)


def have_ref() -> bool:
    return os.path.exists(_REF_PATH)


def _topo(topology: str) -> int:
    if topology not in ("D8", "D4"):
        raise ValueError(f"unknown topology {topology!r}")
    return int(topology == "D4")


def _dem(dem) -> np.ndarray:
    a = np.array(dem, dtype=np.float32, order="C", copy=True)  # (the reference wraps the buffer unowned and non-const)
    assert a.ndim == 2
    return a


class _Backend:
    def __init__(self, path: str, kind: str):
        self.kind = kind
        self.lib = C.CDLL(path)
        prefix = "ref" if kind == "reference" else "orc"
        self._mask = getattr(self.lib, f"{prefix}_pit_mask_f32")
        self._has = getattr(self.lib, f"{prefix}_has_depressions_f32")
        self._mask.argtypes = [C.c_int, _f32p, C.c_int, C.c_int, C.c_float, _u8p]
        self._mask.restype = None if kind == "reference" else C.c_int
        self._has.argtypes = [C.c_int, _f32p, C.c_int, C.c_int]
        self._has.restype = C.c_int

    def pit_mask(self, dem, nodata: float, topology: str = "D8") -> np.ndarray:
        """uint8 mask: 3 NoData, 1 below the filled surface, 0 elsewhere (NoData value 3)."""
        d = _dem(dem)
        h, w = d.shape
        out = np.empty((h, w), np.uint8)
        self._mask(_topo(topology), d, w, h, float(nodata), out)
        return out

    def has_depressions(self, dem, topology: str = "D8") -> bool:
        d = _dem(dem)
        h, w = d.shape
        return bool(self._has(_topo(topology), d, w, h))


_port = None
_ref = None


def port() -> _Backend:
    """The C restatement (depressions.c)."""
    global _port
    if _port is None:
        build()
        _port = _Backend(_PORT_PATH, "port")
    return _port


def ref() -> _Backend:
    """The unmodified reference templates (raises where oracle/_ref was never built)."""
    global _ref
    if _ref is None:
        if not have_ref():
            build()
        if not have_ref():
            raise RuntimeError("oracle/_ref/libref_depressions.so absent (reference tree not available)")
        _ref = _Backend(_REF_PATH, "reference")
    return _ref


def best() -> _Backend:
    """Reference when it was built here, else the port."""
    return ref() if have_ref() else port()
