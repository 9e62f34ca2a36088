"""TEST INFRASTRUCTURE ONLY -- CPU oracles of FillDepressions(epsilon=True), with the two back ends of :mod:`oracle`:

* ``port`` -- ``oracle/libepsilon_fill_oracle.so``: the C restatement in ``oracle/epsilon_fill.c`` of the surface the GPU
  computes (a Dijkstra flood; always buildable).  The GPU's result equals it bit for bit, the sign of a zero aside.
* ``ref``  -- ``oracle/_ref/libref_epsilon_fill.so``: the UNMODIFIED reference template PriorityFloodEpsilon_Barnes2014
  compiled from ``oracle/epsilon_fill_shim.cpp`` (only where the reference tree exists).  Never below the restatement,
  not equal to it (DESIGN.md section 0, f3).

``topology`` is ``"D8"`` or ``"D4"``.  Only tests and tools import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import _HERE

REF = "/root/reference"
_PORT_PATH = os.path.join(_HERE, "libepsilon_fill_oracle.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libref_epsilon_fill.so")
_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")


def _stale(out: str, src: str) -> bool:
    return not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(src)


def build(force: bool = False) -> None:
    """Compile the C restatement (and the reference shim when the reference tree exists)."""
    src = os.path.join(_HERE, "epsilon_fill.c")
    if force or _stale(_PORT_PATH, src):
        # no -ffast-math / -Ofast: they flush subnormals to zero and would let the compiler reorder the comparisons
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-o", _PORT_PATH,
                               src, "-lm"])
    shim = os.path.join(_HERE, "epsilon_fill_shim.cpp")
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


class _Backend:
    def __init__(self, path: str, kind: str):
        self.kind = kind
        self.lib = C.CDLL(path)
        self._fill = getattr(self.lib, "ref_epsilon_fill_f32" if kind == "reference" else "orc_epsilon_fill_f32")
        self._fill.argtypes = [C.c_int, _f32p, C.c_int, C.c_int, C.c_float]
        self._fill.restype = None if kind == "reference" else C.c_int

    def fill(self, dem, nodata: float, topology: str = "D8") -> np.ndarray:
        """The epsilon-filled copy of ``dem`` (float32); cells equal to ``nodata`` are pinned."""
        d = np.array(dem, dtype=np.float32, order="C", copy=True)
        assert d.ndim == 2
        h, w = d.shape
        rc = self._fill(_topo(topology), d, w, h, float(nodata))
        if rc:
            raise MemoryError("orc_epsilon_fill_f32: out of memory")
        return d


_port = None
_ref = None


def port() -> _Backend:
    """The C restatement (epsilon_fill.c)."""
    global _port
    if _port is None:
        build()
        _port = _Backend(_PORT_PATH, "port")
    return _port


def ref() -> _Backend:
    """The unmodified reference template (raises where oracle/_ref was never built)."""
    global _ref
    if _ref is None:
        if not have_ref():
            build()
        if not have_ref():
            raise RuntimeError("oracle/_ref/libref_epsilon_fill.so absent (reference tree not available)")
        _ref = _Backend(_REF_PATH, "reference")
    return _ref
