"""TEST INFRASTRUCTURE ONLY -- the float64 path's spec and its reference.

* :func:`kappa` -- a numpy restatement of the order-preserving float keys (richdem_b200/csrc/f64.cu), the spec the
  kernels are tested against; :func:`kappa_inv_fill` and :func:`advance_ulps` restate the fill's write-back and the
  flats' double apply.
* :func:`ref` -- ``oracle/_ref/libref_f64.so``: the UNMODIFIED reference templates with T = double and T = float
  (oracle/f64_shim.cpp), only where the reference tree exists.

``topology`` is ``"D8"`` or ``"D4"``.  Only tests and tools import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import _HERE

REF = "/root/reference"
_REF_PATH = os.path.join(_HERE, "_ref", "libref_f64.so")
FLT_MAX = float(np.finfo(np.float32).max)
DBL_MAX = float(np.finfo(np.float64).max)
RANK_BASE = 0x00800000
_NAN32 = np.uint32(0x7FC00000).view(np.float32)


def build(force: bool = False) -> None:
    shim = os.path.join(_HERE, "f64_shim.cpp")
    stale = not os.path.exists(_REF_PATH) or os.path.getmtime(_REF_PATH) < os.path.getmtime(shim)
    if os.path.isdir(os.path.join(REF, "include", "richdem")) and (force or stale):
        os.makedirs(os.path.dirname(_REF_PATH), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-DNDEBUG", "-DRICHDEM_NO_PROGRESS", "-fPIC", "-shared",
                               "-I" + os.path.join(REF, "include"), shim, "-o", _REF_PATH])


def have_ref() -> bool:
    return os.path.exists(_REF_PATH)


# ---- the spec -------------------------------------------------------------------------------------------------------
def is_float_raster(z) -> bool:
    """Case 1: every value is NaN, +-inf, or a float-exact double strictly inside (-FLT_MAX, FLT_MAX)."""
    z = np.asarray(z, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = z.astype(np.float32)
        ok = np.isnan(z) | np.isinf(z) | ((f.astype(np.float64) == z) & (np.abs(z) < FLT_MAX))
    return bool(ok.all())


def _image(v: float):
    if np.isnan(v):
        return _NAN32
    if v == np.inf or v == -np.inf:
        return np.float32(v)
    if v == DBL_MAX:
        return np.float32(FLT_MAX)
    if v == -DBL_MAX:
        return np.float32(-FLT_MAX)
    return None


def order_keys(z) -> np.ndarray:
    """The monotone uint64 image of each double (-0.0 just below +0.0)."""
    b = np.ascontiguousarray(z, np.float64).view(np.uint64)
    neg = (b >> np.uint64(63)) != 0
    return np.where(neg, ~b, b | np.uint64(1 << 63))


def kappa(z, nodata: float):
    """(keys float32, kappa(nodata) float32, ranked) as the kernels define them."""
    z = np.ascontiguousarray(z, np.float64)
    if is_float_raster(z):
        keys, ranked = z.astype(np.float32), False
    else:
        flat = z.ravel()
        idx = np.argsort(order_keys(flat), kind="stable")
        sv = flat[idx]
        head = np.ones(sv.size, bool)
        head[1:] = ~(sv[1:] == sv[:-1])  # +-0 share a run, every NaN starts its own
        rank = np.cumsum(head) - 1
        ks = (RANK_BASE + rank).astype(np.uint32).view(np.float32)
        for v, img in ((np.inf, np.float32(np.inf)), (-np.inf, np.float32(-np.inf)), (DBL_MAX, np.float32(FLT_MAX)),
                       (-DBL_MAX, np.float32(-FLT_MAX))):
            ks[sv == v] = img
        ks[np.isnan(sv)] = _NAN32
        keys = np.empty(flat.size, np.float32)
        keys[idx] = ks
        keys, ranked = keys.reshape(z.shape), True
    eq = np.flatnonzero(z.ravel() == nodata)
    if eq.size:
        ndk = keys.ravel()[eq[0]]
    else:
        img = _image(float(nodata))
        ndk = img if img is not None else _NAN32
    return keys, np.float32(ndk), ranked


def kappa_inv_fill(z, keys0, keysf) -> np.ndarray:
    """The fill's write-back: cells whose key changed take the double whose key it is; the others keep their bits."""
    z = np.array(z, np.float64)
    k0 = np.ascontiguousarray(keys0, np.float32).ravel().view(np.uint32)
    kf = np.ascontiguousarray(keysf, np.float32).ravel().view(np.uint32)
    out = z.ravel()
    raised = np.flatnonzero(k0 != kf)
    if raised.size:
        uniq, first = np.unique(k0, return_index=True)  # the fill only copies keys the raster holds
        pos = np.minimum(np.searchsorted(uniq, kf[raised]), uniq.size - 1)
        vals = out[first[pos]]
        vals[np.isnan(kf[raised].view(np.float32))] = np.nan
        out[raised] = vals
    return out.reshape(z.shape)


def advance_ulps(z, k) -> np.ndarray:
    """k successive nextafter(z, +inf), elementwise (k <= 0: z itself)."""
    out = np.array(z, np.float64)
    k = np.asarray(k)
    sel = k > 0
    v, kk = out[sel], k[sel]
    with np.errstate(over="ignore"):  # DBL_MAX -> inf is what nextafter does
        for s in range(int(kk.max()) if kk.size else 0):
            m = kk > s
            v[m] = np.nextafter(v[m], np.inf)
    out[sel] = v
    return out


def apply_flat_mask(z, mask) -> np.ndarray:
    """ResolveFlatsEpsilon's apply (flats/Barnes2014.hpp:496-550): interior cells only."""
    m = np.array(mask, copy=True)
    m[0, :] = m[-1, :] = 0
    m[:, 0] = m[:, -1] = 0
    return advance_ulps(z, m)


# ---- inputs ---------------------------------------------------------------------------------------------------------
def nested_lakes() -> np.ndarray:
    """Two lakes whose spill levels are one double ulp apart, the inner one nested in a wider basin: rounded to float,
    both levels become 5.0 and the lakes merge."""
    z = np.full((11, 15), 10.0)
    z[1:-1, 1:-1] = 7.0
    z[2:9, 2:6] = 1.0                      # lake A
    z[2:9, 8:13] = 2.0                     # lake B, with a nested pit
    z[5, 10] = 0.5
    z[5, 6:8] = 5.0                        # the sill between them
    z[5, 0] = 5.0                          # A's outlet to the edge ...
    z[5, 1] = 5.0
    z[4, 1] = 5.0
    z[8, 14] = np.nextafter(5.0, np.inf)   # ... and B's, one ulp higher
    z[8, 13] = np.nextafter(5.0, np.inf)
    z[5, 6] = np.nextafter(np.nextafter(5.0, np.inf), np.inf)
    z[5, 7] = np.nextafter(np.nextafter(5.0, np.inf), np.inf)
    return z


def cases(seed: int = 0):
    """(name, Z float64, nodata) triples covering the float64 path's ground."""
    from . import fbm_terrain
    rng = np.random.default_rng(seed)
    out = []
    fbm = fbm_terrain(48, 64, seed=3, quantum=0.5).astype(np.float64)
    out.append(("fbm_subfloat", fbm + rng.integers(0, 4, fbm.shape) * 2.0 ** -40, -9999.0))
    g = np.load(os.path.join(_HERE, "..", "tests", "golden", "beauford_crop.npz"))
    b = g["dem"][:96, :128].astype(np.float64)
    nd = float(g["nodata"])
    b = np.where(b == nd, nd, b + rng.random(b.shape) * 1e-9)
    out.append(("beauford_1e-9", b, nd))
    out.append(("nested_lakes", nested_lakes(), -9999.0))
    sp = fbm_terrain(24, 30, seed=5, quantum=1.0).astype(np.float64)
    sp[3:7, 4:9] = DBL_MAX
    sp[10, 3:6] = [FLT_MAX, -FLT_MAX, np.inf]
    sp[12, 10:14] = [-np.inf, 0.0, -0.0, 5e-324]
    sp[14, 4:8] = [1e300, -1e300, -5e-324, 2.2e-308]
    sp[15:18, 15:18] = -0.0
    sp[16, 16] = 0.0
    sp[0, 0] = -DBL_MAX
    out.append(("sentinels", sp, -9999.0))
    out.append(("sentinels_nodata_inf", np.where(sp == np.inf, -np.inf, sp), -np.inf))
    out.append(("sentinels_nodata_dblmax", sp, DBL_MAX))
    nodata_present = fbm.copy()
    nodata_present[10:20, 5:12] = -9999.0
    nodata_present[0, 3] = -9999.0
    out.append(("nodata_present", nodata_present + 2.0 ** -30, -9999.0 + 2.0 ** -30))
    out.append(("nodata_absent", fbm + 2.0 ** -30, 12345.678))
    out.append(("float_raster", fbm, -9999.0))
    out.append(("row_1xN", (rng.random((1, 37)) * 10).round(1), -9999.0))
    out.append(("col_Nx1", (rng.random((29, 1)) * 10).round(1), -9999.0))
    out.append(("square_2x2", np.array([[1.0, np.nextafter(1.0, 2.0)], [0.5, -0.0]]), -9999.0))
    return out


# ---- the reference ------------------------------------------------------------------------------------------------
def _topo(topology: str) -> int:
    if topology not in ("D8", "D4"):
        raise ValueError(f"unknown topology {topology!r}")
    return int(topology == "D4")


class _Ref:
    def __init__(self, path: str):
        L = C.CDLL(path)
        self.lib = L
        for s, T, ct in (("f64", np.float64, C.c_double), ("f32", np.float32, C.c_float)):
            p = np.ctypeslib.ndpointer(T, flags="C_CONTIGUOUS")
            u8 = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
            i32 = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
            f64 = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
            sigs = {"fill": ([C.c_int, p, C.c_int, C.c_int], None),
                    "pit_mask": ([C.c_int, p, C.c_int, C.c_int, ct, u8], None),
                    "has_depressions": ([C.c_int, p, C.c_int, C.c_int], C.c_int),
                    "resolve_flats": ([p, C.c_int, C.c_int, ct], None),
                    "flat_mask": ([p, C.c_int, C.c_int, ct, i32], None),
                    "d8_flow_directions": ([p, C.c_int, C.c_int, ct, u8], None),
                    "fa": ([C.c_int, p, C.c_int, C.c_int, ct, f64], None)}
            for name, (args, res) in sigs.items():
                f = getattr(L, f"ref_{name}_{s}")
                f.argtypes, f.restype = args, res

    @staticmethod
    def _arr(dem):
        a = np.array(dem, copy=True, order="C")
        assert a.ndim == 2 and a.dtype in (np.float32, np.float64)
        return a, "f64" if a.dtype == np.float64 else "f32"

    def _f(self, name, s):
        return getattr(self.lib, f"ref_{name}_{s}")

    def fill(self, dem, topology="D8"):
        a, s = self._arr(dem)
        self._f("fill", s)(_topo(topology), a, a.shape[1], a.shape[0])
        return a

    def pit_mask(self, dem, nodata, topology="D8"):
        a, s = self._arr(dem)
        out = np.empty(a.shape, np.uint8)
        self._f("pit_mask", s)(_topo(topology), a, a.shape[1], a.shape[0], nodata, out)
        return out

    def has_depressions(self, dem, topology="D8"):
        a, s = self._arr(dem)
        return bool(self._f("has_depressions", s)(_topo(topology), a, a.shape[1], a.shape[0]))

    def resolve_flats(self, dem, nodata):
        a, s = self._arr(dem)
        self._f("resolve_flats", s)(a, a.shape[1], a.shape[0], nodata)
        return a

    def flat_mask(self, dem, nodata):
        a, s = self._arr(dem)
        out = np.zeros(a.shape, np.int32)
        self._f("flat_mask", s)(a, a.shape[1], a.shape[0], nodata, out)
        return out

    def d8_flow_directions(self, dem, nodata):
        a, s = self._arr(dem)
        out = np.empty(a.shape, np.uint8)
        self._f("d8_flow_directions", s)(a, a.shape[1], a.shape[0], nodata, out)
        return out

    def fa(self, dem, nodata, topology="D8", weights=None):
        a, s = self._arr(dem)
        acc = np.ones(a.shape, np.float64) if weights is None else np.array(weights, np.float64, order="C")
        self._f("fa", s)(_topo(topology), a, a.shape[1], a.shape[0], nodata, acc)
        return acc


_ref = None


def ref() -> _Ref:
    """The reference templates (raises where oracle/_ref was never built)."""
    global _ref
    if _ref is None:
        if not have_ref():
            build()
        if not have_ref():
            raise RuntimeError("oracle/_ref/libref_f64.so absent (reference tree not available)")
        _ref = _Ref(_REF_PATH)
    return _ref
