"""Writes tests/golden/f64_flowdirs_flats_ref.npz: the reference's barnes_flat_resolution_d8<double, uint8_t> (alter
false and true), GetFlatMask<double> and d8_flow_accum (oracle/f64_flowdirs_shim.cpp) on float64 rasters, the fixtures
of the float64 direction-grid pipeline.

    python tests/golden/make_f64_flowdirs_flats.py   (needs oracle/_ref/libref_f64_flowdirs.so, i.e. the reference tree)

Every raster but the NoData ones is the reference's double fill of a raw raster (stored as <name>/raw), so that it has
long flats.  Inputs:
  fbm_levels        fBm quantised to 16 with levels 20 and 10 float ulps below 1024 and 2048: the float steps cross
                    exponent boundaries (every value a float: the cast route)
  fbm_between       fbm_levels with each level moved by 1/4, 1/2 or 3/4 of its float ulp: the first step rounds down,
                    to even, or up
  fbm_subfloat      fBm with 1e-6 detail, filled: levels that are no float
  above_flt_max     fbm_levels x 1e36: levels below and above FLT_MAX (the float steps give +inf there)
  float_subnormal   fbm_levels centred and x 1e-42, the zero level half -0.0: negative, signed-zero and float-subnormal
                    levels
  double_subnormal  the same x 1e-310: every level rounds to a float zero
  nodata_m32768     fbm_subfloat with NoData patches at -32768
  nodata_1e39       fbm_between with NoData patches at 1e39, a NoData value above FLT_MAX
  beauford          a 120 x 150 crop of beauford_crop.npz (tests/golden), filled, as double
  beauford_1e-9     the same crop with 1e-9 detail, filled
Keys per raster: dem, nodata, dirs0 / dirs1 (alter false / true), dem1 (the altered dem), mask, labels (GetFlatMask)
and area0 (d8_flow_accum of dirs0).
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
OUT = os.path.join(HERE, "f64_flowdirs_flats_ref.npz")
ND = -9999.0


def _float_ulp(v):
    f = np.float32(v)
    return float(np.nextafter(f, np.float32(np.inf))) - float(f)


def _levels():
    import oracle
    q = oracle.fbm_terrain(80, 96, seed=5, amplitude=2000.0, quantum=16.0).astype(np.float64)
    q -= q.min()
    return q + (1024.0 - 20 * 2.0 ** -14) - 16.0 * np.round(q.mean() / 16.0)


def rasters():
    """name -> (raw raster to fill, or None for a raster given as it is, nodata)."""
    import oracle
    rng = np.random.default_rng(23)
    levels = _levels()
    between = levels.copy()
    for k, v in enumerate(np.unique(levels)):
        between[levels == v] = v + (0.25, 0.5, 0.75)[k % 3] * _float_ulp(v)
    sub = oracle.fbm_terrain(80, 96, seed=9, amplitude=500.0, quantum=4.0).astype(np.float64) + rng.random((80, 96)) * 1e-6
    centred = levels - np.median(levels)
    fsub = centred * 1e-42
    fsub[(centred == 0) & (rng.random(centred.shape) < 0.5)] = -0.0
    beau = np.load(os.path.join(HERE, "beauford_crop.npz"))["dem"][100:220, 120:270].astype(np.float64)
    return {
        "fbm_levels": (levels, ND),
        "fbm_between": (between, ND),
        "fbm_subfloat": (sub, ND),
        "above_flt_max": (levels * 1e36, ND),
        "float_subnormal": (fsub, ND),
        "double_subnormal": (centred * 1e-310, ND),
        "beauford": (beau, ND),
        "beauford_1e-9": (beau + rng.random(beau.shape) * 1e-9, ND),
    }


def main() -> None:
    sys.path.insert(0, ROOT)
    from oracle import f64 as F
    from oracle import f64_flowdirs as FD
    F.build()
    FD.build()
    assert F.have_ref() and FD.have_ref(), "the reference tree is needed"
    R, RD = F.ref(), FD.ref()
    out = {}
    filled = {}
    for name, (raw, nd) in rasters().items():
        filled[name] = (raw, R.fill(raw, "D8"), nd)
    rng = np.random.default_rng(29)
    for name, src, nd in (("nodata_m32768", "fbm_subfloat", -32768.0), ("nodata_1e39", "fbm_between", 1e39)):
        dem = filled[src][1].copy()
        for _ in range(6):
            y, x = rng.integers(0, dem.shape[0] - 6), rng.integers(0, dem.shape[1] - 6)
            dem[y:y + rng.integers(1, 6), x:x + rng.integers(1, 6)] = nd
        filled[name] = (None, dem, nd)
    for name, (raw, dem, nd) in filled.items():
        if raw is not None:
            out[f"{name}/raw"] = raw
        out[f"{name}/dem"] = dem
        out[f"{name}/nodata"] = np.float64(nd)
        d0, _ = RD.flowdirs_flats(dem, nd, False)
        d1, dem1 = RD.flowdirs_flats(dem, nd, True)
        m, lab = RD.flat_mask(dem, nd)
        out[f"{name}/dirs0"] = d0
        out[f"{name}/dirs1"] = d1
        out[f"{name}/dem1"] = dem1
        out[f"{name}/mask"] = m
        out[f"{name}/labels"] = lab
        out[f"{name}/area0"] = RD.d8_flow_accum(d0)
        print(f"{name}: {dem.shape}, max increment {m.max()}, altered cells {int(np.sum(dem1.view(np.uint64) != dem.view(np.uint64)))}")
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
