"""Writes tests/golden/f64_flowmet_ref.npz: the reference's double templates of FM_*, FA_* and TA_*
(oracle/f64_flowmet_shim.cpp) on float64 rasters, the fixtures of the float64 D-infinity / MFD / terrain-attribute path.

    python tests/golden/make_f64_flowmet.py        (needs oracle/_ref/libref_f64_flowmet.so, i.e. the reference tree)

Inputs: oracle.f64.cases(), plus
  huge      fBm x 1e200: squared slopes overflow, the differences stay finite
  tiny      fBm x 1e-305: squared slopes underflow, the ratio-test products are subnormal
  near_tie  3x3 cells whose two steepest D-infinity facets differ by one double ulp, for every pair of facet cases
  beauford_data_1e-9  an all-data crop of beauford_crop.npz with 1e-9 detail: the float-rounded raster's D-infinity
            facets differ from the double answer
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
OUT = os.path.join(HERE, "f64_flowmet_ref.npz")

# (method, exponent) as the C ABI numbers methods: 0 D8, 1 Tarboton, 2 D4, 3 Holmgren (Quinn at 1), 4 Freeman.  Holmgren
# and Freeman between them take the exponents 1.0, 0.5, 1.1 and 4.  Every raster gets the full set unless it is one of
# BRIEF: near copies of fbm_subfloat or sentinels, or larger crops, that add ground for D-infinity, attributes and
# NoData handling only.  MFD proportions do not compress, and this keeps the file small.
FM_RUNS = [(0, 1.0), (1, 1.0), (2, 1.0), (3, 1.0), (3, 0.5), (4, 1.1), (4, 4.0)]
FA_RUNS = [(1, 1.0), (3, 1.0), (4, 1.1)]
TA_RUNS = list(range(8))
BRIEF = ("float_raster", "nodata_absent", "nodata_present", "sentinels_nodata_inf", "sentinels_nodata_dblmax",
         "beauford_1e-9", "beauford_data_1e-9")
BRIEF_FM_RUNS = [(1, 1.0)]
BRIEF_FA_RUNS = [(1, 1.0)]
BRIEF_TA_RUNS = [2, 7]
# fbm_subfloat keeps every stencil but the MFD exponents other than 1 (sentinels, huge, tiny and the small rasters take
# those)
FBM_RUNS = (FM_RUNS[:4], [(1, 1.0), (3, 1.0)], TA_RUNS)
TA_ZSCALE = 2.5
TA_CELL = (2.0, 3.0)

# facet tables of Tarboton1997.hpp:48-53 (remapped facets 1..8)
_DY1 = [0, 0, -1, -1, 0, 0, 1, 1, 0]
_DX1 = [0, -1, 0, 0, 1, 1, 0, 0, -1]
_DY2 = [0, -1, -1, -1, -1, 1, 1, 1, 1]
_DX2 = [0, -1, -1, 1, 1, 1, 1, -1, -1]
_DANG = float(np.float32(np.arctan2(1.0, 1.0)))


def dinf_facets(p):
    """The reference's per-facet (case, slope) of the centre of each 3x3 patch p[..., 3, 3] (Tarboton1997.hpp:88-107)."""
    e0 = p[..., 1, 1]
    cases, slopes = [], []
    for n in range(1, 9):
        e1 = p[..., 1 + _DY1[n], 1 + _DX1[n]]
        e2 = p[..., 1 + _DY2[n], 1 + _DX2[n]]
        s1, s2 = e0 - e1, e1 - e2
        with np.errstate(all="ignore"):
            r = np.arctan2(s2, s1)
            c = np.where(r < 1e-7, 0, np.where(r > _DANG - 1e-7, 1, 2))
            s = np.where(c == 0, s1, np.where(c == 1, (e0 - e2) / np.sqrt(2.0), np.sqrt(s1 * s1 + s2 * s2)))
        cases.append(c)
        slopes.append(s)
    return np.stack(cases, -1), np.stack(slopes, -1)


def near_tie() -> np.ndarray:
    """One 3x3 cell (side by side in a 3-row strip, a NoData -9999 column between) per unordered pair of facet cases whose two steepest facets
    differ by exactly one double ulp.  Centre 0, so s1 = -e1 and e0 - e2 = -e2 are exact; the values are slopes 5 in each
    case (case 0: e1 = -5; case 1: e2 = -5 sqrt 2; case 2: s1 = 4, s2 = 3) give or take a few ulps."""
    rng = np.random.default_rng(11)
    u = lambda v, k: v + k * np.spacing(v)  # noqa: E731
    card = np.array([u(-5.0, k) for k in range(-3, 4)] + [-4.0, -1.0, 1.0, 3.0])
    diag = np.array([u(-5.0 * np.sqrt(2.0), k) for k in range(-3, 4)] + [-7.0, u(-7.0, 1), u(-7.0, -1), 8.0, 2.0])
    found = {}
    for _ in range(60):
        m = 200000
        p = np.zeros((m, 3, 3))
        for (yy, xx) in ((0, 1), (1, 0), (1, 2), (2, 1)):
            p[:, yy, xx] = rng.choice(card, m)
        for (yy, xx) in ((0, 0), (0, 2), (2, 0), (2, 2)):
            p[:, yy, xx] = rng.choice(diag, m)
        c, s = dinf_facets(p)
        s = np.where(np.isnan(s), -np.inf, s)
        itop = np.argmax(s, -1)  # the first steepest facet, as the reference's strict `s > smax` picks it
        top = np.take_along_axis(s, itop[:, None], -1)[:, 0]
        below = np.where(s < top[:, None], s, -np.inf)  # the steepest slope of the other facets (twins of top excluded)
        isec = np.argmax(below, -1)
        sec = np.take_along_axis(below, isec[:, None], -1)[:, 0]
        ctop, csec = np.take_along_axis(c, itop[:, None], -1)[:, 0], np.take_along_axis(c, isec[:, None], -1)[:, 0]
        ok = (sec > 0) & (np.nextafter(sec, np.inf) == top)
        for i in np.flatnonzero(ok):
            key = tuple(sorted((int(ctop[i]), int(csec[i]))))
            found.setdefault(key, p[i])
        if len(found) == 6:
            break
    pairs = sorted(found)
    z = np.full((3, 4 * len(pairs) + 1), -9999.0)
    for k, key in enumerate(pairs):
        z[:, 4 * k + 1:4 * k + 4] = found[key]
    return z, pairs


def inputs():
    """(name, Z, nodata) of every fixture raster."""
    sys.path.insert(0, ROOT)
    from oracle import f64 as F
    from oracle import fbm_terrain
    out = list(F.cases())
    fbm = fbm_terrain(24, 32, seed=9, quantum=0.25).astype(np.float64)
    out.append(("huge", fbm * 1e200, -9999.0))
    out.append(("tiny", fbm * 1e-305, -9999.0))
    z, _ = near_tie()
    out.append(("near_tie", z, -9999.0))
    # cases()'s beauford_1e-9 lies mostly in NoData; this crop is all data, and rounding it to float moves D-infinity
    # receivers in several cells
    g = np.load(os.path.join(HERE, "beauford_crop.npz"))
    b = g["dem"][200:240, 250:314].astype(np.float64)
    out.append(("beauford_data_1e-9", b + np.random.default_rng(0).random(b.shape) * 1e-9, float(g["nodata"])))
    return out


def runs(name):
    """(FM runs, FA runs, TA attributes) stored for raster `name`."""
    if name in BRIEF:
        return BRIEF_FM_RUNS, BRIEF_FA_RUNS, BRIEF_TA_RUNS
    if name == "fbm_subfloat":
        return FBM_RUNS
    return FM_RUNS, FA_RUNS, TA_RUNS


def weights(shape):
    """The weights of the stored weighted D-infinity accumulation (fa1_weighted); not stored themselves."""
    return np.random.default_rng(5).random(shape)


def compute(R, name, z, nd):
    """Every fixture output of one raster from the reference's double templates (R = oracle.f64_flowmet.ref())."""
    fm_runs, fa_runs, ta_runs = runs(name)
    d = {}
    for m, x in fm_runs:
        d[f"fm{m}_{x}"] = R.fm(z, nd, m, x)
    for m, x in fa_runs:
        d[f"fa{m}_{x}"] = R.fa(z, nd, m, x)
    if name not in BRIEF:
        d["fa1_weighted"] = R.fa(z, nd, 1, 1.0, weights=weights(z.shape))
    for a in ta_runs:
        d[f"ta{a}"] = R.ta(z, a, nd, TA_ZSCALE, TA_CELL)
    return d


def main():
    sys.path.insert(0, ROOT)
    from oracle import f64_flowmet as FF
    R = FF.ref()
    arrays = {}
    for name, z, nd in inputs():
        arrays[f"{name}/dem"] = z
        arrays[f"{name}/nodata"] = np.float64(nd)
        for k, v in compute(R, name, z, nd).items():
            arrays[f"{name}/{k}"] = v
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
