"""Regenerates tests/golden/depression_masks_ref.npz (run where the reference tree exists).

The reference's pit_mask<D8 / D4> and HasDepressions<D8 / D4> (include/richdem/depressions/Barnes2014.hpp:593-676,
:43-104), compiled unmodified by oracle/depressions.py from oracle/depressions_shim.cpp, on the inputs below: stored in
full for the small rasters, as digests of the masks for the large fBm rasters (which the tests regenerate from their
recipe).  The small inputs reuse two existing fixtures (fill_testdem1.npz: the reference's tests/depressions/testdem1;
beauford_crop.npz: the Beauford crop with NoData) and add seeded synthetic rasters.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from oracle import depressions  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0

# digest-only fixtures: (rows, cols, seed, quantum) of oracle.fbm_terrain
LARGE = {"fbm_large": (1100, 1300, 94, 0.5)}


def inputs():
    """{name: (dem, nodata)} of the fixtures stored in full."""
    t = np.load(f"{OUT}/fill_testdem1.npz")
    b = np.load(f"{OUT}/beauford_crop.npz")
    fbm = oracle.fbm_terrain(150, 170, seed=91, quantum=0.5)
    hole = np.add.outer(np.arange(60, dtype=np.float32), 2 * np.arange(70, dtype=np.float32))  # drains to the corner
    hole[20:31, 25:40] = ND  # ... except an enclosed NoData hole: a depression without a strict pit
    terraced = oracle.fbm_terrain(120, 140, seed=92, quantum=150.0)  # flat-bottomed basins
    inf = oracle.fbm_terrain(64, 80, seed=93, quantum=0.5)
    inf[10:30, 10] = inf[10:30, 30] = inf[10, 10:31] = inf[29, 10:31] = np.inf  # an infinite wall around a basin
    inf[40, 50] = -np.inf
    inf[50, 5:60] = -np.inf
    inf[0, 7] = -np.inf
    return {
        "testdem1": (t["dem"], float(t["nodata"])), "beauford": (b["dem"], float(b["nodata"])), "fbm_q05": (fbm, ND),
        "nodata_hole": (hole, ND), "no_depressions": (oracle.ref().fill_depressions(fbm), ND), "terraced": (terraced, ND),
        "row_1xN": (fbm[40:41, :].copy(), ND), "col_Nx1": (fbm[:, 60:61].copy(), ND), "square_2x2": (fbm[3:5, 3:5].copy(), ND),
        "all_nodata": (np.full((9, 11), ND, np.float32), ND), "infinities": (inf, ND),
    }


def main():
    R = depressions.ref()
    out = {}
    for name, (dem, nd) in inputs().items():
        out[f"{name}__dem"], out[f"{name}__nodata"] = dem.astype(np.float32), np.float32(nd)
        for topo in ("D8", "D4"):
            out[f"{name}__mask_{topo}"] = R.pit_mask(dem, nd, topo)
            out[f"{name}__has_{topo}"] = np.bool_(R.has_depressions(dem, topo))
    for name, (h, w, seed, q) in LARGE.items():
        dem = oracle.fbm_terrain(h, w, seed=seed, quantum=q)
        out[f"{name}__recipe"] = np.array([h, w, seed, q], np.float64)
        for topo in ("D8", "D4"):
            out[f"{name}__mask_{topo}_digest"] = np.array(oracle.digest(R.pit_mask(dem, ND, topo)))
            out[f"{name}__has_{topo}"] = np.bool_(R.has_depressions(dem, topo))
    np.savez_compressed(f"{OUT}/depression_masks_ref.npz", **out)


if __name__ == "__main__":
    main()
