"""Search for terrain on which the packed fixed-point D-infinity walk (accum_dinf_packed) is least accurate, and write the
best patch to tests/golden/dinf_packed_worst.npz.

The walk rounds every share of a two-receiver cell to 2^-24, so the relative error is largest at a cell of small
accumulation that takes several rounded shares.  Each candidate is a 7 x 7 patch of elevations in a NoData frame; 4096 of
them are tiled into one raster, their proportions come from the checker's FM_Tarboton, and the walk is replayed exactly
by oracle/accum_exact.  The score of a patch is the relative error at its centre.  A generation keeps the best patches
and perturbs one to three elevations of each by a random amount between 1e-5 and 10.

    python tools/dinf_packed_worst.py [--seed 2] [--generations 150] [--out tests/golden/dinf_packed_worst.npz]
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from oracle import accum_exact  # noqa: E402

ND = -9999.0
P, K = 9, 64  # patch size (7 x 7 elevations and the NoData frame); K x K patches per batch


def tile(patches):
    dem = np.full((K * P, K * P), ND, np.float32)
    for k, p in enumerate(patches):
        y, x = divmod(k, K)
        dem[y * P + 1:y * P + P - 1, x * P + 1:x * P + P - 1] = p
    return dem


def scores(O, patches):
    e = accumulate_packed(O, tile(patches))
    c = P // 2
    ys, xs = np.divmod(np.arange(len(patches)), K)
    yy, xx = ys * P + c, xs * P + c
    return np.abs(e.packed[yy, xx] - e.ref[yy, xx]) / e.ref[yy, xx]


def accumulate_packed(O, dem):
    return accum_exact.accumulate(O.fm_dinf(dem, ND), mode="packed")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--generations", type=int, default=150)
    ap.add_argument("--out", default=os.path.join("tests", "golden", "dinf_packed_worst.npz"))
    a = ap.parse_args()
    O = oracle.best()
    rng = np.random.default_rng(a.seed)
    pop = [rng.random((P - 2, P - 2)).astype(np.float32) * 100 for _ in range(K * K)]
    best, best_r = None, 0.0
    for gen in range(a.generations):
        r = scores(O, pop)
        i = int(r.argmax())
        if r[i] > best_r:
            best, best_r = pop[i].copy(), float(r[i])
        print(f"generation {gen}: {best_r:.4e} = {best_r / 2.0 ** -22:.3f} x 2^-22", flush=True)
        elite = [pop[j] for j in np.argsort(r)[-16:]] + [best]
        pop = []
        for _ in range(K * K):
            q = elite[rng.integers(len(elite))].copy()
            for _ in range(rng.integers(1, 4)):
                y, x = rng.integers(0, P - 2, 2)
                q[y, x] = np.float32(q[y, x] + rng.normal() * 10.0 ** rng.uniform(-5, 1))
            pop.append(q)
    np.savez_compressed(a.out, patch=best)
    print(f"wrote {a.out}: relative error {best_r:.4e} at the centre")


if __name__ == "__main__":
    main()
