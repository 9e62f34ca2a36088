"""Writes tests/golden/f64_ref.npz: the unmodified reference templates with T = double (oracle/f64_shim.cpp) on the
inputs of oracle.f64.cases() -- fBm with sub-float detail, a Beauford crop with 1e-9 noise, nested lakes one double ulp
apart, DBL_MAX plateaus, +-FLT_MAX, +-inf, +-0, subnormals, +-1e300, NoData present / absent / +-inf, 1 x N, N x 1,
2 x 2.  For every case ``<name>__dem``, ``__nodata``, ``__fill_{D8,D4}``, ``__mask_{D8,D4}``, ``__has_{D8,D4}``,
``__resolved``, ``__dirs``, ``__fa_{D8,D4}`` (unit weights), ``__weights`` and ``__fa_{D8,D4}_w``.

    python tests/golden/make_f64.py
"""
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)

from oracle import f64 as F  # noqa: E402


def main() -> None:
    R = F.ref()
    out = {}
    for name, z, nd in F.cases():
        out[f"{name}__dem"] = z
        out[f"{name}__nodata"] = np.float64(nd)
        w = np.random.default_rng(11).random(z.shape)
        out[f"{name}__weights"] = w
        for topo in ("D8", "D4"):
            out[f"{name}__fill_{topo}"] = R.fill(z, topo)
            out[f"{name}__mask_{topo}"] = R.pit_mask(z, nd, topo)
            out[f"{name}__has_{topo}"] = np.bool_(R.has_depressions(z, topo))
            out[f"{name}__fa_{topo}"] = R.fa(z, nd, topo)
            out[f"{name}__fa_{topo}_w"] = R.fa(z, nd, topo, weights=w)
        out[f"{name}__resolved"] = R.resolve_flats(z, nd)
        out[f"{name}__dirs"] = R.d8_flow_directions(z, nd)
    path = os.path.join(ROOT, "tests", "golden", "f64_ref.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
