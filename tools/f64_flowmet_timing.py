"""Times the float64 flow metrics, accumulations and terrain attributes on one GPU against the float32 path on the same
raster (the fBm of rdb200_dev_generate_fbm_f32 with 2^-30 detail on a sparse lattice of cells for float64, the fBm itself
for float32): FM_Tarboton and FM_Quinn into proportions, unit-weight FA_Tarboton, FA_Quinn, and TA slope_degrees and
profile_curvature.  Every figure is the median of alternating repetitions (each repetition runs every item once, in
turn), timed with CUDA events around the device entry point.  Prints the float64 / float32 ratio per stage and, for the
pure stencil stages, the share of 3.35 TB/s their algorithmic bytes per cell make (props 44 B / 40 B, attributes 12 B /
8 B).  The card and its power limit are printed by the same run.

    python tools/f64_flowmet_timing.py [sizes...]   (default 16384 32768)
"""
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from richdem_b200 import _lib  # noqa: E402

REPS = 5
HBM = 3.35e12
BYTES = {"fm": (44, 40), "ta": (12, 8)}  # per cell, float64 / float32


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return f"{torch.cuda.get_device_name()} ({q})"


def timed(fn, prepare):
    prepare()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def measure(items):
    for fn, prep in items.values():  # warm-up: module load, workspace
        timed(fn, prep)
    times = {k: [] for k in items}
    for _ in range(REPS):
        for k, (fn, prep) in items.items():
            times[k].append(timed(fn, prep))
    return {k: float(np.median(v)) for k, v in times.items()}


def run(n: int) -> dict:
    L = _lib.lib()
    nodata = -9999.0
    z32 = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.check(L.rdb200_dev_generate_fbm_f32(z32.data_ptr(), n, n, 0, 42, 12, 0))
    z64 = z32.double()
    z64[::7, ::5] += 2.0 ** -30
    p32, p64 = z32.data_ptr(), z64.data_ptr()
    none = lambda: None  # noqa: E731
    ms = {}
    # proportions: one (n, n, 9) float buffer, freed before the accumulations allocate their own
    props = torch.empty((n, n, 9), dtype=torch.float32, device="cuda")
    pp = props.data_ptr()
    ms.update(measure({
        "fm_tarboton_f64": (lambda: _lib.check(L.rdb200_dev_fm_method_f64(1, p64, pp, n, n, nodata, 1.0)), none),
        "fm_tarboton_f32": (lambda: _lib.check(L.rdb200_dev_fm_method_f32(1, p32, pp, n, n, nodata, 1.0)), none),
        "fm_quinn_f64": (lambda: _lib.check(L.rdb200_dev_fm_method_f64(3, p64, pp, n, n, nodata, 1.0)), none),
        "fm_quinn_f32": (lambda: _lib.check(L.rdb200_dev_fm_method_f32(3, p32, pp, n, n, nodata, 1.0)), none),
    }))
    del props
    _lib.set_param("trim_workspace", 1)
    torch.cuda.empty_cache()
    acc = torch.empty((n, n), dtype=torch.float64, device="cuda")
    out = torch.empty((n, n), dtype=torch.float32, device="cuda")
    pa, po = acc.data_ptr(), out.data_ptr()
    ones = lambda: acc.fill_(1.0)  # noqa: E731
    ms.update(measure({
        "fa_tarboton_f64": (lambda: _lib.check(L.rdb200_dev_fa_tarboton_f64_f64(p64, pa, n, n, nodata, 1)), none),
        "fa_tarboton_f32": (lambda: _lib.check(L.rdb200_dev_fa_tarboton_f32_f64(p32, pa, n, n, nodata, 1)), none),
        "fa_quinn_f64": (lambda: _lib.check(L.rdb200_dev_fa_method_f64_f64(3, p64, pa, n, n, nodata, 1.0)), ones),
        "fa_quinn_f32": (lambda: _lib.check(L.rdb200_dev_fa_method_f32_f64(3, p32, pa, n, n, nodata, 1.0)), ones),
        "ta_slope_degrees_f64": (lambda: _lib.check(L.rdb200_dev_terrain_attribute_f64(2, p64, po, n, n, nodata, -9999.0,
                                                                                        1.0, 1.0, 1.0)), none),
        "ta_slope_degrees_f32": (lambda: _lib.check(L.rdb200_dev_terrain_attribute_f32(2, p32, po, n, n, nodata, -9999.0,
                                                                                        1.0, 1.0, 1.0)), none),
        "ta_profile_curvature_f64": (lambda: _lib.check(L.rdb200_dev_terrain_attribute_f64(7, p64, po, n, n, nodata,
                                                                                            -9999.0, 1.0, 1.0, 1.0)), none),
        "ta_profile_curvature_f32": (lambda: _lib.check(L.rdb200_dev_terrain_attribute_f32(7, p32, po, n, n, nodata,
                                                                                            -9999.0, 1.0, 1.0, 1.0)), none),
    }))
    res = {"n": n}
    cells = float(n) * n
    for stage in ("fm_tarboton", "fm_quinn", "fa_tarboton", "fa_quinn", "ta_slope_degrees", "ta_profile_curvature"):
        t64, t32 = ms[stage + "_f64"], ms[stage + "_f32"]
        r = {"f64_ms": round(t64, 2), "f32_ms": round(t32, 2), "ratio": round(t64 / t32, 3)}
        kind = stage[:2]
        if kind in BYTES:
            b64, b32 = BYTES[kind]
            r["f64_hbm_share"] = round(cells * b64 / (t64 * 1e-3) / HBM, 3)
            r["f32_hbm_share"] = round(cells * b32 / (t32 * 1e-3) / HBM, 3)
        res[stage] = r
    del z32, z64, acc, out
    _lib.set_param("trim_workspace", 1)
    torch.cuda.empty_cache()
    return res


def main() -> None:
    sizes = [int(a) for a in sys.argv[1:]] or [16384, 32768]
    _lib.init(torch.cuda.current_device())
    print(json.dumps({"card": card()}))
    for n in sizes:
        print(json.dumps(run(n)), flush=True)


if __name__ == "__main__":
    main()
