"""Times the float64 path on one GPU: the key build (the cast case and the rank case separately), the float64 fill
against the float32 fill of the same raster rounded to float and against the float32 fill of its rank keys alone, and
float64 ResolveFlats and FA_D8.  Every figure is
the median of alternating repetitions (each repetition runs every item once, in turn), timed with CUDA events around the
device entry point; inputs are copied in before the start event.  The card and its power limit are printed by the same
run.

    python tools/f64_timing.py [sizes...]   (default 16384 32768)
"""
import ctypes as C
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


def run(n: int) -> dict:
    L = _lib.lib()
    zf = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.check(L.rdb200_dev_generate_fbm_f32(zf.data_ptr(), n, n, 0, 42, 12, 0))
    work = torch.empty((n, n), dtype=torch.float64, device="cuda")
    filled = torch.empty_like(work)
    keys = torch.empty_like(zf)
    nodata = -9999.0
    ndk, rk = C.c_float(0), C.c_int32(0)

    def widened(dst):     # case 1: the float raster, widened
        return lambda: dst.copy_(zf)

    def detailed(dst):    # case 2: sub-float detail on a sparse lattice of cells
        def prep():
            dst.copy_(zf)
            dst[::7, ::5] += 2.0 ** -30
        return prep

    def order_keys():
        _lib.check(L.rdb200_dev_f64_order_keys(work.data_ptr(), keys.data_ptr(), n, n, nodata, C.byref(ndk), C.byref(rk)))

    detailed(filled)()
    _lib.check(L.rdb200_dev_fill_depressions_d8_f64(filled.data_ptr(), n, n))  # flats and FA_D8 run on the filled raster
    items = {
        "keys_case1_cast": (order_keys, widened(work)),
        "keys_case2_rank": (order_keys, detailed(work)),
        "fill_d8_f64_case2": (lambda: _lib.check(L.rdb200_dev_fill_depressions_d8_f64(work.data_ptr(), n, n)), detailed(work)),
        "fill_d8_f32_rounded": (lambda: _lib.check(L.rdb200_dev_fill_depressions_d8_f32(keys.data_ptr(), n, n)),
                                lambda: keys.copy_(zf)),
        # the float engine alone on the rank keys of the same raster: the level schedule on keys spread over many binades
        "fill_d8_f32_on_rank_keys": (lambda: _lib.check(L.rdb200_dev_fill_depressions_d8_f32(keys.data_ptr(), n, n)),
                                     lambda: (detailed(work)(), order_keys())),
        "fill_d8_f64_case1": (lambda: _lib.check(L.rdb200_dev_fill_depressions_d8_f64(work.data_ptr(), n, n)), widened(work)),
        "resolve_flats_f64": (lambda: _lib.check(L.rdb200_dev_resolve_flats_epsilon_f64(work.data_ptr(), n, n, nodata)),
                              lambda: work.copy_(filled)),
        "fa_d8_f64": (lambda: _lib.check(L.rdb200_dev_fa_d8_f64_f64(filled.data_ptr(), work.data_ptr(), n, n, nodata, 1)),
                      lambda: None),
    }
    times = {k: [] for k in items}
    ranked = {}
    for _ in range(REPS):
        for k, (fn, prep) in items.items():
            times[k].append(timed(fn, prep))
            if k.startswith("keys") or k == "fill_d8_f32_on_rank_keys":
                ranked[k] = bool(rk.value)
    out = {"n": n}
    for k, v in times.items():
        out[k + "_ms"] = round(float(np.median(v)), 2)
    out["ranked"] = ranked
    del zf, work, filled, keys
    _lib.set_param("trim_workspace", 1)
    torch.cuda.empty_cache()
    return out


def main() -> None:
    sizes = [int(a) for a in sys.argv[1:]] or [16384, 32768]
    _lib.init(torch.cuda.current_device())
    print(json.dumps({"card": card()}))
    for n in sizes:
        print(json.dumps(run(n)), flush=True)


if __name__ == "__main__":
    main()
