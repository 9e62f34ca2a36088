"""Timing of PitMask and HasDepressions on one GPU (device entry points, raster already in HBM).

    python tools/depression_masks_timing.py [--size 32768] [--repeats 3] [--out timing.json]

Reports, on the benchmark's fBm raster (rdb200_dev_generate_fbm_f32, seed 42):
  * fill      -- rdb200_dev_fill_depressions_d8_f32 on a copy of the raster (the copy is not timed);
  * pit_mask  -- rdb200_dev_pit_mask_d8_f32: a device copy of the raster, the same fill on it, and the fused compare pass
                 (4 B of elevation + 4 B of water level read, 1 B of mask written per cell);
  * has_depressions on the fBm raster, where the strict-pit pass answers, and on its fill, which has no depression and
    no strict pit, so the fill runs after the stencil pass.
Times are host wall clock around calls that end in a device synchronise (the C ABI's calls are synchronous), best of
--repeats after one warm-up call; the GPU's name and power limit are recorded with them.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return f"unknown ({exc})"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=32768)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from richdem_b200 import _lib
    _lib.init(0)
    L = _lib.lib()
    n = a.size
    dem = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.check(L.rdb200_dev_generate_fbm_f32(dem.data_ptr(), n, n, 0, 42, 12, 0.0))
    work = torch.empty_like(dem)
    mask = torch.empty((n, n), dtype=torch.uint8, device="cuda")
    out = C.c_int32(0)

    def best(prepare, call):
        ts = []
        for i in range(a.repeats + 1):
            prepare()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            call()
            torch.cuda.synchronize()
            if i:
                ts.append((time.perf_counter() - t0) * 1e3)
        return min(ts), ts

    nop = lambda: None  # noqa: E731
    res = {"gpu": gpu_info(), "size": n, "cells": n * n}
    res["fill_ms"], res["fill_all_ms"] = best(lambda: work.copy_(dem),
                                               lambda: _lib.check(L.rdb200_dev_fill_depressions_d8_f32(work.data_ptr(), n, n)))
    filled = work.clone()
    res["pit_mask_ms"], res["pit_mask_all_ms"] = best(nop, lambda: _lib.check(
        L.rdb200_dev_pit_mask_d8_f32(dem.data_ptr(), mask.data_ptr(), n, n, -9999.0)))
    res["pit_cells"] = int((mask == 1).sum().item())

    def has(t):
        _lib.check(L.rdb200_dev_has_depressions_d8_f32(t.data_ptr(), n, n, C.byref(out)))
        return out.value

    res["has_fbm_ms"], res["has_fbm_all_ms"] = best(nop, lambda: has(dem))
    res["has_fbm"] = bool(out.value)
    res["has_fbm_launches"] = _lib.stats()["kernel_launches"]
    res["has_filled_ms"], res["has_filled_all_ms"] = best(nop, lambda: has(filled))
    res["has_filled"] = bool(out.value)
    res["pit_mask_minus_fill_ms"] = res["pit_mask_ms"] - res["fill_ms"]
    # the compare pass and the scratch copy at the card's bandwidth: 9 B/cell and 8 B/cell
    res["compare_and_copy_bytes"] = 17 * n * n
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
