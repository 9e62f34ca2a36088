"""The direction-grid pipeline on bench.py's fBm raster (filled), timed with CUDA events, alternating: the row-band
drivers with one band (sharded.d8_flow_directions_band -> rdb200_mgpu_d8_flow_directions_flats_f32 and
sharded.d8_flow_accum_band -> rdb200_mgpu_d8_flow_accum_u8_i32, world 1) and the single-GPU calls
(rdb200_dev_d8_flow_directions_flats_f32 with alter = 0, rdb200_dev_d8_flow_accum_u8_i32).  Both are device-resident; the
directions start from a fresh copy of the filled raster (the copy is not timed), and both accumulations read the same
directions.  This measures what the band machinery costs on one GPU, not a multi-GPU speed-up.
    python tools/d8_dirs_band_timing.py 16384 [--reps 5] [--out result.json]
Prints the card name and power limit with the times, and whether the two results are the same bits."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("n", type=int)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--out")
args = ap.parse_args()
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from richdem_b200 import _lib, sharded  # noqa: E402

ND = -9999.0
N = args.n
L = _lib.lib()
_lib.init(0)
_lib.use_torch_stream()
filled = torch.empty((N, N), dtype=torch.float32, device="cuda")
_lib.check(L.rdb200_dev_generate_fbm_f32(filled.data_ptr(), N, N, 0, 42, 12, 0.0))
_lib.check(L.rdb200_dev_fill_depressions_d8_f32(filled.data_ptr(), N, N))
work = torch.empty_like(filled)
dirs = torch.empty((N, N), dtype=torch.uint8, device="cuda")
area = torch.empty((N, N), dtype=torch.int32, device="cuda")
out = {}


def dirs_band():
    out["dirs"], _ = sharded.d8_flow_directions_band(work, 0, 0, ND)


def dirs_single():
    _lib.check(L.rdb200_dev_d8_flow_directions_flats_f32(work.data_ptr(), dirs.data_ptr(), N, N, ND, 0))
    out["dirs"] = dirs


def accum_band():
    out["area"], _ = sharded.d8_flow_accum_band(out["dirs"], 0, 0)


def accum_single():
    _lib.check(L.rdb200_dev_d8_flow_accum_u8_i32(out["dirs"].data_ptr(), area.data_ptr(), N, N))
    out["area"] = area


def timed(fn, fresh):
    if fresh:
        work.copy_(filled)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


# warm-up, and the results compared below
timed(dirs_band, True)
timed(accum_band, False)
r_dirs, r_area = out["dirs"].clone(), out["area"].clone()
timed(dirs_single, True)
timed(accum_single, False)
same_bits = {"dirs": bool(torch.equal(r_dirs, out["dirs"])), "area": bool(torch.equal(r_area, out["area"]))}
no_flow = int((r_dirs == 0).sum().item())
del r_dirs, r_area
times = {k: [] for k in ("dirs_band_world1", "dirs_single_gpu", "accum_band_world1", "accum_single_gpu")}
for _ in range(args.reps):
    times["dirs_band_world1"].append(timed(dirs_band, True))
    times["accum_band_world1"].append(timed(accum_band, False))
    times["dirs_single_gpu"].append(timed(dirs_single, True))
    times["accum_single_gpu"].append(timed(accum_single, False))
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
result = {"n": N, "reps": args.reps, "gpu": torch.cuda.get_device_name(0),
          "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unavailable",
          "same_bits": same_bits, "no_flow_cells": no_flow,
          "ms": {k: [round(t, 3) for t in v] for k, v in times.items()},
          "median_ms": {k: round(statistics.median(v), 3) for k, v in times.items()}}
print(json.dumps(result), flush=True)
if args.out:
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
