"""FillDepressions<D4> on bench.py's fBm raster, timed with CUDA events, alternating: the row-band driver with one band
(sharded.fill_band(topology="D4") -> rdb200_mgpu_fill_depressions_d4_f32, world 1) and the single-GPU call
(rdb200_dev_fill_depressions_d4_f32).  Both are device-resident and start from a fresh copy of the raster (the copy is not
timed).  This measures what the band machinery costs on one GPU, not a multi-GPU speed-up.
    python tools/d4_fill_band_timing.py 16384 [--reps 5] [--out result.json]
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

N = args.n
L = _lib.lib()
_lib.init(0)
_lib.use_torch_stream()
dem = torch.empty((N, N), dtype=torch.float32, device="cuda")
_lib.check(L.rdb200_dev_generate_fbm_f32(dem.data_ptr(), N, N, 0, 42, 12, 0.0))
work = torch.empty_like(dem)


def band():
    sharded.fill_band(work, 0, 0, topology="D4")


def single():
    _lib.check(L.rdb200_dev_fill_depressions_d4_f32(work.data_ptr(), N, N))


def timed(fn):
    work.copy_(dem)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


timed(band)  # warm-up, and the results compared below
r_band = work.clone()
timed(single)
same_bits = bool(torch.equal(r_band.view(torch.int32), work.view(torch.int32)))
changed = int((r_band != dem).sum().item())
del r_band
times = {"band_world1": [], "single_gpu": []}
for _ in range(args.reps):
    times["band_world1"].append(timed(band))
    times["single_gpu"].append(timed(single))
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
result = {"n": N, "reps": args.reps, "gpu": torch.cuda.get_device_name(0),
          "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unavailable",
          "same_bits": same_bits, "cells_raised": changed,
          "ms": {k: [round(t, 3) for t in v] for k, v in times.items()},
          "median_ms": {k: round(statistics.median(v), 3) for k, v in times.items()}}
print(json.dumps(result), flush=True)
if args.out:
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
