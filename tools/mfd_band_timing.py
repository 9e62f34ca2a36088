"""Unit-weight flow accumulation of one proportions method on bench.py's fBm raster (filled, flats resolved), timed with
CUDA events, alternating: the row-band driver with one band (sharded.fa_band -> rdb200_mgpu_fa_method_f32_f64, world 1)
and the single-GPU call (rdb200_dev_fa_method_f32_f64 after setting the weights to 1).  Both are device-resident.
    python tools/mfd_band_timing.py 16384 [--method Quinn] [--exponent X] [--reps 5] [--out result.json]
Prints the card name and power limit with the times, and the largest relative difference between the two results."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("n", type=int)
ap.add_argument("--method", default="Quinn")
ap.add_argument("--exponent", type=float)
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
mid, xparam = sharded.fa_method_id(args.method, args.exponent)
d = torch.empty((N, N), dtype=torch.float32, device="cuda")
_lib.check(L.rdb200_dev_generate_fbm_f32(d.data_ptr(), N, N, 0, 42, 12, 0.0))
_lib.check(L.rdb200_dev_fill_depressions_d8_f32(d.data_ptr(), N, N))
_lib.check(L.rdb200_dev_resolve_flats_epsilon_f32(d.data_ptr(), N, N, ND))
single_acc = torch.empty((N, N), dtype=torch.float64, device="cuda")


def band():
    return sharded.fa_band(d, 0, 0, ND, method=args.method, exponent=args.exponent)[0]


def single():
    single_acc.fill_(1.0)
    _lib.check(L.rdb200_dev_fa_method_f32_f64(mid, d.data_ptr(), single_acc.data_ptr(), N, N, ND, xparam))
    return single_acc


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


a_band, a_single = band(), single().clone()  # warm-up, and the results compared below
torch.cuda.synchronize()
ok = a_single >= 0
rel = ((a_band - a_single).abs() / a_single.abs().clamp(min=1.0))[ok].max().item()
nodata_same = bool(torch.equal(a_band < 0, a_single < 0))
del a_band, a_single
times = {"band_world1": [], "single_gpu": []}
for _ in range(args.reps):
    times["band_world1"].append(timed(band)[0])
    times["single_gpu"].append(timed(single)[0])
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
result = {"n": N, "method": args.method, "exponent": args.exponent, "reps": args.reps, "gpu": torch.cuda.get_device_name(0),
          "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unavailable",
          "max_rel_diff": rel, "nodata_same": nodata_same,
          "ms": {k: [round(t, 3) for t in v] for k, v in times.items()},
          "median_ms": {k: round(statistics.median(v), 3) for k, v in times.items()}}
print(json.dumps(result), flush=True)
if args.out:
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
