"""Per-kernel device time of unit-weight FA_D8 (rdb200_dev_fa_d8_f32_f64) from torch.profiler, on bench.py's fBm raster
after the fill ("filled") and after the fill and flat resolution ("resolved"):
    python tools/fa_d8_kernels.py 32768 [--reps 5] [--root OTHER_TREE] [--out result.json]
--root loads the library of another checkout (e.g. the parent commit's build) to compare kernels side by side.
Also prints the call's time from CUDA events in a run of its own, without the profiler."""
import argparse
import json
import os
import sys

ap = argparse.ArgumentParser()
ap.add_argument("n", type=int)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--out")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402
from richdem_b200 import _lib  # noqa: E402

ND = -9999.0
N = args.n
L = _lib.lib()
_lib.init(0)
_lib.use_torch_stream()
d = torch.empty((N, N), dtype=torch.float32, device="cuda")
_lib.check(L.rdb200_dev_generate_fbm_f32(d.data_ptr(), N, N, 0, 42, 12, 0.0))
_lib.check(L.rdb200_dev_fill_depressions_d8_f32(d.data_ptr(), N, N))
r = d.clone()
_lib.check(L.rdb200_dev_resolve_flats_epsilon_f32(r.data_ptr(), N, N, ND))
acc = torch.empty((N, N), dtype=torch.float64, device="cuda")


def fa(dem):
    _lib.check(L.rdb200_dev_fa_d8_f32_f64(dem.data_ptr(), acc.data_ptr(), N, N, ND, 1))


result = {"library": os.path.abspath(L._name), "n": N, "reps": args.reps, "gpu": torch.cuda.get_device_name(0)}
for name, dem in (("filled", d), ("resolved", r)):
    fa(dem)  # warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        fa(dem)
    e1.record()
    torch.cuda.synchronize()
    call_ms = e0.elapsed_time(e1) / args.reps
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            fa(dem)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t > 0:
            kernels[ev.key[:90]] = round(t / 1e3 / args.reps, 3)  # ms per call
    result[name] = {"call_ms": round(call_ms, 3), "kernels_ms": dict(sorted(kernels.items(), key=lambda kv: -kv[1]))}
    print(f"{name}: FA_D8 {call_ms:.2f} ms per call (events)", flush=True)
    for k, v in result[name]["kernels_ms"].items():
        print(f"    {v:9.3f} ms  {k}", flush=True)
if args.out:
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
