"""Per-kernel device time of the single-GPU fill (rdb200_dev_fill_depressions_d8_f32) from torch.profiler, on bench.py's
fBm raster, and the device scratch the call leaves in the library's workspace cache:
    python tools/fill_kernels.py 32768 [--reps 3] [--root OTHER_TREE] [--out result.json]
--root loads the library of another checkout (e.g. the parent commit's build) to compare kernels side by side.
`first_round_ms` is the longest sweep launch of a call: the first round of the full-size level, which visits every tile.
`scratch_gib` is the free device memory lost to the first call in a fresh process (cudaMemGetInfo before and after;
the workspace cache only grows, so this bounds the call's peak scratch from above).
`--param k=v` (repeatable) sets a library parameter for every call, e.g. fill_wake_filter=0.  A last call with
fill_profile=1 counts the tile visits, the idle ones (visits that changed nothing) and the neighbour wakes the wake test
dropped, summed over every solver of the call (`wake`; null for a library that does not report them)."""
import argparse
import json
import os
import sys
import tempfile

ap = argparse.ArgumentParser()
ap.add_argument("n", type=int)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--out")
ap.add_argument("--param", action="append", default=[], metavar="K=V")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402
from richdem_b200 import _lib  # noqa: E402

N = args.n
L = _lib.lib()
_lib.init(0)
_lib.use_torch_stream()
params = {k: int(v) for k, v in (p.split("=") for p in args.param)}
for k, v in params.items():
    _lib.set_param(k, v)
dem = torch.empty((N, N), dtype=torch.float32, device="cuda")
_lib.check(L.rdb200_dev_generate_fbm_f32(dem.data_ptr(), N, N, 0, 42, 12, 0.0))
w = torch.empty_like(dem)


def fill():
    w.copy_(dem)
    _lib.check(L.rdb200_dev_fill_depressions_d8_f32(w.data_ptr(), N, N))


torch.cuda.synchronize()
free0 = torch.cuda.mem_get_info()[0]
fill()
torch.cuda.synchronize()
scratch = (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30
st = _lib.stats()
result = {"library": os.path.abspath(L._name), "n": N, "params": params, "reps": args.reps, "gpu": torch.cuda.get_device_name(0),
          "scratch_gib": round(scratch, 3), "rounds": st["fill_rounds"], "visits": st["fill_tile_visits"]}
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(args.reps):
    fill()
e1.record()
torch.cuda.synchronize()
result["call_ms"] = round(e0.elapsed_time(e1) / args.reps, 3)
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.reps):
        fill()
    torch.cuda.synchronize()
kernels = {}
for ev in prof.key_averages():
    t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
    if t > 0:
        kernels[ev.key[:90]] = round(t / 1e3 / args.reps, 3)  # ms per call
result["kernels_ms"] = dict(sorted(kernels.items(), key=lambda kv: -kv[1]))
sweeps = [ev.time_range.elapsed_us() for ev in prof.events() if "fill_sweep_kernel" in ev.name]
result["first_round_ms"] = round(max(sweeps) / 1e3, 3) if sweeps else None
print(f"fill {result['call_ms']:.2f} ms per call (events); first round {result['first_round_ms']} ms; "
      f"scratch {scratch:.2f} GiB; rounds {result['rounds']} visits {result['visits']}", flush=True)
for k, v in result["kernels_ms"].items():
    print(f"    {v:9.3f} ms  {k}", flush=True)


def profiled_counts():
    """one call with fill_profile = 1; its "[fill wake]" lines on stderr (one per solver run), summed"""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            _lib.set_param("fill_profile", 1)
            fill()
            torch.cuda.synchronize()
        finally:
            _lib.set_param("fill_profile", 0)
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        lines = [ln for ln in f.read().splitlines() if ln.startswith("[fill wake]")]
    if not lines:
        return None
    tot = {}
    for ln in lines:
        for kv in ln.split()[2:]:
            k, v = kv.split("=")
            tot[k] = tot.get(k, 0) + int(v)
    return tot


result["wake"] = profiled_counts()
if result["wake"]:
    w = result["wake"]
    print(f"visits {w['visits']}, idle {w['idle_visits']} ({100.0 * w['idle_visits'] / max(1, w['visits']):.1f} %), "
          f"wakes dropped by the wake test {w['wakes_dropped']}  (fill_profile = 1 call)", flush=True)
if args.out:
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
