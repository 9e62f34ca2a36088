"""Times FillDepressions(epsilon=True) on one GPU against the plain fill of the same raster: bench.py's fBm (device
generator, seed 42, 12 octaves) at each size, the plain D8 fill, the epsilon D8 fill and the epsilon D4 fill run in turn
REPS times after one warm-up call each, timed with CUDA events around the device entry point (the input is copied in
before the start event).  Reports the median ms, Mcells/s, fill_rounds and tile visits, with the card and its power limit
read in the same run.

Checks on the same rasters: at the largest size the epsilon surfaces are drained (a plain fill leaves them as they are,
HasDepressions is false); at --check-size (default 8192) both equal the C restatement (oracle/epsilon_fill.c) bit for bit,
the sign of a zero aside, and the reference's single-threaded CPU PriorityFloodEpsilon_Barnes2014 (oracle/_ref, where it
was built) is timed on that raster for comparison.

    python tools/epsilon_fill_timing.py [--check-size N] [--out FILE] [sizes...]   (default 16384 32768)
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from richdem_b200 import _lib  # noqa: E402

REPS = 3
SEED = 42
ND = -9999.0


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return f"{torch.cuda.get_device_name()} ({q})"


def fbm(n: int) -> torch.Tensor:
    z = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().rdb200_dev_generate_fbm_f32(z.data_ptr(), n, n, 0, SEED, 12, 0.0))
    torch.cuda.synchronize()
    return z


def entries():
    L = _lib.lib()
    return {"plain_d8": lambda p, w, h: L.rdb200_dev_fill_depressions_d8_f32(p, w, h),
            "epsilon_d8": lambda p, w, h: L.rdb200_dev_fill_depressions_epsilon_d8_f32(p, w, h, ND),
            "epsilon_d4": lambda p, w, h: L.rdb200_dev_fill_depressions_epsilon_d4_f32(p, w, h, ND)}


def timed(fn, src, work):
    work.copy_(src)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    _lib.check(fn(work.data_ptr(), work.shape[1], work.shape[0]))
    b.record()
    torch.cuda.synchronize()
    s = _lib.stats()
    return a.elapsed_time(b), int(s["fill_rounds"]), int(s["fill_tile_visits"])


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    zero = (a == 0) & (b == 0)
    return bool(torch.equal(a, b)) and bool(torch.equal(a.view(torch.int32)[~zero], b.view(torch.int32)[~zero]))


def run(n: int, check_drained: bool) -> dict:
    src = fbm(n)
    work = torch.empty_like(src)
    fns = entries()
    out = {}
    for name, fn in fns.items():  # warm-up
        timed(fn, src, work)
    runs = {name: [] for name in fns}
    for _ in range(REPS):
        for name, fn in fns.items():
            runs[name].append(timed(fn, src, work))
    for name, rs in runs.items():
        ms = float(np.median([r[0] for r in rs]))
        out[name] = {"ms": round(ms, 2), "ms_all": [round(r[0], 2) for r in rs], "mcells_per_s": round(n * n / ms / 1e3, 1),
                     "fill_rounds": rs[-1][1], "tile_visits": rs[-1][2]}
    if check_drained:
        L = _lib.lib()
        for name in ("epsilon_d8", "epsilon_d4"):
            timed(fns[name], src, work)
            again = work.clone()
            fill = L.rdb200_dev_fill_depressions_d8_f32 if name.endswith("d8") else L.rdb200_dev_fill_depressions_d4_f32
            _lib.check(fill(again.data_ptr(), n, n))
            has = C.c_int32(-1)
            has_fn = L.rdb200_dev_has_depressions_d8_f32 if name.endswith("d8") else L.rdb200_dev_has_depressions_d4_f32
            _lib.check(has_fn(work.data_ptr(), n, n, C.byref(has)))
            torch.cuda.synchronize()
            out[name]["plain_fill_leaves_it"] = bool(torch.equal(again.view(torch.int32), work.view(torch.int32)))
            out[name]["has_depressions"] = bool(has.value)
            del again
    del src, work
    torch.cuda.empty_cache()
    return out


def check_against_restatement(n: int) -> dict:
    import oracle
    from oracle import epsilon_fill as EF
    z = oracle.device_fbm(n, n, seed=SEED)
    src = torch.from_numpy(z).cuda()
    assert torch.equal(src, fbm(n)), "the CPU restatement of the generator differs from the device generator"
    work = torch.empty_like(src)
    fns = entries()
    out = {}
    for name, topo in (("epsilon_d8", "D8"), ("epsilon_d4", "D4")):
        timed(fns[name], src, work)
        t0 = time.perf_counter()
        want = torch.from_numpy(EF.port().fill(z, ND, topo)).cuda()
        out[f"restatement_{topo}_s"] = round(time.perf_counter() - t0, 1)
        out[f"{name}_equals_restatement"] = same_bits(work, want)
        if EF.have_ref():
            t0 = time.perf_counter()
            ref = EF.ref().fill(z, ND, topo)
            out[f"reference_cpu_{topo}_s"] = round(time.perf_counter() - t0, 2)
            out[f"reference_{topo}_never_below"] = bool(torch.all(torch.from_numpy(ref).cuda() >= work))
    out["reference_cpu_note"] = "reference PriorityFloodEpsilon_Barnes2014, one CPU thread (serial priority queue)"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("sizes", nargs="*", type=int, default=[16384, 32768])
    ap.add_argument("--check-size", type=int, default=8192)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    _lib.init(0)
    res = {"card": card(), "reps": REPS, "sizes": {}}
    for n in args.sizes:
        res["sizes"][str(n)] = run(n, n == max(args.sizes))
        print(json.dumps({str(n): res["sizes"][str(n)]}), flush=True)
    if args.check_size:
        res["check"] = {str(args.check_size): check_against_restatement(args.check_size)}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
