"""Times barnes_flat_resolution_d8 (resolved D8 directions, alter false and true) of float64 DEMs on one GPU against the
float32 path on the same raster: the fBm of rdb200_dev_generate_fbm_f32 (quantum 1, so it has flats once filled),
filled by the float32 fill, for float32; the same raster widened to double with 2^-30 relative detail on a sparse
lattice of cells (so the keys are dense ranks) for float64.  Every figure is the median of alternating repetitions
(each repetition runs every item once, in turn), timed with CUDA events around the device entry point; the input is
copied back in place before each call, outside the timed span.  The card and its power limit are printed by the same
run.

    python tools/f64_flowdirs_flats_timing.py [sizes...]   (default 16384 32768)
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


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return f"{torch.cuda.get_device_name()} ({q})"


def run(n: int) -> dict:
    L = _lib.lib()
    _lib.use_torch_stream()
    z32 = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.check(L.rdb200_dev_generate_fbm_f32(z32.data_ptr(), n, n, 0, 2024, 10, 1.0))
    _lib.check(L.rdb200_dev_fill_depressions_d8_f32(z32.data_ptr(), n, n))
    work32 = torch.empty_like(z32)
    work64 = torch.empty((n, n), dtype=torch.float64, device="cuda")
    dirs = torch.empty((n, n), dtype=torch.uint8, device="cuda")

    def prep32():
        work32.copy_(z32)

    def prep64():  # the double raster is rebuilt from the float one, so that only one copy of each is held
        work64.copy_(z32)
        lattice = work64.view(-1)[::97]
        lattice += lattice.abs() * 2.0 ** -30

    items = []
    for alter in (0, 1):
        items.append((f"f32 alter={alter}", prep32, work32, L.rdb200_dev_d8_flow_directions_flats_f32, alter))
        items.append((f"f64 alter={alter}", prep64, work64, L.rdb200_dev_d8_flow_directions_flats_f64, alter))
    times = {name: [] for name, *_ in items}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rep in range(REPS + 1):  # the first repetition warms up every item
        for name, prep, work, fn, alter in items:
            prep()
            torch.cuda.synchronize()
            ev0.record()
            _lib.check(fn(work.data_ptr(), dirs.data_ptr(), n, n, -9999.0, alter))
            ev1.record()
            torch.cuda.synchronize()
            if rep:
                times[name].append(ev0.elapsed_time(ev1))
    out = {"n": n}
    for name, t in times.items():
        out[name + " ms"] = float(np.median(t))
    for alter in (0, 1):
        out[f"f64/f32 alter={alter}"] = out[f"f64 alter={alter} ms"] / out[f"f32 alter={alter} ms"]
    del z32, work32, work64, dirs
    torch.cuda.empty_cache()
    return out


def main() -> None:
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this tool times the GPU and has no CPU fallback")
    sizes = [int(a) for a in sys.argv[1:]] or [16384, 32768]
    _lib.init(torch.cuda.current_device())
    print("card:", card())
    for n in sizes:
        print(json.dumps(run(n)))


if __name__ == "__main__":
    main()
