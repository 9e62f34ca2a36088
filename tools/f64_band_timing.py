"""float64 row bands, timed stage by stage: the order keys kappa_G (sharded.f64_order_keys_band), FillDepressions D8,
ResolveFlats, FA_D8 (unit weights), FM_Quinn and TA_slope_degrees through the sharded band functions with float64
tensors, on an N x N fBm with sub-float detail (so the keys take the global-rank route).  G processes, each with its own
band: over gloo on one device (--gpus 1, the default), or over NCCL with one process per GPU (--gpus G).
    python tools/f64_band_timing.py 8192 --world 2 [--gpus 2] [--reps 3] [--out result.json]
Each stage starts after a barrier and is timed with CUDA events on every rank; the JSON line gives, per stage, the
slowest rank's time of every repetition and their median, with the card name and power limit."""
import argparse
import json
import multiprocessing as mp
import os
import socket
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ND = -9999.0
STAGES = ("keys", "fill_d8", "resolve_flats", "fa_d8", "fm_quinn", "ta_slope_degrees")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, gpus, port, n, reps, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from richdem_b200 import _lib, sharded
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank if gpus > 1 else 0
    torch.cuda.set_device(dev)
    _lib.init(dev)
    dist.init_process_group("nccl" if gpus > 1 else "gloo", rank=rank, world_size=world)
    L = _lib.lib()
    _lib.use_torch_stream()
    r0, r1, gt, gb = sharded.local_rows(n, world, rank)
    h = r1 - r0 + gt + gb
    f = torch.empty((h, n), dtype=torch.float32, device="cuda")
    _lib.check(L.rdb200_dev_generate_fbm_f32(f.data_ptr(), n, h, r0 - gt, 42, 12, 0.0))
    idx = torch.arange((r0 - gt) * n, (r0 - gt + h) * n, dtype=torch.int64, device="cuda").view(h, n)
    dem = f.double() + ((idx * 2654435761) % 4096).double() * 2.0 ** -40  # sub-float detail, the same in every band count

    def stages():
        out = {}
        z = dem.clone()
        out["keys"] = lambda: sharded.f64_order_keys_band(z, gt, gb, ND)
        out["fill_d8"] = lambda: sharded.fill_band(z, gt, gb, row0=r0 - gt, height=n)
        out["resolve_flats"] = lambda: sharded.resolve_flats_band(z, gt, gb, ND)
        out["fa_d8"] = lambda: sharded.fa_band(z, gt, gb, ND, method="D8")
        out["fm_quinn"] = lambda: sharded.flow_proportions_band(z, gt, gb, ND, "Quinn")
        out["ta_slope_degrees"] = lambda: sharded.terrain_attribute_band(z, gt, gb, "slope_degrees", ND)
        return out

    times = {s: [] for s in STAGES}
    for rep in range(reps + 1):  # the first repetition warms up
        for name, fn in stages().items():
            dist.barrier()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            t = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float32, device="cuda" if gpus > 1 else "cpu")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            if rep:
                times[name].append(float(t.item()))
    if rank == 0:
        q.put(times)
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("n", type=int)
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    if args.gpus not in (1, args.world):
        raise SystemExit("--gpus is 1 (every band on one device) or the band count (one band per GPU)")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, args.world, args.gpus, port, args.n, args.reps, q)) for r in range(args.world)]
    for p in procs:
        p.start()
    times = q.get(timeout=3600)
    for p in procs:
        p.join(timeout=120)
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    result = {"n": args.n, "world": args.world, "gpus": args.gpus, "reps": args.reps, "gpu": torch.cuda.get_device_name(0),
              "nvidia_smi": smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else "unavailable",
              "ms": {k: [round(t, 3) for t in v] for k, v in times.items()},
              "median_ms": {k: round(statistics.median(v), 3) for k, v in times.items()}}
    print(json.dumps(result), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
