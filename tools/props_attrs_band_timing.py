"""Flow proportions, accumulation from given proportions and one terrain attribute on bench.py's fBm raster (filled),
timed with CUDA events, alternating: the row-band drivers with one band (sharded.flow_proportions_band ->
rdb200_mgpu_fm_method_f32, sharded.flow_accum_from_props_band -> rdb200_mgpu_flow_accumulation_props_f64 and
sharded.terrain_attribute_band -> rdb200_mgpu_terrain_attribute_f32, world 1) and the single-GPU calls
(rdb200_dev_fm_method_f32, rdb200_dev_flow_accumulation_props_f64, rdb200_dev_terrain_attribute_f32).  Everything is
device-resident; both accumulations read the same proportions and start from unit weights written inside the timed
window.  This measures what the band machinery costs on one GPU, not a multi-GPU speed-up.
    python tools/props_attrs_band_timing.py 16384 [--method Quinn] [--attrib curvature] [--reps 5] [--out result.json]
Prints the card name and power limit with the times, whether the proportions and attributes are the same bits, and the
accumulations' largest relative difference."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("n", type=int)
ap.add_argument("--method", default="Quinn")
ap.add_argument("--exponent", type=float, default=None)
ap.add_argument("--attrib", default="curvature")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--out")
args = ap.parse_args()
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from richdem_b200 import _TERRAIN_ATTRIBS, _lib, sharded  # noqa: E402

ND = -9999.0
N = args.n
L = _lib.lib()
_lib.init(0)
_lib.use_torch_stream()
mid, xparam = sharded._method_id(args.method, args.exponent, "FlowProportions")
dem = torch.empty((N, N), dtype=torch.float32, device="cuda")
_lib.check(L.rdb200_dev_generate_fbm_f32(dem.data_ptr(), N, N, 0, 42, 12, 0.0))
_lib.check(L.rdb200_dev_fill_depressions_d8_f32(dem.data_ptr(), N, N))
props = torch.empty((N, N, 9), dtype=torch.float32, device="cuda")
acc = torch.empty((N, N), dtype=torch.float64, device="cuda")
attr = torch.empty((N, N), dtype=torch.float32, device="cuda")
out = {}


def fm_band():
    out["props"] = sharded.flow_proportions_band(dem, 0, 0, ND, args.method, args.exponent)


def fm_single():
    _lib.check(L.rdb200_dev_fm_method_f32(mid, dem.data_ptr(), props.data_ptr(), N, N, ND, xparam))
    out["props"] = props


def fa_band():
    acc.fill_(1.0)
    out["acc"], _ = sharded.flow_accum_from_props_band(out["props"], 0, 0, weights=acc)


def fa_single():
    acc.fill_(1.0)
    _lib.check(L.rdb200_dev_flow_accumulation_props_f64(out["props"].data_ptr(), acc.data_ptr(), N, N))
    out["acc"] = acc


def ta_band():
    out["attr"] = sharded.terrain_attribute_band(dem, 0, 0, args.attrib, ND)


def ta_single():
    _lib.check(L.rdb200_dev_terrain_attribute_f32(_TERRAIN_ATTRIBS[args.attrib], dem.data_ptr(), attr.data_ptr(), N, N, ND,
                                                  -9999.0, 1.0, 1.0, 1.0))
    out["attr"] = attr


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


# warm-up, and the results compared below
timed(fm_band)
r_props = out["props"]
timed(fa_band)
r_acc = out["acc"].clone()
timed(ta_band)
r_attr = out["attr"]
timed(fm_single)
timed(fa_single)
timed(ta_single)
same_bits = {"props": bool(torch.equal(r_props.view(torch.int32), props.view(torch.int32))),
             "attr": bool(torch.equal(r_attr.view(torch.int32), attr.view(torch.int32)))}
data = acc > 0
acc_rel = float(((r_acc - acc).abs()[data] / acc[data]).max().item())
nodata_same = bool(torch.equal(r_acc == -1, acc == -1))
del r_props, r_acc, r_attr
out.clear()
times = {k: [] for k in ("fm_band_world1", "fm_single_gpu", "fa_band_world1", "fa_single_gpu", "ta_band_world1",
                         "ta_single_gpu")}
for _ in range(args.reps):
    times["fm_band_world1"].append(timed(fm_band))
    times["fa_band_world1"].append(timed(fa_band))
    out.clear()
    times["fm_single_gpu"].append(timed(fm_single))
    times["fa_single_gpu"].append(timed(fa_single))
    times["ta_band_world1"].append(timed(ta_band))
    out.clear()
    times["ta_single_gpu"].append(timed(ta_single))
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
result = {"n": N, "reps": args.reps, "method": args.method, "exponent": args.exponent, "attrib": args.attrib,
          "gpu": torch.cuda.get_device_name(0),
          "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unavailable",
          "same_bits": same_bits, "accum_max_rel_diff": acc_rel, "accum_nodata_same": nodata_same,
          "ms": {k: [round(t, 3) for t in v] for k, v in times.items()},
          "median_ms": {k: round(statistics.median(v), 3) for k, v in times.items()}}
print(json.dumps(result), flush=True)
if args.out:
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
