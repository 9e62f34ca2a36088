"""Multi-GPU check (run under torchrun on N GPUs): sharded fill + FA_D8 / FA_Dinf over NCCL must
equal the single-GPU answer computed on rank 0.  Writes gpurun_out/mgpu_check_<N>.json."""
# Also checked: flat resolution, the direction pipeline on the filled raster (resolved D8 directions, d8_flow_accum), and
# the D4 chain: fill_band(topology="D4") -> resolve_flats_band -> fa_band(method="D4") against FillDepressions<D4> ->
# ResolveFlats -> FA_D4 on one GPU (fill and flats bit for bit, the accumulation to 1e-9 relative).
import json, os, sys, time
import numpy as np
import torch
import torch.distributed as dist
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from richdem_b200 import _lib, sharded

MG = int(os.environ.get("RDB_BAND_MULTIGRID", "0"))  # k >= 2: multigrid start of the band fill (fill_band(..., multigrid=k))
VC = int(os.environ.get("RDB_BAND_VCYCLE", "0"))     # n > 0: coarse-grid correction after every n halo exchanges

rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
_lib.init(lr)
_lib.use_torch_stream()
L = _lib.lib()
ND = -9999.0
res = {"world": world, "cases": []}
for (H, W, q) in [(3000, 2000, 0.5), (8192, 8192, 0.0)]:
    r0, r1, gt, gb = sharded.local_rows(H, world, rank)
    hloc = r1 - r0 + gt + gb
    loc = torch.empty((hloc, W), dtype=torch.float32, device="cuda")
    _lib.check(L.rdb200_dev_generate_fbm_f32(loc.data_ptr(), W, hloc, r0 - gt, 7, 12, q))
    torch.cuda.synchronize(); dist.barrier(); t = time.time()
    filled, frounds = sharded.fill_band(loc.clone(), gt, gb, multigrid=MG, row0=r0 - gt, height=H, vcycle=VC)
    torch.cuda.synchronize(); dist.barrier(); tf = time.time() - t; t = time.time()
    own_f = filled[gt:gt + (r1 - r0)].clone()
    filled_band = filled.clone()
    # flat resolution over bands (in place), then refresh the ghost rows with the neighbours' resolved rows
    seam_iters = sharded.resolve_flats_band(filled, gt, gb, ND)
    sharded.exchange_rows(filled, gt, gb)
    torch.cuda.synchronize(); dist.barrier(); tz = time.time() - t; t = time.time()
    own_r = filled[gt:gt + (r1 - r0)].clone()
    acc, arounds = sharded.fa_band(filled, gt, gb, ND, dinf=False)
    torch.cuda.synchronize(); dist.barrier(); ta = time.time() - t; t = time.time()
    accinf, irounds = sharded.fa_band(filled, gt, gb, ND, dinf=True)
    torch.cuda.synchronize(); dist.barrier(); ti = time.time() - t; t = time.time()
    # the direction-grid pipeline on the filled band (its ghost rows hold the neighbours' filled rows)
    dirs, dseam = sharded.d8_flow_directions_band(filled_band, gt, gb, ND)
    area, drounds = sharded.d8_flow_accum_band(dirs, gt, gb)
    torch.cuda.synchronize(); dist.barrier(); td = time.time() - t
    own_d = dirs[gt:gt + (r1 - r0)].contiguous()
    own_ar = area[gt:gt + (r1 - r0)].contiguous()
    # single-GPU truth on rank 0
    own_a = acc[gt:gt + (r1 - r0)].contiguous()
    own_i = accinf[gt:gt + (r1 - r0)].contiguous()
    if rank == 0:
        full = torch.empty((H, W), dtype=torch.float32, device="cuda")
        _lib.check(L.rdb200_dev_generate_fbm_f32(full.data_ptr(), W, H, 0, 7, 12, q))
        _lib.check(L.rdb200_dev_fill_depressions_d8_f32(full.data_ptr(), W, H))
        full_filled = full.clone()
        d1, z1 = torch.empty((H, W), dtype=torch.uint8, device="cuda"), full_filled.clone()
        _lib.check(L.rdb200_dev_d8_flow_directions_flats_f32(z1.data_ptr(), d1.data_ptr(), W, H, ND, 0))
        del z1
        ar1 = torch.empty((H, W), dtype=torch.int32, device="cuda")
        _lib.check(L.rdb200_dev_d8_flow_accum_u8_i32(d1.data_ptr(), ar1.data_ptr(), W, H))
        _lib.check(L.rdb200_dev_resolve_flats_epsilon_f32(full.data_ptr(), W, H, ND))
        a1 = torch.empty((H, W), dtype=torch.float64, device="cuda")
        _lib.check(L.rdb200_dev_fa_d8_f32_f64(full.data_ptr(), a1.data_ptr(), W, H, ND, 1))
        a2 = torch.empty((H, W), dtype=torch.float64, device="cuda")
        _lib.check(L.rdb200_dev_fa_tarboton_f32_f64(full.data_ptr(), a2.data_ptr(), W, H, ND, 1))
    ok = {}
    for name, own, dtype in (("fill", own_f, torch.float32), ("flats", own_r, torch.float32), ("fa_d8", own_a, torch.float64),
                             ("fa_dinf", own_i, torch.float64), ("d8_dirs", own_d, torch.uint8), ("d8_area", own_ar, torch.int32)):
        if rank == 0:
            ref = {"fill": full_filled, "flats": full, "fa_d8": a1, "fa_dinf": a2, "d8_dirs": d1, "d8_area": ar1}[name]
            good = True
            for g in range(world):
                b0, b1, _, _ = sharded.local_rows(H, world, g)
                if g == 0:
                    part = own
                else:
                    part = torch.empty((b1 - b0, W), dtype=dtype, device="cuda")
                    dist.recv(part, g)
                if name == "fa_dinf":
                    good &= bool(torch.allclose(part, ref[b0:b1], rtol=5e-7, atol=0))
                else:
                    good &= bool(torch.equal(part, ref[b0:b1]))
            ok[name] = good
        else:
            dist.send(own, 0)
    if rank == 0:
        case = {"H": H, "W": W, "q": q, "ok": ok, "fill_s": tf, "flats_s": tz, "flats_seam_iters": seam_iters, "fa_d8_s": ta, "fa_dinf_s": ti,
                "fill_exchange_rounds": frounds, "fa_d8_rounds": arounds, "fa_dinf_rounds": irounds,
                "d8_dirs_accum_s": td, "d8_dirs_seam_iters": dseam, "d8_accum_rounds": drounds}
        print(json.dumps(case), flush=True)
        res["cases"].append(case)
res["d4_cases"] = []
for (H, W, q) in [(3000, 2000, 0.5), (8192, 8192, 0.0)]:
    r0, r1, gt, gb = sharded.local_rows(H, world, rank)
    hloc = r1 - r0 + gt + gb
    loc = torch.empty((hloc, W), dtype=torch.float32, device="cuda")
    _lib.check(L.rdb200_dev_generate_fbm_f32(loc.data_ptr(), W, hloc, r0 - gt, 7, 12, q))
    torch.cuda.synchronize(); dist.barrier(); t = time.time()
    _, frounds = sharded.fill_band(loc, gt, gb, row0=r0 - gt, height=H, topology="D4")
    torch.cuda.synchronize(); dist.barrier(); tf = time.time() - t; t = time.time()
    own_f = loc[gt:gt + (r1 - r0)].clone()
    seam_iters = sharded.resolve_flats_band(loc, gt, gb, ND)
    torch.cuda.synchronize(); dist.barrier(); tz = time.time() - t; t = time.time()
    own_r = loc[gt:gt + (r1 - r0)].clone()
    acc, arounds = sharded.fa_band(loc, gt, gb, ND, method="D4")
    torch.cuda.synchronize(); dist.barrier(); ta = time.time() - t
    own_a = acc[gt:gt + (r1 - r0)].contiguous()
    if rank == 0:
        full = torch.empty((H, W), dtype=torch.float32, device="cuda")
        _lib.check(L.rdb200_dev_generate_fbm_f32(full.data_ptr(), W, H, 0, 7, 12, q))
        _lib.check(L.rdb200_dev_fill_depressions_d4_f32(full.data_ptr(), W, H))
        full_filled = full.clone()
        _lib.check(L.rdb200_dev_resolve_flats_epsilon_f32(full.data_ptr(), W, H, ND))
        a1 = torch.ones((H, W), dtype=torch.float64, device="cuda")
        _lib.check(L.rdb200_dev_fa_method_f32_f64(2, full.data_ptr(), a1.data_ptr(), W, H, ND, 0.0))  # 2: FA_D4
    ok = {}
    for name, own, dtype in (("fill_d4", own_f, torch.float32), ("flats", own_r, torch.float32), ("fa_d4", own_a, torch.float64)):
        if rank == 0:
            ref = {"fill_d4": full_filled, "flats": full, "fa_d4": a1}[name]
            good = True
            for g in range(world):
                b0, b1, _, _ = sharded.local_rows(H, world, g)
                if g == 0:
                    part = own
                else:
                    part = torch.empty((b1 - b0, W), dtype=dtype, device="cuda")
                    dist.recv(part, g)
                if name == "fa_d4":
                    good &= bool(torch.allclose(part, ref[b0:b1], rtol=1e-9, atol=0))
                else:
                    good &= bool(torch.equal(part.view(torch.int32), ref[b0:b1].view(torch.int32)))
            ok[name] = good
        else:
            dist.send(own, 0)
    if rank == 0:
        case = {"H": H, "W": W, "q": q, "ok": ok, "fill_d4_s": tf, "flats_s": tz, "flats_seam_iters": seam_iters,
                "fa_d4_s": ta, "fill_exchange_rounds": frounds, "fa_d4_rounds": arounds}
        print(json.dumps(case), flush=True)
        res["d4_cases"].append(case)
if rank == 0:
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(res, open(f"gpurun_out/mgpu_check_{world}.json", "w"), indent=1)
dist.destroy_process_group()
