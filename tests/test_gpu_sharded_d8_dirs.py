"""The direction-grid pipeline over row bands on the GPU: sharded.d8_flow_directions_band (rdb200_mgpu_d8_flow_directions_
flats_f32) and sharded.d8_flow_accum_band (rdb200_mgpu_d8_flow_accum_u8_i32).  One band must give the single-GPU
FlowDirectionsD8Resolved / D8FlowAccum bits.  G = 2, 3 and 4 processes share the one device over gloo, with the callback
communicator staging every message through host memory; their owned rows must give the same bits, and so must the chain
fill_band -> d8_flow_directions_band -> d8_flow_accum_band against FillDepressions -> FlowDirectionsD8Resolved ->
D8FlowAccum."""
import multiprocessing as mp
import os
import socket

import numpy as np
import pytest

import oracle
import richdem_b200 as rd
from richdem_b200 import sharded

pytestmark = pytest.mark.gpu
ND = -9999.0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rasters(checker, golden):
    """Filled rasters: the Beauford crop (NoData around the data) and a quantised fBm with NoData blocks across the
    seams (an odd width, so the accumulation takes its unpacked path); plus an unfilled quantised fBm for the chain."""
    g = golden["beauford_crop"]
    beauford = np.ascontiguousarray(g["filled"]).astype(np.float32)
    fbm = oracle.fbm_terrain(640, 521, seed=53, quantum=0.5)
    fbm[300:330, 100:180] = ND
    fbm[150:180, 300:330] = ND
    chain = oracle.fbm_terrain(512, 640, seed=54, quantum=0.5)
    return {"beauford": (beauford, float(g["nodata"])), "fbm": (checker.fill_depressions(fbm), ND)}, chain


def single_gpu(dem, nodata):
    out = {}
    for alter in (False, True):
        d = rd.rdarray(dem.copy(), no_data=nodata)
        dirs = np.asarray(rd.FlowDirectionsD8Resolved(d, alter=alter))
        out[alter] = (dirs, np.asarray(d).copy(), np.asarray(rd.D8FlowAccum(dirs)))
    return out


def single_gpu_chain(dem):
    filled = rd.FillDepressions(rd.rdarray(dem.copy(), no_data=ND))
    dirs = np.asarray(rd.FlowDirectionsD8Resolved(rd.rdarray(np.asarray(filled).copy(), no_data=ND)))
    return dirs, np.asarray(rd.D8FlowAccum(dirs))


def test_world_one_equals_single_gpu(checker, golden):
    import torch
    dems, _ = _rasters(checker, golden)
    for name, (dem, nodata) in dems.items():
        expected = single_gpu(dem, nodata)
        assert (expected[False][0] != rd.FlowDirectionsD8(rd.rdarray(dem.copy(), no_data=nodata))).any(), name
        for alter in (False, True):
            t = torch.from_numpy(dem.copy()).cuda().contiguous()
            dirs, it = sharded.d8_flow_directions_band(t, 0, 0, nodata, alter=alter)
            assert it == 0
            assert np.array_equal(dirs.cpu().numpy(), expected[alter][0]), (name, alter)
            assert np.array_equal(t.cpu().numpy().view(np.uint32), expected[alter][1].view(np.uint32)), (name, alter)
            area, rounds = sharded.d8_flow_accum_band(dirs, 0, 0)
            assert rounds == 1
            assert np.array_equal(area.cpu().numpy(), expected[alter][2]), (name, alter)


def _worker(rank, world, port, dems, expected, chain_dem, chain_expected, out_q):
    import torch
    import torch.distributed as dist
    from richdem_b200 import _lib, sharded

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        torch.cuda.set_device(0)
        _lib.init(0)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        res = {}
        for name, (dem, nodata) in dems.items():
            h, w = dem.shape
            r0, r1, gt, gb = sharded.local_rows(h, world, rank)
            for alter in (False, True):
                x_dirs, x_dem, x_area = expected[name][alter]
                local = torch.from_numpy(np.ascontiguousarray(dem[r0 - gt:r1 + gb])).cuda().contiguous()
                dirs, iters = sharded.d8_flow_directions_band(local, gt, gb, nodata, alter=alter)
                d = dirs.cpu().numpy()
                z = local.cpu().numpy().view(np.uint32)
                area, rounds = sharded.d8_flow_accum_band(dirs, gt, gb)
                res[(name, alter)] = {
                    "dirs": bool(np.array_equal(d[gt:gt + r1 - r0], x_dirs[r0:r1])),
                    "dir_ghosts": bool((not gt or np.array_equal(d[0], x_dirs[r0 - 1])) and
                                       (not gb or np.array_equal(d[-1], x_dirs[r1]))),
                    "dem": bool(np.array_equal(z[gt:gt + r1 - r0], x_dem.view(np.uint32)[r0:r1])),
                    "area": bool(np.array_equal(area[gt:gt + r1 - r0].cpu().numpy(), x_area[r0:r1])),
                    "iters": iters, "rounds": rounds}
        h, w = chain_dem.shape
        r0, r1, gt, gb = sharded.local_rows(h, world, rank)
        local = torch.from_numpy(np.ascontiguousarray(chain_dem[r0 - gt:r1 + gb])).cuda().contiguous()
        sharded.fill_band(local, gt, gb)
        dirs, _ = sharded.d8_flow_directions_band(local, gt, gb, ND)
        area, _ = sharded.d8_flow_accum_band(dirs, gt, gb)
        res["chain"] = {"dirs": bool(np.array_equal(dirs[gt:gt + r1 - r0].cpu().numpy(), chain_expected[0][r0:r1])),
                        "area": bool(np.array_equal(area[gt:gt + r1 - r0].cpu().numpy(), chain_expected[1][r0:r1]))}
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_processes_over_gloo_equal_one_gpu(checker, golden, world):
    dems, chain_dem = _rasters(checker, golden)
    expected = {name: single_gpu(dem, nodata) for name, (dem, nodata) in dems.items()}
    chain_expected = single_gpu_chain(chain_dem)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, dems, expected, chain_dem, chain_expected, q))
             for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        chain = res.pop("chain")
        assert chain["dirs"] and chain["area"], (rank, chain)
        for key, r in res.items():
            assert r["dirs"] and r["dir_ghosts"] and r["dem"] and r["area"], (rank, key, r)
            assert r["iters"] >= 2 and r["rounds"] >= 2, (rank, key, r)
    assert all(p.exitcode == 0 for p in procs)
