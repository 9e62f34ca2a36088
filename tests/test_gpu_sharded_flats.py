"""Row-band flat resolution through the C++ driver (rdb200_mgpu_resolve_flats_epsilon_f32, reached through
sharded.resolve_flats_band) on the GPU.  One band must give the single-GPU ResolveFlats bits.  G = 2, 3 and 4 processes
share the one device over gloo, with the callback communicator staging every message through host memory; their bands
must give the same bits, and their ghost rows must come back holding the neighbours' resolved edge rows, so that
fa_band can follow at once (no exchange_rows) and equal the single-GPU FlowAccumulation."""
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
    """Filled rasters: the Beauford crop (NoData around the data) and an fBm with a NoData block across the seams."""
    g = golden["beauford_crop"]
    beauford = np.ascontiguousarray(g["filled"]).astype(np.float32)
    fbm = oracle.fbm_terrain(640, 520, seed=51, quantum=0.5)
    fbm[300:330, 100:180] = ND
    fbm[150:180, 300:330] = ND
    return {"beauford": (beauford, float(g["nodata"])), "fbm": (checker.fill_depressions(fbm), ND)}


def single_gpu(dem, nodata):
    resolved = np.asarray(rd.ResolveFlats(rd.rdarray(dem.copy(), no_data=nodata)))
    acc = np.asarray(rd.FlowAccumulation(rd.rdarray(resolved.copy(), no_data=nodata), "D8"))
    return resolved, acc


def test_world_one_equals_resolve_flats(checker, golden):
    import torch
    for name, (dem, nodata) in _rasters(checker, golden).items():
        expected, _ = single_gpu(dem, nodata)
        assert (expected != dem).any(), name
        t = torch.from_numpy(dem.copy()).cuda().contiguous()
        assert sharded.resolve_flats_band(t, 0, 0, nodata) == 0
        got = t.cpu().numpy()
        assert np.array_equal(got.view(np.uint32), expected.view(np.uint32)), \
            f"{name}: {(got.view(np.uint32) != expected.view(np.uint32)).sum()} cells differ"


def _worker(rank, world, port, dems, expected, out_q):
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
            local = torch.from_numpy(np.ascontiguousarray(dem[r0 - gt:r1 + gb])).cuda().contiguous()
            iters = sharded.resolve_flats_band(local, gt, gb, nodata)
            got = local.cpu().numpy().view(np.uint32)
            x = expected[name][0].view(np.uint32)
            owned = bool(np.array_equal(got[gt:gt + (r1 - r0)], x[r0:r1]))
            ghosts = bool((not gt or np.array_equal(got[0], x[r0 - 1])) and (not gb or np.array_equal(got[-1], x[r1])))
            acc, _ = sharded.fa_band(local, gt, gb, nodata, method="D8")
            fa = bool(np.array_equal(acc[gt:gt + (r1 - r0)].cpu().numpy(), expected[name][1][r0:r1]))
            res[name] = {"owned": owned, "ghosts": ghosts, "fa_d8": fa, "iters": iters}
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_processes_over_gloo_equal_one_gpu(checker, golden, world):
    dems = _rasters(checker, golden)
    expected = {name: single_gpu(dem, nodata) for name, (dem, nodata) in dems.items()}
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, dems, expected, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        for name, r in res.items():
            assert r["owned"] and r["ghosts"] and r["fa_d8"], (rank, name, r)
            assert r["iters"] >= 2, (rank, name, r)
    assert all(p.exitcode == 0 for p in procs)
