"""PitMask / HasDepressions over row bands on the GPU (sharded.pit_mask_band / sharded.has_depressions_band).  G = 2, 4
and 8 processes share the one device over gloo, with the callback communicator staging every message through host
memory; their owned mask rows and their answers must equal the single-GPU PitMask / HasDepressions of the whole raster,
for D8 and D4.  The rasters are those of test_sharded_depression_masks_emulated_gloo.py (a strict pit on a seam row, a
flat-bottomed basin across a seam, a surface without depressions, fBm with NoData blocks across seams) plus the Beauford
crop of the reference fixtures."""
import importlib.util
import multiprocessing as mp
import os
import socket

import numpy as np
import pytest

import richdem_b200 as rd

pytestmark = pytest.mark.gpu
ND = -9999.0
HERE = os.path.dirname(os.path.abspath(__file__))


def _cases():
    spec = importlib.util.spec_from_file_location("depression_band_cases",
                                                  os.path.join(HERE, "test_sharded_depression_masks_emulated_gloo.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


CASES = _cases()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, cases, out_q):
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
        for (name, topo), (dem, bounds, mask, has) in cases.items():
            h = dem.shape[0]
            r0, r1 = bounds[rank]
            gt, gb = int(rank > 0), int(rank < world - 1)
            local = torch.from_numpy(dem[r0 - gt:r1 + gb].copy()).cuda().contiguous()
            got = sharded.pit_mask_band(local, gt, gb, ND, topology=topo, row0=r0 - gt, height=h)
            ok_mask = bool(np.array_equal(got[gt:gt + r1 - r0].cpu().numpy(), mask[r0:r1]))
            got_has = sharded.has_depressions_band(local, gt, gb, topology=topo, row0=r0 - gt, height=h)
            untouched = bool(np.array_equal(local.cpu().numpy().view(np.uint32), dem[r0 - gt:r1 + gb].view(np.uint32)))
            res[(name, topo)] = (ok_mask, got_has == has, untouched)
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_bands_equal_one_gpu(world):
    g = np.load(os.path.join(HERE, "golden", "depression_masks_ref.npz"))
    rasters = CASES.rasters(world)
    beauford = np.ascontiguousarray(g["beauford__dem"])
    rasters["beauford"] = (beauford, CASES.default_bounds(beauford.shape[0], world))
    cases = {}
    for name, (dem, bounds) in rasters.items():
        for topo in ("D8", "D4"):
            src = rd.rdarray(np.ascontiguousarray(dem), no_data=ND)
            cases[(name, topo)] = (dem, bounds, np.asarray(rd.PitMask(src, topology=topo)).copy(),
                                   rd.HasDepressions(src, topology=topo))
    assert np.array_equal(cases[("beauford", "D8")][2], g["beauford__mask_D8"])
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        bad = [key for key, v in res.items() if not all(v)]
        assert not bad, (rank, bad, [res[k] for k in bad])
        assert len(res) == len(cases)
    assert all(p.exitcode == 0 for p in procs)
