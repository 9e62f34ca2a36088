"""Flow proportions, accumulation from given proportions and terrain attributes over row bands on the GPU:
sharded.flow_proportions_band (rdb200_mgpu_fm_method_f32), sharded.flow_accum_from_props_band
(rdb200_mgpu_flow_accumulation_props_f64) and sharded.terrain_attribute_band (rdb200_mgpu_terrain_attribute_f32), on a
2048 x 2048 quantised fBm with NoData patches across the seams.  One band, and G = 2, 3 and 4 processes sharing the one
device over gloo, must give on their owned rows what FlowProportions / TerrainAttribute give on the whole raster, bit for
bit, and what FlowAccumFromProps gives: bit for bit for one-hot proportions with unit weights, within 1e-9 relative
otherwise.  Hand-made proportions send flow across the seams into NoData and out of the raster's edge cells.  With two or
more GPUs the same runs over NCCL, one process per GPU."""
import importlib.util
import multiprocessing as mp
import os
import socket

import numpy as np
import pytest

import oracle
import richdem_b200 as rd
from richdem_b200 import sharded

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0
FM_CASES = [("D8", None), ("Dinf", None), ("D4", None), ("Quinn", None), ("Holmgren", 2.5), ("Freeman", 1.1)]
ATTRIBS = ["slope_riserun", "slope_percentage", "slope_degrees", "slope_radians", "aspect", "curvature",
           "planform_curvature", "profile_curvature"]
ZSCALE, CELL = 2.5, (30.0, 20.0)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _handmade_props(h, w, seed, one_hot):
    path = os.path.join(HERE, "test_sharded_props_attrs_emulated_gloo.py")
    spec = importlib.util.spec_from_file_location("props_attrs_emulated", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.handmade_props(h, w, seed, one_hot)


def _inputs():
    dem = oracle.fbm_terrain(2048, 2048, seed=81, quantum=0.25)
    dem[300:1800, 1000:1030] = ND
    dem[700:1400, 200:260] = ND
    dem[np.random.default_rng(2).random(dem.shape) < 0.01] = ND
    hand = {one_hot: _handmade_props(160, 150, 3, one_hot) for one_hot in (True, False)}
    return np.ascontiguousarray(dem), hand


def _single_gpu_props(dem, m, e):
    return np.asarray(rd.FlowProportions(rd.rdarray(dem, no_data=ND), m, exponent=e))


def _single_gpu_attr(dem, attrib):
    d = rd.rdarray(dem, no_data=ND)
    d.geotransform = [0.0, CELL[0], 0.0, 0.0, 0.0, -CELL[1]]
    return np.asarray(rd.TerrainAttribute(d, attrib, zscale=ZSCALE))


def _single_gpu_accum(props, weights):
    wr = None if weights is None else rd.rdarray(weights.copy(), no_data=-1)
    return np.asarray(rd.FlowAccumFromProps(rd.rd3array(props, no_data=-2), weights=wr))


def _same_accum(got, want, exact):
    if exact:
        return bool(np.array_equal(got, want))
    return bool(np.array_equal(got == -1, want == -1) and np.allclose(got, want, rtol=1e-9, atol=0))


def _run_bands(rank, world, dev, dem, hand, group=None):
    """Every case over this rank's band; returns {case: owned rows match the single-GPU result}."""
    import torch
    h, w = dem.shape
    r0, r1, gt, gb = sharded.local_rows(h, world, rank)
    own = slice(gt, gt + r1 - r0)

    def band(a):
        t = torch.from_numpy(np.ascontiguousarray(a[r0 - gt:r1 + gb]).copy()).to(dev).contiguous()
        if gt:
            t[0] = 7.0  # garbage: the calls refresh the ghost rows themselves
        if gb:
            t[-1] = 0.5
        return t

    res = {}
    rng = np.random.default_rng(17)
    wts = rng.random(dem.shape)
    for m, e in FM_CASES:
        want = _single_gpu_props(dem, m, e)
        local = band(dem)
        got = sharded.flow_proportions_band(local, gt, gb, ND, m, e, group=group)[own].cpu().numpy()
        res[f"fm {m} {e}"] = bool(np.array_equal(got.view(np.uint32), want[r0:r1].view(np.uint32)))
        res[f"fm {m} {e} dem ghosts"] = bool((not gt or np.array_equal(local[0].cpu().numpy(), dem[r0 - 1])) and
                                             (not gb or np.array_equal(local[-1].cpu().numpy(), dem[r1])))
        exact = m in ("D8", "D4")
        for weights in ((None, wts) if m in ("D8", "Dinf", "Holmgren") else (None,)):
            acc_want = _single_gpu_accum(want, weights)
            wl = None if weights is None else torch.from_numpy(weights[r0 - gt:r1 + gb].copy()).to(dev).contiguous()
            acc, rounds = sharded.flow_accum_from_props_band(band(want), gt, gb, weights=wl, group=group)
            key = f"fa {m} {e} {'ones' if weights is None else 'weights'}"
            res[key] = _same_accum(acc[own].cpu().numpy(), acc_want[r0:r1], exact and weights is None)
            res[key + " rounds"] = world == 1 or rounds >= 2
    for attrib in ATTRIBS:
        want = _single_gpu_attr(dem, attrib)
        got = sharded.terrain_attribute_band(band(dem), gt, gb, attrib, ND, zscale=ZSCALE, cell_x=CELL[0], cell_y=CELL[1],
                                             group=group)[own].cpu().numpy()
        res[f"ta {attrib}"] = bool(np.array_equal(got.view(np.uint32), want[r0:r1].view(np.uint32)))
    for one_hot, p in hand.items():
        hh = p.shape[0]
        q0, q1, qt, qb = sharded.local_rows(hh, world, rank)
        for weights in (None, np.random.default_rng(3).random(p.shape[:2])):
            acc_want = _single_gpu_accum(p, weights)
            lp = torch.from_numpy(p[q0 - qt:q1 + qb].copy()).to(dev).contiguous()
            if qt:
                lp[0] = 7.0
            wl = None if weights is None else torch.from_numpy(weights[q0 - qt:q1 + qb].copy()).to(dev).contiguous()
            acc, _ = sharded.flow_accum_from_props_band(lp, qt, qb, weights=wl, group=group)
            res[f"hand {one_hot} {weights is None}"] = _same_accum(acc[qt:qt + q1 - q0].cpu().numpy(), acc_want[q0:q1],
                                                                   one_hot and weights is None)
    return res


def test_one_band_equals_single_gpu():
    dem, hand = _inputs()
    res = _run_bands(0, 1, "cuda", dem, hand)
    assert all(res.values()), {k: v for k, v in res.items() if not v}


def _worker(rank, world, port, backend, dem, hand, out_q):
    import torch
    import torch.distributed as dist
    from richdem_b200 import _lib

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        dev = rank if backend == "nccl" else 0
        torch.cuda.set_device(dev)
        _lib.init(dev)
        dist.init_process_group(backend, rank=rank, world_size=world)
        out_q.put((rank, _run_bands(rank, world, f"cuda:{dev}", dem, hand), None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _spawn(world, backend):
    dem, hand = _inputs()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, dem, hand, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=900) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        assert all(res.values()), (rank, {k: v for k, v in res.items() if not v})
    assert all(p.exitcode == 0 for p in procs)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_processes_over_gloo_equal_one_gpu(world):
    _spawn(world, "gloo")


def test_processes_over_nccl_equal_one_gpu():
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip(f"NCCL bands need two or more GPUs ({n} visible)")
    _spawn(min(n, 4), "nccl")
