"""float64 rasters over row bands on the GPU: the sharded band functions with float64 tensors (rdb200_mgpu_*_f64) on a
2048 x 2048 fBm with sub-float detail and NoData patches across the seams.  One band, and G = 2, 3 and 4 processes
sharing the one device over gloo, must give on their owned rows what richdem_b200.f64 gives on the whole raster:
FillDepressions D8 / D4 (up to the sign of a zero), PitMask, HasDepressions, ResolveFlats, every flow metric and all
eight terrain attributes bit for bit; FA_D8 / FA_D4 with unit weights bit for bit; weighted FA_D8 and D-infinity, Quinn,
Holmgren and Freeman accumulation within 1e-9 relative.  The order keys must keep the order of the values across the
bands.  With two or more GPUs the same runs over NCCL, one process per GPU."""
import multiprocessing as mp
import os
import socket

import numpy as np
import pytest

import oracle
import richdem_b200 as rd
from richdem_b200 import f64, sharded

pytestmark = pytest.mark.gpu
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


def _dem():
    z = oracle.fbm_terrain(2048, 2048, seed=91, quantum=0.25).astype(np.float64)
    rng = np.random.default_rng(4)
    z += rng.random(z.shape) * 1e-6  # sub-float detail: the keys are global ranks
    z[300:1800, 1000:1030] = ND
    z[700:1400, 200:260] = ND
    z[rng.random(z.shape) < 0.01] = ND
    return np.ascontiguousarray(z)


def _rd(a):
    return rd.rdarray(a.copy(), no_data=ND)


def _same_fill(got, want):
    return bool(np.all((got.view(np.uint64) == want.view(np.uint64)) | ((got == 0) & (want == 0))))


def _run_bands(rank, world, dev, dem, group=None):
    """Every case over this rank's band; returns {case: owned rows match the single-GPU float64 result}."""
    import torch
    h, w = dem.shape
    r0, r1, gt, gb = sharded.local_rows(h, world, rank)
    own = slice(gt, gt + r1 - r0)

    def band(a):
        t = torch.from_numpy(np.ascontiguousarray(a[r0 - gt:r1 + gb]).copy()).to(dev).contiguous()
        if gt:
            t[0] = 7.0  # garbage: no float64 driver reads the ghost rows it is handed
        if gb:
            t[-1] = float("nan")
        return t

    res = {}
    filled = {}
    for topo in ("D8", "D4"):
        want = np.asarray(f64.FillDepressions(_rd(dem), topology=topo))
        filled[topo] = want
        out, rounds = sharded.fill_band(band(dem), gt, gb, topology=topo, row0=r0 - gt, height=h, group=group)
        o = out.cpu().numpy()
        res[f"fill {topo}"] = _same_fill(o[own], want[r0:r1])
        res[f"fill {topo} ghosts"] = (not gt or _same_fill(o[0], want[r0 - 1])) and (not gb or _same_fill(o[-1], want[r1]))
    want = np.asarray(f64.PitMask(_rd(dem), topology="D8"))
    got = sharded.pit_mask_band(band(dem), gt, gb, ND, topology="D8", row0=r0 - gt, height=h, group=group)
    res["pit D8"] = bool(np.array_equal(got[own].cpu().numpy(), want[r0:r1]))
    for name, z in (("dem", dem), ("filled", filled["D8"])):
        want = f64.HasDepressions(_rd(z), topology="D8")
        res[f"hasdep {name}"] = sharded.has_depressions_band(band(z), gt, gb, topology="D8", row0=r0 - gt, height=h,
                                                             group=group) == want
    want = np.asarray(f64.ResolveFlats(_rd(filled["D8"])))
    local = band(filled["D8"])
    sharded.resolve_flats_band(local, gt, gb, ND, group=group)
    res["flats"] = bool(np.array_equal(local[own].cpu().numpy().view(np.uint64), want[r0:r1].view(np.uint64)))
    resolved = want
    for m, e in FM_CASES:
        want = np.asarray(f64.FlowProportions(_rd(resolved), m, exponent=e))
        got = sharded.flow_proportions_band(band(resolved), gt, gb, ND, m, e, group=group)[own].cpu().numpy()
        res[f"fm {m} {e}"] = bool(np.array_equal(got.view(np.uint32), want[r0:r1].view(np.uint32)))
    for attrib in ATTRIBS:
        d = _rd(dem)
        d.geotransform = [0.0, CELL[0], 0.0, 0.0, 0.0, -CELL[1]]
        want = np.asarray(f64.TerrainAttribute(d, attrib, zscale=ZSCALE))
        got = sharded.terrain_attribute_band(band(dem), gt, gb, attrib, ND, zscale=ZSCALE, cell_x=CELL[0], cell_y=CELL[1],
                                             group=group)[own].cpu().numpy()
        res[f"ta {attrib}"] = bool(np.array_equal(got.view(np.uint32), want[r0:r1].view(np.uint32)))
    wts = np.random.default_rng(17).random(dem.shape)
    for m, e, weighted in (("D8", None, False), ("D4", None, False), ("D8", None, True), ("Dinf", None, False),
                           ("Quinn", None, False), ("Holmgren", 2.5, False), ("Freeman", 1.1, True)):
        wr = rd.rdarray(wts.copy(), no_data=-1) if weighted else None
        if m in ("D8", "D4"):
            want = np.asarray(f64.FlowAccumulation(_rd(resolved), method=m, weights=wr))
        else:
            want = np.asarray(rd.FlowAccumFromProps(f64.FlowProportions(_rd(resolved), m, exponent=e), weights=wr))
        wl = torch.from_numpy(wts[r0 - gt:r1 + gb].copy()).to(dev).contiguous() if weighted else None
        acc, rounds = sharded.fa_band(band(resolved), gt, gb, ND, method=m, exponent=e, weights=wl, group=group)
        got = acc[own].cpu().numpy()
        key = f"fa {m} {e} {'weights' if weighted else 'ones'}"
        if m in ("D8", "D4") and not weighted:
            res[key] = bool(np.array_equal(got, want[r0:r1]))
        else:
            res[key] = bool(np.array_equal(got == -1, want[r0:r1] == -1) and
                            np.allclose(got, want[r0:r1], rtol=1e-9, atol=0))
        if m not in ("D8", "D4"):  # the proportions walk exchanges after every round that sent flow across a seam
            res[key + " rounds"] = world == 1 or rounds >= 2
    keys, ndk, ranked = sharded.f64_order_keys_band(band(dem), gt, gb, ND, group=group)
    res["keys ranked"] = ranked
    res["keys nodata"] = bool(ndk == keys[own][band(dem)[own] == ND][0].item())
    res["_keys"] = keys[own].cpu().numpy()
    return res


def _check_keys(dem, keys):
    v, k = dem.ravel(), keys.ravel().astype(np.float64)
    o = np.argsort(v, kind="stable")
    vs, ks = v[o], k[o]
    up = vs[1:] > vs[:-1]
    return bool(np.all(ks[1:][up] > ks[:-1][up]) and np.all(ks[1:][~up] == ks[:-1][~up]))


def _assert(results, dem):
    keys = np.concatenate([res.pop("_keys") for _, res, _ in results])
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        assert all(res.values()), (rank, {k: v for k, v in res.items() if not v})
    assert _check_keys(dem, keys)


def test_one_band_equals_single_gpu():
    dem = _dem()
    _assert([(0, _run_bands(0, 1, "cuda", dem), None)], dem)


def _worker(rank, world, port, backend, dem, out_q):
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
        out_q.put((rank, _run_bands(rank, world, f"cuda:{dev}", dem), None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _spawn(world, backend):
    dem = _dem()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, dem, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted((q.get(timeout=1500) for _ in range(world)), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
    _assert(results, dem)
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
