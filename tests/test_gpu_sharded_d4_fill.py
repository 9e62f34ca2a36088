"""The D4 fill over row bands on the GPU: sharded.fill_band(topology="D4") (rdb200_mgpu_fill_depressions_d4_f32).  One
band must give the single-GPU rdb200_dev_fill_depressions_d4_f32 bits.  G = 2, 3 and 4 processes share the one device
over gloo, with the callback communicator staging every message through host memory; their owned rows must give the
same bits, and the chain fill_band(topology="D4") -> resolve_flats_band -> fa_band(method="D4") must match
FillDepressions(topology="D4") -> ResolveFlats -> FlowAccumulation(method="D4").  The rasters are those of
test_sharded_d4_fill_emulated_gloo.py (seams through NoData blocks, an odd width, ghost rows on a tile edge, a band of
one row, a diagonal wall with its one D8 gap on a seam, a checkerboard of pooling blocks) plus the Beauford crop."""
import contextlib
import importlib.util
import multiprocessing as mp
import os
import socket

import numpy as np
import pytest

import oracle
import richdem_b200 as rd
from richdem_b200 import _lib, sharded

pytestmark = pytest.mark.gpu
ND = -9999.0
HERE = os.path.dirname(os.path.abspath(__file__))
FA_RTOL = 1e-9  # FA_D4 over bands sums the same unit flows in another order


def _cases():
    spec = importlib.util.spec_from_file_location("d4_fill_cases", os.path.join(HERE, "test_sharded_d4_fill_emulated_gloo.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


CASES = _cases()


@contextlib.contextmanager
def switches(name):
    """A switch set of the emulated test, with coarse levels allowed down to 16 cells; shipped defaults afterwards."""
    try:
        _lib.set_param("fill_multigrid_min", 16)
        for k, v in CASES.SWITCHES[name].items():
            _lib.set_param(k, v)
        yield
    finally:
        _lib.reset_params()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def single_gpu_d4(dem):
    import torch
    t = torch.from_numpy(dem.copy()).cuda().contiguous()
    _lib.use_torch_stream()
    _lib.check(_lib.lib().rdb200_dev_fill_depressions_d4_f32(t.data_ptr(), dem.shape[1], dem.shape[0]))
    return t.cpu().numpy()


def single_gpu_chain(dem):
    filled = np.asarray(rd.FillDepressions(rd.rdarray(dem.copy(), no_data=ND), topology="D4")).copy()
    resolved = np.asarray(rd.ResolveFlats(rd.rdarray(filled.copy(), no_data=ND))).copy()
    acc = np.asarray(rd.FlowAccumulation(rd.rdarray(resolved.copy(), no_data=ND), method="D4")).copy()
    return filled, resolved, acc


def test_world_one_equals_single_gpu(checker, golden):
    import torch
    g = golden["beauford_crop"]
    for sw in CASES.SWITCHES:
        dems = {name: dem for name, (dem, _) in CASES.rasters(1, CASES.SWITCHES[sw]).items()}
        dems["beauford"] = np.ascontiguousarray(g["dem"]).astype(np.float32)
        with switches(sw):
            for name, dem in dems.items():
                expected = single_gpu_d4(dem)
                assert np.array_equal(expected.view(np.uint32), checker.fill_depressions(dem, "fill_d4").view(np.uint32)), name
                t = torch.from_numpy(dem.copy()).cuda().contiguous()
                out, _ = sharded.fill_band(t, 0, 0, topology="D4")
                assert np.array_equal(out.cpu().numpy().view(np.uint32), expected.view(np.uint32)), (sw, name)


def _worker(rank, world, port, cases, chain_dem, chain_expected, out_q):
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
        for (sw, name), (dem, bounds, expected) in cases.items():
            with switches(sw):
                h = dem.shape[0]
                r0, r1 = bounds[rank]
                gt, gb = int(rank > 0), int(rank < world - 1)
                local = torch.from_numpy(dem[r0 - gt:r1 + gb].copy()).cuda().contiguous()
                out, xr = sharded.fill_band(local, gt, gb, row0=r0 - gt, height=h, topology="D4")
                got = out[gt:gt + r1 - r0].cpu().numpy().view(np.uint32)
                res[(sw, name)] = (bool(np.array_equal(got, expected[r0:r1].view(np.uint32))), xr)
        h, w = chain_dem.shape
        r0, r1, gt, gb = sharded.local_rows(h, world, rank)
        own = slice(gt, gt + r1 - r0)
        local = torch.from_numpy(np.ascontiguousarray(chain_dem[r0 - gt:r1 + gb])).cuda().contiguous()
        sharded.fill_band(local, gt, gb, topology="D4")
        filled_ok = bool(np.array_equal(local[own].cpu().numpy().view(np.uint32), chain_expected[0][r0:r1].view(np.uint32)))
        sharded.resolve_flats_band(local, gt, gb, ND)
        resolved_ok = bool(np.array_equal(local[own].cpu().numpy().view(np.uint32), chain_expected[1][r0:r1].view(np.uint32)))
        acc, _ = sharded.fa_band(local, gt, gb, ND, method="D4")
        a, x = acc[own].cpu().numpy(), chain_expected[2][r0:r1]
        res["chain"] = {"filled": filled_ok, "resolved": resolved_ok,
                        "fa_d4": bool(np.all(np.abs(a - x) <= FA_RTOL * np.abs(x)))}
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_processes_over_gloo_equal_one_gpu(world):
    cases = {}
    for sw in CASES.SWITCHES:
        with switches(sw):
            for name, (dem, bounds) in CASES.rasters(world, CASES.SWITCHES[sw]).items():
                cases[(sw, name)] = (dem, bounds, single_gpu_d4(dem))
    chain_dem = oracle.fbm_terrain(512, 640, seed=81, quantum=0.5)
    chain_dem[200:260, 100:300] = ND
    chain_expected = single_gpu_chain(chain_dem)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, cases, chain_dem, chain_expected, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        chain = res.pop("chain")
        assert all(chain.values()), (rank, chain)
        bad = [key for key, (ok, _) in res.items() if not ok]
        assert not bad, (rank, bad)
        assert len(res) == len(cases)
    assert all(p.exitcode == 0 for p in procs)


def test_python_protocol_and_unknown_topology_raise(monkeypatch):
    import torch
    dem = CASES.fbm(96, 80, seed=76)
    t = torch.from_numpy(dem.copy()).cuda().contiguous()
    with pytest.raises(ValueError, match="C\\+\\+ band driver"):
        sharded.fill_band(t, 0, 0, solver_cls=sharded.CudaBandSolver, topology="D4")
    monkeypatch.setenv("RDB_BAND_DRIVER", "python")
    with pytest.raises(ValueError, match="C\\+\\+ band driver"):
        sharded.fill_band(t, 0, 0, topology="D4")
    monkeypatch.delenv("RDB_BAND_DRIVER")
    with pytest.raises(Exception, match="Unknown topology!"):
        sharded.fill_band(t, 0, 0, topology="D6")
    assert np.array_equal(t.cpu().numpy(), dem)  # nothing ran
