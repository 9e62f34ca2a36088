"""The direction-grid pipeline over row bands -- rdb200_mgpu_d8_flow_directions_flats_f32 and
rdb200_mgpu_d8_flow_accum_u8_i32, reached through sharded.d8_flow_directions_band / d8_flow_accum_band -- over
torch.distributed with the gloo backend, one process per band, on the CPU model of the shipped kernels (tests/emu).

  * Every known-answer D8 grid of the reference's d8_flow_accum tests, cut into 1 to 5 bands, gives its known areas (what
    the reference's parallel_d8_accum test_small.sh asks of its tiles).
  * A filled, quantised fBm with NoData blocks across the seams, a plateau cut by every seam whose only outlet lies in
    the bottom band, and a plateau with no outlet at all: the owned directions equal the checker's
    barnes_flat_resolution_d8 (alter = 0) and the single-GPU call of the whole raster (alter = 1, with its altered
    elevations); the areas of those directions equal the checker's d8_flow_accum of the whole grid; ghost rows come
    back holding the neighbours' edge rows.
  * Wrong ghost flags fail on every rank with an error, before any communication."""
import ctypes as C
import importlib.util
import multiprocessing as mp
import os
import socket
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def plateau_raster(O):
    """A filled fBm (96 x 84) with NoData blocks across the seams and two plateaus cut by every seam of 2 to 5 bands:
    one whose only outlet is a channel leaving through its bottom rim to the raster's bottom edge, and one enclosed
    by a higher rim, with no outlet anywhere."""
    import oracle
    fbm = oracle.fbm_terrain(96, 84, seed=73, quantum=0.5)
    fbm[20:70, 30:40] = ND
    fbm[44:52, 0:12] = ND
    dem = O.fill_depressions(fbm)
    top = float(dem.max())
    low = float(dem[dem != ND].min())
    dem[8:86, 48:72] = top + 10.0  # rim
    dem[9:85, 49:71] = top + 5.0   # drains through the channel below only
    dem[85:, 60] = low - 1.0 - np.arange(11, dtype=np.float32)
    dem[4:60, 74:83] = top + 10.0  # rim
    dem[5:59, 75:82] = top + 4.0   # no outlet
    return dem


def _worker(rank, world, port, lib_path, fixtures, dems, expected, out_q):
    import torch
    import torch.distributed as dist
    from richdem_b200 import _lib, sharded

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        # point this process's Python layer at the kernel emulation (tests only; the loader itself refuses it)
        L = C.CDLL(lib_path)
        for name, argtypes in _lib.SIGNATURES.items():
            f = getattr(L, name)
            f.argtypes = argtypes
            f.restype = C.c_int
        L.rdb200_last_error.restype = C.c_char_p
        L.rdb200_last_error.argtypes = []
        _lib._lib = L
        _lib.use_torch_stream = lambda: None
        sharded._on_device = lambda t: True
        _lib.init(0)
        _lib.set_param("fill_use_tma", 0)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        res = {"fixtures": {}}
        for name, (dirs, area) in fixtures.items():
            h, w = dirs.shape
            r0, r1, gt, gb = sharded.local_rows(h, world, rank)
            local = torch.from_numpy(np.ascontiguousarray(dirs[r0 - gt:r1 + gb]))
            if gt:
                local[0] = 77  # the ghost rows are not read
            if gb:
                local[-1] = 0
            got, _ = sharded.d8_flow_accum_band(local, gt, gb)
            res["fixtures"][name] = bool(np.array_equal(got[gt:gt + r1 - r0].numpy(), area[r0:r1]))
        for dname, dem in dems.items():
            h, w = dem.shape
            r0, r1, gt, gb = sharded.local_rows(h, world, rank)
            x = expected[dname]
            r = {}
            for alter in (0, 1):
                local = torch.from_numpy(np.ascontiguousarray(dem[r0 - gt:r1 + gb]))
                dirs, it = sharded.d8_flow_directions_band(local, gt, gb, ND, alter=bool(alter))
                d = dirs.numpy()
                want = x["dirs"] if not alter else x["dirs_alter"]
                r[f"dirs{alter}"] = bool(np.array_equal(d[gt:gt + r1 - r0], want[r0:r1]))
                r[f"dir_ghosts{alter}"] = bool((not gt or np.array_equal(d[0], want[r0 - 1])) and
                                               (not gb or np.array_equal(d[-1], want[r1])))
                r[f"iters{alter}"] = it
                if alter:
                    z, zx = local.numpy().view(np.uint32), x["altered"].view(np.uint32)
                    r["altered"] = bool(np.array_equal(z[gt:gt + r1 - r0], zx[r0:r1]))
                    r["dem_ghosts"] = bool((not gt or np.array_equal(z[0], zx[r0 - 1])) and
                                           (not gb or np.array_equal(z[-1], zx[r1])))
                else:
                    area, xr = sharded.d8_flow_accum_band(dirs, gt, gb)
                    r["area"] = bool(np.array_equal(area[gt:gt + r1 - r0].numpy(), x["area"][r0:r1]))
                    r["rounds"] = xr
            res[dname] = r
        # bad arguments: every rank fails before the first collective
        dem = dems["fbm"]
        h, w = dem.shape
        r0, r1, gt, gb = sharded.local_rows(h, world, rank)
        local = torch.from_numpy(np.ascontiguousarray(dem[r0 - gt:r1 + gb]))
        dirs = torch.zeros(local.shape, dtype=torch.uint8)
        area = torch.zeros(local.shape, dtype=torch.int32)
        cm = sharded.lib_comm()
        errors = {}
        rc = L.rdb200_mgpu_d8_flow_directions_flats_f32(cm.handle, local.data_ptr(), dirs.data_ptr(), w, local.shape[0], ND,
                                                        1 - gt, 1 - gb, 0, None)
        errors["dirs"] = (rc, (L.rdb200_last_error() or b"").decode())
        rc = L.rdb200_mgpu_d8_flow_accum_u8_i32(cm.handle, dirs.data_ptr(), area.data_ptr(), w, local.shape[0], 1 - gt, 1 - gb,
                                                None)
        errors["accum"] = (rc, (L.rdb200_last_error() or b"").decode())
        rc = L.rdb200_mgpu_d8_flow_accum_u8_i32(cm.handle, dirs.data_ptr(), None, w, local.shape[0], gt, gb, None)
        errors["null area"] = (rc, (L.rdb200_last_error() or b"").decode())
        res["_errors"] = errors
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _single_gpu_alter(lib_path, dem):
    """Directions and elevations of the single-GPU call with alter = 1 on the whole raster, on the same kernel model."""
    from richdem_b200 import _lib
    L = C.CDLL(lib_path)
    f = L.rdb200_dev_d8_flow_directions_flats_f32
    f.argtypes = _lib.SIGNATURES["rdb200_dev_d8_flow_directions_flats_f32"]
    L.rdb200_init.argtypes = [C.c_int32]
    L.rdb200_set_param.argtypes = [C.c_char_p, C.c_int64]
    assert L.rdb200_init(0) == 0 and L.rdb200_set_param(b"fill_use_tma", 0) == 0
    z = np.ascontiguousarray(dem.copy())
    dirs = np.empty(z.shape, np.uint8)
    assert f(z.ctypes.data, dirs.ctypes.data, z.shape[1], z.shape[0], ND, 1) == 0
    return dirs, z


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5])
def test_d8_dirs_band_drivers_on_emulated_kernels(world, golden):
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    import oracle
    lib_path = str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())
    O = oracle.best()
    g = golden["flow_accum_fixtures"]
    fixtures = {}
    for name, nd in zip(g["names"], g["d8_nodata"]):
        d = g[f"{name}__d8"]
        fixtures[str(name)] = (np.where(d == nd, 255, d).astype(np.uint8), g[f"{name}__out"])
    dems = {"fbm": plateau_raster(O)}
    expected = {}
    for k, dem in dems.items():
        dirs = O.d8_flow_directions_flats(dem, ND)[0]
        dirs_alter, altered = _single_gpu_alter(lib_path, dem)
        expected[k] = {"dirs": dirs, "dirs_alter": dirs_alter, "altered": altered, "area": O.d8_flow_accum(dirs)}
    fbm = expected["fbm"]
    assert (fbm["dirs"][9:85, 49:71] != 0).all()  # the plateau with the outlet drains ...
    assert (fbm["dirs"][5:59, 75:82] == 0).all()  # ... the enclosed one does not
    assert (fbm["area"][85:, 60] > 76 * 20).all()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, lib_path, fixtures, dems, expected, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        errors = res.pop("_errors")
        assert all(res.pop("fixtures").values()), (rank, res)
        for dname, r in res.items():
            assert all(v for k, v in r.items() if not k.startswith(("iters", "rounds"))), (rank, dname, r)
            if world > 1:
                assert r["iters0"] >= 2 and r["rounds"] >= 2, (rank, dname, r)
        for case in ("dirs", "accum"):
            assert errors[case][0] != 0 and "ghost_top" in errors[case][1], (rank, errors)
        assert errors["null area"][0] != 0 and "null pointer" in errors["null area"][1], (rank, errors)
    assert all(p.exitcode == 0 for p in procs)
