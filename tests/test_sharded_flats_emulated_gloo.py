"""The C++ row-band flat resolution driver (rdb200_mgpu_resolve_flats_epsilon_f32) over torch.distributed with the gloo
backend, one process per band, on the CPU model of the shipped kernels (tests/emu).  Owned rows must equal the CPU
checker's ResolveFlatsEpsilon bit for bit, and the ghost rows must come back holding the neighbours' resolved edge rows.
Bad arguments must fail on every rank before any communication, so that no rank is left waiting."""
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


def comb_raster():
    """The flat of test_gpu_sharded.py::test_band_flat_resolution_snaking_flat: vertical channels joined at the top,
    one outlet at the bottom, so outlet flags and flat heights cross every seam several times."""
    dem = np.full((96, 64), 10.0, np.float32)
    dem[:, ::4] = 5.0
    dem[2, :] = 5.0
    dem[93, 1::8] = 5.0
    dem[0, :] = dem[-1, :] = 20.0
    dem[:, 0] = dem[:, -1] = 20.0
    dem[94, 4] = 1.0
    dem[95, 4] = 0.0
    return dem


def _worker(rank, world, port, lib_path, dems, expected, out_q):
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
        cm = sharded.lib_comm()
        res = {}
        for dname, dem in dems.items():
            h, w = dem.shape
            local, (r0, r1, gt, gb) = sharded.scatter_rows(dem if rank == 0 else None, h, w, torch.float32, "cpu")
            it = C.c_int32(-1)
            rc = L.rdb200_mgpu_resolve_flats_epsilon_f32(cm.handle, local.data_ptr(), w, local.shape[0], ND, gt, gb,
                                                         C.byref(it))
            got = local.numpy().view(np.uint32)
            x = expected[dname].view(np.uint32)
            res[dname] = {"rc": rc, "owned": bool(np.array_equal(got[gt:gt + (r1 - r0)], x[r0:r1])),
                          "ghosts": bool((not gt or np.array_equal(got[0], x[r0 - 1])) and
                                         (not gb or np.array_equal(got[-1], x[r1]))),
                          "iters": int(it.value)}
        # bad arguments: every rank fails before the first collective
        dem = dems["fbm"]
        h, w = dem.shape
        local, (r0, r1, gt, gb) = sharded.scatter_rows(dem if rank == 0 else None, h, w, torch.float32, "cpu")
        errors = {}
        for case, (rows, t, b) in {"ghost flags": (local.shape[0], 0, 0),
                                   "no owned rows": (gt + gb, gt, gb)}.items():
            rc = L.rdb200_mgpu_resolve_flats_epsilon_f32(cm.handle, local.data_ptr(), w, rows, ND, t, b, None)
            errors[case] = (rc, (L.rdb200_last_error() or b"").decode())
        rc = L.rdb200_mgpu_resolve_flats_epsilon_f32(None, local.data_ptr(), w, local.shape[0], ND, gt, gb, None)
        errors["null comm"] = (rc, (L.rdb200_last_error() or b"").decode())
        res["_errors"] = errors
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_flats_band_driver_on_emulated_kernels(world):
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    import oracle
    lib_path = str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())
    O = oracle.best()
    fbm = oracle.fbm_terrain(96, 84, seed=71, quantum=0.5)
    fbm[20:70, 30:50] = ND  # across every seam
    enclosed = O.fill_depressions(oracle.fbm_terrain(60, 40, seed=72, quantum=0.5))
    enclosed[10:50, 5:35] = ND  # a plateau inside a NoData hole; it crosses every seam and drains into the NoData
    enclosed[14:46, 9:31] = 3.0
    dems = {"fbm": O.fill_depressions(fbm), "comb": O.fill_depressions(comb_raster()),
            "all_flat": np.full((40, 30), 7.0, np.float32), "enclosed": enclosed,
            "one_row": O.fill_depressions(oracle.fbm_terrain(world, 33, seed=world, quantum=2.0))}
    expected = {k: O.resolve_flats(d, ND) for k, d in dems.items()}
    for k in ("fbm", "comb", "all_flat", "enclosed"):
        assert (expected[k] != dems[k]).any(), k  # every raster has something to resolve
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, lib_path, dems, expected, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        errors = res.pop("_errors")
        for dname, r in res.items():
            assert r["rc"] == 0 and r["owned"] and r["ghosts"], (rank, dname, r)
            assert r["iters"] >= 2, (rank, dname, r)  # at least one flag and one height round
        assert res["comb"]["iters"] > 3, (rank, res["comb"])
        assert errors["ghost flags"][0] != 0 and "ghost_top" in errors["ghost flags"][1], (rank, errors)
        assert errors["no owned rows"][0] != 0 and "no owned rows" in errors["no owned rows"][1], (rank, errors)
        assert errors["null comm"][0] != 0 and "null pointer" in errors["null comm"][1], (rank, errors)
    # every rank counted the same merge rounds (they end on the same all-reduced vote)
    for dname in results[0][1]:
        assert len({res[dname]["iters"] for _, res, _ in results}) == 1, dname
    assert all(p.exitcode == 0 for p in procs)
