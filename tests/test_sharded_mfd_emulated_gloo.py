"""The C++ row-band driver for the proportions methods (rdb200_mgpu_fa_method_f32_f64, reached through
sharded.fa_band(method=...)) over torch.distributed with the gloo backend, one process per band, on the CPU model of the
shipped kernels (tests/emu).  This is the collective entry point `torchrun` takes on N GPUs, seam donor masks, parked
outflow messages and termination votes included."""
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
CASES = [("D4", None), ("Quinn", None), ("Holmgren", 2.5), ("Holmgren", 0.7), ("Freeman", 1.1), ("Freeman", 4.0)]


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


def _worker(rank, world, port, lib_path, dems, weights, expected, out_q):
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
        dist.init_process_group("gloo", rank=rank, world_size=world)
        res = {}
        for dname, dem in dems.items():
            h, w = dem.shape
            local, (r0, r1, gt, gb) = sharded.scatter_rows(dem if rank == 0 else None, h, w, torch.float32, "cpu")
            wl, _ = sharded.scatter_rows(weights[dname] if rank == 0 else None, h, w, torch.float64, "cpu")
            own = slice(gt, gt + (r1 - r0))
            for m, e in CASES:
                for wkey, wt in (("ones", None), ("weights", wl.clone())):
                    acc, rounds = sharded.fa_band(local, gt, gb, ND, method=m, exponent=e, weights=wt)
                    a, x = acc[own].numpy(), expected[(dname, m, e, wkey)][r0:r1]
                    ok = bool(np.all(np.abs(a - x) <= 1e-6 * np.abs(x)))  # MFD_ACC_RTOL of the GPU parity tests
                    res[(dname, m, e, wkey)] = (ok, rounds)
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_mfd_band_driver_on_emulated_kernels(world):
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    import oracle
    lib_path = str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())
    gs = _load_module("gpu_sharded_mfd_cases", os.path.join(HERE, "test_gpu_sharded_mfd.py"))
    O = oracle.best()
    fbm = oracle.fbm_terrain(96, 84, seed=61, quantum=0.5)
    fbm[30:70, 20:40] = ND  # across every seam
    dems = {"fbm": O.resolve_flats(O.fill_depressions(fbm), ND), "channel": gs.serpentine_channel(40, 40)}
    rng = np.random.default_rng(world)
    weights = {k: rng.random(d.shape) for k, d in dems.items()}
    expected = {(k, m, e, wkey): O.fa_method(d, ND, m, e, None if wkey == "ones" else weights[k])
                for k, d in dems.items() for m, e in CASES for wkey in ("ones", "weights")}
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, lib_path, dems, weights, expected, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        bad = [k for k, (ok, _) in res.items() if not ok]
        assert not bad, (rank, bad)
        for (dname, m, e, wkey), (_, rounds) in res.items():
            if dname == "channel" and m != "D4":  # the channel crosses every seam many times
                assert rounds > 2, (rank, m, e, wkey, rounds)
    assert all(p.exitcode == 0 for p in procs)
