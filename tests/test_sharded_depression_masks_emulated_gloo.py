"""PitMask and HasDepressions over row bands (rdb200_mgpu_pit_mask_* / rdb200_mgpu_has_depressions_*, reached through
sharded.pit_mask_band / sharded.has_depressions_band) over torch.distributed with the gloo backend, one process per band,
on the CPU model of the shipped kernels (tests/emu).  Every band's owned mask rows and every rank's answer must equal the
single-raster answer of the C restatement (oracle/depressions.c), for D8 and D4, at world sizes 1 to 4.

The rasters put band seams where the band drivers can go wrong:
  * a strict pit on the first owned row of a band: its test needs the ghost row above, and it is the raster's only
    depression, so a rank that ignored its ghost rows would answer "no";
  * an enclosed flat-bottomed basin cut by a seam, the only depression: no strict pit anywhere, so the band fill runs;
  * a surface without depressions (the fill of an fBm raster): both passes run and answer "no";
  * fBm terrain with NoData blocks across the seams.
"""
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


def default_bounds(h, world):
    base, extra = divmod(h, world)
    out, r = [], 0
    for g in range(world):
        n = base + (1 if g < extra else 0)
        out.append((r, r + n))
        r += n
    return out


def plane(h, w):
    """Rises away from the top-left corner: every cell drains, no depression."""
    return np.add.outer(2 * np.arange(h, dtype=np.float32), 3 * np.arange(w, dtype=np.float32))


def rasters(world):
    """{name: (dem, band bounds)}."""
    import oracle
    h, w = 120, 90
    b = default_bounds(h, world)
    seam = b[1][0] if world > 1 else h // 2
    pit = plane(h, w)
    pit[seam, 40] = -5.0  # a strict pit on the first owned row of band 1
    basin = plane(h, w)
    yy, xx = np.mgrid[0:h, 0:w]
    r2 = (yy - seam) ** 2 + (xx - 45) ** 2
    basin[r2 < 12 ** 2] = 500.0   # a ring ...
    basin[r2 < 10 ** 2] = 100.0   # ... around a flat floor, centred on the seam
    fbm = oracle.fbm_terrain(h, w, seed=61, quantum=0.5)
    nodata = fbm.copy()
    nodata[h // 3:h // 3 + h // 4, w // 5:w // 2] = ND
    nodata[h // 2 - 5:h // 2 + 12, 3 * w // 4:w - 6] = ND
    filled = oracle.port().fill_depressions(fbm)
    return {"pit-on-seam": (pit, b), "basin-across-seam": (basin, b), "no-depressions": (filled, b),
            "fbm-nodata": (nodata, b)}


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


def _worker(rank, world, port, lib_path, cases, out_q):
    import torch
    import torch.distributed as dist
    from richdem_b200 import _lib, sharded

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
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
        _lib.set_param("fill_multigrid_min", 16)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        res = {}
        for (name, topo), (dem, bounds, mask, has) in cases.items():
            h = dem.shape[0]
            r0, r1 = bounds[rank]
            gt, gb = int(rank > 0), int(rank < world - 1)
            local = torch.from_numpy(dem[r0 - gt:r1 + gb].copy())
            before = local.clone()
            got = sharded.pit_mask_band(local, gt, gb, ND, topology=topo, row0=r0 - gt, height=h)
            ok_mask = bool(np.array_equal(got[gt:gt + r1 - r0].numpy(), mask[r0:r1]))
            got_has = sharded.has_depressions_band(local, gt, gb, topology=topo)  # row0 / height gathered from the ranks
            untouched = bool(torch.equal(local.view(torch.int32), before.view(torch.int32)))
            res[(name, topo)] = (ok_mask, got_has == has, untouched)
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_depression_masks_over_bands_on_emulated_kernels(world):
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    from oracle import depressions
    lib_path = str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())
    P = depressions.port()
    cases = {}
    for name, (dem, bounds) in rasters(world).items():
        for topo in ("D8", "D4"):
            cases[(name, topo)] = (dem, bounds, P.pit_mask(dem, ND, topo), P.has_depressions(dem, topo))
    assert cases[("pit-on-seam", "D8")][3] and cases[("basin-across-seam", "D4")][3]
    assert not cases[("no-depressions", "D8")][3]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, lib_path, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=900) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        bad = [key for key, v in res.items() if not all(v)]
        assert not bad, (rank, bad, [res[k] for k in bad])
        assert len(res) == len(cases)
    assert all(p.exitcode == 0 for p in procs)
