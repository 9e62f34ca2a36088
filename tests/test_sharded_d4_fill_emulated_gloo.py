"""The C++ row-band fill with D4 topology (rdb200_mgpu_fill_depressions_d4_f32, reached through
sharded.fill_band(topology="D4")) over torch.distributed with the gloo backend, one process per band, on the CPU model of
the shipped kernels (tests/emu).  World 1 is the driver with no neighbours.  Every band's owned rows must equal the
checker's PriorityFlood_Barnes2014<D4> bit for bit, with the multigrid start and the V-cycles on, off and at other
pooling factors.

Two rasters are built to fail if the driver ever mixes in the 8-neighbour stencil:
  * a diagonal wall that is tight under D4 everywhere and under D8 everywhere but one step across a seam;
  * a checkerboard of k x k blocks, k the driver's pooling factor, whose low blocks touch only at corners: a D8 fill of
    the pooled raster would drain them and start the band below the D4 answer, which relaxation never raises.
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
TILE = 64  # rows of a fill tile (csrc/fill.cu TY)

# library switches on top of the shipped defaults (fill_multigrid 8, fill_vcycle 8, fill_band_multigrid 0 = automatic)
SWITCHES = {"defaults": {}, "no-multigrid": {"fill_multigrid": 0}, "no-vcycle": {"fill_vcycle": 0},
            "band-multigrid-2": {"fill_band_multigrid": 2}}


def pooling_factor(world, switches):
    """The pooling factor mgpu_fill_band picks for its coarse level (0: no coarse level)."""
    fm = switches.get("fill_multigrid", 8)
    if fm < 2:
        return 0
    k = switches.get("fill_band_multigrid", 0)
    if k <= 0:
        k = fm * 2 if world > 2 and TILE % (2 * fm) == 0 else fm
    return k


def default_bounds(h, world):
    base, extra = divmod(h, world)
    out, r = [], 0
    for g in range(world):
        n = base + (1 if g < extra else 0)
        out.append((r, r + n))
        r += n
    return out


def _split_after(h, world, head):
    """Bands of the given sizes first, the rest of the rows cut evenly over the remaining bands."""
    out, r = [], 0
    for n in head[:world - 1]:
        out.append((r, r + n))
        r += n
    return out + [(r + a, r + b) for a, b in default_bounds(h - r, world - len(out))]


def fbm(h, w, seed, nodata_blocks=True):
    import oracle
    d = oracle.fbm_terrain(h, w, seed=seed, quantum=0.5)
    if nodata_blocks:
        d[h // 3:h // 3 + h // 4, w // 5:w // 2] = ND      # NoData blocks across the seams
        d[h // 2 - 5:h // 2 + 12, 3 * w // 4:w - 6] = ND
    return d


def diagonal_wall(h, w, seam):
    """A basin in the upper-left corner (interior 0, raster border 10) closed by a wall of height 10 that runs down and to
    the left.  The wall is two cells wide except on row `seam`, so its one D8 gap is the diagonal step from (seam-1, x)
    to (seam, x+1) across the seam, into a plain at height 1 that drains over the raster's edge.  D8 drains the basin
    to 1; D4 fills it to 10."""
    d = np.ones((h, w), np.float32)
    c = seam + w // 2
    for y in range(h):
        lo, hi = c - y, c - y + (0 if y == seam else 1)
        if lo > 0:
            d[y, :min(lo, w)] = 0.0
        d[y, max(lo, 0):max(min(hi + 1, w), 0)] = 10.0
    left = np.zeros((h, w), bool)
    for y in range(h):
        left[y, :max(min(c - y, w), 0)] = True
    border = np.zeros((h, w), bool)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    d[left & border] = 10.0
    return d


def checkerboard(h, w, k, seed):
    """k x k blocks aligned with the driver's pooling blocks: high ones (100 + fBm) and low ones (fBm), touching only at
    their corners.  Under D4 the low blocks inside the raster are pits closed by their four high neighbours; under D8 they
    chain corner to corner to the raster's edge.  The last 6 block columns are plain fBm terrain instead, whose lakes the
    lifted start leaves too high: the V-cycles lower them, so the coarse solver relaxes again and its surface comes back
    through the prolongation."""
    import oracle
    noise = oracle.fbm_terrain(h, w, seed=seed, amplitude=10.0, quantum=0.25)
    plain = oracle.fbm_terrain(h, w, seed=seed + 1, amplitude=60.0, quantum=0.25)
    yy, xx = np.mgrid[0:h, 0:w]
    high = ((yy // k) + (xx // k)) % 2 == 0
    board = np.where(high, 100.0 + noise, noise)
    return np.where(xx < w - 6 * k, board, plain).astype(np.float32)


def rasters(world, switches):
    """{name: (dem, band bounds)} for one world size and switch set."""
    k = pooling_factor(world, switches) or 8
    out = {"fbm": (fbm(190, 200, seed=71), default_bounds(190, world)),
           "odd-width": (fbm(150, 131, seed=72), default_bounds(150, world))}
    # the first band owns one tile of rows and the second 63 rows: both bottom ghost rows are local row 64, the first row
    # of the second tile row
    out["ghost-on-tile-edge"] = (fbm(200, 120, seed=73), _split_after(200, world, [TILE, TILE - 1]))
    # a middle band with a single owned row (an edge band needs two: its local raster has at least three rows)
    out["one-row-band"] = (fbm(90, 100, seed=74), _split_after(90, world, [40, 1]) if world >= 3 else default_bounds(90, world))
    b = default_bounds(160, world)
    out["diagonal-wall"] = (diagonal_wall(160, 150, b[1][0] if world > 1 else 80), b)
    out["checkerboard"] = (checkerboard(16 * k, 24 * k, k, seed=75), default_bounds(16 * k, world))
    return out


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
        for (sw, name, topo), (dem, bounds, expected) in cases.items():
            _lib.reset_params()
            _lib.set_param("fill_use_tma", 0)
            _lib.set_param("fill_multigrid_min", 16)  # coarse levels and V-cycles on these small rasters
            for key, value in SWITCHES[sw].items():
                _lib.set_param(key, value)
            h = dem.shape[0]
            r0, r1 = bounds[rank]
            gt, gb = int(rank > 0), int(rank < world - 1)
            local = torch.from_numpy(dem[r0 - gt:r1 + gb].copy())  # (the fill runs in place)
            filled, _ = sharded.fill_band(local, gt, gb, row0=r0 - gt, height=h, topology=topo)
            got = filled[gt:gt + r1 - r0].numpy().view(np.uint32)
            res[(sw, name, topo)] = bool(np.array_equal(got, expected[r0:r1].view(np.uint32)))
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5])
def test_d4_band_fill_on_emulated_kernels(world):
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    import oracle
    lib_path = str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())
    O = oracle.best()
    cases = {}
    for sw, switches in SWITCHES.items():
        for name, (dem, bounds) in rasters(world, switches).items():
            d4 = O.fill_depressions(dem, "fill_d4")
            cases[(sw, name, "D4")] = (dem, bounds, d4)
            if name == "diagonal-wall":
                d8 = O.fill_depressions(dem)
                assert d8[5, 5] == 1.0 and d4[5, 5] == 10.0  # the basin drains under D8 only
                cases[(sw, name, "D8")] = (dem, bounds, d8)  # ... and the D8 band fill finds the gap across the seam
            if name == "checkerboard":
                assert not np.array_equal(d4, O.fill_depressions(dem))
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
        bad = [key for key, ok in res.items() if not ok]
        assert not bad, (rank, bad)
        assert len(res) == len(cases)
    assert all(p.exitcode == 0 for p in procs)


def test_diagonal_wall_has_one_d8_gap_on_the_seam():
    """The wall raster has the shape the band test relies on: one D8 step through the wall, across the seam."""
    h, w, seam = 160, 150, 53
    d = diagonal_wall(h, w, seam)
    wall = d == 10.0
    inside = np.zeros_like(wall)
    inside[1:-1, 1:-1] = d[1:-1, 1:-1] == 0.0
    gaps = []
    for y in range(h - 1):
        for x in range(w):
            if not inside[y, x]:
                continue
            for dx in (-1, 0, 1):
                for dy in (-1, 0, 1):
                    yy, xx = y + dy, x + dx
                    if 0 <= yy < h and 0 <= xx < w and d[yy, xx] == 1.0:
                        gaps.append((y, x, yy, xx))
    c = seam + w // 2
    assert gaps == [(seam - 1, c - seam, seam, c - seam + 1)]


def test_checkerboard_blocks_touch_only_at_corners():
    k = 8
    d = checkerboard(48, 160, k, seed=1)[:, :160 - 6 * k]
    high = d >= 100.0
    assert high[0, 0] and not high[0, k] and not high[k, 0] and high[k, k]
    low = ~high
    # no two low cells of different blocks are 4-adjacent
    by, bx = np.mgrid[0:d.shape[0], 0:d.shape[1]] // k
    for a, b in ((np.s_[:, 1:], np.s_[:, :-1]), (np.s_[1:, :], np.s_[:-1, :])):
        both = low[a] & low[b]
        assert np.all((by[a] == by[b])[both] & (bx[a] == bx[b])[both])


def test_d4_needs_the_cxx_driver_and_unknown_topology_raises(monkeypatch):
    import torch
    from richdem_b200 import sharded
    t = torch.zeros((8, 8), dtype=torch.float32)
    with pytest.raises(ValueError, match="C\\+\\+ band driver"):
        sharded.fill_band(t, 0, 0, solver_cls=object, topology="D4")
    monkeypatch.setenv("RDB_BAND_DRIVER", "python")
    with pytest.raises(ValueError, match="C\\+\\+ band driver"):
        sharded.fill_band(t, 0, 0, topology="D4")
    with pytest.raises(Exception, match="Unknown topology!"):
        sharded.fill_band(t, 0, 0, topology="d4")
