"""d8_flow_accum of direction grids that no DEM produces: loops, codes that point off the raster or into NoData, all
NoData, strips one cell wide.  D8FlowAccum (rdb200_d8_flow_accum_u8_i32) and the row-band entry
(rdb200_mgpu_d8_flow_accum_u8_i32, reached through sharded.d8_flow_accum_band) must give the checker's d8_flow_accum bit
for bit.  A cell on a loop, or fed by one, never leaves the reference's source queue: it keeps the inflow it received and
never adds its own unit.  Every case runs on the GPU and on the CPU model of the kernels; the band entry also runs with
one process per band over gloo, on both."""
import ctypes as C
import importlib.util
import multiprocessing as mp
import os
import socket
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
NODATA = 255
NO_FLOW, W_, NW, N_, NE, E_, SE, S_, SW = range(9)


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_ek = _load_module("emulated_kernel_fixtures", os.path.join(HERE, "test_emulated_kernels.py"))
emu_lib, emulated = _ek.emu_lib, _ek.emulated


# ---- direction grids ------------------------------------------------------------------------------------------------
def ring(d, y0, x0, y1, x1):
    """The boundary of rows y0..y1 x columns x0..x1 becomes one clockwise loop."""
    d[y0, x0:x1] = E_
    d[y0:y1, x1] = S_
    d[y1, x0 + 1:x1 + 1] = W_
    d[y0 + 1:y1 + 1, x0] = N_
    return d


def random_codes(h, w, seed, nodata_share=0.05):
    rng = np.random.default_rng(seed)
    d = rng.integers(0, 9, (h, w)).astype(np.uint8)
    d[rng.random((h, w)) < nodata_share] = NODATA
    return d


def two_cycle_fed_by_chain():
    """Four cells flow east into a pair of cells that point at each other."""
    d = np.zeros((5, 9), np.uint8)
    d[2, 1:6] = E_
    d[2, 6] = W_
    return d


def long_loop_with_trees(h=150, w=190, seed=3):
    """A loop of 560 cells; the cells inside it flow north into its top row, the cells outside flow towards it, with
    every tenth cell a random code (more loops, trees that end in NoData or off the raster); a long chain winds in from
    the bottom-left corner."""
    rng = np.random.default_rng(seed)
    d = np.zeros((h, w), np.uint8)
    y0, x0, y1, x1 = 20, 25, 120, 165
    d[y0 + 1:y1, x0 + 1:x1] = N_
    d[:y0, :] = S_
    d[y1 + 1:, :] = N_
    d[:, :x0] = E_
    d[:, x1 + 1:] = W_
    noise = rng.random((h, w)) < 0.1
    d[noise] = rng.integers(0, 9, noise.sum())
    d[rng.random((h, w)) < 0.02] = NODATA
    for y in range(h - 1, y1, -2):  # the chain: west-east runs joined by steps north
        xs = range(0, x0) if (h - 1 - y) % 4 == 0 else range(x0 - 1, -1, -1)
        for x in xs:
            d[y, x] = E_ if (h - 1 - y) % 4 == 0 else W_
        d[y, xs[-1]] = N_
        d[y - 1, xs[-1]] = N_
    ring(d, y0, x0, y1, x1)
    return d


def loop_across_tile_seams(h=130, w=140, seed=5):
    """A loop that crosses the 64-cell seams in both directions, in random codes with NoData."""
    return ring(random_codes(h, w, seed), 40, 50, 90, 80)


def off_raster_and_into_nodata(h=70, w=90, seed=7):
    """Border cells point off the raster; chains run into a NoData block and into a NoData column; the rest random."""
    d = random_codes(h, w, seed)
    d[0, :], d[-1, :], d[:, 0], d[:, -1] = N_, S_, W_, E_
    d[0, 0], d[0, -1], d[-1, 0], d[-1, -1] = NW, NE, SW, SE
    d[20:30, 30:50] = NODATA
    d[10:20, 35:45] = S_   # into the block from above
    d[30:40, 35:45] = N_   # and from below
    d[5:60, 70] = NODATA
    d[5:60, 60:70] = E_    # into the column
    return d


def all_nodata():
    return np.full((33, 47), NODATA, np.uint8)


def strip(h, w, seed):
    return random_codes(h, w, seed, nodata_share=0.1)


def band_loops(w, h=61, seed=11):
    """Rows cut into bands of 2 to 5 processes: loops across every row boundary (two columns of vertical 2-cycles, at
    even and odd row pairs), a loop as tall as the raster, and a chain that crosses every seam into a 2-cycle."""
    d = random_codes(h, w, seed)
    ring(d, 1, 2, h - 2, 10)
    d[0:h - 2, 20] = S_
    d[h - 2, 20], d[h - 2, 21] = E_, W_
    for y in range(0, h - 1, 2):
        d[y, 40], d[y + 1, 40] = S_, N_
    for y in range(1, h - 1, 2):
        d[y, 41], d[y + 1, 41] = S_, N_
    return d


CASES = {
    "two_cycle_fed_by_chain": two_cycle_fed_by_chain,
    "long_loop_with_trees": long_loop_with_trees,
    "loop_across_tile_seams": loop_across_tile_seams,
    "random_70x90": lambda: random_codes(70, 90, 13),
    "random_129x260": lambda: random_codes(129, 260, 17, nodata_share=0.2),
    "off_raster_and_into_nodata": off_raster_and_into_nodata,
    "all_nodata": all_nodata,
    "strip_1x300": lambda: strip(1, 300, 19),
    "strip_300x1": lambda: strip(300, 1, 23),
    "strip_1x1": lambda: np.array([[E_]], np.uint8),
    "band_loops_w84": lambda: band_loops(84),
    "band_loops_w83": lambda: band_loops(83),
}


def large_grid():
    """1100 x 1000 cells (above 2^20): random codes, 5 % NoData, and loops of a few thousand cells."""
    d = random_codes(1100, 1000, 29)
    ring(d, 10, 10, 1090, 990)
    ring(d, 300, 200, 800, 700)
    return d


# ---- the cases are what they say --------------------------------------------------------------------------------------
def test_two_cycle_known_answer(checker):
    """The loop cells keep the inflow and never count themselves: 4 and 0 (the chain gives 1, 2, 3, 4 before it)."""
    a = checker.d8_flow_accum(two_cycle_fed_by_chain())
    assert list(a[2, 1:7]) == [1, 2, 3, 4, 4, 0]


def test_loops_where_intended(checker):
    """Cells that never leave the reference's queue show up where the cases put loops."""
    from richdem_b200 import sharded
    a = checker.d8_flow_accum(long_loop_with_trees())
    # the loop passes nothing on: its top row holds what the columns inside bring (noise cuts them short)
    assert (a[20, 25:165] >= 0).all() and a[20, 25:165].sum() > 3000 and a[20, 25:165].max() < 1000
    for world in (2, 3, 4, 5):
        for r0, _ in sharded.band_bounds(61, world)[1:]:
            d = band_loops(84)
            assert d[r0 - 1, 40] + d[r0, 40] == S_ + N_ or d[r0 - 1, 41] + d[r0, 41] == S_ + N_
    assert (checker.d8_flow_accum(all_nodata()) == -1).all()


def _expected(checker, d):
    return checker.d8_flow_accum(d)


def _single(d):
    import richdem_b200 as rd
    return np.asarray(rd.D8FlowAccum(d))


def _band_world_one(d, cuda):
    import torch
    from richdem_b200 import sharded
    t = torch.from_numpy(d.copy())
    if cuda:
        t = t.cuda()
    area, rounds = sharded.d8_flow_accum_band(t.contiguous(), 0, 0)
    assert rounds == 1
    return area.cpu().numpy()


# ---- GPU ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_dirgrid_accum(checker, name):
    d = CASES[name]()
    x = _expected(checker, d)
    assert np.array_equal(_single(d), x), f"{(_single(d) != x).sum()} cells differ"
    assert np.array_equal(_band_world_one(d, True), x)


@pytest.mark.gpu
def test_dirgrid_accum_large(checker):
    """Many warps of sources and walks; width % 4 == 0, so one band takes the packed band walk."""
    from richdem_b200 import _lib
    d = large_grid()
    x = _expected(checker, d)
    assert (x == 0).sum() > 1000  # loop cells without inflow
    assert np.array_equal(_single(d), x)
    assert np.array_equal(_band_world_one(d, True), x)
    try:
        _lib.set_param("accum_walk_lanes", 0)
        assert np.array_equal(_band_world_one(d, True), x)
        _lib.set_param("accum_packed", 0)
        assert np.array_equal(_band_world_one(d, True), x)
    finally:
        _lib.reset_params()


# ---- CPU model of the kernels --------------------------------------------------------------------------------------------
@pytest.fixture()
def host_bands(emulated, monkeypatch):
    from richdem_b200 import _lib, sharded
    monkeypatch.setattr(sharded, "_on_device", lambda t: True)  # "device" memory is host memory here
    monkeypatch.setattr(sharded, "_COMMS", {})                  # communicators of this library only
    monkeypatch.setattr(_lib, "use_torch_stream", lambda: None)
    return emulated


@pytest.mark.parametrize("name", sorted(CASES))
def test_dirgrid_accum_emulated(host_bands, checker, name):
    from richdem_b200 import _lib
    d = CASES[name]()
    x = _expected(checker, d)
    assert np.array_equal(_single(d), x), f"{(_single(d) != x).sum()} cells differ"
    for params in ({}, {"accum_walk_lanes": 0}, {"accum_packed": 0}):
        _lib.reset_params()
        _lib.set_param("fill_use_tma", 0)
        for k, v in params.items():
            _lib.set_param(k, v)
        assert np.array_equal(_band_world_one(d, False), x), params


# ---- one process per band over gloo -------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, lib_path, grids, out_q):
    """lib_path: the CPU model of the kernels, bands in host memory; None: the library on the GPU."""
    import torch
    import torch.distributed as dist
    from richdem_b200 import _lib, sharded

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        if lib_path:
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
        else:
            torch.cuda.set_device(0)
        _lib.init(0)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        res = {}
        for name, (d, x) in grids.items():
            r0, r1, gt, gb = sharded.local_rows(d.shape[0], world, rank)
            local = torch.from_numpy(np.ascontiguousarray(d[r0 - gt:r1 + gb]))
            if gt:
                local[0] = 77  # the ghost rows are not read
            if gb:
                local[-1] = E_
            if not lib_path:
                local = local.cuda()
            area, _ = sharded.d8_flow_accum_band(local, gt, gb)
            got = area[gt:gt + r1 - r0].cpu().numpy()
            res[name] = int((got != x[r0:r1]).sum())
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _run_gloo(world, lib_path, grids):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, lib_path, grids, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        assert all(v == 0 for v in res.values()), (rank, res)  # cells that differ, per grid
    assert all(p.exitcode == 0 for p in procs)


def _gloo_grids(checker):
    names = ("band_loops_w84", "band_loops_w83", "long_loop_with_trees", "two_cycle_fed_by_chain")
    return {k: (CASES[k](), _expected(checker, CASES[k]())) for k in names}


@pytest.mark.parametrize("world", [2, 3, 4, 5])
def test_band_loops_over_gloo_emulated(checker, world):
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    lib_path = str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())
    _run_gloo(world, lib_path, _gloo_grids(checker))


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 4])
def test_band_loops_over_gloo(checker, world):
    grids = _gloo_grids(checker)
    d = large_grid()
    grids["large"] = (d, _expected(checker, d))
    _run_gloo(world, None, grids)
