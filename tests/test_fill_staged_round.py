"""The staged first round of a lifted fill builds each tile's window from the coarse surface and relaxes it, and a tile
edge it lowers must wake the neighbours that already read the lifted value in the same round.  These terrains are where
such a round goes wrong, each run under multigrid configurations that give small rasters a coarse level (so the staged
round runs), for D8 and D4, and compared as uint32 with the CPU checker and with the padded path (fill_external_z = 0,
which loads its first round instead of staging it):
  * a diagonal staircase wall that drains under D8 and not under D4 (a D8 update in the D4 fill lowers cells too far);
  * a serpentine maze with 1-cell corridors (one long path, filled to the level of its outlet);
  * long valleys that cross many tiles diagonally and drain only through tile edges and corners, downstream towards
    the last tiles of the round: an upstream tile reads its downstream neighbour's lifted apron first and must be woken
    when that neighbour drains.  The steep one (more rows than columns) drains down whole columns, so the round's column
    sweeps lower its cells, tile edges included, before the block relaxation sees them.
Pools of 8, 4 and 3 exercise the window build with and without 4 cells per coarse block."""
import importlib.util
import os

import numpy as np
import pytest

from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
WALL = 100.0


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_ez = _load_module("fill_external_z_checks", os.path.join(HERE, "test_fill_external_z.py"))
emu_lib, emulated = _ez.emu_lib, _ez.emulated


def staircase(n, seed):
    """A wall along the diagonal, one cell per row: the cells above it reach the outlet below it through the diagonal
    gaps under D8 and not at all under D4."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:n, 0:n]
    dem = np.where(xx > yy, rng.uniform(0, 5, (n, n)), rng.uniform(0, 3, (n, n))).astype(np.float32)
    dem[yy == xx] = WALL
    dem[0, :] = dem[-1, :] = dem[:, 0] = dem[:, -1] = WALL
    dem[n - 1, 1] = 3.5
    return dem


def serpentine(h, w, seed):
    """1-cell corridors along the rows joined at alternate ends, 1-cell walls; the only outlet is the border cell (0, 1)."""
    rng = np.random.default_rng(seed)
    dem = np.full((h, w), WALL, np.float32)
    rows = list(range(1, h - 1, 2))
    for k, y in enumerate(rows):
        dem[y, 1:w - 1] = rng.uniform(0, 5, w - 2)
        if k + 1 < len(rows):
            dem[y + 1, w - 2 if k % 2 == 0 else 1] = rng.uniform(0, 5)
    dem[0, 1] = 5.5
    return dem


def diagonal_valley(h, w, seed):
    """A 4-connected staircase valley from (1, 1) to (h - 2, w - 2) between walls, its floor falling towards the outlet
    (h - 1, w - 2) on the south border, with noise that leaves small pits along it."""
    rng = np.random.default_rng(seed)
    dem = np.full((h, w), WALL, np.float32)
    y = x = 1
    path = [(y, x)]
    while (y, x) != (h - 2, w - 2):
        # step towards the straight line from (1, 1) to (h - 2, w - 2), right or down
        if y < h - 2 and (x >= w - 2 or (y - 1) * (w - 3) <= (x - 1) * (h - 3)):
            y += 1
        else:
            x += 1
        path.append((y, x))
    n = len(path)
    for i, (py, px) in enumerate(path):
        dem[py, px] = 60.0 - 50.0 * i / n + rng.uniform(0, 2)
    dem[h - 1, w - 2] = 1.0
    return dem


# widths are multiples of 4, so the fill reads Z from the raster and stages its first round
TERRAINS = {"staircase": lambda n: staircase(n, 7), "serpentine_w1": lambda n: serpentine(n + 1, n, 3),
            "diagonal_valley": lambda n: diagonal_valley(n - 10, 2 * n, 5),
            "steep_valley": lambda n: diagonal_valley(2 * n - 20, n - 8, 6)}
# on the GPU the staircase and the valley are large enough for the default configuration's coarse level (sides of
# 1024 and more); the maze's corridor is one path, which the flood walks a tile per round
GPU_SIZES = {"staircase": 1100, "serpentine_w1": 520, "diagonal_valley": 1100, "steep_valley": 1100}
# multigrid configurations whose coarse level exists at these sizes (pool 8, 4 and 3: the window build's coarse column
# and row stepping with and without 4 cells per coarse block)
STAGED_CONFIGS = [{"fill_multigrid": 8, "fill_multigrid_min": 32, "fill_vcycle": 1},
                  {"fill_multigrid": 4, "fill_multigrid_min": 32, "fill_vcycle": 2},
                  {"fill_multigrid": 3, "fill_multigrid_min": 32, "fill_vcycle": 0}]


def _cfg_id(cfg):
    return ",".join(f"{k}={v}" for k, v in cfg.items()) or "defaults"


def check_terrain(L, checker, dem, topo, cfg, on_gpu):
    expected = (checker.fill_depressions(dem) if topo == "D8" else checker.fill_depressions(dem, "fill_d4")).view(np.uint32)
    runs = {}
    try:
        for name, ext in (("external", 1), ("padded", 0)):
            _lib.reset_params()
            if not on_gpu:
                _lib.set_param("fill_use_tma", 0)
            for k, v in cfg.items():
                _lib.set_param(k, v)
            _lib.set_param("fill_external_z", ext)
            runs[name] = _ez.fill_dev(L, dem, topo, 0, on_gpu)
            runs[name + "_stats"] = _lib.stats()
    finally:
        _lib.reset_params()
        if not on_gpu:
            _lib.set_param("fill_use_tma", 0)
    for name in ("external", "padded"):
        got = runs[name].view(np.uint32)
        assert np.array_equal(got, expected), f"{name}: {(got != expected).sum()} cells differ from the checker"
    return runs


def test_terrains_are_what_they_say(checker):
    s = TERRAINS["staircase"](140)
    assert checker.fill_depressions(s, "fill_d4")[5, 100] == WALL and checker.fill_depressions(s)[5, 100] < 6
    v = TERRAINS["diagonal_valley"](140)
    valley = v != WALL
    f = checker.fill_depressions(v, "fill_d4")
    # the valley drains to its outlet through tile after tile: it crosses tile columns and rows
    ys, xs = np.nonzero(valley)
    assert len(np.unique(ys // 64)) >= 2 and len(np.unique(xs // 64)) >= 4
    assert (f[valley] < 70).all() and (f[~valley] == WALL).all()
    v = TERRAINS["steep_valley"](140)
    ys, xs = np.nonzero(v != WALL)
    assert len(np.unique(ys // 64)) >= 4 and len(np.unique(xs // 64)) >= 2 and v.shape[1] % 4 == 0
    m = TERRAINS["serpentine_w1"](140)
    assert (checker.fill_depressions(m)[m != WALL] == np.float32(5.5)).all()


# ---- on the H100 ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", [{}] + STAGED_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("name", sorted(TERRAINS))
def test_staged_round_gpu(checker, name, cfg, topo):
    check_terrain(_lib.lib(), checker, TERRAINS[name](GPU_SIZES[name]), topo, cfg, on_gpu=True)


# ---- on the CPU model of the kernels -------------------------------------------------------------------------------
@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", STAGED_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("name", sorted(TERRAINS))
def test_staged_round_emulated(emulated, checker, name, cfg, topo):
    runs = check_terrain(emulated, checker, TERRAINS[name](140), topo, cfg, on_gpu=False)
    # the CPU model runs the tiles in a fixed order: the staged round must queue exactly the tiles the loaded one does
    for k in ("fill_rounds", "fill_tile_visits"):
        assert runs["external_stats"][k] == runs["padded_stats"][k], k
