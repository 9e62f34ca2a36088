"""Unit-weight D8 by 64 x 64 tiles (csrc/accum.cu, fa_d8_tiles): terrains that stress the in-tile sums of the final pass,
which add each cell's sum to the cell 2^r steps down its path in round r.  In-tile paths of 2^k - 1, 2^k and 2^k + 1
cells pin the round in which a pointer stops being exact, a fishbone sends many cells to the same 2^r-ancestor in one
round, and a funnel brings inflow into a tile through many slots whose paths merge before they leave.  Bit for bit
against the CPU checker, on the GPU and on the CPU model of the kernels, with the harness of
tests/test_fa_d8_tile_roots.py."""
import importlib.util
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


roots = _load_module("fa_d8_tile_root_cases", os.path.join(HERE, "test_fa_d8_tile_roots.py"))
emu_lib, emulated = roots.emu_lib, roots.emulated
tiles, in_tile_path = roots.tiles, roots.in_tile_path
T, ND = roots.T, roots.ND


def d8_codes(dem):
    """The flow codes FA_D8 follows (1..8: W, NW, N, NE, E, SE, S, SW; 0: none; 255: NoData): the first strictly lowest
    data neighbour, none on the raster's border.  (d8_flow_directions also points at NoData neighbours.)"""
    h, w = dem.shape
    data = dem != ND
    codes = np.where(data, 0, 255).astype(np.int64)
    lowest = np.where(data, dem, np.inf)
    inner = (slice(1, h - 1), slice(1, w - 1))
    for n in range(1, 9):
        nb = dem[1 + roots.DY[n]:h - 1 + roots.DY[n], 1 + roots.DX[n]:w - 1 + roots.DX[n]]
        take = data[inner] & (nb != ND) & (nb < lowest[inner])
        lowest[inner][take] = nb[take]
        codes[inner][take] = n
    return codes


def snake_cells():
    """Tile (1, 1)'s cells in the order of a path that winds through rows 1, 3, 5, ... of the tile and ends on the
    tile's right edge in row 1.  Rows are joined by one diagonal step through the row between them, so no two cells of
    the path touch unless they are consecutive, and steepest descent along falling values takes exactly this path."""
    rev, going_left, y = [], True, 1
    while y < T - 1:
        xs = range(T - 1 if y == 1 else T - 2, 0, -1) if going_left else range(1, T - 1)
        rev += [(T + y, T + x) for x in xs]
        rev.append((T + y + 1, T if going_left else 2 * T - 1))  # the turn, in column 0 or 63
        going_left = not going_left
        y += 2
    return rev[::-1]


def in_tile_chain(n, exit):
    """A path of n cells through tile (1, 1) of a 3 x 3 tile raster that is NoData elsewhere.  It ends on the tile's
    right edge: in a pit there, or (exit) continuing into tile (2, 1) for 5 more cells."""
    dem = np.full((3 * T, 3 * T), ND, np.float32)
    path = snake_cells()[-n:]
    if exit:
        end_y, end_x = path[-1]
        path += [(end_y, end_x + 1 + i) for i in range(5)]
    for i, (y, x) in enumerate(path):
        dem[y, x] = 5000.0 - i
    return dem


def fishbone(pit, seed=23):
    """A spine along row 32 of tile (1, 1) falls towards column xp: inside the tile (pit), where the spine ends in a
    pit that all 8 neighbours drain into, or in tile (2, 1).  The ground on either side rises away from the spine, more
    steeply than the spine falls, so every spine cell is joined by side branches from the north-west and south-west;
    noise and scattered NoData cells bend and merge the branches, so their lengths are mixed."""
    rng = np.random.default_rng(seed)
    ys = T + 32
    xp = T + 40 if pit else 2 * T + 20
    yy, xx = np.mgrid[0:3 * T, 0:3 * T].astype(np.float64)
    dem = 1000.0 + np.abs(xx - xp) + 2.0 * np.abs(yy - ys) + rng.uniform(0, 1.5, yy.shape) * (yy != ys)
    near_pit = (np.abs(yy - ys) <= 1) & (np.abs(xx - xp) <= 1)
    dem[(rng.uniform(size=yy.shape) < 0.03) & (yy != ys) & ~near_pit] = ND
    return dem.astype(np.float32)


def funnel(seed=29):
    """Everything falls east and, more steeply, towards row 32 of tile (1, 1): flow from tiles (0, 1) and (1, 0) enters
    tile (1, 1) through many slots on its west and north edges, and those paths merge on row 32 before they leave."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:3 * T, 0:3 * T].astype(np.float64)
    return (1000.0 - xx + 3.0 * np.abs(yy - (T + 32)) + rng.uniform(0, 0.5, yy.shape)).astype(np.float32)


CASES = {f"chain{n}_{'exit' if exit else 'pit'}": (lambda n=n, exit=exit: in_tile_chain(n, exit))
         for k in (5, 10) for n in (2 ** k - 1, 2 ** k, 2 ** k + 1) for exit in (False, True)}
CASES.update({"fishbone_pit": lambda: fishbone(True), "fishbone_exit": lambda: fishbone(False), "funnel": funnel})


@pytest.mark.parametrize("n", [31, 32, 33, 1023, 1024, 1025])
@pytest.mark.parametrize("exit", [False, True])
def test_chain_is_one_in_tile_path(n, exit):
    """The chain's source has exactly n cells on its in-tile path, which ends on the tile's right edge: in a pit, or
    leaving the tile."""
    dem = in_tile_chain(n, exit)
    dirs = d8_codes(dem)
    path = in_tile_path(dirs, *snake_cells()[-n])
    assert len(path) == n and path[-1] == (T + 1, 2 * T - 1)
    assert dirs[path[-1]] == (5 if exit else 0)  # E into tile (2, 1), or none
    assert int((dem != ND).sum()) == n + 5 * exit


def test_fishbone_fan_in():
    """Spine cells of the fishbone have 3 donors (the spine and a branch on either side), and its pit all 8."""
    dem = fishbone(True)
    dirs = d8_codes(dem)
    h, w = dirs.shape
    fan_in = np.zeros((h, w), np.int64)
    ys, xs = np.nonzero((dirs >= 1) & (dirs <= 8))
    np.add.at(fan_in, (ys + roots.DY[dirs[ys, xs]], xs + roots.DX[dirs[ys, xs]]), 1)
    spine = fan_in[T + 32, T + 1:T + 40]
    assert (spine >= 2).all() and spine.max() == 3 and fan_in[T + 32, T + 40] == 8


def test_funnel_enters_through_many_slots():
    """At least 20 cells on the west edge of tile (1, 1) are fed from outside it, and their in-tile paths all leave
    the tile at the same cell."""
    dirs = d8_codes(funnel())
    fed, ends = 0, set()
    for y, x in [(T + i, T) for i in range(T)]:
        for n in range(1, 9):
            sy, sx = y - roots.DY[n], x - roots.DX[n]
            if not (T <= sy < 2 * T and T <= sx < 2 * T) and dirs[sy, sx] == n:
                fed += 1
                ends.add(in_tile_path(dirs, y, x)[-1])
                break
    assert fed >= 20 and len(ends) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_in_tile_sums(checker, name):
    tiles.check(checker, CASES[name]())


@pytest.mark.parametrize("name", sorted(CASES))
def test_in_tile_sums_emulated(emulated, checker, name):
    tiles.check(checker, CASES[name]())
