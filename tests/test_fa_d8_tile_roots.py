"""Unit-weight D8 by 64 x 64 tiles (csrc/accum.cu, fa_d8_tiles) on two tiles that stress how the first pass finds each
cell's root, the last in-tile cell on its path: one path of about 2000 cells that never leaves its tile, so that pointer
jumping runs its full 11-12 rounds, and a tile whose 4096 cells all leave through one exit cell, so that every cell
counts towards the same exit.  Bit for bit against the CPU checker, on the GPU and on the CPU model of the kernels."""
import importlib.util
import os

import numpy as np
import pytest

import oracle

HERE = os.path.dirname(os.path.abspath(__file__))


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_ek = _load_module("emulated_kernel_fixtures", os.path.join(HERE, "test_emulated_kernels.py"))
emu_lib, emulated = _ek.emu_lib, _ek.emulated
tiles = _load_module("fa_d8_tile_cases", os.path.join(HERE, "test_gpu_fa_d8_tiles.py"))
T, ND = tiles.T, tiles.ND
DX = np.array([0, -1, -1, 0, 1, 1, 1, 0, -1])
DY = np.array([0, 0, -1, -1, -1, 0, 1, 1, 1])


def serpentine_in_one_tile(seed=17):
    """A channel that winds through tile (1, 1) of a 3 x 3 tile raster, rows 2 apart, inside high ground that drains
    into it; it ends in a pit inside the tile."""
    dem = (500.0 + oracle.fbm_terrain(3 * T, 3 * T, seed=seed) * 0.01).astype(np.float32)
    path = []
    rows = list(range(T + 1, 2 * T - 1, 2))
    for j, y in enumerate(rows):
        xs = list(range(T + 1, 2 * T - 1)) if j % 2 == 0 else list(range(2 * T - 2, T, -1))
        path += [(y, x) for x in xs]
        if y != rows[-1]:
            path.append((y + 1, xs[-1]))
    for i, (py, px) in enumerate(path):
        dem[py, px] = 100.0 - 0.01 * i
    return dem


def one_exit_tile(seed=19):
    """Tile (1, 1) of a 3 x 3 tile raster is a cone whose lowest cell is its bottom-right corner; the corner drains
    diagonally into a channel through tile (2, 2), the only neighbour it shares with no other cell of the tile.  The
    ground around the tile is higher and drains into it."""
    rng = np.random.default_rng(seed)
    dem = (3000.0 + rng.uniform(0, 50, (3 * T, 3 * T))).astype(np.float32)
    yy, xx = np.mgrid[T:2 * T, T:2 * T].astype(np.float64)
    dem[T:2 * T, T:2 * T] = (1000.0 + np.hypot(yy - (2 * T - 1), xx - (2 * T - 1))).astype(np.float32)
    for k in range(T):
        dem[2 * T + k, 2 * T + k] = 500.0 - k
    return dem


CASES = {"serpentine_in_one_tile": serpentine_in_one_tile, "one_exit_tile": one_exit_tile}


def in_tile_path(dirs, y, x):
    """The cells of (y, x)'s path up to the last one inside its tile."""
    ty, tx, out = y // T, x // T, [(y, x)]
    while dirs[y, x] != 0:
        ny, nx = y + DY[dirs[y, x]], x + DX[dirs[y, x]]
        if (ny // T, nx // T) != (ty, tx):
            break
        y, x = ny, nx
        out.append((y, x))
    return out


def test_serpentine_fills_one_tile(checker):
    """The case really has an in-tile path longer than 2^10 cells that ends inside the tile."""
    dirs = checker.d8_flow_directions(serpentine_in_one_tile(), ND)
    path = in_tile_path(dirs, T + 1, T + 1)
    assert len(path) > 1800
    assert dirs[path[-1]] == 0


def test_one_exit_tile_drains_through_its_corner(checker):
    """Every cell of tile (1, 1) has the tile's corner as its last in-tile cell, and the corner leaves the tile."""
    dirs = checker.d8_flow_directions(one_exit_tile(), ND)
    corner = (2 * T - 1, 2 * T - 1)
    assert dirs[corner] == 6  # SE, into tile (2, 2)
    assert all(in_tile_path(dirs, y, x)[-1] == corner for y in range(T, 2 * T) for x in range(T, 2 * T))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_in_tile_roots(checker, name):
    tiles.check(checker, CASES[name]())


@pytest.mark.parametrize("name", sorted(CASES))
def test_in_tile_roots_emulated(emulated, checker, name):
    tiles.check(checker, CASES[name]())
