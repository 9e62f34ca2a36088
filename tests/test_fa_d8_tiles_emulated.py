"""The tile-by-tile unit-weight D8 accumulation (csrc/accum.cu, fa_d8_tiles) on the CPU model of the kernels
(tests/emu): the cases of test_gpu_fa_d8_tiles.py, bit for bit against the checker.  Also the row-band path's fused
preparation across its 1016-column block seams, which the single-GPU path no longer runs."""
import importlib.util
import os

import numpy as np
import pytest

import oracle
from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_ek = _load_module("emulated_kernel_fixtures", os.path.join(HERE, "test_emulated_kernels.py"))
emu_lib, emulated, band_drivers = _ek.emu_lib, _ek.emulated, _ek.band_drivers
tiles = _load_module("fa_d8_tile_cases", os.path.join(HERE, "test_gpu_fa_d8_tiles.py"))


@pytest.fixture(scope="module")
def tile_cases(checker):
    return dict(tiles.cases(checker))


@pytest.mark.parametrize("name", [f"edge{s}" for s in tiles.tile_edge_shapes()] + [
    "nodata_corners", "tilted_plane", "serpentine_x", "serpentine_y", "all_flat", "all_nodata", "flat_resolved_fbm"])
def test_tile_seam_cases(emulated, checker, tile_cases, name):
    tiles.check(checker, tile_cases[name])


def test_serpentine_reenters_the_same_tile(checker):
    """The serpentine case really is one path that leaves tile column 0 and comes back into it again and again."""
    dem = tiles.serpentine()
    dirs = checker.d8_flow_directions(dem, tiles.ND)
    dx = np.array([0, -1, -1, 0, 1, 1, 1, 0, -1])
    dy = np.array([0, 0, -1, -1, -1, 0, 1, 1, 1])
    y, x, crossings = 4, tiles.T - 26, 0
    while dirs[y, x] != 0:
        ny, nx = y + dy[dirs[y, x]], x + dx[dirs[y, x]]
        crossings += (x < tiles.T) != (nx < tiles.T)
        y, x = ny, nx
    assert crossings > 50


@pytest.mark.parametrize("lanes", [1, 0])
def test_band_preparation_block_seams(band_drivers, checker, lanes):
    """Row bands keep fa_d8_prep_rolling_kernel, whose blocks own 1016 columns and 64 rows: two bands over a raster
    two blocks wide, with NoData across a block seam."""
    nd = -9999.0
    _lib.set_param("accum_walk_lanes", lanes)
    dem = oracle.fbm_terrain(133, 2040, seed=43, quantum=0.5)
    dem[60:70, 1010:1030] = nd
    resolved = checker.resolve_flats(checker.fill_depressions(dem), nd)
    got, _ = band_drivers.emulate_fa_bands(resolved, 2, nd, False)
    assert np.array_equal(got, checker.fa_d8(resolved, nd))
