"""The fill wakes a neighbouring tile only when a changed tile edge can lower one of that tile's cells (the wake test of
fill_sweep_kernel, switched off with fill_wake_filter = 0).  It may not change a bit: every case runs with the test on
and off, in place and in the padded layout (fill_external_z = 0), for D8 and D4, and is compared as uint32 with the CPU
checker:
  * the staged round's terrains: a diagonal staircase, a 1-cell serpentine, valleys that drain only through tile edges
    and corners;
  * partial tiles (widths and heights that are not multiples of 64);
  * lakes whose level is set by a sill cell on a tile edge, and a lake whose only way out crosses a tile corner (a
    diagonal step from one tile's corner cell to its diagonal neighbour's: D8 drains it there, D4 cannot).
With the plain start (fill_multigrid = 0) every tile starts at +inf and is only ever visited because a neighbour woke
it, so a wake the test drops wrongly leaves cells too high; with a coarse level the staged first round runs, whose
neighbours are still being built while a tile tests them.  On the CPU model (one tile after another) the in-place and
the padded layout must queue the same tiles with the test on, as they do with it off."""
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
_sr = _load_module("fill_staged_round_checks", os.path.join(HERE, "test_fill_staged_round.py"))
_ip = _load_module("fill_in_place_checks", os.path.join(HERE, "test_fill_in_place.py"))
emu_lib, emulated = _ez.emu_lib, _ez.emulated


def edge_lakes(n, seed):
    """Walls everywhere but two lakes.  Lake A (tile column 0) spills over a 3-cell sill on the tile column's last
    column into a channel in the next tile column; lake B (tile row 1) over a sill on its tile row's last row into the
    tile row below.  Both channels fall to the border.  The sills set both lakes' level, under D8 and D4 alike."""
    rng = np.random.default_rng(seed)
    dem = np.full((n, n), WALL, np.float32)
    # lake A: rows 70..120, columns 10..63; sill at rows 94..96 of column 63; channel along row 95 to the east border
    dem[70:121, 10:64] = rng.uniform(10, 20, (51, 54))
    dem[94:97, 63] = 25.0
    dem[95, 64:n] = np.linspace(15, 1, n - 64)
    # lake B: rows 130..191, columns 100..170; sill at columns 139..141 of row 191; channel down column 140 to the south
    dem[130:192, 100:171] = rng.uniform(10, 20, (62, 71))
    dem[191, 139:142] = 30.0
    dem[192:n, 140] = np.linspace(15, 1, n - 192)
    return dem


def corner_lake(n, seed):
    """Walls everywhere but a lake in tile (0, 0) whose sill is its corner cell (63, 63) and a channel that starts at
    the diagonal neighbour's corner cell (64, 64) and runs down column 64 to the south border: the only way out is the
    diagonal step across the tile corner.  D8 fills the lake to the sill; D4 leaves it walled in."""
    rng = np.random.default_rng(seed)
    dem = np.full((n, n), WALL, np.float32)
    dem[10:64, 10:64] = rng.uniform(10, 20, (54, 54))
    dem[63, 63] = 25.0
    dem[64:n, 64] = np.linspace(15, 1, n - 64)
    return dem


TERRAINS = dict(_sr.TERRAINS)
TERRAINS["edge_lakes"] = lambda n: edge_lakes(max(n, 256), 11)
TERRAINS["corner_lake"] = lambda n: corner_lake(max(n, 256), 12)
GPU_SIZES = dict(_sr.GPU_SIZES, edge_lakes=1100, corner_lake=1100)
PLAIN = {"fill_multigrid": 0}
EMU_CONFIGS = [PLAIN, _sr.STAGED_CONFIGS[0]]
GPU_CONFIGS = [{}, PLAIN, {"fill_use_tma": 0}] + _sr.STAGED_CONFIGS[:2]


def _cfg_id(cfg):
    return ",".join(f"{k}={v}" for k, v in cfg.items()) or "defaults"


def run_fill(L, dem, topo, cfg, ext, wake, on_gpu):
    try:
        _lib.reset_params()
        if not on_gpu:
            _lib.set_param("fill_use_tma", 0)
        for k, v in cfg.items():
            _lib.set_param(k, v)
        _lib.set_param("fill_external_z", ext)
        _lib.set_param("fill_wake_filter", wake)
        out = _ez.fill_dev(L, dem, topo, 0, on_gpu)
        return out, _lib.stats()
    finally:
        _lib.reset_params()
        if not on_gpu:
            _lib.set_param("fill_use_tma", 0)


def check_wake_filter(L, checker, dem, topo, cfg, on_gpu):
    """in place and padded, wake test on and off: all four equal to the checker; returns their stats"""
    expected = (checker.fill_depressions(dem) if topo == "D8" else checker.fill_depressions(dem, "fill_d4")).view(np.uint32)
    stats = {}
    for layout, ext in (("in_place", 1), ("padded", 0)):
        for wake in (1, 0):
            got, stats[(layout, wake)] = run_fill(L, dem, topo, cfg, ext, wake, on_gpu)
            got = got.view(np.uint32)
            assert np.array_equal(got, expected), \
                f"{layout}, fill_wake_filter={wake}: {(got != expected).sum()} cells differ from the checker"
    return stats


def test_terrains_are_what_they_say(checker):
    e = TERRAINS["edge_lakes"](256)
    for topo in (None, "fill_d4"):
        f = checker.fill_depressions(e, topo)
        assert (f[70:121, 10:63] == np.float32(25)).all() and (f[130:191, 100:171] == np.float32(30)).all()
    c = TERRAINS["corner_lake"](256)
    assert (checker.fill_depressions(c)[10:63, 10:63] == np.float32(25)).all()
    assert (checker.fill_depressions(c, "fill_d4")[10:63, 10:63] == np.float32(WALL)).all()
    # the sills and the corner cells sit on tile edges (column 63, row 191, cells (63, 63) / (64, 64))
    assert e[95, 63] == 25 and e[95, 64] < 25 and e[191, 140] == 30 and e[192, 140] < 30
    assert c[63, 63] == 25 and c[64, 64] < 25 and c[63, 64] == c[64, 63] == WALL


# ---- on the H100 ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", GPU_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("name", sorted(TERRAINS))
def test_wake_filter_terrains_gpu(checker, name, cfg, topo):
    check_wake_filter(_lib.lib(), checker, TERRAINS[name](GPU_SIZES[name]), topo, cfg, on_gpu=True)


@pytest.mark.gpu
@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", [{}, PLAIN], ids=_cfg_id)
@pytest.mark.parametrize("shape", _ip.GPU_TILE_SHAPES, ids=_ip._shape_id)
def test_wake_filter_partial_tiles_gpu(checker, shape, cfg, topo):
    check_wake_filter(_lib.lib(), checker, _ez._dem(shape), topo, cfg, on_gpu=True)


@pytest.mark.gpu
@pytest.mark.parametrize("topo", ["D8", "D4"])
def test_wake_filter_visits_fbm_gpu(topo):
    """On the benchmark's terrain at 4096 x 4096 the test leaves the result as it is and takes visits away."""
    import torch
    L = _lib.lib()
    n = 4096
    dem = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.check(L.rdb200_dev_generate_fbm_f32(dem.data_ptr(), n, n, 0, 42, 12, 0.0))
    fn = L.rdb200_dev_fill_depressions_d8_f32 if topo == "D8" else L.rdb200_dev_fill_depressions_d4_f32
    out, visits = {}, {}
    try:
        for wake in (1, 0):
            _lib.reset_params()
            _lib.set_param("fill_wake_filter", wake)
            w = dem.clone()
            _lib.check(fn(w.data_ptr(), n, n))
            torch.cuda.synchronize()
            out[wake], visits[wake] = w, _lib.stats()["fill_tile_visits"]
    finally:
        _lib.reset_params()
    assert torch.equal(out[1].view(torch.int32), out[0].view(torch.int32))
    assert visits[1] <= visits[0], visits


# ---- on the CPU model of the kernels -------------------------------------------------------------------------------
@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", EMU_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("name", sorted(TERRAINS))
def test_wake_filter_terrains_emulated(emulated, checker, name, cfg, topo):
    stats = check_wake_filter(emulated, checker, TERRAINS[name](140), topo, cfg, on_gpu=False)
    for wake in (1, 0):
        for k in ("fill_rounds", "fill_tile_visits"):
            assert stats[("in_place", wake)][k] == stats[("padded", wake)][k], (k, wake)


@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("shape", [(129, 100), (127, 132)], ids=_ip._shape_id)
def test_wake_filter_partial_tiles_emulated(emulated, checker, shape, topo):
    stats = check_wake_filter(emulated, checker, _ez._dem(shape), topo, PLAIN, on_gpu=False)
    for wake in (1, 0):
        assert stats[("in_place", wake)]["fill_tile_visits"] == stats[("padded", wake)]["fill_tile_visits"]


@pytest.mark.parametrize("topo", ["D8", "D4"])
def test_wake_filter_drops_visits_emulated(emulated, checker, topo):
    """an fBm raster of 5 x 5 tiles with a coarse level: the test takes visits away"""
    stats = check_wake_filter(emulated, checker, _ez._dem((320, 320)), topo, _sr.STAGED_CONFIGS[0], on_gpu=False)
    assert stats[("in_place", 1)]["fill_tile_visits"] < stats[("in_place", 0)]["fill_tile_visits"], stats
