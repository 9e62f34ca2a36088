"""The single-GPU fill relaxes its water surface in the caller's raster when the width is a multiple of 4 and the pointer
is 16-byte aligned, keeping Z in a compact copy that the first sweep round saves tile by tile (or that the start writes,
for a fill without a coarse level).  It may not change a bit: every case is compared as uint32 with the CPU checker and
with the padded layout (fill_external_z = 0), for D8 and D4:
  * partial tiles: widths that are a multiple of 64, a multiple of 4 only, and 4 more than a multiple of 64 (a last tile
    4 columns wide), heights that are a multiple of 64, one more and one less;
  * layout selection: an odd width and a pointer 4 bytes off alignment take the padded layout; on the CPU model the
    launch count shows which one ran (the padded layout copies W out at the end, the in-place one does not), on the
    GPU the device scratch a call takes (one compact Z copy against padded Z and W);
  * staying inside the raster: on the CPU model the raster ends at a page that may not be touched, at heights that are
    not multiples of 64, so a read past its end faults;
  * coarse levels: V-cycle configurations whose coarse rasters are multiples of 4 wide, so the coarse fill and the
    coarse solver run in place, with restriction and prolongation between in-place levels, and a plain start with the
    level schedule active;
  * aliasing: a steep valley two tiles wide, where a tile reads the edge of a neighbour that finished the first round
    before it (from the raster the neighbour has just written its W to).

The GPU part runs the dev entry points on torch buffers; the emulated part runs the same checks on the CPU model of the
kernels (tests/emu, fill_use_tma = 0)."""
import ctypes as C
import importlib.util
import mmap
import os

import numpy as np
import pytest

from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_ez = _load_module("fill_external_z_checks", os.path.join(HERE, "test_fill_external_z.py"))
_sr = _load_module("fill_staged_round_checks", os.path.join(HERE, "test_fill_staged_round.py"))
emu_lib, emulated = _ez.emu_lib, _ez.emulated

# coarse levels: pools 4 and 8 over the shapes below give coarse rasters 4k wide (in place) down to fill_multigrid_min
VCYCLE_CONFIGS = [{"fill_multigrid": 4, "fill_multigrid_min": 32, "fill_vcycle": 2},
                  {"fill_multigrid": 8, "fill_multigrid_min": 32, "fill_vcycle": 1},
                  {"fill_multigrid": 4, "fill_multigrid_min": 128, "fill_vcycle": 1}]
PLAIN = {"fill_multigrid": 0}  # non-lifted start (with the level schedule where the raster is wide enough)


def _cfg_id(cfg):
    return ",".join(f"{k}={v}" for k, v in cfg.items()) or "defaults"


def _shape_id(s):
    return f"{s[0]}x{s[1]}"


def run_fill(L, dem, topo, cfg, ext, offset, on_gpu):
    try:
        _lib.reset_params()
        if not on_gpu:
            _lib.set_param("fill_use_tma", 0)
        for k, v in cfg.items():
            _lib.set_param(k, v)
        _lib.set_param("fill_external_z", ext)
        out = _ez.fill_dev(L, dem, topo, offset, on_gpu)
        return out, _lib.stats()
    finally:
        _lib.reset_params()
        if not on_gpu:
            _lib.set_param("fill_use_tma", 0)


def check_in_place(L, checker, dem, topo, cfg, on_gpu, misaligned=False):
    """in place (when the raster allows it), padded and, optionally, 4 bytes off alignment: all equal to the checker"""
    expected = (checker.fill_depressions(dem) if topo == "D8" else checker.fill_depressions(dem, "fill_d4")).view(np.uint32)
    variants = [("in_place", 1, 0), ("padded", 0, 0)] + ([("misaligned", 1, 1)] if misaligned else [])
    stats = {}
    for name, ext, offset in variants:
        got, stats[name] = run_fill(L, dem, topo, cfg, ext, offset, on_gpu)
        got = got.view(np.uint32)
        assert np.array_equal(got, expected), f"{name}: {(got != expected).sum()} cells differ from the checker"
    return stats


# partial tiles: (height, width) pairs that cover every width with every height
EMU_TILE_SHAPES = [(h, w) for h in (128, 129, 127) for w in (128, 100, 132)]
GPU_TILE_SHAPES = [(h, w) for h in (1088, 1089, 1087) for w in (1088, 1036, 1092)]
# coarse levels: widths whose pooled widths (4 and 8) are multiples of 4
EMU_VCYCLE_SHAPES = [(129, 192), (127, 256), (150, 160)]
GPU_VCYCLE_SHAPES = [(1089, 1088), (1087, 1152)]


def test_shapes_cover_the_cases():
    for shapes in (EMU_TILE_SHAPES, GPU_TILE_SHAPES):
        ws = {w for _, w in shapes}
        hs = {h for h, _ in shapes}
        assert any(w % 64 == 0 for w in ws) and any(w % 4 == 0 and w % 64 not in (0, 4) for w in ws)
        assert any(w % 64 == 4 for w in ws) and all(w % 4 == 0 for w in ws)
        assert {h % 64 for h in hs} == {0, 1, 63}
    for h, w in EMU_VCYCLE_SHAPES + GPU_VCYCLE_SHAPES:
        assert (w // 4) % 4 == 0 and (w // 8) % 4 == 0


# ---- on the H100 ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", [{}, PLAIN, {"fill_use_tma": 0}], ids=_cfg_id)
@pytest.mark.parametrize("shape", GPU_TILE_SHAPES, ids=_shape_id)
def test_in_place_partial_tiles_gpu(checker, shape, cfg, topo):
    check_in_place(_lib.lib(), checker, _ez._dem(shape), topo, cfg, on_gpu=True)


@pytest.mark.gpu
@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", [{}] + VCYCLE_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("shape", GPU_VCYCLE_SHAPES, ids=_shape_id)
def test_in_place_coarse_levels_gpu(checker, shape, cfg, topo):
    check_in_place(_lib.lib(), checker, _ez._dem(shape), topo, cfg, on_gpu=True)


@pytest.mark.gpu
@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", [{}, PLAIN], ids=_cfg_id)
@pytest.mark.parametrize("shape", [(1089, 1036), (1087, 1027)], ids=_shape_id)
def test_padded_layout_selection_gpu(checker, shape, cfg, topo):
    """a pointer 4 bytes off alignment (and an odd width) falls back to the padded layout"""
    check_in_place(_lib.lib(), checker, _ez._dem(shape), topo, cfg, on_gpu=True, misaligned=True)


def gpu_fill_scratch_mib(dem, ext, offset):
    """device memory (MiB) the D8 fill takes from a trimmed workspace, on a buffer `offset` floats past alignment"""
    import torch
    L = _lib.lib()
    h, w = dem.shape
    buf = torch.empty(h * w + 4, dtype=torch.float32, device="cuda")
    v = buf[offset: offset + h * w]
    v.copy_(torch.from_numpy(np.ascontiguousarray(dem).ravel()))
    try:
        _lib.set_param("fill_external_z", ext)
        _lib.set_param("trim_workspace", 1)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        _lib.check(L.rdb200_dev_fill_depressions_d8_f32(v.data_ptr(), w, h))
        torch.cuda.synchronize()
        free1 = torch.cuda.mem_get_info()[0]
    finally:
        _lib.reset_params()
    return (free0 - free1) / 2 ** 20


@pytest.mark.gpu
def test_layout_selection_gpu():
    """The in-place layout keeps one compact Z copy (16 MiB here) where the padded one keeps padded Z and W (34 MiB): the
    scratch a call takes shows which layout ran.  A pointer 4 bytes off alignment and an odd width take the padded one."""
    aligned = _ez._dem((2049, 2052))
    gpu_fill_scratch_mib(aligned, 1, 0)  # (whatever the library sets up once is not part of a call's scratch)
    in_place = gpu_fill_scratch_mib(aligned, 1, 0)
    padded = gpu_fill_scratch_mib(aligned, 0, 0)
    misaligned = gpu_fill_scratch_mib(aligned, 1, 1)
    odd = gpu_fill_scratch_mib(_ez._dem((2049, 2051)), 1, 0)
    assert padded > in_place + 12, (in_place, padded)
    assert misaligned > in_place + 12 and odd > in_place + 12, (in_place, misaligned, odd)


@pytest.mark.gpu
@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", [{}] + _sr.STAGED_CONFIGS[:2], ids=_cfg_id)
def test_in_place_steep_valley_two_tiles_wide_gpu(checker, cfg, topo):
    dem = _sr.diagonal_valley(1100, 128, 6)
    check_in_place(_lib.lib(), checker, dem, topo, {"fill_multigrid_min": 64, **cfg}, on_gpu=True)


# ---- on the CPU model of the kernels -------------------------------------------------------------------------------
@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", [PLAIN, VCYCLE_CONFIGS[0]], ids=_cfg_id)
@pytest.mark.parametrize("shape", EMU_TILE_SHAPES, ids=_shape_id)
def test_in_place_partial_tiles_emulated(emulated, checker, shape, cfg, topo):
    stats = check_in_place(emulated, checker, _ez._dem(shape), topo, cfg, on_gpu=False)
    # the CPU model runs the tiles in a fixed order: both layouts queue the same tiles round for round
    for k in ("fill_rounds", "fill_tile_visits"):
        assert stats["in_place"][k] == stats["padded"][k], k


@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", VCYCLE_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("shape", EMU_VCYCLE_SHAPES, ids=_shape_id)
def test_in_place_coarse_levels_emulated(emulated, checker, shape, cfg, topo):
    stats = check_in_place(emulated, checker, _ez._dem(shape), topo, cfg, on_gpu=False)
    for k in ("fill_rounds", "fill_tile_visits"):
        assert stats["in_place"][k] == stats["padded"][k], k


@pytest.mark.parametrize("topo", ["D8", "D4"])
def test_in_place_level_schedule_emulated(emulated, checker, topo):
    """a plain start with the level schedule active: its histogram reads the compact Z copy, not the raster"""
    stats = check_in_place(emulated, checker, _ez._dem((90, 708)), topo, PLAIN, on_gpu=False)
    for k in ("fill_rounds", "fill_tile_visits"):
        assert stats["in_place"][k] == stats["padded"][k], k


@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("shape", [(129, 132), (127, 131)], ids=_shape_id)
def test_layout_selection_emulated(emulated, checker, shape, topo):
    """The in-place layout saves exactly the final copy (one launch) of a plain fill; a pointer 4 bytes off alignment
    and an odd width take the padded layout, launch for launch what fill_external_z = 0 does."""
    stats = check_in_place(emulated, checker, _ez._dem(shape), topo, {"fill_multigrid": 0, "fill_ordered": 0}, on_gpu=False,
                           misaligned=True)
    launches = {k: v["kernel_launches"] for k, v in stats.items()}
    assert launches["misaligned"] == launches["padded"]
    assert launches["in_place"] == launches["padded"] - (1 if shape[1] % 4 == 0 else 0)


def guarded_raster(h, w):
    """An h x w float32 array of the CPU model whose last cell is followed by a page that may not be touched: a read
    past the end of the raster is a segmentation fault instead of a read of whatever lies there."""
    page = mmap.PAGESIZE
    nbytes = h * w * 4
    total = (nbytes + page - 1) // page * page + page
    m = mmap.mmap(-1, total, prot=mmap.PROT_READ | mmap.PROT_WRITE)
    base = C.addressof(C.c_char.from_buffer(m))
    libc = C.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    libc.mprotect.restype = C.c_int
    assert libc.mprotect(base + total - page, page, 0) == 0, os.strerror(C.get_errno())
    # (w % 4 == 0: the first cell is 16-byte aligned, so the fill works in place)
    return np.frombuffer(m, dtype=np.float32, count=h * w, offset=total - page - nbytes).reshape(h, w)


@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", [PLAIN] + VCYCLE_CONFIGS[:2], ids=_cfg_id)
@pytest.mark.parametrize("shape", [(129, 192), (129, 100), (127, 132), (65, 256)], ids=_shape_id)
def test_in_place_stays_inside_the_raster_emulated(emulated, checker, shape, cfg, topo):
    """The raster ends at a page that may not be touched, with heights that are not multiples of 64: the last tile row
    is partial, and in the staged round its tiles read the apron of neighbours that are done from the raster."""
    h, w = shape
    dem = _ez._dem(shape)
    expected = (checker.fill_depressions(dem) if topo == "D8" else checker.fill_depressions(dem, "fill_d4")).view(np.uint32)
    v = guarded_raster(h, w)
    v[:] = dem
    fn = emulated.rdb200_dev_fill_depressions_d8_f32 if topo == "D8" else emulated.rdb200_dev_fill_depressions_d4_f32
    try:
        for k, val in cfg.items():
            _lib.set_param(k, val)
        _lib.check(fn(v.ctypes.data, w, h))
        stats = _lib.stats()
    finally:
        _lib.reset_params()
        _lib.set_param("fill_use_tma", 0)
    assert np.array_equal(v.view(np.uint32), expected), f"{(v.view(np.uint32) != expected).sum()} cells differ"
    _, padded = run_fill(emulated, dem, topo, cfg, 0, 0, on_gpu=False)
    for k in ("fill_rounds", "fill_tile_visits"):
        assert stats[k] == padded[k], k


@pytest.mark.parametrize("topo", ["D8", "D4"])
@pytest.mark.parametrize("cfg", _sr.STAGED_CONFIGS, ids=_cfg_id)
def test_in_place_steep_valley_two_tiles_wide_emulated(emulated, checker, cfg, topo):
    dem = _sr.diagonal_valley(252, 128, 6)
    stats = check_in_place(emulated, checker, dem, topo, cfg, on_gpu=False)
    for k in ("fill_rounds", "fill_tile_visits"):
        assert stats["in_place"][k] == stats["padded"][k], k
