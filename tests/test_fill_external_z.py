"""The single-GPU fill reads Z straight from the caller's raster (no padded copy) when the width is a multiple of 4 and
the pointer is 16-byte aligned, and builds the first sweep round's W from the lifted start instead of loading it.  Neither
may change a bit: every case is compared as uint32 with the CPU checker and with the padded-copy path
(fill_external_z = 0).  Partial edge tiles (width or height not a multiple of 64) go through the new path; odd widths and a
pointer 4 bytes off alignment take the padded path.

The GPU part runs the dev entry points on torch buffers; the emulated part runs the same checks on the CPU model of the
kernels (tests/emu, fill_use_tma = 0)."""
import ctypes as C
import importlib.util
import os
import sys

import numpy as np
import pytest

import oracle
from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0

# the multigrid / V-cycle configurations of the parity suite, and the plain flood with and without the level schedule
GPU_CONFIGS = [
    {}, {"fill_multigrid": 0}, {"fill_ordered": 0, "fill_multigrid": 0}, {"fill_vcycle": 0}, {"fill_multigrid": 4, "fill_vcycle": 4},
    {"fill_multigrid": 8, "fill_multigrid_min": 256, "fill_vcycle": 2}, {"fill_multigrid": 3, "fill_multigrid_min": 128, "fill_vcycle": 0},
    {"fill_multigrid": 8, "fill_multigrid_min": 32, "fill_vcycle": 1}, {"fill_multigrid": 4, "fill_multigrid_min": 32, "fill_vcycle": 2},
    {"fill_use_tma": 0}, {"fill_use_tma": 0, "fill_multigrid": 0},
]
# heights are not multiples of 64; widths: multiple of 64, multiple of 4 only, odd (padded path)
GPU_SHAPES = [(1100, 1088), (1030, 1036), (1025, 1027)]

EMU_CONFIGS = [
    {"fill_multigrid": 0}, {"fill_ordered": 0, "fill_multigrid": 0}, {"fill_multigrid": 4, "fill_multigrid_min": 32, "fill_vcycle": 2},
    {"fill_multigrid": 8, "fill_multigrid_min": 32, "fill_vcycle": 1}, {"fill_multigrid": 3, "fill_multigrid_min": 32, "fill_vcycle": 0},
]
# (90, 708): 11 tiles across, so the level schedule (and its histogram of Z) is active with fill_multigrid = 0
EMU_SHAPES = [(150, 256), (130, 300), (140, 301), (90, 708)]


def _cfg_id(cfg):
    return ",".join(f"{k}={v}" for k, v in cfg.items()) or "defaults"


def _dem(shape):
    h, w = shape
    dem = oracle.fbm_terrain(h, w, seed=h + w, quantum=0.5)
    dem[h // 4: h // 4 + h // 8, w // 3: w // 3 + w // 6] = ND
    return dem


_expected = {}


def expected_fill(checker, shape, topo):
    key = (shape, topo)
    if key not in _expected:
        dem = _dem(shape)
        _expected[key] = checker.fill_depressions(dem) if topo == "D8" else checker.fill_depressions(dem, "fill_d4")
    return _expected[key]


def fill_dev(L, dem, topo, offset, on_gpu):
    """dev entry point on a buffer whose first cell lies `offset` floats past a 16-byte boundary"""
    h, w = dem.shape
    fn = L.rdb200_dev_fill_depressions_d8_f32 if topo == "D8" else L.rdb200_dev_fill_depressions_d4_f32
    if on_gpu:
        import torch
        buf = torch.empty(h * w + 4, dtype=torch.float32, device="cuda")  # (allocations are 512-byte aligned)
        v = buf[offset: offset + h * w]
        v.copy_(torch.from_numpy(np.ascontiguousarray(dem).ravel()))
        torch.cuda.synchronize()
        _lib.check(fn(v.data_ptr(), w, h))
        torch.cuda.synchronize()
        return v.cpu().numpy().reshape(h, w)
    buf = np.empty(h * w + 8, np.float32)  # the CPU model's device pointers are host pointers
    start = ((-buf.ctypes.data) % 16) // 4 + offset
    v = buf[start: start + h * w]
    v[:] = dem.ravel()
    _lib.check(fn(v.ctypes.data, w, h))
    return v.reshape(h, w).copy()


def check_paths(L, checker, shape, topo, cfg, on_gpu):
    dem = _dem(shape)
    expected = expected_fill(checker, shape, topo).view(np.uint32)
    runs = {}
    try:
        for name, ext, offset in (("external", 1, 0), ("padded", 0, 0), ("misaligned", 1, 1)):
            _lib.reset_params()
            if not on_gpu:
                _lib.set_param("fill_use_tma", 0)
            for k, v in cfg.items():
                _lib.set_param(k, v)
            _lib.set_param("fill_external_z", ext)
            runs[name] = fill_dev(L, dem, topo, offset, on_gpu)
            runs[name + "_stats"] = _lib.stats()
    finally:
        _lib.reset_params()
        if not on_gpu:
            _lib.set_param("fill_use_tma", 0)
    for name in ("external", "padded", "misaligned"):
        got = runs[name].view(np.uint32)
        assert np.array_equal(got, expected), f"{name}: {(got != expected).sum()} cells differ from the checker"
    return runs


# ---- on the H100 ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg", GPU_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("shape", GPU_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_d8_fill_external_z_gpu(checker, shape, cfg):
    check_paths(_lib.lib(), checker, shape, "D8", cfg, on_gpu=True)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [{}, {"fill_multigrid": 0}, {"fill_multigrid": 4, "fill_multigrid_min": 128, "fill_vcycle": 2}],
                         ids=_cfg_id)
@pytest.mark.parametrize("shape", GPU_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_d4_fill_external_z_gpu(checker, shape, cfg):
    check_paths(_lib.lib(), checker, shape, "D4", cfg, on_gpu=True)


# ---- on the CPU model of the kernels -------------------------------------------------------------------------------
def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def emu_lib():
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    build_emu = _load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
    L = C.CDLL(str(build_emu.build()))
    assert L.rdb200_emulated() == 1
    for name, argtypes in _lib.SIGNATURES.items():
        f = getattr(L, name)
        f.argtypes = argtypes
        f.restype = C.c_int
    L.rdb200_last_error.restype = C.c_char_p
    L.rdb200_last_error.argtypes = []
    return L


@pytest.fixture()
def emulated(emu_lib, monkeypatch):
    """Point the Python layer at the emulation for ONE test (TMA / mbarrier PTX is not emulated: fill_use_tma = 0)."""
    monkeypatch.setattr(_lib, "_lib", emu_lib)
    _lib.init(0)
    _lib.set_param("fill_use_tma", 0)
    yield emu_lib
    _lib.reset_params()


@pytest.mark.parametrize("cfg", EMU_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("shape", EMU_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_d8_fill_external_z_emulated(emulated, checker, shape, cfg):
    runs = check_paths(emulated, checker, shape, "D8", cfg, on_gpu=False)
    # the CPU model runs the tiles in a fixed order, so both paths queue the same tiles round for round (a staged tile
    # reads the apron of the neighbours already visited in its round from Wp, as a load would)
    for k in ("fill_rounds", "fill_tile_visits"):
        assert runs["external_stats"][k] == runs["padded_stats"][k], k


@pytest.mark.parametrize("cfg", EMU_CONFIGS[:3], ids=_cfg_id)
@pytest.mark.parametrize("shape", EMU_SHAPES[:3], ids=lambda s: f"{s[0]}x{s[1]}")
def test_d4_fill_external_z_emulated(emulated, checker, shape, cfg):
    check_paths(emulated, checker, shape, "D4", cfg, on_gpu=False)


def test_emulated_shapes_cover_both_paths():
    """The shapes above put partial edge tiles through the external path and an odd width through the padded one."""
    widths = [w for _, w in EMU_SHAPES + GPU_SHAPES]
    heights = [h for h, _ in EMU_SHAPES + GPU_SHAPES]
    assert any(w % 64 == 0 for w in widths) and any(w % 4 == 0 and w % 64 for w in widths) and any(w % 2 for w in widths)
    assert all(h % 64 for h in heights)
