"""The epsilon fill's C ABI (rdb200_fill_depressions_epsilon_d8/_d4_f32 and their rdb200_dev_ twins) on the CPU fiber model
of tests/emu, whose "device memory" is host memory: the engine's fill_sweep_kernel<2> equals the C restatement
(oracle/epsilon_fill.c) bit for bit, the sign of a zero aside, on fBm and quantised fBm, the Beauford crop, degenerate
shapes, shapes one cell either side of a 64 x 64 tile edge, mazes and the special-value fixtures; the in-place layout
(width a multiple of 4) and the padded one both run.  A plain fill of the result changes nothing.  A null raster or a
zero width fails with the argument check's message before any stage runs."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

import oracle
from oracle import epsilon_fill as EF

HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0
TOPOS = ("D8", "D4")


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_ek = _load_module("emulated_kernel_fixtures", os.path.join(HERE, "test_emulated_kernels.py"))
emu_lib = _ek.emu_lib
T = _load_module("epsilon_fill_cpu", os.path.join(HERE, "test_epsilon_fill_cpu.py"))


@pytest.fixture()
def L(emu_lib):
    assert emu_lib.rdb200_init(0) == 0
    assert emu_lib.rdb200_set_param(b"fill_use_tma", 0) == 0  # TMA / mbarrier PTX is not emulated
    yield emu_lib
    emu_lib.rdb200_set_param(b"reset_defaults", 1)


def gpu_eps(L, z, nd, topology, device=False):
    out = np.ascontiguousarray(z, np.float32).copy()
    h, w = out.shape
    name = f"rdb200_{'dev_' if device else ''}fill_depressions_epsilon_{topology.lower()}_f32"
    assert getattr(L, name)(out.ctypes.data, w, h, nd) == 0, L.rdb200_last_error()
    return out


def check(L, z, nd):
    for topology in TOPOS:
        got = gpu_eps(L, z, nd, topology)
        want = EF.port().fill(z, nd, topology)
        assert T.same_surface(got, want), f"{topology}: {np.count_nonzero(got != want)} cells differ"


SHAPES = [(1, 1), (1, 7), (2, 2), (3, 3), (3, 64), (5, 1), (4, 130), (63, 64), (64, 65), (65, 63), (127, 129), (129, 128)]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{h}x{w}" for h, w in SHAPES])
def test_shapes(L, shape):
    h, w = shape
    z = oracle.fbm_terrain(h, w, seed=h * 1000 + w, quantum=0.5)
    if h > 4 and w > 4:
        z[h // 2, w // 2] -= 300.0  # a pit
    check(L, z, ND)


@pytest.mark.parametrize("q", [None, 0.5, 20.0])
def test_fbm(L, q):
    check(L, oracle.fbm_terrain(150, 220, seed=3, quantum=q), ND)  # (220: padded layout)
    check(L, oracle.fbm_terrain(131, 196, seed=4, quantum=q), ND)  # (196: in place)


def test_beauford_crop(L, golden):
    g = golden["beauford_crop"]
    check(L, g["dem"], float(g["nodata"]))


@pytest.mark.parametrize("name", sorted(T.CASES))
def test_fixtures(L, name):
    z, nd = T.case(name)
    check(L, z, nd)


def test_device_twin_and_plain_fill_after(L):
    z = oracle.fbm_terrain(97, 132, seed=8, quantum=1.0)
    for topology in TOPOS:
        host = gpu_eps(L, z, ND, topology)
        dev = gpu_eps(L, z, ND, topology, device=True)
        assert np.array_equal(host.view(np.uint32), dev.view(np.uint32))
        again = host.copy()
        assert getattr(L, f"rdb200_fill_depressions_{topology.lower()}_f32")(again.ctypes.data, 132, 97) == 0
        assert np.array_equal(again.view(np.uint32), host.view(np.uint32))


@pytest.mark.parametrize("entry", ["rdb200_fill_depressions_epsilon_d8_f32", "rdb200_fill_depressions_epsilon_d4_f32",
                                   "rdb200_dev_fill_depressions_epsilon_d8_f32", "rdb200_dev_fill_depressions_epsilon_d4_f32"])
def test_null_dem_and_zero_width_fail_with_their_message(L, entry):
    fn = getattr(L, entry)
    assert fn(None, 5, 4, ND) == 1 and L.rdb200_last_error() == b"fill_depressions_epsilon: null dem"
    z = np.zeros((4, 5), np.float32)
    assert fn(z.ctypes.data, 0, 4, ND) == 1
    assert L.rdb200_last_error() == b"raster dimensions must be positive (got 0 x 4)"
