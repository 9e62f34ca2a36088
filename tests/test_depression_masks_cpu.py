"""PitMask / HasDepressions without a GPU.

* The C restatement (oracle/depressions.c: the fill and one compare) equals the unmodified reference templates
  pit_mask<topo> / HasDepressions<topo> (oracle/depressions_shim.cpp) and the stored fixtures, for D8 and D4.
* The strict-pit fast path never says "yes" where the reference says "no".
* The shipped kernels (csrc/depressions.cu: the strict-pit stencil, the fused mask pass, the fill behind them) run on
  the CPU fiber model of tests/emu and reproduce the fixtures, as tests/test_emulated_kernels.py does for the others.
"""
import ctypes as C
import importlib.util
import os
import sys

import numpy as np
import pytest

import oracle
from oracle import depressions
from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "depression_masks_ref.npz")
TOPOS = ("D8", "D4")


def golden_cases():
    g = np.load(GOLDEN)
    names = sorted({k.split("__")[0] for k in g.files if k.endswith("__dem")})
    return g, names


def strict_pit(dem, topology):
    """numpy statement of the fast path: some interior cell strictly below each of its 8 (4) neighbours."""
    d = np.asarray(dem, np.float32)
    if d.shape[0] < 3 or d.shape[1] < 3:
        return False
    c = d[1:-1, 1:-1]
    offs = [(-1, 0), (1, 0), (0, -1), (0, 1)]
    if topology == "D8":
        offs += [(-1, -1), (-1, 1), (1, -1), (1, 1)]
    pit = np.ones(c.shape, bool)
    for dy, dx in offs:
        pit &= c < d[1 + dy:d.shape[0] - 1 + dy, 1 + dx:d.shape[1] - 1 + dx]
    return bool(pit.any())


@pytest.mark.parametrize("topology", TOPOS)
def test_port_equals_fixtures(topology):
    g, names = golden_cases()
    P = depressions.port()
    assert {"testdem1", "beauford", "fbm_q05", "nodata_hole", "no_depressions", "terraced", "row_1xN", "col_Nx1",
            "square_2x2", "all_nodata", "infinities"} <= set(names)
    for name in names:
        dem, nd = g[f"{name}__dem"], float(g[f"{name}__nodata"])
        assert np.array_equal(P.pit_mask(dem, nd, topology), g[f"{name}__mask_{topology}"]), name
        assert P.has_depressions(dem, topology) == bool(g[f"{name}__has_{topology}"]), name


@pytest.mark.parametrize("topology", TOPOS)
def test_port_equals_reference(topology):
    if not depressions.have_ref():
        depressions.build()
    if not depressions.have_ref():
        pytest.skip("reference tree not available")
    R, P = depressions.ref(), depressions.port()
    g, names = golden_cases()
    dems = {name: (g[f"{name}__dem"], float(g[f"{name}__nodata"])) for name in names}
    for seed in range(6):  # random small rasters with NoData, ties and infinities
        rng = np.random.default_rng(seed)
        h, w = rng.integers(1, 40, 2)
        d = np.round(rng.random((h, w)) * 6).astype(np.float32)
        d[rng.random((h, w)) < 0.1] = -9999.0
        d[rng.random((h, w)) < 0.03] = np.inf
        dems[f"random{seed}"] = (d, -9999.0)
    for name, (dem, nd) in dems.items():
        assert np.array_equal(P.pit_mask(dem, nd, topology), R.pit_mask(dem, nd, topology)), name
        assert P.has_depressions(dem, topology) == R.has_depressions(dem, topology), name


@pytest.mark.parametrize("topology", TOPOS)
def test_strict_pit_never_says_yes_when_the_reference_says_no(topology):
    """The fast path's claim, on the fixtures and on random rasters full of ties, NoData and infinities."""
    B = depressions.best()
    g, names = golden_cases()
    dems = [g[f"{name}__dem"] for name in names]
    for seed in range(40):
        rng = np.random.default_rng(100 + seed)
        h, w = rng.integers(3, 24, 2)
        d = np.round(rng.random((h, w)) * rng.integers(1, 5)).astype(np.float32)
        d[rng.random((h, w)) < 0.15] = -9999.0
        d[rng.random((h, w)) < 0.05] = -np.inf if seed % 2 else np.inf
        dems.append(d)
    hits = 0
    for d in dems:
        if strict_pit(d, topology):
            hits += 1
            assert B.has_depressions(d, topology)
    assert hits >= 10  # the claim was exercised
    # ... and the rasters that need the fill have no strict pit
    for name in ("nodata_hole",) + (("no_depressions",) if topology == "D8" else ()):
        assert not strict_pit(g[f"{name}__dem"], topology), name
    assert bool(g[f"nodata_hole__has_{topology}"])


# ---- the shipped kernels on the CPU fiber model ------------------------------------------------------------------------
def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def emu_lib():
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    path = _load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build()
    L = C.CDLL(str(path))
    assert L.rdb200_emulated() == 1
    for name, argtypes in _lib.SIGNATURES.items():
        f = getattr(L, name)
        f.argtypes = argtypes
        f.restype = C.c_int
    L.rdb200_last_error.restype = C.c_char_p
    L.rdb200_last_error.argtypes = []
    L.rdb200_version.restype = C.c_int
    L.rdb200_shutdown.restype = None
    return L


@pytest.fixture()
def emulated(emu_lib, monkeypatch):
    monkeypatch.setattr(_lib, "_lib", emu_lib)
    _lib.init(0)
    _lib.set_param("fill_use_tma", 0)  # TMA / mbarrier PTX is not emulated
    yield emu_lib
    _lib.reset_params()


@pytest.mark.parametrize("topology", TOPOS)
def test_emulated_kernels_equal_fixtures(emulated, topology):
    import richdem_b200 as rd
    g, names = golden_cases()
    for name in names:
        dem, nd = np.ascontiguousarray(g[f"{name}__dem"]), float(g[f"{name}__nodata"])
        before = dem.copy()
        m = rd.PitMask(rd.rdarray(dem, no_data=nd), topology=topology)
        assert m.dtype == np.uint8 and m.no_data == 3
        assert np.array_equal(np.asarray(m), g[f"{name}__mask_{topology}"]), name
        assert rd.HasDepressions(rd.rdarray(dem, no_data=nd), topology=topology) == bool(g[f"{name}__has_{topology}"]), name
        assert np.array_equal(dem.view(np.uint32), before.view(np.uint32)), name  # the input is not modified


def test_emulated_strict_pit_answers_without_the_fill(emulated):
    import richdem_b200 as rd
    g, _ = golden_cases()
    fbm = np.ascontiguousarray(g["fbm_q05__dem"])
    for topo in TOPOS:
        assert strict_pit(fbm, topo)
        assert rd.HasDepressions(rd.rdarray(fbm, no_data=-9999.0), topology=topo)
        assert _lib.stats()["kernel_launches"] == 1  # the stencil pass alone
        hole = np.ascontiguousarray(g["nodata_hole__dem"])
        assert rd.HasDepressions(rd.rdarray(hole, no_data=-9999.0), topology=topo)
        assert _lib.stats()["kernel_launches"] > 2  # stencil, fill, compare


def test_emulated_unaligned_and_odd_sizes(emulated):
    """The mask pass's scalar path (pointers not 16-byte aligned) and its tail (cells beyond a multiple of 4)."""
    dem = oracle.fbm_terrain(37, 53, seed=5, quantum=0.5)
    dem[5:9, 7:30] = -9999.0
    P = depressions.port()
    buf = np.zeros(dem.size + 1, np.float32)
    d = buf[1:].reshape(dem.shape)
    d[...] = dem
    for topo, fn in (("D8", "rdb200_pit_mask_d8_f32"), ("D4", "rdb200_pit_mask_d4_f32")):
        out = np.zeros(dem.size + 3, np.uint8)
        m = out[3:].reshape(dem.shape)
        _lib.check(getattr(_lib.lib(), fn)(d.ctypes.data, m.ctypes.data, dem.shape[1], dem.shape[0], -9999.0))
        assert np.array_equal(m, P.pit_mask(dem, -9999.0, topo)), topo


def test_argument_validation_matches_fill_depressions():
    import richdem_b200 as rd
    for fn in (rd.PitMask, rd.HasDepressions):
        with pytest.raises(Exception, match="rdarray"):
            fn(np.zeros((4, 4), np.float32))
        with pytest.raises(Exception, match="Unknown topology!"):
            fn(rd.rdarray(np.zeros((4, 4), np.float32), no_data=-1), topology="D6")
        with pytest.raises(Exception, match="float32"):
            fn(rd.rdarray(np.zeros((4, 4), np.float64), no_data=-1))
        with pytest.raises(RuntimeError, match="two dimensions"):
            fn(rd.rdarray(np.zeros((4, 4, 2), np.float32), no_data=-1))
