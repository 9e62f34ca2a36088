"""float64 D-infinity, MFD and terrain attributes without a GPU.

* Every new entry point on the CPU fiber model of tests/emu (host libm in place of the device's atan2 / atan / pow)
  against the reference's double templates stored in tests/golden/f64_flowmet_ref.npz, with the D-infinity filter on
  and off.  Per-cell outputs are bit-exact; accumulations keep the float32 path's tolerances (their sums run in another
  order than the reference's serial walk).
* The premise of the GPU's float32 comparison: on a float-exact raster the reference's double D-infinity, D8, D4 and
  terrain attributes equal its float ones; MFD does not, because it subtracts in the elevation type.
* The fixtures' own ground: huge / tiny hold differences outside [2^-500, 2^500], near_tie holds one-ulp ties, and the
  golden file regenerates to the same bits where the reference tree exists.
"""
import ctypes as C
import importlib.util
import os
import sys

import numpy as np
import pytest

from oracle import f64_flowmet as F
from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "f64_flowmet_ref.npz")


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


M = _load_module("make_f64_flowmet", os.path.join(HERE, "golden", "make_f64_flowmet.py"))
G = np.load(GOLDEN)
NAMES = sorted({k.split("/")[0] for k in G.files})


def fixture(name):
    return G[f"{name}/dem"], float(G[f"{name}/nodata"])


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    u = np.uint32 if a.dtype == np.float32 else np.uint64
    return bool(np.all((a.view(u) == b.view(u)) | (np.isnan(a) & np.isnan(b))))


def close(got, ref, rtol):
    got, ref = np.asarray(got), np.asarray(ref)
    with np.errstate(invalid="ignore"):  # inf - inf
        return bool(np.all((got == ref) | (np.abs(got - ref) <= rtol * np.abs(ref)) | (np.isnan(got) & np.isnan(ref))))


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
    return L


@pytest.fixture()
def emulated(emu_lib, monkeypatch):
    monkeypatch.setattr(_lib, "_lib", emu_lib)
    _lib.init(0)
    yield emu_lib
    _lib.reset_params()


METHOD_NAMES = {0: "D8", 1: "Dinf", 2: "D4", 3: "Holmgren", 4: "Freeman"}


def _method(m, x):
    name = METHOD_NAMES[m]
    if m == 3 and x == 1.0:
        return "Quinn", None
    return name, (x if m in (3, 4) else None)


@pytest.mark.parametrize("tfilter", [1, 0])
@pytest.mark.parametrize("name", NAMES)
def test_emulated_entry_points_equal_the_reference(emulated, name, tfilter):
    import richdem_b200 as rd
    from richdem_b200 import f64
    _lib.set_param("flowmet_tarboton_filter", tfilter)
    z, nd = fixture(name)
    h, w = z.shape
    L = _lib.lib()
    dem = lambda: rd.rdarray(z.copy(), no_data=nd, geotransform=[0, M.TA_CELL[0], 0, 0, 0, -M.TA_CELL[1]])  # noqa: E731
    fm_runs, fa_runs, ta_runs = M.runs(name)
    for m, x in fm_runs:
        method, exponent = _method(m, x)
        ref = G[f"{name}/fm{m}_{x}"]
        assert same_bits(np.asarray(f64.FlowProportions(dem(), method, exponent)), ref), (name, m, x)
        p = np.empty((h, w, 9), np.float32)
        _lib.check(L.rdb200_dev_fm_method_f64(m, _lib.ptr(z), _lib.ptr(p), w, h, nd, x))
        assert same_bits(p, ref), (name, m, x, "dev")
    # FA_Tarboton: the fused engine (packed walk, level kernel) and its weighted form
    for packed, rtol in ((1, 5e-7), (0, 1e-9)):
        _lib.set_param("accum_dinf_packed", packed)
        acc = np.empty((h, w))
        _lib.check(L.rdb200_fa_tarboton_f64_f64(_lib.ptr(z), _lib.ptr(acc), w, h, nd, 1))
        assert close(acc, G[f"{name}/fa1_1.0"], rtol), (name, packed)
    if f"{name}/fa1_weighted" in G:
        acc = M.weights(z.shape)
        _lib.check(L.rdb200_fa_tarboton_f64_f64(_lib.ptr(z), _lib.ptr(acc), w, h, nd, 0))
        assert close(acc, G[f"{name}/fa1_weighted"], 1e-9), name
    for m, x in fa_runs:
        ref = G[f"{name}/fa{m}_{x}"]
        props = G[f"{name}/fm{m}_{x}"]
        if np.isnan(props).any():
            # powers that overflow float make inf shares and inf * (1 / inf) = NaN; the reference then lets a NaN share
            # flow (`<= 0` is false) without counting it as a dependency (`> 0` is false).  The generic accumulation
            # drops it, for float32 as for float64: compare with that engine on the reference's own proportions.
            ref = rd.FlowAccumFromProps(rd.rd3array(props, no_data=-2))
        acc = np.ones((h, w))
        _lib.check(L.rdb200_dev_fa_method_f64_f64(m, _lib.ptr(z), _lib.ptr(acc), w, h, nd, x))
        assert close(acc, ref, 1e-6 if m != 1 else 1e-9), (name, m, x, "dev")
        if m != 1:
            acc = np.ones((h, w))
            fn = {3: L.rdb200_fa_holmgren_f64_f64, 4: L.rdb200_fa_freeman_f64_f64}[m]
            _lib.check(fn(_lib.ptr(z), _lib.ptr(acc), w, h, nd, x))
            assert close(acc, ref, 1e-6), (name, m, x)
        method, exponent = _method(m, x)
        got = rd.FlowAccumFromProps(f64.FlowProportions(dem(), method, exponent))
        assert close(got, ref, 1e-6 if m != 1 else 1e-9), (name, m, x, "from props")
    if (3, 1.0) in fa_runs:
        acc = np.ones((h, w))
        _lib.check(L.rdb200_fa_quinn_f64_f64(_lib.ptr(z), _lib.ptr(acc), w, h, nd))
        props = G[f"{name}/fm3_1.0"]
        quinn = rd.FlowAccumFromProps(rd.rd3array(props, no_data=-2)) if np.isnan(props).any() else G[f"{name}/fa3_1.0"]
        assert close(acc, quinn, 1e-6), name
    attribs = ("slope_riserun", "slope_percentage", "slope_degrees", "slope_radians", "aspect", "curvature",
               "planform_curvature", "profile_curvature")
    for a in ta_runs:
        attrib = attribs[a]
        ref = G[f"{name}/ta{a}"]
        got = f64.TerrainAttribute(dem(), attrib, zscale=M.TA_ZSCALE)
        assert got.dtype == np.float32 and got.no_data == -9999
        assert same_bits(np.asarray(got), ref), (name, attrib)
        o = np.empty((h, w), np.float32)
        _lib.check(L.rdb200_dev_terrain_attribute_f64(a, _lib.ptr(z), _lib.ptr(o), w, h, nd, -9999.0, M.TA_ZSCALE,
                                                      *M.TA_CELL))
        assert same_bits(o, ref), (name, attrib, "dev")


def test_fixtures_reach_the_fallback():
    """huge and tiny hold finite nonzero D-infinity differences outside [2^-500, 2^500] in most cells (so the filter and
    the ratio test are skipped there), and near_tie holds a one-ulp tie of the two steepest facets for each case pair."""
    for name in ("huge", "tiny"):
        z, _ = fixture(name)
        d = np.abs(np.diff(z, axis=1))
        d = d[(d > 0) & np.isfinite(d)]
        out = (d < 2.0 ** -500) | (d > 2.0 ** 500)
        assert out.mean() > 0.9, name
    z, _ = fixture("near_tie")
    _, pairs = M.near_tie()
    assert pairs == [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]
    for k in range(len(pairs)):
        c, s = M.dinf_facets(z[None, :, 4 * k + 1:4 * k + 4])
        s = np.sort(np.unique(s[0][s[0] > 0]))
        assert np.nextafter(s[-2], np.inf) == s[-1], pairs[k]


@pytest.fixture(scope="module")
def R():
    if not F.have_ref():
        F.build()
    if not F.have_ref():
        pytest.skip("reference tree not available")
    return F.ref()


def test_beauford_float_rounding_changes_the_facets(R):
    """On beauford_data_1e-9 (1e-9 detail on a float DEM) the float-rounded raster gives other D-infinity proportions
    than the double answer."""
    z, nd = fixture("beauford_data_1e-9")
    double = G["beauford_data_1e-9/fm1_1.0"]
    rounded = R.fm(z.astype(np.float32), np.float32(nd), 1)
    assert not same_bits(rounded, double)
    assert np.any((rounded[..., 1:] > 0) != (double[..., 1:] > 0))  # other receiving slots, not only other values


def float_exact_raster():
    from oracle import fbm_terrain
    z = fbm_terrain(40, 56, seed=21, quantum=0.0).astype(np.float32)
    rng = np.random.default_rng(3)
    small = rng.random(z.shape) < 0.15
    z[small] = (rng.random(small.sum()) * 1e-3).astype(np.float32)  # float differences across binades round
    z[5, 5:9] = -9999.0
    return z.astype(np.float64)


def test_double_templates_equal_float_ones_on_a_float_exact_raster(R):
    z = float_exact_raster()
    nd = -9999.0
    zf = z.astype(np.float32)
    for m in (0, 1, 2):
        assert same_bits(R.fm(z, nd, m), R.fm(zf, np.float32(nd), m)), m
    for a in range(8):
        assert same_bits(R.ta(z, a, nd, M.TA_ZSCALE, M.TA_CELL), R.ta(zf, a, np.float32(nd), M.TA_ZSCALE, M.TA_CELL)), a
    # MFD: rise = e - ne is computed in the elevation type, so float rounds where double does not
    for m in (3, 4):
        assert not same_bits(R.fm(z, nd, m, 1.0), R.fm(zf, np.float32(nd), m, 1.0)), m


def test_golden_regenerates_to_the_same_bits(R):
    inputs = M.inputs()
    assert sorted(n for n, _, _ in inputs) == NAMES
    for name, z, nd in inputs:
        assert same_bits(z, G[f"{name}/dem"]) and nd == float(G[f"{name}/nodata"]), name
        keys = {k for k in G.files if k.startswith(name + "/")} - {f"{name}/dem", f"{name}/nodata"}
        out = M.compute(R, name, z, nd)
        assert {f"{name}/{k}" for k in out} == keys, name
        for k, v in out.items():
            assert same_bits(np.asarray(v), G[f"{name}/{k}"]), (name, k)


def test_argument_validation():
    import richdem_b200 as rd
    from richdem_b200 import f64
    z = rd.rdarray(np.zeros((4, 4)), no_data=-1)
    for fn, args in ((f64.FlowProportions, ("D8",)), (f64.TerrainAttribute, ("slope_riserun",))):
        with pytest.raises(Exception, match="rdarray"):
            fn(np.zeros((4, 4)), *args)
        with pytest.raises(Exception, match="float64"):
            fn(rd.rdarray(np.zeros((4, 4), np.float32), no_data=-1), *args)
        with pytest.raises(RuntimeError, match="two dimensions"):
            fn(rd.rdarray(np.zeros((4, 4, 2)), no_data=-1), *args)
    with pytest.raises(Exception, match="Invalid FlowProportions method"):
        f64.FlowProportions(z, "nope")
    for m in ("Holmgren", "Freeman"):
        with pytest.raises(Exception, match="requires an exponent"):
            f64.FlowProportions(z, m)
    for m in ("Rho8", "Rho4"):
        with pytest.raises(Exception, match="outside the GPU hot path"):
            f64.FlowProportions(z, m)
    with pytest.raises(Exception, match="Invalid TerrainAttributes attribute"):
        f64.TerrainAttribute(z, "nope")
    with pytest.raises(Exception, match="float32"):  # the float32 functions keep refusing float64
        rd.FlowProportions(z, "D8")
    with pytest.raises(Exception, match="float32"):
        rd.TerrainAttribute(z, "slope_riserun")


def test_emulated_abi_errors(emulated):
    L = _lib.lib()
    z = np.zeros((4, 4))
    p = np.zeros((4, 4, 9), np.float32)
    with pytest.raises(_lib.RichdemB200Error, match="null"):
        _lib.check(L.rdb200_fm_tarboton_f64(None, _lib.ptr(p), 4, 4, 0.0))
    with pytest.raises(_lib.RichdemB200Error, match="positive"):
        _lib.check(L.rdb200_fa_tarboton_f64_f64(_lib.ptr(z), _lib.ptr(z), 0, 4, 0.0, 1))
    with pytest.raises(_lib.RichdemB200Error, match="unknown flow metric"):
        _lib.check(L.rdb200_dev_fm_method_f64(7, _lib.ptr(z), _lib.ptr(p), 4, 4, 0.0, 1.0))
    with pytest.raises(_lib.RichdemB200Error, match="unknown terrain attribute"):
        _lib.check(L.rdb200_terrain_attribute_f64(9, _lib.ptr(z), _lib.ptr(p), 4, 4, 0.0, -9999.0, 1.0, 1.0, 1.0))
    with pytest.raises(_lib.RichdemB200Error, match="cell lengths"):
        _lib.check(L.rdb200_dev_terrain_attribute_f64(0, _lib.ptr(z), _lib.ptr(p), 4, 4, 0.0, -9999.0, 1.0, 0.0, 1.0))
