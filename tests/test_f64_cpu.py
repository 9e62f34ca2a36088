"""float64 elevations without a GPU.

* The argument of DESIGN §0 against the unmodified reference: reference<double>(Z) equals kappa^-1 of
  reference<float>(kappa(Z)) for every function of the float64 path and both topologies (oracle/f64_shim.cpp), bit for
  bit apart from the fill's zero sign; and the float32 path on the rounded raster does not.
* The new kernels (csrc/f64.cu) on the CPU fiber model of tests/emu against the numpy restatement of kappa, and every
  float64 entry point on the emulated library against the reference.
"""
import ctypes as C
import importlib.util
import os
import sys

import numpy as np
import pytest

from oracle import f64 as F
from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
TOPOS = ("D8", "D4")


def same_bits(a, b, zero_sign=False):
    """Bitwise equality; NaN equals NaN; with zero_sign, -0.0 equals +0.0."""
    a, b = np.asarray(a, np.float64).copy(), np.asarray(b, np.float64).copy()
    if a.shape != b.shape:
        return False
    if zero_sign:
        a[a == 0] = 0.0
        b[b == 0] = 0.0
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | nan))


@pytest.fixture(scope="module")
def R():
    if not F.have_ref():
        F.build()
    if not F.have_ref():
        pytest.skip("reference tree not available")
    return F.ref()


CASES = F.cases()


@pytest.mark.parametrize("topology", TOPOS)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_float_keys_give_the_double_answer(R, case, topology):
    name, z, nd = case
    k, ndk, ranked = F.kappa(z, nd)
    assert ranked == (not F.is_float_raster(z))
    # fill: kappa^-1 of the float fill of the keys
    assert same_bits(R.fill(z, topology), F.kappa_inv_fill(z, k, R.fill(k, topology)), zero_sign=True), name
    # pit_mask and HasDepressions: the float templates on the keys, NoData kappa(nodata)
    assert np.array_equal(R.pit_mask(z, nd, topology), R.pit_mask(k, ndk, topology)), name
    assert R.has_depressions(z, topology) == R.has_depressions(k, topology), name
    # accumulation: no elevation values in the output
    assert same_bits(R.fa(z, nd, topology), R.fa(k, ndk, topology)), name
    w = np.random.default_rng(1).random(z.shape)
    assert same_bits(R.fa(z, nd, topology, weights=w), R.fa(k, ndk, topology, weights=w)), name
    if topology == "D8":
        assert np.array_equal(R.d8_flow_directions(z, nd), R.d8_flow_directions(k, ndk)), name
        # flats: the float mask of the keys, applied as double ulps
        assert same_bits(R.resolve_flats(z, nd), F.apply_flat_mask(z, R.flat_mask(k, ndk))), name


def test_the_cast_to_float_changes_the_answer(R):
    """What rounding to float32 first does to nested lakes one double ulp apart."""
    z = F.nested_lakes()
    ref = R.fill(z)
    assert ref[5, 10] == np.nextafter(5.0, np.inf) and ref[5, 3] == 5.0
    rounded = R.fill(z.astype(np.float32)).astype(np.float64)
    assert not same_bits(ref, rounded, zero_sign=True)
    k, _, ranked = F.kappa(z, -9999.0)
    assert ranked
    assert same_bits(ref, F.kappa_inv_fill(z, k, R.fill(k)), zero_sign=True)


def test_kappa_spec():
    z = np.array([[3.0, -0.0, 0.0, np.nextafter(3.0, 4.0)], [np.inf, -F.DBL_MAX, F.DBL_MAX, np.nan]])
    k, ndk, ranked = F.kappa(z, 3.0)
    assert ranked
    assert k[0, 1] == k[0, 2] and k[0, 0] < k[0, 3] and k[0, 1] < k[0, 0]
    assert k[1, 0] == np.inf and k[1, 1] == -F.FLT_MAX and k[1, 2] == F.FLT_MAX and np.isnan(k[1, 3])
    assert ndk == k[0, 0]
    assert 0 < k[0, 1] < k[0, 3] < F.FLT_MAX
    # case 1: the cast; a single FLT_MAX cell sends the raster to case 2
    f = np.array([[1.5, -2.0, np.inf, np.nan]])
    k1, nd1, r1 = F.kappa(f, 7.0)
    assert not r1 and np.array_equal(k1[:, :3], f[:, :3].astype(np.float32)) and np.isnan(nd1)
    assert F.kappa(np.array([[1.5, F.FLT_MAX]]), 0.0)[2]
    assert F.kappa(np.array([[1.5, -F.FLT_MAX]]), 0.0)[2]
    assert F.kappa(np.array([[1.5, 2.0]]), -np.inf)[1] == -np.inf
    assert F.kappa(np.array([[1.5, 2.0]]), F.DBL_MAX)[1] == F.FLT_MAX


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


def key_rasters():
    rng = np.random.default_rng(7)
    out = [(name, z, nd) for name, z, nd in CASES if z.size <= 4000]
    big = rng.random((100, 123)) * 100.0  # three 4096-cell tiles and a partial one
    big[rng.random(big.shape) < 0.1] = -9999.0
    out.append(("three_tiles", big, -9999.0))
    out.append(("all_equal", np.full((9, 11), 1.0 + 2.0 ** -40), 0.0))
    low = np.full((13, 17), 1.0 + 2.0 ** -40).view(np.uint64)
    low = (low + rng.integers(0, 256, low.shape).astype(np.uint64)).view(np.float64)
    out.append(("low_byte_only", low, float(low[3, 3])))
    out.append(("n1_float", np.array([[2.5]]), 2.5))
    out.append(("n1_ranked", np.array([[1.0 + 2.0 ** -40]]), -1.0))
    out.append(("one_flt_max", np.array([[1.0, 2.0, F.FLT_MAX], [0.5, 0.25, 4.0]]), 4.0))
    out.append(("one_minus_flt_max", np.array([[1.0, -F.FLT_MAX, 3.0]]), np.inf))
    out.append(("odd_size", rng.standard_normal((37, 53)), -9999.0))
    return out


def test_emulated_keys_equal_the_spec(emulated):
    from richdem_b200 import f64
    for name, z, nd in key_rasters():
        k, ndk, ranked = f64.OrderKeys(z, nd)
        ks, ndks, rs = F.kappa(z, nd)
        assert ranked == rs, name
        assert np.array_equal(k.view(np.uint32), ks.view(np.uint32)), name
        if np.isnan(ndks):
            assert np.isnan(ndk), name
        else:
            assert ndk.view(np.uint32) == ndks.view(np.uint32), name


def test_emulated_entry_points_equal_the_reference(emulated, R):
    import richdem_b200 as rd
    from richdem_b200 import f64
    small = [c for c in CASES if c[1].size <= 4000]
    for name, z, nd in small:
        before = z.copy()
        a = lambda: rd.rdarray(z.copy(), no_data=nd)
        for topo in TOPOS:
            assert same_bits(f64.FillDepressions(a(), topology=topo), R.fill(z, topo), zero_sign=True), (name, topo)
            assert np.array_equal(f64.PitMask(a(), topology=topo), R.pit_mask(z, nd, topo)), (name, topo)
            assert f64.HasDepressions(a(), topology=topo) == R.has_depressions(z, topo), (name, topo)
            method = "D8" if topo == "D8" else "D4"
            assert same_bits(f64.FlowAccumulation(a(), method=method), R.fa(z, nd, topo)), (name, topo)
            wts = rd.rdarray(np.random.default_rng(2).random(z.shape), no_data=-1)
            got = f64.FlowAccumulation(a(), method=method, weights=wts)
            assert np.allclose(got, R.fa(z, nd, topo, weights=wts), rtol=1e-9, atol=0), (name, topo)
        assert same_bits(f64.ResolveFlats(a()), R.resolve_flats(z, nd)), name
        assert np.array_equal(f64.FlowDirectionsD8(a()), R.d8_flow_directions(z, nd)), name
        assert same_bits(z, before), name


def test_emulated_strict_pit_in_doubles(emulated):
    """A pit one double ulp deep: HasDepressions answers from the stencil pass alone."""
    from richdem_b200 import f64
    import richdem_b200 as rd
    z = np.full((5, 6), 1.0)
    z[2, 3] = np.nextafter(1.0, 0.0)
    for topo in TOPOS:
        assert f64.HasDepressions(rd.rdarray(z, no_data=-9999.0), topology=topo)
        assert _lib.stats()["kernel_launches"] == 1
    flat = np.full((5, 6), 1.0)
    assert not f64.HasDepressions(rd.rdarray(flat, no_data=-9999.0))


def test_argument_validation():
    import richdem_b200 as rd
    from richdem_b200 import f64
    for fn in (f64.PitMask, f64.HasDepressions, f64.FillDepressions):
        with pytest.raises(Exception, match="rdarray"):
            fn(np.zeros((4, 4)))
        with pytest.raises(Exception, match="Unknown topology!"):
            fn(rd.rdarray(np.zeros((4, 4)), no_data=-1), topology="D6")
        with pytest.raises(Exception, match="float64"):
            fn(rd.rdarray(np.zeros((4, 4), np.float32), no_data=-1))
        with pytest.raises(RuntimeError, match="two dimensions"):
            fn(rd.rdarray(np.zeros((4, 4, 2)), no_data=-1))
    for fn in (f64.ResolveFlats, f64.FlowDirectionsD8):
        with pytest.raises(Exception, match="float64"):
            fn(rd.rdarray(np.zeros((4, 4), np.float32), no_data=-1))
    with pytest.raises(Exception, match="not available for float64"):
        f64.FlowAccumulation(rd.rdarray(np.zeros((4, 4)), no_data=-1), method="Dinf")
    with pytest.raises(Exception, match="Invalid FlowAccumulation method"):
        f64.FlowAccumulation(rd.rdarray(np.zeros((4, 4)), no_data=-1), method="nope")
    with pytest.raises(Exception, match="float32"):  # the float32 module keeps refusing float64
        rd.FillDepressions(rd.rdarray(np.zeros((4, 4)), no_data=-1))


def test_emulated_abi_errors(emulated):
    L = _lib.lib()
    z = np.zeros((4, 4))
    with pytest.raises(_lib.RichdemB200Error, match="positive"):
        _lib.check(L.rdb200_fill_depressions_d8_f64(z.ctypes.data, 0, 4))
    with pytest.raises(_lib.RichdemB200Error, match="null"):
        _lib.check(L.rdb200_pit_mask_d4_f64(z.ctypes.data, None, 4, 4, 0.0))
    with pytest.raises(_lib.RichdemB200Error, match="null"):
        _lib.check(L.rdb200_fa_d8_f64_f64(None, z.ctypes.data, 4, 4, 0.0, 1))
