"""Every flow-accumulation engine against exact sums, with signed, zero and non-finite weights.

Two classes of check:

* exact -- weights m * 2^-20 with integers |m| <= 2^20 on rasters of at most ~1 M cells: every partial sum is a double,
  so any summation order gives the same bits.  D8, D4, one-hot proportions and the row-band drivers must then equal the
  CPU checker bit for bit, signs of zero included.
* bounded -- D-infinity and the multi-receiver proportions: |engine - A| <= B cell by cell, where A is the accumulation in
  extended precision over the proportions the library itself returns and B the engine's rigorous error budget
  (oracle/accum_exact.c).  The packed fixed-point D-infinity walk sums integers, so its result is also replayed bit for
  bit.

Special weights (+-0, NaN, +-inf, subnormal, huge) are tested where the answer does not depend on the order of addition:
which cells are NaN and which are +-inf must match the checker exactly, and finite cells stay within the budget.

The checks are plain functions of a device string: the `-m gpu` tests run them on the H100 ("cuda"); the others run them
on the CPU fiber model of the kernels (tests/emu), where "device" memory is host memory ("cpu").
"""
import ctypes as C
import importlib.util
import os
import sys

import numpy as np
import pytest

import oracle
from oracle import accum_exact
from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0
MFD = [("D4", None), ("Quinn", None), ("Holmgren", 2.5), ("Freeman", 1.1)]


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def R(a, nd=ND):
    import richdem_b200 as rd
    return rd.rdarray(np.ascontiguousarray(a), no_data=nd)


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def assert_bits(got, expected, what):
    got, expected = np.asarray(got, np.float64), np.asarray(expected, np.float64)
    bad = bits(got) != bits(expected)
    assert not bad.any(), f"{what}: {bad.sum()} cells differ, first {np.argwhere(bad)[:3].tolist()}: " \
                          f"{got[bad][:3].tolist()} != {expected[bad][:3].tolist()}"


def assert_within_budget(ex: accum_exact.Exact, what):
    q = ex.excess()
    assert q.max() <= 1.0, f"{what}: |got - exact| exceeds the budget {q.max():.3g} x at {np.unravel_index(q.argmax(), q.shape)}"


def assert_special(got, expected, what, zero_signs=False):
    """Same NaN cells, same +inf / -inf cells (and, where asked, the same signs of zero) as the checker."""
    got, expected = np.asarray(got), np.asarray(expected)
    for name, f in (("NaN", np.isnan), ("+inf", np.isposinf), ("-inf", np.isneginf)):
        assert np.array_equal(f(got), f(expected)), f"{what}: {name} cells differ ({f(got).sum()} vs {f(expected).sum()})"
    if zero_signs:
        z = expected == 0
        assert np.array_equal(got == 0, z), what
        assert np.array_equal(np.signbit(got[z]), np.signbit(expected[z])), f"{what}: signs of zero differ"


# ---- terrains --------------------------------------------------------------------------------------------------------
def fbm(checker, shape, seed, patch=True):
    dem = oracle.fbm_terrain(*shape, seed=seed, quantum=0.5)
    if patch:  # NoData patches, one on the raster edge
        h, w = shape
        dem[h // 3:h // 3 + h // 8, w // 4:w // 4 + w // 6] = ND
        dem[h - h // 10:, w // 2:w // 2 + 5] = ND
    return checker.resolve_flats(checker.fill_depressions(dem), ND)


def maze(checker, shape):
    """The serpentine maze: filling makes its corridor one flat, and flat resolution one path through every cell."""
    adv = _load_module("adversarial_terrain", os.path.join(HERE, "test_adversarial_terrain.py"))
    return checker.resolve_flats(checker.fill_depressions(adv.serpentine(*shape, seed=3)), ND)


def tilted_plane(shape, angle=0.3):
    """A plane at a non-grid angle: every interior D-infinity cell has two receivers."""
    yy, xx = np.mgrid[0:shape[0], 0:shape[1]].astype(np.float64)
    return (1000.0 - 0.37 * (xx * np.cos(angle) + yy * np.sin(angle))).astype(np.float32)


def beauford(golden, rows=None):
    g = golden["beauford_crop"]
    dem = np.array(g["resolved"], np.float32)
    nd = float(g["nodata"])
    dem[dem == nd] = ND
    return dem if rows is None else np.ascontiguousarray(dem[:rows])


def packed_worst_case(golden, k):
    """k x k copies of the patch tools/dinf_packed_worst.py found (tests/golden/dinf_packed_worst.npz), each in a NoData
    frame: its centre takes rounded shares whose errors add up to about a quarter of the 2^-22 bound."""
    patch = golden["dinf_packed_worst"]["patch"]
    p = patch.shape[0] + 2
    dem = np.full((k * p, k * p), ND, np.float32)
    for y in range(k):
        for x in range(k):
            dem[y * p + 1:y * p + p - 1, x * p + 1:x * p + p - 1] = patch
    return dem


def exact_weights(shape, seed, nodata_mask=None):
    """m * 2^-20, |m| <= 2^20: signed, with zeros of both signs and cells of exactly -1 (the NoData output value); NaN
    under NoData."""
    rng = np.random.default_rng(seed)
    w = rng.integers(-(1 << 20), (1 << 20) + 1, size=shape).astype(np.float64) * 2.0 ** -20
    k = rng.random(shape)
    w[k < 0.05] = 0.0
    w[(k >= 0.05) & (k < 0.1)] = -0.0
    w[(k >= 0.1) & (k < 0.12)] = -1.0
    w[(k >= 0.12) & (k < 0.14)] = 1.0
    if nodata_mask is not None:
        w[nodata_mask & (k < 0.5)] = np.nan
    return w


# ---- the row-band protocol, every band on one device --------------------------------------------------------------------
def bands(dev, dem, G, weights=None, method=None, exponent=None, dinf=False):
    """Drive G CudaBandAccumulators (rdb200_dev_facc_*) on one device through the fa_band protocol."""
    import torch
    from richdem_b200 import sharded
    h, w = dem.shape
    accs, metas, outs = [], [], []
    for g in range(G):
        r0, r1, gt, gb = sharded.local_rows(h, G, g)
        local = torch.from_numpy(np.ascontiguousarray(dem[r0 - gt:r1 + gb])).to(dev, copy=True).contiguous()
        if weights is None:
            acc = torch.empty(local.shape, dtype=torch.float64, device=dev)
        else:
            acc = torch.from_numpy(np.ascontiguousarray(weights[r0 - gt:r1 + gb])).to(dev, copy=True).contiguous()
        accs.append(sharded.CudaBandAccumulator(local, acc, ND, gt, gb, dinf, weights is None, method=method, exponent=exponent))
        outs.append(acc)
        metas.append((r0, r1, gt, gb))
    for g, (r0, r1, gt, gb) in enumerate(metas):
        if gt:
            accs[g].set_ghost_codes(0, *accs[g - 1].edge_codes(1))
        if gb:
            accs[g].set_ghost_codes(1, *accs[g + 1].edge_codes(0))
    rounds = 0
    while True:
        sent = [A.run() for A in accs]
        rounds += 1
        if not any(a + b for a, b in sent):
            break
        ups = {g: accs[g].take_outflow(0) for g, m in enumerate(metas) if m[2]}
        dns = {g: accs[g].take_outflow(1) for g, m in enumerate(metas) if m[3]}
        for g, (r0, r1, gt, gb) in enumerate(metas):
            if gt:
                accs[g].apply_inflow(0, *dns[g - 1])
            if gb:
                accs[g].apply_inflow(1, *ups[g + 1])
        assert rounds < 10000
    out = np.empty((h, w), np.float64)
    for g, (r0, r1, gt, gb) in enumerate(metas):
        accs[g].finish()
        out[r0:r1] = outs[g][gt:gt + (r1 - r0)].cpu().numpy()
    return out, rounds


def _dev_array(dev, a, misalign=False):
    """A device copy of a float64 raster; misalign: its data pointer 8 bytes off a 16-byte boundary."""
    import torch
    flat = torch.from_numpy(np.ascontiguousarray(a, np.float64).reshape(-1))
    buf = torch.empty(flat.numel() + 2, dtype=torch.float64, device=dev)
    off = 1 if (buf.data_ptr() % 16 == 0) == misalign else 0
    view = buf[off:off + flat.numel()]
    view.copy_(flat)
    assert (view.data_ptr() % 16 == 8) == misalign
    return view


# ======================================================================================================================
# the checks
# ======================================================================================================================
def check_exact_class(dev, checker, dem, seed, G=3):
    """Exact weights: D8, D4, one-hot proportions, float64 DEMs, device and band entry points equal the checker bit for
    bit."""
    import richdem_b200 as rd
    from richdem_b200 import f64
    h, w = dem.shape
    wts = exact_weights(dem.shape, seed, dem == ND)
    exp_d8 = checker.fa_d8(dem, ND, wts)
    exp_d4 = checker.fa_method(dem, ND, "D4", None, wts)
    assert_bits(rd.FlowAccumulation(R(dem), "D8", weights=R(wts, -1)), exp_d8, "D8")
    assert_bits(rd.FlowAccumulation(R(dem), "D4", weights=R(wts, -1)), exp_d4, "D4")
    props = rd.FlowProportions(R(dem), "D8")  # one-hot: d8_flow_accum-style FlowAccumFromProps
    assert_bits(rd.FlowAccumFromProps(props, weights=R(wts, -1)), checker.flow_accumulation(props, wts), "FromProps(D8)")
    d64 = dem.astype(np.float64)
    assert_bits(f64.FlowAccumulation(R(d64), "D8", weights=R(wts, -1)), exp_d8, "f64 D8")
    assert_bits(f64.FlowAccumulation(R(d64), "D4", weights=R(wts, -1)), exp_d4, "f64 D4")
    # the device entry points, on an accumulator 16-byte aligned and 8 bytes off
    L = _lib.lib()
    for mis in (False, True):
        import torch
        d = torch.from_numpy(np.ascontiguousarray(dem)).to(dev)
        a = _dev_array(dev, wts, mis)
        _lib.check(L.rdb200_dev_fa_d8_f32_f64(d.data_ptr(), a.data_ptr(), w, h, ND, 0))
        assert_bits(a.cpu().numpy().reshape(h, w), exp_d8, f"dev D8 misaligned={mis}")
        a = _dev_array(dev, wts, mis)
        _lib.check(L.rdb200_dev_fa_method_f32_f64(2, d.data_ptr(), a.data_ptr(), w, h, ND, 0.0))
        assert_bits(a.cpu().numpy().reshape(h, w), exp_d4, f"dev D4 misaligned={mis}")
    # row bands
    assert_bits(bands(dev, dem, G, wts)[0], exp_d8, f"bands D8 G={G}")
    assert_bits(bands(dev, dem, G, wts, method="D4")[0], exp_d4, f"bands D4 G={G}")


def check_generic_walk_equals_tile_engine(dev, dem):
    """Weights of exactly 1.0 through the generic walk (accum_is_ones = 0) give the unit-weight tile engine's bits."""
    L = _lib.lib()
    h, w = dem.shape
    tile = np.empty((h, w), np.float64)
    _lib.check(L.rdb200_fa_d8_f32_f64(_lib.ptr(dem), _lib.ptr(tile), w, h, ND, 1))
    walk = np.ones((h, w), np.float64)
    _lib.check(L.rdb200_fa_d8_f32_f64(_lib.ptr(dem), _lib.ptr(walk), w, h, ND, 0))
    assert_bits(walk, tile, "generic walk vs tile engine")


def check_bounded_class(dev, checker, dem, seed, G=3):
    """D-infinity and the proportions methods with signed weights: within the double engines' budget of the exact sums
    over the library's own proportions, on one device, over row bands, and from a float64 DEM."""
    import richdem_b200 as rd
    from richdem_b200 import f64
    h, w = dem.shape
    rng = np.random.default_rng(seed)
    wts = rng.standard_normal(dem.shape) * np.exp2(rng.integers(-20, 20, dem.shape))
    pd = rd.FlowProportions(R(dem), "Dinf")

    def ex(p, got):
        return accum_exact.accumulate(p, wts, got=got)

    assert_within_budget(ex(pd, np.asarray(rd.FlowAccumulation(R(dem), "Dinf", weights=R(wts, -1)))), "Dinf weighted")
    assert_within_budget(ex(pd, np.asarray(rd.FlowAccumFromProps(pd, weights=R(wts, -1)))), "FromProps(Dinf)")
    assert_within_budget(ex(pd, bands(dev, dem, G, wts, dinf=True)[0]), f"bands Dinf G={G}")
    for m, e in MFD:
        p = rd.FlowProportions(R(dem), m, e)
        assert_within_budget(ex(p, np.asarray(rd.FlowAccumulation(R(dem), m, e, weights=R(wts, -1)))), m)
        assert_within_budget(ex(p, bands(dev, dem, G, wts, method=m, exponent=e)[0]), f"bands {m} G={G}")
    # float64 DEM (float-exact): the double instantiations
    d64 = dem.astype(np.float64)
    L = _lib.lib()
    got = wts.copy()
    _lib.check(L.rdb200_fa_tarboton_f64_f64(_lib.ptr(d64), _lib.ptr(got), w, h, ND, 0))
    assert_within_budget(ex(f64.FlowProportions(R(d64), "Dinf"), got), "f64 Dinf")
    got = wts.copy()
    _lib.check(L.rdb200_fa_freeman_f64_f64(_lib.ptr(d64), _lib.ptr(got), w, h, ND, 1.1))
    assert_within_budget(ex(f64.FlowProportions(R(d64), "Freeman", 1.1), got), "f64 Freeman")


def check_unit_dinf(dev, dem, G=3):
    """Unit-weight D-infinity on every engine.  The packed fixed-point walk sums integers, so its bits are those of its
    CPU replay, and within the packed budget; the level kernel (accum_dinf_packed 0, W % 4 != 0, an accumulator 8 bytes
    off 16-byte alignment, or mode 2 on a raster where few cells lack a receiver) stays within the double budget.  Both
    against the proportions FlowProportions("Dinf") returns, so FA_Tarboton's fused shares must be those bits.  Returns
    the packed walk's largest relative error (0 if it never ran)."""
    import richdem_b200 as rd
    import torch
    h, w = dem.shape
    pd = rd.FlowProportions(R(dem), "Dinf")
    packed = accum_exact.accumulate(pd, mode="packed")
    L = _lib.lib()
    d = torch.from_numpy(np.ascontiguousarray(dem)).to(dev)
    worst = 0.0

    def check(got, must_pack, what):
        nonlocal worst
        if np.array_equal(got, packed.packed) or np.array_equal(got, packed.packed_fma):
            e = accum_exact.accumulate(pd, mode="packed", got=got)
            assert_within_budget(e, what)
            data = e.ref > 0
            worst = max(worst, float((e.err[data] / e.ref[data]).max()))
        else:
            assert not must_pack, f"{what}: not the packed walk's bits"
            assert_within_budget(accum_exact.accumulate(pd, got=got), what)

    for mode in (0, 1, 2):
        _lib.set_param("accum_dinf_packed", mode)
        for mis in (False, True):
            a = _dev_array(dev, np.zeros((h, w)), mis)
            _lib.check(L.rdb200_dev_fa_tarboton_f32_f64(d.data_ptr(), a.data_ptr(), w, h, ND, 1))
            check(a.cpu().numpy().reshape(h, w), mode == 1 and w % 4 == 0 and not mis,
                  f"Dinf unit accum_dinf_packed={mode} misaligned={mis}")
        check(bands(dev, dem, G, dinf=True)[0], mode != 0 and w % 4 == 0, f"bands Dinf unit accum_dinf_packed={mode}")
    _lib.reset_params()
    return worst


def check_unit_d8_routes(dev, checker, dem, G=3):
    """Unit-weight D8 with accum_packed 0 and 1, on one device and over row bands: the checker's bits."""
    import richdem_b200 as rd
    expected = checker.fa_d8(dem, ND)
    for packed in (0, 1):
        _lib.set_param("accum_packed", packed)
        assert_bits(rd.FlowAccumulation(R(dem), "D8"), expected, f"D8 accum_packed={packed}")
        assert_bits(bands(dev, dem, G)[0], expected, f"bands D8 accum_packed={packed}")
    _lib.reset_params()


SPECIALS = ("neg_zero", "pos_zero", "nan", "pos_inf", "neg_inf", "inf_meets_neg_inf", "subnormal", "huge")


def special_weights(kind, dem, seed):
    """Weights whose accumulation does not depend on the order of addition."""
    rng = np.random.default_rng(seed)
    h, w = dem.shape
    if kind == "neg_zero":
        return np.full((h, w), -0.0)
    if kind == "pos_zero":
        return np.zeros((h, w))
    if kind == "subnormal":
        return rng.integers(1, 1 << 20, (h, w)).astype(np.float64) * 5e-324
    if kind == "huge":
        return rng.uniform(1.0, 2.0, (h, w)) * 1e300
    wts = rng.integers(0, 1 << 10, (h, w)).astype(np.float64) * 2.0 ** -10
    cells = [tuple(rng.integers(1, [h - 1, w - 1])) for _ in range(3)]
    if kind == "nan":
        for c in cells:
            wts[c] = np.nan
    elif kind in ("pos_inf", "neg_inf"):
        for c in cells:
            wts[c] = np.inf if kind == "pos_inf" else -np.inf
    else:  # inf_meets_neg_inf: both in every cell of a row band, so the two meet downstream
        wts[h // 2, 1:w - 1] = np.inf
        wts[h // 2 + 1, 1:w - 1] = -np.inf
    wts[dem == ND] = np.nan  # NoData cells end as -1 whatever they held
    return wts


def check_special_weights(dev, checker, dem, kind, G=3):
    import richdem_b200 as rd
    wts = special_weights(kind, dem, 7)
    zs = kind in ("neg_zero", "pos_zero")
    nd = dem == ND

    def check(got, expected, props, what):
        got = np.asarray(got)
        assert np.all(got[nd] == -1.0), f"{what}: NoData cells must be -1"
        assert_special(got, expected, what, zero_signs=zs)
        fin = np.isfinite(expected)
        ex = accum_exact.accumulate(props, np.where(nd, 0.0, wts), got=np.where(fin, got, 0.0))
        ex.err[~fin] = 0.0
        assert_within_budget(ex, what)

    p8, p4 = rd.FlowProportions(R(dem), "D8"), rd.FlowProportions(R(dem), "D4")
    pd = rd.FlowProportions(R(dem), "Dinf")
    e8, e4, ed = checker.fa_d8(dem, ND, wts), checker.fa_method(dem, ND, "D4", None, wts), checker.fa_dinf(dem, ND, wts)
    check(rd.FlowAccumulation(R(dem), "D8", weights=R(wts, -1)), e8, p8, f"D8 {kind}")
    check(rd.FlowAccumulation(R(dem), "D4", weights=R(wts, -1)), e4, p4, f"D4 {kind}")
    check(rd.FlowAccumulation(R(dem), "Dinf", weights=R(wts, -1)), ed, pd, f"Dinf {kind}")
    check(rd.FlowAccumFromProps(pd, weights=R(wts, -1)), checker.flow_accumulation(pd, wts), pd, f"FromProps(Dinf) {kind}")
    check(bands(dev, dem, G, wts)[0], e8, p8, f"bands D8 {kind}")
    check(bands(dev, dem, G, wts, dinf=True)[0], ed, pd, f"bands Dinf {kind}")
    check(bands(dev, dem, G, wts, method="D4")[0], e4, p4, f"bands D4 {kind}")


# ======================================================================================================================
# on the CPU model of the kernels
# ======================================================================================================================
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
    return L


@pytest.fixture()
def emulated(emu_lib, monkeypatch):
    """The Python layer on the kernel emulation for one test; "device" memory is host memory."""
    from richdem_b200 import sharded
    monkeypatch.setattr(_lib, "_lib", emu_lib)
    monkeypatch.setattr(_lib, "use_torch_stream", lambda: None)
    monkeypatch.setattr(sharded, "_on_device", lambda t: True)
    _lib.init(0)
    _lib.set_param("fill_use_tma", 0)
    yield "cpu"
    _lib.reset_params()


@pytest.mark.parametrize("terrain,shape", [("fbm", (97, 130)), ("fbm", (70, 129)), ("maze", (41, 67)), ("beauford", None)])
def test_exact_weights_emulated(emulated, checker, golden, terrain, shape):
    dem = beauford(golden, 96) if terrain == "beauford" else maze(checker, shape) if terrain == "maze" else \
        fbm(checker, shape, seed=shape[1])
    check_exact_class(emulated, checker, dem, seed=5)


def test_generic_walk_equals_tile_engine_emulated(emulated, checker):
    for shape in ((97, 130), (130, 68)):
        check_generic_walk_equals_tile_engine(emulated, fbm(checker, shape, seed=11))


@pytest.mark.parametrize("terrain", ["fbm", "maze", "plane"])
def test_bounded_weights_emulated(emulated, checker, terrain):
    dem = {"fbm": lambda: fbm(checker, (90, 101), seed=13), "maze": lambda: maze(checker, (33, 48)),
           "plane": lambda: tilted_plane((60, 70))}[terrain]()
    check_bounded_class(emulated, checker, dem, seed=17)


@pytest.mark.parametrize("terrain,shape", [("fbm", (96, 128)), ("fbm", (65, 130)), ("maze", (41, 68)), ("plane", (64, 72))])
def test_unit_dinf_engines_emulated(emulated, checker, terrain, shape):
    dem = maze(checker, shape) if terrain == "maze" else tilted_plane(shape) if terrain == "plane" else \
        fbm(checker, shape, seed=19)
    check_unit_dinf(emulated, dem)


def test_packed_dinf_worst_case_emulated(emulated, golden):
    assert check_unit_dinf(emulated, packed_worst_case(golden, 8)) > 2.0 ** -25


def test_unit_d8_routes_emulated(emulated, checker):
    check_unit_d8_routes(emulated, checker, fbm(checker, (97, 132), seed=23))


@pytest.mark.parametrize("kind", SPECIALS)
def test_special_weights_emulated(emulated, checker, kind):
    check_special_weights(emulated, checker, fbm(checker, (66, 75), seed=29), kind)


# ======================================================================================================================
# on the H100
# ======================================================================================================================
@pytest.fixture()
def cuda():
    _lib.init(0)
    yield "cuda"
    _lib.reset_params()


@pytest.mark.gpu
@pytest.mark.parametrize("terrain,shape", [("fbm", (1000, 1300)), ("fbm", (777, 1003)), ("maze", (201, 333)),
                                           ("beauford", None)])
def test_exact_weights_gpu(cuda, checker, golden, terrain, shape):
    dem = beauford(golden) if terrain == "beauford" else maze(checker, shape) if terrain == "maze" else \
        fbm(checker, shape, seed=shape[1])
    check_exact_class(cuda, checker, dem, seed=5, G=5)


@pytest.mark.gpu
def test_generic_walk_equals_tile_engine_gpu(cuda, checker):
    for shape in ((1000, 1300), (1030, 777), (64, 4096)):
        check_generic_walk_equals_tile_engine(cuda, fbm(checker, shape, seed=11))


@pytest.mark.gpu
@pytest.mark.parametrize("terrain", ["fbm", "maze", "plane", "beauford"])
def test_bounded_weights_gpu(cuda, checker, golden, terrain):
    dem = {"fbm": lambda: fbm(checker, (900, 1101), seed=13), "maze": lambda: maze(checker, (201, 332)),
           "plane": lambda: tilted_plane((600, 700)), "beauford": lambda: beauford(golden)}[terrain]()
    check_bounded_class(cuda, checker, dem, seed=17, G=5)


@pytest.mark.gpu
@pytest.mark.parametrize("terrain,shape", [("fbm", (1024, 1280)), ("fbm", (1000, 1301)), ("maze", (201, 332)),
                                           ("plane", (2048, 2048)), ("beauford", None)])
def test_unit_dinf_engines_gpu(cuda, checker, golden, terrain, shape):
    dem = beauford(golden) if terrain == "beauford" else maze(checker, shape) if terrain == "maze" else \
        tilted_plane(shape) if terrain == "plane" else fbm(checker, shape, seed=19)
    worst = check_unit_dinf(cuda, dem, G=4)
    print(f"packed D-infinity walk, {terrain} {dem.shape}: largest relative error {worst:.3e} (bound 2^-22 = {2.0 ** -22:.3e})")


@pytest.mark.gpu
def test_packed_dinf_worst_case_gpu(cuda, golden):
    worst = check_unit_dinf(cuda, packed_worst_case(golden, 64), G=4)
    print(f"packed D-infinity walk, constructed case: largest relative error {worst:.3e} (bound 2^-22 = {2.0 ** -22:.3e})")
    assert worst > 2.0 ** -25


@pytest.mark.gpu
def test_unit_d8_routes_gpu(cuda, checker):
    check_unit_d8_routes(cuda, checker, fbm(checker, (1000, 1300), seed=23), G=5)
    check_unit_d8_routes(cuda, checker, fbm(checker, (999, 1001), seed=24), G=5)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", SPECIALS)
def test_special_weights_gpu(cuda, checker, kind):
    check_special_weights(cuda, checker, fbm(checker, (700, 901), seed=29), kind, G=5)
