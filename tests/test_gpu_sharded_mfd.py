"""Row-band flow accumulation with the proportions methods (FA_D4, FA_Quinn, FA_Holmgren, FA_Freeman) on the GPU:
G CudaBandAccumulators on one device driven through the fa_band protocol (sequential emulation of G ranks, as in
test_gpu_sharded.py), and the C++ band driver (rdb200_mgpu_fa_method_f32_f64) at world 1.  Results are compared with
the CPU checker and with the single-GPU FlowAccumulation; both sum the same proportions, in different orders."""
import importlib.util
import os

import numpy as np
import pytest

import oracle
import richdem_b200 as rd
from richdem_b200 import _lib, sharded

pytestmark = pytest.mark.gpu
DEV = "cuda"  # tests/test_emulated_mfd_bands.py re-runs these drivers on host memory against the kernel emulation
ND = -9999.0
BAND_RTOL = 1e-9  # band vs single GPU: the same proportions, summed in another order


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_gp = _load_module("gpu_parity_cases", os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_gpu_parity.py"))
METRIC_CASES, MFD_ACC_RTOL = _gp.METRIC_CASES, _gp.MFD_ACC_RTOL


def emulate_fa_bands_method(dem: np.ndarray, G: int, nodata: float, method: str, exponent=None, weights=None):
    """Drive G CudaBandAccumulators for ``method`` on one device through the fa_band protocol: seam donor masks once,
    then rounds of run / take_outflow / apply_inflow until no band parked anything."""
    import torch
    h, w = dem.shape
    accs, metas, outs = [], [], []
    for g in range(G):
        r0, r1, gt, gb = sharded.local_rows(h, G, g)
        local = torch.from_numpy(np.ascontiguousarray(dem[r0 - gt:r1 + gb])).to(DEV, copy=True).contiguous()
        if weights is None:
            acc = torch.empty(local.shape, dtype=torch.float64, device=DEV)
        else:
            acc = torch.from_numpy(np.ascontiguousarray(weights[r0 - gt:r1 + gb])).to(DEV, copy=True).contiguous()
        accs.append(sharded.CudaBandAccumulator(local, acc, nodata, gt, gb, False, weights is None, method=method,
                                                exponent=exponent))
        outs.append(acc)
        metas.append((r0, r1, gt, gb))
    masks = [(A.edge_codes(0) if m[2] else None, A.edge_codes(1) if m[3] else None) for A, m in zip(accs, metas)]
    for g, (r0, r1, gt, gb) in enumerate(metas):
        if gt:
            accs[g].set_ghost_codes(0, *masks[g - 1][1])
        if gb:
            accs[g].set_ghost_codes(1, *masks[g + 1][0])
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


def single_gpu(dem, method, exponent, weights=None):
    w = None if weights is None else rd.rdarray(np.ascontiguousarray(weights), no_data=-1)
    return np.asarray(rd.FlowAccumulation(rd.rdarray(np.ascontiguousarray(dem), no_data=ND), method, exponent=exponent,
                                          weights=w))


def check_bands(checker, dem, G, method, exponent, weights=None):
    got, rounds = emulate_fa_bands_method(dem, G, ND, method, exponent, weights)
    np.testing.assert_allclose(got, checker.fa_method(dem, ND, method, exponent, weights), rtol=MFD_ACC_RTOL, atol=0,
                               err_msg=f"{method} {exponent} G={G} vs checker")
    np.testing.assert_allclose(got, single_gpu(dem, method, exponent, weights), rtol=BAND_RTOL, atol=0,
                               err_msg=f"{method} {exponent} G={G} vs one GPU")
    return rounds


_resolved = {}


def resolved_fbm(checker):
    """Filled, flat-resolved fBm with a NoData block across the seams of every G below."""
    if "dem" not in _resolved:
        dem = oracle.fbm_terrain(640, 500, seed=41, quantum=0.25)
        dem[200:330, 150:190] = ND  # rows 214 (G=3), 240 (G=8), 256 (G=5) and 320 (G=2, 8) are seams
        _resolved["dem"] = checker.resolve_flats(checker.fill_depressions(dem), ND)
    return _resolved["dem"]


@pytest.mark.parametrize("G", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("method,exponent", METRIC_CASES)
def test_band_mfd_accumulation_equals_single(checker, G, method, exponent):
    dem = resolved_fbm(checker)
    check_bands(checker, dem, G, method, exponent)
    wts = np.random.default_rng(G).random(dem.shape)
    check_bands(checker, dem, G, method, exponent, wts)


def serpentine_channel(h=64, w=64, step=4):
    """One channel that runs down and up the raster column after column, so that it crosses every row seam many
    times, cut into a flat plateau (no flow there); it leaves through the raster's bottom edge."""
    dem = np.full((h, w), 10000.0, np.float32)
    cols = list(range(2, w - 2, step))
    if len(cols) % 2 == 0:  # the last column runs down
        cols.pop()
    path = []
    for k, c in enumerate(cols):
        path += [(r, c) for r in (range(1, h - 2) if k % 2 == 0 else range(h - 3, 0, -1))]
        if k + 1 < len(cols):
            turn = h - 3 if k % 2 == 0 else 1
            path += [(turn, cc) for cc in range(c + 1, cols[k + 1])]
    path += [(h - 2, cols[-1]), (h - 1, cols[-1])]
    for z, (r, c) in enumerate(path):
        dem[r, c] = 5000.0 - z
    return dem


@pytest.mark.parametrize("method,exponent", METRIC_CASES)
def test_channel_crossing_seams_needs_several_rounds(checker, method, exponent):
    dem = serpentine_channel()
    for G in (2, 3):
        rounds = check_bands(checker, dem, G, method, exponent)
        if method != "D4":  # (FM_D4's proportions are read as D8 directions, so its flow leaves the channel)
            assert rounds > 2, (method, G, rounds)


@pytest.mark.parametrize("method,exponent", METRIC_CASES)
def test_bands_with_one_owned_row(checker, method, exponent):
    for shape, G in (((6, 40), 6), ((7, 33), 5), ((2, 9), 2), ((4, 12), 4)):
        dem = checker.resolve_flats(checker.fill_depressions(oracle.fbm_terrain(*shape, seed=shape[1], quantum=0.5)), ND)
        check_bands(checker, dem, G, method, exponent)
        check_bands(checker, dem, G, method, exponent, np.random.default_rng(3).random(dem.shape))


@pytest.mark.parametrize("method,exponent", METRIC_CASES)
def test_flow_into_nodata_ghost_cells(checker, method, exponent):
    """NoData on both sides of a seam, so that edge-row cells send shares into NoData ghost cells (dropped, as on one
    GPU) next to shares into ordinary ghost cells."""
    dem = resolved_fbm(checker)[:80, :120].copy()
    dem[40, 10:50] = ND   # first row of band 1 = band 0's bottom ghost row (G = 2)
    dem[39, 60:100] = ND  # last row of band 0 = band 1's top ghost row
    dem[39, 30:35] = ND   # NoData on both sides of the seam
    for G in (2, 4):
        check_bands(checker, dem, G, method, exponent)
        check_bands(checker, dem, G, method, exponent, np.random.default_rng(5).random(dem.shape))


@pytest.mark.parametrize("method,exponent", METRIC_CASES)
def test_cxx_band_driver_world_one(checker, method, exponent):
    """sharded.fa_band(method=...) takes the C++ driver (rdb200_mgpu_fa_method_f32_f64) by default; one band."""
    import torch
    dem = resolved_fbm(checker)
    t = torch.from_numpy(np.ascontiguousarray(dem)).to(DEV).contiguous()
    acc, rounds = sharded.fa_band(t, 0, 0, ND, method=method, exponent=exponent)
    assert rounds == 1
    np.testing.assert_allclose(acc.cpu().numpy(), single_gpu(dem, method, exponent), rtol=BAND_RTOL, atol=0)
    wts = np.random.default_rng(9).random(dem.shape)
    acc, _ = sharded.fa_band(t, 0, 0, ND, method=method, exponent=exponent,
                             weights=torch.from_numpy(wts).to(DEV).contiguous())
    np.testing.assert_allclose(acc.cpu().numpy(), single_gpu(dem, method, exponent, wts), rtol=BAND_RTOL, atol=0)


def test_method_aliases_and_errors():
    import torch
    dem = oracle.fbm_terrain(40, 36, seed=2, quantum=0.5)
    t = torch.from_numpy(dem).to(DEV).contiguous()
    def band(**kw):
        return sharded.fa_band(t, 0, 0, ND, **kw)[0].cpu().numpy()

    def same(a, b, what):  # (multi-receiver sums: atomics may land in another order)
        np.testing.assert_allclose(a, b, rtol=BAND_RTOL, atol=0, err_msg=what)

    ref = {name: band(method=name) for name in ("D8", "Dinf", "D4")}
    for alias, name in (("OCallaghanD8", "D8"), ("Tarboton", "Dinf"), ("OCallaghanD4", "D4")):
        same(band(method=alias), ref[name], alias)
    same(band(dinf=True), ref["Dinf"], "dinf=True")
    same(band(dinf=True, method="Tarboton"), ref["Dinf"], "dinf=True, Tarboton")
    same(band(), ref["D8"], "no method")
    same(band(method="Quinn"), band(method="Holmgren", exponent=1.0), "Quinn")
    same(band(method="Freeman", exponent=2.0), single_gpu(dem, "Freeman", 2.0), "Freeman")

    acc = torch.empty(t.shape, dtype=torch.float64, device=DEV)
    for m in ("Holmgren", "Freeman"):
        with pytest.raises(Exception, match="requires an exponent"):
            sharded.fa_band(t, 0, 0, ND, method=m)
        with pytest.raises(Exception, match="requires an exponent"):
            sharded.CudaBandAccumulator(t, acc, ND, 0, 0, False, True, method=m)
    with pytest.raises(Exception, match="Invalid FlowAccumulation method"):
        sharded.fa_band(t, 0, 0, ND, method="Steepest")
    with pytest.raises(Exception, match="Invalid FlowAccumulation method"):
        sharded.CudaBandAccumulator(t, acc, ND, 0, 0, False, True, method="Steepest")
    with pytest.raises(ValueError, match="dinf=True"):
        sharded.fa_band(t, 0, 0, ND, dinf=True, method="Quinn")

    # the C ABI refuses an unknown method and a non-finite exponent instead of running another method
    import ctypes as C
    L = _lib.lib()
    cm = sharded.lib_comm(None)
    xr = C.c_int32(0)
    for method, x, msg in ((5, 1.0, "unknown method"), (-1, 1.0, "unknown method"), (3, float("nan"), "finite exponent"),
                           (4, float("inf"), "finite exponent")):
        with pytest.raises(_lib.RichdemB200Error, match=msg):
            _lib.check(L.rdb200_mgpu_fa_method_f32_f64(cm.handle, t.data_ptr(), acc.data_ptr(), 36, 40, ND, 0, 0, method, x, 1,
                                                       C.byref(xr)))
        st = C.c_void_p()
        with pytest.raises(_lib.RichdemB200Error, match=msg):
            _lib.check(L.rdb200_dev_facc_begin_method(C.byref(st), t.data_ptr(), acc.data_ptr(), 36, 40, ND, 0, 0, method, x, 1))
