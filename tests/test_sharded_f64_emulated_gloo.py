"""float64 rasters over row bands -- rdb200_mgpu_*_f64 and rdb200_mgpu_f64_order_keys, reached through the sharded band
functions with float64 tensors -- over torch.distributed with the gloo backend, one process per band, on the CPU model
of the shipped kernels (tests/emu).

Every band's owned rows are compared with the single-GPU float64 entry point on the whole raster, under the same model:
  * FillDepressions D8 / D4 (bit for bit up to the sign of a zero), pit_mask, HasDepressions, ResolveFlatsEpsilon, every
    flow metric and all eight terrain attributes (zscale != 1, non-square cells): bit for bit;
  * FA_D8 / FA_D4 with unit weights bit for bit; weighted accumulation and D-infinity / Quinn / Holmgren / Freeman within
    1e-9 relative;
  * the order keys kappa_G: the same order as the values in every band count, equal keys for equal values across bands,
    and kappa_G(nodata) the key of a cell equal to nodata in any band.
The rasters: fBm with sub-float detail (global ranks), a widened float raster (cast route), one float-exact band among
inexact ones, a lake whose spill level lies only in another band, lakes one double ulp apart, DBL_MAX plateaus, +-inf,
NaN, +-0, subnormals and +-1e300, and NoData in one band only, nowhere, and at +-inf; heights 5 and 7 give bands of one
or two rows.  The ghost rows handed in hold garbage.  A lowered rank cap fails on every rank at once, and the next call
works."""
import ctypes as C
import importlib.util
import multiprocessing as mp
import os
import socket
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0
FM_CASES = [("D8", None), ("Dinf", None), ("D4", None), ("Quinn", None), ("Holmgren", 2.5), ("Freeman", 1.1)]
ATTRIBS = ["slope_riserun", "slope_percentage", "slope_degrees", "slope_radians", "aspect", "curvature",
           "planform_curvature", "profile_curvature"]
ZSCALE, CELL = 2.5, (30.0, 20.0)
DMAX = np.finfo(np.float64).max


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _emu_lib(lib_path):
    from richdem_b200 import _lib
    L = C.CDLL(lib_path)
    for name, argtypes in _lib.SIGNATURES.items():
        f = getattr(L, name)
        f.argtypes = argtypes
        f.restype = C.c_int
    L.rdb200_last_error.restype = C.c_char_p
    L.rdb200_last_error.argtypes = []
    assert L.rdb200_init(0) == 0 and L.rdb200_set_param(b"fill_use_tma", 0) == 0
    return L


def _lake(h, w, rng, sill, lake_rows, col):
    """A bowl of cells near 1 in lake_rows, walls near 50 and a corridor in column `col` up to the top edge whose highest
    cell (row 2) is `sill`: the lake fills to `sill`, a value that occurs nowhere else."""
    z = 50.0 + rng.random((h, w)) * 1e-3
    z[lake_rows[0]:lake_rows[1], 2:w - 2] = 1.0 + rng.random((lake_rows[1] - lake_rows[0], w - 4)) * 1e-9
    z[1:lake_rows[0], col] = 5.0 + rng.random(lake_rows[0] - 1) * 1e-9
    z[2, col] = sill
    z[0, col] = 0.5
    return z


def rasters():
    import oracle
    rng = np.random.default_rng(17)
    out = {}
    base = oracle.fbm_terrain(24, 19, seed=71, quantum=0.25).astype(np.float64)
    fbm = base + rng.random(base.shape) * 1e-6  # sub-float detail: the float cast would merge values
    fbm[rng.random(fbm.shape) < 0.04] = ND
    fbm[9:15, 6:9] = ND  # across the seams
    out["fbm"] = fbm
    out["widened"] = oracle.fbm_terrain(22, 17, seed=72, quantum=0.25).astype(np.float32).astype(np.float64)
    mixed = oracle.fbm_terrain(20, 15, seed=73, quantum=0.25).astype(np.float64)
    mixed[6:] += rng.random(mixed[6:].shape) * 1e-7  # the first band(s) float-exact, the others not
    out["mixed"] = mixed
    out["remote_lake"] = _lake(18, 11, rng, 7.123456789012345, (10, 16), 5)
    s = 7.25 + 1e-12
    nest = _lake(18, 13, rng, s, (9, 16), 4)
    nest[1:9, 8] = 5.0 + rng.random(8) * 1e-9  # a second corridor out of the same bowl, its sill one ulp higher
    nest[3, 8] = np.nextafter(s, np.inf)
    nest[0, 8] = 0.5
    nest[12, 2:11] = np.nextafter(s, -np.inf)  # a wall one ulp below the level splits the lake into two
    out["nested_ulp"] = nest
    sp = oracle.fbm_terrain(21, 16, seed=74, quantum=0.25).astype(np.float64) + rng.random((21, 16)) * 1e-8
    sp[3:6, 3:7] = DMAX
    sp[12:15, 9:13] = DMAX
    sp[7, 2], sp[8, 5], sp[16, 4] = np.inf, -np.inf, np.nan
    sp[10, 10], sp[11, 3], sp[17, 12] = 0.0, -0.0, 0.0
    sp[5, 12], sp[18, 7] = 5e-324, -2.5e-310
    sp[2, 9], sp[19, 2] = 1e300, -1e300
    sp[9, 14] = -DMAX
    out["specials"] = sp
    rows5 = oracle.fbm_terrain(5, 23, seed=75, quantum=0.25).astype(np.float64) + rng.random((5, 23)) * 1e-7
    rows5[rng.random(rows5.shape) < 0.05] = ND
    out["rows5"] = rows5
    rows7 = oracle.fbm_terrain(7, 19, seed=76, quantum=0.25).astype(np.float64) + rng.random((7, 19)) * 1e-7
    out["rows7"] = rows7
    # NoData in the last rows only (one band), nowhere, and NoData = -inf
    nd_one = oracle.fbm_terrain(20, 14, seed=77, quantum=0.25).astype(np.float64) + rng.random((20, 14)) * 1e-7
    nd_one[17:19, 4:9] = ND
    out["nd_one_band"] = nd_one
    out["nd_none"] = oracle.fbm_terrain(20, 14, seed=78, quantum=0.25).astype(np.float64) + rng.random((20, 14)) * 1e-7
    nd_inf = oracle.fbm_terrain(20, 14, seed=79, quantum=0.25).astype(np.float64) + rng.random((20, 14)) * 1e-7
    nd_inf[8:13, 5:8] = -np.inf
    out["nd_minus_inf"] = nd_inf
    return {k: np.ascontiguousarray(v) for k, v in out.items()}


NODATA = {"nd_minus_inf": -np.inf}


def _cases():
    dems = rasters()
    cases = {}
    full = ("fbm", "specials")
    for name, dem in dems.items():
        nd = NODATA.get(name, ND)
        c = lambda **kw: dict(dem=dem, nodata=nd, **kw)  # noqa: E731
        cases[f"keys/{name}"] = c(kind="keys")
        for topo in ("D8", "D4"):
            cases[f"fill/{name}/{topo}"] = c(kind="fill", topo=topo)
            if name in full or name.startswith("nd_"):
                cases[f"pit/{name}/{topo}"] = c(kind="pit", topo=topo)
                cases[f"hasdep/{name}/{topo}"] = c(kind="hasdep", topo=topo)
        cases[f"flats/{name}"] = c(kind="flats")
        cases[f"fa/{name}/D8/ones"] = c(kind="fa", method="D8", exponent=None, weights=False)
        if name in full or name in ("rows5", "rows7", "remote_lake"):
            cases[f"fa/{name}/D4/ones"] = c(kind="fa", method="D4", exponent=None, weights=False)
            for m, e in FM_CASES:
                cases[f"fm/{name}/{m}/{e}"] = c(kind="fm", method=m, exponent=e)
            for a in ATTRIBS:
                cases[f"ta/{name}/{a}"] = c(kind="ta", attrib=a)
        if name in ("fbm", "rows7"):
            cases[f"fa/{name}/D8/weights"] = c(kind="fa", method="D8", exponent=None, weights=True)
            for m, e in (("Dinf", None), ("Quinn", None), ("Holmgren", 2.5), ("Freeman", 1.1)):
                cases[f"fa/{name}/{m}/ones"] = c(kind="fa", method=m, exponent=e, weights=False)
            cases[f"fa/{name}/Freeman/weights"] = c(kind="fa", method="Freeman", exponent=1.1, weights=True)
    # hasdep on a raster without depressions: the answer needs the keyed band fill
    cases["hasdep/widened_filled/D8"] = dict(dem=None, nodata=ND, kind="hasdep", topo="D8", fill_first="widened")
    cases["hasdep/fbm_filled/D4"] = dict(dem=None, nodata=ND, kind="hasdep", topo="D4", fill_first="fbm")
    return cases


def _weights(dem):
    return np.random.default_rng(dem.shape[0] * 31 + dem.shape[1]).random(dem.shape)


def _fill_ok(h, world):
    from richdem_b200 import sharded
    return all(r1 - r0 + (g > 0) + (g < world - 1) >= 3 for g, (r0, r1) in enumerate(sharded.band_bounds(h, world)))


def _worker(rank, world, port, lib_path, cases, out_q):
    import torch
    import torch.distributed as dist
    from richdem_b200 import _lib, sharded

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        # point this process's Python layer at the kernel emulation (tests only; the loader itself refuses it)
        L = _emu_lib(lib_path)
        _lib._lib = L
        _lib.use_torch_stream = lambda: None
        sharded._on_device = lambda t: True
        dist.init_process_group("gloo", rank=rank, world_size=world)
        res = {}
        for key, case in cases.items():
            src = case["dem"]
            h = src.shape[0]
            if case["kind"] in ("fill", "pit", "hasdep") and not _fill_ok(h, world):
                continue
            r0, r1, gt, gb = sharded.local_rows(h, world, rank)
            local = torch.from_numpy(np.ascontiguousarray(src[r0 - gt:r1 + gb]).copy())
            if gt:
                local[0] = 7.0  # garbage: no driver may read the ghost rows it is handed
            if gb:
                local[-1] = np.nan
            own = slice(gt, gt + r1 - r0)
            k, nd = case["kind"], case["nodata"]
            if k == "keys":
                keys, ndk, ranked = sharded.f64_order_keys_band(local, gt, gb, nd)
                res[key] = (keys.numpy()[own].copy(), ndk, ranked)
            elif k == "fill":
                out, _ = sharded.fill_band(local, gt, gb, topology=case["topo"])
                g = out.numpy()
                res[key] = g[own].copy()
                res[key + "/ghosts"] = (g[0].copy() if gt else None, g[-1].copy() if gb else None)
            elif k == "pit":
                res[key] = sharded.pit_mask_band(local, gt, gb, nd, topology=case["topo"]).numpy()[own].copy()
            elif k == "hasdep":
                res[key] = sharded.has_depressions_band(local, gt, gb, topology=case["topo"])
            elif k == "flats":
                sharded.resolve_flats_band(local, gt, gb, nd)
                g = local.numpy()
                res[key] = g[own].copy()
                res[key + "/ghosts"] = (g[0].copy() if gt else None, g[-1].copy() if gb else None)
            elif k == "fm":
                res[key] = sharded.flow_proportions_band(local, gt, gb, nd, case["method"], case["exponent"]).numpy()[own].copy()
            elif k == "ta":
                res[key] = sharded.terrain_attribute_band(local, gt, gb, case["attrib"], nd, zscale=ZSCALE, cell_x=CELL[0],
                                                          cell_y=CELL[1]).numpy()[own].copy()
            else:
                wl = None
                if case["weights"]:
                    wl = torch.from_numpy(np.ascontiguousarray(_weights(src)[r0 - gt:r1 + gb]).copy())
                acc, _ = sharded.fa_band(local, gt, gb, nd, method=case["method"], exponent=case["exponent"], weights=wl)
                res[key] = acc.numpy()[own].copy()
        # a rank cap below the raster's distinct values: every rank fails in kappa_G, before any stage; the next call works
        dem = cases["fill/fbm/D8"]["dem"]
        h, w = dem.shape
        r0, r1, gt, gb = sharded.local_rows(h, world, rank)
        local = torch.from_numpy(np.ascontiguousarray(dem[r0 - gt:r1 + gb]).copy())
        errors = {}

        def err(rc):
            return rc, (L.rdb200_last_error() or b"").decode()
        cm = sharded.lib_comm()
        hl = local.shape[0]
        assert L.rdb200_set_param(b"f64_band_rank_cap", 50) == 0
        errors["cap"] = err(L.rdb200_mgpu_fill_depressions_d8_f64(cm.handle, local.data_ptr(), w, hl, gt, gb, r0 - gt, h, None))
        assert L.rdb200_set_param(b"f64_band_rank_cap", 0) == 0
        res["after_cap"] = sharded.fill_band(local.clone(), gt, gb)[0].numpy()[gt:gt + r1 - r0].copy()
        acc = torch.ones(local.shape, dtype=torch.float64)
        mask = torch.zeros(local.shape, dtype=torch.uint8)
        errors["fill ghosts"] = err(L.rdb200_mgpu_fill_depressions_d8_f64(cm.handle, local.data_ptr(), w, hl, 1 - gt, 1 - gb,
                                                                          r0 - gt, h, None))
        errors["pit rows"] = err(L.rdb200_mgpu_pit_mask_d8_f64(cm.handle, local.data_ptr(), mask.data_ptr(), w, hl, ND, gt, gb,
                                                               r0 - gt, r0 - gt + hl - 1))
        errors["fa method"] = err(L.rdb200_mgpu_fa_method_f64_f64(cm.handle, local.data_ptr(), acc.data_ptr(), w, hl, ND, gt, gb,
                                                                  5, 0.0, 1, None))
        props = torch.zeros(local.shape + (9,), dtype=torch.float32)
        errors["fm method"] = err(L.rdb200_mgpu_fm_method_f64(cm.handle, 7, local.data_ptr(), props.data_ptr(), w, hl, ND, gt, gb,
                                                              0.0))
        try:
            sharded.fill_band(local, gt, gb, solver_cls=object)
            errors["python protocol"] = (0, "")
        except ValueError as e:
            errors["python protocol"] = (1, str(e))
        res["_errors"] = errors
        out_q.put((rank, res, None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _method_id(method, exponent):
    from richdem_b200 import sharded
    return sharded._method_id(method, exponent, "FlowProportions")


def _single(L, case):
    """The single-GPU float64 entry point on the whole raster, on the same kernel model."""
    dem, nd, k = case["dem"], case["nodata"], case["kind"]
    h, w = dem.shape
    topo4 = case.get("topo") == "D4"
    if k == "keys":
        return None
    if k == "fill":
        z = dem.copy()
        fn = L.rdb200_dev_fill_depressions_d4_f64 if topo4 else L.rdb200_dev_fill_depressions_d8_f64
        assert fn(z.ctypes.data, w, h) == 0
        return z
    if k == "pit":
        m = np.empty((h, w), np.uint8)
        fn = L.rdb200_dev_pit_mask_d4_f64 if topo4 else L.rdb200_dev_pit_mask_d8_f64
        assert fn(dem.ctypes.data, m.ctypes.data, w, h, nd) == 0
        return m
    if k == "hasdep":
        o = C.c_int32(0)
        fn = L.rdb200_dev_has_depressions_d4_f64 if topo4 else L.rdb200_dev_has_depressions_d8_f64
        assert fn(dem.ctypes.data, w, h, C.byref(o)) == 0
        return bool(o.value)
    if k == "flats":
        z = dem.copy()
        assert L.rdb200_dev_resolve_flats_epsilon_f64(z.ctypes.data, w, h, nd) == 0
        return z
    if k == "fm":
        out = np.empty((h, w, 9), np.float32)
        mid, x = _method_id(case["method"], case["exponent"])
        assert L.rdb200_dev_fm_method_f64(mid, dem.ctypes.data, out.ctypes.data, w, h, nd, x) == 0
        return out
    if k == "ta":
        from richdem_b200 import _TERRAIN_ATTRIBS
        out = np.empty((h, w), np.float32)
        assert L.rdb200_dev_terrain_attribute_f64(_TERRAIN_ATTRIBS[case["attrib"]], dem.ctypes.data, out.ctypes.data, w, h, nd,
                                                  -9999.0, ZSCALE, CELL[0], CELL[1]) == 0
        return out
    mid, x = _method_id(case["method"], case["exponent"])
    acc = _weights(dem) if case["weights"] else np.ones((h, w))
    assert L.rdb200_dev_fa_method_f64_f64(mid, dem.ctypes.data, acc.ctypes.data, w, h, nd, x) == 0
    return acc


def _same_fill(got, want):
    """bit for bit, except that a zero may come back with either sign"""
    gb, wb = got.view(np.uint64), want.view(np.uint64)
    return bool(np.all((gb == wb) | ((got == 0) & (want == 0))))


def _check_keys(key, dem, keys, ndk, nodata):
    """kappa_G is strictly increasing on the values, equal for equal values (+-0 together, NaN to NaN), keeps the images of
    +-inf and +-DBL_MAX, and kappa_G(nodata) is the key of a cell equal to nodata."""
    v, k = dem.ravel(), keys.ravel()
    nan = np.isnan(v)
    assert np.array_equal(nan, np.isnan(k)), key
    v, k = v[~nan], k[~nan].astype(np.float64)
    o = np.argsort(v, kind="stable")
    vs, ks = v[o], k[o]
    up = vs[1:] > vs[:-1]
    assert np.all(ks[1:][up] > ks[:-1][up]), key
    assert np.all(ks[1:][~up] == ks[:-1][~up]), key
    f32max = float(np.finfo(np.float32).max)
    for val, img in ((np.inf, np.inf), (-np.inf, -np.inf), (DMAX, f32max), (-DMAX, -f32max)):
        assert np.all(k[v == val] == img), (key, val)
    if np.any(dem == nodata):
        assert ndk == k[v == nodata][0], key
    elif np.isfinite(nodata):
        assert np.isnan(ndk), key
    else:
        assert ndk == nodata, key


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5])
def test_f64_band_drivers_on_emulated_kernels(world):
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    from richdem_b200 import sharded
    lib_path = str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())
    L = _emu_lib(lib_path)
    cases = _cases()
    for c in cases.values():
        if c.get("fill_first"):
            src = rasters()[c["fill_first"]]
            c["dem"] = _single(L, dict(dem=src, nodata=ND, kind="fill", topo=c["topo"]))
    expected = {k: _single(L, c) for k, c in cases.items()}
    assert expected["hasdep/fbm/D8"] and not expected["hasdep/widened_filled/D8"] and not expected["hasdep/fbm_filled/D4"]
    # the lakes fill to levels that occur in one place only
    for name, sill in (("remote_lake", 7.123456789012345), ("nested_ulp", 7.25 + 1e-12)):
        assert np.sum(cases[f"fill/{name}/D8"]["dem"] == sill) == 1 and np.sum(expected[f"fill/{name}/D8"] == sill) > 20
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, lib_path, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted((q.get(timeout=1800) for _ in range(world)), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        e = res["_errors"]
        assert e["cap"][0] == 1 and "distinct values" in e["cap"][1], (rank, e)
        assert e["fill ghosts"][0] == 1 and "ghost_top" in e["fill ghosts"][1], (rank, e)
        assert e["pit rows"][0] == 1 and "outside the raster" in e["pit rows"][1], (rank, e)
        assert e["fa method"][0] == 1 and "unknown method" in e["fa method"][1], (rank, e)
        assert e["fm method"][0] == 1 and "unknown flow metric" in e["fm method"][1], (rank, e)
        assert e["python protocol"][0] == 1 and "float64" in e["python protocol"][1], (rank, e)
    after = np.concatenate([res["after_cap"] for _, res, _ in results])
    assert _same_fill(after, expected["fill/fbm/D8"])
    checked = 0
    for key, case in cases.items():
        if key not in results[0][1]:
            assert not _fill_ok(case["dem"].shape[0], world), key
            continue
        checked += 1
        kind, want = case["kind"], expected[key]
        if kind == "hasdep":
            assert all(res[key] == want for _, res, _ in results), key
            continue
        if kind == "keys":
            keys = np.concatenate([res[key][0] for _, res, _ in results])
            nds = {np.float32(res[key][1]).view(np.uint32).item() for _, res, _ in results}
            assert len(nds) == 1 and len({res[key][2] for _, res, _ in results}) == 1, key
            _check_keys(key, case["dem"], keys, results[0][1][key][1], case["nodata"])
            ranked = results[0][1][key][2]
            assert ranked == (key != "keys/widened"), key  # one inexact band puts every band on global ranks
            continue
        got = np.concatenate([res[key] for _, res, _ in results])
        if kind == "fill":
            assert _same_fill(got, want), (key, int((got != want).sum()))
        elif kind in ("pit", "flats", "fm", "ta"):
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (key, int((got != want).sum()))
        elif case["method"] in ("D8", "D4") and not case["weights"]:
            assert np.array_equal(got, want), (key, int((got != want).sum()))
        else:
            assert np.array_equal(got == -1, want == -1), key
            np.testing.assert_allclose(got, want, rtol=1e-9, atol=0, err_msg=key)
        if kind in ("fill", "flats"):  # the ghost rows hold the neighbours' results on return
            full = want
            for rank, res, _ in results:
                r0, r1, gt, gb = sharded.local_rows(full.shape[0], world, rank)
                top, bot = res[key + "/ghosts"]
                assert top is None or _same_fill(top, full[r0 - 1]), (key, rank)
                assert bot is None or _same_fill(bot, full[r1]), (key, rank)
    assert checked > 100
    assert all(p.exitcode == 0 for p in procs)
