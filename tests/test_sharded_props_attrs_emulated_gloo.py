"""Flow proportions, accumulation from given proportions and terrain attributes over row bands --
rdb200_mgpu_fm_method_f32, rdb200_mgpu_flow_accumulation_props_f64 and rdb200_mgpu_terrain_attribute_f32, reached through
sharded.flow_proportions_band / flow_accum_from_props_band / terrain_attribute_band -- over torch.distributed with the gloo
backend, one process per band, on the CPU model of the shipped kernels (tests/emu).

Every band's owned rows are compared with the single-GPU entry point on the whole raster, under the same model:
  * proportions of every FM method (Holmgren and Freeman with exponents other than 1) and all eight terrain attributes
    (zscale != 1, non-square cells), bit for bit, on a quantised fBm sprinkled with NoData and on rasters 5 and 7 rows tall,
    where some bands own one or two rows;
  * accumulation of those proportions, and of hand-made proportions that send flow across the seams into NoData cells and
    out of the raster's edge cells: one-hot proportions with unit weights bit for bit, everything else within 1e-9
    relative;
  * one case per function against the stored reference goldens.
The ghost rows handed in hold garbage: the calls must refresh them from the neighbours.  Bad arguments fail on every rank
before any communication."""
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
FM_CASES = [("D8", None), ("Dinf", None), ("D4", None), ("Quinn", None), ("Holmgren", 2.5), ("Holmgren", 0.7),
            ("Freeman", 1.1), ("Freeman", 4.0)]
ATTRIBS = ["slope_riserun", "slope_percentage", "slope_degrees", "slope_radians", "aspect", "curvature",
           "planform_curvature", "profile_curvature"]
ZSCALE, CELL = 2.5, (30.0, 20.0)
DX = [0, -1, -1, 0, 1, 1, 1, 0, -1]  # D8 neighbour n = 1..8: W, NW, N, NE, E, SE, S, SW
DY = [0, 0, -1, -1, -1, 0, 1, 1, 1]


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


def rasters():
    """Elevations: a quantised fBm with NoData blocks across the seams and a 4 % sprinkle of NoData cells (NoData on both
    sides of every seam), and two thin strips whose bands own one or two rows."""
    import oracle
    rng = np.random.default_rng(5)
    out = {}
    for name, (h, w, seed) in {"fbm": (46, 37, 61), "rows5": (5, 23, 62), "rows7": (7, 19, 63)}.items():
        z = oracle.fbm_terrain(h, w, seed=seed, quantum=0.25)
        z[rng.random((h, w)) < 0.04] = ND
        if h > 20:
            z[8:40, 12:16] = ND
        out[name] = np.ascontiguousarray(z)
    return out


def handmade_props(h, w, seed, one_hot):
    """Proportions of a random DAG (shares only go to neighbours of lower rank in a random order): 8 % NoData cells,
    interior cells sending to one or several lower neighbours -- NoData ones included -- and raster-edge cells with flow in
    every direction, off the raster too, which the accumulation must ignore."""
    rng = np.random.default_rng(seed)
    rank = rng.permutation(h * w).reshape(h, w)
    nodata = rng.random((h, w)) < 0.08
    p = np.zeros((h, w, 9), np.float32)
    p[..., 0] = -1.0
    for y in range(h):
        for x in range(w):
            if nodata[y, x]:
                p[y, x, 0] = -2.0
                continue
            edge = x == 0 or y == 0 or x == w - 1 or y == h - 1
            ks = [k for k in range(1, 9) if edge or rank[y + DY[k], x + DX[k]] < rank[y, x]]
            if not ks:
                continue
            if one_hot:
                ks = [ks[rng.integers(len(ks))]]
            else:
                ks = [k for k in ks if rng.random() < 0.7] or ks[:1]
            share = rng.random(len(ks)).astype(np.float32) + np.float32(0.05)
            share = share / share.sum(dtype=np.float32) if not one_hot else np.ones(1, np.float32)
            p[y, x, 0] = 0.0
            p[y, x, ks] = share
    return np.ascontiguousarray(p)


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
            src = case["dem"] if case["kind"] != "fa" else case["props"]
            h = src.shape[0]
            r0, r1, gt, gb = sharded.local_rows(h, world, rank)
            local = torch.from_numpy(np.ascontiguousarray(src[r0 - gt:r1 + gb]).copy())
            if gt:
                local[0] = 7.0  # garbage: the ghost rows must be refreshed by the call
            if gb:
                local[-1] = 0.5
            if case["kind"] == "fm":
                out = sharded.flow_proportions_band(local, gt, gb, ND, case["method"], case["exponent"])
                ghosts_src = local
            elif case["kind"] == "ta":
                out = sharded.terrain_attribute_band(local, gt, gb, case["attrib"], ND, zscale=ZSCALE, cell_x=CELL[0],
                                                     cell_y=CELL[1])
                ghosts_src = local
            else:
                wts = case["weights"]
                wl = None if wts is None else torch.from_numpy(np.ascontiguousarray(wts[r0 - gt:r1 + gb]).copy())
                out, rounds = sharded.flow_accum_from_props_band(local, gt, gb, weights=wl)
                res[key + "/rounds"] = rounds
                ghosts_src = local
            g = ghosts_src.numpy()
            res[key] = out.numpy()[gt:gt + r1 - r0].copy()
            res[key + "/ghosts"] = bool((not gt or np.array_equal(g[0], src[r0 - 1])) and
                                        (not gb or np.array_equal(g[-1], src[r1])))
        # bad arguments: every rank fails before the first collective
        dem = cases["fm/fbm/D8/None"]["dem"]
        h, w = dem.shape
        r0, r1, gt, gb = sharded.local_rows(h, world, rank)
        local = torch.from_numpy(np.ascontiguousarray(dem[r0 - gt:r1 + gb]).copy())
        props = torch.zeros(local.shape + (9,), dtype=torch.float32)
        acc = torch.ones(local.shape, dtype=torch.float64)
        out = torch.zeros(local.shape, dtype=torch.float32)
        cm = sharded.lib_comm()
        hl = local.shape[0]
        errors = {}

        def err(rc):
            return rc, (L.rdb200_last_error() or b"").decode()
        errors["fm ghosts"] = err(L.rdb200_mgpu_fm_method_f32(cm.handle, 0, local.data_ptr(), props.data_ptr(), w, hl, ND,
                                                              1 - gt, 1 - gb, 0.0))
        errors["fm method"] = err(L.rdb200_mgpu_fm_method_f32(cm.handle, 5, local.data_ptr(), props.data_ptr(), w, hl, ND, gt, gb,
                                                              0.0))
        errors["ta attribute"] = err(L.rdb200_mgpu_terrain_attribute_f32(cm.handle, 8, local.data_ptr(), out.data_ptr(), w, hl, ND,
                                                                         ND, 1.0, 1.0, 1.0, gt, gb))
        errors["ta cell"] = err(L.rdb200_mgpu_terrain_attribute_f32(cm.handle, 0, local.data_ptr(), out.data_ptr(), w, hl, ND, ND,
                                                                    1.0, 0.0, 1.0, gt, gb))
        errors["fa ghosts"] = err(L.rdb200_mgpu_flow_accumulation_props_f64(cm.handle, props.data_ptr(), acc.data_ptr(), w, hl,
                                                                            1 - gt, 1 - gb, None))
        errors["fa null"] = err(L.rdb200_mgpu_flow_accumulation_props_f64(cm.handle, props.data_ptr(), None, w, hl, gt, gb, None))
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
    """The single-GPU entry point on the whole raster, on the same kernel model."""
    if case["kind"] == "fm":
        dem = case["dem"]
        h, w = dem.shape
        out = np.empty((h, w, 9), np.float32)
        mid, x = _method_id(case["method"], case["exponent"])
        assert L.rdb200_dev_fm_method_f32(mid, dem.ctypes.data, out.ctypes.data, w, h, ND, x) == 0
        return out
    if case["kind"] == "ta":
        from richdem_b200 import _TERRAIN_ATTRIBS
        dem = case["dem"]
        h, w = dem.shape
        out = np.empty((h, w), np.float32)
        assert L.rdb200_dev_terrain_attribute_f32(_TERRAIN_ATTRIBS[case["attrib"]], dem.ctypes.data, out.ctypes.data, w, h,
                                                  ND, -9999.0, ZSCALE, CELL[0], CELL[1]) == 0
        return out
    p = case["props"]
    h, w = p.shape[:2]
    acc = np.ones((h, w)) if case["weights"] is None else case["weights"].copy()
    assert L.rdb200_dev_flow_accumulation_props_f64(p.ctypes.data, acc.ctypes.data, w, h) == 0
    return acc


def _cases(L, golden):
    dems = rasters()
    g = golden["flow_metrics_ref"]
    dems["s104"] = np.ascontiguousarray(g["s104__resolved"])
    dems["s106"] = np.ascontiguousarray(golden["terrain_attributes_ref"]["s106__dem"])
    cases = {}
    for dname in ("fbm", "rows5", "rows7"):
        for m, e in FM_CASES:
            cases[f"fm/{dname}/{m}/{e}"] = {"kind": "fm", "dem": dems[dname], "method": m, "exponent": e}
        for a in ATTRIBS:
            cases[f"ta/{dname}/{a}"] = {"kind": "ta", "dem": dems[dname], "attrib": a}
    cases["fm/s104/D4/None"] = {"kind": "fm", "dem": dems["s104"], "method": "D4", "exponent": None}
    cases["ta/s106/slope_riserun"] = {"kind": "ta", "dem": dems["s106"], "attrib": "slope_riserun"}
    # accumulation: the single-GPU proportions of the rasters above, and hand-made ones
    rng = np.random.default_rng(9)
    for key in [k for k in cases if k.startswith("fm/")]:
        props = _single(L, cases[key])
        _, dname, m, _e = key.split("/")
        if dname != "fbm" and m not in ("D8", "Holmgren"):
            continue
        exact = m in ("D8", "D4")
        cases["fa" + key[2:] + "/ones"] = {"kind": "fa", "props": props, "weights": None, "exact": exact}
        if dname == "fbm":
            cases["fa" + key[2:] + "/weights"] = {"kind": "fa", "props": props, "weights": rng.random(props.shape[:2]),
                                                  "exact": False}
    for (h, w), seed in (((31, 29), 11), ((5, 17), 12), ((7, 13), 13)):
        for one_hot in (True, False):
            p = handmade_props(h, w, seed, one_hot)
            cases[f"fa/hand/{h}x{w}/{int(one_hot)}/ones"] = {"kind": "fa", "props": p, "weights": None, "exact": one_hot}
            cases[f"fa/hand/{h}x{w}/{int(one_hot)}/weights"] = {"kind": "fa", "props": p, "weights": rng.random((h, w)),
                                                               "exact": False}
    return cases


def _crossings(p, world):
    """(shares across a seam into a NoData cell, raster-edge cells with flow) of proportions p cut into `world` bands."""
    from richdem_b200 import sharded
    h, w = p.shape[:2]
    seams = [r1 for _, r1 in sharded.band_bounds(h, world)[:-1]]
    into_nodata = 0
    for s in seams:
        for y, dys in ((s - 1, (1,)), (s, (-1,))):
            for x in range(1, w - 1):
                if p[y, x, 0] == -2:
                    continue
                for k in range(1, 9):
                    if DY[k] in dys and p[y, x, k] > 0 and p[y + DY[k], x + DX[k], 0] == -2:
                        into_nodata += 1
    edge = np.zeros((h, w), bool)
    edge[[0, -1], :] = True
    edge[:, [0, -1]] = True
    return into_nodata, int((edge & (p[..., 1:] > 0).any(axis=2)).sum())


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_props_attrs_band_drivers_on_emulated_kernels(world, golden):
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    lib_path = str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())
    L = _emu_lib(lib_path)
    cases = _cases(L, golden)
    if world > 1:
        into_nodata, edge_flow = _crossings(cases["fa/hand/31x29/0/ones"]["props"], world)
        assert into_nodata > 0 and edge_flow > 0
    expected = {k: _single(L, c) for k, c in cases.items()}
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, lib_path, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted((q.get(timeout=900) for _ in range(world)), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        errors = res["_errors"]
        assert errors["fm ghosts"][0] != 0 and "ghost_top" in errors["fm ghosts"][1], (rank, errors)
        assert errors["fa ghosts"][0] != 0 and "ghost_top" in errors["fa ghosts"][1], (rank, errors)
        assert errors["fm method"][0] != 0 and "unknown flow metric" in errors["fm method"][1], (rank, errors)
        assert errors["ta attribute"][0] != 0 and "unknown terrain attribute" in errors["ta attribute"][1], (rank, errors)
        assert errors["ta cell"][0] != 0 and "cell lengths" in errors["ta cell"][1], (rank, errors)
        assert errors["fa null"][0] != 0 and "null pointer" in errors["fa null"][1], (rank, errors)
    for key, case in cases.items():
        got = np.concatenate([res[key] for _, res, _ in results])
        want = expected[key]
        assert all(res[key + "/ghosts"] for _, res, _ in results), key
        if case["kind"] != "fa":
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (key, int((got != want).sum()))
        elif case["exact"]:
            assert np.array_equal(got, want), (key, int((got != want).sum()))
        else:
            assert np.array_equal(got == -1, want == -1), key
            np.testing.assert_allclose(got, want, rtol=1e-9, atol=0, err_msg=key)
        if case["kind"] == "fa" and world > 1 and key.startswith("fa/fbm"):
            assert max(res[key + "/rounds"] for _, res, _ in results) >= 2, key
    # one case per function against the reference's stored outputs
    got = {k: np.concatenate([res[k] for _, res, _ in results]) for k in ("fm/s104/D4/None", "ta/s106/slope_riserun")}
    g = golden["flow_metrics_ref"]
    assert np.array_equal(got["fm/s104/D4/None"].reshape(-1, 9)[::11], g["s104__D4_None__fm"])
    assert np.array_equal(got["ta/s106/slope_riserun"][::3, ::3].view(np.uint32),
                          golden["terrain_attributes_ref"]["s106__slope_riserun__2.5"].view(np.uint32))
    assert all(p.exitcode == 0 for p in procs)


def test_golden_accumulation_from_band_props(golden):
    """FlowAccumFromProps of FM_D4 proportions of the s104 raster over three bands against the reference's FA_D4."""
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    lib_path = str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())
    L = _emu_lib(lib_path)
    g = golden["flow_metrics_ref"]
    props = _single(L, {"kind": "fm", "dem": np.ascontiguousarray(g["s104__resolved"]), "method": "D4", "exponent": None})
    world = 3
    cases = {"fm/fbm/D8/None": {"kind": "fm", "dem": rasters()["fbm"], "method": "D8", "exponent": None},
             "fa/s104/D4": {"kind": "fa", "props": props, "weights": None}}
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, lib_path, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted((q.get(timeout=900) for _ in range(world)), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
    got = np.concatenate([res["fa/s104/D4"] for _, res, _ in results])
    np.testing.assert_allclose(got[::3, ::3], g["s104__D4_None__fa"], rtol=1e-9, atol=0)
    assert all(p.exitcode == 0 for p in procs)


def test_band_wrappers_validate_names_as_the_public_api():
    import torch
    from richdem_b200 import sharded
    dem = torch.zeros((4, 5), dtype=torch.float32)
    for m, msg in (("Rho8", 'FlowProportions method "Rho8" is outside the GPU hot path'),
                   ("Rho4", 'FlowProportions method "Rho4" is outside the GPU hot path'),
                   ("Holmgren", 'FlowProportions method "Holmgren" requires an exponent!'),
                   ("Freeman", 'FlowProportions method "Freeman" requires an exponent!'),
                   ("bogus", "Invalid FlowProportions method. Valid methods are: Dinf, Tarboton, Quinn"),
                   (None, "Invalid FlowProportions method")):
        with pytest.raises(Exception) as ei:
            sharded.flow_proportions_band(dem, 0, 0, ND, m)
        assert str(ei.value).startswith(msg), (m, str(ei.value))
    with pytest.raises(Exception, match="Invalid TerrainAttributes attribute. Valid attributes are: slope_riserun"):
        sharded.terrain_attribute_band(dem, 0, 0, "slope", ND)
    with pytest.raises(RuntimeError, match="last of size 9"):
        sharded.flow_accum_from_props_band(torch.zeros((4, 5, 8), dtype=torch.float32), 0, 0)
    # the FlowAccumulation names keep their own messages
    with pytest.raises(Exception, match='FlowAccumulation method "Rho8" is outside'):
        sharded.fa_method_id("Rho8", None)
