"""The float64 direction-grid pipeline without a GPU: barnes_flat_resolution_d8<double, uint8_t> (both alter modes) and
GetFlatMask<double>, on the CPU model of the shipped kernels (tests/emu), against the reference's double templates
stored in tests/golden/f64_flowdirs_flats_ref.npz (tests/golden/make_f64_flowdirs_flats.py).

* The float-step rule: the reference alters a double with nextafterf (flats/flat_resolution.hpp:565-568), so an altered
  cell is m float-ulp steps from the double rounded to float.  The fixtures hold steps that cross float exponent
  boundaries, first roundings down, to even and up, doubles above FLT_MAX (which become +inf) and float- and
  double-subnormal levels; the restatement oracle.f64_flowdirs.float_steps and the emulated kernels both give the
  reference's bits on them.
* The host and device entry points and richdem_b200.f64 on the emulated kernels: directions and altered DEM bit for bit,
  the flat mask bit for bit and its labels equal as a partition.
* The float64 band driver (sharded.d8_flow_directions_band with float64 tensors) over gloo with 1 to 4 bands, bit for
  bit against the single-GPU entry point, ghost rows included.
"""
import ctypes as C
import importlib.util
import multiprocessing as mp
import os
import socket
import sys

import numpy as np
import pytest

from oracle import f64_flowdirs as FD
from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "f64_flowdirs_flats_ref.npz")
FLT_MAX = float(np.finfo(np.float32).max)


def fixtures():
    g = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in g.files})
    return {n: {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(n + "/")} for n in names}


FIX = fixtures()
NAMES = sorted(FIX)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and bool(np.all(a.view(np.uint64) == b.view(np.uint64)))


def same_partition(a, b):
    """Equal labels within one flat, 0 exactly where the other is 0, and one label of a per label of b."""
    a, b = np.asarray(a).ravel(), np.asarray(b).ravel()
    if not np.array_equal(a == 0, b == 0):
        return False
    pairs = np.unique(np.stack([a, b]), axis=1)
    return len(np.unique(pairs[0])) == pairs.shape[1] == len(np.unique(pairs[1]))


def steps_of(f):
    """The increment count the reference applies to every cell: labelled interior cells only."""
    m = np.where(f["labels"] != 0, f["mask"], 0)
    m[0, :] = m[-1, :] = 0
    m[:, 0] = m[:, -1] = 0
    return m


def test_fixtures_cover_the_float_step_cases():
    """What the fixtures promise to exercise, checked on the reference's own output."""
    crossed = rounded_down = rounded_up = tie = overflow = subnormal = False
    for f in FIX.values():
        dem, dem1, m = f["dem"], f["dem1"], steps_of(f)
        sel = (m > 0) & ~np.isnan(dem)
        z, z1 = dem[sel], dem1[sel]
        with np.errstate(over="ignore", invalid="ignore"):
            r = z.astype(np.float32).astype(np.float64)
            ulp = np.abs(np.spacing(z.astype(np.float32)).astype(np.float64))
        fin = np.isfinite(r) & np.isfinite(z1)
        crossed |= bool(np.any(np.frexp(np.abs(r[fin]))[1] != np.frexp(np.abs(z1[fin]))[1]))
        with np.errstate(invalid="ignore"):
            frac = (z - np.floor(z / ulp) * ulp) / ulp
        rounded_down |= bool(np.any((r < z) & np.isfinite(r)))
        rounded_up |= bool(np.any((r > z) & np.isfinite(r)))
        tie |= bool(np.any(np.isclose(frac, 0.5)))
        overflow |= bool(np.any((np.abs(z) > FLT_MAX) & np.isinf(z1)))
        subnormal |= bool(np.any((z1 != 0) & (np.abs(z1) < np.finfo(np.float32).tiny)))
    assert crossed and rounded_down and rounded_up and tie and overflow and subnormal


# Without NoData the flats of the direction grid are those of GetFlatMask, so its mask gives the alteration's counts
@pytest.mark.parametrize("name", [n for n in NAMES if not n.startswith("nodata")])
def test_float_steps_restate_nextafterf(name):
    f = FIX[name]
    assert same_bits(FD.float_steps(f["dem"], steps_of(f)), f["dem1"]), name
    # the double ulps of ResolveFlatsEpsilon<double> are not the rule: they would change the answer here
    if name == "fbm_subfloat":
        from oracle import f64 as F
        assert not same_bits(F.advance_ulps(f["dem"], steps_of(f)), f["dem1"])


def test_golden_regenerates_to_the_same_bits():
    FD.build()
    if not FD.have_ref():
        pytest.skip("reference tree not available")
    from oracle import f64 as F
    F.build()
    mod = _load_module("make_f64_flowdirs_flats", os.path.join(HERE, "golden", "make_f64_flowdirs_flats.py"))
    R, RD = F.ref(), FD.ref()
    for name, (raw, nd) in mod.rasters().items():
        dem = R.fill(raw, "D8")
        assert same_bits(dem, FIX[name]["dem"]), name
        d1, dem1 = RD.flowdirs_flats(dem, nd, True)
        assert np.array_equal(d1, FIX[name]["dirs1"]) and same_bits(dem1, FIX[name]["dem1"]), name


# ---- the emulated kernels ---------------------------------------------------------------------------------------------
def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _emu_lib(path):
    L = C.CDLL(str(path))
    assert L.rdb200_emulated() == 1
    for name, argtypes in _lib.SIGNATURES.items():
        f = getattr(L, name)
        f.argtypes = argtypes
        f.restype = C.c_int
    L.rdb200_last_error.restype = C.c_char_p
    L.rdb200_last_error.argtypes = []
    L.rdb200_shutdown.restype = None
    return L


def _emu_path():
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    return str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())


@pytest.fixture(scope="module")
def emu_lib():
    return _emu_lib(_emu_path())


@pytest.fixture()
def emulated(emu_lib, monkeypatch):
    monkeypatch.setattr(_lib, "_lib", emu_lib)
    _lib.init(0)
    _lib.set_param("fill_use_tma", 0)  # TMA / mbarrier PTX is not emulated
    yield emu_lib
    _lib.reset_params()


def _host(L, dem, nd, alter, dev=False):
    d = np.array(dem, np.float64, copy=True, order="C")
    out = np.empty(d.shape, np.uint8)
    fn = L.rdb200_dev_d8_flow_directions_flats_f64 if dev else L.rdb200_d8_flow_directions_flats_f64
    assert fn(_lib.ptr(d), _lib.ptr(out), d.shape[1], d.shape[0], float(nd), int(alter)) == 0, L.rdb200_last_error()
    return out, d


@pytest.mark.parametrize("name", NAMES)
def test_emulated_entry_points_equal_the_reference(emulated, name):
    import richdem_b200 as rd
    from richdem_b200 import f64
    f = FIX[name]
    nd = float(f["nodata"])
    for dev in (False, True):  # the CPU model runs device entry points on host memory
        d0, z0 = _host(emulated, f["dem"], nd, False, dev)
        assert np.array_equal(d0, f["dirs0"]) and same_bits(z0, f["dem"]), (name, dev)
        d1, z1 = _host(emulated, f["dem"], nd, True, dev)
        assert np.array_equal(d1, f["dirs1"]) and same_bits(z1, f["dem1"]), (name, dev)
    dem = rd.rdarray(f["dem"].copy(), no_data=nd)
    assert np.array_equal(f64.FlowDirectionsD8Resolved(dem), f["dirs0"]) and same_bits(dem, f["dem"])
    assert np.array_equal(f64.FlowDirectionsD8Resolved(dem, alter=True), f["dirs1"]) and same_bits(dem, f["dem1"])
    mask, labels = f64.FlatMask(rd.rdarray(f["dem"].copy(), no_data=nd))
    assert np.array_equal(mask, f["mask"]) and same_partition(labels, f["labels"]), name
    assert np.array_equal(rd.D8FlowAccum(f["dirs0"]), f["area0"]), name


def test_emulated_argument_errors(emulated):
    L = emulated
    z = np.zeros((4, 4))
    d = np.zeros((4, 4), np.uint8)
    assert L.rdb200_d8_flow_directions_flats_f64(None, _lib.ptr(d), 4, 4, -9999.0, 0) == 1
    assert b"d8_flow_directions_flats: null pointer" in L.rdb200_last_error()
    assert L.rdb200_dev_d8_flow_directions_flats_f64(_lib.ptr(z), None, 4, 4, -9999.0, 1) == 1
    assert L.rdb200_get_flat_mask_f64(_lib.ptr(z), None, _lib.ptr(d), 4, 4, -9999.0) == 1
    assert b"get_flat_mask: null pointer" in L.rdb200_last_error()
    assert L.rdb200_d8_flow_directions_flats_f64(_lib.ptr(z), _lib.ptr(d), 0, 4, -9999.0, 0) == 1
    assert b"dimensions" in L.rdb200_last_error()


# ---- row bands over gloo ------------------------------------------------------------------------------------------------
BAND_CASES = ["fbm_subfloat", "fbm_between", "above_flt_max", "float_subnormal", "nodata_m32768", "beauford_1e-9"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, lib_path, cases, out_q):
    import torch
    import torch.distributed as dist
    from richdem_b200 import _lib, sharded

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        # point this process's Python layer at the kernel emulation (tests only; the loader itself refuses it)
        L = _emu_lib(lib_path)
        assert L.rdb200_init(0) == 0 and L.rdb200_set_param(b"fill_use_tma", 0) == 0
        _lib._lib = L
        _lib.use_torch_stream = lambda: None
        sharded._on_device = lambda t: True
        dist.init_process_group("gloo", rank=rank, world_size=world)
        res = {}
        for name, (dem, nd) in cases.items():
            h = dem.shape[0]
            r0, r1, gt, gb = sharded.local_rows(h, world, rank)
            for alter in (False, True):
                local = torch.from_numpy(np.ascontiguousarray(dem[r0 - gt:r1 + gb]).copy())
                dirs, _ = sharded.d8_flow_directions_band(local, gt, gb, nd, alter=alter)
                res[(name, alter)] = (dirs.numpy().copy(), local.numpy().copy(), gt, gb)
        # the argument checks fail before any exchange, on every rank alike
        local = torch.zeros((4, 5), dtype=torch.float64)
        try:
            sharded.d8_flow_directions_band(local, 1 - (rank > 0), 1, -9999.0)
            res["_bad_ghosts"] = None
        except Exception as e:  # noqa: BLE001
            res["_bad_ghosts"] = str(e)
        out_q.put((rank, res, None))
        dist.destroy_process_group()
    except Exception as e:  # noqa: BLE001
        import traceback
        out_q.put((rank, None, traceback.format_exc() + str(e)))


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_f64_band_driver_on_emulated_kernels(world):
    lib_path = _emu_path()
    L = _emu_lib(lib_path)
    assert L.rdb200_init(0) == 0 and L.rdb200_set_param(b"fill_use_tma", 0) == 0
    cases = {n: (FIX[n]["dem"], float(FIX[n]["nodata"])) for n in BAND_CASES}
    want = {(n, a): _host(L, dem, nd, a) for n, (dem, nd) in cases.items() for a in (False, True)}
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
        if world > 1:
            assert res["_bad_ghosts"] and "ghost" in res["_bad_ghosts"], (rank, res["_bad_ghosts"])
    for key, (dirs, dem) in want.items():
        got_d = np.concatenate([res[key][0][res[key][2]:res[key][0].shape[0] - res[key][3]] for _, res, _ in results])
        got_z = np.concatenate([res[key][1][res[key][2]:res[key][1].shape[0] - res[key][3]] for _, res, _ in results])
        assert np.array_equal(got_d, dirs), (key, int((got_d != dirs).sum()))
        assert same_bits(got_z, dem), key
        if key[1]:
            assert np.array_equal(dirs, FIX[key[0]]["dirs1"]) and same_bits(dem, FIX[key[0]]["dem1"])
        for rank, res, _ in results:  # ghost rows hold the neighbours' edge rows on return
            from richdem_b200 import sharded
            r0, r1, gt, gb = sharded.local_rows(dirs.shape[0], world, rank)
            d, z = res[key][0], res[key][1]
            if gt:
                assert np.array_equal(d[0], dirs[r0 - 1]), (key, rank)
                assert not key[1] or same_bits(z[0], dem[r0 - 1]), (key, rank)
            if gb:
                assert np.array_equal(d[-1], dirs[r1]), (key, rank)
                assert not key[1] or same_bits(z[-1], dem[r1]), (key, rank)
    assert all(p.exitcode == 0 for p in procs)
