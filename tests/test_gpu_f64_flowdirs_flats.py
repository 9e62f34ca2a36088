"""The float64 direction-grid pipeline on the H100: barnes_flat_resolution_d8<double, uint8_t> (alter false and true) and
GetFlatMask<double> through the host and device entry points, richdem_b200.f64 and the C++ specialisation, against the
reference's double templates in tests/golden/f64_flowdirs_flats_ref.npz: directions and altered DEM bit for bit, the mask
bit for bit and its labels as a partition.  Then the whole pipeline (f64 fill, resolved directions, D8FlowAccum) from
the raw rasters; the float64 band driver with 1 to 4 processes sharing the GPU over gloo against one GPU; and a
16384 x 16384 fBm whose values are floats, on which the float64 path must give the float32 path's bits."""
import ctypes as C
import multiprocessing as mp
import os
import socket
import subprocess

import numpy as np
import pytest

import richdem_b200 as rd
from richdem_b200 import _lib, f64

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "f64_flowdirs_flats_ref.npz")


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
    a, b = np.asarray(a).ravel(), np.asarray(b).ravel()
    if not np.array_equal(a == 0, b == 0):
        return False
    pairs = np.unique(np.stack([a, b]), axis=1)
    return len(np.unique(pairs[0])) == pairs.shape[1] == len(np.unique(pairs[1]))


@pytest.mark.parametrize("name", NAMES)
def test_entry_points_equal_the_reference(name):
    import torch
    f = FIX[name]
    nd = float(f["nodata"])
    L = _lib.lib()
    h, w = f["dem"].shape
    for alter in (0, 1):
        z = f["dem"].copy()
        d = np.empty(z.shape, np.uint8)
        _lib.check(L.rdb200_d8_flow_directions_flats_f64(_lib.ptr(z), _lib.ptr(d), w, h, nd, alter))
        assert np.array_equal(d, f[f"dirs{alter}"]) and same_bits(z, f["dem1" if alter else "dem"]), (name, alter)
        zt = torch.from_numpy(f["dem"].copy()).cuda()
        dt = torch.empty((h, w), dtype=torch.uint8, device="cuda")
        _lib.use_torch_stream()
        _lib.check(L.rdb200_dev_d8_flow_directions_flats_f64(zt.data_ptr(), dt.data_ptr(), w, h, nd, alter))
        torch.cuda.synchronize()
        assert np.array_equal(dt.cpu().numpy(), f[f"dirs{alter}"]), (name, alter)
        assert same_bits(zt.cpu().numpy(), f["dem1" if alter else "dem"]), (name, alter)
    dem = rd.rdarray(f["dem"].copy(), no_data=nd)
    assert np.array_equal(f64.FlowDirectionsD8Resolved(dem), f["dirs0"]) and same_bits(dem, f["dem"]), name
    assert np.array_equal(f64.FlowDirectionsD8Resolved(dem, alter=True), f["dirs1"]) and same_bits(dem, f["dem1"]), name
    mask, labels = f64.FlatMask(rd.rdarray(f["dem"].copy(), no_data=nd))
    assert np.array_equal(mask, f["mask"]) and same_partition(labels, f["labels"]), name
    assert np.array_equal(rd.D8FlowAccum(f["dirs0"]), f["area0"]), name


@pytest.mark.parametrize("name", [n for n in NAMES if "raw" in FIX[n]])
def test_fill_resolved_directions_accumulation_pipeline(name):
    f = FIX[name]
    nd = float(f["nodata"])
    filled = f64.FillDepressions(rd.rdarray(f["raw"].copy(), no_data=nd))
    z = np.asarray(filled).copy()
    z[z == 0] = 0.0  # the fill's zero sign is not promised
    ref = f["dem"].copy()
    ref[ref == 0] = 0.0
    assert same_bits(z, ref), name
    dirs = f64.FlowDirectionsD8Resolved(filled)
    assert np.array_equal(dirs, f["dirs0"]), name
    assert np.array_equal(rd.D8FlowAccum(dirs), f["area0"]), name


def test_cxx_specialisation_equals_the_reference(tmp_path):
    exe = os.path.join(HERE, "_bin", "cxx_f64_flowdirs_check")
    if not os.path.exists(exe):
        pytest.skip("tests/_bin/cxx_f64_flowdirs_check was not built (the reference headers were absent at build time)")
    for name in NAMES:
        f = FIX[name]
        h, w = f["dem"].shape
        with open(tmp_path / f"{name}.in", "wb") as fh:
            fh.write(np.array([w, h], np.int32).tobytes() + np.float64(f["nodata"]).tobytes() + f["dem"].tobytes())
    subprocess.run([exe, str(tmp_path), *NAMES], check=True, timeout=600)
    for name in NAMES:
        f = FIX[name]
        for alter in (0, 1):
            d = np.fromfile(tmp_path / f"{name}.dirs{alter}.out", np.uint8).reshape(f["dem"].shape)
            z = np.fromfile(tmp_path / f"{name}.dem{alter}.out", np.float64).reshape(f["dem"].shape)
            assert np.array_equal(d, f[f"dirs{alter}"]) and same_bits(z, f["dem1" if alter else "dem"]), (name, alter)
        for line in (tmp_path / f"{name}.launches").read_text().split("\n"):
            if line:
                assert int(line.split()[1]) > 0, (name, line)


# ---- row bands: G processes sharing the GPU over gloo ----------------------------------------------------------------
def _band_rasters():
    import oracle
    rng = np.random.default_rng(8)
    z = oracle.fbm_terrain(1024, 1024, seed=33, quantum=2.0).astype(np.float64) + rng.random((1024, 1024)) * 1e-6
    z[200:700, 400:420] = -9999.0
    big = np.asarray(f64.FillDepressions(rd.rdarray(z, no_data=-9999.0)))
    out = {n: (FIX[n]["dem"], float(FIX[n]["nodata"])) for n in ("fbm_subfloat", "above_flt_max", "nodata_1e39", "beauford_1e-9")}
    out["fbm1024"] = (big, -9999.0)
    return out


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run_bands(rank, world, device, cases):
    import torch
    from richdem_b200 import sharded
    res = {}
    for name, (dem, nd) in cases.items():
        r0, r1, gt, gb = sharded.local_rows(dem.shape[0], world, rank)
        for alter in (False, True):
            local = torch.from_numpy(np.ascontiguousarray(dem[r0 - gt:r1 + gb])).to(device)
            dirs, _ = sharded.d8_flow_directions_band(local, gt, gb, nd, alter=alter)
            torch.cuda.synchronize()
            res[(name, alter)] = (dirs.cpu().numpy()[gt:dirs.shape[0] - gb].copy(), local.cpu().numpy()[gt:local.shape[0] - gb].copy())
    return res


def _worker(rank, world, port, cases, out_q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        torch.cuda.set_device(0)
        _lib.init(0)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        out_q.put((rank, _run_bands(rank, world, "cuda:0", cases), None))
    except Exception as exc:  # surface the failure in the parent instead of a silent non-zero exit
        import traceback
        out_q.put((rank, {}, traceback.format_exc() + repr(exc)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.fixture(scope="module")
def band_cases():
    cases = _band_rasters()
    L = _lib.lib()
    want = {}
    for name, (dem, nd) in cases.items():
        h, w = dem.shape
        for alter in (0, 1):
            z = dem.copy()
            d = np.empty(z.shape, np.uint8)
            _lib.check(L.rdb200_d8_flow_directions_flats_f64(_lib.ptr(z), _lib.ptr(d), w, h, nd, alter))
            want[(name, bool(alter))] = (d, z)
    return cases, want


def _check_bands(results, want):
    for key, (d, z) in want.items():
        got_d = np.concatenate([res[key][0] for _, res, _ in results])
        got_z = np.concatenate([res[key][1] for _, res, _ in results])
        assert np.array_equal(got_d, d), (key, int((got_d != d).sum()))
        assert same_bits(got_z, z), key


def test_one_band_equals_single_gpu(band_cases):
    cases, want = band_cases
    import torch.distributed as dist  # noqa: F401
    _check_bands([(0, _run_bands(0, 1, "cuda", cases), None)], want)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_processes_over_gloo_equal_one_gpu(band_cases, world):
    cases, want = band_cases
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted((q.get(timeout=1500) for _ in range(world)), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
    _check_bands(results, want)
    assert all(p.exitcode == 0 for p in procs)


# ---- 16384^2 ---------------------------------------------------------------------------------------------------------
def test_fbm_16384_float_raster_equals_the_float32_path():
    """Every value of a widened float raster is a float, so the double template and the float template take the same
    decisions and the float steps are the float32 path's ulps: the float64 path must give the float32 path's bits."""
    import torch
    n = 16384
    L = _lib.lib()
    _lib.use_torch_stream()
    z32 = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.check(L.rdb200_dev_generate_fbm_f32(z32.data_ptr(), n, n, 0, 1234, 10, 1.0))
    _lib.check(L.rdb200_dev_fill_depressions_d8_f32(z32.data_ptr(), n, n))
    torch.cuda.synchronize()
    for alter in (0, 1):
        a32 = z32.clone()
        a64 = z32.double()
        d32 = torch.empty((n, n), dtype=torch.uint8, device="cuda")
        d64 = torch.empty((n, n), dtype=torch.uint8, device="cuda")
        _lib.check(L.rdb200_dev_d8_flow_directions_flats_f32(a32.data_ptr(), d32.data_ptr(), n, n, -9999.0, alter))
        flat_cells = int(_lib.stats()["flat_cells_raised"]) if alter else None
        _lib.check(L.rdb200_dev_d8_flow_directions_flats_f64(a64.data_ptr(), d64.data_ptr(), n, n, -9999.0, alter))
        torch.cuda.synchronize()
        assert torch.equal(d32, d64), alter
        assert torch.equal(a32.double().view(torch.int64), a64.view(torch.int64)), alter
        if alter:
            assert flat_cells > 10000
        del a32, a64, d32, d64
    del z32
    torch.cuda.empty_cache()
