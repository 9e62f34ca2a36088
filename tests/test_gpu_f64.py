"""float64 elevations on the H100 against the reference with T = double: the fixtures of tests/golden/f64_ref.npz
(tests/golden/make_f64.py) through the Python API and the device entry points, bit for bit apart from the fill's zero
sign (weighted accumulation within 1e-9 relative); a 4096^2 float64 fBm in both key cases; the keys at 4100^2 (a rank
scan over several steps); one FillDepressions at 32768^2; the C++ specialisations switched on by RICHDEM_B200_F64
(tests/cxx_f64_check.cpp); and the unmodified reference richdem/__init__.py over the pyrichdem module built with them."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
import richdem_b200 as rd
from oracle import f64 as F
from richdem_b200 import _lib
from richdem_b200 import f64

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "f64_ref.npz"))
NAMES = sorted({k.split("__")[0] for k in G.files if k.endswith("__dem")})
TOPOS = ("D8", "D4")


def same_bits(a, b, zero_sign=False):
    a, b = np.asarray(a, np.float64).copy(), np.asarray(b, np.float64).copy()
    if a.shape != b.shape:
        return False
    if zero_sign:
        a[a == 0] = 0.0
        b[b == 0] = 0.0
    return bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def case(name):
    return np.ascontiguousarray(G[f"{name}__dem"]), float(G[f"{name}__nodata"])


@pytest.mark.parametrize("name", NAMES)
def test_python_api_equals_reference(name):
    z, nd = case(name)
    before = z.copy()
    a = lambda: rd.rdarray(z.copy(), no_data=nd)
    for topo in TOPOS:
        assert same_bits(f64.FillDepressions(a(), topology=topo), G[f"{name}__fill_{topo}"], zero_sign=True), topo
        filled = a()
        assert f64.FillDepressions(filled, topology=topo, in_place=True) is None
        assert same_bits(filled, G[f"{name}__fill_{topo}"], zero_sign=True), topo
        m = f64.PitMask(a(), topology=topo)
        assert m.dtype == np.uint8 and m.no_data == 3 and np.array_equal(m, G[f"{name}__mask_{topo}"]), topo
        assert f64.HasDepressions(a(), topology=topo) is bool(G[f"{name}__has_{topo}"]), topo
        method = "D8" if topo == "D8" else "OCallaghanD4"
        assert same_bits(f64.FlowAccumulation(a(), method=method), G[f"{name}__fa_{topo}"]), topo
        wts = rd.rdarray(G[f"{name}__weights"], no_data=-1)
        got = f64.FlowAccumulation(a(), method=method, weights=wts)
        assert np.allclose(got, G[f"{name}__fa_{topo}_w"], rtol=1e-9, atol=0), topo
    assert same_bits(f64.ResolveFlats(a()), G[f"{name}__resolved"])
    d = f64.FlowDirectionsD8(a())
    assert d.no_data == 255 and np.array_equal(d, G[f"{name}__dirs"])
    assert same_bits(z, before)


@pytest.mark.parametrize("name", NAMES)
def test_device_entry_points(name):
    import torch
    z, nd = case(name)
    L = _lib.lib()
    h, w = z.shape
    t = lambda: torch.from_numpy(z.copy()).cuda()
    out = C.c_int32(0)
    for topo, k in (("D8", "d8"), ("D4", "d4")):
        d = t()
        torch.cuda.synchronize()
        _lib.check(getattr(L, f"rdb200_dev_fill_depressions_{k}_f64")(d.data_ptr(), w, h))
        assert same_bits(d.cpu().numpy(), G[f"{name}__fill_{topo}"], zero_sign=True), topo
        d = t()
        m = torch.empty((h, w), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        _lib.check(getattr(L, f"rdb200_dev_pit_mask_{k}_f64")(d.data_ptr(), m.data_ptr(), w, h, nd))
        assert np.array_equal(m.cpu().numpy(), G[f"{name}__mask_{topo}"]), topo
        _lib.check(getattr(L, f"rdb200_dev_has_depressions_{k}_f64")(d.data_ptr(), w, h, C.byref(out)))
        assert bool(out.value) is bool(G[f"{name}__has_{topo}"]), topo
        assert same_bits(d.cpu().numpy(), z), topo  # not modified
        acc = torch.empty((h, w), dtype=torch.float64, device="cuda")
        if topo == "D8":
            _lib.check(L.rdb200_dev_fa_d8_f64_f64(d.data_ptr(), acc.data_ptr(), w, h, nd, 1))
        else:
            acc.fill_(1.0)
            torch.cuda.synchronize()
            _lib.check(L.rdb200_dev_fa_d4_f64_f64(d.data_ptr(), acc.data_ptr(), w, h, nd))
        assert same_bits(acc.cpu().numpy(), G[f"{name}__fa_{topo}"]), topo
    d = t()
    torch.cuda.synchronize()
    _lib.check(L.rdb200_dev_resolve_flats_epsilon_f64(d.data_ptr(), w, h, nd))
    assert same_bits(d.cpu().numpy(), G[f"{name}__resolved"])
    d = t()
    dirs = torch.empty((h, w), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    _lib.check(L.rdb200_dev_d8_flow_directions_f64(d.data_ptr(), dirs.data_ptr(), w, h, nd))
    assert np.array_equal(dirs.cpu().numpy(), G[f"{name}__dirs"])


@pytest.mark.parametrize("name", NAMES)
def test_keys_equal_the_spec(name):
    z, nd = case(name)
    k, ndk, ranked = f64.OrderKeys(z, nd)
    ks, ndks, rs = F.kappa(z, nd)
    assert ranked == rs and np.array_equal(k.view(np.uint32), ks.view(np.uint32))
    assert (np.isnan(ndk) and np.isnan(ndks)) or ndk.view(np.uint32) == ndks.view(np.uint32)


@pytest.fixture(scope="module", params=["float_raster", "ranked"])
def fbm4096(request):
    z = oracle.device_fbm(4096, 4096, seed=7, quantum=0.0).astype(np.float64)
    if request.param == "ranked":
        z = z + np.random.default_rng(3).integers(0, 8, z.shape) * 2.0 ** -36
    z[100:140, 200:260] = -9999.0
    return request.param, z


def test_4096_fbm(fbm4096):
    """Both key cases at 4096^2: the keys equal the spec, and every call equals kappa^-1 of the float path on the keys
    (the float path is bit-exact against the reference on its own); where the reference shim was built, also the
    reference with T = double itself."""
    kind, z = fbm4096
    nd = -9999.0
    k, ndk, ranked = f64.OrderKeys(z, nd)
    ks, ndks, _ = F.kappa(z, nd)
    assert ranked == (kind == "ranked") and np.array_equal(k.view(np.uint32), ks.view(np.uint32)) and ndk == ndks
    R = F.ref() if F.have_ref() else None
    a = lambda arr, nodata: rd.rdarray(arr.copy(), no_data=nodata)
    for topo in TOPOS:
        got = f64.FillDepressions(a(z, nd), topology=topo)
        kf = rd.FillDepressions(a(k, ndk), topology=topo)
        assert same_bits(got, F.kappa_inv_fill(z, k, kf), zero_sign=True), topo
        assert np.array_equal(f64.PitMask(a(z, nd), topology=topo), rd.PitMask(a(k, ndk), topology=topo)), topo
        assert f64.HasDepressions(a(z, nd), topology=topo) == rd.HasDepressions(a(k, ndk), topology=topo), topo
        if R is not None:
            assert same_bits(got, R.fill(z, topo), zero_sign=True), topo
    m, _ = rd.FlatMask(a(k, ndk))
    resolved = f64.ResolveFlats(a(z, nd))
    assert same_bits(resolved, F.apply_flat_mask(z, m))
    assert same_bits(f64.FlowAccumulation(a(z, nd), method="D8"), rd.FlowAccumulation(a(k, ndk), method="D8"))
    assert same_bits(f64.FlowAccumulation(a(z, nd), method="D4"), rd.FlowAccumulation(a(k, ndk), method="D4"))
    assert np.array_equal(f64.FlowDirectionsD8(a(z, nd)), rd.FlowDirectionsD8(a(k, ndk)))


def test_fill_32768_on_one_gpu():
    """One float64 FillDepressions at 32768^2 (8 GiB of doubles) on the device, through the rank keys."""
    import torch
    n = 32768
    zf = torch.empty((n, n), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().rdb200_dev_generate_fbm_f32(zf.data_ptr(), n, n, 0, 42, 12, 0))
    z = zf.double()
    del zf
    z[::7, ::5] += 2.0 ** -30  # sub-float detail: the rank case
    torch.cuda.synchronize()
    before = z[::97, ::89].clone()
    _lib.check(_lib.lib().rdb200_dev_fill_depressions_d8_f64(z.data_ptr(), n, n))
    torch.cuda.synchronize()
    assert bool((z[::97, ::89] >= before).all())
    del z
    _lib.set_param("trim_workspace", 1)
    torch.cuda.empty_cache()


def test_keys_across_several_scan_steps():
    """4100^2 cells: more than 4096 chunks of 4096 run heads, so the rank scan carries across steps of its chunk-sum
    pass; the keys still equal the spec in both routes."""
    n = 4100
    rng = np.random.default_rng(17)
    z = (rng.random((n, n)) * 1000.0).astype(np.float32).astype(np.float64)
    z[rng.random((n, n)) < 0.01] = -9999.0
    for ranked_wanted, zz in ((False, z), (True, z + rng.integers(0, 3, z.shape) * 2.0 ** -40)):
        k, ndk, ranked = f64.OrderKeys(zz, -9999.0)
        ks, ndks, rs = F.kappa(zz, -9999.0)
        assert ranked == rs == ranked_wanted
        assert np.array_equal(k.view(np.uint32), ks.view(np.uint32)) and ndk.view(np.uint32) == ndks.view(np.uint32)


# ---- the C++ drop-in with RICHDEM_B200_F64, and the reference's own Python package built with it ----------------------
def test_cxx_specialisations(tmp_path):
    """tests/cxx_f64_check.cpp calls the reference's template names on Array2D<double> with the macro on; every output
    equals the fixtures, and the library's launch count shows each call ran on the GPU."""
    import subprocess
    exe = os.path.join(HERE, "_bin", "cxx_f64_check")
    if not os.path.exists(exe):
        pytest.skip("tests/_bin/cxx_f64_check was not built (the reference headers were absent at build time)")
    for name in NAMES:
        z, nd = case(name)
        h, w = z.shape
        with open(tmp_path / f"{name}.in", "wb") as f:
            f.write(np.array([w, h], np.int32).tobytes() + np.array([nd], np.float64).tobytes() + z.tobytes())
    r = subprocess.run([exe, str(tmp_path), *NAMES], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    for name in NAMES:
        z, nd = case(name)
        h, w = z.shape
        out = lambda fn, dt: np.fromfile(tmp_path / f"{name}.{fn}.out", dt).reshape(h, w)
        for topo in TOPOS:
            assert same_bits(out(f"fill_{topo}", np.float64), G[f"{name}__fill_{topo}"], zero_sign=True), (name, topo)
            assert np.array_equal(out(f"mask_{topo}", np.uint8), G[f"{name}__mask_{topo}"]), (name, topo)
            has = np.fromfile(tmp_path / f"{name}.has_{topo}.out", np.int32)[0]
            assert bool(has) is bool(G[f"{name}__has_{topo}"]), (name, topo)
            assert same_bits(out(f"fa_{topo}", np.float64), G[f"{name}__fa_{topo}"]), (name, topo)
        assert same_bits(out("zhou", np.float64), G[f"{name}__fill_D8"], zero_sign=True), name
        assert same_bits(out("barnes_D4", np.float64), G[f"{name}__fill_D4"], zero_sign=True), name
        assert same_bits(out("resolved", np.float64), G[f"{name}__resolved"]), name
        assert np.array_equal(out("dirs", np.uint8), G[f"{name}__dirs"]), name
        for line in (tmp_path / f"{name}.launches").read_text().split("\n"):
            if not line:
                continue
            fn, k = line.split()
            if fn.startswith("HasDepressions") and (h < 3 or w < 3):
                continue  # every cell is an edge cell: the call answers without a kernel
            assert int(k) > 0, (name, fn)


_PYRICHDEM_F64_SCRIPT = r"""
import os, sys
import numpy as np
pkg, root, src, dst = sys.argv[1:5]
sys.path.insert(0, pkg)
import richdem
assert os.path.dirname(richdem.__file__).startswith(pkg)
richdem._RichDEMVersion = lambda: "RichDEM (reference Python layer over librichdem_b200)"
sys.path.insert(0, root)
from richdem_b200 import _lib
assert "librichdem_b200.so" in open("/proc/self/maps").read()
g = np.load(src)
names = sorted({k.split("__")[0] for k in g.files if k.endswith("__dem")})
out = {}
def launches():
    return _lib.stats()["kernel_launches"]
for name in names:
    z, nd = np.ascontiguousarray(g[name + "__dem"]), float(g[name + "__nodata"])
    for topo in ("D8", "D4"):
        out[name + "__fill_" + topo] = np.asarray(richdem.FillDepressions(richdem.rdarray(z.copy(), no_data=nd), topology=topo))
        out[name + "__fill_" + topo + "_launches"] = launches()
        out[name + "__fa_" + topo] = np.asarray(richdem.FlowAccumulation(richdem.rdarray(z.copy(), no_data=nd), method=topo))
        out[name + "__fa_" + topo + "_launches"] = launches()
    out[name + "__resolved"] = np.asarray(richdem.ResolveFlats(richdem.rdarray(z.copy(), no_data=nd)))
    out[name + "__resolved_launches"] = launches()
np.savez(dst, **out)
"""


def test_reference_python_package_on_float64(tmp_path):
    """The unmodified reference richdem/__init__.py over tests/_bin/pyrichdem_f64 (the reference binding source compiled
    with RICHDEM_B200_F64), in a subprocess of its own: FillDepressions (D8, D4), ResolveFlats and FlowAccumulation (D8,
    D4) on float64 rdarrays run on the GPU and equal the fixtures."""
    import subprocess
    import sys
    pkg = os.path.join(HERE, "_bin", "pyrichdem_f64")
    if not os.path.exists(os.path.join(pkg, "richdem", "__init__.pyc")) or not any(
            f.startswith("_richdem") for f in os.listdir(pkg)):
        pytest.skip("tests/_bin/pyrichdem_f64 not built (reference tree absent at build time)")
    script, dst = tmp_path / "run.py", tmp_path / "out.npz"
    script.write_text(_PYRICHDEM_F64_SCRIPT)
    r = subprocess.run([sys.executable, str(script), pkg, os.path.dirname(HERE), os.path.join(HERE, "golden", "f64_ref.npz"),
                        str(dst)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.load(dst)
    R = F.ref() if F.have_ref() else None
    for name in NAMES:
        z, nd = case(name)
        # the reference's Array2D.setNoData binding tries its float overload first (pywrapper.hpp:134-135), so its own
        # package hands a float64 raster the NoData value rounded through float: the expected outputs are the
        # reference's with that value
        with np.errstate(over="ignore"):  # DBL_MAX becomes inf, as in the binding
            nd_seen = float(np.float32(nd))
        exact = same_bits(nd_seen, nd)
        for topo in TOPOS:
            assert same_bits(got[f"{name}__fill_{topo}"], G[f"{name}__fill_{topo}"], zero_sign=True), (name, topo)
            assert int(got[f"{name}__fill_{topo}_launches"]) > 0 and int(got[f"{name}__fa_{topo}_launches"]) > 0, (name, topo)
            if exact or R is not None:
                want = G[f"{name}__fa_{topo}"] if exact else R.fa(z, nd_seen, topo)
                assert same_bits(got[f"{name}__fa_{topo}"], want), (name, topo)
        if exact or R is not None:
            want = G[f"{name}__resolved"] if exact else R.resolve_flats(z, nd_seen)
            assert same_bits(got[f"{name}__resolved"], want), name
        assert int(got[f"{name}__resolved_launches"]) > 0, name
