"""FillDepressions(epsilon=True) on the H100 (fill_sweep_kernel<2>): bit for bit the C restatement of its surface
(oracle/epsilon_fill.c), the sign of a zero aside, and never above the reference's PriorityFloodEpsilon_Barnes2014 (stored
in tests/golden/epsilon_fill_ref.npz).

* Layouts and shapes: widths that are a multiple of 4 (the surface relaxes in the caller's raster, TMA loads) and widths
  that are not (padded copy), quantised fBm with wide flats, the Beauford crop with its NoData, a 4096^2 fBm, tall and
  wide rasters, and every fixture of tests/test_epsilon_fill_cpu.py.
* Entry points: the host and device entries give the same bits; a plain fill before and after an epsilon call is the
  same; Python in_place true and false; richdem_b200.f64 refuses epsilon=True.
* Drop-ins: the C++ specialisations behind RICHDEM_B200_EPSILON (tests/cxx_epsilon_fill_check.cpp) and the reference's
  own Python package over the pyrichdem module built with them give the C ABI's bits, on the GPU.
* Other stages on the result (NoData-free rasters): HasDepressions is false, ResolveFlats is the identity and
  FlowDirectionsD8 has no interior cell without a direction.
"""
import ctypes as C
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
import richdem_b200 as rd
from oracle import epsilon_fill as EF
from richdem_b200 import _lib
from richdem_b200 import f64

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0
TOPOS = ("D8", "D4")
G = np.load(os.path.join(HERE, "golden", "epsilon_fill_ref.npz"))


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


T = _load_module("epsilon_fill_cpu", os.path.join(HERE, "test_epsilon_fill_cpu.py"))
same_surface = T.same_surface


def R(a, nd=ND):
    return rd.rdarray(np.ascontiguousarray(a), no_data=nd)


def eps(z, nd, topology):
    return np.asarray(rd.FillDepressions(R(z, nd), epsilon=True, topology=topology))


def want(z, nd, topology):
    return EF.port().fill(z, nd, topology)


SHAPES = [(300, 420), (300, 421), (257, 130), (64, 64), (65, 63), (129, 127), (1, 1), (3, 7), (2, 9), (5, 4)]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{h}x{w}" for h, w in SHAPES])
@pytest.mark.parametrize("topology", TOPOS)
def test_shapes(shape, topology):
    h, w = shape
    z = oracle.fbm_terrain(h, w, seed=h + 7 * w, quantum=0.25)
    if h > 4 and w > 4:
        z[h // 3:h // 3 + 3, w // 3:w // 3 + 3] -= 300.0
    assert same_surface(eps(z, ND, topology), want(z, ND, topology))


@pytest.mark.parametrize("w", [640, 643])
@pytest.mark.parametrize("topology", TOPOS)
def test_quantised_fbm_with_wide_flats(w, topology):
    z = oracle.fbm_terrain(512, w, seed=5, quantum=40.0)
    assert same_surface(eps(z, ND, topology), want(z, ND, topology))


@pytest.mark.parametrize("topology", TOPOS)
def test_beauford_crop(golden, topology):
    g = golden["beauford_crop"]
    z, nd = g["dem"], float(g["nodata"])
    got = eps(z, nd, topology)
    assert same_surface(got, want(z, nd, topology))
    assert np.all(T.stored_reference(G, "beauford", topology, np.ascontiguousarray(z, np.float32)) >= got)
    assert np.array_equal(got[z == nd], z[z == nd])


@pytest.mark.parametrize("topology", TOPOS)
@pytest.mark.parametrize("name", sorted(T.CASES))
def test_fixtures_and_reference(name, topology):
    z, nd = T.case(name)
    got = eps(z, nd, topology)
    assert same_surface(got, want(z, nd, topology))
    assert np.all(T.stored_reference(G, name, topology, z) >= got)


@pytest.mark.parametrize("topology", TOPOS)
def test_4096_fbm(topology):
    z = oracle.device_fbm(4096, 4096, seed=7)
    got = eps(z, ND, topology)
    st = _lib.stats()
    assert st["fill_rounds"] > 0 and st["fill_tile_visits"] > 0
    assert same_surface(got, want(z, ND, topology))


@pytest.mark.parametrize("shape", [(70001, 3), (3, 70001), (20000, 37), (33, 20011)], ids=str)
def test_tall_and_wide(shape):
    z = oracle.fbm_terrain(*shape, seed=11, quantum=0.5)
    for topology in TOPOS:
        assert same_surface(eps(z, ND, topology), want(z, ND, topology)), topology


def test_host_and_device_entries_and_plain_fill_around():
    import torch
    L = _lib.lib()
    z = oracle.fbm_terrain(517, 644, seed=9, quantum=0.5)
    z[100:130, 200:260] = ND
    h, w = z.shape
    plain = np.asarray(rd.FillDepressions(R(z)))
    for topology in TOPOS:
        host = eps(z, ND, topology)
        for width in (w, w - 1):  # in place and padded on the device too
            zz = np.ascontiguousarray(z[:, :width])
            d = torch.from_numpy(zz.copy()).cuda()
            torch.cuda.synchronize()
            _lib.check(getattr(L, f"rdb200_dev_fill_depressions_epsilon_{topology.lower()}_f32")(d.data_ptr(), width, h, ND))
            ref = host if width == w else eps(zz, ND, topology)
            assert np.array_equal(d.cpu().numpy().view(np.uint32), ref.view(np.uint32)), (topology, width)
    assert np.array_equal(np.asarray(rd.FillDepressions(R(z))).view(np.uint32), plain.view(np.uint32))


def test_python_in_place_and_float64_refusal():
    z = oracle.fbm_terrain(200, 300, seed=12, quantum=0.5)
    a = R(z.copy())
    out = rd.FillDepressions(a, epsilon=True, in_place=False)
    assert np.array_equal(np.asarray(a), z) and "epsilon=True" in out.metadata["PROCESSING_HISTORY"]
    assert rd.FillDepressions(a, epsilon=True, in_place=True, topology="D8") is None
    assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(out).view(np.uint32))
    with pytest.raises(Exception, match="float64"):
        f64.FillDepressions(R(z.astype(np.float64)), epsilon=True)


@pytest.mark.parametrize("topology", TOPOS)
def test_other_stages_on_the_result(topology):
    z = oracle.fbm_terrain(400, 500, seed=13, quantum=2.0)
    W = R(eps(z, ND, topology))
    assert not rd.HasDepressions(W, topology=topology)
    assert np.array_equal(np.asarray(rd.ResolveFlats(W)).view(np.uint32), np.asarray(W).view(np.uint32))
    dirs = np.asarray(rd.FlowDirectionsD8(W))
    assert not np.any(dirs[1:-1, 1:-1] == 0)
    assert np.array_equal(np.asarray(rd.FillDepressions(W, topology=topology)).view(np.uint32), np.asarray(W).view(np.uint32))


CXX_NAMES = ["fbm_nodata", "quantised_fbm", "signed_zeros", "spiral"]


def test_cxx_specialisations(tmp_path):
    exe = os.path.join(HERE, "_bin", "cxx_epsilon_fill_check")
    if not os.path.exists(exe):
        pytest.skip("tests/_bin/cxx_epsilon_fill_check was not built (the reference headers were absent at build time)")
    for name in CXX_NAMES:
        z, nd = T.case(name)
        h, w = z.shape
        with open(tmp_path / f"{name}.in", "wb") as f:
            f.write(np.array([w, h], np.int32).tobytes() + np.array([nd], np.float32).tobytes() + z.tobytes())
    r = subprocess.run([exe, str(tmp_path), *CXX_NAMES], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    for name in CXX_NAMES:
        z, nd = T.case(name)
        h, w = z.shape
        for topology in TOPOS:
            abi = eps(z, nd, topology)
            for fn in ("PriorityFloodEpsilon", "FillDepressionsEpsilon"):
                got = np.fromfile(tmp_path / f"{name}.{fn}_{topology}.out", np.float32).reshape(h, w)
                assert np.array_equal(got.view(np.uint32), abi.view(np.uint32)), (name, fn, topology)
        for line in (tmp_path / f"{name}.launches").read_text().split("\n"):
            if line:
                assert int(line.split()[1]) > 0, (name, line)


_PYRICHDEM_SCRIPT = r"""
import os, sys
import numpy as np
pkg, root, dst = sys.argv[1:4]
sys.path.insert(0, pkg)
import richdem
assert os.path.dirname(richdem.__file__).startswith(pkg)
richdem._RichDEMVersion = lambda: "RichDEM (reference Python layer over librichdem_b200)"
sys.path.insert(0, root)
import oracle
from richdem_b200 import _lib
assert "librichdem_b200.so" in open("/proc/self/maps").read()
z = oracle.fbm_terrain(300, 421, seed=17, quantum=0.5)
z[50:80, 100:160] = -9999.0
out = {}
for topo in ("D8", "D4"):
    out[topo] = np.asarray(richdem.FillDepressions(richdem.rdarray(z.copy(), no_data=-9999.0), epsilon=True, topology=topo))
    out[topo + "_launches"] = _lib.stats()["kernel_launches"]
np.savez(dst, **out)
"""


def test_reference_python_package(tmp_path):
    """The unmodified reference richdem/__init__.py over tests/_bin/pyrichdem_epsilon, in a subprocess of its own."""
    pkg = os.path.join(HERE, "_bin", "pyrichdem_epsilon")
    if not os.path.exists(os.path.join(pkg, "richdem", "__init__.pyc")) or not any(
            f.startswith("_richdem") for f in os.listdir(pkg)):
        pytest.skip("tests/_bin/pyrichdem_epsilon not built (reference tree absent at build time)")
    script, dst = tmp_path / "run.py", tmp_path / "out.npz"
    script.write_text(_PYRICHDEM_SCRIPT)
    r = subprocess.run([sys.executable, str(script), pkg, os.path.dirname(HERE), str(dst)], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.load(dst)
    z = oracle.fbm_terrain(300, 421, seed=17, quantum=0.5)
    z[50:80, 100:160] = ND
    for topology in TOPOS:
        assert int(got[topology + "_launches"]) > 0, topology
        assert np.array_equal(got[topology].view(np.uint32), eps(z, ND, topology).view(np.uint32)), topology
