"""PitMask / HasDepressions on the H100 against the reference fixtures (tests/golden/depression_masks_ref.npz, written by
the unmodified pit_mask<topo> / HasDepressions<topo>): every mask bit for bit, every answer -- those the strict-pit pass
gives and those that need the fill -- for D8 and D4, through the Python API, the host and device C entry points and the
C++ drop-in specialisations (tests/cxx_depressions_check.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle
import richdem_b200 as rd
from richdem_b200 import _lib

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "depression_masks_ref.npz"))
NAMES = sorted({k.split("__")[0] for k in G.files if k.endswith("__dem")})
LARGE = sorted({k.split("__")[0] for k in G.files if k.endswith("__recipe")})
TOPOS = ("D8", "D4")


@pytest.mark.parametrize("topology", TOPOS)
@pytest.mark.parametrize("name", NAMES)
def test_python_api_equals_reference(name, topology):
    dem, nd = np.ascontiguousarray(G[f"{name}__dem"]), float(G[f"{name}__nodata"])
    before = dem.copy()
    src = rd.rdarray(dem, no_data=nd, geotransform=[1, 2, 0, 3, 0, -2])
    m = rd.PitMask(src, topology=topology)
    assert type(m) is rd.rdarray and m.dtype == np.uint8 and m.no_data == 3 and m.geotransform == [1, 2, 0, 3, 0, -2]
    assert np.array_equal(np.asarray(m), G[f"{name}__mask_{topology}"])
    assert rd.HasDepressions(src, topology=topology) is bool(G[f"{name}__has_{topology}"])
    assert np.array_equal(dem.view(np.uint32), before.view(np.uint32))


@pytest.mark.parametrize("topology", TOPOS)
@pytest.mark.parametrize("name", LARGE)
def test_large_rasters_equal_reference_digests(name, topology):
    h, w, seed, q = G[f"{name}__recipe"]
    dem = oracle.fbm_terrain(int(h), int(w), seed=int(seed), quantum=float(q))
    m = rd.PitMask(rd.rdarray(dem, no_data=-9999.0), topology=topology)
    assert oracle.digest(np.asarray(m)) == str(G[f"{name}__mask_{topology}_digest"])
    assert rd.HasDepressions(rd.rdarray(dem, no_data=-9999.0), topology=topology) is bool(G[f"{name}__has_{topology}"])


@pytest.mark.parametrize("topology", TOPOS)
def test_device_entry_points(topology):
    import torch
    L = _lib.lib()
    for name in ("beauford", "fbm_q05", "nodata_hole", "no_depressions", "terraced"):
        dem, nd = G[f"{name}__dem"], float(G[f"{name}__nodata"])
        t = torch.from_numpy(np.ascontiguousarray(dem)).cuda()
        m = torch.full(dem.shape, 7, dtype=torch.uint8, device="cuda")
        _lib.use_torch_stream()
        fn = L.rdb200_dev_pit_mask_d8_f32 if topology == "D8" else L.rdb200_dev_pit_mask_d4_f32
        _lib.check(fn(t.data_ptr(), m.data_ptr(), dem.shape[1], dem.shape[0], nd))
        assert np.array_equal(m.cpu().numpy(), G[f"{name}__mask_{topology}"]), name
        out = C.c_int32(-1)
        fn = L.rdb200_dev_has_depressions_d8_f32 if topology == "D8" else L.rdb200_dev_has_depressions_d4_f32
        _lib.check(fn(t.data_ptr(), dem.shape[1], dem.shape[0], C.byref(out)))
        assert out.value == int(bool(G[f"{name}__has_{topology}"])), name
        assert np.array_equal(t.cpu().numpy().view(np.uint32), dem.view(np.uint32)), name
    _lib.set_stream(None)


def test_strict_pit_pass_answers_alone():
    dem = np.ascontiguousarray(G["fbm_q05__dem"])
    for topo in TOPOS:
        assert rd.HasDepressions(rd.rdarray(dem, no_data=-9999.0), topology=topo)
        assert _lib.stats()["kernel_launches"] == 1
        assert rd.HasDepressions(rd.rdarray(np.ascontiguousarray(G["nodata_hole__dem"]), no_data=-9999.0), topology=topo)
        assert _lib.stats()["kernel_launches"] > 2


def test_null_pointers_and_bad_sizes_raise():
    L = _lib.lib()
    out = C.c_int32(0)
    assert L.rdb200_has_depressions_d8_f32(None, 4, 4, C.byref(out)) != 0
    assert L.rdb200_pit_mask_d4_f32(None, None, 4, 4, 0.0) != 0
    d = np.zeros((4, 4), np.float32)
    assert L.rdb200_has_depressions_d4_f32(d.ctypes.data, 0, 4, C.byref(out)) != 0


def test_cxx_dropin_specialisations():
    exe = os.path.join(HERE, "_bin", "cxx_depressions_check")
    if not os.path.exists(exe):
        pytest.skip("tests/_bin/cxx_depressions_check was not built (the reference headers were absent at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "thrown=0" in r.stdout and "mismatches=0" in r.stdout, r.stdout
