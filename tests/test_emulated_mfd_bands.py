"""Row-band FA_D4 / FA_Quinn / FA_Holmgren / FA_Freeman WITHOUT a GPU: the G-bands-on-one-device drivers of
test_gpu_sharded_mfd.py on host memory, against the CPU model of the shipped kernels (tests/emu; see
test_emulated_kernels.py for what that model can and cannot check)."""
import ctypes as C
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_ek = _load_module("emulated_kernel_fixtures", os.path.join(HERE, "test_emulated_kernels.py"))
emu_lib, emulated = _ek.emu_lib, _ek.emulated  # the emulation library, swapped in for one test at a time


@pytest.fixture()
def mfd_drivers(emulated, monkeypatch):
    import torch
    from richdem_b200 import sharded

    def host_view(ptr, shape, typestr, device):
        dt = np.dtype(typestr)
        n = int(np.prod(shape))
        buf = (C.c_char * (n * dt.itemsize)).from_address(int(ptr))
        return torch.from_numpy(np.frombuffer(buf, dtype=dt, count=n).reshape(shape))

    monkeypatch.setattr(sharded, "_on_device", lambda t: True)  # "device" memory is host memory here
    monkeypatch.setattr(sharded, "_view", host_view)
    monkeypatch.setattr(_lib, "use_torch_stream", lambda: None)
    gs = _load_module("gpu_sharded_mfd_drivers", os.path.join(HERE, "test_gpu_sharded_mfd.py"))
    gs.DEV = "cpu"
    return gs


def _resolved(checker, shape, seed, q=0.5):
    return checker.resolve_flats(checker.fill_depressions(oracle.fbm_terrain(*shape, seed=seed, quantum=q)), ND)


@pytest.mark.parametrize("G", [1, 2, 3, 5])
@pytest.mark.parametrize("method,exponent", [("D4", None), ("Quinn", None), ("Holmgren", 2.5), ("Holmgren", 0.7),
                                             ("Freeman", 1.1), ("Freeman", 4.0)])
def test_band_mfd_accumulation(mfd_drivers, checker, G, method, exponent):
    dem = oracle.fbm_terrain(150, 124, seed=41, quantum=0.25)
    dem[40:110, 50:70] = ND  # across the seams of every G
    dem = checker.resolve_flats(checker.fill_depressions(dem), ND)
    mfd_drivers.check_bands(checker, dem, G, method, exponent)
    mfd_drivers.check_bands(checker, dem, G, method, exponent, np.random.default_rng(G).random(dem.shape))


@pytest.mark.parametrize("method,exponent", [("Quinn", None), ("Holmgren", 2.5), ("Freeman", 1.1), ("D4", None)])
def test_band_mfd_channel_crossing_seams(mfd_drivers, checker, method, exponent):
    dem = mfd_drivers.serpentine_channel(40, 40)
    rounds = mfd_drivers.check_bands(checker, dem, 3, method, exponent)
    if method != "D4":
        assert rounds > 2, rounds


@pytest.mark.parametrize("method,exponent", [("Quinn", None), ("Freeman", 4.0), ("D4", None)])
def test_band_mfd_one_owned_row_and_nodata_ghosts(mfd_drivers, checker, method, exponent):
    for shape, G in (((6, 40), 6), ((2, 9), 2), ((5, 17), 3)):
        mfd_drivers.check_bands(checker, _resolved(checker, shape, shape[1]), G, method, exponent)
    dem = _resolved(checker, (40, 60), 7)
    dem[20, 5:25] = ND
    dem[19, 30:50] = ND
    dem[19, 15:18] = ND
    for G in (2, 4):
        mfd_drivers.check_bands(checker, dem, G, method, exponent, np.random.default_rng(G).random(dem.shape))


def test_band_mfd_with_several_blocks():
    """The band walk is one cooperative launch of accum_levels_kernel<2, true>: re-run the cases above with 3 emulated
    SMs (3 blocks side by side, a real grid barrier) and atomics that yield at random."""
    if os.environ.get("RDB_EMU_SMS"):
        pytest.skip("already inside the multi-block run")
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    env = dict(os.environ, RDB_EMU_SMS="3", RDB_EMU_CHAOS="11")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", os.path.abspath(__file__), "-k",
                        "channel or one_owned_row or (band_mfd_accumulation and (Quinn or Freeman-4.0))"],
                       env=env, cwd=os.path.dirname(HERE), capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
