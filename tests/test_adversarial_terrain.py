"""Terrain where a parallel engine and a sequential priority queue part ways: mazes whose single outlet makes the spill
level (fill) and the geodesic distances (flats) travel the whole corridor across 64 x 64 tile seams and band seams,
nested lakes whose levels differ by one ulp, and special float values (signed zeros, infinities, +-FLT_MAX, flats just
below zero whose resolved values cross it).  FillDepressions D8 / D4, FlatMask, ResolveFlats, FlowDirectionsD8Resolved
(alter False / True) and FlowAccumulation D8 / Dinf are held to the checker bit for bit (elevations as uint32, so a zero
of the wrong sign fails -- except in the fill, where the sign of a zero level is documented as free: README, "Exactness"),
on the GPU and on the CPU model of the kernels; the row-band fill and flats on several bands."""
import importlib
import importlib.util
import multiprocessing as mp
import os
import sys

import numpy as np
import pytest

import oracle
from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0
WALL = 100.0
FLT_MAX = float(np.finfo(np.float32).max)
DENORM_MIN = float(np.nextafter(np.float32(0), np.float32(1)))


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_ek = _load_module("emulated_kernel_fixtures", os.path.join(HERE, "test_emulated_kernels.py"))
emu_lib, emulated = _ek.emu_lib, _ek.emulated
gp = _load_module("gpu_parity_checks", os.path.join(HERE, "test_gpu_parity.py"))
gs = _load_module("gpu_sharded_drivers", os.path.join(HERE, "test_gpu_sharded.py"))
FILL_VARIANTS = [v for v in gp.VARIANTS if v and all(k.startswith("fill_") for k in v)]
FLATS_VARIANTS = [v for v in gp.VARIANTS if v and all(k.startswith("flats_") for k in v)]


# ---- mazes ----------------------------------------------------------------------------------------------------------
def serpentine(h, w, width=1, seed=0, nodata_walls=False):
    """Corridors `width` cells wide along the rows, 1-cell walls between them, joined at alternate ends: one path.  The
    floor is random in [0, 5], the only outlet the border cell (0, 1) at 5.5, so the whole path fills to 5.5 and becomes
    one flat draining through that cell.  nodata_walls: every other wall row is NoData."""
    rng = np.random.default_rng(seed)
    dem = np.full((h, w), WALL, np.float32)
    rows = list(range(1, h - width, width + 1))
    for k, y in enumerate(rows):
        dem[y:y + width, 1:w - 1] = rng.uniform(0, 5, (width, w - 2))
        if k + 1 < len(rows):
            xs = slice(w - 1 - width, w - 1) if k % 2 == 0 else slice(1, 1 + width)
            dem[y + width, xs] = rng.uniform(0, 5, width)
            if nodata_walls and k % 2 == 1:
                dem[y + width, 1:w - 1] = np.where(dem[y + width, 1:w - 1] == WALL, ND, dem[y + width, 1:w - 1])
    dem[0, 1] = 5.5
    return dem


def spiral(n, seed=0):
    """A square spiral, 1-cell corridor and walls, from the outlet at (0, 1) inwards."""
    rng = np.random.default_rng(seed)
    dem = np.full((n, n), WALL, np.float32)
    m = (n - 1) // 2
    seen = np.zeros((m, m), bool)
    i = j = 0
    di, dj = 0, 1
    while True:
        seen[i, j] = True
        dem[1 + 2 * i, 1 + 2 * j] = rng.uniform(0, 5)
        for _ in range(2):
            ni, nj = i + di, j + dj
            if 0 <= ni < m and 0 <= nj < m and not seen[ni, nj]:
                break
            di, dj = dj, -di  # turn right
        else:
            break
        dem[1 + 2 * i + di, 1 + 2 * j + dj] = rng.uniform(0, 5)
        i, j = ni, nj
    dem[0, 1] = 5.5
    return dem


def staircase(n, seed=0):
    """A wall along the diagonal, one cell per row: the cells above it reach the outlet below it through the diagonal
    gaps under D8 and not at all under D4."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:n, 0:n]
    dem = np.where(xx > yy, rng.uniform(0, 5, (n, n)), rng.uniform(0, 3, (n, n))).astype(np.float32)
    dem[yy == xx] = WALL
    dem[0, :] = dem[-1, :] = dem[:, 0] = dem[:, -1] = WALL
    dem[n - 1, 1] = 3.5
    return dem


def nested_lakes(n, base, rings=6, seed=0):
    """Concentric square walls 3 cells apart; wall j stands one ulp above wall j - 1 and the outlet (border cell at
    `base`), so lake j fills to exactly one ulp above lake j - 1."""
    rng = np.random.default_rng(seed)
    dem = (np.float32(base) - np.float32(10) - rng.uniform(0, 5, (n, n))).astype(np.float32)
    dem[0, :] = dem[-1, :] = dem[:, 0] = dem[:, -1] = 2 * abs(base) + WALL
    v = np.float32(base)
    dem[0, n // 2] = v
    for j in range(1, rings + 1):
        v = np.nextafter(v, np.float32(np.inf))
        o = 3 * j
        if n - 1 - o <= o:
            break
        dem[o, o:n - o] = dem[n - 1 - o, o:n - o] = dem[o:n - o, o] = dem[o:n - o, n - 1 - o] = v
    return dem


# ---- special values ---------------------------------------------------------------------------------------------------
def _lowland(h, w, seed):
    """Gently sloped ground at about -2 that drains to every border."""
    return (oracle.fbm_terrain(h, w, seed=seed, quantum=0.25) * 0.001 - 2.0).astype(np.float32)


def _basin(dem, y0, x0, y1, x1, floor, outlet, rim=3.0):
    """Rows y0..y1 x columns x0..x1: a ring at `rim` with one outlet cell, the inside at `floor`."""
    dem[y0:y1 + 1, x0:x1 + 1] = rim
    dem[y0 + 1:y1, x0 + 1:x1] = floor
    dem[y0, (x0 + x1) // 2] = outlet


def signed_zeros():
    """Lakes of -0.0 with a +0.0 outlet and the reverse, lakes below zero with either zero as outlet, a +0.0 flat
    next to -1, and zeros of both signs on the border."""
    dem = _lowland(70, 90, 1)
    _basin(dem, 4, 4, 20, 30, -0.0, 0.0)
    _basin(dem, 4, 40, 20, 70, 0.0, -0.0)
    _basin(dem, 30, 4, 50, 30, -1.0, 0.0)
    _basin(dem, 30, 40, 50, 70, -1.0, -0.0)
    dem[55:66, 10:40] = 0.0   # a plateau at +0.0 ...
    dem[60, 41:60] = -1.0     # ... draining east
    dem[0, 20:30] = -0.0
    dem[-1, 60:70] = 0.0
    return dem


def infinities():
    """+inf walls and a +inf plateau inside the raster, -inf pits, +inf and -inf border cells."""
    dem = _lowland(70, 90, 2)
    inf = np.inf
    _basin(dem, 4, 4, 20, 30, -1.0, 0.5, rim=inf)   # a lake behind an infinite wall
    dem[10, 10] = -inf                              # an infinitely deep pit in it
    dem[30:45, 40:70] = inf                         # an infinite plateau, drains into the lowland
    dem[50:60, 10:20] = -inf                        # a block of -inf pits in the open
    dem[0, 30:40] = inf
    dem[-1, 30:40] = -inf
    dem[20:30, 0] = -inf
    return dem


def flt_max_plateaus():
    """A +FLT_MAX plateau (its resolved cells step to +inf), a -FLT_MAX lake and -FLT_MAX on the border."""
    dem = _lowland(70, 90, 3)
    dem[5:30, 5:40] = FLT_MAX
    _basin(dem, 35, 5, 60, 40, -FLT_MAX, 1.0)
    dem[40:50, 50:70] = -FLT_MAX
    dem[-1, 50:70] = -FLT_MAX
    return dem


def flats_below_zero():
    """Flats at -denorm_min and at -0.0, long enough that their resolved values cross zero and climb into the
    denormals; each drains through one cell at -1."""
    dem = _lowland(70, 90, 4)
    dem[5:30, 5:85] = -DENORM_MIN
    dem[17, 85] = -1.0
    dem[40:65, 5:85] = -0.0
    dem[52, 4] = -1.0
    return dem


SPECIAL = {"signed_zeros": signed_zeros, "infinities": infinities, "flt_max_plateaus": flt_max_plateaus,
           "flats_below_zero": flats_below_zero}

# CPU model: at most about 260 x 300
MAZES = {
    "serpentine_w1": lambda: serpentine(140, 131, 1, seed=1),
    "serpentine_w3": lambda: serpentine(131, 140, 3, seed=2),
    "serpentine_w1_columns": lambda: serpentine(130, 141, 1, seed=3).T.copy(),
    "serpentine_w3_columns": lambda: serpentine(129, 150, 3, seed=4).T.copy(),
    "serpentine_nodata_walls": lambda: serpentine(140, 129, 1, seed=5, nodata_walls=True),
    "spiral": lambda: spiral(131, seed=6),
    "staircase": lambda: staircase(140, seed=7),
    "nested_lakes_1000": lambda: nested_lakes(140, 1000.0, rings=20, seed=8),
    "nested_lakes_0": lambda: nested_lakes(130, 0.0, rings=20, seed=9),
}
# GPU: flat geodesic distances up to about 10^5 (a 2048^2 serpentine with 1-cell corridors, 2 x 10^6 cells of path, ran
# longer than 7 minutes through this check with its ten fill / flats variants, and is left out)
GPU_MAZES = dict(MAZES, **{
    "serpentine_w1_512": lambda: serpentine(512, 512, 1, seed=11),
    "serpentine_w3_511": lambda: serpentine(511, 509, 3, seed=12),
    "serpentine_w1_columns_400": lambda: serpentine(400, 403, 1, seed=13).T.copy(),
    "spiral_513": lambda: spiral(513, seed=14),
    "staircase_2048": lambda: staircase(2048, seed=15),
    "nested_lakes_1024": lambda: nested_lakes(1024, 1.0, rings=150, seed=16),
})


def bits(a):
    return np.asarray(a).view(np.uint32)


def same_fill(got, expected, any_zero_sign=False):
    """Bit for bit; any_zero_sign: a zero may carry either sign (README, "Exactness"), every other bit must match."""
    got, expected = np.asarray(got), np.asarray(expected)
    if not any_zero_sign:
        return np.array_equal(bits(got), bits(expected))
    zeros = (got == 0) & (expected == 0)
    return np.array_equal(got, expected) and np.array_equal(bits(got)[~zeros], bits(expected)[~zeros])


def check_terrain(dem, O, variants=False, any_zero_sign=False):
    import richdem_b200 as rd
    R = gp.R
    f_ref = O.fill_depressions(dem)
    assert same_fill(rd.FillDepressions(R(dem)), f_ref, any_zero_sign), "fill D8"
    f4 = O.fill_depressions(dem, "fill_d4")
    assert same_fill(rd.FillDepressions(R(dem), topology="D4"), f4, any_zero_sign), "fill D4"
    m, l = rd.FlatMask(R(f_ref))
    m_ref, l_ref = O.flat_mask(f_ref, ND)
    assert np.array_equal(l != 0, l_ref != 0), "flat labels (membership)"
    assert np.array_equal(m, m_ref), f"flat mask: {(m != m_ref).sum()} cells differ"
    pairs = np.unique(np.stack([l[l != 0], l_ref[l_ref != 0]]), axis=1)
    assert len(np.unique(pairs[0])) == pairs.shape[1] == len(np.unique(pairs[1]))
    r_ref = O.resolve_flats(f_ref, ND)
    assert np.array_equal(bits(rd.ResolveFlats(R(f_ref))), bits(r_ref)), "resolve_flats"
    assert np.array_equal(np.asarray(rd.FlowDirectionsD8Resolved(R(f_ref.copy()))), O.d8_flow_directions_flats(f_ref, ND)[0])
    d = R(f_ref.copy())
    dirs_alt = np.asarray(rd.FlowDirectionsD8Resolved(d, alter=True))
    assert np.array_equal(bits(d), bits(r_ref)), "alter=True elevations"
    assert np.array_equal(dirs_alt, O.d8_flow_directions(r_ref, ND))
    assert np.array_equal(np.asarray(rd.FlowAccumulation(R(r_ref), "D8")), O.fa_d8(r_ref, ND))
    np.testing.assert_allclose(np.asarray(rd.FlowAccumulation(R(r_ref), "Dinf")), O.fa_dinf(r_ref, ND),
                               rtol=gp.DINF_UNIT_RTOL, atol=0)
    if not variants:
        return
    on_cpu_model = hasattr(_lib.lib(), "rdb200_emulated")
    try:
        for cfg in FILL_VARIANTS + FLATS_VARIANTS:
            _lib.reset_params()
            if on_cpu_model:
                _lib.set_param("fill_use_tma", 0)  # TMA / mbarrier PTX is not emulated
            for k, v in cfg.items():
                _lib.set_param(k, v)
            if any(k.startswith("fill_") for k in cfg):
                assert same_fill(rd.FillDepressions(R(dem)), f_ref, any_zero_sign), cfg
                assert same_fill(rd.FillDepressions(R(dem), topology="D4"), f4, any_zero_sign), cfg
            else:
                assert np.array_equal(bits(rd.ResolveFlats(R(f_ref))), bits(r_ref)), cfg
    finally:
        _lib.reset_params()


# ---- the cases are what they say ----------------------------------------------------------------------------------------
def test_mazes_have_one_long_path(checker):
    """The single outlet floods the whole corridor, which becomes one flat."""
    for name in ("serpentine_w1", "serpentine_w3_columns", "spiral"):
        dem = MAZES[name]()
        f = checker.fill_depressions(dem)
        corridor = dem != WALL
        assert (f[corridor] == np.float32(5.5)).all(), name
        m, l = checker.flat_mask(f, ND)
        assert len(np.unique(l[corridor])) == 1 and l[corridor][0] != 0, name
        assert m.max() > corridor.sum() // 2, name  # the geodesic distance runs along the path
    s = MAZES["staircase"]()
    assert (checker.fill_depressions(s, "fill_d4")[5, 100] == WALL) and checker.fill_depressions(s)[5, 100] < 6


def test_nested_lakes_are_one_ulp_apart(checker):
    dem = nested_lakes(140, 1000.0, rings=20)
    f = checker.fill_depressions(dem)
    levels = np.unique(f[1:-1, 1:-1])
    steps = np.diff(levels.view(np.int32))
    assert len(levels) >= 20 and (steps == 1).all()


def test_special_values_are_there(checker):
    r = checker.resolve_flats(checker.fill_depressions(flats_below_zero()), ND)
    assert (r[5:30, 5:85] > 0).all() and (r[40:65, 5:85] > 0).any()  # both flats resolve to values above zero
    r = checker.resolve_flats(checker.fill_depressions(flt_max_plateaus()), ND)
    assert np.isposinf(r[5:30, 5:40]).any()
    z = checker.fill_depressions(signed_zeros())
    assert np.signbit(z[5:20, 5:30]).all() != np.signbit(z[5:20, 41:70]).all()


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GPU_MAZES))
def test_maze(checker, name):
    check_terrain(GPU_MAZES[name](), checker, variants=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SPECIAL))
def test_special_values(checker, name):
    check_terrain(SPECIAL[name](), checker, variants=True, any_zero_sign=name == "signed_zeros")


BAND_MAZES = {"serpentine_w1": lambda n: serpentine(n + 40, n + 1, 1, seed=21),
              "serpentine_w3_columns": lambda n: serpentine(130, n + 40, 3, seed=22).T.copy(),
              "spiral": lambda n: spiral(61, seed=23)}  # (the band drivers of the tests allow 100 flag merges: 15 rings)


def _check_bands(checker, dem, Gs):
    f_ref = checker.fill_depressions(dem)
    r_ref = checker.resolve_flats(f_ref, ND)
    for G in Gs:
        got, rounds = gs.emulate_bands(dem, G)
        assert np.array_equal(bits(got), bits(f_ref)), f"fill G={G} after {rounds} exchanges"
        got, it1, it2 = gs.emulate_flats_bands(f_ref, G, ND)
        assert np.array_equal(bits(got), bits(r_ref)), (G, it1, it2)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BAND_MAZES))
def test_maze_bands(checker, name):
    _check_bands(checker, BAND_MAZES[name](520), (2, 3, 4))


# ---- CPU model of the kernels ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(MAZES))
def test_maze_emulated(emulated, checker, name):
    check_terrain(MAZES[name](), checker)


@pytest.mark.parametrize("name", sorted(SPECIAL))
def test_special_values_emulated(emulated, checker, name):
    check_terrain(SPECIAL[name](), checker, variants=True, any_zero_sign=name == "signed_zeros")


def test_fill_zero_sign_is_the_only_freedom(checker):
    """The signed-zero lakes do take both signs in the reference (so any_zero_sign relaxes something real), and a value
    other than a zero that differs in one bit still fails."""
    z = checker.fill_depressions(signed_zeros())
    flipped = z.copy()
    flipped[z == 0] = -flipped[z == 0]
    assert not np.array_equal(bits(flipped), bits(z)) and same_fill(flipped, z, True)
    bumped = z.copy()
    bumped[60, 20] = np.nextafter(bumped[60, 20], np.float32(1))
    assert not same_fill(bumped, z, True)


def test_maze_variants_emulated(emulated, checker):
    check_terrain(serpentine(130, 133, 1, seed=31), checker, variants=True)


@pytest.fixture()
def host_band_drivers(emulated, monkeypatch):
    import ctypes as C
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
    monkeypatch.setattr(gs, "DEV", "cpu")
    return gs


@pytest.mark.parametrize("name", sorted(BAND_MAZES))
def test_maze_bands_emulated(host_band_drivers, checker, name):
    _check_bands(checker, BAND_MAZES[name](130), (2, 3, 4))


@pytest.mark.parametrize("world", [2, 3, 4])
def test_maze_over_gloo_emulated(world):
    """The C++ band drivers (fill, flats, D8 and Dinf accumulation), one process per band, on a serpentine whose
    corridors cross every seam."""
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    gloo = importlib.import_module("test_sharded_emulated_gloo")  # its worker is pickled by module name
    lib_path = str(_load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build())
    O = oracle.best()
    dem = serpentine(121, 96, 1, seed=41)
    expected = {"fill": O.fill_depressions(dem)}
    expected["flats"] = O.resolve_flats(expected["fill"], ND)
    expected["fa_d8"] = O.fa_d8(expected["flats"], ND)
    expected["fa_dinf"] = O.fa_dinf(expected["flats"], ND)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = gloo._free_port()
    procs = [ctx.Process(target=gloo._worker, args=(r, world, port, lib_path, dem, expected, {}, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in results:
        assert err is None, f"rank {rank}: {err}"
        assert res == {"fill": True, "flats": True, "fa_d8": True, "fa_dinf": True}, (rank, res)
    assert all(p.exitcode == 0 for p in procs)
