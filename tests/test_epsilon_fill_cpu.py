"""FillDepressions(epsilon=True) on the CPU: the C restatement of the surface the GPU computes (oracle/epsilon_fill.c), held
to the definition and to the reference.

With up(x) = nextafterf(x, +inf), the surface W is the unique solution of W = Z on the raster's border and on NoData cells,
W(c) = max(Z(c), min over the neighbours n of up(W(n))) elsewhere (DESIGN.md section 0, f3).

* Definition: the restatement (a Dijkstra flood) equals a brute-force Jacobi iteration of the definition in numpy, from +inf,
  on NoData islands (some inside depressions, one valid cell walled in by NoData), signed zeros, negatives and subnormals,
  +-FLT_MAX and +-inf, nested lakes one ulp apart and mazes whose single path is the longest ulp ramp there is.
* Reference: the reference's PriorityFloodEpsilon_Barnes2014 (stored in tests/golden/epsilon_fill_ref.npz) is never below
  the restatement, on any cell of any fixture, D4 and NoData included.
* Drained: without NoData, and with no elevation at +-inf or +-FLT_MAX (whose ramps saturate at +inf), every non-pinned
  cell has a strictly lower neighbour, and the plain fill
  and ResolveFlats of the checker's C port leave the surface as it is.

This module also defines the fixtures (CASES), which tests/golden/make_epsilon_fill.py stores with the reference's outputs.
"""
import importlib.util
import os

import numpy as np
import pytest

import oracle
from oracle import epsilon_fill as EF

HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0
TOPOS = ("D8", "D4")
DENORM_MIN = float(np.nextafter(np.float32(0), np.float32(1)))


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


adv = _load_module("adversarial_terrain", os.path.join(HERE, "test_adversarial_terrain.py"))


# ---- fixtures ---------------------------------------------------------------------------------------------------------
def fbm_nodata(seed=1, h=48, w=61):
    """fBm with NoData islands: one in the open, one at the bottom of a pit dug into the terrain, one valid cell walled in
    by NoData, and NoData on the border."""
    dem = oracle.fbm_terrain(h, w, seed=seed, quantum=0.5)
    dem[8:12, 20:27] = ND
    dem[28:35, 38:47] -= 400.0  # a pit ...
    dem[31, 42] = ND            # ... with NoData at its bottom
    dem[18:23, 4:9] = ND
    dem[20, 6] = 3.0            # a valid cell whose every neighbour is NoData
    dem[0, 5:9] = ND
    return dem


def fbm_nan_nodata():
    """NaN as the NoData value pins nothing: the surface is the one without NoData."""
    return oracle.fbm_terrain(40, 53, seed=4, quantum=0.25)


def subnormals():
    """Basins whose floors, rims and outlets are subnormal, positive and negative, and a basin around -0.0 whose outlet
    is +denorm_min."""
    dem = adv._lowland(40, 60, 5)
    d = np.float32(DENORM_MIN)
    adv._basin(dem, 3, 3, 15, 25, float(d), float(3 * d), rim=float(64 * d))
    adv._basin(dem, 3, 32, 15, 55, float(-5 * d), float(-d), rim=float(7 * d))
    adv._basin(dem, 22, 3, 36, 25, -0.0, float(d), rim=1.0)
    adv._basin(dem, 22, 32, 36, 55, -1e-30, -0.0, rim=1.0)
    return dem


def quantised_fbm(seed=6, h=70, w=90, q=50.0):
    """Coarsely quantised fBm: wide flats and plateaus, whose cells all become ulp ramps."""
    return oracle.fbm_terrain(h, w, seed=seed, quantum=q)


# name -> (DEM, NoData); the small ones are cheap enough for the brute-force iteration
SMALL = {
    "fbm_nodata": lambda: (fbm_nodata(), ND),
    "fbm_nan_nodata": lambda: (fbm_nan_nodata(), float("nan")),
    "fbm_nodata_zero": lambda: (np.where(fbm_nodata() == ND, np.float32(0), fbm_nodata()).astype(np.float32), 0.0),
    "quantised_fbm": lambda: (quantised_fbm(), ND),
    "signed_zeros": lambda: (adv.signed_zeros(), ND),
    "subnormals": lambda: (subnormals(), ND),
    "infinities": lambda: (adv.infinities(), ND),
    "flt_max_plateaus": lambda: (adv.flt_max_plateaus(), ND),
    "flats_below_zero": lambda: (adv.flats_below_zero(), ND),
    "nested_lakes_0": lambda: (adv.nested_lakes(40, 0.0, rings=6, seed=21), ND),
    "nested_lakes_1000": lambda: (adv.nested_lakes(40, 1000.0, rings=6, seed=22), ND),
    "serpentine_small": lambda: (adv.serpentine(40, 37, 1, seed=23), ND),
    "serpentine_nodata_walls_small": lambda: (adv.serpentine(41, 36, 1, seed=24, nodata_walls=True), ND),
    "spiral_small": lambda: (adv.spiral(41, seed=25), ND),
    "staircase_small": lambda: (adv.staircase(40, seed=26), ND),
}
CASES = dict(SMALL, **{k: (lambda f=f: (f(), ND)) for k, f in adv.MAZES.items()})


def case(name):
    dem, nd = CASES[name]()
    return np.ascontiguousarray(dem, np.float32), nd


# ---- checks -----------------------------------------------------------------------------------------------------------
def offsets(topology):
    if topology == "D4":
        return ((-1, 0), (0, 1), (1, 0), (0, -1))
    return tuple((dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dy or dx)


def pinned(z, nodata):
    p = np.zeros(z.shape, bool)
    p[0, :] = p[-1, :] = p[:, 0] = p[:, -1] = True
    return p | (z == np.float32(nodata))


def neighbour_min(W, topology):
    h, w = W.shape
    P = np.full((h + 2, w + 2), np.inf, np.float32)
    P[1:-1, 1:-1] = W
    m = np.full((h, w), np.inf, np.float32)
    for dy, dx in offsets(topology):
        m = np.fmin(m, P[1 + dy:h + 1 + dy, 1 + dx:w + 1 + dx])
    return m


def brute_force(z, nodata, topology):
    """Jacobi iteration of the definition from +inf on every non-pinned cell, to its fixed point."""
    pin = pinned(z, nodata)
    W = np.where(pin, z, np.float32(np.inf)).astype(np.float32)
    inf = np.float32(np.inf)
    for _ in range(z.size + 1):
        with np.errstate(over="ignore"):  # up(FLT_MAX) = inf
            new = np.where(pin, z, np.maximum(z, np.nextafter(neighbour_min(W, topology), inf))).astype(np.float32)
        if np.array_equal(new, W):
            return W
        W = new
    raise AssertionError("the iteration did not settle")


def same_surface(a, b):
    """Equal as floats and bit for bit away from zero (the sign of a zero is free, as in the plain fill)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    if a.shape != b.shape or not np.array_equal(a, b, equal_nan=True):
        return False
    nz = ~((a == 0) & (b == 0))
    return np.array_equal(a.view(np.uint32)[nz], b.view(np.uint32)[nz])


def stored_reference(g, name, topology, z):
    """The reference's surface for fixture `name` from tests/golden/epsilon_fill_ref.npz (or the dict its maker builds),
    decoded from the form tests/golden/make_epsilon_fill.py stored it in; `z` is the input, checked against its digest."""
    assert str(g[f"{name}__dem_sha"]) == oracle.digest(z), f"{name}: fixture drifted from the stored input"
    k = f"{name}__ref_{topology}"
    if f"{k}__vs_dem" in g:
        bits = z.view(np.uint32) + g[f"{k}__vs_dem"]  # (uint32: wraps, as the subtraction that stored it)
    else:
        bits = np.cumsum(g[f"{k}__row_diff"], axis=1, dtype=np.uint32)
    return bits.view(np.float32)


def drained(W, z, nodata, topology):
    """Every non-pinned cell has a neighbour strictly below it."""
    return bool(np.all((neighbour_min(W, topology) < W) | pinned(z, nodata)))


def _drains(name):
    # no NoData, and no ramp that can climb past FLT_MAX to +inf (up(FLT_MAX) = up(inf) = inf: such cells tie)
    z, nd = case(name)
    return not np.any(z == np.float32(nd)) and bool(np.all(np.abs(z) < np.finfo(np.float32).max))


DRAINED_CASES = [n for n in CASES if _drains(n)]


@pytest.fixture(scope="module")
def eps():
    return EF.port()


@pytest.mark.parametrize("topology", TOPOS)
@pytest.mark.parametrize("name", sorted(SMALL))
def test_restatement_equals_brute_force(eps, name, topology):
    z, nd = case(name)
    W = eps.fill(z, nd, topology)
    assert same_surface(W, brute_force(z, nd, topology)), name
    assert np.all(W >= z) and np.array_equal(W[pinned(z, nd)].view(np.uint32), z[pinned(z, nd)].view(np.uint32))


def test_the_fixtures_are_what_they_say(eps):
    z, nd = case("fbm_nodata")
    W = eps.fill(z, nd, "D8")
    assert W[20, 6] == z[20, 6] and np.all(W[z == ND] == ND)  # the walled-in cell keeps its Z; NoData is never raised
    z, _ = case("fbm_nan_nodata")
    assert same_surface(eps.fill(z, float("nan"), "D8"), eps.fill(z, 1e30, "D8"))
    z, nd = case("subnormals")
    W = eps.fill(z, nd, "D8")
    sub = (W != 0) & (np.abs(W) < np.finfo(np.float32).tiny)
    assert sub.sum() > 100  # the ramps in those basins run through the subnormals
    z, nd = case("nested_lakes_1000")
    assert np.count_nonzero(eps.fill(z, nd, "D8") > z) > 500


@pytest.mark.parametrize("topology", TOPOS)
@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_is_never_below_the_restatement(eps, golden, name, topology):
    g = golden["epsilon_fill_ref"]
    z, nd = case(name)
    ref, W = stored_reference(g, name, topology, z), eps.fill(z, nd, topology)
    assert np.all(ref >= W), f"{np.count_nonzero(ref < W)} cells of the reference lie below the restatement"


def test_reference_is_close_on_nodata_free_fbm(eps, golden):
    """On NoData-free fBm the reference lies a few ulps above the restatement in under 1 % of the cells.  Wide flats
    (coarsely quantised fBm) are where its queue order shows most: there a third of the cells differ, by tens of ulps."""
    g = golden["epsilon_fill_ref"]
    for name, share, ulps in (("fbm_nan_nodata", 0.01, 16), ("quantised_fbm", 0.5, 64)):
        z, nd = case(name)
        for topology in TOPOS:
            ref, W = stored_reference(g, name, topology, z), eps.fill(z, nd, topology)
            d = ref.view(np.int32).astype(np.int64) - W.view(np.int32).astype(np.int64)  # (all values positive here)
            assert 0 <= d.min() and d.max() <= ulps and np.count_nonzero(d) < share * z.size, (name, topology)


@pytest.mark.parametrize("topology", TOPOS)
@pytest.mark.parametrize("name", DRAINED_CASES)
def test_restatement_is_drained(eps, port, name, topology):
    z, nd = case(name)
    W = eps.fill(z, nd, topology)
    assert drained(W, z, nd, topology)
    assert same_surface(port.fill_depressions(W, None if topology == "D8" else "fill_d4"), W)
    assert same_surface(port.resolve_flats(W, nd), W)


def test_float64_refuses_epsilon_before_touching_the_raster():
    """richdem_b200.f64.FillDepressions(epsilon=True) names float64 as not available; the element-type record decides it,
    before any copy or library call, so it needs no GPU."""
    import richdem_b200 as rd
    from richdem_b200 import f64
    a = rd.rdarray(np.zeros((4, 5), np.float64), no_data=ND)
    for in_place in (False, True):
        with pytest.raises(Exception, match="not available for float64"):
            f64.FillDepressions(a, epsilon=True, in_place=in_place)
    assert "PROCESSING_HISTORY" not in a.metadata
