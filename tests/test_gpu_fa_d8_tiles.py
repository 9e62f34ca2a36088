"""Unit-weight D8 accumulation by 64 x 64 tiles (csrc/accum.cu, fa_d8_tiles): rasters whose flow crosses tile seams in
every way the link pass between tiles has to handle, compared bit for bit with the CPU checker.
tests/test_fa_d8_tiles_emulated.py runs the same cases on the CPU model of the kernels."""
import numpy as np
import pytest

import oracle
import richdem_b200 as rd

ND = -9999.0
T = 64  # tile side of the engine


def R(a, nd=ND):
    return rd.rdarray(np.ascontiguousarray(a), no_data=nd)


def tile_edge_shapes():
    """At and around T and 2T, and strips of 1 to 3 rows or columns."""
    return [(1, 1), (1, 64), (2, 65), (3, 63), (64, 1), (65, 2), (63, 3), (64, 64), (65, 65), (63, 129), (128, 128),
            (127, 129), (129, 127), (3, 200), (130, 2)]


def nodata_on_tile_corners(shape=(200, 260), seed=3):
    dem = oracle.fbm_terrain(*shape, seed=seed, quantum=0.5)
    for y, x in ((T, T), (2 * T, T), (T, 3 * T), (3 * T, 2 * T)):
        if y < shape[0] and x < shape[1]:
            dem[y - 5:y + 4, x - 3:x + 6] = ND
    dem[T - 1:T + 1, 2 * T - 1:2 * T + 1] = ND  # exactly the four cells around a corner
    return dem


def tilted_plane(shape=(300, 410), seed=5):
    """Falls towards the far corner, with a little noise: every path crosses many tiles, some of them diagonally
    through tile corners."""
    yy, xx = np.mgrid[0:shape[0], 0:shape[1]].astype(np.float32)
    rng = np.random.default_rng(seed)
    return (1000.0 - 2.0 * xx - 1.5 * yy + rng.uniform(0, 0.9, shape)).astype(np.float32)


def serpentine(shape=(200, 200), seam=T, vertical=True):
    """A channel that crosses one tile seam back and forth (rows 2 apart, turning 26 cells either side of the seam)
    inside high ground that drains into it, so that one path leaves a tile and re-enters it many times."""
    h, w = shape
    dem = (500.0 + oracle.fbm_terrain(h, w, seed=11) * 0.01).astype(np.float32)
    path = []
    y, going_right = 4, True
    while y < h - 4:
        xs = range(seam - 26, seam + 26) if going_right else range(seam + 25, seam - 27, -1)
        path += [(y, x) for x in xs]
        if y + 2 < h - 4:
            x_turn = seam + 25 if going_right else seam - 26
            path.append((y + 1, x_turn))
        y += 2
        going_right = not going_right
    for i, (py, px) in enumerate(path):
        dem[py, px] = 100.0 - 0.01 * i
    return dem if vertical else np.ascontiguousarray(dem.T)


def flat_resolved_fbm(checker, shape=(260, 330), seed=7):
    dem = oracle.fbm_terrain(*shape, seed=seed, quantum=0.5)
    dem[100:130, 60:140] = ND
    return checker.resolve_flats(checker.fill_depressions(dem), ND)


def cases(checker):
    """(name, dem) pairs; every raster is small enough for the CPU model of the kernels."""
    out = []
    for shape in tile_edge_shapes():
        dem = oracle.fbm_terrain(*shape, seed=shape[0] * 131 + shape[1], quantum=0.5)
        if dem.size > 16:
            dem[shape[0] // 2, shape[1] // 2] = ND
        out.append((f"edge{shape}", dem))
    out += [("nodata_corners", nodata_on_tile_corners()), ("tilted_plane", tilted_plane()),
            ("serpentine_x", serpentine()), ("serpentine_y", serpentine(vertical=False)),
            ("all_flat", np.full((130, 140), 5.0, np.float32)), ("all_nodata", np.full((70, 130), ND, np.float32)),
            ("flat_resolved_fbm", flat_resolved_fbm(checker))]
    return out


def check(checker, dem):
    got = np.asarray(rd.FlowAccumulation(R(dem), "D8"))
    expected = checker.fa_d8(dem, ND)
    assert np.array_equal(got, expected), f"{int((got != expected).sum())} of {dem.size} cells differ"


@pytest.mark.gpu
def test_tile_seam_cases(checker):
    for name, dem in cases(checker):
        try:
            check(checker, dem)
        except AssertionError as e:
            raise AssertionError(f"{name}: {e}") from None


@pytest.mark.gpu
@pytest.mark.parametrize("maker", ["tilted_plane", "serpentine", "flat_resolved_fbm"])
def test_tile_seam_cases_large(checker, maker):
    """Paths that cross hundreds of tiles; the serpentine crosses a seam 500 times."""
    if maker == "tilted_plane":
        dem = tilted_plane((2048, 3001))
    elif maker == "serpentine":
        dem = serpentine((1003, 1500), seam=11 * T)
    else:
        dem = flat_resolved_fbm(checker, (1500, 2047), seed=9)
    check(checker, dem)


@pytest.mark.gpu
def test_device_entry_point_without_alignment(checker):
    """rdb200_dev_fa_d8_f32_f64 on a raster that starts one float into its allocation, with an odd width."""
    import torch
    from richdem_b200 import _lib
    dem = flat_resolved_fbm(checker, (515, 771), seed=13)
    d = torch.empty(dem.size + 1, dtype=torch.float32, device="cuda")
    d[1:] = torch.from_numpy(dem.ravel()).cuda()
    acc = torch.empty(dem.size + 1, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().rdb200_dev_fa_d8_f32_f64(d[1:].data_ptr(), acc[1:].data_ptr(), dem.shape[1], dem.shape[0], ND, 1))
    torch.cuda.synchronize()
    assert np.array_equal(acc[1:].cpu().numpy().reshape(dem.shape), checker.fa_d8(dem, ND))
