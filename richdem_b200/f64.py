"""float64 elevations on the GPU: ``FillDepressions``, ``PitMask``, ``HasDepressions``, ``ResolveFlats``,
``FlowAccumulation`` (D8 / OCallaghanD8 / D4 / OCallaghanD4), ``FlowDirectionsD8``, ``FlowDirectionsD8Resolved``,
``FlatMask``, ``FlowProportions`` and ``TerrainAttribute`` for C-contiguous float64 ``rdarray``s, with the arguments,
checks and messages of the float32 functions in :mod:`richdem_b200`.

Each call gives what the reference's ``double`` templates give (the fill's zero sign aside, as for float32), within the
float32 path's tolerances.  The stages that only compare elevations run the float engines on an order-preserving float
key of every value, so two levels one double ulp apart stay apart (DESIGN §0.1).  ``FlowProportions`` and
``TerrainAttribute`` do arithmetic on the elevations and run double instantiations of the float kernels (DESIGN §0.2).
Casting to float32 first gives neither answer.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _lib
from . import (_D4_METHODS, _D8_METHODS, _DINF_METHODS, _EXPONENT_METHODS, _OUT_OF_SCOPE_METHODS, _accum_array,
               _add_analysis, _terrain_attrib_id, rd3array, rdarray)


def _dem_f64(dem: rdarray, what: str) -> np.ndarray:
    if dem.ndim != 2:
        raise RuntimeError("Array must have two dimensions!")  # pywrapper.hpp:118-119
    if dem.dtype != np.float64:
        raise Exception(
            f"{what}: richdem_b200.f64 is built for float64 elevations (got '{dem.dtype}'); "
            "float32 rasters go through richdem_b200 itself.")
    if not dem.flags["C_CONTIGUOUS"]:
        raise Exception(f"{what}: the raster must be C-contiguous")
    return dem


def _nodata_f64(dem) -> float:
    nd = dem.no_data
    if nd is None:
        print("Warning! no_data was None. Setting it to -9999!")  # reference :204-206
        nd = -9999
    return float(nd)


def _check_topology(dem, topology: str) -> None:
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if topology not in ["D8", "D4"]:
        raise Exception("Unknown topology!")


def FillDepressions(dem: rdarray, epsilon: bool = False, in_place: bool = False,
                    topology: str = "D8") -> Optional[rdarray]:
    """FillDepressions<topo, double> (PriorityFlood_Zhou2016 for ``D8``, PriorityFlood_Barnes2014<D4> for ``D4``).
    Returns the filled DEM unless ``in_place``; cells the fill does not raise keep their own bits."""
    _check_topology(dem, topology)
    if epsilon:
        raise Exception("FillDepressions(epsilon=True) is outside the GPU hot path (SURVEY 8f-3)")
    if not in_place:
        dem = dem.copy()
    _add_analysis(dem, f"FillDepressions(dem, epsilon={epsilon})")
    d = _dem_f64(dem, "FillDepressions")
    h, w = d.shape
    L = _lib.lib()
    fn = L.rdb200_fill_depressions_d8_f64 if topology == "D8" else L.rdb200_fill_depressions_d4_f64
    _lib.check(fn(_lib.ptr(d), w, h))
    if not in_place:
        return dem
    return None


def PitMask(dem: rdarray, topology: str = "D8") -> rdarray:
    """pit_mask<topo> of a float64 raster: uint8, 1 below the filled surface, 3 NoData, 0 elsewhere (``no_data`` 3)."""
    _check_topology(dem, topology)
    d = _dem_f64(dem, "PitMask")
    h, w = d.shape
    out = rdarray(np.empty((h, w), np.uint8), meta_obj=dem, no_data=3)
    _add_analysis(out, f"PitMask(dem, topology={topology})")
    L = _lib.lib()
    fn = L.rdb200_pit_mask_d8_f64 if topology == "D8" else L.rdb200_pit_mask_d4_f64
    _lib.check(fn(_lib.ptr(d), _lib.ptr(out), w, h, _nodata_f64(dem)))
    out.no_data = 3
    return out


def HasDepressions(dem: rdarray, topology: str = "D8") -> bool:
    """HasDepressions<topo> of a float64 raster: whether ``FillDepressions`` would raise any cell."""
    _check_topology(dem, topology)
    d = _dem_f64(dem, "HasDepressions")
    h, w = d.shape
    out = C.c_int32(0)
    L = _lib.lib()
    fn = L.rdb200_has_depressions_d8_f64 if topology == "D8" else L.rdb200_has_depressions_d4_f64
    _lib.check(fn(_lib.ptr(d), w, h, C.byref(out)))
    return bool(out.value)


def ResolveFlats(dem: rdarray, in_place: bool = False) -> Optional[rdarray]:
    """ResolveFlatsEpsilon<double>: the Barnes (2014) increment mask, applied as double ulps."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if not in_place:
        dem = dem.copy()
    _add_analysis(dem, f"ResolveFlats(dem, in_place={in_place})")
    d = _dem_f64(dem, "ResolveFlats")
    h, w = d.shape
    _lib.check(_lib.lib().rdb200_resolve_flats_epsilon_f64(_lib.ptr(d), w, h, _nodata_f64(dem)))
    if not in_place:
        return dem
    return None


def FlowAccumulation(dem: rdarray, method: Optional[str] = None, exponent: Optional[float] = None,
                     weights: Optional[rdarray] = None, in_place: bool = False) -> rdarray:
    """FA_D8<double, double> (``D8`` / ``OCallaghanD8``) and FA_D4<double, double> (``D4`` / ``OCallaghanD4``).  The
    other methods are refused here.  Float64 D-infinity, Quinn, Holmgren and Freeman accumulation is available through
    ``richdem_b200.FlowAccumFromProps(f64.FlowProportions(dem, method, exponent))``, through the C ABI
    (``rdb200_fa_{tarboton,quinn,holmgren,freeman}_f64_f64``) and through the C++ specialisations of
    ``include/richdem_b200.hpp`` under ``RICHDEM_B200_F64`` (and so the reference's own Python package built on them)."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    accum, ones = _accum_array(dem, weights, in_place, dem.shape)
    _add_analysis(accum, "FlowAccumulation(dem, method={0}, exponent={1}, weights={2}, in_place={3})".format(
        method, exponent, "None" if weights is None else "weights", in_place))
    d = _dem_f64(dem, "FlowAccumulation")
    h, w = d.shape
    L = _lib.lib()
    nd = _nodata_f64(dem)
    if method in _D8_METHODS:
        _lib.check(L.rdb200_fa_d8_f64_f64(_lib.ptr(d), _lib.ptr(accum), w, h, nd, int(ones)))
    elif method in _D4_METHODS:
        if ones:
            accum[...] = 1.0
        _lib.check(L.rdb200_fa_d4_f64_f64(_lib.ptr(d), _lib.ptr(accum), w, h, nd))
    elif method in _DINF_METHODS + ("Quinn",) + _EXPONENT_METHODS + _OUT_OF_SCOPE_METHODS:
        raise Exception(f'FlowAccumulation method "{method}" is not available for float64 rasters '
                        "(it does arithmetic on elevation differences); valid methods here are: " +
                        ", ".join(_D8_METHODS + _D4_METHODS))
    else:
        raise Exception("Invalid FlowAccumulation method. Valid methods are: " + ", ".join(_D8_METHODS + _D4_METHODS))
    accum.no_data = -1
    return accum


def FlowDirectionsD8(dem: rdarray) -> rdarray:
    """d8_flow_directions<double, uint8_t>: uint8 codes 0..8, 255 NoData."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    d = _dem_f64(dem, "FlowDirectionsD8")
    h, w = d.shape
    out = rdarray(np.empty((h, w), np.uint8), meta_obj=dem, no_data=255)
    _lib.check(_lib.lib().rdb200_d8_flow_directions_f64(_lib.ptr(d), _lib.ptr(out), w, h, _nodata_f64(dem)))
    out.no_data = 255
    return out


def FlowDirectionsD8Resolved(dem: rdarray, alter: bool = False) -> rdarray:
    """barnes_flat_resolution_d8<double, uint8_t>: D8 directions in which drainable flats flow along the Barnes (2014)
    increment mask.  ``alter=True`` raises the flat cells of ``dem`` in place instead, as the reference does for a
    double raster: m float-ulp steps (``nextafterf``) from the value rounded to float32, then the directions again."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    d = _dem_f64(dem, "FlowDirectionsD8Resolved")
    h, w = d.shape
    out = rdarray(np.empty((h, w), np.uint8), meta_obj=dem, no_data=255)
    _lib.check(_lib.lib().rdb200_d8_flow_directions_flats_f64(_lib.ptr(d), _lib.ptr(out), w, h, _nodata_f64(dem),
                                                               int(bool(alter))))
    out.no_data = 255
    return out


def FlatMask(dem: rdarray):
    """GetFlatMask<double>: (mask, labels) int32 arrays; labels are equal within one flat, their values arbitrary."""
    d = _dem_f64(dem, "FlatMask")
    h, w = d.shape
    mask = np.empty((h, w), np.int32)
    labels = np.empty((h, w), np.int32)
    _lib.check(_lib.lib().rdb200_get_flat_mask_f64(_lib.ptr(d), _lib.ptr(mask), _lib.ptr(labels), w, h, _nodata_f64(dem)))
    return mask, labels


def FlowProportions(dem: rdarray, method: Optional[str] = None, exponent: Optional[float] = None) -> rd3array:
    """FM_x<double> (reference FlowProportions, :650-732): (H, W, 9) float32 proportions of a float64 raster, laid out
    as :func:`richdem_b200.FlowProportions` lays them out."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    fprops = rd3array(np.empty(shape=dem.shape + (9,), dtype="float32"), meta_obj=dem, no_data=-2)
    _add_analysis(fprops, f"FlowProportions(dem, method={method}, exponent={exponent})")
    d = _dem_f64(dem, "FlowProportions")
    h, w = d.shape
    L = _lib.lib()
    nd = _nodata_f64(dem)
    if method in _D8_METHODS:
        _lib.check(L.rdb200_fm_d8_f64(_lib.ptr(d), _lib.ptr(fprops), w, h, nd))
    elif method in _DINF_METHODS:
        _lib.check(L.rdb200_fm_tarboton_f64(_lib.ptr(d), _lib.ptr(fprops), w, h, nd))
    elif method in _D4_METHODS:
        _lib.check(L.rdb200_fm_d4_f64(_lib.ptr(d), _lib.ptr(fprops), w, h, nd))
    elif method == "Quinn":
        _lib.check(L.rdb200_fm_quinn_f64(_lib.ptr(d), _lib.ptr(fprops), w, h, nd))
    elif method in _EXPONENT_METHODS:
        if exponent is None:
            raise Exception('FlowProportions method "' + method + '" requires an exponent!')
        fn = L.rdb200_fm_freeman_f64 if method == "Freeman" else L.rdb200_fm_holmgren_f64
        _lib.check(fn(_lib.ptr(d), _lib.ptr(fprops), w, h, nd, float(exponent)))
    elif method in _OUT_OF_SCOPE_METHODS:
        raise Exception(f'FlowProportions method "{method}" is outside the GPU hot path '
                        "(random-walk metric; use the reference CPU implementation)")
    else:
        raise Exception("Invalid FlowProportions method. Valid methods are: " +
                        ", ".join(_DINF_METHODS + ("Quinn",) + _D8_METHODS + _D4_METHODS + _EXPONENT_METHODS +
                                  _OUT_OF_SCOPE_METHODS))
    fprops.no_data = -2
    return fprops


def TerrainAttribute(dem: rdarray, attrib: str, zscale: float = 1.0) -> rdarray:
    """TA_x<double> (reference TerrainAttribute, :735-794) of a float64 raster: float32 result with no_data -9999, cell
    lengths from the geotransform (1 x 1 when there is none), as :func:`richdem_b200.TerrainAttribute`."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    attrib_id = _terrain_attrib_id(attrib)
    d = _dem_f64(dem, "TerrainAttribute")
    h, w = d.shape
    gt = dem.geotransform
    if gt is None:
        print("Warning! No geotransform defined. Choosing a standard one! (Top left cell's top let corner at <0,0>; cells are 1x1.)")
        gt = [0, 1, 0, 0, 0, -1]
    result = rdarray(np.zeros((h, w), np.float32), meta_obj=dem, no_data=-9999)
    _add_analysis(result, f"TerrainAttribute(dem, attrib={attrib}, zscale={zscale})")
    _lib.check(_lib.lib().rdb200_terrain_attribute_f64(attrib_id, _lib.ptr(d), _lib.ptr(result), w, h, _nodata_f64(dem),
                                                        -9999.0, float(zscale), abs(float(gt[1])), abs(float(gt[5]))))
    return result


def OrderKeys(dem: np.ndarray, no_data: float = -9999.0):
    """Diagnostic: the float keys the calls above run the float engines on, ``(keys, nodata_key, ranked)`` with
    ``ranked`` False when every value was a float already (the keys are the cast), True for dense ranks.  The encoding
    is an implementation detail and may change between versions; it is exposed so that tests can check it."""
    d = np.ascontiguousarray(dem, dtype=np.float64)
    if d.ndim != 2:
        raise RuntimeError("Array must have two dimensions!")
    h, w = d.shape
    keys = np.empty((h, w), np.float32)
    ndk, ranked = C.c_float(0), C.c_int32(0)
    _lib.check(_lib.lib().rdb200_f64_order_keys(_lib.ptr(d), _lib.ptr(keys), w, h, float(no_data), C.byref(ndk),
                                                C.byref(ranked)))
    return keys, np.float32(ndk.value), bool(ranked.value)
