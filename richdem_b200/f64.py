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
from . import (_F64, _fill_depressions, _flat_mask, _flow_accumulation, _flow_directions_d8, _flow_directions_d8_resolved,
               _flow_proportions, _has_depressions, _pit_mask, _resolve_flats, _terrain_attribute, rd3array, rdarray)



def FillDepressions(dem: rdarray, epsilon: bool = False, in_place: bool = False,
                    topology: str = "D8") -> Optional[rdarray]:
    """FillDepressions<topo, double> (PriorityFlood_Zhou2016 for ``D8``, PriorityFlood_Barnes2014<D4> for ``D4``).
    Returns the filled DEM unless ``in_place``; cells the fill does not raise keep their own bits.  ``epsilon=True`` is
    not available for float64 rasters and raises."""
    return _fill_depressions(_F64, dem, epsilon, in_place, topology)

def PitMask(dem: rdarray, topology: str = "D8") -> rdarray:
    """pit_mask<topo> of a float64 raster: uint8, 1 below the filled surface, 3 NoData, 0 elsewhere (``no_data`` 3)."""
    return _pit_mask(_F64, dem, topology)


def HasDepressions(dem: rdarray, topology: str = "D8") -> bool:
    """HasDepressions<topo> of a float64 raster: whether ``FillDepressions`` would raise any cell."""
    return _has_depressions(_F64, dem, topology)


def ResolveFlats(dem: rdarray, in_place: bool = False) -> Optional[rdarray]:
    """ResolveFlatsEpsilon<double>: the Barnes (2014) increment mask, applied as double ulps."""
    return _resolve_flats(_F64, dem, in_place)


def FlowAccumulation(dem: rdarray, method: Optional[str] = None, exponent: Optional[float] = None,
                     weights: Optional[rdarray] = None, in_place: bool = False) -> rdarray:
    """FA_D8<double, double> (``D8`` / ``OCallaghanD8``) and FA_D4<double, double> (``D4`` / ``OCallaghanD4``).  The
    other methods are refused here.  Float64 D-infinity, Quinn, Holmgren and Freeman accumulation is available through
    ``richdem_b200.FlowAccumFromProps(f64.FlowProportions(dem, method, exponent))``, through the C ABI
    (``rdb200_fa_{tarboton,quinn,holmgren,freeman}_f64_f64``) and through the C++ specialisations of
    ``include/richdem_b200.hpp`` under ``RICHDEM_B200_F64`` (and so the reference's own Python package built on them)."""
    return _flow_accumulation(_F64, dem, method, exponent, weights, in_place)


def FlowDirectionsD8(dem: rdarray) -> rdarray:
    """d8_flow_directions<double, uint8_t>: uint8 codes 0..8, 255 NoData."""
    return _flow_directions_d8(_F64, dem)


def FlowDirectionsD8Resolved(dem: rdarray, alter: bool = False) -> rdarray:
    """barnes_flat_resolution_d8<double, uint8_t>: D8 directions in which drainable flats flow along the Barnes (2014)
    increment mask.  ``alter=True`` raises the flat cells of ``dem`` in place instead, as the reference does for a
    double raster: m float-ulp steps (``nextafterf``) from the value rounded to float32, then the directions again."""
    return _flow_directions_d8_resolved(_F64, dem, alter)


def FlatMask(dem: rdarray):
    """GetFlatMask<double>: (mask, labels) int32 arrays; labels are equal within one flat, their values arbitrary."""
    return _flat_mask(_F64, dem)


def FlowProportions(dem: rdarray, method: Optional[str] = None, exponent: Optional[float] = None) -> rd3array:
    """FM_x<double> (reference FlowProportions, :650-732): (H, W, 9) float32 proportions of a float64 raster, laid out
    as :func:`richdem_b200.FlowProportions` lays them out."""
    return _flow_proportions(_F64, dem, method, exponent)


def TerrainAttribute(dem: rdarray, attrib: str, zscale: float = 1.0) -> rdarray:
    """TA_x<double> (reference TerrainAttribute, :735-794) of a float64 raster: float32 result with no_data -9999, cell
    lengths from the geotransform (1 x 1 when there is none), as :func:`richdem_b200.TerrainAttribute`."""
    return _terrain_attribute(_F64, dem, attrib, zscale)


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
