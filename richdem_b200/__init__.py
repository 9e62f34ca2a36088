"""richdem_b200 -- H100-native drop-in for RichDEM's fill -> flats -> flow-accumulation path.

The public surface mirrors the part of the reference Python API that lies on that path
(reference: wrappers/pyrichdem/richdem/__init__.py): ``rdarray`` / ``rd3array`` (:155, :226),
``FillDepressions`` (:381), ``ResolveFlats`` (:461), ``FlowAccumulation`` (:490),
``FlowAccumFromProps`` (:599) and ``FlowProportions`` (:650) -- same names, argument meaning,
return conventions and error behaviour (bare ``Exception`` for argument validation,
``RuntimeError`` for engine failures).  Everything is computed by hand-written CUDA kernels in
``librichdem_b200.so`` reached through its C ABI (``include/richdem_b200.h``); there is no CPU
fallback and methods outside the hot path raise.
"""
from __future__ import annotations

import copy
import ctypes as C
import datetime
from typing import Any, Optional

import numpy as np

from . import _lib
from ._lib import RichdemB200Error, init, set_param, shutdown, stats  # noqa: F401

__version__ = "0.1.0"

_D8_METHODS = ("D8", "OCallaghanD8")
_DINF_METHODS = ("Dinf", "Tarboton")
_D4_METHODS = ("D4", "OCallaghanD4")
_EXPONENT_METHODS = ("Freeman", "Holmgren")
# random-walk metrics (Rho8/Rho4 draw from the reference's global RNG; not reproducible on a GPU) stay on the CPU
_OUT_OF_SCOPE_METHODS = ("FairfieldLeymarieD8", "FairfieldLeymarieD4", "Rho8", "Rho4")


def _version_string() -> str:
    return f"richdem_b200 {__version__} (librichdem_b200 {_lib.lib().rdb200_version()})"


def _add_analysis(rda, analysis: str) -> None:
    # PROCESSING_HISTORY provenance, as the reference's _AddAnalysis (:34-48)
    if type(rda) not in (rdarray, rd3array):
        raise Exception("An rdarray or rd3array is required!")
    stamp = datetime.datetime.now(datetime.timezone.utc).strftime("%Y-%m-%d %H:%M:%S.%f UTC")
    if rda.metadata is None:
        rda.metadata = dict()
    rda.metadata["PROCESSING_HISTORY"] = rda.metadata.get("PROCESSING_HISTORY", "") + \
        f"\n{stamp} | {_version_string()} | {analysis}"


class _MetaArray(np.ndarray):
    def __array_finalize__(self, obj):
        if obj is None:
            return
        self.metadata = copy.deepcopy(getattr(obj, "metadata", dict()))
        self.no_data = copy.deepcopy(getattr(obj, "no_data", None))
        self.projection = copy.deepcopy(getattr(obj, "projection", ""))
        self.geotransform = copy.deepcopy(getattr(obj, "geotransform", None))

    def _take_meta(self, meta_obj, no_data, geotransform=None):
        if meta_obj is not None:
            self.metadata = copy.deepcopy(getattr(meta_obj, "metadata", dict()))
            self.no_data = copy.deepcopy(getattr(meta_obj, "no_data", None))
            self.projection = copy.deepcopy(getattr(meta_obj, "projection", ""))
            self.geotransform = copy.deepcopy(getattr(meta_obj, "geotransform", None))
        elif geotransform is not None:
            self.geotransform = geotransform
        if no_data is not None:
            self.no_data = no_data
        if no_data is None:
            raise Exception("A no_data value must be specified!")


class rdarray(_MetaArray):
    """2-D raster with ``no_data`` / ``geotransform`` / ``projection`` / ``metadata``
    (reference rdarray, :155-223)."""

    def __new__(cls, array, meta_obj=None, no_data=None, dtype=None, order=None, geotransform=None,
                copy: bool = False, **kwargs: Any):
        arr = np.array(array, dtype=dtype, order=order, copy=True) if copy else \
            np.asarray(array, dtype=dtype, order=order)
        obj = arr.view(cls)
        obj.metadata = dict()
        obj.projection = ""
        obj.geotransform = None
        obj.no_data = None
        obj._take_meta(meta_obj, no_data, geotransform)
        return obj


class rd3array(_MetaArray):
    """(H, W, 9) float32 flow-proportion array (reference rd3array, :226-279)."""

    def __new__(cls, array, meta_obj=None, no_data=None, order=None, **kwargs: Any):
        obj = np.asarray(array, dtype=np.float32, order=order).view(cls)
        obj.metadata = dict()
        obj.projection = ""
        obj.geotransform = None
        obj.no_data = None
        obj._take_meta(meta_obj, no_data)
        return obj


# ---------------------------------------------------------------------------------------------
def _dem_f32(dem: rdarray, what: str) -> np.ndarray:
    if dem.ndim != 2:
        raise RuntimeError("Array must have two dimensions!")  # pywrapper.hpp:118-119
    if dem.dtype != np.float32:
        raise Exception(
            f"{what}: the H100 path is built for float32 elevations (got '{dem.dtype}'); "
            "convert with dem.astype('float32') -- there is no CPU fallback for other dtypes "
            "(float64 rasters: richdem_b200.f64 computes the float64 answer).")
    if not dem.flags["C_CONTIGUOUS"]:
        raise Exception(f"{what}: the raster must be C-contiguous")
    return dem


def _nodata_f32(dem) -> float:
    nd = dem.no_data
    if nd is None:
        print("Warning! no_data was None. Setting it to -9999!")  # reference :204-206
        nd = -9999
    return float(np.float32(nd))


def FillDepressions(dem: rdarray, epsilon: bool = False, in_place: bool = False,
                    topology: str = "D8") -> Optional[rdarray]:
    """Fills all depressions in a DEM (reference FillDepressions, :381-422 -> PriorityFlood_Zhou2016 for ``D8``,
    PriorityFlood_Barnes2014<D4> for ``D4``).  Returns the filled DEM unless ``in_place``."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if topology not in ["D8", "D4"]:
        raise Exception("Unknown topology!")
    if epsilon:
        raise Exception("FillDepressions(epsilon=True) is outside the GPU hot path (SURVEY 8f-3)")
    if not in_place:
        dem = dem.copy()
    _add_analysis(dem, f"FillDepressions(dem, epsilon={epsilon})")
    d = _dem_f32(dem, "FillDepressions")
    h, w = d.shape
    fn = _lib.lib().rdb200_fill_depressions_d8_f32 if topology == "D8" else _lib.lib().rdb200_fill_depressions_d4_f32
    _lib.check(fn(_lib.ptr(d), w, h))
    if not in_place:
        return dem
    return None


def PitMask(dem: rdarray, topology: str = "D8") -> rdarray:
    """richdem::pit_mask<topo> (depressions/Barnes2014.hpp:593-676; app rd_depressions_mask): uint8 mask of the cells
    that lie in a depression, i.e. below the ``FillDepressions`` surface of ``dem`` (1), NoData cells (3) and all others
    (0), with ``no_data`` 3 and the input's metadata.  ``dem`` is not modified."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if topology not in ["D8", "D4"]:
        raise Exception("Unknown topology!")
    d = _dem_f32(dem, "PitMask")
    h, w = d.shape
    out = rdarray(np.empty((h, w), np.uint8), meta_obj=dem, no_data=3)
    _add_analysis(out, f"PitMask(dem, topology={topology})")
    fn = _lib.lib().rdb200_pit_mask_d8_f32 if topology == "D8" else _lib.lib().rdb200_pit_mask_d4_f32
    _lib.check(fn(_lib.ptr(d), _lib.ptr(out), w, h, _nodata_f32(dem)))
    out.no_data = 3
    return out


def HasDepressions(dem: rdarray, topology: str = "D8") -> bool:
    """richdem::HasDepressions<topo> (depressions/Barnes2014.hpp:43-104; app rd_depressions_has): whether
    ``FillDepressions`` would raise any cell.  NoData is not special, as in the reference."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if topology not in ["D8", "D4"]:
        raise Exception("Unknown topology!")
    d = _dem_f32(dem, "HasDepressions")
    h, w = d.shape
    out = C.c_int32(0)
    fn = _lib.lib().rdb200_has_depressions_d8_f32 if topology == "D8" else _lib.lib().rdb200_has_depressions_d4_f32
    _lib.check(fn(_lib.ptr(d), w, h, C.byref(out)))
    return bool(out.value)


def ResolveFlats(dem: rdarray, in_place: bool = False) -> Optional[rdarray]:
    """Imposes a local gradient on drainable flats (reference ResolveFlats, :461-487 ->
    ResolveFlatsEpsilon)."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if not in_place:
        dem = dem.copy()
    _add_analysis(dem, f"ResolveFlats(dem, in_place={in_place})")
    d = _dem_f32(dem, "ResolveFlats")
    h, w = d.shape
    _lib.check(_lib.lib().rdb200_resolve_flats_epsilon_f32(_lib.ptr(d), w, h, _nodata_f32(dem)))
    if not in_place:
        return dem
    return None


def _accum_array(like, weights, in_place, shape):
    ones = False
    if weights is not None and in_place:
        accum = rdarray(weights, no_data=-1)
    elif weights is not None and not in_place:
        accum = rdarray(weights, copy=True, meta_obj=like, no_data=-1)
    else:
        accum = rdarray(np.empty(shape=shape, dtype="float64"), meta_obj=like, no_data=-1)
        ones = True  # unit weights are generated on the device; nothing is uploaded
    if accum.dtype != "float64":
        raise Exception("Accumulation array must be of type 'float64'!")
    if accum.shape != tuple(shape):
        raise RuntimeError("Accumulation array must have same dimensions as proportions array!")
    if not accum.flags["C_CONTIGUOUS"]:
        raise Exception("Accumulation array must be C-contiguous")
    return accum, ones


def FlowAccumulation(dem: rdarray, method: Optional[str] = None, exponent: Optional[float] = None,
                     weights: Optional[rdarray] = None, in_place: bool = False) -> rdarray:
    """Flow accumulation (reference FlowAccumulation, :490-596).  Methods on the H100 path:
    ``D8`` / ``OCallaghanD8`` (FA_D8), ``Dinf`` / ``Tarboton`` (FA_Tarboton), ``D4`` / ``OCallaghanD4`` (FA_D4),
    ``Quinn``, ``Holmgren`` (exponent), ``Freeman`` (exponent)."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    accum, ones = _accum_array(dem, weights, in_place, dem.shape)
    _add_analysis(accum, "FlowAccumulation(dem, method={0}, exponent={1}, weights={2}, in_place={3})".format(
        method, exponent, "None" if weights is None else "weights", in_place))
    d = _dem_f32(dem, "FlowAccumulation")
    h, w = d.shape
    L = _lib.lib()
    if method in _D8_METHODS:
        _lib.check(L.rdb200_fa_d8_f32_f64(_lib.ptr(d), _lib.ptr(accum), w, h, _nodata_f32(dem), int(ones)))
    elif method in _DINF_METHODS:
        _lib.check(L.rdb200_fa_tarboton_f32_f64(_lib.ptr(d), _lib.ptr(accum), w, h, _nodata_f32(dem), int(ones)))
    elif method in _D4_METHODS or method == "Quinn" or method in _EXPONENT_METHODS:
        # FM_x into a device-resident proportions array + the generic accumulation (flow_accumulation.hpp:18-20,28)
        if ones:
            accum[...] = 1.0
        nd = _nodata_f32(dem)
        if method in _D4_METHODS:
            _lib.check(L.rdb200_fa_d4_f32_f64(_lib.ptr(d), _lib.ptr(accum), w, h, nd))
        elif method == "Quinn":
            _lib.check(L.rdb200_fa_quinn_f32_f64(_lib.ptr(d), _lib.ptr(accum), w, h, nd))
        else:
            if exponent is None:
                raise Exception(f'FlowAccumulation method "{method}" requires an exponent!')
            fn = L.rdb200_fa_freeman_f32_f64 if method == "Freeman" else L.rdb200_fa_holmgren_f32_f64
            _lib.check(fn(_lib.ptr(d), _lib.ptr(accum), w, h, nd, float(exponent)))
    elif method in _OUT_OF_SCOPE_METHODS:
        raise Exception(f'FlowAccumulation method "{method}" is outside the GPU hot path '
                        "(random-walk metric; use the reference CPU implementation)")
    else:
        raise Exception("Invalid FlowAccumulation method. Valid methods are: " +
                        ", ".join(_DINF_METHODS + ("Quinn",) + _D8_METHODS + _D4_METHODS + _EXPONENT_METHODS +
                                  _OUT_OF_SCOPE_METHODS))
    accum.no_data = -1
    return accum


def FlowAccumFromProps(props: rd3array, weights: Optional[rdarray] = None, in_place: bool = False) -> rdarray:
    """Flow accumulation from (H, W, 9) proportions (reference FlowAccumFromProps, :599-647)."""
    if type(props) is not rd3array:
        raise Exception("A richdem.rd3array or numpy.ndarray is required!")
    if props.ndim != 3 or props.shape[2] != 9:
        raise RuntimeError("Array must have three dimensions with the last of size 9!")
    accum, ones = _accum_array(props, weights, in_place, props.shape[0:2])
    if ones:
        accum[...] = 1.0
    _add_analysis(accum, "FlowAccumFromProps(dem, weights={0}, in_place={1})".format(
        "None" if weights is None else "weights", in_place))
    p = np.ascontiguousarray(props, dtype=np.float32)
    h, w = p.shape[0:2]
    _lib.check(_lib.lib().rdb200_flow_accumulation_props_f64(_lib.ptr(p), _lib.ptr(accum), w, h))
    accum.no_data = -1
    return accum


def FlowProportions(dem: rdarray, method: Optional[str] = None, exponent: Optional[float] = None) -> rd3array:
    """Flow proportions (reference FlowProportions, :650-732): (H, W, 9) float32, slot 0 holds
    -2 NoData / -1 no flow / 0 has flow, slots 1..8 the share sent to D8 neighbour n."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    fprops = rd3array(np.empty(shape=dem.shape + (9,), dtype="float32"), meta_obj=dem, no_data=-2)
    _add_analysis(fprops, f"FlowProportions(dem, method={method}, exponent={exponent})")
    d = _dem_f32(dem, "FlowProportions")
    h, w = d.shape
    L = _lib.lib()
    if method in _D8_METHODS:
        _lib.check(L.rdb200_fm_d8_f32(_lib.ptr(d), _lib.ptr(fprops), w, h, _nodata_f32(dem)))
    elif method in _DINF_METHODS:
        _lib.check(L.rdb200_fm_tarboton_f32(_lib.ptr(d), _lib.ptr(fprops), w, h, _nodata_f32(dem)))
    elif method in _D4_METHODS:
        _lib.check(L.rdb200_fm_d4_f32(_lib.ptr(d), _lib.ptr(fprops), w, h, _nodata_f32(dem)))
    elif method == "Quinn":
        _lib.check(L.rdb200_fm_quinn_f32(_lib.ptr(d), _lib.ptr(fprops), w, h, _nodata_f32(dem)))
    elif method in _EXPONENT_METHODS:
        if exponent is None:
            raise Exception('FlowProportions method "' + method + '" requires an exponent!')
        fn = L.rdb200_fm_freeman_f32 if method == "Freeman" else L.rdb200_fm_holmgren_f32
        _lib.check(fn(_lib.ptr(d), _lib.ptr(fprops), w, h, _nodata_f32(dem), float(exponent)))
    elif method in _OUT_OF_SCOPE_METHODS:
        raise Exception(f'FlowProportions method "{method}" is outside the GPU hot path '
                        "(random-walk metric; use the reference CPU implementation)")
    else:
        raise Exception("Invalid FlowProportions method. Valid methods are: " +
                        ", ".join(_DINF_METHODS + ("Quinn",) + _D8_METHODS + _D4_METHODS + _EXPONENT_METHODS +
                                  _OUT_OF_SCOPE_METHODS))
    fprops.no_data = -2
    return fprops


_TERRAIN_ATTRIBS = {"slope_riserun": 0, "slope_percentage": 1, "slope_degrees": 2, "slope_radians": 3, "aspect": 4,
                    "curvature": 5, "planform_curvature": 6, "profile_curvature": 7}


def _terrain_attrib_id(attrib: str) -> int:
    """RDB200_TA_* number of a TerrainAttribute name (also used by sharded.terrain_attribute_band)."""
    if attrib not in _TERRAIN_ATTRIBS:
        raise Exception("Invalid TerrainAttributes attribute. Valid attributes are: " + ", ".join(_TERRAIN_ATTRIBS.keys()))
    return _TERRAIN_ATTRIBS[attrib]


def TerrainAttribute(dem: rdarray, attrib: str, zscale: float = 1.0) -> rdarray:
    """richdem.TerrainAttribute (wrappers/pyrichdem/richdem/__init__.py:735-794) over TA_* (methods/
    terrain_attributes.hpp:370-538): Horn (1981) slope / aspect, Zevenbergen & Thorne (1987) curvatures; float32
    result with no_data -9999.  Cell lengths come from the geotransform (1 x 1 when there is none, as in the
    reference's wrap())."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    attrib_id = _terrain_attrib_id(attrib)
    d = _dem_f32(dem, "TerrainAttribute")
    h, w = d.shape
    gt = dem.geotransform
    if gt is None:
        print("Warning! No geotransform defined. Choosing a standard one! (Top left cell's top let corner at <0,0>; cells are 1x1.)")
        gt = [0, 1, 0, 0, 0, -1]
    result = rdarray(np.zeros((h, w), np.float32), meta_obj=dem, no_data=-9999)
    _add_analysis(result, f"TerrainAttribute(dem, attrib={attrib}, zscale={zscale})")
    _lib.check(_lib.lib().rdb200_terrain_attribute_f32(attrib_id, _lib.ptr(d), _lib.ptr(result), w, h,
                                                        _nodata_f32(dem), -9999.0, float(zscale), abs(float(gt[1])),
                                                        abs(float(gt[5]))))
    return result


# ---- the reference's native cache format (host I/O; nothing runs on the GPU) ---------------------------------------------
_NATIVE_NO_I = 0xFFFFFFFF  # common/Array2D.hpp:103-115: "number of data cells not counted"


def SaveNative(rda: rdarray, filename: str) -> None:
    """Writes ``rda`` in the uncompressed native cache format of richdem::Array2D (`saveToCache`, common/Array2D.hpp:209-241):
    int32 height, width, x offset, y offset | uint32 data-cell count | NoData (the raster's dtype) | 6 doubles geotransform |
    size_t projection length + bytes | the cells, row-major.  The file carries no dtype tag: the reader has to know it
    (`richdem::Array2D<T>(filename, true)`, :420-423)."""
    if type(rda) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if rda.ndim != 2:
        raise RuntimeError("Array must have two dimensions!")
    a = np.ascontiguousarray(rda)
    h, w = a.shape
    nd = rda.no_data if rda.no_data is not None else -9999
    gt = rda.geotransform if rda.geotransform is not None else [0, 1, 0, 0, 0, -1]
    proj = (rda.projection or "").encode()
    with open(filename, "wb") as f:
        f.write(np.array([h, w, 0, 0], np.int32).tobytes())
        f.write(np.array([_NATIVE_NO_I], np.uint32).tobytes())
        f.write(np.array([nd], a.dtype).tobytes())
        f.write(np.array(list(gt), np.float64).reshape(6).tobytes())
        f.write(np.array([len(proj)], np.uint64).tobytes())
        f.write(proj)
        f.write(a.tobytes())


def LoadNative(filename: str, dtype="float32") -> rdarray:
    """Reads a raster written by richdem::Array2D<dtype>::saveToCache (or :func:`SaveNative`); see there for the layout."""
    dt = np.dtype(dtype)
    with open(filename, "rb") as f:
        head = f.read(16 + 4 + dt.itemsize + 48 + 8)
        if len(head) < 16 + 4 + dt.itemsize + 48 + 8:
            raise RuntimeError(f"Failed to load native file '{filename}'!")
        h, w, _xoff, _yoff = np.frombuffer(head, np.int32, 4, 0)
        nd = np.frombuffer(head, dt, 1, 20)[0]
        gt = np.frombuffer(head, np.float64, 6, 20 + dt.itemsize)
        plen = int(np.frombuffer(head, np.uint64, 1, 20 + dt.itemsize + 48)[0])
        if h < 0 or w < 0 or plen > (1 << 20):
            raise RuntimeError(f"'{filename}' is not a native RichDEM raster of dtype {dt}")
        proj = f.read(plen).decode(errors="replace")
        data = np.fromfile(f, dt, int(h) * int(w))
    if data.size != int(h) * int(w):
        raise RuntimeError(f"'{filename}' is truncated: {data.size} of {int(h) * int(w)} cells")
    out = rdarray(data.reshape(int(h), int(w)), no_data=nd.item(), geotransform=[float(g) for g in gt])
    out.projection = proj
    return out


# ---- C++-only functions of the path, exposed for completeness ---------------------------------
def FlowDirectionsD8(dem: rdarray) -> rdarray:
    """richdem::d8_flow_directions (flowmet/d8_flowdirs.hpp:96-123): uint8 codes 0..8, 255 NoData."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    d = _dem_f32(dem, "FlowDirectionsD8")
    h, w = d.shape
    out = rdarray(np.empty((h, w), np.uint8), meta_obj=dem, no_data=255)
    _lib.check(_lib.lib().rdb200_d8_flow_directions_f32(_lib.ptr(d), _lib.ptr(out), w, h, _nodata_f32(dem)))
    out.no_data = 255
    return out


def FlowDirectionsD8Resolved(dem: rdarray, alter: bool = False) -> rdarray:
    """richdem::barnes_flat_resolution_d8 (flats/flat_resolution.hpp:588-607; the pipeline of apps/rd_d8_flowdirs.cpp):
    D8 directions in which drainable flats flow along the Barnes (2014) increment mask.  ``alter=True`` raises the
    flat cells of ``dem`` in place instead (d8_flats_alter_dem) and recomputes the directions."""
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if dem.dtype != np.float32 or not dem.flags["C_CONTIGUOUS"]:
        raise Exception("FlowDirectionsD8Resolved needs a C-contiguous float32 rdarray")
    h, w = dem.shape
    out = rdarray(np.empty((h, w), np.uint8), meta_obj=dem, no_data=255)
    _lib.check(_lib.lib().rdb200_d8_flow_directions_flats_f32(_lib.ptr(dem), _lib.ptr(out), w, h, _nodata_f32(dem), int(alter)))
    out.no_data = 255
    return out


def D8FlowAccum(flowdirs: np.ndarray) -> rdarray:
    """richdem::d8_flow_accum (methods/d8_methods.hpp:47-139) on a uint8 direction grid."""
    f = np.ascontiguousarray(flowdirs, dtype=np.uint8)
    if f.ndim != 2:
        raise RuntimeError("Array must have two dimensions!")
    h, w = f.shape
    out = rdarray(np.empty((h, w), np.int32), no_data=-1)
    _lib.check(_lib.lib().rdb200_d8_flow_accum_u8_i32(_lib.ptr(f), _lib.ptr(out), w, h))
    return out


def FlatMask(dem: rdarray):
    """richdem::GetFlatMask (flats/Barnes2014.hpp:398-467): (mask, labels) int32 arrays."""
    d = _dem_f32(dem, "FlatMask")
    h, w = d.shape
    mask = np.empty((h, w), np.int32)
    labels = np.empty((h, w), np.int32)
    _lib.check(_lib.lib().rdb200_get_flat_mask_f32(_lib.ptr(d), _lib.ptr(mask), _lib.ptr(labels), w, h,
                                                    _nodata_f32(dem)))
    return mask, labels
