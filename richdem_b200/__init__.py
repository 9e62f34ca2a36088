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
from typing import Any, Callable, NamedTuple, Optional, Tuple

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


# ---- one body per stage; an element-type record carries what float32 and float64 DEMs differ in (f64.py binds _F64) -----
class _Elem(NamedTuple):
    dtype: type
    suffix: str  # of the C symbols: rdb200_<stage>_<suffix>
    nodata: Callable[[Any], float]  # a raster's no_data as the C ABI takes it
    refusal: str  # the wrong-dtype message, with {what} and {dtype}
    fa_valid: Tuple[str, ...]  # the methods FlowAccumulation lists as valid
    fa_refused: Tuple[str, ...]  # known methods FlowAccumulation refuses for this element type
    nodata_first: bool  # FlowAccumulation / FlowProportions read no_data before they check the method
    epsilon_refusal: Optional[str]  # why FillDepressions(epsilon=True) is refused for this element type (None: it runs)


_F32 = _Elem(np.float32, "f32", lambda nd: float(np.float32(nd)),
             "{what}: the H100 path is built for float32 elevations (got '{dtype}'); "
             "convert with dem.astype('float32') -- there is no CPU fallback for other dtypes "
             "(float64 rasters: richdem_b200.f64 computes the float64 answer).",
             _DINF_METHODS + ("Quinn",) + _D8_METHODS + _D4_METHODS + _EXPONENT_METHODS + _OUT_OF_SCOPE_METHODS, (), False,
             None)
_F64 = _Elem(np.float64, "f64", float,
             "{what}: richdem_b200.f64 is built for float64 elevations (got '{dtype}'); "
             "float32 rasters go through richdem_b200 itself.",
             _D8_METHODS + _D4_METHODS, _DINF_METHODS + ("Quinn",) + _EXPONENT_METHODS + _OUT_OF_SCOPE_METHODS, True,
             "FillDepressions(epsilon=True) is not available for float64 rasters (its one-ulp steps are double ulps, which "
             "the float engine does not hold); fill float32 rasters with richdem_b200.FillDepressions(epsilon=True)")


def _dem(et: _Elem, dem: rdarray, what: str) -> np.ndarray:
    if dem.ndim != 2:
        raise RuntimeError("Array must have two dimensions!")  # pywrapper.hpp:118-119
    if dem.dtype != et.dtype:
        raise Exception(et.refusal.format(what=what, dtype=dem.dtype))
    if not dem.flags["C_CONTIGUOUS"]:
        raise Exception(f"{what}: the raster must be C-contiguous")
    return dem


def _nodata(et: _Elem, dem) -> float:
    nd = dem.no_data
    if nd is None:
        print("Warning! no_data was None. Setting it to -9999!")  # reference :204-206
        nd = -9999
    return et.nodata(nd)


def _check_topology(dem, topology: str) -> None:
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if topology not in ["D8", "D4"]:
        raise Exception("Unknown topology!")


def _fill_depressions(et, dem, epsilon, in_place, topology):
    _check_topology(dem, topology)
    if epsilon and et.epsilon_refusal:
        raise Exception(et.epsilon_refusal)
    if not in_place:
        dem = dem.copy()
    _add_analysis(dem, f"FillDepressions(dem, epsilon={epsilon})")
    d = _dem(et, dem, "FillDepressions")
    h, w = d.shape
    if epsilon:
        fn = getattr(_lib.lib(), f"rdb200_fill_depressions_epsilon_{topology.lower()}_{et.suffix}")
        _lib.check(fn(_lib.ptr(d), w, h, _nodata(et, dem)))
    else:
        fn = getattr(_lib.lib(), f"rdb200_fill_depressions_{topology.lower()}_{et.suffix}")
        _lib.check(fn(_lib.ptr(d), w, h))
    if not in_place:
        return dem
    return None


def _pit_mask(et, dem, topology):
    _check_topology(dem, topology)
    d = _dem(et, dem, "PitMask")
    h, w = d.shape
    out = rdarray(np.empty((h, w), np.uint8), meta_obj=dem, no_data=3)
    _add_analysis(out, f"PitMask(dem, topology={topology})")
    fn = getattr(_lib.lib(), f"rdb200_pit_mask_{topology.lower()}_{et.suffix}")
    _lib.check(fn(_lib.ptr(d), _lib.ptr(out), w, h, _nodata(et, dem)))
    out.no_data = 3
    return out


def _has_depressions(et, dem, topology):
    _check_topology(dem, topology)
    d = _dem(et, dem, "HasDepressions")
    h, w = d.shape
    out = C.c_int32(0)
    fn = getattr(_lib.lib(), f"rdb200_has_depressions_{topology.lower()}_{et.suffix}")
    _lib.check(fn(_lib.ptr(d), w, h, C.byref(out)))
    return bool(out.value)


def _resolve_flats(et, dem, in_place):
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if not in_place:
        dem = dem.copy()
    _add_analysis(dem, f"ResolveFlats(dem, in_place={in_place})")
    d = _dem(et, dem, "ResolveFlats")
    h, w = d.shape
    fn = getattr(_lib.lib(), f"rdb200_resolve_flats_epsilon_{et.suffix}")
    _lib.check(fn(_lib.ptr(d), w, h, _nodata(et, dem)))
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


def _flow_accumulation(et, dem, method, exponent, weights, in_place):
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    accum, ones = _accum_array(dem, weights, in_place, dem.shape)
    _add_analysis(accum, "FlowAccumulation(dem, method={0}, exponent={1}, weights={2}, in_place={3})".format(
        method, exponent, "None" if weights is None else "weights", in_place))
    d = _dem(et, dem, "FlowAccumulation")
    h, w = d.shape
    L = _lib.lib()
    nd = _nodata(et, dem) if et.nodata_first else None
    if method in et.fa_refused:
        raise Exception(f'FlowAccumulation method "{method}" is not available for {et.dtype.__name__} rasters '
                        "(it does arithmetic on elevation differences); valid methods here are: " + ", ".join(et.fa_valid))
    if method in _OUT_OF_SCOPE_METHODS:
        raise Exception(f'FlowAccumulation method "{method}" is outside the GPU hot path '
                        "(random-walk metric; use the reference CPU implementation)")
    if method not in et.fa_valid:
        raise Exception("Invalid FlowAccumulation method. Valid methods are: " + ", ".join(et.fa_valid))
    if not et.nodata_first:
        nd = _nodata(et, dem)
    if method in _D8_METHODS or method in _DINF_METHODS:
        name = "d8" if method in _D8_METHODS else "tarboton"
        _lib.check(getattr(L, f"rdb200_fa_{name}_{et.suffix}_f64")(_lib.ptr(d), _lib.ptr(accum), w, h, nd, int(ones)))
    else:
        # FM_x into a device-resident proportions array + the generic accumulation (flow_accumulation.hpp:18-20,28)
        if ones:
            accum[...] = 1.0
        name = "d4" if method in _D4_METHODS else method.lower()
        args = ()
        if method in _EXPONENT_METHODS:
            if exponent is None:
                raise Exception(f'FlowAccumulation method "{method}" requires an exponent!')
            args = (float(exponent),)
        _lib.check(getattr(L, f"rdb200_fa_{name}_{et.suffix}_f64")(_lib.ptr(d), _lib.ptr(accum), w, h, nd, *args))
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


def _flow_proportions(et, dem, method, exponent):
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    fprops = rd3array(np.empty(shape=dem.shape + (9,), dtype="float32"), meta_obj=dem, no_data=-2)
    _add_analysis(fprops, f"FlowProportions(dem, method={method}, exponent={exponent})")
    d = _dem(et, dem, "FlowProportions")
    h, w = d.shape
    nd = _nodata(et, dem) if et.nodata_first else None
    if method in _D8_METHODS:
        name = "d8"
    elif method in _DINF_METHODS:
        name = "tarboton"
    elif method in _D4_METHODS:
        name = "d4"
    elif method == "Quinn" or method in _EXPONENT_METHODS:
        if method != "Quinn" and exponent is None:
            raise Exception('FlowProportions method "' + method + '" requires an exponent!')
        name = method.lower()
    elif method in _OUT_OF_SCOPE_METHODS:
        raise Exception(f'FlowProportions method "{method}" is outside the GPU hot path '
                        "(random-walk metric; use the reference CPU implementation)")
    else:
        raise Exception("Invalid FlowProportions method. Valid methods are: " +
                        ", ".join(_DINF_METHODS + ("Quinn",) + _D8_METHODS + _D4_METHODS + _EXPONENT_METHODS +
                                  _OUT_OF_SCOPE_METHODS))
    if not et.nodata_first:
        nd = _nodata(et, dem)
    args = (float(exponent),) if method in _EXPONENT_METHODS else ()
    _lib.check(getattr(_lib.lib(), f"rdb200_fm_{name}_{et.suffix}")(_lib.ptr(d), _lib.ptr(fprops), w, h, nd, *args))
    fprops.no_data = -2
    return fprops


_TERRAIN_ATTRIBS = {"slope_riserun": 0, "slope_percentage": 1, "slope_degrees": 2, "slope_radians": 3, "aspect": 4,
                    "curvature": 5, "planform_curvature": 6, "profile_curvature": 7}


def _terrain_attrib_id(attrib: str) -> int:
    """RDB200_TA_* number of a TerrainAttribute name (also used by sharded.terrain_attribute_band)."""
    if attrib not in _TERRAIN_ATTRIBS:
        raise Exception("Invalid TerrainAttributes attribute. Valid attributes are: " + ", ".join(_TERRAIN_ATTRIBS.keys()))
    return _TERRAIN_ATTRIBS[attrib]


def _terrain_attribute(et, dem, attrib, zscale):
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    attrib_id = _terrain_attrib_id(attrib)
    d = _dem(et, dem, "TerrainAttribute")
    h, w = d.shape
    gt = dem.geotransform
    if gt is None:
        print("Warning! No geotransform defined. Choosing a standard one! (Top left cell's top let corner at <0,0>; cells are 1x1.)")
        gt = [0, 1, 0, 0, 0, -1]
    result = rdarray(np.zeros((h, w), np.float32), meta_obj=dem, no_data=-9999)
    _add_analysis(result, f"TerrainAttribute(dem, attrib={attrib}, zscale={zscale})")
    _lib.check(getattr(_lib.lib(), f"rdb200_terrain_attribute_{et.suffix}")(
        attrib_id, _lib.ptr(d), _lib.ptr(result), w, h, _nodata(et, dem), -9999.0, float(zscale), abs(float(gt[1])),
        abs(float(gt[5]))))
    return result


def _flow_directions_d8(et, dem):
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    d = _dem(et, dem, "FlowDirectionsD8")
    h, w = d.shape
    out = rdarray(np.empty((h, w), np.uint8), meta_obj=dem, no_data=255)
    _lib.check(getattr(_lib.lib(), f"rdb200_d8_flow_directions_{et.suffix}")(_lib.ptr(d), _lib.ptr(out), w, h,
                                                                            _nodata(et, dem)))
    out.no_data = 255
    return out


def _flow_directions_d8_resolved(et, dem, alter):
    if type(dem) is not rdarray:
        raise Exception("A richdem.rdarray or numpy.ndarray is required!")
    if et is _F32:  # the float32 function keeps its own refusal (no ndim check) and hands alter over as given
        if dem.dtype != np.float32 or not dem.flags["C_CONTIGUOUS"]:
            raise Exception("FlowDirectionsD8Resolved needs a C-contiguous float32 rdarray")
        d, alter = dem, int(alter)
    else:
        d, alter = _dem(et, dem, "FlowDirectionsD8Resolved"), int(bool(alter))
    h, w = d.shape
    out = rdarray(np.empty((h, w), np.uint8), meta_obj=dem, no_data=255)
    _lib.check(getattr(_lib.lib(), f"rdb200_d8_flow_directions_flats_{et.suffix}")(_lib.ptr(d), _lib.ptr(out), w, h,
                                                                                  _nodata(et, dem), alter))
    out.no_data = 255
    return out


def _flat_mask(et, dem):  # no rdarray check, in either module
    d = _dem(et, dem, "FlatMask")
    h, w = d.shape
    mask = np.empty((h, w), np.int32)
    labels = np.empty((h, w), np.int32)
    _lib.check(getattr(_lib.lib(), f"rdb200_get_flat_mask_{et.suffix}")(_lib.ptr(d), _lib.ptr(mask), _lib.ptr(labels), w, h,
                                                                       _nodata(et, dem)))
    return mask, labels


# ---------------------------------------------------------------------------------------------
def FillDepressions(dem: rdarray, epsilon: bool = False, in_place: bool = False,
                    topology: str = "D8") -> Optional[rdarray]:
    """Fills all depressions in a DEM (reference FillDepressions, :381-422 -> PriorityFlood_Zhou2016 for ``D8``,
    PriorityFlood_Barnes2014<D4> for ``D4``).  Returns the filled DEM unless ``in_place``.

    ``epsilon=True`` (PriorityFloodEpsilon_Barnes2014) leaves every filled cell one float step above the lowest of its
    neighbours, so the result drains without flats: the unique surface W = max(Z, min over the neighbours of
    nextafter(W, +inf)), with the raster's border and its ``no_data`` cells pinned.  It is never above the reference's
    result, but not bit-identical to it (the reference's depends on its queue's tie order; see
    ``rdb200_fill_depressions_epsilon_d8_f32`` in ``include/richdem_b200.h``)."""
    return _fill_depressions(_F32, dem, epsilon, in_place, topology)


def PitMask(dem: rdarray, topology: str = "D8") -> rdarray:
    """richdem::pit_mask<topo> (depressions/Barnes2014.hpp:593-676; app rd_depressions_mask): uint8 mask of the cells
    that lie in a depression, i.e. below the ``FillDepressions`` surface of ``dem`` (1), NoData cells (3) and all others
    (0), with ``no_data`` 3 and the input's metadata.  ``dem`` is not modified."""
    return _pit_mask(_F32, dem, topology)


def HasDepressions(dem: rdarray, topology: str = "D8") -> bool:
    """richdem::HasDepressions<topo> (depressions/Barnes2014.hpp:43-104; app rd_depressions_has): whether
    ``FillDepressions`` would raise any cell.  NoData is not special, as in the reference."""
    return _has_depressions(_F32, dem, topology)


def ResolveFlats(dem: rdarray, in_place: bool = False) -> Optional[rdarray]:
    """Imposes a local gradient on drainable flats (reference ResolveFlats, :461-487 ->
    ResolveFlatsEpsilon)."""
    return _resolve_flats(_F32, dem, in_place)


def FlowAccumulation(dem: rdarray, method: Optional[str] = None, exponent: Optional[float] = None,
                     weights: Optional[rdarray] = None, in_place: bool = False) -> rdarray:
    """Flow accumulation (reference FlowAccumulation, :490-596).  Methods on the H100 path:
    ``D8`` / ``OCallaghanD8`` (FA_D8), ``Dinf`` / ``Tarboton`` (FA_Tarboton), ``D4`` / ``OCallaghanD4`` (FA_D4),
    ``Quinn``, ``Holmgren`` (exponent), ``Freeman`` (exponent)."""
    return _flow_accumulation(_F32, dem, method, exponent, weights, in_place)


def FlowProportions(dem: rdarray, method: Optional[str] = None, exponent: Optional[float] = None) -> rd3array:
    """Flow proportions (reference FlowProportions, :650-732): (H, W, 9) float32, slot 0 holds
    -2 NoData / -1 no flow / 0 has flow, slots 1..8 the share sent to D8 neighbour n."""
    return _flow_proportions(_F32, dem, method, exponent)


def TerrainAttribute(dem: rdarray, attrib: str, zscale: float = 1.0) -> rdarray:
    """richdem.TerrainAttribute (wrappers/pyrichdem/richdem/__init__.py:735-794) over TA_* (methods/
    terrain_attributes.hpp:370-538): Horn (1981) slope / aspect, Zevenbergen & Thorne (1987) curvatures; float32
    result with no_data -9999.  Cell lengths come from the geotransform (1 x 1 when there is none, as in the
    reference's wrap())."""
    return _terrain_attribute(_F32, dem, attrib, zscale)


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
    return _flow_directions_d8(_F32, dem)


def FlowDirectionsD8Resolved(dem: rdarray, alter: bool = False) -> rdarray:
    """richdem::barnes_flat_resolution_d8 (flats/flat_resolution.hpp:588-607; the pipeline of apps/rd_d8_flowdirs.cpp):
    D8 directions in which drainable flats flow along the Barnes (2014) increment mask.  ``alter=True`` raises the
    flat cells of ``dem`` in place instead (d8_flats_alter_dem) and recomputes the directions."""
    return _flow_directions_d8_resolved(_F32, dem, alter)


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
    return _flat_mask(_F32, dem)
