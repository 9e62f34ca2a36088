"""The C ABI's raster entry points on the CPU fiber model of tests/emu, whose "device memory" is host memory.

* Twins: every host entry point stages its arrays through device workspace and runs the call its rdb200_dev_ twin makes
  on the caller's arrays, so both must give the same bits, for float32 and float64 DEMs, on a width that is a multiple of
  4 and on an odd one.  Outputs the host entry point does not download (the DEM of d8_flow_directions_flats without
  alter) and inputs it does not upload (the accumulator of FA_D8 / FA_Tarboton with accum_is_ones) are covered too.
* Arguments: every host, device and row-band entry point on a raster, given a null array or a zero width, returns 1 with
  its null-pointer message or the dimension check's message, before any stage runs.  Null device pointers are only ever
  handed to the emulation.
"""
import ctypes as C
import importlib.util
import os
import sys

import numpy as np
import pytest

import oracle
from richdem_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
ND = -9999.0
H = 23
WIDTHS = (48, 37)
DIMS_MSG = "raster dimensions must be positive (got 0 x %d)" % H


def _load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def emu_lib():
    if sys.platform != "linux" or os.uname().machine != "x86_64":
        pytest.skip("the fiber switch of tests/emu is x86-64 SysV only")
    path = _load_module("build_emu", os.path.join(HERE, "emu", "build_emu.py")).build()
    L = C.CDLL(str(path))
    assert L.rdb200_emulated() == 1
    for name, argtypes in _lib.SIGNATURES.items():
        f = getattr(L, name)
        f.argtypes = argtypes
        f.restype = C.c_int
    L.rdb200_last_error.restype = C.c_char_p
    L.rdb200_last_error.argtypes = []
    assert L.rdb200_init(0) == 0
    return L


@pytest.fixture()
def L(emu_lib):
    assert emu_lib.rdb200_set_param(b"fill_use_tma", 0) == 0  # TMA / mbarrier PTX is not emulated
    yield emu_lib
    emu_lib.rdb200_set_param(b"reset_defaults", 1)


def _dem(w, dtype):
    dem = oracle.fbm_terrain(H, w, seed=w, quantum=0.5).astype(np.float64)
    dem[3:7, 5:11] = ND
    dem[12, w // 2] -= 40.0  # a pit
    if dtype == np.float64:  # detail below float resolution: the keys take the ranked route
        dem += np.where(dem != ND, np.random.default_rng(w).uniform(0, 1e-9, dem.shape), 0.0)
    return np.ascontiguousarray(dem.astype(dtype))


@pytest.fixture(scope="module")
def inputs(emu_lib):
    """(width, dtype) -> DEM, plus D8 directions and D-infinity proportions of the float32 DEM by width"""
    out = {}
    for w in WIDTHS:
        n = w * H
        for dt in (np.float32, np.float64):
            out[w, dt] = _dem(w, dt)
        dirs, props = np.zeros(n, np.uint8), np.zeros(9 * n, np.float32)
        dem = out[w, np.float32]
        assert emu_lib.rdb200_d8_flow_directions_f32(dem.ctypes.data, dirs.ctypes.data, w, H, ND) == 0
        assert emu_lib.rdb200_fm_tarboton_f32(dem.ctypes.data, props.ctypes.data, w, H, ND) == 0
        out[w, "DIRS"], out[w, "PROPS"] = dirs, props
    return out


# Argument tokens: Z the DEM; U8 / I32 / F32 / P9 (9 floats per cell) output arrays; ACC float64 weights (the
# accumulator); DIRS, PROPS inputs from the fixture; OUT a required int32 result, OPT / OPTF optional int32 / float results;
# COMM a single-rank communicator, COMMOPT one that may be null; W, H, ND; anything else is passed as it is.
ARRAYS = ("Z", "U8", "I32", "F32", "P9", "ACC", "DIRS", "PROPS")
REQUIRED = ARRAYS + ("OUT", "COMM")


def _args(tokens, w, dtype, inputs, comm=None, null_at=None):
    """ctypes arguments for tokens, and what each one points at (for comparing outputs)"""
    n = w * H
    rng = np.random.default_rng(w + 1)
    args, held = [], []
    for i, t in enumerate(tokens):
        obj = None
        if t == "Z":
            obj = inputs[w, dtype].copy()
        elif t == "U8":
            obj = np.full(n, 0xAB, np.uint8)
        elif t == "I32":
            obj = np.full(n, -7, np.int32)
        elif t == "F32":
            obj = np.full(n, 12345.0, np.float32)
        elif t == "P9":
            obj = np.full(9 * n, 12345.0, np.float32)
        elif t == "ACC":
            obj = rng.integers(-(1 << 20), 1 << 20, n).astype(np.float64) * 2.0 ** -20
        elif t in ("DIRS", "PROPS"):
            obj = inputs[w, t].copy()
        elif t in ("OUT", "OPT"):
            obj = C.c_int32(-5)
        elif t == "OPTF":
            obj = C.c_float(-5.0)
        if i == null_at:
            args.append(None)
        elif isinstance(obj, np.ndarray):
            args.append(obj.ctypes.data)
        elif obj is not None:
            args.append(C.byref(obj))
        elif t in ("COMM", "COMMOPT"):
            args.append(comm)
        else:
            args.append({"W": w, "H": H, "ND": ND}.get(t, t))
        if obj is not None:
            held.append(obj)
    return args, held


def _call(L, name, args):
    rc = getattr(L, name)(*args)
    return rc, (L.rdb200_last_error() or b"").decode()


def _outputs(held):
    return [o.tobytes() if isinstance(o, np.ndarray) else bytes(o) for o in held]


# ---- host / device twins: (host entry point, its arguments, device entry point, its arguments) -------------------------
def _twins(t):
    same = []
    for topo in ("d8", "d4"):
        same += [(f"fill_depressions_{topo}_{t}", ["Z", "W", "H"]), (f"pit_mask_{topo}_{t}", ["Z", "U8", "W", "H", "ND"]),
                 (f"has_depressions_{topo}_{t}", ["Z", "W", "H", "OUT"])]
    same += [(f"resolve_flats_epsilon_{t}", ["Z", "W", "H", "ND"]), (f"d8_flow_directions_{t}", ["Z", "U8", "W", "H", "ND"])]
    same += [(f"terrain_attribute_{t}", [a, "Z", "F32", "W", "H", "ND", -1.0, 1.5, 2.0, 3.0]) for a in range(8)]
    renamed = []
    fm = {"d8": (0, 0.0), "tarboton": (1, 0.0), "d4": (2, 0.0), "quinn": (3, 1.0), "holmgren": (3, 4.5), "freeman": (4, 1.3)}
    for metric, (m, x) in fm.items():
        xs = [x] if metric in ("holmgren", "freeman") else []
        renamed.append((f"fm_{metric}_{t}", ["Z", "P9", "W", "H", "ND"] + xs,
                        f"fm_method_{t}", [m, "Z", "P9", "W", "H", "ND", x]))
    fa = dict((k, fm[k]) for k in ("d4", "quinn", "holmgren", "freeman"))
    for metric, (m, x) in fa.items():
        xs = [x] if metric in ("holmgren", "freeman") else []
        renamed.append((f"fa_{metric}_{t}_f64", ["Z", "ACC", "W", "H", "ND"] + xs,
                        f"fa_method_{t}_f64", [m, "Z", "ACC", "W", "H", "ND", x]))
    for ones in (0, 1):
        same += [(f"fa_d8_{t}_f64", ["Z", "ACC", "W", "H", "ND", ones]), (f"fa_tarboton_{t}_f64", ["Z", "ACC", "W", "H", "ND", ones])]
    if t == "f32":
        same += [("d8_flow_directions_flats_f32", ["Z", "U8", "W", "H", "ND", alter]) for alter in (0, 1)]
        same += [("d8_flow_accum_u8_i32", ["DIRS", "I32", "W", "H"]), ("flow_accumulation_props_f64", ["PROPS", "ACC", "W", "H"])]
        same += [(f"fm_{metric}_f32", ["Z", "P9", "W", "H", "ND"]) for metric in ("d8", "tarboton")]
    else:
        same += [("fa_d4_f64_f64", ["Z", "ACC", "W", "H", "ND"]),
                 ("f64_order_keys", ["Z", "F32", "W", "H", "ND", "OPTF", "OPT"])]
    cases = [("rdb200_" + h, a, "rdb200_dev_" + h, a) for h, a in same]
    cases += [("rdb200_" + h, ha, "rdb200_dev_" + d, da) for h, ha, d, da in renamed]
    return cases


TWINS = [(np.float32, c) for c in _twins("f32")] + [(np.float64, c) for c in _twins("f64")]


def _twin_id(case):
    dt, (h, ha, d, da) = case
    return f"{h[7:]}-{d[7:]}-" + "-".join(str(a) for a in da if isinstance(a, (int, float)))


@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("case", TWINS, ids=[_twin_id(c) for c in TWINS])
def test_host_entry_equals_its_device_twin(L, inputs, case, w):
    dtype, (host, host_tokens, dev, dev_tokens) = case
    outs = []
    for name, tokens in ((host, host_tokens), (dev, dev_tokens)):
        args, held = _args(tokens, w, dtype, inputs)
        rc, err = _call(L, name, args)
        assert rc == 0, (name, err)
        outs.append(_outputs(held))
    assert len(outs[0]) == len(outs[1])
    for k, (a, b) in enumerate(zip(*outs)):
        assert a == b, f"{host} and {dev} differ in argument array {k}"


# ---- null arrays and zero widths -------------------------------------------------------------------------------------
def _null_message(name):
    stem = name.replace("rdb200_dev_", "").replace("rdb200_", "")
    for prefix, msg in (("fill_depressions", "fill_depressions: null dem"), ("resolve_flats", "resolve_flats: null dem"),
                        ("pit_mask", "pit_mask: null pointer"), ("has_depressions", "has_depressions: null pointer"),
                        ("d8_flow_directions_flats", "d8_flow_directions_flats: null pointer"),
                        ("d8_flow_directions", "d8_flow_directions: null pointer"),
                        ("d8_flow_accum", "d8_flow_accum: null pointer"), ("fm_", "flow metric: null pointer"),
                        ("terrain_attribute", "terrain attribute: null pointer"),
                        ("flow_accumulation_props", "flow_accumulation: null pointer"),
                        ("fa_", "flow accumulation: null pointer"), ("f64_order_keys", "f64_order_keys: null pointer")):
        if stem.startswith(prefix):
            return msg
    raise KeyError(name)


def _raster_entries():
    """(dtype, entry point, tokens, message for a null array, message for a zero width) of every entry point on a raster"""
    out, seen = [], set()
    for dt, (h, ha, d, da) in TWINS:
        for name, tokens in ((h, ha), (d, da)):
            if name not in seen:
                seen.add(name)
                out.append((dt, name, tokens, _null_message(name), DIMS_MSG))
    out.append((np.float32, "rdb200_get_flat_mask_f32", ["Z", "I32", "I32", "W", "H", "ND"], "get_flat_mask: null pointer",
                DIMS_MSG))
    out.append((np.float32, "rdb200_dev_generate_fbm_f32", ["F32", "W", "H", 0, 7, 4, 0.5], "generate_fbm: null pointer",
                DIMS_MSG))
    band = [
        ("fill_depressions_d8_f32", ["COMMOPT", "Z", "W", "H", 0, 0, 0, "H", "OPT"], "mgpu_fill"),
        ("fill_depressions_d4_f32", ["COMMOPT", "Z", "W", "H", 0, 0, 0, "H", "OPT"], "mgpu_fill"),
        ("pit_mask_d8_f32", ["COMM", "Z", "U8", "W", "H", "ND", 0, 0, 0, "H"], "mgpu_pit_mask"),
        ("pit_mask_d4_f32", ["COMM", "Z", "U8", "W", "H", "ND", 0, 0, 0, "H"], "mgpu_pit_mask"),
        ("has_depressions_d8_f32", ["COMM", "Z", "W", "H", 0, 0, 0, "H", "OUT"], "mgpu_has_depressions"),
        ("has_depressions_d4_f32", ["COMM", "Z", "W", "H", 0, 0, 0, "H", "OUT"], "mgpu_has_depressions"),
        ("fa_f32_f64", ["COMMOPT", "Z", "ACC", "W", "H", "ND", 0, 0, 1, 0, "OPT"], "mgpu_fa"),
        ("fa_method_f32_f64", ["COMMOPT", "Z", "ACC", "W", "H", "ND", 0, 0, 3, 1.0, 0, "OPT"], "mgpu_fa"),
        ("resolve_flats_epsilon_f32", ["COMM", "Z", "W", "H", "ND", 0, 0, "OPT"], "mgpu_resolve_flats"),
        ("d8_flow_directions_flats_f32", ["COMM", "Z", "U8", "W", "H", "ND", 0, 0, 1, "OPT"], "mgpu_d8_flow_directions_flats"),
        ("d8_flow_accum_u8_i32", ["COMM", "DIRS", "I32", "W", "H", 0, 0, "OPT"], "mgpu_d8_flow_accum"),
        ("flow_accumulation_props_f64", ["COMM", "PROPS", "ACC", "W", "H", 0, 0, "OPT"], "mgpu_flow_accumulation_props"),
        ("fm_method_f32", ["COMM", 1, "Z", "P9", "W", "H", "ND", 0, 0, 0.0], "mgpu_fm_method"),
        ("terrain_attribute_f32", ["COMM", 2, "Z", "F32", "W", "H", "ND", -1.0, 1.0, 1.0, 1.0, 0, 0], "mgpu_terrain_attribute"),
    ]
    for name, tokens, what in band:
        # these two check the band geometry first, as every band driver does: a zero width leaves no owned rows
        dims = f"{what}: band has no owned rows (0 x {H})" if what in ("mgpu_fm_method", "mgpu_terrain_attribute") else DIMS_MSG
        out.append((np.float32, "rdb200_mgpu_" + name, tokens, f"{what}: null pointer", dims))
    return out


ENTRIES = _raster_entries()


@pytest.fixture(scope="module")
def comm(emu_lib):
    c = C.c_void_p()
    assert emu_lib.rdb200_comm_create_callbacks(C.byref(c), 0, 1, None, None, None) == 0
    yield c.value
    emu_lib.rdb200_comm_destroy(c.value)


@pytest.mark.parametrize("entry", ENTRIES, ids=[e[1][7:] for e in ENTRIES])
def test_null_arrays_and_zero_width_fail_with_their_message(L, inputs, comm, entry):
    dtype, name, tokens, null_msg, dims_msg = entry
    w = WIDTHS[0]
    nullable = [i for i, t in enumerate(tokens) if t in REQUIRED]
    assert nullable, name
    for i in nullable:
        args, _ = _args(tokens, w, dtype, inputs, comm, null_at=i)
        assert _call(L, name, args) == (1, null_msg), (name, tokens[i])
    args, _ = _args(tokens, w, dtype, inputs, comm)
    args = [0 if t == "W" else a for t, a in zip(tokens, args)]
    assert _call(L, name, args) == (1, dims_msg), name
