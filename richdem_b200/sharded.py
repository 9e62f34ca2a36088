"""Row-band sharding of the hot path across GPUs: one process per GPU, ``torch.distributed`` for
the plumbing (NCCL over NVLink on the GPU box, gloo in the CPU unit tests).

A raster of H rows is cut into G contiguous row bands (row-major memory => a band is one
contiguous slab).  Rank g owns rows [r0, r1) and works on a *local raster* made of its rows plus
one ghost row on every side that touches another band.  The reference's own answer to distribution
is a two-round tile farm over MPI (programs/parallel_priority_flood/main.cpp:603-823); here the
exchange is a one-row halo (W*4 bytes per neighbour) plus a one-int all-reduce per global round.

Fill protocol (every value exchanged is a monotonically decreasing upper bound of the answer):

    state = begin(local raster, ghost rows = +inf)
    repeat:
        run(state)                      # relax the band to its local fixed point (many sweeps)
        send own edge rows to the neighbours, receive theirs
        if no rank's edge rows changed: break
        update ghost rows with what was received
    finish(state)

The band solver is pluggable so that the protocol can be unit-tested on CPU (gloo, world_size 2)
with a stand-in solver supplied by the test; the product always uses :class:`CudaBandSolver`.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Tuple

import numpy as np

try:  # torch is only needed for the distributed entry points
    import torch
    import torch.distributed as dist
except Exception:  # pragma: no cover
    torch = None
    dist = None


def band_bounds(height: int, world: int) -> List[Tuple[int, int]]:
    """Row ranges [r0, r1) of the ``world`` bands (sizes differ by at most one row)."""
    if world < 1:
        raise ValueError("world size must be >= 1")
    if height < world:
        raise ValueError(f"cannot cut {height} rows into {world} bands")
    base, extra = divmod(height, world)
    out, r = [], 0
    for g in range(world):
        n = base + (1 if g < extra else 0)
        out.append((r, r + n))
        r += n
    return out


def local_rows(height: int, world: int, rank: int) -> Tuple[int, int, int, int]:
    """(r0, r1, g_top, g_bot): owned rows and number of ghost rows above / below (0 or 1)."""
    r0, r1 = band_bounds(height, world)[rank]
    return r0, r1, (1 if rank > 0 else 0), (1 if rank < world - 1 else 0)


def _on_device(t) -> bool:
    """Band state lives in HBM: every tensor handed to the rdb200_dev_* entry points must be a CUDA tensor."""
    return bool(t.is_cuda)


class CudaBandSolver:
    """The product band solver: librichdem_b200's row-band fill entry points on device memory."""

    def __init__(self, local_dem: "torch.Tensor", coarse: Optional["torch.Tensor"] = None, pool: int = 0, row_offset: int = 0):
        """``coarse`` (optional): the filled ``pool`` x ``pool`` max-pooled raster of the WHOLE raster; the band then
        starts from its lifted water levels instead of +inf (``row_offset`` = global row of local row 0)."""
        from . import _lib
        assert _on_device(local_dem) and local_dem.dtype == torch.float32 and local_dem.is_contiguous()
        self._lib = _lib
        _lib.use_torch_stream()  # torch ops (halo copies, NCCL) and our kernels share one stream
        self.h, self.w = local_dem.shape
        self.device = local_dem.device
        self._state = C.c_void_p()
        if coarse is None:
            _lib.check(_lib.lib().rdb200_dev_fill_begin(C.byref(self._state), local_dem.data_ptr(), self.w, self.h))
        else:
            assert _on_device(coarse) and coarse.dtype == torch.float32 and coarse.is_contiguous() and pool >= 2
            self._coarse = coarse  # keep it alive until begin has consumed it
            _lib.check(_lib.lib().rdb200_dev_fill_begin_lifted(C.byref(self._state), local_dem.data_ptr(), self.w, self.h,
                                                               coarse.data_ptr(), coarse.shape[1], int(pool), int(row_offset)))

    def run(self) -> int:
        ch = C.c_int32(0)
        self._lib.check(self._lib.lib().rdb200_dev_fill_run(self._state, C.byref(ch)))
        return int(ch.value)

    def read_row(self, y: int) -> "torch.Tensor":
        row = torch.empty(self.w, dtype=torch.float32, device=self.device)
        self._lib.check(self._lib.lib().rdb200_dev_fill_read_row(self._state, y, row.data_ptr()))
        return row

    def update_row(self, y: int, row: "torch.Tensor") -> None:
        assert _on_device(row) and row.dtype == torch.float32 and row.numel() == self.w
        self._lib.check(self._lib.lib().rdb200_dev_fill_update_row(self._state, y, row.contiguous().data_ptr()))

    def blockmax(self, out: "torch.Tensor", pool: int, row_offset: int, skip_top: int, skip_bottom: int) -> None:
        """V-cycle restriction: max-combine the pool x pool block maxima of the owned rows' water surface into ``out``."""
        self._lib.check(self._lib.lib().rdb200_dev_fill_blockmax(self._state, out.data_ptr(), out.shape[1], out.shape[0], int(pool),
                                                             int(row_offset), int(skip_top), int(skip_bottom)))

    def prolong(self, coarse: "torch.Tensor", pool: int, row_offset: int) -> int:
        """V-cycle prolongation: interior cells drop to their block's coarse level where lower; returns tiles touched."""
        n = C.c_int32(0)
        self._lib.check(self._lib.lib().rdb200_dev_fill_prolong(self._state, coarse.data_ptr(), coarse.shape[1], int(pool),
                                                            int(row_offset), C.byref(n)))
        return int(n.value)

    def finish(self) -> "torch.Tensor":
        out = torch.empty((self.h, self.w), dtype=torch.float32, device=self.device)
        self._lib.check(self._lib.lib().rdb200_dev_fill_finish(self._state, out.data_ptr()))
        self._state = None
        return out


# ---- the library's communicator (C++ band drivers: rdb200_mgpu_*) -----------------------------------------------------
_EXCH_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t)
_ALLR_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int)
_COMMS = {}


class LibComm:
    """A rdb200_comm for a torch.distributed process group.  NCCL groups get the library's own NCCL communicator (the
    128-byte unique id travels over torch.distributed once); any other backend gets the callback communicator, whose two
    callbacks move the messages with torch.distributed.  ``cuda``: the bands live in CUDA memory, so the callbacks stage
    every message through host tensors (gloo moves host memory); otherwise (the CPU tests, where "device" memory is host
    memory) they send the buffers in place."""

    def __init__(self, group=None, cuda: bool = False):
        from . import _lib
        self._lib = _lib
        L = _lib.lib()
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.group = group
        self.cuda = bool(cuda)
        self.handle = C.c_void_p()
        backend = dist.get_backend(group) if dist.is_initialized() else "none"
        if backend == "nccl":
            ident = torch.zeros(128, dtype=torch.uint8)
            if self.rank == 0:
                _lib.check(L.rdb200_nccl_unique_id(ident.data_ptr()))
            dev_id = ident.cuda()
            dist.broadcast(dev_id, 0, group=group)
            ident = dev_id.cpu()
            _lib.check(L.rdb200_comm_create_nccl(C.byref(self.handle), self.rank, self.world, ident.data_ptr()))
            self.kind = "nccl"
        else:
            self._exch = _EXCH_FN(self._exchange)
            self._allr = _ALLR_FN(self._allreduce)
            _lib.check(L.rdb200_comm_create_callbacks(C.byref(self.handle), self.rank, self.world, None,
                                                      C.cast(self._exch, C.c_void_p), C.cast(self._allr, C.c_void_p)))
            self.kind = "callbacks"

    @staticmethod
    def _host(ptr, nbytes, dtype):
        buf = (C.c_uint8 * nbytes).from_address(ptr)
        return torch.frombuffer(buf, dtype=dtype)

    def _device(self, ptr, nbytes):
        return _view(ptr, (nbytes,), "|u1", torch.device("cuda", torch.cuda.current_device()))

    def _to_host(self, ptr, nbytes, dtype):
        """Host tensor that holds the message at ``ptr`` (a copy for a CUDA band; the library's stream is synchronised
        before a callback runs, so the copy sees its data)."""
        if self.cuda:
            return self._device(ptr, nbytes).cpu().view(dtype)
        return self._host(ptr, nbytes, dtype)

    def _from_host(self, ptr, host):
        """Put a host tensor received for ``ptr`` in place (a no-op for host memory: it was received there)."""
        if self.cuda:
            self._device(ptr, host.numel() * host.element_size()).copy_(host.view(torch.uint8))

    def _settle(self):
        if self.cuda:  # the callback returns when the data has arrived
            torch.cuda.current_stream().synchronize()

    def _exchange(self, user, su, ru, sd, rd, nbytes):
        try:
            ops, recvs = [], []
            for s_, r_, peer in ((su, ru, self.rank - 1), (sd, rd, self.rank + 1)):
                if s_:
                    recv = torch.empty(nbytes, dtype=torch.uint8) if self.cuda else self._host(r_, nbytes, torch.uint8)
                    recvs.append((r_, recv))
                    ops += [dist.P2POp(dist.isend, self._to_host(s_, nbytes, torch.uint8), peer, self.group),
                            dist.P2POp(dist.irecv, recv, peer, self.group)]
            if ops:
                for req in dist.batch_isend_irecv(ops):
                    req.wait()
            for r_, recv in recvs:
                self._from_host(r_, recv)
            self._settle()
            return 0
        except Exception:  # pragma: no cover
            import traceback
            traceback.print_exc()
            return 1

    def _allreduce(self, user, buf, count, op):
        try:
            dtype = torch.float32 if op in (0, 1) else torch.int32
            t = self._to_host(buf, count * 4, dtype)
            dist.all_reduce(t, op={0: dist.ReduceOp.MAX, 1: dist.ReduceOp.MIN, 2: dist.ReduceOp.MAX, 3: dist.ReduceOp.SUM}[op],
                            group=self.group)
            self._from_host(buf, t)
            self._settle()
            return 0
        except Exception:  # pragma: no cover
            import traceback
            traceback.print_exc()
            return 1


def lib_comm(group=None, cuda: bool = False) -> "LibComm":
    """The library's communicator for ``group`` (made once per group and memory kind); ``cuda``: the bands it connects
    live in CUDA memory."""
    key = (id(group), bool(cuda))
    if key not in _COMMS:
        _COMMS[key] = LibComm(group, cuda)
    return _COMMS[key]


def _neighbour_exchange(send_up, send_dn, g_top, g_bot, rank, group):
    """Send a row to each existing neighbour and receive theirs (batched P2P).  Each of
    send_up / send_dn may be a tensor or a list of tensors; returns matching receive buffers."""
    def as_list(x):
        return list(x) if isinstance(x, (list, tuple)) else [x]
    ops, recv_up, recv_dn = [], None, None
    if g_top:
        su = as_list(send_up)
        recv_up = [torch.empty_like(t) for t in su]
        for t, r in zip(su, recv_up):
            ops += [dist.P2POp(dist.isend, t, rank - 1, group), dist.P2POp(dist.irecv, r, rank - 1, group)]
    if g_bot:
        sd = as_list(send_dn)
        recv_dn = [torch.empty_like(t) for t in sd]
        for t, r in zip(sd, recv_dn):
            ops += [dist.P2POp(dist.isend, t, rank + 1, group), dist.P2POp(dist.irecv, r, rank + 1, group)]
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    return recv_up, recv_dn


def exchange_rows(local: "torch.Tensor", g_top: int, g_bot: int, group=None) -> None:
    """Fill the ghost rows of ``local`` with the neighbouring bands' edge rows (in place)."""
    if not (dist.is_initialized() and dist.get_world_size(group) > 1):
        return
    rank = dist.get_rank(group)
    h = local.shape[0]
    up = local[1].contiguous() if g_top else None
    dn = local[h - 2].contiguous() if g_bot else None
    ru, rd = _neighbour_exchange(up, dn, g_top, g_bot, rank, group)
    if ru is not None:
        local[0].copy_(ru[0])
    if rd is not None:
        local[h - 1].copy_(rd[0])


def coarse_fill(local_dem: "torch.Tensor", g_top: int, g_bot: int, row0: int, height: int, pool: int, group=None,
                keep_elevations: bool = False):
    """The filled ``pool`` x ``pool`` max-pooled raster of the whole (``height`` rows) raster, on every rank: each rank
    pools its owned rows into the coarse rows they touch, a MAX all-reduce merges the bands (a coarse row can straddle a
    seam), and every rank fills the small raster itself -- redundant, but it is 1/pool^2 of the work and saves a
    broadcast.  ``row0`` is the global row of ``local_dem``'s row 0 (the top ghost row if there is one)."""
    from . import _lib
    h, w = local_dem.shape
    wc, hc = (w + pool - 1) // pool, (height + pool - 1) // pool
    coarse = torch.full((hc, wc), float("-inf"), dtype=torch.float32, device=local_dem.device)
    owned = local_dem[g_top:h - g_bot]
    _lib.use_torch_stream()
    _lib.check(_lib.lib().rdb200_dev_maxpool_rows_f32(owned.data_ptr(), w, owned.shape[0], row0 + g_top, pool,
                                                      coarse.data_ptr(), wc, hc))
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(coarse, op=dist.ReduceOp.MAX, group=group)
    elevations = coarse.clone() if keep_elevations else None
    _lib.check(_lib.lib().rdb200_dev_fill_depressions_d8_f32(coarse.data_ptr(), wc, hc))
    return (coarse, elevations) if keep_elevations else coarse


def fill_band(local_dem: "torch.Tensor", g_top: int, g_bot: int, solver_cls=None, group=None,
              max_rounds: int = 100000, return_stats: bool = False, band_rounds: Optional[int] = None,
              multigrid: int = 0, row0: int = 0, height: int = 0, vcycle: int = 0, topology: str = "D8"):
    """Fill this rank's band.  ``local_dem`` is (g_top + owned + g_bot) x W with the ghost rows'
    contents ignored (they are initialised to +inf).  Returns (filled local raster incl. ghost rows,
    number of exchange rounds).  Collective: every rank of ``group`` must call it.

    ``topology`` is that of ``FillDepressions``: ``"D8"`` or ``"D4"`` (PriorityFlood_Barnes2014<D4>, through
    rdb200_mgpu_fill_depressions_d4_f32).  ``"D4"`` needs the C++ driver: the Python protocol (``solver_cls`` or
    RDB_BAND_DRIVER=python) fills with D8 only and refuses it.

    ``multigrid`` = k >= 2 (with ``row0`` = global row of local row 0 and ``height`` = rows of the whole raster): start
    from the lifted fill of the k x k max-pooled raster (see :func:`coarse_fill`) instead of +inf -- an upper bound of
    the answer, so the result is the same, after far fewer dependent rounds and halo exchanges.  ``vcycle`` = n > 0
    adds coarse-grid corrections: after every n halo exchanges that did not end the relaxation, the coarse surface is
    lowered to the block maxima of the bands' surfaces (restriction; MAX all-reduce), relaxed again on every rank and
    handed back (prolongation: fine = min(fine, lifted)) -- a lake that is a little too high is lowered by a sweep
    across the COARSE raster instead of one tile row / halo exchange at a time."""
    if topology not in ("D8", "D4"):
        raise Exception("Unknown topology!")
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    import os
    cxx = solver_cls is None and os.environ.get("RDB_BAND_DRIVER", "cxx") != "python"
    if _is_f64(local_dem):
        if not cxx:
            raise ValueError("fill_band: float64 bands run in the C++ band driver only; the Python band protocol "
                             "(solver_cls, RDB_BAND_DRIVER=python) takes float32")
    elif topology == "D4" and not cxx:
        raise ValueError("fill_band(topology='D4') runs in the C++ band driver only; the Python band protocol "
                         "(solver_cls, RDB_BAND_DRIVER=python) fills with D8")
    if cxx:
        # the product path: the whole band protocol (multigrid start, halo exchanges, V-cycle corrections, termination)
        # runs in C++ over the library's communicator (csrc/fill.cu: mgpu_fill_band); in place on local_dem
        _lib, fn, cm = _band_driver(local_dem, f"fill_depressions_{topology.lower()}_{{}}", group)
        row0, height = _band_geometry(local_dem, g_top, g_bot, row0, height, group)
        h_, w_ = local_dem.shape
        xr = C.c_int32(0)
        _lib.check(fn(cm.handle, local_dem.data_ptr(), w_, h_, int(g_top), int(g_bot), row0, height, C.byref(xr)))
        if return_stats:
            return local_dem, int(xr.value), _lib.stats()
        return local_dem, int(xr.value)
    if solver_cls is None:
        solver_cls = CudaBandSolver
        # halos are exchanged every `band_rounds` sweep rounds instead of after full local convergence,
        # so the flood enters a band from its neighbours when it arrives there rather than after the
        # band has been flooded once from its own raster edges
        import os
        from . import _lib
        if band_rounds is None:
            band_rounds = int(os.environ.get("RDB_BAND_ROUNDS", "64")) if world > 1 else 0
        # the round leash is a process-wide switch of the library: it is put back when this call is over
        with _lib.scoped_param("fill_band_rounds", band_rounds):
            return _fill_band_protocol(local_dem, g_top, g_bot, CudaBandSolver, group, max_rounds, return_stats, multigrid, row0,
                                       height, vcycle, rank, world)
    return _fill_band_protocol(local_dem, g_top, g_bot, solver_cls, group, max_rounds, return_stats, multigrid, row0, height, vcycle,
                               rank, world)


def _band_geometry(local_dem, g_top, g_bot, row0, height, group):
    """(row0, height) of a band: as given, or gathered from every rank's owned rows when ``height`` <= 0."""
    if height > 0:
        return int(row0), int(height)
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    h_ = local_dem.shape[0]
    if world == 1:
        return 0, h_
    hh = torch.tensor([h_ - g_top - g_bot], dtype=torch.int64, device=local_dem.device)
    allh = [torch.zeros_like(hh) for _ in range(world)]
    dist.all_gather(allh, hh, group=group)
    return int(sum(int(t.item()) for t in allh[:rank])) - g_top, int(sum(int(t.item()) for t in allh))


def pit_mask_band(local_dem: "torch.Tensor", g_top: int, g_bot: int, nodata: float, topology: str = "D8", row0: int = 0,
                  height: int = 0, group=None) -> "torch.Tensor":
    """PitMask over this rank's band.  ``local_dem`` is (g_top + owned + g_bot) x W; it is not modified and its ghost rows
    are not read.  ``row0`` / ``height`` as in :func:`fill_band` (gathered from the ranks when ``height`` <= 0).
    Collective.  Returns the uint8 mask of the local shape whose owned rows are the single-GPU bits (ghost rows
    unspecified).  A float64 band gives the bits of :func:`richdem_b200.f64` on the whole raster."""
    if topology not in ("D8", "D4"):
        raise Exception("Unknown topology!")
    _lib, fn, cm = _band_driver(local_dem, f"pit_mask_{topology.lower()}_{{}}", group)
    row0, height = _band_geometry(local_dem, g_top, g_bot, row0, height, group)
    h, w = local_dem.shape
    mask = torch.empty((h, w), dtype=torch.uint8, device=local_dem.device)
    _lib.check(fn(cm.handle, local_dem.data_ptr(), mask.data_ptr(), w, h, float(nodata), int(g_top), int(g_bot), row0, height))
    return mask


def has_depressions_band(local_dem: "torch.Tensor", g_top: int, g_bot: int, topology: str = "D8", row0: int = 0,
                         height: int = 0, group=None) -> bool:
    """HasDepressions of the whole raster, from this rank's band (arguments as :func:`pit_mask_band`).  A strict pit in any
    band answers after one all-reduce; the band fill runs only when there is none.  Collective; every rank gets the
    same answer.  Float64 bands too."""
    if topology not in ("D8", "D4"):
        raise Exception("Unknown topology!")
    _lib, fn, cm = _band_driver(local_dem, f"has_depressions_{topology.lower()}_{{}}", group)
    row0, height = _band_geometry(local_dem, g_top, g_bot, row0, height, group)
    h, w = local_dem.shape
    out = C.c_int32(0)
    _lib.check(fn(cm.handle, local_dem.data_ptr(), w, h, int(g_top), int(g_bot), row0, height, C.byref(out)))
    return bool(out.value)


def _fill_band_protocol(local_dem, g_top, g_bot, solver_cls, group, max_rounds, return_stats, multigrid, row0, height, vcycle, rank,
                        world):
    """The Python band protocol behind :func:`fill_band` (RDB_BAND_DRIVER=python and the CPU tests' solvers).  The ghost rows of
    ``local_dem`` are overwritten in place (with +inf or their lifted levels)."""
    h, w = local_dem.shape
    if multigrid >= 2:
        assert height > 0, "multigrid start needs the global geometry (row0, height)"
        coarse, coarse_z = coarse_fill(local_dem, g_top, g_bot, row0, height, multigrid, group, keep_elevations=True)
        for on, y in ((g_top, 0), (g_bot, h - 1)):  # ghost rows start at their lifted levels too
            if on:
                local_dem[y].copy_(coarse[(row0 + y) // multigrid].repeat_interleave(multigrid)[:w])
        solver = solver_cls(local_dem, coarse, multigrid, row0)
        if vcycle > 0:
            from . import _lib
            rounds = 0
            while True:
                # at least two runs per burst: the first one always exchanges halos (prolongation may have lowered edge
                # rows without the sweep noticing), only a later one can find that nothing moves any more
                r, done = _relax_band(solver, g_top, g_bot, rank, world, group, max_rounds, stop_after=max(2, vcycle))
                rounds += r
                if done:
                    break
                bm = torch.full_like(coarse, float("-inf"))
                solver.blockmax(bm, multigrid, row0, g_top, g_bot)
                if world > 1:
                    dist.all_reduce(bm, op=dist.ReduceOp.MAX, group=group)
                torch.minimum(coarse, bm, out=coarse)
                _lib.check(_lib.lib().rdb200_dev_fill_relax_from_f32(coarse_z.data_ptr(), coarse.data_ptr(), coarse.shape[1],
                                                                     coarse.shape[0]))
                solver.prolong(coarse, multigrid, row0)
            out = solver.finish()
            if return_stats:
                return out, rounds, _lib.stats()
            return out, rounds
    else:
        if g_top:
            local_dem[0].fill_(float("inf"))
        if g_bot:
            local_dem[h - 1].fill_(float("inf"))
        solver = solver_cls(local_dem)
    rounds = _relax_band(solver, g_top, g_bot, rank, world, group, max_rounds)
    out = solver.finish()
    if return_stats:
        from . import _lib
        return out, rounds, _lib.stats()
    return out, rounds


def fa_method_id(method: Optional[str], exponent: Optional[float], dinf: bool = False) -> Tuple[int, float]:
    """(method number of the band entry points, exponent) for a FlowAccumulation method name.  ``method=None`` keeps
    the ``dinf`` switch: D-infinity if set, else D8.  Names and errors are those of :func:`richdem_b200.FlowAccumulation`."""
    from . import _DINF_METHODS
    if method is None:
        return (1 if dinf else 0), 0.0
    if dinf and method not in _DINF_METHODS:
        raise ValueError(f'dinf=True contradicts method "{method}"')
    return _method_id(method, exponent, "FlowAccumulation")


def _method_id(method: Optional[str], exponent: Optional[float], what: str) -> Tuple[int, float]:
    """(method number, exponent) of a flow-metric name; the errors are those of :func:`richdem_b200.FlowAccumulation` or
    :func:`richdem_b200.FlowProportions` (``what``), whose names are the same."""
    from . import _D4_METHODS, _D8_METHODS, _DINF_METHODS, _EXPONENT_METHODS, _OUT_OF_SCOPE_METHODS
    if method in _D8_METHODS:
        return 0, 0.0
    if method in _DINF_METHODS:
        return 1, 0.0
    if method in _D4_METHODS:
        return 2, 0.0
    if method == "Quinn":
        return 3, 1.0
    if method in _EXPONENT_METHODS:
        if exponent is None:
            raise Exception(f'{what} method "{method}" requires an exponent!')
        return (3 if method == "Holmgren" else 4), float(exponent)
    if method in _OUT_OF_SCOPE_METHODS:
        raise Exception(f'{what} method "{method}" is outside the GPU hot path '
                        "(random-walk metric; use the reference CPU implementation)")
    raise Exception(f"Invalid {what} method. Valid methods are: " +
                    ", ".join(_DINF_METHODS + ("Quinn",) + _D8_METHODS + _D4_METHODS + _EXPONENT_METHODS +
                              _OUT_OF_SCOPE_METHODS))


class CudaBandAccumulator:
    """librichdem_b200's row-band accumulation entry points (rdb200_dev_facc_*).  ``method`` / ``exponent`` as in
    :func:`richdem_b200.FlowAccumulation`; without a method, ``dinf`` picks D-infinity or D8."""

    def __init__(self, local_dem, local_accum, nodata: float, g_top: int, g_bot: int, dinf: bool, ones: bool,
                 method: Optional[str] = None, exponent: Optional[float] = None):
        from . import _lib
        mid, xparam = fa_method_id(method, exponent, dinf)
        assert _on_device(local_dem) and local_dem.dtype == torch.float32 and local_dem.is_contiguous()
        assert _on_device(local_accum) and local_accum.dtype == torch.float64 and local_accum.is_contiguous()
        self._lib = _lib
        _lib.use_torch_stream()
        self.L = _lib.lib()
        self.h, self.w = local_dem.shape
        self.dev = local_dem.device
        self.dinf = mid == 1
        self._dem, self._accum = local_dem, local_accum  # the library reads the elevations again at the first run
        self._state = C.c_void_p()
        _lib.check(self.L.rdb200_dev_facc_begin_method(C.byref(self._state), local_dem.data_ptr(), local_accum.data_ptr(),
                                                       self.w, self.h, float(nodata), int(g_top), int(g_bot), mid,
                                                       xparam, int(ones)))

    def edge_codes(self, which: int):
        code = torch.empty(self.w, dtype=torch.uint8, device=self.dev)
        rmax = torch.zeros(self.w, dtype=torch.float32, device=self.dev)
        self._lib.check(self.L.rdb200_dev_facc_get_edge_codes(self._state, which, code.data_ptr(), rmax.data_ptr()))
        return [code, rmax]

    def set_ghost_codes(self, which: int, code, rmax):
        self._lib.check(self.L.rdb200_dev_facc_set_ghost_codes(self._state, which, code.data_ptr(), rmax.data_ptr()))

    def run(self):
        a, b = C.c_int32(0), C.c_int32(0)
        self._lib.check(self.L.rdb200_dev_facc_run(self._state, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def take_outflow(self, which: int):
        s = torch.empty(self.w, dtype=torch.float64, device=self.dev)
        c = torch.empty(self.w, dtype=torch.int32, device=self.dev)
        self._lib.check(self.L.rdb200_dev_facc_take_outflow(self._state, which, s.data_ptr(), c.data_ptr()))
        return [s, c]

    def apply_inflow(self, which: int, s, c):
        self._lib.check(self.L.rdb200_dev_facc_apply_inflow(self._state, which, s.data_ptr(), c.data_ptr()))

    def finish(self):
        self._lib.check(self.L.rdb200_dev_facc_finish(self._state))
        self._state = None


def fa_band(local_dem: "torch.Tensor", g_top: int, g_bot: int, nodata: float, dinf: bool = False,
            weights: Optional["torch.Tensor"] = None, rank_rows=None, group=None, max_rounds: int = 1000000,
            return_stats: bool = False, accumulator_cls=None, method: Optional[str] = None,
            exponent: Optional[float] = None):
    """FlowAccumulation over this rank's band.  ``local_dem`` is (g_top + owned + g_bot) x W and
    its ghost rows must already hold the neighbouring bands' elevations (``fill_band`` leaves them so;
    otherwise call :func:`exchange_rows`).  ``weights`` (float64, same local shape) defaults to ones.
    ``method`` / ``exponent`` as in :func:`richdem_b200.FlowAccumulation` (D8, Dinf, D4, Quinn, Holmgren, Freeman and
    their aliases); without a method, ``dinf`` picks FA_Tarboton or FA_D8.
    Returns (local accumulation incl. scratch ghost rows, exchange rounds[, stats]).  A float64 ``local_dem`` runs
    rdb200_mgpu_fa_method_f64_f64, which does not read its ghost rows."""
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    mid, xparam = fa_method_id(method, exponent, dinf)
    import os
    cxx = accumulator_cls is None and os.environ.get("RDB_BAND_DRIVER", "cxx") != "python"
    if _is_f64(local_dem) and not cxx:
        raise ValueError("fa_band: float64 bands run in the C++ band driver only; the Python band protocol "
                         "(accumulator_cls, RDB_BAND_DRIVER=python) takes float32")
    if cxx:
        _lib, fn, cm = _band_driver(local_dem, "fa_method_{}_f64", group)
        ones = weights is None
        acc = torch.empty(local_dem.shape, dtype=torch.float64, device=local_dem.device) if ones else weights
        assert _on_device(acc) and acc.dtype == torch.float64 and acc.is_contiguous()
        xr = C.c_int32(0)
        _lib.check(fn(cm.handle, local_dem.data_ptr(), acc.data_ptr(), local_dem.shape[1], local_dem.shape[0], float(nodata),
                      int(g_top), int(g_bot), mid, xparam, int(ones), C.byref(xr)))
        if return_stats:
            return acc, int(xr.value), _lib.stats()
        return acc, int(xr.value)
    accumulator_cls = accumulator_cls or CudaBandAccumulator
    ones = weights is None
    acc = torch.empty(local_dem.shape, dtype=torch.float64, device=local_dem.device) if ones else weights
    A = accumulator_cls(local_dem, acc, nodata, g_top, g_bot, dinf, ones, method=method, exponent=exponent)
    if world > 1:
        up = A.edge_codes(0) if g_top else None
        dn = A.edge_codes(1) if g_bot else None
        ru, rd = _neighbour_exchange(up, dn, g_top, g_bot, rank, group)
        if ru is not None:
            A.set_ghost_codes(0, ru[0], ru[1])
        if rd is not None:
            A.set_ghost_codes(1, rd[0], rd[1])
    rounds = 0
    while True:
        sent_t, sent_b = A.run()
        rounds += 1
        if world == 1:
            break
        flag = torch.tensor([1 if (sent_t + sent_b) > 0 else 0], dtype=torch.int32, device=local_dem.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=group)
        if int(flag.item()) == 0:
            break
        up = A.take_outflow(0) if g_top else None
        dn = A.take_outflow(1) if g_bot else None
        ru, rd = _neighbour_exchange(up, dn, g_top, g_bot, rank, group)
        if ru is not None:
            A.apply_inflow(0, ru[0], ru[1])
        if rd is not None:
            A.apply_inflow(1, rd[0], rd[1])
        if rounds >= max_rounds:
            raise RuntimeError("fa_band: exchange rounds exceeded max_rounds")
    A.finish()
    if return_stats:
        from . import _lib
        return acc, rounds, _lib.stats()
    return acc, rounds


def scatter_rows(full: Optional[np.ndarray], height: int, width: int, dtype, device, group=None):
    """Convenience for tests/bench: rank 0 holds ``full`` (H x W numpy); every rank receives its
    local raster (owned rows + ghost rows, ghost contents = neighbour's rows) as a tensor."""
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    r0, r1, gt, gb = local_rows(height, world, rank)
    if world == 1:
        return torch.as_tensor(np.ascontiguousarray(full), device=device).to(dtype).contiguous(), (r0, r1, gt, gb)
    local = torch.empty((r1 - r0 + gt + gb, width), dtype=dtype, device=device)
    if rank == 0:
        for g in range(1, world):
            a0, a1, at, ab = local_rows(height, world, g)
            dist.send(torch.as_tensor(np.ascontiguousarray(full[a0 - at:a1 + ab]), device=device).to(dtype), g, group)
        local.copy_(torch.as_tensor(np.ascontiguousarray(full[r0 - gt:r1 + gb]), device=device).to(dtype))
    else:
        dist.recv(local, 0, group)
    return local, (r0, r1, gt, gb)


# =================================================================================================
# Row-band flat resolution (ResolveFlatsEpsilon over bands)
# =================================================================================================
class _DevArray:
    """Zero-copy torch view of a device array owned by librichdem_b200 (via __cuda_array_interface__)."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2, "strides": None}


def _view(ptr, shape, typestr, device):
    return torch.as_tensor(_DevArray(ptr, shape, typestr), device=device)


class CudaFlatsBand:
    """Stepwise row-band flat resolution on one GPU (rdb200_dev_flats_*).  `local_dem` is the
    (g_top + owned + g_bot) x W float32 raster with the neighbours' rows in the ghost rows; the owned
    rows are modified in place by :meth:`apply`."""

    FT_FLAT, FT_LOW, FT_HIGH, FT_NODATA = 1, 2, 4, 8

    def __init__(self, local_dem, nodata: float, g_top: int, g_bot: int):
        from . import _lib
        assert _on_device(local_dem) and local_dem.dtype == torch.float32 and local_dem.is_contiguous()
        self._lib, self.L = _lib, _lib.lib()
        _lib.use_torch_stream()
        self.h, self.w = local_dem.shape
        self.gt, self.gb = int(g_top), int(g_bot)
        self.dev = local_dem.device
        self._dem = local_dem
        self._state = C.c_void_p()
        _lib.check(self.L.rdb200_dev_flats_begin(C.byref(self._state), local_dem.data_ptr(), self.w, self.h,
                                                 float(nodata), self.gt, self.gb))
        ptrs = (C.c_uint64 * 6)()
        _lib.check(self.L.rdb200_dev_flats_arrays(self._state, ptrs))
        n = self.h * self.w
        self.ft = _view(ptrs[0], (self.h, self.w), "|u1", self.dev)
        self.root = _view(ptrs[1], (self.h, self.w), "<i4", self.dev)    # later: labels
        self.rootflag = _view(ptrs[2], (n,), "|u1", self.dev)
        self.height = _view(ptrs[5], (n,), "<i4", self.dev)

    # rows that face a neighbour: (my edge row, my ghost row) per side
    def rows(self, which: int):
        return (self.gt, 0) if which == 0 else (self.h - 1 - self.gb, self.h - 1)

    def step(self, name: str):
        self._lib.check(getattr(self.L, "rdb200_dev_flats_" + name)(self._state))

    def gradient_begin(self, away: bool):
        st = C.c_void_p()
        self._lib.check(self.L.rdb200_dev_flats_gradient_begin(self._state, int(away), C.byref(st)))
        return _BandStateSolver(st, self.h, self.w, self.dev)

    def gradient_end(self, away: bool, solver: "_BandStateSolver"):
        self._lib.check(self.L.rdb200_dev_flats_gradient_end(self._state, int(away), solver._state))
        solver._state = None

    def finish(self):
        self._lib.check(self.L.rdb200_dev_flats_finish(self._state))
        self._state = None

    # ---- seam payloads (comm-agnostic; the step-wise reference of the seam kernels of csrc/flats.cu, used by the
    # one-device band emulation of the tests) ----
    def flag_payload(self, which: int):
        """uint8 rows [edge, ghost]: outlet flag of the component of every seam cell."""
        e, g = self.rows(which)
        f32 = self.rootflag
        return torch.stack([f32[self.root[e].long()], f32[self.root[g].long()]])

    def merge_flags(self, which: int, theirs) -> bool:
        """theirs = neighbour's flag_payload for the shared seam: their edge row is my ghost row and
        their ghost row is my edge row.  ORs their flags into my roots; True if anything changed."""
        e, g = self.rows(which)
        changed = False
        for my_row, their in ((g, theirs[0]), (e, theirs[1])):
            ok = (self.ft[my_row] & self.FT_NODATA) == 0
            idx = self.root[my_row].long()[ok]
            val = their[ok]
            before = self.rootflag[idx]
            need = (val != 0) & (before == 0)
            if bool(need.any()):
                self.rootflag[idx[need]] = 1
                changed = True
        return changed

    def height_payload(self, which: int):
        """int32 rows [edge, ghost]: flat height (max away level) of the flat of every seam cell (0: none)."""
        e, g = self.rows(which)
        out = []
        for r in (e, g):
            lab = self.root[r].long()      # holds labels now (root + 1, 0 = none)
            hv = self.height[(lab - 1).clamp(min=0)]
            out.append(torch.where(lab > 0, hv, torch.zeros_like(hv)))
        return torch.stack(out)

    def merge_heights(self, which: int, theirs) -> bool:
        e, g = self.rows(which)
        changed = False
        for my_row, their in ((g, theirs[0]), (e, theirs[1])):
            lab = self.root[my_row].long()
            ok = lab > 0
            if not bool(ok.any()):
                continue
            idx = (lab[ok] - 1)
            val = their[ok].to(torch.int32)
            before = self.height[idx]
            if bool((val > before).any()):
                self.height.scatter_reduce_(0, idx, val, reduce="amax", include_self=True)
                changed = True
        return changed


class _BandStateSolver:
    """An existing rdb200_fill_state (here: a band distance state) behind the band-solver interface."""

    def __init__(self, state, h, w, device):
        from . import _lib
        self._lib, self._state, self.h, self.w, self.device = _lib, state, h, w, device

    def run(self) -> int:
        ch = C.c_int32(0)
        self._lib.check(self._lib.lib().rdb200_dev_fill_run(self._state, C.byref(ch)))
        return int(ch.value)

    def read_row(self, y: int):
        row = torch.empty(self.w, dtype=torch.float32, device=self.device)
        self._lib.check(self._lib.lib().rdb200_dev_fill_read_row(self._state, y, row.data_ptr()))
        return row

    def update_row(self, y: int, row):
        self._lib.check(self._lib.lib().rdb200_dev_fill_update_row(self._state, y, row.contiguous().data_ptr()))


def _relax_band(solver, g_top, g_bot, rank, world, group, max_rounds=100000, stop_after=0):
    """The row-band relaxation protocol shared by the fill and the flat-resolution gradients.  ``stop_after`` = n > 0:
    return ``(rounds, done)`` after at most n solver runs (the caller does something -- a coarse-grid correction -- and
    calls again); otherwise run to the end and return the number of rounds."""
    h = solver.h
    rounds = 0
    while True:
        changed = solver.run()
        rounds += 1
        if world == 1:
            if changed & 4:
                if stop_after and rounds >= stop_after:
                    return rounds, False
                continue
            return (rounds, True) if stop_after else rounds
        my_change = 0
        if g_top and (changed & 1 or rounds == 1):
            my_change = 1
        if g_bot and (changed & 2 or rounds == 1):
            my_change = 1
        dev = getattr(solver, "device", "cpu")
        flag = torch.tensor([my_change, 1 if (changed & 4) else 0], dtype=torch.int32, device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=group)
        any_edge, any_active = (int(v) for v in flag.tolist())
        if not any_edge and not any_active:
            return (rounds, True) if stop_after else rounds
        if not any_edge:
            if stop_after and rounds >= stop_after:
                return rounds, False
            continue
        send_up = solver.read_row(1) if g_top else None
        send_dn = solver.read_row(h - 2) if g_bot else None
        recv_up, recv_dn = _neighbour_exchange(send_up, send_dn, g_top, g_bot, rank, group)
        if recv_up is not None:
            solver.update_row(0, recv_up[0])
        if recv_dn is not None:
            solver.update_row(h - 1, recv_dn[0])
        if rounds >= max_rounds:
            raise RuntimeError("band relaxation: exchange rounds exceeded max_rounds")
        if stop_after and rounds >= stop_after:
            return rounds, False


def resolve_flats_band(local_dem: "torch.Tensor", g_top: int, g_bot: int, nodata: float, group=None):
    """ResolveFlatsEpsilon over this rank's band, in place on the owned rows of ``local_dem`` (whose
    ghost rows must hold the neighbours' elevation rows; on return they hold the neighbours' resolved
    edge rows, so :func:`fa_band` can follow without :func:`exchange_rows`).  Collective.  Returns the
    number of seam iterations (flags + heights).  The protocol runs in C++ over the library's
    communicator (csrc/flats.cu: mgpu_resolve_flats_band).  A float64 band takes its increments as double ulps and
    its ghost rows are not read on entry."""
    _lib, fn, cm = _band_driver(local_dem, "resolve_flats_epsilon_{}", group)
    h, w = local_dem.shape
    it = C.c_int32(0)
    _lib.check(fn(cm.handle, local_dem.data_ptr(), w, h, float(nodata), int(g_top), int(g_bot), C.byref(it)))
    return int(it.value)


# =================================================================================================
# The direction-grid pipeline over row bands (FlowDirectionsD8Resolved -> D8FlowAccum)
# =================================================================================================
def d8_flow_directions_band(local_dem: "torch.Tensor", g_top: int, g_bot: int, nodata: float, alter: bool = False,
                            group=None):
    """FlowDirectionsD8Resolved over this rank's band.  ``local_dem`` is (g_top + owned + g_bot) x W and its ghost rows
    must hold the neighbours' elevation rows (:func:`fill_band` leaves them so).  ``alter=True`` raises the flat cells of
    the owned rows in place, as on one GPU.  Collective.  Returns (uint8 directions of the same local shape, whose ghost
    rows hold the neighbours' edge-row directions, seam iterations).  A float64 band takes its directions from the doubles
    and, with ``alter=True``, the reference's float steps (:func:`richdem_b200.f64.FlowDirectionsD8Resolved`)."""
    _lib, fn, cm = _band_driver(local_dem, "d8_flow_directions_flats_{}", group)
    h, w = local_dem.shape
    dirs = torch.empty((h, w), dtype=torch.uint8, device=local_dem.device)
    it = C.c_int32(0)
    _lib.check(fn(cm.handle, local_dem.data_ptr(), dirs.data_ptr(), w, h, float(nodata), int(g_top), int(g_bot),
                  int(bool(alter)), C.byref(it)))
    return dirs, int(it.value)


def d8_flow_accum_band(local_dirs: "torch.Tensor", g_top: int, g_bot: int, group=None):
    """D8FlowAccum over this rank's band of a uint8 direction grid, (g_top + owned + g_bot) x W.  Its ghost rows are not
    read (the edge rows are exchanged here).  Collective.  Returns (int32 upslope-cell counts of the same local shape,
    ghost rows scratch, exchange rounds)."""
    from . import _lib
    assert _on_device(local_dirs) and local_dirs.dtype == torch.uint8 and local_dirs.is_contiguous()
    _lib.use_torch_stream()
    h, w = local_dirs.shape
    area = torch.empty((h, w), dtype=torch.int32, device=local_dirs.device)
    xr = C.c_int32(0)
    cm = lib_comm(group, local_dirs.is_cuda)
    _lib.check(_lib.lib().rdb200_mgpu_d8_flow_accum_u8_i32(cm.handle, local_dirs.data_ptr(), area.data_ptr(), w, h, int(g_top),
                                                           int(g_bot), C.byref(xr)))
    return area, int(xr.value)


# =================================================================================================
# Flow proportions, accumulation from given proportions and terrain attributes over row bands
# =================================================================================================
def flow_proportions_band(local_dem: "torch.Tensor", g_top: int, g_bot: int, nodata: float, method: Optional[str] = None,
                          exponent: Optional[float] = None, group=None):
    """FlowProportions over this rank's band.  ``local_dem`` is (g_top + owned + g_bot) x W; its ghost rows are refreshed
    here with the neighbours' edge rows.  ``method`` / ``exponent`` and their errors are those of
    :func:`richdem_b200.FlowProportions`.  Collective.  Returns float32 proportions of shape (local rows, W, 9) whose owned
    rows are the single-GPU bits (ghost rows scratch)."""
    mid, xparam = _method_id(method, exponent, "FlowProportions")
    _lib, fn, cm = _band_driver(local_dem, "fm_method_{}", group)
    h, w = local_dem.shape
    props = torch.empty((h, w, 9), dtype=torch.float32, device=local_dem.device)
    _lib.check(fn(cm.handle, mid, local_dem.data_ptr(), props.data_ptr(), w, h, float(nodata), int(g_top), int(g_bot), xparam))
    return props


def flow_accum_from_props_band(local_props: "torch.Tensor", g_top: int, g_bot: int, weights: Optional["torch.Tensor"] = None,
                               group=None):
    """FlowAccumFromProps over this rank's band of float32 proportions, (g_top + owned + g_bot) x W x 9.  Their ghost rows
    are not trusted: they are overwritten with the neighbours' edge rows.  ``weights`` (float64, (local rows, W)) defaults
    to ones; when given it receives the accumulation in place.  NoData cells (slot 0 == -2) end as -1.  Collective.
    Returns (float64 accumulation of the local shape, ghost rows scratch, exchange rounds)."""
    from . import _lib
    if local_props.dim() != 3 or local_props.shape[2] != 9:
        raise RuntimeError("Array must have three dimensions with the last of size 9!")
    assert _on_device(local_props) and local_props.dtype == torch.float32 and local_props.is_contiguous()
    h, w = local_props.shape[0:2]
    if weights is None:
        acc = torch.ones((h, w), dtype=torch.float64, device=local_props.device)
    else:
        acc = weights
        assert _on_device(acc) and acc.dtype == torch.float64 and acc.is_contiguous()
        if tuple(acc.shape) != (h, w):
            raise RuntimeError("Accumulation array must have same dimensions as proportions array!")
    _lib.use_torch_stream()
    xr = C.c_int32(0)
    cm = lib_comm(group, local_props.is_cuda)
    _lib.check(_lib.lib().rdb200_mgpu_flow_accumulation_props_f64(cm.handle, local_props.data_ptr(), acc.data_ptr(), w, h,
                                                                  int(g_top), int(g_bot), C.byref(xr)))
    return acc, int(xr.value)


def terrain_attribute_band(local_dem: "torch.Tensor", g_top: int, g_bot: int, attrib: str, nodata: float,
                           zscale: float = 1.0, cell_x: float = 1.0, cell_y: float = 1.0, group=None):
    """TerrainAttribute over this rank's band.  ``local_dem`` is (g_top + owned + g_bot) x W; its ghost rows are refreshed
    here with the neighbours' edge rows.  ``attrib`` and its error are those of :func:`richdem_b200.TerrainAttribute`;
    ``cell_x`` / ``cell_y`` are the cell lengths, |geotransform[1]| and |geotransform[5]|.  Collective.  Returns the
    float32 attribute of the local shape, NoData -9999, whose owned rows are the single-GPU bits (ghost rows scratch)."""
    from . import _terrain_attrib_id
    aid = _terrain_attrib_id(attrib)
    _lib, fn, cm = _band_driver(local_dem, "terrain_attribute_{}", group)
    h, w = local_dem.shape
    out = torch.empty((h, w), dtype=torch.float32, device=local_dem.device)
    _lib.check(fn(cm.handle, aid, local_dem.data_ptr(), out.data_ptr(), w, h, float(nodata), -9999.0, float(zscale),
                  float(cell_x), float(cell_y), int(g_top), int(g_bot)))
    return out


# =================================================================================================
# The C++ band drivers by element type: float32 bands, and float64 bands, which run the float32 drivers on float keys
# every band shares (csrc/f64.cu: kappa_G) and the double flow metrics and attributes (csrc/f64_band.cu).  NoData is a
# double.
# =================================================================================================
def _is_f64(t) -> bool:
    return torch is not None and isinstance(t, torch.Tensor) and t.dtype == torch.float64


def _band_driver(local_dem, name: str, group):
    """(_lib, rdb200_mgpu_<name> with {} the band's element type f32 / f64, the library's communicator for ``group``),
    with the library on torch's current stream."""
    from . import _lib
    f64 = _is_f64(local_dem)
    assert _on_device(local_dem) and local_dem.dtype == (torch.float64 if f64 else torch.float32) and local_dem.is_contiguous()
    _lib.use_torch_stream()
    return _lib, getattr(_lib.lib(), "rdb200_mgpu_" + name.format("f64" if f64 else "f32")), lib_comm(group, local_dem.is_cuda)


def f64_order_keys_band(local_dem: "torch.Tensor", g_top: int, g_bot: int, nodata: float, group=None):
    """Diagnostic (not a stable interface): kappa_G, the float keys the float64 band drivers run the float32 engines on.
    Collective.  Returns (float32 keys of the local shape, whose ghost rows hold the neighbours' keys, kappa_G(nodata),
    True for global ranks / False for the cast to float)."""
    assert _is_f64(local_dem)
    _lib, fn, cm = _band_driver(local_dem, "f64_order_keys", group)
    h, w = local_dem.shape
    keys = torch.empty((h, w), dtype=torch.float32, device=local_dem.device)
    nd, ranked = C.c_float(0), C.c_int32(0)
    _lib.check(fn(cm.handle, local_dem.data_ptr(), keys.data_ptr(), w, h, float(nodata), int(g_top), int(g_bot), C.byref(nd),
                  C.byref(ranked)))
    return keys, float(nd.value), bool(ranked.value)
