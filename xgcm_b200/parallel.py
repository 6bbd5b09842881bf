"""Multi-GPU: one process per GPU (torch.distributed, NCCL over NVLink), sharding as the path allows.

The hot path shards naturally (SURVEY 8e): every operator acts along ONE of X / Y / Z, so any
other dimension — normally ``time`` — is a pure batch dimension.  The production layout is
therefore *contiguous blocks of time steps per rank with NO collective on the data path*
(``shard_bounds`` / ``shard_dataarray``); this is the reference's "broadcast-dim chunks" case
(docs/grid_ufuncs.md:341-376).

Only when the operated axis itself is sharded is there a real exchange step — the analogue of
the reference's ``dask.array.map_overlap(depth=1)`` (xgcm/grid_ufunc.py:1057-1133): each rank
sends ONE boundary plane to a neighbour and receives one (``exchange_halo``; NCCL send/recv over
NVLink on GPUs, gloo on CPU for tests), and the received plane enters the fused stencil kernel
through its ``halo_lo`` / ``halo_hi`` operands (``sharded_stencil2``).  Same restrictions as the
reference: no ``inner`` / ``outer`` outputs (grid_ufunc.py:1136-1159), no cumsum (grid.py:813-816).

Grids with ``face_connections`` (cubed sphere, LLC tiles) add a second natural decomposition: the
FACES.  ``sharded_connected_stencil2`` gives every rank a contiguous block of faces; the one-cell
rims that cross a block boundary — already rotated / flipped / sign-flipped by their owner with the
same signed-stride copies the single-GPU path uses — travel in one NCCL group, everything else is
the single-GPU fused stencil.
"""

from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous block ``[start, stop)`` of ``n`` items owned by ``rank`` (block size ceil(n/world))."""
    if world < 1 or not 0 <= rank < world:
        raise ValueError(f"bad rank/world: {rank}/{world}")
    block = -(-n // world)
    start = min(n, rank * block)
    return start, min(n, start + block)


def shard_dataarray(da, dim: str, rank: Optional[int] = None, world: Optional[int] = None):
    """This rank's contiguous block of ``da`` along ``dim`` (e.g. ``time``)."""
    rank = dist.get_rank() if rank is None else rank
    world = dist.get_world_size() if world is None else world
    start, stop = shard_bounds(da.sizes[dim], world, rank)
    return da.isel({dim: slice(start, stop)})


def _plane(x: torch.Tensor, axis: int, index: int) -> torch.Tensor:
    return x.select(axis, index).contiguous()


def exchange_halo(
    x: torch.Tensor,
    axis: int,
    lo: int,
    hi: int,
    periodic: bool,
    group=None,
    edge_scale_lo: Optional[torch.Tensor] = None,
    edge_scale_hi: Optional[torch.Tensor] = None,
) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """One ring step: returns ``(halo_lo, halo_hi)`` planes for this rank's shard of ``axis``.

    ``halo_lo`` (needed when ``lo``) is the previous rank's LAST plane, ``halo_hi`` (when ``hi``)
    the next rank's FIRST plane.  The ring closes only when ``periodic``; otherwise the edge
    ranks get ``None`` and synthesise the boundary locally (fill / extend in the kernel).
    ``edge_scale_*``: optional metric planes multiplied into the plane before sending (the halo
    must carry ``field * metric`` like the reference's padded array, grid.py:806-808).
    """
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    if world == 1:
        return None, None  # the kernel's own boundary handling covers the single-shard case
    prev_rank, next_rank = (rank - 1) % world, (rank + 1) % world
    has_prev = periodic or rank > 0
    has_next = periodic or rank < world - 1
    ops = []
    recv_lo = recv_hi = None
    keep = []
    if lo:
        # my last plane goes to the next rank; I receive the previous rank's last plane
        if has_next:
            send = _plane(x, axis, x.shape[axis] - 1)
            if edge_scale_hi is not None:
                send = _scale(send, edge_scale_hi)
            keep.append(send)
            ops.append(dist.P2POp(dist.isend, send, _global_rank(next_rank, group), group))
        if has_prev:
            recv_lo = torch.empty_like(_plane(x, axis, 0))
            ops.append(dist.P2POp(dist.irecv, recv_lo, _global_rank(prev_rank, group), group))
    if hi:
        if has_prev:
            send = _plane(x, axis, 0)
            if edge_scale_lo is not None:
                send = _scale(send, edge_scale_lo)
            keep.append(send)
            ops.append(dist.P2POp(dist.isend, send, _global_rank(prev_rank, group), group))
        if has_next:
            recv_hi = torch.empty_like(_plane(x, axis, 0))
            ops.append(dist.P2POp(dist.irecv, recv_hi, _global_rank(next_rank, group), group))
    if ops:
        for req in dist.batch_isend_irecv(ops):  # one ncclGroupStart/End on GPUs
            req.wait()
    return recv_lo, recv_hi


def _global_rank(group_rank: int, group) -> int:
    if group is None:
        return group_rank
    return dist.get_global_rank(group, group_rank)


def _scale(plane: torch.Tensor, metric_plane: torch.Tensor) -> torch.Tensor:
    if plane.is_cuda:
        from . import ops

        return ops.binary("mul", plane, metric_plane.to(plane.dtype), tuple(plane.shape))
    return plane * metric_plane  # CPU tensors only occur in the gloo plumbing tests


class Communicator:
    """The library's own NCCL communicator over the ranks of a torch.distributed group (``xg_comm_init``).

    torch.distributed is only the rendezvous: rank 0 draws the NCCL unique id inside the C library and
    broadcasts its 128 bytes; every rank then joins.  The exchange itself (``xg_halo_exchange`` /
    ``xg_stencil2_sharded``) never goes through Python or torch: pack kernel, one NCCL group on a side stream,
    the local block computed meanwhile, edge planes fixed up from the received halos."""

    def __init__(self, group=None):
        import ctypes as C

        from . import _capi

        if not torch.cuda.is_available():
            raise RuntimeError("xgcm_b200.parallel.Communicator needs CUDA devices (NCCL)")
        self._lib = _capi.load()
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self._ws = None
        try:  # name the NCCL torch ships, so both users share one copy of the library
            import nvidia.nccl as _n  # type: ignore
            import os

            cand = os.path.join(os.path.dirname(_n.__file__), "lib", "libnccl.so.2")
            if os.path.exists(cand):
                self._lib.xg_nccl_load(cand.encode())
        except Exception:
            pass
        ident = (C.c_ubyte * 128)()
        if self.rank == 0:
            _capi.check(self._lib.xg_comm_unique_id(ident))
        payload = [bytes(ident)]
        dist.broadcast_object_list(payload, src=_global_rank(0, group), group=group)
        ident = (C.c_ubyte * 128).from_buffer_copy(payload[0])
        handle = C.c_void_p()
        with torch.cuda.device(torch.cuda.current_device()):
            _capi.check(self._lib.xg_comm_init(ident, self.world, self.rank, C.byref(handle)))
        self._handle = handle

    def close(self):
        if getattr(self, "_handle", None):
            self._lib.xg_comm_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _workspace(self, plane_bytes: int, device) -> torch.Tensor:
        need = 4 * ((plane_bytes + 255) // 256 * 256)
        if self._ws is None or self._ws.numel() < need or self._ws.device != device:
            self._ws = torch.empty(max(need, 256), dtype=torch.uint8, device=device)
        return self._ws

    def stencil2(self, x_local: torch.Tensor, axis: int, op: str, lo: int, hi: int, padding: Optional[str],
                 fill_value: float = 0.0, pre: Optional[torch.Tensor] = None,
                 post: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``xg_stencil2_sharded``: see :func:`sharded_stencil2`."""
        from . import _capi, ops

        if lo + hi != 1:
            raise NotImplementedError(
                "a sharded operated axis supports only length-preserving shifts (center<->left/right), "
                "like map_overlap in the reference"
            )
        if padding not in ("periodic", "fill", "extend"):
            raise ValueError(f"padding must be one of ['periodic', 'fill', 'extend'], but got {padding}")
        x = x_local.contiguous()
        axis = axis % x.dim()
        shape = list(x.shape)
        out = torch.empty_like(x)
        keep_pre, pre_ptr, pre_st = ops._operand(pre, shape, x, "pre metric")
        keep_post, post_ptr, post_st = ops._operand(post, shape, x, "post metric")
        plane = x.numel() // max(shape[axis], 1) * x.element_size()
        ws = self._workspace(plane, x.device)
        with torch.cuda.device(x.device):
            rc = self._lib.xg_stencil2_sharded(
                self._handle, _capi.OPS[op], ops._dtype_code(x), x.data_ptr(), out.data_ptr(), x.dim(),
                _capi.i64_array(shape), axis, lo, hi, _capi.BCS[padding], float(fill_value), pre_ptr, pre_st,
                post_ptr, post_st, ws.data_ptr(), ws.numel(), ops._stream_ptr(x))
        _capi.check(rc)
        return out


def sharded_stencil2(
    x_local: torch.Tensor,
    axis: int,
    op: str,
    lo: int,
    hi: int,
    padding: Optional[str],
    fill_value: float = 0.0,
    pre: Optional[torch.Tensor] = None,
    post: Optional[torch.Tensor] = None,
    group=None,
    comm: Optional["Communicator"] = None,
) -> torch.Tensor:
    """``xg_stencil2`` on a field whose operated ``axis`` is split across the ranks of ``group``
    (contiguous blocks, rank order = axis order).  ``pre`` / ``post`` are the LOCAL shards of the
    metrics.  One plane per neighbour crosses NVLink; everything else is the single-GPU kernel.

    With ``comm`` (a :class:`Communicator`) the whole step is ONE C call, ``xg_stencil2_sharded``: planes
    packed by a kernel, exchanged in one NCCL group on a side stream while the local block is computed.
    Without it the exchange goes through torch.distributed (any backend; the gloo CPU tests use this)."""
    from . import ops

    if comm is not None:
        return comm.stencil2(x_local, axis, op, lo, hi, padding, fill_value, pre=pre, post=post)

    if lo + hi != 1:
        # grid_ufunc.py:1136-1159: shifting to inner/outer would change the chunk length
        raise NotImplementedError(
            "a sharded operated axis supports only length-preserving shifts (center<->left/right), "
            "like map_overlap in the reference"
        )
    axis = axis % x_local.dim()
    scale_lo = scale_hi = None
    if pre is not None:
        pre_b = pre.expand(x_local.shape) if pre.dim() == x_local.dim() else pre
        scale_lo = pre_b.select(axis, 0)
        scale_hi = pre_b.select(axis, x_local.shape[axis] - 1)
    halo_lo, halo_hi = exchange_halo(
        x_local, axis, lo, hi, padding == "periodic", group, edge_scale_lo=scale_lo, edge_scale_hi=scale_hi
    )
    return ops.stencil2(x_local, axis, op, lo, hi, padding, fill_value, pre=pre, post=post,
                        halo_lo=halo_lo, halo_hi=halo_hi)


def sharded_connected_stencil2(grid, da_local, ax_name: str, op: str, lo: int, hi: int, padding=None,
                               fill_value=None, other_component_local=None, post: Optional[torch.Tensor] = None,
                               group=None) -> torch.Tensor:
    """``diff / interp / min / max`` along ``ax_name`` of a field on a grid with face connections
    whose FACES are split across the ranks of ``group``.

    ``grid``: the GLOBAL topology (``Grid(ds, face_connections=...)`` — only dims and links are
    used, so ``ds`` may hold coordinates only).  ``da_local`` (and ``other_component_local`` for a
    vector component, as ``{axis: DataArray}`` like ``Grid.diff``): this rank's contiguous block of
    faces, ``shard_bounds(n_faces, world, rank)`` along the face dim.  Returns the local block of
    the result as a tensor.  Rims whose neighbour face lives on another rank are produced BY THE
    OWNER of that face (slice / swap / flip / negate: ``padding._copy_connected_edge``) and sent
    as thin contiguous slabs; sends and receives of all edges form one ``batch_isend_irecv``.
    """
    from . import ops
    from . import padding as P

    if lo > 1 or hi > 1 or lo + hi == 0:
        raise NotImplementedError("face-sharded operators take one halo cell (center <-> left / right / outer)")
    facedim = grid._facedim
    if facedim is None:
        raise ValueError("the grid has no face connections")
    face_links = grid._face_connections[facedim]
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    n_global = grid._ds.sizes[facedim]
    block = -(-n_global // world)
    start, stop = shard_bounds(n_global, world, rank)
    raw = da_local
    field, isvector, vectoraxis, partner = P._unpack_vector(grid, raw, other_component_local)
    if field.sizes[facedim] != stop - start:
        raise ValueError(
            f"rank {rank} must hold faces [{start}, {stop}) along {facedim!r}, got {field.sizes[facedim]}"
        )
    remote: list = []
    x, halo_lo, halo_hi, _, dims = P.connected_halo_planes(
        raw, grid, ax_name, lo, hi, padding, fill_value, other_component_local,
        face_offset=start, remote_edges=remote)
    planes = (halo_lo, halo_hi)

    # what this rank's faces owe to other ranks: the same enumeration on every rank (global face
    # order, then side) so that sends and receives pair up
    shape = [int(v) for v in x.shape]
    sources = P._connection_sources(field, partner, x)
    fpos = dims.index(facedim)
    tpos = dims.index(P._axis_dim(grid, dims, ax_name))
    slab_shape = list(shape)
    slab_shape[fpos] = 1
    slab_shape[tpos] = 1
    p2p, recvs, keep, batch = [], [], [], []
    for f in range(n_global):
        for side, w in ((0, lo), (1, hi)):
            connection = face_links.get(f, {}).get(ax_name, (None, None))[side] if w else None
            if not connection:
                continue
            owner_f, owner_s = f // block, connection[0] // block
            if owner_f == owner_s:
                continue
            if owner_s == rank:  # I own the neighbour face: build the finished rim and send it
                slab = torch.empty(slab_shape, dtype=x.dtype, device=x.device)
                P._copy_connected_edge(grid, facedim, slab, dims, slab_shape, 0, ax_name, 0, 1, 0,
                                       (connection[0] - start,) + tuple(connection[1:]), bool(side),
                                       sources, isvector, vectoraxis, batch)
                keep.append(slab)
                p2p.append(dist.P2POp(dist.isend, slab, _global_rank(owner_f, group), group))
            elif owner_f == rank:
                buf = torch.empty(slab_shape, dtype=x.dtype, device=x.device)
                recvs.append((side, f - start, buf))
                p2p.append(dist.P2POp(dist.irecv, buf, _global_rank(owner_s, group), group))
    ops.strided_copy_batch(batch)  # all outgoing rims: one launch, before they are sent
    if p2p:
        for req in dist.batch_isend_irecv(p2p):
            req.wait()
    assert sorted((s_, i_) for s_, i_, _ in recvs) == sorted((s_, i_) for s_, i_, _ in remote)
    p_shape = list(shape)
    p_shape[tpos] = 1
    p_strides = P._contiguous_strides(p_shape)
    s_strides = P._contiguous_strides(slab_shape)
    ops.strided_copy_batch([
        (planes[side], i * p_strides[fpos], p_strides, buf, 0, s_strides, slab_shape, False)
        for side, i, buf in recvs
    ])
    return ops.stencil2(x, tpos, op, lo, hi, "fill", 0.0, post=post, halo_lo=halo_lo, halo_hi=halo_hi)
