"""Array-level operators: torch CUDA tensors in/out, numerics in libxgcm_b200.so.

torch is plumbing only (device allocation, streams); every value is produced by
a hand-written sm_90a kernel reached through the C-ABI (``include/xgcm_b200.h``).
There is no CPU path: a non-CUDA tensor raises.
"""

from __future__ import annotations

from typing import Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _capi
from .device import host_device_arg

# the `device` of the *_host functions: None (the current CUDA device), an index, or a sequence of indices, a host
# device group that spreads the call's slabs over those GPUs (device.host_group)
HostDevice = Optional[Union[int, Sequence[int]]]

_TORCH_DTYPE_CODE = {torch.float32: _capi.XG_F32, torch.float64: _capi.XG_F64}


def _require_cuda(t: torch.Tensor, what: str) -> None:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a torch.Tensor, got {type(t)}")
    if not t.is_cuda:
        raise RuntimeError(
            f"{what} lives on {t.device}; xgcm_b200 kernels run on CUDA devices only "
            "(there is no CPU fallback)"
        )


def _dtype_code(t: torch.Tensor) -> int:
    try:
        return _TORCH_DTYPE_CODE[t.dtype]
    except KeyError:
        raise TypeError(f"xgcm_b200 kernels support float32/float64 fields, got {t.dtype}")


def _stream_ptr(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _norm_axis(axis: int, ndim: int) -> int:
    if not -ndim <= axis < ndim:
        raise ValueError(f"axis {axis} out of range for {ndim}-d field")
    return axis % ndim


def _check_padding(padding) -> None:
    if padding not in _capi.BCS:
        raise ValueError(f"padding must be one of ['periodic', 'fill', 'extend'] or None, but got {padding}")


def _stencil_specs(specs, ndim: int, fused: bool):
    """C-ABI values of stencil ``specs`` ``[(axis, op, lo, hi, padding, fill), ...]``: lists of axes, op codes, lo,
    hi, boundary codes and fills.  ``fused`` (one multi-axis launch): the boundary of a padded axis is periodic,
    fill or extend (NotImplementedError for another, ValueError for none) and each axis appears once."""
    axes, opc, los, his, bcs, fills = [], [], [], [], [], []
    for axis, op, lo, hi, padding, fill in specs:
        axes.append(_norm_axis(axis, ndim))
        if op not in _capi.OPS:
            raise ValueError(f"unknown op {op!r}")
        if fused and padding not in ("periodic", "fill", "extend", None):
            raise NotImplementedError(f"fused multi-axis stencils support periodic / fill / extend, not {padding!r}")
        if fused and (lo or hi) and padding is None:
            raise ValueError("no boundary condition was specified but the operation needs to pad the axis")
        _check_padding(padding)
        opc.append(_capi.OPS[op])
        los.append(int(lo))
        his.append(int(hi))
        bcs.append(_capi.BCS[padding] if (lo or hi) else 0)
        fills.append(float(0.0 if fill is None else fill))
    if fused and len(set(axes)) != len(axes):
        raise ValueError("each axis may appear only once")
    return axes, opc, los, his, bcs, fills


def _bins_order(diffs) -> int:
    """``flip`` of monotonic target bins with steps ``diffs``: 1 when they decrease, 0 when they increase
    (transform.py:167-176)."""
    if bool((diffs < 0).all()):
        return 1
    if bool((diffs > 0).all()):
        return 0
    raise ValueError("Target values are not monotonic")


def _operand(m: Optional[torch.Tensor], shape: Sequence[int], like: torch.Tensor, what: str):
    """Return (keepalive tensor, data_ptr, int64[ndim] strides) for a broadcast operand."""
    if m is None:
        return None, None, None
    _require_cuda(m, what)
    if m.dtype != like.dtype:
        m = m.to(like.dtype)
    if m.device != like.device:
        raise RuntimeError(f"{what} is on {m.device}, field on {like.device}")
    try:
        mb = m.expand(tuple(shape))
    except RuntimeError as err:
        raise ValueError(f"{what} of shape {tuple(m.shape)} does not broadcast to {tuple(shape)}") from err
    strides = [0 if s == 1 else st for s, st in zip(shape, mb.stride())]
    if any(st < 0 for st in strides):
        mb = m.contiguous().expand(tuple(shape))
        strides = [0 if s == 1 else st for s, st in zip(shape, mb.stride())]
    return mb, mb.data_ptr(), _capi.i64_array(strides)


def stencil2(
    x: torch.Tensor,
    axis: int,
    op: str,
    lo: int,
    hi: int,
    padding: Optional[str],
    fill_value: float = 0.0,
    pre: Optional[torch.Tensor] = None,
    post: Optional[torch.Tensor] = None,
    halo_lo: Optional[torch.Tensor] = None,
    halo_hi: Optional[torch.Tensor] = None,
    out: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """Fused pad + {diff, interp, min, max} (+ metric) along ``axis``.

    Mirrors padding.py:575-616 + gridops.py:23-24,76-77,123-126,172-175 +
    grid.py:806-808,830-832 of the reference in one HBM pass.
    """
    lib = _capi.load()
    _require_cuda(x, "field")
    if op not in _capi.OPS:
        raise ValueError(f"unknown op {op!r}")
    _check_padding(padding)
    x = x.contiguous()
    axis = _norm_axis(axis, x.dim())
    shape = list(x.shape)
    out_shape = list(shape)
    out_shape[axis] = shape[axis] + lo + hi - 1
    if out_shape[axis] < 0:
        raise ValueError("operated axis too short")
    if out is None:
        out = torch.empty(out_shape, dtype=x.dtype, device=x.device)
    else:
        if list(out.shape) != out_shape or out.dtype != x.dtype or not out.is_contiguous():
            raise ValueError("out has wrong shape/dtype/layout")
    keep_pre, pre_ptr, pre_st = _operand(pre, shape, x, "pre metric")
    keep_post, post_ptr, post_st = _operand(post, out_shape, x, "post metric")
    plane = [s for d, s in enumerate(shape) if d != axis]
    hl = hh = None
    if halo_lo is not None:
        _require_cuda(halo_lo, "halo_lo")
        hl = halo_lo.to(x.dtype).contiguous()
        if hl.numel() != int(np.prod(plane, dtype=np.int64)):
            raise ValueError("halo_lo has wrong size")
    if halo_hi is not None:
        _require_cuda(halo_hi, "halo_hi")
        hh = halo_hi.to(x.dtype).contiguous()
        if hh.numel() != int(np.prod(plane, dtype=np.int64)):
            raise ValueError("halo_hi has wrong size")
    with torch.cuda.device(x.device):
        rc = lib.xg_stencil2(
            _capi.OPS[op], _dtype_code(x), x.data_ptr(), out.data_ptr(), x.dim(),
            _capi.i64_array(shape), axis, lo, hi, _capi.BCS[padding], float(fill_value),
            pre_ptr, pre_st, post_ptr, post_st,
            hl.data_ptr() if hl is not None else None,
            hh.data_ptr() if hh is not None else None,
            _stream_ptr(x),
        )
    _capi.check(rc)
    return out


def stencil_multi(x: torch.Tensor, specs: Sequence[Tuple[int, str, int, int, Optional[str], float]], *,
                  pre: Optional[Sequence[Optional[torch.Tensor]]] = None,
                  post: Optional[Sequence[Optional[torch.Tensor]]] = None) -> torch.Tensor:
    """Fused chain of 2 or 3 single-axis stencils: ``specs`` = [(axis, op, lo, hi, padding, fill), ...]
    in application order.  Bit-identical to the corresponding sequence of :func:`stencil2` calls,
    with one read and one write of the field (reference: one full pass per axis, grid.py:798-832).

    ``pre`` / ``post``: per stage, a metric that broadcasts against the stage's input / output (or None), as
    :func:`stencil2` takes them (``metric_weighted``); the chain then runs ``xg_stencil_multi_weighted``, still one
    launch.  NotImplementedError for a layout the weighted kernel does not address (two or more non-operated dims
    after the last operated one)."""
    import ctypes as C

    lib = _capi.load()
    _require_cuda(x, "field")
    if not 2 <= len(specs) <= 3:
        raise ValueError("stencil_multi fuses 2 or 3 axes")
    x = x.contiguous()
    shape = list(x.shape)
    axes, opc, los, his, bcs, fills = _stencil_specs(specs, x.dim(), fused=True)
    out_shape = _multi_out_shape(shape, axes, los, his)
    pre, post = _stage_list(pre, len(specs), "pre"), _stage_list(post, len(specs), "post")
    if len(set(opc)) != 1:
        # mixed operators: not a Grid-level case; same result through the per-axis kernel
        out = x
        for k, (axis, op, lo, hi, padding, fill) in enumerate(specs):
            out = stencil2(out, axis, op, lo, hi, padding if (lo or hi) else None, fill, pre=pre[k], post=post[k])
        return out
    out = torch.empty(out_shape, dtype=x.dtype, device=x.device)
    n = len(specs)
    IntArr, DblArr = C.c_int * n, C.c_double * n
    weighted = any(m is not None for m in pre + post)
    if weighted:
        keep, met_args = [], []
        for mets, shapes, what in ((pre, _stage_shapes(shape, axes, los, his, 0), "pre"),
                                   (post, _stage_shapes(shape, axes, los, his, 1), "post")):
            ptrs, strides = (C.c_void_p * n)(), []
            for k, (m, s) in enumerate(zip(mets, shapes)):
                mb, ptr, st = _operand(m, s, x, f"{what} metric of stage {k}")
                keep.append(mb)
                ptrs[k] = ptr
                strides += list(st) if st is not None else [0] * len(shape)
            met_args += [ptrs, _capi.i64_array(strides)]
    if out.numel():
        args = (_dtype_code(x), x.data_ptr(), out.data_ptr(), x.dim(), _capi.i64_array(shape), n,
                IntArr(*axes), IntArr(*opc), IntArr(*los), IntArr(*his), IntArr(*bcs), DblArr(*fills))
        with torch.cuda.device(x.device):
            if weighted:
                rc = lib.xg_stencil_multi_weighted(*args, *met_args, _stream_ptr(x))
            else:
                rc = lib.xg_stencil_multi(*args, _stream_ptr(x))
        _capi.check(rc)
    return out


def _stage_list(mets, n, what):
    """``pre`` / ``post`` of a fused chain as a list of one entry (a metric or None) per stage."""
    if mets is None:
        return [None] * n
    mets = list(mets)
    if len(mets) != n:
        raise ValueError(f"{what}: one metric (or None) per stage, got {len(mets)} for {n} stages")
    return mets


def _stage_shapes(shape, axes, los, his, after):
    """Shape of each stage's input (after=0) or output (after=1) of a fused chain."""
    out, cur = [], list(shape)
    for axis, lo, hi in zip(axes, los, his):
        nxt = list(cur)
        nxt[axis] = cur[axis] + lo + hi - 1
        out.append(nxt if after else cur)
        cur = nxt
    return out


def _multi_out_shape(shape, axes, los, his):
    out_shape = list(shape)
    for axis, lo, hi in zip(axes, los, his):
        out_shape[axis] = shape[axis] + lo + hi - 1
    return out_shape


def pad(x: torch.Tensor, axis: int, lo: int, hi: int, padding: Optional[str],
        fill_value: float = 0.0) -> torch.Tensor:
    """The padded array itself (padding.py:575-616), one axis."""
    lib = _capi.load()
    _require_cuda(x, "field")
    _check_padding(padding)
    x = x.contiguous()
    axis = _norm_axis(axis, x.dim())
    shape = list(x.shape)
    out_shape = list(shape)
    out_shape[axis] = shape[axis] + lo + hi
    out = torch.empty(out_shape, dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        rc = lib.xg_pad(_dtype_code(x), x.data_ptr(), out.data_ptr(), x.dim(),
                        _capi.i64_array(shape), axis, lo, hi, _capi.BCS[padding],
                        float(fill_value), _stream_ptr(x))
    _capi.check(rc)
    return out


def fold_rows(x: torch.Tensor, fold_axis: int, seam_axis: int, width: int, skip: int, mirror: int,
              period: int, negate: bool = False, pre: Optional[torch.Tensor] = None,
              out: Optional[torch.Tensor] = None, row0: int = 0) -> torch.Tensor:
    """North-fold halo rows (xg_fold_rows): ``out[..., row0 + r, ..., k, ...] = +-(x * pre)[..., n-1-skip-r, ...,
    (mirror - k) mod period, ...]`` for ``r < width`` along ``fold_axis`` and every ``k`` along ``seam_axis``.

    Without ``out`` the result holds just the ``width`` rows (``width = 1``: the halo plane of
    :func:`stencil2`); with ``out`` (contiguous, ``x``'s shape but any length along ``fold_axis``) the rows
    land at ``row0`` of it."""
    lib = _capi.load()
    _require_cuda(x, "field")
    x = x.contiguous()
    fold_axis = _norm_axis(fold_axis, x.dim())
    seam_axis = _norm_axis(seam_axis, x.dim())
    shape = list(x.shape)
    if out is None:
        out_shape = list(shape)
        out_shape[fold_axis] = int(width)
        out = torch.empty(out_shape, dtype=x.dtype, device=x.device)
    else:
        _require_cuda(out, "out")
        same = [s for d, s in enumerate(out.shape) if d != fold_axis] == [s for d, s in enumerate(shape) if d != fold_axis]
        if out.dim() != x.dim() or not same or out.dtype != x.dtype or not out.is_contiguous():
            raise ValueError("out has wrong shape/dtype/layout")
    keep_pre, pre_ptr, pre_st = _operand(pre, shape, x, "pre metric")
    with torch.cuda.device(x.device):
        rc = lib.xg_fold_rows(_dtype_code(x), x.data_ptr(), out.data_ptr(), x.dim(), _capi.i64_array(shape),
                              fold_axis, seam_axis, int(out.shape[fold_axis]), int(row0), int(width), int(skip),
                              int(mirror), int(period), 1 if negate else 0, pre_ptr, pre_st, _stream_ptr(x))
    _capi.check(rc)
    return out


def strided_copy(dst: torch.Tensor, dst_offset: int, dst_strides: Sequence[int],
                 src: torch.Tensor, src_offset: int, src_strides: Sequence[int],
                 shape: Sequence[int], negate: bool = False) -> None:
    """``dst.flat[dst_offset + i . dst_strides] = +-src.flat[src_offset + i . src_strides]`` for all
    index tuples ``i`` in ``shape`` (xg_strided_copy).  Offsets and strides are in elements of the
    contiguous base tensors; source strides may be negative (flips) or permuted (dim swaps), which
    is how one connected face edge is written (padding.py:414-541)."""
    lib = _capi.load()
    _require_cuda(dst, "dst")
    _require_cuda(src, "src")
    if dst.dtype != src.dtype:
        raise TypeError(f"strided_copy: dtype mismatch {dst.dtype} vs {src.dtype}")
    if not (dst.is_contiguous() and src.is_contiguous()):
        raise ValueError("strided_copy: base tensors must be contiguous")
    shape = [int(v) for v in shape]
    if len(shape) != len(dst_strides) or len(shape) != len(src_strides):
        raise ValueError("strided_copy: shape / strides rank mismatch")
    if any(v == 0 for v in shape):
        return
    # bounds of both index maps (the kernel trusts them)
    for name, t, off, strides in (("dst", dst, dst_offset, dst_strides), ("src", src, src_offset, src_strides)):
        lo = off + sum(min(0, (n - 1) * int(st)) for n, st in zip(shape, strides))
        hi = off + sum(max(0, (n - 1) * int(st)) for n, st in zip(shape, strides))
        if lo < 0 or hi >= t.numel():
            raise IndexError(f"strided_copy: {name} index map leaves the tensor ([{lo}, {hi}] of {t.numel()})")
    es = dst.element_size()
    with torch.cuda.device(dst.device):
        rc = lib.xg_strided_copy(_dtype_code(dst), dst.data_ptr() + int(dst_offset) * es,
                                 _capi.i64_array([int(v) for v in dst_strides]),
                                 src.data_ptr() + int(src_offset) * es,
                                 _capi.i64_array([int(v) for v in src_strides]),
                                 len(shape), _capi.i64_array(shape), 1 if negate else 0,
                                 _stream_ptr(dst))
    _capi.check(rc)


def strided_copy_batch(copies: Sequence[tuple]) -> None:
    """Several :func:`strided_copy` calls — tuples ``(dst, dst_offset, dst_strides, src, src_offset,
    src_strides, shape, negate)`` of one rank and dtype — in ONE launch (xg_strided_copy_batch):
    all connected edges of a field at once.  Falls back to one launch per copy when an index map
    does not collapse to 5 dims."""
    import ctypes as C

    copies = [c for c in copies if all(int(n) > 0 for n in c[6])]
    if not copies:
        return
    if len(copies) == 1:
        return strided_copy(*copies[0])
    lib = _capi.load()
    first = copies[0][0]
    ndim = len(copies[0][6])
    es = first.element_size()
    dptr, sptr, shapes, dstr, sstr, neg, keep = [], [], [], [], [], [], []
    for dst, doff, dstrides, src, soff, sstrides, shape, negate in copies:
        _require_cuda(dst, "dst")
        _require_cuda(src, "src")
        if dst.dtype != first.dtype or src.dtype != first.dtype or dst.device != first.device:
            raise TypeError("strided_copy_batch: all tensors must share dtype and device")
        if not (dst.is_contiguous() and src.is_contiguous()) or len(shape) != ndim:
            raise ValueError("strided_copy_batch: contiguous base tensors and one common rank are required")
        for name, t, off, strides in (("dst", dst, doff, dstrides), ("src", src, soff, sstrides)):
            lo = off + sum(min(0, (int(n) - 1) * int(st)) for n, st in zip(shape, strides))
            hi = off + sum(max(0, (int(n) - 1) * int(st)) for n, st in zip(shape, strides))
            if lo < 0 or hi >= t.numel():
                raise IndexError(f"strided_copy_batch: {name} index map leaves the tensor ([{lo}, {hi}] of {t.numel()})")
        dptr.append(dst.data_ptr() + int(doff) * es)
        sptr.append(src.data_ptr() + int(soff) * es)
        shapes += [int(v) for v in shape]
        dstr += [int(v) for v in dstrides]
        sstr += [int(v) for v in sstrides]
        neg.append(1 if negate else 0)
        keep += [dst, src]
    n = len(copies)
    with torch.cuda.device(first.device):
        rc = lib.xg_strided_copy_batch(
            _dtype_code(first), n, (C.c_void_p * n)(*dptr), (C.c_void_p * n)(*sptr), ndim,
            _capi.i64_array(shapes), _capi.i64_array(dstr), _capi.i64_array(sstr), (C.c_int * n)(*neg),
            _stream_ptr(first))
    if rc == -2:  # XG_ENOTIMPL: an edge with more than 5 collapsed dims
        for c in copies:
            strided_copy(*c)
        return
    _capi.check(rc)


def binary(opname: str, a: torch.Tensor, b: torch.Tensor, shape: Optional[Sequence[int]] = None) -> torch.Tensor:
    """``a (op) b`` with numpy-style broadcasting, on the device (xg_binary).

    The kernel broadcasts ``b`` against ``a``; when ``a`` itself has to be
    broadcast it is expanded first (only happens for metric x metric products).
    """
    lib = _capi.load()
    _require_cuda(a, "a")
    _require_cuda(b, "b")
    if opname not in _capi.BINOPS:
        raise ValueError(f"unknown binary op {opname!r}")
    dt = torch.promote_types(a.dtype, b.dtype)
    if dt not in (torch.float32, torch.float64):
        dt = torch.float64
    a = a.to(dt)
    b = b.to(dt)
    if shape is None:
        shape = torch.broadcast_shapes(a.shape, b.shape)
    shape = tuple(int(s) for s in shape)
    if len(shape) == 0:
        a = a.reshape(1)
        b = b.reshape(1)
        shape = (1,)
        scalar = True
    else:
        scalar = False
    a_full = a.expand(shape).contiguous()
    keep, b_ptr, b_st = _operand(b, shape, a_full, "b")
    out = torch.empty(shape, dtype=dt, device=a.device)
    if out.numel():
        with torch.cuda.device(a.device):
            rc = lib.xg_binary(_capi.BINOPS[opname], _dtype_code(a_full), a_full.data_ptr(), b_ptr,
                               b_st, out.data_ptr(), len(shape), _capi.i64_array(shape),
                               _stream_ptr(a_full))
        _capi.check(rc)
    return out.reshape(()) if scalar else out


def cumscan(
    x: torch.Tensor,
    axis: int,
    reverse: bool = False,
    trim: str = "none",
    pad_lo: int = 0,
    pad_hi: int = 0,
    padding: Optional[str] = None,
    fill_value: float = 0.0,
    pre: Optional[torch.Tensor] = None,
    post: Optional[torch.Tensor] = None,
    skipna: bool = True,
) -> torch.Tensor:
    """Cumulative sum with xgcm's trim / pad table fused (grid.py:1306-1414)."""
    lib = _capi.load()
    _require_cuda(x, "field")
    _check_padding(padding)
    x = x.contiguous()
    axis = _norm_axis(axis, x.dim())
    shape = list(x.shape)
    kept = shape[axis] - (0 if trim == "none" else 1)
    if kept < 0:
        raise ValueError("operated axis too short to trim")
    out_shape = list(shape)
    out_shape[axis] = kept + pad_lo + pad_hi
    out = torch.empty(out_shape, dtype=x.dtype, device=x.device)
    keep_pre, pre_ptr, pre_st = _operand(pre, shape, x, "pre metric")
    keep_post, post_ptr, post_st = _operand(post, out_shape, x, "post metric")
    with torch.cuda.device(x.device):
        rc = lib.xg_cumscan(
            _dtype_code(x), x.data_ptr(), out.data_ptr(), x.dim(), _capi.i64_array(shape), axis,
            int(bool(reverse)), _capi.TRIMS[trim], pad_lo, pad_hi, _capi.BCS[padding],
            float(fill_value), pre_ptr, pre_st, post_ptr, post_st, int(bool(skipna)),
            _stream_ptr(x),
        )
    _capi.check(rc)
    return out


def wreduce(x: torch.Tensor, axis: int, weight: Optional[torch.Tensor] = None, mode: str = "sum",
            skipna: bool = True) -> torch.Tensor:
    """Weighted sum / mean along ``axis`` (grid.py:1598-1605, :1680-1685)."""
    lib = _capi.load()
    _require_cuda(x, "field")
    x = x.contiguous()
    axis = _norm_axis(axis, x.dim())
    shape = list(x.shape)
    out_shape = [s for d, s in enumerate(shape) if d != axis]
    out = torch.empty(out_shape, dtype=x.dtype, device=x.device)
    keep, w_ptr, w_st = _operand(weight, shape, x, "weight")
    if out.numel():
        with torch.cuda.device(x.device):
            rc = lib.xg_wreduce(_dtype_code(x), x.data_ptr(), w_ptr, w_st, out.data_ptr(), x.dim(),
                                _capi.i64_array(shape), axis, _capi.REDUCE[mode],
                                int(bool(skipna)), _stream_ptr(x))
        _capi.check(rc)
    return out


def vinterp_linear(phi: torch.Tensor, theta: torch.Tensor, target: torch.Tensor, axis: int,
                   mask_edges: bool = False, bypass_checks: bool = False,
                   logarithmic: bool = False) -> torch.Tensor:
    """Per-column linear interpolation onto ``target`` levels; new dim LAST
    (transform.py:15-85).  ``theta`` broadcasts against ``phi``.  ``target`` is either a
    shared 1-D level vector or an array whose leading dims broadcast against the column
    dims of ``phi`` (shape-without-axis) and whose LAST dim holds the levels."""
    lib = _capi.load()
    _require_cuda(phi, "phi")
    _require_cuda(theta, "theta")
    _require_cuda(target, "target")
    # numba gufunc loop resolution (transform.py:15-22): float32 only if all are
    if not (phi.dtype == theta.dtype == target.dtype == torch.float32):
        phi, theta, target = phi.to(torch.float64), theta.to(torch.float64), target.to(torch.float64)
    phi = phi.contiguous()
    axis = _norm_axis(axis, phi.dim())
    shape = list(phi.shape)
    m = int(target.shape[-1]) if target.dim() else 1
    keep, th_ptr, th_st = _operand(theta, shape, phi, "theta")
    col_shape = [s for d, s in enumerate(shape) if d != axis]
    tg_st = None
    if target.dim() <= 1:
        target = target.reshape(-1).contiguous()
    else:
        try:
            tb = target.expand(tuple(col_shape) + (m,))
        except RuntimeError as err:
            raise ValueError(
                f"target of shape {tuple(target.shape)} does not broadcast to columns {tuple(col_shape)} + (m,)"
            ) from err
        st = list(tb.stride())
        col_st = [0 if s == 1 else t for s, t in zip(col_shape, st[:-1])]
        full = col_st[:axis] + [st[-1]] + col_st[axis:]
        tg_st = _capi.i64_array(full)
        target = tb
    out_shape = col_shape + [m]
    out = torch.empty(out_shape, dtype=phi.dtype, device=phi.device)
    if out.numel():
        with torch.cuda.device(phi.device):
            rc = lib.xg_vinterp_linear(
                _dtype_code(phi), phi.data_ptr(), th_ptr, th_st, target.data_ptr(), tg_st,
                m, out.data_ptr(), phi.dim(), _capi.i64_array(shape), axis,
                int(bool(mask_edges)), int(bool(bypass_checks)), int(bool(logarithmic)),
                _stream_ptr(phi),
            )
        _capi.check(rc)
    return out


def vinterp_conservative(phi: torch.Tensor, theta: torch.Tensor, target_bins: torch.Tensor,
                         axis: int) -> torch.Tensor:
    """Conservative remapping of an extensive ``phi`` (n cells along ``axis``) bounded by
    ``theta`` (n + 1 bounds along ``axis``, broadcast elsewhere) into the bins delimited by the
    monotonic 1-D ``target_bins`` (transform.py:88-191).  New dim (m - 1 bins) LAST."""
    lib = _capi.load()
    _require_cuda(phi, "phi")
    _require_cuda(theta, "theta")
    _require_cuda(target_bins, "target_bins")
    if not (phi.dtype == theta.dtype == target_bins.dtype == torch.float32):
        phi, theta, target_bins = phi.to(torch.float64), theta.to(torch.float64), target_bins.to(torch.float64)
    if target_bins.dim() != 1:
        raise ValueError("target bins must be 1-D")
    phi = phi.contiguous()
    axis = _norm_axis(axis, phi.dim())
    shape = list(phi.shape)
    tshape = list(shape)
    tshape[axis] = shape[axis] + 1
    if theta.dim() == phi.dim() and theta.shape[axis] != tshape[axis]:
        raise ValueError(
            f"theta needs {tshape[axis]} cell bounds along the axis, got {theta.shape[axis]}"
        )  # transform.py:162 assert phi.shape[-1] == theta.shape[-1] - 1
    flip = _bins_order(target_bins[1:] - target_bins[:-1])
    bins = (torch.flip(target_bins, dims=(0,)) if flip else target_bins).contiguous()
    keep, th_ptr, th_st = _operand(theta, tshape, phi, "theta")
    m = int(bins.numel())
    out_shape = [s for d, s in enumerate(shape) if d != axis] + [m - 1]
    out = torch.empty(out_shape, dtype=phi.dtype, device=phi.device)
    if out.numel():
        with torch.cuda.device(phi.device):
            rc = lib.xg_vinterp_conservative(
                _dtype_code(phi), phi.data_ptr(), th_ptr, th_st, bins.data_ptr(), m, flip,
                out.data_ptr(), phi.dim(), _capi.i64_array(shape), axis, _stream_ptr(phi),
            )
        _capi.check(rc)
    return out


def fill_uniform(out: torch.Tensor, seed: int, offset: int = 0) -> torch.Tensor:
    """Deterministic U(0,1) synthetic field keyed by (seed, offset + flat index)."""
    lib = _capi.load()
    _require_cuda(out, "out")
    if not out.is_contiguous():
        raise ValueError("out must be contiguous")
    with torch.cuda.device(out.device):
        rc = lib.xg_fill_uniform(_dtype_code(out), out.data_ptr(), out.numel(), int(seed),
                                 int(offset), _stream_ptr(out))
    _capi.check(rc)
    return out


def fill_uniform_host(out: np.ndarray, seed: int, offset: int = 0) -> np.ndarray:
    """Host twin of :func:`fill_uniform` (same bits)."""
    lib = _capi.load()
    if not out.flags.c_contiguous:
        raise ValueError("out must be C-contiguous")
    rc = lib.xg_fill_uniform_host(_capi.dtype_code(out.dtype), out.ctypes.data, out.size,
                                  int(seed), int(offset))
    _capi.check(rc)
    return out


def _host_operand(m: Optional[np.ndarray], shape: Sequence[int], dtype, what: str):
    if m is None:
        return None, None, None
    m = np.ascontiguousarray(m, dtype=dtype)
    try:
        mb = np.broadcast_to(m, tuple(shape))
    except ValueError as err:
        raise ValueError(f"{what} of shape {m.shape} does not broadcast to {tuple(shape)}") from err
    es = m.dtype.itemsize
    strides = [0 if s == 1 else st // es for s, st in zip(shape, mb.strides)]
    return m, m.ctypes.data, _capi.i64_array(strides)


def _host_field(x, what, cast=True):
    """``x`` C-contiguous for a host twin (with ``cast``, a non-float field as float64), on a machine with a CUDA
    device."""
    if not isinstance(x, np.ndarray):
        raise TypeError(f"{what} must be a numpy array")
    if not torch.cuda.is_available():
        raise RuntimeError("xgcm_b200 needs a CUDA device: the stencil engine has no CPU fallback")
    if cast and x.dtype not in (np.float32, np.float64):
        x = x.astype(np.float64)
    if not x.flags.c_contiguous:
        x = np.ascontiguousarray(x)
    return x


def _host_out(out, shape, dtype):
    """The page-locked result of a host twin, or the caller's ``out`` after checking it."""
    if out is None:
        return pinned_empty(shape, dtype)
    if list(out.shape) != list(shape) or out.dtype != dtype or not out.flags.c_contiguous:
        raise ValueError("out has wrong shape/dtype/layout")
    return out


def pinned_empty(shape, dtype=np.float32) -> np.ndarray:
    """A page-locked numpy array (torch's caching host allocator owns the memory)."""
    tdt = {np.dtype("float32"): torch.float32, np.dtype("float64"): torch.float64}[np.dtype(dtype)]
    t = torch.empty(tuple(int(s) for s in shape), dtype=tdt, pin_memory=True)
    return t.numpy()


def stencil2_host(
    x: np.ndarray,
    axis: int,
    op: str,
    lo: int,
    hi: int,
    padding: Optional[str],
    fill_value: float = 0.0,
    pre: Optional[np.ndarray] = None,
    post: Optional[np.ndarray] = None,
    out: Optional[np.ndarray] = None,
    device: HostDevice = None,
) -> np.ndarray:
    """Host-buffer twin of :func:`stencil2`: slabs stream H2D -> kernel -> D2H on three
    streams inside ``xg_stencil2_host``.  Page-locked buffers get the full PCIe rate."""
    lib = _capi.load()
    x, shape, axis, out, pre_op, post_op, dev = _host_stencil_prep(x, axis, op, lo, hi, padding, pre, post, out,
                                                                   device, "stencil2_host")
    rc = lib.xg_stencil2_host(
        _capi.OPS[op], _capi.dtype_code(x.dtype), x.ctypes.data, out.ctypes.data, x.ndim,
        _capi.i64_array(shape), axis, lo, hi, _capi.BCS[padding], float(fill_value),
        pre_op[1], pre_op[2], post_op[1], post_op[2], dev,
    )
    _capi.check(rc)
    return out


def _host_stencil_prep(x, axis, op, lo, hi, padding, pre, post, out, device, what):
    """Checks and buffers shared by the host stencil twins: (contiguous x, shape, axis, out, pre operand,
    post operand, device index)."""
    x = _host_field(x, f"{what}: field", cast=False)
    if op not in _capi.OPS:
        raise ValueError(f"unknown op {op!r}")
    _check_padding(padding)
    axis = _norm_axis(axis, x.ndim)
    shape = list(x.shape)
    out_shape = list(shape)
    out_shape[axis] = shape[axis] + lo + hi - 1
    out = _host_out(out, out_shape, x.dtype)
    pre_op = _host_operand(pre, shape, x.dtype, "pre metric")
    post_op = _host_operand(post, out_shape, x.dtype, "post metric")
    dev = host_device_arg(device)
    return x, shape, axis, out, pre_op, post_op, dev


def stencil2_host_fold(x: np.ndarray, axis: int, op: str, lo: int, hi: int, padding: Optional[str],
                       fill_value: float, seam_axis: int, skip: int, mirror: int, period: int,
                       negate: bool = False, pre: Optional[np.ndarray] = None, post: Optional[np.ndarray] = None,
                       out: Optional[np.ndarray] = None, device: HostDevice = None) -> np.ndarray:
    """:func:`stencil2_host` across a north fold along ``axis`` (``xg_stencil2_host_fold``): each slab's
    halo_hi is its folded row (:func:`fold_rows` with ``seam_axis, skip, mirror, period, negate``, of
    ``x * pre``), also halo_lo when the south edge ``padding`` is periodic.  Dim 0 is cut into slabs and must
    be neither ``axis`` nor ``seam_axis``."""
    lib = _capi.load()
    x, shape, axis, out, pre_op, post_op, dev = _host_stencil_prep(x, axis, op, lo, hi, padding, pre, post, out,
                                                                   device, "stencil2_host_fold")
    rc = lib.xg_stencil2_host_fold(
        _capi.OPS[op], _capi.dtype_code(x.dtype), x.ctypes.data, out.ctypes.data, x.ndim,
        _capi.i64_array(shape), axis, lo, hi, _capi.BCS[padding], float(fill_value),
        pre_op[1], pre_op[2], post_op[1], post_op[2], _norm_axis(seam_axis, x.ndim), int(skip), int(mirror),
        int(period), 1 if negate else 0, dev,
    )
    _capi.check(rc)
    return out


_HALO_SOURCES = {"self": 0, "partner": 1, "fill": 2}


def _copy_list_args(program: Sequence[tuple]):
    """C-ABI arguments of a face-connection copy list (``padding.connected_halo_program``): count, rank, sides,
    sources, dst / src offsets, then the flattened shapes, dst strides, src strides and the negate flags."""
    import ctypes as C

    n = len(program)
    cndim = len(program[0][6]) if n else 1
    if any(len(c[6]) != cndim or len(c[2]) != cndim or len(c[5]) != cndim for c in program):
        raise ValueError("every copy of a halo program must have the same rank")
    i32 = lambda vals: (C.c_int * max(n, 1))(*vals)  # noqa: E731
    flat = lambda k: _capi.i64_array([int(v) for c in program for v in c[k]] or [0])  # noqa: E731
    return (n, cndim, i32([int(c[0]) for c in program]), i32([_HALO_SOURCES[c[3]] for c in program]),
            _capi.i64_array([int(c[1]) for c in program] or [0]), _capi.i64_array([int(c[4]) for c in program] or [0]),
            flat(6), flat(2), flat(5), i32([1 if c[7] else 0 for c in program]))


def stencil2_host_connected(x: np.ndarray, axis: int, op: str, lo: int, hi: int, fill_value: float,
                            program: Sequence[tuple], partner: Optional[np.ndarray] = None,
                            post: Optional[np.ndarray] = None, out: Optional[np.ndarray] = None,
                            device: HostDevice = None) -> np.ndarray:
    """:func:`stencil2_host` on a grid with face connections (``xg_stencil2_host_connected``): the halo
    planes of each slab are written by ``program``, the strided copies of
    ``padding.connected_halo_program`` — ``(side, dst offset, dst strides, source ("self", "partner" or
    "fill"), src offset, src strides, shape, negate)`` for the whole field, clipped to each slab by the
    library.  ``partner`` (the other vector component) streams beside ``x``; "fill" reads ``fill_value``."""
    lib = _capi.load()
    x, shape, axis, out, _, post_op, dev = _host_stencil_prep(x, axis, op, lo, hi, "fill" if (lo or hi) else None,
                                                              None, post, out, device, "stencil2_host_connected")
    p_shape = None
    if partner is not None:
        partner = np.ascontiguousarray(partner, dtype=x.dtype)
        p_shape = list(partner.shape)
        if len(p_shape) != x.ndim:
            raise ValueError(f"partner component of shape {tuple(p_shape)} has not the rank of the field {tuple(shape)}")
    n, cndim, side, source, doff, soff, shapes, dstr, sstr, neg = _copy_list_args(program)
    rc = lib.xg_stencil2_host_connected(
        _capi.OPS[op], _capi.dtype_code(x.dtype), x.ctypes.data,
        None if partner is None else partner.ctypes.data, _capi.i64_array(p_shape), out.ctypes.data, x.ndim,
        _capi.i64_array(shape), axis, lo, hi, float(fill_value), post_op[1], post_op[2], n, cndim, side, source,
        doff, soff, shapes, dstr, sstr, neg, dev,
    )
    _capi.check(rc)
    return out


def stencil2_host_connected_weighted(x: np.ndarray, axis: int, op: str, lo: int, hi: int, fill_value: float,
                                     program: Sequence[tuple], pre: np.ndarray, post: Optional[np.ndarray] = None,
                                     out: Optional[np.ndarray] = None, device: HostDevice = None) -> np.ndarray:
    """:func:`stencil2_host_connected` of ``x * pre`` (``xg_stencil2_host_connected_weighted``), divided by ``post``:
    the metric-weighted operator of a scalar field across face connections.  ``program`` is the copy list of
    ``padding.connected_halo_program`` with a metric layout, whose copies also carry the offset and strides of the
    ``pre`` cells they read (the pre-metric broadcast against ``x``, strides 0 where it broadcasts); no partner."""
    lib = _capi.load()
    x, shape, axis, out, pre_op, post_op, dev = _host_stencil_prep(
        x, axis, op, lo, hi, "fill" if (lo or hi) else None, pre, post, out, device,
        "stencil2_host_connected_weighted")
    if pre_op[0] is None:
        raise ValueError("stencil2_host_connected_weighted: a pre-metric is required")
    if any(len(c) != 10 or len(c[9]) != len(c[6]) for c in program):
        raise ValueError("stencil2_host_connected_weighted: every copy must carry the metric offset and strides")
    n, cndim, side, source, doff, soff, shapes, dstr, sstr, neg = _copy_list_args(program)
    poff = _capi.i64_array([int(c[8]) for c in program] or [0])
    pstr = _capi.i64_array([int(v) for c in program for v in c[9]] or [0])
    rc = lib.xg_stencil2_host_connected_weighted(
        _capi.OPS[op], _capi.dtype_code(x.dtype), x.ctypes.data, out.ctypes.data, x.ndim, _capi.i64_array(shape),
        axis, lo, hi, float(fill_value), pre_op[1], pre_op[2], post_op[1], post_op[2], n, cndim, side, source, doff,
        soff, poff, shapes, dstr, sstr, pstr, neg, dev,
    )
    _capi.check(rc)
    return out


def _chain_args(x, specs):
    """C-ABI values of the stages ``specs`` of a host chain (``_stencil_specs``): the count, the page-locked result,
    the int arrays of axes, op codes, lo and hi, the boundary codes, and the fills."""
    import ctypes as C

    n = len(specs)
    axes, opc, los, his, bcs, fills = _stencil_specs(specs, x.ndim, fused=False)
    out = pinned_empty(_multi_out_shape(list(x.shape), axes, los, his), x.dtype)
    i32 = C.c_int * max(n, 1)
    return n, out, (i32(*axes), i32(*opc), i32(*los), i32(*his)), i32(*bcs), (C.c_double * max(n, 1))(*fills)


def stencil_chain_host_fold(x: np.ndarray, stages, device: HostDevice = None) -> np.ndarray:
    """A multi-axis stencil of a host field on a fold grid, stage by stage as the device route launches it
    (``xg_stencil_chain_host_fold``).  ``stages``: 2 or 3 of ``(axis, op, lo, hi, padding, fill, fold)``, each on the
    previous stage's result, ``fold`` None or ``(seam_axis, skip, mirror, period)`` (:func:`fold_rows`, planned for
    that stage's input) when the stage's north edge crosses the fold.  Dim 0 is cut into slabs and must be a batch
    dim."""
    import ctypes as C

    lib = _capi.load()
    x = _host_field(x, "stencil_chain_host_fold: field", cast=False)
    n, out, (axes, opc, los, his), bcs, fills = _chain_args(x, [s[:6] for s in stages])
    plans = [s[6] if s[6] is not None else (0, 0, 0, 1) for s in stages]
    i32 = C.c_int * max(n, 1)
    if out.size:
        rc = lib.xg_stencil_chain_host_fold(
            _capi.dtype_code(x.dtype), x.ctypes.data, out.ctypes.data, x.ndim, _capi.i64_array(x.shape), n, axes,
            opc, los, his, bcs, fills, i32(*[0 if s[6] is None else 1 for s in stages]),
            i32(*[_norm_axis(p[0], x.ndim) for p in plans]), i32(*[int(p[1]) for p in plans]),
            _capi.i64_array([p[2] for p in plans]), _capi.i64_array([p[3] for p in plans]), host_device_arg(device))
        _capi.check(rc)
    return out


def stencil_chain_host_connected(x: np.ndarray, stages, programs, device: HostDevice = None) -> np.ndarray:
    """:func:`stencil_chain_host_fold` on a grid with face connections (``xg_stencil_chain_host_connected``):
    ``stages`` of ``(axis, op, lo, hi, fill)``; ``programs[s]`` writes the halo planes of stage ``s``, the copy list
    of :func:`stencil2_host_connected` (``padding.connected_halo_program``) for that stage's input, sources "self"
    and "fill" (``fill`` of the stage)."""
    import ctypes as C

    lib = _capi.load()
    x = _host_field(x, "stencil_chain_host_connected: field", cast=False)
    if len(programs) != len(stages):
        raise ValueError("stencil_chain_host_connected: one halo program per stage")
    specs = [(axis, op, lo, hi, "fill" if (lo or hi) else None, fill) for axis, op, lo, hi, fill in stages]
    n, out, (axes, opc, los, his), _, fills = _chain_args(x, specs)
    _, cndim, side, source, doff, soff, shapes, dstr, sstr, neg = _copy_list_args([c for p in programs for c in p])
    if out.size:
        rc = lib.xg_stencil_chain_host_connected(
            _capi.dtype_code(x.dtype), x.ctypes.data, out.ctypes.data, x.ndim, _capi.i64_array(x.shape), n, axes,
            opc, los, his, fills, (C.c_int * max(n, 1))(*[len(p) for p in programs]), cndim, side, source, doff, soff,
            shapes, dstr, sstr, neg, host_device_arg(device))
        _capi.check(rc)
    return out


def _pair_specs(spec_a, spec_b, ndim: int):
    """C-ABI values of the two terms of a pair: ``(op_a, lo_a, hi_a, bc_a, fill_a)``, ``(axis_b, op_b, lo_b, hi_b,
    bc_b, fill_b)``."""
    op_a, lo_a, hi_a, pad_a, fill_a = spec_a
    axis_b, op_b, lo_b, hi_b, pad_b, fill_b = spec_b
    for pad_ in (pad_a, pad_b):
        if pad_ not in ("periodic", "fill", "extend"):
            raise ValueError(f"padding must be one of ['periodic', 'fill', 'extend'], but got {pad_}")
    return ((_capi.OPS[op_a], int(lo_a), int(hi_a), _capi.BCS[pad_a], float(0.0 if fill_a is None else fill_a)),
            (_norm_axis(axis_b, ndim), _capi.OPS[op_b], int(lo_b), int(hi_b), _capi.BCS[pad_b],
             float(0.0 if fill_b is None else fill_b)))


def stencil_pair(a: torch.Tensor, b: torch.Tensor, spec_a, spec_b, subtract: int = 0,
                 pre_a: Optional[torch.Tensor] = None, pre_b: Optional[torch.Tensor] = None,
                 post: Optional[torch.Tensor] = None, halo_lo_b: Optional[torch.Tensor] = None,
                 halo_hi_b: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``(OPa(a * pre_a) along the innermost dim  +|-  OPb(b * pre_b) along another dim) / post`` in one pass
    (``xg_stencil_pair_halo``).  ``spec_a = (op, lo, hi, padding, fill)`` acts on the LAST dim, ``spec_b =
    (axis, op, lo, hi, padding, fill)`` on ``axis`` != last.  All arrays share ``a``'s shape; metrics broadcast.

    ``halo_lo_b`` / ``halo_hi_b``: optional planes (``a``'s shape with extent 1 along ``axis``, already
    weighted by ``pre_b``) that pad the term along ``axis`` instead of its padding on their side, e.g. the
    folded north row of :func:`fold_rows`."""
    lib = _capi.load()
    _require_cuda(a, "field a")
    _require_cuda(b, "field b")
    if a.shape != b.shape or a.dtype != b.dtype:
        raise ValueError("stencil_pair: both fields must have the same shape and dtype")
    a, b = a.contiguous(), b.contiguous()
    term_a, term_b = _pair_specs(spec_a, spec_b, a.dim())
    shape = list(a.shape)
    out = torch.empty_like(a)
    k1, pa_ptr, pa_st = _operand(pre_a, shape, a, "pre metric a")
    k2, pb_ptr, pb_st = _operand(pre_b, shape, a, "pre metric b")
    k3, po_ptr, po_st = _operand(post, shape, a, "post metric")
    plane = int(np.prod([s for d, s in enumerate(shape) if d != term_b[0]], dtype=np.int64))
    halos = []
    for h, what in ((halo_lo_b, "halo_lo_b"), (halo_hi_b, "halo_hi_b")):
        if h is not None:
            _require_cuda(h, what)
            if h.device != a.device:
                raise RuntimeError(f"{what} is on {h.device}, field on {a.device}")
            h = h.to(a.dtype).contiguous()
            if h.numel() != plane:
                raise ValueError(f"{what} has wrong size")
        halos.append(h)
    if out.numel():
        with torch.cuda.device(a.device):
            rc = lib.xg_stencil_pair_halo(
                _dtype_code(a), a.data_ptr(), b.data_ptr(), out.data_ptr(), a.dim(), _capi.i64_array(shape),
                *term_a, pa_ptr, pa_st, *term_b, pb_ptr, pb_st, int(subtract), po_ptr, po_st,
                *[None if h is None else h.data_ptr() for h in halos], _stream_ptr(a))
        _capi.check(rc)
    return out


def _host_pair_prep(a, b, spec_a, spec_b, pre_a, pre_b, post, out, device, what):
    """Checks and buffers shared by the host pair twins: (a, b, shape, C-ABI term values, the three operands,
    out, device index)."""
    a, b = _host_field(a, f"{what}: field a", cast=False), _host_field(b, f"{what}: field b", cast=False)
    if a.shape != b.shape or a.dtype != b.dtype:
        raise ValueError(f"{what}: both fields must have the same shape and dtype")
    term_a, term_b = _pair_specs(spec_a, spec_b, a.ndim)
    shape = list(a.shape)
    out = _host_out(out, shape, a.dtype)
    ops_ = [_host_operand(m, shape, a.dtype, w) for m, w in ((pre_a, "pre metric a"), (pre_b, "pre metric b"),
                                                             (post, "post metric"))]
    dev = host_device_arg(device)
    return a, b, shape, term_a, term_b, ops_, out, dev


def stencil_pair_host(a: np.ndarray, b: np.ndarray, spec_a, spec_b, subtract: int = 0,
                      pre_a: Optional[np.ndarray] = None, pre_b: Optional[np.ndarray] = None,
                      post: Optional[np.ndarray] = None, out: Optional[np.ndarray] = None,
                      device: HostDevice = None) -> np.ndarray:
    """Host-buffer twin of :func:`stencil_pair` (``xg_stencil_pair_host``): ``a`` and ``b`` stream through the
    GPU in slabs of dim 0, which must be a batch dim (not ``spec_b``'s axis)."""
    lib = _capi.load()
    a, b, shape, term_a, term_b, (pa, pb, po), out, dev = _host_pair_prep(a, b, spec_a, spec_b, pre_a, pre_b, post,
                                                                           out, device, "stencil_pair_host")
    rc = lib.xg_stencil_pair_host(
        _capi.dtype_code(a.dtype), a.ctypes.data, b.ctypes.data, out.ctypes.data, a.ndim, _capi.i64_array(shape),
        *term_a, pa[1], pa[2], *term_b, pb[1], pb[2], int(subtract), po[1], po[2], dev)
    _capi.check(rc)
    return out


def stencil_pair_host_fold(a: np.ndarray, b: np.ndarray, spec_a, spec_b, seam_axis: int, skip: int, mirror: int,
                           period: int, subtract: int = 0, negate: bool = False, pre_a: Optional[np.ndarray] = None,
                           pre_b: Optional[np.ndarray] = None, post: Optional[np.ndarray] = None,
                           out: Optional[np.ndarray] = None, device: HostDevice = None) -> np.ndarray:
    """:func:`stencil_pair_host` with the term along ``spec_b``'s axis across a north fold
    (``xg_stencil_pair_host_fold``): each slab's ``halo_hi_b`` is the folded row of ``b * pre_b``
    (:func:`fold_rows` with ``seam_axis, skip, mirror, period, negate``), also ``halo_lo_b`` when ``spec_b``
    pads the south edge periodically.  Dim 0 must be neither ``spec_b``'s axis nor ``seam_axis``."""
    lib = _capi.load()
    a, b, shape, term_a, term_b, (pa, pb, po), out, dev = _host_pair_prep(a, b, spec_a, spec_b, pre_a, pre_b, post,
                                                                           out, device, "stencil_pair_host_fold")
    rc = lib.xg_stencil_pair_host_fold(
        _capi.dtype_code(a.dtype), a.ctypes.data, b.ctypes.data, out.ctypes.data, a.ndim, _capi.i64_array(shape),
        *term_a, pa[1], pa[2], *term_b, pb[1], pb[2], int(subtract), po[1], po[2], _norm_axis(seam_axis, a.ndim),
        int(skip), int(mirror), int(period), 1 if negate else 0, dev)
    _capi.check(rc)
    return out


# --------------------------------------------------------------------------- host twins (slab pipelines)


def stencil2_host_multi(x: np.ndarray, specs, outs=None, device: HostDevice = None):
    """One host field up, several stencil results down (``xg_stencil2_host_multi``).

    ``specs``: sequence of ``(axis, op, lo, hi, padding, fill_value)``.  Returns a list of page-locked
    numpy arrays (or fills ``outs``).  Raises NotImplementedError for what the batched pipeline does not
    cover (outer / inner shifts or extrapolate along dim 0) — callers then use :func:`stencil2_host`."""
    lib = _capi.load()
    x = _host_field(x, "field")
    k = len(specs)
    shape = list(x.shape)
    axes, ops_, los, his, bcs, fills = _stencil_specs(specs, x.ndim, fused=False)
    out_shapes = [_multi_out_shape(shape, [axis], [lo], [hi]) for axis, lo, hi in zip(axes, los, his)]
    if outs is None:
        outs = [pinned_empty(s, x.dtype) for s in out_shapes]
    for o, s in zip(outs, out_shapes):
        if list(o.shape) != s or o.dtype != x.dtype or not o.flags.c_contiguous:
            raise ValueError("out has wrong shape/dtype/layout")
    import ctypes as C

    out_ptrs = (C.c_void_p * k)(*[o.ctypes.data for o in outs])
    dev = host_device_arg(device)
    rc = lib.xg_stencil2_host_multi(
        k, (C.c_int * k)(*ops_), _capi.dtype_code(x.dtype), x.ctypes.data, out_ptrs, x.ndim,
        _capi.i64_array(shape), (C.c_int * k)(*axes), (C.c_int * k)(*los), (C.c_int * k)(*his),
        (C.c_int * k)(*bcs), (C.c_double * k)(*fills), dev)
    _capi.check(rc)
    return list(outs)


def stencil_multi_host(x: np.ndarray, specs: Sequence[Tuple[int, str, int, int, Optional[str], float]],
                       device: HostDevice = None, *, pre: Optional[Sequence[Optional[np.ndarray]]] = None,
                       post: Optional[Sequence[Optional[np.ndarray]]] = None) -> np.ndarray:
    """Host twin of :func:`stencil_multi` (``xg_stencil_multi_host``): slabs of the outermost non-operated dim of
    extent > 1 stream through the GPU, one fused launch each.  Raises NotImplementedError for what the slabs do not
    cover (mixed operators; an outer / inner shift or a periodic boundary along the cut dim when every dim of extent
    > 1 is operated) — callers then use :func:`stencil_multi`.

    ``pre`` / ``post``: per-stage host metrics as :func:`stencil_multi` takes them (``xg_stencil_multi_weighted_host``:
    uploaded whole once per device, each slab's launch offset into them)."""
    import ctypes as C

    lib = _capi.load()
    x = _host_field(x, "field")
    if not 2 <= len(specs) <= 3:
        raise ValueError("stencil_multi fuses 2 or 3 axes")
    shape = list(x.shape)
    axes, opc, los, his, bcs, fills = _stencil_specs(specs, x.ndim, fused=True)
    out = pinned_empty(_multi_out_shape(shape, axes, los, his), x.dtype)
    n = len(specs)
    IntArr, DblArr = C.c_int * n, C.c_double * n
    pre, post = _stage_list(pre, n, "pre"), _stage_list(post, n, "post")
    weighted = any(m is not None for m in pre + post)
    keep, met_args = [], []
    if weighted:
        for mets, shapes, what in ((pre, _stage_shapes(shape, axes, los, his, 0), "pre"),
                                   (post, _stage_shapes(shape, axes, los, his, 1), "post")):
            ptrs, strides = (C.c_void_p * n)(), []
            for k, (m, s) in enumerate(zip(mets, shapes)):
                mh, ptr, st = _host_operand(m, s, x.dtype, f"{what} metric of stage {k}")
                keep.append(mh)
                ptrs[k] = ptr
                strides += list(st) if st is not None else [0] * len(shape)
            met_args += [ptrs, _capi.i64_array(strides)]
    dev = host_device_arg(device)
    if out.size:
        args = (_capi.dtype_code(x.dtype), x.ctypes.data, out.ctypes.data, x.ndim, _capi.i64_array(shape), n,
                IntArr(*axes), IntArr(*opc), IntArr(*los), IntArr(*his), IntArr(*bcs), DblArr(*fills))
        if weighted:
            rc = lib.xg_stencil_multi_weighted_host(*args, *met_args, dev)
        else:
            rc = lib.xg_stencil_multi_host(*args, dev)
        _capi.check(rc)
    return out


def cumscan_host(x: np.ndarray, axis: int, reverse: bool = False, trim: str = "none", pad_lo: int = 0,
                 pad_hi: int = 0, padding: Optional[str] = None, fill_value: float = 0.0,
                 pre: Optional[np.ndarray] = None, post: Optional[np.ndarray] = None, skipna: bool = True,
                 device: HostDevice = None) -> np.ndarray:
    """Host twin of :func:`cumscan` (``xg_cumscan_host``): slabs of a non-operated dim stream through the GPU."""
    lib = _capi.load()
    _check_padding(padding)
    x, shape, axis, out, pre_op, post_op, dev = _host_scan_prep(x, axis, trim, pad_lo, pad_hi, pre, post, device)
    if out.size:
        rc = lib.xg_cumscan_host(
            _capi.dtype_code(x.dtype), x.ctypes.data, out.ctypes.data, x.ndim, _capi.i64_array(shape), axis,
            int(bool(reverse)), _capi.TRIMS[trim], pad_lo, pad_hi, _capi.BCS[padding], float(fill_value),
            pre_op[1], pre_op[2], post_op[1], post_op[2], int(bool(skipna)), dev)
        _capi.check(rc)
    return out


def _host_scan_prep(x, axis, trim, pad_lo, pad_hi, pre, post, device):
    """Checks and buffers shared by the host cumscan twins: (contiguous x, shape, axis, out, pre operand, post
    operand, device index)."""
    x = _host_field(x, "field")
    axis = _norm_axis(axis, x.ndim)
    shape = list(x.shape)
    kept = shape[axis] - (0 if trim == "none" else 1)
    if kept < 0:
        raise ValueError("operated axis too short to trim")
    out_shape = list(shape)
    out_shape[axis] = kept + pad_lo + pad_hi
    out = pinned_empty(out_shape, x.dtype)
    pre_op = _host_operand(pre, shape, x.dtype, "pre metric")
    post_op = _host_operand(post, out_shape, x.dtype, "post metric")
    return x, shape, axis, out, pre_op, post_op, host_device_arg(device)


def cumscan_host_fold(x: np.ndarray, axis: int, reverse: bool, trim: str, seam_axis: int, skip: int, mirror: int,
                      period: int, pre: Optional[np.ndarray] = None, post: Optional[np.ndarray] = None,
                      skipna: bool = True, device: HostDevice = None) -> np.ndarray:
    """:func:`cumscan_host` whose north edge is padded across a fold (``xg_cumscan_host_fold``): bit for bit
    :func:`cumscan` (``pre``, no post), then the folded row of the scanned field as one row above it
    (:func:`fold_rows` with ``seam_axis, skip, mirror, period``, planned for the scanned shape), then ``/ post``.
    Dim 0 is cut into slabs and must be neither ``axis`` nor ``seam_axis``."""
    lib = _capi.load()
    x, shape, axis, out, pre_op, post_op, dev = _host_scan_prep(x, axis, trim, 0, 1, pre, post, device)
    if out.size:
        rc = lib.xg_cumscan_host_fold(
            _capi.dtype_code(x.dtype), x.ctypes.data, out.ctypes.data, x.ndim, _capi.i64_array(shape), axis,
            int(bool(reverse)), _capi.TRIMS[trim], 0, 1, pre_op[1], pre_op[2], post_op[1], post_op[2],
            int(bool(skipna)), _norm_axis(seam_axis, x.ndim), int(skip), int(mirror), int(period), dev)
        _capi.check(rc)
    return out


def cumscan_host_connected(x: np.ndarray, axis: int, reverse: bool, trim: str, pad_lo: int, pad_hi: int,
                           fill_value: float, program: Sequence[tuple], pre: Optional[np.ndarray] = None,
                           post: Optional[np.ndarray] = None, skipna: bool = True,
                           device: HostDevice = None) -> np.ndarray:
    """:func:`cumscan_host` on a grid with face connections (``xg_cumscan_host_connected``): bit for bit
    :func:`cumscan` (``pre``, no post), then the halo planes written by ``program`` — the copy list of
    :func:`stencil2_host_connected`, built by ``padding.connected_halo_program`` for the SCANNED field's shape,
    sources "self" and "fill" — then ``/ post``."""
    lib = _capi.load()
    x, shape, axis, out, pre_op, post_op, dev = _host_scan_prep(x, axis, trim, pad_lo, pad_hi, pre, post, device)
    if out.size:
        n, cndim, side, source, doff, soff, shapes, dstr, sstr, neg = _copy_list_args(program)
        rc = lib.xg_cumscan_host_connected(
            _capi.dtype_code(x.dtype), x.ctypes.data, out.ctypes.data, x.ndim, _capi.i64_array(shape), axis,
            int(bool(reverse)), _capi.TRIMS[trim], pad_lo, pad_hi, float(fill_value), pre_op[1], pre_op[2],
            post_op[1], post_op[2], int(bool(skipna)), n, cndim, side, source, doff, soff, shapes, dstr, sstr, neg,
            dev)
        _capi.check(rc)
    return out


def wreduce_host(x: np.ndarray, axis: int, weight: Optional[np.ndarray] = None, mode: str = "sum",
                 skipna: bool = True, device: HostDevice = None) -> np.ndarray:
    """Host twin of :func:`wreduce` (``xg_wreduce_host``)."""
    lib = _capi.load()
    x = _host_field(x, "field")
    axis = _norm_axis(axis, x.ndim)
    shape = list(x.shape)
    out_shape = [s for d, s in enumerate(shape) if d != axis]
    out = pinned_empty(out_shape if out_shape else [1], x.dtype)
    kw, w_ptr, w_st = _host_operand(weight, shape, x.dtype, "weight")
    dev = host_device_arg(device)
    if out.size and x.size:
        rc = lib.xg_wreduce_host(_capi.dtype_code(x.dtype), x.ctypes.data, w_ptr, w_st, out.ctypes.data, x.ndim,
                                 _capi.i64_array(shape), axis, _capi.REDUCE[mode], int(bool(skipna)), dev)
        _capi.check(rc)
    return out if out_shape else out.reshape(())


def wreduce_host_multi(x: np.ndarray, axes: Sequence[int], weight: Optional[np.ndarray] = None, mode: str = "sum",
                       skipna: bool = True, device: HostDevice = None) -> np.ndarray:
    """Weighted sum / mean of a host field over several ``axes`` (``xg_wreduce_host_multi``), bit for bit the
    chain of :func:`wreduce` calls ``Grid.integrate`` / ``Grid.average`` run on the device.  Raises
    NotImplementedError for what the slabs do not cover (an empty reduced dim, or no reduced dim of extent > 1
    inside the slab dim) — callers then use :func:`wreduce`."""
    import ctypes as C

    lib = _capi.load()
    x = _host_field(x, "field")
    axes = [_norm_axis(a, x.ndim) for a in axes]
    shape = list(x.shape)
    out_shape = [s for d, s in enumerate(shape) if d not in axes]
    out = pinned_empty(out_shape if out_shape else [1], x.dtype)
    kw, w_ptr, w_st = _host_operand(weight, shape, x.dtype, "weight")
    dev = host_device_arg(device)
    if out.size:
        n = len(axes)
        rc = lib.xg_wreduce_host_multi(_capi.dtype_code(x.dtype), x.ctypes.data, w_ptr, w_st, out.ctypes.data,
                                       x.ndim, _capi.i64_array(shape), n, (C.c_int * n)(*axes), _capi.REDUCE[mode],
                                       int(bool(skipna)), dev)
        _capi.check(rc)
    return out if out_shape else out.reshape(())


def vinterp_linear_host(phi: np.ndarray, theta: np.ndarray, target: np.ndarray, axis: int,
                        mask_edges: bool = False, bypass_checks: bool = False, logarithmic: bool = False,
                        device: HostDevice = None) -> np.ndarray:
    """Host twin of :func:`vinterp_linear` for a shared 1-D ``target`` (``xg_vinterp_linear_host``); ``theta``
    broadcasts against ``phi`` (the 1-D coordinate or a full field)."""
    lib = _capi.load()
    phi = _host_field(phi, "phi")
    theta = np.asarray(theta)
    target = np.asarray(target)
    if target.ndim > 1:
        raise NotImplementedError("vinterp_linear_host: per-column targets; use the device entry point")
    if not (phi.dtype == theta.dtype == target.dtype == np.float32):  # numba loop resolution, transform.py:15-22
        phi, theta, target = phi.astype(np.float64, copy=False), theta.astype(np.float64), target.astype(np.float64)
    phi = np.ascontiguousarray(phi)
    axis = _norm_axis(axis, phi.ndim)
    shape = list(phi.shape)
    target = np.ascontiguousarray(target.reshape(-1))
    m = int(target.size)
    kt, th_ptr, th_st = _host_operand(theta, shape, phi.dtype, "theta")
    out_shape = [s for d, s in enumerate(shape) if d != axis] + [m]
    out = pinned_empty(out_shape, phi.dtype)
    dev = host_device_arg(device)
    if out.size:
        rc = lib.xg_vinterp_linear_host(
            _capi.dtype_code(phi.dtype), phi.ctypes.data, th_ptr, th_st, target.ctypes.data, None, m,
            out.ctypes.data, phi.ndim, _capi.i64_array(shape), axis, int(bool(mask_edges)),
            int(bool(bypass_checks)), int(bool(logarithmic)), dev)
        _capi.check(rc)
    return out


def vinterp_conservative_host(phi: np.ndarray, theta: np.ndarray, target_bins: np.ndarray, axis: int,
                              theta_at_centers: bool = False, device: HostDevice = None) -> np.ndarray:
    """Host twin of :func:`vinterp_conservative` (``xg_vinterp_conservative_host``): slabs of ``phi`` (and of
    ``theta`` when it is a full field) stream through the GPU.  With ``theta_at_centers``, ``theta`` holds n
    cell-centre values along ``axis`` and its bounds are those of ``grid.interp(theta, axis, padding="extend")``."""
    lib = _capi.load()
    phi = _host_field(phi, "phi")
    theta = np.asarray(theta)
    target_bins = np.asarray(target_bins)
    if not (phi.dtype == theta.dtype == target_bins.dtype == np.float32):
        phi, theta, target_bins = (phi.astype(np.float64, copy=False), theta.astype(np.float64, copy=False),
                                   target_bins.astype(np.float64, copy=False))
    if target_bins.ndim != 1:
        raise ValueError("target bins must be 1-D")
    phi = np.ascontiguousarray(phi)
    axis = _norm_axis(axis, phi.ndim)
    shape = list(phi.shape)
    tshape = list(shape)
    tshape[axis] = shape[axis] + (0 if theta_at_centers else 1)
    if theta.ndim == phi.ndim and theta.shape[axis] != tshape[axis]:
        what = "cell-centre values" if theta_at_centers else "cell bounds"
        raise ValueError(f"theta needs {tshape[axis]} {what} along the axis, got {theta.shape[axis]}")
    flip = _bins_order(target_bins[1:] - target_bins[:-1])
    bins = np.ascontiguousarray(target_bins[::-1] if flip else target_bins)
    kt, th_ptr, th_st = _host_operand(theta, tshape, phi.dtype, "theta")
    m = int(bins.size)
    out_shape = [s for d, s in enumerate(shape) if d != axis] + [m - 1]
    out = pinned_empty(out_shape, phi.dtype)
    dev = host_device_arg(device)
    if out.size:
        rc = lib.xg_vinterp_conservative_host(
            _capi.dtype_code(phi.dtype), phi.ctypes.data, th_ptr, th_st, int(bool(theta_at_centers)),
            bins.ctypes.data, m, flip, out.ctypes.data, phi.ndim, _capi.i64_array(shape), axis, dev)
        _capi.check(rc)
    return out
