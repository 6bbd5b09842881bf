"""``pad``: halo padding of labelled arrays (reference ``xgcm/padding.py:765-871``).

On simply connected grids the built-in operators never call this (their halo
is fused into the stencil kernel); it exists for user-defined grid ufuncs and
for API parity, and the copy runs on the device in ``xg_pad``.

On grids with ``face_connections`` (cubed sphere, LLC tiles) every operator
pads through ``_pad_face_connections`` (reference padding.py:260-572): faces
are pre-padded with the ordinary boundary condition, then the halo of every
connected edge is overwritten with the neighbour face's rim — sliced, swapped,
flipped and sign-flipped as the connection demands.  Each of those edge
transfers is one ``xg_strided_copy`` launch whose signed strides encode the
whole index map.

On grids with a north fold (tripolar ocean grids, ``padding={"X": "periodic",
"Y": {"fold": pivot}}``, reference padding.py:21-181, :619-762) the north edge of
the fold axis is padded by ``_pad_fold``: its halo rows are interior rows mirrored
along the periodic seam axis about the pole (``xg_fold_rows``), the south edge
and every other axis are padded as usual, in that order.  Operators take the
folded row as a halo plane of the fused stencil (``fold_halo_plane``).
"""

from __future__ import annotations

from typing import Dict, Mapping, Optional, Tuple, Union

from .labeled import DataArray

# reference padding.py:15-19
_XGCM_BOUNDARY_KWARG_TO_XARRAY_PAD_KWARG = {
    "periodic": "wrap",
    "fill": "constant",
    "extend": "edge",
}

# ---------------------------------------------------------------------------------------------- north fold
# The pivot names the sublattice the pole sits on along the seam (X) and fold (Y) axes: a cell
# centre or a cell edge (T / F / U / V points of ocean models).  The fold is experimental in the
# reference too; Grid construction warns.
_PIVOT_ALIASES = {
    "center": {"seam": "center", "fold": "center"},
    "t": {"seam": "center", "fold": "center"},
    "corner": {"seam": "edge", "fold": "edge"},
    "f": {"seam": "edge", "fold": "edge"},
    "u": {"seam": "edge", "fold": "center"},
    "v": {"seam": "center", "fold": "edge"},
}

# seam position -> (2 * offset of its cell coordinate, cells - length); the mirror partner of seam
# index k is (C - k - 2 * offset) mod N with N the number of cells, C = 0 (edge pivot) or 1 (centre)
_SEAM_POSITION = {"center": (1, 0), "left": (0, 0), "right": (2, 0), "outer": (0, -1), "inner": (2, 1)}


def _is_fold_padding(padding) -> bool:
    return isinstance(padding, Mapping) and "fold" in padding


def _position_kind(position: str) -> str:
    return "center" if position == "center" else "edge"


def _parse_fold_padding(padding: Mapping) -> Dict:
    """Validate a fold spec ``{"fold": pivot, "south": mode}``; returns it normalised (south defaults to fill)."""
    if not _is_fold_padding(padding):
        raise ValueError(f"Not a fold padding value: {padding!r}")
    extra = set(padding) - {"fold", "south"}
    if extra:
        raise ValueError(
            f"Unknown keys {sorted(extra)} in fold padding {dict(padding)!r}. "
            "Allowed keys are 'fold' (pivot type) and 'south' (south-edge mode)."
        )
    pivot = padding["fold"]
    if isinstance(pivot, str):
        if pivot.lower() not in _PIVOT_ALIASES:
            raise ValueError(
                f"Unknown fold pivot {pivot!r}. Use one of {sorted(_PIVOT_ALIASES)} "
                "or an explicit {axis: position} mapping."
            )
    elif isinstance(pivot, Mapping):
        if not pivot:
            raise ValueError("Explicit fold pivot mapping must not be empty.")
        bad = {ax: pos for ax, pos in pivot.items() if pos not in _SEAM_POSITION}
        if bad:
            raise ValueError(
                f"Invalid position(s) {bad} in explicit fold pivot {dict(pivot)!r}. "
                f"Each must be one of {sorted(_SEAM_POSITION)}."
            )
    else:
        raise ValueError(
            f"Fold pivot must be a name ({sorted(_PIVOT_ALIASES)}) or an {{axis: position}} mapping, got {pivot!r}."
        )
    south = padding.get("south", "fill")
    if south not in _XGCM_BOUNDARY_KWARG_TO_XARRAY_PAD_KWARG:
        raise ValueError(
            f"Fold 'south' mode must be one of {list(_XGCM_BOUNDARY_KWARG_TO_XARRAY_PAD_KWARG)}, got {south!r}."
        )
    return {"fold": pivot, "south": south}


def _resolve_pivot(pivot, fold_axis: str, seam_axis: str) -> Dict[str, str]:
    """``{"seam": center|edge, "fold": center|edge}`` of an alias or an ``{axis: position}`` mapping."""
    if isinstance(pivot, str):
        return dict(_PIVOT_ALIASES[pivot.lower()])
    roles = {}
    for axname, position in pivot.items():
        if axname == fold_axis:
            roles["fold"] = _position_kind(position)
        elif axname == seam_axis:
            roles["seam"] = _position_kind(position)
        else:
            raise ValueError(
                f"Fold pivot axis {axname!r} is neither the fold axis {fold_axis!r} nor the seam axis {seam_axis!r}."
            )
    roles.setdefault("seam", "center")
    roles.setdefault("fold", "center")
    return roles


def fold_edges(grid, ax_name: str, ax_padding, hi: int):
    """How an axis is padded with respect to a north fold: ``(north folds, boundary mode of the other edges)``.

    On a fold axis the north edge folds whenever it is padded (``hi > 0``), whatever the per-call
    ``padding`` says; a per-call string only sets the south edge, which otherwise takes the spec's
    ``south`` mode (reference padding.py:744-757).  Every fast path that picks itself from the padding
    value asks this first.  Other axes: ``(False, ax_padding)``."""
    info = grid._folds.get(ax_name)
    if info is None:
        return False, ax_padding
    return hi > 0, (ax_padding if isinstance(ax_padding, str) else info["south"])


def _fold_plan(grid, fold_axis: str, dims, shape, width: int):
    """(fold dim number, seam dim number, skip, mirror, period) of the north halo of a field with ``dims``."""
    info = grid._folds[fold_axis]
    seam_axis = info["seam_axis"]
    roles = _resolve_pivot(info["pivot"], fold_axis, seam_axis)
    probe = DataArray.__new__(DataArray)
    probe._dims = tuple(dims)
    fold_pos, fold_dim = grid.axes[fold_axis]._get_position_name(probe)
    seam_pos, seam_dim = grid.axes[seam_axis]._get_position_name(probe)
    f, s = dims.index(fold_dim), dims.index(seam_dim)
    n = int(shape[f])
    skip = 1 if _position_kind(fold_pos) == roles["fold"] else 0
    if width > n - skip:
        raise ValueError(
            f"North-fold halo width {width} requested on fold axis {fold_axis!r} exceeds the {n - skip} "
            f"interior row(s) available to mirror along {fold_dim!r} (grid length {n}"
            f"{', minus 1 redundant pole row' if skip else ''})."
        )
    two_off, extra = _SEAM_POSITION[seam_pos]
    length = int(shape[s])
    period = length + extra
    mirror = (0 if roles["seam"] == "edge" else 1) - two_off
    # a partner >= length exists only when period > length (inner), hit by k = (mirror - length) mod period
    if period > length and (mirror - length) % period < length:
        raise NotImplementedError(
            f"A {seam_pos!r} seam position is incompatible with a center-type fold pivot (seam role "
            f"{roles['seam']!r}): the mirror about a cell-center pole has no partner on this sublattice. "
            "Use an edge-type pivot, or a center/left/right/outer seam position."
        )
    return f, s, skip, mirror, period


def fold_halo_plane(grid, fold_axis: str, dims, x, pre=None, negate: bool = False):
    """The folded north row of the device tensor ``x`` (dims ``dims``) as a halo plane for ``xg_stencil2``:
    ``x``'s shape with length 1 along the fold dim, ``x * pre`` read at the mirrored cell, sign-flipped
    for vector components.  One ``xg_fold_rows`` launch."""
    from . import ops

    f, s, skip, mirror, period = _fold_plan(grid, fold_axis, tuple(dims), list(x.shape), 1)
    return ops.fold_rows(x, f, s, 1, skip, mirror, period, negate=negate, pre=pre)


def fold_halo_planes(grid, fold_axis: str, dims, x, lo: int, south, pre=None, negate: bool = False):
    """``(halo_lo, halo_hi)`` of a one-cell stencil whose north edge crosses the fold of ``fold_axis``:
    halo_hi is the folded row (:func:`fold_halo_plane`).  A periodic south edge wraps the row above the top,
    which is that same fold row (reference padding.py:723-762), so it is halo_lo too when the stencil pads
    the south edge (``lo``); otherwise halo_lo is None and the boundary condition ``south`` pads that edge."""
    halo_hi = fold_halo_plane(grid, fold_axis, dims, x, pre=pre, negate=negate)
    return (halo_hi if lo and south == "periodic" else None), halo_hi


def _pad_fold(data, grid, padding_width, padding, fill_value):
    """Padding on a grid with a north fold (reference padding.py:687-762), on the device.

    Same order as the reference: the fold halo first, built from the unpadded field (so the seam
    mirror sees the whole periodic row), then the south edge of the fold axis and every other axis
    with the ordinary boundary conditions, on the array that already holds the fold rows — a
    periodic south edge therefore wraps the fold row, and a seam padded in the same call wraps the
    folded rows.  A vector component ``{axis: da}`` changes sign across the fold; it needs no
    partner component (the fold is a point reflection, not a rotation)."""
    from . import ops
    from .device import as_device_tensor, result_like

    if isinstance(data, dict):
        isvector = True
        [da] = list(data.values())
    else:
        isvector, da = False, data
    fold_axes = [ax for ax in padding_width if ax in grid._folds and padding_width[ax][1] > 0]
    if len(fold_axes) > 1:
        raise NotImplementedError(
            f"Padding more than one north-fold axis at once is not supported (got fold axes {sorted(fold_axes)})."
        )
    for fax in fold_axes:
        width = int(padding_width[fax][1])
        dims = tuple(da.dims)
        x, was_host = as_device_tensor(da.data, grid._device_for(da))
        f, s, skip, mirror, period = _fold_plan(grid, fax, dims, list(x.shape), width)
        n = int(x.shape[f])
        out = ops.pad(x, f, 0, width, "fill", 0.0)
        ops.fold_rows(x, f, s, width, skip, mirror, period, negate=isvector, out=out, row0=n)
        da = DataArray(result_like(out, was_host), dims=dims, name=da.name, attrs=da.attrs)
    basic_width, basic_padding = {}, {}
    for ax, widths in padding_width.items():
        if ax in grid._folds:
            basic_width[ax] = (widths[0], 0)
            basic_padding[ax] = fold_edges(grid, ax, padding[ax], 0)[1]
        else:
            basic_width[ax] = widths
            basic_padding[ax] = padding[ax]
    return _pad_basic(da, grid, basic_width, basic_padding, fill_value)


def _strip_all_coords(data):
    """Padding cannot invent coordinate values: drop them all (padding.py:220-227)."""
    if isinstance(data, dict):
        return {k: v.drop_vars(list(v.coords)) for k, v in data.items()}
    return data.drop_vars(list(data.coords))


def missing_boundary_error(ax_name) -> ValueError:
    """The error of an operator that has to pad ``ax_name`` when no boundary condition is set for it."""
    return ValueError(
        f"No boundary condition was specified for axis {ax_name!r}, but the "
        f"requested operation needs to pad it. Set a boundary condition, "
        f"e.g. ``padding='fill'`` (or 'extend'/'periodic'), on the Grid "
        f"(``Grid(..., padding=...)``) or pass ``padding=`` to the "
        f"grid method."
    )


def _pad_basic(da: DataArray, grid, padding_width, padding, fill_value):
    from . import ops
    from .device import as_device_tensor, result_like

    out = da.copy(deep=False)
    for ax, widths in padding_width.items():
        if all(w == 0 for w in widths):
            continue  # padding.py:592-593
        axis = grid.axes[ax]
        _, dim = axis._get_position_name(out)
        ax_padding = padding[ax]
        if ax_padding is None:
            raise missing_boundary_error(ax)
        x, was_host = as_device_tensor(out.data, grid._device_for(out))
        fv = fill_value[ax] if fill_value[ax] is not None else 0.0
        y = ops.pad(x, out.get_axis_num(dim), int(widths[0]), int(widths[1]), ax_padding, fv)
        out = DataArray(result_like(y, was_host), dims=out.dims, name=out.name, attrs=out.attrs)
    return out


def _get_all_connection_axes(connections, facedim):
    all_axes = []
    for c in connections[facedim].values():
        all_axes.extend(list(c.keys()))
    return list(dict.fromkeys(all_axes))


def _infer_vector_component_axis(grid, da) -> str:
    """The axis a bare vector component is aligned with: the only axis on which it is not at
    the cell centre (padding.py:230-257)."""
    edge_axes = []
    for axname, axis in grid.axes.items():
        try:
            position, _ = axis._get_position_name(da)
        except KeyError:
            continue
        if position != "center":
            edge_axes.append(axname)
    if len(edge_axes) == 1:
        return edge_axes[0]
    raise ValueError(
        "Could not unambiguously infer the axis of the vector component being "
        f"padded from its staggered position (edge axes found: {edge_axes}). "
        "Pass the component as a `{axis_name: DataArray}` dict so its "
        "orientation is explicit, e.g. "
        "`pad({'Y': v}, ..., other_component={'X': u})`."
    )


def _contiguous_strides(shape):
    strides, acc = [], 1
    for n in reversed(shape):
        strides.append(acc)
        acc *= int(n)
    return list(reversed(strides))


def broadcast_strides(m_shape, shape):
    """Element strides of a C-contiguous operand of shape ``m_shape`` (1 where it broadcasts) read over ``shape``:
    0 along every dim of extent 1 in either, as the kernels' operands take them."""
    m_strides = _contiguous_strides(m_shape)
    return [0 if int(m) == 1 or int(n) == 1 else st for m, n, st in zip(m_shape, shape, m_strides)]


def _axis_dim(grid, dims, axname):
    for d in grid.axes[axname].coords.values():
        if d in dims:
            return d
    raise KeyError(f"None of the DataArray's dims {dims} were found in axis coords.")


def _source_dim_for(grid, target_dim, s_dims):
    """The source dim a target dim reads from: same name, else the source's dim on the same grid
    axis (padding.py:183-198 renames the partner component's dims this way)."""
    if target_dim in s_dims:
        return target_dim
    for axname in grid.axes:
        positions = list(grid.axes[axname].coords.values())
        if target_dim in positions:
            for d in positions:
                if d in s_dims:
                    return d
    raise ValueError(f"cannot match dimension {target_dim!r} against the source dims {s_dims}")


def _copy_connected_edge(grid, facedim, dst, d_dims, d_shape, face, axname, d_start, width, prepad,
                         connection, is_right, sources, isvector, vectoraxis, batch, cross_pads=None):
    """Write the ``width`` halo cells of one connected edge of ``face`` into ``dst`` (dims
    ``d_dims``, starting at index ``d_start`` along the dim of ``axname``) from the neighbour
    named by ``connection`` (padding.py:414-541): ONE strided copy, appended to ``batch`` (all edges
    of a field go out in one ``xg_strided_copy_batch`` launch).

    ``sources``: {"self": (tensor, dims, shape, strides), "partner": ...}; the source arrays carry
    ``prepad`` halo cells on the sliced dim (the reference slices pre-padded arrays; the operator
    fast path reads the bare field, prepad = 0).  Every dim of ``dst`` other than the face dim and
    the padded one is copied over its full extent, which must match the source's.

    ``cross_pads`` (with prepad = 0): ``{dst dim: (lo, hi)}`` for ONE other dim of ``dst`` that is
    itself padded.  The reference takes the rim from the PRE-PADDED neighbour, so along that dim the
    slab continues into the neighbour's own basic halo (fill constant / edge cell / wrapped cells,
    ``cross_pads["modes"][axis] = (mode, fill value)``): those corner blocks are written by extra
    strided copies with zero or wrapped source strides.
    """
    source_face, source_axis, reverse = connection
    swap_axis = axname != source_axis
    s, s_dims, s_shape, s_strides = sources["partner" if (isvector and swap_axis) else "self"]
    # positional face index like the reference's isel
    if source_face < 0 or source_face >= s_shape[s_dims.index(facedim)]:
        raise IndexError(f"face {source_face} is not a valid index for {facedim!r}")
    d_strides = _contiguous_strides(d_shape)
    target_dim = _axis_dim(grid, d_dims, axname)
    loop_dims = [d for d in d_dims if d != facedim]
    shape = [width if d == target_dim else d_shape[d_dims.index(d)] for d in loop_dims]
    dst_strides = [d_strides[d_dims.index(d)] for d in loop_dims]
    dst_offset = face * d_strides[d_dims.index(facedim)] + d_start * d_strides[d_dims.index(target_dim)]

    src_offset = source_face * s_strides[s_dims.index(facedim)]
    src_strides = []
    if swap_axis:
        cross_dim = _axis_dim(grid, d_dims, source_axis)        # target dim along the seam
        s_sliced = _source_dim_for(grid, cross_dim, s_dims)    # source dim along source_axis
        s_along = _source_dim_for(grid, target_dim, s_dims)    # source dim along axname
    else:
        cross_dim = None
        s_sliced = _source_dim_for(grid, target_dim, s_dims)
        s_along = None
    s_len = s_shape[s_dims.index(s_sliced)]
    if is_right:  # padding.py:443-459: the neighbour's first cells, or its last ones if reversed
        s0 = s_len - prepad - width if reverse else prepad
    else:
        s0 = prepad if reverse else s_len - prepad - width
    negate = isvector and (
        (reverse and vectoraxis == axname) or (swap_axis and not reverse and vectoraxis != axname)
    )
    # per loop dim: segments (dst start, length, src start, src stride, constant or None)
    per_dim = []
    for d, n in zip(loop_dims, shape):
        if d == target_dim:
            st = s_strides[s_dims.index(s_sliced)]
            if reverse:  # flip across the seam (padding.py:478-487)
                per_dim.append([(0, n, (s0 + width - 1) * st, -st, None)])
            else:
                per_dim.append([(0, n, s0 * st, st, None)])
            continue
        lo_d, hi_d = (cross_pads or {}).get(d, (0, 0))
        n_in = n - lo_d - hi_d
        if swap_axis and d == cross_dim:
            sd, flip, src_axis_name = s_along, not reverse, axname  # flip along the seam (padding.py:489-498)
            if s_shape[s_dims.index(sd)] != n_in:
                raise ValueError(
                    "a face connection that swaps axes needs faces of equal size along "
                    f"{axname!r} and {source_axis!r}"
                )
        else:
            sd, flip = _source_dim_for(grid, d, s_dims), False
            src_axis_name = next((ax for ax in grid.axes if sd in grid.axes[ax].coords.values()), None)
            if s_shape[s_dims.index(sd)] != n_in:
                raise ValueError(f"dimension {d!r} differs between connected arrays")
        st = s_strides[s_dims.index(sd)]
        segs = [(lo_d, n_in, (n_in - 1) * st if flip else 0, -st if flip else st, None)]
        if lo_d or hi_d:
            mode, fv = cross_pads["modes"][src_axis_name]
            for length, lower in ((lo_d, True), (hi_d, False)):
                if not length:
                    continue
                dst0 = 0 if lower else lo_d + n_in
                # the neighbour's halo this dst halo reads: its lower one, or the upper one if flipped
                src_lower = lower != flip
                if mode == "fill":
                    segs.append((dst0, length, 0, 0, float(fv if fv is not None else 0.0)))
                elif mode == "extend":
                    segs.append((dst0, length, 0 if src_lower else (n_in - 1) * st, 0, None))
                else:  # periodic: the cells at the other end, in dst order
                    if src_lower:   # virtual source index -length .. -1  (or reversed when flipped)
                        first, last = n_in - length, n_in - 1
                    else:           # virtual source index n .. n + length - 1
                        first, last = 0, length - 1
                    # identity walks the virtual index upwards; the flip walks it downwards
                    if flip:
                        # dst lower halo (D = -length..-1) -> u = n-1-D = n-1+length .. n  -> wrapped: length-1 .. 0
                        # dst upper halo (D = n..n+length-1) -> u = -1 .. -length -> wrapped: n-1 .. n-length
                        segs.append((dst0, length, last * st, -st, None))
                    else:
                        segs.append((dst0, length, first * st, st, None))
        per_dim.append(segs)
    import itertools

    for combo in itertools.product(*per_dim):
        const = [c[4] for c in combo if c[4] is not None]
        sub_shape = [c[1] for c in combo]
        d_off = dst_offset + sum(c[0] * ds for c, ds in zip(combo, dst_strides))
        if const:
            cval = cross_pads["const"](const[0])
            batch.append((dst, d_off, dst_strides, cval, 0, [0] * len(sub_shape), sub_shape, negate))
        else:
            s_off = src_offset + sum(c[2] for c in combo)
            batch.append((dst, d_off, dst_strides, s, s_off, [c[3] for c in combo], sub_shape, negate))


def _unpack_vector(grid, da, other_component):
    """(field, is vector, its axis, partner component) — padding.py:277-303."""
    if isinstance(da, dict):
        vectoraxis, da = dict(da).popitem()
        isvector = True
    elif other_component is not None:
        isvector = True
        vectoraxis = _infer_vector_component_axis(grid, da)
    else:
        return da, False, None, None
    if other_component is None:
        raise ValueError("Padding vector components requires `other_component` input.")
    _, da_partner = dict(other_component).popitem()
    return da, isvector, vectoraxis, da_partner


def _require_connected_edges(grid, ax_name, lo, hi, n_face, face_offset=0):
    """Raise when a halo of ``lo`` / ``hi`` cells along ``ax_name`` pads an edge without a face connection on one
    of the faces ``face_offset .. face_offset + n_face - 1``: the caller has no boundary condition for such edges."""
    face_links = grid._face_connections[grid._facedim]
    for side, w in ((0, lo), (1, hi)):
        if not w:
            continue
        unconnected = [face_offset + i for i in range(n_face)
                       if face_links.get(face_offset + i, {}).get(ax_name, (None, None))[side] is None]
        if unconnected:
            raise ValueError(
                f"No boundary condition was specified for axis {ax_name!r}, "
                f"but the requested operation needs to pad the {'right' if side else 'left'} "
                f"edge of face(s) {unconnected}, which have no face "
                f"connection there. Set a boundary condition, e.g. "
                f"``padding='fill'`` (or 'extend'/'periodic'), on the Grid "
                f"(``Grid(..., padding=...)``) or pass ``padding=`` to the "
                f"grid method."
            )


def _connection_sources(da, partner, x):
    """The ``sources`` of :func:`_copy_connected_edge`: ``"self"``, the field ``da`` as the device tensor ``x``, and
    for a vector component (``partner`` not None) ``"partner"``, the other component on ``x``'s device in its dtype."""
    from .device import as_device_tensor

    sources = {"self": (x, tuple(da.dims), [int(v) for v in x.shape], _contiguous_strides(x.shape))}
    if partner is not None:
        q = as_device_tensor(partner.data, x.device)[0].to(x.dtype)
        sources["partner"] = (q, tuple(partner.dims), [int(v) for v in q.shape], _contiguous_strides(q.shape))
    return sources


def connected_edge_mode(grid, ax_name, lo, hi, padding, fill_value, n_face, face_offset=0):
    """``(mode, fill value)`` of the unconnected edges of ``ax_name`` on a grid with face connections, after
    the same validation the simply connected path performs in ``ops.stencil2`` / ``_apply_fused_stencil``."""
    paddings = grid._complete_user_kwargs_using_axis_defaults(padding, "padding")
    fills = grid._complete_user_kwargs_using_axis_defaults(fill_value, "fill_value")
    ax_padding = paddings[ax_name]
    # an unknown string must not silently become a periodic halo on the unconnected edges
    if isinstance(ax_padding, Mapping):
        raise NotImplementedError(
            "fold / per-side padding mappings are not supported on grids with face connections"
        )
    if ax_padding not in (None, "periodic", "fill", "extend"):
        if ax_padding == "extrapolate":
            raise NotImplementedError(
                "padding='extrapolate' (an opt-in extension without a reference counterpart) is not available "
                "for operators on grids with face connections; use fill / extend / periodic"
            )
        raise ValueError(
            f"padding must be one of ['periodic', 'fill', 'extend'] or None, but got {ax_padding!r}"
        )
    if ax_padding is None:
        _require_connected_edges(grid, ax_name, lo, hi, n_face, face_offset)
    fv = fills[ax_name] if fills[ax_name] is not None else 0.0
    return (ax_padding if ax_padding is not None else "fill"), float(fv)


def _connected_edge_plan(grid, ax_name, lo, hi, dims, shape, vectoraxis, partner_layout, face_offset=0,
                        remote_edges=None, self_strides=None):
    """The strided copies that write the neighbour rims of every connected edge into the one-cell halo
    planes of a field with ``dims`` / ``shape`` along ``ax_name``: a list of ``(side, dst offset, dst strides,
    source ("self" or "partner"), src offset, src strides, shape, negate)``, offsets and strides in elements
    of the contiguous plane (``shape`` with extent 1 along the axis) and source arrays.  ``partner_layout``:
    ``(dims, shape)`` of the other vector component, or None for a scalar.

    The index maps depend only on the topology and the array layout, not on the values: they are derived
    once per (axis, widths, layout) and kept on the grid.  ``face_offset`` / ``remote_edges`` as in
    :func:`connected_halo_planes` (such plans are not cached).  ``self_strides``: element strides "self" is read
    with instead of the contiguous ones of ``shape`` -- a metric broadcast against the field, 0 where it
    broadcasts, whose plan replays the field's index maps over the metric's cells."""
    facedim = grid._facedim
    face_links = grid._face_connections[facedim]
    isvector = partner_layout is not None
    cache = grid.__dict__.setdefault("_halo_plan_cache", {})
    self_strides = _contiguous_strides(shape) if self_strides is None else [int(v) for v in self_strides]
    key = (ax_name, lo, hi, tuple(dims), tuple(shape), vectoraxis, partner_layout, tuple(self_strides), face_offset)
    plan = cache.get(key) if remote_edges is None else None
    if plan is not None:
        return plan
    sources = {"self": ("self", tuple(dims), list(shape), self_strides)}
    if isvector:
        p_dims, p_shape = partner_layout
        sources["partner"] = ("partner", tuple(p_dims), list(p_shape), _contiguous_strides(p_shape))
    t = list(dims).index(_axis_dim(grid, dims, ax_name))
    n_face = shape[list(dims).index(facedim)]
    p_shape = list(shape)
    p_shape[t] = 1
    plan = []
    for side, w in ((0, lo), (1, hi)):
        if not w:
            continue
        for i in range(n_face):
            connection = face_links.get(face_offset + i, {}).get(ax_name, (None, None))[side]
            if not connection:
                continue
            src_local = connection[0] - face_offset
            if remote_edges is not None and not 0 <= src_local < n_face:
                remote_edges.append((side, i, connection))
                continue
            _copy_connected_edge(grid, facedim, side, tuple(dims), p_shape, i, ax_name, 0, 1, 0,
                                 (src_local,) + tuple(connection[1:]), bool(side), sources, isvector,
                                 vectoraxis, plan)
    if remote_edges is None:
        cache[key] = plan
    return plan


def connected_halo_program(grid, ax_name, lo, hi, dims, shape, mode, vectoraxis=None, partner_layout=None,
                           pre_strides=None, face_offset=0, remote_edges=None):
    """Every strided copy that builds the one-cell halo planes of a field with ``dims`` / ``shape`` along
    ``ax_name``: the neighbour rims of :func:`_connected_edge_plan` plus, on each face without a connection on a
    padded side, the basic boundary value (``mode``: fill from the constant, source ``"fill"``; extend: the
    nearest row; periodic: the row at the other end).  Each face's plane is written by exactly one copy.
    :func:`connected_halo_planes` runs the list on device tensors; the host slab pipeline
    (``xg_stencil2_host_connected``) replays it on each slab.

    ``pre_strides``: the element strides of a pre-metric read over ``shape`` (:func:`broadcast_strides`).  Each
    copy then also carries ``(pre offset, pre strides)``, the metric cells under the field cells it reads (the
    same index map over the metric; offset 0, strides 0 for a fill copy, whose weight is 1), for
    ``xg_stencil2_host_connected_weighted``: the halo of ``x * pre``.

    ``face_offset`` / ``remote_edges`` as in :func:`connected_halo_planes`: an edge whose neighbour lives in
    another block of faces gets no copy.  The program is kept on the grid, except when ``remote_edges`` is given."""
    cache = grid.__dict__.setdefault("_halo_program_cache", {})
    key = (ax_name, lo, hi, tuple(dims), tuple(shape), mode, vectoraxis, partner_layout,
           None if pre_strides is None else tuple(int(v) for v in pre_strides), face_offset)
    if remote_edges is None and key in cache:
        return cache[key]
    facedim = grid._facedim
    face_links = grid._face_connections[facedim]
    dims = tuple(dims)
    t = dims.index(_axis_dim(grid, dims, ax_name))
    f = dims.index(facedim)
    n = shape[t]
    strides = _contiguous_strides(shape)
    p_shape = list(shape)
    p_shape[t] = 1
    p_strides = _contiguous_strides(p_shape)
    loop = [d for d in range(len(dims)) if d != f]
    program = list(_connected_edge_plan(grid, ax_name, lo, hi, dims, shape, vectoraxis, partner_layout,
                                        face_offset, remote_edges))
    if pre_strides is not None:
        ms = [int(v) for v in pre_strides]
        weights = _connected_edge_plan(grid, ax_name, lo, hi, dims, shape, vectoraxis, partner_layout, face_offset,
                                       None if remote_edges is None else [], self_strides=ms)
        program = [c + (w[4], w[5]) for c, w in zip(program, weights)]
    for side, w in ((0, lo), (1, hi)):
        if not w:
            continue
        for i in range(shape[f]):
            if face_links.get(face_offset + i, {}).get(ax_name, (None, None))[side] is not None:
                continue
            c_shape = [p_shape[d] for d in loop]
            dst = (side, i * p_strides[f], [p_strides[d] for d in loop])
            if mode == "fill":
                copy = dst + ("fill", 0, [0] * len(loop), c_shape, False)
                weight = (0, [0] * len(loop))
            else:
                row = ((n - 1) if side else 0) if mode == "extend" else (0 if side else (n - 1))
                copy = dst + ("self", i * strides[f] + row * strides[t], [strides[d] for d in loop], c_shape, False)
                if pre_strides is not None:
                    weight = (i * ms[f] + row * ms[t], [ms[d] for d in loop])
            program.append(copy if pre_strides is None else copy + weight)
    if remote_edges is None:
        cache[key] = program
    return program


def connected_halo_planes(da, grid, ax_name, lo, hi, padding, fill_value, other_component=None,
                          face_offset=0, remote_edges=None, pre=None):
    """The one-cell halo planes of ``da`` along ``ax_name`` on a grid with face connections, for
    the fused stencil kernel (``xg_stencil2`` takes them as ``halo_lo`` / ``halo_hi``).

    Equals the first / last plane of ``pad(da, {ax_name: (lo, hi)})`` — basic boundary values on
    unconnected edges, the neighbour's rim (rotated, flipped, sign-flipped) on connected ones —
    without materialising the padded field: the planes are thin, so an operator on a connected
    grid costs one read and one write of the field like on a simple one.  Returns
    ``(field tensor, halo_lo or None, halo_hi or None, was_host, dims)``.

    ``face_offset`` / ``remote_edges``: ``da`` holds the contiguous block of faces that starts at
    global face ``face_offset`` (faces sharded across GPUs, ``parallel.sharded_connected_stencil2``);
    edges whose neighbour lives in another block are not filled here but appended to
    ``remote_edges`` as ``(side, local face, connection)``.

    ``pre`` (a device tensor that broadcasts against the scalar field, 1 where it broadcasts): the planes are
    those of ``x * pre``, the halo of a metric-weighted operator, whose fused stencil then takes ``pre`` for the
    interior cells.  The same copies run over the metric into weight planes (1 on a fill edge, which stays the
    bare fill value, as the reference pads the already weighted array); one ``xg_binary`` launch multiplies the
    two, so each halo cell is the gathered ``x`` times the gathered metric, rounded once in the field's dtype.

    The copies of :func:`connected_halo_program` (and their weight copies) go out in one
    ``xg_strided_copy_batch`` launch.
    """
    import torch

    from . import ops
    from .device import as_device_constant, as_device_tensor

    da, isvector, vectoraxis, da_partner = _unpack_vector(grid, da, other_component)
    x, was_host = as_device_tensor(da.data, grid._device_for(da))
    dims = tuple(da.dims)
    shape = [int(v) for v in x.shape]
    sources = _connection_sources(da, da_partner, x)
    mode, fv = connected_edge_mode(grid, ax_name, lo, hi, padding, fill_value, shape[dims.index(grid._facedim)],
                                   face_offset)
    partner_layout = None if not isvector else (sources["partner"][1], tuple(sources["partner"][2]))
    pre_strides = None
    if pre is not None:
        if isvector:
            raise NotImplementedError(
                "metric weighting of vector components across face connections is not implemented")
        m = pre.to(x.dtype).contiguous()
        pre_strides = broadcast_strides(list(m.shape), shape)
    program = connected_halo_program(grid, ax_name, lo, hi, dims, shape, mode, vectoraxis, partner_layout,
                                     pre_strides, face_offset, remote_edges)
    p_shape = list(shape)
    p_shape[dims.index(_axis_dim(grid, dims, ax_name))] = 1
    sides = [side for side, w in ((0, lo), (1, hi)) if w]
    # the x planes, then the weight planes side by side: one product over both at the end
    stack = torch.empty([len(sides) * (1 if pre is None else 2)] + p_shape, dtype=x.dtype, device=x.device)
    planes = {side: stack[k] for k, side in enumerate(sides)}
    tensors = {key: src[0] for key, src in sources.items()}
    if any(c[3] == "fill" for c in program):  # the fill value, then the weight of a fill edge
        tensors["fill"] = as_device_constant(torch.tensor([fv, 1.0], dtype=x.dtype).numpy(), x.device)
    batch = [(planes[side], doff, dstr, tensors[src], soff, sstr, shp, neg)
             for side, doff, dstr, src, soff, sstr, shp, neg, *_ in program]
    if pre is not None:  # the same index maps over the metric's cells
        batch += [(stack[len(sides) + sides.index(side)], doff, dstr, tensors["fill"] if src == "fill" else m,
                   1 if src == "fill" else poff, pstr, shp, False)
                  for side, doff, dstr, src, _, _, shp, _, poff, pstr in program]
    ops.strided_copy_batch(batch)
    if pre is not None and sides:
        weighted = ops.binary("mul", stack[:len(sides)], stack[len(sides):])
        planes = {side: weighted[k] for k, side in enumerate(sides)}
    return x, planes.get(0), planes.get(1), was_host, dims


def _pad_face_connections(da, grid, padding_width, padding, fill_value, other_component=None):
    """Padding across face connections (padding.py:260-572), on the device.

    Same steps as the reference: (1) pad every face on every connection axis to the largest
    requested width with the ordinary boundary condition, (2) overwrite the halo of each
    CONNECTED edge with the neighbour's rim, always read from the pre-padded arrays, (3) trim
    back to the requested widths.  Step 2 is one batched strided-copy launch per axis.  When
    one or two axes are padded the three steps collapse into ``xg_pad`` + one batched copy per axis.

    The reference visits the axes in ``set`` order (hash-seed dependent, padding.py:307-309);
    only halo corners depend on it.  Here the order is that of ``grid.axes``.
    """
    from . import ops
    from .device import as_device_tensor, result_like

    facedim = grid._facedim
    connections = grid._face_connections
    if connections is None:
        raise ValueError("Grid connections cannot be None")
    if facedim is None:
        raise ValueError("Face dimension cannot be None")

    da, isvector, vectoraxis, da_partner = _unpack_vector(grid, da, other_component)
    if isvector:
        da_partner = _strip_all_coords(da_partner)

    wanted = set(_get_all_connection_axes(connections, facedim)) | set(padding_width.keys())
    pad_axes = [ax for ax in grid.axes if ax in wanted] + [ax for ax in wanted if ax not in grid.axes]
    padding_width = {ax: tuple(padding_width.get(ax, (0, 0))) for ax in pad_axes}
    width = max(max(w) for w in padding_width.values())
    max_padding_width = {ax: (width, width) for ax in pad_axes}

    n_facedim = da.sizes[facedim]
    face_links = connections[facedim]
    prepad_padding = dict(padding)
    for axname in pad_axes:
        if prepad_padding.get(axname) is None:
            _require_connected_edges(grid, axname, *padding_width[axname], n_facedim)
            # every padded edge of this axis is connected: its pre-padded halo is a placeholder
            prepad_padding[axname] = "fill"

    active = [ax for ax in pad_axes if any(padding_width[ax])]
    if len(active) in (1, 2):
        # One padded axis (every built-in operator, most user ufuncs) or two (2-D stencils of user ufuncs): no
        # pre-padded copies.  Basic-pad the padded axes straight into the final shape (one pass); then, axis by
        # axis in the reference's order, overwrite the connected halos from the UNPADDED neighbours.  With two
        # axes each halo slab spans the FULL extent of the other axis -- its corner blocks are the neighbour's
        # own basic halo (what the reference finds in the pre-padded neighbour), produced by zero-stride /
        # wrapped strided copies.  Same values as the general route below, two passes over the field instead
        # of five.
        import torch

        padded = _pad_basic(da, grid, {ax: padding_width[ax] for ax in active}, prepad_padding, fill_value)
        out, was_host = as_device_tensor(padded.data, grid._device_for(padded))  # fresh: xg_pad allocated it
        o_dims = tuple(padded.dims)
        o_shape = [int(v) for v in out.shape]
        x, _ = as_device_tensor(da.data, out.device)
        sources = _connection_sources(da, da_partner, x)
        consts = {}

        def const(value):
            key = repr(float(value))
            if key not in consts:
                consts[key] = torch.full((1,), float(value), dtype=out.dtype, device=out.device)
            return consts[key]

        modes = {ax: (prepad_padding[ax], fill_value.get(ax)) for ax in pad_axes}
        for ax in active:
            other = next((a for a in active if a != ax), None)
            cross = None if other is None else {_axis_dim(grid, o_dims, other): padding_width[other], "modes": modes,
                                                "const": const}
            lo, hi = padding_width[ax]
            t_len = o_shape[o_dims.index(_axis_dim(grid, o_dims, ax))]
            batch = []
            for i in range(n_facedim):
                links = face_links.get(i, {}).get(ax, (None, None))
                for connection, is_right, w in ((links[0], False, lo), (links[1], True, hi)):
                    if connection and w:
                        _copy_connected_edge(grid, facedim, out, o_dims, o_shape, i, ax, (t_len - w) if is_right else 0,
                                             w, 0, connection, is_right, sources, isvector, vectoraxis, batch,
                                             cross_pads=cross)
            ops.strided_copy_batch(batch)  # the second axis overwrites the corners, like the reference
        return DataArray(result_like(out, was_host), dims=o_dims, name=padded.name, attrs=padded.attrs)

    prepadded = _pad_basic(da, grid, max_padding_width, prepad_padding, fill_value)
    p, was_host = as_device_tensor(prepadded.data, grid._device_for(prepadded))
    p_dims = tuple(prepadded.dims)
    p_shape = [int(v) for v in p.shape]
    p_strides = _contiguous_strides(p_shape)
    partner = _pad_basic(da_partner, grid, max_padding_width, prepad_padding, fill_value) if isvector else None
    sources = _connection_sources(prepadded, partner, p)

    out = p.clone()
    face_pos = p_dims.index(facedim)

    by_axis = {}
    if width > 0:
        for i in range(n_facedim):
            connection_single = face_links.get(i, {})
            for axname in pad_axes:
                left_connection, right_connection = connection_single.get(axname, (None, None))
                target_dim = _axis_dim(grid, p_dims, axname)
                t_len = p_shape[p_dims.index(target_dim)]
                for connection, is_right in [(left_connection, False), (right_connection, True)]:
                    if not connection:
                        continue
                    _copy_connected_edge(
                        grid, facedim, out, p_dims, p_shape, i, axname,
                        (t_len - width) if is_right else 0, width, width, connection, is_right,
                        sources, isvector, vectoraxis, by_axis.setdefault(axname, []),
                    )
    # Edges only read the pre-padded arrays and, halo corners aside, write disjoint cells; corner
    # cells are written by both axes, so the axes go out in order (one launch each).
    for axname in pad_axes:
        ops.strided_copy_batch(by_axis.get(axname, []))

    # trim back to the requested widths (padding.py:557-572)
    starts, final_shape = [], []
    for d, n in zip(p_dims, p_shape):
        lo_cut = hi_cut = 0
        for axname in pad_axes:
            if d in grid.axes[axname].coords.values():
                lo_cut = width - padding_width[axname][0]
                hi_cut = width - padding_width[axname][1]
        starts.append(lo_cut)
        final_shape.append(n - lo_cut - hi_cut)
    if any(starts) or final_shape != p_shape:
        trimmed = out.new_empty(final_shape)
        offset = sum(st * k for st, k in zip(p_strides, starts))
        ops.strided_copy(trimmed, 0, _contiguous_strides(final_shape), out, offset, p_strides, final_shape)
        out = trimmed
    return DataArray(result_like(out, was_host), dims=p_dims, name=prepadded.name, attrs=prepadded.attrs)


def pad(
    data: Union[DataArray, Dict[str, DataArray]],
    grid,
    padding_width: Optional[Dict[str, Tuple[int, int]]],
    padding: Optional[Union[str, Mapping[str, str]]] = None,
    fill_value: Optional[Union[float, Mapping[str, float]]] = None,
    other_component: Optional[Dict[str, DataArray]] = None,
    **kwargs,
):
    """Pad ``data`` along the given grid axes according to the boundary conditions."""
    if "boundary" in kwargs:
        raise ValueError(
            "Argument 'boundary' has been renamed to 'padding'. Please use 'padding' instead."
        )
    if "boundary_width" in kwargs:
        raise ValueError(
            "Argument 'boundary_width' has been renamed to 'padding_width'. "
            "Please use 'padding_width' instead."
        )
    padding = grid._complete_user_kwargs_using_axis_defaults(padding, "padding")
    fill_value = grid._complete_user_kwargs_using_axis_defaults(fill_value, "fill_value")

    if padding_width is None or all(tuple(w) == (0, 0) for w in padding_width.values()):
        return data  # padding.py:831-836

    data = _strip_all_coords(data)
    if grid._face_connections is not None:
        return _pad_face_connections(
            data, grid, padding_width, padding, fill_value, other_component=other_component
        )
    if grid._folds and any(ax in grid._folds for ax in padding_width):
        return _pad_fold(data, grid, padding_width, padding, fill_value)
    if isinstance(data, dict):
        [data] = list(data.values())
    return _pad_basic(data, grid, padding_width, padding, fill_value)
