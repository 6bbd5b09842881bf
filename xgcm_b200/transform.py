"""``Grid.transform``: 1-D coordinate transformation along an axis.

Mid-level logic (argument checks, target parsing, naming, output dim order)
follows the reference's ``xgcm/transform.py:279-514``; the per-column numerics
(``_interp_1d_linear``, transform.py:15-41, a numba CPU gufunc in the reference)
run in the ``xg_vinterp_linear`` CUDA kernel; ``method="conservative"``
(transform.py:88-191, 252-276) runs in ``xg_vinterp_conservative``.
"""

from __future__ import annotations

import warnings

import numpy as np

from .labeled import DataArray


def interp_1d_linear(phi, theta, target_theta_levels, mask_edges=False, bypass_checks=False,
                     logarithmic=False):
    """Array-level entry point with the reference's signature (transform.py:44-85):
    ``phi[..., n], theta[..., n], target[m] -> [..., m]`` along the LAST axis.
    numpy in -> numpy out (through the GPU); CUDA tensors stay on the device."""
    from . import ops
    from .device import as_device_tensor, result_like

    p, host = as_device_tensor(phi)
    th, _ = as_device_tensor(theta, p.device)
    tg, _ = as_device_tensor(target_theta_levels, p.device)
    if th.dim() < p.dim():
        th = th.reshape((1,) * (p.dim() - th.dim()) + tuple(th.shape))
    out = ops.vinterp_linear(p, th, tg, -1, mask_edges, bypass_checks, logarithmic)
    return result_like(out, host)


def linear_interpolation(phi, theta, target_theta_levels, phi_dim, theta_dim, target_dim,
                         mask_edges=True, bypass_checks=False, logarithmic=False, suffix="",
                         grid=None):
    """Labelled wrapper (transform.py:197-249): broadcast dims by name, new dim LAST.

    ``target_theta_levels`` may be 1-D (shared levels) or carry extra dims (one level vector per
    column, e.g. terrain-following target depths); dims it has that ``phi`` lacks become
    broadcast dims of the output, like ``xr.apply_ufunc`` does.
    """
    from . import ops
    from .device import as_device_constant, as_device_tensor, result_like

    if theta_dim not in theta.dims:
        raise ValueError(f"`target_data` must have the dimension {theta_dim!r} of the transform axis")
    if target_dim not in target_theta_levels.dims:
        raise ValueError(
            f"The specified `target_dim` {target_dim} is not within the dimensions of the target: [{target_theta_levels.dims}]."
        )
    device = grid._device_for(phi) if grid is not None else None
    # theta dims other than the core dim must already be dims of phi
    extra = [d for d in theta.dims if d not in phi.dims and d != theta_dim]
    if extra:
        raise ValueError(f"target data has dimensions {extra} that the data does not have")
    tgt_other = [d for d in target_theta_levels.dims if d != target_dim]
    if (not phi.is_device and not tgt_other and not theta.is_device
            and np.asarray(phi.data).dtype in (np.float32, np.float64)):
        # numpy-backed field, shared target levels: slabs of a non-operated dim stream through the GPU
        # (xg_vinterp_linear_host: H2D || kernel || D2H) instead of one upload + one download
        th_dims = [d if d != theta_dim else phi_dim for d in theta.dims]
        th = np.asarray(theta.values)
        present = [d for d in phi.dims if d in th_dims]
        perm = [th_dims.index(d) for d in present]
        if perm != list(range(len(perm))):
            th = np.transpose(th, perm)
        sizes = dict(zip(th_dims, theta.shape))
        if sizes[phi_dim] != phi.sizes[phi_dim]:
            raise ValueError(
                f"conflicting sizes for dimension {phi_dim!r}: {phi.sizes[phi_dim]} on the data, "
                f"{sizes[phi_dim]} on the target data"
            )
        th = th.reshape([sizes[d] if d in th_dims else 1 for d in phi.dims])
        out = ops.vinterp_linear_host(np.asarray(phi.data), th, np.asarray(target_theta_levels.values),
                                      phi.get_axis_num(phi_dim), mask_edges, bypass_checks, logarithmic,
                                      device=None if grid is None else grid._host_device(phi))
        out_dims = tuple(d for d in phi.dims if d != phi_dim) + (target_dim,)
        coords = {k: c for k, c in phi.coords.items()
                  if phi_dim not in c.dims and k != target_dim and all(d in out_dims for d in c.dims)}
        for k, c in target_theta_levels.coords.items():
            if all(d in out_dims for d in c.dims):
                coords[k] = c
        res = DataArray(out, dims=out_dims, coords=coords)
        if phi.name:
            res.name = phi.name + suffix
        return res
    x, host = as_device_tensor(phi.data, device)
    new_dims = [d for d in tgt_other if d not in phi.dims]
    for d in tgt_other:
        if d in phi.dims and phi.sizes[d] != target_theta_levels.sizes[d]:
            raise ValueError(f"conflicting sizes for dimension {d!r} between the data and the target")
    work_dims = list(phi.dims) + new_dims  # phi gains broadcast dims the target introduces
    if new_dims:
        shape = list(x.shape) + [target_theta_levels.sizes[d] for d in new_dims]
        x = x.reshape(list(x.shape) + [1] * len(new_dims)).expand(shape).contiguous()
    axis_num = work_dims.index(phi_dim)
    # theta -> tensor broadcastable against the working dims
    th_dims = [d if d != theta_dim else phi_dim for d in theta.dims]
    th_t = as_device_constant(theta.data, x.device)  # read-only: the 1-D coordinate is uploaded once per content
    present = [d for d in work_dims if d in th_dims]
    perm = [th_dims.index(d) for d in present]
    if perm != list(range(len(perm))):
        th_t = th_t.permute(*perm)
    sizes = dict(zip(th_dims, theta.shape))
    if sizes[phi_dim] != phi.sizes[phi_dim]:
        raise ValueError(
            f"conflicting sizes for dimension {phi_dim!r}: {phi.sizes[phi_dim]} on the data, "
            f"{sizes[phi_dim]} on the target data"
        )
    th_t = th_t.reshape([sizes[d] if d in th_dims else 1 for d in work_dims])
    # target -> (column dims..., m)
    col_dims = [d for d in work_dims if d != phi_dim]
    tg_t = as_device_constant(target_theta_levels.data, x.device)
    if tgt_other:
        tdims = list(target_theta_levels.dims)
        order = [d for d in col_dims if d in tdims] + [target_dim]
        perm = [tdims.index(d) for d in order]
        if perm != list(range(len(perm))):
            tg_t = tg_t.permute(*perm)
        tsz = target_theta_levels.sizes
        tg_t = tg_t.reshape([tsz[d] if d in tdims else 1 for d in col_dims] + [tsz[target_dim]])
    out = ops.vinterp_linear(x, th_t, tg_t, axis_num, mask_edges, bypass_checks, logarithmic)
    out_dims = tuple(col_dims) + (target_dim,)
    # like xr.apply_ufunc with exclude_dims: nothing that lives on the consumed core dim survives
    coords = {k: c for k, c in phi.coords.items()
              if phi_dim not in c.dims and k != target_dim and all(d in out_dims for d in c.dims)}
    for k, c in target_theta_levels.coords.items():
        if all(d in out_dims for d in c.dims):
            coords[k] = c
    res = DataArray(result_like(out, host), dims=out_dims, coords=coords)
    if phi.name:
        res.name = phi.name + suffix
    return res


def interp_1d_conservative(phi, theta, target_theta_bins):
    """Array-level entry point with the reference's signature (transform.py:145-191):
    ``phi[..., n], theta[..., n+1], bins[m] -> [..., m-1]`` along the LAST axis.
    numpy in -> numpy out (slabs streamed through the GPU); CUDA tensors stay on the device."""
    from . import ops
    from .device import as_device_tensor, result_like
    from .labeled import is_device_array

    if not any(is_device_array(a) for a in (phi, theta, target_theta_bins)) and _cuda_device() is not None:
        p, th, tb = np.asarray(phi), np.asarray(theta), np.asarray(target_theta_bins)
        if p.shape[-1] != th.shape[-1] - 1:
            raise AssertionError("phi needs one value per cell: phi.shape[-1] == theta.shape[-1] - 1")
        if tb.ndim != 1:
            raise AssertionError("target_theta_bins must be 1-D")
        return ops.vinterp_conservative_host(p, th, tb, -1)
    p, host = as_device_tensor(phi)
    th, _ = as_device_tensor(theta, p.device)
    tb, _ = as_device_tensor(target_theta_bins, p.device)
    if p.shape[-1] != th.shape[-1] - 1:
        raise AssertionError("phi needs one value per cell: phi.shape[-1] == theta.shape[-1] - 1")
    if tb.dim() != 1:
        raise AssertionError("target_theta_bins must be 1-D")
    if th.dim() < p.dim():
        th = th.reshape((1,) * (p.dim() - th.dim()) + tuple(th.shape))
    return result_like(ops.vinterp_conservative(p, th, tb, -1), host)


def _cuda_device(phi=None, grid=None):
    """The CUDA device a call on ``phi`` runs on, or None without one (the device route then raises its own error)."""
    from . import device as _device

    try:
        dev = grid._device_for(phi) if grid is not None else _device.default_device()
    except RuntimeError:
        return None
    return dev if dev.type == "cuda" else None


def _conservative_host_device(phi, theta, target_theta_levels, grid):
    """The CUDA device through which ``xg_vinterp_conservative_host`` streams a numpy-backed remap, or None when
    the device route applies: device or mixed inputs, a field that is not f32 / f64, no CUDA device."""
    if (phi.is_device or theta.is_device or target_theta_levels.is_device
            or np.asarray(phi.data).dtype not in (np.float32, np.float64)):
        return None
    return _cuda_device(phi, grid)


def conservative_interpolation(phi, theta, target_theta_levels, phi_dim, theta_dim, target_dim,
                               suffix="", grid=None):
    """Labelled wrapper (transform.py:252-276): bins along ``target_dim`` (one fewer than the
    levels), coordinate = bin centres."""
    return _conservative_interpolation(phi, theta, target_theta_levels, phi_dim, theta_dim, target_dim, suffix,
                                       grid)


def _conservative_interpolation(phi, theta, target_theta_levels, phi_dim, theta_dim, target_dim, suffix="",
                                grid=None, theta_at_centers=False):
    """:func:`conservative_interpolation`; with ``theta_at_centers`` (numpy inputs only) ``theta`` holds the n cell
    centres along ``theta_dim`` and the remap uses the bounds ``grid.interp(theta, axis, padding="extend")`` gives,
    made slab by slab on the device."""
    from . import ops
    from .device import as_device_tensor, result_like

    if theta_dim not in theta.dims:
        raise ValueError(f"`target_data` must have the cell-bounds dimension {theta_dim!r}")
    if target_theta_levels.ndim != 1:
        raise NotImplementedError(
            "Conservative transformation is not yet supported for multi-dimensional targets."
        )
    host_dev = _conservative_host_device(phi, theta, target_theta_levels, grid)
    if theta_at_centers and host_dev is None:
        raise ValueError("theta at cell centres is taken by the host route only (numpy inputs, a CUDA device)")
    extra = [d for d in theta.dims if d not in phi.dims and d != theta_dim]
    if host_dev is not None:
        # numpy-backed fields: slabs of phi (and of a full theta field) stream through the GPU
        # (xg_vinterp_conservative_host: H2D || kernel || D2H) instead of one upload + one download
        if extra:
            raise ValueError(f"target data has dimensions {extra} that the data does not have")
        th_dims = [d if d != theta_dim else phi_dim for d in theta.dims]
        th = np.asarray(theta.values)
        present = [d for d in phi.dims if d in th_dims]
        perm = [th_dims.index(d) for d in present]
        if perm != list(range(len(perm))):
            th = np.transpose(th, perm)
        sizes = dict(zip(th_dims, theta.shape))
        need = phi.sizes[phi_dim] + (0 if theta_at_centers else 1)
        if sizes[phi_dim] != need:
            what = "cell-centre values" if theta_at_centers else "cell bounds"
            raise ValueError(f"`target_data` needs {need} {what} along {theta_dim!r}, got {sizes[phi_dim]}")
        th = th.reshape([sizes[d] if d in th_dims else 1 for d in phi.dims])
        out = ops.vinterp_conservative_host(np.asarray(phi.data), th, np.asarray(target_theta_levels.values),
                                            phi.get_axis_num(phi_dim), theta_at_centers,
                                            device=host_dev.index if grid is None else grid._host_device(phi))
        return _conservative_result(out, phi, phi_dim, target_theta_levels, target_dim, suffix)
    device = grid._device_for(phi) if grid is not None else None
    x, host = as_device_tensor(phi.data, device)
    if extra:
        raise ValueError(f"target data has dimensions {extra} that the data does not have")
    axis_num = phi.get_axis_num(phi_dim)
    th_dims = [d if d != theta_dim else phi_dim for d in theta.dims]
    th_t, _ = as_device_tensor(theta.data, x.device)
    present = [d for d in phi.dims if d in th_dims]
    perm = [th_dims.index(d) for d in present]
    if perm != list(range(len(perm))):
        th_t = th_t.permute(*perm)
    sizes = dict(zip(th_dims, theta.shape))
    if sizes[phi_dim] != phi.sizes[phi_dim] + 1:
        raise ValueError(
            f"`target_data` needs {phi.sizes[phi_dim] + 1} cell bounds along {theta_dim!r}, got {sizes[phi_dim]}"
        )
    th_t = th_t.reshape([sizes[d] if d in th_dims else 1 for d in phi.dims])
    tg_t, _ = as_device_tensor(target_theta_levels.data, x.device)
    out = ops.vinterp_conservative(x, th_t, tg_t, axis_num)
    return _conservative_result(result_like(out, host), phi, phi_dim, target_theta_levels, target_dim, suffix)


def _conservative_result(out, phi, phi_dim, target_theta_levels, target_dim, suffix):
    out_dims = tuple(d for d in phi.dims if d != phi_dim) + (target_dim,)
    coords = {k: c for k, c in phi.coords.items()
              if phi_dim not in c.dims and k != target_dim and all(d in out_dims for d in c.dims)}
    levels = target_theta_levels.values
    coords[target_dim] = ((target_dim,), (levels[1:] + levels[:-1]) / 2)  # transform.py:270-272
    res = DataArray(out, dims=out_dims, coords=coords)
    if phi.name:
        res.name = phi.name + suffix
    return res


def _fuse_centre_bounds(phi, theta, target, grid):
    """Whether the remap of numpy fields may make theta's bounds itself: the host route applies, and theta's dtype
    is the remap's, so the center -> outer interp rounds as grid.interp's would (grid.interp works in theta's own
    dtype, integers in f64; the remap works in f32 only when phi, theta and the bins all are f32)."""
    if _conservative_host_device(phi, theta, target, grid) is None:
        return False
    th_dt = np.asarray(theta.data).dtype
    th_dt = th_dt if th_dt in (np.float32, np.float64) else np.dtype(np.float64)
    all_f32 = np.asarray(phi.data).dtype == th_dt == np.asarray(target.data).dtype == np.float32
    return th_dt == (np.float32 if all_f32 else np.float64)


def transform(grid, axis_name, da, target, target_data=None, target_dim=None, method="linear",
              mask_edges=True, bypass_checks=False, suffix="_transformed"):
    """See ``Grid.transform``; argument handling as in reference transform.py:279-514."""
    axis = grid.axes[axis_name]
    if axis.padding == "periodic":
        raise ValueError(
            "`transform` can only be used on axes that are non-periodic. Set a "
            "non-periodic boundary (e.g. `padding='fill'`, or leave it unset) "
            "for this axis on `xgcm.Grid`."
        )
    for var_name, variable, allowed in [
        ("da", da, (DataArray,)),
        ("target", target, (DataArray, np.ndarray)),
        ("target_data", target_data, (DataArray,)),
    ]:
        if not (isinstance(variable, allowed) or variable is None):
            raise ValueError(
                f"`{var_name}` needs to be a {' or '.join([str(a) for a in allowed])}. Found {type(variable)}"
            )

    def _check_other_dims(target_da):
        da_other = set(da.dims) - set(axis.coords.values())
        tgt_other = set(target_da.dims) - set(axis.coords.values())
        if not tgt_other.issubset(da_other):
            raise ValueError(
                f"Found additional dimensions [{tgt_other - da_other}]"
                "in `target_data` not found in `da`. This could mean that the target "
                "array is not on the same position along other axes."
                " If the additional dimensions are associated witha staggered axis, "
                "use grid.interp() to move values to other grid position. "
                "If additional dimensions are not related to the grid (e.g. climate "
                "model ensemble members or similar), use xr.broadcast() before using transform."
            )

    def _parse_target(target, target_dim, target_data_dim, target_data):
        if target_data is None:
            target_data = grid._ds[target_data_dim]  # transform.py:427-428
        if target_dim is None:
            if isinstance(target, DataArray):
                if len(target.dims) == 1:
                    target_dim = list(target.dims)[0]
            else:
                if target_data.name is None:
                    warnings.warn(
                        "Input`target_data` has no name, but we need a name for the transformed dimension. The name `TRANSFORMED_DIMENSION` will be used. To avoid this warning, call `.rename` on `target_data` before calling `transform`."
                    )
                    target_data.name = "TRANSFORMED_DIMENSION"
                target_dim = target_data.name
        if not isinstance(target, DataArray):
            target = DataArray(target, dims=[target_dim], coords={target_dim: target})
        if target_dim is None:
            raise ValueError(
                "`target` has more than one dimension: `target_dim` must be given explicitly"
            )
        if target_dim not in target.dims:
            raise ValueError(
                f"The specified `target_dim` {target_dim} is not within the dimensions of the target: [{target.dims}]."
            )
        _check_other_dims(target_data)
        return target, target_dim, target_data

    _, dim = axis._get_position_name(da)
    if method in ("linear", "log"):
        target, target_dim, target_data = _parse_target(target, target_dim, dim, target_data)
        theta_dim = dim
        if dim not in target_data.dims:
            raise ValueError(
                f"`target_data` must be located on the same position ({dim}) as `da` along axis {axis_name}"
            )
        return linear_interpolation(
            da, target_data, target, dim, theta_dim, target_dim,
            mask_edges=mask_edges, bypass_checks=bypass_checks, logarithmic=(method == "log"),
            grid=grid,
            # NB: like the reference (transform.py:455-466) the Grid-level `suffix` is NOT forwarded:
            # the output keeps the input's name; only the mid-level wrapper honours `suffix`.
        )
    if method == "conservative":
        if isinstance(target, DataArray) and len(target.dims) > 1:
            raise NotImplementedError(
                "Conservative transformation is not yet supported for multi-dimensional targets."
            )
        try:
            target_data_dim = axis.coords["outer"]
        except KeyError:
            raise RuntimeError(
                "In order to use the method `conservative` the grid object needs to have `outer` coordinates."
            )
        target, target_dim, target_data = _parse_target(target, target_dim, target_data_dim, target_data)
        if target_data_dim not in target_data.dims:
            warnings.warn(
                "The `target data` input is not located on the cell bounds. This method will continue with linear interpolation with repeated boundary values. For most accurate results provide values on cell bounds.",
                UserWarning,
            )
            center = axis.coords.get("center")
            if (center is not None and center in target_data.dims and axis.default_shifts.get("center") == "outer"
                    and target_data.sizes[center] == da.sizes[dim] and _fuse_centre_bounds(da, target_data, target, grid)):
                # numpy fields: the n + 1 bounds grid.interp would give are made slab by slab on the device, beside
                # the remap, instead of a round trip of the bounds through host memory
                return _conservative_interpolation(da, target_data, target, dim, center, target_dim, grid=grid,
                                                   theta_at_centers=True)
            target_data = grid.interp(target_data, axis_name, padding="extend")
        return conservative_interpolation(da, target_data, target, dim, target_data_dim, target_dim, grid=grid)
    raise ValueError(f"unknown transform method {method!r}")
