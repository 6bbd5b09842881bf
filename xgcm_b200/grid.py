"""``Grid``: the user-facing façade, API-compatible with the reference's ``xgcm.Grid``.

Method names, kwargs (``axis, to, padding, fill_value, metric_weighted, reverse,
other_component``), kwarg precedence (per call > ufunc default > Axis default,
reference grid.py:315-332), default shifts, metric selection rules
(``get_metric`` conditions 1-4, grid.py:534-657) and error behaviour follow the
reference.  What differs is where the numbers come from: every array value is
produced by a CUDA kernel behind the C-ABI:

* ``diff / interp / min / max`` (+ ``metric_weighted``) and ``derivative``:
  one fused ``xg_stencil2`` launch per axis (reference: np.pad copy + ufunc +
  up to two metric passes, grid.py:800-832,1576-1578);
* ``cumsum / cumint``: one ``xg_cumscan`` launch per axis (grid.py:1306-1414);
* ``integrate / average``: one ``xg_wreduce`` launch per axis (grid.py:1598-1605,1680-1685);
* ``transform`` (linear / log): ``xg_vinterp_linear`` (transform.py).

Host (numpy-backed) inputs are streamed through the GPU and come back as numpy;
CUDA-resident inputs stay resident.

A north fold (tripolar grids, ``padding={"X": "periodic", "Y": {"fold": pivot}}``,
reference grid.py:411-470) is recorded in ``grid._folds``; an operator across it
takes the folded row as a halo plane of its ``xg_stencil2`` launch (one
``xg_fold_rows`` launch beside it).  Out of scope (raise ``NotImplementedError``):
dask chunking.
"""

from __future__ import annotations

import inspect
import itertools
import warnings
from collections import OrderedDict
from typing import Any, Callable, Dict, Iterable, List, Mapping, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np

from . import gridops
from .axis import Axis, _is_dataset
from .grid_ufunc import (
    GridUFunc,
    _check_data_input,
    _GridUFuncSignature,
    _halo_core_dims,
    _host_stream_route,
    _is_host_float,
    _maybe_unpack_vector_component,
    _reattach_coords,
    _stencil_boundary,
    apply_as_grid_ufunc,
)
from .labeled import DataArray, Dataset, is_device_array
from .metrics import iterate_axis_combinations
from .padding import (  # noqa: F401  (pad: re-exported like the reference's grid module)
    _get_all_connection_axes,
    connected_edge_mode,
    fold_edges,
    missing_boundary_error,
    pad,
)


def _maybe_promote_str_to_list(a):
    return [a] if isinstance(a, str) else a


def _host_devices_arg(host_devices):
    """``Grid(host_devices=...)``: None, "all", or a non-empty tuple of CUDA device indices."""
    if host_devices is None or (isinstance(host_devices, str) and host_devices == "all"):
        return host_devices
    if isinstance(host_devices, (str, bytes)) or not isinstance(host_devices, Iterable):
        raise TypeError(f"host_devices must be None, 'all' or a sequence of CUDA device indices, got {host_devices!r}")
    devices = tuple(host_devices)
    if not devices or not all(isinstance(d, (int, np.integer)) and not isinstance(d, bool) and d >= 0
                              for d in devices):
        raise ValueError(f"host_devices must hold one or more non-negative CUDA device indices, got {host_devices!r}")
    return tuple(int(d) for d in devices)


class Grid:
    """A collection of :class:`Axis` objects plus grid metrics, bound to a dataset.

    ``device``: the CUDA device of the calls on numpy fields (default: the current one).  ``host_devices``: None,
    a sequence of CUDA device indices, or "all" (every visible GPU): calls that stream numpy fields through the GPU
    in slabs spread those slabs over these GPUs, each streaming a contiguous block of the result through its own
    PCIe link.  Results are bit for bit those of one GPU.  Device tensors, and numpy fields on routes that do not
    stream, keep using ``device``."""

    def __init__(
        self,
        ds,
        coords: Optional[Mapping[str, Mapping[str, str]]] = None,
        fill_value: Optional[Union[float, Mapping[str, float]]] = None,
        default_shifts: Optional[Mapping[str, str]] = None,
        padding: Optional[Union[str, Mapping[str, str]]] = None,
        face_connections: Optional[Dict[str, Any]] = None,
        metrics: Optional[Mapping[Tuple[str], List[str]]] = None,
        autoparse_metadata: bool = True,
        device=None,
        host_devices=None,
        **kwargs,
    ):
        if "boundary" in kwargs:
            raise ValueError(
                "Argument 'boundary' has been renamed to 'padding'. Please use 'padding' instead."
            )
        self._xarray_io = False
        if not _is_dataset(ds):
            raise TypeError(
                f"ds argument to `xgcm.Grid` must be of type xarray.Dataset, but is of type {type(ds)}"
            )
        if not isinstance(ds, Dataset):
            from . import interop

            ds = interop.dataset_from_xarray(ds)
            self._xarray_io = True
        self._ds = ds
        self._device = device
        self._host_devices = _host_devices_arg(host_devices)

        if autoparse_metadata and coords is None:
            from .metadata import parse_comodo

            parsed = parse_comodo(ds)
            if parsed:
                coords = parsed

        if "periodic" in kwargs:
            raise ValueError(
                "The `periodic` argument has been removed. Use "
                "`padding='periodic'` (per axis if needed, e.g. "
                "`padding={'X': 'periodic', 'Y': 'fill'}`) instead. "
                "Previously `periodic=False` corresponded to `padding='fill'`."
            )
        if kwargs:
            raise TypeError(
                f"Grid.__init__() got unexpected keyword argument(s): "
                f"{', '.join(repr(k) for k in kwargs)}"
            )
        if fill_value:
            warnings.warn(
                "The default fill_value will be changed to nan (from 0.0 previously) "
                "in future versions. Provide `fill_value=0.0` to preserve previous behavior.",
                category=DeprecationWarning,
            )
        if coords is None:
            raise ValueError(
                "Could not determine Axis names - please provide them in the coords kwarg "
                "or provide a dataset from which they can be parsed"
            )
        if face_connections is not None and face_connections:  # grid.py:256-261
            self._facedim = list(face_connections.keys())[0]
            self._face_connections = face_connections
        else:
            self._facedim = None
            self._face_connections = None

        all_axes = list(coords.keys())
        padding_dict = self._map_kwargs_over_axes(padding, axes=all_axes)
        shifts_dict = self._map_kwargs_over_axes(default_shifts, axes=all_axes)
        fill_dict = self._map_kwargs_over_axes(fill_value, axes=all_axes)
        self._explicitly_periodic_axes = {ax for ax, p in padding_dict.items() if p == "periodic"}

        self.axes: "OrderedDict[str, Axis]" = OrderedDict()
        for name in all_axes:
            self.axes[name] = Axis(
                ds,
                name,
                coords=coords[name],
                default_shifts=shifts_dict.get(name, None),
                padding=padding_dict.get(name, None),
                fill_value=fill_dict.get(name, None),
            )

        if face_connections is not None:
            self._assign_face_connections(face_connections)
        self._validate_folds()

        self._metrics: Dict[frozenset, List[DataArray]] = {}
        self._metric_cache: Dict[Any, Any] = {}
        if metrics is not None:
            for key, value in metrics.items():
                self.set_metrics(key, value)

    # ------------------------------------------------------------------ topology
    def _assign_face_connections(self, fc):
        """Check that every link of a face-connection dict is mirrored by its neighbour and hand
        each Axis its links (grid.py:334-409).  Structure: ``{facedim: {face: {axis: (left,
        right)}}}`` with a link ``(neighbour face, neighbour axis, reverse)`` or None."""
        if len(fc) > 1:
            raise ValueError(
                "Only one face dimension is supported for now. Instead found %r" % repr(fc.keys())
            )
        facedim = list(fc.keys())[0]
        if facedim not in self._ds.dims:
            raise ValueError(
                f"Face dimension {facedim} does not exist in the dataset. "
                f"Found {list(self._ds.dims)} instead"
            )
        face_values = list(np.asarray(self._ds[facedim].values).tolist())
        face_links = fc[facedim]
        axis_connections: Dict[str, Dict[Any, Any]] = {}
        for fidx, face_axis_links in face_links.items():
            for axis, axis_links in face_axis_links.items():
                axis_connections.setdefault(axis, {})
                link_left, link_right = axis_links

                def check_neighbor(link, position):
                    if link is None:
                        return None
                    idx, ax, rev = link
                    # a reversed link arrives at the same side of the neighbour
                    correct_position = int(not position) if rev else position
                    try:
                        neighbor_link = face_links[idx][ax][correct_position]
                    except (KeyError, IndexError):
                        raise KeyError(
                            "Couldn't find a face link for face %r"
                            "in axis %r at position %r" % (idx, ax, correct_position)
                        )
                    idx_n, ax_n, rev_n = neighbor_link
                    if ax not in self.axes:
                        raise KeyError("axis %r is not a valid axis" % ax)
                    if ax_n not in self.axes:
                        raise KeyError("axis %r is not a valid axis" % ax_n)
                    for i in (idx, idx_n):
                        if i not in face_values:
                            raise IndexError(
                                "%r is not a valid index for face dimension %r" % (i, facedim)
                            )
                    if (idx_n != fidx) or (ax_n != axis) or (rev_n != rev):
                        raise ValueError(
                            "Face link mismatch: neighbor doesn't correctly link back to this face. "
                            "face: %r, axis: %r, position: %r, rev: %r, link: %r, neighbor_link: %r"
                            % (fidx, axis, position, rev, link, neighbor_link)
                        )
                    return idx, self.axes[ax], rev

                left = check_neighbor(link_left, 1)
                right = check_neighbor(link_right, 0)
                axis_connections[axis][fidx] = (left, right)
        for axis, axis_links in axis_connections.items():
            self.axes[axis]._facedim = facedim
            self.axes[axis]._face_connections = axis_links

    def _validate_folds(self):
        """Record every north fold in ``self._folds[fold axis] = {"seam_axis", "pivot", "south"}``
        (grid.py:411-470).  The seam is the one OTHER axis whose padding was given as "periodic";
        an axis with no padding is not a candidate."""
        self._folds: Dict[str, Dict[str, Any]] = {}
        for axname, axis in self.axes.items():
            spec = axis._padding
            if not isinstance(spec, Mapping):
                continue
            seams = [other for other in self.axes if other != axname and other in self._explicitly_periodic_axes]
            if not seams:
                raise ValueError(
                    f"A fold padding on axis {axname!r} requires an explicitly periodic seam axis (the zonal "
                    "wrap), but no other axis was explicitly marked periodic. Set e.g. "
                    "padding={'X': 'periodic', '" + str(axname) + "': {'fold': ...}}."
                )
            if len(seams) > 1:
                raise ValueError(
                    f"A fold padding on axis {axname!r} is ambiguous: more than one explicitly periodic "
                    f"axis could be the seam ({seams}). Multiple candidate seam axes are not supported."
                )
            self._folds[axname] = {"seam_axis": seams[0], "pivot": spec["fold"], "south": spec["south"]}
        if self._folds and self._face_connections is not None:
            raise NotImplementedError(
                "Combining a north-fold boundary with face_connections is not supported "
                f"(fold axes: {sorted(self._folds)}). Use one or the other."
            )
        if self._folds:
            warnings.warn(
                "The north-fold (tripolar) boundary condition is experimental. Its API and numerical "
                "behavior may change in future releases; please review results carefully.",
                category=UserWarning,
            )

    # ------------------------------------------------------------------ kwargs plumbing
    def _map_kwargs_over_axes(self, kwargs, axes: Optional[Iterable[str]] = None) -> Dict[str, Any]:
        """``'fill'`` -> ``{'X': 'fill', 'Y': 'fill'}``; dicts pass through (grid.py:291-313)."""
        if axes is None:
            axes = self.axes
        if isinstance(kwargs, dict):
            return kwargs
        return {name: kwargs for name in axes}

    def _complete_user_kwargs_using_axis_defaults(self, user_kwargs, property: str) -> Dict[str, Any]:
        """Per-call value wins, else the Axis default (grid.py:315-332)."""
        defaults = {ax: getattr(self.axes[ax], property) for ax in self.axes}
        if user_kwargs is None:
            return defaults
        return {**defaults, **self._map_kwargs_over_axes(user_kwargs)}

    # ------------------------------------------------------------------ device plumbing
    def _device_for(self, da=None):
        import torch

        if da is not None and is_device_array(getattr(da, "data", None)):
            return da.data.device
        if self._device is not None:
            return torch.device(self._device)
        from .device import default_device

        return default_device()

    def _host_device(self, da=None):
        """The ``device`` of the ``ops.*_host`` call that streams numpy field ``da``: the grid's ``host_devices``
        group when it has one, else the index of the CUDA device the call runs on."""
        if self._host_devices is None:
            return self._device_for(da).index
        if self._host_devices == "all":
            import torch

            return tuple(range(torch.cuda.device_count()))
        return self._host_devices

    def _metric_tensor(self, metric: DataArray, field_dims: Sequence[str], like):
        """Device tensor of ``metric`` shaped to broadcast against ``field_dims`` (size-1 elsewhere)."""
        import torch

        missing = [d for d in metric.dims if d not in field_dims]
        if missing:
            raise ValueError(f"metric dims {metric.dims} are not a subset of the field dims {tuple(field_dims)}")
        key = (id(metric.data), tuple(metric.dims), tuple(field_dims), str(like.dtype), str(like.device))
        hit = self._metric_cache.get(key)
        if hit is not None and hit[0] is metric.data:
            return hit[1]
        data = metric.data
        if not is_device_array(data):
            arr = np.ascontiguousarray(np.asarray(data))
            if arr.dtype.kind != "f":
                arr = arr.astype(np.float64)
            data = torch.from_numpy(arr).to(like.device)
        data = data.to(like.dtype)
        present = [d for d in field_dims if d in metric.dims]
        perm = [metric.dims.index(d) for d in present]
        if perm != list(range(len(perm))):
            data = data.permute(*perm).contiguous()
        shape = [metric.sizes[d] if d in metric.dims else 1 for d in field_dims]
        t = data.reshape(shape)
        if len(self._metric_cache) > 64:
            self._metric_cache.clear()
        self._metric_cache[key] = (metric.data, t)
        return t

    def _metric_host(self, metric: DataArray, field_dims: Sequence[str], dtype) -> np.ndarray:
        """Host array of ``metric`` shaped to broadcast against ``field_dims``."""
        missing = [d for d in metric.dims if d not in field_dims]
        if missing:
            raise ValueError(f"metric dims {metric.dims} are not a subset of the field dims {tuple(field_dims)}")
        arr = metric.values
        present = [d for d in field_dims if d in metric.dims]
        perm = [metric.dims.index(d) for d in present]
        if perm != list(range(len(perm))):
            arr = np.transpose(arr, perm)
        shape = [metric.sizes[d] if d in metric.dims else 1 for d in field_dims]
        return np.ascontiguousarray(arr, dtype=dtype).reshape(shape)

    def _wrap_in(self, obj):
        """Accept real xarray objects when xarray is installed."""
        if isinstance(obj, DataArray) or obj is None:
            return obj, False
        if isinstance(obj, dict):  # vector input {axis: DataArray} / other_component: convert the values
            out, any_x = {}, False
            for k, v in obj.items():
                out[k], was = self._wrap_in(v)
                any_x = any_x or was
            return out, any_x
        if type(obj).__name__ == "DataArray" and hasattr(obj, "dims"):
            from . import interop

            return interop.dataarray_from_xarray(obj), True
        return obj, False

    def _wrap_out(self, res, as_xarray: bool):
        if not as_xarray:
            return res
        from . import interop

        return interop.dataarray_to_xarray(res)

    # ------------------------------------------------------------------ metrics
    def set_metrics(self, key, value, overwrite=False):
        """Register dataset variables as metrics for a set of axes (grid.py:472-514)."""
        metric_axes = frozenset(_maybe_promote_str_to_list(key))
        missing = [ma for ma in metric_axes if ma not in self.axes]
        if missing:
            raise KeyError(f"Metric axes {missing!r} not compatible with grid axes {tuple(self.axes)!r}")
        names = _maybe_promote_str_to_list(value)
        for name in names:
            if name not in self._ds.variables:
                raise KeyError(f"Metric variable {name} not found in dataset.")
        self._metric_cache.clear()
        if metric_axes in self._metrics:
            existing = self._metrics[metric_axes]
            new = self._ds[name].reset_coords(drop=True)
            replaced = False
            for idx, old in enumerate(existing):
                if set(new.dims) == set(old.dims):
                    if not overwrite:
                        raise ValueError(
                            f"Metric variable {old.name} with dimensions {old.dims} already assigned in metrics."
                            f" Overwrite {old.name} with {name} by setting overwrite=True."
                        )
                    existing[idx] = new
                    replaced = True
            if not replaced:
                existing.append(new)
        else:
            self._metrics[metric_axes] = [self._ds[n].reset_coords(drop=True) for n in names]

    def _get_dims_from_axis(self, da, axis) -> List[str]:
        da = _maybe_unpack_vector_component(da)
        dims = []
        for ax in _maybe_promote_str_to_list(axis):
            if ax not in self.axes:
                raise KeyError(f"Did not find axis {ax} from data array {da.name}")
            matching = [d for d in self.axes[ax].coords.values() if d in da.dims]
            if len(matching) != 1:
                raise ValueError(
                    f"Did not find single matching dimension {da.dims} from {da.name} corresponding to axis {ax}, got {matching}."
                )
            dims.append(matching[0])
        return dims

    def _metric_product(self, metrics: Sequence[DataArray]) -> DataArray:
        """Product of metrics (dx * dy ...), computed on the device (reference:
        ``functools.reduce(operator.mul, ...)``, grid.py:617-619)."""
        if len(metrics) == 1:
            return metrics[0]
        key = ("prod",) + tuple(id(m.data) for m in metrics)
        hit = self._metric_cache.get(key)
        if hit is not None and all(a is b.data for a, b in zip(hit[0], metrics)):
            return hit[1]
        dev = self._device_for(None)
        out = metrics[0] if metrics[0].is_device else metrics[0].to_device(dev)
        for m in metrics[1:]:
            out = out * (m if m.is_device else m.to_device(dev))
        self._metric_cache[key] = (tuple(m.data for m in metrics), out)
        return out

    def get_metric(self, array, axes):
        """The metric for ``axes`` that broadcasts against ``array`` (only its dims matter).

        Selection follows the reference (grid.py:534-657): (1) a metric registered under
        exactly these axes whose dims fit; (2) else that metric interpolated to the array's
        position; (3) else a product of sub-axis metrics whose dims fit; (4) else the
        interpolated product.
        """
        array_dims = set(array.dims)
        self._get_dims_from_axis(array, frozenset(axes))
        registered = set(tuple(k) for k in self._metrics.keys())
        overlap = registered.intersection(set(itertools.permutations(tuple(axes))))
        found = None
        if overlap:
            key = frozenset(*overlap)
            candidates = self._metrics[key]
            for mv in candidates:
                if set(mv.dims).issubset(array_dims):
                    found = mv
                    break
            if found is None:
                mv = candidates[-1]
                warnings.warn(
                    f"Metric at {array.dims} being interpolated from metrics at dimensions {mv.dims}. Boundary value set to 'extend'."
                )
                found = self.interp_like(mv, array, "extend", None)
        else:
            fallback = None
            locked = False
            for combo in iterate_axis_combinations(axes):
                try:
                    pools = [self._metrics[ac] for ac in combo]
                except KeyError:
                    continue
                for choice in itertools.product(*pools):
                    dims = set(d for mv in choice for d in mv.dims)
                    if dims.issubset(array_dims):
                        found = self._metric_product(choice)
                        break
                    if not locked:
                        fallback = choice
                if found is not None:
                    break
                locked = True
            if found is None and fallback is not None:
                warnings.warn(
                    f"Metric at {array.dims} being interpolated from metrics at dimensions {[pc.dims for pc in fallback]}. Boundary value set to 'extend'."
                )
                found = self._metric_product(
                    tuple(self.interp_like(pc, array, "extend", None) for pc in fallback)
                )
        if found is None:
            raise KeyError(
                f"Unable to find any combinations of metrics for array dims {array_dims!r} and axes {axes!r}"
            )
        return found

    def interp_like(self, array, like, padding=None, fill_value=None, **kwargs):
        """Interpolate ``array`` to the grid positions of ``like`` (grid.py:659-716)."""
        if "boundary" in kwargs:
            raise ValueError(
                "Argument 'boundary' has been renamed to 'padding'. Please use 'padding' instead."
            )
        interp_axes = []
        for name, axis in self.axes.items():
            try:
                pos_array, _ = axis._get_position_name(array)
                pos_like, _ = axis._get_position_name(like)
            except KeyError:
                continue
            if pos_like != pos_array:
                interp_axes.append(name)
        return self.interp(array, interp_axes, fill_value=fill_value, padding=padding)

    def __repr__(self):
        lines = ["<xgcm.Grid>"]
        for name, axis in self.axes.items():
            kind = "periodic" if axis._periodic else "not periodic"
            lines.append("%s Axis (%s, padding=%r):" % (name, kind, axis.padding))
            lines += axis._coord_desc()
        return "\n".join(lines)

    # ------------------------------------------------------------------ 1-D operator dispatch
    def _create_1d_grid_ufunc_signatures(self, da, axis, to) -> List[_GridUFuncSignature]:
        sigs = []
        for ax_name in axis:
            ax = self.axes[ax_name]
            from_pos, _ = ax._get_position_name(da)
            to_pos = to[ax_name] if to.get(ax_name) is not None else None
            if to_pos is None:
                to_pos = ax._default_shifts[from_pos]
            sigs.append(_GridUFuncSignature.from_string(f"({ax_name}:{from_pos})->({ax_name}:{to_pos})"))
        return sigs

    def _1d_grid_ufunc_dispatch(self, funcname, data, axis, to=None, metric_weighted=None,
                                other_component=None, _divide_by_metric_of=None, **kwargs):
        """Apply the built-in 1-D grid ufunc along each axis in turn (grid.py:728-836).

        ``metric_weighted`` (and the divide of ``derivative``) are handed to the kernel as
        pre-multiply / post-divide operands instead of separate full-array passes.
        """
        if "keep_coords" in kwargs:
            raise ValueError(
                "The 'keep_coords' argument has been removed. Coordinates "
                "compatible with the output are now always preserved."
            )
        if isinstance(axis, str):
            axis = [axis]
        data, as_xarray = self._wrap_in(data)
        if other_component is not None:
            other_component, _ = self._wrap_in(other_component)
        data = _check_data_input(data, self)
        unpacked = _maybe_unpack_vector_component(data)
        for ax_name in axis:
            if ax_name not in self.axes:
                raise KeyError(f"Did not find axis {ax_name} in grid axes {list(self.axes)}")
        to = self._map_kwargs_over_axes(to)
        if isinstance(metric_weighted, str):
            metric_weighted = (metric_weighted,)
        metric_weighted = self._map_kwargs_over_axes(metric_weighted)
        signatures = self._create_1d_grid_ufunc_signatures(unpacked, axis=axis, to=to)

        host_input = not unpacked.is_device
        array = unpacked.copy(deep=False)
        n_axes = len(axis)
        weights = {ax: metric_weighted.get(ax) for ax in axis if metric_weighted.get(ax)}
        if (
            n_axes in (2, 3)
            and len(set(axis)) == n_axes
            and (not weights or other_component is None)
            and _divide_by_metric_of is None
            and not isinstance(data, dict)
            and set(kwargs) <= {"padding", "fill_value"}
        ):
            fused = self._fused_multi_axis(funcname, array, axis, to, kwargs, weights)
            if fused is None and other_component is None and not weights:  # a scalar field: no vector halo
                fused = self._multi_axis_halo_host(funcname, array, axis, to, kwargs)
            if fused is not None:
                return self._wrap_out(fused, as_xarray)
        if host_input and n_axes > 1:
            # several passes: upload once, keep the intermediates resident, download once
            array = array.to_device(self._device_for(None))

        for sig, ax_name in zip(signatures, axis):
            grid_ufunc, remaining = _select_grid_ufunc(funcname, sig, module=gridops, **kwargs)
            weighted = metric_weighted.get(ax_name) if isinstance(metric_weighted, dict) else None
            extra = {}
            post_fns = []
            if weighted:
                extra["_pre_metric"] = self.get_metric(array, weighted)
                post_fns.append(lambda probe, _w=weighted: self.get_metric(probe, _w))
            if _divide_by_metric_of is not None:
                post_fns.append(lambda probe, _a=_divide_by_metric_of: self.get_metric(probe, _a))
            if post_fns:
                extra["_post_metric"] = post_fns[0]
            arg = {ax_name_key: array for ax_name_key in data} if isinstance(data, dict) else array
            array = grid_ufunc(
                self, arg, axis=[(ax_name,)], dask="forbidden", map_overlap=False,
                other_component=other_component, **remaining, **extra,
            )
            for fn in post_fns[1:]:  # metric_weighted AND derivative: second divide, own pass
                array = array / fn(array)
        if host_input and array.is_device:
            from .device import result_like

            array = array._replace(data=result_like(array.data, True))
        return self._wrap_out(array, as_xarray)

    def _fused_multi_axis(self, funcname, array, axis, to, kwargs, weights=None):
        """All axes of a multi-axis diff / interp / min / max in ONE kernel launch
        (``xg_stencil_multi``): same values as the per-axis loop of grid.py:800-832, one read and
        one write of the field instead of one pass per axis.  ``weights`` (axis name -> the
        ``metric_weighted`` axes of its stage) gives each weighted stage the pre- and post-metric
        the loop would take, ``get_metric`` of the stage's input and output dims
        (``xg_stencil_multi_weighted``).  Returns None when the fused kernel does not cover the case
        (then the caller runs the per-axis launches)."""
        from . import ops
        from .device import as_device_tensor, result_like
        from .grid_ufunc import _ShapeProbe

        if self._face_connections is not None:
            return None  # halos come from other faces: per-axis pad + stencil
        weights = weights or {}
        paddings = self._complete_user_kwargs_using_axis_defaults(kwargs.get("padding"), "padding")
        fills = self._complete_user_kwargs_using_axis_defaults(kwargs.get("fill_value"), "fill_value")
        specs, rename = [], {}
        dims, shape = tuple(array.dims), list(array.shape)
        stages = []  # per stage: its metric_weighted axes, input dims and shape, output dims and shape
        for ax_name in axis:
            t = _stencil_term(self, funcname, array, ax_name, to.get(ax_name), paddings, fills)
            if t.folded:
                return None  # the fold row is a halo plane of the per-axis launch
            if t.pad_mode not in ("periodic", "fill", "extend", None):
                return None  # e.g. the opt-in extrapolate extension: per-axis path
            specs.append((t.axis_num, funcname, t.lo, t.hi, t.pad_mode if (t.lo or t.hi) else None, t.fill))
            rename[t.in_dim] = t.out_dim
            out_dims = tuple(t.out_dim if d == t.in_dim else d for d in dims)
            out_shape = list(shape)
            out_shape[t.axis_num] += t.lo + t.hi - 1
            stages.append((weights.get(ax_name), dims, shape, out_dims, out_shape))
            dims, shape = out_dims, out_shape
        if array.shape[-1] < 32:
            return None  # tiny rows: the one-block-per-row kernel has nothing to chew on
        stage_mets = [None if not w else (self.get_metric(_ShapeProbe(d, s), w), d,
                                          self.get_metric(_ShapeProbe(od, os_), w), od)
                      for w, d, s, od, os_ in stages]

        def metrics(convert):
            if not weights:
                return {}
            pre = [None if sm is None else convert(sm[0], sm[1]) for sm in stage_mets]
            post = [None if sm is None else convert(sm[2], sm[3]) for sm in stage_mets]
            return {"pre": pre, "post": post}

        out = None
        dev = self._device_for(array)
        if _is_host_float(array) and dev.type == "cuda":
            # numpy-backed field: slabs stream through the GPU (xg_stencil_multi_host), so input, result and the
            # device footprint need not fit in HBM together
            x = np.asarray(array.data)
            try:
                out = ops.stencil_multi_host(x, specs, device=self._host_device(array),
                                             **metrics(lambda m, d: self._metric_host(m, d, x.dtype)))
            except NotImplementedError:
                out = None  # a cut along an operated dim the slabs cannot pad: the whole field on the device
        if out is None:
            x, was_host = as_device_tensor(array.data, dev)
            try:
                y = ops.stencil_multi(x, specs, **metrics(lambda m, d: self._metric_tensor(m, d, x)))
            except NotImplementedError:
                return None  # a metric layout the weighted kernel does not address: per-axis launches
            out = result_like(y, was_host)
        out_dims = tuple(rename.get(d, d) for d in array.dims)
        res = DataArray(out, dims=out_dims, name=array.name, attrs=array.attrs)
        return _reattach_coords([res], self, None, set(rename.values()), [array])[0]

    def _multi_axis_halo_host(self, funcname, array, axis, to, kwargs):
        """A multi-axis diff / interp / min / max of a numpy field on a face-connected grid, or across a north fold,
        streamed through the GPU in slabs (``xg_stencil_chain_host_connected`` / ``_fold``) instead of uploaded
        whole: per slab, the device route's per-axis launches in the order given, each stage's halo planes built
        from its own input, so the values are those of the device route.  Each stage is resolved against the
        intermediate's dims and shape, and its errors are raised before anything streams.  Returns the result, or
        None for the whole-field route: no face connection and no folded term, a device array, no CUDA device, a
        boundary the halo stencils do not take (extrapolate), no batch dim in front of the operated, seam and face
        dims (``_host_stream_route``), a fold the plan cannot mirror."""
        from . import ops
        from .padding import connected_halo_program

        connected = self._face_connections is not None
        if not (connected or self._folds) or not _is_host_float(array) or self._device_for(array).type != "cuda":
            return None
        padding, fill_value = kwargs.get("padding"), kwargs.get("fill_value")
        paddings = self._complete_user_kwargs_using_axis_defaults(padding, "padding")
        fills = self._complete_user_kwargs_using_axis_defaults(fill_value, "fill_value")
        if connected:  # every padded edge takes its value from connected_edge_mode below, which raises its own errors
            paddings = {k: "fill" if v is None else v for k, v in paddings.items()}
        dims, shape = tuple(array.dims), [int(v) for v in array.shape]
        stages = []  # (term, the stage's input dims and shape, edge mode and fill of a connected stage)
        probe = DataArray.__new__(DataArray)
        for ax_name in axis:
            probe._dims = dims
            t = _stencil_term(self, funcname, probe, ax_name, to.get(ax_name), paddings, fills)
            mode = None
            if connected:
                mode = connected_edge_mode(self, ax_name, t.lo, t.hi, padding, fill_value,
                                           shape[dims.index(self._facedim)])
            elif t.pad_mode not in ("periodic", "fill", "extend", None):
                return None  # e.g. the opt-in extrapolate extension
            stages.append((t, dims, shape, mode))
            dims = tuple(t.out_dim if d == t.in_dim else d for d in dims)
            shape = list(shape)
            shape[t.axis_num] += t.lo + t.hi - 1
        if not connected and not any(t.folded for t, *_ in stages):
            return None
        in_dims = stages[0][1]
        fold_axis = next((t.ax_name for t, *_ in stages if t.folded), None)
        core = [t.in_dim for t, *_ in stages] + _halo_core_dims(self, in_dims, fold_axis)
        cut = _host_stream_route("connected" if connected else "fold", in_dims, stages[0][2], core,
                                 max(t.lo for t, *_ in stages), max(t.hi for t, *_ in stages))
        if cut is None:
            return None
        specs, programs = [], []
        for t, s_dims, s_shape, mode in stages:
            m_dims, m_shape = cut.dims(s_dims), cut.shape(s_shape)
            if connected:
                specs.append((cut.axis(t.axis_num), funcname, t.lo, t.hi, mode[1]))
                programs.append(connected_halo_program(self, t.ax_name, t.lo, t.hi, m_dims, m_shape, mode[0]))
                continue
            plan = cut.fold_plan(self, t.ax_name, s_dims, s_shape) if t.folded else None
            if t.folded and plan is None:
                return None
            specs.append((cut.axis(t.axis_num), funcname, t.lo, t.hi, t.pad_mode if (t.lo or t.hi) else None, t.fill,
                          plan))
        x, device = cut.cut(array.data), self._host_device(array)
        if connected:
            y = ops.stencil_chain_host_connected(x, specs, programs, device=device)
        else:
            y = ops.stencil_chain_host_fold(x, specs, device=device)
        res = DataArray(y.reshape(shape), dims=dims, name=array.name, attrs=array.attrs)
        return _reattach_coords([res], self, None, {t.out_dim for t, *_ in stages}, [array])[0]

    def apply_many(self, da, requests, padding=None, fill_value=None):
        """Several single-axis operators of ONE field in one call (an extension; the reference has no
        counterpart and would re-read the field per call, grid.py:796-832).

        ``requests``: sequence of ``(funcname, axis)`` or ``(funcname, axis, to)`` with funcname in
        diff / interp / min / max.  Returns a list of DataArrays, one per request, identical to calling
        ``getattr(grid, funcname)(da, axis, to=to)`` one by one.  For a numpy-backed field the batch goes
        through ``xg_stencil2_host_multi``: the field crosses PCIe once and every result streams back
        while later slabs are still being computed.  Device-resident fields just loop."""
        from . import ops

        da, as_xarray = self._wrap_in(da)
        reqs = []
        for r in requests:
            funcname, ax_name = r[0], r[1]
            to = r[2] if len(r) > 2 else None
            if funcname not in ("diff", "interp", "min", "max"):
                raise ValueError(f"apply_many supports diff / interp / min / max, got {funcname!r}")
            if ax_name not in self.axes:
                raise KeyError(f"Did not find axis {ax_name} in grid axes {list(self.axes)}")
            reqs.append((funcname, ax_name, to))
        kw = {}
        if padding is not None:
            kw["padding"] = padding
        if fill_value is not None:
            kw["fill_value"] = fill_value

        def one_by_one():
            return [self._wrap_out(self._1d_grid_ufunc_dispatch(f, da, a, to=t, **kw), as_xarray)
                    for f, a, t in reqs]

        host_ok = (not isinstance(da, dict) and _is_host_float(da) and self._face_connections is None
                   and 1 <= len(reqs) <= 8)
        if not host_ok:
            return one_by_one()
        paddings = self._complete_user_kwargs_using_axis_defaults(padding, "padding")
        fills = self._complete_user_kwargs_using_axis_defaults(fill_value, "fill_value")
        specs, renames = [], []
        for funcname, ax_name, to in reqs:
            t = _stencil_term(self, funcname, da, ax_name, self._map_kwargs_over_axes(to).get(ax_name), paddings,
                              fills)
            if t.folded:
                return one_by_one()  # the host pipeline takes no halo planes
            if t.pad_mode not in ("periodic", "fill", "extend", None):
                return one_by_one()
            if t.axis_num == 0 and (t.lo + t.hi != 1):
                return one_by_one()  # outer / inner shift along the slab dimension
            specs.append((t.axis_num, funcname, t.lo, t.hi, t.pad_mode if (t.lo or t.hi) else None, t.fill))
            renames.append((t.in_dim, t.out_dim, ax_name, (t.lo, t.hi)))
        outs = ops.stencil2_host_multi(np.asarray(da.data), specs, device=self._host_device(da))
        results = []
        for arr, (in_dim, out_dim, ax_name, width) in zip(outs, renames):
            out_dims = tuple(out_dim if d == in_dim else d for d in da.dims)
            res = DataArray(arr, dims=out_dims, name=da.name, attrs=da.attrs)
            res = _reattach_coords([res], self, {ax_name: width}, {out_dim}, [da])[0]
            results.append(self._wrap_out(res, as_xarray))
        return results

    # ------------------------------------------------------------------ two-field composites (extension)
    def pair(self, funcname_a, da_a, axis_a, funcname_b, da_b, axis_b, combine="add", metric_a=None,
             metric_b=None, divide_by=None, to=None, padding=None, fill_value=None, _components=None):
        """``(f_a(da_a * metric_a, axis_a)  +|-  f_b(da_b * metric_b, axis_b)) / metric_out`` — what users chain
        from ``Grid.diff`` / ``Grid.interp`` and xarray arithmetic for divergence-like quantities
        (docs/ufunc_examples.md:105-153), evaluated in ONE kernel (``xg_stencil_pair``) when both terms are
        length-preserving stencils along different dims of same-shaped fields; rounding is that of the chain.

        ``metric_a`` / ``metric_b``: axes whose metric (``get_metric`` at the input's position) multiplies the
        input; ``divide_by``: axes whose metric at the OUTPUT position divides the result; ``combine``: "add" or
        "sub" (term a minus term b).  Anything the fused kernel does not cover runs as the explicit chain.

        ``_components``: the vector-component axes of ``da_a`` / ``da_b`` (divergence, vorticity); a term
        across a north fold then folds its input as that component, which changes its sign.

        On a fold grid the term along the non-innermost dim may cross the fold: its folded row is the kernel's
        halo plane (one ``xg_fold_rows`` launch beside the pair).  Numpy fields with a batch dim in front of
        the operated (and seam) dims stream through the GPU in slabs (``xg_stencil_pair_host``)."""
        from . import ops
        from .device import as_device_tensor, result_like
        from .padding import fold_halo_planes

        if combine not in ("add", "sub"):
            raise ValueError(f"combine must be 'add' or 'sub', got {combine!r}")
        da_a, xr_a = self._wrap_in(da_a)
        da_b, xr_b = self._wrap_in(da_b)
        as_xarray = xr_a or xr_b
        to = self._map_kwargs_over_axes(to)
        kw = {}
        if padding is not None:
            kw["padding"] = padding
        if fill_value is not None:
            kw["fill_value"] = fill_value

        def as_tuple(m):
            return (m,) if isinstance(m, str) else (tuple(m) if m is not None else None)

        metric_a, metric_b, divide_by = as_tuple(metric_a), as_tuple(metric_b), as_tuple(divide_by)

        def chain():
            xa = da_a * self.get_metric(da_a, metric_a) if metric_a else da_a
            xb = da_b * self.get_metric(da_b, metric_b) if metric_b else da_b
            if _components is not None:
                xa = {_components[0]: xa} if axis_a in self._folds else xa
                xb = {_components[1]: xb} if axis_b in self._folds else xb
            ta = self._1d_grid_ufunc_dispatch(funcname_a, xa, axis_a, to={axis_a: to.get(axis_a)}, **kw)
            tb = self._1d_grid_ufunc_dispatch(funcname_b, xb, axis_b, to={axis_b: to.get(axis_b)}, **kw)
            if ta.dims != tb.dims:
                raise ValueError(f"the two terms land on different positions: {ta.dims} vs {tb.dims}")
            r = ta + tb if combine == "add" else ta - tb
            if divide_by:
                r = r / self.get_metric(r, divide_by)
            r.name = da_a.name
            return self._wrap_out(r, as_xarray)

        if (isinstance(da_a, dict) or isinstance(da_b, dict) or self._face_connections is not None
                or axis_a == axis_b or da_a.shape != da_b.shape or da_a.is_device != da_b.is_device):
            return chain()
        paddings = self._complete_user_kwargs_using_axis_defaults(padding, "padding")
        fills = self._complete_user_kwargs_using_axis_defaults(fill_value, "fill_value")
        terms = []
        for funcname, da, ax_name in ((funcname_a, da_a, axis_a), (funcname_b, da_b, axis_b)):
            if funcname not in ("diff", "interp", "min", "max") or ax_name not in self.axes:
                return chain()
            try:
                t = _stencil_term(self, funcname, da, ax_name, to.get(ax_name), paddings, fills)
            except ValueError:
                return chain()  # no such position, or no boundary condition: the chain raises its own error
            if t.lo + t.hi != 1 or t.pad_mode not in ("periodic", "fill", "extend"):
                return chain()
            terms.append(t)
        ta, tb = terms
        out_dims_a = tuple(ta.out_dim if d == ta.in_dim else d for d in da_a.dims)
        out_dims_b = tuple(tb.out_dim if d == tb.in_dim else d for d in da_b.dims)
        # each term leaves the other's operated dim untouched: the sum needs both to land on the same dims
        if out_dims_a != out_dims_b:
            raise ValueError(f"the two terms land on different positions: {out_dims_a} vs {out_dims_b}")
        last = da_a.ndim - 1
        if ta.axis_num == last and tb.axis_num != last:
            first, second, fa, fb, ma_ax, mb_ax = ta, tb, da_a, da_b, metric_a, metric_b
            sub = 0 if combine == "add" else 1
        elif tb.axis_num == last and ta.axis_num != last:
            first, second, fa, fb, ma_ax, mb_ax = tb, ta, da_b, da_a, metric_b, metric_a
            sub = 0 if combine == "add" else 2  # kernel: innermost term first; we want (a - b) = strided - innermost
        else:
            return chain()  # neither (or both) terms act on the innermost dim
        host = not da_a.is_device
        dev = self._device_for(da_a)
        # the kernel takes halo planes for the term along the strided dim only; the fold plane and the host twins
        # are CUDA launches (as in grid_ufunc._apply_fused_stencil, a fold off a CUDA device keeps the chain)
        if first.folded or (second.folded and dev.type != "cuda"):
            return chain()
        spec_a = (first.op, first.lo, first.hi, first.pad_mode, first.fill)
        spec_b = (second.axis_num, second.op, second.lo, second.hi, second.pad_mode, second.fill)
        negate = _components is not None  # a vector component changes sign across the fold
        probe = DataArray.__new__(DataArray)
        probe._dims = out_dims_a

        def finish(data):
            res = DataArray(data, dims=out_dims_a, name=da_a.name)
            res = _reattach_coords([res], self, None, {ta.out_dim, tb.out_dim}, [da_a, da_b])[0]
            return self._wrap_out(res, as_xarray)

        if host and dev.type == "cuda" and _is_host_float(fa) and _is_host_float(fb) and fa.data.dtype == fb.data.dtype:
            # numpy fields: slabs of the leading batch dims H2D -> xg_stencil_pair_halo -> D2H
            dims, shape, dt = tuple(fb.dims), list(fb.shape), fa.data.dtype
            pre_a = self._metric_host(self.get_metric(fa, ma_ax), fa.dims, dt) if ma_ax else None
            pre_b = self._metric_host(self.get_metric(fb, mb_ax), fb.dims, dt) if mb_ax else None
            post = self._metric_host(self.get_metric(probe, divide_by), out_dims_a, dt) if divide_by else None
            core = [second.in_dim, dims[-1]] + _halo_core_dims(self, dims, second.ax_name if second.folded else None)
            cut = _host_stream_route("pair", dims, shape, core, 0, 1,
                                     operand_shapes=[m.shape for m in (pre_a, pre_b, post) if m is not None])
            plan = cut.fold_plan(self, second.ax_name, dims, shape) if second.folded and cut is not None else None
            if cut is not None and (plan is not None or not second.folded):
                kw = dict(pre_a=cut.cut(pre_a), pre_b=cut.cut(pre_b), post=cut.cut(post), device=self._host_device(da_a))
                spec_b = (cut.axis(spec_b[0]),) + spec_b[1:]
                if second.folded:
                    y = ops.stencil_pair_host_fold(cut.cut(fa.data), cut.cut(fb.data), spec_a, spec_b, *plan, sub,
                                                   negate=negate, **kw)
                else:
                    y = ops.stencil_pair_host(cut.cut(fa.data), cut.cut(fb.data), spec_a, spec_b, sub, **kw)
                return finish(y.reshape(shape))
        xa, _ = as_device_tensor(fa.data, dev)
        xb, _ = as_device_tensor(fb.data, dev)
        if xa.dtype != xb.dtype:
            return chain()
        pre_a = self._metric_tensor(self.get_metric(fa, ma_ax), fa.dims, xa) if ma_ax else None
        pre_b = self._metric_tensor(self.get_metric(fb, mb_ax), fb.dims, xb) if mb_ax else None
        post = self._metric_tensor(self.get_metric(probe, divide_by), out_dims_a, xa) if divide_by else None
        halo = {}
        if second.folded:
            halo["halo_lo_b"], halo["halo_hi_b"] = fold_halo_planes(self, second.ax_name, fb.dims, xb, second.lo,
                                                                    second.pad_mode, pre=pre_b, negate=negate)
        y = ops.stencil_pair(xa, xb, spec_a, spec_b, sub, pre_a=pre_a, pre_b=pre_b, post=post, **halo)
        return finish(result_like(y, host))

    def divergence(self, u, v, axis_u="X", axis_v="Y", **kwargs):
        """Finite-volume horizontal divergence ``(diff(u * dy, X) + diff(v * dx, Y)) / area`` on a C-grid, metrics
        from ``get_metric`` (u * its Y-metric, v * its X-metric, area at the output position); one fused pass."""
        return self.pair("diff", u, axis_u, "diff", v, axis_v, combine="add", metric_a=(axis_v,), metric_b=(axis_u,),
                         divide_by=(axis_u, axis_v), _components=(axis_u, axis_v), **kwargs)

    def vorticity(self, u, v, axis_u="X", axis_v="Y", **kwargs):
        """Vertical relative vorticity ``(diff(v * dy, X) - diff(u * dx, Y)) / area`` on a C-grid; one fused pass."""
        return self.pair("diff", v, axis_u, "diff", u, axis_v, combine="sub", metric_a=(axis_v,), metric_b=(axis_u,),
                         divide_by=(axis_u, axis_v), _components=(axis_v, axis_u), **kwargs)

    def apply_as_grid_ufunc(self, func: Callable, *args, axis=None, signature="", padding_width=None,
                            padding=None, fill_value=None, dask="forbidden", map_overlap=False,
                            **kwargs):
        """Apply a user function in a grid-aware manner (grid.py:866-968)."""
        if "boundary" in kwargs:
            raise ValueError(
                "Argument 'boundary' has been renamed to 'padding'. Please use 'padding' instead."
            )
        if "boundary_width" in kwargs:
            raise ValueError(
                "Argument 'boundary_width' has been renamed to 'padding_width'. "
                "Please use 'padding_width' instead."
            )
        return apply_as_grid_ufunc(
            func, *args, axis=axis, grid=self, signature=signature, padding_width=padding_width,
            padding=padding, fill_value=fill_value, dask=dask, map_overlap=map_overlap, **kwargs,
        )

    def interp(self, da, axis, **kwargs):
        """Interpolate neighbouring points to the intermediate position along ``axis``."""
        return self._1d_grid_ufunc_dispatch("interp", da, axis, **kwargs)

    def diff(self, da, axis, **kwargs):
        """Difference of neighbouring points, landing on the intermediate position."""
        return self._1d_grid_ufunc_dispatch("diff", da, axis, **kwargs)

    def min(self, da, axis, **kwargs):
        """Minimum of neighbouring points (NaN-propagating, like np.min)."""
        return self._1d_grid_ufunc_dispatch("min", da, axis, **kwargs)

    def max(self, da, axis, **kwargs):
        """Maximum of neighbouring points (NaN-propagating, like np.max)."""
        return self._1d_grid_ufunc_dispatch("max", da, axis, **kwargs)

    def derivative(self, da, axis, **kwargs):
        """Centered-difference derivative: ``diff(da, axis) / get_metric(diff, (axis,))``
        (grid.py:1534-1578), the divide fused into the stencil launch."""
        if not isinstance(axis, str):
            raise ValueError("derivative acts on a single axis; pass its name as a string")
        return self._1d_grid_ufunc_dispatch("diff", da, axis, _divide_by_metric_of=(axis,), **kwargs)

    # ------------------------------------------------------------------ cumsum family
    def cumsum(self, da, axis, to=None, padding=None, fill_value=None, metric_weighted=None,
               reverse=False, _pre_weight=None, **kwargs):
        """Cumulative sum moving to the intermediate position (grid.py:1183-1418).

        Per axis ONE ``xg_cumscan`` launch does metric multiply, (reverse) sequential
        cumsum, trim, boundary pad of the cumsum'd data and metric divide.
        """
        from . import ops
        from .device import as_device_tensor, result_like

        if "boundary" in kwargs:
            raise ValueError(
                "Argument 'boundary' has been renamed to 'padding'. Please use 'padding' instead."
            )
        if "keep_coords" in kwargs:
            raise ValueError(
                "The 'keep_coords' argument has been removed. Coordinates "
                "compatible with the output are now always preserved."
            )
        if kwargs:
            raise TypeError(f"cumsum() got unexpected keyword argument(s): {list(kwargs)}")
        da, as_xarray = self._wrap_in(da)
        if isinstance(axis, str):
            axis = [axis]
        to = self._map_kwargs_over_axes(to)
        if isinstance(reverse, dict):
            extra = [name for name in reverse if name not in axis]
            if extra:
                raise ValueError(
                    f"`reverse` was given for axes {extra} which are not being "
                    f"cumulatively summed (axis={axis}). Only pass `reverse` for "
                    f"the axes in `axis`."
                )
        reverse = self._map_kwargs_over_axes(reverse)
        if isinstance(metric_weighted, str):
            metric_weighted = (metric_weighted,)
        metric_weighted = self._map_kwargs_over_axes(metric_weighted)
        paddings = self._complete_user_kwargs_using_axis_defaults(padding, "padding")
        fills = self._complete_user_kwargs_using_axis_defaults(fill_value, "fill_value")

        def plan(ax_name):
            return self._cumsum_axis(da, ax_name, to, reverse, metric_weighted, paddings, fills)

        if len(axis) == 1 and _is_host_float(da):
            res = self._cumsum_host(da, plan(axis[0]), paddings, padding, fill_value, _pre_weight)
            if res is not None:
                return self._wrap_out(res, as_xarray)
        x, _ = as_device_tensor(da.data, self._device_for(da))
        data = da._replace(data=x)
        for ax_i, ax_name in enumerate(axis):
            s = plan(ax_name)
            input_da = data
            out_dims = tuple(s.new_dim if d == s.dim else d for d in data.dims)
            axis_num = data.get_axis_num(s.dim)
            pre_t = post_t = None
            probe = DataArray.__new__(DataArray)
            probe._dims = out_dims
            if s.weighted:
                pre_t = self._metric_tensor(self.get_metric(data, s.weighted), data.dims, data.data)
                post_t = self._metric_tensor(self.get_metric(probe, s.weighted), out_dims, data.data)
            if _pre_weight is not None and ax_i == 0:
                w_t = self._metric_tensor(_pre_weight, data.dims, data.data)
                if pre_t is None:
                    pre_t = w_t  # (da * w) is formed inside the scan kernel: 8 B/cell instead of 20
                else:  # two roundings in the reference, (da * w) * metric: keep them
                    data = data._replace(data=ops.binary("mul", data.data, w_t))
            if (self._face_connections is not None and (s.pad_lo or s.pad_hi)) or s.folded:
                # the reference pads the cumsum'd data with ``pad`` (grid.py:1385-1391), which on a
                # connected grid takes the halo from the neighbour face and across a north fold
                # mirrors the scanned rows: scan + trim in the kernel, halo through ``pad``, metric
                # divide last
                y = ops.cumscan(data.data, axis_num, s.reverse, s.trim, 0, 0, None, s.fill, pre=pre_t,
                                post=None, skipna=True)
                scanned = DataArray(y, dims=data.dims, name=da.name, attrs=da.attrs)
                y = pad(scanned, grid=self, padding_width={ax_name: (s.pad_lo, s.pad_hi)}, padding=padding,
                        fill_value=fill_value).data
                if post_t is not None:
                    y = ops.binary("div", y, post_t)
            else:
                y = ops.cumscan(data.data, axis_num, s.reverse, s.trim, s.pad_lo, s.pad_hi, s.bc, s.fill, pre=pre_t,
                                post=post_t, skipna=True)
            coordless = DataArray(y, dims=out_dims, name=da.name, attrs=da.attrs)
            data = _reattach_coords(
                [coordless], grid=self, padding_width={ax_name: (s.pad_lo, s.pad_hi)},
                out_core_dim_names={s.new_dim}, input_args=[input_da],
            )[0]
        if not da.is_device:
            data = data._replace(data=result_like(data.data, True))
        return self._wrap_out(data, as_xarray)

    def _cumsum_axis(self, da, ax_name, to, reverse, metric_weighted, paddings, fills) -> "_ScanAxis":
        """The shift table entry, boundary and metric of one axis of ``cumsum``; raises for an invalid shift and
        for a padded axis without a boundary condition."""
        ax = self.axes[ax_name]
        pos, dim = ax._get_position_name(da)
        ax_reverse = bool(reverse.get(ax.name, False))
        weighted = metric_weighted.get(ax.name) if isinstance(metric_weighted, dict) else None
        ax_to = to.get(ax.name) if isinstance(to, dict) else None
        if ax_to is None:
            ax_to = ax._default_shifts[pos]
        try:
            trim, (pad_lo, pad_hi) = (_CUMSUM_REV if ax_reverse else _CUMSUM_FWD)[(pos, ax_to)]
        except KeyError:
            raise ValueError(
                f"From `{pos}` to `{ax_to}` is not a valid position "
                f"shift for cumsum operation along axis {ax}."
            )
        folded, ax_padding = fold_edges(self, ax.name, paddings[ax.name], pad_hi)
        if (pad_lo or pad_hi) and ax_padding is None and self._face_connections is None:
            raise missing_boundary_error(ax.name)
        fv = fills[ax.name] if fills[ax.name] is not None else 0.0
        return _ScanAxis(ax.name, dim, ax.coords[ax_to], ax_reverse, weighted, trim, pad_lo, pad_hi, folded,
                         ax_padding if (pad_lo or pad_hi) else None, fv)

    def _cumsum_host(self, da, s, paddings, padding, fill_value, pre_weight):
        """One axis of ``cumsum`` on the numpy field ``da`` streamed through the GPU in slabs instead of one
        un-overlapped upload + download around the kernel: ``xg_cumscan_host``, or ``xg_cumscan_host_fold`` /
        ``_connected`` where the padded edge crosses a north fold or a face connection.  Those two run per slab
        the device route's scan, halo of the scanned field (as ``pad`` builds it) and divide by the post metric;
        their slabs are cut as the stencils cut them (``grid_ufunc._host_stream_route``) and the halo is planned
        for the scanned, merged layout.  Returns the result, or None: the whole-field route (a call with both
        cumint and metric_weighted, a per-side padding mapping, no batch dim in front of the halo dims, a fold the
        plan cannot mirror)."""
        from . import ops
        from .padding import connected_halo_program

        bc, fv, halo = s.bc, s.fill, None  # halo: the fold or face connection the padded edge crosses
        if self._face_connections is not None or s.ax_name in self._folds:
            if s.weighted and pre_weight is not None:
                return None
            if self._face_connections is not None and (s.pad_lo or s.pad_hi):
                if paddings[s.ax_name] not in (None, "periodic", "fill", "extend"):
                    return None  # e.g. a per-side mapping: pad() has the say
                if s.ax_name in _get_all_connection_axes(self._face_connections, self._facedim):
                    halo = "connected"
                else:  # e.g. Z on LLC: the basic boundary, checked as pad() checks it
                    bc, fv = connected_edge_mode(self, s.ax_name, s.pad_lo, s.pad_hi, padding, fill_value,
                                                 da.sizes[self._facedim])
            elif s.folded:
                halo = "fold"
        x, dims, shape = da.data, tuple(da.dims), [int(v) for v in da.shape]
        out_dims = tuple(s.new_dim if d == s.dim else d for d in dims)
        axis_num = dims.index(s.dim)
        pre = post = None
        if s.weighted:
            probe = DataArray.__new__(DataArray)
            probe._dims = out_dims
            pre = self._metric_host(self.get_metric(da, s.weighted), dims, x.dtype)
            post = self._metric_host(self.get_metric(probe, s.weighted), out_dims, x.dtype)
        if pre_weight is not None:  # cumint: the metric product rides on the kernel's pre operand
            if pre is not None:
                return None  # cumint with metric_weighted: two pre weights, the whole-field route
            pre = self._metric_host(pre_weight, dims, x.dtype)
        device = self._host_device(da)
        if halo is None:
            y = ops.cumscan_host(x, axis_num, s.reverse, s.trim, s.pad_lo, s.pad_hi, bc, fv, pre=pre, post=post,
                                 skipna=True, device=device)
        else:
            core = [s.dim] + _halo_core_dims(self, dims, s.ax_name)
            cut = _host_stream_route(halo, dims, shape, core, s.pad_lo, s.pad_hi,
                                     operand_shapes=[m.shape for m in (pre, post) if m is not None])
            if cut is None:
                return None
            scanned = list(shape)
            scanned[axis_num] -= 0 if s.trim == "none" else 1
            m_dims, m_scanned = cut.dims(dims), cut.shape(scanned)
            kw = dict(pre=cut.cut(pre), post=cut.cut(post), skipna=True, device=device)
            if halo == "fold":
                plan = cut.fold_plan(self, s.ax_name, dims, scanned)
                if plan is None:
                    return None
                y = ops.cumscan_host_fold(cut.cut(x), cut.axis(axis_num), s.reverse, s.trim, *plan, **kw)
            else:
                mode, fv = connected_edge_mode(self, s.ax_name, s.pad_lo, s.pad_hi, padding, fill_value,
                                               shape[dims.index(self._facedim)])
                program = connected_halo_program(self, s.ax_name, s.pad_lo, s.pad_hi, m_dims, m_scanned, mode)
                y = ops.cumscan_host_connected(cut.cut(x), cut.axis(axis_num), s.reverse, s.trim, s.pad_lo,
                                               s.pad_hi, fv, program, **kw)
            scanned[axis_num] += s.pad_lo + s.pad_hi
            y = y.reshape(scanned)
        coordless = DataArray(y, dims=out_dims, name=da.name, attrs=da.attrs)
        return _reattach_coords([coordless], grid=self, padding_width={s.ax_name: (s.pad_lo, s.pad_hi)},
                                out_core_dim_names={s.new_dim}, input_args=[da])[0]

    def cumint(self, da, axis, **kwargs):
        """Cumulative integral: ``cumsum(da * get_metric(da, axis), axis)`` (grid.py:1607-1660)."""
        da, as_xarray = self._wrap_in(da)
        weight = self.get_metric(da, axis)
        # the product da * metric is formed inside the scan kernel (its `pre` operand): one pass
        res = self.cumsum(da, axis, _pre_weight=weight, **kwargs)
        return self._wrap_out(res, as_xarray)

    # ------------------------------------------------------------------ reductions
    def _weighted_reduce(self, da, axis, mode, kwargs):
        from . import ops
        from .device import as_device_tensor, result_like

        da, as_xarray = self._wrap_in(da)
        skipna = kwargs.pop("skipna", None)
        min_count = kwargs.pop("min_count", None)
        keep_attrs = kwargs.pop("keep_attrs", None)  # accepted, attrs are dropped like xarray's default
        if kwargs:
            raise TypeError(f"unexpected keyword argument(s): {list(kwargs)}")
        if min_count is not None:
            # the reference forwards it to DataArray.sum; not fused here: refuse rather than ignore
            raise NotImplementedError("min_count is not supported by the fused integrate / average")
        if skipna is None:
            skipna = True  # xarray default for float data
        weight = self.get_metric(da, axis)
        dims = self._get_dims_from_axis(da, axis)

        def with_coords(res):
            return res.assign_coords({k: c for k, c in da.coords.items() if all(d in res.dims for d in c.dims)})

        y = self._weighted_reduce_host(da, dims, weight, mode, skipna) if _is_host_float(da) else None
        if y is not None:
            res = DataArray(y, dims=tuple(x_ for x_ in da.dims if x_ not in dims), name=da.name)
            return self._wrap_out(with_coords(res), as_xarray)
        x, _ = as_device_tensor(da.data, self._device_for(da))
        cur = da._replace(data=x)
        wt = self._metric_tensor(weight, cur.dims, x)
        # several axes: the first pass (innermost listed dim) applies the weights, the others are plain sums
        order = sorted(dims, key=lambda d: cur.get_axis_num(d), reverse=True)
        if mode == "mean" and len(order) > 1:
            # weighted mean over several dims = sum(x w over valid) / sum(w over valid): numerator and
            # denominator are reduced side by side (the kernel masks NaN cells itself: no full-size temp)
            num, den_src, first = cur, None, True
            for d in order:
                axn = num.get_axis_num(d)
                if first:
                    den = ops.wreduce(cur.data, axn, wt, "wvalid", bool(skipna))
                    numer = ops.wreduce(num.data, axn, wt, "sum", bool(skipna))
                    first = False
                else:
                    numer = ops.wreduce(num.data, axn, None, "sum", bool(skipna))
                    den = ops.wreduce(den_src.data, axn, None, "sum", False)
                keep = tuple(x_ for x_ in num.dims if x_ != d)
                num = DataArray(numer, dims=keep)
                den_src = DataArray(den, dims=keep)
            res = DataArray(ops.binary("divnz", num.data, den_src.data), dims=num.dims, name=da.name)
        else:
            first = True
            for d in order:
                axn = cur.get_axis_num(d)
                y = ops.wreduce(cur.data, axn, wt if first else None, mode, bool(skipna))
                first = False
                cur = DataArray(y, dims=tuple(x_ for x_ in cur.dims if x_ != d), name=da.name)
            res = cur
        res = with_coords(res)
        if not da.is_device:
            res = res._replace(data=result_like(res.data, True))
        return self._wrap_out(res, as_xarray)

    def _weighted_reduce_host(self, da, dims, weight, mode, skipna):
        """``integrate`` / ``average`` of the numpy field ``da`` over ``dims`` streamed through the GPU in slabs:
        ``xg_wreduce_host`` for one dim, ``xg_wreduce_host_multi`` for several (the launches of the device route
        run per slab, with a weight that spans the slab dim streamed beside the field).  Returns the reduced
        array, or None: the whole-field route."""
        from . import ops

        if len(dims) == 1:
            w_np = self._metric_host(weight, da.dims, da.data.dtype)
            return ops.wreduce_host(da.data, da.get_axis_num(dims[0]), w_np, mode, bool(skipna),
                                    device=self._host_device(da))
        if not (len(set(dims)) == len(dims) > 1 and self._device_for(da).type == "cuda"):
            return None
        w_np = self._metric_host(weight, da.dims, da.data.dtype)
        try:
            return ops.wreduce_host_multi(da.data, [da.get_axis_num(d) for d in dims], w_np, mode, bool(skipna),
                                          device=self._host_device(da))
        except NotImplementedError:
            return None  # an empty reduced dim, or a single line: the whole field on the device

    def integrate(self, da, axis, **kwargs):
        """Finite-volume integral ``(da * metric).sum(dim)`` (grid.py:1580-1605), fused."""
        return self._weighted_reduce(da, axis, "sum", dict(kwargs))

    def average(self, da, axis, **kwargs):
        """Metric-weighted mean ignoring NaNs (grid.py:1662-1685), fused."""
        return self._weighted_reduce(da, axis, "mean", dict(kwargs))

    # ------------------------------------------------------------------ vertical transform
    def transform(self, da, axis, target, **kwargs):
        """Convert ``da`` to new 1-D coordinates along ``axis`` (grid.py:1687-1776)."""
        from .transform import transform

        da, as_xarray = self._wrap_in(da)
        if "target_data" in kwargs and kwargs["target_data"] is not None:
            kwargs["target_data"], _ = self._wrap_in(kwargs["target_data"])
        target, _ = self._wrap_in(target)
        return self._wrap_out(transform(self, axis, da, target, **kwargs), as_xarray)

    # deprecated 2-D vector wrappers of the reference (grid.py:1420-1532) are not carried over
    def _apply_vector_function(self, function, vector, **kwargs):
        """Apply diff / interp to both components of a C-grid vector, each padded with the other
        as its partner across rotated face connections (grid.py:1420-1474)."""
        if not (isinstance(vector, dict) and len(vector) == 2):
            raise ValueError(
                "Input is expected to be a dictionary with two key/value pairs which map grid axis "
                "to the vector component parallel to that axis"
            )
        warnings.warn(
            "`interp_2d_vector` and `diff_2d_vector` will be removed from future releases."
            "The same functionality will be accessible under the `xgcm.Grid.diff` and "
            "`xgcm.Grid.interp` methods, please see those docstrings for details.",
            category=DeprecationWarning,
        )
        to = kwargs.get("to", "center")
        if to != "center":
            raise NotImplementedError(
                "Only vector interpolation to cell center is implemented, but got to=%r" % to
            )
        for axis_name, component in vector.items():
            position, _ = self.axes[axis_name]._get_position_name(component)
            if position == "center":
                raise NotImplementedError(
                    "Only vector interpolation to cell center is implemented, but vector %s "
                    "component is defined at center (dims: %r)" % (axis_name, component.dims)
                )
        x_axis_name, y_axis_name = list(vector)
        x_component = function(
            {x_axis_name: vector[x_axis_name]}, x_axis_name,
            other_component={y_axis_name: vector[y_axis_name]}, **kwargs,
        )
        y_component = function(
            {y_axis_name: vector[y_axis_name]}, y_axis_name,
            other_component={x_axis_name: vector[x_axis_name]}, **kwargs,
        )
        return {x_axis_name: x_component, y_axis_name: y_component}

    def diff_2d_vector(self, vector, **kwargs):
        """Difference a 2-D vector to the intermediate grid point (grid.py:1476-1495)."""
        return self._apply_vector_function(self.diff, vector, **kwargs)

    def interp_2d_vector(self, vector, **kwargs):
        """Interpolate a 2-D vector to the intermediate grid point (grid.py:1497-1530)."""
        return self._apply_vector_function(self.interp, vector, **kwargs)


class _StencilTerm(NamedTuple):
    """One built-in stencil (diff / interp / min / max) of a field along one axis, as the fused launches take it."""

    op: str
    ax_name: str
    lo: int
    hi: int
    in_dim: str
    out_dim: str
    axis_num: int
    pad_mode: Optional[str]
    fill: float
    folded: bool


def _stencil_term(grid, funcname, da, ax_name, to, paddings, fills) -> _StencilTerm:
    """Resolve ``funcname`` of ``da`` along ``ax_name`` to position ``to`` (None: the axis default shift): the
    gridops ufunc and its padding, the dims in and out, the boundary (``paddings`` / ``fills`` completed with
    the Axis defaults) and whether the north edge folds.  Raises for a position the axis does not have and for
    a padded axis without a boundary condition."""
    sig = grid._create_1d_grid_ufunc_signatures(da, axis=[ax_name], to={ax_name: to})[0]
    grid_ufunc, _ = _select_grid_ufunc(funcname, sig, module=gridops)
    dummy = grid_ufunc.signature.in_ax_names[0][0]  # the ufunc's own dummy axis name ("X")
    lo, hi = (grid_ufunc.padding_width or {}).get(dummy, (0, 0))
    from_pos, to_pos = sig.in_ax_positions[0][0], sig.out_ax_positions[0][0]
    coords = grid.axes[ax_name].coords
    if to_pos not in coords:
        raise ValueError(f"Axis position ({ax_name}:{to_pos}) does not exist in grid")
    folded, pad_mode, fill = _stencil_boundary(grid, ax_name, lo, hi, paddings, fills)
    in_dim = coords[from_pos]
    return _StencilTerm(funcname, ax_name, lo, hi, in_dim, coords[to_pos], da.get_axis_num(in_dim), pad_mode, fill,
                        folded)


class _ScanAxis(NamedTuple):
    """One axis of ``Grid.cumsum``: its dims, direction, metric, shift table entry and boundary."""

    ax_name: str
    dim: str
    new_dim: str
    reverse: bool
    weighted: Any
    trim: str
    pad_lo: int
    pad_hi: int
    folded: bool
    bc: Optional[str]
    fill: float


# (from, to) -> (trim, (pad_lo, pad_hi)); transcription of the enumerated shifts of
# reference grid.py:1326-1383
_CUMSUM_FWD = {
    ("center", "right"): ("none", (0, 0)),
    ("left", "center"): ("none", (0, 0)),
    ("center", "left"): ("drop_last", (1, 0)),
    ("right", "center"): ("drop_last", (1, 0)),
    ("center", "inner"): ("drop_last", (0, 0)),
    ("outer", "center"): ("drop_last", (0, 0)),
    ("center", "outer"): ("none", (1, 0)),
    ("inner", "center"): ("none", (1, 0)),
}
_CUMSUM_REV = {
    ("center", "left"): ("none", (0, 0)),
    ("right", "center"): ("none", (0, 0)),
    ("center", "right"): ("drop_first", (0, 1)),
    ("left", "center"): ("drop_first", (0, 1)),
    ("center", "inner"): ("drop_first", (0, 0)),
    ("outer", "center"): ("drop_first", (0, 0)),
    ("center", "outer"): ("none", (0, 1)),
    ("inner", "center"): ("none", (0, 1)),
}


_SELECTED_UFUNCS: Dict[tuple, "GridUFunc"] = {}


def _select_grid_ufunc(funcname, signature: _GridUFuncSignature, module, **kwargs):
    """Pick the GridUFunc of ``module`` whose name starts with ``funcname`` and whose
    signature is equivalent (grid.py:1779-1824).  The scan is memoised per (module, name,
    signature text): it is pure, and at BASELINE configs[0] sizes it cost more than the kernel."""
    key = (module.__name__, funcname, str(signature))
    hit = _SELECTED_UFUNCS.get(key)
    if hit is not None:
        return hit, kwargs
    candidates = inspect.getmembers(module, lambda obj: isinstance(obj, GridUFunc))
    by_name = [f for name, f in candidates if name.startswith(funcname)]
    if not by_name:
        raise NotImplementedError(f"Could not find any pre-defined {funcname} grid ufuncs")
    matching = [f for f in by_name if f.signature.equivalent(signature)]
    if not matching:
        raise NotImplementedError(
            f"Could not find any pre-defined {funcname} grid ufuncs with signature {signature}"
        )
    if len(matching) > 1:
        raise ValueError(
            f"Function {funcname} with signature='{signature}' and kwargs={kwargs} is an ambiguous selection"
        )
    _SELECTED_UFUNCS[key] = matching[0]
    return matching[0], kwargs
