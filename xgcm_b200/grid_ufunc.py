"""Grid-ufunc engine: signatures, ``GridUFunc``, ``as_grid_ufunc``, ``apply_as_grid_ufunc``.

Same public surface and error behaviour as the reference's ``xgcm/grid_ufunc.py``
(signature grammar :31-43,266-362; ``equivalent`` :230-263; ``GridUFunc`` :373-562;
``apply_as_grid_ufunc`` :661-951), but the numerics are different by design:

* a built-in 1-D operator (``gridops.*``, tagged with ``kernel_op``) never
  materialises a padded copy — halo, operator and optional metric weighting run
  as ONE ``xg_stencil2`` launch (the reference does ``pad`` -> ``apply_ufunc`` ->
  two more metric passes, grid_ufunc.py:905-924, grid.py:806-832);
* a user-supplied python ufunc still works: its inputs are padded on the device
  (``xg_pad``) and handed to the user's function as numpy arrays with the core
  dims moved last, exactly as ``xr.apply_ufunc`` would.

dask ``map_overlap`` (grid_ufunc.py:1057-1223) is out of scope: the multi-GPU
analogue is ``xgcm_b200.parallel``.
"""

from __future__ import annotations

import re
import string
import collections.abc
from typing import Any, Callable, Dict, List, Mapping, Optional, Sequence, Tuple, Union, get_type_hints

import numpy as np

from .labeled import DataArray
from .padding import pad

_AXIS_NAME = r"\w+"
_AXIS_POSITION = "(?:center|left|right|inner|outer)"
_PAIR = f"{_AXIS_NAME}:{_AXIS_POSITION}"
_PAIR_LIST = f"(?:{_PAIR}(?:,{_PAIR})*,?)*"
_ARGUMENT = rf"\({_PAIR_LIST}\)"
_ARGUMENT_LIST = f"{_ARGUMENT}(?:,{_ARGUMENT})*"
_SIGNATURE = f"^{_ARGUMENT_LIST}->{_ARGUMENT_LIST}$"

T_AX_POS_LIST = List[Tuple[str, ...]]


def _maybe_unpack_vector_component(data):
    if isinstance(data, dict):
        [da] = list(data.values())
        return da
    return data


def _is_dataarray(obj) -> bool:
    return isinstance(obj, DataArray)


def _check_data_input(data, grid):
    """A scalar field (DataArray) or a single vector component ({axis: DataArray})."""
    if data is None:
        return data
    if not (_is_dataarray(data) or isinstance(data, dict)):
        raise TypeError(
            f"All data arguments must be either a DataArray or Dictionary Got {type(data)}."
        )
    if isinstance(data, dict):
        if len(data) != 1:
            raise ValueError(
                "Vector components provided as dictionaries should contain exactly one key/value pair."
                f" Found {len(data)}. Full input:{data}"
            )
        [(key, value)] = data.items()
        if key not in grid.axes:
            raise ValueError(
                f"Vector component with unknown axis provided. Grid has axes ({list(grid.axes)}), got  ({key})"
            )
        if not _is_dataarray(value):
            raise TypeError(f"Dictionary inputs must have a DataArray as value. Got {type(value)}.")
    return data


class _GridUFuncSignature:
    """Axis names and positions of every input / output of a grid ufunc."""

    _REPLACEMENT_DUMMY_INDEX_NAMES = [f"__{c}" for c in string.ascii_letters]

    def __init__(self, in_ax_names, in_ax_positions, out_ax_names, out_ax_positions):
        if not in_ax_names or not in_ax_positions:
            raise ValueError(
                "At least one input argument of the Grid UFunc signature must have "
                "axis names and positions"
            )
        self.in_ax_names = in_ax_names
        self.in_ax_positions = in_ax_positions
        self.out_ax_names = out_ax_names
        self.out_ax_positions = out_ax_positions

    @staticmethod
    def _side(names, positions):
        args = [",".join(f"{a}:{p}" for a, p in zip(n, ps)) for n, ps in zip(names, positions)]
        return ",".join(f"({a})" for a in args)

    def __str__(self):
        text = self.__dict__.get("_text")
        if text is None:
            text = self._text = (
                f"{self._side(self.in_ax_names, self.in_ax_positions)}->"
                f"{self._side(self.out_ax_names, self.out_ax_positions)}"
            )
        return text

    def __repr__(self):
        return f"_GridUFuncSignature('{self}')"

    _PARSED: Dict[str, "_GridUFuncSignature"] = {}

    @classmethod
    def from_string(cls, signature: str) -> "_GridUFuncSignature":
        # signatures are never mutated after construction, so the parse is shared
        hit = cls._PARSED.get(signature) if cls is _GridUFuncSignature else None
        if hit is None:
            hit = cls(*_parse_signature_from_string(signature))
            if cls is _GridUFuncSignature and len(cls._PARSED) < 4096:
                cls._PARSED[signature] = hit
        return hit

    @classmethod
    def from_type_hints(cls, hints: Dict[str, Any]) -> "_GridUFuncSignature":
        return cls(*_parse_signature_from_type_hints(hints))

    def equivalent(self, other: "_GridUFuncSignature") -> bool:
        """Equal up to a consistent renaming of the dummy axis names."""

        def first_seen(sig):
            order = []
            for side in (sig.in_ax_names, sig.out_ax_names):
                for arg in side:
                    for ax in arg:
                        if ax not in order:
                            order.append(ax)
            return order

        mine, theirs = first_seen(self), first_seen(other)
        if len(mine) != len(theirs):
            return False

        def canon(sig, order):
            ren = dict(zip(order, self._REPLACEMENT_DUMMY_INDEX_NAMES))
            return (
                [tuple(ren[a] for a in arg) for arg in sig.in_ax_names],
                [tuple(p) for p in sig.in_ax_positions],
                [tuple(ren[a] for a in arg) for arg in sig.out_ax_names],
                [tuple(p) for p in sig.out_ax_positions],
            )

        return canon(self, mine) == canon(other, theirs)


def _split_args(txt):
    names, positions = [], []
    for arg in re.findall(_ARGUMENT, txt):
        positions.append(tuple(re.findall(_AXIS_POSITION, arg)))
        only_names = re.sub(_AXIS_POSITION, "", arg)
        names.append(tuple(re.findall(_AXIS_NAME, only_names)))
    return names, positions


def _parse_signature_from_string(signature: str):
    signature = signature.replace(" ", "")
    if not re.match(_SIGNATURE, signature):
        raise ValueError(f"Not a valid grid ufunc signature: {signature}")
    in_txt, out_txt = signature.split("->")
    in_names, in_pos = _split_args(in_txt)
    out_names, out_pos = _split_args(out_txt)
    return in_names, in_pos, out_names, out_pos


def _maybe_multiple_return_vals(return_hint):
    if getattr(return_hint, "_name", None) == "Tuple":
        return list(return_hint.__args__)
    return [return_hint]


def _annotation_strings(hints):
    return [h.__metadata__[0] for h in hints if hasattr(h, "__metadata__")]


def _parse_signature_from_type_hints(hints: Dict[str, Any]):
    hints = dict(hints)
    if "return" in hints:
        ret = _annotation_strings(_maybe_multiple_return_vals(hints.pop("return")))
        out_names, out_pos = [], []
        for ann in ret:
            out_pos.append(tuple(re.findall(_AXIS_POSITION, ann)))
            out_names.append(tuple(re.findall(_AXIS_NAME, re.sub(_AXIS_POSITION, "", ann))))
    else:
        out_names, out_pos = [()], [()]
    in_names, in_pos = [], []
    for ann in _annotation_strings(hints.values()):
        in_pos.append(tuple(re.findall(_AXIS_POSITION, ann)))
        in_names.append(tuple(re.findall(_AXIS_NAME, re.sub(_AXIS_POSITION, "", ann))))
    text = str(_GridUFuncSignature(in_names, in_pos, out_names, out_pos))
    if not re.match(_SIGNATURE, text):
        raise ValueError(f"Not a valid grid ufunc signature: {text}")
    return in_names, in_pos, out_names, out_pos


def _deprecated_kwargs(kwargs):
    if "boundary" in kwargs:
        raise ValueError(
            "Argument 'boundary' has been renamed to 'padding'. Please use 'padding' instead."
        )
    if "boundary_width" in kwargs:
        raise ValueError(
            "Argument 'boundary_width' has been renamed to 'padding_width'. "
            "Please use 'padding_width' instead."
        )


class GridUFunc:
    """A function bound to a grid signature; calling it goes through ``apply_as_grid_ufunc``.

    ``kernel_op`` (one of ``diff, interp, min, max``) marks the built-in operators
    whose pad + arithmetic + metric weighting run fused in ``xg_stencil2``.
    """

    def __init__(self, ufunc: Callable, **kwargs):
        self.ufunc = ufunc
        _deprecated_kwargs(kwargs)
        str_sig = kwargs.pop("signature")
        self.signature = self._get_signature_from_str_or_type_hints(ufunc, str_sig)
        self.padding_width = kwargs.pop("padding_width", None)
        self.padding = kwargs.pop("padding", None)
        self.fill_value = kwargs.pop("fill_value", None)
        self.dask = kwargs.pop("dask", "forbidden")
        self.map_overlap = kwargs.pop("map_overlap", False)
        self.pad_before_func = kwargs.pop("pad_before_func", True)
        self.kernel_op = kwargs.pop("kernel_op", getattr(ufunc, "kernel_op", None))
        if kwargs:
            raise TypeError(f"Unsupported keyword argument(s) provided: {list(kwargs.keys())}")

    @staticmethod
    def _get_signature_from_str_or_type_hints(ufunc, str_sig):
        try:
            hints = get_type_hints(ufunc, include_extras=True)
        except Exception:
            hints = {}

        def has_annotations(h):
            if "return" in h:
                if any(hasattr(x, "__metadata__") for x in _maybe_multiple_return_vals(h["return"])):
                    return True
            return any(hasattr(x, "__metadata__") for x in h.values())

        if str_sig:
            if has_annotations(hints):
                raise ValueError(
                    "Must specify axis positions through only one of either type hints or signature kwarg, not both."
                )
            return _GridUFuncSignature.from_string(str_sig)
        if not has_annotations(hints):
            raise ValueError("Must specify axis positions through either type hints or signature kwarg")
        return _GridUFuncSignature.from_type_hints(hints)

    def __repr__(self):
        return (
            f"GridUFunc(ufunc={self.ufunc}, signature='{self.signature}', padding_width='{self.padding_width}', "
            f"          padding='{self.padding}', dask='{self.dask})', map_overlap={self.map_overlap}, pad_before_func={self.pad_before_func})"
        )

    @property
    def boundary(self):
        raise AttributeError(
            "Attribute 'boundary' has been renamed to 'padding'. Please use 'padding' instead."
        )

    @property
    def boundary_width(self):
        raise AttributeError(
            "Attribute 'boundary_width' has been renamed to 'padding_width'. "
            "Please use 'padding_width' instead."
        )

    def __call__(self, grid=None, *args, axis, **kwargs):
        if "boundary" in kwargs:
            raise ValueError(
                "Argument 'boundary' has been renamed to 'padding'. Please use 'padding' instead."
            )
        padding = kwargs.pop("padding", self.padding)
        fill_value = kwargs.pop("fill_value", self.fill_value)
        dask = kwargs.pop("dask", self.dask)
        map_overlap = kwargs.pop("map_overlap", self.map_overlap)
        pad_before_func = kwargs.pop("pad_before_func", self.pad_before_func)
        return apply_as_grid_ufunc(
            self.ufunc,
            *args,
            axis=axis,
            grid=grid,
            signature=self.signature,
            padding_width=self.padding_width,
            padding=padding,
            fill_value=fill_value,
            dask=dask,
            map_overlap=map_overlap,
            pad_before_func=pad_before_func,
            _kernel_op=self.kernel_op,
            **kwargs,
        )


def as_grid_ufunc(signature: str = "", padding_width=None, **kwargs) -> Callable:
    """Decorator turning an array function into a grid-aware ufunc (grid_ufunc.py:565-658)."""
    _deprecated_kwargs(kwargs)
    allowed = {"padding", "fill_value", "dask", "map_overlap", "pad_before_func", "kernel_op"}
    forbidden = list(kwargs.keys() - allowed)
    if forbidden:
        raise TypeError(f"Unsupported keyword argument(s) provided: {forbidden}")

    def _as_grid_ufunc(ufunc):
        return GridUFunc(ufunc, signature=signature, padding_width=padding_width, **kwargs)

    return _as_grid_ufunc


def _promote_to_sequence_and_check(data, grid):
    if not isinstance(data, (list, tuple, collections.abc.Sequence)):  # (typing.Sequence checks are ~10x slower)
        data = [data]
    return [_check_data_input(d, grid) for d in data]


def _identify_dummy_axes_with_real_axes(sig_in_dummy_ax_names, axis) -> Mapping[str, str]:
    if len(axis) != len(sig_in_dummy_ax_names):
        raise ValueError(
            "Number of entries in `axis` does not match the number of variables in the input signature"
        )
    for i, (arg_axes, dummy_arg_axes) in enumerate(zip(axis, sig_in_dummy_ax_names)):
        if len(arg_axes) != len(dummy_arg_axes):
            raise ValueError(
                f"Number of Axes in `axis` entry number {i} does not match the number of Axes in that entry in the input signature"
            )
    unique_dummy = list(dict.fromkeys(ax for arg in sig_in_dummy_ax_names for ax in arg))
    unique_real = list(dict.fromkeys(ax for arg in axis for ax in arg))
    if len(unique_dummy) != len(unique_real):
        raise ValueError(
            f"Found {len(unique_dummy)} unique input axes in signature but {len(unique_real)} "
            f"real unique input axes were supplied to the grid ufunc when called"
        )
    return dict(zip(unique_dummy, unique_real))


def _substitute_dummy_axis_names(padding_width, mapping):
    if padding_width:
        return {mapping[ax]: tuple(width) for ax, width in padding_width.items()}
    return {real: (0, 0) for real in mapping.values()}


def _grid_coords_on(grid, dims):
    """The coordinates of ``grid._ds`` that live on ``dims`` only.  Memoised per grid and dim tuple (keyed on
    the dataset's coordinate and variable names, so a dataset edited in place is seen): building the dataset's
    coordinate view costs more host time per call than the kernel of a small field."""
    ds = grid._ds
    stamp = (tuple(getattr(ds, "_coord_names", ())), len(getattr(ds, "_vars", ())))
    cache = grid.__dict__.setdefault("_coords_on_cache", {})
    hit = cache.get(dims)
    if hit is not None and hit[0] == stamp:
        return hit[1]
    dimset = set(dims)
    found = {cname: c for cname, c in ds.coords.items() if all(d in dimset for d in c.dims)}
    cache[dims] = (stamp, found)
    return found


def _reattach_coords(results, grid, padding_width, out_core_dim_names=None, input_args=None):
    """Coordinates of position-shifted dims come from ``grid._ds``; coordinates living
    purely on untouched dims are kept from the inputs (grid_ufunc.py:1262-1320)."""
    out_core_dim_names = set(out_core_dim_names or ())
    input_coords = {}
    for arg in input_args or []:
        for cname, c in arg.coords.items():
            if any(d in out_core_dim_names for d in c.dims):
                continue
            input_coords.setdefault(cname, c)
    out = []
    for res in results:
        matching = dict(_grid_coords_on(grid, tuple(res.dims)))
        for cname, c in input_coords.items():
            if all(d in res.dims for d in c.dims):
                matching[cname] = c
        try:
            res = res.assign_coords(matching)
        except ValueError as err:
            if padding_width and str(err).startswith("conflicting sizes"):
                raise ValueError(
                    f"{str(err)} - does your grid ufunc correctly trim off the same number of elements "
                    f"which were added by padding using padding_width={padding_width}?"
                )
            raise
        out.append(res)
    return out


def _restore_input_dim_order(results, args, sig, in_core_dims, out_core_dims):
    """Outputs follow the inputs' dim order, core dims renamed (grid_ufunc.py:56-103)."""
    dummy_in = {
        ax: dim
        for names, dims in zip(sig.in_ax_names, in_core_dims)
        for ax, dim in zip(names, dims)
    }
    dummy_out = {
        ax: dim
        for names, dims in zip(sig.out_ax_names, out_core_dims)
        for ax, dim in zip(names, dims)
    }
    rename = {dummy_in[ax]: dummy_out[ax] for ax in dummy_in if ax in dummy_out}
    order: List[str] = []
    for arg in args:
        for d in _maybe_unpack_vector_component(arg).dims:
            d = rename.get(d, d)
            if d not in order:
                order.append(d)
    out = []
    for res in results:
        want = [d for d in order if d in res.dims] + [d for d in res.dims if d not in order]
        out.append(res.transpose(*want))
    return tuple(out)


def apply_as_grid_ufunc(
    func: Callable,
    *args,
    axis: Optional[Sequence[Sequence[str]]] = None,
    grid=None,
    signature: Union[str, _GridUFuncSignature] = "",
    padding_width: Optional[Mapping[str, Tuple[int, int]]] = None,
    padding=None,
    fill_value=None,
    dask: str = "forbidden",
    map_overlap: bool = False,
    pad_before_func: bool = True,
    other_component=None,
    **kwargs,
):
    """Apply ``func`` to labelled arrays in a grid-aware manner (grid_ufunc.py:661-951)."""
    _deprecated_kwargs(kwargs)
    if "keep_coords" in kwargs:
        raise ValueError(
            "The 'keep_coords' argument has been removed. Coordinates "
            "compatible with the output are now always preserved."
        )
    kernel_op = kwargs.pop("_kernel_op", getattr(func, "kernel_op", None))
    pre_metric = kwargs.pop("_pre_metric", None)
    post_metric_fn = kwargs.pop("_post_metric", None)

    if grid is None:
        raise ValueError("Must provide a grid object to describe the Axes")
    if map_overlap:
        raise NotImplementedError(
            "dask map_overlap is outside the scope of xgcm_b200; use xgcm_b200.parallel for "
            "multi-GPU sharding (with a halo exchange when the operated axis is sharded)"
        )

    args = _promote_to_sequence_and_check(args, grid)
    other_component = _promote_to_sequence_and_check(other_component, grid)
    if len(other_component) == 1 and other_component[0] is None:
        other_component = other_component * len(args)
    if len(args) != len(other_component):
        raise ValueError(
            "When providing multiple input arguments, `other_component`"
            " needs to provide one dictionary per input."
        )
    if axis is None:
        raise ValueError("Must provide an axis along which to apply the grid ufunc")
    if len(args) != len(axis):
        raise ValueError(
            "Number of entries in `axis` does not match the number of data arguments supplied"
        )

    sig = signature if isinstance(signature, _GridUFuncSignature) else _GridUFuncSignature.from_string(signature)
    dummy_to_real = _identify_dummy_axes_with_real_axes(sig.in_ax_names, axis)
    out_ax_names = [[dummy_to_real[ax] for ax in arg] for arg in sig.out_ax_names]

    # inputs must sit on the positions the signature states (grid_ufunc.py:827-842)
    for i, (arg_ns, arg_ps, arg) in enumerate(zip(axis, sig.in_ax_positions, args)):
        for n, p in zip(arg_ns, arg_ps):
            try:
                ax_pos = grid.axes[n].coords[p]
            except KeyError:
                raise ValueError(f"Axis position ({n}:{p}) does not exist in grid")
            arr = _maybe_unpack_vector_component(arg)
            if ax_pos not in arr.dims:
                raise ValueError(
                    f"Mismatch between signature and input argument {i}: "
                    f"Signature specified data to lie at Axis Position ({n}:{p}), "
                    f"but the corresponding grid coordinate {grid.axes[n].coords[p]} "
                    f"does not appear in argument"
                    f"{arr}"
                )

    in_core_dims = [
        [grid.axes[n].coords[p] for n, p in zip(arg_ns, arg_ps)]
        for arg_ns, arg_ps in zip(axis, sig.in_ax_positions)
    ]
    try:
        out_core_dims = [
            [grid.axes[n].coords[p] for n, p in zip(arg_ns, arg_ps)]
            for arg_ns, arg_ps in zip(out_ax_names, sig.out_ax_positions)
        ]
    except KeyError as err:
        raise ValueError(f"Output axis position {err} does not exist in grid")

    padding_width_real = _substitute_dummy_axis_names(padding_width, dummy_to_real)
    input_arrays = [_maybe_unpack_vector_component(a) for a in args]

    fused = (
        kernel_op is not None
        and pad_before_func
        and len(args) == 1
        and len(in_core_dims[0]) == 1
        and len(out_core_dims) == 1
        and len(out_core_dims[0]) == 1
    )
    if fused:
        results = (
            _apply_fused_stencil(
                kernel_op, input_arrays[0], grid, axis[0][0], in_core_dims[0][0],
                out_core_dims[0][0], padding_width_real, padding, fill_value,
                pre_metric, post_metric_fn, raw_arg=args[0], other_component=other_component[0],
            ),
        )
    else:
        if pre_metric is not None or post_metric_fn is not None:
            raise NotImplementedError("metric fusion is only available for built-in 1-D operators")
        results = _apply_generic(
            func, args, input_arrays, grid, in_core_dims, out_core_dims, padding_width_real,
            padding, fill_value, other_component, pad_before_func, kwargs,
        )

    out_core_dim_names = set(d for arg in out_core_dims for d in arg)
    results = _reattach_coords(results, grid, padding_width, out_core_dim_names, input_arrays)
    results = _restore_input_dim_order(results, args, sig, in_core_dims, out_core_dims)
    if len(results) == 1:
        (results,) = results
    return results


def _apply_connected_stencil(op, da, raw_arg, other_component, grid, ax_name, in_dim, out_dim,
                             padding_width_real, padding, fill_value, pre_metric, post_metric_fn):
    """Built-in operator on a grid with face connections: the halo is not an affine function of
    the field any more (it comes from other faces, rotated), so it is materialised once by
    ``pad`` -> ``xg_strided_copy`` and the stencil then runs on the padded array without a
    boundary condition (reference: grid_ufunc.py:903-921 pads, then applies the kernel)."""
    from . import ops
    from .device import as_device_tensor, result_like
    from .padding import pad

    lo, hi = padding_width_real.get(ax_name, (0, 0))
    if pre_metric is None and lo <= 1 and hi <= 1:
        streamed = _stream_connected_stencil(op, raw_arg, other_component, grid, ax_name, in_dim, out_dim, lo, hi,
                                             padding, fill_value, post_metric_fn)
        if streamed is not None:
            return streamed
        # halo planes gathered from the neighbour faces, then the ordinary fused launch
        from .padding import connected_halo_planes

        x, halo_lo, halo_hi, was_host, dims = connected_halo_planes(
            raw_arg, grid, ax_name, lo, hi, padding, fill_value, other_component)
        axis_num = dims.index(in_dim)
        out_dims = tuple(out_dim if d == in_dim else d for d in dims)
        out_shape = list(x.shape)
        out_shape[axis_num] = x.shape[axis_num] + lo + hi - 1
        post_da = post_metric_fn(_ShapeProbe(out_dims, out_shape)) if post_metric_fn is not None else None
        post_t = grid._metric_tensor(post_da, out_dims, x) if post_da is not None else None
        out = ops.stencil2(x, axis_num, op, lo, hi, "fill" if (lo or hi) else None, 0.0,
                           post=post_t, halo_lo=halo_lo, halo_hi=halo_hi)
        return DataArray(result_like(out, was_host), dims=out_dims, name=da.name, attrs=da.attrs)
    if pre_metric is not None:
        if isinstance(raw_arg, dict):
            raise NotImplementedError(
                "metric weighting of vector components across face connections is not implemented"
            )
        x, was_host = as_device_tensor(da.data, grid._device_for(da))
        x = ops.binary("mul", x, grid._metric_tensor(pre_metric, da.dims, x))
        weighted = DataArray(result_like(x, was_host), dims=da.dims, name=da.name, attrs=da.attrs)
        raw_arg = weighted
    padded = pad(raw_arg, grid=grid, padding_width={ax_name: (lo, hi)}, padding=padding,
                 fill_value=fill_value, other_component=other_component)
    if isinstance(padded, dict):  # zero-width request: pad returns its input untouched
        [padded] = list(padded.values())
    axis_num = padded.get_axis_num(in_dim)
    out_dims = tuple(out_dim if d == in_dim else d for d in padded.dims)
    out_shape = list(padded.shape)
    out_shape[axis_num] = padded.shape[axis_num] - 1
    post_da = post_metric_fn(_ShapeProbe(out_dims, out_shape)) if post_metric_fn is not None else None
    x, was_host = as_device_tensor(padded.data, grid._device_for(padded))
    post_t = grid._metric_tensor(post_da, out_dims, x) if post_da is not None else None
    out = ops.stencil2(x, axis_num, op, 0, 0, None, post=post_t)
    return DataArray(result_like(out, was_host), dims=out_dims, name=da.name, attrs=da.attrs)


def _apply_fused_stencil(op, da, grid, ax_name, in_dim, out_dim, padding_width_real, padding,
                         fill_value, pre_metric, post_metric_fn, raw_arg=None, other_component=None):
    """One ``xg_stencil2`` launch: halo + operator + metric weighting."""
    from . import ops
    from .device import as_device_tensor, result_like

    if grid._face_connections is not None:
        return _apply_connected_stencil(
            op, da, da if raw_arg is None else raw_arg, other_component, grid, ax_name, in_dim,
            out_dim, padding_width_real, padding, fill_value, pre_metric, post_metric_fn,
        )
    from .padding import fold_edges, fold_halo_planes

    lo, hi = padding_width_real.get(ax_name, (0, 0))
    paddings = grid._complete_user_kwargs_using_axis_defaults(padding, "padding")
    fills = grid._complete_user_kwargs_using_axis_defaults(fill_value, "fill_value")
    folded, ax_padding = fold_edges(grid, ax_name, paddings[ax_name], hi)
    if (lo or hi) and ax_padding is None:
        raise ValueError(
            f"No boundary condition was specified for axis {ax_name!r}, but the "
            f"requested operation needs to pad it. Set a boundary condition, "
            f"e.g. ``padding='fill'`` (or 'extend'/'periodic'), on the Grid "
            f"(``Grid(..., padding=...)``) or pass ``padding=`` to the "
            f"grid method."
        )
    axis_num = da.get_axis_num(in_dim)
    out_dims = tuple(out_dim if d == in_dim else d for d in da.dims)
    out_shape = list(da.shape)
    out_shape[axis_num] = da.shape[axis_num] + lo + hi - 1
    post_da = post_metric_fn(_ShapeProbe(out_dims, out_shape)) if post_metric_fn is not None else None
    bc = ax_padding if (lo or hi) else None
    fv = fills[ax_name] if fills[ax_name] is not None else 0.0

    if _is_host_float(da) and (not folded or grid._device_for(da).type == "cuda"):
        # host field: stream slabs H2D -> kernel -> D2H inside the library (xg_stencil2_host, or
        # xg_stencil2_host_fold with the folded row of each slab as its north halo)
        dims, shape = tuple(da.dims), list(da.shape)
        pre_h = None if pre_metric is None else grid._metric_host(pre_metric, dims, da.data.dtype)
        post_h = None if post_da is None else grid._metric_host(post_da, out_dims, da.data.dtype)
        core = [in_dim]
        if folded:
            from .padding import _axis_dim, _fold_plan

            core.append(_axis_dim(grid, dims, grid._folds[ax_name]["seam_axis"]))
        route = _host_stream_route("fold" if folded else "plain", dims, shape, core, lo, hi,
                                   operand_shapes=[m.shape for m in (pre_h, post_h) if m is not None])
        if route is not None:
            _, ndrop, nmerge = route
            cut = lambda a: _merge_leading(a, ndrop, nmerge)  # noqa: E731
            x = cut(da.data)
            ax = axis_num - ndrop - nmerge + 1
            kw = dict(pre=None if pre_h is None else cut(pre_h), post=None if post_h is None else cut(post_h),
                      device=grid._host_device(da))
            try:
                if folded:
                    _, seam, skip, mirror, period = _fold_plan(grid, ax_name, dims, shape, 1)
                    out = ops.stencil2_host_fold(x, ax, op, lo, hi, bc, fv, seam - ndrop - nmerge + 1, skip, mirror,
                                                 period, negate=isinstance(raw_arg, dict), **kw)
                else:
                    out = ops.stencil2_host(x, ax, op, lo, hi, bc, fv, **kw)
                return DataArray(out.reshape(out_shape), dims=out_dims, name=da.name, attrs=da.attrs)
            except NotImplementedError:
                pass  # e.g. periodic halo + pre-metric along the outermost axis: whole-field path below

    x, was_host = as_device_tensor(da.data, grid._device_for(da))
    pre_t = grid._metric_tensor(pre_metric, da.dims, x) if pre_metric is not None else None
    post_t = grid._metric_tensor(post_da, out_dims, x) if post_da is not None else None
    halo_lo = halo_hi = None
    if folded:
        # the north halo is the folded row of x * pre, sign-flipped for a vector component
        halo_lo, halo_hi = fold_halo_planes(grid, ax_name, da.dims, x, lo, ax_padding, pre=pre_t,
                                            negate=isinstance(raw_arg, dict))
    out = ops.stencil2(x, axis_num, op, lo, hi, bc, fv, pre=pre_t, post=post_t, halo_lo=halo_lo, halo_hi=halo_hi)
    return DataArray(result_like(out, was_host), dims=out_dims, name=da.name, attrs=da.attrs)


def _is_host_float(da) -> bool:
    return not da.is_device and isinstance(da.data, np.ndarray) and da.data.dtype in (np.float32, np.float64)


def _host_stream_route(kind, dims, shape, core_dims, lo, hi, pre=False, partner_ok=True, operand_shapes=()):
    """Whether a numpy field streams through a host slab pipeline, and how it is cut.

    ``kind``: "plain" (``xg_stencil2_host``), "fold" (the operator crosses a north fold), "connected" (face
    connections) or "pair" (``xg_stencil_pair_host`` and its fold variant); ``core_dims``: the dims the
    operator or any halo source indexes (operated dims; seam dim; face dim and the dims of the connection
    axes).  The slabs are cut along dim 0: leading size-1 dims are dropped first, then the leading batch dims
    (those before the first core dim) are merged into one dim 0 -- as far as every broadcast operand (metric
    ``operand_shapes``, 1 where it broadcasts) merges with them.  A plain grid cuts the field's own dim 0 (no
    merge), which may be the operated dim.  Returns ``(kind, dims dropped, dims merged)``, or None for the
    whole-field device path: a fold, connected or pair field with no batch dim in front, a halo wider than
    one cell, a pre-metric or a partner component that cannot stream beside the field on a connected grid."""
    first = min(list(dims).index(d) for d in core_dims)
    ndrop = 0
    while ndrop < first and shape[ndrop] == 1:
        ndrop += 1
    if kind == "plain":
        return kind, ndrop, 1
    if lo > 1 or hi > 1 or first == ndrop or (kind == "connected" and (pre or not partner_ok)):
        return None
    nmerge = first - ndrop

    def merges(m, k):
        sizes = [(int(a), int(b)) for a, b in zip(m[ndrop:ndrop + k], shape[ndrop:ndrop + k]) if b != 1]
        return all(a == b for a, b in sizes) or all(a == 1 for a, _ in sizes)

    while nmerge > 1 and not all(merges(m, nmerge) for m in operand_shapes):
        nmerge -= 1
    return kind, ndrop, nmerge


def _merge_leading(a, ndrop, nmerge):
    """``a`` (C-contiguous, or a metric with 1 where it broadcasts) without its first ``ndrop`` dims and with
    the next ``nmerge`` merged into one (``_host_stream_route`` checked that this is a reshape)."""
    a = np.ascontiguousarray(a)
    return a.reshape((int(np.prod(a.shape[ndrop:ndrop + nmerge])),) + a.shape[ndrop + nmerge:])


def _stream_connected_stencil(op, raw_arg, other_component, grid, ax_name, in_dim, out_dim, lo, hi, padding,
                              fill_value, post_metric_fn):
    """A built-in operator on a numpy field of a grid with face connections through the host slab pipeline
    (``xg_stencil2_host_connected``), or None when the field does not stream (``_host_stream_route``)."""
    from . import ops
    from .padding import (_axis_dim, _get_all_connection_axes, _unpack_vector, connected_edge_mode,
                          connected_halo_program)

    da, isvector, vectoraxis, partner = _unpack_vector(grid, raw_arg, other_component)
    if not _is_host_float(da) or grid._device_for(da).type != "cuda":
        return None
    dims, shape = tuple(da.dims), [int(v) for v in da.shape]
    facedim = grid._facedim
    core = [in_dim, facedim]
    for axname in _get_all_connection_axes(grid._face_connections, facedim):
        core += [d for d in grid.axes[axname].coords.values() if d in dims]
    mode, fv = connected_edge_mode(grid, ax_name, lo, hi, padding, fill_value, shape[dims.index(facedim)])
    axis_num = dims.index(in_dim)
    out_dims = tuple(out_dim if d == in_dim else d for d in dims)
    out_shape = list(shape)
    out_shape[axis_num] = shape[axis_num] + lo + hi - 1
    post_da = post_metric_fn(_ShapeProbe(out_dims, out_shape)) if post_metric_fn is not None else None
    post_h = None if post_da is None else grid._metric_host(post_da, out_dims, da.data.dtype)
    first = min(dims.index(d) for d in core)
    partner_ok = not isvector or (
        not partner.is_device and isinstance(partner.data, np.ndarray) and len(partner.dims) == len(dims)
        and tuple(partner.dims[:first]) == dims[:first] and tuple(partner.shape[:first]) == tuple(shape[:first]))
    route = _host_stream_route("connected", dims, shape, core, lo, hi, partner_ok=partner_ok,
                               operand_shapes=[post_h.shape] if post_h is not None else [])
    if route is None:
        return None
    _, ndrop, nmerge = route
    cut = lambda a: _merge_leading(a, ndrop, nmerge)  # noqa: E731
    lead = ndrop + nmerge
    m_dims = dims[ndrop:ndrop + 1] + dims[lead:]  # the merged batch dim keeps the name of its first dim
    x = cut(da.data)
    q = partner_layout = None
    if isvector:
        q = cut(partner.data)
        partner_layout = (tuple(partner.dims[ndrop:ndrop + 1] + partner.dims[lead:]), tuple(q.shape))
    program = connected_halo_program(grid, ax_name, lo, hi, m_dims, list(x.shape), mode, vectoraxis,
                                     partner_layout)
    out = ops.stencil2_host_connected(x, m_dims.index(in_dim), op, lo, hi, fv, program, partner=q,
                                      post=None if post_h is None else cut(post_h),
                                      device=grid._host_device(da))
    return DataArray(out.reshape(out_shape), dims=out_dims, name=da.name, attrs=da.attrs)


class _ShapeProbe:
    """Dims-only stand-in handed to ``Grid.get_metric`` (which only looks at dims)."""

    def __init__(self, dims, shape):
        self.dims = tuple(dims)
        self.shape = tuple(shape)
        self.name = None

    @property
    def sizes(self):
        return dict(zip(self.dims, self.shape))


def _apply_generic(func, args, input_arrays, grid, in_core_dims, out_core_dims,
                   padding_width_real, padding, fill_value, other_component, pad_before_func,
                   kwargs):
    """User-defined ufunc: device pad (xg_pad), then the user's function on host arrays with the
    core dims last — the contract of ``xr.apply_ufunc`` (grid_ufunc.py:954-990)."""
    from .labeled import to_numpy

    def run(arrs):
        moved = []
        for a, core in zip(arrs, in_core_dims):
            a = _maybe_unpack_vector_component(a)
            order = [d for d in a.dims if d not in core] + list(core)
            moved.append(a.transpose(*order))
        # broadcast non-core dims by name
        bdims: List[str] = []
        for a, core in zip(moved, in_core_dims):
            for d in a.dims:
                if d not in core and d not in bdims:
                    bdims.append(d)
        raw = []
        for a, core in zip(moved, in_core_dims):
            v = to_numpy(a.data)
            nb = [d for d in a.dims if d not in core]
            shape = [a.sizes[d] if d in nb else 1 for d in bdims] + [a.sizes[d] for d in core]
            src_order = [nb.index(d) for d in bdims if d in nb]
            v = np.transpose(v, src_order + list(range(len(nb), v.ndim)))
            raw.append(v.reshape(shape))
        res = func(*raw, **kwargs)
        if not isinstance(res, tuple):
            res = (res,)
        if len(res) != len(out_core_dims):
            raise ValueError(
                f"grid ufunc returned {len(res)} outputs but the signature declares {len(out_core_dims)}"
            )
        out = []
        for r, core in zip(res, out_core_dims):
            r = np.asarray(r)
            dims = tuple(bdims) + tuple(core)
            if r.ndim != len(dims):
                raise ValueError(
                    f"applied function returned data with unexpected number of dimensions. "
                    f"Received {r.ndim} dimension(s) but expected {len(dims)} dimensions with names: {dims!r}"
                )
            out.append(DataArray(r, dims=dims))
        return out

    def pad_all(arrs, core_dims_unused):
        return [
            pad(a, grid=grid, padding_width=padding_width_real, padding=padding,
                fill_value=fill_value, other_component=oc)
            for a, oc in zip(arrs, other_component)
        ]

    if pad_before_func:
        results = run(pad_all(args, in_core_dims))
    else:
        results = pad_all(run(args), out_core_dims)
    # sizes of the new core dims must match the grid (apply_ufunc output_sizes check)
    for res in results:
        for d in res.dims:
            if d in grid._ds.dims and grid._ds.sizes[d] != res.sizes[d]:
                raise ValueError(
                    f"conflicting sizes for dimension {d!r}: length {res.sizes[d]} on the data but "
                    f"length {grid._ds.sizes[d]} on the grid - does your grid ufunc correctly trim off "
                    f"the same number of elements which were added by padding using "
                    f"padding_width={padding_width_real}?"
                )
    return tuple(results)
