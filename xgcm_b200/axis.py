"""``Axis``: one direction of the model grid with its staggered positions.

Host-side metadata only (no array math).  Behaviour mirrors the reference's
``xgcm/axis.py`` — position names, default shifts (axis.py:11-17,126-146),
padding validation (:152-165) and the 0.0 fill default (:167-171) — because the
resolved (position, dim, shift, boundary, fill) tuple is what parameterises the
CUDA kernels.
"""

from __future__ import annotations

from typing import Mapping, Optional, Tuple, Union

from .labeled import Dataset
from .padding import _parse_fold_padding

VALID_POSITION_NAMES = "center|left|right|inner|outer"
_VALID_POSITIONS = tuple(VALID_POSITION_NAMES.split("|"))

# shift tried, in order, when the user gives no `to` (reference axis.py:11-17)
FALLBACK_SHIFTS = {
    "center": ("left", "right", "outer", "inner"),
    "left": ("center",),
    "right": ("center",),
    "outer": ("center",),
    "inner": ("center",),
}

# reference padding.py:15-19; "extrapolate" is this package's opt-in extension
VALID_PADDINGS = ("periodic", "fill", "extend")
EXTENSION_PADDINGS = ("extrapolate",)

# number of points of each position relative to `center` (docs/grids.md:77-79)
POSITION_LENGTH_OFFSET = {"center": 0, "left": 0, "right": 0, "outer": 1, "inner": -1}


def _is_dataset(obj) -> bool:
    if isinstance(obj, Dataset):
        return True
    return type(obj).__name__ == "Dataset" and hasattr(obj, "dims") and hasattr(obj, "coords")


class Axis:
    """A single direction along a model grid, holding one dim name per cell position."""

    def __init__(
        self,
        ds,
        name: str,
        coords: Mapping[str, str],
        default_shifts: Optional[Mapping[str, str]] = None,
        padding: Optional[Union[str, Mapping]] = None,
        fill_value: Optional[float] = None,
        **kwargs,
    ):
        if "boundary" in kwargs:
            raise ValueError(
                "Argument 'boundary' has been renamed to 'padding'. Please use 'padding' instead."
            )
        if not isinstance(name, str):
            raise TypeError(f"name argument must be of type str, but is of type {type(name)}")
        if not _is_dataset(ds):
            raise TypeError(f"ds argument must be of type xarray.Dataset, but is of type {type(ds)}")
        self._name = name

        for pos, dim in coords.items():
            if pos not in _VALID_POSITIONS:
                raise ValueError(
                    f"Axis position must be one of {list(_VALID_POSITIONS)}, but got {pos}"
                )
            if dim not in ds.dims:
                raise ValueError(
                    f"Could not find dimension `{dim}` (for the `{pos}` position on axis `{name}`) in input dataset."
                )
        dims = list(coords.values())
        duplicates = sorted({d for d in dims if dims.count(d) > 1})
        if duplicates:
            raise ValueError(
                f"The same dimension cannot be assigned to multiple positions on axis `{name}`. "
                f"Duplicate dimension(s): {duplicates}"
            )
        self._coords = dict(coords)

        user_shifts = dict(default_shifts or {})
        self._default_shifts = {}
        for pos in self._coords:
            if pos in user_shifts:
                self._default_shifts[pos] = user_shifts[pos]
            else:
                for candidate in FALLBACK_SHIFTS[pos]:
                    if candidate in self._coords:
                        self._default_shifts[pos] = candidate
                        break
            if self._default_shifts.get(pos) == pos:
                raise ValueError(f"Can't set the default shift for {pos} to be to {pos}")

        if isinstance(padding, Mapping):
            # a north-fold spec, e.g. {"fold": "corner"}; its seam axis is inferred by Grid._validate_folds
            padding = _parse_fold_padding(padding)
        elif padding is not None and padding not in VALID_PADDINGS + EXTENSION_PADDINGS:
            raise ValueError(
                f"padding must be one of {list(VALID_PADDINGS)} "
                f"or a fold spec (e.g. {{'fold': 'corner'}}) or None, but got {padding}"
            )
        self._padding = padding

        if fill_value is None:
            fill_value = 0.0
        if not isinstance(fill_value, (int, float)):
            raise TypeError("fill value must be an integer or a float")
        self._fill_value = fill_value
        self._periodic = padding == "periodic"
        # set by Grid._assign_face_connections (grid.py:407-409)
        self._facedim = None
        self._face_connections = None

    @property
    def periodic(self) -> bool:
        return self._periodic

    @property
    def fill_value(self) -> float:
        return self._fill_value

    @property
    def name(self) -> str:
        return self._name

    @property
    def coords(self) -> Mapping[str, str]:
        return self._coords

    @property
    def default_shifts(self) -> Mapping[str, str]:
        return self._default_shifts

    @property
    def padding(self) -> Optional[Union[str, Mapping]]:
        return self._padding

    @property
    def boundary(self):
        raise AttributeError(
            "Attribute 'boundary' has been renamed to 'padding'. Please use 'padding' instead."
        )

    def __repr__(self):
        kind = "periodic" if self._periodic else "not periodic"
        lines = [f"<xgcm.Axis '{self.name}' ({kind}, padding={self.padding!r})>", "Axis Coordinates:"]
        return "\n".join(lines + self._coord_desc())

    def _coord_desc(self):
        out = []
        for pos, dim in self.coords.items():
            line = "  * %-8s %s" % (pos, dim)
            if pos in self._default_shifts:
                line += " --> %s" % self._default_shifts[pos]
            out.append(line)
        return out

    def _get_position_name(self, da) -> Tuple[str, str]:
        """(position, dim) of this axis on ``da`` (reference axis.py:232-251)."""
        candidates = set(da.dims).intersection(self.coords.values())
        if len(candidates) == 0:
            raise KeyError(f"None of the DataArray's dims {da.dims} were found in axis coords.")
        if len(candidates) > 1:
            raise KeyError(f"DataArray cannot have more than 1 axis dimension, but found {candidates}")
        for pos, dim in self.coords.items():
            if dim in da.dims:
                return pos, dim
        raise KeyError(f"None of the DataArray's dims {da.dims} were found in axis coords.")

    def _get_axis_dim_num(self, da):
        _, dim = self._get_position_name(da)
        return da.get_axis_num(dim)
