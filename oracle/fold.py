"""CPU oracle of north-fold padding (tripolar grids), restated in numpy from the rules of the reference.

TEST INFRASTRUCTURE ONLY.  Nothing under ``xgcm_b200/`` may import this.

The north halo of width W along the fold axis (reference xgcm/padding.py:619-684):
  * halo row r (r = 0..W-1, going north) is interior row n-1-skip-r, with skip = 1 when the field's
    fold-axis position kind (center, or edge for left/right/outer/inner) equals the pivot's fold role;
  * the row is mirrored along the seam axis: seam index k reads (C - k - 2*off) mod N with C = 0 for an
    edge pivot and 1 for a center pivot, 2*off = 1 center, 0 left, 2 right, 0 outer, 2 inner, and N the
    seam length (minus 1 for outer, plus 1 for inner);
  * vector components change sign.
Padding order (padding.py:723-762): the fold rows are concatenated first, from the unpadded field; then
the south edge of the fold axis and every other axis are padded with ``np.pad`` on that array.
``tests/test_fold_host.py`` pins the pivot table and partner maps against ``tests/golden/fold_ref.json``,
recorded from the reference's own helpers by ``oracle/make_fold_golden.py``.
"""

from __future__ import annotations

import numpy as np

from .stencil import pad_axis

PIVOT_ALIASES = {
    "center": ("center", "center"),  # (seam role, fold role)
    "t": ("center", "center"),
    "corner": ("edge", "edge"),
    "f": ("edge", "edge"),
    "u": ("edge", "center"),
    "v": ("center", "edge"),
}
TWO_OFFSET = {"center": 1, "left": 0, "right": 2, "outer": 0, "inner": 2}
CELLS_MINUS_LENGTH = {"center": 0, "left": 0, "right": 0, "outer": -1, "inner": 1}


def kind(position):
    return "center" if position == "center" else "edge"


def resolve_pivot(pivot, fold_axis, seam_axis):
    """``{"seam": role, "fold": role}`` of an alias (case-insensitive) or an ``{axis: position}`` mapping."""
    if isinstance(pivot, str):
        seam, fold = PIVOT_ALIASES[pivot.lower()]
        return {"seam": seam, "fold": fold}
    roles = {"seam": "center", "fold": "center"}
    for ax, pos in pivot.items():
        if ax == fold_axis:
            roles["fold"] = kind(pos)
        elif ax == seam_axis:
            roles["seam"] = kind(pos)
        else:
            raise ValueError(f"pivot axis {ax!r} is neither the fold nor the seam axis")
    return roles


def seam_partner_indices(position, seam_role, length):
    """Source seam index of every output seam index k: (C - k - 2*off) mod N."""
    c = 0 if seam_role == "edge" else 1
    n_cells = length + CELLS_MINUS_LENGTH[position]
    return np.array([(c - k - TWO_OFFSET[position]) % n_cells for k in range(length)], dtype=np.int64)


def north_rows(a, fold_axis, seam_axis, fold_position, seam_position, roles, width, vector=False):
    """The ``width`` folded rows of ``a`` (ordered going north), stacked along ``fold_axis``."""
    a = np.asarray(a)
    n = a.shape[fold_axis]
    skip = 1 if kind(fold_position) == roles["fold"] else 0
    if width > n - skip:
        raise ValueError(f"north halo width {width} exceeds the {n - skip} interior row(s)")
    idx = seam_partner_indices(seam_position, roles["seam"], a.shape[seam_axis])
    if idx.max() >= a.shape[seam_axis]:
        raise NotImplementedError("seam position incompatible with the pivot")
    rows = np.take(a, [n - 1 - skip - r for r in range(width)], axis=fold_axis)
    rows = np.take(rows, idx, axis=seam_axis)
    return -rows if vector else rows


def pad_fold(a, fold_axis, seam_axis, fold_position, seam_position, roles, widths, modes, fills=None,
             vector=False):
    """``pad()`` on a fold grid: ``widths`` / ``modes`` / ``fills`` map dim numbers to (lo, hi), a boundary
    mode and a fill value; the fold dim's mode is its south mode (its north edge always folds)."""
    fills = fills or {}
    a = np.asarray(a)
    lo, hi = widths.get(fold_axis, (0, 0))
    if hi:
        halo = north_rows(a, fold_axis, seam_axis, fold_position, seam_position, roles, hi, vector)
        a = np.concatenate([a, halo], axis=fold_axis)
    for d, (w_lo, w_hi) in widths.items():
        if d == fold_axis:
            w_hi = 0
        a = pad_axis(a, d, w_lo, w_hi, modes.get(d), fills.get(d, 0.0))
    return a
