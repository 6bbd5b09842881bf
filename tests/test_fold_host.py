"""North-fold (tripolar) boundary on the CPU: spec parsing and Grid validation (the cases of the reference's
xgcm/test/test_fold.py:76-279), the oracle against the reference's own helpers (tests/golden/fold_ref.json) and
its known answers, and the routing of every operator across the fold with the kernels replaced by the oracle
(tests/_mock_fold.py): a per-call padding string must never turn the folded north edge into a plain one."""

import json
import os
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from _mock_fold import install
from oracle import fold as F
from oracle import stencil as S

Nx, Ny = 8, 5
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fold_ref.json")


@pytest.fixture
def mock(monkeypatch):
    install(monkeypatch)


def _ds():
    """One field per staggering: c (yh, xh), u (yh, xl), v (yl, xh), q (yl, xl), all arange(40)."""
    base = np.arange(Ny * Nx, dtype=float).reshape(Ny, Nx)
    return xg.Dataset(
        data_vars={"c": (("yh", "xh"), base.copy()), "u": (("yh", "xl"), base.copy()),
                   "v": (("yl", "xh"), base.copy()), "q": (("yl", "xl"), base.copy())},
        coords={"xh": np.arange(Nx), "xl": np.arange(Nx), "yh": np.arange(Ny), "yl": np.arange(Ny)},
    )


def _grid(ds, pivot, **spec):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        return xg.Grid(ds, coords={"X": {"center": "xh", "left": "xl"}, "Y": {"center": "yh", "left": "yl"}},
                       padding={"X": "periodic", "Y": {"fold": pivot, **spec}}, autoparse_metadata=False)


# ---------------------------------------------------------------------------------------------- parsing
@pytest.mark.parametrize("alias, seam, fold", [("center", "center", "center"), ("T", "center", "center"),
                                               ("corner", "edge", "edge"), ("F", "edge", "edge"),
                                               ("U", "edge", "center"), ("V", "center", "edge")])
def test_pivot_aliases(alias, seam, fold):
    grid = _grid(_ds(), alias)
    assert grid._folds["Y"] == {"seam_axis": "X", "pivot": alias, "south": "fill"}
    from xgcm_b200.padding import _resolve_pivot

    assert _resolve_pivot(alias, "Y", "X") == {"seam": seam, "fold": fold}
    assert F.resolve_pivot(alias, "Y", "X") == {"seam": seam, "fold": fold}


def test_explicit_pivot_and_left_right_equivalence():
    from xgcm_b200.padding import _resolve_pivot

    assert _resolve_pivot({"X": "right", "Y": "center"}, "Y", "X") == {"seam": "edge", "fold": "center"}
    left = _resolve_pivot({"X": "left", "Y": "left"}, "Y", "X")
    right = _resolve_pivot({"X": "right", "Y": "right"}, "Y", "X")
    assert left == right == {"seam": "edge", "fold": "edge"}


def test_fold_requires_periodic_seam():
    with pytest.raises(ValueError, match="periodic seam axis"):
        xg.Grid(_ds(), coords={"X": {"center": "xh"}, "Y": {"center": "yh"}},
                padding={"X": "fill", "Y": {"fold": "corner"}}, autoparse_metadata=False)


def test_seam_inferred_and_unspecified_axis_ignored():
    ds = _ds()
    ds = xg.Dataset(data_vars={k: ds[k] for k in ("c",)}, coords={"xh": np.arange(Nx), "xl": np.arange(Nx),
                                                                    "yh": np.arange(Ny), "yl": np.arange(Ny),
                                                                    "zh": np.arange(3)})
    with pytest.warns(UserWarning, match="experimental"):
        grid = xg.Grid(ds, coords={"X": {"center": "xh", "left": "xl"}, "Y": {"center": "yh", "left": "yl"},
                                   "Z": {"center": "zh"}},
                       padding={"X": "periodic", "Y": {"fold": "corner"}}, autoparse_metadata=False)
    assert grid._folds["Y"]["seam_axis"] == "X"
    assert "Z" not in grid._explicitly_periodic_axes
    with pytest.raises(ValueError, match="ambiguous"):
        xg.Grid(ds, coords={"X": {"center": "xh", "left": "xl"}, "Y": {"center": "yh", "left": "yl"},
                            "Z": {"center": "zh"}},
                padding={"X": "periodic", "Z": "periodic", "Y": {"fold": "corner"}}, autoparse_metadata=False)


def test_fold_warns_exactly_once_and_plain_grids_do_not():
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        xg.Grid(_ds(), coords={"X": {"center": "xh"}, "Y": {"center": "yh"}},
                padding={"X": "periodic", "Y": {"fold": "corner"}}, autoparse_metadata=False)
        plain = xg.Grid(_ds(), coords={"X": {"center": "xh"}, "Y": {"center": "yh"}},
                        padding="periodic", autoparse_metadata=False)
    folds = [w for w in rec if issubclass(w.category, UserWarning) and "experimental" in str(w.message)]
    assert len(folds) == 1
    assert plain._folds == {}


@pytest.mark.parametrize("spec, match", [({"fold": "banana"}, "Unknown fold pivot"),
                                         ({"fold": {"X": "centre", "Y": "center"}}, "Invalid position"),
                                         ({"fold": {"X": "banana"}}, "Invalid position"),
                                         ({"fold": "corner", "north": "fill"}, "Unknown keys"),
                                         ({"fold": "corner", "south": "wrap"}, "south")])
def test_bad_specs_raise(spec, match):
    with pytest.raises(ValueError, match=match):
        xg.Grid(_ds(), coords={"X": {"center": "xh"}, "Y": {"center": "yh"}},
                padding={"X": "periodic", "Y": spec}, autoparse_metadata=False)


def test_fold_rejects_face_connections():
    ds = xg.Dataset(coords={"face": np.array([0, 1]), "xh": np.arange(Nx), "xl": np.arange(Nx),
                            "yh": np.arange(Ny), "yl": np.arange(Ny)})
    fc = {"face": {0: {"X": (None, (1, "X", False))}, 1: {"X": ((0, "X", False), None)}}}
    with pytest.raises(NotImplementedError, match="face_connections"):
        xg.Grid(ds, coords={"X": {"center": "xh", "left": "xl"}, "Y": {"center": "yh", "left": "yl"}},
                padding={"X": "periodic", "Y": {"fold": "corner"}}, face_connections=fc, autoparse_metadata=False)


@pytest.mark.parametrize("pivot", ["center", "V"])
def test_inner_seam_position_center_pivot_raises(mock, pivot):
    ds = xg.Dataset(data_vars={"f": (("yl", "xi"), np.zeros((Ny, Nx - 1)))},
                    coords={"xh": np.arange(Nx), "xi": np.arange(Nx - 1), "yh": np.arange(Ny), "yl": np.arange(Ny)})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords={"X": {"center": "xh", "inner": "xi"}, "Y": {"center": "yh", "left": "yl"}},
                       padding={"X": "periodic", "Y": {"fold": pivot}}, autoparse_metadata=False)
    with pytest.raises(NotImplementedError, match="incompatible"):
        xg.pad(ds["f"], grid, padding_width={"Y": (0, 1)})


# ---------------------------------------------------------------------------------------------- oracle vs golden
def test_oracle_matches_reference_helpers():
    ref = json.load(open(GOLDEN))
    for key, want in ref["partners"].items():
        position, role, length = key.split("|")
        np.testing.assert_array_equal(F.seam_partner_indices(position, role, int(length)), want, err_msg=key)
    for key, want in ref["pivots"].items():
        pivot = json.loads(key) if key.startswith("{") else key
        assert F.resolve_pivot(pivot, "Y", "X") == want, key
    from xgcm_b200.padding import _parse_fold_padding

    for label, case in ref["specs"].items():
        if "raises" in case:
            with pytest.raises(ValueError):
                _parse_fold_padding(case["spec"])
        else:
            assert _parse_fold_padding(case["spec"]) == case["result"], label


# ---------------------------------------------------------------------------------------------- known answers
B = np.arange(Ny * Nx, dtype=float).reshape(Ny, Nx)
ROW4_REV = [39.0, 38, 37, 36, 35, 34, 33, 32]
ROW3_REV = [31.0, 30, 29, 28, 27, 26, 25, 24]
CORNER = F.resolve_pivot("corner", "Y", "X")


def _north(fold_pos, seam_pos, pivot, width=1, vector=False, a=B):
    return F.north_rows(a, 0, 1, fold_pos, seam_pos, F.resolve_pivot(pivot, "Y", "X"), width, vector)


def test_oracle_known_answers():
    # test_corner_pivot_all_positions
    np.testing.assert_array_equal(_north("center", "center", "corner")[0], ROW4_REV)
    np.testing.assert_array_equal(_north("center", "left", "corner", vector=True)[0],
                                  [-32.0, -39, -38, -37, -36, -35, -34, -33])
    np.testing.assert_array_equal(_north("left", "center", "corner", vector=True)[0], [-v for v in ROW3_REV])
    np.testing.assert_array_equal(_north("left", "left", "corner")[0], [24.0, 31, 30, 29, 28, 27, 26, 25])
    # test_u_pivot_redundant_row
    np.testing.assert_array_equal(_north("center", "center", "U")[0], ROW3_REV)
    np.testing.assert_array_equal(_north("left", "center", "U")[0], ROW4_REV)
    # test_vector_flips_scalar_does_not
    np.testing.assert_array_equal(_north("left", "center", "corner", vector=True),
                                  -_north("left", "center", "corner"))
    # test_multi_row_halo
    np.testing.assert_array_equal(_north("center", "center", "corner", width=2), [ROW4_REV, ROW3_REV])
    # test_north_halo_wider_than_interior_raises
    assert F.pad_fold(B, 0, 1, "center", "center", CORNER, {0: (0, Ny)}, {0: "fill"}).shape == (2 * Ny, Nx)
    with pytest.raises(ValueError, match="exceeds the .* interior row"):
        F.pad_fold(B, 0, 1, "center", "center", CORNER, {0: (0, Ny + 1)}, {0: "fill"})
    # test_fold_with_simultaneous_seam_padding
    out = F.pad_fold(B, 0, 1, "center", "center", CORNER, {1: (1, 1), 0: (0, 1)}, {1: "periodic", 0: "fill"})
    np.testing.assert_array_equal(out[-1], [32.0] + ROW4_REV + [39.0])
    # test_fold_south_edge_respects_per_call_padding
    out = F.pad_fold(B, 0, 1, "center", "center", CORNER, {0: (1, 1)}, {0: "extend"})
    np.testing.assert_array_equal(out[0], B[0])
    np.testing.assert_array_equal(out[-1], ROW4_REV)
    np.testing.assert_array_equal(F.pad_fold(B, 0, 1, "center", "center", CORNER, {0: (1, 0)}, {0: "fill"})[0], 0.0)
    # a periodic south wraps the fold row when the north is padded too, else interior row n-1
    np.testing.assert_array_equal(F.pad_fold(B, 0, 1, "center", "center", CORNER, {0: (1, 1)}, {0: "periodic"})[0],
                                  ROW4_REV)
    np.testing.assert_array_equal(F.pad_fold(B, 0, 1, "center", "center", CORNER, {0: (1, 0)}, {0: "periodic"})[0],
                                  B[-1])


def test_oracle_center_and_edge_mirror_same_pole():
    def fn(x):
        return np.sin(2 * np.pi * x / Nx) + 0.3 * np.cos(6 * np.pi * x / Nx)

    xc, xe = np.arange(Nx) + 0.5, np.arange(Nx).astype(float)
    np.testing.assert_allclose(_north("center", "center", "corner", a=np.tile(fn(xc), (Ny, 1)))[0], fn((-xc) % Nx),
                               atol=1e-12)
    np.testing.assert_allclose(_north("center", "left", "corner", a=np.tile(fn(xe), (Ny, 1)))[0], fn((-xe) % Nx),
                               atol=1e-12)


def test_oracle_outer_symmetric_memory():
    def fn(x, y):
        return np.sin(2 * np.pi * x / Nx) + 0.5 * y

    xq, yq, xc = np.arange(Nx + 1), np.arange(Ny + 1), np.arange(Nx) + 0.5
    v = fn(xc[None, :], yq[:, None])
    q = fn(xq[None, :], yq[:, None])
    np.testing.assert_allclose(_north("outer", "center", "corner", a=v)[0], fn((-xc) % Nx, Ny - 1), atol=1e-12)
    np.testing.assert_allclose(_north("outer", "outer", "corner", a=q)[0],
                               [fn((-j) % Nx, Ny - 1) for j in range(Nx + 1)], atol=1e-12)


def test_oracle_interp_diff_across_seam_known_answer():
    """The operator answers of the reference's test: a left -> center Y shift straddles the fold row."""
    def straddle(halo):
        fp = np.vstack([B, np.asarray(halo, dtype=float)[None, :]])
        return 0.5 * (fp[:-1] + fp[1:]), fp[1:] - fp[:-1]

    cases = [("corner", "center", False, ROW3_REV), ("corner", "center", True, [-v for v in ROW3_REV]),
             ("corner", "left", False, [24.0, 31, 30, 29, 28, 27, 26, 25]), ("U", "center", False, ROW4_REV)]
    for pivot, seam_pos, vector, halo in cases:
        padded = F.pad_fold(B, 0, 1, "left", seam_pos, F.resolve_pivot(pivot, "Y", "X"), {0: (0, 1)}, {0: "fill"},
                            vector=vector)
        exp_i, exp_d = straddle(halo)
        np.testing.assert_array_equal(S.stencil2("interp", padded, 0, 0, 0, None), exp_i)
        np.testing.assert_array_equal(S.stencil2("diff", padded, 0, 0, 0, None), exp_d)


# ---------------------------------------------------------------------------------------------- the package, mocked
def _expect(op, a, fold_pos, seam_pos, pivot, lo, hi, south, vector=False, fold_axis=0, seam_axis=1):
    padded = F.pad_fold(a, fold_axis, seam_axis, fold_pos, seam_pos, F.resolve_pivot(pivot, "Y", "X"),
                        {fold_axis: (lo, hi)}, {fold_axis: south}, vector=vector)
    return S.stencil2(op, padded, fold_axis, 0, 0, None)


def test_pad_known_answers(mock):
    ds = _ds()
    grid = _grid(ds, "corner")
    np.testing.assert_array_equal(xg.pad(ds["c"], grid, padding_width={"Y": (0, 1)}).values[-1], ROW4_REV)
    out = xg.pad({"X": ds["u"]}, grid, padding_width={"Y": (0, 1)}, other_component={"Y": ds["v"]})
    np.testing.assert_array_equal(out.values[-1], [-32.0, -39, -38, -37, -36, -35, -34, -33])
    out = xg.pad({"Y": ds["v"]}, grid, padding_width={"Y": (0, 1)})
    np.testing.assert_array_equal(out.values[-1], [-v for v in ROW3_REV])
    out = xg.pad(ds["c"], grid, padding_width={"X": (1, 1), "Y": (0, 1)})
    assert out.shape == (Ny + 1, Nx + 2)
    np.testing.assert_array_equal(out.values[-1], [32.0] + ROW4_REV + [39.0])
    out = xg.pad(ds["c"], grid, padding_width={"Y": (1, 1)}, padding={"Y": "extend"})
    np.testing.assert_array_equal(out.values[0], B[0])
    np.testing.assert_array_equal(out.values[-1], ROW4_REV)
    np.testing.assert_array_equal(xg.pad(ds["c"], grid, padding_width={"Y": (1, 0)}).values[0], 0.0)
    with pytest.raises(ValueError, match="exceeds the .* interior row"):
        xg.pad(ds["c"], grid, padding_width={"Y": (0, Ny + 1)})
    assert xg.pad(ds["c"], grid, padding_width={"Y": (0, Ny)}).sizes["yh"] == 2 * Ny


@pytest.mark.parametrize("per_call", [None, "extend", "fill", "periodic"])
def test_operators_fold_whatever_the_per_call_padding(mock, per_call):
    ds = _ds()
    grid = _grid(ds, "corner", south="periodic")
    kw = {} if per_call is None else {"padding": per_call}
    south = per_call or "periodic"
    q = ds["q"]
    for op in ("diff", "interp", "min", "max"):
        want = _expect(op, B, "left", "left", "corner", 0, 1, south)
        np.testing.assert_array_equal(getattr(grid, op)(q, "Y", **kw).values, want)                  # numpy input
        dev = xg.DataArray(torch.from_numpy(B.copy()), dims=("yl", "xl"))
        np.testing.assert_array_equal(np.asarray(getattr(grid, op)(dev, "Y", **kw).data), want)      # device input
    c = ds["c"]
    # center -> left pads only the south edge
    want = _expect("diff", B, "center", "center", "corner", 1, 0, south)
    np.testing.assert_array_equal(grid.diff(c, "Y", to="left", **kw).values, want)
    # the vector component changes sign across the fold
    want = _expect("interp", B, "left", "center", "corner", 0, 1, south, vector=True)
    np.testing.assert_array_equal(grid.interp({"Y": ds["v"]}, "Y", **kw).values, want)
    # apply_many (numpy field: the batched host pipeline would take no fold halo)
    got = grid.apply_many(q, [("diff", "Y"), ("interp", "X")], **kw)
    np.testing.assert_array_equal(got[0].values, _expect("diff", B, "left", "left", "corner", 0, 1, south))
    np.testing.assert_array_equal(got[1].values, S.stencil2("interp", B, 1, 0, 1, per_call or "periodic"))
    # multi-axis interp: per-axis launches, the Y one across the fold
    got = grid.interp(q, ["X", "Y"], **kw)
    step = S.stencil2("interp", B, 1, 0, 1, per_call or "periodic")
    np.testing.assert_array_equal(got.values, _expect("interp", step, "left", "center", "corner", 0, 1, south))


def test_pair_divergence_and_cumsum_across_the_fold(mock):
    rng = np.random.default_rng(3)
    u, v = rng.random((Ny, Nx)), rng.random((Ny, Nx))
    ds = xg.Dataset(data_vars={"u": (("yh", "xl"), u), "v": (("yl", "xh"), v), "c": (("yh", "xh"), u.copy()),
                               "dx": (("yh", "xh"), 1 + rng.random((Ny, Nx))),
                               "dy": (("yh", "xh"), 1 + rng.random((Ny, Nx)))},
                    coords={"xh": np.arange(Nx), "xl": np.arange(Nx), "yh": np.arange(Ny), "yl": np.arange(Ny),
                            "yr": np.arange(Ny)})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords={"X": {"center": "xh", "left": "xl"},
                                   "Y": {"center": "yh", "left": "yl", "right": "yr"}},
                       padding={"X": "periodic", "Y": {"fold": "corner"}}, autoparse_metadata=False)
    for kw in ({}, {"padding": "extend"}):
        south = kw.get("padding", "fill")
        want = (S.stencil2("diff", u, 1, 0, 1, kw.get("padding", "periodic"))
                + _expect("diff", v, "left", "center", "corner", 0, 1, south))
        np.testing.assert_array_equal(grid.pair("diff", ds["u"], "X", "diff", ds["v"], "Y", **kw).values, want)
        # a term given as a vector component folds with a sign change
        wdiv = (S.stencil2("diff", u, 1, 0, 1, kw.get("padding", "periodic"))
                + _expect("diff", v, "left", "center", "corner", 0, 1, south, vector=True))
        got = grid.pair("diff", ds["u"], "X", "diff", ds["v"], "Y", _components=("X", "Y"), **kw)
        np.testing.assert_array_equal(got.values, wdiv)
        # cumsum c -> right reversed pads the north edge: scan, fold the scanned rows, no divide
        scanned = np.flip(np.cumsum(np.flip(u, 0), 0), 0)[1:]
        want = F.pad_fold(scanned, 0, 1, "center", "center", CORNER, {0: (0, 1)}, {0: south})
        got = grid.cumsum(ds["c"], "Y", to="right", reverse=True, **kw)
        np.testing.assert_array_equal(got.values, want)
        # forward c -> left pads only the south edge: the spec's south mode unless overridden
        fwd = np.cumsum(u, 0)[:-1]
        np.testing.assert_array_equal(grid.cumsum(ds["c"], "Y", to="left", **kw).values,
                                      S.pad_axis(fwd, 0, 1, 0, south))


def test_divergence_folds_v_as_a_vector(mock):
    rng = np.random.default_rng(5)
    u, v = rng.random((Ny, Nx)), rng.random((Ny, Nx))
    dyu, dxv, area = 1 + rng.random((Ny, Nx)), 1 + rng.random((Ny, Nx)), 1 + rng.random((Ny, Nx))
    ds = xg.Dataset(data_vars={"u": (("yh", "xl"), u), "v": (("yl", "xh"), v), "dyu": (("yh", "xl"), dyu),
                               "dxv": (("yl", "xh"), dxv), "area": (("yh", "xh"), area)},
                    coords={"xh": np.arange(Nx), "xl": np.arange(Nx), "yh": np.arange(Ny), "yl": np.arange(Ny)})
    grid = _grid(ds, "corner")
    grid.set_metrics("Y", "dyu")
    grid.set_metrics("X", "dxv")
    grid.set_metrics(("X", "Y"), "area")
    for kw in ({}, {"padding": "extend"}):
        tx = S.stencil2("diff", u * dyu, 1, 0, 1, kw.get("padding", "periodic"))
        ty = _expect("diff", v * dxv, "left", "center", "corner", 0, 1, kw.get("padding", "fill"), vector=True)
        np.testing.assert_array_equal(grid.divergence(ds["u"], ds["v"], **kw).values, (tx + ty) / area)
