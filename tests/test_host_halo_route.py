"""Host-side planning of the streamed halo pipelines, without a GPU: which numpy fields stream through the
slab pipelines and how they are cut (``grid_ufunc._host_stream_route``), and the face-connection copy list
``padding.connected_halo_program`` replayed in numpy against oracle/faces.py."""

import itertools

import numpy as np
import pytest

import xgcm_b200 as xg
from oracle.faces import pad_face_connections
from xgcm_b200.grid_ufunc import _host_stream_route, _merge_leading
from xgcm_b200.padding import connected_halo_program

CORE_FACES = ["face", "y", "x", "yl", "xl"]


def test_route_cuts_leading_batch_dims():
    r = _host_stream_route
    # xmitgcm layouts on a face-connected grid: (time, k, face, j, i), (k, face, j, i), (1, k, face, j, i)
    assert r("connected", ("t", "k", "face", "y", "x"), [3, 5, 6, 8, 8], CORE_FACES[:3], 0, 1) == ("connected", 0, 2)
    assert r("connected", ("k", "face", "y", "x"), [5, 6, 8, 8], CORE_FACES[:3], 1, 1) == ("connected", 0, 1)
    assert r("connected", ("o", "k", "face", "y", "x"), [1, 5, 6, 8, 8], CORE_FACES[:3], 1, 0) == ("connected", 1, 1)
    # NEMO (time_counter, deptht, y, x) across a fold
    assert r("fold", ("t", "z", "y", "x"), [12, 75, 30, 40], ["y", "x"], 0, 1) == ("fold", 0, 2)
    # a plain grid cuts its own dim 0, after dropping leading size-1 dims (it may become the operated dim)
    assert r("plain", ("o", "z", "y", "x"), [1, 75, 24, 36], ["y"], 0, 1) == ("plain", 1, 1)
    assert r("plain", ("o", "z", "y", "x"), [1, 75, 24, 36], ["z"], 0, 1) == ("plain", 1, 1)
    assert r("plain", ("z", "y", "x"), [75, 24, 36], ["z"], 0, 1) == ("plain", 0, 1)


def test_route_merges_only_what_the_metrics_allow():
    r = _host_stream_route
    dims, shape = ("t", "z", "y", "x"), [4, 5, 30, 40]
    assert r("fold", dims, shape, ["y", "x"], 0, 1, operand_shapes=[(1, 1, 30, 40)]) == ("fold", 0, 2)
    assert r("fold", dims, shape, ["y", "x"], 0, 1, operand_shapes=[(4, 5, 30, 40)]) == ("fold", 0, 2)
    # a per-level metric broadcast over time is not a reshape of (t * z): cut along t alone
    assert r("fold", dims, shape, ["y", "x"], 0, 1, operand_shapes=[(1, 5, 30, 40)]) == ("fold", 0, 1)
    assert _merge_leading(np.zeros((1, 1, 3, 4)), 0, 2).shape == (1, 3, 4)
    assert _merge_leading(np.zeros((1, 4, 5, 3)), 1, 2).shape == (20, 3)


def test_route_falls_back():
    r = _host_stream_route
    # no batch dim in front: (face, k, j, i), 2-D (face, j, i), a fold field (y, x)
    assert r("connected", ("face", "k", "y", "x"), [6, 5, 8, 8], CORE_FACES[:3], 0, 1) is None
    assert r("connected", ("face", "y", "x"), [6, 8, 8], CORE_FACES[:3], 0, 1) is None
    assert r("connected", ("o", "face", "y", "x"), [1, 6, 8, 8], CORE_FACES[:3], 0, 1) is None
    assert r("fold", ("y", "x"), [30, 40], ["y", "x"], 0, 1) is None
    # a pre-metric on a face-connected grid, a partner that cannot stream, a halo wider than one cell
    dims, shape = ("t", "face", "y", "x"), [3, 6, 8, 8]
    assert r("connected", dims, shape, CORE_FACES[:3], 0, 1, pre=True) is None
    assert r("connected", dims, shape, CORE_FACES[:3], 0, 1, partner_ok=False) is None
    assert r("fold", ("t", "y", "x"), [3, 30, 40], ["y", "x"], 0, 2) is None


COORDS = {"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"}}
AXES = {"X": ("x", "xl"), "Y": ("y", "yl")}
# xgcm/test/test_faceconnections.py:99-127: same-axis, swapped and reversed seams
CUBED_SPHERE = {
    "face": {
        0: {"X": ((3, "X", False), (1, "X", False)), "Y": ((4, "Y", False), (5, "Y", False))},
        1: {"X": ((0, "X", False), (2, "X", False)), "Y": ((4, "X", False), (5, "X", True))},
        2: {"X": ((1, "X", False), (3, "X", False)), "Y": ((4, "Y", True), (5, "Y", True))},
        3: {"X": ((2, "X", False), (0, "X", False)), "Y": ((4, "X", True), (5, "X", False))},
        4: {"X": ((3, "Y", True), (1, "Y", False)), "Y": ((2, "Y", True), (0, "Y", False))},
        5: {"X": ((3, "Y", False), (1, "Y", True)), "Y": ((0, "Y", False), (2, "Y", True))},
    }
}


def _replay(program, x, partner, fill, p_shape):
    planes = [np.full(p_shape, np.inf), np.full(p_shape, np.inf)]
    written = [np.zeros(p_shape, int), np.zeros(p_shape, int)]
    srcs = {"self": x.ravel(), "partner": None if partner is None else partner.ravel(), "fill": np.array([fill])}
    for side, doff, dstr, src, soff, sstr, shp, neg in program:
        for idx in itertools.product(*[range(n) for n in shp]):
            d = doff + sum(i * s for i, s in zip(idx, dstr))
            v = srcs[src][soff + sum(i * s for i, s in zip(idx, sstr))]
            planes[side].ravel()[d] = -v if neg else v
            written[side].ravel()[d] += 1
    return planes, written


@pytest.mark.parametrize("mode", ["fill", "extend", "periodic"])
def test_connected_halo_program_matches_oracle(mode):
    """Every copy spans dim 0 in full (what the slab pipeline clips per slab); each face's plane is written
    exactly once; the planes equal the first / last plane of the oracle's padded field."""
    n = 6
    rng = np.random.default_rng(0)
    lead = (2, 3)
    coords = {"x": np.arange(n) + 0.0, "xl": np.arange(n) - 0.5, "y": np.arange(n) + 0.0,
              "yl": np.arange(n) - 0.5, "face": np.arange(6)}
    ds = xg.Dataset(data_vars={
        "c": (("t", "k", "face", "y", "x"), rng.random(lead + (6, n, n))),
        "u": (("t", "k", "face", "y", "xl"), rng.random(lead + (6, n, n))),
        "v": (("t", "k", "face", "yl", "x"), rng.random(lead + (6, n, n)))}, coords=coords)
    grid = xg.Grid(ds, coords=COORDS, face_connections=CUBED_SPHERE)
    for ax, (lo, hi), vec in itertools.product(["X", "Y"], [(1, 0), (0, 1), (1, 1)], [None, "X", "Y"]):
        da, partner = {None: (ds["c"], None), "X": (ds["u"], ds["v"]), "Y": (ds["v"], ds["u"])}[vec]
        dims, shape = da.dims, list(da.shape)
        layout = None if partner is None else (tuple(partner.dims), tuple(partner.shape))
        program = connected_halo_program(grid, ax, lo, hi, dims, shape, mode, vec, layout)
        assert all(c[6][0] == shape[0] for c in program)
        t = dims.index([d for d in dims if d in AXES[ax]][0])
        p_shape = list(shape)
        p_shape[t] = 1
        planes, written = _replay(program, da.values, None if partner is None else partner.values, 1.5, p_shape)
        want = pad_face_connections(
            da.values, dims, AXES, "face", CUBED_SPHERE["face"], {ax: (lo, hi)}, {a: mode for a in AXES},
            {a: 1.5 for a in AXES}, vector_axis=vec, partner=None if partner is None else partner.values,
            partner_dims=None if partner is None else partner.dims)
        for side, w, row in ((0, lo, 0), (1, hi, want.shape[t] - 1)):
            if w:
                assert (written[side] == 1).all()
                np.testing.assert_array_equal(planes[side], np.take(want, [row], axis=t), err_msg=f"{ax} {vec}")
