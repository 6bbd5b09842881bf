"""The device halo of a face-connected operator without a GPU (mock backend): ``padding.connected_halo_planes`` runs
the copy list of ``connected_halo_program`` in one batched strided copy (and one product for a metric-weighted halo),
and its planes are the first / last plane of oracle/faces.py's padding of ``x`` (or ``x * m``), on whole fields and
on blocks of faces whose remote edges are left to the caller."""

import itertools

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from _mock_backend import install
from oracle.faces import pad_face_connections
from xgcm_b200 import ops
from xgcm_b200.padding import _connected_edge_plan, connected_halo_planes

N = 4
AXES = {"X": ("x", "xl"), "Y": ("y", "yl")}
COORDS = {"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"}}
# xgcm/test/test_faceconnections.py:99-127, and the two-face seams of xgcm/test/test_padding.py
TOPOLOGIES = {
    "cubed_sphere": {
        0: {"X": ((3, "X", False), (1, "X", False)), "Y": ((4, "Y", False), (5, "Y", False))},
        1: {"X": ((0, "X", False), (2, "X", False)), "Y": ((4, "X", False), (5, "X", True))},
        2: {"X": ((1, "X", False), (3, "X", False)), "Y": ((4, "Y", True), (5, "Y", True))},
        3: {"X": ((2, "X", False), (0, "X", False)), "Y": ((4, "X", True), (5, "X", False))},
        4: {"X": ((3, "Y", True), (1, "Y", False)), "Y": ((2, "Y", True), (0, "Y", False))},
        5: {"X": ((3, "Y", False), (1, "Y", True)), "Y": ((0, "Y", False), (2, "Y", True))},
    },
    "right_left_same_axis": {0: {"X": (None, (1, "X", False))}, 1: {"X": ((0, "X", False), None)}},
    "right_right_same_axis": {0: {"X": (None, (1, "X", True))}, 1: {"X": (None, (0, "X", True))}},
    "right_left_swap_axis": {0: {"X": (None, (1, "Y", False))}, 1: {"Y": ((0, "X", False), None)}},
    "right_right_swap_axis": {0: {"X": (None, (1, "Y", True))}, 1: {"Y": (None, (0, "X", True))}},
}


@pytest.fixture
def counts(monkeypatch):
    """Oracle-backed ops; the number of batched copies, single copies and products each call issues."""
    if torch.cuda.is_available():
        pytest.skip("real kernels available: the connected operators are covered by the gpu-marked modules")
    install(monkeypatch)
    n = {"strided_copy_batch": 0, "strided_copy": 0, "binary": 0}
    for name in n:
        def spy(*a, _fn=getattr(ops, name), _name=name, **kw):
            n[_name] += 1
            return _fn(*a, **kw)

        monkeypatch.setattr(ops, name, spy)
    return n


def _blocks(n_face):
    """The whole field, and contiguous blocks of faces as a face-sharded rank holds them."""
    return [(0, n_face)] + ([(0, 1), (1, 1)] if n_face == 2 else [(0, 3), (2, 2), (5, 1)])


# the weighted product also runs over the planes' remote edges, which hold whatever the allocation held
@pytest.mark.filterwarnings("ignore:overflow encountered in multiply:RuntimeWarning")
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("mode", ["fill", "extend", "periodic"])
@pytest.mark.parametrize("name", sorted(TOPOLOGIES))
def test_halo_planes_match_oracle(counts, name, mode, dtype):
    links = TOPOLOGIES[name]
    nf = len(links)
    rng = np.random.default_rng(len(name))
    data = {k: rng.standard_normal((2, nf, N, N)).astype(dtype) for k in "cuv"}
    data["m"] = (0.5 + rng.random((1, nf, N, N))).astype(dtype)
    dims = {"c": ("t", "face", "y", "x"), "u": ("t", "face", "y", "xl"), "v": ("t", "face", "yl", "x")}
    ds = xg.Dataset(coords={"face": np.arange(nf), "t": np.arange(2.0), "x": np.arange(N) + 0.0,
                            "xl": np.arange(N) - 0.5, "y": np.arange(N) + 0.0, "yl": np.arange(N) - 0.5})
    grid = xg.Grid(ds, coords=COORDS, face_connections={"face": links}, autoparse_metadata=False)
    fill = 0.1
    cases = [("c", None, False), ("c", None, True), ("u", "X", False), ("v", "Y", False)]
    for ax, (lo, hi), (key, vec, weighted), (f0, nb) in itertools.product(
            ["X", "Y"], [(1, 0), (0, 1), (1, 1)], cases, _blocks(nf)):
        block = slice(f0, f0 + nb)
        partner_key = {"X": "v", "Y": "u"}.get(vec)
        arr = lambda k: xg.DataArray(torch.from_numpy(np.ascontiguousarray(data[k][:, block])), dims=dims[k])  # noqa
        da, other = (arr(key), None) if vec is None else ({vec: arr(key)}, {"Y" if vec == "X" else "X": arr(partner_key)})
        pre = torch.from_numpy(np.ascontiguousarray(data["m"][:, block])) if weighted else None
        remote = [] if nb < nf else None
        for k in counts:
            counts[k] = 0
        x, halo_lo, halo_hi, _, out_dims = connected_halo_planes(
            da, grid, ax, lo, hi, mode, fill, other, face_offset=f0, remote_edges=remote, pre=pre)
        what = f"{ax} {(lo, hi)} {key} pre={weighted} faces {f0}..{f0 + nb - 1}"
        assert (counts["strided_copy_batch"], counts["strided_copy"]) == (1, 0), what
        assert counts["binary"] == (1 if weighted else 0), what
        assert out_dims == dims[key]

        t = out_dims.index([d for d in out_dims if d in AXES[ax]][0])
        shape = list(x.shape)
        layout = None if vec is None else (dims[partner_key], tuple(shape))
        want_remote = [] if remote is not None else None
        _connected_edge_plan(grid, ax, lo, hi, out_dims, shape, vec, layout, f0, want_remote)
        assert remote == want_remote, what

        field = data[key] * data["m"] if weighted else data[key]
        want = pad_face_connections(
            field, dims[key], AXES, "face", links, {ax: (lo, hi)}, {a: mode for a in AXES}, {a: fill for a in AXES},
            vector_axis=vec, partner=None if vec is None else data[partner_key],
            partner_dims=None if vec is None else dims[partner_key])
        for side, plane, row in ((0, halo_lo, 0), (1, halo_hi, want.shape[t] - 1)):
            if not (lo, hi)[side]:
                assert plane is None, what
                continue
            assert plane.dtype == x.dtype and list(plane.shape) == shape[:t] + [1] + shape[t + 1:], what
            for i in range(nb):  # remote edges are the caller's to write
                if (side, i) not in {(s, j) for s, j, _ in remote or []}:
                    np.testing.assert_array_equal(plane.numpy()[:, i], np.take(want, [row], axis=t)[:, f0 + i],
                                                  err_msg=f"{what} side {side} face {f0 + i}")
