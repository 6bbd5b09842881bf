"""Every host-buffer entry point streams through one device workspace: a fold stencil call and a cumscan_host call
on numpy fields share its slot buffers, and both workspace queries report that one workspace."""

import ctypes as C

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from oracle import stencil as S
from test_host_halo_gpu import NX, NY, _fold_grid, _fold_oracle, _host
from xgcm_b200 import _capi, ops

pytestmark = pytest.mark.gpu


def _both_queries():
    lib = _capi.load()
    got = []
    for query in (lib.xg_host_workspace_bytes, lib.xg_host_pipe_workspace_bytes):
        v = C.c_int64(-1)
        _capi.check(query(torch.cuda.current_device(), C.byref(v)))
        got.append(v.value)
    return got


def test_stencil_and_pipe_calls_share_one_workspace(monkeypatch):
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")
    lib = _capi.load()
    _, grid = _fold_grid("periodic", "corner", np.float32)
    a = np.random.default_rng(3).standard_normal((12, 20, NY, NX)).astype(np.float32)
    da = xg.DataArray(a, dims=("time", "z", "yleft", "xcenter"))
    rng = np.random.default_rng(4)
    c = rng.random((30, 64, 100)).astype(np.float32)
    pre = (rng.random(c.shape) + 0.5).astype(np.float32)

    def fold():  # xg_stencil2_host_fold, several slabs
        got = grid.diff(da, "Y", to="center")
        np.testing.assert_array_equal(_host(got), _fold_oracle("diff", a, "left", "center", "corner", 0, 1, "periodic"))

    def scan():  # xg_cumscan_host, several slabs
        got = ops.cumscan_host(c, 1, pre=pre)
        np.testing.assert_array_equal(got, S.cumscan(c, 1, False, "none", 0, 0, None, 0.0, pre, None, True))

    alone = []
    for call in (fold, scan):
        _capi.check(lib.xg_host_workspace_release())
        assert _both_queries() == [0, 0]
        call()
        stencil_bytes, pipe_bytes = _both_queries()
        assert stencil_bytes == pipe_bytes > 0
        alone.append(stencil_bytes)

    _capi.check(lib.xg_host_workspace_release())
    fold()
    scan()
    stencil_bytes, pipe_bytes = _both_queries()
    assert stencil_bytes == pipe_bytes
    assert max(alone) <= stencil_bytes < sum(alone), (alone, stencil_bytes)
    _capi.check(lib.xg_host_workspace_release())
    assert _both_queries() == [0, 0]
