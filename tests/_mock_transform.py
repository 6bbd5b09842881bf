"""CPU stand-in for the C-ABI of the conservative transform's host twin, for the HOST-LOGIC tests of
tests/test_transform_host.py.  Never imported by the package.

On top of the oracle-backed ops of ``_mock_backend``, ``xg_vinterp_conservative_host`` is replaced by its
definition (the oracle on the host buffers it is handed), so ``ops.vinterp_conservative_host`` runs for real:
promotion, bin flip and theta strides included.  Every call is recorded in ``CALLS``.  The grids report a CUDA
device (``cuda``, never touched: every array stays a CPU tensor or a numpy array)."""

import ctypes as C

import numpy as np
import torch

from _mock_backend import install as install_backend
from oracle import stencil as oracle

CALLS = []


def _host_array(addr, dtype, count):
    buf = (C.c_char * (int(count) * np.dtype(dtype).itemsize)).from_address(int(addr))
    return np.frombuffer(buf, dtype=dtype, count=int(count))


def xg_vinterp_conservative_host(dtype, phi, theta, theta_strides, theta_at_centers, bins, m, flip, out, ndim, shape,
                                 axis, device):
    """The definition of xg_vinterp_conservative_host on host buffers."""
    dt = np.float32 if dtype == 0 else np.float64
    es = np.dtype(dt).itemsize
    shape = [int(shape[d]) for d in range(ndim)]
    strides = [int(theta_strides[d]) for d in range(ndim)]
    tshape = list(shape)
    tshape[axis] += 0 if theta_at_centers else 1
    span = 1 + sum((t - 1) * s for t, s in zip(tshape, strides) if t > 1)
    th = np.lib.stride_tricks.as_strided(_host_array(theta, dt, span), tshape, [s * es for s in strides])
    if theta_at_centers:  # grid.interp(theta, axis, padding="extend"): the center -> outer shift
        th = oracle.stencil2("interp", np.ascontiguousarray(th), axis, 1, 1, "extend").astype(dt)
    p = _host_array(phi, dt, np.prod(shape)).reshape(shape)
    r = oracle.vinterp_conservative(p, th, _host_array(bins, dt, m), axis)
    if flip:
        r = r[..., ::-1]
    _host_array(out, dt, r.size)[:] = r.reshape(-1)
    CALLS.append(dict(dtype=dt, axis=axis, shape=tuple(shape), theta_shape=tuple(tshape), theta_strides=tuple(strides),
                      theta_at_centers=int(theta_at_centers), flip=int(flip), m=int(m)))
    return 0


class _Lib:
    xg_vinterp_conservative_host = staticmethod(xg_vinterp_conservative_host)


def install(monkeypatch):
    from xgcm_b200 import _capi, device, ops

    install_backend(monkeypatch)
    CALLS.clear()
    monkeypatch.setattr(device, "default_device", lambda: torch.device("cuda"))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(ops, "pinned_empty", lambda shape, dtype=np.float32: np.empty(tuple(shape), dtype))
    monkeypatch.setattr(_capi, "load", lambda: _Lib())
