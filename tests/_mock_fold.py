"""CPU stand-in for ``xg_fold_rows`` on top of the oracle-backed kernels of ``_mock_backend``, for the HOST-LOGIC
tests of the north fold (tests/test_fold_host.py).  Never imported by the package."""

import numpy as np

from _mock_backend import _np, _t
from _mock_backend import install as install_backend


def fold_rows(x, fold_axis, seam_axis, width, skip, mirror, period, negate=False, pre=None, out=None, row0=0):
    """The definition of xg_fold_rows (include/xgcm_b200.h), including its argument checks."""
    a = _np(x) if pre is None else _np(x) * np.broadcast_to(_np(pre), _np(x).shape)
    n, length = a.shape[fold_axis], a.shape[seam_axis]
    if fold_axis == seam_axis or width < 1 or width > n - skip:
        raise ValueError("xg_fold_rows: bad fold / seam axes or halo width")
    src = [(mirror - k) % period for k in range(length)]
    if max(src) >= length:
        raise NotImplementedError("xg_fold_rows: seam position incompatible with the pivot")
    rows = np.take(np.take(a, [n - 1 - skip - r for r in range(width)], axis=fold_axis), src, axis=seam_axis)
    rows = (-rows if negate else rows).astype(_np(x).dtype)
    if out is None:
        return _t(rows)
    o = out.numpy()
    sl = [slice(None)] * o.ndim
    sl[fold_axis] = slice(row0, row0 + width)
    o[tuple(sl)] = rows
    return out


def install(monkeypatch):
    from xgcm_b200 import ops

    install_backend(monkeypatch)
    monkeypatch.setattr(ops, "fold_rows", fold_rows)
