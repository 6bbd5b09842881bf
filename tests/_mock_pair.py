"""CPU stand-ins for the two-field composites across a north fold, on top of the oracle-backed kernels of
``_mock_fold``, for the HOST-LOGIC tests of Grid.pair (tests/test_fold_pair_host.py).  Never imported by the package.

The fold halo plane and the host twins are CUDA launches, so Grid.pair takes them only on a CUDA device: the grids
here report one (``cuda``, never touched: every array stays a CPU tensor or a numpy array)."""

import numpy as np
import torch

from _mock_backend import _np, _t
from _mock_fold import fold_rows
from _mock_fold import install as install_fold
from oracle import stencil as oracle


def install(monkeypatch):
    from xgcm_b200 import device, ops

    install_fold(monkeypatch)
    monkeypatch.setattr(device, "default_device", lambda: torch.device("cuda"))
    plain_pair, stencil2 = ops.stencil_pair, ops.stencil2

    def stencil_pair(a, b, spec_a, spec_b, subtract=0, pre_a=None, pre_b=None, post=None, halo_lo_b=None,
                     halo_hi_b=None):
        """The definition of xg_stencil_pair_halo: the term along axis_b with its halo planes (the halo form of the
        stencil2 stand-in), then the chain's arithmetic, each step rounded to the field dtype."""
        if halo_lo_b is None and halo_hi_b is None:
            return plain_pair(a, b, spec_a, spec_b, subtract, pre_a, pre_b, post)
        op_a, lo_a, hi_a, pad_a, fill_a = spec_a
        axis_b, op_b, lo_b, hi_b, pad_b, fill_b = spec_b
        aa = _np(a)
        ta = oracle.stencil2(op_a, aa, aa.ndim - 1, lo_a, hi_a, pad_a, fill_a, _np(pre_a))
        tb = _np(stencil2(b, axis_b, op_b, lo_b, hi_b, pad_b, fill_b, pre=pre_b, halo_lo=halo_lo_b, halo_hi=halo_hi_b))
        r = ta + tb if not subtract else (ta - tb if int(subtract) == 1 else tb - ta)
        if post is not None:
            with np.errstate(invalid="ignore", divide="ignore"):
                r = r / _np(post)
        return _t(r.astype(aa.dtype))

    def stencil_pair_host(a, b, spec_a, spec_b, subtract=0, pre_a=None, pre_b=None, post=None, out=None,
                          device=None):
        return ops.stencil_pair(_t(a), _t(b), spec_a, spec_b, subtract, pre_a=pre_a, pre_b=pre_b, post=post).numpy()

    def stencil_pair_host_fold(a, b, spec_a, spec_b, seam_axis, skip, mirror, period, subtract=0, negate=False,
                               pre_a=None, pre_b=None, post=None, out=None, device=None):
        """The definition of xg_stencil_pair_host_fold: b's folded row is halo_hi_b, and halo_lo_b under a
        periodic south edge."""
        axis_b, _, lo_b, _, pad_b, _ = spec_b
        halo_hi = fold_rows(_t(b), axis_b, seam_axis, 1, skip, mirror, period, negate=negate, pre=pre_b)
        halo_lo = halo_hi if lo_b and pad_b == "periodic" else None
        return ops.stencil_pair(_t(a), _t(b), spec_a, spec_b, subtract, pre_a=pre_a, pre_b=pre_b, post=post,
                                halo_lo_b=halo_lo, halo_hi_b=halo_hi).numpy()

    for name, fn in dict(stencil_pair=stencil_pair, stencil_pair_host=stencil_pair_host,
                         stencil_pair_host_fold=stencil_pair_host_fold).items():
        monkeypatch.setattr(ops, name, fn)
