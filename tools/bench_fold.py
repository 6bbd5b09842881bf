"""The north fold at C3 size: Grid.diff('Y') + Grid.interp('Y') of a (75, 2400, 3600) fp32 field at the Y `left`
position (its north edge is padded) on a tripolar grid with a corner pivot, beside the same calls on a plain
`fill` grid, timed alternately in one process; plus xg_fold_rows on its own.  Prints one JSON line.

Usage (on the GPU box): python tools/bench_fold.py [--shape 75 2400 3600] [--rounds 3]
"""

import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import xgcm_b200 as xg  # noqa: E402
from xgcm_b200 import _capi, ops  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet


def timed(fn, iters=5, reps=4, warmup=2):
    """median over `iters` of (time of `reps` back-to-back calls) / reps, CUDA events."""
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) / reps)
    return statistics.median(ts)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return out or None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", type=int, nargs=3, default=[75, 2400, 3600])
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    nz, ny, nx = args.shape
    x = torch.empty((nz, ny, nx), dtype=torch.float32, device="cuda:0")
    ops.fill_uniform(x, 0xC0FFEE)
    ds = xg.Dataset(coords={"XC": np.arange(nx) + 0.5, "YC": np.arange(ny) + 0.5, "YG": np.arange(ny) + 0.0})
    coords = {"X": {"center": "XC"}, "Y": {"center": "YC", "left": "YG"}}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)  # the fold is flagged experimental
        g_fold = xg.Grid(ds, coords=coords, padding={"X": "periodic", "Y": {"fold": "corner"}},
                         autoparse_metadata=False)
    g_plain = xg.Grid(ds, coords=coords, padding={"X": "periodic", "Y": "fill"}, autoparse_metadata=False)
    da = xg.DataArray(x, dims=("Z", "YG", "XC"))

    def f_plain():
        g_plain.diff(da, "Y")
        g_plain.interp(da, "Y")

    def f_fold():
        g_fold.diff(da, "Y")
        g_fold.interp(da, "Y")

    n0 = _capi.load().xg_launch_count()
    f_fold()
    launches = int(_capi.load().xg_launch_count() - n0)
    ms_p, ms_f = [], []
    for _ in range(args.rounds):
        ms_p.append(timed(f_plain))
        ms_f.append(timed(f_fold))
    ms_p, ms_f = statistics.median(ms_p), statistics.median(ms_f)
    cells, row = x.numel(), nz * nx
    bytes_plain = 2 * 8 * cells
    bytes_fold = 2 * (8 * cells + 12 * row)  # + per op: the mirrored row read and written, and read as the halo
    ms_rows = timed(lambda: ops.fold_rows(x, 1, 2, 1, 1, 0, nx), iters=20, reps=1)
    print(json.dumps({
        "card": card(), "shape": [nz, ny, nx], "launches_per_pair_fold": launches,
        "ms_per_pair_fold": ms_f, "ms_per_pair_plain": ms_p, "fold_over_plain": ms_f / ms_p,
        "frac_of_peak_fold": bytes_fold / (ms_f * 1e-3) / 1e9 / PEAK_GBS,
        "frac_of_peak_plain": bytes_plain / (ms_p * 1e-3) / 1e9 / PEAK_GBS,
        "ms_xg_fold_rows_alone": ms_rows,
    }))


if __name__ == "__main__":
    main()
