"""The north fold at C3 size: Grid.diff('Y') + Grid.interp('Y') of a (75, 2400, 3600) fp32 field at the Y `left`
position (its north edge is padded) on a tripolar grid with a corner pivot, beside the same calls on a plain
`fill` grid, timed alternately in one process; plus xg_fold_rows on its own.  Then the two-field composites on the
same grids: Grid.divergence (v crosses the fold) and Grid.vorticity (u crosses it) of fp32 fields of that shape with
(Y, X) metrics, fold vs plain alternated `--pair-rounds` times, beside the explicit chain a user writes on the fold
grid (Grid.diff calls and array arithmetic); and the divergence of numpy (T, Z, Y, X) fields in page-locked memory
through the host twin (xg_stencil_pair_host_fold).  Prints one JSON line, with the card name and power limit.

Usage (on the GPU box): python tools/bench_fold.py [--shape 75 2400 3600] [--rounds 3] [--pair-rounds 5]
                        [--host-lead 2 20]
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
    ap.add_argument("--pair-rounds", type=int, default=5)
    ap.add_argument("--host-lead", type=int, nargs=2, default=[2, 20])
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
    del x, da
    result = {
        "card": card(), "shape": [nz, ny, nx], "launches_per_pair_fold": launches,
        "ms_per_pair_fold": ms_f, "ms_per_pair_plain": ms_p, "fold_over_plain": ms_f / ms_p,
        "frac_of_peak_fold": bytes_fold / (ms_f * 1e-3) / 1e9 / PEAK_GBS,
        "frac_of_peak_plain": bytes_plain / (ms_p * 1e-3) / 1e9 / PEAK_GBS,
        "ms_xg_fold_rows_alone": ms_rows,
    }
    result.update(bench_composites(nz, ny, nx, args.pair_rounds, args.host_lead))
    result["card_after"] = card()
    print(json.dumps(result))


def bench_composites(nz, ny, nx, rounds, host_lead):
    """divergence / vorticity on the fold and the plain grid, the user chain on the fold grid, the host twin."""
    rng = np.random.default_rng(0)
    pos = {"C": ("YC", "XC"), "U": ("YC", "XG"), "V": ("YG", "XC"), "F": ("YG", "XG")}
    data = {}
    for p, dims in pos.items():
        for name in ("dx", "dy", "area"):
            data[f"{name}_{p}"] = (dims, (0.5 + rng.random((ny, nx))).astype(np.float32))
    ds = xg.Dataset(data_vars=data, coords={"XC": np.arange(nx) + 0.5, "XG": np.arange(nx) + 0.0,
                                            "YC": np.arange(ny) + 0.5, "YG": np.arange(ny) + 0.0})
    coords = {"X": {"center": "XC", "left": "XG"}, "Y": {"center": "YC", "left": "YG"}}
    metrics = {("X",): [f"dx_{p}" for p in pos], ("Y",): [f"dy_{p}" for p in pos],
               ("X", "Y"): [f"area_{p}" for p in pos]}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        g_fold = xg.Grid(ds, coords=coords, padding={"X": "periodic", "Y": {"fold": "corner"}}, metrics=metrics,
                         autoparse_metadata=False)
    g_plain = xg.Grid(ds, coords=coords, padding={"X": "periodic", "Y": "fill"}, metrics=metrics,
                      autoparse_metadata=False)
    a = torch.empty((nz, ny, nx), dtype=torch.float32, device="cuda:0")
    b = torch.empty_like(a)
    ops.fill_uniform(a, 11)
    ops.fill_uniform(b, 12)
    # divergence: u at U points, v at V points (v crosses the fold); vorticity: v at C points, u at F points (u
    # crosses the fold), both landing where their two terms meet
    u_div, v_div = xg.DataArray(a, dims=("Z",) + pos["U"]), xg.DataArray(b, dims=("Z",) + pos["V"])
    u_vor, v_vor = xg.DataArray(b, dims=("Z",) + pos["F"]), xg.DataArray(a, dims=("Z",) + pos["C"])
    to_div, to_vor = {"X": "center", "Y": "center"}, {"X": "left", "Y": "center"}

    def chain_div():
        t = g_fold.diff(u_div * g_fold.get_metric(u_div, ("Y",)), "X", to="center") + g_fold.diff(
            {"Y": v_div * g_fold.get_metric(v_div, ("X",))}, "Y", to="center")
        return t / g_fold.get_metric(t, ("X", "Y"))

    def chain_vor():
        t = g_fold.diff(v_vor * g_fold.get_metric(v_vor, ("Y",)), "X", to="left") - g_fold.diff(
            {"Y": u_vor * g_fold.get_metric(u_vor, ("X",))}, "Y", to="center")
        return t / g_fold.get_metric(t, ("X", "Y"))

    out = {"composite_shape": [nz, ny, nx]}
    cells = nz * ny * nx
    for name, fused, args, to, chain in (("divergence", "divergence", (u_div, v_div), to_div, chain_div),
                                         ("vorticity", "vorticity", (u_vor, v_vor), to_vor, chain_vor)):
        fold = lambda: getattr(g_fold, fused)(*args, to=to)  # noqa: E731
        plain = lambda: getattr(g_plain, fused)(*args, to=to)  # noqa: E731
        got, want = fold().data, chain().data
        n0 = _capi.load().xg_launch_count()
        fold()
        out[f"{name}_launches_fold"] = int(_capi.load().xg_launch_count() - n0)
        out[f"{name}_label_fold"] = _capi.last_launch()
        out[f"{name}_fold_equals_chain"] = bool(torch.equal(torch.nan_to_num(got), torch.nan_to_num(want)))
        del got, want
        ms_f, ms_p, ms_c = [], [], []
        for _ in range(rounds):
            ms_p.append(timed(plain))
            ms_f.append(timed(fold))
            ms_c.append(timed(chain, iters=3, reps=2, warmup=1))
        ms_f, ms_p, ms_c = statistics.median(ms_f), statistics.median(ms_p), statistics.median(ms_c)
        out.update({f"{name}_ms_fold": ms_f, f"{name}_ms_plain": ms_p, f"{name}_ms_chain_fold": ms_c,
                    f"{name}_fold_minus_plain_us": (ms_f - ms_p) * 1e3, f"{name}_chain_over_fused": ms_c / ms_f,
                    # read a, read b, write out (the fold row and the (Y, X) metrics are not counted)
                    f"{name}_frac_of_peak_fold": 3 * 4 * cells / (ms_f * 1e-3) / 1e9 / PEAK_GBS})
    del a, b, u_div, v_div, u_vor, v_vor
    torch.cuda.empty_cache()
    # numpy (T, Z, Y, X): the host twin streams T*Z slabs through the GPU
    lead = tuple(host_lead)
    hu, hv = ops.pinned_empty(lead + (ny, nx)), ops.pinned_empty(lead + (ny, nx))
    ops.fill_uniform_host(hu, 21)
    ops.fill_uniform_host(hv, 22)
    du = xg.DataArray(hu, dims=("T", "Z") + pos["U"])
    dv = xg.DataArray(hv, dims=("T", "Z") + pos["V"])
    host = lambda: g_fold.divergence(du, dv, to=to_div)  # noqa: E731
    ms_h = timed(host, iters=3, reps=1, warmup=1)
    out.update({"host_divergence_shape": list(lead) + [ny, nx], "host_divergence_ms": ms_h,
                # PCIe: two fields up, one down
                "host_divergence_GBs": 3 * hu.nbytes / (ms_h * 1e-3) / 1e9})
    return out


if __name__ == "__main__":
    main()
