"""Metric-weighted multi-axis Grid.diff / interp on a C3-sized (75, 2400, 3600) fp32 field (Z, Y, X), X periodic,
Y fill, Z extend.  Cases:

  interp_xy_area    interp(["X", "Y"], metric_weighted=["X", "Y"]) with 2-D areas registered at every position
  interp_xy_volume  the same with a 3-D volume-like metric at every position
  diff_xyz          diff(["X", "Y", "Z"], metric_weighted={"X": "X", "Y": "Y"}) with 1-D dx / dy

For each case, alternated in one process with CUDA events after warm-up:

  grid      the Grid call as a user makes it (its last launch label is reported: the route Grid chose)
  fused     ops.stencil_multi with the stage metrics Grid resolves (xg_stencil_multi_weighted)
  per_axis  the single-axis weighted calls in series
  l2_met    the fused launch with every metric replaced by one row (1, X) of it: the same instructions with metric
            reads that stay in L1 / L2, so fused - l2_met is what the metrics' memory traffic costs
  free      the metric-free fused launch on the same field, the ceiling

The fused and per-axis outputs are compared bit for bit.  Algorithmic bytes: the field in and the result out, plus
each distinct metric array the chain reads, once.  With --host, the first case also runs on a page-locked numpy field
(host clock around each synchronous call): streamed (xg_stencil_multi_weighted_host) against the Grid route for the
same field resident on the device (upload, the device call Grid chooses, download), compared bit for bit.  Prints one
JSON line with the card name and power limit.
"""

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import xgcm_b200 as xg  # noqa: E402
from xgcm_b200 import _capi, ops  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=10).stdout.strip()
    return out or None


def timed_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def make_grid(shape, case, rng):
    nz, ny, nx = shape
    sizes = {"Z": nz, "Y": ny, "X": nx}
    coords = {ax: {"center": ax + "C", "left": ax + "G"} for ax in "ZYX"}
    ds_coords = {ax + s: np.arange(n) + off for ax, n in sizes.items() for s, off in (("C", 0.5), ("G", 0.0))}
    data_vars, metrics = {}, {}
    if case == "interp_xy_area":
        for py in "CG":
            for px in "CG":
                data_vars[f"area_{py}{px}"] = (("Y" + py, "X" + px), rng.random((ny, nx), dtype=np.float32) + 0.5)
        metrics[("X", "Y")] = list(data_vars)
    elif case == "interp_xy_volume":
        for py in "CG":
            for px in "CG":
                data_vars[f"vol_{py}{px}"] = (("ZC", "Y" + py, "X" + px),
                                              rng.random((nz, ny, nx), dtype=np.float32) + 0.5)
        metrics[("X", "Y")] = list(data_vars)
    else:
        for ax, n in (("X", nx), ("Y", ny)):
            names = []
            for p in "CG":
                data_vars[f"d{ax.lower()}_{p}"] = ((ax + p,), rng.random(n, dtype=np.float32) + 0.5)
                names.append(f"d{ax.lower()}_{p}")
            metrics[(ax,)] = names
    ds = xg.Dataset(data_vars=data_vars, coords=ds_coords)
    grid = xg.Grid(ds, coords=coords, padding={"X": "periodic", "Y": "fill", "Z": "extend"}, metrics=metrics,
                   autoparse_metadata=False)
    return grid, sum(v[1].nbytes for v in data_vars.values())


def stage_operands(grid, da, axes, op, w, x):
    """Specs and per-stage device metrics of the chain "every axis to the left" (what Grid resolves)."""
    pads = {"X": "periodic", "Y": "fill", "Z": "extend"}
    dims, shape = list(da.dims), list(da.shape)
    specs, pre, post = [], [], []
    for ax in axes:
        num = dims.index(ax + "C")
        specs.append((num, op, 1, 0, pads[ax], 0.0))
        out_dims = list(dims)
        out_dims[num] = ax + "G"
        wa = w.get(ax) if isinstance(w, dict) else w
        if wa:
            probe_in = xg.DataArray(np.empty((1,) * len(dims), np.float32), dims=tuple(dims))
            probe_out = xg.DataArray(np.empty((1,) * len(dims), np.float32), dims=tuple(out_dims))
            pre.append(grid._metric_tensor(grid.get_metric(probe_in, wa), dims, x))
            post.append(grid._metric_tensor(grid.get_metric(probe_out, wa), out_dims, x))
        else:
            pre.append(None)
            post.append(None)
        dims = out_dims
    return specs, pre, post


CASES = {
    "interp_xy_area": ("interp", ["X", "Y"], ["X", "Y"]),
    "interp_xy_volume": ("interp", ["X", "Y"], ["X", "Y"]),
    "diff_xyz": ("diff", ["X", "Y", "Z"], {"X": "X", "Y": "Y"}),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", type=int, nargs=3, default=[75, 2400, 3600])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multi_weighted needs a CUDA device")
    shape = tuple(args.shape)
    rng = np.random.default_rng(0)
    x = torch.rand(shape, dtype=torch.float32, device="cuda")
    da = xg.DataArray(x, dims=("ZC", "YC", "XC"))
    field_bytes = x.numel() * 4
    result = {"card": card(), "shape": list(shape), "dtype": "float32", "cases": {}}
    for name, (op, axes, w) in CASES.items():
        grid, _ = make_grid(shape, name, rng)
        to = {ax: "left" for ax in axes}
        fn = getattr(grid, op)

        def per_axis():
            cur = da
            for ax in axes:
                cur = fn(cur, ax, to={ax: "left"}, metric_weighted=w.get(ax) if isinstance(w, dict) else w)
            return cur

        specs, pre, post = stage_operands(grid, da, axes, op, w, x)
        read = {m.data_ptr(): m.numel() * m.element_size() for m in pre + post if m is not None}
        metric_bytes = sum(read.values())
        rows = lambda ms: [None if m is None else m[..., :1, :].contiguous() for m in ms]  # noqa: E731
        pre_r, post_r = rows(pre), rows(post)
        fused = lambda: ops.stencil_multi(x, specs, pre=pre, post=post)  # noqa: E731
        l2_met = lambda: ops.stencil_multi(x, specs, pre=pre_r, post=post_r)  # noqa: E731
        free = lambda: ops.stencil_multi(x, specs)  # noqa: E731
        user = lambda: fn(da, axes, to=to, metric_weighted=w)  # noqa: E731
        got = xg.DataArray(fused(), dims=da.dims)
        label = _capi.last_launch()
        user()
        grid_label = _capi.last_launch()
        want = per_axis()
        same = bool(torch.equal(torch.nan_to_num(got.data, nan=7.0), torch.nan_to_num(want.data, nan=7.0))
                    and torch.equal(torch.isnan(got.data), torch.isnan(want.data)))
        del got, want
        free()
        l2_met()
        times = {"grid": [], "fused": [], "per_axis": [], "l2_met": [], "free": []}
        fns = {"grid": user, "fused": fused, "per_axis": per_axis, "l2_met": l2_met, "free": free}
        for _ in range(args.rounds):
            for k, f in fns.items():
                times[k].append(timed_ms(f))
        med = {k: statistics.median(v) for k, v in times.items()}
        alg = 2 * field_bytes + metric_bytes
        result["cases"][name] = {
            "fused_label": label, "grid_label": grid_label, "bit_equal": same,
            "ms": {k: round(v, 3) for k, v in med.items()},
            "algorithmic_bytes": alg,
            "fused_GBps": round(alg / med["fused"] / 1e6, 1),
            "free_GBps": round(2 * field_bytes / med["free"] / 1e6, 1),
            "fused_speedup_vs_per_axis": round(med["per_axis"] / med["fused"], 3),
        }
        torch.cuda.empty_cache()
    if args.host:
        op, axes, w = CASES["interp_xy_area"]
        grid, _ = make_grid(shape, "interp_xy_area", rng)
        a = ops.pinned_empty(shape, np.float32)
        a[...] = x.cpu().numpy()
        hda = xg.DataArray(a, dims=("ZC", "YC", "XC"))
        to = {ax: "left" for ax in axes}

        def streamed():
            return grid.interp(hda, axes, to=to, metric_weighted=w)

        def whole():
            out = grid.interp(xg.DataArray(torch.from_numpy(a).cuda(), dims=hda.dims), axes, to=to,
                              metric_weighted=w)
            return out.data.cpu().numpy()

        s_out, w_out = np.asarray(streamed().data), whole()
        th = {"streamed": [], "whole_field": []}
        for _ in range(args.rounds):
            for k, f in (("streamed", streamed), ("whole_field", whole)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                f()
                torch.cuda.synchronize()
                th[k].append(time.perf_counter() - t0)
        result["host_interp_xy_area"] = {
            "bit_equal": bool(np.array_equal(s_out, w_out, equal_nan=True)),
            "s": {k: round(statistics.median(v), 4) for k, v in th.items()},
        }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
