"""Numpy fields on face-connected and north-fold grids through the host slab pipelines, beside the plain-grid
host call on the same shape (the ceiling: same slabs, no halo stage) and beside the old whole-field route
(upload, device call, download): Grid.diff, and Grid.cumsum across the faces (X to outer: a trimmed shift such as
X to left raises across the cubed sphere's axis-swapping seams), along Z, and reversed across the fold; and the
multi-axis chains, Grid.diff(["X", "Y"]) across the faces and Grid.interp(["X", "Y"]) across the fold, beside the
same call on a plain grid (xg_stencil_multi_host, one fused launch per slab), the old route and the single-axis
streamed call.
Page-locked inputs, host clock around each synchronous call, the variants alternated `--rounds` times in one
process.  Prints one JSON line with the card, its power limit, the median seconds and GB/s (bytes in + out over
time) of every variant, its ratio to the plain-grid ceiling and to the old route, and tools/bench_pcie.py's copy
rates.

    python tools/bench_host_halo.py [--faces 90 6 2160 2160] [--fold [T] 75 3059 4322] [--rounds 5]

If MemAvailable allows about 2.2x of it, a year of monthly ORCA12-like temperature (12, 75, 3059, 4322) fp32
(47.6 GB) also streams across the fold (diff, then the reverse cumsum), with sampled time steps checked against
oracle/fold.py.  The old route runs only where its device buffers fit on the card with room to spare.
"""

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import xgcm_b200 as xg  # noqa: E402
from xgcm_b200 import ops  # noqa: E402

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


def card():
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out or None


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def pinned_random(shape, seed):
    a = ops.pinned_empty(shape, np.float32)
    ops.fill_uniform_host(a.reshape(-1), seed)
    return a


def timed_call(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def old_route(grid, method, da, dims, other=None, **kw):
    """Upload, device call, download: what a numpy field on these grids did before it streamed."""
    def run():
        x = xg.DataArray(torch.from_numpy(da).to("cuda:0", non_blocking=True), dims=dims)
        extra = {}
        if other is not None:
            (oax, (q, qdims)), = other.items()
            extra["other_component"] = {oax: xg.DataArray(torch.from_numpy(q).to("cuda:0", non_blocking=True),
                                                          dims=qdims)}
        return getattr(grid, method)(x, **kw, **extra).data.cpu()
    return run


def faces_variants(shape):
    nt, nf, ny, nx = shape
    coords = {"x": np.arange(nx) + 0.0, "xl": np.arange(nx) - 0.5, "xo": np.arange(nx + 1) - 0.5,
              "y": np.arange(ny) + 0.0, "yl": np.arange(ny) - 0.5, "face": np.arange(nf), "k": np.arange(nt) + 0.0,
              "kl": np.arange(nt) - 0.5}
    ds = xg.Dataset(coords=coords)
    axes = {"X": {"center": "x", "left": "xl", "outer": "xo"}, "Y": {"center": "y", "left": "yl"},
            "Z": {"center": "k", "left": "kl"}}
    grid = xg.Grid(ds, coords=axes, face_connections=CUBED_SPHERE)
    plain = xg.Grid(ds, coords=axes, padding="fill")
    c = pinned_random(shape, 1)
    v = pinned_random(shape, 2)
    cd, ud, vd = ("k", "face", "y", "x"), ("k", "face", "y", "xl"), ("k", "face", "yl", "x")
    fits = 3 * c.nbytes < 0.8 * torch.cuda.mem_get_info()[0]
    variants = {
        "faces_scalar_diffX": lambda: grid.diff(xg.DataArray(c, dims=cd), "X", padding="fill"),
        "faces_vector_diffX": lambda: grid.diff({"X": xg.DataArray(c, dims=ud)}, "X",
                                                other_component={"Y": xg.DataArray(v, dims=vd)}, padding="fill"),
        "plain_diffX": lambda: plain.diff(xg.DataArray(c, dims=cd), "X"),
        "faces_cumsumX": lambda: grid.cumsum(xg.DataArray(c, dims=cd), "X", to="outer"),
        "plain_cumsumX": lambda: plain.cumsum(xg.DataArray(c, dims=cd), "X", to="outer"),
        "faces_cumsumZ": lambda: grid.cumsum(xg.DataArray(c, dims=cd), "Z", padding="fill"),
        "plain_cumsumZ": lambda: plain.cumsum(xg.DataArray(c, dims=cd), "Z"),
        "faces_diffXY": lambda: grid.diff(xg.DataArray(c, dims=cd), ["X", "Y"], padding="fill"),
        "plain_diffXY": lambda: plain.diff(xg.DataArray(c, dims=cd), ["X", "Y"]),
    }
    if fits:  # input, intermediate, result
        variants["faces_diffXY_old"] = old_route(grid, "diff", c, cd, axis=["X", "Y"], padding="fill")
        variants["faces_scalar_diffX_old"] = old_route(grid, "diff", c, cd, axis="X", padding="fill")
        variants["faces_vector_diffX_old"] = old_route(grid, "diff", c, ud, {"Y": (v, vd)}, axis="X", padding="fill")
    if 4 * c.nbytes < 0.8 * torch.cuda.mem_get_info()[0]:  # input, scan, padded copy, result
        variants["faces_cumsumX_old"] = old_route(grid, "cumsum", c, cd, axis="X", to="outer")
        variants["faces_cumsumZ_old"] = old_route(grid, "cumsum", c, cd, axis="Z", padding="fill")
    return variants, 2 * c.nbytes, {"faces_vector_diffX": 3 * c.nbytes, "faces_vector_diffX_old": 3 * c.nbytes}


def fold_grid(ny, nx):
    coords = {"xc": np.arange(nx), "xl": np.arange(nx), "yc": np.arange(ny), "yl": np.arange(ny)}
    ds = xg.Dataset(coords=coords)
    axes = {"X": {"center": "xc", "left": "xl"}, "Y": {"center": "yc", "left": "yl"}}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords=axes, padding={"X": "periodic", "Y": {"fold": "T", "south": "fill"}},
                       autoparse_metadata=False)
    return grid, xg.Grid(ds, coords=axes, padding={"X": "periodic", "Y": "fill"}, autoparse_metadata=False)


def fold_variants(shape):
    grid, plain = fold_grid(shape[-2], shape[-1])
    a = pinned_random(shape, 3)
    dims = ("t", "z", "yl", "xc")[-len(shape):]
    variants = {
        "fold_interpXY": lambda: grid.interp(xg.DataArray(a, dims=dims), ["X", "Y"], to={"Y": "center"}),
        "plain_fold_shape_interpXY": lambda: plain.interp(xg.DataArray(a, dims=dims), ["X", "Y"], to={"Y": "center"}),
        "fold_diffY": lambda: grid.diff(xg.DataArray(a, dims=dims), "Y", to="center"),
        "plain_fold_shape_diffY": lambda: plain.diff(xg.DataArray(a, dims=dims), "Y", to="center"),
        "fold_cumsumY_reverse": lambda: grid.cumsum(xg.DataArray(a, dims=dims), "Y", to="center", reverse=True),
        "plain_fold_shape_cumsumY_reverse": lambda: plain.cumsum(xg.DataArray(a, dims=dims), "Y", to="center",
                                                                 reverse=True),
    }
    if 2 * a.nbytes < 0.8 * torch.cuda.mem_get_info()[0]:
        variants["fold_diffY_old"] = old_route(grid, "diff", a, dims, axis="Y", to="center")
    if 3 * a.nbytes < 0.8 * torch.cuda.mem_get_info()[0]:  # input, intermediate, result
        variants["fold_interpXY_old"] = old_route(grid, "interp", a, dims, axis=["X", "Y"], to={"Y": "center"})
    if 4 * a.nbytes < 0.8 * torch.cuda.mem_get_info()[0]:  # input, scan, padded copy, result
        variants["fold_cumsumY_reverse_old"] = old_route(grid, "cumsum", a, dims, axis="Y", to="center", reverse=True)
    return variants, 2 * a.nbytes, {}


def pcie():
    try:
        out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_pcie.py")], capture_output=True,
                             text=True, timeout=600).stdout.strip().splitlines()
        return json.loads(out[-1])
    except Exception as err:  # the ceiling is context, not the measurement
        return {"error": repr(err)}


def orca_year(rounds):
    shape = (12, 75, 3059, 4322)
    nbytes = int(np.prod(shape)) * 4
    if mem_available() < 2.2 * nbytes:
        return {"skipped": f"MemAvailable {mem_available() / 1e9:.1f} GB < 2.2 x {nbytes / 1e9:.1f} GB"}
    from oracle import fold as F
    from oracle import stencil as S

    grid, _ = fold_grid(shape[2], shape[3])
    a = pinned_random(shape, 4)
    da = xg.DataArray(a, dims=("t", "z", "yl", "xc"))
    roles = F.resolve_pivot("T", "Y", "X")
    steps = ((0, 0), (5, 40), (11, 74))
    result = {"shape": shape, "checked_steps": [list(s) for s in steps]}
    for name, call, want in (
            ("diffY", lambda: grid.diff(da, "Y", to="center"),
             lambda s: S.stencil2("diff", F.pad_fold(s, 0, 1, "left", "center", roles, {0: (0, 1)}, {0: "fill"}),
                                  0, 0, 0, None)),
            ("cumsumY_reverse", lambda: grid.cumsum(da, "Y", to="center", reverse=True),
             lambda s: F.pad_fold(S.cumscan(s, 0, True, "drop_first"), 0, 1, "left", "center", roles, {0: (0, 1)},
                                  {0: "fill"}))):
        ts = []
        for _ in range(max(1, rounds // 2)):
            out = [None]
            ts.append(timed_call(lambda: out.__setitem__(0, call())))
        got = out[0].data
        for t, z in steps:
            np.testing.assert_array_equal(got[t, z], want(a[t, z]))
        del out, got
        result[name] = {"s": statistics.median(ts), "GBps": 2 * nbytes / statistics.median(ts) / 1e9}
    return result


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--faces", type=int, nargs=4, default=[90, 6, 2160, 2160])
    p.add_argument("--fold", type=int, nargs="+", default=[75, 3059, 4322])
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--skip-year", action="store_true")
    args = p.parse_args()
    torch.cuda.init()
    result = {"card": card(), "pcie": pcie()}
    for nbytes, build in ((4 * int(np.prod(args.faces)), lambda: faces_variants(tuple(args.faces))),
                          (4 * int(np.prod(args.fold)), lambda: fold_variants(tuple(args.fold)))):
        if mem_available() < 6 * nbytes:  # inputs, partner and pinned outputs
            result.setdefault("skipped", []).append(f"{nbytes / 1e9:.1f} GB field: MemAvailable too small")
            continue
        variants, moved, moved_by = build()
        times = {k: [] for k in variants}
        for fn in variants.values():  # warm-up: workspace, plans, allocator
            fn()
        for _ in range(args.rounds):
            for k, fn in variants.items():
                times[k].append(timed_call(fn))
        for k, ts in times.items():
            med = statistics.median(ts)
            result[k] = {"s": med, "min_s": min(ts), "GBps": moved_by.get(k, moved) / med / 1e9}
        del variants
    for name, ceiling in (("faces_scalar_diffX", "plain_diffX"), ("faces_vector_diffX", "plain_diffX"),
                          ("fold_diffY", "plain_fold_shape_diffY"), ("faces_cumsumX", "plain_cumsumX"),
                          ("faces_cumsumZ", "plain_cumsumZ"),
                          ("fold_cumsumY_reverse", "plain_fold_shape_cumsumY_reverse"),
                          ("faces_diffXY", "plain_diffXY"), ("fold_interpXY", "plain_fold_shape_interpXY")):
        if name in result and ceiling in result:
            result[name]["vs_plain"] = result[name]["s"] / result[ceiling]["s"]
        if name in result and name + "_old" in result:
            result[name]["vs_old"] = result[name]["s"] / result[name + "_old"]["s"]
    for name, single in (("faces_diffXY", "faces_scalar_diffX"), ("fold_interpXY", "fold_diffY")):
        if name in result and single in result:
            result[name]["vs_single_axis"] = result[name]["s"] / result[single]["s"]
    result["orca_year"] = {"skipped": "--skip-year"} if args.skip_year else orca_year(args.rounds)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
