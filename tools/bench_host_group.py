"""Grid calls on numpy fields spread over host device groups, against the single-device call.

    python tools/bench_host_group.py [--reps 3] [--T T]

Page-locked fp32 (T, 75, 2400, 3600) fields, T >= the largest group (default: that size, at least 1), on a grid with
X periodic, Y fill, Z extend.  Calls:

  e2e         Grid.apply_many: diff + interp along X, Y and Z (six results), once per time step -- apply_many cuts
              dim 0 into slabs, so each (75, 2400, 3600) step is one call whose Z rows the group's members share
  divergence  Grid.divergence(u, v) of (T, 75, 2400, 3600) fields, the (T * 75) leading rows shared
  transform   Grid.transform(theta, "Z", 100 levels, method="linear") with theta a (T, 75, 2400, 3600) field

Routes: the grid without host_devices (one GPU), and Grid(host_devices=(0, .., k - 1)) for k = 1, 2, 4, 8 as far as
GPUs are visible, alternated --reps times; medians in seconds and in host bytes moved per second (in + out), beside
the ceiling of tools/bench_pcie.py taken in the same run, with the card name and power limit.  Every group's results
are compared bit for bit with the single-device call of the same round.  Prints one JSON line.
"""
import argparse
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import xgcm_b200 as xg  # noqa: E402
from bench_transform_host import _card, _mem_available, _pcie, _timed  # noqa: E402
from xgcm_b200 import ops  # noqa: E402

NZ, NY, NX = 75, 2400, 3600
DIMS = ("t", "z", "y", "x")
LEVELS = 100


def _grid(host_devices, metrics):
    ds = xg.Dataset(data_vars=metrics,
                    coords={"z": np.arange(NZ) + 0.5, "zl": np.arange(NZ) + 0.0, "y": np.arange(NY) + 0.5,
                            "yl": np.arange(NY) + 0.0, "x": np.arange(NX) + 0.5, "xl": np.arange(NX) + 0.0})
    return xg.Grid(ds, coords={"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"},
                               "Z": {"center": "z", "left": "zl"}},
                   padding={"X": "periodic", "Y": "fill", "Z": "extend"}, fill_value=0.0, autoparse_metadata=False,
                   metrics={("X",): ["dx"], ("Y",): ["dy"], ("X", "Y"): ["area"]}, host_devices=host_devices)


def _field(T, seed):
    a = ops.pinned_empty((T, NZ, NY, NX), np.float32)
    ops.fill_uniform_host(a, seed=seed)
    return a


def _equal(a, b):
    return all(np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32)) for x, y in zip(a, b))


def _run(calls, routes, reps):
    """calls(grid) -> list of numpy results; per rep every route once, in order; medians and bit-identity."""
    for g in routes.values():  # warm-up: workspaces, threads' contexts, allocators
        calls(g)
    times = {k: [] for k in routes}
    same = {k: True for k in routes if k != "single"}
    for _ in range(reps):
        ref = None
        for k, g in routes.items():
            dt, out = _timed(lambda: calls(g))
            times[k].append(dt)
            if k == "single":
                ref = out
            else:
                same[k] = same[k] and _equal(ref, out)
            del out
        del ref
    return {k: float(np.median(v)) for k, v in times.items()}, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--T", type=int, default=0)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    n_gpu = torch.cuda.device_count()
    sizes = [k for k in (1, 2, 4, 8) if k <= n_gpu]
    T = max(args.T, sizes[-1])
    card, power = _card()
    pcie = _pcie()  # before the big host buffers exist
    field = NZ * NY * NX * 4
    res = {"card": card, "power_limit": power, "gpus_visible": n_gpu, "dtype": "float32", "reps": args.reps,
           "shape": [T, NZ, NY, NX], "slab_mb": os.environ.get("XG_HOST_SLAB_MB", "128 (default)"),
           "pcie_ceiling": pcie, "mem_available_gb": _mem_available() / 1e9, "cases": {}}
    for k in (2, 4, 8):
        if k not in sizes:
            res.setdefault("not_measured", []).append(f"group of {k}: {n_gpu} GPU(s) visible")
    rng = np.random.default_rng(0)
    metrics = {"dx": (("yl", "x"), (0.5 + rng.random((NY, NX))).astype(np.float32)),
               "dy": (("y", "xl"), (0.5 + rng.random((NY, NX))).astype(np.float32)),
               "area": (("y", "x"), (0.5 + rng.random((NY, NX))).astype(np.float32))}
    routes = {"single": _grid(None, metrics)}
    routes.update({f"group{k}": _grid(tuple(range(k)), metrics) for k in sizes})

    def record(name, med, same, bytes_io):
        res["cases"][name] = {"seconds_median": med, "host_GBps_in_plus_out": {k: bytes_io / v / 1e9
                                                                               for k, v in med.items()},
                              "speedup_vs_single": {k: med["single"] / v for k, v in med.items()},
                              "bit_identical_to_single": same}

    # e2e: apply_many per time step
    phi = _field(T, 1)
    reqs = [(f, a) for a in ("X", "Y", "Z") for f in ("diff", "interp")]
    steps = [xg.DataArray(phi[t], dims=DIMS[1:]) for t in range(T)]
    med, same = _run(lambda g: [r.data for s in steps for r in g.apply_many(s, reqs)], routes, args.reps)
    record("e2e_apply_many", med, same, 7 * T * field)
    del steps

    # divergence of (u, v) on the C grid: u at (center, left), v at (left, center)
    v = _field(T, 2)
    du = xg.DataArray(phi, dims=("t", "z", "y", "xl"))
    dv = xg.DataArray(v, dims=("t", "z", "yl", "x"))
    to = {"X": "center", "Y": "center"}
    med, same = _run(lambda g: [g.divergence(du, dv, to=to).data], routes, args.reps)
    record("divergence", med, same, 3 * T * field)
    del v, du, dv

    # linear transform to 100 levels of a monotonic theta field
    theta = _field(T, 3)
    theta += np.arange(NZ, dtype=np.float32)[None, :, None, None]
    levels = np.linspace(0.5, NZ - 0.5, LEVELS).astype(np.float32)
    da, dth = xg.DataArray(phi, dims=DIMS), xg.DataArray(theta, dims=DIMS)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        med, same = _run(lambda g: [g.transform(da, "Z", levels, target_data=dth, method="linear").data], routes,
                         args.reps)
    record("transform_linear_100", med, same, 2 * T * field + T * field * LEVELS // NZ)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
