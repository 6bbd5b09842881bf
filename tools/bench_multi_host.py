"""Multi-axis Grid calls on numpy fields: the streamed host twins against the whole-field route.

    python tools/bench_multi_host.py [--reps 5]

Page-locked fp32 C3 fields (75, 2400, 3600) on a grid with X periodic, Y fill, Z extend.  Cases, each timed as

  streamed  the Grid call on the numpy field (xg_stencil_multi_host / xg_wreduce_host_multi: upload || kernel ||
            download, slab by slab)
  whole     upload the field (and the weight) whole from the same page-locked arrays, the Grid call on the device
            field, download the result

  interp_xyz  grid.interp(theta, ["X", "Y", "Z"], to="left")
  interp_xy   grid.interp(theta, ["X", "Y"], to="left") of a (T, 75, 2400, 3600) field, T = 4 when the host has the
              memory (MemAvailable), else less (reported)
  average_xyz grid.average(theta, ["X", "Y", "Z"]) with a (75, 2400, 3600) volume weight, one registered metric

Routes alternated --reps times, medians reported, in seconds and GB/s of bytes in + out, beside the PCIe ceiling of
tools/bench_pcie.py run in the same command, with the card name and power limit.  Each case's two routes are compared
bit for bit.  Prints one JSON line.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import xgcm_b200 as xg  # noqa: E402
from bench_transform_host import _card, _mem_available, _pcie, _timed  # noqa: E402
from xgcm_b200 import ops  # noqa: E402

NZ, NY, NX = 75, 2400, 3600
DIMS = ("z", "y", "x")


def _grid(vol=None):
    ds = xg.Dataset(data_vars={} if vol is None else {"vol": (DIMS, vol)},
                    coords={"z": np.arange(NZ) + 0.5, "zl": np.arange(NZ) + 0.0, "y": np.arange(NY) + 0.5,
                            "yl": np.arange(NY) + 0.0, "x": np.arange(NX) + 0.5, "xl": np.arange(NX) + 0.0})
    return xg.Grid(ds, coords={"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"},
                               "Z": {"center": "z", "left": "zl"}},
                   padding={"X": "periodic", "Y": "fill", "Z": "extend"}, fill_value=0.0,
                   metrics=None if vol is None else {("X", "Y", "Z"): ["vol"]}, autoparse_metadata=False)


def _download(res):
    host = ops.pinned_empty(tuple(res.data.shape), np.float32)
    torch.from_numpy(host).copy_(res.data)
    return host


def _run(routes, reps):
    for fn in routes.values():  # warm-up: workspace, allocator, kernel attributes
        fn()
    times = {k: [] for k in routes}
    last = {}
    for _ in range(reps):
        for k, fn in routes.items():
            last[k] = None  # the previous result's host memory can serve this one
            dt, last[k] = _timed(fn)
            times[k].append(dt)
    med = {k: float(np.median(v)) for k, v in times.items()}
    same = bool(np.array_equal(*[np.asarray(v).view(np.uint32) for v in last.values()]))
    return med, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    card, power = _card()
    pcie = _pcie()  # before the big host buffers exist
    field = NZ * NY * NX * 4
    res = {"card": card, "power_limit": power, "dtype": "float32", "reps": args.reps, "shape": [NZ, NY, NX],
           "slab_mb": os.environ.get("XG_HOST_SLAB_MB", "128 (default)"), "pcie_ceiling": pcie, "cases": {}}

    def record(name, med, same, bytes_io):
        res["cases"][name] = {"seconds_median": med, "GBps_in_plus_out": {k: bytes_io / v / 1e9 for k, v in med.items()},
                              "bit_identical": same}

    # interp_xyz and average_xyz on one C3 field and its volume weight
    theta = ops.pinned_empty((NZ, NY, NX), np.float32)
    vol = ops.pinned_empty((NZ, NY, NX), np.float32)
    ops.fill_uniform_host(theta, seed=1)
    ops.fill_uniform_host(vol, seed=2)
    vol += 0.5
    grid = _grid()
    da = xg.DataArray(theta, dims=DIMS)

    def whole_interp(g, a, axes):
        d = torch.from_numpy(a).cuda(non_blocking=True)
        return _download(g.interp(xg.DataArray(d, dims=("t",) * (a.ndim - 3) + DIMS), axes, to="left"))

    med, same = _run({"streamed": lambda: grid.interp(da, ["X", "Y", "Z"], to="left").data,
                      "whole": lambda: whole_interp(grid, theta, ["X", "Y", "Z"])}, args.reps)
    record("interp_xyz", med, same, 2 * field)

    wgrid = _grid(vol)

    def whole_average():
        g = _grid(vol)  # a new grid: its metric cache does not keep the weight on the device between calls
        d = torch.from_numpy(theta).cuda(non_blocking=True)
        return g.average(xg.DataArray(d, dims=DIMS), ["X", "Y", "Z"]).data.cpu().numpy()

    med, same = _run({"streamed": lambda: np.asarray(wgrid.average(da, ["X", "Y", "Z"]).data),
                      "whole": whole_average}, args.reps)
    record("average_xyz", med, same, 2 * field)
    del theta, vol, da, wgrid

    # interp_xy of a (T, Z, Y, X) field: input, and the results of both routes alive at once
    avail = _mem_available()
    T = 4
    while T > 1 and 3 * T * field * 1.3 > avail:
        T -= 1
    res["interp_xy_T"] = T
    if T < 4:
        res["note"] = f"interp_xy with T = {T}: MemAvailable {avail / 1e9:.1f} GB is short of what T = 4 needs"
    theta4 = ops.pinned_empty((T, NZ, NY, NX), np.float32)
    ops.fill_uniform_host(theta4, seed=3)
    da4 = xg.DataArray(theta4, dims=("t",) + DIMS)
    med, same = _run({"streamed": lambda: grid.interp(da4, ["X", "Y"], to="left").data,
                      "whole": lambda: whole_interp(grid, theta4, ["X", "Y"])}, args.reps)
    record("interp_xy", med, same, 2 * T * field)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
