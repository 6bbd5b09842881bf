"""Conservative Grid.transform of numpy fields: the streamed host twin against today's whole-field route.

    python tools/bench_transform_host.py [--reps 5]

Input: page-locked fp32 phi (T, 75, 2400, 3600), theta bounds (T, 76, 2400, 3600), 61 bin edges; T = 2 when the
host has the memory (MemAvailable), else T = 1 (reported).  Routes, alternated --reps times, medians reported:

  a  ops.vinterp_conservative_host (slabs of phi and theta stream; upload || k_vconserv || download)
  b  upload phi and theta whole from the same page-locked arrays, ops.vinterp_conservative, download
  c  theta at cell centres (T, 75, 2400, 3600): fused (theta_at_centers) against grid.interp(extend) + the twin

Seconds and GB/s of bytes in + out per route, beside the PCIe ceiling of tools/bench_pcie.py run in the same
command, with the card name and power limit.  The routes' outputs are compared bit for bit.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import xgcm_b200 as xg  # noqa: E402
from xgcm_b200 import ops  # noqa: E402

NZ, NY, NX, M = 75, 2400, 3600, 61


def _mem_available():
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as exc:  # the numbers stay valid; the label is missing
        return torch.cuda.get_device_name(0), f"unknown ({exc!r})"


def _pcie():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_pcie.py")], capture_output=True, text=True,
                       timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    return json.loads(lines[-1]) if lines else {"error": r.stderr[-500:]}


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    card, power = _card()
    pcie = _pcie()  # before the big host buffers exist

    per_t = 4 * NY * NX * (NZ + (NZ + 1) + NZ + 4 * (M - 1))  # phi, bounds, centres, four results
    avail = _mem_available()
    T = 2 if avail > 2 * per_t * 1.3 else 1
    note = None if T == 2 else f"T = 1: MemAvailable {avail / 1e9:.1f} GB is short of what T = 2 needs"

    phi = ops.pinned_empty((T, NZ, NY, NX), np.float32)
    th = ops.pinned_empty((T, NZ + 1, NY, NX), np.float32)
    tc = ops.pinned_empty((T, NZ, NY, NX), np.float32)
    ops.fill_uniform_host(phi, seed=1)
    ops.fill_uniform_host(th, seed=2)
    ops.fill_uniform_host(tc, seed=3)
    th += np.arange(NZ + 1, dtype=np.float32)[None, :, None, None]  # increasing bounds, one unit per level
    tc += np.arange(NZ, dtype=np.float32)[None, :, None, None]
    bins = np.linspace(-1.0, NZ + 1.0, M).astype(np.float32)

    grid = xg.Grid(xg.Dataset(coords={"z": np.arange(NZ) + 0.5, "zo": np.arange(NZ + 1.0)}),
                   coords={"Z": {"center": "z", "outer": "zo"}})
    tc_da = xg.DataArray(tc, dims=("t", "z", "y", "x"))

    def route_a():
        return ops.vinterp_conservative_host(phi, th, bins, 1)

    def route_b():
        d_phi = torch.from_numpy(phi).cuda(non_blocking=True)
        d_th = torch.from_numpy(th).cuda(non_blocking=True)
        d_bins = torch.from_numpy(bins).cuda()
        out = ops.vinterp_conservative(d_phi, d_th, d_bins, 1)
        host = ops.pinned_empty(out.shape, np.float32)
        torch.from_numpy(host).copy_(out)
        return host

    def route_c_fused():
        return ops.vinterp_conservative_host(phi, tc, bins, 1, theta_at_centers=True)

    def route_c_interp():
        bounds = grid.interp(tc_da, "Z", padding="extend")
        return ops.vinterp_conservative_host(phi, bounds.values, bins, 1)

    routes = {"a_twin": route_a, "b_whole_field": route_b, "c_centres_fused": route_c_fused,
              "c_interp_then_twin": route_c_interp}
    bytes_io = {
        "a_twin": phi.nbytes + th.nbytes,
        "b_whole_field": phi.nbytes + th.nbytes,
        "c_centres_fused": phi.nbytes + tc.nbytes,
        "c_interp_then_twin": phi.nbytes + tc.nbytes,  # what the user hands in; the bounds' round trip is the cost
    }
    out_bytes = T * NY * NX * (M - 1) * 4
    for fn in routes.values():  # warm-up: workspaces, allocator, kernel attributes
        fn()
    times = {k: [] for k in routes}
    last = {}
    for _ in range(args.reps):
        for k, fn in routes.items():
            dt, out = _timed(fn)
            times[k].append(dt)
            last[k] = out
    med = {k: float(np.median(v)) for k, v in times.items()}
    res = {
        "card": card, "power_limit": power, "T": T, "note": note,
        "shape_phi": [T, NZ, NY, NX], "bins": M, "dtype": "float32", "reps": args.reps,
        "seconds_median": med,
        "GBps_in_plus_out": {k: (bytes_io[k] + out_bytes) / med[k] / 1e9 for k in routes},
        "pcie_ceiling": pcie,
        "bit_identical": {
            "a_vs_b": bool(np.array_equal(last["a_twin"].view(np.uint32), last["b_whole_field"].view(np.uint32))),
            "c_fused_vs_interp": bool(np.array_equal(last["c_centres_fused"].view(np.uint32),
                                                     last["c_interp_then_twin"].view(np.uint32))),
        },
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
