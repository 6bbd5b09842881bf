"""Metric-weighted Grid.interp along X across face connections at an LLC-like size: a (50, 13, 540, 540) fp32 field
(k, face, j, i) on 13 faces joined in a ring along X, with a (face, j, i) metric.  Times, alternated in one process:

  fused    grid.interp(x, "X", metric_weighted="X") on a device tensor: halo planes of x * dx, one xg_stencil2
  composed the route it replaces, spelled out: ops.binary (x * dx) -> padding.pad -> ops.stencil2 (/ dx_l)

and checks that the two agree bit for bit.  Then the same call on a numpy field of that shape with a leading time
dim (`--host-time`) in page-locked memory, streamed in slabs (xg_stencil2_host_connected_weighted), against the
page-locked copy time of the same bytes (the measurement of tools/bench_pcie.py: the field up and the result down at
once).  Prints one JSON line, with the card name and power limit.

Usage (on the GPU box): python tools/bench_faces_weighted.py [--shape 50 13 540 540] [--rounds 5] [--host-time 2]
"""

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import xgcm_b200 as xg  # noqa: E402
from xgcm_b200 import ops  # noqa: E402
from xgcm_b200.padding import pad  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return out or None
    except Exception:
        return None


def ring(nf):
    """nf faces in a ring along X (their Y edges unconnected)."""
    links = {}
    for i in range(nf):
        left, right = (i - 1) % nf, (i + 1) % nf
        links.setdefault(i, {})["X"] = ((left, "X", False), (right, "X", False))
    return {"face": links}


def timed_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", type=int, nargs=4, default=[50, 13, 540, 540])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host-time", type=int, default=2)
    args = ap.parse_args()
    nz, nf, ny, nx = args.shape
    rng = np.random.default_rng(0)
    coords = {"i": np.arange(nx) + 0.5, "i_g": np.arange(nx) + 0.0, "j": np.arange(ny) + 0.5, "face": np.arange(nf)}
    ds = xg.Dataset(data_vars={"dxC": (("face", "j", "i"), (0.5 + rng.random((nf, ny, nx))).astype(np.float32)),
                               "dxG": (("face", "j", "i_g"), (0.5 + rng.random((nf, ny, nx))).astype(np.float32))},
                    coords=coords)
    fc = ring(nf)
    grid = xg.Grid(ds, coords={"X": {"center": "i", "left": "i_g"}, "Y": {"center": "j"}}, face_connections=fc,
                   metrics={("X",): ["dxC", "dxG"]}, padding="fill", autoparse_metadata=False)
    x = torch.empty((nz, nf, ny, nx), dtype=torch.float32, device="cuda:0")
    ops.fill_uniform(x, 0xFACE)
    da = xg.DataArray(x, dims=("k", "face", "j", "i"))
    dims = da.dims
    pre = grid._metric_tensor(ds["dxC"], dims, x)
    post = grid._metric_tensor(ds["dxG"], ("k", "face", "j", "i_g"), x)

    def fused():
        return grid.interp(da, "X", metric_weighted="X").data

    def composed():
        w = xg.DataArray(ops.binary("mul", x, pre), dims=dims)
        p = pad(w, grid=grid, padding_width={"X": (1, 0)}, padding="fill").data
        return ops.stencil2(p, 3, "interp", 0, 0, None, post=post)

    same = bool(torch.equal(fused(), composed()))
    t_fused, t_composed = [], []
    for _ in range(args.rounds):
        t_fused.append(timed_ms(fused))
        t_composed.append(timed_ms(composed))
    field_bytes = x.numel() * 4
    fused_ms, composed_ms = statistics.median(t_fused), statistics.median(t_composed)

    # numpy field (time, k, face, j, i) in page-locked memory, streamed in slabs
    hshape = (args.host_time, nz, nf, ny, nx)
    host = ops.pinned_empty(hshape, np.float32)
    host[...] = x.cpu().numpy()[None]
    hda = xg.DataArray(host, dims=("time",) + dims)
    grid.interp(hda, "X", metric_weighted="X")  # warm-up: workspace and plan
    t_host = []
    for _ in range(max(2, args.rounds // 2)):
        t_host.append(timed_ms(lambda: grid.interp(hda, "X", metric_weighted="X")))
    host_ms = statistics.median(t_host)
    # the copy rate of the same bytes: the field up and the result down at once, page-locked (tools/bench_pcie.py)
    out_h = ops.pinned_empty(hshape, np.float32)
    up_d = torch.empty(hshape, dtype=torch.float32, device="cuda:0")
    dn_d = torch.zeros(hshape, dtype=torch.float32, device="cuda:0")
    up_h, dn_h = torch.from_numpy(host), torch.from_numpy(out_h)
    s_up, s_dn = torch.cuda.Stream(), torch.cuda.Stream()

    def copies():
        with torch.cuda.stream(s_up):
            up_d.copy_(up_h, non_blocking=True)
        with torch.cuda.stream(s_dn):
            dn_h.copy_(dn_d, non_blocking=True)
        s_up.synchronize()
        s_dn.synchronize()

    copies()
    copy_ms = statistics.median([timed_ms(copies) for _ in range(3)])
    host_bytes = host.nbytes
    print(json.dumps({
        "card": card(),
        "shape": [nz, nf, ny, nx],
        "device_fused_ms": round(fused_ms, 3),
        "device_composed_ms": round(composed_ms, 3),
        "device_speedup": round(composed_ms / fused_ms, 3),
        "device_fused_GBps": round(2 * field_bytes / fused_ms / 1e6, 1),
        "bitwise_equal": same,
        "host_shape": list(hshape),
        "host_ms": round(host_ms, 3),
        "host_copy_ms": round(copy_ms, 3),
        "host_vs_copy": round(copy_ms / host_ms, 3),
        "host_GBps_each_way": round(host_bytes / host_ms / 1e6, 1),
        "note": "fused vs composed alternated; host_vs_copy = page-locked copy time / streamed call time",
    }))


if __name__ == "__main__":
    main()
