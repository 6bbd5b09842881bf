"""Per-kernel timing on the C3 field (75, 2400, 3600) fp32: GB/s of algorithmic bytes.

Usage (on the GPU box): python tools/kernel_bench.py [--shape 75 2400 3600] [--dtype f32]
"""

import argparse
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xgcm_b200 import ops  # noqa: E402


def time_call(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for s, e in ev:
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    ts = sorted(s.elapsed_time(e) for s, e in ev)
    return ts[len(ts) // 2], ts[0]


def copy_stream_lib():
    """tools/micro/copy_stream.cu (16-byte ld.global.cs / st.global.cs copy) built into a temporary directory,
    keyed by the source hash, so the tree stays read-only."""
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "micro", "copy_stream.cu")
    tag = hashlib.sha256(open(src, "rb").read()).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), f"xgcm_b200_copy_stream_{tag}.so")
    if not os.path.exists(so):
        nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
        subprocess.run([nvcc, "-O3", "-shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-o", so + ".tmp", src], check=True)
        os.replace(so + ".tmp", so)
    lib = ctypes.CDLL(so)
    lib.copy_stream.restype = ctypes.c_int
    lib.copy_stream.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", type=int, nargs="+", default=[75, 2400, 3600])
    ap.add_argument("--dtype", default="f32")
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    dt = torch.float32 if args.dtype == "f32" else torch.float64
    es = 4 if args.dtype == "f32" else 8
    x = torch.rand(args.shape, dtype=dt, device="cuda")
    cells = x.numel()
    peak = None
    try:
        peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    y = torch.empty_like(x)
    med, best = time_call(lambda: y.copy_(x), args.iters)
    print(f"torch copy_            : {med:8.3f} ms  {2*cells*es/med/1e6:8.1f} GB/s (best {2*cells*es/best/1e6:.1f})")
    lib = copy_stream_lib()
    for bps in (4, 8):
        y.zero_()
        fn = lambda: lib.copy_stream(x.data_ptr(), y.data_ptr(), cells * es, bps, torch.cuda.current_stream().cuda_stream)
        med, best = time_call(fn, args.iters)
        assert torch.equal(x, y)
        print(f"ld/st.global.cs copy {bps}x: {med:8.3f} ms  {2*cells*es/med/1e6:8.1f} GB/s (best {2*cells*es/best/1e6:.1f})")
    names = "ZYX" if len(args.shape) == 3 else [str(i) for i in range(len(args.shape))]
    for axis in range(len(args.shape)):
        for op in ("diff", "interp"):
            for (lo, hi, bc) in ((1, 0, "periodic"), (0, 1, "fill"), (1, 0, "extend")):
                out = torch.empty_like(x)
                fn = lambda: ops.stencil2(x, axis, op, lo, hi, bc, 0.0, out=out)
                med, best = time_call(fn, args.iters)
                gbs = 2 * cells * es / med / 1e6
                frac = f" {gbs/peak:5.2f} of measured peak" if peak else ""
                print(f"{op:6s} axis={names[axis]} lo={lo} hi={hi} {bc:8s}: {med:8.3f} ms  {gbs:8.1f} GB/s{frac}  "
                      f"{cells/med/1e6:7.1f} Gcell/s")


if __name__ == "__main__":
    main()
