"""Build recipe for the C-ABI shared library (nvcc, sm_90a only, in-tree).

``python -m xgcm_b200._build`` or ``__graft_entry__.build()``.  The library
links only against the (static) CUDA runtime: no torch, no python.
"""

from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
import warnings
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
INCLUDE = PKG_DIR.parent / "include"
BUILD_DIR = PKG_DIR / "csrc" / "build"
LIB_PATH = PKG_DIR / "libxgcm_b200.so"

ARCH = "arch=compute_90a,code=sm_90a"  # H100 (Hopper)

NVCC_FLAGS = [
    "-gencode",
    ARCH,
    "-lineinfo",
    "-O3",
    "-std=c++17",
    # numpy rounds after every ufunc: no FMA contraction, IEEE div/sqrt
    "--fmad=false",
    "--prec-div=true",
    "--prec-sqrt=true",
    "--ftz=false",
    "-Xcompiler",
    "-fPIC",
    "-Xcompiler",
    "-fvisibility=hidden",
    "-DXG_BUILDING",
]


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; cannot build libxgcm_b200.so")
    return nvcc


def sources():
    return sorted(CSRC.glob("*.cu"))


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _compile_one(src: Path, verbose: bool) -> Path:
    obj = BUILD_DIR / (src.stem + ".o")
    cmd = [_nvcc(), *NVCC_FLAGS, "-I", str(INCLUDE), "-I", str(CSRC), "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{res.stdout}\n{res.stderr}")
    if verbose:
        sys.stderr.write(res.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every ``csrc/*.cu`` for sm_90a and link ``libxgcm_b200.so``."""
    srcs = sources()
    stamp = BUILD_DIR / "digest.txt"
    digest = current_digest()
    if not force and LIB_PATH.exists() and stamp.exists() and stamp.read_text() == digest:
        if not (BUILD_DIR / "kernels.txt").exists():
            try:
                write_manifest(digest)
            except (OSError, RuntimeError, subprocess.CalledProcessError) as err:
                # the library itself is current; only the kernel list for the tests is missing
                warnings.warn(f"kernels.txt not written (needs cuobjdump and c++filt): {err}")
        return LIB_PATH
    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile_one(s, verbose), srcs))
    cmd = [
        _nvcc(),
        "-shared",
        "-gencode",
        ARCH,
        "-o",
        str(LIB_PATH),
        *[str(o) for o in objs],
        "-cudart",
        "static",
    ]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    write_manifest(digest)
    stamp.write_text(digest)
    return LIB_PATH


def kernel_entries(lib: Path = LIB_PATH):
    """``[(source stem, demangled name)]`` of every ``__global__`` instance linked into ``lib``: the
    STO_ENTRY symbols of ``cuobjdump -symbols``, demangled by ``c++filt`` into the names the CUDA
    profiler (kineto) reports."""
    cuobjdump = Path(_nvcc()).with_name("cuobjdump")
    res = subprocess.run([str(cuobjdump), "-symbols", str(lib)], capture_output=True, text=True, check=True)
    stems, mangled = [], []
    stem = "?"
    for line in res.stdout.splitlines():
        if line.startswith("identifier = "):
            stem = Path(line.split("=", 1)[1].strip()).stem
        elif "STO_ENTRY" in line:
            stems.append(stem)
            mangled.append(line.split()[-1])
    res = subprocess.run(["c++filt"], input="\n".join(mangled) + "\n", capture_output=True, text=True, check=True)
    names = res.stdout.splitlines()
    if len(names) != len(mangled):
        raise RuntimeError("c++filt returned a different number of names than it was given")
    return sorted(zip(stems, names))


def write_manifest(digest: str) -> Path:
    """``BUILD_DIR/kernels.txt``: the build digest on the first line, then one ``stem<TAB>name`` line per
    kernel instance.  The GPU tests compare it with the kernels the profiler saw launch."""
    lines = [f"# digest {digest}"] + [f"{s}\t{n}" for s, n in kernel_entries()]
    path = BUILD_DIR / "kernels.txt"
    path.write_text("\n".join(lines) + "\n")
    return path


def read_manifest(path: Path = BUILD_DIR / "kernels.txt"):
    """``(digest, [(stem, name)])`` of a manifest written by :func:`write_manifest`."""
    lines = path.read_text().splitlines()
    if not lines or not lines[0].startswith("# digest "):
        raise ValueError(f"{path}: no digest line")
    entries = []
    for ln in lines[1:]:
        stem, sep, name = ln.partition("\t")
        if not sep or not name.startswith("void "):
            raise ValueError(f"{path}: malformed entry {ln!r}")
        entries.append((stem, name))
    return lines[0][len("# digest "):], entries


def current_digest() -> str:
    """Digest of the sources and flags the library is built from (what ``digest.txt`` holds after a build)."""
    return _digest(sources() + sorted(CSRC.glob("*.cuh")) + sorted(INCLUDE.glob("*.h")))


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
