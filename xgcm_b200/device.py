"""Device residency helpers (torch = allocator / stream owner only).

Host arrays handed to a Grid method are copied to the GPU, processed by the
CUDA kernels and copied back; CUDA tensors stay resident.  There is no CPU
compute path: without a CUDA device these helpers raise.
"""

from __future__ import annotations

from typing import Sequence, Tuple

import numpy as np
import torch

_FLOAT = (np.dtype("float32"), np.dtype("float64"))
_SMALL_BYTES = 64 * 1024
_small_cache: dict = {}


def default_device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError(
            "xgcm_b200 needs a CUDA device: the stencil engine has no CPU fallback"
        )
    return torch.device("cuda", torch.cuda.current_device())


def as_device_tensor(data, device=None) -> Tuple[torch.Tensor, bool]:
    """Return ``(contiguous CUDA tensor, was_host)``.

    Integer / bool fields are promoted to float64 (the kernels are fp32/fp64).
    """
    if isinstance(data, torch.Tensor):
        if not data.is_cuda:
            raise RuntimeError("CPU torch tensors are not supported; pass numpy arrays or CUDA tensors")
        t = data
        if t.dtype not in (torch.float32, torch.float64):
            t = t.to(torch.float64)
        return t.contiguous(), False
    arr = np.asarray(data)
    if arr.dtype not in _FLOAT:
        arr = arr.astype(np.float64)
    if not arr.flags.c_contiguous:
        arr = np.ascontiguousarray(arr)
    if not arr.flags.writeable:
        arr = arr.copy()
    dev = device if device is not None else default_device()
    return torch.from_numpy(arr).to(dev, non_blocking=True), True


def as_device_constant(data, device=None) -> torch.Tensor:
    """Device copy of a SMALL read-only host operand (coordinate vector, target levels, 1-D metric), uploaded once
    per content.  A pageable upload blocks the host until the copy has drained behind whatever kernel is running
    — for a 1 ms kernel that serialises consecutive calls — so identical small operands are re-used.  The returned
    tensor is shared: callers must never write to it (fields go through :func:`as_device_tensor`)."""
    if isinstance(data, torch.Tensor):
        return as_device_tensor(data, device)[0]
    arr = np.asarray(data)
    if arr.dtype not in _FLOAT:
        arr = arr.astype(np.float64)
    if not arr.flags.c_contiguous:
        arr = np.ascontiguousarray(arr)
    if arr.nbytes > _SMALL_BYTES:
        return as_device_tensor(arr, device)[0]
    dev = device if device is not None else default_device()
    key = (arr.dtype.str, arr.shape, str(dev), hash(arr.tobytes()))
    hit = _small_cache.get(key)
    if hit is None:
        if len(_small_cache) >= 256:
            _small_cache.clear()
        hit = torch.from_numpy(arr.copy()).to(dev)
        _small_cache[key] = hit
    return hit


_host_groups: dict = {}


def host_group(devices: Sequence[int]) -> int:
    """Handle of the host device group ``devices`` (``xg_host_group``), cached per member list.

    Passed as the ``device`` of an ``ops.*_host`` call, it spreads the call's slabs over the members: the result
    rows are cut into one contiguous block per member, and each member streams its block through its own PCIe
    link.  A member may repeat; its blocks then take turns on that GPU."""
    key = tuple(int(d) for d in devices)
    hit = _host_groups.get(key)
    if hit is None:
        import ctypes as C

        from . import _capi

        handle = C.c_int(0)
        _capi.check(_capi.load().xg_host_group(len(key), (C.c_int * max(len(key), 1))(*key), C.byref(handle)))
        hit = _host_groups[key] = handle.value
    return hit


def host_device_arg(device) -> int:
    """The ``int device`` argument of a ``*_host`` entry point: the current CUDA device for None, an index, or the
    handle of the group a sequence of indices names."""
    if device is None:
        return torch.cuda.current_device()
    if isinstance(device, (int, np.integer)):
        return int(device)
    return host_group(device)


def result_like(t: torch.Tensor, was_host: bool):
    """Give the result the residency of the input: numpy for host inputs."""
    if was_host:
        host = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)  # torch's caching host allocator
        host.copy_(t)
        return host.numpy()
    return t


# --------------------------------------------------------------------------- NUMA placement of the host side
def _parse_cpulist(text: str):
    cpus = set()
    for part in text.strip().split(","):
        if not part:
            continue
        if "-" in part:
            a, b = part.split("-")
            cpus.update(range(int(a), int(b) + 1))
        else:
            cpus.add(int(part))
    return cpus


def gpu_numa_node(index: int | None = None) -> int:
    """NUMA node the GPU hangs off (sysfs), or -1 when the platform does not say."""
    idx = torch.cuda.current_device() if index is None else int(index)
    p = torch.cuda.get_device_properties(idx)
    try:
        bdf = f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
        with open(f"/sys/bus/pci/devices/{bdf}/numa_node") as f:
            return int(f.read().strip())
    except Exception:
        return -1


def bind_to_gpu_numa(index: int | None = None) -> dict:
    """Pin the calling thread (and the memory it touches from now on) to the NUMA node of GPU ``index``.

    Host-streamed calls are bound by host-memory / root-complex bandwidth once several GPUs share a socket:
    page-locked buffers should live on the socket their GPU is attached to.  Call this BEFORE allocating
    pinned buffers (``ops.pinned_empty``) — one process per GPU, as torchrun launches them.  Returns what was
    done (for logs); never raises."""
    import ctypes
    import os
    import platform

    info = {"gpu": torch.cuda.current_device() if index is None else int(index), "numa_node": -1,
            "cpus_bound": 0, "mempolicy": None}
    try:
        node = gpu_numa_node(index)
        info["numa_node"] = node
        if node < 0:
            info["note"] = "sysfs reports no NUMA node for this GPU"
            return info
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            cpus = _parse_cpulist(f.read())
        allowed = os.sched_getaffinity(0)
        use = cpus & allowed
        if use:
            os.sched_setaffinity(0, use)
            info["cpus_bound"] = len(use)
        else:
            info["note"] = "node cpus not in this process's cpuset"
        # set_mempolicy(MPOL_PREFERRED, {node}): page-locked allocations after this land on the GPU's socket
        nr = {"x86_64": 238, "aarch64": 237}.get(platform.machine())
        if nr is not None:
            nbits = 1024
            mask = (ctypes.c_ulong * (nbits // (8 * ctypes.sizeof(ctypes.c_ulong))))()
            mask[node // (8 * ctypes.sizeof(ctypes.c_ulong))] |= 1 << (node % (8 * ctypes.sizeof(ctypes.c_ulong)))
            libc = ctypes.CDLL(None, use_errno=True)
            rc = libc.syscall(nr, 1, ctypes.byref(mask), nbits + 1)  # MPOL_PREFERRED = 1
            info["mempolicy"] = "preferred" if rc == 0 else f"failed (errno {ctypes.get_errno()})"
    except Exception as exc:  # placement is an optimisation, never an error
        info["note"] = repr(exc)
    return info
