"""Pinned host memory placed on the NUMA node next to the GPU.

The streaming path (dca_stream_*) copies every batch host->device over PCIe.  On a two-socket host a
pinned buffer whose pages sit on the far socket crosses the socket interconnect on every copy, so pinned
buffers are allocated while the calling thread is restricted to the CPUs NVML reports as local to the GPU;
the previous affinity is restored afterwards (pages stay where they were pinned).  Best effort: the gain
is host-dependent and has not been measured on H100 hosts.
No reference counterpart (the reference never leaves the host).
"""
from __future__ import annotations

import contextlib
import os

import numpy as np
import torch


def gpu_local_cpus(device_index: int):
    """CPUs local to CUDA device `device_index` (set of ints) or None when it cannot be determined."""
    try:
        p = torch.cuda.get_device_properties(device_index)
        bus = "%08x:%02x:%02x.0" % (p.pci_domain_id, p.pci_bus_id, p.pci_device_id)
    except Exception:
        return None
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByPciBusId(bus.encode())
        ncpu = os.cpu_count() or 1
        words = pynvml.nvmlDeviceGetCpuAffinity(h, (ncpu + 63) // 64)
        cpus = {64 * w + b for w, m in enumerate(words) for b in range(64) if (int(m) >> b) & 1}
        if cpus:
            return cpus
    except Exception:
        pass
    try:
        with open("/sys/bus/pci/devices/%s/local_cpulist" % bus[4:]) as f:      # sysfs uses a 4-digit domain
            cpus = set()
            for part in f.read().strip().split(","):
                lo, _, hi = part.partition("-")
                cpus.update(range(int(lo), int(hi or lo) + 1))
            return cpus or None
    except Exception:
        return None


@contextlib.contextmanager
def near_gpu(device_index: int):
    """Restrict the calling thread to the GPU-local CPUs for the duration of the block (best effort)."""
    prev = None
    try:
        cpus = gpu_local_cpus(device_index)
        if cpus and hasattr(os, "sched_getaffinity"):
            cur = os.sched_getaffinity(0)
            want = cur & cpus
            if want and want != cur:
                os.sched_setaffinity(0, want)
                prev = cur
    except Exception:
        prev = None
    try:
        yield
    finally:
        if prev is not None:
            try:
                os.sched_setaffinity(0, prev)
            except Exception:
                pass


def pin_near_gpu(a, device_index: int = 0) -> torch.Tensor:
    """Pinned host copy of a numpy array / host tensor, pages on the GPU's NUMA node (plain tensor without CUDA)."""
    t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    if not torch.cuda.is_available():
        return t
    with near_gpu(device_index):
        out = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
        out.copy_(t)
    return out
