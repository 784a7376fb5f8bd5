"""Preprocessing on the host (io.normalize) against the device (device_data.DeviceDataset), one JSON line per size.

    python tests/diag_preprocess.py [--sizes 8192x20000,68000x20000] [--epochs 5] [--batch 4096] [--reps 5]

Per size: host io.normalize wall time; device upload / totals / moments / write times by CUDA events (median of
--reps after a warm-up) with each kernel's bytes over its time against the data-sheet 3.35 TB/s of the H100 SXM;
dca(..., epochs, batch_size) wall time with training_kwds preprocess 'host' against 'device'; the card's name and power
limit, read in the same run.  Counts are seeded synthetic Poisson counts generated in row chunks.  Needs a GPU.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12


def synth_poisson(n, g, seed=0, chunk=4096):
    rng = np.random.default_rng(seed)
    gene_mean = np.exp(rng.normal(-1.2, 1.3, size=g)).astype(np.float64)
    Y = np.empty((n, g), np.float32)
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        depth = np.exp(rng.normal(0, 0.3, size=(e - s, 1)))
        Y[s:e] = rng.poisson(depth * gene_mean[None, :])
    Y[Y.sum(1) == 0, 0] = 1
    Y[0, Y.sum(0) == 0] = 1
    return Y


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as e:                                   # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown (%s)" % e


def time_events(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def measure(n, g, epochs, batch, reps):
    from dca_b200 import io, _lib
    from dca_b200.anndata_lite import AnnData
    from dca_b200.api import dca
    from dca_b200.device_data import DeviceDataset, _upload_dense
    lib = _lib.load()
    dev = torch.device("cuda:0")
    Y = synth_poisson(n, g)
    res = {"cells": n, "genes": g, "nonzero_frac": float(np.count_nonzero(Y) / Y.size)}

    t0 = time.perf_counter()
    io.normalize(AnnData(Y.copy()), filter_min_counts=False)
    res["host_normalize_s"] = time.perf_counter() - t0

    Yd = torch.empty((n, g), dtype=torch.float32, device=dev)
    res["upload_ms"] = time_events(lambda: _upload_dense(Y, Yd), reps)
    res["upload_GBps"] = n * g * 4 / res["upload_ms"] / 1e6
    wsb = C.c_size_t()
    _lib.check(lib.dca_preprocess_workspace_bytes(n, g, C.byref(wsb)))
    ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)
    nc = torch.empty(n, dtype=torch.float64, device=dev)
    gt = torch.empty(g, dtype=torch.float64, device=dev)
    bad = torch.zeros(1, dtype=torch.int64, device=dev)
    mean = torch.empty(g, dtype=torch.float64, device=dev)
    std = torch.empty(g, dtype=torch.float64, device=dev)
    X = torch.empty((n, g), dtype=torch.float32, device=dev)
    s = lambda: torch.cuda.current_stream().cuda_stream                          # noqa: E731
    ms = time_events(lambda: _lib.check(lib.dca_count_totals(Yd.data_ptr(), g, n, g, nc.data_ptr(), gt.data_ptr(),
                                                             bad.data_ptr(), ws.data_ptr(), ws.numel(), s())), reps)
    med = float(np.median(nc.cpu().numpy()))
    mbytes = n * g * 4
    kernels = {"totals": (ms, mbytes)}
    ms = time_events(lambda: _lib.check(lib.dca_log_moments(Yd.data_ptr(), g, n, g, nc.data_ptr(), med, 7, mean.data_ptr(),
                                                            std.data_ptr(), ws.data_ptr(), ws.numel(), s())), reps)
    kernels["moments"] = (ms, 2 * mbytes)
    ms = time_events(lambda: _lib.check(lib.dca_normalize_write(Yd.data_ptr(), g, n, g, nc.data_ptr(), med, 7, mean.data_ptr(),
                                                                std.data_ptr(), X.data_ptr(), _lib.F32, g, s())), reps)
    kernels["write_fp32"] = (ms, 2 * mbytes)
    for k, (t, b) in kernels.items():
        res[k + "_ms"] = t
        res[k + "_bytes"] = b
        res[k + "_TBps"] = b / t / 1e9
        res[k + "_of_3.35TBps"] = b / t / 1e9 / (HBM_BYTES_PER_S / 1e12)
    del Yd, X, ws
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    DeviceDataset.from_counts(Y, dev)
    torch.cuda.synchronize()
    res["device_from_counts_s"] = time.perf_counter() - t0
    torch.cuda.empty_cache()

    for mode in ("host", "device"):
        a = AnnData(Y.copy())
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dca(a, ae_type="zinb-conddisp", epochs=epochs, batch_size=batch, training_kwds={"preprocess": mode})
        torch.cuda.synchronize()
        res["dca_%s_s" % mode] = time.perf_counter() - t0
        del a
        torch.cuda.empty_cache()
    name, limit = card()
    res["gpu"], res["power_limit"] = name, limit
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192x20000,68000x20000")
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("diag_preprocess needs a CUDA device")
    for sz in a.sizes.split(","):
        n, g = (int(v) for v in sz.split("x"))
        print(json.dumps(measure(n, g, a.epochs, a.batch, a.reps)), flush=True)


if __name__ == "__main__":
    main()
