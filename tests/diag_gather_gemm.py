"""The encoder GEMMs reading the batch's rows of X in place against gathering the batch first, one JSON line.

    python tests/diag_gather_gemm.py [--cells 68000] [--genes 20000] [--batch 4096] [--reps 9]

On a resident [cells x genes] bf16 X and a random batch of row indices, times by CUDA events (median of --reps launches,
L2 flushed before each): K1 (encoder forward, dca_tc_gene_gemm_rows mode 1) and K5 (encoder backward, mode 2) reading
X through the row indices; the copy of the batch into a contiguous [batch x genes] bf16 buffer (torch index_select,
the same bytes as the engine's former gather_rows_bf16_kernel: one read and one write of the batch) and K1 / K5 on that
buffer.  Reports each one's algorithmic bytes over its time, against the data-sheet 3.35 TB/s of the H100 SXM, the
two totals, and the card's name and power limit, read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as e:                                   # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=68000)
    ap.add_argument("--genes", type=int, default=20000)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    from dca_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    N, G, B = a.cells, a.genes, a.batch
    g = torch.Generator(device=dev); g.manual_seed(0)
    X = torch.empty((N, G), dtype=torch.bfloat16, device=dev)
    for s in range(0, N, 8192):
        X[s:s + 8192] = torch.randn((min(8192, N - s), G), generator=g, device=dev).to(torch.bfloat16)
    rows = torch.randperm(N, generator=g, device=dev)[:B].to(torch.int32).contiguous()
    Xb = torch.empty((B, G), dtype=torch.bfloat16, device=dev)
    W1 = (torch.randn((G, 64), generator=g, device=dev) * 0.05).to(torch.bfloat16)
    dA = (torch.randn((B, 64), generator=g, device=dev) * 1e-3).to(torch.bfloat16)
    out = torch.zeros((B, 64), device=dev); dW = torch.zeros((G, 64), device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def k1(Z, ld, r):
        _lib.check(lib.dca_tc_gene_gemm_rows(1, Z.data_ptr(), None, None, ld, None if r is None else r.data_ptr(), B, G, 1,
                                             None, W1.data_ptr(), out.data_ptr(), None, None, None, 64, 0, None, None,
                                             None, stream, 0), "K1")

    def k5(Z, ld, r):
        _lib.check(lib.dca_tc_gene_gemm_rows(2, Z.data_ptr(), None, None, ld, None if r is None else r.data_ptr(), B, G, 1,
                                             dA.data_ptr(), None, None, dW.data_ptr(), None, None, 64, 0, None, None,
                                             None, stream, 0), "K5")

    def gather():
        torch.index_select(X, 0, rows.long(), out=Xb)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(a.reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return float(np.median(ms))

    zb = B * G * 2                                  # the batch of X, bf16
    parts = {
        "K1_rows": (lambda: k1(X, G, rows), zb + G * 64 * 2 + B * 64 * 4 * 2),
        "K5_rows": (lambda: k5(X, G, rows), zb + B * 64 * 2 + G * 64 * 4 * 2),
        "gather_index_select": (gather, 2 * zb),
        "K1_contiguous": (lambda: k1(Xb, G, None), zb + G * 64 * 2 + B * 64 * 4 * 2),
        "K5_contiguous": (lambda: k5(Xb, G, None), zb + B * 64 * 2 + G * 64 * 4 * 2),
    }
    res = {}
    for name, (fn, nbytes) in parts.items():
        ms = timed(fn)
        res[name] = {"ms": round(ms, 4), "bytes": nbytes, "GB_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
                     "frac_of_datasheet_hbm": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}
    name, limit = card()
    print(json.dumps({"shape": {"cells": N, "genes": G, "batch": B}, "reps": a.reps, "card": name, "power_limit": limit,
                      "kernels": res,
                      "total_rows_ms": round(res["K1_rows"]["ms"] + res["K5_rows"]["ms"], 4),
                      "total_gather_then_contiguous_ms": round(res["gather_index_select"]["ms"] + res["K1_contiguous"]["ms"]
                                                               + res["K5_contiguous"]["ms"], 4)}))


if __name__ == "__main__":
    main()
