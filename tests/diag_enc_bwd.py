"""Where the encoder side of the training step spends its time, one JSON line.

    python tests/diag_enc_bwd.py [--steps 20] [--reps 21]

On the benchmark's workload (bench.py's shape, data generator and step, imported unchanged: 68k x 20k resident bf16
X, batch 4096, zinb-conddisp), an engine after 5 steps, CUDA graphs off:
  * per-step device time of K5 (encoder backward dW1 = X[rows]^T . dA1), mid_backward, K1 (encoder forward) and
    mid_forward, from torch.profiler (CUDA activities) over --steps steps, and of all kernels of the step;
  * K5 alone through dca_tc_gene_gemm_rows mode 2 on a batch of the same X, by CUDA events, median of --reps launches
    with L2 flushed before each, and its algorithmic bytes over that time against the data-sheet 3.35 TB/s of the H100
    SXM;
  * the card's name and power limit, read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["DCA_GRAPH"] = "0"                       # every kernel of the step shows in the trace as a launch

HBM_BYTES_PER_S = 3.35e12
# kernel name -> part; K5 is gene_gemm_enc_bwd_kernel, or the (a)-only instantiation of gene_gemm_kernel before it
PARTS = {
    "K5": lambda n: "enc_bwd_kernel" in n or n.startswith("void dca::tc::gg::gene_gemm_kernel<true, false, false"),
    "mid_backward": lambda n: "mid_backward_kernel" in n,
    "K1": lambda n: n.startswith("void dca::tc::gg::gene_gemm_kernel<false, true, false, false"),
    "mid_forward": lambda n: "mid_forward_kernel" in n,
}


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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--trace", default=None, help="also write the Chrome trace here")
    a = ap.parse_args()
    import bench
    from dca_b200 import _lib
    from dca_b200.engine import DeviceEngine
    if not torch.cuda.is_available():
        raise SystemExit("diag_enc_bwd.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cells, genes, ae_type, _ = bench.WORKLOADS["c3"]
    batch = 4096
    X, Y, sf, *_ = bench.synth_on_device(cells, genes, dev, 1234, torch.bfloat16)
    eng = DeviceEngine(genes, genes, bench.HIDDEN, ae_type, True, max_batch=batch, x_dtype="bfloat16", device=dev, seed=0)
    total = a.warmup + a.steps
    gperm = torch.Generator(device=dev); gperm.manual_seed(99)
    n_train = int(cells * 0.9)
    idx = torch.cat([torch.randperm(n_train, generator=gperm, device=dev)
                     for _ in range(total * batch // n_train + 1)])[:total * batch].to(torch.int32).contiguous()
    torch.cuda.synchronize()
    side = torch.cuda.Stream(dev)
    torch.cuda.set_stream(side)

    def step(i):
        eng.train_step(X, Y, sf, rows=idx[i * batch:(i + 1) * batch])
        eng.apply_update(1e-3, 5.0, 1.0)

    for i in range(a.warmup):
        step(i)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(a.warmup, total):
            step(i)
        torch.cuda.synchronize()
    if a.trace:
        prof.export_chrome_trace(a.trace)
    per = {k: {"us_per_step": 0.0, "launches": 0, "kernel": None} for k in PARTS}
    all_us = 0.0
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or ev.name.startswith("Memcpy") or ev.name.startswith("Memset"):
            continue
        us = ev.device_time_total
        all_us += us
        for k, match in PARTS.items():
            if match(ev.name):
                per[k]["us_per_step"] += us / a.steps; per[k]["launches"] += 1; per[k]["kernel"] = ev.name[:80]
    for v in per.values():
        v["us_per_step"] = round(v["us_per_step"], 2)

    # K5 alone: the benchmark's first batch of X, dA1 of the same shape
    lib = _lib.load()
    g = torch.Generator(device=dev); g.manual_seed(0)
    rows = idx[:batch]
    dA = (torch.randn((batch, 64), generator=g, device=dev) * 1e-3).to(torch.bfloat16)
    dW = torch.zeros((genes, 64), device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def k5():
        _lib.check(lib.dca_tc_gene_gemm_rows(2, X.data_ptr(), None, None, genes, rows.data_ptr(), batch, genes, 1,
                                             dA.data_ptr(), None, None, dW.data_ptr(), None, None, 64, 0, None, None,
                                             None, stream, 0), "K5")

    k5()
    torch.cuda.synchronize()
    ms = []
    for _ in range(a.reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); k5(); e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    k5_ms = float(np.median(ms))
    nbytes = batch * genes * 2 + batch * 64 * 2 + genes * 64 * 4 * 2     # X rows, dA1, dW1 read + written
    name, limit = card()
    print(json.dumps({"card": name, "power_limit": limit, "shape": {"cells": cells, "genes": genes, "batch": batch},
                      "profiled_steps": a.steps, "in_step": per, "all_kernels_us_per_step": round(all_us / a.steps, 2),
                      "K5_alone": {"ms_median": round(k5_ms, 4), "ms_min": round(min(ms), 4), "reps": a.reps,
                                   "bytes": nbytes, "GB_per_s": round(nbytes / (k5_ms * 1e-3) / 1e9, 1),
                                   "frac_of_datasheet_hbm": round(nbytes / (k5_ms * 1e-3) / HBM_BYTES_PER_S, 3)}}))
    eng.close()


if __name__ == "__main__":
    main()
