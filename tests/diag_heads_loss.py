"""Time the heads + loss kernel (dca_tc_heads_loss, K2+3) alone on the benchmark's inputs, one JSON line.

    python tests/diag_heads_loss.py [--cells 68000] [--genes 20000] [--batch 4096] [--steps 5] [--reps 30]

The counts come from bench.py's generator (synth_on_device, same seed).  An engine built as bench.py builds it trains
--steps steps on random batches; the head weights and biases are then read from it, and H3 (the last hidden layer's
output) of the next batch is computed from its weights by the oracle's hidden-stack formula (training-mode BatchNorm,
relu) with torch on the device.  The kernel reads the batch's counts through the row indices, as in the step.  Times are
CUDA-event timings of back-to-back launches (the batch's 328 MB of counts do not stay in L2): the median, min and max of
--reps launches after 3 warm-up launches, with the byte floor (count in, three bf16 gradients out: 10 B per element) at
the data-sheet 3.35 TB/s of the H100 SXM and the card's name and power limit, read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests.diag_gather_gemm import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=68000)
    ap.add_argument("--genes", type=int, default=20000)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    import ctypes as C
    from bench import synth_on_device, HIDDEN
    from dca_b200 import _lib
    from dca_b200.engine import DeviceEngine
    from oracle import dca_oracle as O
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    N, G, B = a.cells, a.genes, a.batch
    X, Y, sf, _, _, _ = synth_on_device(N, G, dev, 1234, torch.bfloat16)
    eng = DeviceEngine(G, G, HIDDEN, "zinb-conddisp", True, max_batch=B, x_dtype="bfloat16", device=dev, seed=0)
    g = torch.Generator(device=dev); g.manual_seed(99)
    n_train = int(N * 0.9)
    batches = [torch.randperm(n_train, generator=g, device=dev)[:B].to(torch.int32).contiguous() for _ in range(a.steps + 1)]
    for rows in batches[:-1]:
        eng.train_step(X, Y, sf, rows=rows)
        eng.apply_update(1e-3, 5.0)
    torch.cuda.synchronize()
    w = {k: torch.from_numpy(np.asarray(v, np.float32)).to(dev) for k, v in eng.get_weights().items()}
    rows = batches[-1]
    with torch.no_grad():
        h = X.index_select(0, rows.long()).float()
        for i, nm in enumerate(O.layer_names(len(HIDDEN))):
            k = w[nm + "/kernel"].to(torch.bfloat16).float() if i == 0 else w[nm + "/kernel"]
            z = h @ k + w[nm + "/bias"]
            z = (z - z.mean(0)) / torch.sqrt(z.var(0, unbiased=False) + O.KERAS_DEFAULTS["bn_eps"]) + w[nm + "/bn_beta"]
            h = torch.relu(z)
    heads = O.head_names("zinb-conddisp")
    Hb = h.to(torch.bfloat16).contiguous()
    Wk = torch.stack([w[nm + "/kernel"] for nm in heads]).to(torch.bfloat16).contiguous()       # [3][64][G]
    bias = torch.cat([w[nm + "/bias"] for nm in heads]).contiguous()
    dz = [torch.empty((B, G), dtype=torch.bfloat16, device=dev) for _ in range(3)]
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    nb = C.c_size_t(); _lib.check(lib.dca_zinb_loss_workspace_bytes(B, G, C.byref(nb)), "workspace")
    ws = torch.zeros(nb.value, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def launch():
        _lib.check(lib.dca_tc_heads_loss(Hb.data_ptr(), B, Wk.data_ptr(), bias.data_ptr(), G, Y.data_ptr(), G, rows.data_ptr(),
                                         sf.data_ptr(), 0.0, 1.0 / (B * G), dz[0].data_ptr(), dz[1].data_ptr(), dz[2].data_ptr(),
                                         G, loss.data_ptr(), ws.data_ptr(), nb.value, stream), "dca_tc_heads_loss")

    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.reps)]
    for e0, e1 in ev:
        e0.record(); launch(); e1.record()
    torch.cuda.synchronize()
    ms = np.array([e0.elapsed_time(e1) for e0, e1 in ev])
    floor_ms = 10.0 * B * G / HBM_BYTES_PER_S * 1e3
    name, limit = card()
    print(json.dumps({"shape": {"cells": N, "genes": G, "batch": B}, "train_steps": a.steps, "reps": a.reps,
                      "card": name, "power_limit": limit,
                      "heads_loss_ms": {"median": round(float(np.median(ms)), 4), "min": round(float(ms.min()), 4),
                                        "max": round(float(ms.max()), 4)},
                      "byte_floor_ms": round(floor_ms, 4), "loss_sum": float(loss.item()),
                      "zero_fraction": float((Y.index_select(0, rows.long()) == 0).float().mean().item())}))


if __name__ == "__main__":
    main()
