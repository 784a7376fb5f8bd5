"""The head backward (gene-GEMM mode 3) alone: one band-ordered launch against the two launches, one JSON line.

    python tests/diag_head_bwd.py [--batch 4096] [--genes 20000] [--heads 3] [--reps 21] [--staggers 0,1300]

On seeded bf16 dZ [heads x batch x genes], H3 [batch x 64] and head kernels, times dca_tc_gene_gemm mode 3 on the device
(torch.profiler kernel times, first gene-GEMM kernel to the end of the slot reduction) with the L2 flushed before every
call, alternating the two launches (head_bwd_banded = 0) and the banded launch at each --staggers value call by call in
one process (median of --reps calls each).  Reports each path's time, one read of dZ over that time (the bytes a single pass
needs) against the data-sheet 3.35 TB/s of the H100 SXM, whether the two paths gave bit-identical outputs, and the
card's name and power limit, read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.diag_gather_gemm import HBM_BYTES_PER_S, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--genes", type=int, default=20000)
    ap.add_argument("--heads", type=int, default=3)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--staggers", default="0,1300", help="head_bwd_stagger values of the banded launch to time (SM cycles)")
    a = ap.parse_args()
    from dca_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    B, G, nh = a.batch, a.genes, a.heads
    g = torch.Generator(device=dev); g.manual_seed(0)
    Z = [(torch.randn((B, G), generator=g, device=dev) * 1e-3).to(torch.bfloat16) for _ in range(nh)]
    H = torch.relu(torch.randn((B, 64), generator=g, device=dev)).to(torch.bfloat16)
    W = (torch.randn((nh, 64, G), generator=g, device=dev) * 0.2).to(torch.bfloat16).contiguous()
    outs = {v: (torch.zeros((B, 64), device=dev), [torch.zeros((64, G), device=dev) for _ in range(nh)],
                [torch.zeros(G, device=dev) for _ in range(nh)]) for v in (0, 1)}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def run(v):
        out, dW, db = outs[v]
        z = [Z[i].data_ptr() if i < nh else None for i in range(3)]
        w = [dW[i].data_ptr() if i < nh else None for i in range(3)]
        b = [db[i].data_ptr() if i < nh else None for i in range(3)]
        _lib.set_tunable("head_bwd_banded", v)
        _lib.check(lib.dca_tc_gene_gemm(3, z[0], z[1], z[2], G, B, G, nh, H.data_ptr(), W.data_ptr(), out.data_ptr(),
                                        w[0], w[1], w[2], G, 1, b[0], b[1], b[2], stream), "dca_tc_gene_gemm")

    staggers = [int(s) for s in a.staggers.split(",") if s]
    paths = [("two_launches", 0, 0)] + [("banded" if s == 0 else "banded_stagger_%d" % s, 1, s) for s in staggers]
    try:
        for v in (0, 1):                                     # warm-up, and one call each from zeroed outputs
            run(v)
        torch.cuda.synchronize()
        same = all(torch.equal(x, y) for x, y in zip([outs[0][0]] + outs[0][1] + outs[0][2],
                                                     [outs[1][0]] + outs[1][1] + outs[1][2]))
        # device time of each call: first gene-GEMM kernel start to reduce kernel end (the C entry also allocates its
        # workspace, which host-side events would time too); calls separated by the L2 flush
        from torch.profiler import ProfilerActivity, profile
        order = []
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                for name, v, s in paths:
                    flush.zero_()
                    _lib.set_tunable("head_bwd_stagger", s)
                    run(v); order.append(name)
            torch.cuda.synchronize()
    finally:
        _lib.set_tunable("head_bwd_banded", 1)
        _lib.set_tunable("head_bwd_stagger", 1300)
    ks = sorted((e for e in prof.events() if "gene_gemm" in e.name), key=lambda e: e.time_range.start)
    spans, cur = [], None
    for e in ks:
        if cur is None:
            cur = [e.time_range.start, e.time_range.end]
        cur[1] = e.time_range.end
        if "reduce" in e.name:
            spans.append(cur[1] - cur[0]); cur = None
    assert len(spans) == len(order), (len(spans), len(order))
    one_read = nh * B * G * 2
    res = {}
    for name, _, _ in paths:
        us = [t for t, n in zip(spans, order) if n == name]
        m = float(np.median(us))
        res[name] = {"us": round(m, 1), "us_min": round(min(us), 1), "us_max": round(max(us), 1),
                     "one_read_GB_per_s": round(one_read / (m * 1e-6) / 1e9, 1),
                     "one_read_frac_of_datasheet_hbm": round(one_read / (m * 1e-6) / HBM_BYTES_PER_S, 3)}
    name, limit = card()
    print(json.dumps({"shape": {"batch": B, "genes": G, "heads": nh}, "reps": a.reps, "card": name, "power_limit": limit,
                      "dZ_bytes": one_read, "paths": res, "bit_identical_first_call": same,
                      "speedup_best_banded": round(res["two_launches"]["us"] / min(r["us"] for n, r in res.items() if n != "two_launches"), 3)}))


if __name__ == "__main__":
    main()
