"""Sweep of the loss kernel's launch tunables (dca_set_tunable) on synthetic head outputs.

Not a test: run by hand on a GPU box,  python tests/diag_loss_sweep.py > loss_sweep.log
Prints one line per (shape, gradient dtype, target blocks, producer/consumer sleep): median ms over
launches with the L2 flushed in between, and the algorithmic GB/s (28 B / element fp32 gradients,
22 B / element bf16 gradients).
"""
import ctypes as C
import itertools
import sys

import numpy as np
import torch

from dca_b200 import _lib


def main():
    lib = _lib.load()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev); g.manual_seed(0)
    shapes = [(4096, 2000), (4096, 20000)]
    if len(sys.argv) > 1:
        shapes = [tuple(int(v) for v in s.split("x")) for s in sys.argv[1:]]
    flush = torch.empty(160 * 1024 * 1024, dtype=torch.uint8, device=dev)
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for (B, G) in shapes:
        lam = torch.rand(G, device=dev, generator=g) * 0.4
        Y = torch.poisson(lam.expand(B, G).contiguous(), generator=g)
        m = torch.exp(torch.randn(B, G, device=dev, generator=g) * 0.5)
        d = torch.nn.functional.softplus(torch.randn(B, G, device=dev, generator=g))
        p = torch.sigmoid(torch.randn(B, G, device=dev, generator=g))
        sf = torch.ones(B, device=dev)
        rows = torch.randperm(B, device=dev, generator=g).int()
        nb = C.c_size_t(); lib.dca_zinb_loss_workspace_bytes(B, G, C.byref(nb))
        ws = torch.zeros(nb.value, dtype=torch.uint8, device=dev); loss = torch.zeros(1, dtype=torch.float64, device=dev)
        print("shape %dx%d zero fraction %.3f" % (B, G, float((Y == 0).float().mean())), flush=True)
        for gdt, gbytes in ((_lib.BF16, 2), (_lib.F32, 4)):
            tdt = torch.bfloat16 if gbytes == 2 else torch.float32
            gm = torch.empty((B, G), dtype=tdt, device=dev); gd = torch.empty_like(gm); gp = torch.empty_like(gm)
            ref = None
            for tb, (ps, cs), bf in itertools.product((0, 2368, 444), ((0, 0),), (0, 1)):
                for k, v in (("loss_target_blocks", tb), ("loss_producer_sleep_ns", ps), ("loss_consumer_sleep_ns", cs), ("loss_branch_free", bf)):
                    _lib.check(lib.dca_set_tunable(k.encode(), v), k)
                times = []
                for it in range(7):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    rc = lib.dca_zinb_loss_fwd_bwd(Y.data_ptr(), G, rows.data_ptr(), sf.data_ptr(), m.data_ptr(), d.data_ptr(),
                                                   p.data_ptr(), G, B, G, 0, 0.0, 1.0 / (B * G), gm.data_ptr(), gd.data_ptr(),
                                                   gp.data_ptr(), gdt, None, loss.data_ptr(), ws.data_ptr(), nb.value, st)
                    e1.record(); torch.cuda.synchronize(dev)
                    _lib.check(rc, "dca_zinb_loss_fwd_bwd")
                    if it >= 2:
                        times.append(e0.elapsed_time(e1))
                val = float(loss.item())
                if ref is None:
                    ref = val
                ms = float(np.median(times)); byts = B * G * (16 + 3 * gbytes)
                print("  grad=%s blocks=%4d sleep=%4d/%3d bf=%d  ms=%.4f  %.0f GB/s  loss_sum_rel_dev=%.1e"
                      % ("bf16" if gbytes == 2 else "fp32", tb, ps, cs, bf, ms, byts / ms / 1e6, abs(val - ref) / abs(ref)), flush=True)


if __name__ == "__main__":
    main()
