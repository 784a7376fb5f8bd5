"""A/B of the two ZINB loss kernels (dca_set_tunable "loss_ring": 0 = block-wide bulk-copy ring, 1 = per-thread
cp.async ring with f32x2 arithmetic) on realistic operands: timing (L2 flushed, CUDA events) and a numerical check
of loss + the three gradient tensors against a float64 torch statement of dca/loss.py:122-148 on sampled rows.

Not a test: run by hand on a GPU box,  python tests/diag_loss_ab.py > loss_ab.log
"""
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dca_b200 import _lib  # noqa: E402


def ref64(y, m, sf, d, p, cond):
    """float64 autograd statement of ZINB.loss (sum over the given elements) and d/d pre-activations."""
    eps = 1e-10
    zm = torch.log(m.double()).requires_grad_(True)
    mm = torch.clamp(torch.exp(zm), 1e-5, 1e6)
    if cond:
        zd = torch.log(torch.expm1(d.double())).requires_grad_(True)          # softplus^-1
        th = torch.clamp(torch.nn.functional.softplus(zd), 1e-4, 1e4)
    else:
        zd = d.double().clone().requires_grad_(True); th = zd
    zp = torch.logit(p.double()).requires_grad_(True)
    pi = torch.sigmoid(zp)
    mu = mm * sf.double()[:, None]
    th = torch.clamp(th, max=1e6)
    t1 = torch.lgamma(th + eps) + torch.lgamma(y + 1.0) - torch.lgamma(y + th + eps)
    t2 = (th + y) * torch.log(1.0 + mu / (th + eps)) + y * (torch.log(th + eps) - torch.log(mu + eps))
    nb = t1 + t2 - torch.log(1.0 - pi + eps)
    zero = -torch.log(pi + (1.0 - pi) * torch.pow(th / (th + mu + eps), th) + eps)
    el = torch.where(y < 1e-8, zero, nb)
    tot = el.sum()
    tot.backward()
    return float(tot), zm.grad, zd.grad, zp.grad


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
        logm = torch.randn(G, device=dev, generator=g) * 1.5 - 2.0
        depth = torch.exp(torch.randn(B, 1, device=dev, generator=g) * 0.35)
        lam = torch._standard_gamma(torch.full((B, G), 2.0, device=dev), generator=g) * depth * torch.exp(logm)[None, :] / 2.0
        Y = torch.poisson(lam, generator=g)
        Y[torch.rand(B, G, device=dev, generator=g) < 0.2] = 0
        m = torch.exp(logm[None, :] + torch.randn(B, G, device=dev, generator=g) * 0.5).clamp(1e-5, 1e6)
        d = torch.nn.functional.softplus(torch.randn(B, G, device=dev, generator=g) * 1.5).clamp(1e-4, 1e4)
        p = torch.sigmoid(torch.randn(B, G, device=dev, generator=g))
        sf = depth.flatten().contiguous()
        thg = torch.exp(torch.randn(G, device=dev, generator=g)).clamp(1e-3, 1e4)
        rows = torch.randperm(B, device=dev, generator=g).int()
        nb = C.c_size_t(); lib.dca_zinb_loss_workspace_bytes(B, G, C.byref(nb))
        ws = torch.zeros(nb.value, dtype=torch.uint8, device=dev); loss = torch.zeros(1, dtype=torch.float64, device=dev)
        print("shape %dx%d zero fraction %.3f, max count %d, counts>16: %.4f" % (
            B, G, float((Y == 0).float().mean()), int(Y.max()), float((Y > 16).float().mean())), flush=True)
        samp = torch.arange(0, B, max(1, B // 64), device=dev)[:64]            # kernel rows checked against float64
        inv_n = 1.0 / (B * G)
        for ae, cond in ((0, True), (1, False)):
            dd = d if cond else thg
            ysamp = Y[rows[samp].long()].double()
            rl, rgm, rgd, rgp = ref64(ysamp, m[samp], sf[rows[samp].long()], d[samp] if cond else thg[None, :].expand(len(samp), G), p[samp], cond)
            for gdt, gbytes in ((_lib.BF16, 2), (_lib.F32, 4)):
                tdt = torch.bfloat16 if gbytes == 2 else torch.float32
                gm = torch.zeros((B, G), dtype=tdt, device=dev); gd = torch.zeros_like(gm); gp = torch.zeros_like(gm)
                dth = torch.zeros(G, device=dev)
                base = None
                for ring, tb in ((0, 0), (1, 0), (2, 0), (2, 148 * 12), (2, 148 * 24), (1, 148 * 24)):
                    _lib.check(lib.dca_set_tunable(b"loss_ring", ring), "loss_ring")
                    _lib.check(lib.dca_set_tunable(b"loss_target_blocks", tb), "loss_target_blocks")
                    times = []
                    for it in range(7):
                        flush.zero_()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        rc = lib.dca_zinb_loss_fwd_bwd(Y.data_ptr(), G, rows.data_ptr(), sf.data_ptr(), m.data_ptr(), dd.data_ptr(),
                                                       p.data_ptr(), G, B, G, ae, 0.0, inv_n, gm.data_ptr(),
                                                       gd.data_ptr() if cond else None, gp.data_ptr(), gdt,
                                                       None if cond else dth.data_ptr(), loss.data_ptr(), ws.data_ptr(), nb.value, st)
                        e1.record(); torch.cuda.synchronize(dev)
                        _lib.check(rc, "dca_zinb_loss_fwd_bwd")
                        if it >= 2:
                            times.append(e0.elapsed_time(e1))
                    val = float(loss.item())
                    if base is None:
                        base = val
                    # gradients of the sampled rows against float64 (per-tensor scale)
                    def err(got, ref):
                        ref = ref * inv_n
                        return float((got[samp].double() - ref).abs().max() / ref.abs().max())
                    e_m = err(gm, rgm); e_p = err(gp, rgp)
                    e_d = err(gd, rgd) if cond else float(((dth.double() * 1.0) - 0).abs().max() * 0)   # dtheta is checked by pytest
                    ms = float(np.median(times)); byts = B * G * (4 + 4 * (3 if cond else 2) + (3 if cond else 2) * gbytes)
                    print("  ae=%d grad=%s ring=%d blocks=%4d  ms=%.4f  %.0f GB/s  loss_rel_dev_vs_ring0=%.1e  grad err vs f64 (of tensor max): m %.1e d %.1e pi %.1e"
                          % (ae, "bf16" if gbytes == 2 else "fp32", ring, tb, ms, byts / ms / 1e6, abs(val - base) / abs(base), e_m, e_d, e_p), flush=True)
    _lib.check(lib.dca_set_tunable(b"loss_ring", 1), "loss_ring")
    _lib.check(lib.dca_set_tunable(b"loss_target_blocks", 0), "loss_target_blocks")


if __name__ == "__main__":
    main()
