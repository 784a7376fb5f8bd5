"""The stand-alone ZINB loss (dca_zinb_loss_fwd_bwd) on a batch too tall for the ring kernel's launch plan.

The ring kernel walks at most 256 rows per block and puts the row chunks on the grid's y dimension, so it covers at most
65535 * 256 rows.  A batch of 65535 * 256 + 1 rows (8 genes, about 0.54 GB per fp32 tensor) needs 65536 row chunks and
runs on the generic vectorised kernel (zinb_loss_kernel + fold_partials_kernel) instead.  Checked for zinb-conddisp
and zinb (constant dispersion, dL/dtheta summed per gene), with fp32 and bf16 gradients: the gradients of sampled rows
against the float64 oracle, dL/dtheta and the loss sum against float64 sums over every row (oracle/torch_ref.py in
float64 on the device, in row chunks; dL/dtheta by autograd).  The workspace dca_zinb_loss_workspace_bytes asks for
holds zinb's dL/dtheta partials of every row chunk of the plan; one without room for them is refused."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import dca_oracle as O
from oracle import torch_ref as T
from tests.util import rel_err

DEV = "cuda:0"
B, G = 65535 * 256 + 1, 8
CHUNK = 1 << 21                                   # rows per float64 reference chunk


def _inputs(cond, seed):
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    mean = torch.exp(torch.randn(G, device=DEV, generator=g))
    sf = torch.exp(torch.randn(B, device=DEV, generator=g) * 0.35)
    Y = torch.poisson(mean[None, :] * sf[:, None], generator=g)
    Y[torch.rand(B, G, device=DEV, generator=g) < 0.3] = 0
    Y[-1] = torch.tensor([0., 1., 17., 40., 1000., 30000., 5., 0.], device=DEV)
    m = (mean[None, :] * torch.exp(torch.randn(B, G, device=DEV, generator=g) * 0.5)).clamp(1e-5, 1e6)
    dshape = (B, G) if cond else (G,)
    d = torch.nn.functional.softplus(torch.randn(dshape, device=DEV, generator=g) * 2.0).clamp(1e-4, 1e4)
    p = torch.sigmoid(torch.randn(B, G, device=DEV, generator=g) * 2.0)
    return Y, sf, m, d, p


def _oracle_rows(ae_type, y, m, sf, d, pi, inv_n):
    """float64 oracle of the sampled rows: dzm, dzp and (conddisp) dzd, scaled by 1 / N."""
    cond = ae_type.endswith("conddisp")
    y, m, sf, d, pi = [np.asarray(a, np.float64) for a in (y, m, sf, d, pi)]
    mu = m * sf[:, None]
    th = d if cond else np.broadcast_to(d[None, :], mu.shape)
    dmu, dth, dpi = O.loss_partials(y, mu, th, pi)
    out = {"dzm": dmu * mu * ((m > 1e-5) & (m < 1e6)) * inv_n, "dzp": dpi * pi * (1 - pi) * inv_n}
    if cond:
        out["dzd"] = dth * (1.0 - np.exp(-d)) * ((d > 1e-4) & (d < 1e4)) * inv_n
    return out


def _reference_sums(cond, Y, sf, m, d, p):
    """float64 loss sum over every row and (constant dispersion) dL/dtheta per gene, in row chunks."""
    theta = d.double().requires_grad_(not cond)
    total = torch.zeros((), dtype=torch.float64, device=DEV)
    for r0 in range(0, B, CHUNK):
        sl = slice(r0, min(B, r0 + CHUNK))
        th = theta[sl] if cond else theta[None, :]
        el = T.zinb_elem(Y[sl].double(), m[sl].double() * sf[sl].double()[:, None], th, p[sl].double())
        s = el.sum()
        if not cond:
            s.backward()
        total += s.detach()
    return total.item(), (None if cond else theta.grad)


@pytest.mark.gpu
@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "zinb"])
def test_loss_past_the_ring_plan_vs_oracle(ae_type):
    from dca_b200 import _lib as L
    lib = L.load()
    assert -(-B // 256) > 65535                   # more row chunks than the ring kernel's grid can hold
    cond = ae_type.endswith("conddisp")
    Y, sf, m, d, p = _inputs(cond, 7)
    inv_n = 1.0 / (B * G)
    ref_sum, ref_dth = _reference_sums(cond, Y, sf, m, d, p)
    rng = np.random.default_rng(8)
    samp = np.unique(np.concatenate([[0, 1, 65535 * 256 - 1, B - 1], rng.choice(B, 60, replace=False)]))
    ts = torch.as_tensor(samp, device=DEV)
    ref = _oracle_rows(ae_type, Y[ts].cpu().numpy(), m[ts].cpu().numpy(), sf[ts].cpu().numpy(),
                       (d[ts] if cond else d).cpu().numpy(), p[ts].cpu().numpy(), inv_n)
    nb = C.c_size_t(); assert lib.dca_zinb_loss_workspace_bytes(B, G, C.byref(nb)) == 0
    # loss partials of 65536 blocks (double) + 256 bytes, then one float per (row chunk, gene): at most the ring plan's
    # cdiv(B, 256) = 65536 row chunks
    base = 8 * 65536 + 256
    assert nb.value >= base + 4 * 65536 * G, nb.value
    ws = torch.zeros(nb.value, dtype=torch.uint8, device=DEV)
    if not cond:
        # declared a workspace of the loss partials alone (the buffer behind it is the full one)
        gm = torch.empty((B, G), device=DEV); gp = torch.empty_like(gm)
        dth = torch.empty(G, device=DEV)
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        st = lib.dca_zinb_loss_fwd_bwd(Y.data_ptr(), G, None, sf.data_ptr(), m.data_ptr(), d.data_ptr(), p.data_ptr(), G,
                                       B, G, L.AE_TYPE_IDS[ae_type], 0.0, inv_n, gm.data_ptr(), None, gp.data_ptr(), L.F32,
                                       dth.data_ptr(), loss.data_ptr(), ws.data_ptr(), base, None)
        torch.cuda.synchronize()
        assert st == -1 and b"workspace too small" in lib.dca_last_error(), (st, lib.dca_last_error())
        del gm, gp
    for gdt, tol in ((L.F32, 3e-4), (L.BF16, 6e-3)):
        tdt = torch.bfloat16 if gdt == L.BF16 else torch.float32
        gm = torch.empty((B, G), dtype=tdt, device=DEV); gp = torch.empty_like(gm)
        gd = torch.empty_like(gm) if cond else None
        dth = torch.empty(G, device=DEV)
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        L.check(lib.dca_zinb_loss_fwd_bwd(Y.data_ptr(), G, None, sf.data_ptr(), m.data_ptr(), d.data_ptr(), p.data_ptr(), G,
                                          B, G, L.AE_TYPE_IDS[ae_type], 0.0, inv_n, gm.data_ptr(),
                                          gd.data_ptr() if cond else None, gp.data_ptr(), gdt,
                                          None if cond else dth.data_ptr(), loss.data_ptr(), ws.data_ptr(), nb.value, None),
                "dca_zinb_loss_fwd_bwd")
        torch.cuda.synchronize()
        total = float(loss.item())
        assert abs(total - ref_sum) <= 2e-5 * abs(ref_sum), (ae_type, gdt, total, ref_sum)
        got = {"dzm": gm, "dzp": gp}
        if cond:
            got["dzd"] = gd
        for nm, t in got.items():
            e = rel_err(t[ts].float().cpu().numpy(), ref[nm])
            assert e < tol, (ae_type, gdt, nm, e)
        if not cond:
            assert rel_err(dth.cpu().numpy(), ref_dth.cpu().numpy()) < 3e-4, (gdt, dth, ref_dth)
        del gm, gp, gd


def test_deleted_loss_tunables_are_unknown_names():
    """The loss kernel has one backward variant: its former selectors fail like any other unknown name."""
    from dca_b200 import _lib as L
    lib = L.load()
    for name in (b"loss_ring", b"loss_branch_free", b"loss_producer_sleep_ns", b"loss_consumer_sleep_ns"):
        assert lib.dca_set_tunable(name, 1) == -1, name          # DCA_ERR_BAD_ARG
    assert lib.dca_set_tunable(b"loss_target_blocks", 0) == 0    # the launch-plan override stays
