"""Parity of the CUDA path (through the C ABI) with the CPU oracle.  Needs an H100: -m gpu."""
import ctypes as C
import os
import subprocess
import sys
import numpy as np
import pytest
import torch

from oracle import dca_oracle as O
from tests.util import synth_counts, rel_err

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _lib():
    from dca_b200 import _lib
    return _lib


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


def _problem(B, G, seed=0):
    Y = synth_counts(B, G, seed)
    X, sf = O.normalize_inputs(Y)
    return X, Y, sf


def _post_act(B, G, seed):
    rng = np.random.default_rng(seed)
    m = np.exp(rng.normal(0, 1.5, (B, G))).astype(np.float32)
    d = np.exp(rng.normal(0, 1.5, (B, G))).astype(np.float32).clip(2e-4, 9e3)
    pi = (1 / (1 + np.exp(-rng.normal(0, 2, (B, G))))).astype(np.float32)
    return m, d, pi


def _oracle_loss(ae_type, Y, sf, m, d, pi, ridge, rows=None):
    Yb = Y[rows] if rows is not None else Y
    sfb = sf[rows] if rows is not None else sf
    m64, d64, pi64 = [a.astype(np.float64) for a in (m, d, pi)]
    mu = m64 * sfb.astype(np.float64)[:, None]
    has_pi = ae_type.startswith("zinb"); cond = ae_type.endswith("conddisp")
    th = d64 if cond else np.broadcast_to(d64[0:1, :], mu.shape)
    Yb = Yb.astype(np.float64)
    if has_pi:
        el = O.zinb_loss_elem(Yb, mu, th, pi64, ridge); dmu, dth, dpi = O.loss_partials(Yb, mu, th, pi64, ridge)
    else:
        el = O.nb_loss_elem(Yb, mu, th); dmu, dth, dpi = O.loss_partials(Yb, mu, th)
    n = el.size
    out = {"sum": el.sum(), "dzm": dmu * mu / n}
    if cond:
        out["dzd"] = dth * (1 - np.exp(-d64)) / n
    else:
        out["dtheta"] = dth.sum(0)
    if has_pi:
        out["dzp"] = dpi * pi64 * (1 - pi64) / n
    return out


@pytest.mark.parametrize("ae_type", O.AE_TYPES)
@pytest.mark.parametrize("shape", [(37, 203), (64, 256), (200, 1028)])
def test_loss_kernel_vs_oracle(ae_type, shape):
    L = _lib(); lib = L.load()
    B, G = shape
    N = B + 13
    Y = synth_counts(N, G, 1)
    Y[0, :4] = [0, 17, 40, 3000]
    sf = np.exp(np.random.default_rng(2).normal(0, 0.3, N)).astype(np.float32)
    rows = np.random.default_rng(3).permutation(N)[:B].astype(np.int32)
    m, d, pi = _post_act(B, G, 4)
    cond = ae_type.endswith("conddisp"); has_pi = ae_type.startswith("zinb")
    ref = _oracle_loss(ae_type, Y, sf, m, d, pi, 0.01, rows)
    Yd, sfd, rd = _t(Y), _t(sf), torch.as_tensor(rows).to(DEV)
    md, dd, pd = _t(m), (_t(d) if cond else _t(d[0])), _t(pi)
    gm, gd, gp = torch.empty_like(md), torch.empty_like(md), torch.empty_like(md)
    dth = torch.zeros(G, device=DEV)
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    nb = C.c_size_t(); assert lib.dca_zinb_loss_workspace_bytes(B, G, C.byref(nb)) == 0
    ws = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    st = lib.dca_zinb_loss_fwd_bwd(Yd.data_ptr(), G, rd.data_ptr(), sfd.data_ptr(), md.data_ptr(), dd.data_ptr(),
                                   pd.data_ptr() if has_pi else None, G, B, G, L.AE_TYPE_IDS[ae_type], 0.01,
                                   1.0 / (B * G), gm.data_ptr(), gd.data_ptr() if cond else None,
                                   gp.data_ptr() if has_pi else None, L.F32, dth.data_ptr(), loss.data_ptr(),
                                   ws.data_ptr(), nb.value, None)
    L.check(st, "dca_zinb_loss_fwd_bwd")
    torch.cuda.synchronize()
    assert abs(loss.item() - ref["sum"]) <= 2e-5 * abs(ref["sum"])
    assert rel_err(gm.cpu().numpy(), ref["dzm"]) < 3e-4
    if cond:
        assert rel_err(gd.cpu().numpy(), ref["dzd"]) < 3e-4
    else:
        assert rel_err(dth.cpu().numpy(), ref["dtheta"]) < 3e-4
    if has_pi:
        assert rel_err(gp.cpu().numpy(), ref["dzp"]) < 3e-4
    # forward-only kernel accumulates
    loss2 = torch.full((1,), 5.0, dtype=torch.float64, device=DEV)
    L.check(lib.dca_zinb_loss_fwd(Yd.data_ptr(), G, rd.data_ptr(), sfd.data_ptr(), md.data_ptr(), dd.data_ptr(),
                                  pd.data_ptr() if has_pi else None, G, B, G, L.AE_TYPE_IDS[ae_type], 0.01,
                                  loss2.data_ptr(), ws.data_ptr(), nb.value, None))
    torch.cuda.synchronize()
    assert abs(loss2.item() - 5.0 - ref["sum"]) <= 2e-5 * abs(ref["sum"])


def test_loss_kernel_inplace_and_bf16():
    L = _lib(); lib = L.load()
    B, G = 128, 512
    Y = synth_counts(B, G, 5); sf = np.ones(B, np.float32)
    m, d, pi = _post_act(B, G, 6)
    ref = _oracle_loss("zinb-conddisp", Y, sf, m, d, pi, 0.0)
    nb = C.c_size_t(); lib.dca_zinb_loss_workspace_bytes(B, G, C.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    Yd, sfd = _t(Y), _t(sf)
    # in place: gradients overwrite the activations
    md, dd, pd = _t(m), _t(d), _t(pi)
    L.check(lib.dca_zinb_loss_fwd_bwd(Yd.data_ptr(), G, None, sfd.data_ptr(), md.data_ptr(), dd.data_ptr(), pd.data_ptr(),
                                      G, B, G, 0, 0.0, 1.0 / (B * G), md.data_ptr(), dd.data_ptr(), pd.data_ptr(), L.F32,
                                      None, loss.data_ptr(), ws.data_ptr(), nb.value, None))
    torch.cuda.synchronize()
    assert rel_err(md.cpu().numpy(), ref["dzm"]) < 3e-4 and rel_err(pd.cpu().numpy(), ref["dzp"]) < 3e-4
    # bf16 gradient storage
    md, dd, pd = _t(m), _t(d), _t(pi)
    g = [torch.empty((B, G), dtype=torch.bfloat16, device=DEV) for _ in range(3)]
    L.check(lib.dca_zinb_loss_fwd_bwd(Yd.data_ptr(), G, None, sfd.data_ptr(), md.data_ptr(), dd.data_ptr(), pd.data_ptr(),
                                      G, B, G, 0, 0.0, 1.0 / (B * G), g[0].data_ptr(), g[1].data_ptr(), g[2].data_ptr(),
                                      L.BF16, None, loss.data_ptr(), ws.data_ptr(), nb.value, None))
    torch.cuda.synchronize()
    assert rel_err(g[0].float().cpu().numpy(), ref["dzm"]) < 6e-3      # bf16: 2^-8 relative
    assert rel_err(g[1].float().cpu().numpy(), ref["dzd"]) < 6e-3


def test_loss_kernel_golden_biochemists(golden_dir):
    """KAT: summed NLL at R's MLE (reference fixtures data/biochemists-*.tsv) through the CUDA kernel."""
    L = _lib(); lib = L.load()
    bio = dict(np.load(os.path.join(golden_dir, "biochemists.npz")))
    y = bio["y"].astype(np.float32).reshape(-1, 1); B = y.shape[0]
    nb = C.c_size_t(); lib.dca_zinb_loss_workspace_bytes(B, 1, C.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    sf = _t(np.ones(B, np.float32)); Yd = _t(y)
    g = [torch.empty((B, 1), device=DEV) for _ in range(3)]
    # NB, per-gene theta (ae_type 'nb')
    m = _t(bio["nb_pred"].reshape(-1, 1)); th = _t(np.array([float(bio["nb_theta"])]))
    dth = torch.zeros(1, device=DEV)
    L.check(lib.dca_zinb_loss_fwd_bwd(Yd.data_ptr(), 1, None, sf.data_ptr(), m.data_ptr(), th.data_ptr(), None, 1, B, 1, 3,
                                      0.0, 1.0, g[0].data_ptr(), None, None, L.F32, dth.data_ptr(), loss.data_ptr(),
                                      ws.data_ptr(), nb.value, None))
    torch.cuda.synchronize()
    assert abs(loss.item() - 1560.9583383552) < 2e-2
    assert abs(dth.item()) < 2e-2                          # stationary in theta at the MLE
    # ZINB
    m = _t(bio["zinb_pred_count"].reshape(-1, 1)); p = _t(bio["zinb_pred_zero"].reshape(-1, 1))
    th = _t(np.array([float(bio["zinb_theta"])]))
    L.check(lib.dca_zinb_loss_fwd_bwd(Yd.data_ptr(), 1, None, sf.data_ptr(), m.data_ptr(), th.data_ptr(), p.data_ptr(), 1, B, 1,
                                      1, 0.0, 1.0, g[0].data_ptr(), None, g[2].data_ptr(), L.F32, dth.data_ptr(),
                                      loss.data_ptr(), ws.data_ptr(), nb.value, None))
    torch.cuda.synchronize()
    assert abs(loss.item() - 1549.9908867856) < 2e-2
    design = bio["design"]
    assert np.max(np.abs(design.T @ g[0].cpu().numpy().astype(np.float64))) < 5e-2   # d/d beta_count = 0
    assert np.max(np.abs(design.T @ g[2].cpu().numpy().astype(np.float64))) < 5e-2   # d/d beta_zero = 0


def test_heads_fwd_vs_oracle():
    L = _lib(); lib = L.load()
    B, K, G = 50, 64, 300
    rng = np.random.default_rng(0)
    H = rng.normal(0, 1, (B, K)).astype(np.float32)
    W = [rng.normal(0, 0.3, (K, G)).astype(np.float32) for _ in range(3)]
    b = [rng.normal(0, 0.5, G).astype(np.float32) for _ in range(3)]
    sf = np.exp(rng.normal(0, 0.3, B)).astype(np.float32)
    outs = [torch.empty((B, G), device=DEV) for _ in range(3)]
    Hd, Wd, bd, sfd = _t(H), [_t(w) for w in W], [_t(x) for x in b], _t(sf)
    L.check(lib.dca_dense_heads_fwd(Hd.data_ptr(), K, B, K, G, Wd[0].data_ptr(), bd[0].data_ptr(), Wd[1].data_ptr(),
                                    bd[1].data_ptr(), Wd[2].data_ptr(), bd[2].data_ptr(), sfd.data_ptr(),
                                    outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), G, None))
    torch.cuda.synchronize()
    H64 = H.astype(np.float64)
    z = [H64 @ W[i].astype(np.float64) + b[i] for i in range(3)]
    np.testing.assert_allclose(outs[0].cpu().numpy(), O.mean_act(z[0]) * sf[:, None], rtol=2e-4)
    np.testing.assert_allclose(outs[1].cpu().numpy(), O.disp_act(z[1]), rtol=2e-4)
    np.testing.assert_allclose(outs[2].cpu().numpy(), O.sigmoid(z[2]), rtol=2e-4, atol=1e-7)


CASES = [("zinb-conddisp", True, (64, 32, 64)), ("zinb", True, (16, 8, 16)), ("nb-conddisp", False, (10, 2, 10)),
         ("nb", True, (12,)), ("zinb-conddisp", True, ()), ("zinb-conddisp", False, (64, 32, 64))]


def _make_pair(ae_type, batchnorm, hidden, B, G, seed=0, ridge=0.0, **eng_kw):
    from dca_b200.engine import DeviceEngine
    p0 = O.init_params(G, G, hidden, ae_type, batchnorm, seed=seed, dtype=np.float32)
    rng = np.random.default_rng(seed + 1)
    for k in p0:
        if k.endswith(("/bias", "/bn_beta", "/theta")):
            p0[k] = rng.normal(0, 0.2, p0[k].shape).astype(np.float32)
    net = O.OracleNet(G, G, hidden, ae_type, batchnorm, ridge=ridge, dtype=np.float64, params=p0, **{
        k: v for k, v in eng_kw.items() if k in ("l1", "l2", "l1_enc", "l2_enc")})
    eng = DeviceEngine(G, G, hidden, ae_type, batchnorm, max_batch=B, ridge=ridge, seed=None, gemm_path="generic", **eng_kw)
    eng.set_weights(p0)
    return net, eng


@pytest.mark.parametrize("ae_type,batchnorm,hidden", CASES)
def test_train_step_vs_oracle(ae_type, batchnorm, hidden):
    B, G = 96, 200
    X, Y, sf = _problem(B + 20, G, 7)
    rows = np.random.default_rng(0).permutation(B + 20)[:B].astype(np.int32)
    net, eng = _make_pair(ae_type, batchnorm, hidden, B, G, ridge=0.02, l2=1e-4, l1_enc=1e-5)
    Xd, Yd, sfd, rd = _t(X), _t(Y), _t(sf), torch.as_tensor(rows).to(DEV)
    eng.train_step(Xd, Yd, sfd, rows=rd)
    loss = eng.read_loss()
    oloss, og = net.loss_and_grads(X[rows].astype(np.float64), Y[rows].astype(np.float64), sf[rows].astype(np.float64))
    assert abs(loss - oloss) < 1e-4 * abs(oloss)
    g = eng.grads.cpu().numpy()
    for name, off, r, c in eng.param_info:
        ref = og[name].reshape(-1)
        got = g[off: off + r * c]
        if name.endswith("/bias") and batchnorm and not name.startswith(("mean", "dispersion", "pi")):
            assert np.max(np.abs(got)) < 1e-6          # exactly zero in exact arithmetic (BN removes it)
            continue
        assert rel_err(got, ref, 2e-3) < 2e-3, name
    # update + BN moving statistics
    net.rmsprop_step(og, lr=1e-3, clip=5.0)
    eng.apply_update(1e-3, 5.0, 1.0)
    w = eng.get_weights()
    for k, v in net.params.items():
        if k.endswith("/bias") and batchnorm and not k.startswith(("mean", "dispersion", "pi")):
            continue                                      # noise/(sqrt(noise^2)+eps): not comparable
        np.testing.assert_allclose(w[k], v, rtol=2e-3, atol=2e-4, err_msg=k)


def test_trajectory_five_steps():
    B, G = 64, 120
    X, Y, sf = _problem(B, G, 9)
    net, eng = _make_pair("zinb-conddisp", True, (64, 32, 64), B, G)
    Xd, Yd, sfd = _t(X), _t(Y), _t(sf)
    for _ in range(5):
        eng.train_step(Xd, Yd, sfd)
        eng.apply_update(1e-3, 5.0)
        l_o = net.train_step(X.astype(np.float64), Y.astype(np.float64), sf.astype(np.float64))
        assert abs(eng.read_loss() - l_o) < 5e-4 * abs(l_o)
    acc = eng.read_epoch_acc()
    assert acc[1] == 5 * B


@pytest.mark.parametrize("ae_type", O.AE_TYPES)
def test_predict_and_eval_vs_oracle(ae_type):
    B, G = 80, 150
    X, Y, sf = _problem(B, G, 11)
    net, eng = _make_pair(ae_type, True, (64, 32, 64), B, G)
    rng = np.random.default_rng(1)
    w = eng.get_weights()
    for k in list(w):
        if k.endswith("moving_mean"): w[k] = rng.normal(0, 0.3, w[k].shape).astype(np.float32)
        if k.endswith("moving_var"): w[k] = rng.uniform(0.5, 2.0, w[k].shape).astype(np.float32)
    eng.set_weights(w)
    for k in w: net.params[k] = w[k].astype(np.float64)
    ref = net.predict(X.astype(np.float64), sf.astype(np.float64))
    cond = ae_type.endswith("conddisp"); has_pi = ae_type.startswith("zinb")
    mean = torch.empty((B, G), device=DEV); pi = torch.empty((B, G), device=DEV) if has_pi else None
    disp = torch.empty((B, G) if cond else (G,), device=DEV); lat = torch.empty((B, 32), device=DEV)
    eng.predict(_t(X), _t(sf), mean=mean, disp=disp, pi=pi, latent=lat)
    torch.cuda.synchronize()
    np.testing.assert_allclose(mean.cpu().numpy(), ref["mean"], rtol=5e-4)
    np.testing.assert_allclose(disp.cpu().numpy(), ref["dispersion"], rtol=5e-4)
    np.testing.assert_allclose(lat.cpu().numpy(), ref["latent"], rtol=5e-4, atol=1e-5)
    if has_pi:
        np.testing.assert_allclose(pi.cpu().numpy(), ref["pi"], rtol=5e-4, atol=1e-7)
    eng.read_epoch_acc(reset=True)
    eng.eval_step(_t(X), _t(Y), _t(sf))
    acc = eng.read_epoch_acc()
    oval = net.loss(X.astype(np.float64), Y.astype(np.float64), sf.astype(np.float64), training=False)
    assert acc[3] == B * G and abs(acc[2] / acc[3] - oval) < 1e-4 * abs(oval)


def test_engine_errors_are_loud():
    from dca_b200.engine import DeviceEngine
    with pytest.raises(NotImplementedError):
        DeviceEngine(10, 10, (4,), "gaussian")
    with pytest.raises(Exception, match="one decoder layer"):
        DeviceEngine(10, 10, (8, 4, 8, 8, 8), "zinb-fork")             # forks: exactly one layer after 'center'
    eng = DeviceEngine(10, 10, (4, 2, 4), "zinb", max_batch=8)
    X = torch.zeros((9, 10), device=DEV); Y = torch.zeros((9, 10), device=DEV); sf = torch.ones(9, device=DEV)
    with pytest.raises(ValueError):
        eng.train_step(X, Y, sf)                       # batch > max_batch
    with pytest.raises(ValueError):
        eng.train_step(X[:4].double(), Y[:4], sf[:4])  # wrong dtype


def test_full_size_properties_c2():
    """C2 shape (10k x 2k zinb-conddisp, batch 4096): size-independent properties."""
    from dca_b200.engine import DeviceEngine
    N, G, B = 10000, 2000, 4096
    Y = synth_counts(N, G, 3); X, sf = O.normalize_inputs(Y)
    eng = DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=1)
    Xd, Yd, sfd = _t(X), _t(Y), _t(sf)
    rows = torch.randperm(9000, device=DEV)[:B].to(torch.int32)
    eng.train_step(Xd, Yd, sfd, rows=rows); l1 = eng.read_loss(); g1 = eng.grads.clone()
    eng.train_step(Xd, Yd, sfd, rows=rows); l2 = eng.read_loss(); g2 = eng.grads.clone()
    assert np.isfinite(l1) and l1 == l2                                        # repeatable: every sum has a fixed order
    assert torch.isfinite(g1).all()
    assert torch.equal(g1, g2)
    # loss of the batch == mean of the losses of its two halves (checksum of checksums)
    eng.read_epoch_acc(reset=True)
    eng.eval_step(Xd, Yd, sfd, rows=rows); a = eng.read_epoch_acc()
    eng.eval_step(Xd, Yd, sfd, rows=rows[: B // 2].contiguous()); eng.eval_step(Xd, Yd, sfd, rows=rows[B // 2:].contiguous())
    b = eng.read_epoch_acc()
    assert abs(a[2] - b[2]) < 1e-6 * abs(a[2]) and a[3] == b[3]
    # a few steps reduce the loss
    l0 = l1
    for _ in range(10):
        eng.train_step(Xd, Yd, sfd, rows=rows); eng.apply_update(1e-3, 5.0)
    assert eng.read_loss() < l0


# ---------------------------------------------------------------------------------------------
# tcgen05 path (bf16 operands, fp32 accumulation) inside the engine
TC_CASES = [("zinb-conddisp", True), ("zinb", True), ("nb-conddisp", False), ("nb", True)]


def _make_pair_tc(ae_type, batchnorm, B, G, seed=0):
    from dca_b200.engine import DeviceEngine
    hidden = (64, 32, 64)
    p0 = O.init_params(G, G, hidden, ae_type, batchnorm, seed=seed, dtype=np.float32)
    rng = np.random.default_rng(seed + 1)
    for k in p0:
        if k.endswith(("/bias", "/bn_beta", "/theta")):
            p0[k] = rng.normal(0, 0.2, p0[k].shape).astype(np.float32)
    net = O.OracleNet(G, G, hidden, ae_type, batchnorm, dtype=np.float64, params=p0, emulate_bf16=True)
    eng = DeviceEngine(G, G, hidden, ae_type, batchnorm, max_batch=B, seed=None, gemm_path="tcgen05")
    eng.set_weights(p0)
    return net, eng


@pytest.mark.parametrize("ae_type,batchnorm", TC_CASES)
def test_tc_train_step_vs_oracle(ae_type, batchnorm):
    """Whole step through the tensor-core kernels vs the SAME-ROUNDING fp64 oracle (GEMM operands of the
    gene-wide layers rounded to bf16 exactly where the kernels round them, everything else exact).
    ReLU-mask flips make the exact-oracle comparison discontinuous (a 2^-9 perturbation of W1 moves
    single columns of dW1 by ~10 % at batch 300), so parity of the bf16 path is defined against this."""
    B, G = 300, 264
    X, Y, sf = _problem(B + 40, G, 21)
    rows = np.random.default_rng(1).permutation(B + 40)[:B].astype(np.int32)
    net, eng = _make_pair_tc(ae_type, batchnorm, B, G)
    Xd, Yd, sfd, rd = _t(X), _t(Y), _t(sf), torch.as_tensor(rows).to(DEV)
    eng.train_step(Xd, Yd, sfd, rows=rd)
    loss = eng.read_loss()
    oloss, og = net.loss_and_grads(X[rows].astype(np.float64), Y[rows].astype(np.float64), sf[rows].astype(np.float64))
    assert abs(loss - oloss) < 5e-5 * abs(oloss), (loss, oloss)
    exact = O.OracleNet(G, G, (64, 32, 64), ae_type, batchnorm, dtype=np.float64, params=net.params)
    assert abs(loss - exact.loss(X[rows].astype(np.float64), Y[rows].astype(np.float64), sf[rows].astype(np.float64), training=True)) < 5e-3 * abs(oloss)
    g = eng.grads.cpu().numpy()
    for name, off, r, c in eng.param_info:
        ref = og[name].reshape(-1); got = g[off: off + r * c]
        if name.endswith("/bias") and batchnorm and not name.startswith(("mean", "dispersion", "pi")):
            continue
        err = np.max(np.abs(got - ref)) / (np.max(np.abs(ref)) + 1e-30)
        assert err < 2e-3, "%s: %.3g" % (name, err)
    # bf16 X storage takes the same path without the conversion copy
    from dca_b200.engine import DeviceEngine
    eng2 = DeviceEngine(G, G, (64, 32, 64), ae_type, batchnorm, max_batch=B, seed=None, gemm_path="tcgen05", x_dtype="bfloat16")
    eng2.set_weights(eng.get_weights())
    eng2.train_step(_t(X[rows], torch.bfloat16), _t(Y[rows]), _t(sf[rows]))
    assert abs(eng2.read_loss() - oloss) < 4e-3 * abs(oloss)


def test_tc_trajectory_and_predict():
    B, G = 256, 200
    X, Y, sf = _problem(B, G, 23)
    net, eng = _make_pair_tc("zinb-conddisp", True, B, G)
    Xd, Yd, sfd = _t(X), _t(Y), _t(sf)
    for _ in range(8):
        eng.train_step(Xd, Yd, sfd); eng.apply_update(1e-3, 5.0)
        l_o = net.train_step(X.astype(np.float64), Y.astype(np.float64), sf.astype(np.float64))
        assert abs(eng.read_loss() - l_o) < 1e-2 * abs(l_o)
    ref = net.predict(X.astype(np.float64), sf.astype(np.float64))
    mean = torch.empty((B, G), device=DEV); disp = torch.empty((B, G), device=DEV); pi = torch.empty((B, G), device=DEV)
    lat = torch.empty((B, 32), device=DEV)
    eng.predict(Xd, sfd, mean=mean, disp=disp, pi=pi, latent=lat)
    torch.cuda.synchronize()
    for got, key in ((mean, "mean"), (disp, "dispersion"), (pi, "pi")):
        r = ref[key]; gnp = got.cpu().numpy()
        assert np.median(np.abs(gnp - r) / (np.abs(r) + 1e-6)) < 2e-2, key
    with pytest.raises(Exception):
        from dca_b200.engine import DeviceEngine
        DeviceEngine(100, 100, (10, 2, 10), "zinb", max_batch=8, gemm_path="tcgen05")   # shape does not qualify


def test_stream_from_host_counts_matches_resident_path():
    """dca_stream_step (uint16 counts from pinned host memory, on-device normalisation) == dca_train_step on the
    host-normalised matrix (dca/io.py:99-109 restated on the device)."""
    from dca_b200.engine import DeviceEngine
    N, G, B = 700, 264, 256
    Y = synth_counts(N, G, 31); X, sf = O.normalize_inputs(Y)
    l = np.log1p(Y / sf[:, None].astype(np.float32)).astype(np.float32)
    mean = l.mean(0, dtype=np.float64); std = np.sqrt(l.var(0, ddof=1, dtype=np.float64))
    for gemm_path, tol in (("tcgen05", 2e-3), ("generic", 2e-5)):
        e1 = DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=3, gemm_path=gemm_path)
        e2 = DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=3, gemm_path=gemm_path)
        e2.set_input_transform(mean, std, True, True)
        cnt = torch.from_numpy(Y.astype(np.uint16)).pin_memory(); sfh = torch.from_numpy(sf).pin_memory()
        e2.stream_begin(cnt, sfh, B)
        nb = (N + B - 1) // B
        for i in range(nb):
            s, e = i * B, min(N, (i + 1) * B)
            e1.train_step(_t(X[s:e]), _t(Y[s:e]), _t(sf[s:e])); e1.apply_update(1e-3, 5.0)
            e2.stream_step(i, i + 1 if i + 1 < nb else -1); e2.apply_update(1e-3, 5.0)
            l1, l2 = e1.read_loss(), e2.read_loss()
            assert abs(l1 - l2) < tol * abs(l1), (gemm_path, i, l1, l2)
        e2.stream_end()


@pytest.mark.parametrize("bits", [4, 8, 16, "dense", "sparse", "auto"])
def test_stream_packed_counts_equals_uint16_stream(bits):
    """dca_stream_begin_packed (4/8/16 bits per entry + overflow list) and dca_stream_begin_sparse (non-zero bitmap +
    4-bit codes of the non-zero counts) expand to the same Y and X as the plain uint16 stream: loss trajectories are
    identical; large counts travel through the overflow list."""
    from dca_b200.engine import DeviceEngine
    from dca_b200 import io
    N, G, B = 600, 264, 256
    Y = synth_counts(N, G, 37)
    rng = np.random.default_rng(5)
    for _ in range(400):                                    # counts that need the escape in every width
        Y[rng.integers(N), rng.integers(G)] = float(rng.choice([15, 16, 40, 254, 255, 256, 3000, 60000]))
    _, sf = O.normalize_inputs(Y)
    l = np.log1p(Y / sf[:, None].astype(np.float32)).astype(np.float32)
    mean = l.mean(0, dtype=np.float64); std = np.sqrt(l.var(0, ddof=1, dtype=np.float64))
    pc = io.pack_counts(Y, bits, batch=B)
    assert np.array_equal(io.unpack_counts(pc), Y.astype(np.float32))
    e1 = DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=3, gemm_path="generic")
    e2 = DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=3, gemm_path="generic")
    sfh = torch.from_numpy(sf).pin_memory()
    for e in (e1, e2):
        e.set_input_transform(mean, std, True, True)
    e1.stream_begin(torch.from_numpy(Y.astype(np.uint16)).pin_memory(), sfh, B)
    e2.stream_begin(pc, sfh, B)
    nb = (N + B - 1) // B
    for i in range(nb):
        nxt = i + 1 if i + 1 < nb else -1
        e1.stream_step(i, nxt); e1.apply_update(1e-3, 5.0)
        e2.stream_step(i, nxt); e2.apply_update(1e-3, 5.0)
        l1, l2 = e1.read_loss(), e2.read_loss()
        assert abs(l1 - l2) <= 1e-6 * abs(l1), (bits, i, l1, l2)
    e1.stream_end(); e2.stream_end()
    # capacity check: a batch with too many escapes is refused with a message
    dense = np.full((B, G), 20.0, dtype=np.float32)
    with pytest.raises(ValueError, match="overflow"):
        e2.stream_begin(io.pack_counts(dense, 4), None, B)


@pytest.mark.parametrize("shape", [(256, 264), (300, 2000), (4096, 2000), (128, 64)])
def test_fused_heads_kernel_equals_three_kernel_path(shape):
    """flash_zinb.cu (heads forward + ZINB loss/gradient + head backward in one kernel) against the unfused
    K2 + K3 + K4 sequence: same rounding points, so loss and every gradient agree to accumulation-order noise;
    ragged cell blocks (B % 128 != 0), a partial gene tile (G % 64 != 0) and row gather are covered."""
    from dca_b200.engine import DeviceEngine
    from dca_b200 import _lib
    B, G = shape
    N = B + 37
    Y = synth_counts(N, G, 51); Y[0, :4] = [0, 17, 40, 3000]
    X, sf = O.normalize_inputs(Y)
    rows = torch.as_tensor(np.random.default_rng(3).permutation(N)[:B].astype(np.int32)).to(DEV)
    engines = []
    for fused in (1, 0):
        _lib.set_tunable("fused_heads", fused)
        engines.append(DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=9, gemm_path="tcgen05", ridge=0.01))
    _lib.set_tunable("fused_heads", 0)                                   # back to the default
    e1, e2 = engines
    Xd, Yd, sfd = _t(X), _t(Y), _t(sf)
    for step in range(3):                        # direct call, graph capture, graph replay
        for e in (e1, e2):
            e.train_step(Xd, Yd, sfd, rows=rows)
        torch.cuda.synchronize()
        l1, l2 = e1.read_loss(), e2.read_loss()
        assert abs(l1 - l2) <= 2e-6 * abs(l2), (step, l1, l2)
        G1, G2 = e1.grads.cpu().numpy(), e2.grads.cpu().numpy()
        scale = float(np.max(np.abs(G2[: e2.n_params])))     # (biases in front of a BatchNorm have a pure-noise gradient)
        for name, off, r, c in e2.param_info:
            g1, g2 = G1[off: off + r * c], G2[off: off + r * c]
            # dW1 sits behind the bf16 rounding of dA1: an fp32 ulp of order noise in dH3 can flip that rounding (2^-9)
            # the other hidden-stack tensors see that flip diluted through the 64 -> 32 -> 64 layers
            head = name.startswith(("mean", "dispersion", "pi"))
            rtol = 3e-2 if name == "enc0/kernel" else (2e-4 if head else 2e-3)
            # absolute floor 1e-4 of the largest hidden gradient: tensors whose own gradient is tiny (center/kernel: 1e-4 of
            # it) carry the same absolute order noise as their neighbours (measured 8e-5 in 2 of 5 runs)
            assert np.max(np.abs(g1 - g2)) <= rtol * np.max(np.abs(g2)) + 1e-4 * scale, (step, name, np.max(np.abs(g1 - g2)), np.max(np.abs(g2)), scale)
        for e in (e1, e2):
            e.apply_update(1e-3, 5.0)
        # keep the replicas identical: RMSprop's first steps amplify accumulation-order noise in near-zero gradients
        torch.cuda.synchronize()
        e1.params.copy_(e2.params); e1.rms.copy_(e2.rms); e1.bn_state.copy_(e2.bn_state); e1.params_changed()


def test_loss_ring_mirrors_every_step_loss():
    """dca_set_loss_ring: slot k % n of the pinned host ring holds the loss of the k-th update."""
    from dca_b200.engine import DeviceEngine
    B, G = 128, 264
    X, Y, sf = _problem(B, G, 43)
    e = DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=5, gemm_path="generic")
    Xd, Yd, sfd = _t(X), _t(Y), _t(sf)
    ring = torch.full((4,), -1.0).pin_memory()
    with pytest.raises(ValueError):
        e.set_loss_ring(torch.zeros(4))                     # not pinned
    e.set_loss_ring(ring)
    want = []
    for k in range(6):
        e.train_step(Xd, Yd, sfd); e.apply_update(1e-3, 5.0)
        want.append(e.read_loss())
        torch.cuda.synchronize()
        assert ring[k % 4].item() == pytest.approx(want[-1], rel=1e-6), (k, ring, want)
    e.set_loss_ring(None)
    e.train_step(Xd, Yd, sfd); e.apply_update(1e-3, 5.0); torch.cuda.synchronize()
    assert ring[2].item() == pytest.approx(want[2], rel=1e-6)      # untouched after switching off


@pytest.mark.parametrize("gemm_path", ["generic", "tcgen05"])
def test_two_phase_step_equals_single_call(gemm_path):
    """dca_train_step_phase(1) + (2) == dca_train_step; after phase 1 the head bucket of the gradient is final."""
    from dca_b200.engine import DeviceEngine
    B, G = 256, 264
    X, Y, sf = _problem(B, G, 41)
    e1 = DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=5, gemm_path=gemm_path)
    e2 = DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=5, gemm_path=gemm_path)
    Xd, Yd, sfd = _t(X), _t(Y), _t(sf)
    for _ in range(3):                       # 3 rounds: direct call, graph capture, graph replay
        e1.train_step(Xd, Yd, sfd)
        e2.train_step(Xd, Yd, sfd, phase=1)
        head_after_1 = e2.grads[e2.head_bucket:].clone()
        e2.train_step(Xd, Yd, sfd, phase=2)
        torch.cuda.synchronize()
        assert torch.equal(head_after_1, e2.grads[e2.head_bucket:])
        if gemm_path == "tcgen05":
            # the two halves launch the same kernels as the single call, and no sum on this path depends on timing
            assert torch.equal(e1.grads, e2.grads)
        else:
            # the fp32 path's split-K GEMMs add their partial products with atomics: order noise only
            g1, g2 = e1.grads.cpu().numpy(), e2.grads.cpu().numpy()
            assert np.max(np.abs(g1 - g2)) <= 1e-5 * np.max(np.abs(g1)) + 1e-12
        e1.apply_update(1e-3, 5.0); e2.apply_update(1e-3, 5.0)


def test_tc_step_is_bit_reproducible():
    """Two engines with the same seed and inputs compute bit-identical gradients and parameters on the tensor-core path
    (direct call, graph capture and replay on a side stream): every gradient of the step is summed in a fixed order.
    The shape spreads the gene-wide products over several cell blocks, gene ranges and partial slots."""
    from dca_b200.engine import DeviceEngine
    N, G, B = 1100, 2000, 1024
    Y = synth_counts(N, G, 7); X, sf = O.normalize_inputs(Y)
    rows = torch.as_tensor(np.random.default_rng(1).permutation(N)[:B].astype(np.int32)).to(DEV)
    engines = [DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=3, gemm_path="tcgen05") for _ in range(2)]
    Xd, Yd, sfd = _t(X), _t(Y), _t(sf)
    side = torch.cuda.Stream(DEV)
    with torch.cuda.stream(side):
        for step in range(4):
            for e in engines:
                e.train_step(Xd, Yd, sfd, rows=rows)
                e.apply_update(1e-3, 5.0)
            side.synchronize()
            assert torch.equal(engines[0].grads, engines[1].grads), step
            assert torch.equal(engines[0].params, engines[1].params), step
            assert torch.equal(engines[0].bn_state, engines[1].bn_state), step


# ---------------------------------------------------------------------------------------------------------------------
# The launch plans the tensor-core step chooses by batch size, model shape and SM budget, each against the oracle.
def _grad_errors(g, param_info, ref, batchnorm):
    """max |g - ref| / max |ref| per gradient tensor of the flat buffer g; ref: tensor name -> array, or a second flat
    buffer.  Hidden biases in front of a BatchNorm are skipped: exactly zero in exact arithmetic, pure noise here."""
    errs = {}
    for name, off, r, c in param_info:
        if batchnorm and name.endswith("/bias") and not name.startswith(("mean", "dispersion", "pi")):
            continue
        want = ref[name].reshape(-1) if isinstance(ref, dict) else ref[off: off + r * c]
        got = g[off: off + r * c]
        errs[name] = float(np.max(np.abs(got - want)) / (np.max(np.abs(want)) + 1e-30))
    return errs


# the bounds of test_tc_train_step_at_20k_genes_vs_both_oracles: loss 1e-4 relative, head tensors 3e-3 and hidden-stack
# tensors 3e-2 of their largest element (the hidden ones sit behind the bf16 rounding of dA1 in front of the encoder
# backward: an fp32 ulp of difference upstream can move one element of dW1 by 2^-9 of its size)
def _assert_step_bounds(errs, tag):
    for name, e in errs.items():
        head = name.startswith(("mean", "dispersion", "pi"))
        assert e < (3e-3 if head else 3e-2), (tag, name, e)


def _fmt_errs(errs):
    heads = max((e for n, e in errs.items() if n.startswith(("mean", "dispersion", "pi"))), default=0.0)
    hidden = max((e for n, e in errs.items() if not n.startswith(("mean", "dispersion", "pi"))), default=0.0)
    return "worst head %.2e, worst hidden %.2e" % (heads, hidden)


# (B, G, batchnorm, fused hidden stack): B <= 4096 runs 32-row strips on up to 128 CTAs; 4096 < B <= 8192 128 CTAs of
# 36-64 rows; B > 8192 the per-layer hidden kernels and the tensor-core encoder backward of that path.
#   6001: 126 strips of 48 rows with a 1-row last strip, 47 cell blocks of 128 with a 113-row last block
#   8192: 128 strips of 64 rows
#   129 x 56: one partial gene tile, one cell past a block
TC_REGIMES = [(4096, 2000, True, True), (6001, 2000, True, True), (8192, 2000, True, True), (8200, 2000, True, False),
              (8200, 2000, False, False), (129, 56, True, True)]


@pytest.mark.parametrize("B,G,batchnorm,fused", TC_REGIMES)
def test_tc_train_step_batch_regimes_vs_oracle(B, G, batchnorm, fused):
    """One tensor-core step (zinb-conddisp, row gather from a larger dataset) in every batch regime of the hidden stack
    against the same-rounding float64 oracle: loss, every gradient tensor, and the BatchNorm moving statistics after
    the step.  Without BatchNorm the hidden biases carry a real gradient and are compared too."""
    N = B + 300
    X, Y, sf = _problem(N, G, 29)
    rows = np.random.default_rng(2).permutation(N)[:B].astype(np.int32)
    net, eng = _make_pair_tc("zinb-conddisp", batchnorm, B, G)
    info = eng.info()
    assert info["tc_heads"] and info["tc_encoder"] and info["fused_hidden"] == fused, info
    w0 = eng.get_weights()
    eng.train_step(_t(X), _t(Y), _t(sf), rows=torch.as_tensor(rows).to(DEV))
    loss = eng.read_loss()
    oloss, og = net.loss_and_grads(X[rows].astype(np.float64), Y[rows].astype(np.float64), sf[rows].astype(np.float64))
    errs = _grad_errors(eng.grads.cpu().numpy(), eng.param_info, og, batchnorm)
    # moving statistics: recover the batch statistics from the update m' = mom * m + (1 - mom) * s of both
    mom = O.KERAS_DEFAULTS["bn_momentum"]
    w1 = eng.get_weights()
    bn_err = 0.0
    for k in (w0 if batchnorm else ()):
        if "bn_moving" not in k:
            continue
        s_got = (w1[k].astype(np.float64) - mom * w0[k]) / (1 - mom)
        s_ref = (net.params[k] - mom * w0[k]) / (1 - mom)
        bn_err = max(bn_err, float(np.max(np.abs(s_got - s_ref)) / (np.max(np.abs(s_ref)) + 1e-30)))
    print("\n[tc step B=%d G=%d bn=%d] loss rel %.2e, %s, batch statistics %.2e"
          % (B, G, batchnorm, abs(loss - oloss) / abs(oloss), _fmt_errs(errs), bn_err))
    assert abs(loss - oloss) < 1e-4 * abs(oloss), (loss, oloss)
    _assert_step_bounds(errs, (B, G, batchnorm))
    assert bn_err < 1e-3, bn_err


# gemm_path="auto" picks the tensor-core heads (last hidden width 64, n_out % 8 == 0) and the tensor-core encoder (first
# hidden width 64, n_in % 8 == 0) independently: (n_in, n_out), hidden, tc_heads, tc_encoder
MIXED_AUTO = [((264, 264), (64, 32), False, True), ((264, 264), (32, 64), True, False), ((264, 264), (64,), True, True),
              ((1000, 1004), (64, 32, 64), False, True), ((1004, 1000), (64, 32, 64), True, False)]


@pytest.mark.parametrize("io,hidden,tc_heads,tc_enc", MIXED_AUTO)
def test_auto_mixed_paths_vs_oracle(io, hidden, tc_heads, tc_enc):
    """Models whose tensor-core encoder and heads are chosen independently by gemm_path="auto" (one side bf16 wgmma,
    the other fp32), including a single hidden layer (L = 1, center 0) and n_in != n_out: the engine reports the path
    it chose, and loss and gradients match the oracle that rounds exactly that side to bf16."""
    from dca_b200.engine import DeviceEngine
    n_in, n_out = io
    B = 300; N = B + 40
    X, _ = O.normalize_inputs(synth_counts(N, n_in, 33))
    Y = synth_counts(N, n_out, 34); _, sf = O.normalize_inputs(Y)
    rows = np.random.default_rng(5).permutation(N)[:B].astype(np.int32)
    p0 = O.init_params(n_in, n_out, hidden, "zinb-conddisp", True, seed=3, dtype=np.float32)
    rng = np.random.default_rng(4)
    for k in p0:
        if k.endswith(("/bias", "/bn_beta")):
            p0[k] = rng.normal(0, 0.2, p0[k].shape).astype(np.float32)
    side = {(True, True): "both", (True, False): "heads", (False, True): "encoder"}[(tc_heads, tc_enc)]
    net = O.OracleNet(n_in, n_out, hidden, "zinb-conddisp", True, dtype=np.float64, params=p0, emulate_bf16=side)
    eng = DeviceEngine(n_in, n_out, hidden, "zinb-conddisp", True, max_batch=B, seed=None)
    eng.set_weights(p0)
    info = eng.info()
    assert (info["tc_heads"], info["tc_encoder"]) == (tc_heads, tc_enc), info
    eng.train_step(_t(X), _t(Y), _t(sf), rows=torch.as_tensor(rows).to(DEV))
    loss = eng.read_loss()
    oloss, og = net.loss_and_grads(X[rows].astype(np.float64), Y[rows].astype(np.float64), sf[rows].astype(np.float64))
    errs = _grad_errors(eng.grads.cpu().numpy(), eng.param_info, og, True)
    print("\n[auto %s hidden %s: bf16 %s] loss rel %.2e, %s" % (io, hidden, side, abs(loss - oloss) / abs(oloss), _fmt_errs(errs)))
    assert abs(loss - oloss) < 1e-4 * abs(oloss), (loss, oloss)
    _assert_step_bounds(errs, (io, hidden))


DP_CONFIGS = {"defaults": {}, "reserve_sms_32": {"DCA_DP_RESERVE_SMS": "32"},
              # 132 - 100 = 32 CTAs cannot hold 4096 rows in 64-row strips: 64 CTAs of 64 rows instead of 128 of 32
              "reserve_sms_100": {"DCA_DP_RESERVE_SMS": "100"}, "split_heads": {"DCA_DP_SPLIT_HEADS": "1"}}


@pytest.fixture(scope="module")
def dp_plain_and_oracle():
    """dca_train_step and the same-rounding oracle on the problem of tests/run_dp_one_rank.py (computed once)."""
    from dca_b200.engine import DeviceEngine
    from tests.run_dp_one_rank import problem, B, G, HIDDEN
    X, Y, sf, rows, p0 = problem()
    eng = DeviceEngine(G, G, HIDDEN, "zinb-conddisp", True, max_batch=B, seed=None)
    eng.set_weights(p0)
    eng.train_step(_t(X), _t(Y), _t(sf), rows=torch.as_tensor(rows).to(DEV))
    torch.cuda.synchronize()
    plain = {"grads": eng.grads.cpu().numpy(), "bn_state": eng.bn_state.cpu().numpy(), "P": eng.n_params,
             "head_bucket": eng.head_bucket, "param_info": eng.param_info}
    eng.close()
    net = O.OracleNet(G, G, HIDDEN, "zinb-conddisp", True, dtype=np.float64, params=p0, emulate_bf16=True)
    oloss, og = net.loss_and_grads(X[rows].astype(np.float64), Y[rows].astype(np.float64), sf[rows].astype(np.float64))
    return plain, oloss, og


@pytest.mark.parametrize("config", list(DP_CONFIGS))
def test_dp_step_one_rank_launch_plans_vs_plain_step_and_oracle(config, dp_plain_and_oracle, tmp_path):
    """dca_train_step_dp on a one-rank communicator (B = 4096, G = 2000) with the default launch plan, SMs reserved for
    the collective (32: a narrower hidden-stack backward grid whose strips differ from the forward's; 100: 64-row
    strips) and one head-backward launch per head.  Each runs in its own process (the switches are read once).
    Three calls (direct, graph capture, replay) give the same bits; the BatchNorm state and the head gradients (the
    phase before the reserve applies; per-head launches own the same dW / db elements as one launch) equal the plain
    step's bits; the default plan equals it everywhere; the rest is within the step bounds of the plain step and of
    the oracle."""
    plain, oloss, og = dp_plain_and_oracle
    env = {k: v for k, v in os.environ.items() if not k.startswith("DCA_DP_")}
    env.update(DP_CONFIGS[config])
    out = tmp_path / "dp.npz"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "tests", "run_dp_one_rank.py"), str(out)], env=env, cwd=root,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    d = np.load(out)
    runs = d["grads"]
    assert int(d["step_graphs"]) >= 1
    for it in (1, 2):
        assert np.array_equal(runs[it], runs[0]), (config, "call %d differs from the direct call" % it)
    g, P, hb = runs[0], plain["P"], plain["head_bucket"]
    assert np.array_equal(d["bn_state"], plain["bn_state"]), config
    assert np.array_equal(g[hb:], plain["grads"][hb:]), config            # head kernels / biases, loss slot, flag
    if config == "defaults":
        assert np.array_equal(g, plain["grads"])
    loss = float(g[P])
    e_plain = _grad_errors(g, plain["param_info"], plain["grads"], True)
    e_oracle = _grad_errors(g, plain["param_info"], og, True)
    print("\n[dp one rank, %s] vs plain step: %s; vs oracle: loss rel %.2e, %s"
          % (config, _fmt_errs(e_plain), abs(loss - oloss) / abs(oloss), _fmt_errs(e_oracle)))
    assert abs(loss - oloss) < 1e-4 * abs(oloss), (loss, oloss)
    _assert_step_bounds(e_plain, (config, "plain"))
    _assert_step_bounds(e_oracle, (config, "oracle"))
