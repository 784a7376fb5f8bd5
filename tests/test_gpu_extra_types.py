"""The remaining registry keys of dca/network.py:763-768 (poisson, normal, nb-shared, zinb-shared, zinb-elempi [+ sharedpi],
nb-fork, zinb-fork) through the C ABI against the float64 AUTOGRAD statement of the same networks
(oracle/torch_ref.py:TorchExtraNet -- autograd plays the role TF autodiff plays in the reference): one training step
(loss, every gradient tensor), a short trajectory with the RMSprop update and BatchNorm moving statistics, validation
loss and predict outputs.  Needs an H100: -m gpu."""
import numpy as np
import pytest
import torch

from oracle import dca_oracle as O
from oracle.torch_ref import TorchExtraNet, extra_init_params, EXTRA_TYPES
from tests.util import synth_counts, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = [(t, False) for t in EXTRA_TYPES] + [("zinb-elempi", True)]


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


def _pair(ae_type, sharedpi, B, G, hidden=(16, 8, 16), batchnorm=True, ridge=0.0, seed=0):
    from dca_b200.engine import DeviceEngine
    p0 = extra_init_params(G, G, hidden, ae_type, batchnorm, seed=seed, sharedpi=sharedpi)
    rng = np.random.default_rng(seed + 1)
    for k in p0:
        if k.endswith(("/bias", "/bn_beta")):
            p0[k] = rng.normal(0, 0.2, p0[k].shape).astype(np.float32)
    net = TorchExtraNet(p0, hidden, ae_type, batchnorm, ridge=ridge)
    eng = DeviceEngine(G, G, hidden, ae_type, batchnorm, max_batch=B, ridge=ridge, seed=None, sharedpi=sharedpi)
    assert sorted(n for n, *_ in eng.param_info) == sorted(k for k in p0 if k.endswith(("/kernel", "/bias", "/bn_beta"))), \
        (sorted(n for n, *_ in eng.param_info), sorted(p0))
    eng.set_weights(p0)
    return net, eng


@pytest.mark.parametrize("ae_type,sharedpi", CASES)
@pytest.mark.parametrize("batchnorm", [True, False])
def test_extra_type_train_step_vs_autograd(ae_type, sharedpi, batchnorm):
    B, G = 96, 120
    Y = synth_counts(B + 20, G, 7); X, sf = O.normalize_inputs(Y)
    rows = np.random.default_rng(0).permutation(B + 20)[:B].astype(np.int32)
    net, eng = _pair(ae_type, sharedpi, B, G, batchnorm=batchnorm, ridge=0.02 if ae_type.startswith("zinb") else 0.0)
    eng.train_step(_t(X), _t(Y), _t(sf), rows=torch.as_tensor(rows).to(DEV))
    loss = eng.read_loss()
    T = lambda a: torch.tensor(a, dtype=torch.float64)
    oloss, og, _ = net.loss_and_grads(T(X[rows]), T(Y[rows]), T(sf[rows]))
    assert abs(loss - oloss) < 1e-4 * abs(oloss), (ae_type, loss, oloss)
    g = eng.grads.cpu().numpy()
    for name, off, r, c in eng.param_info:
        ref = og[name].numpy().reshape(-1); got = g[off: off + r * c]
        if name.endswith("/bias") and batchnorm and not name.startswith(("mean", "dispersion", "pi")):
            assert np.max(np.abs(got)) < 1e-5          # exactly zero in exact arithmetic (BatchNorm removes it)
            continue
        assert rel_err(got, ref, 2e-3) < 3e-3, (ae_type, name, rel_err(got, ref, 2e-3))


@pytest.mark.parametrize("ae_type,sharedpi", CASES)
def test_extra_type_trajectory_eval_and_predict(ae_type, sharedpi):
    B, G = 64, 80
    Y = synth_counts(B, G, 9); X, sf = O.normalize_inputs(Y)
    net, eng = _pair(ae_type, sharedpi, B, G)
    T = lambda a: torch.tensor(a, dtype=torch.float64)
    Xd, Yd, sfd = _t(X), _t(Y), _t(sf)
    for _ in range(4):
        eng.train_step(Xd, Yd, sfd); eng.apply_update(1e-3, 5.0)
        l_o = net.train_step(T(X), T(Y), T(sf))
        assert abs(eng.read_loss() - l_o) < 5e-4 * abs(l_o), ae_type
    # validation loss (inference-mode BatchNorm)
    eng.read_epoch_acc(reset=True)
    eng.eval_step(Xd, Yd, sfd)
    acc = eng.read_epoch_acc()
    with torch.no_grad():
        oval = float(net.loss(T(X), T(Y), T(sf), training=False)[0])
    assert abs(acc[2] / acc[3] - oval) < 2e-4 * abs(oval), (ae_type, acc, oval)
    # predict
    ref = net.predict(T(X), T(sf))
    shared = ae_type in ("nb-shared", "zinb-shared")
    mean = torch.empty((B, G), device=DEV); lat = torch.empty((B, 8), device=DEV)
    disp = torch.empty((B, 1 if shared else G), device=DEV) if "dispersion" in ref else None
    pi = torch.empty((B, 1 if shared else G), device=DEV) if "pi" in ref else None
    eng.predict(Xd, sfd, mean=mean, disp=disp, pi=pi, latent=lat)
    torch.cuda.synchronize()
    # tolerances relative to the tensor scale (linear outputs cross zero: 'normal' mean, latent)
    np.testing.assert_allclose(mean.cpu().numpy(), ref["mean"], rtol=2e-3, atol=5e-4 * np.abs(ref["mean"]).max())
    np.testing.assert_allclose(lat.cpu().numpy(), ref["latent"], rtol=2e-3, atol=5e-4 * np.abs(ref["latent"]).max())
    if disp is not None:
        np.testing.assert_allclose(disp.cpu().numpy().reshape(ref["dispersion"].shape), ref["dispersion"], rtol=2e-3)
    if pi is not None:
        np.testing.assert_allclose(pi.cpu().numpy().reshape(ref["pi"].shape), ref["pi"], rtol=2e-3, atol=1e-7)


def test_poisson_nan_targets_are_left_out_of_the_mean():
    """poisson_loss (dca/loss.py:40-46): NaN targets count as zero and are excluded from the element count."""
    from dca_b200.engine import DeviceEngine
    B, G = 32, 40
    Y = synth_counts(B, G, 3); X, sf = O.normalize_inputs(Y)
    Yn = Y.copy(); Yn[3, 5] = np.nan; Yn[10, :4] = np.nan
    net, eng = _pair("poisson", False, B, G)
    T = lambda a: torch.tensor(a, dtype=torch.float64)
    eng.train_step(_t(X), _t(Yn), _t(sf))
    oloss, og, _ = net.loss_and_grads(T(X), T(Yn), T(sf))
    assert np.isfinite(oloss) and abs(eng.read_loss() - oloss) < 1e-4 * abs(oloss)
    g = eng.grads.cpu().numpy()
    name, off, r, c = [t for t in eng.param_info if t[0] == "mean/kernel"][0]
    assert rel_err(g[off: off + r * c], og[name].numpy().reshape(-1), 2e-3) < 3e-3
