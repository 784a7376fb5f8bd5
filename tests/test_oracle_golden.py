"""Pin the oracle against the reference's own fixtures (data/biochemists-*.tsv, via
tests/golden/biochemists.npz) and against autograd.  CPU only."""
import os
import numpy as np
import pytest
import torch

from oracle import dca_oracle as O
from oracle import torch_ref as T


@pytest.fixture(scope="module")
def bio(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "biochemists.npz")))


def test_nb_predictions_match_R(bio):
    mu = np.exp(bio["design"] @ bio["nb_beta"])
    assert np.max(np.abs(mu - bio["nb_pred"])) < 1e-12


def test_zinb_predictions_match_R(bio):
    mu = np.exp(bio["design"] @ bio["zinb_count"])
    pi = 1 / (1 + np.exp(-(bio["design"] @ bio["zinb_zero"])))
    assert np.max(np.abs(mu - bio["zinb_pred_count"])) < 1e-12
    assert np.max(np.abs(pi - bio["zinb_pred_zero"])) < 1e-12


def test_kat_nb_sum_nll(bio):
    y = bio["y"]; mu = bio["nb_pred"]
    s = np.sum(O.nb_loss_elem(y, mu, np.full_like(y, float(bio["nb_theta"]))))
    assert abs(s - 1560.9583383552) < 1e-6           # SURVEY.md 8c KAT-1
    assert abs(s - float(bio["kat_nb_sum_nll"])) < 1e-9


def test_kat_zinb_sum_nll(bio):
    y = bio["y"]
    s = np.sum(O.zinb_loss_elem(y, bio["zinb_pred_count"], np.full_like(y, float(bio["zinb_theta"])),
                                bio["zinb_pred_zero"]))
    assert abs(s - 1549.9908867856) < 1e-6           # SURVEY.md 8c KAT-2


def test_nb_gradient_vanishes_at_R_mle(bio):
    """R's glm.nb MLE is a stationary point of dca/loss.py:87-88 => pins the NB formula."""
    y = bio["y"]; Xd = bio["design"]; th = float(bio["nb_theta"])
    mu = np.exp(Xd @ bio["nb_beta"])
    dmu, dth, _ = O.loss_partials(y, mu, np.full_like(y, th))
    g_beta = Xd.T @ (dmu * mu)
    assert np.max(np.abs(g_beta)) < 1e-4
    assert abs(np.sum(dth)) < 1e-4


def test_zinb_gradient_vanishes_at_R_mle(bio):
    y = bio["y"]; Xd = bio["design"]; th = float(bio["zinb_theta"])
    mu = np.exp(Xd @ bio["zinb_count"]); pi = 1 / (1 + np.exp(-(Xd @ bio["zinb_zero"])))
    dmu, dth, dpi = O.loss_partials(y, mu, np.full_like(y, th), pi)
    assert np.max(np.abs(Xd.T @ (dmu * mu))) < 1e-3
    assert np.max(np.abs(Xd.T @ (dpi * pi * (1 - pi)))) < 1e-3
    assert abs(np.sum(dth)) < 1e-3


def _rand_problem(B, G, seed, hidden=(16, 8, 16)):
    rng = np.random.default_rng(seed)
    lam = rng.gamma(2.0, 1.0, size=(B, G)) * np.exp(rng.normal(-1, 1, size=(1, G)))
    Y = rng.poisson(lam).astype(np.float64)
    Y[rng.random((B, G)) < 0.3] = 0
    Y[:, Y.sum(0) == 0] = 1
    Y[Y.sum(1) == 0, 0] = 1
    X, sf = O.normalize_inputs(Y)
    return X.astype(np.float64), Y, sf.astype(np.float64)


@pytest.mark.parametrize("ae_type", O.AE_TYPES)
@pytest.mark.parametrize("batchnorm", [True, False])
def test_closed_form_grads_match_autograd(ae_type, batchnorm):
    B, G = 24, 40
    X, Y, sf = _rand_problem(B, G, 3)
    net = O.OracleNet(G, G, (16, 8, 16), ae_type, batchnorm, ridge=0.1, dtype=np.float64,
                      params=O.init_params(G, G, (16, 8, 16), ae_type, batchnorm, seed=1, dtype=np.float64))
    # make biases/theta non-trivial
    rng = np.random.default_rng(5)
    for k in net.params:
        if k.endswith(("/bias", "/bn_beta", "/theta")):
            net.params[k] = rng.normal(0, 0.3, net.params[k].shape)
    ref = T.TorchRefNet(net.params, (16, 8, 16), ae_type, batchnorm, ridge=0.1, dtype=torch.float64)
    loss, g = net.loss_and_grads(X, Y, sf, update_bn=False)
    tl, tg, _ = ref.loss_and_grads(torch.tensor(X), torch.tensor(Y), torch.tensor(sf))
    assert abs(loss - tl) < 1e-10 * max(1, abs(tl))
    assert set(g) == set(tg)
    for k in g:
        np.testing.assert_allclose(g[k], tg[k].numpy(), rtol=1e-8, atol=1e-12, err_msg=k)


def test_train_steps_match_torch_ref():
    B, G = 32, 30
    X, Y, sf = _rand_problem(B, G, 11)
    p0 = O.init_params(G, G, (8, 4, 8), "zinb-conddisp", True, seed=2, dtype=np.float64)
    net = O.OracleNet(G, G, (8, 4, 8), "zinb-conddisp", True, dtype=np.float64, params=p0)
    ref = T.TorchRefNet(p0, (8, 4, 8), "zinb-conddisp", True, dtype=torch.float64)
    for _ in range(5):
        l1 = net.train_step(X, Y, sf)
        l2 = ref.train_step(torch.tensor(X), torch.tensor(Y), torch.tensor(sf))
        assert abs(l1 - l2) < 1e-9
    for k in net.params:
        np.testing.assert_allclose(net.params[k], ref.p[k].detach().numpy(), rtol=1e-7, atol=1e-10, err_msg=k)


def test_loss_edge_cases_finite():
    y = np.array([0, 0, 1, 5, 1000, 0, 3.0])
    mu = np.array([1e-5, 1e6, 1e-5, 1e6, 50.0, 2.0, 2.0])
    th = np.array([1e-4, 1e4, 1e4, 1e-4, 1.0, 1e-3, 1e4])
    pi = np.array([0.0, 1.0, 1e-9, 1 - 1e-9, 0.5, 0.999, 0.001])
    el = O.zinb_loss_elem(y, mu, th, pi)
    assert np.all(np.isfinite(el))
    d = O.loss_partials(y, mu, th, pi)
    assert all(np.all(np.isfinite(x)) for x in d)


def test_fit_keras_semantics_history_keys():
    X, Y, sf = _rand_problem(50, 12, 4)
    net = O.OracleNet(12, 12, (4, 2, 4), "nb-conddisp", True)
    h = O.fit(net, X, Y, sf, epochs=3, batch_size=8)
    assert set(h) == {"loss", "val_loss", "lr"} and len(h["loss"]) == 3 and len(h["val_loss"]) == 3


def test_oracle_bf16_emulation_per_side():
    """emulate_bf16 rounds the encoder side (X, first kernel, dA of the first layer), the head side (last hidden
    activation, head kernels, dZ), both (True) or neither (False), independently -- the engine chooses its tensor-core
    encoder and heads independently."""
    from tests.util import synth_counts
    n_in, n_out, hidden, B = 24, 16, (8, 4, 8), 20
    X, _ = O.normalize_inputs(synth_counts(B, n_in, 1))
    Y = synth_counts(B, n_out, 2); _, sf = O.normalize_inputs(Y)
    X, Y, sf = X.astype(np.float64), Y.astype(np.float64), sf.astype(np.float64)
    p0 = O.init_params(n_in, n_out, hidden, "zinb-conddisp", True, seed=0)
    nets = {s: O.OracleNet(n_in, n_out, hidden, "zinb-conddisp", True, params=p0, emulate_bf16=s)
            for s in (True, False, "both", "none", "encoder", "heads")}
    out = {s: n.forward(X, sf, training=True) for s, n in nets.items()}
    grads = {s: n.loss_and_grads(X, Y, sf, update_bn=False)[1] for s, n in nets.items()}
    for a, b in ((True, "both"), (False, "none")):
        for k in grads[a]:
            assert np.array_equal(grads[a][k], grads[b][k]), (a, k)
    # the encoder side alone decides the hidden stack's forward; the head side the heads' rounding
    assert np.array_equal(out["encoder"]["latent"], out["both"]["latent"])
    assert np.array_equal(out["heads"]["latent"], out["none"]["latent"])
    assert not np.array_equal(out["encoder"]["latent"], out["none"]["latent"])
    h = out["heads"]["decoded"]
    zm = O.bf16_round(h) @ O.bf16_round(p0["mean/kernel"].astype(np.float64)) + p0["mean/bias"]
    assert np.array_equal(out["heads"]["z"]["mean"], zm)
    assert np.array_equal(out["encoder"]["z"]["mean"], out["encoder"]["decoded"] @ p0["mean/kernel"].astype(np.float64) + p0["mean/bias"])
    # all four variants differ in the first kernel's gradient
    g0 = [grads[s]["enc0/kernel"] for s in ("both", "none", "encoder", "heads")]
    assert all(not np.array_equal(g0[i], g0[j]) for i in range(4) for j in range(i + 1, 4))
    with pytest.raises(AssertionError):
        O.OracleNet(n_in, n_out, hidden, "zinb-conddisp", True, params=p0, emulate_bf16="decoder")
