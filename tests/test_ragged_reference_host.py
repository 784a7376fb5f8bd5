"""The row-chunked float64 reference (oracle/torch_ref.py: loss_and_grads_chunked) that checks the fp32 training step at
full gene counts on the device: the same mean loss and gradients as the one-piece autograd step, and as the NumPy
oracle's closed-form backward.  Runs on the CPU."""
import numpy as np
import pytest
import torch

from oracle import dca_oracle as O
from oracle.torch_ref import TorchRefNet, TorchExtraNet, extra_init_params
from tests.util import synth_counts

HIDDEN = (16, 8, 16)


def _problem(B, G, seed):
    """The first B rows of a 70-row normalised dataset (one row has no per-gene variance of its own)."""
    Y = synth_counts(70, G, seed)
    X, sf = O.normalize_inputs(Y)
    return X[:B].astype(np.float64), Y[:B].astype(np.float64), sf[:B].astype(np.float64)


def _nontrivial(p, seed):
    rng = np.random.default_rng(seed)
    for k in p:
        if k.endswith(("/bias", "/bn_beta", "/theta")):
            p[k] = rng.normal(0, 0.2, p[k].shape)
    return p


def _assert_grads_close(got, want, tol, tag):
    """Per tensor, max |got - want| <= tol * max |want|, with the largest gradient of the step as the floor: at B = 1
    with BatchNorm every gradient in front of the first BatchNorm is zero in exact arithmetic."""
    assert set(got) == set(want), tag
    floor = max(float(np.max(np.abs(np.asarray(v)))) for v in want.values())
    for k in want:
        g, w = np.asarray(got[k], np.float64), np.asarray(want[k], np.float64)
        assert np.max(np.abs(g - w)) <= tol * max(float(np.max(np.abs(w))), 1e-6 * floor), (tag, k)


@pytest.mark.parametrize("B", [70, 1])
@pytest.mark.parametrize("batchnorm", [True, False])
@pytest.mark.parametrize("ae_type", O.AE_TYPES)
def test_chunked_reference_equals_unchunked_and_oracle(ae_type, batchnorm, B):
    G = 203
    X, Y, sf = _problem(B, G, 3)
    p0 = _nontrivial(O.init_params(G, G, HIDDEN, ae_type, batchnorm, seed=1, dtype=np.float64), 2)
    T = lambda a: torch.tensor(a, dtype=torch.float64)
    one = TorchRefNet(p0, HIDDEN, ae_type, batchnorm, ridge=0.02, dtype=torch.float64)
    l1, g1, s1 = one.loss_and_grads(T(X), T(Y), T(sf))
    chunked = TorchRefNet(p0, HIDDEN, ae_type, batchnorm, ridge=0.02, dtype=torch.float64)
    l2, g2, s2 = chunked.loss_and_grads_chunked(T(X), T(Y), T(sf), chunk=16)
    assert abs(l2 - l1) <= 1e-12 * abs(l1)
    _assert_grads_close({k: v.numpy() for k, v in g2.items()}, {k: v.numpy() for k, v in g1.items()}, 1e-12, "chunked")
    assert [n for n, _, _ in s1] == [n for n, _, _ in s2]
    for (_, m1, v1), (_, m2, v2) in zip(s1, s2):
        assert torch.equal(m1, m2) and torch.equal(v1, v2)
    net = O.OracleNet(G, G, HIDDEN, ae_type, batchnorm, ridge=0.02, dtype=np.float64, params=p0)
    lo, go = net.loss_and_grads(X, Y, sf, update_bn=False)
    assert abs(l2 - lo) <= 1e-9 * abs(lo)
    _assert_grads_close({k: v.numpy() for k, v in g2.items()}, go, 1e-9, "oracle")


@pytest.mark.parametrize("ae_type", ["zinb-shared", "zinb-fork", "poisson"])
@pytest.mark.parametrize("B", [70, 1])
def test_chunked_extra_reference_equals_unchunked(ae_type, B):
    """Per-cell heads (zinb-shared), one decoder layer per head (zinb-fork: three leaves), and the poisson mean over
    the non-NaN targets of the whole batch."""
    G = 203
    X, Y, sf = _problem(B, G, 5)
    if ae_type == "poisson":
        Y[0, 3] = np.nan; Y[-1, 10:14] = np.nan
    p0 = _nontrivial(extra_init_params(G, G, HIDDEN, ae_type, True, seed=4, dtype="float64"), 6)
    T = lambda a: torch.tensor(a, dtype=torch.float64)
    l1, g1, _ = TorchExtraNet(p0, HIDDEN, ae_type, True, ridge=0.02).loss_and_grads(T(X), T(Y), T(sf))
    l2, g2, _ = TorchExtraNet(p0, HIDDEN, ae_type, True, ridge=0.02).loss_and_grads_chunked(T(X), T(Y), T(sf), chunk=16)
    assert np.isfinite(l1) and abs(l2 - l1) <= 1e-12 * abs(l1)
    _assert_grads_close({k: v.numpy() for k, v in g2.items()}, {k: v.numpy() for k, v in g1.items()}, 1e-12, ae_type)


@pytest.mark.parametrize("side", ["both", "encoder", "heads", "none"])
@pytest.mark.parametrize("batchnorm", [True, False])
@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "nb"])
def test_same_rounding_reference_equals_oracle(ae_type, batchnorm, side):
    """TorchRefNet(emulate_bf16=side), the same-rounding reference of the tensor-core path for every activation and
    dropout, rounds exactly where OracleNet(emulate_bf16=side)'s closed form does for relu models: the same loss and
    gradients, in one piece and in row chunks.  The rounding is visible: "both" is far from the exact statement."""
    G, B = 48, 70
    X, Y, sf = _problem(B, G, 9)
    p0 = _nontrivial(O.init_params(G, G, HIDDEN, ae_type, batchnorm, seed=3, dtype=np.float64), 4)
    net = O.OracleNet(G, G, HIDDEN, ae_type, batchnorm, dtype=np.float64, params=p0, emulate_bf16=side)
    oloss, og = net.loss_and_grads(X, Y, sf, update_bn=False)
    T = lambda a: torch.tensor(a, dtype=torch.float64)
    ref = TorchRefNet(p0, HIDDEN, ae_type, batchnorm, dtype=torch.float64, emulate_bf16=side)
    for tag, (loss, g, _) in (("one piece", ref.loss_and_grads(T(X), T(Y), T(sf))),
                              ("chunked", ref.loss_and_grads_chunked(T(X), T(Y), T(sf), chunk=16))):
        assert abs(loss - oloss) <= 1e-10 * abs(oloss), (side, tag, loss, oloss)
        # hidden biases in front of a BatchNorm are zero in exact arithmetic: the two float64 evaluations leave ~1e-17
        floor = 1e-4 * max(float(np.max(np.abs(v))) for v in og.values())
        assert set(g) == set(og), tag
        for k, w in og.items():
            err = float(np.max(np.abs(g[k].numpy().reshape(w.shape) - w)))
            assert err <= 1e-10 * max(float(np.max(np.abs(w))), floor), (side, tag, k, err)
    if side == "both":
        exact = TorchRefNet(p0, HIDDEN, ae_type, batchnorm, dtype=torch.float64)
        _, ge, _ = exact.loss_and_grads(T(X), T(Y), T(sf))
        diff = max(float((ge[k] - g[k]).abs().max() / ge[k].abs().max()) for k in ("enc0/kernel", "mean/kernel"))
        assert diff > 1e-4, diff
