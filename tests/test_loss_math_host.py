"""The per-element arithmetic of the CUDA loss kernel (dca_b200/csrc/zinb_math.cuh), compiled for
the host and exported as dca_zinb_elem_host, against the float64 oracle.  Runs without a GPU."""
import ctypes as C
import numpy as np
import pytest

from oracle import dca_oracle as O
from dca_b200 import _lib


def _host_elem(ae_type, y, m, sf, d, pi, ridge, kernel_variant=False):
    lib = _lib.load()
    out = (C.c_float * 4)()
    res = np.zeros((len(y), 4), np.float32)
    t = _lib.AE_TYPE_IDS[ae_type] | ({False: 0, "ring": 0x200}[kernel_variant])
    for i in range(len(y)):
        assert lib.dca_zinb_elem_host(t, float(y[i]), float(m[i]), float(sf[i]), float(d[i]), float(pi[i]),
                                      float(ridge), C.byref(out)) == 0
        res[i] = list(out)
    return res


def _oracle_elem(ae_type, y, m, sf, d, pi, ridge):
    """Oracle element loss and gradients w.r.t. pre-activations given POST-activation values
    strictly inside the clip ranges (so the activation chain factors are well defined)."""
    y, m, sf, d, pi = [np.asarray(a, np.float64) for a in (y, m, sf, d, pi)]
    mu = m * sf
    has_pi = ae_type.startswith("zinb")
    cond = ae_type.endswith("conddisp")
    if has_pi:
        el = O.zinb_loss_elem(y, mu, d, pi, ridge)
        dmu, dth, dpi = O.loss_partials(y, mu, d, pi, ridge)
    else:
        el = O.nb_loss_elem(y, mu, d)
        dmu, dth, _ = O.loss_partials(y, mu, d)
        dpi = np.zeros_like(y)
    gm = dmu * mu * ((m > 1e-5) & (m < 1e6))
    gd = dth * (1.0 - np.exp(-d)) * ((d > 1e-4) & (d < 1e4)) if cond else dth
    gp = dpi * pi * (1 - pi) if has_pi else np.zeros_like(y)
    return np.stack([el, gm, gd, gp], 1)


def _cases(n, seed):
    rng = np.random.default_rng(seed)
    y = rng.poisson(rng.gamma(0.7, 3.0, n)).astype(np.float64)
    y[rng.random(n) < 0.5] = 0
    y[:8] = [0, 1, 2, 16, 17, 40, 1000, 30000]
    m = np.exp(rng.normal(0, 2.5, n))
    sf = np.exp(rng.normal(0, 0.4, n))
    d = np.exp(rng.normal(0, 2.5, n)).clip(2e-4, 9e3)
    pi = 1 / (1 + np.exp(-rng.normal(0, 3, n)))
    return y, m, sf, d, pi


@pytest.mark.parametrize("ae_type", O.AE_TYPES)
def test_host_math_matches_oracle(ae_type):
    y, m, sf, d, pi = _cases(3000, 7)
    # the kernel sees float32 inputs: evaluate the oracle at the float32-rounded values
    y, m, sf, d, pi = [a.astype(np.float32).astype(np.float64) for a in (y, m, sf, d, pi)]
    got = _host_elem(ae_type, y, m, sf, d, pi, 0.05).astype(np.float64)
    ref = _oracle_elem(ae_type, y, m, sf, d, pi, 0.05)
    names = ["loss", "dzm", "dzd", "dzp"]
    for j in range(4):
        scale = np.maximum(np.abs(ref[:, j]), 1e-3 * np.max(np.abs(ref[:, j])) + 1e-30)
        err = np.abs(got[:, j] - ref[:, j]) / scale
        k = int(np.argmax(err))
        assert err[k] < 2e-4, "%s %s: rel err %.3g at y=%g m=%g sf=%g d=%g pi=%g got=%g ref=%g" % (
            ae_type, names[j], err[k], y[k], m[k], sf[k], d[k], pi[k], got[k, j], ref[k, j])


def test_host_math_clip_bounds():
    """Values AT the clip bounds: zero gradient through the clipped activation (tf.clip_by_value)."""
    y = np.array([0, 3, 0, 3.0]); sf = np.ones(4)
    m = np.array([1e-5, 1e-5, 1e6, 1e6], np.float32).astype(np.float64)
    d = np.array([1e-4, 1e4, 1e-4, 1e4], np.float32).astype(np.float64)
    pi = np.array([0.3, 0.6, 0.0, 1.0])
    got = _host_elem("zinb-conddisp", y, m, sf, d, pi, 0.0)
    assert np.all(got[:, 1] == 0) and np.all(got[:, 2] == 0)
    assert np.all(np.isfinite(got))
    ref = O.zinb_loss_elem(y, m * sf, d, pi)
    np.testing.assert_allclose(got[:, 0], ref, rtol=2e-4, atol=1e-5)


@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "zinb"])
@pytest.mark.parametrize("ridge", [0.0, 0.05])
def test_ring_formulation_equals_the_reference_formulation(ae_type, ridge):
    """The formulation of the ring and heads + loss kernels (zinb_zero_pair, zinb_nb_raw, finish_factors_pair) returns
    what the plain per-element function returns -- including the series / MUFU switch points (q = 1/16, d = 1/32), the
    clip bounds and rows with extreme size factors."""
    y, m, sf, d, pi = _cases(4000, 11)
    m[:6] = [1e-5, 1e6, 2e-5, 5e5, 1.0, 1.0]; d[:6] = [1e-4, 1e4, 0.03125, 0.031, 0.0313, 9e3]
    sf[6:10] = [1e-3, 1e3, 1.0, 1.0]
    # q = mu / (theta + mu) around 1/16
    m[10:14] = [1.0 / 15.0, 0.0666, 0.0667, 0.07]; sf[10:14] = 1.0; d[10:14] = 1.0; y[10:14] = 0
    y, m, sf, d, pi = [a.astype(np.float32).astype(np.float64) for a in (y, m, sf, d, pi)]
    a = _host_elem(ae_type, y, m, sf, d, pi, ridge).astype(np.float64)
    # "ring": the f32x2 pair functions, the masked rising-product groups and the shared finishing factors of
    # zinb_loss_bwd_ring_kernel and heads_loss_kernel
    b = _host_elem(ae_type, y, m, sf, d, pi, ridge, kernel_variant="ring").astype(np.float64)
    assert np.all(np.isfinite(a) == np.isfinite(b))
    fin = np.isfinite(a)
    scale = np.maximum(np.abs(a), 1e-3 * np.max(np.abs(np.where(fin, a, 0.0)), axis=0, keepdims=True) + 1e-30)
    err = np.where(fin, np.abs(a - b) / scale, 0.0)
    k = np.unravel_index(int(np.argmax(err)), err.shape)
    assert err[k] <= 2e-5, (ae_type, ridge, k, a[k], b[k], y[k[0]], m[k[0]], sf[k[0]], d[k[0]], pi[k[0]])


@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "zinb"])
def test_ring_kernel_formulation_matches_oracle(ae_type):
    """The default loss kernel's formulation (variant 0x200) straight against the float64 oracle, with the counts that
    walk every path of the masked rising product (1..4 one group, 5..16 further groups, > 16 / non-integer Stirling)."""
    y, m, sf, d, pi = _cases(3000, 13)
    y[8:30] = [3, 4, 5, 6, 7, 8, 9, 12, 13, 15, 16, 17, 18, 2.5, 0.5, 100, 63, 64, 65, 5000, 1, 2]
    y, m, sf, d, pi = [a.astype(np.float32).astype(np.float64) for a in (y, m, sf, d, pi)]
    got = _host_elem(ae_type, y, m, sf, d, pi, 0.05, kernel_variant="ring").astype(np.float64)
    ref = _oracle_elem(ae_type, y, m, sf, d, pi, 0.05)
    for j, nm in enumerate(["loss", "dzm", "dzd", "dzp"]):
        scale = np.maximum(np.abs(ref[:, j]), 1e-3 * np.max(np.abs(ref[:, j])) + 1e-30)
        err = np.abs(got[:, j] - ref[:, j]) / scale
        k = int(np.argmax(err))
        assert err[k] < 2e-4, "%s %s: rel err %.3g at y=%g m=%g sf=%g d=%g pi=%g got=%g ref=%g" % (
            ae_type, nm, err[k], y[k], m[k], sf[k], d[k], pi[k], got[k, j], ref[k, j])
