"""Host mirrors of the hidden-layer activation / dropout arithmetic (csrc/activations.cuh, the same source the device
kernels compile) against torch autograd and against the statistics a Bernoulli(1 - rate) mask must have.
Reference behaviour: dca/network.py:129-138 (Activation / LeakyReLU / PReLU, Dropout), :98-99 (input dropout).
CPU only: loads the C-ABI library but launches nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

from dca_b200 import _lib
from oracle.torch_ref import hidden_activation


def _act(lib, name, x, alpha=0.0):
    out = (C.c_float * 2)()
    assert lib.dca_activation_host(_lib.ACTIVATION_IDS[name], C.c_float(x), C.c_float(alpha), C.byref(out)) == 0
    return out[0], out[1]


@pytest.mark.parametrize("name", sorted(_lib.ACTIVATION_IDS))
def test_activation_value_and_derivative_match_autograd(name):
    lib = _lib.load()
    xs = np.concatenate([np.linspace(-6, 6, 49), [-30.0, -1e-3, 1e-3, 25.0]]).astype(np.float32)
    xs = xs[np.abs(xs) > 1e-6]                       # kinks at 0 are measure-zero; conventions differ between frameworks
    if name == "hard_sigmoid":
        xs = xs[np.abs(np.abs(xs) - 2.5) > 1e-3]
    alpha = 0.17
    for x in xs:
        t = torch.tensor(float(x), dtype=torch.float64, requires_grad=True)
        y = hidden_activation(name, t, torch.tensor(alpha, dtype=torch.float64))
        (g,) = torch.autograd.grad(y, t)
        v, d = _act(lib, name, float(x), alpha)
        assert abs(v - float(y)) <= 2e-6 * max(1.0, abs(float(y))), (name, x, v, float(y))
        assert abs(d - float(g)) <= 3e-6 * max(1.0, abs(float(g))), (name, x, d, float(g))


def test_unknown_activation_is_rejected():
    lib = _lib.load()
    out = (C.c_float * 2)()
    assert lib.dca_activation_host(99, C.c_float(0.5), C.c_float(0.0), C.byref(out)) != 0


def _mask(lib, seed, step, layer, n, rate):
    m = np.empty(n, np.uint8)
    assert lib.dca_dropout_mask_host(C.c_uint64(seed), C.c_uint64(step), layer, n, C.c_float(rate),
                                     m.ctypes.data_as(C.c_void_p)) == 0
    return m


def test_dropout_mask_statistics_and_streams():
    lib = _lib.load()
    n = 200_000
    for rate in (0.1, 0.5, 0.8):
        m = _mask(lib, 7, 1, 0, n, rate)
        keep = 1.0 - rate
        assert abs(m.mean() - keep) < 5 * np.sqrt(keep * rate / n)         # Bernoulli(1 - rate)
        # no serial correlation between neighbours (a counter hash, not a shifted sequence)
        a = m[:-1].astype(np.float64) - keep; b = m[1:].astype(np.float64) - keep
        assert abs((a * b).mean()) < 5 * keep * rate / np.sqrt(n)
    base = _mask(lib, 7, 1, 0, n, 0.5)
    assert np.array_equal(base, _mask(lib, 7, 1, 0, n, 0.5))              # deterministic
    for other in (_mask(lib, 8, 1, 0, n, 0.5), _mask(lib, 7, 2, 0, n, 0.5), _mask(lib, 7, 1, 1, n, 0.5),
                  _mask(lib, 7, 1, -1, n, 0.5)):
        assert abs((base == other).mean() - 0.5) < 0.01                     # independent streams per seed / step / layer
    assert _mask(lib, 1, 1, 0, 1000, 0.0).all()                            # rate 0 keeps everything
    assert lib.dca_dropout_mask_host(C.c_uint64(1), C.c_uint64(1), 0, 10, C.c_float(1.0), base.ctypes.data_as(C.c_void_p)) != 0


def test_config_carries_activation_and_dropout_fields():
    cfg = _lib.default_config()
    assert cfg.activation == 0 and cfg.input_dropout == 0.0 and all(cfg.hidden_dropout[i] == 0.0 for i in range(_lib.DCA_MAX_HIDDEN))
    lib = _lib.load()
    nbytes = C.c_size_t()
    cfg.n_in = cfg.n_out = 40; cfg.max_batch = 8
    assert lib.dca_arena_bytes(C.byref(cfg), C.byref(nbytes)) == 0
    base = nbytes.value
    cfg.activation = _lib.ACTIVATION_IDS["PReLU"]; cfg.input_dropout = 0.2
    assert lib.dca_arena_bytes(C.byref(cfg), C.byref(nbytes)) == 0 and nbytes.value > base   # slope scratch + dropped input
    cfg.activation = 12
    assert lib.dca_arena_bytes(C.byref(cfg), C.byref(nbytes)) != 0
    cfg.activation = 0; cfg.hidden_dropout[1] = 1.0
    assert lib.dca_arena_bytes(C.byref(cfg), C.byref(nbytes)) != 0
    cfg.hidden_dropout[1] = 0.0; cfg.activation = _lib.ACTIVATION_IDS["PReLU"]; cfg.ae_type = _lib.AE_TYPE_IDS["nb-fork"]
    assert lib.dca_arena_bytes(C.byref(cfg), C.byref(nbytes)) != 0         # Activation('PReLU') does not exist in Keras


def test_dropout_mask_known_answers():
    """Pins the mask generator (constants of the 64-bit mix, key derivation, 24-bit threshold): a run with the same
    `random_state` must draw the same masks in a later version of the library.  Bit i of the word = keep flag of element i."""
    lib = _lib.load()
    kat = {(7, 1, 0, 0.5): 0xa072e29d8ef8d62c, (7, 1, -1, 0.25): 0x726fbf93e775fdbe, (12345678901234567, 3, 8, 0.8): 0x20340000460401}
    for (seed, step, layer, rate), want in kat.items():
        m = _mask(lib, seed, step, layer, 64, rate)
        got = sum(int(b) << i for i, b in enumerate(m))
        assert got == want, (seed, step, layer, rate, hex(got))


def _bwd(lib, name, x, rate, kept, g=1.0, alpha=0.0):
    out = (C.c_float * 2)()
    assert lib.dca_activation_bwd_host(_lib.ACTIVATION_IDS[name], C.c_float(x), C.c_float(alpha), C.c_float(rate), kept,
                                       C.c_float(g), C.byref(out)) == 0
    return out[0], out[1]


@pytest.mark.parametrize("rate", [0.01, 0.11, 0.15, 0.23, 0.77])
def test_saturated_hard_sigmoid_has_no_gradient_under_dropout(rate):
    """hard_sigmoid is flat outside (-2.5, 2.5).  At these rates the stored output of a saturated, kept unit times keep
    is 1 - 2^-24 in fp32, not 1: the backward element must take the slope from the input, not from that value."""
    lib = _lib.load()
    keep = np.float32(1) - np.float32(rate)
    assert (np.float32(1) / keep) * keep != np.float32(1)              # the rounding this case is about
    for x in (2.6, 3.0, 7.5, -2.6, -9.0):
        h, dx = _bwd(lib, "hard_sigmoid", x, rate, 1, g=0.75)
        assert h == np.float32(1) / keep if x > 0 else h == 0.0, (x, h)
        assert dx == 0.0, (rate, x, dx)
    for x in (-2.4, -0.3, 0.0, 1.1, 2.4):                              # the linear part: 0.2 g / keep
        h, dx = _bwd(lib, "hard_sigmoid", x, rate, 1, g=0.75)
        assert dx == pytest.approx(0.2 * 0.75 / (1 - rate), rel=1e-6), (rate, x, dx)
        assert _bwd(lib, "hard_sigmoid", x, rate, 0, g=0.75) == (0.0, 0.0)      # dropped


@pytest.mark.parametrize("name", sorted(_lib.ACTIVATION_IDS))
def test_backward_element_matches_autograd_through_dropout(name):
    """dca_activation_bwd_host (the element act_bwd_kernel computes) against autograd of dropout(act(x)) in float64."""
    lib = _lib.load()
    xs = np.array([-4.0, -2.6, -1.3, -0.2, 0.3, 1.7, 2.6, 4.5], np.float32)
    alpha = 0.17
    for rate in (0.0, 0.11, 0.77):
        for kept in (1, 0) if rate > 0 else (1,):
            for x in xs:
                t = torch.tensor(float(x), dtype=torch.float64, requires_grad=True)
                y = hidden_activation(name, t, torch.tensor(alpha, dtype=torch.float64)) * kept / (1.0 - rate)
                (gref,) = torch.autograd.grad(y * 0.6, t)
                h, dx = _bwd(lib, name, float(x), rate, kept, g=0.6, alpha=alpha)
                assert abs(h - float(y)) <= 2e-6 * max(1.0, abs(float(y))), (name, rate, kept, x, h, float(y))
                assert abs(dx - float(gref)) <= 3e-6 * max(1.0, abs(float(gref))), (name, rate, kept, x, dx, float(gref))
