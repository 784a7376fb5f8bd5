"""Hidden activations other than relu, PReLU's trainable slopes and dropout (input + hidden) through the C ABI against the
float64 AUTOGRAD statement of the same network (oracle/torch_ref.py) -- autograd plays the role TF autodiff plays in the
reference.  Dropout masks are a counter-based stream (dca_dropout_mask_host reproduces the mask of any layer / step), so
the oracle applies exactly the mask the device applied: the comparison is element-exact, not distributional.
Reference behaviour: dca/network.py:98-99 (input dropout), :129-138 (activation layer, hidden dropout), :41; the CLI
flags --activation / --dropoutrate / --inputdropout.  Needs an H100: -m gpu."""
import ctypes as C

import numpy as np
import pytest
import torch

from dca_b200 import _lib
from oracle import dca_oracle as O
from oracle.torch_ref import TorchRefNet, TorchExtraNet, extra_init_params
from tests.util import synth_counts, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ACTS = [a for a in sorted(_lib.ACTIVATION_IDS) if a != "relu"]
T = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64)


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


def _mask(seed, step, layer, shape, rate):
    n = int(np.prod(shape))
    m = np.empty(n, np.uint8)
    assert _lib.load().dca_dropout_mask_host(C.c_uint64(seed), C.c_uint64(step), layer, n, C.c_float(rate),
                                             m.ctypes.data_as(C.c_void_p)) == 0
    return torch.tensor(m.reshape(shape), dtype=torch.float64)


def _params(G, hidden, ae_type, batchnorm, activation, seed=0, extra=False):
    p0 = (extra_init_params if extra else O.init_params)(G, G, hidden, ae_type, batchnorm, seed=seed)
    rng = np.random.default_rng(seed + 1)
    for k in list(p0):
        if k.endswith(("/bias", "/bn_beta", "/theta")):
            p0[k] = rng.normal(0, 0.2, p0[k].shape).astype(np.float32)
    if activation == "PReLU":                      # Keras initialises the slopes to 0; non-zero values exercise both gradients
        names = [k[: -len("/kernel")] for k in p0 if k.endswith("/kernel") and not k.startswith(("mean", "dispersion", "pi"))]
        for nm in names:
            p0[nm + "_act/alpha"] = rng.uniform(-0.2, 0.4, p0[nm + "/bias"].shape).astype(np.float32)
    return p0


def _engine(G, hidden, ae_type, batchnorm, B, p0, **kw):
    from dca_b200.engine import DeviceEngine
    eng = DeviceEngine(G, G, hidden, ae_type, batchnorm, max_batch=B, seed=None, **kw)
    trainable = sorted(k for k in p0 if not k.endswith(("moving_mean", "moving_var")))
    assert sorted(n for n, *_ in eng.param_info) == trainable, (sorted(n for n, *_ in eng.param_info), trainable)
    eng.set_weights(p0)
    return eng


def _check_grads(eng, og, batchnorm, tol, skip_hidden_bias=True):
    g = eng.grads.cpu().numpy()
    for name, off, r, c in eng.param_info:
        ref = og[name].numpy().reshape(-1); got = g[off: off + r * c]
        if skip_hidden_bias and name.endswith("/bias") and batchnorm and not name.startswith(("mean", "dispersion", "pi")):
            assert np.max(np.abs(got)) < 1e-5          # BatchNorm removes the Dense bias from the loss
            continue
        if np.max(np.abs(ref)) < 1e-8:                 # structurally zero (e.g. a linear layer's beta in front of another BatchNorm)
            assert np.max(np.abs(got)) < 1e-6, name
            continue
        assert rel_err(got, ref, 2e-3) < tol, (name, rel_err(got, ref, 2e-3))


@pytest.mark.parametrize("activation", ACTS)
@pytest.mark.parametrize("batchnorm", [True, False])
def test_activation_train_step_vs_autograd(activation, batchnorm):
    B, G, hidden = 96, 160, (24, 8, 24)
    Y = synth_counts(B + 16, G, 3); X, sf = O.normalize_inputs(Y)
    rows = np.random.default_rng(0).permutation(B + 16)[:B].astype(np.int32)
    p0 = _params(G, hidden, "zinb-conddisp", batchnorm, activation)
    if activation == "exponential":      # exp(.) hidden units drive the heads into their clips (mu 2e6, theta 1e-4), where the
        for k in p0:                     # reference's own float32 formula is 1e-3 off its float64 value (the engine agrees
            if k.endswith("/kernel"): p0[k] *= 0.05     # with the float32 evaluation to 1e-7 there): stay inside the clips
    net = TorchRefNet(p0, hidden, "zinb-conddisp", batchnorm, ridge=0.01, dtype=torch.float64, activation=activation)
    eng = _engine(G, hidden, "zinb-conddisp", batchnorm, B, p0, ridge=0.01, gemm_path="generic", activation=activation)
    eng.train_step(_t(X), _t(Y), _t(sf), rows=torch.as_tensor(rows).to(DEV))
    oloss, og, _ = net.loss_and_grads(T(X[rows]), T(Y[rows]), T(sf[rows]))
    assert abs(eng.read_loss() - oloss) < 1e-4 * abs(oloss), (activation, eng.read_loss(), oloss)
    _check_grads(eng, og, batchnorm, 3e-3)


def test_prelu_slopes_are_named_and_trained_like_keras():
    """keras.layers.PReLU(name='<layer>_act') owns one zero-initialised slope per unit; RMSprop updates it."""
    from dca_b200.engine import DeviceEngine
    B, G, hidden = 64, 96, (16, 4, 16)
    eng = DeviceEngine(G, G, hidden, "nb", True, max_batch=B, seed=3, activation="PReLU", gemm_path="generic")
    w = eng.get_weights()
    for nm in ("enc0", "center", "dec1"):
        assert nm + "_act/alpha" in w and not w[nm + "_act/alpha"].any()
    Y = synth_counts(B, G, 5); X, sf = O.normalize_inputs(Y)
    net = TorchRefNet(w, hidden, "nb", True, dtype=torch.float64, activation="PReLU")
    for _ in range(4):                                   # the 2nd+ steps replay the captured graph
        eng.train_step(_t(X), _t(Y), _t(sf)); eng.apply_update(1e-3, 5.0)
        lo = net.train_step(T(X), T(Y), T(sf))
        assert abs(eng.read_loss() - lo) < 5e-4 * abs(lo)
    w2 = eng.get_weights()
    for nm in ("enc0", "center", "dec1"):
        a = w2[nm + "_act/alpha"]; ref = net.p[nm + "_act/alpha"].detach().numpy()
        assert np.abs(a).max() > 1e-4
        live = np.abs(ref) > 5e-4            # sign-like first RMSprop steps: units with a ~0 gradient are noise / (|noise| + eps)
        np.testing.assert_allclose(a[live], ref[live], rtol=5e-2, atol=2e-4)


@pytest.mark.parametrize("activation,batchnorm", [("relu", True), ("elu", True), ("tanh", False), ("PReLU", True)])
def test_dropout_trajectory_vs_autograd_with_the_same_masks(activation, batchnorm):
    """Input + hidden dropout over four steps (direct call, then graph replay): every step's loss and gradients equal the
    autograd statement evaluated with the masks dca_dropout_mask_host returns for that step."""
    B, G, hidden = 80, 128, (32, 8, 32)
    rates, in_rate, seed = [0.2, 0.35, 0.1], 0.25, 4242
    Y = synth_counts(B, G, 13); X, sf = O.normalize_inputs(Y)
    p0 = _params(G, hidden, "zinb-conddisp", batchnorm, activation, seed=2)
    net = TorchRefNet(p0, hidden, "zinb-conddisp", batchnorm, dtype=torch.float64, activation=activation)
    eng = _engine(G, hidden, "zinb-conddisp", batchnorm, B, p0, gemm_path="generic", activation=activation,
                  hidden_dropout=rates, input_dropout=in_rate, dropout_seed=seed)
    losses = []
    for step in range(1, 5):
        net.masks = {-1: _mask(seed, step, -1, (B, G), in_rate)}; net.rates = {-1: in_rate}
        for i, (h, r) in enumerate(zip(hidden, rates)):
            net.masks[i] = _mask(seed, step, i, (B, h), r); net.rates[i] = r
        eng.train_step(_t(X), _t(Y), _t(sf))
        oloss, og, stats = net.loss_and_grads(T(X), T(Y), T(sf))
        losses.append(eng.read_loss())
        assert abs(eng.read_loss() - oloss) < 1e-4 * abs(oloss), (step, eng.read_loss(), oloss)
        _check_grads(eng, og, batchnorm, 4e-3)
        eng.apply_update(1e-3, 5.0)
        net._apply(og, stats, 1e-3, 5.0)
    assert len(set(round(l, 6) for l in losses)) == 4          # fresh masks every step, also under graph replay
    # inference: no mask (Keras Dropout is the identity outside training)
    eng.read_epoch_acc(reset=True)
    eng.eval_step(_t(X), _t(Y), _t(sf))
    acc = eng.read_epoch_acc()
    with torch.no_grad():
        oval = float(net.loss(T(X), T(Y), T(sf), training=False)[0])
    assert abs(acc[2] / acc[3] - oval) < 3e-4 * abs(oval)


def test_dropout_on_the_tcgen05_path():
    """Flagship shape (64-wide outer layers): encoder / head GEMMs on the tensor cores read the dropped input batch and the
    dropped last hidden layer; bf16 operand rounding bounds the distance to the exact statement (DESIGN.md section 3)."""
    B, G, hidden = 256, 512, (64, 32, 64)
    rates, in_rate, seed = [0.1, 0.0, 0.2], 0.15, 99
    Y = synth_counts(B, G, 17); X, sf = O.normalize_inputs(Y)
    p0 = _params(G, hidden, "zinb-conddisp", True, "elu", seed=5)
    net = TorchRefNet(p0, hidden, "zinb-conddisp", True, dtype=torch.float64, activation="elu")
    for x_dtype, tdt in (("float32", torch.float32), ("bfloat16", torch.bfloat16)):
        eng = _engine(G, hidden, "zinb-conddisp", True, B, p0, gemm_path="tcgen05", activation="elu", hidden_dropout=rates,
                      input_dropout=in_rate, dropout_seed=seed, x_dtype=x_dtype)
        Xin = X.astype(np.float32)
        if x_dtype == "bfloat16":
            Xin = torch.tensor(Xin).to(torch.bfloat16).to(torch.float32).numpy()
        for step in (1, 2, 3):
            net.masks = {-1: _mask(seed, step, -1, (B, G), in_rate)}; net.rates = {-1: in_rate}
            for i, (h, r) in enumerate(zip(hidden, rates)):
                if r > 0: net.masks[i] = _mask(seed, step, i, (B, h), r); net.rates[i] = r
            eng.train_step(_t(Xin, tdt), _t(Y), _t(sf))
            oloss, og, _ = net.loss_and_grads(T(Xin), T(Y), T(sf))
            assert abs(eng.read_loss() - oloss) < 2e-3 * abs(oloss), (x_dtype, step, eng.read_loss(), oloss)
            g = eng.grads.cpu().numpy()
            for name, off, r, c in eng.param_info:
                if name.endswith("/kernel"):
                    ref = og[name].numpy().reshape(-1); got = g[off: off + r * c]
                    err = np.linalg.norm(got - ref) / (np.linalg.norm(ref) + 1e-30)
                    assert err < (2e-2 if name.startswith(("mean", "dispersion", "pi")) else 0.15), (x_dtype, name, err)
        eng.close()


@pytest.mark.parametrize("ae_type,activation", [("poisson", "selu"), ("zinb-fork", "LeakyReLU"), ("nb-shared", "PReLU"),
                                                ("zinb-elempi", "softplus")])
def test_extra_types_with_activation_and_dropout(ae_type, activation):
    B, G, hidden = 72, 100, (16, 8, 16)
    rates, in_rate, seed = [0.1, 0.2, 0.3], 0.2, 31
    Y = synth_counts(B + 8, G, 19); X, sf = O.normalize_inputs(Y)
    rows = np.random.default_rng(2).permutation(B + 8)[:B].astype(np.int32)
    p0 = _params(G, hidden, ae_type, True, activation, seed=4, extra=True)
    if activation == "PReLU":
        assert "enc0_act/alpha" in p0
    net = TorchExtraNet(p0, hidden, ae_type, True, activation=activation)
    eng = _engine(G, hidden, ae_type, True, B, p0, activation=activation, hidden_dropout=rates, input_dropout=in_rate,
                  dropout_seed=seed)
    for step in (1, 2, 3):
        net.masks = {-1: _mask(seed, step, -1, (B, G), in_rate)}; net.rates = {-1: in_rate}
        for i, (h, r) in enumerate(zip(hidden, rates)):
            net.masks[i] = _mask(seed, step, i, (B, h), r); net.rates[i] = r
        for b in range(3):                                         # fork branches: the last decoder layer's rate
            net.masks[8 + b] = _mask(seed, step, 8 + b, (B, hidden[-1]), rates[-1]); net.rates[8 + b] = rates[-1]
        eng.train_step(_t(X), _t(Y), _t(sf), rows=torch.as_tensor(rows).to(DEV))
        oloss, og, stats = net.loss_and_grads(T(X[rows]), T(Y[rows]), T(sf[rows]))
        assert abs(eng.read_loss() - oloss) < 1e-4 * abs(oloss), (ae_type, step, eng.read_loss(), oloss)
        _check_grads(eng, og, True, 4e-3)
        eng.apply_update(1e-3, 5.0)
        TorchRefNet._apply(net, og, stats, 1e-3, 5.0)


def test_public_api_accepts_activation_and_dropout():
    """dca(adata, activation=..., hidden_dropout=..., network_kwds={'input_dropout': ...}) -- dca/api.py:26-28,170-180;
    the reference's hyper-parameter search samples exactly these knobs (dca/hyper.py:32-37)."""
    from dca_b200.anndata_lite import AnnData
    from dca_b200.api import dca
    adata = AnnData(synth_counts(600, 120, 23))
    ret, net = dca(adata, mode="denoise", ae_type="zinb-conddisp", hidden_size=(32, 8, 32), activation="selu",
                   hidden_dropout=0.1, network_kwds={"input_dropout": 0.1}, epochs=8, batch_size=64, copy=True,
                   return_info=True, return_model=True, random_state=0)
    assert np.isfinite(ret.X).all()
    assert net.engine.activation == "selu" and net.engine.input_dropout == pytest.approx(0.1)
    hist = ret.uns["dca_loss_history"]
    assert hist["loss"][-1] < hist["loss"][0]
    with pytest.raises(NotImplementedError):
        dca(AnnData(synth_counts(100, 40, 1)), activation="softmax", epochs=1)


@pytest.mark.parametrize("optimizer", ["SGD", "Adagrad", "Adadelta", "Adam", "Adamax", "Nadam", "rmsprop"])
def test_keras_optimizers_vs_restated_update_rules(optimizer):
    """`opt.__dict__[optimizer](clipvalue=clip_grad)` (dca/train.py:54-57, CLI --optimizer): six steps with each Keras
    optimizer against the float64 restatement of keras/optimizers.py in oracle/torch_ref.py (class-default
    hyper-parameters and learning rate)."""
    from dca_b200 import _lib as L
    B, G, hidden = 64, 96, (16, 4, 16)
    Y = synth_counts(B, G, 29); X, sf = O.normalize_inputs(Y)
    p0 = _params(G, hidden, "zinb-conddisp", False, "relu", seed=6)
    net = TorchRefNet(p0, hidden, "zinb-conddisp", False, dtype=torch.float64)
    net.optimizer = {"rmsprop": "RMSprop"}.get(optimizer, optimizer)
    eng = _engine(G, hidden, "zinb-conddisp", False, B, p0, gemm_path="generic")
    lr = eng.set_optimizer(optimizer)
    assert lr == L.OPTIMIZERS[optimizer][1]
    clip = 0.02 if optimizer == "SGD" else 5.0          # exercise clipvalue where the step is proportional to the gradient
    for step in range(6):
        eng.train_step(_t(X), _t(Y), _t(sf)); eng.apply_update(lr, clip)
        lo = net.train_step(T(X), T(Y), T(sf), lr=lr, clip=clip)
        assert abs(eng.read_loss() - lo) < 2e-4 * abs(lo), (optimizer, step, eng.read_loss(), lo)
    w = eng.get_weights()
    for k in net.train_keys:
        ref = net.p[k].detach().numpy(); got = w[k].reshape(ref.shape)
        d0 = np.abs(ref - p0[k].astype(np.float64).reshape(ref.shape)).max()
        assert np.abs(got - ref).max() < 2e-2 * d0 + 1e-6, (optimizer, k, np.abs(got - ref).max(), d0)
    # a fresh optimizer forgets its state
    eng.reset_optimizer()
    assert not eng.rms.any()
    with pytest.raises(NotImplementedError):
        eng.set_optimizer("TFOptimizer")
