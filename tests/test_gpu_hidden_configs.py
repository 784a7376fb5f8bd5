"""Everything a user can choose for the hidden layers, at real sizes, on every GEMM path: --hiddensize (one to eight
layers, widths 1 to 128), --activation (all twelve), --dropoutrate, --inputdropout, batchnorm on and off and PReLU's
slopes -- against the float64 autograd reference (oracle/torch_ref.py) on the same device, its head and loss graph
evaluated in row chunks, with the dropout masks the device drew (dca_dropout_mask_host).

Which path a case takes is decided by the widths and asserted from DeviceEngine.info():
  * first width 64 / last width 64 (G % 8 == 0): the tensor-core encoder / heads.  They round their GEMM operands to
    bf16, so the reference rounds at the same points (TorchRefNet(emulate_bf16=...), DESIGN section 3) and the bounds
    are those the relu model meets at the same shape (test_gpu_parity._assert_step_bounds): loss 1e-4 relative, head
    gradients 3e-3 and hidden-stack gradients 3e-2 of the tensor's largest element (the hidden ones sit behind the
    bf16 rounding of dA of the first layer: an fp32 ulp upstream can move one element of dW1 by 2^-9 of its size).
  * any other first / last width: the fp32 split-K GEMMs, against the exact float64 statement: loss 1e-4 relative,
    every gradient rel_err(got, ref, 2e-3) < 2e-3, predict outputs 5e-4 relative (test_gpu_ragged_genes).
  * the fused hidden stack (mid_stack.cu, one launch) only for relu without dropout, widths <= 64 and B <= 8192; any
    other model or batch runs the per-layer kernels.

Reference behaviour: dca/network.py:92-141 (hidden stack), dca/hyper.py:27-37 (the search grid), dca/__main__.py
(--activation, --dropoutrate, --inputdropout, --hiddensize).  Every tensor's worst error is printed (-s), as is each
case's peak device memory and wall time.  Needs an H100: -m gpu."""
import ctypes as C
import functools
import gc
import time

import numpy as np
import pytest
import torch

from dca_b200 import _lib
from oracle import dca_oracle as O
from oracle.torch_ref import TorchRefNet, hidden_activation, apply_dropout
from tests.util import synth_counts

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
AE = "zinb-conddisp"
EXTRA = 300                         # each batch is gathered from a dataset this many rows larger
LOSS_TOL, GRAD_TOL, GRAD_FLOOR, PRED_TOL = 1e-4, 2e-3, 2e-3, 5e-4
# tensor-core path: max |got - ref| / max |ref| per tensor against the same-rounding reference (module docstring)
TC_HEAD_TOL, TC_HIDDEN_TOL = 3e-3, 3e-2
# tensor-core predict against the same-rounding reference: the bf16 rounding of the last hidden activation can land on
# the other side of a rounding boundary when fp32 sums differ in their last bit (2^-9 of one operand of one head sum)
TC_PRED_TOL = 2e-3
# Gradients that are zero in exact arithmetic (hidden biases in front of a BatchNorm; at B = 1 with BatchNorm everything
# upstream of the last BatchNorm): fp32 leaves the rounding of B terms of a sum whose exact value is 0, far below 1e-5
# of the step's largest gradient.
ZERO_TOL = 1e-5
# BatchNorm statistics recovered from the moving averages m' = mom * m + (1 - mom) * s: the fp32 rounding of m' (2^-24
# of |m|) becomes 100x larger in s, so the error is taken relative to max |s| + max |m|.
BN_TOL = 1e-3
PEAK_BUDGET = 16 << 30
HIDDEN_RATE, INPUT_RATE = 0.11, 0.23
HEAD_LAYERS = ("mean", "dispersion", "pi")


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


def _chunk(G):
    return max(256, 5_000_000 // G)            # reference rows per head / loss chunk: ~1.5 GB of float64 graph at most


@functools.lru_cache(maxsize=2)
def _dataset(G):
    """Normalised synthetic counts with enough rows for the largest batch of this gene count (host arrays)."""
    N = (8200 if G < 10000 else 4096) + EXTRA
    Y = synth_counts(N, G, 2000 + G)
    X, sf = O.normalize_inputs(Y)
    return X, Y, sf


def _batch(G, B, x_dtype=torch.float32):
    """Device X, Y, sf of a dataset B + 300 rows long and a permuted int32 gather of B of its rows."""
    X, Y, sf = _dataset(G)
    N = B + EXTRA
    rows = np.random.default_rng(B).permutation(N)[:B].astype(np.int32)
    return _t(X[:N], x_dtype), _t(Y[:N]), _t(sf[:N]), torch.as_tensor(rows).to(DEV)


def _params(G, hidden, batchnorm, activation, seed=0):
    """Glorot kernels; random non-zero biases, betas and dispersions; PReLU slopes of both signs.  hard_sigmoid: biases
    and betas of U(-3.5, 3.5), so that a good share of every layer's units sits on either flat part.  exponential:
    kernels scaled by 0.05 so that exp(.) units keep the heads inside their clips (test_gpu_activations)."""
    p0 = O.init_params(G, G, hidden, AE, batchnorm, seed=seed, dtype=np.float32)
    rng = np.random.default_rng(seed + 1)
    for k in list(p0):
        if k.endswith(("/bias", "/bn_beta", "/theta")):
            hidden_layer = not k.startswith(HEAD_LAYERS)
            if activation == "hard_sigmoid" and hidden_layer:
                p0[k] = rng.uniform(-3.5, 3.5, p0[k].shape).astype(np.float32)
            else:
                p0[k] = rng.normal(0, 0.2, p0[k].shape).astype(np.float32)
        if activation == "exponential" and k.endswith("/kernel"):
            p0[k] = p0[k] * np.float32(0.05)
    if activation == "PReLU":
        for nm in O.layer_names(len(hidden)):
            p0[nm + "_act/alpha"] = rng.uniform(-0.2, 0.4, p0[nm + "/bias"].shape).astype(np.float32)
    return p0


def _engine(G, hidden, batchnorm, B, p0, activation="relu", rates=None, in_rate=0.0, seed=77, **kw):
    from dca_b200.engine import DeviceEngine
    eng = DeviceEngine(G, G, hidden, AE, batchnorm, max_batch=B, seed=None, activation=activation,
                       hidden_dropout=list(rates) if rates else 0.0, input_dropout=in_rate, dropout_seed=seed, **kw)
    eng.set_weights(p0)
    return eng


def _expect_path(eng, hidden, activation, dropout, B, gemm_path="auto"):
    """The path the widths and the model select; asserted so that a change of the selection is noticed here.  The
    tensor-core heads read their kernels in place from the flat bf16 parameter copy, whose TMA base must be 16-byte
    aligned: with inner widths that put a head kernel at an offset off a multiple of 8 parameters the heads run on the
    fp32 path (and are compared as such)."""
    info = eng.info()
    tc = gemm_path != "generic"
    off = {name: o for name, o, *_ in eng.param_info}
    aligned = all(off[k] % 8 == 0 for k in ("mean/kernel", "dispersion/kernel", "pi/kernel"))
    want = {"tc_encoder": tc and hidden[0] == 64, "tc_heads": tc and hidden[-1] == 64 and aligned,
            "fused_hidden": activation == "relu" and not dropout and max(hidden) <= 64 and B <= 8192}
    got = {k: info[k] for k in want}
    assert got == want, (hidden, activation, dropout, B, info)
    return got


def _side(path):
    return {(True, True): "both", (True, False): "encoder", (False, True): "heads", (False, False): "none"}[
        (path["tc_encoder"], path["tc_heads"])]


def _mask(seed, step, layer, shape, rate):
    n = int(np.prod(shape))
    m = np.empty(n, np.uint8)
    assert _lib.load().dca_dropout_mask_host(C.c_uint64(seed), C.c_uint64(step), layer, n, C.c_float(rate),
                                             m.ctypes.data_as(C.c_void_p)) == 0
    return torch.from_numpy(m.reshape(shape)).to(DEV, torch.float64)


def _set_masks(ref, seed, step, B, G, hidden, rates, in_rate):
    """The masks the device applies at training step `step` (1 = the engine's first train_step)."""
    ref.masks, ref.rates = {}, {}
    if in_rate > 0:
        ref.masks[-1] = _mask(seed, step, -1, (B, G), in_rate); ref.rates[-1] = in_rate
    for i, (h, r) in enumerate(zip(hidden, rates or [0.0] * len(hidden))):
        if r > 0:
            ref.masks[i] = _mask(seed, step, i, (B, h), r); ref.rates[i] = r


@pytest.fixture(autouse=True)
def _device_budget(request):
    """Each case frees its engine and tensors before the next; peak device memory and wall time are printed."""
    gc.collect(); torch.cuda.empty_cache()
    torch.empty(1, device=DEV)                           # the allocator's statistics exist once it has allocated
    torch.cuda.reset_peak_memory_stats(DEV)
    t0 = time.perf_counter()
    yield
    peak = torch.cuda.max_memory_allocated(DEV)
    print("[%s] peak device memory %.2f GB, %.1f s" % (request.node.name, peak / 1e9, time.perf_counter() - t0))
    gc.collect(); torch.cuda.empty_cache()
    assert peak < PEAK_BUDGET, peak


def _check_grads(tag, g, param_info, og, tc):
    """Every gradient tensor against the reference; prints the worst error of each.  Tensors whose reference is zero
    (<= 1e-10 of the step's largest gradient: exact zeros left as float64 rounding) are held to ZERO_TOL of that."""
    ref = {k: v.detach().double().cpu().numpy().reshape(-1) for k, v in og.items()}
    scale = max(float(np.max(np.abs(v))) for v in ref.values())
    bad = []
    for name, off, r, c in param_info:
        got = g[off: off + r * c].astype(np.float64); want = ref[name]
        head = name.startswith(HEAD_LAYERS)
        if np.max(np.abs(want)) <= 1e-10 * scale:
            err = float(np.max(np.abs(got))) / scale
            print("  %-20s zero: |got| %.2e of the largest gradient" % (name, err))
            ok = err < ZERO_TOL
        elif tc["tc_heads"] or (tc["tc_encoder"] and not head):
            # behind a bf16 rounding (heads: dZ and H; hidden stack: dA1, or the rounded dZ the heads pass down)
            err = float(np.max(np.abs(got - want)) / np.max(np.abs(want)))
            print("  %-20s max err %.2e of its largest element (same rounding)" % (name, err))
            ok = err < (TC_HEAD_TOL if head else TC_HIDDEN_TOL)
        else:
            e = np.abs(got - want) / np.maximum(np.abs(want), GRAD_FLOOR * np.max(np.abs(want)))
            i = int(np.argmax(e)); err = float(e[i])
            print("  %-20s rel_err %.2e at %s (got %.6e, ref %.6e)" % (name, err, np.unravel_index(i, (r, c)), got[i], want[i]))
            ok = err < GRAD_TOL
        if not ok:
            bad.append((name, err))
    assert not bad, (tag, bad)


def _bn_error(w0, w1, stats):
    mom = O.KERAS_DEFAULTS["bn_momentum"]
    err = 0.0
    for nm, mean, var in stats:
        for key, s in (("mean", mean), ("var", var)):
            k = "%s/bn_moving_%s" % (nm, key)
            s_ref = s.double().cpu().numpy()
            s_got = (w1[k].astype(np.float64) - mom * w0[k]) / (1 - mom)
            err = max(err, float(np.max(np.abs(s_got - s_ref)) / (np.max(np.abs(s_ref)) + np.max(np.abs(w0[k])))))
    return err


def _load(ref, w):
    """The reference at the engine's weights and moving statistics."""
    with torch.no_grad():
        for k, v in w.items():
            ref.p[k].copy_(torch.as_tensor(v).reshape(ref.p[k].shape))


def _step(tag, eng, ref, data, path, batchnorm):
    """One engine training step against the reference (its masks already set): loss, every gradient tensor and the
    BatchNorm batch statistics the step folds into the moving averages."""
    Xd, Yd, sfd, rd = data
    w0 = eng.get_weights()
    _load(ref, w0)
    eng.train_step(Xd, Yd, sfd, rows=rd)
    loss = eng.read_loss()
    g = eng.grads.cpu().numpy()
    w1 = eng.get_weights()
    rl = rd.long()
    oloss, og, stats = ref.loss_and_grads_chunked(Xd[rl].double(), Yd[rl].double(), sfd[rl].double(),
                                                  chunk=_chunk(Yd.shape[1]))
    bn_err = _bn_error(w0, w1, stats) if batchnorm else 0.0
    print("\n[%s] path %s: loss %.6f ref %.6f rel %.2e, batch statistics %.2e"
          % (tag, path, loss, oloss, abs(loss - oloss) / abs(oloss), bn_err))
    _check_grads(tag, g, eng.param_info, og, path)
    assert abs(loss - oloss) < LOSS_TOL * abs(oloss), (tag, loss, oloss)
    assert bn_err < BN_TOL, (tag, bn_err)
    return loss


def _eval_and_predict(tag, eng, ref, data, path):
    """eval_step loss (inference BatchNorm, no dropout) and predict (mean, dispersion, pi, latent) at the engine's
    weights against the reference's inference forward, row chunk by row chunk."""
    Xd, Yd, sfd, rd = data
    B, G, lat_w = rd.numel(), Yd.shape[1], ref.hidden[len(ref.hidden) // 2]
    _load(ref, eng.get_weights())
    eng.read_epoch_acc(reset=True)
    eng.eval_step(Xd, Yd, sfd, rows=rd)
    acc = eng.read_epoch_acc()
    out = {k: torch.empty((B, G), device=DEV) for k in ("mean", "dispersion", "pi")}
    out["latent"] = torch.empty((B, lat_w), device=DEV)
    eng.predict(Xd, sfd, rows=rd, mean=out["mean"], disp=out["dispersion"], pi=out["pi"], latent=out["latent"])
    torch.cuda.synchronize()
    rl = rd.long()
    errs = {k: 0.0 for k in out}
    loss_sum = 0.0
    chunk = _chunk(G)
    with torch.no_grad():
        h, _, lat = ref.hidden_stack(Xd[rl].double(), training=False)
        for s in range(0, B, chunk):
            mu, theta, pi = ref.head_outputs(h[s:s + chunk], sfd[rl[s:s + chunk]].double())
            loss_sum += float(ref._elem(Yd[rl[s:s + chunk]].double(), mu, theta, pi).sum())
            want = {"mean": mu, "dispersion": theta, "pi": pi, "latent": lat[s:s + chunk]}
            for k, o in out.items():
                # absolute floors: pi as test_gpu_parity; the latent (pre-BatchNorm, linear, crosses zero): 1/10 of its
                # largest element
                floor = {"pi": 1e-7 / PRED_TOL, "latent": 0.1 * float(lat.abs().max())}.get(k, 0.0)
                e = ((o[s:s + chunk].double() - want[k]).abs() / (want[k].abs() + floor)).max().item()
                errs[k] = max(errs[k], e)
    oval = loss_sum / (B * G)
    val = acc[2] / acc[3]
    print("[%s] eval loss %.6f ref %.6f rel %.2e; predict worst relative error %s"
          % (tag, val, oval, abs(val - oval) / abs(oval), {k: "%.2e" % e for k, e in errs.items()}))
    assert acc[3] == B * G and abs(val - oval) < LOSS_TOL * abs(oval), (tag, val, oval)
    tol = TC_PRED_TOL if (path["tc_encoder"] or path["tc_heads"]) else PRED_TOL
    assert all(e < tol for e in errs.values()), (tag, errs)


def _reference(p0, hidden, batchnorm, activation, path):
    return TorchRefNet(p0, hidden, AE, batchnorm, dtype=torch.float64, activation=activation, device=DEV,
                       emulate_bf16=_side(path))


# ------------------------------------------------------------------------------------------------------------------
# a. The reference's hyper-parameter search grid (dca/hyper.py:27-37)
GRID_HIDDEN = [(64, 32, 64), (32, 16, 32), (64, 64), (32, 32), (16, 16), (16,), (32,), (64,), (128,)]
GRID_ACTS = ["relu", "selu", "elu", "PReLU", "linear", "LeakyReLU"]


def _grid_step(G, B, hidden, activation, batchnorm, dropout):
    rates = [HIDDEN_RATE] * len(hidden) if dropout else None
    in_rate = INPUT_RATE if dropout else 0.0
    data = _batch(G, B)
    p0 = _params(G, hidden, batchnorm, activation)
    eng = _engine(G, hidden, batchnorm, B, p0, activation, rates, in_rate)
    path = _expect_path(eng, hidden, activation, dropout, B)
    ref = _reference(p0, hidden, batchnorm, activation, path)
    _set_masks(ref, 77, 1, B, G, hidden, rates, in_rate)
    _step((G, B, hidden, activation, batchnorm, dropout), eng, ref, data, path, batchnorm)
    eng.close()


@pytest.mark.parametrize("batchnorm", [True, False])
@pytest.mark.parametrize("activation", GRID_ACTS)
@pytest.mark.parametrize("hidden", GRID_HIDDEN, ids=str)
def test_search_grid_step(hidden, activation, batchnorm):
    """Every hidden size x activation x batchnorm of the search grid, hidden dropout 0.11 and input dropout 0.23, at
    2000 genes and batches of 1024: loss, every gradient (PReLU slopes included) and the moving statistics."""
    _grid_step(2000, 1024, hidden, activation, batchnorm, True)


# every hidden size once (relu) and every other activation once on the default sizes, batchnorm and dropout rotated
GRID_20K = [(h, "relu", i % 2 == 0, i % 3 != 2) for i, h in enumerate(GRID_HIDDEN)] + \
           [((64, 32, 64), a, i % 2 == 1, i % 3 != 1) for i, a in enumerate(GRID_ACTS[1:])]


@pytest.mark.parametrize("hidden,activation,batchnorm,dropout", GRID_20K, ids=str)
def test_search_grid_step_at_20k_genes(hidden, activation, batchnorm, dropout):
    _grid_step(20000, 4096, hidden, activation, batchnorm, dropout)


# ------------------------------------------------------------------------------------------------------------------
# b. Every activation with dropout, four steps (direct call, graph capture, replays), then eval and predict
def _saturated_fraction(ref, Xr):
    """Per hidden layer: the share of units that hard_sigmoid saturates at 1 and dropout keeps in the reference's
    training forward (the units whose gradient must be 0)."""
    out, h = [], apply_dropout(Xr, ref.masks[-1], ref.rates[-1])
    with torch.no_grad():
        for i, nm in enumerate(ref.names):
            a = h @ ref.p[nm + "/kernel"] + ref.p[nm + "/bias"]
            if ref.batchnorm:
                a = (a - a.mean(0)) / torch.sqrt(a.var(0, unbiased=False) + ref.bn_eps) + ref.p[nm + "/bn_beta"]
            v = hidden_activation("hard_sigmoid", a)
            out.append(float(((v == 1.0) & (ref.masks[i] > 0)).double().mean()))
            h = apply_dropout(v, ref.masks[i], ref.rates[i])
    return out


@pytest.mark.parametrize("activation", sorted(_lib.ACTIVATION_IDS))
@pytest.mark.parametrize("gemm_path", ["auto", "generic"])
def test_every_activation_with_dropout_four_steps(activation, gemm_path):
    """Hidden dropout 0.11 and input dropout 0.77 on the tensor-core path (batchnorm) and on the fp32 path (no
    batchnorm), four training steps: the step graph is captured on the second call and replayed after, so every step
    must draw fresh masks (the reference applies that step's).  Each step starts the reference at the engine's weights.
    hard_sigmoid saturates at least 5 % of every layer's units at 1: at rate 0.11 their stored output times keep is
    1 - 2^-24, and the gradient must still be 0 there."""
    G, B, hidden, seed = 2000, 1024, (64, 32, 64), 4242
    # exponential after a BatchNorm: x_hat of the heavy-tailed exp(.) units of the layer before reaches ~sqrt(B), and
    # exp of that overflows the heads in any precision; that case runs without BatchNorm on both paths
    batchnorm = gemm_path == "auto" and activation != "exponential"
    rates, in_rate = [HIDDEN_RATE] * 3, 0.77
    data = _batch(G, B)
    p0 = _params(G, hidden, batchnorm, activation, seed=3)
    eng = _engine(G, hidden, batchnorm, B, p0, activation, rates, in_rate, seed=seed, gemm_path=gemm_path)
    path = _expect_path(eng, hidden, activation, True, B, gemm_path)
    ref = _reference(p0, hidden, batchnorm, activation, path)
    losses = []
    for step in range(1, 5):
        _set_masks(ref, seed, step, B, G, hidden, rates, in_rate)
        if activation == "hard_sigmoid" and step == 1:
            _load(ref, eng.get_weights())
            frac = _saturated_fraction(ref, data[0][data[3].long()].double())
            print("\nhard_sigmoid units at 1 and kept, per layer: %s" % ["%.3f" % f for f in frac])
            assert min(frac) >= 0.05, frac
        losses.append(_step((activation, gemm_path, "step %d" % step), eng, ref, data, path, batchnorm))
        eng.apply_update(1e-3, 5.0)
    assert len(set(losses)) == 4, losses
    _eval_and_predict((activation, gemm_path), eng, ref, data, path)
    eng.close()


# ------------------------------------------------------------------------------------------------------------------
# c. Depths 1 to 8: 64-wide ends (tensor-core encoder), inner widths off every multiple of 4 and 16.  The heads take the
# tensor cores where the head kernels land 16-byte aligned in the flat parameters (_expect_path): with batchnorm for
# (64, 3, 10, 64), (64, 48, 3, 10, 64), (64, 50, 3, 9, 17, 64) and (64, 36, 100, 36, 64), always for (64,), (64, 64),
# (64, 61, 30, 1, 1, 3, 64), (64, 40, 24, 12, 12, 24, 40, 64) and (64, 128, 64), never for (64, 33, 64).
DEPTHS = [(64,), (64, 64), (64, 33, 64), (64, 3, 10, 64), (64, 48, 3, 10, 64), (64, 50, 3, 9, 17, 64),
          (64, 61, 30, 1, 1, 3, 64), (64, 40, 24, 12, 12, 24, 40, 64),
          (64, 128, 64), (64, 36, 100, 36, 64)]                 # a middle layer wider than 64: per-layer middle
# every mid-stack regime (1 row; 129 rows, one past a 128-row block; 4096: 32-row strips on 128 CTAs; 8192: 128 x 64
# rows, its limit) and B = 8200 (per-layer hidden kernels)
DEPTH_BATCHES = [1, 129, 4096, 8192, 8200]


@pytest.mark.parametrize("batchnorm", [True, False])
@pytest.mark.parametrize("B", DEPTH_BATCHES)
@pytest.mark.parametrize("hidden", DEPTHS, ids=str)
def test_depths_on_the_fused_hidden_stack(hidden, B, batchnorm):
    """relu without dropout: one step (loss, every gradient, moving statistics), then eval loss and predict, whose
    latent is the pre-BatchNorm output of layer L // 2 (the reference's 'center')."""
    G = 2000
    data = _batch(G, B)
    p0 = _params(G, hidden, batchnorm, "relu", seed=len(hidden))
    eng = _engine(G, hidden, batchnorm, B, p0)
    path = _expect_path(eng, hidden, "relu", False, B)
    ref = _reference(p0, hidden, batchnorm, "relu", path)
    tag = (hidden, B, batchnorm)
    _step(tag, eng, ref, data, path, batchnorm)
    _eval_and_predict(tag, eng, ref, data, path)
    eng.close()


def test_nine_hidden_layers_are_rejected():
    from dca_b200.engine import DeviceEngine
    assert _lib.DCA_MAX_HIDDEN == 8
    with pytest.raises(ValueError, match="at most 8 hidden layers"):
        DeviceEngine(256, 256, (64,) * 9, AE, True, max_batch=16, seed=0)


# ------------------------------------------------------------------------------------------------------------------
# d. Dropout through every dataset kind: the resident, streamed and packed datasets give the same bits
@pytest.mark.parametrize("x_dtype", ["float32", "bfloat16"])
def test_dropout_training_is_bit_identical_across_dataset_kinds(x_dtype):
    """train() for two epochs with input dropout 0.2, hidden dropout 0.11, elu and the tensor-core model from one
    random_state on a DeviceDataset, a StreamedDataset and a PackedDeviceDataset of the same counts: history, weights
    and BatchNorm state bit-identical.  With fp32 X the expanded batches stay fp32 under input dropout, so that the
    mask scales the fp32 value and the encoder's gather rounds it once, as on the resident X."""
    from dca_b200.device_data import DeviceDataset
    from dca_b200.network import AE_types
    from dca_b200.packed_data import PackedDeviceDataset
    from dca_b200.stream_data import StreamedDataset
    from dca_b200.train import train
    G, bs = 2000, 256
    Y = synth_counts(1500, G, 12)
    kinds = {"device_data": DeviceDataset.from_counts(Y, torch.device(DEV), x_dtype=x_dtype),
             "stream_data": StreamedDataset.from_counts(Y, torch.device(DEV), x_dtype=x_dtype, batch=bs),
             "packed_data": PackedDeviceDataset.from_counts(Y, torch.device(DEV), x_dtype=x_dtype)}
    runs = {}
    for kind, ds in kinds.items():
        net = AE_types[AE](input_size=G, output_size=G, hidden_size=(64, 32, 64), x_dtype=x_dtype, activation="elu",
                           hidden_dropout=0.11, input_dropout=0.2)
        net.build(max_batch=bs, seed=5)
        info = net.engine.info()
        assert info["tc_heads"] and info["tc_encoder"] and not info["fused_hidden"], info
        np.random.seed(3)
        hist = train(None, net, epochs=2, batch_size=bs, validation_split=0.1, verbose=False, shuffle=False,
                     **{kind: ds}).history
        runs[kind] = (hist, net.engine.get_weights())
        print("\n[%s X %s] loss %s val_loss %s" % (kind, x_dtype, hist["loss"], hist["val_loss"]))
        net.engine.close()
    h_d, w_d = runs["device_data"]
    for kind in ("stream_data", "packed_data"):
        h, w = runs[kind]
        differ = [k for k in w_d if not np.array_equal(w_d[k], w[k])]
        assert h == h_d and not differ, (kind, x_dtype, h, h_d, differ)
