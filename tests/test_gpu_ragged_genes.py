"""The fp32 path at real sizes: gene counts off a multiple of 8 (what ``io.normalize``'s gene filter leaves seven times out
of eight) keep the default model off the tensor-core kernels, so its heads, encoder and head backward run on the
split-K CUDA-core GEMM (dense_generic.cu), its loss on the scalar (G % 4 != 0) or vector (G % 4 == 0, partial last
column block) loss kernels, its bias and BatchNorm sums through col_sums.  Each case runs that path at 20 000 genes and
batches of 1 to 8200 rows against the float64 autograd reference (oracle/torch_ref.py) on the same device, its head
and loss graph evaluated in row chunks.  Needs an H100: -m gpu.

Bounds (README; DESIGN section 3): loss 1e-4 relative, every gradient tensor rel_err(got, ref, 2e-3) < 2e-3, predict
outputs 5e-4 relative.  Every tensor's worst error and its location is printed (-s), as is the peak device memory."""
import functools
import gc
import time

import numpy as np
import pytest
import torch

from oracle import dca_oracle as O
from oracle.torch_ref import TorchRefNet, TorchExtraNet, extra_init_params, EXTRA_TYPES
from tests.util import synth_counts

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
HIDDEN = (64, 32, 64)
NAMES = O.layer_names(len(HIDDEN))
HEAD_LAYERS = ("mean", "dispersion", "pi", "mean_no_act")
EXTRA = 300                         # each batch is gathered from a dataset this many rows larger
CHUNK = 256                         # reference rows per head / loss chunk: ~1.5 GB of float64 graph at 20 004 genes
LOSS_TOL, GRAD_TOL, GRAD_FLOOR, PRED_TOL = 1e-4, 2e-3, 2e-3, 5e-4
# Gradients that are zero in exact arithmetic (hidden biases in front of a BatchNorm; at B = 1 with BatchNorm x_hat = 0,
# so everything upstream of the last BatchNorm): fp32 leaves the rounding of B terms of a sum whose exact value is 0,
# about sqrt(B) * 2^-24 of the terms, far below 1e-5 of the step's largest gradient.
ZERO_TOL = 1e-5
# BatchNorm statistics recovered from the moving averages m' = mom * m + (1 - mom) * s: the fp32 rounding of m' (2^-24
# of |m|) becomes 100x larger in s, so the error is taken relative to max |s| + max |m|.
BN_TOL = 1e-3
PEAK_BUDGET = 16 << 30


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


@functools.lru_cache(maxsize=3)
def _dataset(G):
    """Normalised synthetic counts with enough rows for the largest batch of this gene count (host arrays)."""
    N = (8200 if G < 10000 else 4096) + EXTRA
    Y = synth_counts(N, G, 1000 + G)
    Y[0, :4] = [0, 17, 40, 3000]
    X, sf = O.normalize_inputs(Y)
    return X, Y, sf


def _batch(G, B, x_dtype=torch.float32):
    """Device X, Y, sf of a dataset B + 300 rows long and a permuted int32 gather of B of its rows."""
    X, Y, sf = _dataset(G)
    N = B + EXTRA
    rows = np.random.default_rng(B).permutation(N)[:B].astype(np.int32)
    return _t(X[:N], x_dtype), _t(Y[:N]), _t(sf[:N]), torch.as_tensor(rows).to(DEV)


def _params(p0, seed):
    """Random non-zero biases, BatchNorm betas and per-gene dispersions (test_gpu_parity._make_pair)."""
    rng = np.random.default_rng(seed + 1)
    for k in p0:
        if k.endswith(("/bias", "/bn_beta", "/theta")):
            p0[k] = rng.normal(0, 0.2, p0[k].shape).astype(np.float32)
    return p0


def _engine(G, ae_type, B, p0, batchnorm=True, fused=True, **kw):
    from dca_b200.engine import DeviceEngine
    eng = DeviceEngine(G, G, HIDDEN, ae_type, batchnorm, max_batch=B, seed=None, **kw)
    eng.set_weights(p0)
    info = eng.info()
    # the shapes must stay on the fp32 path: if a change moves them elsewhere this file tests something else
    assert not info["tc_heads"] and not info["tc_encoder"] and info["fused_hidden"] == fused, info
    return eng


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


def _is_head(name):
    return name.split("/")[0] in HEAD_LAYERS


def _zero_tensors(param_info, batchnorm, B):
    """Gradient tensors that are exactly zero in exact arithmetic."""
    if not batchnorm:
        return set()
    hidden = [n for n, *_ in param_info if not _is_head(n)]
    zero = {n for n in hidden if n.endswith("/bias")}
    if B == 1:
        # x_hat = 0 in every layer, so dL/da = 0 behind every BatchNorm: only the last layer's beta sees the heads' gradient
        zero |= {n for n in hidden if n != NAMES[-1] + "/bn_beta"}
    return zero


def _check_grads(tag, g, param_info, og, batchnorm, B, verbose=True):
    """Every gradient tensor against the reference; prints the worst error of each and where it sits.  Returns the
    worst error: relative for most tensors, as a fraction of the step's largest gradient for the zero ones."""
    ref = {k: v.detach().double().cpu().numpy().reshape(-1) for k, v in og.items()}
    scale = max(float(np.max(np.abs(v))) for v in ref.values())
    zero = _zero_tensors(param_info, batchnorm, B)
    bad, worst = [], 0.0
    for name, off, r, c in param_info:
        got = g[off: off + r * c].astype(np.float64); want = ref[name]
        if name in zero:
            i = int(np.argmax(np.abs(got)))
            err = abs(got[i]) / scale
            if verbose:
                print("  %-24s zero: |got| %.2e of the largest gradient at %s (ref max %.1e)"
                      % (name, err, np.unravel_index(i, (r, c)), np.max(np.abs(want)) / scale))
            ok = err < ZERO_TOL and np.max(np.abs(want)) <= 1e-12 * scale
        else:
            e = np.abs(got - want) / np.maximum(np.abs(want), GRAD_FLOOR * np.max(np.abs(want)) + 1e-30)
            i = int(np.argmax(e)); err = float(e[i])
            if verbose:
                print("  %-24s rel_err %.2e at %s (got %.6e, ref %.6e)" % (name, err, np.unravel_index(i, (r, c)), got[i], want[i]))
            ok = err < GRAD_TOL
        worst = max(worst, err)
        if not ok:
            bad.append((name, err))
    assert not bad, (tag, bad)
    return worst


@torch.no_grad()
def _near_zero_units(ref, Xr):
    """ReLU inputs of the reference's training forward within fp32 error of zero (1e-5 of the layer's largest): units
    whose mask the fp32 step may flip.  Printed so that a failing hidden-stack tensor can be read from one run."""
    h, out = Xr, []
    for nm in ref.names:
        a = h @ ref.p[nm + "/kernel"] + ref.p[nm + "/bias"]
        if ref.batchnorm:
            a = (a - a.mean(0)) / torch.sqrt(a.var(0, unbiased=False) + ref.bn_eps) + ref.p[nm + "/bn_beta"]
        out.append(int((a.abs() < 1e-5 * a.abs().max()).sum()))
        h = torch.relu(a)
    return out


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


def _one_step(ae_type, G, B, batchnorm=True, x_dtype="float32"):
    """One training step of the engine (rows gathered from a larger dataset) against the chunked float64 reference:
    loss, every gradient tensor and the BatchNorm batch statistics the step folds into the moving averages."""
    Xd, Yd, sfd, rd = _batch(G, B, torch.bfloat16 if x_dtype == "bfloat16" else torch.float32)
    p0 = _params(O.init_params(G, G, HIDDEN, ae_type, batchnorm, seed=0, dtype=np.float32), 0)
    eng = _engine(G, ae_type, B, p0, batchnorm, fused=B <= 8192, x_dtype=x_dtype)
    w0 = eng.get_weights()
    eng.train_step(Xd, Yd, sfd, rows=rd)
    loss = eng.read_loss()
    g = eng.grads.cpu().numpy()
    w1 = eng.get_weights()
    param_info = eng.param_info
    eng.close(); del eng
    rl = rd.long()
    # bf16 X: the reference reads the same bf16 values; every weight stays fp32 (the fp32 GEMM converts X on load)
    Xr, Yr, sfr = Xd[rl].double(), Yd[rl].double(), sfd[rl].double()
    ref = TorchRefNet(p0, HIDDEN, ae_type, batchnorm, dtype=torch.float64, device=DEV)
    oloss, og, stats = ref.loss_and_grads_chunked(Xr, Yr, sfr, chunk=CHUNK)
    flips = _near_zero_units(ref, Xr)
    bn_err = _bn_error(w0, w1, stats) if batchnorm else 0.0
    print("\n[%s G=%d B=%d bn=%d X %s] loss %.6f ref %.6f rel %.2e, batch statistics %.2e, ReLU inputs near 0 per layer %s"
          % (ae_type, G, B, batchnorm, x_dtype, loss, oloss, abs(loss - oloss) / abs(oloss), bn_err, flips))
    _check_grads((ae_type, G, B), g, param_info, og, batchnorm, B)
    assert abs(loss - oloss) < LOSS_TOL * abs(oloss), (loss, oloss)
    assert bn_err < BN_TOL, bn_err


# G = 20001: the scalar loss kernel (G % 4 != 0); G = 20004: the vector loss kernels, last 128-gene block 36 genes wide.
# B = 1 (a one-row last batch), 32 (the default batch: split-K over the genes in the head backward), 4096.
STEP_CASES = [(G, B, t) for G in (20001, 20004) for B in (1, 32, 4096) for t in O.AE_TYPES]


@pytest.mark.parametrize("G,B,ae_type", STEP_CASES)
def test_fp32_step_vs_float64(G, B, ae_type):
    _one_step(ae_type, G, B)


def test_fp32_step_per_layer_hidden_path():
    """B > 8192: the hidden stack runs as per-layer kernels instead of the one-launch mid_stack."""
    _one_step("zinb-conddisp", 2003, 8200)


def test_fp32_step_bf16_x():
    """bf16 X storage on the fp32 path: gemm_kernel<__nv_bfloat16> reads X, the weights stay fp32."""
    _one_step("zinb-conddisp", 20001, 4096, x_dtype="bfloat16")


def test_fp32_trajectory_five_steps():
    """Five train_step + apply_update (RMSprop, clip 5) at the default batch against the reference's train_step: loss at
    every step, then every parameter and moving statistic."""
    G, B = 20001, 32
    Xd, Yd, sfd, rd = _batch(G, B)
    p0 = _params(O.init_params(G, G, HIDDEN, "zinb-conddisp", True, seed=0, dtype=np.float32), 0)
    eng = _engine(G, "zinb-conddisp", B, p0)
    ref = TorchRefNet(p0, HIDDEN, "zinb-conddisp", True, dtype=torch.float64, device=DEV)
    rl = rd.long()
    Xr, Yr, sfr = Xd[rl].double(), Yd[rl].double(), sfd[rl].double()
    for step in range(5):
        eng.train_step(Xd, Yd, sfd, rows=rd)
        eng.apply_update(1e-3, 5.0)
        loss = eng.read_loss()
        oloss = ref.train_step(Xr, Yr, sfr, lr=1e-3, clip=5.0)
        print("\n  step %d: loss %.6f ref %.6f rel %.2e" % (step, loss, oloss, abs(loss - oloss) / abs(oloss)))
        assert abs(loss - oloss) < LOSS_TOL * abs(oloss), (step, loss, oloss)
    w = eng.get_weights()
    eng.close(); del eng
    bad = []
    for k, v in ref.p.items():
        if k.endswith("/bias") and not _is_head(k):
            continue                                      # noise / (sqrt(noise^2) + eps) in front of a BatchNorm
        want = v.detach().double().cpu().numpy().reshape(w[k].shape)
        e = np.abs(w[k] - want) - 2e-3 * np.abs(want)
        i = int(np.argmax(e))
        print("  %-24s worst |got - ref| - 2e-3 |ref| = %.2e at %s" % (k, e.flat[i], np.unravel_index(i, want.shape)))
        if e.flat[i] > 2e-4:
            bad.append((k, float(e.flat[i])))
    assert not bad, bad


@pytest.mark.parametrize("G", [20001, 20004])
@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "nb"])
def test_fp32_eval_and_predict(ae_type, G):
    """eval_step loss and predict outputs (mean, dispersion, pi, latent) with non-trivial moving statistics against
    the reference's inference forward, row chunk by row chunk on the device."""
    B = 4096
    Xd, Yd, sfd, rd = _batch(G, B)
    p0 = _params(O.init_params(G, G, HIDDEN, ae_type, True, seed=0, dtype=np.float32), 0)
    rng = np.random.default_rng(1)
    for k in p0:
        if k.endswith("moving_mean"): p0[k] = rng.normal(0, 0.3, p0[k].shape).astype(np.float32)
        if k.endswith("moving_var"): p0[k] = rng.uniform(0.5, 2.0, p0[k].shape).astype(np.float32)
    eng = _engine(G, ae_type, B, p0)
    eng.read_epoch_acc(reset=True)
    eng.eval_step(Xd, Yd, sfd, rows=rd)
    acc = eng.read_epoch_acc()
    cond, has_pi = ae_type.endswith("conddisp"), ae_type.startswith("zinb")
    out = {"mean": torch.empty((B, G), device=DEV), "latent": torch.empty((B, HIDDEN[1]), device=DEV),
           "dispersion": torch.empty((B, G) if cond else (G,), device=DEV)}
    if has_pi:
        out["pi"] = torch.empty((B, G), device=DEV)
    eng.predict(Xd, sfd, rows=rd, mean=out["mean"], disp=out["dispersion"], pi=out.get("pi"), latent=out["latent"])
    torch.cuda.synchronize()
    eng.close(); del eng
    ref = TorchRefNet(p0, HIDDEN, ae_type, True, dtype=torch.float64, device=DEV)
    rl = rd.long()
    # absolute floors: pi as test_gpu_parity; the latent (pre-BatchNorm 'center', linear, crosses zero) carries the
    # first layer's fp32 error, ~1e-5 of its scale after 20 000 terms: 5e-5 of its largest element
    errs = {k: 0.0 for k in out}
    loss_sum = 0.0
    with torch.no_grad():
        for s in range(0, B, CHUNK):
            r = rl[s:s + CHUNK]
            Xr, Yr, sfr = Xd[r].double(), Yd[r].double(), sfd[r].double()
            h, _, lat = ref.hidden_stack(Xr, training=False)
            mu, theta, pi = ref.head_outputs(h, sfr)
            loss_sum += float(ref._elem(Yr, mu, theta, pi).sum())
            want = {"mean": mu, "latent": lat, "dispersion": theta if cond else theta.reshape(-1), "pi": pi}
            for k, o in out.items():
                got = o if (k == "dispersion" and not cond) else o[s:s + CHUNK]
                floor = {"pi": 1e-7 / PRED_TOL, "latent": 0.1 * float(lat.abs().max())}.get(k, 0.0)
                e = ((got.double() - want[k]).abs() / (want[k].abs() + floor)).max().item()
                errs[k] = max(errs[k], e)
    oval = loss_sum / (B * G)
    val = acc[2] / acc[3]
    print("\n[%s G=%d B=%d] eval loss %.6f ref %.6f rel %.2e; predict worst relative error %s"
          % (ae_type, G, B, val, oval, abs(val - oval) / abs(oval), {k: "%.2e" % e for k, e in errs.items()}))
    assert acc[3] == B * G and abs(val - oval) < LOSS_TOL * abs(oval), (val, oval)
    assert all(e < PRED_TOL for e in errs.values()), errs


EXTRA_CASES = [(t, False) for t in EXTRA_TYPES] + [("zinb-elempi", True)]


@pytest.mark.parametrize("B", [32, 1000])
@pytest.mark.parametrize("ae_type,sharedpi", EXTRA_CASES)
def test_extra_type_step_and_predict(ae_type, sharedpi, B):
    """The seven other AE types (extra_types.cu; fp32 path only) with the default hidden sizes: one step against the
    autograd reference on the device, then predict with the same weights."""
    from dca_b200.engine import DeviceEngine
    G = 2003
    Xd, Yd, sfd, rd = _batch(G, B)
    ridge = 0.02 if ae_type.startswith("zinb") else 0.0
    p0 = extra_init_params(G, G, HIDDEN, ae_type, True, seed=0, sharedpi=sharedpi)
    rng = np.random.default_rng(1)
    for k in p0:
        if k.endswith(("/bias", "/bn_beta")):
            p0[k] = rng.normal(0, 0.2, p0[k].shape).astype(np.float32)
    eng = DeviceEngine(G, G, HIDDEN, ae_type, True, max_batch=B, ridge=ridge, seed=None, sharedpi=sharedpi)
    eng.set_weights(p0)
    info = eng.info()
    assert not info["tc_heads"] and not info["tc_encoder"] and not info["fused_hidden"], info
    shared = ae_type in ("nb-shared", "zinb-shared")
    rl = rd.long()
    Xr, Yr, sfr = Xd[rl].double(), Yd[rl].double(), sfd[rl].double()
    net = TorchExtraNet(p0, HIDDEN, ae_type, True, ridge=ridge, device=DEV)
    ref = net.predict(Xr, sfr)
    out = {"mean": torch.empty((B, G), device=DEV), "latent": torch.empty((B, HIDDEN[1]), device=DEV)}
    if "dispersion" in ref:
        out["dispersion"] = torch.empty((B, 1 if shared else G), device=DEV)
    if "pi" in ref:
        out["pi"] = torch.empty((B, 1 if shared else G), device=DEV)
    # predict first: the training step moves the BatchNorm moving statistics
    eng.predict(Xd, sfd, rows=rd, mean=out["mean"], disp=out.get("dispersion"), pi=out.get("pi"), latent=out["latent"])
    eng.train_step(Xd, Yd, sfd, rows=rd)
    loss = eng.read_loss()
    g = eng.grads.cpu().numpy()
    param_info = eng.param_info
    eng.close(); del eng
    oloss, og, _ = net.loss_and_grads_chunked(Xr, Yr, sfr, chunk=CHUNK)
    print("\n[%s%s G=%d B=%d] loss %.6f ref %.6f rel %.2e" % (ae_type, " sharedpi" if sharedpi else "", G, B, loss, oloss,
                                                            abs(loss - oloss) / abs(oloss)))
    _check_grads((ae_type, sharedpi, B), g, param_info, og, True, B)
    assert abs(loss - oloss) < LOSS_TOL * abs(oloss), (loss, oloss)
    errs = {}
    for k, o in out.items():
        want = ref[k].reshape(o.shape)
        # linear outputs cross zero ('normal' mean, latent): absolute floor of 5e-5 of the largest element
        floor = 0.1 * np.abs(want).max() if (k == "latent" or ae_type == "normal") else (1e-7 / PRED_TOL if k == "pi" else 0.0)
        errs[k] = float(np.max(np.abs(o.cpu().numpy() - want) / (np.abs(want) + floor)))
    print("  predict worst relative error %s" % {k: "%.2e" % e for k, e in errs.items()})
    assert all(e < PRED_TOL for e in errs.values()), errs


def test_train_defaults_on_filtered_genes_every_step_vs_float64():
    """train() end to end with every default: 1033 cells x 20 000 genes of which 7 have no counts, so io.normalize
    keeps 19 993 genes (fp32 path); validation split 0.1 leaves 929 training cells, whose last batch of 32 is one row.

    Every training step train() runs (the one-row batch included) is checked against the float64 reference evaluated
    at the engine's weights of that moment: loss and every gradient tensor; every validation batch likewise; the
    history is the row-weighted mean of those losses, lr the default.  The weights are not compared with an
    independent float64 run of the same schedule: at this shape RMSprop's normalisation of tiny gradients (eps 1e-7)
    makes the trajectory chaotic.  A float64 run whose first kernel is perturbed by 1e-7 relative, below fp32
    resolution, departs from the unperturbed one by 1e-3 in the step loss within 20 steps, as torch's own fp32 step
    does; no fp32 implementation can follow one float64 trajectory over two epochs to 1e-4."""
    from dca_b200.anndata_lite import AnnData
    from dca_b200 import io
    from dca_b200.network import AE_types
    from dca_b200.train import train
    N, G0, bs, epochs = 1033, 20000, 32, 2
    Y = synth_counts(N, G0, 23)
    Y[:, np.random.default_rng(4).choice(G0, 7, replace=False)] = 0
    ad = io.normalize(io.read_dataset(AnnData(Y.copy())))
    G = ad.X.shape[1]
    assert G == G0 - 7 and G % 8 != 0
    split_at = int(N * 0.9)
    assert split_at == 929 and split_at % bs == 1
    net = AE_types["zinb-conddisp"](input_size=G, output_size=G)
    net.build(max_batch=bs, seed=3)
    eng = net.engine
    info = eng.info()
    assert not info["tc_heads"] and not info["tc_encoder"] and info["fused_hidden"], info
    ref = TorchRefNet(eng.get_weights(), HIDDEN, "zinb-conddisp", True, dtype=torch.float64, device=DEV)
    steps, vals = [], []
    engine_step, engine_eval = eng.train_step, eng.eval_step

    def at_engine_weights():
        with torch.no_grad():
            for k, v in eng.get_weights().items():            # synchronises the device
                ref.p[k].copy_(torch.as_tensor(v).reshape(ref.p[k].shape))

    def checked_step(X, Y, sf, rows=None, **kw):
        at_engine_weights()
        engine_step(X, Y, sf, rows=rows, **kw)
        loss = eng.read_loss()
        rl = rows.long()
        oloss, og, _ = ref.loss_and_grads(X[rl].double(), Y[rl].double(), sf[rl].double())
        gerr = _check_grads(("train step", len(steps)), eng.grads.cpu().numpy(), eng.param_info, og, True, rows.numel(),
                            verbose=False)
        steps.append((rows.numel(), loss, oloss, gerr))

    def checked_eval(X, Y, sf, **kw):
        at_engine_weights()
        engine_eval(X, Y, sf, **kw)
        with torch.no_grad():
            oval = float(ref.loss(X.double(), Y.double(), sf.double(), training=False)[0])
        vals.append((X.shape[0], oval))

    eng.train_step, eng.eval_step = checked_step, checked_eval
    np.random.seed(11)
    hist = train(ad, net, epochs=epochs, batch_size=bs, verbose=False).history
    per_epoch = (split_at + bs - 1) // bs
    assert len(steps) == epochs * per_epoch and [b for b, *_ in steps[:per_epoch]] == [bs] * (per_epoch - 1) + [1]
    for i, (b, loss, oloss, gerr) in enumerate(steps):
        print("  step %2d B %2d loss %.6f ref %.6f rel %.2e, worst gradient error %.2e" % (i, b, loss, oloss, abs(loss - oloss) / oloss, gerr))
        assert abs(loss - oloss) < LOSS_TOL * abs(oloss), (i, b, loss, oloss)
    n_va = N - split_at
    for e in range(epochs):
        ep = steps[e * per_epoch:(e + 1) * per_epoch]
        ref_loss = sum(b * ol for b, _, ol, _ in ep) / split_at
        va = vals[e * len(vals) // epochs:(e + 1) * len(vals) // epochs]
        assert sum(b for b, _ in va) == n_va
        ref_val = sum(b * ov for b, ov in va) / n_va
        print("[train defaults G=%d epoch %d] loss %.6f ref %.6f, val_loss %.6f ref %.6f, lr %g"
              % (G, e, hist["loss"][e], ref_loss, hist["val_loss"][e], ref_val, hist["lr"][e]))
        assert abs(hist["loss"][e] - ref_loss) < LOSS_TOL * ref_loss
        assert abs(hist["val_loss"][e] - ref_val) < LOSS_TOL * ref_val
    np.testing.assert_allclose(hist["lr"], [O.KERAS_DEFAULTS["rms_lr"]] * epochs, rtol=1e-6)
