"""The zinb, nb-conddisp and nb models on the tensor-core path at 20 000 genes.  zinb-conddisp computes its head
activations inside the loss kernel; these three types do not: their heads run the tensor-core heads kernel with two
head slots (zinb: mean + pi, nb-conddisp: mean + dispersion) or one (nb), their loss runs the ring kernel (zinb) or the
vectorised loss kernel (nb-conddisp, nb) into bf16 slot gradients, the per-gene dispersion of zinb / nb is clipped
and its gradient finished from dL/dtheta, and the head backward runs with one or two slots.

 * one training step in every batch regime of the hidden stack (B = 1, the default 32, the two fused-stack strip plans
   4096 and 8192, the per-layer path 8200; with and without BatchNorm; bf16 X) against the float64 autograd reference
   (oracle/torch_ref.py) on the device, both the same-rounding one (bf16 operands where the kernels round) and the
   exact one;
 * eval_step and every output subset the Python API asks predict() for;
 * two engines with the same seed give the same bits through a direct step, a graph capture and a graph replay;
 * every optimizer but RMSprop refreshes the bf16 copy of the parameters that the tensor-core kernels read.

Every tensor's worst error and where it sits is printed (-s), as are each case's peak device memory and wall time.
Needs an H100: -m gpu."""
import functools
import gc
import time

import numpy as np
import pytest
import torch

from oracle import dca_oracle as O
from oracle.torch_ref import TorchRefNet
from tests.util import synth_counts
from tests.test_gpu_parity_full import TC_VS_EXACT
from tests.test_gpu_ragged_genes import _params, _zero_tensors, _bn_error, _is_head

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
G = 20000
HIDDEN = (64, 32, 64)
EXTRA = 300                         # each batch is gathered from a dataset this many rows larger
CHUNK = 256                         # reference rows per head / loss chunk
TYPES = ("zinb", "nb-conddisp", "nb")
SLOTS = {"zinb-conddisp": 3, "zinb": 2, "nb-conddisp": 2, "nb": 1}
# same-rounding reference: the bounds of test_gpu_parity._assert_step_bounds, the BatchNorm batch statistics of
# test_tc_train_step_batch_regimes_vs_oracle
LOSS_TOL, HEAD_TOL, HIDDEN_TOL, BN_TOL = 1e-4, 3e-3, 3e-2, 1e-3
# dL/dtheta is summed over the cells from fp32 element derivatives; entries whose sum cancels are held to an absolute
# floor of this fraction of the tensor's largest entry
THETA_FLOOR = 2e-3
ZERO_TOL = 1e-5                     # gradients that are zero in exact arithmetic, relative to the step's largest gradient
PRED_TOL = 5e-4
PEAK_BUDGET = 16 << 30
# raw dispersion/theta entries whose exp lies outside the clip range [1e-3, 1e4]: their gradient is exactly zero
CLIPPED_THETA = {7: -8.0, 1234: 10.0, 19999: -9.5}


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


@functools.lru_cache(maxsize=1)
def _dataset():
    """Normalised synthetic counts with enough rows for the largest batch (host arrays)."""
    Y = synth_counts(8200 + EXTRA, G, 1000 + G)
    Y[0, :4] = [0, 17, 40, 3000]
    X, sf = O.normalize_inputs(Y)
    return X, Y, sf


def _batch(B, x_dtype=torch.float32, seed=None):
    """Device X, Y, sf of a dataset B + 300 rows long and a permuted int32 gather of B of its rows."""
    X, Y, sf = _dataset()
    N = B + EXTRA
    rows = np.random.default_rng(B if seed is None else seed).permutation(N)[:B].astype(np.int32)
    return _t(X[:N], x_dtype), _t(Y[:N]), _t(sf[:N]), torch.as_tensor(rows).to(DEV)


def _ridge(ae_type):
    return 0.02 if ae_type.startswith("zinb") else 0.0


def _start_params(ae_type, batchnorm=True, moving_stats=False):
    p0 = _params(O.init_params(G, G, HIDDEN, ae_type, batchnorm, seed=0, dtype=np.float32), 0)
    if "dispersion/theta" in p0:
        for g, v in CLIPPED_THETA.items():
            p0["dispersion/theta"][g] = v
    if moving_stats:
        rng = np.random.default_rng(1)
        for k in p0:
            if k.endswith("moving_mean"): p0[k] = rng.normal(0, 0.3, p0[k].shape).astype(np.float32)
            if k.endswith("moving_var"): p0[k] = rng.uniform(0.5, 2.0, p0[k].shape).astype(np.float32)
    return p0


def _engine(ae_type, B, p0=None, batchnorm=True, seed=None, **kw):
    from dca_b200.engine import DeviceEngine
    eng = DeviceEngine(G, G, HIDDEN, ae_type, batchnorm, max_batch=B, ridge=_ridge(ae_type), seed=seed, **kw)
    if p0 is not None:
        eng.set_weights(p0)
    info = eng.info()
    # the shapes must stay on the tensor-core path: if a change moves them elsewhere this file tests something else
    assert info["tc_heads"] and info["tc_encoder"] and info["fused_hidden"] == (B <= 8192), info
    assert info["head_slots"] == SLOTS[ae_type], info
    return eng


def _ref(p0, ae_type, batchnorm=True, emulate_bf16=True):
    return TorchRefNet(p0, HIDDEN, ae_type, batchnorm, ridge=_ridge(ae_type), dtype=torch.float64, device=DEV,
                       emulate_bf16=emulate_bf16)


@pytest.fixture(autouse=True)
def _device_budget(request):
    """Each case frees its engines and tensors before the next; peak device memory and wall time are printed."""
    gc.collect(); torch.cuda.empty_cache()
    torch.empty(1, device=DEV)                           # the allocator's statistics exist once it has allocated
    torch.cuda.reset_peak_memory_stats(DEV)
    t0 = time.perf_counter()
    yield
    peak = torch.cuda.max_memory_allocated(DEV)
    print("[%s] peak device memory %.2f GB, %.1f s" % (request.node.name, peak / 1e9, time.perf_counter() - t0))
    gc.collect(); torch.cuda.empty_cache()
    assert peak < PEAK_BUDGET, peak


def _normwise(got, want):
    return float(np.linalg.norm(got - want) / (np.linalg.norm(want) + 1e-300))


def _grad_errors(g, param_info, og_same, og_exact, batchnorm, B):
    """Every gradient tensor against both references; prints each tensor's worst error and where it sits and returns
    the list of (tensor, which bound, error, bound) that fail."""
    same = {k: v.detach().double().cpu().numpy().reshape(-1) for k, v in og_same.items()}
    exact = {k: v.detach().double().cpu().numpy().reshape(-1) for k, v in og_exact.items()}
    scale = max(float(np.max(np.abs(v))) for v in exact.values())
    zero = _zero_tensors(param_info, batchnorm, B)
    bad = []
    for name, off, r, c in param_info:
        got = g[off: off + r * c].astype(np.float64)
        s, x = same[name], exact[name]
        shape = (r, c)
        if name in zero:
            i = int(np.argmax(np.abs(got)))
            err = abs(got[i]) / scale
            ref_max = max(np.max(np.abs(s)), np.max(np.abs(x))) / scale
            print("  %-24s zero: |got| %.2e of the largest gradient at %s (references' max %.1e)"
                  % (name, err, np.unravel_index(i, shape), ref_max))
            if not (err < ZERO_TOL and ref_max <= 1e-12):
                bad.append((name, "zero", err, ZERO_TOL))
            continue
        head = _is_head(name)
        if name == "dispersion/theta":
            e = np.abs(got - s) / np.maximum(np.abs(s), THETA_FLOOR * np.max(np.abs(s)))
            kind = "rel (floor %.0e)" % THETA_FLOOR
        else:
            e = np.abs(got - s) / np.max(np.abs(s))
            kind = "of max"
        i = int(np.argmax(e)); e_same = float(e[i])
        e_exact = _normwise(got, x)
        b_same = HEAD_TOL if head else HIDDEN_TOL
        b_exact = TC_VS_EXACT["grad_head"] if head else TC_VS_EXACT["grad_hidden"]
        print("  %-24s same %.2e %s at %s (got %.6e, ref %.6e); exact norm-wise %.4e"
              % (name, e_same, kind, np.unravel_index(i, shape), got[i], s[i], e_exact))
        if not e_same < b_same:
            bad.append((name, "same", e_same, b_same))
        if not e_exact < b_exact:
            bad.append((name, "exact", e_exact, b_exact))
    return bad


# (B, BatchNorm): a one-row last batch, the CLI's default batch, the two strip plans of the fused hidden stack and the
# per-layer hidden path past 8192 rows
STEP_REGIMES = [(1, True), (32, True), (4096, True), (8192, True), (8200, True), (4096, False), (8200, False)]
STEP_CASES = [(t, B, bn, "float32") for t in TYPES for B, bn in STEP_REGIMES] + [("nb", 4096, True, "bfloat16")]


@pytest.mark.parametrize("ae_type,B,batchnorm,x_dtype", STEP_CASES)
def test_tc_step_vs_float64(ae_type, B, batchnorm, x_dtype):
    """One training step (rows gathered from a larger dataset) against the same-rounding and the exact float64
    reference: loss, every gradient tensor (the clipped theta entries included) and the BatchNorm batch statistics."""
    Xd, Yd, sfd, rd = _batch(B, torch.bfloat16 if x_dtype == "bfloat16" else torch.float32)
    p0 = _start_params(ae_type, batchnorm)
    eng = _engine(ae_type, B, p0, batchnorm, x_dtype=x_dtype)
    w0 = eng.get_weights()
    eng.train_step(Xd, Yd, sfd, rows=rd)
    loss = eng.read_loss()
    g = eng.grads.cpu().numpy()
    w1 = eng.get_weights()
    param_info = eng.param_info
    eng.close(); del eng
    rl = rd.long()
    Xr, Yr, sfr = Xd[rl].double(), Yd[rl].double(), sfd[rl].double()
    l_same, og_same, stats = _ref(p0, ae_type, batchnorm, True).loss_and_grads_chunked(Xr, Yr, sfr, chunk=CHUNK)
    l_exact, og_exact, _ = _ref(p0, ae_type, batchnorm, False).loss_and_grads_chunked(Xr, Yr, sfr, chunk=CHUNK)
    bn_err = _bn_error(w0, w1, stats) if batchnorm else 0.0
    print("\n[%s B=%d bn=%d X %s] loss %.7f, same-rounding %.7f (rel %.2e), exact %.7f (rel %.2e); batch statistics %.2e"
          % (ae_type, B, batchnorm, x_dtype, loss, l_same, abs(loss - l_same) / abs(l_same), l_exact,
             abs(loss - l_exact) / abs(l_exact), bn_err))
    if "dispersion/theta" in og_same:
        name, off, r, c = [t for t in param_info if t[0] == "dispersion/theta"][0]
        clipped = g[off + np.array(list(CLIPPED_THETA))]
        print("  dL/dtheta of the clipped entries %s" % clipped)
        assert not clipped.any(), clipped
    bad = _grad_errors(g, param_info, og_same, og_exact, batchnorm, B)
    assert abs(loss - l_same) < LOSS_TOL * abs(l_same), (loss, l_same)
    assert abs(loss - l_exact) < TC_VS_EXACT["loss"] * abs(l_exact), (loss, l_exact)
    assert bn_err < BN_TOL, bn_err
    assert not bad, bad


# The output subsets the Python API asks predict() for (network.py): mode='denoise' (mean), the latent alone,
# mode='full' (mean + latent), return_info=True (everything) and the per-gene theta call of _predict_batches.
SUBSETS = {"denoise": ("mean",), "latent": ("latent",), "full": ("mean", "latent"),
           "info": ("mean", "dispersion", "pi", "latent"), "theta": ("dispersion",)}


def _head_outputs(ae_type):
    """The outputs of predict() that are head slots of the tensor-core heads kernel."""
    return ("mean",) + (("dispersion",) if ae_type.endswith("conddisp") else ()) + (("pi",) if ae_type.startswith("zinb") else ())


@pytest.mark.parametrize("ae_type", TYPES)
def test_tc_eval_and_predict(ae_type):
    """eval_step's loss and predict()'s outputs for every subset, with random BatchNorm moving statistics, against the
    inference forward of the references, row chunk by row chunk on the device.

    heads_forward runs the tensor-core heads kernel only when every head slot has an output; a subset that leaves one
    out (zinb and nb-conddisp: mode='denoise' and 'full'; nb-conddisp: the dispersion alone) runs the heads on the fp32
    CUDA-core GEMM from the fp32 last hidden layer instead.  Its outputs are held to the reference that rounds the
    encoder's operands to bf16 and keeps the heads exact; the tensor-core subsets to the same-rounding reference.  The
    per-gene theta of zinb / nb is clip(exp(raw), 1e-3, 1e4) of the stored parameter, bit for bit."""
    B = 4096
    Xd, Yd, sfd, rd = _batch(B)
    p0 = _start_params(ae_type, moving_stats=True)
    eng = _engine(ae_type, B, p0)
    cond, has_pi = ae_type.endswith("conddisp"), ae_type.startswith("zinb")
    eng.read_epoch_acc(reset=True)
    eng.eval_step(Xd, Yd, sfd, rows=rd)
    acc = eng.read_epoch_acc()
    outs = {}
    for sub, keys in SUBSETS.items():
        o = {}
        for k in keys:
            if k == "latent":
                o[k] = torch.full((B, HIDDEN[1]), float("nan"), device=DEV)
            elif k == "pi" and not has_pi:
                continue
            else:
                o[k] = torch.full((B, G) if (k != "dispersion" or cond) else (G,), float("nan"), device=DEV)
        eng.predict(Xd, sfd, rows=rd, mean=o.get("mean"), disp=o.get("dispersion"), pi=o.get("pi"), latent=o.get("latent"))
        outs[sub] = o
    torch.cuda.synchronize()
    eng.close(); del eng
    heads = _head_outputs(ae_type)
    tc_subsets = {sub for sub, keys in SUBSETS.items() if all(k in keys for k in heads)}
    fp32_subsets = {sub for sub, o in outs.items() if sub not in tc_subsets and any(k in heads for k in o)}
    print("\n[%s] predict subsets on the tensor-core heads: %s; on the fp32 CUDA-core heads: %s"
          % (ae_type, sorted(tc_subsets), sorted(fp32_subsets)))
    refs = {"same": _ref(p0, ae_type, emulate_bf16=True), "encoder": _ref(p0, ae_type, emulate_bf16="encoder"),
            "exact": _ref(p0, ae_type, emulate_bf16=False)}
    rel = {}                                      # (subset, output, reference) -> worst relative error
    nrm = {}                                      # (subset, output) -> [||got - exact||^2, ||exact||^2]
    loss_sum = {k: 0.0 for k in refs}
    rl = rd.long()
    with torch.no_grad():
        for s in range(0, B, CHUNK):
            r = rl[s:s + CHUNK]
            Xr, Yr, sfr = Xd[r].double(), Yd[r].double(), sfd[r].double()
            for rk, ref in refs.items():
                h, _, lat = ref.hidden_stack(Xr, training=False)
                mu, theta, pi = ref.head_outputs(h, sfr)
                loss_sum[rk] += float(ref._elem(Yr, mu, theta, pi).sum())
                want = {"mean": mu, "latent": lat, "dispersion": theta if cond else None, "pi": pi}
                for sub, o in outs.items():
                    for k, got in o.items():
                        if want[k] is None:
                            continue
                        got = got[s:s + CHUNK].double()
                        # absolute floors: pi as test_gpu_ragged_genes; the latent (pre-BatchNorm, crosses zero) 0.1 of its
                        # largest element
                        floor = {"pi": 1e-7 / PRED_TOL, "latent": 0.1 * float(lat.abs().max())}.get(k, 0.0)
                        e = ((got - want[k]).abs() / (want[k].abs() + floor)).max().item()
                        rel[(sub, k, rk)] = max(rel.get((sub, k, rk), 0.0), e)
                        if rk == "exact":
                            a = nrm.setdefault((sub, k), [0.0, 0.0])
                            a[0] += float(((got - want[k]) ** 2).sum()); a[1] += float((want[k] ** 2).sum())
    val = acc[2] / acc[3]
    ev = {rk: loss_sum[rk] / (B * G) for rk in refs}
    print("  eval loss %.7f, same-rounding %.7f (rel %.2e), exact %.7f (rel %.2e)"
          % (val, ev["same"], abs(val - ev["same"]) / ev["same"], ev["exact"], abs(val - ev["exact"]) / ev["exact"]))
    bad = []
    for sub, o in outs.items():
        for k in o:
            if k == "dispersion" and not cond:
                continue
            e_n = (nrm[(sub, k)][0] / nrm[(sub, k)][1]) ** 0.5
            print("  %-8s %-10s relative: same-rounding %.2e, bf16 encoder %.2e, exact %.2e; exact norm-wise %.2e"
                  % (sub, k, rel[(sub, k, "same")], rel[(sub, k, "encoder")], rel[(sub, k, "exact")], e_n))
            if k == "latent":
                checks = [("encoder", PRED_TOL), ("norm", TC_VS_EXACT["latent_same_weights"])]
            elif sub in tc_subsets:
                checks = [("same", PRED_TOL), ("norm", TC_VS_EXACT["predict_same_weights"])]
            else:
                checks = [("encoder", PRED_TOL), ("norm", TC_VS_EXACT["predict_same_weights"])]
            for rk, bound in checks:
                e = e_n if rk == "norm" else rel[(sub, k, rk)]
                if not e < bound:
                    bad.append((sub, k, rk, e, bound))
    if not cond:
        raw = torch.as_tensor(p0["dispersion/theta"]).to(DEV)
        theta = torch.clamp(torch.exp(raw), 1e-3, 1e4)
        for sub in ("info", "theta"):
            d = outs[sub]["dispersion"]
            print("  %-8s theta: %d of %d entries differ from clip(exp(raw))" % (sub, int((d != theta).sum()), G))
            assert torch.equal(d, theta), sub
    assert acc[3] == B * G
    assert abs(val - ev["same"]) < LOSS_TOL * ev["same"], (val, ev["same"])
    assert abs(val - ev["exact"]) < TC_VS_EXACT["loss"] * ev["exact"], (val, ev["exact"])
    assert not bad, bad


@pytest.mark.parametrize("ae_type", ["zinb", "nb"])
def test_tc_step_bits_run_to_run(ae_type):
    """Two engines with the same seed, three steps with updates on a side stream: the first a direct call, the second
    captured into a CUDA graph and launched, the third a graph replay.  Gradients, parameters and BatchNorm state
    agree bit for bit after every step: nothing on the path, dL/dtheta included, is summed in a run-dependent order."""
    B = 4096
    Xd, Yd, sfd, rd = _batch(B)
    stream = torch.cuda.Stream(DEV)
    with torch.cuda.stream(stream):
        a, b = _engine(ae_type, B, seed=7), _engine(ae_type, B, seed=7)
        assert torch.equal(a.params, b.params)
        for step in range(3):
            for e in (a, b):
                e.train_step(Xd, Yd, sfd, rows=rd)
                e.apply_update(1e-3, 5.0)
            stream.synchronize()
            same = {k: torch.equal(getattr(a, k), getattr(b, k)) for k in ("grads", "params", "bn_state")}
            diff = {k: int((getattr(a, k) != getattr(b, k)).sum()) for k, v in same.items() if not v}
            print("\n  [%s] step %d (graphs %d): identical %s, differing elements %s"
                  % (ae_type, step, a.info()["step_graphs"], same, diff))
            assert all(same.values()), (step, diff)
        assert a.info()["step_graphs"] >= 1 and b.info()["step_graphs"] >= 1
        a.close(); b.close()
    torch.cuda.synchronize()


@pytest.mark.parametrize("ae_type", ["nb", "zinb-conddisp"])
@pytest.mark.parametrize("optimizer", ["SGD", "Adagrad", "Adadelta", "Adam", "Adamax", "Nadam"])
def test_tc_optimizers_refresh_bf16_operands(optimizer, ae_type):
    """The tensor-core kernels read a bf16 copy of the parameters that the update kernel rewrites.  Engine A trains
    three steps with the optimizer; engine B starts from A's weights (set_weights casts the copy afresh).  One more step
    of both on a fresh batch gives bit-identical gradients, so no element of A's copy was left stale.  A's losses follow
    the same-rounding float64 reference running the same update rule."""
    B = 512
    Xd, Yd, sfd, rd = _batch(B)
    _, _, _, rd2 = _batch(B, seed=B + 1)
    p0 = _start_params(ae_type)
    a = _engine(ae_type, B, p0)
    lr = a.set_optimizer(optimizer)
    ref = _ref(p0, ae_type)
    ref.optimizer = optimizer
    rl = rd.long()
    Xr, Yr, sfr = Xd[rl].double(), Yd[rl].double(), sfd[rl].double()
    for step in range(3):
        a.train_step(Xd, Yd, sfd, rows=rd)
        a.apply_update(lr, 5.0)
        loss = a.read_loss()
        oloss, og, stats = ref.loss_and_grads_chunked(Xr, Yr, sfr, chunk=CHUNK)
        ref._apply(og, stats, lr, 5.0)
        print("\n  [%s %s] step %d: loss %.7f ref %.7f rel %.2e" % (optimizer, ae_type, step, loss, oloss, abs(loss - oloss) / oloss))
        assert abs(loss - oloss) < 5e-3 * abs(oloss), (step, loss, oloss)
    b = _engine(ae_type, B, a.get_weights())
    for e in (a, b):
        e.train_step(Xd, Yd, sfd, rows=rd2)
    torch.cuda.synchronize()
    n_diff = int((a.grads != b.grads).sum())
    print("  gradients of the fresh batch: %d of %d elements differ" % (n_diff, a.grads.numel()))
    assert torch.equal(a.grads, b.grads), n_diff
    a.close(); b.close()
