"""torch-CPU restatement of the reference training step -- TEST INFRASTRUCTURE ONLY.

Purpose (a) an autograd-based cross-check of the closed-form gradients in
``oracle/dca_oracle.py`` (autograd plays the role TF autodiff plays in the reference);
(b) the CPU baseline timed by ``bench.py`` ("torch-CPU restatement of the reference
path (TensorFlow unavailable in image)").

The op sequence mirrors what Keras executes for
  dca/network.py:92-141 (Dense -> BatchNormalization(center, no scale) -> relu),
  dca/network.py:366-393 / 496-522 / 293-316 (heads),  dca/layers.py:85 (mean * sf),
  dca/loss.py:72-156 (NB / ZINB NLL, every epsilon kept),
  dca/train.py:54-57 (RMSprop with clipvalue).
Never imported by the product package.
"""
from __future__ import annotations

import math
from typing import Dict, Sequence

import torch

from .dca_oracle import KERAS_DEFAULTS, layer_names, head_names

EPS = 1e-10


def hidden_activation(name, x, alpha=None):
    """Keras `Activation(name)` / `LeakyReLU()` / `PReLU()` as the reference applies them after every hidden layer
    (dca/network.py:129-135), written with torch's own functions (independent of the engine's closed forms)."""
    F = torch.nn.functional
    if name == "relu": return torch.relu(x)
    if name == "linear": return x
    if name == "elu": return F.elu(x)
    if name == "selu": return F.selu(x)
    if name == "tanh": return torch.tanh(x)
    if name == "sigmoid": return torch.sigmoid(x)
    if name == "hard_sigmoid": return torch.clamp(0.2 * x + 0.5, 0.0, 1.0)
    if name == "softplus": return F.softplus(x)
    if name == "softsign": return F.softsign(x)
    if name == "exponential": return torch.exp(x)
    if name == "LeakyReLU": return F.leaky_relu(x, 0.3)
    if name == "PReLU": return torch.relu(x) - alpha * torch.relu(-x)
    raise ValueError(name)


def bf16_round(t):
    """Round-to-nearest-even to bfloat16 of t's float32 value, returned in t's dtype (dca_oracle.bf16_round)."""
    return t.to(torch.float32).to(torch.bfloat16).to(t.dtype)


class RoundOperand(torch.autograd.Function):
    """A tensor-core GEMM operand: rounded to bf16 going forward; the gradient passes straight through to the fp32
    tensor it was rounded from (the engine keeps fp32 masters and activations)."""

    @staticmethod
    def forward(ctx, x):
        return bf16_round(x)

    @staticmethod
    def backward(ctx, g):
        return g


class RoundGrad(torch.autograd.Function):
    """Identity going forward; the gradient arriving here is rounded to bf16, as the engine rounds dZ and dA of the
    first layer before the tensor-core GEMMs read them."""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return bf16_round(g)


def apply_dropout(x, mask, rate):
    """keras.layers.Dropout in training mode with the mask handed in: x * mask / (1 - rate)  (dca/network.py:98-99,137-138)."""
    return x * mask.to(x.dtype).reshape(x.shape) / (1.0 - rate)


def nb_elem(y, mu, theta):
    theta = torch.clamp(theta, max=1e6)                                   # dca/loss.py:85
    t1 = torch.lgamma(theta + EPS) + torch.lgamma(y + 1.0) - torch.lgamma(y + theta + EPS)   # :87
    t2 = (theta + y) * torch.log(1.0 + (mu / (theta + EPS))) \
        + (y * (torch.log(theta + EPS) - torch.log(mu + EPS)))            # :88
    final = t1 + t2
    return torch.where(torch.isnan(final), torch.full_like(final, float("inf")), final)


def zinb_elem(y, mu, theta, pi, ridge=0.0):
    nb_case = nb_elem(y, mu, theta) - torch.log(1.0 - pi + EPS)           # :130
    th = torch.clamp(theta, max=1e6)
    zero_nb = torch.pow(th / (th + mu + EPS), th)                         # :136
    zero_case = -torch.log(pi + ((1.0 - pi) * zero_nb) + EPS)             # :137
    res = torch.where(y < 1e-8, zero_case, nb_case)                       # :138
    return res + ridge * pi * pi                                          # :139-140


def poisson_elem_sum_and_count(y, mu):
    """dca/loss.py:33-48: sum of  mu - y log(mu + 1e-10) + lgamma(y + 1)  over the non-NaN targets, and their count."""
    ok = ~torch.isnan(y)
    nelem = ok.to(mu.dtype).sum()
    nelem = torch.where(nelem == 0, torch.ones_like(nelem), nelem)
    y0 = torch.where(ok, y, torch.zeros_like(y))
    ret = mu - y0 * torch.log(mu + EPS) + torch.lgamma(y0 + 1.0)
    return ret.sum(), nelem


# ------------------------------------------------------------------------------------------------------------------
# The remaining registry keys of dca/network.py:763-768 (SURVEY.md 8f-4), each a re-parameterisation of the heads:
#   poisson      :233-246   mean head (MeanAct), poisson_loss (dca/loss.py:33-48)
#   normal       :143-156   LINEAR mean head, keras mean_squared_error
#   nb-shared    :341-363   dispersion = Dense(1, DispAct): one theta per CELL
#   zinb-shared  :465-493   pi = Dense(1, sigmoid) and dispersion = Dense(1, DispAct) per cell
#   zinb-elempi  :424-462   t = -Dense(G)(h); mean = MeanAct(t); pi = sigmoid(t * k + c) (ElementwiseDense, dca/layers.py:50-81;
#                           sharedpi: scalar k, c)
#   nb-fork / zinb-fork :553-760   the decoder layer(s) after 'center' exist once PER HEAD (own Dense + BatchNorm + act)
EXTRA_TYPES = ("poisson", "normal", "nb-shared", "zinb-shared", "zinb-elempi", "nb-fork", "zinb-fork")
FORK_BRANCHES = {"nb-fork": ("mean", "disp"), "zinb-fork": ("mean", "disp", "pi")}
BRANCH_HEAD = {"mean": "mean", "disp": "dispersion", "pi": "pi"}


def extra_init_params(n_in, n_out, hidden, ae_type, batchnorm=True, seed=0, dtype="float32", sharedpi=False):
    """Parameter dict (reference layer names) of the extra types, Glorot-uniform kernels / zero biases like Keras."""
    import numpy as np
    rng = np.random.default_rng(seed)
    hidden = tuple(hidden)
    names = layer_names(len(hidden))
    center = len(hidden) // 2
    p = {}

    def dense(name, fi, fo, shape=None):
        lim = math.sqrt(6.0 / (fi + fo))
        p[name + "/kernel"] = rng.uniform(-lim, lim, size=shape if shape is not None else (fi, fo)).astype(dtype)
        p[name + "/bias"] = np.zeros(fo if shape is None else shape, dtype)

    def bn(name, h):
        if batchnorm:
            p[name + "/bn_beta"] = np.zeros(h, dtype); p[name + "/bn_moving_mean"] = np.zeros(h, dtype)
            p[name + "/bn_moving_var"] = np.ones(h, dtype)
    prev = n_in
    fork = FORK_BRANCHES.get(ae_type)
    last = {}
    for i, (nm, h) in enumerate(zip(names, hidden)):
        if fork and i > center:
            for br in fork:                               # every fork layer starts from the trunk (dca/network.py:586-596)
                dense("%s_last_%s" % (nm, br), prev, h); bn("%s_last_%s" % (nm, br), h); last[br] = h
            continue
        dense(nm, prev, h); bn(nm, h); prev = h
    kin = lambda br: last.get(br, prev)
    if ae_type in ("poisson", "normal"):
        dense("mean", prev, n_out)
    elif ae_type == "nb-shared":
        dense("dispersion", prev, 1); dense("mean", prev, n_out)
    elif ae_type == "zinb-shared":
        dense("pi", prev, 1); dense("dispersion", prev, 1); dense("mean", prev, n_out)
    elif ae_type == "zinb-elempi":
        dense("dispersion", prev, n_out); dense("mean_no_act", prev, n_out)
        npi = 1 if sharedpi else n_out
        dense("pi", npi, npi, shape=(npi,))               # 1-D kernel: Keras computes fan_in = fan_out = shape[0]
    elif ae_type == "nb-fork":
        dense("dispersion", kin("disp"), n_out); dense("mean", kin("mean"), n_out)
    elif ae_type == "zinb-fork":
        dense("pi", kin("pi"), n_out); dense("dispersion", kin("disp"), n_out); dense("mean", kin("mean"), n_out)
    else:
        raise KeyError(ae_type)
    return p


class TorchExtraNet:
    """float64 autograd statement of one training step of the extra types (the role TF autodiff plays in the reference);
    same parameter names as the engine.  TEST INFRASTRUCTURE ONLY."""

    def __init__(self, params, hidden, ae_type, batchnorm=True, ridge=0.0, dtype=torch.float64, activation="relu",
                 device="cpu"):
        assert ae_type in EXTRA_TYPES
        self.hidden = tuple(hidden); self.ae_type = ae_type; self.batchnorm = batchnorm; self.ridge = ridge; self.dtype = dtype
        self.activation = activation; self.device = torch.device(device)
        self.masks = {}; self.rates = {}      # dropout: layer id (-1 input, i hidden, 8 + b fork branch) -> keep mask / rate
        self.names = layer_names(len(self.hidden)); self.center = len(self.hidden) // 2
        self.p = {k: torch.as_tensor(v).to(self.device, dtype).clone() for k, v in params.items()}
        self.train_keys = [k for k in self.p if k.endswith(("/kernel", "/bias", "/bn_beta", "_act/alpha"))]
        for k in self.train_keys:
            self.p[k].requires_grad_(True)
        self.rms = {k: torch.zeros_like(self.p[k]) for k in self.train_keys}
        self.mom = KERAS_DEFAULTS["bn_momentum"]; self.bn_eps = KERAS_DEFAULTS["bn_eps"]

    def _layer(self, h, nm, training, stats, lid=None):
        a = h @ self.p[nm + "/kernel"] + self.p[nm + "/bias"]
        pre = a
        if self.batchnorm:
            if training:
                mean = a.mean(0); var = a.var(0, unbiased=False)
                stats.append((nm, mean.detach(), var.detach()))
            else:
                mean = self.p[nm + "/bn_moving_mean"]; var = self.p[nm + "/bn_moving_var"]
            pre = (a - mean) / torch.sqrt(var + self.bn_eps) + self.p[nm + "/bn_beta"]
        out = hidden_activation(self.activation, pre, self.p.get(nm + "_act/alpha"))
        if training and lid in self.masks:
            out = apply_dropout(out, self.masks[lid], self.rates[lid])
        return a, out

    def hidden_stack(self, X, training=True):
        """(head inputs {branch: activation}, latent, BatchNorm batch statistics): everything in front of the heads."""
        stats = []
        h = X; latent = None
        if training and -1 in self.masks:
            h = apply_dropout(h, self.masks[-1], self.rates[-1])
        fork = FORK_BRANCHES.get(self.ae_type)
        branch = {}
        for i, nm in enumerate(self.names):
            if fork and i > self.center:
                for b, br in enumerate(fork):
                    _, branch[br] = self._layer(h, "%s_last_%s" % (nm, br), training, stats, 8 + b)
                continue
            a, h = self._layer(h, nm, training, stats, i)
            if nm == "center":
                latent = a
        return {br: branch.get(br, h) for br in ("mean", "disp", "pi")}, latent, stats

    def forward(self, X, sf, training=True):
        ins, latent, stats = self.hidden_stack(X, training)
        out = self.heads(ins, sf)
        out.update(latent=latent, stats=stats)
        return out

    def heads(self, ins, sf):
        """mean / dispersion / pi of the rows of ``ins`` (one activation per branch; all three are the trunk's
        last activation except for the fork types)."""
        h = ins["mean"]
        dense = lambda nm, x: x @ self.p[nm + "/kernel"] + self.p[nm + "/bias"]
        sfc = sf.reshape(-1, 1)
        out = {}
        t = self.ae_type
        if t == "normal":
            out["mean"] = dense("mean", h) * sfc
        elif t == "zinb-elempi":
            tt = -dense("mean_no_act", h)
            out["pi"] = torch.sigmoid(tt * self.p["pi/kernel"] + self.p["pi/bias"]) * torch.ones_like(tt)
            out["mean"] = torch.clamp(torch.exp(tt), 1e-5, 1e6) * sfc
            out["dispersion"] = torch.clamp(torch.nn.functional.softplus(dense("dispersion", h)), 1e-4, 1e4)
        else:
            out["mean"] = torch.clamp(torch.exp(dense("mean", ins["mean"])), 1e-5, 1e6) * sfc
            if t != "poisson":
                out["dispersion"] = torch.clamp(torch.nn.functional.softplus(dense("dispersion", ins["disp"])), 1e-4, 1e4)
            if t in ("zinb-shared", "zinb-fork"):
                out["pi"] = torch.sigmoid(dense("pi", ins["pi"]))
        return out

    def _loss_sum(self, o, Y):
        """Sum of the element losses of the rows in ``o`` (not divided by the element count)."""
        mu = o["mean"]
        if self.ae_type == "normal":
            return ((mu - Y) ** 2).sum()                                 # keras mean_squared_error
        if self.ae_type == "poisson":
            return poisson_elem_sum_and_count(Y, mu)[0]
        if "pi" in o:
            return zinb_elem(Y, mu, o["dispersion"].expand_as(mu), o["pi"].expand_as(mu), self.ridge).sum()
        return nb_elem(Y, mu, o["dispersion"].expand_as(mu)).sum()

    def _n_elem(self, Y):
        """The loss is a mean over this many elements (poisson: the non-NaN targets, at least one)."""
        if self.ae_type == "poisson":
            return poisson_elem_sum_and_count(Y, torch.ones_like(Y))[1]
        return Y.numel()

    def loss(self, X, Y, sf, training=True):
        o = self.forward(X, sf, training)
        return self._loss_sum(o, Y) / self._n_elem(Y), o["stats"]

    def _grads(self):
        return {k: (self.p[k].grad.detach().clone() if self.p[k].grad is not None else torch.zeros_like(self.p[k]))
                for k in self.train_keys}

    def loss_and_grads(self, X, Y, sf):
        for k in self.train_keys:
            self.p[k].grad = None
        loss, stats = self.loss(X, Y, sf, True)
        loss.backward()
        return float(loss.detach()), self._grads(), stats

    def loss_and_grads_chunked(self, X, Y, sf, chunk=256):
        """loss_and_grads with the heads and the loss evaluated ``chunk`` rows at a time, so that the autograd graph of
        the B x G head and loss tensors exists for one chunk only.  The hidden stack runs on the whole batch (BatchNorm
        needs the batch statistics); its outputs become leaves whose gradient the chunks accumulate, and that gradient
        is then backpropagated through the stack once.  Same mean loss and gradients as loss_and_grads."""
        for k in self.train_keys:
            self.p[k].grad = None
        ins, _, stats = self.hidden_stack(X, True)
        leaves = {}                                       # one leaf per distinct tensor (branches may share the trunk)
        for v in ins.values():
            if id(v) not in leaves:
                leaves[id(v)] = (v, v.detach().requires_grad_(True))
        lins = {br: leaves[id(v)][1] for br, v in ins.items()}
        n = self._n_elem(Y)
        total = 0.0
        for s in range(0, X.shape[0], chunk):
            o = self.heads({br: v[s:s + chunk] for br, v in lins.items()}, sf[s:s + chunk])
            part = self._loss_sum(o, Y[s:s + chunk])
            (part / n).backward()
            total += float(part.detach())
        outs = [(v, leaf.grad) for v, leaf in leaves.values() if v.requires_grad and leaf.grad is not None]
        if outs:
            torch.autograd.backward([v for v, _ in outs], [g for _, g in outs])
        return total / float(n), self._grads(), stats

    _apply = None

    def train_step(self, X, Y, sf, lr=KERAS_DEFAULTS["rms_lr"], clip=KERAS_DEFAULTS["clipvalue"]):
        loss, grads, stats = self.loss_and_grads(X, Y, sf)
        TorchRefNet._apply(self, grads, stats, lr, clip)
        return loss

    @torch.no_grad()
    def predict(self, X, sf):
        o = self.forward(X, sf, False)
        return {k: v.detach().cpu().numpy() for k, v in o.items() if k != "stats" and v is not None}


class TorchRefNet:
    """Same parameter names / layouts as oracle.dca_oracle.OracleNet.

    emulate_bf16 ("both" | "encoder" | "heads" | "none", True / False = "both" / "none") has OracleNet's meaning: the
    same-rounding statement of the tensor-core path (DESIGN section 3).  "encoder" rounds X (after input dropout) and the
    first kernel going forward and dA of the first layer going backward; "heads" rounds the last hidden activation
    (after dropout) and the head kernels going forward and dZ going backward.  Everything else stays in ``dtype``."""

    def __init__(self, params: Dict[str, "torch.Tensor"], hidden: Sequence[int], ae_type: str,
                 batchnorm=True, ridge=0.0, dtype=torch.float32, activation="relu", device="cpu", emulate_bf16=False):
        side = {True: "both", False: "none"}.get(emulate_bf16, emulate_bf16)
        assert side in ("both", "none", "encoder", "heads"), emulate_bf16
        self.rnd_enc = side in ("both", "encoder"); self.rnd_heads = side in ("both", "heads")
        self.hidden = tuple(hidden); self.ae_type = ae_type; self.batchnorm = batchnorm
        self.ridge = ridge; self.dtype = dtype; self.activation = activation; self.device = torch.device(device)
        self.masks = {}; self.rates = {}      # dropout: layer id (-1 input, i hidden) -> keep mask / rate
        self.names = layer_names(len(self.hidden)); self.heads = head_names(ae_type)
        self.p = {k: torch.as_tensor(v).to(self.device, dtype).clone() for k, v in params.items()}
        self.train_keys = [k for k in self.p if k.endswith(("/kernel", "/bias", "/bn_beta", "/theta", "_act/alpha"))]
        for k in self.train_keys:
            self.p[k].requires_grad_(True)
        self.rms = {k: torch.zeros_like(self.p[k]) for k in self.train_keys}
        self.mom = KERAS_DEFAULTS["bn_momentum"]; self.bn_eps = KERAS_DEFAULTS["bn_eps"]

    def forward(self, X, sf, training=True):
        h, stats, _ = self.hidden_stack(X, training)
        return self.head_outputs(h, sf) + (stats,)

    def hidden_stack(self, X, training=True):
        """(last hidden activation, BatchNorm batch statistics, latent: the pre-BatchNorm output of 'center')."""
        h = X; latent = None
        if training and -1 in self.masks:
            if self.rnd_enc:
                # the device scales fp32 X by fp32(1 / keep) and rounds that product to bf16: a 1-ulp difference in the
                # scale would move ~2^-16 of the elements across a bf16 rounding boundary, by 2^-8 of their value.  The
                # product of two fp32 values is exact in float64; its float32 rounding is the device's product.
                one = torch.tensor(1.0, dtype=torch.float32)
                inv_keep = float(one / (one - torch.tensor(self.rates[-1], dtype=torch.float32)))
                h = (h * self.masks[-1].to(h.dtype).reshape(h.shape) * inv_keep).to(torch.float32).to(h.dtype)
            else:
                h = apply_dropout(h, self.masks[-1], self.rates[-1])
        stats = []
        for i, nm in enumerate(self.names):
            if i == 0 and self.rnd_enc:
                a = RoundGrad.apply(RoundOperand.apply(h) @ RoundOperand.apply(self.p[nm + "/kernel"])) + self.p[nm + "/bias"]
            else:
                a = h @ self.p[nm + "/kernel"] + self.p[nm + "/bias"]
            if nm == "center":
                latent = a
            if self.batchnorm:
                if training:
                    mean = a.mean(0); var = a.var(0, unbiased=False)
                    stats.append((nm, mean.detach(), var.detach()))
                else:
                    mean = self.p[nm + "/bn_moving_mean"]; var = self.p[nm + "/bn_moving_var"]
                a = (a - mean) / torch.sqrt(var + self.bn_eps) + self.p[nm + "/bn_beta"]
            h = hidden_activation(self.activation, a, self.p.get(nm + "_act/alpha"))
            if training and i in self.masks:
                h = apply_dropout(h, self.masks[i], self.rates[i])
        return h, stats, latent

    def head_outputs(self, h, sf):
        """(mu, theta, pi) of the rows of h; theta is [1 x G] for the per-gene dispersion types, pi None for NB."""
        if self.rnd_heads:
            hr = RoundOperand.apply(h)
            z = {nm: RoundGrad.apply(hr @ RoundOperand.apply(self.p[nm + "/kernel"]) + self.p[nm + "/bias"]) for nm in self.heads}
        else:
            z = {nm: h @ self.p[nm + "/kernel"] + self.p[nm + "/bias"] for nm in self.heads}
        m = torch.clamp(torch.exp(z["mean"]), 1e-5, 1e6)
        mu = m * sf.reshape(-1, 1)
        if "dispersion" in z:
            theta = torch.clamp(torch.nn.functional.softplus(z["dispersion"]), 1e-4, 1e4)
        else:
            theta = torch.clamp(torch.exp(self.p["dispersion/theta"]), 1e-3, 1e4).reshape(1, -1)
        pi = torch.sigmoid(z["pi"]) if "pi" in z else None
        return mu, theta, pi

    def _elem(self, Y, mu, theta, pi):
        theta = theta.expand_as(mu)
        return zinb_elem(Y, mu, theta, pi, self.ridge) if pi is not None else nb_elem(Y, mu, theta)

    def loss(self, X, Y, sf, training=True):
        mu, theta, pi, stats = self.forward(X, sf, training)
        return self._elem(Y, mu, theta, pi).mean(), stats

    def loss_and_grads(self, X, Y, sf):
        for k in self.train_keys:
            self.p[k].grad = None
        loss, stats = self.loss(X, Y, sf, True)
        loss.backward()
        return float(loss.detach()), {k: self.p[k].grad.detach().clone() for k in self.train_keys}, stats

    def loss_and_grads_chunked(self, X, Y, sf, chunk=256):
        """loss_and_grads with the heads and the loss evaluated ``chunk`` rows at a time, so that the autograd graph of
        the B x G head and loss tensors exists for one chunk only (a 4096 x 20000 float64 ZINB graph in one piece
        holds tens of GB).  The hidden stack runs on the whole batch (BatchNorm needs the batch statistics); its last
        activation becomes a leaf whose gradient the chunks accumulate, and that gradient is then backpropagated
        through the stack once.  Same mean loss and gradients as loss_and_grads."""
        for k in self.train_keys:
            self.p[k].grad = None
        h, stats, _ = self.hidden_stack(X, True)
        leaf = h.detach().requires_grad_(True)
        n = Y.numel()
        total = 0.0
        for s in range(0, X.shape[0], chunk):
            mu, theta, pi = self.head_outputs(leaf[s:s + chunk], sf[s:s + chunk])
            part = self._elem(Y[s:s + chunk], mu, theta, pi).sum()
            (part / n).backward()
            total += float(part.detach())
        if h.requires_grad:
            h.backward(leaf.grad)
        grads = {k: (self.p[k].grad.detach().clone() if self.p[k].grad is not None else torch.zeros_like(self.p[k]))
                 for k in self.train_keys}
        return total / n, grads, stats

    @torch.no_grad()
    def _apply(self, grads, stats, lr, clip):
        """Optimizer step.  self.optimizer (default 'RMSprop') names a keras.optimizers class; the rules restate
        `get_updates` of Keras 2.x keras/optimizers.py (a dependency of the reference, pinned `keras>=2.0.8` in its
        setup.py, not vendored) with every hyper-parameter but lr / clipvalue at the class default, epsilon = K.epsilon()
        = 1e-7, decay 0 -- what `opt.__dict__[optimizer](clipvalue=clip_grad[, lr=...])` (dca/train.py:54-57) builds."""
        kind = getattr(self, "optimizer", "RMSprop")
        rho = KERAS_DEFAULTS["rms_rho"]; eps = KERAS_DEFAULTS["rms_eps"]
        if kind != "RMSprop":
            if not hasattr(self, "opt2"):
                self.opt2 = {k: torch.zeros_like(v) for k, v in self.rms.items()}; self.opt_t = 0; self.m_sched = 1.0
            self.opt_t += 1
            t = self.opt_t; b1, b2 = 0.9, 0.999
            if kind == "Nadam":
                mu_t = b1 * (1.0 - 0.5 * 0.96 ** (t * 0.004)); mu_t1 = b1 * (1.0 - 0.5 * 0.96 ** ((t + 1) * 0.004))
                sched_new = self.m_sched * mu_t; sched_next = sched_new * mu_t1; self.m_sched = sched_new
        for k, g in grads.items():
            g = g.clamp(-clip, clip)
            if kind == "RMSprop":
                self.rms[k].mul_(rho).addcmul_(g, g, value=1.0 - rho)
                self.p[k].sub_(lr * g / (self.rms[k].sqrt() + eps))
                continue
            a, b2s = self.rms[k], self.opt2[k]
            if kind == "SGD":
                self.p[k].sub_(lr * g)
            elif kind == "Adagrad":
                a.add_(g * g); self.p[k].sub_(lr * g / (a.sqrt() + eps))
            elif kind == "Adadelta":
                a.mul_(0.95).add_(0.05 * g * g)
                upd = g * (b2s + eps).sqrt() / (a + eps).sqrt()
                self.p[k].sub_(lr * upd)
                b2s.mul_(0.95).add_(0.05 * upd * upd)
            elif kind == "Adam":
                lr_t = lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
                a.mul_(b1).add_((1 - b1) * g); b2s.mul_(b2).add_((1 - b2) * g * g)
                self.p[k].sub_(lr_t * a / (b2s.sqrt() + eps))
            elif kind == "Adamax":
                lr_t = lr / (1.0 - b1 ** t)
                a.mul_(b1).add_((1 - b1) * g); torch.maximum(b2 * b2s, g.abs(), out=b2s)
                self.p[k].sub_(lr_t * a / (b2s + eps))
            elif kind == "Nadam":
                gp = g / (1.0 - sched_new)
                a.mul_(b1).add_((1 - b1) * g); mp = a / (1.0 - sched_next)
                b2s.mul_(b2).add_((1 - b2) * g * g); vp = b2s / (1.0 - b2 ** t)
                mbar = (1.0 - mu_t) * gp + mu_t1 * mp
                self.p[k].sub_(lr * mbar / (vp.sqrt() + eps))
            else:
                raise ValueError(kind)
        for nm, mean, var in stats:
            self.p[nm + "/bn_moving_mean"].mul_(self.mom).add_((1 - self.mom) * mean)
            self.p[nm + "/bn_moving_var"].mul_(self.mom).add_((1 - self.mom) * var)

    def train_step(self, X, Y, sf, lr=KERAS_DEFAULTS["rms_lr"], clip=KERAS_DEFAULTS["clipvalue"]):
        loss, grads, stats = self.loss_and_grads(X, Y, sf)
        self._apply(grads, stats, lr, clip)
        return loss
