"""CPU oracle for the DCA training hot path -- TEST INFRASTRUCTURE ONLY.

This module is a NumPy restatement (float64 by default, float32 on request) of the
arithmetic that theislab/dca executes through Keras/TensorFlow on the path

    dca/train.py:35-100  ->  dca/network.py:92-141,366-393  ->  dca/loss.py:60-156

It is the checker for the CUDA kernels in ``dca_b200/csrc``.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s cpu-baseline / ``--impl reference``
legs may import it; the product package ``dca_b200`` never does.

PARITY STATUS: "parity unpinned" for the autoencoder path.  TensorFlow / Keras /
scanpy are not installable in this image (SURVEY.md section 8c), so this restatement
cannot be run against the reference itself.  What IS pinned: the NB / ZINB loss
formulas are checked against the reference's own R-fitted fixtures
(data/biochemists-*.tsv, see tests/golden/make_golden.py and
tests/test_oracle_golden.py).  Third-party defaults that are restated from API
knowledge are collected in ``KERAS_DEFAULTS`` below so they can be corrected in
one place.

Every function cites the reference file:line it follows (paths relative to the
reference repository root).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
from scipy import special as _sp

# ----------------------------------------------------------------------------
# Third-party defaults (Keras 2.4 / TF 2.x / scanpy) -- SURVEY.md Appendix B.
# ----------------------------------------------------------------------------
KERAS_DEFAULTS = dict(
    bn_momentum=0.99,      # keras.layers.BatchNormalization(momentum=0.99)
    bn_eps=1e-3,           # keras.layers.BatchNormalization(epsilon=1e-3)
    rms_lr=1e-3,           # keras.optimizers.RMSprop(lr=0.001)
    rms_rho=0.9,           # rho=0.9
    rms_eps=1e-7,          # epsilon=K.epsilon()=1e-7, added OUTSIDE the sqrt
    clipvalue=5.0,         # dca/train.py:37 clip_grad=5.
    plateau_factor=0.1,    # ReduceLROnPlateau(factor=0.1, min_delta=1e-4, cooldown=0, min_lr=0)
    plateau_min_delta=1e-4,
    validation_split=0.1,  # dca/train.py:38
)

LOSS_EPS = 1e-10           # dca/loss.py:65

AE_TYPES = ("zinb-conddisp", "zinb", "nb-conddisp", "nb")


def bf16_round(a):
    """Round-to-nearest-even to bfloat16 precision (8-bit mantissa), returned in a's dtype.
    Used by the "same-rounding" oracle that mirrors where the tcgen05 path rounds its GEMM operands."""
    a = np.asarray(a)
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    r = ((u >> 16) & 1) + np.uint32(0x7FFF)
    out = ((u + r) & np.uint32(0xFFFF0000)).view(np.float32)
    return out.astype(a.dtype).reshape(a.shape)


# ----------------------------------------------------------------------------
# Activations (dca/network.py:38-39, 369)
# ----------------------------------------------------------------------------
def softplus(x):
    x = np.asarray(x)
    return np.logaddexp(x, np.zeros_like(x))


def sigmoid(x):
    x = np.asarray(x)
    return np.where(x >= 0, 1.0 / (1.0 + np.exp(-np.abs(x))),
                    np.exp(-np.abs(x)) / (1.0 + np.exp(-np.abs(x)))).astype(x.dtype)


def mean_act(x):
    """MeanAct = clip(exp(x), 1e-5, 1e6) -- dca/network.py:38."""
    with np.errstate(over="ignore"):
        return np.clip(np.exp(x), 1e-5, 1e6).astype(np.asarray(x).dtype)


def disp_act(x):
    """DispAct = clip(softplus(x), 1e-4, 1e4) -- dca/network.py:39."""
    return np.clip(softplus(x), 1e-4, 1e4).astype(np.asarray(x).dtype)


def theta_const(theta_raw):
    """ConstantDispersionLayer: clip(exp(theta), 1e-3, 1e4) -- dca/layers.py:17-21."""
    with np.errstate(over="ignore"):
        return np.clip(np.exp(theta_raw), 1e-3, 1e4)


# ----------------------------------------------------------------------------
# Loss (dca/loss.py:72-156), element-wise, no reduction
# ----------------------------------------------------------------------------
def nb_loss_elem(y, mu, theta, eps=LOSS_EPS):
    """NB.loss with mean=False -- dca/loss.py:85-105 (scale_factor=1, masking=False)."""
    dt = np.result_type(y, mu, theta)
    y = np.asarray(y, dt); mu = np.asarray(mu, dt); theta = np.asarray(theta, dt)
    theta = np.minimum(theta, dt.type(1e6))                                   # :85
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        t1 = _sp.gammaln(theta + eps) + _sp.gammaln(y + 1.0) - _sp.gammaln(y + theta + eps)   # :87
        t2 = (theta + y) * np.log(1.0 + (mu / (theta + eps))) \
            + (y * (np.log(theta + eps) - np.log(mu + eps)))                  # :88
        final = t1 + t2
    final = np.where(np.isnan(final), np.inf, final)                          # :105 _nan2inf
    return final.astype(dt)


def zinb_loss_elem(y, mu, theta, pi, ridge=0.0, eps=LOSS_EPS):
    """ZINB.loss with mean=False -- dca/loss.py:130-140."""
    dt = np.result_type(y, mu, theta, pi)
    y = np.asarray(y, dt); mu = np.asarray(mu, dt)
    theta = np.asarray(theta, dt); pi = np.asarray(pi, dt)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        nb_case = nb_loss_elem(y, mu, theta, eps) - np.log(1.0 - pi + eps)    # :130
        th = np.minimum(theta, dt.type(1e6))                                  # :134
        zero_nb = np.power(th / (th + mu + eps), th)                          # :136
        zero_case = -np.log(pi + ((1.0 - pi) * zero_nb) + eps)                # :137
        result = np.where(y < 1e-8, zero_case, nb_case)                       # :138
        result = result + ridge * np.square(pi)                               # :139-140
    return result.astype(dt)


def reduce_loss(elem):
    """tf.reduce_mean followed by _nan2inf -- dca/loss.py:107-111, 142-148."""
    m = np.mean(elem, dtype=np.float64) if elem.size else np.float64("nan")
    return np.inf if np.isnan(m) else float(m)


def nb_loss(y, mu, theta):
    return reduce_loss(nb_loss_elem(y, mu, theta))


def zinb_loss(y, mu, theta, pi, ridge=0.0):
    return reduce_loss(zinb_loss_elem(y, mu, theta, pi, ridge))


# ----------------------------------------------------------------------------
# Closed-form derivatives of the element-wise loss with respect to (mu, theta, pi)
# (what TF autodiff produces for dca/loss.py; SURVEY.md A.4).  NOT divided by N.
# ----------------------------------------------------------------------------
def loss_partials(y, mu, theta, pi=None, ridge=0.0, eps=LOSS_EPS):
    """Return (dL/dmu, dL/dtheta, dL/dpi) per element. pi=None -> NB only (dpi = None)."""
    dt = np.result_type(y, mu, theta)
    y = np.asarray(y, dt); mu = np.asarray(mu, dt); theta = np.asarray(theta, dt)
    th = np.minimum(theta, dt.type(1e6))
    th_pass = (theta <= 1e6).astype(dt)           # gradient of tf.minimum(theta, 1e6)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        te = th + eps
        # nb branch
        dmu_nb = (th + y) / (te + mu) - y / (mu + eps)
        dth_nb = (_sp.digamma(te) - _sp.digamma(y + te) + np.log(1.0 + mu / te)
                  - (th + y) * mu / (te * (te + mu)) + y / te)
        if pi is None:
            return dmu_nb, dth_nb * th_pass, None
        pi = np.asarray(pi, dt)
        dpi_nb = 1.0 / (1.0 - pi + eps)
        # zero branch
        den = th + mu + eps
        r = th / den
        z = np.power(r, th)
        D = pi + (1.0 - pi) * z + eps
        w = (1.0 - pi) / D * z
        dmu_z = w * th / den
        # d/dtheta [theta * log(theta/(theta+mu+eps))] = log r + 1 - r   (r = theta/den)
        dth_z = -w * (np.log(r) + 1.0 - r)
        dpi_z = -(1.0 - z) / D
        zero = y < 1e-8
        dmu = np.where(zero, dmu_z, dmu_nb)
        dth = np.where(zero, dth_z, dth_nb) * th_pass
        dpi = np.where(zero, dpi_z, dpi_nb) + 2.0 * ridge * pi
    return dmu, dth, dpi


def head_grads_from_preact(y, sf, zm, zd=None, zp=None, theta_raw=None, ridge=0.0,
                           n_norm=None):
    """Forward loss + gradients w.r.t. head pre-activations.

    zm: mean pre-activation (B,G); zd: dispersion pre-activation or None (const-disp,
    then theta_raw (G,) is used); zp: pi pre-activation or None (NB models).
    Returns dict(loss, dzm, dzd|dtheta_raw, dzp, m, d, pi).  Gradients are of the MEAN
    loss (divided by n_norm = B*G by default).
    Follows dca/network.py:366-393 (heads), dca/layers.py:85 (mean*sf), dca/loss.py.
    """
    zm = np.asarray(zm)
    dt = zm.dtype
    B, G = zm.shape
    n = float(B * G) if n_norm is None else float(n_norm)
    sf = np.asarray(sf, dt).reshape(-1, 1)
    with np.errstate(over="ignore"):
        em = np.exp(zm)
    m = np.clip(em, 1e-5, 1e6).astype(dt)
    m_pass = ((em >= 1e-5) & (em <= 1e6)).astype(dt)    # tf.clip_by_value grad, inclusive
    mu = m * sf
    out = {"m": m}
    if zd is not None:
        sp = softplus(np.asarray(zd, dt))
        d = np.clip(sp, 1e-4, 1e4).astype(dt)
        d_pass = ((sp >= 1e-4) & (sp <= 1e4)).astype(dt)
        theta = d
    else:
        with np.errstate(over="ignore"):
            et = np.exp(np.asarray(theta_raw, dt))
        theta_g = np.clip(et, 1e-3, 1e4).astype(dt)
        t_pass = ((et >= 1e-3) & (et <= 1e4)).astype(dt)
        theta = np.broadcast_to(theta_g.reshape(1, -1), (B, G))
        d = theta_g
    out["d"] = d
    pi = None
    if zp is not None:
        pi = sigmoid(np.asarray(zp, dt))
        out["pi"] = pi
        elem = zinb_loss_elem(y, mu, theta, pi, ridge)
    else:
        elem = nb_loss_elem(y, mu, theta)
    out["elem"] = elem
    out["loss"] = reduce_loss(elem) if n_norm is None else float(np.sum(elem, dtype=np.float64) / n)
    dmu, dth, dpi = loss_partials(y, mu, theta, pi, ridge)
    out["dzm"] = (dmu * sf * m * m_pass / n).astype(dt)
    if zd is not None:
        out["dzd"] = (dth * sigmoid(np.asarray(zd, dt)) * d_pass / n).astype(dt)
    else:
        out["dtheta_raw"] = (np.sum(dth, axis=0) * theta_g * t_pass / n).astype(dt)
    if zp is not None:
        out["dzp"] = (dpi * pi * (1.0 - pi) / n).astype(dt)
    return out


# ----------------------------------------------------------------------------
# Pre-processing restatement (dca/io.py:88-111 + the scanpy calls it makes)
# ----------------------------------------------------------------------------
def normalize_inputs(Y, size_factors=True, logtrans_input=True, normalize_input=True):
    """Return (X, sf) from raw counts Y (cells x genes), float32 like scanpy.

    sc.pp.normalize_per_cell: X = Y / n_counts * median(n_counts)      (dca/io.py:99-100)
    sf = n_counts / median(n_counts)                                   (dca/io.py:101)
    sc.pp.log1p (natural log)                                          (dca/io.py:105-106)
    sc.pp.scale: per-gene zero mean / unit variance, ddof=1, no clip   (dca/io.py:108-109)
    """
    Y = np.asarray(Y, dtype=np.float32)
    n_counts = Y.sum(axis=1, dtype=np.float64)
    if size_factors:
        med = np.median(n_counts)
        sf = (n_counts / med)
        X = (Y / sf[:, None].astype(np.float32)).astype(np.float32)
    else:
        sf = np.ones(Y.shape[0], dtype=np.float64)
        X = Y.copy()
    if logtrans_input:
        X = np.log1p(X)
    if normalize_input:
        mean = X.mean(axis=0, dtype=np.float64)
        var = X.var(axis=0, ddof=1, dtype=np.float64)
        std = np.sqrt(var)
        std[std == 0] = 1.0
        X = ((X - mean) / std).astype(np.float32)
    return X.astype(np.float32), sf.astype(np.float32)


# ----------------------------------------------------------------------------
# The network (dca/network.py) as plain arrays, with manual backprop
# ----------------------------------------------------------------------------
def layer_names(n_hidden: int) -> List[str]:
    """enc{i} / center / dec{i} naming -- dca/network.py:102-111."""
    center = int(np.floor(n_hidden / 2.0))
    names = []
    for i in range(n_hidden):
        if i == center:
            names.append("center")
        elif i < center:
            names.append("enc%d" % i)
        else:
            names.append("dec%d" % (i - center))
    return names


def head_names(ae_type: str) -> List[str]:
    return {"zinb-conddisp": ["mean", "dispersion", "pi"],
            "zinb": ["mean", "pi"],
            "nb-conddisp": ["mean", "dispersion"],
            "nb": ["mean"]}[ae_type]


def glorot_uniform(rng, fan_in, fan_out, dtype=np.float32):
    lim = math.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-lim, lim, size=(fan_in, fan_out)).astype(dtype)


def init_params(n_in, n_out, hidden=(64, 32, 64), ae_type="zinb-conddisp", batchnorm=True,
                seed=0, dtype=np.float32) -> Dict[str, np.ndarray]:
    """Parameter dict with the reference's tensor names (Keras layer names)."""
    rng = np.random.default_rng(seed)
    p: Dict[str, np.ndarray] = {}
    prev = n_in
    for nm, h in zip(layer_names(len(hidden)), hidden):
        p[nm + "/kernel"] = glorot_uniform(rng, prev, h, dtype)
        p[nm + "/bias"] = np.zeros(h, dtype)
        if batchnorm:
            p[nm + "/bn_beta"] = np.zeros(h, dtype)
            p[nm + "/bn_moving_mean"] = np.zeros(h, dtype)
            p[nm + "/bn_moving_var"] = np.ones(h, dtype)
        prev = h
    for nm in head_names(ae_type):
        p[nm + "/kernel"] = glorot_uniform(rng, prev, n_out, dtype)
        p[nm + "/bias"] = np.zeros(n_out, dtype)
    if ae_type in ("zinb", "nb"):
        p["dispersion/theta"] = np.zeros(n_out, dtype)      # dca/layers.py:17-20
    return p


TRAINABLE_SUFFIX = ("/kernel", "/bias", "/bn_beta", "/theta")


def trainable_names(p):
    return [k for k in p if k.endswith(TRAINABLE_SUFFIX)]


@dataclass
class OracleNet:
    n_in: int
    n_out: int
    hidden: Sequence[int] = (64, 32, 64)
    ae_type: str = "zinb-conddisp"
    batchnorm: bool = True
    ridge: float = 0.0
    l1: float = 0.0
    l2: float = 0.0
    l1_enc: float = 0.0
    l2_enc: float = 0.0
    dtype: type = np.float64
    params: Dict[str, np.ndarray] = field(default_factory=dict)
    rms: Dict[str, np.ndarray] = field(default_factory=dict)
    bn_momentum: float = KERAS_DEFAULTS["bn_momentum"]
    bn_eps: float = KERAS_DEFAULTS["bn_eps"]
    # same-rounding emulation of the tcgen05 path: GEMM operands of the gene-wide layers are rounded
    # to bf16 (X, first kernel, last hidden activation, head kernels, dZ, dA of the first layer).
    # The engine picks the tensor-core encoder and heads independently, so either side can be emulated
    # alone: "encoder" (X, first kernel, dA of the first layer), "heads" (last hidden activation, head
    # kernels, dZ), "both" (= True) or "none" (= False).
    emulate_bf16: Union[bool, str] = False

    def __post_init__(self):
        assert self.ae_type in AE_TYPES
        side = {True: "both", False: "none"}.get(self.emulate_bf16, self.emulate_bf16)
        assert side in ("both", "none", "encoder", "heads"), self.emulate_bf16
        self._rnd_enc = bf16_round if side in ("both", "encoder") else (lambda t: t)
        self._rnd_heads = bf16_round if side in ("both", "heads") else (lambda t: t)
        self.names = layer_names(len(self.hidden))
        self.heads = head_names(self.ae_type)
        if not self.params:
            self.params = init_params(self.n_in, self.n_out, self.hidden, self.ae_type,
                                      self.batchnorm, dtype=self.dtype)
        self.params = {k: np.asarray(v, self.dtype).copy() for k, v in self.params.items()}

    # -- regulariser coefficients per layer: dca/network.py:113-122, 125
    def _reg(self, idx):
        center = int(np.floor(len(self.hidden) / 2.0))
        enc_stage = idx <= center
        l1 = self.l1_enc if (self.l1_enc != 0.0 and enc_stage) else self.l1
        l2 = self.l2_enc if (self.l2_enc != 0.0 and enc_stage) else self.l2
        return l1, l2

    # -- forward: dca/network.py:92-141 (hidden stack) + :366-393 (heads)
    def forward(self, X, sf, training: bool, cache: Optional[dict] = None):
        dt = self.dtype
        h = np.asarray(X, dt)
        c = {"h_in": [h]} if cache is not None else None
        latent = None
        rnd_e, rnd_h = self._rnd_enc, self._rnd_heads
        for i, nm in enumerate(self.names):
            if i == 0:
                a = rnd_e(h) @ rnd_e(self.params[nm + "/kernel"]) + self.params[nm + "/bias"]
            else:
                a = h @ self.params[nm + "/kernel"] + self.params[nm + "/bias"]
            if nm == "center":
                latent = a                                  # dca/network.py:184-185 (pre-BN)
            if self.batchnorm:
                if training:
                    mean = a.mean(axis=0)
                    var = a.var(axis=0)                    # biased
                else:
                    mean = self.params[nm + "/bn_moving_mean"]
                    var = self.params[nm + "/bn_moving_var"]
                inv = 1.0 / np.sqrt(var + self.bn_eps)
                xhat = (a - mean) * inv
                pre = xhat + self.params[nm + "/bn_beta"]   # center=True, scale=False
                if cache is not None:
                    c.setdefault("bn", []).append((xhat, inv, mean, var))
            else:
                pre = a
            h = np.maximum(pre, 0)                         # Activation('relu')
            if cache is not None:
                c.setdefault("pre", []).append(pre)
                c["h_in"].append(h)
        out = {"latent": latent, "decoded": h}
        z = {}
        for nm in self.heads:
            z[nm] = rnd_h(h) @ rnd_h(self.params[nm + "/kernel"]) + self.params[nm + "/bias"]
        out["z"] = z
        out["mean_norm"] = mean_act(z["mean"])
        sfc = np.asarray(sf, dt).reshape(-1, 1)
        out["mean"] = out["mean_norm"] * sfc               # ColwiseMultLayer, dca/layers.py:85
        if "dispersion" in z:
            out["dispersion"] = disp_act(z["dispersion"])
        elif "dispersion/theta" in self.params:
            out["dispersion"] = theta_const(self.params["dispersion/theta"]).astype(dt)
        if "pi" in z:
            out["pi"] = sigmoid(z["pi"])
        if cache is not None:
            cache.update(c)
        return out

    def penalty(self):
        """Keras kernel_regularizer l1_l2 terms -- dca/network.py:125,370,375,379."""
        tot = 0.0
        for i, nm in enumerate(self.names):
            l1, l2 = self._reg(i)
            W = self.params[nm + "/kernel"]
            tot += l1 * np.abs(W).sum() + l2 * np.square(W).sum()
        for nm in self.heads:
            W = self.params[nm + "/kernel"]
            tot += self.l1 * np.abs(W).sum() + self.l2 * np.square(W).sum()
        return float(tot)

    def loss(self, X, Y, sf, training=False):
        out = self.forward(X, sf, training)
        theta = out["dispersion"]
        if theta.ndim == 1:
            theta = np.broadcast_to(theta.reshape(1, -1), out["mean"].shape)
        if "pi" in out:
            data = zinb_loss(np.asarray(Y, self.dtype), out["mean"], theta, out["pi"], self.ridge)
        else:
            data = nb_loss(np.asarray(Y, self.dtype), out["mean"], theta)
        return data + self.penalty()

    # -- backward: TF autodiff restated in closed form (SURVEY.md A.4)
    def loss_and_grads(self, X, Y, sf, update_bn=True) -> Tuple[float, Dict[str, np.ndarray]]:
        dt = self.dtype
        cache: dict = {}
        out = self.forward(X, sf, True, cache)
        z = out["z"]
        hg = head_grads_from_preact(np.asarray(Y, dt), sf, z["mean"], z.get("dispersion"),
                                    z.get("pi"), self.params.get("dispersion/theta"),
                                    self.ridge)
        loss = hg["loss"] + self.penalty()
        g: Dict[str, np.ndarray] = {}
        rnd_e, rnd_h = self._rnd_enc, self._rnd_heads
        h_last = cache["h_in"][-1]
        dh = np.zeros_like(h_last)
        for nm, key in (("mean", "dzm"), ("dispersion", "dzd"), ("pi", "dzp")):
            if nm in z:
                dz = rnd_h(hg[key])
                W = self.params[nm + "/kernel"]
                g[nm + "/kernel"] = rnd_h(h_last).T @ dz + self.l1 * np.sign(W) + 2 * self.l2 * W
                g[nm + "/bias"] = dz.sum(axis=0)
                dh = dh + dz @ rnd_h(W).T
        if "dtheta_raw" in hg:
            g["dispersion/theta"] = hg["dtheta_raw"]
        for i in reversed(range(len(self.names))):
            nm = self.names[i]
            pre = cache["pre"][i]
            dpre = dh * (pre > 0)
            if self.batchnorm:
                xhat, inv, mean, var = cache["bn"][i]
                g[nm + "/bn_beta"] = dpre.sum(axis=0)
                da = inv * (dpre - dpre.mean(axis=0) - xhat * (dpre * xhat).mean(axis=0))
            else:
                da = dpre
            W = self.params[nm + "/kernel"]
            l1, l2 = self._reg(i)
            if i == 0:
                g[nm + "/kernel"] = rnd_e(cache["h_in"][i]).T @ rnd_e(da) + l1 * np.sign(W) + 2 * l2 * W
            else:
                g[nm + "/kernel"] = cache["h_in"][i].T @ da + l1 * np.sign(W) + 2 * l2 * W
            g[nm + "/bias"] = da.sum(axis=0)
            dh = da @ W.T
        if update_bn and self.batchnorm:
            mom = self.bn_momentum
            for i, nm in enumerate(self.names):
                _, _, mean, var = cache["bn"][i]
                self.params[nm + "/bn_moving_mean"] = mom * self.params[nm + "/bn_moving_mean"] + (1 - mom) * mean
                self.params[nm + "/bn_moving_var"] = mom * self.params[nm + "/bn_moving_var"] + (1 - mom) * var
        return loss, g

    # -- optimizer: keras RMSprop(clipvalue=5) -- dca/train.py:54-57 (SURVEY.md A.6)
    def rmsprop_step(self, grads, lr=KERAS_DEFAULTS["rms_lr"], clip=KERAS_DEFAULTS["clipvalue"],
                     rho=KERAS_DEFAULTS["rms_rho"], eps=KERAS_DEFAULTS["rms_eps"]):
        for k, gk in grads.items():
            gk = np.clip(gk, -clip, clip) if clip else gk
            r = self.rms.get(k)
            if r is None:
                r = np.zeros_like(self.params[k])
            r = rho * r + (1.0 - rho) * np.square(gk)
            self.rms[k] = r
            self.params[k] = self.params[k] - lr * gk / (np.sqrt(r) + eps)

    def train_step(self, X, Y, sf, lr=KERAS_DEFAULTS["rms_lr"], clip=KERAS_DEFAULTS["clipvalue"]):
        loss, g = self.loss_and_grads(X, Y, sf)
        self.rmsprop_step(g, lr, clip)
        return loss

    # -- predict: dca/network.py:188-211, 395-405 (inference-mode BN, all cells)
    def predict(self, X, sf):
        out = self.forward(X, sf, False)
        res = {"mean": out["mean"], "latent": out["latent"], "mean_norm": out["mean_norm"]}
        if "dispersion" in out:
            res["dispersion"] = out["dispersion"]
        if "pi" in out:
            res["pi"] = out["pi"]
        return res


# ----------------------------------------------------------------------------
# Keras Model.fit semantics as used at dca/train.py:91-98 (SURVEY.md A.7)
# ----------------------------------------------------------------------------
def fit(net: OracleNet, X, Y, sf, epochs=300, batch_size=32, validation_split=0.1,
        reduce_lr=10, early_stop=15, lr=None, clip=5.0, rng=None, batch_order=None):
    """Returns history dict {'loss','val_loss','lr'}.  ``batch_order`` (list of index
    arrays per epoch) overrides the shuffle so a CUDA run can be replayed exactly."""
    rng = np.random.default_rng(0) if rng is None else rng
    N = X.shape[0]
    split_at = int(N * (1.0 - validation_split)) if validation_split else N
    lr = KERAS_DEFAULTS["rms_lr"] if lr is None else lr
    hist = {"loss": [], "val_loss": [], "lr": []}
    best = np.inf; wait = 0; es_best = np.inf; es_wait = 0
    for ep in range(epochs):
        order = batch_order[ep] if batch_order is not None else rng.permutation(split_at)
        tot = 0.0; cnt = 0
        for s in range(0, split_at, batch_size):
            idx = order[s:s + batch_size]
            l = net.train_step(X[idx], Y[idx], sf[idx], lr=lr, clip=clip)
            tot += l * len(idx); cnt += len(idx)
        hist["loss"].append(tot / max(cnt, 1))
        hist["lr"].append(lr)
        if split_at < N:
            vt = 0.0; vc = 0
            for s in range(split_at, N, batch_size):
                e = min(s + batch_size, N)
                vt += net.loss(X[s:e], Y[s:e], sf[s:e], training=False) * (e - s); vc += e - s
            val = vt / vc
            hist["val_loss"].append(val)
            # ReduceLROnPlateau(monitor='val_loss', patience=reduce_lr, factor=0.1, min_delta=1e-4)
            if reduce_lr:
                if val < best - KERAS_DEFAULTS["plateau_min_delta"]:
                    best = val; wait = 0
                else:
                    wait += 1
                    if wait >= reduce_lr:
                        lr = lr * KERAS_DEFAULTS["plateau_factor"]; wait = 0
            # EarlyStopping(monitor='val_loss', patience=early_stop, min_delta=0)
            if early_stop:
                if val < es_best:
                    es_best = val; es_wait = 0
                else:
                    es_wait += 1
                    if es_wait >= early_stop:
                        break
    return hist
