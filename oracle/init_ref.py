"""NumPy restatement of the kernel initializers (Keras 2 / tf.keras 2.x `kernel_initializer`, dca/network.py:124-126)
and of the counter-based draws the library takes for them (include/dca_b200.h, "initializers").  Test infrastructure
only: written from the formulas, it shares no code with the library.

draw(name, seed, sid, shape) gives the float32 kernel the library's initializer of that name writes for the kernel with
stream id sid and Keras shape `shape` ((n,) for a 1-D kernel, (in, out) for a 2-D one)."""
import numpy as np

# name -> (kind, arguments), the table of Keras defaults (snake_case names; CAMEL holds the class names)
VS = "variance_scaling"
SPECS = {
    "glorot_uniform": (VS, dict(scale=1.0, mode="fan_avg", distribution="uniform")),
    "glorot_normal": (VS, dict(scale=1.0, mode="fan_avg", distribution="truncated_normal")),
    "he_uniform": (VS, dict(scale=2.0, mode="fan_in", distribution="uniform")),
    "he_normal": (VS, dict(scale=2.0, mode="fan_in", distribution="truncated_normal")),
    "lecun_uniform": (VS, dict(scale=1.0, mode="fan_in", distribution="uniform")),
    "lecun_normal": (VS, dict(scale=1.0, mode="fan_in", distribution="truncated_normal")),
    "variance_scaling": (VS, dict(scale=1.0, mode="fan_in", distribution="truncated_normal")),
    "random_normal": ("random_normal", dict(stddev=0.05)),
    "random_uniform": ("random_uniform", dict(minval=-0.05, maxval=0.05)),
    "truncated_normal": ("truncated_normal", dict(stddev=0.05)),
    "zeros": ("constant", dict(value=0.0)),
    "ones": ("constant", dict(value=1.0)),
    "constant": ("constant", dict(value=0.0)),
    "orthogonal": ("orthogonal", dict(gain=1.0)),
    "identity": ("identity", dict(gain=1.0)),
}
ALIASES = {"normal": "random_normal", "uniform": "random_uniform", "zero": "zeros", "one": "ones"}
CAMEL = {"GlorotUniform": "glorot_uniform", "GlorotNormal": "glorot_normal", "HeUniform": "he_uniform",
         "HeNormal": "he_normal", "LecunUniform": "lecun_uniform", "LecunNormal": "lecun_normal",
         "VarianceScaling": "variance_scaling", "RandomNormal": "random_normal", "RandomUniform": "random_uniform",
         "TruncatedNormal": "truncated_normal", "Zeros": "zeros", "Ones": "ones", "Constant": "constant",
         "Orthogonal": "orthogonal", "Identity": "identity"}
TRUNC_SD = 0.87962566103423978        # standard deviation of a standard normal truncated to [-2, 2]
TRUNC_ATTEMPTS = 16


def canonical(name):
    return CAMEL.get(name, ALIASES.get(name, name))


def fans(shape):
    """Keras _compute_fans for the kernels of this model: (n,) -> (n, n); (in, out) -> (in, out)."""
    if len(shape) == 1:
        return int(shape[0]), int(shape[0])
    return int(shape[0]), int(shape[1])


def target(name, shape):
    """The distribution of one element: ("uniform", lo, hi), ("normal", sigma), ("truncated", sigma) -- a normal of
    that sigma restricted to [-2 sigma, 2 sigma] --, ("constant", v), ("identity", gain) or ("orthogonal", gain)."""
    kind, a = SPECS[canonical(name)]
    if kind == VS:
        fi, fo = fans(shape)
        n = {"fan_in": fi, "fan_out": fo, "fan_avg": (fi + fo) / 2.0}[a["mode"]]
        s = a["scale"] / max(1.0, n)
        if a["distribution"] == "uniform":
            lim = np.sqrt(3.0 * s)
            return ("uniform", -lim, lim)
        if a["distribution"] == "truncated_normal":
            return ("truncated", np.sqrt(s) / TRUNC_SD)
        return ("normal", np.sqrt(s))
    if kind == "random_normal":
        return ("normal", a["stddev"])
    if kind == "truncated_normal":
        return ("truncated", a["stddev"])
    if kind == "random_uniform":
        return ("uniform", a["minval"], a["maxval"])
    if kind == "constant":
        return ("constant", a["value"])
    if len(shape) != 2:
        raise ValueError("%s needs a 2-D kernel, got shape %s" % (kind, tuple(shape)))
    return (kind, a["gain"])


FLAGSHIP = ("zinb-conddisp", "zinb", "nb-conddisp", "nb")
HEAD_SID = {"mean": 100, "dispersion": 101, "pi": 102}


def kernels(ae_type, n_in, n_out, hidden=(64, 32, 64), sharedpi=False):
    """[(name, Keras shape, stream id)] of every kernel of a model: the flagship types number their hidden layers 0, 1,
    ... and their heads 100 (mean), 101 (dispersion), 102 (pi); the other types number their kernels in creation
    order."""
    from oracle import dca_oracle, torch_ref
    if ae_type in FLAGSHIP:
        p = dca_oracle.init_params(n_in, n_out, hidden, ae_type, batchnorm=False)
    else:
        p = torch_ref.extra_init_params(n_in, n_out, hidden, ae_type, batchnorm=False, sharedpi=sharedpi)
    out = []
    for i, nm in enumerate(k for k in p if k.endswith("/kernel")):
        layer = nm[:-len("/kernel")]
        sid = (HEAD_SID[layer] if layer in HEAD_SID else i) if ae_type in FLAGSHIP else i
        out.append((nm, tuple(p[nm].shape), sid))
    return out


# ---- the counter-based draws
_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(x):
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def element_hash(seed, sid, n):
    with np.errstate(over="ignore"):
        key = splitmix64(np.uint64(seed) ^ (np.uint64(sid) * np.uint64(0xD1B54A32D192ED03)))
        return splitmix64(key + np.arange(n, dtype=np.uint64))


def std_normal(h, attempt):
    """Box-Muller in float64 of draw `attempt` of the elements with hashes h."""
    with np.errstate(over="ignore"):
        h1 = splitmix64(h ^ (np.uint64(0x632BE59BD9B4E019) * np.uint64(2 * attempt + 1)))
        h2 = splitmix64(h ^ (np.uint64(0x632BE59BD9B4E019) * np.uint64(2 * attempt + 2)))
    u1 = ((h1 >> np.uint64(11)) + np.uint64(1)).astype(np.float64) * 2.0 ** -53
    u2 = (h2 >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def truncated_std_normal(h):
    z = np.zeros(h.shape, np.float64)
    todo = np.ones(h.shape, bool)
    for a in range(TRUNC_ATTEMPTS):
        t = std_normal(h, a)
        ok = todo & (np.abs(t) < 2.0)
        z[ok] = t[ok]
        todo &= ~ok
        if not todo.any():
            break
    return z


def normal_matrix(seed, sid, shape):
    """The standard normals (rounded to float32) whose QR gives an orthogonal kernel of this shape:
    (max(rows, cols), min(rows, cols))."""
    r, c = shape
    m, n = max(r, c), min(r, c)
    return std_normal(element_hash(seed, sid, m * n), 0).astype(np.float32).reshape(m, n)


def orthogonal_from(A, shape, gain=1.0):
    """Keras Orthogonal on the normal matrix A: Q R = qr(A) (reduced), Q * sign(diag R), transposed when rows < cols;
    float64."""
    q, r = np.linalg.qr(A.astype(np.float64))
    q = q * np.sign(np.diag(r))
    if shape[0] < shape[1]:
        q = q.T
    return gain * q


def draw(name, seed, sid, shape):
    """The kernel as the library draws it, restated: float32, Keras shape.  Uniform draws are the library's float
    arithmetic (bit for bit); normal ones are float64 Box-Muller rounded once (the library's values within 1 ulp)."""
    t = target(name, shape)
    size = int(np.prod(shape))
    if t[0] == "constant":
        return np.full(shape, t[1], np.float32)
    if t[0] == "identity":
        return (t[1] * np.eye(*shape)).astype(np.float32)
    if t[0] == "orthogonal":
        return orthogonal_from(normal_matrix(seed, sid, shape), shape, t[1]).astype(np.float32)
    h = element_hash(seed, sid, size)
    if t[0] == "uniform":
        lo, hi = t[1], t[2]
        if canonical(name) in SPECS and SPECS[canonical(name)][0] == VS:
            # the limit in float32, as the library computes it: sqrt(3 scale / n)
            a = SPECS[canonical(name)][1]
            fi, fo = fans(shape)
            n = {"fan_in": np.float32(fi), "fan_out": np.float32(fo),
                 "fan_avg": np.float32(0.5) * np.float32(fi + fo)}[a["mode"]]
            half = np.sqrt(np.float32(3.0) * np.float32(a["scale"]) / max(np.float32(1.0), n), dtype=np.float32)
            center = np.float32(0.0)
        else:
            center = np.float32(0.5) * (np.float32(lo) + np.float32(hi))
            half = np.float32(0.5) * (np.float32(hi) - np.float32(lo))
        u = (h >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
        x = np.float32(2.0) * u - np.float32(1.0)
        # fmaf(x, half, center): x * half is exact in float64 (24 x 24 bits), so one rounding to float32 restates it
        # whenever center + x * half is exact in float64 too (center 0 for every Keras default)
        w = (x.astype(np.float64) * np.float64(half) + np.float64(center)).astype(np.float32)
        return w.reshape(shape)
    z = std_normal(h, 0) if t[0] == "normal" else truncated_std_normal(h)
    return (z * np.float64(t[1])).astype(np.float32).reshape(shape)
