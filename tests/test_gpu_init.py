"""Kernel initializers on the GPU (dca_init_params_ex; --init, dca/network.py:124-126): every Keras name, all eleven AE
types, at 2 000 and 20 000 genes, against the host restatement of the draws (dca_init_fill_host) and NumPy's QR, plus
the target distributions, the untouched non-kernel tensors, the bf16 copy the tensor-core path reads, and training end
to end.  Needs a GPU."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
from scipy import stats

from dca_b200 import _lib
from oracle import init_ref as R
from tests.util import synth_counts

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HIDDEN = (64, 32, 64)
NAMES = sorted(R.SPECS)
SEED = 7


def _engine(ae_type, G, init, seed=SEED, **kw):
    from dca_b200.engine import DeviceEngine
    return DeviceEngine(G, G, HIDDEN, ae_type, True, max_batch=64, init=init, seed=seed, **kw)


def _host(name, seed, sid, shape):
    ndim, rows, cols = (1, 1, shape[0]) if len(shape) == 1 else (2, shape[0], shape[1])
    out = np.empty(rows * cols, np.float32)
    assert _lib.load().dca_init_fill_host(C.byref(_lib.initializer(name)), C.c_uint64(seed), C.c_uint64(sid), ndim,
                                          rows, cols, out.ctypes.data_as(C.c_void_p)) == 0
    return out


def _ulps(a, b):
    a = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    b = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return np.abs(np.where(a < 0, -(a & 0x7FFFFFFF), a) - np.where(b < 0, -(b & 0x7FFFFFFF), b))


def _ks_p(w, t):
    x = w.astype(np.float64).ravel()
    if t[0] == "uniform":
        return stats.kstest(x, stats.uniform(loc=t[1], scale=t[2] - t[1]).cdf).pvalue
    if t[0] == "normal":
        return stats.kstest(x, stats.norm(scale=t[1]).cdf).pvalue
    return stats.kstest(x, stats.truncnorm(-2.0, 2.0, scale=t[1]).cdf).pvalue


def _check_kernel(ae_type, G, init, name, shape, sid, dev):
    t = R.target(init, shape)
    what = "%s %d %s %s" % (ae_type, G, init, name)
    if t[0] == "orthogonal":
        A = _host(init, SEED, sid, shape).reshape(max(shape), min(shape))
        ref = R.orthogonal_from(A, shape, t[1])
        err = np.abs(dev.reshape(shape).astype(np.float64) - ref).max()
        assert err <= 1e-6, (what, err)
        W = dev.reshape(shape).astype(np.float64)
        g = W.T @ W if shape[0] >= shape[1] else W @ W.T
        assert np.abs(g - np.eye(g.shape[0])).max() <= 1e-5, what
        return
    host = _host(init, SEED, sid, shape)
    if t[0] in ("uniform", "constant", "identity"):
        np.testing.assert_array_equal(dev.ravel(), host, err_msg=what)
    else:
        assert _ulps(dev.ravel(), host).max() <= 1, what
    if t[0] == "truncated":
        assert np.abs(dev.astype(np.float64)).max() < 2 * t[1] * (1 + 2.0 ** -23), what
    if G == 20000 and shape == (64, G) and t[0] in ("uniform", "normal", "truncated"):
        p = _ks_p(dev, t)
        assert p > 1e-3, (what, p)


@pytest.mark.parametrize("G", [2000, 20000])
@pytest.mark.parametrize("ae_type", list(_lib.AE_TYPE_IDS))
def test_every_initializer_matches_the_host_draws(ae_type, G):
    table = R.kernels(ae_type, G, G, HIDDEN)
    for init in NAMES:
        if ae_type == "zinb-elempi" and init in ("orthogonal", "identity"):
            with pytest.raises(ValueError, match="2-D"):
                _engine(ae_type, G, init)
            continue
        eng = _engine(ae_type, G, init)
        w = eng.get_weights()
        for name, shape, sid in table:
            _check_kernel(ae_type, G, init, name, shape, sid, w[name])
        # biases, BatchNorm beta and moving statistics, theta: as dca_init_params leaves them
        for name, a in w.items():
            if name.endswith("/kernel"):
                continue
            expect = 1.0 if name.endswith("moving_var") else 0.0
            assert np.all(a == expect), (ae_type, init, name)
        # the bf16 copy of the tensor-core path holds the new values: a predict right after init equals one after
        # set_weights of the same values on a fresh engine
        if ae_type in R.FLAGSHIP:
            other = _engine(ae_type, G, "zeros", seed=None)
            other.set_weights(w)
            np.testing.assert_array_equal(_predict(eng), _predict(other), err_msg="%s %s" % (ae_type, init))
            other.close()
        eng.close()


def _predict(eng):
    import torch
    dev = eng.device
    g = torch.Generator(device="cpu").manual_seed(1)
    X = torch.randn(48, eng.n_in, generator=g).to(dev)
    sf = torch.ones(48, device=dev)
    mean = torch.empty(48, eng.n_out, device=dev)
    eng.predict(X, sf, mean=mean)
    torch.cuda.synchronize(dev)
    return mean.cpu().numpy()


@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "nb", "zinb-elempi", "zinb-fork"])
def test_seed_keys_the_draws(ae_type):
    for init in ("he_normal", "glorot_uniform", "orthogonal", "random_uniform", "truncated_normal"):
        if ae_type == "zinb-elempi" and init == "orthogonal":
            continue
        a = _engine(ae_type, 2000, init, seed=3)
        b = _engine(ae_type, 2000, init, seed=3)
        c = _engine(ae_type, 2000, init, seed=4)
        pa, pb, pc = (e.params.cpu().numpy() for e in (a, b, c))
        assert pa.tobytes() == pb.tobytes(), (ae_type, init)
        assert pa.tobytes() != pc.tobytes(), (ae_type, init)
        for e in (a, b, c):
            e.close()


@pytest.mark.parametrize("G", [2000, 20000])
def test_glorot_uniform_through_init_params_ex_is_dca_init_params(G):
    import torch
    for ae_type in _lib.AE_TYPE_IDS:
        eng = _engine(ae_type, G, "glorot_uniform", seed=11)      # dca_init_params_ex
        ex = eng.params.cpu().numpy().copy()
        ex_bf = eng.get_weights()
        _lib.check(eng.lib.dca_init_params(eng.handle, C.c_uint64(11), eng._stream()), "dca_init_params")
        torch.cuda.synchronize(eng.device)
        assert eng.params.cpu().numpy().tobytes() == ex.tobytes(), ae_type
        assert all(np.array_equal(v, eng.get_weights()[k]) for k, v in ex_bf.items())
        eng.close()


def test_an_invalid_spec_changes_nothing():
    import torch
    eng = _engine("zinb-elempi", 2000, "he_uniform")
    before = eng.params.cpu().numpy().copy()
    with pytest.raises(ValueError, match="2-D"):
        _lib.check(eng.lib.dca_init_params_ex(eng.handle, C.c_uint64(1), C.byref(_lib.initializer("orthogonal")),
                                              eng._stream()), "dca_init_params_ex")
    torch.cuda.synchronize(eng.device)
    assert eng.params.cpu().numpy().tobytes() == before.tobytes()
    eng.close()


@pytest.mark.parametrize("init", NAMES)
def test_dca_trains_with_every_initializer(init):
    from dca_b200.anndata_lite import AnnData
    from dca_b200.api import dca
    adata = AnnData(synth_counts(300, 120, 2))
    ret = dca(adata, init=init, epochs=2, copy=True, return_info=True, batch_size=64)
    loss = ret.uns['dca_loss_history']['loss']
    assert 1 <= len(loss) <= 2 and np.all(np.isfinite(loss)), (init, loss)
    assert np.all(np.isfinite(ret.X))


def test_cli_init_he_normal(tmp_path):
    Y = synth_counts(120, 60, 4).astype(int)
    df = pd.DataFrame(Y.T, index=["g%d" % i for i in range(60)], columns=["c%d" % i for i in range(120)])
    inp = tmp_path / "counts.tsv"; df.to_csv(inp, sep="\t")
    out = tmp_path / "out"
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", "dca_b200", str(inp), str(out), "--init", "he_normal", "-e", "2"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    for f in ("mean.tsv", "latent.tsv", "dispersion.tsv"):          # the default type, nb-conddisp, has no dropout
        assert (out / f).exists(), f
    mean = pd.read_csv(out / "mean.tsv", sep="\t", index_col=0)
    assert mean.shape == (60, 120) and np.all(np.isfinite(mean.values))


@pytest.mark.parametrize("ae_type", ["poisson", "zinb-elempi", "nb-fork"])
def test_one_row_kernels_of_the_other_types(ae_type):
    """A hidden width of 1 gives the extra types a 2-D kernel with one row ("dec0" here): its draws take fan_in = its
    length, the rule glorot_uniform has always used for these types, and orthogonal / identity treat it as 2-D."""
    from dca_b200.engine import DeviceEngine
    hidden = (16, 1, 16)
    for init in ("glorot_uniform", "he_normal", "orthogonal", "identity"):
        if ae_type == "zinb-elempi" and init in ("orthogonal", "identity"):
            continue
        eng = DeviceEngine(40, 40, hidden, ae_type, True, max_batch=8, init=init, seed=5)
        w = eng.get_weights()
        table = R.kernels(ae_type, 40, 40, hidden)
        for name, shape, sid in table:
            dev = w[name].ravel()
            if init in ("orthogonal", "identity"):
                if init == "identity":
                    np.testing.assert_array_equal(dev, np.eye(*shape, dtype=np.float32).ravel())
                else:
                    W = dev.reshape(shape).astype(np.float64)
                    g = W.T @ W if shape[0] >= shape[1] else W @ W.T
                    assert np.abs(g - np.eye(g.shape[0])).max() <= 1e-5, name
                continue
            host_shape = (shape[-1],) if shape[0] == 1 or len(shape) == 1 else shape
            host = _host(init, 5, sid, host_shape)
            assert _ulps(dev, host).max() <= (0 if init == "glorot_uniform" else 1), (ae_type, init, name)
        assert any(s[0] == 1 and len(s) == 2 for _, s, _ in table)
        eng.close()
