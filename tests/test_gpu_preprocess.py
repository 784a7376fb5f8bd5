"""On-device preprocessing (csrc/preprocess.cu, dca_b200/device_data.py) against the host path io.normalize and the
NumPy statement of the device arithmetic (device_data.normalize_reference), and training / prediction / dca() / CLI
on the resident dataset against the host arm holding the same values.  Needs a GPU."""
import ctypes as C
import itertools

import numpy as np
import pandas as pd
import pytest
import torch

from tests.util import synth_counts

pytestmark = pytest.mark.gpu


def _adata(Y):
    from dca_b200.anndata_lite import AnnData
    return AnnData(np.array(Y, dtype=np.float32))


def _within_ulp(a, b, n=1):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.all(np.abs(a.astype(np.float64) - b) <= n * np.spacing(np.maximum(np.abs(a), np.abs(b))))


def _dd(Y, **kw):
    from dca_b200.device_data import DeviceDataset
    return DeviceDataset.from_counts(Y, torch.device("cuda:0"), **kw)


def _host(t):
    return t.cpu().numpy()


def _parity_cases():
    yield "4096x2000", synth_counts(4096, 2000, 0)
    Y = synth_counts(1024, 20000, 1)
    Y[3, 7] = 1e6
    yield "1024x20000", Y


@pytest.mark.parametrize("case", ["4096x2000", "1024x20000"])
def test_parity_with_host_normalize(case):
    from dca_b200 import io
    from dca_b200.device_data import normalize_reference
    Y = dict(_parity_cases())[case]
    host = io.normalize(_adata(Y), filter_min_counts=False)
    dd = _dd(Y)
    ref = normalize_reference(Y)
    assert np.array_equal(_host(dd.n_counts), np.asarray(host.obs['n_counts']))
    assert np.array_equal(_host(dd.sf), np.asarray(host.obs['size_factors']))
    np.testing.assert_allclose(_host(dd.mean), ref["mean"], rtol=1e-9, atol=1e-300)
    np.testing.assert_allclose(_host(dd.std), ref["std"], rtol=1e-9)
    X = _host(dd.X)
    assert _within_ulp(X, ref["X"])
    Xh = np.asarray(host.X)
    assert np.all(np.abs(X - Xh) <= 4e-6 * np.maximum(1.0, np.abs(Xh)))
    assert np.array_equal(dd.gene_totals_host, Y.sum(0, dtype=np.float64)) and dd.n_bad == 0


@pytest.mark.parametrize("flags", list(itertools.product([False, True], repeat=3)))
def test_all_flag_combinations(flags):
    from dca_b200 import io
    from dca_b200.device_data import normalize_reference
    sfac, logt, norm = flags
    Y = synth_counts(300, 130, 5)
    dd = _dd(Y, size_factors=sfac, logtrans_input=logt, normalize_input=norm)
    ref = normalize_reference(Y, sfac, logt, norm)
    host = io.normalize(_adata(Y), filter_min_counts=False, size_factors=sfac, logtrans_input=logt, normalize_input=norm)
    assert np.array_equal(_host(dd.sf), np.broadcast_to(np.asarray(host.obs['size_factors'], np.float32), (300,)))
    if sfac:
        assert np.array_equal(_host(dd.n_counts), np.asarray(host.obs['n_counts']))
    np.testing.assert_allclose(_host(dd.mean), ref["mean"], rtol=1e-9, atol=1e-300)
    np.testing.assert_allclose(_host(dd.std), ref["std"], rtol=1e-9)
    X = _host(dd.X)
    assert _within_ulp(X, ref["X"])
    Xh = np.asarray(host.X)
    assert np.all(np.abs(X - Xh) <= 4e-6 * np.maximum(1.0, np.abs(Xh)))
    if not (sfac or logt or norm):
        assert np.array_equal(X, Y)


def test_filter_min_counts_matches_host():
    from dca_b200 import io
    Y = synth_counts(500, 90, 6)
    Y[:, [3, 40, 89]] = 0          # all-zero genes
    Y[[0, 17, 499], :] = 0         # all-zero cells
    Y[250, :] = 0
    Y[250, 3] = 0
    a_h, a_d = _adata(Y), _adata(Y)
    io.normalize(a_h)
    io.normalize(a_d, device=torch.device("cuda:0"))
    dd = a_d.uns['dca_device_data']
    assert list(a_h.var_names) == list(a_d.var_names) and list(a_h.obs_names) == list(a_d.obs_names)
    assert a_h.X.shape == a_d.X.shape == (496, 87)
    assert np.array_equal(a_h.raw.X, a_d.raw.X) and list(a_h.raw.var_names) == list(a_d.raw.var_names)
    assert np.array_equal(np.asarray(a_h.obs['n_counts']), np.asarray(a_d.obs['n_counts']))
    assert np.array_equal(np.asarray(a_h.obs['size_factors']), np.asarray(a_d.obs['size_factors']))
    assert np.all(np.abs(a_d.X - a_h.X) <= 4e-6 * np.maximum(1.0, np.abs(a_h.X)))
    assert np.array_equal(a_d.X, dd.host_x()) and np.array_equal(_host(dd.Y), a_h.raw.X)


def _raw_pipeline(Y, ldy, ldx, x_dtype, flags=7):
    """The five entry points called directly, Y / X with leading dimensions ldy / ldx and NaN guard bands."""
    from dca_b200 import _lib
    lib = _lib.load()
    N, G = Y.shape
    dev = torch.device("cuda:0")
    Yp = torch.full((N, ldy), float("nan"), dtype=torch.float32, device=dev)
    Yp[:, :G] = torch.from_numpy(Y).to(dev)
    xdt = torch.bfloat16 if x_dtype == _lib.BF16 else torch.float32
    Xp = torch.full((N + 1, ldx), float("nan"), dtype=xdt, device=dev)
    ws_b = C.c_size_t()
    assert lib.dca_preprocess_workspace_bytes(N, G, C.byref(ws_b)) == 0
    ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
    nc = torch.empty(N, dtype=torch.float64, device=dev)
    gt = torch.empty(G, dtype=torch.float64, device=dev)
    bad = torch.zeros(1, dtype=torch.int64, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.dca_count_totals(Yp.data_ptr(), ldy, N, G, nc.data_ptr(), gt.data_ptr(), bad.data_ptr(), ws.data_ptr(),
                                    ws.numel(), s))
    med = float(np.median(_host(nc)))
    mean = torch.empty(G, dtype=torch.float64, device=dev)
    std = torch.empty(G, dtype=torch.float64, device=dev)
    _lib.check(lib.dca_log_moments(Yp.data_ptr(), ldy, N, G, nc.data_ptr(), med, flags, mean.data_ptr(), std.data_ptr(),
                                   ws.data_ptr(), ws.numel(), s))
    _lib.check(lib.dca_normalize_write(Yp.data_ptr(), ldy, N, G, nc.data_ptr(), med, flags, mean.data_ptr(), std.data_ptr(),
                                       Xp.data_ptr(), x_dtype, ldx, s))
    torch.cuda.synchronize()
    return _host(nc), _host(gt), int(bad.item()), _host(mean), _host(std), Xp


@pytest.mark.parametrize("G", [1, 37, 2000])
@pytest.mark.parametrize("N", [1, 203])
def test_shapes_and_guard_band(N, G):
    from dca_b200 import _lib
    from dca_b200.device_data import normalize_reference
    Y = synth_counts(N, G, 7 + G)
    if G > 1 and N > 1:
        Y[:, G // 2] = 0           # an all-zero (constant) gene
        Y[Y.sum(1) == 0, 0] = 1
    ref = normalize_reference(Y)
    first = {}
    # G + 8: the 128-bit path where G allows it; G + 1: the scalar path (unaligned rows) for every G
    for ldy, ldx in ((G, G), (G + 8, G + 8), (G + 1, G + 1), (G, G + 1)):
        for xd in (_lib.F32, _lib.BF16):
            nc, gt, bad, mean, std, Xp = _raw_pipeline(Y, ldy, ldx, xd)
            assert np.array_equal(nc, ref["n_counts"]) and bad == 0
            np.testing.assert_allclose(mean, ref["mean"], rtol=1e-9, atol=1e-300)
            np.testing.assert_allclose(std, ref["std"], rtol=1e-9)
            Xf = Xp.float()
            assert torch.isnan(Xf[:N, G:]).all() and torch.isnan(Xf[N:]).all(), "write outside [N x G]"
            X = _host(Xf[:N, :G])
            if xd == _lib.F32:
                assert _within_ulp(X, ref["X"])
                X32 = Xp[:N, :G].contiguous()
            else:
                assert torch.equal(Xp[:N, :G], X32.to(torch.bfloat16))     # bf16 = fp32 X rounded once
            first.setdefault(xd, Xp[:N, :G].contiguous())
            assert torch.equal(Xp[:N, :G], first[xd]), (ldy, ldx)            # every write path gives the same bits
    if N == 1:
        assert np.all(std == 1.0)


def test_two_pass_variance():
    """A gene of counts 1e6 + 0..4 over 3001 cells: a one-pass variance (sum l^2 - N mean^2, even with the product
    fused) is off by about 6e-6 of the std without log1p and by more than half of it with log1p.  (With a power-of-two
    number of cells and integer l, the fused one-pass form happens to be exact, so N is odd here.)"""
    from dca_b200.device_data import normalize_reference
    Y = synth_counts(3001, 64, 20)
    Y[:, 10] = 1e6 + np.random.default_rng(0).integers(0, 5, 3001)
    for flags in ((False, False, True), (False, True, True)):
        dd = _dd(Y, size_factors=flags[0], logtrans_input=flags[1], normalize_input=flags[2])
        ref = normalize_reference(Y, *flags)
        np.testing.assert_allclose(_host(dd.std), ref["std"], rtol=1e-9)
        assert _within_ulp(_host(dd.X), ref["X"])


def _emulate_moments(l):
    """Gene mean / std summed in the order of preprocess.cu: a CTA per (256-gene block, slice of rows) whose 8 warps
    take every 8th row of the slice; warps added in order; slots (slices) added in slot order."""
    N, G = l.shape
    gblocks = -(-G // 256)
    s = min(-(-1056 // gblocks), max(1, -(-N // 64)))
    rps = -(-N // s)
    slices = -(-N // rps)

    def colsum(v):
        tot = np.zeros(G)
        for sl in range(slices):
            r0, r1 = sl * rps, min(N, (sl + 1) * rps)
            cta = np.zeros(G)
            for w in range(8):
                acc = np.zeros(G)
                for r in range(r0 + w, r1, 8):
                    acc = acc + v[r]
                cta = cta + acc
            tot = tot + cta
        return tot
    L = l.astype(np.float64)
    mean = colsum(L) / N
    d = L - mean
    std = np.sqrt(colsum(d * d) / (N - 1)) if N > 1 else np.ones(G)
    std[std == 0] = 1.0
    return mean, std


@pytest.mark.parametrize("shape", [(4096, 2000), (1000, 300)])
def test_fold_order_is_slot_order(shape):
    """mean and std bit-exact against a NumPy emulation of the kernels' summation order (from the device's l)."""
    Y = synth_counts(*shape, 21)
    l = _host(_dd(Y, normalize_input=False).X)
    mean, std = _emulate_moments(l)
    dd = _dd(Y)
    assert np.array_equal(_host(dd.mean), mean)
    assert np.array_equal(_host(dd.std), std)


def test_bad_entries_are_counted_not_rejected():
    Y = synth_counts(64, 40, 8)
    Y[1, 2], Y[3, 4], Y[5, 6] = -1.0, 0.5, np.inf
    dd = _dd(Y, size_factors=False, logtrans_input=False, normalize_input=False)
    assert dd.n_bad == 3


def test_csr_input_same_bits_and_two_calls_identical():
    import scipy.sparse as sp
    Y = synth_counts(777, 1031, 9)
    Y[2, 5] = 123456.0
    d1, d2 = _dd(Y), _dd(Y)
    dc = _dd(sp.csr_matrix(Y))
    for name in ("Y", "n_counts", "mean", "std", "X", "sf"):
        assert torch.equal(getattr(d1, name), getattr(d2, name)), name
        assert torch.equal(getattr(d1, name), getattr(dc, name)), name
    # an unsorted CSR with duplicate entries (each count split in two halves, listed in reverse gene order) is
    # canonicalised on a copy; the caller's matrix is left as it is
    m = sp.csr_matrix(Y)
    indptr, indices, data = [0], [], []
    for r in range(Y.shape[0]):
        ix, v = m.indices[m.indptr[r]:m.indptr[r + 1]][::-1], m.data[m.indptr[r]:m.indptr[r + 1]][::-1] / 2
        indices += [ix, ix]; data += [v, v]; indptr.append(indptr[-1] + 2 * ix.size)
    dup = sp.csr_matrix((np.concatenate(data), np.concatenate(indices), np.asarray(indptr)), shape=Y.shape)
    assert not dup.has_canonical_format
    assert torch.equal(_dd(dup).X, d1.X) and not dup.has_canonical_format


def _bf16_rne(x):
    """float64 -> the nearest bfloat16 (ties to even), as float64"""
    m, e = np.frexp(np.asarray(x, np.float64))
    return np.ldexp(np.round(m * 256.0) / 256.0, e)


def test_bf16_x_is_fp32_x_rounded():
    Y = synth_counts(4096, 2000, 10)
    d32, d16 = _dd(Y), _dd(Y, x_dtype="bfloat16")
    assert d16.X.dtype == torch.bfloat16
    assert torch.equal(d16.X, d32.X.to(torch.bfloat16))
    # entries whose fp32 value is a bf16 tie while the double value is not: rounding the double straight to bf16 gives
    # a different result there.  The data must contain some, or the check above would not tell the two apart.
    l = _host(_dd(Y, normalize_input=False).X).astype(np.float64)
    x64 = (l - _host(d32.mean)) / _host(d32.std)                     # the device's double value, same IEEE operations
    assert np.array_equal(x64.astype(np.float32), _host(d32.X))
    direct = _bf16_rne(x64)
    split = direct != _bf16_rne(x64.astype(np.float32))
    assert split.sum() >= 10, int(split.sum())
    assert np.all(_host(d16.X.float())[split] != direct[split])
    Y2 = synth_counts(100, 37, 11)                                 # G % 8 != 0: the scalar write path
    assert torch.equal(_dd(Y2, x_dtype="bfloat16").X, _dd(Y2).X.to(torch.bfloat16))


# ------------------------------------------------------------------------------------------ training / prediction
def _host_arm(dd, Y):
    """An AnnData holding the device X / size factors on the host, raw = the counts."""
    from dca_b200.anndata_lite import AnnData
    a = AnnData(dd.host_x())
    a.obs['size_factors'] = dd.host_size_factors()
    a.raw = AnnData(np.ascontiguousarray(Y, dtype=np.float32))
    return a


def _net(ae_type, G, seed=0):
    from dca_b200.network import AE_types
    net = AE_types[ae_type](input_size=G, output_size=G, hidden_size=(64, 32, 64))
    net.build(max_batch=256, seed=seed)
    return net


def _fit(net, adata, **kw):
    from dca_b200.train import train
    np.random.seed(3)
    return train(adata, net, epochs=2, batch_size=256, validation_split=0.1, verbose=False, **kw).history


def _state(net):
    w = net.engine.get_weights()
    return {k: v for k, v in w.items()}


@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "nb"])
def test_train_and_predict_match_host_arm(ae_type):
    """zinb-conddisp: loss history, weights and BatchNorm state bit-identical.  'nb' sums its per-gene dispersion
    gradient with atomics (zinb_loss.cu), so two host-arm runs already differ in the last bits: there the device arm
    is held to 1e-5 of the host arm.  Prediction from the same weights is bit-identical for both."""
    G = 2000
    Y = synth_counts(1500, G, 12)
    dd = _dd(Y)
    host = _host_arm(dd, Y)
    n_h, n_d = _net(ae_type, G), _net(ae_type, G)
    if ae_type == "zinb-conddisp":
        assert n_d.engine.info()["tc_heads"]
    h_h = _fit(n_h, host)
    h_d = _fit(n_d, host, device_data=dd)
    w_h, w_d = _state(n_h), _state(n_d)
    assert w_h.keys() == w_d.keys()
    if ae_type == "zinb-conddisp":
        assert h_h == h_d
        assert all(np.array_equal(w_h[k], w_d[k]) for k in w_h)
    else:
        # the atomics' summation order differs from run to run and training amplifies it (two host-arm runs differ by
        # 1e-10 to 1e-7 relative after two epochs)
        for k in ("loss", "val_loss"):
            np.testing.assert_allclose(h_d[k], h_h[k], rtol=1e-5)
        for k in w_h:
            assert np.max(np.abs(w_h[k] - w_d[k]), initial=0.0) <= 1e-4 * max(np.max(np.abs(w_h[k]), initial=0.0), 1.0), k
    r_h = n_d._run_predict(host, True, True, True, True)
    r_d = n_d._run_predict(host, True, True, True, True, device_data=dd)
    for k in ("mean", "dispersion", "pi", "latent"):
        if r_h.get(k) is None:
            assert r_d.get(k) is None
        else:
            assert np.array_equal(r_h[k], r_d[k]), k


def test_train_on_take_subset_bit_identical():
    G = 2000
    Y = synth_counts(1200, G, 13)
    dd = _dd(Y)
    mask = np.random.default_rng(0).random(1200) < 0.6
    sub = dd.take(mask)
    assert sub.n == int(mask.sum()) and sub.X.data_ptr() == dd.X.data_ptr()
    host = _host_arm(dd, Y)[mask]
    n_h, n_d = _net("zinb-conddisp", G), _net("zinb-conddisp", G)
    assert _fit(n_h, host) == _fit(n_d, host, device_data=sub)
    w_h, w_d = _state(n_h), _state(n_d)
    assert all(np.array_equal(w_h[k], w_d[k]) for k in w_h)


def test_train_errors():
    from dca_b200.train import train
    Y = synth_counts(300, 64, 14)
    dd = _dd(Y)
    net = _net("nb", 64)
    host = _host_arm(dd, Y)
    with pytest.raises(ValueError, match="stream"):
        train(host, net, epochs=1, batch_size=64, device_data=dd, stream=True, verbose=False)
    with pytest.raises(ValueError, match="output_subset"):
        train(host, net, epochs=1, batch_size=64, device_data=dd, output_subset=list(host.raw.var_names[:2]), verbose=False)


def test_dataset_larger_than_free_memory(monkeypatch):
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a, **k: (1 << 20, 80 << 30))
    with pytest.raises(MemoryError, match="stream=True"):
        _dd(synth_counts(512, 1024, 15))


# ------------------------------------------------------------------------------------------ end to end
def test_dca_device_preprocess_matches_host_mode():
    from dca_b200.api import dca
    Y = synth_counts(1000, 300, 16)
    kw = dict(ae_type="zinb-conddisp", epochs=4, batch_size=128, return_info=True, copy=True)
    a_h = dca(_adata(Y), **kw)
    a_d = dca(_adata(Y), training_kwds={"preprocess": "device"}, **kw)
    assert a_h.X.shape == a_d.X.shape and set(a_h.obsm_keys()) == set(a_d.obsm_keys())
    assert set(a_h.uns_keys()) == set(a_d.uns_keys()) and 'dca_device_data' not in a_d.uns_keys()
    for k in a_h.obsm_keys():
        assert a_h.obsm[k].shape == a_d.obsm[k].shape
    assert np.array_equal(a_h.raw.X, a_d.raw.X)
    for k in ("n_counts", "size_factors"):
        assert np.array_equal(np.asarray(a_h.obs[k]), np.asarray(a_d.obs[k])), k
    lh, ld = a_h.uns['dca_loss_history'], a_d.uns['dca_loss_history']
    assert lh.keys() == ld.keys()
    for k in ("loss", "val_loss"):
        np.testing.assert_allclose(ld[k], lh[k], rtol=1e-3)
    a_l = dca(_adata(Y), mode="latent", training_kwds={"preprocess": "device"}, epochs=1, copy=True)
    assert np.array_equal(a_l.X, Y) and a_l.obsm['X_dca'].shape == (1000, 32)


def test_cli_device_preprocess_round_trip(tmp_path):
    from dca_b200.__main__ import main
    Y = synth_counts(240, 80, 17).astype(int)
    Y[:, 5] = 0                                    # filtered out by the CLI's filter_min_counts
    genes = ["g%d" % i for i in range(80)]
    df = pd.DataFrame(Y.T, index=genes, columns=["c%d" % i for i in range(240)])
    inp = tmp_path / "counts.tsv"
    df.to_csv(inp, sep="\t")
    subset = tmp_path / "genes.txt"
    subset.write_text("\n".join(["g3", "g10", "g42", "g77"]))
    outs = {}
    for mode in ("host", "device"):
        out = tmp_path / mode
        main([str(inp), str(out), "--type", "zinb-conddisp", "-e", "2", "-b", "64", "--testsplit",
              "--denoisesubset", str(subset), "--preprocess", mode])
        outs[mode] = out
    files = sorted(p.name for p in outs["host"].iterdir())
    assert files == sorted(p.name for p in outs["device"].iterdir())
    for f in ("mean.tsv", "latent.tsv", "dispersion.tsv", "dropout.tsv"):
        hdr = 0 if f == "mean.tsv" else None                            # only mean.tsv has a header line
        h = pd.read_csv(outs["host"] / f, sep="\t", index_col=0, header=hdr)
        d = pd.read_csv(outs["device"] / f, sep="\t", index_col=0, header=hdr)
        assert h.shape == d.shape and list(h.index) == list(d.index), f
        if hdr is not None:
            assert list(h.columns) == list(d.columns), f
    assert pd.read_csv(outs["device"] / "mean.tsv", sep="\t", index_col=0).shape == (4, 240)
