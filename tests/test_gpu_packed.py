"""Packed counts resident in device memory (packed_data.PackedDeviceDataset): the GPU packer against the host packer
byte for byte, statistics and filters, the row-indexed exact expansion, training, prediction and the end-to-end paths --
bit-identical to the resident DeviceDataset on the same counts."""
import itertools

import numpy as np
import pandas as pd
import pytest
import torch

from tests.util import synth_counts

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FORMATS = ["sparse", 4, 8, 16]


def _dd(Y, **kw):
    from dca_b200.device_data import DeviceDataset
    return DeviceDataset.from_counts(Y, DEV, **kw)


def _pd(Y, **kw):
    from dca_b200.packed_data import PackedDeviceDataset
    return PackedDeviceDataset.from_counts(Y, DEV, **kw)


def _np(t):
    if isinstance(t, torch.Tensor):
        return (t.view(torch.int16) if t.dtype == torch.bfloat16 else t).cpu().numpy()
    return np.asarray(t)


def _eq(a, b):
    a, b = _np(a), _np(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _bytes_eq(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.nbytes == b.nbytes and np.array_equal(a.reshape(-1).view(np.uint8), b.reshape(-1).view(np.uint8))


_CASES = {}


def _case(name):
    if not _CASES:
        _CASES["1000x304"] = synth_counts(1000, 304, 0)
        _CASES["4096x2000"] = synth_counts(4096, 2000, 1)
        Y = synth_counts(1024, 20000, 2)
        Y[3, 7] = 1e6                                      # an overflow entry in every packing width
        _CASES["1024x20000"] = Y
    return _CASES[name]


# ------------------------------------------------------------------------------------------------ packer
@pytest.mark.parametrize("bits", ["sparse", 4, 8, 16, "auto"])
@pytest.mark.parametrize("csr", [False, True])
@pytest.mark.parametrize("case", ["1000x304", "4096x2000", "1024x20000"])
def test_packer_bytes_are_the_host_packers(case, csr, bits):
    import scipy.sparse as sp
    from dca_b200 import io
    Y = _case(case)
    N = Y.shape[0]
    ref = io.pack_rows(Y, bits, batch=None)
    chunks = (1, 7, 64, N - 1, N) if N <= 1000 else (7, 64, N - 1, N)
    for chunk in chunks:
        pdd = _pd(sp.csr_matrix(Y) if csr else Y, bits=bits, chunk_rows=chunk, size_factors=False,
                  normalize_input=False)          # (no moment passes: only the packing is under test here)
        got = pdd.host_packed()
        assert got.bits == ref.bits, chunk
        assert _bytes_eq(got.packed, ref.packed) and _bytes_eq(got.indptr, ref.indptr), chunk
        assert _bytes_eq(got.entries, ref.entries), chunk
        if ref.bits == 1:
            assert _bytes_eq(got.nib_indptr, ref.nib_indptr) and _bytes_eq(got.nibbles, ref.nibbles), chunk


def test_packer_rejects_what_the_host_packer_rejects():
    from dca_b200 import io
    for bad in (0.5, -1.0):
        Y = synth_counts(100, 64, 3)
        Y[5, 9] = bad
        with pytest.raises(ValueError, match="non-negative integers"):
            io.pack_rows(Y, "auto")
        with pytest.raises(ValueError, match="non-negative integers"):
            _pd(Y)
    with pytest.raises(ValueError, match="bits must be"):
        _pd(synth_counts(10, 64, 4), bits=5)


# ------------------------------------------------------------------------------------------------ statistics
@pytest.mark.parametrize("flags", list(itertools.product([False, True], repeat=3)))
def test_statistics_and_filters_are_the_resident_bits(flags):
    Y = synth_counts(1000, 312, 5)
    Y[17] = 0                                            # a cell without counts: dropped by size factors / the filter
    Y[:, 100:108] = 0                                    # eight all-zero genes: 304 remain after filtering
    for filt, chunk in ((False, 7), (True, 64)):
        kw = dict(size_factors=flags[0], logtrans_input=flags[1], normalize_input=flags[2], filter_min_counts=filt)
        dd, pdd = _dd(Y, **kw), _pd(Y, chunk_rows=chunk, **kw)
        assert _eq(pdd.n_counts_host, dd.n_counts_host) and _eq(pdd.size_factors_host, dd.size_factors_host)
        assert _eq(pdd.mean, dd.mean) and _eq(pdd.std, dd.std) and pdd.median == dd.median and pdd.flags == dd.flags
        assert _eq(pdd.gene_totals_host, dd.gene_totals_host) and _eq(pdd.input_gene_totals, dd.input_gene_totals)
        for m in ("gene_mask", "cell_mask", "sf_mask"):
            assert np.array_equal(getattr(pdd, m), getattr(dd, m)), m
        Yp, Xp, sfp = pdd.expand()
        assert _eq(Yp, dd.Y) and _eq(Xp, dd.X) and _eq(sfp, dd.sf)


def test_filter_to_a_gene_count_off_the_packed_width_raises():
    Y = synth_counts(300, 96, 6)
    Y[:, 8:15] = 0                                       # seven all-zero genes: 89 would remain
    with pytest.raises(ValueError, match="multiple of 8"):
        _pd(Y, filter_min_counts=True)
    with pytest.raises(ValueError, match="multiple of 8"):
        _pd(synth_counts(10, 12, 7))


# ------------------------------------------------------------------------------------------------ expansion
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("x_dtype", ["float32", "bfloat16"])
def test_row_indexed_expansion_is_the_resident_rows(fmt, x_dtype):
    Y = synth_counts(700, 512, 8)
    Y[3, 7], Y[400, 511], Y[650, 0] = 1e6, 300, 70000      # overflow entries at every width
    dd = _dd(Y, x_dtype=x_dtype)
    pdd = _pd(Y, x_dtype=x_dtype, bits=fmt)
    assert pdd.bits == (1 if fmt == "sparse" else fmt) and int(pdd.ovf_indptr[-1]) > 0
    rng = np.random.default_rng(0)
    lists = {"random": rng.permutation(700)[:300], "repeated": np.array([3, 3, 400, 3, 650, 650, 0]),
             "descending": np.arange(699, -1, -1), "single": np.array([400]),
             "max_batch": rng.integers(0, 700, 4096)}
    for name, rows in lists.items():
        Yp, Xp, sfp = pdd.take(rows).expand()
        r = torch.from_numpy(rows).to(DEV)
        assert _eq(Yp, dd.Y[r]) and _eq(Xp, dd.X[r]) and _eq(sfp, dd.sf[r]), name


# ------------------------------------------------------------------------------------------------ training
def _net(ae_type, G, x_dtype="float32", gemm_path="auto", seed=0):
    from dca_b200.network import AE_types
    net = AE_types[ae_type](input_size=G, output_size=G, hidden_size=(64, 32, 64), x_dtype=x_dtype, gemm_path=gemm_path)
    net.build(max_batch=256, seed=seed)
    return net


def _fit(net, **kw):
    from dca_b200.train import train
    np.random.seed(3)
    return train(None, net, epochs=3, batch_size=256, validation_split=0.1, verbose=False, **kw).history


@pytest.mark.parametrize("ae_type,x_dtype,gemm_path", [("zinb-conddisp", "float32", "auto"),
                                                       ("zinb-conddisp", "bfloat16", "auto"),
                                                       ("nb", "float32", "auto"),
                                                       ("zinb-conddisp", "float32", "generic")])
def test_train_matches_resident(ae_type, x_dtype, gemm_path):
    """Rows reshuffled every epoch (shuffle=True) from the same NumPy seed.  zinb-conddisp and nb on the tensor-core
    path: history, weights and BatchNorm state bit-identical.  The generic path splits K with atomics, so two resident
    runs already differ: held to the tolerances of the streamed arm in test_gpu_out_of_core.test_train_matches_resident,
    for the same reason."""
    G = 2000
    Y = synth_counts(1500, G, 12)
    dd, pdd = _dd(Y, x_dtype=x_dtype), _pd(Y, x_dtype=x_dtype)
    n_d, n_p = _net(ae_type, G, x_dtype, gemm_path), _net(ae_type, G, x_dtype, gemm_path)
    if gemm_path == "auto" and ae_type == "zinb-conddisp":
        assert n_p.engine.info()["tc_heads"] and n_p.engine.info()["tc_encoder"]
    h_d = _fit(n_d, device_data=dd)
    h_p = _fit(n_p, packed_data=pdd)
    w_d, w_p = n_d.engine.get_weights(), n_p.engine.get_weights()
    if gemm_path == "auto":
        assert h_d == h_p
        assert all(np.array_equal(w_d[k], w_p[k]) for k in w_d)     # weights and BatchNorm moving statistics
    else:
        for k in ("loss", "val_loss"):
            np.testing.assert_allclose(h_p[k], h_d[k], rtol=1e-3)
        for k in w_d:
            assert np.max(np.abs(w_d[k] - w_p[k]), initial=0.0) <= 2e-2 * max(np.max(np.abs(w_d[k]), initial=0.0), 1.0), k


# ------------------------------------------------------------------------------------------------ prediction
@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "nb", "zinb-shared"])
def test_predict_matches_resident(ae_type):
    G, N = 512, 5000                                      # two predict batches: 4096 + 904
    Y = synth_counts(N, G, 15)
    dd, pdd = _dd(Y), _pd(Y)
    net = _net(ae_type, G)
    r_d = net._run_predict(None, True, True, True, True, device_data=dd)
    r_p = net._run_predict(None, True, True, True, True, packed_data=pdd)
    for k in ("mean", "dispersion", "pi", "latent"):
        if r_d.get(k) is None:
            assert r_p.get(k) is None, k
        elif ae_type == "zinb-shared":
            # split-K atomics of the fp32 generic GEMMs: the rule of test_gpu_out_of_core.test_predict_matches_resident
            a, b = r_d[k], r_p[k]
            assert a.shape == b.shape and np.max(np.abs(a - b)) <= 2e-6 * np.max(np.abs(a)), k
        else:
            assert _eq(r_d[k], r_p[k]), k


# ------------------------------------------------------------------------------------------------ end to end
def _adata(Y):
    from dca_b200.anndata_lite import AnnData
    return AnnData(np.array(Y, dtype=np.float32))


def _same_adata(a, b):
    assert _eq(a.X, b.X) and _eq(a.raw.X, b.raw.X)
    assert set(a.obsm_keys()) == set(b.obsm_keys()) and all(_eq(a.obsm[k], b.obsm[k]) for k in a.obsm_keys())
    assert list(a.var.columns) == list(b.var.columns)
    assert list(a.obs.columns) == list(b.obs.columns)
    for k in ("n_counts", "size_factors"):
        assert _eq(np.asarray(a.obs[k]), np.asarray(b.obs[k])), k
    assert a.uns.get('dca_loss_history') == b.uns.get('dca_loss_history')


def test_dca_packed_matches_device_preprocess():
    from dca_b200.api import dca
    Y = synth_counts(1000, 304, 16)
    Y[11] = 0                                             # dropped by normalize_per_cell in both modes
    kw = dict(ae_type="zinb-conddisp", epochs=3, batch_size=128, return_info=True, copy=True)
    a_d = dca(_adata(Y), training_kwds={"preprocess": "device"}, **kw)
    a_p = dca(_adata(Y), training_kwds={"preprocess": "device", "packed": True}, **kw)
    assert a_p.n_obs == 999
    _same_adata(a_d, a_p)
    l_d = dca(_adata(Y), mode="latent", training_kwds={"preprocess": "device"}, epochs=1, copy=True)
    l_p = dca(_adata(Y), mode="latent", training_kwds={"preprocess": "device", "packed": True}, epochs=1, copy=True)
    assert _eq(l_d.obsm['X_dca'], l_p.obsm['X_dca']) and _eq(l_d.X, l_p.X)


def test_cli_packed_round_trip(tmp_path):
    from dca_b200.__main__ import main
    Y = synth_counts(240, 88, 17).astype(int)
    Y[:, 40:48] = 0                                       # eight genes filtered out by the CLI's filter_min_counts
    genes = ["g%d" % i for i in range(88)]
    df = pd.DataFrame(Y.T, index=genes, columns=["c%d" % i for i in range(240)])
    inp = tmp_path / "counts.tsv"
    df.to_csv(inp, sep="\t")
    outs = {}
    for name, extra in (("device", []), ("packed", ["--packed"])):
        out = tmp_path / name
        main([str(inp), str(out), "--type", "zinb-conddisp", "-e", "2", "-b", "64", "--testsplit",
              "--preprocess", "device"] + extra)
        outs[name] = out
    files = sorted(p.name for p in outs["device"].iterdir())
    assert files == sorted(p.name for p in outs["packed"].iterdir())
    for f in ("mean.tsv", "latent.tsv", "dispersion.tsv", "dropout.tsv"):
        hdr = 0 if f == "mean.tsv" else None
        d = pd.read_csv(outs["device"] / f, sep="\t", index_col=0, header=hdr)
        p = pd.read_csv(outs["packed"] / f, sep="\t", index_col=0, header=hdr)
        assert d.shape == p.shape and list(d.index) == list(p.index), f
        if hdr is not None:
            assert list(d.columns) == list(p.columns), f
    assert pd.read_csv(outs["packed"] / "mean.tsv", sep="\t", index_col=0).shape == (80, 240)


# ------------------------------------------------------------------------------------------------ errors
def test_train_errors(monkeypatch):
    from dca_b200 import dist
    from dca_b200.train import train
    Y = synth_counts(300, 64, 14)
    pdd = _pd(Y)
    net = _net("nb", 64)
    for other in (dict(stream=True), dict(device_data=_dd(Y)), dict(stream_data=object())):
        with pytest.raises(ValueError, match="cannot be combined"):
            train(None, net, epochs=1, batch_size=64, packed_data=pdd, verbose=False, **other)
    with pytest.raises(ValueError, match="use_raw_as_output"):
        train(None, net, epochs=1, batch_size=64, packed_data=pdd, use_raw_as_output=False, verbose=False)
    with pytest.raises(NotImplementedError, match="output_subset"):
        train(None, net, epochs=1, batch_size=64, packed_data=pdd, output_subset=["a"], verbose=False)
    monkeypatch.setattr(dist, "rank_world", lambda: (0, 2))
    with pytest.raises(NotImplementedError, match="one GPU"):
        train(None, net, epochs=1, batch_size=64, packed_data=pdd, verbose=False)
