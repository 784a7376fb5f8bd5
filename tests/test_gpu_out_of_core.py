"""Out-of-core mode (stream_data.StreamedDataset): statistics from chunked column passes over packed host counts, the
exact expansion of streamed batches, streamed training and prediction -- bit-identical to the resident DeviceDataset
on the same counts."""
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


def _sd(Y, **kw):
    from dca_b200.stream_data import StreamedDataset
    return StreamedDataset.from_counts(Y, DEV, **kw)


def _np(t):
    if isinstance(t, torch.Tensor):
        return (t.view(torch.int16) if t.dtype == torch.bfloat16 else t).cpu().numpy()
    return np.asarray(t)


def _eq(a, b):
    a, b = _np(a), _np(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _cases():
    yield "1000x304", synth_counts(1000, 304, 0)
    yield "4096x2000", synth_counts(4096, 2000, 1)
    Y = synth_counts(1024, 20000, 2)
    Y[3, 7] = 1e6                                          # an overflow entry in every packing width
    yield "1024x20000", Y


# ------------------------------------------------------------------------------------------------ statistics
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("case", ["1000x304", "4096x2000", "1024x20000"])
def test_chunked_statistics_are_the_whole_matrix_bits(case, fmt):
    from dca_b200 import io
    from dca_b200.stream_data import _moments, _totals
    Y = dict(_cases())[case]
    N = Y.shape[0]
    dd = _dd(Y)
    pc = io.pack_counts(Y, fmt)
    for chunk in (1, 7, 64, 1000, N, N + 5):             # chunks straddle slices and are not multiples of 8
        if chunk == 1 and N > 1024:
            continue                                      # (4096 one-row chunks: covered by the smaller shapes)
        nc, gt, bad = _totals(pc, DEV, chunk_rows=min(chunk, N))
        assert _eq(nc, dd.n_counts) and _eq(gt, dd.gene_totals_host) and bad == dd.n_bad == 0, chunk
        mean, std = _moments(pc, nc, dd.median, dd.flags, DEV, chunk_rows=min(chunk, N))
        assert _eq(mean, dd.mean) and _eq(std, dd.std), chunk


@pytest.mark.parametrize("flags", list(itertools.product([False, True], repeat=3)))
def test_all_flag_combinations(flags):
    Y = synth_counts(1000, 304, 3)
    Y[17] = 0                                            # a cell without counts: dropped by size factors / the filter
    for filt, chunk in ((False, 7), (True, 64)):          # the carried passes split across chunks for every flag set
        kw = dict(size_factors=flags[0], logtrans_input=flags[1], normalize_input=flags[2], filter_min_counts=filt)
        dd, sd = _dd(Y, **kw), _sd(Y, chunk_rows=chunk, **kw)
        assert _eq(sd.n_counts_host, dd.n_counts_host) and _eq(sd.size_factors_host, dd.size_factors_host)
        assert _eq(sd.mean, dd.mean) and _eq(sd.std, dd.std) and sd.median == dd.median and sd.flags == dd.flags
        assert _eq(sd.gene_totals_host, dd.gene_totals_host) and _eq(sd.input_gene_totals, dd.input_gene_totals)
        for m in ("gene_mask", "cell_mask", "sf_mask"):
            assert np.array_equal(getattr(sd, m), getattr(dd, m)), m
        Ys, Xs, sfs = sd.expand()
        assert _eq(Ys, dd.Y) and _eq(Xs, dd.X) and _eq(sfs, dd.sf)


def test_two_pass_variance():
    Y = synth_counts(3001, 64, 20)
    Y[:, 10] = 1e6 + np.random.default_rng(0).integers(0, 5, 3001)
    for flags in ((False, False, True), (False, True, True)):
        kw = dict(size_factors=flags[0], logtrans_input=flags[1], normalize_input=flags[2])
        dd = _dd(Y, **kw)
        for chunk in (7, 64, 3001):
            sd = _sd(Y, chunk_rows=chunk, **kw)
            assert _eq(sd.std, dd.std) and _eq(sd.mean, dd.mean), chunk


def test_csr_input_and_gene_filter():
    import scipy.sparse as sp
    Y = synth_counts(600, 96, 4)
    Y[:, 8:16] = 0                                       # eight all-zero genes: 88 remain after filtering
    dd = _dd(Y, filter_min_counts=True)
    sd = _sd(sp.csr_matrix(Y), filter_min_counts=True)
    assert sd.n_genes == 88 and np.array_equal(sd.gene_mask, dd.gene_mask)
    assert _eq(sd.mean, dd.mean) and _eq(sd.std, dd.std) and _eq(sd.n_counts_host, dd.n_counts_host)
    Y[:, 0] = 0                                          # 87 genes would remain: not a packed width
    with pytest.raises(ValueError, match="multiple of 8"):
        _sd(Y, filter_min_counts=True)
    with pytest.raises(ValueError, match="multiple of 8"):
        _sd(synth_counts(10, 12, 5))


# ------------------------------------------------------------------------------------------------ transform
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("big", [False, True])
@pytest.mark.parametrize("x_dtype", ["float32", "bfloat16"])
def test_exact_expansion_is_the_resident_rows(fmt, big, x_dtype):
    Y = synth_counts(700, 512, 6)
    if big:
        Y[3, 7], Y[400, 511] = 1e6, 300
    dd = _dd(Y, x_dtype=x_dtype)
    sd = _sd(Y, x_dtype=x_dtype, bits=fmt)
    assert sd.pc.bits == (1 if fmt == "sparse" else fmt)
    if big:
        assert len(sd.pc.entries) > 0
    rows = np.arange(123, 611)
    Ys, Xs, sfs = sd.take(rows).expand()
    r = torch.from_numpy(rows).to(DEV)
    assert _eq(Ys, dd.Y[r]) and _eq(Xs, dd.X[r]) and _eq(sfs, dd.sf[r])


# ------------------------------------------------------------------------------------------------ training
def _net(ae_type, G, x_dtype="float32", gemm_path="auto", seed=0):
    from dca_b200.network import AE_types
    net = AE_types[ae_type](input_size=G, output_size=G, hidden_size=(64, 32, 64), x_dtype=x_dtype, gemm_path=gemm_path)
    net.build(max_batch=256, seed=seed)
    return net


def _fit(net, **kw):
    from dca_b200.train import train
    np.random.seed(3)
    return train(None, net, epochs=2, batch_size=256, validation_split=0.1, verbose=False, **kw).history


@pytest.mark.parametrize("ae_type,x_dtype,gemm_path", [("zinb-conddisp", "float32", "auto"),
                                                       ("zinb-conddisp", "bfloat16", "auto"),
                                                       ("nb", "float32", "auto"),
                                                       ("zinb-conddisp", "float32", "generic")])
def test_train_matches_resident(ae_type, x_dtype, gemm_path):
    """zinb-conddisp and nb on the tensor-core path: history, weights and BatchNorm state bit-identical.  The generic
    path splits K with atomics: there two runs of the SAME arm already differ, and RMSprop turns last-bit gradient noise
    into learning-rate-sized steps, so it is held to 1e-3 of the losses and 2e-2 of each weight tensor's scale."""
    G = 2000
    Y = synth_counts(1500, G, 12)
    dd, sd = _dd(Y, x_dtype=x_dtype), _sd(Y, x_dtype=x_dtype, batch=256)
    n_d, n_s = _net(ae_type, G, x_dtype, gemm_path), _net(ae_type, G, x_dtype, gemm_path)
    if gemm_path == "auto" and ae_type == "zinb-conddisp":
        assert n_s.engine.info()["tc_heads"] and n_s.engine.info()["tc_encoder"]
    h_d = _fit(n_d, device_data=dd, shuffle=False)
    h_s = _fit(n_s, stream_data=sd, shuffle=False)
    w_d, w_s = n_d.engine.get_weights(), n_s.engine.get_weights()
    if gemm_path == "auto":
        assert h_d == h_s
        assert all(np.array_equal(w_d[k], w_s[k]) for k in w_d)
    else:
        for k in ("loss", "val_loss"):
            np.testing.assert_allclose(h_s[k], h_d[k], rtol=1e-3)
        for k in w_d:
            assert np.max(np.abs(w_d[k] - w_s[k]), initial=0.0) <= 2e-2 * max(np.max(np.abs(w_d[k]), initial=0.0), 1.0), k


def test_shuffled_training_replays_on_resident_batches():
    """shuffle=True: the rows are shuffled once and every epoch permutes whole batches; replaying that order with
    resident steps on the DeviceDataset gives the same bits."""
    from dca_b200.train import train
    G, N, bs, epochs = 2000, 1100, 256, 2
    Y = synth_counts(N, G, 13)
    dd, sd = _dd(Y), _sd(Y, batch=bs)
    n_s, n_r = _net("zinb-conddisp", G), _net("zinb-conddisp", G)
    np.random.seed(5)
    hist = train(None, n_s, epochs=epochs, batch_size=bs, validation_split=0.1, verbose=False, stream_data=sd).history
    assert np.all(np.isfinite(hist["loss"])) and np.all(np.isfinite(hist["val_loss"]))
    np.random.seed(5)
    n_tr = int(N * 0.9)
    order0 = np.arange(n_tr)
    np.random.shuffle(order0)
    nb = (n_tr + bs - 1) // bs
    e = n_r.engine
    e.set_optimizer("RMSprop"); e.reset_optimizer()
    rows_all = dd.rows
    losses = []
    for _ in range(epochs):
        border = np.random.permutation(nb)
        e.read_epoch_acc(reset=True)
        for k in border:
            r = torch.from_numpy(order0[k * bs: min(n_tr, (k + 1) * bs)].astype(np.int32)).to(DEV)
            e.train_step(dd.X, dd.Y, dd.sf, rows=rows_all[r.long()])
            e.apply_update(1e-3, 5.0, 1.0)
        for s0 in range(n_tr, N, bs):
            e.eval_step(dd.X, dd.Y, dd.sf, rows=rows_all[s0:min(N, s0 + bs)])
        acc = e.read_epoch_acc(reset=False)
        losses.append((acc[0] / acc[1], acc[2] / acc[3]))
    assert [float(a) for a, _ in losses] == hist["loss"] and [float(b) for _, b in losses] == hist["val_loss"]
    w_s, w_r = n_s.engine.get_weights(), e.get_weights()
    assert all(np.array_equal(w_s[k], w_r[k]) for k in w_s)


def test_train_errors():
    from dca_b200.train import train
    Y = synth_counts(300, 64, 14)
    sd = _sd(Y)
    net = _net("nb", 64)
    with pytest.raises(ValueError, match="use_raw_as_output"):
        train(None, net, epochs=1, batch_size=64, stream_data=sd, use_raw_as_output=False, verbose=False)
    with pytest.raises(NotImplementedError, match="output_subset"):
        train(None, net, epochs=1, batch_size=64, stream_data=sd, output_subset=["a"], verbose=False)
    with pytest.raises(ValueError, match="not both"):
        train(None, net, epochs=1, batch_size=64, stream_data=sd, device_data=_dd(Y), verbose=False)


def test_overflow_heavy_counts_stream_at_every_batch_size():
    """Deep counts packed for a training batch of 32 (4 bits) overflow the staging of a 4096-row predict batch: the
    streaming calls widen the packing where a batch would not fit, and training and prediction still give the resident
    bits."""
    from tests.test_packed_rows_host import _deep_counts
    from dca_b200 import io
    G = 2000
    Y = _deep_counts(8192, G, 7)
    dd, sd = _dd(Y), _sd(Y, batch=32)
    assert sd.pc.bits == 4 and io._worst_batch(sd.pc.indptr, 4096) > max(4096, 4096 * G // 32)
    n_d, n_s = _net("zinb-conddisp", G), _net("zinb-conddisp", G)
    h_d = _fit(n_d, device_data=dd, shuffle=False)
    h_s = _fit(n_s, stream_data=sd, shuffle=False)
    assert h_d == h_s
    w_d, w_s = n_d.engine.get_weights(), n_s.engine.get_weights()
    assert all(np.array_equal(w_d[k], w_s[k]) for k in w_d)
    r_d = n_d._run_predict(None, True, True, True, True, device_data=dd)
    r_s = n_d._run_predict(None, True, True, True, True, stream_data=sd)
    for k in ("mean", "dispersion", "pi", "latent"):
        assert _eq(r_d[k], r_s[k]), k
    from dca_b200.train import train
    np.random.seed(1)                                     # batch 32, rows shuffled into a new order before streaming
    h = train(None, n_s, epochs=1, batch_size=32, validation_split=0.1, verbose=False, stream_data=sd).history
    assert np.all(np.isfinite(h["loss"])) and np.all(np.isfinite(h["val_loss"]))


# ------------------------------------------------------------------------------------------------ prediction
@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "nb", "zinb-shared"])
def test_predict_matches_resident(ae_type):
    G, N = 512, 5000                                      # two predict batches: 4096 + 904
    Y = synth_counts(N, G, 15)
    dd, sd = _dd(Y), _sd(Y)
    net = _net(ae_type, G)
    r_d = net._run_predict(None, True, True, True, True, device_data=dd)
    r_s = net._run_predict(None, True, True, True, True, stream_data=sd)
    for k in ("mean", "dispersion", "pi", "latent"):
        if r_d.get(k) is None:
            assert r_s.get(k) is None, k
        elif ae_type == "zinb-shared":
            # the extra AE types run the fp32 generic GEMMs, whose split-K atomics make two resident predictions differ:
            # up to 2.7e-7 of an output's largest value on an H100 (streamed against resident: 3.1e-7); held to 2e-6
            a, b = r_d[k], r_s[k]
            assert a.shape == b.shape and np.max(np.abs(a - b)) <= 2e-6 * np.max(np.abs(a)), k
        else:
            assert _eq(r_d[k], r_s[k]), k


# ------------------------------------------------------------------------------------------------ end to end
def _adata(Y):
    from dca_b200.anndata_lite import AnnData
    return AnnData(np.array(Y, dtype=np.float32))


def _same_adata(a, b):
    assert _eq(a.X, b.X) and _eq(a.raw.X, b.raw.X)
    assert set(a.obsm_keys()) == set(b.obsm_keys()) and all(_eq(a.obsm[k], b.obsm[k]) for k in a.obsm_keys())
    assert list(a.var.columns) == list(b.var.columns)
    for k in ("n_counts", "size_factors"):
        assert _eq(np.asarray(a.obs[k]), np.asarray(b.obs[k])), k
    assert a.uns.get('dca_loss_history') == b.uns.get('dca_loss_history')


def test_dca_stream_matches_device_preprocess(monkeypatch):
    from dca_b200.api import dca
    Y = synth_counts(1000, 304, 16)
    Y[11] = 0                                             # dropped by normalize_per_cell in both modes
    kw = dict(ae_type="zinb-conddisp", epochs=3, batch_size=128, return_info=True, copy=True)
    a_d = dca(_adata(Y), training_kwds={"preprocess": "device", "shuffle": False}, **kw)
    a_s = dca(_adata(Y), training_kwds={"preprocess": "device", "stream": True, "shuffle": False}, **kw)
    assert a_s.n_obs == 999
    _same_adata(a_d, a_s)
    l_d = dca(_adata(Y), mode="latent", training_kwds={"preprocess": "device", "shuffle": False}, epochs=1, copy=True)
    l_s = dca(_adata(Y), mode="latent", training_kwds={"preprocess": "device", "stream": True, "shuffle": False},
              epochs=1, copy=True)
    assert _eq(l_d.obsm['X_dca'], l_s.obsm['X_dca']) and _eq(l_d.X, l_s.X)
    # 'auto': the streamed mode when the resident dataset does not fit, the resident one otherwise; the same results
    import dca_b200.stream_data as S
    import dca_b200.device_data as Dd
    used = []
    orig = S.StreamedDataset.from_counts

    def recording(cls, *a, **k):
        used.append("stream")
        return orig(*a, **k)
    monkeypatch.setattr(S.StreamedDataset, "from_counts", classmethod(recording))
    auto = dict(kw, epochs=1)
    a1 = dca(_adata(Y), training_kwds={"preprocess": "device", "stream": "auto", "shuffle": False}, **auto)
    assert used == []
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a, **k: (1 << 20, 80 << 30))
    a2 = dca(_adata(Y), training_kwds={"preprocess": "device", "stream": "auto", "shuffle": False}, **auto)
    assert used == ["stream"]
    monkeypatch.undo()
    _same_adata(a1, a2)
    assert Dd.DeviceDataset.device_bytes(Y) > 1 << 20


def test_cli_stream_round_trip(tmp_path):
    from dca_b200.__main__ import main
    Y = synth_counts(240, 88, 17).astype(int)
    Y[:, 40:48] = 0                                       # eight genes filtered out by the CLI's filter_min_counts
    genes = ["g%d" % i for i in range(88)]
    df = pd.DataFrame(Y.T, index=genes, columns=["c%d" % i for i in range(240)])
    inp = tmp_path / "counts.tsv"
    df.to_csv(inp, sep="\t")
    outs = {}
    for name, extra in (("device", []), ("stream", ["--stream"])):
        out = tmp_path / name
        main([str(inp), str(out), "--type", "zinb-conddisp", "-e", "2", "-b", "64", "--testsplit",
              "--preprocess", "device"] + extra)
        outs[name] = out
    files = sorted(p.name for p in outs["device"].iterdir())
    assert files == sorted(p.name for p in outs["stream"].iterdir())
    for f in ("mean.tsv", "latent.tsv", "dispersion.tsv", "dropout.tsv"):
        hdr = 0 if f == "mean.tsv" else None
        d = pd.read_csv(outs["device"] / f, sep="\t", index_col=0, header=hdr)
        s = pd.read_csv(outs["stream"] / f, sep="\t", index_col=0, header=hdr)
        assert d.shape == s.shape and list(d.index) == list(s.index), f
        if hdr is not None:
            assert list(d.columns) == list(s.columns), f
    assert pd.read_csv(outs["stream"] / "mean.tsv", sep="\t", index_col=0).shape == (80, 240)
    subset = tmp_path / "genes.txt"
    subset.write_text("g3\ng10")
    with pytest.raises(NotImplementedError, match="denoisesubset"):
        main([str(inp), str(tmp_path / "x"), "-e", "1", "--preprocess", "device", "--stream", "--denoisesubset", str(subset)])
    with pytest.raises(ValueError, match="--preprocess device"):
        main([str(inp), str(tmp_path / "y"), "-e", "1", "--stream"])
