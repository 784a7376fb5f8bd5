"""Streamed and packed datasets of any gene count (``pad_genes=True``): the rows are stored zero-padded to the next
multiple of 8, and preprocessing, training, prediction and the written files are those of the resident
``DeviceDataset`` on the same counts.  The pad genes never reach the model: a count planted in one changes no bit.

Determinism.  A gene count off a multiple of 8 trains on the fp32 CUDA-core path, whose split-K GEMMs (K >= 256, fewer
output tiles than two per SM) add their partial sums with atomics, and 'nb' sums its theta gradient with atomics.  Two
resident runs of the same model can then differ in the last bits.  Below 256 genes and batches under 256 rows no GEMM
splits, and 'zinb-conddisp' is deterministic: there the comparisons are bit for bit ('poisson' sums its loss with
double atomics).  At about 20 000 genes a second resident run measures the path's own spread: when it reproduces the
first run bit for bit the streamed and packed runs must too; otherwise they are held to the tolerances of
tests/test_gpu_out_of_core.py for the same atomics (loss rtol 1e-4, weights 2e-2 of the largest weight), or four
times the rerun's own gap where that is larger."""
import ctypes as C
import itertools

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
import torch

from tests.util import synth_counts

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
WIDTHS = ["sparse", 4, 8, 16, "auto"]


def _dd(Y, **kw):
    from dca_b200.device_data import DeviceDataset
    return DeviceDataset.from_counts(Y, DEV, **kw)


def _sd(Y, **kw):
    from dca_b200.stream_data import StreamedDataset
    return StreamedDataset.from_counts(Y, DEV, pad_genes=True, **kw)


def _pd(Y, **kw):
    from dca_b200.packed_data import PackedDeviceDataset
    return PackedDeviceDataset.from_counts(Y, DEV, pad_genes=True, **kw)


KINDS = {"stream_data": _sd, "packed_data": _pd}


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


def _ragged_counts(n, g, seed):
    """Counts with a cell without counts, three all-zero genes (the filter leaves g - 3 genes) and overflow entries at
    every width."""
    Y = synth_counts(n, g, seed)
    Y[17] = 0
    Y[:, [5, 6, g - 2]] = 0
    Y[3, 7], Y[n // 2, 0], Y[n - 1, g - 1] = 1e6, 300, 70000
    return Y


# ------------------------------------------------------------------------------------------------ 1. preprocessing
@pytest.mark.parametrize("bits", WIDTHS)
@pytest.mark.parametrize("flags", list(itertools.product([False, True], repeat=3)))
def test_preprocessing_is_the_resident_bits(flags, bits):
    G0 = 97
    Y = _ragged_counts(700, G0, 1)
    for filt, chunk in ((False, 7), (True, 64)):
        kw = dict(size_factors=flags[0], logtrans_input=flags[1], normalize_input=flags[2], filter_min_counts=filt)
        dd = _dd(Y, **kw)
        G = dd.Y.shape[1]
        assert G == (94 if filt else 97) and G % 8 != 0
        for kind, make in KINDS.items():
            for csr in (False, True):
                ds = make(sp.csr_matrix(Y) if csr else Y, bits=bits, chunk_rows=chunk, **kw)
                where = (kind, csr, filt)
                assert ds.n_genes == G, where
                assert _eq(ds.n_counts_host, dd.n_counts_host) and _eq(ds.size_factors_host, dd.size_factors_host), where
                assert _eq(ds.mean, dd.mean) and _eq(ds.std, dd.std), where
                assert ds.median == dd.median and ds.flags == dd.flags, where
                assert _eq(ds.gene_totals_host, dd.gene_totals_host), where
                assert _eq(ds.input_gene_totals, dd.input_gene_totals), where
                for m in ("gene_mask", "cell_mask", "sf_mask"):
                    assert np.array_equal(getattr(ds, m), getattr(dd, m)), (where, m)
                Ye, Xe, sfe = ds.expand()
                assert Ye.shape == (dd.n, G), where
                assert _eq(Ye, dd.Y) and _eq(Xe, dd.X) and _eq(sfe, dd.sf), where


@pytest.mark.parametrize("x_dtype", ["float32", "bfloat16"])
def test_expansion_at_20k_genes_is_the_resident_rows(x_dtype):
    for G in (19999, 20004, 20007):
        Y = _ragged_counts(300, G, G)
        dd = _dd(Y, x_dtype=x_dtype)
        rows = np.random.default_rng(0).permutation(dd.n)[:123]
        r = torch.from_numpy(rows).to(DEV)
        for kind, make in KINDS.items():
            ds = make(Y, x_dtype=x_dtype)
            Ye, Xe, sfe = ds.take(rows).expand()
            assert _eq(Ye, dd.Y[r]) and _eq(Xe, dd.X[r]) and _eq(sfe, dd.sf[r]), (G, kind)


@pytest.mark.parametrize("bits", WIDTHS)
@pytest.mark.parametrize("csr", [False, True])
def test_gpu_packer_bytes_are_the_host_packers(csr, bits):
    from dca_b200 import io
    for G in (89, 20001):
        Y = _ragged_counts(400 if G < 1000 else 120, G, 2)
        Y[17, 3] = 1                                     # every cell keeps counts: no row is dropped
        gene_mask = Y.sum(0) >= 1
        for filt in (False, True):
            src = Y[:, gene_mask] if filt else Y
            ref = io.pack_rows(src, bits, batch=None, pad_genes=True)
            for chunk in (7, 64, Y.shape[0]):
                pdd = _pd(sp.csr_matrix(Y) if csr else Y, bits=bits, chunk_rows=chunk, size_factors=False,
                          normalize_input=False, filter_min_counts=filt)
                got = pdd.host_packed()
                where = (G, filt, chunk)
                assert got.genes == ref.genes == src.shape[1] and got.n_genes == ref.n_genes, where
                assert got.bits == ref.bits, where
                assert _bytes_eq(got.packed, ref.packed) and _bytes_eq(got.indptr, ref.indptr), where
                assert _bytes_eq(got.entries, ref.entries), where
                if ref.bits == 1:
                    assert _bytes_eq(got.nib_indptr, ref.nib_indptr) and _bytes_eq(got.nibbles, ref.nibbles), where


def test_default_still_refuses_ragged_gene_counts():
    from dca_b200.packed_data import PackedDeviceDataset
    from dca_b200.stream_data import StreamedDataset
    Y = synth_counts(50, 12, 3)
    for cls in (StreamedDataset, PackedDeviceDataset):
        with pytest.raises(ValueError, match="multiple of 8"):
            cls.from_counts(Y, DEV)


# ------------------------------------------------------------------------------------------------ 2. training
def _net(ae_type, G, x_dtype, max_batch, seed=0):
    from dca_b200.network import AE_types
    net = AE_types[ae_type](input_size=G, output_size=G, x_dtype=x_dtype)
    net.build(max_batch=max_batch, seed=seed)
    return net


def _fit(ae_type, G, x_dtype, bs, **data):
    from dca_b200.train import train
    net = _net(ae_type, G, x_dtype, bs)
    info = net.engine.info()
    assert not info["tc_heads"] and not info["tc_encoder"], info
    np.random.seed(3)
    hist = train(None, net, epochs=2, batch_size=bs, validation_split=0.1, verbose=False, shuffle=False, **data).history
    w = net.engine.get_weights()                          # weights and BatchNorm moving statistics
    net.engine.close()
    return hist, w


def _max_weight_gap(w_a, w_b):
    return max(float(np.max(np.abs(w_a[k] - w_b[k]), initial=0.0)) / max(float(np.max(np.abs(w_a[k]), initial=0.0)), 1.0)
               for k in w_a)


def _same_run(a, b):
    return a[0] == b[0] and all(np.array_equal(a[1][k], b[1][k]) for k in a[1])


def _loss_gap(h_a, h_b):
    return max(abs(a - b) / abs(a) for k in ("loss", "val_loss") for a, b in zip(h_a[k], h_b[k]))


def _check_runs(ref, ref2, runs, exact, loss_tol=1e-4, w_tol=2e-2):
    """runs {kind: (history, weights)} against the resident run ref; ref2: a second resident run (None: exact).  When
    the rerun differs, each kind is held to the larger of the given tolerances and four times the rerun's own gap."""
    exact = exact or (ref2 is not None and _same_run(ref, ref2))
    if ref2 is not None:
        lg, wg = _loss_gap(ref[0], ref2[0]), _max_weight_gap(ref[1], ref2[1])
        print("  resident rerun: bit-identical %s, loss gap %.2e, weight gap %.2e" % (_same_run(ref, ref2), lg, wg))
        loss_tol, w_tol = max(loss_tol, 4 * lg), max(w_tol, 4 * wg)
    for kind, run in runs.items():
        print("  %s: bit-identical %s, loss gap %.2e, weight gap %.2e"
              % (kind, _same_run(ref, run), _loss_gap(ref[0], run[0]), _max_weight_gap(ref[1], run[1])))
        assert set(run[1]) == set(ref[1]) and all(run[1][k].shape == ref[1][k].shape for k in ref[1])
        if exact:
            assert _same_run(ref, run), kind
        else:
            assert _loss_gap(ref[0], run[0]) <= loss_tol, kind
            assert _max_weight_gap(ref[1], run[1]) <= w_tol, kind


TRAIN_CASES = [("zinb-conddisp", "float32"), ("zinb-conddisp", "bfloat16"), ("nb", "float32"), ("nb", "bfloat16"),
               ("poisson", "float32")]


@pytest.mark.parametrize("ae_type,x_dtype", TRAIN_CASES)
@pytest.mark.parametrize("G,N,bs", [(19999, 8600, 4096), (20004, 700, 32)])
def test_train_at_20k_genes_matches_resident(G, N, bs, ae_type, x_dtype):
    """Two epochs with validation.  At batch 4096 (4 steps per epoch) the tolerances of the module docstring.  At batch
    32 (20 steps per epoch) RMSprop turns the last-bit differences of the atomics into a chaotic trajectory: on an H100
    two resident runs of these cases differed by up to 2.8e-3 of a loss and 3.3e-2 of the largest weight, so the kinds
    are held to 1e-2 and 1e-1 there (or four times the rerun's gap)."""
    Y = synth_counts(N, G, G + bs)
    dd = _dd(Y, x_dtype=x_dtype)
    ref = _fit(ae_type, G, x_dtype, bs, device_data=dd)
    ref2 = _fit(ae_type, G, x_dtype, bs, device_data=dd)
    runs = {"stream_data": _fit(ae_type, G, x_dtype, bs, stream_data=_sd(Y, x_dtype=x_dtype, batch=bs)),
            "packed_data": _fit(ae_type, G, x_dtype, bs, packed_data=_pd(Y, x_dtype=x_dtype))}
    print("\n[train G=%d B=%d %s %s] loss %s" % (G, bs, ae_type, x_dtype, ref[0]["loss"]))
    _check_runs(ref, ref2, runs, False, *((1e-4, 2e-2) if bs >= 4096 else (1e-2, 1e-1)))


@pytest.mark.parametrize("x_dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("bits", ["sparse", 4, 16])
def test_train_below_256_genes_is_the_resident_bits(bits, x_dtype):
    ae_type, G, N, bs = "zinb-conddisp", 89, 900, 128
    Y = synth_counts(N, G, 7)
    Y[5, 3] = 1e6
    dd = _dd(Y, x_dtype=x_dtype)
    ref = _fit(ae_type, G, x_dtype, bs, device_data=dd)
    runs = {"stream_data": _fit(ae_type, G, x_dtype, bs, stream_data=_sd(Y, x_dtype=x_dtype, batch=bs, bits=bits)),
            "packed_data": _fit(ae_type, G, x_dtype, bs, packed_data=_pd(Y, x_dtype=x_dtype, bits=bits))}
    _check_runs(ref, None, runs, exact=True)


# ------------------------------------------------------------------------------------------------ 3. predict
def _predict_all(net, **data):
    return net._run_predict(None, True, True, True, True, **data)


def _same_outputs(r_a, r_b):
    return all((r_a.get(k) is None and r_b.get(k) is None) or _eq(r_a[k], r_b[k])
               for k in ("mean", "dispersion", "pi", "latent"))


@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "nb", "zinb-shared"])
def test_predict_and_written_files_match_resident(ae_type, tmp_path):
    """Below 256 genes every output and file bit for bit; at 19 999 genes (two predict batches, 4096 + 904) bit for
    bit when the resident path reproduces itself, else within 2e-6 of each output's largest value.  'zinb-shared' runs
    the shape-general path of the extra AE types (its per-cell outputs are written through predict and write, which
    need an AnnData: no files here)."""
    for G, N, exact in ((89, 5000, True), (19999, 5000, False)):
        Y = synth_counts(N, G, 11)
        dd = _dd(Y)
        net = _net(ae_type, G, "float32", 32)
        r_d = _predict_all(net, device_data=dd)
        exact = exact or _same_outputs(r_d, _predict_all(net, device_data=dd))
        for kind, make in KINDS.items():
            ds = make(Y)
            r = _predict_all(net, **{kind: ds})
            for k in ("mean", "dispersion", "pi", "latent"):
                if r_d.get(k) is None:
                    assert r.get(k) is None, (G, kind, k)
                    continue
                assert r[k].shape == r_d[k].shape, (G, kind, k)
                if exact:
                    assert _eq(r[k], r_d[k]), (G, kind, k)
                else:
                    a, b = _np(r_d[k]), _np(r[k])
                    assert np.max(np.abs(a - b)) <= 2e-6 * np.max(np.abs(a)), (G, kind, k)
            if G < 256 and ae_type != "zinb-shared":
                rownames, colnames = ["c%d" % i for i in range(N)], ["g%d" % i for i in range(G)]
                d_dir, k_dir = tmp_path / ("d%d" % G), tmp_path / ("%s%d" % (kind, G))
                net.write_predictions(str(d_dir), rownames, colnames, device_data=dd)
                net.write_predictions(str(k_dir), rownames, colnames, **{kind: ds})
                files = sorted(p.name for p in d_dir.iterdir())
                assert files == sorted(p.name for p in k_dir.iterdir()) and "mean.tsv" in files
                for f in files:
                    assert (d_dir / f).read_bytes() == (k_dir / f).read_bytes(), (kind, f)
        net.engine.close()


# ------------------------------------------------------------------------------------------------ 4. pad isolation
def _plant(packed, bits, G, value):
    """Set pad gene G (the first pad column) of every row of a dense-width packed matrix (uint8 [rows, bytes])."""
    if bits == 4:
        byte = packed[:, G // 2]
        packed[:, G // 2] = (byte & 0x0F) | (value << 4) if G % 2 else (byte & 0xF0) | value
    elif bits == 8:
        packed[:, G] = value
    else:
        packed.view(np.uint16)[:, G] = value


@pytest.mark.parametrize("bits", [4, 8, 16])
def test_counts_in_pad_genes_change_no_bit(bits):
    """Counts planted in a pad gene of every stored row (streamed and packed): the same training, validation and
    predict bits as the clean rows."""
    from dca_b200.train import train
    G, N, bs = 89, 900, 128
    Y = synth_counts(N, G, 9)
    results = {}
    for kind, make in KINDS.items():
        for planted in (False, True):
            ds = make(Y, bits=bits) if kind == "packed_data" else make(Y, bits=bits, batch=bs)
            if planted:
                if kind == "packed_data":
                    host = ds.packed.cpu().numpy().reshape(ds.n, -1)
                    _plant(host, bits, G, 9)
                    ds.packed.copy_(torch.from_numpy(host.reshape(-1)))
                else:
                    _plant(ds.pc.packed.view(np.uint8), bits, G, 9)
                    ds.pc._pinned = None                 # pin the planted bytes
            net = _net("zinb-conddisp", G, "float32", bs)
            np.random.seed(3)
            hist = train(None, net, epochs=2, batch_size=bs, validation_split=0.1, verbose=False, shuffle=False,
                         **{kind: ds}).history
            out = _predict_all(net, **{kind: ds})
            results[(kind, planted)] = (hist, net.engine.get_weights(), out)
            net.engine.close()
        clean, dirty = results[(kind, False)], results[(kind, True)]
        assert _same_run(clean[:2], dirty[:2]), kind
        assert _same_outputs(clean[2], dirty[2]), kind


# ------------------------------------------------------------------------------------------------ 5. ABI
def test_descriptor_of_the_wrong_width_is_refused():
    from dca_b200 import _lib
    from dca_b200 import io
    G = 89
    Y = synth_counts(200, G, 4)
    pdd = _pd(Y)
    net = _net("zinb-conddisp", G, "float32", 64)
    eng = net.engine
    pdd._bind(eng)
    lib = _lib.load()
    rows = pdd.rows[:64]
    assert lib.dca_packed_train_step(eng.handle, C.byref(pdd.desc), rows.data_ptr(), 64, eng._stream()) == 0
    for genes in (88, 89, 104):
        bad = _lib.PackedCountsDesc.from_buffer_copy(pdd.desc)
        bad.genes = genes
        for fn in ("dca_packed_train_step", "dca_packed_eval_step"):
            assert getattr(lib, fn)(eng.handle, C.byref(bad), rows.data_ptr(), 64, eng._stream()) != 0, (fn, genes)
        assert lib.dca_packed_predict(eng.handle, C.byref(bad), rows.data_ptr(), 64, None, None, None, G, None,
                                      eng._stream()) != 0, genes
        assert b"genes" in lib.dca_last_error(), genes
    torch.cuda.synchronize()
    pc = io.pack_rows(Y, 4, pad_genes=True)
    with pytest.raises(ValueError, match="genes"):
        eng.stream_begin(io.pack_rows(np.zeros((10, 96), np.float32), 4), None, 64)
    # the host stream of a ragged engine needs the exact transform; the float one is refused with an error
    eng.set_input_transform(None, None)
    with pytest.raises((ValueError, _lib.DcaError), match="exact transform"):
        eng.stream_begin(pc, None, 64)
    eng.close()


# ------------------------------------------------------------------------------------------------ 6. CLI
def test_cli_packed_and_stream_write_the_device_files(tmp_path, monkeypatch):
    """A gene x cell TSV with five all-zero genes: the CLI's gene filter leaves 99 genes.  Shuffling is switched off
    (np.random.shuffle / permutation keep the order), so the streamed epoch visits the resident batches in the
    resident order; the files are then byte-identical."""
    from dca_b200.__main__ import main
    G0, N = 104, 300
    Y = synth_counts(N, G0, 17).astype(int)
    Y[:, [3, 40, 41, 77, 100]] = 0
    genes = ["g%d" % i for i in range(G0)]
    df = pd.DataFrame(Y.T, index=genes, columns=["c%d" % i for i in range(N)])
    inp = tmp_path / "counts.tsv"
    df.to_csv(inp, sep="\t")
    monkeypatch.setattr(np.random, "shuffle", lambda a: None)
    monkeypatch.setattr(np.random, "permutation", lambda n: np.arange(n) if np.isscalar(n) else np.asarray(n).copy())
    outs = {}
    for name, extra in (("device", []), ("packed", ["--packed"]), ("stream", ["--stream"])):
        out = tmp_path / name
        main([str(inp), str(out), "--type", "zinb-conddisp", "-e", "2", "-b", "64", "--preprocess", "device"] + extra)
        outs[name] = out
    assert pd.read_csv(outs["device"] / "mean.tsv", sep="\t", index_col=0).shape == (99, N)
    for name in ("packed", "stream"):
        for f in ("mean.tsv", "dispersion.tsv", "dropout.tsv", "latent.tsv"):
            assert (outs["device"] / f).read_bytes() == (outs[name] / f).read_bytes(), (name, f)
