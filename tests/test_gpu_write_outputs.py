"""The GPU writer of the '%.6f' TSV files (io.write_text_matrix_device, csrc/write_text.cu) and the gene-block output
path built on it (Autoencoder.write_predictions): the same bytes as Python's '%.6f', as io.write_text_matrix, and as
predict + write, from every input source and in every CLI mode; host memory that does not grow with the cell count."""
import os
import tracemalloc

import numpy as np
import pandas as pd
import pytest
import torch

from tests.util import synth_counts

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _ref6(values):
    return ["" if v != v else "%.6f" % v for v in np.asarray(values, dtype=np.float32).astype(np.float64).tolist()]


def _device_text(bits, tmp_path, cols=1024):
    """The file write_text_matrix_device writes for the float32 bit patterns `bits` (rows of `cols` values)."""
    from dca_b200.io import write_text_matrix_device
    t = torch.from_numpy(bits.view(np.float32).reshape(-1, cols).copy()).to(DEV)
    path = str(tmp_path / "fmt.tsv")
    write_text_matrix_device(t, path)
    with open(path, "rb") as f:
        return f.read()


def _expected_text(bits, cols=1024):
    f = _ref6(bits.view(np.float32))
    return "".join("\t".join(f[i:i + cols]) + "\n" for i in range(0, len(f), cols)).encode()


# ------------------------------------------------------------------------------------------------ number format
def _formatter_cases():
    rng = np.random.default_rng(0)
    e = np.arange(256, dtype=np.uint32) << 23
    parts = [rng.integers(0, 2 ** 32, 2 ** 23, dtype=np.uint64).astype(np.uint32)]
    for m in (0, 1, 2, 2 ** 23 - 1):
        parts += [e | m, e | m | 0x80000000]
    per_exp = (2 ** 24 - sum(p.size for p in parts)) // 512
    parts.append((e[:, None] | rng.integers(0, 2 ** 23, (256, per_exp), dtype=np.uint32)).ravel())
    parts.append((e[:, None] | 0x80000000 | rng.integers(0, 2 ** 23, (256, per_exp), dtype=np.uint32)).ravel())
    bits = np.concatenate(parts)
    pad = (-bits.size) % 1024
    return np.concatenate([bits, rng.integers(0, 2 ** 32, pad, dtype=np.uint64).astype(np.uint32)])


def test_format_2_24_patterns(tmp_path):
    bits = _formatter_cases()
    assert bits.size >= 2 ** 24
    step = 2 ** 20
    for s in range(0, bits.size, step):
        b = bits[s:s + step]
        assert _device_text(b, tmp_path) == _expected_text(b), s


def test_format_ties_boundaries_and_extremes(tmp_path):
    j = np.arange(1, 64)
    k = np.arange(1, 2 ** 12)
    ties = (k[None, :].astype(np.float64) / 2.0 ** j[:, None]).astype(np.float32)       # exact k / 2^j
    ties = ties[ties.astype(np.float64) * 2.0 ** j[:, None] == k[None, :]]
    bnd = ((np.arange(0, 2 ** 20) + 0.5) / 1e6).astype(np.float32)                       # ...5 boundaries and neighbours
    big = np.float32(8e9) * (1 + np.arange(-2000, 2000, dtype=np.float32) * np.float32(1e-7))
    fmax = np.finfo(np.float32).max
    special = np.array([0.0078125, -0.0078125, 5e-7, -5e-7, 1.5e-6, 2.5e-6, 0.0, -0.0, -1e-7, -4.9e-7, -1e-30, 1e-45,
                        -1e-45, 1.17549435e-38, fmax, -fmax, 2.0 ** 64, 2.0 ** 100, np.nan, -np.nan, np.inf, -np.inf],
                       dtype=np.float32)
    denorm = np.arange(1, 2 ** 16, dtype=np.uint32).view(np.float32)
    v = np.concatenate([ties, -ties, bnd, np.nextafter(bnd, np.float32(np.inf)), np.nextafter(bnd, np.float32(-np.inf)),
                        -bnd, big, np.geomspace(1e9, fmax, 50000).astype(np.float32), special, denorm, -denorm])
    bits = v.astype(np.float32).view(np.uint32)
    bits = np.concatenate([bits, np.zeros((-bits.size) % 1024, np.uint32)])
    assert _device_text(bits, tmp_path) == _expected_text(bits)


# ------------------------------------------------------------------------------------------------ matrix writer
_ODD = ["plain", "tab\there", 'quo"te', "new\nline", "cr\rx", "", "ünï"]


def _names(prefix, n):
    return [_ODD[i] if i < len(_ODD) else "%s%d" % (prefix, i) for i in range(n)]


@pytest.mark.parametrize("shape", [(1, 1), (1, 300), (300, 1), (37, 300), (513, 7)])
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("labels", ["none", "rows", "cols", "both"])
def test_matrix_writer_matches_host(tmp_path, shape, transpose, labels):
    from dca_b200.io import write_text_matrix, write_text_matrix_device
    rng = np.random.default_rng(shape[0] * 1000 + shape[1])
    m = (rng.standard_normal(shape) * 10.0 ** rng.integers(-8, 9, shape)).astype(np.float32)
    m.ravel()[:: 17] = np.nan
    rn = _names("r", shape[0]) if labels in ("rows", "both") else None
    cn = _names("c", shape[1]) if labels in ("cols", "both") else None
    a, b = str(tmp_path / "host.tsv"), str(tmp_path / "dev.tsv")
    write_text_matrix(m, a, rownames=rn, colnames=cn, transpose=transpose)
    write_text_matrix_device(torch.from_numpy(m).to(DEV), b, rownames=rn, colnames=cn, transpose=transpose)
    assert open(a, "rb").read() == open(b, "rb").read()


@pytest.mark.parametrize("transpose", [False, True])
def test_matrix_writer_many_chunks_and_strided(tmp_path, transpose):
    from dca_b200.io import write_text_matrix, write_text_matrix_device
    rng = np.random.default_rng(5)
    full = rng.standard_normal((700, 900)).astype(np.float32)
    view = torch.from_numpy(full).to(DEV)[:, 100:800]                     # leading dimension 900
    m = full[:, 100:800]
    rn, cn = _names("r", 700), _names("c", 700)
    a, b = str(tmp_path / "host.tsv"), str(tmp_path / "dev.tsv")
    write_text_matrix(m, a, rownames=rn, colnames=cn, transpose=transpose)
    info = np.zeros(4, dtype=np.int64)
    write_text_matrix_device(view, b, rownames=rn, colnames=cn, transpose=transpose, chunk_bytes=10000, info=info)
    data = open(a, "rb").read()
    assert open(b, "rb").read() == data
    assert info[0] == len(data) and info[1] > 10 and len(data) > 50 * 10000


def test_matrix_writer_append_blocks(tmp_path):
    from dca_b200.io import write_text_matrix, write_text_matrix_device
    m = np.random.default_rng(6).standard_normal((50, 40)).astype(np.float32)
    rn, cn = _names("r", 50), _names("c", 40)
    a, b = str(tmp_path / "host.tsv"), str(tmp_path / "dev.tsv")
    write_text_matrix(m, a, rownames=rn, colnames=cn, transpose=True)
    t = torch.from_numpy(m).to(DEV)
    for g0 in range(0, 40, 13):
        write_text_matrix_device(t[:, g0:g0 + 13], b, rownames=rn if g0 == 0 else None, colnames=cn[g0:g0 + 13],
                                 transpose=True, append=g0 > 0)
    assert open(a, "rb").read() == open(b, "rb").read()


# ------------------------------------------------------------------------------------------------ predictions
N_CELLS, N_GENES = 5000, 512                               # two predict batches: 4096 + 904


@pytest.fixture(scope="module")
def counts():
    return synth_counts(N_CELLS, N_GENES, 21)


@pytest.fixture(scope="module")
def cell_names():
    return _names("cell", N_CELLS)


@pytest.fixture(scope="module")
def gene_names():
    return _names("gene", N_GENES)


def _net(ae_type, n_out=N_GENES, gemm_path="auto"):
    from dca_b200.network import AE_types
    net = AE_types[ae_type](input_size=N_GENES, output_size=n_out, hidden_size=(64, 32, 64), gemm_path=gemm_path)
    net.build(max_batch=256, seed=4)
    return net


def _source(kind, Y):
    from dca_b200.anndata_lite import AnnData
    from dca_b200 import io
    if kind == "host":
        return {}, io.normalize(AnnData(Y.copy()), filter_min_counts=False)
    if kind == "device":
        from dca_b200.device_data import DeviceDataset
        return {"device_data": DeviceDataset.from_counts(Y, DEV)}, None
    if kind == "stream":
        from dca_b200.stream_data import StreamedDataset
        return {"stream_data": StreamedDataset.from_counts(Y, DEV)}, None
    from dca_b200.packed_data import PackedDeviceDataset
    return {"packed_data": PackedDeviceDataset.from_counts(Y, DEV)}, None


def _reference_files(net, out, adata, src, cells, genes, mode="full", return_info=True):
    """The files of predict + write for the source."""
    from dca_b200.anndata_lite import AnnData
    if adata is None:
        adata = AnnData(np.zeros((N_CELLS, len(genes)), np.float32), obs=pd.DataFrame(index=cells),
                        var=pd.DataFrame(index=genes))
    else:
        adata = adata.copy()
        adata.obs.index = pd.Index(cells)
    net.predict(adata, mode=mode, return_info=return_info, **src)
    net.write(adata, str(out), mode=mode, colnames=genes)


def _same_files(a, b):
    fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
    assert fa == fb
    for f in fa:
        assert open(os.path.join(a, f), "rb").read() == open(os.path.join(b, f), "rb").read(), f
    return fa


def _heads(net):
    return 1 + (net.ae_type not in ("nb", "zinb")) + bool(net.has_pi)


@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "nb-conddisp", "nb"])
@pytest.mark.parametrize("kind", ["host", "device", "stream", "packed"])
@pytest.mark.parametrize("blocks", ["one", "many"])
def test_write_predictions_matches_predict_write(tmp_path, counts, cell_names, gene_names, ae_type, kind, blocks):
    net = _net(ae_type)
    src, adata = _source(kind, counts)
    _reference_files(net, tmp_path / "ref", adata, src, cell_names, gene_names)
    cap = None if blocks == "one" else 70 * 4 * N_CELLS * _heads(net)          # 70 genes: 8 blocks, the last of 22
    net.write_predictions(str(tmp_path / "new"), cell_names, gene_names, mode="full", return_info=True, adata=adata,
                          max_block_bytes=cap, chunk_bytes=1 << 20, **src)
    files = _same_files(tmp_path / "ref", tmp_path / "new")
    assert {"mean.tsv", "latent.tsv", "dispersion.tsv"} <= set(files)


@pytest.mark.parametrize("mode", ["denoise", "latent"])
def test_write_predictions_modes(tmp_path, counts, cell_names, gene_names, mode):
    net = _net("zinb-conddisp")
    src, adata = _source("host", counts)
    _reference_files(net, tmp_path / "ref", adata, src, cell_names, gene_names, mode=mode, return_info=False)
    net.write_predictions(str(tmp_path / "new"), cell_names, gene_names, mode=mode, return_info=False,
                          adata=adata, max_block_bytes=100 * 4 * N_CELLS, **src)
    _same_files(tmp_path / "ref", tmp_path / "new")


def test_write_predictions_output_subset(tmp_path, counts, cell_names, gene_names):
    sub = [3, 17, 100, 101, 250, 511, 64, 0, 9, 300, 301, 302, 77]
    net = _net("zinb-conddisp", n_out=len(sub))
    src, adata = _source("device", counts)
    names = [gene_names[i] for i in sub]
    _reference_files(net, tmp_path / "ref", adata, src, cell_names, names)
    net.write_predictions(str(tmp_path / "new"), cell_names, names, max_block_bytes=4 * 4 * N_CELLS * 3, **src)
    _same_files(tmp_path / "ref", tmp_path / "new")


def _read(path, header):
    return pd.read_csv(path, sep="\t", index_col=0, header=0 if header else None, keep_default_na=False,
                       na_values=[""], quoting=0)


@pytest.mark.parametrize("ae_type,gemm_path,return_info", [("nb-conddisp", "generic", True),
                                                            ("zinb-shared", "auto", False)])
def test_write_predictions_not_reproducible_paths(tmp_path, counts, ae_type, gemm_path, return_info):
    """Split-K atomics differ run to run in the last bits: the files are held to the rule of
    test_gpu_packed.test_predict_matches_resident."""
    cell_names, gene_names = ["c%d" % i for i in range(N_CELLS)], ["g%d" % i for i in range(N_GENES)]
    net = _net(ae_type, gemm_path=gemm_path)
    src, adata = _source("device", counts)
    _reference_files(net, tmp_path / "ref", adata, src, cell_names, gene_names, return_info=return_info)
    net.write_predictions(str(tmp_path / "new"), cell_names, gene_names, return_info=return_info,
                          max_block_bytes=70 * 4 * N_CELLS * 3, **src)
    files = sorted(os.listdir(tmp_path / "ref"))
    assert files == sorted(os.listdir(tmp_path / "new"))
    for f in files:
        a, b = _read(tmp_path / "ref" / f, f == "mean.tsv"), _read(tmp_path / "new" / f, f == "mean.tsv")
        assert list(a.index) == list(b.index) and list(a.columns) == list(b.columns), f
        x, y = a.to_numpy(np.float64), b.to_numpy(np.float64)
        assert x.shape == y.shape and np.max(np.abs(x - y)) <= 2e-6 * np.max(np.abs(x)) + 1e-6, f


def test_write_predictions_shared_keeps_predict_write(tmp_path, counts, cell_names, gene_names):
    """nb-shared's per-cell dispersion is not cells x genes: predict + write run as before, their error included."""
    net = _net("nb-shared")
    src, adata = _source("host", counts)
    with pytest.raises(ValueError, match="labels"):
        _reference_files(net, tmp_path / "ref", adata, src, cell_names, gene_names)
    with pytest.raises(ValueError, match="labels"):
        net.write_predictions(str(tmp_path / "new"), cell_names, gene_names, adata=adata.copy())


# ------------------------------------------------------------------------------------------------ CLI
@pytest.mark.parametrize("mode", [["--preprocess", "host"], ["--preprocess", "device"],
                                  ["--preprocess", "device", "--stream"], ["--preprocess", "device", "--packed"]])
def test_cli_outputs_match_predict_write(tmp_path, monkeypatch, mode):
    from dca_b200.__main__ import main
    from dca_b200.network import Autoencoder
    Y = synth_counts(600, 96, 23).astype(int)
    genes = _names("g", 96)
    genes[2] = "gene two"
    df = pd.DataFrame(Y.T, index=genes, columns=["c%d" % i for i in range(600)])
    inp = tmp_path / "counts.tsv"
    df.to_csv(inp, sep="\t")
    orig = Autoencoder.write_predictions
    ref = tmp_path / "ref"

    def both(self, file_path, rownames, colnames, mode='full', return_info=True, device_data=None, stream_data=None,
             packed_data=None, adata=None, **kw):
        orig(self, file_path, rownames, colnames, mode=mode, return_info=return_info, device_data=device_data,
             stream_data=stream_data, packed_data=packed_data, adata=adata, max_block_bytes=4 * 600 * 3 * 20, **kw)
        self.predict(adata, mode=mode, return_info=return_info, device_data=device_data, stream_data=stream_data,
                     packed_data=packed_data)
        self.write(adata, str(ref), mode=mode, colnames=colnames)
    monkeypatch.setattr(Autoencoder, "write_predictions", both)
    out = tmp_path / "out"
    main([str(inp), str(out), "--type", "zinb-conddisp", "-e", "2", "-b", "64"] + mode)
    for f in ("mean.tsv", "latent.tsv", "dispersion.tsv", "dropout.tsv"):
        assert open(out / f, "rb").read() == open(ref / f, "rb").read(), f


# ------------------------------------------------------------------------------------------------ host memory
def test_write_predictions_host_memory_bounded(tmp_path):
    """One 32768 x 2048 float32 output is 256 MB: the traced host peak stays under 1/8 of it."""
    from dca_b200.device_data import DeviceDataset
    from dca_b200.network import AE_types
    n, g = 32768, 2048
    dd = DeviceDataset.from_counts(synth_counts(n, g, 24), DEV)
    net = AE_types["nb"](input_size=g, output_size=g, hidden_size=(64, 32, 64))
    net.build(max_batch=256, seed=1)
    cells, genes = ["c%d" % i for i in range(n)], ["g%d" % i for i in range(g)]
    torch.cuda.synchronize()
    tracemalloc.start()
    try:
        net.write_predictions(str(tmp_path / "out"), cells, genes, mode="full", return_info=True, device_data=dd)
        peak = tracemalloc.get_traced_memory()[1]
    finally:
        tracemalloc.stop()
    assert peak < n * g * 4 // 8, peak
    assert os.path.getsize(tmp_path / "out" / "mean.tsv") > n * g * 8
