"""GPU reader of Cell Ranger matrix directories (io.read_counts_10x, csrc/read_mtx.cu with a feature map) against the
host statement io._read_10x_scipy: the same CSR arrays in dtype and bytes, the same names and var columns, for the v2
and v3 layouts, gzip and plain, both orientations, non-expression rows dropped inside the parse, across chunks; the
map entry points with no map against the plain readers; and the CLI from a directory against a TSV of the same counts
with the same labels."""
import gzip
import os

import numpy as np
import pandas as pd
import pytest
import scipy.io
import scipy.sparse as sp

from dca_b200 import io

pytestmark = pytest.mark.gpu


def assert_same_csr(a, b):
    assert a.shape == b.shape and a.format == b.format == "csr"
    for f in ("indptr", "indices", "data"):
        x, y = getattr(a, f), getattr(b, f)
        assert x.dtype == y.dtype, (f, x.dtype, y.dtype)
        assert x.tobytes() == y.tobytes(), f


def assert_same(ad, ref, transpose):
    assert_same_csr(ad.X, ref.X)
    pd.testing.assert_index_equal(ad.obs_names, ref.obs_names)
    pd.testing.assert_index_equal(ad.var_names, ref.var_names)
    genes, ref_genes = (ad.var, ref.var) if transpose else (ad.obs, ref.obs)
    ref_genes = ref_genes[[c for c in ref_genes.columns if c != "dca_split"]]
    pd.testing.assert_frame_equal(genes[[c for c in genes.columns if c != "dca_split"]], ref_genes)


def feature_rows(n_gex, n_peaks, n_ab=0, seed=0):
    """Interleaved features (id, symbol, type): gene blocks between larger peak blocks, a few antibody rows, and
    duplicate symbols.  Returns the rows and the boolean mask of gene rows."""
    rng = np.random.default_rng(seed)
    kinds = np.array(["Gene Expression"] * n_gex + ["Peaks"] * n_peaks + ["Antibody Capture"] * n_ab)
    # blocks of about 10 genes / 25 peaks in file order
    order = np.argsort(np.concatenate([np.arange(n_gex) * 2.5, rng.uniform(0, n_gex * 2.5, n_peaks),
                                       rng.uniform(0, n_gex * 2.5, n_ab)]), kind="stable")
    kinds = kinds[order]
    rows, g = [], 0
    for k, t in enumerate(kinds):
        if t == "Gene Expression":
            sym = "Gene%d" % g if g % 7 else "Dup"              # every 7th gene symbol is "Dup"
            rows.append(("ENSG%05d" % g, sym, t))
            g += 1
        elif t == "Peaks":
            rows.append(("chr1:%d-%d" % (100 * k, 100 * k + 50), "chr1:%d-%d" % (100 * k, 100 * k + 50), t))
        else:
            rows.append(("AB%d" % k, "CD%d" % k, t))
    return rows, kinds == "Gene Expression"


def counts(features, cells, seed=1, density=0.1):
    rng = np.random.default_rng(seed)
    M = (rng.poisson(3.0, (features, cells)) + 1) * (rng.random((features, cells)) < density)
    return sp.csr_matrix(M.astype(np.int64))


def make_dir(path, M, features, gz, legacy=False, cell_major=True, prefix=""):
    """M: features x cells.  cell_major: entries ordered by cell (Cell Ranger's layout, CSR order of the transposed
    output); otherwise by feature."""
    os.makedirs(path)
    sfx = ".gz" if gz else ""

    def put(name, data):
        with open(os.path.join(path, prefix + name + sfx), "wb") as f:
            f.write(gzip.compress(data, 6) if gz else data)
    tmp = os.path.join(path, "tmp.mtx")
    scipy.io.mmwrite(tmp, sp.csc_matrix(M) if cell_major else sp.csr_matrix(M), field="integer")
    with open(tmp, "rb") as f:
        put("matrix.mtx", f.read())
    os.remove(tmp)
    cols = 2 if legacy else 3
    put("genes.tsv" if legacy else "features.tsv", "".join("\t".join(r[:cols]) + "\n" for r in features).encode())
    put("barcodes.tsv", "".join("%s-1\n" % bc for bc in barcodes(M.shape[1])).encode())
    return path


def barcodes(n):
    rng = np.random.default_rng(n)
    return ["".join(s) for s in rng.choice(list("ACGT"), (n, 16))]


def no_scipy(monkeypatch):
    def f(*a, **k):
        raise AssertionError("the scipy reader was used")
    monkeypatch.setattr(io, "_read_10x_scipy", f)


@pytest.mark.parametrize("legacy", [False, True], ids=["v3", "v2"])
@pytest.mark.parametrize("gz", [True, False], ids=["gz", "plain"])
@pytest.mark.parametrize("transpose", [True, False])
def test_same_as_scipy(tmp_path, monkeypatch, legacy, gz, transpose):
    features, _ = feature_rows(40, 0 if legacy else 90, 0 if legacy else 5)
    M = counts(len(features), 70)
    d = make_dir(str(tmp_path / "d"), M, features, gz, legacy, cell_major=transpose)
    ref = io._read_10x_scipy(d, transpose)
    no_scipy(monkeypatch)
    assert_same(io.read_counts_10x(d, transpose), ref, transpose)
    assert_same(io.read_dataset(d, transpose=transpose), ref, transpose)


@pytest.mark.parametrize("chunk_bytes", [0, 4096, 65536])
@pytest.mark.parametrize("transpose", [True, False])
def test_peaks_outnumber_genes(tmp_path, transpose, chunk_bytes):
    """A multiome-like directory: 300 gene rows among 1400 peak rows and 20 antibody rows, read in chunks whose
    boundaries fall inside peak blocks, so whole chunks and groups hold no kept entry."""
    features, keep = feature_rows(300, 1400, 20, seed=3)
    M = counts(len(features), 400, seed=4, density=0.05)
    d = make_dir(str(tmp_path / "d"), M, features, True, cell_major=transpose)
    ref = io._read_10x_scipy(d, transpose)
    assert ref.X.shape == ((400, 300) if transpose else (300, 400))
    assert 0 < ref.X.nnz < M.nnz
    assert_same(io.read_counts_10x(d, transpose, chunk_bytes=chunk_bytes), ref, transpose)


def test_only_peaks_in_a_run_of_chunks(tmp_path):
    """All gene rows at the end of the file's row order and cells whose entries are peaks only: chunks with no kept
    entry at all carry the slot and the last key unchanged."""
    features = [("chr1:%d" % k, "chr1:%d" % k, "Peaks") for k in range(500)] + \
               [("ENSG%d" % k, "G%d" % k, "Gene Expression") for k in range(12)]
    M = counts(len(features), 200, seed=5, density=0.08).toarray()
    M[500:, 40:120] = 0                                          # 80 cells with peak entries only
    M[500:, 199] = 0                                             # and the last cell
    d = make_dir(str(tmp_path / "d"), sp.csr_matrix(M), features, False)
    ref = io._read_10x_scipy(d, True)
    assert_same(io.read_counts_10x(d, True, chunk_bytes=2048), ref, True)


@pytest.mark.parametrize("transpose", [True, False])
def test_explicit_zeros(tmp_path, transpose):
    features, _ = feature_rows(30, 50, 3, seed=6)
    M = counts(len(features), 40, seed=7, density=0.3)
    M.data[::4] = 0                                              # stored zeros stay stored
    d = make_dir(str(tmp_path / "d"), M, features, True, cell_major=transpose)
    ref = io._read_10x_scipy(d, transpose)
    assert (ref.X.data == 0).any()
    assert_same(io.read_counts_10x(d, transpose, chunk_bytes=4096), ref, transpose)


@pytest.mark.parametrize("gz", [True, False], ids=["gz", "plain"])
def test_gene_expression_only(tmp_path, gz):
    """Every feature kept: the map path gives the bytes of the plain Matrix Market readers on the same file."""
    features = [("ENSG%d" % k, "G%d" % (k % 50), "Gene Expression") for k in range(80)]
    M = counts(80, 90, seed=8)
    d = make_dir(str(tmp_path / "d"), M, features, gz)
    m = os.path.join(d, "matrix.mtx" + (".gz" if gz else ""))
    plain = io.read_counts_gzip(m, True) if gz else io.read_counts_mtx(m, True)
    ad = io.read_counts_10x(d, True)
    assert_same_csr(ad.X, plain.X)
    assert_same(ad, io._read_10x_scipy(d, True), True)


@pytest.mark.parametrize("gz", [True, False], ids=["gz", "plain"])
@pytest.mark.parametrize("transpose", [True, False])
def test_map_entry_points_without_map(tmp_path, gz, transpose):
    """dca_read_mtx_counts_map / _gz_map with a NULL map, and with the identity map, give the bytes of
    dca_read_mtx_counts / _gz."""
    M = counts(60, 50, seed=9, density=0.2)
    p = str(tmp_path / "m.mtx")
    scipy.io.mmwrite(p, sp.csc_matrix(M) if transpose else sp.csr_matrix(M), field="integer")
    if gz:
        with open(p, "rb") as f:
            data = f.read()
        p += ".gz"
        with open(p, "wb") as f:
            f.write(gzip.compress(data))
    base = "dca_read_mtx_counts_gz" if gz else "dca_read_mtx_counts"
    want = io._read_mtx_gpu(p, transpose, 4096, None, base)
    for fmap in (None, np.arange(60, dtype=np.int32)):
        got = io._read_mtx_gpu(p, transpose, 4096, None, base + "_map", fmap)
        assert_same_csr(got.X, want.X)


def test_bad_map_is_an_error(tmp_path):
    M = counts(6, 5, seed=10, density=0.5)
    p = str(tmp_path / "m.mtx")
    scipy.io.mmwrite(p, sp.csc_matrix(M), field="integer")
    from dca_b200._lib import DcaError
    for fmap in (np.array([0, 1, 2], np.int32), np.array([0, 2, -1, 1, 3, 4], np.int32)):
        with pytest.raises((ValueError, DcaError), match="feature_map"):
            io._read_mtx_gpu(p, True, 0, None, "dca_read_mtx_counts_map", fmap)


def test_declined_falls_back(tmp_path):
    """Cell Ranger's cell-major file read without transpose is not in CSR order of the output: the GPU reader declines
    it and read_dataset gives the host statement's result."""
    features, _ = feature_rows(25, 40, 2, seed=11)
    M = counts(len(features), 30, seed=12, density=0.3)
    d = make_dir(str(tmp_path / "d"), M, features, True, cell_major=True)
    assert io.read_counts_10x(d, False) is None
    assert_same(io.read_dataset(d, transpose=False), io._read_10x_scipy(d, False), False)


# ------------------------------------------------------------------------------------------------------------- CLI
N_CELLS, N_GENES = 300, 64


@pytest.fixture(scope="module")
def cli_inputs(tmp_path_factory):
    """A v3 gzipped directory of 300 cells, 64 gene rows among 150 peak and 6 antibody rows, and a TSV of its gene
    counts (genes x cells) labelled with the reader's unique symbols and the barcodes."""
    from tests.util import synth_counts
    tmp = tmp_path_factory.mktemp("cli")
    features, keep = feature_rows(N_GENES, 150, 6, seed=13)
    Y = synth_counts(N_CELLS, N_GENES, 14).astype(np.int64)       # cells x genes
    M = counts(len(features), N_CELLS, seed=15, density=0.05).toarray()
    M[keep] = Y.T
    d = make_dir(str(tmp / "dir"), sp.csr_matrix(M), features, True, prefix="GSM9_")
    ref = io._read_10x_scipy(d, True)
    symbols, cells = list(ref.var_names), list(ref.obs_names)
    assert "Dup-1" in symbols
    tsv = tmp / "counts.tsv"
    tsv.write_text("\t" + "\t".join(cells) + "\n" +
                   "".join("%s\t%s\n" % (symbols[g], "\t".join(str(v) for v in Y[:, g])) for g in range(N_GENES)))
    subset = tmp / "subset.txt"
    subset.write_text("\n".join(["Gene1", "Dup", "Dup-1", "Gene20", "Gene40"]) + "\n")
    return d, str(tsv), str(subset), symbols, cells


def run_pair(tmp_path, cli_inputs, monkeypatch, extra, name):
    from dca_b200.__main__ import main
    d, tsv, subset, _, _ = cli_inputs
    extra = [subset if a == "SUBSET" else a for a in extra]
    args = ["--type", "zinb-conddisp", "-e", "2", "-b", "64"] + extra
    main([tsv, str(tmp_path / (name + "_tsv"))] + args)
    with monkeypatch.context() as m:
        no_scipy(m)
        main([d, str(tmp_path / (name + "_dir"))] + args)
    out_tsv, out_dir = tmp_path / (name + "_tsv"), tmp_path / (name + "_dir")
    files = sorted(f for f in os.listdir(out_tsv) if f.endswith(".tsv"))
    assert "mean.tsv" in files and "latent.tsv" in files
    for f in files:
        assert (out_dir / f).read_bytes() == (out_tsv / f).read_bytes(), f
    return out_dir


@pytest.mark.parametrize("mode", ["device", "packed", "stream"])
def test_cli_directory_against_tsv(tmp_path, cli_inputs, monkeypatch, mode):
    extra = ["--preprocess", "device"] + {"device": [], "packed": ["--packed"], "stream": ["--stream"]}[mode]
    out = run_pair(tmp_path, cli_inputs, monkeypatch, extra, mode)
    _, _, _, symbols, cells = cli_inputs
    mean = pd.read_csv(out / "mean.tsv", sep="\t", index_col=0)
    assert list(mean.columns) == cells
    assert set(mean.index) <= set(symbols) and mean.index.is_unique and len(mean.index) > N_GENES // 2


@pytest.mark.parametrize("preprocess", ["host", "device"])
def test_cli_denoisesubset_symbols(tmp_path, cli_inputs, monkeypatch, preprocess):
    out = run_pair(tmp_path, cli_inputs, monkeypatch, ["--preprocess", preprocess, "--denoisesubset", "SUBSET"],
                   preprocess)
    mean = pd.read_csv(out / "mean.tsv", sep="\t", index_col=0)
    assert sorted(mean.index) == sorted(["Gene1", "Dup", "Dup-1", "Gene20", "Gene40"])


@pytest.mark.parametrize("flag", ["--packed", "--stream"])
def test_cli_denoisesubset_rejected(tmp_path, cli_inputs, flag):
    from dca_b200.__main__ import main
    d, _, subset, _, _ = cli_inputs
    with pytest.raises(Exception, match="denoisesubset"):
        main([d, str(tmp_path / "out"), "-e", "1", "--preprocess", "device", flag, "--denoisesubset", subset])
