"""The host statement of the Cell Ranger directory reader (io._read_10x_scipy) against hand-written expectations:
scanpy's read_10x_mtx(path, var_names='gene_symbols', make_unique=True, gex_only=True) in both orientations, for the
v2 and v3 layouts, GEO prefixes, duplicate symbols, non-expression features and the errors."""
import gzip
import os

import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp

from dca_b200 import io

# 5 features x 3 cells, as the file holds them (genes x cells)
COUNTS = np.array([[1, 0, 2],
                   [0, 7, 0],
                   [4, 0, 0],
                   [0, 3, 5],
                   [6, 0, 1]])
BARCODES = ["AAAC-1", "CCCG-1", "GGGT-1"]


def make_dir(tmp_path, features, counts=COUNTS, barcodes=BARCODES, prefix="", gz=False, legacy=False, name="d"):
    """A Cell Ranger directory: features is a list of tuples, one per row of counts (the tab-separated columns)."""
    d = tmp_path / name
    d.mkdir()
    suffix = ".gz" if gz else ""

    def put(fname, data):
        (d / (prefix + fname + suffix)).write_bytes(gzip.compress(data) if gz else data)
    p = str(tmp_path / "m.mtx")
    scipy.io.mmwrite(p, sp.csc_matrix(np.asarray(counts)), field="integer")
    put("matrix.mtx", open(p, "rb").read())
    os.remove(p)
    put("genes.tsv" if legacy else "features.tsv", "".join("\t".join(f) + "\n" for f in features).encode())
    put("barcodes.tsv", "".join(b + "\n" for b in barcodes).encode())
    return str(d)


def gex(ids, symbols):
    return [(i, s, "Gene Expression") for i, s in zip(ids, symbols)]


IDS = ["ENSG1", "ENSG2", "ENSG3", "ENSG4", "ENSG5"]
SYMBOLS = ["Sox2", "Actb", "Gapdh", "Mt-co1", "Cd4"]


def check(ad, X, obs, var, transpose):
    """X: the expected dense matrix in the output orientation; obs / var the expected names."""
    assert ad.X.format == "csr" and ad.X.dtype == np.float32
    assert ad.X.indptr.dtype == np.int32 and ad.X.indices.dtype == np.int32
    assert np.array_equal(ad.X.toarray(), np.asarray(X, dtype=np.float32))
    assert list(ad.obs_names) == obs and list(ad.var_names) == var


@pytest.mark.parametrize("transpose", [True, False])
def test_v2_plain(tmp_path, transpose):
    d = make_dir(tmp_path, [(i, s) for i, s in zip(IDS, SYMBOLS)], legacy=True)
    ad = io._read_10x_scipy(d, transpose)
    genes = ad.var if transpose else ad.obs
    if transpose:
        check(ad, COUNTS.T, BARCODES, SYMBOLS, True)
    else:
        check(ad, COUNTS, SYMBOLS, BARCODES, False)
    assert list(genes.columns) == ["gene_ids"] and list(genes["gene_ids"]) == IDS


@pytest.mark.parametrize("transpose", [True, False])
def test_v3_gzip(tmp_path, transpose):
    d = make_dir(tmp_path, gex(IDS, SYMBOLS), gz=True)
    assert sorted(os.listdir(d)) == ["barcodes.tsv.gz", "features.tsv.gz", "matrix.mtx.gz"]
    ad = io._read_10x_scipy(d, transpose)
    if transpose:
        check(ad, COUNTS.T, BARCODES, SYMBOLS, True)
    else:
        check(ad, COUNTS, SYMBOLS, BARCODES, False)
    genes = ad.var if transpose else ad.obs
    assert list(genes["gene_ids"]) == IDS and list(genes["feature_types"]) == ["Gene Expression"] * 5


def test_geo_prefix(tmp_path):
    d = make_dir(tmp_path, gex(IDS, SYMBOLS), prefix="GSM123_", gz=True)
    (tmp_path / "d" / "GSM123_README.txt").write_text("not part of the triple\n")
    check(io._read_10x_scipy(d, True), COUNTS.T, BARCODES, SYMBOLS, True)


def test_gzip_by_magic_bytes(tmp_path):
    """A gzip file without the .gz name and a plain file with it read alike."""
    d = make_dir(tmp_path, gex(IDS, SYMBOLS))
    m = os.path.join(d, "matrix.mtx")
    data = open(m, "rb").read()
    os.remove(m)
    open(m + ".gz", "wb").write(data)                            # plain bytes under a .gz name
    b = os.path.join(d, "barcodes.tsv")
    data = open(b, "rb").read()
    open(b, "wb").write(gzip.compress(data))                     # gzip bytes under a plain name
    check(io._read_10x_scipy(d, True), COUNTS.T, BARCODES, SYMBOLS, True)


def test_duplicate_symbols(tmp_path):
    symbols = ["A", "A", "A-1", "B", "A"]
    d = make_dir(tmp_path, gex(IDS, symbols))
    ad = io._read_10x_scipy(d, True)
    check(ad, COUNTS.T, BARCODES, ["A", "A-2", "A-1", "B", "A-3"], True)
    assert list(ad.var["gene_ids"]) == IDS


def test_make_index_unique():
    assert list(io.make_index_unique(["A", "A", "A-1"])) == ["A", "A-2", "A-1"]
    assert list(io.make_index_unique(["x", "y", "x", "x-1", "x", "y"])) == ["x", "y", "x-2", "x-1", "x-3", "y-1"]
    assert list(io.make_index_unique(["p", "q"])) == ["p", "q"]


def test_feature_filter(tmp_path):
    """Antibody-capture and peak rows interleaved with gene rows are dropped, after the symbols are made unique over
    all rows (as read_10x_mtx does)."""
    features = [("ENSG1", "A", "Gene Expression"), ("CD3", "A", "Antibody Capture"),
                ("ENSG3", "A", "Gene Expression"), ("chr1:10-20", "chr1:10-20", "Peaks"),
                ("ENSG5", "Cd4", "Gene Expression")]
    d = make_dir(tmp_path, features)
    keep = [0, 2, 4]
    ad = io._read_10x_scipy(d, True)
    check(ad, COUNTS[keep].T, BARCODES, ["A", "A-2", "Cd4"], True)
    assert list(ad.var["gene_ids"]) == ["ENSG1", "ENSG3", "ENSG5"]
    assert list(ad.var["feature_types"]) == ["Gene Expression"] * 3
    ad = io._read_10x_scipy(d, False)
    check(ad, COUNTS[keep], ["A", "A-2", "Cd4"], BARCODES, False)
    assert list(ad.obs["gene_ids"]) == ["ENSG1", "ENSG3", "ENSG5"]


def test_six_column_features(tmp_path):
    """Cell Ranger ARC's features.tsv (id, name, type, chromosome, start, end) is read by its first three columns."""
    features = [(i, s, t, "chr1", str(100 * k), str(100 * k + 50))
                for k, (i, s, t) in enumerate(gex(IDS, SYMBOLS))]
    features[1] = ("chr2:5-9", "chr2:5-9", "Peaks", "chr2", "5", "9")
    d = make_dir(tmp_path, features, gz=True)
    ad = io._read_10x_scipy(d, True)
    keep = [0, 2, 3, 4]
    check(ad, COUNTS[keep].T, BARCODES, [SYMBOLS[k] for k in keep], True)
    assert list(ad.var.columns) == ["gene_ids", "feature_types"]


def test_missing_file(tmp_path):
    d = make_dir(tmp_path, gex(IDS, SYMBOLS))
    os.remove(os.path.join(d, "barcodes.tsv"))
    with pytest.raises(ValueError, match=r"missing barcodes\.tsv\[\.gz\].*matrix\.mtx"):
        io._read_10x_scipy(d, True)
    empty = tmp_path / "empty"
    empty.mkdir()
    with pytest.raises(ValueError, match="not a Cell Ranger matrix directory"):
        io._read_10x_scipy(str(empty), True)


def test_two_triples(tmp_path):
    d = make_dir(tmp_path, gex(IDS, SYMBOLS), prefix="GSM1_")
    for f in ("matrix.mtx", "features.tsv", "barcodes.tsv"):
        os.link(os.path.join(d, "GSM1_" + f), os.path.join(d, "GSM2_" + f))
    with pytest.raises(ValueError, match=r"2 candidate .*GSM1_matrix\.mtx.*GSM2_matrix\.mtx"):
        io._read_10x_scipy(d, True)


def test_label_count_mismatch(tmp_path):
    d = make_dir(tmp_path, gex(IDS, SYMBOLS), barcodes=BARCODES + ["TTTT-1"])
    with pytest.raises(ValueError, match=r"matrix\.mtx is 5 x 3.*features\.tsv lists 5 features.*barcodes\.tsv 4"):
        io._read_10x_scipy(d, True)
    d = make_dir(tmp_path, gex(IDS[:4], SYMBOLS[:4]), name="e")
    with pytest.raises(ValueError, match=r"features\.tsv lists 4 features"):
        io._read_10x_scipy(d, False)


def test_read_dataset_without_gpu(tmp_path, monkeypatch):
    """Without a CUDA device read_dataset takes a directory through the host statement, cells x genes by default in
    the CLI's orientation (transpose=True)."""
    monkeypatch.setattr(io, "_cuda_available", lambda: False)
    d = make_dir(tmp_path, gex(IDS, SYMBOLS))
    ad = io.read_dataset(d, transpose=True)
    check(ad, COUNTS.T, BARCODES, SYMBOLS, True)
    assert list(ad.obs["dca_split"]) == ["train"] * 3
