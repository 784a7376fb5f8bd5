"""GPU reader of Matrix Market count files (io.read_counts_mtx, csrc/read_mtx.cu) against scipy's reader: the same CSR
arrays, in dtype and bytes, in both orientations; scipy's result for every file it does not take; the CLI from a .mtx
file against the same counts as a TSV; and a file past 2^32 bytes against the generator's own arrays.  Files of more
than 2^31 entries are not tested."""
import gzip
import os
import shutil
import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.io
import scipy.sparse as sp
import torch

from dca_b200 import io

pytestmark = pytest.mark.gpu

BANNER = "%%MatrixMarket matrix coordinate {} general"


def scipy_csr(path, transpose):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        X = sp.csr_matrix(scipy.io.mmread(path).astype(np.float32))
    return X.T.tocsr() if transpose else X


def mtx_text(entries, m, n, field="integer", comments=(), eol="\n", final_eol=True, nnz=None):
    """entries: (i, j, value token) with 1-based indices, in file order."""
    lines = [BANNER.format(field)] + ["%" + c for c in comments] + ["%d %d %d" % (m, n, len(entries) if nnz is None else nnz)]
    lines += ["%d %d %s" % e for e in entries]
    return eol.join(lines) + (eol if final_eol else "")


def entries_of(X, transpose):
    """The entries of the cells x genes CSR X in CSR order, as a file read with (transpose) or without must hold them:
    genes x cells (i = gene) with transpose, cells x genes otherwise."""
    coo = X.tocoo()
    r, c, v = coo.row + 1, coo.col + 1, coo.data
    order = np.lexsort((c, r))
    r, c, v = r[order], c[order], v[order]
    return [((cc, rr, str(int(vv))) if transpose else (rr, cc, str(int(vv)))) for rr, cc, vv in zip(r, c, v)]


def write(tmp_path, text, name="m.mtx"):
    p = tmp_path / name
    p.write_bytes(text.encode() if isinstance(text, str) else text)
    return str(p)


def assert_same_csr(a, b):
    assert a.shape == b.shape and a.format == b.format == "csr"
    for f in ("indptr", "indices", "data"):
        x, y = getattr(a, f), getattr(b, f)
        assert x.dtype == y.dtype, (f, x.dtype, y.dtype)
        assert x.tobytes() == y.tobytes(), f


def check(path, transpose, chunk_bytes=0):
    ad = io.read_counts_mtx(path, transpose, chunk_bytes=chunk_bytes)
    assert ad is not None, "the GPU reader did not take %s" % path
    assert_same_csr(ad.X, scipy_csr(path, transpose))
    n, g = ad.X.shape
    assert list(ad.obs_names) == [str(i) for i in range(n)] and list(ad.var_names) == [str(i) for i in range(g)]
    return ad


def check_both(tmp_path, X, **kw):
    """X: cells x genes; the file for transpose (genes x cells, column-major) and the one without (row-major)."""
    m, n = X.shape
    check(write(tmp_path, mtx_text(entries_of(X, False), m, n, **kw), "rows.mtx"), False)
    check(write(tmp_path, mtx_text(entries_of(X, True), n, m, **kw), "cols.mtx"), True)


def counts(n, g, seed=0, density=0.08, lam=3.0):
    rng = np.random.default_rng(seed)
    M = rng.poisson(lam, (n, g)) * (rng.random((n, g)) < density)
    return sp.csr_matrix(M.astype(np.int64))


def test_mmwrite_files(tmp_path):
    X = counts(40, 24, 1)                                        # cells x genes
    p = str(tmp_path / "csc.mtx")
    scipy.io.mmwrite(p, X.T.tocsc(), field="integer")           # genes x cells, column-major: Cell Ranger's layout
    check(p, True)
    p = str(tmp_path / "csr.mtx")
    scipy.io.mmwrite(p, X.astype(np.float64).tocsr(), field="integer")
    check(p, False)


@pytest.mark.parametrize("case", ["one", "single_entry", "empty", "empty_rows", "wide", "tall", "explicit_zeros",
                                  "rounding", "real_field", "comments_crlf_no_final_eol"])
def test_same_arrays_as_scipy(tmp_path, case):
    kw = {}
    if case == "one":
        X = sp.csr_matrix(np.array([[5]]))
    elif case == "single_entry":
        X = sp.csr_matrix(([7], ([3], [4])), shape=(6, 9))
    elif case == "empty":
        X = sp.csr_matrix((5, 3), dtype=np.int64)
    elif case == "empty_rows":
        M = counts(12, 7, 2, density=0.5).toarray()
        M[[0, 1, 5, 6, 10, 11]] = 0                           # leading, inner and trailing empty rows
        X = sp.csr_matrix(M)
    elif case == "wide":
        X = counts(20, 100000, 3, density=0.02)
    elif case == "tall":
        X = counts(50000, 8, 4, density=0.3)
    elif case == "explicit_zeros":
        X = counts(9, 11, 5, density=0.4)
        X.data[::3] = 0                                        # stored zeros stay stored
    elif case == "rounding":
        vals = [2 ** 24 + 1, 2 ** 31, 10 ** 18 - 1, 2 ** 24 + 3, 123456789012345678]
        X = sp.csr_matrix((np.array(vals, dtype=np.int64), ([0, 0, 1, 2, 2], [0, 3, 1, 0, 2])), shape=(3, 4))
    elif case == "real_field":
        X, kw = counts(10, 10, 6, density=0.5, lam=1e6), dict(field="real")
    else:
        X, kw = counts(13, 9, 7, density=0.4), dict(comments=("", " written by a test", "%"), eol="\r\n", final_eol=False)
    check_both(tmp_path, X, **kw)


@pytest.mark.parametrize("where", ["index", "value", "space", "cr_lf", "line_end"])
def test_chunk_boundaries(tmp_path, where):
    X = counts(12, 30, 8, density=0.5, lam=500)
    data = mtx_text(entries_of(X, True), 30, 12, eol="\r\n").encode()
    head = data.index(b"\n", data.index(b"\n") + 1) + 1          # banner and size line
    start = data.index(b"\n", head) + 1                          # from the second entry line on:
    while data.index(b" ", start) - start < 2:                   # the first line whose row index has two digits
        start = data.index(b"\n", start) + 1
    seg = data[start:data.index(b"\n", start) + 1]
    v0 = seg.rindex(b" ") + 1
    assert seg[v0:v0 + 2].isdigit()
    k = {"index": 1, "value": v0 + 1, "space": seg.index(b" ") + 1, "cr_lf": seg.index(b"\r") + 1,
         "line_end": len(seg)}[where]
    p = write(tmp_path, data)
    check(p, True, chunk_bytes=start - head + k)                  # the first chunk read ends at that byte


def declined_file(case):
    """(text or bytes, transpose) of a file the GPU reader declines."""
    X = counts(6, 5, 9, density=0.6)
    ent = entries_of(X, False)
    m, n, tr, field, text = 6, 5, False, "integer", None
    if case == "order_rows":                 # column-major file read without transpose
        ent.sort(key=lambda e: (e[1], e[0]))
    elif case == "order_cols":               # row-major genes x cells file read with transpose
        ent, m, n, tr = [(j, i, v) for (i, j, v) in ent], 5, 6, True
        ent.sort()
    elif case == "duplicate":
        ent = ent[:3] + [ent[2]] + ent[3:]
    elif case == "symmetric":
        text = mtx_text([(2, 1, "3"), (4, 2, "5")], 6, 6).replace("general", "symmetric")
    elif case == "pattern":
        text = "%%MatrixMarket matrix coordinate pattern general\n6 5 2\n1 2\n3 4\n"
    elif case == "array":
        M = X.toarray()
        text = "%%MatrixMarket matrix array integer general\n6 5\n" + "".join("%d\n" % v for v in M.T.reshape(-1))
    elif case in ("fraction", "exponent", "sign", "negative", "digits19"):
        i, j, _ = ent[2]
        ent[2] = (i, j, {"fraction": "1.5", "exponent": "1e3", "sign": "+3", "negative": "-3",
                         "digits19": "1234567890123456789"}[case])
    elif case in ("two_spaces", "tab", "trailing_space"):
        text = mtx_text(ent, m, n).split("\n")
        k = 4
        text[k] = {"two_spaces": text[k].replace(" ", "  ", 1), "tab": text[k].replace(" ", "\t", 1),
                   "trailing_space": text[k] + " "}[case]
        text = "\n".join(text)
    elif case in ("blank_line", "comment_line"):
        text = mtx_text(ent, m, n).split("\n")
        text.insert(5, "" if case == "blank_line" else "% a comment")
        text = "\n".join(text)
    elif case == "fewer":
        text = mtx_text(ent, m, n, nnz=len(ent) + 1)
    elif case == "more":
        text = mtx_text(ent, m, n, nnz=len(ent) - 1)
    elif case == "index0":
        ent[1] = (0, ent[1][1], ent[1][2])
    elif case == "index_above":
        ent[-1] = (ent[-1][0], n + 1, ent[-1][2])
    elif case == "gzip":
        return gzip.compress(mtx_text(ent, m, n).encode()), tr, ".mtx.gz"
    if text is None:
        text = mtx_text(ent, m, n, field)
    return text, tr, ".mtx"


@pytest.mark.parametrize("case", ["order_rows", "order_cols", "duplicate", "symmetric", "pattern", "array", "fraction",
                                  "exponent", "sign", "negative", "two_spaces", "tab", "trailing_space", "blank_line",
                                  "comment_line", "fewer", "more", "index0", "index_above", "digits19", "gzip"])
def test_declined(tmp_path, case):
    text, tr, ext = declined_file(case)
    p = write(tmp_path, text, "m" + ext)
    assert io.read_counts_mtx(p, tr) is None
    try:
        ref = io._read_mtx_scipy(p)
    except Exception as e:                                       # scipy refuses it: so does read_dataset
        with pytest.raises(type(e)):
            io.read_dataset(p, transpose=tr)
        return
    sub = ref.X[:10].toarray()
    if not np.all(sub.astype(int) == sub):
        with pytest.raises(AssertionError, match="unnormalized count data"):
            io.read_dataset(p, transpose=tr)
        return
    ad = io.read_dataset(p, transpose=tr)
    assert_same_csr(ad.X, scipy_csr(p, tr))


def test_read_dataset_round_trip(tmp_path, monkeypatch):
    M = counts(50, 40, 10, density=0.3).toarray()
    M[:, 0] = 1
    X = sp.csr_matrix(M)
    p = write(tmp_path, mtx_text(entries_of(sp.csr_matrix(X), True), 40, 50))
    exp = io.read_dataset(io._read_mtx_scipy(p), transpose=True, test_split=True)

    def no_scipy(*a, **k):
        raise AssertionError("the scipy reader was used")
    monkeypatch.setattr(io, "_read_mtx_scipy", no_scipy)
    ad = io.read_dataset(p, transpose=True, test_split=True)
    assert_same_csr(ad.X, exp.X)
    pd.testing.assert_index_equal(ad.obs_names, exp.obs_names)
    pd.testing.assert_index_equal(ad.var_names, exp.var_names)
    assert list(ad.obs["dca_split"]) == list(exp.obs["dca_split"])
    assert ad.obs["dca_split"].dtype == exp.obs["dca_split"].dtype


def test_cli_mtx_against_tsv(tmp_path, monkeypatch):
    from dca_b200.__main__ import main
    from tests.util import synth_counts
    Y = synth_counts(300, 64, 11)                                # cells x genes, 10x-like
    X = sp.csr_matrix(Y.astype(np.int64))
    mtx = write(tmp_path, mtx_text(entries_of(X, True), 64, 300), "counts.mtx")
    tsv = tmp_path / "counts.tsv"
    G = Y.T.astype(np.int64)                                     # genes x cells
    tsv.write_text("\t" + "\t".join(str(c) for c in range(300)) + "\n" +
                   "".join("%d\t%s\n" % (g, "\t".join(str(v) for v in G[g])) for g in range(64)))
    args = ["--type", "zinb-conddisp", "-e", "3", "-b", "64", "--testsplit", "--preprocess", "device", "--packed"]
    main([str(tsv), str(tmp_path / "tsv")] + args)

    def guarded(orig):
        def f(self, *a, **k):
            if self.shape[0] > 16:
                raise AssertionError("a dense host copy of %d rows of the input" % self.shape[0])
            return orig(self, *a, **k)
        return f
    monkeypatch.setattr(sp.csr_matrix, "toarray", guarded(sp.csr_matrix.toarray))
    monkeypatch.setattr(sp.csr_matrix, "todense", guarded(sp.csr_matrix.todense))

    def no_scipy(*a, **k):
        raise AssertionError("the scipy reader was used")
    monkeypatch.setattr(io, "_read_mtx_scipy", no_scipy)
    main([mtx, str(tmp_path / "mtx")] + args)
    for f in ("mean.tsv", "dispersion.tsv", "dropout.tsv", "latent.tsv"):
        assert (tmp_path / "mtx" / f).read_bytes() == (tmp_path / "tsv" / f).read_bytes(), f


# -------------------------------------------------------------------------------------------------- past 2^32 bytes
GENES, DENSITY = 2000, 0.05
# fixed-width fields (leading zeros are unsigned decimals too): 25 bytes per entry line
WG, WC, WV = 8, 9, 5


def _digits(x, width):
    out = np.empty((x.size, width), dtype=np.uint8)
    x = x.astype(np.int64)
    for k in range(width - 1, -1, -1):
        out[:, k] = 48 + x % 10
        x //= 10
    return out


def _write_large(path, n_cells, seed=0, block=20000):
    """A seeded genes x cells file in column-major order; returns the cells x genes CSR arrays it holds."""
    rng = np.random.default_rng(seed)
    indptr = np.zeros(n_cells + 1, dtype=np.int64)
    idx_parts, val_parts = [], []
    with open(path, "wb") as f:
        f.write(b"%%MatrixMarket matrix coordinate integer general\n")
        size_at = f.tell()
        f.write(b" " * 40 + b"\n")                               # the size line, padded until NNZ is known
        nnz = 0
        for c0 in range(0, n_cells, block):
            c1 = min(n_cells, c0 + block)
            cells, genes = np.nonzero(rng.integers(0, 1000, (c1 - c0, GENES), dtype=np.int16) < DENSITY * 1000)
            vals = rng.integers(1, 99999, cells.size).astype(np.int64)
            lines = np.empty((cells.size, WG + WC + WV + 3), dtype=np.uint8)
            lines[:, :WG] = _digits(genes + 1, WG)
            lines[:, WG] = 32
            lines[:, WG + 1:WG + 1 + WC] = _digits(cells + c0 + 1, WC)
            lines[:, WG + 1 + WC] = 32
            lines[:, WG + 2 + WC:-1] = _digits(vals, WV)
            lines[:, -1] = 10
            f.write(lines.tobytes())
            indptr[c0 + 1:c1 + 1] = np.bincount(cells, minlength=c1 - c0)
            idx_parts.append(genes.astype(np.int32))
            val_parts.append(vals.astype(np.float32))
            nnz += cells.size
        header_end = size_at + 41
        f.seek(size_at)
        size = b"%d %d %d" % (GENES, n_cells, nnz)
        f.write(b"%" * (39 - len(size)) + b"\n" + size)           # the padding becomes a comment line
    np.cumsum(indptr, out=indptr)
    return indptr, np.concatenate(idx_parts), np.concatenate(val_parts), header_end


def test_past_2_pow_32_bytes(tmp_path):
    line = WG + WC + WV + 3
    n_cells = int((2 ** 32 + 2 ** 28) / (line * GENES * DENSITY)) + 1
    need = n_cells * GENES * DENSITY * line * 1.05
    if shutil.disk_usage(str(tmp_path)).free < need + (1 << 30):
        pytest.skip("needs %.1f GB of free disk" % (need / 1e9))
    nnz_est = n_cells * GENES * DENSITY
    if torch.cuda.mem_get_info()[0] < 8 * nnz_est + (4 << 30):
        pytest.skip("needs %.1f GB of free device memory" % ((8 * nnz_est + (4 << 30)) / 1e9))
    p = str(tmp_path / "large.mtx")
    indptr, indices, data, header_end = _write_large(p, n_cells)
    size = os.path.getsize(p)
    assert size > 2 ** 32
    # the entry whose line holds byte 2^32, and its cell
    k = (2 ** 32 - header_end) // line
    cell = int(np.searchsorted(indptr, k, side="right") - 1)
    assert header_end + indptr[cell] * line <= 2 ** 32 < header_end + indptr[cell + 1] * line
    ad = io.read_counts_mtx(p, transpose=True)
    assert ad is not None
    X = ad.X
    assert X.shape == (n_cells, GENES) and X.indptr.dtype == np.int32 and X.indices.dtype == np.int32
    for r in (cell - 1, cell, cell + 1):                         # rows on both sides of the 2^32-byte offset
        a, b = indptr[r], indptr[r + 1]
        assert X.indptr[r] == a and X.indptr[r + 1] == b
        assert np.array_equal(X.indices[a:b], indices[a:b]) and np.array_equal(X.data[a:b], data[a:b])
    assert np.array_equal(X.indptr, indptr)
    assert np.array_equal(X.indices, indices)
    assert X.data.tobytes() == data.tobytes()
