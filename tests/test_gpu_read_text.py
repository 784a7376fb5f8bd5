"""GPU reader of TSV / CSV count tables (io.read_counts_text, csrc/read_text.cu) against the pandas reader: the same
matrix bytes and labels in both orientations, and the pandas result for every file it does not take."""
import gzip

import numpy as np
import pandas as pd
import pytest

from dca_b200 import io
from dca_b200.anndata_lite import AnnData

pytestmark = pytest.mark.gpu

BOM = "\ufeff"


def table_text(M, rows, cols, sep="\t", eol="\n", final_eol=True, index_name="", tokens=None):
    """Text of a gene x cell table: header (index_name, cols), one line per row label; tokens[i][j] overrides M."""
    lines = [sep.join([index_name] + list(cols))]
    for i, r in enumerate(rows):
        vals = [str(int(v)) for v in M[i]]
        if tokens is not None:
            vals = [tokens[i][j] if tokens[i][j] is not None else v for j, v in enumerate(vals)]
        lines.append(sep.join([r] + vals))
    return eol.join(lines) + (eol if final_eol else "")


def write(tmp_path, text, name="counts.tsv"):
    p = tmp_path / name
    p.write_bytes(text.encode("utf-8") if isinstance(text, str) else text)
    return str(p)


def counts(n, g, seed=0, density=0.35, lam=3.0):
    rng = np.random.default_rng(seed)
    return (rng.poisson(lam, (n, g)) * (rng.random((n, g)) < density)).astype(np.int64)


def assert_same(ad, exp):
    assert ad.X.dtype == np.float32 and ad.X.shape == exp.X.shape
    assert ad.X.tobytes() == exp.X.tobytes()
    pd.testing.assert_index_equal(ad.obs_names, exp.obs_names)
    pd.testing.assert_index_equal(ad.var_names, exp.var_names)
    assert ad.obs_names.name == exp.obs_names.name and ad.var_names.name == exp.var_names.name


def check_fast(path, sep="\t", chunk_bytes=0):
    ref = io._read_text_pandas(path, sep)
    for tr in (False, True):
        ad = io.read_counts_text(path, sep, tr, chunk_bytes=chunk_bytes)
        assert ad is not None, "the GPU reader did not take %s" % path
        assert_same(ad, ref.transpose() if tr else ref)
    return ref


def names(prefix, n):
    return ["%s%d" % (prefix, i) for i in range(n)]


@pytest.mark.parametrize("sep", ["\t", ","])
@pytest.mark.parametrize("eol", ["\n", "\r\n"])
@pytest.mark.parametrize("final_eol", [True, False])
def test_separators_and_line_ends(tmp_path, sep, eol, final_eol):
    M = counts(7, 13, 1)
    p = write(tmp_path, table_text(M, names("g", 7), names("c", 13), sep, eol, final_eol),
              "counts.csv" if sep == "," else "counts.tsv")
    check_fast(p, sep)


@pytest.mark.parametrize("index_name", ["", "gene", BOM + "gene", BOM])
def test_index_headers(tmp_path, index_name):
    M = counts(5, 6, 2)
    check_fast(write(tmp_path, table_text(M, names("g", 5), names("c", 6), index_name=index_name)))


@pytest.mark.parametrize("rows", [
    ["007", "1.50", "3"],          # float index: 7.0, 1.5, 3.0
    ["007", "12", "3"],            # int index: 7, 12, 3
    ["NA", "x", "y"],              # NaN -> 'nan'
    ["NA", "", "nan"],             # all missing
    ["TRUE", "False", "true"],     # bool index
    ["a", "a", "b"],               # duplicates stay duplicates
    ["", "x", "TRUE"],             # an empty label
])
def test_row_labels(tmp_path, rows):
    M = counts(3, 4, 3)
    check_fast(write(tmp_path, table_text(M, rows, ["c", "c", "d", "c"])))     # duplicate column labels: c, c.1, ...


def test_dot_tokens_and_rounding(tmp_path):
    vals = [0, 2 ** 24 + 1, 2 ** 31, 10 ** 18 - 1, 2 ** 53 + 1, 2 ** 24 + 3, 16777217, 123456789012345678]
    M = np.array([vals, vals[::-1]], dtype=np.int64)
    check_fast(write(tmp_path, table_text(M, ["a", "b"], names("c", len(vals)))))
    M2 = counts(4, 5, 4)
    tok = [[None] * 5 for _ in range(4)]
    tok[0][1], tok[2][3], tok[3][0] = "5.0", "7.", "12.000"
    M2[0, 1], M2[2, 3], M2[3, 0] = 5, 7, 12
    check_fast(write(tmp_path, table_text(M2, names("g", 4), names("c", 5), tokens=tok), "dots.tsv"))


def test_shapes(tmp_path):
    check_fast(write(tmp_path, table_text(np.array([[4]]), ["g"], ["c"]), "one.tsv"))
    check_fast(write(tmp_path, table_text(counts(20, 100000, 5), names("g", 20), names("c", 100000)), "wide.tsv"))
    check_fast(write(tmp_path, table_text(counts(50000, 8, 6), names("g", 50000), names("c", 8)), "tall.tsv"))
    for d in (0.0, 0.05, 0.9, 1.0):
        check_fast(write(tmp_path, table_text(counts(37, 53, 7, density=d, lam=40), names("g", 37), names("c", 53)),
                         "sparse.tsv"))


@pytest.mark.parametrize("where", ["token", "separator", "cr_lf", "line_end"])
def test_chunk_boundaries(tmp_path, where):
    M = counts(12, 9, 8, density=0.8, lam=500)
    text = table_text(M, names("g", 12), names("c", 9), eol="\r\n")
    data = text.encode()
    head = data.index(b"\n") + 1
    line2 = data.index(b"\n", data.index(b"\n", head) + 1) + 1     # the third data line starts here
    seg = data[line2:data.index(b"\n", line2) + 1]
    if where == "token":
        k = next(i for i in range(1, len(seg)) if chr(seg[i - 1]).isdigit() and chr(seg[i]).isdigit())
    elif where == "separator":
        k = seg.index(b"\t") + 1
    elif where == "cr_lf":
        k = seg.index(b"\r") + 1
    else:
        k = len(seg)
    p = write(tmp_path, data)
    check_fast(p, "\t", chunk_bytes=line2 - head + k)      # the first chunk read ends at that byte


@pytest.mark.parametrize("case", ["sign", "fraction", "exponent", "na_value", "space", "ragged", "blank_line",
                                  "implicit_index", "quote", "empty_value", "digits", "big_with_dot", "long_line",
                                  "mixed_label_chunks", "gzip"])
def test_fallback(tmp_path, case):
    M = counts(6, 5, 9)
    rows, cols = names("g", 6), names("c", 5)
    tok = [[None] * 5 for _ in range(6)]
    text, name, chunk, sep = None, "counts.tsv", 0, "\t"
    if case in ("sign", "fraction", "exponent", "na_value", "space", "empty_value", "digits", "big_with_dot"):
        tok[2][3] = {"sign": "-1", "fraction": "1.5", "exponent": "1e3", "na_value": "NA", "space": " 4",
                     "empty_value": "", "digits": "1234567890123456789", "big_with_dot": "9007199254740993"}[case]
        if case == "big_with_dot":
            tok[4][1] = "2.0"
    elif case == "quote":
        rows[1] = '"g1"'
    elif case == "ragged":                             # one data line with an extra field
        lines = table_text(M, rows, cols).split("\n")
        lines[2] += "\t7"
        text = "\n".join(lines)
    elif case == "blank_line":
        lines = table_text(M, rows, cols).split("\n")
        lines.insert(3, "")
        text = "\n".join(lines)
    elif case == "implicit_index":
        text = table_text(M, rows, cols).split("\n", 1)[1]
        text = "\t".join(cols) + "\n" + text
    elif case == "long_line":
        chunk = 8
    elif case == "mixed_label_chunks":                 # 8-row inference chunks of a 100001-field table: int, then str
        M = counts(20, 100000, 10)
        rows, cols = [str(i) for i in range(8)] + names("g", 12), names("c", 100000)
        tok = None
    if text is None:
        text = table_text(M, rows, cols, tokens=tok)
    if case == "gzip":
        name = "counts.tsv.gz"
        p = write(tmp_path, gzip.compress(text.encode()), name)
        assert io.read_counts_text(p, sep) is None
        ad = io.read_dataset(p)
        ref = AnnData(M.astype(np.float32), obs=pd.DataFrame(index=pd.Index(rows)), var=pd.DataFrame(index=pd.Index(cols)))
        assert ad.X.tobytes() == ref.X.tobytes()
        return
    p = write(tmp_path, text, name)
    assert io.read_counts_text(p, sep, False, chunk_bytes=chunk) is None
    assert io.read_counts_text(p, sep, True, chunk_bytes=chunk) is None
    try:
        ref = io._read_text_pandas(p, sep)
    except Exception as e:                                # pandas refuses it: so does read_dataset
        with pytest.raises(type(e)):
            io.read_dataset(p)
        return
    X_sub = ref.X[:10]
    if not np.all(X_sub.astype(int) == X_sub):
        with pytest.raises(AssertionError, match="unnormalized count data"):
            io.read_dataset(p)
        return
    ad = io.read_dataset(p)
    assert_same(ad, ref)


def test_fractional_table_fails_the_count_check(tmp_path):
    p = write(tmp_path, table_text(counts(4, 4, 11), names("g", 4), names("c", 4)).replace("\t0", "\t0.5"))
    assert io.read_counts_text(p, "\t") is None
    with pytest.raises(AssertionError, match="unnormalized count data"):
        io.read_dataset(p)


def test_read_dataset_round_trip(tmp_path, monkeypatch):
    M = counts(30, 50, 12)
    p = write(tmp_path, table_text(M, names("g", 30), names("c", 50), index_name="gene"))
    exp = io.read_dataset(io._read_text_pandas(p, "\t"), transpose=True, test_split=True)

    def no_pandas(*a, **k):
        raise AssertionError("the pandas reader was used")
    monkeypatch.setattr(io, "_read_text_pandas", no_pandas)
    ad = io.read_dataset(p, transpose=True, test_split=True)
    assert_same(ad, exp)
    assert list(ad.obs["dca_split"]) == list(exp.obs["dca_split"])
    assert ad.obs["dca_split"].dtype == exp.obs["dca_split"].dtype
