"""Host half of the GPU text reader: the row labels it rebuilds from the first field of every line (io._row_labels) and
the row chunks pandas infers column types in, against pandas reading the whole file.  No GPU needed."""
import numpy as np
import pandas as pd
import pytest

from dca_b200 import io


def table(rows, n_cols, index_name="gene"):
    head = "\t".join([index_name] + ["c%d" % j for j in range(n_cols)])
    body = "".join("%s\t%s\n" % (r, "\t".join(["1"] * n_cols)) for r in rows)
    return (head + "\n" + body).encode()


def rebuilt(path, rows, n_cols):
    """_row_labels from what the device returns: the raw first-field bytes of every data line and their offsets."""
    raw = [r.encode() for r in rows]
    offsets = np.zeros(len(raw) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in raw], out=offsets[1:])
    return io._row_labels(path, b"\t", b"".join(raw), offsets, n_cols + 1)


@pytest.mark.parametrize("rows,index_name", [
    (["007", "1.50", "3"], "gene"), (["007", "12", "3"], ""), (["NA", "x", "y"], "\ufeffgene"), (["NA", "", "nan"], ""),
    (["TRUE", "False", "true"], "g"), (["a", "a", "b"], "\ufeff"), (["", "x", "TRUE"], ""), (["-0", "1e3", "inf"], "x"),
])
def test_row_labels_match_pandas(tmp_path, rows, index_name):
    p = tmp_path / "t.tsv"
    p.write_bytes(table(rows, 3, index_name))
    exp = pd.read_csv(p, sep="\t", index_col=0).index.astype(str)
    got = rebuilt(str(p), rows, 3)
    assert got is not None
    pd.testing.assert_index_equal(got.astype(str), exp)


def test_pandas_type_inference_chunks(tmp_path):
    # 2044 value columns: 2045 fields, chunks of 256 rows; an int chunk then a str chunk mix into one object column
    assert io._pandas_chunk_rows(2045) == 256 and io._pandas_chunk_rows(2044) == 512
    rows = ["007"] * 300 + ["abc"]
    p = tmp_path / "t.tsv"
    p.write_bytes(table(rows, 2044))
    idx = list(pd.read_csv(p, sep="\t", index_col=0, low_memory=True).index.astype(str))
    assert idx[255] == "7" and idx[256] == "007"
    assert rebuilt(str(p), rows, 2044) is None                   # mixed chunks: left to pandas
    rows = ["g%d" % i for i in range(300)] + ["abc"]             # every chunk str: the same strings
    p.write_bytes(table(rows, 2044))
    got = rebuilt(str(p), rows, 2044)
    pd.testing.assert_index_equal(got.astype(str), pd.read_csv(p, sep="\t", index_col=0).index.astype(str))
