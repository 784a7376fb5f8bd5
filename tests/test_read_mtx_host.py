"""Host half of the Matrix Market route: .mtx and .mtx.gz paths without a GPU go to the scipy statement, and the lite
AnnData keeps a CSR X through copy, transpose, raw and subsetting, with the values of the dense AnnData.  No GPU
needed."""
import gzip

import numpy as np
import pandas as pd
import pytest
import scipy.io
import scipy.sparse as sp

from dca_b200 import io
from dca_b200.anndata_lite import AnnData


def counts_csr(n, g, seed=0, density=0.3):
    rng = np.random.default_rng(seed)
    M = (rng.poisson(4.0, (n, g)) * (rng.random((n, g)) < density)).astype(np.float32)
    M[:, 0] += 1                                   # no all-zero cell
    M[0] += 1                                      # no all-zero gene
    return sp.csr_matrix(M)


def csr_ad(X, seed=1):
    ad = AnnData(X, keep_sparse=True)
    ad.obs["g"] = np.random.default_rng(seed).integers(0, 3, X.shape[0])
    return ad


def assert_same_x(a, b):
    """a: CSR, b: dense; same values and dtype."""
    assert sp.issparse(a) and a.format == "csr"
    assert a.dtype == b.dtype and a.shape == b.shape
    assert a.toarray().tobytes() == np.asarray(b).tobytes()


@pytest.mark.parametrize("gz", [False, True])
def test_routing_without_cuda(tmp_path, monkeypatch, gz):
    A = counts_csr(30, 12).T.tocsc()                                     # genes x cells, written column-major
    p = tmp_path / "m.mtx"
    scipy.io.mmwrite(str(p), A, field="integer")
    if gz:
        q = tmp_path / "m.mtx.gz"
        q.write_bytes(gzip.compress(p.read_bytes()))
        p = q
    monkeypatch.setattr(io, "_cuda_available", lambda: False)
    called = []
    monkeypatch.setattr(io, "read_counts_mtx", lambda *a, **k: called.append(a))
    ad, transposed = io._read_path(str(p), True)
    assert not called and not transposed
    exp = io._read_mtx_scipy(str(p))
    for got in (ad, exp):
        assert sp.issparse(got.X) and got.X.format == "csr" and got.X.dtype == np.float32
    assert (ad.X != exp.X).nnz == 0
    assert list(ad.obs_names) == [str(i) for i in range(12)] and list(ad.var_names) == [str(i) for i in range(30)]
    rd = io.read_dataset(str(p), transpose=True, test_split=True)
    assert sp.issparse(rd.X) and rd.X.shape == (30, 12)
    assert rd.X.toarray().tobytes() == np.ascontiguousarray(A.T.toarray().astype(np.float32)).tobytes()


def test_csr_operations_stay_csr():
    X = counts_csr(40, 16, 2)
    s, d = csr_ad(X), csr_ad(X.toarray())
    assert sp.issparse(s.X) and not sp.issparse(d.X)
    assert_same_x(s.copy().X, d.copy().X)
    assert_same_x(s.transpose().X, d.transpose().X)
    assert s.transpose().obs_names.equals(d.transpose().obs_names)
    s.raw = s
    d.raw = d
    assert_same_x(s.raw.X, d.raw.X)
    s2, d2 = s.copy(), d.copy()
    s2.raw, d2.raw = s2.copy(), d2.copy()
    assert_same_x(s2.raw.X, d2.raw.X)
    mask = np.arange(16) % 3 != 1
    rows = np.arange(40) % 4 != 2
    s2._inplace_subset_var(mask)
    d2._inplace_subset_var(mask)
    s2._inplace_subset_obs(rows)
    d2._inplace_subset_obs(rows)
    assert_same_x(s2.X, d2.X)
    assert_same_x(s2.raw.X, d2.raw.X)
    assert s2.obs.equals(d2.obs) and s2.var.equals(d2.var)
    sel = pd.Series(np.arange(40) % 5 == 0)
    assert_same_x(s[sel].X, d[sel].X)
    assert_same_x(s[sel].raw.X, d[sel].raw.X)
    assert_same_x(s[np.array([3, 1, 7])].X, d[np.array([3, 1, 7])].X)


def test_constructor_still_densifies():
    X = counts_csr(5, 8, 3)
    ad = AnnData(X)
    assert isinstance(ad.X, np.ndarray) and ad.X.tobytes() == X.toarray().tobytes()
    assert sp.issparse(AnnData(X, keep_sparse=True).X)
    assert AnnData(X.astype(np.float64), keep_sparse=True).X.dtype == np.float32


def test_host_normalize_matches_dense():
    M = counts_csr(60, 24, 4, density=0.2).toarray()
    M[5] = 0                                         # a cell the filter drops
    M[:, 7] = 0                                      # a gene the filter drops
    X = sp.csr_matrix(M)
    s, d = AnnData(X, keep_sparse=True), AnnData(X.toarray())
    io.normalize(s)
    io.normalize(d)
    assert not sp.issparse(s.X)
    assert s.X.tobytes() == d.X.tobytes()
    assert_same_x(s.raw.X, d.raw.X)
    pd.testing.assert_frame_equal(s.obs, d.obs)
    assert s.var_names.equals(d.var_names)


def test_check_counts_rejects_fractional_csr():
    X = counts_csr(12, 8, 5)
    X.data[0] = 0.5
    with pytest.raises(AssertionError, match="unnormalized count data"):
        io.read_dataset(AnnData(X, keep_sparse=True))
    with pytest.raises(AssertionError, match="unnormalized count data"):
        io.read_dataset(AnnData(X.toarray()))
