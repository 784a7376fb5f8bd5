"""A minimal AnnData stand-in (anndata / scanpy / h5py are not in the image).

Implements only what the DCA surface touches (dca/io.py, dca/api.py, dca/network.py):
X, obs, var, obsm, uns, raw, n_obs, n_vars, obs_names, var_names, copy(), transpose(),
boolean row subsetting, obsm_keys(), var_keys(), uns_keys().  When the real ``anndata``
package is importable the host code accepts its objects as well (duck typing).

X is a dense ndarray, or a scipy.sparse CSR matrix when the constructor is asked to keep one
(``keep_sparse=True``, as the Matrix Market readers do); copies, the transpose, raw and every
subset of a CSR AnnData stay CSR.
"""
from __future__ import annotations

import numpy as np
import pandas as pd


class _Raw:
    def __init__(self, X, var):
        self.X = X
        self.var = var

    @property
    def var_names(self):
        return self.var.index

    def __getitem__(self, idx):
        return _Raw(self.X[idx], self.var)


def _is_sparse(X):
    return hasattr(X, "toarray")


def _copy_x(X):
    return X.copy() if _is_sparse(X) else np.array(X, copy=True)


class AnnData:
    def __init__(self, X, obs=None, var=None, obsm=None, uns=None, raw=None, dtype=np.float32, *, keep_sparse=False):
        """A sparse X is densified unless keep_sparse=True, which keeps it as a CSR matrix of `dtype`."""
        if _is_sparse(X) and keep_sparse:
            X = X.tocsr()
            self.X = X if X.dtype == dtype else X.astype(dtype)
        else:
            if _is_sparse(X):
                X = X.toarray()
            self.X = np.asarray(X, dtype=dtype)
        if self.X.ndim != 2:
            raise ValueError("X must be 2-dimensional (cells x genes)")
        n, g = self.X.shape
        self.obs = obs.copy() if obs is not None else pd.DataFrame(index=pd.Index([str(i) for i in range(n)]))
        self.var = var.copy() if var is not None else pd.DataFrame(index=pd.Index([str(i) for i in range(g)]))
        if len(self.obs) != n or len(self.var) != g:
            raise ValueError("obs/var length does not match X")
        self.obsm = dict(obsm) if obsm else {}
        self.uns = dict(uns) if uns else {}
        self._raw = raw

    # -- basic properties
    @property
    def n_obs(self): return self.X.shape[0]
    @property
    def n_vars(self): return self.X.shape[1]
    @property
    def shape(self): return self.X.shape
    @property
    def obs_names(self): return self.obs.index
    @property
    def var_names(self): return self.var.index

    @property
    def raw(self): return self._raw

    @raw.setter
    def raw(self, value):
        if value is None or isinstance(value, _Raw):
            self._raw = value
        else:   # anndata semantics: adata.raw = adata  freezes X and var
            self._raw = _Raw(_copy_x(value.X), value.var.copy())

    def obsm_keys(self): return list(self.obsm.keys())
    def var_keys(self): return list(self.var.columns)
    def obs_keys(self): return list(self.obs.columns)
    def uns_keys(self): return list(self.uns.keys())

    def copy(self):
        raw = None if self._raw is None else _Raw(self._raw.X.copy(), self._raw.var.copy())
        return AnnData(self.X.copy(), self.obs, self.var, {k: np.array(v, copy=True) for k, v in self.obsm.items()},
                       dict(self.uns), raw, dtype=self.X.dtype, keep_sparse=True)

    def transpose(self):
        X = self.X.T.tocsr() if _is_sparse(self.X) else self.X.T.copy()
        return AnnData(X, self.var, self.obs, None, dict(self.uns), None, dtype=self.X.dtype, keep_sparse=True)

    T = property(transpose)

    # in-place boolean subsetting with anndata's (private but long-stable) method names: what scanpy's filter_* and
    # normalize_per_cell call on the caller's object
    def _inplace_subset_obs(self, mask):
        mask = np.asarray(mask)
        self.X = self.X[mask]
        self.obs = self.obs[mask] if mask.dtype == bool else self.obs.iloc[mask]
        self.obsm = {k: np.asarray(v)[mask] for k, v in self.obsm.items()}
        if self._raw is not None:
            self._raw = self._raw[mask]

    def _inplace_subset_var(self, mask):
        mask = np.asarray(mask)
        self.X = self.X[:, mask]
        self.var = self.var[mask] if mask.dtype == bool else self.var.iloc[mask]

    def __getitem__(self, idx):
        if isinstance(idx, tuple):
            raise NotImplementedError("anndata_lite supports row subsetting only")
        if isinstance(idx, pd.Series):
            idx = idx.values
        idx = np.asarray(idx)
        raw = None if self._raw is None else self._raw[idx]
        return AnnData(self.X[idx], self.obs.iloc[idx] if idx.dtype != bool else self.obs[idx], self.var,
                       {k: np.asarray(v)[idx] for k, v in self.obsm.items()}, dict(self.uns), raw, dtype=self.X.dtype,
                       keep_sparse=True)

    def __repr__(self):
        return "AnnData(lite) n_obs x n_vars = %d x %d" % self.shape


def is_anndata(obj) -> bool:
    if isinstance(obj, AnnData):
        return True
    try:
        import anndata  # type: ignore
        return isinstance(obj, anndata.AnnData)
    except Exception:
        return False
