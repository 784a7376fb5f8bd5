"""Data preparation and text I/O with the surface of dca/io.py:53-131.

scanpy / anndata are not available in the image, so the four ``sc.pp`` calls the reference
makes (dca/io.py:91-109, dca/api.py:163) are restated in NumPy (semantics in SURVEY.md A.1 /
Appendix B); real AnnData objects are accepted when ``anndata`` is importable.
"""
from __future__ import annotations

import os
import pickle

import numpy as np
import pandas as pd

from .anndata_lite import AnnData, is_anndata


def _dense(X):
    return X.toarray() if hasattr(X, "toarray") else np.asarray(X)


def read_text_or_h5ad(path: str):
    """sc.read(path, first_column_names=True) -- dca/io.py:59.  Text tables go through the GPU reader when it can take
    them (read_counts_text), otherwise through pandas; Matrix Market files through read_counts_mtx, otherwise through
    scipy; gzip files of either through read_counts_gzip first; all give the same AnnData.  A Cell Ranger matrix
    directory goes through read_counts_10x, otherwise through _read_10x_scipy."""
    return _read_path(path, False)[0]


_TEXT_EXTS = (".tsv", ".txt", ".csv")
# magic numbers of the compressed formats pandas would decompress (or choke on) under a plain text extension
_COMPRESSED_MAGIC = (b"\x1f\x8b", b"BZh", b"\xfd7zXZ\x00", b"\x28\xb5\x2f\xfd", b"PK\x03\x04")


def _read_path(path, transpose):
    """(AnnData, transposed): transposed is True when the reader already returned the cells x genes orientation."""
    if os.path.isdir(path):
        if _cuda_available():
            ad = read_counts_10x(path, transpose)
            if ad is not None:
                return ad, transpose
        return _read_10x_scipy(path, transpose), transpose
    ext = os.path.splitext(path)[1].lower()
    if ext == ".h5ad":
        try:
            import anndata  # type: ignore
        except ImportError as e:
            raise ImportError("reading .h5ad needs the anndata package, which is not installed") from e
        return anndata.read_h5ad(path), False
    if ext == ".gz" and _cuda_available() and _is_gzip(path):
        ad = read_counts_gzip(path, transpose)
        if ad is not None:
            return ad, transpose
    if path.lower().endswith(".mtx.gz"):         # Cell Ranger >= 3 writes its matrix gzipped: scipy decompresses it
        return _read_mtx_scipy(path), False
    if ext == ".mtx":
        if _cuda_available():
            ad = read_counts_mtx(path, transpose)
            if ad is not None:
                return ad, transpose
        return _read_mtx_scipy(path), False
    sep = "," if ext == ".csv" else "\t"
    if ext in _TEXT_EXTS and _cuda_available():
        ad = read_counts_text(path, sep, transpose)
        if ad is not None:
            return ad, transpose
    return _read_text_pandas(path, sep), False


def _read_text_pandas(path, sep):
    """The pandas reader of a text table (genes x cells as in the file)."""
    tab = pd.read_csv(path, sep=sep, index_col=0)
    return AnnData(tab.values.astype(np.float32), obs=pd.DataFrame(index=tab.index.astype(str)),
                   var=pd.DataFrame(index=tab.columns.astype(str)))


def _is_gzip(path):
    with open(path, "rb") as f:
        return f.read(2) == b"\x1f\x8b"


def _cuda_available():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def read_counts_text(path, sep, transpose=False, chunk_bytes=0, device=None):
    """The AnnData _read_text_pandas(path, sep) gives (its .transpose() with transpose=True), parsed on a CUDA device
    by dca_read_text_counts (csrc/read_text.cu), bit for bit; None when the file is not one the GPU reader takes
    exactly (include/dca_b200.h lists them), is compressed, or its matrix does not fit in free device memory.

    The file's bytes go to the device in chunks of chunk_bytes (0: 64 MB) and the float32 matrix comes back.  Column
    labels come from pandas reading the header alone; row labels from pandas reading a two-column table made of the
    header's first field and every line's first field, in the row chunks pandas' own reader infers types in, so they
    are the same strings (numeric-looking labels, NA tokens, booleans, duplicates, the index name, a BOM)."""
    with open(path, "rb") as f:
        if any(f.read(6).startswith(m) for m in _COMPRESSED_MAGIC):
            return None
    return _read_text_gpu(path, sep, transpose, chunk_bytes, device, "dca_read_text_counts")


def _read_text_gpu(path, sep, transpose, chunk_bytes, device, entry):
    """read_counts_text through the native reader `entry` (the file's bytes, or those of its inflated stream)."""
    import ctypes as C
    import torch
    from . import _lib
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise ValueError("read_counts_text parses on a CUDA device (got %s)" % dev)
    lib = _lib.load()
    read = getattr(lib, entry)
    sep_b = sep.encode()
    if len(sep_b) != 1:
        return None
    info = np.zeros(4, dtype=np.int64)
    stream = torch.cuda.current_stream(dev)
    with torch.cuda.device(dev):
        st = read(os.fsencode(path), sep_b[0], int(bool(transpose)), int(chunk_bytes), dev.index,
                  C.c_void_p(stream.cuda_stream), None, 0, None, None, 0, info.ctypes.data)
        if st == -3:
            return None
        _lib.check(st, entry)
        rows, cols, nlab, work = (int(v) for v in info)
        if rows * cols * 4 + work > torch.cuda.mem_get_info(dev)[0]:
            return None
        columns = pd.read_csv(path, sep=sep, index_col=0, nrows=0).columns
        if len(columns) != cols:
            return None
        out = torch.empty((cols, rows) if transpose else (rows, cols), dtype=torch.float32, device=dev)
        offsets = np.zeros(rows + 1, dtype=np.int64)
        labels = np.zeros(max(nlab, 1), dtype=np.uint8)
        st = read(os.fsencode(path), sep_b[0], int(bool(transpose)), int(chunk_bytes), dev.index,
                  C.c_void_p(stream.cuda_stream), C.c_void_p(out.data_ptr()), out.numel(),
                  offsets.ctypes.data, labels.ctypes.data, nlab, info.ctypes.data)
        if st == -3:                 # the file changed between the two passes
            return None
        _lib.check(st, entry)
        X = out.cpu().numpy()
    del out
    index = _row_labels(path, sep_b, labels[:nlab].tobytes(), offsets, cols + 1)
    if index is None:
        return None
    obs = pd.DataFrame(index=index.astype(str))
    var = pd.DataFrame(index=columns.astype(str))
    return AnnData(X, obs=var, var=obs) if transpose else AnnData(X, obs=obs, var=var)


def _read_mtx_scipy(path):
    """scanpy's reader of a .mtx path (anndata.read_mtx): csr_matrix(scipy.io.mmread(path).astype('float32')), with
    the names '0', '1', ... of both axes."""
    import warnings
    import scipy.io
    import scipy.sparse as sp
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)        # scipy >= 1.15: spmatrix -> sparse array default
        X = sp.csr_matrix(scipy.io.mmread(path).astype(np.float32))
    return AnnData(X, keep_sparse=True)


def read_counts_mtx(path, transpose=False, chunk_bytes=0, device=None):
    """The AnnData _read_mtx_scipy(path) gives (its .transpose() with transpose=True), parsed on a CUDA device by
    dca_read_mtx_counts (csrc/read_mtx.cu): X is a float32 scipy.sparse.csr_matrix whose indptr, indices and data equal
    scipy's in dtype and bytes.  None when the GPU reader does not take the file (include/dca_b200.h lists the files it
    takes: entries in CSR order of the output, as Cell Ranger writes them for transpose=True), the file is compressed,
    or the arrays do not fit in free device memory.

    The file's bytes go to the device in chunks of chunk_bytes (0: 64 MB) in one pass, and the CSR arrays come back.
    The index arrays are int32 unless NNZ or a dimension reaches 2^31, as scipy chooses."""
    with open(path, "rb") as f:
        if any(f.read(6).startswith(m) for m in _COMPRESSED_MAGIC):
            return None
    return _read_mtx_gpu(path, transpose, chunk_bytes, device, "dca_read_mtx_counts")


def _read_mtx_gpu(path, transpose, chunk_bytes, device, entry, feature_map=None):
    """read_counts_mtx through the native reader `entry` (the file's bytes, or those of its inflated stream).  The
    '_map' entries take feature_map (int32 per file row: its output index, or -1 to drop it; None keeps every row)."""
    import ctypes as C
    import torch
    import scipy.sparse as sp
    from . import _lib
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise ValueError("read_counts_mtx parses on a CUDA device (got %s)" % dev)
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    read = getattr(_lib.load(), entry)
    info = np.zeros(4, dtype=np.int64)
    stream = torch.cuda.current_stream(dev)
    with torch.cuda.device(dev):
        args = (os.fsencode(path), int(bool(transpose)), int(chunk_bytes), dev.index, C.c_void_p(stream.cuda_stream))
        tail = ()
        if entry.endswith("_map"):
            fmap = None if feature_map is None else np.ascontiguousarray(feature_map, dtype=np.int32)
            tail = (None, 0) if fmap is None else (fmap.ctypes.data, fmap.size)
        st = read(*args, None, None, None, info.ctypes.data, *tail)
        if st == -3:
            return None
        _lib.check(st, entry)
        rows, cols, nnz, work = (int(v) for v in info)
        if 8 * (rows + 1) + 8 * nnz + work > torch.cuda.mem_get_info(dev)[0]:
            return None
        indptr = torch.empty(rows + 1, dtype=torch.int64, device=dev)
        indices = torch.empty(max(nnz, 1), dtype=torch.int32, device=dev)
        data = torch.empty(max(nnz, 1), dtype=torch.float32, device=dev)
        st = read(*args, C.c_void_p(indptr.data_ptr()), C.c_void_p(indices.data_ptr()), C.c_void_p(data.data_ptr()),
                  info.ctypes.data, *tail)
        if st == -3:
            return None
        _lib.check(st, entry)
        nnz = int(info[2])                           # the entries kept (all of them without a feature map)
        indptr, indices, data = indptr.cpu().numpy(), indices[:nnz].cpu().numpy(), data[:nnz].cpu().numpy()
    if max(rows, cols, nnz) < 2 ** 31:
        indptr = indptr.astype(np.int32)
    else:
        indices = indices.astype(np.int64)
    X = sp.csr_matrix((data, indices, indptr), shape=(rows, cols), copy=False)
    return AnnData(X, keep_sparse=True)


def read_counts_gzip(path, transpose=False, chunk_bytes=0, device=None):
    """The AnnData today's route gives for a gzip file (scipy's reader for a .mtx.gz path, else pandas' with the tab
    separator _read_path uses for a '.gz' extension), inflated and parsed on a CUDA device: dca_read_mtx_counts_gz or
    dca_read_text_counts_gz (csrc/inflate.cu) with the outputs, labels and orientation of read_counts_mtx and
    read_counts_text.  None when the file is not gzip, the inflate declines it (include/dca_b200.h, dca_gunzip), the
    parser does not take its inflated bytes, or the outputs do not fit in free device memory."""
    if not _is_gzip(path):
        return None
    if path.lower().endswith(".mtx.gz"):
        return _read_mtx_gpu(path, transpose, chunk_bytes, device, "dca_read_mtx_counts_gz")
    return _read_text_gpu(path, "\t", transpose, chunk_bytes, device, "dca_read_text_counts_gz")


# Cell Ranger's matrix directory: the files of each role, by suffix after the shared prefix (GEO's sample prefix, or '')
_10X_ROLES = (("matrix", ("matrix.mtx.gz", "matrix.mtx")),
              ("features", ("features.tsv.gz", "features.tsv", "genes.tsv.gz", "genes.tsv")),
              ("barcodes", ("barcodes.tsv.gz", "barcodes.tsv")))
_10X_WANT = {"matrix": "matrix.mtx[.gz]", "features": "features.tsv[.gz] (or genes.tsv[.gz])",
             "barcodes": "barcodes.tsv[.gz]"}


def _find_10x(path):
    """(matrix, features, barcodes): the paths of the one Cell Ranger triple in directory `path` that share a prefix;
    ValueError naming the files when a file is missing or there is more than one triple."""
    found = {}                                   # prefix -> role -> [file names]
    for name in sorted(os.listdir(path)):
        if not os.path.isfile(os.path.join(path, name)):
            continue
        for role, suffixes in _10X_ROLES:
            suf = next((x for x in suffixes if name.endswith(x)), None)
            if suf is not None:
                found.setdefault(name[:-len(suf)], {}).setdefault(role, []).append(name)
                break
    triples = []
    for prefix, roles in found.items():
        if len(roles) == 3:
            triples += [(m, f, b) for m in roles["matrix"] for f in roles["features"] for b in roles["barcodes"]]
    if len(triples) > 1:
        raise ValueError("%s holds %d candidate Cell Ranger matrix triples (matrix, features, barcodes): %s" % (
            path, len(triples), "; ".join(", ".join(t) for t in triples)))
    if not triples:
        if not found:
            raise ValueError("%s is not a Cell Ranger matrix directory: it has no %s, %s or %s" % (
                path, _10X_WANT["matrix"], _10X_WANT["features"], _10X_WANT["barcodes"]))
        missing = ["%s (beside %s)" % (prefix + _10X_WANT[role], ", ".join(sum(roles.values(), [])))
                   for prefix, roles in sorted(found.items()) for role, _ in _10X_ROLES if role not in roles]
        raise ValueError("%s is not a Cell Ranger matrix directory: missing %s" % (path, "; ".join(missing)))
    return tuple(os.path.join(path, n) for n in triples[0])


def _read_tsv_columns(path, most):
    """The first `most` tab-separated columns of a headerless label file (gzip or plain, by magic bytes) as strings,
    taken literally (no NA values, no quoting)."""
    import csv
    try:
        tab = pd.read_csv(path, sep="\t", header=None, dtype=str, na_filter=False, quoting=csv.QUOTE_NONE,
                          compression="gzip" if _is_gzip(path) else None)
    except pd.errors.EmptyDataError:
        return [np.empty(0, dtype=object)]
    return [tab[c].to_numpy(dtype=object) for c in tab.columns[:most]]


def make_index_unique(names, join="-"):
    """anndata.utils.make_index_unique: the first occurrence of a name stays; each later duplicate v takes v-1, v-2, ...
    (one counter per name), skipping any candidate already among the names or already given."""
    idx = pd.Index(names)
    if idx.is_unique:
        return idx
    values = idx.to_numpy(dtype=object).copy()
    taken = set(values)
    counter = {}
    for i in np.flatnonzero(idx.duplicated(keep="first")):
        v = values[i]
        while True:
            counter[v] = counter.get(v, 0) + 1
            cand = "%s%s%d" % (v, join, counter[v])
            if cand not in taken:
                taken.add(cand)
                values[i] = cand
                break
    return pd.Index(values, name=idx.name)


def _mtx_size(path):
    """(M, N) of a Matrix Market file's size line (gzip or plain, by magic bytes); None when there is none."""
    import gzip
    with (gzip.open if _is_gzip(path) else open)(path, "rb") as f:
        for line in f:
            if not line.startswith(b"%"):
                parts = line.split()
                return (int(parts[0]), int(parts[1])) if len(parts) >= 2 and parts[0].isdigit() and \
                    parts[1].isdigit() else None
    return None


def _10x_labels(path, shape=None):
    """(matrix path, barcodes, var, keep) of the Cell Ranger directory `path`: var (one row per feature of the file,
    indexed by the unique gene symbols) holds gene_ids and, for the v3 layout, feature_types; keep marks the rows
    read_10x_mtx(gex_only=True) keeps.  shape: (M, N) of the matrix, checked against the label counts (ValueError)."""
    matrix, features, barcodes = _find_10x(path)
    cols = _read_tsv_columns(features, 3)
    v3 = os.path.basename(features)[:-len(".tsv.gz" if features.endswith(".gz") else ".tsv")].endswith("features")
    bc = _read_tsv_columns(barcodes, 1)[0]
    if len(cols) < 2:
        raise ValueError("%s: a features file needs gene ids and symbols (2 tab-separated columns)" % features)
    if shape is None:
        shape = _mtx_size(matrix)
    if shape is not None and (len(cols[0]), len(bc)) != tuple(shape):
        raise ValueError("%s is %d x %d (features x barcodes), but %s lists %d features and %s %d barcodes" % (
            matrix, shape[0], shape[1], features, len(cols[0]), barcodes, len(bc)))
    var = pd.DataFrame({"gene_ids": cols[0]}, index=make_index_unique(cols[1]))
    keep = np.ones(len(var), dtype=bool)
    if v3 and len(cols) > 2:
        var["feature_types"] = cols[2]
        keep = cols[2] == "Gene Expression"
    return matrix, pd.Index(bc), var, keep


def _10x_anndata(X, barcodes, var, keep, transpose):
    """The AnnData of a Cell Ranger read: X cells x genes (transpose) or genes x cells, with the kept features."""
    var = var[keep]
    obs = pd.DataFrame(index=barcodes)
    return AnnData(X, obs=obs, var=var, keep_sparse=True) if transpose else \
        AnnData(X, obs=var, var=obs, keep_sparse=True)


def _read_10x_scipy(path, transpose):
    """scanpy's read_10x_mtx(path, var_names='gene_symbols', make_unique=True, gex_only=True), transposed to genes x
    cells unless `transpose`: X = csr_matrix(mmread(matrix).astype(float32)), .T.tocsr() with transpose, then the
    Gene Expression features (columns with transpose, rows without); labels as _10x_labels reads them."""
    import gzip
    import warnings
    import scipy.io
    import scipy.sparse as sp
    matrix, barcodes, var, keep = _10x_labels(path)
    with warnings.catch_warnings(), (gzip.open if _is_gzip(matrix) else open)(matrix, "rb") as f:
        warnings.simplefilter("ignore", DeprecationWarning)
        X = sp.csr_matrix(scipy.io.mmread(f).astype(np.float32))
    if X.shape != (len(var), len(barcodes)):
        raise ValueError("%s is %d x %d, but its directory lists %d features and %d barcodes" % (
            matrix, X.shape[0], X.shape[1], len(var), len(barcodes)))
    if transpose:
        X = X.T.tocsr()
    if not keep.all():
        kept = np.flatnonzero(keep)
        X = X[:, kept] if transpose else X[kept]
    return _10x_anndata(X, barcodes, var, keep, transpose)


def read_counts_10x(path, transpose=False, chunk_bytes=0, device=None):
    """The AnnData _read_10x_scipy(path, transpose) gives, with the matrix parsed on a CUDA device by
    dca_read_mtx_counts_map / dca_read_mtx_counts_gz_map (csrc/read_mtx.cu, gzip detected by magic bytes): the
    features other than Gene Expression are dropped inside the parse, so they never reach the CSR arrays, whose
    indptr, indices and data equal scipy's in dtype and bytes.  The labels are read on the host (_10x_labels).  None
    when the GPU reader does not take the matrix (as read_counts_mtx), or the arrays do not fit in free device memory.
    ValueError when the directory is not one Cell Ranger triple or its label counts do not match the matrix."""
    matrix, barcodes, var, keep = _10x_labels(path)
    fmap = None if keep.all() else np.where(keep, np.cumsum(keep) - 1, -1).astype(np.int32)
    entry = "dca_read_mtx_counts_gz_map" if _is_gzip(matrix) else "dca_read_mtx_counts_map"
    ad = _read_mtx_gpu(matrix, transpose, chunk_bytes, device, entry, fmap)
    if ad is None:
        return None
    return _10x_anndata(ad.X, barcodes, var, keep, transpose)


def _pandas_chunk_rows(width):
    """Rows per chunk in which pandas' C reader (low_memory=True) infers column types for a table of `width` fields:
    the largest power of two below half of 2**20 // width."""
    heuristic = 2 ** 20 // width
    n = 1
    while n * 2 < heuristic:
        n *= 2
    return n


def _row_labels(path, sep, labels, offsets, width):
    """The index pd.read_csv(path, sep=sep, index_col=0) gives, from the header's first field and the first field of
    every data line: pandas reads them as a two-column table (a second column keeps an empty label from being a blank
    line), chunk by chunk in the chunks its reader of the `width`-field file infers types in.  None when the chunks
    infer different types (pandas then mixes them into one object column, which this does not restate)."""
    import gzip
    import io as _io
    with (gzip.open if _is_gzip(path) else open)(path, "rb") as f:
        header = f.readline()
    head = header.split(sep, 1)[0]
    n = len(offsets) - 1
    starts, ends = offsets[:-1], offsets[1:]
    body = b"".join([labels[a:b] + sep + b"0\n" for a, b in zip(starts.tolist(), ends.tolist())])
    text = head + sep + b"x\n" + body
    try:
        whole = pd.read_csv(_io.BytesIO(text), sep=sep.decode(), index_col=0, low_memory=False).index
        step = _pandas_chunk_rows(width)
        if n > step and whole.dtype != np.int64:
            kinds = {c.index.dtype for c in pd.read_csv(_io.BytesIO(text), sep=sep.decode(), index_col=0, chunksize=step,
                                                        low_memory=False)}
            if len(kinds) != 1:
                return None
    except Exception:
        return None
    return whole


def read_dataset(adata, transpose=False, test_split=False, copy=False, check_counts=True):
    """dca/io.py:53-85.  A path to a text table is read on the GPU when read_counts_text takes it, and a Matrix Market
    file when read_counts_mtx takes it; both transpose on the device and only return integer counts, so the check below
    passes in either orientation.  A .mtx file gives a CSR X (as the reference's AnnData has)."""
    transposed = False
    if is_anndata(adata):
        if copy:
            adata = adata.copy()
    elif isinstance(adata, str):
        adata, transposed = _read_path(adata, transpose)
    else:
        raise NotImplementedError

    if check_counts:
        # check if observations are unnormalized using first 10           (dca/io.py:63-70)
        X_subset = _dense(adata.X[:10])
        norm_error = 'Make sure that the dataset (adata.X) contains unnormalized count data.'
        assert np.all(X_subset.astype(int) == X_subset), norm_error

    if transpose and not transposed:
        adata = adata.transpose()

    if test_split:
        from sklearn.model_selection import train_test_split
        train_idx, test_idx = train_test_split(np.arange(adata.n_obs), test_size=0.1, random_state=42)
        spl = pd.Series(['train'] * adata.n_obs)
        spl.iloc[test_idx] = 'test'
        adata.obs['dca_split'] = spl.values
    else:
        adata.obs['dca_split'] = 'train'

    adata.obs['dca_split'] = adata.obs['dca_split'].astype('category')
    print('dca: Successfully preprocessed {} genes and {} cells.'.format(adata.n_vars, adata.n_obs))
    return adata


def filter_genes_mask(X, min_counts=1):
    """sc.pp.filter_genes(X, min_counts=1) -> (mask, counts)   (dca/api.py:163)."""
    counts = np.asarray(_dense(X).sum(axis=0)).reshape(-1)
    return counts >= min_counts, counts


def _inplace_subset(adata, rows=None, cols=None):
    """Boolean-mask subsetting IN PLACE (what scanpy's filter_genes / filter_cells / normalize_per_cell do to the
    caller's object): anndata.AnnData and the lite stand-in both provide _inplace_subset_var / _inplace_subset_obs."""
    if cols is not None:
        adata._inplace_subset_var(np.asarray(cols))
    if rows is not None:
        adata._inplace_subset_obs(np.asarray(rows))


def apply_device_normalize(adata, dd, filter_min_counts, set_x=True):
    """The AnnData mutations of normalize() from a DeviceDataset built with the same flags (device_data.py): in-place
    filtering, raw, obs['n_counts'] / obs['size_factors'] and (set_x) X as a host fp32 copy of the device X."""
    if filter_min_counts:
        if not dd.gene_mask.all():
            _inplace_subset(adata, cols=dd.gene_mask)
        if not dd.cell_mask.all():
            _inplace_subset(adata, rows=dd.cell_mask)
    if dd.flags:
        adata.raw = adata.copy()
    else:
        adata.raw = adata
    if dd.flags & 1:
        if not dd.sf_mask.all():
            _inplace_subset(adata, rows=dd.sf_mask)
        adata.obs['n_counts'] = dd.n_counts_host
        adata.obs['size_factors'] = dd.size_factors_host
    else:
        adata.obs['size_factors'] = np.float32(1.0)
    if set_x:
        adata.X = np.ascontiguousarray(dd.host_x(), dtype=np.float32)
    return adata


def normalize(adata, filter_min_counts=True, size_factors=True, normalize_input=True, logtrans_input=True, device=None,
              stream=False, packed=False):
    """dca/io.py:88-111 with scanpy's arithmetic restated:
    filter_genes/filter_cells(min_counts=1); raw copy; normalize_per_cell (each cell scaled to the
    median total count; zero-count cells dropped as scanpy does); size_factors = n_counts/median;
    log1p (natural); scale (zero mean, unit variance with ddof=1, no clipping).

    Like the reference, this MUTATES the object it is given -- X, obs['n_counts'], obs['size_factors'], raw and (when
    filtering) the set of cells / genes -- and returns the same object, for the lite stand-in and for a real
    anndata.AnnData alike (only attribute assignment and the two in-place subsetting methods are used).

    device (None: the NumPy path above): a CUDA device to compute all of this on (device_data.DeviceDataset, same
    flags).  The AnnData is mutated the same way, X becomes a host fp32 copy of the device X, and the resident
    dataset is returned in adata.uns['dca_device_data'] for train(device_data=...) and predict(device_data=...).
    Size factors and n_counts are bit-identical to the host path; X agrees to a few fp32 ulp (device_data.py).  There
    is no fallback: without a CUDA device this raises.

    stream=True (with a device): out of core instead (stream_data.StreamedDataset, same flags, same bits as the resident
    dataset): the raw counts stay packed in host memory, adata.X keeps the (filtered) raw counts -- no normalised matrix
    exists on the host -- and the dataset is returned in adata.uns['dca_stream_data'] for train(stream_data=...) and
    predict(stream_data=...).

    packed=True (with a device): the raw counts are packed on the device and stay there, packed
    (packed_data.PackedDeviceDataset, same flags): adata.X keeps the (filtered) raw counts and the dataset is returned in
    adata.uns['dca_packed_data'] for train(packed_data=...) and predict(packed_data=...)."""
    if device is not None or stream or packed:
        if device is None:
            raise ValueError("%s=True preprocesses on a device: give device=" % ("packed" if packed else "stream"))
        if stream and packed:
            raise ValueError("give stream=True or packed=True, not both")
        from .device_data import build_dataset
        ds = build_dataset(adata.X, device, "float32", stream=stream, packed=packed, size_factors=size_factors,
                           logtrans_input=logtrans_input, normalize_input=normalize_input,
                           filter_min_counts=filter_min_counts)
        apply_device_normalize(adata, ds, filter_min_counts, set_x=not (stream or packed))
        adata.uns['dca_' + ds.kind] = ds
        return adata
    if filter_min_counts:
        gmask, _ = filter_genes_mask(adata.X, 1)                       # dca/io.py:90-92
        if not gmask.all():
            _inplace_subset(adata, cols=gmask)
        cmask = np.asarray(_dense(adata.X).sum(axis=1)).reshape(-1) >= 1
        if not cmask.all():
            _inplace_subset(adata, rows=cmask)

    if size_factors or normalize_input or logtrans_input:              # dca/io.py:94-97
        adata.raw = adata.copy()
    else:
        adata.raw = adata

    X = _dense(adata.X)
    if size_factors:                                                   # dca/io.py:99-101
        n_counts = np.asarray(X.sum(axis=1, dtype=np.float64)).reshape(-1)
        keep = n_counts >= 1                         # normalize_per_cell filters cells with < 1 count
        if not keep.all():
            _inplace_subset(adata, rows=keep)        # anndata subsets .raw along obs as well
            X = _dense(adata.X)
            n_counts = n_counts[keep]
        med = np.median(n_counts)
        adata.obs['n_counts'] = n_counts
        X = (X / (n_counts / med)[:, None]).astype(np.float32)
        adata.obs['size_factors'] = (n_counts / med).astype(np.float32)
    else:
        adata.obs['size_factors'] = np.float32(1.0)                    # dca/io.py:102-103

    if logtrans_input:                                                 # dca/io.py:105-106
        X = np.log1p(X)

    if normalize_input:                                                # dca/io.py:108-109
        mean = X.mean(axis=0, dtype=np.float64)
        var = X.var(axis=0, ddof=1, dtype=np.float64) if X.shape[0] > 1 else np.ones(X.shape[1])
        std = np.sqrt(var)
        std[std == 0] = 1.0
        X = ((X - mean) / std).astype(np.float32)

    adata.X = np.ascontiguousarray(X, dtype=np.float32)
    return adata


def read_genelist(filename):
    genelist = list(set(open(filename, 'rt').read().strip().split('\n')))
    assert len(genelist) > 0, 'No genes detected in genelist file'
    print('dca: Subset of {} genes will be denoised.'.format(len(genelist)))
    return genelist


def write_text_matrix(matrix, filename, rownames=None, colnames=None, transpose=False, threads=0, gzip=False,
                      device=None):
    """TSV with '%.6f' values, the files of dca/io.py:120-129 byte for byte.  float32 / float64 matrices go through
    the multi-threaded native writer (dca_write_text_matrix); anything else through pandas like the reference.

    gzip=True writes the same text gzip-compressed on the CUDA device `device` (default: the current one): the text
    goes to a temporary file beside `filename`, which gzip_file_device compresses in pieces and then removes."""
    if gzip:
        tmp = "%s.%d.tmp" % (filename, os.getpid())
        try:
            write_text_matrix(matrix, tmp, rownames, colnames, transpose, threads)
            gzip_file_device(tmp, filename, device=device)
        finally:
            if os.path.exists(tmp):
                os.remove(tmp)
        return
    import ctypes as C
    m = np.asarray(matrix)
    native = m.ndim == 2 and m.dtype in (np.float32, np.float64) and m.size > 0
    if native:
        from . import _lib
        lib = _lib.load()           # raises when libdca_b200.so has not been built
    if not native:                  # non-float / empty / 1-d input: the reference's own pandas call
        if transpose:
            m = m.T
            rownames, colnames = colnames, rownames
        pd.DataFrame(m, index=rownames, columns=colnames).to_csv(
            filename, sep='\t', index=(rownames is not None), header=(colnames is not None), float_format='%.6f')
        return
    m = np.ascontiguousarray(m)

    def labels(names, n):
        if names is None:
            return None, None
        vals = [str(v).encode() for v in list(names)]
        if len(vals) != n:
            raise ValueError("got %d labels for %d rows/columns" % (len(vals), n))
        arr = (C.c_char_p * n)(*vals)
        return arr, vals
    rn, _keep_r = labels(rownames, m.shape[0])
    cn, _keep_c = labels(colnames, m.shape[1])
    _lib.check(lib.dca_write_text_matrix(os.fsencode(filename), m.ctypes.data, int(m.dtype == np.float64), m.shape[0],
                                         m.shape[1], m.shape[1], rn, cn, int(bool(transpose)), int(threads)),
               "dca_write_text_matrix")


def quote_label(name):
    """The bytes of one label in the files write_text_matrix writes: str(name) in UTF-8, quoted csv.QUOTE_MINIMAL style
    (inside '"', quotes doubled) only when it holds a tab, a quote, '\\n' or '\\r'."""
    b = str(name).encode()
    if any(c in b for c in b'\t"\n\r'):
        return b'"' + b.replace(b'"', b'""') + b'"'
    return b


def label_bytes(names, n):
    """(bytes, int64 offsets[n + 1]) of the quoted labels `names` back to back: the label block dca_write_text_device
    takes."""
    vals = [quote_label(v) for v in list(names)]
    if len(vals) != n:
        raise ValueError("got %d labels for %d rows/columns" % (len(vals), n))
    offsets = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(v) for v in vals], out=offsets[1:])
    return b"".join(vals), offsets


def header_bytes(colnames, has_rownames):
    """The header line of write_text_matrix: the quoted column labels joined by tabs, after an empty cell when the
    lines have labels."""
    return (b"\t" if has_rownames else b"") + b"\t".join(quote_label(v) for v in list(colnames)) + b"\n"


def gzip_device(data, device=None, info=None):
    """One gzip member of `data` (bytes, or a 1-d uint8 CUDA tensor) compressed on a CUDA device by dca_gzip_device
    (csrc/deflate.cu), as a uint8 CUDA tensor.  Bytes go to `device` (default: the current one) first.  info: an int64
    array of 3, filled with the member's bytes, blocks and stored blocks."""
    import ctypes as C
    import torch
    from . import _lib
    if isinstance(data, torch.Tensor):
        if not data.is_cuda or data.dtype != torch.uint8 or data.dim() != 1:
            raise ValueError("gzip_device takes bytes or a 1-d uint8 CUDA tensor")
        src = data.contiguous()
    else:
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        src = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(dev) if len(data) else \
            torch.empty(0, dtype=torch.uint8, device=dev)
    lib = _lib.load()
    n = src.numel()
    info_arr = np.zeros(3, dtype=np.int64)
    _lib.check(lib.dca_gzip_device(None, n, None, 0, 0, None, info_arr.ctypes.data), "dca_gzip_device")
    out = torch.empty(int(info_arr[0]), dtype=torch.uint8, device=src.device)
    stream = torch.cuda.current_stream(src.device)
    with torch.cuda.device(src.device):
        _lib.check(lib.dca_gzip_device(C.c_void_p(src.data_ptr() if n else 0), n, C.c_void_p(out.data_ptr()), out.numel(),
                                       src.device.index, C.c_void_p(stream.cuda_stream), info_arr.ctypes.data),
                   "dca_gzip_device")
    if info is not None:
        info[:] = info_arr
    return out[:int(info_arr[0])]


def gzip_file_device(src, dst, device=None, piece_bytes=64 << 20):
    """dst = src gzip-compressed on a CUDA device: one gzip member per piece of piece_bytes, so host memory holds one
    piece whatever the file's size."""
    with open(src, "rb") as f, open(dst, "wb") as g:
        while True:
            data = f.read(piece_bytes)
            g.write(gzip_device(data, device).cpu().numpy().tobytes())
            if len(data) < piece_bytes:
                break


def write_text_matrix_device(tensor, filename, rownames=None, colnames=None, transpose=False, append=False,
                             header=True, chunk_bytes=0, info=None, gzip=False):
    """write_text_matrix(tensor.cpu().numpy(), filename, rownames, colnames, transpose) byte for byte, formatted on the
    tensor's CUDA device (dca_write_text_device, csrc/write_text.cu): a float32 matrix in device memory becomes text
    without a host copy of it.  The text reaches the file in pinned pieces of chunk_bytes (0: 16 MB), the write of one
    overlapping the formatting of the next.

    append=True appends to the file instead of creating it, and header=False leaves out the header line, so that a
    matrix can be written in blocks of output lines.  info: an int64 array of 4, filled with the bytes written, line
    groups, microseconds of formatting kernels and microseconds waiting for the file writes.  An empty matrix goes
    through write_text_matrix.

    gzip=True writes the text as one gzip member instead (appended as one more member with append=True), compressed
    on the device before it leaves it (dca_write_text_device_gz): the file decompresses to the bytes gzip=False writes,
    and info[0] counts compressed bytes."""
    import ctypes as C
    import torch
    from . import _lib
    t = tensor
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or t.dim() != 2:
        raise ValueError("write_text_matrix_device takes a 2-d float32 CUDA tensor")
    if t.numel() == 0:
        if append or not header:
            raise ValueError("an empty matrix is written whole")
        write_text_matrix(t.cpu().numpy(), filename, rownames, colnames, transpose, gzip=gzip, device=t.device)
        return
    if t.stride(1) != 1 or t.stride(0) < t.shape[1]:
        t = t.contiguous()
    rows, cols = t.shape
    line_names, head_names = (colnames, rownames) if transpose else (rownames, colnames)
    out_rows, out_cols = (cols, rows) if transpose else (rows, cols)
    labels, offsets = label_bytes(line_names, out_rows) if line_names is not None else (None, None)
    if head_names is not None:
        names = list(head_names)
        if len(names) != out_cols:
            raise ValueError("got %d labels for %d rows/columns" % (len(names), out_cols))
        head = header_bytes(names, line_names is not None) if header else b""
    else:
        head = b""
    lib = _lib.load()
    dev = t.device
    info_arr = np.zeros(4, dtype=np.int64)
    stream = torch.cuda.current_stream(dev)
    with torch.cuda.device(dev):
        entry = "dca_write_text_device_gz" if gzip else "dca_write_text_device"
        _lib.check(getattr(lib, entry)(os.fsencode(filename), int(bool(append)), C.c_void_p(t.data_ptr()), rows, cols,
                                       t.stride(0), int(bool(transpose)), head, len(head), labels,
                                       None if offsets is None else offsets.ctypes.data, int(chunk_bytes), dev.index,
                                       C.c_void_p(stream.cuda_stream), info_arr.ctypes.data),
                   entry)
    if info is not None:
        info[:] = info_arr


def read_pickle(inputfile):
    return pickle.load(open(inputfile, "rb"))


# ------------------------------------------------------------------------------------------------
# Packed host format of a raw count matrix for the streaming path (dca_stream_begin_packed, include/dca_b200.h).
# No counterpart in the reference (it feeds float matrices to Keras, dca/train.py:78-98); scRNA-seq counts
# are >80 % zeros and mostly < 15, so 4 bits per entry + a short overflow list carry the same information
# as the float32 matrix in 1/8 of the bytes that cross PCIe every step.
class PackedCounts:
    """bits-per-entry matrix + CSR overflow list; see pack_counts().  bits == 1 is the SPARSE format: ``packed`` is the
    non-zero bitmap (n_genes/8 bytes per row), ``nibbles`` the 4-bit codes of the non-zero counts in gene order (each row
    starts on a byte boundary at ``nib_indptr[row]``), codes of 15 escape into the overflow list.  ``n_genes`` is the
    stored width (a multiple of 8), ``genes`` the matrix's gene count: smaller when a ragged matrix was packed as its
    zero-padded form (pack_counts(..., pad_genes=True)), whose last n_genes - genes columns are all zero."""

    def __init__(self, packed, bits, n_genes, indptr, entries, nib_indptr=None, nibbles=None, genes=None):
        self.packed, self.bits, self.n_genes, self.indptr, self.entries = packed, bits, n_genes, indptr, entries
        self.nib_indptr, self.nibbles = nib_indptr, nibbles
        self.genes = n_genes if genes is None else int(genes)
        self._pinned = None            # pinned host copies, made by DeviceEngine.stream_begin on first use

    @property
    def n_rows(self):
        return self.packed.shape[0]

    @property
    def nbytes(self):
        extra = (self.nib_indptr.nbytes + self.nibbles.nbytes) if self.bits == 1 else 0
        return self.packed.nbytes + self.indptr.nbytes + self.entries.nbytes + extra

    def bytes_for_rows(self, r0, r1):
        """host->device bytes of one batch [r0, r1): tile + indptr segment + overflow entries (+ nibble stream)."""
        b = (r1 - r0) * self.packed.shape[1] * self.packed.itemsize + 8 * (r1 - r0 + 1) + \
            8 * int(self.indptr[r1] - self.indptr[r0])
        if self.bits == 1:
            b += 8 * (r1 - r0 + 1) + int(self.nib_indptr[r1] - self.nib_indptr[r0])
        return b

    def take_rows(self, idx, block=65536):
        """The rows ``idx`` (integer positions, in that order) as a new PackedCounts, copied on the packed arrays without
        unpacking: the bytes pack_counts writes for the selected rows at the same width.  Works in blocks of rows so
        that the index arrays stay small."""
        idx = np.asarray(idx, dtype=np.int64).reshape(-1)
        if idx.size and (idx.min() < 0 or idx.max() >= self.n_rows):
            raise IndexError("row index out of range for %d rows" % self.n_rows)
        if idx.size <= block:
            return self._take_block(idx)
        return concat_packed([self._take_block(idx[i:i + block]) for i in range(0, idx.size, block)])

    def _take_block(self, idx):
        indptr, entries = _gather_segments(self.indptr, self.entries, idx)
        if self.bits != 1:
            return PackedCounts(np.ascontiguousarray(self.packed[idx]), self.bits, self.n_genes, indptr, entries,
                                genes=self.genes)
        nib_indptr, nib = _gather_segments(self.nib_indptr, self.nibbles, idx)
        nibbles = np.zeros(nib.size + 16, dtype=np.uint8)            # + slack: the device reads whole bytes
        nibbles[:nib.size] = nib
        return PackedCounts(np.ascontiguousarray(self.packed[idx]), 1, self.n_genes, indptr, entries, nib_indptr, nibbles,
                            genes=self.genes)


def _gather_segments(indptr, data, idx):
    """CSR row selection: (new indptr, data of rows idx concatenated in that order)."""
    lens = indptr[idx + 1] - indptr[idx]
    out_ptr = np.zeros(idx.size + 1, dtype=np.int64)
    np.cumsum(lens, out=out_ptr[1:])
    row = np.repeat(np.arange(idx.size, dtype=np.int64), lens)
    src = indptr[idx][row] + np.arange(int(out_ptr[-1]), dtype=np.int64) - out_ptr[:-1][row]
    return out_ptr, data[src]


def concat_packed(parts):
    """Row concatenation of PackedCounts of one format (same width and gene count): the bytes pack_counts writes for
    the stacked matrix at that width."""
    parts = list(parts)
    if not parts:
        raise ValueError("nothing to concatenate")
    bits, g, genes = parts[0].bits, parts[0].n_genes, parts[0].genes
    if any(p.bits != bits or p.n_genes != g or p.genes != genes for p in parts):
        raise ValueError("packed parts differ in width or gene count")

    def cat_ptr(ptrs):
        out = [np.zeros(1, dtype=np.int64)]
        off = 0
        for p in ptrs:
            out.append(p[1:] - p[0] + off)
            off += int(p[-1] - p[0])
        return np.concatenate(out)
    packed = np.concatenate([p.packed for p in parts])
    indptr = cat_ptr([p.indptr for p in parts])
    entries = np.concatenate([p.entries for p in parts]) if parts else np.empty(0, OVERFLOW_ENTRY)
    if bits != 1:
        return PackedCounts(packed, bits, g, indptr, entries, genes=genes)
    nib_indptr = cat_ptr([p.nib_indptr for p in parts])
    nibbles = np.zeros(int(nib_indptr[-1]) + 16, dtype=np.uint8)
    for p, o in zip(parts, nib_indptr[np.cumsum([0] + [p.n_rows for p in parts[:-1]])]):
        n = int(p.nib_indptr[-1] - p.nib_indptr[0])
        nibbles[o:o + n] = p.nibbles[:n]
    return PackedCounts(packed, 1, g, indptr, entries, nib_indptr, nibbles, genes=genes)


def pack_rows(counts, bits="auto", batch=None, chunk_rows=16384, threads=0, pad_genes=False):
    """pack_counts of a dense matrix or a scipy.sparse CSR matrix, ``chunk_rows`` rows at a time (a CSR matrix is
    never dense on the host as a whole), concatenated with concat_packed: the bytes pack_counts writes for the whole
    matrix.  bits='auto' / 'sparse' / 'dense' decide the format once, from the whole matrix as pack_counts does.
    pad_genes: as for pack_counts (each chunk is padded as it is densified)."""
    csr = hasattr(counts, "tocsr") and getattr(counts, "format", None) == "csr"
    n, g = (int(s) for s in counts.shape)
    gp = _packed_width(g, pad_genes)
    if n <= chunk_rows and not csr:
        return pack_counts(counts, bits, batch=batch, threads=threads, pad_genes=pad_genes)
    if bits in ("auto", "sparse", "dense"):
        bits = _choose_format(counts, csr, bits, batch, chunk_rows, gp)

    def rows(r0, r1):
        m = counts[r0:r1]
        return m.toarray() if csr else np.asarray(m)
    return concat_packed([pack_counts(rows(r0, min(n, r0 + chunk_rows)), bits, threads=threads, pad_genes=pad_genes)
                          for r0 in range(0, n, chunk_rows)])


def _packed_width(g, pad_genes):
    """The stored width of g genes: g itself when it is a multiple of 8, else g rounded up with pad_genes."""
    if g % 8 == 0:
        return g
    if not pad_genes:
        raise ValueError("the number of genes must be a multiple of 8 for the packed format (got %d)" % g)
    return (g + 7) // 8 * 8


def _zero_padded(C, gp):
    """C (n x g) with gp - g all-zero columns appended."""
    if C.shape[1] == gp:
        return C
    out = np.zeros((C.shape[0], gp), dtype=C.dtype)
    out[:, :C.shape[1]] = C
    return out


def _choose_format(counts, csr, bits, batch, chunk_rows, g):
    """The width pack_counts(counts, bits, batch) would choose (1 = sparse), from per-row statistics gathered chunk by
    chunk (the native escape counter; non-integer or negative counts raise)."""
    n = counts.shape[0]                                  # g: the stored width (pad genes hold no count)
    nnz = np.zeros(n, dtype=np.int64)
    per_row = np.zeros((3, n), dtype=np.int64)
    for r0 in range(0, n, chunk_rows):
        r1 = min(n, r0 + chunk_rows)
        m = counts[r0:r1]
        m = m.toarray() if csr else np.asarray(m)
        nnz[r0:r1] = np.count_nonzero(m, axis=1)
        per_row[:, r0:r1] = _escapes_native(m)
    if bits in ("sparse", "auto") and n > 0:
        if bits == "sparse" or _prefer_sparse(int(nnz.sum()), n * g):
            nib = np.zeros(n + 1, dtype=np.int64)
            np.cumsum((nnz + 1) // 2, out=nib[1:])
            if _worst_batch(nib, batch) <= _nibble_cap(batch, g):
                return "sparse"
            if bits == "sparse":
                raise ValueError("more than 50 % non-zero entries in a batch: use a dense width (bits=4)")
    return _choose_bits(per_row, n, g, batch)


def _prefer_sparse(nnz, size):
    """pack_counts' choice of the sparse over the dense formats: fewer than 45 % non-zeros, and 1 bit per entry + 4 bits
    per non-zero at least 20 % below the 4 bits per entry of the dense 4-bit width."""
    return nnz < 0.45 * size and size / 8.0 + nnz / 2.0 < 0.8 * size / 2.0


def _worst_batch(indptr, batch):
    """Largest span of a CSR indptr over consecutive batches of `batch` rows (0 without a batch)."""
    n = len(indptr) - 1
    if not batch or n <= 0:
        return 0
    return int(np.max(np.diff(indptr[np.r_[np.arange(0, n, batch), n]])))


def _nibble_cap(batch, g):
    """Bytes of non-zero codes a streamed batch of the sparse format may carry (50 % non-zeros; engine.cu nib_cap)."""
    return batch * g // 4 + 64 if batch else 0


def _escapes_native(C, threads=0):
    """int64 [3][rows]: entries of each row that need the overflow list at 4, 8 and 16 bits (dca_count_escapes)."""
    from . import _lib
    lib = _lib.load()
    if C.dtype not in _NATIVE_DTYPES:
        C = C.astype(np.float64 if C.dtype.kind == "f" else np.int64)
    C = np.ascontiguousarray(C)
    n, g = C.shape
    per_row = np.zeros((3, n), dtype=np.int64)
    if n == 0:
        return per_row
    st = lib.dca_count_escapes(C.ctypes.data, _NATIVE_DTYPES[C.dtype], n, g, g, per_row.ctypes.data, int(threads))
    if st != 0:
        msg = lib.dca_last_error().decode("utf-8", "replace")
        raise ValueError("counts must be non-negative integers" if "non-negative" in msg else msg)
    return per_row


def fit_batches(pc, batch, ovf_cap, nib_cap, chunk_rows=16384):
    """``pc`` when every batch of ``batch`` consecutive rows carries at most ``ovf_cap`` overflow entries (and, in the
    sparse format, at most ``nib_cap`` bytes of non-zero codes) -- what a streaming engine can stage
    (DeviceEngine.stream_capacity); otherwise the same counts repacked, chunk by chunk, at the narrowest dense width
    whose batches fit.  The counts are the same, so the expanded Y and X are the same bits."""
    if (_worst_batch(pc.indptr, batch) <= ovf_cap
            and (pc.bits != 1 or _worst_batch(pc.nib_indptr, batch) <= nib_cap)):
        return pc
    n = pc.n_rows
    per_row = np.zeros((3, n), dtype=np.int64)
    for r0 in range(0, n, chunk_rows):
        r1 = min(n, r0 + chunk_rows)
        per_row[:, r0:r1] = _escapes_native(unpack_counts(pc.take_rows(np.arange(r0, r1))))
    for w, b in enumerate((4, 8, 16)):
        ptr = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(per_row[w], out=ptr[1:])
        if _worst_batch(ptr, batch) <= ovf_cap:
            out = concat_packed([pack_counts(unpack_counts(pc.take_rows(np.arange(r0, min(n, r0 + chunk_rows)))), b)
                                 for r0 in range(0, n, chunk_rows)])
            out.genes = pc.genes
            return out
    raise ValueError("a batch of %d rows holds more than %d counts >= 65535 (the overflow capacity of one streamed batch)"
                     % (batch, ovf_cap))


OVERFLOW_ENTRY = np.dtype([("gene", "<i4"), ("count", "<f4")])


_NATIVE_DTYPES = {np.dtype(np.float32): 0, np.dtype(np.float64): 1, np.dtype(np.uint16): 2, np.dtype(np.int32): 3,
                  np.dtype(np.int64): 4}


def _choose_bits(per_row, n, g, batch):
    """Smallest total bytes among 4 / 8 / 16 bits whose per-batch overflow fits the device staging capacity.
    per_row: int64 [3][n] escapes per row at each width."""
    best = None
    for w, b in enumerate((4, 8, 16)):
        pr = per_row[w]
        if batch:
            cap = max(4096, batch * g // 32)
            worst = max(int(pr[i:i + batch].sum()) for i in range(0, max(n, 1), batch)) if n else 0
            if worst > cap:
                continue
        total = n * g * b / 8.0 + 8.0 * float(pr.sum())
        if best is None or total < best[0]:
            best = (total, b)
    if best is None:
        raise ValueError("no packing width fits the overflow capacity")
    return best[1]


def _pack_sparse_native(C, batch, threads=0):
    """Multi-threaded packer of the library (dca_sparse_counts + dca_pack_sparse)."""
    from . import _lib
    lib = _lib.load()
    if C.dtype not in _NATIVE_DTYPES:
        C = C.astype(np.float64 if C.dtype.kind == "f" else np.int64)
    C = np.ascontiguousarray(C)
    n, g = C.shape
    if g > 65536:
        raise ValueError("the sparse format supports at most 65536 genes")
    dt = _NATIVE_DTYPES[C.dtype]
    nnz = np.zeros(n, dtype=np.int64); esc = np.zeros(n, dtype=np.int64)
    st = lib.dca_sparse_counts(C.ctypes.data, dt, n, g, g, nnz.ctypes.data, esc.ctypes.data, int(threads))
    if st != 0:
        msg = lib.dca_last_error().decode("utf-8", "replace")
        raise ValueError("counts must be non-negative integers" if "non-negative" in msg else msg)
    nib_indptr = np.zeros(n + 1, dtype=np.int64); np.cumsum((nnz + 1) // 2, out=nib_indptr[1:])
    indptr = np.zeros(n + 1, dtype=np.int64); np.cumsum(esc, out=indptr[1:])
    if _worst_batch(nib_indptr, batch) > _nibble_cap(batch, g):
        raise ValueError("more than 50 % non-zero entries in a batch: use a dense width (bits=4)")
    bitmap = np.empty((n, g // 8), dtype=np.uint8)
    nibbles = np.zeros(int(nib_indptr[-1]) + 16, dtype=np.uint8)
    entries = np.empty(int(indptr[-1]), dtype=OVERFLOW_ENTRY)
    _lib.check(lib.dca_pack_sparse(C.ctypes.data, dt, n, g, g, bitmap.ctypes.data, nib_indptr.ctypes.data, nibbles.ctypes.data,
                                   indptr.ctypes.data, entries.ctypes.data if len(entries) else None, int(threads)), "dca_pack_sparse")
    return PackedCounts(bitmap, 1, g, indptr, entries, nib_indptr, nibbles)


def _pack_sparse(C, batch):
    """NumPy statement of the sparse format (dca_stream_begin_sparse, include/dca_b200.h)."""
    n, g = C.shape
    if g > 65536:
        raise ValueError("the sparse format supports at most 65536 genes")
    nz = C != 0
    bitmap = np.packbits(nz, axis=1, bitorder="little")                    # [n, g/8]
    rows, cols = np.nonzero(nz)                                             # row-major: by row, then gene
    vals = C[rows, cols]
    codes = np.minimum(vals, 15).astype(np.uint8)
    cnt = np.bincount(rows, minlength=n).astype(np.int64)
    nib_indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum((cnt + 1) // 2, out=nib_indptr[1:])                          # every row starts on a byte boundary
    first = np.zeros(n + 1, dtype=np.int64); np.cumsum(cnt, out=first[1:])
    k = np.arange(rows.shape[0], dtype=np.int64) - first[rows]             # index of the code inside its row
    byte = nib_indptr[rows] + (k >> 1)
    nibbles = np.zeros(int(nib_indptr[-1]) + 16, dtype=np.uint8)           # + slack: the device reads whole bytes
    even = (k & 1) == 0
    nibbles[byte[even]] = codes[even]
    nibbles[byte[~even]] |= (codes[~even] << 4).astype(np.uint8)
    over = vals >= 15
    orow, ocol = rows[over], cols[over]
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(orow, minlength=n), out=indptr[1:])
    entries = np.empty(orow.shape[0], dtype=OVERFLOW_ENTRY)
    entries["gene"] = ocol; entries["count"] = vals[over]
    if _worst_batch(nib_indptr, batch) > _nibble_cap(batch, g):
        raise ValueError("more than 50 % non-zero entries in a batch: use a dense width (bits=4)")
    return PackedCounts(np.ascontiguousarray(bitmap), 1, g, indptr, entries, nib_indptr, nibbles)


def pack_counts(counts, bits="auto", batch=None, native=True, threads=0, pad_genes=False):
    """Pack an integer-valued count matrix (cells x genes, any numeric dtype) into `bits` bits per entry.

    Counts >= 2**bits - 1 are stored as the escape value 2**bits - 1 and listed (row-sorted) in the overflow
    CSR: indptr int64[n_rows+1], entries {int32 gene, float32 count}.  bits='auto' picks the width in
    (4, 8, 16) with the fewest total bytes whose per-batch overflow (when `batch` is given) stays under
    batch*genes/32 entries (the device staging capacity).  native=True runs the multi-threaded packer of the
    library (dca_count_escapes / dca_pack_counts); native=False is the NumPy statement of the same format.
    The gene count must be a multiple of 8; with pad_genes=True any gene count packs as its zero-padded form: the
    bytes of the matrix with all-zero columns appended up to the next multiple of 8 (PackedCounts.genes records the
    gene count, n_genes the stored width)."""
    C = np.asarray(counts)
    if C.ndim != 2:
        raise ValueError("counts must be a 2-d matrix")
    genes = C.shape[1]
    C = _zero_padded(C, _packed_width(genes, pad_genes))
    pc = _pack_padded(C, bits, batch, native, threads)
    pc.genes = genes
    return pc


def _pack_padded(C, bits, batch, native, threads):
    n, g = C.shape
    if bits not in ("auto", "sparse", "dense") and bits not in (4, 8, 16):
        raise ValueError("bits must be 4, 8, 16, 'sparse', 'dense' (best dense width) or 'auto' (smallest of all)")
    if bits in ("sparse", "auto") and n > 0:
        if not native and C.size and (C.min() < 0 or np.any(C != np.floor(C))):
            raise ValueError("counts must be non-negative integers")
        nnz = int(np.count_nonzero(C))
        # sparse: 1 bit per entry + 4 bits per non-zero (+ 8 B per count >= 15); dense 4-bit: 4 bits per entry
        if bits == "sparse" or _prefer_sparse(nnz, C.size):
            try:
                return _pack_sparse_native(C, batch, threads) if native else _pack_sparse(C, batch)
            except ValueError:
                if bits == "sparse":
                    raise
    if bits in ("sparse", "dense"):
        bits = "auto"
    if native and n > 0:
        return _pack_counts_native(C, bits, batch, threads)
    if C.size and (C.min() < 0 or np.any(C != np.floor(C))):
        raise ValueError("counts must be non-negative integers")
    if bits == "auto":
        per_row = np.stack([(C >= (1 << b) - 1).sum(1) for b in (4, 8, 16)]).astype(np.int64)
        bits = _choose_bits(per_row, n, g, batch)
    esc = (1 << bits) - 1
    over = C >= esc
    base = np.where(over, esc, C).astype(np.uint16 if bits == 16 else np.uint8)
    if bits == 4:
        packed = (base[:, 0::2] | (base[:, 1::2] << 4)).astype(np.uint8)
    else:
        packed = base
    rows, cols = np.nonzero(over)                     # row-major order: sorted by row, then gene
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=indptr[1:])
    entries = np.empty(rows.shape[0], dtype=OVERFLOW_ENTRY)
    entries["gene"] = cols
    entries["count"] = C[rows, cols]
    return PackedCounts(np.ascontiguousarray(packed), bits, g, indptr, entries)


def _pack_counts_native(C, bits, batch, threads):
    from . import _lib
    lib = _lib.load()
    if C.dtype not in _NATIVE_DTYPES:
        C = C.astype(np.float64 if C.dtype.kind == "f" else np.int64)
    C = np.ascontiguousarray(C)
    n, g = C.shape
    dt = _NATIVE_DTYPES[C.dtype]
    per_row = _escapes_native(C, threads)
    if bits == "auto":
        bits = _choose_bits(per_row, n, g, batch)
    w = (4, 8, 16).index(bits)
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(per_row[w], out=indptr[1:])
    packed = np.empty((n, g // 2) if bits == 4 else (n, g), dtype=np.uint16 if bits == 16 else np.uint8)
    entries = np.empty(int(indptr[-1]), dtype=OVERFLOW_ENTRY)
    _lib.check(lib.dca_pack_counts(C.ctypes.data, dt, n, g, g, bits, packed.ctypes.data, indptr.ctypes.data,
                                   entries.ctypes.data if len(entries) else None, int(threads)), "dca_pack_counts")
    return PackedCounts(packed, bits, g, indptr, entries)


def unpack_counts(pc: PackedCounts):
    """Inverse of pack_counts (float32 matrix) -- the host statement of what the device expansion produces."""
    if pc.bits == 1:
        nz = np.unpackbits(pc.packed, axis=1, bitorder="little")[:, :pc.n_genes].astype(bool)
        out = np.zeros((pc.n_rows, pc.n_genes), dtype=np.float32)
        rows, cols = np.nonzero(nz)
        cnt = np.bincount(rows, minlength=pc.n_rows).astype(np.int64)
        first = np.zeros(pc.n_rows + 1, dtype=np.int64); np.cumsum(cnt, out=first[1:])
        k = np.arange(rows.shape[0], dtype=np.int64) - first[rows]
        b = pc.nibbles[pc.nib_indptr[rows] + (k >> 1)]
        out[rows, cols] = np.where(k & 1, b >> 4, b & 0xF)
        orow = np.repeat(np.arange(pc.n_rows), np.diff(pc.indptr))
        out[orow, pc.entries["gene"]] = pc.entries["count"]
        return out
    if pc.bits == 4:
        out = np.empty((pc.n_rows, pc.n_genes), dtype=np.float32)
        out[:, 0::2] = pc.packed & 0xF
        out[:, 1::2] = pc.packed >> 4
    else:
        out = pc.packed.astype(np.float32)
    rows = np.repeat(np.arange(pc.n_rows), np.diff(pc.indptr))
    out[rows, pc.entries["gene"]] = pc.entries["count"]
    return out
