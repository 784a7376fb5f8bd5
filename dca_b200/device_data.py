"""A count matrix preprocessed in HBM and kept there for training and prediction.

``DeviceDataset.from_counts`` uploads the raw counts once, as the fp32 target matrix Y the training step reads, and
computes the library sizes, size factors, gene statistics and the normalised input X on the device
(csrc/preprocess.cu, ``dca_count_totals`` ... ``dca_normalize_write`` in include/dca_b200.h).  That is
dca/io.py:88-111 -- what ``io.normalize`` restates in NumPy on the host -- without a host copy of the normalised matrix.

The arithmetic is ``normalize_reference`` below.  Size factors and ``n_counts`` are bit-identical to ``io.normalize``;
X differs from it only where NumPy's float32 ``log1p`` differs from the float rounding of the double ``log1p`` (a few
ulp).
"""
from __future__ import annotations

import contextlib
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import check

PRE_SIZE_FACTORS, PRE_LOG1P, PRE_SCALE = 1, 2, 4
_UPLOAD_CHUNK_BYTES = 64 << 20


def preprocess_flags(size_factors=True, logtrans_input=True, normalize_input=True) -> int:
    return PRE_SIZE_FACTORS * bool(size_factors) | PRE_LOG1P * bool(logtrans_input) | PRE_SCALE * bool(normalize_input)


def normalize_reference(counts, size_factors=True, logtrans_input=True, normalize_input=True):
    """NumPy statement of the device arithmetic (no filtering; every cell needs a count when size_factors):
    sf64 = n_counts / median, q = float32(y / sf64), l = float32(log1p(float64(q))), fp64 gene
    mean and two-pass std (ddof=1; 1 for one cell or a constant gene), X = float32((l - mean) / std)."""
    Y = np.asarray(counts, dtype=np.float32)
    N = Y.shape[0]
    n_counts = Y.sum(axis=1, dtype=np.float64)
    med = np.median(n_counts)
    if size_factors:
        q = (Y / (n_counts / med)[:, None]).astype(np.float32)
        sf = (n_counts / med).astype(np.float32)
    else:
        q, sf = Y, np.ones(N, np.float32)
    l = np.log1p(q.astype(np.float64)).astype(np.float32) if logtrans_input else q
    if normalize_input:
        mean = l.mean(axis=0, dtype=np.float64)
        var = ((l - mean) ** 2).sum(axis=0) / (N - 1) if N > 1 else np.ones(Y.shape[1])
        std = np.sqrt(var)
        std[std == 0] = 1.0
        X = ((l - mean) / std).astype(np.float32)
    else:
        mean, std, X = np.zeros(Y.shape[1]), np.ones(Y.shape[1]), l
    return dict(n_counts=n_counts, size_factors=sf, mean=mean, std=std, X=X)


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _is_csr(counts):
    return hasattr(counts, "tocsr") and getattr(counts, "format", None) == "csr"


def _device(device):
    """The CUDA device a dataset is built on (None or an index-less 'cuda': the current one)."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    return torch.device("cuda", torch.cuda.current_device()) if dev.index is None else dev


_X_DTYPES = {"float32": torch.float32, "bfloat16": torch.bfloat16, torch.float32: torch.float32,
             torch.bfloat16: torch.bfloat16}


def _counts_matrix(counts):
    """counts as a scipy CSR matrix or a dense ndarray, checked to be a non-empty cells x genes matrix."""
    if not _is_csr(counts):
        counts = np.asarray(counts.toarray() if hasattr(counts, "toarray") else counts)
    if counts.ndim != 2 or counts.shape[0] < 1 or counts.shape[1] < 1:
        raise ValueError("counts must be a non-empty cells x genes matrix")
    if counts.shape[0] >= 2 ** 31:
        raise ValueError("at most 2**31 - 1 cells")
    return counts


def _size_factors(nc, size_factors):
    """(median, fp32 size factors) of the row totals nc: n_counts / median, or (1, ones) without size factors."""
    if not size_factors:
        return 1.0, np.ones(nc.shape[0], np.float32)
    med = float(np.median(nc))
    return med, (nc / med).astype(np.float32)


def build_dataset(counts, device=None, x_dtype="float32", stream=False, packed=False, batch=32, **flags):
    """The dataset of the device preprocessing of ``counts`` with the flags of io.normalize (``flags``): resident
    (DeviceDataset), out of core from packed host counts (stream: stream_data.StreamedDataset, packed for a training
    batch of ``batch`` rows) or packed in device memory (packed: packed_data.PackedDeviceDataset).  The packed kinds
    take any gene count, before and after the gene filter: their rows are stored zero-padded to a multiple of 8
    (pad_genes=True)."""
    if packed:
        from .packed_data import PackedDeviceDataset
        return PackedDeviceDataset.from_counts(counts, device, x_dtype, pad_genes=True, **flags)
    if stream:
        from .stream_data import StreamedDataset
        return StreamedDataset.from_counts(counts, device, x_dtype, batch=batch, pad_genes=True, **flags)
    return DeviceDataset.from_counts(counts, device, x_dtype, **flags)


def _one_dataset(device_data=None, stream_data=None, packed_data=None, stream=False):
    """The dataset given to train / predict / write_predictions through its keyword, or None (input from the AnnData).
    stream: train()'s host-streaming switch, which only a StreamedDataset goes with."""
    given = [d for d in (device_data, stream_data, packed_data) if d is not None]
    if packed_data is not None and (len(given) > 1 or stream):
        raise ValueError("packed_data is resident in HBM: it cannot be combined with stream, device_data or "
                         "stream_data")
    if len(given) > 1:
        raise ValueError("give device_data or stream_data, not both")
    if device_data is not None and stream:
        raise ValueError("device_data is resident in HBM: it cannot be combined with stream=True")
    return given[0] if given else None


def _resident_fit(eng, n_tr, n, batch, shuffle, step, evaluate, rows_map=None):
    """(epoch, validate) over n cells of which the first n_tr train: every epoch reshuffles the training rows with the
    global NumPy RNG as Keras does (np.random.shuffle of the index array) and runs step(rows) on each batch, rows an
    int32 device tensor of storage rows (positions mapped through rows_map when given), then update(); validate runs
    evaluate(s, e) over the held-out positions [n_tr, n) in batches.  check(positions of the batch's cells), when given,
    runs after every step, before its update."""
    def epoch(update, check=None):
        order = np.arange(n_tr)
        if shuffle:
            np.random.shuffle(order)
        order_d = torch.from_numpy(order.astype(np.int32)).to(eng.device)
        if rows_map is not None:
            order_d = rows_map[order_d.long()]
        for s in range(0, n_tr, batch):
            step(order_d[s:s + batch])
            if check:
                check(order[s:s + batch])
            update()

    def validate(check=None):
        for s in range(n_tr, n, batch):             # inference-mode BN over the held-out tail
            e = min(s + batch, n)
            evaluate(s, e)
            if check:
                check(np.arange(s, e))
    return epoch, validate


class _Dataset:
    """What train() and predict() know of a dataset kind, the same on DeviceDataset, stream_data.StreamedDataset and
    packed_data.PackedDeviceDataset:
      ``kind``: the keyword of train / predict / write_predictions that takes it and the suffix of its adata.uns key;
      ``_bind(eng)``: its checks against the engine and, where the kind needs it, the exact input transform;
      ``_fit(eng, n_tr, batch, shuffle)`` -> (epoch, validate): epoch(update) runs one epoch's training steps over the
      first n_tr cells, calling update() after each, and validate() the validation pass over the others; with a
      second argument check, both call check(positions of the batch's cells) after every step, before its update;
      ``_predictor(eng, bs)`` -> (run, theta, session): run(i, s, e, buffers) is the inference of batch i, cells
      [s, e), into the device buffers {"mean", "disp", "pi", "latent"} (any subset); theta(th) writes the per-gene
      dispersion of the const-disp types; a pass of run over the batches, and theta, go inside ``with session():``."""
    kind = None
    _on = "lives on"

    # the buffers are never written after from_counts: copies of an AnnData share them instead of duplicating memory
    def __copy__(self):
        return self

    def __deepcopy__(self, memo):
        return self

    def _positions(self, mask_or_index):
        """int64 positions in [0, n) of the cells ``mask_or_index`` selects (a boolean mask over this dataset's cells
        or integer positions, negative ones counting from the end), in that order."""
        idx = np.asarray(mask_or_index)
        if idx.dtype == bool:
            if idx.shape != (self.n,):
                raise ValueError("a mask must have one entry per cell (%d), got shape %s" % (self.n, idx.shape))
            idx = np.flatnonzero(idx)
        idx = idx.astype(np.int64).reshape(-1)
        if idx.size and (idx.min() < -self.n or idx.max() >= self.n):
            raise IndexError("cell index out of range for %d cells" % self.n)
        return idx % max(self.n, 1)

    def _cover(self, adata):
        if adata is not None and adata.n_obs != self.n:
            raise ValueError("%s covers %d cells, adata has %d" % (self.kind, self.n, adata.n_obs))

    def _check_genes(self, eng):
        if eng.n_in != self.n_genes or eng.n_out != self.n_genes:
            raise ValueError("%s has %d genes, the network %d inputs and %d outputs"
                             % (self.kind, self.n_genes, eng.n_in, eng.n_out))

    def _bind(self, eng):
        if self.device != eng.device:
            raise ValueError("%s %s %s, the network on %s" % (self.kind, self._on, self.device, eng.device))
        if self.x_dtype != eng.x_dtype:
            raise ValueError("%s X is %s, the network expects %s (network_kwds x_dtype)"
                             % (self.kind, self.x_dtype, eng.x_dtype))

    def host_size_factors(self) -> np.ndarray:
        return self.size_factors_host


class DeviceDataset(_Dataset):
    """Resident Y (fp32 raw counts), X (fp32 or bf16 normalised input), sf (fp32 size factors), n_counts, gene mean /
    std (fp64) and ``rows``, the int32 storage rows of the cells this dataset covers, in order.  ``take`` makes a
    dataset over a subset of them without copying a matrix.  ``y_cols`` names the input genes Y holds when it holds a
    subset of them (``with_output_genes``), otherwise None.  Training and prediction gather their batches through
    ``rows`` (the interface of _Dataset, keyword ``device_data``).

    Host copies of the per-cell and per-gene results (``n_counts_host``, ``size_factors_host``, ``gene_totals_host``)
    and the masks of the filtering steps (``gene_mask``, ``cell_mask``, ``sf_mask``) are what ``io.normalize`` needs to
    mutate an AnnData the way the host path does."""
    kind = "device_data"

    def __init__(self, Y, X, sf, n_counts, mean, std, rows, y_cols=None):
        self.Y, self.X, self.sf, self.n_counts, self.mean, self.std = Y, X, sf, n_counts, mean, std
        self.rows = rows
        self.y_cols = y_cols
        self.device = X.device

    @property
    def n(self) -> int:
        return int(self.rows.numel())

    @property
    def n_genes(self) -> int:
        return int(self.X.shape[1])

    @property
    def x_dtype(self):
        return self.X.dtype

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_counts(cls, counts, device=None, x_dtype="float32", size_factors=True, logtrans_input=True,
                    normalize_input=True, filter_min_counts=False):
        """counts: cells x genes, a dense ndarray or a scipy.sparse CSR matrix of raw counts.  The filtering and
        normalisation steps of io.normalize, with the same flags; x_dtype 'float32' | 'bfloat16'."""
        lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.DcaError("DeviceDataset needs a CUDA device (H100); there is no CPU fallback")
        dev, xdt = _device(device), _X_DTYPES[x_dtype]
        counts = _counts_matrix(counts)
        csr = _is_csr(counts)
        N, G = (int(s) for s in counts.shape)
        ws_bytes = C.c_size_t()
        check(lib.dca_preprocess_workspace_bytes(N, G, C.byref(ws_bytes)), "dca_preprocess_workspace_bytes")
        need = cls.device_bytes(counts, xdt, size_factors, filter_min_counts)
        free = torch.cuda.mem_get_info(dev)[0]
        if need > free:
            raise MemoryError("preprocessing %d x %d counts on %s needs %.2f GB of device memory and %.2f GB are free; "
                              "train from host memory instead: train(..., stream=True) or training_kwds={'stream': True} "
                              "(with 'preprocess': 'device', stream_data.StreamedDataset: out of core, same results)"
                              % (N, G, dev, need / 1e9, free / 1e9))
        with torch.cuda.device(dev):
            Y = torch.empty((N, G), dtype=torch.float32, device=dev)
            if csr:
                _upload_csr(lib, counts, Y, dev)
            else:
                _upload_dense(counts, Y)
            ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=dev)
            return cls._normalize(lib, Y, ws, dev, xdt, size_factors, logtrans_input, normalize_input, filter_min_counts)

    @staticmethod
    def device_bytes(counts, x_dtype="float32", size_factors=True, filter_min_counts=False) -> int:
        """Device memory from_counts needs for ``counts`` (cells x genes, dense or scipy CSR) with these flags."""
        xdt = _X_DTYPES[x_dtype]
        N, G = (int(s) for s in counts.shape)
        ws_bytes = C.c_size_t()
        check(_lib.load().dca_preprocess_workspace_bytes(N, G, C.byref(ws_bytes)), "dca_preprocess_workspace_bytes")
        need = N * G * (4 + xdt.itemsize) + ws_bytes.value + N * 24
        if filter_min_counts or size_factors:
            need += N * G * 4                          # a filtered copy of Y exists next to the unfiltered one
        if _is_csr(counts):
            need += counts.nnz * 8 + (N + 1) * 8
        return need

    @classmethod
    def _normalize(cls, lib, Y, ws, dev, xdt, size_factors, logtrans_input, normalize_input, filter_min_counts):
        N0, G0 = Y.shape
        n_counts, gene_tot, n_bad = _totals(lib, Y, ws, dev)
        input_gene_totals, input_n_bad = gene_tot.cpu().numpy(), int(n_bad.item())
        gene_mask = np.ones(G0, bool)
        cell_mask = np.ones(N0, bool)
        if filter_min_counts:                                            # dca/io.py:90-92
            gene_mask = input_gene_totals >= 1
            if not gene_mask.all():
                Y = _gather(lib, Y, None, np.flatnonzero(gene_mask), dev)
                n_counts, gene_tot, _ = _totals(lib, Y, ws, dev)
            cell_mask = n_counts.cpu().numpy() >= 1
            if not cell_mask.all():
                Y = _gather(lib, Y, np.flatnonzero(cell_mask), None, dev)
                n_counts, gene_tot, _ = _totals(lib, Y, ws, dev)
        nc = n_counts.cpu().numpy()
        sf_mask = np.ones(nc.shape[0], bool)
        if size_factors:                                                 # normalize_per_cell drops cells without counts
            sf_mask = nc >= 1
            if not sf_mask.all():
                Y = _gather(lib, Y, np.flatnonzero(sf_mask), None, dev)
                n_counts, gene_tot, _ = _totals(lib, Y, ws, dev)
                nc = n_counts.cpu().numpy()
        med, sf_h = _size_factors(nc, size_factors)
        N, G = Y.shape
        flags = preprocess_flags(size_factors, logtrans_input, normalize_input)
        s = _stream(dev)
        mean = torch.empty(G, dtype=torch.float64, device=dev)
        std = torch.empty(G, dtype=torch.float64, device=dev)
        check(lib.dca_log_moments(Y.data_ptr(), G, N, G, n_counts.data_ptr(), med, flags, mean.data_ptr(), std.data_ptr(),
                                  ws.data_ptr(), ws.numel(), s), "dca_log_moments")
        X = torch.empty((N, G), dtype=xdt, device=dev)
        check(lib.dca_normalize_write(Y.data_ptr(), G, N, G, n_counts.data_ptr(), med, flags, mean.data_ptr(),
                                      std.data_ptr(), X.data_ptr(), _lib.BF16 if xdt == torch.bfloat16 else _lib.F32, G, s),
              "dca_normalize_write")
        sf = torch.from_numpy(sf_h).to(dev)
        dd = cls(Y, X, sf, n_counts, mean, std, torch.arange(N, dtype=torch.int32, device=dev))
        dd.flags, dd.median = flags, med
        dd.n_counts_host, dd.size_factors_host = nc, sf_h
        dd.gene_totals_host = gene_tot.cpu().numpy()
        dd.input_gene_totals, dd.n_bad = input_gene_totals, input_n_bad
        dd.gene_mask, dd.cell_mask, dd.sf_mask = gene_mask, cell_mask, sf_mask
        return dd

    # ------------------------------------------------------------------ views
    def _derive(self, rows=None, Y=None, y_cols=None):
        dd = DeviceDataset.__new__(DeviceDataset)
        dd.__dict__.update(self.__dict__)
        if rows is not None:
            dd.rows = rows
        if Y is not None:
            dd.Y, dd.y_cols = Y, y_cols
        return dd

    def take(self, mask_or_index):
        """The cells ``mask_or_index`` (a boolean mask over this dataset's cells or integer positions) selects, in
        that order: only ``rows`` is composed, the matrices are shared."""
        sel = torch.from_numpy(self._positions(mask_or_index)).to(self.device)
        return self._derive(rows=self.rows[sel].contiguous())

    def with_output_genes(self, cols):
        """A dataset whose Y holds only the input genes ``cols`` (positions, in that order): the training target of
        ``output_subset`` / the CLI's --denoisesubset.  X is shared."""
        if self.y_cols is not None:
            raise ValueError("Y already holds a subset of the genes")
        cols = np.asarray(cols, dtype=np.int64).reshape(-1)
        if cols.size == 0 or cols.min() < 0 or cols.max() >= self.n_genes:
            raise IndexError("gene positions out of range for %d genes" % self.n_genes)
        Y = _gather(_lib.load(), self.Y, None, cols, self.device)
        return self._derive(Y=Y, y_cols=cols)

    def host_x(self) -> np.ndarray:
        """fp32 host copy of X over this dataset's cells."""
        return self.X[self.rows.long()].float().cpu().numpy()

    def host_size_factors(self) -> np.ndarray:
        return self.sf[self.rows.long()].cpu().numpy()

    # ------------------------------------------------------------------ training and prediction
    def _fit(self, eng, n_tr, batch, shuffle):
        return _resident_fit(eng, n_tr, self.n, batch, shuffle,
                             lambda rows: eng.train_step(self.X, self.Y, self.sf, rows=rows),
                             lambda s, e: eng.eval_step(self.X, self.Y, self.sf, rows=self.rows[s:e]), self.rows)

    def _predictor(self, eng, bs):
        def run(i, s, e, b):
            eng.predict(self.X, self.sf, rows=self.rows[s:e], mean=b.get("mean"), disp=b.get("disp"), pi=b.get("pi"),
                        latent=b.get("latent"))

        def theta(th):
            eng.predict(self.X, self.sf, rows=self.rows[:1], disp=th)
        return run, theta, contextlib.nullcontext


# ---------------------------------------------------------------------- helpers
def _upload_dense(counts, Y):
    """Row chunks of at most 64 MB through torch copies (pageable memory); integer counts are converted per chunk."""
    N, G = counts.shape
    step = max(1, _UPLOAD_CHUNK_BYTES // (4 * G))
    for r0 in range(0, N, step):
        r1 = min(N, r0 + step)
        Y[r0:r1].copy_(torch.from_numpy(np.ascontiguousarray(counts[r0:r1], dtype=np.float32)))


def _upload_csr(lib, counts, Y, dev):
    m = counts
    if not m.has_canonical_format:
        m = m.copy()
        m.sum_duplicates()
        m.sort_indices()
    N, G = Y.shape
    if m.nnz and (int(m.indices.min()) < 0 or int(m.indices.max()) >= G):
        raise ValueError("CSR column index out of range")
    indptr = torch.from_numpy(np.ascontiguousarray(m.indptr, dtype=np.int64)).to(dev)
    indices = torch.from_numpy(np.ascontiguousarray(m.indices, dtype=np.int32)).to(dev)
    data = torch.from_numpy(np.ascontiguousarray(m.data, dtype=np.float32)).to(dev)
    check(lib.dca_counts_csr_to_dense(indptr.data_ptr(), indices.data_ptr() if m.nnz else None,
                                      data.data_ptr() if m.nnz else None, N, G, Y.data_ptr(), G, _stream(dev)),
          "dca_counts_csr_to_dense")


def _totals(lib, Y, ws, dev):
    N, G = Y.shape
    n_counts = torch.empty(N, dtype=torch.float64, device=dev)
    gene_tot = torch.empty(G, dtype=torch.float64, device=dev)
    n_bad = torch.zeros(1, dtype=torch.int64, device=dev)
    check(lib.dca_count_totals(Y.data_ptr(), G, N, G, n_counts.data_ptr(), gene_tot.data_ptr(), n_bad.data_ptr(),
                               ws.data_ptr(), ws.numel(), _stream(dev)), "dca_count_totals")
    return n_counts, gene_tot, n_bad


def _gather(lib, Y, rows, cols, dev):
    """Y[rows][:, cols] into a new contiguous matrix (None: all)."""
    N, G = Y.shape
    r = None if rows is None else torch.from_numpy(np.ascontiguousarray(rows, dtype=np.int32)).to(dev)
    c = None if cols is None else torch.from_numpy(np.ascontiguousarray(cols, dtype=np.int32)).to(dev)
    nr = N if r is None else r.numel()
    nc = G if c is None else c.numel()
    out = torch.empty((nr, nc), dtype=torch.float32, device=dev)
    check(lib.dca_gather_counts(Y.data_ptr(), Y.stride(0), None if r is None else r.data_ptr(), nr,
                                None if c is None else c.data_ptr(), nc, out.data_ptr(), nc, _stream(dev)),
          "dca_gather_counts")
    return out
