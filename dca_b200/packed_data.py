"""A count matrix packed on the GPU and kept packed in device memory for training and prediction.

``PackedDeviceDataset.from_counts`` uploads the raw counts in row chunks twice: once for the library sizes, gene totals
and the per-row statistics the format is chosen from (``dca_count_totals_rows`` + ``dca_pack_count_rows``), once to pack
them into dataset-wide device arrays at offsets from device prefix sums (``dca_pack_rows_device``).  The formats are
those of io.pack_counts: about 0.3 bytes per entry in the sparse format at 35 % non-zeros, against 6 - 8 bytes for the
fp32 Y and the X of the resident ``device_data.DeviceDataset``.  The gene moments are computed from chunks expanded from
the packed arrays, with no further host traffic.  Every training, validation and predict batch is then expanded by row
index on the device (``dca_packed_train_step`` ... in include/dca_b200.h): nothing crosses PCIe per step and the rows are
reshuffled every epoch as Keras does.

On the same counts every result is bit-identical to ``DeviceDataset``: size factors, n_counts, gene totals, mean, std
and every X the training step and predict read.  The counts must be non-negative integers.  With ``pad_genes=True``
any gene count is accepted, before and after filtering: the rows are packed at the gene count rounded up to a multiple
of 8, the pad genes all zero (the bytes of io.pack_rows(..., pad_genes=True)), and the statistics, the expansion and
the model see the real genes only.  With the default ``pad_genes=False`` the gene count after filtering must be a
multiple of 8.
"""
from __future__ import annotations

import contextlib
import ctypes as C
from types import SimpleNamespace

import numpy as np
import torch

from . import _lib
from . import io as dio
from ._lib import check
from .device_data import (_counts_matrix, _Dataset, _device, _is_csr, _resident_fit, _size_factors, _stream, _X_DTYPES,
                          preprocess_flags)
from .stream_data import _chunk_rows, _moments, _pad_stats, _totals

_ESC_ROW = {1: 1, 4: 1, 8: 2, 16: 3}           # row of the count-pass statistics holding a width's overflow entries


def choose_format(nnz, per_row, n, g, bits="auto"):
    """The width io.pack_rows(counts, bits, batch=None) packs a matrix with (1: the sparse format), from its total
    non-zeros ``nnz`` and ``per_row`` (int64 [3][n]: entries >= 15, 255, 65535 per row), with the same errors."""
    if bits not in ("auto", "sparse", "dense") and bits not in (4, 8, 16):
        raise ValueError("bits must be 4, 8, 16, 'sparse', 'dense' (best dense width) or 'auto' (smallest of all)")
    if bits in ("sparse", "auto") and n > 0:
        if bits == "sparse" or dio._prefer_sparse(int(nnz), n * g):
            if g <= 65536:
                return 1
            if bits == "sparse":
                raise ValueError("the sparse format supports at most 65536 genes")
    if bits in (4, 8, 16):
        return bits
    return dio._choose_bits(per_row, n, g, None)


class _HostChunks:
    """fn(r0, n, Y) for consecutive row chunks of a host matrix (dense, or scipy CSR densified on the device by
    dca_counts_csr_to_dense: a CSR matrix is never dense on the host as a whole); Y = the chunk's fp32 counts, ``ld``
    wide: the gene count rounded up to a multiple of 8, whose pad columns stay zero (the packer's count pass reads whole
    16-byte groups)."""

    def __init__(self, counts, dev):
        self.counts, self.dev, self.csr = counts, dev, _is_csr(counts)
        self.N, self.G = (int(s) for s in counts.shape)
        self.ld = (self.G + 7) // 8 * 8

    def __call__(self, chunk, fn):
        Y = torch.zeros((chunk, self.ld), dtype=torch.float32, device=self.dev)
        for r0 in range(0, self.N, chunk):
            r1 = min(self.N, r0 + chunk)
            self._upload(r0, r1, Y)
            fn(r0, r1 - r0, Y)

    def _upload(self, r0, r1, Y):
        if not self.csr:
            Y[: r1 - r0, : self.G].copy_(torch.from_numpy(np.ascontiguousarray(self.counts[r0:r1], dtype=np.float32)))
            return
        m = self.counts[r0:r1]
        if not m.has_canonical_format:
            m = m.copy()
            m.sum_duplicates()
            m.sort_indices()
        if m.nnz and (int(m.indices.min()) < 0 or int(m.indices.max()) >= self.G):
            raise ValueError("CSR column index out of range")
        indptr = torch.from_numpy(np.ascontiguousarray(m.indptr, dtype=np.int64)).to(self.dev)
        indices = torch.from_numpy(np.ascontiguousarray(m.indices, dtype=np.int32)).to(self.dev)
        data = torch.from_numpy(np.ascontiguousarray(m.data, dtype=np.float32)).to(self.dev)
        check(_lib.load().dca_counts_csr_to_dense(indptr.data_ptr(), indices.data_ptr() if m.nnz else None,
                                                  data.data_ptr() if m.nnz else None, r1 - r0, self.G, Y.data_ptr(),
                                                  self.ld, _stream(self.dev)), "dca_counts_csr_to_dense")


class PackedDeviceDataset(_Dataset):
    """Raw counts packed in device memory (``packed``, ``ovf_indptr``, ``entries`` and, in the sparse format (bits 1),
    ``nib_indptr`` and ``nibbles``: the arrays of io.PackedCounts with absolute offsets), their fp64 row totals
    ``n_counts`` and ``rows``, the int32 storage rows of the cells this dataset covers, in order (``take`` composes it,
    as DeviceDataset.take does).  The statistics and masks are those of StreamedDataset (``n_counts_host``,
    ``size_factors_host``, ``mean``, ``std``, ``median``, ``flags``, ``gene_mask``, ``cell_mask``, ``sf_mask``,
    ``gene_totals_host``, ``input_gene_totals``, ``n_bad``), so io.apply_device_normalize(adata, pd, ..., set_x=False)
    mutates an AnnData the same way.  Training, validation and prediction expand every batch from the packed arrays by
    row index with the exact transform (the interface of device_data._Dataset, keyword ``packed_data``); training
    reshuffles the rows every epoch as DeviceDataset does."""
    kind = "packed_data"

    @property
    def n(self) -> int:
        return int(self.rows.numel())

    @property
    def n_genes(self) -> int:
        return int(getattr(self, "genes", self.desc.genes))        # the real genes; desc.genes is the stored width

    @classmethod
    def from_counts(cls, counts, device=None, x_dtype="float32", size_factors=True, logtrans_input=True,
                    normalize_input=True, filter_min_counts=False, bits="auto", chunk_rows=None, pad_genes=False):
        """counts: cells x genes, a dense ndarray or a scipy.sparse CSR matrix of raw counts.  The filtering and
        normalisation steps of io.normalize with the same flags; x_dtype 'float32' | 'bfloat16' (the X the training
        step reads); bits: the packing as io.pack_rows(counts, bits) chooses it ('auto', 'sparse', 'dense', 4, 8, 16);
        chunk_rows: rows per uploaded / expanded chunk (default: 256 MB of fp32 counts); pad_genes: accept a gene count
        off a multiple of 8, before and after the gene filter (stored zero-padded to the next multiple of 8,
        ``desc.genes``; ``genes`` and every result cover the real genes)."""
        lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.DcaError("PackedDeviceDataset needs a CUDA device (H100); there is no CPU fallback")
        dev, xdt = _device(device), _X_DTYPES[x_dtype]
        counts = _counts_matrix(counts)
        N0, G0 = (int(s) for s in counts.shape)
        if G0 % 8 != 0 and not pad_genes:
            raise ValueError("the packed format needs a gene count that is a multiple of 8 (got %d)" % G0)
        choose_format(0, np.zeros((3, 0), np.int64), 0, dio._packed_width(G0, pad_genes), bits)          # reject a bad `bits` before any work
        host = _HostChunks(counts, dev)
        with torch.cuda.device(dev):
            # pass 1 over the host counts: totals (the chunked column pass) and the per-row statistics of the packer
            stats = torch.empty((5, N0), dtype=torch.int64, device=dev)

            def upload_and_count(chunk, fn):
                def both(r0, n, Y):                          # (the pad columns of a ragged chunk hold no count)
                    check(lib.dca_pack_count_rows(Y.data_ptr(), host.ld, n, host.ld, stats.data_ptr() + 8 * r0, N0,
                                                  _stream(dev)), "dca_pack_count_rows")
                    fn(r0, n, Y[:, :G0])
                host(chunk, both)
            nc, gene_tot, n_bad = _totals(SimpleNamespace(n_rows=N0, n_genes=G0), dev, chunk_rows, upload_and_count)
            st = stats.cpu().numpy()
            if st[4].any():
                raise ValueError("counts must be non-negative integers")
            input_gene_totals, input_n_bad = gene_tot, n_bad
            # filters (dca/io.py:90-92, normalize_per_cell): a dropped gene or cell holds no non-zero and no escape, so
            # the kept rows' statistics stand; the totals are recomputed from the packed rows as the other paths do
            gene_mask = np.ones(G0, bool)
            cell_mask = np.ones(N0, bool)
            if filter_min_counts:
                gene_mask = gene_tot >= 1
                if not gene_mask.all() and gene_mask.sum() % 8 != 0 and not pad_genes:
                    raise ValueError("filtering leaves %d genes; the packed format needs a multiple of 8 "
                                     "(filter the genes before, or use the resident device path)" % gene_mask.sum())
                cell_mask = nc >= 1
            keep = np.flatnonzero(cell_mask)
            sf_mask = np.ones(keep.size, bool)
            if size_factors:
                sf_mask = nc[keep] >= 1
                keep = keep[sf_mask]
            cols = np.flatnonzero(gene_mask)
            N, G = int(keep.size), int(cols.size)
            if N < 1:
                raise ValueError("no cell with counts is left")
            pd = cls._pack(lib, host, st, keep, cols, gene_mask.all(), bits, dev, chunk_rows)
            pd.x_dtype, pd.device = xdt, dev
            filtered = N != N0 or G != G0
            if filtered:
                nc, gene_tot, _ = _totals(SimpleNamespace(n_rows=N, n_genes=G), dev, chunk_rows, pd._chunks)
            med, sf_h = _size_factors(nc, size_factors)
            flags = preprocess_flags(size_factors, logtrans_input, normalize_input)
            pd.n_counts = torch.from_numpy(np.ascontiguousarray(nc, dtype=np.float64)).to(dev)
            pd.desc.n_counts = pd.n_counts.data_ptr()
            mean, std = _moments(SimpleNamespace(n_rows=N, n_genes=G), nc, med, flags, dev, chunk_rows, pd._chunks)
        pd.n_counts_host, pd.size_factors_host, pd.mean, pd.std, pd.median, pd.flags = nc, sf_h, mean, std, med, flags
        Gp = int(pd.desc.genes)                          # the expansion reads per-gene statistics at the stored width
        pd._mean_d = torch.from_numpy(_pad_stats(mean, Gp, 0.0)).to(dev)
        pd._std_d = torch.from_numpy(_pad_stats(std, Gp, 1.0)).to(dev)
        pd.gene_totals_host, pd.input_gene_totals, pd.n_bad = gene_tot, input_gene_totals, input_n_bad
        pd.gene_mask, pd.cell_mask, pd.sf_mask = gene_mask, cell_mask, sf_mask
        return pd

    @classmethod
    def _pack(cls, lib, host, st, keep, cols, all_genes, bits, dev, chunk_rows):
        """Pass 2 over the host counts: the kept rows ``keep`` and genes ``cols`` packed into new device arrays, at the
        stored width Gp (the gene count rounded up to a multiple of 8; the pad genes hold no count, so the per-row
        statistics ``st`` stand for the padded rows)."""
        N0, G0 = host.N, host.G
        N, G = int(keep.size), int(cols.size)
        Gp = (G + 7) // 8 * 8
        w = choose_format(int(st[0, keep].sum()), st[1:4, keep], N, Gp, bits)
        keep_d = torch.from_numpy(keep).to(dev)
        pd = cls.__new__(cls)
        pd.bits, pd.genes = w, G
        row_bytes = Gp // 8 if w == 1 else Gp * w // 8
        pd.packed = torch.empty(N * row_bytes, dtype=torch.uint8, device=dev)
        pd.ovf_indptr = torch.zeros(N + 1, dtype=torch.int64, device=dev)
        pd.ovf_indptr[1:] = torch.cumsum(torch.from_numpy(st[_ESC_ROW[w]]).to(dev)[keep_d], 0)
        n_ovf = int(pd.ovf_indptr[-1].item())
        pd.entries = torch.empty(max(n_ovf, 1) * 8, dtype=torch.uint8, device=dev)
        max_nib = 0
        if w == 1:
            nnz = torch.from_numpy(st[0]).to(dev)[keep_d]
            pd.nib_indptr = torch.zeros(N + 1, dtype=torch.int64, device=dev)
            pd.nib_indptr[1:] = torch.cumsum((nnz + 1) // 2, 0)
            pd.nibbles = torch.zeros(int(pd.nib_indptr[-1].item()) + 16, dtype=torch.uint8, device=dev)   # + slack
            max_nib = int(((st[0, keep] + 1) // 2).max())
        else:
            pd.nib_indptr = pd.nibbles = None
        pd.rows = torch.arange(N, dtype=torch.int32, device=dev)
        pd.desc = _lib.PackedCountsDesc(
            C.sizeof(_lib.PackedCountsDesc), w, N, Gp, max_nib, pd.packed.data_ptr(),
            pd.ovf_indptr.data_ptr() if n_ovf else None, pd.entries.data_ptr() if n_ovf else None,
            pd.nib_indptr.data_ptr() if w == 1 else None, pd.nibbles.data_ptr() if w == 1 else None, None)
        cols_d = None if all_genes else torch.from_numpy(cols.astype(np.int32)).to(dev)
        chunk = min(N0, chunk_rows or _chunk_rows(G0))
        # the kept rows and genes of a chunk, Gp wide: the pad columns are zeroed once and never written
        sel = (torch.zeros((chunk, Gp), dtype=torch.float32, device=dev)
               if (cols_d is not None or N != N0 or Gp != G) else None)

        def pack(r0, n, Y):
            a, b = np.searchsorted(keep, [r0, r0 + n])
            if b == a:
                return
            src = Y
            if sel is not None:                          # the kept rows and genes of the chunk (dca_gather_counts)
                local = torch.from_numpy((keep[a:b] - r0).astype(np.int32)).to(dev)
                check(lib.dca_gather_counts(Y.data_ptr(), host.ld, local.data_ptr(), int(b - a),
                                            None if cols_d is None else cols_d.data_ptr(), G, sel.data_ptr(), Gp,
                                            _stream(dev)), "dca_gather_counts")
                src = sel
            check(lib.dca_pack_rows_device(src.data_ptr(), src.stride(0), int(b - a), int(a), C.byref(pd.desc),
                                           _stream(dev)),
                  "dca_pack_rows_device")
        host(chunk, pack)
        return pd

    def _chunks(self, chunk, fn):
        """fn(r0, n, Y) for consecutive row chunks of every storage row, Y expanded from the packed arrays (the
        statistics passes read the counts from here: no second host upload); Y holds the real genes, a view with row
        stride desc.genes that drops the pad genes."""
        lib = _lib.load()
        dev, G, N = self.device, int(self.desc.genes), int(self.desc.n_rows)
        Y = torch.empty((chunk, G), dtype=torch.float32, device=dev)
        X = torch.empty((chunk, G), dtype=torch.bfloat16, device=dev)
        sf = torch.empty(chunk, dtype=torch.float32, device=dev)
        zero, one = torch.zeros(G, dtype=torch.float64, device=dev), torch.ones(G, dtype=torch.float64, device=dev)
        for r0 in range(0, N, chunk):
            n = min(chunk, N - r0)
            r = torch.arange(r0, r0 + n, dtype=torch.int32, device=dev)
            check(lib.dca_expand_rows_exact(C.byref(self.desc), r.data_ptr(), n, 1.0, 0, zero.data_ptr(), one.data_ptr(),
                                            Y.data_ptr(), X.data_ptr(), _lib.BF16, sf.data_ptr(), _stream(dev)),
                  "dca_expand_rows_exact")
            fn(r0, n, Y[:, :self.n_genes])

    # ------------------------------------------------------------------ views
    def take(self, mask_or_index):
        """The cells ``mask_or_index`` (a boolean mask over this dataset's cells or integer positions) selects, in
        that order: only ``rows`` (and the host per-cell arrays) are composed, no packed byte is copied."""
        idx = self._positions(mask_or_index)
        pd = PackedDeviceDataset.__new__(PackedDeviceDataset)
        pd.__dict__.update(self.__dict__)
        pd.rows = self.rows[torch.from_numpy(idx).to(self.device)].contiguous()
        pd.n_counts_host = self.n_counts_host[idx]
        pd.size_factors_host = self.size_factors_host[idx]
        return pd

    def expand(self):
        """(Y, X, sf) of this dataset's cells on the device, expanded by row index (dca_expand_rows_exact): the rows of
        a DeviceDataset's Y, X and sf for the same cells (expanded at the stored width, returned over the real genes)."""
        n, G = self.n, int(self.desc.genes)
        Y = torch.empty((n, G), dtype=torch.float32, device=self.device)
        X = torch.empty((n, G), dtype=self.x_dtype, device=self.device)
        sf = torch.empty(n, dtype=torch.float32, device=self.device)
        check(_lib.load().dca_expand_rows_exact(C.byref(self.desc), self.rows.data_ptr(), n, self.median, self.flags,
                                                self._mean_d.data_ptr(), self._std_d.data_ptr(), Y.data_ptr(),
                                                X.data_ptr(), _lib.BF16 if self.x_dtype == torch.bfloat16 else _lib.F32,
                                                sf.data_ptr(), _stream(self.device)), "dca_expand_rows_exact")
        if G != self.n_genes:
            Y, X = Y[:, :self.n_genes].contiguous(), X[:, :self.n_genes].contiguous()
        torch.cuda.synchronize(self.device)
        return Y, X, sf

    def host_packed(self):
        """Host copy of the packed arrays as an io.PackedCounts over every storage row (the bytes io.pack_rows writes
        for the same counts, pad genes included)."""
        N, G = int(self.desc.n_rows), int(self.desc.genes)
        packed = self.packed.cpu().numpy()
        if self.bits == 16:
            packed = packed.view(np.uint16)
        packed = packed.reshape(N, -1)
        indptr = self.ovf_indptr.cpu().numpy()
        entries = self.entries.cpu().numpy()[: 8 * int(indptr[-1])].view(dio.OVERFLOW_ENTRY)
        if self.bits != 1:
            return dio.PackedCounts(packed, self.bits, G, indptr, entries, genes=self.n_genes)
        return dio.PackedCounts(packed, 1, G, indptr, entries, self.nib_indptr.cpu().numpy(), self.nibbles.cpu().numpy(),
                                genes=self.n_genes)

    def device_bytes(self) -> int:
        """Device memory the dataset holds: packed arrays, row totals and the row map."""
        ts = [self.packed, self.ovf_indptr, self.entries, self.nib_indptr, self.nibbles, self.n_counts, self.rows,
              self._mean_d, self._std_d]
        return sum(t.numel() * t.element_size() for t in ts if t is not None)

    # ------------------------------------------------------------------ training and prediction
    def _bind(self, eng):
        self._check_genes(eng)
        super()._bind(eng)
        eng.set_input_transform_exact(self.mean, self.std, self.median, self.flags)

    def _fit(self, eng, n_tr, batch, shuffle):
        return _resident_fit(eng, n_tr, self.n, batch, shuffle, lambda rows: eng.packed_train_step(self, rows),
                             lambda s, e: eng.packed_eval_step(self, self.rows[s:e]), self.rows)

    def _predictor(self, eng, bs):
        def run(i, s, e, b):
            eng.packed_predict(self, self.rows[s:e], mean=b.get("mean"), disp=b.get("disp"), pi=b.get("pi"),
                               latent=b.get("latent"))

        def theta(th):
            eng.packed_predict(self, self.rows[:1], disp=th)
        return run, theta, contextlib.nullcontext
