"""A count matrix preprocessed out of core: packed raw counts in pinned host memory, statistics computed on the device.

``StreamedDataset.from_counts`` packs the raw counts once (io.pack_rows: about 0.2 bytes per entry in the sparse format,
0.5 in the 4-bit one) and computes library sizes, size factors and the gene mean / std from chunks of rows streamed
through the device (the chunked column passes ``dca_count_totals_rows`` ... ``dca_log_moments_finish`` of
include/dca_b200.h).  Training and prediction then stream batches from the same packed bytes and normalise them on the
device with the exact transform (``dca_set_input_transform_exact``).  Neither the normalised matrix nor the whole count
matrix ever exists in device memory, and no normalised matrix exists on the host.

On the same counts every result is bit-identical to ``device_data.DeviceDataset`` (dca/io.py:88-111 computed in HBM):
size factors, n_counts, gene totals, mean, std and every X the training step and predict read.  The counts must be
non-negative integers.  With ``pad_genes=True`` any gene count is accepted, before and after filtering: the rows are
packed at the gene count rounded up to a multiple of 8, the pad genes all zero (io.pack_rows(..., pad_genes=True)),
and the statistics, the expansion and the model see the real genes only.  With the default ``pad_genes=False`` the
gene count must be a multiple of 8.
"""
from __future__ import annotations

import contextlib
import ctypes as C

import numpy as np
import torch

from . import _lib
from . import io as dio
from ._lib import check
from .device_data import (PRE_SIZE_FACTORS, _counts_matrix, _Dataset, _device, _size_factors, _stream, _X_DTYPES,
                          preprocess_flags)

_CHUNK_BYTES = 256 << 20          # fp32 counts of one chunk of rows on the device


def pin_packed(pc, device_index=0):
    """Pinned host copies of a PackedCounts' arrays, made once and kept on the object (pc._pinned):
    (packed bytes, overflow indptr, overflow entry bytes[, nibble indptr, nibbles])."""
    from .hostmem import pin_near_gpu
    if getattr(pc, "_pinned", None) is None:          # cudaHostAlloc costs milliseconds: pin once per PackedCounts
        def pinned(a, view):
            return pin_near_gpu(np.ascontiguousarray(a).view(view), device_index)
        pc._pinned = (pinned(pc.packed, np.uint8), pinned(pc.indptr, np.int64),
                      pinned(pc.entries if len(pc.entries) else np.zeros(1, dtype=pc.entries.dtype), np.uint8))
        if pc.bits == 1:
            pc._pinned += (pinned(pc.nib_indptr, np.int64), pinned(pc.nibbles, np.uint8))
    return pc._pinned


class _DevicePack:
    """Device copies of rows [r0, r1) of a PackedCounts (any format), sized for the largest chunk it will hold."""

    def __init__(self, pc, dev, max_rows, max_entries, max_nib):
        rb = pc.packed.shape[1] * pc.packed.itemsize
        self.packed = torch.empty(max_rows * rb + 16, dtype=torch.uint8, device=dev)
        self.indptr = torch.empty(max_rows + 1, dtype=torch.int64, device=dev)
        self.entries = torch.empty(max(1, max_entries) * 8, dtype=torch.uint8, device=dev)
        if pc.bits == 1:
            self.nib_indptr = torch.empty(max_rows + 1, dtype=torch.int64, device=dev)
            self.nibbles = torch.empty(max_nib + 16, dtype=torch.uint8, device=dev)
        self.rb = rb

    def upload(self, pc, pins, r0, r1):
        """Asynchronous copies on the current stream (pins: pin_packed(pc)); returns (has_overflow, max row nibble bytes)."""
        n = r1 - r0
        self.packed[: n * self.rb].copy_(pins[0].reshape(-1)[r0 * self.rb: r1 * self.rb], non_blocking=True)
        e0, e1 = int(pc.indptr[r0]), int(pc.indptr[r1])
        if e1 > e0:
            self.indptr[: n + 1].copy_(pins[1][r0: r1 + 1], non_blocking=True)
            self.entries[: 8 * (e1 - e0)].copy_(pins[2][8 * e0: 8 * e1], non_blocking=True)
        max_nib = 0
        if pc.bits == 1:
            b0, b1 = int(pc.nib_indptr[r0]), int(pc.nib_indptr[r1])
            self.nib_indptr[: n + 1].copy_(pins[3][r0: r1 + 1], non_blocking=True)
            if b1 > b0:
                self.nibbles[: b1 - b0].copy_(pins[4][b0: b1], non_blocking=True)
            max_nib = int(np.diff(pc.nib_indptr[r0: r1 + 1]).max())
        return e1 > e0, max_nib

    def expand(self, lib, pc, n, has_ovf, max_nib, Y, X, x_dtype, dev, exact=None):
        """The rows uploaded last into Y (fp32) and X: the float transform with no scaling (X = y) when exact is None,
        else the exact transform, exact = (n_counts device fp64 of these rows, median, flags, mean, std)."""
        ovp = self.indptr.data_ptr() if has_ovf else None
        ove = self.entries.data_ptr() if has_ovf else None
        xdt = _lib.BF16 if x_dtype == torch.bfloat16 else _lib.F32
        G = pc.n_genes
        s = _stream(dev)
        if exact is None:
            if pc.bits == 1:
                check(lib.dca_expand_sparse_counts(self.packed.data_ptr(), self.nib_indptr.data_ptr(), self.nibbles.data_ptr(),
                                                   max_nib, ovp, ove, None, n, G, None, None, 0, 0, Y.data_ptr(),
                                                   X.data_ptr(), xdt, None, s), "dca_expand_sparse_counts")
            else:
                check(lib.dca_expand_packed_counts(self.packed.data_ptr(), pc.bits, ovp, ove, None, n, G, None, None, 0, 0,
                                                   Y.data_ptr(), X.data_ptr(), xdt, None, s), "dca_expand_packed_counts")
            return
        nc, med, flags, mean, std, sf_out = exact
        ncp = nc.data_ptr() if nc is not None else None
        if pc.bits == 1:
            check(lib.dca_expand_sparse_counts_exact(self.packed.data_ptr(), self.nib_indptr.data_ptr(),
                                                     self.nibbles.data_ptr(), max_nib, ovp, ove, ncp, n, G, med, flags,
                                                     mean.data_ptr(), std.data_ptr(), Y.data_ptr(), X.data_ptr(), xdt,
                                                     sf_out.data_ptr(), s), "dca_expand_sparse_counts_exact")
        else:
            check(lib.dca_expand_packed_counts_exact(self.packed.data_ptr(), pc.bits, ovp, ove, ncp, n, G, med, flags,
                                                     mean.data_ptr(), std.data_ptr(), Y.data_ptr(), X.data_ptr(), xdt,
                                                     sf_out.data_ptr(), s), "dca_expand_packed_counts_exact")


def _chunk_bounds(pc, chunk_rows):
    n = pc.n_rows
    b = list(range(0, n, chunk_rows)) + [n]
    max_e = max(int(pc.indptr[b[i + 1]] - pc.indptr[b[i]]) for i in range(len(b) - 1))
    max_nib = max(int(pc.nib_indptr[b[i + 1]] - pc.nib_indptr[b[i]]) for i in range(len(b) - 1)) if pc.bits == 1 else 0
    return b, max_e, max_nib


def for_each_chunk(pc, dev, chunk_rows, fn):
    """fn(r0, n, Y) for consecutive row chunks of pc in order, Y = the chunk's fp32 counts of the pc.genes real genes
    on the device (a view with row stride pc.n_genes: the pad genes are dropped).  The packed bytes
    of the next chunk are copied host->device on a side stream while the current one is expanded and processed
    (two staging buffers); everything else runs on the current stream."""
    lib = _lib.load()
    bounds, max_e, max_nib = _chunk_bounds(pc, chunk_rows)
    pins = pin_packed(pc, dev.index or 0)
    G = pc.n_genes
    Y = torch.empty((chunk_rows, G), dtype=torch.float32, device=dev)
    X = torch.empty((chunk_rows, G), dtype=torch.bfloat16, device=dev)       # the expansion's X: not used here
    stage = [_DevicePack(pc, dev, chunk_rows, max_e, max_nib) for _ in range(2)]
    comp = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(dev)
    freed = [None, None]

    def upload(k):
        slot = k % 2
        with torch.cuda.stream(side):
            if freed[slot] is not None:
                side.wait_event(freed[slot])
            info = stage[slot].upload(pc, pins, bounds[k], bounds[k + 1])
            ev = torch.cuda.Event()
            ev.record(side)
        return ev, info

    nk = len(bounds) - 1
    pending = upload(0)
    for k in range(nk):
        ev, (has_ovf, mnib) = pending
        if k + 1 < nk:
            pending = upload(k + 1)
        comp.wait_event(ev)
        n = bounds[k + 1] - bounds[k]
        stage[k % 2].expand(lib, pc, n, has_ovf, mnib, Y, X, torch.bfloat16, dev)
        freed[k % 2] = torch.cuda.Event()
        freed[k % 2].record(comp)
        fn(bounds[k], n, Y[:, :pc.genes])
    torch.cuda.synchronize(dev)


def expand_exact(pc, n_counts, median, flags, mean, std, x_dtype, dev):
    """Y (fp32), X (x_dtype) and sf (fp32) of every row of pc on the device through the exact expansion: the rows of a
    DeviceDataset's Y, X and sf for the same cells (pc.genes columns).  n_counts: host fp64 [pc.n_rows]; mean / std:
    host fp64 [pc.genes].  The rows are expanded at the stored width, the pad genes with mean 0 and std 1."""
    lib = _lib.load()
    n, G = pc.n_rows, pc.n_genes
    _, max_e, max_nib = _chunk_bounds(pc, max(n, 1))
    pk = _DevicePack(pc, dev, n, max_e, max_nib)
    pins = pin_packed(pc, dev.index or 0)
    has_ovf, mnib = pk.upload(pc, pins, 0, n)
    Y = torch.empty((n, G), dtype=torch.float32, device=dev)
    X = torch.empty((n, G), dtype=x_dtype, device=dev)
    sf = torch.empty(n, dtype=torch.float32, device=dev)
    nc = torch.from_numpy(np.ascontiguousarray(n_counts, dtype=np.float64)).to(dev)
    md = torch.from_numpy(_pad_stats(mean, G, 0.0)).to(dev)
    sd = torch.from_numpy(_pad_stats(std, G, 1.0)).to(dev)
    pk.expand(lib, pc, n, has_ovf, mnib, Y, X, x_dtype, dev, exact=(nc, median, flags, md, sd, sf))
    if pc.genes != G:
        Y, X = Y[:, :pc.genes].contiguous(), X[:, :pc.genes].contiguous()
    torch.cuda.synchronize(dev)
    return Y, X, sf


def _pad_stats(v, width, fill):
    """fp64 per-gene vector v extended to ``width`` entries with ``fill`` (the pad genes' neutral mean 0 / std 1)."""
    out = np.full(width, fill, dtype=np.float64)
    out[:len(v)] = v
    return out


def stream_epoch(eng, n, batch, shuffle, begin, positions):
    """epoch(update) over the n rows of a host stream that begin() starts, in batches of ``batch`` rows: the batches
    in a new random order every epoch (global NumPy RNG; in order with shuffle=False), update() after each step and
    before it check(positions of the batch's cells) when given -- ``positions``: each streamed row's, in stream order."""
    nb = (n + batch - 1) // batch

    def epoch(update, check=None):
        border = np.random.permutation(nb) if shuffle else np.arange(nb)
        begin()
        try:                                       # a failing check leaves no stream open
            for k in range(nb):
                b = int(border[k])
                eng.stream_step(b, int(border[k + 1]) if k + 1 < nb else -1)
                if check:
                    check(positions[b * batch: (b + 1) * batch])
                update()
        finally:
            eng.stream_end()
    return epoch


class StreamedDataset(_Dataset):
    """Packed raw counts ``pc`` (io.PackedCounts, cells in order) with the statistics of the device preprocessing:
    ``n_counts_host`` (fp64), ``size_factors_host`` (fp32), ``mean`` / ``std`` (fp64 per gene), ``median``, ``flags``.
    The masks of the filtering steps (``gene_mask``, ``cell_mask``, ``sf_mask``), ``gene_totals_host``,
    ``input_gene_totals`` and ``n_bad`` are those of DeviceDataset, so io.apply_device_normalize(adata, sd, ...,
    set_x=False) mutates an AnnData the same way.  Training, validation and prediction stream their batches from the
    packed counts (the interface of device_data._Dataset, keyword ``stream_data``); training shuffles the rows once
    and permutes whole batches every epoch."""
    kind = "stream_data"
    _on = "is for"

    def __init__(self, pc, n_counts_host, size_factors_host, mean, std, median, flags, x_dtype, device):
        self.pc, self.n_counts_host, self.size_factors_host = pc, n_counts_host, size_factors_host
        self.mean, self.std, self.median, self.flags = mean, std, median, flags
        self.x_dtype, self.device = x_dtype, device

    @property
    def n(self) -> int:
        return self.pc.n_rows

    @property
    def n_genes(self) -> int:
        return self.pc.genes

    @classmethod
    def from_counts(cls, counts, device=None, x_dtype="float32", size_factors=True, logtrans_input=True,
                    normalize_input=True, filter_min_counts=False, batch=32, bits="auto", chunk_rows=None,
                    pad_genes=False):
        """counts: cells x genes, a dense ndarray or a scipy.sparse CSR matrix of raw counts (a CSR matrix is packed in
        row chunks and never densified whole).  The filtering and normalisation steps of io.normalize with the same
        flags; x_dtype 'float32' | 'bfloat16' (the X the training step reads); batch: the training batch the packing
        the format is chosen for (overflow entries per batch; the streaming calls check and, where needed, widen the
        packing for the batch they stream in: stream_batches); chunk_rows: rows per chunk of the statistics passes
        (default: 256 MB of fp32 counts); pad_genes: accept a gene count off a multiple of 8, before and after the
        gene filter (the rows are packed zero-padded to the next multiple of 8; every result covers the real genes)."""
        if not torch.cuda.is_available():
            raise _lib.DcaError("StreamedDataset needs a CUDA device (H100); there is no CPU fallback")
        dev, xdt = _device(device), _X_DTYPES[x_dtype]
        counts = _counts_matrix(counts)
        N0, G0 = (int(s) for s in counts.shape)
        if G0 % 8 != 0 and not pad_genes:
            raise ValueError("streaming from packed counts needs a gene count that is a multiple of 8 (got %d)" % G0)
        with torch.cuda.device(dev):
            pc = dio.pack_rows(counts, bits, batch=batch, pad_genes=pad_genes)
            nc, gene_tot, n_bad = _totals(pc, dev, chunk_rows)
            input_gene_totals, input_n_bad = gene_tot, n_bad
            gene_mask = np.ones(G0, bool)
            cell_mask = np.ones(N0, bool)
            if filter_min_counts:                                            # dca/io.py:90-92
                gene_mask = gene_tot >= 1
                if not gene_mask.all():
                    if gene_mask.sum() % 8 != 0 and not pad_genes:
                        raise ValueError("filtering leaves %d genes; streaming from packed counts needs a multiple of 8 "
                                         "(filter the genes before, or use the resident device path)" % gene_mask.sum())
                    counts = counts[:, np.flatnonzero(gene_mask)]
                    pc = dio.pack_rows(counts, bits, batch=batch, pad_genes=pad_genes)
                    nc, gene_tot, _ = _totals(pc, dev, chunk_rows)
                cell_mask = nc >= 1
                if not cell_mask.all():
                    pc = pc.take_rows(np.flatnonzero(cell_mask))
                    nc, gene_tot, _ = _totals(pc, dev, chunk_rows)
            sf_mask = np.ones(nc.shape[0], bool)
            if size_factors:                                                 # normalize_per_cell drops cells without counts
                sf_mask = nc >= 1
                if not sf_mask.all():
                    pc = pc.take_rows(np.flatnonzero(sf_mask))
                    nc, gene_tot, _ = _totals(pc, dev, chunk_rows)
            med, sf_h = _size_factors(nc, size_factors)
            flags = preprocess_flags(size_factors, logtrans_input, normalize_input)
            mean, std = _moments(pc, nc, med, flags, dev, chunk_rows)
        sd = cls(pc, nc, sf_h, mean, std, med, flags, xdt, dev)
        sd.gene_totals_host, sd.input_gene_totals, sd.n_bad = gene_tot, input_gene_totals, input_n_bad
        sd.gene_mask, sd.cell_mask, sd.sf_mask = gene_mask, cell_mask, sf_mask
        return sd

    def take(self, mask_or_index):
        """The cells ``mask_or_index`` (a boolean mask over this dataset's cells or integer positions) selects, in that
        order; the packed rows are copied (io.PackedCounts.take_rows) unless the selection is every cell in order."""
        idx = self._positions(mask_or_index)
        if idx.size == self.n and np.array_equal(idx, np.arange(self.n)):
            return self
        sd = StreamedDataset.__new__(StreamedDataset)
        sd.__dict__.update(self.__dict__)
        sd._stream_cache = {}
        sd.pc = self.pc.take_rows(idx)
        sd.n_counts_host = self.n_counts_host[idx]
        sd.size_factors_host = self.size_factors_host[idx]
        return sd

    def rows(self, r0, r1):
        """A dataset over cells [r0, r1)."""
        return self.take(np.arange(r0, r1))

    def stream_batches(self, eng, batch):
        """Start streaming this dataset through engine ``eng`` in batches of ``batch`` rows with the exact transform
        (dca_set_input_transform_exact + dca_stream_begin* + dca_stream_row_totals).  The packing is checked against
        what one batch of the engine may carry and widened when a batch would not fit (io.fit_batches); the widened
        copy is kept for the next call with the same batch."""
        from .hostmem import pin_near_gpu
        ovf_cap, nib_cap = eng.stream_capacity()
        key = (batch, ovf_cap, nib_cap)
        cache = self.__dict__.setdefault("_stream_cache", {})
        if key not in cache:
            nc = pin_near_gpu(torch.from_numpy(np.ascontiguousarray(self.n_counts_host, dtype=np.float64)),
                              self.device.index or 0)
            cache.clear()
            cache[key] = (dio.fit_batches(self.pc, batch, ovf_cap, nib_cap), nc)
        pc, nc = cache[key]
        eng.set_input_transform_exact(self.mean, self.std, self.median, self.flags)
        eng.stream_begin(pc, None, batch)
        eng.stream_row_totals(nc)

    def expand(self):
        """(Y, X, sf) of every cell on the device, through the exact expansion: the rows of a DeviceDataset's Y, X and sf."""
        return expand_exact(self.pc, self.n_counts_host, self.median, self.flags, self.mean, self.std, self.x_dtype,
                            self.device)

    # ------------------------------------------------------------------ training and prediction
    def _bind(self, eng):
        self._check_genes(eng)
        super()._bind(eng)

    def _fit(self, eng, n_tr, batch, shuffle):
        """The training rows shuffled ONCE (a packed copy in that order), every epoch permuting whole batches; the
        validation rows streamed as well (dca_stream_eval), so device memory does not grow with the dataset."""
        order0 = np.arange(n_tr)
        if shuffle:
            np.random.shuffle(order0)
        tr = self.take(order0)
        va = self.rows(n_tr, self.n) if n_tr < self.n else None
        nb_va = (self.n - n_tr + batch - 1) // batch

        def validate(check=None):
            if va is None:
                return
            va.stream_batches(eng, batch)
            try:
                for k in range(nb_va):
                    eng.stream_eval(k, k + 1 if k + 1 < nb_va else -1)
                    if check:
                        check(np.arange(n_tr + k * batch, min(n_tr + (k + 1) * batch, self.n)))
            finally:
                eng.stream_end()
        return stream_epoch(eng, n_tr, batch, shuffle, lambda: tr.stream_batches(eng, batch), order0), validate

    def _predictor(self, eng, bs):
        nb = (self.n + bs - 1) // bs

        def run(i, s, e, b):
            eng.stream_predict(i, i + 1 if i + 1 < nb else -1, mean=b.get("mean"), disp=b.get("disp"),
                               pi=b.get("pi"), latent=b.get("latent"))

        def theta(th):
            eng.stream_predict(0, -1, disp=th)

        @contextlib.contextmanager
        def session():
            self.stream_batches(eng, bs)
            try:
                yield
            finally:
                eng.stream_end()
        return run, theta, session


def _genes(pc):
    return getattr(pc, "genes", pc.n_genes)


def _chunk_rows(G):
    return max(1, _CHUNK_BYTES // (4 * G))


def _workspace(lib, N, G, chunk, dev):
    ws_bytes = C.c_size_t()
    check(lib.dca_stats_workspace_bytes(N, G, chunk, C.byref(ws_bytes)), "dca_stats_workspace_bytes")
    return torch.empty(ws_bytes.value, dtype=torch.uint8, device=dev)


def _totals(pc, dev, chunk_rows=None, chunks=None):
    """(n_counts fp64 [N], gene totals fp64 [G], number of bad entries) on the host.  chunks(chunk, fn) feeds the row
    chunks of the matrix to fn(r0, n, Y) (default: for_each_chunk over the packed host counts pc); pc then only needs
    n_rows and n_genes.  G: pc.genes when pc has it (the real genes of padded rows), else pc.n_genes; Y may have a row
    stride above G."""
    lib = _lib.load()
    N, G = pc.n_rows, _genes(pc)
    chunk = min(N, chunk_rows or _chunk_rows(G))
    ws = _workspace(lib, N, G, chunk, dev)
    n_counts = torch.empty(N, dtype=torch.float64, device=dev)
    gene_tot = torch.empty(G, dtype=torch.float64, device=dev)
    n_bad = torch.zeros(1, dtype=torch.int64, device=dev)
    check(lib.dca_stats_begin(N, G, ws.data_ptr(), ws.numel(), _stream(dev)), "dca_stats_begin")

    def rows(r0, n, Y):
        check(lib.dca_count_totals_rows(Y.data_ptr(), Y.stride(0), r0, n, N, G, n_counts.data_ptr(), ws.data_ptr(), ws.numel(),
                                        _stream(dev)), "dca_count_totals_rows")
    (chunks or (lambda c, fn: for_each_chunk(pc, dev, c, fn)))(chunk, rows)
    check(lib.dca_count_totals_finish(N, G, gene_tot.data_ptr(), n_bad.data_ptr(), ws.data_ptr(), ws.numel(),
                                      _stream(dev)), "dca_count_totals_finish")
    return n_counts.cpu().numpy(), gene_tot.cpu().numpy(), int(n_bad.item())


def _moments(pc, nc_host, median, flags, dev, chunk_rows=None, chunks=None):
    """Gene mean and std (fp64, host) of l over the rows of pc: passes 1 and 2 of dca_log_moments (chunks: as for
    _totals)."""
    lib = _lib.load()
    N, G = pc.n_rows, _genes(pc)
    chunk = min(N, chunk_rows or _chunk_rows(G))
    ws = _workspace(lib, N, G, chunk, dev)
    nc = torch.from_numpy(np.ascontiguousarray(nc_host, dtype=np.float64)).to(dev) if flags & PRE_SIZE_FACTORS else None
    ncp = nc.data_ptr() if nc is not None else None
    out = [torch.empty(G, dtype=torch.float64, device=dev) for _ in range(2)]
    for p in (1, 2):
        check(lib.dca_stats_begin(N, G, ws.data_ptr(), ws.numel(), _stream(dev)), "dca_stats_begin")
        if flags & 4:                           # DCA_PRE_SCALE: otherwise mean = 0, std = 1 without reading the counts
            def rows(r0, n, Y, p=p):
                check(lib.dca_log_moments_rows(p, Y.data_ptr(), Y.stride(0), r0, n, N, G, ncp, median, flags, out[0].data_ptr(),
                                               ws.data_ptr(), ws.numel(), _stream(dev)), "dca_log_moments_rows")
            (chunks or (lambda c, fn: for_each_chunk(pc, dev, c, fn)))(chunk, rows)
        check(lib.dca_log_moments_finish(p, N, G, flags, out[p - 1].data_ptr(), ws.data_ptr(), ws.numel(), _stream(dev)),
              "dca_log_moments_finish")
    return out[0].cpu().numpy(), out[1].cpu().numpy()
