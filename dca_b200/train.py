"""Training driver with the surface of dca/train.py:35-191.

``train()`` replaces ``model.compile`` + ``model.fit`` (dca/train.py:54-98): the data stay
resident in HBM, every batch is one dca_train_step + gradient all-reduce (when launched under
torch.distributed) + dca_apply_update, validation is the tail ``validation_split`` of the rows
(taken before shuffling, as Keras does), and ReduceLROnPlateau / EarlyStopping are evaluated on
the host from one scalar per epoch (SURVEY.md A.7).
"""
from __future__ import annotations

import os
import random
from typing import Optional

import numpy as np
import torch

from . import dist as D
from .engine import KERAS_DEFAULTS


class History:
    """Stand-in for keras.callbacks.History (only ``.history`` is used, dca/api.py:206)."""

    def __init__(self):
        self.history = {"loss": [], "val_loss": [], "lr": []}
        self.epoch = []


class PlateauAndStop:
    """ReduceLROnPlateau(monitor='val_loss', factor=0.1, min_delta=1e-4, cooldown=0, min_lr=0)
    followed by EarlyStopping(monitor='val_loss', min_delta=0) -- dca/train.py:70-75."""

    def __init__(self, lr, reduce_lr, early_stop, verbose=False):
        self.lr, self.reduce_lr, self.early_stop, self.verbose = lr, reduce_lr, early_stop, verbose
        self.best = np.inf; self.wait = 0
        self.es_best = np.inf; self.es_wait = 0
        self.stopped_epoch = None

    def on_epoch_end(self, epoch, monitor) -> bool:
        """Returns True when training should stop."""
        if monitor is None:
            return False
        if self.reduce_lr:
            if monitor < self.best - 1e-4:
                self.best = monitor; self.wait = 0
            else:
                self.wait += 1
                if self.wait >= self.reduce_lr:
                    new_lr = self.lr * 0.1
                    if self.verbose:
                        print("\nEpoch %05d: ReduceLROnPlateau reducing learning rate to %s." % (epoch + 1, new_lr))
                    self.lr = new_lr; self.wait = 0
        if self.early_stop:
            if monitor < self.es_best:
                self.es_best = monitor; self.es_wait = 0
            else:
                self.es_wait += 1
                if self.es_wait >= self.early_stop:
                    self.stopped_epoch = epoch
                    if self.verbose:
                        print("Epoch %05d: early stopping" % (epoch + 1))
                    return True
        return False


def _to_device(a, dtype, device):
    t = torch.as_tensor(np.ascontiguousarray(a))
    return t.to(device=device, dtype=dtype, non_blocking=False).contiguous()


def train(adata, network, output_dir=None, optimizer='RMSprop', learning_rate=None,
          epochs=300, reduce_lr=10, output_subset=None, use_raw_as_output=True,
          early_stop=15, batch_size=32, clip_grad=5., save_weights=False,
          validation_split=0.1, tensorboard=False, verbose=True, threads=None,
          **kwds):
    """Same signature as dca/train.py:35-39.  ``threads`` is accepted and ignored (GPU path).

    Extra keyword (``training_kwds`` of ``dca()``): ``stream`` -- False (default): the shard lives in HBM for the whole
    run, rows are reshuffled every epoch exactly like Keras; True / 'auto': train from HOST memory through
    dca_stream_* (raw counts bit-packed in pinned memory, every step copies its batch host->device while the previous
    one computes and normalises it on the device, dca/io.py:99-109 restated) -- for matrices that do not fit the GPU
    ('auto' switches when X + Y would exceed 60 % of the free device memory).  In streaming mode the training rows are
    shuffled ONCE and every epoch visits the batches in a new random order (documented deviation from Keras' per-epoch
    row shuffle).  Other keywords of the reference's model.fit (e.g. shuffle=False) are honoured or rejected loudly.

    ``device_data``: a device_data.DeviceDataset of the cells of ``adata`` (in order), preprocessed in HBM.  X, the
    raw-count target and the size factors are then read there (steps gather their rows through the dataset's
    ``rows``) and adata's matrices are not used; the updates are those of the host arrays holding the same values.
    Single process only, use_raw_as_output only, and with ``output_subset`` the dataset's Y must already hold those
    genes (DeviceDataset.with_output_genes).  adata is then only read for ``raw.var_names`` (output_subset) and may be
    None otherwise.

    ``packed_data``: a packed_data.PackedDeviceDataset of the cells of ``adata`` (in order): raw counts packed in HBM,
    every batch expanded on the device by row index.  The resident loop as with device_data (rows reshuffled every
    epoch exactly like Keras) and the same updates; single process only, use_raw_as_output only, no output_subset."""
    stream = kwds.pop('stream', False)
    shuffle = kwds.pop('shuffle', True)
    device_data = kwds.pop('device_data', None)
    stream_data = kwds.pop('stream_data', None)
    packed_data = kwds.pop('packed_data', None)
    if kwds:
        raise TypeError("train() got keyword arguments the accelerated fit loop does not implement: %s" % sorted(kwds))
    from . import _lib as _L
    if optimizer not in _L.OPTIMIZERS:
        raise NotImplementedError("optimizer %r is not on the accelerated path (supported: %s)"
                                  % (optimizer, sorted(k for k in _L.OPTIMIZERS if not k.islower())))
    if tensorboard:
        raise NotImplementedError("tensorboard logging is not part of the accelerated path")
    if output_dir is not None:
        os.makedirs(output_dir, exist_ok=True)
    if packed_data is not None:
        if device_data is not None or stream_data is not None or stream:
            raise ValueError("packed_data is resident in HBM: it cannot be combined with stream, device_data or "
                             "stream_data")
        return _train_packed_data(adata, network, packed_data, output_subset, use_raw_as_output, optimizer,
                                  learning_rate, batch_size, validation_split, epochs, reduce_lr, early_stop, clip_grad,
                                  verbose, save_weights, output_dir, shuffle)
    if stream_data is not None:
        if device_data is not None:
            raise ValueError("give device_data or stream_data, not both")
        return _train_stream_data(adata, network, stream_data, output_subset, use_raw_as_output, optimizer, learning_rate,
                                  batch_size, validation_split, epochs, reduce_lr, early_stop, clip_grad, verbose,
                                  save_weights, output_dir, shuffle)
    if device_data is not None:
        return _train_device_data(adata, network, device_data, stream, output_subset, use_raw_as_output, optimizer,
                                  learning_rate, batch_size, validation_split, epochs, reduce_lr, early_stop, clip_grad,
                                  verbose, save_weights, output_dir, shuffle)

    X = np.asarray(adata.X, dtype=np.float32)
    sf = np.asarray(adata.obs['size_factors'], dtype=np.float32).reshape(-1)
    if output_subset:
        raw_names = np.asarray(adata.raw.var_names)
        gene_idx = [np.where(raw_names == x)[0][0] for x in output_subset]
        Yh = adata.raw.X[:, gene_idx] if use_raw_as_output else adata.X[:, gene_idx]
    else:
        Yh = adata.raw.X if use_raw_as_output else adata.X
    Yh = np.asarray(Yh.toarray() if hasattr(Yh, "toarray") else Yh, dtype=np.float32)

    N = X.shape[0]
    split_at = int(N * (1. - validation_split)) if validation_split and 0. < validation_split < 1. else N
    rank, world = D.rank_world()

    # cells shard across ranks (SURVEY.md 8e): contiguous row ranges, equal count per rank
    tr_lo, tr_hi = D.shard_bounds(split_at, rank, world, equal=True)
    va_lo, va_hi = D.shard_bounds(N - split_at, rank, world, equal=False)
    va_lo += split_at; va_hi += split_at

    if world > 1 and rank == 0 and (split_at % world) and verbose:
        print("dca: %d training cells do not divide over %d ranks; the last %d are left out of every epoch"
              % (split_at, world, split_at % world))
    eng = network.ensure_engine(max_batch=batch_size)
    dev = eng.device
    if stream == 'auto':
        free = torch.cuda.mem_get_info(dev)[0]
        stream = (tr_hi - tr_lo + va_hi - va_lo) * X.shape[1] * (4 + eng.params.element_size()) > 0.6 * free
    # opt.__dict__[optimizer](clipvalue=clip_grad[, lr=learning_rate])                   (dca/train.py:54-57)
    default_lr = eng.set_optimizer(optimizer)
    if learning_rate is None:
        learning_rate = default_lr
    if stream:
        return _fit_stream(eng, network, X, Yh, sf, (tr_lo, tr_hi), (va_lo, va_hi), batch_size, epochs, learning_rate, reduce_lr,
                           early_stop, clip_grad, world, rank, verbose, save_weights, output_dir, shuffle)
    Xd = _to_device(np.concatenate([X[tr_lo:tr_hi], X[va_lo:va_hi]]), eng.x_dtype, dev)
    Yd = _to_device(np.concatenate([Yh[tr_lo:tr_hi], Yh[va_lo:va_hi]]), torch.float32, dev)
    sfd = _to_device(np.concatenate([sf[tr_lo:tr_hi], sf[va_lo:va_hi]]), torch.float32, dev)
    n_tr = tr_hi - tr_lo
    n_va = va_hi - va_lo

    if world > 1:
        D.broadcast_(eng.params, src=0); D.broadcast_(eng.bn_state, src=0)
        eng.params_changed()
        if torch.distributed.get_backend() == "nccl":
            eng.comm_init()          # gradient exchange inside the library: one CUDA graph per step (dca_train_step_dp)
    eng.reset_optimizer()

    lr = float(learning_rate)
    ctl = PlateauAndStop(lr, reduce_lr, early_stop, verbose)
    hist = History()
    if verbose:
        print(network.summary())

    steps = (n_tr + batch_size - 1) // batch_size
    gscale = 1.0 / world
    # run on a non-default stream (CUDA-graph replay of the step needs a capturable stream)
    torch.cuda.synchronize(dev)
    prev_stream = torch.cuda.current_stream(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))
    try:
        hist = _fit_loop(eng, network, Xd, Yd, sfd, n_tr, n_va, steps, batch_size, epochs, ctl, clip_grad, gscale, world, rank,
                         dev, hist, verbose, save_weights, output_dir, shuffle)
    finally:
        torch.cuda.synchronize(dev)
        torch.cuda.set_stream(prev_stream)
    if not hist.history["val_loss"]:
        del hist.history["val_loss"]
    return hist


def _epoch_end(eng, network, hist, ctl, epoch, epochs, n_va, world, rank, dev, verbose, save_weights, output_dir, best_val):
    """Epoch bookkeeping shared by the resident and the streaming loop: reduce the accumulators over ranks, history,
    ModelCheckpoint, ReduceLROnPlateau / EarlyStopping.  Returns (stop, best_val)."""
    acc = np.asarray(eng.read_epoch_acc(reset=True), dtype=np.float64)
    if world > 1:
        acc = D.all_reduce_sum_host(acc, dev)
        if eng.bn_state.numel():
            D.all_reduce_sum_(eng.bn_state); eng.bn_state.mul_(1.0 / world)
    loss = acc[0] / acc[1] if acc[1] > 0 else float("nan")
    if not np.isfinite(loss):
        loss = float("inf")                       # _nan2inf convention, dca/loss.py:148
    val = None
    if n_va > 0 or (world > 1 and acc[3] > 0):
        val = acc[2] / acc[3] + network.penalty_value()
        if not np.isfinite(val):
            val = float("inf")
    hist.epoch.append(epoch)
    hist.history["loss"].append(float(loss))
    hist.history["lr"].append(float(ctl.lr))
    if val is not None:
        hist.history["val_loss"].append(float(val))
    if verbose and rank == 0:
        print("Epoch %d/%d - loss: %.4f%s - lr: %g" % (epoch + 1, epochs, loss,
                                                    "" if val is None else " - val_loss: %.4f" % val, ctl.lr))
    if save_weights and output_dir is not None and rank == 0:
        mon = val if val is not None else loss
        if mon < best_val:                       # ModelCheckpoint(save_best_only=True), dca/train.py:64-69
            best_val = mon
            network.save_weights(os.path.join(output_dir, "weights.npz"))
    return ctl.on_epoch_end(epoch, val), best_val


def _fit_stream(eng, network, X, Yh, sf, tr, va, batch_size, epochs, learning_rate, reduce_lr, early_stop, clip_grad, world, rank,
                verbose, save_weights, output_dir, shuffle):
    """Training from host memory (dca_stream_*): see train().  X is only used for the (small, resident) validation rows;
    the training rows travel as bit-packed raw counts and are normalised on the device."""
    from . import io as dio
    from .hostmem import pin_near_gpu
    dev = eng.device
    (tr_lo, tr_hi), (va_lo, va_hi) = tr, va
    if eng.n_in != eng.n_out or Yh.shape[1] != X.shape[1]:
        raise NotImplementedError("stream=True needs the raw counts of the input genes as the target (no output_subset)")
    n_tr, n_va = tr_hi - tr_lo, va_hi - va_lo
    order0 = np.arange(tr_lo, tr_hi)
    if shuffle:
        np.random.shuffle(order0)                 # ONE row shuffle; the epochs permute whole batches
    Ytr = np.ascontiguousarray(Yh[order0]); sftr = np.ascontiguousarray(sf[order0])
    # the transform X = (log1p(y / sf) - mean_g) / std_g the host normalisation applied (dca/io.py:99-109), recovered from
    # (X, raw) of a few hundred rows: two unknowns per gene
    l = np.log1p(Yh / sf[:, None]) if n_tr + n_va <= 4096 else None
    if l is None:
        pick = np.linspace(0, Yh.shape[0] - 1, 4096).astype(np.int64)
        l = np.log1p(Yh[pick] / sf[pick, None]); xs = X[pick]
    else:
        xs = X
    lm, xm = l.mean(0, dtype=np.float64), xs.mean(0, dtype=np.float64)
    lv = ((l - lm) * (xs - xm)).sum(0, dtype=np.float64); xv = ((xs - xm) ** 2).sum(0, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        std = np.where(xv > 0, lv / xv, 1.0)       # l = mean + std * x  =>  std = cov(l, x) / var(x)
    std[~np.isfinite(std) | (std <= 0)] = 1.0
    mean = lm - std * xm
    if float(np.max(np.abs((l - mean) / std - xs))) > 1e-2:
        raise NotImplementedError("stream=True supports the default preprocessing only (size factors + log1p [+ scale], "
                                  "dca/io.py:99-109): adata.X is not (log1p(raw / size_factors) - mean_g) / std_g")
    eng.set_input_transform(mean, std, True, True)
    packed = dio.pack_counts(Ytr, "auto", batch=batch_size)
    sf_h = pin_near_gpu(torch.from_numpy(sftr.astype(np.float32)), dev.index or 0)
    Xv = _to_device(X[va_lo:va_hi], eng.x_dtype, dev) if n_va else None
    Yv = _to_device(Yh[va_lo:va_hi], torch.float32, dev) if n_va else None
    sfv = _to_device(sf[va_lo:va_hi], torch.float32, dev) if n_va else None
    if world > 1:
        D.broadcast_(eng.params, src=0); D.broadcast_(eng.bn_state, src=0)
        eng.params_changed()
        if torch.distributed.get_backend() == "nccl":
            eng.comm_init()
    eng.reset_optimizer()
    lr = float(learning_rate)
    ctl = PlateauAndStop(lr, reduce_lr, early_stop, verbose)
    hist = History()
    nb = (n_tr + batch_size - 1) // batch_size
    gscale = 1.0 / world
    torch.cuda.synchronize(dev)
    prev_stream = torch.cuda.current_stream(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))
    best_val = np.inf
    try:
        for epoch in range(epochs):
            border = np.random.permutation(nb) if shuffle else np.arange(nb)
            eng.read_epoch_acc(reset=True)
            eng.stream_begin(packed, sf_h, batch_size)
            for k in range(nb):
                eng.stream_step(int(border[k]), int(border[k + 1]) if k + 1 < nb else -1)
                if world > 1:
                    eng.allreduce_grads() if getattr(eng, "_comm", False) else D.all_reduce_sum_(eng.grads)
                eng.apply_update(ctl.lr, clip_grad, gscale)
            eng.stream_end()
            for s0 in range(0, n_va, batch_size):
                e = min(s0 + batch_size, n_va)
                eng.eval_step(Xv[s0:e], Yv[s0:e], sfv[s0:e])
            stop, best_val = _epoch_end(eng, network, hist, ctl, epoch, epochs, n_va, world, rank, dev, verbose, save_weights,
                                        output_dir, best_val)
            if stop:
                break
    finally:
        torch.cuda.synchronize(dev)
        torch.cuda.set_stream(prev_stream)
    if not hist.history["val_loss"]:
        del hist.history["val_loss"]
    return hist


def _train_stream_data(adata, network, sd, output_subset, use_raw_as_output, optimizer, learning_rate, batch_size,
                       validation_split, epochs, reduce_lr, early_stop, clip_grad, verbose, save_weights, output_dir, shuffle):
    """train() on a stream_data.StreamedDataset: the split and stream semantics of _fit_stream (the training rows shuffled
    once, every epoch permuting whole batches; in order with shuffle=False), with batches normalised by the exact transform
    of the device preprocessing.  The validation rows are streamed as well (dca_stream_eval), so device memory does not
    grow with the dataset."""
    if D.rank_world()[1] > 1:
        raise NotImplementedError("stream_data trains on one GPU; a torch.distributed world larger than 1 is not supported")
    if not use_raw_as_output:
        raise ValueError("stream_data holds the raw counts as the target: use_raw_as_output=False is not supported")
    if output_subset:
        raise NotImplementedError("stream_data needs the raw counts of the input genes as the target (no output_subset)")
    if adata is not None and adata.n_obs != sd.n:
        raise ValueError("stream_data covers %d cells, adata has %d" % (sd.n, adata.n_obs))
    eng = network.ensure_engine(max_batch=batch_size)
    if eng.n_in != sd.n_genes or eng.n_out != sd.n_genes:
        raise ValueError("stream_data has %d genes, the network %d inputs and %d outputs" % (sd.n_genes, eng.n_in, eng.n_out))
    if sd.device != eng.device:
        raise ValueError("stream_data is for %s, the network on %s" % (sd.device, eng.device))
    if sd.x_dtype != eng.x_dtype:
        raise ValueError("stream_data X is %s, the network expects %s (network_kwds x_dtype)" % (sd.x_dtype, eng.x_dtype))
    dev = eng.device
    N = sd.n
    n_tr = int(N * (1. - validation_split)) if validation_split and 0. < validation_split < 1. else N
    n_va = N - n_tr
    order0 = np.arange(n_tr)
    if shuffle:
        np.random.shuffle(order0)                 # ONE row shuffle; the epochs permute whole batches (as _fit_stream)
    tr = sd.take(order0)
    va = sd.rows(n_tr, N) if n_va else None
    nb_va = (n_va + batch_size - 1) // batch_size
    default_lr = eng.set_optimizer(optimizer)
    if learning_rate is None:
        learning_rate = default_lr
    eng.reset_optimizer()
    ctl = PlateauAndStop(float(learning_rate), reduce_lr, early_stop, verbose)
    hist = History()
    if verbose:
        print(network.summary())
    nb = (n_tr + batch_size - 1) // batch_size
    torch.cuda.synchronize(dev)
    prev_stream = torch.cuda.current_stream(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))
    best_val = np.inf
    try:
        for epoch in range(epochs):
            border = np.random.permutation(nb) if shuffle else np.arange(nb)
            eng.read_epoch_acc(reset=True)
            tr.stream_batches(eng, batch_size)
            for k in range(nb):
                eng.stream_step(int(border[k]), int(border[k + 1]) if k + 1 < nb else -1)
                eng.apply_update(ctl.lr, clip_grad, 1.0)
            eng.stream_end()
            if n_va:
                va.stream_batches(eng, batch_size)
                for k in range(nb_va):
                    eng.stream_eval(k, k + 1 if k + 1 < nb_va else -1)
                eng.stream_end()
            stop, best_val = _epoch_end(eng, network, hist, ctl, epoch, epochs, n_va, 1, 0, dev, verbose, save_weights,
                                        output_dir, best_val)
            if stop:
                break
    finally:
        torch.cuda.synchronize(dev)
        torch.cuda.set_stream(prev_stream)
    if not hist.history["val_loss"]:
        del hist.history["val_loss"]
    return hist


def _train_device_data(adata, network, dd, stream, output_subset, use_raw_as_output, optimizer, learning_rate, batch_size,
                       validation_split, epochs, reduce_lr, early_stop, clip_grad, verbose, save_weights, output_dir, shuffle):
    """train() on a DeviceDataset: the resident loop of train() with positions mapped through dd.rows."""
    if stream:
        raise ValueError("device_data is resident in HBM: it cannot be combined with stream=True")
    if D.rank_world()[1] > 1:
        raise NotImplementedError("device_data trains on one GPU; a torch.distributed world larger than 1 is not supported")
    if not use_raw_as_output:
        raise ValueError("device_data holds the raw counts as the target: use_raw_as_output=False is not supported")
    if output_subset:
        if adata is None:
            raise ValueError("output_subset names genes of adata.raw: pass the AnnData with device_data")
        raw_names = np.asarray(adata.raw.var_names)
        gene_idx = [int(np.where(raw_names == x)[0][0]) for x in output_subset]
        if dd.y_cols is None or list(dd.y_cols) != gene_idx:
            raise ValueError("output_subset needs a dataset whose Y holds those genes: "
                             "device_data.with_output_genes(<their positions in adata.raw.var_names>)")
    elif dd.y_cols is not None:
        raise ValueError("the dataset's Y holds a subset of the genes, but no output_subset was given")
    if adata is not None and adata.n_obs != dd.n:
        raise ValueError("device_data covers %d cells, adata has %d" % (dd.n, adata.n_obs))
    eng = network.ensure_engine(max_batch=batch_size)
    if dd.X.device != eng.device:
        raise ValueError("device_data lives on %s, the network on %s" % (dd.X.device, eng.device))
    if dd.x_dtype != eng.x_dtype:
        raise ValueError("device_data X is %s, the network expects %s (network_kwds x_dtype)" % (dd.x_dtype, eng.x_dtype))
    N = dd.n
    n_tr = int(N * (1. - validation_split)) if validation_split and 0. < validation_split < 1. else N
    n_va = N - n_tr
    default_lr = eng.set_optimizer(optimizer)
    if learning_rate is None:
        learning_rate = default_lr
    eng.reset_optimizer()
    ctl = PlateauAndStop(float(learning_rate), reduce_lr, early_stop, verbose)
    hist = History()
    if verbose:
        print(network.summary())
    steps = (n_tr + batch_size - 1) // batch_size
    dev = eng.device
    torch.cuda.synchronize(dev)
    prev_stream = torch.cuda.current_stream(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))
    try:
        hist = _fit_loop(eng, network, dd.X, dd.Y, dd.sf, n_tr, n_va, steps, batch_size, epochs, ctl, clip_grad, 1.0, 1, 0,
                         dev, hist, verbose, save_weights, output_dir, shuffle, rows_map=dd.rows)
    finally:
        torch.cuda.synchronize(dev)
        torch.cuda.set_stream(prev_stream)
    if not hist.history["val_loss"]:
        del hist.history["val_loss"]
    return hist


def _train_packed_data(adata, network, pd, output_subset, use_raw_as_output, optimizer, learning_rate, batch_size,
                       validation_split, epochs, reduce_lr, early_stop, clip_grad, verbose, save_weights, output_dir, shuffle):
    """train() on a PackedDeviceDataset: the resident loop of train() with every batch expanded from the packed counts
    by row index (dca_packed_train_step / dca_packed_eval_step) with the exact transform of the device preprocessing."""
    if D.rank_world()[1] > 1:
        raise NotImplementedError("packed_data trains on one GPU; a torch.distributed world larger than 1 is not supported")
    if not use_raw_as_output:
        raise ValueError("packed_data holds the raw counts as the target: use_raw_as_output=False is not supported")
    if output_subset:
        raise NotImplementedError("packed_data needs the raw counts of the input genes as the target (no output_subset)")
    if adata is not None and adata.n_obs != pd.n:
        raise ValueError("packed_data covers %d cells, adata has %d" % (pd.n, adata.n_obs))
    eng = network.ensure_engine(max_batch=batch_size)
    if eng.n_in != pd.n_genes or eng.n_out != pd.n_genes:
        raise ValueError("packed_data has %d genes, the network %d inputs and %d outputs" % (pd.n_genes, eng.n_in, eng.n_out))
    if pd.device != eng.device:
        raise ValueError("packed_data lives on %s, the network on %s" % (pd.device, eng.device))
    if pd.x_dtype != eng.x_dtype:
        raise ValueError("packed_data X is %s, the network expects %s (network_kwds x_dtype)" % (pd.x_dtype, eng.x_dtype))
    N = pd.n
    n_tr = int(N * (1. - validation_split)) if validation_split and 0. < validation_split < 1. else N
    n_va = N - n_tr
    default_lr = eng.set_optimizer(optimizer)
    if learning_rate is None:
        learning_rate = default_lr
    eng.reset_optimizer()
    eng.set_input_transform_exact(pd.mean, pd.std, pd.median, pd.flags)
    ctl = PlateauAndStop(float(learning_rate), reduce_lr, early_stop, verbose)
    hist = History()
    if verbose:
        print(network.summary())
    steps = (n_tr + batch_size - 1) // batch_size
    dev = eng.device
    torch.cuda.synchronize(dev)
    prev_stream = torch.cuda.current_stream(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))
    try:
        hist = _fit_loop(eng, network, None, None, None, n_tr, n_va, steps, batch_size, epochs, ctl, clip_grad, 1.0, 1, 0,
                         dev, hist, verbose, save_weights, output_dir, shuffle, rows_map=pd.rows, packed=pd)
    finally:
        torch.cuda.synchronize(dev)
        torch.cuda.set_stream(prev_stream)
    if not hist.history["val_loss"]:
        del hist.history["val_loss"]
    return hist


def _fit_loop(eng, network, Xd, Yd, sfd, n_tr, n_va, steps, batch_size, epochs, ctl, clip_grad, gscale, world, rank, dev, hist,
              verbose, save_weights, output_dir, shuffle=True, rows_map=None, packed=None):
    """rows_map (int32 device tensor, n_tr + n_va entries): the storage row of each position in Xd / Yd / sfd; None:
    position = row.  packed: a PackedDeviceDataset whose storage rows rows_map names (Xd, Yd, sfd unused): every batch
    is expanded from its packed counts."""
    best_val = np.inf
    for epoch in range(epochs):
        # Keras: np.random.shuffle(index_array) with the global NumPy RNG (seeded in api.dca / CLI)
        order = np.arange(n_tr)
        if shuffle:
            np.random.shuffle(order)
        order_d = torch.from_numpy(order.astype(np.int32)).to(dev)
        if rows_map is not None:
            order_d = rows_map[order_d.long()]
        eng.read_epoch_acc(reset=True)
        for s in range(steps):
            rows = order_d[s * batch_size: min((s + 1) * batch_size, n_tr)]
            if packed is not None:
                eng.packed_train_step(packed, rows)
            elif world > 1:
                eng.train_step_allreduce(Xd, Yd, sfd, rows=rows)     # NCCL all-reduce overlapped with the backward tail
            else:
                eng.train_step(Xd, Yd, sfd, rows=rows)
            eng.apply_update(ctl.lr, clip_grad, gscale)
        # validation pass: inference-mode BN over the held-out tail
        for s in range(n_tr, n_tr + n_va, batch_size):
            e = min(s + batch_size, n_tr + n_va)
            if packed is not None:
                eng.packed_eval_step(packed, rows_map[s:e])
            elif rows_map is not None:
                eng.eval_step(Xd, Yd, sfd, rows=rows_map[s:e])
            else:
                eng.eval_step(Xd[s:e], Yd[s:e], sfd[s:e])
        stop, best_val = _epoch_end(eng, network, hist, ctl, epoch, epochs, n_va, world, rank, dev, verbose, save_weights,
                                    output_dir, best_val)
        if stop:
            break
    return hist


def train_with_args(args):
    """CLI orchestration -- dca/train.py:103-191."""
    from . import io
    from .network import AE_types

    # set seed for reproducibility                                        (dca/train.py:114-117)
    random.seed(42)
    np.random.seed(42)
    torch.manual_seed(42)
    os.environ['PYTHONHASHSEED'] = '0'

    if args.hyper:
        raise NotImplementedError("--hyper (hyperopt search, dca/hyper.py) is outside the accelerated path")

    adata = io.read_dataset(args.input,
                            transpose=(not args.transpose),  # assume gene x cell by default
                            check_counts=args.checkcounts,
                            test_split=args.testsplit)

    preprocess = getattr(args, 'preprocess', 'host')
    if preprocess not in ('host', 'device'):
        raise ValueError("--preprocess must be 'host' or 'device'")
    stream = bool(getattr(args, 'stream', False))
    if stream and preprocess != 'device':
        raise ValueError("--stream needs --preprocess device")
    packed = bool(getattr(args, 'packed', False))
    if packed and preprocess != 'device':
        raise ValueError("--packed needs --preprocess device")
    if packed and stream:
        raise ValueError("--packed and --stream exclude each other: the counts stay packed in GPU or in host memory")
    if packed and args.denoisesubset:
        raise NotImplementedError("--packed trains on every input gene (the expanded batches need n_in == n_out): "
                                  "--denoisesubset is not supported with it")
    if stream and args.denoisesubset:
        raise NotImplementedError("--stream trains on every input gene (the streamed batches need n_in == n_out): "
                                  "--denoisesubset is not supported with it")
    adata = io.normalize(adata,
                         size_factors=args.sizefactors,
                         logtrans_input=args.loginput,
                         normalize_input=args.norminput,
                         device=torch.device('cuda', torch.cuda.current_device()) if preprocess == 'device' else None,
                         stream=stream, packed=packed)
    dd = adata.uns.pop('dca_device_data', None)
    sd = adata.uns.pop('dca_stream_data', None)
    pdd = adata.uns.pop('dca_packed_data', None)

    if args.denoisesubset:
        genelist = list(set(io.read_genelist(args.denoisesubset)))
        assert len(set(genelist) - set(adata.var_names.values)) == 0, \
            'Gene list is not overlapping with genes from the dataset'
        output_size = len(genelist)
    else:
        genelist = None
        output_size = adata.n_vars

    hidden_size = [int(x) for x in args.hiddensize.split(',')] if args.hiddensize.strip() else []
    hidden_dropout = [float(x) for x in args.dropoutrate.split(',')]
    if len(hidden_dropout) == 1:
        hidden_dropout = hidden_dropout[0]

    assert args.type in AE_types, 'loss type not supported'
    input_size = adata.n_vars

    net = AE_types[args.type](input_size=input_size,
                              output_size=output_size,
                              hidden_size=hidden_size,
                              l2_coef=args.l2,
                              l1_coef=args.l1,
                              l2_enc_coef=args.l2enc,
                              l1_enc_coef=args.l1enc,
                              ridge=args.ridge,
                              hidden_dropout=hidden_dropout,
                              input_dropout=args.inputdropout,
                              batchnorm=args.batchnorm,
                              activation=args.activation,
                              init=args.init,
                              debug=args.debug,
                              file_path=args.outputdir)
    net.save()
    net.build()

    train_mask = np.asarray(adata.obs.dca_split == 'train')
    extra = {}
    if dd is not None:
        dd_train = dd.take(train_mask)
        if genelist:
            raw_names = np.asarray(adata.raw.var_names)
            dd_train = dd_train.with_output_genes([int(np.where(raw_names == x)[0][0]) for x in genelist])
        extra['device_data'] = dd_train
    if sd is not None:
        extra['stream_data'] = sd.take(train_mask)
    if pdd is not None:
        extra['packed_data'] = pdd.take(train_mask)
    losses = train(adata[adata.obs.dca_split == 'train'], net,
                   output_dir=args.outputdir,
                   learning_rate=args.learningrate,
                   epochs=args.epochs, batch_size=args.batchsize,
                   early_stop=args.earlystop,
                   reduce_lr=args.reducelr,
                   output_subset=genelist,
                   optimizer=args.optimizer,
                   clip_grad=args.gradclip,
                   save_weights=args.saveweights,
                   tensorboard=args.tensorboard,
                   verbose=True, **extra)

    if genelist:
        predict_columns = adata.var_names[[np.where(adata.var_names == x)[0][0] for x in genelist]]
    else:
        predict_columns = adata.var_names

    # the files of net.predict(adata, mode='full', return_info=True, ...) + net.write(...), written in gene blocks
    # from the device: host memory holds the labels and the text buffers, never a cells x genes output
    net.write_predictions(args.outputdir, adata.obs_names.values, predict_columns, mode='full', return_info=True,
                          device_data=dd, stream_data=sd, packed_data=pdd, adata=adata)
    return losses
