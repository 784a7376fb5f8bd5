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

    ``device_data`` / ``stream_data`` / ``packed_data``: a dataset of the cells of ``adata`` (in order) preprocessed on
    the device -- device_data.DeviceDataset (resident in HBM), stream_data.StreamedDataset (packed counts in pinned
    host memory, streamed as above) or packed_data.PackedDeviceDataset (packed counts in HBM, every batch expanded on
    the device by row index).  X, the raw-count target and the size factors then come from the dataset and adata's
    matrices are not used; the updates are those of the host arrays holding the same values.  Single process only,
    use_raw_as_output only, and ``output_subset`` only with a DeviceDataset whose Y already holds those genes
    (DeviceDataset.with_output_genes).  adata is then only read for ``raw.var_names`` (output_subset) and may be None
    otherwise."""
    stream = kwds.pop('stream', False)
    shuffle = kwds.pop('shuffle', True)
    device_data = kwds.pop('device_data', None)
    stream_data = kwds.pop('stream_data', None)
    packed_data = kwds.pop('packed_data', None)
    if kwds:
        raise TypeError("train() got keyword arguments the accelerated fit loop does not implement: %s" % sorted(kwds))
    from . import _lib as _L
    from .device_data import _one_dataset
    if optimizer not in _L.OPTIMIZERS:
        raise NotImplementedError("optimizer %r is not on the accelerated path (supported: %s)"
                                  % (optimizer, sorted(k for k in _L.OPTIMIZERS if not k.islower())))
    if tensorboard:
        raise NotImplementedError("tensorboard logging is not part of the accelerated path")
    if output_dir is not None:
        os.makedirs(output_dir, exist_ok=True)
    fit = dict(optimizer=optimizer, learning_rate=learning_rate, epochs=epochs, reduce_lr=reduce_lr,
               early_stop=early_stop, clip_grad=clip_grad, verbose=verbose, save_weights=save_weights,
               output_dir=output_dir)
    fit["names"] = _cell_gene_names(adata, output_subset)
    data = _one_dataset(device_data, stream_data, packed_data, stream)
    if data is not None:
        _check_target(data, adata, output_subset, use_raw_as_output)
        eng = network.ensure_engine(max_batch=batch_size)
        data._bind(eng)
        n_tr = _split(data.n, validation_split)
        epoch, validate = data._fit(eng, n_tr, batch_size, shuffle)
        return _fit(eng, network, epoch, validate, data.n - n_tr, **fit)

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
    split_at = _split(N, validation_split)
    rank, world = D.rank_world()

    # cells shard across ranks (SURVEY.md 8e): contiguous row ranges, equal count per rank
    tr_lo, tr_hi = D.shard_bounds(split_at, rank, world, equal=True)
    va_lo, va_hi = D.shard_bounds(N - split_at, rank, world, equal=False)
    tr, va = (tr_lo, tr_hi), (va_lo + split_at, va_hi + split_at)

    if world > 1 and rank == 0 and (split_at % world) and verbose:
        print("dca: %d training cells do not divide over %d ranks; the last %d are left out of every epoch"
              % (split_at, world, split_at % world))
    eng = network.ensure_engine(max_batch=batch_size)
    if stream == 'auto':
        free = torch.cuda.mem_get_info(eng.device)[0]
        stream = (tr_hi - tr_lo + va_hi - va_lo) * X.shape[1] * (4 + eng.params.element_size()) > 0.6 * free
    feed = _host_stream if stream else _host_resident
    epoch, validate = feed(eng, X, Yh, sf, tr, va, batch_size, shuffle, world)
    if world > 1:
        D.broadcast_(eng.params, src=0); D.broadcast_(eng.bn_state, src=0)
        eng.params_changed()
        if torch.distributed.get_backend() == "nccl":
            eng.comm_init()          # gradient exchange inside the library: one CUDA graph per step (dca_train_step_dp)
    return _fit(eng, network, epoch, validate, va[1] - va[0], gscale=1.0 / world, world=world, rank=rank, **fit)


def _cell_gene_names(adata, output_subset):
    """(cell names, output gene names) of an AnnData for the debug checks' messages; None where unknown."""
    if adata is None:
        return None, None
    genes = list(output_subset) if output_subset else getattr(adata, "var_names", None)
    return getattr(adata, "obs_names", None), genes


def _split(n, validation_split):
    """Training rows of n: the tail ``validation_split`` validates (taken before shuffling, as Keras does)."""
    return int(n * (1. - validation_split)) if validation_split and 0. < validation_split < 1. else n


def _check_target(data, adata, output_subset, use_raw_as_output):
    """The rules every dataset kind trains under: one process, the raw counts of its cells as the target, and an
    output_subset only through a DeviceDataset whose Y holds those genes (y_cols)."""
    if D.rank_world()[1] > 1:
        raise NotImplementedError("%s trains on one GPU; a torch.distributed world larger than 1 is not supported"
                                  % data.kind)
    if not use_raw_as_output:
        raise ValueError("%s holds the raw counts as the target: use_raw_as_output=False is not supported" % data.kind)
    if not hasattr(data, "y_cols"):
        if output_subset:
            raise NotImplementedError("%s needs the raw counts of the input genes as the target (no output_subset)"
                                      % data.kind)
    elif output_subset:
        if adata is None:
            raise ValueError("output_subset names genes of adata.raw: pass the AnnData with device_data")
        raw_names = np.asarray(adata.raw.var_names)
        gene_idx = [int(np.where(raw_names == x)[0][0]) for x in output_subset]
        if data.y_cols is None or list(data.y_cols) != gene_idx:
            raise ValueError("output_subset needs a dataset whose Y holds those genes: "
                             "device_data.with_output_genes(<their positions in adata.raw.var_names>)")
    elif data.y_cols is not None:
        raise ValueError("the dataset's Y holds a subset of the genes, but no output_subset was given")
    data._cover(adata)


def _host_resident(eng, X, Yh, sf, tr, va, batch_size, shuffle, world):
    """(epoch, validate) of the rows tr + va of the host arrays, copied to the device once: the training rows
    reshuffled every epoch as Keras does, the gradients all-reduced over the ranks in the step when world > 1."""
    from .device_data import _resident_fit
    (tr_lo, tr_hi), (va_lo, va_hi) = tr, va
    dev = eng.device
    Xd = _to_device(np.concatenate([X[tr_lo:tr_hi], X[va_lo:va_hi]]), eng.x_dtype, dev)
    Yd = _to_device(np.concatenate([Yh[tr_lo:tr_hi], Yh[va_lo:va_hi]]), torch.float32, dev)
    sfd = _to_device(np.concatenate([sf[tr_lo:tr_hi], sf[va_lo:va_hi]]), torch.float32, dev)
    n_tr = tr_hi - tr_lo
    step = eng.train_step_allreduce if world > 1 else eng.train_step     # NCCL all-reduce overlapped with the backward
    epoch, validate = _resident_fit(eng, n_tr, n_tr + va_hi - va_lo, batch_size, shuffle,
                                    lambda rows: step(Xd, Yd, sfd, rows=rows),
                                    lambda s, e: eng.eval_step(Xd[s:e], Yd[s:e], sfd[s:e]))

    def cells(check):                             # positions in the copied rows -> rows of adata
        return check and (lambda p: check(np.where(p < n_tr, tr_lo + p, va_lo + p - n_tr)))
    return (lambda update, check=None: epoch(update, cells(check))), (lambda check=None: validate(cells(check)))


def _host_stream(eng, X, Yh, sf, tr, va, batch_size, shuffle, world):
    """Training from host memory (dca_stream_*): see train().  X is only used for the (small, resident) validation rows;
    the training rows travel as bit-packed raw counts and are normalised on the device."""
    from . import io as dio
    from .hostmem import pin_near_gpu
    from .stream_data import stream_epoch
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
    steps = stream_epoch(eng, n_tr, batch_size, shuffle, lambda: eng.stream_begin(packed, sf_h, batch_size), order0)

    def epoch(update, check=None):
        if world == 1:
            return steps(update, check)

        def reduced():                            # the gradients summed over the ranks before every update
            eng.allreduce_grads() if getattr(eng, "_comm", False) else D.all_reduce_sum_(eng.grads)
            update()
        steps(reduced, check)

    def validate(check=None):
        for s0 in range(0, n_va, batch_size):
            e = min(s0 + batch_size, n_va)
            eng.eval_step(Xv[s0:e], Yv[s0:e], sfv[s0:e])
            if check:
                check(np.arange(va_lo + s0, va_lo + e))
    return epoch, validate


def _fit(eng, network, epoch, validate, n_va, optimizer, learning_rate, epochs, reduce_lr, early_stop, clip_grad, verbose,
         save_weights, output_dir, names=(None, None), gscale=1.0, world=1, rank=0):
    """The fit loop of every input: optimizer, ReduceLROnPlateau / EarlyStopping, history and ModelCheckpoint around
    epoch(update) -- one epoch's training steps, update() after each -- and validate(), the pass over the n_va
    validation rows.  With network.debug, both also get a check of every step's debug report (_DebugChecks)."""
    debug = bool(getattr(network, "debug", False))
    if debug or getattr(eng, "debug_checks", False) is True:       # a run without --debug touches no engine state
        eng.set_debug_checks(debug)
    # opt.__dict__[optimizer](clipvalue=clip_grad[, lr=learning_rate])                   (dca/train.py:54-57)
    default_lr = eng.set_optimizer(optimizer)
    eng.reset_optimizer()
    ctl = PlateauAndStop(float(default_lr if learning_rate is None else learning_rate), reduce_lr, early_stop, verbose)
    hist = History()
    if verbose:
        print(network.summary())
    dev = eng.device
    # run on a non-default stream (CUDA-graph replay of the step needs a capturable stream)
    torch.cuda.synchronize(dev)
    prev_stream = torch.cuda.current_stream(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))
    best_val = np.inf
    try:
        for e in range(epochs):
            eng.read_epoch_acc(reset=True)
            update = lambda: eng.apply_update(ctl.lr, clip_grad, gscale)     # noqa: E731
            if debug:
                dbg = _DebugChecks(eng, e + 1, names, world, dev)
                epoch(update, dbg.training)
                validate(dbg.validation)
                dbg.end_validation()
            else:
                epoch(update)
                validate()
            stop, best_val = _epoch_end(eng, network, hist, ctl, e, epochs, n_va, world, rank, dev, verbose, save_weights,
                                        output_dir, best_val)
            if stop:
                break
    finally:
        torch.cuda.synchronize(dev)
        torch.cuda.set_stream(prev_stream)
    if not hist.history["val_loss"]:
        del hist.history["val_loss"]
    return hist


DEBUG_TERMS = ("y_pred", "t1", "t2")


def debug_message(report, epoch, phase, batch, positions, obs_names=None, gene_names=None):
    """The FloatingPointError message of a failing debug report: the reference's message for the first failing term,
    in the order y_pred, t1, t2 (dca/loss.py:87-100), then where -- epoch (from 1), 'training' or 'validation', the
    batch index (from 0), the cell (its position in the dataset, positions[batch row], and its name) and the gene of
    that term's first non-finite element -- and the three counts.  report: engine.read_debug_report()'s dict, with
    counts summed over the ranks; its "first" entry is None when the element lies in another rank's share."""
    counts = [int(c) for c in report["count"]]
    k = next(i for i in range(3) if counts[i] > 0)

    def named(names, i):
        return "" if names is None or i >= len(names) else " (%s)" % names[i]
    msg = "%s has inf/nans: epoch %d, %s batch %d" % (DEBUG_TERMS[k], epoch, phase, batch)
    first = report["first"][k]
    if first is None:
        msg += ", in another rank's share of the batch"
    else:
        row, gene = first
        cell = int(positions[row])
        msg += ", cell %d%s, gene %d%s" % (cell, named(obs_names, cell), gene, named(gene_names, gene))
    return msg + "; non-finite elements: y_pred %d, t1 %d, t2 %d" % tuple(counts)


class _DebugChecks:
    """--debug in the fit loop of one epoch: the report of every training step is read before its update, so a
    failing batch's update is never applied (the network keeps the weights from before it, as the reference's abort
    leaves them, and the BatchNorm moving statistics that batch's forward pass moved are put back); the report of every
    validation batch after it.  With world > 1 the training counts are summed over
    the ranks every step, so every rank raises at the same step; the validation counts once after the pass (the ranks'
    validation shares need not have the same number of batches)."""

    def __init__(self, eng, epoch, names, world, dev):
        self.eng, self.epoch, self.world, self.dev = eng, epoch, world, dev
        self.obs_names, self.gene_names = names
        self.n_train = self.n_val = 0
        self.val_failure = None
        self.bn = eng.bn_state.clone() if eng.bn_state.numel() else None      # as after the last clean step

    def _summed(self, counts):
        return [int(c) for c in D.all_reduce_sum_host(np.asarray(counts, dtype=np.float64), self.dev)]

    def training(self, positions):
        r = self.eng.read_debug_report()
        if self.world > 1:
            r["count"] = self._summed(r["count"])
        batch, self.n_train = self.n_train, self.n_train + 1
        if any(r["count"]):
            if self.bn is not None:
                self.eng.bn_state.copy_(self.bn)
            raise FloatingPointError(debug_message(r, self.epoch, "training", batch, positions, self.obs_names,
                                                   self.gene_names))
        if self.bn is not None:
            self.bn.copy_(self.eng.bn_state)

    def validation(self, positions):
        r = self.eng.read_debug_report()
        batch, self.n_val = self.n_val, self.n_val + 1
        if any(r["count"]) and self.val_failure is None:
            self.val_failure = debug_message(r, self.epoch, "validation", batch, positions, self.obs_names,
                                             self.gene_names)
            if self.world == 1:
                raise FloatingPointError(self.val_failure)

    def end_validation(self):
        failed = self.val_failure is not None
        if self.world > 1:
            failed = self._summed([int(failed)])[0] > 0
        if failed:
            raise FloatingPointError(self.val_failure or "validation has inf/nans on another rank: epoch %d" % self.epoch)


def _epoch_end(eng, network, hist, ctl, epoch, epochs, n_va, world, rank, dev, verbose, save_weights, output_dir, best_val):
    """Epoch bookkeeping: reduce the accumulators over ranks, history, ModelCheckpoint, ReduceLROnPlateau /
    EarlyStopping.  Returns (stop, best_val)."""
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
    ds = next((adata.uns.pop(k) for k in ('dca_device_data', 'dca_stream_data', 'dca_packed_data') if k in adata.uns),
              None)

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
    if ds is not None:
        ds_train = ds.take(train_mask)
        if genelist:                              # a DeviceDataset: --stream and --packed reject --denoisesubset
            raw_names = np.asarray(adata.raw.var_names)
            ds_train = ds_train.with_output_genes([int(np.where(raw_names == x)[0][0]) for x in genelist])
        extra[ds.kind] = ds_train
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
                          adata=adata, gzip=bool(getattr(args, 'gzip', False)),
                          **({ds.kind: ds} if ds is not None else {}))
    return losses
