"""Python face of the C-ABI engine (include/dca_b200.h).

``DeviceEngine`` owns a torch uint8 arena (torch is only the allocator), hands its device
pointer to ``dca_create`` and exposes the parameter / gradient / state regions as torch views
so that ``torch.distributed`` can all-reduce the flat gradient buffer in place.
All compute happens inside libdca_b200.so; nothing here falls back to torch ops.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import check

# Keras / TF defaults the reference relies on (SURVEY.md Appendix B) -- single place to correct.
KERAS_DEFAULTS = dict(bn_momentum=0.99, bn_eps=1e-3, rms_rho=0.9, rms_eps=1e-7, rms_lr=1e-3)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


class DeviceEngine:
    def __init__(self, n_in: int, n_out: int, hidden: Sequence[int] = (64, 32, 64),
                 ae_type: str = "zinb-conddisp", batchnorm: bool = True, max_batch: int = 32,
                 x_dtype: str = "float32", ridge: float = 0.0, l1: float = 0.0, l2: float = 0.0,
                 l1_enc: float = 0.0, l2_enc: float = 0.0, gemm_path: str = "auto",
                 device: Optional[torch.device] = None, seed: Optional[int] = 0, sharedpi: bool = False,
                 sync_bn: bool = False, activation: str = "relu", hidden_dropout=0.0, input_dropout: float = 0.0,
                 dropout_seed: Optional[int] = None, init: str = "glorot_uniform"):
        if ae_type not in _lib.AE_TYPE_IDS:
            raise NotImplementedError("ae_type %r is not on the accelerated path (supported: %s)"
                                      % (ae_type, sorted(_lib.AE_TYPE_IDS)))
        self.lib = _lib.load()
        self.init = init
        self._init_spec = _lib.initializer(init)         # kernel_initializer of every kernel (dca/network.py:124-126)
        if not torch.cuda.is_available():
            raise _lib.DcaError("dca_b200 needs a CUDA device (H100); there is no CPU fallback")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.n_in, self.n_out, self.hidden = int(n_in), int(n_out), tuple(int(h) for h in hidden)
        self.ae_type, self.batchnorm, self.max_batch = ae_type, bool(batchnorm), int(max_batch)
        self.x_dtype = {"float32": torch.float32, "bfloat16": torch.bfloat16}[x_dtype]
        cfg = _lib.default_config()
        cfg.n_in, cfg.n_out = self.n_in, self.n_out
        if len(self.hidden) > _lib.DCA_MAX_HIDDEN:
            raise ValueError("at most %d hidden layers" % _lib.DCA_MAX_HIDDEN)
        cfg.n_hidden = len(self.hidden)
        for i, h in enumerate(self.hidden):
            cfg.hidden[i] = h
        cfg.ae_type = _lib.AE_TYPE_IDS[ae_type]
        cfg.batchnorm = int(self.batchnorm)
        cfg.max_batch = self.max_batch
        cfg.x_dtype = _lib.BF16 if self.x_dtype == torch.bfloat16 else _lib.F32
        cfg.gemm_path = {"auto": _lib.GEMM_AUTO, "generic": _lib.GEMM_GENERIC, "tcgen05": _lib.GEMM_TCGEN05}[gemm_path]
        cfg.ridge, cfg.l1, cfg.l2, cfg.l1_enc, cfg.l2_enc = ridge, l1, l2, l1_enc, l2_enc
        cfg.elempi_shared = int(bool(sharedpi))          # zinb-elempi only (dca/network.py:425-427)
        cfg.sync_bn = int(bool(sync_bn))                 # BatchNorm over the global batch in data-parallel runs (comm_init)
        # hidden activation + dropout (dca/network.py:98-99,129-138); anything but relu / rate 0 takes the per-layer hidden path
        if activation not in _lib.ACTIVATION_IDS:
            raise NotImplementedError("activation %r is not on the accelerated path (supported: %s)"
                                      % (activation, sorted(_lib.ACTIVATION_IDS)))
        cfg.activation = _lib.ACTIVATION_IDS[activation]
        rates = list(hidden_dropout) if isinstance(hidden_dropout, (list, tuple)) else [hidden_dropout] * len(self.hidden)
        if len(rates) != len(self.hidden):
            raise ValueError("hidden_dropout needs one rate per hidden layer")
        for i, r in enumerate(rates):
            cfg.hidden_dropout[i] = float(r)
        cfg.input_dropout = float(input_dropout)
        self.activation, self.hidden_dropout, self.input_dropout = activation, [float(r) for r in rates], float(input_dropout)
        if dropout_seed is None:                        # data-parallel replicas draw different masks
            rank = torch.distributed.get_rank() if (torch.distributed.is_available() and torch.distributed.is_initialized()) else 0
            dropout_seed = (seed or 0) * 1000003 + 12345 + 7919 * rank
        self.dropout_seed = int(dropout_seed) & (2 ** 64 - 1)
        cfg.dropout_seed = self.dropout_seed
        cfg.bn_momentum, cfg.bn_eps = KERAS_DEFAULTS["bn_momentum"], KERAS_DEFAULTS["bn_eps"]
        cfg.rms_rho, cfg.rms_eps = KERAS_DEFAULTS["rms_rho"], KERAS_DEFAULTS["rms_eps"]
        self.cfg = cfg
        self.debug_checks = False
        nbytes = C.c_size_t()
        check(self.lib.dca_arena_bytes(C.byref(cfg), C.byref(nbytes)), "dca_arena_bytes")
        with torch.cuda.device(self.device):
            self.arena = torch.empty(nbytes.value + 256, dtype=torch.uint8, device=self.device)
            base = self.arena.data_ptr()
            self._arena_off = (-base) % 256
            self.handle = C.c_void_p()
            check(self.lib.dca_create(C.byref(cfg), C.c_void_p(base + self._arena_off), nbytes.value,
                                      C.byref(self.handle)), "dca_create")
        self.params = self._region(_lib.REGION_PARAMS, torch.float32)
        self.grads = self._region(_lib.REGION_GRADS, torch.float32)       # [P+2]: ..., loss, nonfinite
        self.rms = self._region(_lib.REGION_RMS, torch.float32)
        self.bn_state = self._region(_lib.REGION_BN_STATE, torch.float32)
        self.epoch_acc = self._region(_lib.REGION_EPOCH_ACC, torch.float64)
        self.n_params = self.params.numel()
        hb = C.c_int64()
        check(self.lib.dca_grad_buckets(self.handle, C.byref(hb)), "dca_grad_buckets")
        self.head_bucket = int(hb.value)
        self.param_info = self._infos(self.lib.dca_param_count, self.lib.dca_param_info)
        self.state_info = self._infos(self.lib.dca_state_count, self.lib.dca_state_info)
        if seed is not None:
            try:
                self.init_params(seed)
            except ValueError:
                self.close()
                raise

    # ------------------------------------------------------------------ plumbing
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _region(self, rid, dtype):
        p, n = C.c_void_p(), C.c_int64()
        check(self.lib.dca_region(self.handle, rid, C.byref(p), C.byref(n)), "dca_region")
        if n.value == 0:
            return torch.empty(0, dtype=dtype, device=self.device)
        off = p.value - self.arena.data_ptr()
        item = torch.empty(0, dtype=dtype).element_size()
        return self.arena[off: off + n.value * item].view(dtype)

    def _infos(self, count_fn, info_fn):
        n, nt = C.c_int64(), C.c_int32()
        check(count_fn(self.handle, C.byref(n), C.byref(nt)))
        out = []
        for i in range(nt.value):
            ti = _lib.TensorInfo()
            check(info_fn(self.handle, i, C.byref(ti)))
            out.append((ti.name.decode(), int(ti.offset), int(ti.rows), int(ti.cols)))
        return out

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle.value:
            if getattr(self, "_comm", False):
                self.lib.dca_comm_destroy(self.handle); self._comm = False
            self.lib.dca_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ parameters
    def init_params(self, seed: int):
        """Kernels drawn by the engine's initializer (``init``), biases, BatchNorm and theta at their Keras defaults.
        ValueError when the initializer does not apply to a kernel of the model (orthogonal / identity on the 1-D
        'pi/kernel' of zinb-elempi)."""
        check(self.lib.dca_init_params_ex(self.handle, C.c_uint64(seed & (2 ** 64 - 1)), C.byref(self._init_spec),
                                          self._stream()), "dca_init_params_ex")

    def params_changed(self):
        check(self.lib.dca_params_changed(self.handle, self._stream()), "dca_params_changed")

    def get_weights(self) -> Dict[str, np.ndarray]:
        """All tensors (trainable + BatchNorm moving statistics) by reference name, Keras layouts."""
        torch.cuda.synchronize(self.device)
        flat = self.params.detach().cpu().numpy()
        out = {}
        for name, off, r, c in self.param_info:
            a = flat[off: off + r * c]
            out[name] = a.reshape(r, c).copy() if name.endswith("/kernel") else a.copy()
        sflat = self.bn_state.detach().cpu().numpy()
        for name, off, r, c in self.state_info:
            out[name] = sflat[off: off + r * c].copy()
        return out

    def set_weights(self, weights: Dict[str, np.ndarray], strict: bool = True):
        flat = self.params.detach().cpu().numpy().copy()
        sflat = self.bn_state.detach().cpu().numpy().copy()
        seen = set()
        for name, off, r, c in self.param_info:
            if name in weights:
                w = np.asarray(weights[name], np.float32).reshape(-1)
                if w.size != r * c:
                    raise ValueError("shape mismatch for %s: expected %d values, got %d" % (name, r * c, w.size))
                flat[off: off + r * c] = w; seen.add(name)
            elif strict:
                raise KeyError("missing weight %r" % name)
        for name, off, r, c in self.state_info:
            if name in weights:
                sflat[off: off + r * c] = np.asarray(weights[name], np.float32).reshape(-1); seen.add(name)
            elif strict:
                raise KeyError("missing state %r" % name)
        self.params.copy_(torch.from_numpy(flat))
        if sflat.size:
            self.bn_state.copy_(torch.from_numpy(sflat))
        self.params_changed()

    def reset_optimizer(self):
        """Clear the optimizer state (accumulators + iteration count) -- what compiling a fresh Keras optimizer does."""
        check(self.lib.dca_reset_optimizer(self.handle, self._stream()), "dca_reset_optimizer")

    def set_optimizer(self, name: str) -> float:
        """Select the update rule of apply_update by its keras.optimizers name (dca/train.py:54-57); returns the Keras
        default learning rate of that class (used when learning_rate is None)."""
        if name not in _lib.OPTIMIZERS:
            raise NotImplementedError("optimizer %r is not on the accelerated path (supported: %s)"
                                      % (name, sorted(k for k in _lib.OPTIMIZERS if not k.islower())))
        kind, default_lr = _lib.OPTIMIZERS[name]
        check(self.lib.dca_set_optimizer(self.handle, kind, self._stream()), "dca_set_optimizer")
        self.optimizer = name
        return default_lr

    # ------------------------------------------------------------------ hot path
    def _check_inputs(self, X, Y, sf, rows, batch):
        if X.dtype != self.x_dtype:
            raise ValueError("X dtype %s does not match engine x_dtype %s" % (X.dtype, self.x_dtype))
        if X.dim() != 2 or X.shape[1] != self.n_in or X.stride(1) != 1:
            raise ValueError("X must be (rows, %d) row-major" % self.n_in)
        if Y is not None and (Y.dtype != torch.float32 or Y.dim() != 2 or Y.shape[1] != self.n_out or Y.stride(1) != 1):
            raise ValueError("Y must be float32 (rows, %d) row-major" % self.n_out)
        if sf is not None and (sf.dtype != torch.float32 or sf.dim() != 1 or not sf.is_contiguous()):
            raise ValueError("size factors must be a contiguous float32 vector")
        if rows is not None:
            if rows.dtype != torch.int32 or not rows.is_contiguous():
                raise ValueError("rows must be a contiguous int32 tensor")
            batch = rows.numel() if batch is None else batch
        else:
            batch = X.shape[0] if batch is None else batch
        if batch > self.max_batch:
            raise ValueError("batch %d > max_batch %d" % (batch, self.max_batch))
        return int(batch)

    def train_step(self, X, Y, sf, rows=None, batch=None, phase=0):
        """Forward + loss + backward into ``self.grads`` (no update).  phase 1 / 2 run the two halves
        (see dca_train_step_phase): after phase 1 ``self.grads[self.head_bucket:]`` is final."""
        b = self._check_inputs(X, Y, sf, rows, batch)
        if phase == 0:
            check(self.lib.dca_train_step(self.handle, _ptr(X), X.stride(0), _ptr(Y), Y.stride(0), _ptr(sf), _ptr(rows),
                                          b, self._stream()), "dca_train_step")
        else:
            check(self.lib.dca_train_step_phase(self.handle, _ptr(X), X.stride(0), _ptr(Y), Y.stride(0), _ptr(sf),
                                                _ptr(rows), b, phase, self._stream()), "dca_train_step_phase")

    def comm_init(self, single_rank: bool = False):
        """Create the engine's own NCCL communicator (dca_comm_init) over the ranks of the default torch.distributed
        group: rank 0 draws the unique id, torch.distributed carries its 128 bytes to the others.  Afterwards
        train_step_allreduce runs the gradient exchange inside the library (one CUDA graph per step).

        single_rank=True builds a one-rank communicator without torch.distributed: the data-parallel step
        (dca_train_step_dp, with its DCA_DP_* launch plans) then runs on this GPU alone and its all-reduces leave the
        gradients as they are -- the way to exercise that step on a single GPU."""
        if single_rank:
            buf = (C.c_char * 128)()
            check(self.lib.dca_comm_unique_id(buf), "dca_comm_unique_id")
            with torch.cuda.device(self.device):
                check(self.lib.dca_comm_init(self.handle, buf.raw, 0, 1), "dca_comm_init")
            self._comm = True
            return True
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
            return False
        ident = torch.zeros(128, dtype=torch.uint8)
        if dist.get_rank() == 0:
            buf = (C.c_char * 128)()
            check(self.lib.dca_comm_unique_id(buf), "dca_comm_unique_id")
            ident = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
        ident = ident.to(self.device)
        dist.broadcast(ident, 0)
        raw = bytes(ident.cpu().numpy().tobytes())
        with torch.cuda.device(self.device):
            check(self.lib.dca_comm_init(self.handle, raw, dist.get_rank(), dist.get_world_size()), "dca_comm_init")
        self._comm = True
        return True

    def allreduce_grads(self):
        """Sum all-reduce of the flat gradient buffer (+ loss slot, flag) over the engine's communicator."""
        check(self.lib.dca_allreduce(self.handle, self._stream()), "dca_allreduce")

    def train_step_allreduce(self, X, Y, sf, rows=None):
        """Data-parallel step: the all-reduce of the head-gradient bucket overlaps the hidden-stack backward.  With an
        engine communicator (comm_init) the whole sequence is one library call / one CUDA graph."""
        if getattr(self, "_comm", False):
            b = self._check_inputs(X, Y, sf, rows, None)
            check(self.lib.dca_train_step_dp(self.handle, _ptr(X), X.stride(0), _ptr(Y), Y.stride(0), _ptr(sf), _ptr(rows),
                                             b, self._stream()), "dca_train_step_dp")
            return
        import torch.distributed as dist
        self.train_step(X, Y, sf, rows=rows, phase=1)
        w1 = dist.all_reduce(self.grads[self.head_bucket:], async_op=True)
        self.train_step(X, Y, sf, rows=rows, phase=2)
        w2 = dist.all_reduce(self.grads[:self.head_bucket], async_op=True) if self.head_bucket > 0 else None
        w1.wait()
        if w2 is not None:
            w2.wait()

    def apply_update(self, lr: float, clip: float = 5.0, grad_scale: float = 1.0):
        check(self.lib.dca_apply_update(self.handle, lr, clip, grad_scale, self._stream()), "dca_apply_update")

    def eval_step(self, X, Y, sf, rows=None, batch=None):
        b = self._check_inputs(X, Y, sf, rows, batch)
        check(self.lib.dca_eval_step(self.handle, _ptr(X), X.stride(0), _ptr(Y), Y.stride(0), _ptr(sf), _ptr(rows),
                                     b, self._stream()), "dca_eval_step")

    def predict(self, X, sf, rows=None, batch=None, mean=None, disp=None, pi=None, latent=None):
        """mean (* size factor), dispersion, pi: [batch x n_out] -- for the per-cell heads of 'nb-shared' / 'zinb-shared'
        dispersion and pi are [batch] (or [batch x 1]); latent: [batch x hidden[center]]."""
        b = self._check_inputs(X, None, sf, rows, batch)
        ld = None
        for t in (mean, disp, pi):
            if t is not None and t.dim() == 2 and t.shape[1] > 1:
                ld = t.stride(0) if ld is None else ld
                if t.stride(0) != ld:
                    raise ValueError("outputs must share a leading dimension")
        check(self.lib.dca_predict(self.handle, _ptr(X), X.stride(0), _ptr(sf), _ptr(rows), b, _ptr(mean), _ptr(disp),
                                   _ptr(pi), ld or self.n_out, _ptr(latent), self._stream()), "dca_predict")

    def read_loss(self):
        l, nf = C.c_float(), C.c_int32()
        check(self.lib.dca_read_loss(self.handle, C.byref(l), C.byref(nf), self._stream()), "dca_read_loss")
        return float("inf") if nf.value else l.value

    def read_epoch_acc(self, reset=True):
        acc = (C.c_double * 4)()
        check(self.lib.dca_read_epoch_acc(self.handle, C.byref(acc), int(reset), self._stream()), "dca_read_epoch_acc")
        return list(acc)

    def set_debug_checks(self, on: bool):
        """The reference's debug checks (dca/loss.py:87-100) inside the loss kernels of every later training and
        validation step (dca_set_debug_checks); read each step's report with read_debug_report."""
        check(self.lib.dca_set_debug_checks(self.handle, int(bool(on))), "dca_set_debug_checks")
        self.debug_checks = bool(on)

    def read_debug_report(self):
        """The debug report of the last step (waits for it): {"count": [y_pred, t1, t2] non-finite elements,
        "first": per term (batch row, gene) of its first non-finite element in row-major order, or None}."""
        r = _lib.DebugReport()
        r.struct_bytes = C.sizeof(_lib.DebugReport)
        check(self.lib.dca_read_debug_report(self.handle, C.byref(r), self._stream()), "dca_read_debug_report")
        return {"count": [int(c) for c in r.count],
                "first": [None if r.first_row[k] < 0 else (int(r.first_row[k]), int(r.first_gene[k])) for k in range(3)]}

    def train_step_host(self, x_host: torch.Tensor, y_host: torch.Tensor, sf_host: Optional[torch.Tensor],
                        lr: float, clip: float = 5.0) -> float:
        """End-to-end step from HOST (pinned) buffers through dca_train_step_host: x_host [b x n_in] of the engine's
        x_dtype, y_host float32 [b x n_out], sf_host float32 [b] or None, all contiguous."""
        def host(t, dtype, shape, what):
            if t.is_cuda or t.dtype != dtype or tuple(t.shape) != shape or not t.is_contiguous():
                raise ValueError("train_step_host: %s must be a contiguous %s HOST tensor of shape %s (got %s %s%s)"
                                 % (what, dtype, shape, t.dtype, tuple(t.shape), " on the device" if t.is_cuda else ""))
        b = x_host.shape[0] if x_host.dim() == 2 else -1
        host(x_host, self.x_dtype, (b, self.n_in), "x_host")
        host(y_host, torch.float32, (b, self.n_out), "y_host")
        if sf_host is not None:
            host(sf_host, torch.float32, (b,), "sf_host")
        out = C.c_float()
        check(self.lib.dca_train_step_host(self.handle, x_host.data_ptr(), y_host.data_ptr(),
                                           None if sf_host is None else sf_host.data_ptr(), b, lr, clip,
                                           C.byref(out), self._stream()), "dca_train_step_host")
        return out.value

    # ------------------------------------------------------------------ streaming from host counts
    def set_input_transform(self, gene_mean=None, gene_std=None, use_size_factors=True, use_log1p=True):
        """On-device restatement of io.normalize for streamed batches: X = ((log1p)(y/sf) - mean)/std."""
        if gene_mean is None:
            check(self.lib.dca_set_input_transform(self.handle, None, None, int(use_size_factors), int(use_log1p), self._stream()),
                  "dca_set_input_transform")
            return
        mean = np.ascontiguousarray(gene_mean, dtype=np.float32)
        std = np.asarray(gene_std, dtype=np.float64).copy(); std[std == 0] = 1.0
        inv = np.ascontiguousarray(1.0 / std, dtype=np.float32)
        if mean.size != self.n_in or inv.size != self.n_in:
            raise ValueError("gene_mean / gene_std must have %d entries" % self.n_in)
        check(self.lib.dca_set_input_transform(self.handle, mean.ctypes.data, inv.ctypes.data, int(use_size_factors),
                                               int(use_log1p), self._stream()), "dca_set_input_transform")

    def set_input_transform_exact(self, gene_mean, gene_std, median: float, flags: int):
        """The exact transform of the device preprocessing for streamed batches (dca_set_input_transform_exact): the X
        DeviceDataset stores for the same counts.  gene_mean / gene_std: fp64 per gene; flags: device_data.PRE_*."""
        mean = np.ascontiguousarray(gene_mean, dtype=np.float64)
        std = np.ascontiguousarray(gene_std, dtype=np.float64)
        if mean.size != self.n_in or std.size != self.n_in:
            raise ValueError("gene_mean / gene_std must have %d entries" % self.n_in)
        check(self.lib.dca_set_input_transform_exact(self.handle, mean.ctypes.data, std.ctypes.data, float(median),
                                                     int(flags), self._stream()), "dca_set_input_transform_exact")

    def stream_row_totals(self, n_counts: torch.Tensor):
        """Per-row fp64 totals of the active stream's rows for the exact transform: a pinned HOST float64 tensor, kept
        until stream_end."""
        if n_counts.is_cuda or n_counts.dtype != torch.float64 or not n_counts.is_contiguous():
            raise ValueError("the row totals must be a contiguous float64 HOST tensor")
        self._stream_keep = tuple(self._stream_keep or ()) + (n_counts,)
        check(self.lib.dca_stream_row_totals(self.handle, n_counts.data_ptr()), "dca_stream_row_totals")

    def stream_begin(self, counts, sf: Optional[torch.Tensor], batch: int):
        """Train from HOST memory.  counts: a HOST uint16 tensor [n_rows x n_in] (pin it, hostmem.pin_near_gpu), or an
        io.PackedCounts (4/8/16 bits per entry + overflow list, see io.pack_counts) whose arrays are pinned
        here (with n_in off a multiple of 8: packed with pad_genes=True, and the exact transform set); sf: HOST
        float32 [n_rows] or None."""
        if sf is not None and sf.is_cuda:
            raise ValueError("stream_begin takes HOST tensors")
        if isinstance(counts, torch.Tensor):
            if counts.dtype != torch.uint16 or counts.dim() != 2 or counts.shape[1] != self.n_in or counts.stride(1) != 1:
                raise ValueError("counts must be a uint16 (rows, %d) row-major host tensor" % self.n_in)
            if counts.is_cuda:
                raise ValueError("stream_begin takes HOST tensors")
            self._stream_keep = (counts, sf)
            check(self.lib.dca_stream_begin(self.handle, counts.data_ptr(), counts.stride(0),
                                            None if sf is None else sf.data_ptr(), counts.shape[0], batch, self._stream()),
                  "dca_stream_begin")
            return
        pc = counts
        if pc.genes != self.n_in or pc.n_genes != (self.n_in + 7) // 8 * 8:
            raise ValueError("packed counts have %d genes (stored %d wide), the engine %d"
                             % (pc.genes, pc.n_genes, self.n_in))

        from .stream_data import pin_packed
        packed, indptr, entries = pin_packed(pc, self.device.index or 0)[:3]
        self._stream_keep = pc._pinned + (sf,)
        if pc.bits == 1:                              # sparse format: bitmap + nibble stream (dca_stream_begin_sparse)
            check(self.lib.dca_stream_begin_sparse(self.handle, packed.data_ptr(), pc._pinned[3].data_ptr(), pc._pinned[4].data_ptr(),
                                                   indptr.data_ptr(), entries.data_ptr(), None if sf is None else sf.data_ptr(),
                                                   pc.n_rows, batch, self._stream()), "dca_stream_begin_sparse")
            return
        check(self.lib.dca_stream_begin_packed(self.handle, packed.data_ptr(), pc.bits, packed.shape[-1] if packed.dim() == 2 else 0,
                                               indptr.data_ptr(), entries.data_ptr(), None if sf is None else sf.data_ptr(),
                                               pc.n_rows, batch, self._stream()), "dca_stream_begin_packed")

    # ------------------------------------------------------------------ packed counts resident in device memory
    def _packed_rows(self, pd, rows):
        if pd.device != self.device or pd.x_dtype != self.x_dtype:
            raise ValueError("packed_data X is %s on %s, the engine expects %s on %s"
                             % (pd.x_dtype, pd.device, self.x_dtype, self.device))
        if rows.dtype != torch.int32 or not rows.is_contiguous() or not rows.is_cuda:
            raise ValueError("rows must be a contiguous int32 device tensor")
        if rows.numel() > self.max_batch:
            raise ValueError("batch %d > max_batch %d" % (rows.numel(), self.max_batch))
        return C.byref(pd.desc), rows.data_ptr(), int(rows.numel())

    def packed_train_step(self, pd, rows):
        """train_step on rows ``rows`` (int32 device tensor of storage rows) of a packed_data.PackedDeviceDataset: the
        rows are expanded on the device with the transform of set_input_transform_exact (dca_packed_train_step)."""
        src, r, b = self._packed_rows(pd, rows)
        check(self.lib.dca_packed_train_step(self.handle, src, r, b, self._stream()), "dca_packed_train_step")

    def packed_eval_step(self, pd, rows):
        src, r, b = self._packed_rows(pd, rows)
        check(self.lib.dca_packed_eval_step(self.handle, src, r, b, self._stream()), "dca_packed_eval_step")

    def packed_predict(self, pd, rows, mean=None, disp=None, pi=None, latent=None):
        """predict() on rows ``rows`` of a PackedDeviceDataset (outputs as there)."""
        src, r, b = self._packed_rows(pd, rows)
        ld = None
        for t in (mean, disp, pi):
            if t is not None and t.dim() == 2 and t.shape[1] > 1:
                ld = t.stride(0) if ld is None else ld
                if t.stride(0) != ld:
                    raise ValueError("outputs must share a leading dimension")
        check(self.lib.dca_packed_predict(self.handle, src, r, b, _ptr(mean), _ptr(disp), _ptr(pi), ld or self.n_out,
                                          _ptr(latent), self._stream()), "dca_packed_predict")

    def set_loss_ring(self, ring: Optional[torch.Tensor]):
        """Mirror every step's loss into the pinned host float32 tensor `ring` (slot k % len for the k-th
        apply_update after this call); None switches it off."""
        if ring is None:
            check(self.lib.dca_set_loss_ring(self.handle, None, 0), "dca_set_loss_ring"); self._ring_keep = None
            return
        if ring.dtype != torch.float32 or ring.is_cuda or not ring.is_pinned() or not ring.is_contiguous():
            raise ValueError("the loss ring must be a contiguous pinned float32 host tensor")
        self._ring_keep = ring
        check(self.lib.dca_set_loss_ring(self.handle, ring.data_ptr(), ring.numel()), "dca_set_loss_ring")

    def stream_step(self, batch_index: int, next_batch_index: int = -1):
        """Forward + loss + backward of host batch `batch_index`; the copy of `next_batch_index` overlaps it."""
        check(self.lib.dca_stream_step(self.handle, batch_index, next_batch_index, self._stream()), "dca_stream_step")

    def stream_eval(self, batch_index: int, next_batch_index: int = -1):
        """eval_step on host batch `batch_index` of the active stream (validation pass); the copy and expansion of
        `next_batch_index` overlap it."""
        check(self.lib.dca_stream_eval(self.handle, batch_index, next_batch_index, self._stream()), "dca_stream_eval")

    def stream_capacity(self):
        """(overflow entries, bytes of sparse non-zero codes) one streamed batch may carry (dca_stream_capacity)."""
        ovf, nib = C.c_int64(), C.c_int64()
        check(self.lib.dca_stream_capacity(self.handle, C.byref(ovf), C.byref(nib)), "dca_stream_capacity")
        return int(ovf.value), int(nib.value)

    def stream_predict(self, batch_index: int, next_batch_index: int = -1, mean=None, disp=None, pi=None, latent=None):
        """predict() on host batch `batch_index` of the active stream (outputs as there); the copy and expansion of
        `next_batch_index` overlap it."""
        ld = None
        for t in (mean, disp, pi):
            if t is not None and t.dim() == 2 and t.shape[1] > 1:
                ld = t.stride(0) if ld is None else ld
                if t.stride(0) != ld:
                    raise ValueError("outputs must share a leading dimension")
        check(self.lib.dca_stream_predict(self.handle, batch_index, next_batch_index, _ptr(mean), _ptr(disp), _ptr(pi),
                                          ld or self.n_out, _ptr(latent), self._stream()), "dca_stream_predict")

    def stream_end(self):
        check(self.lib.dca_stream_end(self.handle, self._stream()), "dca_stream_end")
        self._stream_keep = None

    PHASES = ("hidden_fwd", "heads_fwd", "loss_fwd_bwd", "heads_bwd", "hidden_bwd", "update")

    def profile(self, on: bool):
        check(self.lib.dca_profile_enable(self.handle, int(on)), "dca_profile_enable")

    def profile_read(self, reset=True):
        """{phase: (total_ms, count)} measured with CUDA events inside the library."""
        ms, cnt = (C.c_double * 6)(), (C.c_int64 * 6)()
        check(self.lib.dca_profile_read(self.handle, C.byref(ms), C.byref(cnt), int(reset)), "dca_profile_read")
        return {p: (ms[i], int(cnt[i])) for i, p in enumerate(self.PHASES)}

    def info(self):
        a = (C.c_int32 * 8)()
        check(self.lib.dca_engine_info(self.handle, C.byref(a)), "dca_engine_info")
        return {"tc_heads": bool(a[0]), "tc_encoder": bool(a[1]), "fused_hidden": bool(a[2]), "head_slots": a[3],
                "sm_count": a[4], "grad_bytes": a[5], "step_graphs": a[6], "graphs_enabled": bool(a[7])}

    @property
    def latent_dim(self):
        return self.hidden[len(self.hidden) // 2] if self.hidden else 0


def launch_count() -> int:
    return int(_lib.load().dca_launch_count())
