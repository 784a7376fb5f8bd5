"""ctypes binding of libdca_b200.so (C ABI in include/dca_b200.h).

There is NO fallback: if the shared library is missing or has no usable CUDA device the
import / first call fails loudly.  PyTorch is used by callers only as the device allocator.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdca_b200.so")

DCA_MAX_HIDDEN = 8
DCA_NAME_LEN = 48

ACTIVATION_IDS = {"relu": 0, "linear": 1, "elu": 2, "selu": 3, "tanh": 4, "sigmoid": 5, "hard_sigmoid": 6,
                  "softplus": 7, "softsign": 8, "exponential": 9, "LeakyReLU": 10, "PReLU": 11}
# keras.optimizers module attributes the reference's `opt.__dict__[optimizer]` resolves (dca/train.py:54-57): class names and
# the lower-case aliases keras/optimizers.py defines; value = (dca_optimizer id, the class's default learning rate)
OPTIMIZERS = {"RMSprop": (0, 1e-3), "SGD": (1, 1e-2), "Adagrad": (2, 1e-2), "Adadelta": (3, 1.0), "Adam": (4, 1e-3),
              "Adamax": (5, 2e-3), "Nadam": (6, 2e-3)}
OPTIMIZERS.update({k.lower(): v for k, v in list(OPTIMIZERS.items())})
AE_TYPE_IDS = {"zinb-conddisp": 0, "zinb": 1, "nb-conddisp": 2, "nb": 3,
               # the remaining registry keys of dca/network.py:763-768: shape-general fp32 path (csrc/extra_types.cu)
               "poisson": 4, "normal": 5, "nb-shared": 6, "zinb-shared": 7, "zinb-elempi": 8, "nb-fork": 9, "zinb-fork": 10}
F32, BF16 = 0, 1
GEMM_AUTO, GEMM_GENERIC, GEMM_TCGEN05 = 0, 1, 2
REGION_PARAMS, REGION_GRADS, REGION_RMS, REGION_BN_STATE, REGION_EPOCH_ACC = 0, 1, 2, 3, 4


INIT_VARIANCE_SCALING, INIT_RANDOM_NORMAL, INIT_RANDOM_UNIFORM, INIT_TRUNCATED_NORMAL = 0, 1, 2, 3
INIT_CONSTANT, INIT_ORTHOGONAL, INIT_IDENTITY = 4, 5, 6
FAN_MODES = {"fan_in": 0, "fan_out": 1, "fan_avg": 2}
DISTRIBUTIONS = {"truncated_normal": 0, "untruncated_normal": 1, "uniform": 2}


def _vs(scale, mode, distribution):
    return dict(kind=INIT_VARIANCE_SCALING, scale=scale, mode=FAN_MODES[mode], distribution=DISTRIBUTIONS[distribution])


# Keras 2 / tf.keras 2.x `kernel_initializer` names (the CLI's --init, dca/network.py:124-126) with their default
# arguments: the snake_case names and the class names
_INITS = {
    "glorot_uniform": _vs(1.0, "fan_avg", "uniform"), "glorot_normal": _vs(1.0, "fan_avg", "truncated_normal"),
    "he_uniform": _vs(2.0, "fan_in", "uniform"), "he_normal": _vs(2.0, "fan_in", "truncated_normal"),
    "lecun_uniform": _vs(1.0, "fan_in", "uniform"), "lecun_normal": _vs(1.0, "fan_in", "truncated_normal"),
    "variance_scaling": _vs(1.0, "fan_in", "truncated_normal"),
    "random_normal": dict(kind=INIT_RANDOM_NORMAL, stddev=0.05),
    "random_uniform": dict(kind=INIT_RANDOM_UNIFORM, minval=-0.05, maxval=0.05),
    "truncated_normal": dict(kind=INIT_TRUNCATED_NORMAL, stddev=0.05),
    "zeros": dict(kind=INIT_CONSTANT, value=0.0), "ones": dict(kind=INIT_CONSTANT, value=1.0),
    "constant": dict(kind=INIT_CONSTANT, value=0.0),
    "orthogonal": dict(kind=INIT_ORTHOGONAL, gain=1.0), "identity": dict(kind=INIT_IDENTITY, gain=1.0),
}
_INIT_ALIASES = {
    "GlorotUniform": "glorot_uniform", "GlorotNormal": "glorot_normal", "HeUniform": "he_uniform", "HeNormal": "he_normal",
    "LecunUniform": "lecun_uniform", "LecunNormal": "lecun_normal", "VarianceScaling": "variance_scaling",
    "normal": "random_normal", "RandomNormal": "random_normal", "uniform": "random_uniform",
    "RandomUniform": "random_uniform", "TruncatedNormal": "truncated_normal", "zero": "zeros", "Zeros": "zeros",
    "one": "ones", "Ones": "ones", "Constant": "constant", "Orthogonal": "orthogonal", "Identity": "identity",
}
INITIALIZERS = dict(_INITS, **{k: _INITS[v] for k, v in _INIT_ALIASES.items()})


class DcaError(RuntimeError):
    pass


class Config(C.Structure):
    _fields_ = [
        ("struct_bytes", C.c_int32), ("n_in", C.c_int32), ("n_out", C.c_int32),
        ("n_hidden", C.c_int32), ("hidden", C.c_int32 * DCA_MAX_HIDDEN),
        ("ae_type", C.c_int32), ("batchnorm", C.c_int32), ("max_batch", C.c_int32),
        ("x_dtype", C.c_int32), ("gemm_path", C.c_int32),
        ("ridge", C.c_float), ("l1", C.c_float), ("l2", C.c_float),
        ("l1_enc", C.c_float), ("l2_enc", C.c_float),
        ("bn_momentum", C.c_float), ("bn_eps", C.c_float),
        ("rms_rho", C.c_float), ("rms_eps", C.c_float),
        ("elempi_shared", C.c_int32), ("sync_bn", C.c_int32),
        ("activation", C.c_int32), ("input_dropout", C.c_float),
        ("hidden_dropout", C.c_float * DCA_MAX_HIDDEN), ("dropout_seed", C.c_uint64),
    ]


class TensorInfo(C.Structure):
    _fields_ = [("name", C.c_char * DCA_NAME_LEN), ("offset", C.c_int64),
                ("rows", C.c_int32), ("cols", C.c_int32)]


class PackedCountsDesc(C.Structure):
    """dca_packed_counts: device pointers of one packed count matrix (include/dca_b200.h)."""
    _fields_ = [
        ("struct_bytes", C.c_int32), ("bits", C.c_int32), ("n_rows", C.c_int64), ("genes", C.c_int32),
        ("max_row_nibble_bytes", C.c_int32), ("packed", C.c_void_p), ("ovf_indptr", C.c_void_p),
        ("ovf_entries", C.c_void_p), ("nib_indptr", C.c_void_p), ("nibbles", C.c_void_p), ("n_counts", C.c_void_p),
    ]


class Initializer(C.Structure):
    """dca_initializer: a kernel initializer (include/dca_b200.h)."""
    _fields_ = [("struct_bytes", C.c_int32), ("kind", C.c_int32), ("scale", C.c_float), ("mode", C.c_int32),
                ("distribution", C.c_int32), ("stddev", C.c_float), ("minval", C.c_float), ("maxval", C.c_float),
                ("value", C.c_float), ("gain", C.c_float)]


def initializer(name: str) -> Initializer:
    """The dca_initializer of a Keras initializer name; ValueError for a name Keras would not resolve here."""
    if not isinstance(name, str) or name not in INITIALIZERS:
        raise ValueError("unknown initializer %r (accepted: %s)" % (name, ", ".join(sorted(INITIALIZERS))))
    return Initializer(struct_bytes=C.sizeof(Initializer), **INITIALIZERS[name])


class DebugReport(C.Structure):
    """dca_debug_report: the debug checks' report of the last step (include/dca_b200.h)."""
    _fields_ = [("struct_bytes", C.c_int32), ("reserved", C.c_int32), ("count", C.c_int64 * 3),
                ("first_row", C.c_int32 * 3), ("first_gene", C.c_int32 * 3)]


# name -> (restype, argtypes); every symbol declared in include/dca_b200.h
_vp, _i32, _i64, _f, _sz = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_size_t
PROTOTYPES = {
    "dca_version": (C.c_int, []),
    "dca_last_error": (C.c_char_p, []),
    "dca_config_default": (None, [C.POINTER(Config)]),
    "dca_arena_bytes": (C.c_int, [C.POINTER(Config), C.POINTER(_sz)]),
    "dca_create": (C.c_int, [C.POINTER(Config), _vp, _sz, C.POINTER(_vp)]),
    "dca_destroy": (C.c_int, [_vp]),
    "dca_param_count": (C.c_int, [_vp, C.POINTER(_i64), C.POINTER(_i32)]),
    "dca_param_info": (C.c_int, [_vp, _i32, C.POINTER(TensorInfo)]),
    "dca_state_count": (C.c_int, [_vp, C.POINTER(_i64), C.POINTER(_i32)]),
    "dca_state_info": (C.c_int, [_vp, _i32, C.POINTER(TensorInfo)]),
    "dca_region": (C.c_int, [_vp, _i32, C.POINTER(_vp), C.POINTER(_i64)]),
    "dca_init_params": (C.c_int, [_vp, C.c_uint64, _vp]),
    "dca_init_params_ex": (C.c_int, [_vp, C.c_uint64, C.POINTER(Initializer), _vp]),
    "dca_init_fill_host": (C.c_int, [C.POINTER(Initializer), C.c_uint64, C.c_uint64, _i32, _i32, _i32, _vp]),
    "dca_params_changed": (C.c_int, [_vp, _vp]),
    "dca_train_step": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp, _i32, _vp]),
    "dca_train_step_phase": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp, _i32, _i32, _vp]),
    "dca_grad_buckets": (C.c_int, [_vp, C.POINTER(_i64)]),
    "dca_comm_unique_id": (C.c_int, [_vp]),
    "dca_comm_init": (C.c_int, [_vp, _vp, _i32, _i32]),
    "dca_comm_destroy": (C.c_int, [_vp]),
    "dca_allreduce": (C.c_int, [_vp, _vp]),
    "dca_train_step_dp": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp, _i32, _vp]),
    "dca_set_optimizer": (C.c_int, [_vp, _i32, _vp]),
    "dca_reset_optimizer": (C.c_int, [_vp, _vp]),
    "dca_apply_update": (C.c_int, [_vp, _f, _f, _f, _vp]),
    "dca_eval_step": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp, _i32, _vp]),
    "dca_predict": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp, _vp]),
    "dca_read_loss": (C.c_int, [_vp, C.POINTER(_f), C.POINTER(_i32), _vp]),
    "dca_read_epoch_acc": (C.c_int, [_vp, C.POINTER(C.c_double * 4), _i32, _vp]),
    "dca_set_debug_checks": (C.c_int, [_vp, _i32]),
    "dca_read_debug_report": (C.c_int, [_vp, C.POINTER(DebugReport), _vp]),
    "dca_debug_check": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _i64, _vp, _i64, _i32, _i32, _vp, C.POINTER(DebugReport), _vp]),
    "dca_train_step_host": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _f, _f, C.POINTER(_f), _vp]),
    "dca_set_input_transform": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _vp]),
    "dca_set_loss_ring": (C.c_int, [_vp, _vp, _i32]),
    "dca_stream_begin": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _i32, _vp]),
    "dca_stream_begin_packed": (C.c_int, [_vp, _vp, _i32, _i64, _vp, _vp, _vp, _i64, _i32, _vp]),
    "dca_stream_begin_sparse": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp]),
    "dca_stream_step": (C.c_int, [_vp, _i64, _i64, _vp]),
    "dca_stream_end": (C.c_int, [_vp, _vp]),
    "dca_expand_packed_counts": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _vp,
                                           _vp]),
    "dca_expand_sparse_counts": (C.c_int, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _i32, _vp, _vp,
                                           _i32, _vp, _vp]),
    "dca_zinb_loss_fwd_bwd": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _f, _f,
                                        _vp, _vp, _vp, _i32, _vp, _vp, _vp, _sz, _vp]),
    "dca_zinb_loss_workspace_bytes": (C.c_int, [_i32, _i32, C.POINTER(_sz)]),
    "dca_zinb_loss_fwd": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _f,
                                    _vp, _vp, _sz, _vp]),
    "dca_zinb_elem_host": (C.c_int, [_i32, _f, _f, _f, _f, _f, _f, C.POINTER(_f * 4)]),
    "dca_dropout_mask_host": (C.c_int, [C.c_uint64, C.c_uint64, _i32, _i64, _f, _vp]),
    "dca_activation_host": (C.c_int, [_i32, _f, _f, C.POINTER(_f * 2)]),
    "dca_activation_bwd_host": (C.c_int, [_i32, _f, _f, _f, _i32, _f, C.POINTER(_f * 2)]),
    "dca_dense_heads_fwd": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                      _vp, _vp, _vp, _i64, _vp]),
    "dca_tc_heads_fwd": (C.c_int, [_vp, _i32, _vp, _vp, _i32, _i32, C.POINTER(_i32 * 3), _vp, _vp, _vp, _vp, _i64, _vp]),
    "dca_tc_heads_loss": (C.c_int, [_vp, _i32, _vp, _vp, _i32, _vp, _i64, _vp, _vp, _f, _f, _vp, _vp, _vp, _i64, _vp,
                                    _vp, _sz, _vp]),
    "dca_tc_gene_gemm": (C.c_int, [_i32, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32,
                                   _vp, _vp, _vp, _vp]),
    "dca_tc_gene_gemm_sms": (C.c_int, [_i32, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i64,
                                       _i32, _vp, _vp, _vp, _vp, _i32]),
    "dca_tc_gene_gemm_rows": (C.c_int, [_i32, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                        _i64, _i32, _vp, _vp, _vp, _vp, _i32]),
    "dca_head_bwd_schedule": (C.c_int, [_i32, _i32, _i32, _i32, _i32, _vp, _i64, C.POINTER(_i64), _vp]),
    "dca_enc_bwd_schedule": (C.c_int, [_i32, _i32, _vp, _i64, _vp]),
    "dca_tc_probe": (C.c_int, [_vp, _i32, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32,
                               _vp, _vp]),
    "dca_profile_enable": (C.c_int, [_vp, _i32]),
    "dca_profile_read": (C.c_int, [_vp, C.POINTER(C.c_double * 6), C.POINTER(C.c_int64 * 6), _i32]),
    "dca_engine_info": (C.c_int, [_vp, C.POINTER(_i32 * 8)]),
    "dca_write_text_matrix": (C.c_int, [C.c_char_p, _vp, _i32, _i64, _i64, _i64, _vp, _vp, _i32, _i32]),
    "dca_write_text_device": (C.c_int, [C.c_char_p, _i32, _vp, _i64, _i64, _i64, _i32, _vp, _i64, _vp, _vp, _i64, _i32, _vp,
                                        _vp]),
    "dca_write_text_device_gz": (C.c_int, [C.c_char_p, _i32, _vp, _i64, _i64, _i64, _i32, _vp, _i64, _vp, _vp, _i64, _i32,
                                           _vp, _vp]),
    "dca_format_fixed6_host": (C.c_int, [_vp, _i64, _vp, _vp]),
    "dca_read_text_counts": (C.c_int, [C.c_char_p, _i32, _i32, _i64, _i32, _vp, _vp, _i64, _vp, _vp, _i64, _vp]),
    "dca_read_mtx_counts": (C.c_int, [C.c_char_p, _i32, _i64, _i32, _vp, _vp, _vp, _vp, _vp]),
    "dca_read_text_counts_gz": (C.c_int, [C.c_char_p, _i32, _i32, _i64, _i32, _vp, _vp, _i64, _vp, _vp, _i64, _vp]),
    "dca_read_mtx_counts_gz": (C.c_int, [C.c_char_p, _i32, _i64, _i32, _vp, _vp, _vp, _vp, _vp]),
    "dca_read_mtx_counts_map": (C.c_int, [C.c_char_p, _i32, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i64]),
    "dca_read_mtx_counts_gz_map": (C.c_int, [C.c_char_p, _i32, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i64]),
    "dca_gunzip": (C.c_int, [C.c_char_p, _i32, _vp, _vp, _i64, _vp]),
    "dca_inflate_span_host": (C.c_int, [_vp, _i64, _i32, _i64, _i64, _vp, _i64, _vp]),
    "dca_inflate_find_host": (C.c_int, [_vp, _i64, _i64, _i64, _vp]),
    "dca_gzip_device": (C.c_int, [_vp, _i64, _vp, _i64, _i32, _vp, _vp]),
    "dca_gzip_host": (C.c_int, [_vp, _i64, _vp, _i64, C.POINTER(_i64)]),
    "dca_count_escapes": (C.c_int, [_vp, _i32, _i64, _i64, _i64, _vp, _i32]),
    "dca_pack_counts": (C.c_int, [_vp, _i32, _i64, _i64, _i64, _i32, _vp, _vp, _vp, _i32]),
    "dca_sparse_counts": (C.c_int, [_vp, _i32, _i64, _i64, _i64, _vp, _vp, _i32]),
    "dca_pack_sparse": (C.c_int, [_vp, _i32, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i32]),
    "dca_preprocess_workspace_bytes": (C.c_int, [_i64, _i32, C.POINTER(_sz)]),
    "dca_counts_csr_to_dense": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _vp, _i64, _vp]),
    "dca_count_totals": (C.c_int, [_vp, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "dca_gather_counts": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i32, _vp, _i64, _vp]),
    "dca_log_moments": (C.c_int, [_vp, _i64, _i64, _i32, _vp, C.c_double, _i32, _vp, _vp, _vp, _sz, _vp]),
    "dca_normalize_write": (C.c_int, [_vp, _i64, _i64, _i32, _vp, C.c_double, _i32, _vp, _vp, _vp, _i32, _i64, _vp]),
    "dca_stats_workspace_bytes": (C.c_int, [_i64, _i32, _i64, C.POINTER(_sz)]),
    "dca_stats_begin": (C.c_int, [_i64, _i32, _vp, _sz, _vp]),
    "dca_count_totals_rows": (C.c_int, [_vp, _i64, _i64, _i64, _i64, _i32, _vp, _vp, _sz, _vp]),
    "dca_count_totals_finish": (C.c_int, [_i64, _i32, _vp, _vp, _vp, _sz, _vp]),
    "dca_log_moments_rows": (C.c_int, [_i32, _vp, _i64, _i64, _i64, _i64, _i32, _vp, C.c_double, _i32, _vp, _vp, _sz,
                                       _vp]),
    "dca_log_moments_finish": (C.c_int, [_i32, _i64, _i32, _i32, _vp, _vp, _sz, _vp]),
    "dca_set_input_transform_exact": (C.c_int, [_vp, _vp, _vp, C.c_double, _i32, _vp]),
    "dca_stream_row_totals": (C.c_int, [_vp, _vp]),
    "dca_stream_predict": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _i64, _vp, _vp]),
    "dca_stream_eval": (C.c_int, [_vp, _i64, _i64, _vp]),
    "dca_stream_capacity": (C.c_int, [_vp, C.POINTER(_i64), C.POINTER(_i64)]),
    "dca_expand_packed_counts_exact": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _i32, _i32, C.c_double, _i32, _vp, _vp, _vp,
                                                 _vp, _i32, _vp, _vp]),
    "dca_expand_sparse_counts_exact": (C.c_int, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i32, _i32, C.c_double, _i32, _vp,
                                                 _vp, _vp, _vp, _i32, _vp, _vp]),
    "dca_pack_count_rows": (C.c_int, [_vp, _i64, _i64, _i32, _vp, _i64, _vp]),
    "dca_pack_rows_device": (C.c_int, [_vp, _i64, _i64, _i64, C.POINTER(PackedCountsDesc), _vp]),
    "dca_expand_rows_exact": (C.c_int, [C.POINTER(PackedCountsDesc), _vp, _i32, C.c_double, _i32, _vp, _vp, _vp, _vp, _i32,
                                        _vp, _vp]),
    "dca_packed_train_step": (C.c_int, [_vp, C.POINTER(PackedCountsDesc), _vp, _i32, _vp]),
    "dca_packed_eval_step": (C.c_int, [_vp, C.POINTER(PackedCountsDesc), _vp, _i32, _vp]),
    "dca_packed_predict": (C.c_int, [_vp, C.POINTER(PackedCountsDesc), _vp, _i32, _vp, _vp, _vp, _i64, _vp, _vp]),
    "dca_launch_count": (C.c_int64, []),
    "dca_set_tunable": (C.c_int, [C.c_char_p, C.c_int64]),
}

_lib = None


def load():
    """Load the shared library (once).  Raises ImportError with build instructions if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "dca_b200: %s not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C dca_b200/csrc`). There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)      # AttributeError if the library does not export it
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int, what: str = ""):
    if status != 0:
        msg = load().dca_last_error().decode("utf-8", "replace")
        if status == -1:
            raise ValueError("%s: %s" % (what or "dca_b200", msg))
        raise DcaError("%s failed (status %d): %s" % (what or "dca_b200", status, msg))


def set_tunable(name: str, value: int):
    """Process-wide launch tunables / switches (dca_set_tunable in include/dca_b200.h)."""
    check(load().dca_set_tunable(name.encode(), int(value)), "dca_set_tunable")


def default_config() -> Config:
    cfg = Config()
    load().dca_config_default(C.byref(cfg))
    return cfg
