"""ctypes binding of the C-ABI in include/lfmq.h (lfm_quant_b200/_lfmq.so).

There is no CPU fallback: if the shared library is missing or a call fails, this module raises.
"""
from __future__ import annotations

import ctypes as C
import os

# LFMQ_LIB_PATH: an alternative build of the same ABI (A/B measurements of kernel variants, tools/)
_LIB_PATH = os.environ.get('LFMQ_LIB_PATH') or os.path.join(os.path.dirname(os.path.abspath(__file__)), '_lfmq.so')

OPTIMIZERS = {'Adadelta': 0, 'Adam': 1, 'RMSprop': 2, 'SGD': 3}
PREC_FP32, PREC_BF16, PREC_BF16X3, PREC_TF32 = 0, 1, 2, 3
# LFMQ_TAIL_*: the slots of the gradient vector's tail, grads[n_trainable + TAIL_*], and its length
TAIL_LOSS, TAIL_MSE0, TAIL_GRAD_NORM, TAIL_CLIP_SCALE, TAIL_UQ_LOSS_LAST_TAR, TAIL_LEN = 0, 1, 2, 3, 4, 8
CELLS = {'lstm': 0, 'gru': 1}           # LFMQ_CELL_*
ABI_VERSION = 4                         # LFMQ_ABI_VERSION in include/lfmq.h (4: lfmq_chain_*, forecast_steps > 1)


class LfmqConfig(C.Structure):
    _fields_ = [('struct_size', C.c_int32), ('max_batch', C.c_int32), ('seq_len', C.c_int32),
                ('n_inputs', C.c_int32), ('n_outputs', C.c_int32), ('num_hidden', C.c_int32),
                ('num_layers', C.c_int32), ('target_idx', C.c_int32), ('train', C.c_int32),
                ('precision', C.c_int32), ('optimizer', C.c_int32), ('forward_only', C.c_int32),
                ('rnn_cell', C.c_int32), ('uq', C.c_int32),
                ('dropout', C.c_float), ('recurrent_dropout', C.c_float), ('target_lambda', C.c_float),
                ('rnn_lambda', C.c_float), ('max_grad_norm', C.c_float), ('max_norm', C.c_float),
                ('sgd_momentum', C.c_float), ('bn_epsilon', C.c_float), ('seed', C.c_uint64)]


class LfmqDenseConfig(C.Structure):
    _fields_ = [('struct_size', C.c_int32), ('max_batch', C.c_int32), ('seq_len', C.c_int32), ('n_inputs', C.c_int32),
                ('n_outputs', C.c_int32), ('target_idx', C.c_int32), ('precision', C.c_int32), ('optimizer', C.c_int32),
                ('forward_only', C.c_int32), ('huber_loss', C.c_int32), ('target_lambda', C.c_float),
                ('huber_delta', C.c_float), ('max_grad_norm', C.c_float), ('sgd_momentum', C.c_float)]


class LfmqGatherArgs(C.Structure):
    _fields_ = [('struct_size', C.c_int32), ('n_rows', C.c_int32), ('n_cols', C.c_int32), ('B', C.c_int32),
                ('T', C.c_int32), ('F', C.c_int32), ('O', C.c_int32), ('stride', C.c_int32),
                ('seq_norm_col', C.c_int32), ('log_squasher', C.c_int32), ('aux_masking', C.c_int32),
                ('table', C.c_void_p), ('inp_idx', C.c_void_p), ('tar_idx', C.c_void_p),
                ('inp_cols', C.c_void_p), ('fin_cols', C.c_void_p), ('center', C.c_void_p),
                ('scale', C.c_void_p), ('scale_flag', C.c_void_p), ('aux_flag', C.c_void_p),
                ('x', C.c_void_p), ('y', C.c_void_p), ('seq_norm', C.c_void_p)]


class LfmqWindowIndexArgs(C.Structure):
    _fields_ = [('struct_size', C.c_int32), ('n', C.c_int32), ('train', C.c_int32), ('stride', C.c_int32),
                ('forecast_n', C.c_int32), ('min_unrollings', C.c_int32), ('max_unrollings', C.c_int32),
                ('start_date', C.c_int32), ('end_date', C.c_int32), ('last_train_date', C.c_int32), ('cap', C.c_int32),
                ('key', C.c_void_p), ('active', C.c_void_p), ('date', C.c_void_p), ('inp_idx', C.c_void_p),
                ('tar_idx', C.c_void_p), ('rows', C.c_void_p), ('count', C.c_void_p), ('work', C.c_void_p)]


# every symbol include/lfmq.h declares: name -> (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    'lfmq_last_error': (C.c_char_p, []),
    'lfmq_abi_version': (C.c_int32, []),
    'lfmq_workspace_bytes': (C.c_int32, [C.POINTER(LfmqConfig), C.POINTER(C.c_uint64)]),
    'lfmq_create': (C.c_int32, [C.POINTER(LfmqConfig), _P, C.c_uint64, C.POINTER(_P)]),
    'lfmq_destroy': (C.c_int32, [_P]),
    'lfmq_dense_workspace_bytes': (C.c_int32, [C.POINTER(LfmqDenseConfig), C.POINTER(C.c_uint64)]),
    'lfmq_dense_create': (C.c_int32, [C.POINTER(LfmqDenseConfig), _P, C.c_uint64, C.POINTER(_P)]),
    'lfmq_set_device_share': (C.c_int32, [_P, C.c_int32, C.c_int32]),
    'lfmq_persistent_cta_budget': (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int64)]),
    'lfmq_param_count': (C.c_int32, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    'lfmq_param_spec': (C.c_int32, [_P, C.c_int32, C.c_char_p, C.c_int32, C.POINTER(C.c_int32),
                                     C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    'lfmq_params_ptr': (C.c_int32, [_P, C.POINTER(_P)]),
    'lfmq_grads_ptr': (C.c_int32, [_P, C.POINTER(_P)]),
    'lfmq_opt_state_ptr': (C.c_int32, [_P, C.POINTER(_P), C.POINTER(C.c_int64)]),
    'lfmq_set_params': (C.c_int32, [_P, _P, C.c_int64, _P]),
    'lfmq_get_params': (C.c_int32, [_P, _P, C.c_int64, _P]),
    'lfmq_forward': (C.c_int32, [_P, _P, C.c_int32, C.c_int64, C.c_int64, _P, _P]),
    'lfmq_forward_uq': (C.c_int32, [_P, _P, C.c_int32, C.c_int64, C.c_int64, _P, _P, _P]),
    'lfmq_loss': (C.c_int32, [_P, _P, _P, C.c_int32, _P, _P]),
    'lfmq_loss_uq': (C.c_int32, [_P, _P, _P, _P, C.c_int32, _P, _P]),
    'lfmq_mask_count': (C.c_int32, [_P, _P, C.c_int32, _P, _P]),
    'lfmq_backward': (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int64, C.c_int64, _P, _P]),
    'lfmq_apply': (C.c_int32, [_P, C.c_float, C.c_int64, _P]),
    'lfmq_train_step': (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int64, C.c_int64, C.c_float, _P, _P]),
    'lfmq_chain_forward': (C.c_int32, [_P, C.c_int32, _P, C.c_int32, C.c_int64, C.c_int64, _P, _P, _P]),
    'lfmq_chain_forward_uq': (C.c_int32, [_P, C.c_int32, _P, C.c_int32, C.c_int64, C.c_int64, _P, _P, _P, _P]),
    'lfmq_forward_uq_mc_work_bytes': (C.c_int32, [_P, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    'lfmq_forward_uq_mc': (C.c_int32, [_P, _P, C.c_int32, C.c_int64, C.c_int64, C.c_int32, _P, _P, _P, _P, _P,
                                        C.c_uint64, _P]),
    'lfmq_chain_forward_uq_mc_work_bytes': (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    'lfmq_chain_forward_uq_mc': (C.c_int32, [_P, C.c_int32, _P, C.c_int32, C.c_int64, C.c_int64, C.c_int32, _P, _P, _P,
                                              _P, _P, C.c_uint64, _P]),
    'lfmq_chain_forward_uq_dist_work_bytes': (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                          C.POINTER(C.c_uint64)]),
    'lfmq_chain_forward_uq_dist': (C.c_int32, [_P, C.c_int32, _P, _P, C.c_int32, C.c_int64, C.c_int64, C.c_int32, _P,
                                                C.c_int32, _P, _P, _P, _P, _P, _P, _P, C.c_uint64, _P]),
    'lfmq_integrated_gradients_work_bytes': (C.c_int32, [_P, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    'lfmq_integrated_gradients': (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P, _P, _P, _P, C.c_uint64, _P]),
    'lfmq_chain_permutation_importance_work_bytes': (C.c_int32, [_P, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    'lfmq_chain_permutation_importance': (C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_int32, _P, C.c_int32, C.c_int32,
                                                       C.c_uint64, C.c_int64, _P, _P, C.c_uint64, _P]),
    'lfmq_permutation_index': (C.c_int32, [C.c_int32, C.c_uint64, C.c_int32, C.c_int32, C.c_int32,
                                           C.POINTER(C.c_int32)]),
    'lfmq_chain_shapley_work_bytes': (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                  C.POINTER(C.c_uint64)]),
    'lfmq_chain_shapley': (C.c_int32, [_P, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_uint64, C.c_int64,
                                        _P, _P, _P, _P, C.c_uint64, _P]),
    'lfmq_chain_ale_work_bytes': (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    'lfmq_chain_ale': (C.c_int32, [_P, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int64, _P, _P, _P, _P,
                                    _P, _P, _P, C.c_uint64, _P]),
    'lfmq_influence_features_work_bytes': (C.c_int32, [_P, C.POINTER(C.c_uint64)]),
    'lfmq_influence_train_features': (C.c_int32, [_P, _P, _P, C.c_int32, _P, _P, C.c_uint64, _P]),
    'lfmq_influence_query_features': (C.c_int32, [_P, _P, C.c_int32, _P, _P, _P, C.c_uint64, _P]),
    'lfmq_influence_topk_work_bytes': (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                   C.POINTER(C.c_uint64)]),
    'lfmq_influence_topk': (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P,
                                         _P, _P, _P, C.c_uint64, _P]),
    'lfmq_nearest_topk_work_bytes': (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    'lfmq_nearest_topk': (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P,
                                       C.c_uint64, _P]),
    'lfmq_conformal_scores_work_bytes': (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    'lfmq_conformal_scores': (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int32, _P, _P, C.c_uint64, _P]),
    'lfmq_conformal_calibrate_work_bytes': (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    'lfmq_conformal_calibrate': (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, _P, _P,
                                              C.c_uint64, _P]),
    'lfmq_conformal_apply_work_bytes': (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                    C.POINTER(C.c_uint64)]),
    'lfmq_conformal_apply': (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int32, _P, _P, _P, C.c_int32, C.c_int32, _P, _P,
                                          _P, _P, C.c_uint64, _P]),
    'lfmq_factor_eval_work_bytes': (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                C.POINTER(C.c_uint64)]),
    'lfmq_factor_eval': (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_int32, _P, _P, _P,
                                      _P, _P, _P, _P, _P, C.c_uint64, _P]),
    'lfmq_chain_loss':(C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_int32, _P, _P]),
    'lfmq_chain_loss_uq': (C.c_int32, [_P, C.c_int32, _P, _P, _P, _P, C.c_int32, _P, _P]),
    'lfmq_chain_backward': (C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_int32, C.c_int64, C.c_int64, _P, _P, _P]),
    'lfmq_chain_apply': (C.c_int32, [_P, C.c_int32, C.c_float, C.c_int64, _P]),
    'lfmq_mask_count_uq': (C.c_int32, [_P, _P, C.c_int32, _P, _P]),
    'lfmq_set_row_weights': (C.c_int32, [_P, _P]),
    'lfmq_row_weights': (C.c_int32, [_P, C.c_int64, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                     C.c_int32, _P, _P]),
    'lfmq_chain_mask_count': (C.c_int32, [_P, C.c_int32, _P, C.c_int32, _P, _P]),
    'lfmq_chain_backward_dp': (C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_int32, C.c_int64, C.c_int64, _P, _P, _P,
                                           _P]),
    'lfmq_chain_grad_pack_size': (C.c_int32, [_P, C.c_int32, C.POINTER(C.c_int64)]),
    'lfmq_chain_grad_pack': (C.c_int32, [_P, C.c_int32, _P, _P]),
    'lfmq_chain_grad_unpack': (C.c_int32, [_P, C.c_int32, _P, _P, _P, _P]),
    'lfmq_window_index': (C.c_int32, [C.POINTER(LfmqWindowIndexArgs), _P]),
    'lfmq_gather_batch': (C.c_int32, [C.POINTER(LfmqGatherArgs), _P]),
    'lfmq_unscale': (C.c_int32, [_P, _P, C.c_int64, C.c_int32, _P, _P, C.c_int32, _P]),
    'lfmq_launch_count': (C.c_int64, []),
    'lfmq_profile_enable': (C.c_int32, [_P, C.c_int32]),
    'lfmq_profile_read': (C.c_int32, [_P, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int32)]),
}

_lib = None


class LfmqError(RuntimeError):
    pass


def lib_path():
    return _LIB_PATH


def load():
    """Loads _lfmq.so (once) and types every entry point.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(_LIB_PATH):
        raise LfmqError('%s not found: build it with `make` or `python -c "import __graft_entry__ as g; g.build()"` '
                        '(there is no CPU fallback)' % _LIB_PATH)
    lib = C.CDLL(_LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if lib.lfmq_abi_version() != ABI_VERSION:
        raise LfmqError('ABI version mismatch: %d' % lib.lfmq_abi_version())
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise LfmqError('lfmq error %d: %s' % (rc, load().lfmq_last_error().decode('utf-8', 'replace')))
