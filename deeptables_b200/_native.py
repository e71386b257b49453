"""ctypes binding of the C ABI declared in include/deeptables_b200.h.

The product path has NO CPU fallback: if the shared library is missing this module raises at
import time with the build command, and every op raises ``RuntimeError`` carrying
``dtb_last_error()`` when the library reports a failure.
"""
import ctypes
import os
import re
from ctypes import c_int, c_int64, c_longlong, c_ulonglong, c_float, c_double, c_void_p, c_size_t, c_char_p, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, '_native', 'libdeeptables_b200.so')
HEADER_PATH = os.path.join(os.path.dirname(_HERE), 'include', 'deeptables_b200.h')

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f'{LIB_PATH} is missing: the sm_90a extension is not built. Run '
        f'`python -c "import __graft_entry__ as g; g.build()"` (or `python deeptables_b200/build.py`) '
        f'from the repo root. There is no CPU fallback.')

lib = ctypes.CDLL(LIB_PATH)

P = c_void_p   # every device pointer travels as void*
_IP = POINTER(c_int)


class OptimParams(ctypes.Structure):
    """``dtb_optim_params`` (host memory, read at call time): hyperparameters of SGD / RMSprop / Adagrad."""
    _fields_ = [('kind', c_int), ('flag', c_int), ('lr', c_float), ('momentum', c_float), ('rho', c_double),
                ('eps', c_float)]


OPTIM_SGD, OPTIM_RMSPROP, OPTIM_ADAGRAD = 1, 2, 3
_OPP = POINTER(OptimParams)

METRIC_MAX_LISTS, METRIC_MAX_THRESHOLDS = 8, 2048


class MetricPlan(ctypes.Structure):
    """``dtb_metric_plan`` (host memory, read at call time): what one ``dtb_metrics_update`` accumulates."""
    _fields_ = [('cols', c_int), ('n_lists', c_int), ('list_len', c_int * METRIC_MAX_LISTS),
                ('list_off', c_int * METRIC_MAX_LISTS), ('sums', c_int), ('argmax', c_int), ('top_k', c_int)]


_MPP = POINTER(MetricPlan)


class LossParams(ctypes.Structure):
    """``dtb_loss_params`` (host memory, read at call time): the loss ``dtb_keras_loss_fwd_bwd`` computes."""
    _fields_ = [('loss', c_int), ('delta', c_float), ('label_smoothing', c_float), ('scratch', c_void_p)]


_LPP = POINTER(LossParams)


class GbdtSplitRec(ctypes.Structure):
    """``dtb_gbdt_split_rec``: a leaf's integer sums and its best split (feature -1: none)."""
    _fields_ = [('gain', c_double), ('g', c_int64), ('h', c_int64), ('left_g', c_int64), ('left_h', c_int64),
                ('count', ctypes.c_int32), ('left_count', ctypes.c_int32), ('feature', ctypes.c_int32),
                ('bin', ctypes.c_int32)]


class GbdtSplitParams(ctypes.Structure):
    """``dtb_gbdt_split_params`` (host memory, read at call time)."""
    _fields_ = [('lambda_l2', c_double), ('lambda_l1', c_double), ('min_split_gain', c_double),
                ('min_child_weight', c_double), ('scale_g', c_double), ('scale_h', c_double),
                ('min_child_samples', ctypes.c_int32)]


GBDT_BINARY, GBDT_L2, GBDT_SOFTMAX = 0, 1, 2
GBDT_STAGE_NODES = 2048

_SIGNATURES = {
    'dtb_version': (c_int, []),
    'dtb_last_error': (c_char_p, []),
    'dtb_device_sm_count': (c_int, [_IP]),
    'dtb_capture_status': (c_int, [P]),
    'dtb_launch_count': (c_longlong, []),
    'dtb_launch_count_add': (None, [c_longlong]),
    'dtb_embedding_gather': (c_int, [P, P, P, P, c_int, c_int, c_int, P, P]),
    'dtb_embedding_scatter_add': (c_int, [P, P, P, P, c_int, c_int, c_int, P]),
    'dtb_fm_linear_fwd': (c_int, [P, P, P, P, P, P, P, c_int, c_int, c_int, c_int, P, P]),
    'dtb_fm_linear_bwd': (c_int, [P, P, P, P, P, P, P, P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_linear_dense_grad': (c_int, [P, P, P, c_int, c_int, P]),
    'dtb_concat_emb_dense_fwd': (c_int, [P, P, P, P, P, c_int, c_int, c_int, c_int, P, P]),
    'dtb_concat_emb_dense_bwd': (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_ragged_concat_emb_dense_fwd': (c_int, [P, P, P, _IP, P, P, c_int, c_int, c_int, c_int, P, P]),
    'dtb_ragged_concat_emb_dense_bwd': (c_int, [P, P, _IP, P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_batchnorm_train_fwd': (c_int, [P, P, P, P, P, P, P, P, P, c_int, c_int, c_float, c_float, P]),
    'dtb_batchnorm_infer_fwd': (c_int, [P, P, P, P, P, P, c_int, c_int, c_float, P]),
    'dtb_batchnorm_infer_bwd': (c_int, [P, P, P, P, c_int, c_int, c_float, P]),
    'dtb_batchnorm_bwd': (c_int, [P, P, P, P, P, P, P, P, P, c_int, c_int, c_float, P]),
    'dtb_dense_workspace_bytes': (c_size_t, [c_int, c_int]),
    'dtb_dense_fwd': (c_int, [P, P, P, P, P, c_size_t, c_int, c_int, c_int, c_int, P]),
    'dtb_dense_bwd': (c_int, [P, P, P, P, P, P, P, P, c_size_t, c_int, c_int, c_int, c_int, P]),
    'dtb_dropout': (c_int, [P, P, c_int64, c_float, c_ulonglong, P]),
    'dtb_dropout_dev': (c_int, [P, P, c_int64, c_float, P, P]),
    'dtb_seed_advance': (c_int, [P, c_int, P]),
    'dtb_loss_fwd_bwd': (c_int, [P, P, P, P, P, P, c_int, c_int, c_int, P]),
    'dtb_focal_loss_fwd_bwd': (c_int, [P, P, P, P, P, c_int, c_int, c_int, c_float, c_float, P]),
    'dtb_keras_loss_fwd_bwd': (c_int, [P, P, P, P, P, P, c_int, c_int, c_int, _LPP, P]),
    'dtb_adam_dense': (c_int, [P, P, P, P, c_int64, c_float, c_double, c_double, c_float, c_int, P]),
    'dtb_adam_rows_catchup': (c_int, [P, P, P, P, P, P, P, c_int, c_double, c_double, c_float,
                                      c_int, c_int, c_int, P]),
    'dtb_adam_rows_apply': (c_int, [P, P, P, P, P, P, P, P, c_int, c_double, c_double, c_float,
                                    c_int, c_int, c_int, P]),
    'dtb_adam_dense_dev': (c_int, [P, P, P, P, c_int64, P, P, c_double, c_double, c_float, c_int, P]),
    'dtb_adam_rows_catchup_dev': (c_int, [P, P, P, P, P, P, P, P, c_double, c_double, c_float, c_int, c_int, c_int, P]),
    'dtb_adam_rows_apply_dev': (c_int, [P, P, P, P, P, P, P, P, P, c_double, c_double, c_float, c_int, c_int, c_int, P]),
    'dtb_step_increment': (c_int, [P, P]),
    'dtb_adam_rows_flush': (c_int, [P, P, P, P, P, c_int, c_double, c_double, c_float, c_int64, c_int, P]),
    'dtb_optim_dense': (c_int, [P, P, P, P, P, c_int64, _OPP, c_int, P]),
    'dtb_optim_rows_catchup': (c_int, [P, P, P, P, P, P, P, c_int, _OPP, c_int, c_int, c_int, P]),
    'dtb_optim_rows_apply': (c_int, [P, P, P, P, P, P, P, P, c_int, _OPP, c_int, c_int, c_int, P]),
    'dtb_optim_rows_flush': (c_int, [P, P, P, P, P, c_int, _OPP, c_int64, c_int, P]),
    'dtb_optim_rows_catchup_dev': (c_int, [P, P, P, P, P, P, P, P, _OPP, c_int, c_int, c_int, P]),
    'dtb_optim_rows_apply_dev': (c_int, [P, P, P, P, P, P, P, P, P, _OPP, c_int, c_int, c_int, P]),
    'dtb_optim_rows_flush_dev': (c_int, [P, P, P, P, P, P, _OPP, c_int64, c_int, P]),
    'dtb_reg_grad': (c_int, [P, P, c_int64, c_float, c_float, P, c_double, P]),
    'dtb_adam_dense_reg': (c_int, [P, P, P, P, c_int64, c_float, c_double, c_double, c_float, c_int, c_float, c_float,
                                   P, c_double, P]),
    'dtb_adam_dense_reg_dev': (c_int, [P, P, P, P, c_int64, P, P, c_double, c_double, c_float, c_int, c_float, c_float,
                                       P, c_double, P]),
    'dtb_optim_dense_reg': (c_int, [P, P, P, P, P, c_int64, _OPP, c_int, c_float, c_float, P, c_double, P]),
    'dtb_optim_dense_lr': (c_int, [P, P, P, P, P, c_int64, _OPP, P, c_int, P, c_int, P]),
    'dtb_optim_rows_apply_lr': (c_int, [P, P, P, P, P, P, P, P, P, c_int, P, _OPP, c_int, c_int, c_int, P]),
    'dtb_optim_dense_reg_lr': (c_int, [P, P, P, P, P, c_int64, _OPP, P, c_int, P, c_int, c_float, c_float, P, c_double,
                                       P]),
    'dtb_metrics_state_bytes': (c_size_t, [_MPP]),
    'dtb_metrics_reset': (c_int, [P, _MPP, P]),
    'dtb_metrics_update': (c_int, [P, P, P, P, c_int, _MPP, P]),
    'dtb_perm_keys': (c_int, [P, c_int64, c_ulonglong, c_int, c_int, P]),
    'dtb_shuffle_column': (c_int, [P, P, P, c_int64, c_int, c_int, P]),
    'dtb_importance_scratch_bytes': (c_size_t, [c_int]),
    'dtb_importance_auc': (c_int, [P, P, P, c_int64, P, P, P]),
    'dtb_importance_labels': (c_int, [c_int, P, P, c_int64, c_int, c_int, P, P, P]),
    'dtb_importance_sums': (c_int, [c_int, P, P, P, c_int64, c_int, c_double, P, P, P]),
    'dtb_shap_compose': (c_int, [P, P, P, P, P, c_int, P, P, P, c_int64, c_int, c_int, c_int, P, P, P]),
    'dtb_shap_means': (c_int, [P, c_int64, c_int, c_int, c_int, P, P]),
    'dtb_pdp_block_sums': (c_int, [P, P, c_int64, c_int, c_int, c_int, P, P]),
    'dtb_gradshap_compose': (c_int, [P, P, P, P, P, P, P, c_int, P, P, P, c_int64, c_int, c_int, c_int, P, P, P]),
    'dtb_gradshap_reduce': (c_int, [P, P, P, P, P, P, P, c_int, P, P, c_int64, c_int, c_int, P, P, P, P]),
    'dtb_gradshap_means': (c_int, [P, c_int64, c_int, c_int, P, P]),
    'dtb_gradshap_output_grad': (c_int, [P, c_int64, c_int, c_int, c_int, P, P]),
    'dtb_probe_loss_grad': (c_int, [P, c_int64, P, P, c_int64, c_int, c_int, c_int, c_int, P, P]),
    'dtb_probe_tile_rows': (c_int, [c_int, c_int]),
    'dtb_probe_join': (c_int, [P, c_int64, c_int, P, P]),
    'dtb_probe_predict': (c_int, [P, c_int64, P, c_int64, c_int, c_int, c_int, P, P, P]),
    'dtb_probe_correct': (c_int, [P, P, c_int64, P, P]),
    'dtb_te_remap': (c_int, [P, P, c_int64, c_int, P, P]),
    'dtb_te_keys': (c_int, [P, P, P, c_int64, c_int, c_int, c_int, P, P]),
    'dtb_te_segment_starts': (c_int, [P, c_int64, c_int64, P, P]),
    'dtb_te_segment_stats': (c_int, [P, P, P, P, P, c_int64, c_int, P, P]),
    'dtb_te_segment_join': (c_int, [P, P, c_int64, P, P]),
    'dtb_te_encodings': (c_int, [P, P, P, P, P, P, c_int64, c_int, c_int, c_int, c_double, P, P, P]),
    'dtb_te_gather': (c_int, [P, P, P, P, P, P, c_int64, c_int, c_int, c_int, c_int, P, P]),
    'dtb_gbdt_bin':(c_int, [P, c_int, P, c_int, P, P, P, c_int64, c_int, P, P]),
    'dtb_gbdt_grad': (c_int, [P, P, c_int64, c_int, c_int, c_int, P, P, P, P]),
    'dtb_gbdt_fixed': (c_int, [P, P, c_int64, c_int, c_int, P, P, P]),
    'dtb_gbdt_hist': (c_int, [P, P, c_int64, c_int64, P, P, c_int, c_int, P, P, P, P]),
    'dtb_gbdt_hist_sub': (c_int, [P, P, P, P, P, P, c_int64, c_int, P]),
    'dtb_gbdt_split': (c_int, [P, P, P, P, c_int, P, c_int, c_int, POINTER(GbdtSplitParams), P, P]),
    'dtb_gbdt_partition': (c_int, [P, c_int, P, c_int64, c_int64, c_int, c_int, c_int64, P, P]),
    'dtb_gbdt_update': (c_int, [P, P, P, c_int, c_int64, P, P, c_int, c_int, P, c_int64, P]),
    'dtb_gbdt_leaves': (c_int, [P, c_int, P, c_int, P, P, P, P, P, P, c_int, c_int, c_int64, P, P, c_int, c_int, P]),
    'dtb_discretize': (c_int, [P, c_int, c_int64, P, P, P, c_int, P, c_int, c_int, P]),
    'dtb_dae_swap_batch': (c_int, [P, c_int, P, P, P, P, c_int, c_int, c_int, c_ulonglong, P, P, P]),
    'dtb_grad_rows_pack':(c_int, [P, P, P, P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_grad_rows_unpack': (c_int, [P, P, P, P, c_int, c_int, c_int, P]),
    'dtb_cin_saved_bytes': (c_size_t, [c_int, c_int, c_int, _IP, c_int, c_int]),
    'dtb_cin_workspace_bytes': (c_size_t, [c_int, c_int, c_int, _IP, c_int, c_int, c_int]),
    'dtb_cin_fwd': (c_int, [P, P, P, P, P, P, P, P, c_size_t, c_int, c_int, c_int, _IP, c_int, c_int,
                            c_int, c_int, P, P]),
    'dtb_cin_bwd': (c_int, [P, P, P, P, P, P, P, P, P, P, c_size_t, c_int, c_int, c_int, _IP, c_int,
                            c_int, c_int, c_int, P]),
    'dtb_cin_bwd_phase': (c_int, [P, P, P, P, P, P, P, P, P, P, c_size_t, c_int, c_int, c_int, _IP, c_int,
                                  c_int, c_int, c_int, c_int, P]),
    'dtb_cin_tc_supported': (c_int, [c_int, c_int, _IP, c_int, c_int]),
    'dtb_cin_resolved_precision': (c_int, [c_int, c_int, _IP, c_int, c_int, c_int]),
    'dtb_tc_selftest': (c_int, [P, P, P, P, c_int, c_int, c_int, P]),
    'dtb_cross_fwd': (c_int, [P, P, P, P, P, c_int, c_int, c_int, P]),
    'dtb_cross_bwd_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'dtb_cross_bwd': (c_int, [P, P, P, P, P, P, P, P, P, c_size_t, c_int, c_int, c_int, P]),
    'dtb_pnn_fwd': (c_int, [P, P, P, P, P, P, c_int, c_int, c_int, c_int, P, P]),
    'dtb_pnn_bwd': (c_int, [P, P, P, P, P, P, P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_afm_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'dtb_afm_fwd': (c_int, [P, P, P, P, P, P, P, c_int, c_int, c_int, c_int, c_int, P, P]),
    'dtb_afm_bwd': (c_int, [P, P, P, P, P, P, P, P, P, P, P, P, c_size_t, c_int, c_int, c_int, c_int, c_int, P]),
    'dtb_bilinear_fwd': (c_int, [P, P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_bilinear_bwd': (c_int, [P, P, P, P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_senet_pool_fwd': (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_senet_pool_bwd': (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_senet_scale_fwd': (c_int, [P, P, P, c_int, c_int, c_int, P]),
    'dtb_senet_scale_bwd': (c_int, [P, P, P, P, P, c_int, c_int, c_int, P]),
    'dtb_conv_fields_fwd': (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    'dtb_conv_fields_bwd': (c_int, [P, P, P, P, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    'dtb_maxpool_fields_fwd': (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_maxpool_fields_bwd': (c_int, [P, P, P, c_int, c_int, c_int, c_int, P]),
    'dtb_attention_core_fwd': (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, P]),
    'dtb_attention_core_bwd': (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    'dtb_attention_core_dropout_fwd': (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, c_float, c_ulonglong, P,
                                               c_longlong, P]),
    'dtb_attention_core_dropout_bwd': (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_float,
                                               c_ulonglong, P, c_longlong, P]),
}


def declared_symbols():
    """Every ``dtb_*`` function the public header declares."""
    with open(HEADER_PATH) as f:
        text = f.read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(dtb_[a-z0-9_]+)\s*\(', text)))


for _name, (_res, _args) in _SIGNATURES.items():
    _fn = getattr(lib, _name)      # AttributeError here = header/library mismatch: fail loudly
    _fn.restype = _res
    _fn.argtypes = _args


def last_error():
    msg = lib.dtb_last_error()
    return msg.decode() if msg else ''


_DEBUG_CAPTURE = os.environ.get('DTB_DEBUG_CAPTURE', '') == '1'


def check(rc, what=''):
    if rc != 0:
        raise RuntimeError(f'deeptables_b200 native call {what} failed (code {rc}): {last_error()}')
    if _DEBUG_CAPTURE:          # debug aid: name the first native call after which a stream capture is no longer valid
        st = lib.dtb_capture_status(stream_ptr())
        if st not in (0, 1):
            raise RuntimeError(f'stream capture status {st} right after native call {what!r}')


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return None
    return c_void_p(t.data_ptr())


def int_array(values):
    arr = (c_int * len(values))(*[int(v) for v in values])
    return arr


def stream_ptr():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)
