"""ctypes binding of libopenglue_b200.so (include/openglue_b200.h).

The library is the product: there is NO Python/torch fallback for any kernel.  If the shared
object is missing or a call fails, this module raises - loudly - instead of computing the
result some other way.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libopenglue_b200.so')

OG_OK = 0
OG_PREC_FP32, OG_PREC_TF32X3, OG_PREC_FP16X3 = 0, 1, 2
OG_MAX_HIDDEN = 8
(OG_T_KENC_W, OG_T_KENC_B, OG_T_QKV_W, OG_T_QKV_B, OG_T_FC1_W, OG_T_FC1_B, OG_T_FC2_W, OG_T_FC2_B,
 OG_T_PROJ_W, OG_T_PROJ_B, OG_T_PROJ_RMIX, OG_T_DUSTBIN) = range(12)


class OgConfig(C.Structure):
    _fields_ = [('descriptor_dim', C.c_int32), ('num_heads', C.c_int32), ('num_layers', C.c_int32),
                ('side_info_size', C.c_int32), ('num_hidden', C.c_int32), ('hidden', C.c_int32 * OG_MAX_HIDDEN),
                ('sinkhorn_iters', C.c_int32), ('sinkhorn_reg', C.c_float), ('match_threshold', C.c_float),
                ('precision', C.c_int32), ('no_descriptors', C.c_int32)]


class OgLinearArgs(C.Structure):
    _fields_ = [('A', C.c_void_p), ('lda', C.c_int64), ('strideA', C.c_int64),
                ('A2', C.c_void_p), ('lda2', C.c_int64), ('strideA2', C.c_int64),
                ('k1', C.c_int32), ('k2', C.c_int32),
                ('W', C.c_void_p), ('ldw', C.c_int64), ('strideW', C.c_int64),
                ('bias', C.c_void_p),
                ('rows', C.c_int32), ('nout', C.c_int32), ('batch', C.c_int32),
                ('alpha', C.c_float), ('relu', C.c_int32),
                ('R', C.c_void_p), ('ldr', C.c_int64), ('strideR', C.c_int64),
                ('rscale', C.c_void_p),
                ('Y', C.c_void_p), ('ldy', C.c_int64), ('strideY', C.c_int64),
                ('Yt', C.c_void_p), ('ldyt', C.c_int64), ('strideYt', C.c_int64)]


# every symbol include/openglue_b200.h declares: (restype, argtypes)
_P, _I, _L, _F, _D = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_double
_CFG = C.POINTER(OgConfig)
class OgGtTransform(C.Structure):       # include/openglue_b200.h: og_gt_transform
    _fields_ = [('type', C.c_int32), ('H', C.c_void_p), ('K0', C.c_void_p), ('K1', C.c_void_p), ('R', C.c_void_p),
                ('T', C.c_void_p), ('depth0', C.c_void_p), ('depth1', C.c_void_p), ('depth_is_image', C.c_int32),
                ('depth0_h', C.c_int32), ('depth0_w', C.c_int32), ('depth1_h', C.c_int32), ('depth1_w', C.c_int32)]


OG_GT_PERSPECTIVE, OG_GT_3D_REPROJECTION = 0, 1

SYMBOLS = {
    'og_version': (_I, []),
    'og_last_error': (C.c_char_p, []),
    'og_device_info': (_I, [C.POINTER(C.c_int)] * 3),
    'og_packed_weight_floats': (_L, [_CFG]),
    'og_packed_offset': (_L, [_CFG, _I, _I]),
    'og_workspace_bytes': (_L, [_CFG, _I, _I, _I]),
    'og_split_tf32': (_I, [_P, _P, _P, _L, _P]),
    'og_linear_tc_fwd': (_I, [C.POINTER(OgLinearArgs), _P, _P, _P, _P, _P, _P, _I, _P]),
    'og_superglue_forward': (_I, [_CFG, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, C.POINTER(C.c_float),
                                  _P, _P, _P, _P, _P, _P, _P, _P, _L, _P]),
    'og_superglue_forward_f16': (_I, [_CFG, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, C.POINTER(C.c_float),
                                      _P, _P, _P, _P, _P, _P, _P, _P, _L, _P]),
    'og_workspace_bytes_padded': (_L, [_CFG, _I, _I, _I]),
    'og_superglue_forward_padded': (_I, [_CFG, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P,
                                         _P, _P, _P, _P, _P, _P, _P, _P, _L, _P]),
    'og_f16_meta_floats': (_L, [_CFG]),
    'og_pack_f16': (_I, [_CFG, _P, _P, _P, _P, _P]),
    'og_weight_split_f16': (_I, [_P, _P, _I, _I, _P, _P, _P, _P]),
    'og_amax': (_I, [_P, _L, _P, _P]),
    'og_linear_f16_fwd': (_I, [C.POINTER(OgLinearArgs), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    'og_attention_f16_fwd': (_I, [_P, _L, _L, _P, _P, _P, _L, _P, _P, _P, _L, _P, _P, _L, _L, _P, _I, _I, _I, _I, _I, _I, _P]),
    'og_last_forward_launches': (_I, []),
    'og_set_tuning': (_I, [_I, _I]),
    'og_set_fusion': (_I, [_I]),
    'og_linear_fwd': (_I, [C.POINTER(OgLinearArgs), _I, _P]),
    'og_attention_fwd': (_I, [_P, _L, _L, _P, _L, _L, _P, _L, _L, _P, _L, _L, _I, _I, _I, _I, _I, _I, _P]),
    'og_attention_tc_fwd': (_I, [_P, _L, _L, _P, _P, _L, _P, _P, _L, _P, _L, _L, _I, _I, _I, _I, _I, _P]),
    'og_attention_fwd_padded': (_I, [_P, _L, _L, _P, _L, _L, _P, _L, _L, _P, _L, _L, _I, _I, _I, _I, _I, _P, _P]),
    'og_attention_tc_fwd_padded': (_I, [_P, _L, _L, _P, _P, _L, _P, _P, _L, _P, _L, _L, _I, _I, _I, _I, _I, _P, _P]),
    'og_attention_f16_fwd_padded': (_I, [_P, _L, _L, _P, _P, _P, _L, _P, _P, _P, _L, _P, _P, _L, _L, _P, _I, _I, _I, _I, _I, _P, _P]),
    'og_sinkhorn_workspace_bytes': (_L, [_I, _I, _I]),
    'og_set_sinkhorn_resident': (_I, [_I]),
    'og_sinkhorn_plan': (_I, [_I, _I, _I, _P]),
    'og_sinkhorn_fwd': (_I, [_P, _L, _L, _P, _I, _I, _I, _I, _F, _P, _P, _L, _P]),
    'og_sinkhorn_fwd_padded': (_I, [_P, _L, _L, _P, _I, _I, _I, _P, _I, _F, _P, _P, _L, _P]),
    'og_sinkhorn_consts': (_I, [_I, _I, C.POINTER(C.c_float)]),
    'og_sinkhorn_consts_padded': (_I, [_P, _I, _I, _I, _P, _P]),
    'og_sinkhorn_hist_floats': (_L, [_I, _I, _I, _I]),
    'og_sinkhorn_train_fwd': (_I, [_P, _L, _L, _P, _I, _I, _I, _I, _F, _P, _P, _P, _L, _P]),
    'og_sinkhorn_bwd_workspace_bytes': (_L, [_I, _I, _I, _I]),
    'og_sinkhorn_bwd': (_I, [_P, _L, _L, _P, _I, _I, _I, _I, _F, _P, _P, _P, _P, _P, _L, _P]),
    'og_sinkhorn_train_fwd_padded': (_I, [_P, _L, _L, _P, _I, _I, _I, _P, _I, _F, _P, _P, _P, _L, _P]),
    'og_sinkhorn_bwd_padded': (_I, [_P, _L, _L, _P, _I, _I, _I, _P, _I, _F, _P, _P, _P, _P, _P, _L, _P]),
    'og_match_workspace_bytes': (_L, [_I, _I, _I]),
    'og_match_fwd': (_I, [_P, _I, _I, _I, _F, _P, _P, _P, _P, _P, _L, _P]),
    'og_match_fwd_padded': (_I, [_P, _I, _I, _I, _P, _F, _P, _P, _P, _P, _P, _L, _P]),
    'og_gt_matches_workspace_bytes': (_L, [_I, _I, _I]),
    'og_collate_fwd': (_I, [_P, _P, _P, _P, _P, _I, _P, _I, _I, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'og_criterion_workspace_bytes': (_L, [_I]),
    'og_criterion_fwd': (_I, [_P, _P, _P, _I, _I, _I, _P, _P, _F, _P, _L, _P]),
    'og_criterion_fwd_padded': (_I, [_P, _P, _P, _I, _I, _I, _P, _P, _P, _F, _P, _L, _P]),
    'og_metric_loss_workspace_bytes': (_L, [_I, _I, _I, _I, _I, _I]),
    'og_metric_loss_fwd': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _I, _P, _P, _P, _P, _P, _P, _P, _F, _P, _L, _P]),
    'og_gt_matches_fwd': (_I, [_P, _P, _I, _I, _I, C.POINTER(OgGtTransform), _P, _P, _P, _L, _P]),
    'og_gt_matches_fwd_padded': (_I, [_P, _P, _I, _I, _I, _P, C.POINTER(OgGtTransform), _P, _P, _P, _L, _P]),
    # training-step operators (row f1)
    'og_train_workspace_floats': (_L, [_I]),
    'og_linear_auto_scratch_floats': (_L, [C.POINTER(OgLinearArgs)]),
    'og_linear_auto_fwd': (_I, [C.POINTER(OgLinearArgs), _I, _P, _P]),
    'og_transpose': (_I, [_P, _L, _L, _P, _L, _L, _I, _I, _I, _I, _P]),
    'og_colsum': (_I, [_P, _L, _P, _L, _P, _L, _I, _I, _P, _P, _P]),
    'og_bn_train_fwd': (_I, [_P, _L, _I, _I, _I, _P, _P, _F, _F, _P, _L, _P, _P, _P, _P, _P, _P]),
    'og_bn_train_bwd': (_I, [_P, _L, _P, _L, _I, _I, _I, _P, _P, _P, _P, _L, _P, _P, _P, _P]),
    'og_softmax_rows': (_I, [_P, _L, _L, _I, _P]),
    'og_softmax_bwd_rows': (_I, [_P, _P, _L, _L, _I, _F, _P]),
    'og_axpby': (_I, [_P, _P, _F, _F, _P, _L, _P]),
    'og_sum_batches': (_I, [_P, _I, _I, _I, _P, _L, _I, _P]),
    'og_mix_fwd': (_I, [_P, _P, _P, _P, _L, _I, _P]),
    'og_mix_bwd': (_I, [_P, _P, _P, _P, _L, _I, _P]),
    'og_mix_param_grad': (_I, [_P, _P, _P, _I, _P]),
    'og_kenc_input': (_I, [_P, _P, _I, _I, _F, _F, _P, _P]),
    'og_bn_train_fwd_padded': (_I, [_P, _L, _I, _I, _P, _I, _I, _P, _P, _F, _F, _P, _L, _P, _P, _P, _P, _P, _P]),
    'og_bn_train_bwd_padded': (_I, [_P, _L, _P, _L, _I, _I, _P, _I, _I, _P, _P, _P, _P, _L, _P, _P, _P, _P]),
    'og_softmax_rows_padded': (_I, [_P, _L, _I, _L, _I, _P, _P]),
    'og_softmax_bwd_rows_padded': (_I, [_P, _P, _L, _I, _L, _I, _F, _P, _P]),
    'og_kenc_input_padded': (_I, [_P, _P, _I, _I, _P, _I, _P, _P, _P]),
    'og_mask_padded_rows': (_I, [_P, _I, _I, _I, _P, _P, _P]),
    'og_train_guard': (_I, [_P, _I, _P, _P]),
    'og_bn_train_fwd_guarded': (_I, [_P, _L, _I, _I, _P, _I, _I, _P, _P, _F, _F, _P, _L, _P, _P, _P, _P, _P, _P, _P, _P]),
    'og_train_skip_outputs': (_I, [_P, _P, _I, _P, _L, _P]),
    # SuperPoint front-end operators (row f4)
    'og_sp_im2col3x3': (_I, [_P, _I, _I, _I, _I, _P, _P]),
    'og_sp_maxpool2x2': (_I, [_P, _I, _I, _I, _I, _P, _P]),
    'og_row_normalize': (_I, [_P, _L, _I, _I, _F, _P]),
    'og_sp_heat_nms': (_I, [_P, _I, _I, _I, _I, _F, _I, _P, _P]),
    'og_sp_compact': (_I, [_P, _I, _I, _I, _P, _P, _P, _P]),
    'og_sp_select': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P]),
    'og_sp_sample_desc': (_I, [_P, _I, _I, _I, _I, _P, _P, _I, _I, _I, _P, _P]),
    # OpenCV SIFT front-end (row f7)
    'og_sift_workspace_bytes': (_L, [_I, _I, _I, _I]),
    'og_sift_workspace_layout': (_I, [_I, _I, _I, _I, _P, _I]),
    'og_sift_detect': (_I, [_P, _I, _I, _I, _I, _I, _P, _L, _P, _P, _P, _P]),
    'og_sift_detect_padded': (_I, [_P, _I, _I, _I, _I, _I, _P, _L, _P, _P, _P, _P, _P]),
    'og_sift_select_workspace_bytes': (_L, [_I, _I]),
    'og_sift_select': (_I, [_P, _P, _I, _I, _F, _I, _P, _L, _P, _P, _P]),
    'og_sift_describe': (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P]),
    'og_sift_rootsift_laf': (_I, [_P, _P, _L, _I, _P, _P, _P, _P]),
    'og_sift_fast_atan2': (_I, [_P, _P, _L, _I, _P, _P]),
    'og_sift_gaussian_taps': (_I, [_D, _P, _I]),
    'og_ksift_workspace_bytes': (_L, [_I, _I, _I, _I]),
    'og_ksift_workspace_layout': (_I, [_I, _I, _I, _I, _P, _I]),
    'og_ksift_pyramid': (_I, [_P, _I, _I, _I, _I, _P, _L, _P]),
    'og_ksift_detect': (_I, [_I, _I, _I, _I, _P, _L, _P, _P, _P, _P]),
    'og_ksift_select_workspace_bytes': (_L, [_I, _I]),
    'og_ksift_select': (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _L, _P, _P, _P]),
    'og_ksift_describe': (_I, [_P, _I, _I, _I, _I, _P, _L, _P, _P, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P]),
    # kornia GFTT / AffNet / HardNet front-end
    'og_kgftt_workspace_bytes': (_L, [_I, _I, _I, _I]),
    'og_kgftt_workspace_layout': (_I, [_I, _I, _I, _I, _P, _I]),
    'og_kgftt_pyramid': (_I, [_P, _I, _I, _I, _I, _P, _L, _P]),
    'og_kgftt_detect': (_I, [_I, _I, _I, _I, _P, _L, _P, _P, _P, _P]),
    'og_kgftt_affnet_patches': (_I, [_P, _I, _I, _I, _I, _P, _L, _P, _I, _P, _P, _I, _I, _I, _P, _P]),
    'og_kgftt_frames': (_I, [_P, _I, _I, _I, _I, _P, _L, _P, _P, _I, _P, _P, _I, _I, _I, _P, _I, _P, _P, _P, _P, _P]),
    'og_kgftt_im2col3x3_s2': (_I, [_P, _I, _I, _I, _I, _P, _P]),
    'og_kgftt_desc_finish': (_I, [_P, _I, _I, _P, _P]),
    # DoG (cv2) / AffNet / OriNet / HardNet front-end
    'og_dogaff_workspace_bytes': (_L, [_I, _I, _I]),
    'og_dogaff_workspace_layout': (_I, [_I, _I, _I, _P, _I]),
    'og_dogaff_pyramid': (_I, [_P, _I, _I, _I, _P, _L, _P]),
    'og_dogaff_affnet_patches': (_I, [_P, _I, _I, _I, _P, _L, _P, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P]),
    'og_dogaff_frames': (_I, [_P, _I, _I, _I, _P, _L, _P, _I, _I, _I, _P, _P, _P, _P]),
    'og_dogaff_orinet_head': (_I, [_P, _I, _I, _I, _P, _L, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    # local features -> matcher inputs, matches -> compact list
    'og_prepare_features': (_I, [_P, _P, _L, _I, _I, _P, _P, _P]),
    'og_match_compact': (_I, [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'og_keypoint_counts': (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P]),
    'og_mask_empty_pairs': (_I, [_P, _P, _I, _I, _I, _P, _P, _P, _P, _P]),
    # homography-pretraining pairs
    'og_homography_pairs': (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    # optimiser step: clip_grad_norm_ -> Adam -> StepLR
    'og_optim_state_bytes': (_L, []),
    'og_optim_workspace_bytes': (_L, [_I]),
    'og_clip_adam_step': (_I, [_P, _I, _L, _D, _D, _D, _D, _D, _P, _P, _L, _P]),
    'og_clip_adam_step_guarded': (_I, [_P, _I, _L, _D, _D, _D, _D, _D, _P, _P, _L, _P, _P]),
    'og_adam_schedule': (_I, [_L, _D, _D, _D, _D, _P, _P, _P, _P]),
}

_lib: Optional[C.CDLL] = None


class OpenGlueB200Error(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raise if it is not built."""
    global _lib
    if _lib is None:
        path = os.environ.get('OG_LIB') or LIB_PATH     # OG_LIB: an experimental build of the same sources (A/B timing)
        if not os.path.exists(path):
            raise OpenGlueB200Error(
                f'{path} is missing: build it with `python -m openglue_b200.build` '
                '(there is no fallback implementation)')
        handle = C.CDLL(path)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(handle, name)          # AttributeError if the symbol is not exported
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc: int, what: str) -> None:
    if rc != OG_OK:
        msg = lib().og_last_error()
        raise OpenGlueB200Error(f'{what} failed with status {rc}: {msg.decode() if msg else "?"}')


def check_size(n: int, what: str) -> int:
    """The result of a ``*_workspace_bytes`` / ``*_floats`` query; a negative one (rejected arguments) raises."""
    n = int(n)
    if n < 0:
        check(n, what)
    return n


def ptr(t: Optional[torch.Tensor], off: int = 0) -> Optional[C.c_void_p]:
    """Device pointer to element ``off`` of ``t`` (None for None), as the C ABI takes it."""
    return None if t is None else C.c_void_p(t.data_ptr() + off * t.element_size())


def stream(dev=None) -> C.c_void_p:
    """The current CUDA stream of ``dev`` (default: the current device), as the C ABI takes it."""
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def make_config(config: dict, match_threshold: float = 0.2, precision: int = OG_PREC_FP32) -> OgConfig:
    """Translate the reference's nested config dict (superglue.py:12-27) to og_config."""
    pe, gnn = config['positional_encoding'], config['attention_gnn']
    hidden = list(pe.get('hidden_layers_sizes') or [])
    if len(hidden) > OG_MAX_HIDDEN:
        raise ValueError(f'at most {OG_MAX_HIDDEN} hidden layers in the positional encoder')
    c = OgConfig()
    c.descriptor_dim = int(config['descriptor_dim'])
    c.num_heads = int(gnn['num_heads'])
    c.num_layers = 2 * int(gnn['num_stages'])
    c.side_info_size = int(pe.get('side_info_size', 1))
    c.num_hidden = len(hidden)
    for i, h in enumerate(hidden):
        c.hidden[i] = int(h)
    c.sinkhorn_iters = int(config['otp']['num_iters'])
    c.sinkhorn_reg = float(config['otp']['reg'])
    c.match_threshold = float(match_threshold)
    c.precision = int(precision)
    c.no_descriptors = int(bool(config.get('no_descriptors', False)))
    return c
