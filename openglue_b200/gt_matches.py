"""Ground-truth match generation on the GPU: drop-in for ``models.gt_matches_generation.generate_gt_matches``
(reference models/gt_matches_generation.py:17-93), the step that runs right before the matching core in the
reference's ``training_step`` / ``validation_step`` (models/matching_module.py:84-93).

Same signature, same return value ``(data, y_true)``, same constants.  ``positive_threshold`` / ``negative_threshold``
are accepted and - exactly as in the reference, whose refinements write through boolean-mask copies - change nothing.
All arithmetic runs in ``libopenglue_b200.so`` (``og_gt_matches_fwd``); there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Dict, Optional, Tuple

import torch

from . import _cabi
from .superglue import is_padded, padded_lengths

UNMATCHED_INDEX = -1      # reference models/gt_matches_generation.py:13
IGNORE_INDEX = -2         # reference models/gt_matches_generation.py:14

__all__ = ['generate_gt_matches', 'gt_matches', 'UNMATCHED_INDEX', 'IGNORE_INDEX']


def _f32(t: torch.Tensor, dev: torch.device) -> torch.Tensor:
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


def gt_matches(kpts0: torch.Tensor, kpts1: torch.Tensor, transformation: Dict[str, Any],
               lengths: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """-> (gt_matches0 [B, N] int64, gt_matches1 [B, M] int64) on the keypoints' (CUDA) device.  ``lengths`` (padded batch,
    int32 [2B] on the device: n_0 .. n_{B-1}, m_0 .. m_{B-1}): pair b's labels come from its first n_b / m_b keypoints alone and
    are ``IGNORE_INDEX`` past them."""
    dev = kpts0.device
    if dev.type != 'cuda':
        raise RuntimeError('openglue_b200.gt_matches needs CUDA tensors (sm_90a); there is no CPU path')
    if kpts0.dim() != 3 or kpts1.dim() != 3 or kpts0.shape[-1] != 2 or kpts1.shape[-1] != 2 or kpts0.shape[0] != kpts1.shape[0]:
        raise ValueError('keypoints must be [B, N, 2] and [B, M, 2]')
    B, n, m = kpts0.shape[0], kpts0.shape[1], kpts1.shape[1]
    if n == 0 or m == 0:
        raise ValueError('empty keypoint set')
    kind = transformation['type'][0]                       # reference utils/misc.py:23: one type per batch
    tf = _cabi.OgGtTransform()
    keep = []                                              # tensors the struct points into

    def ptr(name, shape):
        t = _f32(transformation[name], dev)
        if tuple(t.shape) != shape:
            raise ValueError(f'transformation[{name!r}] has shape {tuple(t.shape)}, expected {shape}')
        keep.append(t)
        return t.data_ptr()

    if kind == 'perspective':
        tf.type = _cabi.OG_GT_PERSPECTIVE
        tf.H = ptr('H', (B, 3, 3))
    elif kind == '3d_reprojection':
        tf.type = _cabi.OG_GT_3D_REPROJECTION
        tf.K0, tf.K1, tf.R, tf.T = ptr('K0', (B, 3, 3)), ptr('K1', (B, 3, 3)), ptr('R', (B, 3, 3)), ptr('T', (B, 3))
        d0, d1 = transformation['depth0'], transformation['depth1']
        if d0.dim() == 2:                                  # reference utils/misc.py:87-89: depth per keypoint
            tf.depth_is_image = 0
            tf.depth0, tf.depth1 = ptr('depth0', (B, n)), ptr('depth1', (B, m))
        else:                                              # utils/misc.py:90-97: depth images [B, H, W]
            tf.depth_is_image = 1
            tf.depth0_h, tf.depth0_w, tf.depth1_h, tf.depth1_w = d0.shape[-2], d0.shape[-1], d1.shape[-2], d1.shape[-1]
            tf.depth0 = ptr('depth0', (B, d0.shape[-2], d0.shape[-1]))
            tf.depth1 = ptr('depth1', (B, d1.shape[-2], d1.shape[-1]))
    else:
        raise ValueError(f'Unknown transformation type {kind}.')      # reference utils/misc.py:34
    k0, k1 = _f32(kpts0, dev), _f32(kpts1, dev)
    lib = _cabi.lib()
    with torch.cuda.device(dev):
        ws_bytes = _cabi.check_size(lib.og_gt_matches_workspace_bytes(B, n, m), 'og_gt_matches_workspace_bytes')
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        gt0 = torch.empty(B, n, dtype=torch.int64, device=dev)
        gt1 = torch.empty(B, m, dtype=torch.int64, device=dev)
        if lengths is not None:
            rc = lib.og_gt_matches_fwd_padded(_cabi.ptr(k0), _cabi.ptr(k1), B, n, m, _cabi.ptr(lengths), C.byref(tf), _cabi.ptr(gt0),
                                              _cabi.ptr(gt1), _cabi.ptr(ws), ws_bytes, _cabi.stream(dev))
            _cabi.check(rc, 'og_gt_matches_fwd_padded')
        else:
            rc = lib.og_gt_matches_fwd(_cabi.ptr(k0), _cabi.ptr(k1), B, n, m, C.byref(tf), _cabi.ptr(gt0), _cabi.ptr(gt1), _cabi.ptr(ws),
                                       ws_bytes, _cabi.stream(dev))
            _cabi.check(rc, 'og_gt_matches_fwd')
        # the kernels are only enqueued: keep their inputs alive on this stream
        for t in keep + [k0, k1, ws] + ([lengths] if lengths is not None else []):
            t.record_stream(torch.cuda.current_stream(dev))
    return gt0, gt1


def generate_gt_matches(data: Dict[str, Any], features0: Dict[str, torch.Tensor], features1: Dict[str, torch.Tensor],
                        positive_threshold: float, negative_threshold: Optional[float] = None
                        ) -> Tuple[Optional[Dict[str, Any]], Optional[Dict[str, torch.Tensor]]]:
    """Same contract as the reference function (models/gt_matches_generation.py:17-93).  A padded batch (``data`` with
    ``num_keypoints0`` / ``num_keypoints1``) labels each pair from its own keypoints, and ``y_true`` carries the lengths on to
    :func:`~openglue_b200.criterion`."""
    kpts0, kpts1 = features0['keypoints'], features1['keypoints']
    if kpts0.size(1) == 0 or kpts1.size(1) == 0:           # reference :33-35
        return None, None
    lengths, y_len = None, {}
    if is_padded(data):
        y_len = padded_lengths(data, kpts0.shape[0], kpts0.shape[1], kpts1.shape[1])
        lengths = torch.cat([y_len['num_keypoints0'].to(kpts0.device), y_len['num_keypoints1'].to(kpts0.device)]).contiguous()
        y_len = {k: data[k] for k in y_len}
    gt0, gt1 = gt_matches(kpts0, kpts1, data['transformation'], lengths)
    data = {**data,
            'keypoints0': kpts0, 'keypoints1': kpts1,
            'local_descriptors0': features0['local_descriptors'], 'local_descriptors1': features1['local_descriptors'],
            'side_info0': features0['side_info'], 'side_info1': features1['side_info']}
    return data, {'gt_matches0': gt0, 'gt_matches1': gt1, **y_len}
