"""Matching loss on the GPU: drop-in for ``utils.losses.criterion`` (reference utils/losses.py:7-53), the call that
follows the matching core in the reference's ``training_step`` (models/matching_module.py:101).

Same signature and return value ``{'loss', 'metric_loss'}``.  ``margin=None`` (the value in every shipped config,
config/*.yaml ``margin: null`` with ``metric_weight: 0.0``) is the implemented case: ``metric_loss`` is then identically 0
in the reference too (utils/losses.py:56-58, 83-85).  The arithmetic runs in ``libopenglue_b200.so``
(``og_criterion_fwd``, deterministic); there is no CPU path.  ``criterion_with_grad`` also returns
d loss / d scores - the sparse scatter that starts the backward pass.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from . import _cabi
from ._cabi import ptr, stream

__all__ = ['criterion', 'criterion_with_grad']


def _run(y_true: Dict[str, torch.Tensor], y_pred: Dict[str, torch.Tensor], want_grad: bool, grad_scale: float):
    scores = y_pred['scores']
    dev = scores.device
    if dev.type != 'cuda':
        raise RuntimeError('openglue_b200.criterion needs CUDA tensors (sm_90a); there is no CPU path')
    scores = scores.detach().float().contiguous()
    B, n1, m1 = scores.shape
    gt0 = y_true['gt_matches0'].to(device=dev, dtype=torch.int64).contiguous()
    gt1 = y_true['gt_matches1'].to(device=dev, dtype=torch.int64).contiguous()
    if gt0.shape != (B, n1 - 1) or gt1.shape != (B, m1 - 1):
        raise ValueError(f'gt_matches shapes {tuple(gt0.shape)}, {tuple(gt1.shape)} do not fit scores {tuple(scores.shape)}')
    lib = _cabi.lib()
    with torch.cuda.device(dev):
        wsb = _cabi.check_size(lib.og_criterion_workspace_bytes(B), 'og_criterion_workspace_bytes')
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        loss = torch.empty(2, dtype=torch.float32, device=dev)
        dscores = torch.zeros_like(scores) if want_grad else None
        rc = lib.og_criterion_fwd(ptr(scores), ptr(gt0), ptr(gt1), B, n1 - 1, m1 - 1, ptr(loss), ptr(dscores), float(grad_scale), ptr(ws), wsb,
                                  stream(dev))
        _cabi.check(rc, 'og_criterion_fwd')
    return loss, dscores


class _Criterion(torch.autograd.Function):
    """loss = criterion(scores): the same kernel call also writes d loss / d scores, which the backward pass scales."""

    @staticmethod
    def forward(ctx, scores, gt0, gt1):
        loss, dscores = _run({'gt_matches0': gt0, 'gt_matches1': gt1}, {'scores': scores}, True, 1.0)
        ctx.save_for_backward(dscores)
        ctx.dtype = scores.dtype
        return loss

    @staticmethod
    def backward(ctx, gloss):
        dscores, = ctx.saved_tensors
        return (dscores * gloss[0]).to(ctx.dtype), None, None          # metric_loss (loss[1]) is identically 0


def criterion(y_true: Dict[str, torch.Tensor], y_pred: Dict[str, torch.Tensor], margin: Optional[float] = None
              ) -> Dict[str, torch.Tensor]:
    """reference utils/losses.py:7-53 -> {'loss', 'metric_loss'} (0-dim tensors on the scores' device).  Differentiable
    with respect to ``y_pred['scores']`` (the sparse scatter the gather's backward pass is), so
    ``criterion(...)['loss'].backward()`` drives the training step as it does in the reference (matching_module.py:101-105)."""
    if margin is not None:
        raise NotImplementedError('openglue_b200.criterion implements margin=None (every shipped reference config); '
                                  'the triplet terms of utils/losses.py:56-99 are not built')
    if torch.is_grad_enabled() and y_pred['scores'].requires_grad:
        loss = _Criterion.apply(y_pred['scores'], y_true['gt_matches0'], y_true['gt_matches1'])
    else:
        loss, _ = _run(y_true, y_pred, False, 1.0)
    return {'loss': loss[0], 'metric_loss': loss[1]}


def criterion_with_grad(y_true, y_pred, grad_scale: float = 1.0) -> Tuple[Dict[str, torch.Tensor], torch.Tensor]:
    """-> ({'loss', 'metric_loss'}, grad_scale * d loss / d scores [B, N+1, M+1])."""
    loss, dscores = _run(y_true, y_pred, True, grad_scale)
    return {'loss': loss[0], 'metric_loss': loss[1]}, dscores
