"""Matching loss on the GPU: drop-in for ``utils.losses.criterion`` (reference utils/losses.py:7-53), the call that
follows the matching core in the reference's ``training_step`` (models/matching_module.py:101).

Same signature and return value ``{'loss', 'metric_loss'}``.  With ``margin=None`` (the value in every shipped config,
config/*.yaml ``margin: null`` with ``metric_weight: 0.0``) ``metric_loss`` is identically 0, as in the reference
(utils/losses.py:56-58, 83-85).  With a margin, ``metric_loss`` holds the triplet and margin terms on the half cosine distance
of the context descriptors (utils/losses.py:56-99), hard negatives mined on the GPU, and is differentiable with respect to
``context_descriptors0/1``.  The arithmetic runs in ``libopenglue_b200.so`` (``og_criterion_fwd``, ``og_metric_loss_fwd``,
both deterministic); there is no CPU path.  ``criterion_with_grad`` also returns d loss / d scores - the sparse scatter that
starts the backward pass; ``metric_loss_with_grad`` returns the metric term with its hard negatives and gradient.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from . import _cabi
from ._cabi import ptr, stream
from .superglue import is_padded, padded_lengths

__all__ = ['criterion', 'criterion_with_grad', 'metric_loss_with_grad']


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
    lens = None
    if is_padded(y_true):                                  # each pair's loss on its own block, dustbins at its lengths
        ln = padded_lengths(y_true, B, n1 - 1, m1 - 1)
        lens = torch.cat([ln['num_keypoints0'].to(dev), ln['num_keypoints1'].to(dev)]).contiguous()
    lib = _cabi.lib()
    with torch.cuda.device(dev):
        wsb = _cabi.check_size(lib.og_criterion_workspace_bytes(B), 'og_criterion_workspace_bytes')
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        loss = torch.empty(2, dtype=torch.float32, device=dev)
        dscores = torch.zeros_like(scores) if want_grad else None
        if lens is not None:
            rc = lib.og_criterion_fwd_padded(ptr(scores), ptr(gt0), ptr(gt1), B, n1 - 1, m1 - 1, ptr(lens), ptr(loss), ptr(dscores),
                                             float(grad_scale), ptr(ws), wsb, stream(dev))
            _cabi.check(rc, 'og_criterion_fwd_padded')
            return loss, dscores
        rc = lib.og_criterion_fwd(ptr(scores), ptr(gt0), ptr(gt1), B, n1 - 1, m1 - 1, ptr(loss), ptr(dscores), float(grad_scale), ptr(ws), wsb,
                                  stream(dev))
        _cabi.check(rc, 'og_criterion_fwd')
    return loss, dscores


class _Criterion(torch.autograd.Function):
    """loss = criterion(scores): the same kernel call also writes d loss / d scores, which the backward pass scales."""

    @staticmethod
    def forward(ctx, scores, y_true):
        loss, dscores = _run(y_true, {'scores': scores}, True, 1.0)
        ctx.save_for_backward(dscores)
        ctx.dtype = scores.dtype
        return loss

    @staticmethod
    def backward(ctx, gloss):
        dscores, = ctx.saved_tensors
        return (dscores * gloss[0]).to(ctx.dtype), None                # metric_loss (loss[1]) is identically 0


def _metric_run(gt0: torch.Tensor, gt1: torch.Tensor, c0: torch.Tensor, c1: torch.Tensor, margin: float, want_grad: bool,
                grad_scale: float, out: Optional[torch.Tensor] = None):
    """og_metric_loss_fwd -> (metric_loss [1] (or ``out``, written in place), (n0, u0, n1, u1), dc0, dc1).  ``gt0``/``gt1`` int64
    on the device; c0 [B, d, n], c1 [B, d, m] float32 contiguous."""
    dev = c0.device
    B, d, n = c0.shape
    m = c1.shape[2]
    lib = _cabi.lib()
    prec = _cabi.OG_PREC_TF32X3
    with torch.cuda.device(dev):
        wsb = _cabi.check_size(lib.og_metric_loss_workspace_bytes(B, d, n, m, int(want_grad), prec), 'og_metric_loss_workspace_bytes')
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        metric = out if out is not None else torch.empty(1, dtype=torch.float32, device=dev)
        n0, u0 = torch.empty(B, n, dtype=torch.int64, device=dev), torch.empty(B, n, dtype=torch.int64, device=dev)
        n1, u1 = torch.empty(B, m, dtype=torch.int64, device=dev), torch.empty(B, m, dtype=torch.int64, device=dev)
        dc0 = torch.empty_like(c0) if want_grad else None
        dc1 = torch.empty_like(c1) if want_grad else None
        rc = lib.og_metric_loss_fwd(ptr(c0), ptr(c1), ptr(gt0), ptr(gt1), B, d, n, m, float(margin), prec, ptr(metric), ptr(n0), ptr(u0),
                                    ptr(n1), ptr(u1), ptr(dc0), ptr(dc1), float(grad_scale), ptr(ws), wsb, stream(dev))
        _cabi.check(rc, 'og_metric_loss_fwd')
    return metric, (n0, u0, n1, u1), dc0, dc1


def _metric_inputs(y_true, y_pred):
    """labels and context descriptors of a criterion call with a margin, checked against the scores' shape"""
    if 'context_descriptors0' not in y_pred or 'context_descriptors1' not in y_pred:
        raise NotImplementedError('criterion(margin=...) computes its metric terms on the context descriptors: y_pred needs '
                                  "'context_descriptors0' and 'context_descriptors1' (SuperGlue.forward's outputs) besides 'scores'")
    scores = y_pred['scores']
    dev = scores.device
    if dev.type != 'cuda':
        raise RuntimeError('openglue_b200.criterion needs CUDA tensors (sm_90a); there is no CPU path')
    c0, c1 = y_pred['context_descriptors0'], y_pred['context_descriptors1']
    B, n1, m1 = scores.shape
    if c0.dim() != 3 or c1.dim() != 3 or c0.shape[0] != B or c1.shape[0] != B or c0.shape[1] != c1.shape[1] \
            or c0.shape[2] != n1 - 1 or c1.shape[2] != m1 - 1:
        raise ValueError(f'context descriptors {tuple(c0.shape)}, {tuple(c1.shape)} do not fit scores {tuple(scores.shape)}')
    if c0.device != dev or c1.device != dev:
        raise RuntimeError('scores and context descriptors must be on the same device')
    gt0 = y_true['gt_matches0'].to(device=dev, dtype=torch.int64).contiguous()
    gt1 = y_true['gt_matches1'].to(device=dev, dtype=torch.int64).contiguous()
    return gt0, gt1, c0, c1


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().float().contiguous()


class _CriterionMetric(torch.autograd.Function):
    """[loss, metric_loss] = criterion(scores, c0, c1; margin): both kernel calls also write their gradients (d loss / d scores,
    d metric_loss / d c0, c1), which the backward pass scales by the incoming gradient of each output."""

    @staticmethod
    def forward(ctx, scores, c0, c1, gt0, gt1, margin):
        loss, dscores = _run({'gt_matches0': gt0, 'gt_matches1': gt1}, {'scores': scores}, True, 1.0)
        _, _, dc0, dc1 = _metric_run(gt0, gt1, _f32(c0), _f32(c1), margin, True, 1.0, out=loss[1:])
        ctx.save_for_backward(dscores, dc0, dc1)
        ctx.dtypes = (scores.dtype, c0.dtype, c1.dtype)
        return loss

    @staticmethod
    def backward(ctx, gloss):
        dscores, dc0, dc1 = ctx.saved_tensors
        need = ctx.needs_input_grad
        return ((dscores * gloss[0]).to(ctx.dtypes[0]) if need[0] else None,
                (dc0 * gloss[1]).to(ctx.dtypes[1]) if need[1] else None,
                (dc1 * gloss[1]).to(ctx.dtypes[2]) if need[2] else None, None, None, None)


def criterion(y_true: Dict[str, torch.Tensor], y_pred: Dict[str, torch.Tensor], margin: Optional[float] = None
              ) -> Dict[str, torch.Tensor]:
    """reference utils/losses.py:7-99 -> {'loss', 'metric_loss'} (0-dim tensors on the scores' device).  Differentiable
    with respect to ``y_pred['scores']`` (the sparse scatter the gather's backward pass is) and, with a margin, to
    ``y_pred['context_descriptors0/1']``, so ``(nll_weight * out['loss'] + metric_weight * out['metric_loss']).backward()``
    drives the training step as it does in the reference (matching_module.py:101-105).

    A padded batch (``y_true`` with ``num_keypoints0`` / ``num_keypoints1``, as :func:`generate_gt_matches` returns it) takes
    each pair's loss on its own block of ``scores`` (dustbins at its lengths), ignores its labels past them and averages the B
    pairs; ``d loss / d scores`` is 0 outside the blocks.  The metric terms (``margin``) are not built for padded batches."""
    if margin is not None and is_padded(y_true):
        raise NotImplementedError('criterion(margin=...) on a padded batch (num_keypoints0 / num_keypoints1) is not built')
    if margin is not None:
        gt0, gt1, c0, c1 = _metric_inputs(y_true, y_pred)
        scores = y_pred['scores']
        if torch.is_grad_enabled() and (scores.requires_grad or c0.requires_grad or c1.requires_grad):
            loss = _CriterionMetric.apply(scores, c0, c1, gt0, gt1, float(margin))
        else:
            loss, _ = _run(y_true, y_pred, False, 1.0)
            _metric_run(gt0, gt1, _f32(c0), _f32(c1), float(margin), False, 1.0, out=loss[1:])
        return {'loss': loss[0], 'metric_loss': loss[1]}
    if torch.is_grad_enabled() and y_pred['scores'].requires_grad:
        loss = _Criterion.apply(y_pred['scores'], y_true)
    else:
        loss, _ = _run(y_true, y_pred, False, 1.0)
    return {'loss': loss[0], 'metric_loss': loss[1]}


def criterion_with_grad(y_true, y_pred, grad_scale: float = 1.0) -> Tuple[Dict[str, torch.Tensor], torch.Tensor]:
    """-> ({'loss', 'metric_loss'}, grad_scale * d loss / d scores [B, N+1, M+1])."""
    loss, dscores = _run(y_true, y_pred, True, grad_scale)
    return {'loss': loss[0], 'metric_loss': loss[1]}, dscores


def metric_loss_with_grad(y_true, y_pred, margin: float, grad_scale: float = 1.0, want_grad: bool = True) -> Dict[str, torch.Tensor]:
    """The metric term alone (``y_pred``: ``context_descriptors0/1``; ``scores`` only for its shape check when present) ->
    {'metric_loss' (0-dim), 'n0', 'u0' [B, n], 'n1', 'u1' [B, m] (the hard negatives: n0 / n1 the argmins with each matched
    pair masked, u0 / u1 the unmasked ones), 'dc0' [B, d, n], 'dc1' [B, d, m] (grad_scale * d metric_loss / d c0, c1; None
    without ``want_grad``)}."""
    if 'scores' not in y_pred:
        c0 = y_pred['context_descriptors0']
        y_pred = dict(y_pred, scores=c0.new_empty(c0.shape[0], c0.shape[2] + 1, y_pred['context_descriptors1'].shape[2] + 1))
    gt0, gt1, c0, c1 = _metric_inputs(y_true, y_pred)
    metric, (n0, u0, n1, u1), dc0, dc1 = _metric_run(gt0, gt1, _f32(c0), _f32(c1), float(margin), want_grad, grad_scale)
    return {'metric_loss': metric[0], 'n0': n0, 'u0': u0, 'n1': n1, 'u1': u1, 'dc0': dc0, 'dc1': dc1}
