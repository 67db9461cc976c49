"""CPU oracle for the metric terms of the matching loss  --  TEST INFRASTRUCTURE, NOT PRODUCT.

Restates ``criterion(..., margin=mu)['metric_loss']`` (reference utils/losses.py:56-99 on the half cosine distance of
utils/misc.py:106-113) as plain torch, in the reference's order of operations, and also returns what the loss selected: the four
hard-negative index vectors, each selection's gap (runner-up minus minimum) and every hinge argument.  Differentiable with respect
to the context descriptors through torch autograd.  Pinned by tests/golden/metric_*.pt, minted by oracle/gen_golden_metric_loss.py
from the UNMODIFIED reference function (tests/test_metric_loss_oracle.py).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle.loss_oracle import _mean_weights

Tensor = torch.Tensor


def half_cosine_dist(c0: Tensor, c1: Tensor) -> Tensor:
    """c0 [B, d, n], c1 [B, d, m] -> 0.25 |normalize(x_i) - normalize(y_j)|^2 [B, n, m], through torch.cdist as the reference"""
    x = F.normalize(c0.transpose(2, 1).contiguous(), dim=-1)
    y = F.normalize(c1.transpose(2, 1).contiguous(), dim=-1)
    return 0.25 * torch.cdist(x, y).pow(2)


def _gap(v: Tensor, dim: int) -> Tensor:
    """runner-up minus minimum along ``dim`` (inf with a single candidate)"""
    if v.shape[dim] < 2:
        return torch.full(v.select(dim, 0).shape, float('inf'), dtype=v.dtype)
    two = torch.topk(v, 2, dim=dim, largest=False).values
    return two.select(dim, 1) - two.select(dim, 0)


def metric_terms(gt0: Tensor, gt1: Tensor, c0: Tensor, c1: Tensor, margin: float) -> Dict[str, Tensor]:
    """-> {'metric_loss', 'dist', 'n0', 'u0' [B, n], 'n1', 'u1' [B, m], 'gap_n0', 'gap_u0', 'gap_n1', 'gap_u1' (same shapes),
    'a0', 'a1' (hinge arguments of the matched rows, in torch.where order), 'au0', 'au1' (of the unmatched rows / columns)}"""
    dist = half_cosine_dist(c0, c1)
    zero = torch.zeros((), dtype=dist.dtype)
    B = c0.shape[0]
    # matched rows: positive against the hardest negative of its row and of its column, the positives masked out
    b, i = torch.where(gt0 >= 0)
    j = gt0[b, i]
    w = _mean_weights(b)
    masked = dist.detach().clone()
    masked[b, i, j] = float('inf')
    n0, n1 = masked.argmin(dim=2), masked.argmin(dim=1)
    free = dist.detach()
    u0, u1 = free.argmin(dim=2), free.argmin(dim=1)
    pos = dist[b, i, j]
    a0 = pos - dist[b, i, n0[b, i]] + margin
    a1 = pos - dist[b, n1[b, j], j] + margin
    matched = (torch.maximum(a0, zero) * w).sum() + (torch.maximum(a1, zero) * w).sum()
    # unmatched rows of image 0 and columns of image 1: their nearest neighbour pushed beyond the margin
    b, i = torch.where(gt0 == -1)
    au0 = margin - dist[b, i, u0[b, i]]
    un0 = (torch.maximum(au0, zero) * _mean_weights(b)).sum()
    b, j = torch.where(gt1 == -1)
    au1 = margin - dist[b, u1[b, j], j]
    un1 = (torch.maximum(au1, zero) * _mean_weights(b)).sum()
    return {'metric_loss': (matched + un0 + un1) / B, 'dist': dist,
            'n0': n0, 'u0': u0, 'n1': n1, 'u1': u1,
            'gap_n0': _gap(masked, 2), 'gap_u0': _gap(free, 2), 'gap_n1': _gap(masked, 1), 'gap_u1': _gap(free, 1),
            'a0': a0.detach(), 'a1': a1.detach(), 'au0': au0.detach(), 'au1': au1.detach()}


def used_margins(gt0: Tensor, gt1: Tensor, out: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """The gaps of the selections the loss reads (n0 of matched rows, n1 of the columns they name, u0 of unmatched rows, u1 of
    unmatched columns) and |hinge argument| of every term: how far each decision the loss makes is from flipping."""
    b, i = torch.where(gt0 >= 0)
    j = gt0[b, i]
    b0, i0 = torch.where(gt0 == -1)
    b1, j1 = torch.where(gt1 == -1)
    return {'gap_n0': out['gap_n0'][b, i], 'gap_n1': out['gap_n1'][b, j], 'gap_u0': out['gap_u0'][b0, i0], 'gap_u1': out['gap_u1'][b1, j1],
            'a0': out['a0'].abs(), 'a1': out['a1'].abs(), 'au0': out['au0'].abs(), 'au1': out['au1'].abs()}


def smallest_margin(gt0: Tensor, gt1: Tensor, out: Dict[str, Tensor]) -> float:
    return min([float(v.min()) for v in used_margins(gt0, gt1, out).values() if v.numel()] + [float('inf')])
