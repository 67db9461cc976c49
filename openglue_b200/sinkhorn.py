"""Differentiable dustbin-augmented log-domain Sinkhorn on the GPU: the forward AND the backward pass of the reference's
``SuperGlue.get_matching_probs`` + ``log_otp_solver`` (reference models/superglue/superglue.py:88-111,
models/superglue/optimal_transport.py:4-28) as hand-written kernels behind ``og_sinkhorn_train_fwd`` / ``og_sinkhorn_bwd``.

``matching_log_probs(S, dustbin_score, num_iters, reg)`` returns the [B, N+1, M+1] log-assignment and is a
``torch.autograd.Function``: its backward runs the T unrolled iterations in reverse from the scaling-vector history the
forward recorded (what torch autograd does for the reference in ``training_step``, models/matching_module.py:99-105, without
the T x (N+1)(M+1) tape).  There is no CPU path.
"""
from __future__ import annotations

import torch

from . import _cabi
from ._ops import _Ops

__all__ = ['matching_log_probs']


class _Sinkhorn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, S: torch.Tensor, dustbin: torch.Tensor, num_iters: int, reg: float):
        dev = S.device
        if dev.type != 'cuda':
            raise RuntimeError('openglue_b200.matching_log_probs needs CUDA tensors (sm_90a); there is no CPU path')
        B, n, m = S.shape
        lds = (m + 3) // 4 * 4
        Sp = torch.zeros(B, n, lds, dtype=torch.float32, device=dev)       # 16-byte aligned rows (the kernels' layout)
        Sp[:, :, :m] = S.detach().float()
        dust = dustbin.detach().float().reshape(1).contiguous()
        with torch.cuda.device(dev):
            scores, hist = _Ops(dev, _cabi.OG_PREC_FP32).sinkhorn_fwd(Sp, dust, B, n, m, int(num_iters), float(reg))
        ctx.save_for_backward(Sp, dust, hist)
        ctx.meta = (B, n, m, lds, int(num_iters), float(reg), dustbin.shape, S.dtype, dustbin.dtype)
        return scores

    @staticmethod
    def backward(ctx, G: torch.Tensor):
        Sp, dust, hist = ctx.saved_tensors
        B, n, m, lds, T, reg, dshape, sdt, ddt = ctx.meta
        dev = Sp.device
        G = G.detach().float().contiguous()
        with torch.cuda.device(dev):
            dZ, dd = _Ops(dev, _cabi.OG_PREC_FP32).sinkhorn_bwd(Sp, dust, hist, G, B, n, m, T, reg)
        return dZ[:, :n, :m].to(sdt), dd.reshape(dshape).to(ddt), None, None


def matching_log_probs(S: torch.Tensor, dustbin_score: torch.Tensor, num_iters: int, reg: float = 1.0) -> torch.Tensor:
    """reference SuperGlue.get_matching_probs(S) (superglue.py:88-111): S [B, N, M] -> log-assignment [B, N+1, M+1];
    differentiable with respect to ``S`` and ``dustbin_score``."""
    return _Sinkhorn.apply(S, dustbin_score, num_iters, reg)
