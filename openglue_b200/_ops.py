"""ctypes wrappers of the library's operator-level entry points on torch-owned buffers: the toolbox the training step
(openglue_b200/training.py) and the SuperPoint front-end (openglue_b200/superpoint.py) schedule their kernels with.  torch only
allocates; every arithmetic operation is a kernel of libopenglue_b200.so (include/openglue_b200.h)."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch

from . import _cabi
from ._cabi import ptr


def _pad4(n: int) -> int:
    return (n + 3) // 4 * 4


class _Ops:
    """ctypes wrappers of the training operators on the current stream of ``dev`` (fp32 CUDA tensors in, out).

    A padded batch passes per-pair lengths ``lens`` (device int32 [B]: the first ``lens[b]`` of pair b's ``cap`` rows are real;
    for the Sinkhorn, the B row lengths then the B column lengths); without them every operator runs its uniform form."""

    def __init__(self, dev: torch.device, precision: int):
        self.dev, self.prec = dev, precision
        self.lib = _cabi.lib()
        self._ws: Dict[int, torch.Tensor] = {}

    def st(self):
        return _cabi.stream(self.dev)

    def empty(self, *shape):
        return torch.empty(*shape, dtype=torch.float32, device=self.dev)

    def zeros(self, *shape):
        return torch.zeros(*shape, dtype=torch.float32, device=self.dev)

    def ws(self, cols: int) -> torch.Tensor:
        t = self._ws.get(cols)
        if t is None:
            t = self._ws[cols] = self.empty(_cabi.check_size(self.lib.og_train_workspace_floats(cols), 'og_train_workspace_floats'))
        return t

    # ---- Y[b] = alpha [A | A2][b] . W[b]^T + bias (+ relu) (+ R[b]);  pointers = (tensor, float offset) ----
    def gemm(self, A, lda, k1, W, ldw, rows, nout, Y, ldy, *, a_off=0, w_off=0, y_off=0, A2=None, lda2=0, k2=0, a2_off=0, bias=None,
             relu=False, alpha=1.0, R=None, ldr=0, r_off=0, batch=1, strideA=0, strideA2=0, strideW=0, strideY=0, strideR=0,
             Yt=None, ldyt=0, strideYt=0, yt_off=0):
        a = _cabi.OgLinearArgs()
        a.A, a.lda, a.strideA = ptr(A, a_off), lda, strideA
        a.A2, a.lda2, a.strideA2 = ptr(A2, a2_off), lda2, strideA2
        a.k1, a.k2 = k1, k2
        a.W, a.ldw, a.strideW = ptr(W, w_off), ldw, strideW
        a.bias = ptr(bias)
        a.rows, a.nout, a.batch = rows, nout, batch
        a.alpha, a.relu = float(alpha), int(relu)
        a.R, a.ldr, a.strideR = ptr(R, r_off), ldr, strideR
        a.rscale = None
        a.Y, a.ldy, a.strideY = ptr(Y, y_off), ldy, strideY
        a.Yt, a.ldyt, a.strideYt = ptr(Yt, yt_off), ldyt, strideYt
        scratch = None
        if self.prec != _cabi.OG_PREC_FP32:
            scratch = self.empty(max(int(self.lib.og_linear_auto_scratch_floats(C.byref(a))), 4))
        _cabi.check(self.lib.og_linear_auto_fwd(C.byref(a), self.prec, ptr(scratch), self.st()), 'og_linear_auto_fwd')

    def linear(self, X, W, bias=None, *, relu=False, A2=None, R=None, out=None):
        """X [rows, k1] (| A2 [rows, k2]) . W[nout, k1 + k2]^T + bias (+ R) -> [rows, nout]"""
        rows, k1 = X.shape
        k2 = A2.shape[1] if A2 is not None else 0
        nout = W.shape[0]
        Y = out if out is not None else self.empty(rows, nout)
        self.gemm(X, X.stride(0), k1, W, k1 + k2, rows, nout, Y, Y.stride(0), A2=A2, lda2=(A2.stride(0) if A2 is not None else 0), k2=k2,
                  bias=bias, relu=relu, R=R, ldr=(R.stride(0) if R is not None else 0))
        return Y

    def transpose(self, X, *, batch=1, rows=None, cols=None, pad=True):
        """[batch][rows, cols] (dense) -> zero-padded [batch][cols, pad4(rows)]"""
        if rows is None:
            rows, cols = X.shape[-2], X.shape[-1]
        rp = _pad4(rows) if pad else rows
        out = self.zeros(batch, cols, rp) if rp != rows else self.empty(batch, cols, rp)
        self.transpose_raw(X, 0, cols, rows * cols, out, rp, cols * rp, batch, rows, cols, True)
        return out

    def colsum(self, X, Y=None, Z=None):
        rows, cols = X.shape
        out = self.empty(cols)
        _cabi.check(self.lib.og_colsum(ptr(X), X.stride(0), ptr(Y), Y.stride(0) if Y is not None else 0, ptr(Z), Z.stride(0) if Z is not None else 0,
                                       rows, cols, ptr(out), ptr(self.ws(cols)), self.st()), 'og_colsum')
        return out

    def axpby(self, x, y, a=1.0, b=1.0, out=None):
        out = out if out is not None else torch.empty_like(x)
        _cabi.check(self.lib.og_axpby(ptr(x), ptr(y), float(a), float(b), ptr(out), x.numel(), self.st()), 'og_axpby')
        return out

    def transpose_raw(self, X, x_off, ld_in, stride_in, out, ld_out, stride_out, batch, rows, cols, transpose):
        _cabi.check(self.lib.og_transpose(ptr(X, x_off), ld_in, stride_in, ptr(out), ld_out, stride_out, batch, rows, cols, int(transpose), self.st()),
                    'og_transpose')

    def kenc_input(self, kpts, side, rows, S, width, height, lens=None, pair_wh=None):
        """``pair_wh``: padded batch, (W, H) of pair b's image at pair_wh[b, :2] (rows 4 floats apart)"""
        out = self.empty(rows, 2 + S)
        if lens is not None:
            B = lens.numel()
            _cabi.check(self.lib.og_kenc_input_padded(ptr(kpts), ptr(side) if S else None, B, rows // B, ptr(lens), S, ptr(pair_wh), ptr(out),
                                                      self.st()), 'og_kenc_input_padded')
            return out
        _cabi.check(self.lib.og_kenc_input(ptr(kpts), ptr(side) if S else None, rows, S, float(width), float(height), ptr(out), self.st()), 'og_kenc_input')
        return out

    def mask_rows(self, X, lens):
        """X [B * cap, cols] -> a copy with the rows past each pair's length zeroed"""
        rows, cols = X.shape
        B = lens.numel()
        out = self.empty(rows, cols)
        _cabi.check(self.lib.og_mask_padded_rows(ptr(X), B, rows // B, cols, ptr(lens), ptr(out), self.st()), 'og_mask_padded_rows')
        return out

    def attention(self, q, k, v, B, nq, nk, H, dh, klen=None):
        """fused softmax attention (forward): the wgmma 3xTF32 kernel for head_dim 32 / 64 (K and V^T as tf32 hi/lo operands),
        the fp32 CUDA-core kernel otherwise / in fp32 mode; ``klen``: sequence b attends to its first klen[b] keys"""
        d = H * dh
        o = self.empty(B * nq, d)
        if self.prec != _cabi.OG_PREC_FP32 and dh in (32, 64):
            khi, klo = torch.empty_like(k), torch.empty_like(k)
            _cabi.check(self.lib.og_split_tf32(ptr(k), ptr(khi), ptr(klo), k.numel(), self.st()), 'og_split_tf32')
            vt = self.transpose(v, batch=B, rows=nk, cols=d)            # [B, d, pad4(nk)], zero padded
            vthi, vtlo = torch.empty_like(vt), torch.empty_like(vt)
            _cabi.check(self.lib.og_split_tf32(ptr(vt), ptr(vthi), ptr(vtlo), vt.numel(), self.st()), 'og_split_tf32')
            if klen is not None:
                _cabi.check(self.lib.og_attention_tc_fwd_padded(ptr(q), d, nq * d, ptr(khi), ptr(klo), d, ptr(vthi), ptr(vtlo), vt.shape[2], ptr(o),
                                                                d, nq * d, B, nq, nk, H, dh, ptr(klen), self.st()), 'og_attention_tc_fwd_padded')
                return o
            _cabi.check(self.lib.og_attention_tc_fwd(ptr(q), d, nq * d, ptr(khi), ptr(klo), d, ptr(vthi), ptr(vtlo), vt.shape[2], ptr(o), d, nq * d,
                                                     B, nq, nk, H, dh, self.st()), 'og_attention_tc_fwd')
            return o
        if klen is not None:
            _cabi.check(self.lib.og_attention_fwd_padded(ptr(q), d, nq * d, ptr(k), d, nk * d, ptr(v), d, nk * d, ptr(o), d, nq * d, B, nq, nk, H,
                                                         dh, ptr(klen), self.st()), 'og_attention_fwd_padded')
            return o
        _cabi.check(self.lib.og_attention_fwd(ptr(q), d, nq * d, ptr(k), d, nk * d, ptr(v), d, nk * d, ptr(o), d, nq * d, B, nq, nk, H, dh,
                                              _cabi.OG_PREC_FP32, self.st()), 'og_attention_fwd')
        return o

    def softmax_rows(self, P, ld, rows, cols, klen=None):
        """``klen``: rows are [B, rows / B] and sequence b's rows take its first klen[b] columns (P = 0 past them)"""
        if klen is not None:
            B = klen.numel()
            _cabi.check(self.lib.og_softmax_rows_padded(ptr(P), ld, B, rows // B, cols, ptr(klen), self.st()), 'og_softmax_rows_padded')
            return
        _cabi.check(self.lib.og_softmax_rows(ptr(P), ld, rows, cols, self.st()), 'og_softmax_rows')

    def softmax_bwd_rows(self, P, dP, ld, rows, cols, scale, klen=None):
        if klen is not None:
            B = klen.numel()
            _cabi.check(self.lib.og_softmax_bwd_rows_padded(ptr(P), ptr(dP), ld, B, rows // B, cols, float(scale), ptr(klen), self.st()),
                        'og_softmax_bwd_rows_padded')
            return
        _cabi.check(self.lib.og_softmax_bwd_rows(ptr(P), ptr(dP), ld, rows, cols, float(scale), self.st()), 'og_softmax_bwd_rows')

    def mix_fwd(self, g, l, mix):
        rows, d = g.shape
        out = self.empty(rows, d)
        _cabi.check(self.lib.og_mix_fwd(ptr(g), ptr(l), ptr(mix), ptr(out), rows, d, self.st()), 'og_mix_fwd')
        return out

    def mix_bwd(self, dm, mix):
        rows, d = dm.shape
        dg, dl = self.empty(rows, d), self.empty(rows, d)
        _cabi.check(self.lib.og_mix_bwd(ptr(dm), ptr(mix), ptr(dg), ptr(dl), rows, d, self.st()), 'og_mix_bwd')
        return dg, dl

    def mix_param_grad(self, csum, mix):
        d = mix.numel()
        out = self.empty(d)
        _cabi.check(self.lib.og_mix_param_grad(ptr(csum), ptr(mix), ptr(out), d, self.st()), 'og_mix_param_grad')
        return out

    def bn_fwd(self, a, gamma, beta, eps, momentum, running_mean, running_var, lens=None, skip=None, num_batches_tracked=None):
        """``lens``: statistics over the real rows of every pair (rows [B, cap]).  ``skip`` (device int32 flag): the guarded form,
        which leaves the running statistics untouched when the flag is set and adds 1 - skip to ``num_batches_tracked``."""
        rows, cols = a.shape
        y, mean, invstd = self.empty(rows, cols), self.empty(cols), self.empty(cols)
        if skip is not None:
            B = 1 if lens is None else lens.numel()
            _cabi.check(self.lib.og_bn_train_fwd_guarded(ptr(a), a.stride(0), B, rows // B, ptr(lens), cols, 1, ptr(gamma), ptr(beta), float(eps),
                                                         float(momentum), ptr(y), cols, ptr(mean), ptr(invstd), ptr(running_mean),
                                                         ptr(running_var), ptr(skip), ptr(num_batches_tracked), ptr(self.ws(cols)), self.st()),
                        'og_bn_train_fwd_guarded')
            return y, mean, invstd
        if lens is not None:
            B = lens.numel()
            _cabi.check(self.lib.og_bn_train_fwd_padded(ptr(a), a.stride(0), B, rows // B, ptr(lens), cols, 1, ptr(gamma), ptr(beta), float(eps),
                                                        float(momentum), ptr(y), cols, ptr(mean), ptr(invstd), ptr(running_mean),
                                                        ptr(running_var), ptr(self.ws(cols)), self.st()), 'og_bn_train_fwd_padded')
            return y, mean, invstd
        _cabi.check(self.lib.og_bn_train_fwd(ptr(a), a.stride(0), rows, cols, 1, ptr(gamma), ptr(beta), float(eps), float(momentum), ptr(y), cols,
                                             ptr(mean), ptr(invstd), ptr(running_mean), ptr(running_var), ptr(self.ws(cols)), self.st()), 'og_bn_train_fwd')
        return y, mean, invstd

    def bn_bwd(self, dy, a, gamma, mean, invstd, lens=None):
        rows, cols = a.shape
        da, dgamma, dbeta = self.empty(rows, cols), self.empty(cols), self.empty(cols)
        if lens is not None:
            B = lens.numel()
            _cabi.check(self.lib.og_bn_train_bwd_padded(ptr(dy), dy.stride(0), ptr(a), a.stride(0), B, rows // B, ptr(lens), cols, 1, ptr(gamma),
                                                        ptr(mean), ptr(invstd), ptr(da), cols, ptr(dgamma), ptr(dbeta), ptr(self.ws(cols)),
                                                        self.st()), 'og_bn_train_bwd_padded')
            return da, dgamma, dbeta
        _cabi.check(self.lib.og_bn_train_bwd(ptr(dy), dy.stride(0), ptr(a), a.stride(0), rows, cols, 1, ptr(gamma), ptr(mean), ptr(invstd), ptr(da), cols,
                                             ptr(dgamma), ptr(dbeta), ptr(self.ws(cols)), self.st()), 'og_bn_train_bwd')
        return da, dgamma, dbeta

    def sinkhorn_fwd(self, Sp, dust, B, n, m, iters, reg, lens=None):
        """``lens``: [2B] row then column lengths of a padded batch"""
        lib, lds = self.lib, Sp.shape[2]
        scores = self.empty(B, n + 1, m + 1)
        hist = self.empty(max(int(lib.og_sinkhorn_hist_floats(B, n, m, iters)), 1))
        wsb = _cabi.check_size(lib.og_sinkhorn_workspace_bytes(B, n, m), 'og_sinkhorn_workspace_bytes')
        ws = torch.empty(wsb, dtype=torch.uint8, device=self.dev)
        if lens is not None:
            _cabi.check(lib.og_sinkhorn_train_fwd_padded(ptr(Sp), lds, n * lds, ptr(dust), B, n, m, ptr(lens), iters, reg, ptr(scores), ptr(hist),
                                                         ptr(ws), wsb, self.st()), 'og_sinkhorn_train_fwd_padded')
            return scores, hist
        _cabi.check(lib.og_sinkhorn_train_fwd(ptr(Sp), lds, n * lds, ptr(dust), B, n, m, iters, reg, ptr(scores), ptr(hist), ptr(ws), wsb, self.st()),
                    'og_sinkhorn_train_fwd')
        return scores, hist

    def sinkhorn_bwd(self, Sp, dust, hist, G, B, n, m, iters, reg, lens=None):
        lib, lds = self.lib, Sp.shape[2]
        dZ, dd = self.empty(B, n + 1, m + 1), self.empty(1)
        wsb = _cabi.check_size(lib.og_sinkhorn_bwd_workspace_bytes(B, n, m, iters), 'og_sinkhorn_bwd_workspace_bytes')
        ws = torch.empty(wsb, dtype=torch.uint8, device=self.dev)
        if lens is not None:
            _cabi.check(lib.og_sinkhorn_bwd_padded(ptr(Sp), lds, n * lds, ptr(dust), B, n, m, ptr(lens), iters, reg, ptr(hist), ptr(G), ptr(dZ),
                                                   ptr(dd), ptr(ws), wsb, self.st()), 'og_sinkhorn_bwd_padded')
            return dZ, dd
        _cabi.check(lib.og_sinkhorn_bwd(ptr(Sp), lds, n * lds, ptr(dust), B, n, m, iters, reg, ptr(hist), ptr(G), ptr(dZ), ptr(dd), ptr(ws), wsb, self.st()),
                    'og_sinkhorn_bwd')
        return dZ, dd

    def sum_batches(self, part, S, rows, cols, out, out_off, ld, accumulate=True):
        _cabi.check(self.lib.og_sum_batches(ptr(part), S, rows, cols, ptr(out, out_off), ld, int(accumulate), self.st()), 'og_sum_batches')

    def _transpose_chunks(self, X, S, Kc):
        """[rows, cols] -> zero-padded [S, cols, Kc]: chunk s holds rows [s Kc, (s + 1) Kc) transposed"""
        rows, cols = X.shape
        out = self.zeros(S, cols, Kc) if rows != S * Kc else self.empty(S, cols, Kc)
        nfull = rows // Kc
        if nfull:
            self.transpose_raw(X, 0, cols, Kc * cols, out, Kc, cols * Kc, nfull, Kc, cols, True)
        if rows - nfull * Kc:
            self.transpose_raw(X, nfull * Kc * cols, cols, 0, out[nfull], Kc, 0, 1, rows - nfull * Kc, cols, True)
        return out

    SPLIT_K = 512

    def grad_weight(self, dY, X, into, col_off=0):
        """into[:, col_off : col_off + K] += dY^T X   (dY [rows, nout], X [rows, K], into [nout, ld]).  The contraction runs over the
        rows (thousands) while the output is one or four GEMM tiles: it is split into chunks of SPLIT_K rows that run as ONE batched
        GEMM (enough tiles for the whole GPU) and are summed in a fixed order."""
        rows, nout = dY.shape
        K = X.shape[1]
        ld = into.stride(0)
        Kc = self.SPLIT_K
        S = (rows + Kc - 1) // Kc
        if S <= 1:
            dYt = self.transpose(dY)                  # [1, nout, rp]
            Xt = self.transpose(X)                    # [1, K, rp]
            rp = dYt.shape[2]
            self.gemm(dYt, rp, rp, Xt, rp, nout, K, into, ld, y_off=col_off, R=into, ldr=ld, r_off=col_off)
            return
        dYt = self._transpose_chunks(dY, S, Kc)       # [S, nout, Kc]
        Xt = self._transpose_chunks(X, S, Kc)         # [S, K, Kc]
        part = self.empty(S, nout, K)
        self.gemm(dYt, Kc, Kc, Xt, Kc, nout, K, part, K, batch=S, strideA=nout * Kc, strideW=K * Kc, strideY=nout * K)
        self.sum_batches(part, S, nout, K, into, col_off, ld, True)

    def grad_input(self, dY, W, k_off=0, k=None):
        """dY [rows, nout] . W[:, k_off : k_off + k] -> [rows, k]   (W [nout, ldw] row-major)"""
        nout, ldw = W.shape
        k = ldw - k_off if k is None else k
        Wt = self.zeros(k, _pad4(nout)) if nout % 4 else self.empty(k, nout)
        self.transpose_raw(W, k_off, ldw, 0, Wt, Wt.stride(0), 0, 1, nout, k, True)
        rows = dY.shape[0]
        out = self.empty(rows, k)
        # K of this GEMM = nout; a dY whose row length is not a multiple of 4 goes through the fp32 kernel (og_linear_auto_fwd decides)
        self.gemm(dY, dY.stride(0), nout, Wt, Wt.stride(0), rows, k, out, k)
        return out
