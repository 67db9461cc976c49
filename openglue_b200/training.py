"""Training-mode forward AND backward of the matching core (SURVEY.md section 8, row f1): what ``SuperGlue.forward`` and
torch autograd compute for the reference inside ``MatchingTrainingModule.training_step`` (reference
models/matching_module.py:71-105) - BatchNorm with batch statistics (models/utils.py:48-58: Conv1d -> ReLU -> BatchNorm1d),
running-statistics updates, and the gradient of every parameter (and of the local descriptors).

Nothing here is differentiated by torch: :class:`TrainStep` records the activations of the forward pass and runs the backward
pass as an explicit schedule of the library's kernels (``include/openglue_b200.h``: the wgmma 3xTF32 / fp32 GEMMs for
``dX = dY W`` and ``dW = dY^T X``, the fused attention kernel forward, the materialised-softmax attention gradient, the
Sinkhorn backward pass, batch-norm / bias / mix reductions).  torch only owns the buffers and routes the resulting gradients
to the ``nn.Parameter`` objects (``_TrainFunction``).  There is no CPU path.

Layout: every activation is row-major ``[rows, channels]`` with ``rows = batch x keypoints`` of ONE image - the reference's
``[B, C, N]`` tensors transposed; BatchNorm statistics therefore run over the rows of one call, exactly the reference's
per-call ``(B, N)`` statistics (attention_gnn.py:58-77 calls the shared module once per image).

Padded batches (``num_keypoints0`` / ``num_keypoints1`` in ``data``, as for inference): pair b owns rows [0, n_b) / [0, m_b) of
the capacities N, M.  Attention, Sinkhorn and the loss run on each pair alone; BatchNorm pools the real rows of every pair in
the call (mean and biased variance over sum_b n_b rows).  Local descriptors are read through a copy with the padding zeroed, so
the padding's contents never reach a result, and every gradient at a padding row is 0.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

from . import _cabi, _graphs
from ._ops import _Ops, _pad4  # noqa: F401  (tests build their torch double of the kernels on _Ops' composite helpers)
from .features import (_check_image_pair, _frontend_storage, _image_pair_inputs, get_laf_to_sideinfo_converter, padded_capacity,
                       weights_key)
from .superglue import _MATCHER_KEYS, _matcher_inputs, is_padded, padded_inputs

__all__ = ['TrainStep', 'train_forward', 'GraphedTrainStep', 'ImagePairTrainStep']


class _BN:
    """One BatchNorm1d call site: parameters, running buffers and what the backward pass needs."""

    def __init__(self, mod: torch.nn.BatchNorm1d, lens: Optional[torch.Tensor] = None, skip: Optional[torch.Tensor] = None):
        self.mod = mod
        self.pk = {} if lens is None else {'lens': lens}           # padded batch: statistics over the real rows of every pair
        self.skip = skip                                           # device flag: a skipped step moves no running buffer

    def forward(self, ops: _Ops, a: torch.Tensor) -> torch.Tensor:
        m = self.mod
        self.a = a
        if m.momentum is None:
            raise NotImplementedError('BatchNorm1d(momentum=None) (cumulative average) is not built')
        track = m.track_running_stats and m.running_mean is not None
        if self.skip is not None:                                  # num_batches_tracked += 1 - skip on the device
            y, self.mean, self.invstd = ops.bn_fwd(a, m.weight, m.bias, m.eps, m.momentum, m.running_mean if track else None,
                                                   m.running_var if track else None, skip=self.skip,
                                                   num_batches_tracked=m.num_batches_tracked if track else None, **self.pk)
            return y
        y, self.mean, self.invstd = ops.bn_fwd(a, m.weight, m.bias, m.eps, m.momentum, m.running_mean if track else None,
                                               m.running_var if track else None, **self.pk)
        if track:
            m.num_batches_tracked += 1
        return y

    def backward(self, ops: _Ops, dy: torch.Tensor):
        return ops.bn_bwd(dy, self.a, self.mod.weight, self.mean, self.invstd, **self.pk)


class TrainStep:
    """One training-mode forward pass of ``model`` (an ``openglue_b200.SuperGlue`` in ``train()`` mode) with everything its
    backward pass needs.  ``forward()`` -> (scores [B,N+1,M+1], ctx0 [B,d,N], ctx1 [B,d,M]); ``backward(dscores, dctx0, dctx1)`` ->
    ``{parameter name: gradient}`` (+ ``'local_descriptors0/1'``).

    A padded batch (``num_keypoints0`` / ``num_keypoints1``, per-pair ``image0_size`` / ``image1_size`` optional, validated by
    :func:`~openglue_b200.superglue.padded_inputs`) gives each pair's outputs on its own block: ``scores[b, :n_b+1, :m_b+1]``
    (dustbins at n_b, m_b) and ``-inf`` elsewhere, context descriptors 0 past the lengths.  ``backward`` reads ``dscores`` on
    those blocks and ``dctx`` on the real columns only; the local-descriptor gradients are 0 on the padding rows.

    ``skip`` (device int32 [] flag, as ``og_train_guard`` writes it): the BatchNorm running statistics and ``num_batches_tracked``
    move only when it reads 0; the outputs are computed either way."""

    def __init__(self, model, data: dict, ops=None, skip: Optional[torch.Tensor] = None):
        model._check_head_dim()                         # before the forward pass moves any BatchNorm running buffer
        self.model = model
        cfg = model.config
        self.d = cfg['descriptor_dim']
        self.H = cfg['attention_gnn']['num_heads']
        self.use_offset = bool(cfg['attention_gnn'].get('use_offset', False))
        self.residual = bool(model.residual)
        self.no_desc = bool(cfg.get('no_descriptors', False))
        self.iters, self.reg = int(cfg['otp']['num_iters']), float(cfg['otp']['reg'])
        self.S = cfg['positional_encoding'].get('side_info_size', 1)
        k0 = data['keypoints0']
        self.dev = k0.device
        if ops is None:
            if self.dev.type != 'cuda':
                raise RuntimeError('openglue_b200 training needs CUDA tensors (sm_90a); there is no CPU path')
            for p in model.parameters():
                if p.device != self.dev or p.dtype != torch.float32:
                    raise RuntimeError('openglue_b200 training needs float32 parameters on the device of the data')
            prec = model._precision()
            ops = _Ops(self.dev, _cabi.OG_PREC_FP32 if prec == _cabi.OG_PREC_FP32 else _cabi.OG_PREC_TF32X3)
        self.ops = ops                                  # (tests inject a torch double of the kernels to check this schedule on the CPU)
        self.skip = skip
        f = lambda t, last: self._prep(t, last)
        self.kpts = [f(data['keypoints0'], 2), f(data['keypoints1'], 2)]
        self.side = [f(data['side_info0'], self.S), f(data['side_info1'], self.S)]
        self.ldesc = [f(data['local_descriptors0'], self.d), f(data['local_descriptors1'], self.d)]
        self.B = self.kpts[0].shape[0]
        self.N = [self.kpts[0].shape[1], self.kpts[1].shape[1]]
        if min(self.N) == 0:
            raise ValueError('empty keypoint set')
        self.padded = is_padded(data)
        self.lens = None
        if self.padded:
            extra = padded_inputs(data, self.B, self.N[0], self.N[1])
            lh = [extra['num_keypoints0'], extra['num_keypoints1']]
            for i, t in enumerate(lh):
                if t.device.type == 'cpu' and int(t.sum()) < 2:
                    # what BatchNorm1d raises for one value per channel: the statistics of a call pool the real rows
                    raise ValueError(f'Expected more than 1 value per channel when training: num_keypoints{i} sums to 1')
            self.lens = torch.cat([t.to(self.dev) for t in lh]).contiguous()          # [2B]: n_0 .. n_{B-1}, m_0 .. m_{B-1}
            self.pair_wh = torch.cat([extra['image0_size'].to(self.dev), extra['image1_size'].to(self.dev)], 1).contiguous()   # [B, 4]
            self.wh = [(0.0, 0.0), (0.0, 0.0)]
        else:
            self.wh = [model._image_wh(data, 0), model._image_wh(data, 1)]
        self.grads: Dict[str, torch.Tensor] = {}

    def _len(self, i):
        """image i's per-pair lengths (device int32 [B]), or None for a uniform batch"""
        return None if self.lens is None else self.lens[i * self.B:(i + 1) * self.B]

    def _lk(self):
        return {} if self.lens is None else {'lens': self.lens}

    @staticmethod
    def _prep(t, last):
        t = t.detach()
        if t.dtype != torch.float32:
            t = t.float()
        if t.shape[-1] != last:
            raise ValueError(f'expected last dimension {last}, got {tuple(t.shape)}')
        return t.contiguous()

    # ------------------------------------------------------------------ helpers
    def _device_ctx(self):
        import contextlib
        return torch.cuda.device(self.dev) if self.dev.type == 'cuda' else contextlib.nullcontext()

    @staticmethod
    def _w2(conv):
        return conv.weight.view(conv.weight.shape[0], conv.weight.shape[1])

    def _acc(self, name: str, g: torch.Tensor):
        """grads[name] += g (parameters shared by both images / both cross directions)"""
        if name in self.grads:
            self.ops.axpby(self.grads[name], g, 1.0, 1.0, out=self.grads[name])
        else:
            self.grads[name] = g

    def _acc_weight(self, name: str, conv, dY, X, X2=None):
        """d conv.weight (+)= dY^T [X | X2], d conv.bias (+)= colsum dY"""
        ops = self.ops
        wname, bname = name + '.weight', name + '.bias'
        if wname not in self.grads:
            self.grads[wname] = ops.zeros(conv.weight.shape[0], conv.weight.shape[1])
        ops.grad_weight(dY, X, self.grads[wname])
        if X2 is not None:
            ops.grad_weight(dY, X2, self.grads[wname], col_off=X.shape[1])
        self._acc(bname, ops.colsum(dY))

    # ------------------------------------------------------------------ forward
    def forward(self):
        ops, model, B, d = self.ops, self.model, self.B, self.d
        with self._device_ctx():
            enc = model.positional_encoding.encoder
            nl = (len(enc) + 2) // 3                                   # Conv (ReLU BN Conv)*
            self.kenc = []                                             # per image: list of (input, _BN) per hidden layer + last input
            x = []
            if self.padded:                                            # the residuals read the descriptors with the padding zeroed
                self.ldesc = [ops.mask_rows(self.ldesc[i].view(B * self.N[i], d), self._len(i)).view(B, self.N[i], d) for i in range(2)]
            for i in range(2):
                rows = B * self.N[i]
                if self.padded:
                    h = ops.kenc_input(self.kpts[i], self.side[i], rows, self.S, 0.0, 0.0, lens=self._len(i), pair_wh=self.pair_wh[:, 2 * i:])
                else:
                    h = ops.kenc_input(self.kpts[i], self.side[i], rows, self.S, self.wh[i][0], self.wh[i][1])
                rec = []
                for j in range(nl - 1):
                    conv, bn = enc[3 * j], _BN(enc[3 * j + 2], self._len(i), self.skip)
                    a = ops.linear(h, self._w2(conv), conv.bias)
                    rec.append((h, bn))
                    h = bn.forward(ops, a)
                conv = enc[3 * (nl - 1)]
                xi = ops.linear(h, self._w2(conv), conv.bias, R=None if self.no_desc else self.ldesc[i].view(rows, d))
                rec.append((h, None))
                self.kenc.append(rec)
                x.append(xi)
            self.calls = []                                            # message-passing calls in execution order
            for l, layer in enumerate(model.attention_gnn.layers):
                mod = layer.module
                name = f'attention_gnn.layers.{l}.module'
                if l % 2 == 0:                                         # self (attention_gnn.py:58-61)
                    x[0] = self._prop(name, mod, x[0], x[0], 0, 0)
                    x[1] = self._prop(name, mod, x[1], x[1], 1, 1)
                else:                                                  # cross, sequential (attention_gnn.py:74-77)
                    x[0] = self._prop(name, mod, x[0], x[1], 0, 1)
                    x[1] = self._prop(name, mod, x[1], x[0], 1, 0)
            self.x_final = x
            proj = model.linear_proj
            self.g = [ops.linear(x[i], self._w2(proj), proj.bias) for i in range(2)]
            if self.residual:
                self.mix = model.mix_coefs.detach().reshape(d)
                self.m = [ops.mix_fwd(self.g[i], self.ldesc[i].view(B * self.N[i], d), self.mix) for i in range(2)]
            else:
                self.m = self.g
            if self.padded:                                            # context descriptors are 0 past the lengths
                self.m = [ops.mask_rows(self.m[i], self._len(i)) for i in range(2)]
            n, m_ = self.N
            # context descriptors in the reference's [B, d, N] layout; their zero-padded copies are the transposed operands of the backward pass
            self.mT = [ops.transpose(self.m[i], batch=B, rows=self.N[i], cols=d) for i in range(2)]          # [B, d, pad4(N)]
            ctx = [self.mT[i][:, :, :self.N[i]].contiguous() if self.mT[i].shape[2] != self.N[i] else self.mT[i] for i in range(2)]
            lds = _pad4(m_)
            self.Sp = ops.zeros(B, n, lds)
            ops.gemm(self.m[0], d, d, self.m[1], d, n, m_, self.Sp, lds, alpha=d ** -0.5, batch=B, strideA=n * d, strideW=m_ * d, strideY=n * lds)
            self.dust = model.dustbin_score.detach().reshape(1).contiguous()
            scores, self.hist = ops.sinkhorn_fwd(self.Sp, self.dust, B, n, m_, self.iters, self.reg, **self._lk())
        return scores, ctx[0], ctx[1]

    def _prop(self, name, mod, xq, xkv, iq, ikv):
        """ResidualAttentionMessagePropagation.forward (attention_gnn.py:43-55) on row-major activations."""
        ops, d, H, B = self.ops, self.d, self.H, self.B
        nq, nk = self.N[iq], self.N[ikv]
        mha = mod.mha
        q = ops.linear(xq, self._w2(mha.in_proj_q), mha.in_proj_q.bias)
        k = ops.linear(xkv, self._w2(mha.in_proj_k), mha.in_proj_k.bias)
        v = ops.linear(xkv, self._w2(mha.in_proj_v), mha.in_proj_v.bias)
        kl = {} if self.lens is None else {'klen': self._len(ikv)}
        o = ops.attention(q, k, v, B, nq, nk, H, d // H, **kl)
        msg = ops.linear(o, self._w2(mha.out_proj), mha.out_proj.bias)
        c1 = ops.axpby(xq, msg, 1.0, -1.0) if self.use_offset else xq
        fc = mod.fc
        a = ops.linear(c1, self._w2(fc[0]), fc[0].bias, A2=msg)
        bn = _BN(fc[2], self._len(iq), self.skip)
        hbn = bn.forward(ops, a)
        out = ops.linear(hbn, self._w2(fc[3]), fc[3].bias, R=xq)
        self.calls.append(dict(name=name, mod=mod, xq=xq, xkv=xkv, iq=iq, ikv=ikv, q=q, k=k, v=v, o=o, msg=msg, c1=c1, bn=bn, hbn=hbn, **kl))
        return out

    # ------------------------------------------------------------------ backward
    def backward(self, dscores: Optional[torch.Tensor], dctx0: Optional[torch.Tensor] = None, dctx1: Optional[torch.Tensor] = None
                 ) -> Dict[str, torch.Tensor]:
        ops, model, B, d = self.ops, self.model, self.B, self.d
        n, m_ = self.N
        self.grads = {}
        with self._device_ctx():
            dm = [ops.zeros(B * n, d), ops.zeros(B * m_, d)]
            if dscores is not None:
                G = dscores.detach().float().contiguous()
                dZ, dd = ops.sinkhorn_bwd(self.Sp, self.dust, self.hist, G, B, n, m_, self.iters, self.reg, **self._lk())
                self.grads['dustbin_score'] = dd.reshape(model.dustbin_score.shape)
                # S = m0 m1^T d^-0.5:  dm0 = dS m1 d^-0.5,  dm1 = dS^T m0 d^-0.5   (superglue.py:64, 80-85)
                mp, np_ = _pad4(m_), _pad4(n)
                dS = ops.zeros(B, n, mp)
                ops.transpose_raw(dZ, 0, m_ + 1, (n + 1) * (m_ + 1), dS, mp, n * mp, B, n, m_, False)
                dSt = ops.zeros(B, m_, np_)
                ops.transpose_raw(dZ, 0, m_ + 1, (n + 1) * (m_ + 1), dSt, np_, m_ * np_, B, n, m_, True)
                sc = d ** -0.5
                ops.gemm(dS, mp, mp, self.mT[1], mp, n, d, dm[0], d, alpha=sc, batch=B, strideA=n * mp, strideW=d * mp, strideY=n * d)
                ops.gemm(dSt, np_, np_, self.mT[0], np_, m_, d, dm[1], d, alpha=sc, batch=B, strideA=m_ * np_, strideW=d * np_, strideY=m_ * d)
            for i, dctx in enumerate((dctx0, dctx1)):
                if dctx is not None:                                    # gradient arriving at the [B, d, N] context descriptors
                    t = ops.transpose(dctx.detach().float().contiguous(), batch=B, rows=d, cols=self.N[i], pad=False)     # -> [B, N, d]
                    ops.axpby(dm[i], t.view(B * self.N[i], d), 1.0, 1.0, out=dm[i])
            if self.padded:     # backward of the forward's mask: drops the dustbin gradients at n_b, m_b and any dctx past the lengths
                dm = [ops.mask_rows(dm[i], self._len(i)) for i in range(2)]
            dl = [None, None]
            if self.residual:
                dg = []
                csum = None
                for i in range(2):
                    rows = B * self.N[i]
                    gi, li = ops.mix_bwd(dm[i], self.mix)
                    dg.append(gi)
                    dl[i] = li
                    c = ops.colsum(dm[i], self.g[i], self.ldesc[i].view(rows, d))
                    csum = c if csum is None else ops.axpby(csum, c, 1.0, 1.0)
                self.grads['mix_coefs'] = ops.mix_param_grad(csum, self.mix).reshape(model.mix_coefs.shape)
            else:
                dg = dm
            proj = model.linear_proj
            dx = []
            for i in range(2):
                self._acc_weight('linear_proj', proj, dg[i], self.x_final[i])
                dx.append(ops.grad_input(dg[i], self._w2(proj)))
            # message passing, in reverse execution order
            for call in reversed(self.calls):
                iq, ikv = call['iq'], call['ikv']
                dxq, dxkv = self._prop_bwd(call, dx[iq])
                if iq == ikv:
                    dx[iq] = ops.axpby(dxq, dxkv, 1.0, 1.0, out=dxq)
                else:
                    dx[iq] = dxq
                    dx[ikv] = ops.axpby(dx[ikv], dxkv, 1.0, 1.0, out=dxkv)
            # keypoint encoder (+ the descriptors that were added to its output, superglue.py:52-55)
            enc = model.positional_encoding.encoder
            for i in range(2):
                rec = self.kenc[i]
                if not self.no_desc:
                    dl[i] = dx[i] if dl[i] is None else ops.axpby(dl[i], dx[i], 1.0, 1.0, out=dl[i])
                g = dx[i]
                for j in range(len(rec) - 1, -1, -1):
                    h, bn = rec[j]
                    conv = enc[3 * j]
                    self._acc_weight(f'positional_encoding.encoder.{3 * j}', conv, g, h)
                    if j == 0:
                        break                                           # no gradient with respect to the keypoints / side info
                    gh = ops.grad_input(g, self._w2(conv))
                    g, dgam, dbet = rec[j - 1][1].backward(ops, gh)
                    self._acc(f'positional_encoding.encoder.{3 * (j - 1) + 2}.weight', dgam)
                    self._acc(f'positional_encoding.encoder.{3 * (j - 1) + 2}.bias', dbet)
            for i in range(2):
                if dl[i] is not None:
                    self.grads[f'local_descriptors{i}'] = dl[i].view(B, self.N[i], d)
        return self.grads

    def _prop_bwd(self, call, dout):
        ops, d = self.ops, self.d
        mod, name = call['mod'], call['name']
        fc, mha = mod.fc, mod.mha
        xq, xkv = call['xq'], call['xkv']
        # out = xq + hbn W2^T + b2
        self._acc_weight(name + '.fc.3', fc[3], dout, call['hbn'])
        dhbn = ops.grad_input(dout, self._w2(fc[3]))
        da, dgam, dbet = call['bn'].backward(ops, dhbn)
        self._acc(name + '.fc.2.weight', dgam)
        self._acc(name + '.fc.2.bias', dbet)
        # a = [c1 | msg] W1^T + b1
        self._acc_weight(name + '.fc.0', fc[0], da, call['c1'], call['msg'])
        W1 = self._w2(fc[0])
        dc1 = ops.grad_input(da, W1, 0, d)
        dmsg = ops.grad_input(da, W1, d, d)
        if self.use_offset:                                             # c1 = xq - msg
            dmsg = ops.axpby(dmsg, dc1, 1.0, -1.0, out=dmsg)
        dxq = ops.axpby(dout, dc1, 1.0, 1.0, out=dc1)
        # msg = o Wo^T + bo
        self._acc_weight(name + '.mha.out_proj', mha.out_proj, dmsg, call['o'])
        do = ops.grad_input(dmsg, self._w2(mha.out_proj))
        dq, dk, dv = self._attention_bwd(call, do)
        self._acc_weight(name + '.mha.in_proj_q', mha.in_proj_q, dq, xq)
        self._acc_weight(name + '.mha.in_proj_k', mha.in_proj_k, dk, xkv)
        self._acc_weight(name + '.mha.in_proj_v', mha.in_proj_v, dv, xkv)
        ops.axpby(dxq, ops.grad_input(dq, self._w2(mha.in_proj_q)), 1.0, 1.0, out=dxq)
        dxkv = ops.grad_input(dk, self._w2(mha.in_proj_k))
        ops.axpby(dxkv, ops.grad_input(dv, self._w2(mha.in_proj_v)), 1.0, 1.0, out=dxkv)
        return dxq, dxkv

    def _attention_bwd(self, call, do):
        """Gradient of softmax_attention (models/superglue/attention.py:8-19) per head, with the probabilities re-materialised:
        P = softmax(q k^T s);  dV = P^T dO;  dP = dO V^T;  dS = s P (dP - rowsum(P dP));  dQ = dS K;  dK = dS^T Q."""
        ops, d, H, B = self.ops, self.d, self.H, self.B
        dh = d // H
        nq, nk = self.N[call['iq']], self.N[call['ikv']]
        q, k, v = call['q'], call['k'], call['v']
        nqp, nkp = _pad4(nq), _pad4(nk)
        scale = dh ** -0.5
        qT = ops.transpose(q, batch=B, rows=nq, cols=d)                 # [B, d, nqp]
        kT = ops.transpose(k, batch=B, rows=nk, cols=d)                 # [B, d, nkp]
        doT = ops.transpose(do, batch=B, rows=nq, cols=d)               # [B, d, nqp]
        dq, dk, dv = ops.empty(B * nq, d), ops.empty(B * nk, d), ops.empty(B * nk, d)
        P, dP = ops.zeros(B, nq, nkp), ops.zeros(B, nq, nkp)
        PT, dST = ops.zeros(B, nk, nqp), ops.zeros(B, nk, nqp)
        kl = {'klen': call['klen']} if 'klen' in call else {}   # P = 0 past each sequence's keys: dQ, dK, dV vanish there
        for h in range(H):
            c = h * dh
            ops.gemm(q, d, dh, k, d, nq, nk, P, nkp, a_off=c, w_off=c, alpha=scale, batch=B, strideA=nq * d, strideW=nk * d, strideY=nq * nkp)
            ops.softmax_rows(P, nkp, B * nq, nk, **kl)
            ops.gemm(do, d, dh, v, d, nq, nk, dP, nkp, a_off=c, w_off=c, batch=B, strideA=nq * d, strideW=nk * d, strideY=nq * nkp)
            ops.transpose_raw(P, 0, nkp, nq * nkp, PT, nqp, nk * nqp, B, nq, nk, True)
            ops.gemm(PT, nqp, nqp, doT, nqp, nk, dh, dv, d, w_off=c * nqp, y_off=c, batch=B, strideA=nk * nqp, strideW=d * nqp, strideY=nk * d)
            ops.softmax_bwd_rows(P, dP, nkp, B * nq, nk, scale, **kl)
            ops.gemm(dP, nkp, nkp, kT, nkp, nq, dh, dq, d, w_off=c * nkp, y_off=c, batch=B, strideA=nq * nkp, strideW=d * nkp, strideY=nq * d)
            ops.transpose_raw(dP, 0, nkp, nq * nkp, dST, nqp, nk * nqp, B, nq, nk, True)
            ops.gemm(dST, nqp, nqp, qT, nqp, nk, dh, dk, d, w_off=c * nqp, y_off=c, batch=B, strideA=nk * nqp, strideW=d * nqp, strideY=nk * d)
        return dq, dk, dv


class _TrainFunction(torch.autograd.Function):
    """Routes the explicit backward pass of :class:`TrainStep` into torch's autograd graph: inputs are the local descriptors and
    every parameter of the model, outputs the three tensors of the reference's ``forward``."""

    @staticmethod
    def forward(ctx, model, data, names, ld0, ld1, *params):
        ctx.set_materialize_grads(False)
        step = TrainStep(model, data)
        scores, c0, c1 = step.forward()
        ctx.step, ctx.names = step, names
        ctx.shapes = [p.shape for p in params]
        ctx.ld_dtypes = (ld0.dtype, ld1.dtype)
        return scores, c0, c1

    @staticmethod
    def backward(ctx, dscores, dc0, dc1):
        g = ctx.step.backward(dscores, dc0, dc1)
        ctx.step = None                                                 # the activations are released with the step
        need = ctx.needs_input_grad
        gl = [g.get('local_descriptors0'), g.get('local_descriptors1')]
        out: List[Optional[torch.Tensor]] = [None, None, None]
        for i in range(2):
            out.append(gl[i].to(ctx.ld_dtypes[i]) if need[3 + i] and gl[i] is not None else None)
        for j, nme in enumerate(ctx.names):
            gj = g.get(nme) if need[5 + j] else None
            out.append(None if gj is None else gj.reshape(ctx.shapes[j]))
        return tuple(out)


def train_forward(model, data: dict) -> Dict[str, torch.Tensor]:
    """``SuperGlue.forward`` in training mode: same outputs as the reference module (superglue.py:66-70), differentiable."""
    names, params = zip(*[(n, p) for n, p in model.named_parameters()])
    scores, c0, c1 = _TrainFunction.apply(model, data, names, data['local_descriptors0'], data['local_descriptors1'], *params)
    return {'context_descriptors0': c0, 'context_descriptors1': c1, 'scores': scores}


def _bind_grads(params, grads, dev):
    """p.grad = views of one buffer (16-byte aligned slices) -> (buffer, views), passed back in as ``grads``: a skipped step zeroes
    every gradient in one launch, and a captured graph's gradients stay where ``p.grad`` points after ``zero_grad()``"""
    if grads is None or grads[0].device != dev or any(p.device != dev for _, p in params):
        sizes = [(p.numel() + 3) // 4 * 4 for _, p in params]
        flat = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
        views, off = [], 0
        for (_, p), n in zip(params, sizes):
            views.append(flat[off:off + p.numel()].view(p.shape))
            off += n
        grads = (flat, views)
    for (_, p), g in zip(params, grads[1]):
        if p.grad is not g:
            p.grad = g
    return grads


def _pointers(model, params) -> tuple:
    """The storage of the parameters, buffers and gradients a captured step reads; not their versions, which every step bumps"""
    return (tuple(t.data_ptr() for t in list(model.parameters()) + list(model.buffers())),
            tuple(None if p.grad is None else p.grad.data_ptr() for _, p in params))


class _WarmupGuard:
    """The warm-up run before a capture is not a training step: the BatchNorm buffers and, with an optimiser, the parameters
    and its state are put back after it.  ``guarded``: the replayed optimiser step may have been skipped on the device."""

    def __init__(self, model, optimizer, guarded: bool):
        self.model, self.opt, self.guarded = model, optimizer, guarded

    def save(self) -> None:
        self._saved = [b.clone() for b in self.model.buffers()], None if self.opt is None else self.opt._snapshot()

    def restore(self) -> None:
        for b, s in zip(self.model.buffers(), self._saved[0]):
            b.copy_(s)
        if self.opt is not None:
            self.opt._restore(self._saved[1])

    def captured(self):
        snap, self._saved = self._saved[1], None
        if self.opt is not None:                                         # the capture ran nothing: no parameter has new state
            self.opt._stepped = list(snap[-1])
            return self.opt._last_idx

    def replayed(self, idx) -> None:
        if self.opt is not None:                                         # the kernels wrote the parameters through raw pointers
            self.opt._stepped_now(idx, guarded=self.guarded)


class GraphedTrainStep:
    """The whole training step of one batch shape - train-mode forward, ``criterion``, backward, gradients into ``param.grad`` and,
    with ``optimizer`` (a :class:`~openglue_b200.optim.ClippedAdam`), the optimiser step - captured ONCE into a CUDA graph and
    replayed: the eager step issues ~5000 kernel launches from Python and is launch-rate-bound, the replay costs the kernels' own
    time.  Labels (``generate_gt_matches``) stay outside::

        opt = ClippedAdam.from_config(model, config['train'])  # clip_grad_norm_ -> Adam -> StepLR, on the device
        step = GraphedTrainStep(model, data, y_true, optimizer=opt)   # model.train(); captures on the first batch
        for data, y_true in loader:                           # same shapes
            loss = step(data, y_true)                         # {'loss', 'metric_loss'}: one replay is the whole iteration

    Without ``optimizer`` the graph ends with the gradients in ``p.grad`` and any optimiser runs after the replay (in-place
    updates keep the captured parameter addresses valid).  The capture's warm-up run is not a training step: the BatchNorm
    buffers, and with ``optimizer`` the parameters and its state, are restored after it, so the first replay is step 1.

    The graph reads the parameters and BatchNorm buffers in place (so optimiser steps and running statistics carry over) and the
    inputs from static copies.  Every call must keep the captured shapes and, for a uniform batch, the captured image sizes, which
    the graph bakes in: another shape or size raises ``ValueError``.  ``p.grad`` is bound again on every call (``zero_grad()``
    may have set it to None), and the step is captured again when a parameter, buffer or gradient is re-allocated (``p.data =
    ...``; ``load_state_dict`` keeps storage).  Results are bit-identical to the eager step (same kernels, same order).

    ``margin`` / ``metric_weight`` (the reference's ``train.margin`` / ``train.metric_weight``, matching_module.py:101-105): with a
    margin the graph also computes ``metric_loss`` on the context descriptors (``og_metric_loss_fwd``) and backpropagates
    ``nll_weight * loss + metric_weight * metric_loss``, as ``criterion(..., margin=)`` does in the eager step; ``margin=None``
    captures the margin-free step exactly as before.

    Padded batches (``num_keypoints0`` / ``num_keypoints1`` in ``data`` and ``y_true``, per-pair ``image0_size`` /
    ``image1_size`` optional): the lengths and sizes live in static device buffers like the other inputs, so one capture per
    capacity (B, N, M) replays every set of lengths; the step is :class:`TrainStep`'s padded step with :func:`criterion`'s
    per-pair loss.  ``margin`` is not built for padded batches."""

    def __init__(self, model, data: dict, y_true: dict, nll_weight: float = 1.0, optimizer=None, margin: Optional[float] = None,
                 metric_weight: float = 0.0):
        from .losses import _metric_run
        from .losses import _run as criterion_run
        from .optim import ClippedAdam
        if not model.training:
            raise RuntimeError('GraphedTrainStep captures the training-mode step: call model.train() first')
        dev = data['keypoints0'].device
        if dev.type != 'cuda':
            raise RuntimeError('openglue_b200 training needs CUDA tensors (sm_90a); there is no CPU path')
        if optimizer is not None and not isinstance(optimizer, ClippedAdam):
            raise TypeError('GraphedTrainStep captures the optimiser step of openglue_b200.ClippedAdam only '
                            f'(got {type(optimizer).__name__}): run other optimisers after the replay')
        self.padded = is_padded(data)
        if self.padded and margin is not None:
            raise NotImplementedError('GraphedTrainStep(margin=...) on a padded batch (num_keypoints0 / num_keypoints1) is not built')
        self.model, self.dev, self.optimizer = model, dev, optimizer
        self.params = list(model.named_parameters())
        self._guard = _WarmupGuard(model, optimizer, guarded=False)
        inputs, self._key, consts = self._inputs(data, y_true)

        def chain(s):                         # s: the static inputs; a padded batch's labels read its lengths there too
            step = TrainStep(model, {**s, **consts})
            scores, c0, c1 = step.forward()
            loss, dscores = criterion_run(s, {'scores': scores}, True, float(nll_weight))
            if margin is None:
                grads = step.backward(dscores)
            else:                                                        # metric_loss into loss[1]; its gradient scaled as autograd
                _, _, dc0, dc1 = _metric_run(s['gt_matches0'], s['gt_matches1'], c0, c1, float(margin), True, 1.0, out=loss[1:])
                for dc in (dc0, dc1):                                    # scales the eager step's unit gradients (one rounding)
                    step.ops.axpby(dc, None, float(metric_weight), 0.0, out=dc)
                grads = step.backward(dscores, dc0, dc1)
            for name, p in self.params:
                p.grad.copy_(grads[name].reshape(p.shape))
            if optimizer is not None:
                optimizer.step()
            return loss
        self._chain = chain
        self._grads = _bind_grads(self.params, None, dev)
        with torch.cuda.device(dev):
            self._graphs = {self._key: _graphs.capture(inputs, chain, dev, f32=True, version=self._version, guard=self._guard)}

    def _inputs(self, data: dict, y_true: dict):
        """-> (static inputs, key, key constants) of a batch"""
        tensors, consts = _matcher_inputs(data)
        # labels as int64, whatever dtype they come in: og_metric_loss_fwd reads the static buffer as int64
        tensors.update({k: y_true[k].to(torch.int64) for k in ('gt_matches0', 'gt_matches1')})
        return tensors, (tuple(tuple(data[k].shape) for k in _MATCHER_KEYS), tuple(consts.values())), consts

    def _version(self) -> tuple:
        return _pointers(self.model, self.params)

    def __call__(self, data: dict, y_true: dict) -> Dict[str, torch.Tensor]:
        if is_padded(data) != self.padded:
            raise ValueError('the batch must be padded (num_keypoints0 / num_keypoints1) exactly when the captured one was')
        inputs, key, _ = self._inputs(data, y_true)
        for k, shape, want in zip(_MATCHER_KEYS, key[0], self._key[0]):
            if shape != want:
                raise ValueError(f'{k}: shape {shape} differs from the captured {want}')
        if key[1] != self._key[1]:
            raise ValueError(f'image sizes (W, H) {key[1]} differ from the captured {self._key[1]}: a uniform batch bakes them into '
                             'the graph')
        self._grads = _bind_grads(self.params, self._grads, self.dev)
        with torch.cuda.device(self.dev):
            loss = _graphs.run(self._graphs, 1, self._key, self._version, inputs, self._chain, self.dev, f32=True, guard=self._guard)
        return {'loss': loss[0], 'metric_loss': loss[1]}


# transformation type -> {tensor key: shape with B, h, w filled in by _transformation}
_TF_KEYS = {'perspective': ('H',), '3d_reprojection': ('K0', 'K1', 'R', 'T', 'depth0', 'depth1')}


class ImagePairTrainStep:
    """The reference's ``training_step`` from images (models/matching_module.py:71-105 with features computed online, as
    ``train.py`` and ``pretrain_homography.py`` run it), replayed as one CUDA graph::

        opt = ClippedAdam.from_config(superglue, config['train'])
        step = ImagePairTrainStep(local_feature, superglue.train(), config, optimizer=opt)
        out = step(batch)                      # batch: 'image0' [B,1,H0,W0], 'image1' [B,1,H1,W1], 'transformation'
        out = step.pretrain(images_u8, offset) # homography pretraining: uint8 RGB [B,H,W,3] -> synthesized pairs -> the same step

    One call runs ``extract_padded`` on both images (K rows per image, ``capacity`` or the front-end's ``max_keypoints``),
    ``prepare_features_output``, the per-pair image sizes, ``gt_matches`` with the device counts, the padded :class:`TrainStep`
    forward, ``criterion``, the backward pass, the gradients into ``p.grad`` and, with ``optimizer`` (a
    :class:`~openglue_b200.optim.ClippedAdam`), its step.  Without an optimiser the call ends with the gradients in ``p.grad``.
    ``batch['transformation']`` is ``{'type': ['perspective'] * B, 'H' [B,3,3]}`` or ``{'type': ['3d_reprojection'] * B, 'K0',
    'K1', 'R' [B,3,3], 'T' [B,3], 'depth0' [B,h0,w0], 'depth1' [B,h1,w1]}`` (depth images, as MegaDepth's loader gives them).
    ``pretrain(images_u8, offset)`` draws each image's corner offsets with ``torch.randint`` on the default CUDA generator (new ones
    on every replay; ``torch.cuda.manual_seed`` reproduces them), synthesizes the pairs (``synthesize_homography_pairs``) and runs
    the same step.

    The reference skips a batch in which an image has no keypoint (``data is None``); a batch in which one side's real rows total
    fewer than 2 makes ``BatchNorm1d`` raise there.  Both are decided here on the device (``og_train_guard``): such a batch is
    skipped - parameters, BatchNorm buffers and optimiser state keep their bits, ``p.grad`` is 0, the loss is NaN and
    ``skipped`` is 1 - with no host synchronisation.

    Returns device tensors: ``loss``, ``metric_loss`` (0-dim), ``skipped`` (int32, 0-dim), ``num_keypoints0`` /
    ``num_keypoints1`` and ``overflow0`` / ``overflow1`` (int32 [B]: the front-end's flags, an image cut to K rows trains on its
    first K) and, from ``pretrain``, ``warp_offset`` (int32 [B,4,2]) - copies, or the graph's own buffers with ``borrow=True``
    (overwritten by the next call).

    ``use_cuda_graph=True`` captures one graph per (image shapes and dtypes, K, transformation type and tensor shapes, precision,
    device) after one eager warm-up run, which is not a training step: the BatchNorm buffers, the parameters and the optimiser
    state are restored after it.  A graph is captured again when a parameter, buffer or gradient of the matcher is reallocated
    or a weight of the front-end changes; at most ``max_graphs`` are kept.  ``use_cuda_graph=False`` runs the same chain
    eagerly, with the same results bit for bit.

    Not built: ``train.margin`` (the metric loss on padded batches), colour augmentation (``train.augmentations.name`` other
    than ``'none'``) and fine-tuning the front-end (``features.finetune``)."""

    _OUT_KEYS = ('loss', 'metric_loss', 'skipped', 'num_keypoints0', 'num_keypoints1', 'overflow0', 'overflow1')

    def __init__(self, local_feature: torch.nn.Module, superglue, config: dict, optimizer=None, capacity: Optional[int] = None,
                 use_cuda_graph: bool = True):
        from .optim import ClippedAdam
        from .superglue import SuperGlue
        if not isinstance(superglue, SuperGlue):
            raise TypeError('openglue_b200.ImagePairTrainStep trains an openglue_b200.SuperGlue')
        if not superglue.training:
            raise RuntimeError('ImagePairTrainStep runs the training-mode step: call superglue.train() first')
        if not callable(getattr(local_feature, 'extract_padded', None)):
            raise TypeError('openglue_b200.ImagePairTrainStep takes a front-end with extract_padded (OpenCVSIFT, SIFT, GFTTAffNetHardNet, '
                            'DoGOpenCVAffNetHardNet, SuperPointNet[Bn])')
        if (config.get('features') or {}).get('finetune', False):
            raise NotImplementedError('fine-tuning the front-end (features.finetune) is not built: openglue_b200 front-ends run in eval mode')
        train = config['train']
        if train.get('margin') is not None:
            raise NotImplementedError('criterion(margin=...) on a padded batch (num_keypoints0 / num_keypoints1) is not built')
        aug = (train.get('augmentations') or {}).get('name', 'none')
        if aug != 'none':
            raise NotImplementedError(f"train.augmentations.name = {aug!r}: colour augmentation is not built (only 'none')")
        if optimizer is not None and not isinstance(optimizer, ClippedAdam):
            raise TypeError('ImagePairTrainStep runs the optimiser step of openglue_b200.ClippedAdam only '
                            f'(got {type(optimizer).__name__}): pass optimizer=None and step other optimisers after the call')
        superglue._check_head_dim()
        sg_cfg = config['superglue']
        self.laf_converter = get_laf_to_sideinfo_converter(sg_cfg['laf_to_sideinfo_method'])
        side = superglue.config['positional_encoding'].get('side_info_size', 1)
        if side != 1 + self.laf_converter.side_info_dim:
            raise ValueError(f"side_info_size {side} of the matcher does not fit laf_to_sideinfo_method "
                             f"{sg_cfg['laf_to_sideinfo_method']!r} (1 + {self.laf_converter.side_info_dim} columns)")
        d = superglue.config['descriptor_dim']
        fd = getattr(local_feature, 'descriptor_dim', 128)                 # OpenCVSIFT: 128
        if fd != d:
            raise ValueError(f'the front-end describes keypoints in {fd} dimensions, the matcher takes {d}')
        self.log_response = bool(sg_cfg.get('log_transform_response', False))
        self.positive_threshold = float(train['gt_positive_threshold'])  # as in the reference, the labels do not depend on them
        self.negative_threshold = train.get('gt_negative_threshold')
        self.nll_weight = float(train.get('nll_weight', 1.0))
        self.metric_weight = float(train.get('metric_weight', 0.0))      # multiplies metric_loss = 0 (margin None)
        local_feature.eval()                                               # matching_module.py:77-78
        self.local_feature, self.superglue, self.optimizer = local_feature, superglue, optimizer
        self.capacity, self.use_cuda_graph = capacity, use_cuda_graph
        self.params = list(superglue.named_parameters())
        self._grads = None                                                 # one zero-padded buffer behind every p.grad
        self._guard = _WarmupGuard(superglue, optimizer, guarded=True)
        self._graphs: Dict[tuple, _graphs.Entry] = {}
        self.max_graphs = 4

    # ------------------------------------------------------------------ the chain
    def _chain(self, image0: torch.Tensor, image1: torch.Tensor, tf: dict, K: int) -> Dict[str, torch.Tensor]:
        from .gt_matches import gt_matches
        from .losses import _run as criterion_run
        dev = image0.device
        B = image0.shape[0]
        lib, st = _cabi.lib(), _cabi.stream(dev)
        data, feats = _image_pair_inputs(self.local_feature, self.laf_converter, self.log_response, image0, image1, K)
        out = {k: feats[k] for k in ('num_keypoints0', 'num_keypoints1', 'overflow0', 'overflow1')}
        lens = torch.cat([out['num_keypoints0'], out['num_keypoints1']])
        skip = torch.empty((), dtype=torch.int32, device=dev)
        _cabi.check(lib.og_train_guard(_cabi.ptr(lens), B, _cabi.ptr(skip), st), 'og_train_guard')
        gt0, gt1 = gt_matches(data['keypoints0'], data['keypoints1'], tf, lens)
        y_true = {'gt_matches0': gt0, 'gt_matches1': gt1, 'num_keypoints0': out['num_keypoints0'], 'num_keypoints1': out['num_keypoints1']}
        step = TrainStep(self.superglue, data, skip=skip)
        scores, _, _ = step.forward()
        loss, dscores = criterion_run(y_true, {'scores': scores}, True, self.nll_weight)
        grads = step.backward(dscores)
        for name, p in self.params:
            p.grad.copy_(grads[name].reshape(p.shape))
        flat = self._grads[0]
        if self.optimizer is None:                                         # loss = NaN and every p.grad = 0 when skipped
            _cabi.check(lib.og_train_skip_outputs(_cabi.ptr(skip), _cabi.ptr(loss), 2, _cabi.ptr(flat), flat.numel(), st), 'og_train_skip_outputs')
        else:                                                              # the guarded optimiser step zeroes the gradients
            _cabi.check(lib.og_train_skip_outputs(_cabi.ptr(skip), _cabi.ptr(loss), 2, None, 0, st), 'og_train_skip_outputs')
            self.optimizer.step(skip=skip)
        out.update(loss=loss[0], metric_loss=loss[1], skipped=skip)
        return out

    # ------------------------------------------------------------------ arguments
    def _K(self) -> int:
        return padded_capacity(self.local_feature.max_keypoints, self.capacity)

    def _check_model(self, dev) -> None:
        for _, p in self.params:
            if p.device != dev or p.dtype != torch.float32:
                raise RuntimeError('openglue_b200 training needs float32 parameters on the device of the images')
        if not self.superglue.training:
            raise RuntimeError('ImagePairTrainStep runs the training-mode step: call superglue.train() first')
        if self.optimizer is not None and self.optimizer.dev != dev:
            raise RuntimeError(f'the optimiser holds its state on {self.optimizer.dev}, the images are on {dev}')

    @staticmethod
    def _transformation(tf: dict, B: int) -> Tuple[str, Dict[str, torch.Tensor]]:
        """-> (type, {key: tensor}) of batch['transformation'], shapes checked (depth: images [B, h, w])"""
        kind = tf['type'][0] if isinstance(tf['type'], (list, tuple)) else tf['type']
        if kind not in _TF_KEYS:
            raise ValueError(f'Unknown transformation type {kind}.')
        want = {'H': (B, 3, 3), 'K0': (B, 3, 3), 'K1': (B, 3, 3), 'R': (B, 3, 3), 'T': (B, 3)}
        out = {}
        for k in _TF_KEYS[kind]:
            t = tf[k]
            if not torch.is_tensor(t):
                raise TypeError(f'transformation[{k!r}] must be a tensor')
            ok = tuple(t.shape) == want[k] if k in want else (t.dim() == 3 and t.shape[0] == B)
            if not ok:
                raise ValueError(f"transformation[{k!r}] has shape {tuple(t.shape)}, expected {want.get(k, f'[{B}, h, w]')}")
            out[k] = t
        return kind, out

    # ------------------------------------------------------------------ graphs
    def _versions(self) -> tuple:
        return _pointers(self.superglue, self.params), weights_key(self.local_feature)

    def _run(self, key: tuple, inputs: Dict[str, torch.Tensor], chain) -> Dict[str, torch.Tensor]:
        """Replay (capturing on first use) the graph of ``chain(static inputs)`` for ``key``; the inputs are copied into its
        static buffers.  Eager when use_cuda_graph is False."""
        dev = self.superglue.dustbin_score.device
        self._grads = _bind_grads(self.params, self._grads, dev)
        if not self.use_cuda_graph:
            return chain(inputs)
        return _graphs.run(self._graphs, self.max_graphs, key, self._versions, inputs, chain, dev, f32=True,
                           hold=lambda: _frontend_storage(self.local_feature), guard=self._guard)

    # ------------------------------------------------------------------ public
    def __call__(self, batch: dict, borrow: bool = False) -> Dict[str, torch.Tensor]:
        """One training step on ``batch`` (``image0``, ``image1``, ``transformation``).  ``borrow=True`` (CUDA-graph mode): the graph's
        own output buffers instead of copies."""
        image0, image1 = batch['image0'], batch['image1']
        _check_image_pair(image0, image1)
        B = image0.shape[0]
        kind, tf = self._transformation(batch['transformation'], B)
        K = self._K()
        if image0.device.type != 'cuda' or image1.device != image0.device:
            raise RuntimeError('openglue_b200.ImagePairTrainStep needs both images on one CUDA device (sm_90a); there is no CPU path')
        dev = image0.device
        self._check_model(dev)
        inputs = {'image0': image0, 'image1': image1, **tf}

        def chain(x):
            t = {'type': [kind] * B, **{k: x[k] for k in tf}}
            return self._chain(x['image0'], x['image1'], t, K)
        key = (tuple(image0.shape), tuple(image1.shape), image0.dtype, image1.dtype, K, kind,
               tuple((k, tuple(v.shape)) for k, v in tf.items()), self.superglue._precision(), str(dev))
        with torch.cuda.device(dev):
            out = self._run(key, inputs, chain)
        return out if borrow or not self.use_cuda_graph else {k: v.clone() for k, v in out.items()}

    def pretrain(self, images_u8: torch.Tensor, offset: int, borrow: bool = False) -> Dict[str, torch.Tensor]:
        """Homography pretraining (``pretrain_homography.py``): ``synthesize_homography_pairs(images_u8, offset)`` with offsets drawn
        on the device, then the step; the result also holds ``warp_offset`` [B, 4, 2]."""
        from .homography import _check_images, _pairs
        B, _, _, offset = _check_images(images_u8, offset)
        K = self._K()
        if images_u8.device.type != 'cuda':
            raise RuntimeError('openglue_b200: images_u8 must be a CUDA tensor (sm_90a); there is no CPU path')
        dev = images_u8.device
        self._check_model(dev)

        def chain(x):
            wo = torch.randint(-offset, offset, (B, 4, 2), device=dev, dtype=torch.int32)   # the default generator: graph-safe
            pairs = _pairs(x['images_u8'], offset, wo)
            out = self._chain(pairs['image0'], pairs['image1'], pairs['transformation'], K)
            out['warp_offset'] = wo
            return out
        key = ('pretrain', tuple(images_u8.shape), offset, K, self.superglue._precision(), str(dev))
        with torch.cuda.device(dev):
            out = self._run(key, {'images_u8': images_u8}, chain)
        return out if borrow or not self.use_cuda_graph else {k: v.clone() for k, v in out.items()}
