"""Training on padded batches without a GPU.

* The checks TrainStep and criterion run on a padded batch before any kernel.
* The CPU leg: ``TrainStep`` with per-pair lengths driven by the float64 torch double of the kernels (``_PaddedCpuOps``, the
  ``_CpuOps`` of tests/test_training.py with the lengths arguments), against
  - at B = 1 with capacity > length, the unmodified reference (oracle/_ref) differentiated by float64 autograd on the trimmed pair;
  - at B >= 3 with mixed lengths (one pair with n_b = 1), ``restated_reference``: the reference module with its BatchNorm pooling
    the real columns of every pair, its attention masked to each sequence's keys, its keypoint normalisation per pair and its
    Sinkhorn run pair by pair - itself checked against the plain reference at full lengths.
  Outputs, every parameter gradient, the local-descriptor gradients (0 on the padding) and the BatchNorm buffers are compared.
The GPU file (tests/test_padded_training.py) runs the same two comparisons on the device.
"""
import copy
import types

import pytest
import torch
import torch.nn.functional as F

from openglue_b200.losses import criterion
from openglue_b200.superglue import SuperGlue
from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
from openglue_b200.training import TrainStep
from test_training import _CpuOps
from test_training_reference import _reference_class, perturb_bn

OUTS = ('scores', 'context_descriptors0', 'context_descriptors1')


# ----------------------------------------------------------------------------------------------------- validation
def _data(n0=(10, 1, 4), n1=(7, 7, 1)):
    d = synthetic_pairs(3, 10, 7, 32, 1, seed=0)
    d['num_keypoints0'] = torch.tensor(n0)
    d['num_keypoints1'] = torch.tensor(n1)
    return d


def _model():
    return SuperGlue(default_config(descriptor_dim=32, num_stages=1)).train()


@pytest.mark.parametrize('key,value', [('num_keypoints0', [0, 1, 4]), ('num_keypoints0', [11, 1, 4]),
                                       ('num_keypoints1', [7, -1, 1]), ('num_keypoints1', [7, 8, 1])])
def test_lengths_outside_the_capacity_are_refused(key, value):
    d = _data()
    d[key] = torch.tensor(value)
    with pytest.raises(ValueError, match='capacity'):
        TrainStep(_model(), d, ops=_CpuOps())


def test_lengths_come_in_pairs():
    d = _data()
    del d['num_keypoints1']
    with pytest.raises(ValueError, match='both'):
        TrainStep(_model(), d, ops=_CpuOps())


def test_one_real_row_in_a_batchnorm_call_is_refused_as_batchnorm1d_does():
    d = synthetic_pairs(1, 10, 7, 32, 1, seed=0)
    d['num_keypoints0'], d['num_keypoints1'] = torch.tensor([1]), torch.tensor([5])
    with pytest.raises(ValueError, match='more than 1 value per channel'):
        TrainStep(_model(), d, ops=_CpuOps())
    with pytest.raises(ValueError, match='more than 1 value per channel'):
        torch.nn.BatchNorm1d(4).train()(torch.zeros(1, 4))


def test_margin_on_a_padded_batch_is_not_built():
    y = {'gt_matches0': torch.zeros(3, 10, dtype=torch.int64), 'gt_matches1': torch.zeros(3, 7, dtype=torch.int64),
         'num_keypoints0': torch.tensor([10, 1, 4]), 'num_keypoints1': torch.tensor([7, 7, 1])}
    with pytest.raises(NotImplementedError, match='padded'):
        criterion(y, {'scores': torch.zeros(3, 11, 8)}, margin=0.5)


# ----------------------------------------------------------------------------------------------------- the float64 double
def _real(lens, cap):
    """[B * cap] bool: the real rows of a padded [B, cap] layout"""
    return (torch.arange(cap)[None, :] < lens.reshape(-1, 1).long()).reshape(-1)


class _PaddedCpuOps(_CpuOps):
    """_CpuOps with the lengths arguments of openglue_b200._ops._Ops (the kernels' padded forms restated in float64)."""

    def kenc_input(self, kpts, side, rows, S, width, height, lens=None, pair_wh=None):
        if lens is None:
            return super().kenc_input(kpts, side, rows, S, width, height)
        B = lens.numel()
        wh = pair_wh[:, :2].to(self.dt).repeat_interleave(rows // B, 0)
        xy = 2 * kpts.reshape(rows, 2).to(self.dt) / (wh - 1) - 1
        out = torch.cat([xy, side.reshape(rows, S).to(self.dt)], 1) if S else xy
        return torch.where(_real(lens, rows // B)[:, None], out, torch.zeros((), dtype=self.dt))

    def mask_rows(self, X, lens):
        return torch.where(_real(lens, X.shape[0] // lens.numel())[:, None], X, torch.zeros((), dtype=X.dtype))

    def attention(self, q, k, v, B, nq, nk, H, dh, klen=None):
        if klen is None:
            return super().attention(q, k, v, B, nq, nk, H, dh)
        qh = q.view(B, nq, H, dh).permute(0, 2, 1, 3)
        kh = k.view(B, nk, H, dh).permute(0, 2, 1, 3)
        vh = v.view(B, nk, H, dh).permute(0, 2, 1, 3)
        s = qh @ kh.transpose(2, 3) * dh ** -0.5
        s = s.masked_fill(torch.arange(nk)[None, None, None, :] >= klen.long()[:, None, None, None], -float('inf'))
        return (s.softmax(-1) @ vh).permute(0, 2, 1, 3).reshape(B * nq, H * dh).contiguous()

    def softmax_rows(self, P, ld, rows, cols, klen=None):
        if klen is None:
            return super().softmax_rows(P, ld, rows, cols)
        v = self._view(P, 0, rows, cols, ld)
        keep = torch.arange(cols)[None, :] < klen.long().repeat_interleave(rows // klen.numel())[:, None]
        v.copy_(v.masked_fill(~keep, -float('inf')).softmax(-1))

    def softmax_bwd_rows(self, P, dP, ld, rows, cols, scale, klen=None):
        super().softmax_bwd_rows(P, dP, ld, rows, cols, scale)     # P = 0 past the keys: dS = 0 there

    def bn_fwd(self, a, gamma, beta, eps, momentum, running_mean, running_var, lens=None):
        if lens is None:
            return super().bn_fwd(a, gamma, beta, eps, momentum, running_mean, running_var)
        real = _real(lens, a.shape[0] // lens.numel())
        r = a.clamp_min(0)
        mean, var = r[real].mean(0), r[real].var(0, unbiased=False)
        invstd = (var + eps).rsqrt()
        if running_mean is not None:
            n = int(real.sum())
            running_mean.mul_(1 - momentum).add_((momentum * mean).to(running_mean.dtype))
            running_var.mul_(1 - momentum).add_((momentum * var * n / max(n - 1, 1)).to(running_var.dtype))
        return (r - mean) * invstd * gamma.detach().to(self.dt) + beta.detach().to(self.dt), mean, invstd

    def bn_bwd(self, dy, a, gamma, mean, invstd, lens=None):
        if lens is None:
            return super().bn_bwd(dy, a, gamma, mean, invstd)
        real = _real(lens, a.shape[0] // lens.numel())[:, None]
        dy = torch.where(real, dy, torch.zeros((), dtype=dy.dtype))
        r = a.clamp_min(0)
        xhat = (r - mean) * invstd
        dbeta, dgamma = dy.sum(0), (dy * xhat).sum(0)
        n = int(real.sum())
        dr = gamma.detach().to(self.dt) * invstd * (dy - dbeta / n - xhat * dgamma / n)
        return torch.where(real, dr * (a > 0), torch.zeros((), dtype=dr.dtype)), dgamma, dbeta

    def sinkhorn_fwd(self, Sp, dust, B, n, m, iters, reg, lens=None):
        if lens is None:
            return super().sinkhorn_fwd(Sp, dust, B, n, m, iters, reg)
        from oracle.sinkhorn_grad_oracle import forward_with_history
        out = torch.full((B, n + 1, m + 1), -float('inf'), dtype=self.dt)
        for b in range(B):
            nb, mb = int(lens[b]), int(lens[B + b])
            out[b, :nb + 1, :mb + 1] = forward_with_history(Sp[b:b + 1, :nb, :mb].to(self.dt), dust.to(self.dt).reshape(()), iters, reg)[0][0]
        return out, None

    def sinkhorn_bwd(self, Sp, dust, hist, G, B, n, m, iters, reg, lens=None):
        if lens is None:
            return super().sinkhorn_bwd(Sp, dust, hist, G, B, n, m, iters, reg)
        from oracle.sinkhorn_grad_oracle import backward
        dZ = self.zeros(B, n + 1, m + 1)
        dd = 0.0
        for b in range(B):
            nb, mb = int(lens[b]), int(lens[B + b])
            dS, d1 = backward(Sp[b:b + 1, :nb, :mb].to(self.dt), dust.to(self.dt).reshape(()), iters, reg,
                              G[b:b + 1, :nb + 1, :mb + 1].to(self.dt))
            dZ[b, :nb, :mb] = dS[0]
            dZ[b, nb, :mb + 1] = 1e3              # like the kernel, the pair's dustbin row and column hold (here: arbitrary) gradients
            dZ[b, :nb, mb] = 1e3                  # that the score GEMM's backward must not pass on
            dd = dd + d1
        return dZ, dd.reshape(1)


# ----------------------------------------------------------------------------------------------------- the restated reference
def restated_reference(SG, cfg, sd, lens0, lens1, wh0, wh1, dtype):
    """The reference module (class SG, float ``dtype``, train mode) restated for a padded batch whose capacities differ (N != M):
    BatchNorm with statistics over the real columns of every pair (running_var with the unbiased factor of their count), attention
    masked to each sequence's keys, keypoints normalised with each pair's (W, H) (wh0 / wh1 [B, 2]) and the Sinkhorn of each pair on
    its own block, -inf elsewhere.  At full lengths and one image size it is the reference."""
    model = SG(copy.deepcopy(cfg))
    model.load_state_dict(sd, strict=True)
    model = model.to(dtype).train()
    N = M = None

    def lens_of(L):
        return lens0.long() if L == N else lens1.long()

    def norm(kpts, _shape):
        wh = (wh0 if kpts.shape[1] == N else wh1).to(kpts.dtype)
        return 2 * kpts / (wh[:, None, :] - 1) - 1

    def attention(query, key, value):
        q = query.transpose(2, 3)
        a = torch.matmul(q, key) * query.size(2) ** -0.5
        L = key.shape[-1]
        a = a.masked_fill(torch.arange(L)[None, None, None, :] >= lens_of(L)[:, None, None, None], -float('inf')).softmax(-1)
        return torch.matmul(a, value.transpose(2, 3)).transpose(2, 3).contiguous(), a

    def bn(self, x):
        L = x.shape[2]
        keep = torch.arange(L)[None, :] < lens_of(L)[:, None]
        xs = x.permute(0, 2, 1)[keep]
        mean, var = xs.mean(0), xs.var(0, unbiased=False)
        cnt = xs.shape[0]
        with torch.no_grad():
            self.running_mean.mul_(1 - self.momentum).add_(self.momentum * mean)
            self.running_var.mul_(1 - self.momentum).add_(self.momentum * var * cnt / (cnt - 1))
            self.num_batches_tracked += 1
        return (x - mean[None, :, None]) * (var + self.eps).rsqrt()[None, :, None] * self.weight[None, :, None] + self.bias[None, :, None]

    def matching(S):
        out = []
        for b in range(S.shape[0]):
            nb, mb = int(lens0[b]), int(lens1[b])
            p = type(model).get_matching_probs(model, S[b:b + 1, :nb, :mb])
            out.append(F.pad(p, (0, M - mb, 0, N - nb), value=-float('inf')))
        return torch.cat(out)

    def forward(data):
        nonlocal N, M
        N, M = data['keypoints0'].shape[1], data['keypoints1'].shape[1]
        assert N != M, 'the restatement tells the images apart by their capacities'
        return type(model).forward(model, data)

    model.normalize_keypoints = norm
    model.get_matching_probs = matching
    for mod in model.modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            mod.forward = types.MethodType(bn, mod)
        if hasattr(mod, 'attention_func'):
            mod.attention_func = attention
    model.forward = forward
    return model


# ----------------------------------------------------------------------------------------------------- cases
# name: (default_config kwargs, extra config keys, pairs [(n_b, m_b)], capacity (N, M), seed)
CASES = {
    'mixed': (dict(descriptor_dim=64, num_stages=2, num_iters=10), {}, [(21, 9), (1, 17), (14, 2)], (24, 19), 51),
    'mixed_offset_nodesc': (dict(descriptor_dim=32, num_heads=4, num_stages=2, num_iters=10, use_offset=True, residual=False),
                            dict(no_descriptors=True), [(9, 30), (30, 1), (2, 11), (17, 17)], (31, 33), 52),
    'one_pair': (dict(descriptor_dim=64, num_stages=2, num_iters=10), {}, [(29, 22)], (36, 25), 53),
}
SIZES = [(640., 480.), (321., 200.), (1000., 777.), (90., 130.)]


def case_config(case):
    kw, extra, _, _, _ = CASES[case]
    return dict(default_config(**kw), **extra)


def case_state(case):
    seed = CASES[case][4]
    return perturb_bn(synthetic_state_dict(case_config(case), seed=seed), seed)


def case_batch(case, fill=0.0):
    """(padded data, upstream gradients G on the real entries, lens0, lens1, wh0, wh1): every pair and image has its own size"""
    cfg = case_config(case)
    _, _, pairs, (N, M), seed = CASES[case]
    B, d, S = len(pairs), cfg['descriptor_dim'], cfg['positional_encoding']['side_info_size']
    lens0 = torch.tensor([p[0] for p in pairs], dtype=torch.int32)
    lens1 = torch.tensor([p[1] for p in pairs], dtype=torch.int32)
    wh0 = torch.tensor([SIZES[b % 4] for b in range(B)], dtype=torch.float64)
    wh1 = torch.tensor([SIZES[(b + 1) % 4] for b in range(B)], dtype=torch.float64)
    data = synthetic_pairs(B, N, M, d, S, family='planted', seed=seed)
    data.pop('planted_matches0', None)
    for i, (lens, cap) in enumerate(((lens0, N), (lens1, M))):
        pad = ~_real(lens, cap).reshape(B, cap)
        for k in ('keypoints', 'side_info', 'local_descriptors'):
            data[f'{k}{i}'] = data[f'{k}{i}'].masked_fill(pad[..., None], fill)
        data[f'num_keypoints{i}'] = lens
    data['image0_size'], data['image1_size'] = wh0.float(), wh1.float()
    g = torch.Generator().manual_seed(seed + 1)
    G = {'scores': torch.randn(B, N + 1, M + 1, generator=g).double(),
         'context_descriptors0': torch.randn(B, d, N, generator=g).double(),
         'context_descriptors1': torch.randn(B, d, M, generator=g).double()}
    valid = masks(lens0, lens1, N, M, d)
    G = {k: G[k] * valid[k] for k in OUTS}
    return data, G, lens0, lens1, wh0, wh1


def masks(lens0, lens1, N, M, d):
    """{output: bool mask of its real entries}"""
    l0, l1 = lens0.long(), lens1.long()
    r0, r1 = torch.arange(N + 1)[None, :] <= l0[:, None], torch.arange(M + 1)[None, :] <= l1[:, None]
    return {'scores': r0[:, :, None] & r1[:, None, :],
            'context_descriptors0': (torch.arange(N)[None, :] < l0[:, None])[:, None, :].expand(-1, d, -1),
            'context_descriptors1': (torch.arange(M)[None, :] < l1[:, None])[:, None, :].expand(-1, d, -1)}


def reference_run(case, dtype, restated=True, trimmed=False):
    """float64 / float32 autograd of the restated reference on a case (or of the plain reference on its trimmed single pair, or at
    full lengths): {'outs', 'grads', 'dld', 'bufs'} on the CPU in float64, padded layout."""
    SG = _reference_class(True)
    cfg, sd = case_config(case), case_state(case)
    data, G, lens0, lens1, wh0, wh1 = case_batch(case)
    if trimmed:                                          # one pair: the reference on its real keypoints, no restatement
        n, m = int(lens0[0]), int(lens1[0])
        d = {f'{k}{i}': data[f'{k}{i}'][:, :L] for k in ('keypoints', 'side_info', 'local_descriptors') for i, L in ((0, n), (1, m))}
        d['image0_size'], d['image1_size'] = tuple(wh0[0].tolist()), tuple(wh1[0].tolist())
        G = {'scores': G['scores'][:, :n + 1, :m + 1], 'context_descriptors0': G['context_descriptors0'][:, :, :n],
             'context_descriptors1': G['context_descriptors1'][:, :, :m]}
        model = SG(copy.deepcopy(cfg))
        model.load_state_dict(sd, strict=True)
        model = model.to(dtype).train()
    elif restated:
        d = {k: v for k, v in data.items() if not k.startswith('num_keypoints')}
        d['image0_size'] = d['image1_size'] = (640., 480.)   # the restatement reads the per-pair sizes
        model = restated_reference(SG, cfg, sd, lens0, lens1, wh0, wh1, dtype)
    else:                                                # plain reference at full lengths, one image size
        d = {k: v for k, v in data.items() if not k.startswith('num_keypoints')}
        d['image0_size'] = d['image1_size'] = (640., 480.)
        model = SG(copy.deepcopy(cfg))
        model.load_state_dict(sd, strict=True)
        model = model.to(dtype).train()
    d = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}
    for i in (0, 1):
        d[f'local_descriptors{i}'] = d[f'local_descriptors{i}'].clone().requires_grad_(True)
    y = model(d)
    L = 0
    for k in OUTS:
        out = y[k]
        L = L + (G[k].to(dtype) * torch.where(torch.isfinite(out), out, torch.zeros((), dtype=dtype))).sum()
    L.backward()
    res = {'outs': {k: y[k].detach().double() for k in OUTS},
           'grads': {k: p.grad.detach().double() for k, p in model.named_parameters() if p.grad is not None},
           'dld': [None if d[f'local_descriptors{i}'].grad is None else d[f'local_descriptors{i}'].grad.detach().double() for i in (0, 1)],
           'bufs': {k: v.detach().clone() for k, v in model.named_buffers()}}
    if trimmed:                                          # back into the padded layout of the case
        _, _, pairs, (N, M), _ = CASES[case]
        n, m = pairs[0]
        sc = torch.full((1, N + 1, M + 1), -float('inf'), dtype=torch.float64)
        sc[:, :n + 1, :m + 1] = res['outs']['scores']
        res['outs']['scores'] = sc
        res['outs']['context_descriptors0'] = F.pad(res['outs']['context_descriptors0'], (0, N - n))
        res['outs']['context_descriptors1'] = F.pad(res['outs']['context_descriptors1'], (0, M - m))
        res['dld'] = [None if g is None else F.pad(g, (0, 0, 0, c - L)) for g, c, L in ((res['dld'][0], N, n), (res['dld'][1], M, m))]
    return res


def train_step_run(case, ops, model, fill=0.0):
    """TrainStep on the padded case with the given kernels (the CPU double or the device's), L = sum <G, out> on the real entries:
    same dict as reference_run, float64 on the CPU, with the raw outputs under 'raw'."""
    data, G, *_ = case_batch(case, fill)
    dev = next(model.parameters()).device
    dt = next(model.parameters()).dtype
    data = {k: (v.to(dev, dt) if torch.is_tensor(v) and v.is_floating_point() and not k.startswith('image') else
                v.to(dev) if torch.is_tensor(v) else v) for k, v in data.items()}
    step = TrainStep(model, data, ops=ops)
    outs = dict(zip(OUTS, step.forward()))
    grads = step.backward(*[G[k].to(dev, dt) for k in OUTS])
    return {'outs': {k: v.detach().cpu().double() for k, v in outs.items()},
            'grads': {k: v.detach().cpu().double() for k, v in grads.items() if not k.startswith('local_descriptors')},
            'dld': [grads[f'local_descriptors{i}'].detach().cpu().double() if f'local_descriptors{i}' in grads else None for i in (0, 1)],
            'bufs': {k: v.detach().cpu().clone() for k, v in model.named_buffers()}}


def check_against(got, refs, lens0, lens1, chk):
    """chk(what, got, *refs) on the real entries (refs: reference runs, the first one float64); the padding of got must be -inf
    (scores) / 0 (context descriptors, local-descriptor gradients) exactly."""
    ref = refs[0]
    N, M = got['outs']['context_descriptors0'].shape[2], got['outs']['context_descriptors1'].shape[2]
    d = got['outs']['context_descriptors0'].shape[1]
    mk = masks(lens0, lens1, N, M, d)
    for k in OUTS:
        g, r = got['outs'][k], ref['outs'][k]
        chk(k, g[mk[k]], *[R['outs'][k][mk[k]] for R in refs])
        pad = g[~mk[k]]
        assert bool((torch.isneginf(pad) if k == 'scores' else pad == 0).all()), k
    assert set(got['grads']) == set(ref['grads'])
    for k, r in ref['grads'].items():
        chk(f'grad {k}', got['grads'][k].reshape(r.shape), *[R['grads'][k] for R in refs])
    for i, lens in enumerate((lens0, lens1)):
        assert (got['dld'][i] is None) == (ref['dld'][i] is None), i
        if ref['dld'][i] is None:
            continue
        real = _real(lens, got['dld'][i].shape[1])
        g = got['dld'][i].reshape(-1, d)
        chk(f'grad local_descriptors{i}', g[real], *[R['dld'][i].reshape(-1, d)[real] for R in refs])
        assert bool((g[~real] == 0).all()), i
    for k, r in ref['bufs'].items():
        if k.endswith('num_batches_tracked'):
            assert int(got['bufs'][k]) == int(r), k
        else:
            chk(f'buffer {k}', got['bufs'][k].double(), *[R['bufs'][k].double() for R in refs])


def _close(tol):
    def chk(what, g, r, *_):
        assert torch.isfinite(g).all(), what
        assert float((g - r).abs().max()) <= tol * max(1.0, float(r.abs().max())), what
    return chk


def _double_model(case):
    model = SuperGlue(case_config(case))
    model.load_state_dict(case_state(case), strict=True)
    return model.double().train()


# ----------------------------------------------------------------------------------------------------- CPU leg
@pytest.mark.parametrize('case', ['mixed', 'mixed_offset_nodesc'])
def test_restated_reference_is_the_reference_at_full_lengths(case):
    """At full lengths and one image size the restatement's masks are no-ops: it is the plain reference (float64)."""
    kw, extra, pairs, (N, M), seed = CASES[case]
    CASES[case + '_full'] = (kw, extra, [(N, M)] * len(pairs), (N, M), seed)
    try:
        global SIZES
        sizes, SIZES = SIZES, [(640., 480.)] * 4
        try:
            a = reference_run(case + '_full', torch.float64, restated=True)
            b = reference_run(case + '_full', torch.float64, restated=False)
        finally:
            SIZES = sizes
    finally:
        del CASES[case + '_full']
    lens0 = torch.full((len(pairs),), N, dtype=torch.int32)
    lens1 = torch.full((len(pairs),), M, dtype=torch.int32)
    check_against(a, [b], lens0, lens1, _close(1e-12))


@pytest.mark.parametrize('case', ['mixed', 'mixed_offset_nodesc'])
def test_padded_schedule_on_the_cpu_double_matches_the_restated_reference(case):
    ref = reference_run(case, torch.float64)
    _, _, lens0, lens1, _, _ = case_batch(case)
    for fill in (0.0, float('nan')):
        got = train_step_run(case, _PaddedCpuOps(), _double_model(case), fill)
        check_against(got, [ref], lens0, lens1, _close(2e-6))


def test_one_pair_on_the_cpu_double_matches_the_reference_on_the_trimmed_pair():
    ref = reference_run('one_pair', torch.float64, trimmed=True)
    _, _, lens0, lens1, _, _ = case_batch('one_pair')
    got = train_step_run('one_pair', _PaddedCpuOps(), _double_model('one_pair'), float('nan'))
    check_against(got, [ref], lens0, lens1, _close(2e-6))
