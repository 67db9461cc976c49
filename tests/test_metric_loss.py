"""Metric terms of the matching loss on the GPU (og_metric_loss_fwd through openglue_b200.criterion(margin=...)): the operator
against the reference-minted fixtures (tests/golden/metric_*.pt), an edge table against the oracle on the same tensors, its launch
count, the training step with a margin against the reference's autograd (tests/golden/train_metric.pt), and the graphed step
against the eager one.

Selections: an entry is compared where the fp64 fixture marks it decisive (runner-up minus minimum > 1e-5) or as an exact tie
(gap 0: the lowest index wins, as torch.argmin); entries in between are undecidable in fp32 and are only counted."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import metric_loss_oracle as M                         # noqa: E402  (checker only)
from oracle.gen_golden_metric_loss import metric_inputs, CASES     # noqa: E402

DEV = 'cuda:0'
SEL = ('n0', 'u0', 'n1', 'u1')
DECISIVE = 1e-5


def _fx(name):
    return torch.load(os.path.join(ROOT, 'tests', 'golden', name + '.pt'), weights_only=False)


def _inputs(name, fx):
    if 'c0' in fx:
        return fx['gt_matches0'], fx['gt_matches1'], fx['c0'], fx['c1']
    return metric_inputs(*CASES[name])


def _run(gt0, gt1, c0, c1, margin, grad_scale=1.0, want_grad=True):
    from openglue_b200.losses import metric_loss_with_grad
    yt = {'gt_matches0': gt0.to(DEV), 'gt_matches1': gt1.to(DEV)}
    yp = {'context_descriptors0': c0.to(DEV), 'context_descriptors1': c1.to(DEV)}
    return metric_loss_with_grad(yt, yp, margin, grad_scale, want_grad)


def _check_selections(out, sel, where):
    undecided = 0
    for k in SEL:
        got, ref, gap = out[k].cpu(), sel[k], sel['gap_' + k].double()
        judged = (gap > DECISIVE) | (gap == 0)
        bad = judged & (got != ref)
        assert not bad.any(), (where, k, torch.nonzero(bad)[:5].tolist())
        undecided += int((~judged).sum())
    return undecided


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['metric_small', 'metric_empty', 'metric_ties', 'metric_m01', 'metric_m1', 'metric_large'])
def test_operator_matches_reference(name):
    fx = _fx(name)
    gt0, gt1, c0, c1 = _inputs(name, fx)
    margin = fx['case'][8]
    out = _run(gt0, gt1, c0, c1, margin)
    undecided = _check_selections(out, fx['selections'], name)
    print(f'{name}: {undecided} undecided selection entries (gap <= {DECISIVE:g})')
    ref = float(fx['metric_loss_f64'])
    assert abs(float(out['metric_loss']) - ref) <= 1e-5 * max(1.0, abs(ref))
    if 'dc0_f64' in fx:
        for k in ('dc0', 'dc1'):
            want = fx[k + '_f64']
            assert float((out[k].cpu().double() - want).abs().max()) <= 2e-4 * float(want.abs().max()), k
    again = _run(gt0, gt1, c0, c1, margin)                     # deterministic
    for k in ('metric_loss',) + SEL + (('dc0', 'dc1') if 'dc0_f64' in fx else ()):
        assert torch.equal(out[k], again[k]), k
    if name == 'metric_ties':                                  # duplicated columns: each row picks the lower copy
        half = c1.shape[2] // 2
        assert (out['u0'] < half).all()


def _edge_case(B, n, m, d, seed, labels):
    g = torch.Generator().manual_seed(seed)
    gt0 = torch.full((B, n), -1, dtype=torch.int64)
    gt1 = torch.full((B, m), -1, dtype=torch.int64)
    for b in range(B):
        k = max(1, min(n, m) // 2)
        src, dst = torch.randperm(n, generator=g)[:k], torch.randperm(m, generator=g)[:k]
        gt0[b, src], gt1[b, dst] = dst, src
        gt0[b, (torch.rand(n, generator=g) < 0.1) & (gt0[b] < 0)] = -2
        gt1[b, (torch.rand(m, generator=g) < 0.1) & (gt1[b] < 0)] = -2
        if labels == 'shared' and n > 1:                        # two rows name one column
            gt0[b, 1] = gt0[b, 0] if gt0[b, 0] >= 0 else 0
            gt0[b, 0] = gt0[b, 1]
    if labels == 'empty_one':                                  # pair 0: no matched row, no unmatched column
        gt0[0][gt0[0] >= 0] = -1
        gt1[0][gt1[0] == -1] = -2
    elif labels == 'empty_all':                                # no set in any pair: every key point ignored
        gt0[:] = -2
        gt1[:] = -2
    c0 = torch.randn(B, d, n, generator=g)
    c1 = torch.randn(B, d, m, generator=g)
    return gt0, gt1, c0, c1


EDGES = [(B, n, m, d, lab) for (B, n, m, d, lab) in [
    (1, 1, 1, 64, 'plain'), (1, 1, 37, 128, 'plain'), (3, 37, 1, 256, 'plain'), (1, 37, 37, 64, 'plain'), (3, 128, 131, 64, 'plain'),
    (3, 131, 128, 128, 'shared'), (1, 128, 37, 256, 'shared'), (3, 131, 131, 256, 'empty_one'), (3, 37, 128, 64, 'empty_all'),
    (1, 131, 1, 128, 'shared'), (3, 128, 128, 256, 'plain'), (1, 37, 131, 128, 'empty_one')]]


@pytest.mark.gpu
@pytest.mark.parametrize('B,n,m,d,labels', EDGES)
def test_edges_against_the_oracle(B, n, m, d, labels):
    gt0, gt1, c0, c1 = _edge_case(B, n, m, d, 7 * n + m + d + B, labels)
    x0, x1 = c0.double().requires_grad_(True), c1.double().requires_grad_(True)
    ref = M.metric_terms(gt0, gt1, x0, x1, 0.5)
    ref['metric_loss'].backward()
    out = _run(gt0, gt1, c0, c1, 0.5, grad_scale=0.75)
    _check_selections(out, ref, (B, n, m, d, labels))
    want = float(ref['metric_loss'].detach())
    assert abs(float(out['metric_loss']) - want) <= 1e-5 * max(1.0, abs(want))
    if M.smallest_margin(gt0, gt1, ref) > DECISIVE:            # the gradient is only defined away from flipping decisions
        for g, r in ((out['dc0'], x0.grad), (out['dc1'], x1.grad)):
            r = 0.75 * r
            assert float((g.cpu().double() - r).abs().max()) <= 2e-4 * max(float(r.abs().max()), 1e-30)
    if labels == 'empty_all':
        assert float(out['metric_loss']) == 0.0 and float(out['dc0'].abs().max()) == 0.0


@pytest.mark.gpu
def test_launch_counts():
    from openglue_b200 import _cabi
    from openglue_b200._cabi import ptr, stream
    lib = _cabi.lib()
    gt0, gt1, c0, c1 = _edge_case(2, 128, 96, 64, 3, 'plain')
    gt0, gt1, c0, c1 = (t.to(DEV) for t in (gt0, gt1, c0, c1))
    B, d, n, m = 2, 64, 128, 96
    idx = [torch.empty(B, k, dtype=torch.int64, device=DEV) for k in (n, n, m, m)]
    loss = torch.empty(1, device=DEV)
    for prec, fwd, grad in ((_cabi.OG_PREC_FP32, 9, 16), (_cabi.OG_PREC_TF32X3, 10, 19)):
        for want_grad, count in ((0, fwd), (1, grad)):
            wsb = lib.og_metric_loss_workspace_bytes(B, d, n, m, want_grad, prec)
            ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
            dc0, dc1 = (torch.empty_like(c0), torch.empty_like(c1)) if want_grad else (None, None)
            before = lib.og_last_forward_launches()
            rc = lib.og_metric_loss_fwd(ptr(c0), ptr(c1), ptr(gt0), ptr(gt1), B, d, n, m, 0.5, prec, ptr(loss), *[ptr(t) for t in idx],
                                        ptr(dc0), ptr(dc1), 1.0, ptr(ws), wsb, stream())
            _cabi.check(rc, 'og_metric_loss_fwd')
            assert lib.og_last_forward_launches() - before == count, (prec, want_grad)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_criterion_with_a_margin_is_differentiable():
    from openglue_b200 import criterion
    fx = _fx('metric_small')
    gt0, gt1, c0, c1 = _inputs('metric_small', fx)
    B, n, m = gt0.shape[0], gt0.shape[1], gt1.shape[1]
    scores = (-8.0 * torch.rand(B, n + 1, m + 1, generator=torch.Generator().manual_seed(0)) - 0.05).to(DEV).requires_grad_(True)
    x0, x1 = c0.to(DEV).requires_grad_(True), c1.to(DEV).requires_grad_(True)
    yt = {'gt_matches0': gt0.to(DEV), 'gt_matches1': gt1.to(DEV)}
    out = criterion(yt, {'scores': scores, 'context_descriptors0': x0, 'context_descriptors1': x1}, margin=0.5)
    plain = criterion(yt, {'scores': scores.detach()}, margin=None)
    assert torch.equal(out['loss'].detach(), plain['loss'])
    ref = float(fx['metric_loss_f64'])
    assert abs(float(out['metric_loss'].detach()) - ref) <= 1e-5 * max(1.0, ref)
    (1.0 * out['loss'] + 0.25 * out['metric_loss']).backward()
    for g, k in ((x0.grad, 'dc0_f64'), (x1.grad, 'dc1_f64')):
        want = 0.25 * fx[k]
        assert float((g.cpu().double() - want).abs().max()) <= 2e-4 * float(want.abs().max())
    with torch.no_grad():
        again = criterion(yt, {'scores': scores, 'context_descriptors0': x0, 'context_descriptors1': x1}, margin=0.5)
    assert torch.equal(again['metric_loss'], out['metric_loss'].detach())
    with pytest.raises(NotImplementedError, match='context_descriptors0'):
        criterion(yt, {'scores': scores.detach()}, margin=0.5)


def _train_model(fx, precision):
    from openglue_b200 import SuperGlue
    from openglue_b200.synthetic import synthetic_state_dict
    sd = synthetic_state_dict(fx['config'], seed=fx['weights_seed'])
    sd.update(fx['bn_buffers'])
    model = SuperGlue(dict(fx['config'], precision=precision))
    model.load_state_dict(sd, strict=True)
    return model.to(DEV).train()


def _rel(a, b):
    return float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_training_step_with_a_margin_matches_reference(precision):
    from openglue_b200 import criterion
    fx = _fx('train_metric')
    model = _train_model(fx, precision)
    data = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in fx['data'].items()}
    data['local_descriptors0'] = data['local_descriptors0'].clone().requires_grad_(True)
    data['local_descriptors1'] = data['local_descriptors1'].clone().requires_grad_(True)
    gt0, gt1 = fx['gt_matches0'], fx['gt_matches1']
    out = model(data)
    # forward accuracy first: the oracle, run on the GPU's context descriptors, must select what the fp64 reference selected
    sel = M.metric_terms(gt0, gt1, out['context_descriptors0'].detach().cpu().double(), out['context_descriptors1'].detach().cpu().double(),
                         fx['margin'])
    for k in SEL:
        assert torch.equal(sel[k], fx['selections'][k]), ('forward accuracy', k)
    loss = criterion({'gt_matches0': gt0.to(DEV), 'gt_matches1': gt1.to(DEV)}, out, margin=fx['margin'])
    assert abs(float(loss['loss'].detach()) - float(fx['loss_f64'])) <= 1e-4 * max(1.0, abs(float(fx['loss_f64'])))
    assert abs(float(loss['metric_loss'].detach()) - float(fx['metric_loss_f64'])) <= 1e-4 * max(1.0, abs(float(fx['metric_loss_f64'])))
    (fx['nll_weight'] * loss['loss'] + fx['metric_weight'] * loss['metric_loss']).backward()
    worst = ('', 0.0)
    for k, p in model.named_parameters():
        ref = fx['grads'][k]
        assert p.grad is not None, k
        g = p.grad.detach().cpu()
        scale = float(ref.abs().max())
        if scale < 1e-9:
            assert float(g.abs().max()) < 1e-6, k
            continue
        r = _rel(g, ref)
        worst = max(worst, (k, r), key=lambda t: t[1])
        assert r <= 1e-3, (k, r)
        assert float((g - ref).abs().max()) <= 1e-3 * scale, k
    print(f'train_metric {precision}: worst relative gradient error {worst[1]:.2e} ({worst[0]})')
    for i in (0, 1):
        assert _rel(data[f'local_descriptors{i}'].grad.cpu(), fx[f'dlocal_descriptors{i}']) <= 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize('with_optimizer', [False, True])
def test_graphed_step_with_a_margin_is_bit_identical_to_the_eager_step(with_optimizer):
    from openglue_b200 import ClippedAdam, criterion
    from openglue_b200.training import GraphedTrainStep
    fx = _fx('train_metric')
    data = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in fx['data'].items()}
    y_true = {'gt_matches0': fx['gt_matches0'].to(DEV), 'gt_matches1': fx['gt_matches1'].to(DEV)}
    eager, graphed = _train_model(fx, 'tf32x3'), _train_model(fx, 'tf32x3')
    if with_optimizer:
        opt_e, opt_g = ClippedAdam(eager.parameters()), ClippedAdam(graphed.parameters())
    else:
        opt_e, opt_g = torch.optim.SGD(eager.parameters(), lr=1e-3), torch.optim.SGD(graphed.parameters(), lr=1e-3)
    step = GraphedTrainStep(graphed, data, y_true, optimizer=opt_g if with_optimizer else None, margin=0.5, metric_weight=0.5)
    for it in range(3):
        opt_e.zero_grad()
        out = criterion(y_true, eager(data), margin=0.5)
        (1.0 * out['loss'] + 0.5 * out['metric_loss']).backward()
        opt_e.step()
        got = step(data, y_true)
        if not with_optimizer:
            opt_g.step()
        assert torch.equal(out['loss'].detach(), got['loss']), it
        assert torch.equal(out['metric_loss'].detach(), got['metric_loss']), it
        assert float(got['metric_loss']) > 0
        for (k, pe), (_, pg) in zip(eager.named_parameters(), graphed.named_parameters()):
            assert torch.equal(pe.grad, pg.grad), (it, k)
            assert torch.equal(pe, pg), (it, k)
    for (k, be), (_, bg) in zip(eager.named_buffers(), graphed.named_buffers()):
        assert torch.equal(be, bg), k
