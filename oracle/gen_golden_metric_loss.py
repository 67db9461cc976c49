"""Mint golden vectors for the metric terms of the matching loss (``criterion(..., margin=mu)['metric_loss']``) by running the
UNMODIFIED reference ``utils.losses.criterion`` (ucuapps/OpenGlue @ /root/reference) and torch autograd through it.

TEST INFRASTRUCTURE.  Runs only in the build container; outputs are committed under tests/golden/metric_*.pt and
tests/golden/train_metric.pt and pin ``oracle/metric_loss_oracle.py`` (tests/test_metric_loss_oracle.py) and the CUDA path
(tests/test_metric_loss.py).

    python oracle/gen_golden_metric_loss.py

Criterion-level cases keep: inputs (or, for metric_large, the seed that regenerates them), labels, the loss and the gradients with
respect to both context descriptors in fp32 and fp64, and from the fp64 run the four hard-negative index vectors, each selection's
gap (runner-up minus minimum, masked or unmasked as used) and every hinge argument.

train_metric: the reference SuperGlue in ``train()`` mode, ``1.0 * loss + 0.5 * metric_loss`` backpropagated, every parameter
gradient kept (fp64 run, stored as fp32).  Data seeds are searched in order until every selection gap and every hinge argument the
loss reads is >= 1e-4 in the fp64 run, so that a correct fp32 forward pass cannot flip a decision.
"""
from __future__ import annotations

import copy
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get('OPENGLUE_REFERENCE', '/root/reference')
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from oracle import metric_loss_oracle as M  # noqa: E402
from gen_golden_loss import synthetic_labels  # noqa: E402

CASES = {
    # name: (batch, n, m, d, seed, matched share, ignore share, empty_sets, margin, duplicated columns, positive noise)
    'metric_small': (3, 37, 52, 64, 1, 0.5, 0.1, False, 0.5, False, 0.6),
    'metric_empty': (3, 20, 24, 64, 3, 0.5, 0.1, True, 0.5, False, 0.6),
    'metric_ties':  (2, 30, 40, 64, 5, 0.5, 0.1, False, 0.5, True, 0.0),     # c1 = [c1' | c1']: bit-equal duplicates, exact ties
    'metric_m01':   (2, 60, 45, 128, 7, 0.6, 0.05, False, 0.1, False, 1.5),   # few hinges active
    'metric_m1':    (2, 60, 45, 128, 8, 0.6, 0.05, False, 1.0, False, 0.6),   # every hinge active
    'metric_large': (2, 1024, 1024, 256, 9, 0.5, 0.05, False, 0.5, False, 0.6),
}
STORE_INPUTS = {'metric_small', 'metric_empty', 'metric_ties', 'metric_m01', 'metric_m1'}
TRAIN_MIN_MARGIN = 1e-4


def metric_inputs(batch, n, m, d, seed, matched, ignore, empty_sets, margin, dup, noise):
    """labels (synthetic_labels) and context descriptors in which a matched column is its row's descriptor plus noise, so that
    positives are near and the margin decides how many hinges are active"""
    gt0, gt1, _ = synthetic_labels(batch, n, m, seed, matched, ignore, empty_sets)
    g = torch.Generator().manual_seed(1000 + seed)
    c0 = torch.randn(batch, d, n, generator=g)
    c1 = torch.randn(batch, d, m // 2 if dup else m, generator=g)
    if dup:
        c1 = torch.cat([c1, c1], dim=2)
    else:
        b, i = torch.where(gt0 >= 0)
        c1[b, :, gt0[b, i]] = c0[b, :, i] + noise * torch.randn(len(b), d, generator=g)
    return gt0, gt1, c0, c1


def _selections(gt0, gt1, c0, c1, margin):
    out = M.metric_terms(gt0, gt1, c0.double(), c1.double(), margin)
    keep = ('n0', 'u0', 'n1', 'u1', 'gap_n0', 'gap_u0', 'gap_n1', 'gap_u1', 'a0', 'a1', 'au0', 'au1')
    return {k: out[k].detach().clone() for k in keep}, M.smallest_margin(gt0, gt1, out)


def mint_criterion_cases(criterion, out_dir):
    for name, case in CASES.items():
        gt0, gt1, c0, c1 = metric_inputs(*case)
        margin = case[8]
        fx = {'case': case, 'gt_matches0': gt0, 'gt_matches1': gt1,
              'reference': 'utils/losses.py:7-99 @ /root/reference, torch ' + torch.__version__}
        if name in STORE_INPUTS:
            fx['c0'], fx['c1'] = c0, c1
        for dtype, tag in ((torch.float32, 'f32'), (torch.float64, 'f64')):
            x0 = c0.to(dtype).clone().requires_grad_(True)
            x1 = c1.to(dtype).clone().requires_grad_(True)
            B, n, m = gt0.shape[0], gt0.shape[1], gt1.shape[1]
            scores = torch.zeros(B, n + 1, m + 1, dtype=dtype)
            out = criterion({'gt_matches0': gt0, 'gt_matches1': gt1}, {'context_descriptors0': x0, 'context_descriptors1': x1,
                                                                       'scores': scores}, margin=margin)
            fx[f'metric_loss_{tag}'] = out['metric_loss'].detach().clone()
            if name in STORE_INPUTS:
                out['metric_loss'].backward()
                fx[f'dc0_{tag}'] = x0.grad.detach().clone()
                fx[f'dc1_{tag}'] = x1.grad.detach().clone()
        fx['selections'], smallest = _selections(gt0, gt1, c0, c1, margin)
        if name == 'metric_large':
            fx['selections'] = {k: (v.float() if v.is_floating_point() else v) for k, v in fx['selections'].items()}
        torch.save(fx, os.path.join(out_dir, name + '.pt'))
        a = [fx['selections'][k] for k in ('a0', 'a1', 'au0', 'au1')]
        active = sum(int((t > 0).sum()) for t in a)
        print(f'{name}: metric_loss {float(fx["metric_loss_f64"]):.6f}  hinges active {active}/{sum(t.numel() for t in a)}  '
              f'smallest used gap / |hinge| {smallest:.2e}')


def mint_train_metric(out_dir):
    from gen_golden import _stub_modules
    from gen_golden_train import perturb_bn
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
    _stub_modules()
    from models.superglue.superglue import SuperGlue as RefSuperGlue          # the reference, unmodified
    from utils.losses import criterion
    batch, n, m, margin, metric_weight = 2, 40, 56, 0.5, 0.5
    cfg = default_config(descriptor_dim=64, num_stages=2, num_iters=10)
    wseed = 31
    sd = perturb_bn(synthetic_state_dict(cfg, seed=wseed), wseed)

    def run(seed, dtype):
        data = synthetic_pairs(batch, n, m, cfg['descriptor_dim'], cfg['positional_encoding']['side_info_size'], family='planted', seed=seed)
        gt0, gt1, _ = synthetic_labels(batch, n, m, seed, 0.5, 0.1, False)
        model = RefSuperGlue(copy.deepcopy(cfg))
        model.load_state_dict(sd, strict=True)
        model = model.to(dtype).train()
        d = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in data.items()}
        d['local_descriptors0'] = d['local_descriptors0'].clone().requires_grad_(True)
        d['local_descriptors1'] = d['local_descriptors1'].clone().requires_grad_(True)
        y_pred = model(d)
        out = criterion({'gt_matches0': gt0, 'gt_matches1': gt1}, y_pred, margin=margin)
        (1.0 * out['loss'] + metric_weight * out['metric_loss']).backward()
        return data, gt0, gt1, model, d, y_pred, out

    for seed in range(100, 400):
        data, gt0, gt1, model, d, y_pred, out = run(seed, torch.float64)
        sel, smallest = _selections(gt0, gt1, y_pred['context_descriptors0'].detach(), y_pred['context_descriptors1'].detach(), margin)
        if smallest >= TRAIN_MIN_MARGIN:
            break
    else:
        raise RuntimeError('no data seed with every decision of the metric loss >= 1e-4 from flipping')
    assert smallest >= TRAIN_MIN_MARGIN
    fx = {'config': cfg, 'weights_seed': wseed, 'data_seed': seed, 'bn_buffers': {k: v for k, v in sd.items() if 'running_' in k},
          'data': data, 'gt_matches0': gt0, 'gt_matches1': gt1, 'margin': margin, 'nll_weight': 1.0, 'metric_weight': metric_weight,
          'selections': sel, 'smallest_margin': smallest,
          'reference': 'models/superglue/superglue.py + utils/losses.py @ /root/reference, train() mode, torch ' + torch.__version__}
    fx['loss_f64'] = out['loss'].detach().clone()
    fx['metric_loss_f64'] = out['metric_loss'].detach().clone()
    fx['context_descriptors0_f64'] = y_pred['context_descriptors0'].detach().float()
    fx['context_descriptors1_f64'] = y_pred['context_descriptors1'].detach().float()
    fx['grads'] = {k: p.grad.detach().float() for k, p in model.named_parameters()}
    fx['dlocal_descriptors0'] = d['local_descriptors0'].grad.detach().float()
    fx['dlocal_descriptors1'] = d['local_descriptors1'].grad.detach().float()
    _, _, _, m32, d32, _, out32 = run(seed, torch.float32)
    fx['metric_loss_f32'] = out32['metric_loss'].detach().clone()
    fx['grads_f32_vs_f64_max_abs'] = max(float((p.grad.double() - fx['grads'][k].double()).abs().max()) for k, p in m32.named_parameters())
    torch.save(fx, os.path.join(out_dir, 'train_metric.pt'))
    print(f'train_metric: data seed {seed}  loss {float(fx["loss_f64"]):.6f}  metric_loss {float(fx["metric_loss_f64"]):.6f}  '
          f'smallest margin {smallest:.2e}  max |g32 - g64| {fx["grads_f32_vs_f64_max_abs"]:.2e}')


def main():
    from utils.losses import criterion                                   # the reference, unmodified
    out_dir = os.path.join(ROOT, 'tests', 'golden')
    mint_criterion_cases(criterion, out_dir)
    mint_train_metric(out_dir)


if __name__ == '__main__':
    main()
