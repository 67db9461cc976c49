"""Time the metric terms of the matching loss (criterion with a margin), in one process:
  (1) CUDA events around ``criterion(y_true, y_pred, margin=0.5)`` - the NLL term plus og_metric_loss_fwd - without and with the
      gradient (inputs requiring grad: the call also writes d metric_loss / d context descriptors), at B x N x M = 4 x 1024^2 and
      16 x 2048^2, d = 256;
  (2) the graph-replayed training iteration (GraphedTrainStep with ClippedAdam) without and with a margin (metric_weight 0.5),
      alternated round by round, at the shapes of tools/train_step_timing.py (d = 256, 9 stages, 4 heads, 20 Sinkhorn
      iterations, 1024 keypoints, batch 4 and 2).
Prints one JSON object with the GPU's name and power limit beside the numbers.

    python tools/metric_loss_timing.py [--iters 20] [--rounds 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics

import torch

from gpu_timing import card, rounds_ms
from train_step_timing import _labels


def _criterion_case(B, n, m, d, seed, dev):
    g = torch.Generator().manual_seed(seed)
    gt0 = torch.full((B, n), -1, dtype=torch.int64)
    gt1 = torch.full((B, m), -1, dtype=torch.int64)
    for b in range(B):
        k = min(n, m) // 2
        src, dst = torch.randperm(n, generator=g)[:k], torch.randperm(m, generator=g)[:k]
        gt0[b, src], gt1[b, dst] = dst, src
    c0, c1 = torch.randn(B, d, n, generator=g), torch.randn(B, d, m, generator=g)
    scores = -8.0 * torch.rand(B, n + 1, m + 1, generator=g) - 0.05
    return ({'gt_matches0': gt0.to(dev), 'gt_matches1': gt1.to(dev)},
            {'scores': scores.to(dev), 'context_descriptors0': c0.to(dev), 'context_descriptors1': c1.to(dev)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--batches', type=int, nargs='+', default=[4, 2])
    ap.add_argument('--keypoints', type=int, default=1024)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('metric_loss_timing needs a CUDA device')
    from openglue_b200 import ClippedAdam, SuperGlue, criterion
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
    from openglue_b200.training import GraphedTrainStep
    dev = torch.device('cuda:0')
    res = {'card': card(), 'iters': args.iters, 'rounds': args.rounds, 'criterion': {}, 'train_step': {}}

    for B, N in ((4, 1024), (16, 2048)):
        y_true, y_pred = _criterion_case(B, N, N, 256, 0, dev)
        yg = dict(y_pred, context_descriptors0=y_pred['context_descriptors0'].clone().requires_grad_(True),
                  context_descriptors1=y_pred['context_descriptors1'].clone().requires_grad_(True))
        plain = lambda: criterion(y_true, y_pred, margin=None)
        fwd = lambda: criterion(y_true, y_pred, margin=0.5)
        grad = lambda: criterion(y_true, yg, margin=0.5)
        for f in (plain, fwd, grad):
            for _ in range(2):
                f()
        tp, tf, tg = rounds_ms({'plain': plain, 'fwd': fwd, 'grad': grad}, args.iters, args.rounds).values()
        res['criterion'][f'{B}x{N}x{N} d=256'] = {'margin_none_ms': statistics.median(tp), 'margin_ms': statistics.median(tf),
                                                   'margin_with_grad_ms': statistics.median(tg), 'rounds_ms': [tp, tf, tg]}
        del y_true, y_pred, yg
        torch.cuda.empty_cache()

    cfg = default_config(descriptor_dim=256, num_stages=9, num_heads=4, num_iters=20)
    sd = synthetic_state_dict(cfg, seed=0)
    res['config'] = 'd=256, 9 stages, 4 heads, 20 Sinkhorn iterations, tf32x3 training GEMMs, ClippedAdam in the graph'

    def model():
        m = SuperGlue(dict(cfg, precision='tf32x3'))
        m.load_state_dict(copy.deepcopy(sd))
        return m.to(dev).train()

    opt = lambda m: ClippedAdam.from_config(m, {'lr': 1e-4, 'grad_clip': 10.0, 'scheduler_gamma': 0.999994})
    for B in args.batches:
        pairs = synthetic_pairs(B, args.keypoints, args.keypoints, 256, 1, family='planted', seed=7)
        y_true = _labels(pairs, dev)
        data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in pairs.items()}
        ma, mb = model(), model()
        step_a = GraphedTrainStep(ma, data, y_true, optimizer=opt(ma))
        step_b = GraphedTrainStep(mb, data, y_true, optimizer=opt(mb), margin=0.5, metric_weight=0.5)
        fa, fb = (lambda: step_a(data, y_true)), (lambda: step_b(data, y_true))
        for f in (fa, fb):
            for _ in range(3):
                f()
        ta, tb = rounds_ms({'a': fa, 'b': fb}, args.iters, args.rounds).values()
        res['train_step'][f'B={B}'] = {'no_margin_ms': ta, 'margin_ms': tb, 'median_no_margin_ms': statistics.median(ta),
                                       'median_margin_ms': statistics.median(tb)}
        del step_a, step_b, ma, mb
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
