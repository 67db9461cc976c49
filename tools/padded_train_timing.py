"""Time one training iteration on a padded batch against the two uniform batches a user could build from the same pairs:
  padded     B pairs at capacity N x M, each with its own keypoint counts (lengths uniform in [N / 2, N]), all keypoints kept;
  min_stack  the same pairs trimmed to the smallest counts of the batch (the reference's collation), a uniform batch;
  full       a uniform batch at the full capacity N x M.
Each is one GraphedTrainStep replay with ClippedAdam inside (labels outside), d = 256, 9 stages, 4 heads, 20 Sinkhorn iterations,
tf32x3.  The three forms alternate in one process; CUDA events around `iters` replays, medians of `rounds` rounds.  Prints one
JSON object with the GPU's name and power limit beside the numbers.

    python tools/padded_train_timing.py [--batch 4] [--capacity 2048] [--iters 20] [--rounds 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import statistics

import torch

from gpu_timing import card, rounds_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--capacity', type=int, default=2048)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('padded_train_timing needs a CUDA device')
    from openglue_b200 import SuperGlue
    from openglue_b200.optim import ClippedAdam
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
    from openglue_b200.training import GraphedTrainStep
    dev = torch.device('cuda:0')
    B, N = args.batch, args.capacity
    g = torch.Generator().manual_seed(args.seed)
    n0 = torch.randint(N // 2, N + 1, (B,), generator=g)
    n1 = torch.randint(N // 2, N + 1, (B,), generator=g)
    cfg = default_config(descriptor_dim=256, num_stages=9, num_heads=4, num_iters=20)
    cfg['precision'] = 'tf32x3'
    full = synthetic_pairs(B, N, N, 256, 1, family='planted', seed=args.seed)
    full.pop('planted_matches0', None)
    full = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in full.items()}
    gt0 = torch.randint(-2, N, (B, N), generator=g).to(dev)
    gt1 = torch.randint(-2, N, (B, N), generator=g).to(dev)
    keys = ('keypoints', 'side_info', 'local_descriptors')
    padded = dict(full, num_keypoints0=n0, num_keypoints1=n1)
    y_padded = {'gt_matches0': gt0, 'gt_matches1': gt1, 'num_keypoints0': n0, 'num_keypoints1': n1}
    a, b = int(n0.min()), int(n1.min())
    trimmed = dict(full, **{f'{k}0': full[f'{k}0'][:, :a].contiguous() for k in keys}, **{f'{k}1': full[f'{k}1'][:, :b].contiguous() for k in keys})
    y_trimmed = {'gt_matches0': gt0[:, :a].clamp(max=b - 1).contiguous(), 'gt_matches1': gt1[:, :b].clamp(max=a - 1).contiguous()}
    y_full = {'gt_matches0': gt0, 'gt_matches1': gt1}
    forms = {}
    for name, (data, y) in {'padded': (padded, y_padded), 'min_stack': (trimmed, y_trimmed), 'full': (full, y_full)}.items():
        model = SuperGlue(cfg)
        model.load_state_dict(synthetic_state_dict(cfg, seed=1), strict=True)
        model = model.to(dev).train()
        step = GraphedTrainStep(model, data, y, optimizer=ClippedAdam(model.parameters(), lr=1e-4))
        forms[name] = (lambda s=step, d=data, yy=y: s(d, yy))
        for _ in range(3):
            forms[name]()
    ms = rounds_ms(forms, args.iters, args.rounds)
    res = {'card': card(), 'batch': B, 'capacity': N, 'lengths0': n0.tolist(), 'lengths1': n1.tolist(),
           'kept_keypoints': {'padded': int(n0.sum() + n1.sum()), 'min_stack': B * (a + b), 'full': 2 * B * N},
           'config': 'd 256, 9 stages, 4 heads, 20 Sinkhorn iterations, tf32x3, GraphedTrainStep + ClippedAdam',
           'ms_per_iteration_median': {k: statistics.median(v) for k, v in ms.items()}, 'ms_per_iteration_rounds': ms}
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
