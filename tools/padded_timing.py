"""Time a padded batch (pairs with their own keypoint counts in one call) against the ways to match the same pairs without it:
one pair at a time at B = 1 (eager, and CUDA-graphed with one graph per pair shape), and the uniform batch at the full capacity.
Capacity 16 pairs x 2048 x 2048, descriptor_dim 256, 9 stages, 100 Sinkhorn iterations, MatchingCore (matches only); lengths
from a fixed seed: uniform in [1024, 2048], and a skewed set (one pair at the capacity, the others in [128, 512]).  CUDA events,
the median of three rounds.  Prints one JSON line per measurement, with the GPU's name and power limit.

    python tools/padded_timing.py [--iters 10] [--warmup 2] [--precision fp16x3]
"""
from __future__ import annotations

import argparse
import json
import statistics

import torch

from gpu_timing import card, events_ms

B, CAP, D, STAGES, ITERS = 16, 2048, 256, 9, 100


def length_sets():
    g = torch.Generator().manual_seed(0)
    uniform = (torch.randint(1024, CAP + 1, (B,), generator=g), torch.randint(1024, CAP + 1, (B,), generator=g))
    skew0, skew1 = torch.randint(128, 513, (B,), generator=g), torch.randint(128, 513, (B,), generator=g)
    skew0[0] = skew1[0] = CAP
    return {'uniform_1024_2048': uniform, 'skewed': (skew0, skew1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--precision', default='fp16x3', choices=['fp32', 'tf32x3', 'fp16x3'])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('padded_timing: no CUDA device (the measurement needs the GPU; there is nothing to fall back to)')
    from openglue_b200.superglue import MatchingCore, SuperGlue
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict

    dev = torch.device('cuda', 0)
    cfg = dict(default_config(descriptor_dim=D, num_stages=STAGES, num_iters=ITERS), precision=args.precision)
    model = SuperGlue(cfg).eval()
    model.load_state_dict(synthetic_state_dict(cfg, seed=0))
    model = model.to(dev)
    full = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in synthetic_pairs(B, CAP, CAP, D, 1, seed=1).items()}
    info = dict(card=card(), precision=args.precision, batch=B, capacity=CAP, descriptor_dim=D, stages=STAGES, sinkhorn_iters=ITERS,
                iters=args.iters)
    eager = MatchingCore(model)
    graphed = MatchingCore(model, use_cuda_graph=True)
    graphed.max_graphs = 2 * B + 2                       # one graph per pair shape at B = 1, and the batches

    def report(forms, **what):                           # each form on its own: warm-up, then the median of three rounds
        for mode, fn in forms.items():
            ms = statistics.median([events_ms(fn, args.iters, args.warmup), events_ms(fn, args.iters), events_ms(fn, args.iters)])
            print(json.dumps(dict(info, **what, mode=mode, ms=ms)), flush=True)

    report({'uniform_full_capacity_eager': lambda: eager(full), 'uniform_full_capacity_graph': lambda: graphed(full)})
    for name, (n0, n1) in length_sets().items():
        padded = dict(full, num_keypoints0=n0, num_keypoints1=n1)
        pairs = [{k: (v[b:b + 1, :(n0 if k.endswith('0') else n1)[b]] if torch.is_tensor(v) else v) for k, v in full.items()}
                 for b in range(B)]
        report({'padded_eager': lambda: eager(padded), 'padded_graph': lambda: graphed(padded),
                'one_at_a_time_eager': lambda: [eager(p) for p in pairs], 'one_at_a_time_graph': lambda: [graphed(p) for p in pairs]},
               lengths=name, mean_n=float(n0.float().mean()), mean_m=float(n1.float().mean()))


if __name__ == '__main__':
    main()
