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
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from sift_timing import gpu_info  # noqa: E402

B, CAP, D, STAGES, ITERS = 16, 2048, 256, 9, 100


def length_sets():
    g = torch.Generator().manual_seed(0)
    uniform = (torch.randint(1024, CAP + 1, (B,), generator=g), torch.randint(1024, CAP + 1, (B,), generator=g))
    skew0, skew1 = torch.randint(128, 513, (B,), generator=g), torch.randint(128, 513, (B,), generator=g)
    skew0[0] = skew1[0] = CAP
    return {'uniform_1024_2048': uniform, 'skewed': (skew0, skew1)}


def time_ms(fn, iters: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    rounds = []
    for _ in range(3):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(iters):
            fn()
        ev[1].record()
        ev[1].synchronize()
        rounds.append(ev[0].elapsed_time(ev[1]) / iters)
    return statistics.median(rounds)


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
    info = dict(gpu_info(), precision=args.precision, batch=B, capacity=CAP, descriptor_dim=D, stages=STAGES, sinkhorn_iters=ITERS,
                iters=args.iters)
    eager = MatchingCore(model)
    graphed = MatchingCore(model, use_cuda_graph=True)
    graphed.max_graphs = 2 * B + 2                       # one graph per pair shape at B = 1, and the batches

    print(json.dumps(dict(info, mode='uniform_full_capacity_eager', ms=time_ms(lambda: eager(full), args.iters, args.warmup))), flush=True)
    print(json.dumps(dict(info, mode='uniform_full_capacity_graph', ms=time_ms(lambda: graphed(full), args.iters, args.warmup))), flush=True)
    for name, (n0, n1) in length_sets().items():
        padded = dict(full, num_keypoints0=n0, num_keypoints1=n1)
        pairs = [{k: (v[b:b + 1, :(n0 if k.endswith('0') else n1)[b]] if torch.is_tensor(v) else v) for k, v in full.items()}
                 for b in range(B)]
        res = {'padded_eager': time_ms(lambda: eager(padded), args.iters, args.warmup),
               'padded_graph': time_ms(lambda: graphed(padded), args.iters, args.warmup),
               'one_at_a_time_eager': time_ms(lambda: [eager(p) for p in pairs], args.iters, args.warmup),
               'one_at_a_time_graph': time_ms(lambda: [graphed(p) for p in pairs], args.iters, args.warmup)}
        for mode, ms in res.items():
            print(json.dumps(dict(info, lengths=name, mean_n=float(n0.float().mean()), mean_m=float(n1.float().mean()), mode=mode, ms=ms)),
                  flush=True)


if __name__ == '__main__':
    main()
