"""Time the reference's training iteration after labels, in two forms, alternating them in one process:
  (a) GraphedTrainStep replay, then torch's clip_grad_norm_(params, 10) -> Adam.step() -> StepLR.step() eagerly (Lightning's loop);
  (b) GraphedTrainStep(optimizer=ClippedAdam) replay: the whole iteration in one graph.
and the optimiser alone: ClippedAdam.step() (eager, and replayed from a CUDA graph) against torch's eager foreach sequence.

Shape of the reference's config_cached_sp_magicleap.yaml: d = 256, 9 stages, 4 heads, 20 Sinkhorn iterations, 1024 keypoints,
batch 4 (the config) and 2.  Prints one JSON object with the GPU's name and power limit beside the numbers.

    python tools/train_step_timing.py [--batches 4 2] [--iters 20] [--rounds 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics

import torch

from gpu_timing import card, rounds_ms


def _labels(pairs, dev):
    gt0 = pairs['planted_matches0'].to(torch.int64)
    B, n = gt0.shape
    m = pairs['keypoints1'].shape[1]
    gt1 = torch.full((B, m), -1, dtype=torch.int64)
    for b in range(B):
        idx = torch.nonzero(gt0[b] >= 0).flatten()
        gt1[b, gt0[b, idx]] = idx
    return {'gt_matches0': gt0.to(dev), 'gt_matches1': gt1.to(dev)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, nargs='+', default=[4, 2])
    ap.add_argument('--keypoints', type=int, default=1024)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('train_step_timing needs a CUDA device')
    from openglue_b200 import ClippedAdam, SuperGlue
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
    from openglue_b200.training import GraphedTrainStep
    dev = torch.device('cuda:0')
    cfg = default_config(descriptor_dim=256, num_stages=9, num_heads=4, num_iters=20)
    sd = synthetic_state_dict(cfg, seed=0)
    res = {'card': card(), 'config': 'd=256, 9 stages, 4 heads, 20 Sinkhorn iterations, tf32x3 training GEMMs',
           'keypoints': args.keypoints, 'iters': args.iters, 'rounds': args.rounds, 'train_step': {}, 'optimizer_alone': {}}

    def model():
        m = SuperGlue(dict(cfg, precision='tf32x3'))
        m.load_state_dict(copy.deepcopy(sd))
        return m.to(dev).train()

    for B in args.batches:
        pairs = synthetic_pairs(B, args.keypoints, args.keypoints, 256, 1, family='planted', seed=7)
        y_true = _labels(pairs, dev)
        data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in pairs.items()}
        ma, mb = model(), model()
        pa = list(ma.parameters())
        adam = torch.optim.Adam(pa, lr=1e-4)
        sched = torch.optim.lr_scheduler.StepLR(adam, step_size=1, gamma=0.999994)
        step_a = GraphedTrainStep(ma, data, y_true)
        step_b = GraphedTrainStep(mb, data, y_true, optimizer=ClippedAdam.from_config(mb, {'lr': 1e-4, 'grad_clip': 10.0,
                                                                                                'scheduler_gamma': 0.999994}))

        def form_a():
            step_a(data, y_true)
            torch.nn.utils.clip_grad_norm_(pa, 10.0)
            adam.step()
            sched.step()

        def form_b():
            step_b(data, y_true)

        for f in (form_a, form_b):
            for _ in range(3):
                f()
        ta, tb = rounds_ms({'a': form_a, 'b': form_b}, args.iters, args.rounds).values()
        res['train_step'][f'B={B}'] = {'a_graph_plus_eager_torch_optimizer_ms': ta, 'b_graph_with_clipped_adam_ms': tb,
                                       'median_a_ms': statistics.median(ta), 'median_b_ms': statistics.median(tb)}
        del step_a, step_b, ma, mb, adam, sched, pa
        torch.cuda.empty_cache()

    # the optimiser alone, on the default model's 11,957,249 parameters with gradients of norm ~5 (the unclipped regime)
    m0, m1 = model(), model()
    n = sum(p.numel() for p in m0.parameters())
    g = torch.Generator(device=dev).manual_seed(0)
    for p, q in zip(m0.parameters(), m1.parameters()):
        p.grad = torch.randn(p.shape, device=dev, generator=g) * (5.0 / n ** 0.5)
        q.grad = p.grad.clone()
    p0 = list(m0.parameters())
    adam = torch.optim.Adam(p0, lr=1e-4)
    sched = torch.optim.lr_scheduler.StepLR(adam, step_size=1, gamma=0.999994)
    ours = ClippedAdam(m1.parameters())

    def torch_seq():
        torch.nn.utils.clip_grad_norm_(p0, 10.0)
        adam.step()
        sched.step()

    ours.step()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ours.step()
    for f in (torch_seq, ours.step, graph.replay):
        for _ in range(3):
            f()
    tt, to, tg = rounds_ms({'torch': torch_seq, 'eager': ours.step, 'graph': graph.replay}, args.iters * 5, args.rounds).values()
    hbm = 36 * n                                        # norm pass 4 B + fused pass 32 B per parameter (from shapes)
    res['optimizer_alone'] = {'parameters': n, 'torch_foreach_clip_adam_steplr_ms': tt, 'clipped_adam_eager_ms': to,
                              'clipped_adam_graph_replay_ms': tg, 'bytes_per_step': hbm,
                              'clipped_adam_graph_GBps': hbm / (statistics.median(tg) * 1e-3) / 1e9}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
