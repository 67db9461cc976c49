"""Time images -> matches for B pairs of 960 x 720 images, three ways, with SIFT (max_keypoints 2048) and SuperPoint (1024):
  pairwise  OpenGlueMatcher, one pair at a time (the reference's inference loop; each call reads counts back to the host);
  eager     ImagePairMatcher(use_cuda_graph=False): the batch through extract_padded, the padded matcher and the match
            extraction, without a host synchronisation;
  graph     ImagePairMatcher(use_cuda_graph=True): the same chain replayed as one CUDA graph (borrowed outputs).
Every form ends in matches0 / matching_scores0 on the device (the compact list is not built).  SuperGlue: d = 128 (SIFT) or 256
(SuperPoint), 9 stages, 4 heads, 100 Sinkhorn iterations, fp16x3; synthetic weights.  Images: bicubic-upsampled noise.
CUDA events around `iters` calls, medians of `rounds` rounds, the forms alternating in one process.  Prints one JSON object with
the GPU's name and power limit beside the numbers (ms per batch and per pair).

    python tools/image_matching_timing.py [--batches 1 4 16] [--iters 5] [--rounds 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import statistics

import torch

from gpu_timing import card, rounds_ms


def _images(B, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    low = torch.rand(B, 1, 72, 96, generator=g, device=dev)
    img = torch.nn.functional.interpolate(low, size=(744, 984), mode='bicubic', align_corners=False).clamp(0, 1)
    return img[:, :, :720, :960].contiguous(), img[:, :, 24:, 24:].contiguous()      # two views shifted by (24, 24)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, nargs='+', default=[1, 4, 16])
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('image_matching_timing needs a CUDA device')
    from gen_golden_superpoint import synthetic_superpoint_state_dict
    from openglue_b200 import OpenCVSIFT, SuperGlue, SuperPointNet
    from openglue_b200.features import ImagePairMatcher, OpenGlueMatcher
    from openglue_b200.synthetic import default_config, synthetic_state_dict
    dev = torch.device('cuda:0')
    mc = {'superglue': {'laf_to_sideinfo_method': 'none'}, 'inference': {'match_threshold': 0.2}}
    result = {'card': card(), 'iters': args.iters, 'rounds': args.rounds, 'image': [720, 960], 'results': []}
    for name in ('sift', 'superpoint'):
        if name == 'sift':
            fe, D = OpenCVSIFT(max_keypoints=2048), 128
        else:
            fe, D = SuperPointNet(max_keypoints=1024, keypoint_threshold=0.005), 256
            fe.load_state_dict(synthetic_superpoint_state_dict(7), strict=True)
            fe = fe.to(dev).eval()
        cfg = default_config(descriptor_dim=D, num_stages=9, num_heads=4, num_iters=100)
        sg = SuperGlue(cfg)
        sg.load_state_dict(synthetic_state_dict(cfg, seed=1), strict=True)
        sg = sg.to(dev).eval()
        pairwise = OpenGlueMatcher(fe, sg, mc)
        eager = ImagePairMatcher(fe, sg, mc, use_cuda_graph=False)
        graph = ImagePairMatcher(fe, sg, mc, use_cuda_graph=True)
        for B in args.batches:
            i0, i1 = _images(B, B, dev)
            if name == 'sift':
                i0, i1 = (255 * i0).round().to(torch.uint8), (255 * i1).round().to(torch.uint8)
            forms = {
                'pairwise': lambda: [pairwise({'image0': i0[b:b + 1], 'image1': i1[b:b + 1]}) for b in range(B)],
                'eager': lambda: eager(i0, i1),
                'graph': lambda: graph(i0, i1, borrow=True),
            }
            for fn in forms.values():                                          # warm-up (and the one capture)
                fn()
            out = eager(i0, i1)
            counts = (out['num_keypoints0'].tolist(), out['num_keypoints1'].tolist())
            times = rounds_ms(forms, args.iters, args.rounds)
            row = {'features': name, 'batch': B, 'keypoints0': counts[0], 'keypoints1': counts[1],
                   'overflow': int(out['overflow0'].sum() + out['overflow1'].sum())}
            for k, v in times.items():
                row[f'{k}_ms'] = round(statistics.median(v), 3)
                row[f'{k}_ms_per_pair'] = round(statistics.median(v) / B, 3)
                row[f'{k}_rounds_ms'] = [round(x, 3) for x in v]
            result['results'].append(row)
            print(json.dumps(row), flush=True)
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
