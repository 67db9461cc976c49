"""Time the kornia SIFT front-end (openglue_b200.SIFT, max_keypoints 1024) per image at B = 1 and B = 16 on a 960 x 720 texture:
``forward``, ``extract_padded``, and for comparison the float32 restatement of kornia (oracle/kornia_sift_oracle.py, run on CUDA
tensors: a stand-in for what the reference does with kornia on a GPU, not kornia itself).  CUDA events around warm-up-excluded
repetitions; prints the card's name and power limit from the same run.

    python tools/kornia_sift_timing.py [--reps 10] [--oracle-reps 2]
"""
from __future__ import annotations

import argparse
import json

import torch

from gpu_timing import card, events_ms  # first: it makes the package and the oracle importable
from openglue_b200 import SIFT
from oracle import kornia_sift_oracle as KO


def texture(B, H, W, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.zeros(B, 1, H, W, device=dev)
    for s in (4, 16, 64):
        n = torch.rand(B, 1, H // s + 2, W // s + 2, generator=g, device=dev)
        x += torch.nn.functional.interpolate(n, size=(H, W), mode='bicubic', align_corners=False) * (s / 64.0)
    return (x / x.amax()).clamp(0, 1)


def oracle_forward(img, nf):
    resp, lafs = KO.detect(img, nf)
    lafs = KO.laf_orienter(lafs, img, 19)
    return lafs, resp, KO.laf_descriptors(img, lafs, 41)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--oracle-reps', type=int, default=2)
    args = ap.parse_args()
    dev = 'cuda:0'
    sift = SIFT(max_keypoints=1024)
    rows = []
    for B in (1, 16):
        img = texture(B, 720, 960, 7, dev)
        t_fwd = events_ms(lambda: sift(img), args.reps, warmup=2)
        t_pad = events_ms(lambda: sift.extract_padded(img), args.reps, warmup=2)
        with torch.no_grad():
            t_or = events_ms(lambda: oracle_forward(img, 1024), args.oracle_reps, warmup=1) if B == 1 else None
        rows.append(dict(B=B, forward_ms_per_image=t_fwd / B, extract_padded_ms_per_image=t_pad / B,
                         oracle_f32_cuda_ms_per_image=None if t_or is None else t_or / B))
        print(json.dumps(rows[-1]))
    print(json.dumps(dict(card=card(), image='960x720', max_keypoints=1024, rows=rows)))


if __name__ == '__main__':
    main()
