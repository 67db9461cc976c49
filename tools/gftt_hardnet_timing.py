"""Time the GFTT / AffNet / HardNet front-end (openglue_b200.GFTTAffNetHardNet, max_keypoints 1024, synthetic weights) per image at
B = 1 and B = 16 on a 960 x 720 texture: ``forward``, ``extract_padded``, the share of ``forward`` the two patch CNNs take (the
time saved when their GEMMs are skipped), and for comparison the float32 restatement of kornia (oracle/kornia_gftt_oracle.py, run
on CUDA tensors: a stand-in for what the reference does with kornia on a GPU, not kornia itself).  CUDA events around
warm-up-excluded repetitions; prints the card's name and power limit from the same run.

    python tools/gftt_hardnet_timing.py [--reps 10] [--oracle-reps 2]
"""
from __future__ import annotations

import argparse
import json

import torch

from gpu_timing import card, events_ms  # first: it makes the package and the oracle importable
from kornia_sift_timing import texture
from openglue_b200 import GFTTAffNetHardNet
from openglue_b200 import _patch_cnn as PC
from oracle import kornia_gftt_oracle as KG


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--oracle-reps', type=int, default=2)
    args = ap.parse_args()
    dev = 'cuda:0'
    w = {'affnet': KG.synthetic_affnet_state_dict(), 'hardnet': KG.synthetic_hardnet_state_dict()}
    fe = GFTTAffNetHardNet(max_keypoints=1024, weights=w)
    rows = []
    for B in (1, 16):
        img = texture(B, 720, 960, 7, dev)
        t_fwd = events_ms(lambda: fe(img), args.reps, warmup=2)
        t_pad = events_ms(lambda: fe.extract_padded(img), args.reps, warmup=2)
        cnn = PC.run_cnn
        PC.run_cnn = lambda ops, layers, x, rows, convs, col, acts, out: out     # everything but the CNN GEMMs and im2col
        t_rest = events_ms(lambda: fe(img), args.reps, warmup=2)
        PC.run_cnn = cnn
        with torch.no_grad():
            t_or = events_ms(lambda: KG.run(img, 1024), args.oracle_reps, warmup=1) if B == 1 else None
        rows.append(dict(B=B, forward_ms_per_image=t_fwd / B, extract_padded_ms_per_image=t_pad / B, cnn_share=1 - t_rest / t_fwd,
                         oracle_f32_cuda_ms_per_image=None if t_or is None else t_or / B))
        print(json.dumps(rows[-1]))
    print(json.dumps(dict(card=card(), image='960x720', max_keypoints=1024, rows=rows)))


if __name__ == '__main__':
    main()
