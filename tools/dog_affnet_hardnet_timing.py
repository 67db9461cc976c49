"""Time the DoG / AffNet / OriNet / HardNet front-end (openglue_b200.DoGOpenCVAffNetHardNet, max_keypoints 2048, synthetic weights)
per image on a 960 x 720 texture: ``forward`` at B = 1 (the reference takes one image), ``extract_batch`` at B = 16,
``extract_padded`` at both, the share of the time the three patch CNNs take (the time saved when their im2col and GEMMs are
skipped), and for comparison the float32 restatement of kornia (oracle/dog_affnet_oracle.py, run on CUDA tensors: a stand-in for
what the reference does with kornia on a GPU, not kornia itself) on the same selected keypoints, plus cv2's SIFT detection on the
host when cv2 is importable.  CUDA events around warm-up-excluded repetitions; prints the card's name and power limit from the
same run.

    python tools/dog_affnet_hardnet_timing.py [--reps 10] [--oracle-reps 2]
"""
from __future__ import annotations

import argparse
import json
import time

import torch

from gpu_timing import card, events_ms  # first: it makes the package and the oracle importable
from kornia_sift_timing import texture
from openglue_b200 import DoGOpenCVAffNetHardNet
from openglue_b200 import _patch_cnn as PC
from oracle import dog_affnet_oracle as KD
from oracle import kornia_gftt_oracle as KG

NF = 2048


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--oracle-reps', type=int, default=2)
    args = ap.parse_args()
    dev = 'cuda:0'
    w = {'affnet': KG.synthetic_affnet_state_dict(), 'orinet': KD.synthetic_orinet_state_dict(), 'hardnet': KG.synthetic_hardnet_state_dict()}
    fe = DoGOpenCVAffNetHardNet(max_keypoints=NF, weights=w)
    rows = []
    for B in (1, 16):
        img = texture(B, 720, 960, 7, dev)
        run = (lambda: fe(img)) if B == 1 else (lambda: fe.extract_batch(img))
        n = [int(t[0].shape[1]) for t in fe.extract_batch(img)]
        t_fwd = events_ms(run, args.reps, warmup=2)
        t_pad = events_ms(lambda: fe.extract_padded(img, NF), args.reps, warmup=2)
        cnn = PC.run_cnn
        PC.run_cnn = lambda ops, layers, x, rows, convs, col, acts, out: acts[1] if out is None else out   # all but the CNNs
        t_rest = events_ms(run, args.reps, warmup=2)
        PC.run_cnn = cnn
        row = dict(B=B, keypoints_per_image=sum(n) / B, forward_ms_per_image=t_fwd / B, extract_padded_ms_per_image=t_pad / B,
                   cnn_share=1 - t_rest / t_fwd)
        if B == 1:
            det = fe._detect_select(img, True)
            kp1 = det.kp[0, det.sel[0, :int(det.n_sel[0])].long()][None].contiguous()
            with torch.no_grad():
                row['oracle_f32_cuda_describe_ms'] = events_ms(lambda: KD.describe(img, kp1), args.oracle_reps, warmup=1)
            try:
                import cv2
                u8 = (img[0, 0].cpu().numpy() * 255).astype('uint8')
                sift = cv2.SIFT_create(contrastThreshold=-10000, edgeThreshold=-10000)
                sift.detect(u8, None)
                t0 = time.perf_counter()
                for _ in range(args.oracle_reps):
                    sift.detect(u8, None)
                row['cv2_host_detect_ms'] = (time.perf_counter() - t0) * 1e3 / args.oracle_reps
            except ImportError:
                row['cv2_host_detect_ms'] = None
        rows.append(row)
        print(json.dumps(row))
    print(json.dumps(dict(card=card(), image='960x720', max_keypoints=NF, rows=rows)))


if __name__ == '__main__':
    main()
