"""Time the OpenCV SIFT front-end (openglue_b200.OpenCVSIFT: OPENCV_SIFT with max_keypoints 2048, nms_diameter 9, RootSIFT) on a
960 x 720 image, with CUDA events, at batch 1 (forward) and batch 16 (extract_batch), and - when cv2 and the reference checkout
are present - the reference's detect_and_compute on the host cores.  Prints one JSON line per measurement, with the GPU's name
and power limit.

    python tools/sift_timing.py [--iters 20] [--warmup 3] [--reference /path/to/reference]
"""
from __future__ import annotations

import argparse
import json
import os
import time

import numpy as np
import torch

from gpu_timing import card, events_ms


def image(seed: int, H: int = 720, W: int = 960) -> torch.Tensor:
    """a smooth multi-scale texture in [0, 1]: [1, 1, H, W]"""
    g = torch.Generator().manual_seed(seed)
    x = sum(torch.nn.functional.interpolate(torch.rand(1, 1, H // s, W // s, generator=g), size=(H, W), mode='bicubic', align_corners=False) * s
            for s in (6, 24, 96))
    x = torch.nn.functional.avg_pool2d(x, 5, 1, 2)
    return ((x - x.min()) / (x.max() - x.min())).clamp(0, 1)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reference', default=os.environ.get('OG_REFERENCE_ROOT', '/root/reference'))
    a = ap.parse_args()
    if torch.cuda.is_available():
        from openglue_b200 import OpenCVSIFT
        info = {'card': card()}
        m = OpenCVSIFT(max_keypoints=2048, nms_diameter=9., rootsift=True)
        one = image(0).cuda()
        batch = torch.cat([image(s) for s in range(16)]).cuda()
        n = m(one)[1].shape[1]
        ms1 = events_ms(lambda: m(one), a.iters, a.warmup)
        print(json.dumps({'what': 'OpenCVSIFT.forward', 'batch': 1, 'H': 720, 'W': 960, 'keypoints': n, 'ms_per_image': round(ms1, 3), **info}))
        ms16 = events_ms(lambda: m.extract_batch(batch), max(2, a.iters // 4), 1)
        print(json.dumps({'what': 'OpenCVSIFT.extract_batch', 'batch': 16, 'H': 720, 'W': 960, 'ms_per_image': round(ms16 / 16, 3), **info}))
    else:
        print(json.dumps({'what': 'OpenCVSIFT', 'gpu': 'not measured (no CUDA device)'}))
    try:
        import cv2  # noqa: F401
        os.environ['OG_REFERENCE_ROOT'] = a.reference
        from gen_golden_sift import import_reference
        sift_create, _ = import_reference()
    except Exception as e:                                     # noqa: BLE001
        print(json.dumps({'what': 'reference detect_and_compute', 'cpu': f'not measured ({type(e).__name__})'}))
        return
    feats = sift_create(max_keypoints=2048, nms_diameter=9., rootsift=True)
    u8 = (255. * image(0)[0, 0].numpy()).astype(np.uint8)
    feats.detect_and_compute(u8)
    t = []
    for _ in range(max(3, a.iters // 4)):
        t0 = time.perf_counter()
        feats.detect_and_compute(u8)
        t.append(time.perf_counter() - t0)
    print(json.dumps({'what': 'reference detect_and_compute (host CPU)', 'batch': 1, 'ms_per_image': round(1e3 * float(np.median(t)), 1),
                      'cpu_threads': cv2.getNumThreads(), 'cpus': os.cpu_count()}))


if __name__ == '__main__':
    main()
