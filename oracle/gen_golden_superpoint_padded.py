"""Mint golden vectors for SuperPoint's padded output (``SuperPointNet.extract_padded``): the UNMODIFIED reference
``models.features.superpoint.model.SuperPointNet.forward`` (model.py:80-129) run on each image of a batch ALONE, so no
``min_stack`` trims an image to the batch's smallest count.  The layer outputs are injected as in gen_golden_superpoint_post.py
(``torch.rand`` draws from a recorded seed, ``post_inputs``), for two ``max_keypoints``: -1 (every keypoint, raster order) and one
that cuts some images of the batch and not others.

TEST INFRASTRUCTURE.  Runs only where the reference is checked out; the output is committed as tests/golden/sp_padded_240.pt.

    python oracle/gen_golden_superpoint_padded.py
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

from gen_golden_superpoint_post import BORDER, desc_subset, inputs_sha256, post_inputs  # noqa: E402

NAME = 'sp_padded_240'
# batch, H, W, nms_kernel, keypoint_threshold, seed; levels 0.  The thresholds differ per image (applied by scaling its scores)
# so the counts spread widely.
CASE = dict(batch=3, h=240, w=320, nms=9, thr=0.005, seed=21)
SCALES = (1.0, 0.00515, 0.00502)     # image b's cell scores times SCALES[b]: the threshold then cuts its NMS survivors
MAXKS = (-1, 500)


def padded_inputs():
    c = CASE
    scores, desc = post_inputs(c['batch'], c['h'], c['w'], c['seed'])
    scores = scores * torch.tensor(SCALES).view(-1, 1, 1, 1)
    return scores, desc


def main():
    from gen_golden import _stub_modules
    from gen_golden_superpoint import REF, nms2d
    sys.path.insert(0, REF)
    _stub_modules()
    import kornia.geometry.subpix as subpix                              # the stub module
    subpix.nms2d = nms2d
    from models.features.superpoint.model import SuperPointNet as RefSuperPoint     # the reference, unmodified
    c = CASE
    scores, desc = padded_inputs()
    fx = {'case': dict(c, border=BORDER, scales=SCALES), 'sha256': inputs_sha256(scores, desc), 'maxk': {},
          'reference': 'models/features/superpoint/model.py:80-129 per image (kornia nms2d restated), torch ' + torch.__version__}
    for maxk in MAXKS:
        model = RefSuperPoint(max_keypoints=maxk, nms_kernel=c['nms'], remove_borders_size=BORDER, keypoint_threshold=c['thr']).eval()
        per = []
        for b in range(c['batch']):
            model._forward_layers = lambda image, mask=None, b=b: (desc[b:b + 1], scores[b:b + 1])
            with torch.no_grad():
                lafs, kp_scores, descriptors = model(torch.zeros(1, 1, c['h'], c['w']))
            kpts = lafs[0, :, :, 2].contiguous()
            kp16 = kpts.to(torch.int16)
            assert torch.equal(kp16.float(), kpts)                       # pixel positions, exactly
            idx = desc_subset(kpts, c['h'], c['w'])
            per.append({'keypoints': kp16, 'scores': kp_scores[0].contiguous(), 'desc_idx': idx, 'descriptors': descriptors[0, idx].contiguous()})
        fx['maxk'][maxk] = per
        print(f'{NAME} max_keypoints {maxk}: keypoints per image {[p["keypoints"].shape[0] for p in per]}')
    torch.save(fx, os.path.join(ROOT, 'tests', 'golden', NAME + '.pt'))


if __name__ == '__main__':
    main()
