"""Mint golden vectors for the kornia SIFT front-end (openglue_b200.SIFT) by running the UNMODIFIED reference
``models/features/sift.py`` and ``models/features/base.py`` (the ``SIFT`` features of config/features_online/sift.yaml).

TEST INFRASTRUCTURE.  Runs only where the reference is checked out; outputs are committed under tests/golden/ksift_*.pt.  kornia
is not installed: the two files are loaded by path under a stub package, and every ``kornia.*`` name they import is the
restatement in oracle/kornia_sift_oracle.py (kornia 0.6.3).  The reference's wiring, constructor arguments, ``run_nms`` and
min-stack are therefore executed, not restated.

Images are the committed OpenCV SIFT fixtures' (tests/golden/sift_{tiny,small,odd,warp,uniform}.npz), as ``image / 255.`` in
float32.  Stored per case (config: max_keypoints 1024, nms_diameter 9, rootsift, upright False):
  image_u8     uint8 [B, 1, H, W]   the images; ``load_fixture`` adds ``image``, the float32 input ``image_u8 / 255.``
  det_resp     [B, 1024]        the detector's responses (ScaleSpaceDetector.detect, bonus included)
  det_lafs     [B, 1024, 2, 3]  its LAFs before orientation
  angles       [B, 1024]        LAFOrienter's dominant orientation (radians) of every detector LAF
  sel          [B, N] int64     which detector output each output row is (run_nms's selection, min-stacked)
  lafs, responses              the reference's outputs [B, N, 2, 3], [B, N]
  descriptors  float16 [B, N, 128]

    python oracle/gen_golden_kornia_sift.py
"""
from __future__ import annotations

import importlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
REF_ROOT = os.environ.get('OG_REFERENCE_ROOT', '/root/reference')
sys.path.insert(0, ROOT)

from oracle import kornia_sift_oracle as KO  # noqa: E402

MAX_KEYPOINTS, NMS_DIAMETER = 1024, 9
CASES = {                                   # name: the sift_*.npz images of the batch
    'ksift_tiny': ['sift_tiny'],
    'ksift_small': ['sift_small'],
    'ksift_odd': ['sift_odd'],
    'ksift_warp': ['sift_warp'],
    'ksift_uniform': ['sift_uniform'],
    'ksift_pair': ['sift_small', 'sift_warp'],           # a two-image batch: run_nms's min-stack
}


def import_reference():
    """The reference's ``SIFT`` class, its kornia imports resolved to the restatement."""
    mods = {
        'kornia': {}, 'kornia.feature': dict(LAFDescriptor=KO.LAFDescriptor),
        'kornia.feature.scale_space_detector': dict(ScaleSpaceDetector=KO.ScaleSpaceDetector),
        'kornia.feature.orientation': dict(LAFOrienter=KO.LAFOrienter, PassLAF=KO.PassLAF),
        'kornia.geometry': {}, 'kornia.geometry.subpix': dict(ConvQuadInterp3d=KO.ConvQuadInterp3d, nms2d=KO.nms2d),
        'kornia.geometry.transform': dict(ScalePyramid=KO.ScalePyramid),
        'kornia.feature.responses': dict(BlobDoG=KO.BlobDoG, CornerGFTT=KO.CornerGFTT),
        'kornia.feature.siftdesc': dict(SIFTDescriptor=KO.SIFTDescriptor),
    }
    saved = {name: sys.modules.get(name) for name in mods}
    for name, attrs in mods.items():
        m = types.ModuleType(name)
        m.__path__ = []
        m.__dict__.update(attrs)
        sys.modules[name] = m
    pkg = types.ModuleType('_ref_features')
    pkg.__path__ = [os.path.join(REF_ROOT, 'models', 'features')]
    sys.modules['_ref_features'] = pkg
    try:
        return importlib.import_module('_ref_features.sift').SIFT
    finally:                                  # the stubs stand in for kornia only while the reference files import
        for name, m in saved.items():
            if m is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = m


def load_images(names):
    """uint8 [B, 1, H, W] of the named sift_*.npz fixtures"""
    return torch.from_numpy(np.stack([np.load(os.path.join(GOLDEN, n + '.npz'))['image'] for n in names])[:, None])


def to_input(images_u8: torch.Tensor) -> torch.Tensor:
    """the float32 image the reference runs on: ``image / 255.`` in float64, rounded to float32"""
    return torch.from_numpy(images_u8.numpy().astype(np.float64) / 255.).float()


def load_fixture(path: str) -> dict:
    """a ksift_*.pt fixture with its float32 input ``image`` (stored as uint8 to keep the fixtures small)"""
    fx = torch.load(path)
    fx['image'] = to_input(fx['image_u8'])
    return fx


def mint(name, SIFT):
    img_u8 = load_images(CASES[name])
    img = to_input(img_u8)
    feats = SIFT(descriptor_dim=128, max_keypoints=MAX_KEYPOINTS, nms_diameter=NMS_DIAMETER, rootsift=True).eval()
    with torch.no_grad():
        lafs, resp, desc = feats(img)
    call = feats.detector.calls[-1]
    det_lafs, det_resp = call['det_lafs'], call['det_resp']
    oriented, angles = KO.laf_orienter(det_lafs, img, 19, want_angles=True)
    # which detector output each output row is: its oriented LAF and response name it uniquely
    sel = []
    for b in range(img.shape[0]):
        key = {oriented[b, j].numpy().tobytes() + det_resp[b, j].numpy().tobytes(): j for j in range(det_resp.shape[1])}
        sel.append([key[lafs[b, i].numpy().tobytes() + resp[b, i].numpy().tobytes()] for i in range(resp.shape[1])])
    return dict(image_u8=img_u8, det_resp=det_resp, det_lafs=det_lafs, angles=angles, sel=torch.tensor(sel, dtype=torch.int64).view(img.shape[0], -1),
                lafs=lafs, responses=resp, descriptors=desc.half(),
                reference='models/features/sift.py + base.py (unmodified), kornia 0.6.3 restated by oracle/kornia_sift_oracle.py, torch ' + torch.__version__)


def main():
    SIFT = import_reference()
    only = sys.argv[1:]
    for name in CASES:
        if only and name not in only:
            continue
        fx = mint(name, SIFT)
        torch.save(fx, os.path.join(GOLDEN, name + '.pt'))
        print(f'{name}: image {tuple(fx["image_u8"].shape)}, {fx["responses"].shape[1]} keypoints')


if __name__ == '__main__':
    main()
