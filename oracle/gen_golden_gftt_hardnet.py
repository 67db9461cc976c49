"""Mint golden vectors for the GFTT / AffNet / HardNet front-end (openglue_b200.GFTTAffNetHardNet) by running the UNMODIFIED
reference ``models/features/hardnet.py`` and ``models/features/base.py`` (config/features_online/gftt_affnet_hardnet.yaml).

TEST INFRASTRUCTURE.  Runs only where the reference is checked out; outputs are committed under tests/golden/gftt_*.pt.  kornia
is not installed: the two files are loaded by path under a stub package, and every ``kornia.*`` name they import is the
restatement in oracle/kornia_gftt_oracle.py (kornia 0.6.3).  The reference's wiring, constructor arguments, ``run_nms`` and
min-stack are therefore executed, not restated.  The networks carry the seeded synthetic weights (the pretrained checkpoints
are not available offline); they are regenerated from the stored seeds, not stored.

Images are the committed OpenCV SIFT fixtures' (tests/golden/sift_{tiny,small,odd,warp,uniform}.npz).  Stored per case (config:
max_keypoints 1024, nms_diameter 9, upright False):
  image_u8     uint8 [B, 1, H, W]   the images; ``load_fixture`` adds ``image``, the float32 input ``image_u8 / 255.``
  det_resp     [B, 1024]        the detector's responses (bonus included)
  det_lafs     [B, 1024, 2, 3]  its LAFs, before AffNet
  aff_lafs     [B, 1024, 2, 3]  AffNet's LAFs of every detection
  angles       [B, 1024]        LAFOrienter's dominant orientation (radians) of every AffNet LAF
  sel          [B, N] int64     which detector output each output row is (run_nms's selection, min-stacked)
  lafs, responses              the reference's outputs [B, N, 2, 3], [B, N]
  descriptors  float16 [B, N, 128]
  affnet_seed, hardnet_seed, affnet_sha256, hardnet_sha256   the synthetic weights

    python oracle/gen_golden_gftt_hardnet.py
"""
from __future__ import annotations

import importlib
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
REF_ROOT = os.environ.get('OG_REFERENCE_ROOT', '/root/reference')
sys.path.insert(0, ROOT)

from oracle import kornia_gftt_oracle as KG  # noqa: E402
from oracle import kornia_sift_oracle as KO  # noqa: E402
from oracle.gen_golden_kornia_sift import load_images, to_input  # noqa: E402

MAX_KEYPOINTS, NMS_DIAMETER = 1024, 9
CASES = {                                   # name: the sift_*.npz images of the batch
    'gftt_tiny': ['sift_tiny'],
    'gftt_small': ['sift_small'],
    'gftt_odd': ['sift_odd'],
    'gftt_warp': ['sift_warp'],
    'gftt_uniform': ['sift_uniform'],
    'gftt_pair': ['sift_small', 'sift_warp'],           # a two-image batch: run_nms's min-stack
}


def import_reference():
    """The reference's ``GFTTAffNetHardNet`` class, its kornia imports resolved to the restatement."""
    mods = {
        'kornia': {}, 'kornia.feature': dict(LAFDescriptor=KG.LAFDescriptor),
        'kornia.feature.affine_shape': dict(LAFAffNetShapeEstimator=KG.LAFAffNetShapeEstimator),
        'kornia.feature.scale_space_detector': dict(ScaleSpaceDetector=KG.ScaleSpaceDetector),
        'kornia.feature.orientation': dict(LAFOrienter=KG.LAFOrienter, PassLAF=KG.PassLAF),
        'kornia.feature.responses': dict(CornerGFTT=KG.CornerGFTT),
        'kornia.geometry': {}, 'kornia.geometry.subpix': dict(ConvQuadInterp3d=KG.ConvQuadInterp3d, nms2d=KO.nms2d),
        'kornia.geometry.transform': dict(ScalePyramid=KG.ScalePyramid),
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
        return importlib.import_module('_ref_features.hardnet').GFTTAffNetHardNet
    finally:                                  # the stubs stand in for kornia only while the reference files import
        for name, m in saved.items():
            if m is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = m


def load_fixture(path: str) -> dict:
    """a gftt_*.pt fixture with its float32 input ``image`` (stored as uint8 to keep the fixtures small)"""
    fx = torch.load(path)
    fx['image'] = to_input(fx['image_u8'])
    return fx


def mint(name, GFTTAffNetHardNet):
    img_u8 = load_images(CASES[name])
    img = to_input(img_u8)
    feats = GFTTAffNetHardNet(descriptor_dim=128, max_keypoints=MAX_KEYPOINTS, nms_diameter=NMS_DIAMETER).eval()
    with torch.no_grad():
        lafs, resp, desc = feats(img)
    call = feats.detector.calls[-1]
    det_lafs, det_resp, aff_lafs = call['det_lafs'], call['det_resp'], call['aff_lafs']
    oriented, angles = KO.laf_orienter(aff_lafs, img, 19, want_angles=True)
    # which detector output each output row is: its oriented LAF and response name it uniquely
    sel = []
    for b in range(img.shape[0]):
        key = {oriented[b, j].numpy().tobytes() + det_resp[b, j].numpy().tobytes(): j for j in range(det_resp.shape[1])}
        sel.append([key[lafs[b, i].numpy().tobytes() + resp[b, i].numpy().tobytes()] for i in range(resp.shape[1])])
    return dict(image_u8=img_u8, det_resp=det_resp, det_lafs=det_lafs, aff_lafs=aff_lafs, angles=angles,
                sel=torch.tensor(sel, dtype=torch.int64).view(img.shape[0], -1), lafs=lafs, responses=resp, descriptors=desc.half(),
                affnet_seed=KG.AFFNET_SEED, hardnet_seed=KG.HARDNET_SEED,
                affnet_sha256=KG.state_dict_checksum(KG.synthetic_affnet_state_dict(KG.AFFNET_SEED)),
                hardnet_sha256=KG.state_dict_checksum(KG.synthetic_hardnet_state_dict(KG.HARDNET_SEED)),
                reference='models/features/hardnet.py + base.py (unmodified), kornia 0.6.3 restated by oracle/kornia_gftt_oracle.py, torch '
                          + torch.__version__)


def main():
    cls = import_reference()
    only = sys.argv[1:]
    for name in CASES:
        if only and name not in only:
            continue
        fx = mint(name, cls)
        torch.save(fx, os.path.join(GOLDEN, name + '.pt'))
        print(f'{name}: image {tuple(fx["image_u8"].shape)}, {fx["responses"].shape[1]} keypoints')


if __name__ == '__main__':
    main()
