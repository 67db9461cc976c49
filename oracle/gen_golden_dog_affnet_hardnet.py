"""Mint golden vectors for the DoG / AffNet / OriNet / HardNet front-end (openglue_b200.DoGOpenCVAffNetHardNet) by running the
UNMODIFIED reference ``models/features/opencv/dog_affnet_harnet.py`` and ``models/features/opencv/base.py``
(config/features/dog_opencv_affnet_hardnet.yaml) with the installed cv2 and scipy.

TEST INFRASTRUCTURE.  Runs only where the reference, cv2 and scipy are present; outputs are committed under tests/golden/dogaff_*.pt.
kornia and kornia_moons are not installed: the two files are loaded by path under a stub package, and every ``kornia``,
``kornia.feature`` and ``kornia_moons.feature`` name they use is the restatement in oracle/dog_affnet_oracle.py.  The reference's
wiring, cv2 detection, KDTree NMS and top-k are therefore executed, not restated.  The networks carry the seeded synthetic weights
(the pretrained checkpoints are not available offline); they are regenerated from the stored seeds, not stored.

Images are the committed OpenCV SIFT fixtures' (tests/golden/sift_{tiny,small,odd,warp,uniform}.npz), one per case: the reference
takes B = 1.  Stored per case (config: max_keypoints 2048, nms_diameter 9), rows in the reference's (argpartition) order:
  image_u8     uint8 [1, 1, H, W]   the image; ``load_fixture`` adds ``image``, the float32 input ``image_u8 / 255.``
  kp           [1, N, 5]        the selected cv2 keypoints (x, y, size, angle, response)
  moons_lafs   [1, N, 2, 3]     laf_from_opencv_SIFT_kpts
  aff_lafs     [1, N, 2, 3]     AffNet's LAFs
  angles       [1, N]           OriNet's angles (radians) on the AffNet LAFs
  lafs, scores                 the reference's outputs [1, N, 2, 3], [1, N]
  descriptors  float16 [1, N, 128]
  affnet_seed, orinet_seed, hardnet_seed and their sha256, cv2_version
``sift_uniform`` has no keypoints, where the reference fails (scipy's KDTree of an empty array): that case stores N = 0 and
``reference_fails=True`` instead of a reference run.

    python oracle/gen_golden_dog_affnet_hardnet.py
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

from oracle import dog_affnet_oracle as KD  # noqa: E402
from oracle import kornia_gftt_oracle as KG  # noqa: E402
from oracle.gen_golden_kornia_sift import load_images, to_input  # noqa: E402

MAX_KEYPOINTS, NMS_DIAMETER = 2048, 9
CASES = {'dogaff_tiny': 'sift_tiny', 'dogaff_small': 'sift_small', 'dogaff_odd': 'sift_odd', 'dogaff_warp': 'sift_warp',
         'dogaff_uniform': 'sift_uniform'}


def import_reference():
    """The reference's ``DoGOpenCVAffNetHardNet`` class, its kornia and kornia_moons imports resolved to the restatement."""
    mods = {
        'kornia': dict(tensor_to_image=KD.tensor_to_image, image_to_tensor=KD.image_to_tensor),
        'kornia.feature': dict(HardNet=KD.HardNet, LAFAffNetShapeEstimator=KD.LAFAffNetShapeEstimator, LAFOrienter=KD.LAFOrienter,
                               OriNet=KD.OriNet, extract_patches_from_pyramid=KD.extract_patches_from_pyramid),
        'kornia_moons': {}, 'kornia_moons.feature': dict(laf_from_opencv_SIFT_kpts=KD.laf_from_opencv_SIFT_kpts),
    }
    saved = {name: sys.modules.get(name) for name in mods}
    for name, attrs in mods.items():
        m = types.ModuleType(name)
        m.__path__ = []
        m.__dict__.update(attrs)
        sys.modules[name] = m
    sys.modules['kornia'].feature = sys.modules['kornia.feature']
    sys.modules['kornia_moons'].feature = sys.modules['kornia_moons.feature']
    pkg = types.ModuleType('_ref_opencv_features')          # the package's own __init__ (which imports the others) is not run
    pkg.__path__ = [os.path.join(REF_ROOT, 'models', 'features', 'opencv')]
    sys.modules['_ref_opencv_features'] = pkg
    try:
        return importlib.import_module('_ref_opencv_features.dog_affnet_harnet').DoGOpenCVAffNetHardNet
    finally:                                  # the stubs stand in for kornia only while the reference files import
        for name, m in saved.items():
            if m is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = m


def load_fixture(path: str) -> dict:
    """a dogaff_*.pt fixture with its float32 input ``image`` (stored as uint8 to keep the fixtures small)"""
    fx = torch.load(path)
    fx['image'] = to_input(fx['image_u8'])
    return fx


def mint(name, DoGOpenCVAffNetHardNet):
    import cv2
    img_u8 = load_images([CASES[name]])
    img = to_input(img_u8)
    feats = DoGOpenCVAffNetHardNet(max_keypoints=MAX_KEYPOINTS, nms_diameter=float(NMS_DIAMETER)).eval()
    fx = dict(image_u8=img_u8, affnet_seed=KG.AFFNET_SEED, orinet_seed=KD.ORINET_SEED, hardnet_seed=KG.HARDNET_SEED,
              affnet_sha256=KG.state_dict_checksum(KG.synthetic_affnet_state_dict(KG.AFFNET_SEED)),
              orinet_sha256=KG.state_dict_checksum(KD.synthetic_orinet_state_dict(KD.ORINET_SEED)),
              hardnet_sha256=KG.state_dict_checksum(KG.synthetic_hardnet_state_dict(KG.HARDNET_SEED)),
              cv2_version=cv2.__version__, reference_fails=False,
              reference='models/features/opencv/dog_affnet_harnet.py + base.py (unmodified), cv2 ' + cv2.__version__
                        + ', kornia 0.6.3 and kornia_moons restated by oracle/dog_affnet_oracle.py, torch ' + torch.__version__)
    quantised = (KD.tensor_to_image(img) * 255).astype('uint8')
    if len(feats.features.detect(quantised, None)) == 0:
        e = torch.zeros(1, 0, 2, 3)
        fx.update(reference_fails=True, kp=torch.zeros(1, 0, 5), moons_lafs=e, aff_lafs=e, angles=torch.zeros(1, 0), lafs=e,
                  scores=torch.zeros(1, 0), descriptors=torch.zeros(1, 0, 128, dtype=torch.float16))
        return fx
    captured = {}
    mod = sys.modules[DoGOpenCVAffNetHardNet.__module__]
    detect = mod.detect_kpts_opencv

    def spy(*a, **k):                       # the selected cv2 keypoints, as the reference receives them
        kpts, scores = detect(*a, **k)
        captured['kp'] = torch.tensor([[k_.pt[0], k_.pt[1], k_.size, k_.angle, k_.response] for k_ in kpts], dtype=torch.float32)
        return kpts, scores
    mod.detect_kpts_opencv = spy
    try:
        with torch.no_grad():
            lafs, scores, desc = feats(img)
    finally:
        mod.detect_kpts_opencv = detect
    aff, ori = feats.affnet.calls[-1], feats.orinet.calls[-1]
    fx.update(kp=captured['kp'][None], moons_lafs=aff['lafs_in'], aff_lafs=aff['lafs_out'], angles=ori['angles'], lafs=lafs,
              scores=scores.float(), descriptors=desc.half())
    return fx


def main():
    cls = import_reference()
    only = sys.argv[1:]
    for name in CASES:
        if only and name not in only:
            continue
        fx = mint(name, cls)
        torch.save(fx, os.path.join(GOLDEN, name + '.pt'))
        print(f'{name}: image {tuple(fx["image_u8"].shape)}, {fx["lafs"].shape[1]} keypoints')


if __name__ == '__main__':
    main()
