"""Mint golden vectors for the OpenCV SIFT front-end (openglue_b200.OpenCVSIFT) by running the UNMODIFIED reference
``models/features/opencv/base.py`` and ``_features.py`` (``sift_create``: ``cv2.SIFT_create(contrastThreshold=-10000,
edgeThreshold=-10000)``, radius NMS, top-k, RootSIFT, LAFs) with cv2 4.13 on the host CPU.

TEST INFRASTRUCTURE.  Runs only where the reference is checked out and cv2 is installed; outputs are committed under
tests/golden/sift_*.npz.  The two reference files need only cv2, numpy and scipy; the package ``__init__`` pulls in kornia, so
the files are loaded by path under a stub package and the ``__init__`` never runs.

Images are deterministic synthetic uint8 textures (``make_image``: numpy's PCG64 from a fixed seed, plus cv2 resizes / blurs /
a perspective warp, all stored in the fixture, so nothing has to regenerate them bit for bit).  Stored per image:
  image                   uint8 [H, W]
  kp_pt, kp_size, kp_angle, kp_response, kp_octave
                          cv2's raw keypoints of ``detectAndCompute`` (cv2's order: x, y, size desc, angle, ...)
  desc_raw                uint8 [N, 128]  cv2's raw descriptors (integer-valued float32 in cv2: lossless as uint8)
  ref_lafs, ref_scores, ref_index
                          the reference's ``detect_and_compute`` outputs (max_keypoints 2048, nms_diameter 9, rootsift:
                          config/features/sift_opencv.yaml), in its (argpartition) order.  Its descriptors are stored as
                          ref_index, the raw keypoint each output is: they equal the reference's ``normalize_descriptors`` of
                          ``desc_raw[ref_index]`` bit for bit (asserted while minting; ``ref_descriptors`` rebuilds them)
and sift_atan.npz holds a ``cv2.fastAtan2`` table (y, x, angle in degrees).

    python oracle/gen_golden_sift.py
"""
from __future__ import annotations

import importlib
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
REF_ROOT = os.environ.get('OG_REFERENCE_ROOT', '/root/reference')

# name: (H, W, kind, seed, final blur sigma)
CASES = {
    'sift_tiny': (64, 80, 'noise', 1, 0.0),
    'sift_small': (240, 320, 'mixed', 2, 0.0),
    'sift_odd': (375, 500, 'grating', 3, 1.2),          # neither side a multiple of 8
    'sift_vga': (720, 960, 'mixed', 4, 4.5),
    'sift_warp': (240, 320, 'warp', 2, 0.0),            # a homography of sift_small's texture
    'sift_uniform': (96, 128, 'uniform', 5, 0.0),       # no extremum: zero keypoints
}
MAX_KEYPOINTS, NMS_DIAMETER, ROOTSIFT = 2048, 9.0, True


def import_reference():
    """(sift_create, nms_keypoints) from the reference files, loaded by path under a stub package."""
    d = os.path.join(REF_ROOT, 'models', 'features', 'opencv')
    pkg = types.ModuleType('_ref_opencv')
    pkg.__path__ = [d]
    sys.modules['_ref_opencv'] = pkg
    feats = importlib.import_module('_ref_opencv._features')
    base = importlib.import_module('_ref_opencv.base')
    return feats.sift_create, base.nms_keypoints


def make_image(H: int, W: int, kind: str, seed: int, blur: float = 0.0) -> np.ndarray:
    import cv2
    rng = np.random.default_rng(seed)
    if kind == 'uniform':
        return np.full((H, W), 117, np.uint8)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    img = np.zeros((H, W))
    for s in (6, 24, 96):                                            # multi-scale noise
        n = rng.random((H // s + 2, W // s + 2))
        img += cv2.resize(n, (W, H), interpolation=cv2.INTER_CUBIC) * (s / 96.0) * 60
    if kind in ('grating', 'mixed'):
        for f, a in ((0.07, 0.3), (0.19, 1.1)):
            img += 25 * np.sin(2 * np.pi * f * (xx * np.cos(a) + yy * np.sin(a)))
    if kind in ('mixed', 'noise'):
        for _ in range(max(4, H * W // 3000)):                        # Gaussian blobs of both signs
            cy, cx, r, amp = rng.random() * H, rng.random() * W, 1.5 + rng.random() * 10, rng.choice([-1, 1]) * (30 + 60 * rng.random())
            img += amp * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r))
    img += rng.normal(0, 1, (H, W))
    if blur > 0:                                                     # a smoother texture: fewer fine-scale extrema
        img = cv2.GaussianBlur(img, (0, 0), blur)
    img = np.clip(img + 40, 0, 255).astype(np.uint8)
    return img


def warp_image(img: np.ndarray, seed: int) -> np.ndarray:
    import cv2
    H, W = img.shape
    rng = np.random.default_rng(seed + 100)
    src = np.float32([[0, 0], [W, 0], [W, H], [0, H]])
    dst = src + rng.uniform(-0.12, 0.12, (4, 2)).astype(np.float32) * np.float32([W, H])
    M = cv2.getPerspectiveTransform(src, dst)
    return cv2.warpPerspective(img, M, (W, H), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT)


def mint(name: str, sift_create) -> dict:
    import cv2
    H, W, kind, seed, blur = CASES[name]
    img = warp_image(make_image(H, W, 'mixed', seed), seed) if kind == 'warp' else make_image(H, W, kind, seed, blur)
    sift = cv2.SIFT_create(contrastThreshold=-10000, edgeThreshold=-10000)
    kpts, desc = sift.detectAndCompute(img, None)
    n = len(kpts)
    out = dict(image=img,
               kp_pt=np.array([k.pt for k in kpts], np.float32).reshape(n, 2),
               kp_size=np.array([k.size for k in kpts], np.float32),
               kp_angle=np.array([k.angle for k in kpts], np.float32),
               kp_response=np.array([k.response for k in kpts], np.float32),
               kp_octave=np.array([k.octave for k in kpts], np.int32),
               desc_raw=(np.zeros((0, 128), np.uint8) if desc is None else desc.astype(np.uint8)))
    if desc is not None:
        assert np.array_equal(out['desc_raw'].astype(np.float32), desc), 'cv2 descriptors are integer-valued'
        feats = sift_create(max_keypoints=MAX_KEYPOINTS, nms_diameter=NMS_DIAMETER, rootsift=ROOTSIFT)
        lafs, scores, d = feats.detect_and_compute(img)
        # which raw keypoint each output is: the reference's own LAF of every raw keypoint, with its response, names it uniquely
        raw_lafs = feats.lafs_from_opencv_kpts(kpts, mr_size=feats.laf_scale_mr_size)
        key = {raw_lafs[j].tobytes() + out['kp_response'][j].tobytes(): j for j in range(n)}
        assert len(key) == n
        index = np.array([key[lafs[i].astype(np.float32).tobytes() + np.float32(scores[i]).tobytes()] for i in range(len(scores))], np.int32)
        # the descriptors are then the reference's normalisation of those raw descriptors: stored as the index, checked here bit for bit
        assert np.array_equal(feats.normalize_descriptors(desc[index], ROOTSIFT).view(np.int32), d.astype(np.float32).view(np.int32))
        out.update(ref_lafs=lafs.astype(np.float32), ref_scores=scores.astype(np.float32), ref_index=index)
    else:                                                    # the reference fails here (descriptors is None): nothing to store
        out.update(ref_lafs=np.zeros((0, 2, 3), np.float32), ref_scores=np.zeros(0, np.float32), ref_index=np.zeros(0, np.int32))
    return out


def ref_descriptors(fx: dict) -> np.ndarray:
    """The reference's output descriptors of a fixture: ``OpenCVFeatures.normalize_descriptors(desc_raw[ref_index], root_norm=True)``
    restated with the same numpy operations (the minting asserts the two agree bit for bit)."""
    d = fx['desc_raw'][fx['ref_index']].astype(np.float32)
    d /= np.linalg.norm(d, ord=1, axis=1, keepdims=True)
    return np.sqrt(d)


def atan_table() -> dict:
    import cv2
    rng = np.random.default_rng(7)
    y = (rng.integers(-300, 301, 6000) * rng.random(6000)).astype(np.float32)
    x = (rng.integers(-300, 301, 6000) * rng.random(6000)).astype(np.float32)
    ints = np.arange(-4, 5, dtype=np.float32)                    # the axes, the diagonals, 0 / 0
    gy, gx = np.meshgrid(ints, ints, indexing='ij')
    y, x = np.concatenate([y, gy.ravel(), [1.0]]).astype(np.float32), np.concatenate([x, gx.ravel(), [2.0]]).astype(np.float32)
    a = np.array([cv2.fastAtan2(float(v), float(u)) for v, u in zip(y, x)], np.float32)
    return dict(y=y, x=x, angle=a)


def main() -> None:
    sift_create, _ = import_reference()
    os.makedirs(GOLDEN, exist_ok=True)
    for name in CASES:
        fx = mint(name, sift_create)
        np.savez_compressed(os.path.join(GOLDEN, name + '.npz'), **fx)
        print(f'{name}: {fx["image"].shape} {len(fx["kp_size"])} raw keypoints, {len(fx["ref_scores"])} selected')
    np.savez_compressed(os.path.join(GOLDEN, 'sift_atan.npz'), **atan_table())


if __name__ == '__main__':
    main()
