"""Mint golden vectors for the homography-pretraining pairs (openglue_b200.synthesize_homography_pairs) by running the UNMODIFIED
reference ``data.oxford_paris_dataset.OxfordParis1MDataset.__getitem__`` (data/oxford_paris_dataset.py:27-66) with cv2 4.13.

TEST INFRASTRUCTURE.  Runs only where the reference is checked out; outputs are committed under tests/golden/hg_*.pt.
  - albumentations is not installed here: its ``Compose`` is stubbed to the identity (the colour augmentation is random and is
    not part of the GPU path), and the fixtures say so in their ``reference`` string;
  - ``np.random.randint`` is patched to hand out the case's corner offsets (the call's arguments are checked);
  - every image is written as a lossless PNG already at ``resize_shape``, so ``cv2.imread`` returns it unchanged and the
    INTER_AREA resize is an identity copy (asserted on every call).
The images are regenerated from a seed by ``pair_images`` (integer arithmetic only, bit-identical on every CPU); the fixture
records their sha256, which the tests check.

Stored: the corner offsets, ``H_true`` as the reference's float32 tensor and as cv2's float64, and ``image0`` / ``image1`` as uint8
gray (round(image * 255), exact: every value is k / 255).  For the pretraining size, the per-pair sha256 of the two uint8 images and
a few of their rows instead of the images.

    python oracle/gen_golden_homography.py [case ...]
"""
from __future__ import annotations

import glob
import hashlib
import os
import sys
import tempfile
import types
from unittest import mock

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))

CASES = {
    # name: (batch, resize_shape (W, H), offset, offsets ('random' | 'zero' | 'low' | 'high' | 'fold'), seed, store_full)
    'hg_pretrain': (4, (1472, 1232), 256, 'random', 31, False),      # config/homography_pretraining.yaml: 1472 x 1232, offset 256
    'hg_odd': (3, (37, 40), 8, 'random', 32, True),                  # odd width, W not a multiple of 4, below one 64-column block
    'hg_wide': (3, (98, 64), 16, 'random', 33, True),                # non-square, two column blocks
    'hg_tall': (2, (50, 133), 10, 'random', 34, True),               # taller than wide, W % 4 == 2
    'hg_zero': (2, (70, 52), 12, 'zero', 35, True),                  # H_true = identity, image1 = image0
    'hg_low': (2, (66, 46), 9, 'low', 36, True),                     # every corner at -offset
    'hg_high': (2, (66, 46), 9, 'high', 37, True),                   # every corner at offset - 1
    'hg_fold': (4, (40, 36), 14, 'fold', 38, True),                  # folded corners: samples outside the image, partial border blends
}
ROWS = (0, 1, 359, 360, 718, 719)                                    # rows of the pretraining-size crops stored in full


def pair_images(batch: int, H: int, W: int, seed: int) -> torch.Tensor:
    """[batch, H, W, 3] uint8 RGB with texture at several scales: 4 x 4 blocks of uniform colour, a 3 x 3 box blur, +-8 noise.
    Integer arithmetic only, so every CPU regenerates the same bytes from the seed."""
    g = torch.Generator().manual_seed(seed)
    coarse = torch.randint(0, 256, (batch, H // 4 + 3, W // 4 + 3, 3), generator=g, dtype=torch.int64)
    big = coarse.repeat_interleave(4, 1).repeat_interleave(4, 2)[:, :H + 2, :W + 2]
    blur = sum(big[:, dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)) // 9
    noise = torch.randint(-8, 9, (batch, H, W, 3), generator=g, dtype=torch.int64)
    return (blur + noise).clamp(0, 255).to(torch.uint8).contiguous()


def case_offsets(kind: str, batch: int, offset: int, seed: int) -> torch.Tensor:
    """[batch, 4, 2] int32 corner offsets (x, y) in [-offset, offset)"""
    g = torch.Generator().manual_seed(seed + 1000)
    if kind == 'random':
        return torch.randint(-offset, offset, (batch, 4, 2), generator=g, dtype=torch.int32)
    if kind == 'zero':
        return torch.zeros(batch, 4, 2, dtype=torch.int32)
    if kind == 'low':
        return torch.full((batch, 4, 2), -offset, dtype=torch.int32)
    if kind == 'high':
        return torch.full((batch, 4, 2), offset - 1, dtype=torch.int32)
    if kind == 'fold':
        # corners pushed across the crop (the crop is narrower than 2 offset): the source quadrilateral is concave or crossed,
        # the homography's horizon crosses the crop and part of it samples outside the image, some of it one pixel across the
        # border.  Pairs 0 and 1 were picked (for offset 14) from draws that blend partially with the border; pair 2 is the
        # crop turned by 180 degrees.
        o = torch.randint(-offset, offset, (batch, 4, 2), generator=g, dtype=torch.int32)
        o[0] = torch.tensor([[3, 1], [1, 12], [-7, 8], [4, -14]])
        o[1] = torch.tensor([[-12, 10], [-14, 1], [-12, -6], [-1, -3]])
        o[2] = torch.tensor([[offset - 1, offset - 1], [offset - 1, -offset], [-offset, offset - 1], [-offset, -offset]])
        return o
    raise ValueError(kind)


def images_sha256(images: torch.Tensor) -> str:
    return hashlib.sha256(images.contiguous().numpy().tobytes()).hexdigest()


def u8(image: torch.Tensor) -> torch.Tensor:
    """[1, h, w] float k / 255 -> [h, w] uint8 k (exact)"""
    return torch.round(image[0].double() * 255.0).to(torch.uint8)


def _dataset_class():
    import numpy as np  # noqa: F401
    sys.path.insert(0, os.environ.get('OPENGLUE_REFERENCE', '/root/reference'))
    alb = types.ModuleType('albumentations')                           # colour augmentation: identity

    class Compose:
        def __init__(self, transforms):
            pass

        def __call__(self, image):
            return {'image': image}

    alb.Compose = Compose
    alb.RandomBrightnessContrast = alb.ColorJitter = alb.GaussNoise = lambda *a, **k: None
    sys.modules['albumentations'] = alb
    from gen_golden import _stub_modules
    _stub_modules()
    import importlib.util
    path = os.path.join(os.environ.get('OPENGLUE_REFERENCE', '/root/reference'), 'data', 'oxford_paris_dataset.py')
    spec = importlib.util.spec_from_file_location('oxford_paris_dataset', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)                                       # the reference, unmodified
    return mod


def mint(name, out_dir):
    import cv2
    import numpy as np
    mod = _dataset_class()
    batch, (W, H), offset, kind, seed, full = CASES[name]
    images = pair_images(batch, H, W, seed)
    offsets = case_offsets(kind, batch, offset, seed)
    fx = {'name': name, 'case': dict(batch=batch, H=H, W=W, offset=offset, kind=kind, seed=seed), 'sha256': images_sha256(images),
          'warp_offset': offsets, 'H_true': [], 'H_true_f64': [],
          'reference': 'data/oxford_paris_dataset.py:27-66 OxfordParis1MDataset.__getitem__ with albumentations Compose stubbed to '
                       'the identity (no colour augmentation), cv2 ' + cv2.__version__ + ', torch ' + torch.__version__}
    real_resize = cv2.resize

    def resize(img, dsize, interpolation=None):
        out = real_resize(img, dsize, interpolation=interpolation)
        assert out.shape == img.shape and np.array_equal(out, img), 'the INTER_AREA resize must be an identity copy here'
        return out

    real_gpt = cv2.getPerspectiveTransform
    fits = []

    def gpt(src, dst, *a):
        M = real_gpt(src, dst, *a)
        fits.append(M)
        return M

    img0, img1 = [], []
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, 'scene'))
        for b in range(batch):
            path = os.path.join(tmp, 'scene', f'{b:03d}.jpg')              # the dataset globs *.jpg; the bytes are a PNG
            ok, buf = cv2.imencode('.png', cv2.cvtColor(images[b].numpy(), cv2.COLOR_RGB2BGR))
            assert ok
            with open(path, 'wb') as f:
                f.write(buf.tobytes())
        ds = mod.OxfordParis1MDataset(__import__('pathlib').Path(tmp), resize_shape=(W, H), offset=offset)
        ds.images_list = sorted(glob.glob(os.path.join(tmp, 'scene', '*.jpg')))
        assert len(ds) == batch
        for b in range(batch):
            want = offsets[b].numpy().astype(np.int64)

            def randint(low, high=None, size=None, dtype=int, _want=want):
                assert (low, high, tuple(size)) == (-offset, offset, (4, 2))
                return _want.copy()

            fits.clear()
            with mock.patch.object(mod.np.random, 'randint', randint), mock.patch.object(mod.cv2, 'resize', resize), \
                    mock.patch.object(mod.cv2, 'getPerspectiveTransform', gpt):
                item = ds[b]
            assert item['transformation']['type'] == 'perspective'
            # every homography came from a successful LU solve (cv2 4.13 falls back to an SVD otherwise: M[8] != 1)
            assert all(M[2, 2] == 1.0 for M in fits), f'{name}[{b}]: cv2 left its LU path'
            fx['H_true'].append(item['transformation']['H'])
            fx['H_true_f64'].append(torch.from_numpy(fits[1].copy()))
            img0.append(u8(item['image0']))
            img1.append(u8(item['image1']))
            assert torch.equal(img0[-1].float() / 255., item['image0'][0]) and torch.equal(img1[-1].float() / 255., item['image1'][0])
            if kind == 'fold':                                               # the border enters: count the samples it touches
                bw = cv2.warpPerspective(images[b].numpy(), fits[0], (W, H), borderValue=(255, 255, 255))
                b0 = cv2.warpPerspective(images[b].numpy(), fits[0], (W, H))
                crop = (slice(offset, H - offset), slice(offset, W - offset))
                d = (bw[crop].astype(int) - b0[crop].astype(int))
                fx.setdefault('border_samples', []).append(int((d != 0).any(-1).sum()))
                fx.setdefault('partial_border_samples', []).append(int(((d > 0) & (d < 255)).any(-1).sum()))
    fx['H_true'] = torch.stack(fx['H_true'])
    fx['H_true_f64'] = torch.stack(fx['H_true_f64'])
    img0, img1 = torch.stack(img0), torch.stack(img1)
    if full:
        fx['image0'], fx['image1'] = img0, img1
    else:
        fx['image0_sha256'] = [images_sha256(t) for t in img0]
        fx['image1_sha256'] = [images_sha256(t) for t in img1]
        fx['rows'] = ROWS
        fx['image0_rows'] = img0[:, list(ROWS)].clone()
        fx['image1_rows'] = img1[:, list(ROWS)].clone()
    if kind == 'zero':
        assert torch.equal(img0, img1) and all(torch.equal(h, torch.eye(3)) for h in fx['H_true'])
    if kind == 'fold':
        assert sum(fx['partial_border_samples']) > 0, 'no partial border blend in the folded case'
    torch.save(fx, os.path.join(out_dir, name + '.pt'))
    extra = f', border samples {fx["border_samples"]}, partial {fx["partial_border_samples"]}' if kind == 'fold' else ''
    print(f'{name}: {batch} x {H} x {W}, offset {offset} -> {tuple(img0.shape)}{extra}')


def main():
    out_dir = os.path.join(ROOT, 'tests', 'golden')
    only = sys.argv[1:]
    for name in CASES:
        if not only or name in only:
            mint(name, out_dir)


if __name__ == '__main__':
    main()
