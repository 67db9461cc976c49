"""kornia SIFT front-end without a GPU: the float32 oracle against its float64 form stage by stage, the committed fixtures against
the unmodified reference (where it is checked out), the oracle against kornia's own modules (where kornia is installed), and the
argument checks of openglue_b200.SIFT and its C entry points."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import kornia_sift_oracle as KO  # noqa: E402
from oracle.gen_golden_kornia_sift import load_fixture  # noqa: E402
from openglue_b200 import SIFT, _cabi  # noqa: E402

REF = os.environ.get('OG_REFERENCE_ROOT', '/root/reference')


def _fx(name):
    return load_fixture(os.path.join(HERE, 'golden', name + '.pt'))


def test_oracle_float32_against_float64_stage_by_stage():
    img = _fx('ksift_tiny')['image']
    p32, s32 = KO.scale_pyramid(img)
    p64, _ = KO.scale_pyramid(img.double())
    assert [p.shape for p in p32] == [(1, 1, 6, 128, 160), (1, 1, 6, 64, 80)]
    # bounds: about 4x what was measured (levels 1.0e-6, responses 5.4e-7, descriptors 2.4e-5, angles 3.2e-7)
    for a, b in zip(p32, p64):
        assert float((a.double() - b).abs().max()) <= 4e-6                     # levels in [0, 1]
        assert float((KO.dog_response(a).double() - KO.dog_response(b)).abs().max()) <= 4e-6
    r32, l32 = KO.detect(img, 256)
    r64, l64 = KO.detect(img.double(), 256)
    assert float((r32.double() - r64).abs().max()) <= 2e-6
    top = r64[0] > 10                                                           # the strict extrema (bonus 10)
    a, b = l64[0][top].flatten(1), l32[0][r32[0] > 10].double().flatten(1)       # near-equal responses may swap ranks
    # sift_tiny's extrema have DoG values near 1e-3, so float32 moves their interpolated LAFs by up to 1e-2 (9.5e-3 measured); one
    # of the 9 sits at the |offset| > 0.7 decision
    close = torch.cdist(a, b).min(1).values <= 2e-2
    assert float(close.float().mean()) >= 0.8
    d32 = KO.laf_descriptors(img, l64[:, :16].float())
    d64 = KO.laf_descriptors(img.double(), l64[:, :16])
    assert float((d32.double() - d64).abs().max()) <= 1e-4
    a32 = KO.laf_orienter(l64[:, :16].float(), img, 19, want_angles=True)[1]
    a64 = KO.laf_orienter(l64[:, :16], img.double(), 19, want_angles=True)[1]
    assert float((a32.double() - a64).abs().max()) <= 1e-5


def test_patch_pyramid_level_float32_against_float64():
    """the level of LAFs at scale 16 2^k (1 + d): float32 and float64 agree away from the boundaries and differ by at most one level
    next to them; the clamp to min(h, w) // 32 - 1 holds in both; the levels are the ones extract_patches_from_pyramid samples"""
    H, W = 160, 171
    d = torch.tensor([-1e-2, -4e-4, -2.0 ** -22, 0.0, 2.0 ** -22, 4e-4, 1e-2], dtype=torch.float64)
    s = (16.0 * 2.0 ** torch.arange(6, dtype=torch.float64)[:, None] * (1 + d)).flatten()
    laf = torch.zeros(1, s.numel(), 2, 3, dtype=torch.float64)
    laf[0, :, 0, 0], laf[0, :, 1, 1], laf[0, :, 0, 2], laf[0, :, 1, 2] = s, s, 80.0, 70.0
    l64 = KO.patch_pyramid_level(laf, H, W, 32).flatten()
    l32 = KO.patch_pyramid_level(laf.float(), H, W, 32).flatten()
    far = (d.abs() >= 4e-4).repeat(6)
    assert torch.equal(l32[far], l64[far]) and int((l32 - l64).abs().max()) <= 1
    assert int(l64.max()) == min(H, W) // 32 - 1 and int(l64.min()) == 0
    k = torch.log2(s / 16).floor().clamp(0, 4).long()                 # the nominal level of each row
    assert torch.equal(l64[far], k[far])
    img = torch.rand(1, 1, H, W, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    p = KO.extract_patches_from_pyramid(img, laf, 32).flatten(2)
    past = l64 >= KO.patch_pyramid_levels(H, W, 32)                    # levels never visited: zero patches
    assert bool(past.any()) and not p[0, past].any() and bool((p[0, ~past].abs().amax(1) > 0).all())


def test_fixture_consistency():
    for name in ['ksift_tiny', 'ksift_small', 'ksift_odd', 'ksift_warp', 'ksift_uniform', 'ksift_pair']:
        fx = _fx(name)
        B = fx['image'].shape[0]
        assert fx['det_resp'].shape == (B, 1024) and fx['det_lafs'].shape == (B, 1024, 2, 3)
        N = fx['lafs'].shape[1]
        assert fx['responses'].shape == (B, N) and fx['descriptors'].shape == (B, N, 128) and fx['sel'].shape == (B, N)
        for b in range(B):
            assert torch.equal(fx['responses'][b], fx['det_resp'][b, fx['sel'][b]])
    assert _fx('ksift_uniform')['lafs'].shape[1] == 0


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, 'models', 'features', 'sift.py')), reason='the reference is not checked out')
def test_the_fixture_script_reproduces_the_committed_fixtures():
    sys.path.insert(0, os.path.join(ROOT, 'oracle'))
    import gen_golden_kornia_sift as G
    SIFTRef = G.import_reference()
    for name in ['ksift_tiny', 'ksift_uniform']:
        got, want = G.mint(name, SIFTRef), torch.load(os.path.join(HERE, 'golden', name + '.pt'))
        for k, v in want.items():
            if torch.is_tensor(v):
                assert torch.equal(got[k], v), (name, k)


def test_oracle_against_kornia():
    """The only pin of the restatement to an execution of kornia: module by module on random inputs."""
    kornia = pytest.importorskip('kornia')
    g = torch.Generator().manual_seed(0)
    img = torch.rand(1, 1, 80, 96, generator=g)
    pyr, _, _ = kornia.geometry.transform.ScalePyramid(3, 1.6, 32, double_image=True)(img)
    mine, _ = KO.scale_pyramid(img)
    for a, b in zip(pyr, mine):
        assert torch.allclose(a, b, atol=1e-6)
    dog = KO.dog_response(mine[0])
    c_k, y_k = kornia.geometry.subpix.ConvQuadInterp3d(10)(dog)
    c_m, y_m = KO.conv_quad_interp3d(dog)
    assert torch.allclose(y_k, y_m, atol=1e-5) and torch.allclose(c_k, c_m, atol=1e-4)
    resp, lafs = kornia.feature.ScaleSpaceDetector(256, resp_module=kornia.feature.BlobDoG(), nms_module=kornia.geometry.subpix.ConvQuadInterp3d(10),
                                                   scale_pyr_module=kornia.geometry.transform.ScalePyramid(3, 1.6, 32, double_image=True),
                                                   ori_module=kornia.feature.PassLAF(), scale_space_response=True, minima_are_also_good=True,
                                                   mr_size=6.0).detect(img, 256)
    r_m, l_m = KO.detect(img, 256)
    assert torch.allclose(resp.sort(descending=True).values, r_m, atol=1e-5)
    patches = torch.rand(8, 1, 41, 41, generator=g)
    assert torch.allclose(kornia.feature.SIFTDescriptor(41, rootsift=True)(patches), KO.sift_descriptor(patches), atol=1e-5)
    p19 = torch.rand(8, 1, 19, 19, generator=g)
    assert torch.equal(kornia.feature.orientation.PatchDominantGradientOrientation(19)(p19), KO.dominant_orientation(p19))
    assert torch.allclose(kornia.feature.extract_patches_from_pyramid(img, l_m[:, :8], 41), KO.extract_patches_from_pyramid(img, l_m[:, :8], 41),
                          atol=1e-6)


def test_arguments_are_checked():
    with pytest.raises(ValueError):
        SIFT(patch_size=32)
    with pytest.raises(ValueError):
        SIFT(descriptor_dim=256)
    with pytest.raises(ValueError):
        SIFT(max_keypoints=10000)
    with pytest.raises(ValueError):
        SIFT(nms_diameter=8)
    s = SIFT(max_keypoints=1024, device=torch.device('cpu')).eval()
    assert (s.max_keypoints, s.descriptor_dim) == (1024, 128)
    with pytest.raises(RuntimeError, match='CUDA'):
        s(torch.rand(1, 1, 64, 64))
    with pytest.raises(RuntimeError, match='CUDA'):
        s.extract_padded(torch.rand(1, 1, 64, 64))
    with pytest.raises(ValueError):
        s(torch.rand(1, 3, 64, 64))
    with pytest.raises(TypeError):
        s(torch.rand(1, 1, 64, 64).numpy())


def test_workspace_queries():
    lib = _cabi.lib()
    assert lib.og_ksift_workspace_bytes(1, 720, 960, 1024) > 0
    assert lib.og_ksift_workspace_bytes(1, 720, 960, 9000) < 0          # above 8192 keypoints
    assert lib.og_ksift_workspace_bytes(0, 720, 960, 1024) < 0
    assert lib.og_ksift_select_workspace_bytes(2, 1024) > 0
    import numpy as np
    out = np.zeros(128, np.int64)
    n = lib.og_ksift_workspace_layout(1, 64, 80, 1024, out.ctypes.data, 128)
    assert out[0] == 2 and tuple(out[1:3]) == (128, 160) and tuple(out[6:8]) == (64, 80)
    assert out[n - 1] == lib.og_ksift_workspace_bytes(1, 64, 80, 1024)
    assert lib.og_ksift_select(None, None, None, 1, 64, 64, 16, 1, 9, 16, 1, None, 0, None, None, None) < 0
