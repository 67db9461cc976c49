"""Host-side checks of the padded front-end outputs and ImagePairMatcher: arguments are refused before any kernel launch, and the
new C entry points reject null pointers and bad sizes with OG_EINVAL without touching a GPU."""
import pytest
import torch

from openglue_b200 import OpenCVSIFT, SuperGlue, SuperPointNet, SuperPointNetBn, _cabi
from openglue_b200.features import ImagePairMatcher, padded_capacity
from openglue_b200.synthetic import default_config

MC = {'superglue': {'laf_to_sideinfo_method': 'none'}, 'inference': {'match_threshold': 0.2}}


def test_padded_capacity():
    assert padded_capacity(1024) == 1024 and padded_capacity(1024, 300) == 300 and padded_capacity(-1, 5) == 5
    with pytest.raises(ValueError, match='needs a capacity'):
        padded_capacity(-1)
    for bad in (0, -3):
        with pytest.raises(ValueError, match='at least 1'):
            padded_capacity(-1, bad)
    with pytest.raises(ValueError, match='at least 1'):
        padded_capacity(0)


@pytest.mark.parametrize('cls', [SuperPointNet, SuperPointNetBn])
def test_superpoint_extract_padded_refuses_before_any_launch(cls):
    """CPU tensors reach no kernel: each refusal below comes first, so it is the one raised"""
    img = torch.zeros(2, 1, 64, 80)
    with pytest.raises(ValueError, match='needs a capacity'):
        cls(max_keypoints=-1).extract_padded(img)
    with pytest.raises(ValueError, match='at least 1'):
        cls(max_keypoints=512).extract_padded(img, 0)
    for shape in ((2, 1, 60, 80), (2, 1, 64, 84), (2, 3, 64, 80), (64, 80)):
        with pytest.raises(ValueError, match='multiples of 8'):
            cls(max_keypoints=512).extract_padded(torch.zeros(shape))
    with pytest.raises(RuntimeError, match='CUDA'):
        cls(max_keypoints=512).extract_padded(img)


def test_sift_extract_padded_refuses_before_any_launch():
    img = torch.zeros(2, 1, 64, 80, dtype=torch.uint8)
    with pytest.raises(ValueError, match='needs a capacity'):
        OpenCVSIFT().extract_padded(img)
    with pytest.raises(ValueError, match='at least 1'):
        OpenCVSIFT(max_keypoints=100).extract_padded(img, 0)
    with pytest.raises(ValueError, match=r'\[B, 1, H, W\]'):
        OpenCVSIFT(max_keypoints=100).extract_padded(torch.zeros(2, 3, 64, 80))
    with pytest.raises(RuntimeError, match='CUDA'):
        OpenCVSIFT(max_keypoints=100).extract_padded(img)


def _superglue(d=128):
    return SuperGlue(default_config(descriptor_dim=d, num_heads=4, num_stages=1, num_iters=5)).eval()


def test_image_pair_matcher_refuses_before_any_launch():
    with pytest.raises(TypeError, match='SuperGlue'):
        ImagePairMatcher(OpenCVSIFT(max_keypoints=100), torch.nn.Identity(), MC)
    with pytest.raises(TypeError, match='extract_padded'):
        ImagePairMatcher(torch.nn.Identity(), _superglue(), MC)
    with pytest.raises(NameError):
        ImagePairMatcher(OpenCVSIFT(max_keypoints=100), _superglue(), {'superglue': {'laf_to_sideinfo_method': 'shape'}, 'inference': {}})
    m = ImagePairMatcher(OpenCVSIFT(max_keypoints=100), _superglue(), MC)
    a, b = torch.zeros(2, 1, 64, 80), torch.zeros(3, 1, 64, 80)
    with pytest.raises(ValueError, match='same number of images'):
        m(a, b)
    with pytest.raises(ValueError, match=r'image1 must be \[B, 1, H, W\]'):
        m(a, torch.zeros(2, 64, 80))
    with pytest.raises(ValueError, match='needs a capacity'):
        ImagePairMatcher(OpenCVSIFT(), _superglue(), MC)(a, a)
    with pytest.raises(ValueError, match='at least 1'):
        ImagePairMatcher(OpenCVSIFT(), _superglue(), MC, capacity=0)(a, a)
    with pytest.raises(RuntimeError, match='CUDA'):
        m(a, a)


def test_new_entry_points_reject_bad_arguments():
    lib = _cabi.lib()
    buf = torch.zeros(64, dtype=torch.int32)
    p = _cabi.ptr(buf)
    EINVAL = -1
    # og_keypoint_counts(count, B, cap, max_keypoints, K, n_out, mode, overflow, stream)
    assert lib.og_keypoint_counts(None, 2, 10, -1, 5, p, p, p, None) == EINVAL
    assert lib.og_keypoint_counts(p, 2, 10, -1, 5, None, p, p, None) == EINVAL
    assert lib.og_keypoint_counts(p, 2, 10, -1, 5, p, p, None, None) == EINVAL
    for B, cap, K in ((0, 10, 5), (2, 0, 5), (2, 10, 0), (-1, 10, 5)):
        assert lib.og_keypoint_counts(p, B, cap, -1, K, p, p, p, None) == EINVAL
    # og_mask_empty_pairs(len0, len1, B, n, m, matches0, mscores0, matches1, mscores1, stream)
    for i in range(6):
        args = [p] * 6
        args[i] = None
        assert lib.og_mask_empty_pairs(args[0], args[1], 2, 4, 4, *args[2:], None) == EINVAL
    for B, n, m in ((0, 4, 4), (2, 0, 4), (2, 4, 0)):
        assert lib.og_mask_empty_pairs(p, p, B, n, m, p, p, p, p, None) == EINVAL
    # og_sift_detect_padded(image, dtype, B, H, W, cap, ws, ws_bytes, kp, octave, count, overflow, stream)
    assert lib.og_sift_detect_padded(p, 0, 1, 64, 64, 100, p, 1 << 20, p, p, p, None, None) == EINVAL
    assert lib.og_sift_detect_padded(None, 0, 1, 64, 64, 100, p, 1 << 20, p, p, p, p, None) == EINVAL
    assert lib.og_sift_detect_padded(p, 0, 0, 64, 64, 100, p, 1 << 20, p, p, p, p, None) == EINVAL
    assert lib.og_sift_detect_padded(p, 0, 1, 64, 64, 100, p, 16, p, p, p, p, None) == EINVAL       # workspace too small
