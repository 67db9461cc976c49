"""Host-side checks of ImagePairTrainStep and the guarded training entry points: every refusal happens before any kernel launch
(CPU tensors reach no kernel, so the refusal under test is the one raised), and the new C entry points reject null pointers and
bad sizes with OG_EINVAL without touching a GPU."""
import copy

import pytest
import torch

from openglue_b200 import ImagePairTrainStep, OpenCVSIFT, SuperGlue, SuperPointNet, _cabi
from openglue_b200.synthetic import default_config

CONFIG = {'superglue': {'laf_to_sideinfo_method': 'none', 'log_transform_response': False},
          'train': {'gt_positive_threshold': 2, 'gt_negative_threshold': 7, 'margin': None, 'nll_weight': 1.0, 'metric_weight': 0.0,
                    'augmentations': {'name': 'none'}, 'lr': 1e-4, 'grad_clip': 10.0, 'scheduler_gamma': 0.999994}}


def _superglue(d=128, side=1):
    return SuperGlue(default_config(descriptor_dim=d, num_heads=4, num_stages=1, num_iters=5, side_info_size=side)).train()


def _config(**train):
    c = copy.deepcopy(CONFIG)
    c['train'].update(train)
    return c


def _batch(B=2, H=64, W=80, **over):
    b = {'image0': torch.zeros(B, 1, H, W), 'image1': torch.zeros(B, 1, H, W),
         'transformation': {'type': ['perspective'] * B, 'H': torch.eye(3).expand(B, 3, 3)}}
    b.update(over)
    return b


def test_constructor_refusals():
    sift = OpenCVSIFT(max_keypoints=100)
    with pytest.raises(TypeError, match='SuperGlue'):
        ImagePairTrainStep(sift, torch.nn.Linear(2, 2), CONFIG)
    with pytest.raises(RuntimeError, match=r'train\(\)'):
        ImagePairTrainStep(sift, _superglue().eval(), CONFIG)
    with pytest.raises(TypeError, match='extract_padded'):
        ImagePairTrainStep(torch.nn.Identity(), _superglue(), CONFIG)
    with pytest.raises(NotImplementedError, match='finetune'):
        ImagePairTrainStep(sift, _superglue(), {**CONFIG, 'features': {'finetune': True}})
    with pytest.raises(NotImplementedError, match='margin'):
        ImagePairTrainStep(sift, _superglue(), _config(margin=0.5, metric_weight=1.0))
    with pytest.raises(NotImplementedError, match='augmentation'):
        ImagePairTrainStep(sift, _superglue(), _config(augmentations={'name': 'weak_color_aug'}))
    sg = _superglue()
    with pytest.raises(TypeError, match='ClippedAdam'):
        ImagePairTrainStep(sift, sg, CONFIG, optimizer=torch.optim.Adam(sg.parameters()))
    with pytest.raises(NameError):
        ImagePairTrainStep(sift, sg, {**CONFIG, 'superglue': {'laf_to_sideinfo_method': 'shape'}})
    with pytest.raises(ValueError, match='side_info_size'):
        ImagePairTrainStep(sift, _superglue(side=4), CONFIG)
    with pytest.raises(ValueError, match='dimensions'):
        ImagePairTrainStep(sift, _superglue(d=256), CONFIG)
    with pytest.raises(ValueError, match='dimensions'):
        ImagePairTrainStep(SuperPointNet(max_keypoints=100), _superglue(d=128), CONFIG)
    ImagePairTrainStep(sift, _superglue(side=4), {**CONFIG, 'superglue': {'laf_to_sideinfo_method': 'scale_rotation'}})
    with pytest.raises(ValueError, match='head_dim'):
        ImagePairTrainStep(sift, SuperGlue(default_config(descriptor_dim=128, num_heads=1, num_stages=1, num_iters=5)).train(), CONFIG)


def test_call_refusals_before_any_launch():
    step = ImagePairTrainStep(OpenCVSIFT(max_keypoints=100), _superglue(), CONFIG)
    with pytest.raises(ValueError, match=r'image1 must be \[B, 1, H, W\]'):
        step(_batch(image1=torch.zeros(2, 64, 80)))
    with pytest.raises(ValueError, match=r'image0 must be \[B, 1, H, W\]'):
        step(_batch(image0=torch.zeros(2, 3, 64, 80)))
    with pytest.raises(ValueError, match='same number of images'):
        step(_batch(image1=torch.zeros(3, 1, 64, 80)))
    with pytest.raises(ValueError, match='Unknown transformation type'):
        step(_batch(transformation={'type': ['affine'] * 2, 'H': torch.zeros(2, 3, 3)}))
    with pytest.raises(ValueError, match=r"transformation\['H'\]"):
        step(_batch(transformation={'type': ['perspective'] * 2, 'H': torch.zeros(3, 3, 3)}))
    tf = {'type': ['3d_reprojection'] * 2, 'K0': torch.zeros(2, 3, 3), 'K1': torch.zeros(2, 3, 3), 'R': torch.zeros(2, 3, 3),
          'T': torch.zeros(2, 3), 'depth0': torch.zeros(2, 64, 80), 'depth1': torch.zeros(2, 64, 80)}
    for k, bad in (('T', torch.zeros(2, 3, 1)), ('depth1', torch.zeros(2, 64)), ('K0', torch.zeros(2, 4, 4))):
        with pytest.raises(ValueError, match=rf"transformation\['{k}'\]"):
            step(_batch(transformation={**tf, k: bad}))
    with pytest.raises(KeyError):
        step(_batch(transformation={k: v for k, v in tf.items() if k != 'R'}))
    with pytest.raises(ValueError, match='needs a capacity'):
        ImagePairTrainStep(OpenCVSIFT(), _superglue(), CONFIG)(_batch())
    with pytest.raises(ValueError, match='at least 1'):
        ImagePairTrainStep(OpenCVSIFT(), _superglue(), CONFIG, capacity=0)(_batch())
    with pytest.raises(RuntimeError, match='CUDA'):
        step(_batch())
    with pytest.raises(RuntimeError, match='CUDA'):
        step(_batch(transformation=tf))


def test_pretrain_refusals_before_any_launch():
    step = ImagePairTrainStep(OpenCVSIFT(max_keypoints=100), _superglue(), CONFIG)
    with pytest.raises(TypeError, match='uint8'):
        step.pretrain(torch.zeros(2, 96, 128, 3), 8)
    with pytest.raises(ValueError, match=r'\[B, H, W, 3\]'):
        step.pretrain(torch.zeros(2, 96, 128, 1, dtype=torch.uint8), 8)
    with pytest.raises(ValueError, match='offset'):
        step.pretrain(torch.zeros(2, 96, 128, 3, dtype=torch.uint8), 48)
    with pytest.raises(TypeError, match='integer'):
        step.pretrain(torch.zeros(2, 96, 128, 3, dtype=torch.uint8), 8.5)
    with pytest.raises(RuntimeError, match='CUDA'):
        step.pretrain(torch.zeros(2, 96, 128, 3, dtype=torch.uint8), 8)


def test_guarded_entry_points_reject_bad_arguments():
    lib = _cabi.lib()
    buf = torch.zeros(64, dtype=torch.int32)
    p = _cabi.ptr(buf)
    EINVAL = -1
    # og_train_guard(lengths, B, skip, stream)
    assert lib.og_train_guard(None, 2, p, None) == EINVAL
    assert lib.og_train_guard(p, 2, None, None) == EINVAL
    for B in (0, -1):
        assert lib.og_train_guard(p, B, p, None) == EINVAL
    # og_train_skip_outputs(skip, loss, nloss, x, n, stream)
    assert lib.og_train_skip_outputs(None, p, 2, p, 4, None) == EINVAL
    assert lib.og_train_skip_outputs(p, None, 2, p, 4, None) == EINVAL
    assert lib.og_train_skip_outputs(p, p, 2, None, 4, None) == EINVAL
    for nloss, n in ((-1, 4), (257, 4), (2, -1)):
        assert lib.og_train_skip_outputs(p, p, nloss, p, n, None) == EINVAL
    assert lib.og_train_skip_outputs(p, None, 0, None, 0, None) == 0             # nothing to write: no launch
    # og_bn_train_fwd_guarded(a, lda, batch, cap, lengths, cols, relu, gamma, beta, eps, momentum, y, ldy, mean, invstd,
    #                         running_mean, running_var, skip, num_batches_tracked, workspace, stream)
    def bn(**kw):
        a = dict(a=p, batch=2, cap=8, cols=4, gamma=p, beta=p, y=p, mean=p, invstd=p, ws=p)
        a.update(kw)
        return lib.og_bn_train_fwd_guarded(a['a'], 4, a['batch'], a['cap'], p, a['cols'], 1, a['gamma'], a['beta'], 1e-5, 0.1, a['y'], 4,
                                           a['mean'], a['invstd'], p, p, p, p, a['ws'], None)
    for k in ('a', 'gamma', 'beta', 'y', 'mean', 'invstd', 'ws'):
        assert bn(**{k: None}) == EINVAL, k
    for sizes in (dict(batch=0), dict(cap=0), dict(cols=0), dict(batch=1 << 16, cap=1 << 16)):
        assert bn(**sizes) == EINVAL, sizes
    # og_clip_adam_step_guarded(segments, nseg, ntiles, b1, b2, eps, max_norm, lr_gamma, state, ws, ws_bytes, skip, stream)
    def adam(segs=p, nseg=1, ntiles=1, b1=0.9, clip=10.0, state=p, ws=p, wsb=1 << 12):
        return lib.og_clip_adam_step_guarded(segs, nseg, ntiles, b1, 0.999, 1e-8, clip, 0.99, state, ws, wsb, p, None)
    for kw in (dict(segs=None), dict(state=None), dict(ws=None), dict(nseg=0), dict(ntiles=0), dict(b1=1.0), dict(clip=0.0)):
        assert adam(**kw) == EINVAL, kw
    assert adam(wsb=8) < 0                                                      # workspace too small
