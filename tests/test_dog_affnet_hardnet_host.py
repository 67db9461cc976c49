"""CPU checks of the DoG / AffNet / OriNet / HardNet front-end (openglue_b200.DoGOpenCVAffNetHardNet): the oracle in float32
against float64 stage by stage, the fixtures reproduced from their stored images, keypoints and seeds, the BatchNorm fold, the
refusals and the weight loading, and that nothing downloads."""
from __future__ import annotations

import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
REF = os.environ.get('OG_REFERENCE_ROOT', '/root/reference')

from oracle import dog_affnet_oracle as KD  # noqa: E402
from oracle import kornia_gftt_oracle as KG  # noqa: E402
from oracle import kornia_sift_oracle as KO  # noqa: E402
from oracle.gen_golden_dog_affnet_hardnet import CASES, load_fixture  # noqa: E402
from openglue_b200 import DoGOpenCVAffNetHardNet  # noqa: E402
from openglue_b200 import dog_affnet_hardnet as DA  # noqa: E402


def _fx(name):
    return load_fixture(os.path.join(GOLDEN, name + '.pt'))


def _weights():
    return dict(affnet=KG.synthetic_affnet_state_dict(), orinet=KD.synthetic_orinet_state_dict(), hardnet=KG.synthetic_hardnet_state_dict())


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def test_moons_lafs_from_keypoints_equal_the_cv2_keypoint_path():
    class Kp:                                                # the cv2.KeyPoint fields kornia_moons reads
        def __init__(self, r):
            self.pt, self.size, self.angle, self.response = (float(r[0]), float(r[1])), float(r[2]), float(r[3]), float(r[4])
    kp = _fx('dogaff_small')['kp']
    want = KD.laf_from_opencv_SIFT_kpts([Kp(r) for r in kp[0].tolist()])
    assert torch.equal(KD.lafs_from_kp(kp), want)
    l64 = KD.lafs_from_kp(kp, torch.float64)
    assert float((want.double() - l64).abs().max() / l64.abs().max()) < 4e-7
    # the rotation: [[s cos t, s sin t], [-s sin t, s cos t]], t = -angle in radians (kornia's pi is float32)
    t = -kp[0, :, 3].double() * torch.pi / 180
    s = 6.0 * kp[0, :, 2].double()
    for got, want in ((l64[0, :, 0, 0], s * torch.cos(t)), (l64[0, :, 0, 1], s * torch.sin(t)), (l64[0, :, 1, 0], -s * torch.sin(t)),
                      (l64[0, :, 1, 1], s * torch.cos(t))):
        torch.testing.assert_close(got, want, rtol=0, atol=1e-6 * float(s.max()))


def test_oracle_float32_agrees_with_float64_stage_by_stage():
    fx = _fx('dogaff_small')
    img, kp = fx['image'], fx['kp'][:, :400]
    assert (kp[..., 3] != 0).float().mean() > 0.9            # AffNet on LAFs with non-zero cv2 orientations
    s32 = KD.describe(img, kp)
    s64 = KD.describe(img.double(), kp)
    assert _rel(s32['moons_lafs'], s64['moons_lafs']) < 1e-6
    assert _rel(s32['aff_lafs'], s64['aff_lafs']) < 1e-4
    # angles: the float64 angle on the float32 pipeline's own AffNet LAFs isolates OriNet
    ori64 = KD.orinet_in(torch.float64)
    with torch.no_grad():
        _, a64 = KD.laf_orienter(s32['aff_lafs'].double(), img.double(), ori64, want_angles=True)
    assert float((s32['angles'].double() - a64).abs().max()) < 1e-4
    cos = F.cosine_similarity(s32['descriptors'].double(), s64['descriptors'], dim=-1)
    assert float(cos.min()) > 0.9999


def test_orinet_padded_head_equals_conv2d_in_float64():
    f = KD.orinet_in(torch.float64)
    g = torch.Generator().manual_seed(3)
    x = torch.relu(torch.randn(5, 64, 8, 8, generator=g, dtype=torch.float64))
    head = f[KD.ORINET_HEAD]
    assert head.padding == (1, 1) and head.kernel_size == (8, 8)
    y = torch.tanh(F.conv2d(x, head.weight, head.bias, padding=1))
    assert y.shape == (5, 2, 3, 3)
    want = y.mean(dim=(2, 3))
    with torch.no_grad():
        got = f[KD.ORINET_HEAD + 2](f[KD.ORINET_HEAD + 1](head(x))).view(5, 2)
    torch.testing.assert_close(got, want, rtol=1e-14, atol=1e-14)
    # the synthetic head keeps (y0, y1) far from atan2's singularity on real patches
    fx = _fx('dogaff_small')
    with torch.no_grad():
        xy = KD.orinet_xy(KD.extract_patches_from_pyramid(fx['image'], fx['aff_lafs'], 32).view(-1, 1, 32, 32), KD.orinet_in(torch.float32))
    assert float(xy.norm(dim=1).min()) > 0.2


@pytest.mark.parametrize('name', list(CASES))
def test_fixtures_reproduce_from_images_keypoints_and_seeds(name):
    fx = _fx(name)
    assert fx['affnet_sha256'] == KG.state_dict_checksum(KG.synthetic_affnet_state_dict(fx['affnet_seed']))
    assert fx['orinet_sha256'] == KG.state_dict_checksum(KD.synthetic_orinet_state_dict(fx['orinet_seed']))
    assert fx['hardnet_sha256'] == KG.state_dict_checksum(KG.synthetic_hardnet_state_dict(fx['hardnet_seed']))
    n = fx['kp'].shape[1]
    assert n <= 2048 and fx['scores'].shape == (1, n) and fx['descriptors'].shape == (1, n, 128)
    if n == 0:
        assert fx['reference_fails']
        return
    assert torch.equal(fx['scores'], fx['kp'][..., 4])
    s = KD.describe(fx['image'], fx['kp'])
    for k in ('moons_lafs', 'aff_lafs', 'angles', 'lafs'):
        assert torch.equal(s[k], fx[k]), k
    assert torch.equal(s['descriptors'].half(), fx['descriptors'])


@pytest.mark.parametrize('name', [n for n in CASES if n != 'dogaff_uniform'])
def test_fresh_reference_run_equals_the_fixture(name):
    if not os.path.isfile(os.path.join(REF, 'models', 'features', 'opencv', 'dog_affnet_harnet.py')):
        pytest.skip('the reference is not checked out here')
    cv2 = pytest.importorskip('cv2')
    pytest.importorskip('scipy')
    from oracle.gen_golden_dog_affnet_hardnet import import_reference, mint
    fx, new = _fx(name), mint(name, import_reference())
    if cv2.__version__ != fx['cv2_version']:
        pytest.skip(f'cv2 {cv2.__version__} here, the fixture was made with {fx["cv2_version"]}')
    for k in ('kp', 'moons_lafs', 'aff_lafs', 'angles', 'lafs', 'scores', 'descriptors'):
        assert torch.equal(new[k], fx[k]), k


def test_orinet_batchnorm_fold_equals_conv_then_batchnorm():
    m = DoGOpenCVAffNetHardNet(max_keypoints=64, weights=_weights())
    f = m.orinet.angle_detector.features
    x = torch.randn(3, 16, 12, 12, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    conv, bn = f[3], f[4]
    w, b = DA.fold(conv.weight, bn)
    with torch.no_grad():
        want = F.batch_norm(F.conv2d(x, conv.weight.double(), padding=1), bn.running_mean.double(), bn.running_var.double(), eps=bn.eps)
    got = F.conv2d(x, w.double().view(16, 3, 3, 16).permute(0, 3, 1, 2), b.double(), padding=1)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)
    hw, hb = m._weights_on(torch.device('cpu'))['orinet'][-1]
    assert hw.shape == (2, 8 * 8 * 64) and torch.equal(hw.view(2, 8, 8, 64).permute(0, 3, 1, 2), f[19].weight.float())
    assert torch.equal(hb, f[19].bias.float())


@pytest.mark.parametrize('kwargs', [dict(max_keypoints=0), dict(max_keypoints=-2), dict(precision='fp16')])
def test_argument_refusals(kwargs):
    with pytest.raises(ValueError):
        DoGOpenCVAffNetHardNet(**kwargs, weights=_weights())


def test_input_refusals():
    import numpy as np
    m = DoGOpenCVAffNetHardNet(max_keypoints=64, weights=_weights())
    with pytest.raises(TypeError):
        m(np.zeros((32, 32), np.uint8))
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 1, 32, 32))
    with pytest.raises(RuntimeError):
        m.extract_padded(torch.zeros(2, 1, 32, 32), 16)
    with pytest.raises(ValueError):
        m(torch.zeros(1, 3, 32, 32))
    with pytest.raises(RuntimeError):
        m.train()


def test_weights_load_from_kornia_layout_reference_modules_and_files(tmp_path):
    w = _weights()
    m = DoGOpenCVAffNetHardNet(max_keypoints=64, weights=w)
    assert torch.equal(m.affnet.features[19].bias, w['affnet']['features.19.bias'])
    assert torch.equal(m.orinet.angle_detector.features[19].weight, w['orinet']['features.19.weight'])
    assert torch.equal(m.hardnet.features[15].weight, w['hardnet']['features.15.weight'])
    for k, (fname, _) in DA.CHECKPOINTS.items():
        torch.save({'state_dict': w[k], 'epoch': 1}, tmp_path / fname)
    m2 = DoGOpenCVAffNetHardNet(weights={k: str(tmp_path / f) for k, (f, _) in DA.CHECKPOINTS.items()})
    assert list(m.state_dict()) == list(m2.state_dict())
    for a, b in zip(m.state_dict().values(), m2.state_dict().values()):
        assert torch.equal(a, b)
    if os.path.isfile(os.path.join(REF, 'models', 'features', 'opencv', 'dog_affnet_harnet.py')) and _has('cv2') and _has('scipy'):
        from oracle.gen_golden_dog_affnet_hardnet import import_reference
        sd = import_reference()(max_keypoints=64).state_dict()
    else:
        sd = m.state_dict()
    prefixes = ('affnet.features.', 'orinet.angle_detector.features.', 'hardnet.features.')
    assert all(any(k.startswith(p) for k in sd) for p in prefixes) and all(k.startswith(prefixes) for k in sd)
    m3 = DoGOpenCVAffNetHardNet(max_keypoints=64, weights=w)
    m3.load_state_dict(sd, strict=True)
    with pytest.raises(KeyError):
        DoGOpenCVAffNetHardNet(weights={**w, 'orinet': {'features.0.weight': torch.zeros(16, 1, 3, 3)}})
    with pytest.raises(ValueError):
        DoGOpenCVAffNetHardNet(weights={'affnet': w['affnet'], 'hardnet': w['hardnet']})


def _has(mod):
    try:
        __import__(mod)
        return True
    except ImportError:
        return False


def test_no_download(tmp_path, monkeypatch):
    import urllib.request

    def refuse(*a, **k):
        raise AssertionError('nothing may be downloaded')
    monkeypatch.setenv('TORCH_HOME', str(tmp_path))
    monkeypatch.setattr(torch.hub, 'load_state_dict_from_url', refuse)
    monkeypatch.setattr(torch.hub, 'download_url_to_file', refuse)
    monkeypatch.setattr(urllib.request, 'urlopen', refuse)
    monkeypatch.setattr(urllib.request, 'urlretrieve', refuse)
    ck = tmp_path / 'hub' / 'checkpoints'
    ck.mkdir(parents=True)
    w = _weights()
    for name, (fname, url) in DA.CHECKPOINTS.items():
        with pytest.raises(FileNotFoundError, match=fname) as e:
            DoGOpenCVAffNetHardNet()
        assert url in str(e.value)
        torch.save({'state_dict': w[name]}, ck / fname)
    m = DoGOpenCVAffNetHardNet()
    assert torch.equal(m.orinet.angle_detector.features[19].bias, w['orinet']['features.19.bias'])


def test_graphs_hold_the_nested_detector_workspaces():
    """a captured graph reads the workspaces of the OpenCVSIFT the module detects through, so what a graph holds includes them"""
    from openglue_b200.features import _frontend_storage
    m = DoGOpenCVAffNetHardNet(max_keypoints=64, weights=_weights())
    own, det = torch.zeros(4), (torch.zeros(8), torch.zeros(2))
    m._ws['describe'] = own
    m._sift._ws['detect'] = det
    held, _ = _frontend_storage(m)
    assert any(h is own for h in held) and any(h is det for h in held)
