"""GFTT / AffNet / HardNet front-end without a GPU: the float32 oracle against its float64 form stage by stage, the committed
fixtures against their images and weight seeds (and against the unmodified reference where it is checked out), the BatchNorm
fold, the argument and weight-loading checks of openglue_b200.GFTTAffNetHardNet, and that nothing downloads.  Parity of the
restatement with kornia itself is checked only where kornia is installed; elsewhere it is unverified."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import kornia_gftt_oracle as KG  # noqa: E402
from oracle import kornia_sift_oracle as KO  # noqa: E402
from oracle.gen_golden_gftt_hardnet import load_fixture  # noqa: E402
from openglue_b200 import GFTTAffNetHardNet  # noqa: E402
from openglue_b200 import gftt_hardnet as GH  # noqa: E402

REF = os.environ.get('OG_REFERENCE_ROOT', '/root/reference')
CASES = ['gftt_tiny', 'gftt_small', 'gftt_odd', 'gftt_warp', 'gftt_uniform', 'gftt_pair']


def _fx(name):
    return load_fixture(os.path.join(HERE, 'golden', name + '.pt'))


def _weights():
    return {'affnet': KG.synthetic_affnet_state_dict(), 'hardnet': KG.synthetic_hardnet_state_dict()}


def test_oracle_float32_against_float64_stage_by_stage():
    fx = _fx('gftt_small')
    img = fx['image']
    pyr, sig = KO.scale_pyramid(img, double_image=False)
    pyr64, sig64 = KO.scale_pyramid(img.double(), double_image=False)
    assert pyr[0].shape[-2:] == img.shape[-2:]                                  # no doubling
    for o in range(len(pyr)):
        r32 = KG.octave_response(pyr[o], sig[o]).double()
        r64 = KG.octave_response(pyr64[o], sig64[o])
        assert r32.shape[2] == 5
        # the smaller eigenvalue cancels in float32: bounded relative to the octave's largest response (2.4e-5 measured)
        assert float((r32 - r64).abs().max()) <= 1e-4 * float(r64.abs().max()) + 1e-9, o
    r32, l32 = KG.detect(img, 1024)
    r64, l64 = KG.detect(img.double(), 1024)
    assert float((r32.double() - r64).abs().max()) <= 1e-4 * float(r64.abs().max())
    aff, hard = KG.features_in(torch.float32)
    aff64, hard64 = KG.features_in(torch.float64)
    lafs = l64[:, :64]
    a32 = KG.affnet_shape(lafs.float(), img, aff).double()
    a64 = KG.affnet_shape(lafs, img.double(), aff64)
    assert float((a32 - a64).abs().max()) <= 1e-4 * float(a64[..., :2].abs().max())
    p = KO.extract_patches_from_pyramid(img.double(), a64, 32).view(-1, 1, 32, 32)
    d32 = KG.hardnet(p.float(), hard).double()
    d64 = KG.hardnet(p, hard64)
    assert float(F.cosine_similarity(d32, d64, dim=1).min()) >= 1 - 1e-6


def test_fixtures_reproduce_from_images_and_seeds():
    for name in CASES:
        fx = _fx(name)
        B = fx['image'].shape[0]
        assert fx['affnet_sha256'] == KG.state_dict_checksum(KG.synthetic_affnet_state_dict(fx['affnet_seed']))
        assert fx['hardnet_sha256'] == KG.state_dict_checksum(KG.synthetic_hardnet_state_dict(fx['hardnet_seed']))
        N = fx['lafs'].shape[1]
        assert fx['det_lafs'].shape == fx['aff_lafs'].shape == (B, 1024, 2, 3) and fx['sel'].shape == (B, N)
        for b in range(B):
            assert torch.equal(fx['responses'][b], fx['det_resp'][b, fx['sel'][b]])
            assert torch.equal(fx['lafs'][b, :, :, 2], fx['det_lafs'][b, fx['sel'][b], :, 2])     # AffNet and the orienter keep centres
        if name in ('gftt_tiny', 'gftt_small'):
            r, l = KG.detect(fx['image'], 1024)
            assert torch.equal(r, fx['det_resp']) and torch.equal(l, fx['det_lafs'])
            aff, _ = KG.features_in(torch.float32)
            with torch.no_grad():
                assert torch.equal(KG.affnet_shape(l, fx['image'], aff), fx['aff_lafs'])
    assert _fx('gftt_uniform')['lafs'].shape[1] == 0


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, 'models', 'features', 'hardnet.py')), reason='the reference is not checked out')
def test_fixtures_equal_a_fresh_run_of_the_reference():
    from oracle.gen_golden_gftt_hardnet import import_reference, mint
    cls = import_reference()
    for name in ('gftt_small', 'gftt_pair'):
        fx, new = _fx(name), mint(name, cls)
        for k in ('det_resp', 'det_lafs', 'aff_lafs', 'sel', 'lafs', 'responses', 'descriptors'):
            assert torch.equal(fx[k], new[k]), (name, k)


def test_batchnorm_fold_equals_conv_then_batchnorm():
    sd = KG.synthetic_hardnet_state_dict()
    net = GH._HardNet()
    net.load_state_dict(sd)
    x = torch.randn(3, 32, 10, 10, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    conv, bn = net.features[3], net.features[4]
    want = F.batch_norm(F.conv2d(x, conv.weight.double(), padding=1), bn.running_mean.double(), bn.running_var.double(), eps=bn.eps)
    w, b = GH._fold(conv.weight, bn)
    cols = F.unfold(x, 3, padding=1).view(3, 32, 9, 100).permute(0, 3, 2, 1).reshape(3, 100, 9 * 32)    # (ky, kx, c) columns
    got = (cols @ w.double().t() + b.double()).permute(0, 2, 1).reshape(3, 32, 10, 10)
    assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max())
    head, hbn = net.features[19], net.features[20]
    y = torch.randn(2, 128, 8, 8, dtype=torch.float64)
    want = F.batch_norm(F.conv2d(y, head.weight.double()), hbn.running_mean.double(), hbn.running_var.double(), eps=hbn.eps).flatten(1)
    w, b = GH._fold(head.weight, hbn)
    got = y.permute(0, 2, 3, 1).reshape(2, -1) @ w.double().t() + b.double()
    assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max())


@pytest.mark.parametrize('kwargs', [dict(patch_size=41), dict(descriptor_dim=256), dict(max_keypoints=0), dict(max_keypoints=8193),
                                    dict(nms_diameter=8), dict(precision='fp16')])
def test_argument_refusals(kwargs):
    with pytest.raises(ValueError):
        GFTTAffNetHardNet(**kwargs, weights=_weights())


def test_weights_load_from_kornia_layout_reference_modules_and_files(tmp_path):
    w = _weights()
    m = GFTTAffNetHardNet(max_keypoints=64, weights=w)
    assert torch.equal(m.detector.aff.features[19].bias, w['affnet']['features.19.bias'])
    assert torch.equal(m.descriptor.descriptor.features[15].weight, w['hardnet']['features.15.weight'])
    # kornia's checkpoint files: a dict holding 'state_dict'
    for k, (fname, _) in GH.CHECKPOINTS.items():
        torch.save({'state_dict': w[k], 'epoch': 1}, tmp_path / fname)
    m2 = GFTTAffNetHardNet(weights={k: str(tmp_path / f) for k, (f, _) in GH.CHECKPOINTS.items()})
    for a, b in zip(m.state_dict().values(), m2.state_dict().values()):
        assert torch.equal(a, b)
    # the reference module (its kornia modules stood in by the restatement): its state_dict loads, strictly
    if os.path.isfile(os.path.join(REF, 'models', 'features', 'hardnet.py')):
        from oracle.gen_golden_gftt_hardnet import import_reference
        ref = import_reference()(max_keypoints=64)
        sd = ref.state_dict()
    else:
        sd = m.state_dict()
    assert any(k.startswith('detector.aff.features.') for k in sd) and any(k.startswith('descriptor.descriptor.features.') for k in sd)
    m3 = GFTTAffNetHardNet(max_keypoints=64, weights=w)
    m3.load_state_dict(sd, strict=True)
    with pytest.raises(KeyError):
        GFTTAffNetHardNet(weights={'affnet': w['affnet'], 'hardnet': {'features.0.weight': torch.zeros(32, 1, 3, 3)}})


def test_no_download(tmp_path, monkeypatch):
    def refuse(*a, **k):
        raise AssertionError('load_state_dict_from_url must not be called')
    monkeypatch.setenv('TORCH_HOME', str(tmp_path))
    monkeypatch.setattr(torch.hub, 'load_state_dict_from_url', refuse)
    monkeypatch.setattr(torch.hub, 'download_url_to_file', refuse)
    with pytest.raises(FileNotFoundError, match='AffNet.pth'):
        GFTTAffNetHardNet()
    # with both files in kornia's cache the module loads them
    ck = tmp_path / 'hub' / 'checkpoints'
    ck.mkdir(parents=True)
    w = _weights()
    torch.save({'state_dict': w['affnet']}, ck / 'AffNet.pth')
    with pytest.raises(FileNotFoundError, match='checkpoint_liberty_with_aug.pth'):
        GFTTAffNetHardNet()
    torch.save({'state_dict': w['hardnet']}, ck / 'checkpoint_liberty_with_aug.pth')
    GFTTAffNetHardNet()


def test_parity_with_kornia():
    kornia = pytest.importorskip('kornia')
    img = _fx('gftt_small')['image']
    torch.testing.assert_close(kornia.feature.responses.gftt_response(img), KG.gftt_response(img))
    hn = kornia.feature.HardNet(False).eval()
    hn.load_state_dict(KG.synthetic_hardnet_state_dict())
    an = kornia.feature.LAFAffNetShapeEstimator(False).eval()
    an.load_state_dict(KG.synthetic_affnet_state_dict(), strict=False)
    aff, hard = KG.features_in(torch.float32)
    r, l = KG.detect(img, 256)
    with torch.no_grad():
        torch.testing.assert_close(an(l, img), KG.affnet_shape(l, img, aff))
        p = torch.rand(8, 1, 32, 32, generator=torch.Generator().manual_seed(0))
        torch.testing.assert_close(hn(p), KG.hardnet(p, hard))
        det = kornia.feature.ScaleSpaceDetector(256, resp_module=kornia.feature.responses.CornerGFTT(),
                                                nms_module=kornia.geometry.subpix.ConvQuadInterp3d(10, 1e-5),
                                                scale_pyr_module=kornia.geometry.transform.ScalePyramid(3, 1.6, 32, double_image=False),
                                                ori_module=kornia.feature.orientation.PassLAF(), mr_size=6.0)
        lk, rk = det(img)
        torch.testing.assert_close(rk, r, atol=1e-4, rtol=1e-4)
