"""Padded batches without a GPU: the Python validation of host lengths, shapes and train mode, pad_features, the C ABI's padded
workspace query and the host Sinkhorn constants the padded kernels' tables must reproduce."""
import ctypes as C
import ctypes.util

import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200.features import pad_features
from openglue_b200.superglue import SuperGlue, is_padded, padded_inputs
from openglue_b200.synthetic import default_config, synthetic_pairs


def _data(B=3, n=10, m=7):
    d = synthetic_pairs(B, n, m, 32, 1, seed=0)
    d['num_keypoints0'] = torch.tensor([10, 1, 4])
    d['num_keypoints1'] = torch.tensor([7, 7, 1])
    return d


def test_host_lengths_and_sizes_become_per_pair_tensors():
    d = _data()
    assert is_padded(d) and not is_padded({'keypoints0': None})
    out = padded_inputs(d, 3, 10, 7)
    assert out['num_keypoints0'].dtype == torch.int32 and out['num_keypoints0'].tolist() == [10, 1, 4]
    assert out['image0_size'].shape == (3, 2) and out['image0_size'][0].tolist() == list(map(float, d['image0_size']))
    d['image1_size'] = torch.tensor([[640., 480.], [320., 240.], [100., 50.]])
    assert padded_inputs(d, 3, 10, 7)['image1_size'][2].tolist() == [100., 50.]


@pytest.mark.parametrize('key,value,msg', [
    ('num_keypoints0', torch.tensor([0, 1, 4]), r'\[1, 10\]'),
    ('num_keypoints0', torch.tensor([11, 1, 4]), r'\[1, 10\]'),
    ('num_keypoints1', torch.tensor([7, -1, 1]), r'\[1, 7\]'),
    ('num_keypoints1', torch.tensor([7, 8, 1]), r'\[1, 7\]'),
    ('num_keypoints0', torch.tensor([1, 2]), 'shape'),
    ('num_keypoints0', torch.tensor([[1, 2, 3]]), 'shape'),
    ('num_keypoints0', torch.tensor([1., 2., 3.]), 'integer'),
    ('image0_size', torch.ones(2, 2), r'\[3, 2\]'),
])
def test_bad_padded_inputs_are_refused(key, value, msg):
    d = _data()
    d[key] = value
    with pytest.raises(ValueError, match=msg):
        padded_inputs(d, 3, 10, 7)


def test_lengths_come_in_pairs():
    d = _data()
    del d['num_keypoints1']
    with pytest.raises(ValueError, match='both'):
        padded_inputs(d, 3, 10, 7)


def test_train_mode_with_lengths_is_not_implemented():
    model = SuperGlue(default_config(descriptor_dim=32, num_stages=1)).train()
    with pytest.raises(NotImplementedError, match='eval mode'):
        model(_data())
    with pytest.raises(NotImplementedError, match='eval mode'):
        model.run(_data(), want_matches=True)


def test_pad_features_keeps_every_keypoint():
    g = torch.Generator().manual_seed(0)
    feats = [(torch.randn(1, k, 2, 3, generator=g), torch.rand(1, k, generator=g), torch.randn(1, k, 5, generator=g)) for k in (4, 9, 1)]
    lafs, resp, desc, counts = pad_features(feats)
    assert counts.tolist() == [4, 9, 1] and counts.device.type == 'cpu'
    assert lafs.shape == (3, 9, 2, 3) and resp.shape == (3, 9) and desc.shape == (3, 9, 5)
    for b, (l, r, d) in enumerate(feats):
        k = l.shape[1]
        assert torch.equal(lafs[b, :k], l[0]) and torch.equal(resp[b, :k], r[0]) and torch.equal(desc[b, :k], d[0])
        assert (lafs[b, k:] == 0).all() and (resp[b, k:] == 0).all() and (desc[b, k:] == 0).all()
    assert pad_features([(f[0][0], f[1][0], f[2][0]) for f in feats], capacity=12)[0].shape == (3, 12, 2, 3)
    with pytest.raises(ValueError, match='capacity'):
        pad_features(feats, capacity=8)


def test_padded_workspace_holds_the_masked_descriptors():
    lib = _cabi.lib()
    cfg = _cabi.make_config(default_config())
    B, n, m = 4, 300, 200
    extra = lib.og_workspace_bytes_padded(cfg, B, n, m) - lib.og_workspace_bytes(cfg, B, n, m)
    assert extra >= B * (n + m) * 256 * 4
    assert lib.og_workspace_bytes_padded(cfg, 0, n, m) < 0


def test_host_sinkhorn_constants_are_the_references():
    """og_sinkhorn_consts is what the Sinkhorn uses for a uniform batch and what a padded batch's tables must reproduce bit for bit:
    norm = -log(n + m) in float32 (the host's logf), log_a_last = norm + log(m), log_b_last = norm + log(n)."""
    lib = _cabi.lib()
    libm = C.CDLL(ctypes.util.find_library('m'))
    libm.logf.restype, libm.logf.argtypes = C.c_float, [C.c_float]
    out = (C.c_float * 3)()
    for n, m in [(1, 1), (2048, 2048), (1579, 3100), (65536, 8192), (7, 4935)]:
        assert lib.og_sinkhorn_consts(n, m, out) == 0
        norm = -C.c_float(libm.logf(float(n + m))).value
        f32 = lambda x: torch.tensor(x, dtype=torch.float32)
        assert out[0] == norm
        assert out[1] == float(f32(norm) + f32(torch.log(torch.tensor(float(m), dtype=torch.float64)).item()))
        assert out[2] == float(f32(norm) + f32(torch.log(torch.tensor(float(n), dtype=torch.float64)).item()))
