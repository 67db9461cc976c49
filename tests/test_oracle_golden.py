"""Pin the oracle: it must reproduce the reference's own outputs (tests/golden/, minted by
oracle/gen_golden.py from the unmodified reference) before anything is compared against it."""
import pytest
import torch

from oracle import superglue_oracle as O
from conftest import GOLDEN_BIG, GOLDEN_FULL, GOLDEN_SAMPLED


@pytest.mark.parametrize('name', GOLDEN_FULL)
def test_oracle_matches_reference_full(golden, name):
    fx = golden(name)
    out = O.run(fx['state_dict'], fx['config'], fx['data'], fx['match_threshold'])
    # same ATen ops, same order => fp32 agreement to rounding noise
    assert (out['scores'] - fx['scores_f32']).abs().max() <= 2e-6
    assert (out['context_descriptors0'] - fx['context_descriptors0_f32']).abs().max() <= 1e-5
    assert (out['context_descriptors1'] - fx['context_descriptors1_f32']).abs().max() <= 1e-5
    assert torch.equal(out['matches0'], fx['matches0'])
    assert (out['matching_scores0'] - fx['matching_scores0']).abs().max() <= 2e-6
    # fp64 oracle vs fp64 reference
    out64 = O.run(fx['state_dict'], fx['config'], fx['data'], fx['match_threshold'], dtype=torch.float64)
    assert (out64['scores'] - fx['scores_f64']).abs().max() <= 1e-10


@pytest.mark.parametrize('name', GOLDEN_SAMPLED)
def test_oracle_matches_reference_c1(golden, name):
    """BASELINE.json configs[0]: 1 pair, N=M=512, d=256, 9 stages, 20 Sinkhorn iterations."""
    fx = golden(name)
    out = O.run(fx['state_dict'], fx['config'], fx['data'], fx['match_threshold'])
    s = out['scores']
    assert (s[:, ::7, ::5] - fx['scores_f32_sample']).abs().max() <= 5e-6
    assert (s[:, -1, :] - fx['scores_f32_lastrow']).abs().max() <= 5e-6
    assert (s[:, :, -1] - fx['scores_f32_lastcol']).abs().max() <= 5e-6
    assert (out['context_descriptors0'][:, ::4, ::8] - fx['ctx0_f32_sample']).abs().max() <= 2e-5
    assert torch.equal(out['matches0'], fx['matches0'])
    assert (out['matching_scores0'] - fx['matching_scores0']).abs().max() <= 5e-6
    rel = (s.double().sum(2) - fx['scores_f64_rowsum']).abs().max() / fx['scores_f64_rowsum'].abs().max()
    assert rel < 1e-6


@pytest.mark.parametrize('name', GOLDEN_BIG)
def test_oracle_matches_reference_big(golden, name):
    """BASELINE.json configs[1], [2], [4] at full depth: the oracle on the fixture's scored pairs (the first two of the
    batch bench.py times) against the reference's fp32 run of the same pairs."""
    fx = golden(name)
    k = fx['scored_pairs']
    data = {key: (v[:k] if torch.is_tensor(v) else v) for key, v in fx['data'].items()}
    out = O.run(fx['state_dict'], fx['config'], data, fx['match_threshold'])
    s, (sr, sc) = out['scores'], fx['sample_stride']
    # same ATen ops on the same B = k batch: rounding noise only (|scores| reaches ~80 on the planted inputs)
    assert (s[:, ::sr, ::sc] - fx['scores_f32_sample']).abs().max() <= 2e-5
    assert (s[:, -1, :] - fx['scores_f32_lastrow']).abs().max() <= 2e-5
    assert (s[:, :, -1] - fx['scores_f32_lastcol']).abs().max() <= 2e-5
    assert (out['context_descriptors0'][:, ::4, ::8] - fx['ctx0_f32_sample']).abs().max() <= 5e-5
    # matches0 / matching_scores0 of the fixture come from the reference's MatchingTrainingModule.forward over the WHOLE batch
    assert torch.equal(out['matches0'], fx['matches0'][:k])
    assert (out['matching_scores0'] - fx['matching_scores0'][:k]).abs().max() <= 2e-5
    rel = (s.double().sum(2) - fx['scores_f64_rowsum']).abs().max() / fx['scores_f64_rowsum'].abs().max()
    assert rel < 2e-5                       # fp32 run against the fp64 reference (ref32-vs-ref64 is ~1e-4 absolute here)
    if 'planted' in name:
        planted = fx['data']['planted_matches0']
        has = planted >= 0
        assert (fx['matches0'][has] == planted[has]).float().mean() > 0.995


def test_planted_matches_are_recovered(golden):
    fx = golden('C1_planted')
    planted = fx['data']['planted_matches0']
    m0 = fx['matches0']
    has = planted >= 0
    assert has.sum() >= 300
    assert torch.equal(m0[has], planted[has])              # every planted pair is recovered


def test_sinkhorn_marginals():
    """Property of the algorithm (optimal_transport.py:20-28): after the v update the column
    marginals of exp(Z+u+v) equal b exactly, the row marginals approximately."""
    torch.manual_seed(0)
    s = torch.randn(2, 30, 41, dtype=torch.float64) * 3
    lp = O.matching_log_probs(s, torch.tensor(1.0, dtype=torch.float64), 200, 1.0)
    m, n = 30, 41
    p = (lp + (-torch.log(torch.tensor(float(m + n))))).exp()
    col = p.sum(1)
    assert torch.allclose(col[:, :-1], torch.full((2, n), 1.0 / (m + n), dtype=torch.float64), atol=1e-12)
    assert torch.allclose(col[:, -1], torch.full((2,), m / (m + n), dtype=torch.float64), atol=1e-12)
    assert torch.allclose(p.sum(2)[:, :-1], torch.full((2, m), 1.0 / (m + n), dtype=torch.float64), atol=1e-6)


def test_extract_matches_ties_first_index():
    s = torch.full((1, 4, 4), -5.0)
    s[0, 0, 1] = s[0, 0, 2] = -0.1          # row tie -> first index (1)
    s[0, 1, 1] = -0.2
    out = O.extract_matches(s, 0.2)
    assert out['matches0'][0, 0].item() == 1
    assert out['matches0'][0, 1].item() == -1      # column 1's best row is 0, not mutual


def test_oracle_equals_staged_reference():
    """oracle/_ref (oracle/build_ref.py: the unmodified reference files, staged so that they travel to the GPU box and serve as
    bench.py's `cpu_baseline.kind = "reference"`): the live reference module and the oracle restatement must agree bit for bit
    on fresh seeds - including `use_offset`, a regularisation != 1 and 6 side-info channels, which no committed fixture of the
    big configurations covers."""
    from oracle.build_ref import import_reference
    ref = import_reference()
    if ref is None:
        pytest.skip('oracle/_ref is not staged (run `python oracle/build_ref.py` where /root/reference exists)')
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
    SuperGlueRef = ref[0]
    # the option rows of tests/test_gpu_parity.py::test_forward_matches_oracle; `images`: sizes from image tensors, which take
    # precedence over image*_size (set wrong on purpose)
    for seed, kw, (n, m), images in [
            (11, dict(descriptor_dim=64, num_stages=2, num_iters=15), (97, 61), False),
            (12, dict(descriptor_dim=128, num_stages=2, num_iters=7, side_info_size=6, use_offset=True, reg=0.7), (50, 75), False),
            (13, dict(descriptor_dim=192, num_heads=3, num_stages=2, num_iters=10), (40, 33), False),
            (14, dict(descriptor_dim=64, num_heads=1, num_stages=2, num_iters=10), (40, 33), False),
            (15, dict(descriptor_dim=96, num_heads=3, num_stages=2, num_iters=10), (40, 33), False),
            (16, dict(descriptor_dim=32, num_heads=4, num_stages=2, num_iters=10), (40, 33), False),
            (17, dict(descriptor_dim=64, num_stages=2, num_iters=10, hidden_layers_sizes=()), (40, 33), False),
            (18, dict(descriptor_dim=64, num_stages=2, num_iters=10, hidden_layers_sizes=(30, 50)), (40, 33), False),
            (19, dict(descriptor_dim=64, num_stages=2, num_iters=10, side_info_size=0), (40, 33), False),
            (20, dict(descriptor_dim=64, num_stages=2, num_iters=10), (40, 33), True)]:
        cfg = default_config(**kw)
        sd = synthetic_state_dict(cfg, seed=seed)
        data = synthetic_pairs(2, n, m, cfg['descriptor_dim'], cfg['positional_encoding']['side_info_size'], family='planted', seed=seed)
        if images:
            data['image0'], data['image1'] = torch.zeros(2, 1, 500, 700), torch.zeros(2, 1, 640, 480)
            data['image0_size'] = data['image1_size'] = (2000, 1000)
        model = SuperGlueRef(dict(cfg)).eval()
        model.load_state_dict(sd, strict=True)
        with torch.no_grad():
            want = model(data)
        got = O.run(sd, cfg, data, 0.2)
        for key in ('scores', 'context_descriptors0', 'context_descriptors1'):
            assert torch.equal(got[key], want[key]), (kw, key)


def test_label_and_loss_oracles_equal_staged_reference():
    """The two neighbouring steps on fresh seeds, live against the staged reference (oracle/_ref): ground-truth matches from a
    homography (models/gt_matches_generation.py:17-93 vs oracle/gt_matches_oracle.py) and the matching loss
    (utils/losses.py:7-53 vs oracle/loss_oracle.py), both bit for bit."""
    from oracle.build_ref import import_reference
    ref = import_reference()
    if ref is None:
        pytest.skip('oracle/_ref is not staged (run `python oracle/build_ref.py` where /root/reference exists)')
    from oracle import gt_matches_oracle as G
    from oracle import loss_oracle as L
    _, ref_criterion, ref_generate = ref
    for seed, (b, n, m) in [(21, (2, 60, 45)), (22, (3, 33, 80))]:
        g = torch.Generator().manual_seed(seed)
        k0 = torch.rand(b, n, 2, generator=g) * torch.tensor([640.0, 480.0])
        H = torch.tensor([[0.9, 0.05, 20.0], [-0.04, 0.95, 12.0], [1e-5, 2e-5, 1.0]]).repeat(b, 1, 1)
        k0h = torch.cat([k0, torch.ones(b, n, 1)], -1) @ H.transpose(1, 2)
        k0w = k0h[..., :2] / k0h[..., 2:]
        npl = min(n, m // 2)
        k1 = torch.cat([k0w[:, :npl] + 0.3 * torch.randn(b, npl, 2, generator=g),            # planted correspondences + clutter
                        torch.rand(b, m - npl, 2, generator=g) * torch.tensor([640.0, 480.0])], 1)
        tf = {'type': ['perspective'] * b, 'H': H}
        feat = lambda k: {'keypoints': k, 'local_descriptors': torch.zeros(b, k.shape[1], 4), 'side_info': torch.zeros(b, k.shape[1], 1)}
        _, y_true = ref_generate({'transformation': tf}, feat(k0), feat(k1), positive_threshold=3.0, negative_threshold=5.0)
        g0, g1, _ = G.gt_matches(k0, k1, tf)
        assert torch.equal(g0, y_true['gt_matches0']) and torch.equal(g1, y_true['gt_matches1'])
        assert int((g0 >= 0).sum()) > 0
        scores = torch.log_softmax(torch.randn(b, n + 1, m + 1, generator=g), dim=-1)
        y_pred = {'scores': scores, 'context_descriptors0': torch.randn(b, 8, n, generator=g), 'context_descriptors1': torch.randn(b, 8, m, generator=g)}
        want = ref_criterion(y_true, y_pred, margin=None)
        got = L.criterion({'gt_matches0': g0, 'gt_matches1': g1}, {'scores': scores})
        assert torch.equal(got['loss'], want['loss']) and float(got['metric_loss']) == float(want['metric_loss']) == 0.0
