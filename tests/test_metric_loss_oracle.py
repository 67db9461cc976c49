"""Metric terms of the matching loss (criterion with a margin), on the CPU: the oracle (oracle/metric_loss_oracle.py) against the
fixtures minted from the UNMODIFIED reference ``utils.losses.criterion`` with autograd (oracle/gen_golden_metric_loss.py), against
the staged reference itself on fresh inputs, the fixtures' own contents, and the argument checks of og_metric_loss_fwd."""
import ctypes as C
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import metric_loss_oracle as M                         # noqa: E402  (checker only)
from oracle.gen_golden_metric_loss import metric_inputs, CASES     # noqa: E402  (input generator, no reference import at module level)

GOLDEN = ['metric_small', 'metric_empty', 'metric_ties', 'metric_m01', 'metric_m1']
SELECTIONS = ('n0', 'u0', 'n1', 'u1')


def _fx(name):
    return torch.load(os.path.join(ROOT, 'tests', 'golden', name + '.pt'), weights_only=False)


@pytest.mark.parametrize('name', GOLDEN)
def test_oracle_matches_reference_fixture(name):
    fx = _fx(name)
    gt0, gt1, margin = fx['gt_matches0'], fx['gt_matches1'], fx['case'][8]
    x0 = fx['c0'].double().requires_grad_(True)
    x1 = fx['c1'].double().requires_grad_(True)
    out = M.metric_terms(gt0, gt1, x0, x1, margin)
    assert abs(float(out["metric_loss"].detach()) - float(fx["metric_loss_f64"])) <= 1e-12
    out['metric_loss'].backward()
    for g, ref in ((x0.grad, fx['dc0_f64']), (x1.grad, fx['dc1_f64'])):
        assert float((g - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max()))
    for k in SELECTIONS:
        assert torch.equal(out[k], fx['selections'][k]), k
    for k in ('a0', 'a1', 'au0', 'au1', 'gap_n0', 'gap_u0', 'gap_n1', 'gap_u1'):
        assert torch.equal(out[k], fx['selections'][k]), k
    o32 = M.metric_terms(gt0, gt1, fx['c0'], fx['c1'], margin)
    assert abs(float(o32['metric_loss']) - float(fx['metric_loss_f32'])) <= 1e-6 * max(1.0, abs(float(fx['metric_loss_f32'])))


def test_fixture_contents():
    small = _fx('metric_small')
    assert (small['gt_matches0'] == -2).any() and (small['gt_matches1'] == -2).any()          # ignore entries present
    empty = _fx('metric_empty')
    assert not (empty['gt_matches0'][1] >= 0).any() and not (empty['gt_matches1'][2] == -1).any()
    ties = _fx('metric_ties')
    half = ties['c1'].shape[2] // 2
    assert torch.equal(ties['c1'][:, :, :half], ties['c1'][:, :, half:])
    assert (ties['selections']['gap_u0'] == 0).all()                                          # every row argmin is an exact tie
    act = lambda fx: sum(int((fx['selections'][k] > 0).sum()) for k in ('a0', 'a1', 'au0', 'au1'))
    tot = lambda fx: sum(fx['selections'][k].numel() for k in ('a0', 'a1', 'au0', 'au1'))
    m01, m1 = _fx('metric_m01'), _fx('metric_m1')
    assert m01['case'][8] == 0.1 and 0 < act(m01) < tot(m01) // 10                           # a few hinges active
    assert m1['case'][8] == 1.0 and act(m1) == tot(m1)                                        # all of them
    large = _fx('metric_large')
    assert 'c0' not in large and large['case'][:4] == (2, 1024, 1024, 256)
    assert large['selections']['n0'].shape == (2, 1024)


def test_train_metric_decisions_are_far_from_flipping():
    fx = _fx('train_metric')
    sel = fx['selections']
    out = dict(sel)
    gt0, gt1 = fx['gt_matches0'], fx['gt_matches1']
    used = M.used_margins(gt0, gt1, out)
    assert all(v.numel() > 0 for v in used.values())
    assert min(float(v.min()) for v in used.values()) >= 1e-4
    assert fx['smallest_margin'] >= 1e-4
    assert fx['margin'] == 0.5 and fx['metric_weight'] == 0.5 and fx['nll_weight'] == 1.0
    ref = M.metric_terms(gt0, gt1, fx['context_descriptors0_f64'].double(), fx['context_descriptors1_f64'].double(), fx['margin'])
    for k in SELECTIONS:                                       # the fp32-rounded descriptors select the same negatives
        assert torch.equal(ref[k], sel[k]), k


def _reference():
    from oracle.build_ref import import_reference
    got = import_reference()
    if got is None:
        pytest.skip('oracle/_ref is not staged')
    return got[1]


def _random_case(B, n, m, d, seed, dup=False):
    g = torch.Generator().manual_seed(seed)
    gt0 = torch.full((B, n), -1, dtype=torch.int64)
    gt1 = torch.full((B, m), -1, dtype=torch.int64)
    for b in range(B):
        k = min(n, m) // 2 if min(n, m) > 1 else 1
        src, dst = torch.randperm(n, generator=g)[:k], torch.randperm(m, generator=g)[:k]
        gt0[b, src], gt1[b, dst] = dst, src
        gt0[b, (torch.rand(n, generator=g) < 0.1) & (gt0[b] < 0)] = -2
    c0 = torch.randn(B, d, n, generator=g)
    c1 = torch.randn(B, d, m, generator=g)
    if dup:
        c1 = torch.cat([c1[:, :, : m // 2], c1[:, :, : m - m // 2]], dim=2)
    return gt0, gt1, c0, c1


@pytest.mark.parametrize('B,n,m,d,seed,dup', [(2, 40, 33, 32, 51, False), (3, 37, 1, 16, 52, False), (2, 1, 30, 16, 53, False),
                                              (2, 30, 40, 24, 54, True), (1, 300, 257, 64, 55, False), (2, 20, 18, 8, 56, False)])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_oracle_equals_staged_reference(B, n, m, d, seed, dup, dtype):
    """Fresh seeds, torch.equal: value, gradients (m == 1: the positive is its own negative; duplicated columns: exact ties)."""
    criterion = _reference()
    gt0, gt1, c0, c1 = _random_case(B, n, m, d, seed, dup)
    res = []
    for f in ('ref', 'oracle'):
        x0, x1 = c0.to(dtype).requires_grad_(True), c1.to(dtype).requires_grad_(True)
        if f == 'ref':
            v = criterion({'gt_matches0': gt0, 'gt_matches1': gt1}, {'context_descriptors0': x0, 'context_descriptors1': x1,
                                                                     'scores': torch.zeros(B, n + 1, m + 1, dtype=dtype)}, margin=0.5)['metric_loss']
        else:
            v = M.metric_terms(gt0, gt1, x0, x1, 0.5)['metric_loss']
        v.backward()
        res.append((v.detach(), x0.grad, x1.grad))
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_metric_inputs_regenerate_metric_large():
    fx = _fx('metric_large')
    gt0, gt1, c0, c1 = metric_inputs(*CASES['metric_large'])
    assert torch.equal(gt0, fx['gt_matches0']) and torch.equal(gt1, fx['gt_matches1'])
    assert c0.shape == (2, 256, 1024) and c1.shape == (2, 256, 1024)


def test_metric_abi_rejects_bad_arguments_without_a_gpu():
    from openglue_b200 import _cabi
    lib = _cabi.lib()
    FP32, TF32X3 = _cabi.OG_PREC_FP32, _cabi.OG_PREC_TF32X3
    assert lib.og_metric_loss_workspace_bytes(2, 64, 37, 52, 1, TF32X3) > lib.og_metric_loss_workspace_bytes(2, 64, 37, 52, 0, TF32X3) > 0
    assert lib.og_metric_loss_workspace_bytes(2, 64, 37, 52, 0, FP32) > 0
    for args in ((0, 64, 37, 52), (65536, 64, 37, 52), (2, 0, 37, 52), (2, 64, 0, 52), (2, 64, 37, 0)):
        assert lib.og_metric_loss_workspace_bytes(*args, 0, FP32) == -1, args
    assert lib.og_metric_loss_workspace_bytes(2, 64, 37, 52, 0, _cabi.OG_PREC_FP16X3) == -1
    p = C.c_void_p(256)                                      # never dereferenced: every call below fails its checks first
    good = dict(c0=p, c1=p, gt0=p, gt1=p, B=2, d=64, n=37, m=52, mu=0.5, prec=FP32, loss=p, n0=p, u0=p, n1=p, u1=p, dc0=None, dc1=None,
                gs=1.0, ws=p, wsb=1 << 30, st=None)

    def call(**kw):
        a = dict(good, **kw)
        return lib.og_metric_loss_fwd(*a.values())

    for k in ('c0', 'c1', 'gt0', 'gt1', 'loss', 'n0', 'u0', 'n1', 'u1', 'ws'):
        assert call(**{k: None}) == -1, k                    # OG_EINVAL, no CUDA call made
    assert call(dc0=p) == -1 and call(dc1=p) == -1
    for kw in (dict(B=0), dict(B=65536), dict(d=0), dict(n=0), dict(m=-1), dict(prec=_cabi.OG_PREC_FP16X3)):
        assert call(**kw) == -1, kw
    assert b'metric_loss' in lib.og_last_error()


def test_product_does_not_import_the_metric_oracle():
    pkg = os.path.join(ROOT, 'openglue_b200')
    for name in os.listdir(pkg):
        if name.endswith('.py'):
            with open(os.path.join(pkg, name)) as f:
                assert 'metric_loss_oracle' not in f.read(), name
