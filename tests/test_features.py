"""Local features -> matcher inputs (csrc/features.cuh, openglue_b200/features.py): the LAF side information of
prepare_features_output, the ordered compaction of the matches, and OpenGlueMatcher end to end.

1. CPU: converter names / dimensions / NameError as in the reference; the kornia restatements with which the fixtures were minted
   (oracle/gen_golden_features.py) reproduce them; the matcher inputs regenerate bit for bit; CPU tensors are refused.
2. GPU, og_prepare_features through the C ABI into NaN-poisoned outputs followed by guard regions: every method x log_response,
   1 .. 32 x 4096 keypoints.  Non-log columns bit-equal to the reference's fp32 result (by at most 2 ulp on the few frames where
   ATen's CPU square root is not correctly rounded, and there bit-equal to an IEEE restatement), log columns within 2 ulp of it
   and within 1e-6 of its fp64 result.
3. GPU, og_match_compact against torch boolean indexing, on crafted matches (valid rows with a zero score, invalid rows with a
   positive one).
4. GPU, OpenGlueMatcher on the two reference-minted matcher fixtures in every precision, and on a SuperPointNet image pair against
   a by-hand composition of the same public pieces.
"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'oracle'))
from gen_golden_features import (MATCH_CASES, METHODS, get_laf_center, get_laf_scale, inputs_sha256,  # noqa: E402
                                 match_config, matcher_inputs)

import openglue_b200  # noqa: E402
from openglue_b200 import features as FT  # noqa: E402
from openglue_b200._cabi import ptr as _p, stream as _st  # noqa: E402

GOLDEN = os.path.join(HERE, 'golden')
DEV = 'cuda:0'
GUARD = 1024
INT_POISON = -0x5a5a5a5a
TOL = 1e-4
DIMS = {'none': 0, 'scale': 1, 'rotation': 2, 'scale_rotation': 3, 'affine': 5}
CODES = {'none': 0, 'scale': 1, 'rotation': 2, 'scale_rotation': 3, 'affine': 4}
_cache = {}


def _fx(name):
    if name not in _cache:
        _cache[name] = torch.load(os.path.join(GOLDEN, name + '.pt'), weights_only=False)
    return _cache[name]


def log_columns(method, log_response):
    """indices of the side-information columns that are logarithms"""
    cols = [0] if log_response else []
    return cols + ([1] if method in ('scale', 'scale_rotation', 'affine') else [])


def side_restated(lafs, responses, method, log_response):
    """the reference's prepare_features_output + converter (models/laf_converter.py, models/features/utils.py:54-65) in plain torch
    on the restated kornia helpers"""
    r = responses.unsqueeze(-1)
    if log_response:
        r = (r + 0.1).log()
    s = get_laf_scale(lafs).squeeze(-1)                        # [B, N, 1]
    cols = [r]
    if method in ('scale', 'scale_rotation', 'affine'):
        cols.append(torch.log(s))
    if method in ('rotation', 'scale_rotation'):
        cols.append(torch.flip(lafs[..., 0, :-1], dims=(-1,)) / s)
    if method == 'affine':
        cols.append(torch.flatten(lafs[..., :-1], start_dim=2) / s)
    return torch.cat(cols, -1)


def side_ieee(lafs, responses, method, log_response):
    """what og_prepare_features computes: the same operations in numpy float32, each one IEEE-rounded (numpy's float32 square root
    is correctly rounded), the logarithms correctly rounded from float64.  [B, N, 1 + dim]"""
    f32 = np.float32
    L = lafs.reshape(-1, 2, 3).numpy()
    a00, a01, a10, a11 = L[:, 0, 0], L[:, 0, 1], L[:, 1, 0], L[:, 1, 1]
    r = responses.reshape(-1).numpy()
    if log_response:
        r = np.log((r + f32(0.1)).astype(np.float64)).astype(f32)
    s = np.sqrt(np.abs((a00 * a11 - a10 * a01) + f32(1e-10)))
    cols = [r]
    if method in ('scale', 'scale_rotation', 'affine'):
        cols.append(np.log(s.astype(np.float64)).astype(f32))
    if method in ('rotation', 'scale_rotation'):
        cols += [a01 / s, a00 / s]
    if method == 'affine':
        cols += [a00 / s, a01 / s, a10 / s, a11 / s]
    return torch.from_numpy(np.stack(cols, -1)).view(*lafs.shape[:2], -1)


def sqrt_not_rounded(fx):
    """[B, N]: frames whose scale the reference's float32 run got from a square root that is not correctly rounded.  ATen's CPU
    sqrt (vectorised, Sleef) can be 1 ulp off the IEEE result; on those frames every quotient by s may differ by up to 2 ulp from
    the kernel's, which uses the correctly rounded square root (as torch does on CUDA)."""
    ref = fx['side'][('affine', False)][..., 2:]
    return (side_ieee(fx['lafs'], fx['responses'], 'affine', False)[..., 2:] != ref).any(-1)


def ulp(x):
    x = x.abs().float()
    return torch.nextafter(x, torch.full_like(x, float('inf'))) - x


# ---------------------------------------------------------------------------------------------------------------------
# CPU

def test_converter_names_dimensions_and_errors():
    for name, dim in DIMS.items():
        for spelled in (name, name.upper(), name.title()):
            conv = openglue_b200.get_laf_to_sideinfo_converter(spelled)
            assert conv.side_info_dim == dim
    assert openglue_b200.get_laf_to_sideinfo_converter().side_info_dim == 0
    with pytest.raises(NameError, match='^Unexpected name for the method: Scale-Rotation$'):
        openglue_b200.get_laf_to_sideinfo_converter('Scale-Rotation')


def test_restated_kornia_helpers_reproduce_the_fixtures():
    fx = _fx('feat_convert')
    lafs, resp = fx['lafs'], fx['responses']
    assert torch.equal(get_laf_center(lafs), fx['keypoints'])
    # frames where the square root of the fixture's run or of this CPU's ATen is not the correctly rounded one: an ulp there
    # moves every column derived from s by a few ulp
    off = sqrt_not_rounded(fx)
    here = (side_restated(lafs, resp, 'affine', False)[..., 2:] != side_ieee(lafs, resp, 'affine', False)[..., 2:]).any(-1)
    exact = ~(off | here)
    for method in METHODS:
        for lr in (False, True):
            for dt, ref in ((torch.float32, fx['side'][(method, lr)]), (torch.float64, fx['side_f64'][(method, lr)])):
                ours = side_restated(lafs.to(dt), resp.to(dt), method, lr)
                assert ours.shape == ref.shape == (*lafs.shape[:2], 1 + DIMS[method])
                if dt == torch.float64:
                    assert ((ours - ref).abs() <= 1e-14 * ref.abs().clamp_min(1)).all(), (method, lr)
                    continue
                logs = log_columns(method, lr)
                rest = [c for c in range(ours.shape[-1]) if c not in logs]
                assert torch.equal(ours[exact][:, rest], ref[exact][:, rest]), (method, lr)
                assert ((ours - ref).abs() <= 4 * ulp(ref) + 3e-7 * len(logs)).all(), (method, lr)
                if logs:
                    assert ((ours[exact][:, logs] - ref[exact][:, logs]).abs() <= 2 * ulp(ref[exact][:, logs])).all(), (method, lr)
    # the kernel's arithmetic (the IEEE restatement) is the reference's, up to ATen's CPU square root on a few frames
    assert int(off.sum()) <= 0.005 * off.numel()
    for method in METHODS:
        ieee, ref = side_ieee(lafs, resp, method, False), fx['side'][(method, False)]
        rest = [c for c in range(ref.shape[-1]) if c not in log_columns(method, False)]
        assert torch.equal(ieee[~off][:, rest], ref[~off][:, rest])
        assert ((ieee[off][:, rest] - ref[off][:, rest]).abs() <= 2 * ulp(ref[off][:, rest])).all()
    # the frames the fixture promises: reflections, near-singular frames where the 1e-10 dominates, identity frames, zero responses
    det = lafs[..., 0, 0].double() * lafs[..., 1, 1] - lafs[..., 1, 0].double() * lafs[..., 0, 1]
    assert (det < 0).sum() > 50 and (det.abs() < 1e-11).sum() >= 60 and (resp == 0).sum() > 50
    assert (lafs[..., :2] == torch.eye(2)).all(-1).all(-1).sum() >= 64


@pytest.mark.parametrize('name', list(MATCH_CASES))
def test_matcher_inputs_regenerate(name):
    """the matcher fixtures store no inputs: they regenerate bit for bit from the seed, and the reference gathered its LAFs from them"""
    fx = _fx(name)
    c = fx['case']
    inputs = matcher_inputs(c['batch'], c['n'], c['m'], fx['config']['descriptor_dim'], c['seed'])
    assert inputs_sha256(inputs) == fx['sha256']
    ref = fx['f32']
    bi, ij = ref['batch_indexes'], ref['original_matching_idxs']
    assert torch.equal(ref['lafs0'][0], inputs['lafs0'][bi, ij[:, 0]])
    assert torch.equal(ref['lafs1'][0], inputs['lafs1'][bi, ij[:, 1]])


def test_cpu_tensors_are_refused():
    from openglue_b200 import SuperGlue
    from openglue_b200.synthetic import default_config
    fx = _fx('feat_convert')
    lafs, resp = fx['lafs'], fx['responses']
    conv = openglue_b200.get_laf_to_sideinfo_converter('affine')
    with pytest.raises(RuntimeError, match='CUDA'):
        conv(lafs)
    with pytest.raises(RuntimeError, match='CUDA'):
        openglue_b200.get_laf_to_sideinfo_converter('none')(lafs)
    with pytest.raises(RuntimeError, match='CUDA'):
        openglue_b200.prepare_features_output(lafs, resp, torch.zeros(*lafs.shape[:2], 8), conv)
    with pytest.raises(RuntimeError, match='CUDA'):
        FT.compact_matches(torch.full(lafs.shape[:2], -1), torch.zeros(lafs.shape[:2]), lafs, lafs)
    sg = SuperGlue(default_config(descriptor_dim=32, num_stages=1, side_info_size=6))
    with pytest.raises(TypeError):
        openglue_b200.OpenGlueMatcher(None, torch.nn.Identity(), match_config(False))
    matcher = openglue_b200.OpenGlueMatcher(None, sg, match_config(False))
    data = {'lafs0': lafs, 'responses0': resp, 'descriptors0': torch.zeros(*lafs.shape[:2], 32),
            'lafs1': lafs, 'responses1': resp, 'descriptors1': torch.zeros(*lafs.shape[:2], 32),
            'image0': torch.zeros(2, 1, 8, 8), 'image1': torch.zeros(2, 1, 8, 8)}
    with pytest.raises(RuntimeError, match='CUDA'):
        matcher(data)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the two kernels through the C ABI

def _lib():
    from openglue_b200 import _cabi
    return _cabi.lib()


def _check(rc, what):
    from openglue_b200 import _cabi
    _cabi.check(rc, what)


def _poisoned(n, dtype=torch.float32):
    return torch.full((n + GUARD,), float('nan') if dtype.is_floating_point else INT_POISON, dtype=dtype, device=DEV)


def _untouched(t):
    return bool((torch.isnan(t) if t.is_floating_point() else t == INT_POISON).all())


@pytest.mark.gpu
@pytest.mark.parametrize('R', [1, 33, 1034, 4097, 32 * 4096])
@pytest.mark.parametrize('log_response', [False, True])
@pytest.mark.parametrize('method', METHODS)
def test_prepare_features_kernel(method, log_response, R):
    fx = _fx('feat_convert')
    rows = fx['lafs'].shape[0] * fx['lafs'].shape[1]
    idx = torch.arange(R) % rows                                       # the fixture's frames, repeated to R keypoints
    lafs = fx['lafs'].view(rows, 2, 3)[idx].to(DEV)
    resp = fx['responses'].view(rows)[idx].to(DEV)
    ref = fx['side'][(method, log_response)].view(rows, -1)[idx]
    ref64 = fx['side_f64'][(method, log_response)].view(rows, -1)[idx]
    ieee = side_ieee(fx['lafs'], fx['responses'], method, log_response).view(rows, -1)[idx]
    off = sqrt_not_rounded(fx).view(rows)[idx]
    width = 1 + DIMS[method]
    kpts, side = _poisoned(2 * R), _poisoned(width * R)
    _check(_lib().og_prepare_features(_p(lafs), _p(resp), R, CODES[method], int(log_response), _p(kpts), _p(side), _st()),
           'og_prepare_features')
    torch.cuda.synchronize()
    assert _untouched(kpts[2 * R:]) and _untouched(side[width * R:])
    assert torch.equal(kpts[:2 * R].view(R, 2).cpu(), fx['keypoints'].view(rows, 2)[idx])
    ours = side[:width * R].view(R, width).cpu()
    logs = log_columns(method, log_response)
    rest = [c for c in range(width) if c not in logs]
    # non-log columns: bit-equal to the reference's fp32 result, except by an ulp where its square root was not correctly
    # rounded (then a quotient by s moves by at most 2 ulp); bit-equal to the IEEE restatement everywhere
    assert torch.equal(ours[:, rest], ieee[:, rest])
    assert torch.equal(ours[~off][:, rest], ref[~off][:, rest])
    assert ((ours[off][:, rest] - ref[off][:, rest]).abs() <= 2 * ulp(ref[off][:, rest])).all()
    if logs:
        e_ulp = float(((ours[~off][:, logs] - ref[~off][:, logs]).abs() / ulp(ref[~off][:, logs])).max()) if (~off).any() else 0.0
        e_ieee = float(((ours[:, logs] - ieee[:, logs]).abs() / ulp(ieee[:, logs])).max())
        e64 = float((ours[:, logs].double() - ref64[:, logs]).abs().max())
        print(f'\n[{method} log_response={log_response} R={R}] log columns: {e_ulp:.1f} ulp from the reference fp32 (bound 2), '
              f'{e_ieee:.1f} ulp from the correctly rounded log (bound 2), {e64:.2e} from fp64 (bound 1e-6); '
              f'{int(off.sum())} frames with a 1-ulp reference sqrt')
        assert e_ulp <= 2 and e_ieee <= 2 and e64 <= 1e-6


@pytest.mark.gpu
def test_converter_and_prepare_features_output():
    fx = _fx('feat_convert')
    lafs, resp = fx['lafs'].to(DEV), fx['responses'].to(DEV)
    desc = torch.randn(*lafs.shape[:2], 16, device=DEV)
    for method in METHODS:
        conv = openglue_b200.get_laf_to_sideinfo_converter(method)
        alone = conv(lafs)                                             # the converter alone: no response column
        assert alone.shape == (*lafs.shape[:2], DIMS[method]) and alone.is_cuda
        for lr in (False, True):
            out = openglue_b200.prepare_features_output(lafs, resp, desc, conv, log_response=lr)
            assert set(out) == {'keypoints', 'side_info', 'local_descriptors'}
            assert torch.equal(out['keypoints'].cpu(), fx['keypoints'])
            assert torch.equal(out['side_info'][..., 1:], alone)
            ieee = side_ieee(fx['lafs'], fx['responses'], method, lr)
            rest = [c for c in range(ieee.shape[-1]) if c not in log_columns(method, lr)]
            assert torch.equal(out['side_info'].cpu()[..., rest], ieee[..., rest])
            assert out['local_descriptors'] is desc
    out = openglue_b200.prepare_features_output(lafs, resp, desc, conv, permute_desc=True)
    assert out['local_descriptors'].shape == (lafs.shape[0], 16, lafs.shape[1])


def _compact_ref(matches0, mscores0, lafs0, lafs1):
    """inference.py:192-209 in plain torch: boolean indexing with matches0 != -1"""
    B, n = matches0.shape
    mask = matches0 != -1
    arange0 = torch.arange(n, device=matches0.device)[None].expand(B, -1)
    bi = torch.arange(B, device=matches0.device)[:, None].expand(-1, n)[mask]
    i, j = arange0[mask], matches0[mask]
    l0, l1 = lafs0[bi, i][None], lafs1[bi, j][None]
    return {'original_matching_idxs': torch.stack([i, j], -1), 'batch_indexes': bi, 'confidence': mscores0[mask],
            'lafs0': l0, 'lafs1': l1, 'keypoints0': l0[..., 2][0], 'keypoints1': l1[..., 2][0]}


@pytest.mark.gpu
@pytest.mark.parametrize('B,n,m,share', [(3, 2500, 700, 0.4), (1, 1, 1, 1.0), (2, 1024, 1030, 1.0), (2, 300, 50, 0.0)])
def test_match_compact_kernel(B, n, m, share):
    g = torch.Generator().manual_seed(B * n + m)
    matches0 = torch.randint(0, m, (B, n), generator=g)
    matches0[torch.rand(B, n, generator=g) >= share] = -1
    if B > 1 and share < 1:
        matches0[1] = -1                                               # a pair without a match
    mscores0 = torch.rand(B, n, generator=g)
    mscores0[:, ::5] = 0.0                                             # valid rows with a zero score (exp underflow, negative threshold),
    lafs0, lafs1 = torch.randn(B, n, 2, 3, generator=g), torch.randn(B, m, 2, 3, generator=g)   # invalid rows with a positive one
    dev = [t.to(DEV) for t in (matches0, mscores0, lafs0, lafs1)]
    cap = B * n
    pair, ij, total = _poisoned(cap, torch.int64), _poisoned(2 * cap, torch.int64), _poisoned(1, torch.int64)
    conf, l0, l1, k0, k1 = _poisoned(cap), _poisoned(6 * cap), _poisoned(6 * cap), _poisoned(2 * cap), _poisoned(2 * cap)
    _check(_lib().og_match_compact(*[_p(t) for t in dev], B, n, m, _p(pair), _p(ij), _p(conf), _p(l0), _p(l1), _p(k0), _p(k1), _p(total),
                                   _st()), 'og_match_compact')
    torch.cuda.synchronize()
    nc = int(total[0])
    ref = _compact_ref(matches0, mscores0, lafs0, lafs1)
    assert nc == ref['confidence'].numel()
    assert _untouched(total[1:])
    for buf, w in ((pair, 1), (ij, 2), (conf, 1), (l0, 6), (l1, 6), (k0, 2), (k1, 2)):
        assert _untouched(buf[w * nc:])                                # rows past the count and the guard
    assert torch.equal(pair[:nc].cpu(), ref['batch_indexes'])
    assert torch.equal(ij[:2 * nc].view(nc, 2).cpu(), ref['original_matching_idxs'])
    assert torch.equal(conf[:nc].cpu(), ref['confidence'])
    assert torch.equal(l0[:6 * nc].view(1, nc, 2, 3).cpu(), ref['lafs0'])
    assert torch.equal(l1[:6 * nc].view(1, nc, 2, 3).cpu(), ref['lafs1'])
    assert torch.equal(k0[:2 * nc].view(nc, 2).cpu(), ref['keypoints0'])
    assert torch.equal(k1[:2 * nc].view(nc, 2).cpu(), ref['keypoints1'])
    # the Python form returns the same, with the reference's shapes
    out = FT.compact_matches(*dev)
    for k, v in ref.items():
        assert out[k].shape == v.shape and torch.equal(out[k].cpu(), v), k


# ---------------------------------------------------------------------------------------------------------------------
# GPU: OpenGlueMatcher

def _superglue(cfg, precision):
    from openglue_b200 import SuperGlue
    from openglue_b200.synthetic import synthetic_state_dict
    cfg = dict(cfg)
    cfg['precision'] = precision
    sg = SuperGlue(cfg).eval()
    sg.load_state_dict(synthetic_state_dict(cfg, seed=0), strict=True)
    return sg.to(DEV)


def _dense(out, B, n):
    """compact list -> matches0 [B, n] (-1: no match)"""
    m0 = torch.full((B, n), -1, dtype=torch.int64)
    ij = out['original_matching_idxs'].cpu()
    m0[out['batch_indexes'].cpu(), ij[:, 0]] = ij[:, 1]
    return m0


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['fp16x3', 'tf32x3', 'fp32'])
@pytest.mark.parametrize('name', list(MATCH_CASES))
def test_matcher_matches_reference(name, precision):
    fx = _fx(name)
    c = fx['case']
    B, n = c['batch'], c['n']
    inputs = matcher_inputs(B, n, c['m'], fx['config']['descriptor_dim'], c['seed'])
    assert inputs_sha256(inputs) == fx['sha256']
    data = {k: v.to(DEV) for k, v in inputs.items()}
    data['image0'] = torch.empty(B, 1, *c['image_hw'], device=DEV)
    data['image1'] = torch.empty(B, 1, *c['image_hw'], device=DEV)
    sg = _superglue(fx['config'], precision)
    matcher = openglue_b200.OpenGlueMatcher(None, sg, match_config(c['log_transform_response'], fx['match_threshold']))
    out = matcher(dict(data))
    ref = fx['f32']
    for k, v in ref.items():                                           # [NC, ...] / [1, NC, 2, 3], as the reference's
        assert out[k].dtype == v.dtype and out[k].dim() == v.dim() and out[k].is_cuda, k
        assert out[k].shape[-1] == v.shape[-1] and (not k.startswith('lafs') or out[k].shape[0] == 1), k
    # decisive rows (the parity tests' rule): row / column top-2 gap and distance to the threshold beyond 2 x the bound
    bound = max(TOL, 2 * fx['ref32_vs_ref64_max_abs'])
    i0 = fx['row_argmax_f64']
    decisive = (fx['row_top2_gap_f64'] > 2 * bound) & (fx['col_top2_gap_f64'].gather(1, i0) > 2 * bound) & \
               ((fx['matching_scores0_f64'] - fx['match_threshold']).abs() > 2 * bound)
    ours_m0, ref_m0 = _dense(out, B, n), _dense(ref, B, n)
    bi, ii = out['batch_indexes'].cpu(), out['original_matching_idxs'][:, 0].cpu()
    rb, ri = ref['batch_indexes'], ref['original_matching_idxs'][:, 0]
    keep_ours, keep_ref = decisive[bi, ii], decisive[rb, ri]
    print(f'\n[{name} {precision}] {out["confidence"].numel()} matches (reference {ref["confidence"].numel()}), '
          f'{int((~decisive).sum())} rows not decisive, {int((ours_m0 != ref_m0).sum())} rows differ; bound {bound:.2e}')
    assert torch.equal(ours_m0[decisive], ref_m0[decisive])
    assert torch.equal(out['original_matching_idxs'].cpu()[keep_ours], ref['original_matching_idxs'][keep_ref])
    assert torch.equal(bi[keep_ours], rb[keep_ref])
    # confidence of the matches both sides report, against the reference's fp32 and fp64 runs
    both = (ours_m0 >= 0) & (ours_m0 == ref_m0)
    conf_ours = torch.full((B, n), float('nan'))
    conf_ours[bi, ii] = out['confidence'].cpu()
    conf_ref = torch.full((B, n), float('nan'))
    conf_ref[rb, ri] = ref['confidence']
    r64 = fx['f64']
    conf_64 = torch.full((B, n), float('nan'), dtype=torch.float64)
    conf_64[r64['batch_indexes'], r64['original_matching_idxs'][:, 0]] = r64['confidence']
    assert both.sum() > 0.9 * ref['confidence'].numel()
    assert (conf_ours[both] - conf_ref[both]).abs().max() <= TOL
    both64 = both & ~torch.isnan(conf_64)
    assert (conf_ours[both64].double() - conf_64[both64]).abs().max() <= TOL
    # gathered LAFs and keypoints: exact copies of the inputs
    ij = out['original_matching_idxs']
    assert torch.equal(out['lafs0'][0], data['lafs0'][out['batch_indexes'], ij[:, 0]])
    assert torch.equal(out['lafs1'][0], data['lafs1'][out['batch_indexes'], ij[:, 1]])
    assert torch.equal(out['keypoints0'], out['lafs0'][0, :, :, 2]) and torch.equal(out['keypoints1'], out['lafs1'][0, :, :, 2])
    # a repeat call is bit-identical
    again = matcher(dict(data))
    for k in ref:
        assert torch.equal(out[k], again[k]), k
    # nothing clears a threshold of 1: the reference's empty outputs
    empty = _fx('feat_match_affine')
    matcher.match_config = match_config(c['log_transform_response'], 1.0)
    none = matcher(dict(data))
    for k, shape in empty['empty_shapes'].items():
        assert tuple(none[k].shape) == shape and str(none[k].dtype) == empty['empty_dtypes'][k], k


@pytest.mark.gpu
@pytest.mark.parametrize('method', ['none', 'scale_rotation'])
def test_superpoint_image_pair(method):
    """SuperPointNet -> OpenGlueMatcher on a 480 x 640 pair equals the by-hand composition of SuperPointNet,
    prepare_features_output, MatchingCore and a torch boolean-index compaction"""
    from openglue_b200 import MatchingCore, SuperPointNet
    from openglue_b200.synthetic import default_config
    torch.manual_seed(0)
    net = SuperPointNet(max_keypoints=1024, keypoint_threshold=0.005).eval().to(DEV)

    class Front(torch.nn.Module):
        """the front-end with its unit descriptors scaled by 32 (as synthetic.py's desc_scale does): with random SuperGlue weights,
        unit descriptors leave the scores so flat that a single mutual match remains; scaled, a few survive, enough for the
        threshold to cut through them.  The match count is printed; the fixture tests above are the ones with many matches."""

        def forward(self, image):
            lafs, scores, desc = net(image)
            return lafs, scores, 32.0 * desc

    sp = Front()
    g = torch.Generator().manual_seed(7)
    base = torch.nn.functional.interpolate(torch.rand(1, 1, 64, 84, generator=g), size=(512, 672), mode='bilinear', align_corners=False)
    im0 = base[..., :480, :640].contiguous().to(DEV)
    im1 = base[..., 24:504, 16:656].contiguous().to(DEV)               # the same scene, shifted
    cfg = default_config(descriptor_dim=256, num_stages=2, num_iters=20, side_info_size=1 + DIMS[method])
    sg = _superglue(cfg, 'fp16x3')
    conv = openglue_b200.get_laf_to_sideinfo_converter(method)
    # by hand
    lafs0, sc0, d0 = sp(im0)
    lafs1, sc1, d1 = sp(im1)
    f0 = openglue_b200.prepare_features_output(lafs0, sc0, d0, conv)
    f1 = openglue_b200.prepare_features_output(lafs1, sc1, d1, conv)
    inp = {'image0': im0, 'image1': im1, **{k + '0': v for k, v in f0.items()}, **{k + '1': v for k, v in f1.items()}}
    probe = MatchingCore(sg, -1.0)(inp)                                # every mutual match: pick a threshold that cuts through them
    ms = probe['matching_scores0'][probe['matches0'] >= 0]
    thr = float(ms.median())
    res = MatchingCore(sg, thr)(inp)
    ref = _compact_ref(res['matches0'], res['matching_scores0'], lafs0, lafs1)
    # the matcher
    config = {'superglue': {'laf_to_sideinfo_method': method}, 'inference': {'match_threshold': thr}}
    data = {'image0': im0, 'image1': im1}
    out = openglue_b200.OpenGlueMatcher(sp, sg, config)(data)
    print(f'\n[{method}] {lafs0.shape[1]} / {lafs1.shape[1]} keypoints, {ms.numel()} mutual, {ref["confidence"].numel()} above {thr:.3f}')
    assert data['image0_size'] == [640, 480] and data['image1_size'] == [640, 480]
    assert 0 < ref['confidence'].numel() < ms.numel()
    for k, v in ref.items():
        assert out[k].shape == v.shape and torch.equal(out[k], v), k
