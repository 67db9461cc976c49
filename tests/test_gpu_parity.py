"""GPU parity tests (`pytest -m gpu` on an H100).  Everything goes through the C ABI
(libopenglue_b200.so via ctypes) and is checked against the oracle (oracle/superglue_oracle.py,
itself pinned to the reference's outputs by tests/test_oracle_golden.py) and directly against
the committed golden vectors minted from the reference.

Tolerances (BASELINE.json north_star): log-scores within 1e-4 absolute of the reference fp32
path (for inputs whose scores reach |30..80| the reference's own fp32-vs-fp64 error is of that
order, so the bound is max(1e-4, 2*err(ref32, ref64)) there); matches0 identical on every row
whose decision margin exceeds 2x the tolerance (ties are counted, not asserted);
matching_scores0 within 1e-4."""
import ctypes as C

import pytest
import torch

from conftest import GOLDEN_BIG, GOLDEN_FULL, GOLDEN_SAMPLED
from openglue_b200 import _cabi
from openglue_b200._cabi import ptr as _ptr, stream as _stream
from openglue_b200.superglue import MatchingCore, SuperGlue
from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
from oracle import superglue_oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-4
DEV = 'cuda:0'


def _to_dev(data):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in data.items()}


def _model(cfg, sd, precision='fp32'):
    cfg = dict(cfg)
    cfg['precision'] = precision
    model = SuperGlue(cfg).eval()
    model.load_state_dict(sd, strict=True)
    return model.to(DEV)


def decisive_rows(scores_ref, margin):
    """rows/cols of the inner block whose top-2 gap exceeds `margin` (argmax is then well defined)."""
    inner = scores_ref[:, :-1, :-1].double()
    b, n, m = inner.shape
    row_ok = torch.ones(b, n, dtype=torch.bool)
    col_ok = torch.ones(b, m, dtype=torch.bool)
    if m >= 2:
        t2r = inner.topk(2, dim=2).values
        row_ok = (t2r[..., 0] - t2r[..., 1]) > margin
    if n >= 2:
        t2c = inner.topk(2, dim=1).values
        col_ok = (t2c[:, 0] - t2c[:, 1]) > margin
    return row_ok, col_ok


def check_matches(ours, ref, scores_ref, tol):
    row_ok, col_ok = decisive_rows(scores_ref, 2 * tol)
    m0, r0 = ours['matches0'].cpu(), ref['matches0']
    # a row's match decision involves its own argmax and the column argmax of the chosen column
    i0 = scores_ref[:, :-1, :-1].argmax(2)
    decisive = row_ok & col_ok.gather(1, i0)
    ms_ref = ref['matching_scores0']
    decisive &= (ms_ref - 0.2).abs() > 2 * tol                # threshold not within tolerance either
    assert torch.equal(m0[decisive], r0[decisive])
    if decisive.any():                                        # (a 1-keypoint image can leave no decisive row at all)
        assert (ours['matching_scores0'].cpu()[decisive] - ms_ref[decisive]).abs().max() <= tol
    return int((~decisive).sum())


# --------------------------------------------------------------------------- whole path vs golden
@pytest.mark.parametrize('name', GOLDEN_FULL)
def test_forward_matches_reference_golden(golden, name):
    fx = golden(name)
    model = _model(fx['config'], fx['state_dict'])
    core = MatchingCore(model, fx['match_threshold'])
    data = _to_dev(fx['data'])
    out = model(data)
    bound = max(TOL, 2 * fx['ref32_vs_ref64_max_abs'])
    assert out['scores'].shape == fx['scores_f32'].shape
    assert (out['scores'].cpu().double() - fx['scores_f64']).abs().max() <= bound
    assert (out['scores'].cpu() - fx['scores_f32']).abs().max() <= bound
    assert (out['context_descriptors0'].cpu() - fx['context_descriptors0_f32']).abs().max() <= 1e-4
    assert (out['context_descriptors1'].cpu() - fx['context_descriptors1_f32']).abs().max() <= 1e-4
    res = core(data)
    ref = {'matches0': fx['matches0'], 'matching_scores0': fx['matching_scores0']}
    check_matches(res, ref, fx['scores_f64'], bound)
    if 'planted' in name:
        assert torch.equal(res['matches0'].cpu(), fx['matches0'])          # decisive inputs: bit-exact


@pytest.mark.parametrize('name', GOLDEN_SAMPLED)
def test_forward_matches_reference_c1(golden, name):
    """BASELINE.json configs[0]: 1 pair, N=M=512, d=256, 9 stages, 20 Sinkhorn iterations."""
    fx = golden(name)
    model = _model(fx['config'], fx['state_dict'])
    data = _to_dev(fx['data'])
    res = MatchingCore(model, fx['match_threshold'])(data, want_scores=True)
    s = res['scores'].cpu()
    bound = max(TOL, 2 * fx['ref32_vs_ref64_max_abs'])
    assert (s[:, ::7, ::5].double() - fx['scores_f64_sample']).abs().max() <= bound
    assert (s[:, ::7, ::5] - fx['scores_f32_sample']).abs().max() <= bound
    assert (s[:, -1, :] - fx['scores_f32_lastrow']).abs().max() <= bound
    assert (s[:, :, -1] - fx['scores_f32_lastcol']).abs().max() <= bound
    # row arg-max identical wherever the reference's own margin is decisive
    gap_ok = fx['row_top2_gap_f64'] > 2 * bound
    assert torch.equal(s[:, :-1, :-1].argmax(2)[gap_ok], fx['row_argmax_f64'][gap_ok])
    if name == 'C1_planted':
        assert torch.equal(res['matches0'].cpu(), fx['matches0'])
        assert (res['matching_scores0'].cpu() - fx['matching_scores0']).abs().max() <= TOL


# --------------------------------------------------------------------------- the configs the numbers are quoted on
@pytest.mark.parametrize('precision,pair', [('fp16x3', 1), ('fp16x3', 0), ('tf32x3', 1), ('tf32x3', 0), ('fp32', 1)])
@pytest.mark.parametrize('name', GOLDEN_BIG)
def test_forward_matches_reference_big(golden, name, precision, pair):
    """BASELINE.json configs[1] (C2), [2] (C3, headline: the 16 pairs bench.py times on rank 0) and [4] (C5, 18 stages,
    S = 6) at FULL depth against fixtures minted from the unmodified reference: log-scores of the scored pairs against the
    reference's fp32 and fp64 runs, matches0 / matching_scores0 of EVERY pair of the batch against the reference's
    MatchingTrainingModule.forward.  `pair` is accepted and has no effect on sm_90 (one kernel form)."""
    fx = golden(name)
    if precision == 'fp32' and name == 'C2_planted':
        pytest.skip('fp32 CUDA-core mode: covered by C3 / C5 (saves box time)')
    lib = _cabi.lib()
    lib.og_set_tuning(pair, pair)
    try:
        model = _model(fx['config'], fx['state_dict'], precision)
        res = MatchingCore(model, fx['match_threshold'])(_to_dev(fx['data']), want_scores=True)
        torch.cuda.synchronize()
    finally:
        lib.og_set_tuning(1, 1)
    k, (sr, sc) = fx['scored_pairs'], fx['sample_stride']
    s = res['scores'][:k].cpu()
    bound = max(TOL, 2 * fx['ref32_vs_ref64_max_abs'])
    e64 = float((s[:, ::sr, ::sc].double() - fx['scores_f64_sample']).abs().max())
    e32 = float((s[:, ::sr, ::sc] - fx['scores_f32_sample']).abs().max())
    edb = max(float((s[:, -1, :] - fx['scores_f32_lastrow']).abs().max()), float((s[:, :, -1] - fx['scores_f32_lastcol']).abs().max()))
    rel = float((s.double().sum(2) - fx['scores_f64_rowsum']).abs().max() / fx['scores_f64_rowsum'].abs().max())
    # matches: decisive rows of the scored pairs (row / column top-2 gap and distance to the threshold beyond 2 x bound)
    m0, ms0 = res['matches0'].cpu(), res['matching_scores0'].cpu()
    i0 = fx['row_argmax_f64']
    decisive = (fx['row_top2_gap_f64'] > 2 * bound) & (fx['col_top2_gap_f64'].gather(1, i0) > 2 * bound) & \
               ((fx['matching_scores0'][:k] - 0.2).abs() > 2 * bound)
    excluded = int((~decisive).sum())
    mism_all = int((m0 != fx['matches0']).sum())
    ems = float((ms0 - fx['matching_scores0']).abs().max())
    print(f'\n[{name} {precision} pair={pair}] max|dscore| vs ref64 {e64:.2e}, vs ref32 {e32:.2e} (bound {bound:.2e}, ref32-vs-ref64 '
          f'{fx["ref32_vs_ref64_max_abs"]:.2e}); dustbin row/col {edb:.2e}; row-sum rel {rel:.1e}; matches0 mismatches over all '
          f'{fx["batch"]} pairs: {mism_all}; rows excluded as near-ties (scored pairs): {excluded}; max|dmatching_scores0| {ems:.2e}')
    assert e64 <= bound and e32 <= bound and edb <= bound and rel < 2e-5
    assert torch.equal(s[:, :-1, :-1].argmax(2)[fx['row_top2_gap_f64'] > 2 * bound], i0[fx['row_top2_gap_f64'] > 2 * bound])
    assert torch.equal(m0[:k][decisive], fx['matches0'][:k][decisive])
    mutual = decisive & (fx['matching_scores0'][:k] > 0)                                  # non-mutual rows carry 0
    assert (ms0[:k][mutual] - fx['matching_scores0_f64'][mutual]).abs().max() <= TOL     # exp(max_j) of the fp64 reference
    assert (ms0[:k][decisive & ~mutual] == 0).all()
    if 'planted' in name:                                        # decisive inputs: identical on EVERY pair of the batch
        assert mism_all == 0
        assert ems <= bound
    else:
        assert int((m0 >= 0).sum()) == 0                         # flat inputs: nothing clears the threshold


# --------------------------------------------------------------------------- whole path vs oracle
@pytest.mark.parametrize('batch,n,m,kw,family', [
    (2, 130, 97, dict(descriptor_dim=64, num_stages=2, num_iters=30), 'planted'),      # ragged n != m, m % 4 != 0
    (1, 1, 5, dict(descriptor_dim=32, num_stages=1, num_iters=5), 'flat'),             # single keypoint
    (3, 7, 3, dict(descriptor_dim=32, num_stages=1, num_iters=0), 'flat'),             # zero Sinkhorn iterations
    (1, 300, 513, dict(descriptor_dim=128, num_stages=2, num_iters=40, side_info_size=6), 'planted'),
    (2, 256, 1100, dict(descriptor_dim=64, num_stages=1, num_iters=15, reg=0.5, use_offset=True,
                        residual=False), 'flat'),                                     # V=16 path, reg != 1
    (1, 4096, 1024, dict(descriptor_dim=128, num_stages=1, num_iters=50, side_info_size=6), 'planted'),   # configs[4] shape
    (2, 330, 197, dict(descriptor_dim=256, num_stages=2, num_iters=30), 'planted'),    # head_dim 64 (the fp16x3 GNN path), ragged n != m
    (1, 200, 200, dict(descriptor_dim=256, num_stages=3, num_iters=20, use_offset=True), 'flat'),        # head_dim 64, n == m (joint self layers)
    (1, 1, 5, dict(descriptor_dim=256, num_stages=1, num_iters=5), 'flat'),            # head_dim 64: a single keypoint / single key block tail
    (3, 64, 1, dict(descriptor_dim=256, num_stages=2, num_iters=0), 'flat'),           # head_dim 64: one key, zero Sinkhorn iterations
    (2, 129, 257, dict(descriptor_dim=128, num_heads=2, num_stages=2, num_iters=10, residual=False), 'planted'),   # head_dim 64 with d = 128
    (2, 150, 97, dict(descriptor_dim=192, num_heads=3, num_stages=2, num_iters=20), 'planted'),     # fp16 GNN with d % 128 != 0: unfused runs
    (2, 70, 83, dict(descriptor_dim=64, num_heads=1, num_stages=2, num_iters=20), 'planted'),       # fp16 GNN narrower than one 128-wide tile
    (2, 90, 61, dict(descriptor_dim=96, num_heads=3, num_stages=2, num_iters=20), 'planted'),       # tf32 attention, head_dim 32, d not 2^k
    (2, 45, 50, dict(descriptor_dim=32, num_heads=4, num_stages=2, num_iters=20), 'planted'),       # head_dim 8: CUDA-core attention everywhere
    (2, 60, 71, dict(descriptor_dim=64, num_stages=2, num_iters=20, hidden_layers_sizes=()), 'planted'),        # encoder without hidden layer
    (2, 60, 71, dict(descriptor_dim=64, num_stages=2, num_iters=20, hidden_layers_sizes=(30, 50)), 'planted'),  # widths not multiples of 4
    (2, 60, 71, dict(descriptor_dim=64, num_stages=2, num_iters=20, side_info_size=0), 'planted'),   # no side info
    (2, 60, 71, dict(descriptor_dim=64, num_stages=2, num_iters=20), 'planted+images'),              # sizes from image tensors
])
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3', 'fp16x3'])
def test_forward_matches_oracle(batch, n, m, kw, family, precision):
    cfg = default_config(**kw)
    sd = synthetic_state_dict(cfg, seed=3)
    family, _, images = family.partition('+')
    data = synthetic_pairs(batch, n, m, cfg['descriptor_dim'], cfg['positional_encoding']['side_info_size'],
                           family=family, seed=77)
    if images:                        # image tensors [B, 1, H, W] take precedence over image*_size (set wrong here on purpose)
        data['image0'], data['image1'] = torch.zeros(batch, 1, 500, 700), torch.zeros(batch, 1, 640, 480)
        data['image0_size'] = data['image1_size'] = (2000, 1000)
    ref = O.run(sd, cfg, data, 0.2)
    ref64 = O.run(sd, cfg, data, 0.2, dtype=torch.float64)
    bound = max(TOL, 2 * float((ref['scores'].double() - ref64['scores']).abs().max()))
    model = _model(cfg, sd, precision)
    res = MatchingCore(model, 0.2)(_to_dev(data), want_scores=True)
    assert (res['scores'].cpu().double() - ref64['scores']).abs().max() <= bound
    check_matches(res, ref, ref64['scores'], bound)
    # context descriptors (superglue.py:66-69)
    out = model(_to_dev(data))
    for i in (0, 1):
        c = out[f'context_descriptors{i}'].cpu().double()
        assert torch.isfinite(c).all()
        assert (c - ref64[f'context_descriptors{i}']).abs().max() <= 1e-4 * max(1.0, float(ref64[f'context_descriptors{i}'].abs().max()))
    # matches1 (inference.py:176-190): same decisive rule, seen from image 1
    row_ok, col_ok = decisive_rows(ref64['scores'], 2 * bound)
    i1 = ref64['scores'][:, :-1, :-1].argmax(1)
    dec1 = col_ok & row_ok.gather(1, i1) & ((ref['matching_scores1'] - 0.2).abs() > 2 * bound)
    dec1 &= (ref['matching_scores0'].gather(1, i1) - 0.2).abs() > 2 * bound
    assert torch.equal(res['matches1'].cpu()[dec1], ref['matches1'][dec1])
    if dec1.any():
        assert (res['matching_scores1'].cpu()[dec1] - ref['matching_scores1'][dec1]).abs().max() <= bound


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3', 'fp16x3'])
def test_no_descriptors_option(precision):
    """config['no_descriptors'] (reference superglue.py:45-49): the GNN starts from the positional encoding alone; the residual
    mix (:59-62) still blends the raw descriptors in."""
    cfg = default_config(descriptor_dim=256, num_stages=2, num_iters=20)
    cfg['no_descriptors'] = True
    sd = synthetic_state_dict(cfg, seed=4)
    data = synthetic_pairs(2, 150, 131, 256, 1, family='planted', seed=9)
    ref64 = O.run(sd, cfg, data, 0.2, dtype=torch.float64)
    ref = O.run(sd, cfg, data, 0.2)
    with_desc = O.run(sd, {**cfg, 'no_descriptors': False}, data, 0.2)
    assert (with_desc['scores'] - ref['scores']).abs().max() > 1e-2          # the option changes the answer
    bound = max(TOL, 2 * float((ref['scores'].double() - ref64['scores']).abs().max()))
    res = MatchingCore(_model(cfg, sd, precision), 0.2)(_to_dev(data), want_scores=True)
    assert (res['scores'].cpu().double() - ref64['scores']).abs().max() <= bound
    check_matches(res, ref, ref64['scores'], bound)


@pytest.mark.parametrize('mode', ['eval', 'train'])
def test_unsupported_head_dim_is_rejected_before_any_kernel(mode):
    """d = 256 with 2 heads (head_dim 128, which the reference accepts) loads, then fails with a ValueError naming head_dim
    before any kernel runs: in train mode no BatchNorm running buffer has moved."""
    cfg = default_config(descriptor_dim=256, num_heads=2, num_stages=1, num_iters=5)
    model = SuperGlue(dict(cfg, precision='tf32x3'))
    model.load_state_dict(synthetic_state_dict(cfg, seed=1), strict=True)
    model = model.to(DEV).train(mode == 'train')
    before = {k: v.clone() for k, v in model.named_buffers()}
    data = _to_dev(synthetic_pairs(2, 40, 30, 256, 1, family='flat', seed=2))
    err = None
    try:
        model(data)
    except Exception as e:                   # (checked below, after the buffers)
        err = e
    torch.cuda.synchronize()
    moved = [k for k, v in model.named_buffers() if not torch.equal(v, before[k])]
    assert not moved, f'buffers moved before the error: {moved}'
    assert isinstance(err, ValueError) and 'head_dim' in str(err), repr(err)


def test_host_buffers_roundtrip(golden):
    """MatchingCore with HOST tensors (the e2e path of bench.py): same answer as device tensors."""
    fx = golden('tiny_planted')
    core = MatchingCore(_model(fx['config'], fx['state_dict']), fx['match_threshold'], device=DEV)
    host = {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in fx['data'].items()}
    res = core(host)
    assert res['matches0'].device.type == 'cpu'
    assert torch.equal(res['matches0'], fx['matches0'])


def test_cuda_graph_replay_matches_eager(golden):
    """MatchingCore(use_cuda_graph=True): same answers as eager launches, across replays and new inputs."""
    fx = golden('small_planted')
    model = _model(fx['config'], fx['state_dict'], 'tf32x3')
    eager = MatchingCore(model, fx['match_threshold'])
    graphed = MatchingCore(model, fx['match_threshold'], use_cuda_graph=True)
    data = _to_dev(fx['data'])
    ref = eager(data, want_scores=True)
    for _ in range(3):
        got = graphed(data, want_scores=True)
        assert torch.equal(got['matches0'], ref['matches0']) and torch.equal(got['scores'], ref['scores'])
    data2 = dict(data)
    data2['keypoints0'] = data['keypoints0'].flip(1).contiguous()            # same shapes, different values
    data2['local_descriptors0'] = data['local_descriptors0'].flip(1).contiguous()
    data2['side_info0'] = data['side_info0'].flip(1).contiguous()
    ref2 = eager(data2, want_scores=True)
    got2 = graphed(data2, want_scores=True)
    assert torch.equal(got2['matches0'], ref2['matches0']) and torch.equal(got2['scores'], ref2['scores'])
    host = {k: (v.cpu().pin_memory() if torch.is_tensor(v) else v) for k, v in data2.items()}
    got3 = graphed(host)
    assert got3['matches0'].device.type == 'cpu' and torch.equal(got3['matches0'], ref2['matches0'].cpu())


@pytest.mark.parametrize('graph', [False, True])
def test_submit_pipeline_matches_blocking_forward(golden, graph):
    """MatchingCore.submit()/wait() with two batches in flight: every batch gets the answer the blocking call gives."""
    fx = golden('small_planted')
    model = _model(fx['config'], fx['state_dict'], 'tf32x3')
    blocking = MatchingCore(model, fx['match_threshold'], device=DEV)
    piped = MatchingCore(model, fx['match_threshold'], device=DEV, use_cuda_graph=graph)
    batches = []
    for i in range(5):
        h = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in fx['data'].items()}
        if i % 2:
            for k in ('keypoints0', 'local_descriptors0', 'side_info0'):
                h[k] = h[k].flip(1).contiguous()
        if i >= 3:
            h['local_descriptors1'] = torch.nn.functional.normalize(h['local_descriptors1'] + 0.05 * i, dim=-1)
        batches.append({k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in h.items()})
    want = [{k: v.clone() for k, v in blocking(h).items()} for h in batches]
    got, pend = [], None
    for h in batches:
        nxt = piped.submit(h)
        if pend is not None:
            got.append({k: v.clone() for k, v in pend.wait().items()})
        pend = nxt
    got.append({k: v.clone() for k, v in pend.wait().items()})
    for w, g in zip(want, got):
        for k in ('matches0', 'matches1', 'matching_scores0', 'matching_scores1'):
            assert g[k].device.type == 'cpu' and torch.equal(w[k], g[k]), k
    with pytest.raises(ValueError):
        piped.submit(_to_dev(fx['data']))


# --------------------------------------------------------------------------- operators
@pytest.mark.parametrize('rows,k1,k2,nout,relu,resid,batch', [
    (200, 3, 0, 32, True, False, 1), (513, 256, 256, 512, True, False, 1), (130, 512, 0, 256, False, True, 1),
    (64, 64, 0, 100, False, False, 3), (1, 7, 5, 9, False, True, 2)])
def test_linear_operator(rows, k1, k2, nout, relu, resid, batch):
    g = torch.Generator().manual_seed(1)
    A = torch.randn(batch, rows, k1, generator=g)
    A2 = torch.randn(batch, rows, k2, generator=g) if k2 else None
    W = torch.randn(batch, nout, k1 + k2, generator=g)
    bias = torch.randn(nout, generator=g)
    R = torch.randn(batch, rows, nout, generator=g) if resid else None
    rs = torch.rand(nout, generator=g) if resid else None
    X = torch.cat([A, A2], -1) if k2 else A
    ref = 0.7 * (X.double() @ W.double().transpose(1, 2)) + bias.double()
    if relu:
        ref = ref.relu()
    if resid:
        ref = ref + rs.double() * R.double()
    dA, dA2, dW, db = A.to(DEV), (A2.to(DEV) if k2 else None), W.to(DEV), bias.to(DEV)
    dR, drs = (R.to(DEV), rs.to(DEV)) if resid else (None, None)
    Y = torch.empty(batch, rows, nout, device=DEV)
    Yt = torch.empty(batch, nout, rows, device=DEV)
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.strideA = dA.data_ptr(), k1, rows * k1
    if k2:
        a.A2, a.lda2, a.strideA2 = dA2.data_ptr(), k2, rows * k2
    a.k1, a.k2 = k1, k2
    a.W, a.ldw, a.strideW = dW.data_ptr(), k1 + k2, nout * (k1 + k2)
    a.bias = db.data_ptr()
    a.rows, a.nout, a.batch, a.alpha, a.relu = rows, nout, batch, 0.7, int(relu)
    if resid:
        a.R, a.ldr, a.strideR, a.rscale = dR.data_ptr(), nout, rows * nout, drs.data_ptr()
    a.Y, a.ldy, a.strideY = Y.data_ptr(), nout, rows * nout
    a.Yt, a.ldyt, a.strideYt = Yt.data_ptr(), rows, nout * rows
    _cabi.check(_cabi.lib().og_linear_fwd(C.byref(a), _cabi.OG_PREC_FP32, _stream()), 'og_linear_fwd')
    scale = ref.abs().max()
    assert (Y.cpu().double() - ref).abs().max() <= 2e-6 * scale
    assert torch.equal(Yt.cpu(), Y.cpu().transpose(1, 2))


@pytest.mark.parametrize('B,H,dh,nq,nk', [(2, 4, 64, 200, 333), (1, 4, 32, 65, 64), (3, 2, 16, 10, 129), (1, 4, 8, 64, 1)])
def test_attention_operator(B, H, dh, nq, nk):
    g = torch.Generator().manual_seed(2)
    d = H * dh
    q, k, v = (3 * torch.randn(B, n_, d, generator=g) for n_ in (nq, nk, nk))
    # oracle layout: [B, H, Dh, n]
    to_ref = lambda t: t.transpose(1, 2).reshape(B, H, dh, -1)
    ref = O.softmax_attention(to_ref(q).double(), to_ref(k).double(), to_ref(v).double()).reshape(B, d, nq).transpose(1, 2)
    dq, dk, dv = q.to(DEV), k.to(DEV), v.to(DEV)
    out = torch.empty(B, nq, d, device=DEV)
    rc = _cabi.lib().og_attention_fwd(_ptr(dq), d, nq * d, _ptr(dk), d, nk * d, _ptr(dv), d, nk * d, _ptr(out), d, nq * d,
                                      B, nq, nk, H, dh, _cabi.OG_PREC_FP32, _stream())
    _cabi.check(rc, 'og_attention_fwd')
    assert (out.cpu().double() - ref).abs().max() <= 5e-6 * ref.abs().max()


@pytest.mark.parametrize('B,n,m,iters,reg,scale', [(2, 30, 41, 50, 1.0, 3.0), (1, 513, 512, 20, 1.0, 10.0),
                                                   (3, 100, 1025, 10, 0.7, 2.0), (1, 2048, 2048, 100, 1.0, 8.0),
                                                   (20, 64, 64, 30, 1.0, 5.0), (1, 4, 2048, 3, 1.0, 1.0),
                                                   (1, 300, 3000, 15, 1.0, 3.0), (2, 1500, 4100, 10, 0.8, 4.0), (1, 64, 8192, 5, 1.0, 2.0),
                                                   (3, 700, 513, 25, 1.0, 6.0), (1, 2048, 1030, 40, 1.0, 8.0)])
def test_sinkhorn_operator(B, n, m, iters, reg, scale):
    g = torch.Generator().manual_seed(5)
    S = scale * torch.randn(B, n, m, generator=g)
    dust = torch.tensor(1.3)
    ref = O.matching_log_probs(S.double(), dust.double(), iters, reg)
    lds = (m + 3) // 4 * 4
    dS = torch.zeros(B, n, lds, device=DEV)
    dS[:, :, :m] = S.to(DEV)
    scores = torch.empty(B, n + 1, m + 1, device=DEV)
    lib = _cabi.lib()
    wsb = lib.og_sinkhorn_workspace_bytes(B, n, m)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    rc = lib.og_sinkhorn_fwd(_ptr(dS), lds, n * lds, _ptr(dust.to(DEV)), B, n, m, iters, reg, _ptr(scores), _ptr(ws), wsb,
                             _stream())
    _cabi.check(rc, 'og_sinkhorn_fwd')
    assert (scores.cpu().double() - ref).abs().max() <= 2e-5
    # property (size independent): after the last v-update the column marginals are exactly b
    if iters > 0:
        p = (scores.cpu().double() - torch.log(torch.tensor(float(n + m)))).exp().sum(1)
        assert (p[:, :-1] * (n + m) - 1).abs().max() < 1e-4
        assert (p[:, -1] * (n + m) / n - 1).abs().max() < 1e-4


@pytest.mark.parametrize('B,n,m', [(2, 50, 70), (1, 513, 300), (3, 64, 64)])
def test_match_operator_ties_and_threshold(B, n, m):
    g = torch.Generator().manual_seed(9)
    scores = -3 * torch.rand(B, n + 1, m + 1, generator=g)
    scores = (scores * 4).round() / 4                       # many exact ties -> first-index rule matters
    ref = O.extract_matches(scores, 0.2)
    ds = scores.to(DEV)
    lib = _cabi.lib()
    wsb = lib.og_match_workspace_bytes(B, n, m)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    m0 = torch.empty(B, n, dtype=torch.int64, device=DEV); s0 = torch.empty(B, n, device=DEV)
    m1 = torch.empty(B, m, dtype=torch.int64, device=DEV); s1 = torch.empty(B, m, device=DEV)
    _cabi.check(lib.og_match_fwd(_ptr(ds), B, n, m, 0.2, _ptr(m0), _ptr(s0), _ptr(m1), _ptr(s1), _ptr(ws), wsb, _stream()),
                'og_match_fwd')
    assert torch.equal(m0.cpu(), ref['matches0'])
    assert torch.equal(m1.cpu(), ref['matches1'])
    assert (s0.cpu() - ref['matching_scores0']).abs().max() <= 1e-6
    assert (s1.cpu() - ref['matching_scores1']).abs().max() <= 1e-6


# --------------------------------------------------------------------------- full size properties
def test_headline_shape_properties():
    """N = M = 2048, d = 256, 9 stages, 100 iterations (BASELINE.json headline shape, 2 pairs):
    too big for the oracle in seconds, so check size-independent properties."""
    cfg = default_config(num_iters=100)
    sd = synthetic_state_dict(cfg, seed=0)
    data = synthetic_pairs(2, 2048, 2048, 256, 1, family='planted', seed=1234)
    model = _model(cfg, sd, 'tf32x3')
    core = MatchingCore(model, 0.2)
    res = core(_to_dev(data), want_scores=True)
    s = res['scores'].double()
    assert torch.isfinite(s).all()
    n = m = 2048
    col = (s - torch.log(torch.tensor(float(n + m)))).exp().sum(1)
    assert (col[:, :-1] * (n + m) - 1).abs().max() < 1e-3          # column marginals = b after the last v-update
    row = (s - torch.log(torch.tensor(float(n + m)))).exp().sum(2)
    assert (row[:, :-1] * (n + m) - 1).abs().max() < 0.05          # rows nearly converged after 100 iterations
    m0, m1 = res['matches0'], res['matches1']
    idx = torch.arange(n, device=m0.device)[None].expand_as(m0)
    ok = m0 >= 0
    assert torch.equal(m1.gather(1, m0.clamp(min=0))[ok], idx[ok])  # matches are mutual
    planted = data['planted_matches0'].to(m0.device)
    has = planted >= 0
    assert (m0[has] == planted[has]).float().mean() > 0.99          # planted correspondences recovered
    res2 = core(_to_dev(data), want_scores=True)
    assert torch.equal(res2['scores'], res['scores'])               # deterministic (no atomics on data)
    assert model.last_launches > 100
