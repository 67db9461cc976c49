"""The persistent, warp-specialized Hopper GEMM (csrc/linear_sm90.cuh): min(tiles, SMs) CTAs walk the output tiles in a static
schedule.  Scheduler edges (tile counts around the SM count), ragged rows / columns, batched operands with per-batch weights,
the forward's GEMM forms, and position independence (a tile's result does not depend on which CTA or which round computes it),
for both operand forms, against float64 references with the bounds of test_gpu_f16.py / test_gpu_tc.py."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200._cabi import ptr as _p, stream as _st

DEV = 'cuda:0'
F16_BOUND, TF32_BOUND = 2e-6, 1.5e-6


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _operands(rows, k1, k2, nout, batch, per_batch_b, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    A = 3 * torch.randn(batch, rows, k1, generator=g, device=DEV)
    A2 = torch.randn(batch, rows, k2, generator=g, device=DEV) if k2 else None
    W = torch.randn(batch if per_batch_b else 1, nout, k1 + k2, generator=g, device=DEV) / 8
    bias = torch.randn(nout, generator=g, device=DEV)
    return A, A2, W, bias


def _reference(A, A2, W, bias, alpha, relu, R=None):
    X = torch.cat([A, A2], -1) if A2 is not None else A
    ref = alpha * (X.double() @ W.double().transpose(1, 2)) + bias.double()
    if relu:
        ref = ref.relu()
    return ref + R.double() if R is not None else ref


def _args(A, A2, W, bias, alpha, relu, per_batch_b):
    batch, rows, k1 = A.shape
    k2 = A2.shape[2] if A2 is not None else 0
    nout = W.shape[1]
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.strideA = A.data_ptr(), k1, rows * k1
    if k2:
        a.A2, a.lda2, a.strideA2 = A2.data_ptr(), k2, rows * k2
    a.k1, a.k2, a.ldw, a.strideW = k1, k2, k1 + k2, (nout * (k1 + k2) if per_batch_b else 0)
    a.bias = bias.data_ptr()
    a.rows, a.nout, a.batch, a.alpha, a.relu = rows, nout, batch, alpha, int(relu)
    return a


def _split16(W):
    hi = torch.empty(W.shape, dtype=torch.float16, device=DEV)
    lo = torch.empty_like(hi)
    meta = torch.zeros(4, device=DEV)
    w2 = W.reshape(-1, W.shape[-1])
    _cabi.check(_cabi.lib().og_weight_split_f16(_p(w2), None, w2.shape[0], w2.shape[1], _p(hi), _p(lo), _p(meta), _st()), 'split16')
    return hi, lo, meta


def _amax(*xs):
    slot = torch.zeros(1, device=DEV)
    x = torch.cat([t.flatten() for t in xs if t is not None])
    _cabi.check(_cabi.lib().og_amax(_p(x), x.numel(), _p(slot), _st()), 'og_amax')
    return slot


def run_f16(A, A2, W, bias, alpha=0.7, relu=False, per_batch_b=False, kind='y', R=None, Y=None, pad=0):
    """og_linear_f16_fwd; kind 'y' (fp32 Y, optional residual R; Y may be R: the in-place form of fc2), 'split' (row-major fp16
    hi/lo) or 'tsplit' (transposed fp16 hi/lo); pad widens the row stride of the fp16 outputs beyond a multiple of 8 elements.
    Returns the output decoded to float64 and, for 'y', the tracked amax."""
    batch, rows, _ = A.shape
    nout = W.shape[1]
    a = _args(A, A2, W, bias, alpha, relu, per_batch_b)
    Wh, Wl, meta = _split16(W)
    meta[2] = bias.abs().max()                         # max |bias| (the split above covers the weights only)
    lib = _cabi.lib()
    a_amax = _amax(A, A2)
    amax_out, scale_out = torch.zeros(1, device=DEV), torch.zeros(1, device=DEV)
    if kind == 'y':
        if Y is None:
            Y = torch.full((batch, rows, nout), float('nan'), device=DEV)
        a.Y, a.ldy, a.strideY = Y.data_ptr(), nout, rows * nout
        if R is not None:
            a.R, a.ldr, a.strideR = R.data_ptr(), nout, rows * nout
        _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(a_amax), _p(amax_out), None, None, None, None, None, 0, _st()), 'linear_f16')
        return Y, float(amax_out)
    if kind == 'split':
        ldy = (nout + 7) // 8 * 8 + pad
        Yh = torch.zeros(batch, rows, ldy, dtype=torch.float16, device=DEV)
        Yl = torch.zeros_like(Yh)
        a.ldy, a.strideY = ldy, rows * ldy
        _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(a_amax), None, _p(scale_out), _p(Yh), _p(Yl), None, None, 0, _st()), 'linear_f16')
        return (Yh[:, :, :nout].double() + Yl[:, :, :nout].double()) / float(scale_out), None
    ldyt = (rows + 7) // 8 * 8 + pad
    Yth = torch.zeros(batch, nout, ldyt, dtype=torch.float16, device=DEV)
    Ytl = torch.zeros_like(Yth)
    a.ldyt, a.strideYt = ldyt, nout * ldyt
    _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(a_amax), None, _p(scale_out), None, None, _p(Yth), _p(Ytl), 0, _st()), 'linear_f16')
    return ((Yth[:, :, :rows].double() + Ytl[:, :, :rows].double()) / float(scale_out)).transpose(1, 2), None


def run_tf32(A, A2, W, bias, alpha=0.5, relu=False, per_batch_b=False, R=None):
    """og_linear_tc_fwd with fp32 Y (optional residual R); returns Y."""
    batch, rows, _ = A.shape
    nout = W.shape[1]
    a = _args(A, A2, W, bias, alpha, relu, per_batch_b)
    lib = _cabi.lib()
    Whi, Wlo = torch.empty_like(W), torch.empty_like(W)
    _cabi.check(lib.og_split_tf32(_p(W), _p(Whi), _p(Wlo), W.numel(), _st()), 'og_split_tf32')
    Y = torch.full((batch, rows, nout), float('nan'), device=DEV)
    a.Y, a.ldy, a.strideY = Y.data_ptr(), nout, rows * nout
    if R is not None:
        a.R, a.ldr, a.strideR = R.data_ptr(), nout, rows * nout
    _cabi.check(lib.og_linear_tc_fwd(C.byref(a), _p(Whi), _p(Wlo), None, None, None, None, 2, _st()), 'og_linear_tc_fwd')
    return Y


def _check(form, A, A2, W, bias, relu=False, per_batch_b=False, kind='y', R=None, in_place=False, pad=0):
    alpha = 0.7 if form == 'f16' else 0.5
    ref = _reference(A, A2, W, bias, alpha, relu, R)
    if form == 'f16':
        Y, amax = run_f16(A, A2, W, bias, alpha, relu, per_batch_b, kind, R, Y=R if in_place else None, pad=pad)
    else:
        Y, amax = run_tf32(A, A2, W, bias, alpha, relu, per_batch_b, R), None
    torch.cuda.synchronize()
    err = float((Y.double() - ref).abs().max() / ref.abs().max())
    assert err <= (F16_BOUND if form == 'f16' else TF32_BOUND), err
    if amax is not None:
        assert amax == float(Y.abs().max())              # tracked amax = the true maximum of the output
    return Y


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['f16', 'tf32'])
@pytest.mark.parametrize('tiles', ['1', 'sms-1', 'sms', 'sms+1', '3sms+5'])
def test_scheduler_edges(form, tiles):
    """Tile counts around the SM count: fewer tiles than SMs, exactly one round, one tile more, several rounds plus a tail.
    Ragged rows: the last row tile holds 77 of 128 rows."""
    sms = _sms()
    n = {'1': 1, 'sms-1': sms - 1, 'sms': sms, 'sms+1': sms + 1, '3sms+5': 3 * sms + 5}[tiles]
    A, A2, W, bias = _operands(128 * n - 51, 192 if form == 'f16' else 96, 0, 128, 1, False, seed=n)   # 3 K blocks
    _check(form, A, A2, W, bias)


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['f16', 'tf32'])
@pytest.mark.parametrize('rows,nout,batch,per_batch_b', [(1000, 392, 1, False), (2049, 200, 3, False), (300, 2048, 4, True),
                                                       (517, 334, 5, True)])
def test_ragged_and_batched(form, rows, nout, batch, per_batch_b):
    """Ragged rows and columns; batch > 1 with a batch stride of A and, per_batch_b, a per-batch weight block (b_rows_per_batch:
    the score GEMM's form).  Tiles of one batch item are spread over several CTAs and rounds."""
    A, A2, W, bias = _operands(rows, 256, 0, nout, batch, per_batch_b, seed=rows + nout)
    _check(form, A, A2, W, bias, per_batch_b=per_batch_b)


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['f16', 'tf32'])
def test_concatenated_operand(form):
    """fc1 of the forward: A | A2 (x | message) with ReLU, K = 512, nout = 512, many rounds of tiles."""
    A, A2, W, bias = _operands(8192 + 37, 256, 256, 512, 1, False, seed=3)
    _check(form, A, A2, W, bias, relu=True)


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['f16', 'tf32'])
def test_in_place_residual(form):
    """fc2 of the forward: Y = x + W h with R == Y (f16: the residual read and the write of one element by the same thread)."""
    A, A2, W, bias = _operands(8192 + 100, 512, 0, 256, 1, False, seed=4)
    g = torch.Generator(device=DEV).manual_seed(5)
    R = torch.randn(1, A.shape[1], 256, generator=g, device=DEV)
    _check(form, A, A2, W, bias, R=R.clone() if form == 'tf32' else R, in_place=form == 'f16')


@pytest.mark.gpu
@pytest.mark.parametrize('pad', [0, 2])
@pytest.mark.parametrize('kind', ['split', 'tsplit'])
@pytest.mark.parametrize('rows,nout,batch', [(4096 + 77, 256, 1), (2048 + 3, 256, 2), (1000, 200, 5), (77, 100, 3)])
def test_f16_operand_outputs_ragged(kind, rows, nout, batch, pad):
    """K (row-major fp16 hi/lo) and V^T (transposed fp16 hi/lo) outputs over many tiles with ragged rows and columns.  K with pad 0:
    16-byte-aligned rows, stored as 16-byte runs after a quad exchange (partial runs at the ragged column edge); pad 2: rows that
    are not, stored element pair by element pair."""
    A, A2, W, bias = _operands(rows, 256, 0, nout, batch, False, seed=rows)
    _check('f16', A, A2, W, bias, kind=kind, pad=pad)


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['f16', 'tf32'])
def test_position_independence(form):
    """One launch over many tiles equals, bit for bit, the same rows computed by separate launches of fewer tiles: each tile
    lands on another CTA and in another round of the schedule, and its result must not change."""
    sms = _sms()
    rows = 128 * (3 * sms + 5)
    A, A2, W, bias = _operands(rows, 256, 256, 256, 1, False, seed=9)
    cuts = (0, 128, 128 * 7, 128 * (sms + 2), rows)
    # the fp16 form scales A by a power of two that follows the binade of max |A|: give every slice the same one
    A.clamp_(-16, 16)
    A[:, list(cuts[:-1]), 0] = 20.0
    run = run_f16 if form == 'f16' else run_tf32
    pick = (lambda r: r[0]) if form == 'f16' else (lambda r: r)
    whole = pick(run(A, A2, W, bias))
    for r0, r1 in zip(cuts[:-1], cuts[1:]):
        sub = pick(run(A[:, r0:r1].contiguous(), A2[:, r0:r1].contiguous(), W, bias))
        assert torch.equal(sub, whole[:, r0:r1]), (r0, r1)


@pytest.mark.gpu
@pytest.mark.parametrize('batch,n,m', [(4, 1500, 900), (2, 2048, 2048)])
def test_stacked_projections_many_tiles(batch, n, m):
    """Q | K | V (nkinds 3, self layers) and K | V (nkinds 2, cross layers) as one launch each over many tiles with ragged rows:
    the whole path's outputs equal those of one launch per projection, bit for bit."""
    from openglue_b200 import SuperGlue
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
    cfg = default_config(descriptor_dim=256, num_stages=2, num_iters=10)
    cfg['precision'] = 'fp16x3'
    model = SuperGlue(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=8), strict=True)
    model = model.to(DEV).eval()
    data = synthetic_pairs(batch, n, m, 256, 1, family='planted', seed=31)
    data = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in data.items()}
    lib = _cabi.lib()
    prev = lib.og_set_fusion(1)
    try:
        with torch.no_grad():
            fused = {k: v.clone() for k, v in model(data).items()}
            lib.og_set_fusion(0)
            plain = {k: v.clone() for k, v in model(data).items()}
    finally:
        lib.og_set_fusion(prev)
    for k in fused:
        assert torch.equal(fused[k], plain[k]), k


@pytest.mark.gpu
def test_stacked_projections_against_float64():
    """The stacked Q | K | V (nkinds 3) and K | V (nkinds 2) launches over several rounds of ragged tiles (1500 and 900 keypoints
    per image), checked through the whole path against the float64 oracle with the bounds of test_gpu_parity.py."""
    from oracle import superglue_oracle as O
    from openglue_b200 import MatchingCore, SuperGlue
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
    batch, n, m = 2, 1500, 900
    cfg = default_config(descriptor_dim=256, num_stages=1, num_iters=20)
    sd = synthetic_state_dict(cfg, seed=3)
    data = synthetic_pairs(batch, n, m, 256, 1, family='planted', seed=77)
    ref = O.run(sd, cfg, data, 0.2)
    ref64 = O.run(sd, cfg, data, 0.2, dtype=torch.float64)
    bound = max(1e-4, 2 * float((ref['scores'].double() - ref64['scores']).abs().max()))
    cfg = dict(cfg, precision='fp16x3')
    model = SuperGlue(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.to(DEV).eval()
    dev_data = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in data.items()}
    lib = _cabi.lib()
    prev = lib.og_set_fusion(1)
    try:
        res = MatchingCore(model, 0.2)(dev_data, want_scores=True)
        with torch.no_grad():
            out = model(dev_data)
    finally:
        lib.og_set_fusion(prev)
    assert (res['scores'].cpu().double() - ref64['scores']).abs().max() <= bound
    for i in (0, 1):
        c, r = out[f'context_descriptors{i}'].cpu().double(), ref64[f'context_descriptors{i}']
        assert (c - r).abs().max() <= 1e-4 * max(1.0, float(r.abs().max()))


def test_gemm_kernels_are_warp_specialized_without_spills():
    """Static check of the built library (cuobjdump, no GPU; OG_LIB names another build): both GEMM instantiations move registers
    between warpgroups (USETMAXREG) and touch no local memory (STL / LDL: spills)."""
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    path = os.environ.get('OG_LIB') or _cabi.LIB_PATH
    assert os.path.exists(path), f'library not built: {path}'
    res = subprocess.run([tool, '-sass', path], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    funcs, cur = {}, None
    for line in res.stdout.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = funcs.setdefault(m.group(1), []) if 'linear_sm90_kernel' in m.group(1) else None
            continue
        m = re.match(r'\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P(?:\d+|T)\s+)?([A-Z0-9_.]+)', line)
        if m and cur is not None:
            cur.append(m.group(1).split('.')[0])
    assert len(funcs) == 2, sorted(funcs)                # F16LinearArgs and TcLinearArgs
    for name, ops in funcs.items():
        assert 'USETMAXREG' in ops and 'HGMMA' in ops, name
        assert 'STL' not in ops and 'LDL' not in ops, name
