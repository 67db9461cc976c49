"""The training kernels at training sizes, each against a float64 reference that shares none of its code.

a. The Sinkhorn training forward (og_sinkhorn_train_fwd) and backward (og_sinkhorn_bwd) through the C ABI, at both edges of every
   column band of the instantiation table (csrc/sinkhorn.cuh: sinkhorn_plan), against the reverse-recurrence
   oracle (oracle/sinkhorn_grad_oracle.py, pinned to the reference's autograd by tests/test_sinkhorn_grad.py).
b. The operators of csrc/train_ops.cuh (transpose / copy, column sums, BatchNorm forward and backward, row softmax and its backward,
   the split-K reduction, axpby, the residual mix, the keypoint-encoder input) against float64 torch, autograd where the operator is
   a gradient, with strided inputs and NaN-poisoned outputs.
c. The whole TrainStep at a production-size batch against the same TrainStep driven by the float64 torch double of its kernels.

Bounds come from an error model (a recursive fp32 sum of k terms is within k 2^-24 sum|terms| of the exact sum) or from the distance
between the float64 reference and the same reference run in float32; every case prints the error it measured next to its bound.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from openglue_b200._cabi import ptr as _p, stream as _st
from oracle import loss_oracle as L
from oracle import sinkhorn_grad_oracle as SG

U = 2.0 ** -24                                  # unit roundoff of float32
DEV = 'cuda:0'


def _lib():
    from openglue_b200 import _cabi
    return _cabi.lib()


def _check(rc, what):
    from openglue_b200 import _cabi
    _cabi.check(rc, what)


def _sm_count():
    sms = C.c_int(0)
    _check(_lib().og_device_info(C.byref(sms), None, None), 'og_device_info')
    return sms.value


def _nan(*shape):
    return torch.full(shape, float('nan'), dtype=torch.float32, device=DEV)


def _strided(x, ld, fill=float('nan')):
    """x [rows, cols] (CPU) -> device [rows, ld] buffer holding x in its first cols columns, `fill` elsewhere, and the [rows, cols] view"""
    rows, cols = x.shape
    buf = torch.full((rows, ld), fill, dtype=torch.float32, device=DEV)
    buf[:, :cols] = x.to(DEV)
    return buf, buf[:, :cols]


def _report(tag, err, bound):
    print(f'\n[{tag}] max error {err:.3e}, bound {bound:.3e} ({err / bound if bound > 0 else 0.0:.2f} of it)')


# ---------------------------------------------------------------------------------------------------------------------
# a. Sinkhorn training forward + backward across every instantiation
#    (B, n, m, iters, reg, upstream): upstream 'dense' = a random dense d loss / d scores, 'labels' = the criterion's gradient
SINK_CASES = [
    (1, 300, 512, 10, 1.0, 'labels'),        # V4 W1, top of the band
    (2, 257, 513, 10, 0.7, 'dense'),         # V4 W2, bottom (m % 4 = 1)
    (1, 200, 1024, 8, 1.0, 'labels'),        # V4 W2, top
    (1, 330, 1025, 6, 0.5, 'dense'),         # V8 W2, bottom (m % 4 = 1)
    (1, 150, 2048, 5, 1.0, 'labels'),        # V8 W2, top
    (1, 301, 2049, 8, 1.0, 'dense'),         # V16 W2, bottom (m % 4 = 1)
    (1, 260, 2050, 100, 1.0, 'labels'),      # V16 W2, T = 100 (m % 4 = 2)
    (2, 200, 3071, 5, 0.7, 'dense'),         # V16 W2 (m % 4 = 3)
    (1, 1500, 4096, 8, 1.0, 'labels'),       # V16 W2, top
    (1, 150, 4097, 5, 0.5, 'dense'),         # V16 W4, bottom (m % 4 = 1)
    (1, 100, 8192, 3, 1.0, 'labels'),        # V16 W4, top
    (1, 4096, 1024, 5, 1.0, 'dense'),        # N >> M: 32 strips, ragged rows per strip
    (1, 1, 700, 5, 1.0, 'dense'),            # N = 1
    (1, 600, 1, 5, 1.0, 'labels'),           # M = 1
    (1, 100, 2500, 0, 1.0, 'dense'),         # no iteration
    (1, 120, 600, 1, 0.7, 'labels'),         # one iteration
]


def _sink_inputs(B, n, m, upstream, seed):
    g = torch.Generator().manual_seed(seed)
    S = 4.0 * torch.randn(B, n, m, generator=g)
    dust = torch.tensor(0.8)
    if upstream == 'dense':
        G = torch.randn(B, n + 1, m + 1, generator=g, dtype=torch.float64) / (n + m)
    else:
        gt0 = torch.full((B, n), -1, dtype=torch.int64)
        gt1 = torch.full((B, m), -1, dtype=torch.int64)
        k = (2 * min(n, m)) // 3
        for b in range(B):
            src, dst = torch.randperm(n, generator=g)[:k], torch.randperm(m, generator=g)[:k]
            gt0[b, src] = dst
            gt1[b, dst] = src
        G = L.criterion_grad({'gt_matches0': gt0, 'gt_matches1': gt1}, (B, n + 1, m + 1))
    return S, dust, G.float()


def _sink_run(S, dust, G, iters, reg):
    """og_sinkhorn_train_fwd + og_sinkhorn_bwd on padded rows (lds > m, strideS > n lds; the padding is NaN) into NaN-poisoned outputs"""
    lib = _lib()
    B, n, m = S.shape
    lds = (m + 3) // 4 * 4 + 8
    strideS = n * lds + 64
    Sbuf = torch.full((B * strideS,), float('nan'), dtype=torch.float32, device=DEV)
    Sbuf.as_strided((B, n, m), (strideS, lds, 1)).copy_(S.to(DEV))
    d = dust.reshape(1).to(DEV)
    scores = _nan(B, n + 1, m + 1)
    hist = _nan(max(int(lib.og_sinkhorn_hist_floats(B, n, m, iters)), 1))
    wsb = int(lib.og_sinkhorn_workspace_bytes(B, n, m))
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    _check(lib.og_sinkhorn_train_fwd(_p(Sbuf), lds, strideS, _p(d), B, n, m, iters, reg, _p(scores), _p(hist), _p(ws), wsb, _st()),
           'og_sinkhorn_train_fwd')
    Gd = G.to(DEV).contiguous()
    dZ, dd = _nan(B, n + 1, m + 1), _nan(1)
    wsb = int(lib.og_sinkhorn_bwd_workspace_bytes(B, n, m, iters))
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    _check(lib.og_sinkhorn_bwd(_p(Sbuf), lds, strideS, _p(d), B, n, m, iters, reg, _p(hist), _p(Gd), _p(dZ), _p(dd), _p(ws), wsb, _st()),
           'og_sinkhorn_bwd')
    torch.cuda.synchronize()
    return scores.cpu(), hist.cpu(), dZ.cpu(), dd.cpu()


def _sink_oracle(S, dust, G, iters, reg, dtype):
    scores, _, us, vs, _, _ = SG.forward_with_history(S.to(dtype), dust.to(dtype), iters, reg)
    dS, dd = SG.backward(S.to(dtype), dust.to(dtype), iters, reg, G.to(dtype))
    return scores.double(), [u.double() for u in us], [v.double() for v in vs], dS.double(), float(dd)


def _deviation_bound(x64, x32, k=4.0):
    """k x the float32 reference's own distance from float64, and never below k ulps of the largest magnitude"""
    return k * max(float((x32 - x64).abs().max()), 2 * U * float(x64.abs().max()))


def _check_sinkhorn(B, n, m, iters, reg, upstream, seed):
    S, dust, G = _sink_inputs(B, n, m, upstream, seed)
    scores, hist, dZ, dd = _sink_run(S, dust, G, iters, reg)
    tag = f'B={B} {n}x{m} T={iters} reg={reg} {upstream}'
    assert torch.isfinite(scores).all() and torch.isfinite(hist[:int(_lib().og_sinkhorn_hist_floats(B, n, m, iters))]).all()
    assert torch.isfinite(dZ).all() and torch.isfinite(dd).all(), tag
    r64 = _sink_oracle(S, dust, G, iters, reg, torch.float64)
    r32 = _sink_oracle(S, dust, G, iters, reg, torch.float32)
    # scores
    err, bound = float((scores.double() - r64[0]).abs().max()), _deviation_bound(r64[0], r32[0])
    _report(tag + ' scores', err, bound)
    assert err <= bound
    # recorded history: u [B][T][n+1], then v [B][T+1][m+1] (v_0 = 0)
    hu = hist[:B * iters * (n + 1)].view(B, iters, n + 1).double()
    hv = hist[B * iters * (n + 1):B * iters * (n + 1) + B * (iters + 1) * (m + 1)].view(B, iters + 1, m + 1).double()
    assert torch.equal(hv[:, 0], torch.zeros(B, m + 1, dtype=torch.float64))
    for t in range(iters):
        for name, got, w64, w32 in (('u', hu[:, t], r64[1][t], r32[1][t]), ('v', hv[:, t + 1], r64[2][t + 1], r32[2][t + 1])):
            err, bound = float((got - w64).abs().max()), _deviation_bound(w64, w32)
            if t in (0, iters - 1):
                _report(f'{tag} {name}_{t + 1}', err, bound)
            assert err <= bound, (name, t + 1)
    # d loss / d S: 2e-4 of max|dS| (tests/test_sinkhorn_grad.py), or the float32 reference's own distance if that is larger
    dS = dZ[:, :n, :m].double()
    scale = float(r64[3].abs().max())
    err, bound = float((dS - r64[3]).abs().max()), max(2e-4 * scale, 4 * float((r64[3] - r32[3]).abs().max()))
    _report(tag + ' dS', err, bound)
    assert err <= bound
    # d loss / d dustbin
    err = abs(float(dd) - r64[4])
    bound = max(2e-4 * max(abs(r64[4]), 1e-3), 4 * abs(r32[4] - r64[4]))
    _report(tag + ' d dustbin', err, bound)
    assert err <= bound
    # ... which is the sum of the dustbin row and column of dS_aug (a recursive fp32 sum of n + m + 1 terms per pair, then B pairs)
    terms = torch.cat([dZ[:, n, :].reshape(-1), dZ[:, :n, m].reshape(-1)]).double()
    bound = (n + m + 1 + B) * U * float(terms.abs().sum())
    assert abs(float(dd) - float(terms.sum())) <= bound
    # deterministic, bit for bit
    again = _sink_run(S, dust, G, iters, reg)
    for a, b in zip((scores, hist, dZ, dd), again):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize('case', SINK_CASES, ids=lambda c: f'B{c[0]}_{c[1]}x{c[2]}_T{c[3]}_reg{c[4]}_{c[5]}')
def test_sinkhorn_train_fwd_bwd_matches_oracle(case):
    _check_sinkhorn(*case, seed=SINK_CASES.index(case))


@pytest.mark.gpu
def test_sinkhorn_train_launch_loop_over_pairs():
    """More pairs than one cooperative launch holds, in both passes: the forward runs two CTAs per SM, the backward (1545 <= m <= 2048)
    one, so the two passes split the batch differently and each runs its loop over launches with per-launch history offsets."""
    sms = _sm_count()
    fwd_pairs, bwd_pairs = min(2 * sms, 256), min(sms, 256)
    B = fwd_pairs + 4
    assert B > bwd_pairs
    _check_sinkhorn(B, 6, 1800, 5, 1.0, 'labels', seed=11)


# ---------------------------------------------------------------------------------------------------------------------
# b. csrc/train_ops.cuh operators
ROWS = [1, 63, 64, 65, 16385, 2 * 16 * 2048]
COLS = [1, 3, 64, 65, 256, 264]


def _colred_shape(rows):
    """chunking of colreduce_launch: the row chunks and rows per chunk of the two-stage column reduction"""
    chunks = max(1, min(256, -(-rows // 64)))
    rpc = -(-max(rows, 1) // chunks)
    return max(1, -(-rows // rpc)), rpc


def _sum_bound(terms, rows):
    """|fp32 column sum - exact| <= (terms summed in sequence + slack) u sum|terms| for the two-stage reduction"""
    chunks, rpc = _colred_shape(rows)
    return 2 * (rpc + chunks + 4) * U * terms.abs().sum(0)


def _ws(cols):
    return torch.empty(int(_lib().og_train_workspace_floats(cols)), dtype=torch.float32, device=DEV)


def _poison_intact(buf, cols):
    return bool(torch.isnan(buf[:, cols:]).all()) if buf.shape[1] > cols else True


@pytest.mark.gpu
@pytest.mark.parametrize('rows', ROWS)
def test_colsum_matches_float64(rows):
    lib = _lib()
    g = torch.Generator().manual_seed(rows)
    for cols in COLS:
        x, y, z = (torch.randn(rows, cols, generator=g) for _ in range(3))
        xb, _ = _strided(x, cols + 5)
        yb, _ = _strided(y, cols + 3)
        zb, _ = _strided(z, cols + 7)
        x64, y64, z64 = x.double(), y.double(), z.double()
        for use_y, use_z in ((False, False), (True, False), (True, True)):
            terms = x64 * ((y64 - (z64 if use_z else 0)) if use_y else 1)
            out = _nan(cols + 1)
            _check(lib.og_colsum(_p(xb), xb.stride(0), _p(yb if use_y else None), yb.stride(0), _p(zb if use_z else None), zb.stride(0),
                                 rows, cols, _p(out), _p(_ws(cols)), _st()), 'og_colsum')
            got = out[:cols].cpu().double()
            assert torch.isnan(out[cols]).item()
            err = (got - terms.sum(0)).abs()
            bound = _sum_bound(terms, rows) + 4 * U * terms.sum(0).abs()
            assert bool((err <= bound).all()), (cols, use_y, use_z)
        _report(f'colsum {rows}x{cols}', float(err.max()), float(bound.max()))


def _bn_reference(a, gamma, beta, eps, momentum, rm, rv, relu, dy):
    """float64 F.batch_norm(training=True) on relu?(a) with autograd for the backward (rows = 1: the formulas, which torch refuses)"""
    a = a.double().requires_grad_(True)
    r = torch.relu(a) if relu else a                          # (relu: gradient 0 at a = 0, as nn.ReLU)
    rm, rv = rm.double().clone(), rv.double().clone()
    if a.shape[0] > 1:
        y = F.batch_norm(r, rm, rv, gamma.double(), beta.double(), training=True, momentum=momentum, eps=eps)
    else:
        y = (r - r) * gamma.double() + beta.double()
        rm.mul_(1 - momentum).add_(momentum * r.detach()[0])
        rv.mul_(1 - momentum)
    (da,) = torch.autograd.grad(y, a, dy.double())
    mean = r.detach().mean(0)
    var = r.detach().var(0, unbiased=False)
    dbeta = dy.double().sum(0)
    dgamma = (dy.double() * (r.detach() - mean) / (var + eps).sqrt()).sum(0)
    return y.detach(), mean, var, rm, rv, da, dgamma, dbeta


@pytest.mark.gpu
@pytest.mark.parametrize('relu', [False, True], ids=['linear', 'relu'])
@pytest.mark.parametrize('rows', ROWS)
def test_batchnorm_train_fwd_bwd_matches_autograd(rows, relu):
    lib = _lib()
    g = torch.Generator().manual_seed(1000 + rows)
    eps, momentum = 1e-5, 0.1
    for cols in COLS:
        a = 1.5 * torch.randn(rows, cols, generator=g) + 0.3
        gamma, beta = 1 + 0.5 * torch.randn(cols, generator=g), torch.randn(cols, generator=g)
        rm, rv = torch.randn(cols, generator=g), 0.5 + torch.rand(cols, generator=g)
        dy = torch.randn(rows, cols, generator=g)
        y64, mu64, var64, rm64, rv64, da64, dg64, db64 = _bn_reference(a, gamma, beta, eps, momentum, rm, rv, relu, dy)
        ab, _ = _strided(a, cols + 4)
        yb = _nan(rows, cols + 3)
        mean, invstd = _nan(cols), _nan(cols)
        rmd, rvd = rm.to(DEV), rv.to(DEV)
        gd, bd = gamma.to(DEV), beta.to(DEV)
        _check(lib.og_bn_train_fwd(_p(ab), ab.stride(0), rows, cols, int(relu), _p(gd), _p(bd), eps, momentum, _p(yb), yb.stride(0),
                                   _p(mean), _p(invstd), _p(rmd), _p(rvd), _p(_ws(cols)), _st()), 'og_bn_train_fwd')
        r64 = torch.relu(a.double()) if relu else a.double()
        chunks, rpc = _colred_shape(rows)
        k = 2 * (rpc + chunks + 4) * U
        # error model: mean within k mean|r|; the two-pass variance within k var + (mean error)^2; invstd to half var's relative error
        e_mu = k * r64.abs().mean(0) + 2 * U * mu64.abs()
        e_var = k * var64 + e_mu ** 2
        rel_is = 0.5 * e_var / (var64 + eps) + 4 * U
        is64 = 1 / (var64 + eps).sqrt()
        xhat = (r64 - mu64) * is64
        e_y = gamma.double().abs() * (e_mu * is64 + xhat.abs() * (rel_is + 4 * U)) + 2 * U * (y64.abs() + beta.double().abs())
        got = yb[:, :cols].cpu().double()
        assert _poison_intact(yb.cpu(), cols)
        assert bool(((got - y64).abs() <= e_y).all()), ('y', cols)
        assert bool(((mean.cpu().double() - mu64).abs() <= e_mu).all()), ('mean', cols)
        assert bool(((invstd.cpu().double() - is64).abs() <= rel_is * is64).all()), ('invstd', cols)
        n_ub = rows / (rows - 1) if rows > 1 else 1.0
        assert bool(((rmd.cpu().double() - rm64).abs() <= momentum * e_mu + 4 * U * (rm64.abs() + momentum * mu64.abs())).all()), cols
        assert bool(((rvd.cpu().double() - rv64).abs() <= momentum * n_ub * e_var + 4 * U * (rv64.abs() + momentum * n_ub * var64)).all()), cols
        _report(f'bn fwd {rows}x{cols} relu={relu}', float((got - y64).abs().max()), float(e_y.max()))
        # backward from the kernel's own saved statistics; the reference differentiates the float64 forward
        dyb, _ = _strided(dy, cols + 2)
        dab = _nan(rows, cols + 1)
        dgam, dbet = _nan(cols), _nan(cols)
        _check(lib.og_bn_train_bwd(_p(dyb), dyb.stride(0), _p(ab), ab.stride(0), rows, cols, int(relu), _p(gd), _p(mean), _p(invstd),
                                   _p(dab), dab.stride(0), _p(dgam), _p(dbet), _p(_ws(cols)), _st()), 'og_bn_train_bwd')
        dy64 = dy.double()
        # xhat as the kernel forms it, from statistics that carry the forward's errors
        e_xhat = is64 * (e_mu + 2 * U * r64.abs()) + xhat.abs() * (rel_is + 2 * U)
        e_db = _sum_bound(dy64, rows)
        e_dg = _sum_bound(dy64 * xhat, rows) + (dy64.abs() * e_xhat).sum(0)
        e_da = gamma.double().abs() * is64 * (4 * U * dy64.abs() + (e_db + 4 * U * db64.abs()) / rows
                                              + (xhat.abs() * (e_dg + 4 * U * dg64.abs()) + e_xhat * dg64.abs()) / rows) \
            + da64.abs() * (rel_is + 4 * U)
        assert bool(((dbet.cpu().double() - db64).abs() <= e_db).all()), ('dbeta', cols)
        assert bool(((dgam.cpu().double() - dg64).abs() <= e_dg).all()), ('dgamma', cols)
        got = dab[:, :cols].cpu().double()
        assert _poison_intact(dab.cpu(), cols)
        assert bool(((got - da64).abs() <= e_da).all()), ('da', cols)
        _report(f'bn bwd {rows}x{cols} relu={relu}', float((got - da64).abs().max()), float(e_da.max()))


SOFTMAX_COLS = [1, 31, 32, 33, 2100, 4097]


@pytest.mark.gpu
@pytest.mark.parametrize('cols', SOFTMAX_COLS)
def test_softmax_rows_and_backward_match_autograd(cols):
    lib = _lib()
    g = torch.Generator().manual_seed(cols)
    rows, ld, scale = 37, cols + 6, 0.125
    x = 3.0 * torch.randn(rows, cols, generator=g)
    dP = torch.randn(rows, cols, generator=g)
    x64 = x.double().requires_grad_(True)
    P64 = torch.softmax(x64, -1)
    (dx64,) = torch.autograd.grad(P64, x64, dP.double())
    P64 = P64.detach()
    dS64 = scale * dx64
    # forward, in place on a strided buffer whose padding is NaN (a read of the padding would poison the row)
    buf, _ = _strided(x, ld)
    _check(lib.og_softmax_rows(_p(buf), ld, rows, cols, _st()), 'og_softmax_rows')
    got = buf.cpu()
    assert _poison_intact(got, cols)
    P = got[:, :cols].double()
    # exp of (x - max) carries u |x - max| + 2u; the warp's sum (cols / 32 + 5 terms in sequence) and the scaling two more
    xm = (x.double() - x.double().max(-1, keepdim=True).values).abs()
    rel = 2 * (U * xm + (U * xm).max(-1, keepdim=True).values + (cols / 32 + 10) * U)
    err, bound = (P - P64).abs(), rel * P64
    _report(f'softmax {rows}x{cols}', float(err.max()), float(bound.max()))
    assert bool((err <= bound).all())
    # backward from the kernel's P: dS = scale P (dP - sum_j P dP)
    Pd, _ = _strided(P.float(), ld)
    gd, _ = _strided(dP, ld)
    _check(lib.og_softmax_bwd_rows(_p(Pd), _p(gd), ld, rows, cols, scale, _st()), 'og_softmax_bwd_rows')
    got = gd.cpu()
    assert _poison_intact(got, cols)
    dS = got[:, :cols].double()
    dP64 = dP.double()
    dot = (P64 * dP64).sum(-1, keepdim=True)
    e_dot = (cols / 32 + 8) * U * (P64 * dP64).abs().sum(-1, keepdim=True) * 2 + (bound * dP64.abs()).sum(-1, keepdim=True)
    e = scale * (bound * (dP64 - dot).abs() + P64 * (e_dot + 4 * U * (dP64.abs() + dot.abs())))
    err = (dS - dS64).abs()
    _report(f'softmax bwd {rows}x{cols}', float(err.max()), float(e.max()))
    assert bool((err <= e).all())


@pytest.mark.gpu
@pytest.mark.parametrize('S', [1, 3, 130])
@pytest.mark.parametrize('accumulate', [0, 1])
def test_sum_batches_matches_float64(S, accumulate):
    lib = _lib()
    g = torch.Generator().manual_seed(S * 10 + accumulate)
    for rows, cols in ((1, 1), (63, 65), (256, 264), (257, 3)):
        part = torch.randn(S, rows, cols, generator=g)
        init = torch.randn(rows, cols, generator=g)
        ld = cols + 9
        out, _ = _strided(init, ld) if accumulate else (_nan(rows, ld), None)
        pd = part.to(DEV)
        _check(lib.og_sum_batches(_p(pd), S, rows, cols, _p(out), ld, accumulate, _st()), 'og_sum_batches')
        got = out.cpu()
        assert _poison_intact(got, cols)
        want = part.double().sum(0) + (init.double() if accumulate else 0)
        terms_abs = part.double().abs().sum(0) + (init.double().abs() if accumulate else 0)
        bound = (S + 2) * U * terms_abs
        err = (got[:, :cols].double() - want).abs()
        assert bool((err <= bound).all()), (rows, cols)
    _report(f'sum_batches S={S} acc={accumulate}', float(err.max()), float(bound.max()))


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['transpose', 'copy'])
def test_transpose_and_copy_are_exact(mode):
    lib = _lib()
    g = torch.Generator().manual_seed(3)
    t = mode == 'transpose'
    shapes = [(3, 1, 1), (2, 33, 65), (1, 4097, 31), (2, 64, 264)]
    if not t:
        shapes += [(1, 5000, 300), (1, 3, 17000)]          # grid-stride loops over rows (> 4096) and over columns (> 64 x 256)
    for batch, rows, cols in shapes:
        x = torch.randn(batch, rows, cols + 3, generator=g)
        src = x.to(DEV)
        ld_in, stride_in = cols + 3, rows * (cols + 3)
        orows, ocols = (cols, rows) if t else (rows, cols)
        ld_out = ocols + 5
        stride_out = orows * ld_out + 7
        out = _nan(batch * stride_out)
        _check(lib.og_transpose(_p(src), ld_in, stride_in, _p(out), ld_out, stride_out, batch, rows, cols, int(t), _st()), 'og_transpose')
        got = out.cpu()
        want = x[:, :, :cols].transpose(1, 2) if t else x[:, :, :cols]
        view = got.as_strided((batch, orows, ocols), (stride_out, ld_out, 1))
        assert torch.equal(view, want), (batch, rows, cols)
        written = torch.zeros_like(got, dtype=torch.bool)
        written.as_strided((batch, orows, ocols), (stride_out, ld_out, 1)).fill_(True)
        assert bool(torch.isnan(got[~written]).all()), (batch, rows, cols)


@pytest.mark.gpu
def test_elementwise_kernels_within_a_few_ulp():
    lib = _lib()
    g = torch.Generator().manual_seed(5)
    rows, d = 2 * 16 * 2048, 256                           # more elements than one grid covers: the grid-stride loops run
    x, y = torch.randn(rows * d, generator=g), torch.randn(rows * d, generator=g)
    xd, yd = x.to(DEV), y.to(DEV)
    a_, b_ = 0.37, -1.9
    for use_y in (True, False):
        out = _nan(rows * d + 1)
        _check(lib.og_axpby(_p(xd), _p(yd if use_y else None), a_, b_, _p(out), rows * d, _st()), 'og_axpby')
        got = out.cpu()
        assert torch.isnan(got[-1]).item()
        ax, by = float(torch.tensor(a_, dtype=torch.float32)) * x.double(), float(torch.tensor(b_, dtype=torch.float32)) * y.double()
        want = ax + by if use_y else ax
        bound = 2 * U * (ax.abs() + (by.abs() if use_y else 0))
        err = (got[:-1].double() - want).abs()
        _report(f'axpby y={use_y}', float(err.max()), float(bound.max()))
        assert bool((err <= bound).all())
    # residual mix: out = alpha g + (1 - alpha) l, alpha = sigmoid(mix); backward and d mix through autograd
    gm, lm = x.view(rows, d), y.view(rows, d)
    mix = 1.5 * torch.randn(d, generator=g)
    dm = torch.randn(rows, d, generator=g)
    mix64 = mix.double().requires_grad_(True)
    g64, l64 = gm.double().requires_grad_(True), lm.double().requires_grad_(True)
    al64 = torch.sigmoid(mix64)
    out64 = al64 * g64 + (1 - al64) * l64
    dg64, dl64, dmix64 = torch.autograd.grad(out64, (g64, l64, mix64), dm.double())
    al = al64.detach()
    e_al = 8 * U * al                                       # expf, add, divide
    e_1mal = e_al + 2 * U * (1 - al)
    mixd, gd, ld_, dmd = mix.to(DEV), gm.to(DEV).contiguous(), lm.to(DEV).contiguous(), dm.to(DEV)
    out = _nan(rows * d + 1)
    _check(lib.og_mix_fwd(_p(gd), _p(ld_), _p(mixd), _p(out), rows, d, _st()), 'og_mix_fwd')
    got = out.cpu()
    assert torch.isnan(got[-1]).item()
    bound = gm.double().abs() * e_al + lm.double().abs() * e_1mal + 3 * U * (al * gm.double().abs() + (1 - al) * lm.double().abs())
    err = (got[:-1].view(rows, d).double() - out64.detach()).abs()
    _report('mix fwd', float(err.max()), float(bound.max()))
    assert bool((err <= bound).all())
    dg, dl = _nan(rows * d + 1), _nan(rows * d + 1)
    _check(lib.og_mix_bwd(_p(dmd), _p(mixd), _p(dg), _p(dl), rows, d, _st()), 'og_mix_bwd')
    dg, dl = dg.cpu(), dl.cpu()
    assert torch.isnan(dg[-1]).item() and torch.isnan(dl[-1]).item()
    for got, want, e in ((dg, dg64, e_al + U * al), (dl, dl64, e_1mal + U * (1 - al))):
        err, bound = (got[:-1].view(rows, d).double() - want).abs(), dm.double().abs() * e
        assert bool((err <= bound).all())
    _report('mix bwd', float(err.max()), float(bound.max()))
    # d mix = colsum(dm (g - l)) alpha (1 - alpha): the training step's two kernels in sequence
    cs = _nan(d)
    _check(lib.og_colsum(_p(dmd), d, _p(gd), d, _p(ld_), d, rows, d, _p(cs), _p(_ws(d)), _st()), 'og_colsum')
    dmix = _nan(d + 1)
    _check(lib.og_mix_param_grad(_p(cs), _p(mixd), _p(dmix), d, _st()), 'og_mix_param_grad')
    got = dmix.cpu()
    assert torch.isnan(got[-1]).item()
    terms = dm.double() * (gm.double() - lm.double())
    w = al * (1 - al)
    csum = terms.sum(0)
    bound = w * _sum_bound(terms, rows) + csum.abs() * (e_al * (1 - al) + e_1mal * al + 4 * U * w)
    err = (got[:-1].double() - dmix64).abs()
    _report('d mix', float(err.max()), float(bound.max()))
    assert bool((err <= bound).all())
    # keypoint-encoder input [2 x / (W - 1) - 1, 2 y / (H - 1) - 1, side info]
    for S_ in (0, 1, 6):
        n = 3000
        kp = torch.rand(n, 2, generator=g) * torch.tensor([639.0, 479.0])
        side = torch.rand(n, max(S_, 1), generator=g)
        kd, sd = kp.to(DEV), side.to(DEV)
        out = _nan(n * (2 + S_) + 1)
        _check(lib.og_kenc_input(_p(kd), _p(sd) if S_ else None, n, S_, 640.0, 480.0, _p(out), _st()), 'og_kenc_input')
        got = out.cpu()
        assert torch.isnan(got[-1]).item()
        got = got[:-1].view(n, 2 + S_)
        q = 2 * kp.double() / torch.tensor([639.0, 479.0], dtype=torch.float64)
        assert bool(((got[:, :2].double() - (q - 1)).abs() <= 2 * U * (q.abs() + 1)).all()), S_
        if S_:
            assert torch.equal(got[:, 2:], side[:, :S_])


# ---------------------------------------------------------------------------------------------------------------------
# c. The whole training step at training sizes, against the float64 torch double of its kernels
STEP_CASES = {
    # B = 2, N = 700, M = 2100: 1400 and 4200 rows per image -> split-K weight gradients of 3 and 9 chunks (the last ragged);
    # M = 2100 puts the Sinkhorn backward in its 2048 < m <= 4096 band; d = 256, 4 heads: head_dim 64, the tf32 attention
    'd256_h4': dict(B=2, N=700, M=2100, cfg=dict(descriptor_dim=256, num_stages=2, num_heads=4, num_iters=20)),
    'offset_reg05': dict(B=2, N=701, M=1030, cfg=dict(descriptor_dim=128, num_stages=2, num_heads=4, num_iters=20, reg=0.5,
                                                      use_offset=True)),
}


def _step_inputs(case):
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
    c = STEP_CASES[case]
    cfg = default_config(**c['cfg'])
    sd = synthetic_state_dict(cfg, seed=3)
    data = synthetic_pairs(c['B'], c['N'], c['M'], cfg['descriptor_dim'], 1, family='planted', seed=17)
    gt0 = data['planted_matches0']
    gt1 = torch.full((c['B'], c['M']), -1, dtype=torch.int64)
    for b in range(c['B']):
        src = torch.nonzero(gt0[b] >= 0).flatten()
        gt1[b, gt0[b, src]] = src
    return cfg, sd, data, {'gt_matches0': gt0, 'gt_matches1': gt1}


def _run_step(cfg, sd, data, labels, dtype=None, precision=None):
    """one TrainStep: on the GPU (precision given) or on the torch double of its kernels in `dtype` -> every output as float64 on the CPU"""
    from openglue_b200 import SuperGlue
    from openglue_b200.training import TrainStep
    from test_training import _CpuOps
    model = SuperGlue(dict(cfg, precision=precision or 'fp32'))
    model.load_state_dict(sd, strict=True)
    keys = ('keypoints0', 'keypoints1', 'side_info0', 'side_info1', 'local_descriptors0', 'local_descriptors1')
    if precision is None:
        model = model.to(dtype).train()
        d = {k: (v.to(dtype) if k in keys else v) for k, v in data.items()}
        step = TrainStep(model, d, ops=_CpuOps(dtype))
    else:
        model = model.to(DEV).train()
        d = {k: (v.to(DEV) if k in keys else v) for k, v in data.items()}
        step = TrainStep(model, d)
    scores, _, _ = step.forward()
    scores = scores.detach().double().cpu()
    loss = float(L.criterion(labels, {'scores': scores})['loss'])
    G = L.criterion_grad(labels, tuple(scores.shape))
    grads = step.backward(G.to(dtype or torch.float32).to(scores.device if precision is None else DEV))
    out = {'scores': scores, 'loss': torch.tensor(loss, dtype=torch.float64)}
    out.update({k: v.detach().double().cpu().reshape(-1) for k, v in grads.items()})
    out.update({'buffer.' + k: v.detach().double().cpu() for k, v in model.named_buffers() if 'running_' in k})
    return out


@pytest.fixture(scope='module')
def step_refs():
    cache = {}

    def get(case):
        if case not in cache:
            inputs = _step_inputs(case)
            cache[case] = inputs, _run_step(*inputs, dtype=torch.float64), _run_step(*inputs, dtype=torch.float32)
        return cache[case]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['tf32x3', 'fp32'])
@pytest.mark.parametrize('case', list(STEP_CASES))
def test_training_step_at_training_size(step_refs, case, precision):
    inputs, r64, r32 = step_refs(case)
    got = _run_step(*inputs, precision=precision)
    assert set(got) == set(r64)
    # scores and BatchNorm buffers: 8 x the float32 double's own distance from float64 (the problem's conditioning at this size).
    # The loss is a weighted sum of scores (weights d loss / d scores): sum |weights| x the scores' bound.
    # Gradients: the larger of that distance and tests/test_training.py's elementwise rule, 1e-3 of the tensor's largest entry.  The
    # fp32 kernels reduce over rows in sequential chunks and the Sinkhorn backward is held to 2e-4 of max|dS|; the float32 double sums
    # pairwise with exact exponentials, so its distance alone under-states the kernels' rounding on gradients that cancel (the
    # biases in front of a BatchNorm).
    scores_bound = max(8 * float((r32['scores'] - r64['scores']).abs().max()), 4 * U * float(r64['scores'].abs().max()))
    weights = float(L.criterion_grad(inputs[3], tuple(r64['scores'].shape)).abs().sum())
    worst = ('', 0.0)
    for k in sorted(r64):
        g, w64, w32 = got[k], r64[k], r32[k]
        assert g.shape == w64.shape, k
        assert bool(torch.isfinite(g).all()), k
        scale = float(w64.abs().max())
        if scale < 1e-9:                                    # the key biases: a shift of every logit of a row, gradient 0 (tests/test_training.py's rule)
            assert float(g.abs().max()) < 1e-6, k
            continue
        if k == 'scores':
            bound = scores_bound
        elif k == 'loss':
            bound = weights * scores_bound
        elif k.startswith('buffer.'):
            bound = max(8 * float((w32 - w64).abs().max()), 4 * U * scale)
        else:
            bound = max(8 * float((w32 - w64).abs().max()), 1e-3 * scale)
        err = float((g - w64).abs().max())
        assert err <= bound, (k, err, bound)
        worst = max(worst, (k, err / bound if bound else 0.0), key=lambda t: t[1])
    print(f'\n[{case} {precision}] {len(r64)} tensors; worst error/bound {worst[1]:.2f} ({worst[0]})')
