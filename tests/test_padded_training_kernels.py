"""The padded forms of the training kernels at training sizes, pair by pair against float64 references on each trimmed pair.

A padded batch holds pair b as the [n_b, m_b] block of a shared capacity N x M; what lies outside the block is padding of any bits.
Each operator is checked where its uniform form was checked in tests/test_training_kernels.py, and with the lengths that cut its
tiles, chunks, strips and column bands:
  1. the Sinkhorn with history and its backward (og_sinkhorn_train_fwd_padded, og_sinkhorn_bwd_padded) at capacities that select
     every column band, against oracle/sinkhorn_grad_oracle.py; junk padding (NaN, +-inf, 1e30) gives the zero-padding bits;
  2. masked BatchNorm forward, backward and the guarded form, against float64 autograd on the real rows;
  3. the masked row softmax and its backward;
  4. the padded criterion and its gradient scatter;
  5. the padded labels (og_gt_matches_fwd_padded) at a capacity above the nearest-neighbour tile, against oracle/gt_matches_oracle.py;
  6. the keypoint-encoder input and the row mask;
  7. fp16x3 attention with key lengths.
Bounds come from an error model or from the float32 reference's own distance to float64; every case prints its error next to its
bound."""
import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200._cabi import ptr as _p, stream as _st
from oracle import gt_matches_oracle as GO
from oracle import loss_oracle as L
from test_attention_kernels import CONTRACT, Operands, _reference
from test_gt_matches import _checkable
from test_training_kernels import (U, _bn_reference, _colred_shape, _deviation_bound, _nan, _report, _sink_inputs, _sink_oracle,
                                   _sm_count, _sum_bound, _ws)

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
FILLS = [float('nan'), float('inf'), -float('inf'), 1e30]


def _lib():
    return _cabi.lib()


def _bits(t):
    return t.view(torch.int32)


def _same_bits(a, b, what):
    assert torch.equal(_bits(a), _bits(b)), f'{what}: {int((_bits(a) != _bits(b)).sum())} elements differ'


# ---------------------------------------------------------------------------------------------------------------------
# 1. Sinkhorn with history and its backward, padded
def _sink_batch(pairs, N, M, upstream, seed):
    """per-pair inputs (S_b [1, n, m], G_b [1, n + 1, m + 1]) of `pairs` [(n, m)]"""
    out = []
    for b, (n, m) in enumerate(pairs):
        S, dust, G = _sink_inputs(1, n, m, upstream, seed * 1000 + b)
        out.append((S, G))
    return out, dust


def _sink_padded_run(inputs, dust, N, M, iters, reg, fill=0.0, padded=True):
    """og_sinkhorn_train_fwd(_padded) + og_sinkhorn_bwd(_padded) with S's padding (rows >= n_b, columns >= m_b, the row tails past M)
    and dscores outside each block set to `fill`; outputs NaN-poisoned.  padded=False: the uniform entry points (every pair at the
    capacity)."""
    lib = _lib()
    B = len(inputs)
    lds = (M + 3) // 4 * 4 + 4
    strideS = N * lds + 64
    Sbuf = torch.full((B * strideS,), fill, dtype=torch.float32)
    Sv = Sbuf.as_strided((B, N, lds), (strideS, lds, 1))
    G = torch.full((B, N + 1, M + 1), fill, dtype=torch.float32)
    for b, (S_b, G_b) in enumerate(inputs):
        n, m = S_b.shape[1:]
        Sv[b, :n, :m] = S_b[0]
        G[b, :n + 1, :m + 1] = G_b[0]
    Sd, Gd, d = Sbuf.to(DEV), G.to(DEV), dust.reshape(1).to(DEV)
    lens = torch.tensor([x[0].shape[1] for x in inputs] + [x[0].shape[2] for x in inputs], dtype=torch.int32, device=DEV)
    scores = _nan(B, N + 1, M + 1)
    hist = _nan(max(int(lib.og_sinkhorn_hist_floats(B, N, M, iters)), 1))
    wsb = int(lib.og_sinkhorn_workspace_bytes(B, N, M))
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    if padded:
        rc = lib.og_sinkhorn_train_fwd_padded(_p(Sd), lds, strideS, _p(d), B, N, M, _p(lens), iters, reg, _p(scores), _p(hist), _p(ws), wsb,
                                              _st())
    else:
        rc = lib.og_sinkhorn_train_fwd(_p(Sd), lds, strideS, _p(d), B, N, M, iters, reg, _p(scores), _p(hist), _p(ws), wsb, _st())
    _cabi.check(rc, 'og_sinkhorn_train_fwd_padded')
    dZ, dd = _nan(B, N + 1, M + 1), _nan(1)
    wsb = int(lib.og_sinkhorn_bwd_workspace_bytes(B, N, M, iters))
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    if padded:
        rc = lib.og_sinkhorn_bwd_padded(_p(Sd), lds, strideS, _p(d), B, N, M, _p(lens), iters, reg, _p(hist), _p(Gd), _p(dZ), _p(dd), _p(ws),
                                        wsb, _st())
    else:
        rc = lib.og_sinkhorn_bwd(_p(Sd), lds, strideS, _p(d), B, N, M, iters, reg, _p(hist), _p(Gd), _p(dZ), _p(dd), _p(ws), wsb, _st())
    _cabi.check(rc, 'og_sinkhorn_bwd_padded')
    torch.cuda.synchronize()
    return scores.cpu(), hist.cpu(), dZ.cpu(), dd.cpu()


def _check_sink_pairs(tag, inputs, dust, N, M, iters, reg, out):
    """every pair of `out` against the float64 oracle on the trimmed pair (float32 oracle for the bounds)"""
    scores, hist, dZ, dd = out
    B = len(inputs)
    hu = hist[:B * iters * (N + 1)].view(B, iters, N + 1).double()
    hv = hist[B * iters * (N + 1):B * iters * (N + 1) + B * (iters + 1) * (M + 1)].view(B, iters + 1, M + 1).double()
    dd64 = dd_bound = dd_terms = 0.0
    worst = {}
    for b, (S_b, G_b) in enumerate(inputs):
        n, m = S_b.shape[1:]
        r64 = _sink_oracle(S_b, dust, G_b, iters, reg, torch.float64)
        r32 = _sink_oracle(S_b, dust, G_b, iters, reg, torch.float32)
        checks = [('scores', scores[b, :n + 1, :m + 1].double(), r64[0][0], _deviation_bound(r64[0], r32[0]))]
        assert torch.equal(hv[b, 0, :m + 1], torch.zeros(m + 1, dtype=torch.float64)), b
        # u_t and v_t are log-sum-exps whose arguments reach max|scores|: each rounding moves them by ulps of that magnitude, which the
        # float32 oracle's distance need not show on a pair of one or two columns
        floor = 16 * U * float(r64[0].abs().max())
        for t in range(iters):
            checks.append((f'u_{t + 1}', hu[b, t, :n + 1], r64[1][t][0], max(_deviation_bound(r64[1][t], r32[1][t]), floor)))
            checks.append((f'v_{t + 1}', hv[b, t + 1, :m + 1], r64[2][t + 1][0], max(_deviation_bound(r64[2][t + 1], r32[2][t + 1]), floor)))
        scale = float(r64[3].abs().max())
        checks.append(('dS', dZ[b, :n, :m].double(), r64[3][0], max(2e-4 * scale, 4 * float((r64[3] - r32[3]).abs().max()))))
        for name, got, want, bound in checks:
            err = float((got - want).abs().max())
            assert err <= bound, (tag, b, (n, m), name, err, bound)
            key = name if name[0] not in 'uv' else name[0]
            ratio = err / bound if bound > 0 else 0.0
            if ratio >= worst.get(key, (-1.0,))[0]:
                worst[key] = (ratio, err, bound, (n, m))
        # outside the block: scores -inf, dS_aug exactly 0
        blk = scores[b].clone()
        blk[:n + 1, :m + 1] = -float('inf')
        assert torch.isneginf(blk).all(), (tag, b)
        rest = dZ[b].clone()
        rest[:n + 1, :m + 1] = 0
        assert (rest == 0).all() and not torch.isnan(rest).any(), (tag, b)
        # d dustbin of this pair is the sum of its dustbin row and column of dS_aug (a recursive fp32 sum of n + m + 1 terms)
        terms = torch.cat([dZ[b, n, :m + 1], dZ[b, :n, m]]).double()
        assert abs(float(terms.sum()) - r64[4]) <= max(2e-4 * max(abs(r64[4]), 1e-3), 4 * abs(r32[4] - r64[4])) + \
            (n + m + 1) * U * float(terms.abs().sum()), (tag, b)
        dd64 += r64[4]
        dd_bound += max(2e-4 * max(abs(r64[4]), 1e-3), 4 * abs(r32[4] - r64[4]))
        dd_terms += float(terms.abs().sum())
    for key, (ratio, err, bound, nm) in sorted(worst.items()):
        _report(f'{tag} {key} (worst pair {nm[0]}x{nm[1]})', err, bound)
    dd_bound += (N + M + 1 + B) * U * dd_terms                     # the kernel's fp32 sums: per pair, then over the pairs
    err = abs(float(dd) - dd64)
    _report(f'{tag} d dustbin', err, dd_bound)
    assert err <= dd_bound


def _sink_case(N, M, pairs, iters, reg, upstream, seed, tag):
    inputs, dust = _sink_batch(pairs, N, M, upstream, seed)
    zero = _sink_padded_run(inputs, dust, N, M, iters, reg)
    _check_sink_pairs(tag, inputs, dust, N, M, iters, reg, zero)
    names = ('scores', 'hist', 'dS_aug', 'd dustbin')
    for a, b, what in zip(zero, _sink_padded_run(inputs, dust, N, M, iters, reg), names):
        _same_bits(a, b, f'second run: {what}')
    for fill in FILLS:
        for a, b, what in zip(zero, _sink_padded_run(inputs, dust, N, M, iters, reg, fill=fill), names):
            _same_bits(a, b, f'padding {fill}: {what}')


# (N, M, pairs, T, reg, upstream): per capacity, a pair at full size, n_b = 1, m_b = 1, m_b % 4 in {1, 2, 3}, and a pair whose m_b
# falls in a narrower column band than the capacity's
SINK_CASES = {
    'M512_V4W1': (300, 512, [(300, 512), (1, 509), (300, 1), (150, 257), (77, 510), (299, 511), (40, 60)], 10, 1.0, 'labels'),
    'M1024_V4W2': (200, 1024, [(200, 1024), (1, 1021), (200, 1), (60, 1022), (199, 1023), (33, 500)], 7, 0.7, 'dense'),
    'M2048_V8W2': (150, 2048, [(150, 2048), (1, 2047), (150, 1), (80, 1025), (149, 2046), (10, 100)], 100, 1.0, 'labels'),
    'M4096_V16W2_bwd_one_slot': (100, 4096, [(100, 4096), (1, 4093), (100, 1), (57, 4094), (99, 4095), (20, 600)], 5, 0.7, 'dense'),
    'M8192_V16W4': (64, 8192, [(64, 8192), (1, 8191), (64, 1), (30, 4097), (63, 8190), (64, 100)], 3, 1.0, 'labels'),
    # n_b leaves more than half of the 32 strips of the capacity empty
    'empty_strips': (1000, 700, [(1000, 700), (100, 650), (3, 699)], 4, 1.0, 'dense'),
    'T0': (40, 300, [(40, 300), (1, 1), (17, 299)], 0, 0.7, 'dense'),
    'T1': (64, 130, [(64, 130), (2, 129), (63, 3)], 1, 1.0, 'labels'),
}


@pytest.mark.parametrize('case', list(SINK_CASES))
def test_sinkhorn_padded_fwd_bwd_per_pair_against_oracle(case):
    N, M, pairs, iters, reg, upstream = SINK_CASES[case]
    _sink_case(N, M, pairs, iters, reg, upstream, seed=list(SINK_CASES).index(case), tag=f'{case} T={iters} reg={reg}')


def test_sinkhorn_padded_training_shaped_batch():
    """4 pairs at capacity 2048 x 2048, lengths uniform in [1024, 2048] as tools/padded_train_timing.py draws them"""
    g = torch.Generator().manual_seed(2048)
    n0, n1 = torch.randint(1024, 2049, (4,), generator=g), torch.randint(1024, 2049, (4,), generator=g)
    _sink_case(2048, 2048, list(zip(n0.tolist(), n1.tolist())), 20, 1.0, 'labels', seed=20, tag='2048x2048 training-shaped T=20')


def test_sinkhorn_padded_launch_loop_over_pairs():
    """More pairs than one cooperative launch holds (the shape of test_sinkhorn_train_launch_loop_over_pairs), with ragged lengths:
    both passes loop over launches and offset the lengths by each launch's first pair."""
    B = min(2 * _sm_count(), 256) + 4
    g = torch.Generator().manual_seed(11)
    pairs = [(int(torch.randint(1, 7, (1,), generator=g)), int(torch.randint(1, 1801, (1,), generator=g))) for _ in range(B)]
    pairs[0], pairs[-1] = (6, 1800), (1, 1)
    _sink_case(6, 1800, pairs, 5, 1.0, 'labels', seed=21, tag=f'B={B} 6x1800 launch loop T=5')


@pytest.mark.parametrize('M', [512, 1024, 2048, 4096, 8192])
def test_sinkhorn_padded_at_capacity_is_the_uniform_kernel_bit_for_bit(M):
    N = 70
    inputs, dust = _sink_batch([(N, M)] * 3, N, M, 'dense', seed=M)
    for iters, reg in ((5, 0.7), (2, 1.0)):
        for a, b, what in zip(_sink_padded_run(inputs, dust, N, M, iters, reg), _sink_padded_run(inputs, dust, N, M, iters, reg, padded=False),
                              ('scores', 'hist', 'dS_aug', 'd dustbin')):
            _same_bits(a, b, f'M={M} T={iters}: {what}')


# ---------------------------------------------------------------------------------------------------------------------
# 2. masked BatchNorm
BN_SHAPES = {'16x2048': (16, 2048), '33x1000_chunks_straddle_pairs': (33, 1000)}


def _bn_lengths(B, cap, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, cap + 1, (B,), generator=g)
    lens[:3] = torch.tensor([1, cap - 1, cap])
    return lens


@pytest.mark.parametrize('relu', [False, True], ids=['linear', 'relu'])
@pytest.mark.parametrize('shape', list(BN_SHAPES))
def test_masked_batchnorm_against_float64(shape, relu):
    lib = _lib()
    B, cap = BN_SHAPES[shape]
    rows = B * cap
    lens = _bn_lengths(B, cap, seed=rows)
    real = torch.cat([torch.arange(b * cap, b * cap + int(n)) for b, n in enumerate(lens)])
    pad = torch.ones(rows, dtype=torch.bool).index_fill_(0, real, False)
    ld = torch.tensor(lens.tolist(), dtype=torch.int32, device=DEV)
    chunks, rpc = _colred_shape(rows)
    if shape.startswith('33'):
        assert rpc == 129 and cap % rpc                      # the column reduction's row chunks straddle pairs
    eps, momentum = 1e-5, 0.1
    g = torch.Generator().manual_seed(7 + rows + relu)
    for cols in (64, 256, 512):
        a = 1.5 * torch.randn(rows, cols, generator=g) + 0.3
        gamma, beta = 1 + 0.5 * torch.randn(cols, generator=g), torch.randn(cols, generator=g)
        rm, rv = torch.randn(cols, generator=g), 0.5 + torch.rand(cols, generator=g)
        dy = torch.randn(rows, cols, generator=g)
        y64, mu64, var64, rm64, rv64, da64, dg64, db64 = _bn_reference(a[real], gamma, beta, eps, momentum, rm, rv, relu, dy[real])
        n_real = real.numel()

        def run(fill, guarded=None):
            ad, dyd = a.clone(), dy.clone()
            ad[pad], dyd[pad] = fill, fill
            ad, dyd = ad.to(DEV), dyd.to(DEV)
            y, dab = _nan(rows, cols), _nan(rows, cols)
            mean, invstd, dgam, dbet = _nan(cols), _nan(cols), _nan(cols), _nan(cols)
            rmd, rvd = rm.to(DEV), rv.to(DEV)
            gd, bd = gamma.to(DEV), beta.to(DEV)
            nbt = torch.full((1,), 41, dtype=torch.int64, device=DEV)
            if guarded is None:
                rc = lib.og_bn_train_fwd_padded(_p(ad), cols, B, cap, _p(ld), cols, int(relu), _p(gd), _p(bd), eps, momentum, _p(y), cols, _p(mean),
                                                _p(invstd), _p(rmd), _p(rvd), _p(_ws(cols)), _st())
            else:
                skip = torch.tensor([guarded], dtype=torch.int32, device=DEV)
                rc = lib.og_bn_train_fwd_guarded(_p(ad), cols, B, cap, _p(ld), cols, int(relu), _p(gd), _p(bd), eps, momentum, _p(y), cols,
                                                 _p(mean), _p(invstd), _p(rmd), _p(rvd), _p(skip), _p(nbt), _p(_ws(cols)), _st())
            _cabi.check(rc, 'og_bn_train_fwd_padded')
            _cabi.check(lib.og_bn_train_bwd_padded(_p(dyd), cols, _p(ad), cols, B, cap, _p(ld), cols, int(relu), _p(gd), _p(mean), _p(invstd),
                                                   _p(dab), cols, _p(dgam), _p(dbet), _p(_ws(cols)), _st()), 'og_bn_train_bwd_padded')
            torch.cuda.synchronize()
            return {'y': y.cpu()[real], 'mean': mean.cpu(), 'invstd': invstd.cpu(), 'running_mean': rmd.cpu(), 'running_var': rvd.cpu(),
                    'da': dab.cpu(), 'dgamma': dgam.cpu(), 'dbeta': dbet.cpu(), 'num_batches_tracked': nbt.cpu()}

        got = run(0.0)
        # forward: the error model of test_batchnorm_train_fwd_bwd_matches_autograd, over the real rows of the padded reduction
        r64 = torch.relu(a[real].double()) if relu else a[real].double()
        k = 2 * (rpc + chunks + 4) * U
        e_mu = k * r64.abs().mean(0) + 2 * U * mu64.abs()
        e_var = k * var64 + e_mu ** 2
        rel_is = 0.5 * e_var / (var64 + eps) + 4 * U
        is64 = 1 / (var64 + eps).sqrt()
        xhat = (r64 - mu64) * is64
        e_y = gamma.double().abs() * (e_mu * is64 + xhat.abs() * (rel_is + 4 * U)) + 2 * U * (y64.abs() + beta.double().abs())
        err = (got['y'].double() - y64).abs()
        _report(f'bn fwd {shape} cols={cols} relu={relu}', float(err.max()), float(e_y.max()))
        assert bool((err <= e_y).all()), ('y', cols)
        assert bool(((got['mean'].double() - mu64).abs() <= e_mu).all()), ('mean', cols)
        n_ub = n_real / (n_real - 1)
        assert bool(((got['running_mean'].double() - rm64).abs() <= momentum * e_mu + 4 * U * (rm64.abs() + momentum * mu64.abs())).all())
        assert bool(((got['running_var'].double() - rv64).abs() <= momentum * n_ub * e_var + 4 * U * (rv64.abs() + momentum * n_ub * var64)).all())
        # backward from the kernel's own statistics
        dy64 = dy[real].double()
        e_xhat = is64 * (e_mu + 2 * U * r64.abs()) + xhat.abs() * (rel_is + 2 * U)
        e_db = _sum_bound(dy64, rows)
        e_dg = _sum_bound(dy64 * xhat, rows) + (dy64.abs() * e_xhat).sum(0)
        e_da = gamma.double().abs() * is64 * (4 * U * dy64.abs() + (e_db + 4 * U * db64.abs()) / n_real
                                              + (xhat.abs() * (e_dg + 4 * U * dg64.abs()) + e_xhat * dg64.abs()) / n_real) \
            + da64.abs() * (rel_is + 4 * U)
        assert bool(((got['dbeta'].double() - db64).abs() <= e_db).all()), ('dbeta', cols)
        assert bool(((got['dgamma'].double() - dg64).abs() <= e_dg).all()), ('dgamma', cols)
        err = (got['da'][real].double() - da64).abs()
        _report(f'bn bwd {shape} cols={cols} relu={relu}', float(err.max()), float(e_da.max()))
        assert bool((err <= e_da).all()), ('da', cols)
        assert (got['da'][pad] == 0).all()
        # NaN padding (in a and dy) changes no real-row output; the guarded form is the padded form, or with skip = 1 leaves the
        # running statistics and num_batches_tracked untouched
        junk = run(float('nan'))
        for key in ('y', 'mean', 'invstd', 'running_mean', 'running_var', 'dgamma', 'dbeta', 'da'):
            _same_bits(junk[key], got[key], f'NaN padding: {key}')
        kept = run(0.0, guarded=0)
        for key in got:
            if key != 'num_batches_tracked':
                _same_bits(kept[key], got[key], f'guarded, skip = 0: {key}')
        assert int(kept['num_batches_tracked']) == 42
        skipped = run(0.0, guarded=1)
        assert torch.equal(skipped['running_mean'], rm) and torch.equal(skipped['running_var'], rv)
        assert int(skipped['num_batches_tracked']) == 41


# ---------------------------------------------------------------------------------------------------------------------
# 3. masked softmax and its backward
def test_masked_softmax_and_backward_against_float64():
    lib = _lib()
    key_lens = [1, 31, 32, 33, 1024, 2047, 2048]
    B, seq, cap = len(key_lens), 4 * 512, 2048                       # 4 heads x 512 queries per sequence, 2048 key columns
    ld, scale = cap + 4, 0.125
    g = torch.Generator().manual_seed(33)
    x = 3.0 * torch.randn(B * seq, cap, generator=g)
    dP = torch.randn(B * seq, cap, generator=g)
    kl = torch.tensor(key_lens, dtype=torch.int32, device=DEV)

    def run(fill):
        xs, ds = x.clone(), dP.clone()
        for b, n in enumerate(key_lens):
            xs[b * seq:(b + 1) * seq, n:] = fill
            ds[b * seq:(b + 1) * seq, n:] = fill
        P = torch.full((B * seq, ld), float('nan'), device=DEV)
        P[:, :cap] = xs.to(DEV)
        _cabi.check(lib.og_softmax_rows_padded(_p(P), ld, B, seq, cap, _p(kl), _st()), 'og_softmax_rows_padded')
        dS = torch.full((B * seq, ld), float('nan'), device=DEV)
        dS[:, :cap] = ds.to(DEV)
        _cabi.check(lib.og_softmax_bwd_rows_padded(_p(P), _p(dS), ld, B, seq, cap, scale, _p(kl), _st()), 'og_softmax_bwd_rows_padded')
        torch.cuda.synchronize()
        return P.cpu(), dS.cpu()

    P, dS = run(0.0)
    assert torch.isnan(P[:, cap:]).all() and torch.isnan(dS[:, cap:]).all()
    for b, n in enumerate(key_lens):
        r = slice(b * seq, (b + 1) * seq)
        x64 = x[r, :n].double().requires_grad_(True)
        P64 = torch.softmax(x64, -1)
        (dx64,) = torch.autograd.grad(P64, x64, dP[r, :n].double())
        P64 = P64.detach()
        xm = (x[r, :n].double() - x[r, :n].double().max(-1, keepdim=True).values).abs()
        rel = 2 * (U * xm + (U * xm).max(-1, keepdim=True).values + (n / 32 + 10) * U)
        err, bound = (P[r, :n].double() - P64).abs(), rel * P64
        _report(f'masked softmax len={n}', float(err.max()), float(bound.max()))
        assert bool((err <= bound).all()), n
        # backward from the kernel's P, as in test_softmax_rows_and_backward_match_autograd
        Pk = P[r, :n].double()
        dP64 = dP[r, :n].double()
        dot = (P64 * dP64).sum(-1, keepdim=True)
        e_dot = (n / 32 + 8) * U * (P64 * dP64).abs().sum(-1, keepdim=True) * 2 + (bound * dP64.abs()).sum(-1, keepdim=True)
        e = scale * (bound * (dP64 - dot).abs() + P64 * (e_dot + 4 * U * (dP64.abs() + dot.abs())))
        err = (dS[r, :n].double() - scale * dx64).abs()
        _report(f'masked softmax bwd len={n}', float(err.max()), float(e.max()))
        assert bool((err <= e).all()), n
        assert (Pk >= 0).all()
        assert (P[r, n:cap] == 0).all() and (dS[r, n:cap] == 0).all(), n
    Pn, dSn = run(float('nan'))
    _same_bits(Pn, P, 'NaN past the lengths: P')
    _same_bits(dSn, dS, 'NaN past the lengths: dS')


# ---------------------------------------------------------------------------------------------------------------------
# 4. the padded criterion
def test_padded_criterion_is_the_mean_of_the_trimmed_pairs():
    from openglue_b200.losses import criterion_with_grad
    B, N, M = 16, 2048, 2048
    g = torch.Generator().manual_seed(44)
    ns, ms = torch.randint(1, N + 1, (B,), generator=g), torch.randint(1, M + 1, (B,), generator=g)
    ns[:4], ms[:4] = torch.tensor([1, N, 700, 2047]), torch.tensor([M, 1, 900, 2048])
    scores = torch.full((B, N + 1, M + 1), float('nan'))
    gt0, gt1 = torch.full((B, N), 5, dtype=torch.int64), torch.full((B, M), 7, dtype=torch.int64)     # junk past the lengths
    pairs = []
    for b in range(B):
        n, m = int(ns[b]), int(ms[b])
        s = torch.log_softmax(torch.randn(n + 1, m + 1, generator=g), -1)
        g0, g1 = torch.randint(-2, m, (n,), generator=g), torch.randint(-2, n, (m,), generator=g)
        if b == 2:                                       # no -1 rows
            g0 = torch.randint(0, m, (n,), generator=g)
        if b == 3:                                       # every label ignored
            g0, g1 = torch.full((n,), -2, dtype=torch.int64), torch.full((m,), -2, dtype=torch.int64)
        scores[b, :n + 1, :m + 1], gt0[b, :n], gt1[b, :m] = s, g0, g1
        pairs.append((n, m, s, g0, g1))
    y = {'gt_matches0': gt0.to(DEV), 'gt_matches1': gt1.to(DEV), 'num_keypoints0': ns, 'num_keypoints1': ms}
    loss, ds = criterion_with_grad(y, {'scores': scores.to(DEV)})
    ds = ds.cpu()
    ref, terms_abs = 0.0, 0.0
    for b, (n, m, s, g0, g1) in enumerate(pairs):
        yb = {'gt_matches0': g0[None], 'gt_matches1': g1[None]}
        ref += float(L.criterion(yb, {'scores': s[None].double()})['loss'])
        w = L.criterion_grad(yb, (1, n + 1, m + 1))[0]
        terms_abs += float((w * s.double()).abs().sum())
        # the scatter of the weights -1 / (B c), -0.5 / (B c): the kernel divides once, correctly rounded
        want = torch.zeros(n + 1, m + 1, dtype=torch.float64)
        for sel, wt in (((g0 >= 0), 1.0), ((g0 == -1), 0.5)):
            c = int(sel.sum())
            if c:
                i = torch.nonzero(sel).flatten()
                want[i, g0[i] if wt == 1.0 else m] = -wt / (c * B)
        sel = g1 == -1
        if int(sel.sum()):
            want[n, torch.nonzero(sel).flatten()] = -0.5 / (int(sel.sum()) * B)
        assert torch.equal(ds[b, :n + 1, :m + 1], want.float()), b
        rest = ds[b].clone()
        rest[:n + 1, :m + 1] = 0
        assert (rest == 0).all() and not torch.isnan(rest).any(), b
    assert float(ds[3].abs().sum()) == 0.0
    ref /= B
    bound = 2 * (N + M + B + 8) * U * terms_abs / B + 2 * U * abs(ref)
    err = abs(float(loss['loss']) - ref)
    _report(f'criterion B={B} {N}x{M}', err, bound)
    assert err <= bound


# ---------------------------------------------------------------------------------------------------------------------
# 5. padded labels above the nearest-neighbour tile
@pytest.mark.parametrize('kind', ['perspective', '3d_keypoint', '3d_image'])
def test_padded_labels_above_the_tile_against_oracle(kind):
    from openglue_b200.gt_matches import IGNORE_INDEX, gt_matches
    from openglue_b200.synthetic import synthetic_gt_scene
    N, M = 4096, 3000                                    # above GT_TILE = 2048
    ns, ms = [2047, 2048, 2049, 2500, N], [3000, 2049, 2048, 2047, 2500]
    B = len(ns)
    sc = synthetic_gt_scene(B, N, M, 'perspective' if kind == 'perspective' else '3d_reprojection', seed=55, depth_image=kind == '3d_image')
    k0, k1, tf = sc['keypoints0'], sc['keypoints1'], sc['transformation']
    kp0, kp1 = k0.clone(), k1.clone()
    for b, (n, m) in enumerate(zip(ns, ms)):
        kp0[b, n:], kp1[b, m:] = float('nan'), float('nan')
    tfd = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in tf.items()}
    if kind == '3d_keypoint':
        for i, L_ in ((0, ns), (1, ms)):
            d = tf[f'depth{i}'].clone()
            for b, n in enumerate(L_):
                d[b, n:] = float('nan')
            tfd[f'depth{i}'] = d.to(DEV)
    lens = torch.tensor(ns + ms, dtype=torch.int32, device=DEV)
    g0, g1 = gt_matches(kp0.to(DEV), kp1.to(DEV), tfd, lens)
    g0, g1 = g0.cpu(), g1.cpu()
    for b, (n, m) in enumerate(zip(ns, ms)):
        tb = {k: (v[b:b + 1] if torch.is_tensor(v) else v[:1]) for k, v in tf.items()}
        if kind == '3d_keypoint':
            tb['depth0'], tb['depth1'] = tf['depth0'][b:b + 1, :n], tf['depth1'][b:b + 1, :m]
        scene = {'keypoints0': k0[b:b + 1, :n], 'keypoints1': k1[b:b + 1, :m], 'transformation': tb}
        w0, w1, _ = GO.gt_matches(scene['keypoints0'], scene['keypoints1'], tb)
        c0, c1 = _checkable(scene)
        assert c0.float().mean() >= 0.9 and c1.float().mean() >= 0.9, (b, 'too many near-tie rows')
        assert torch.equal(g0[b:b + 1, :n][c0], w0[c0]), (b, int((g0[b:b + 1, :n][c0] != w0[c0]).sum()))
        assert torch.equal(g1[b:b + 1, :m][c1], w1[c1]), (b, int((g1[b:b + 1, :m][c1] != w1[c1]).sum()))
        assert (g0[b, n:] == IGNORE_INDEX).all() and (g1[b, m:] == IGNORE_INDEX).all(), b
        print(f'\n[labels {kind} pair {n}x{m}] {int(c0.sum())}/{n} and {int(c1.sum())}/{m} rows checked exactly, '
              f'{int((w0 >= 0).sum())} matches')


# ---------------------------------------------------------------------------------------------------------------------
# 6. keypoint-encoder input and row mask
@pytest.mark.parametrize('side_info_size', [0, 1])
def test_kenc_input_and_row_mask_are_exact(side_info_size):
    lib = _lib()
    B, cap, S = 16, 2048, side_info_size
    g = torch.Generator().manual_seed(66 + S)
    lens = torch.randint(1, cap + 1, (B,), generator=g)
    lens[:3] = torch.tensor([1, cap - 1, cap])
    wh = torch.stack([torch.randint(2, 2000, (B,), generator=g), torch.randint(2, 2000, (B,), generator=g)], 1).float()
    wh[0] = torch.tensor([2.0, 2.0])
    pair_wh = torch.zeros(B, 4)
    pair_wh[:, :2] = wh
    kp = torch.rand(B, cap, 2, generator=g) * (wh[:, None] - 1)
    side = torch.rand(B, cap, max(S, 1), generator=g)
    kp_j, side_j = kp.clone(), side.clone()
    for b, n in enumerate(lens.tolist()):
        kp_j[b, n:], side_j[b, n:] = float('nan'), float('nan')
    ld = torch.tensor(lens.tolist(), dtype=torch.int32, device=DEV)
    outs = []
    for k_, s_ in ((kp, side), (kp_j, side_j)):
        out = _nan(B * cap * (2 + S) + 1)
        kd, sd = k_.to(DEV), s_[..., :max(S, 1)].contiguous().to(DEV)
        _cabi.check(lib.og_kenc_input_padded(_p(kd), _p(sd) if S else None, B, cap, _p(ld), S, _p(pair_wh.to(DEV)), _p(out), _st()),
                    'og_kenc_input_padded')
        outs.append(out.cpu())
    got, junk = outs
    assert torch.isnan(got[-1]) and torch.isnan(junk[-1])
    got, junk = got[:-1].view(B, cap, 2 + S), junk[:-1].view(B, cap, 2 + S)
    # torch float32: 2 x / (w - 1) - 1 per coordinate with the pair's own image size
    want = 2 * kp / (wh[:, None] - 1) - 1
    for b, n in enumerate(lens.tolist()):
        assert torch.equal(got[b, :n, :2], want[b, :n]), b
        if S:
            assert torch.equal(got[b, :n, 2:], side[b, :n, :S]), b
        assert (got[b, n:] == 0).all() and not torch.isnan(got[b, n:]).any(), b
    _same_bits(junk, got, 'NaN padding')
    # og_mask_padded_rows: the rows past each length zeroed, the rest copied
    cols = 257
    X = torch.randn(B * cap, cols, generator=g)
    X[::7] = float('nan')
    out = _nan(B * cap, cols)
    _cabi.check(lib.og_mask_padded_rows(_p(X.to(DEV)), B, cap, cols, _p(ld), _p(out), _st()), 'og_mask_padded_rows')
    real = torch.zeros(B * cap, dtype=torch.bool)
    for b, n in enumerate(lens.tolist()):
        real[b * cap:b * cap + n] = True
    want = torch.where(real[:, None], X, torch.zeros(()))
    _same_bits(out.cpu(), want, 'og_mask_padded_rows')


# ---------------------------------------------------------------------------------------------------------------------
# 7. fp16x3 attention with key lengths
def test_f16_attention_key_lengths_against_float64():
    H, dh, nq, nk = 2, 64, 130, 300
    lens = [1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300]            # those of test_attention_key_lengths
    B, d = len(lens), H * dh
    g = torch.Generator(device=DEV).manual_seed(77)
    q, k, v = (1.5 * torch.randn(B, n, d, generator=g, device=DEV) for n in (nq, nk, nk))
    for b, L_ in enumerate(lens):                                         # the padding keys as the path produces them: zero
        k[b, L_:], v[b, L_:] = 0.0, 0.0
    ops = Operands('fp16', dh, H, q, k, v)
    out = ops.new_out()
    out_amax = torch.zeros(1, device=DEV)
    kl = torch.tensor(lens, dtype=torch.int32, device=DEV)
    _cabi.check(_lib().og_attention_f16_fwd_padded(_p(ops.Q), ops.ldq, ops.sq, _p(ops.qamax), _p(ops.khi), _p(ops.klo), ops.ldk, _p(ops.kmeta),
                                                   _p(ops.vthi), _p(ops.vtlo), ops.ldvt, _p(ops.vmeta), _p(out), ops.ldo, ops.so, _p(out_amax), B,
                                                   nq, nk, H, dh, _p(kl), _st()), 'og_attention_f16_fwd_padded')
    torch.cuda.synchronize()
    got = ops.out_view(out).double().cpu()
    assert torch.isfinite(got).all()
    worst = 0.0
    for b, L_ in enumerate(lens):
        ref = _reference(q[b:b + 1, :, :], k[b:b + 1, :L_], v[b:b + 1, :L_], H).cpu()[0]
        bound = CONTRACT['fp16'] * float(ref.abs().max())
        err = float((got[b] - ref).abs().max())
        assert err <= bound, (L_, err, bound)
        worst = max(worst, err / bound)
        if L_ in (1, 128, 129, 300):
            _report(f'fp16x3 attention key length {L_}', err, bound)
    print(f'\n[fp16x3 attention key lengths] worst error / bound {worst:.2f}')
    assert float(out_amax) == float(ops.out_view(out).abs().max())
