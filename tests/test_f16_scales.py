"""The power-of-two scales of the fp16 hi/lo ("3xFP16") operands, tested where they can fail: tensor magnitudes far from 1,
one operand skewed against another, a bias that dominates the output, |alpha| < 1, all-zero inputs, and whole-path weights
and inputs of the kind trained models and unnormalised features produce.

Every fp16 operand carries a scale from tc::f16_scale_for (csrc/tc_common.cuh) that puts a BOUND on its magnitudes into
[2^14, 2^15): the tracked amax of an fp32 tensor, or, for the fp16 K / V^T outputs of a GEMM (written before their maximum is
known), |alpha| amax(A) max_n ||W_n||_1 + max |b|.  A bound that is too low makes hi = fp16(x s) overflow.

References are float64.  Bounds are the operators' contracts (test_gpu_f16.py): 2e-6 of max |ref| for the GEMM, 5e-6 for
attention; where a case is ill-conditioned on purpose, the float32 reference's own distance from float64 (x 4) where that is
larger.  Every case prints its error next to its bound."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200._cabi import ptr as _p, stream as _st
from openglue_b200.superglue import MatchingCore, SuperGlue
from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
from oracle import superglue_oracle as O
from test_gpu_parity import check_matches

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GEMM_BOUND, ATTN_BOUND, TF32_ATTN_BOUND = 2e-6, 5e-6, 1e-5
F16_MAX = 65504.0


def _report(tag, err, bound):
    print(f'\n[{tag}] max error {err:.3e}, bound {bound:.3e} ({err / bound if bound > 0 else 0.0:.2f} of it)')


def _exponent(x):
    """the biased exponent field of float32(x)"""
    return (int(np.array(x, dtype=np.float32).view(np.uint32)) >> 23) & 0xff


def f16_scale_for(bound):
    """tc::f16_scale_for: 2^(14 - e) for the float32 exponent e of `bound`, e clamped to [-40, 60]"""
    return 2.0 ** (14 - (min(max(_exponent(bound), 87), 187) - 127))


def f16_out_scale(alpha, a_amax, w_l1, b_max):
    """the scale of a GEMM's fp16 output: f16_scale_for(fmaf(|alpha| a_amax, w_l1, b_max)), the product |alpha| a_amax rounded
    to float32 as the kernel does (float64 holds the exact product of two floats; only the exponent of the sum matters)"""
    ab = np.float32(abs(np.float32(alpha))) * np.float32(a_amax)
    return f16_scale_for(float(ab) * float(w_l1) + float(b_max))


def _split16(w, bias=None):
    hi = torch.full(w.shape, float('nan'), dtype=torch.float16, device=DEV)
    lo = torch.full_like(hi, float('nan'))
    meta = torch.full((4,), float('nan'), device=DEV)
    _cabi.check(_cabi.lib().og_weight_split_f16(_p(w), _p(bias), w.shape[0], w.shape[1], _p(hi), _p(lo), _p(meta), _st()), 'split16')
    return hi, lo, meta


def _amax(x):
    slot = torch.full((1,), float('nan'), device=DEV)                 # og_amax resets the slot itself
    _cabi.check(_cabi.lib().og_amax(_p(x), x.numel(), _p(slot), _st()), 'og_amax')
    return slot


def _bits(x):
    return int(torch.as_tensor(x, dtype=torch.float32).reshape(()).cpu().view(torch.int32))


# --------------------------------------------------------------------------------------------------------------------- a. scale rule
def test_weight_scale_follows_the_rule_across_the_clamp_range():
    """meta[0] of og_weight_split_f16 = f16_scale_for(amax) for amax at and one ulp below 2^k, k in [-45, 65] (past both clamp ends,
    2^-40 and 2^60); inside the clamp range hi / lo are finite and represent x s to max(2^-22 |x s|, 2^-25)."""
    g = torch.Generator(device=DEV).manual_seed(11)
    base = torch.rand(48, 80, generator=g, device=DEV) * 2 - 1                  # |base| < 1
    bad = []
    for k in range(-45, 66):
        top = 2.0 ** k
        for amax in (top, float(np.nextafter(np.float32(top), np.float32(0)))):
            w = base * amax
            w[7, 13] = -amax                                                  # the maximum is a negative element
            hi, lo, meta = _split16(w)
            scale = float(meta[0])
            want = f16_scale_for(amax)
            if scale != want:
                bad.append(f'amax {amax:.9g}: scale {scale!r}, rule {want!r}')
            if 87 <= _exponent(amax) <= 187:                                  # 2^-40 <= amax < 2^61: the scale is not clamped
                xs = w.double() * scale
                pair = hi.double() + lo.double()
                tol = torch.clamp(xs.abs() * 2.0 ** -22, min=2.0 ** -25)
                ok = bool(torch.isfinite(pair).all()) and bool(((pair - xs).abs() <= tol).all())
                if not ok:
                    bad.append(f'amax {amax:.9g}: hi/lo do not represent x s (max |hi| {float(hi.float().abs().max())})')
    hi, lo, meta = _split16(torch.zeros(16, 64, device=DEV))
    print(f'\n[weight split scale] 222 magnitudes 2^-45 .. 2^65: {len(bad)} off the rule; all-zero tensor: scale {float(meta[0])!r}')
    assert float(meta[0]) == 2.0 ** 54 and not bool(hi.float().abs().max()) and not bool(lo.float().abs().max())
    assert not bad, '\n'.join(bad)


def test_amax_is_exact():
    """og_amax = max |x| bit for bit: a negative maximum, -0.0, float32 subnormals, a single element, and a tensor long enough that
    the grid is capped at 1184 blocks and every thread strides several times."""
    g = torch.Generator(device=DEV).manual_seed(12)
    cases = {}
    x = torch.randn(10000, generator=g, device=DEV)
    x[4321] = -17.25
    cases['negative maximum'] = (x, 17.25)
    cases['-0.0 everywhere'] = (torch.full((3000,), -0.0, device=DEV), 0.0)
    sub = torch.arange(1, 4097, dtype=torch.float64, device=DEV) * 2.0 ** -149     # k * 2^-149: every one a float32 subnormal
    sub = (sub * torch.where(torch.rand(4096, generator=g, device=DEV) < 0.5, -1.0, 1.0)).float()[torch.randperm(4096, generator=g, device=DEV)]
    cases['subnormals'] = (sub, 4096 * 2.0 ** -149)
    cases['n = 1'] = (torch.tensor([-3.0e-30], device=DEV), 3.0e-30)
    n = 1184 * 2048 * 2 + 12345                                               # grid capped at 1184 x 256 threads: 16 strides each
    big = torch.randn(n, generator=g, device=DEV)
    for pos in (0, 777777, n - 1):
        y = big.clone()
        y[pos] = -1000.5
        cases[f'n = {n}, maximum at {pos}'] = (y, 1000.5)
    for name, (x, want) in cases.items():
        got = _amax(x)
        ref = float(x.abs().max())
        print(f'\n[og_amax {name}] {float(got)!r} (max |x| {ref!r})')
        assert _bits(got) == _bits(torch.tensor(want, dtype=torch.float32)) == _bits(torch.tensor(ref)), name


# --------------------------------------------------------------------------------------------------------------------- b. fp16 GEMM
def _gemm_f16(A, A2, W, bias, alpha, kind, relu=False, R=None, Y=None):
    """og_linear_f16_fwd with one output kind, into NaN-poisoned buffers: 'y' (fp32 Y, optional residual R; Y may be R), 'k'
    (row-major hi / lo) or 'vt' (transposed hi / lo).  A, A2: [batch, rows, k]; W [nout, K] split with its bias, as the forward
    packs it.  Returns the decoded output [batch, rows, nout] (float64), the raw outputs, the published scale (split kinds) or the
    tracked amax (fp32 kind), the input amax slot and the weight meta."""
    batch, rows, k1 = A.shape
    k2 = A2.shape[2] if A2 is not None else 0
    nout = W.shape[0]
    Wh, Wl, meta = _split16(W, bias)
    a_amax = _amax(torch.cat([A.flatten(), A2.flatten()]) if k2 else A)
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.strideA = A.data_ptr(), k1, rows * k1
    if k2:
        a.A2, a.lda2, a.strideA2 = A2.data_ptr(), k2, rows * k2
    a.k1, a.k2, a.ldw, a.strideW = k1, k2, k1 + k2, 0
    a.bias = bias.data_ptr() if bias is not None else None
    a.rows, a.nout, a.batch, a.alpha, a.relu = rows, nout, batch, alpha, int(relu)
    lib = _cabi.lib()
    amax_out, scale_out = torch.zeros(1, device=DEV), torch.full((1,), float('nan'), device=DEV)
    if kind == 'y':
        if Y is None:
            Y = torch.full((batch, rows, nout), float('nan'), device=DEV)
        a.Y, a.ldy, a.strideY = Y.data_ptr(), nout, rows * nout
        if R is not None:
            a.R, a.ldr, a.strideR = R.data_ptr(), nout, rows * nout
        _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(a_amax), _p(amax_out), None, None, None, None, None, 0, _st()), 'linear_f16')
        return Y.double(), (Y,), float(amax_out), float(a_amax), meta.cpu()
    if kind == 'k':
        hi = torch.full((batch, rows, nout), float('nan'), dtype=torch.float16, device=DEV)
        lo = torch.full_like(hi, float('nan'))
        a.ldy, a.strideY = nout, rows * nout
        _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(a_amax), None, _p(scale_out), _p(hi), _p(lo), None, None, 0, _st()), 'linear_f16')
        sc = float(scale_out)
        return (hi.double() + lo.double()) / sc, (hi, lo), sc, float(a_amax), meta.cpu()
    hi = torch.full((batch, nout, rows), float('nan'), dtype=torch.float16, device=DEV)
    lo = torch.full_like(hi, float('nan'))
    a.ldyt, a.strideYt = rows, nout * rows
    _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(a_amax), None, _p(scale_out), None, None, _p(hi), _p(lo), 0, _st()), 'linear_f16')
    sc = float(scale_out)
    return ((hi.double() + lo.double()) / sc).transpose(1, 2), (hi, lo), sc, float(a_amax), meta.cpu()


def _gemm_check(tag, kind, alpha, ref, res, fails):
    """finite outputs, max |hi| <= 65504, the published scale = the rule, the decoded output within the contract.  A split
    output resolves x s to 2^-25 (tc_common.cuh), which limits its absolute precision to 2^-25 / s where the scale is clamped
    (output bounds below 2^-40): the bound is never below 2^-24 / s."""
    out, raw, sc, a_amax, meta = res
    scale_ref = float(ref.abs().max())
    finite = all(bool(torch.isfinite(t).all()) for t in raw)
    bound = GEMM_BOUND * scale_ref
    msg = []
    if kind != 'y':
        hmax = float(raw[0].float().abs().max())
        want = f16_out_scale(alpha, a_amax, float(meta[1]), float(meta[2]))
        bound = max(bound, 2.0 ** -24 / sc)
        if not hmax <= F16_MAX:
            msg.append(f'max |hi| {hmax}')
        if sc != want:
            msg.append(f'scale 2^{np.log2(sc):.0f}, rule 2^{np.log2(want):.0f}')
    err = float((out - ref).abs().max()) if finite else float('nan')
    if not finite:
        msg.append('non-finite ' + ('Y' if kind == 'y' else 'halves'))
    elif not err <= bound:
        msg.append('error above bound')
    _report(tag + (' FAIL: ' + ', '.join(msg) if msg else ''), err, bound)
    if msg:
        fails.append(f'{tag}: {", ".join(msg)} (error {err:.3e}, bound {bound:.3e})')


GEMM_EXPS = (-30, -10, 0, 10, 30)
ALPHAS = (1.0, 0.7, 0.25, 0.0625, -0.5)
BIAS_LEVELS = {'no bias': 0.0, 'bias ~ product': 1.0, 'bias 1024 x product': 1024.0}


@pytest.mark.parametrize('bias_level', list(BIAS_LEVELS))
@pytest.mark.parametrize('alpha', ALPHAS)
@pytest.mark.parametrize('kind', ['y', 'k', 'vt'])
def test_gemm_f16_across_magnitudes(kind, alpha, bias_level):
    """A = 2^kA randn, W = 2^kW randn / 8 over kA, kW in {-30, -10, 0, 10, 30}; bias absent, of the product's size, or dominant.
    Split outputs whose bound passes 2^60 (the top of the scale clamp: kA = kW = 30) are out of range by design and skipped."""
    rows, K, nout = 200, 256, 192
    g = torch.Generator(device=DEV).manual_seed(21)
    A0 = torch.randn(1, rows, K, generator=g, device=DEV)
    W0 = torch.randn(nout, K, generator=g, device=DEV) / 8
    b0 = torch.randn(nout, generator=g, device=DEV)
    fails, skipped = [], 0
    for ka in GEMM_EXPS:
        for kw in GEMM_EXPS:
            A, W = A0 * 2.0 ** ka, W0 * 2.0 ** kw                            # powers of two: exact
            prod = alpha * (A.double() @ W.double().t())
            bias = (BIAS_LEVELS[bias_level] * float(prod.abs().max()) * b0).float() if BIAS_LEVELS[bias_level] else None
            ref = prod + bias.double() if bias is not None else prod
            tag = f'f16 gemm {kind} alpha={alpha} A 2^{ka} W 2^{kw} {bias_level}'
            if kind != 'y':
                l1 = float(W.double().abs().sum(1).max())
                bmax = float(bias.abs().max()) if bias is not None else 0.0
                if abs(alpha) * float(A.abs().max()) * l1 + bmax >= 2.0 ** 60:
                    skipped += 1
                    continue
            res = _gemm_f16(A, None, W, bias, alpha, kind)
            _gemm_check(tag, kind, alpha, ref, res, fails)
            if kind == 'y':                                                 # tracked amax = the true maximum of the output
                if res[2] != float(res[1][0].abs().max()):
                    fails.append(f'{tag}: amax_out {res[2]} != max |Y| {float(res[1][0].abs().max())}')
    print(f'\n[f16 gemm {kind} alpha={alpha} {bias_level}] {len(fails)} failing, {skipped} skipped (bound >= 2^60)')
    assert not fails, '\n'.join(fails)


@pytest.mark.parametrize('alpha', [1.0, 0.25])
@pytest.mark.parametrize('kind', ['y', 'k', 'vt'])
def test_gemm_f16_concatenated_operand_skewed(kind, alpha):
    """fc1's form Y = relu(alpha [A | A2] . W^T + b): A2 2^20 and 2^-20 times A.  One amax slot bounds both operands."""
    rows, k1, k2, nout = 200, 128, 128, 256
    g = torch.Generator(device=DEV).manual_seed(22)
    A = 3 * torch.randn(1, rows, k1, generator=g, device=DEV)
    A20 = torch.randn(1, rows, k2, generator=g, device=DEV)
    W = torch.randn(nout, k1 + k2, generator=g, device=DEV) / 8
    b0 = torch.randn(nout, generator=g, device=DEV)
    relu = kind == 'y'
    fails = []
    for skew in (20, -20):
        A2 = A20 * 2.0 ** skew
        prod = alpha * (torch.cat([A, A2], -1).double() @ W.double().t())
        for level, c in BIAS_LEVELS.items():
            bias = (c * float(prod.abs().max()) * b0).float() if c else None
            ref = prod + bias.double() if bias is not None else prod
            ref = ref.relu() if relu else ref
            res = _gemm_f16(A, A2, W, bias, alpha, kind, relu=relu)
            _gemm_check(f'f16 gemm {kind} [A | 2^{skew} A2] alpha={alpha} {level}', kind, alpha, ref, res, fails)
    assert not fails, '\n'.join(fails)


@pytest.mark.parametrize('kind', ['y', 'k', 'vt'])
def test_gemm_f16_all_zero_input(kind):
    """A = 0: the amax slot stays 0 and the operand scale clamps (2^54); the output is the bias, exactly in fp32."""
    rows, K, nout = 130, 128, 128
    g = torch.Generator(device=DEV).manual_seed(23)
    A = torch.zeros(1, rows, K, device=DEV)
    W = torch.randn(nout, K, generator=g, device=DEV)
    fails = []
    for alpha in (1.0, 0.25):
        for bias in (None, 5 * torch.randn(nout, generator=g, device=DEV)):
            ref = (bias.double() if bias is not None else torch.zeros(nout, dtype=torch.float64, device=DEV)).expand(1, rows, nout)
            res = _gemm_f16(A, None, W, bias, alpha, kind)
            tag = f'f16 gemm {kind} A = 0 alpha={alpha} {"bias" if bias is not None else "no bias"}'
            assert res[3] == 0.0, tag                                          # the amax slot
            if kind == 'y':
                Y = res[1][0]
                assert torch.equal(Y, ref.float()), tag
                assert res[2] == float(ref.abs().max()), tag                    # amax_out = max |b|
                print(f'\n[{tag}] Y == bias exactly')
            else:
                _gemm_check(tag, kind, alpha, ref, res, fails)
                if bias is None:
                    assert res[2] == 2.0 ** 54 and not bool(res[1][0].float().abs().max()), tag
    assert not fails, '\n'.join(fails)


@pytest.mark.parametrize('alpha', [1.0, 0.25])
def test_gemm_f16_in_place_residual_skewed(alpha):
    """fc2's form Y += alpha A . W^T + b in place (R = Y), the residual 2^20 and 2^-20 times the product; amax_out = max |Y|."""
    batch, rows, K, nout = 2, 200, 512, 256
    g = torch.Generator(device=DEV).manual_seed(24)
    A = torch.randn(batch, rows, K, generator=g, device=DEV)
    W = torch.randn(nout, K, generator=g, device=DEV) / 16
    bias = torch.randn(nout, generator=g, device=DEV) / 4
    R0 = torch.randn(batch, rows, nout, generator=g, device=DEV)
    prod = alpha * (A.double() @ W.double().t()) + bias.double()
    fails = []
    for skew in (20, 0, -20):
        R = R0 * (2.0 ** skew * float(prod.abs().max()))
        ref = prod + R.double()
        Y = R.clone()
        res = _gemm_f16(A, None, W, bias, alpha, 'y', R=Y, Y=Y)
        _gemm_check(f'f16 gemm y += residual 2^{skew} x product alpha={alpha}', 'y', alpha, ref, res, fails)
        if res[2] != float(Y.abs().max()):
            fails.append(f'residual 2^{skew}: amax_out {res[2]} != max |Y| {float(Y.abs().max())}')
    assert not fails, '\n'.join(fails)


# --------------------------------------------------------------------------------------------------------------------- c. attention
ATT_B, ATT_NQ, ATT_NK, ATT_D = 2, 200, 333, 256                 # 333 keys: a partial last key block in both forms
LDVT = (ATT_NK + 7) // 8 * 8


def _orthogonal(d, g):
    q, r = torch.linalg.qr(torch.randn(d, d, generator=g, device=DEV, dtype=torch.float64))
    return (q * torch.sign(torch.diagonal(r))).float().contiguous()          # (QR returns Q column-major)


def _attention_inputs(case, g):
    """Q [B, nq, d] and the K / V projections' inputs: K = Xk Wk^T + bk, V = Xv Wv^T + bv with orthogonal Wk, Wv, so that the
    designed K, V come out of the projection GEMMs (whose fp16 forms write them with scales from the GEMM's bound)."""
    B, nq, nk, d = ATT_B, ATT_NQ, ATT_NK, ATT_D
    r = lambda *s: torch.randn(*s, generator=g, device=DEV)
    q, k, v, bk, bv = r(B, nq, d), r(B, nk, d), 3 * r(B, nk, d), r(d), r(d)
    pick = lambda keys: k.gather(1, keys[..., None].expand(-1, -1, d))
    if case == 'Q x 2^10':
        q = q * 2.0 ** 10
    elif case == 'Q x 2^-10':
        q = q * 2.0 ** -10
    elif case == 'K bias-dominated':                              # a shared offset (cancels in the softmax) + small per-key part
        bk = 64 * r(d)
        k = bk + 2.0 ** -6 * r(B, nk, d)
        q = 8 * q
    elif case == 'near one-hot rows':
        q = 1.5 * pick(torch.randint(0, nk, (B, nq), generator=g, device=DEV)) + 0.1 * r(B, nq, d)
    elif case == 'row maxima in the last partial block':          # keys 320 .. 332: the last block of 128 (fp16) and of 64 (tf32)
        q = 1.5 * pick(torch.randint(320, nk, (B, nq), generator=g, device=DEV)) + 0.1 * r(B, nq, d)
    elif case == 'logits rising block by block':                  # every key block raises the running maximum
        k = 0.3 * k + (4.0 * torch.arange(nk, device=DEV) / nk)[None, :, None]
        q = 0.5 + 0.1 * q
    elif case == 'Q all zero':                                    # uniform weights: the mean of V
        q = torch.zeros_like(q)
    Wk, Wv = _orthogonal(d, g), _orthogonal(d, g)
    Xk, Xv = (k - bk) @ Wk, (v - bv) @ Wv
    return q.contiguous(), Xk.contiguous(), Wk, bk, Xv.contiguous(), Wv, bv


def _attention_reference(q, Xk, Wk, bk, Xv, Wv, bv, H, dtype):
    """projections and attention in `dtype` on the CPU (float32: the reference's own rounding, for the ill-conditioned bound)"""
    B, nq, d = q.shape
    nk, dh = Xk.shape[1], d // H
    c = lambda t: t.cpu().to(dtype)
    k = c(Xk) @ c(Wk).t() + c(bk)
    v = c(Xv) @ c(Wv).t() + c(bv)
    hv = lambda t, n: c(t).reshape(B, n, H, dh).permute(0, 2, 1, 3)
    o = torch.softmax(hv(q, nq) @ hv(k, nk).transpose(2, 3) / dh ** 0.5, dim=-1) @ hv(v, nk)
    return o.permute(0, 2, 1, 3).reshape(B, nq, d).double()


def _projection_args(X, W, bias):
    B, n, d = X.shape
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.strideA = X.data_ptr(), d, n * d
    a.k1, a.k2, a.ldw, a.strideW = d, 0, d, 0
    a.bias = bias.data_ptr()
    a.rows, a.nout, a.batch, a.alpha, a.relu = n, W.shape[0], B, 1.0, 0
    return a


def _attention_f16(q, Xk, Wk, bk, Xv, Wv, bv):
    """K (row-major) and V^T (transposed) hi / lo from og_linear_f16_fwd, then og_attention_f16_fwd (head_dim 64)."""
    B, nq, d = q.shape
    nk = Xk.shape[1]
    lib = _cabi.lib()
    kh = torch.full((B * nk, d), float('nan'), dtype=torch.float16, device=DEV)
    kl = torch.full_like(kh, float('nan'))
    vth = torch.full((B * d, LDVT), float('nan'), dtype=torch.float16, device=DEV)   # columns past nk stay NaN: never read
    vtl = torch.full_like(vth, float('nan'))
    ks, vs = torch.full((1,), float('nan'), device=DEV), torch.full((1,), float('nan'), device=DEV)
    for X, W, b, outs, sc in ((Xk, Wk, bk, (kh, kl, None, None), ks), (Xv, Wv, bv, (None, None, vth, vtl), vs)):
        Wh, Wl, meta = _split16(W, b)
        a = _projection_args(X, W, b)
        a.ldy, a.strideY, a.ldyt, a.strideYt = d, nk * d, LDVT, d * LDVT
        _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(_amax(X)), None, _p(sc), *(_p(t) for t in outs), 0, _st()),
                    'linear_f16')
    assert torch.isfinite(kh).all() and torch.isfinite(kl).all()
    assert torch.isfinite(vth[:, :nk]).all() and torch.isfinite(vtl[:, :nk]).all()
    out = torch.full((B, nq, d), float('nan'), device=DEV)
    oamax = torch.zeros(1, device=DEV)
    _cabi.check(lib.og_attention_f16_fwd(_p(q), d, nq * d, _p(_amax(q)), _p(kh), _p(kl), d, _p(ks), _p(vth), _p(vtl), LDVT, _p(vs),
                                         _p(out), d, nq * d, _p(oamax), B, nq, nk, d // 64, 64, 0, _st()), 'og_attention_f16_fwd')
    return out, float(oamax)


def _attention_tf32(q, Xk, Wk, bk, Xv, Wv, bv, H):
    """K and V^T tf32 hi / lo from og_linear_tc_fwd, then og_attention_tc_fwd (head_dim d / H)."""
    B, nq, d = q.shape
    nk = Xk.shape[1]
    lib = _cabi.lib()
    k = torch.full((B * nk, d), float('nan'), device=DEV)
    khi, klo = torch.full_like(k, float('nan')), torch.full_like(k, float('nan'))
    vt = torch.full((B * d, LDVT), float('nan'), device=DEV)
    vthi, vtlo = torch.full_like(vt, float('nan')), torch.full_like(vt, float('nan'))
    for X, W, b, is_v in ((Xk, Wk, bk, False), (Xv, Wv, bv, True)):
        Whi, Wlo = torch.empty_like(W), torch.empty_like(W)
        _cabi.check(lib.og_split_tf32(_p(W), _p(Whi), _p(Wlo), W.numel(), _st()), 'og_split_tf32')
        a = _projection_args(X, W, b)
        if is_v:
            a.Yt, a.ldyt, a.strideYt = vt.data_ptr(), LDVT, d * LDVT
            outs = (None, None, vthi, vtlo)
        else:
            a.Y, a.ldy, a.strideY = k.data_ptr(), d, nk * d
            outs = (khi, klo, None, None)
        _cabi.check(lib.og_linear_tc_fwd(C.byref(a), _p(Whi), _p(Wlo), *(_p(t) for t in outs), 2, _st()), 'og_linear_tc_fwd')
    out = torch.full((B, nq, d), float('nan'), device=DEV)
    _cabi.check(lib.og_attention_tc_fwd(_p(q), d, nq * d, _p(khi), _p(klo), d, _p(vthi), _p(vtlo), LDVT, _p(out), d, nq * d,
                                        B, nq, nk, H, d // H, _st()), 'og_attention_tc_fwd')
    return out


@pytest.mark.parametrize('case', ['Q x 2^10', 'Q x 2^-10', 'K bias-dominated', 'near one-hot rows',
                                  'row maxima in the last partial block', 'logits rising block by block', 'Q all zero'])
def test_attention_f16_scales(case):
    """og_attention_f16_fwd on K / V^T written by the fp16 GEMM, and the same inputs through the tf32 GEMM and og_attention_tc_fwd
    (head_dim 64 and 32): where the fp16 form fails and the tf32 form passes, the fault is in the scaling.  Large logits
    (Q x 2^10, a large shared K offset, sharp or rising rows) make the float32 reference itself deviate from float64 by up to
    100x the contract, so the bound is the contract or 4x that deviation, whichever is larger (for Q x 2^-10 and Q = 0: the
    contract)."""
    g = torch.Generator(device=DEV).manual_seed(31)
    inputs = _attention_inputs(case, g)
    q, Xv, Wv, bv = inputs[0], inputs[4], inputs[5], inputs[6]
    if case == 'Q all zero':                                      # uniform weights (the query scale clamps): the mean of V
        vmean = (Xv.double() @ Wv.double().t() + bv.double()).mean(1, keepdim=True).expand(-1, ATT_NQ, -1).cpu()
        assert (_attention_reference(*inputs, 4, torch.float64) - vmean).abs().max() <= 1e-12 * vmean.abs().max()
    out16, oamax = _attention_f16(*inputs)
    results = {'fp16 dh=64': (out16, 4, ATTN_BOUND),
               'tf32 dh=64': (_attention_tf32(*inputs, 4), 4, TF32_ATTN_BOUND),
               'tf32 dh=32': (_attention_tf32(*inputs, 8), 8, TF32_ATTN_BOUND)}
    torch.cuda.synchronize()
    fails = []
    for form, (out, H, contract) in results.items():
        ref64 = _attention_reference(*inputs, H, torch.float64)
        bound = max(contract * float(ref64.abs().max()),
                    4 * float((_attention_reference(*inputs, H, torch.float32) - ref64).abs().max()))
        finite = bool(torch.isfinite(out).all())
        err = float((out.cpu().double() - ref64).abs().max()) if finite else float('nan')
        _report(f'attention {form} {case}', err, bound)
        if not err <= bound:
            fails.append(f'{form}: error {err:.3e}, bound {bound:.3e}')
    if oamax != float(out16.abs().max()):                         # tracked amax of the fp16 form's output
        fails.append(f'fp16 out_amax {oamax} != max |out| {float(out16.abs().max())}')
    assert not fails, '\n'.join(fails)


# --------------------------------------------------------------------------------------------------------------------- d. whole path
# (name, batch, n, m, stages): state dicts edited the way trained weights or unnormalised features plausibly look
WHOLE_PATH = [('BN running_var ~ 1e-3', 1, 256, 256, 2),
              ('Q / K projections x 8', 2, 200, 131, 2),
              ('projection biases x 64', 1, 256, 256, 3),
              ('descriptors x 30', 1, 300, 300, 2),
              ('descriptors x 1e-3', 1, 300, 300, 2)]
# Ill-conditioned on purpose: scores reach 4e7 (BN) and 3e4 (x 30), and the float32 oracle's own context descriptors are off
# float64 by 3.7e-4 and 3.2e-4 of their maximum, beyond the 1e-4 the well-conditioned cases are held to.
ILL_CONDITIONED = {'BN running_var ~ 1e-3', 'descriptors x 30'}


@functools.lru_cache(maxsize=None)
def _whole_path_case(name, batch, n, m, stages):
    cfg = default_config(descriptor_dim=256, num_stages=stages, num_iters=20)
    sd = synthetic_state_dict(cfg, seed=6)
    g = torch.Generator().manual_seed(7)
    for key in sd:
        if name.startswith('BN') and key.startswith('attention_gnn.') and key.endswith('fc.2.running_var'):
            sd[key] = 1e-3 * (0.5 + torch.rand(sd[key].shape, generator=g))         # folded MLP weights ~30x larger
        elif name.startswith('Q / K') and ('mha.in_proj_q.weight' in key or 'mha.in_proj_k.weight' in key):
            sd[key] = 8 * sd[key]                                                     # sharp attention
        elif name.startswith('projection biases') and '.mha.' in key and key.endswith('.bias'):
            sd[key] = 64 * sd[key]                                                    # |b| up to 4 (default init: 1 / 16)
    data = synthetic_pairs(batch, n, m, 256, 1, family='planted', seed=78)
    if name.startswith('descriptors'):
        s = 30.0 if name.endswith('30') else 1e-3
        for i in (0, 1):
            data[f'local_descriptors{i}'] = data[f'local_descriptors{i}'] * s
    return cfg, sd, data, O.run(sd, cfg, data, 0.2), O.run(sd, cfg, data, 0.2, dtype=torch.float64)


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3', 'fp16x3'])
@pytest.mark.parametrize('name,batch,n,m,stages', WHOLE_PATH)
def test_whole_path_adverse_weights(name, batch, n, m, stages, precision):
    """The forward against the float64 oracle with test_gpu_parity.py::test_forward_matches_oracle's bounds: scores within
    max(1e-4, 2 err(ref32, ref64)), matches on the decisive rows, context descriptors within 1e-4 relative.  The ill-conditioned
    cases take 4 err(ref32, ref64) (the pattern of the operator tests) for the scores and the context descriptors where that is
    larger."""
    cfg, sd, data, ref, ref64 = _whole_path_case(name, batch, n, m, stages)
    k = 4 if name in ILL_CONDITIONED else 2
    cfg = dict(cfg, precision=precision)
    model = SuperGlue(cfg).eval()
    model.load_state_dict(sd, strict=True)
    model = model.to(DEV)
    dev = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in data.items()}
    res = MatchingCore(model, 0.2)(dev, want_scores=True)
    bound = max(1e-4, k * float((ref['scores'].double() - ref64['scores']).abs().max()))
    s = res['scores'].cpu().double()
    assert torch.isfinite(s).all()
    err = float((s - ref64['scores']).abs().max())
    _report(f'whole path {precision} {name} B{batch} {n}x{m} {stages} stages: scores (max |score| {float(ref64["scores"].abs().max()):.1f})', err, bound)
    assert err <= bound
    excluded = check_matches(res, ref, ref64['scores'], bound)
    out = model(dev)
    for i in (0, 1):
        c = out[f'context_descriptors{i}'].cpu().double()
        r = ref64[f'context_descriptors{i}']
        cbound = 1e-4 * max(1.0, float(r.abs().max()))
        if name in ILL_CONDITIONED:
            cbound = max(cbound, 4 * float((ref[f'context_descriptors{i}'].double() - r).abs().max()))
        cerr = float((c - r).abs().max()) if bool(torch.isfinite(c).all()) else float('nan')
        _report(f'whole path {precision} {name}: context descriptors {i}', cerr, cbound)
        assert cerr <= cbound
    print(f'[whole path {precision} {name}] rows excluded from the match check as near-ties: {excluded}')
