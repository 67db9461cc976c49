"""GPU tests of the fp16 hi/lo ("3xFP16", wgmma with fp16 operands) operators through the C ABI: og_weight_split_f16, og_amax,
og_linear_f16_fwd, og_attention_f16_fwd, against float64 references (the attention one is the oracle's softmax_attention).
Accuracy contract = the tf32x3 kernels': fp32-GEMM grade (a few 1e-7 relative to the largest output)."""
import ctypes as C

import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200._cabi import ptr as _p, stream as _st
from oracle import superglue_oracle as O

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def split16(x2d, bias=None):
    """fp32 [rows, cols] -> (hi16, lo16, meta[4]) on the device through og_weight_split_f16"""
    hi = torch.empty(x2d.shape, dtype=torch.float16, device=DEV)
    lo = torch.empty_like(hi)
    meta = torch.zeros(4, device=DEV)
    _cabi.check(_cabi.lib().og_weight_split_f16(_p(x2d), _p(bias), x2d.shape[0], x2d.shape[1], _p(hi), _p(lo), _p(meta), _st()), 'split16')
    return hi, lo, meta


def amax_of(x):
    slot = torch.zeros(1, device=DEV)
    _cabi.check(_cabi.lib().og_amax(_p(x), x.numel(), _p(slot), _st()), 'og_amax')
    return slot


def test_weight_split_f16_represents_the_tensor():
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(300, 200, generator=g) * torch.logspace(-6, 1, 200)).to(DEV)      # 7 decades of dynamic range
    b = torch.randn(300, generator=g).to(DEV)
    hi, lo, meta = split16(w, b)
    scale, l1, bmax = (float(x) for x in meta[:3].cpu())
    amax = float(w.abs().max())
    assert 2 ** 14 <= amax * scale < 2 ** 15 and scale == 2.0 ** round(torch.log2(torch.tensor(scale)).item())
    assert abs(l1 / float(w.abs().sum(1).max()) - 1) < 1e-3 and abs(bmax - float(b.abs().max())) < 1e-6
    back = (hi.double() + lo.double()) / scale
    err = (back - w.double()).abs()
    assert bool((err <= torch.maximum(w.double().abs() * 2.0 ** -21, torch.tensor(2.0 ** -24 / scale, device=DEV, dtype=torch.float64))).all())
    assert float(amax_of(w)) == amax


def _linear_case(rows, k1, k2, nout, relu, resid, batch, kind, swap=0, seed=1):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(batch, rows, k1, generator=g) * 3
    A2 = torch.randn(batch, rows, k2, generator=g) * 0.5 if k2 else None
    W = torch.randn(nout, k1 + k2, generator=g) / 8
    bias = torch.randn(nout, generator=g)
    R = torch.randn(batch, rows, nout, generator=g) if resid else None
    X = torch.cat([A, A2], -1) if k2 else A
    ref = 0.7 * (X.double() @ W.double().t()) + bias.double()
    if relu:
        ref = ref.relu()
    if resid:
        ref = ref + R.double()
    dA, dW, db = A.to(DEV), W.to(DEV), bias.to(DEV)
    dA2 = A2.to(DEV) if k2 else None
    dR = R.to(DEV) if resid else None
    Wh, Wl, meta = split16(dW, db)
    a_amax = amax_of(torch.cat([dA.flatten(), dA2.flatten()]) if k2 else dA)
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.strideA = dA.data_ptr(), k1, rows * k1
    if k2:
        a.A2, a.lda2, a.strideA2 = dA2.data_ptr(), k2, rows * k2
    a.k1, a.k2, a.ldw, a.strideW = k1, k2, k1 + k2, 0
    a.bias = db.data_ptr()
    a.rows, a.nout, a.batch, a.alpha, a.relu = rows, nout, batch, 0.7, int(relu)
    if resid:
        a.R, a.ldr, a.strideR = dR.data_ptr(), nout, rows * nout
    lib = _cabi.lib()
    amax_out, scale_out = torch.zeros(1, device=DEV), torch.zeros(1, device=DEV)
    scale_ref = float(ref.abs().max())
    if kind == 'y':
        Y = torch.full((batch, rows, nout), float('nan'), device=DEV)
        a.Y, a.ldy, a.strideY = Y.data_ptr(), nout, rows * nout
        _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(a_amax), _p(amax_out), None, None, None, None, None, swap, _st()), 'linear_f16')
        err = float((Y.cpu().double() - ref).abs().max()) / scale_ref
        return err, float(amax_out), float(Y.abs().max())
    if kind == 'split':
        ldy = (nout + 7) // 8 * 8
        Yh = torch.zeros(batch, rows, ldy, dtype=torch.float16, device=DEV)
        Yl = torch.zeros_like(Yh)
        a.ldy, a.strideY = ldy, rows * ldy
        _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(a_amax), None, _p(scale_out), _p(Yh), _p(Yl), None, None, swap, _st()), 'linear_f16')
        sc = float(scale_out)
        back = (Yh[:, :, :nout].double() + Yl[:, :, :nout].double()).cpu() / sc
        return float((back - ref).abs().max()) / scale_ref, sc, float(Yh.float().abs().max())
    ldyt = (rows + 7) // 8 * 8
    Yth = torch.zeros(batch, nout, ldyt, dtype=torch.float16, device=DEV)
    Ytl = torch.zeros_like(Yth)
    a.ldyt, a.strideYt = ldyt, nout * ldyt
    _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(Wh), _p(Wl), _p(meta), _p(a_amax), None, _p(scale_out), None, None, _p(Yth), _p(Ytl), swap, _st()), 'linear_f16')
    sc = float(scale_out)
    back = (Yth[:, :, :rows].double() + Ytl[:, :, :rows].double()).cpu().transpose(1, 2) / sc
    return float((back - ref).abs().max()) / scale_ref, sc, float(Yth.float().abs().max())


def test_f16_tmem_operand_layout_probe():
    """Which half of a packed 32-bit A-operand register is K element 2c?  The production packing (swap = 0: low half) must be the right one.
    (The name is kept from the earlier form of the kernels, which held this operand in tensor memory.)"""
    e0, _, _ = _linear_case(128, 64, 0, 128, False, False, 1, 'y', swap=0)
    e1, _, _ = _linear_case(128, 64, 0, 128, False, False, 1, 'y', swap=1)
    print(f'\n[f16 register A-operand layout] rel. error with element 2c in the LOW half: {e0:.2e}, in the HIGH half: {e1:.2e}')
    assert e0 < 2e-6 < e1


@pytest.mark.parametrize('rows,k1,k2,nout,relu,resid,batch', [
    (128, 64, 0, 128, False, False, 1), (128, 256, 0, 128, False, False, 1), (300, 256, 0, 200, True, False, 1),
    (513, 256, 256, 512, True, False, 1), (130, 512, 0, 256, False, True, 1), (257, 64, 0, 128, False, False, 3),
    (1000, 320, 0, 392, False, False, 1), (200, 96, 0, 72, True, False, 2)])
def test_linear_f16_fp32_output(rows, k1, k2, nout, relu, resid, batch):
    err, amax_out, ymax = _linear_case(rows, k1, k2, nout, relu, resid, batch, 'y')
    print(f'\n[linear_f16 {rows}x{k1}+{k2}->{nout} b{batch}] rel err {err:.2e}')
    assert err <= 2e-6
    assert amax_out == ymax                                   # tracked amax = the true maximum of the output


@pytest.mark.parametrize('kind', ['split', 'tsplit'])
@pytest.mark.parametrize('rows,k1,nout,batch', [(128, 64, 128, 1), (300, 256, 256, 2), (2048, 256, 256, 2), (77, 128, 64, 3)])
def test_linear_f16_split_outputs(kind, rows, k1, nout, batch):
    err, sc, hmax = _linear_case(rows, k1, 0, nout, False, False, batch, kind)
    print(f'\n[linear_f16 {kind} {rows}x{k1}->{nout} b{batch}] rel err {err:.2e}, scale 2^{torch.log2(torch.tensor(sc)).item():.0f}, max|hi| {hmax:.0f}')
    assert err <= 2e-6
    assert 0 < hmax < 2 ** 15                                 # the bound-derived scale keeps the halves in range


@pytest.mark.parametrize('pair', [1, 0])                 # og_set_tuning(-1, pair): accepted, no effect on sm_90 (one kernel form)
@pytest.mark.parametrize('B,H,nq,nk', [(2, 4, 200, 333), (1, 4, 128, 64), (1, 2, 65, 1), (3, 4, 512, 2048), (1, 4, 300, 130)])
def test_attention_f16_operator(B, H, nq, nk, pair):
    dh = 64
    g = torch.Generator().manual_seed(2)
    d = H * dh
    q, k, v = (3 * torch.randn(B, n_, d, generator=g) for n_ in (nq, nk, nk))
    to_ref = lambda t: t.transpose(1, 2).reshape(B, H, dh, -1)
    ref = O.softmax_attention(to_ref(q).double(), to_ref(k).double(), to_ref(v).double()).reshape(B, d, nq).transpose(1, 2)
    dq = q.to(DEV)
    kh, kl, kmeta = split16(k.reshape(B * nk, d).to(DEV))
    ldvt = (nk + 7) // 8 * 8
    vt = torch.zeros(B * d, ldvt, device=DEV)
    vt[:, :nk] = v.transpose(1, 2).reshape(B * d, nk).to(DEV)
    vth, vtl, vmeta = split16(vt)
    out = torch.full((B, nq, d), float('nan'), device=DEV)
    oamax = torch.zeros(1, device=DEV)
    lib = _cabi.lib()
    lib.og_set_tuning(-1, pair)
    try:
        rc = lib.og_attention_f16_fwd(_p(dq), d, nq * d, _p(amax_of(dq)), _p(kh), _p(kl), d, _p(kmeta), _p(vth), _p(vtl), ldvt, _p(vmeta),
                                      _p(out), d, nq * d, _p(oamax), B, nq, nk, H, dh, 0, _st())
        _cabi.check(rc, 'og_attention_f16_fwd')
        torch.cuda.synchronize()
    finally:
        lib.og_set_tuning(-1, 1)
    err = float((out.cpu().double() - ref).abs().max() / ref.abs().max())
    print(f'\n[attention_f16 B{B} H{H} {nq}x{nk} pair={pair}] rel err {err:.2e}')
    assert err <= 5e-6
    assert float(oamax) == float(out.abs().max())


@pytest.mark.parametrize('B,H,nq,nk,pair', [
    (10, 4, 1024, 1216, 1),      # 320 CTAs, 19 key blocks each: the stage ring wraps several times, a partial last block
    (12, 4, 1000, 1100, 1),      # 384 CTAs, 18 key blocks, ragged query rows and keys
    (6, 4, 700, 64, 1),          # one key block per CTA: the ring is never refilled
    (5, 4, 1024, 1216, 0)])      # og_set_tuning(-1, 0): accepted, no effect on sm_90 (one kernel form)
def test_attention_f16_many_tiles(B, H, nq, nk, pair):
    """Many CTAs and long key loops of the fp16 attention kernel: the mbarrier phases of the K / V stage ring across many
    refills, partial key blocks and ragged query tiles.  Reference: plain torch float64 on the device (the same arithmetic as
    oracle.softmax_attention)."""
    dh = 64
    g = torch.Generator(device=DEV).manual_seed(2)
    d = H * dh
    q, k, v = (3 * torch.randn(B, n_, d, generator=g, device=DEV) for n_ in (nq, nk, nk))
    hv = lambda t, n: t.double().reshape(B, n, H, dh).permute(0, 2, 1, 3)
    ref = (torch.softmax(hv(q, nq) @ hv(k, nk).transpose(2, 3) / dh ** 0.5, dim=-1) @ hv(v, nk)).permute(0, 2, 1, 3).reshape(B, nq, d)
    kh, kl, kmeta = split16(k.reshape(B * nk, d))
    ldvt = (nk + 7) // 8 * 8
    vt = torch.zeros(B * d, ldvt, device=DEV)
    vt[:, :nk] = v.transpose(1, 2).reshape(B * d, nk)
    vth, vtl, vmeta = split16(vt)
    out = torch.full((B, nq, d), float('nan'), device=DEV)
    oamax = torch.zeros(1, device=DEV)
    lib = _cabi.lib()
    lib.og_set_tuning(-1, pair)
    try:
        for _ in range(2):                           # the second launch reuses nothing: barriers are per launch
            rc = lib.og_attention_f16_fwd(_p(q), d, nq * d, _p(amax_of(q)), _p(kh), _p(kl), d, _p(kmeta), _p(vth), _p(vtl), ldvt, _p(vmeta),
                                          _p(out), d, nq * d, _p(oamax), B, nq, nk, H, dh, 0, _st())
            _cabi.check(rc, 'og_attention_f16_fwd')
        torch.cuda.synchronize()
    finally:
        lib.og_set_tuning(-1, 1)
    err = float((out.double() - ref).abs().max() / ref.abs().max())
    print(f'\n[attention_f16 many tiles B{B} H{H} {nq}x{nk} pair={pair}] rel err {err:.2e}')
    assert err <= 5e-6
    assert float(oamax) == float(out.abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize('batch,n,m', [(2, 330, 197), (1, 256, 256), (3, 64, 1)])
def test_fused_projections_are_bit_identical(batch, n, m):
    """One launch over the stacked Q | K | V (self) or K | V (cross) weights (linear_sm90.cuh, F16LinearArgs::nkinds) computes the same tiles with the
    same arithmetic as one launch per projection: the whole path's outputs must not change by a single bit."""
    import torch
    from openglue_b200 import SuperGlue, _cabi
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
    dev = torch.device('cuda:0')
    cfg = default_config(descriptor_dim=256, num_stages=2, num_iters=10)
    cfg['precision'] = 'fp16x3'
    model = SuperGlue(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=8), strict=True)
    model = model.to(dev).eval()
    data = synthetic_pairs(batch, n, m, 256, 1, family='planted', seed=31)
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in data.items()}
    lib = _cabi.lib()
    prev = lib.og_set_fusion(1)
    try:
        with torch.no_grad():
            fused = {k: v.clone() for k, v in model(data).items()}
            n_fused = model.last_launches
            lib.og_set_fusion(0)
            plain = {k: v.clone() for k, v in model(data).items()}
            n_plain = model.last_launches
    finally:
        lib.og_set_fusion(prev)
    for k in fused:
        assert torch.equal(fused[k], plain[k]), k
    stages = cfg['attention_gnn']['num_stages']
    same = 2 if n != m else 1                                  # self layers: one launch per image when n != m
    assert n_plain - n_fused == stages * (2 * same + 2 * 1)     # self: Q,K,V -> 1 (2 saved per call); cross: K,V -> 1 (1 saved per call, 2 calls)
