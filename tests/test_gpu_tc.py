"""GPU tests of the wgmma (3xTF32) kernels: operator-level vs fp64, and the whole path in
precision='tf32x3' against the reference golden vectors (same 1e-4 bound as the fp32 mode)."""
import ctypes as C

import pytest
import torch

from conftest import GOLDEN_FULL
from openglue_b200 import _cabi
from openglue_b200._cabi import ptr as _p
from openglue_b200.superglue import MatchingCore, SuperGlue

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.mark.parametrize('mode', [2, 0, 1])
@pytest.mark.parametrize('rows,k1,k2,nout,batch,per_batch_b', [(128, 32, 0, 128, 1, False), (1000, 256, 256, 392, 1, False),
                                                              (257, 64, 0, 200, 3, True), (300, 512, 0, 256, 2, False)])
def test_linear_tc_operator(mode, rows, k1, k2, nout, batch, per_batch_b):
    g = torch.Generator().manual_seed(0)
    K = k1 + k2
    A = 3 * torch.randn(batch, rows, k1, generator=g)
    A2 = torch.randn(batch, rows, k2, generator=g) if k2 else None
    W = torch.randn(batch if per_batch_b else 1, nout, K, generator=g)
    bias = torch.randn(nout, generator=g)
    R = torch.randn(batch, rows, nout, generator=g)
    X = torch.cat([A, A2], -1) if k2 else A
    ref = (0.5 * (X.double() @ W.double().transpose(1, 2)) + bias.double()).relu() + R.double()
    lib = _cabi.lib()
    st = _cabi.stream()
    dA, dW, db, dR = A.to(DEV), W.to(DEV), bias.to(DEV), R.to(DEV)
    dA2 = A2.to(DEV) if k2 else None
    Whi, Wlo = torch.empty_like(dW), torch.empty_like(dW)
    _cabi.check(lib.og_split_tf32(_p(dW), _p(Whi), _p(Wlo), dW.numel(), st), 'og_split_tf32')
    Y = torch.full((batch, rows, nout), float('nan'), device=DEV)
    Yhi, Ylo = torch.zeros_like(Y), torch.zeros_like(Y)
    Yt = torch.full((batch, nout, rows), float('nan'), device=DEV)
    Ythi, Ytlo = torch.zeros_like(Yt), torch.zeros_like(Yt)
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.strideA = dA.data_ptr(), k1, rows * k1
    if k2:
        a.A2, a.lda2, a.strideA2 = dA2.data_ptr(), k2, rows * k2
    a.k1, a.k2, a.ldw, a.strideW = k1, k2, K, (nout * K if per_batch_b else 0)
    a.bias = db.data_ptr()
    a.rows, a.nout, a.batch, a.alpha, a.relu = rows, nout, batch, 0.5, 1
    a.R, a.ldr, a.strideR = dR.data_ptr(), nout, rows * nout
    a.Y, a.ldy, a.strideY = Y.data_ptr(), nout, rows * nout
    a.Yt, a.ldyt, a.strideYt = Yt.data_ptr(), rows, nout * rows
    _cabi.check(lib.og_linear_tc_fwd(C.byref(a), _p(Whi), _p(Wlo), _p(Yhi), _p(Ylo), _p(Ythi), _p(Ytlo), mode, st),
                'og_linear_tc_fwd')
    scale = ref.abs().max()
    # mode 2 (chunked accumulation) is as accurate as an fp32 FMA GEMM; modes 0/1 carry the tensor core's
    # truncating accumulator over the whole K (still ~100x better than single-pass tf32)
    assert (Y.cpu().double() - ref).abs().max() <= (1.5e-6 if mode == 2 else 1e-5) * scale
    assert torch.equal(Yt.transpose(1, 2), Y)
    assert (Yhi.double() + Ylo.double() - Y.double()).abs().max() <= 2.0 ** -21 * scale
    assert torch.equal(Ythi.transpose(1, 2), Yhi) and torch.equal(Ytlo.transpose(1, 2), Ylo)


@pytest.mark.parametrize('B,H,dh,nq,nk', [(2, 4, 64, 200, 333), (1, 4, 32, 129, 64), (3, 2, 64, 64, 1), (1, 4, 64, 1000, 2048)])
def test_attention_tc_operator(B, H, dh, nq, nk):
    from oracle import superglue_oracle as O
    g = torch.Generator().manual_seed(2)
    d = H * dh
    q, k, v = (3 * torch.randn(B, n_, d, generator=g) for n_ in (nq, nk, nk))
    to_ref = lambda t: t.transpose(1, 2).reshape(B, H, dh, -1)
    ref = O.softmax_attention(to_ref(q).double(), to_ref(k).double(), to_ref(v).double()).reshape(B, d, nq).transpose(1, 2)
    lib = _cabi.lib()
    st = _cabi.stream()
    dq, dk = q.to(DEV), k.to(DEV)
    ldv = (nk + 3) // 4 * 4
    dvt = torch.zeros(B, d, ldv, device=DEV)
    dvt[:, :, :nk] = v.to(DEV).transpose(1, 2)
    khi, klo, vthi, vtlo = (torch.empty_like(t) for t in (dk, dk, dvt, dvt))
    _cabi.check(lib.og_split_tf32(_p(dk), _p(khi), _p(klo), dk.numel(), st), 'split k')
    _cabi.check(lib.og_split_tf32(_p(dvt), _p(vthi), _p(vtlo), dvt.numel(), st), 'split v')
    out = torch.full((B, nq, d), float('nan'), device=DEV)
    rc = lib.og_attention_tc_fwd(_p(dq), d, nq * d, _p(khi), _p(klo), d, _p(vthi), _p(vtlo), ldv, _p(out), d, nq * d,
                                 B, nq, nk, H, dh, st)
    _cabi.check(rc, 'og_attention_tc_fwd')
    torch.cuda.synchronize()
    assert (out.cpu().double() - ref).abs().max() <= 1e-5 * ref.abs().max()


# ids = the two values of og_set_tuning's switches, named as the C ABI documents them for callers of earlier builds
@pytest.fixture(params=[0, 1], ids=['single_cta', 'cta_pair'])
def kernel_form(request):
    """og_set_tuning is kept in the C ABI for callers of earlier builds: sm_90 has one GEMM and one attention form, so either
    setting must be accepted and must leave the results unchanged (the same kernels run)."""
    _cabi.check(_cabi.lib().og_set_tuning(request.param, request.param), 'og_set_tuning')
    yield request.param
    _cabi.check(_cabi.lib().og_set_tuning(1, 1), 'og_set_tuning')


def test_both_kernel_forms_match_reference(golden, kernel_form):
    """Either setting of the (no-op on sm_90) kernel-form switch is accepted and the results still match the reference."""
    for name in ('small_planted', 'C1_planted'):
        test_forward_tf32x3_matches_reference(golden, name)
    test_attention_tc_operator(2, 4, 64, 200, 333)
    test_attention_tc_operator(1, 4, 32, 129, 64)
    test_linear_tc_operator(2, 1000, 256, 256, 392, 1, False)
    test_linear_tc_operator(2, 300, 512, 0, 256, 2, False)


@pytest.mark.parametrize('name', ['tiny_planted', 'small_planted', 'C1_planted', 'C1_flat'])
def test_forward_tf32x3_matches_reference(golden, name):
    fx = golden(name)
    cfg = dict(fx['config'])
    cfg['precision'] = 'tf32x3'
    model = SuperGlue(cfg).eval()
    model.load_state_dict(fx['state_dict'])
    model = model.to(DEV)
    data = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in fx['data'].items()}
    res = MatchingCore(model, fx['match_threshold'])(data, want_scores=True)
    bound = max(1e-4, 2 * fx['ref32_vs_ref64_max_abs'])
    s = res['scores'].cpu()
    if 'scores_f64' in fx:
        assert (s.double() - fx['scores_f64']).abs().max() <= bound
    else:
        assert (s[:, ::7, ::5].double() - fx['scores_f64_sample']).abs().max() <= bound
    if 'planted' in name:
        assert torch.equal(res['matches0'].cpu(), fx['matches0'])
        assert (res['matching_scores0'].cpu() - fx['matching_scores0']).abs().max() <= 1e-4
