"""How operator calls reach their kernels, and the launch count that follows from it.

1. CPU, on the sources: every kernel of the library is enqueued by one helper, og::launch (csrc/common.cuh), which is the only
   place that counts launches; the only other write of the counter is the reset at the start of a forward pass.  The Python
   modules hand tensors and streams to the C ABI only through _cabi.ptr / _cabi.stream.
2. GPU: each operator entry point moves og_last_forward_launches() by exactly the number of kernels it enqueues, and a forward
   pass reports its own launches whatever ran before it.
"""
import ctypes as C
import os
import re

import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200._cabi import ptr, stream

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'openglue_b200')
CSRC = os.path.join(PKG, 'csrc')
DEV = 'cuda:0'


def _sources(directory, suffixes):
    for name in sorted(os.listdir(directory)):
        if name.endswith(suffixes):
            with open(os.path.join(directory, name)) as f:
                yield name, f.read()


def test_kernels_are_launched_only_by_the_helper():
    chevrons = [name for name, text in _sources(CSRC, ('.cu', '.cuh')) if '<<<' in text]
    assert chevrons == []
    ex = [(name, text.count('cudaLaunchKernelEx')) for name, text in _sources(CSRC, ('.cu', '.cuh')) if 'cudaLaunchKernelEx' in text]
    assert ex == [('common.cuh', 1)]


def test_launch_counter_is_written_only_by_the_helper_and_the_forward_reset():
    write = re.compile(r'(\+\+|--)\s*launch_counter\(\)|launch_counter\(\)\s*(\+\+|--|[-+]?=(?!=))')
    writes = [(name, line.strip()) for name, text in _sources(CSRC, ('.cu', '.cuh')) for line in text.splitlines() if write.search(line)]
    assert writes == [('api.cu', 'launch_counter() = 0;'), ('common.cuh', '++launch_counter();')]
    api = dict(_sources(CSRC, ('.cu',)))['api.cu']
    assert api.index('static int forward_impl(') < api.index('launch_counter() = 0;') < api.index('int og_superglue_forward(')


def test_python_passes_tensors_and_streams_through_cabi():
    raw_ptr = re.compile(r'c_void_p\([^)]*data_ptr\(\)')
    offenders = [name for name, text in _sources(PKG, ('.py',))
                 if name != '_cabi.py' and ('.cuda_stream' in text or raw_ptr.search(text))]
    assert offenders == []


def test_ptr_offsets_count_elements():
    t = torch.zeros(8, dtype=torch.float64)
    assert ptr(None) is None
    assert ptr(t).value == t.data_ptr()
    assert ptr(t, 3).value == t.data_ptr() + 3 * 8


def test_check_size_raises_on_a_rejected_query():
    assert _cabi.check_size(_cabi.lib().og_criterion_workspace_bytes(4), 'og_criterion_workspace_bytes') > 0
    with pytest.raises(_cabi.OpenGlueB200Error):
        _cabi.check_size(_cabi.lib().og_criterion_workspace_bytes(0), 'og_criterion_workspace_bytes')


# ---- GPU: launches per operator call ----
def _f32(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(*shape, generator=g).to(DEV)


def _split_tf32():
    x = _f32(1000)
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    return lambda: _cabi.lib().og_split_tf32(ptr(x), ptr(hi), ptr(lo), x.numel(), stream())


def _weight_split_f16():
    w, b = _f32(64, 128), _f32(64)
    hi = torch.empty(64 * 128, dtype=torch.float16, device=DEV)
    lo, meta = torch.empty_like(hi), torch.empty(4, device=DEV)
    return lambda: _cabi.lib().og_weight_split_f16(ptr(w), ptr(b), 64, 128, ptr(hi), ptr(lo), ptr(meta), stream())


def _amax():
    x, slot = _f32(5000), torch.empty(1, device=DEV)
    return lambda: _cabi.lib().og_amax(ptr(x), x.numel(), ptr(slot), stream())


def _match():
    B, n, m = 2, 50, 70
    scores = -3 * _f32(B, n + 1, m + 1)
    wsb = _cabi.check_size(_cabi.lib().og_match_workspace_bytes(B, n, m), 'og_match_workspace_bytes')
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    m0, m1 = torch.empty(B, n, dtype=torch.int64, device=DEV), torch.empty(B, m, dtype=torch.int64, device=DEV)
    s0, s1 = torch.empty(B, n, device=DEV), torch.empty(B, m, device=DEV)
    return lambda: _cabi.lib().og_match_fwd(ptr(scores), B, n, m, 0.2, ptr(m0), ptr(s0), ptr(m1), ptr(s1), ptr(ws), wsb, stream())


def _gt_matches():
    B, n, m = 2, 40, 30
    k0, k1 = 100 * _f32(B, n, 2, seed=1), 100 * _f32(B, m, 2, seed=2)
    H = torch.eye(3).repeat(B, 1, 1).to(DEV)
    tf = _cabi.OgGtTransform()
    tf.type, tf.H = _cabi.OG_GT_PERSPECTIVE, H.data_ptr()
    wsb = _cabi.check_size(_cabi.lib().og_gt_matches_workspace_bytes(B, n, m), 'og_gt_matches_workspace_bytes')
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    gt0, gt1 = torch.empty(B, n, dtype=torch.int64, device=DEV), torch.empty(B, m, dtype=torch.int64, device=DEV)
    return lambda H=H: _cabi.lib().og_gt_matches_fwd(ptr(k0), ptr(k1), B, n, m, C.byref(tf), ptr(gt0), ptr(gt1), ptr(ws), wsb, stream())


def _criterion():
    B, n, m = 2, 20, 30
    scores = -3 * _f32(B, n + 1, m + 1)
    gt0, gt1 = torch.full((B, n), -1, dtype=torch.int64, device=DEV), torch.full((B, m), -1, dtype=torch.int64, device=DEV)
    loss = torch.empty(2, device=DEV)
    wsb = _cabi.check_size(_cabi.lib().og_criterion_workspace_bytes(B), 'og_criterion_workspace_bytes')
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    return lambda: _cabi.lib().og_criterion_fwd(ptr(scores), ptr(gt0), ptr(gt1), B, n, m, ptr(loss), None, 1.0, ptr(ws), wsb, stream())


def _ops(precision=_cabi.OG_PREC_FP32):
    from openglue_b200._ops import _Ops
    return _Ops(torch.device(DEV), precision)


def _sinkhorn(backward):
    B, n, m, T = 1, 40, 60, 5
    ops = _ops()
    Sp, dust = torch.zeros(B, n, 60, device=DEV), torch.ones(1, device=DEV)
    Sp[:] = _f32(B, n, m)
    if not backward:
        return lambda: ops.sinkhorn_fwd(Sp, dust, B, n, m, T, 1.0)
    _, hist = ops.sinkhorn_fwd(Sp, dust, B, n, m, T, 1.0)
    G = _f32(B, n + 1, m + 1)
    return lambda: ops.sinkhorn_bwd(Sp, dust, hist, G, B, n, m, T, 1.0)


def _bn(backward):
    ops, a = _ops(), _f32(300, 64)
    gamma, beta, rm, rv = _f32(64), _f32(64), torch.zeros(64, device=DEV), torch.ones(64, device=DEV)
    if not backward:
        return lambda: ops.bn_fwd(a, gamma, beta, 1e-5, 0.1, rm, rv)
    _, mean, invstd = ops.bn_fwd(a, gamma, beta, 1e-5, 0.1, rm, rv)
    dy = _f32(300, 64)
    return lambda: ops.bn_bwd(dy, a, gamma, mean, invstd)


def _transpose(transpose):
    ops, x = _ops(), _f32(100, 48)
    out = torch.empty(48, 100, device=DEV) if transpose else torch.empty(100, 48, device=DEV)
    ld = 100 if transpose else 48
    return lambda: ops.transpose_raw(x, 0, 48, 0, out, ld, 0, 1, 100, 48, transpose)


def _gemm(precision):
    ops, x, w = _ops(precision), _f32(256, 128), _f32(64, 128)
    out = torch.empty(256, 64, device=DEV)
    return lambda: ops.linear(x, w, out=out)


def _colsum():
    ops, x = _ops(), _f32(500, 33)
    return lambda: ops.colsum(x)


# operator -> (set-up returning the call, kernels the call enqueues)
LAUNCHES = {
    'og_split_tf32': (_split_tf32, 1),
    'og_weight_split_f16': (_weight_split_f16, 3),
    'og_amax': (_amax, 1),
    'og_match_fwd': (_match, 4),
    'og_gt_matches_fwd': (_gt_matches, 7),
    'og_criterion_fwd': (_criterion, 1),
    'og_sinkhorn_train_fwd': (lambda: _sinkhorn(False), 1),
    'og_sinkhorn_bwd': (lambda: _sinkhorn(True), 6),          # 3 initial sums, the cooperative sweep, dZ, d dustbin
    'og_bn_train_fwd': (lambda: _bn(False), 6),               # 2 two-stage column reductions, stats, apply
    'og_bn_train_bwd': (lambda: _bn(True), 3),
    'og_colsum': (_colsum, 2),
    'og_transpose': (lambda: _transpose(True), 1),
    'og_transpose_copy': (lambda: _transpose(False), 1),
    'og_linear_auto_fwd_fp32': (lambda: _gemm(_cabi.OG_PREC_FP32), 1),
    'og_linear_auto_fwd_tf32x3': (lambda: _gemm(_cabi.OG_PREC_TF32X3), 2),    # weight split + GEMM
}


@pytest.mark.gpu
@pytest.mark.parametrize('op', sorted(LAUNCHES))
def test_operator_counts_its_launches(op):
    setup, kernels = LAUNCHES[op]
    call = setup()
    torch.cuda.synchronize()
    lib = _cabi.lib()
    before = lib.og_last_forward_launches()
    rc = call()
    if isinstance(rc, int):
        _cabi.check(rc, op)
    torch.cuda.synchronize()
    assert lib.og_last_forward_launches() - before == kernels


@pytest.mark.gpu
def test_forward_reports_its_own_launches():
    from openglue_b200.superglue import SuperGlue
    from openglue_b200.synthetic import default_config, synthetic_pairs, synthetic_state_dict
    cfg = default_config(descriptor_dim=64, num_stages=1, num_iters=10)
    model = SuperGlue(dict(cfg)).eval()
    model.load_state_dict(synthetic_state_dict(cfg, seed=0))
    model = model.to(DEV)
    data = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in synthetic_pairs(1, 64, 48, 64, 1, seed=3).items()}
    model.run(data, want_matches=True)
    first = model.last_launches
    assert first == _cabi.lib().og_last_forward_launches() > 0
    _split_tf32()()                              # an operator between two forward passes ...
    assert _cabi.lib().og_last_forward_launches() == first + 1
    model.run(data, want_matches=True)
    assert model.last_launches == first          # ... is not counted in the next one
