"""Output stores of the fp16 Hopper GEMM (csrc/linear_sm90.cuh): each consumer stages half a tile in shared memory and stores it by
TMA when every output has 16-byte aligned rows, and with its threads otherwise.  The outputs are written into NaN-poisoned buffers
with guard rows, guard columns and (V^T) padding past the sequence length: the guards must stay untouched and the results must
equal the float64 reference within the bounds of test_gpu_f16.py."""
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
BOUND = 2e-6
GUARD = 5                                                # guard rows / channels past the output


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _case(rows, k, nout, batch, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    A = 3 * torch.randn(batch, rows, k, generator=g, device=DEV)
    W = torch.randn(nout, k, generator=g, device=DEV) / 8
    bias = torch.randn(nout, generator=g, device=DEV)
    hi, lo = torch.empty(W.shape, dtype=torch.float16, device=DEV), torch.empty(W.shape, dtype=torch.float16, device=DEV)
    meta = torch.zeros(4, device=DEV)
    lib = _cabi.lib()
    _cabi.check(lib.og_weight_split_f16(_p(W), _p(bias), nout, k, _p(hi), _p(lo), _p(meta), _st()), 'split16')
    amax = torch.zeros(1, device=DEV)
    _cabi.check(lib.og_amax(_p(A), A.numel(), _p(amax), _st()), 'og_amax')
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.strideA, a.k1, a.ldw = A.data_ptr(), k, rows * k, k, k
    a.bias, a.rows, a.nout, a.batch, a.alpha = bias.data_ptr(), rows, nout, batch, 0.7
    ref = 0.7 * (A.double() @ W.double().t()) + bias.double()
    return a, (hi, lo, meta, amax, A, bias), ref          # the operands stay referenced while `a` points at them


def _rel(x, ref):
    return float((x.double() - ref).abs().max() / ref.abs().max())


# ldy / ldyt = the output's extent + extra: extra % 4 (fp32) or % 8 (fp16) == 0 keeps the rows 16-byte aligned (TMA stores), any
# other value makes the threads store them
SHAPES = [(128 * 2 - 51, 128, 1), (1000, 392, 1), (517, 334, 3), (2049, 200, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize('extra', [8, 6])
@pytest.mark.parametrize('rows,nout,batch', SHAPES)
@pytest.mark.parametrize('resid', [False, True])
def test_fp32_output_keeps_its_guards(rows, nout, batch, resid, extra):
    """Kind 1 (fp32 Y, bias, amax), also with the residual read from Y itself (fc2's in-place form)."""
    a, (hi, lo, meta, amax, *_keep), ref = _case(rows, 256, nout, batch, seed=rows + nout)
    ld = nout + (extra if nout % 4 == 0 else 4 - nout % 4 + extra)
    buf = torch.full((batch, rows + GUARD, ld), float('nan'), device=DEV)
    if resid:
        R = torch.randn(batch, rows, nout, device=DEV)
        buf[:, :rows, :nout] = R
        ref = ref + R.double()
        a.R, a.ldr, a.strideR = buf.data_ptr(), ld, (rows + GUARD) * ld
    a.Y, a.ldy, a.strideY = buf.data_ptr(), ld, (rows + GUARD) * ld
    amax_out = torch.zeros(1, device=DEV)
    _cabi.check(_cabi.lib().og_linear_f16_fwd(C.byref(a), _p(hi), _p(lo), _p(meta), _p(amax), _p(amax_out), None, None, None, None,
                                              None, 0, _st()), 'linear_f16')
    torch.cuda.synchronize()
    Y = buf[:, :rows, :nout]
    assert _rel(Y, ref) <= BOUND
    assert float(amax_out) == float(Y.abs().max())
    assert bool(buf[:, rows:].isnan().all()) and bool(buf[:, :, nout:].isnan().all())


@pytest.mark.gpu
@pytest.mark.parametrize('extra', [8, 2])
@pytest.mark.parametrize('rows,nout,batch', SHAPES)
@pytest.mark.parametrize('kind', ['k', 'vt'])
def test_fp16_operand_outputs_keep_their_guards(kind, rows, nout, batch, extra):
    """Kind 2 (row-major fp16 hi / lo, the K operand) and kind 3 (transposed, V^T: [batch, nout, ldyt] with ldyt past the
    sequence length, the padding the attention kernel's operand rows carry)."""
    a, (hi, lo, meta, amax, *_keep), ref = _case(rows, 256, nout, batch, seed=rows * 3 + nout)
    scale = torch.zeros(1, device=DEV)
    nan = float('nan')
    if kind == 'k':
        ld = (nout + 7) // 8 * 8 + extra
        shape, strides = (batch, rows + GUARD, ld), ('ldy', 'strideY')
    else:
        ld = (rows + 7) // 8 * 8 + extra
        shape, strides = (batch, nout + GUARD, ld), ('ldyt', 'strideYt')
    bh = torch.full(shape, nan, dtype=torch.float16, device=DEV)
    bl = torch.full(shape, nan, dtype=torch.float16, device=DEV)
    setattr(a, strides[0], ld)
    setattr(a, strides[1], shape[1] * ld)
    outs = (_p(bh), _p(bl), None, None) if kind == 'k' else (None, None, _p(bh), _p(bl))
    _cabi.check(_cabi.lib().og_linear_f16_fwd(C.byref(a), _p(hi), _p(lo), _p(meta), _p(amax), None, _p(scale), *outs, 0, _st()),
                'linear_f16')
    torch.cuda.synchronize()
    if kind == 'k':
        inner, outer = nout, rows
    else:
        inner, outer = rows, nout
    for b in (bh, bl):
        assert bool(b[:, outer:].isnan().all()) and bool(b[:, :, inner:].isnan().all())
        assert not bool(b[:, :outer, :inner].isnan().any())
    Y = (bh[:, :outer, :inner].double() + bl[:, :outer, :inner].double()) / float(scale)
    assert _rel(Y if kind == 'k' else Y.transpose(1, 2), ref) <= BOUND


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['y', 'k', 'vt'])
def test_many_tiles_per_cta(kind):
    """Several rounds of tiles per CTA with ragged rows: every round reuses the staging buffers of the previous one."""
    sms = _sms()
    rows, nout = 128 * (2 * sms + 3) - 77, 256
    a, (hi, lo, meta, amax, *_keep), ref = _case(rows, 512, nout, 1, seed=11)
    lib = _cabi.lib()
    if kind == 'y':
        Y = torch.full((rows, nout), float('nan'), device=DEV)
        a.Y, a.ldy = Y.data_ptr(), nout
        _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(hi), _p(lo), _p(meta), _p(amax), None, None, None, None, None, None, 0, _st()), 'f16')
        torch.cuda.synchronize()
        assert _rel(Y, ref[0]) <= BOUND
        return
    scale = torch.zeros(1, device=DEV)
    shape = (rows, nout) if kind == 'k' else (nout, (rows + 7) // 8 * 8)
    bh = torch.full(shape, float('nan'), dtype=torch.float16, device=DEV)
    bl = torch.full(shape, float('nan'), dtype=torch.float16, device=DEV)
    if kind == 'k':
        a.ldy = nout
        outs = (_p(bh), _p(bl), None, None)
    else:
        a.ldyt = shape[1]
        outs = (None, None, _p(bh), _p(bl))
    _cabi.check(lib.og_linear_f16_fwd(C.byref(a), _p(hi), _p(lo), _p(meta), _p(amax), None, _p(scale), *outs, 0, _st()), 'f16')
    torch.cuda.synchronize()
    Y = (bh.double() + bl.double()) / float(scale)
    if kind == 'vt':
        assert bool(bh[:, rows:].isnan().all())
        Y = Y[:, :rows].t()
    assert _rel(Y, ref[0]) <= BOUND


def test_fp16_gemm_stores_its_tiles_by_tma():
    """Static check of the built library (cuobjdump, no GPU; OG_LIB names another build): the fp16 GEMM stores its output tiles
    with TMA (UTMASTG) from shared memory it writes with stmatrix (STSM)."""
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    path = os.environ.get('OG_LIB') or _cabi.LIB_PATH
    assert os.path.exists(path), f'library not built: {path}'
    res = subprocess.run([tool, '-sass', path], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    ops, cur = [], None
    for line in res.stdout.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = 'linear_sm90_kernel' in m.group(1) and 'F16LinearArgs' in m.group(1)
            continue
        m = re.match(r'\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P(?:\d+|T)\s+)?([A-Z0-9_.]+)', line)
        if m and cur:
            ops.append(m.group(1).split('.')[0])
    assert ops, 'fp16 GEMM kernel not found'
    assert 'UTMASTG' in ops and 'STSM' in ops
