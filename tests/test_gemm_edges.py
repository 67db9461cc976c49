"""The 3xTF32 and fp32 GEMMs and the training step's GEMM dispatch at their K, tile, batch and layout edges, against float64.

Entry points: og_linear_fwd (the fp32 CUDA-core kernel, 128 x 128 x 8 tiles), og_linear_tc_fwd (the 3xTF32 wgmma kernel, 128 x 128
output tiles, K blocks of 32, W pre-split by og_split_tf32) and og_linear_auto_fwd (the training step's dispatcher, at OG_PREC_FP32
and OG_PREC_TF32X3: it splits W on the fly and runs the tensor-core kernel where the shape is tileable, the fp32 kernel otherwise).

Every operand and output lives in a larger NaN-filled buffer: rows longer than the data (lda > k1, ldw > K, ldy > nout, ...), gaps
between batch items, other heads' columns next to a head slice, and guard floats before and after.  A read past K, past a head or
past an item therefore shows up as NaN in the result, and after the call every output element the GEMM must not write is checked to
be still NaN.  All reads stay inside the buffers, so a wrong kernel produces NaN rather than a fault.

The reference is float64 torch on the device: alpha [A | A2] W^T + bias, then ReLU, then + rscale R or + R.  Bounds:
- the operators' contracts, relative to max |ref|: 2e-6 for the fp32 kernel (test_gpu_parity.py), 1.5e-6 for the 3xTF32 kernel
  (test_gpu_tc.py);
- per element, an error model: |y - ref| <= c u (|alpha| sum_k |a_k w_k| + |bias| + |s r|), u = 2^-24.
  fp32 kernel: one FMA per k in K order, so c = K + 4 (K roundings of the running sum, then alpha, bias and the residual).
  3xTF32 kernel: a w is carried as a_hi w_hi + a_hi w_lo + a_lo w_hi with hi = rna_tf32(x), lo = rna_tf32(x - hi), so the dropped
  a_lo w_lo and the rounding of the two lo parts cost at most 16 u |a w|; inside each 64-element chunk the tensor core adds the 3 x 64
  exact products into an fp32 accumulator that may truncate, up to 2 u of the running sum per product, 6 min(K, 64); the chunks are
  added with round-to-nearest, one u each.  c = 16 + 6 min(K, 64) + ceil(K / 64) + 4.
The per-element bound holds for every case; the cases built with cancellation (half the rows sum x w and then -(1 - 2^-10) x w over
the same weights, so the result is ~2^-10 of the partial sums) put it where the contract, relative to max |ref|, says little.  Every
case prints its errors next to both bounds.
"""
import ctypes as C
import math
import types

import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200._cabi import ptr as _p, stream as _st

DEV = 'cuda:0'
NAN = float('nan')
U = 2.0 ** -24
GUARD = 64                                      # poisoned floats before and after every buffer
CONTRACT = {'simt': 2e-6, 'tf32': 1.5e-6}
OG_EUNSUPPORTED = -2
GRID_ROWS = 65535 * 128                         # rows one launch of the fp32 kernel covers (grid.y <= 65535)


def _pad4(n):
    return (n + 3) // 4 * 4


def _report(tag, err, bound, extra=''):
    print(f'\n[{tag}] max error {err:.3e}, bound {bound:.3e} ({err / bound if bound > 0 else 0.0:.2f} of it){extra}')


# --------------------------------------------------------------------------------------------------------------------- buffers
class Poisoned:
    """`items` matrices [rows, cols] in one NaN buffer: element (b, r, c) at base + b stride + (roff + r) ld + coff + c.  The GEMM
    gets the pointer to (0, 0, 0); everything else in the buffer (other rows, other columns, gaps, guards) stays NaN."""

    def __init__(self, items, rows, cols, ld, stride=None, roff=0, coff=0, shift=0):
        assert ld >= coff + cols
        self.items, self.rows, self.cols, self.ld = items, rows, cols, ld
        self.stride = (roff + rows) * ld + 8 if stride is None else stride
        self.off = GUARD + shift + roff * ld + coff
        span = (items - 1) * self.stride + (rows - 1) * ld + cols if items else 0
        self.buf = torch.full((self.off + span + GUARD,), NAN, device=DEV)

    def ptr(self):
        return _p(self.buf, self.off)

    def view(self, buf=None):
        """[items, rows, cols] view of the data region of `buf` (default: this buffer)"""
        b = self.buf if buf is None else buf
        return b.as_strided((self.items, self.rows, self.cols), (self.stride, self.ld, 1), self.off)

    def mask(self):
        m = torch.zeros(self.buf.shape, dtype=torch.bool, device=DEV)
        self.view(m).fill_(True)
        return m

    def set(self, t):
        self.view().copy_(t.reshape(self.items, self.rows, self.cols))
        return self

    def untouched(self, buf=None):
        """every element outside the data region is still NaN"""
        b = self.buf if buf is None else buf
        return bool(torch.isnan(b[~self.mask()]).all())


# --------------------------------------------------------------------------------------------------------------------- cases
def case(name, rows, k1, nout, batch=1, k2=0, **kw):
    """One GEMM: sizes, epilogue and layout.  Layout defaults: every row padded by 4 NaN floats past the next multiple of 4, 8 NaN
    floats between batch items, W per batch item when wbatch (one NaN row between items), A broadcast over the batch when abcast."""
    K = k1 + k2
    c = types.SimpleNamespace(name=name, rows=rows, k1=k1, k2=k2, K=K, nout=nout, batch=batch, alpha=0.75, bias=True, relu=False,
                              res=None, rscale=False, wbatch=False, abcast=False, cancel=False, outs=('Y', 'Yt', 'split', 'tsplit'), seed=0,
                              lda=_pad4(k1) + 4, lda2=_pad4(k2) + 4, ldw=_pad4(K) + 4, ldy=_pad4(nout) + 4, ldyt=_pad4(rows) + 4,
                              ldr=_pad4(nout) + 8, strideA=None, strideA2=None, strideW=None, strideY=None, strideYt=None,
                              acoff=0, ycoff=0, wroff=0, wcoff=0, wrows=None, ashift=0, a2shift=0, wshift=0)
    for k, v in kw.items():
        assert hasattr(c, k), k
        setattr(c, k, v)
    return c


def _operands(c):
    """NaN-poisoned A (A2), W, bias, rscale, R and the float64 reference and error scale (alpha |X| |W|^T + |b| + |s r|)"""
    g = torch.Generator(device=DEV).manual_seed(c.seed)
    r = lambda *s: torch.randn(*s, generator=g, device=DEV)
    ia = 1 if c.abcast else c.batch
    iw = c.batch if c.wbatch else 1
    X = 2 * r(ia, c.rows, c.K)
    W = r(iw, c.nout, c.K) / 4
    if c.cancel:                                                       # rows 1, 3, ...: x w, then -(1 - 2^-10) x w
        h = c.K // 2
        W[:, :, h:2 * h] = W[:, :, :h]
        X[:, 1::2, h:2 * h] = -(1 - 2.0 ** -10) * X[:, 1::2, :h]
    bias = r(c.nout) if c.bias else None
    A = Poisoned(ia, c.rows, c.k1, c.lda, c.strideA, coff=c.acoff, shift=c.ashift).set(X[:, :, :c.k1])
    A2 = Poisoned(ia, c.rows, c.k2, c.lda2, c.strideA2, shift=c.a2shift).set(X[:, :, c.k1:]) if c.k2 else None
    wrows = c.wrows if c.wrows is not None else (c.nout + 1 if c.wbatch else c.nout)
    strideW = c.strideW if c.strideW is not None else (wrows * c.ldw if c.wbatch else 0)
    Wp = Poisoned(iw, c.nout, c.K, c.ldw, strideW if c.wbatch else None, roff=c.wroff, coff=c.wcoff, shift=c.wshift).set(W)
    Wp.gemm_stride = strideW
    R = s = None
    if c.res:
        R = r(c.batch, c.rows, c.nout)
        s = torch.rand(c.nout, generator=g, device=DEV) + 0.5 if c.rscale else None
    ref = c.alpha * (X.double() @ W.double().transpose(1, 2))
    scale = abs(c.alpha) * (X.double().abs() @ W.double().abs().transpose(1, 2))
    if ref.shape[0] != c.batch:
        ref, scale = ref.expand(c.batch, -1, -1), scale.expand(c.batch, -1, -1)
    if bias is not None:
        ref, scale = ref + bias.double(), scale + bias.double().abs()
    if c.relu:
        ref = ref.relu()
    if R is not None:
        sr = R.double() * (s.double() if s is not None else 1.0)
        ref, scale = ref + sr, scale + sr.abs()
    return types.SimpleNamespace(A=A, A2=A2, W=Wp, bias=bias, R=R, s=s, ref=ref, scale=scale)


def _outputs(c, ops, outs):
    """NaN-poisoned output buffers (Y, Yt, Yhi / Ylo, Ythi / Ytlo) for the requested outputs; R aliasing Y is written into Y"""
    y = lambda: Poisoned(c.batch, c.rows, c.nout, c.ldy, c.strideY, coff=c.ycoff)
    yt = lambda: Poisoned(c.batch, c.nout, c.rows, c.ldyt, c.strideYt)
    o = {}
    if 'Y' in outs or c.res == 'alias':
        o['Y'] = y()
    if 'Yt' in outs:
        o['Yt'] = yt()
    if 'split' in outs:
        o['Yhi'], o['Ylo'] = y(), y()
    if 'tsplit' in outs:
        o['Ythi'], o['Ytlo'] = yt(), yt()
    if c.res == 'alias':
        o['Y'].set(ops.R)
    elif c.res:
        o['R'] = Poisoned(c.batch, c.rows, c.nout, c.ldr).set(ops.R)
    return o


def _args(c, ops, o):
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.strideA = ops.A.ptr(), c.lda, (0 if c.abcast else ops.A.stride)
    if ops.A2 is not None:
        a.A2, a.lda2, a.strideA2 = ops.A2.ptr(), c.lda2, (0 if c.abcast else ops.A2.stride)
    a.k1, a.k2 = c.k1, c.k2
    a.W, a.ldw, a.strideW = ops.W.ptr(), c.ldw, ops.W.gemm_stride
    a.bias = _p(ops.bias)
    a.rows, a.nout, a.batch, a.alpha, a.relu = c.rows, c.nout, c.batch, c.alpha, int(c.relu)
    if c.res == 'alias':
        a.R, a.ldr, a.strideR = o['Y'].ptr(), o['Y'].ld, o['Y'].stride
    elif c.res:
        a.R, a.ldr, a.strideR = o['R'].ptr(), o['R'].ld, o['R'].stride
    a.rscale = _p(ops.s)
    if 'Y' in o:
        a.Y, a.ldy, a.strideY = o['Y'].ptr(), o['Y'].ld, o['Y'].stride
    if 'Yt' in o:
        a.Yt, a.ldyt, a.strideYt = o['Yt'].ptr(), o['Yt'].ld, o['Yt'].stride
    if 'Yhi' in o and 'Y' not in o:                                    # the split outputs share Y's (Yt's) layout
        a.ldy, a.strideY = o['Yhi'].ld, o['Yhi'].stride
    if 'Ythi' in o and 'Yt' not in o:
        a.ldyt, a.strideYt = o['Ythi'].ld, o['Ythi'].stride
    return a


def _split_w(W):
    hi, lo = torch.empty_like(W.buf), torch.empty_like(W.buf)
    _cabi.check(_cabi.lib().og_split_tf32(_p(W.buf), _p(hi), _p(lo), W.buf.numel(), _st()), 'og_split_tf32')
    return _p(hi, W.off), _p(lo, W.off), (hi, lo)


def launch(entry, c, ops, o):
    """Runs case c through one entry point: 'simt' og_linear_fwd, 'tf32' og_linear_tc_fwd, 'auto_fp32' / 'auto_tf32'
    og_linear_auto_fwd.  Returns the status."""
    lib = _cabi.lib()
    a = _args(c, ops, o)
    if entry == 'simt':
        return lib.og_linear_fwd(C.byref(a), _cabi.OG_PREC_FP32, _st())
    if entry == 'tf32':
        hi, lo, keep = _split_w(ops.W)
        rc = lib.og_linear_tc_fwd(C.byref(a), hi, lo, *(_p(o[k].buf, o[k].off) if k in o else None for k in ('Yhi', 'Ylo', 'Ythi', 'Ytlo')),
                                  2, _st())
        torch.cuda.synchronize()
        return rc
    prec = _cabi.OG_PREC_FP32 if entry == 'auto_fp32' else _cabi.OG_PREC_TF32X3
    n = _cabi.check_size(lib.og_linear_auto_scratch_floats(C.byref(a)), 'og_linear_auto_scratch_floats')
    scratch = torch.full((max(n, 4),), NAN, device=DEV)
    rc = lib.og_linear_auto_fwd(C.byref(a), prec, _p(scratch), _st())
    torch.cuda.synchronize()
    return rc


def _bits(t):
    return t.contiguous().view(torch.int32)


def check(entry, c, allowed=None):
    """Runs c through `entry` with every output the entry point and the case allow, checks values, layout and poisoning; returns
    the outputs (for bit comparisons between entry points)."""
    outs = [k for k in c.outs if entry == 'tf32' or k in ('Y', 'Yt')] or ['Y', 'Yt']     # split outputs: the tensor-core form only
    if allowed is not None:
        outs = [k for k in outs if k in allowed]
    ops = _operands(c)
    o = _outputs(c, ops, outs)
    _cabi.check(launch(entry, c, ops, o), f'{entry} {c.name}')
    torch.cuda.synchronize()
    # the kernel that ran (c.kernel: auto_tf32 runs the fp32 kernel on untileable shapes) sets the bounds
    form = getattr(c, 'kernel', 'tf32' if entry in ('tf32', 'auto_tf32') else 'simt')
    K = c.K
    cm = K + 4 if form == 'simt' else 16 + 6 * min(K, 64) + math.ceil(K / 64) + 4
    ref, scale = ops.ref, ops.scale
    bound_c = CONTRACT[form] * float(ref.abs().max())
    vals = {}
    if 'Y' in outs:
        vals['Y'] = o['Y'].view().double()
    if 'Yt' in outs:
        vals['Yt'] = o['Yt'].view().double().transpose(1, 2)
    if 'Yhi' in o:
        vals['Yhi+Ylo'] = o['Yhi'].view().double() + o['Ylo'].view().double()
    if 'Ythi' in o:
        vals['Ythi+Ytlo'] = (o['Ythi'].view().double() + o['Ytlo'].view().double()).transpose(1, 2)
    split_slack = 2.0 ** -21 * ref.abs()                               # hi + lo of Y: <= 2^-21 |Y| from Y
    for k, v in vals.items():
        assert bool(torch.isfinite(v).all()), f'{entry} {c.name}: {k} has non-finite values'
        d = (v - ref).abs()
        extra = split_slack if '+' in k else 0.0
        err = float(d.max())
        ratio = float((d / (cm * U * scale + extra + 1e-300)).max())
        _report(f'{entry} {c.name} {k}', err, bound_c, f'; per element {ratio:.2f} of c u sum|a w| (c = {cm})')
        assert err <= bound_c + (float(split_slack.max()) if '+' in k else 0.0), f'{entry} {c.name}: {k} over the contract'
        assert ratio <= 1.0, f'{entry} {c.name}: {k} over the error model'
    for k, t in o.items():
        if k != 'R':
            assert t.untouched(), f'{entry} {c.name}: {k} written outside its layout'
    if 'Y' in outs and 'Yt' in outs:
        assert torch.equal(_bits(o['Yt'].view().transpose(1, 2)), _bits(o['Y'].view())), f'{c.name}: Yt != Y^T'
    if 'Yhi' in o:
        hi, lo = o['Yhi'].view(), o['Ylo'].view()
        assert bool(((_bits(hi) & 0x1FFF) == 0).all()), f'{c.name}: Yhi not tf32-exact'
        if 'Y' in outs:
            y = o['Y'].view()
            assert bool(((hi.double() + lo.double() - y.double()).abs() <= 2.0 ** -21 * y.double().abs()).all()), f'{c.name}: Yhi + Ylo != Y'
    if 'Yhi' in o and 'Ythi' in o:
        assert torch.equal(_bits(o['Ythi'].view().transpose(1, 2)), _bits(o['Yhi'].view()))
        assert torch.equal(_bits(o['Ytlo'].view().transpose(1, 2)), _bits(o['Ylo'].view()))
    return {k: t.view().clone() for k, t in o.items() if k != 'R'}


# --------------------------------------------------------------------------------------------------------------------- case table
def _training_forms():
    """The training step's GEMM calls (openglue_b200/training.py), restated at small sizes with its strides"""
    cs = []
    B, n, m, d = 2, 37, 50, 64
    lds = _pad4(m)
    # score GEMM: Sp[b] = m0[b] m1[b]^T d^-0.5, ldy = lds > m, per-batch W (m rows per item)
    cs.append(case('score gemm', n, d, m, B, alpha=d ** -0.5, bias=False, wbatch=True, wrows=m, lda=d, ldw=d, ldy=lds,
                   strideA=n * d, strideY=n * lds))
    # dm0 = dS m1 d^-0.5: dS [B, n, mp], mT[1] [B, d, mp]
    mp = _pad4(m)
    cs.append(case('dm', n, mp, d, B, alpha=d ** -0.5, bias=False, wbatch=True, wrows=d, lda=mp, ldw=mp, ldy=d,
                   strideA=n * mp, strideY=n * d))
    # attention gradient, head 1 of H: the other heads' columns (rows of the transposed operands) are NaN
    for dh in (8, 16, 32, 64):
        H = 3 if dh < 64 else 2
        dd, c0 = H * dh, dh
        nq, nk = 37, 45
        nqp, nkp = _pad4(nq), _pad4(nk)
        # P = q_h k_h^T s and dP = do_h v_h^T: head-offset A and W, K = dh
        cs.append(case(f'attn P, dP dh{dh}', nq, dh, nk, B, alpha=dh ** -0.5, bias=False, wbatch=True, wrows=nk, lda=dd, ldw=dd,
                       acoff=c0, wcoff=c0, strideA=nq * dd, strideW=nk * dd, ldy=nkp, strideY=nq * nkp))
        # dv_h = P^T do_h and dk_h = dS^T q_h (dq_h = dS k_h): W = rows c0 .. c0 + dh of a [B, d, nqp] operand, Y head-offset
        cs.append(case(f'attn dV, dK dh{dh}', nk, nqp, dh, B, bias=False, wbatch=True, wrows=dd, wroff=c0, lda=nqp, ldw=nqp,
                       strideA=nk * nqp, strideW=dd * nqp, ldy=dd, ycoff=c0, strideY=nk * dd))
        cs.append(case(f'attn dQ dh{dh}', nq, nkp, dh, B, bias=False, wbatch=True, wrows=dd, wroff=c0, lda=nkp, ldw=nkp,
                       strideA=nq * nkp, strideW=dd * nkp, ldy=dd, ycoff=c0, strideY=nq * dd))
    # A broadcast over the batch with a per-batch W
    cs.append(case('A broadcast', 100, 64, 40, 3, abcast=True, wbatch=True))
    # grad_weight, split-K batched: part[s] = dYt[s] Xt[s]^T, K = 512 per chunk
    cs.append(case('grad_weight split-K', 64, 512, 40, 3, bias=False, alpha=1.0, wbatch=True, wrows=40, lda=512, ldw=512,
                   ldy=40, strideA=64 * 512, strideY=64 * 40, strideW=40 * 512))
    # grad_weight, one chunk of 300 rows: into[:, off:off + K] += dY^T X (R is Y)
    cs.append(case('grad_weight 300 rows', 64, 300, 40, bias=False, alpha=1.0, res='alias', ldy=100, ycoff=52, lda=300, ldw=300))
    return cs


def _cases():
    cs = []
    for K in (32, 36, 60, 64, 100, 132, 260, 300, 516, 576, 1152):
        cs.append(case(f'K {K}', 129, K, 129, cancel=K >= 64, seed=K))
    for k1 in (32, 64, 256):
        for k2 in (4, 36, 100, 256):
            cs.append(case(f'k1 {k1} k2 {k2}', 130, k1, 72, 2, k2=k2, cancel=True, seed=k1 + k2))
    for rows, nout, batch in ((1, 64, 1), (127, 1, 2), (128, 3, 1), (129, 127, 3), (257, 128, 1), (1, 129, 5), (128, 392, 2),
                              (257, 392, 1), (127, 129, 4)):
        cs.append(case(f'rows {rows} nout {nout} batch {batch}', rows, 96, nout, batch, seed=rows + nout))
    cs.append(case('no bias, relu, alpha -1.25', 200, 128, 100, 2, bias=False, relu=True, alpha=-1.25))
    cs.append(case('R with its own ldr', 200, 64, 100, 2, res='R', ldr=132))
    cs.append(case('R with rscale', 200, 64, 100, 2, res='R', rscale=True, relu=True))
    cs.append(case('R is Y (in-place fc2)', 150, 128, 64, 2, res='alias', ldy=68))
    cs.append(case('R is Y with rscale (final projection)', 150, 64, 64, res='alias', rscale=True, ldy=64))
    cs.append(case('Yt only', 129, 64, 130, 2, outs=('Yt',)))
    cs.append(case('split outputs only', 129, 64, 130, 2, outs=('split', 'tsplit')))
    cs.append(case('Y and split, no Yt', 100, 64, 50, outs=('Y', 'split')))
    return cs + _training_forms()


CASES = {c.name: c for c in _cases()}
SIMT_ONLY = {f'K {K}': case(f'K {K}', 129, K, 129, cancel=K >= 64, seed=K) for K in (9, 34, 65)}


def _tileable(c):
    return c.K >= 32 and c.k1 % 4 == 0 and c.k2 % 4 == 0 and (not c.k2 or c.k1 % 32 == 0)


# every case through every entry point that takes it (the tensor-core form rejects untileable shapes: test_dispatch_decisions)
TABLE = [(e, n) for n, c in {**CASES, **SIMT_ONLY}.items() for e in ('simt', 'tf32', 'auto_fp32', 'auto_tf32') if e != 'tf32' or _tileable(c)]


@pytest.mark.gpu
@pytest.mark.parametrize('entry,name', TABLE)
def test_case_table(entry, name):
    c = CASES.get(name) or SIMT_ONLY[name]
    if entry == 'auto_tf32' and not _tileable(c):
        c = types.SimpleNamespace(**vars(c), kernel='simt')           # the dispatcher runs the fp32 kernel: its contract
    check(entry, c)


# --------------------------------------------------------------------------------------------------------------------- dispatch
DISPATCH = [
    # (name, tileable, case)
    ('K 28', False, case('K 28', 100, 28, 70)),
    ('K 32', True, case('K 32', 100, 32, 70)),
    ('K 34 (K % 4)', False, case('K 34', 100, 34, 70)),
    ('k1 36 with A2', False, case('k1 36 A2', 100, 36, 70, k2=28)),
    ('k1 32 with A2', True, case('k1 32 A2', 100, 32, 70, k2=36)),
    ('A offset by one float', False, case('A +1', 100, 64, 70, ashift=1)),
    ('A2 offset by one float', False, case('A2 +1', 100, 64, 70, k2=32, a2shift=1)),
    ('W offset by one float', False, case('W +1', 100, 64, 70, wshift=1)),
    ('lda % 4', False, case('lda % 4', 100, 64, 70, lda=67)),
    ('strideA % 4', False, case('strideA % 4', 100, 64, 70, 2, strideA=100 * 68 + 2)),
    ('ldw % 4', False, case('ldw % 4', 100, 64, 70, ldw=66)),
    ('strideW % ldw', False, case('strideW % ldw', 100, 64, 70, 2, wbatch=True, strideW=71 * 68 + 4)),
    ('strideW whole rows', True, case('strideW rows', 100, 64, 70, 2, wbatch=True, strideW=72 * 68)),
]


@pytest.mark.gpu
@pytest.mark.parametrize('name', [d[0] for d in DISPATCH])
def test_dispatch_decisions(name):
    """og_linear_auto_fwd at TF32X3 equals, bit for bit, the kernel that should run: og_linear_tc_fwd on the same split where the
    shape is tileable, og_linear_fwd otherwise; og_linear_tc_fwd rejects an untileable shape before any launch; at FP32 the
    dispatcher always runs og_linear_fwd."""
    _, tileable, c = next(d for d in DISPATCH if d[0] == name)
    c = types.SimpleNamespace(**vars(c), kernel='tf32' if tileable else 'simt')
    c.outs = ('Y', 'Yt')
    auto = check('auto_tf32', c)
    auto32 = check('auto_fp32', types.SimpleNamespace(**{**vars(c), 'kernel': 'simt'}))
    simt = check('simt', types.SimpleNamespace(**{**vars(c), 'kernel': 'simt'}))
    lib = _cabi.lib()
    if tileable:
        want = check('tf32', c, allowed=('Y', 'Yt'))
    else:
        want = simt
        ops = _operands(c)
        o = _outputs(c, ops, ('Y', 'Yt'))
        hi, lo, keep = _split_w(ops.W)
        before = lib.og_last_forward_launches()
        rc = lib.og_linear_tc_fwd(C.byref(_args(c, ops, o)), hi, lo, None, None, None, None, 2, _st())
        assert rc == OG_EUNSUPPORTED, (rc, lib.og_last_error())
        assert lib.og_last_forward_launches() == before
        torch.cuda.synchronize()
        assert all(bool(torch.isnan(o[k].buf).all()) for k in ('Y', 'Yt'))
    for k in ('Y', 'Yt'):
        assert torch.equal(_bits(auto[k]), _bits(want[k])), f'{name}: auto_tf32 {k} differs from the expected kernel'
        assert torch.equal(_bits(auto32[k]), _bits(simt[k])), f'{name}: auto_fp32 {k} differs from og_linear_fwd'


def test_auto_scratch_is_the_weight_footprint():
    """og_linear_auto_scratch_floats covers what the split reads: batch - 1 blocks of strideW, then nout - 1 rows of ldw and K
    elements.  A head slice of a wider matrix (W at column c of rows of ldw) ends K elements into its last row, not ldw."""
    lib = _cabi.lib()
    for batch, nout, K, ldw, strideW in ((1, 64, 16, 64, 0), (2, 45, 32, 96, 45 * 96), (3, 16, 40, 40, 64 * 40), (1, 1, 9, 9, 0)):
        a = _cabi.OgLinearArgs()
        a.k1, a.nout, a.ldw, a.strideW, a.batch = K, nout, ldw, strideW, batch
        foot = (batch - 1) * strideW + (nout - 1) * ldw + K
        assert lib.og_linear_auto_scratch_floats(C.byref(a)) == 2 * ((foot + 63) // 64 * 64)


# --------------------------------------------------------------------------------------------------------------------- grid limits
@pytest.mark.gpu
def test_batch_past_the_grid_is_rejected_before_any_launch():
    lib = _cabi.lib()
    x = torch.full((64,), NAN, device=DEV)
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.k1, a.W, a.ldw, a.Y, a.ldy = _p(x), 4, 4, _p(x), 4, _p(x), 4
    a.rows, a.nout, a.batch, a.alpha = 1, 1, 65536, 1.0
    for call in (lambda: lib.og_linear_fwd(C.byref(a), _cabi.OG_PREC_FP32, _st()),
                 lambda: lib.og_linear_auto_fwd(C.byref(a), _cabi.OG_PREC_FP32, None, _st())):
        before = lib.og_last_forward_launches()
        assert call() == OG_EUNSUPPORTED
        assert b'65535' in lib.og_last_error()
        assert lib.og_last_forward_launches() == before
    torch.cuda.synchronize()
    assert bool(torch.isnan(x).all())


def _sampled_rows(rows):
    """the first tile, the rows around the first launch's end (row 65535 * 128) and the last 200"""
    idx = torch.cat([torch.arange(0, 128), torch.arange(GRID_ROWS - 200, min(GRID_ROWS + 200, rows)), torch.arange(rows - 200, rows)])
    return idx.unique().to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize('extra', [1, 129])
def test_fp32_gemm_rows_past_the_grid(extra):
    """SuperPoint's conv1a shape ([B H W, 9] x [64, 9]) with more rows than one launch's grid covers (28 images of 480 x 640 have
    8.6 M), through og_linear_fwd and og_linear_auto_fwd: every row written and finite, sampled rows against float64."""
    rows, K, nout = GRID_ROWS + extra, 9, 64
    g = torch.Generator(device=DEV).manual_seed(extra)
    A = torch.randn(rows, K, generator=g, device=DEV)
    W = torch.randn(nout, K, generator=g, device=DEV)
    bias = torch.randn(nout, generator=g, device=DEV)
    Y = torch.empty(rows, nout, device=DEV)
    idx = _sampled_rows(rows)
    ref = (A[idx].double() @ W.double().T + bias.double()).relu()
    lib = _cabi.lib()
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.k1, a.W, a.ldw, a.bias = _p(A), K, K, _p(W), K, _p(bias)
    a.rows, a.nout, a.batch, a.alpha, a.relu = rows, nout, 1, 1.0, 1
    a.Y, a.ldy = _p(Y), nout
    for name, call in (('og_linear_fwd', lambda: lib.og_linear_fwd(C.byref(a), _cabi.OG_PREC_FP32, _st())),
                       ('og_linear_auto_fwd fp32', lambda: lib.og_linear_auto_fwd(C.byref(a), _cabi.OG_PREC_FP32, None, _st())),
                       ('og_linear_auto_fwd tf32x3', lambda: lib.og_linear_auto_fwd(C.byref(a), _cabi.OG_PREC_TF32X3, _p(W.new_empty(4096)), _st()))):
        Y.fill_(NAN)
        _cabi.check(call(), name)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(Y).all()), f'{name}: rows left unwritten'
        err = float((Y[idx].double() - ref).abs().max())
        bound = CONTRACT['simt'] * float(ref.abs().max())
        _report(f'{name} rows {rows}', err, bound)
        assert err <= bound
    del A, Y
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_tf32_gemm_rows_past_the_grid():
    """The persistent tensor-core schedule has no row limit: 2^23 + 129 rows with K = nout = 32."""
    rows, K, nout = 2 ** 23 + 129, 32, 32
    g = torch.Generator(device=DEV).manual_seed(7)
    A = torch.randn(rows, K, generator=g, device=DEV)
    W = torch.randn(nout, K, generator=g, device=DEV)
    Whi, Wlo = torch.empty_like(W), torch.empty_like(W)
    lib = _cabi.lib()
    _cabi.check(lib.og_split_tf32(_p(W), _p(Whi), _p(Wlo), W.numel(), _st()), 'og_split_tf32')
    Y = torch.full((rows, nout), NAN, device=DEV)
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.k1, a.ldw = _p(A), K, K, K
    a.rows, a.nout, a.batch, a.alpha = rows, nout, 1, 1.0
    a.Y, a.ldy = _p(Y), nout
    _cabi.check(lib.og_linear_tc_fwd(C.byref(a), _p(Whi), _p(Wlo), None, None, None, None, 2, _st()), 'og_linear_tc_fwd')
    torch.cuda.synchronize()
    assert bool(torch.isfinite(Y).all())
    idx = _sampled_rows(rows)
    ref = A[idx].double() @ W.double().T
    err, bound = float((Y[idx].double() - ref).abs().max()), CONTRACT['tf32'] * float(ref.abs().max())
    _report(f'og_linear_tc_fwd rows {rows}', err, bound)
    assert err <= bound
    del A, Y
    torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------------------------------- position
def _dense_gemm(entry, A, W, bias, Y, rows, batch, a_off=0, y_off=0, strideA=0, strideW=0, strideY=0, Yt=None, yt_off=0, ldyt=0, strideYt=0):
    K, nout = A.shape[-1], W.shape[-2]
    a = _cabi.OgLinearArgs()
    a.A, a.lda, a.strideA, a.k1 = _p(A, a_off), K, strideA, K
    a.W, a.ldw, a.strideW, a.bias = _p(W), K, strideW, _p(bias)
    a.rows, a.nout, a.batch, a.alpha = rows, nout, batch, 0.75
    a.Y, a.ldy, a.strideY = _p(Y, y_off), nout, strideY
    if Yt is not None:
        a.Yt, a.ldyt, a.strideYt = _p(Yt, yt_off), ldyt, strideYt
    lib = _cabi.lib()
    if entry == 'simt':
        _cabi.check(lib.og_linear_fwd(C.byref(a), _cabi.OG_PREC_FP32, _st()), 'og_linear_fwd')
    else:
        hi, lo = torch.empty_like(W), torch.empty_like(W)
        _cabi.check(lib.og_split_tf32(_p(W), _p(hi), _p(lo), W.numel(), _st()), 'og_split_tf32')
        _cabi.check(lib.og_linear_tc_fwd(C.byref(a), _p(hi), _p(lo), None, None, None, None, 2, _st()), 'og_linear_tc_fwd')
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize('entry', ['simt', 'tf32'])
def test_repeated_launches_are_bit_identical(entry):
    g = torch.Generator(device=DEV).manual_seed(3)
    A, W, bias = torch.randn(3, 300, 132, generator=g, device=DEV), torch.randn(3, 200, 132, generator=g, device=DEV), torch.randn(200, device=DEV)
    outs = []
    for _ in range(3):
        Y = torch.full((3, 300, 200), NAN, device=DEV)
        _dense_gemm(entry, A, W, bias, Y, 300, 3, strideA=300 * 132, strideW=200 * 132, strideY=300 * 200)
        outs.append(_bits(Y))
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


@pytest.mark.gpu
def test_fp32_gemm_position_independence():
    """One batched launch = the per-item launches, and row ranges cut at multiples of 128 = the whole, bit for bit (Y and Yt):
    the host's row ranges past the grid limit rely on it."""
    g = torch.Generator(device=DEV).manual_seed(4)
    B, rows, K, nout = 3, 300, 67, 130
    A, W, bias = torch.randn(B, rows, K, generator=g, device=DEV), torch.randn(B, nout, K, generator=g, device=DEV), torch.randn(nout, device=DEV)
    whole, whole_t = torch.full((B, rows, nout), NAN, device=DEV), torch.full((B, nout, rows), NAN, device=DEV)
    _dense_gemm('simt', A, W, bias, whole, rows, B, strideA=rows * K, strideW=nout * K, strideY=rows * nout,
                Yt=whole_t, ldyt=rows, strideYt=nout * rows)
    for b in range(B):
        y, yt = torch.full((rows, nout), NAN, device=DEV), torch.full((nout, rows), NAN, device=DEV)
        _dense_gemm('simt', A[b].contiguous(), W[b].contiguous(), bias, y, rows, 1, Yt=yt, ldyt=rows)
        assert torch.equal(_bits(y), _bits(whole[b])) and torch.equal(_bits(yt), _bits(whole_t[b]))
        parts, parts_t = torch.full_like(y, NAN), torch.full_like(yt, NAN)
        Ab = A[b].contiguous()
        for r0, r1 in ((0, 128), (128, 256), (256, rows)):
            _dense_gemm('simt', Ab, W[b].contiguous(), bias, parts, r1 - r0, 1, a_off=r0 * K, y_off=r0 * nout, Yt=parts_t, yt_off=r0, ldyt=rows)
        assert torch.equal(_bits(parts), _bits(whole[b])) and torch.equal(_bits(parts_t), _bits(whole_t[b]))
