"""The three attention kernels at their tile, batch and layout edges, and the training step's attention gradient, against float64.

a. og_attention_fwd (fp32 CUDA cores, head_dim 8 / 16 / 32 / 64, tiles of 64 queries x 64 keys), og_attention_tc_fwd (3xTF32,
   head_dim 32 / 64, 128 queries x 64 keys) and og_attention_f16_fwd (3xFP16, head_dim 64, 128 queries x 128 keys) run one case
   table: nq and nk at every tile edge and around the 3-stage K / V ring, the benchmark's shapes, keys of the next batch item that
   would take the whole softmax if the key mask failed, the layouts the forward passes (the interleaved qkv buffer, padded rows,
   gaps between batch items), and adverse magnitudes at 1000 x 4097.  Every operand's padding and every output element a kernel
   must not write is NaN; after the call the output's padding columns, the gaps between batch items and the rows past the last
   item are checked to be still NaN.
b. Position independence (one launch over B items or H heads = one launch per item / per head subset, bit for bit), determinism,
   and agreement of the three forms at head_dim 64.
c. TrainStep._attention_bwd (the per-head materialised-softmax gradient) against float64 autograd, in the fp32 and tf32x3 operator
   precisions, and a gradient confined to one head leaving the other heads' dq, dk, dv exactly zero.

The reference is plain torch on the device in float64, the arithmetic of oracle.softmax_attention.  Bounds, relative to
max |ref|: the operators' contracts (5e-6 for the fp32 and fp16 forms, 1e-5 for the tf32 form); for ill-conditioned inputs
(logits of tens to thousands), the larger of the contract and 4x the float32 reference's own distance from float64.  Every case
prints its error next to its bound.
"""
import types

import pytest
import torch

from openglue_b200 import _cabi
from openglue_b200._cabi import ptr as _p, stream as _st

DEV = 'cuda:0'
NAN = float('nan')

BLOCKS = {'simt': (64, 64), 'tf32': (128, 64), 'fp16': (128, 128)}     # (queries, keys) per tile
HEAD_DIMS = {'simt': (8, 16, 32, 64), 'tf32': (32, 64), 'fp16': (64,)}
CONTRACT = {'simt': 5e-6, 'tf32': 1e-5, 'fp16': 5e-6}
FORM_DH = [(f, dh) for f in BLOCKS for dh in HEAD_DIMS[f]]
TAIL_ROWS = 3                                                             # poisoned output rows past the last batch item


def _report(tag, err, bound, extra=''):
    print(f'\n[{tag}] max error {err:.3e}, bound {bound:.3e} ({err / bound if bound > 0 else 0.0:.2f} of it){extra}')


# --------------------------------------------------------------------------------------------------------------------- reference
def _reference(q, k, v, H, dtype=torch.float64):
    """softmax(q k^T dh^-0.5) v per head, in `dtype`: q [B, nq, d], k, v [B, nk, d] -> [B, nq, d]"""
    B, nq, d = q.shape
    nk, dh = k.shape[1], d // H
    hv = lambda t, n: t.to(dtype).reshape(B, n, H, dh).permute(0, 2, 1, 3)
    o = torch.softmax(hv(q, nq) @ hv(k, nk).transpose(2, 3) * dh ** -0.5, dim=-1) @ hv(v, nk)
    return o.permute(0, 2, 1, 3).reshape(B, nq, d)


# --------------------------------------------------------------------------------------------------------------------- inputs
# recipes whose logits reach tens to thousands: the float32 reference itself moves away from float64 by more than the contract
ILL_CONDITIONED = {'Q x 2^10', 'K offset-dominated', 'near one-hot rows', 'row maxima in the last partial block',
                   'logits rising block by block', 'logits spanning +-80', 'next item dominates'}
MAGNITUDES = ['Q x 2^10', 'Q x 2^-10', 'K offset-dominated', 'near one-hot rows', 'row maxima in the last partial block',
              'logits rising block by block', 'logits spanning +-80', 'Q all zero']


def _per_head(t, H):
    return t.view(*t.shape[:-1], H, t.shape[-1] // H)


def _inputs(recipe, form, B, H, nq, nk, dh, seed):
    """q [B, nq, d], k, v [B, nk, d] (float32, on the device) of one recipe"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    d = H * dh
    r = lambda *s: torch.randn(*s, generator=g, device=DEV)
    q, k, v = 1.5 * r(B, nq, d), 1.5 * r(B, nk, d), r(B, nk, d)          # logits ~ N(0, 2.25^2)
    bk = BLOCKS[form][1]
    if recipe == 'Q x 2^10':
        q = q * 2.0 ** 10
    elif recipe == 'Q x 2^-10':
        q = q * 2.0 ** -10
    elif recipe == 'K offset-dominated':                           # a shared offset (cancels in the softmax) + a small per-key part
        k = 64 * r(d) + 2.0 ** -6 * r(B, nk, d)
        q = 8 * q
    elif recipe in ('near one-hot rows', 'row maxima in the last partial block'):
        k = r(B, nk, d)
        lo = 0 if recipe == 'near one-hot rows' else (nk - 1) // bk * bk      # the last (partial) key block of this form
        keys = torch.randint(lo, nk, (B, nq), generator=g, device=DEV)
        q = 1.5 * (64 / dh) ** 0.5 * k.gather(1, keys[..., None].expand(-1, -1, d)) + 0.1 * r(B, nq, d)
    elif recipe == 'logits rising block by block':                 # row i's logits rise (or fall) along the keys at its own rate
        k = 0.3 * k / 1.5 + (8.0 * torch.arange(nk, device=DEV) / nk)[None, :, None]
        q = (2 * torch.rand(B, nq, 1, generator=g, device=DEV) - 1) + 0.1 * r(B, nq, d)
    elif recipe == 'logits spanning +-80':                         # logit(i, j) ~ c_i t_j: the running maximum jumps by up to 160,
        e = torch.full((d,), dh ** -0.5, device=DEV)               # so the correction factors of the early blocks underflow
        t = (-80 + 160 * torch.arange(nk, device=DEV) / max(nk - 1, 1))[None, :, None] + 5 * r(B, nk, 1)
        c = torch.where(torch.rand(B, nq, 1, generator=g, device=DEV) < 0.5, -1.0, 1.0) * (0.5 + 0.5 * torch.rand(B, nq, 1, generator=g, device=DEV))
        q = c * e
        k = dh ** 0.5 * t.clamp(-80, 80) * e + 0.5 * r(B, nk, d)
    elif recipe == 'Q all zero':
        q = torch.zeros_like(q)
    elif recipe == 'next item dominates':
        q, k = _next_item_dominates(q, k, H, dh, nk, bk)
    else:
        assert recipe == 'random', recipe
    return q.contiguous(), k.contiguous(), v.contiguous()


def _next_item_dominates(q, k, H, dh, nk, bk):
    """The last, partial key block of item b loads the first keys of item b + 1 (the tensor-core forms' K map spans batch * nk
    rows).  Two of those keys get a logit 50 above the largest logit of item b for every query, so an unmasked one takes the whole
    softmax.  The last item's logits are all <= -50, so the zero-filled keys past its end (logit 0) would take it too."""
    B = q.shape[0]
    pad = -nk % bk
    assert pad, 'nk must not be a multiple of the key block'
    s = dh ** -0.5
    qh = _per_head(q, H)
    qh.sub_(qh.mean(-1, keepdim=True)).add_(1.0)                   # every query: sum of its channels per head = dh
    kh = _per_head(k, H)
    hot = sorted({0, min(pad, nk) - 1})
    logits_max = lambda b: (torch.einsum('ihc,jhc->hij', qh[b], kh[b]) * s).amax((1, 2))     # [H]
    for b in range(B - 1):
        gamma = (logits_max(b) + 50) / (s * dh)                    # s q . (gamma 1) = s gamma dh for every query
        kh[b + 1, hot] = gamma[:, None].expand(-1, dh)
    delta = (logits_max(B - 1) + 50) / (s * dh)
    kh[B - 1] -= delta[:, None]
    return q, k


# --------------------------------------------------------------------------------------------------------------------- launching
def _poisoned(n, dtype=torch.float32):
    return torch.full((n,), NAN, dtype=dtype, device=DEV)


def _fill(buf, t, rows, ld, cols, off=0):
    """buf[off + r ld + c] = t[r, c] for r < rows, c < cols"""
    buf[off:off + rows * ld].view(rows, ld)[:, :cols] = t.reshape(rows, cols)


def _split16(x2d):
    hi = torch.empty(x2d.shape, dtype=torch.float16, device=DEV)
    lo = torch.empty_like(hi)
    meta = torch.full((4,), NAN, device=DEV)
    _cabi.check(_cabi.lib().og_weight_split_f16(_p(x2d), None, x2d.shape[0], x2d.shape[1], _p(hi), _p(lo), _p(meta), _st()), 'split16')
    return hi, lo, meta


def _split_tf32(x):
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    _cabi.check(_cabi.lib().og_split_tf32(_p(x), _p(hi), _p(lo), x.numel(), _st()), 'og_split_tf32')
    return hi, lo


class Operands:
    """The operands of one form in HBM, laid out as `layout` says, every padding element NaN:
      'compact'   Q, K (V) with rows of d; V^T rows padded to the form's alignment;
      'padded'    ldq = ldo = d + 2, ldk = d + 4 (tf32) / + 8 (fp16) / + 3 (simt, also ldv), ldvt 8 past its alignment,
                  strideq / strideo 10 floats past nq ld;
      'qkv self'  (simt) Q | K | V interleaved in one [B n, 3d] buffer, as the fp32 forward's self layers pass it;
      'qkv cross' (simt) the same buffer over the rows of both images: Q of image 0, K and V of image 1.
    The tensor-core operands are split before their padding is poisoned; the fp16 form's q_amax is taken over Q alone."""

    def __init__(self, form, dh, H, q, k, v, layout='compact'):
        B, nq, d = q.shape
        nk = k.shape[1]
        self.form, self.dh, self.H, self.B, self.nq, self.nk, self.d = form, dh, H, B, nq, nk, d
        padded = layout == 'padded'
        self.ldo = d + (2 if padded else 0)
        self.so = nq * self.ldo + (10 if padded else 0)
        if layout.startswith('qkv'):
            assert form == 'simt'
            self_layer = layout == 'qkv self'
            assert not self_layer or nq == nk
            rows = B * nq + (0 if self_layer else B * nk)
            buf = _poisoned(rows * 3 * d)
            view = buf.view(rows, 3 * d)
            view[:B * nq, :d] = q.reshape(B * nq, d)
            kv0 = 0 if self_layer else B * nq
            view[kv0:kv0 + B * nk, d:2 * d] = k.reshape(B * nk, d)
            view[kv0:kv0 + B * nk, 2 * d:] = v.reshape(B * nk, d)
            self.bufs = (buf,)
            self.Q, self.q_off, self.ldq, self.sq = buf, 0, 3 * d, nq * 3 * d
            self.K, self.k_off, self.ldk, self.sk = buf, kv0 * 3 * d + d, 3 * d, nk * 3 * d
            self.V, self.v_off, self.ldv, self.sv = buf, kv0 * 3 * d + 2 * d, 3 * d, nk * 3 * d
            return
        self.ldq = d + (2 if padded else 0)
        self.sq = nq * self.ldq + (10 if padded else 0)
        self.Q, self.q_off = _poisoned(B * self.sq), 0
        for b in range(B):
            _fill(self.Q, q[b], nq, self.ldq, d, b * self.sq)
        if form == 'simt':
            self.ldk = self.ldv = d + (3 if padded else 0)
            self.sk = self.sv = nk * self.ldk
            self.K, self.V = _poisoned(B * self.sk), _poisoned(B * self.sv)
            self.k_off = self.v_off = 0
            _fill(self.K, k, B * nk, self.ldk, d)
            _fill(self.V, v, B * nk, self.ldv, d)
            return
        align = 4 if form == 'tf32' else 8
        self.ldk = d + (align if padded else 0)
        self.ldvt = (nk + align - 1) // align * align + (8 if padded else 0)
        kc = k.reshape(B * nk, d).contiguous()
        vtc = v.transpose(1, 2).reshape(B * d, nk).contiguous()
        dtype = torch.float32 if form == 'tf32' else torch.float16
        if form == 'tf32':
            ksplit, vsplit = _split_tf32(kc), _split_tf32(vtc)
        else:
            *ksplit, self.kmeta = _split16(kc)
            *vsplit, self.vmeta = _split16(vtc)
            self.qamax = torch.full((1,), NAN, device=DEV)
            _cabi.check(_cabi.lib().og_amax(_p(q), q.numel(), _p(self.qamax), _st()), 'og_amax')
        self.khi, self.klo = (_poisoned(B * nk * self.ldk, dtype) for _ in range(2))
        self.vthi, self.vtlo = (_poisoned(B * d * self.ldvt, dtype) for _ in range(2))
        for dst, src in ((self.khi, ksplit[0]), (self.klo, ksplit[1])):
            _fill(dst, src, B * nk, self.ldk, d)
        for dst, src in ((self.vthi, vsplit[0]), (self.vtlo, vsplit[1])):
            _fill(dst, src, B * d, self.ldvt, nk)

    def new_out(self):
        return _poisoned(self.B * self.so + TAIL_ROWS * self.ldo)

    def out_view(self, out):
        return out.as_strided((self.B, self.nq, self.d), (self.so, self.ldo, 1))

    def launch(self, out, b0=0, nb=None, h0=0, nh=None, out_amax=None):
        """items b0 .. b0 + nb - 1, heads h0 .. h0 + nh - 1, by pointer offsets and smaller batch / num_heads"""
        nb = self.B - b0 if nb is None else nb
        nh = self.H - h0 if nh is None else nh
        dh, lib = self.dh, _cabi.lib()
        c = h0 * dh
        q = _p(self.Q, self.q_off + b0 * self.sq + c)
        o = _p(out, b0 * self.so + c)
        if self.form == 'simt':
            rc = lib.og_attention_fwd(q, self.ldq, self.sq, _p(self.K, self.k_off + b0 * self.sk + c), self.ldk, self.sk,
                                      _p(self.V, self.v_off + b0 * self.sv + c), self.ldv, self.sv, o, self.ldo, self.so,
                                      nb, self.nq, self.nk, nh, dh, _cabi.OG_PREC_FP32, _st())
            return _cabi.check(rc, 'og_attention_fwd')
        # the V^T map counts nb * nh * dh rows from its base: a head subset is one batch item
        assert nh == self.H or nb == 1
        ko, vo = b0 * self.nk * self.ldk + c, (b0 * self.d + c) * self.ldvt
        kv = (_p(self.khi, ko), _p(self.klo, ko), self.ldk)
        vt = (_p(self.vthi, vo), _p(self.vtlo, vo), self.ldvt)
        if self.form == 'tf32':
            rc = lib.og_attention_tc_fwd(q, self.ldq, self.sq, *kv, *vt, o, self.ldo, self.so, nb, self.nq, self.nk, nh, dh, _st())
            return _cabi.check(rc, 'og_attention_tc_fwd')
        rc = lib.og_attention_f16_fwd(q, self.ldq, self.sq, _p(self.qamax), *kv, _p(self.kmeta), *vt, _p(self.vmeta), o, self.ldo, self.so,
                                      _p(out_amax), nb, self.nq, self.nk, nh, dh, 0, _st())
        return _cabi.check(rc, 'og_attention_f16_fwd')


def _unwritten(ops, out):
    """the output elements no launch may write: padding columns, gaps between batch items, rows past the last item"""
    mask = torch.ones(out.shape, dtype=torch.bool, device=DEV)
    mask.as_strided((ops.B, ops.nq, ops.d), (ops.so, ops.ldo, 1)).fill_(False)
    return out[mask]


# --------------------------------------------------------------------------------------------------------------------- case table
def _edges(block):
    """1, block - 1, block, block + 1, and 3 / 4 blocks +- 1 (the K / V ring has 3 stages)"""
    return [1, block - 1, block, block + 1, 3 * block - 1, 3 * block + 1, 4 * block - 1, 4 * block + 1]


def _cases():
    cases = []
    add = lambda form, dh, B, H, nq, nk, recipe, layout='compact': cases.append(
        pytest.param(form, dh, B, H, nq, nk, recipe, layout, id=f'{form}-dh{dh}-B{B}H{H}-{nq}x{nk}-{recipe}' + (f'-{layout}' if layout != 'compact' else '')))
    for form, dh in FORM_DH:
        bq, bk = BLOCKS[form]
        # tile edges: every nk edge once, paired with the nq edges in turn; B 1 .. 3, H 1 .. 4
        for j, nk in enumerate(_edges(bk)):
            nq = _edges(bq)[(3 * j) % 8]
            add(form, dh, 1 + j % 3, 1 + j % 4, nq, nk, 'tile edges')
        # keys of the next item dominate: a partial last block of a few keys, and one of a single key
        add(form, dh, 3, 2, 100, 2 * bk + 5, 'next item dominates')
        add(form, dh, 2, 1, bq + 3, 1, 'next item dominates')
        add(form, dh, 3, 2, bq + 2, bk + 37, 'random', 'padded')
        for recipe in MAGNITUDES:
            add(form, dh, 1, 2, 1000, 4097, recipe)
    add('simt', 64, 2, 2, 150, 150, 'random', 'qkv self')
    add('simt', 16, 2, 4, 150, 97, 'random', 'qkv cross')
    add('simt', 8, 3, 4, 70, 130, 'next item dominates', 'qkv cross')
    # many tiles at the benchmark's shapes: C5 (d 128, 4 heads) self and cross layers, C3 (d 256, 4 heads) self layers at B 2
    for nq, nk in ((4096, 4096), (4096, 1024), (1024, 4096)):
        add('tf32', 32, 1, 4, nq, nk, 'many tiles')
    for form in ('fp16', 'tf32', 'simt'):
        add(form, 64, 2, 4, 2048, 2048, 'many tiles')
    for dh in (8, 16):                                             # the fp32 kernel's long key loops at small head dims
        add('simt', dh, 2, 4, 300, 4097, 'many tiles')
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize('form,dh,B,H,nq,nk,recipe,layout', _cases())
def test_attention_matches_float64(form, dh, B, H, nq, nk, recipe, layout):
    seed = 1000 * dh + 10 * B + H + nq + 7 * nk
    q, k, v = _inputs('random' if recipe in ('tile edges', 'many tiles') else recipe, form, B, H, nq, nk, dh, seed)
    ops = Operands(form, dh, H, q, k, v, layout)
    out = ops.new_out()
    out_amax = torch.zeros(1, device=DEV) if form == 'fp16' else None
    ops.launch(out, out_amax=out_amax)
    got = ops.out_view(out).double()
    ref = _reference(q, k, v, H)
    ref32_err = float((_reference(q, k, v, H, torch.float32).double() - ref).abs().max())
    scale = float(ref.abs().max())
    bound = CONTRACT[form] * scale
    if recipe in ILL_CONDITIONED:
        bound = max(bound, 4 * ref32_err)
    finite = bool(torch.isfinite(got).all())
    err = float((got - ref).abs().max()) if finite else NAN
    _report(f'{form} dh={dh} B{B} H{H} {nq}x{nk} {recipe} {layout}', err, bound, f'; float32 reference {ref32_err:.3e}, max |ref| {scale:.3e}')
    assert finite, 'non-finite output'
    assert err <= bound
    if recipe == 'Q all zero':                                     # uniform weights: the mean of V
        assert (ref - v.double().mean(1, keepdim=True)).abs().max() <= 1e-12 * v.abs().max()
    assert bool(torch.isnan(_unwritten(ops, out)).all()), 'written outside the output rows / columns'
    if form == 'fp16':
        assert float(out_amax) == float(ops.out_view(out).abs().max())     # the tracked amax of the output


# --------------------------------------------------------------------------------------------------------------------- b. position
@pytest.mark.gpu
@pytest.mark.parametrize('form,dh', [pytest.param(f, dh, id=f'{f}-dh{dh}-B3H4-200x333') for f, dh in FORM_DH])
def test_position_independence_and_determinism(form, dh):
    """A CTA's result does not depend on the batch item or head slice it is launched with: one launch over B items = B launches of
    one item (pointer offsets), one launch over H heads = a launch over a head subset (pointer offset h dh, num_heads reduced), and
    two identical launches agree, all bit for bit.  The tensor-core forms' V^T map counts batch * num_heads * head_dim rows from
    its base, so their head subsets are launched one item at a time."""
    B, H, nq, nk = 3, 4, 200, 333
    q, k, v = _inputs('random', form, B, H, nq, nk, dh, 77)
    ops = Operands(form, dh, H, q, k, v, 'padded')
    full, again = ops.new_out(), ops.new_out()
    ops.launch(full)
    ops.launch(again)
    view = ops.out_view
    assert torch.equal(view(full), view(again)), 'two identical launches differ'
    per_item = ops.new_out()
    for b in range(B):
        ops.launch(per_item, b0=b, nb=1)
    assert torch.equal(view(full), view(per_item)), 'per-item launches differ from one launch over the batch'
    h0, nh = 1, 2
    sub = ops.new_out()
    items = range(B) if form == 'simt' else [B - 1]
    if form == 'simt':
        ops.launch(sub, h0=h0, nh=nh)
    else:
        ops.launch(sub, b0=B - 1, nb=1, h0=h0, nh=nh)
    cols = slice(h0 * dh, (h0 + nh) * dh)
    for b in items:
        assert torch.equal(view(full)[b, :, cols], view(sub)[b, :, cols]), f'head subset {h0} .. {h0 + nh - 1} of item {b} differs'
    sub_rest = view(sub).clone()
    sub_rest[list(items), :, cols] = NAN
    assert bool(torch.isnan(sub_rest).all()) and bool(torch.isnan(_unwritten(ops, sub)).all()), 'a head subset wrote outside its columns'
    print(f'\n[{form} dh={dh} B{B} H{H} {nq}x{nk}] repeat, per-item and head-subset launches bit-identical')


@pytest.mark.gpu
def test_forms_agree_at_head_dim_64():
    """The three forms on the same operands at head_dim 64 agree within the sum of their contracts (relative to max |ref|)."""
    B, H, nq, nk = 2, 4, 300, 700
    q, k, v = _inputs('random', 'simt', B, H, nq, nk, 64, 78)
    ref = _reference(q, k, v, H)
    scale = float(ref.abs().max())
    outs = {}
    for form in BLOCKS:
        ops = Operands(form, 64, H, q, k, v)
        out = ops.new_out()
        ops.launch(out)
        outs[form] = ops.out_view(out).double()
    fails = []
    for a, b in (('simt', 'tf32'), ('simt', 'fp16'), ('tf32', 'fp16')):
        err, bound = float((outs[a] - outs[b]).abs().max()), (CONTRACT[a] + CONTRACT[b]) * scale
        _report(f'{a} vs {b} dh=64 B{B} H{H} {nq}x{nk}', err, bound)
        if not err <= bound:
            fails.append(f'{a} vs {b}: {err:.3e} > {bound:.3e}')
    assert not fails, '\n'.join(fails)


# --------------------------------------------------------------------------------------------------------------------- c. gradient
def _poisoned_ops(precision):
    """the training operators, with every buffer they leave uninitialised NaN: an element of the backward schedule that is read
    before it is written, or never written, shows in its result"""
    from openglue_b200._ops import _Ops

    class PoisonedOps(_Ops):
        def empty(self, *shape):
            return torch.full(shape, NAN, dtype=torch.float32, device=self.dev)
    return PoisonedOps(torch.device(DEV), precision)


def _attention_bwd(precision, B, H, nq, nk, q, k, v, do):
    """TrainStep._attention_bwd on a stand-in holding exactly what it reads"""
    from openglue_b200.training import TrainStep
    d = q.shape[1]
    step = types.SimpleNamespace(ops=_poisoned_ops(precision), d=d, H=H, B=B, N=[nq, nk])
    call = dict(iq=0, ikv=1, q=q, k=k, v=v)
    return TrainStep._attention_bwd(step, call, do)


def _autograd(B, H, nq, nk, q, k, v, do, dtype):
    d = q.shape[1]
    leaves = [t.detach().to(dtype).requires_grad_() for t in (q, k, v)]
    o = _reference(leaves[0].view(B, nq, d), leaves[1].view(B, nk, d), leaves[2].view(B, nk, d), H, dtype)
    o.backward(do.to(dtype).view(B, nq, d))
    return [t.grad for t in leaves]


def _grad_inputs(B, H, nq, nk, dh, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    d = H * dh
    r = lambda *s: torch.randn(*s, generator=g, device=DEV)
    return 1.5 * r(B * nq, d), 1.5 * r(B * nk, d), r(B * nk, d), r(B * nq, d)


PRECISIONS = {'fp32': _cabi.OG_PREC_FP32, 'tf32x3': _cabi.OG_PREC_TF32X3}
GRAD_SHAPES = [(37, 50), (65, 131), (99, 129)]         # nq, nk not multiples of 4; nq = 65 and nk = 129 are 1 mod 64


@pytest.mark.gpu
@pytest.mark.parametrize('nq,nk', GRAD_SHAPES, ids=[f'B2-{nq}x{nk}' for nq, nk in GRAD_SHAPES])
@pytest.mark.parametrize('dh,H', [(8, 3), (16, 2), (32, 3), (64, 2)], ids=['dh8-H3', 'dh16-H2', 'dh32-H3', 'dh64-H2'])
@pytest.mark.parametrize('prec', list(PRECISIONS))
def test_attention_gradient_matches_autograd(prec, dh, H, nq, nk):
    """dq, dk, dv of TrainStep._attention_bwd against float64 autograd through softmax(q k^T s) v for a random dO.  Per tensor:
    |got - ref64| <= max(4 |ref32 - ref64|, 1e-5 max |ref64|)."""
    B = 2
    q, k, v, do = _grad_inputs(B, H, nq, nk, dh, 100 * dh + nq + nk)
    got = _attention_bwd(PRECISIONS[prec], B, H, nq, nk, q, k, v, do)
    ref64 = _autograd(B, H, nq, nk, q, k, v, do, torch.float64)
    ref32 = _autograd(B, H, nq, nk, q, k, v, do, torch.float32)
    fails = []
    for name, gt, r64, r32 in zip(('dq', 'dk', 'dv'), got, ref64, ref32):
        bound = max(4 * float((r32.double() - r64).abs().max()), 1e-5 * float(r64.abs().max()))
        err = float((gt.double() - r64).abs().max()) if bool(torch.isfinite(gt).all()) else NAN
        _report(f'attention backward {prec} {name} dh={dh} H{H} B{B} {nq}x{nk}', err, bound)
        if not err <= bound:
            fails.append(f'{name}: error {err:.3e}, bound {bound:.3e}')
    assert not fails, '\n'.join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize('dh,H', [(8, 3), (16, 4), (32, 3), (64, 2)], ids=['dh8-H3', 'dh16-H4', 'dh32-H3', 'dh64-H2'])
@pytest.mark.parametrize('prec', list(PRECISIONS))
def test_attention_gradient_of_one_head(prec, dh, H):
    """dO zero outside head h: the other heads' dq, dk, dv are exactly zero, and head h's match float64 autograd."""
    B, nq, nk = 2, 37, 130
    q, k, v, do = _grad_inputs(B, H, nq, nk, dh, 7 * dh + H)
    for h in range(H):
        cols = slice(h * dh, (h + 1) * dh)
        doh = torch.zeros_like(do)
        doh[:, cols] = do[:, cols]
        got = _attention_bwd(PRECISIONS[prec], B, H, nq, nk, q, k, v, doh)
        ref64 = _autograd(B, H, nq, nk, q, k, v, doh, torch.float64)
        ref32 = _autograd(B, H, nq, nk, q, k, v, doh, torch.float32)
        for name, gt, r64, r32 in zip(('dq', 'dk', 'dv'), got, ref64, ref32):
            rest = gt.clone()
            rest[:, cols] = 0
            assert torch.equal(rest, torch.zeros_like(rest)), f'head {h}: {name} of the other heads is not exactly zero'
            bound = max(4 * float((r32.double() - r64).abs().max()), 1e-5 * float(r64.abs().max()))
            err = float((gt[:, cols].double() - r64[:, cols]).abs().max()) if bool(torch.isfinite(gt).all()) else NAN
            _report(f'attention backward {prec} {name} dh={dh} H{H}, dO on head {h} only', err, bound)
            assert err <= bound, f'head {h}: {name}'
