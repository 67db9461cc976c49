"""The SuperPoint front-end (csrc/superpoint.cuh, openglue_b200/superpoint.py) operator by operator and at real image sizes.

1. Every C-ABI entry point of the front-end against an exact or float64 torch restatement of the operation it implements, at the
   shapes and edges where such kernels go wrong (odd sizes, both vector paths, offsets past 2^31 floats, plateaus and ties, edge
   peaks, lists over capacity, sorts of up to 16384 candidates).  Outputs are NaN-poisoned, with a guard region after them that
   must stay poisoned.
2. The post-processing chain (SuperPointNet._keypoints) at 240x320 .. 720x960 on injected layer outputs, against fixtures minted
   by the unmodified reference forward (oracle/gen_golden_superpoint_post.py).
3. The whole network at 480x640 and 720x960 against a float64 restatement of the reference's layers, run on the device.

Every GPU case prints what it measured next to its bound (run with -s).
"""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'oracle'))
from gen_golden_superpoint_post import CASES as POST_CASES, inputs_sha256, post_inputs  # noqa: E402
from test_superpoint import _decisions, _disagreements  # noqa: E402
from openglue_b200._cabi import ptr as _p, stream as _st  # noqa: E402

DEV = 'cuda:0'
U = 2.0 ** -24                  # unit roundoff of float32
GUARD = 1024                    # poisoned elements after every output buffer
INT_POISON = -0x5a5a5a5a
SP_MAX_CAND = 16384             # csrc/common.cuh (CTA_TOPK_MAX): the sort capacity of og_sp_select
OG_EUNSUPPORTED = -2


def _lib():
    from openglue_b200 import _cabi
    return _cabi.lib()


def _check(rc, what):
    from openglue_b200 import _cabi
    _cabi.check(rc, what)


def _poisoned(n, dtype=torch.float32):
    """a device buffer of n elements followed by GUARD guard elements, all NaN (integers: INT_POISON)"""
    return torch.full((n + GUARD,), float('nan') if dtype.is_floating_point else INT_POISON, dtype=dtype, device=DEV)


def _untouched(t):
    return bool((torch.isnan(t) if t.is_floating_point() else t == INT_POISON).all())


def _n2(n):
    return 1 << max(n - 1, 0).bit_length()


def _report(tag, err, bound):
    print(f'\n[{tag}] max error {err:.3e}, bound {bound:.3e}')


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------------------------------
# restatements (plain torch; float32 where the operation is exact, float64 otherwise)

def im2col_ref(x):
    """x [B, H, W, C] -> [B H W, 9 C] with column (3 ky + kx) C + c: F.unfold (k 3, pad 1), whose rows are c 9 + tap, reordered"""
    B, H, W, Cc = x.shape
    u = F.unfold(x.permute(0, 3, 1, 2), 3, padding=1)
    return u.view(B, Cc, 9, H * W).permute(0, 3, 2, 1).reshape(B * H * W, 9 * Cc)


def pixel_heat(probs):
    """cell probabilities [B, Hc, Wc, 65] -> pixel scores [B, 8 Hc, 8 Wc] (the pixel shuffle of model.py:86-88)"""
    B, Hc, Wc, _ = probs.shape
    return probs[..., :64].reshape(B, Hc, Wc, 8, 8).permute(0, 1, 3, 2, 4).reshape(B, 8 * Hc, 8 * Wc)


def cell_probs(heat, last=0.0):
    """inverse of pixel_heat; channel 64 ("no keypoint") = `last`"""
    B, H, W = heat.shape
    p = heat.reshape(B, H // 8, 8, W // 8, 8).permute(0, 1, 3, 2, 4).reshape(B, H // 8, W // 8, 64)
    return torch.cat([p, torch.full_like(p[..., :1], last)], -1).contiguous()


def nms_threshold_borders(heat, nms, thr, border):
    """kornia nms2d (x * (x > max(0, the other k*k - 1 values of the replicate-padded window)); oracle/gen_golden_superpoint.py::nms2d),
    F.threshold(s, thr, 0) (model.py:93) and remove_borders (utils.py:4-11) on [B, H, W]: the score where the pixel is kept, else 0"""
    B, H, W = heat.shape
    r = nms // 2
    mx = torch.zeros_like(heat)                                         # the centre channel of nms2d's kernel is all zero
    if nms > 1:
        win = F.pad(heat[:, None], [r, r, r, r], mode='replicate')[:, 0].unfold(1, nms, 1).unfold(2, nms, 1).reshape(B, H, W, nms * nms)
        c = nms * nms // 2
        mx = torch.cat([win[..., :c], win[..., c + 1:]], -1).amax(-1).clamp_min(0)
    s = F.threshold(heat * (heat > mx).to(heat.dtype), thr, 0.)
    inb = torch.zeros_like(s, dtype=torch.bool)
    inb[:, border:H - border, border:W - border] = True
    return torch.where(inb, s, torch.zeros_like(s))


def sample_desc_ref(coarse, kpts, cell, dtype):
    """sample_desc_from_points (utils.py:14-31) for one image in `dtype`: coarse [Hc, Wc, D] (NHWC), kpts [n, 2] (x, y) -> [n, D]"""
    Hc, Wc, D = coarse.shape
    H, W = Hc * cell, Wc * cell
    pts = kpts.to(dtype) - cell / 2 + 0.5
    pts = pts / torch.tensor([W - cell / 2 - 0.5, H - cell / 2 - 0.5], dtype=dtype, device=kpts.device)
    pts = pts.view(1, 1, -1, 2) * 2 - 1
    d = F.grid_sample(coarse.permute(2, 0, 1)[None].to(dtype), pts, align_corners=False).view(D, -1)
    return F.normalize(d, p=2, dim=0).t()


def layers_ref(sd, image, dtype, bn=False):
    """The reference's _forward_layers (model.py:61-78; SuperPointNetBn model.py:180-199) from its state dict, in `dtype`:
    image [B, 1, H, W] -> (descriptor map [B, D, Hc, Wc] with unit columns, pixel heat map [B, H, W])"""
    t = lambda k: sd[k].to(device=image.device, dtype=dtype)

    def conv(x, name, relu=True):
        w = t(name + '.weight')
        y = F.conv2d(x, w, t(name + '.bias'), padding=w.shape[-1] // 2)
        if bn:
            b = 'bn' + name[4:]
            y = F.batch_norm(y, t(b + '.running_mean'), t(b + '.running_var'), t(b + '.weight'), t(b + '.bias'), False, 0.0, 1e-5)
        return y.relu() if relu else y
    x = image.to(dtype)
    for i in range(4):
        x = conv(conv(x, f'conv{i + 1}a'), f'conv{i + 1}b')
        if i != 3:
            x = F.max_pool2d(x, 2, 2)
    desc = conv(conv(x, 'convDa'), 'convDb', relu=False)
    desc = desc.div(torch.norm(desc, p=2, dim=1).unsqueeze(1))
    cell = F.softmax(conv(conv(x, 'convPa'), 'convPb', relu=False), 1)[:, :-1]
    return desc, pixel_heat(cell.permute(0, 2, 3, 1))


# =====================================================================================================================
# 1. operators
# ---------------------------------------------------------------------------------------------------------------------
# og_sp_im2col3x3: bit-exact against F.unfold.  C % 4 == 0 takes the float4 path, other C the scalar path.
IM2COL_CASES = [(3, 15, 20, 1), (3, 15, 20, 3), (3, 15, 20, 64), (3, 15, 20, 128), (3, 45, 60, 3), (3, 45, 60, 64),
                (3, 1, 1, 1), (3, 1, 1, 64), (3, 2, 3, 3), (3, 2, 3, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize('B,H,W,Cc', IM2COL_CASES)
def test_im2col3x3_is_unfold(B, H, W, Cc):
    x = torch.randn(B, H, W, Cc, generator=_gen(H * 1000 + Cc)).to(DEV)
    n = B * H * W * 9 * Cc
    out = _poisoned(n)
    _check(_lib().og_sp_im2col3x3(_p(x), B, H, W, Cc, _p(out), _st()), 'og_sp_im2col3x3')
    ref = im2col_ref(x)
    assert torch.equal(out[:n].view_as(ref), ref)
    assert _untouched(out[n:])


@pytest.mark.gpu
def test_im2col3x3_past_2_31_floats():
    """B = 6 images of 720 x 960 x 64: the output is 2.39e9 floats, so its offsets pass 2^31.  The image holding the row that crosses
    2^31 and the first and last images are compared against F.unfold; every element of the others must have been written."""
    B, H, W, Cc = 6, 720, 960, 64
    row = 9 * Cc
    n = B * H * W * row
    torch.cuda.empty_cache()                                             # blocks earlier tests left in torch's cache count as free
    free = torch.cuda.mem_get_info()[0]
    need = 4 * (n + B * H * W * Cc) + n + 3 * 4 * H * W * row + (1 << 30)
    if free < need:
        pytest.skip(f'needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free')
    x = torch.rand(B, H, W, Cc, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5)) - 0.5
    out = _poisoned(n)
    _check(_lib().og_sp_im2col3x3(_p(x), B, H, W, Cc, _p(out), _st()), 'og_sp_im2col3x3')
    p_cross = (1 << 31) // row
    b_cross = p_cross // (H * W)
    print(f'\n[im2col 6 x 720 x 960 x 64] {n} floats out; offset 2^31 falls in output row {p_cross} (image {b_cross}, '
          f'y {p_cross % (H * W) // W}, x {p_cross % W})')
    assert n > (1 << 31)
    for b in sorted({0, b_cross, B - 1}):
        ref = im2col_ref(x[b:b + 1])
        assert torch.equal(out[b * H * W * row:(b + 1) * H * W * row].view_as(ref), ref), b
        del ref
    assert not bool(torch.isnan(out[:n]).any())
    assert _untouched(out[n:])
    del out, x
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# og_sp_maxpool2x2: bit-exact against F.max_pool2d
@pytest.mark.gpu
@pytest.mark.parametrize('B,H,W,Cc', [(3, 30, 42, 3), (3, 30, 42, 64), (2, 18, 26, 128), (1, 2, 2, 64), (2, 6, 10, 1)])
def test_maxpool2x2_is_max_pool2d(B, H, W, Cc):
    g = _gen(H * 100 + Cc)
    x = torch.randn(B, H, W, Cc, generator=g) - 1.0                      # mostly negative: a zero-initialised max would show
    x[0] = -torch.rand(H, W, Cc, generator=g) - 0.5                     # all negative
    x = x.to(DEV)
    n = B * (H // 2) * (W // 2) * Cc
    out = _poisoned(n)
    _check(_lib().og_sp_maxpool2x2(_p(x), B, H, W, Cc, _p(out), _st()), 'og_sp_maxpool2x2')
    ref = F.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).contiguous()
    assert torch.equal(out[:n].view_as(ref), ref)
    assert _untouched(out[n:])


# ---------------------------------------------------------------------------------------------------------------------
# og_row_normalize: mode 0 = x / ||x|| (model.py:72-73: zero rows give NaN), mode 1 = F.normalize (eps 1e-12: zero rows give 0).
# Error model: per lane a recursive sum of ceil(C / 32) squares, a 5-level warp tree, sqrt, division: relative error of every
# output element <= (ceil(C / 32) + 8) u.
@pytest.mark.gpu
@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('Cc', [256, 65, 33, 1])
def test_row_normalize(Cc, mode):
    rows = 10 ** 6
    g = torch.Generator(device=DEV).manual_seed(Cc + 7 * mode)
    x = torch.randn(rows, Cc, device=DEV, generator=g)
    zero, tiny = [0, 4097, rows - 1], [3, 5, rows - 2]
    x[zero] = 0.0
    x[tiny] *= 1e-14                                                     # norm below F.normalize's eps
    buf = _poisoned(rows * Cc)
    buf[:rows * Cc] = x.view(-1)
    _check(_lib().og_row_normalize(_p(buf), rows, Cc, mode, 1e-12, _st()), 'og_row_normalize')
    y = buf[:rows * Cc].view(rows, Cc)
    x64 = x.double()
    ref = x64 / x64.norm(dim=1, keepdim=True) if mode == 0 else F.normalize(x64, p=2, dim=1, eps=1e-12)
    nz = torch.ones(rows, dtype=torch.bool, device=DEV)
    nz[zero] = False
    if mode == 0:
        assert bool(torch.isnan(y[zero]).all())
    else:
        assert bool((y[zero] == 0).all())
    rel = float(((y[nz].double() - ref[nz]).abs() / ref[nz].abs().clamp_min(1e-300)).max())
    bound = (math.ceil(Cc / 32) + 8) * U
    _report(f'row_normalize C {Cc} mode {mode}, {rows} rows (relative)', rel, bound)
    assert rel <= bound
    assert _untouched(buf[rows * Cc:])


# ---------------------------------------------------------------------------------------------------------------------
# og_sp_heat_nms: bit-exact against the restatement, from quantised probabilities (k / 64: plateaus and exact ties) with planted
# peaks on the edge rows and columns and in the corners.  Under replicate padding an edge pixel compares against itself, so it
# never survives when nms_kernel > 1.
def _nms_input(B, Hc, Wc, seed):
    g = _gen(seed)
    heat = torch.randint(0, 65, (B, 8 * Hc, 8 * Wc), generator=g).float() / 64
    H, W = 8 * Hc, 8 * Wc
    for b in range(B):
        peaks = [(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1)]
        peaks += [(0, int(x)) for x in torch.randint(0, W, (3,), generator=g)] + [(H - 1, int(x)) for x in torch.randint(0, W, (3,), generator=g)]
        peaks += [(int(y), 0) for y in torch.randint(0, H, (3,), generator=g)] + [(int(y), W - 1) for y in torch.randint(0, H, (3,), generator=g)]
        for y, x in peaks:                                               # a strict maximum of its 9 x 9 window, itself excepted
            heat[b, max(y - 4, 0):y + 5, max(x - 4, 0):x + 5] *= 0.5
        for y, x in peaks:
            heat[b, y, x] = 1.0
    return heat


@pytest.mark.gpu
@pytest.mark.parametrize('nms', [1, 3, 5, 9])
def test_heat_nms_is_nms2d_threshold_borders(nms):
    lib = _lib()
    for Hc, Wc in [(5, 7), (9, 13)]:
        heat = _nms_input(3, Hc, Wc, 100 * nms + Hc)
        probs = cell_probs(heat, last=0.25).to(DEV)
        B, H, W = heat.shape
        for border in (0, 4, 9):
            for thr in (0.0, 0.005, 0.02):
                out = _poisoned(B * H * W)
                _check(lib.og_sp_heat_nms(_p(probs), B, Hc, Wc, nms, thr, border, _p(out), _st()), 'og_sp_heat_nms')
                ref = nms_threshold_borders(heat, nms, thr, border)
                if nms > 1 and border == 0:                              # the planted edge peaks are all suppressed
                    assert not bool(ref[:, [0, -1], :].any()) and not bool(ref[:, :, [0, -1]].any())
                got = out[:B * H * W].view(B, H, W).cpu()
                assert torch.equal(got, ref), (Hc, Wc, border, thr, int((got != ref).sum()))
                assert _untouched(out[B * H * W:])
                print(f'nms {nms} {H}x{W} border {border} thr {thr}: survivors {[(int((r != 0).sum())) for r in ref]}')


def test_nms_restatement_is_gen_golden_nms2d():
    """the restatement above agrees with the conv-based nms2d the fixtures were minted with (float64: the one-hot conv is exact)"""
    from gen_golden_superpoint import nms2d
    heat = _nms_input(2, 5, 7, 3).double()
    for k in (1, 3, 5, 9):
        assert torch.equal(nms_threshold_borders(heat, k, 0.0, 0), nms2d(heat[:, None], (k, k))[:, 0])


# ---------------------------------------------------------------------------------------------------------------------
# og_sp_compact: torch.nonzero order, bit-exact indices / scores / counts; an image over capacity reports its true count, stores
# its first cap candidates and leaves the other images alone
def _sparse_rows(B, HW, densities, seed):
    g = _gen(seed)
    rows = torch.zeros(B, HW)
    for b, d in enumerate(densities):
        on = torch.rand(HW, generator=g) < d
        v = (torch.randint(1, 65, (HW,), generator=g).float() / 64) * torch.where(torch.rand(HW, generator=g) < 0.2, -1.0, 1.0)
        rows[b] = torch.where(on, v, torch.where(torch.rand(HW, generator=g) < 0.1, -0.0, 0.0))   # -0.0 is zero too
    return rows


COMPACT_CASES = {                # name: (B, HW, cap, per-image densities)
    'hw1': (3, 1, 1, [1.0, 0.0, 0.0]),
    'hw1000': (3, 1000, 1000, [0.3, 0.0, 1.0]),
    'hw3001': (3, 3001, 3001, [0.01, 0.5, 1.0]),
    'hw307200': (2, 480 * 640, SP_MAX_CAND, [1 / 81, 1 / 49]),
    'over_cap': (3, 5000, 300, [0.02, 0.5, 0.05]),
}


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(COMPACT_CASES))
def test_compact_is_nonzero(name):
    B, HW, cap, dens = COMPACT_CASES[name]
    rows = _sparse_rows(B, HW, dens, len(name) * HW)
    heat = rows.to(DEV)
    idx, sc, cnt = _poisoned(B * cap, torch.int32), _poisoned(B * cap), _poisoned(B, torch.int32)
    _check(_lib().og_sp_compact(_p(heat), B, HW, cap, _p(idx), _p(sc), _p(cnt), _st()), 'og_sp_compact')
    idx, sc, cnt = idx.cpu(), sc.cpu(), cnt.cpu()
    counts = []
    for b in range(B):
        nz = torch.nonzero(rows[b])[:, 0]
        counts.append(nz.numel())
        k = min(nz.numel(), cap)
        assert int(cnt[b]) == nz.numel()
        assert torch.equal(idx[b * cap:b * cap + k].long(), nz[:k])
        assert torch.equal(sc[b * cap:b * cap + k], rows[b, nz[:k]])
        assert _untouched(idx[b * cap + k:(b + 1) * cap]) and _untouched(sc[b * cap + k:(b + 1) * cap])
    assert _untouched(idx[B * cap:]) and _untouched(sc[B * cap:]) and _untouched(cnt[B:])
    print(f'\ncompact {name}: HW {HW}, cap {cap}, counts {counts}' + (' (over cap)' if max(counts) > cap else ''))
    if name == 'over_cap':
        assert counts[1] > cap and counts[0] < cap and counts[2] < cap


# ---------------------------------------------------------------------------------------------------------------------
# og_sp_select: mode 0 keeps the candidate order, mode 1 is a stable descending sort on (score, candidate position): ties go to
# the lower position.  Caller contract, not exercised here: n_out[b] <= count[b] (a larger n_out reads unwritten candidates).
def _select_ref(idx, sc, cnt, n, mode, W):
    order = torch.sort(sc[:cnt], descending=True, stable=True).indices[:n] if mode else torch.arange(n)
    p = idx[order].long()
    return torch.stack([p % W, p // W], -1).float(), sc[order]


SELECT_CASES = {                 # name: (counts, modes, n_out, quantised score levels per image (0: continuous))
    'small': ([1, 2, 1023, 1025], [1, 0, 1, 1], [1, 2, 1000, 1025], [0, 8, 32, 4]),
    'n2_4096': ([4097, 3000, 2049], [1, 1, 0], [4097, 100, 2049], [16, 0, 0]),
    'n2_16384': ([16384, 16383, 4097, 9000], [1, 1, 1, 0], [16384, 2048, 4000, 8999], [32, 0, 8, 0]),
}


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(SELECT_CASES))
def test_select_is_stable_topk(name):
    counts, modes, n_out, levels = SELECT_CASES[name]
    B, cap, H, W = len(counts), SP_MAX_CAND, 720, 960
    out_cap = max(n_out) + 3                                             # rows past every n_out stay untouched
    g = _gen(len(name))
    idx = torch.full((B, cap), INT_POISON, dtype=torch.int32)
    sc = torch.full((B, cap), float('nan'))
    for b, (c, q) in enumerate(zip(counts, levels)):
        idx[b, :c] = torch.randperm(H * W, generator=g)[:c].sort().values.int()
        sc[b, :c] = (torch.randint(1, q + 1, (c,), generator=g).float() / q) if q else torch.rand(c, generator=g)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=DEV)
    args = [idx.to(DEV), sc.to(DEV), i32(counts), i32(n_out), i32(modes)]          # held: their memory must outlive the launch
    kp, so = _poisoned(B * out_cap * 2), _poisoned(B * out_cap)
    lib = _lib()
    before = lib.og_last_forward_launches()
    _check(lib.og_sp_select(*[_p(t) for t in args], B, cap, W, out_cap, max(counts), _p(kp), _p(so), _st()), 'og_sp_select')
    assert lib.og_last_forward_launches() == before + 1
    kp, so = kp.cpu(), so.cpu()
    for b in range(B):
        rk, rs = _select_ref(idx[b], sc[b], counts[b], n_out[b], modes[b], W)
        n = n_out[b]
        got_k = kp[b * out_cap * 2:(b * out_cap + n) * 2].view(n, 2)
        assert torch.equal(got_k, rk), (b, int((got_k != rk).any(-1).sum()))
        assert torch.equal(so[b * out_cap:b * out_cap + n], rs)
        assert _untouched(kp[(b * out_cap + n) * 2:(b + 1) * out_cap * 2]) and _untouched(so[b * out_cap + n:(b + 1) * out_cap])
        ties = int((rs[1:] == rs[:-1]).sum()) if modes[b] else 0
        print(f'select {name} image {b}: count {counts[b]}, n2 {_n2(counts[b])}, mode {modes[b]}, n_out {n}, tied neighbours {ties}')
    assert _untouched(kp[B * out_cap * 2:]) and _untouched(so[B * out_cap:])


@pytest.mark.gpu
def test_select_refuses_more_than_16384_candidates():
    lib = _lib()
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32, device=DEV)
    idx, sc = torch.zeros(SP_MAX_CAND, dtype=torch.int32, device=DEV), torch.zeros(SP_MAX_CAND, device=DEV)
    kp, so = _poisoned(2), _poisoned(1)
    before = lib.og_last_forward_launches()
    count, n_out, mode = i32(SP_MAX_CAND), i32(1), i32(1)
    rc = lib.og_sp_select(_p(idx), _p(sc), _p(count), _p(n_out), _p(mode), 1, SP_MAX_CAND, 960, 1, SP_MAX_CAND + 1, _p(kp), _p(so), _st())
    torch.cuda.synchronize()
    assert rc == OG_EUNSUPPORTED
    assert lib.og_last_forward_launches() == before
    assert _untouched(kp) and _untouched(so)


# ---------------------------------------------------------------------------------------------------------------------
# og_sp_sample_desc: float64 restatement of sample_desc_from_points; bound = 2 x the distance of the same restatement run in float32
def _sample_kpts(Hc, Wc, n, seed):
    H, W = 8 * Hc, 8 * Wc
    border = [(x, 0) for x in range(W)] + [(x, H - 1) for x in range(W)] + [(0, y) for y in range(H)] + [(W - 1, y) for y in range(H)]
    g = _gen(seed)
    frac = torch.rand(n, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0])
    return torch.cat([torch.tensor(border, dtype=torch.float32), frac])


@pytest.mark.gpu
@pytest.mark.parametrize('Hc,Wc,D', [(5, 7, 256), (6, 9, 65), (3, 4, 1), (1, 6, 256), (4, 1, 65), (1, 1, 1)])
def test_sample_desc(Hc, Wc, D):
    B, cell = 3, 8
    coarse = (2 * torch.rand(B, Hc, Wc, D, generator=_gen(D + Hc)) - 1).to(DEV)
    pts = _sample_kpts(Hc, Wc, 200, Wc)
    n_out = [pts.shape[0], pts.shape[0] // 2, 1]
    out_cap = pts.shape[0] + 5
    kp = torch.full((B, out_cap, 2), float('nan'))
    for b in range(B):
        kp[b, :n_out[b]] = pts[torch.randperm(pts.shape[0], generator=_gen(b))[:n_out[b]]] if b else pts
    kp = kp.to(DEV)
    out = _poisoned(B * out_cap * D)
    n_dev = torch.tensor(n_out, dtype=torch.int32, device=DEV)
    _check(_lib().og_sp_sample_desc(_p(coarse), B, Hc, Wc, D, _p(kp), _p(n_dev), out_cap, max(n_out), cell, _p(out), _st()), 'og_sp_sample_desc')
    got = out[:B * out_cap * D].view(B, out_cap, D)
    err = dist32 = 0.0
    for b in range(B):
        n = n_out[b]
        r64 = sample_desc_ref(coarse[b], kp[b, :n], cell, torch.float64)
        r32 = sample_desc_ref(coarse[b], kp[b, :n], cell, torch.float32)
        err = max(err, float((got[b, :n].double() - r64).abs().max()))
        dist32 = max(dist32, float((r32.double() - r64).abs().max()))
        assert _untouched(got[b, n:])
    bound = max(2 * dist32, 1e-6)
    _report(f'sample_desc Hc {Hc} Wc {Wc} D {D}, n_out {n_out}', err, bound)
    assert err <= bound
    assert _untouched(out[B * out_cap * D:])


# =====================================================================================================================
# 2. the post-processing chain at real sizes against fixtures minted by the reference's own forward
def _post(name):
    fx = torch.load(os.path.join(HERE, 'golden', name + '.pt'), weights_only=False)
    c = fx['case']
    scores, desc = post_inputs(c['batch'], c['h'], c['w'], c['seed'], c['levels'])
    assert inputs_sha256(scores, desc) == fx['sha256'], 'the regenerated inputs differ from the ones the fixture was minted from'
    if fx['candidates'] is None:                                         # the output is every candidate, in order
        fx['candidates'] = [(k[:, 1].int() * c['w'] + k[:, 0].int()) for k in fx['keypoints']]
    else:
        fx['candidates'] = list(fx['candidates'].split(fx['counts'].tolist()))
    assert [len(x) for x in fx['candidates']] == fx['counts'].tolist()
    return fx, scores, desc


def _modes(counts, maxk):
    """the module's selection (superpoint.py, top_k_keypoints + min_stack): per image (n kept, sorted top-k or not)"""
    keep = [c if (maxk == -1 or maxk >= c) else maxk for c in counts]
    mode = [0 if (maxk == -1 or maxk >= c) else 1 for c in counts]
    if any(v != min(keep) for v in keep):
        keep, mode = [min(keep)] * len(counts), [1] * len(counts)
    return keep, mode


def _same_up_to_ties(pos, sc, ref_pos, ref_sc, cand_pos, cand_sc, topk):
    """pos / ref_pos: keypoint positions (y W + x) of one image, sc / ref_sc their scores (lists).  Identical sequences, except that
    the reference's top-k (torch.topk) orders equal scores arbitrarily: inside a run of equal scores the positions are compared as
    sets, ours ascending; the last run may be cut, where the reference may keep any candidates of that score and ours keeps the
    lowest positions.  Returns the number of keypoints in tie runs."""
    assert sc == ref_sc
    if not topk:
        assert pos == ref_pos
        return 0
    pool = {}
    for p, s in zip(cand_pos, cand_sc):
        pool.setdefault(s, []).append(p)
    n, i, tied = len(sc), 0, 0
    while i < n:
        j = i
        while j < n and sc[j] == sc[i]:
            j += 1
        ours, theirs = pos[i:j], ref_pos[i:j]
        assert ours == sorted(ours), i
        if j < n or len(pool[sc[i]]) == j - i:
            assert set(ours) == set(theirs), i
        else:
            assert ours == sorted(pool[sc[i]])[:j - i] and set(theirs) <= set(pool[sc[i]]), i
        tied += j - i if j - i > 1 else 0
        i = j
    return tied


def test_post_fixtures_follow_the_restated_rules():
    """CPU: each fixture's inputs regenerate to the recorded bytes, its candidates are the restated NMS / threshold / border rule on
    them, its keypoints the restated selection (up to exact ties), and each reaches the regime its case claims."""
    seen = {}
    for name in POST_CASES:
        fx, scores, desc = _post(name)
        c = fx['case']
        heat = pixel_heat(scores.permute(0, 2, 3, 1))
        kept = nms_threshold_borders(heat, c['nms'], c['thr'], c['border'])
        counts = fx['counts'].tolist()
        keep, mode = _modes(counts, c['maxk'])
        for b in range(c['batch']):
            cand = torch.nonzero(kept[b].view(-1))[:, 0]
            assert torch.equal(fx['candidates'][b].long(), cand)
            cand_sc = kept[b].view(-1)[cand]
            kp = fx['keypoints'][b].long()
            pos = (kp[:, 1] * c['w'] + kp[:, 0]).tolist()
            assert torch.equal(fx['scores'][b], heat[b].view(-1)[pos])
            order = torch.sort(cand_sc, descending=True, stable=True).indices[:keep[b]] if mode[b] else torch.arange(keep[b])
            _same_up_to_ties(cand[order].tolist(), cand_sc[order].tolist(), pos, fx['scores'][b].tolist(), cand.tolist(), cand_sc.tolist(), mode[b])
        seen[name] = (counts, keep, mode)
        print(f'{name}: candidates {counts}, kept {keep}, sorted {mode}, n2 {[_n2(x) for x in counts]}')
    assert all(_n2(x) == 4096 for x in seen['sp_post_480_top2048'][0]) and seen['sp_post_480_top2048'][2] == [1, 1]
    assert seen['sp_post_720_all'][2] == [0] and 8192 < seen['sp_post_720_all'][0][0] <= SP_MAX_CAND
    assert seen['sp_post_720_top2048'][2] == [1] and _n2(seen['sp_post_720_top2048'][0][0]) == SP_MAX_CAND
    assert len(set(seen['sp_post_240_minstack'][0])) == 3 and seen['sp_post_240_minstack'][2] == [1, 1, 1]
    fx, _, _ = _post('sp_post_240_ties')
    assert all(int((s[1:] == s[:-1]).sum()) > 50 for s in fx['scores'])


def _probs_coarse(scores, desc):
    """injected layer outputs -> the module's NHWC layout: probs [B hc wc, 65] (channel 64 unused: 0), coarse [B hc wc, D]"""
    return (cell_probs(pixel_heat(scores.permute(0, 2, 3, 1))).view(-1, 65).to(DEV),
            desc.permute(0, 2, 3, 1).reshape(-1, desc.shape[1]).contiguous().to(DEV))


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(POST_CASES))
def test_post_chain_matches_reference(name):
    from openglue_b200 import SuperPointNet
    fx, scores, desc = _post(name)
    c = fx['case']
    h, w = c['h'], c['w']
    model = SuperPointNet(max_keypoints=c['maxk'], nms_kernel=c['nms'], remove_borders_size=c['border'], keypoint_threshold=c['thr']).to(DEV).eval()
    probs, coarse = _probs_coarse(scores, desc)
    lafs, sc, ds = [t.cpu() for t in model._keypoints(probs, coarse, h, w)]
    counts = fx['counts'].tolist()
    keep, mode = _modes(counts, c['maxk'])
    assert lafs.shape == (c['batch'], keep[0], 2, 3) and ds.shape == (c['batch'], keep[0], 256)
    assert torch.equal(sc, fx['scores'])                                 # copies of the input: bit-equal
    err = err64 = dist32 = 0.0
    tied = []
    for b in range(c['batch']):
        kp = lafs[b, :, :, 2]
        pos = (kp[:, 1].long() * w + kp[:, 0].long()).tolist()
        ref_kp = fx['keypoints'][b]
        ref_pos = (ref_kp[:, 1].long() * w + ref_kp[:, 0].long()).tolist()
        cand = fx['candidates'][b].long()
        cand_sc = pixel_heat(scores.permute(0, 2, 3, 1))[b].view(-1)[cand]
        tied.append(_same_up_to_ties(pos, sc[b].tolist(), ref_pos, fx['scores'][b].tolist(), cand.tolist(), cand_sc.tolist(), mode[b]))
        at = {p: i for i, p in enumerate(pos)}
        for j, d in zip(fx['desc_idx'][b].tolist(), fx['descriptors'][b]):
            if ref_pos[j] in at:
                err = max(err, float((ds[b, at[ref_pos[j]]] - d).abs().max()))
        cb = coarse.view(c['batch'], h // 8, w // 8, -1)[b]
        r64 = sample_desc_ref(cb, kp.to(DEV), 8, torch.float64)
        r32 = sample_desc_ref(cb, kp.to(DEV), 8, torch.float32)
        err64 = max(err64, float((ds[b].double() - r64.cpu()).abs().max()))
        dist32 = max(dist32, float((r32.double() - r64).abs().max()))
    bound64 = max(2 * dist32, 1e-6)
    print(f'\n[{name}] candidates {counts}, n2 {[_n2(x) for x in counts]}, keypoints {keep[0]} per image, sorted {mode}, '
          f'keypoints in exact-tie runs {tied}; descriptors: max |ours - reference fp32| {err:.2e} (bound 1e-6), '
          f'max |ours - float64| {err64:.2e} (bound {bound64:.1e})')
    assert err <= 1e-6 and err64 <= bound64


@pytest.mark.gpu
def test_post_chain_over_capacity():
    """720 x 960 with nms_kernel 5: more NMS survivors than the 16384 candidates one image holds.  The module raises its host error;
    og_sp_compact reports the true count."""
    from openglue_b200 import SuperPointNet
    scores, desc = post_inputs(1, 720, 960, 12)
    probs, coarse = _probs_coarse(scores, desc)
    ref = int((nms_threshold_borders(pixel_heat(scores.permute(0, 2, 3, 1)), 5, 0.005, 4) != 0).sum())
    model = SuperPointNet(max_keypoints=2048, nms_kernel=5, keypoint_threshold=0.005).to(DEV).eval()
    with pytest.raises(RuntimeError, match='survive non-maximum suppression'):
        model._keypoints(probs, coarse, 720, 960)
    lib = _lib()
    heat = _poisoned(720 * 960)
    _check(lib.og_sp_heat_nms(_p(probs), 1, 90, 120, 5, 0.005, 4, _p(heat), _st()), 'og_sp_heat_nms')
    idx, sc, cnt = _poisoned(SP_MAX_CAND, torch.int32), _poisoned(SP_MAX_CAND), _poisoned(1, torch.int32)
    _check(lib.og_sp_compact(_p(heat), 1, 720 * 960, SP_MAX_CAND, _p(idx), _p(sc), _p(cnt), _st()), 'og_sp_compact')
    print(f'\n[over capacity] 720x960 nms 5: {int(cnt[0])} candidates (restated rule: {ref}), capacity {SP_MAX_CAND}')
    assert ref > SP_MAX_CAND and int(cnt[0]) == ref
    assert _untouched(idx[SP_MAX_CAND:]) and _untouched(sc[SP_MAX_CAND:]) and _untouched(cnt[1:])
    assert not bool(torch.isnan(sc[:SP_MAX_CAND]).any())


# =====================================================================================================================
# 3. the whole network at real size against the float64 restatement of the reference's layers
@pytest.mark.parametrize('name', ['superpoint_all', 'superpoint_topk', 'superpoint_thr', 'superpoint_bn'])
def test_layers_restatement_reproduces_the_reference(name):
    """CPU: layers_ref in float64 reproduces the float64 run of the unmodified reference module the fixtures store (as float32)"""
    from gen_golden_superpoint import synthetic_superpoint_bn_state_dict, synthetic_superpoint_state_dict
    fx = torch.load(os.path.join(HERE, 'golden', name + '.pt'), weights_only=False)
    seed = fx['case'][5]
    bn = name.endswith('_bn')
    sd = synthetic_superpoint_bn_state_dict(seed) if bn else synthetic_superpoint_state_dict(seed)
    desc, heat = layers_ref(sd, fx['image'], torch.float64, bn)
    e_heat = float((heat - fx['heat_f64'].double()).abs().max())
    e_desc = float((desc - fx['desc_map_f64'].double()).abs().max())
    print(f'{name}: max |heat - ref64| {e_heat:.1e}, max |desc - ref64| {e_desc:.1e} (bound 1e-7: the fixture is rounded to float32)')
    assert e_heat <= 1e-7 and e_desc <= 1e-7


_REF_CACHE = {}


def _network_ref(B, H, W, bn, seed):
    """(sd, image, desc64, heat64, float32-restatement distances) for one configuration, run on the device"""
    key = (B, H, W, bn, seed)
    if key not in _REF_CACHE:
        from gen_golden_superpoint import synthetic_images, synthetic_superpoint_bn_state_dict, synthetic_superpoint_state_dict
        sd = synthetic_superpoint_bn_state_dict(seed) if bn else synthetic_superpoint_state_dict(seed)
        img = synthetic_images(B, H, W, seed).to(DEV)
        d64, h64 = layers_ref(sd, img, torch.float64, bn)
        tf32 = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            d32, h32 = layers_ref(sd, img, torch.float32, bn)
        finally:
            torch.backends.cudnn.allow_tf32 = tf32
        _REF_CACHE.clear()
        _REF_CACHE[key] = (sd, img, d64, h64, float((h32.double() - h64).abs().max()), float((d32.double() - d64).abs().max()))
    return _REF_CACHE[key]


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('bn', [False, True], ids=['plain', 'bn'])
@pytest.mark.parametrize('B,H,W', [(2, 480, 640), (1, 720, 960)])
def test_network_at_real_size(B, H, W, bn, precision):
    """The reference config (max_keypoints 2048, nms_kernel 9, keypoint_threshold 0.005, borders 4)"""
    from openglue_b200 import SuperPointNet, SuperPointNetBn
    sd, img, d64, h64, dh32, dd32 = _network_ref(B, H, W, bn, 21)
    cls = SuperPointNetBn if bn else SuperPointNet
    thr = 0.005
    model = cls(max_keypoints=2048, nms_kernel=9, keypoint_threshold=thr, precision=precision)
    model.load_state_dict(sd, strict=True)
    model = model.to(DEV).eval()
    lafs, sc, ds = model(img)
    lafs2, sc2, ds2 = model(img)
    assert torch.equal(lafs, lafs2) and torch.equal(sc, sc2) and torch.equal(ds, ds2)           # deterministic
    probs, coarse = model._network(img)
    heat = pixel_heat(probs.view(B, H // 8, W // 8, 65)).double()
    dmap = coarse.view(B, H // 8, W // 8, -1).permute(0, 3, 1, 2).double()
    e_heat, e_desc = float((heat - h64).abs().max()), float((dmap - d64).abs().max())
    b_heat, b_desc = max(1e-5, 5 * dh32), max(1e-5, 5 * dd32)
    # NMS decisions of the module's own heat map, pixel by pixel, against the rule on the float64 map
    out = _poisoned(B * H * W)
    _check(_lib().og_sp_heat_nms(_p(probs), B, H // 8, W // 8, 9, thr, 4, _p(out), _st()), 'og_sp_heat_nms')
    ours_keep = (out[:B * H * W].view(B, H, W) != 0).cpu()
    margin = 10 * max(e_heat, 1e-7)
    h64c = h64.float().cpu()
    keep, decisive = _decisions(h64c, 9, thr, 4, margin)
    assert int(((ours_keep != keep) & decisive).sum()) == 0
    # the keypoints: the reference's top-k of its kept pixels, by float64 score, then min_stack
    lafs, ds = lafs.cpu(), ds.cpu()
    counts = keep.view(B, -1).sum(1).tolist()
    n_ref = min(min(c, 2048) for c in counts)
    bad, e_kd = 0, 0.0
    for b in range(B):
        kept = torch.nonzero(keep[b].view(-1))[:, 0]
        top = kept[torch.sort(h64c[b].view(-1)[kept], descending=True, stable=True).indices[:n_ref]]
        ref_pts = [(int(p) % W, int(p) // W) for p in top]
        ours = [(int(x), int(y)) for x, y in lafs[b, :, :, 2].tolist()]
        bad += _disagreements(ours, ref_pts, keep[b], decisive[b], h64c[b], margin)
        r64 = sample_desc_ref(d64[b].permute(1, 2, 0), lafs[b, :, :, 2].to(DEV), 8, torch.float64)
        e_kd = max(e_kd, float((ds[b].double() - r64.cpu()).abs().max()))
    print(f'\n[{cls.__name__} {precision} {B}x{H}x{W}] heat {e_heat:.2e} (bound {b_heat:.1e}), descriptor map {e_desc:.2e} '
          f'(bound {b_desc:.1e}); candidates {counts}, n2 {[_n2(c) for c in counts]}, keypoints {tuple(lafs.shape[:2])}; '
          f'non-decisive pixels {int((~decisive).sum())}, decisive disagreements {bad}; keypoint descriptors {e_kd:.2e} (bound 1e-4)')
    assert e_heat <= b_heat and e_desc <= b_desc
    assert bad == 0
    if bool(decisive.all()):
        assert lafs.shape[1] == n_ref
    assert e_kd <= 1e-4


@pytest.mark.gpu
def test_network_without_keypoints_and_bad_sizes():
    from gen_golden_superpoint import synthetic_images, synthetic_superpoint_state_dict
    from openglue_b200 import SuperPointNet
    model = SuperPointNet(max_keypoints=2048, keypoint_threshold=1.0)            # no probability exceeds 1
    model.load_state_dict(synthetic_superpoint_state_dict(21), strict=True)
    model = model.to(DEV).eval()
    lafs, sc, ds = model(synthetic_images(2, 64, 96, 3).to(DEV))
    assert lafs.shape == (2, 0, 2, 3) and sc.shape == (2, 0) and ds.shape == (2, 0, 256)
    for h, w in [(60, 96), (64, 100), (63, 63)]:
        with pytest.raises(ValueError):
            model(torch.zeros(1, 1, h, w, device=DEV))
