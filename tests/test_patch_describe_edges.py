"""The describe path the AffNet / OriNet / HardNet front-ends share (``GFTTAffNetHardNet``, ``DoGOpenCVAffNetHardNet``) at its edges,
against the float64 restatements in oracle/: the patch CNNs layer by layer at every partial-chunk row count, both im2col kernels,
``ks_patch``'s pyramid-level choice, clamps and borders, the row mapping of a chunk that spans images, the AffNet frame algebra
at tanh saturation, and the descriptor normalisation."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import dog_affnet_oracle as KD  # noqa: E402
from oracle import kornia_gftt_oracle as KG  # noqa: E402
from oracle import kornia_sift_oracle as KO  # noqa: E402
from openglue_b200 import DoGOpenCVAffNetHardNet, GFTTAffNetHardNet, _cabi  # noqa: E402
from openglue_b200._cabi import ptr  # noqa: E402
from openglue_b200._ops import _Ops  # noqa: E402
from openglue_b200._patch_cnn import AFFNET_CONVS, CHUNK, HARDNET_CONVS, HEAD, PS, cnn_buffers, fold, nhwc_head, run_cnn  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
PREC = {'fp32': _cabi.OG_PREC_FP32, 'tf32x3': _cabi.OG_PREC_TF32X3}


def _lib():
    return _cabi.lib()


def _st():
    return _cabi.stream(torch.device(DEV))


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ulps(a, b):
    """|a - b| in units of b's float32 ulp, per element (b float64, rounded to float32 for its ulp)"""
    bf = b.float().abs()
    return (a.double() - b).abs() / (torch.nextafter(bf, torch.tensor(float('inf'))) - bf).double()


# ------------------------------------------------------------------ im2col
def _unfold64(x, stride):
    """The float64 3x3, padding-1 im2col of NHWC x [B, H, W, C]: [B * Ho * Wo, 9 C], column (3 ky + kx) C + c"""
    B, H, W, C = x.shape
    xp = F.pad(x.double().permute(0, 3, 1, 2), (1, 1, 1, 1))
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    taps = [xp[:, :, ky:ky + stride * (Ho - 1) + 1:stride, kx:kx + stride * (Wo - 1) + 1:stride] for ky in range(3) for kx in range(3)]
    return torch.stack(taps, 1).permute(0, 3, 4, 1, 2).reshape(B * Ho * Wo, 9 * C)


def _im2col(x, stride, out=None):
    """og_sp_im2col3x3 (stride 1) or og_kgftt_im2col3x3_s2 (stride 2) of NHWC x on the GPU: [B * Ho * Wo, 9 C]"""
    B, H, W, C = x.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    if out is None:
        out = torch.empty(B * Ho * Wo * 9 * C, device=DEV)
    fn = 'og_sp_im2col3x3' if stride == 1 else 'og_kgftt_im2col3x3_s2'
    _cabi.check(getattr(_lib(), fn)(ptr(x), B, H, W, C, ptr(out), _st()), fn)
    return out[:B * Ho * Wo * 9 * C].view(B * Ho * Wo, 9 * C)


@pytest.mark.parametrize('C', [1, 3, 16, 64])
@pytest.mark.parametrize('H,W', [(31, 17), (1, 5), (2, 3), (16, 16), (32, 32)])
def test_im2col_is_the_float64_unfold_bit_for_bit(H, W, C):
    """a copy: equal to the float64 unfold exactly, the scalar (C % 4 != 0) and float4 paths, odd sizes ((H + 1) / 2 outputs), and
    nothing written past the output"""
    x = torch.randn(2, H, W, C, generator=_gen(H * 1000 + W * 10 + C)).to(DEV)
    for stride in (1, 2):
        want = _unfold64(x.cpu(), stride)
        buf = torch.full((want.numel() + 256,), float('nan'), device=DEV)
        got = _im2col(x, stride, buf)
        torch.cuda.synchronize()
        assert torch.equal(got.cpu().double(), want), stride
        assert bool(buf[want.numel():].isnan().all()), stride


# ------------------------------------------------------------------ patch CNNs by layer and by row count
ROWS = [1, 63, 64, 65, 127, 128]
NETS = {'affnet': AFFNET_CONVS, 'orinet': AFFNET_CONVS, 'hardnet': HARDNET_CONVS}


def _net(name, dtype, sd=None):
    if name == 'affnet':
        return KG.features_in(dtype, affnet_sd=sd)[0]
    if name == 'hardnet':
        return KG.features_in(dtype, hardnet_sd=sd)[1]
    return KD.orinet_in(dtype, sd)


def _packed(name, net):
    """the front-ends' GEMM layers (as their _weights_on packs them): folded 3x3 layers, then the head (none for OriNet, whose head
    is og_dogaff_orinet_head)"""
    layers = [fold(net[i].weight, net[i + 1]) for i, *_ in NETS[name]]
    if name == 'affnet':
        layers.append(nhwc_head(net[HEAD]))
    elif name == 'hardnet':
        layers.append(fold(net[HEAD].weight, net[HEAD + 1]))
    return [(w.to(DEV), b.to(DEV)) for w, b in layers]


def _stepwise(ops, layers, convs, x, rows, head_out):
    """run_cnn's layers one at a time on rows NHWC patches x: [(im2col, NHWC output)] per 3x3 layer, and the head into head_out"""
    out = []
    h = w = PS
    for li, (_, ci, co, s) in enumerate(convs):
        col = _im2col(x.view(rows, h, w, ci), s)
        h, w = (h - 1) // s + 1, (w - 1) // s + 1
        wt, b = layers[li]
        y = ops.linear(col, wt, b, relu=True, out=torch.empty(rows * h * w, co, device=DEV))
        out.append((col, y.view(rows, h, w, co)))
        x = y
    if head_out is not None:
        wt, b = layers[len(convs)]
        ops.linear(x.view(rows, -1), wt, b, out=head_out)
    return out


def _nchw64(t):
    return t.permute(0, 3, 1, 2).double()


@pytest.mark.parametrize('case', ['affnet', 'orinet', 'hardnet', 'affnet_var0'])
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_cnn_layers_at_every_row_count_against_float64(case, precision):
    """Each 3x3 layer (im2col bit for bit, then the GEMM with folded BatchNorm and ReLU) on the kernel's own input to it, and the
    head, against float64 conv2d + BatchNorm + ReLU; the first r rows of a 128-row pass equal an r-row pass bit for bit (neither
    GEMM splits K, so no output row's reduction depends on M); run_cnn gives the same bits, with AffNet's [r, 3] head at its
    12-byte stride and nothing past it.  ``affnet_var0``: one BatchNorm's running_var near 0, so the fold's 1 / sqrt(var + eps)
    is ~300."""
    name = case.split('_')[0]
    sd = None
    if case == 'affnet_var0':
        sd = KG.synthetic_affnet_state_dict()
        sd['features.4.running_var'] = 1e-7 * torch.rand(16, generator=_gen(11))
    net64, net32 = _net(name, torch.float64, sd), _net(name, torch.float32, sd)
    net64d = _net(name, torch.float64, sd).to(DEV)
    convs = NETS[name]
    layers = _packed(name, net64)
    ops = _Ops(torch.device(DEV), PREC[precision])
    nout = {'affnet': 3, 'hardnet': 128, 'orinet': None}[name]
    x = KG.normalize_input(torch.rand(CHUNK, 1, PS, PS, generator=_gen(5))).view(CHUNK, PS, PS, 1).to(DEV).contiguous()
    head = torch.empty(CHUNK, nout, device=DEV) if nout else None
    full = _stepwise(ops, layers, convs, x, CHUNK, head)
    torch.cuda.synchronize()
    # each layer against float64, on the kernel's input to it
    inp = x
    with torch.no_grad():
        for li, ((i, ci, co, s), (col, y)) in enumerate(zip(convs, full)):
            assert torch.equal(col.cpu().double(), _unfold64(inp.cpu(), s)), li
            x64 = _nchw64(inp).to(DEV)
            want = torch.relu(net64d[i + 1](net64d[i](x64))).cpu()
            ref32 = torch.relu(net32[i + 1](net32[i](_nchw64(inp).float().cpu()))).double()
            # eps: 3xTF32 drops the lo x lo product (< 2^-22 |w||x| per term) and the folded weights and bias are rounded to
            # float32 once (2^-24 relative); 2^-20 sum |w||x| + |b| covers both twice over
            wf, bf = layers[li]
            mag = F.conv2d(x64.abs(), wf.double().view(co, 3, 3, ci).permute(0, 3, 1, 2).abs(), stride=s, padding=1) + bf.double().abs().view(1, -1, 1, 1)
            bound = 4 * float((ref32 - want).abs().max()) + 2.0 ** -20 * float(mag.max())
            err = float((_nchw64(y).cpu() - want).abs().max())
            print(f'{case} {precision} layer {li}: err {err:.3e}, bound {bound:.3e} (max |y| {float(want.abs().max()):.3e})')
            assert err <= bound, (li, err, bound)
            inp = y
        if nout:
            x64 = _nchw64(inp).to(DEV)
            want = (net64d[HEAD](x64) if name == 'affnet' else net64d[HEAD + 1](net64d[HEAD](x64))).flatten(1).cpu()
            x32 = _nchw64(inp).float().cpu()
            ref32 = (net32[HEAD](x32) if name == 'affnet' else net32[HEAD + 1](net32[HEAD](x32))).flatten(1).double()
            wf, bf = layers[-1]
            mag = inp.reshape(CHUNK, -1).double().abs().cpu() @ wf.double().abs().t().cpu() + bf.double().abs().cpu()
            bound = 4 * float((ref32 - want).abs().max()) + 2.0 ** -20 * float(mag.max())
            err = float((head.cpu().double() - want).abs().max())
            print(f'{case} {precision} head: err {err:.3e}, bound {bound:.3e}')
            assert err <= bound, (err, bound)
    # partial chunks: bit for bit the prefix of the full pass, through the stepwise layers and through run_cnn
    patches, col, a0, a1, _ = cnn_buffers({}, torch.device(DEV))
    patches[:CHUNK * PS * PS].copy_(x.flatten())
    for r in ROWS:
        h_r = torch.empty(r, nout, device=DEV) if nout else None
        part = _stepwise(ops, layers, convs, x[:r].contiguous(), r, h_r)
        out = torch.full((CHUNK * 3 + 64,), float('nan'), device=DEV) if name == 'affnet' else (
            torch.empty(r, nout, device=DEV) if nout else None)
        got = run_cnn(ops, layers, patches, r, convs, col, (a0, a1), out[:r * 3].view(r, 3) if name == 'affnet' else out)
        torch.cuda.synchronize()
        for li, ((_, yf), (_, yr)) in enumerate(zip(full, part)):
            assert torch.equal(yr, yf[:r]), (r, li)
        if nout:
            assert torch.equal(h_r, head[:r]), r
            run_head = out[:r * 3].view(r, 3) if name == 'affnet' else out
            assert torch.equal(run_head, head[:r]), r
            if name == 'affnet':
                assert bool(out[r * 3:].isnan().all()), r
        else:
            assert torch.equal(got.view(r, 8, 8, 64), full[-1][1][:r]), r


# ------------------------------------------------------------------ ks_patch at its boundaries
SIZES = [(160, 171), (64, 97), (33, 47), (31, 40)]
BOUNDARY_D = [-1e-2, -4e-4, -2.0 ** -22, 0.0, 2.0 ** -22, 4e-4, 1e-2]


def _shapes():
    """unit-determinant 2x2 parts: identity, two rotations, a shear, a strongly anisotropic rotated ellipse"""
    def rot(deg):
        t = torch.tensor(deg, dtype=torch.float64) * torch.pi / 180
        return torch.stack([torch.stack([t.cos(), t.sin()]), torch.stack([-t.sin(), t.cos()])])
    sh = torch.tensor([[1.0, 0.8], [0.0, 1.0]], dtype=torch.float64)
    an = torch.diag(torch.tensor([4.0, 0.25], dtype=torch.float64))
    return [torch.eye(2, dtype=torch.float64), rot(30.0), rot(-135.0), sh, rot(60.0) @ an]


def _laf_table(H, W):
    """(LAFs [1, N, 2, 3] float64, nominal scales [N], rotation angles in degrees [N] for the isotropic rows (nan otherwise)):
    scales 16 2^k (1 + d) next to every level boundary, below level 0 and far past the pyramid, on centres on the first and last
    pixel, half a pixel and far outside and inside, with rotated, sheared and anisotropic shapes"""
    scales = [4.0, 12.0, 16.0] + [16.0 * 2 ** k * (1 + d) for k in range(1, 6) for d in BOUNDARY_D] + [1024.0]
    cx, cy = (W - 1) / 2, (H - 1) / 2
    centres = [(0.0, 0.0), (W - 1.0, H - 1.0), (-0.5, cy), (W - 0.5, cy / 2), (cx, -0.5), (cx / 2, H - 0.5), (-40.0, cy), (W + 40.0, cy),
               (cx + 0.25, cy + 0.75)]
    shapes = _shapes()
    angles = [0.0, 30.0, -135.0, float('nan'), float('nan')]
    rows, s_nom, ang = [], [], []
    for s in scales:
        for ci, (x, y) in enumerate(centres):
            for si in ((ci + k) % len(shapes) for k in range(2)):      # two shapes per centre, every shape on every scale
                a = torch.zeros(2, 3, dtype=torch.float64)
                a[:, :2] = s * shapes[si]
                a[0, 2], a[1, 2] = x, y
                rows.append(a)
                s_nom.append(s)
                ang.append(angles[si])
    return torch.stack(rows)[None], torch.tensor(s_nom, dtype=torch.float64), torch.tensor(ang, dtype=torch.float64)


def _img(H, W, B, seed):
    return torch.rand(B, 1, H, W, generator=_gen(seed))


def _gftt_ws(m, img):
    B, _, H, W = img.shape
    ws, _ = m._workspace(img.device, B, H, W)
    _cabi.check(_lib().og_kgftt_pyramid(ptr(img), B, H, W, m.max_keypoints, ptr(ws), ws.numel(), _st()), 'og_kgftt_pyramid')
    return ws


def _gftt_model(nf=16, **kw):
    return GFTTAffNetHardNet(max_keypoints=nf, weights={'affnet': KG.synthetic_affnet_state_dict(), 'hardnet': KG.synthetic_hardnet_state_dict()},
                             **kw)


def _dog_model(**kw):
    w = dict(affnet=KG.synthetic_affnet_state_dict(), orinet=KD.synthetic_orinet_state_dict(), hardnet=KG.synthetic_hardnet_state_dict())
    return DoGOpenCVAffNetHardNet(weights=w, **kw)


def _check_patches(tag, got, img, lafs, want_fn, s_nom, upright):
    """got [N, 32, 32] against want_fn(img, lafs) in float64, where the float32 and float64 oracles pick the same level (of the LAF
    made upright when want_fn samples it so); where they pick different levels, against either oracle; exact zeros past the pyramid"""
    H, W = img.shape[-2:]
    p64 = want_fn(img.double(), lafs.double()).view(-1, PS, PS)
    p32 = want_fn(img, lafs.float()).view(-1, PS, PS).double()
    up = KO.make_upright if upright else (lambda t: t)
    l64 = KO.patch_pyramid_level(up(lafs.double()), H, W, PS).flatten()
    l32 = KO.patch_pyramid_level(up(lafs.float()), H, W, PS).flatten()
    got = got.double()
    same = l32 == l64
    # + one float32 ulp at the standardised patches' magnitude (|x| < 8: 8 2^-23 ~ 1e-6)
    bound = 4 * float((p32 - p64)[same].abs().max()) + 1e-6
    e64 = (got - p64).abs().flatten(1).amax(1)
    e32 = (got - p32).abs().flatten(1).amax(1)
    print(f'{tag} {H}x{W}: {len(got)} rows, max err {float(e64[same].max()):.3e} (bound {bound:.3e}), {int((~same).sum())} rows where '
          f'the float32 and float64 oracles pick different levels (err {float(torch.minimum(e64, e32)[~same].max()) if (~same).any() else 0:.3e})')
    assert float(e64[same].max()) <= bound
    assert bool((torch.minimum(e64, e32)[~same] <= bound).all())
    past = same & (l64 >= KO.patch_pyramid_levels(H, W, PS))
    assert not got[past].any() and not p64[past].any()
    # the table straddles every level boundary the clamp leaves open
    for k in range(1, max(0, min(H, W) // PS - 1) + 1):
        sk = 16.0 * 2 ** k
        assert bool(((l64 == k - 1) & (s_nom > 0.98 * sk) & (s_nom < sk)).any()) and bool(((l64 == k) & (s_nom >= sk) & (s_nom < 1.02 * sk)).any()), k
    return past


@pytest.mark.parametrize('H,W', SIZES)
def test_patch_sampler_at_levels_clamps_and_borders(H, W):
    """ks_patch through the three kernels that cut AffNet's and HardNet's patches, on a table of LAFs straddling every pyramid level
    boundary, past the clamp and past the last level, centred on and outside the border"""
    img = _img(H, W, 1, H + W)
    lafs, s_nom, ang = _laf_table(H, W)
    N = lafs.shape[1]
    dev_img = img.to(DEV)
    n = torch.tensor([N], dtype=torch.int32, device=DEV)
    l32 = lafs.float().to(DEV).contiguous()
    # GFTT: AffNet's standardised patch of make_upright(LAF)
    m = _gftt_model()
    ws = _gftt_ws(m, dev_img)
    out = torch.empty(N, PS, PS, device=DEV)
    _cabi.check(_lib().og_kgftt_affnet_patches(ptr(dev_img), 1, H, W, m.max_keypoints, ptr(ws), ws.numel(), ptr(l32), N, None, ptr(n), N, 0, N,
                                               ptr(out), _st()), 'og_kgftt_affnet_patches')
    torch.cuda.synchronize()
    past = _check_patches('kgftt_affnet_patches', out.cpu(), img, lafs.float(), KG.affnet_patches, s_nom, True)
    if H == 160:
        assert bool(past.any())                                         # scales 256 and up sample the missing level 4
    # GFTT frames, upright, xy = 0: HardNet's patch of the frame (the LAF's scale and orientation)
    xy = torch.zeros(N, 3, device=DEV)
    resp = torch.arange(N, dtype=torch.float32, device=DEV)
    lo, sc = torch.empty(1, N, 2, 3, device=DEV), torch.empty(1, N, device=DEV)
    _cabi.check(_lib().og_kgftt_frames(ptr(dev_img), 1, H, W, m.max_keypoints, ptr(ws), ws.numel(), ptr(l32), ptr(resp), N, None, ptr(n), N, 0, N,
                                       ptr(xy), 1, ptr(lo), ptr(sc), None, ptr(out), _st()), 'og_kgftt_frames')
    torch.cuda.synchronize()
    assert torch.equal(sc.cpu(), resp.cpu()[None]) and torch.equal(lo.cpu()[..., 2], l32.cpu()[..., 2])
    _check_patches('kgftt_frames', out.cpu(), img, lo.cpu(),
                   lambda im, la: KG.normalize_input(KO.extract_patches_from_pyramid(im, la, PS).view(-1, 1, PS, PS)), s_nom, False)
    # DoG: kornia_moons' LAF of a cv2 keypoint (isotropic rows only), then AffNet's patch
    iso = ~ang.isnan()
    kp = torch.stack([lafs[0, iso, 0, 2], lafs[0, iso, 1, 2], s_nom[iso] / 6, ang[iso], torch.arange(int(iso.sum()), dtype=torch.float64)], 1)
    kp = kp.float()[None].to(DEV).contiguous()
    Nk = kp.shape[1]
    dm = _dog_model()
    dws = dm._workspace(torch.device(DEV), 1, H, W)
    args = (ptr(dev_img), 1, H, W, ptr(dws), dws.numel())
    _cabi.check(_lib().og_dogaff_pyramid(*args, _st()), 'og_dogaff_pyramid')
    sel = torch.arange(Nk, dtype=torch.int32, device=DEV)
    nk = torch.tensor([Nk], dtype=torch.int32, device=DEV)
    dl, ds = torch.empty(1, Nk, 2, 3, device=DEV), torch.empty(1, Nk, device=DEV)
    _cabi.check(_lib().og_dogaff_affnet_patches(*args, ptr(kp), Nk, ptr(sel), ptr(nk), Nk, 0, Nk, ptr(dl), ptr(ds), ptr(out), _st()),
                'og_dogaff_affnet_patches')
    torch.cuda.synchronize()
    assert torch.equal(ds.cpu(), kp.cpu()[..., 4])
    _check_patches('dogaff_affnet_patches', out[:Nk].cpu(), img, dl.cpu(), KG.affnet_patches, s_nom[iso], True)


# ------------------------------------------------------------------ row mapping and batch structure
B3, CAP_IN, OUT_CAP, COUNTS = 3, 256, 150, [150, 37, 0]


def _det_table(B, H, W, cap, seed):
    """detector-like rows per image: centres inside, scales 6 .. 40, random orientations; (lafs [B, cap, 2, 3], resp [B, cap],
    cv2-style keypoints [B, cap, 5])"""
    g = _gen(seed)
    x = 8 + (W - 16) * torch.rand(B, cap, generator=g)
    y = 8 + (H - 16) * torch.rand(B, cap, generator=g)
    s = 6 + 34 * torch.rand(B, cap, generator=g)
    t = 360 * torch.rand(B, cap, generator=g) - 180
    r = torch.rand(B, cap, generator=g)
    rad = t * torch.pi / 180
    lafs = torch.stack([torch.stack([s * rad.cos(), s * rad.sin(), x], -1), torch.stack([-s * rad.sin(), s * rad.cos(), y], -1)], -2)
    return lafs, r, torch.stack([x, y, s / 6, t, r], -1)


def _describe(m, img, args, n, out_cap):
    """The module's _describe of the selected rows (``args``: what it takes before n), keeping through its tap every chunk's patches
    of each stage ('p_affnet', 'p_orinet', 'p_hardnet') and the angles"""
    B = img.shape[0]
    R = B * out_cap
    o = {}

    def tap(stage, r0, rows, t):
        if stage == 'angles':
            o['angles'] = t.clone()
        else:
            p = o.setdefault(f'p_{stage}', torch.full((R, PS, PS), float('nan'), device=DEV))
            p[r0:r0 + rows] = t[:rows * PS * PS].view(rows, PS, PS)
    out = m._describe(img, *args, n, out_cap, tap)
    torch.cuda.synchronize()
    o.update(zip(('lafs', 'scores', 'desc', 'angles'), out))            # DoG returns the angles, GFTT gives them to the tap
    return {key: t.cpu() for key, t in o.items()}


@pytest.mark.parametrize('front', ['gftt', 'dog'])
def test_row_mapping_across_images_and_chunks(front):
    """B = 3 images, out_cap = 150, n = [150, 37, 0] and a random sel: chunk 0 ends inside image 0's rows, chunk 1 spans images 0
    and 1, chunk 2 images 1 and 2.  Every row (b, j < n[b]) equals the same stages run on image b alone with sel[b, j] resolved on
    the host; every row past n[b], and all of image 2, is exactly zero in every output and patch."""
    H, W = 96, 120
    img = _img(H, W, B3, 7).to(DEV)
    lafs, resp, kp = _det_table(B3, H, W, CAP_IN, 8)
    sel = torch.stack([torch.randperm(CAP_IN, generator=_gen(20 + b)) for b in range(B3)]).int()
    n = torch.tensor(COUNTS, dtype=torch.int32)
    if front == 'gftt':
        m = _gftt_model(CAP_IN)
        run = lambda im, src, s, nn, oc: _describe(m, im, (_gftt_ws(m, im), src[0].to(DEV).contiguous(), src[1].to(DEV).contiguous(), s),
                                                   nn, oc)
        src = (lafs, resp)
        pick = lambda b, idx: (lafs[b:b + 1, idx], resp[b:b + 1, idx])
    else:
        m = _dog_model(capacity=CAP_IN)
        assert m.capacity == CAP_IN
        run = lambda im, src, s, nn, oc: _describe(m, im, (src.to(DEV).contiguous(), s), nn, oc)
        src = kp
        pick = lambda b, idx: kp[b:b + 1, idx]
    got = run(img, src, sel.to(DEV), n.to(DEV), OUT_CAP)
    for key, t in got.items():
        t = t.view(B3, OUT_CAP, -1)
        for b, nb in enumerate(COUNTS):
            assert not t[b, nb:].any(), (key, b)
    for b, nb in enumerate(COUNTS[:2]):
        idx = sel[b, :nb].long()
        one = pick(b, idx)
        pad = lambda t: torch.cat([t, t.new_zeros(1, CAP_IN - nb, *t.shape[2:])], 1)     # the single run's inputs at capacity
        one = tuple(pad(t) for t in one) if isinstance(one, tuple) else pad(one)
        s1 = torch.arange(CAP_IN, dtype=torch.int32, device=DEV)[None].contiguous() if front == 'dog' else None
        alone = run(img[b:b + 1].contiguous(), one, s1, torch.tensor([nb], dtype=torch.int32, device=DEV), nb)
        for key, t in alone.items():
            assert torch.equal(got[key].view(B3, OUT_CAP, -1)[b, :nb], t.view(1, nb, -1)[0]), (key, b)


# ------------------------------------------------------------------ AffNet frame algebra
XY = [0.0, 1e-3, -1e-3, 1.0, -1.0, 5.0, -5.0, 12.0, -12.0]


def _frame_table():
    """(xy [N, 3] before tanh, detector LAFs [1, N, 2, 3] float32): every xy triple of XY on isotropic LAFs of three scales and
    three orientations"""
    v = torch.tensor(XY, dtype=torch.float32)
    xy = torch.cartesian_prod(v, v, v)
    det = []
    for s in (4.0, 20.0, 60.0):
        for deg in (0.0, 50.0, -170.0):
            t = torch.tensor(deg, dtype=torch.float64) * torch.pi / 180
            det.append(torch.tensor([[s * t.cos(), s * t.sin(), 60.25], [-s * t.sin(), s * t.cos(), 47.5]], dtype=torch.float64))
    xy = xy.repeat(len(det), 1)
    lafs = torch.stack(det).repeat_interleave(len(XY) ** 3, 0)[None].float()
    return xy, lafs


def _tanh32_variants(xy):
    """float32 tanh and its values 1 and 2 ulp either side (CUDA's tanhf is within 2 ulp)"""
    t = torch.tanh(xy)
    out = [t]
    for d in (float('inf'), -float('inf')):
        u = t
        for _ in range(2):
            u = torch.nextafter(u, torch.tensor(d))
            out.append(u)
    return out


@pytest.mark.parametrize('front', ['gftt', 'dog'])
def test_affnet_frames_at_tanh_saturation(front):
    """og_kgftt_frames (upright) and og_dogaff_frames on pre-tanh xy in {0, +-1e-3, +-1, +-5, +-12}^3: centres and scores exact,
    the 2x2 part within the float32 oracle's error per row (its tanh moved by up to 2 ulp, as CUDA's tanhf may be), every value
    finite and the determinant the input's (scale_orig^2) up to the float32 rounding of the output's entries"""
    xy, lafs = _frame_table()
    N = xy.shape[0]
    H, W = 96, 120
    img = _img(H, W, 1, 9).to(DEV)
    n = torch.tensor([N], dtype=torch.int32, device=DEV)
    out = torch.empty(N, PS, PS, device=DEV)
    xy_d, lafs_d = xy.to(DEV).contiguous(), lafs.to(DEV).contiguous()
    if front == 'gftt':
        m = _gftt_model()
        ws = _gftt_ws(m, img)
        resp = torch.rand(N, generator=_gen(3)).to(DEV)
        lo, sc = torch.empty(1, N, 2, 3, device=DEV), torch.empty(1, N, device=DEV)
        _cabi.check(_lib().og_kgftt_frames(ptr(img), 1, H, W, m.max_keypoints, ptr(ws), ws.numel(), ptr(lafs_d), ptr(resp), N,
                                           None, ptr(n), N, 0, N, ptr(xy_d), 1, ptr(lo), ptr(sc), None, ptr(out), _st()),
                    'og_kgftt_frames')
        torch.cuda.synchronize()
        assert torch.equal(sc.cpu()[0], resp.cpu())
    else:
        m = _dog_model()
        ws = m._workspace(torch.device(DEV), 1, H, W)
        args = (ptr(img), 1, H, W, ptr(ws), ws.numel())
        _cabi.check(_lib().og_dogaff_pyramid(*args, _st()), 'og_dogaff_pyramid')
        lo = lafs_d.clone()
        _cabi.check(_lib().og_dogaff_frames(*args, ptr(n), N, 0, N, ptr(xy_d), ptr(lo), ptr(out), _st()), 'og_dogaff_frames')
        torch.cuda.synchronize()
    lo = lo.cpu()[0].double()
    assert torch.equal(lo[:, :, 2], lafs[0, :, :, 2].double())
    assert bool(lo.isfinite().all()) and bool(out.isfinite().all())
    want = KG.affnet_frames(torch.tanh(xy.double()), lafs.double())[0]
    ref_err = torch.stack([(KG.affnet_frames(t, lafs)[0].double() - want)[:, :, :2].abs().flatten(1).amax(1) for t in _tanh32_variants(xy)]).amax(0)
    s2 = (lafs[0, :, 0, 0].double() * lafs[0, :, 1, 1] - lafs[0, :, 1, 0].double() * lafs[0, :, 0, 1] + 1e-10).abs()
    err = (lo[:, :, :2] - want[:, :, :2]).abs().flatten(1).amax(1)
    bound = 4 * ref_err + 2.0 ** -20 * s2.sqrt()
    worst = int((err / bound).argmax())
    print(f'{front}: {N} rows, max err / bound {float((err / bound).max()):.3f} (row {worst}: xy {xy[worst].tolist()}, err {float(err[worst]):.3e}, '
          f'bound {float(bound[worst]):.3e}); max err where no tanh saturates {float(err[(xy.abs() < 5).all(1)].max()):.3e}')
    assert bool((err <= bound).all())
    # the frame keeps the input's scale: det = scale_orig^2, up to the rounding of the entries (2^-24 each) through ~30 float32
    # operations: 2^-16 of |a00 a11| + |a01 a10|
    d = lo[:, 0, 0] * lo[:, 1, 1] - lo[:, 0, 1] * lo[:, 1, 0]
    scale = (lo[:, 0, 0] * lo[:, 1, 1]).abs() + (lo[:, 0, 1] * lo[:, 1, 0]).abs()
    rel = (d - s2).abs() / scale
    print(f'{front}: max |det - scale_orig^2| / (|a00 a11| + |a01 a10|) {float(rel.max()):.3e}')
    assert bool((rel <= 2.0 ** -16).all())


# ------------------------------------------------------------------ descriptor normalisation
def test_desc_finish_normalises_and_zeroes():
    """og_kgftt_desc_finish on B = 2: random rows over six decades, a zero row, rows of norm ~1e-20 (below the 1e-12 clamp) and rows
    past n[b].  Bit for bit the float32 restatement of its order (per lane (x^2 + y^2) + (z^2 + w^2), then the xor tree 16 .. 1);
    within 4.5 ulp of F.normalize in float64 (the squared norm rounds 7 times along that tree, 3.5 ulp after the square root,
    plus the root's and the division's half ulp each); zeros exact."""
    B, cap, n = 2, 40, [30, 7]
    g = _gen(4)
    desc = torch.randn(B, cap, 128, generator=g) * torch.logspace(-3, 3, B * cap).view(B, cap, 1)
    desc[0, 3] = 0.0
    desc[1, 2] = 0.0
    desc[0, 5] = torch.randn(128, generator=g) * 1e-21
    desc[1, 4] = torch.randn(128, generator=g) * 3e-22
    d = desc.to(DEV).contiguous()
    _cabi.check(_lib().og_kgftt_desc_finish(ptr(d), B, cap, ptr(torch.tensor(n, dtype=torch.int32, device=DEV)), _st()), 'og_kgftt_desc_finish')
    got = d.cpu()
    x = desc.view(B, cap, 32, 4)
    s = (x[..., 0] * x[..., 0] + x[..., 1] * x[..., 1]) + (x[..., 2] * x[..., 2] + x[..., 3] * x[..., 3])
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., torch.arange(32) ^ o]
    emu = desc / torch.clamp(torch.sqrt(s[..., :1]), min=1e-12)
    want = F.normalize(desc.double(), dim=-1)
    for b in range(B):
        assert not got[b, n[b]:].any()
        assert torch.equal(got[b, :n[b]], emu[b, :n[b]])
        u = _ulps(got[b, :n[b]], want[b, :n[b]])
        print(f'image {b}: max {float(u.max()):.2f} ulp from float64')
        assert float(u.max()) <= 4.5
    assert not got[0, 3].any() and not got[1, 2].any()
