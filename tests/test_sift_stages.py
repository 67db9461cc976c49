"""The OpenCV SIFT front-end (csrc/sift.cuh) stage by stage.  Each stage is checked on the kernels' own inputs for it, read back
from og_sift_detect's workspace (og_sift_workspace_layout), so an error in one stage does not spread into the next.  Every GPU
test runs a batch of three different images of one size, so the planes of images b > 0 are exercised at every stage.

  P  pyramid, exact: octave 0 level 0 = the blur of the x2 INTER_LINEAR upsample; every later level = the blur of the kernels'
     previous level; DoG = the float32 difference of adjacent levels; the first level of an octave = the nearest x2 downsample of
     level 3 of the one before.  The blur restatement (exact float32 FMA) is also held to a float64 convolution, and, where cv2
     is installed, to cv2.resize / cv2.GaussianBlur on the host.
  X  extrema + interpolation: the located records equal a float32 restatement bit for bit (size within 1 ulp: the kernel's and
     numpy's double exp2 are not both correctly rounded) and a float64 one within tolerances, except candidates that float64
     puts within a margin of a decision.
  O  orientations against a float64 histogram on the kernels' Gaussian levels.
  S  cv2's keypoint order and duplicate removal, exact; the padded entry point's count / overflow.
  N  NMS + top-k on synthetic keypoints against test_sift.greedy_select, at its edges.
  D  descriptors against cv2's calcSIFTDescriptor in float64 on the kernels' Gaussian level, synthetic keypoints at the image
     borders, octaves, sizes and angles where it goes wrong, and every selected keypoint of real images.

Crop widths are chosen so that the octave widths cover every residue of w mod 8 (the blurs' fused / unfused tails), and one batch
is 8 x 13, whose late octaves are narrower than the 27-tap kernel.  Measured distributions are printed (pytest -s).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from test_sift import greedy_select

DEV = 'cuda:0'
F32_EPS = float(np.finfo(np.float32).eps)
LOC_DTYPE = np.dtype([('o', '<i4'), ('layer', '<i4'), ('r', '<i4'), ('c', '<i4'), ('octw', '<i4'),
                      ('x', '<f4'), ('y', '<f4'), ('size', '<f4'), ('response', '<f4')])     # struct SiftLoc (36 bytes)
CAP = 1 << 13


def gpu(test):
    """a GPU test; skipped where there is no CUDA device, so the host tests of this file run anywhere"""
    return pytest.mark.gpu(pytest.mark.skipif(not torch.cuda.is_available(), reason='needs a CUDA device')(test))


def _lib():
    from openglue_b200 import _cabi
    return _cabi


def _image(name):
    return np.load(os.path.join(GOLDEN_DIR, name + '.npz'))['image']


# three different images of one size per batch; octave widths 2W, W, W/2, ...: 326 163 81 40 20 10 5 and 234 117 58 29 14 7 3
# cover every residue mod 8
BATCHES = {
    'w163': (120, 163, [('sift_small', 37, 101), ('sift_warp', 0, 0), ('sift_odd', 211, 300)]),
    'w117': (100, 117, [('sift_vga', 300, 411), ('sift_small', 140, 203), ('sift_odd', 5, 17)]),
    'w13': (8, 13, [('sift_tiny', 20, 30), ('sift_small', 100, 100), ('sift_warp', 51, 7)]),
}


def batch_images(key):
    H, W, crops = BATCHES[key]
    return np.stack([_image(n)[y:y + H, x:x + W] for n, y, x in crops])


# ---------------------------------------------------------------------------------------------------------------------
# host restatements

def fma32(a, b, c):
    """float32 fma(a, b, c), correctly rounded: the product is exact in float64; the float64 sum's rounding error (TwoSum) breaks a
    float32 tie, so the double rounding float64 -> float32 never happens"""
    p = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
    c = np.asarray(c, np.float32).astype(np.float64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    nb = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    tie = (s != r64) & (s == (r64 + nb.astype(np.float64)) * 0.5) & (e != 0)
    up = (e > 0) == (nb > r)                                   # the exact sum lies on e's side of the tie
    return np.where(tie & up, nb, r).astype(np.float32)


def reflect101(p, n):
    p = np.asarray(p)
    if n == 1:
        return np.zeros_like(p)
    while True:
        bad = (p < 0) | (p >= n)
        if not bad.any():
            return p
        p = np.where(p < 0, -p, np.where(p >= n, 2 * n - p - 2, p))


def gaussian_taps(sigma):
    buf = (C.c_float * 32)()
    n = _lib().lib().og_sift_gaussian_taps(float(sigma), C.cast(buf, C.c_void_p), 32)
    assert n > 0
    return np.array(buf[:n], np.float32)


def blur32(src, sigma):
    """the kernels' separable blur of src [..., h, w]: rows a running FMA except the last w mod 4 columns, columns symmetric pairs
    by FMA except the last w mod 8, BORDER_REFLECT_101"""
    k = gaussian_taps(sigma)
    n, R = len(k), len(k) // 2
    h, w = src.shape[-2:]
    xs, ys = np.arange(w), np.arange(h)
    sf, su = np.zeros(src.shape, np.float32), np.zeros(src.shape, np.float32)
    for t in range(n):
        v = src[..., reflect101(xs + t - R, w)]
        sf = fma32(v, k[t], sf)
        su = su + v * k[t]
    tmp = np.where(xs < (w & ~3), sf, su)
    sf, su = fma32(tmp, k[R], np.float32(0)), tmp * k[R]
    for t in range(1, R + 1):
        pr = tmp[..., reflect101(ys + t, h), :] + tmp[..., reflect101(ys - t, h), :]
        sf = fma32(pr, k[R + t], sf)
        su = su + pr * k[R + t]
    return np.where(xs < (w & ~7), sf, su)


def blur64(src, sigma):
    """the same convolution in float64 with the same float taps"""
    k = gaussian_taps(sigma).astype(np.float64)
    R = len(k) // 2
    h, w = src.shape[-2:]
    x = src.astype(np.float64)
    xs, ys = np.arange(w), np.arange(h)
    tmp = sum(k[t] * x[..., reflect101(xs + t - R, w)] for t in range(len(k)))
    return sum(k[t] * tmp[..., reflect101(ys + t - R, h), :] for t in range(len(k)))


def upsample2(u8):
    """cv2.resize INTER_LINEAR at exactly x2 of a uint8 image [..., H, W] (exact in float32)"""
    H, W = u8.shape[-2:]
    s = u8.astype(np.float64)

    def axis(n):
        i = np.arange(2 * n)
        lo = np.where(i & 1, i >> 1, (i >> 1) - 1)
        f = np.where(i & 1, 0.25, 0.75)
        return np.maximum(lo, 0), np.minimum(lo + 1, n - 1), f
    xa, xb, fx = axis(W)
    ya, yb, fy = axis(H)
    rows = s[..., xa] * (1 - fx) + s[..., xb] * fx
    return (rows[..., ya, :] * (1 - fy)[:, None] + rows[..., yb, :] * fy[:, None]).astype(np.float32)


def pyramid_sigmas():
    """(the initial blur, cv2's per-level sigmas in double)"""
    s32 = np.float32(1.6)
    sig_diff = float(np.sqrt(np.float32(max(s32 * s32 - np.float32(1.0), np.float32(0.01)))))
    k = 2.0 ** (1.0 / 3)
    sig = [1.6]
    for i in range(1, 6):
        prev = k ** (i - 1) * 1.6
        sig.append(float(np.sqrt((prev * k) ** 2 - prev ** 2)))
    return sig_diff, sig


def num_octaves(H, W):
    return int(np.rint(np.log2(2.0 * min(H, W)) - 2)) + 1


def host_pyramid(u8):
    """the restated pyramid of u8 [B, H, W]: ([gauss [6, B, h, w]], [dog [5, B, h, w]]) per octave"""
    sig_diff, sig = pyramid_sigmas()
    gauss, dog = [], []
    for o in range(num_octaves(*u8.shape[1:])):
        g = [blur32(upsample2(u8), sig_diff) if o == 0 else gauss[-1][3][:, ::2, ::2][:, :gauss[-1].shape[2] // 2, :gauss[-1].shape[3] // 2]]
        for i in range(1, 6):
            g.append(blur32(g[-1], sig[i]))
        gauss.append(np.stack(g))
        dog.append(gauss[-1][1:] - gauss[-1][:-1])
    return gauss, dog


# ---- extrema + interpolation (cv2's adjustLocalExtrema, both thresholds negative) ----

def extrema_candidates(dog):
    """26-neighbour extrema of layers 1..3 inside the 5-pixel border: arrays (b, layer, r, c)"""
    _, B, h, w = dog.shape
    if h <= 10 or w <= 10:
        return [np.zeros(0, np.int64)] * 4
    cen = dog[1:4, :, 5:h - 5, 5:w - 5]
    ge, le = np.ones(cen.shape, bool), np.ones(cen.shape, bool)
    for dl in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                nb = dog[1 + dl:4 + dl, :, 5 + dy:h - 5 + dy, 5 + dx:w - 5 + dx]
                ge &= cen >= nb
                le &= cen <= nb
    l, b, r, c = np.nonzero(((cen > 0) & ge) | ((cen < 0) & le))
    return b, l + 1, r + 5, c + 5


def adjust(dog, o, b, layer, r, c, dt):
    """sift_adjust for every candidate at once, in the kernel's operation order, in dtype dt (float32: bit for bit; float64: the
    reference).  Returns (ok, records [LOC_DTYPE] of the accepted (size from the float64 exp2), margin): margin is float64's
    relative distance from a decision: an offset near 0.5 (the convergence test and the step's rounding), det near 0."""
    _, B, h, w = dog.shape
    D = dog.astype(dt)
    f = dt
    img_scale = f(1) / f(255)
    deriv, second, cross = img_scale * f(0.5), img_scale, img_scale * f(0.25)
    n = len(b)
    b, layer, r, c = (np.array(a, np.int64) for a in (b, layer, r, c))
    alive, done = np.ones(n, bool), np.zeros(n, bool)
    X = [np.zeros(n, dt) for _ in range(3)]
    margin = np.full(n, np.inf)

    def at(dl, dy, dx, m):
        return D[layer[m] + dl, b[m], r[m] + dy, c[m] + dx]

    def derivs(m):
        v2 = at(0, 0, 0, m) * f(2)
        g = [(at(0, 0, 1, m) - at(0, 0, -1, m)) * deriv, (at(0, 1, 0, m) - at(0, -1, 0, m)) * deriv, (at(1, 0, 0, m) - at(-1, 0, 0, m)) * deriv]
        dxx = (at(0, 0, 1, m) + at(0, 0, -1, m) - v2) * second
        dyy = (at(0, 1, 0, m) + at(0, -1, 0, m) - v2) * second
        dss = (at(1, 0, 0, m) + at(-1, 0, 0, m) - v2) * second
        dxy = (at(0, 1, 1, m) - at(0, 1, -1, m) - at(0, -1, 1, m) + at(0, -1, -1, m)) * cross
        dxs = (at(1, 0, 1, m) - at(1, 0, -1, m) - at(-1, 0, 1, m) + at(-1, 0, -1, m)) * cross
        dys = (at(1, 1, 0, m) - at(1, -1, 0, m) - at(-1, 1, 0, m) + at(-1, -1, 0, m)) * cross
        return g, dxx, dyy, dss, dxy, dxs, dys

    with np.errstate(all='ignore'):
        for _ in range(5):
            m = alive & ~done
            if not m.any():
                break
            (b0, b1, b2), a00, a11, a22, a01, a02, a12 = derivs(m)
            a10, a20, a21 = a01, a02, a12
            det = (a00 * (a11 * a22 - a21 * a12) - a01 * (a10 * a22 - a20 * a12)) + a02 * (a10 * a21 - a20 * a11)
            d = np.where(det != 0, f(1) / det, f(0))
            X0 = d * ((b0 * (a11 * a22 - a12 * a21) - a01 * (b1 * a22 - a12 * b2)) + a02 * (b1 * a21 - a11 * b2))
            X1 = d * ((a00 * (b1 * a22 - a12 * b2) - b0 * (a10 * a22 - a12 * a20)) + a02 * (a10 * b2 - b1 * a20))
            X2 = d * ((a00 * (a11 * b2 - b1 * a21) - a01 * (a10 * b2 - b1 * a20)) + b0 * (a10 * a21 - a11 * a20))
            xi, xr, xc = -X2, -X1, -X0
            scale = np.abs(a00 * a11 * a22) + np.abs(a01 * a12 * a20) * 2 + np.abs(a02 * a02 * a11) + np.abs(a12 * a12 * a00) + np.abs(a01 * a01 * a22)
            mg = np.abs(det) / np.maximum(scale, 1e-300)
            for x in (xi, xr, xc):
                ax = np.abs(x.astype(np.float64))
                mg = np.minimum(mg, np.where(ax < 1e6, np.abs(ax - np.floor(ax) - 0.5), np.inf))
            idx = np.nonzero(m)[0]
            margin[idx] = np.minimum(margin[idx], mg)
            conv = (np.abs(xi) < f(0.5)) & (np.abs(xr) < f(0.5)) & (np.abs(xc) < f(0.5))
            for k, x in enumerate((xc, xr, xi)):
                X[k][idx] = x
            done[idx[conv]] = True
            big = f(np.float32(2147483647 // 3))
            step = idx[~conv]
            xs = [x[~conv] for x in (xi, xr, xc)]
            bad = (np.abs(xs[0]) > big) | (np.abs(xs[1]) > big) | (np.abs(xs[2]) > big)
            alive[step[bad]] = False
            step, xs = step[~bad], [x[~bad] for x in xs]
            c[step] += np.rint(xs[2]).astype(np.int64)
            r[step] += np.rint(xs[1]).astype(np.int64)
            layer[step] += np.rint(xs[0]).astype(np.int64)
            out = (layer[step] < 1) | (layer[step] > 3) | (c[step] < 5) | (c[step] >= w - 5) | (r[step] < 5) | (r[step] >= h - 5)
            alive[step[out]] = False
            layer[step[out]], r[step[out]], c[step[out]] = 1, 5, 5          # keeps the gathers of the dead in bounds
        ok = alive & done
        m = ok.copy()
        (dx, dy, ds), dxx, dyy, _, dxy, _, _ = derivs(m)
        xc, xr, xi = X[0][m], X[1][m], X[2][m]
        t = (dx * xc + dy * xr) + ds * xi
        contr = at(0, 0, 0, m) * img_scale + t * f(0.5)
        det = dxx * dyy - dxy * dxy
        dmg = np.abs(det.astype(np.float64)) / np.maximum(np.abs(dxx * dyy).astype(np.float64) + (dxy * dxy).astype(np.float64), 1e-300)
        idx = np.nonzero(m)[0]
        margin[idx] = np.minimum(margin[idx], dmg)
        keep = det > 0
        ok[idx[~keep]] = False
        sel = keep
        rec = np.zeros(int(sel.sum()), LOC_DTYPE)
        p = 1 << o
        rec['o'], rec['layer'], rec['r'], rec['c'] = o, layer[m][sel], r[m][sel], c[m][sel]
        rec['x'] = ((c[m][sel].astype(dt) + xc[sel]) * f(p)).astype(np.float32)
        rec['y'] = ((r[m][sel].astype(dt) + xr[sel]) * f(p)).astype(np.float32)
        rec['octw'] = o + (layer[m][sel] << 8) + (np.rint((xi[sel].astype(np.float64) + 0.5) * 255.0).astype(np.int64) << 16)
        e = ((layer[m][sel].astype(dt) + xi[sel]) / f(3)).astype(np.float32)
        size = ((np.float32(1.6) * np.exp2(e.astype(np.float64)).astype(np.float32)) * np.float32(p)) * np.float32(2)
        rec['size'] = size if dt == np.float32 else (1.6 * np.exp2((layer[m][sel] + xi[sel].astype(np.float64)) / 3) * p * 2)
        rec['response'] = np.abs(contr[sel]).astype(np.float32)
    return ok, rec, margin


def _loc_order(rec):
    return np.lexsort([rec[k].view(np.int32) if rec[k].dtype == np.float32 else rec[k]
                       for k in ('response', 'y', 'x', 'octw', 'c', 'r', 'layer', 'o')])


# ---- orientation (calcOrientationHist + the peak loop), float64 ----

_P = [v * 180 / np.pi for v in (0.9997878412794807, -0.3258083974640975, 0.1555786518463281, -0.04432655554792128)]


def fast_atan2_64(y, x):
    """cv::hal::fastAtan2's polynomial, in float64 (degrees in [0, 360])"""
    ax, ay = np.abs(x), np.abs(y)
    c = np.where(ax >= ay, ay / (ax + np.finfo(np.float64).eps), ax / (ay + np.finfo(np.float64).eps))
    c2 = c * c
    a = (((_P[3] * c2 + _P[2]) * c2 + _P[1]) * c2 + _P[0]) * c
    a = np.where(ax >= ay, a, 90 - a)
    a = np.where(x < 0, 180 - a, a)
    return np.where(y < 0, 360 - a, a)


def orientation_ref(img, L, tol):
    """the peaks of one located extremum on its Gaussian level img [h, w]: [(angle, peak, marginal)].  A bin within tol * max of
    the 0.8 threshold or of a neighbour is listed as marginal, peak or not; so is every peak when a sample's bin is within 1e-6 of
    a rounding boundary."""
    h, w = img.shape
    scl = np.float32(np.float32(L['size'] * np.float32(0.5)) / np.float32(1 << int(L['o'])))
    radius = int(np.rint(np.float32(np.float32(4.5) * scl)))
    sigma = 1.5 * float(scl)
    r0, c0 = int(L['r']), int(L['c'])
    ylo, yhi, xlo, xhi = max(-radius, 1 - r0), min(radius, h - 2 - r0), max(-radius, 1 - c0), min(radius, w - 2 - c0)
    ii, jj = np.meshgrid(np.arange(ylo, yhi + 1), np.arange(xlo, xhi + 1), indexing='ij')
    ii, jj = ii.ravel(), jj.ravel()
    y, x = r0 + ii, c0 + jj
    g = img.astype(np.float64)
    dx, dy = g[y, x + 1] - g[y, x - 1], g[y - 1, x] - g[y + 1, x]
    wt = np.exp((ii * ii + jj * jj) * (-1.0 / (2 * sigma * sigma)))
    binf = 36 / 360 * fast_atan2_64(dy, dx)
    amb = bool((np.abs(binf - np.floor(binf) - 0.5) < 1e-6).any())
    bins = np.rint(binf).astype(np.int64) % 36
    hist = np.bincount(bins, wt * np.hypot(dx, dy), 36)
    hs = (np.roll(hist, 2) + np.roll(hist, -2)) / 16 + (np.roll(hist, 1) + np.roll(hist, -1)) * 4 / 16 + hist * 6 / 16
    mx = hs.max()
    thr = 0.8 * mx
    out = []
    for j in range(36):
        hl, hr, hj = hs[j - 1], hs[(j + 1) % 36], hs[j]
        peak = hj > hl and hj > hr and hj >= thr
        near = min(abs(hj - thr), abs(hj - hl), abs(hj - hr)) <= tol * mx
        if peak or near:
            den = hl - 2 * hj + hr
            b = j + (0.5 * (hl - hr) / den if den != 0 else 0.0)
            b = b + 36 if b < 0 else b - 36 if b >= 36 else b
            a = 360 - 10 * b
            out.append((0.0 if abs(a - 360) < F32_EPS else a, peak, near or amb))
    return out


# ---- descriptors (calcSIFTDescriptor), float64 ----

def describe_ref(gauss, b, x, y, size, angle, octw):
    """cv2's descriptor of one keypoint on the Gaussian level its octave word names, in float64, before the rounding to integers.
    The keypoint's geometry (pixel, radius, rotation) is the kernel's float32 one; every weight and sum is float64."""
    f = np.float32
    octave, layer = octw & 255, (octw >> 8) & 255
    octave = octave if octave < 128 else octave - 256
    scale = f(1) / f(1 << octave) if octave >= 0 else f(1 << -octave)
    img = gauss[octave + 1][layer, b].astype(np.float64)
    rows, cols = img.shape
    sz, ptx, pty = f(f(size) * scale), f(f(x) * scale), f(f(y) * scale)
    ori = f(f(360) - f(angle))
    if abs(f(ori - f(360))) < F32_EPS:
        ori = f(0)
    scl = f(sz * f(0.5))
    px, py = int(np.rint(ptx)), int(np.rint(pty))
    orad = f(ori * f(np.pi / 180))
    cos_t, sin_t = f(np.cos(np.float64(orad))), f(np.sin(np.float64(orad)))
    hist_width = f(f(3) * scl)
    radius = int(np.rint(f(f(f(hist_width * f(1.4142135623730951)) * f(5)) * f(0.5))))
    radius = min(radius, int(np.sqrt(float(cols) * cols + float(rows) * rows)))
    cos_t, sin_t = float(f(cos_t / hist_width)), float(f(sin_t / hist_width))
    ii, jj = np.meshgrid(np.arange(-radius, radius + 1), np.arange(-radius, radius + 1), indexing='ij')
    ii, jj = ii.ravel(), jj.ravel()
    c_rot, r_rot = jj * cos_t - ii * sin_t, jj * sin_t + ii * cos_t
    rbin, cbin = r_rot + 1.5, c_rot + 1.5
    r, c = py + ii, px + jj
    m = (rbin > -1) & (rbin < 4) & (cbin > -1) & (cbin < 4) & (r > 0) & (r < rows - 1) & (c > 0) & (c < cols - 1)
    rbin, cbin, r, c, c_rot, r_rot = rbin[m], cbin[m], r[m], c[m], c_rot[m], r_rot[m]
    dx, dy = img[r, c + 1] - img[r, c - 1], img[r - 1, c] - img[r + 1, c]
    mag = np.hypot(dx, dy) * np.exp((c_rot * c_rot + r_rot * r_rot) * -0.125)
    obin = (fast_atan2_64(dy, dx) - float(ori)) * (8 / 360)
    r0, c0, o0 = np.floor(rbin).astype(np.int64), np.floor(cbin).astype(np.int64), np.floor(obin).astype(np.int64)
    rf, cf, of = rbin - r0, cbin - c0, obin - o0
    o0 = np.where(o0 < 0, o0 + 8, np.where(o0 >= 8, o0 - 8, o0))
    hist = np.zeros((6, 6, 10))
    for dr, wr in ((0, 1 - rf), (1, rf)):
        for dc, wc in ((0, 1 - cf), (1, cf)):
            for do, wo in ((0, 1 - of), (1, of)):
                np.add.at(hist, (r0 + 1 + dr, c0 + 1 + dc, o0 + do), mag * wr * wc * wo)
    hist[:, :, 0] += hist[:, :, 8]
    hist[:, :, 1] += hist[:, :, 9]
    v = hist[1:5, 1:5, :8].ravel()
    v = np.minimum(v, np.sqrt((v * v).sum()) * 0.2)
    return v * (512 / max(np.sqrt((v * v).sum()), F32_EPS))


# ---------------------------------------------------------------------------------------------------------------------
# host tests

def test_workspace_layout():
    """og_sift_workspace_layout writes sift_layout's offsets: octave sizes halve, the regions do not overlap, the total is
    og_sift_workspace_bytes"""
    lib = _lib().lib()
    for B, H, W, cap in ((3, 120, 163, CAP), (1, 8, 13, 7), (2, 375, 500, 1000)):
        out = (C.c_int64 * 64)()
        n = lib.og_sift_workspace_layout(B, H, W, cap, C.cast(out, C.c_void_p), 64)
        nO = num_octaves(H, W)
        assert n == 1 + 4 * nO + 5 and out[0] == nO
        v = np.array(out[:n], np.int64)
        oc = v[1:1 + 4 * nO].reshape(nO, 4)
        loc_off, kp_off, oct_off, cnt_off, total = v[1 + 4 * nO:]
        h, w = 2 * H, 2 * W
        end = 0
        for o in range(nO):
            assert tuple(oc[o, :2]) == (h, w)
            assert oc[o, 2] >= end and oc[o, 3] >= oc[o, 2] + 6 * B * h * w * 4
            end = oc[o, 3] + 5 * B * h * w * 4
            h, w = h // 2, w // 2
        assert end <= loc_off and loc_off + B * cap * 36 <= kp_off and kp_off + B * cap * 20 <= oct_off and oct_off + B * cap * 4 <= cnt_off
        assert cnt_off + 8 * B <= total == lib.og_sift_workspace_bytes(B, H, W, cap)
        assert lib.og_sift_workspace_layout(B, H, W, cap, C.cast(out, C.c_void_p), n - 1) == -1
    assert lib.og_sift_workspace_layout(1, 1, 1, 10, C.cast((C.c_int64 * 64)(), C.c_void_p), 64) == -2


def test_fma32_is_correctly_rounded():
    """the float32 FMA restatement against exact rational arithmetic, on ties built to double-round in float64"""
    from fractions import Fraction
    rng = np.random.default_rng(0)
    a = rng.standard_normal(2000).astype(np.float32)
    b = rng.standard_normal(2000).astype(np.float32)
    c = rng.standard_normal(2000).astype(np.float32) * np.float32(1e-3)
    # c = a float32 midpoint minus a product: the float64 sum lands on the tie, with the error term deciding
    a2 = np.float32(1) + np.arange(1, 200, dtype=np.float32) * np.float32(2 ** -23)
    b2 = np.float32(1) + np.float32(2 ** -23)
    c2 = np.float32(2 ** -24) * np.float32(1) + (-(a2.astype(np.float64) * float(b2))).astype(np.float32)
    A, Bv, Cv = np.concatenate([a, a2]), np.concatenate([b, np.full(len(a2), b2, np.float32)]), np.concatenate([c, c2])
    got = fma32(A, Bv, Cv)
    for x, y, z, g in zip(A, Bv, Cv, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        errs = [abs(Fraction(float(q)) - exact) for q in cands]
        best = min(errs)
        assert abs(Fraction(float(g)) - exact) == best, (x, y, z)


@pytest.mark.parametrize('shape', [(37, 53), (61, 90), (40, 29), (8, 13)])
def test_restated_blur_equals_cv2(shape):
    """the restated upsample, blurs and downsample equal cv2.resize / cv2.GaussianBlur bit for bit, for every pyramid sigma"""
    cv2 = pytest.importorskip('cv2')
    H, W = shape
    u8 = _image('sift_small')[:H, :W]
    up = upsample2(u8)
    assert np.array_equal(up, cv2.resize(u8.astype(np.float32), (2 * W, 2 * H), interpolation=cv2.INTER_LINEAR))
    assert np.array_equal(up[::2, ::2], cv2.resize(up, (W, H), interpolation=cv2.INTER_NEAREST))
    sig_diff, sig = pyramid_sigmas()
    for img in (u8.astype(np.float32), up):
        for s in [sig_diff] + sig[1:]:
            a = blur32(img, s)
            ref = cv2.GaussianBlur(img, (0, 0), s, sigmaY=s, borderType=cv2.BORDER_REFLECT_101)
            assert np.array_equal(a.view(np.int32), ref.view(np.int32)), (shape, s, int((a != ref).sum()))


def _blur_error_ratio(out, src, sigma):
    """max |out - float64 convolution| in units of eps * sum |k| |x| (x >= 0 here, so that sum is the float64 blur of |x|)"""
    ref = blur64(np.abs(src.astype(np.float64)), sigma)
    return float((np.abs(out.astype(np.float64) - blur64(src, sigma)) / np.maximum(ref * F32_EPS, 1e-300)).max())


def test_restated_blur_is_a_gaussian():
    """the restatement is the float64 convolution to a few eps * sum |k| |x| (the independent check of P)"""
    u8 = _image('sift_odd')[:61, :90]
    _, sig = pyramid_sigmas()
    x = upsample2(u8)
    worst = 0.0
    for s in sig[1:]:
        y = blur32(x, s)
        worst = max(worst, _blur_error_ratio(y, x, s))
        x = y
    print(f'\nblur restatement against float64: max error {worst:.2f} eps * sum |k||x|')
    assert worst <= 4


# ---------------------------------------------------------------------------------------------------------------------
# GPU

class Detected:
    """og_sift_detect of one batch, with every stage's results read back from its workspace"""

    def __init__(self, u8, cap=CAP):
        cab = _lib()
        lib = cab.lib()
        B, H, W = u8.shape
        self.u8, self.B, self.H, self.W, self.cap = u8, B, H, W, cap
        self.ws = torch.empty(cab.check_size(lib.og_sift_workspace_bytes(B, H, W, cap), 'ws'), dtype=torch.uint8, device=DEV)
        self.img = torch.from_numpy(u8).to(DEV)
        self.kp_d = torch.empty(B, cap, 5, device=DEV)
        self.oct_d = torch.empty(B, cap, dtype=torch.int32, device=DEV)
        self.count_d = torch.empty(B, dtype=torch.int32, device=DEV)
        cab.check(lib.og_sift_detect(cab.ptr(self.img), 0, B, H, W, cap, cab.ptr(self.ws), self.ws.numel(), cab.ptr(self.kp_d), cab.ptr(self.oct_d),
                                     cab.ptr(self.count_d), cab.stream()), 'og_sift_detect')
        out = (C.c_int64 * 128)()
        n = lib.og_sift_workspace_layout(B, H, W, cap, C.cast(out, C.c_void_p), 128)
        v = np.array(out[:n], np.int64)
        nO = int(v[0])
        oc = v[1:1 + 4 * nO].reshape(nO, 4)
        loc_off, kp_off, oct_off, cnt_off, total = (int(t) for t in v[1 + 4 * nO:])
        assert total == self.ws.numel()
        ws = self.ws.cpu().numpy()

        def arr(off, dtype, shape):
            return ws[off:off + int(np.prod(shape)) * np.dtype(dtype).itemsize].view(dtype).reshape(shape)
        self.gauss = [arr(int(g), np.float32, (6, B, int(h), int(w))) for h, w, g, _ in oc]
        self.dog = [arr(int(d), np.float32, (5, B, int(h), int(w))) for h, w, _, d in oc]
        cnt = arr(cnt_off, np.int32, (2, B))
        self.loc_count, self.kp_count = cnt[0].copy(), cnt[1].copy()
        assert (self.loc_count <= cap).all() and (self.kp_count <= cap).all()
        locs = arr(loc_off, LOC_DTYPE, (B, cap))
        self.locs = [locs[b, :self.loc_count[b]].copy() for b in range(B)]
        kp = arr(kp_off, np.float32, (B, cap, 5))
        octs = arr(oct_off, np.int32, (B, cap))
        self.raw_kp = [kp[b, :self.kp_count[b]].copy() for b in range(B)]
        self.raw_oct = [octs[b, :self.kp_count[b]].copy() for b in range(B)]
        self.count = self.count_d.cpu().numpy()
        self.kp = [self.kp_d[b, :self.count[b]].cpu().numpy() for b in range(B)]
        self.octave = [self.oct_d[b, :self.count[b]].cpu().numpy() for b in range(B)]


_DETECTED = {}


def detected(key):
    if key not in _DETECTED:
        _DETECTED[key] = Detected(batch_images(key))
    return _DETECTED[key]


@gpu
@pytest.mark.parametrize('key', list(BATCHES))
def test_pyramid_exact(key):
    """P: every Gaussian and DoG level of every octave and image, bit for bit, each from the kernels' own previous level; and the
    float64 convolution within a few eps * sum |k| |x|"""
    d = detected(key)
    sig_diff, sig = pyramid_sigmas()
    assert len(d.gauss) == num_octaves(d.H, d.W)
    worst = 0.0
    for o, (g, dg) in enumerate(zip(d.gauss, d.dog)):
        if o == 0:
            up = upsample2(d.u8)
            want = blur32(up, sig_diff)
            worst = max(worst, _blur_error_ratio(g[0], up, sig_diff))
        else:
            p = d.gauss[o - 1][3]
            want = p[:, ::2, ::2][:, :p.shape[1] // 2, :p.shape[2] // 2]
        assert np.array_equal(g[0].view(np.int32), want.view(np.int32)), (key, o, 0, int((g[0] != want).sum()))
        for i in range(1, 6):
            want = blur32(g[i - 1], sig[i])
            bad = g[i] != want
            assert not bad.any(), (key, o, i, 'images', sorted(set(np.nonzero(bad)[0].tolist())), 'columns', sorted(set(np.nonzero(bad)[2].tolist()))[:16])
            worst = max(worst, _blur_error_ratio(g[i], g[i - 1], sig[i]))
        assert np.array_equal(dg.view(np.int32), (g[1:] - g[:-1]).view(np.int32)), (key, o)
    print(f'\n[{key}] P: {len(d.gauss)} octaves, widths {[x.shape[3] for x in d.gauss]}; blur against float64 <= {worst:.2f} eps * sum |k||x|')
    assert worst <= 4


def _restated_extrema(d):
    """per octave, over every 26-neighbour candidate of every image: (image, ok32, records32, ok64, records64, float64 margin)"""
    per = []
    for o, dog in enumerate(d.dog):
        b, l, r, c = extrema_candidates(dog)
        ok32, rec32, _ = adjust(dog, o, b, l, r, c, np.float32)
        ok64, rec64, margin = adjust(dog, o, b, l, r, c, np.float64)
        per.append((b, ok32, rec32, ok64, rec64, margin))
    return per


@gpu
@pytest.mark.parametrize('key', list(BATCHES))
def test_extrema_and_interpolation(key):
    """X: the located records equal the float32 restatement (multiset: atomics fix their order) bit for bit, size within 1 ulp;
    against float64 every candidate agrees within tolerances unless float64 puts it within a margin of a decision"""
    d = detected(key)
    per = _restated_extrema(d)
    n_cand = sum(len(p[0]) for p in per)
    one_sided, max_dpos, max_dpos_all, max_dresp = 0, 0.0, 0.0, 0.0
    for b in range(d.B):
        gpu = d.locs[b]
        ref = np.concatenate([p[2][p[0][p[1]] == b] for p in per])
        assert len(gpu) == len(ref), (key, b, len(gpu), len(ref))
        g, r = gpu[_loc_order(gpu)], ref[_loc_order(ref)]
        for k in ('o', 'layer', 'r', 'c', 'octw', 'x', 'y', 'response'):
            assert np.array_equal(g[k].view(np.int32), r[k].view(np.int32)), (key, b, k)
        ulp = np.abs(g['size'].view(np.int32).astype(np.int64) - r['size'].view(np.int32))
        assert ulp.max(initial=0) <= 1, (key, b)
    for _, ok32, rec32, ok64, rec64, margin in per:
        # per candidate: the float32 and float64 restatements, in candidate order
        i32, i64 = np.cumsum(ok32) - 1, np.cumsum(ok64) - 1
        both = ok32 & ok64
        same = np.zeros(len(ok32), bool)
        a, z = rec32[i32[both]], rec64[i64[both]]
        same_px = (a['layer'] == z['layer']) & (a['r'] == z['r']) & (a['c'] == z['c'])
        same[np.nonzero(both)[0][same_px]] = True
        diff = ~same & (ok32 | ok64)
        assert (margin[diff] <= 1e-3).all(), (key, margin[diff].max())
        one_sided += int(diff.sum())
        if same_px.any():
            a, z = a[same_px], z[same_px]
            scale = (1 << a['o']).astype(np.float64)
            dpos = np.maximum(np.abs(a['x'] - z['x'].astype(np.float64)), np.abs(a['y'] - z['y'].astype(np.float64))) / scale
            m = margin[np.nonzero(both)[0][same_px]]
            max_dpos = max(max_dpos, float(dpos[m > 1e-3].max(initial=0)))
            max_dpos_all = max(max_dpos_all, float(dpos.max(initial=0)))
            dresp = np.abs(a['response'] - z['response'].astype(np.float64)) / np.maximum(z['response'], 1e-12)
            max_dresp = max(max_dresp, float(dresp.max(initial=0)))
            assert np.array_equal(a['octw'] & 0xffff, z['octw'] & 0xffff)
    print(f'\n[{key}] X: {n_cand} candidates, {sum(len(x) for x in d.locs)} located; float32 vs float64: {one_sided} on one side only (all near a '
          f'decision), max |dpos| {max_dpos:.2e} octave px away from decisions ({max_dpos_all:.2e} overall), max relative |dresponse| {max_dresp:.2e}')
    assert one_sided <= max(2, n_cand // 200)
    assert max_dpos <= 1e-3 and max_dresp <= 1e-3


@gpu
@pytest.mark.parametrize('key', list(BATCHES))
def test_orientations(key):
    """O: the raw keypoints equal, as a multiset, the float64 histogram's peaks of every located extremum; angles within 1e-2
    degrees; a peak within a margin of the 0.8 threshold or of a neighbour may be on one side only"""
    d = detected(key)
    tol = 1e-4
    n_marg, max_da, n_kp = 0, 0.0, 0
    for b in range(d.B):
        gk, go = d.raw_kp[b], d.raw_oct[b]
        groups = {}
        for k, o in zip(gk, go):
            groups.setdefault((k[0], k[1], k[2], k[4], int(o)), []).append(float(k[3]))
        refs = {}
        for L in d.locs[b]:
            key_ = (np.float32(L['x'] * np.float32(0.5)), np.float32(L['y'] * np.float32(0.5)), np.float32(L['size'] * np.float32(0.5)),
                    L['response'], int((L['octw'] & ~255) | ((L['octw'] - 1) & 255)))
            refs.setdefault(key_, []).extend(orientation_ref(d.gauss[L['o']][L['layer'], b], L, tol))
        assert set(groups) <= set(refs), (key, b, 'keypoints at no located extremum')
        for k_, peaks in refs.items():
            got = sorted(groups.get(k_, []))
            left = list(peaks)
            for a in got:
                dist = [min(abs(a - p) % 360, 360 - abs(a - p) % 360) for p, _, _ in left]
                j = int(np.argmin(dist)) if dist else -1
                assert j >= 0 and (dist[j] <= 1e-2 or left[j][2]), (key, b, k_, got, peaks)
                _, peak, marginal = left.pop(j)
                if marginal:
                    n_marg += int(not peak or dist[j] > 1e-2)                # a peak of the kernels' only
                else:
                    assert peak
                    max_da = max(max_da, dist[j])
            assert all(m or not p for _, p, m in left), (key, b, k_, got, peaks)
            n_marg += sum(int(p) for _, p, _ in left)                          # a peak of float64's only
            n_kp += len(got)
    print(f'\n[{key}] O: {n_kp} raw keypoints from {sum(len(x) for x in d.locs)} extrema; max |dangle| {max_da:.2e} deg; {n_marg} marginal peaks '
          f'on one side only')
    assert n_marg <= max(2, n_kp // 200)


def _cv_sort_unique(kp, octv):
    order = np.lexsort((-octv.astype(np.int64), -kp[:, 4], kp[:, 3], -kp[:, 2], kp[:, 1], kp[:, 0]))
    kp, octv = kp[order], octv[order]
    keep = np.ones(len(kp), bool)
    keep[1:] = (kp[1:, :4] != kp[:-1, :4]).any(1)
    return kp[keep], octv[keep]


@gpu
@pytest.mark.parametrize('key', list(BATCHES))
def test_sort_unique_exact(key):
    """S: og_sift_detect's keypoints are the raw buffer in cv2's KeyPoint12_LessThan order without (x, y, size, angle) repeats"""
    d = detected(key)
    dups = 0
    for b in range(d.B):
        kp, octv = _cv_sort_unique(d.raw_kp[b], d.raw_oct[b])
        dups += d.kp_count[b] - len(kp)
        assert d.count[b] == len(kp)
        assert np.array_equal(d.kp[b].view(np.int32), kp.view(np.int32)) and np.array_equal(d.octave[b], octv)
    print(f'\n[{key}] S: {d.count.tolist()} keypoints, {dups} duplicates removed')


@gpu
def test_padded_count_and_overflow():
    """S: at a capacity that cuts one image of the batch, the others' outputs equal the uncut run's, the cut image is flagged, and
    og_sift_detect reports its count above the capacity"""
    cab = _lib()
    lib = cab.lib()
    full = detected('w163')
    cut = int(np.argmax(full.kp_count))
    others = [b for b in range(full.B) if b != cut]
    cap = int(max(full.kp_count[others].max(), full.loc_count[others].max()))
    assert cap < full.kp_count[cut]
    B, H, W = full.u8.shape
    ws = torch.empty(cab.check_size(lib.og_sift_workspace_bytes(B, H, W, cap), 'ws'), dtype=torch.uint8, device=DEV)
    kp, octv = torch.empty(B, cap, 5, device=DEV), torch.empty(B, cap, dtype=torch.int32, device=DEV)
    count, ovf = torch.empty(B, dtype=torch.int32, device=DEV), torch.full((B,), 7, dtype=torch.int32, device=DEV)
    cab.check(lib.og_sift_detect_padded(cab.ptr(full.img), 0, B, H, W, cap, cab.ptr(ws), ws.numel(), cab.ptr(kp), cab.ptr(octv), cab.ptr(count),
                                        cab.ptr(ovf), cab.stream()), 'og_sift_detect_padded')
    count_h, ovf_h = count.cpu().numpy(), ovf.cpu().numpy()
    assert ovf_h.tolist() == [int(b == cut) for b in range(B)]
    assert 0 < count_h[cut] <= cap
    for b in others:
        assert count_h[b] == full.count[b]
        assert np.array_equal(kp[b, :count_h[b]].cpu().numpy().view(np.int32), full.kp[b].view(np.int32))
        assert np.array_equal(octv[b, :count_h[b]].cpu().numpy(), full.octave[b])
    cab.check(lib.og_sift_detect(cab.ptr(full.img), 0, B, H, W, cap, cab.ptr(ws), ws.numel(), cab.ptr(kp), cab.ptr(octv), cab.ptr(count),
                                 cab.stream()), 'og_sift_detect')
    c2 = count.cpu().numpy()
    assert c2[cut] > cap and [c2[b] for b in others] == [full.count[b] for b in others]


def _select(kps, cap, radius, max_kp):
    """og_sift_select of a batch of keypoint lists (x, y, response), padded to cap"""
    cab = _lib()
    lib = cab.lib()
    B = len(kps)
    kp = np.zeros((B, cap, 5), np.float32)
    for b, k in enumerate(kps):
        kp[b, :len(k), 0], kp[b, :len(k), 1], kp[b, :len(k), 4] = k[:, 0], k[:, 1], k[:, 2]
        kp[b, :len(k), 2] = 3.0
    kp_d = torch.from_numpy(kp).to(DEV)
    count = torch.tensor([len(k) for k in kps], dtype=torch.int32, device=DEV)
    work = torch.empty(cab.check_size(lib.og_sift_select_workspace_bytes(B, cap), 'ws'), dtype=torch.uint8, device=DEV)
    sel, n_sel = torch.full((B, cap), -1, dtype=torch.int32, device=DEV), torch.empty(B, dtype=torch.int32, device=DEV)
    cab.check(lib.og_sift_select(cab.ptr(kp_d), cab.ptr(count), B, cap, float(radius), int(max_kp), cab.ptr(work), work.numel(), cab.ptr(sel),
                                 cab.ptr(n_sel), cab.stream()), 'og_sift_select')
    n_sel = n_sel.cpu().numpy()
    return [sel[b, :n_sel[b]].cpu().numpy().tolist() for b in range(B)]


def _greedy(k, radius, max_kp):
    if radius <= 0:                                            # no NMS at all (greedy_select would still merge coincident points)
        order = sorted(range(len(k)), key=lambda i: (-float(k[i, 2]), i))
        return order[:max_kp] if max_kp > 0 else order
    return greedy_select(k[:, :2], k[:, 2], np.float32(radius), max_kp)


def _kps(n, seed, extent=60.0, levels=None):
    rng = np.random.default_rng(seed)
    k = np.zeros((n, 3), np.float32)
    k[:, :2] = np.round(rng.random((n, 2)) * extent * 4) / 4                      # quarter pixels: many exact distances
    k[:, 2] = rng.integers(0, levels, n) if levels else rng.random(n)
    return k


@gpu
def test_select_edges():
    """N: greedy radius NMS + top-k against the host restatement at its edges"""
    r = np.float32(4.5)
    on = np.float32([[0, 0, 1.0], [4.5, 0, 0.9], [0, 4.5, 0.8], [-4.5, 0, 0.7], [20, 20, 0.6], [23, 24, 0.5], [40, 40, 0.4]])
    out = np.float32([[0, 0, 1.0], [np.nextafter(np.float32(4.5), np.float32(9)), 0, 0.9], [20, 20, 0.8],
                      [20, np.nextafter(np.float32(24.5), np.float32(99)), 0.7]])
    same_x = np.float32([[10, y, 1 - 0.01 * y] for y in np.arange(0, 30, 1.5)])
    eq = _kps(300, 1, levels=1)                                                   # all responses equal
    cases = [([on], r, -1), ([on], np.float32(5.0), -1), ([out], r, -1), ([same_x], r, -1), ([eq], r, -1), ([eq], 0.0, -1), ([eq], -1.0, 10)]
    n = 200
    k = _kps(n, 2, levels=40)
    for m in (1, n - 1, n, n + 1, 0):
        cases.append(([k], r, m))
        cases.append(([k], 0.0, m))
    for batch, rad, m in cases:
        cap = max(len(x) for x in batch)
        got = _select(batch, cap, rad, m)
        for b, x in enumerate(batch):
            assert got[b] == _greedy(x, rad, m), (rad, m, len(x))


@gpu
@pytest.mark.parametrize('cap', [1000, 1025, 4097])
def test_select_batch_counts_and_caps(cap):
    """N: a batch whose counts are 0, 1 and cap, at capacities that are not powers of two, more than 1024 keypoints per CTA"""
    n = min(cap, 3000)
    big = _kps(cap, cap, extent=np.sqrt(n) * 4, levels=n // 3)
    batch = [np.zeros((0, 3), np.float32), _kps(1, 5), big, _kps(n - 7, cap + 1, extent=np.sqrt(n) * 3, levels=50)]
    for rad, m in ((4.5, -1), (4.5, 300), (0.0, 1025), (2.0, cap - 1)):
        got = _select(batch, cap, rad, m)
        for b, x in enumerate(batch):
            assert got[b] == _greedy(x, rad, m), (cap, rad, m, b)


def _describe(d, kp_list, oct_list):
    """og_sift_describe of supplied keypoints on d's pyramid: raw descriptors per image"""
    cab = _lib()
    lib = cab.lib()
    B, cap = d.B, d.cap
    n = max(len(k) for k in kp_list)
    kp, octv = np.zeros((B, cap, 5), np.float32), np.zeros((B, cap), np.int32)
    for b in range(B):
        kp[b, :len(kp_list[b])], octv[b, :len(kp_list[b])] = kp_list[b], oct_list[b]
    kp_d, oct_d = torch.from_numpy(kp).to(DEV), torch.from_numpy(octv).to(DEV)
    sel = torch.arange(cap, dtype=torch.int32, device=DEV).repeat(B, 1)
    n_sel = torch.tensor([len(k) for k in kp_list], dtype=torch.int32, device=DEV)
    out = [torch.empty(B, n, *s, device=DEV) for s in ((2, 3), (), (128,), (128,))]
    cab.check(lib.og_sift_describe(cab.ptr(d.ws), B, d.H, d.W, cap, cab.ptr(kp_d), cab.ptr(oct_d), cab.ptr(sel), cab.ptr(n_sel), n, n, 1,
                                   *[cab.ptr(t) for t in out], cab.stream()), 'og_sift_describe')
    raw = out[3].cpu().numpy()
    return [raw[b, :len(kp_list[b])] for b in range(B)]


def _check_descriptors(d, kp_list, oct_list, raw, margin=0.05):
    """every entry within 1 of the float64 value rounded, and equal to it wherever that value is further than margin from .5"""
    n_entries, n_near, worst = 0, 0, 0.0
    for b in range(d.B):
        for k, o, g in zip(kp_list[b], oct_list[b], raw[b]):
            v = describe_ref(d.gauss, b, k[0], k[1], k[2], k[3], int(o))
            want = np.clip(np.rint(v), 0, 255)
            diff = np.abs(g - want)
            near = np.abs(v - np.floor(v) - 0.5) <= margin
            assert diff.max() <= 1 and (diff[~near] == 0).all(), (b, k, o, np.nonzero(diff)[0], v[diff > 0], g[diff > 0])
            n_entries += len(v)
            n_near += int((diff > 0).sum())
            worst = max(worst, float(np.abs(g - np.clip(v, 0, 255)).max()))
    return n_entries, n_near, worst


@gpu
def test_descriptors_synthetic():
    """D: keypoints on and near every border, octave -1 to the last octave with a level, every layer, sizes up to the radius clamp,
    angles 0, 359.99 and within FLT_EPSILON of 360"""
    d = detected('w117')
    angles = np.float32([0, 1e-7, np.nextafter(np.float32(360), np.float32(0)), 359.99, 90, 180.5, 271.25])
    kp_list, oct_list = [], []
    for b in range(d.B):
        kps, octs = [], []
        t = b
        for oi, g in enumerate(d.gauss):
            rows, cols = g.shape[2:]
            octave = oi - 1
            scale = 2.0 ** octave                                          # base coordinates = octave coordinates * 2^octave
            xs = [0, 0.4, 0.51, 1, 1.5, cols / 2, cols - 2, cols - 1.5, cols - 1, cols - 0.6]
            ys = [0, 0.6, 1, 1.49, rows / 2, rows - 2, rows - 1.49, rows - 1]
            pts = [(x, rows / 2) for x in xs] + [(cols / 2, y) for y in ys] + [(0, 0), (cols - 1, rows - 1), (0.5, rows - 1.5)]
            diag = np.hypot(rows, cols)
            sizes = [3.2, 5.0] + ([diag / 4, diag] if diag < 40 else [9.0])
            for x, y in pts:
                t += 1
                layer = 1 + t % 3
                s = sizes[t % len(sizes)]
                kps.append((x * scale, y * scale, s * scale, angles[t % len(angles)], 1.0))
                octs.append((octave & 255) | (layer << 8) | (128 << 16))
        kp_list.append(np.array(kps, np.float32))
        oct_list.append(np.array(octs, np.int32))
    raw = _describe(d, kp_list, oct_list)
    n, near, worst = _check_descriptors(d, kp_list, oct_list, raw)
    print(f'\n[w117] D synthetic: {sum(len(k) for k in kp_list)} keypoints, {n} entries, {near} one apart (all near .5), max |raw - float64| {worst:.3f}')


@gpu
def test_descriptors_of_selected_keypoints():
    """D: every keypoint the selection keeps (radius 4.5, top 2048) on the real crops, against the float64 descriptor"""
    cab = _lib()
    lib = cab.lib()
    d = detected('w117')
    B, cap = d.B, d.cap
    work = torch.empty(cab.check_size(lib.og_sift_select_workspace_bytes(B, cap), 'ws'), dtype=torch.uint8, device=DEV)
    sel, n_sel = torch.empty(B, cap, dtype=torch.int32, device=DEV), torch.empty(B, dtype=torch.int32, device=DEV)
    cab.check(lib.og_sift_select(cab.ptr(d.kp_d), cab.ptr(d.count_d), B, cap, 4.5, 2048, cab.ptr(work), work.numel(), cab.ptr(sel), cab.ptr(n_sel),
                                 cab.stream()), 'og_sift_select')
    n_sel = n_sel.cpu().numpy()
    idx = [sel[b, :n_sel[b]].cpu().numpy() for b in range(B)]
    kp_list = [d.kp[b][idx[b]] for b in range(B)]
    oct_list = [d.octave[b][idx[b]] for b in range(B)]
    raw = _describe(d, kp_list, oct_list)
    n, near, worst = _check_descriptors(d, kp_list, oct_list, raw)
    print(f'\n[w117] D selected: {n_sel.tolist()} keypoints, {n} entries, {near} one apart (all near .5), max |raw - float64| {worst:.3f}')
    assert min(n_sel) > 20
