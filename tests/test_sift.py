"""OpenCV SIFT front-end (openglue_b200.OpenCVSIFT, csrc/sift.cuh) against fixtures minted from the unmodified reference with cv2
4.13 (oracle/gen_golden_sift.py).  The GPU tests read only tests/golden/; they need neither cv2 nor the reference.

Exact:     E1 the uint8 quantisation; E2 NMS + top-k, RootSIFT and LAFs driven by cv2's own raw keypoints and descriptors;
           E3 the fastAtan2 restatement.
Measured:  A1 raw keypoints against cv2's (recall and precision); A2 descriptors of matched keypoints; A3 the final outputs
           against the reference's.  The measured distributions are printed (pytest -s).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from oracle.gen_golden_sift import ref_descriptors

IMAGES = ['sift_tiny', 'sift_small', 'sift_odd', 'sift_vga', 'sift_warp']
ALL = IMAGES + ['sift_uniform']
DEV = 'cuda:0'
MAX_KP, RADIUS = 2048, 4.5
# A1's match criterion
PT_TOL, SIZE_RTOL, ANGLE_TOL, RESP_RTOL = 0.01, 1e-4, 0.05, 1e-3


def _fx(name):
    return dict(np.load(os.path.join(GOLDEN_DIR, name + '.npz')))


def _lib():
    from openglue_b200 import _cabi
    return _cabi


def _ulp_diff(a, b):
    a = np.ascontiguousarray(a, np.float32).view(np.int32).astype(np.int64)
    b = np.ascontiguousarray(b, np.float32).view(np.int32).astype(np.int64)
    a = np.where(a < 0, -(a & 0x7fffffff), a)
    b = np.where(b < 0, -(b & 0x7fffffff), b)
    return np.abs(a - b)


# ---------------------------------------------------------------------------------------------------------------------
# host restatements (no GPU)

def greedy_select(pt, resp, radius, max_kp):
    """nms_keypoints + the top-k of detect_kpts_opencv with the kernels' tie rule (response desc, index asc): kept indices in
    output order."""
    order = sorted(range(len(resp)), key=lambda i: (-float(resp[i]), i))
    p = pt.astype(np.float64)
    removed = np.zeros(len(resp), bool)
    kept = []
    for i in order:
        if removed[i]:
            continue
        kept.append(i)
        d2 = ((p - p[i]) ** 2).sum(1)
        removed |= d2 <= radius * radius
    return kept[:max_kp] if max_kp > 0 else kept


def rootsift_laf(pt, size, angle, resp, raw):
    """normalize_descriptors(root_norm=True) + lafs_from_opencv_kpts as the kernels compute them (scale * cos / sin rounded once
    from double)"""
    d = raw.astype(np.float32)
    d = np.sqrt(d / np.abs(d).sum(1, keepdims=True, dtype=np.float32)).astype(np.float32)
    s = (6.0 * size.astype(np.float64)).astype(np.float32)
    th = (-angle.astype(np.float32)) * np.float32(np.pi / 180)
    sc = (s.astype(np.float64) * np.cos(th.astype(np.float64))).astype(np.float32)
    ss = (s.astype(np.float64) * np.sin(th.astype(np.float64))).astype(np.float32)
    lafs = np.empty((len(s), 2, 3), np.float32)
    lafs[:, 0, 0], lafs[:, 0, 1], lafs[:, 1, 0], lafs[:, 1, 1] = sc, ss, -ss, sc
    lafs[:, :, 2] = pt
    return lafs, resp.astype(np.float32), d


def check_selection(fx, kept, lafs, scores, desc):
    """E2's rule: the selected responses equal the reference's as a multiset; a keypoint whose response is unique among the raw
    keypoints is the reference's own (LAF within 1 ulp, descriptor within 2 ulp); a tied one is some member of its class."""
    ref_s = fx['ref_scores']
    assert len(kept) == len(ref_s)
    assert np.array_equal(np.sort(scores), np.sort(ref_s))
    vals, counts = np.unique(fx['kp_response'], return_counts=True)
    unique = set(vals[counts == 1].tolist())
    pos = {float(s): i for i, s in enumerate(ref_s)}
    ref_desc = ref_descriptors(fx)
    n_unique, laf_ulps = 0, []
    for j, s in enumerate(scores):
        if float(s) in unique:
            i = pos[float(s)]
            laf_ulps.append(int(_ulp_diff(lafs[j], fx['ref_lafs'][i]).max()))
            assert _ulp_diff(desc[j], ref_desc[i]).max() <= 2
            n_unique += 1
    # numpy's float32 cos / sin (the reference's) are not correctly rounded: one LAF entry in a few thousand is 2 ulp away
    laf_ulps = np.array(laf_ulps, np.int64)
    assert laf_ulps.size == 0 or (laf_ulps.max() <= 2 and (laf_ulps <= 1).mean() >= 0.995), np.bincount(laf_ulps)
    return n_unique


@pytest.mark.parametrize('name', IMAGES)
def test_selection_restatement_matches_reference(name):
    """E2 on the host: the greedy restatement on cv2's raw keypoints gives the reference's selection, RootSIFT and LAFs"""
    fx = _fx(name)
    kept = greedy_select(fx['kp_pt'], fx['kp_response'], RADIUS, MAX_KP)
    lafs, scores, desc = rootsift_laf(fx['kp_pt'][kept], fx['kp_size'][kept], fx['kp_angle'][kept], fx['kp_response'][kept], fx['desc_raw'][kept])
    assert check_selection(fx, kept, lafs, scores, desc) > 0


def test_fixtures_reproduce_from_cv2():
    """the stored raw keypoints and descriptors are what cv2 computes for the stored images"""
    cv2 = pytest.importorskip('cv2')
    for name in ALL:
        fx = _fx(name)
        kpts, desc = cv2.SIFT_create(contrastThreshold=-10000, edgeThreshold=-10000).detectAndCompute(fx['image'], None)
        assert len(kpts) == len(fx['kp_size']), name
        if not kpts:
            continue
        assert np.array_equal(np.array([k.pt for k in kpts], np.float32), fx['kp_pt'])
        assert np.array_equal(np.array([k.angle for k in kpts], np.float32), fx['kp_angle'])
        assert np.array_equal(np.array([k.octave for k in kpts], np.int32), fx['kp_octave'])
        assert np.array_equal(desc, fx['desc_raw'].astype(np.float32))


def test_gaussian_taps():
    """og_sift_gaussian_taps: cv2's float Gaussian kernel for the pyramid's sigmas (against cv2 where it is installed)"""
    cab = _lib()
    lib = cab.lib()
    buf = (C.c_float * 32)()
    k = 2 ** (1 / 3)
    sigmas = [float(np.sqrt(np.float32(1.6) * np.float32(1.6) - np.float32(1.0)).astype(np.float32))] + \
             [1.6 * np.sqrt((k ** i) ** 2 - (k ** (i - 1)) ** 2) for i in range(1, 6)]
    for s in sigmas:
        n = lib.og_sift_gaussian_taps(s, C.cast(buf, C.c_void_p), 32)
        assert n == (int(np.rint(s * 8 + 1)) | 1)
        taps = np.array(buf[:n], np.float32)
        assert np.array_equal(taps, taps[::-1]) and abs(float(taps.sum(dtype=np.float64)) - 1) < 1e-6
        try:
            import cv2
        except ImportError:
            continue
        assert np.array_equal(taps, cv2.getGaussianKernel(n, s, cv2.CV_32F).ravel()), s
    assert lib.og_sift_gaussian_taps(30.0, C.cast(buf, C.c_void_p), 32) == -2          # OG_EUNSUPPORTED
    assert lib.og_sift_gaussian_taps(-1.0, C.cast(buf, C.c_void_p), 32) == -1


def test_argument_validation():
    """the C entry points refuse bad arguments before touching the GPU"""
    cab = _lib()
    lib = cab.lib()
    p = C.c_void_p(16)
    assert lib.og_sift_workspace_bytes(0, 64, 64, 100) == -1
    assert lib.og_sift_workspace_bytes(1, 64, 64, 0) == -1
    assert lib.og_sift_workspace_bytes(1, 1, 1, 10) == -2                           # no octave
    n = lib.og_sift_workspace_bytes(2, 64, 80, 1000)
    assert n > 2 * 11 * 4 * 64 * 80 * 4
    assert lib.og_sift_detect(None, 0, 1, 64, 80, 1000, p, n, p, p, p, None) == -1
    assert lib.og_sift_detect(p, 2, 1, 64, 80, 1000, p, n, p, p, p, None) == -1       # dtype
    assert lib.og_sift_detect(p, 0, 2, 64, 80, 1000, p, n - 1, p, p, p, None) == -1   # workspace too small
    m = lib.og_sift_select_workspace_bytes(1, 1000)
    assert m == 4 * 1024 * 4
    assert lib.og_sift_select(p, p, 1, 1000, 4.5, 10, p, m - 1, p, p, None) == -1
    assert lib.og_sift_select(p, p, 1, 1000, float('nan'), 10, p, m, p, p, None) == -1
    assert lib.og_sift_select(None, p, 1, 1000, 4.5, 10, p, m, p, p, None) == -1
    assert lib.og_sift_describe(p, 1, 64, 80, 1000, p, p, p, p, 0, 1, 1, p, p, p, None, None) == -1
    assert lib.og_sift_describe(None, 1, 64, 80, 1000, p, p, p, p, 8, 1, 1, p, p, p, None, None) == -1
    assert lib.og_sift_rootsift_laf(p, p, -1, 1, p, p, p, None) == -1
    assert lib.og_sift_fast_atan2(p, None, 4, 0, p, None) == -1


def test_module_refuses_cpu_and_batches_in_forward():
    import openglue_b200
    m = openglue_b200.OpenCVSIFT(max_keypoints=2048)
    assert openglue_b200.sift_create_torch(2048, 9., True).max_keypoints == 2048
    with pytest.raises(RuntimeError, match='CUDA'):
        m(torch.zeros(1, 1, 64, 64))
    with pytest.raises(AssertionError):
        m(torch.zeros(2, 1, 64, 64))
    with pytest.raises(TypeError):
        m(np.zeros((64, 64), np.uint8))


# ---------------------------------------------------------------------------------------------------------------------
# GPU

def _detect_all(fx):
    """og_sift_detect on the fixture image, then og_sift_describe of EVERY keypoint: (pt, size, angle, response, octave, raw desc)"""
    from openglue_b200 import OpenCVSIFT
    cab = _lib()
    lib = cab.lib()
    img = torch.from_numpy(fx['image']).to(DEV)[None, None]
    m = OpenCVSIFT(max_keypoints=-1, nms_diameter=0.0)                   # nms off, no top-k: sel = every keypoint by response
    r = m._detect_select(m._image(img))
    n = int(r.count[0])
    H, W = img.shape[2:]
    sel = torch.arange(m.capacity, dtype=torch.int32, device=DEV)[None]
    n_sel = torch.tensor([n], dtype=torch.int32, device=DEV)
    oc = max(n, 1)
    out = [torch.empty(1, oc, *s, device=DEV) for s in ((2, 3), (), (128,), (128,))]
    st = cab.stream()
    cab.check(lib.og_sift_describe(cab.ptr(r.ws), 1, H, W, m.capacity, cab.ptr(r.kp), cab.ptr(r.octave), cab.ptr(sel), cab.ptr(n_sel), oc, n, 1,
                                   *[cab.ptr(t) for t in out], st), 'og_sift_describe')
    kp = r.kp[0, :n].cpu().numpy()
    return dict(pt=kp[:, :2], size=kp[:, 2], angle=kp[:, 3], response=kp[:, 4], octave=r.octave[0, :n].cpu().numpy(),
                raw=out[3][0, :n].cpu().numpy())


def match_keypoints(a_pt, a_size, a_angle, a_resp, a_oct, b_pt, b_size, b_angle, b_resp, b_oct):
    """for each keypoint of a, the index of a keypoint of b meeting A1's criterion (-1: none)"""
    order = np.argsort(b_pt[:, 0], kind='stable')
    bx = b_pt[order, 0]
    out = np.full(len(a_pt), -1, np.int64)
    for i in range(len(a_pt)):
        lo, hi = np.searchsorted(bx, a_pt[i, 0] - PT_TOL, 'left'), np.searchsorted(bx, a_pt[i, 0] + PT_TOL, 'right')
        for j in order[lo:hi]:
            da = abs(float(a_angle[i]) - float(b_angle[j])) % 360.0
            if ((a_oct[i] & 0xffff) == (b_oct[j] & 0xffff) and np.hypot(*(a_pt[i] - b_pt[j])) <= PT_TOL
                    and abs(a_size[i] - b_size[j]) <= SIZE_RTOL * b_size[j] and min(da, 360 - da) <= ANGLE_TOL
                    and abs(a_resp[i] - b_resp[j]) <= RESP_RTOL * b_resp[j]):
                out[i] = j
                break
    return out


@pytest.mark.gpu
def test_fast_atan2_bit_exact():
    """E3: the kernels' scalar fastAtan2 equals cv2.fastAtan2 on the fixture table, bit for bit"""
    cab = _lib()
    t = _fx('sift_atan')
    y, x = torch.from_numpy(t['y']).to(DEV), torch.from_numpy(t['x']).to(DEV)
    out = torch.empty_like(y)
    cab.check(cab.lib().og_sift_fast_atan2(cab.ptr(y), cab.ptr(x), y.numel(), 0, cab.ptr(out), cab.stream()), 'og_sift_fast_atan2')
    assert np.array_equal(out.cpu().numpy().view(np.int32), t['angle'].view(np.int32))


@pytest.mark.gpu
@pytest.mark.parametrize('name', IMAGES)
def test_select_and_finish_on_cv2_keypoints(name):
    """E2: og_sift_select + og_sift_rootsift_laf driven by cv2's raw keypoints and descriptors give the reference's outputs"""
    cab = _lib()
    lib = cab.lib()
    fx = _fx(name)
    n = len(fx['kp_size'])
    kp = np.stack([fx['kp_pt'][:, 0], fx['kp_pt'][:, 1], fx['kp_size'], fx['kp_angle'], fx['kp_response']], 1).astype(np.float32)
    kp_d = torch.from_numpy(kp).to(DEV)[None]
    count = torch.tensor([n], dtype=torch.int32, device=DEV)
    work = torch.empty(cab.check_size(lib.og_sift_select_workspace_bytes(1, n), 'ws'), dtype=torch.uint8, device=DEV)
    sel, n_sel = torch.empty(1, n, dtype=torch.int32, device=DEV), torch.empty(1, dtype=torch.int32, device=DEV)
    st = cab.stream()
    cab.check(lib.og_sift_select(cab.ptr(kp_d), cab.ptr(count), 1, n, RADIUS, MAX_KP, cab.ptr(work), work.numel(), cab.ptr(sel), cab.ptr(n_sel), st),
              'og_sift_select')
    k = int(n_sel[0])
    kept = sel[0, :k].cpu().numpy().tolist()
    assert kept == greedy_select(fx['kp_pt'], fx['kp_response'], RADIUS, MAX_KP)
    raw = torch.from_numpy(fx['desc_raw'][kept].astype(np.float32)).to(DEV)
    sk = kp_d[0, kept].contiguous()
    lafs, scores, desc = torch.empty(k, 2, 3, device=DEV), torch.empty(k, device=DEV), torch.empty(k, 128, device=DEV)
    cab.check(lib.og_sift_rootsift_laf(cab.ptr(sk), cab.ptr(raw), k, 1, cab.ptr(lafs), cab.ptr(scores), cab.ptr(desc), st), 'og_sift_rootsift_laf')
    n_unique = check_selection(fx, kept, lafs.cpu().numpy(), scores.cpu().numpy(), desc.cpu().numpy())
    print(f'\n[{name}] E2: {k} selected of {n}, {n_unique} with a unique response checked to the ulp')


@pytest.mark.gpu
def test_quantisation_matches_wrapper():
    """E1: a float image gives what its uint8(255 * x) image gives (the wrapper's conversion), on every value k / 255 and between"""
    from openglue_b200 import OpenCVSIFT
    g = torch.Generator().manual_seed(3)
    x = torch.nn.functional.interpolate(torch.rand(1, 1, 30, 40, generator=g), size=(120, 160), mode='bilinear', align_corners=False)
    x = torch.where(torch.rand(x.shape, generator=g) < 0.3, torch.randint(0, 256, x.shape, generator=g).float() / 255, x)
    u8 = torch.from_numpy((255. * x[0, 0].numpy()).astype(np.uint8))[None, None]
    m = OpenCVSIFT()
    a, b = m(x.to(DEV)), m(u8.to(DEV))
    assert a[0].shape[1] > 50
    for p, q in zip(a, b):
        assert torch.equal(p, q)


@pytest.mark.gpu
@pytest.mark.parametrize('name', IMAGES)
def test_raw_keypoints_and_descriptors_against_cv2(name):
    """A1: raw keypoints against cv2's (recall, precision >= 99.9 %); A2: descriptors of matched keypoints (>= 99.8 % identical,
    no entry more than 1 apart, every cosine >= 0.999)"""
    fx = _fx(name)
    ours = _detect_all(fx)
    ref = dict(pt=fx['kp_pt'], size=fx['kp_size'], angle=fx['kp_angle'], response=fx['kp_response'], octave=fx['kp_octave'])
    keys = ('pt', 'size', 'angle', 'response', 'octave')
    r2o = match_keypoints(*[ref[k] for k in keys], *[ours[k] for k in keys])
    o2r = match_keypoints(*[ours[k] for k in keys], *[ref[k] for k in keys])
    recall, precision = (r2o >= 0).mean(), (o2r >= 0).mean()
    m = r2o >= 0
    a, b = fx['desc_raw'][m].astype(np.float64), ours['raw'][r2o[m]].astype(np.float64)
    same = (a == b).all(1)
    cos = (a * b).sum(1) / np.maximum(np.linalg.norm(a, axis=1) * np.linalg.norm(b, axis=1), 1e-30)
    dpt = np.hypot(*(ref['pt'][m] - ours['pt'][r2o[m]]).T)
    for i in np.nonzero(r2o < 0)[0][:5]:
        print(f'  cv2 keypoint without a match: pt {ref["pt"][i]}, size {ref["size"][i]}, angle {ref["angle"][i]}, response {ref["response"][i]}, '
              f'octave {ref["octave"][i] & 0xffff:#x}')
        if len(ours['pt']):
            j = int(np.argmin(np.hypot(*(ours['pt'] - ref['pt'][i]).T)))
            print(f'    nearest of ours: pt {ours["pt"][j]}, size {ours["size"][j]}, angle {ours["angle"][j]}, response {ours["response"][j]}, '
                  f'octave {ours["octave"][j] & 0xffff:#x}')
    print(f'\n[{name}] A1: cv2 {len(ref["size"])} / ours {len(ours["size"])} keypoints, recall {recall:.4f}, precision {precision:.4f}, '
          f'max |dpt| {dpt.max() if dpt.size else 0:.2e};  A2: identical {same.mean() if same.size else 1:.4f}, min cosine '
          f'{cos.min() if cos.size else 1:.6f}, max |d| {np.abs(a - b).max() if a.size else 0:.0f}')
    assert recall >= 0.999 and precision >= 0.999
    assert same.mean() >= 0.998 and (a.size == 0 or np.abs(a - b).max() <= 1) and cos.min() >= 0.999


@pytest.mark.gpu
@pytest.mark.parametrize('name', IMAGES)
def test_end_to_end_against_reference(name):
    """A3: OpenCVSIFT(2048, 9, rootsift) outputs against the reference's detect_and_compute: >= 99.9 % of its keypoints present,
    with scores, LAFs and descriptors within the A1 / A2 tolerances; the output is in descending response"""
    from openglue_b200 import OpenCVSIFT
    fx = _fx(name)
    lafs, scores, desc = OpenCVSIFT(max_keypoints=MAX_KP, nms_diameter=9., rootsift=True)(torch.from_numpy(fx['image']).to(DEV)[None, None])
    assert lafs.shape[0] == 1 and lafs.shape[2:] == (2, 3) and desc.shape[2] == 128 and lafs.is_cuda
    lafs, scores, desc = lafs[0].cpu().numpy(), scores[0].cpu().numpy(), desc[0].cpu().numpy()
    assert np.all(np.diff(scores) <= 0)
    assert len(scores) <= MAX_KP

    def frame(l):
        s = np.hypot(l[:, 0, 0], l[:, 0, 1])
        ang = np.rad2deg(np.arctan2(-l[:, 0, 1].astype(np.float64), l[:, 0, 0])) % 360
        return l[:, :, 2], s / 6, ang
    rp, rs, ra = frame(fx['ref_lafs'])
    op, os_, oa = frame(lafs)
    # A keypoint whose response several raw keypoints share (mostly one location with several orientations) is the reference's
    # arbitrary pick inside that class (numpy's argsort order): there, any orientation of the class is accepted.
    vals, counts = np.unique(fx['kp_response'], return_counts=True)
    tied = np.isin(fx['ref_scores'], vals[counts > 1])
    z = np.zeros(len(rs), np.int32)
    hit = match_keypoints(rp, rs, ra, fx['ref_scores'], z, op, os_, oa, scores, np.zeros(len(os_), np.int32))
    free = hit < 0
    free[~tied] = False
    if free.any():                                                      # tied: match without the angle, then check the class's angles
        hit_free = match_keypoints(rp[free], rs[free], np.zeros(free.sum()), fx['ref_scores'][free], z[free], op, os_, np.zeros(len(oa)), scores,
                                   np.zeros(len(os_), np.int32))
        raw_angles = {}
        for r, a in zip(fx['kp_response'], fx['kp_angle']):
            raw_angles.setdefault(float(r), []).append(float(a))
        for i, j in zip(np.nonzero(free)[0], hit_free):
            if j >= 0 and any(min(abs(oa[j] - a) % 360, 360 - abs(oa[j] - a) % 360) <= ANGLE_TOL for a in raw_angles[float(fx['ref_scores'][i])]):
                hit[i] = -2 - j                                         # present, a different member of the class
    present = (hit != -1).mean()
    m = hit >= 0
    cos = (ref_descriptors(fx)[m].astype(np.float64) * desc[hit[m]]).sum(1)       # unit vectors
    print(f'\n[{name}] A3: reference {len(rs)} / ours {len(scores)} keypoints ({tied.sum()} in tied classes), present {present:.4f} '
          f'({(hit <= -2).sum()} as another member of their class), min cosine {cos.min() if cos.size else 1:.6f}')
    assert present >= 0.999 and (cos.size == 0 or cos.min() >= 0.999)


@pytest.mark.gpu
def test_uniform_image_has_no_keypoints():
    from openglue_b200 import OpenCVSIFT
    fx = _fx('sift_uniform')
    lafs, scores, desc = OpenCVSIFT(max_keypoints=MAX_KP)(torch.from_numpy(fx['image']).to(DEV)[None, None])
    assert lafs.shape == (1, 0, 2, 3) and scores.shape == (1, 0) and desc.shape == (1, 0, 128)


@pytest.mark.gpu
def test_batch_equals_forward_and_runs_are_identical():
    """extract_batch of B images equals forward of each, bit for bit; two runs are bit-identical"""
    from openglue_b200 import OpenCVSIFT
    imgs = [_fx('sift_small')['image'], _fx('sift_warp')['image'], np.full((240, 320), 90, np.uint8)]
    batch = torch.from_numpy(np.stack(imgs)).to(DEV)[:, None].float() / 255
    m = OpenCVSIFT(max_keypoints=1000)
    outs = m.extract_batch(batch)
    again = m.extract_batch(batch)
    assert len(outs) == 3 and outs[2][0].shape[1] == 0
    for b, o in enumerate(outs):
        single = m(batch[b:b + 1])
        for p, q, r in zip(o, single, again[b]):
            assert torch.equal(p, q) and torch.equal(p, r)


@pytest.mark.gpu
def test_matcher_with_sift_front_end():
    """OpenGlueMatcher(OpenCVSIFT, SuperGlue(d = 128, 'scale_rotation')) runs end to end on an image pair"""
    import openglue_b200
    from openglue_b200 import OpenCVSIFT, SuperGlue
    from openglue_b200.synthetic import default_config, synthetic_state_dict
    cfg = default_config(descriptor_dim=128, num_stages=2, num_iters=20, side_info_size=1 + 3)
    cfg['laf_to_sideinfo_method'] = 'scale_rotation'
    sg = SuperGlue(cfg).eval()
    sg.load_state_dict(synthetic_state_dict(cfg, seed=0), strict=True)
    sg = sg.to(DEV)
    im0 = torch.from_numpy(_fx('sift_small')['image']).to(DEV)[None, None].float() / 255
    im1 = torch.from_numpy(_fx('sift_warp')['image']).to(DEV)[None, None].float() / 255
    config = {'superglue': {'laf_to_sideinfo_method': 'scale_rotation'}, 'inference': {'match_threshold': 0.0}}
    out = openglue_b200.OpenGlueMatcher(OpenCVSIFT(max_keypoints=512), sg, config)({'image0': im0, 'image1': im1})
    assert out['lafs0'].is_cuda and out['lafs0'].shape[-2:] == (2, 3)
    assert torch.isfinite(out['confidence']).all()
