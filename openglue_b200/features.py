"""Local features -> matcher inputs, and the stand-alone image-pair matcher.  Drop-ins for the reference's

    models.laf_converter.get_laf_to_sideinfo_converter(method_name)       (models/laf_converter.py:108-128)
    models.features.utils.prepare_features_output(lafs, responses, desc, laf_converter, permute_desc, log_response)   (utils.py:54-65)
    inference.OpenGlueMatcher(local_feature, matcher, match_config)       (inference.py:81-211)

The geometry of each keypoint's local affine frame (LAF) - log-scale, orientation or the full affine shape - becomes the side
information the keypoint encoder of ``SuperGlue`` takes next to the response.  ``prepare_features_output`` is ONE launch of
``og_prepare_features`` (csrc/features.cuh): keypoints and side information come out of the same pass over the LAFs, and every
column except the logarithms equals the reference's fp32 result bit for bit (the square root is the correctly rounded one, which
ATen's vectorised CPU form misses by an ulp on a few frames in a thousand).  ``OpenGlueMatcher`` runs an image pair (or
pre-extracted features) through the front-end, this step, ``SuperGlue`` with ``MatchingCore``'s match extraction, and the ordered
compaction ``og_match_compact`` to the reference's compact match list; reading the number of matches is its one host
synchronisation, where the reference's boolean indexing synchronises too.  ``ImagePairMatcher`` runs batches of image pairs
through the same chain on padded front-end outputs (``extract_padded``) with the keypoint counts on the device: no host
synchronisation at all, so the whole chain replays as one CUDA graph.

CUDA tensors only, and no autograd: the reference never differentiates these outputs.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import _cabi, _graphs
from ._cabi import ptr, stream
from .superglue import SuperGlue

__all__ = ['LAFConverter', 'get_laf_to_sideinfo_converter', 'prepare_features_output', 'compact_matches', 'pad_features',
           'padded_capacity', 'OpenGlueMatcher', 'ImagePairMatcher']

# method name -> (og_laf_method, side-information columns after the response)
_METHODS = {'none': (0, 0), 'scale': (1, 1), 'rotation': (2, 2), 'scale_rotation': (3, 3), 'affine': (4, 5)}


def _device_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not torch.is_tensor(t) or t.device.type != 'cuda':
        raise RuntimeError(f'openglue_b200: {name} must be a CUDA tensor (sm_90a); there is no CPU path')
    t = t.detach()
    return (t if t.dtype == torch.float32 else t.float()).contiguous()


def _lafs(lafs: torch.Tensor) -> torch.Tensor:
    lafs = _device_f32(lafs, 'lafs')
    if lafs.dim() != 4 or lafs.shape[2:] != (2, 3):
        raise ValueError(f'lafs must be [B, N, 2, 3], got {tuple(lafs.shape)}')
    return lafs


class LAFConverter:
    """LAF -> side information for one method (the reference's ``LAFConverter`` with its conversion functions):
    ``side_info_dim`` columns per keypoint, ``__call__(lafs [B,N,2,3]) -> [B,N,side_info_dim]``."""

    def __init__(self, method: str):
        self.method = method
        self._code, self._dim = _METHODS[method]

    @property
    def side_info_dim(self) -> int:
        return self._dim

    def __call__(self, lafs: torch.Tensor) -> torch.Tensor:
        lafs = _lafs(lafs)
        B, N = lafs.shape[:2]
        out = torch.empty(B, N, self._dim, dtype=torch.float32, device=lafs.device)
        if self._dim and B * N:
            with torch.cuda.device(lafs.device):
                _cabi.check(_cabi.lib().og_prepare_features(ptr(lafs), None, B * N, self._code, 0, None, ptr(out), stream(lafs.device)),
                            'og_prepare_features')
        return out

    def __repr__(self):
        return f'LAFConverter({self.method!r})'


def get_laf_to_sideinfo_converter(method_name: str = 'none') -> LAFConverter:
    """The converter ``superglue.laf_to_sideinfo_method`` names: 'none' | 'scale' | 'rotation' | 'scale_rotation' | 'affine'
    (case-insensitive; anything else raises the reference's ``NameError``)."""
    name = method_name.lower()
    if name not in _METHODS:
        raise NameError('Unexpected name for the method: {}'.format(method_name))
    return LAFConverter(name)


def prepare_features_output(lafs, responses, desc, laf_converter: LAFConverter, permute_desc: bool = False,
                            log_response: bool = False) -> Dict[str, torch.Tensor]:
    """-> {'keypoints' [B,N,2], 'side_info' [B,N,1+dim], 'local_descriptors'}: the reference's dict, from one kernel launch.
    side_info = [response (log(response + 0.1) when ``log_response``), laf_converter(lafs)]."""
    if not isinstance(laf_converter, LAFConverter):
        raise TypeError('laf_converter must come from openglue_b200.get_laf_to_sideinfo_converter')
    lafs = _lafs(lafs)
    B, N = lafs.shape[:2]
    responses = _device_f32(responses, 'responses')
    if tuple(responses.shape) != (B, N):
        raise ValueError(f'responses must be [B, N] = {(B, N)}, got {tuple(responses.shape)}')
    if not torch.is_tensor(desc) or desc.device.type != 'cuda':
        raise RuntimeError('openglue_b200: desc must be a CUDA tensor (sm_90a); there is no CPU path')
    dev = lafs.device
    kpts = torch.empty(B, N, 2, dtype=torch.float32, device=dev)
    side = torch.empty(B, N, 1 + laf_converter.side_info_dim, dtype=torch.float32, device=dev)
    if B * N:
        with torch.cuda.device(dev):
            _cabi.check(_cabi.lib().og_prepare_features(ptr(lafs), ptr(responses), B * N, laf_converter._code, int(bool(log_response)),
                                                        ptr(kpts), ptr(side), stream(dev)), 'og_prepare_features')
    return {'keypoints': kpts, 'side_info': side, 'local_descriptors': desc.permute(0, 2, 1) if permute_desc else desc}


def compact_matches(matches0: torch.Tensor, mscores0: torch.Tensor, lafs0: torch.Tensor, lafs1: torch.Tensor) -> Dict[str, torch.Tensor]:
    """The compact match list of ``OpenGlueMatcher.forward`` (inference.py:192-209) from ``matches0`` [B,n] (-1: no match) and
    ``matching_scores0`` [B,n]: every (b, i) with ``matches0[b, i] >= 0``, pair-major then by i, as the reference's boolean
    indexing orders them.  One kernel launch, then one read of the count."""
    dev = matches0.device
    if dev.type != 'cuda':
        raise RuntimeError('openglue_b200: matches0 must be a CUDA tensor (sm_90a); there is no CPU path')
    matches0 = matches0.detach().long().contiguous()
    mscores0 = _device_f32(mscores0, 'matching_scores0')
    lafs0, lafs1 = _lafs(lafs0), _lafs(lafs1)
    B, n = matches0.shape
    m = lafs1.shape[1]
    if tuple(mscores0.shape) != (B, n) or lafs0.shape[:2] != (B, n) or lafs1.shape[0] != B:
        raise ValueError('inconsistent batch / keypoint counts')
    cap = B * n
    i64 = dict(dtype=torch.int64, device=dev)
    f32 = dict(dtype=torch.float32, device=dev)
    pair, ij, conf = torch.empty(cap, **i64), torch.empty(cap, 2, **i64), torch.empty(cap, **f32)
    l0, l1 = torch.empty(cap, 2, 3, **f32), torch.empty(cap, 2, 3, **f32)
    k0, k1 = torch.empty(cap, 2, **f32), torch.empty(cap, 2, **f32)
    total = torch.empty(1, **i64)
    if cap and m:
        with torch.cuda.device(dev):
            _cabi.check(_cabi.lib().og_match_compact(ptr(matches0), ptr(mscores0), ptr(lafs0), ptr(lafs1), B, n, m, ptr(pair), ptr(ij), ptr(conf),
                                                     ptr(l0), ptr(l1), ptr(k0), ptr(k1), ptr(total), stream(dev)), 'og_match_compact')
        nc = int(total.item())                  # the one host synchronisation (the reference's boolean indexing)
    else:
        nc = 0
    return {'original_matching_idxs': ij[:nc], 'batch_indexes': pair[:nc], 'confidence': conf[:nc],
            'lafs0': l0[:nc][None], 'lafs1': l1[:nc][None], 'keypoints0': k0[:nc], 'keypoints1': k1[:nc]}


def pad_features(features: Sequence[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]], capacity: Optional[int] = None
                 ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """One batch from images with their own keypoint counts, without dropping any: the lossless counterpart of the reference's
    ``min_stack`` (models/features/utils.py:28-52), which trims every image to the smallest count.  ``features``: one
    ``(lafs [1,N_b,2,3] | [N_b,2,3], responses [1,N_b] | [N_b], descriptors [1,N_b,D] | [N_b,D])`` per image, as
    ``OpenCVSIFT.extract_batch`` returns them.  -> zero-padded ``lafs`` [B,N,2,3], ``responses`` [B,N], ``descriptors`` [B,N,D]
    with N = ``capacity`` (default: the largest N_b), and ``num_keypoints`` [B] (int64, on the host): the matcher's
    ``num_keypoints0`` / ``num_keypoints1``."""
    feats: List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = []
    for lafs, resp, desc in features:
        if lafs.dim() == 4:
            lafs, resp, desc = lafs[0], resp[0], desc[0]
        if lafs.dim() != 3 or lafs.shape[1:] != (2, 3) or resp.shape != lafs.shape[:1] or desc.dim() != 2 or desc.shape[0] != lafs.shape[0]:
            raise ValueError('each feature set must be (lafs [N,2,3], responses [N], descriptors [N,D]), optionally with a leading 1')
        feats.append((lafs, resp, desc))
    if not feats:
        raise ValueError('pad_features needs at least one feature set')
    counts = [f[0].shape[0] for f in feats]
    D = feats[0][2].shape[1]
    if any(f[2].shape[1] != D for f in feats):
        raise ValueError('descriptors of different widths')
    N = max(counts) if capacity is None else int(capacity)
    if N < max(counts):
        raise ValueError(f'capacity {N} is below the largest keypoint count {max(counts)}')
    dev = feats[0][0].device
    B = len(feats)
    lafs = torch.zeros(B, N, 2, 3, dtype=torch.float32, device=dev)
    resp = torch.zeros(B, N, dtype=torch.float32, device=dev)
    desc = torch.zeros(B, N, D, dtype=torch.float32, device=dev)
    for b, (l, r, d) in enumerate(feats):
        k = l.shape[0]
        lafs[b, :k], resp[b, :k], desc[b, :k] = l, r, d
    return lafs, resp, desc, torch.tensor(counts, dtype=torch.int64)


def padded_capacity(max_keypoints: int, capacity: Optional[int] = None) -> int:
    """K, the rows per image of a front-end's ``extract_padded``: ``capacity``, by default ``max_keypoints``."""
    if capacity is None:
        if int(max_keypoints) == -1:
            raise ValueError('extract_padded needs a capacity when max_keypoints is -1 (every keypoint kept)')
        capacity = max_keypoints
    if int(capacity) < 1:
        raise ValueError(f'capacity must be at least 1, got {capacity}')
    return int(capacity)


class OpenGlueMatcher(nn.Module):
    """Drop-in for the reference's ``inference.OpenGlueMatcher`` (inference.py:81-211): correspondences between two images from
    local features followed by SuperGlue.

    ``local_feature``: the front-end, ``image [B,1,H,W] -> (lafs, responses, descriptors)`` (e.g. ``openglue_b200.SuperPointNet``);
    ``matcher``: an ``openglue_b200.SuperGlue``; ``match_config``: the reference's config with ``superglue.laf_to_sideinfo_method``,
    optional ``superglue.log_transform_response`` and ``inference.match_threshold``.

    ``forward(data)`` takes ``image0`` / ``image1`` [B,1,H,W] and, optionally, pre-extracted ``lafs{0,1}``, ``descriptors{0,1}``,
    ``responses{0,1}`` (the images then only give their sizes) - padded to a capacity with ``num_keypoints0`` /
    ``num_keypoints1`` (``pad_features``), they are matched as one batch with each pair's own counts; it sets
    ``data['image{0,1}_size']`` as the reference does and
    returns ``original_matching_idxs`` [NC,2], ``batch_indexes`` [NC], ``confidence`` [NC], ``lafs0`` / ``lafs1`` [1,NC,2,3],
    ``keypoints0`` / ``keypoints1`` [NC,2]."""

    def __init__(self, local_feature: nn.Module, matcher: SuperGlue, match_config: Dict = {}) -> None:
        super().__init__()
        if not isinstance(matcher, SuperGlue):
            raise TypeError('openglue_b200.OpenGlueMatcher takes an openglue_b200.SuperGlue as its matcher')
        self.local_feature = local_feature
        self.laf_converter = get_laf_to_sideinfo_converter(match_config['superglue']['laf_to_sideinfo_method'])
        self.matcher = matcher
        self.match_config = match_config
        self.eval()

    def extract_features(self, image: torch.Tensor, mask=None) -> Dict[str, torch.Tensor]:
        lafs, resps, descs = self.local_feature(image)
        return {'lafs': lafs, 'responses': resps, 'descriptors': descs}

    @torch.no_grad()
    def forward(self, data: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        feats = []
        for i in (0, 1):
            if f'lafs{i}' not in data or f'descriptors{i}' not in data:
                f = self.extract_features(data[f'image{i}'])
                feats.append((f['lafs'], f['descriptors'], f['responses']))
            else:
                feats.append((data[f'lafs{i}'], data[f'descriptors{i}'], data[f'responses{i}']))
        (lafs0, descs0, resps0), (lafs1, descs1, resps1) = feats
        _, _, h0, w0 = data['image0'].shape
        _, _, h1, w1 = data['image1'].shape
        data['image0_size'], data['image1_size'] = [w0, h0], [w1, h1]
        log_response = self.match_config['superglue'].get('log_transform_response', False)
        f0 = prepare_features_output(lafs0, resps0, descs0, self.laf_converter, log_response=log_response)
        f1 = prepare_features_output(lafs1, resps1, descs1, self.laf_converter, log_response=log_response)
        inputs = {**data, **{k + '0': v for k, v in f0.items()}, **{k + '1': v for k, v in f1.items()}}
        # MatchingCore's path: SuperGlue + mutual-argmax extraction in one call
        res = self.matcher.run(inputs, want_matches=True, want_context=False,
                               match_threshold=float(self.match_config['inference']['match_threshold']))
        return compact_matches(res['matches0'], res['matching_scores0'], lafs0, lafs1)


def weights_key(module: nn.Module) -> tuple:
    """Changes whenever a parameter or buffer of ``module`` is written or replaced: the key of its packed weights, and of a
    captured graph that has a front-end's packed weights baked in"""
    return tuple((t._version, t.data_ptr()) for t in list(module.parameters()) + list(module.buffers()))


def _frontend_storage(module: nn.Module) -> tuple:
    """The cached workspaces and packed weights of the front-end and of every module inside it (``DoGOpenCVAffNetHardNet``
    detects through its own ``OpenCVSIFT``): a captured graph reads them, so it holds them even if a module drops them later"""
    mods = list(module.modules())
    return tuple(v for m in mods for v in getattr(m, '_ws', {}).values()), tuple(getattr(m, '_packed', None) for m in mods)


def _check_image_pair(image0, image1) -> None:
    for i, img in ((0, image0), (1, image1)):
        if not torch.is_tensor(img) or img.dim() != 4 or img.shape[1] != 1:
            raise ValueError(f'image{i} must be [B, 1, H, W], got {tuple(img.shape) if torch.is_tensor(img) else type(img)}')
    if image0.shape[0] != image1.shape[0] or image0.shape[0] < 1:
        raise ValueError(f'image0 and image1 must hold the same number of images, got {image0.shape[0]} and {image1.shape[0]}')


def _image_pair_inputs(local_feature: nn.Module, laf_converter: LAFConverter, log_response: bool, image0: torch.Tensor,
                       image1: torch.Tensor, K: int) -> Tuple[Dict[str, torch.Tensor], Dict[str, torch.Tensor]]:
    """The image-pair front-end: ``extract_padded`` on both images (K rows each), ``prepare_features_output`` and the per-pair
    image sizes -> (the padded matcher inputs, {``lafs{i}``, ``keypoints{i}``, ``num_keypoints{i}``, ``overflow{i}``})."""
    dev = image0.device
    B = image0.shape[0]
    data, feats = {}, {}
    for i, img in ((0, image0), (1, image1)):
        lafs, resp, desc, num, over = local_feature.extract_padded(img, K)
        f = prepare_features_output(lafs, resp, desc, laf_converter, log_response=log_response)
        size = torch.empty(B, 2, dtype=torch.float32, device=dev)        # (W, H) per pair, filled on the device
        size[:, 0] = float(img.shape[3])
        size[:, 1] = float(img.shape[2])
        data.update({f'keypoints{i}': f['keypoints'], f'side_info{i}': f['side_info'], f'local_descriptors{i}': desc,
                     f'num_keypoints{i}': num, f'image{i}_size': size})
        feats.update({f'lafs{i}': lafs, f'keypoints{i}': f['keypoints'], f'num_keypoints{i}': num, f'overflow{i}': over})
    return data, feats


class ImagePairMatcher(nn.Module):
    """Batches of image pairs to matches with no host synchronisation, replayed as one CUDA graph by default.

    ``local_feature``: an ``OpenCVSIFT``, ``SIFT``, ``GFTTAffNetHardNet``, ``DoGOpenCVAffNetHardNet`` or ``SuperPointNet`` /
    ``SuperPointNetBn``; ``matcher``: an ``openglue_b200.SuperGlue``;
    ``match_config``: ``OpenGlueMatcher``'s (``superglue.laf_to_sideinfo_method``, optional ``superglue.log_transform_response``,
    ``inference.match_threshold``).  ``capacity``: the keypoint rows K per image (default: the front-end's ``max_keypoints``).

    ``forward(image0 [B,1,H0,W0], image1 [B,1,H1,W1])`` runs ``extract_padded`` on both images, ``prepare_features_output``,
    ``SuperGlue.run`` on the padded batch with the device counts, and the match extraction.  Each pair's matches are those of
    the pair matched alone.  It returns device tensors: ``matches0`` / ``matching_scores0`` [B,K], ``matches1`` /
    ``matching_scores1`` [B,K] (-1 / 0 past the counts, and everywhere in a pair with no keypoint in either image),
    ``lafs0`` / ``lafs1`` [B,K,2,3], ``keypoints0`` / ``keypoints1`` [B,K,2], ``num_keypoints0`` / ``num_keypoints1`` [B] int32 and
    ``overflow0`` / ``overflow1`` [B] int32 (the front-ends' flags: an image cut to the capacity).  ``compact_matches(matches0,
    matching_scores0, lafs0, lafs1)`` gives ``OpenGlueMatcher``'s list.

    ``use_cuda_graph=True`` captures the chain once per (B, H0, W0, H1, W1, K, image dtype, device, precision, match threshold)
    after one eager warm-up run, and replays it with the images copied into static buffers.  A graph is captured again when the
    matcher's buffers are reallocated or a weight of the matcher or the front-end changes; at most ``max_graphs`` are kept.
    The first call packs the weights and copies them to the device; every later call runs without a host synchronisation."""

    _OUT_KEYS = ('matches0', 'matching_scores0', 'matches1', 'matching_scores1', 'lafs0', 'lafs1', 'keypoints0', 'keypoints1',
                 'num_keypoints0', 'num_keypoints1', 'overflow0', 'overflow1')

    def __init__(self, local_feature: nn.Module, matcher: SuperGlue, match_config: Dict, use_cuda_graph: bool = True,
                 capacity: Optional[int] = None) -> None:
        super().__init__()
        if not isinstance(matcher, SuperGlue):
            raise TypeError('openglue_b200.ImagePairMatcher takes an openglue_b200.SuperGlue as its matcher')
        if not callable(getattr(local_feature, 'extract_padded', None)):
            raise TypeError('openglue_b200.ImagePairMatcher takes a front-end with extract_padded (OpenCVSIFT, SIFT, GFTTAffNetHardNet, '
                            'DoGOpenCVAffNetHardNet, SuperPointNet[Bn])')
        self.local_feature = local_feature
        self.matcher = matcher
        self.laf_converter = get_laf_to_sideinfo_converter(match_config['superglue']['laf_to_sideinfo_method'])
        self.log_response = bool(match_config['superglue'].get('log_transform_response', False))
        self.match_threshold = float(match_config['inference']['match_threshold'])
        self.capacity = capacity
        self.use_cuda_graph = use_cuda_graph
        self._graphs: Dict[tuple, _graphs.Entry] = {}
        self.max_graphs = 4
        self.eval()

    def _chain(self, image0: torch.Tensor, image1: torch.Tensor, K: int) -> Dict[str, torch.Tensor]:
        dev = image0.device
        B = image0.shape[0]
        data, out = _image_pair_inputs(self.local_feature, self.laf_converter, self.log_response, image0, image1, K)
        res = self.matcher.run(data, want_matches=True, want_context=False, match_threshold=self.match_threshold)
        m0, s0, m1, s1 = res['matches0'], res['matching_scores0'], res['matches1'], res['matching_scores1']
        with torch.cuda.device(dev):
            _cabi.check(_cabi.lib().og_mask_empty_pairs(ptr(out['num_keypoints0']), ptr(out['num_keypoints1']), B, K, K, ptr(m0), ptr(s0),
                                                        ptr(m1), ptr(s1), stream(dev)), 'og_mask_empty_pairs')
        out.update(matches0=m0, matching_scores0=s0, matches1=m1, matching_scores1=s1)
        return out

    def _versions(self) -> tuple:
        return (getattr(self.matcher, '_alloc_gen', 0), self.matcher._weights_version(), weights_key(self.local_feature))

    def _run_graph(self, image0: torch.Tensor, image1: torch.Tensor, K: int) -> Dict[str, torch.Tensor]:
        """Replay (capturing on first use) the CUDA graph for these shapes; the images are copied into its static buffers."""
        dev = image0.device
        key = (tuple(image0.shape), tuple(image1.shape), image0.dtype, image1.dtype, K, str(dev), self.matcher._precision(),
               self.match_threshold)
        return _graphs.run(self._graphs, self.max_graphs, key, self._versions, {'image0': image0, 'image1': image1},
                           lambda s: self._chain(s['image0'], s['image1'], K), dev, f32=False,
                           hold=lambda: _frontend_storage(self.local_feature))

    @torch.no_grad()
    def forward(self, image0: torch.Tensor, image1: torch.Tensor, borrow: bool = False) -> Dict[str, torch.Tensor]:
        """``borrow=True`` (CUDA-graph mode): return the graph's own output buffers instead of copies; the next call on this
        matcher overwrites them (use it when the results are consumed on the same stream right away)."""
        _check_image_pair(image0, image1)
        K = padded_capacity(self.local_feature.max_keypoints, self.capacity)
        if image0.device.type != 'cuda' or image1.device != image0.device:
            raise RuntimeError('openglue_b200.ImagePairMatcher needs both images on one CUDA device (sm_90a); there is no CPU path')
        with torch.cuda.device(image0.device):
            if not self.use_cuda_graph:
                return self._chain(image0, image1, K)
            out = self._run_graph(image0, image1, K)
        return out if borrow else {k: v.clone() for k, v in out.items()}
