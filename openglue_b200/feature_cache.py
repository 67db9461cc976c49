"""Cached local features -> batches for the matching core, on the GPU (SURVEY.md section 8, row f3).

What the reference does on the host for the cached-features pipeline (``use_cached_features: True``):

* ``extract_features.py:251-262`` writes, per image, four deepdish HDF5 files ``<name>_{lafs,scores,descriptors,size}.h5``;
* ``MegaDepthPairsDatasetFeatures.__getitem__`` (data/megadepth_dataset.py:203-282) loads them for both images of a pair,
  crops keypoints to the target size and returns ``lafs{0,1} [K,2,3]``, ``scores{0,1} [K]``, ``descriptors{0,1} [K,D]`` (variable
  K), the transformation (intrinsics, pose, depth images) and the image sizes;
* ``MegaDepthPairsDataModuleFeatures.stack_keypoints_batch`` (data/megadepth_datamodule.py:105-168) is the DataLoader's
  ``collate_fn``: top-``num_keypoints`` by confidence (validation) or a random subset (training), zero padding, per-keypoint depth.

Here: ``FeatureStore`` reads a features directory into PINNED host tensors once (the reference's ``.h5`` quadruples when ``deepdish``
or ``h5py`` is importable, or the ``.npz`` files ``convert_h5_to_npz`` writes from them - this image has neither HDF5 library, so the
tests use the ``.npz`` form), and ``collate_features`` is the drop-in for ``stack_keypoints_batch``: same arguments, same returned
dict, but the selection / gather / depth lookup run in ``og_collate_fwd`` on the device and the result is already device-resident for
``generate_gt_matches`` -> ``SuperGlue``.  One pinned staging copy per batch; there is no CPU fallback for the collation itself.
"""
from __future__ import annotations

import os
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _cabi
from ._cabi import ptr, stream

__all__ = ['FeatureStore', 'collate_features', 'convert_h5_to_npz', 'save_features_npz']

_FIELDS = ('lafs', 'scores', 'descriptors', 'size')


def _load_h5(path: str):
    """One array the way extract_features.py:251-262 saved it (deepdish.io.save of a numpy array)."""
    try:
        import deepdish as dd                                   # the reference's own reader
        return np.asarray(dd.io.load(path))
    except ImportError:
        pass
    try:
        import h5py                                             # deepdish stores a bare ndarray as the dataset '/data'
    except ImportError as e:
        raise ImportError('reading the reference\'s .h5 feature files needs deepdish or h5py (neither is installed here); '
                          'convert them once with convert_h5_to_npz on a machine that has one of them') from e
    with h5py.File(path, 'r') as f:
        return np.asarray(f['data'])


def save_features_npz(directory: str, base_name: str, lafs, scores, descriptors, size) -> str:
    """The four arrays of extract_features.save_outputs (extract_features.py:251-262) in ONE uncompressed .npz."""
    os.makedirs(directory, exist_ok=True)
    path = os.path.join(directory, base_name + '.npz')
    np.savez(path, lafs=np.asarray(lafs, np.float32), scores=np.asarray(scores, np.float32),
             descriptors=np.asarray(descriptors, np.float32), size=np.asarray(size, np.int64))
    return path


def convert_h5_to_npz(features_dir: str, out_dir: Optional[str] = None) -> int:
    """<name>_{lafs,scores,descriptors,size}.h5 (reference format) -> <name>.npz, for every image of a scene directory."""
    out_dir = out_dir or features_dir
    names = sorted({f[:-len('_lafs.h5')] for f in os.listdir(features_dir) if f.endswith('_lafs.h5')})
    for n in names:
        arrs = [_load_h5(os.path.join(features_dir, f'{n}_{k}.h5')) for k in _FIELDS]
        save_features_npz(out_dir, n, *arrs)
    return len(names)


class FeatureStore:
    """Features of one scene directory, resident in pinned host memory.  ``store[name]`` -> dict of torch tensors
    (``lafs [K,2,3]``, ``scores [K]``, ``descriptors [K,D]``, ``size`` (w, h)) - what the reference re-reads from disk for every pair."""

    def __init__(self, features_dir: str, pin: bool = True):
        self.dir = features_dir
        self.pin = pin and torch.cuda.is_available()
        self._items: Dict[str, Dict[str, Any]] = {}

    def names(self) -> List[str]:
        found = {f[:-4] for f in os.listdir(self.dir) if f.endswith('.npz')}
        found |= {f[:-len('_lafs.h5')] for f in os.listdir(self.dir) if f.endswith('_lafs.h5')}
        return sorted(found)

    def __getitem__(self, name: str) -> Dict[str, Any]:
        it = self._items.get(name)
        if it is None:
            npz = os.path.join(self.dir, name + '.npz')
            if os.path.exists(npz):
                with np.load(npz) as z:
                    arrs = {k: z[k] for k in _FIELDS}
            else:
                arrs = {k: _load_h5(os.path.join(self.dir, f'{name}_{k}.h5')) for k in _FIELDS}
            it = {'lafs': torch.from_numpy(np.ascontiguousarray(arrs['lafs'], np.float32)),
                  'scores': torch.from_numpy(np.ascontiguousarray(arrs['scores'], np.float32)),
                  'descriptors': torch.from_numpy(np.ascontiguousarray(arrs['descriptors'], np.float32)),
                  'size': tuple(int(x) for x in arrs['size'])}
            if self.pin:
                it = {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in it.items()}
            self._items[name] = it
        return it


def collate_features(batch: Sequence[Dict[str, Any]], target_num_keypoints: int, random: bool = False,
                     device: Optional[torch.device] = None, generator: Optional[torch.Generator] = None) -> Dict[str, Any]:
    """Drop-in for ``MegaDepthPairsDataModuleFeatures.stack_keypoints_batch(batch, target_num_keypoints, random)``
    (reference data/megadepth_datamodule.py:105-168): same input (a list of the cached-feature dataset's items), same returned
    dict (``lafs{0,1}``, ``scores{0,1}``, ``descriptors{0,1}``, ``image{0,1}_size``, ``transformation`` with per-keypoint depths),
    tensors on ``device``.  ``random=True`` draws ``torch.randperm`` on the host exactly as the reference does (same generator
    state -> same selection)."""
    dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    if dev.type != 'cuda':
        raise RuntimeError('openglue_b200.collate_features runs on a CUDA device (sm_90a); there is no CPU path')
    B, K = len(batch), int(target_num_keypoints)
    D = batch[0]['descriptors0'].size(1)
    counts, select = [], None
    for item in batch:
        for img in (0, 1):
            counts.append(int(item[f'lafs{img}'].size(0)))
    offsets = np.zeros(2 * B + 1, np.int32)
    offsets[1:] = np.cumsum(counts)
    total = int(offsets[-1])
    # one pinned staging buffer per field, one H2D copy each
    stage = {'lafs': torch.empty(max(total, 1), 2, 3).pin_memory(), 'scores': torch.empty(max(total, 1)).pin_memory(),
             'desc': torch.empty(max(total, 1), D).pin_memory()}
    if random:
        select = torch.zeros(2 * B, K, dtype=torch.int32)
    i = 0
    for item in batch:
        for img in (0, 1):
            o, c = int(offsets[i]), counts[i]
            stage['lafs'][o:o + c] = item[f'lafs{img}']
            stage['scores'][o:o + c] = item[f'scores{img}']
            stage['desc'][o:o + c] = item[f'descriptors{img}']
            if random and c > K:                                 # reference :147-148
                perm = torch.randperm(c, generator=generator) if generator is not None else torch.randperm(c)
                select[i] = perm[:K].to(torch.int32)
            i += 1
    tf = batch[0]['transformation']
    depth = [None, None]
    if 'depth0' in tf:
        depth = [torch.stack([x['transformation'][f'depth{img}'] for x in batch]).float().contiguous() for img in (0, 1)]
    lib = _cabi.lib()
    with torch.cuda.device(dev):
        d_lafs, d_scores, d_desc = (stage[k].to(dev, non_blocking=True) for k in ('lafs', 'scores', 'desc'))
        d_off = torch.from_numpy(offsets).to(dev, non_blocking=True)
        d_sel = select.to(dev, non_blocking=True) if select is not None else None
        d_depth = [d.to(dev, non_blocking=True) if d is not None else None for d in depth]
        out = {f'lafs{i}': torch.empty(B, K, 2, 3, device=dev) for i in (0, 1)}
        out.update({f'scores{i}': torch.empty(B, K, device=dev) for i in (0, 1)})
        out.update({f'descriptors{i}': torch.empty(B, K, D, device=dev) for i in (0, 1)})
        kdepth = [torch.empty(B, K, device=dev) if d is not None else None for d in d_depth]
        rc = lib.og_collate_fwd(ptr(d_lafs), ptr(d_scores), ptr(d_desc), ptr(d_off), ptr(d_sel), max(counts),
                                ptr(d_depth[0]), 0 if d_depth[0] is None else d_depth[0].shape[-2], 0 if d_depth[0] is None else d_depth[0].shape[-1],
                                ptr(d_depth[1]), 0 if d_depth[1] is None else d_depth[1].shape[-2], 0 if d_depth[1] is None else d_depth[1].shape[-1],
                                B, K, D, ptr(out['lafs0']), ptr(out['lafs1']), ptr(out['scores0']), ptr(out['scores1']),
                                ptr(out['descriptors0']), ptr(out['descriptors1']), ptr(kdepth[0]), ptr(kdepth[1]),
                                stream(dev))
        _cabi.check(rc, 'og_collate_fwd')
        for t in (d_lafs, d_scores, d_desc, d_off, d_sel, *d_depth):
            if t is not None:
                t.record_stream(torch.cuda.current_stream(dev))
    out['image0_size'] = batch[0]['image0_size']
    out['image1_size'] = batch[0]['image1_size']
    transformation = {'type': ['3d_reprojection'] if 'K0' in tf else [tf.get('type', 'perspective')]}
    for k in ('K0', 'K1', 'R', 'T', 'H'):
        if k in tf:
            transformation[k] = torch.stack([x['transformation'][k] for x in batch]).to(dev)
    if kdepth[0] is not None:
        transformation['depth0'], transformation['depth1'] = kdepth
    out['transformation'] = transformation
    return out
