"""Time one homography-pretraining step from images (pretrain_homography.py's setting: 1472 x 1232 uint8 RGB, offset 256, so 960 x
720 pairs; B = 4), three ways, with SuperPoint (max_keypoints 1024, d = 256) and SIFT (max_keypoints 2048, d = 128):
  hand      the chain wired by hand, eagerly: synthesize_homography_pairs -> extract_padded -> prepare_features_output ->
            generate_gt_matches -> TrainStep -> criterion_with_grad -> backward -> ClippedAdam.step;
  eager     ImagePairTrainStep.pretrain with use_cuda_graph=False: the same chain behind the device-side skip;
  graph     ImagePairTrainStep.pretrain replayed as one CUDA graph (borrowed outputs).
SuperGlue: 9 stages, 4 heads, 20 Sinkhorn iterations, tf32x3, synthetic weights; ClippedAdam from the reference's train config.
Each form trains its own copy of the model.  CUDA events around `iters` steps, medians of `rounds` rounds, the forms alternating in
one process.  Prints one JSON object with the GPU's name and power limit beside the numbers (ms per step).

    python tools/image_train_timing.py [--batch 4] [--iters 5] [--rounds 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import statistics

import torch

from gpu_timing import card, rounds_ms

CONFIG = {'superglue': {'laf_to_sideinfo_method': 'none', 'log_transform_response': False},
          'train': {'gt_positive_threshold': 2, 'gt_negative_threshold': 7, 'margin': None, 'nll_weight': 1.0, 'metric_weight': 0.0,
                    'augmentations': {'name': 'none'}, 'lr': 1e-4, 'grad_clip': 10.0, 'scheduler_gamma': 0.999994}}


def _rgb(B, dev):
    g = torch.Generator(device=dev).manual_seed(B)
    low = torch.rand(B, 3, 1232 // 12, 1472 // 12, generator=g, device=dev)
    img = torch.nn.functional.interpolate(low, size=(1232, 1472), mode='bicubic', align_corners=False).clamp(0, 1) * 255
    return img.to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('image_train_timing needs a CUDA device')
    from gen_golden_superpoint import synthetic_superpoint_state_dict
    from openglue_b200 import ClippedAdam, ImagePairTrainStep, OpenCVSIFT, SuperGlue, SuperPointNet, synthesize_homography_pairs
    from openglue_b200.features import get_laf_to_sideinfo_converter, prepare_features_output
    from openglue_b200.gt_matches import generate_gt_matches
    from openglue_b200.losses import criterion_with_grad
    from openglue_b200.synthetic import default_config, synthetic_state_dict
    from openglue_b200.training import TrainStep
    dev = torch.device('cuda:0')
    B, offset = args.batch, 256
    imgs = _rgb(B, dev)
    conv = get_laf_to_sideinfo_converter('none')
    result = {'card': card(), 'iters': args.iters, 'rounds': args.rounds, 'batch': B, 'image': [1232, 1472], 'offset': offset, 'results': []}
    for name in ('superpoint', 'sift'):
        if name == 'sift':
            fe, D, K = OpenCVSIFT(max_keypoints=2048), 128, 2048
        else:
            fe, D, K = SuperPointNet(max_keypoints=1024, keypoint_threshold=0.005), 256, 1024
            fe.load_state_dict(synthetic_superpoint_state_dict(7), strict=True)
            fe = fe.to(dev).eval()
        cfg = default_config(descriptor_dim=D, num_stages=9, num_heads=4, num_iters=20)
        cfg['precision'] = 'tf32x3'
        models = []
        for _ in range(3):
            m = SuperGlue(cfg)
            m.load_state_dict(synthetic_state_dict(cfg, seed=1), strict=True)
            m = m.to(dev).train()
            models.append((m, ClippedAdam.from_config(m, CONFIG['train'])))
        eager = ImagePairTrainStep(fe, models[1][0], CONFIG, optimizer=models[1][1], use_cuda_graph=False)
        graph = ImagePairTrainStep(fe, models[2][0], CONFIG, optimizer=models[2][1])
        m_h, o_h = models[0]

        def hand():
            raw = synthesize_homography_pairs(imgs, offset)
            feats = []
            for i in (0, 1):
                lafs, resp, desc, n, _ = fe.extract_padded(raw[f'image{i}'], K)
                feats.append(prepare_features_output(lafs, resp, desc, conv))
                raw[f'num_keypoints{i}'] = n
            data, y = generate_gt_matches(raw, feats[0], feats[1], 2, 7)
            st = TrainStep(m_h, data)
            scores, _, _ = st.forward()
            _, ds = criterion_with_grad(y, {'scores': scores})
            g = st.backward(ds)
            for k, p in m_h.named_parameters():
                p.grad = g[k].reshape(p.shape)
            o_h.step()

        forms = {'hand': hand, 'eager': lambda: eager.pretrain(imgs, offset), 'graph': lambda: graph.pretrain(imgs, offset, borrow=True)}
        for fn in forms.values():                                              # warm-up (and the one capture)
            fn()
        out = eager.pretrain(imgs, offset)
        row = {'features': name, 'keypoints_capacity': K, 'keypoints0': out['num_keypoints0'].tolist(),
               'keypoints1': out['num_keypoints1'].tolist(), 'overflow': int(out['overflow0'].sum() + out['overflow1'].sum()),
               'skipped': int(out['skipped'])}
        for k, v in rounds_ms(forms, args.iters, args.rounds).items():
            row[f'{k}_ms'] = round(statistics.median(v), 3)
            row[f'{k}_rounds_ms'] = [round(x, 3) for x in v]
        result['results'].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
