"""openglue_b200: the OpenGlue matching core (SuperGlue-style GNN + Sinkhorn) on the H100 (sm_90a).

Public surface mirrors the reference for this one path:
    SuperGlue(config).forward(data)  -> {'context_descriptors0', 'context_descriptors1', 'scores'}
    MatchingCore(superglue)(data)    -> {'matches0', 'matching_scores0', 'matches1', 'matching_scores1'}
and, for the step right before it in the reference's training / validation step:
    generate_gt_matches(data, features0, features1, positive_threshold, negative_threshold) -> (data, y_true)
and the steps either side of those:
    collate_features(batch, target_num_keypoints, random)     (the cached-feature DataLoader's collate_fn, on the GPU)
    criterion(y_true, y_pred, margin=None) -> {'loss', 'metric_loss'}
    matching_log_probs(S, dustbin_score, num_iters, reg)      (differentiable Sinkhorn: forward + backward kernels)
    SuperGlue(config).train()(data)                           (training mode: batch-statistics BatchNorm, explicit backward pass)
    ClippedAdam.from_config(superglue, config['train'])       (clip_grad_norm_ -> Adam -> StepLR, one device call, graph-capturable)
    SuperPointNet(max_keypoints, ...)(image) -> (lafs, scores, descriptors)   (the detector / descriptor front-end; SuperPointNetBn: its BatchNorm variant)
    OpenCVSIFT(max_keypoints, nms_diameter, rootsift)(image) -> (lafs, scores, descriptors)   (OPENCV_SIFT: cv2's SIFT + radius NMS + RootSIFT)
    SIFT(max_keypoints=8000, nms_diameter=9, upright, rootsift)(images) -> (lafs, responses, descriptors)   (SIFT: kornia's DoG detector + run_nms + RootSIFT)
    GFTTAffNetHardNet(max_keypoints=8000, nms_diameter=9, upright, weights=...)(images) -> (lafs, responses, descriptors)   (GFTT + AffNet + run_nms + HardNet)
    DoGOpenCVAffNetHardNet(max_keypoints=-1, nms_diameter=9., weights=...)(image) -> (lafs, scores, descriptors)   (OPENCVDoGAffNetHardNet: cv2's SIFT detector + AffNet + OriNet + HardNet)
    prepare_features_output(lafs, responses, desc, get_laf_to_sideinfo_converter(method), ...)   (front-end output -> SuperGlue input)
    OpenGlueMatcher(local_feature, superglue, match_config)(data) -> compact match list   (stand-alone image-pair inference)
    ImagePairMatcher(local_feature, superglue, match_config)(image0, image1) -> padded matches   (batches of pairs, one CUDA graph)
    synthesize_homography_pairs(images_u8, offset, warp_offset, generator)   (the homography-pretraining dataset's pairs, batched)
    ImagePairTrainStep(local_feature, superglue, config, optimizer)(batch)   (training_step from images, one CUDA graph)
"""
from .gt_matches import generate_gt_matches  # noqa: F401
from .homography import synthesize_homography_pairs  # noqa: F401
from .feature_cache import FeatureStore, collate_features  # noqa: F401
from .features import ImagePairMatcher, OpenGlueMatcher, get_laf_to_sideinfo_converter, prepare_features_output  # noqa: F401
from .losses import criterion  # noqa: F401
from .optim import ClippedAdam  # noqa: F401
from .sinkhorn import matching_log_probs  # noqa: F401
from .superglue import MatchingCore, PendingMatches, SuperGlue  # noqa: F401
from .sift import OpenCVSIFT, sift_create_torch  # noqa: F401
from .kornia_sift import SIFT  # noqa: F401
from .gftt_hardnet import GFTTAffNetHardNet  # noqa: F401
from .dog_affnet_hardnet import DoGOpenCVAffNetHardNet  # noqa: F401
from .superpoint import SuperPointNet, SuperPointNetBn  # noqa: F401
from .training import ImagePairTrainStep  # noqa: F401

__version__ = '0.1.0'
