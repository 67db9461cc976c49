// Batch collation of cached local features (SURVEY.md section 8, row f3): the GPU form of
// MegaDepthPairsDataModuleFeatures.stack_keypoints_batch (reference data/megadepth_datamodule.py:105-168), the step that
// turns the per-image outputs of the cached-feature dataset (data/megadepth_dataset.py:203-282; variable keypoint counts)
// into the fixed-size batch the matching core consumes:
//   * more keypoints than the target  -> the `target` most confident ones, in descending score order (torch.topk; validation)
//                                        or a caller-supplied random selection (torch.randperm on the host; training),
//   * fewer                           -> all of them in their original order, zero padding behind (virtual keypoints:
//                                        depth 0 marks them as ignored for the ground-truth generation),
//   * the depth of every kept keypoint is looked up in the pair's depth image at (int(y), int(x)).
// One CTA per (pair, image).  Selection = bitonic sort of (score, index) in shared memory (ties: lower index first); the
// rest is a gather: HBM-bound, ~(6 + 1 + D) floats in and out per kept keypoint.  Index work: bit-exact.
#pragma once
#include "common.cuh"

namespace og {

struct CollateArgs {
  const float* lafs;            // [total, 2, 3] raw local affine frames of all images, image order (b, 0), (b, 1), ...
  const float* scores;          // [total]
  const float* desc;            // [total, D]
  const int* offsets;           // [2 B + 1] first raw keypoint of every image
  const int* select;            // optional [2 B, K]: caller's selection for images with more than K keypoints (random mode)
  const float* depth0;          // optional [B, H0, W0] depth images of image 0 (NULL: no depth output)
  const float* depth1;          // optional [B, H1, W1]
  int B, K, D, h0, w0, h1, w1;
  float* out_lafs0; float* out_lafs1;       // [B, K, 2, 3]
  float* out_scores0; float* out_scores1;   // [B, K]
  float* out_desc0; float* out_desc1;       // [B, K, D]
  float* out_depth0; float* out_depth1;     // [B, K] (optional)
  int sort_n;                   // shared-memory sort capacity (power of two >= the largest image)
};

constexpr int COLLATE_THREADS = 256;

__global__ void __launch_bounds__(COLLATE_THREADS) collate_kernel(CollateArgs a) {
  extern __shared__ __align__(16) unsigned char og_collate_smem[];
  float* key = reinterpret_cast<float*>(og_collate_smem);             // [sort_n]
  int* val = reinterpret_cast<int*>(key + a.sort_n);                  // [sort_n]
  const int b = blockIdx.x, img = blockIdx.y;
  const int i = 2 * b + img;
  const int first = a.offsets[i], cnt = a.offsets[i + 1] - first;
  const int K = a.K, D = a.D;
  const int keep = min(cnt, K);
  if (cnt > K && a.select == nullptr) cta_topk_sort<COLLATE_THREADS>(a.scores + first, cnt, key, val);
  float* o_lafs = (img ? a.out_lafs1 : a.out_lafs0) + (int64_t)b * K * 6;
  float* o_sc = (img ? a.out_scores1 : a.out_scores0) + (int64_t)b * K;
  float* o_desc = (img ? a.out_desc1 : a.out_desc0) + (int64_t)b * K * D;
  float* o_dep = img ? a.out_depth1 : a.out_depth0;
  const float* dimg = img ? a.depth1 : a.depth0;
  const int dh = img ? a.h1 : a.h0, dw = img ? a.w1 : a.w0;
  auto source = [&](int j) -> int {                  // raw keypoint behind output slot j (j < keep)
    if (cnt <= K) return j;
    return a.select ? a.select[(int64_t)i * K + j] : val[j];
  };
  for (int j = threadIdx.x; j < K; j += COLLATE_THREADS) {
    float l[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, s = 0.f, dep = 0.f;
    if (j < keep) {
      const int src = first + source(j);
#pragma unroll
      for (int e = 0; e < 6; ++e) l[e] = a.lafs[(int64_t)src * 6 + e];
      s = a.scores[src];
      if (dimg) {                                    // depth[int(y), int(x)]: lafs[:, 1, 2] = y, lafs[:, 0, 2] = x (truncation like .type(int64))
        int yy = (int)l[5], xx = (int)l[2];
        yy = min(max(yy, 0), dh - 1); xx = min(max(xx, 0), dw - 1);
        dep = dimg[((int64_t)b * dh + yy) * dw + xx];
      }
    }
#pragma unroll
    for (int e = 0; e < 6; ++e) o_lafs[(int64_t)j * 6 + e] = l[e];
    o_sc[j] = s;
    if (o_dep) o_dep[(int64_t)b * K + j] = dep;
  }
  // descriptors: one warp per kept row, coalesced along the channel dimension
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = warp; j < K; j += COLLATE_THREADS / 32) {
    float* dst = o_desc + (int64_t)j * D;
    if (j < keep) {
      const float* src = a.desc + (int64_t)(first + source(j)) * D;
      for (int c = lane; c < D; c += 32) dst[c] = src[c];
    } else {
      for (int c = lane; c < D; c += 32) dst[c] = 0.f;
    }
  }
}

inline int collate_launch(CollateArgs a, int max_count, cudaStream_t stream) {
  size_t smem;
  if (const int rc = cta_topk_smem<collate_kernel>(max_count, "collate: %d keypoints in one image > %d", &smem)) return rc;
  a.sort_n = pow2_ceil(max_count);
  return OG_LAUNCH(collate_kernel, dim3(a.B, 2), COLLATE_THREADS, smem, stream, a);
}

}  // namespace og
