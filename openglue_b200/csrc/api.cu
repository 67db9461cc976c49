// extern "C" entry points of libopenglue_b200.so (see include/openglue_b200.h) and the
// host-side schedule of the whole matching-core forward pass.
#include "common.cuh"
#include "linear_simt.cuh"
#include "linear_sm90.cuh"
#include "attention_simt.cuh"
#include "attention_sm90.cuh"
#include "sinkhorn.cuh"
#include "sinkhorn_bwd.cuh"
#include "match.cuh"
#include "gt_matches.cuh"
#include "criterion.cuh"
#include "metric_loss.cuh"
#include "collate.cuh"
#include "train_ops.cuh"
#include "superpoint.cuh"
#include "sift.cuh"
#include "kornia_sift.cuh"
#include "kornia_gftt.cuh"
#include "features.cuh"
#include "homography.cuh"
#include "optim.cuh"
#include <math.h>
#include <string.h>
#include <vector>

namespace og {

// Padded batch: row r of one image's [B, cap] rows is slot r % cap of pair b = r / cap, real below len[b] (clamped into [1, cap]).
__device__ __forceinline__ bool padded_row_real(int64_t r, int cap, const int* len) {
  const int b = (int)(r / cap);
  return (int)(r - (int64_t)b * cap) < padded_length(len, b, cap);
}

// keypoint normalisation + concat with side info:  in0[r] = [2*x/(W-1) - 1, 2*y/(H-1) - 1, side...]
// (reference superglue.py:74-78 and positional_encoding.py:16-18).  A padded batch (len non-null) takes each pair's (W - 1, H - 1)
// from wh (rows 4 floats apart: the image's (W, H) of the pair) and zeroes the rows past its length (whatever the padding slots
// hold, every row from here on is finite).
__global__ void __launch_bounds__(256) kenc_input_kernel(const float* __restrict__ kpts, const float* __restrict__ side,
                                                          int rows, int S, float wm1, float hm1, int cap, const int* __restrict__ len,
                                                          const float* __restrict__ wh, float* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float* o = out + (int64_t)r * (2 + S);
  if (len) {
    if (!padded_row_real(r, cap, len)) {
      for (int s = 0; s < 2 + S; ++s) o[s] = 0.f;
      return;
    }
    const int b = r / cap;
    wm1 = __ldg(wh + 4 * b) - 1.f;
    hm1 = __ldg(wh + 4 * b + 1) - 1.f;
  }
  o[0] = __fdiv_rn(2.f * __ldg(kpts + 2 * (int64_t)r), wm1) - 1.f;
  o[1] = __fdiv_rn(2.f * __ldg(kpts + 2 * (int64_t)r + 1), hm1) - 1.f;
  for (int s = 0; s < S; ++s) o[2 + s] = __ldg(side + (int64_t)r * S + s);
}

// dst = src [rows, d] with the rows past each pair's length zeroed (the descriptors a padded batch's residuals read)
__global__ void __launch_bounds__(256) mask_padded_rows_kernel(const float* __restrict__ src, int64_t rows, int cap, int d,
                                                                const int* __restrict__ len, float* __restrict__ dst) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows * d; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = padded_row_real(i / d, cap, len) ? __ldg(src + i) : 0.f;
}

// ctx [B, d, cap] (channel-first context descriptors): zero the columns past each pair's length
__global__ void __launch_bounds__(256) zero_padded_cols_kernel(float* __restrict__ ctx, int B, int d, int cap, const int* __restrict__ len) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (int64_t)B * d * cap; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / ((int64_t)d * cap));
    if ((int)(i % cap) >= padded_length(len, b, cap)) ctx[i] = 0.f;
  }
}

// out[b] = the Sinkhorn constants (norm, log_a_last, log_b_last) the padded kernels derive for pair b
__global__ void sinkhorn_consts_kernel(SinkArgs a, float* out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  const SinkPair p(a, b);
  out[3 * b] = p.norm; out[3 * b + 1] = p.log_a_last; out[3 * b + 2] = p.log_b_last;
}

struct Layout {           // float offsets of the packed weights
  std::vector<int64_t> kenc_w, kenc_b;
  std::vector<int64_t> qkv_w, qkv_b, fc1_w, fc1_b, fc2_w, fc2_b;
  int64_t proj_w, proj_b, proj_rmix, dustbin, total;
  std::vector<int> kenc_sizes;
};

static int check_config(const og_config* c) {
  OG_CHECK_ARG(c != nullptr, "config is null");
  OG_CHECK_ARG(c->descriptor_dim > 0 && c->num_heads > 0 && c->descriptor_dim % c->num_heads == 0,
               "descriptor_dim %d must be a positive multiple of num_heads %d", c->descriptor_dim, c->num_heads);
  OG_CHECK_ARG(c->num_layers >= 0 && c->num_layers % 2 == 0, "num_layers must be 2 * num_stages");
  OG_CHECK_ARG(c->side_info_size >= 0, "side_info_size < 0");
  OG_CHECK_ARG(c->num_hidden >= 0 && c->num_hidden <= OG_MAX_HIDDEN, "num_hidden out of range");
  OG_CHECK_ARG(c->sinkhorn_iters >= 0 && c->sinkhorn_reg > 0.f, "bad sinkhorn parameters");
  OG_CHECK_ARG(c->descriptor_dim % 4 == 0, "descriptor_dim must be a multiple of 4");
  return OG_OK;
}

static Layout make_layout(const og_config* c) {
  Layout L;
  const int64_t d = c->descriptor_dim;
  L.kenc_sizes.push_back(2 + c->side_info_size);
  for (int i = 0; i < c->num_hidden; ++i) L.kenc_sizes.push_back(c->hidden[i]);
  L.kenc_sizes.push_back((int)d);
  int64_t off = 0;
  auto take = [&](int64_t nfl) { int64_t o = off; off += (nfl + 3) / 4 * 4; return o; };   // keep 16-byte alignment
  for (size_t i = 1; i < L.kenc_sizes.size(); ++i) {
    L.kenc_w.push_back(take((int64_t)L.kenc_sizes[i] * L.kenc_sizes[i - 1]));
    L.kenc_b.push_back(take(L.kenc_sizes[i]));
  }
  for (int l = 0; l < c->num_layers; ++l) {
    L.qkv_w.push_back(take(3 * d * d)); L.qkv_b.push_back(take(3 * d));
    L.fc1_w.push_back(take(4 * d * d)); L.fc1_b.push_back(take(2 * d));
    L.fc2_w.push_back(take(2 * d * d)); L.fc2_b.push_back(take(d));
  }
  L.proj_w = take(d * d); L.proj_b = take(d); L.proj_rmix = take(d); L.dustbin = take(1);
  L.total = off;
  return L;
}

struct Workspace {
  float *in0, *h0, *h1, *x, *qkv, *o, *hid, *g, *ghi, *glo, *sbuf;
  float *q, *khi, *klo, *vthi, *vtlo;     // tensor-core attention operands (OG_PREC_TF32X3)
  int64_t ldn, ldm;                       // padded row lengths of the channel-major V^T buffers
  void *sink, *match;
  float* slots;                           // amax / scale scalars of the fp16 path (zeroed at the start of a forward pass)
  int nslots;
  float* desc;                            // padded batch: the descriptors of both images with their padding rows zeroed
  int64_t lds, sink_bytes, match_bytes, total;
};

static int plan_workspace(const og_config* c, int B, int n, int m, void* base, Workspace* w, bool padded = false) {
  const int64_t d = c->descriptor_dim, R = (int64_t)B * (n + m);
  int maxh = (int)d;
  for (int i = 0; i < c->num_hidden; ++i) maxh = std::max(maxh, c->hidden[i]);
  char* p = static_cast<char*>(base);
  int64_t off = 0;
  auto take = [&](int64_t bytes) { int64_t o = off; off += align_up(bytes, 256); return p ? (void*)(p + o) : nullptr; };
  w->in0 = (float*)take(R * (2 + c->side_info_size) * 4);
  w->h0 = (float*)take(R * maxh * 4);
  w->h1 = (float*)take(R * maxh * 4);
  w->x = (float*)take(R * d * 4);
  w->qkv = (float*)take(R * 3 * d * 4);
  w->o = (float*)take(R * d * 4);
  w->hid = (float*)take(R * 2 * d * 4);
  w->g = (float*)take(R * d * 4);
  w->ghi = (float*)take((int64_t)B * m * d * 4);          // tf32 split of image-1 descriptors (score GEMM B operand)
  w->glo = (float*)take((int64_t)B * m * d * 4);
  w->ldn = align_up(n, 8); w->ldm = align_up(m, 8);          // 16-byte rows for the fp16 form as well
  w->nslots = 16 * c->num_layers + 16;
  w->slots = (float*)take((int64_t)w->nslots * 4);
  if (c->precision == OG_PREC_TF32X3 || c->precision == OG_PREC_FP16X3) {
    w->q = (float*)take(R * d * 4);
    w->khi = (float*)take(R * d * 4);
    w->klo = (float*)take(R * d * 4);
    w->vthi = (float*)take((int64_t)B * d * (w->ldn + w->ldm) * 4);
    w->vtlo = (float*)take((int64_t)B * d * (w->ldn + w->ldm) * 4);
  } else {
    w->q = w->khi = w->klo = w->vthi = w->vtlo = nullptr;
  }
  w->lds = align_up(m, 4);
  w->sbuf = (float*)take((int64_t)B * n * w->lds * 4);
  w->sink_bytes = sinkhorn_workspace_bytes(B, n, m);
  if (w->sink_bytes < 0) return OG_EUNSUPPORTED;
  w->sink = take(w->sink_bytes);
  w->match_bytes = match_workspace_bytes(B, n, m);
  w->match = take(w->match_bytes);
  w->desc = padded ? (float*)take(R * d * 4) : nullptr;
  w->total = off;
  return OG_OK;
}

static og_linear_args lin(const float* A, int64_t lda, int k, const float* W, const float* bias, int rows, int nout,
                          float* Y, int64_t ldy) {
  og_linear_args a;
  memset(&a, 0, sizeof(a));
  a.A = A; a.lda = lda; a.k1 = k; a.W = W; a.ldw = k; a.bias = bias; a.rows = rows; a.nout = nout; a.batch = 1;
  a.alpha = 1.f; a.Y = Y; a.ldy = ldy;
  return a;
}

// The fields of the tensor-core GEMM arguments (TcLinearArgs or F16LinearArgs) that come from og_linear_args; the split and
// fp16 outputs and the fp16 operand scales are the caller's.  The fp16 form has no rscale or fp32 transposed output (a.Y: run F16_Y).
template <class T> static T gemm_args(const og_linear_args& a) {
  T t;
  memset(&t, 0, sizeof(t));
  t.A = a.A; t.lda = a.lda; t.strideA = a.strideA; t.A2 = a.A2; t.lda2 = a.lda2; t.strideA2 = a.strideA2;
  t.k1 = a.k1; t.k2 = a.k2;
  t.b_rows_per_batch = a.strideW ? (int)(a.strideW / a.ldw) : 0;
  t.bias = a.bias; t.rows = a.rows; t.nout = a.nout; t.batch = a.batch; t.alpha = a.alpha; t.relu = a.relu;
  t.R = a.R; t.ldr = a.ldr; t.strideR = a.strideR;
  if constexpr (std::is_same<T, TcLinearArgs>::value) {
    t.Y = a.Y; t.ldy = a.ldy; t.strideY = a.strideY; t.Yt = a.Yt; t.ldyt = a.ldyt; t.strideYt = a.strideYt; t.rscale = a.rscale;
  } else {
    t.out[F16_Y] = {a.Y, nullptr, nullptr, a.ldy, a.strideY, nullptr}; t.kind0 = F16_Y; t.nkinds = 1; t.kind_cols = a.nout;
  }
  return t;
}

// Whether the tensor-core GEMM can run t = gemm_args(a) + the caller's fields on the weight split Bhi / Blo (a.W's layout): every
// batch item starts at a whole row of B, and linear_sm90_eligible holds.
template <class T, class BT>
static bool gemm_tileable(const og_linear_args& a, const T& t, const BT* Bhi, const BT* Blo) {
  return (!a.strideW || a.strideW % a.ldw == 0) && linear_sm90_eligible(t, Bhi, Blo, a.ldw);
}

// Launches the tensor-core GEMM t on a shape gemm_tileable accepted.
template <class T, class BT>
static int gemm_launch(const og_linear_args& a, const T& t, const BT* Bhi, const BT* Blo, cudaStream_t s) {
  // rows the B tensor map may touch: the LAST batch item only owns nout rows (a map declared over b_rows_per_batch * batch rows
  // would let a 128-row TMA box read past the end of a head-sliced or exactly-sized operand; rows beyond the map are zero-filled)
  const int64_t brows = a.strideW ? (int64_t)t.b_rows_per_batch * (a.batch - 1) + a.nout : a.nout;
  return linear_sm90_launch(t, Bhi, Blo, a.ldw, brows, s);
}

// gemm_launch, where an untileable shape fails with "who: why"
template <class T, class BT>
static int linear_sm90_run(const og_linear_args& a, const T& t, const BT* Bhi, const BT* Blo, const char* who, const char* why,
                           cudaStream_t s) {
  if (!gemm_tileable(a, t, Bhi, Blo))
    return fail(OG_EUNSUPPORTED, "%s: %s", who, a.strideW && a.strideW % a.ldw != 0 ? "strideW must be a multiple of ldw" : why);
  return gemm_launch(a, t, Bhi, Blo, s);
}

// Split-output request for the tensor-core path (the fp32 CUDA-core path ignores it).
struct SplitOut { float *Yhi = nullptr, *Ylo = nullptr, *Ythi = nullptr, *Ytlo = nullptr; };

static TcLinearArgs tc_args(const og_linear_args& a, const SplitOut& so) {
  TcLinearArgs t = gemm_args<TcLinearArgs>(a);
  t.Yhi = so.Yhi; t.Ylo = so.Ylo; t.Ythi = so.Ythi; t.Ytlo = so.Ytlo;
  return t;
}

// Kernel selection for one linear layer: the wgmma 3xTF32 GEMM when asked for and the shape is tileable,
// otherwise the fp32 CUDA-core kernel (tiny K such as the 3-channel keypoint-encoder input).
static int linear_dispatch(const og_linear_args& a, int precision, cudaStream_t s, const float* Whi = nullptr,
                           const float* Wlo = nullptr, const SplitOut& so = SplitOut()) {
  if (precision == OG_PREC_TF32X3 && Whi && Wlo) {
    const TcLinearArgs t = tc_args(a, so);
    if (gemm_tileable(a, t, Whi, Wlo)) return gemm_launch(a, t, Whi, Wlo, s);
  }
  if (so.Yhi || so.Ythi) return fail(OG_EUNSUPPORTED, "split outputs need the tensor-core path");
  return linear_simt_launch(a, s);
}

// floats of W a GEMM reads: batch weight blocks strideW apart, the last of them nout rows of ldw of which the last ends after
// K elements (a head-sliced W, such as a column block of K, ends there; a whole last row of ldw would run past it)
static int64_t weight_floats(const og_linear_args& a) {
  const int64_t last = (int64_t)(a.nout - 1) * a.ldw + a.k1 + a.k2;
  return (a.batch > 1 && a.strideW) ? (int64_t)(a.batch - 1) * a.strideW + last : last;
}

}  // namespace og

using namespace og;

extern "C" {

int og_version(void) { return OG_VERSION; }
const char* og_last_error(void) { return err_buf(); }

int og_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  const DeviceInfo& d = device_info();
  if (!d.ok) return fail(OG_ECUDA, "no CUDA device");
  if (sm_count) *sm_count = d.sm_count;
  if (cc_major) *cc_major = d.cc_major;
  if (cc_minor) *cc_minor = d.cc_minor;
  return OG_OK;
}

int64_t og_packed_weight_floats(const og_config* cfg) {
  if (check_config(cfg) != OG_OK) return -1;
  return make_layout(cfg).total;
}

int64_t og_packed_offset(const og_config* cfg, int tensor_id, int index) {
  if (check_config(cfg) != OG_OK) return -1;
  Layout L = make_layout(cfg);
  auto at = [&](const std::vector<int64_t>& v) -> int64_t {
    return (index >= 0 && index < (int)v.size()) ? v[index] : (int64_t)fail(OG_EINVAL, "index %d out of range", index);
  };
  switch (tensor_id) {
    case OG_T_KENC_W: return at(L.kenc_w);
    case OG_T_KENC_B: return at(L.kenc_b);
    case OG_T_QKV_W: return at(L.qkv_w);
    case OG_T_QKV_B: return at(L.qkv_b);
    case OG_T_FC1_W: return at(L.fc1_w);
    case OG_T_FC1_B: return at(L.fc1_b);
    case OG_T_FC2_W: return at(L.fc2_w);
    case OG_T_FC2_B: return at(L.fc2_b);
    case OG_T_PROJ_W: return L.proj_w;
    case OG_T_PROJ_B: return L.proj_b;
    case OG_T_PROJ_RMIX: return L.proj_rmix;
    case OG_T_DUSTBIN: return L.dustbin;
    default: return fail(OG_EINVAL, "unknown tensor id %d", tensor_id);
  }
}

int64_t og_workspace_bytes(const og_config* cfg, int batch, int n, int m) {
  if (check_config(cfg) != OG_OK) return -1;
  if (batch <= 0 || n <= 0 || m <= 0) return fail(OG_EINVAL, "batch, n, m must be positive");
  Workspace w;
  if (plan_workspace(cfg, batch, n, m, nullptr, &w) != OG_OK) return -1;
  return w.total;
}

int og_last_forward_launches(void) { return launch_counter(); }

static int& fuse_qkv_mode() {
  static int v = [] { const char* e = getenv("OG_FUSE_QKV"); return e ? (atoi(e) != 0) : 1; }();
  return v;
}
int og_set_fusion(int fuse_projections) {
  const int prev = fuse_qkv_mode();
  if (fuse_projections >= 0) fuse_qkv_mode() = fuse_projections ? 1 : 0;
  return prev;
}

int og_set_tuning(int gemm_pair, int attention_pair) {
  (void)gemm_pair; (void)attention_pair;           // CTA-pair MMAs do not exist on sm_90: one kernel form per operator
  return OG_OK;
}

int og_linear_fwd(const og_linear_args* a, int precision, void* stream) {
  OG_CHECK_ARG(a && a->A && a->W && (a->Y || a->Yt), "linear: null pointer");
  OG_CHECK_ARG(precision == OG_PREC_FP32, "linear: the tensor-core form takes pre-split weights (og_linear_tc_fwd)");
  OG_CHECK_ARG(a->rows > 0 && a->nout > 0 && a->batch > 0 && a->k1 > 0 && a->k2 >= 0, "linear: bad sizes");
  OG_CHECK_ARG(a->k2 == 0 || a->A2, "linear: k2 > 0 needs A2");
  return linear_simt_launch(*a, (cudaStream_t)stream);
}

int og_linear_tc_fwd(const og_linear_args* a, const float* Whi, const float* Wlo, float* Yhi, float* Ylo, float* Ythi,
                     float* Ytlo, int mode, void* stream) {
  OG_CHECK_ARG(a && a->A && Whi && Wlo && (a->Y || a->Yt || Yhi || Ythi), "linear_tc: null pointer");
  OG_CHECK_ARG(a->rows > 0 && a->nout > 0 && a->batch > 0 && a->k1 > 0 && a->k2 >= 0, "linear_tc: bad sizes");
  OG_CHECK_ARG((Yhi == nullptr) == (Ylo == nullptr) && (Ythi == nullptr) == (Ytlo == nullptr), "linear_tc: hi/lo come in pairs");
  (void)mode;                                      // every mode runs the one sm_90 kernel (see the header)
  SplitOut so; so.Yhi = Yhi; so.Ylo = Ylo; so.Ythi = Ythi; so.Ytlo = Ytlo;
  return linear_sm90_run(*a, tc_args(*a, so), Whi, Wlo, "linear_tc",
                         "needs K >= 32, K % 4 == 0, k1 % 32 == 0 with a second operand and 16-byte aligned rows", (cudaStream_t)stream);
}

// one GEMM of the training step: wgmma 3xTF32 when the shape is tileable (W is split on the fly into split_scratch, 2 x the
// W footprint in floats), the exact fp32 CUDA-core kernel otherwise
int64_t og_linear_auto_scratch_floats(const og_linear_args* a) {
  if (!a || a->nout <= 0 || a->ldw <= 0 || a->batch <= 0) return -1;
  return 2 * align_up(weight_floats(*a), 64);
}
int og_linear_auto_fwd(const og_linear_args* a, int precision, float* split_scratch, void* stream) {
  OG_CHECK_ARG(a && a->A && a->W && (a->Y || a->Yt), "linear_auto: null pointer");
  OG_CHECK_ARG(a->rows > 0 && a->nout > 0 && a->batch > 0 && a->k1 > 0 && a->k2 >= 0, "linear_auto: bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  if (precision != OG_PREC_FP32 && split_scratch && aligned16(a->W)) {
    const int64_t wf = weight_floats(*a);
    float* hi = split_scratch; float* lo = split_scratch + align_up(wf, 64);
    const TcLinearArgs t = gemm_args<TcLinearArgs>(*a);
    if (gemm_tileable(*a, t, hi, lo)) {
      if (const int rc = OG_LAUNCH(split_tf32_kernel, (unsigned)((wf + 255) / 256), 256, 0, st, a->W, hi, lo, wf)) return rc;
      return gemm_launch(*a, t, hi, lo, st);
    }
  }
  return linear_simt_launch(*a, st);
}

int og_split_tf32(const float* src, float* hi, float* lo, int64_t n, void* stream) {
  OG_CHECK_ARG(src && hi && lo && n > 0, "split_tf32: bad arguments");
  return OG_LAUNCH(split_tf32_kernel, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, src, hi, lo, n);
}

static int attention_fwd_impl(const float* q, int64_t ldq, int64_t strideq, const float* k, int64_t ldk, int64_t stridek,
                              const float* v, int64_t ldv, int64_t stridev, float* out, int64_t ldo, int64_t strideo,
                              int batch, int nq, int nk, int num_heads, int head_dim, const int* klen, void* stream) {
  OG_CHECK_ARG(q && k && v && out, "attention: null pointer");
  OG_CHECK_ARG(batch > 0 && nq > 0 && nk > 0 && num_heads > 0 && head_dim > 0, "attention: bad sizes");
  AttnArgs a{q, ldq, strideq, k, ldk, stridek, v, ldv, stridev, out, ldo, strideo, batch, nq, nk, num_heads,
             (float)pow((double)head_dim, -0.5), klen};
  return attention_simt_launch(a, head_dim, (cudaStream_t)stream);
}

int og_attention_fwd(const float* q, int64_t ldq, int64_t strideq, const float* k, int64_t ldk, int64_t stridek,
                     const float* v, int64_t ldv, int64_t stridev, float* out, int64_t ldo, int64_t strideo,
                     int batch, int nq, int nk, int num_heads, int head_dim, int precision, void* stream) {
  (void)precision;                                   // raw fp32 operands: always the exact kernel (see the header)
  return attention_fwd_impl(q, ldq, strideq, k, ldk, stridek, v, ldv, stridev, out, ldo, strideo, batch, nq, nk, num_heads, head_dim,
                            nullptr, stream);
}

int og_attention_fwd_padded(const float* q, int64_t ldq, int64_t strideq, const float* k, int64_t ldk, int64_t stridek,
                            const float* v, int64_t ldv, int64_t stridev, float* out, int64_t ldo, int64_t strideo,
                            int batch, int nq, int nk, int num_heads, int head_dim, const int* key_lengths, void* stream) {
  OG_CHECK_ARG(key_lengths, "attention_padded: null key_lengths");
  return attention_fwd_impl(q, ldq, strideq, k, ldk, stridek, v, ldv, stridev, out, ldo, strideo, batch, nq, nk, num_heads, head_dim,
                            key_lengths, stream);
}

static int attention_tc_fwd_impl(const float* q, int64_t ldq, int64_t strideq, const float* khi, const float* klo, int64_t ldk,
                                 const float* vthi, const float* vtlo, int64_t ldvt, float* out, int64_t ldo, int64_t strideo,
                                 int batch, int nq, int nk, int num_heads, int head_dim, const int* klen, void* stream) {
  OG_CHECK_ARG(q && khi && klo && vthi && vtlo && out, "attention_tc: null pointer");
  OG_CHECK_ARG(batch > 0 && nq > 0 && nk > 0 && num_heads > 0, "attention_tc: bad sizes");
  if (!attention_tc_eligible(head_dim, ldq, ldk, ldvt, ldo))
    return fail(OG_EUNSUPPORTED, "attention_tc: head_dim in {32, 64} and 16-byte aligned rows required");
  TcAttnArgs a{q, ldq, strideq, out, ldo, strideo, batch, nq, nk, num_heads, num_heads * head_dim,
               (float)pow((double)head_dim, -0.5), klen};
  return attention_tc_launch(a, khi, klo, ldk, vthi, vtlo, ldvt, head_dim, (cudaStream_t)stream);
}

int og_attention_tc_fwd(const float* q, int64_t ldq, int64_t strideq, const float* khi, const float* klo, int64_t ldk,
                        const float* vthi, const float* vtlo, int64_t ldvt, float* out, int64_t ldo, int64_t strideo,
                        int batch, int nq, int nk, int num_heads, int head_dim, void* stream) {
  return attention_tc_fwd_impl(q, ldq, strideq, khi, klo, ldk, vthi, vtlo, ldvt, out, ldo, strideo, batch, nq, nk, num_heads, head_dim,
                               nullptr, stream);
}

int og_attention_tc_fwd_padded(const float* q, int64_t ldq, int64_t strideq, const float* khi, const float* klo, int64_t ldk,
                               const float* vthi, const float* vtlo, int64_t ldvt, float* out, int64_t ldo, int64_t strideo,
                               int batch, int nq, int nk, int num_heads, int head_dim, const int* key_lengths, void* stream) {
  OG_CHECK_ARG(key_lengths, "attention_tc_padded: null key_lengths");
  return attention_tc_fwd_impl(q, ldq, strideq, khi, klo, ldk, vthi, vtlo, ldvt, out, ldo, strideo, batch, nq, nk, num_heads, head_dim,
                               key_lengths, stream);
}

int64_t og_sinkhorn_workspace_bytes(int batch, int n, int m) { return sinkhorn_workspace_bytes(batch, n, m); }

int og_set_sinkhorn_resident(int resident) {
  const int prev = sink_resident_mode();
  if (resident >= 0) sink_resident_mode() = resident ? 1 : 0;
  return prev;
}

int og_sinkhorn_plan(int batch, int n, int m, int64_t* plan) {
  OG_CHECK_ARG(plan, "sinkhorn_plan: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0, "sinkhorn_plan: bad sizes");
  SinkPlan p;
  const bool resident = sink_resident_mode() && sinkhorn_resident_plan(batch, n, m, &p);
  if (!resident) {
    if (const int rc = sinkhorn_plan(false, batch, n, m, &p)) return rc;
    p.rows_reg = p.rows_smem = 0;
  }
  const int64_t v[10] = {resident, p.V, p.W, p.SP, p.rows_per_strip, p.pairs_per_launch, p.rows_reg, p.rows_smem,
                         (int64_t)p.smem, p.occ};
  for (int i = 0; i < 10; ++i) plan[i] = v[i];
  return OG_OK;
}

int og_sinkhorn_fwd(const float* S, int64_t lds, int64_t strideS, const float* dustbin, int batch, int n, int m,
                    int iters, float reg, float* scores, void* workspace, int64_t workspace_bytes, void* stream) {
  OG_CHECK_ARG(S && dustbin && scores && workspace, "sinkhorn: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0 && iters >= 0 && reg > 0.f, "sinkhorn: bad sizes");
  return sinkhorn_launch(S, lds, strideS, dustbin, batch, n, m, iters, reg, scores, workspace, workspace_bytes,
                         (cudaStream_t)stream);
}

int og_sinkhorn_fwd_padded(const float* S, int64_t lds, int64_t strideS, const float* dustbin, int batch, int n, int m,
                           const int* lengths, int iters, float reg, float* scores, void* workspace, int64_t workspace_bytes,
                           void* stream) {
  OG_CHECK_ARG(S && dustbin && lengths && scores && workspace, "sinkhorn_padded: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0 && iters >= 0 && reg > 0.f, "sinkhorn_padded: bad sizes");
  return sinkhorn_launch(S, lds, strideS, dustbin, batch, n, m, iters, reg, scores, workspace, workspace_bytes,
                         (cudaStream_t)stream, nullptr, nullptr, lengths);
}

int og_sinkhorn_consts(int n, int m, float* out) {
  OG_CHECK_ARG(out && n > 0 && m > 0, "sinkhorn_consts: bad arguments");
  const SinkConsts k = sinkhorn_consts(n, m);
  out[0] = k.norm; out[1] = k.log_a_last; out[2] = k.log_b_last;
  return OG_OK;
}

int og_sinkhorn_consts_padded(const int* lengths, int batch, int n, int m, float* out, void* stream) {
  OG_CHECK_ARG(lengths && out && batch > 0 && n > 0 && m > 0, "sinkhorn_consts_padded: bad arguments");
  OG_CHECK_ARG(n <= SINK_MAX_ROWS && m <= SINK_MAX_COLS, "sinkhorn_consts_padded: at most %d rows and %d columns", SINK_MAX_ROWS,
               SINK_MAX_COLS);
  cudaStream_t st = (cudaStream_t)stream;
  if (const int rc = sinkhorn_log_tables(st)) return rc;
  SinkArgs a;
  memset(&a, 0, sizeof(a));
  a.B = batch; a.n = n; a.m = m; a.len_n = lengths; a.len_m = lengths + batch;
  return OG_LAUNCH(sinkhorn_consts_kernel, cdiv(batch, 256), 256, 0, st, a, out);
}

int64_t og_sinkhorn_hist_floats(int batch, int n, int m, int iters) {
  return (batch > 0 && n > 0 && m > 0 && iters >= 0) ? sinkhorn_hist_floats(batch, n, m, iters) : -1;
}

int og_sinkhorn_train_fwd(const float* S, int64_t lds, int64_t strideS, const float* dustbin, int batch, int n, int m,
                          int iters, float reg, float* scores, float* hist, void* workspace, int64_t workspace_bytes, void* stream) {
  OG_CHECK_ARG(S && dustbin && scores && workspace && hist, "sinkhorn_train_fwd: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0 && iters >= 0 && reg > 0.f, "sinkhorn_train_fwd: bad sizes");
  return sinkhorn_launch(S, lds, strideS, dustbin, batch, n, m, iters, reg, scores, workspace, workspace_bytes, (cudaStream_t)stream,
                         hist, hist + (int64_t)batch * iters * (n + 1));
}

int og_sinkhorn_train_fwd_padded(const float* S, int64_t lds, int64_t strideS, const float* dustbin, int batch, int n, int m,
                                 const int* lengths, int iters, float reg, float* scores, float* hist, void* workspace,
                                 int64_t workspace_bytes, void* stream) {
  OG_CHECK_ARG(S && dustbin && lengths && scores && workspace && hist, "sinkhorn_train_fwd_padded: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0 && iters >= 0 && reg > 0.f, "sinkhorn_train_fwd_padded: bad sizes");
  return sinkhorn_launch(S, lds, strideS, dustbin, batch, n, m, iters, reg, scores, workspace, workspace_bytes, (cudaStream_t)stream,
                         hist, hist + (int64_t)batch * iters * (n + 1), lengths);
}

int64_t og_sinkhorn_bwd_workspace_bytes(int batch, int n, int m, int iters) {
  return (batch > 0 && n > 0 && m > 0 && iters >= 0) ? sinkhorn_bwd_workspace_bytes(batch, n, m, iters) : -1;
}

int og_sinkhorn_bwd(const float* S, int64_t lds, int64_t strideS, const float* dustbin, int batch, int n, int m, int iters, float reg,
                    const float* hist, const float* dscores, float* dS_aug, float* ddustbin, void* workspace, int64_t workspace_bytes,
                    void* stream) {
  OG_CHECK_ARG(S && dustbin && hist && dscores && dS_aug && ddustbin && workspace, "sinkhorn_bwd: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0 && iters >= 0 && reg > 0.f, "sinkhorn_bwd: bad sizes");
  return sinkhorn_bwd_launch(S, lds, strideS, dustbin, batch, n, m, iters, reg, hist, dscores, dS_aug, ddustbin, workspace,
                             workspace_bytes, (cudaStream_t)stream);
}

int og_sinkhorn_bwd_padded(const float* S, int64_t lds, int64_t strideS, const float* dustbin, int batch, int n, int m,
                           const int* lengths, int iters, float reg, const float* hist, const float* dscores, float* dS_aug,
                           float* ddustbin, void* workspace, int64_t workspace_bytes, void* stream) {
  OG_CHECK_ARG(S && dustbin && lengths && hist && dscores && dS_aug && ddustbin && workspace, "sinkhorn_bwd_padded: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0 && iters >= 0 && reg > 0.f, "sinkhorn_bwd_padded: bad sizes");
  return sinkhorn_bwd_launch(S, lds, strideS, dustbin, batch, n, m, iters, reg, hist, dscores, dS_aug, ddustbin, workspace,
                             workspace_bytes, (cudaStream_t)stream, lengths);
}

int64_t og_match_workspace_bytes(int batch, int n, int m) { return match_workspace_bytes(batch, n, m); }

int og_match_fwd(const float* scores, int batch, int n, int m, float threshold, int64_t* matches0, float* mscores0,
                 int64_t* matches1, float* mscores1, void* workspace, int64_t workspace_bytes, void* stream) {
  OG_CHECK_ARG(scores && workspace, "match: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0, "match: bad sizes");
  return match_launch(scores, batch, n, m, threshold, matches0, mscores0, matches1, mscores1, workspace,
                      workspace_bytes, (cudaStream_t)stream);
}

int og_match_fwd_padded(const float* scores, int batch, int n, int m, const int* lengths, float threshold, int64_t* matches0,
                        float* mscores0, int64_t* matches1, float* mscores1, void* workspace, int64_t workspace_bytes, void* stream) {
  OG_CHECK_ARG(scores && lengths && workspace, "match_padded: null pointer");
  OG_CHECK_ARG(batch > 0 && batch <= 65535 && n > 0 && m > 0, "match_padded: bad sizes");
  return match_launch(scores, batch, n, m, threshold, matches0, mscores0, matches1, mscores1, workspace,
                      workspace_bytes, (cudaStream_t)stream, lengths);
}

int64_t og_gt_matches_workspace_bytes(int batch, int n, int m) {
  if (batch <= 0 || n <= 0 || m <= 0) return -1;
  return gt_matches_workspace_bytes(batch, n, m);
}

static int gt_matches_impl(const float* kpts0, const float* kpts1, int batch, int n, int m, const int* lens, const og_gt_transform* tf,
                           int64_t* gt_matches0, int64_t* gt_matches1, void* workspace, int64_t workspace_bytes, void* stream) {
  OG_CHECK_ARG(kpts0 && kpts1 && tf && gt_matches0 && gt_matches1 && workspace, "gt_matches: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0, "gt_matches: bad sizes (the reference returns (None, None) for an empty keypoint set)");
  OG_CHECK_ARG(tf->type == OG_GT_PERSPECTIVE || tf->type == OG_GT_3D_REPROJECTION, "gt_matches: unknown transformation type %d", tf->type);
  if (tf->type == OG_GT_PERSPECTIVE) {
    OG_CHECK_ARG(tf->H, "gt_matches: perspective transformation needs H");
  } else {
    OG_CHECK_ARG(tf->K0 && tf->K1 && tf->R && tf->T && tf->depth0 && tf->depth1, "gt_matches: 3d_reprojection needs K0, K1, R, T, depth0, depth1");
    OG_CHECK_ARG(!tf->depth_is_image || (tf->depth0_h > 0 && tf->depth0_w > 0 && tf->depth1_h > 0 && tf->depth1_w > 0),
                 "gt_matches: depth image sizes");
  }
  return gt_matches_launch(kpts0, kpts1, batch, n, m, *tf, gt_matches0, gt_matches1, workspace, workspace_bytes, (cudaStream_t)stream,
                           lens);
}

int og_gt_matches_fwd(const float* kpts0, const float* kpts1, int batch, int n, int m, const og_gt_transform* tf,
                      int64_t* gt_matches0, int64_t* gt_matches1, void* workspace, int64_t workspace_bytes, void* stream) {
  return gt_matches_impl(kpts0, kpts1, batch, n, m, nullptr, tf, gt_matches0, gt_matches1, workspace, workspace_bytes, stream);
}

int og_gt_matches_fwd_padded(const float* kpts0, const float* kpts1, int batch, int n, int m, const int* lengths,
                             const og_gt_transform* tf, int64_t* gt_matches0, int64_t* gt_matches1, void* workspace,
                             int64_t workspace_bytes, void* stream) {
  OG_CHECK_ARG(lengths, "gt_matches_padded: null lengths");
  return gt_matches_impl(kpts0, kpts1, batch, n, m, lengths, tf, gt_matches0, gt_matches1, workspace, workspace_bytes, stream);
}

int og_collate_fwd(const float* lafs, const float* scores, const float* desc, const int* offsets, const int* select, int max_count,
                   const float* depth0, int depth0_h, int depth0_w, const float* depth1, int depth1_h, int depth1_w,
                   int batch, int target_keypoints, int descriptor_dim,
                   float* out_lafs0, float* out_lafs1, float* out_scores0, float* out_scores1, float* out_desc0, float* out_desc1,
                   float* out_depth0, float* out_depth1, void* stream) {
  OG_CHECK_ARG(lafs && scores && desc && offsets && out_lafs0 && out_lafs1 && out_scores0 && out_scores1 && out_desc0 && out_desc1,
               "collate: null pointer");
  OG_CHECK_ARG(batch > 0 && target_keypoints > 0 && descriptor_dim > 0 && max_count >= 0, "collate: bad sizes");
  OG_CHECK_ARG((depth0 == nullptr) == (out_depth0 == nullptr) && (depth1 == nullptr) == (out_depth1 == nullptr), "collate: depth in / out come together");
  OG_CHECK_ARG(!depth0 || (depth0_h > 0 && depth0_w > 0), "collate: depth0 size");
  OG_CHECK_ARG(!depth1 || (depth1_h > 0 && depth1_w > 0), "collate: depth1 size");
  CollateArgs a;
  a.lafs = lafs; a.scores = scores; a.desc = desc; a.offsets = offsets; a.select = select; a.depth0 = depth0; a.depth1 = depth1;
  a.B = batch; a.K = target_keypoints; a.D = descriptor_dim; a.h0 = depth0_h; a.w0 = depth0_w; a.h1 = depth1_h; a.w1 = depth1_w;
  a.out_lafs0 = out_lafs0; a.out_lafs1 = out_lafs1; a.out_scores0 = out_scores0; a.out_scores1 = out_scores1;
  a.out_desc0 = out_desc0; a.out_desc1 = out_desc1; a.out_depth0 = out_depth0; a.out_depth1 = out_depth1; a.sort_n = 1;
  return collate_launch(a, std::max(max_count, 1), (cudaStream_t)stream);
}

int64_t og_criterion_workspace_bytes(int batch) { return batch > 0 ? criterion_workspace_bytes(batch) : -1; }

int og_criterion_fwd(const float* scores, const int64_t* gt_matches0, const int64_t* gt_matches1, int batch, int n, int m,
                     float* loss, float* dscores, float grad_scale, void* workspace, int64_t workspace_bytes, void* stream) {
  OG_CHECK_ARG(scores && gt_matches0 && gt_matches1 && loss && workspace, "criterion: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0, "criterion: bad sizes");
  return criterion_launch(scores, gt_matches0, gt_matches1, batch, n, m, loss, dscores, grad_scale, workspace, workspace_bytes,
                          (cudaStream_t)stream);
}

int og_criterion_fwd_padded(const float* scores, const int64_t* gt_matches0, const int64_t* gt_matches1, int batch, int n, int m,
                            const int* lengths, float* loss, float* dscores, float grad_scale, void* workspace, int64_t workspace_bytes,
                            void* stream) {
  OG_CHECK_ARG(scores && gt_matches0 && gt_matches1 && lengths && loss && workspace, "criterion_padded: null pointer");
  OG_CHECK_ARG(batch > 0 && n > 0 && m > 0, "criterion_padded: bad sizes");
  return criterion_launch(scores, gt_matches0, gt_matches1, batch, n, m, loss, dscores, grad_scale, workspace, workspace_bytes,
                          (cudaStream_t)stream, lengths);
}

static bool metric_sizes_ok(int batch, int d, int n, int m, int precision) {
  return batch >= 1 && batch <= 65535 && d >= 1 && n >= 1 && m >= 1 && (precision == OG_PREC_FP32 || precision == OG_PREC_TF32X3);
}
int64_t og_metric_loss_workspace_bytes(int batch, int d, int n, int m, int want_grad, int precision) {
  return metric_sizes_ok(batch, d, n, m, precision) ? metric_workspace_bytes(batch, n, m, d, want_grad, precision) : -1;
}
int og_metric_loss_fwd(const float* c0, const float* c1, const int64_t* gt_matches0, const int64_t* gt_matches1, int batch, int d,
                       int n, int m, float margin, int precision, float* metric_loss, int64_t* n0, int64_t* u0, int64_t* n1,
                       int64_t* u1, float* dc0, float* dc1, float grad_scale, void* workspace, int64_t workspace_bytes,
                       void* stream) {
  OG_CHECK_ARG(c0 && c1 && gt_matches0 && gt_matches1 && metric_loss && n0 && u0 && n1 && u1 && workspace, "metric_loss: null pointer");
  OG_CHECK_ARG((dc0 == nullptr) == (dc1 == nullptr), "metric_loss: dc0 and dc1 come together");
  OG_CHECK_ARG(metric_sizes_ok(batch, d, n, m, precision), "metric_loss: bad sizes or precision");
  return metric_loss_launch(c0, c1, gt_matches0, gt_matches1, batch, d, n, m, margin, precision, metric_loss, n0, u0, n1, u1, dc0, dc1,
                            grad_scale, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ---- training-step operators (row f1; csrc/train_ops.cuh) ----
int64_t og_train_workspace_floats(int cols) { return cols > 0 ? colreduce_workspace_floats(cols) + 2 * (int64_t)cols : -1; }

int og_transpose(const float* in, int64_t ld_in, int64_t stride_in, float* out, int64_t ld_out, int64_t stride_out,
                 int batch, int rows, int cols, int transpose, void* stream) {
  OG_CHECK_ARG(in && out, "transpose: null pointer");
  OG_CHECK_ARG(batch >= 0 && rows >= 0 && cols >= 0 && ld_in >= cols && ld_out >= (transpose ? rows : cols), "transpose: bad sizes");
  return transpose_launch(in, ld_in, stride_in, out, ld_out, stride_out, batch, rows, cols, transpose, (cudaStream_t)stream);
}

int og_colsum(const float* x, int64_t ldx, const float* y, int64_t ldy, const float* z, int64_t ldz, int rows, int cols,
              float* out, float* workspace, void* stream) {
  OG_CHECK_ARG(x && out && workspace, "colsum: null pointer");
  OG_CHECK_ARG(rows >= 0 && cols > 0 && (!z || y), "colsum: bad arguments");
  ColReduceArgs a = {};
  a.x = x; a.ldx = ldx; a.y = y; a.ldy = ldy; a.z = z; a.ldz = ldz; a.rows = rows; a.cols = cols; a.partial = workspace; a.out0 = out;
  return colreduce_launch<0>(a, (cudaStream_t)stream);
}

static int bn_train_fwd_impl(const float* a_, int64_t lda, int rows, int cols, int relu, const float* gamma, const float* beta,
                             float eps, float momentum, float* y, int64_t ldy, float* save_mean, float* save_invstd,
                             float* running_mean, float* running_var, float* workspace, const int* len, int cap, const int* skip,
                             long long* num_batches_tracked, void* stream) {
  OG_CHECK_ARG(a_ && gamma && beta && y && save_mean && save_invstd && workspace, "bn_train_fwd: null pointer");
  OG_CHECK_ARG(rows > 0 && cols > 0, "bn_train_fwd: bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  float* var = workspace;                                   // [cols]
  ColReduceArgs r = {};
  r.x = a_; r.ldx = lda; r.rows = rows; r.cols = cols; r.relu = relu; r.partial = workspace + 2 * (int64_t)cols; r.out0 = save_mean;
  r.len = len; r.cap = cap;
  int rc = colreduce_launch<1>(r, st);
  if (rc != OG_OK) return rc;
  r.mu = save_mean; r.out0 = var;
  if ((rc = colreduce_launch<2>(r, st)) != OG_OK) return rc;
  if ((rc = OG_LAUNCH(bn_finish_stats_kernel, cdiv(cols, 256), 256, 0, st, save_mean, var, cols, rows, len, cap, eps, momentum, save_invstd,
                      running_mean, running_var, skip, num_batches_tracked)) != OG_OK) return rc;
  return OG_LAUNCH(bn_apply_kernel, eltwise_grid((int64_t)rows * cols), 256, 0, st, a_, lda, rows, cols, relu, save_mean, save_invstd, gamma,
                   beta, y, ldy);
}

int og_bn_train_fwd(const float* a_, int64_t lda, int rows, int cols, int relu, const float* gamma, const float* beta,
                    float eps, float momentum, float* y, int64_t ldy, float* save_mean, float* save_invstd,
                    float* running_mean, float* running_var, float* workspace, void* stream) {
  return bn_train_fwd_impl(a_, lda, rows, cols, relu, gamma, beta, eps, momentum, y, ldy, save_mean, save_invstd, running_mean, running_var,
                           workspace, nullptr, rows, nullptr, nullptr, stream);
}

int og_bn_train_fwd_padded(const float* a_, int64_t lda, int batch, int cap, const int* lengths, int cols, int relu, const float* gamma,
                           const float* beta, float eps, float momentum, float* y, int64_t ldy, float* save_mean, float* save_invstd,
                           float* running_mean, float* running_var, float* workspace, void* stream) {
  OG_CHECK_ARG(lengths && batch > 0 && cap > 0 && (int64_t)batch * cap <= INT32_MAX, "bn_train_fwd_padded: bad lengths or sizes");
  return bn_train_fwd_impl(a_, lda, batch * cap, cols, relu, gamma, beta, eps, momentum, y, ldy, save_mean, save_invstd, running_mean,
                           running_var, workspace, lengths, cap, nullptr, nullptr, stream);
}

int og_bn_train_fwd_guarded(const float* a_, int64_t lda, int batch, int cap, const int* lengths, int cols, int relu, const float* gamma,
                            const float* beta, float eps, float momentum, float* y, int64_t ldy, float* save_mean, float* save_invstd,
                            float* running_mean, float* running_var, const int* skip, int64_t* num_batches_tracked, float* workspace,
                            void* stream) {
  OG_CHECK_ARG(batch > 0 && cap > 0 && (int64_t)batch * cap <= INT32_MAX, "bn_train_fwd_guarded: bad sizes");
  return bn_train_fwd_impl(a_, lda, batch * cap, cols, relu, gamma, beta, eps, momentum, y, ldy, save_mean, save_invstd, running_mean,
                           running_var, workspace, lengths, cap, skip, reinterpret_cast<long long*>(num_batches_tracked), stream);
}

int og_train_guard(const int* lengths, int B, int* skip, void* stream) {
  OG_CHECK_ARG(lengths && skip, "train_guard: null pointer");
  OG_CHECK_ARG(B > 0 && B <= INT32_MAX / 2, "train_guard: B = %d must be positive", B);
  return OG_LAUNCH(train_guard_kernel, 1, 32, 0, (cudaStream_t)stream, lengths, B, skip);
}

int og_train_skip_outputs(const int* skip, float* loss, int nloss, float* x, int64_t n, void* stream) {
  OG_CHECK_ARG(skip && (loss || nloss == 0) && (x || n == 0), "train_skip_outputs: null pointer");
  OG_CHECK_ARG(nloss >= 0 && nloss <= 256 && n >= 0, "train_skip_outputs: bad sizes");
  if (nloss == 0 && n == 0) return OG_OK;
  return OG_LAUNCH(train_skip_outputs_kernel, std::max(eltwise_grid(n), 1u), 256, 0, (cudaStream_t)stream, skip, loss, nloss, x, n);
}

static int bn_train_bwd_impl(const float* dy, int64_t lddy, const float* a_, int64_t lda, int rows, int cols, int relu,
                             const float* gamma, const float* save_mean, const float* save_invstd,
                             float* da, int64_t ldda, float* dgamma, float* dbeta, float* workspace, const int* len, int cap, void* stream) {
  OG_CHECK_ARG(dy && a_ && gamma && save_mean && save_invstd && da && dgamma && dbeta && workspace, "bn_train_bwd: null pointer");
  OG_CHECK_ARG(rows > 0 && cols > 0, "bn_train_bwd: bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  ColReduceArgs r = {};
  r.x = dy; r.ldx = lddy; r.y = a_; r.ldy = lda; r.mu = save_mean; r.invstd = save_invstd; r.rows = rows; r.cols = cols; r.relu = relu;
  r.partial = workspace + 2 * (int64_t)cols; r.out0 = dbeta; r.out1 = dgamma;
  r.len = len; r.cap = cap;
  int rc = colreduce_launch<3>(r, st);
  if (rc != OG_OK) return rc;
  return OG_LAUNCH(bn_bwd_apply_kernel, eltwise_grid((int64_t)rows * cols), 256, 0, st, dy, lddy, a_, lda, rows, cols, relu, save_mean,
                   save_invstd, gamma, dgamma, dbeta, da, ldda, len, cap);
}

int og_bn_train_bwd(const float* dy, int64_t lddy, const float* a_, int64_t lda, int rows, int cols, int relu,
                    const float* gamma, const float* save_mean, const float* save_invstd,
                    float* da, int64_t ldda, float* dgamma, float* dbeta, float* workspace, void* stream) {
  return bn_train_bwd_impl(dy, lddy, a_, lda, rows, cols, relu, gamma, save_mean, save_invstd, da, ldda, dgamma, dbeta, workspace,
                           nullptr, rows, stream);
}

int og_bn_train_bwd_padded(const float* dy, int64_t lddy, const float* a_, int64_t lda, int batch, int cap, const int* lengths, int cols,
                           int relu, const float* gamma, const float* save_mean, const float* save_invstd,
                           float* da, int64_t ldda, float* dgamma, float* dbeta, float* workspace, void* stream) {
  OG_CHECK_ARG(lengths && batch > 0 && cap > 0 && (int64_t)batch * cap <= INT32_MAX, "bn_train_bwd_padded: bad lengths or sizes");
  return bn_train_bwd_impl(dy, lddy, a_, lda, batch * cap, cols, relu, gamma, save_mean, save_invstd, da, ldda, dgamma, dbeta, workspace,
                           lengths, cap, stream);
}

int og_softmax_rows(float* S, int64_t ld, int64_t rows, int cols, void* stream) {
  OG_CHECK_ARG(S && rows >= 0 && cols > 0 && ld >= cols, "softmax_rows: bad arguments");
  if (rows == 0) return OG_OK;
  OG_CHECK_ARG((rows + 7) / 8 <= 0x7fffffffLL, "softmax_rows: too many rows");
  return OG_LAUNCH(softmax_rows_kernel, (unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream, S, ld, rows, cols, nullptr, rows);
}

int og_softmax_rows_padded(float* S, int64_t ld, int batch, int64_t seq_rows, int cols, const int* key_lengths, void* stream) {
  OG_CHECK_ARG(S && key_lengths && batch > 0 && seq_rows > 0 && cols > 0 && ld >= cols, "softmax_rows_padded: bad arguments");
  const int64_t rows = (int64_t)batch * seq_rows;
  OG_CHECK_ARG((rows + 7) / 8 <= 0x7fffffffLL, "softmax_rows_padded: too many rows");
  return OG_LAUNCH(softmax_rows_kernel, (unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream, S, ld, rows, cols, key_lengths, seq_rows);
}

int og_softmax_bwd_rows(const float* P, float* dP, int64_t ld, int64_t rows, int cols, float scale, void* stream) {
  OG_CHECK_ARG(P && dP && rows >= 0 && cols > 0 && ld >= cols, "softmax_bwd_rows: bad arguments");
  if (rows == 0) return OG_OK;
  OG_CHECK_ARG((rows + 7) / 8 <= 0x7fffffffLL, "softmax_bwd_rows: too many rows");
  return OG_LAUNCH(softmax_bwd_rows_kernel, (unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream, P, dP, ld, rows, cols, scale, nullptr, rows);
}

int og_softmax_bwd_rows_padded(const float* P, float* dP, int64_t ld, int batch, int64_t seq_rows, int cols, float scale,
                               const int* key_lengths, void* stream) {
  OG_CHECK_ARG(P && dP && key_lengths && batch > 0 && seq_rows > 0 && cols > 0 && ld >= cols, "softmax_bwd_rows_padded: bad arguments");
  const int64_t rows = (int64_t)batch * seq_rows;
  OG_CHECK_ARG((rows + 7) / 8 <= 0x7fffffffLL, "softmax_bwd_rows_padded: too many rows");
  return OG_LAUNCH(softmax_bwd_rows_kernel, (unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream, P, dP, ld, rows, cols, scale,
                   key_lengths, seq_rows);
}

int og_sum_batches(const float* part, int S, int rows, int cols, float* out, int64_t ld_out, int accumulate, void* stream) {
  OG_CHECK_ARG(part && out && S > 0 && rows > 0 && cols > 0 && ld_out >= cols, "sum_batches: bad arguments");
  return OG_LAUNCH(sum_batches_kernel, eltwise_grid((int64_t)rows * cols), 256, 0, (cudaStream_t)stream, part, S, rows, cols, out, ld_out,
                   accumulate);
}

int og_axpby(const float* x, const float* y, float a_, float b, float* out, int64_t n, void* stream) {
  OG_CHECK_ARG(x && out && n >= 0, "axpby: bad arguments");
  if (n == 0) return OG_OK;
  return OG_LAUNCH(axpby_kernel, eltwise_grid(n), 256, 0, (cudaStream_t)stream, x, y, a_, b, out, n);
}

int og_mix_fwd(const float* g, const float* l, const float* mix, float* out, int64_t rows, int d, void* stream) {
  OG_CHECK_ARG(g && l && mix && out && rows > 0 && d > 0, "mix_fwd: bad arguments");
  return OG_LAUNCH(mix_fwd_kernel, eltwise_grid(rows * d), 256, 0, (cudaStream_t)stream, g, l, mix, out, rows, d);
}

int og_mix_bwd(const float* dm, const float* mix, float* dg, float* dl, int64_t rows, int d, void* stream) {
  OG_CHECK_ARG(dm && mix && (dg || dl) && rows > 0 && d > 0, "mix_bwd: bad arguments");
  return OG_LAUNCH(mix_bwd_kernel, eltwise_grid(rows * d), 256, 0, (cudaStream_t)stream, dm, mix, dg, dl, rows, d);
}

int og_mix_param_grad(const float* colsum, const float* mix, float* dmix, int d, void* stream) {
  OG_CHECK_ARG(colsum && mix && dmix && d > 0, "mix_param_grad: bad arguments");
  return OG_LAUNCH(mix_param_grad_kernel, cdiv(d, 256), 256, 0, (cudaStream_t)stream, colsum, mix, dmix, d);
}

int og_kenc_input(const float* kpts, const float* side, int rows, int side_info_size, float width, float height, float* out, void* stream) {
  OG_CHECK_ARG(kpts && out && rows > 0 && side_info_size >= 0 && (side_info_size == 0 || side), "kenc_input: bad arguments");
  return OG_LAUNCH(kenc_input_kernel, cdiv(rows, 256), 256, 0, (cudaStream_t)stream, kpts, side, rows, side_info_size, width - 1.f,
                   height - 1.f, rows, nullptr, nullptr, out);
}

int og_kenc_input_padded(const float* kpts, const float* side, int batch, int cap, const int* lengths, int side_info_size,
                         const float* pair_wh, float* out, void* stream) {
  OG_CHECK_ARG(kpts && out && lengths && pair_wh && batch > 0 && cap > 0 && (int64_t)batch * cap <= INT32_MAX && side_info_size >= 0 &&
               (side_info_size == 0 || side), "kenc_input_padded: bad arguments");
  const int rows = batch * cap;
  return OG_LAUNCH(kenc_input_kernel, cdiv(rows, 256), 256, 0, (cudaStream_t)stream, kpts, side, rows, side_info_size, 0.f, 0.f, cap,
                   lengths, pair_wh, out);
}

int og_mask_padded_rows(const float* src, int batch, int cap, int cols, const int* lengths, float* dst, void* stream) {
  OG_CHECK_ARG(src && dst && lengths && batch > 0 && cap > 0 && cols > 0, "mask_padded_rows: bad arguments");
  const int64_t rows = (int64_t)batch * cap;
  return OG_LAUNCH(mask_padded_rows_kernel, eltwise_grid(rows * cols), 256, 0, (cudaStream_t)stream, src, rows, cap, cols, lengths, dst);
}

// ---- SuperPoint front-end operators (row f4; csrc/superpoint.cuh) ----
int og_sp_im2col3x3(const float* x, int B, int H, int W, int C, float* out, void* stream) {
  OG_CHECK_ARG(x && out && B > 0 && H > 0 && W > 0 && C > 0, "sp_im2col3x3: bad arguments");
  return OG_LAUNCH(im2col3x3_kernel, sp_grid((int64_t)B * H * W * 9 * ((C % 4 == 0) ? C / 4 : C)), 256, 0, (cudaStream_t)stream, x, B, H, W,
                   C, out);
}
int og_sp_maxpool2x2(const float* x, int B, int H, int W, int C, float* out, void* stream) {
  OG_CHECK_ARG(x && out && B > 0 && H > 0 && W > 0 && C > 0 && H % 2 == 0 && W % 2 == 0, "sp_maxpool2x2: bad arguments");
  return OG_LAUNCH(maxpool2x2_kernel, sp_grid((int64_t)B * (H / 2) * (W / 2) * C), 256, 0, (cudaStream_t)stream, x, B, H, W, C, out);
}
int og_row_normalize(float* x, int64_t rows, int C, int mode, float eps, void* stream) {
  OG_CHECK_ARG(x && rows >= 0 && C > 0 && (mode == 0 || mode == 1), "row_normalize: bad arguments");
  if (rows == 0) return OG_OK;
  return OG_LAUNCH(row_normalize_kernel, (unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream, x, rows, C, mode, eps);
}
int og_sp_heat_nms(const float* probs, int B, int Hc, int Wc, int nms_kernel, float threshold, int border, float* heat, void* stream) {
  OG_CHECK_ARG(probs && heat && B > 0 && Hc > 0 && Wc > 0 && nms_kernel > 0 && nms_kernel % 2 == 1 && border >= 0, "sp_heat_nms: bad arguments");
  return OG_LAUNCH(sp_heat_nms_kernel, sp_grid((int64_t)B * Hc * Wc * 64), 256, 0, (cudaStream_t)stream, probs, B, Hc, Wc, nms_kernel,
                   threshold, border, heat);
}
int og_sp_compact(const float* heat, int B, int HW, int cap, int* cand_idx, float* cand_score, int* count, void* stream) {
  OG_CHECK_ARG(heat && cand_idx && cand_score && count && B > 0 && HW > 0 && cap > 0, "sp_compact: bad arguments");
  return OG_LAUNCH(sp_compact_kernel, B, 1024, 0, (cudaStream_t)stream, heat, HW, cap, cand_idx, cand_score, count);
}
int og_sp_select(const int* cand_idx, const float* cand_score, const int* count, const int* n_out, const int* mode, int B, int cap, int W,
                 int out_cap, int max_count, float* kpts, float* scores, void* stream) {
  OG_CHECK_ARG(cand_idx && cand_score && count && n_out && mode && kpts && scores, "sp_select: null pointer");
  OG_CHECK_ARG(B > 0 && cap > 0 && W > 0 && out_cap > 0 && max_count >= 0, "sp_select: bad sizes");
  size_t smem;
  if (const int rc = cta_topk_smem<sp_select_kernel>(max_count, "sp_select: %d candidates in one image exceed the sort capacity %d",
                                                     &smem))
    return rc;
  return OG_LAUNCH(sp_select_kernel, B, 1024, smem, (cudaStream_t)stream, cand_idx, cand_score, count, n_out, mode, cap, W, out_cap, kpts,
                   scores);
}
int og_sp_sample_desc(const float* coarse, int B, int Hc, int Wc, int D, const float* kpts, const int* n_out, int out_cap, int max_n, int cell,
                      float* desc, void* stream) {
  OG_CHECK_ARG(coarse && kpts && n_out && desc && B > 0 && Hc > 0 && Wc > 0 && D > 0 && out_cap > 0 && cell > 0, "sp_sample_desc: bad arguments");
  if (max_n <= 0) return OG_OK;
  return OG_LAUNCH(sp_sample_desc_kernel, dim3(cdiv(max_n, 8), B), 256, 0, (cudaStream_t)stream, coarse, Hc, Wc, D, kpts, n_out, out_cap,
                   cell, desc);
}

// ---- OpenCV SIFT front-end (csrc/sift.cuh) ----
int64_t og_sift_workspace_bytes(int B, int H, int W, int cap) {
  SiftLayout L;
  if (B <= 0 || B > 65535 || H <= 0 || W <= 0 || cap <= 0 || cap > (1 << 24)) return fail(OG_EINVAL, "sift_workspace_bytes: bad sizes");
  if (!sift_layout(B, H, W, cap, L)) return fail(OG_EUNSUPPORTED, "sift: a %d x %d image has no octave or more than %d", H, W, SIFT_MAX_OCTAVES);
  return L.total;
}
int og_sift_workspace_layout(int B, int H, int W, int cap, int64_t* out, int n) {
  OG_CHECK_ARG(out, "sift_workspace_layout: null pointer");
  const int64_t bytes = og_sift_workspace_bytes(B, H, W, cap);
  if (bytes < 0) return (int)bytes;
  SiftLayout L;
  sift_layout(B, H, W, cap, L);
  const int need = 1 + 4 * L.nO + 5;
  OG_CHECK_ARG(n >= need, "sift_workspace_layout: %d entries, %d needed", n, need);
  int i = 0;
  out[i++] = L.nO;
  for (int o = 0; o < L.nO; ++o) {
    out[i++] = L.h[o]; out[i++] = L.w[o]; out[i++] = L.gauss_off[o]; out[i++] = L.dog_off[o];
  }
  out[i++] = L.loc_off; out[i++] = L.kp_off; out[i++] = L.oct_off; out[i++] = L.cnt_off; out[i++] = L.total;
  return i;
}
int og_sift_gaussian_taps(double sigma, float* taps, int cap) {
  OG_CHECK_ARG(taps && sigma > 0 && cap > 0, "sift_gaussian_taps: bad arguments");
  const int n = sift_gaussian_taps(sigma, taps, cap);
  if (n < 0) return fail(OG_EUNSUPPORTED, "sift_gaussian_taps: sigma %g needs more than %d taps", sigma, cap);
  return n;
}
static int sift_blur(const float* src, int B, int h, int w, double sigma, float* tmp, float* dst, float* dog, cudaStream_t st) {
  SiftTaps t;
  t.n = sift_gaussian_taps(sigma, t.k, SIFT_MAX_TAPS);
  if (t.n < 0) return fail(OG_EUNSUPPORTED, "sift: sigma %g needs more than %d taps", sigma, SIFT_MAX_TAPS);
  const int64_t n = (int64_t)B * h * w;
  if (const int rc = OG_LAUNCH(sift_blur_rows_kernel, sift_grid(n), 256, 0, st, src, B, h, w, t, tmp)) return rc;
  return OG_LAUNCH(sift_blur_cols_kernel, sift_grid(n), 256, 0, st, tmp, B, h, w, t, dst, src, dog);
}
// og_sift_detect, and with overflow non-null og_sift_detect_padded (see sift_sort_unique_kernel)
static int sift_detect(const void* image, int dtype, int B, int H, int W, int cap, void* ws, int64_t ws_bytes, float* kp, int* octave,
                       int* count, int* overflow, void* stream) {
  OG_CHECK_ARG(image && ws && kp && octave && count, "sift_detect: null pointer");
  OG_CHECK_ARG(dtype == 0 || dtype == 1, "sift_detect: dtype must be 0 (uint8) or 1 (float32)");
  const int64_t need = og_sift_workspace_bytes(B, H, W, cap);
  if (need < 0) return (int)need;
  OG_CHECK_ARG(ws_bytes >= need, "sift_detect: workspace of %lld bytes, %lld needed", (long long)ws_bytes, (long long)need);
  SiftLayout L;
  sift_layout(B, H, W, cap, L);
  unsigned char* w8 = static_cast<unsigned char*>(ws);
  cudaStream_t st = (cudaStream_t)stream;
  const SiftPyramid P = sift_pyramid(w8, L, B);
  float* tmp = reinterpret_cast<float*>(w8 + L.tmp_off);
  int* loc_count = reinterpret_cast<int*>(w8 + L.cnt_off);
  int* kp_count = loc_count + B;
  SiftLoc* loc = reinterpret_cast<SiftLoc*>(w8 + L.loc_off);
  float* kp_raw = reinterpret_cast<float*>(w8 + L.kp_off);
  int* oct_raw = reinterpret_cast<int*>(w8 + L.oct_off);
  int* work = reinterpret_cast<int*>(w8 + L.work_off);
  const uint8_t* u8 = static_cast<const uint8_t*>(image);
  if (dtype == 1) {
    uint8_t* q = w8 + L.u8_off;
    const int64_t n = (int64_t)B * H * W;
    if (const int rc = OG_LAUNCH(sift_quantize_kernel, sift_grid(n), 256, 0, st, static_cast<const float*>(image), n, q)) return rc;
    u8 = q;
  }
  OG_CUDA(cudaMemsetAsync(loc_count, 0, 2 * B * sizeof(int), st));
  // createInitialImage: x2 INTER_LINEAR, then the blur from the assumed 0.5 (x2: 1.0) to sigma
  float* up = P.oct[0].dog;                            // scratch until the first DoG level is written
  if (const int rc = OG_LAUNCH(sift_upsample_kernel, sift_grid((int64_t)B * L.h[0] * L.w[0]), 256, 0, st, u8, B, H, W, up)) return rc;
  const float sig_diff = sqrtf(std::max(SIFT_SIGMA * SIFT_SIGMA - 0.5f * 0.5f * 4, 0.01f));
  if (const int rc = sift_blur(up, B, L.h[0], L.w[0], (double)sig_diff, tmp, P.oct[0].gauss, nullptr, st)) return rc;
  // buildGaussianPyramid / buildDoGPyramid
  double sig[SIFT_GAUSS];
  sig[0] = SIFT_SIGMA_D;
  const double k = pow(2., 1. / SIFT_LAYERS);
  for (int i = 1; i < SIFT_GAUSS; ++i) {
    const double prev = pow(k, (double)(i - 1)) * SIFT_SIGMA_D, total = prev * k;
    sig[i] = sqrt(total * total - prev * prev);
  }
  for (int o = 0; o < L.nO; ++o) {
    const SiftOctave& oc = P.oct[o];
    const int64_t plane = (int64_t)B * oc.h * oc.w;
    if (o > 0) {
      const SiftOctave& pv = P.oct[o - 1];
      if (const int rc = OG_LAUNCH(sift_downsample_kernel, sift_grid(plane), 256, 0, st, pv.gauss + (int64_t)SIFT_LAYERS * B * pv.h * pv.w,
                                   B, pv.h, pv.w, oc.gauss)) return rc;
    }
    for (int i = 1; i < SIFT_GAUSS; ++i)
      if (const int rc = sift_blur(oc.gauss + (i - 1) * plane, B, oc.h, oc.w, sig[i], tmp, oc.gauss + i * plane, oc.dog + (i - 1) * plane, st)) return rc;
  }
  // findScaleSpaceExtrema: extrema + interpolation, orientations
  for (int o = 0; o < L.nO; ++o) {
    const SiftOctave& oc = P.oct[o];
    const int64_t n = (int64_t)B * SIFT_LAYERS * std::max(oc.h - 2 * SIFT_BORDER, 0) * std::max(oc.w - 2 * SIFT_BORDER, 0);
    if (n == 0) continue;
    if (const int rc = OG_LAUNCH(sift_extrema_kernel, sift_grid(n), 256, 0, st, oc, B, o, loc, L.loc_cap, loc_count)) return rc;
  }
  if (const int rc = OG_LAUNCH(sift_orientation_kernel, dim3(cdiv(L.loc_cap, 8), B), 256, 0, st, P, (const SiftLoc*)loc, L.loc_cap,
                               (const int*)loc_count, kp_raw, oct_raw, cap, kp_count)) return rc;
  // KeyPointsFilter::removeDuplicatedSorted
  return OG_LAUNCH(sift_sort_unique_kernel, B, 1024, 0, st, (const float*)kp_raw, (const int*)oct_raw, (const int*)kp_count,
                   (const int*)loc_count, L.loc_cap, cap, L.n2max, work, kp, octave, count, overflow);
}
int og_sift_detect(const void* image, int dtype, int B, int H, int W, int cap, void* ws, int64_t ws_bytes, float* kp, int* octave,
                   int* count, void* stream) {
  return sift_detect(image, dtype, B, H, W, cap, ws, ws_bytes, kp, octave, count, nullptr, stream);
}
int og_sift_detect_padded(const void* image, int dtype, int B, int H, int W, int cap, void* ws, int64_t ws_bytes, float* kp, int* octave,
                          int* count, int* overflow, void* stream) {
  OG_CHECK_ARG(overflow, "sift_detect_padded: null pointer");
  return sift_detect(image, dtype, B, H, W, cap, ws, ws_bytes, kp, octave, count, overflow, stream);
}
int64_t og_sift_select_workspace_bytes(int B, int cap) {
  if (B <= 0 || B > 65535 || cap <= 0 || cap > (1 << 24)) return fail(OG_EINVAL, "sift_select_workspace_bytes: bad sizes");
  return (int64_t)B * 4 * pow2_ceil(cap) * 4;
}
int og_sift_select(const float* kp, const int* count, int B, int cap, float nms_radius, int max_keypoints, void* work, int64_t work_bytes,
                   int* sel, int* n_sel, void* stream) {
  OG_CHECK_ARG(kp && count && work && sel && n_sel, "sift_select: null pointer");
  const int64_t need = og_sift_select_workspace_bytes(B, cap);
  if (need < 0) return (int)need;
  OG_CHECK_ARG(work_bytes >= need, "sift_select: workspace of %lld bytes, %lld needed", (long long)work_bytes, (long long)need);
  OG_CHECK_ARG(nms_radius == nms_radius, "sift_select: nms_radius is NaN");
  return OG_LAUNCH(sift_select_kernel, B, 1024, 0, (cudaStream_t)stream, kp, count, cap, nms_radius, max_keypoints, pow2_ceil(cap),
                   static_cast<int*>(work), sel, n_sel);
}
int og_sift_describe(const void* ws, int B, int H, int W, int cap, const float* kp, const int* octave, const int* sel, const int* n_sel,
                     int out_cap, int max_n, int rootsift, float* lafs, float* scores, float* desc, float* raw_desc, void* stream) {
  OG_CHECK_ARG(ws && kp && octave && sel && n_sel && lafs && scores && desc, "sift_describe: null pointer");
  OG_CHECK_ARG(out_cap > 0 && max_n >= 0, "sift_describe: bad sizes");
  SiftLayout L;
  if (og_sift_workspace_bytes(B, H, W, cap) < 0) return OG_EINVAL;
  sift_layout(B, H, W, cap, L);
  if (max_n == 0) return OG_OK;
  const SiftPyramid P = sift_pyramid(static_cast<unsigned char*>(const_cast<void*>(ws)), L, B);
  return OG_LAUNCH(sift_describe_kernel, dim3(cdiv(std::min(max_n, out_cap), 8), B), 256, 0, (cudaStream_t)stream, P, kp, octave, cap, sel, n_sel,
                   out_cap, rootsift, lafs, scores, desc, raw_desc);
}
int og_sift_rootsift_laf(const float* kp, const float* raw_desc, int64_t N, int rootsift, float* lafs, float* scores, float* desc, void* stream) {
  OG_CHECK_ARG(kp && raw_desc && lafs && scores && desc && N >= 0, "sift_rootsift_laf: bad arguments");
  if (N == 0) return OG_OK;
  return OG_LAUNCH(sift_rootsift_laf_kernel, (unsigned)((N + 7) / 8), 256, 0, (cudaStream_t)stream, kp, raw_desc, N, rootsift, lafs, scores, desc);
}
int og_sift_fast_atan2(const float* y, const float* x, int64_t n, int fused, float* out, void* stream) {
  OG_CHECK_ARG(y && x && out && n >= 0, "sift_fast_atan2: bad arguments");
  if (n == 0) return OG_OK;
  return OG_LAUNCH(sift_fast_atan2_kernel, sift_grid(n), 256, 0, (cudaStream_t)stream, y, x, n, fused, out);
}

// ---- local features -> matcher inputs, matches -> compact list (csrc/features.cuh) ----
int og_prepare_features(const float* lafs, const float* responses, int64_t R, int method, int log_response, float* kpts, float* side,
                        void* stream) {
  OG_CHECK_ARG(method >= OG_LAF_NONE && method <= OG_LAF_AFFINE, "prepare_features: unknown LAF method %d", method);
  const int width = (responses ? 1 : 0) + laf_side_dim(method);
  OG_CHECK_ARG(lafs && R >= 0 && (width == 0 || side), "prepare_features: bad arguments");
  if (R == 0 || (width == 0 && !kpts)) return OG_OK;
  return OG_LAUNCH(prepare_features_kernel, (unsigned)((R + 255) / 256), 256, 0, (cudaStream_t)stream, lafs, responses, R, method,
                   log_response, kpts, side, width);
}
int og_match_compact(const int64_t* matches0, const float* mscores0, const float* lafs0, const float* lafs1, int B, int n, int m,
                     int64_t* pair, int64_t* ij, float* confidence, float* out_lafs0, float* out_lafs1, float* out_kpts0,
                     float* out_kpts1, int64_t* total, void* stream) {
  OG_CHECK_ARG(matches0 && mscores0 && lafs0 && lafs1 && pair && ij && confidence && out_lafs0 && out_lafs1 && out_kpts0 && out_kpts1 && total,
               "match_compact: null pointer");
  OG_CHECK_ARG(B > 0 && n > 0 && m > 0 && (int64_t)B * n <= INT32_MAX - 1024, "match_compact: bad sizes");
  return OG_LAUNCH(match_compact_kernel, 1, 1024, 0, (cudaStream_t)stream, matches0, mscores0, lafs0, lafs1, B * n, n, m, pair, ij, confidence,
                   out_lafs0, out_lafs1, out_kpts0, out_kpts1, total);
}

// ---- kornia SIFT front-end (csrc/kornia_sift.cuh) ----
static int ks_check_sizes(int B, int H, int W, int k, KsLayout& L, const char* who) {
  if (B <= 0 || B > 65535 || H <= 0 || W <= 0 || k <= 0) return fail(OG_EINVAL, "%s: bad sizes", who);
  if (k > KS_MAX_FEATURES) return fail(OG_EUNSUPPORTED, "%s: num_features %d above %d", who, k, KS_MAX_FEATURES);
  if (min(H, W) < 2 || (int64_t)5 * 4 * H * W > 0xffffffffLL) return fail(OG_EUNSUPPORTED, "%s: a %d x %d image is not supported", who, H, W);
  if (!ks_layout(B, H, W, k, L)) return fail(OG_EUNSUPPORTED, "%s: a %d x %d image has more than %d octaves", who, H, W, KS_MAX_OCTAVES);
  return OG_OK;
}
int64_t og_ksift_workspace_bytes(int B, int H, int W, int num_features) {
  KsLayout L;
  if (const int rc = ks_check_sizes(B, H, W, num_features, L, "ksift_workspace_bytes")) return rc;
  return L.bytes;
}
int og_ksift_workspace_layout(int B, int H, int W, int num_features, int64_t* out, int n) {
  OG_CHECK_ARG(out, "ksift_workspace_layout: null pointer");
  KsLayout L;
  if (const int rc = ks_check_sizes(B, H, W, num_features, L, "ksift_workspace_layout")) return rc;
  const int need = 1 + 5 * L.nO + 1 + 3 * L.np + 1;
  OG_CHECK_ARG(n >= need, "ksift_workspace_layout: %d entries, %d needed", n, need);
  int i = 0;
  out[i++] = L.nO;
  for (int o = 0; o < L.nO; ++o) {
    out[i++] = L.oct[o].h; out[i++] = L.oct[o].w;
    out[i++] = 4 * L.oct[o].gauss; out[i++] = 4 * L.oct[o].dog; out[i++] = 4 * L.oct[o].resp;
  }
  out[i++] = L.np;
  for (int l = 0; l < L.np; ++l) { out[i++] = L.ph[l]; out[i++] = L.pw[l]; out[i++] = l == 0 ? -1 : 4 * L.pyr[l]; }
  out[i++] = L.bytes;
  return i;
}
static int ks_blur(float* ws_f, const KsLayout& L, int B, int h, int w, const float* src, int64_t src_stride, double sigma,
                   float* dst, int64_t dst_stride, cudaStream_t st) {
  KsTaps t;
  const int k = ks_kernel_size(sigma, h, w);
  if (k > KS_MAX_TAPS) return fail(OG_EUNSUPPORTED, "ksift: sigma %g needs more than %d taps", sigma, KS_MAX_TAPS);
  ks_gaussian_taps(k, sigma, t);
  const int64_t plane = (int64_t)h * w;
  float* tmp = ws_f + L.tmp;
  if (const int rc = OG_LAUNCH(ks_blur_kernel, sift_grid(B * plane), 256, 0, st, src, src_stride, B, h, w, t, 0, tmp, plane)) return rc;
  return OG_LAUNCH(ks_blur_kernel, sift_grid(B * plane), 256, 0, st, (const float*)tmp, plane, B, h, w, t, 1, dst, dst_stride);
}
static int ks_args(void* ws, int64_t ws_bytes, int B, int H, int W, int k, KsLayout& L, const char* who) {
  OG_CHECK_ARG(ws, "%s: null workspace", who);
  if (const int rc = ks_check_sizes(B, H, W, k, L, who)) return rc;
  OG_CHECK_ARG(ws_bytes >= L.bytes, "%s: workspace of %lld bytes, %lld needed", who, (long long)ws_bytes, (long long)L.bytes);
  return OG_OK;
}
// The Gaussian levels 1 .. 5 of octave o (and its level 0, the previous octave's level 3 at [::2, ::2], for o > 0)
static int ks_octave_levels(float* f, const KsLayout& L, int B, int o, cudaStream_t st) {
  const KsOctave& oc = L.oct[o];
  const int64_t plane = (int64_t)oc.h * oc.w;
  float* g = f + oc.gauss;
  if (o > 0) {
    const KsOctave& pv = L.oct[o - 1];
    if (const int rc = OG_LAUNCH(ks_subsample_kernel, sift_grid(B * plane), 256, 0, st, (const float*)(f + pv.gauss), B, pv.h, pv.w,
                                 oc.h, oc.w, g)) return rc;
  }
  const double step = std::pow(2.0, 1.0 / 3.0);
  double cur = 1.6;
  for (int l = 1; l < KS_LEVELS; ++l) {
    const double sigma = cur * std::sqrt(step * step - 1.0);
    if (const int rc = ks_blur(f, L, B, oc.h, oc.w, g + (l - 1) * plane, KS_LEVELS * plane, sigma, g + l * plane, KS_LEVELS * plane, st)) return rc;
    cur *= step;
  }
  return OG_OK;
}
int og_ksift_pyramid(const float* image, int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, void* stream) {
  KsLayout L;
  if (const int rc = ks_args(ws, ws_bytes, B, H, W, num_features, L, "ksift_pyramid")) return rc;
  OG_CHECK_ARG(image, "ksift_pyramid: null image");
  cudaStream_t st = (cudaStream_t)stream;
  float* f = static_cast<float*>(ws);
  const KsOctave& o0 = L.oct[0];
  const int64_t p0 = (int64_t)o0.h * o0.w;
  float* g0 = f + o0.gauss;
  if (const int rc = OG_LAUNCH(ks_upsample_kernel, sift_grid(B * p0), 256, 0, st, image, B, H, W, g0)) return rc;
  // the upsampled image has sigma 1.0; the first level is blurred to 1.6
  if (const int rc = ks_blur(f, L, B, o0.h, o0.w, g0, KS_LEVELS * p0, std::max(std::sqrt(1.6 * 1.6 - 1.0), 0.01), g0, KS_LEVELS * p0, st)) return rc;
  for (int o = 0; o < L.nO; ++o) {
    const KsOctave& oc = L.oct[o];
    const int64_t plane = (int64_t)oc.h * oc.w;
    if (const int rc = ks_octave_levels(f, L, B, o, st)) return rc;
    if (const int rc = OG_LAUNCH(ks_dog_kernel, sift_grid(B * KS_DOG * plane), 256, 0, st, (const float*)(f + oc.gauss), B, (int)plane,
                                 f + oc.dog)) return rc;
  }
  return OG_OK;
}
// The detector on the volumes in ws: the responses of every voxel (SIFT: extrema of DoG and -DoG; GFTT: maxima of levels 0 .. 4),
// the exact per-octave top-k, the border test and the global top-k
static int ks_detect(const KsLayout& L, int B, int H, int W, bool gftt, void* ws, float* lafs, float* resp, int* count, cudaStream_t st) {
  float* f = static_cast<float*>(ws);
  char* c = static_cast<char*>(ws);
  const int segs = B * L.nO, k = L.k;
  KsSel* sel = reinterpret_cast<KsSel*>(c + L.state);
  unsigned int* hist = reinterpret_cast<unsigned int*>(c + L.hist);
  unsigned long long* cand = reinterpret_cast<unsigned long long*>(c + L.cand);
  int* cnt = reinterpret_cast<int*>(c + L.count);
  if (const int rc = OG_LAUNCH(ks_select_init_kernel, cdiv(segs, 128), 128, 0, st, L, segs, sel, hist, cnt)) return rc;
  for (int o = 0; o < L.nO; ++o) {
    const KsOctave& oc = L.oct[o];
    const int64_t per = (int64_t)KS_DOG * oc.h * oc.w;
    if (gftt) {
      if (const int rc = OG_LAUNCH(kg_response_kernel, sift_grid(B * per), 256, 0, st, (const float*)(f + oc.dog), B, oc.h, oc.w, f + oc.resp)) return rc;
    } else {
      if (const int rc = OG_LAUNCH(ks_response_kernel, sift_grid(B * per), 256, 0, st, (const float*)(f + oc.dog), B, oc.h, oc.w, f + oc.resp)) return rc;
    }
    const dim3 grid((unsigned)std::min<int64_t>(cdiv((int)std::min<int64_t>(per, INT_MAX), 2048), 512), B);
    for (int pass = 0; pass < 8; ++pass) {
      if (const int rc = OG_LAUNCH(ks_hist_kernel, grid, 256, 0, st, (const float*)(f + oc.resp), per, o, L.nO, (const KsSel*)sel, hist)) return rc;
      if (const int rc = OG_LAUNCH(ks_pick_kernel, cdiv(B, 128), 128, 0, st, B, o, L.nO, sel, hist)) return rc;
    }
    if (const int rc = OG_LAUNCH(ks_compact_kernel, grid, 256, 0, st, (const float*)(f + oc.resp), per, o, L.nO, (const KsSel*)sel, k, cand, cnt)) return rc;
  }
  const size_t smem = (size_t)pow2_ceil(k) * 8;
  KsCand* list = reinterpret_cast<KsCand*>(c + L.list);
  KsCand* scratch = reinterpret_cast<KsCand*>(c + L.scratch);
  if (gftt) {
    if (const int rc = smem_opt_in<ks_octave_list_kernel<512, 1>>((int)((size_t)KS_MAX_FEATURES * 8))) return rc;
    if (const int rc = OG_LAUNCH((ks_octave_list_kernel<512, 1>), segs, 512, smem, st, (const float*)f, L, B, H, W, (const int*)cnt, scratch,
                                 list, (const unsigned long long*)cand)) return rc;
  } else {
    if (const int rc = smem_opt_in<ks_octave_list_kernel<512>>((int)((size_t)KS_MAX_FEATURES * 8))) return rc;
    if (const int rc = OG_LAUNCH(ks_octave_list_kernel<512>, segs, 512, smem, st, (const float*)f, L, B, H, W, (const int*)cnt, scratch, list,
                                 (const unsigned long long*)cand)) return rc;
  }
  if (const int rc = OG_LAUNCH(ks_merge_kernel, dim3(cdiv(k, 256), L.nO, B), 256, 0, st, (const KsCand*)list, (const int*)cnt, L.nO, k,
                               lafs, resp, count)) return rc;
  return OG_LAUNCH(ks_det_tail_kernel, dim3(cdiv(k, 256), B), 256, 0, st, (const int*)count, k, lafs, resp);
}
int og_ksift_detect(int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, float* lafs, float* resp, int* count, void* stream) {
  KsLayout L;
  if (const int rc = ks_args(ws, ws_bytes, B, H, W, num_features, L, "ksift_detect")) return rc;
  OG_CHECK_ARG(lafs && resp && count, "ksift_detect: null pointer");
  return ks_detect(L, B, H, W, false, ws, lafs, resp, count, (cudaStream_t)stream);
}
int64_t og_ksift_select_workspace_bytes(int B, int cap) {
  if (B <= 0 || B > 65535 || cap <= 0 || cap > KS_MAX_FEATURES) return fail(OG_EINVAL, "ksift_select_workspace_bytes: bad sizes");
  return align_up((int64_t)B * cap, 256) + (int64_t)B * 4;
}
int og_ksift_select(const float* lafs, const float* resp, const int* count, int B, int H, int W, int cap, int nms, int nms_diameter,
                    int max_keypoints, int min_stack, void* work, int64_t work_bytes, int* sel, int* n_sel, void* stream) {
  OG_CHECK_ARG(lafs && resp && count && work && sel && n_sel, "ksift_select: null pointer");
  OG_CHECK_ARG(H > 0 && W > 0, "ksift_select: bad image size");
  OG_CHECK_ARG(!nms || (nms_diameter > 0 && nms_diameter % 2 == 1), "ksift_select: nms_diameter must be odd and positive, got %d", nms_diameter);
  const int64_t need = og_ksift_select_workspace_bytes(B, cap);
  if (need < 0) return (int)need;
  OG_CHECK_ARG(work_bytes >= need, "ksift_select: workspace of %lld bytes, %lld needed", (long long)work_bytes, (long long)need);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* keep = static_cast<unsigned char*>(work);
  int* kept = reinterpret_cast<int*>(keep + align_up((int64_t)B * cap, 256));
  const size_t smem = (size_t)pow2_ceil(cap) * 16;
  if (const int rc = smem_opt_in<ks_nms_kernel<1024>>((int)((size_t)KS_MAX_FEATURES * 16))) return rc;
  if (const int rc = OG_LAUNCH(ks_nms_kernel<1024>, B, 1024, smem, st, lafs, resp, count, cap, H, W, nms_diameter / 2, nms, keep, kept)) return rc;
  return OG_LAUNCH(ks_select_kernel, B, 1024, 0, st, (const unsigned char*)keep, (const int*)kept, B, cap, max_keypoints, min_stack, sel, n_sel);
}
// kornia's pyrdown patch pyramid: level 0 is the image, level l > 0 in ws
static KsPyr ks_patch_pyramid(const KsLayout& L, const float* image, void* ws) {
  float* f = static_cast<float*>(ws);
  KsPyr P{};
  P.n = L.np;
  for (int l = 0; l < L.np; ++l) {
    P.h[l] = L.ph[l]; P.w[l] = L.pw[l];
    P.p[l] = l == 0 ? image : f + L.pyr[l];
    if (l > 0 && (L.ph[l] < 1 || L.pw[l] < 1)) { P.n = l; break; }
  }
  return P;
}
static int ks_build_patch_pyramid(const KsLayout& L, int B, const KsPyr& P, void* ws, cudaStream_t st) {
  float* f = static_cast<float*>(ws);
  for (int l = 1; l < P.n; ++l) {
    const int64_t m = (int64_t)B * L.ph[l - 1] * L.pw[l - 1];
    if (const int rc = OG_LAUNCH(ks_pyrdown_blur_kernel, sift_grid(m), 256, 0, st, P.p[l - 1], B, L.ph[l - 1], L.pw[l - 1], f + L.tmp)) return rc;
    if (const int rc = OG_LAUNCH(ks_pyrdown_resize_kernel, sift_grid((int64_t)B * L.ph[l] * L.pw[l]), 256, 0, st, (const float*)(f + L.tmp), B,
                                 L.ph[l - 1], L.pw[l - 1], L.ph[l], L.pw[l], f + L.pyr[l])) return rc;
  }
  return OG_OK;
}
int og_ksift_describe(const float* image, int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, const float* lafs,
                      const float* resp, int cap, const int* sel, const int* n, int out_cap, int upright, int rootsift, float* lafs_out,
                      float* scores, float* desc, float* angle, void* stream) {
  KsLayout L;
  if (const int rc = ks_args(ws, ws_bytes, B, H, W, num_features, L, "ksift_describe")) return rc;
  OG_CHECK_ARG(image && lafs && resp && n && lafs_out && scores && desc, "ksift_describe: null pointer");
  OG_CHECK_ARG(cap > 0 && out_cap > 0 && out_cap <= 65535, "ksift_describe: bad capacities");
  cudaStream_t st = (cudaStream_t)stream;
  const KsPyr P = ks_patch_pyramid(L, image, ws);
  if (const int rc = ks_build_patch_pyramid(L, B, P, ws, st)) return rc;
  KsDescConst* K = reinterpret_cast<KsDescConst*>(static_cast<char*>(ws) + L.consts);
  if (const int rc = OG_LAUNCH(ks_desc_const_kernel, 1, 32, 0, st, K)) return rc;
  return OG_LAUNCH(ks_describe_kernel<256>, dim3(out_cap, B), 256, 0, st, P, H, W, lafs, resp, cap, sel, n, out_cap, upright, rootsift,
                   (const KsDescConst*)K, lafs_out, scores, desc, angle);
}

// ---- kornia GFTT / AffNet / HardNet front-end (csrc/kornia_gftt.cuh) ----
static int kg_check_sizes(int B, int H, int W, int k, KsLayout& L, const char* who) {
  if (B <= 0 || B > 65535 || H <= 0 || W <= 0 || k <= 0) return fail(OG_EINVAL, "%s: bad sizes", who);
  if (k > KS_MAX_FEATURES) return fail(OG_EUNSUPPORTED, "%s: num_features %d above %d", who, k, KS_MAX_FEATURES);
  if (min(H, W) < 2 || (int64_t)6 * H * W > 0xffffffffLL) return fail(OG_EUNSUPPORTED, "%s: a %d x %d image is not supported", who, H, W);
  if (!ks_layout(B, H, W, k, L, false, KS_LEVELS)) return fail(OG_EUNSUPPORTED, "%s: a %d x %d image has more than %d octaves", who, H, W, KS_MAX_OCTAVES);
  return OG_OK;
}
static int kg_args(const void* ws, int64_t ws_bytes, int B, int H, int W, int k, KsLayout& L, const char* who) {
  OG_CHECK_ARG(ws, "%s: null workspace", who);
  if (const int rc = kg_check_sizes(B, H, W, k, L, who)) return rc;
  OG_CHECK_ARG(ws_bytes >= L.bytes, "%s: workspace of %lld bytes, %lld needed", who, (long long)ws_bytes, (long long)L.bytes);
  return OG_OK;
}
int64_t og_kgftt_workspace_bytes(int B, int H, int W, int num_features) {
  KsLayout L;
  if (const int rc = kg_check_sizes(B, H, W, num_features, L, "kgftt_workspace_bytes")) return rc;
  return L.bytes;
}
int og_kgftt_workspace_layout(int B, int H, int W, int num_features, int64_t* out, int n) {
  OG_CHECK_ARG(out, "kgftt_workspace_layout: null pointer");
  KsLayout L;
  if (const int rc = kg_check_sizes(B, H, W, num_features, L, "kgftt_workspace_layout")) return rc;
  const int need = 1 + 5 * L.nO + 1 + 3 * L.np + 1;
  OG_CHECK_ARG(n >= need, "kgftt_workspace_layout: %d entries, %d needed", n, need);
  int i = 0;
  out[i++] = L.nO;
  for (int o = 0; o < L.nO; ++o) {
    out[i++] = L.oct[o].h; out[i++] = L.oct[o].w;
    out[i++] = 4 * L.oct[o].gauss; out[i++] = 4 * L.oct[o].dog; out[i++] = 4 * L.oct[o].resp;
  }
  out[i++] = L.np;
  for (int l = 0; l < L.np; ++l) { out[i++] = L.ph[l]; out[i++] = L.pw[l]; out[i++] = l == 0 ? -1 : 4 * L.pyr[l]; }
  out[i++] = L.bytes;
  return i;
}
int og_kgftt_pyramid(const float* image, int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, void* stream) {
  KsLayout L;
  if (const int rc = kg_args(ws, ws_bytes, B, H, W, num_features, L, "kgftt_pyramid")) return rc;
  OG_CHECK_ARG(image, "kgftt_pyramid: null image");
  cudaStream_t st = (cudaStream_t)stream;
  float* f = static_cast<float*>(ws);
  const KsOctave& o0 = L.oct[0];
  const int64_t p0 = (int64_t)o0.h * o0.w;
  // the input has sigma 0.5; the first level is blurred to 1.6
  if (const int rc = ks_blur(f, L, B, H, W, image, p0, std::max(std::sqrt(1.6 * 1.6 - 0.25), 0.01), f + o0.gauss, KS_LEVELS * p0, st)) return rc;
  KgGftt g;
  KsTaps t;
  ks_gaussian_taps(7, 1.0, t);
  for (int i = 0; i < 7; ++i) for (int j = 0; j < 7; ++j) g.k2[i * 7 + j] = t.k[i] * t.k[j];
  const double step = std::pow(2.0, 1.0 / 3.0);
  double cur = 1.6;
  for (int l = 0; l < KS_LEVELS; ++l) { g.s4[l] = powf((float)cur, 4.f); cur *= step; }     // the level sigmas, float32, to the 4th
  for (int o = 0; o < L.nO; ++o) {
    const KsOctave& oc = L.oct[o];
    if (const int rc = ks_octave_levels(f, L, B, o, st)) return rc;
    const dim3 grid(cdiv(oc.w, KG_TILE), cdiv(oc.h, KG_TILE), B * KS_LEVELS);
    if (const int rc = OG_LAUNCH(kg_gftt_kernel, grid, dim3(KG_TILE, KG_TILE), 0, st, (const float*)(f + oc.gauss), oc.h, oc.w, g, f + oc.dog)) return rc;
  }
  const KsPyr P = ks_patch_pyramid(L, image, ws);
  if (const int rc = ks_build_patch_pyramid(L, B, P, ws, st)) return rc;
  return OG_LAUNCH(ks_desc_const_kernel, 1, 32, 0, st, reinterpret_cast<KsDescConst*>(static_cast<char*>(ws) + L.consts));
}
int og_kgftt_detect(int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, float* lafs, float* resp, int* count, void* stream) {
  KsLayout L;
  if (const int rc = kg_args(ws, ws_bytes, B, H, W, num_features, L, "kgftt_detect")) return rc;
  OG_CHECK_ARG(lafs && resp && count, "kgftt_detect: null pointer");
  return ks_detect(L, B, H, W, true, ws, lafs, resp, count, (cudaStream_t)stream);
}
static int kg_rows_args(const float* image, const float* lafs, const int* n, int cap, int out_cap, int B, int r0, int rows, const char* who) {
  OG_CHECK_ARG(image && lafs && n, "%s: null pointer", who);
  OG_CHECK_ARG(cap > 0 && out_cap > 0 && rows >= 0 && r0 >= 0 && (int64_t)r0 + rows <= (int64_t)B * out_cap && (int64_t)B * out_cap <= INT32_MAX,
               "%s: bad rows [%d, %d + %d) of %d x %d", who, r0, r0, rows, B, out_cap);
  return OG_OK;
}
int og_kgftt_affnet_patches(const float* image, int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, const float* lafs, int cap,
                            const int* sel, const int* n, int out_cap, int r0, int rows, float* patches, void* stream) {
  KsLayout L;
  if (const int rc = kg_args(ws, ws_bytes, B, H, W, num_features, L, "kgftt_affnet_patches")) return rc;
  if (const int rc = kg_rows_args(image, lafs, n, cap, out_cap, B, r0, rows, "kgftt_affnet_patches")) return rc;
  OG_CHECK_ARG(patches, "kgftt_affnet_patches: null pointer");
  if (rows == 0) return OG_OK;
  return OG_LAUNCH(kg_affnet_patch_kernel<256>, rows, 256, 0, (cudaStream_t)stream, ks_patch_pyramid(L, image, ws), H, W, lafs, cap, sel, n, out_cap,
                   r0, patches);
}
int og_kgftt_frames(const float* image, int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, const float* lafs, const float* resp,
                    int cap, const int* sel, const int* n, int out_cap, int r0, int rows, const float* xy, int upright, float* lafs_out,
                    float* scores, float* angle, float* patches, void* stream) {
  KsLayout L;
  if (const int rc = kg_args(ws, ws_bytes, B, H, W, num_features, L, "kgftt_frames")) return rc;
  if (const int rc = kg_rows_args(image, lafs, n, cap, out_cap, B, r0, rows, "kgftt_frames")) return rc;
  OG_CHECK_ARG(resp && xy && lafs_out && scores && patches, "kgftt_frames: null pointer");
  if (rows == 0) return OG_OK;
  const KsDescConst* K = reinterpret_cast<const KsDescConst*>(static_cast<const char*>(ws) + L.consts);
  return OG_LAUNCH(kg_frame_kernel<256>, rows, 256, 0, (cudaStream_t)stream, ks_patch_pyramid(L, image, ws), H, W, lafs, resp, cap, sel, n,
                   out_cap, r0, xy, upright, K, lafs_out, scores, angle, patches);
}
int og_kgftt_im2col3x3_s2(const float* x, int B, int H, int W, int C, float* out, void* stream) {
  OG_CHECK_ARG(x && out && B > 0 && H > 0 && W > 0 && C > 0, "kgftt_im2col3x3_s2: bad arguments");
  const int64_t cols = (int64_t)B * ((H + 1) / 2) * ((W + 1) / 2) * 9 * ((C % 4 == 0) ? C / 4 : C);
  return OG_LAUNCH(kg_im2col3x3_s2_kernel, sp_grid(cols), 256, 0, (cudaStream_t)stream, x, B, H, W, C, out);
}
int og_kgftt_desc_finish(float* desc, int B, int out_cap, const int* n, void* stream) {
  OG_CHECK_ARG(desc && n && B > 0 && out_cap > 0, "kgftt_desc_finish: bad arguments");
  const int64_t rows = (int64_t)B * out_cap;
  return OG_LAUNCH(kg_desc_finish_kernel, (unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream, desc, B, out_cap, n);
}

int og_keypoint_counts(const int* count, int B, int cap, int max_keypoints, int K, int* n_out, int* mode, int* overflow, void* stream) {
  OG_CHECK_ARG(count && n_out && overflow, "keypoint_counts: null pointer");
  OG_CHECK_ARG(B > 0 && cap > 0 && K > 0, "keypoint_counts: bad sizes");
  return OG_LAUNCH(keypoint_counts_kernel, cdiv(B, 256), 256, 0, (cudaStream_t)stream, count, B, cap, max_keypoints, K, n_out, mode,
                   overflow);
}
int og_mask_empty_pairs(const int* len0, const int* len1, int B, int n, int m, int64_t* matches0, float* mscores0, int64_t* matches1,
                        float* mscores1, void* stream) {
  OG_CHECK_ARG(len0 && len1 && matches0 && mscores0 && matches1 && mscores1, "mask_empty_pairs: null pointer");
  OG_CHECK_ARG(B > 0 && n > 0 && m > 0, "mask_empty_pairs: bad sizes");
  const int64_t total = (int64_t)B * ((int64_t)n + m);
  return OG_LAUNCH(mask_empty_pairs_kernel, eltwise_grid(total), 256, 0, (cudaStream_t)stream, len0, len1, B, n, m, matches0, mscores0,
                   matches1, mscores1);
}

// ---- homography-pretraining pairs (csrc/homography.cuh) ----
int og_homography_pairs(const uint8_t* rgb, int B, int H, int W, int offset, const int32_t* warp_offset, float* image0, float* image1,
                        float* H_true, void* stream) {
  OG_CHECK_ARG(rgb && warp_offset && image0 && image1 && H_true, "homography_pairs: null pointer");
  OG_CHECK_ARG(B >= 1 && B <= 65535, "homography_pairs: B = %d must be in [1, 65535]", B);
  OG_CHECK_ARG(offset >= 1 && H > 0 && W > 0 && 2 * (int64_t)offset < (H < W ? H : W),
               "homography_pairs: offset %d must be >= 1 with 2 offset < min(H, W) = min(%d, %d)", offset, H, W);
  OG_CHECK_ARG((int64_t)HG_ROWS * W <= INT32_MAX, "homography_pairs: W = %d too large", W);
  const int h = H - 2 * offset;
  return OG_LAUNCH(homography_pairs_kernel, dim3(cdiv(h, HG_ROWS), B), HG_THREADS, 0, (cudaStream_t)stream, rgb, H, W, offset,
                   hg_block_width(H, W), warp_offset, image0, image1, H_true);
}

// ---- optimiser step (csrc/optim.cuh) ----
int64_t og_optim_state_bytes(void) { return (int64_t)sizeof(og_optim_state); }
int64_t og_optim_workspace_bytes(int nseg) { return nseg > 0 ? optim_workspace_bytes(nseg) : -1; }

static bool unit_beta(double b) { return b >= 0.0 && b < 1.0; }

static int clip_adam_impl(const og_optim_segment* segments, int nseg, int64_t ntiles, double beta1, double beta2, double eps,
                          double max_norm, double lr_gamma, og_optim_state* state, void* workspace, int64_t workspace_bytes,
                          const int* skip, void* stream) {
  OG_CHECK_ARG(segments && state && workspace, "clip_adam_step: null pointer");
  OG_CHECK_ARG(nseg > 0 && ntiles > 0, "clip_adam_step: nseg = %d and ntiles = %lld must be positive", nseg, (long long)ntiles);
  OG_CHECK_ARG(max_norm > 0.0, "clip_adam_step: max_norm = %g must be positive", max_norm);
  OG_CHECK_ARG(unit_beta(beta1) && unit_beta(beta2), "clip_adam_step: betas (%g, %g) must lie in [0, 1)", beta1, beta2);
  OG_CHECK_ARG(eps >= 0.0, "clip_adam_step: eps = %g must be >= 0", eps);
  OG_CHECK_ARG(lr_gamma > 0.0, "clip_adam_step: lr_gamma = %g must be positive", lr_gamma);
  if (workspace_bytes < optim_workspace_bytes(nseg)) return fail(OG_EWORKSPACE, "clip_adam_step: workspace too small");
  const OptHyper h = {beta1, beta2, eps, max_norm, lr_gamma};
  return optim_step_launch(segments, nseg, ntiles, h, state, workspace, skip, (cudaStream_t)stream);
}

int og_clip_adam_step(const og_optim_segment* segments, int nseg, int64_t ntiles, double beta1, double beta2, double eps,
                      double max_norm, double lr_gamma, og_optim_state* state, void* workspace, int64_t workspace_bytes, void* stream) {
  return clip_adam_impl(segments, nseg, ntiles, beta1, beta2, eps, max_norm, lr_gamma, state, workspace, workspace_bytes, nullptr, stream);
}

int og_clip_adam_step_guarded(const og_optim_segment* segments, int nseg, int64_t ntiles, double beta1, double beta2, double eps,
                              double max_norm, double lr_gamma, og_optim_state* state, void* workspace, int64_t workspace_bytes,
                              const int* skip, void* stream) {
  return clip_adam_impl(segments, nseg, ntiles, beta1, beta2, eps, max_norm, lr_gamma, state, workspace, workspace_bytes, skip, stream);
}

int og_adam_schedule(int64_t nsteps, double lr, double lr_gamma, double beta1, double beta2, double* lr_out, float* step_size,
                     float* bc2_sqrt, void* stream) {
  OG_CHECK_ARG(lr_out && step_size && bc2_sqrt, "adam_schedule: null pointer");
  OG_CHECK_ARG(nsteps > 0 && nsteps < (1 << 24), "adam_schedule: nsteps = %lld must lie in [1, 2^24)", (long long)nsteps);
  OG_CHECK_ARG(unit_beta(beta1) && unit_beta(beta2) && lr_gamma > 0.0, "adam_schedule: bad hyper-parameters");
  cudaStream_t st = (cudaStream_t)stream;
  if (const int rc = OG_LAUNCH(adam_lr_chain_kernel, 1, 1, 0, st, nsteps, lr, lr_gamma, lr_out)) return rc;
  return OG_LAUNCH(adam_scalars_kernel, (unsigned)std::min<int64_t>((nsteps + 255) / 256, 4096), 256, 0, st, nsteps, (const double*)lr_out,
                   beta1, beta2, step_size, bc2_sqrt);
}

static int forward_impl(const og_config* cfg, const float* Wp, const float* Whi, const float* Wlo, const __half* W16h,
                        const __half* W16l, const float* meta16, int B, int n, int m,
                         const float* kpts0,
                         const float* kpts1, const float* side0, const float* side1, const float* desc0,
                         const float* desc1, const float* img_wh, float* ctx0, float* ctx1, float* scores,
                         int64_t* matches0, float* mscores0, int64_t* matches1, float* mscores1, void* workspace,
                         int64_t workspace_bytes, void* stream_, const int* lens = nullptr, const float* pair_wh = nullptr) {
  int rc = check_config(cfg);
  if (rc != OG_OK) return rc;
  // padded batch (lens, pair_wh): pair b owns rows [0, lens[b]) of image 0 and [0, lens[B + b]) of image 1 of the capacity n, m
  const bool padded = lens != nullptr;
  OG_CHECK_ARG(Wp && kpts0 && kpts1 && desc0 && desc1 && (padded ? pair_wh != nullptr : img_wh != nullptr) && scores && workspace,
               "forward: null pointer");
  OG_CHECK_ARG(cfg->side_info_size == 0 || (side0 && side1), "forward: side info missing");
  OG_CHECK_ARG(B > 0 && n > 0 && m > 0, "forward: batch, n, m must be positive");
  OG_CHECK_ARG(cfg->precision == OG_PREC_FP32 || (Whi && Wlo), "forward: the tensor-core modes need packed_hi / packed_lo");
  OG_CHECK_ARG(cfg->precision != OG_PREC_FP16X3 || (W16h && W16l && meta16), "forward: OG_PREC_FP16X3 needs the fp16 weight split (og_pack_f16)");
  const bool tcp = (cfg->precision != OG_PREC_FP32) && cfg->descriptor_dim >= 32;   // K >= 32 for the tensor-core tiles
  // fp16 hi/lo form of the GNN (projections, attention, message MLP): head_dim 64, d a multiple of 64; everything else
  // (Dh = 32, the final projection, the score GEMM) runs the tf32 hi/lo form - same accuracy class
  const bool f16p = tcp && cfg->precision == OG_PREC_FP16X3 && cfg->descriptor_dim % 64 == 0 &&
                    cfg->descriptor_dim / cfg->num_heads == 64;
  auto WH = [&](int64_t off) { return tcp ? Whi + off : nullptr; };
  auto WL = [&](int64_t off) { return tcp ? Wlo + off : nullptr; };
  OG_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "forward: workspace must be 256-byte aligned");
  cudaStream_t st = (cudaStream_t)stream_;
  const int prec = cfg->precision == OG_PREC_FP16X3 ? OG_PREC_TF32X3 : cfg->precision;     // what the non-f16 launches run as
  const Layout L = make_layout(cfg);
  Workspace w;
  rc = plan_workspace(cfg, B, n, m, workspace, &w, padded);
  if (rc != OG_OK) return rc;
  if (workspace_bytes < w.total) return fail(OG_EWORKSPACE, "forward: workspace %lld < %lld bytes",
                                             (long long)workspace_bytes, (long long)w.total);
  launch_counter() = 0;
  const int d = cfg->descriptor_dim, H = cfg->num_heads, dh = d / H, S = cfg->side_info_size;
  const int R0 = B * n, R1 = B * m, R = R0 + R1;
  float* x0 = w.x; float* x1 = w.x + (int64_t)R0 * d;

  // ---- keypoint encoder (positional_encoding.py:16-19) + descriptors (superglue.py:52-55) ----
  // A padded batch zeroes its padding rows here and reads its descriptors from a copy with them zeroed: from the first kernel on
  // every row is finite (the fp16 amax slots see every row, and a masked key with a NaN value would poison P.V: 0 * NaN = NaN).
  const float* dsc0 = desc0;
  const float* dsc1 = desc1;
  // each image's (W - 1, H - 1), or in a padded batch its lengths and per-pair sizes (the kernel reads these when len is set)
  const float wm0 = padded ? 0.f : img_wh[0] - 1.f, hm0 = padded ? 0.f : img_wh[1] - 1.f;
  const float wm1 = padded ? 0.f : img_wh[2] - 1.f, hm1 = padded ? 0.f : img_wh[3] - 1.f;
  const int* len0 = padded ? lens : nullptr;
  const int* len1 = padded ? lens + B : nullptr;
  const float* wh0 = padded ? pair_wh : nullptr;
  const float* wh1 = padded ? pair_wh + 2 : nullptr;
  if ((rc = OG_LAUNCH(kenc_input_kernel, cdiv(R0, 256), 256, 0, st, kpts0, side0, R0, S, wm0, hm0, n, len0, wh0, w.in0)) != OG_OK) return rc;
  if ((rc = OG_LAUNCH(kenc_input_kernel, cdiv(R1, 256), 256, 0, st, kpts1, side1, R1, S, wm1, hm1, m, len1, wh1,
                      w.in0 + (int64_t)R0 * (2 + S))) != OG_OK)
    return rc;
  if (padded) {
    float* d1m = w.desc + (int64_t)R0 * d;
    if ((rc = OG_LAUNCH(mask_padded_rows_kernel, eltwise_grid((int64_t)R0 * d), 256, 0, st, desc0, (int64_t)R0, n, d, lens, w.desc)) != OG_OK)
      return rc;
    if ((rc = OG_LAUNCH(mask_padded_rows_kernel, eltwise_grid((int64_t)R1 * d), 256, 0, st, desc1, (int64_t)R1, m, d, lens + B, d1m)) != OG_OK)
      return rc;
    dsc0 = w.desc; dsc1 = d1m;
  }
  {
    const float* cur = w.in0;
    float* bufs[2] = {w.h0, w.h1};
    const int nl = (int)L.kenc_sizes.size() - 1;
    for (int i = 0; i < nl; ++i) {
      const int kin = L.kenc_sizes[i], kout = L.kenc_sizes[i + 1];
      if (i < nl - 1) {
        og_linear_args a = lin(cur, kin, kin, Wp + L.kenc_w[i], Wp + L.kenc_b[i], R, kout, bufs[i & 1], kout);
        a.relu = 1;
        if ((rc = linear_dispatch(a, OG_PREC_FP32, st)) != OG_OK) return rc;
        cur = bufs[i & 1];
      } else {                        // last layer: + local descriptors, per image (separate user tensors)
        og_linear_args a = lin(cur, kin, kin, Wp + L.kenc_w[i], Wp + L.kenc_b[i], R0, kout, x0, d);
        if (!cfg->no_descriptors) { a.R = dsc0; a.ldr = d; }           // superglue.py:45-55
        if ((rc = linear_dispatch(a, OG_PREC_FP32, st)) != OG_OK) return rc;
        og_linear_args b = lin(cur + (int64_t)R0 * kin, kin, kin, Wp + L.kenc_w[i], Wp + L.kenc_b[i], R1, kout, x1, d);
        if (!cfg->no_descriptors) { b.R = dsc1; b.ldr = d; }
        if ((rc = linear_dispatch(b, OG_PREC_FP32, st)) != OG_OK) return rc;
      }
    }
  }

  // ---- attentional GNN (attention_gnn.py:58-93) ----
  // One layer schedule for three forms of attention.  They differ in how the projection writes Q / K / V, how attention reads
  // them and how the GEMMs get their operand scales:
  //   FP32: Q | K | V interleaved in qkv [R, 3d], exact attention on CUDA cores (fp32, d < 32 or head_dim not in {32, 64});
  //   TF32: Q fp32, K split hi/lo keypoint-major and V split hi/lo channel-major (= the reference's own [B, d, M] layout), which
  //         are exactly the operand layouts csrc/attention_sm90.cuh stages with TMA;
  //   F16:  the same layouts in fp16 hi/lo, every operand scaled from device slots (below).
  enum class Att { FP32, TF32, F16 };
  const Att att = f16p ? Att::F16 : (tcp && (dh == 32 || dh == 64)) ? Att::TF32 : Att::FP32;
  // `count` sequences of `len` keypoints from row `row0` on, of image `img` (2: both)
  struct Seqs { int row0, len, count, img; int rows() const { return len * count; } };
  const Seqs img[2] = {{0, n, B, 0}, {R0, m, B, 1}};
  const Seqs all{0, R, 1, 2};                                // every row at once, for the GEMMs only
  // Granularity of a self layer with n != m, which each form keeps as it is:
  //   FP32 projects both images in one launch (its GEMMs see rows, not sequences);
  //   F16 runs the MLP per image, so that each image keeps its own amax slot: one shared slot would change the fp16 scales.
  const bool project_all_rows = att == Att::FP32, mlp_per_image = att == Att::F16;
  // V^T of image 0 (or of both images when n == m) at offset 0 with rows ldn apart, V^T of image 1 after it with rows ldm apart
  auto vt_ld = [&](const Seqs& kv) { return kv.row0 == 0 ? w.ldn : w.ldm; };
  auto vt_off = [&](const Seqs& kv) { return kv.row0 == 0 ? 0 : (int64_t)B * d * w.ldn; };

  // F16: every activation tensor has a device slot with its tracked amax (fp32 tensors) or the scale it was written with (fp16
  // K / V^T); a consumer derives its operand scale from the producers' slots, so no scale ever passes through the host.
  int nslot = 0;
  auto new_slot = [&]() -> float* { return w.slots + (nslot < w.nslots - 1 ? nslot++ : w.nslots - 1); };
  float* sx[2] = {};                                         // amax slots of the current x0 / x1
  struct SeqSlots { float *q, *k, *v, *o; } ss[2] = {};      // of the last projection of image 0 (or both images) / image 1
  auto xslot = [&](const Seqs& g, int i) { return g.img == 2 ? sx[i] : i == 0 ? sx[g.img] : nullptr; };   // amax of x's rows g
  __half* kh16 = reinterpret_cast<__half*>(w.khi); __half* kl16 = reinterpret_cast<__half*>(w.klo);
  __half* vth16 = reinterpret_cast<__half*>(w.vthi); __half* vtl16 = reinterpret_cast<__half*>(w.vtlo);
  if (att == Att::F16) {
    OG_CUDA(cudaMemsetAsync(w.slots, 0, (size_t)w.nslots * 4, st));
    sx[0] = sx[1] = new_slot();
    const int64_t nx = (int64_t)R * d;
    if ((rc = OG_LAUNCH(amax_kernel, (unsigned)std::min<int64_t>((nx + 2047) / 2048, 1184), 256, 0, st, w.x, nx, sx[0])) != OG_OK) return rc;
  }
  // the fp16 GEMM of `a`: operand amax slots am0 .. am2 (of A, A2) and the meta of weight t of layer l (og_pack_f16)
  auto args16 = [&](const og_linear_args& a, float* am0, float* am1, float* am2, int l, int t) {
    F16LinearArgs g = gemm_args<F16LinearArgs>(a);
    g.amax_in[0] = am0; g.amax_in[1] = am1; g.amax_in[2] = am2; g.w_meta = meta16 + ((int64_t)l * 5 + t) * 4;
    return g;
  };
  auto run16 = [&](const og_linear_args& a, const F16LinearArgs& g, int64_t woff) {
    return linear_sm90_run(a, g, W16h + woff, W16l + woff, "forward", "a layer is not tileable by the fp16 GEMM", st);
  };
  // F16 with d % 128 == 0 (every shipped config): the projections that share their input run as ONE launch over the stacked
  // weights (one run of kinds): Q | K | V in a self layer (same keypoints), K | V in a cross layer (+ Q on its own).
  const bool fuse_qkv = fuse_qkv_mode() && d % tcf::BN == 0;

  // Q of the rows q, K and V of the rows kv (q itself in a self layer)
  auto project = [&](int l, const Seqs& q, const Seqs& kv) -> int {
    const bool self = q.row0 == kv.row0;
    const int64_t wq = L.qkv_w[l], bq = L.qkv_b[l], dd = (int64_t)d * d;
    const float* xq = w.x + (int64_t)q.row0 * d;
    const float* xkv = w.x + (int64_t)kv.row0 * d;
    int r;
    if (att == Att::FP32) {       // qkv[g, c0 : c0 + nout] = x[g] . Wqkv[c0 : c0 + nout]^T + b: Q | K | V in one launch in a self layer
      auto part = [&](const Seqs& g, int c0, int nout) {
        og_linear_args a = lin(w.x + (int64_t)g.row0 * d, d, d, Wp + wq + (int64_t)c0 * d, Wp + bq + c0, g.rows(), nout,
                               w.qkv + (int64_t)g.row0 * 3 * d + c0, 3 * d);
        return linear_dispatch(a, prec, st, WH(wq + (int64_t)c0 * d), WL(wq + (int64_t)c0 * d));
      };
      if (self) return part(q, 0, 3 * d);
      return (r = part(q, 0, d)) != OG_OK ? r : part(kv, d, 2 * d);
    }
    const int64_t ldv = vt_ld(kv), voff = vt_off(kv);
    if (att == Att::TF32) {
      og_linear_args aq = lin(xq, d, d, Wp + wq, Wp + bq, q.rows(), d, w.q + (int64_t)q.row0 * d, d);
      og_linear_args ak = lin(xkv, d, d, Wp + wq + dd, Wp + bq + d, kv.rows(), d, nullptr, d);
      og_linear_args av = lin(xkv, d, d, Wp + wq + 2 * dd, Wp + bq + 2 * d, kv.len, d, nullptr, d);   // V^T batched per sequence
      av.batch = kv.count; av.strideA = (int64_t)kv.len * d; av.ldyt = ldv; av.strideYt = (int64_t)d * ldv;
      SplitOut sk, sv;
      sk.Yhi = w.khi + (int64_t)kv.row0 * d; sk.Ylo = w.klo + (int64_t)kv.row0 * d;
      sv.Ythi = w.vthi + voff; sv.Ytlo = w.vtlo + voff;
      if ((r = linear_dispatch(aq, prec, st, WH(wq), WL(wq))) != OG_OK) return r;
      if ((r = linear_dispatch(ak, prec, st, WH(wq + dd), WL(wq + dd), sk)) != OG_OK) return r;
      return linear_dispatch(av, prec, st, WH(wq + 2 * dd), WL(wq + 2 * dd), sv);
    }
    SeqSlots& s = ss[q.img == 1];
    s = {new_slot(), new_slot(), new_slot(), new_slot()};
    // Q of the rows q, K and V^T of the rows kv, each with its batch stride per sequence
    const F16Out out[F16_KINDS] = {
        {w.q + (int64_t)q.row0 * d, nullptr, nullptr, d, (int64_t)q.len * d, nullptr},
        {nullptr, kh16 + (int64_t)kv.row0 * d, kl16 + (int64_t)kv.row0 * d, d, (int64_t)kv.len * d, s.k},
        {nullptr, vth16 + voff, vtl16 + voff, ldv, (int64_t)d * ldv, s.v}};
    // The kinds k0 .. k0 + nk - 1 of the rows g in one launch over their stacked weights.  A run that writes V^T is batched per
    // sequence, as V^T's layout is; Q or K alone is one batch item of all rows of g.
    auto run = [&](const Seqs& g, int k0, int nk) {
      const bool per_seq = k0 + nk == F16_KINDS;
      og_linear_args a = lin(w.x + (int64_t)g.row0 * d, d, d, Wp + wq + k0 * dd, Wp + bq + k0 * d, per_seq ? g.len : g.rows(), nk * d, nullptr, d);
      if (per_seq) { a.batch = g.count; a.strideA = (int64_t)g.len * d; }
      F16LinearArgs ga = args16(a, xslot(g, 0), xslot(g, 1), nullptr, l, k0);
      std::copy(out, out + F16_KINDS, ga.out);
      ga.kind0 = k0; ga.nkinds = nk; ga.kind_cols = d; ga.amax_out = s.q;
      return run16(a, ga, wq + k0 * dd);
    };
    if (fuse_qkv && self) return run(q, F16_Y, 3);
    if (fuse_qkv) return (r = run(q, F16_Y, 1)) != OG_OK ? r : run(kv, F16_K, 2);
    for (int k = F16_Y; k < F16_KINDS; ++k)
      if ((r = run(k == F16_Y ? q : kv, k, 1)) != OG_OK) return r;
    return OG_OK;
  };

  // o[q] = attention of the queries q over the keys / values kv.  A padded batch gives each sequence its keys' length: lens is
  // n_0 .. n_{B-1}, m_0 .. m_{B-1}, so image 0 (or both images as 2B sequences) starts at lens, image 1 at lens + B.
  auto attend = [&](const Seqs& q, const Seqs& kv) -> int {
    const float scale = (float)pow((double)dh, -0.5);
    const int* klen = padded ? lens + (kv.img == 1 ? B : 0) : nullptr;
    if (att == Att::FP32) {
      const float* qkv_q = w.qkv + (int64_t)q.row0 * 3 * d;
      const float* qkv_kv = w.qkv + (int64_t)kv.row0 * 3 * d;
      AttnArgs a{qkv_q, 3 * d, (int64_t)q.len * 3 * d, qkv_kv + d, 3 * d, (int64_t)kv.len * 3 * d, qkv_kv + 2 * d, 3 * d,
                 (int64_t)kv.len * 3 * d, w.o + (int64_t)q.row0 * d, d, (int64_t)q.len * d, q.count, q.len, kv.len, H, scale, klen};
      return attention_simt_launch(a, dh, st);
    }
    const int64_t ldv = vt_ld(kv), voff = vt_off(kv), k0 = (int64_t)kv.row0 * d;
    TcAttnArgs a{w.q + (int64_t)q.row0 * d, d, (int64_t)q.len * d, w.o + (int64_t)q.row0 * d, d, (int64_t)q.len * d,
                 q.count, q.len, kv.len, H, d, scale, klen};
    if (att == Att::TF32) return attention_tc_launch(a, w.khi + k0, w.klo + k0, d, w.vthi + voff, w.vtlo + voff, ldv, dh, st);
    const SeqSlots& s = ss[q.img == 1];
    return attention_f16_launch(a, F16AttnScales{s.q, s.k, s.v, s.o, 0}, kh16 + k0, kl16 + k0, d, vth16 + voff, vtl16 + voff, ldv, dh, st);
  };

  // x[g] <- x[g] + W2 . relu(W1 . [x[g] ; o[g]] + b1) + b2     (out_proj and BN folded into W1 / W2 on the host)
  auto mlp = [&](int l, const Seqs& g) -> int {
    float* xr = w.x + (int64_t)g.row0 * d;
    float* hr = w.hid + (int64_t)g.row0 * 2 * d;
    og_linear_args a1 = lin(xr, d, d, Wp + L.fc1_w[l], Wp + L.fc1_b[l], g.rows(), 2 * d, hr, 2 * d);
    a1.A2 = w.o + (int64_t)g.row0 * d; a1.lda2 = d; a1.k2 = d; a1.ldw = 2 * d; a1.relu = 1;
    og_linear_args a2 = lin(hr, 2 * d, 2 * d, Wp + L.fc2_w[l], Wp + L.fc2_b[l], g.rows(), d, xr, d);
    a2.R = xr; a2.ldr = d;
    int r;
    if (att != Att::F16) {
      if ((r = linear_dispatch(a1, prec, st, WH(L.fc1_w[l]), WL(L.fc1_w[l]))) != OG_OK) return r;
      return linear_dispatch(a2, prec, st, WH(L.fc2_w[l]), WL(L.fc2_w[l]));
    }
    // F16: [x ; o] scaled by the slots of x and of the attention output, the hidden layer by the amax fc1 tracked
    float* sh = new_slot();
    float* sn = new_slot();
    F16LinearArgs g1 = args16(a1, xslot(g, 0), xslot(g, 1), ss[g.img == 1].o, l, 3);
    g1.amax_out = sh;
    if ((r = run16(a1, g1, L.fc1_w[l])) != OG_OK) return r;
    F16LinearArgs g2 = args16(a2, sh, nullptr, nullptr, l, 4);
    g2.amax_out = sn;
    if ((r = run16(a2, g2, L.fc2_w[l])) != OG_OK) return r;
    if (g.img != 1) sx[0] = sn;
    if (g.img != 0) sx[1] = sn;
    return OG_OK;
  };

  for (int l = 0; l < cfg->num_layers; ++l) {
    if (l % 2 == 1) {                                      // cross: SEQUENTIAL (attention_gnn.py:74-77)
      for (int i = 0; i < 2; ++i) {                        // image 1's K / V come from the UPDATED image 0
        if ((rc = project(l, img[i], img[1 - i])) != OG_OK) return rc;
        if ((rc = attend(img[i], img[1 - i])) != OG_OK) return rc;
        if ((rc = mlp(l, img[i])) != OG_OK) return rc;
      }
    } else if (n == m) {                                   // self: both images as one batch of 2B sequences
      const Seqs both{0, n, 2 * B, 2};
      if ((rc = project(l, both, both)) != OG_OK) return rc;
      if ((rc = attend(both, both)) != OG_OK) return rc;
      if ((rc = mlp(l, both)) != OG_OK) return rc;
    } else {                                               // self: one image at a time
      if (project_all_rows && (rc = project(l, all, all)) != OG_OK) return rc;
      for (int i = 0; i < 2; ++i) {
        if (!project_all_rows && (rc = project(l, img[i], img[i])) != OG_OK) return rc;
        if ((rc = attend(img[i], img[i])) != OG_OK) return rc;
      }
      for (int i = 0; i < (mlp_per_image ? 2 : 1); ++i)
        if ((rc = mlp(l, mlp_per_image ? img[i] : all)) != OG_OK) return rc;
    }
  }

  // ---- final projection + residual mix (superglue.py:58-62); channel-first context descriptors ----
  for (int img = 0; img < 2; ++img) {
    const int nn = img ? m : n;
    float* xr = img ? x1 : x0;
    float* gr = w.g + (img ? (int64_t)R0 * d : 0);
    og_linear_args a = lin(xr, d, d, Wp + L.proj_w, Wp + L.proj_b, nn, d, gr, d);
    a.batch = B; a.strideA = (int64_t)nn * d; a.strideY = (int64_t)nn * d;
    a.R = img ? dsc1 : dsc0; a.ldr = d; a.strideR = (int64_t)nn * d; a.rscale = Wp + L.proj_rmix;
    float* ctx = img ? ctx1 : ctx0;
    if (ctx) { a.Yt = ctx; a.ldyt = nn; a.strideYt = (int64_t)d * nn; }
    SplitOut so;
    if (tcp && img == 1) { so.Yhi = w.ghi; so.Ylo = w.glo; }      // image-1 descriptors are the score GEMM's B operand
    if ((rc = linear_dispatch(a, prec, st, WH(L.proj_w), WL(L.proj_w), so)) != OG_OK) return rc;
    if (padded && ctx &&
        (rc = OG_LAUNCH(zero_padded_cols_kernel, eltwise_grid((int64_t)B * d * nn), 256, 0, st, ctx, B, d, nn, lens + (img ? B : 0))) != OG_OK)
      return rc;
  }
  // ---- score matrix (superglue.py:64,80-86): S = g0^T g1 * d^-0.5, written with padded rows ----
  {
    og_linear_args a = lin(w.g, d, d, w.g + (int64_t)R0 * d, nullptr, n, m, w.sbuf, w.lds);
    a.batch = B; a.strideA = (int64_t)n * d; a.strideW = (int64_t)m * d; a.strideY = (int64_t)n * w.lds;
    a.alpha = (float)pow((double)d, -0.5);
    if ((rc = linear_dispatch(a, prec, st, tcp ? w.ghi : nullptr, tcp ? w.glo : nullptr)) != OG_OK) return rc;
  }
  // ---- optimal transport (superglue.py:88-111) + matches (matching_module.py:174-187) ----
  rc = sinkhorn_launch(w.sbuf, w.lds, (int64_t)n * w.lds, Wp + L.dustbin, B, n, m, cfg->sinkhorn_iters,
                       cfg->sinkhorn_reg, scores, w.sink, w.sink_bytes, st, nullptr, nullptr, lens);
  if (rc != OG_OK) return rc;
  if (matches0 || mscores0 || matches1 || mscores1) {
    rc = match_launch(scores, B, n, m, cfg->match_threshold, matches0, mscores0, matches1, mscores1, w.match,
                      w.match_bytes, st, lens);
    if (rc != OG_OK) return rc;
  }
  return OG_OK;
}

int og_superglue_forward(const og_config* cfg, const float* Wp, const float* Whi, const float* Wlo, int B, int n, int m,
                         const float* kpts0, const float* kpts1, const float* side0, const float* side1, const float* desc0,
                         const float* desc1, const float* img_wh, float* ctx0, float* ctx1, float* scores,
                         int64_t* matches0, float* mscores0, int64_t* matches1, float* mscores1, void* workspace,
                         int64_t workspace_bytes, void* stream) {
  if (cfg && cfg->precision == OG_PREC_FP16X3) return fail(OG_EINVAL, "forward: OG_PREC_FP16X3 takes og_superglue_forward_f16");
  return forward_impl(cfg, Wp, Whi, Wlo, nullptr, nullptr, nullptr, B, n, m, kpts0, kpts1, side0, side1, desc0, desc1, img_wh, ctx0, ctx1,
                      scores, matches0, mscores0, matches1, mscores1, workspace, workspace_bytes, stream);
}

int og_superglue_forward_f16(const og_config* cfg, const float* Wp, const float* Whi, const float* Wlo, const void* W16h,
                             const void* W16l, const float* meta16, int B, int n, int m,
                             const float* kpts0, const float* kpts1, const float* side0, const float* side1, const float* desc0,
                             const float* desc1, const float* img_wh, float* ctx0, float* ctx1, float* scores,
                             int64_t* matches0, float* mscores0, int64_t* matches1, float* mscores1, void* workspace,
                             int64_t workspace_bytes, void* stream) {
  return forward_impl(cfg, Wp, Whi, Wlo, static_cast<const __half*>(W16h), static_cast<const __half*>(W16l), meta16, B, n, m, kpts0, kpts1,
                      side0, side1, desc0, desc1, img_wh, ctx0, ctx1, scores, matches0, mscores0, matches1, mscores1, workspace,
                      workspace_bytes, stream);
}

int64_t og_workspace_bytes_padded(const og_config* cfg, int batch, int n, int m) {
  if (check_config(cfg) != OG_OK) return -1;
  if (batch <= 0 || n <= 0 || m <= 0) return fail(OG_EINVAL, "batch, n, m must be positive");
  Workspace w;
  if (plan_workspace(cfg, batch, n, m, nullptr, &w, true) != OG_OK) return -1;
  return w.total;
}

int og_superglue_forward_padded(const og_config* cfg, const float* Wp, const float* Whi, const float* Wlo, const void* W16h,
                                const void* W16l, const float* meta16, int B, int n, int m, const int* lengths,
                                const float* image_sizes, const float* kpts0, const float* kpts1, const float* side0,
                                const float* side1, const float* desc0, const float* desc1, float* ctx0, float* ctx1, float* scores,
                                int64_t* matches0, float* mscores0, int64_t* matches1, float* mscores1, void* workspace,
                                int64_t workspace_bytes, void* stream) {
  OG_CHECK_ARG(lengths && image_sizes, "forward_padded: null lengths / image_sizes");
  OG_CHECK_ARG(B <= 65535, "forward_padded: batch %d > 65535", B);
  return forward_impl(cfg, Wp, Whi, Wlo, static_cast<const __half*>(W16h), static_cast<const __half*>(W16l), meta16, B, n, m, kpts0, kpts1,
                      side0, side1, desc0, desc1, nullptr, ctx0, ctx1, scores, matches0, mscores0, matches1, mscores1, workspace,
                      workspace_bytes, stream, lengths, image_sizes);
}

int64_t og_f16_meta_floats(const og_config* cfg) {
  if (check_config(cfg) != OG_OK) return -1;
  return (int64_t)cfg->num_layers * 5 * 4;
}

int og_weight_split_f16(const float* w, const float* bias, int rows, int cols, void* hi16, void* lo16, float* meta, void* stream) {
  OG_CHECK_ARG(w && hi16 && lo16 && meta && rows > 0 && cols > 0, "weight_split_f16: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  OG_CUDA(cudaMemsetAsync(meta, 0, 4 * sizeof(float), st));
  int rc;
  if ((rc = OG_LAUNCH(weight_meta_kernel, cdiv(rows, 8), 256, 0, st, w, bias, rows, cols, meta)) != OG_OK) return rc;
  const int64_t nel = (int64_t)rows * cols;
  if ((rc = OG_LAUNCH(split_f16_kernel, (unsigned)((nel + 255) / 256), 256, 0, st, w, static_cast<__half*>(hi16), static_cast<__half*>(lo16),
                      nel, meta)) != OG_OK)
    return rc;
  return OG_LAUNCH(finish_meta_kernel, 1, 1, 0, st, meta);
}

int og_pack_f16(const og_config* cfg, const float* Wp, void* hi16, void* lo16, float* meta, void* stream) {
  int rc = check_config(cfg);
  if (rc != OG_OK) return rc;
  OG_CHECK_ARG(Wp && hi16 && lo16 && meta, "pack_f16: null pointer");
  const Layout L = make_layout(cfg);
  const int64_t d = cfg->descriptor_dim;
  __half* h = static_cast<__half*>(hi16); __half* lo = static_cast<__half*>(lo16);
  for (int l = 0; l < cfg->num_layers; ++l) {
    struct T { int64_t woff, boff; int rows, cols; } ts[5] = {
      {L.qkv_w[l], L.qkv_b[l], (int)d, (int)d}, {L.qkv_w[l] + d * d, L.qkv_b[l] + d, (int)d, (int)d},
      {L.qkv_w[l] + 2 * d * d, L.qkv_b[l] + 2 * d, (int)d, (int)d},
      {L.fc1_w[l], L.fc1_b[l], (int)(2 * d), (int)(2 * d)}, {L.fc2_w[l], L.fc2_b[l], (int)d, (int)(2 * d)}};
    for (int t = 0; t < 5; ++t)
      if ((rc = og_weight_split_f16(Wp + ts[t].woff, Wp + ts[t].boff, ts[t].rows, ts[t].cols, h + ts[t].woff, lo + ts[t].woff,
                                    meta + ((int64_t)l * 5 + t) * 4, stream)) != OG_OK) return rc;
  }
  return OG_OK;
}

int og_amax(const float* x, int64_t n, float* slot, void* stream) {
  OG_CHECK_ARG(x && slot && n > 0, "amax: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  OG_CUDA(cudaMemsetAsync(slot, 0, sizeof(float), st));
  return OG_LAUNCH(amax_kernel, (unsigned)std::min<int64_t>((n + 2047) / 2048, 1184), 256, 0, st, x, n, slot);
}

int og_linear_f16_fwd(const og_linear_args* a, const void* Wh16, const void* Wl16, const float* w_meta, const float* a_amax,
                      float* amax_out, float* scale_out, void* Yh, void* Yl, void* Yth, void* Ytl, int swap_halves, void* stream) {
  OG_CHECK_ARG(a && a->A && Wh16 && Wl16 && w_meta && a_amax, "linear_f16: null pointer");
  OG_CHECK_ARG(a->rows > 0 && a->nout > 0 && a->batch > 0 && a->k1 > 0 && a->k2 >= 0, "linear_f16: bad sizes");
  OG_CHECK_ARG(!a->rscale && !a->Yt, "linear_f16: rscale / fp32 transposed outputs are not part of the fp16 form");
  F16LinearArgs g = gemm_args<F16LinearArgs>(*a);
  g.out[F16_K] = {nullptr, static_cast<__half*>(Yh), static_cast<__half*>(Yl), a->ldy, a->strideY, scale_out};
  g.out[F16_VT] = {nullptr, static_cast<__half*>(Yth), static_cast<__half*>(Ytl), a->ldyt, a->strideYt, scale_out};
  g.kind0 = a->Y ? F16_Y : Yh ? F16_K : F16_VT;
  g.nkinds = (a->Y != nullptr) + (Yh != nullptr) + (Yth != nullptr) == 1;   // no output or several: an empty run, not tileable
  g.amax_in[0] = a_amax; g.w_meta = w_meta; g.amax_out = amax_out; g.swap_halves = swap_halves;
  return linear_sm90_run(*a, g, static_cast<const __half*>(Wh16), static_cast<const __half*>(Wl16), "linear_f16",
                         "needs K >= 64, 16-byte aligned rows, exactly one output kind (Y | Yh,Yl | Yth,Ytl)", (cudaStream_t)stream);
}

static int attention_f16_fwd_impl(const float* q, int64_t ldq, int64_t strideq, const float* q_amax, const void* khi, const void* klo,
                                  int64_t ldk, const float* k_scale, const void* vthi, const void* vtlo, int64_t ldvt,
                                  const float* v_scale, float* out, int64_t ldo, int64_t strideo, float* out_amax, int batch, int nq,
                                  int nk, int num_heads, int head_dim, int swap_halves, const int* klen, void* stream) {
  OG_CHECK_ARG(q && q_amax && khi && klo && k_scale && vthi && vtlo && v_scale && out, "attention_f16: null pointer");
  OG_CHECK_ARG(batch > 0 && nq > 0 && nk > 0 && num_heads > 0, "attention_f16: bad sizes");
  if (!attention_f16_eligible(head_dim, ldq, ldk, ldvt, ldo))
    return fail(OG_EUNSUPPORTED, "attention_f16: head_dim 64 and 16-byte aligned rows required");
  TcAttnArgs a{q, ldq, strideq, out, ldo, strideo, batch, nq, nk, num_heads, num_heads * head_dim, (float)pow((double)head_dim, -0.5),
               klen};
  F16AttnScales sc{q_amax, k_scale, v_scale, out_amax, swap_halves};
  return attention_f16_launch(a, sc, static_cast<const __half*>(khi), static_cast<const __half*>(klo), ldk,
                                static_cast<const __half*>(vthi), static_cast<const __half*>(vtlo), ldvt, head_dim, (cudaStream_t)stream);
}

int og_attention_f16_fwd(const float* q, int64_t ldq, int64_t strideq, const float* q_amax, const void* khi, const void* klo,
                         int64_t ldk, const float* k_scale, const void* vthi, const void* vtlo, int64_t ldvt, const float* v_scale,
                         float* out, int64_t ldo, int64_t strideo, float* out_amax, int batch, int nq, int nk, int num_heads,
                         int head_dim, int swap_halves, void* stream) {
  return attention_f16_fwd_impl(q, ldq, strideq, q_amax, khi, klo, ldk, k_scale, vthi, vtlo, ldvt, v_scale, out, ldo, strideo, out_amax,
                                batch, nq, nk, num_heads, head_dim, swap_halves, nullptr, stream);
}

int og_attention_f16_fwd_padded(const float* q, int64_t ldq, int64_t strideq, const float* q_amax, const void* khi, const void* klo,
                                int64_t ldk, const float* k_scale, const void* vthi, const void* vtlo, int64_t ldvt,
                                const float* v_scale, float* out, int64_t ldo, int64_t strideo, float* out_amax, int batch, int nq,
                                int nk, int num_heads, int head_dim, const int* key_lengths, void* stream) {
  OG_CHECK_ARG(key_lengths, "attention_f16_padded: null key_lengths");
  return attention_f16_fwd_impl(q, ldq, strideq, q_amax, khi, klo, ldk, k_scale, vthi, vtlo, ldvt, v_scale, out, ldo, strideo, out_amax,
                                batch, nq, nk, num_heads, head_dim, 0, key_lengths, stream);
}

}  // extern "C"
