/*
 * openglue_b200.h  --  C ABI of libopenglue_b200.so
 *
 * An H100 (sm_90a) implementation of ONE path of ucuapps/OpenGlue: the SuperGlue-style
 * matching core (reference models/superglue/*, models/matching_module.py:149-187).
 * The reference is pure Python and has no FFI; these entry points are what a binding for
 * this path binds (ctypes today, see INTEGRATION.md).  Each function names the reference
 * code it replaces (paths relative to the reference repo root).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to caller-owned memory unless the name ends in
 *     `_host`; nothing is allocated, freed or synchronised behind the caller's back;
 *   - every call enqueues work on `stream` and returns immediately;
 *   - return value: OG_OK (0) or a negative og_status; og_last_error() gives a
 *     thread-local message for the last failure on the calling thread;
 *   - activations are keypoint-major: row = keypoint, `d` channels contiguous.  The
 *     reference's channel-first [B, d, n] tensors appear only at the Python-visible
 *     outputs (context descriptors);
 *   - all floating-point data is IEEE fp32; match indices are int64 (torch.int64).
 */
#ifndef OPENGLUE_B200_H_
#define OPENGLUE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OG_VERSION 100          /* major*10000 + minor*100 + patch */

typedef enum og_status {
  OG_OK = 0,
  OG_EINVAL = -1,               /* bad argument (null pointer, non-positive size, misalignment) */
  OG_EUNSUPPORTED = -2,         /* shape / option outside what the kernels cover               */
  OG_ECUDA = -3,                /* a CUDA runtime call failed (message has the CUDA error)      */
  OG_EWORKSPACE = -4            /* workspace too small                                          */
} og_status;

/* arithmetic of the GEMM-shaped contractions */
typedef enum og_precision {
  OG_PREC_FP32 = 0,             /* CUDA-core FFMA, fp32 accumulate: the exact mode                 */
  OG_PREC_TF32X3 = 1,           /* wgmma tf32, hi/lo operand split, 3 products, fp32 accum     */
  OG_PREC_FP16X3 = 2            /* wgmma f16: fp16 hi/lo operands with power-of-two tensor scales (same 10-bit
                                   mantissas, twice the MMA rate, half the operand bytes); GNN layers with head_dim 64,
                                   everything else as OG_PREC_TF32X3.  Entry point: og_superglue_forward_f16          */
} og_precision;

#define OG_MAX_HIDDEN 8

/* Mirrors the reference's nested config dict (models/superglue/superglue.py:12-27). */
typedef struct og_config {
  int32_t descriptor_dim;       /* d;  config['descriptor_dim']                                  */
  int32_t num_heads;            /* H;  attention_gnn.num_heads, heads = contiguous channel blocks */
  int32_t num_layers;           /* 2 * attention_gnn.num_stages (even = self, odd = cross)        */
  int32_t side_info_size;       /* S;  positional_encoding.side_info_size                          */
  int32_t num_hidden;           /* len(positional_encoding.hidden_layers_sizes)                    */
  int32_t hidden[OG_MAX_HIDDEN];
  int32_t sinkhorn_iters;       /* otp.num_iters                                                   */
  float   sinkhorn_reg;         /* otp.reg                                                         */
  float   match_threshold;      /* inference.match_threshold (config/config.yaml:40)               */
  int32_t precision;            /* og_precision                                                    */
  int32_t no_descriptors;       /* config.get('no_descriptors'): the GNN starts from the positional encoding alone
                                   (superglue.py:45-49); the residual mix still uses the raw descriptors (:59-62) */
} og_config;

int         og_version(void);
const char* og_last_error(void);
/* Number of SMs / compute capability of the current device (capability cache, read-only). */
int         og_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---------------------------------------------------------------------------------------------
 * Packed weights.  The host side folds eval-mode BatchNorm forward into the following conv
 * (reference models/utils.py:48-58: Conv -> ReLU -> BN), folds `out_proj` into `fc.0`
 * (attention_gnn.py:32,52-55) and sigmoid(mix_coefs) into `linear_proj` (superglue.py:58-62),
 * in float64, and lays the result out as one flat fp32 buffer:
 *
 *   kenc:   for i in 0..num_hidden:  W_i [out_i, in_i],  b_i [out_i]      (in_0 = 2 + S)
 *   layer l (0..num_layers-1):  Wqkv [3d, d], bqkv [3d], W1 [2d, 2d], b1 [2d], W2 [d, 2d], b2 [d]
 *   final:  Wp [d, d], bp [d], rmix [d]   (rmix = 1 - sigmoid(mix_coefs), zeros without residual)
 *   dustbin_score [1]
 *
 * og_packed_offset() returns the float offset of a tensor inside that buffer.
 * ------------------------------------------------------------------------------------------- */
typedef enum og_tensor_id {
  OG_T_KENC_W = 0, OG_T_KENC_B = 1,               /* index = kenc linear layer 0..num_hidden     */
  OG_T_QKV_W = 2, OG_T_QKV_B = 3, OG_T_FC1_W = 4, OG_T_FC1_B = 5, OG_T_FC2_W = 6, OG_T_FC2_B = 7,
                                                  /* index = GNN layer                           */
  OG_T_PROJ_W = 8, OG_T_PROJ_B = 9, OG_T_PROJ_RMIX = 10, OG_T_DUSTBIN = 11   /* index ignored    */
} og_tensor_id;

int64_t og_packed_weight_floats(const og_config* cfg);
/* hi = round-to-nearest tf32(src), lo = round-to-nearest tf32(src - hi): the operand split of the
 * OG_PREC_TF32X3 kernels (x ~= hi + lo to 2^-23 |x|).  Device pointers, n floats each.            */
int og_split_tf32(const float* src, float* hi, float* lo, int64_t n, void* stream);
int64_t og_packed_offset(const og_config* cfg, int tensor_id, int index);

/* ---------------------------------------------------------------------------------------------
 * The whole path.  Replaces SuperGlue.forward (models/superglue/superglue.py:29-72) plus the
 * match extraction of MatchingTrainingModule.forward (models/matching_module.py:174-187) and
 * its reverse direction (inference.py:176-190).
 *
 *   kpts{0,1}  [B, n|m, 2] pixel (x, y);  side{0,1} [B, n|m, S];  desc{0,1} [B, n|m, d]
 *   img_wh     host array {W0, H0, W1, H1}  (superglue.py:35-41, 74-78)
 *   ctx{0,1}   [B, d, n|m]  channel-first context descriptors   (may be NULL)
 *   scores     [B, n+1, m+1] log assignment incl. dustbins
 *   matches0   [B, n] int64 (-1 = no match), mscores0 [B, n];  matches1/mscores1 [B, m] (may be NULL)
 *   packed_hi/lo  tf32 split of packed_weights (og_split_tf32), same offsets; required when
 *              cfg->precision == OG_PREC_TF32X3, ignored (may be NULL) for OG_PREC_FP32
 *   workspace  >= og_workspace_bytes(cfg, B, n, m), 256-byte aligned
 * ------------------------------------------------------------------------------------------- */
int64_t og_workspace_bytes(const og_config* cfg, int batch, int n, int m);

int og_superglue_forward(const og_config* cfg, const float* packed_weights,
                         const float* packed_hi, const float* packed_lo,
                         int batch, int n, int m,
                         const float* kpts0, const float* kpts1,
                         const float* side0, const float* side1,
                         const float* desc0, const float* desc1,
                         const float* img_wh_host,
                         float* ctx0, float* ctx1, float* scores,
                         int64_t* matches0, float* mscores0,
                         int64_t* matches1, float* mscores1,
                         void* workspace, int64_t workspace_bytes, void* stream);

/* OG_PREC_FP16X3 form of the whole path: additionally takes the fp16 hi/lo split of the GNN weights and its per-tensor
 * meta data (og_pack_f16; same element offsets as packed_weights).  packed_hi / packed_lo (tf32) are still required: the
 * final projection and the score GEMM run the tf32 form.                                                            */
int64_t og_f16_meta_floats(const og_config* cfg);
int og_pack_f16(const og_config* cfg, const float* packed_weights, void* hi16, void* lo16, float* meta, void* stream);
int og_superglue_forward_f16(const og_config* cfg, const float* packed_weights,
                             const float* packed_hi, const float* packed_lo,
                             const void* packed_hi16, const void* packed_lo16, const float* meta16,
                             int batch, int n, int m,
                             const float* kpts0, const float* kpts1,
                             const float* side0, const float* side1,
                             const float* desc0, const float* desc1,
                             const float* img_wh_host,
                             float* ctx0, float* ctx1, float* scores,
                             int64_t* matches0, float* mscores0,
                             int64_t* matches1, float* mscores1,
                             void* workspace, int64_t workspace_bytes, void* stream);

/* Padded batch: pairs with their own keypoint counts in one call, in every precision (packed_hi16 / packed_lo16 / meta16 may be
 * NULL unless cfg->precision == OG_PREC_FP16X3).  kpts, side, desc, ctx, scores and matches are laid out as in
 * og_superglue_forward at the capacity n, m; pair b owns rows [0, n_b) of image 0 and [0, m_b) of image 1, and each pair's result
 * is the whole path run on that pair alone.
 *   lengths      device int32 [2B]: n_0 .. n_{B-1}, then m_0 .. m_{B-1}.  Not checked: the kernels clamp each into [1, n] / [1, m].
 *   image_sizes  device float [B, 4]: (W0, H0, W1, H1) of each pair
 *   The padding slots of kpts, side and desc may hold anything (NaN, inf); they influence no valid output.  Outputs past the
 *   lengths: scores -inf (each pair's dustbin row is row n_b, its dustbin column m_b), matches -1, mscores 0, ctx 0.
 *   n <= 65536, batch <= 65535;  workspace >= og_workspace_bytes_padded(cfg, B, n, m), 256-byte aligned.
 *   The first padded call on a device uploads the Sinkhorn's constant tables synchronously: it must not be stream-captured. */
int64_t og_workspace_bytes_padded(const og_config* cfg, int batch, int n, int m);
int og_superglue_forward_padded(const og_config* cfg, const float* packed_weights,
                                const float* packed_hi, const float* packed_lo,
                                const void* packed_hi16, const void* packed_lo16, const float* meta16,
                                int batch, int n, int m, const int* lengths, const float* image_sizes,
                                const float* kpts0, const float* kpts1,
                                const float* side0, const float* side1,
                                const float* desc0, const float* desc1,
                                float* ctx0, float* ctx1, float* scores,
                                int64_t* matches0, float* mscores0,
                                int64_t* matches1, float* mscores1,
                                void* workspace, int64_t workspace_bytes, void* stream);

/* Number of kernels this thread has enqueued since the last og_superglue_forward (or _f16) began, that forward's own
 * launches included.  Every operator entry point adds the kernels it launches.                                      */
int og_last_forward_launches(void);

/* Kernel-variant switches kept for callers of earlier builds.  sm_90 has no CTA-pair MMA, so there is one GEMM and one
 * attention form and both switches are accepted and ignored.                                                         */
int og_set_tuning(int gemm_pair, int attention_pair);
/* fuse_projections = 1 (default; env OG_FUSE_QKV): the Q / K / V projections that share their input run as one launch over the
 * stacked weights (fp16x3 path, descriptor_dim % 128 == 0); 0: one launch per projection.  Bit-identical results (tested).
 * Returns the previous setting; a negative argument only queries.                                                   */
int og_set_fusion(int fuse_projections);

/* ---------------------------------------------------------------------------------------------
 * Operator-level entry points (what the whole-path call is built from; tested one by one
 * against the matching oracle function).
 * ------------------------------------------------------------------------------------------- */

/* Y = epilogue( alpha * [A | A2] . W^T + bias ).   Replaces every Conv1d(k=1) of the path
 * (attention_gnn.py:16-20,24-26,32; models/utils.py:53-57; superglue.py:58) and, batched,
 * calculate_matching_score (superglue.py:80-86).
 *   A  [batch][rows, k1] (lda, strideA)   A2 [batch][rows, k2] or NULL (concat along K)
 *   W  [nout, k1+k2] (ldw; strideW != 0 => one W per batch item)     bias [nout] or NULL
 *   relu: clamp at 0 after bias.   R/rscale: Y += rscale[o] * R[r, o]  (rscale NULL => 1)
 *   Y  [rows, nout] (ldy) and/or Yt [nout, rows] (ldyt) - either may be NULL              */
typedef struct og_linear_args {
  const float* A;  int64_t lda;  int64_t strideA;
  const float* A2; int64_t lda2; int64_t strideA2;
  int32_t k1, k2;
  const float* W;  int64_t ldw;  int64_t strideW;
  const float* bias;
  int32_t rows, nout, batch;
  float   alpha;
  int32_t relu;
  const float* R;  int64_t ldr;  int64_t strideR;
  const float* rscale;
  float* Y;  int64_t ldy;  int64_t strideY;
  float* Yt; int64_t ldyt; int64_t strideYt;
} og_linear_args;
int og_linear_fwd(const og_linear_args* args, int precision, void* stream);
/* Tensor-core (wgmma, 3xTF32) form of og_linear_fwd: W is given pre-split (Whi/Wlo, same layout as
 * args->W, which is ignored).  One kernel (TMA-fed, chunked accumulation folded with round-to-nearest adds)
 * serves every `mode` (0, 1, 2 name kernel forms of earlier builds).  A second operand A2 needs k1 % 32 == 0.
 * Yhi/Ylo (Ythi/Ytlo): optional split copies of Y (Yt) for use as the next kernel's B operand; same ld/stride as Y (Yt). */
int og_linear_tc_fwd(const og_linear_args* args, const float* Whi, const float* Wlo,
                     float* Yhi, float* Ylo, float* Ythi, float* Ytlo, int mode, void* stream);

/* out[b, i, h*Dh + c] = sum_j softmax_j(q_i . k_j * Dh^-0.5) v_j[c]  per head h.
 * Replaces softmax_attention (models/superglue/attention.py:8-19) inside
 * MultiheadAttention.forward (attention_gnn.py:22-32); the N x M probabilities are never
 * materialised.  q [batch][nq, *] row stride ldq; k, v [batch][nk, *]; heads are contiguous
 * channel blocks of width Dh = d / H.  Raw fp32 operands: this entry point always runs the exact
 * fp32 kernel whatever `precision` says; the tensor-core forms take operands that the projection
 * GEMMs have already split (og_attention_tc_fwd, og_attention_f16_fwd).                        */
int og_attention_fwd(const float* q, int64_t ldq, int64_t strideq,
                     const float* k, int64_t ldk, int64_t stridek,
                     const float* v, int64_t ldv, int64_t stridev,
                     float* out, int64_t ldo, int64_t strideo,
                     int batch, int nq, int nk, int num_heads, int head_dim,
                     int precision, void* stream);

/* Tensor-core (wgmma, 3xTF32) form of og_attention_fwd.  Operands as the projection GEMM leaves them:
 *   q fp32 [batch][nq, ldq];  khi/klo tf32-split [batch*nk, ldk] keypoint-major;
 *   vthi/vtlo tf32-split [batch*d, ldvt] channel-major (d = num_heads*head_dim; ldvt >= nk, multiple of 4).
 * head_dim must be 32 or 64.                                                                        */
int og_attention_tc_fwd(const float* q, int64_t ldq, int64_t strideq,
                        const float* khi, const float* klo, int64_t ldk,
                        const float* vthi, const float* vtlo, int64_t ldvt,
                        float* out, int64_t ldo, int64_t strideo,
                        int batch, int nq, int nk, int num_heads, int head_dim, void* stream);

/* fp16 hi/lo ("3xFP16") forms of the two tensor-core operators (OG_PREC_FP16X3).  Operand scales never pass through the
 * host: every tensor has a device scalar - its tracked max |x| (fp32 tensors) or the power-of-two scale it was written
 * with (fp16 tensors).
 *   og_weight_split_f16: w [rows, cols] fp32 (+ bias [rows] or NULL) -> hi16 / lo16 (fp16, same layout) and
 *       meta[4] = {scale, max_n ||w_n||_1, max |bias|, 0}; also the way to split an activation tensor for a test.
 *   og_amax: slot = max |x|.
 *   og_linear_f16_fwd: args as og_linear_fwd (W, rscale, Yt ignored / must be NULL); exactly ONE output kind:
 *       args->Y (fp32, + optional R residual, amax_out) | Yh,Yl (fp16 [rows, nout], ldy) | Yth,Ytl (fp16 [nout, rows], ldyt);
 *       fp16 outputs are written with *scale_out (derived from a bound: |alpha| * a_amax * meta[1] + meta[2]).
 *   og_attention_f16_fwd: q fp32 with its amax; khi/klo fp16 [batch*nk, ldk] with k_scale; vthi/vtlo fp16 [batch*d, ldvt]
 *       with v_scale; head_dim 64.  swap_halves is a layout probe and must be 0.                                      */
int og_weight_split_f16(const float* w, const float* bias, int rows, int cols, void* hi16, void* lo16, float* meta, void* stream);
int og_amax(const float* x, int64_t n, float* slot, void* stream);
int og_linear_f16_fwd(const og_linear_args* args, const void* Wh16, const void* Wl16, const float* w_meta, const float* a_amax,
                      float* amax_out, float* scale_out, void* Yh, void* Yl, void* Yth, void* Ytl, int swap_halves, void* stream);
int og_attention_f16_fwd(const float* q, int64_t ldq, int64_t strideq, const float* q_amax,
                         const void* khi, const void* klo, int64_t ldk, const float* k_scale,
                         const void* vthi, const void* vtlo, int64_t ldvt, const float* v_scale,
                         float* out, int64_t ldo, int64_t strideo, float* out_amax,
                         int batch, int nq, int nk, int num_heads, int head_dim, int swap_halves, void* stream);

/* Padded forms of the three attention operators: sequence b attends to its first key_lengths[b] keys (device int32 [batch],
 * clamped into [1, nk]); the operands keep the layout of the capacity nk.  Every query row is computed. */
int og_attention_fwd_padded(const float* q, int64_t ldq, int64_t strideq,
                            const float* k, int64_t ldk, int64_t stridek,
                            const float* v, int64_t ldv, int64_t stridev,
                            float* out, int64_t ldo, int64_t strideo,
                            int batch, int nq, int nk, int num_heads, int head_dim,
                            const int* key_lengths, void* stream);
int og_attention_tc_fwd_padded(const float* q, int64_t ldq, int64_t strideq,
                               const float* khi, const float* klo, int64_t ldk,
                               const float* vthi, const float* vtlo, int64_t ldvt,
                               float* out, int64_t ldo, int64_t strideo,
                               int batch, int nq, int nk, int num_heads, int head_dim,
                               const int* key_lengths, void* stream);
int og_attention_f16_fwd_padded(const float* q, int64_t ldq, int64_t strideq, const float* q_amax,
                                const void* khi, const void* klo, int64_t ldk, const float* k_scale,
                                const void* vthi, const void* vtlo, int64_t ldvt, const float* v_scale,
                                float* out, int64_t ldo, int64_t strideo, float* out_amax,
                                int batch, int nq, int nk, int num_heads, int head_dim,
                                const int* key_lengths, void* stream);

/* Dustbin-augmented log-domain Sinkhorn.  Replaces SuperGlue.get_matching_probs
 * (superglue.py:88-111) + log_otp_solver (optimal_transport.py:4-28).
 *   S       [B][n, lds]  inner score block (lds >= m, multiple of 4, 16-byte aligned rows)
 *   dustbin device scalar;   scores [B, n+1, m+1]
 *   workspace >= og_sinkhorn_workspace_bytes(B, n, m)                                          */
int64_t og_sinkhorn_workspace_bytes(int batch, int n, int m);
/* resident = 1 (default; env OG_SINK_RESIDENT): the forward Sinkhorn (og_sinkhorn_fwd, og_superglue_forward*) keeps each pair's
 * score rows on chip for all its iterations wherever that plan fits (og_sinkhorn_plan); 0: the streaming kernel, which reads the
 * score matrix from HBM in every iteration.  The column sums are added in another order, so scores agree to the last bits; both
 * forms are deterministic.  The training form always streams.  Returns the previous setting; a negative argument only queries. */
int og_set_sinkhorn_resident(int resident);
/* How og_sinkhorn_fwd runs (batch, n, m) on the current device under the current setting: plan[0..9] = resident (1) or streaming
 * (0), float4s per lane, warps per row, strips per pair, rows per strip, pairs per launch, rows per warp held in registers, rows
 * per warp held in shared memory, dynamic shared memory per CTA (bytes), CTAs per SM. */
int og_sinkhorn_plan(int batch, int n, int m, int64_t* plan);
int og_sinkhorn_fwd(const float* S, int64_t lds, int64_t strideS, const float* dustbin,
                    int batch, int n, int m, int iters, float reg,
                    float* scores, void* workspace, int64_t workspace_bytes, void* stream);
/* Padded form: pair b is the [n_b, m_b] block of the capacity n x m (lengths: device int32 [2B], n_0 .. n_{B-1}, m_0 .. m_{B-1},
 * clamped into [1, n] / [1, m]; n <= 65536); scores[b, :n_b+1, :m_b+1] is its augmented log-assignment (dustbin row n_b, column
 * m_b), -inf elsewhere.  The plan and workspace are the capacity's.  og_sinkhorn_consts: the host's (norm, log_a_last,
 * log_b_last) of an n x m pair; og_sinkhorn_consts_padded: out [B, 3] (device), what the padded kernels use for each pair, bit
 * for bit the host's.  The first padded call on a device uploads tables synchronously: it must not be stream-captured.  */
int og_sinkhorn_fwd_padded(const float* S, int64_t lds, int64_t strideS, const float* dustbin,
                           int batch, int n, int m, const int* lengths, int iters, float reg,
                           float* scores, void* workspace, int64_t workspace_bytes, void* stream);
int og_sinkhorn_consts(int n, int m, float* out);
int og_sinkhorn_consts_padded(const int* lengths, int batch, int n, int m, float* out, void* stream);

/* Training form of the Sinkhorn operator (SURVEY.md section 8, row f1).  og_sinkhorn_train_fwd = og_sinkhorn_fwd that also
 * records the scaling vectors of every iteration (hist: og_sinkhorn_hist_floats floats: u [B][T][n+1], v [B][T+1][m+1]);
 * og_sinkhorn_bwd = the gradient through all T unrolled iterations, as torch autograd computes it for the reference's
 * get_matching_probs / log_otp_solver in training_step (matching_module.py:99-105):
 *   dscores [B,n+1,m+1] = d loss / d scores (dense)  ->  dS_aug [B,n+1,m+1] = d loss / d S_aug (its [:n,:m] block is
 *   d loss / d S of the score GEMM, reg included) and ddustbin[0] = d loss / d dustbin_score.  Deterministic.        */
int64_t og_sinkhorn_hist_floats(int batch, int n, int m, int iters);
int og_sinkhorn_train_fwd(const float* S, int64_t lds, int64_t strideS, const float* dustbin,
                          int batch, int n, int m, int iters, float reg, float* scores, float* hist,
                          void* workspace, int64_t workspace_bytes, void* stream);
int64_t og_sinkhorn_bwd_workspace_bytes(int batch, int n, int m, int iters);
int og_sinkhorn_bwd(const float* S, int64_t lds, int64_t strideS, const float* dustbin,
                    int batch, int n, int m, int iters, float reg, const float* hist,
                    const float* dscores, float* dS_aug, float* ddustbin,
                    void* workspace, int64_t workspace_bytes, void* stream);
/* Padded forms (lengths as og_sinkhorn_fwd_padded; same hist size and workspace): pair b runs on its [n_b, m_b] block with its own
 * marginals; hist keeps the capacity's strides (pair b's dustbin entries at n_b / m_b).  The backward pass reads dscores on each
 * pair's [n_b + 1, m_b + 1] block only, writes dS_aug there and 0 on the rest of the capacity, and ddustbin sums each pair's own
 * dustbin row and column.  Both need the tables og_sinkhorn_fwd_padded uploads (one padded call before a stream capture). */
int og_sinkhorn_train_fwd_padded(const float* S, int64_t lds, int64_t strideS, const float* dustbin,
                                 int batch, int n, int m, const int* lengths, int iters, float reg, float* scores, float* hist,
                                 void* workspace, int64_t workspace_bytes, void* stream);
int og_sinkhorn_bwd_padded(const float* S, int64_t lds, int64_t strideS, const float* dustbin,
                           int batch, int n, int m, const int* lengths, int iters, float reg, const float* hist,
                           const float* dscores, float* dS_aug, float* ddustbin,
                           void* workspace, int64_t workspace_bytes, void* stream);

/* Mutual-argmax match extraction on scores[:, :n, :m].  Replaces
 * models/matching_module.py:174-187 and inference.py:176-190 (ties -> lowest index).
 *   workspace >= og_match_workspace_bytes(B, n, m)                                             */
int64_t og_match_workspace_bytes(int batch, int n, int m);
int og_match_fwd(const float* scores, int batch, int n, int m, float threshold,
                 int64_t* matches0, float* mscores0, int64_t* matches1, float* mscores1,
                 void* workspace, int64_t workspace_bytes, void* stream);
/* Padded form (lengths as og_sinkhorn_fwd_padded; batch <= 65535): pair b's matches on scores[b, :n_b, :m_b]; -1 / 0 past them. */
int og_match_fwd_padded(const float* scores, int batch, int n, int m, const int* lengths, float threshold,
                        int64_t* matches0, float* mscores0, int64_t* matches1, float* mscores1,
                        void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Ground-truth match generation: the step immediately BEFORE the matching core in the reference's
 * training / validation step (models/matching_module.py:84-93).  Replaces
 * generate_gt_matches (models/gt_matches_generation.py:17-93) with reproject_keypoints /
 * get_inverse_transformation (utils/misc.py:21-103): reprojection of both keypoint sets, the two
 * N x M torch.cdist + min, the mutual check and the UNMATCHED (-1) / IGNORE (-2) marks.  The
 * reference's threshold refinements (:56-67, :76-78) assign through boolean-mask copies and have
 * no effect; they are not reproduced, so the thresholds are not parameters here.
 * ------------------------------------------------------------------------------------------- */
enum { OG_GT_PERSPECTIVE = 0, OG_GT_3D_REPROJECTION = 1 };   /* transformation['type'] (utils/misc.py:23-34) */
typedef struct og_gt_transform {
  int32_t type;
  const float* H;                    /* perspective: [B,3,3]                                            */
  const float* K0; const float* K1;  /* 3d: intrinsics [B,3,3]                                          */
  const float* R;  const float* T;   /* 3d: relative pose [B,3,3], [B,3]  (x1 = R x0 + T)               */
  const float* depth0;               /* 3d: per-keypoint depth [B,n] / [B,m], or depth images           */
  const float* depth1;               /*     [B,depth{0,1}_h,depth{0,1}_w] when depth_is_image           */
  int32_t depth_is_image;
  int32_t depth0_h, depth0_w, depth1_h, depth1_w;
} og_gt_transform;

int64_t og_gt_matches_workspace_bytes(int batch, int n, int m);
/* kpts0 [B,n,2], kpts1 [B,m,2] pixel coordinates; gt_matches0 [B,n], gt_matches1 [B,m] int64
 * (index of the match, -1 unmatched, -2 ignore).  All pointers are device memory.                  */
int og_gt_matches_fwd(const float* kpts0, const float* kpts1, int batch, int n, int m, const og_gt_transform* tf,
                      int64_t* gt_matches0, int64_t* gt_matches1, void* workspace, int64_t workspace_bytes, void* stream);
/* Padded form (lengths as og_sinkhorn_fwd_padded): pair b's nearest neighbours and mutual check run over its first n_b / m_b
 * keypoints; its labels past them are -2 (ignore).  Per-keypoint depths keep the capacity's layout [B,n] / [B,m].            */
int og_gt_matches_fwd_padded(const float* kpts0, const float* kpts1, int batch, int n, int m, const int* lengths,
                             const og_gt_transform* tf, int64_t* gt_matches0, int64_t* gt_matches1, void* workspace,
                             int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Batch collation of cached local features: the step that FEEDS the path from the cached-feature dataset.  Replaces
 * MegaDepthPairsDataModuleFeatures.stack_keypoints_batch (data/megadepth_datamodule.py:105-168): per image, the
 * `target_keypoints` most confident keypoints in descending score order (select == NULL; torch.topk, ties -> lower
 * index) or the caller's selection (select [2*batch, target_keypoints] int32: torch.randperm indices, training), all of
 * them + zero padding when an image has fewer; depth{0,1} [batch, H, W] images are sampled at (int(y), int(x)) of every
 * kept keypoint (NULL: no depth).  Raw inputs are the images' features concatenated in the order (pair 0, image 0),
 * (pair 0, image 1), (pair 1, image 0) ...: lafs [total,2,3], scores [total], desc [total,D], offsets [2*batch+1] int32;
 * max_count = the largest image (<= 16384).  Outputs [batch, target, ...] per image side.  Index work: bit-exact.      */
int og_collate_fwd(const float* lafs, const float* scores, const float* desc, const int* offsets, const int* select, int max_count,
                   const float* depth0, int depth0_h, int depth0_w, const float* depth1, int depth1_h, int depth1_w,
                   int batch, int target_keypoints, int descriptor_dim,
                   float* out_lafs0, float* out_lafs1, float* out_scores0, float* out_scores1, float* out_desc0, float* out_desc1,
                   float* out_depth0, float* out_depth1, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Matching loss: the step immediately AFTER the matching core in the reference's training step
 * (models/matching_module.py:101).  Replaces criterion (utils/losses.py:7-53) for margin = None (every
 * shipped config): loss[0] = 'loss' (negative log-likelihood of the ground-truth assignment, mean per set and
 * per pair), loss[1] = 'metric_loss' = 0.  gt_matches0 [B,n] / gt_matches1 [B,m] int64 as og_gt_matches_fwd
 * writes them (-1 unmatched, -2 ignore).  dscores (optional, [B,n+1,m+1], ZERO-FILLED by the caller) receives
 * grad_scale * d loss / d scores (a sparse scatter: the backward pass of the gather).  Deterministic.      */
int64_t og_criterion_workspace_bytes(int batch);
int og_criterion_fwd(const float* scores, const int64_t* gt_matches0, const int64_t* gt_matches1, int batch, int n, int m,
                     float* loss, float* dscores, float grad_scale, void* workspace, int64_t workspace_bytes, void* stream);
/* Padded form (lengths as og_sinkhorn_fwd_padded): pair b's loss reads its [n_b + 1, m_b + 1] block of scores (dustbins at n_b,
 * m_b) and its first n_b / m_b labels; loss[0] is the mean of the B pairs' losses.  dscores outside each block stays 0.        */
int og_criterion_fwd_padded(const float* scores, const int64_t* gt_matches0, const int64_t* gt_matches1, int batch, int n, int m,
                            const int* lengths, float* loss, float* dscores, float grad_scale, void* workspace,
                            int64_t workspace_bytes, void* stream);

/* Metric terms of the same loss for a margin mu: criterion(..., margin=mu)['metric_loss'] (utils/losses.py:56-99 on the
 * half cosine distance of utils/misc.py:106-113, dist = 0.25 |normalize(c0_i) - normalize(c1_j)|^2).
 *   c0 [B, d, n], c1 [B, d, m]: the context descriptors (SuperGlue.forward's context_descriptors0/1);
 *   gt_matches0/1 as og_criterion_fwd;  metric_loss [1] receives the value;
 *   n0, u0 [B, n] and n1, u1 [B, m] (int64) receive the hard negatives: n0 / n1 = argmin over the row / column of dist with
 *   every (i, gt0[i]) of a matched row masked, u0 / u1 the unmasked argmins (ties: the lowest index, as torch.argmin);
 *   dc0 [B, d, n], dc1 [B, d, m] (both or neither) receive grad_scale * d metric_loss / d c0, c1 (overwritten).
 * precision OG_PREC_FP32 or OG_PREC_TF32X3 selects the GEMMs behind the Gram X Y^T and the gradient.  Launches:
 * 9 (16 with dc0/dc1) with OG_PREC_FP32; OG_PREC_TF32X3 adds one operand-split launch per GEMM that runs on the tensor cores:
 * the Gram when d % 4 == 0 and d >= 32, with dc0/dc1 also dX when m rounded up to 4 is >= 32 and dY when n rounded up to 4 is
 * >= 32 (other shapes run the exact fp32 kernel).  Deterministic, no host synchronisation.  OG_EINVAL without a
 * launch: a null pointer, dc0 without dc1 (or the reverse), B outside [1, 65535], n, m or d < 1, another precision.
 * og_metric_loss_workspace_bytes: -1 for such sizes.                                                          */
int64_t og_metric_loss_workspace_bytes(int batch, int d, int n, int m, int want_grad, int precision);
int og_metric_loss_fwd(const float* c0, const float* c1, const int64_t* gt_matches0, const int64_t* gt_matches1, int batch, int d,
                       int n, int m, float margin, int precision, float* metric_loss, int64_t* n0, int64_t* u0, int64_t* n1,
                       int64_t* u1, float* dc0, float* dc1, float grad_scale, void* workspace, int64_t workspace_bytes,
                       void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training-step operators (SURVEY.md section 8, row f1): what nn.BatchNorm1d in training mode and torch autograd do for the
 * reference around the contractions of SuperGlue.forward in MatchingTrainingModule.training_step
 * (models/matching_module.py:71-105).  The contractions themselves (dX = dY W, dW = dY^T X, the attention gradients
 * dV = P^T dO, dP = dO V^T, dQ = dS K, dK = dS^T Q) run on og_linear_fwd / og_linear_tc_fwd with transposed operands.
 * Activations are row-major [rows, channels], rows = batch x keypoints.  All reductions are deterministic.
 *   og_transpose        transpose != 0: out[b][c, r] = in[b][r, c];  == 0: pitch-changing copy.  Padding is left untouched.
 *   og_colsum           out[c] = sum_r x[r,c] * (y ? y[r,c] - (z ? z[r,c] : 0) : 1)           (bias / mix gradients)
 *   og_bn_train_fwd     y = gamma (r - mean) invstd + beta, r = relu ? max(a, 0) : a, batch statistics over the rows
 *                       (biased variance), save_mean / save_invstd [cols] kept for the backward pass, running_mean /
 *                       running_var (optional) updated with `momentum` (unbiased variance): models/utils.py:48-58,
 *                       torch.nn.BatchNorm1d(training=True)
 *   og_bn_train_bwd     da (through the fused ReLU), dgamma, dbeta from dy
 *   og_softmax_rows     in-place row softmax of the materialised attention scores (models/superglue/attention.py:12-13)
 *   og_softmax_bwd_rows dP <- scale * P * (dP - sum_j P dP)
 *   og_axpby            out = a x + b y (y NULL: a x)
 *   og_mix_fwd / _bwd / _param_grad   residual mix alpha = sigmoid(mix_coefs) (superglue.py:59-62) and its gradients
 *   og_kenc_input       [2 x / (W - 1) - 1, 2 y / (H - 1) - 1, side info]  (superglue.py:74-78, positional_encoding.py:16-18)
 * workspace: >= og_train_workspace_floats(cols) floats.                                                           */
int64_t og_train_workspace_floats(int cols);
/* One GEMM of the training step, args as og_linear_fwd: the wgmma 3xTF32 kernel when the shape is tileable (K >= 32,
 * K % 4 == 0, 16-byte aligned rows, dense batches; W is split into split_scratch, og_linear_auto_scratch_floats(args)
 * floats, on the fly), the exact fp32 CUDA-core kernel otherwise or when precision == OG_PREC_FP32.               */
int64_t og_linear_auto_scratch_floats(const og_linear_args* args);
int og_linear_auto_fwd(const og_linear_args* args, int precision, float* split_scratch, void* stream);
int og_transpose(const float* in, int64_t ld_in, int64_t stride_in, float* out, int64_t ld_out, int64_t stride_out,
                 int batch, int rows, int cols, int transpose, void* stream);
int og_colsum(const float* x, int64_t ldx, const float* y, int64_t ldy, const float* z, int64_t ldz, int rows, int cols,
              float* out, float* workspace, void* stream);
int og_bn_train_fwd(const float* a, int64_t lda, int rows, int cols, int relu, const float* gamma, const float* beta,
                    float eps, float momentum, float* y, int64_t ldy, float* save_mean, float* save_invstd,
                    float* running_mean, float* running_var, float* workspace, void* stream);
int og_bn_train_bwd(const float* dy, int64_t lddy, const float* a, int64_t lda, int rows, int cols, int relu,
                    const float* gamma, const float* save_mean, const float* save_invstd,
                    float* da, int64_t ldda, float* dgamma, float* dbeta, float* workspace, void* stream);
int og_softmax_rows(float* S, int64_t ld, int64_t rows, int cols, void* stream);
int og_softmax_bwd_rows(const float* P, float* dP, int64_t ld, int64_t rows, int cols, float scale, void* stream);
int og_axpby(const float* x, const float* y, float a, float b, float* out, int64_t n, void* stream);
/* out[r, c] (+)= sum_s part[s][r, c] (s ascending; out row stride ld_out): reduction of the split-K weight gradients      */
int og_sum_batches(const float* part, int S, int rows, int cols, float* out, int64_t ld_out, int accumulate, void* stream);
int og_mix_fwd(const float* g, const float* l, const float* mix, float* out, int64_t rows, int d, void* stream);
int og_mix_bwd(const float* dm, const float* mix, float* dg, float* dl, int64_t rows, int d, void* stream);
int og_mix_param_grad(const float* colsum, const float* mix, float* dmix, int d, void* stream);
int og_kenc_input(const float* kpts, const float* side, int rows, int side_info_size, float width, float height,
                  float* out, void* stream);
/* Padded forms of the training-step operators.  Rows are [batch, cap]: row r is slot r % cap of pair r / cap, real below
 * lengths[r / cap] (device int32 [batch], clamped into [1, cap]).
 *   og_bn_train_fwd_padded / _bwd_padded  batch statistics over the real rows of every pair: mean and biased variance over
 *                       sum_b n_b rows, running_var with the unbiased factor sum n / (sum n - 1); dgamma / dbeta over the real
 *                       rows; da = 0 on the padding rows.  Padding rows of y are finite when a is.
 *   og_softmax_rows_padded / og_softmax_bwd_rows_padded   rows [batch, seq_rows]: sequence b's rows take its first
 *                       key_lengths[b] columns of `cols`; P = 0 (dS = 0) on the others
 *   og_kenc_input_padded   og_kenc_input with each pair's (W, H) from pair_wh (rows 4 floats apart) and the padding rows 0
 *   og_mask_padded_rows    dst = src [batch * cap, cols] with the padding rows 0 (dst may not alias src)                  */
int og_bn_train_fwd_padded(const float* a, int64_t lda, int batch, int cap, const int* lengths, int cols, int relu, const float* gamma,
                           const float* beta, float eps, float momentum, float* y, int64_t ldy, float* save_mean, float* save_invstd,
                           float* running_mean, float* running_var, float* workspace, void* stream);
int og_bn_train_bwd_padded(const float* dy, int64_t lddy, const float* a, int64_t lda, int batch, int cap, const int* lengths, int cols,
                           int relu, const float* gamma, const float* save_mean, const float* save_invstd,
                           float* da, int64_t ldda, float* dgamma, float* dbeta, float* workspace, void* stream);
int og_softmax_rows_padded(float* S, int64_t ld, int batch, int64_t seq_rows, int cols, const int* key_lengths, void* stream);
int og_softmax_bwd_rows_padded(const float* P, float* dP, int64_t ld, int batch, int64_t seq_rows, int cols, float scale,
                               const int* key_lengths, void* stream);
int og_kenc_input_padded(const float* kpts, const float* side, int batch, int cap, const int* lengths, int side_info_size,
                         const float* pair_wh, float* out, void* stream);
int og_mask_padded_rows(const float* src, int batch, int cap, int cols, const int* lengths, float* dst, void* stream);
/* Guarded forms: the skip of the reference's training_step (models/matching_module.py:96-97) decided on the device, so that a
 * training step from images runs without a host synchronisation.  `skip` is a device int32 flag; a skipped step changes no
 * training state.
 *   og_train_guard          skip = 1 when some lengths[i] <= 0 (an image without keypoints: the reference's `data is None`) or
 *                           when the B row lengths or the B column lengths total fewer than 2 (BatchNorm1d's "more than 1 value
 *                           per channel"), else 0.  lengths [2B] device int32: n_0 .. n_{B-1}, m_0 .. m_{B-1}.
 *   og_bn_train_fwd_guarded og_bn_train_fwd_padded (og_bn_train_fwd over batch x cap rows when lengths is NULL) with: running_mean /
 *                           running_var left untouched when *skip != 0; num_batches_tracked (int64, optional) += 1 - *skip on
 *                           the device.  y, save_mean and save_invstd are written either way.  skip NULL: never skipped.
 *   og_train_skip_outputs   when *skip != 0: loss[0 .. nloss) = NaN, x[0 .. n) = 0 (gradients); nothing otherwise.  nloss <= 256.
 * With skip NULL or *skip == 0 every guarded form equals its unguarded entry point bit for bit.                         */
int og_train_guard(const int* lengths, int B, int* skip, void* stream);
int og_bn_train_fwd_guarded(const float* a, int64_t lda, int batch, int cap, const int* lengths, int cols, int relu, const float* gamma,
                            const float* beta, float eps, float momentum, float* y, int64_t ldy, float* save_mean, float* save_invstd,
                            float* running_mean, float* running_var, const int* skip, int64_t* num_batches_tracked, float* workspace,
                            void* stream);
int og_train_skip_outputs(const int* skip, float* loss, int nloss, float* x, int64_t n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * SuperPoint front-end operators (SURVEY.md section 8, row f4): SuperPointNet.forward (models/features/superpoint/model.py:61-129)
 * on NHWC activations.  Convolutions = og_sp_im2col3x3 (3x3, pad 1) + og_linear_auto_fwd (bias / ReLU fused; 1x1: the GEMM alone).
 *   og_sp_im2col3x3     out[p, (3 ky + kx) C + c] = x[b, y + ky - 1, x + kx - 1, c] (zero padding);  x [B,H,W,C], out [B H W, 9 C]
 *   og_sp_maxpool2x2    nn.MaxPool2d(2, 2) on NHWC
 *   og_row_normalize    mode 0: x /= ||x||_2 per row (model.py:70-71);  mode 1: F.normalize (x /= max(||x||_2, eps))
 *   og_sp_heat_nms      probs [B,Hc,Wc,65] (channel softmax done) -> heat [B, 8 Hc, 8 Wc]: pixel shuffle (model.py:84-86), nms2d
 *                       (kornia >= 0.6.1, restated: x > max(0, the other k*k - 1 values of the replicate-padded window)),
 *                       F.threshold + nonzero (model.py:89-92) and remove_borders (utils.py:4-11): the score where kept, else 0
 *   og_sp_compact       per image: surviving pixels in row-major order (torch.nonzero) -> cand_idx / cand_score [B, cap], count [B]
 *   og_sp_select        per image: n_out[b] keypoints, mode[b] = 0 in candidate order | 1 = the largest scores, descending (torch.topk,
 *                       equal scores: lower index first; top_k_keypoints utils.py:34-39, min_stack models/features/utils.py:28-56);
 *                       kpts [B,out_cap,2] as (x, y) floats, scores [B,out_cap];  max_count = the largest count (<= 16384);
 *                       the caller guarantees n_out[b] <= min(count[b], cap, out_cap) (a larger n_out reads unwritten candidates)
 *   og_sp_sample_desc   sample_desc_from_points (utils.py:14-31): bilinear grid_sample (align_corners False) of the coarse descriptors
 *                       [B,Hc,Wc,D] at the keypoints + F.normalize -> desc [B,out_cap,D]                                        */
int og_sp_im2col3x3(const float* x, int B, int H, int W, int C, float* out, void* stream);
int og_sp_maxpool2x2(const float* x, int B, int H, int W, int C, float* out, void* stream);
int og_row_normalize(float* x, int64_t rows, int C, int mode, float eps, void* stream);
int og_sp_heat_nms(const float* probs, int B, int Hc, int Wc, int nms_kernel, float threshold, int border, float* heat, void* stream);
int og_sp_compact(const float* heat, int B, int HW, int cap, int* cand_idx, float* cand_score, int* count, void* stream);
int og_sp_select(const int* cand_idx, const float* cand_score, const int* count, const int* n_out, const int* mode, int B, int cap, int W,
                 int out_cap, int max_count, float* kpts, float* scores, void* stream);
int og_sp_sample_desc(const float* coarse, int B, int Hc, int Wc, int D, const float* kpts, const int* n_out, int out_cap, int max_n, int cell,
                      float* desc, void* stream);

/* ---------------------------------------------------------------------------------------------
 * OpenCV SIFT front-end (OPENCV_SIFT: cv2.SIFT_create(contrastThreshold=-10000, edgeThreshold=-10000) + the reference's radius NMS,
 * top-k, RootSIFT and LAFs; models/features/opencv/_features.py:10-18, base.py:14-182).  B same-size images per call.
 * Keypoints are kp [B, cap, 5] = (x, y, size, angle, response) floats and octave [B, cap] (cv2's packed octave word), per image in
 * cv2's order (x, y, size desc, angle, response desc, octave desc) without exact duplicates.
 *   og_sift_workspace_bytes  the workspace of og_sift_detect / og_sift_describe (Gaussian and DoG pyramids, candidate lists);
 *                            < 0 (OG_EUNSUPPORTED) when the image has no octave or more than 16
 *   og_sift_detect           image [B, H, W] (dtype 0: uint8; 1: float32, quantised as the torch wrapper does: uint8(255 * x))
 *                            -> kp, octave, count [B]; count[b] > cap means cap was too small and the outputs are incomplete.
 *                            The pyramid stays in ws for og_sift_describe.
 *   og_sift_select_workspace_bytes / og_sift_select
 *                            greedy radius NMS (visit by response desc, equal responses by index asc; a kept point removes every
 *                            point within nms_radius, inclusive; none when nms_radius <= 0) then the max_keypoints largest
 *                            responses (all when <= 0): sel [B, cap] indices into kp by response desc, index asc; n_sel [B].
 *                            Takes any keypoints, e.g. cv2's own; count[b] is clamped to [0, cap].
 *   og_sift_describe         cv2's descriptors of kp[b, sel[b, j]], j < n_sel[b] (and < out_cap), from og_sift_detect's pyramid in ws
 *                            (same B, H, W, cap), then normalize_descriptors (rootsift: L1 + sqrt, else L2) and lafs_from_opencv_kpts
 *                            (mr_size 6): lafs [B, out_cap, 2, 3], scores [B, out_cap], desc [B, out_cap, 128], raw_desc (optional)
 *                            [B, out_cap, 128] cv2's integer-valued descriptor.  max_n >= every n_sel[b] sizes the grid.
 *   og_sift_detect_padded    og_sift_detect for outputs padded to a fixed capacity: count[b] is always the number of keypoints
 *                            written (<= cap) and overflow[b] = 1 marks an image that exceeded a capacity (its keypoints are then
 *                            incomplete), 0 otherwise.  Nothing is read back to the host.
 *   og_sift_rootsift_laf     normalize_descriptors + lafs_from_opencv_kpts of supplied kp [N, 5] and raw descriptors [N, 128]
 *   og_sift_fast_atan2       out[i] = cv2's fastAtan2(y[i], x[i]) in degrees: fused = cv::hal::fastAtan2's vector form, 0 = the
 *                            scalar one (cv2.fastAtan2)
 *   og_sift_gaussian_taps    host only: cv2's float Gaussian kernel for sigma (taps computed in double, rounded to float); returns the
 *                            number of taps, or OG_EUNSUPPORTED when it exceeds cap
 *   og_sift_workspace_layout host only: where og_sift_detect keeps each stage's results in its workspace, for reading them back.
 *                            out[0] = the octave count nO; out[1 + 4 o ..] = h, w, Gaussian offset, DoG offset of octave o (levels
 *                            [6][B][h][w] and [5][B][h][w] float32); then the byte offsets of the located extrema (the SiftLoc
 *                            records of csrc/sift.cuh, [B][cap]), the raw keypoints ([B][cap][5] float32), their octave words
 *                            ([B][cap] int32) and the counts (int32: located [B], then raw keypoints [B]), and the workspace
 *                            size.  Returns the number of entries written (1 + 4 nO + 5), or < 0 when n is too small       */
int64_t og_sift_workspace_bytes(int B, int H, int W, int cap);
int og_sift_workspace_layout(int B, int H, int W, int cap, int64_t* out, int n);
int og_sift_detect(const void* image, int dtype, int B, int H, int W, int cap, void* ws, int64_t ws_bytes, float* kp, int* octave,
                   int* count, void* stream);
int og_sift_detect_padded(const void* image, int dtype, int B, int H, int W, int cap, void* ws, int64_t ws_bytes, float* kp, int* octave,
                          int* count, int* overflow, void* stream);
int64_t og_sift_select_workspace_bytes(int B, int cap);
int og_sift_select(const float* kp, const int* count, int B, int cap, float nms_radius, int max_keypoints, void* work, int64_t work_bytes,
                   int* sel, int* n_sel, void* stream);
int og_sift_describe(const void* ws, int B, int H, int W, int cap, const float* kp, const int* octave, const int* sel, const int* n_sel,
                     int out_cap, int max_n, int rootsift, float* lafs, float* scores, float* desc, float* raw_desc, void* stream);
int og_sift_rootsift_laf(const float* kp, const float* raw_desc, int64_t N, int rootsift, float* lafs, float* scores, float* desc, void* stream);
int og_sift_fast_atan2(const float* y, const float* x, int64_t n, int fused, float* out, void* stream);
int og_sift_gaussian_taps(double sigma, float* taps, int cap);

/* ---------------------------------------------------------------------------------------------
 * kornia's DoG SIFT front-end (the reference's SIFT, models/features/sift.py on base.py: ScaleSpaceDetector + run_nms + LAFDescriptor
 * of kornia 0.6.3; csrc/kornia_sift.cuh).  B same-size float32 images [B, H, W] in [0, 1]; num_features (<= 8192) keypoints per image
 * leave the detector.  Every stage is its own call, so a caller (or a test) can feed any stage its own inputs.
 *   og_ksift_workspace_bytes   the workspace of pyramid / detect / describe (same B, H, W, num_features): octaves, responses,
 *                              the selection state and the patch pyramid; < 0 when the image is not supported
 *   og_ksift_workspace_layout  host only: out[0] = the octave count nO; out[1 + 5 o ..] = h, w, and the byte offsets of the Gaussian
 *                              levels ([B][6][h][w]), the DoG ([B][5][h][w]) and the voxel responses ([B][5][h][w]) of octave o; then
 *                              the patch-pyramid level count nP and per level h, w, byte offset (-1: level 0 is the image); then
 *                              the workspace size.  Returns the number of entries written
 *   og_ksift_pyramid           ScalePyramid(3, 1.6, 32, double_image=True) and BlobDoG into ws
 *   og_ksift_detect            from the DoG in ws: conv_quad_interp3d on DoG and -DoG, the per-octave top-k of every voxel (response
 *                              desc, voxel index asc), laf_is_inside_image, the global top-k (response desc, octave asc, per-octave
 *                              rank asc) -> lafs [B, num_features, 2, 3] in image pixels (before orientation), resp [B, num_features],
 *                              count [B] (rows past it are 0)
 *   og_ksift_select_workspace_bytes / og_ksift_select
 *                              base.py's run_nms on detector outputs lafs [B, cap, 2, 3], resp [B, cap], count [B] of H x W images:
 *                              nms = 0 keeps every output; otherwise the float32 key sort (equal keys by index), unique positions,
 *                              nms2d(nms_diameter, odd) on the scattered scores, then the first min(survivors, max_keypoints)
 *                              survivors in detector order (their top-k; max_keypoints <= 0: no cap), survivors = the batch minimum
 *                              when min_stack -> sel [B, cap] detector indices, n_sel [B]
 *   og_ksift_describe          rows j < n[b] of lafs_out [B, out_cap, 2, 3], scores, desc [B, out_cap, 128] and angle (optional,
 *                              [B, out_cap]: LAFOrienter's dominant orientation in radians) for detector output sel[b][j] (sel NULL:
 *                              j): LAFOrienter(19) unless upright, then SIFTDescriptor(41, rootsift) on kornia's pyrdown patch pyramid
 *                              of image; rows past n[b] are written as 0                                                       */
int64_t og_ksift_workspace_bytes(int B, int H, int W, int num_features);
int og_ksift_workspace_layout(int B, int H, int W, int num_features, int64_t* out, int n);
int og_ksift_pyramid(const float* image, int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, void* stream);
int og_ksift_detect(int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, float* lafs, float* resp, int* count, void* stream);
int64_t og_ksift_select_workspace_bytes(int B, int cap);
int og_ksift_select(const float* lafs, const float* resp, const int* count, int B, int H, int W, int cap, int nms, int nms_diameter,
                    int max_keypoints, int min_stack, void* work, int64_t work_bytes, int* sel, int* n_sel, void* stream);
int og_ksift_describe(const float* image, int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, const float* lafs,
                      const float* resp, int cap, const int* sel, const int* n, int out_cap, int upright, int rootsift, float* lafs_out,
                      float* scores, float* desc, float* angle, void* stream);

/* ---------------------------------------------------------------------------------------------
 * kornia's GFTT / AffNet / HardNet front-end (the reference's GFTTAffNetHardNet, models/features/hardnet.py on base.py, kornia 0.6.3;
 * csrc/kornia_gftt.cuh).  Same images and num_features as og_ksift_*; selection is og_ksift_select.  The two patch CNNs are run by
 * the caller between the describe stages (NHWC im2col: og_sp_im2col3x3 / og_kgftt_im2col3x3_s2, then og_linear_auto_fwd), over
 * chunks of output rows [r0, r0 + rows) of the [B, out_cap] output, so their scratch is bounded by the chunk size.
 *   og_kgftt_workspace_bytes / og_kgftt_workspace_layout   as og_ksift_*; octave 0 is H x W and the second volume of each octave
 *                              holds the GFTT responses of all 6 Gaussian levels ([B][6][h][w])
 *   og_kgftt_pyramid           ScalePyramid(3, 1.6, 32, double_image=False), CornerGFTT on every level (times sigma^4), and the
 *                              pyrdown patch pyramid of image, into ws
 *   og_kgftt_detect            conv_quad_interp3d (maxima only) on levels 0 .. 4 of the responses, then og_ksift_detect's top-k,
 *                              border test and merge -> lafs [B, num_features, 2, 3] (before AffNet), resp, count [B]
 *   og_kgftt_affnet_patches    patches [rows, 32, 32]: AffNet's standardised input ((x - mean) / (std + 1e-6), Bessel's std) on
 *                              make_upright of detector output sel[b][j] (sel NULL: j), zeros for rows with j >= n[b]
 *   og_kgftt_frames            from AffNet's 8x8-conv output xy [rows, 3] (before tanh): the affine LAF (preserve_orientation),
 *                              LAFOrienter(19) unless upright -> lafs_out, scores, angle (optional) rows of [B, out_cap], and
 *                              patches [rows, 32, 32], HardNet's standardised input on the final LAF; rows past n[b] are 0
 *   og_kgftt_im2col3x3_s2      3x3, stride 2, pad 1 im2col on NHWC: out [B ceil(H/2) ceil(W/2), 9 C], columns (3 ky + kx) C + c
 *   og_kgftt_desc_finish       desc [B, out_cap, 128]: rows j < n[b] divided by max(||row||_2, 1e-12) (F.normalize), others 0  */
int64_t og_kgftt_workspace_bytes(int B, int H, int W, int num_features);
int og_kgftt_workspace_layout(int B, int H, int W, int num_features, int64_t* out, int n);
int og_kgftt_pyramid(const float* image, int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, void* stream);
int og_kgftt_detect(int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, float* lafs, float* resp, int* count, void* stream);
int og_kgftt_affnet_patches(const float* image, int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, const float* lafs, int cap,
                            const int* sel, const int* n, int out_cap, int r0, int rows, float* patches, void* stream);
int og_kgftt_frames(const float* image, int B, int H, int W, int num_features, void* ws, int64_t ws_bytes, const float* lafs, const float* resp,
                    int cap, const int* sel, const int* n, int out_cap, int r0, int rows, const float* xy, int upright, float* lafs_out,
                    float* scores, float* angle, float* patches, void* stream);
int og_kgftt_im2col3x3_s2(const float* x, int B, int H, int W, int C, float* out, void* stream);
int og_kgftt_desc_finish(float* desc, int B, int out_cap, const int* n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * The DoG / AffNet / OriNet / HardNet front-end (the reference's OPENCVDoGAffNetHardNet, models/features/opencv/dog_affnet_harnet.py:
 * cv2 SIFT keypoints, kornia_moons' LAFs, kornia 0.6.3's AffNet, OriNet and HardNet; csrc/dog_affnet.cuh).  Detection and selection
 * are og_sift_detect (dtype 1) and og_sift_select; these stages describe the selected keypoints from the float image [B, H, W].
 * The three CNNs are run by the caller between the stages (as og_kgftt_*), over chunks of output rows [r0, r0 + rows) of the
 * [B, out_cap] output.  lafs [B, out_cap, 2, 3] carries each row's LAF between the stages: each stage reads its rows and rewrites them.
 *   og_dogaff_workspace_bytes / og_dogaff_workspace_layout   the float image's pyrdown patch pyramid for 32-pixel patches.
 *                              layout (host only): out[0] = levels np; out[1 + 3 l ..] = h, w, byte offset of level l (-1: the
 *                              image); then the workspace bytes.  Returns the entries written.
 *   og_dogaff_pyramid          builds the patch pyramid of image into ws
 *   og_dogaff_affnet_patches   row (b, j), j < n[b]: keypoint kp[b, sel[b, j]] (kp [B, cap, 5] = x, y, size, angle, response) ->
 *                              lafs = laf_from_opencv_SIFT_kpts (mrSize 6), scores = response, patches [rows, 32, 32] = AffNet's
 *                              standardised input on make_upright(laf); rows past n[b] are 0
 *   og_dogaff_frames           from AffNet's 8x8-conv output xy [rows, 3] (before tanh): lafs <- the affine LAF (preserve_orientation),
 *                              patches = OriNet's standardised input on it
 *   og_dogaff_orinet_head      from OriNet's last 3x3-conv activations act [rows, 8, 8, 64] (NHWC, 16-byte aligned), the head's
 *                              weight [2, 8, 8, 64] ((ky, kx, c) order, 8-byte aligned) and bias [2]: Conv2d(64, 2, 8, padding=1),
 *                              tanh, mean, angle = atan2(y0 + 1e-8, y1 + 1e-8); lafs <- set_laf_orientation(laf, rad2deg(angle) +
 *                              get_laf_orientation(laf)), angle [B, out_cap], patches = HardNet's standardised input on the new LAF */
int64_t og_dogaff_workspace_bytes(int B, int H, int W);
int og_dogaff_workspace_layout(int B, int H, int W, int64_t* out, int n);
int og_dogaff_pyramid(const float* image, int B, int H, int W, void* ws, int64_t ws_bytes, void* stream);
int og_dogaff_affnet_patches(const float* image, int B, int H, int W, void* ws, int64_t ws_bytes, const float* kp, int cap, const int* sel,
                             const int* n, int out_cap, int r0, int rows, float* lafs, float* scores, float* patches, void* stream);
int og_dogaff_frames(const float* image, int B, int H, int W, void* ws, int64_t ws_bytes, const int* n, int out_cap, int r0, int rows,
                     const float* xy, float* lafs, float* patches, void* stream);
int og_dogaff_orinet_head(const float* image, int B, int H, int W, void* ws, int64_t ws_bytes, const int* n, int out_cap, int r0, int rows,
                          const float* act, const float* weight, const float* bias, float* lafs, float* angle, float* patches, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Local features -> matcher inputs, and matches -> the compact match list of stand-alone inference.
 *   og_prepare_features  prepare_features_output (models/features/utils.py:54-65) with the LAF -> side-information converter
 *                        superglue.laf_to_sideinfo_method names (models/laf_converter.py:108-128).  One thread per keypoint.
 *                        lafs [R,2,3] = [[a00, a01, x], [a10, a11, y]];  s = sqrt(|(a00 a11 - a10 a01) + 1e-10|) (kornia get_laf_scale)
 *                          kpts [R,2] = (x, y)  (may be NULL: not written)
 *                          side [R, (responses ? 1 : 0) + dim]:  r, or log(r + 0.1) when log_response  (responses NULL: no column),
 *                          then by method:  NONE  -                                              (dim 0)
 *                                           SCALE  log s                                         (dim 1)
 *                                           ROTATION  a01/s, a00/s                               (dim 2)
 *                                           SCALE_ROTATION  log s, a01/s, a00/s                  (dim 3)
 *                                           AFFINE  log s, a00/s, a01/s, a10/s, a11/s            (dim 5)
 *                        Separately rounded IEEE operations in ATen's order (no FMA contraction): every column except the
 *                        logarithms equals the reference's fp32 result bit for bit (where ATen's square root is correctly
 *                        rounded: its vectorised CPU form is 1 ulp off on a few frames in a thousand).
 *   og_match_compact     the boolean indexing of OpenGlueMatcher.forward (inference.py:192-209) on og_match_fwd's output: every
 *                        (b, i) with matches0[b, i] >= 0, in pair-major then i order (deterministic) ->
 *                          pair [B n] int64 (batch_indexes), ij [B n, 2] int64 (i, j = original_matching_idxs),
 *                          confidence [B n] = mscores0[b, i], out_lafs0/1 [B n, 2, 3] = lafs0[b, i] / lafs1[b, j],
 *                          out_kpts0/1 [B n, 2] = their centres;  total [1] int64 = the number of matches (rows past it are
 *                          not written).  matches0 [B,n] int64, mscores0 [B,n], lafs0 [B,n,2,3], lafs1 [B,m,2,3].
 *                        The predicate is matches0 >= 0, never the score: a mutual match whose exp underflowed to 0 is kept
 *                        when the threshold is negative.
 *   og_keypoint_counts   the kept keypoints of each image of a front-end output padded to K rows, on the device: of count[b]
 *                        keypoints the first min(count[b], cap) were stored; max_keypoints >= 0 below that number keeps the
 *                        max_keypoints best (mode[b] = 1), otherwise all are kept in stored order (mode[b] = 0); n_out[b] = the
 *                        kept number clamped to K; overflow[b] |= 1 when count[b] > cap or the kept number exceeds K (the caller
 *                        initialises overflow).  count, n_out, mode (may be NULL), overflow: int32 [B].
 *   og_mask_empty_pairs  matches0 / mscores0 [B,n] and matches1 / mscores1 [B,m] (og_match_fwd_padded's outputs) = -1 / 0 in every
 *                        slot of a pair whose len0[b] or len1[b] (int32 [B], device) is 0: the padded kernels clamp lengths to
 *                        at least 1, so they match row 0 of an image without keypoints.                               */
typedef enum og_laf_method {
  OG_LAF_NONE = 0, OG_LAF_SCALE = 1, OG_LAF_ROTATION = 2, OG_LAF_SCALE_ROTATION = 3, OG_LAF_AFFINE = 4
} og_laf_method;
int og_prepare_features(const float* lafs, const float* responses, int64_t R, int method, int log_response, float* kpts, float* side,
                        void* stream);
int og_match_compact(const int64_t* matches0, const float* mscores0, const float* lafs0, const float* lafs1, int B, int n, int m,
                     int64_t* pair, int64_t* ij, float* confidence, float* out_lafs0, float* out_lafs1, float* out_kpts0,
                     float* out_kpts1, int64_t* total, void* stream);
int og_keypoint_counts(const int* count, int B, int cap, int max_keypoints, int K, int* n_out, int* mode, int* overflow, void* stream);
int og_mask_empty_pairs(const int* len0, const int* len1, int B, int n, int m, int64_t* matches0, float* mscores0, int64_t* matches1,
                        float* mscores1, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Homography-pretraining image pairs (OxfordParis1MDataset.__getitem__, data/oxford_paris_dataset.py:27-66, without the decode,
 * the INTER_AREA resize and the colour augmentation).  One launch for B images:
 *   rgb [B,H,W,3] uint8 (rows of 3 W bytes, no alignment required);  warp_offset [B,4,2] int32 device, (x, y) per corner in the
 *   order (off, off), (off, H-off-1), (W-off-1, off), (W-off-1, H-off-1), each in [-offset, offset) (the caller checks the range)
 *   -> image0 [B,h,w] fp32 = gray(crop) / 255,  image1 [B,h,w] = gray(crop(warpPerspective(rgb, H_warp))) / 255,
 *      H_true [B,3,3] fp32 (the homography relating the crops),  h = H - 2 offset, w = W - 2 offset.
 *   cv2's arithmetic throughout (getPerspectiveTransform by LU, warpPerspective's fixed-point INTER_LINEAR with a constant-0
 *   border, cvtColor RGB2GRAY): equal to cv2 4.13 bit for bit wherever its LU solve succeeds.  A pivot below 100 DBL_EPSILON
 *   gives H = [[0,0,0],[0,0,0],[0,0,1]] (OpenCV's LU rule; cv2 4.13 falls back to an SVD there instead); no error is reported.
 *   OG_EINVAL without a launch: a null pointer, B outside [1, 65535], offset < 1 or 2 offset >= min(H, W).                   */
int og_homography_pairs(const uint8_t* rgb, int B, int H, int W, int offset, const int32_t* warp_offset, float* image0, float* image1,
                        float* H_true, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Optimiser step of the reference's training loop (train.py, train_cached.py, pretrain_homography.py under Lightning):
 *   torch.nn.utils.clip_grad_norm_(params, max_norm) -> torch.optim.Adam.step() -> StepLR(step_size=1, gamma).step()
 * (models/matching_module.py:133-147; Lightning's gradient_clip_val), in one call of two kernels and with no host
 * synchronisation, so that it can be captured in a CUDA graph.
 *   segments  device table of nseg og_optim_segment: every fp32 parameter with a gradient, its Adam moments and its step
 *             count (torch's per-parameter state['step']).  Segment s covers tiles tile0 .. tile0 + ceil(numel / OG_OPTIM_TILE) - 1
 *             of the step; tile0 starts at 0 and runs on without gaps; ntiles = the total.  Pointers need 4-byte alignment;
 *             a segment whose four arrays are 16-byte aligned runs the vector path.
 *   state     og_optim_state: lr (read, then multiplied by lr_gamma), grad_norm / clip_coef (written), sched_steps
 *             (incremented).  Zero-fill it once and set lr before the first call; the CTA counter is reset by the kernel.
 *   workspace >= og_optim_workspace_bytes(nseg), 8-byte aligned.
 * Per element, torch's foreach arithmetic, bit for bit (same rounding points and FMA contractions):
 *   g *= clip_coef (written back);  m = lerp(m, g, 1 - beta1);  v = v beta2 + (1 - beta2) g g;
 *   p += step_size (m / (sqrt(v) / bc2_sqrt + eps))
 * with clip_coef = min(max_norm / (norm + 1e-6), 1) in fp32 (NaN norm -> NaN), the norm a deterministic fp64 reduction
 * rounded once to fp32, and per segment step += 1, bc1 = 1 - beta1^step, bc2_sqrt = (1 - beta2^step)^0.5,
 * step_size = -lr / bc1 in fp64, rounded once to fp32.
 * OG_EINVAL without touching the GPU: null pointers, nseg or ntiles <= 0, max_norm <= 0, beta outside [0, 1), eps < 0,
 * lr_gamma <= 0, a small workspace (OG_EWORKSPACE).
 * og_clip_adam_step_guarded: the same step behind a device int32 flag `skip` (NULL: og_clip_adam_step).  When *skip != 0
 * only the gradients are written, with 0: parameters, moments, step counts, lr, grad_norm and sched_steps keep their bits.
 * og_adam_schedule (tests): the same device-derived scalars for steps 1 .. nsteps from an initial lr:
 * lr_out[k] = the lr of step k + 1, step_size[k] / bc2_sqrt[k] its fp32 scalars.                        */
#define OG_OPTIM_TILE 2048
typedef struct og_optim_segment {
  float* param; float* grad; float* exp_avg; float* exp_avg_sq;
  float* step;                  /* one fp32 step count                                               */
  int64_t numel;
  int64_t tile0;
} og_optim_segment;
typedef struct og_optim_state {
  double   lr;
  float    grad_norm;           /* what clip_grad_norm_ returns                                      */
  float    clip_coef;
  uint32_t counter;             /* CTA counter of the norm kernel: zero between calls               */
  uint32_t sched_steps;         /* scheduler steps taken (StepLR's last_epoch): +1 per call          */
} og_optim_state;
int64_t og_optim_state_bytes(void);
int64_t og_optim_workspace_bytes(int nseg);
int og_clip_adam_step(const og_optim_segment* segments, int nseg, int64_t ntiles, double beta1, double beta2, double eps,
                      double max_norm, double lr_gamma, og_optim_state* state, void* workspace, int64_t workspace_bytes, void* stream);
int og_clip_adam_step_guarded(const og_optim_segment* segments, int nseg, int64_t ntiles, double beta1, double beta2, double eps,
                              double max_norm, double lr_gamma, og_optim_state* state, void* workspace, int64_t workspace_bytes,
                              const int* skip, void* stream);
int og_adam_schedule(int64_t nsteps, double lr, double lr_gamma, double beta1, double beta2, double* lr_out, float* step_size,
                     float* bc2_sqrt, void* stream);

#ifdef __cplusplus
}
#endif
#endif  /* OPENGLUE_B200_H_ */
