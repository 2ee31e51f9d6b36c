/* pf_b200.h — C ABI of libpf_b200.so: the H100 (sm_90a) kernels behind PocketFlow's
 * compression-aware training step.
 *
 * The reference (Tencent/PocketFlow) has no FFI: its de-facto operator boundary is the set of
 * private learner methods that emit TensorFlow op chains.  Each entry point below replaces one
 * such chain; the comment above it cites the reference file:line it stands in for.
 *
 * Conventions (SURVEY.md §8b):
 *   - every function returns int: 0 = ok, <0 = pf_status, >0 = cudaError_t;
 *     pf_last_error() returns a thread-local human-readable message for the last failure.
 *   - the caller owns every buffer (inputs, outputs, workspaces, descriptor tables); kernels
 *     never allocate.  Pointers named *_dev are device pointers; `stream` is a cudaStream_t
 *     passed as void* (0 = legacy default stream).
 *   - all calls are asynchronous with respect to the host (enqueue only) unless stated.
 *   - fp32 everywhere ("u32"/"u8" where noted); tensors are dense, NHWC activations,
 *     HWIO ([kh,kw,cin,cout]) kernels — the TF layouts the reference uses.
 *   - there is NO CPU fallback anywhere in this library.
 */
#ifndef PF_B200_H_
#define PF_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PF_B200_ABI_VERSION 1

typedef enum pf_status {
  PF_OK = 0,
  PF_ERR_INVALID_ARG = -1,  /* bad size / null pointer / unsupported mode (Python raises ValueError) */
  PF_ERR_UNSUPPORTED = -2,  /* shape outside what the kernel implements                              */
  PF_ERR_NO_DEVICE = -3,    /* no CUDA device / driver                                              */
  PF_ERR_NCCL = -4,         /* NCCL missing or returned an error                                    */
  PF_ERR_INTERNAL = -5
} pf_status;

int pf_abi_version(void);
const char* pf_last_error(void);
/* Number of kernel launches this library has enqueued in this process (bench.py "gpu_launches"). */
int64_t pf_launch_count(void);
void pf_launch_count_reset(void);
/* Device query helper: SM count of the current device (132 on H100 SXM). */
int pf_sm_count(int* out);

/* ---------------------------------------------------------------------------------------------
 * Ordered-uint encoding of float min/max slots.  enc(f) is monotone in f, so atomicMin/atomicMax
 * on uint32 implement float min/max.  A min slot starts at 0xFFFFFFFF, a max slot at 0.
 *   enc(f) = bits(f) ^ (bits(f) >> 31 ? 0xFFFFFFFF : 0x80000000)
 * ------------------------------------------------------------------------------------------- */

/* ---------------------------------------------------------------------------------------------
 * a1  Weight fake-quantization, multi-tensor (one launch pair for every layer).
 *     Replaces UniformQuantization.__uniform_quantize(mode='weight') + __scale + __inv_scale +
 *     __channel_bucket / __split_bucket — learners/uniform_quantization/utils.py:163-289.
 *
 *     Every tensor is described by one pf_uq_seg.  Bucket id of flat element i is (i % ncols):
 *       per-layer  (use_buckets=False): ncols = 1,              padded = numel
 *       'channel'  (reshape [-1,cout], reduce axis 0): ncols = cout, padded = numel
 *       'split'    (pad with copies of the LAST element to a multiple of bucket_size, reshape
 *                   [bucket_size,-1], reduce axis 0): ncols = padded/bucket_size; elements
 *                   i in [numel,padded) read src[numel-1]   (utils.py:247-274: strided buckets)
 *     qw = alpha*(rint((w-beta)/alpha*k)/k)+beta, alpha=(max-min)+1e-10f, beta=min,
 *     k=float(2^bits-1); round-half-even; every op individually rounded (no FMA contraction).
 * ------------------------------------------------------------------------------------------- */
typedef struct pf_uq_seg {
  const float* src;   /* device; 16-byte aligned                                  */
  float* dst;         /* device; 16-byte aligned; may equal src                   */
  int64_t numel;      /* < 2^31                                                    */
  int64_t padded;     /* >= numel; multiple of ncols                               */
  int32_t ncols;      /* number of buckets of this tensor                          */
  int32_t bucket0;    /* first slot of this tensor in mn_enc/mx_enc (multiple of 4)*/
  int32_t bits;       /* 1..32                                                     */
  int32_t reserved;
} pf_uq_seg;

/* One unit of CTA work.  kind 0: flat chunk [start, start+count) of seg (elementwise kernels and
 * per-layer min/max).  kind 1: column tile for bucketed min/max: columns [c0, c0+ncol_tile),
 * rows [start, start+count) of the [padded/ncols, ncols] view. */
typedef struct pf_work {
  int32_t seg;
  int32_t kind;
  int64_t start;
  int32_t count;
  int32_t c0;
  int32_t ncol_tile;
  int32_t reserved;
} pf_work;

/* Phase 1: per-bucket min/max into ordered-uint slots (caller pre-fills mn_enc with 0xFF bytes and
 * mx_enc with 0 — pf_fill_u32 does both).  work table = kind-0 chunks (per-layer) / kind-1 tiles. */
int pf_uq_weight_minmax(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work,
                        uint32_t* mn_enc_dev, uint32_t* mx_enc_dev, void* stream);
/* Phase 1b: scales_dev[0..n) = alpha = (max-min)+1e-10f, [n..2n) = beta = min, [2n..3n) = RN(1/alpha)
 * (n = n_buckets, a multiple of 4).  The reciprocal feeds an exact (correctly rounded) division by
 * residual correction, so results stay bit-identical to true fp32 division. */
int pf_uq_weight_scales(const uint32_t* mn_enc_dev, const uint32_t* mx_enc_dev, int n_buckets,
                        float* scales_dev, void* stream);
/* Phase 2: quantize.  work table: kind-0 chunks.  (The second read of the weights is an L2 hit:
 * all weights of ResNet-50 are 94 MB < 126 MB L2.) */
int pf_uq_weight_quant(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work,
                       const float* scales_dev, int n_buckets, void* stream);
/* a3  STE backward of the weight quantizer as a stand-alone op, in place on the gradient:
 *     g <- (((g*alpha)/k)*k)/alpha   (gradient_override_map Round->Identity, utils.py:185-186;
 *     min/max under stop_gradient, :224-225).  segs[i].src/dst point at the gradient. */
int pf_uq_weight_ste_bwd(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work,
                         const float* scales_dev, int n_buckets, void* stream);

/* a2  Activation fake-quantization (per-TENSOR min/max, utils.py:51-79, 215-231).
 *     minmax: accumulates into minmax_enc_dev[0] (min) / [1] (max) (pre-filled 0xFFFFFFFF / 0).
 *     quant : y = Q(x) with the scalar range; src may equal dst. */
int pf_uq_act_minmax(const float* x_dev, int64_t n, uint32_t* minmax_enc_dev, void* stream);
int pf_uq_act_quant(const float* x_dev, float* y_dev, int64_t n, const uint32_t* minmax_enc_dev,
                    int bits, void* stream);
/* same, (also) writing y as split-bf16 planes for the tensor-core conv that consumes it (y_dev may be NULL) */
int pf_uq_act_quant_planes(const float* x_dev, float* y_dev, void* y_hi_dev, void* y_lo_dev, int64_t n,
                           const uint32_t* minmax_enc_dev, int bits, void* stream);
/* static range (a calibrated model): y = Q(clamp(x, lo, hi)) with range_enc_dev[0..1] = the encoded lo / hi, written
 * once by the caller; one pass, no range pass.  Bit-identical to pf_uq_act_quant when lo / hi is x's own range. */
int pf_uq_act_quant_static(const float* x_dev, float* y_dev, int64_t n, const uint32_t* range_enc_dev, int bits,
                           void* stream);

int pf_fill_u32(uint32_t* p_dev, int64_t n, uint32_t value, void* stream);
/* (min,max) ordered-uint pairs <- (0xFFFFFFFF, 0): one launch resets every activation range slot. */
int pf_minmax_reset(uint32_t* pairs_dev, int64_t n_pairs, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a5  Magnitude-threshold mask build, multi-tensor.
 *     Replaces WeightSparseLearner.__build_masks — learners/weight_sparsification/learner.py:260-294:
 *        bkup = where(mask > 0.5, w, bkup); thr = percentile(|bkup|, 100*s) ('nearest': the
 *        element at index rank_desc of the DESCENDING sort); mask = float(|bkup| > thr);
 *        w = bkup*mask.
 *     The order statistic is found exactly by a 4-pass radix select on the IEEE bit pattern of
 *     |bkup| (no sort, no approximation) so masks are bit-exact.
 *     ranks_desc_dev[i] = clip(int32(rint((n-1)*(1-q/100))),0,n-1), computed on the host in
 *     float64 exactly as tf.contrib.distributions.percentile does.
 *     workspace_dev: n_seg * PF_WS_WORKSPACE_U32_PER_SEG uint32 (zeroed by the call).
 *     thr_out_dev (optional, n_seg floats) receives each tensor's threshold.
 * ------------------------------------------------------------------------------------------- */
typedef struct pf_ws_seg {
  float* w;
  float* bkup;
  float* mask;
  int64_t numel;
} pf_ws_seg;
#define PF_WS_WORKSPACE_U32_PER_SEG (256 + 8)

int pf_ws_mask_build(const pf_ws_seg* segs_dev, int n_seg, const pf_work* work_dev, int n_work,
                     const int64_t* ranks_desc_dev, uint32_t* workspace_dev, float* thr_out_dev,
                     void* stream);

/* Exact k-th order statistic of plain values (not |.|), multi-tensor, used by the codebook
 * quantile initialisation (learners/nonuniform_quantization/utils.py:349-366).  Query q reads
 * segs[qseg[q]].bkup (numel floats) and returns the element at descending index ranks_desc[q]. */
int pf_select_desc(const pf_ws_seg* segs_dev, const int32_t* qseg_dev, int n_query,
                   const pf_work* work_dev, int n_work, /* work[].seg indexes QUERIES */
                   const int64_t* ranks_desc_dev, uint32_t* workspace_dev, float* out_dev,
                   void* stream);

/* ---------------------------------------------------------------------------------------------
 * a6/a9  Fused optimizer steps over flat fp32 ranges.
 *   momentum: replaces __calc_grads_pruned (weight_sparsification/learner.py:314-332) +
 *     MomentumOptimizer.apply_gradients (:201,:212), with the Horovod average
 *     (utils/multi_gpu_wrapper.py:82-89) and the l2_loss gradient folded in:
 *        gt = g*grad_scale + wd*w ; gt *= mask (if mask) ; acc = acc*mom + gt ; w -= lr*acc
 *   adam: TF-1.x ApplyAdam (uniform_quantization/learner.py:244):
 *        gt as above (no mask); alpha = lr*sqrt(1-b2p)/(1-b1p);
 *        m += (gt-m)*(1-b1); v += (gt*gt-v)*(1-b2); w -= (m*alpha)/(sqrt(v)+eps)
 *   lr/b1p/b2p are read from device scalars (hp_dev) so the step is CUDA-graph replayable:
 *     momentum: hp_dev[0]=lr ; adam: hp_dev[0]=lr, [1]=beta1_power, [2]=beta2_power.
 * ------------------------------------------------------------------------------------------- */
int pf_momentum_step(float* w_dev, float* acc_dev, const float* g_dev, const float* mask_dev,
                     int64_t n, const float* hp_dev, float momentum, float wd, float grad_scale,
                     void* stream);
int pf_adam_step(float* w_dev, float* m_dev, float* v_dev, const float* g_dev, int64_t n,
                 const float* hp_dev, float beta1, float beta2, float eps, float wd,
                 float grad_scale, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a7/a8  Losses.
 *   pf_softmax_ce_fwd_bwd replaces tf.losses.softmax_cross_entropy(onehot, logits)
 *     (nets/resnet_at_cifar10.py:104) and DistillationHelper.calc_loss
 *     (learners/distillation_helper.py:86-103) in one pass over the N x K logits:
 *        hard = mean_n CE(labels_n, s_n)
 *        dst  = w_dst * mean_n CE(softmax(t_n/T), s_n/T)        (teacher_dev may be NULL)
 *        dlogits = d(hard+dst)/ds ; correct_n = [argmax labels == argmax s]
 *     out_dev[0]=hard, [1]=dst, [2]=accuracy (top-1), [3]=top-5 accuracy.
 *     row_ws_dev: 4*N floats of scratch.  Deterministic (fixed-order final reduction).
 *   pf_l2_loss: out_dev[0] = scale * sum(v^2)/2 over a flat range (tf.nn.l2_loss summed by add_n,
 *     nets/resnet_at_cifar10.py:105-107).  partial_ws_dev: PF_L2_PARTIALS floats.
 * ------------------------------------------------------------------------------------------- */
int pf_softmax_ce_fwd_bwd(const float* logits_dev, const float* labels_dev,
                          const float* teacher_dev, int n, int k, float tempr, float w_dst,
                          float* dlogits_dev, float* out_dev, float* row_ws_dev, void* stream);
#define PF_L2_PARTIALS 1024
int pf_l2_loss(const float* v_dev, int64_t n, float scale, int accumulate, float* out_dev,
               float* partial_ws_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a11 Codebook (non-uniform) weight quantization, multi-tensor, per-layer range.
 *     Replaces NonUniformQuantization.__nonuni_quantize / __build_norm_quant_point —
 *     learners/nonuniform_quantization/utils.py:168-194, 284-307:
 *        xn=(w-beta)/alpha; idx=argmin_j|xn-c_j| (first index on ties);
 *        q=c[idx]*sign(xn+1e-6); out=alpha*q+beta.
 *     Uses pf_uq_seg (ncols must be 1; bits = log2(#centroids) <= 8) and the scales of
 *     pf_uq_weight_minmax + pf_uq_weight_scales.  clusters_dev: per seg 2^bits floats at offset seg*256.
 *     idx_out_dev (optional): uint8 centroid index per element, laid out like the weights
 *     (idx_base_dev[seg] = byte offset of the tensor), for the codebook gradient.
 * ------------------------------------------------------------------------------------------- */
int pf_nuq_weight_quant(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work,
                        const float* scales_dev, int n_buckets,
                        const float* clusters_dev, uint8_t* idx_out_dev,
                        const int64_t* idx_base_dev, void* stream);
/* same, with the codebook of tensor `seg` at clusters_base_dev + cluster_off_dev[seg] (floats): codebooks that live
 * among the model's trainable variables (the reference's `clusters` variables, utils.py:297) */
int pf_nuq_weight_quant_ex(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work,
                           const float* scales_dev, int n_buckets, const float* clusters_base_dev,
                           const int64_t* cluster_off_dev, uint8_t* idx_out_dev, const int64_t* idx_base_dev,
                           void* stream);
/* f4  Codebook gradient of the `cluster` / `both` optimisation modes (learners/nonuniform_quantization/
 *     learner.py:252-261): backward of tf.gather(c, min_index) under the Mul->Add / Sign->Identity override
 *     (utils.py:303-306) through the inverse scale alpha*q+beta (:433):
 *        dL/dc_j = alpha * sum_{i : idx_i = j} g_i ,   g = gradient w.r.t. the quantized tensor.
 *     gsegs[i].src = g of tensor i (numel floats; bits, bucket0 as in the forward's segs); work: kind-0 chunks, all
 *     chunks of a tensor contiguous, work_first_dev[seg .. seg+1) = its range (n_seg + 1 entries); idx/idx_base: what
 *     pf_nuq_weight_quant wrote; partial_ws_dev: n_work * 256 floats; result at grad_base_dev + cluster_off_dev[seg].
 *     Deterministic (fixed-order two-stage reduction). */
int pf_nuq_cluster_grad(const pf_uq_seg* gsegs_dev, int n_seg, const pf_work* work_dev, int n_work,
                        const int32_t* work_first_dev, const uint8_t* idx_dev, const int64_t* idx_base_dev,
                        const float* scales_dev, float* partial_ws_dev, float* grad_base_dev,
                        const int64_t* cluster_off_dev, void* stream);

/* f5  Bucketed codebooks (NonUniformQuantization.__bucket_quantize, utils.py:196-243).  segs as for the bucketed
 *     pf_uq_weight_minmax (ncols = nb buckets, bucket of flat element i = i % nb, split padding = copies of the last
 *     element), scales from pf_uq_weight_minmax + pf_uq_weight_scales on those segs.  The codebook of bucket b of
 *     tensor seg is column b of a [K, nb] matrix: c[j, b] = clusters_base[cluster_off[seg] + j * nb + b], K >= 2^bits.
 *     Quantize / gradient work: kind-1 tiles (columns [c0, c0 + ncol_tile), rows [start, start + count)) with
 *     ncol_tile <= min(256, 8192 / 2^bits); the tile's codebooks are staged in shared memory.  Only the real elements
 *     (flat index < numel) are quantized, indexed and differentiated. */
#define PF_NUQ_BUCKET_MAX_ROWS 16384
int pf_nuq_bucket_quant(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work, const float* scales_dev,
                        int n_buckets, const float* clusters_base_dev, const int64_t* cluster_off_dev,
                        uint8_t* idx_out_dev, const int64_t* idx_base_dev, void* stream);
/* c[j, b] = (sorted_b[pos[seg*256 + j]] - beta_b) / alpha_b for j < 2^bits, 0 for 2^bits <= j < K: exact order
 *     statistics of every bucket (its padded rows included).  work: one item per bucket, seg, c0 = bucket,
 *     count = rows of the bucket (<= PF_NUQ_BUCKET_MAX_ROWS = max_rows bound), ncol_tile = K.  pos: ascending
 *     positions, 256 per seg. */
int pf_nuq_bucket_quantile_init(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work, int max_rows,
                                const int32_t* pos_dev, const float* scales_dev, int n_buckets,
                                float* clusters_base_dev, const int64_t* cluster_off_dev, void* stream);
/* dL/dc[j, b] = alpha_b * sum_{i in b, i < numel, idx_i = j} g_i.  work = the quantize tiles, each with
 *     reserved = float offset of its 2^bits * ncol_tile partials in partial_ws_dev; tiles_dev: one item per column
 *     tile, start / count = its range of `work` (row order), c0 / ncol_tile as there.  Deterministic. */
int pf_nuq_bucket_cluster_grad(const pf_uq_seg* gsegs_dev, const pf_work* work_dev, int n_work,
                               const pf_work* tiles_dev, int n_tiles, const uint8_t* idx_dev,
                               const int64_t* idx_base_dev, const float* scales_dev, float* partial_ws_dev,
                               float* grad_base_dev, const int64_t* cluster_off_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a4  Convolution / dense layers, exact-fp32 CUDA-core path (pf_conv.cu).
 *     Replaces tf.nn.conv2d / tf.matmul re-created on the quantized weight
 *     (learners/uniform_quantization/utils.py:88-113) and their autodiff (learner.py:247).
 *     x: NHWC [n,h,w,c]; w: HWIO [r,s,c,k]; y: NHWC [n,p,q,k]; pad_t/pad_l = leading padding
 *     (TF 'SAME': pad_total//2; fixed_padding: (k-1)//2 — utils/external/resnet_model.py:71-103).
 *     A dense layer is the h=w=r=s=1 case.
 * ------------------------------------------------------------------------------------------- */
typedef struct pf_conv_desc {
  int32_t n, h, w, c;      /* input  */
  int32_t k, r, s;         /* filters, kernel height/width */
  int32_t p, q;            /* output height/width */
  int32_t stride_h, stride_w, pad_t, pad_l;
} pf_conv_desc;            /* HOST struct, passed by pointer */
#define PF_CONV_WGRAD_MAX_SPLITS 64
#define PF_BN_MAX_SPLITS 1024

/* cols[m][k] (m = output pixel, k = (r*S+s)*C + c, zero-padded to kpad columns): explicit im2col for
 * first layers whose Cin (3) the tensor-core path cannot take; the conv then runs as a 1x1 conv over
 * kpad channels. */
int pf_im2col(const pf_conv_desc* d, const float* x_dev, int kpad, float* cols_dev, void* stream);
/* Space-to-depth form of a stride-2 first layer: x' [n, hp, wp, cpad] (split-bf16 planes) with
 * x'[.., y', x', (dy*2+dx)*c + cc] = x[.., 2y'+dy-pad_t, 2x'+dx-pad_l, cc]; the RxS stride-2 conv equals a stride-1
 * ceil(R/2) x ceil(S/2) conv over x' whose kernel rows are re-arranged with pf_gather_rows (idx < 0: zero row). */
int pf_s2d_planes(const float* x_dev, int n, int h, int w, int c, int pad_t, int pad_l, int hp, int wp, int cpad,
                  void* hi_dev, void* lo_dev, void* stream);
int pf_gather_rows(const float* src_dev, const int32_t* idx_dev, int n_rows, int row_len, float* dst_dev, void* stream);
/* same, written directly as split-bf16 operand planes [N*P*Q, kpad] (kpad % 8 == 0) */
int pf_im2col_planes(const pf_conv_desc* d, const float* x_dev, int kpad, void* cols_hi_dev, void* cols_lo_dev,
                     void* stream);
/* y = conv(x, w) (+ bias[k]) (relu if relu != 0) */
int pf_conv2d_fwd(const pf_conv_desc* d, const float* x_dev, const float* w_dev, const float* bias_dev,
                  int relu, float* y_dev, void* stream);
/* dx (+)= conv_transpose(dy, w).  wt_ws_dev: r*s*c*k floats of scratch (per-tap transposed weight). */
int pf_conv2d_dgrad(const pf_conv_desc* d, const float* dy_dev, const float* w_dev, float* wt_ws_dev,
                    int accumulate, float* dx_dev, void* stream);
/* dw = x (*) dy, split-K with a fixed-order reduction (deterministic).
 * ws_dev: pf_conv2d_wgrad_workspace_bytes(d) bytes. */
int64_t pf_conv2d_wgrad_workspace_bytes(const pf_conv_desc* d);
int pf_conv2d_wgrad(const pf_conv_desc* d, const float* x_dev, const float* dy_dev, float* ws_dev,
                    float* dw_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a4  Convolution forward / dgrad on the Hopper tensor cores (wgmma, pf_conv_tc.cu), same semantics as
 *     pf_conv2d_fwd / pf_conv2d_dgrad.  fp32 operands are split x = hi + lo (bf16 each) and each
 *     k-slice issues hi*hi + hi*lo + lo*hi into one fp32 register accumulator (error ~2^-17 relative).
 *     Requires Cin % 16 == 0 and Cout % 16 == 0 (pf_conv2d_tc_supported).
 *     Weights are pre-split and laid out K-major once per step by pf_conv2d_tc_prep_weight into
 *     caller-owned bf16 buffers of pf_conv2d_tc_weight_elems(d, dgrad) elements each, which the caller
 *     zero-fills ONCE at allocation (padding columns are never written).
 * ------------------------------------------------------------------------------------------- */
int pf_conv2d_tc_supported(const pf_conv_desc* d);
int64_t pf_conv2d_tc_weight_elems(const pf_conv_desc* d, int dgrad);
int pf_conv2d_tc_prep_weight(const pf_conv_desc* d, const float* w_dev, void* fwd_hi_dev, void* fwd_lo_dev,
                             void* dgrad_hi_dev, void* dgrad_lo_dev, void* stream);
/* y = conv(x, w) (+ bias) (relu) (+ residual_dev: the fused residual add of resnet_model.py:199,314;
 * NULL = none) */
int pf_conv2d_tc_fwd(const pf_conv_desc* d, const float* x_dev, const void* w_hi_dev, const void* w_lo_dev,
                     const float* bias_dev, int relu, const float* residual_dev, float* y_dev, void* stream);
int pf_conv2d_tc_dgrad(const pf_conv_desc* d, const float* dy_dev, const void* wd_hi_dev, const void* wd_lo_dev,
                       int accumulate, float* dx_dev, void* stream);
/* multi-tensor weight preparation: every conv kernel of a network in ONE launch.  segs: one entry per kernel
 * (kpad = pf_conv2d_tc_weight_elems / rows; dgrad pointers may be NULL), work: one item per 32 x 64 tile of the
 * [R*S*Cin, Cout] matrix (start = first row, c0 = first column). */
typedef struct pf_tc_prep_seg {
  const float* w;          /* HWIO fp32 */
  void* fwd_hi;
  void* fwd_lo;
  void* dgrad_hi;
  void* dgrad_lo;
  int32_t rs, c, k;        /* R*S, Cin, Cout */
  int32_t kpad_f, kpad_d;  /* row pitches of the fwd / dgrad copies (multiples of 64) */
  int32_t q_bits;          /* 0: w holds the values to split.  1..8: w holds the UNQUANTIZED kernel and the copies are
                            * derived with the weight quantizer's own op chain (a1): fwd_hi <- bf16(level - 2^(bits-1))
                            * (integer levels, fwd_lo untouched), dgrad_hi / dgrad_lo <- split of the quantized value */
  const float* q_alpha;    /* bucket scales of pf_uq_weight_scales at this tensor's first bucket: alpha, */
  const float* q_beta;     /*   beta, */
  const float* q_ralpha;   /*   RN(1 / alpha) */
  int32_t q_ncols;         /* 1 (per layer) or k (per output channel) */
  int32_t reserved;
} pf_tc_prep_seg;
int pf_conv2d_tc_prep_weights_multi(const pf_tc_prep_seg* segs_dev, const pf_work* work_dev, int n_work, void* stream);
/* dw = x (*) dy on the tensor cores (MN-major operands, split-K with a fixed-order reduction).
 * Requires Cin % 16 == 0 and Cout % 64 == 0; ws_dev: pf_conv2d_tc_wgrad_workspace_bytes(d) bytes. */
#define PF_CONV_TC_WGRAD_MAX_SPLITS 148
int pf_conv2d_tc_wgrad_supported(const pf_conv_desc* d);
int64_t pf_conv2d_tc_wgrad_workspace_bytes(const pf_conv_desc* d);
int pf_conv2d_tc_wgrad(const pf_conv_desc* d, const float* x_dev, const float* dy_dev, float* ws_dev,
                       float* dw_dev, void* stream);
/* fp32 -> split-bf16 planes: hi = bf16(x), lo = bf16(x - hi) (n % 8 == 0, 16-byte aligned); the operand format of
 * the tensor-core kernels.  pf_conv2d_tc_wgrad splits x and dy into its workspace and then runs the same
 * persistent kernel as pf_conv2d_tc_wgrad_planes, which takes operands that are already split. */
int pf_split_bf16(const float* src_dev, void* hi_dev, void* lo_dev, int64_t n, void* stream);
int64_t pf_conv2d_tc_wgrad_planes_workspace_bytes(const pf_conv_desc* d);   /* split-K partials only */
/* the same fwd / dgrad kernels with the activation operand already split (written by pf_bn_apply_planes,
 * pf_uq_act_quant_planes, pf_bn_bwd_planes or pf_split_bf16): producers are pure cp.async copies */
int pf_conv2d_tc_fwd_planes(const pf_conv_desc* d, const void* x_hi_dev, const void* x_lo_dev, const void* w_hi_dev,
                            const void* w_lo_dev, const float* bias_dev, int relu, const float* residual_dev,
                            float* y_dev, void* stream);
int pf_conv2d_tc_dgrad_planes(const pf_conv_desc* d, const void* dy_hi_dev, const void* dy_lo_dev, const void* wd_hi_dev,
                              const void* wd_lo_dev, int accumulate, float* dx_dev, void* stream);
/* Inference-mode batch norm of the conv's output, applied in the forward epilogue: after bias, ReLU and the residual
 * add, the value stored to y_dev also goes through act(((v - mean) * rsqrt(var + eps)) * gamma + beta) with the op
 * chain (and rounding) of pf_bn_apply_eval, and is stored as split-bf16 planes and / or fp32.  Bit-identical to the
 * plain forward followed by pf_bn_apply_eval(y_dev, ...); y_dev itself is still written.  Every pointer is a device
 * pointer: the four per-channel vectors ([Cout] each) and y 16-byte aligned, the planes 8-byte aligned. */
typedef struct pf_tc_bn_out {
  const float* mean;       /* moving mean */
  const float* var;        /* moving variance */
  const float* gamma;
  const float* beta;
  float eps;               /* >= 0 */
  int32_t act;             /* 0 none, 1 ReLU, 2 ReLU6 */
  float* y;                /* post-BN fp32 tensor, or NULL */
  void* hi;                /* post-BN split-bf16 planes (layout of y_dev), or NULL; at least one of y / hi */
  void* lo;
} pf_tc_bn_out;
int pf_conv2d_tc_fwd_bn(const pf_conv_desc* d, const float* x_dev, const void* w_hi_dev, const void* w_lo_dev,
                        const float* bias_dev, int relu, const float* residual_dev, float* y_dev, const pf_tc_bn_out* bn,
                        void* stream);
int pf_conv2d_tc_fwd_planes_bn(const pf_conv_desc* d, const void* x_hi_dev, const void* x_lo_dev, const void* w_hi_dev,
                               const void* w_lo_dev, const float* bias_dev, int relu, const float* residual_dev,
                               float* y_dev, const pf_tc_bn_out* bn, void* stream);
/* dw_dev == NULL: leave the split-K partials [splits][R*S*Cin][Cout] in ws_dev (pf_conv2d_tc_wgrad_splits(d) of
 * them) for ONE deferred pf_conv2d_tc_wgrad_reduce_multi over every layer of the step */
typedef struct pf_tc_reduce_seg {
  const float* partial;    /* [splits][n] */
  float* out;              /* [n] */
  int64_t n;               /* multiple of 4 */
  int32_t splits;
  int32_t reserved;
} pf_tc_reduce_seg;
int pf_conv2d_tc_wgrad_splits(const pf_conv_desc* d);
int pf_conv2d_tc_wgrad_reduce_multi(const pf_tc_reduce_seg* segs_dev, const pf_work* work_dev, int n_work, void* stream);
int pf_conv2d_tc_wgrad_planes(const pf_conv_desc* d, const void* x_hi_dev, const void* x_lo_dev, const void* dy_hi_dev,
                              const void* dy_lo_dev, float* ws_dev, float* dw_dev, void* stream);
/* ---- TMA-fed kernels with EXACT quantizer-level operands (pf_conv_tma.cu; SURVEY §7 hard part 1b) ----
 * When channel counts are multiples of 64 the same entry points above feed the tensor cores with TMA
 * (cp.async.bulk.tensor: im2col-mode tensor maps for the NHWC operand, tiled maps for the weight / gradient matrices;
 * PF_TC_FEED=lsu forces the cp.async kernels).  The *_ex entry points additionally accept operands of <= 8-bit
 * fake-quantized tensors as their INTEGER LEVELS, which bf16 represents exactly, so one MMA per k-slice replaces
 * three (two where the other operand is a split-bf16 gradient):
 *   activation (reference: learners/uniform_quantization/utils.py:51-79, 175-199):  qa = scale * level,
 *     plane0 = levels (plane1 unused) when the tensor's minimum is 0, otherwise plane0/plane1 = hi/lo of qa and
 *     scale = 1 — the producer (pf_bn_apply_quant_levels) decides on the device and records it in `hdr`;
 *     csum[pixel][nseg] = sums of the stored plane values over channel segments of min(C,128) (for the rank-1
 *     correction that the weight offset needs: sum_k qa[m,k] over the filter window);
 *   weights (utils.py:81-113, 224-245):  qw = (alpha_c / k) (level - centre) + (beta_c + centre alpha_c / k),
 *     plane0 = bf16(level - centre), centre = 2^(bits-1), k = 2^bits - 1; alpha / beta = the quantizer's bucket
 *     scales (per layer or per output channel).  plane1 != NULL, alpha == NULL: plain split-bf16 weights. */
typedef struct pf_tc_act_hdr {
  float scale;             /* value of one level (1.0 when the planes hold hi / lo) */
  int32_t nplanes;         /* 1: plane0 = integer levels; 2: plane0 / plane1 = hi / lo */
} pf_tc_act_hdr;
typedef struct pf_tc_act {
  const void* plane0;      /* bf16, layout of the fp32 tensor */
  const void* plane1;      /* bf16 or NULL (then hdr must say 1 plane, or hdr == NULL and the tensor is bf16-exact) */
  const pf_tc_act_hdr* hdr;/* device, or NULL: nplanes = (plane1 ? 2 : 1), scale = 1 */
  const float* csum;       /* device [pixels][nseg] or NULL (only needed with weight levels) */
  int32_t nseg;
  int32_t reserved;
} pf_tc_act;
typedef struct pf_tc_wt {
  const void* plane0;      /* bf16 K-major [rows][kpad] as written by pf_conv2d_tc_prep_weight* */
  const void* plane1;      /* lo plane, or NULL with levels */
  const float* alpha;      /* device bucket scales (levels) or NULL */
  const float* beta;
  int32_t per_channel;     /* 1: one bucket per output channel; 0: one per layer */
  int32_t bits;
} pf_tc_wt;
int pf_conv2d_tc_tma_supported(const pf_conv_desc* d, int pass /* 0 fwd, 1 dgrad, 2 wgrad */);
/* producer of a pf_tc_act: Q(act(bn(x))) with a known range (as pf_bn_apply_quant), written as levels / planes +
 * header + channel sums (csum_dev: m * ceil(c / 128) floats).  C must be a power of two >= 16.  y_dev (fp32 copy) may
 * be NULL.  Reference ops: utils/external/resnet_model.py:55-62 + learners/uniform_quantization/utils.py:51-79. */
int pf_bn_apply_quant_levels(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                             const float* gamma_dev, const float* beta_dev, int act, const uint32_t* range_enc_dev,
                             int bits, float* y_dev, void* plane0_dev, void* plane1_dev, pf_tc_act_hdr* hdr_dev,
                             float* csum_dev, void* stream);
/* operand feed of the tensor-core kernels: 1 = TMA where eligible (default), 0 = cp.async everywhere, -1 = back to the
 * PF_TC_FEED environment default.  Process-wide; used by the tests to run both kernels on the same inputs. */
int pf_conv2d_tc_set_feed(int mode);
int pf_conv2d_tc_fwd_ex(const pf_conv_desc* d, const pf_tc_act* x, const pf_tc_wt* w, const float* bias_dev, int relu,
                        const float* residual_dev, float* y_dev, void* stream);
/* dgrad with a pf_tc_act gradient operand.  The weights must be split-bf16 planes (wd->alpha == NULL): dgrad reduces
 * over output channels, along which per-channel weight scales vary, so weight levels cannot be corrected by a column
 * epilogue; they are refused with PF_ERR_INVALID_ARG. */
int pf_conv2d_tc_dgrad_ex(const pf_conv_desc* d, const pf_tc_act* dy, const pf_tc_wt* wd, int accumulate, float* dx_dev,
                          void* stream);
int pf_conv2d_tc_wgrad_ex(const pf_conv_desc* d, const pf_tc_act* x, const pf_tc_act* dy, float* ws_dev, float* dw_dev,
                          void* stream);
/* ---- u8 x u8 inference forward (pf_conv_tma.cu; reference: learners/uniform_quantization/utils.py:92-104, 163-199,
 * the conv of the fake-quantized weight and activation) ----
 * The TMA-fed ping-pong forward with BOTH operands as the uniform quantizers' own unsigned levels, one byte each:
 *   x->plane0 = u8 activation levels q_a in [0, k_a] (layout of the NHWC tensor), x->plane1 = NULL, x->hdr = {scale =
 *   alpha_a / k_a, nplanes = 1} and x->csum / x->nseg = ceil(Cin / 128) per-pixel channel-segment level sums, all written
 *   by pf_bn_eval_levels_u8;  w->plane0 = u8 weight levels q_w in [0, k_w], K-major [Cout][R*S*Cin] (row pitch R*S*Cin),
 *   w->plane1 = NULL, w->alpha / w->beta = the weight quantizer's bucket scales (per layer, or per output channel with
 *   w->per_channel = 1), w->bits = log2(k_w + 1) <= 8.
 * One u8 x u8 -> s32 wgmma per 32-wide k-slice gives S[m,n] = sum_K q_a q_w exactly (K * 255^2 < 2^31 for K < 33,000);
 * the epilogue computes
 *   y[m,n] = (scale * alpha_n / k_w) * S[m,n] + (scale * beta_n) * J[m],   J[m] = sum_K q_a (from csum),
 * rounding only there, then bias, ReLU (relu != 0), the residual (residual_dev) and, with bn != NULL, the folded inference
 * batch norm as pf_conv2d_tc_fwd_bn applies it.  A header with nplanes != 1 (the activation's minimum was not 0, so
 * its values are not scale * level) makes every output NaN.  The shape picks the kernel: where
 * pf_conv2d_u8_supported(d) holds (Cin % 64 == 0, Cout % 64 == 0, strides <= 8, filters <= 16 x 16) the TMA-fed one,
 * otherwise a cp.async-fed one (pf_conv_tc.cu) with the same arithmetic, which needs Cin % 16 == 0, Cout % 16 == 0 and
 * R*S*Cin <= 32768; pf_conv2d_u8_narrow_supported(d) tells whether either kernel takes d. */
int pf_conv2d_u8_supported(const pf_conv_desc* d);
int pf_conv2d_u8_narrow_supported(const pf_conv_desc* d);
int pf_conv2d_u8_fwd(const pf_conv_desc* d, const pf_tc_act* x, const pf_tc_wt* w, const float* bias_dev, int relu,
                     const float* residual_dev, float* y_dev, const pf_tc_bn_out* bn, void* stream);
/* producer of the u8 operand (reference: utils/external/resnet_model.py:55-62 inference BN, then
 * learners/uniform_quantization/utils.py:51-79 with the range of this batch): y = act(bn(x)) with the moving statistics
 * (pf_bn_apply_eval's op chain), quantized per tensor, written as levels rint(((y - min) / alpha) * k) into levels_dev
 * (m * c bytes) + hdr + csum (m * ceil(c / 128) floats).  have_range = 0: range_enc_dev[0..1] is reset and filled with
 * min / max of y first (a pass of its own: the whole range is needed before any level); 1: it already holds them (a
 * pf_bn_apply_eval of the same x with minmax_enc_dev = range_enc_dev).  C a multiple of 16 (a power of two, or not:
 * each runs a kernel of its own, with the same levels and sums), bits 1..8.  x and the four per-channel vectors
 * 16-byte aligned, levels_dev and hdr_dev 8-byte aligned. */
int pf_bn_eval_levels_u8(const float* x_dev, int64_t m, int c, const float* moving_mean_dev, const float* moving_var_dev,
                         float eps, const float* gamma_dev, const float* beta_dev, int act, int bits,
                         uint32_t* range_enc_dev, int have_range, void* levels_dev, pf_tc_act_hdr* hdr_dev,
                         float* csum_dev, void* stream);
/* the same producer with a static (calibrated) range in range_enc_dev[0..1] (ordered-uint lo / hi, read only): y is
 * clamped to [lo, hi] and quantized with lo / hi in place of the batch's min / max, in ONE pass with no atomics (4 B
 * read + 1 B written per element).  Levels, csum and header equal pf_bn_eval_levels_u8's whenever lo / hi is the
 * batch's range of y.  Same shapes, bits and alignments as pf_bn_eval_levels_u8. */
int pf_bn_eval_levels_u8_static(const float* x_dev, int64_t m, int c, const float* moving_mean_dev,
                                const float* moving_var_dev, float eps, const float* gamma_dev, const float* beta_dev,
                                int act, int bits, const uint32_t* range_enc_dev, void* levels_dev,
                                pf_tc_act_hdr* hdr_dev, float* csum_dev, void* stream);
/* host-side decisions of the most recent tensor-core conv launch (fwd / dgrad / wgrad, either feed), recorded by the
 * launcher from the values it launches with, so that tests can tell which kernel variant a call exercised.  One
 * process-wide record, not synchronised: read it from the thread that launched.  Returns PF_ERR_INVALID_ARG when
 * out is NULL or no launch has been recorded yet. */
typedef struct pf_tc_plan {
  int32_t seq;             /* number of launches recorded so far (this one included) */
  int32_t feed;            /* 1: TMA-fed kernel, 0: cp.async-fed kernel */
  int32_t pass;            /* 0 fwd, 1 dgrad, 2 wgrad */
  int32_t classes;         /* dgrad: 1 = strided dgrad by pixel-parity classes */
  int32_t bn;              /* tile width */
  int32_t aff;             /* epilogue: 0 plain, 1 activation-level scale, 2 weight levels (scale + rank-1 term) */
  int32_t na, nb;          /* operand planes as seen by the host (na: upper bound when a device header decides) */
  int32_t a_fp32;          /* cp.async fwd / dgrad: 1 = the activation is fp32, split by the producers */
  int32_t ring;            /* depth of the residual / accumulate cp.async ring: 0 = none, 2 or 4 */
  int32_t b_stationary;    /* cp.async fwd / dgrad: weights loaded once per CTA */
  int32_t stages;          /* cp.async: pipeline stages; TMA: stage budget in bytes (stages = budget / stage bytes) */
  int32_t tiles;           /* output tiles (fwd / dgrad) or work units (wgrad: tiles x splits) */
  int32_t grid;            /* CTAs launched */
  int32_t splits, pps;     /* wgrad: split-K factor and pixels per split */
} pf_tc_plan;
int pf_conv2d_tc_last_plan(pf_tc_plan* out);
/* hardware probe used by tests/test_tc_gpu.py to pin the descriptor conventions (not a product op) */
int pf_tc_probe(const void* a_dev, const void* b_dev, float* d_dev, int n, int k, int mode, uint32_t lbo_a,
                uint32_t sbo_a, uint32_t lbo_b, uint32_t sbo_b, uint32_t kstep_a, uint32_t kstep_b, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a4  Depthwise convolution, depth multiplier 1 (pf_dwconv.cu): slim.separable_conv2d's depthwise half
 *     (utils/external/mobilenet_v1.py:273-280; TF op DepthwiseConv2dNative).  x NHWC, w [r,s,c,1],
 *     descriptor with k == c, c % 4 == 0, r*s <= 9.  HBM-bound.  wgrad: ws_dev of
 *     pf_dwconv_wgrad_workspace_bytes(d) bytes; deterministic.
 * ------------------------------------------------------------------------------------------- */
#define PF_DWCONV_MAX_SPLITS 1024
int pf_dwconv_fwd(const pf_conv_desc* d, const float* x_dev, const float* w_dev, float* y_dev, void* stream);
int pf_dwconv_dgrad(const pf_conv_desc* d, const float* dy_dev, const float* w_dev, int accumulate, float* dx_dev,
                    void* stream);
int64_t pf_dwconv_wgrad_workspace_bytes(const pf_conv_desc* d);
int pf_dwconv_wgrad(const pf_conv_desc* d, const float* x_dev, const float* dy_dev, float* ws_dev, float* dw_dev,
                    void* stream);
/* which kernel the most recent pf_dwconv_fwd / _dgrad / _wgrad call launched (one of the PF_DW_* below; 0 before the
 * first launch), chosen on the host from the shape and PF_DW_ROWS, so that tests can tell which dispatch target a call
 * exercised.  One process-wide record, not synchronised: read it from the thread that launched. */
enum {
  PF_DW_FWD_ROWS = 1,        /* 3x3 stride 1, 4 output rows per thread */
  PF_DW_FWD_3X3_S1,
  PF_DW_FWD_3X3_S2,
  PF_DW_FWD_GENERIC,
  PF_DW_DGRAD_ROWS,
  PF_DW_DGRAD_3X3_S1,
  PF_DW_DGRAD_BLOCK_P0,      /* 3x3 stride 2, 2 x 2 input pixels per thread, pad 0 */
  PF_DW_DGRAD_BLOCK_P1,      /* the same, pad 1 */
  PF_DW_DGRAD_3X3_S2,
  PF_DW_DGRAD_GENERIC,
  PF_DW_WGRAD_ROWS,
  PF_DW_WGRAD_3X3_S1,
  PF_DW_WGRAD_3X3_S2,
  PF_DW_WGRAD_GENERIC
};
int pf_dwconv_last_variant(void);
/* u8 forward of the integer inference model (reference: learners/uniform_quantization/utils.py:92-104, 163-199, the
 * depthwise conv of the fake-quantized weight and activation), on CUDA cores:
 *   x->plane0 = u8 activation levels q_a [N,H,W,C], x->hdr = {scale = alpha_a / k_a, nplanes = 1} as
 *   pf_bn_eval_levels_u8 writes them (x->plane1 = NULL; x->csum is not read);  w->plane0 = u8 weight levels q_w [R*S][C]
 *   (the [R,S,C,1] kernel's layout), w->plane1 = NULL, w->alpha / w->beta = the weight quantizer's bucket scales ([C]
 *   with w->per_channel = 1, else [1]), w->bits = log2(k_w + 1) in 1..8.
 * Per output pixel and channel, S = sum_taps q_a q_w and J = sum_taps q_a are exact integers (padding taps are level 0,
 * the value 0 of an activation whose range starts at 0), and
 *   y = (scale * alpha_c / k_w) * S + (scale * beta_c) * J
 * is rounded once, in fp32.  A header with nplanes != 1 makes every output NaN.  Requires pf_dwconv_u8_supported(d):
 * k == c, C % 16 == 0 (16 channels per 128-bit load), C <= 65536, r * s <= 9, strides 1 or 2, zero padding, fewer than
 * 2^31 input and output elements; 3 x 3 filters with equal strides run a row-blocked kernel, the rest one pixel per
 * item. */
int pf_dwconv_u8_supported(const pf_conv_desc* d);
int pf_dwconv_u8_fwd(const pf_conv_desc* d, const pf_tc_act* x, const pf_tc_wt* w, float* y_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a13 The HBM-bound layers between the convolutions (pf_nn.cu); tensors viewed as [m, c], c % 4 == 0.
 *     tf.layers.batch_normalization(momentum, eps, fused) — utils/external/resnet_model.py:55-62:
 *       stats : batch mean / biased variance / rstd (+ moving-stat update, unbiased moving variance);
 *               ws_dev: 3*c*PF_BN_MAX_SPLITS floats.
 *       apply : y = act(((x-mean)*rstd)*gamma+beta), act 0 none / 1 relu / 2 relu6; when
 *               minmax_enc_dev != NULL also accumulates the per-tensor min/max of y for the
 *               activation quantizer (utils.py:51-79) — the reference's two extra reduction passes.
 *       bwd   : dgamma, dbeta, dx (+)= through act and training-mode BN; ws_dev as for stats.
 * ------------------------------------------------------------------------------------------- */
int pf_bn_train_stats(const float* x_dev, int64_t m, int c, float eps, float momentum, float* mean_dev,
                      float* var_dev, float* rstd_dev, float* moving_mean_dev, float* moving_var_dev,
                      float* ws_dev, void* stream);
/* stats + the per-tensor range of y = act(bn(x)) for the activation quantizer, evaluated from the per-channel
 * extremes of x (every step of bn/act is monotone in x, so the result is bit-identical to a min/max pass over
 * y); accumulates into minmax_enc_dev[0..1] (ordered-uint).  ws_dev: 5 * C * PF_BN_MAX_SPLITS floats. */
int pf_bn_train_stats_range(const float* x_dev, int64_t m, int c, float eps, float momentum, float* mean_dev,
                            float* var_dev, float* rstd_dev, float* moving_mean_dev, float* moving_var_dev,
                            const float* gamma_dev, const float* beta_dev, int act, uint32_t* minmax_enc_dev,
                            float* ws_dev, void* stream);
int pf_bn_eval_prepare(const float* moving_var_dev, int c, float eps, float* rstd_dev, void* stream);
/* inference-mode BN in one launch: rstd = rsqrt(moving_var + eps) is formed in the kernel (same roundings as
 * pf_bn_eval_prepare + pf_bn_apply); fp32 and/or split-bf16 plane output */
int pf_bn_apply_eval(const float* x_dev, int64_t m, int c, const float* moving_mean_dev, const float* moving_var_dev,
                     float eps, const float* gamma_dev, const float* beta_dev, int act, float* y_dev, void* y_hi_dev,
                     void* y_lo_dev, uint32_t* minmax_enc_dev, void* stream);
/* inference-mode BN + act + fake-quant with a static (calibrated) range in one pass: y = Q(clamp(act(bn(x)), lo, hi))
 * with range_enc_dev[0..1] = the encoded lo / hi; fp32 and/or split-bf16 planes.  Bit-identical to pf_bn_apply_eval
 * followed by pf_uq_act_quant(_planes) when lo / hi is the batch's range of act(bn(x)). */
int pf_bn_apply_eval_quant_static(const float* x_dev, int64_t m, int c, const float* moving_mean_dev,
                                  const float* moving_var_dev, float eps, const float* gamma_dev, const float* beta_dev,
                                  int act, const uint32_t* range_enc_dev, int bits, float* y_dev, void* y_hi_dev,
                                  void* y_lo_dev, void* stream);
/* y = Q(act(bn(x))) in one pass with a known range (pf_bn_train_stats_range): fp32 and/or split-bf16 planes */
int pf_bn_apply_quant(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                      const float* gamma_dev, const float* beta_dev, int act, const uint32_t* range_enc_dev, int bits,
                      float* y_dev, void* y_hi_dev, void* y_lo_dev, void* stream);
int pf_bn_apply(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                const float* gamma_dev, const float* beta_dev, int act, float* y_dev,
                uint32_t* minmax_enc_dev, void* stream);
int pf_bn_bwd(const float* dy_dev, const float* x_dev, int64_t m, int c, const float* mean_dev,
              const float* rstd_dev, const float* gamma_dev, const float* beta_dev, int act,
              float* dgamma_dev, float* dbeta_dev, float* dx_dev, int accumulate, float* ws_dev,
              void* stream);
/* variants that (also) write the result as split-bf16 planes — the operand format of the tensor-core convs that
 * consume it (y: next conv's fwd + wgrad; dx: the producing conv's dgrad + wgrad).  The fp32 output pointer may
 * be NULL when every consumer takes planes; `accumulate` needs the fp32 dx. */
int pf_bn_apply_planes(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                       const float* gamma_dev, const float* beta_dev, int act, float* y_dev, void* y_hi_dev,
                       void* y_lo_dev, uint32_t* minmax_enc_dev, void* stream);
int pf_bn_bwd_planes(const float* dy_dev, const float* x_dev, int64_t m, int c, const float* mean_dev,
                     const float* rstd_dev, const float* gamma_dev, const float* beta_dev, int act,
                     float* dgamma_dev, float* dbeta_dev, float* dx_dev, int accumulate, void* dx_hi_dev,
                     void* dx_lo_dev, float* ws_dev, void* stream);
/* linear bottleneck + residual (MobileNet-v2, conv_blocks.py:289-313): y = bn(x) + res, BN without activation, in one
 * pass — the training form with batch statistics (mean / rstd of pf_bn_train_stats), the _eval form with moving
 * statistics (rstd formed in the kernel as in pf_bn_apply_eval).  Writes the fp32 sum and / or its split-bf16 planes
 * (the operand of the next block's expand conv); at least one output.  The add is one __fadd_rn after the BN op
 * chain: bit-identical to pf_bn_apply + pf_add.  8 B/element read, 4 (fp32) and / or 4 (planes) written. */
int pf_bn_apply_add(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                    const float* gamma_dev, const float* beta_dev, const float* res_dev, float* y_dev, void* y_hi_dev,
                    void* y_lo_dev, void* stream);
int pf_bn_apply_add_eval(const float* x_dev, int64_t m, int c, const float* moving_mean_dev, const float* moving_var_dev,
                         float eps, const float* gamma_dev, const float* beta_dev, const float* res_dev, float* y_dev,
                         void* y_hi_dev, void* y_lo_dev, void* stream);
/* channel gathers of the compact (channel-pruned) inference graph, pocketflow_b200/compact.py: NHWC viewed as
 * [m, cin] -> [m, cout], y[:, j] = x[:, idx[j]], and 0 where idx[j] < 0 (zero padding channels); cout % 4 == 0,
 * idx_dev 16-byte aligned.
 *   pf_gather_channels       input fp32 (x_dev) OR split-bf16 planes (x_hi_dev / x_lo_dev); output fp32 and / or
 *                            planes.  fp32 -> planes is the split of pf_split_bf16; planes -> planes copies the bits;
 *                            planes -> fp32 is hi + lo.
 *   pf_bn_apply_eval_gather  y = gather(act(bn(x))) with the moving statistics, bit-identical to pf_bn_apply_eval at
 *                            full width followed by pf_gather_channels (mean / var / gamma / beta have cin entries). */
int pf_gather_channels(const float* x_dev, const void* x_hi_dev, const void* x_lo_dev, int64_t m, int cin, int cout,
                       const int32_t* idx_dev, float* y_dev, void* y_hi_dev, void* y_lo_dev, void* stream);
int pf_bn_apply_eval_gather(const float* x_dev, int64_t m, int cin, const float* moving_mean_dev,
                            const float* moving_var_dev, float eps, const float* gamma_dev, const float* beta_dev, int act,
                            int cout, const int32_t* idx_dev, float* y_dev, void* y_hi_dev, void* y_lo_dev,
                            void* stream);
/* training of the compact graph (fine-tuning a channel-pruned model at its pruned width):
 *   pf_bn_apply_gather   y = gather(act(bn(x))) with the batch statistics mean / rstd of pf_bn_train_stats (cin entries,
 *                        taken at the BN's own width), bit-identical to pf_bn_apply at full width followed by
 *                        pf_gather_channels; reads 4 B per kept element, writes 4 B (fp32) and / or 4 B (planes).
 *   pf_scatter_channels  the backward of pf_gather_channels: dx[:, idx[j]] (+)= dy[:, j] for idx[j] >= 0.  dy is
 *                        [m, cout], dx [m, cin] (cin % 4 == 0); inv_dev[cin] is the inverse of the gather's table
 *                        (inv[c] = j with idx[j] == c, else -1; 16-byte aligned) — positions are unique, so every
 *                        element of dx has one writer and there are no atomics.  accumulate == 0 writes ALL of dx (zeros
 *                        where inv < 0); accumulate != 0 adds into the fp32 dx and leaves ungathered channels alone.
 *                        dx may also (or only, without accumulate) be written as split-bf16 planes of the final value,
 *                        the convention of pf_bn_bwd_planes.  4 B read per compact element + 4 B written per element
 *                        of dx (+ 4 B read per touched element when accumulating). */
int pf_bn_apply_gather(const float* x_dev, int64_t m, int cin, const float* mean_dev, const float* rstd_dev,
                       const float* gamma_dev, const float* beta_dev, int act, int cout, const int32_t* idx_dev,
                       float* y_dev, void* y_hi_dev, void* y_lo_dev, void* stream);
int pf_scatter_channels(const float* dy_dev, int64_t m, int cin, int cout, const int32_t* inv_dev, int accumulate,
                        float* dx_dev, void* dx_hi_dev, void* dx_lo_dev, void* stream);
/* dropout (slim.dropout, mobilenet.py:369; TF 1.x nn_ops.dropout): y = (x / keep) * floor(keep + u), u in [0, 1) from
 * Philox4x32-10 keyed by (seed, rank) with counter (element index / 4 [64 bits], step [low 32 bits], stream_id);
 * mask_dev[i] <- floor(keep + u) (0 / 1).  stream_id tells the Dropout ops of one graph apart (each passes its own
 * state).  state_dev[0] is the step, state_dev[1] scratch (both 0 initially): the launch reads the step and advances it
 * by one, so a replayed CUDA graph draws a fresh mask each time.  Backward: dx (+)= (dy * mask) / keep. */
int pf_dropout_fwd(const float* x_dev, int64_t n, float keep_prob, uint32_t seed, uint32_t rank, uint32_t stream_id,
                   uint64_t* state_dev, float* y_dev, uint8_t* mask_dev, void* stream);
/* the same draw for a channel-pruned tensor [n / c, c] whose channel j is channel layout_dev[j] of the full-width
 * tensor [n / c, cfull] (layout_dev: c int32 on the device, -1 for a zero padding channel): element (row, j) takes the
 * uniform full-width element row * cfull + layout_dev[j] takes under pf_dropout_fwd with the same seed, rank, stream_id
 * and step, so the mask is the full-width one gathered by the layout; a padding channel gets mask 0.  layout_dev NULL:
 * exactly pf_dropout_fwd. */
int pf_dropout_fwd_mapped(const float* x_dev, int64_t n, float keep_prob, uint32_t seed, uint32_t rank,
                          uint32_t stream_id, const int32_t* layout_dev, int c, int cfull, uint64_t* state_dev,
                          float* y_dev, uint8_t* mask_dev, void* stream);
int pf_dropout_bwd(const float* dy_dev, const uint8_t* mask_dev, int64_t n, float keep_prob, int accumulate, float* dx_dev,
                   void* stream);
/* out (+)= a (+ b): residual add (resnet_model.py:199,314) / gradient fan-out; b_dev may be NULL */
int pf_add(const float* a_dev, const float* b_dev, int64_t n, int accumulate, float* out_dev, void* stream);
/* dst[i][j] = sum_b src[b*m+i][b*n+j] (src is (g*m) x (g*n) row-major): folds the diagonal blocks of a weight gradient that
 * the tensor cores computed from g pixels per GEMM row (convs with fewer than 64 output channels) */
int pf_fold_diag_blocks(const float* src_dev, int g, int m, int n, float* dst_dev, void* stream);
/* dx (+)= dy * [y > 0] (and [y < 6] for act == 2) */
int pf_relu_bwd(const float* dy_dev, const float* y_dev, int64_t n, int act, int accumulate, float* dx_dev,
                void* stream);
/* out[c] = sum_m a[m][c] (bias gradient) */
int pf_colsum(const float* a_dev, int64_t m, int c, float* out_dev, void* stream);
/* max pooling (kernel r x s, strides, leading pads from the descriptor; k unused; c % 4 == 0).  The
 * forward records the window position of the FIRST maximum in row-major order (uint8 per output
 * element; argmax_dev may be NULL for inference) and the backward routes each gradient there, like
 * TF's MaxPoolGrad.  Gather form, deterministic. */
int pf_maxpool_fwd(const pf_conv_desc* d, const float* x_dev, float* y_dev, uint8_t* argmax_dev, void* stream);
int pf_maxpool_bwd(const pf_conv_desc* d, const float* dy_dev, const uint8_t* argmax_dev, int accumulate,
                   float* dx_dev, void* stream);
/* ILSVRC-12 preprocessing of a mini-batch of decoded uint8 RGB crops in one launch — what
 * utils/external/imagenet_preprocessing.py:225-260 does after decoding: TF1 bilinear resize (align_corners=False, no
 * half-pixel centres) of the [h, w, 3] crop at crops_dev + offset to [rh, rw], optional left-right flip of the SOURCE
 * (training flips before resizing), the [out_h, out_w] window at (top, left) of the resized image (evaluation:
 * central crop of the 256-short-side resize; training: rh = out_h, rw = out_w, top = left = 0), minus the channel
 * means.  dst_dev: fp32 [n, out_h, out_w, 3].  Bit-identical to the host restatement in
 * pocketflow_b200/datasets/ilsvrc12_dataset.py (every operation individually rounded). */
typedef struct pf_img_desc {
  int64_t offset;        /* byte offset of this crop in crops_dev */
  int32_t h, w;          /* crop size */
  int32_t rh, rw;        /* size it is resized to */
  int32_t top, left;     /* window origin inside the resized image */
  int32_t flip;          /* != 0: mirror the crop left-right before resizing */
  int32_t reserved;
} pf_img_desc;
int pf_preprocess_images(const uint8_t* crops_dev, const pf_img_desc* desc_dev, int n, int out_h, int out_w,
                         float mean_r, float mean_g, float mean_b, float* dst_dev, void* stream);

/* Baseline JPEG decoding for the input pipeline (pf_jpeg.cu), bit for bit with libjpeg-turbo's default
 * decompression (islow IDCT, fancy upsampling, YCbCr -> RGB) as Pillow runs it.  The host parses the headers
 * (pocketflow_b200/datasets/jpeg.py) and only hands over files the device supports: 8-bit, one interleaved sequential
 * Huffman scan, grey or YCbCr with luma sampling 1x1, 2x1 or 2x2 and chroma 1x1.
 *   data_dev    : every image's entropy-coded segment (desc.scan_offset / scan_bytes)
 *   coef_ws_dev : int16 workspace, 64 per block of MCU rows [0, mcu_rows) of each image from desc.coef_offset on
 *                 (mcus_per_row * mcu_rows * blocks per MCU * 128 bytes per image)
 *   crops_dev   : uint8 [crop_h, crop_w, 3] RGB written at desc.crop_offset
 *   status_dev  : int32 [n], 0 = decoded; otherwise the image's data is anomalous (1 bad Huffman code, 2 data ends
 *                 early, 3 bad restart marker, 4 run past coefficient 63, 5 bad descriptor: a field out of range, or an
 *                 MCU window that does not hold every block the crop and its upsampling context read), its crop is
 *                 not written and the host has to decode it.  An anomaly never touches another image's crop or
 *                 workspace.  The caller guarantees that data_dev, coef_ws_dev and crops_dev hold what each
 *                 descriptor's offsets and sizes point at (datasets/jpeg.py: pack, workspace_elems). */
typedef struct pf_jpeg_huff {
  int16_t lookup[256];    /* next 8 bits -> (code length << 8) | symbol; 0: the code is longer than 8 bits */
  int32_t maxcode[18];    /* largest code of each length (-1: none), as jdhuff.c derives it */
  int32_t valoffset[18];  /* huffval index = code + valoffset[length] */
  uint8_t huffval[256];
} pf_jpeg_huff;
typedef struct pf_jpeg_desc {
  int64_t scan_offset;     /* first byte of the entropy-coded segment in data_dev */
  int64_t coef_offset;     /* first int16 of this image's workspace (a multiple of 64) */
  int64_t crop_offset;     /* first byte of the crop in crops_dev */
  int32_t scan_bytes;
  int32_t height, width;
  int32_t ncomp;           /* 1 (grey) or 3 (YCbCr) */
  int32_t hs, vs;          /* luma sampling factors; chroma is 1x1 */
  int32_t restart_interval;/* MCUs per restart interval, 0: none */
  int32_t mcus_per_row;
  int32_t mcu_rows;        /* MCU rows entropy-decoded: through the last one the crop needs */
  int32_t mcu_row0, mcu_col0, mcu_col1;  /* MCU window inverse-transformed: rows [mcu_row0, mcu_rows) */
  int32_t crop_y, crop_x, crop_h, crop_w;
  int32_t dc_tbl[3], ac_tbl[3];          /* per component: index into huff[] */
  uint16_t quant[3][64];   /* per component, zig-zag order */
  pf_jpeg_huff huff[4];
} pf_jpeg_desc;
int pf_jpeg_decode(const uint8_t* data_dev, const pf_jpeg_desc* desc_dev, int n, int16_t* coef_ws_dev,
                   uint8_t* crops_dev, int32_t* status_dev, void* stream);
/* tf.reduce_mean over H,W (resnet_model.py:547-548) */
int pf_global_avgpool_fwd(const float* x_dev, int n, int hw, int c, float* y_dev, void* stream);
int pf_global_avgpool_bwd(const float* dy_dev, int n, int hw, int c, int accumulate, float* dx_dev, void* stream);
/* row softmax and its backward (nets/lenet_at_cifar10.py:66) */
int pf_softmax_fwd(const float* x_dev, int n, int k, float* y_dev, void* stream);
int pf_softmax_bwd(const float* dy_dev, const float* y_dev, int n, int k, float* dx_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * f4  Layer-wise channel selection of the channel-pruning learner (pf_cpg.cu).
 *     Replaces, per proximal-gradient iteration of ChannelPrunedGpuLearner.__choose_channels
 *     (learners/channel_pruning_gpu/learner.py:445-518), the TF ops of __build_extra_losses (:339-354) and
 *     __build_layer_ops (:356-402); kernels W are [R,S,Cin,Cout] row-major, rs = R*S:
 *   pf_cpg_diff_l2     diff = a - b ; loss[0] = sum(diff^2)/2    (tf.nn.l2_loss of the two conv outputs, :352;
 *                      with a = pruned, b = full, diff is also d loss / d a).  partial_ws: PF_L2_PARTIALS floats.
 *   pf_cpg_group_norms norms[c] = sqrt(sum_{rs,k} (w - lr*g)^2)  (:378-379; g NULL: the norm of w itself, :256)
 *   pf_cpg_prox_apply  w = (w - lr*g) * max(1 - thr[0] / norms[c], 0)   (:378-382; thr = the percentile of norms)
 *   pf_cpg_channel_mask mask[rs,c,k] = norms[c] > 0               (:256-259)
 *   pf_mul             out = a * b                                 (masked gradient g * mask, :438)
 * ------------------------------------------------------------------------------------------- */
int pf_cpg_diff_l2(const float* a_dev, const float* b_dev, int64_t n, float* diff_dev, float* loss_dev,
                   float* partial_ws_dev, void* stream);
int pf_cpg_group_norms(const float* w_dev, const float* g_dev, float lr, int rs, int cin, int cout,
                       float* norms_dev, void* stream);
int pf_cpg_prox_apply(float* w_dev, const float* g_dev, float lr, const float* norms_dev, const float* thr_dev,
                      int rs, int cin, int cout, void* stream);
int pf_cpg_channel_mask(const float* norms_dev, int rs, int cin, int cout, float* mask_dev, void* stream);
int pf_mul(const float* a_dev, const float* b_dev, int64_t n, float* out_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * f5  Channel selection of the remastered channel-pruning learner (pf_cpr.cu).
 *     Replaces the numpy float64 / small-TF-graph work of ChannelPrunedRmtLearner.__choose_channels
 *     (learners/channel_pruning_rmt/learner.py:546-842); kernels W are [R,S,Cin,Cout] row-major, rs = R*S,
 *     K = rs*Cin; patch rows are HWIO-ordered, so X * reshape(W, [K, Cout]) is the conv:
 *   pf_cpr_sample   rows_dev int32 [n_rows, 4] = (n, oh, ow, dst) (16-byte aligned; dst < 0: skip the row):
 *                   X[dst, (r*S+s)*Cin + c] = x[n, oh*sh - pad_t + r, ow*sw - pad_l + s, c] (0 outside the image),
 *                   Y[dst, k] = y[n, oh, ow, k] - bias[k]   (:679-703; bias_dev may be NULL).  The input is x_dev
 *                   when non-NULL, else hi + lo of the split-bf16 planes x_hi_dev / x_lo_dev.  Exact (a gather).
 *   pf_cpr_gram     over the n_idx rows idx_dev of X / Y (:751-769):
 *                     F[(j,o), c] = sum_t X[idx[j], t*Cin + c] * W[t, c, o]  (float64),  y[(j,o)] = Y[idx[j], o]
 *                     G = F^T F, b = F^T y, nrm = ||G||_F;  g_dev = (Cin+1)^2 + 1 doubles:
 *                     g[i*(Cin+1) + j] = G[i][j] / nrm, g[i*(Cin+1) + Cin] = b[i] / nrm (i, j < Cin),
 *                     g[(Cin+1)^2] = nrm;  gf_dev [Cin*Cin] / bf_dev [Cin] = the same in float32.
 *                   F is formed chunk_rows rows of X at a time in ws_dev (pf_cpr_gram_ws_doubles doubles).
 *                   CUDA-core FP64, fixed summation order (deterministic).
 *   pf_cpr_ista     iters steps of m <- prox(m - lr*(G m - b), gamma*lr) in float32 from m0 (:449-452, :780-781),
 *                   one cooperative launch; m_dev [Cin] = result, nnz_dev[0] = its count of non-zeros;
 *                   ws_dev: 2*Cin floats.  Deterministic (fixed-order row sums).
 *   pf_cpr_mask_channels  a[row, t, c, k] *= (|m[c]| > 0) for a of shape [rows, rs, Cin, inner]   (:817-820, :839)
 * ------------------------------------------------------------------------------------------- */
int pf_cpr_sample(const pf_conv_desc* d, const float* x_dev, const void* x_hi_dev, const void* x_lo_dev,
                  const float* y_dev, const float* bias_dev, const int32_t* rows_dev, int n_rows, float* X_dev,
                  float* Y_dev, void* stream);
int64_t pf_cpr_gram_ws_doubles(int cin, int cout, int64_t chunk_rows);
int pf_cpr_gram(const float* X_dev, const float* Y_dev, const int32_t* idx_dev, int n_idx, const float* w_dev, int rs,
                int cin, int cout, double* ws_dev, int64_t chunk_rows, double* g_dev, float* gf_dev, float* bf_dev,
                void* stream);
int pf_cpr_ista(const float* g_dev, const float* b_dev, const float* m0_dev, int cin, float lr, float gamma, int iters,
                float* m_dev, float* ws_dev, int32_t* nnz_dev, void* stream);
int pf_cpr_mask_channels(float* a_dev, int64_t rows, int rs, int cin, int inner, const float* m_dev, void* stream);

/* f5b Channel selection of the LASSO channel-pruning learner (pf_cpr.cu, /root/reference/learners/channel_pruning).
 *   pf_cp_sample     rows_dev int32 [n_rows, 8] = (n, oh, ow, dst, rh, rw, 0, 0) (16-byte aligned; dst < 0: skip):
 *                    X[dst] = the R x S x C input patch at (n, oh, ow) as pf_cpr_sample gathers it, and in float64
 *                    Y[dst, k] = (y - bias)[n, oh, ow, k] + (res_full - res_cur)[n, rh, rw, k] (res_* [N, res_h,
 *                    res_w, K], both NULL: no residual term).
 *   pf_cp_gram       G_aug [(cin+1)^2 (+1 scratch)] = [P | y]^T [P | y] over the n_idx sampled rows idx_dev, where
 *                    P[(j, o), c] = sum_t X[idx[j], t, c] W[t, c, o] and y[(j, o)] = Y[idx[j], o]; float64, formed
 *                    chunk_rows rows at a time in ws_dev ((cin+1) * chunk_rows * cout doubles).
 *   pf_cp_normal_eq  G_aug [(ncols+cout)^2 (+1 scratch)] = [X_k | Y]^T [X_k | Y] over all n_rows rows, X_k = the columns
 *                    cols_dev of X [n_rows, K]; ws_dev holds (ncols + cout) * chunk_rows doubles.
 */
int pf_cp_sample(const pf_conv_desc* d, const float* x_dev, const void* x_hi_dev, const void* x_lo_dev,
                 const float* y_dev, const float* bias_dev, const float* res_full_dev, const float* res_cur_dev,
                 int res_h, int res_w, const int32_t* rows_dev, int n_rows, float* X_dev, double* Y_dev, void* stream);
int pf_cp_gram(const float* X_dev, const double* Y_dev, const int32_t* idx_dev, int n_idx, const float* w_dev, int rs,
               int cin, int cout, double* ws_dev, int64_t chunk_rows, double* g_dev, void* stream);
int pf_cp_normal_eq(const float* X_dev, const double* Y_dev, int64_t n_rows, int64_t K, int cout, const int32_t* cols_dev,
                    int ncols, double* ws_dev, int64_t chunk_rows, double* g_dev, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a10 The collective of the data-parallel step (pf_comm.cu).  Replaces mgw.DistributedOptimizer's per-variable
 *     Horovod all-reduces and mgw.broadcast_global_variables (utils/multi_gpu_wrapper.py:82-98; call sites
 *     learners/uniform_quantization/learner.py:245-247, :271): ONE in-place ncclAllReduce (sum, fp32) over the flat
 *     gradient buffer — or over contiguous buckets of it as the backward pass completes them — enqueued on the
 *     caller's stream (CUDA-graph capturable); the division by the worker count is the optimizers' grad_scale.
 *     NCCL (libnccl.so.2, or the path in PF_NCCL_LIB) is bound at run time, not linked.
 *       pf_comm_unique_id  rank 0: 128 bytes to distribute to every rank (any host-side channel)
 *       pf_comm_init       collective over all ranks, on the calling thread's current device; *comm_out = handle
 *       pf_allreduce_flat / pf_broadcast_flat   asynchronous on `stream`
 * ------------------------------------------------------------------------------------------- */
int pf_comm_nccl_version(int* version_out);
int pf_comm_unique_id(void* id128_out);
int pf_comm_init(const void* id128, int n_ranks, int rank, void** comm_out);
int pf_comm_destroy(void* comm);
int pf_allreduce_flat(void* comm, float* buf_dev, int64_t n, void* stream);
int pf_broadcast_flat(void* comm, float* buf_dev, int64_t n, int root, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PF_B200_H_ */
