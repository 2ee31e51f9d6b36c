// pf_nuq.cu — codebook (non-uniform) weight quantization, multi-tensor.
//
// Replaces NonUniformQuantization.__nonuni_quantize / __build_norm_quant_point
// (/root/reference/learners/nonuniform_quantization/utils.py:168-194, 284-307), which materialises
// tile(x, [...,2^b]) (a x16 temporary at 4 bits: 1.5 GB on ResNet-50), abs(sub), argmin, gather,
// mul(sign) and the inverse scale as separate TF kernels.  Here the codebook of a tensor sits in
// shared memory and the nearest-centroid search runs in registers: 8 B/element of HBM traffic
// (+1 B/element when the centroid index is kept for the codebook gradient).
#include "pf_common.cuh"

namespace {
constexpr int kThreads = 256;

__device__ __forceinline__ float nuq_one(float w, float alpha, float beta, float ralpha,
                                         const float* __restrict__ c, int nc, uint8_t* idx_out) {
  const float xn = pf_div_r(__fsub_rn(w, beta), alpha, ralpha);
  float best = fabsf(__fsub_rn(xn, c[0]));
  int bi = 0;
  for (int j = 1; j < nc; ++j) {
    const float d = fabsf(__fsub_rn(xn, c[j]));
    if (d < best) {  // strict: first index wins on ties (tf.argmin)
      best = d;
      bi = j;
    }
  }
  if (idx_out) *idx_out = (uint8_t)bi;
  const float t = __fadd_rn(xn, 1e-6f);
  const float sgn = t > 0.f ? 1.f : (t < 0.f ? -1.f : 0.f);
  return __fadd_rn(__fmul_rn(alpha, __fmul_rn(c[bi], sgn)), beta);
}

__global__ void __launch_bounds__(kThreads)
nuq_quant_kernel(const pf_uq_seg* __restrict__ segs, const pf_work* __restrict__ work,
                 const float* __restrict__ scales, int n_buckets,
                 const float* __restrict__ clusters, const int64_t* __restrict__ cluster_off,
                 uint8_t* __restrict__ idx_out, const int64_t* __restrict__ idx_base) {
  __shared__ float sc[256];
  const pf_work w = work[blockIdx.x];
  const pf_uq_seg s = segs[w.seg];
  const int nc = 1 << s.bits;
  // the codebook of this tensor: at cluster_off[seg] floats from `clusters` (codebooks that live among the model's
  // trainable variables), or at seg * 256 (a [segments, 256] table)
  const float* cb = clusters + (cluster_off ? (size_t)cluster_off[w.seg] : (size_t)w.seg * 256);
  if ((int)threadIdx.x < nc) sc[threadIdx.x] = cb[threadIdx.x];
  __syncthreads();
  const float alpha = __ldg(scales + s.bucket0), mn = __ldg(scales + n_buckets + s.bucket0);
  const float ra = __ldg(scales + 2 * n_buckets + s.bucket0);
  uint8_t* io = idx_out ? idx_out + idx_base[w.seg] : nullptr;
  const int64_t end = w.start + w.count;
  for (int64_t i = w.start + (int64_t)threadIdx.x * 4; i < end; i += kThreads * 4) {
    if (i + 3 < end) {
      float4 v = pf_ld4(s.src + i);
      uint8_t id[4];
      v.x = nuq_one(v.x, alpha, mn, ra, sc, nc, io ? &id[0] : nullptr);
      v.y = nuq_one(v.y, alpha, mn, ra, sc, nc, io ? &id[1] : nullptr);
      v.z = nuq_one(v.z, alpha, mn, ra, sc, nc, io ? &id[2] : nullptr);
      v.w = nuq_one(v.w, alpha, mn, ra, sc, nc, io ? &id[3] : nullptr);
      pf_st_stream(s.dst + i, v);
      if (io) *reinterpret_cast<uchar4*>(io + i) = make_uchar4(id[0], id[1], id[2], id[3]);
    } else {
      for (int64_t j = i; j < end; ++j) s.dst[j] = nuq_one(s.src[j], alpha, mn, ra, sc, nc, io ? io + j : nullptr);
    }
  }
}

// ---- codebook gradient (cluster / both optimisation modes): the gather's backward is a segment sum,
//   dL/dc_j = alpha * sum_{i: idx_i = j} g_i        (g = dL/d(quantized weight); inverse scale alpha*q + beta)
// Deterministic two-stage reduction: every CTA sums its chunk per centroid in registers (16 centroids per pass, the
// chunk is re-read from L2 for codebooks with more), block-reduces, and writes partial[work][j]; the final kernel adds
// the partials of a tensor in work order and applies alpha.
constexpr int kNcPass = 16;

__global__ void __launch_bounds__(kThreads)
nuq_cluster_grad_partial_kernel(const pf_uq_seg* __restrict__ segs, const pf_work* __restrict__ work,
                                const uint8_t* __restrict__ idx, const int64_t* __restrict__ idx_base,
                                float* __restrict__ partial) {
  __shared__ float sh[kThreads / 32][kNcPass];
  const pf_work w = work[blockIdx.x];
  const pf_uq_seg s = segs[w.seg];
  const int nc = 1 << s.bits;
  const uint8_t* io = idx + idx_base[w.seg];
  const float* g = s.src;                       // the gradient w.r.t. the quantized tensor
  const int64_t end = w.start + w.count;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j0 = 0; j0 < nc; j0 += kNcPass) {
    float acc[kNcPass];
#pragma unroll
    for (int j = 0; j < kNcPass; ++j) acc[j] = 0.f;
    for (int64_t i = w.start + threadIdx.x; i < end; i += kThreads) {
      const int id = (int)io[i] - j0;
      const float gv = g[i];
#pragma unroll
      for (int j = 0; j < kNcPass; ++j) acc[j] += (id == j) ? gv : 0.f;
    }
#pragma unroll
    for (int j = 0; j < kNcPass; ++j) {
      const float t = pf_warp_sum(acc[j]);
      if (lane == 0) sh[warp][j] = t;
    }
    __syncthreads();
    if (threadIdx.x < kNcPass && j0 + (int)threadIdx.x < nc) {
      float t = 0.f;
#pragma unroll
      for (int wv = 0; wv < kThreads / 32; ++wv) t += sh[wv][threadIdx.x];
      partial[(size_t)blockIdx.x * 256 + j0 + threadIdx.x] = t;
    }
    __syncthreads();
  }
}

// one CTA per tensor: sum the partials of its work items (a contiguous range of the work table) in order
__global__ void __launch_bounds__(256)
nuq_cluster_grad_final_kernel(const pf_uq_seg* __restrict__ segs, const int32_t* __restrict__ work_first,
                              const float* __restrict__ partial, const float* __restrict__ scales,
                              float* __restrict__ grad_base, const int64_t* __restrict__ cluster_off) {
  const int seg = blockIdx.x;
  const pf_uq_seg s = segs[seg];
  const int nc = 1 << s.bits;
  const int j = threadIdx.x;
  if (j >= nc) return;
  float t = 0.f;
  for (int wi = work_first[seg]; wi < work_first[seg + 1]; ++wi) t += partial[(size_t)wi * 256 + j];
  grad_base[cluster_off[seg] + j] = __fmul_rn(t, __ldg(scales + s.bucket0));     // * alpha
}

// ================================================================== bucketed codebooks
// NonUniformQuantization.__bucket_quantize (utils.py:196-243): a tensor is viewed as [rows, nb] (bucket of flat element
// i = i % nb; split buckets pad with copies of the last element), bucket b has its own range (alpha_b, beta_b from
// pf_uq_weight_minmax / pf_uq_weight_scales) and its own codebook, column b of a [K, nb] matrix (K >= 2^bits rows):
//   c[j, b] = clusters_base[cluster_off[seg] + j * nb + b].
// Work items are kind-1 tiles: columns [c0, c0 + ncol_tile) x rows [start, start + count); ncol_tile <= 8192 / 2^bits,
// so a tile's codebooks ([2^bits][ncol_tile] floats, <= 32 KB) sit in shared memory whatever nb is.
constexpr int kBucketSmemFloats = 8192;

__device__ __forceinline__ float nuq_one_col(float w, float alpha, float beta, float ralpha,
                                             const float* __restrict__ c, int ld, int nc, int* idx_out) {
  const float xn = pf_div_r(__fsub_rn(w, beta), alpha, ralpha);
  float best = fabsf(__fsub_rn(xn, c[0]));
  int bi = 0;
  for (int j = 1; j < nc; ++j) {
    const float d = fabsf(__fsub_rn(xn, c[j * ld]));
    if (d < best) {  // strict: first index wins on ties (tf.argmin)
      best = d;
      bi = j;
    }
  }
  *idx_out = bi;
  const float t = __fadd_rn(xn, 1e-6f);
  const float sgn = t > 0.f ? 1.f : (t < 0.f ? -1.f : 0.f);
  return __fadd_rn(__fmul_rn(alpha, __fmul_rn(c[bi * ld], sgn)), beta);
}

// one thread per column of the tile, kThreads / tile-width row groups; only real elements (r * nb + col < numel) are
// read and written, padding copies take no part in the assignment
__global__ void __launch_bounds__(kThreads)
nuq_bucket_quant_kernel(const pf_uq_seg* __restrict__ segs, const pf_work* __restrict__ work,
                        const float* __restrict__ scales, int n_buckets, const float* __restrict__ clusters,
                        const int64_t* __restrict__ cluster_off, uint8_t* __restrict__ idx_out,
                        const int64_t* __restrict__ idx_base) {
  __shared__ float sc[kBucketSmemFloats];
  const pf_work w = work[blockIdx.x];
  const pf_uq_seg s = segs[w.seg];
  const int nc = 1 << s.bits, tc = w.ncol_tile, nb = s.ncols;
  const float* cb = clusters + cluster_off[w.seg] + w.c0;
  for (int t = threadIdx.x; t < nc * tc; t += kThreads) {
    const int j = t / tc, col = t - j * tc;
    sc[t] = cb[(int64_t)j * nb + col];
  }
  __syncthreads();
  const int tx = threadIdx.x % tc, ty = threadIdx.x / tc, nty = kThreads / tc;
  if (ty >= nty) return;
  const int col = w.c0 + tx;
  const float alpha = __ldg(scales + s.bucket0 + col), beta = __ldg(scales + n_buckets + s.bucket0 + col);
  const float ra = __ldg(scales + 2 * n_buckets + s.bucket0 + col);
  uint8_t* io = idx_out ? idx_out + idx_base[w.seg] : nullptr;
  const int64_t rend = w.start + w.count;
  for (int64_t r = w.start + ty; r < rend; r += nty) {
    const int64_t i = r * nb + col;
    if (i >= s.numel) break;
    int id;
    s.dst[i] = nuq_one_col(__ldg(s.src + i), alpha, beta, ra, sc + tx, tc, nc, &id);
    if (io) io[i] = (uint8_t)id;
  }
}

// quantile init, one CTA per bucket: the bucket's rows (padding copies included, as in the reference's percentile over
// the padded [bucket_size, nb] matrix) are bitonic-sorted ascending in shared memory; centroid j is the element at
// ascending position pos[seg * 256 + j] (= rows - 1 - the descending 'nearest' rank), normalised with the bucket's fp32
// (w - beta) / alpha.  x -> x_n is monotone non-decreasing, so sorting the raw weights selects the same element.
// Rows 2^bits .. K-1 of the codebook are zeroed.  work[]: seg, c0 = bucket, count = rows, ncol_tile = K.
constexpr int kQinitThreads = 512;

__global__ void __launch_bounds__(kQinitThreads)
nuq_bucket_qinit_kernel(const pf_uq_seg* __restrict__ segs, const pf_work* __restrict__ work,
                        const int32_t* __restrict__ pos, const float* __restrict__ scales, int n_buckets,
                        float* __restrict__ clusters, const int64_t* __restrict__ cluster_off) {
  extern __shared__ float sv[];
  const pf_work w = work[blockIdx.x];
  const pf_uq_seg s = segs[w.seg];
  const int nb = s.ncols, b = w.c0, rows = w.count;
  int p2 = 1;
  while (p2 < rows) p2 <<= 1;
  for (int r = threadIdx.x; r < p2; r += kQinitThreads) {
    int64_t i = (int64_t)r * nb + b;
    sv[r] = r < rows ? __ldg(s.src + (i < s.numel ? i : s.numel - 1)) : INFINITY;
  }
  __syncthreads();
  for (int k = 2; k <= p2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < p2; t += kQinitThreads) {
        const int u = t ^ j;
        if (u > t) {
          const float a = sv[t], c = sv[u];
          const bool up = (t & k) == 0;
          if (up ? (a > c) : (a < c)) {
            sv[t] = c;
            sv[u] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  const int nc = 1 << s.bits;
  const float alpha = __ldg(scales + s.bucket0 + b), beta = __ldg(scales + n_buckets + s.bucket0 + b);
  const float ra = __ldg(scales + 2 * n_buckets + s.bucket0 + b);
  float* cb = clusters + cluster_off[w.seg] + b;
  for (int j = threadIdx.x; j < w.ncol_tile; j += kQinitThreads)
    cb[(int64_t)j * nb] = j < nc ? pf_div_r(__fsub_rn(sv[pos[w.seg * 256 + j]], beta), alpha, ra) : 0.f;
}

// codebook gradient, stage 1: per work tile (the quantize kernel's tiles), one thread per column sums g over its rows
// in row order into smem acc[j][col] (the thread owns the column: no atomics), then writes partial[reserved + ...]
__global__ void __launch_bounds__(kThreads)
nuq_bucket_grad_partial_kernel(const pf_uq_seg* __restrict__ segs, const pf_work* __restrict__ work,
                               const uint8_t* __restrict__ idx, const int64_t* __restrict__ idx_base,
                               float* __restrict__ partial) {
  __shared__ float acc[kBucketSmemFloats];
  const pf_work w = work[blockIdx.x];
  const pf_uq_seg s = segs[w.seg];
  const int nc = 1 << s.bits, tc = w.ncol_tile, nb = s.ncols;
  for (int t = threadIdx.x; t < nc * tc; t += blockDim.x) acc[t] = 0.f;
  __syncthreads();
  const int tx = threadIdx.x;
  if (tx < tc) {
    const uint8_t* io = idx + idx_base[w.seg];
    const int col = w.c0 + tx;
    const int64_t rend = w.start + w.count;
    for (int64_t r = w.start; r < rend; ++r) {
      const int64_t i = r * nb + col;
      if (i >= s.numel) break;
      acc[(int)io[i] * tc + tx] += __ldg(s.src + i);
    }
  }
  __syncthreads();
  float* out = partial + w.reserved;
  for (int t = threadIdx.x; t < nc * tc; t += blockDim.x) out[t] = acc[t];
}

// stage 2, one CTA per column tile: tiles[].start / .count = its range of stage-1 work items (in row order); adds their
// partials in that order and applies alpha_b:  grad[j, b] = alpha_b * sum.  Rows >= 2^bits are not written.
__global__ void __launch_bounds__(kThreads)
nuq_bucket_grad_final_kernel(const pf_uq_seg* __restrict__ segs, const pf_work* __restrict__ tiles,
                             const pf_work* __restrict__ work, const float* __restrict__ partial,
                             const float* __restrict__ scales, float* __restrict__ grad_base,
                             const int64_t* __restrict__ cluster_off) {
  const pf_work tl = tiles[blockIdx.x];
  const pf_uq_seg s = segs[tl.seg];
  const int nc = 1 << s.bits, tc = tl.ncol_tile, nb = s.ncols;
  for (int t = threadIdx.x; t < nc * tc; t += kThreads) {
    float sum = 0.f;
    for (int64_t wi = tl.start; wi < tl.start + tl.count; ++wi) sum += partial[work[wi].reserved + t];
    const int j = t / tc, col = tl.c0 + t - j * tc;
    grad_base[cluster_off[tl.seg] + (int64_t)j * nb + col] = __fmul_rn(sum, __ldg(scales + s.bucket0 + col));
  }
}
}  // namespace

extern "C" {

int pf_nuq_weight_quant(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work,
                        const float* scales_dev, int n_buckets,
                        const float* clusters_dev, uint8_t* idx_out_dev,
                        const int64_t* idx_base_dev, void* stream) {
  PF_REQUIRE(n_work >= 0, "pf_nuq_weight_quant: n_work < 0");
  if (n_work == 0) return PF_OK;
  PF_REQUIRE(segs_dev && work_dev && scales_dev && clusters_dev,
             "pf_nuq_weight_quant: null pointer");
  PF_REQUIRE((idx_out_dev == nullptr) == (idx_base_dev == nullptr),
             "pf_nuq_weight_quant: idx_out and idx_base must be given together");
  nuq_quant_kernel<<<n_work, kThreads, 0, (cudaStream_t)stream>>>(
      segs_dev, work_dev, scales_dev, n_buckets, clusters_dev, nullptr, idx_out_dev, idx_base_dev);
  PF_CHECK_LAUNCH("pf_nuq_weight_quant");
  return PF_OK;
}

int pf_nuq_weight_quant_ex(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work,
                           const float* scales_dev, int n_buckets, const float* clusters_base_dev,
                           const int64_t* cluster_off_dev, uint8_t* idx_out_dev, const int64_t* idx_base_dev,
                           void* stream) {
  PF_REQUIRE(n_work >= 0, "pf_nuq_weight_quant_ex: n_work < 0");
  if (n_work == 0) return PF_OK;
  PF_REQUIRE(segs_dev && work_dev && scales_dev && clusters_base_dev && cluster_off_dev,
             "pf_nuq_weight_quant_ex: null pointer");
  PF_REQUIRE((idx_out_dev == nullptr) == (idx_base_dev == nullptr),
             "pf_nuq_weight_quant_ex: idx_out and idx_base must be given together");
  nuq_quant_kernel<<<n_work, kThreads, 0, (cudaStream_t)stream>>>(
      segs_dev, work_dev, scales_dev, n_buckets, clusters_base_dev, cluster_off_dev, idx_out_dev, idx_base_dev);
  PF_CHECK_LAUNCH("pf_nuq_weight_quant_ex");
  return PF_OK;
}

int pf_nuq_cluster_grad(const pf_uq_seg* gsegs_dev, int n_seg, const pf_work* work_dev, int n_work,
                        const int32_t* work_first_dev, const uint8_t* idx_dev, const int64_t* idx_base_dev,
                        const float* scales_dev, float* partial_ws_dev, float* grad_base_dev,
                        const int64_t* cluster_off_dev, void* stream) {
  PF_REQUIRE(n_seg >= 0 && n_work >= 0, "pf_nuq_cluster_grad: negative count");
  if (n_seg == 0 || n_work == 0) return PF_OK;
  PF_REQUIRE(gsegs_dev && work_dev && work_first_dev && idx_dev && idx_base_dev && scales_dev && partial_ws_dev &&
                 grad_base_dev && cluster_off_dev, "pf_nuq_cluster_grad: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  nuq_cluster_grad_partial_kernel<<<n_work, kThreads, 0, st>>>(gsegs_dev, work_dev, idx_dev, idx_base_dev, partial_ws_dev);
  PF_CHECK_LAUNCH("pf_nuq_cluster_grad(partial)");
  nuq_cluster_grad_final_kernel<<<n_seg, 256, 0, st>>>(gsegs_dev, work_first_dev, partial_ws_dev, scales_dev, grad_base_dev,
                                                      cluster_off_dev);
  PF_CHECK_LAUNCH("pf_nuq_cluster_grad(final)");
  return PF_OK;
}

int pf_nuq_bucket_quant(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work, const float* scales_dev,
                        int n_buckets, const float* clusters_base_dev, const int64_t* cluster_off_dev,
                        uint8_t* idx_out_dev, const int64_t* idx_base_dev, void* stream) {
  PF_REQUIRE(n_work >= 0, "pf_nuq_bucket_quant: n_work < 0");
  if (n_work == 0) return PF_OK;
  PF_REQUIRE(segs_dev && work_dev && scales_dev && clusters_base_dev && cluster_off_dev,
             "pf_nuq_bucket_quant: null pointer");
  PF_REQUIRE((idx_out_dev == nullptr) == (idx_base_dev == nullptr),
             "pf_nuq_bucket_quant: idx_out and idx_base must be given together");
  nuq_bucket_quant_kernel<<<n_work, kThreads, 0, (cudaStream_t)stream>>>(
      segs_dev, work_dev, scales_dev, n_buckets, clusters_base_dev, cluster_off_dev, idx_out_dev, idx_base_dev);
  PF_CHECK_LAUNCH("pf_nuq_bucket_quant");
  return PF_OK;
}

int pf_nuq_bucket_quantile_init(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work, int max_rows,
                                const int32_t* pos_dev, const float* scales_dev, int n_buckets,
                                float* clusters_base_dev, const int64_t* cluster_off_dev, void* stream) {
  PF_REQUIRE(n_work >= 0, "pf_nuq_bucket_quantile_init: n_work < 0");
  if (n_work == 0) return PF_OK;
  PF_REQUIRE(segs_dev && work_dev && pos_dev && scales_dev && clusters_base_dev && cluster_off_dev,
             "pf_nuq_bucket_quantile_init: null pointer");
  PF_REQUIRE(max_rows >= 1 && max_rows <= PF_NUQ_BUCKET_MAX_ROWS,
             "pf_nuq_bucket_quantile_init: bucket rows must be in [1, %d]", PF_NUQ_BUCKET_MAX_ROWS);
  int p2 = 1;
  while (p2 < max_rows) p2 <<= 1;
  const size_t smem = (size_t)p2 * sizeof(float);
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(nuq_bucket_qinit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)smem);
    PF_REQUIRE(e == cudaSuccess, "pf_nuq_bucket_quantile_init: %s", cudaGetErrorString(e));
  }
  nuq_bucket_qinit_kernel<<<n_work, kQinitThreads, smem, (cudaStream_t)stream>>>(
      segs_dev, work_dev, pos_dev, scales_dev, n_buckets, clusters_base_dev, cluster_off_dev);
  PF_CHECK_LAUNCH("pf_nuq_bucket_quantile_init");
  return PF_OK;
}

int pf_nuq_bucket_cluster_grad(const pf_uq_seg* gsegs_dev, const pf_work* work_dev, int n_work,
                               const pf_work* tiles_dev, int n_tiles, const uint8_t* idx_dev,
                               const int64_t* idx_base_dev, const float* scales_dev, float* partial_ws_dev,
                               float* grad_base_dev, const int64_t* cluster_off_dev, void* stream) {
  PF_REQUIRE(n_work >= 0 && n_tiles >= 0, "pf_nuq_bucket_cluster_grad: negative count");
  if (n_work == 0 || n_tiles == 0) return PF_OK;
  PF_REQUIRE(gsegs_dev && work_dev && tiles_dev && idx_dev && idx_base_dev && scales_dev && partial_ws_dev &&
                 grad_base_dev && cluster_off_dev, "pf_nuq_bucket_cluster_grad: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  nuq_bucket_grad_partial_kernel<<<n_work, kThreads, 0, st>>>(gsegs_dev, work_dev, idx_dev, idx_base_dev,
                                                              partial_ws_dev);
  PF_CHECK_LAUNCH("pf_nuq_bucket_cluster_grad(partial)");
  nuq_bucket_grad_final_kernel<<<n_tiles, kThreads, 0, st>>>(gsegs_dev, tiles_dev, work_dev, partial_ws_dev, scales_dev,
                                                            grad_base_dev, cluster_off_dev);
  PF_CHECK_LAUNCH("pf_nuq_bucket_cluster_grad(final)");
  return PF_OK;
}

}  // extern "C"
