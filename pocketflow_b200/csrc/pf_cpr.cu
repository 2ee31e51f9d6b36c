// pf_cpr.cu — the channel-selection phase of the remastered channel-pruning learner (SURVEY §8 f5).
//
// Reference: /root/reference/learners/channel_pruning_rmt/learner.py
//   :651-725  sample R x S x Cin input patches of the pruned model and Cout outputs of the full model at random output
//             positions (zero-filled outside the image; SAME's leading pads :665-672), check patch * W == output
//   :748-769  feature matrix F[(n,o), c] = sum_rs X[n, rs, c] W[rs, c, o], response y[(n,o)] = Y[n, o];
//             G = F^T F, b = F^T y in float64, both divided by ||G||_F
//   :432-468  ISTA in float32: m <- prox(m - lr (G m - b), gamma lr), prox(x, t) = x - t | x + t | 0
//   :817-839  least-squares refit on the kept channels: X with the dropped channels' columns zeroed, W * [|m| > 0]
// The refit's GEMMs are the ordinary 1x1 conv fwd / wgrad kernels over N "pixels" of K = R*S*Cin channels and its
// update is pf_adam_step; this file holds what has no counterpart elsewhere:
//   pf_cpr_sample         one launch per cached mini-batch: a row gather, exact (hi + lo where the executor keeps only
//                         split-bf16 planes of the conv input: the operand the conv consumed)
//   pf_cpr_gram           F in float64 over bounded row chunks, G_aug += F_aug^T F_aug on the CUDA-core FP64 pipes
//                         (F_aug = [F | y], so b is G_aug's last column), upper-triangle tiles then mirrored, one
//                         fixed-order Frobenius norm, the normalised G / b in float64 and their float32 copies for ISTA
//   pf_cpr_ista           all iterations of one gamma in ONE cooperative launch (grid-wide sync between iterations);
//                         one warp per row of G m, fixed lane order and shuffle tree, so the mask and its nnz count
//                         are the same bits run after run whatever the grid size
//   pf_cpr_mask_channels  a[.., t, c, k] *= [|m[c]| > 0]  (the kept-channel patch matrix and the final W * bnry)
// Every reduction has a fixed order: results are deterministic.
//
// The LASSO channel-pruning learner (/root/reference/learners/channel_pruning/channel_pruner.py) has its own entry
// points here, on the same Gram machinery:
//   pf_cp_sample      the patches of the current model's conv input and the full model's conv outputs at positions
//                     shared by a whole batch (:263-341, :391-412); Y in float64, plus the residual branch difference
//                     full - current of the block's Add output, gathered at the Add's own positions (:579-586)
//   pf_cp_gram        the design matrix product[(s, o), c] = sum_hw X[s, hw, c] W2[hw, c, o] over the sampled rows
//                     (:468-476) and G_aug = [P | y]^T [P | y] in float64, unnormalised
//   pf_cp_normal_eq   [X_k | Y]^T [X_k | Y] in float64 over every row: the normal equations of the refit of the kept
//                     input channels (:569-573)
#include <cooperative_groups.h>
#include <cuda_bf16.h>

#include "pf_common.cuh"

namespace cg = cooperative_groups;

namespace {

// ------------------------------------------------------------------------------------------------ shared pieces
// the R x S x C input patch at output position (n, oh, ow) into xr (zero outside the image), one block per row
__device__ __forceinline__ void gather_patch(const pf_conv_desc& d, const float* __restrict__ x,
                                             const __nv_bfloat16* __restrict__ xhi,
                                             const __nv_bfloat16* __restrict__ xlo, int n, int oh, int ow,
                                             float* __restrict__ xr) {
  const int K = d.r * d.s * d.c;
  for (int e = threadIdx.x; e < K; e += blockDim.x) {
    const int t = e / d.c, c = e - t * d.c;
    const int r = t / d.s, s = t - r * d.s;
    const int ih = oh * d.stride_h - d.pad_t + r, iw = ow * d.stride_w - d.pad_l + s;
    float v = 0.f;
    if (ih >= 0 && ih < d.h && iw >= 0 && iw < d.w) {
      const size_t i = (((size_t)n * d.h + ih) * d.w + iw) * d.c + c;
      v = x ? x[i] : __fadd_rn(__bfloat162float(xhi[i]), __bfloat162float(xlo[i]));
    }
    xr[e] = v;
  }
}

// sum_t X[src, t, c] W[t, c, o] in float64, in t order
__device__ __forceinline__ double patch_times_kernel(const float* __restrict__ X, const float* __restrict__ w,
                                                     int64_t src, int64_t K, int rs, int cin, int cout, int c, int o) {
  double acc = 0.0;
  const float* xr = X + src * K + c;
  for (int t = 0; t < rs; ++t) acc = fma((double)xr[(int64_t)t * cin], (double)w[((int64_t)t * cin + c) * cout + o], acc);
  return acc;
}

// ------------------------------------------------------------------------------------------------ sampler
__global__ void __launch_bounds__(256)
cpr_sample_kernel(pf_conv_desc d, const float* __restrict__ x, const __nv_bfloat16* __restrict__ xhi,
                  const __nv_bfloat16* __restrict__ xlo, const float* __restrict__ y, const float* __restrict__ bias,
                  const int32_t* __restrict__ rows, float* __restrict__ X, float* __restrict__ Y) {
  const int4 row = reinterpret_cast<const int4*>(rows)[blockIdx.x];    // (n, oh, ow, dst)
  if (row.w < 0) return;
  const int K = d.r * d.s * d.c;
  gather_patch(d, x, xhi, xlo, row.x, row.y, row.z, X + (size_t)row.w * K);
  const float* yr = y + (((size_t)row.x * d.p + row.y) * d.q + row.z) * d.k;
  for (int k = threadIdx.x; k < d.k; k += blockDim.x)
    Y[(size_t)row.w * d.k + k] = bias ? __fsub_rn(yr[k], bias[k]) : yr[k];
}

// ------------------------------------------------------------------------------------------------ Gram matrix
// Ft[c][m] (c-major, ld = mcap): m = j*cout + o over the chunk's rows j; c < cin: F, c == cin: y
__global__ void __launch_bounds__(256)
cpr_feature_kernel(const float* __restrict__ X, const float* __restrict__ Y, const int32_t* __restrict__ idx, int j0,
                   int nj, const float* __restrict__ w, int rs, int cin, int cout, double* __restrict__ Ft,
                   int64_t mcap) {
  const int64_t m_n = (int64_t)nj * cout, total = m_n * (cin + 1);
  const int64_t K = (int64_t)rs * cin;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / m_n);
    const int64_t m = i - (int64_t)c * m_n;
    const int j = (int)(m / cout), o = (int)(m - (int64_t)j * cout);
    const int64_t src = idx[j0 + j];
    double acc;
    if (c == cin) {
      acc = (double)Y[src * cout + o];
    } else {
      acc = patch_times_kernel(X, w, src, K, rs, cin, cout, c, o);
    }
    Ft[(int64_t)c * mcap + m] = acc;
  }
}

constexpr int GT = 64, GK = 16;    // G tile 64 x 64, k-step 16; 256 threads x (4 x 4) accumulators

// G[i][j] += sum_m Ft[i][m] Ft[j][m] for the tiles with ti <= tj (n = cin + 1 rows of Ft)
__global__ void __launch_bounds__(256)
cpr_syrk_kernel(const double* __restrict__ Ft, int64_t mcap, int64_t m_n, int n, double* __restrict__ G) {
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (ti > tj) return;
  __shared__ double sa[GK][GT + 1], sb[GK][GT + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int i0 = ti * GT, j0 = tj * GT;
  double acc[4][4] = {};
  for (int64_t m0 = 0; m0 < m_n; m0 += GK) {
    for (int e = threadIdx.x; e < GK * GT; e += 256) {
      const int r = e / GK, kk = e - r * GK;           // consecutive threads: consecutive m (coalesced)
      const int64_t m = m0 + kk;
      const bool in_m = m < m_n;
      sa[kk][r] = (in_m && i0 + r < n) ? Ft[(int64_t)(i0 + r) * mcap + m] : 0.0;
      sb[kk][r] = (in_m && j0 + r < n) ? Ft[(int64_t)(j0 + r) * mcap + m] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GK; ++kk) {
      double a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        a[u] = sa[kk][ty + 16 * u];
        b[u] = sb[kk][tx + 16 * u];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = fma(a[u], b[v], acc[u][v]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int i = i0 + ty + 16 * u, j = j0 + tx + 16 * v;
      if (i < n && j < n) G[(int64_t)i * n + j] += acc[u][v];
    }
}

// mirror the upper triangle and sum the squares of G (the first cin x cin block) in a fixed order: one block
__global__ void __launch_bounds__(1024)
cpr_norm_kernel(double* __restrict__ G, int n, int cin, double* __restrict__ norm_out) {
  __shared__ double sh[1024];
  double acc = 0.0;
  for (int64_t e = threadIdx.x; e < (int64_t)n * n; e += 1024) {
    const int i = (int)(e / n), j = (int)(e - (int64_t)i * n);
    if (i > j) continue;
    const double v = G[e];
    if (i < j) G[(int64_t)j * n + i] = v;
    if (j < cin) acc = fma(v, v, (i < j) ? fma(v, v, acc) : acc);   // (i, j) and (j, i)
  }
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 512; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) norm_out[0] = sqrt(sh[0]);
}

// G /= ||G||, b /= ||G|| in float64 and their float32 copies (the float32 placeholders of the LASSO graph, :438-439)
__global__ void __launch_bounds__(256)
cpr_scale_kernel(double* __restrict__ G, int n, int cin, const double* __restrict__ norm, float* __restrict__ gf,
                 float* __restrict__ bf) {
  const double s = norm[0];
  for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < (int64_t)cin * n; e += (int64_t)gridDim.x * 256) {
    const int i = (int)(e / n), j = (int)(e - (int64_t)i * n);
    const double v = G[e] / s;
    G[e] = v;
    if (j < cin) gf[(int64_t)i * cin + j] = (float)v;
    else bf[i] = (float)v;
  }
}

// ------------------------------------------------------------------------------------------------ ISTA
__global__ void __launch_bounds__(256)
cpr_ista_kernel(const float* __restrict__ G, const float* __restrict__ b, const float* __restrict__ m0, int cin,
                float lr, float thr, int iters, float* m_out, float* ws, int* __restrict__ nnz) {
  // (m_out / ws are written and re-read across the grid-wide barrier: plain loads, never the read-only path)
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31;
  const int warp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int nwarps = (int)((gridDim.x * blockDim.x) >> 5);
  int count = 0;
  for (int it = 0; it < iters; ++it) {
    const float* cur = it == 0 ? m0 : ws + (size_t)(it & 1) * cin;
    float* nxt = it == iters - 1 ? m_out : ws + (size_t)((it + 1) & 1) * cin;
    for (int i = warp; i < cin; i += nwarps) {
      const float* gr = G + (size_t)i * cin;
      float acc = 0.f;
      for (int j = lane; j < cin; j += 32) acc = fmaf(gr[j], cur[j], acc);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
      // mask - lr * (matmul(xt_x, mask) - xt_y), then prox_mapping(., gamma * lr)  (:450-452)
      const float x = __fsub_rn(cur[i], __fmul_rn(lr, __fsub_rn(acc, b[i])));
      const float y = x > thr ? __fsub_rn(x, thr) : (x < -thr ? __fadd_rn(x, thr) : 0.f);
      if (lane == 0) {
        nxt[i] = y;
        if (it == iters - 1) count += (y != 0.f);
      }
    }
    if (it < iters - 1) grid.sync();
  }
  if (iters == 0)
    for (int i = warp; i < cin; i += nwarps)
      if (lane == 0) {
        m_out[i] = m0[i];
        count += (m0[i] != 0.f);
      }
  if (lane == 0 && count) atomicAdd(nnz, count);
}

__global__ void __launch_bounds__(256)
cpr_mask_channels_kernel(float* __restrict__ a, int64_t total, int cin, int inner, const float* __restrict__ m) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int c = (int)((i / inner) % cin);
    a[i] = __fmul_rn(a[i], fabsf(m[c]) > 0.f ? 1.f : 0.f);
  }
}

// ------------------------------------------------------------------------------------------------ LASSO learner
// rows: int32 [n, 8] = (n, oh, ow, dst, rh, rw, -, -): the conv's output position and the Add's (when res_full is set)
__global__ void __launch_bounds__(256)
cp_sample_kernel(pf_conv_desc d, const float* __restrict__ x, const __nv_bfloat16* __restrict__ xhi,
                 const __nv_bfloat16* __restrict__ xlo, const float* __restrict__ y, const float* __restrict__ bias,
                 const float* __restrict__ res_full, const float* __restrict__ res_cur, int res_h, int res_w,
                 const int32_t* __restrict__ rows, float* __restrict__ X, double* __restrict__ Y) {
  const int4 row = reinterpret_cast<const int4*>(rows)[2 * blockIdx.x];
  const int4 rrow = reinterpret_cast<const int4*>(rows)[2 * blockIdx.x + 1];
  if (row.w < 0) return;
  const int K = d.r * d.s * d.c;
  gather_patch(d, x, xhi, xlo, row.x, row.y, row.z, X + (size_t)row.w * K);
  const float* yr = y + (((size_t)row.x * d.p + row.y) * d.q + row.z) * d.k;
  const size_t ri = (((size_t)row.x * res_h + rrow.x) * res_w + rrow.y) * d.k;
  for (int k = threadIdx.x; k < d.k; k += blockDim.x) {
    double v = (double)(bias ? __fsub_rn(yr[k], bias[k]) : yr[k]);
    if (res_full) v = v + ((double)res_full[ri + k] - (double)res_cur[ri + k]);
    Y[(size_t)row.w * d.k + k] = v;
  }
}

// Ft[c][m] (ld = mcap), m = j*cout + o over the chunk's sampled rows j: c < cin the design matrix, c == cin y
__global__ void __launch_bounds__(256)
cp_product_kernel(const float* __restrict__ X, const double* __restrict__ Y, const int32_t* __restrict__ idx, int j0,
                  int nj, const float* __restrict__ w, int rs, int cin, int cout, double* __restrict__ Ft, int64_t mcap) {
  const int64_t m_n = (int64_t)nj * cout, total = m_n * (cin + 1);
  const int64_t K = (int64_t)rs * cin;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / m_n);
    const int64_t m = i - (int64_t)c * m_n;
    const int j = (int)(m / cout), o = (int)(m - (int64_t)j * cout);
    const int64_t src = idx[j0 + j];
    double acc;
    if (c == cin) {
      acc = Y[src * cout + o];
    } else {
      acc = patch_times_kernel(X, w, src, K, rs, cin, cout, c, o);
    }
    Ft[(int64_t)c * mcap + m] = acc;
  }
}

// Ft[c][m] (ld = mcap) over the chunk's rows m: c < ncols column cols[c] of X, then the cout columns of Y
__global__ void __launch_bounds__(256)
cp_columns_kernel(const float* __restrict__ X, const double* __restrict__ Y, const int32_t* __restrict__ cols, int ncols,
                  int64_t K, int cout, int64_t r0, int64_t nr, double* __restrict__ Ft, int64_t mcap) {
  const int64_t total = nr * (ncols + cout);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / nr);
    const int64_t m = i - (int64_t)c * nr, row = r0 + m;
    Ft[(int64_t)c * mcap + m] = c < ncols ? (double)X[row * K + cols[c]] : Y[row * cout + (c - ncols)];
  }
}

inline unsigned grid_for(int64_t n, int per_sm) {
  int64_t g = (n + 255) / 256;
  const int64_t cap = (int64_t)PF_NUM_SMS * per_sm;
  if (g > cap) g = cap;
  return (unsigned)(g < 1 ? 1 : g);
}

}  // namespace

extern "C" {

int pf_cpr_sample(const pf_conv_desc* d, const float* x_dev, const void* x_hi_dev, const void* x_lo_dev,
                  const float* y_dev, const float* bias_dev, const int32_t* rows_dev, int n_rows, float* X_dev,
                  float* Y_dev, void* stream) {
  PF_REQUIRE(d != nullptr && n_rows >= 0, "pf_cpr_sample: bad arguments");
  PF_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0 && d->c > 0 && d->k > 0 && d->r > 0 && d->s > 0 && d->p > 0 &&
                 d->q > 0 && d->stride_h > 0 && d->stride_w > 0 && d->pad_t >= 0 && d->pad_l >= 0,
             "pf_cpr_sample: non-positive dimension in conv descriptor");
  PF_REQUIRE(x_dev || (x_hi_dev && x_lo_dev), "pf_cpr_sample: no input (fp32 tensor or hi/lo planes)");
  PF_REQUIRE(y_dev && X_dev && Y_dev, "pf_cpr_sample: null pointer");
  if (n_rows == 0) return PF_OK;
  PF_REQUIRE(rows_dev && ((uintptr_t)rows_dev & 15) == 0, "pf_cpr_sample: rows must be 16-byte aligned int32 [n, 4]");
  cpr_sample_kernel<<<n_rows, 256, 0, (cudaStream_t)stream>>>(*d, x_dev, (const __nv_bfloat16*)x_hi_dev,
                                                               (const __nv_bfloat16*)x_lo_dev, y_dev, bias_dev, rows_dev,
                                                               X_dev, Y_dev);
  PF_CHECK_LAUNCH("pf_cpr_sample");
  return PF_OK;
}

int64_t pf_cpr_gram_ws_doubles(int cin, int cout, int64_t chunk_rows) {
  if (cin < 1 || cout < 1 || chunk_rows < 1) return 0;
  return (int64_t)(cin + 1) * chunk_rows * cout;
}

int pf_cpr_gram(const float* X_dev, const float* Y_dev, const int32_t* idx_dev, int n_idx, const float* w_dev, int rs,
                int cin, int cout, double* ws_dev, int64_t chunk_rows, double* g_dev, float* gf_dev, float* bf_dev,
                void* stream) {
  PF_REQUIRE(n_idx >= 1 && rs >= 1 && cin >= 1 && cout >= 1 && chunk_rows >= 1, "pf_cpr_gram: bad shape");
  PF_REQUIRE(X_dev && Y_dev && idx_dev && w_dev && ws_dev && g_dev && gf_dev && bf_dev, "pf_cpr_gram: null pointer");
  PF_REQUIRE(cin < 65536 && (int64_t)rs * cin < (1ll << 31), "pf_cpr_gram: kernel too large");
  cudaStream_t st = (cudaStream_t)stream;
  const int n = cin + 1;
  PF_CUDA(cudaMemsetAsync(g_dev, 0, sizeof(double) * ((size_t)n * n + 1), st));
  const int64_t mcap = chunk_rows * cout;
  const dim3 tiles((n + GT - 1) / GT, (n + GT - 1) / GT);
  for (int j0 = 0; j0 < n_idx; j0 += (int)chunk_rows) {
    const int nj = (int)((n_idx - j0) < chunk_rows ? (n_idx - j0) : chunk_rows);
    const int64_t m_n = (int64_t)nj * cout;
    cpr_feature_kernel<<<grid_for(m_n * n, 16), 256, 0, st>>>(X_dev, Y_dev, idx_dev, j0, nj, w_dev, rs, cin, cout,
                                                              ws_dev, mcap);
    PF_CHECK_LAUNCH("pf_cpr_gram/feature");
    cpr_syrk_kernel<<<tiles, 256, 0, st>>>(ws_dev, mcap, m_n, n, g_dev);
    PF_CHECK_LAUNCH("pf_cpr_gram/syrk");
  }
  double* norm = g_dev + (size_t)n * n;
  cpr_norm_kernel<<<1, 1024, 0, st>>>(g_dev, n, cin, norm);
  PF_CHECK_LAUNCH("pf_cpr_gram/norm");
  cpr_scale_kernel<<<grid_for((int64_t)cin * n, 8), 256, 0, st>>>(g_dev, n, cin, norm, gf_dev, bf_dev);
  PF_CHECK_LAUNCH("pf_cpr_gram/scale");
  return PF_OK;
}

int pf_cpr_ista(const float* g_dev, const float* b_dev, const float* m0_dev, int cin, float lr, float gamma, int iters,
                float* m_dev, float* ws_dev, int32_t* nnz_dev, void* stream) {
  PF_REQUIRE(cin >= 1 && iters >= 0, "pf_cpr_ista: bad shape");
  PF_REQUIRE(g_dev && b_dev && m0_dev && m_dev && ws_dev && nnz_dev, "pf_cpr_ista: null pointer");
  PF_REQUIRE(m_dev != m0_dev, "pf_cpr_ista: m and m0 must not alias");
  cudaStream_t st = (cudaStream_t)stream;
  static int max_blocks = 0;
  if (max_blocks == 0) {
    int per_sm = 0;
    PF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cpr_ista_kernel, 256, 0));
    max_blocks = per_sm * PF_NUM_SMS;
    PF_REQUIRE(max_blocks > 0, "pf_cpr_ista: kernel cannot be resident");
  }
  int blocks = (cin + 7) / 8;                         // 8 warps per block, one row each per sweep
  if (blocks > max_blocks) blocks = max_blocks;
  PF_CUDA(cudaMemsetAsync(nnz_dev, 0, sizeof(int32_t), st));
  // gamma * lr in float32 (the gamma placeholder times the python-float learning rate, :452)
  float thr = gamma * lr;
  void* args[] = {(void*)&g_dev, (void*)&b_dev, (void*)&m0_dev, (void*)&cin, (void*)&lr, (void*)&thr, (void*)&iters,
                  (void*)&m_dev, (void*)&ws_dev, (void*)&nnz_dev};
  PF_CUDA(cudaLaunchCooperativeKernel((const void*)cpr_ista_kernel, dim3(blocks), dim3(256), args, 0, st));
  PF_CHECK_LAUNCH("pf_cpr_ista");
  return PF_OK;
}

int pf_cpr_mask_channels(float* a_dev, int64_t rows, int rs, int cin, int inner, const float* m_dev, void* stream) {
  PF_REQUIRE(rows >= 0 && rs >= 1 && cin >= 1 && inner >= 1, "pf_cpr_mask_channels: bad shape");
  if (rows == 0) return PF_OK;
  PF_REQUIRE(a_dev && m_dev, "pf_cpr_mask_channels: null pointer");
  const int64_t total = rows * rs * cin * (int64_t)inner;
  cpr_mask_channels_kernel<<<grid_for(total, 8), 256, 0, (cudaStream_t)stream>>>(a_dev, total, cin, inner, m_dev);
  PF_CHECK_LAUNCH("pf_cpr_mask_channels");
  return PF_OK;
}


int pf_cp_sample(const pf_conv_desc* d, const float* x_dev, const void* x_hi_dev, const void* x_lo_dev,
                 const float* y_dev, const float* bias_dev, const float* res_full_dev, const float* res_cur_dev,
                 int res_h, int res_w, const int32_t* rows_dev, int n_rows, float* X_dev, double* Y_dev, void* stream) {
  PF_REQUIRE(d != nullptr && n_rows >= 0, "pf_cp_sample: bad arguments");
  PF_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0 && d->c > 0 && d->k > 0 && d->r > 0 && d->s > 0 && d->p > 0 &&
                 d->q > 0 && d->stride_h > 0 && d->stride_w > 0 && d->pad_t >= 0 && d->pad_l >= 0,
             "pf_cp_sample: non-positive dimension in conv descriptor");
  PF_REQUIRE(x_dev || (x_hi_dev && x_lo_dev), "pf_cp_sample: no input (fp32 tensor or hi/lo planes)");
  PF_REQUIRE(y_dev && X_dev && Y_dev, "pf_cp_sample: null pointer");
  PF_REQUIRE(!res_full_dev == !res_cur_dev, "pf_cp_sample: the residual needs both the full and the current tensor");
  PF_REQUIRE(!res_full_dev || (res_h > 0 && res_w > 0), "pf_cp_sample: bad residual shape");
  if (n_rows == 0) return PF_OK;
  PF_REQUIRE(rows_dev && ((uintptr_t)rows_dev & 15) == 0, "pf_cp_sample: rows must be 16-byte aligned int32 [n, 8]");
  cp_sample_kernel<<<n_rows, 256, 0, (cudaStream_t)stream>>>(*d, x_dev, (const __nv_bfloat16*)x_hi_dev,
                                                              (const __nv_bfloat16*)x_lo_dev, y_dev, bias_dev,
                                                              res_full_dev, res_cur_dev, res_h, res_w, rows_dev, X_dev,
                                                              Y_dev);
  PF_CHECK_LAUNCH("pf_cp_sample");
  return PF_OK;
}

int pf_cp_gram(const float* X_dev, const double* Y_dev, const int32_t* idx_dev, int n_idx, const float* w_dev, int rs,
               int cin, int cout, double* ws_dev, int64_t chunk_rows, double* g_dev, void* stream) {
  PF_REQUIRE(n_idx >= 1 && rs >= 1 && cin >= 1 && cout >= 1 && chunk_rows >= 1, "pf_cp_gram: bad shape");
  PF_REQUIRE(X_dev && Y_dev && idx_dev && w_dev && ws_dev && g_dev, "pf_cp_gram: null pointer");
  PF_REQUIRE(cin < 65536 && (int64_t)rs * cin < (1ll << 31), "pf_cp_gram: kernel too large");
  cudaStream_t st = (cudaStream_t)stream;
  const int n = cin + 1;
  PF_CUDA(cudaMemsetAsync(g_dev, 0, sizeof(double) * ((size_t)n * n + 1), st));
  const int64_t mcap = chunk_rows * cout;
  const dim3 tiles((n + GT - 1) / GT, (n + GT - 1) / GT);
  for (int j0 = 0; j0 < n_idx; j0 += (int)chunk_rows) {
    const int nj = (int)((n_idx - j0) < chunk_rows ? (n_idx - j0) : chunk_rows);
    const int64_t m_n = (int64_t)nj * cout;
    cp_product_kernel<<<grid_for(m_n * n, 16), 256, 0, st>>>(X_dev, Y_dev, idx_dev, j0, nj, w_dev, rs, cin, cout, ws_dev,
                                                             mcap);
    PF_CHECK_LAUNCH("pf_cp_gram/product");
    cpr_syrk_kernel<<<tiles, 256, 0, st>>>(ws_dev, mcap, m_n, n, g_dev);
    PF_CHECK_LAUNCH("pf_cp_gram/syrk");
  }
  cpr_norm_kernel<<<1, 1024, 0, st>>>(g_dev, n, cin, g_dev + (size_t)n * n);     // (mirrors; the norm is not used)
  PF_CHECK_LAUNCH("pf_cp_gram/mirror");
  return PF_OK;
}

int pf_cp_normal_eq(const float* X_dev, const double* Y_dev, int64_t n_rows, int64_t K, int cout, const int32_t* cols_dev,
                    int ncols, double* ws_dev, int64_t chunk_rows, double* g_dev, void* stream) {
  PF_REQUIRE(n_rows >= 1 && K >= 1 && cout >= 1 && ncols >= 1 && ncols <= K && chunk_rows >= 1,
             "pf_cp_normal_eq: bad shape");
  PF_REQUIRE(X_dev && Y_dev && cols_dev && ws_dev && g_dev, "pf_cp_normal_eq: null pointer");
  PF_REQUIRE((int64_t)ncols + cout < 65536, "pf_cp_normal_eq: too many columns");
  cudaStream_t st = (cudaStream_t)stream;
  const int n = ncols + cout;
  PF_CUDA(cudaMemsetAsync(g_dev, 0, sizeof(double) * ((size_t)n * n + 1), st));
  const dim3 tiles((n + GT - 1) / GT, (n + GT - 1) / GT);
  for (int64_t r0 = 0; r0 < n_rows; r0 += chunk_rows) {
    const int64_t nr = (n_rows - r0) < chunk_rows ? (n_rows - r0) : chunk_rows;
    cp_columns_kernel<<<grid_for(nr * n, 16), 256, 0, st>>>(X_dev, Y_dev, cols_dev, ncols, K, cout, r0, nr, ws_dev,
                                                             chunk_rows);
    PF_CHECK_LAUNCH("pf_cp_normal_eq/columns");
    cpr_syrk_kernel<<<tiles, 256, 0, st>>>(ws_dev, chunk_rows, nr, n, g_dev);
    PF_CHECK_LAUNCH("pf_cp_normal_eq/syrk");
  }
  cpr_norm_kernel<<<1, 1024, 0, st>>>(g_dev, n, n, g_dev + (size_t)n * n);        // (mirrors; the norm is not used)
  PF_CHECK_LAUNCH("pf_cp_normal_eq/mirror");
  return PF_OK;
}

}  // extern "C"
