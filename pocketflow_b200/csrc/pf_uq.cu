// pf_uq.cu — uniform fake-quantization kernels (HBM-bound; 8 B/element algorithmic).
//
// Replaces the TensorFlow op chain emitted by UniformQuantization.__uniform_quantize
// (/root/reference/learners/uniform_quantization/utils.py:163-289): reduce_max, reduce_min, sub,
// add(eps), sub, realdiv, mul, round, realdiv, mul, add (+reshape/concat/slice for buckets) — 9-12
// separate full-tensor kernels per layer in the reference — by
//   (1) one multi-tensor min/max launch for every layer's buckets (warp-shuffle + smem + one
//       ordered-uint atomic per bucket per CTA), and
//   (2) one multi-tensor quantize launch (128-bit loads/stores, the weights re-read from L2).
// Activations (per-tensor range, up to 784 MiB each on ResNet-50) use the same two phases with
// persistent grid-stride kernels sized to a multiple of the SM count.
#include "pf_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxColTile = 1024;

// ------------------------------------------------------------------ weight min/max (multi-tensor)
__device__ __forceinline__ float ld_clamped(const float* __restrict__ src, int64_t i, int64_t numel) {
  return __ldg(src + (i < numel ? i : numel - 1));
}

template <int V>
__device__ __forceinline__ void minmax_coltile(const pf_uq_seg& s, const pf_work& w,
                                               uint32_t* __restrict__ mn_enc,
                                               uint32_t* __restrict__ mx_enc, uint32_t* smn,
                                               uint32_t* smx) {
  const int tc = w.ncol_tile;
  const int nvec = tc / V;
  const int nty = kThreads / nvec;
  const int tx = threadIdx.x % nvec;
  const int ty = threadIdx.x / nvec;
  for (int t = threadIdx.x; t < tc; t += kThreads) {
    smn[t] = 0xFFFFFFFFu;
    smx[t] = 0u;
  }
  __syncthreads();
  float mn[V], mx[V];
#pragma unroll
  for (int j = 0; j < V; ++j) {
    mn[j] = INFINITY;
    mx[j] = -INFINITY;
  }
  if (ty < nty) {
    const int64_t rend = w.start + w.count;
    const int64_t col = (int64_t)w.c0 + (int64_t)tx * V;
    for (int64_t r = w.start + ty; r < rend; r += nty) {
      const int64_t i = r * (int64_t)s.ncols + col;
      if (V == 4 && i + 3 < s.numel) {
        float4 v = pf_ld_stream(s.src + i);
        mn[0] = fminf(mn[0], v.x); mx[0] = fmaxf(mx[0], v.x);
        mn[1 % V] = fminf(mn[1 % V], v.y); mx[1 % V] = fmaxf(mx[1 % V], v.y);
        mn[2 % V] = fminf(mn[2 % V], v.z); mx[2 % V] = fmaxf(mx[2 % V], v.z);
        mn[3 % V] = fminf(mn[3 % V], v.w); mx[3 % V] = fmaxf(mx[3 % V], v.w);
      } else {
#pragma unroll
        for (int j = 0; j < V; ++j) {
          float v = ld_clamped(s.src, i + j, s.numel);
          mn[j] = fminf(mn[j], v);
          mx[j] = fmaxf(mx[j], v);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < V; ++j) {
      if (mn[j] <= mx[j]) {  // thread saw at least one row
        atomicMin(&smn[tx * V + j], pf_enc(mn[j]));
        atomicMax(&smx[tx * V + j], pf_enc(mx[j]));
      }
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < tc; t += kThreads) {
    if (smx[t] != 0u || smn[t] != 0xFFFFFFFFu) {
      atomicMin(&mn_enc[s.bucket0 + w.c0 + t], smn[t]);
      atomicMax(&mx_enc[s.bucket0 + w.c0 + t], smx[t]);
    }
  }
}

__device__ __forceinline__ void block_minmax_to_slot(float mn, float mx, uint32_t* mn_slot,
                                                     uint32_t* mx_slot) {
  __shared__ float s_mn[kThreads / 32], s_mx[kThreads / 32];
  mn = pf_warp_min(mn);
  mx = pf_warp_max(mx);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) {
    s_mn[wid] = mn;
    s_mx[wid] = mx;
  }
  __syncthreads();
  if (wid == 0) {
    mn = lane < kThreads / 32 ? s_mn[lane] : INFINITY;
    mx = lane < kThreads / 32 ? s_mx[lane] : -INFINITY;
    mn = pf_warp_min(mn);
    mx = pf_warp_max(mx);
    if (lane == 0 && mn <= mx) {
      atomicMin(mn_slot, pf_enc(mn));
      atomicMax(mx_slot, pf_enc(mx));
    }
  }
}

__global__ void __launch_bounds__(kThreads)
uq_weight_minmax_kernel(const pf_uq_seg* __restrict__ segs, const pf_work* __restrict__ work,
                        uint32_t* __restrict__ mn_enc, uint32_t* __restrict__ mx_enc) {
  __shared__ uint32_t smn[kMaxColTile], smx[kMaxColTile];
  const pf_work w = work[blockIdx.x];
  const pf_uq_seg s = segs[w.seg];
  if (w.kind == 1) {
    if ((s.ncols & 3) == 0)
      minmax_coltile<4>(s, w, mn_enc, mx_enc, smn, smx);
    else
      minmax_coltile<1>(s, w, mn_enc, mx_enc, smn, smx);
    return;
  }
  // kind 0: per-layer range over a flat chunk (start is a multiple of 4)
  float mn = INFINITY, mx = -INFINITY;
  const int64_t end = w.start + w.count;
  for (int64_t i = w.start + (int64_t)threadIdx.x * 4; i < end; i += kThreads * 4) {
    if (i + 3 < end) {
      float4 v = pf_ld_stream(s.src + i);
      mn = fminf(fminf(mn, v.x), fminf(v.y, fminf(v.z, v.w)));
      mx = fmaxf(fmaxf(mx, v.x), fmaxf(v.y, fmaxf(v.z, v.w)));
    } else {
      for (int64_t j = i; j < end; ++j) {
        float v = __ldg(s.src + j);
        mn = fminf(mn, v);
        mx = fmaxf(mx, v);
      }
    }
  }
  block_minmax_to_slot(mn, mx, mn_enc + s.bucket0, mx_enc + s.bucket0);
}

// ------------------------------------------------------------------ weight quantize / STE backward
enum { kModeQuant = 0, kModeSteBwd = 1 };

// per bucket: alpha = (max-min)+1e-10, beta = min, ralpha = RN(1/alpha)  ->  scales[3][n_buckets]
__global__ void __launch_bounds__(kThreads)
uq_scales_kernel(const uint32_t* __restrict__ mn_enc, const uint32_t* __restrict__ mx_enc, int n,
                 float* __restrict__ scales) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const float mn = pf_dec(mn_enc[i]), mx = pf_dec(mx_enc[i]);
  const float alpha = __fadd_rn(__fsub_rn(mx, mn), 1e-10f);
  scales[i] = alpha;
  scales[n + i] = mn;
  scales[2 * n + i] = __frcp_rn(alpha);
}

template <int MODE>
__device__ __forceinline__ float apply_one(float x, float alpha, float beta, float ralpha, float k, float rk) {
  if (MODE == kModeQuant) return pf_fake_quant(x, alpha, beta, k, ralpha, rk);
  // STE: Mul(alpha) -> RealDiv(k) -> Mul(k) -> RealDiv(alpha) gradients, in that order
  return pf_div_r(__fmul_rn(pf_div_r(__fmul_rn(x, alpha), k, rk), k), alpha, ralpha);
}

template <int MODE>
__global__ void __launch_bounds__(kThreads)
uq_weight_apply_kernel(const pf_uq_seg* __restrict__ segs, const pf_work* __restrict__ work,
                       const float* __restrict__ scales, int n_buckets) {
  const pf_work w = work[blockIdx.x];
  const pf_uq_seg s = segs[w.seg];
  const float k = pf_uq_kf(s.bits);
  const float rk = __frcp_rn(k);
  const int64_t end = w.start + w.count;
  const uint32_t ncols = (uint32_t)s.ncols;
  const float* __restrict__ pa = scales + s.bucket0;
  const float* __restrict__ pb = scales + n_buckets + s.bucket0;
  const float* __restrict__ pr = scales + 2 * n_buckets + s.bucket0;
  int64_t i = w.start + (int64_t)threadIdx.x * 4;
  if (ncols == 1) {
    const float al = __ldg(pa), be = __ldg(pb), ra = __ldg(pr);
    for (; i < end; i += kThreads * 4) {
      if (i + 3 < end) {
        float4 v = pf_ld4(s.src + i);
        v.x = apply_one<MODE>(v.x, al, be, ra, k, rk);
        v.y = apply_one<MODE>(v.y, al, be, ra, k, rk);
        v.z = apply_one<MODE>(v.z, al, be, ra, k, rk);
        v.w = apply_one<MODE>(v.w, al, be, ra, k, rk);
        pf_st_stream(s.dst + i, v);
      } else {
        for (int64_t j = i; j < end; ++j) s.dst[j] = apply_one<MODE>(s.src[j], al, be, ra, k, rk);
      }
    }
    return;
  }
  // bucketed: bucket of flat element i is i % ncols; keep the column incrementally
  uint32_t c = (uint32_t)((uint64_t)i % ncols);
  const uint32_t step = (uint32_t)(kThreads * 4) % ncols;
  const bool aligned = (ncols & 3u) == 0;
  for (; i < end; i += kThreads * 4) {
    if (aligned && i + 3 < end) {
      float4 v = pf_ld4(s.src + i);
      const float4 a = __ldg(reinterpret_cast<const float4*>(pa + c));
      const float4 b = __ldg(reinterpret_cast<const float4*>(pb + c));
      const float4 r = __ldg(reinterpret_cast<const float4*>(pr + c));
      v.x = apply_one<MODE>(v.x, a.x, b.x, r.x, k, rk);
      v.y = apply_one<MODE>(v.y, a.y, b.y, r.y, k, rk);
      v.z = apply_one<MODE>(v.z, a.z, b.z, r.z, k, rk);
      v.w = apply_one<MODE>(v.w, a.w, b.w, r.w, k, rk);
      pf_st_stream(s.dst + i, v);
    } else {
      for (int j = 0; j < 4 && i + j < end; ++j) {
        const uint32_t cj = (c + j) % ncols;
        s.dst[i + j] = apply_one<MODE>(s.src[i + j], __ldg(pa + cj), __ldg(pb + cj), __ldg(pr + cj), k, rk);
      }
    }
    c += step;
    if (c >= ncols) c -= ncols;
  }
}

// ------------------------------------------------------------------ activations (per-tensor range)
constexpr int kActUnroll = 4;

__global__ void __launch_bounds__(kThreads)
uq_act_minmax_kernel(const float* __restrict__ x, int64_t n, uint32_t* __restrict__ minmax_enc) {
  float mn = INFINITY, mx = -INFINITY;
  const int64_t nvec = n >> 2;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  for (; i + (kActUnroll - 1) * stride < nvec; i += kActUnroll * stride) {
    float4 v[kActUnroll];
#pragma unroll
    for (int u = 0; u < kActUnroll; ++u) v[u] = pf_ld_stream(x + ((i + u * stride) << 2));
#pragma unroll
    for (int u = 0; u < kActUnroll; ++u) {
      mn = fminf(fminf(mn, v[u].x), fminf(v[u].y, fminf(v[u].z, v[u].w)));
      mx = fmaxf(fmaxf(mx, v[u].x), fmaxf(v[u].y, fmaxf(v[u].z, v[u].w)));
    }
  }
  for (; i < nvec; i += stride) {
    float4 v = pf_ld_stream(x + (i << 2));
    mn = fminf(fminf(mn, v.x), fminf(v.y, fminf(v.z, v.w)));
    mx = fmaxf(fmaxf(mx, v.x), fmaxf(v.y, fmaxf(v.z, v.w)));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    float v = __ldg(x + (nvec << 2) + threadIdx.x);
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
  block_minmax_to_slot(mn, mx, minmax_enc, minmax_enc + 1);
}

// CLAMP (pf_uq_act_quant_static): minmax_enc holds a calibrated range and x is clamped to it before the quantizer.
template <bool CLAMP = false>
__global__ void __launch_bounds__(kThreads)
uq_act_quant_kernel(const float* x, float* y, int64_t n, const uint32_t* __restrict__ minmax_enc,
                    int bits, void* __restrict__ y_hi, void* __restrict__ y_lo) {
  const float mn = pf_dec(__ldg(minmax_enc)), mx = pf_dec(__ldg(minmax_enc + 1));
  auto in = [&](float v) { return CLAMP ? pf_clamp(v, mn, mx) : v; };
  const float alpha = __fadd_rn(__fsub_rn(mx, mn), 1e-10f);
  const float k = pf_uq_kf(bits);
  const float ra = __frcp_rn(alpha), rk = __frcp_rn(k);
  const int64_t nvec = n >> 2;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  for (; i + (kActUnroll - 1) * stride < nvec; i += kActUnroll * stride) {
    float4 v[kActUnroll];
#pragma unroll
    for (int u = 0; u < kActUnroll; ++u) v[u] = pf_ld4(x + ((i + u * stride) << 2));
#pragma unroll
    for (int u = 0; u < kActUnroll; ++u) {
      v[u].x = pf_fake_quant(in(v[u].x), alpha, mn, k, ra, rk);
      v[u].y = pf_fake_quant(in(v[u].y), alpha, mn, k, ra, rk);
      v[u].z = pf_fake_quant(in(v[u].z), alpha, mn, k, ra, rk);
      v[u].w = pf_fake_quant(in(v[u].w), alpha, mn, k, ra, rk);
      if (y) pf_st_stream(y + ((i + u * stride) << 2), v[u]);
      if (y_hi) pf_st_planes4(y_hi, y_lo, (i + u * stride) << 2, v[u]);
    }
  }
  for (; i < nvec; i += stride) {
    float4 v = pf_ld4(x + (i << 2));
    v.x = pf_fake_quant(in(v.x), alpha, mn, k, ra, rk);
    v.y = pf_fake_quant(in(v.y), alpha, mn, k, ra, rk);
    v.z = pf_fake_quant(in(v.z), alpha, mn, k, ra, rk);
    v.w = pf_fake_quant(in(v.w), alpha, mn, k, ra, rk);
    if (y) pf_st_stream(y + (i << 2), v);
    if (y_hi) pf_st_planes4(y_hi, y_lo, i << 2, v);
  }
  if (y && blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t j = (nvec << 2) + threadIdx.x;
    y[j] = pf_fake_quant(in(x[j]), alpha, mn, k, ra, rk);
  }
}

inline unsigned act_grid(int64_t n) {
  // persistent-style: a multiple of the SM count, 8 resident CTAs of 256 threads per SM at most
  int64_t want = ((n >> 2) + kThreads * kActUnroll - 1) / (kThreads * kActUnroll);
  int64_t cap = (int64_t)PF_NUM_SMS * 8;
  if (want < 1) want = 1;
  return (unsigned)(want < cap ? want : cap);
}

}  // namespace

extern "C" {

int pf_uq_weight_minmax(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work,
                        uint32_t* mn_enc_dev, uint32_t* mx_enc_dev, void* stream) {
  PF_REQUIRE(n_work >= 0, "pf_uq_weight_minmax: n_work < 0");
  if (n_work == 0) return PF_OK;
  PF_REQUIRE(segs_dev && work_dev && mn_enc_dev && mx_enc_dev, "pf_uq_weight_minmax: null pointer");
  uq_weight_minmax_kernel<<<n_work, kThreads, 0, (cudaStream_t)stream>>>(segs_dev, work_dev,
                                                                        mn_enc_dev, mx_enc_dev);
  PF_CHECK_LAUNCH("pf_uq_weight_minmax");
  return PF_OK;
}

int pf_uq_weight_scales(const uint32_t* mn_enc_dev, const uint32_t* mx_enc_dev, int n_buckets,
                        float* scales_dev, void* stream) {
  PF_REQUIRE(n_buckets >= 0, "pf_uq_weight_scales: n_buckets < 0");
  if (n_buckets == 0) return PF_OK;
  PF_REQUIRE(mn_enc_dev && mx_enc_dev && scales_dev, "pf_uq_weight_scales: null pointer");
  PF_REQUIRE((n_buckets & 3) == 0 && ((uintptr_t)scales_dev & 15) == 0,
             "pf_uq_weight_scales: n_buckets must be a multiple of 4 and scales 16-byte aligned");
  uq_scales_kernel<<<(n_buckets + kThreads - 1) / kThreads, kThreads, 0, (cudaStream_t)stream>>>(
      mn_enc_dev, mx_enc_dev, n_buckets, scales_dev);
  PF_CHECK_LAUNCH("pf_uq_weight_scales");
  return PF_OK;
}

int pf_uq_weight_quant(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work,
                       const float* scales_dev, int n_buckets, void* stream) {
  PF_REQUIRE(n_work >= 0, "pf_uq_weight_quant: n_work < 0");
  if (n_work == 0) return PF_OK;
  PF_REQUIRE(segs_dev && work_dev && scales_dev, "pf_uq_weight_quant: null pointer");
  uq_weight_apply_kernel<kModeQuant><<<n_work, kThreads, 0, (cudaStream_t)stream>>>(
      segs_dev, work_dev, scales_dev, n_buckets);
  PF_CHECK_LAUNCH("pf_uq_weight_quant");
  return PF_OK;
}

int pf_uq_weight_ste_bwd(const pf_uq_seg* segs_dev, const pf_work* work_dev, int n_work,
                         const float* scales_dev, int n_buckets, void* stream) {
  PF_REQUIRE(n_work >= 0, "pf_uq_weight_ste_bwd: n_work < 0");
  if (n_work == 0) return PF_OK;
  PF_REQUIRE(segs_dev && work_dev && scales_dev, "pf_uq_weight_ste_bwd: null pointer");
  uq_weight_apply_kernel<kModeSteBwd><<<n_work, kThreads, 0, (cudaStream_t)stream>>>(
      segs_dev, work_dev, scales_dev, n_buckets);
  PF_CHECK_LAUNCH("pf_uq_weight_ste_bwd");
  return PF_OK;
}

int pf_uq_act_minmax(const float* x_dev, int64_t n, uint32_t* minmax_enc_dev, void* stream) {
  PF_REQUIRE(n >= 0, "pf_uq_act_minmax: n < 0");
  if (n == 0) return PF_OK;
  PF_REQUIRE(x_dev && minmax_enc_dev, "pf_uq_act_minmax: null pointer");
  PF_REQUIRE(((uintptr_t)x_dev & 15) == 0, "pf_uq_act_minmax: x must be 16-byte aligned");
  uq_act_minmax_kernel<<<act_grid(n), kThreads, 0, (cudaStream_t)stream>>>(x_dev, n, minmax_enc_dev);
  PF_CHECK_LAUNCH("pf_uq_act_minmax");
  return PF_OK;
}

int pf_uq_act_quant_planes(const float* x_dev, float* y_dev, void* y_hi_dev, void* y_lo_dev, int64_t n,
                           const uint32_t* minmax_enc_dev, int bits, void* stream) {
  PF_REQUIRE(n >= 0, "pf_uq_act_quant: n < 0");
  PF_REQUIRE(bits >= 1 && bits <= 32, "pf_uq_act_quant: bits must be in [1, 32]");
  if (n == 0) return PF_OK;
  PF_REQUIRE(x_dev && (y_dev || y_hi_dev) && minmax_enc_dev, "pf_uq_act_quant: null pointer");
  PF_REQUIRE((y_hi_dev == nullptr) == (y_lo_dev == nullptr), "pf_uq_act_quant: planes come in pairs");
  PF_REQUIRE(y_hi_dev == nullptr || (n & 3) == 0, "pf_uq_act_quant: plane output needs n %% 4 == 0");
  PF_REQUIRE((((uintptr_t)x_dev | (uintptr_t)y_dev) & 15) == 0 && (((uintptr_t)y_hi_dev | (uintptr_t)y_lo_dev) & 7) == 0,
             "pf_uq_act_quant: x and y must be 16-byte aligned (planes: 8)");
  uq_act_quant_kernel<><<<act_grid(n), kThreads, 0, (cudaStream_t)stream>>>(x_dev, y_dev, n, minmax_enc_dev, bits,
                                                                         y_hi_dev, y_lo_dev);
  PF_CHECK_LAUNCH("pf_uq_act_quant");
  return PF_OK;
}

int pf_uq_act_quant_static(const float* x_dev, float* y_dev, int64_t n, const uint32_t* range_enc_dev, int bits,
                           void* stream) {
  PF_REQUIRE(n >= 0, "pf_uq_act_quant_static: n < 0");
  PF_REQUIRE(bits >= 1 && bits <= 32, "pf_uq_act_quant_static: bits must be in [1, 32]");
  if (n == 0) return PF_OK;
  PF_REQUIRE(x_dev && y_dev && range_enc_dev, "pf_uq_act_quant_static: null pointer");
  PF_REQUIRE((((uintptr_t)x_dev | (uintptr_t)y_dev) & 15) == 0, "pf_uq_act_quant_static: x and y must be 16-byte aligned");
  uq_act_quant_kernel<true><<<act_grid(n), kThreads, 0, (cudaStream_t)stream>>>(x_dev, y_dev, n, range_enc_dev, bits,
                                                                               nullptr, nullptr);
  PF_CHECK_LAUNCH("pf_uq_act_quant_static");
  return PF_OK;
}

int pf_uq_act_quant(const float* x_dev, float* y_dev, int64_t n, const uint32_t* minmax_enc_dev,
                    int bits, void* stream) {
  PF_REQUIRE(n >= 0, "pf_uq_act_quant: n < 0");
  PF_REQUIRE(n == 0 || y_dev != nullptr, "pf_uq_act_quant: null pointer");
  return pf_uq_act_quant_planes(x_dev, y_dev, nullptr, nullptr, n, minmax_enc_dev, bits, stream);
}

}  // extern "C"
