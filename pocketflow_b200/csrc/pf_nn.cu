// pf_nn.cu — the HBM-bound layers around the convolutions (SURVEY.md §8 a13): batch-norm
// (training statistics, apply(+ReLU/ReLU6)(+activation range), backward), max/mean pooling,
// residual add, ReLU backward, bias gradient.  NHWC fp32; every tensor is viewed as [M, C].
//
// Reference semantics: tf.layers.batch_normalization(momentum .997, eps 1e-5, fused)
// (/root/reference/utils/external/resnet_model.py:55-62), tf.nn.relu (:144), max_pooling2d 3x3 s2
// SAME (:521-525), reduce_mean over H,W (:547-548), residual add (:199,:314).
// Design: one pass computes the batch statistics (shifted sums, fp64 combine), one pass applies
// BN+ReLU AND accumulates the per-tensor min/max the activation quantizer needs
// (uniform_quantization/utils.py:51-79), so the separate reduce_max/reduce_min passes of the
// reference disappear.
#include <cstdlib>
#include <numeric>

#include "pf_common.cuh"

namespace {

constexpr int NT = 256;
constexpr int kColTile = 256;  // columns per CTA (64 float4 lanes)

// ------------------------------------------------------------------ column-reduction scaffolding
struct ColTile {
  int c0, tc, nvec, nty, tx, ty;
  __device__ ColTile(int C) {
    c0 = blockIdx.x * kColTile;
    tc = min(kColTile, C - c0);
    nvec = tc >> 2;
    nty = NT / nvec;
    tx = threadIdx.x % nvec;
    ty = threadIdx.x / nvec;
  }
};

// BN statistics partials: per (split, channel): K (shift), s1 = sum(x-K), s2 = sum((x-K)^2)
// RANGE: also min(x), max(x) per channel.  y = act(bn(x)) is a composition of correctly-rounded monotone steps, so
// the per-tensor range of y needed by the activation quantizer (utils.py:51-79) is attained at the per-channel
// extremes of x: the final kernel evaluates it from these, and no pass over y is needed.
template <bool RANGE>
__global__ void __launch_bounds__(NT)
bn_stats_partial_kernel(const float* __restrict__ x, int M, int C, int rows_per_split,
                        float* __restrict__ part /* [splits][3 or 5][C] */) {
  __shared__ float sh[RANGE ? 4 : 2][NT * 4];
  constexpr int NF = RANGE ? 5 : 3;
  const ColTile t(C);
  const int r0 = blockIdx.y * rows_per_split;
  const int r1 = min(M, r0 + rows_per_split);
  const int col = t.c0 + t.tx * 4;
  float4 K = make_float4(0.f, 0.f, 0.f, 0.f), s1 = K, s2 = K;
  float4 mn = make_float4(INFINITY, INFINITY, INFINITY, INFINITY), mx = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  if (t.ty < t.nty) {
    K = __ldg(reinterpret_cast<const float4*>(x + (size_t)r0 * C + col));
    auto acc = [&](const float4 v) {
      if (RANGE) {
        mn.x = fminf(mn.x, v.x); mn.y = fminf(mn.y, v.y); mn.z = fminf(mn.z, v.z); mn.w = fminf(mn.w, v.w);
        mx.x = fmaxf(mx.x, v.x); mx.y = fmaxf(mx.y, v.y); mx.z = fmaxf(mx.z, v.z); mx.w = fmaxf(mx.w, v.w);
      }
      const float dx = v.x - K.x, dy = v.y - K.y, dz = v.z - K.z, dw = v.w - K.w;
      s1.x += dx; s1.y += dy; s1.z += dz; s1.w += dw;
      s2.x = fmaf(dx, dx, s2.x); s2.y = fmaf(dy, dy, s2.y); s2.z = fmaf(dz, dz, s2.z); s2.w = fmaf(dw, dw, s2.w);
    };
    int r = r0 + t.ty;
    for (; r + 3 * t.nty < r1; r += 4 * t.nty) {   // 4 independent 128-bit loads in flight per thread
      const float4 v0 = pf_ld_stream(x + (size_t)r * C + col);
      const float4 v1 = pf_ld_stream(x + (size_t)(r + t.nty) * C + col);
      const float4 v2 = pf_ld_stream(x + (size_t)(r + 2 * t.nty) * C + col);
      const float4 v3 = pf_ld_stream(x + (size_t)(r + 3 * t.nty) * C + col);
      acc(v0); acc(v1); acc(v2); acc(v3);
    }
    for (; r < r1; r += t.nty) acc(pf_ld_stream(x + (size_t)r * C + col));
    float* a = &sh[0][(t.ty * t.nvec + t.tx) * 4];
    float* b = &sh[1][(t.ty * t.nvec + t.tx) * 4];
    a[0] = s1.x; a[1] = s1.y; a[2] = s1.z; a[3] = s1.w;
    b[0] = s2.x; b[1] = s2.y; b[2] = s2.z; b[3] = s2.w;
    if (RANGE) {
      float* lo = &sh[RANGE ? 2 : 0][(t.ty * t.nvec + t.tx) * 4];
      float* hi = &sh[RANGE ? 3 : 0][(t.ty * t.nvec + t.tx) * 4];
      lo[0] = mn.x; lo[1] = mn.y; lo[2] = mn.z; lo[3] = mn.w;
      hi[0] = mx.x; hi[1] = mx.y; hi[2] = mx.z; hi[3] = mx.w;
    }
  }
  __syncthreads();
  // fixed-order combine over ty: deterministic
  for (int c = threadIdx.x; c < t.tc; c += NT) {
    float a = 0.f, b = 0.f, lo = INFINITY, hi = -INFINITY;
    for (int y = 0; y < t.nty; ++y) {
      a += sh[0][(y * t.nvec + (c >> 2)) * 4 + (c & 3)];
      b += sh[1][(y * t.nvec + (c >> 2)) * 4 + (c & 3)];
      if (RANGE) {
        lo = fminf(lo, sh[RANGE ? 2 : 0][(y * t.nvec + (c >> 2)) * 4 + (c & 3)]);
        hi = fmaxf(hi, sh[RANGE ? 3 : 0][(y * t.nvec + (c >> 2)) * 4 + (c & 3)]);
      }
    }
    float* p = part + (size_t)blockIdx.y * NF * C;
    p[t.c0 + c] = __ldg(x + (size_t)r0 * C + t.c0 + c);
    p[C + t.c0 + c] = a;
    p[2 * C + t.c0 + c] = b;
    if (RANGE) {
      p[3 * C + t.c0 + c] = lo;
      p[4 * C + t.c0 + c] = hi;
    }
  }
}

// Combine the partials in fp64; emit mean, biased var, rstd; update moving stats.  Every split's shifted sums are
// re-based to ONE common shift K0 (the first split's), after which they simply add:
//     d = K - K0;  S1' = s1 + n d;  S2' = s2 + 2 d s1 + n d^2        (exact algebra, fp64)
// and mean = K0 + S1/N, m2 = S2 - S1^2/N.  No divisions inside the loop (the first version merged Chan-style
// moments pairwise: four fp64 divisions per split on a GPU with 1/64-rate fp64 — 36 us per launch).
// kFinalWarps warps per channel stride over the splits; fixed-order shuffle + smem tree: deterministic.
constexpr int kFinalWarps = 4;
__global__ void __launch_bounds__(NT)
bn_stats_final_kernel(const float* __restrict__ part, int M, int C, int splits, int rows_per_split,
                      float eps, float momentum, float* __restrict__ mean, float* __restrict__ var,
                      float* __restrict__ rstd, float* __restrict__ mov_mean, float* __restrict__ mov_var,
                      int nf, const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                      uint32_t* __restrict__ minmax_enc) {
  constexpr int CPB = NT / 32 / kFinalWarps;      // channels per block
  __shared__ double sh1[NT / 32], sh2[NT / 32];
  __shared__ float shlo[NT / 32], shhi[NT / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cl = warp / kFinalWarps, sub = warp % kFinalWarps;
  const int c = blockIdx.x * CPB + cl;
  double S1 = 0.0, S2 = 0.0;
  float xlo = INFINITY, xhi = -INFINITY;
  const double K0 = c < C ? (double)part[c] : 0.0;
  if (c < C) {
    for (int s = sub * 32 + lane; s < splits; s += 32 * kFinalWarps) {
      const int r0 = s * rows_per_split;
      const double n = (double)(min(M, r0 + rows_per_split) - r0);
      const float* p = part + (size_t)s * nf * C;
      const double d = (double)p[c] - K0, s1 = p[C + c], s2 = p[2 * C + c];
      S1 += s1 + n * d;
      S2 += s2 + 2.0 * d * s1 + n * d * d;
      if (nf == 5) {
        xlo = fminf(xlo, p[3 * C + c]);
        xhi = fmaxf(xhi, p[4 * C + c]);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    S1 += __shfl_down_sync(0xffffffffu, S1, o);
    S2 += __shfl_down_sync(0xffffffffu, S2, o);
  }
  xlo = pf_warp_min(xlo);
  xhi = pf_warp_max(xhi);
  if (lane == 0) { sh1[warp] = S1; sh2[warp] = S2; shlo[warp] = xlo; shhi[warp] = xhi; }
  __syncthreads();
  if (c >= C || sub != 0 || lane != 0) return;
  for (int w = 1; w < kFinalWarps; ++w) {
    S1 += sh1[warp + w];
    S2 += sh2[warp + w];
    xlo = fminf(xlo, shlo[warp + w]);
    xhi = fmaxf(xhi, shhi[warp + w]);
  }
  struct { double n, mean, m2; } acc;
  acc.n = (double)M;
  acc.mean = K0 + S1 / acc.n;
  acc.m2 = fmax(S2 - S1 * S1 / acc.n, 0.0);
  const float mu = (float)acc.mean;
  const float v = (float)(acc.m2 / acc.n);
  mean[c] = mu;
  var[c] = v;
  const float rs_ = __frsqrt_rn(__fadd_rn(v, eps));
  rstd[c] = rs_;
  if (nf == 5 && minmax_enc && xlo <= xhi) {
    // range of y = act(bn(x)) over this channel: attained at the extremes of x (monotone in x)
    const float ya = pf_bn_act(xlo, mu, rs_, gamma[c], beta[c], act), yb = pf_bn_act(xhi, mu, rs_, gamma[c], beta[c], act);
    atomicMin(minmax_enc, pf_enc(fminf(ya, yb)));
    atomicMax(minmax_enc + 1, pf_enc(fmaxf(ya, yb)));
  }
  if (mov_mean) {
    // moving = moving*momentum + batch*(1-momentum); the moving variance uses the unbiased estimate
    const float om = __fsub_rn(1.f, momentum);
    const float vu = acc.n > 1.0 ? (float)(acc.m2 / (acc.n - 1.0)) : v;
    mov_mean[c] = __fadd_rn(__fmul_rn(mov_mean[c], momentum), __fmul_rn(mu, om));
    mov_var[c] = __fadd_rn(__fmul_rn(mov_var[c], momentum), __fmul_rn(vu, om));
  }
}

__global__ void __launch_bounds__(NT)
bn_eval_prepare_kernel(const float* __restrict__ mov_var, int C, float eps, float* __restrict__ rstd) {
  const int c = blockIdx.x * NT + threadIdx.x;
  if (c < C) rstd[c] = __frsqrt_rn(__fadd_rn(mov_var[c], eps));
}

// y = act(bn(x)); optionally accumulates the per-tensor min/max of y (ordered-uint slots)
// RES: y = bn(x) + res — a linear-bottleneck BN (no activation) feeding a residual Add (MobileNet-v2,
// conv_blocks.py:289-313) in one pass; the add is one more correctly rounded step after the BN chain, so the result is
// bit-identical to BN apply followed by pf_add.  8 B/element read (x, res) instead of 4 + 8 + 8 for the three passes.
// CLAMP (static range, pf_bn_apply_eval_quant_static): act(bn(x)) is clamped to [min, max] of q_range before the
// fake-quant, so values outside a calibrated range take its end levels; inside it the result is the unclamped one.
template <bool RES, bool CLAMP = false>
__global__ void __launch_bounds__(NT)
bn_apply_kernel(const float* __restrict__ x, int64_t total, int C, const float* __restrict__ mean,
                const float* __restrict__ rstd, const float* __restrict__ gamma,
                const float* __restrict__ beta, int act, float* __restrict__ y,
                uint32_t* __restrict__ minmax_enc, void* __restrict__ y_hi, void* __restrict__ y_lo,
                const uint32_t* __restrict__ q_range, int q_bits, float var_eps, const float* __restrict__ res) {
  // var_eps >= 0: `rstd` holds the (moving) VARIANCE and rstd = rsqrt(var + eps) is formed here (inference mode;
  // same two roundings as bn_eval_prepare_kernel, one launch less per layer)
  __shared__ float s_mn[NT / 32], s_mx[NT / 32];
  // fused activation fake-quant (range known beforehand: pf_bn_train_stats_range)
  float q_alpha = 1.f, q_beta = 0.f, q_k = 1.f, q_ra = 1.f, q_rk = 1.f, q_hi = 0.f;
  if (q_range) {
    const float qmn = pf_dec(__ldg(q_range)), qmx = pf_dec(__ldg(q_range + 1));
    q_hi = qmx;
    q_alpha = __fadd_rn(__fsub_rn(qmx, qmn), 1e-10f);
    q_beta = qmn;
    q_k = pf_uq_kf(q_bits);
    q_ra = __frcp_rn(q_alpha);
    q_rk = __frcp_rn(q_k);
  }
  const int64_t nvec = total >> 2;
  const int64_t stride = (int64_t)gridDim.x * NT;
  int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x;
  uint32_t c = (uint32_t)((i << 2) % (uint32_t)C);
  const uint32_t step = (uint32_t)((stride << 2) % (uint32_t)C);
  float mn = INFINITY, mx = -INFINITY;
  auto apply4 = [&](float4 v, const float4& mu, const float4& rs, const float4& ga, const float4& be, int64_t idx) {
    v.x = pf_bn_act(v.x, mu.x, rs.x, ga.x, be.x, act);
    v.y = pf_bn_act(v.y, mu.y, rs.y, ga.y, be.y, act);
    v.z = pf_bn_act(v.z, mu.z, rs.z, ga.z, be.z, act);
    v.w = pf_bn_act(v.w, mu.w, rs.w, ga.w, be.w, act);
    if (RES) {
      const float4 r = pf_ld_stream(res + (idx << 2));
      v.x = __fadd_rn(v.x, r.x); v.y = __fadd_rn(v.y, r.y); v.z = __fadd_rn(v.z, r.z); v.w = __fadd_rn(v.w, r.w);
    }
    if (q_range) {
      if (CLAMP) {
        v.x = pf_clamp(v.x, q_beta, q_hi); v.y = pf_clamp(v.y, q_beta, q_hi);
        v.z = pf_clamp(v.z, q_beta, q_hi); v.w = pf_clamp(v.w, q_beta, q_hi);
      }
      v.x = pf_fake_quant(v.x, q_alpha, q_beta, q_k, q_ra, q_rk);
      v.y = pf_fake_quant(v.y, q_alpha, q_beta, q_k, q_ra, q_rk);
      v.z = pf_fake_quant(v.z, q_alpha, q_beta, q_k, q_ra, q_rk);
      v.w = pf_fake_quant(v.w, q_alpha, q_beta, q_k, q_ra, q_rk);
    }
    if (y) pf_st_stream(y + (idx << 2), v);
    if (y_hi) pf_st_planes4(y_hi, y_lo, idx << 2, v);
    mn = fminf(fminf(mn, v.x), fminf(v.y, fminf(v.z, v.w)));
    mx = fmaxf(fmaxf(mx, v.x), fmaxf(v.y, fmaxf(v.z, v.w)));
  };
  if (step == 0) {
    // the grid stride is a multiple of C: this thread's 4 channels never change -> parameters live in
    // registers and the loop is a pure 8 B/element stream with 4 independent loads in flight
    const float4 mu = __ldg(reinterpret_cast<const float4*>(mean + c));
    float4 rs = __ldg(reinterpret_cast<const float4*>(rstd + c));
    if (var_eps >= 0.f) {
      rs.x = __frsqrt_rn(__fadd_rn(rs.x, var_eps)); rs.y = __frsqrt_rn(__fadd_rn(rs.y, var_eps));
      rs.z = __frsqrt_rn(__fadd_rn(rs.z, var_eps)); rs.w = __frsqrt_rn(__fadd_rn(rs.w, var_eps));
    }
    const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c));
    const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c));
    for (; i + 3 * stride < nvec; i += 4 * stride) {
      const float4 v0 = pf_ld_stream(x + (i << 2));
      const float4 v1 = pf_ld_stream(x + ((i + stride) << 2));
      const float4 v2 = pf_ld_stream(x + ((i + 2 * stride) << 2));
      const float4 v3 = pf_ld_stream(x + ((i + 3 * stride) << 2));
      apply4(v0, mu, rs, ga, be, i);
      apply4(v1, mu, rs, ga, be, i + stride);
      apply4(v2, mu, rs, ga, be, i + 2 * stride);
      apply4(v3, mu, rs, ga, be, i + 3 * stride);
    }
    for (; i < nvec; i += stride) apply4(pf_ld_stream(x + (i << 2)), mu, rs, ga, be, i);
  } else {
    for (; i < nvec; i += stride) {
      const float4 mu = __ldg(reinterpret_cast<const float4*>(mean + c));
      float4 rs = __ldg(reinterpret_cast<const float4*>(rstd + c));
      if (var_eps >= 0.f) {
        rs.x = __frsqrt_rn(__fadd_rn(rs.x, var_eps)); rs.y = __frsqrt_rn(__fadd_rn(rs.y, var_eps));
        rs.z = __frsqrt_rn(__fadd_rn(rs.z, var_eps)); rs.w = __frsqrt_rn(__fadd_rn(rs.w, var_eps));
      }
      const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c));
      const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c));
      apply4(pf_ld_stream(x + (i << 2)), mu, rs, ga, be, i);
      c += step;
      if (c >= (uint32_t)C) c -= (uint32_t)C;
    }
  }
  if (minmax_enc) {
    mn = pf_warp_min(mn);
    mx = pf_warp_max(mx);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) { s_mn[wid] = mn; s_mx[wid] = mx; }
    __syncthreads();
    if (wid == 0) {
      mn = lane < NT / 32 ? s_mn[lane] : INFINITY;
      mx = lane < NT / 32 ? s_mx[lane] : -INFINITY;
      mn = pf_warp_min(mn);
      mx = pf_warp_max(mx);
      if (lane == 0 && mn <= mx) {
        atomicMin(minmax_enc, pf_enc(mn));
        atomicMax(minmax_enc + 1, pf_enc(mx));
      }
    }
  }
}

// BN + activation + fake-quant (known range) writing the tensor-core operand as INTEGER LEVELS where it can:
// y = act(bn(x)), qa = Q(y).  When the tensor's minimum is exactly 0 (every ReLU / ReLU6 output in practice) and
// bits <= 8, qa = scale * level with level in [0, 2^bits - 1] exactly representable in bf16: plane0 <- bf16(level),
// plane1 is not written, hdr <- {scale = alpha / k, 1} and a consuming MMA needs ONE operand plane instead of two.
// Otherwise plane0 / plane1 <- hi / lo of qa and hdr <- {1, 2}.  Either way csum[pixel][segment] receives the sum of
// the stored plane values over channel segments of min(C, 128) — the rank-1 term the weight quantizer's offset needs
// (pf_conv_tma.cu).  One warp owns whole segments (C a power of two >= 16), reduced by a fixed xor butterfly: the sums
// are deterministic, and exact for levels.  HBM traffic: 4 B read + 2 B (levels) or 4 B (planes) written per element.
// LEVELS_ONLY: no fp32 output wanted and the operand CAN travel as levels (host: bits <= 8) — the dequantized value is
// then never formed (the level alone is 13 fp32 ops per element against 21; the general form ran at 3.4 TB/s on the
// 822 MB tensors of stage 1, issue-bound).  A range that does not start at 0 (device-side condition) falls back to the
// general path inside the same kernel.
template <bool LEVELS_ONLY>
__global__ void __launch_bounds__(NT)
bn_apply_levels_kernel(const float* __restrict__ x, int64_t total, int C, int cshift, const float* __restrict__ mean,
                       const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                       int act, float* __restrict__ y, void* __restrict__ p0, void* __restrict__ p1,
                       const uint32_t* __restrict__ q_range, int q_bits, pf_tc_act_hdr* __restrict__ hdr,
                       float* __restrict__ csum, int nseg) {
  const float qmn = pf_dec(__ldg(q_range)), qmx = pf_dec(__ldg(q_range + 1));
  const float q_alpha = __fadd_rn(__fsub_rn(qmx, qmn), 1e-10f), q_beta = qmn;
  const float q_k = pf_uq_kf(q_bits), q_ra = __frcp_rn(q_alpha), q_rk = __frcp_rn(q_k);
  const bool lev = q_bits <= 8 && q_beta == 0.f;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    hdr->scale = lev ? __fdiv_rn(q_alpha, q_k) : 1.f;
    hdr->nplanes = lev ? 1 : 2;
  }
  const int lane = threadIdx.x & 31;
  const int L = min(C >> 2, 32);                       // lanes per channel segment
  const int64_t nvec = total >> 2;
  const int64_t stride = (int64_t)gridDim.x * NT;      // a multiple of C / 4 (host): this thread's channels never change
  const int64_t first = (int64_t)blockIdx.x * NT + threadIdx.x;
  const uint32_t c = (uint32_t)((first << 2) & (int64_t)(C - 1));
  const float4 mu = __ldg(reinterpret_cast<const float4*>(mean + c));
  const float4 rs = __ldg(reinterpret_cast<const float4*>(rstd + c));
  const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c));
  const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c));
  auto emit = [&](float4 v, int64_t i, bool valid) {
    float4 lv;
    if (LEVELS_ONLY && lev) {
      lv.x = pf_quant_level(pf_bn_act(v.x, mu.x, rs.x, ga.x, be.x, act), q_alpha, q_beta, q_k, q_ra);
      lv.y = pf_quant_level(pf_bn_act(v.y, mu.y, rs.y, ga.y, be.y, act), q_alpha, q_beta, q_k, q_ra);
      lv.z = pf_quant_level(pf_bn_act(v.z, mu.z, rs.z, ga.z, be.z, act), q_alpha, q_beta, q_k, q_ra);
      lv.w = pf_quant_level(pf_bn_act(v.w, mu.w, rs.w, ga.w, be.w, act), q_alpha, q_beta, q_k, q_ra);
    } else {
      v.x = pf_fake_quant_lv(pf_bn_act(v.x, mu.x, rs.x, ga.x, be.x, act), q_alpha, q_beta, q_k, q_ra, q_rk, lv.x);
      v.y = pf_fake_quant_lv(pf_bn_act(v.y, mu.y, rs.y, ga.y, be.y, act), q_alpha, q_beta, q_k, q_ra, q_rk, lv.y);
      v.z = pf_fake_quant_lv(pf_bn_act(v.z, mu.z, rs.z, ga.z, be.z, act), q_alpha, q_beta, q_k, q_ra, q_rk, lv.z);
      v.w = pf_fake_quant_lv(pf_bn_act(v.w, mu.w, rs.w, ga.w, be.w, act), q_alpha, q_beta, q_k, q_ra, q_rk, lv.w);
    }
    const float4 s = lev ? lv : v;
    float part = 0.f;
    if (valid) {
      const int64_t e = i << 2;
      if (!LEVELS_ONLY && y) pf_st_stream(y + e, v);
      if (lev) {
        const __nv_bfloat162 a = __floats2bfloat162_rn(s.x, s.y), b = __floats2bfloat162_rn(s.z, s.w);
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p0) + e) =
            make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
      } else {
        pf_st_planes4(p0, p1, e, s);
      }
      part = (s.x + s.y) + (s.z + s.w);
    }
    for (int o = L >> 1; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (valid && (lane & (L - 1)) == 0) {
      const int64_t e = i << 2;
      csum[(e >> cshift) * nseg + (int)((e & (int64_t)(C - 1)) >> 7)] = part;
    }
  };
  // warp-uniform trip count (the segment reduction uses full-warp shuffles); FOUR independent loads in flight per thread
  // (with two, this kernel and its plane-writing sibling both read at ~2.5 TB/s: bound by the latency of the reads)
  const int64_t wbase = first - lane;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int64_t off = 0; wbase + off < nvec; off += 4 * stride) {
    const int64_t i0 = first + off, i1 = i0 + stride, i2 = i1 + stride, i3 = i2 + stride;
    const bool v0 = i0 < nvec, v1 = i1 < nvec, v2 = i2 < nvec, v3 = i3 < nvec;
    const float4 a = v0 ? pf_ld_stream(x + (i0 << 2)) : zero4;
    const float4 b = v1 ? pf_ld_stream(x + (i1 << 2)) : zero4;
    const float4 c4 = v2 ? pf_ld_stream(x + (i2 << 2)) : zero4;
    const float4 d = v3 ? pf_ld_stream(x + (i3 << 2)) : zero4;
    emit(a, i0, v0);
    emit(b, i1, v1);
    emit(c4, i2, v2);
    emit(d, i3, v3);
  }
}

// The u8 operand of pf_conv2d_u8_fwd (inference): y = act(bn(x)) with the moving statistics (pf_bn_apply_eval's op
// chain, rstd formed in the kernel), quantized with the per-tensor range of THIS batch, written as unsigned 8-bit levels
// rint(((y - min) / alpha) * k) — the levels act_quant rebuilds its values from — plus the per-pixel channel-segment
// level sums (csum, as bn_apply_levels_kernel writes them) and the header {alpha / k, 1}.  The range needs a grid-wide
// reduction before any level is written, so this runs twice: RANGE = min / max of y into range_enc (ordered-uint, as
// pf_bn_apply_eval accumulates it), then the levels.  A range that does not start at 0 (an activation offset the u8
// convolution has no term for) is recorded as header {1, 0}.  Channel-stationary grid (host: chan_grid), C a power of
// two >= 16.  HBM traffic: 4 B read per element and pass, 1 B written.
// CLAMP (pf_bn_eval_levels_u8_static): range_enc holds a calibrated range and only the level pass runs; y is clamped
// to it first (a value above max gets level k), so with the batch's own range the levels and sums are these.  4 B read
// and 1 B written per element, no atomics.
template <bool RANGE, bool CLAMP = false>
__global__ void __launch_bounds__(NT)
bn_eval_levels_u8_kernel(const float* __restrict__ x, int64_t total, int C, int cshift, const float* __restrict__ mean,
                         const float* __restrict__ var, float eps, const float* __restrict__ gamma,
                         const float* __restrict__ beta, int act, uint32_t* __restrict__ range_enc, int q_bits,
                         uint8_t* __restrict__ levels, pf_tc_act_hdr* __restrict__ hdr, float* __restrict__ csum,
                         int nseg) {
  const int lane = threadIdx.x & 31;
  const int64_t nvec = total >> 2;
  const int64_t stride = (int64_t)gridDim.x * NT;
  const int64_t first = (int64_t)blockIdx.x * NT + threadIdx.x;
  const uint32_t c = (uint32_t)((first << 2) & (int64_t)(C - 1));
  const float4 mu = __ldg(reinterpret_cast<const float4*>(mean + c));
  float4 rs = __ldg(reinterpret_cast<const float4*>(var + c));
  rs.x = __frsqrt_rn(__fadd_rn(rs.x, eps)); rs.y = __frsqrt_rn(__fadd_rn(rs.y, eps));
  rs.z = __frsqrt_rn(__fadd_rn(rs.z, eps)); rs.w = __frsqrt_rn(__fadd_rn(rs.w, eps));
  const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c));
  const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c));
  auto bn4 = [&](float4 v) {
    return make_float4(pf_bn_act(v.x, mu.x, rs.x, ga.x, be.x, act), pf_bn_act(v.y, mu.y, rs.y, ga.y, be.y, act),
                       pf_bn_act(v.z, mu.z, rs.z, ga.z, be.z, act), pf_bn_act(v.w, mu.w, rs.w, ga.w, be.w, act));
  };
  if (RANGE) {
    __shared__ float s_mn[NT / 32], s_mx[NT / 32];
    float mn = INFINITY, mx = -INFINITY;
    for (int64_t i = first; i < nvec; i += stride) {
      const float4 y = bn4(pf_ld_stream(x + (i << 2)));
      mn = fminf(fminf(mn, y.x), fminf(y.y, fminf(y.z, y.w)));
      mx = fmaxf(fmaxf(mx, y.x), fmaxf(y.y, fmaxf(y.z, y.w)));
    }
    mn = pf_warp_min(mn);
    mx = pf_warp_max(mx);
    if (lane == 0) {
      s_mn[threadIdx.x >> 5] = mn;
      s_mx[threadIdx.x >> 5] = mx;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      mn = lane < NT / 32 ? s_mn[lane] : INFINITY;
      mx = lane < NT / 32 ? s_mx[lane] : -INFINITY;
      mn = pf_warp_min(mn);
      mx = pf_warp_max(mx);
      if (lane == 0 && mn <= mx) {
        atomicMin(range_enc, pf_enc(mn));
        atomicMax(range_enc + 1, pf_enc(mx));
      }
    }
    return;
  }
  const float qmn = pf_dec(__ldg(range_enc)), qmx = pf_dec(__ldg(range_enc + 1));
  const float q_alpha = __fadd_rn(__fsub_rn(qmx, qmn), 1e-10f);
  const float q_k = pf_uq_kf(q_bits), q_ra = __frcp_rn(q_alpha);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    hdr->scale = qmn == 0.f ? __fdiv_rn(q_alpha, q_k) : 1.f;
    hdr->nplanes = qmn == 0.f ? 1 : 0;
  }
  const int L = min(C >> 2, 32);                       // lanes per channel segment
  const int64_t wbase = first - lane;
  for (int64_t i = first; wbase + (i - first) < nvec; i += stride) {   // warp-uniform trip count (segment shuffles)
    const bool valid = i < nvec;
    float part = 0.f;
    if (valid) {
      float4 y = bn4(pf_ld_stream(x + (i << 2)));
      if (CLAMP) {
        y.x = pf_clamp(y.x, qmn, qmx); y.y = pf_clamp(y.y, qmn, qmx);
        y.z = pf_clamp(y.z, qmn, qmx); y.w = pf_clamp(y.w, qmn, qmx);
      }
      const float lx = pf_quant_level(y.x, q_alpha, qmn, q_k, q_ra), ly = pf_quant_level(y.y, q_alpha, qmn, q_k, q_ra);
      const float lz = pf_quant_level(y.z, q_alpha, qmn, q_k, q_ra), lw = pf_quant_level(y.w, q_alpha, qmn, q_k, q_ra);
      *reinterpret_cast<uint32_t*>(levels + (i << 2)) =
          (uint32_t)lx | ((uint32_t)ly << 8) | ((uint32_t)lz << 16) | ((uint32_t)lw << 24);
      part = (lx + ly) + (lz + lw);
    }
    for (int o = L >> 1; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (valid && (lane & (L - 1)) == 0) {
      const int64_t e = i << 2;
      csum[(e >> cshift) * nseg + (int)((e & (int64_t)(C - 1)) >> 7)] = part;
    }
  }
}

// The same two passes for a C that is a multiple of 16 but not a power of two (MobileNet-v2's 96 .. 960 channels):
// an item is one pixel's channel segment (128 channels, the last one partial, as csum counts them), owned by a group
// of 8 lanes of 16 channels each (lanes past C idle); a lane reads 64 bytes, writes 16 bytes of levels (as two 8-byte stores), and the group's
// level sum is a 3-step xor butterfly (integers below 2^24: exact).  The item index is the csum index.  Segment-
// stationary grid: the number of groups is a multiple of nseg (host: seg_grid), so every lane keeps its 16 channels
// and their batch-norm constants.  The levels are pf_quant_level of the same values as in bn_eval_levels_u8_kernel
// (CLAMP as there).
template <bool RANGE, bool CLAMP = false>
__global__ void __launch_bounds__(NT)
bn_eval_levels_u8_seg_kernel(const float* __restrict__ x, int64_t items, int C, int nseg, const float* __restrict__ mean,
                             const float* __restrict__ var, float eps, const float* __restrict__ gamma,
                             const float* __restrict__ beta, int act, uint32_t* __restrict__ range_enc, int q_bits,
                             uint8_t* __restrict__ levels, pf_tc_act_hdr* __restrict__ hdr, float* __restrict__ csum) {
  const int lane = threadIdx.x & 31, sub = threadIdx.x & 7;
  const int64_t first = ((int64_t)blockIdx.x * NT + threadIdx.x) >> 3;       // this lane's group
  const int64_t stride = (int64_t)gridDim.x * (NT / 8);
  const int c0 = (int)(first % nseg) * 128 + sub * 16;
  const bool cok = c0 < C;
  float mu[16], rs[16], ga[16], be[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = cok ? c0 + j : 0;
    mu[j] = __ldg(mean + c);
    rs[j] = __frsqrt_rn(__fadd_rn(__ldg(var + c), eps));
    ga[j] = __ldg(gamma + c);
    be[j] = __ldg(beta + c);
  }
  auto load_bn = [&](int64_t item, float (&y)[16]) {
    const float* src = x + (item / nseg) * C + c0;
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const float4 a = pf_ld_stream(src + 4 * v);
      y[4 * v] = pf_bn_act(a.x, mu[4 * v], rs[4 * v], ga[4 * v], be[4 * v], act);
      y[4 * v + 1] = pf_bn_act(a.y, mu[4 * v + 1], rs[4 * v + 1], ga[4 * v + 1], be[4 * v + 1], act);
      y[4 * v + 2] = pf_bn_act(a.z, mu[4 * v + 2], rs[4 * v + 2], ga[4 * v + 2], be[4 * v + 2], act);
      y[4 * v + 3] = pf_bn_act(a.w, mu[4 * v + 3], rs[4 * v + 3], ga[4 * v + 3], be[4 * v + 3], act);
    }
  };
  if (RANGE) {
    __shared__ float s_mn[NT / 32], s_mx[NT / 32];
    float mn = INFINITY, mx = -INFINITY;
    if (cok) {
      for (int64_t i = first; i < items; i += stride) {
        float y[16];
        load_bn(i, y);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          mn = fminf(mn, y[j]);
          mx = fmaxf(mx, y[j]);
        }
      }
    }
    mn = pf_warp_min(mn);
    mx = pf_warp_max(mx);
    if (lane == 0) {
      s_mn[threadIdx.x >> 5] = mn;
      s_mx[threadIdx.x >> 5] = mx;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      mn = lane < NT / 32 ? s_mn[lane] : INFINITY;
      mx = lane < NT / 32 ? s_mx[lane] : -INFINITY;
      mn = pf_warp_min(mn);
      mx = pf_warp_max(mx);
      if (lane == 0 && mn <= mx) {
        atomicMin(range_enc, pf_enc(mn));
        atomicMax(range_enc + 1, pf_enc(mx));
      }
    }
    return;
  }
  const float qmn = pf_dec(__ldg(range_enc)), qmx = pf_dec(__ldg(range_enc + 1));
  const float q_alpha = __fadd_rn(__fsub_rn(qmx, qmn), 1e-10f);
  const float q_k = pf_uq_kf(q_bits), q_ra = __frcp_rn(q_alpha);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    hdr->scale = qmn == 0.f ? __fdiv_rn(q_alpha, q_k) : 1.f;
    hdr->nplanes = qmn == 0.f ? 1 : 0;
  }
  const int64_t wbase = first - (lane >> 3);           // the warp's first group
  for (int64_t i = first; wbase + (i - first) < items; i += stride) {   // warp-uniform trip count (group shuffles)
    float part = 0.f;
    if (i < items && cok) {
      float y[16];
      load_bn(i, y);
      if (CLAMP) {
#pragma unroll
        for (int j = 0; j < 16; ++j) y[j] = pf_clamp(y[j], qmn, qmx);
      }
      uint32_t w[4];
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const float l0 = pf_quant_level(y[4 * v], q_alpha, qmn, q_k, q_ra);
        const float l1 = pf_quant_level(y[4 * v + 1], q_alpha, qmn, q_k, q_ra);
        const float l2 = pf_quant_level(y[4 * v + 2], q_alpha, qmn, q_k, q_ra);
        const float l3 = pf_quant_level(y[4 * v + 3], q_alpha, qmn, q_k, q_ra);
        w[v] = (uint32_t)l0 | ((uint32_t)l1 << 8) | ((uint32_t)l2 << 16) | ((uint32_t)l3 << 24);
        part += (l0 + l1) + (l2 + l3);
      }
      // two 8-byte stores: the entry point promises to work with an 8-byte-aligned levels buffer
      uint2* dst = reinterpret_cast<uint2*>(levels + (i / nseg) * C + c0);
      dst[0] = make_uint2(w[0], w[1]);
      dst[1] = make_uint2(w[2], w[3]);
    }
    part += __shfl_xor_sync(0xffffffffu, part, 4);
    part += __shfl_xor_sync(0xffffffffu, part, 2);
    part += __shfl_xor_sync(0xffffffffu, part, 1);
    if (i < items && sub == 0) csum[i] = part;
  }
}

// BN backward, phase 1: per channel sum(dz) and sum(dz * xhat), dz = dy masked by the activation.
__global__ void __launch_bounds__(NT)
bn_bwd_partial_kernel(const float* __restrict__ dy, const float* __restrict__ x, int M, int C,
                      int rows_per_split, const float* __restrict__ mean, const float* __restrict__ rstd,
                      const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                      float* __restrict__ part /* [splits][2][C] */) {
  __shared__ float sh[2][NT * 4];
  const ColTile t(C);
  const int r0 = blockIdx.y * rows_per_split;
  const int r1 = min(M, r0 + rows_per_split);
  const int col = t.c0 + t.tx * 4;
  float a[4] = {0.f, 0.f, 0.f, 0.f}, b[4] = {0.f, 0.f, 0.f, 0.f};
  if (t.ty < t.nty) {
    const float4 mu4 = __ldg(reinterpret_cast<const float4*>(mean + col));
    const float4 rs4 = __ldg(reinterpret_cast<const float4*>(rstd + col));
    const float4 ga4 = __ldg(reinterpret_cast<const float4*>(gamma + col));
    const float4 be4 = __ldg(reinterpret_cast<const float4*>(beta + col));
    const float mu[4] = {mu4.x, mu4.y, mu4.z, mu4.w}, rs[4] = {rs4.x, rs4.y, rs4.z, rs4.w};
    const float ga[4] = {ga4.x, ga4.y, ga4.z, ga4.w}, be[4] = {be4.x, be4.y, be4.z, be4.w};
    for (int r = r0 + t.ty; r < r1; r += t.nty) {
      const float4 d4 = pf_ld_stream(dy + (size_t)r * C + col);
      const float4 x4 = pf_ld_stream(x + (size_t)r * C + col);
      const float d[4] = {d4.x, d4.y, d4.z, d4.w}, xv[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xh = __fmul_rn(__fsub_rn(xv[j], mu[j]), rs[j]);
        float dz = d[j];
        if (act) {
          const float z = __fadd_rn(__fmul_rn(xh, ga[j]), be[j]);
          if (!(z > 0.f) || (act == 2 && !(z < 6.f))) dz = 0.f;
        }
        a[j] += dz;
        b[j] = fmaf(dz, xh, b[j]);
      }
    }
    float* pa = &sh[0][(t.ty * t.nvec + t.tx) * 4];
    float* pb = &sh[1][(t.ty * t.nvec + t.tx) * 4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { pa[j] = a[j]; pb[j] = b[j]; }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < t.tc; c += NT) {
    float sa = 0.f, sb = 0.f;
    for (int y = 0; y < t.nty; ++y) {
      sa += sh[0][(y * t.nvec + (c >> 2)) * 4 + (c & 3)];
      sb += sh[1][(y * t.nvec + (c >> 2)) * 4 + (c & 3)];
    }
    float* p = part + (size_t)blockIdx.y * 2 * C;
    p[t.c0 + c] = sa;
    p[C + t.c0 + c] = sb;
  }
}

__global__ void __launch_bounds__(NT)
bn_bwd_final_kernel(const float* __restrict__ part, int C, int splits, float* __restrict__ dgamma,
                    float* __restrict__ dbeta) {
  // kFinalWarps warps per channel, lanes over the splits, fixed-order shuffle + smem tree (deterministic)
  constexpr int CPB = NT / 32 / kFinalWarps;
  __shared__ double sha[NT / 32], shb[NT / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cl = warp / kFinalWarps, sub = warp % kFinalWarps;
  const int c = blockIdx.x * CPB + cl;
  double sa = 0.0, sb = 0.0;
  if (c < C) {
    for (int s = sub * 32 + lane; s < splits; s += 32 * kFinalWarps) {
      sa += part[(size_t)s * 2 * C + c];
      sb += part[(size_t)s * 2 * C + C + c];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sa += __shfl_down_sync(0xffffffffu, sa, o);
    sb += __shfl_down_sync(0xffffffffu, sb, o);
  }
  if (lane == 0) { sha[warp] = sa; shb[warp] = sb; }
  __syncthreads();
  if (c < C && sub == 0 && lane == 0) {
    for (int w = 1; w < kFinalWarps; ++w) { sa += sha[warp + w]; sb += shb[warp + w]; }
    dbeta[c] = (float)sa;
    dgamma[c] = (float)sb;
  }
}

// phase 2: dx = gamma*rstd*(dz - dbeta/M - xhat*dgamma/M)   (training-mode BN)
__global__ void __launch_bounds__(NT)
bn_bwd_apply_kernel(const float* __restrict__ dy, const float* __restrict__ x, int64_t total, int C,
                    float inv_m, const float* __restrict__ mean, const float* __restrict__ rstd,
                    const float* __restrict__ gamma, const float* __restrict__ beta,
                    const float* __restrict__ dgamma, const float* __restrict__ dbeta, int act,
                    int accumulate, float* __restrict__ dx, void* __restrict__ dx_hi, void* __restrict__ dx_lo) {
  const int64_t nvec = total >> 2;
  const int64_t stride = (int64_t)gridDim.x * NT;
  int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x;
  uint32_t c = (uint32_t)((i << 2) % (uint32_t)C);
  const uint32_t step = (uint32_t)((stride << 2) % (uint32_t)C);
  auto one = [&](const float4 d4, const float4 x4, const float4 mu4, const float4 rs4, const float4 ga4,
                 const float4 be4, const float4 dg4, const float4 db4, int64_t idx) {
    const float d[4] = {d4.x, d4.y, d4.z, d4.w}, xv[4] = {x4.x, x4.y, x4.z, x4.w};
    const float mu[4] = {mu4.x, mu4.y, mu4.z, mu4.w}, rs[4] = {rs4.x, rs4.y, rs4.z, rs4.w};
    const float ga[4] = {ga4.x, ga4.y, ga4.z, ga4.w}, be[4] = {be4.x, be4.y, be4.z, be4.w};
    const float dg[4] = {dg4.x, dg4.y, dg4.z, dg4.w}, db[4] = {db4.x, db4.y, db4.z, db4.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float xh = __fmul_rn(__fsub_rn(xv[j], mu[j]), rs[j]);
      float dz = d[j];
      if (act) {
        const float z = __fadd_rn(__fmul_rn(xh, ga[j]), be[j]);
        if (!(z > 0.f) || (act == 2 && !(z < 6.f))) dz = 0.f;
      }
      o[j] = ga[j] * rs[j] * (dz - db[j] * inv_m - xh * dg[j] * inv_m);
    }
    float4 r = make_float4(o[0], o[1], o[2], o[3]);
    if (accumulate) {
      const float4 old = *reinterpret_cast<const float4*>(dx + (idx << 2));
      r.x += old.x; r.y += old.y; r.z += old.z; r.w += old.w;
    }
    if (dx) pf_st_stream(dx + (idx << 2), r);
    if (dx_hi) pf_st_planes4(dx_hi, dx_lo, idx << 2, r);
  };
  if (step == 0) {
    const float4 mu4 = __ldg(reinterpret_cast<const float4*>(mean + c)), rs4 = __ldg(reinterpret_cast<const float4*>(rstd + c));
    const float4 ga4 = __ldg(reinterpret_cast<const float4*>(gamma + c)), be4 = __ldg(reinterpret_cast<const float4*>(beta + c));
    const float4 dg4 = __ldg(reinterpret_cast<const float4*>(dgamma + c)), db4 = __ldg(reinterpret_cast<const float4*>(dbeta + c));
    for (; i + stride < nvec; i += 2 * stride) {
      const float4 d0 = pf_ld_stream(dy + (i << 2)), x0 = pf_ld_stream(x + (i << 2));
      const float4 d1 = pf_ld_stream(dy + ((i + stride) << 2)), x1 = pf_ld_stream(x + ((i + stride) << 2));
      one(d0, x0, mu4, rs4, ga4, be4, dg4, db4, i);
      one(d1, x1, mu4, rs4, ga4, be4, dg4, db4, i + stride);
    }
    for (; i < nvec; i += stride)
      one(pf_ld_stream(dy + (i << 2)), pf_ld_stream(x + (i << 2)), mu4, rs4, ga4, be4, dg4, db4, i);
  } else {
    for (; i < nvec; i += stride) {
      one(pf_ld_stream(dy + (i << 2)), pf_ld_stream(x + (i << 2)), __ldg(reinterpret_cast<const float4*>(mean + c)),
          __ldg(reinterpret_cast<const float4*>(rstd + c)), __ldg(reinterpret_cast<const float4*>(gamma + c)),
          __ldg(reinterpret_cast<const float4*>(beta + c)), __ldg(reinterpret_cast<const float4*>(dgamma + c)),
          __ldg(reinterpret_cast<const float4*>(dbeta + c)), i);
      c += step;
      if (c >= (uint32_t)C) c -= (uint32_t)C;
    }
  }
}

// ------------------------------------------------------------------ elementwise helpers
// out = a + b (residual add) ; or out (+)= a  when b == nullptr (gradient fan-out)
__global__ void __launch_bounds__(NT)
add_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, int accumulate,
           float* __restrict__ out) {
  const int64_t nvec = n >> 2;
  const int64_t stride = (int64_t)gridDim.x * NT;
  for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < nvec; i += stride) {
    float4 v = pf_ld4(a + (i << 2));
    if (b) {
      const float4 w = pf_ld4(b + (i << 2));
      v.x = __fadd_rn(v.x, w.x); v.y = __fadd_rn(v.y, w.y); v.z = __fadd_rn(v.z, w.z); v.w = __fadd_rn(v.w, w.w);
    }
    if (accumulate) {
      const float4 o = pf_ld4(out + (i << 2));
      v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
    }
    pf_st_stream(out + (i << 2), v);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t j = (nvec << 2) + threadIdx.x;
    float v = a[j] + (b ? b[j] : 0.f);
    out[j] = accumulate ? out[j] + v : v;
  }
}

// dx (+)= dy * [y > 0] (and [y < 6] for relu6)
__global__ void __launch_bounds__(NT)
relu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, int64_t n, int act,
                int accumulate, float* __restrict__ dx) {
  const int64_t stride = (int64_t)gridDim.x * NT;
  for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < n; i += stride) {
    const float yy = y[i];
    float v = (yy > 0.f && (act != 2 || yy < 6.f)) ? dy[i] : 0.f;
    dx[i] = accumulate ? dx[i] + v : v;
  }
}

// out[c] = sum_m a[m][c]   (bias gradient); fixed order per column -> deterministic
__global__ void __launch_bounds__(NT)
colsum_kernel(const float* __restrict__ a, int M, int C, float* __restrict__ out) {
  __shared__ float sh[NT];
  const int c = blockIdx.x;
  float s = 0.f;
  for (int m = threadIdx.x; m < M; m += NT) s += a[(size_t)m * C + c];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = NT / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[c] = sh[0];
}

// ------------------------------------------------------------------ pooling
// Forward also records, per output element, which window position (r*kw + q) holds the FIRST maximum
// in row-major scan order (TF's MaxPoolGrad routes the gradient there); 255 = empty window.
__global__ void __launch_bounds__(NT)
maxpool_fwd_kernel(const float* __restrict__ x, int N, int H, int W, int C, int P, int Q, int kh, int kw,
                   int sh, int sw, int pt, int pl, float* __restrict__ y, uint8_t* __restrict__ argmax) {
  // N*P*Q < 2^31 (checked on the host): 32-bit pixel index, one division chain per 4 channels
  const uint32_t C4 = (uint32_t)(C >> 2);
  const uint32_t total = (uint32_t)N * P * Q * C4;         // < 2^31 (checked on the host)
  const uint32_t stride = gridDim.x * NT;
  for (uint32_t i = blockIdx.x * NT + threadIdx.x; i < total; i += stride) {
    const uint32_t pix = i / C4;
    const int c = (int)((i - pix * C4) << 2);
    const uint32_t t1 = pix / (uint32_t)Q;
    const int ow = (int)(pix - t1 * (uint32_t)Q);
    const int n = (int)(t1 / (uint32_t)P);
    const int oh = (int)(t1 - (uint32_t)n * (uint32_t)P);
    float m[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    int a[4] = {255, 255, 255, 255};
    for (int r = 0; r < kh; ++r) {
      const int ih = oh * sh - pt + r;
      if (ih < 0 || ih >= H) continue;
      for (int q = 0; q < kw; ++q) {
        const int iw = ow * sw - pl + q;
        if (iw < 0 || iw >= W) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * H + ih) * W + iw) * C + c));
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (vv[j] > m[j]) { m[j] = vv[j]; a[j] = r * kw + q; }
      }
    }
    const size_t o = ((((size_t)n * P + oh) * Q + ow) * C + c);
    *reinterpret_cast<float4*>(y + o) = make_float4(m[0], m[1], m[2], m[3]);
    if (argmax) *reinterpret_cast<uchar4*>(argmax + o) = make_uchar4((uint8_t)a[0], (uint8_t)a[1], (uint8_t)a[2], (uint8_t)a[3]);
  }
}

// 3x3 / stride 2 (the ResNet stem pool, resnet_model.py:521-525): taps unrolled, all nine loads issued before the
// first compare (the generic kernel's data-dependent `continue`s serialise them: 2.5 TB/s -> see profiles/)
__global__ void __launch_bounds__(NT)
maxpool3x3s2_fwd_kernel(const float* __restrict__ x, int N, int H, int W, int C, int P, int Q, int pt, int pl,
                        float* __restrict__ y, uint8_t* __restrict__ argmax) {
  const uint32_t C4 = (uint32_t)(C >> 2);
  const uint32_t total = (uint32_t)N * P * Q * C4;
  const uint32_t stride = gridDim.x * NT;
  for (uint32_t i = blockIdx.x * NT + threadIdx.x; i < total; i += stride) {
    const uint32_t pix = i / C4;
    const int c = (int)((i - pix * C4) << 2);
    const uint32_t t1 = pix / (uint32_t)Q;
    const int ow = (int)(pix - t1 * (uint32_t)Q);
    const int n = (int)(t1 / (uint32_t)P);
    const int oh = (int)(t1 - (uint32_t)n * (uint32_t)P);
    const int ih0 = oh * 2 - pt, iw0 = ow * 2 - pl;
    float4 v[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int ih = ih0 + r, iw = iw0 + q;
        const bool ok = ih >= 0 && ih < H && iw >= 0 && iw < W;
        v[r * 3 + q] = ok ? __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * H + ih) * W + iw) * C + c))
                          : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
      }
    float m[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    int a[4] = {255, 255, 255, 255};
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const float vv[4] = {v[t].x, v[t].y, v[t].z, v[t].w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (vv[j] > m[j]) { m[j] = vv[j]; a[j] = t; }
    }
    const size_t o = (size_t)pix * C + c;
    *reinterpret_cast<float4*>(y + o) = make_float4(m[0], m[1], m[2], m[3]);
    if (argmax) *reinterpret_cast<uchar4*>(argmax + o) = make_uchar4((uint8_t)a[0], (uint8_t)a[1], (uint8_t)a[2], (uint8_t)a[3]);
  }
}

// backward of the same pool: an input position belongs to at most 2x2 windows; their argmax bytes and dy values are
// all requested up front
__global__ void __launch_bounds__(NT)
maxpool3x3s2_bwd_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ argmax, int N, int H, int W, int C,
                        int P, int Q, int pt, int pl, int accumulate, float* __restrict__ dx) {
  const uint32_t C4 = (uint32_t)(C >> 2);
  const uint32_t total = (uint32_t)N * H * W * C4;
  const uint32_t stride = gridDim.x * NT;
  for (uint32_t i = blockIdx.x * NT + threadIdx.x; i < total; i += stride) {
    const uint32_t pix = i / C4;
    const int c = (int)((i - pix * C4) << 2);
    const uint32_t t1 = pix / (uint32_t)W;
    const int iw = (int)(pix - t1 * (uint32_t)W);
    const int n = (int)(t1 / (uint32_t)H);
    const int ih = (int)(t1 - (uint32_t)n * (uint32_t)H);
    // windows oh in {ceil((ih+pt-2)/2) .. floor((ih+pt)/2)}: at most two per axis
    const int ohb = (ih + pt) >> 1, owb = (iw + pl) >> 1;
    uchar4 a[4];
    float4 d[4];
    int code[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int oh = ohb - (k >> 1), ow = owb - (k & 1);
      const int r = ih + pt - oh * 2, q = iw + pl - ow * 2;
      const bool ok = oh >= 0 && oh < P && ow >= 0 && ow < Q && r >= 0 && r < 3 && q >= 0 && q < 3;
      code[k] = ok ? r * 3 + q : 254;
      const size_t o = (((size_t)n * P + (ok ? oh : 0)) * Q + (ok ? ow : 0)) * C + c;
      a[k] = ok ? __ldg(reinterpret_cast<const uchar4*>(argmax + o)) : make_uchar4(255, 255, 255, 255);
      d[k] = ok ? __ldg(reinterpret_cast<const float4*>(dy + o)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    // same accumulation order as the generic kernel: oh ascending, then ow ascending
    float g[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 3; k >= 0; --k) {
      if (a[k].x == code[k]) g[0] += d[k].x;
      if (a[k].y == code[k]) g[1] += d[k].y;
      if (a[k].z == code[k]) g[2] += d[k].z;
      if (a[k].w == code[k]) g[3] += d[k].w;
    }
    float4 o4 = make_float4(g[0], g[1], g[2], g[3]);
    float* p = dx + ((size_t)i << 2);
    if (accumulate) {
      const float4 old = *reinterpret_cast<const float4*>(p);
      o4.x += old.x; o4.y += old.y; o4.z += old.z; o4.w += old.w;
    }
    *reinterpret_cast<float4*>(p) = o4;
  }
}

// dx[n,ih,iw,c] (+)= sum of dy over the windows whose recorded argmax is (ih,iw).  Gather form: no
// atomics, deterministic; each input position belongs to at most ceil(kh/sh)*ceil(kw/sw) windows.
__global__ void __launch_bounds__(NT)
maxpool_bwd_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ argmax, int N, int H, int W, int C,
                   int P, int Q, int kh, int kw, int sh, int sw, int pt, int pl, int accumulate,
                   float* __restrict__ dx) {
  const uint32_t C4 = (uint32_t)(C >> 2);
  const uint32_t total = (uint32_t)N * H * W * C4;         // < 2^31 (checked on the host)
  const uint32_t stride = gridDim.x * NT;
  for (uint32_t i = blockIdx.x * NT + threadIdx.x; i < total; i += stride) {
    const uint32_t pix = i / C4;
    const int c = (int)((i - pix * C4) << 2);
    const uint32_t t1 = pix / (uint32_t)W;
    const int iw = (int)(pix - t1 * (uint32_t)W);
    const int n = (int)(t1 / (uint32_t)H);
    const int ih = (int)(t1 - (uint32_t)n * (uint32_t)H);
    float g[4] = {0.f, 0.f, 0.f, 0.f};
    const int oh_lo = max(0, (ih + pt - kh + sh) / sh), oh_hi = min(P - 1, (ih + pt) / sh);
    const int ow_lo = max(0, (iw + pl - kw + sw) / sw), ow_hi = min(Q - 1, (iw + pl) / sw);
    for (int oh = oh_lo; oh <= oh_hi; ++oh) {
      const int r = ih + pt - oh * sh;
      for (int ow = ow_lo; ow <= ow_hi; ++ow) {
        const int q = iw + pl - ow * sw;
        const int code = r * kw + q;
        const size_t o = (((size_t)n * P + oh) * Q + ow) * C + c;
        const uchar4 a = __ldg(reinterpret_cast<const uchar4*>(argmax + o));
        if (a.x == code || a.y == code || a.z == code || a.w == code) {
          const float4 d = __ldg(reinterpret_cast<const float4*>(dy + o));
          if (a.x == code) g[0] += d.x;
          if (a.y == code) g[1] += d.y;
          if (a.z == code) g[2] += d.z;
          if (a.w == code) g[3] += d.w;
        }
      }
    }
    float4 o4 = make_float4(g[0], g[1], g[2], g[3]);
    float* p = dx + ((size_t)i << 2);
    if (accumulate) {
      const float4 old = *reinterpret_cast<const float4*>(p);
      o4.x += old.x; o4.y += old.y; o4.z += old.z; o4.w += old.w;
    }
    *reinterpret_cast<float4*>(p) = o4;
  }
}

// y[n][c] = mean over HW ; one CTA per (n, 64-channel tile)
__global__ void __launch_bounds__(NT)
gap_fwd_kernel(const float* __restrict__ x, int HW, int C, float* __restrict__ y) {
  __shared__ float sh[NT];
  const int n = blockIdx.y;
  const int cl = threadIdx.x & 63, part = threadIdx.x >> 6;  // 64 channels x 4 row-lanes
  const int c = blockIdx.x * 64 + cl;
  float s = 0.f;
  if (c < C)
    for (int p = part; p < HW; p += 4) s += __ldg(x + ((size_t)n * HW + p) * C + c);
  sh[threadIdx.x] = s;
  __syncthreads();
  if (part == 0 && c < C) {
    const float tot = (sh[cl] + sh[64 + cl]) + (sh[128 + cl] + sh[192 + cl]);
    y[(size_t)n * C + c] = __fdiv_rn(tot, (float)HW);
  }
}

__global__ void __launch_bounds__(NT)
gap_bwd_kernel(const float* __restrict__ dy, int64_t total, int HW, int C, int accumulate,
               float* __restrict__ dx) {
  const int64_t stride = (int64_t)gridDim.x * NT;
  const float inv = 1.f / (float)HW;
  for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < total; i += stride) {
    const int c = (int)(i % C);
    const int64_t n = i / ((int64_t)HW * C);
    const float g = __ldg(dy + n * C + c) * inv;
    dx[i] = accumulate ? dx[i] + g : g;
  }
}

// row softmax (LeNet ends in tf.nn.softmax, nets/lenet_at_cifar10.py:66) and its backward
__global__ void __launch_bounds__(NT)
softmax_fwd_kernel(const float* __restrict__ x, int n, int k, float* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (NT / 32) + (threadIdx.x >> 5);
  if (row >= n) return;
  const float* r = x + (size_t)row * k;
  float m = -INFINITY;
  for (int j = lane; j < k; j += 32) m = fmaxf(m, r[j]);
  m = pf_warp_max(m);
  float s = 0.f;
  for (int j = lane; j < k; j += 32) s += expf(r[j] - m);
  s = pf_warp_sum(s);
  for (int j = lane; j < k; j += 32) y[(size_t)row * k + j] = __fdiv_rn(expf(r[j] - m), s);
}
__global__ void __launch_bounds__(NT)
softmax_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, int n, int k,
                   float* __restrict__ dx) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (NT / 32) + (threadIdx.x >> 5);
  if (row >= n) return;
  float dot = 0.f;
  for (int j = lane; j < k; j += 32) dot += dy[(size_t)row * k + j] * y[(size_t)row * k + j];
  dot = pf_warp_sum(dot);
  for (int j = lane; j < k; j += 32) {
    const size_t o = (size_t)row * k + j;
    dx[o] = (dy[o] - dot) * y[o];
  }
}

// grid whose stride (gridDim*NT float4s) is a multiple of C/4, so that threads keep their channels
inline int bn_grid_cap() {                // PF_BN_GRIDCAP, read per launch
  const char* v = getenv("PF_BN_GRIDCAP");
  return (v && *v) ? atoi(v) : 8;
}
inline unsigned chan_grid(int64_t nvec, int C) {
  int64_t want = (nvec + NT - 1) / NT;
  const int64_t cap = (int64_t)PF_NUM_SMS * bn_grid_cap();
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  const int c4 = C >> 2;
  int64_t mult = 1;
  while ((mult * NT) % c4 != 0 && mult < 64) mult <<= 1;   // C/4 is 2^a * odd; NT = 256 covers 2^a <= 256
  if ((mult * NT) % c4 == 0) want = (want + mult - 1) / mult * mult;
  return (unsigned)want;
}

inline unsigned ew_grid(int64_t work_items) {
  int64_t want = (work_items + NT - 1) / NT;
  const int64_t cap = (int64_t)PF_NUM_SMS * 8;
  if (want < 1) want = 1;
  return (unsigned)(want < cap ? want : cap);
}

inline int bn_splits(int M, int C, int* rows_per_split) {
  const int col_tiles = (C + kColTile - 1) / kColTile;
  int splits = (8 * PF_NUM_SMS + col_tiles - 1) / col_tiles;
  const int max_by_rows = (M + 63) / 64;
  if (splits > max_by_rows) splits = max_by_rows;
  if (splits > PF_BN_MAX_SPLITS) splits = PF_BN_MAX_SPLITS;
  if (splits < 1) splits = 1;
  int rps = (M + splits - 1) / splits;
  *rows_per_split = rps;
  return (M + rps - 1) / rps;
}

// dst[i][j] = sum_b src[b*m + i][b*n + j]: the diagonal blocks of a (g*m) x (g*n) matrix folded onto each other — the
// weight gradient of a conv with fewer than 64 output channels, computed on the tensor cores from g pixels per GEMM row
// (engine: the 3 -> 32 stem of MobileNet-v1)
__global__ void __launch_bounds__(NT)
fold_diag_blocks_kernel(const float* __restrict__ src, int g, int m, int n, float* __restrict__ dst) {
  const int i = blockIdx.x * NT + threadIdx.x;
  if (i >= m * n) return;
  const int r = i / n, c = i - r * n;
  float acc = 0.f;
  for (int b = 0; b < g; ++b) acc += src[(size_t)(b * m + r) * (g * n) + b * n + c];
  dst[i] = acc;
}
}  // namespace

extern "C" {

int pf_bn_train_stats_range(const float* x_dev, int64_t m, int c, float eps, float momentum, float* mean_dev,
                            float* var_dev, float* rstd_dev, float* moving_mean_dev, float* moving_var_dev,
                            const float* gamma_dev, const float* beta_dev, int act, uint32_t* minmax_enc_dev,
                            float* ws_dev, void* stream) {
  PF_REQUIRE(m > 0 && c > 0 && m < (1ll << 31), "pf_bn_train_stats: bad shape");
  PF_REQUIRE((c & 3) == 0, "pf_bn_train_stats: C must be a multiple of 4 (got %d)", c);
  PF_REQUIRE(x_dev && mean_dev && var_dev && rstd_dev && ws_dev, "pf_bn_train_stats: null pointer");
  PF_REQUIRE((moving_mean_dev == nullptr) == (moving_var_dev == nullptr), "pf_bn_train_stats: moving stats come in pairs");
  PF_REQUIRE(minmax_enc_dev == nullptr || (gamma_dev && beta_dev && act >= 0 && act <= 2),
             "pf_bn_train_stats_range: the output range needs gamma, beta and act in {0,1,2}");
  int rps;
  const int splits = bn_splits((int)m, c, &rps);
  dim3 grid((c + kColTile - 1) / kColTile, splits);
  cudaStream_t st = (cudaStream_t)stream;
  const int nf = minmax_enc_dev ? 5 : 3;
  if (minmax_enc_dev) bn_stats_partial_kernel<true><<<grid, NT, 0, st>>>(x_dev, (int)m, c, rps, ws_dev);
  else bn_stats_partial_kernel<false><<<grid, NT, 0, st>>>(x_dev, (int)m, c, rps, ws_dev);
  PF_CHECK_LAUNCH("pf_bn_train_stats/partial");
  constexpr int kCPB = NT / 32 / kFinalWarps;
  bn_stats_final_kernel<<<(c + kCPB - 1) / kCPB, NT, 0, st>>>(ws_dev, (int)m, c, splits, rps, eps, momentum, mean_dev,
                                                         var_dev, rstd_dev, moving_mean_dev, moving_var_dev, nf, gamma_dev,
                                                         beta_dev, act, minmax_enc_dev);
  PF_CHECK_LAUNCH("pf_bn_train_stats/final");
  return PF_OK;
}

int pf_bn_train_stats(const float* x_dev, int64_t m, int c, float eps, float momentum, float* mean_dev,
                      float* var_dev, float* rstd_dev, float* moving_mean_dev, float* moving_var_dev,
                      float* ws_dev, void* stream) {
  return pf_bn_train_stats_range(x_dev, m, c, eps, momentum, mean_dev, var_dev, rstd_dev, moving_mean_dev, moving_var_dev,
                                 nullptr, nullptr, 0, nullptr, ws_dev, stream);
}

int pf_bn_eval_prepare(const float* moving_var_dev, int c, float eps, float* rstd_dev, void* stream) {
  PF_REQUIRE(c > 0 && moving_var_dev && rstd_dev, "pf_bn_eval_prepare: bad arguments");
  bn_eval_prepare_kernel<<<(c + NT - 1) / NT, NT, 0, (cudaStream_t)stream>>>(moving_var_dev, c, eps, rstd_dev);
  PF_CHECK_LAUNCH("pf_bn_eval_prepare");
  return PF_OK;
}

static int bn_apply_impl(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                         const float* gamma_dev, const float* beta_dev, int act, float* y_dev, void* y_hi_dev,
                         void* y_lo_dev, uint32_t* minmax_enc_dev, const uint32_t* q_range_dev, int q_bits, void* stream,
                         float var_eps = -1.f, const float* res_dev = nullptr, bool clamp = false) {
  PF_REQUIRE(m > 0 && c > 0 && (c & 3) == 0, "pf_bn_apply: bad shape (C must be a multiple of 4)");
  PF_REQUIRE(act >= 0 && act <= 2, "pf_bn_apply: act must be 0 (none), 1 (relu) or 2 (relu6)");
  PF_REQUIRE(x_dev && mean_dev && rstd_dev && gamma_dev && beta_dev, "pf_bn_apply: null pointer");
  PF_REQUIRE(y_dev || y_hi_dev, "pf_bn_apply: no output");
  PF_REQUIRE((y_hi_dev == nullptr) == (y_lo_dev == nullptr), "pf_bn_apply: planes come in pairs");
  PF_REQUIRE((((uintptr_t)y_hi_dev | (uintptr_t)y_lo_dev) & 7) == 0, "pf_bn_apply: planes must be 8-byte aligned");
  const int64_t total = m * c;
  const unsigned grid = chan_grid(total >> 2, c);
  if (clamp)
    bn_apply_kernel<false, true><<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, total, c, mean_dev, rstd_dev, gamma_dev, beta_dev,
                                                                        act, y_dev, nullptr, y_hi_dev, y_lo_dev, q_range_dev,
                                                                        q_bits, var_eps, nullptr);
  else if (res_dev)
    bn_apply_kernel<true><<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, total, c, mean_dev, rstd_dev, gamma_dev, beta_dev, act,
                                                                 y_dev, minmax_enc_dev, y_hi_dev, y_lo_dev, q_range_dev, q_bits,
                                                                 var_eps, res_dev);
  else
    bn_apply_kernel<false><<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, total, c, mean_dev, rstd_dev, gamma_dev, beta_dev, act,
                                                                  y_dev, minmax_enc_dev, y_hi_dev, y_lo_dev, q_range_dev, q_bits,
                                                                  var_eps, nullptr);
  PF_CHECK_LAUNCH("pf_bn_apply");
  return PF_OK;
}

int pf_bn_apply_planes(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                       const float* gamma_dev, const float* beta_dev, int act, float* y_dev, void* y_hi_dev,
                       void* y_lo_dev, uint32_t* minmax_enc_dev, void* stream) {
  return bn_apply_impl(x_dev, m, c, mean_dev, rstd_dev, gamma_dev, beta_dev, act, y_dev, y_hi_dev, y_lo_dev, minmax_enc_dev,
                       nullptr, 0, stream);
}

int pf_bn_apply_eval(const float* x_dev, int64_t m, int c, const float* moving_mean_dev, const float* moving_var_dev,
                     float eps, const float* gamma_dev, const float* beta_dev, int act, float* y_dev, void* y_hi_dev,
                     void* y_lo_dev, uint32_t* minmax_enc_dev, void* stream) {
  PF_REQUIRE(eps >= 0.f, "pf_bn_apply_eval: eps < 0");
  return bn_apply_impl(x_dev, m, c, moving_mean_dev, moving_var_dev, gamma_dev, beta_dev, act, y_dev, y_hi_dev, y_lo_dev,
                       minmax_enc_dev, nullptr, 0, stream, eps);
}

int pf_bn_apply_eval_quant_static(const float* x_dev, int64_t m, int c, const float* moving_mean_dev,
                                  const float* moving_var_dev, float eps, const float* gamma_dev, const float* beta_dev,
                                  int act, const uint32_t* range_enc_dev, int bits, float* y_dev, void* y_hi_dev,
                                  void* y_lo_dev, void* stream) {
  PF_REQUIRE(eps >= 0.f, "pf_bn_apply_eval_quant_static: eps < 0");
  PF_REQUIRE(range_enc_dev != nullptr, "pf_bn_apply_eval_quant_static: null range");
  PF_REQUIRE(bits >= 1 && bits <= 32, "pf_bn_apply_eval_quant_static: bits must be in [1, 32]");
  return bn_apply_impl(x_dev, m, c, moving_mean_dev, moving_var_dev, gamma_dev, beta_dev, act, y_dev, y_hi_dev, y_lo_dev,
                       nullptr, range_enc_dev, bits, stream, eps, nullptr, true);
}

int pf_bn_apply_quant(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                      const float* gamma_dev, const float* beta_dev, int act, const uint32_t* range_enc_dev, int bits,
                      float* y_dev, void* y_hi_dev, void* y_lo_dev, void* stream) {
  PF_REQUIRE(range_enc_dev != nullptr, "pf_bn_apply_quant: null range");
  PF_REQUIRE(bits >= 1 && bits <= 32, "pf_bn_apply_quant: bits must be in [1, 32]");
  return bn_apply_impl(x_dev, m, c, mean_dev, rstd_dev, gamma_dev, beta_dev, act, y_dev, y_hi_dev, y_lo_dev, nullptr,
                       range_enc_dev, bits, stream);
}

int pf_bn_apply_quant_levels(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                             const float* gamma_dev, const float* beta_dev, int act, const uint32_t* range_enc_dev,
                             int bits, float* y_dev, void* plane0_dev, void* plane1_dev, pf_tc_act_hdr* hdr_dev,
                             float* csum_dev, void* stream) {
  PF_REQUIRE(m > 0 && c >= 16 && (c & (c - 1)) == 0, "pf_bn_apply_quant_levels: C must be a power of two >= 16 (got %d)", c);
  PF_REQUIRE(act >= 0 && act <= 2, "pf_bn_apply_quant_levels: act must be 0 (none), 1 (relu) or 2 (relu6)");
  PF_REQUIRE(bits >= 1 && bits <= 32, "pf_bn_apply_quant_levels: bits must be in [1, 32]");
  PF_REQUIRE(x_dev && mean_dev && rstd_dev && gamma_dev && beta_dev && range_enc_dev && plane0_dev && plane1_dev && hdr_dev &&
                 csum_dev, "pf_bn_apply_quant_levels: null pointer");
  PF_REQUIRE((((uintptr_t)plane0_dev | (uintptr_t)plane1_dev | (uintptr_t)hdr_dev) & 7) == 0,
             "pf_bn_apply_quant_levels: planes / header must be 8-byte aligned");
  const int64_t total = m * c;
  int cshift = 0;
  while ((1 << cshift) < c) ++cshift;
  const int nseg = (c + 127) / 128;
  // grid: a multiple of (C/4)/gcd(C/4, NT) blocks so that every thread keeps its 4 channels (C/4 <= NT * 64 here)
  unsigned grid = chan_grid(total >> 2, c);
  PF_REQUIRE(((int64_t)grid * NT) % (c >> 2) == 0, "pf_bn_apply_quant_levels: C = %d too large for the channel-stationary grid", c);
  if (y_dev == nullptr && bits <= 8)
    bn_apply_levels_kernel<true><<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, total, c, cshift, mean_dev, rstd_dev, gamma_dev,
                                                                       beta_dev, act, nullptr, plane0_dev, plane1_dev,
                                                                       range_enc_dev, bits, hdr_dev, csum_dev, nseg);
  else
    bn_apply_levels_kernel<false><<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, total, c, cshift, mean_dev, rstd_dev, gamma_dev,
                                                                        beta_dev, act, y_dev, plane0_dev, plane1_dev,
                                                                        range_enc_dev, bits, hdr_dev, csum_dev, nseg);
  PF_CHECK_LAUNCH("pf_bn_apply_quant_levels");
  return PF_OK;
}

// have_range: 0 = reset range_enc and run the range pass first, 1 = range_enc holds this batch's range, 2 = it holds
// a calibrated range (the clamping level pass only)
static int bn_eval_levels_u8_impl(const char* who, const float* x_dev, int64_t m, int c, const float* moving_mean_dev,
                                  const float* moving_var_dev, float eps, const float* gamma_dev, const float* beta_dev,
                                  int act, int bits, uint32_t* range_enc_dev, int have_range, void* levels_dev,
                                  pf_tc_act_hdr* hdr_dev, float* csum_dev, void* stream) {
  PF_REQUIRE(m > 0 && c >= 16 && c % 16 == 0, "%s: C must be a multiple of 16 (got %d)", who, c);
  PF_REQUIRE(act >= 0 && act <= 2, "%s: act must be 0 (none), 1 (relu) or 2 (relu6)", who);
  PF_REQUIRE(bits >= 1 && bits <= 8, "%s: u8 levels need 1..8 bits", who);
  PF_REQUIRE(eps >= 0.f, "%s: eps < 0", who);
  PF_REQUIRE(x_dev && moving_mean_dev && moving_var_dev && gamma_dev && beta_dev && range_enc_dev && levels_dev && hdr_dev &&
                 csum_dev, "%s: null pointer", who);
  PF_REQUIRE((((uintptr_t)x_dev | (uintptr_t)moving_mean_dev | (uintptr_t)moving_var_dev | (uintptr_t)gamma_dev |
               (uintptr_t)beta_dev) & 15) == 0 && (((uintptr_t)levels_dev | (uintptr_t)hdr_dev) & 7) == 0,
             "%s: fp32 tensors must be 16-byte aligned, levels / header 8-byte aligned", who);
  const int64_t total = m * c;
  const int nseg = (c + 127) / 128;
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* lv = reinterpret_cast<uint8_t*>(levels_dev);
  if (c & (c - 1)) {
    // groups of 8 lanes per (pixel, segment) item; a multiple of nseg groups in the grid
    const int64_t items = m * nseg;
    int64_t grid = std::min((items * 8 + NT - 1) / NT, (int64_t)PF_NUM_SMS * bn_grid_cap());
    const int64_t mult = nseg / std::gcd(nseg, NT / 8);
    grid = std::max<int64_t>(1, (grid + mult - 1) / mult) * mult;
    if (have_range == 2) {
      bn_eval_levels_u8_seg_kernel<false, true><<<(unsigned)grid, NT, 0, st>>>(x_dev, items, c, nseg, moving_mean_dev,
                                                                               moving_var_dev, eps, gamma_dev, beta_dev, act,
                                                                               range_enc_dev, bits, lv, hdr_dev, csum_dev);
      PF_CHECK_LAUNCH(who);
      return PF_OK;
    }
    if (!have_range) {
      const int rc = pf_minmax_reset(range_enc_dev, 1, stream);
      if (rc) return rc;
      bn_eval_levels_u8_seg_kernel<true><<<(unsigned)grid, NT, 0, st>>>(x_dev, items, c, nseg, moving_mean_dev,
                                                                        moving_var_dev, eps, gamma_dev, beta_dev, act,
                                                                        range_enc_dev, bits, lv, hdr_dev, csum_dev);
      PF_CHECK_LAUNCH(who);
    }
    bn_eval_levels_u8_seg_kernel<false><<<(unsigned)grid, NT, 0, st>>>(x_dev, items, c, nseg, moving_mean_dev,
                                                                       moving_var_dev, eps, gamma_dev, beta_dev, act,
                                                                       range_enc_dev, bits, lv, hdr_dev, csum_dev);
    PF_CHECK_LAUNCH(who);
    return PF_OK;
  }
  int cshift = 0;
  while ((1 << cshift) < c) ++cshift;
  const unsigned grid = chan_grid(total >> 2, c);
  PF_REQUIRE(((int64_t)grid * NT) % (c >> 2) == 0, "%s: C = %d too large for the channel-stationary grid", who, c);
  if (have_range == 2) {
    bn_eval_levels_u8_kernel<false, true><<<grid, NT, 0, st>>>(x_dev, total, c, cshift, moving_mean_dev, moving_var_dev,
                                                               eps, gamma_dev, beta_dev, act, range_enc_dev, bits, lv,
                                                               hdr_dev, csum_dev, nseg);
    PF_CHECK_LAUNCH(who);
    return PF_OK;
  }
  if (!have_range) {
    const int rc = pf_minmax_reset(range_enc_dev, 1, stream);
    if (rc) return rc;
    bn_eval_levels_u8_kernel<true><<<grid, NT, 0, st>>>(x_dev, total, c, cshift, moving_mean_dev, moving_var_dev, eps,
                                                        gamma_dev, beta_dev, act, range_enc_dev, bits, lv, hdr_dev,
                                                        csum_dev, nseg);
    PF_CHECK_LAUNCH(who);
  }
  bn_eval_levels_u8_kernel<false><<<grid, NT, 0, st>>>(x_dev, total, c, cshift, moving_mean_dev, moving_var_dev, eps,
                                                       gamma_dev, beta_dev, act, range_enc_dev, bits, lv, hdr_dev, csum_dev,
                                                       nseg);
  PF_CHECK_LAUNCH(who);
  return PF_OK;
}

int pf_bn_eval_levels_u8(const float* x_dev, int64_t m, int c, const float* moving_mean_dev, const float* moving_var_dev,
                         float eps, const float* gamma_dev, const float* beta_dev, int act, int bits,
                         uint32_t* range_enc_dev, int have_range, void* levels_dev, pf_tc_act_hdr* hdr_dev,
                         float* csum_dev, void* stream) {
  return bn_eval_levels_u8_impl("pf_bn_eval_levels_u8", x_dev, m, c, moving_mean_dev, moving_var_dev, eps, gamma_dev,
                                beta_dev, act, bits, range_enc_dev, have_range ? 1 : 0, levels_dev, hdr_dev, csum_dev,
                                stream);
}

int pf_bn_eval_levels_u8_static(const float* x_dev, int64_t m, int c, const float* moving_mean_dev,
                                const float* moving_var_dev, float eps, const float* gamma_dev, const float* beta_dev,
                                int act, int bits, const uint32_t* range_enc_dev, void* levels_dev,
                                pf_tc_act_hdr* hdr_dev, float* csum_dev, void* stream) {
  // the kernels read range_enc only in the level pass (have_range 2 launches no other)
  return bn_eval_levels_u8_impl("pf_bn_eval_levels_u8_static", x_dev, m, c, moving_mean_dev, moving_var_dev, eps,
                                gamma_dev, beta_dev, act, bits, const_cast<uint32_t*>(range_enc_dev), 2, levels_dev,
                                hdr_dev, csum_dev, stream);
}

int pf_bn_apply_add(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                    const float* gamma_dev, const float* beta_dev, const float* res_dev, float* y_dev, void* y_hi_dev,
                    void* y_lo_dev, void* stream) {
  PF_REQUIRE(res_dev != nullptr, "pf_bn_apply_add: null residual");
  PF_REQUIRE((((uintptr_t)res_dev | (uintptr_t)x_dev | (uintptr_t)y_dev) & 15) == 0, "pf_bn_apply_add: fp32 tensors must be 16-byte aligned");
  return bn_apply_impl(x_dev, m, c, mean_dev, rstd_dev, gamma_dev, beta_dev, 0, y_dev, y_hi_dev, y_lo_dev, nullptr, nullptr, 0,
                       stream, -1.f, res_dev);
}

int pf_bn_apply_add_eval(const float* x_dev, int64_t m, int c, const float* moving_mean_dev, const float* moving_var_dev,
                         float eps, const float* gamma_dev, const float* beta_dev, const float* res_dev, float* y_dev,
                         void* y_hi_dev, void* y_lo_dev, void* stream) {
  PF_REQUIRE(eps >= 0.f, "pf_bn_apply_add_eval: eps < 0");
  PF_REQUIRE(res_dev != nullptr, "pf_bn_apply_add_eval: null residual");
  PF_REQUIRE((((uintptr_t)res_dev | (uintptr_t)x_dev | (uintptr_t)y_dev) & 15) == 0,
             "pf_bn_apply_add_eval: fp32 tensors must be 16-byte aligned");
  return bn_apply_impl(x_dev, m, c, moving_mean_dev, moving_var_dev, gamma_dev, beta_dev, 0, y_dev, y_hi_dev, y_lo_dev, nullptr,
                       nullptr, 0, stream, eps, res_dev);
}

int pf_bn_apply(const float* x_dev, int64_t m, int c, const float* mean_dev, const float* rstd_dev,
                const float* gamma_dev, const float* beta_dev, int act, float* y_dev,
                uint32_t* minmax_enc_dev, void* stream) {
  PF_REQUIRE(y_dev != nullptr, "pf_bn_apply: null pointer");
  return pf_bn_apply_planes(x_dev, m, c, mean_dev, rstd_dev, gamma_dev, beta_dev, act, y_dev, nullptr, nullptr,
                            minmax_enc_dev, stream);
}

int pf_bn_bwd_planes(const float* dy_dev, const float* x_dev, int64_t m, int c, const float* mean_dev,
                     const float* rstd_dev, const float* gamma_dev, const float* beta_dev, int act,
                     float* dgamma_dev, float* dbeta_dev, float* dx_dev, int accumulate, void* dx_hi_dev,
                     void* dx_lo_dev, float* ws_dev, void* stream) {
  PF_REQUIRE(m > 0 && c > 0 && (c & 3) == 0 && m < (1ll << 31), "pf_bn_bwd: bad shape (C must be a multiple of 4)");
  PF_REQUIRE(dy_dev && x_dev && mean_dev && rstd_dev && gamma_dev && beta_dev && dgamma_dev && dbeta_dev && ws_dev,
             "pf_bn_bwd: null pointer");
  PF_REQUIRE(dx_dev || dx_hi_dev, "pf_bn_bwd: no output");
  PF_REQUIRE((dx_hi_dev == nullptr) == (dx_lo_dev == nullptr), "pf_bn_bwd: planes come in pairs");
  PF_REQUIRE(!accumulate || dx_dev, "pf_bn_bwd: accumulate needs the fp32 dx");
  PF_REQUIRE((((uintptr_t)dx_hi_dev | (uintptr_t)dx_lo_dev) & 7) == 0, "pf_bn_bwd: planes must be 8-byte aligned");
  int rps;
  const int splits = bn_splits((int)m, c, &rps);
  dim3 grid((c + kColTile - 1) / kColTile, splits);
  cudaStream_t st = (cudaStream_t)stream;
  bn_bwd_partial_kernel<<<grid, NT, 0, st>>>(dy_dev, x_dev, (int)m, c, rps, mean_dev, rstd_dev, gamma_dev, beta_dev,
                                            act, ws_dev);
  PF_CHECK_LAUNCH("pf_bn_bwd/partial");
  bn_bwd_final_kernel<<<(c + NT / 32 / kFinalWarps - 1) / (NT / 32 / kFinalWarps), NT, 0, st>>>(ws_dev, c, splits, dgamma_dev, dbeta_dev);
  PF_CHECK_LAUNCH("pf_bn_bwd/final");
  const int64_t total = m * c;
  bn_bwd_apply_kernel<<<chan_grid(total >> 2, c), NT, 0, st>>>(dy_dev, x_dev, total, c, 1.f / (float)m, mean_dev, rstd_dev,
                                                        gamma_dev, beta_dev, dgamma_dev, dbeta_dev, act, accumulate,
                                                        dx_dev, dx_hi_dev, dx_lo_dev);
  PF_CHECK_LAUNCH("pf_bn_bwd/apply");
  return PF_OK;
}

int pf_bn_bwd(const float* dy_dev, const float* x_dev, int64_t m, int c, const float* mean_dev,
              const float* rstd_dev, const float* gamma_dev, const float* beta_dev, int act,
              float* dgamma_dev, float* dbeta_dev, float* dx_dev, int accumulate, float* ws_dev,
              void* stream) {
  PF_REQUIRE(dx_dev != nullptr, "pf_bn_bwd: null pointer");
  return pf_bn_bwd_planes(dy_dev, x_dev, m, c, mean_dev, rstd_dev, gamma_dev, beta_dev, act, dgamma_dev, dbeta_dev,
                          dx_dev, accumulate, nullptr, nullptr, ws_dev, stream);
}

int pf_fold_diag_blocks(const float* src_dev, int g, int m, int n, float* dst_dev, void* stream) {
  PF_REQUIRE(g >= 1 && m >= 1 && n >= 1 && (int64_t)m * n < (1ll << 30), "pf_fold_diag_blocks: bad shape");
  PF_REQUIRE(src_dev && dst_dev, "pf_fold_diag_blocks: null pointer");
  fold_diag_blocks_kernel<<<(m * n + NT - 1) / NT, NT, 0, (cudaStream_t)stream>>>(src_dev, g, m, n, dst_dev);
  PF_CHECK_LAUNCH("pf_fold_diag_blocks");
  return PF_OK;
}

int pf_add(const float* a_dev, const float* b_dev, int64_t n, int accumulate, float* out_dev, void* stream) {
  PF_REQUIRE(n >= 0, "pf_add: n < 0");
  if (n == 0) return PF_OK;
  PF_REQUIRE(a_dev && out_dev, "pf_add: null pointer");
  PF_REQUIRE((((uintptr_t)a_dev | (uintptr_t)b_dev | (uintptr_t)out_dev) & 15) == 0, "pf_add: 16-byte alignment required");
  add_kernel<<<ew_grid(n >> 2), NT, 0, (cudaStream_t)stream>>>(a_dev, b_dev, n, accumulate, out_dev);
  PF_CHECK_LAUNCH("pf_add");
  return PF_OK;
}

int pf_relu_bwd(const float* dy_dev, const float* y_dev, int64_t n, int act, int accumulate, float* dx_dev,
                void* stream) {
  PF_REQUIRE(n >= 0 && (act == 1 || act == 2), "pf_relu_bwd: bad arguments");
  if (n == 0) return PF_OK;
  PF_REQUIRE(dy_dev && y_dev && dx_dev, "pf_relu_bwd: null pointer");
  relu_bwd_kernel<<<ew_grid(n), NT, 0, (cudaStream_t)stream>>>(dy_dev, y_dev, n, act, accumulate, dx_dev);
  PF_CHECK_LAUNCH("pf_relu_bwd");
  return PF_OK;
}

int pf_colsum(const float* a_dev, int64_t m, int c, float* out_dev, void* stream) {
  PF_REQUIRE(m > 0 && c > 0 && m < (1ll << 31) && a_dev && out_dev, "pf_colsum: bad arguments");
  colsum_kernel<<<c, NT, 0, (cudaStream_t)stream>>>(a_dev, (int)m, c, out_dev);
  PF_CHECK_LAUNCH("pf_colsum");
  return PF_OK;
}

int pf_maxpool_fwd(const pf_conv_desc* d, const float* x_dev, float* y_dev, uint8_t* argmax_dev, void* stream) {
  PF_REQUIRE(d && x_dev && y_dev && d->n > 0 && d->c > 0 && d->p > 0 && d->q > 0, "pf_maxpool_fwd: bad arguments");
  PF_REQUIRE((d->c & 3) == 0 && d->r * d->s < 255, "pf_maxpool_fwd: C must be a multiple of 4 and the window < 255");
  const int64_t total = (int64_t)d->n * d->p * d->q * (d->c >> 2);
  PF_REQUIRE(total < (1ll << 31), "pf_maxpool_fwd: tensor too large");
  if (d->r == 3 && d->s == 3 && d->stride_h == 2 && d->stride_w == 2) {
    maxpool3x3s2_fwd_kernel<<<ew_grid(total), NT, 0, (cudaStream_t)stream>>>(x_dev, d->n, d->h, d->w, d->c, d->p, d->q,
                                                                            d->pad_t, d->pad_l, y_dev, argmax_dev);
    PF_CHECK_LAUNCH("pf_maxpool_fwd");
    return PF_OK;
  }
  maxpool_fwd_kernel<<<ew_grid(total), NT, 0, (cudaStream_t)stream>>>(x_dev, d->n, d->h, d->w, d->c, d->p, d->q, d->r,
                                                                     d->s, d->stride_h, d->stride_w, d->pad_t,
                                                                     d->pad_l, y_dev, argmax_dev);
  PF_CHECK_LAUNCH("pf_maxpool_fwd");
  return PF_OK;
}

int pf_maxpool_bwd(const pf_conv_desc* d, const float* dy_dev, const uint8_t* argmax_dev, int accumulate,
                   float* dx_dev, void* stream) {
  PF_REQUIRE(d && dy_dev && argmax_dev && dx_dev && d->n > 0 && d->c > 0, "pf_maxpool_bwd: bad arguments");
  PF_REQUIRE((d->c & 3) == 0, "pf_maxpool_bwd: C must be a multiple of 4");
  const int64_t total = (int64_t)d->n * d->h * d->w * (d->c >> 2);
  PF_REQUIRE(total < (1ll << 31), "pf_maxpool_bwd: tensor too large");
  if (d->r == 3 && d->s == 3 && d->stride_h == 2 && d->stride_w == 2) {
    maxpool3x3s2_bwd_kernel<<<ew_grid(total), NT, 0, (cudaStream_t)stream>>>(dy_dev, argmax_dev, d->n, d->h, d->w, d->c, d->p,
                                                                            d->q, d->pad_t, d->pad_l, accumulate, dx_dev);
    PF_CHECK_LAUNCH("pf_maxpool_bwd");
    return PF_OK;
  }
  maxpool_bwd_kernel<<<ew_grid(total), NT, 0, (cudaStream_t)stream>>>(dy_dev, argmax_dev, d->n, d->h, d->w, d->c,
                                                                     d->p, d->q, d->r, d->s, d->stride_h,
                                                                     d->stride_w, d->pad_t, d->pad_l, accumulate,
                                                                     dx_dev);
  PF_CHECK_LAUNCH("pf_maxpool_bwd");
  return PF_OK;
}

int pf_global_avgpool_fwd(const float* x_dev, int n, int hw, int c, float* y_dev, void* stream) {
  PF_REQUIRE(n > 0 && hw > 0 && c > 0 && x_dev && y_dev, "pf_global_avgpool_fwd: bad arguments");
  dim3 grid((c + 63) / 64, n);
  gap_fwd_kernel<<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, hw, c, y_dev);
  PF_CHECK_LAUNCH("pf_global_avgpool_fwd");
  return PF_OK;
}

int pf_global_avgpool_bwd(const float* dy_dev, int n, int hw, int c, int accumulate, float* dx_dev, void* stream) {
  PF_REQUIRE(n > 0 && hw > 0 && c > 0 && dy_dev && dx_dev, "pf_global_avgpool_bwd: bad arguments");
  const int64_t total = (int64_t)n * hw * c;
  gap_bwd_kernel<<<ew_grid(total), NT, 0, (cudaStream_t)stream>>>(dy_dev, total, hw, c, accumulate, dx_dev);
  PF_CHECK_LAUNCH("pf_global_avgpool_bwd");
  return PF_OK;
}

int pf_softmax_fwd(const float* x_dev, int n, int k, float* y_dev, void* stream) {
  PF_REQUIRE(n > 0 && k > 0 && x_dev && y_dev, "pf_softmax_fwd: bad arguments");
  softmax_fwd_kernel<<<(n + 7) / 8, NT, 0, (cudaStream_t)stream>>>(x_dev, n, k, y_dev);
  PF_CHECK_LAUNCH("pf_softmax_fwd");
  return PF_OK;
}

int pf_softmax_bwd(const float* dy_dev, const float* y_dev, int n, int k, float* dx_dev, void* stream) {
  PF_REQUIRE(n > 0 && k > 0 && dy_dev && y_dev && dx_dev, "pf_softmax_bwd: bad arguments");
  softmax_bwd_kernel<<<(n + 7) / 8, NT, 0, (cudaStream_t)stream>>>(dy_dev, y_dev, n, k, dx_dev);
  PF_CHECK_LAUNCH("pf_softmax_bwd");
  return PF_OK;
}

}  // extern "C"
