// pf_dropout.cu — dropout in the training step (slim.dropout, MobileNet-v2's head, mobilenet.py:369 with
// keep_prob = 0.8 from training_scope, :418).  TF 1.x semantics (nn_ops.dropout): y = (x / keep) * floor(keep + u)
// with u uniform in [0, 1), each step rounded in fp32; the backward is dx = (dy * mask) / keep.
//
// The uniforms come from Philox4x32-10 (Salmon et al., SC'11), keyed by (seed, rank); the 128-bit counter is
// (element group [2 words], step [low 32 bits], stream): one Philox block gives the 4 uniforms of elements 4g .. 4g+3,
// and `stream` (the Dropout op's index in the graph, each op with its own step counter) keeps the masks of several
// Dropout ops of one graph independent (the step wraps after 2^32 launches).  u = float(0x3f800000 | (word & 0x7fffff))
// - 1, the 23-bit conversion of TF's random_uniform.  The step lives in device memory and the
// forward advances it once every CTA has read it, so a captured CUDA graph draws a new mask on every replay and the
// eager step i and the graph replay of step i draw the same mask.  TF's own stream (Philox keyed by the graph seed,
// counters in its own order) cannot be reproduced: the distribution and the scaling are the same, the draws are not.
#include "pf_common.cuh"

namespace {

constexpr int NT = 256;

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k.x += W0; k.y += W1; }
    const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
    const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

__device__ __forceinline__ float u01(uint32_t w) { return __uint_as_float(0x3f800000u | (w & 0x7fffffu)) - 1.f; }

// state[0]: step counter; state[1]: ticket of the CTAs that have read it this launch.  VEC: n % 4 == 0 and 16-byte
// aligned x / y (4-byte aligned mask): one float4 load, one float4 store and one 4-byte mask store per group.
template <bool VEC>
__global__ void __launch_bounds__(NT)
dropout_fwd_kernel(const float* __restrict__ x, int64_t n, float keep, uint2 key, uint32_t stream,
                   unsigned long long* state, float* __restrict__ y, uint8_t* __restrict__ mask) {
  __shared__ unsigned long long s_step;
  if (threadIdx.x == 0) s_step = __ldcg(state);
  __syncthreads();
  const unsigned long long step = s_step;
  const int64_t ngroups = (n + 3) >> 2;
  for (int64_t g = (int64_t)blockIdx.x * NT + threadIdx.x; g < ngroups; g += (int64_t)gridDim.x * NT) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), (uint32_t)step, stream), key);
    const float m0 = floorf(__fadd_rn(keep, u01(r.x))), m1 = floorf(__fadd_rn(keep, u01(r.y)));
    const float m2 = floorf(__fadd_rn(keep, u01(r.z))), m3 = floorf(__fadd_rn(keep, u01(r.w)));
    if (VEC) {
      const float4 v = *reinterpret_cast<const float4*>(x + 4 * g);
      *reinterpret_cast<float4*>(y + 4 * g) = make_float4(__fmul_rn(__fdiv_rn(v.x, keep), m0), __fmul_rn(__fdiv_rn(v.y, keep), m1),
                                                          __fmul_rn(__fdiv_rn(v.z, keep), m2), __fmul_rn(__fdiv_rn(v.w, keep), m3));
      *reinterpret_cast<uint32_t*>(mask + 4 * g) =
          (uint32_t)m0 | ((uint32_t)m1 << 8) | ((uint32_t)m2 << 16) | ((uint32_t)m3 << 24);
    } else {
      const float m[4] = {m0, m1, m2, m3};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int64_t i = 4 * g + j;
        if (i < n) {
          y[i] = __fmul_rn(__fdiv_rn(x[i], keep), m[j]);
          mask[i] = (uint8_t)m[j];
        }
      }
    }
  }
  if (threadIdx.x == 0) {
    // the last CTA to take a ticket advances the step: every CTA has read the old value by then
    __threadfence();
    if (atomicAdd(state + 1, 1ull) == gridDim.x - 1) {
      state[1] = 0ull;
      state[0] = step + 1ull;
      __threadfence();
    }
  }
}

// The channel-mapped draw of a compact tensor [rows, c] whose channel j is channel layout[j] of a full-width tensor
// [rows, cfull]: element (row, j) takes the uniform of full-width element f = row * cfull + layout[j], i.e. component
// f & 3 of Philox block f >> 2 at the same step and stream, so the mask is the full-width mask gathered by the layout.
// A padding channel (layout[j] < 0) gets mask 0.  One Philox block per element: a compact Dropout is a head layer.
__global__ void __launch_bounds__(NT)
dropout_fwd_mapped_kernel(const float* __restrict__ x, int64_t n, int c, int cfull, const int32_t* __restrict__ layout,
                          float keep, uint2 key, uint32_t stream, unsigned long long* state, float* __restrict__ y,
                          uint8_t* __restrict__ mask) {
  __shared__ unsigned long long s_step;
  if (threadIdx.x == 0) s_step = __ldcg(state);
  __syncthreads();
  const unsigned long long step = s_step;
  for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < n; i += (int64_t)gridDim.x * NT) {
    const int64_t row = i / c;
    const int l = layout[i - row * c];
    float m = 0.f;
    if (l >= 0) {
      const int64_t f = row * cfull + l, g = f >> 2;
      const uint4 r = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), (uint32_t)step, stream), key);
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};
      m = floorf(__fadd_rn(keep, u01(w[f & 3])));
    }
    y[i] = __fmul_rn(__fdiv_rn(x[i], keep), m);
    mask[i] = (uint8_t)m;
  }
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(state + 1, 1ull) == gridDim.x - 1) {
      state[1] = 0ull;
      state[0] = step + 1ull;
      __threadfence();
    }
  }
}

__global__ void __launch_bounds__(NT)
dropout_bwd_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ mask, int64_t n, float keep, int accumulate,
                   float* __restrict__ dx) {
  for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < n; i += (int64_t)gridDim.x * NT) {
    const float v = __fdiv_rn(__fmul_rn(dy[i], (float)mask[i]), keep);
    dx[i] = accumulate ? __fadd_rn(dx[i], v) : v;
  }
}

unsigned grid_of(int64_t items) {
  int64_t g = (items + NT - 1) / NT;
  const int64_t cap = (int64_t)PF_NUM_SMS * 8;
  if (g > cap) g = cap;
  return (unsigned)(g < 1 ? 1 : g);
}

}  // namespace

int pf_dropout_fwd(const float* x_dev, int64_t n, float keep_prob, uint32_t seed, uint32_t rank, uint32_t stream_id,
                   uint64_t* state_dev, float* y_dev, uint8_t* mask_dev, void* stream) {
  PF_REQUIRE(n > 0 && x_dev && y_dev && mask_dev && state_dev, "pf_dropout_fwd: bad arguments");
  PF_REQUIRE(keep_prob > 0.f && keep_prob <= 1.f, "pf_dropout_fwd: keep_prob must be in (0, 1]");
  PF_REQUIRE(((uintptr_t)state_dev & 7) == 0, "pf_dropout_fwd: state must be 8-byte aligned");
  const bool vec = (n & 3) == 0 && (((uintptr_t)x_dev | (uintptr_t)y_dev) & 15) == 0 && ((uintptr_t)mask_dev & 3) == 0;
  auto* st = reinterpret_cast<unsigned long long*>(state_dev);
  if (vec)
    dropout_fwd_kernel<true><<<grid_of(n >> 2), NT, 0, (cudaStream_t)stream>>>(x_dev, n, keep_prob, make_uint2(seed, rank),
                                                                               stream_id, st, y_dev, mask_dev);
  else
    dropout_fwd_kernel<false><<<grid_of((n + 3) >> 2), NT, 0, (cudaStream_t)stream>>>(x_dev, n, keep_prob,
                                                                                      make_uint2(seed, rank), stream_id, st,
                                                                                      y_dev, mask_dev);
  PF_CHECK_LAUNCH("pf_dropout_fwd");
  return PF_OK;
}

int pf_dropout_fwd_mapped(const float* x_dev, int64_t n, float keep_prob, uint32_t seed, uint32_t rank,
                          uint32_t stream_id, const int32_t* layout_dev, int c, int cfull, uint64_t* state_dev,
                          float* y_dev, uint8_t* mask_dev, void* stream) {
  if (!layout_dev)
    return pf_dropout_fwd(x_dev, n, keep_prob, seed, rank, stream_id, state_dev, y_dev, mask_dev, stream);
  PF_REQUIRE(n > 0 && x_dev && y_dev && mask_dev && state_dev, "pf_dropout_fwd_mapped: bad arguments");
  PF_REQUIRE(keep_prob > 0.f && keep_prob <= 1.f, "pf_dropout_fwd_mapped: keep_prob must be in (0, 1]");
  PF_REQUIRE(((uintptr_t)state_dev & 7) == 0, "pf_dropout_fwd_mapped: state must be 8-byte aligned");
  PF_REQUIRE(c > 0 && c <= cfull && n % c == 0, "pf_dropout_fwd_mapped: need 0 < c <= cfull and n % c == 0");
  dropout_fwd_mapped_kernel<<<grid_of(n), NT, 0, (cudaStream_t)stream>>>(x_dev, n, c, cfull, layout_dev, keep_prob,
                                                                        make_uint2(seed, rank), stream_id,
                                                                        reinterpret_cast<unsigned long long*>(state_dev),
                                                                        y_dev, mask_dev);
  PF_CHECK_LAUNCH("pf_dropout_fwd_mapped");
  return PF_OK;
}

int pf_dropout_bwd(const float* dy_dev, const uint8_t* mask_dev, int64_t n, float keep_prob, int accumulate, float* dx_dev,
                   void* stream) {
  PF_REQUIRE(n > 0 && dy_dev && mask_dev && dx_dev, "pf_dropout_bwd: bad arguments");
  PF_REQUIRE(keep_prob > 0.f && keep_prob <= 1.f, "pf_dropout_bwd: keep_prob must be in (0, 1]");
  dropout_bwd_kernel<<<grid_of(n), NT, 0, (cudaStream_t)stream>>>(dy_dev, mask_dev, n, keep_prob, accumulate, dx_dev);
  PF_CHECK_LAUNCH("pf_dropout_bwd");
  return PF_OK;
}
