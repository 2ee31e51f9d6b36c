// pf_compact.cu — channel gathers of the compact (channel-pruned) graph, and their backward (a channel scatter).
//
// A channel-pruned network runs at its pruned width (pocketflow_b200/compact.py): a convolution whose kernel has zero
// rows for some input channels reads a narrower copy of its input, `gather(x, nnzs)` of the reference's
// tools/conversion/export_chn_pruned_tflite_model.py.  Both kernels here produce that copy: NHWC viewed as [M, Cin] ->
// [M, Cout] through an index table idx[Cout] of input channels (idx < 0: a zero padding channel).
//  * gather_kernel<NO_BN>: a plain gather of fp32 or split-bf16 planes, to fp32 and / or planes.
//  * gather_kernel<BN_EVAL>: the inference-mode BN apply (+ ReLU / ReLU6) fused in front of the gather: every kept value
//    goes through the op chain of bn_apply_kernel (pf_nn.cu, rstd formed from the moving variance as there), so it is
//    bit-identical to pf_bn_apply_eval at full width followed by the gather, without the full-width tensor.
//  * gather_kernel<BN_TRAIN>: the same with the batch statistics of pf_bn_train_stats: `var` holds rstd.
//  * scatter_kernel: the backward of the gather, dx[m, idx[j]] (+)= dy[m, j].  It walks the FULL width through the
//    inverse table inv[Cin] (compact position of a full channel, -1: nobody gathered it), so every element of dx has
//    one writer: no atomics, and without `accumulate` the zeros of the dropped channels come from the same pass.
// One thread = 4 consecutive output channels of one row; when the 4 source channels are consecutive and 4-aligned the
// source is read with one 128-bit (fp32) / 64-bit (planes) load, otherwise element by element.  Planes are written with
// the split of pf_st_planes4, which is the split of pf_split_bf16.
#include "pf_common.cuh"

namespace {

constexpr int NT = 256;

enum { NO_BN = 0, BN_EVAL = 1, BN_TRAIN = 2 };

__device__ __forceinline__ float bf16_bits_to_float(uint16_t b) { return __uint_as_float((uint32_t)b << 16); }

template <int BN>
__global__ void __launch_bounds__(NT)
gather_kernel(const float* __restrict__ x, const uint16_t* __restrict__ x_hi, const uint16_t* __restrict__ x_lo,
              int64_t m, int cin, int cout, const int32_t* __restrict__ idx, const float* __restrict__ mean,
              const float* __restrict__ var, float eps, const float* __restrict__ gamma, const float* __restrict__ beta,
              int act, float* __restrict__ y, void* __restrict__ y_hi, void* __restrict__ y_lo) {
  const int groups = cout >> 2;
  const int64_t total = m * groups;
  const bool vec_ok = (cin & 3) == 0;
  for (int64_t g = (int64_t)blockIdx.x * NT + threadIdx.x; g < total; g += (int64_t)gridDim.x * NT) {
    const int64_t row = g / groups;
    const int j = (int)(g - row * groups) << 2;
    const int4 s = __ldg(reinterpret_cast<const int4*>(idx + j));
    const int si[4] = {s.x, s.y, s.z, s.w};
    const bool run = vec_ok && s.x >= 0 && (s.x & 3) == 0 && s.y == s.x + 1 && s.z == s.x + 2 && s.w == s.x + 3;
    float v[4];
    if (x_hi != nullptr) {
      // planes in: planes out are a copy of the source bits; fp32 out is hi + lo
      uint16_t h[4], l[4];
      if (run) {
        const uint2 a = __ldg(reinterpret_cast<const uint2*>(x_hi + row * cin + s.x));
        const uint2 b = __ldg(reinterpret_cast<const uint2*>(x_lo + row * cin + s.x));
        h[0] = a.x & 0xffffu; h[1] = a.x >> 16; h[2] = a.y & 0xffffu; h[3] = a.y >> 16;
        l[0] = b.x & 0xffffu; l[1] = b.x >> 16; l[2] = b.y & 0xffffu; l[3] = b.y >> 16;
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          h[k] = si[k] >= 0 ? __ldg(x_hi + row * cin + si[k]) : (uint16_t)0;
          l[k] = si[k] >= 0 ? __ldg(x_lo + row * cin + si[k]) : (uint16_t)0;
        }
      }
      if (y_hi) {
        uint2* ph = reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(y_hi) + row * cout + j);
        uint2* pl = reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(y_lo) + row * cout + j);
        *ph = make_uint2((uint32_t)h[0] | ((uint32_t)h[1] << 16), (uint32_t)h[2] | ((uint32_t)h[3] << 16));
        *pl = make_uint2((uint32_t)l[0] | ((uint32_t)l[1] << 16), (uint32_t)l[2] | ((uint32_t)l[3] << 16));
      }
      if (y) {
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = __fadd_rn(bf16_bits_to_float(h[k]), bf16_bits_to_float(l[k]));
        pf_st_stream(y + row * cout + j, make_float4(v[0], v[1], v[2], v[3]));
      }
      continue;
    }
    if (run) {
      const float4 a = pf_ld_stream(x + row * cin + s.x);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = si[k] >= 0 ? __ldg(x + row * cin + si[k]) : 0.f;
    }
    if (BN != NO_BN) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (si[k] < 0) { v[k] = 0.f; continue; }
        const float s2 = __ldg(var + si[k]);
        const float rs = BN == BN_EVAL ? __frsqrt_rn(__fadd_rn(s2, eps)) : s2;
        v[k] = pf_bn_act(v[k], __ldg(mean + si[k]), rs, __ldg(gamma + si[k]), __ldg(beta + si[k]), act);
      }
    }
    const float4 o = make_float4(v[0], v[1], v[2], v[3]);
    if (y) pf_st_stream(y + row * cout + j, o);
    if (y_hi) pf_st_planes4(y_hi, y_lo, row * cout + j, o);
  }
}

// One thread = 4 consecutive channels of one row of dx.  `run`: the 4 compact sources are consecutive and 4-aligned
// (one 128-bit load of dy).  With ACC a group nobody gathered is left alone (nothing to add) unless planes are wanted.
template <bool ACC>
__global__ void __launch_bounds__(NT)
scatter_kernel(const float* __restrict__ dy, int64_t m, int cin, int cout, const int32_t* __restrict__ inv,
               float* dx, void* __restrict__ dx_hi, void* __restrict__ dx_lo) {
  const int groups = cin >> 2;
  const int64_t total = m * groups;
  const bool vec_ok = (cout & 3) == 0;
  for (int64_t g = (int64_t)blockIdx.x * NT + threadIdx.x; g < total; g += (int64_t)gridDim.x * NT) {
    const int64_t row = g / groups;
    const int c = (int)(g - row * groups) << 2;
    const int4 s = __ldg(reinterpret_cast<const int4*>(inv + c));
    const int si[4] = {s.x, s.y, s.z, s.w};
    float v[4];
    if (vec_ok && s.x >= 0 && (s.x & 3) == 0 && s.y == s.x + 1 && s.z == s.x + 2 && s.w == s.x + 3) {
      const float4 a = pf_ld_stream(dy + row * cout + s.x);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    } else {
      if (ACC && dx_hi == nullptr && (s.x & s.y & s.z & s.w) < 0) continue;
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = si[k] >= 0 ? __ldg(dy + row * cout + si[k]) : 0.f;
    }
    float4 o = make_float4(v[0], v[1], v[2], v[3]);
    if (ACC) {
      const float4 p = pf_ld4(dx + row * cin + c);
      o = make_float4(__fadd_rn(p.x, o.x), __fadd_rn(p.y, o.y), __fadd_rn(p.z, o.z), __fadd_rn(p.w, o.w));
    }
    if (dx) pf_st_stream(dx + row * cin + c, o);
    if (dx_hi) pf_st_planes4(dx_hi, dx_lo, row * cin + c, o);
  }
}

unsigned gather_grid(int64_t total) {
  int64_t blocks = (total + NT - 1) / NT;
  const int64_t cap = (int64_t)PF_NUM_SMS * 16;
  if (blocks > cap) blocks = cap;
  return (unsigned)(blocks > 0 ? blocks : 1);
}

int check_common(const char* who, int64_t m, int cin, int cout, const int32_t* idx_dev, const float* y_dev,
                 const void* y_hi_dev, const void* y_lo_dev) {
  PF_REQUIRE(m > 0 && cin > 0 && cout > 0 && (cout & 3) == 0, "%s: bad shape (m > 0, cin > 0, cout a multiple of 4)", who);
  PF_REQUIRE(idx_dev != nullptr && ((uintptr_t)idx_dev & 15) == 0, "%s: the index table must be 16-byte aligned", who);
  PF_REQUIRE(y_dev || y_hi_dev, "%s: no output", who);
  PF_REQUIRE((y_hi_dev == nullptr) == (y_lo_dev == nullptr), "%s: planes come in pairs", who);
  PF_REQUIRE((((uintptr_t)y_hi_dev | (uintptr_t)y_lo_dev) & 7) == 0 && ((uintptr_t)y_dev & 15) == 0,
             "%s: fp32 output must be 16-byte and planes 8-byte aligned", who);
  return PF_OK;
}

}  // namespace

int pf_gather_channels(const float* x_dev, const void* x_hi_dev, const void* x_lo_dev, int64_t m, int cin, int cout,
                       const int32_t* idx_dev, float* y_dev, void* y_hi_dev, void* y_lo_dev, void* stream) {
  const char* who = "pf_gather_channels";
  int rc = check_common(who, m, cin, cout, idx_dev, y_dev, y_hi_dev, y_lo_dev);
  if (rc) return rc;
  PF_REQUIRE((x_dev != nullptr) != (x_hi_dev != nullptr), "%s: give the input as fp32 or as planes, not both", who);
  PF_REQUIRE((x_hi_dev == nullptr) == (x_lo_dev == nullptr), "%s: planes come in pairs", who);
  PF_REQUIRE((((uintptr_t)x_dev) & 15) == 0 && (((uintptr_t)x_hi_dev | (uintptr_t)x_lo_dev) & 7) == 0,
             "%s: fp32 input must be 16-byte and planes 8-byte aligned", who);
  gather_kernel<NO_BN><<<gather_grid(m * (cout >> 2)), NT, 0, (cudaStream_t)stream>>>(
      x_dev, (const uint16_t*)x_hi_dev, (const uint16_t*)x_lo_dev, m, cin, cout, idx_dev, nullptr, nullptr, 0.f, nullptr,
      nullptr, 0, y_dev, y_hi_dev, y_lo_dev);
  PF_CHECK_LAUNCH(who);
  return PF_OK;
}

int pf_bn_apply_eval_gather(const float* x_dev, int64_t m, int cin, const float* moving_mean_dev,
                            const float* moving_var_dev, float eps, const float* gamma_dev, const float* beta_dev, int act,
                            int cout, const int32_t* idx_dev, float* y_dev, void* y_hi_dev, void* y_lo_dev,
                            void* stream) {
  const char* who = "pf_bn_apply_eval_gather";
  int rc = check_common(who, m, cin, cout, idx_dev, y_dev, y_hi_dev, y_lo_dev);
  if (rc) return rc;
  PF_REQUIRE(eps >= 0.f, "%s: eps < 0", who);
  PF_REQUIRE(act >= 0 && act <= 2, "%s: act must be 0 (none), 1 (relu) or 2 (relu6)", who);
  PF_REQUIRE(x_dev && moving_mean_dev && moving_var_dev && gamma_dev && beta_dev, "%s: null pointer", who);
  PF_REQUIRE(((uintptr_t)x_dev & 15) == 0, "%s: fp32 input must be 16-byte aligned", who);
  gather_kernel<BN_EVAL><<<gather_grid(m * (cout >> 2)), NT, 0, (cudaStream_t)stream>>>(
      x_dev, nullptr, nullptr, m, cin, cout, idx_dev, moving_mean_dev, moving_var_dev, eps, gamma_dev, beta_dev, act,
      y_dev, y_hi_dev, y_lo_dev);
  PF_CHECK_LAUNCH(who);
  return PF_OK;
}

int pf_bn_apply_gather(const float* x_dev, int64_t m, int cin, const float* mean_dev, const float* rstd_dev,
                       const float* gamma_dev, const float* beta_dev, int act, int cout, const int32_t* idx_dev,
                       float* y_dev, void* y_hi_dev, void* y_lo_dev, void* stream) {
  const char* who = "pf_bn_apply_gather";
  int rc = check_common(who, m, cin, cout, idx_dev, y_dev, y_hi_dev, y_lo_dev);
  if (rc) return rc;
  PF_REQUIRE(act >= 0 && act <= 2, "%s: act must be 0 (none), 1 (relu) or 2 (relu6)", who);
  PF_REQUIRE(x_dev && mean_dev && rstd_dev && gamma_dev && beta_dev, "%s: null pointer", who);
  PF_REQUIRE(((uintptr_t)x_dev & 15) == 0, "%s: fp32 input must be 16-byte aligned", who);
  gather_kernel<BN_TRAIN><<<gather_grid(m * (cout >> 2)), NT, 0, (cudaStream_t)stream>>>(
      x_dev, nullptr, nullptr, m, cin, cout, idx_dev, mean_dev, rstd_dev, 0.f, gamma_dev, beta_dev, act, y_dev, y_hi_dev,
      y_lo_dev);
  PF_CHECK_LAUNCH(who);
  return PF_OK;
}

int pf_scatter_channels(const float* dy_dev, int64_t m, int cin, int cout, const int32_t* inv_dev, int accumulate,
                        float* dx_dev, void* dx_hi_dev, void* dx_lo_dev, void* stream) {
  const char* who = "pf_scatter_channels";
  PF_REQUIRE(m > 0 && cin > 0 && cout > 0 && (cin & 3) == 0, "%s: bad shape (m > 0, cout > 0, cin a multiple of 4)", who);
  PF_REQUIRE(dy_dev != nullptr && ((uintptr_t)dy_dev & 15) == 0, "%s: dy must be 16-byte aligned", who);
  PF_REQUIRE(inv_dev != nullptr && ((uintptr_t)inv_dev & 15) == 0, "%s: the inverse table must be 16-byte aligned", who);
  PF_REQUIRE(dx_dev || dx_hi_dev, "%s: no output", who);
  PF_REQUIRE(dx_dev || !accumulate, "%s: accumulate needs the fp32 dx", who);
  PF_REQUIRE((dx_hi_dev == nullptr) == (dx_lo_dev == nullptr), "%s: planes come in pairs", who);
  PF_REQUIRE((((uintptr_t)dx_hi_dev | (uintptr_t)dx_lo_dev) & 7) == 0 && ((uintptr_t)dx_dev & 15) == 0,
             "%s: fp32 output must be 16-byte and planes 8-byte aligned", who);
  const unsigned grid = gather_grid(m * (cin >> 2));
  if (accumulate)
    scatter_kernel<true><<<grid, NT, 0, (cudaStream_t)stream>>>(dy_dev, m, cin, cout, inv_dev, dx_dev, dx_hi_dev, dx_lo_dev);
  else
    scatter_kernel<false><<<grid, NT, 0, (cudaStream_t)stream>>>(dy_dev, m, cin, cout, inv_dev, dx_dev, dx_hi_dev, dx_lo_dev);
  PF_CHECK_LAUNCH(who);
  return PF_OK;
}
