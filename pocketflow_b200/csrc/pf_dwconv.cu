// pf_dwconv.cu — depthwise convolution (depth multiplier 1) forward / dgrad / wgrad, NHWC x [R,S,C,1].
//
// slim.separable_conv2d(num_outputs=None) of MobileNet-v1
// (/root/reference/utils/external/mobilenet_v1.py:273-280; op type DepthwiseConv2dNative, which the
// quantizers re-create on the quantized weight, learners/uniform_quantization/utils.py:92-104).
// 2*R*S FLOP per output element against >= 8 bytes of traffic: an HBM-bound kernel (SURVEY §8 a4:
// "depthwise is bandwidth-bound"), so: one thread per (pixel, 4 channels), 128-bit loads of the
// R*S taps (neighbouring taps hit L1/L2), no tensor cores.
#include <stdlib.h>

#include "pf_common.cuh"

namespace {
constexpr int NT = 256;

struct DwGeom {
  int N, H, W, C, R, S, P, Q, sh, sw, pt, pl;
};

__global__ void __launch_bounds__(NT)
dw_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, DwGeom g, float* __restrict__ y) {
  const int C4 = g.C >> 2;
  const int64_t total = (int64_t)g.N * g.P * g.Q * C4;
  const int64_t stride = (int64_t)gridDim.x * NT;
  for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < total; i += stride) {
    const int c = (int)(i % C4) << 2;
    int64_t t = i / C4;
    const int ow = (int)(t % g.Q); t /= g.Q;
    const int oh = (int)(t % g.P);
    const int n = (int)(t / g.P);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = 0; r < g.R; ++r) {
      const int ih = oh * g.sh - g.pt + r;
      if (ih < 0 || ih >= g.H) continue;
      for (int s = 0; s < g.S; ++s) {
        const int iw = ow * g.sw - g.pl + s;
        if (iw < 0 || iw >= g.W) continue;
        const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * g.H + ih) * g.W + iw) * g.C + c));
        const float4 wv = __ldg(reinterpret_cast<const float4*>(w + ((size_t)r * g.S + s) * g.C + c));
        acc.x = fmaf(xv.x, wv.x, acc.x); acc.y = fmaf(xv.y, wv.y, acc.y);
        acc.z = fmaf(xv.z, wv.z, acc.z); acc.w = fmaf(xv.w, wv.w, acc.w);
      }
    }
    pf_st_stream(y + (i << 2), acc);
  }
}

// dx[n,ih,iw,c] (+)= sum over taps of dy[n,oh,ow,c] * w[r,s,c] with oh*sh - pt + r == ih
__global__ void __launch_bounds__(NT)
dw_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, DwGeom g, int accumulate,
                float* __restrict__ dx) {
  const int C4 = g.C >> 2;
  const int64_t total = (int64_t)g.N * g.H * g.W * C4;
  const int64_t stride = (int64_t)gridDim.x * NT;
  for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < total; i += stride) {
    const int c = (int)(i % C4) << 2;
    int64_t t = i / C4;
    const int iw = (int)(t % g.W); t /= g.W;
    const int ih = (int)(t % g.H);
    const int n = (int)(t / g.H);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = 0; r < g.R; ++r) {
      const int th = ih + g.pt - r;
      if (th < 0 || th % g.sh) continue;
      const int oh = th / g.sh;
      if (oh >= g.P) continue;
      for (int s = 0; s < g.S; ++s) {
        const int tw = iw + g.pl - s;
        if (tw < 0 || tw % g.sw) continue;
        const int ow = tw / g.sw;
        if (ow >= g.Q) continue;
        const float4 dv = __ldg(reinterpret_cast<const float4*>(dy + (((size_t)n * g.P + oh) * g.Q + ow) * g.C + c));
        const float4 wv = __ldg(reinterpret_cast<const float4*>(w + ((size_t)r * g.S + s) * g.C + c));
        acc.x = fmaf(dv.x, wv.x, acc.x); acc.y = fmaf(dv.y, wv.y, acc.y);
        acc.z = fmaf(dv.z, wv.z, acc.z); acc.w = fmaf(dv.w, wv.w, acc.w);
      }
    }
    float* p = dx + (i << 2);
    if (accumulate) {
      const float4 o = *reinterpret_cast<const float4*>(p);
      acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
    }
    pf_st_stream(p, acc);
  }
}

// dw[r,s,c] = sum over output pixels of x[n, oh*sh-pt+r, ow*sw-pl+s, c] * dy[n,oh,ow,c]
// grid: (channel tiles of 128, pixel splits); thread = 4 channels x all taps (R*S <= 9) over a pixel
// stride; partials [split][R*S][C] -> fixed-order final reduction (deterministic).
constexpr int kMaxTaps = 9;
__global__ void __launch_bounds__(NT)
dw_wgrad_partial_kernel(const float* __restrict__ x, const float* __restrict__ dy, DwGeom g, int pix_per_split,
                        float* __restrict__ part) {
  __shared__ float sh[NT * 4];
  const int taps = g.R * g.S;
  const int c0 = blockIdx.x * 128;
  const int tc = min(128, g.C - c0);
  const int nvec = tc >> 2, nty = NT / nvec;
  const int tx = threadIdx.x % nvec, ty = threadIdx.x / nvec;
  const int npix = g.N * g.P * g.Q;
  const int p0 = blockIdx.y * pix_per_split, p1 = min(npix, p0 + pix_per_split);
  float acc[kMaxTaps][4];
#pragma unroll
  for (int t = 0; t < kMaxTaps; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;
  const int c = c0 + tx * 4;
  if (ty < nty) {
    for (int p = p0 + ty; p < p1; p += nty) {
      const int pq = g.P * g.Q;
      const int n = p / pq;
      const int rem = p - n * pq;
      const int oh = rem / g.Q, ow = rem - oh * g.Q;
      const float4 dv = pf_ld_stream(dy + (size_t)p * g.C + c);
#pragma unroll
      for (int t = 0; t < kMaxTaps; ++t) {
        if (t < taps) {
          const int r = t / g.S, s = t - r * g.S;
          const int ih = oh * g.sh - g.pt + r, iw = ow * g.sw - g.pl + s;
          if (ih >= 0 && ih < g.H && iw >= 0 && iw < g.W) {
            const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * g.H + ih) * g.W + iw) * g.C + c));
            acc[t][0] = fmaf(xv.x, dv.x, acc[t][0]); acc[t][1] = fmaf(xv.y, dv.y, acc[t][1]);
            acc[t][2] = fmaf(xv.z, dv.z, acc[t][2]); acc[t][3] = fmaf(xv.w, dv.w, acc[t][3]);
          }
        }
      }
    }
  }
  // combine over ty per tap, fixed order
  for (int t = 0; t < taps; ++t) {
    __syncthreads();
    if (ty < nty) {
      float* a = &sh[(ty * nvec + tx) * 4];
      a[0] = acc[t][0]; a[1] = acc[t][1]; a[2] = acc[t][2]; a[3] = acc[t][3];
    }
    __syncthreads();
    for (int cc = threadIdx.x; cc < tc; cc += NT) {
      float s = 0.f;
      for (int y = 0; y < nty; ++y) s += sh[(y * nvec + (cc >> 2)) * 4 + (cc & 3)];
      part[((size_t)blockIdx.y * taps + t) * g.C + c0 + cc] = s;
    }
  }
}

__global__ void __launch_bounds__(NT)
dw_wgrad_final_kernel(const float* __restrict__ part, int n, int splits, float* __restrict__ dw) {
  const int i = blockIdx.x * NT + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int z = 0; z < splits; ++z) s += part[(size_t)z * n + i];
  dw[i] = (float)s;
}


// ---------------------------------------------------------------------------------------------------------------
// 3x3 specialisations (every depthwise layer of MobileNet-v1), stride ST in {1, 2}: taps unrolled with predicated
// loads (all nine in flight at once instead of a chain of data-dependent `continue`s), 32-bit index arithmetic, and
// the 9 x 4 filter values of the thread's channels hoisted into registers (256 threads per block is a multiple of
// C/4 for every power-of-two C <= 1024, so a thread's channels never change).  The generic kernels above ran the
// 13 depthwise layers at ~1 TB/s: 15.3 of the 32 ms of the MobileNet step.
template <int ST>
__global__ void __launch_bounds__(NT)
dw3x3_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, DwGeom g, float* __restrict__ y) {
  const uint32_t C4 = (uint32_t)(g.C >> 2);
  const uint32_t total = (uint32_t)g.N * g.P * g.Q * C4;
  const uint32_t stride = gridDim.x * NT;
  uint32_t i = blockIdx.x * NT + threadIdx.x;
  const int c = (int)((i % C4) << 2);
  float4 wv[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wv[t] = __ldg(reinterpret_cast<const float4*>(w + (size_t)t * g.C + c));
  for (; i < total; i += stride) {
    const uint32_t pix = i / C4;
    const uint32_t t1 = pix / (uint32_t)g.Q;
    const int ow = (int)(pix - t1 * (uint32_t)g.Q);
    const int n = (int)(t1 / (uint32_t)g.P);
    const int oh = (int)(t1 - (uint32_t)n * (uint32_t)g.P);
    const int ih0 = oh * ST - g.pt, iw0 = ow * ST - g.pl;
    const float* xn = x + (size_t)n * g.H * g.W * g.C + c;
    float4 xv[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int ih = ih0 + r, iw = iw0 + q;
        const bool ok = ih >= 0 && ih < g.H && iw >= 0 && iw < g.W;
        xv[r * 3 + q] = ok ? __ldg(reinterpret_cast<const float4*>(xn + ((size_t)ih * g.W + iw) * g.C)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int t = 0; t < 9; ++t) {     // same accumulation order as the generic kernel (taps ascending); skipped taps add 0*w
      acc.x = fmaf(xv[t].x, wv[t].x, acc.x); acc.y = fmaf(xv[t].y, wv[t].y, acc.y);
      acc.z = fmaf(xv[t].z, wv[t].z, acc.z); acc.w = fmaf(xv[t].w, wv[t].w, acc.w);
    }
    pf_st_stream(y + ((size_t)i << 2), acc);
  }
}

template <int ST>
__global__ void __launch_bounds__(NT)
dw3x3_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, DwGeom g, int accumulate,
                   float* __restrict__ dx) {
  const uint32_t C4 = (uint32_t)(g.C >> 2);
  const uint32_t total = (uint32_t)g.N * g.H * g.W * C4;
  const uint32_t stride = gridDim.x * NT;
  uint32_t i = blockIdx.x * NT + threadIdx.x;
  const int c = (int)((i % C4) << 2);
  float4 wv[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wv[t] = __ldg(reinterpret_cast<const float4*>(w + (size_t)t * g.C + c));
  for (; i < total; i += stride) {
    const uint32_t pix = i / C4;
    const uint32_t t1 = pix / (uint32_t)g.W;
    const int iw = (int)(pix - t1 * (uint32_t)g.W);
    const int n = (int)(t1 / (uint32_t)g.H);
    const int ih = (int)(t1 - (uint32_t)n * (uint32_t)g.H);
    const float* dn = dy + (size_t)n * g.P * g.Q * g.C + c;
    float4 dv[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int th = ih + g.pt - r, tw = iw + g.pl - q;
        bool ok = th >= 0 && tw >= 0;
        if (ST == 2) ok = ok && ((th | tw) & 1) == 0;
        const int oh = ST == 2 ? th >> 1 : th, ow = ST == 2 ? tw >> 1 : tw;
        ok = ok && oh < g.P && ow < g.Q;
        dv[r * 3 + q] = ok ? __ldg(reinterpret_cast<const float4*>(dn + ((size_t)oh * g.Q + ow) * g.C)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      acc.x = fmaf(dv[t].x, wv[t].x, acc.x); acc.y = fmaf(dv[t].y, wv[t].y, acc.y);
      acc.z = fmaf(dv[t].z, wv[t].z, acc.z); acc.w = fmaf(dv[t].w, wv[t].w, acc.w);
    }
    float* p = dx + ((size_t)i << 2);
    if (accumulate) {
      const float4 o = *reinterpret_cast<const float4*>(p);
      acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
    }
    pf_st_stream(p, acc);
  }
}

template <int ST>
__global__ void __launch_bounds__(NT)
dw3x3_wgrad_partial_kernel(const float* __restrict__ x, const float* __restrict__ dy, DwGeom g, int pix_per_split,
                           float* __restrict__ part) {
  __shared__ float sh[NT * 4];
  const int c0 = blockIdx.x * 128;
  const int tc = min(128, g.C - c0);
  const int nvec = tc >> 2, nty = NT / nvec;
  const int tx = threadIdx.x % nvec, ty = threadIdx.x / nvec;
  const uint32_t npix = (uint32_t)g.N * g.P * g.Q, pq = (uint32_t)g.P * g.Q;
  const uint32_t p0 = blockIdx.y * (uint32_t)pix_per_split, p1 = min(npix, p0 + (uint32_t)pix_per_split);
  float acc[9][4];
#pragma unroll
  for (int t = 0; t < 9; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;
  const int c = c0 + tx * 4;
  if (ty < nty) {
    for (uint32_t p = p0 + ty; p < p1; p += nty) {
      const uint32_t n = p / pq;
      const uint32_t rem = p - n * pq;
      const int oh = (int)(rem / (uint32_t)g.Q), ow = (int)(rem - (uint32_t)oh * g.Q);
      const int ih0 = oh * ST - g.pt, iw0 = ow * ST - g.pl;
      const float* xn = x + (size_t)n * g.H * g.W * g.C + c;
      const float4 dv = pf_ld_stream(dy + (size_t)p * g.C + c);
      float4 xv[9];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          const int ih = ih0 + r, iw = iw0 + q;
          const bool ok = ih >= 0 && ih < g.H && iw >= 0 && iw < g.W;
          xv[r * 3 + q] = ok ? __ldg(reinterpret_cast<const float4*>(xn + ((size_t)ih * g.W + iw) * g.C)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        acc[t][0] = fmaf(xv[t].x, dv.x, acc[t][0]); acc[t][1] = fmaf(xv[t].y, dv.y, acc[t][1]);
        acc[t][2] = fmaf(xv[t].z, dv.z, acc[t][2]); acc[t][3] = fmaf(xv[t].w, dv.w, acc[t][3]);
      }
    }
  }
  for (int t = 0; t < 9; ++t) {     // combine over ty per tap, fixed order
    __syncthreads();
    if (ty < nty) {
      float* a = &sh[(ty * nvec + tx) * 4];
      a[0] = acc[t][0]; a[1] = acc[t][1]; a[2] = acc[t][2]; a[3] = acc[t][3];
    }
    __syncthreads();
    for (int cc = threadIdx.x; cc < tc; cc += NT) {
      float s = 0.f;
      for (int y = 0; y < nty; ++y) s += sh[(y * nvec + (cc >> 2)) * 4 + (cc & 3)];
      part[((size_t)blockIdx.y * 9 + t) * g.C + c0 + cc] = s;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Stride-1 3x3, ROW-BLOCKED: a thread produces RB vertically adjacent outputs of its (column, 4 channels) and streams the
// RB + 2 input rows they share through registers — 3 (RB + 2) loads for RB outputs instead of 9 RB (RB = 4: 4.5 per
// output), with every row read once per thread.  The 9-loads-per-output form above moved ~3.4x the tensor through
// L2 -> SM (horizontal neighbours hit L1, the two vertical neighbours did not): 8.3 ms of MobileNet's 25 ms step against
// 2.4 ms of HBM time (profiles/r1_bench_mobilenet_cpg50_b256_final.json).  Same accumulation order per output as the
// kernels above (rows r ascending, columns q ascending) for fwd: bit-identical results.
constexpr int kRB = 4;

__global__ void __launch_bounds__(NT)
dw3x3s1_fwd_rows_kernel(const float* __restrict__ x, const float* __restrict__ w, DwGeom g, float* __restrict__ y) {
  const uint32_t C4 = (uint32_t)(g.C >> 2), PB = (uint32_t)(g.P + kRB - 1) / kRB;
  const uint32_t total = (uint32_t)g.N * PB * g.Q * C4;
  const uint32_t stride = gridDim.x * NT;
  uint32_t i = blockIdx.x * NT + threadIdx.x;
  const int c = (int)((i % C4) << 2);
  float4 wv[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wv[t] = __ldg(reinterpret_cast<const float4*>(w + (size_t)t * g.C + c));
  for (; i < total; i += stride) {
    const uint32_t pix = i / C4;
    const uint32_t t1 = pix / (uint32_t)g.Q;
    const int ow = (int)(pix - t1 * (uint32_t)g.Q);
    const int n = (int)(t1 / PB);
    const int oh0 = (int)(t1 - (uint32_t)n * PB) * kRB;
    const int ih0 = oh0 - g.pt, iw0 = ow - g.pl;
    const float* xn = x + (size_t)n * g.H * g.W * g.C + c;
    float4 acc[kRB];
#pragma unroll
    for (int j = 0; j < kRB; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int rr = 0; rr < kRB + 2; ++rr) {
      const int ih = ih0 + rr;
      const bool okh = ih >= 0 && ih < g.H;
      float4 xv[3];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int iw = iw0 + q;
        const bool ok = okh && iw >= 0 && iw < g.W;
        xv[q] = ok ? __ldg(reinterpret_cast<const float4*>(xn + ((size_t)ih * g.W + iw) * g.C)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int j = 0; j < kRB; ++j) {
        const int r = rr - j;
        if (r >= 0 && r < 3) {
#pragma unroll
          for (int q = 0; q < 3; ++q) {
            acc[j].x = fmaf(xv[q].x, wv[r * 3 + q].x, acc[j].x); acc[j].y = fmaf(xv[q].y, wv[r * 3 + q].y, acc[j].y);
            acc[j].z = fmaf(xv[q].z, wv[r * 3 + q].z, acc[j].z); acc[j].w = fmaf(xv[q].w, wv[r * 3 + q].w, acc[j].w);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kRB; ++j)
      if (oh0 + j < g.P) pf_st_stream(y + (((size_t)n * g.P + oh0 + j) * g.Q + ow) * g.C + c, acc[j]);
  }
}

// dx(ih, iw) = sum_{r,q} dy(ih + pt - r, iw + pl - q) w[r][q]: RB input rows per thread, the RB + 2 dy rows they read
// streamed in ascending order
__global__ void __launch_bounds__(NT)
dw3x3s1_dgrad_rows_kernel(const float* __restrict__ dy, const float* __restrict__ w, DwGeom g, int accumulate,
                          float* __restrict__ dx) {
  const uint32_t C4 = (uint32_t)(g.C >> 2), HB = (uint32_t)(g.H + kRB - 1) / kRB;
  const uint32_t total = (uint32_t)g.N * HB * g.W * C4;
  const uint32_t stride = gridDim.x * NT;
  uint32_t i = blockIdx.x * NT + threadIdx.x;
  const int c = (int)((i % C4) << 2);
  float4 wv[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wv[t] = __ldg(reinterpret_cast<const float4*>(w + (size_t)t * g.C + c));
  for (; i < total; i += stride) {
    const uint32_t pix = i / C4;
    const uint32_t t1 = pix / (uint32_t)g.W;
    const int iw = (int)(pix - t1 * (uint32_t)g.W);
    const int n = (int)(t1 / HB);
    const int ih0 = (int)(t1 - (uint32_t)n * HB) * kRB;
    const float* dn = dy + (size_t)n * g.P * g.Q * g.C + c;
    float4 acc[kRB];
#pragma unroll
    for (int j = 0; j < kRB; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int rr = 0; rr < kRB + 2; ++rr) {
      const int oh = ih0 + g.pt - 2 + rr;
      const bool okh = oh >= 0 && oh < g.P;
      float4 dv[3];                                  // dv[q] = dy(oh, iw + pl - q)
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int ow = iw + g.pl - q;
        const bool ok = okh && ow >= 0 && ow < g.Q;
        dv[q] = ok ? __ldg(reinterpret_cast<const float4*>(dn + ((size_t)oh * g.Q + ow) * g.C)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int j = 0; j < kRB; ++j) {
        const int r = j + 2 - rr;                    // oh = (ih0 + j) + pt - r
        if (r >= 0 && r < 3) {
#pragma unroll
          for (int q = 0; q < 3; ++q) {
            acc[j].x = fmaf(dv[q].x, wv[r * 3 + q].x, acc[j].x); acc[j].y = fmaf(dv[q].y, wv[r * 3 + q].y, acc[j].y);
            acc[j].z = fmaf(dv[q].z, wv[r * 3 + q].z, acc[j].z); acc[j].w = fmaf(dv[q].w, wv[r * 3 + q].w, acc[j].w);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kRB; ++j) {
      if (ih0 + j >= g.H) continue;
      float* p = dx + (((size_t)n * g.H + ih0 + j) * g.W + iw) * g.C + c;
      float4 a = acc[j];
      if (accumulate) {
        const float4 o = *reinterpret_cast<const float4*>(p);
        a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w;
      }
      pf_st_stream(p, a);
    }
  }
}

// dw[r,q,c] = sum over outputs of x(oh + r - pt, ow + q - pl) dy(oh, ow): work item = (image, block of RB output rows,
// column); the RB + 2 input rows are read once per item.  Items are split over blockIdx.y like the pixels above.
__global__ void __launch_bounds__(NT)
dw3x3s1_wgrad_rows_kernel(const float* __restrict__ x, const float* __restrict__ dy, DwGeom g, int items_per_split,
                          float* __restrict__ part) {
  __shared__ float sh[NT * 4];
  const int c0 = blockIdx.x * 128;
  const int tc = min(128, g.C - c0);
  const int nvec = tc >> 2, nty = NT / nvec;
  const int tx = threadIdx.x % nvec, ty = threadIdx.x / nvec;
  const uint32_t PB = (uint32_t)(g.P + kRB - 1) / kRB;
  const uint32_t nitems = (uint32_t)g.N * PB * g.Q;
  const uint32_t i0 = blockIdx.y * (uint32_t)items_per_split, i1 = min(nitems, i0 + (uint32_t)items_per_split);
  float acc[9][4];
#pragma unroll
  for (int t = 0; t < 9; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;
  const int c = c0 + tx * 4;
  if (ty < nty) {
    for (uint32_t it = i0 + ty; it < i1; it += nty) {
      const uint32_t t1 = it / (uint32_t)g.Q;
      const int ow = (int)(it - t1 * (uint32_t)g.Q);
      const int n = (int)(t1 / PB);
      const int oh0 = (int)(t1 - (uint32_t)n * PB) * kRB;
      const int ih0 = oh0 - g.pt, iw0 = ow - g.pl;
      const float* xn = x + (size_t)n * g.H * g.W * g.C + c;
      float4 dv[kRB];
#pragma unroll
      for (int j = 0; j < kRB; ++j)
        dv[j] = (oh0 + j < g.P) ? pf_ld_stream(dy + (((size_t)n * g.P + oh0 + j) * g.Q + ow) * g.C + c)
                                : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int rr = 0; rr < kRB + 2; ++rr) {
        const int ih = ih0 + rr;
        const bool okh = ih >= 0 && ih < g.H;
        float4 xv[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          const int iw = iw0 + q;
          const bool ok = okh && iw >= 0 && iw < g.W;
          xv[q] = ok ? __ldg(reinterpret_cast<const float4*>(xn + ((size_t)ih * g.W + iw) * g.C)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < kRB; ++j) {
          const int r = rr - j;
          if (r >= 0 && r < 3) {
#pragma unroll
            for (int q = 0; q < 3; ++q) {
              acc[r * 3 + q][0] = fmaf(xv[q].x, dv[j].x, acc[r * 3 + q][0]); acc[r * 3 + q][1] = fmaf(xv[q].y, dv[j].y, acc[r * 3 + q][1]);
              acc[r * 3 + q][2] = fmaf(xv[q].z, dv[j].z, acc[r * 3 + q][2]); acc[r * 3 + q][3] = fmaf(xv[q].w, dv[j].w, acc[r * 3 + q][3]);
            }
          }
        }
      }
    }
  }
  for (int t = 0; t < 9; ++t) {     // combine over ty per tap, fixed order
    __syncthreads();
    if (ty < nty) {
      float* a = &sh[(ty * nvec + tx) * 4];
      a[0] = acc[t][0]; a[1] = acc[t][1]; a[2] = acc[t][2]; a[3] = acc[t][3];
    }
    __syncthreads();
    for (int cc = threadIdx.x; cc < tc; cc += NT) {
      float s = 0.f;
      for (int y = 0; y < nty; ++y) s += sh[(y * nvec + (cc >> 2)) * 4 + (cc & 3)];
      part[((size_t)blockIdx.y * 9 + t) * g.C + c0 + cc] = s;
    }
  }
}

// Stride-2 3x3 dgrad, 2 x 2 input pixels per thread: the four pixels (2a + u, 2b + v) of a block read the SAME 2 x 2
// neighbourhood of dy — dy(a - 1 + d + PAD, b - 1 + e + PAD), d, e in {0, 1} — each through the taps its parity allows
// (r = u - PAD + 2 - 2d, q likewise; 1 + 2 + 2 + 4 = 9 tap uses in all).  4 loads for 4 outputs, where the
// one-pixel-per-thread kernel issued 9 predicated loads per output (1.5 ms for MobileNet's 4 strided layers, 1.1 TB/s).
template <int PAD>
__global__ void __launch_bounds__(NT)
dw3x3s2_dgrad_block_kernel(const float* __restrict__ dy, const float* __restrict__ w, DwGeom g, int accumulate,
                           float* __restrict__ dx) {
  const uint32_t C4 = (uint32_t)(g.C >> 2), HB = (uint32_t)(g.H + 1) >> 1, WB = (uint32_t)(g.W + 1) >> 1;
  const uint32_t total = (uint32_t)g.N * HB * WB * C4;
  const uint32_t stride = gridDim.x * NT;
  uint32_t i = blockIdx.x * NT + threadIdx.x;
  const int c = (int)((i % C4) << 2);
  float4 wv[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wv[t] = __ldg(reinterpret_cast<const float4*>(w + (size_t)t * g.C + c));
  for (; i < total; i += stride) {
    const uint32_t pix = i / C4;
    const uint32_t t1 = pix / WB;
    const int b = (int)(pix - t1 * WB);
    const int n = (int)(t1 / HB);
    const int a = (int)(t1 - (uint32_t)n * HB);
    const float* dn = dy + (size_t)n * g.P * g.Q * g.C + c;
    float4 dv[2][2];
#pragma unroll
    for (int d = 0; d < 2; ++d)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int oh = a - 1 + d + PAD, ow = b - 1 + e + PAD;
        const bool ok = oh >= 0 && oh < g.P && ow >= 0 && ow < g.Q;
        dv[d][e] = ok ? __ldg(reinterpret_cast<const float4*>(dn + ((size_t)oh * g.Q + ow) * g.C)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
      for (int v = 0; v < 2; ++v) {
        const int ih = 2 * a + u, iw = 2 * b + v;
        if (ih >= g.H || iw >= g.W) continue;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int d = 0; d < 2; ++d) {
          const int r = u - PAD + 2 - 2 * d;
          if (r < 0 || r > 2) continue;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int q = v - PAD + 2 - 2 * e;
            if (q < 0 || q > 2) continue;
            acc.x = fmaf(dv[d][e].x, wv[r * 3 + q].x, acc.x); acc.y = fmaf(dv[d][e].y, wv[r * 3 + q].y, acc.y);
            acc.z = fmaf(dv[d][e].z, wv[r * 3 + q].z, acc.z); acc.w = fmaf(dv[d][e].w, wv[r * 3 + q].w, acc.w);
          }
        }
        float* p = dx + (((size_t)n * g.H + ih) * g.W + iw) * g.C + c;
        if (accumulate) {
          const float4 o = *reinterpret_cast<const float4*>(p);
          acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
        }
        pf_st_stream(p, acc);
      }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// u8 forward of the integer inference model (pf_dwconv_u8_fwd): activation and weights are the uniform quantizers'
// unsigned levels, one byte each, so one 128-bit load holds 16 channels of a pixel and a thread works on 16 channels.
// Per output, S = sum_taps q_a q_w and J = sum_taps q_a are exact integers (S <= 9 * 255^2 < 2^20, J <= 9 * 255 < 2^12)
// and share one 32-bit accumulator, S in bits 0..19 and J in bits 20..31; the affine epilogue is the only rounding:
//   y = fma(S, e1, J * e2),   e1 = (alpha_c * (1 / k_w)) * s_a,   e2 = beta_c * s_a,   s_a = alpha_a / k_a (header)
// (the u8 tensor-core convolution's epilogue with weight centre 0).  A header with nplanes != 1 makes s_a NaN.
struct DwU8Epi {
  const float* alpha;      // weight bucket scales: [C] with per_channel, else [1]
  const float* beta;
  const pf_tc_act_hdr* hdr;
  int per_channel;
  float rk;                // 1 / (2^bits - 1)
};

constexpr int kU8Ch = 16;                 // channels per thread
constexpr uint32_t kJOne = 1u << 20;      // J's unit in the shared accumulator
constexpr int kU8RB = 2;                  // output rows per item of the 3 x 3 kernel
constexpr int kU8NT = 128, kU8MinBlocks = 3;   // <= 168 registers: 12 warps per SM

// the 16 (S, J) accumulators of one output pixel through the epilogue, as four streaming float4 stores
__device__ __forceinline__ void dw_u8_store(const uint32_t (&acc)[kU8Ch], const DwU8Epi& e, float a_s, int c,
                                            float* __restrict__ out) {
#pragma unroll
  for (int v = 0; v < kU8Ch / 4; ++v) {
    float4 al, be;
    if (e.per_channel) {
      al = __ldg(reinterpret_cast<const float4*>(e.alpha + c + 4 * v));
      be = __ldg(reinterpret_cast<const float4*>(e.beta + c + 4 * v));
    } else {
      const float a0 = __ldg(e.alpha), b0 = __ldg(e.beta);
      al = make_float4(a0, a0, a0, a0);
      be = make_float4(b0, b0, b0, b0);
    }
    const float a4[4] = {al.x, al.y, al.z, al.w}, b4[4] = {be.x, be.y, be.z, be.w};
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t t = acc[4 * v + k];
      const float e1 = (a4[k] * e.rk) * a_s, e2 = b4[k] * a_s;
      o[k] = fmaf((float)(t & (kJOne - 1)), e1, (float)(t >> 20) * e2);
    }
    pf_st_stream(out + 4 * v, make_float4(o[0], o[1], o[2], o[3]));
  }
}

// 16 channels of three horizontally adjacent taps (a, b, c: one uint4 each) regrouped per channel: byte q of out[k] is
// tap q of channel k (byte 3 is a copy of byte 0, for the caller to mask or multiply by a zero weight byte)
__device__ __forceinline__ void dw_u8_taps3(const uint4& a, const uint4& b, const uint4& c, uint32_t (&out)[kU8Ch]) {
  const uint32_t av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w}, cv[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t lo = __byte_perm(av[i], bv[i], 0x5140), hi = __byte_perm(av[i], bv[i], 0x7362);
    out[4 * i + 0] = __byte_perm(lo, cv[i], 0x0410);
    out[4 * i + 1] = __byte_perm(lo, cv[i], 0x0532);
    out[4 * i + 2] = __byte_perm(hi, cv[i], 0x0610);
    out[4 * i + 3] = __byte_perm(hi, cv[i], 0x0732);
  }
}

// Items are (image, block of RB output rows, column, 16 channels), in a grid-stride loop whose stride is a multiple of
// C / 16, so a thread's channels never change and its 3 x 16 packed weight words (byte q = w[r][q][c], byte 3 = 0) are
// formed once.  An item streams the (RB - 1) * ST + 3 input rows its outputs share, row-blocked as the fp32 stride-1
// kernel above; each row's three taps of a channel sit in one word, so one dp4a with the weights of row r adds a row's
// three products to S, and one dp4a with 0x00010101 gives the row's level sum for J.
template <int ST, int RB>
__global__ void __launch_bounds__(kU8NT, kU8MinBlocks)
dw3x3_u8_fwd_rows_kernel(const uint8_t* __restrict__ x, const uint8_t* __restrict__ w, DwU8Epi e, DwGeom g,
                         float* __restrict__ y) {
  const uint32_t C16 = (uint32_t)(g.C / kU8Ch), PB = (uint32_t)(g.P + RB - 1) / RB;
  const uint32_t total = (uint32_t)g.N * PB * g.Q * C16;
  const uint32_t lanes = (gridDim.x * kU8NT) / C16 * C16;
  const uint32_t tid = blockIdx.x * kU8NT + threadIdx.x;
  if (tid >= lanes) return;
  const int c = (int)(tid % C16) * kU8Ch;
  uint32_t wp[3][kU8Ch];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const uint8_t* wr = w + (size_t)(3 * r) * g.C + c;
    dw_u8_taps3(__ldg(reinterpret_cast<const uint4*>(wr)), __ldg(reinterpret_cast<const uint4*>(wr + g.C)),
                __ldg(reinterpret_cast<const uint4*>(wr + 2 * g.C)), wp[r]);
#pragma unroll
    for (int k = 0; k < kU8Ch; ++k) wp[r][k] &= 0x00ffffffu;
  }
  const float a_s = __ldg(&e.hdr->nplanes) == 1 ? __ldg(&e.hdr->scale) : __int_as_float(0x7fc00000);
  for (uint32_t i = tid; i < total; i += lanes) {
    const uint32_t pix = i / C16;
    const uint32_t t1 = pix / (uint32_t)g.Q;
    const int ow = (int)(pix - t1 * (uint32_t)g.Q);
    const int n = (int)(t1 / PB);
    const int oh0 = (int)(t1 - (uint32_t)n * PB) * RB;
    const int ih0 = oh0 * ST - g.pt, iw0 = ow * ST - g.pl;
    const uint8_t* xn = x + (size_t)n * g.H * g.W * g.C + c;
    uint32_t acc[RB][kU8Ch];
#pragma unroll
    for (int j = 0; j < RB; ++j)
#pragma unroll
      for (int k = 0; k < kU8Ch; ++k) acc[j][k] = 0u;
#pragma unroll
    for (int rr = 0; rr < (RB - 1) * ST + 3; ++rr) {
      const int ih = ih0 + rr;
      const bool okh = ih >= 0 && ih < g.H;
      uint4 xv[3];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int iw = iw0 + q;
        const bool ok = okh && iw >= 0 && iw < g.W;
        xv[q] = ok ? __ldg(reinterpret_cast<const uint4*>(xn + ((size_t)ih * g.W + iw) * g.C)) : make_uint4(0u, 0u, 0u, 0u);
      }
      uint32_t xp[kU8Ch];
      dw_u8_taps3(xv[0], xv[1], xv[2], xp);
#pragma unroll
      for (int k = 0; k < kU8Ch; ++k) {
        const uint32_t rs = __dp4a(xp[k], 0x00010101u, 0u) << 20;
#pragma unroll
        for (int j = 0; j < RB; ++j) {
          const int r = rr - j * ST;
          if (r >= 0 && r < 3) acc[j][k] = __dp4a(xp[k], wp[r][k], acc[j][k] + rs);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < RB; ++j)
      if (oh0 + j < g.P) dw_u8_store(acc[j], e, a_s, c, y + (((size_t)n * g.P + oh0 + j) * g.Q + ow) * g.C + c);
  }
}

// any other filter of <= kMaxTaps taps and either stride: one output pixel x 16 channels per item, tap by tap;
// q_a * (q_w + 2^20) adds the product to S and q_a to J in one multiply-add
__global__ void __launch_bounds__(kU8NT, kU8MinBlocks)
dw_u8_fwd_kernel(const uint8_t* __restrict__ x, const uint8_t* __restrict__ w, DwU8Epi e, DwGeom g,
                 float* __restrict__ y) {
  const uint32_t C16 = (uint32_t)(g.C / kU8Ch);
  const uint32_t total = (uint32_t)g.N * g.P * g.Q * C16;
  const uint32_t lanes = (gridDim.x * kU8NT) / C16 * C16;
  const uint32_t tid = blockIdx.x * kU8NT + threadIdx.x;
  if (tid >= lanes) return;
  const int c = (int)(tid % C16) * kU8Ch;
  const float a_s = __ldg(&e.hdr->nplanes) == 1 ? __ldg(&e.hdr->scale) : __int_as_float(0x7fc00000);
  for (uint32_t i = tid; i < total; i += lanes) {
    const uint32_t pix = i / C16;
    const uint32_t t1 = pix / (uint32_t)g.Q;
    const int ow = (int)(pix - t1 * (uint32_t)g.Q);
    const int n = (int)(t1 / (uint32_t)g.P);
    const int oh = (int)(t1 - (uint32_t)n * (uint32_t)g.P);
    const uint8_t* xn = x + (size_t)n * g.H * g.W * g.C + c;
    uint32_t acc[kU8Ch];
#pragma unroll
    for (int k = 0; k < kU8Ch; ++k) acc[k] = 0u;
    for (int r = 0; r < g.R; ++r) {
      const int ih = oh * g.sh - g.pt + r;
      if (ih < 0 || ih >= g.H) continue;
      for (int s = 0; s < g.S; ++s) {
        const int iw = ow * g.sw - g.pl + s;
        if (iw < 0 || iw >= g.W) continue;
        const uint4 xv = __ldg(reinterpret_cast<const uint4*>(xn + ((size_t)ih * g.W + iw) * g.C));
        const uint4 wv = __ldg(reinterpret_cast<const uint4*>(w + (size_t)(r * g.S + s) * g.C + c));
        const uint32_t xa[4] = {xv.x, xv.y, xv.z, xv.w}, wa[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
        for (int k = 0; k < kU8Ch; ++k) {
          const uint32_t qa = (xa[k >> 2] >> (8 * (k & 3))) & 0xffu, qw = (wa[k >> 2] >> (8 * (k & 3))) & 0xffu;
          acc[k] += qa * (qw + kJOne);
        }
      }
    }
    dw_u8_store(acc, e, a_s, c, y + (size_t)pix * g.C + c);
  }
}

inline bool dw_rows_enabled() {           // PF_DW_ROWS=0: the one-output-per-thread kernels everywhere (read per launch)
  const char* v = getenv("PF_DW_ROWS");
  return !(v && v[0] == '0');
}

int g_last_variant = 0;                   // pf_dwconv_last_variant: PF_DW_* of the most recent launch, 0 = none yet
inline bool dw_rows(const DwGeom& g) {   // the row-blocked stride-1 kernels
  return dw_rows_enabled() && g.sh == 1 && g.sw == 1 && g.P >= kRB && g.H >= kRB;
}

inline bool dw_is3x3(const DwGeom& g) {
  const int c4 = g.C >> 2;
  return g.R == 3 && g.S == 3 && g.sh == g.sw && (g.sh == 1 || g.sh == 2) && c4 > 0 && (NT % c4) == 0 &&
         (int64_t)g.N * g.H * g.W * c4 < (1ll << 31) && (int64_t)g.N * g.P * g.Q * c4 < (1ll << 31);
}

int dw_geom(const pf_conv_desc* d, DwGeom* g, const char* who) {
  PF_REQUIRE(d != nullptr, "%s: null descriptor", who);
  PF_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0 && d->c > 0 && d->r > 0 && d->s > 0 && d->p > 0 && d->q > 0 &&
                 d->stride_h > 0 && d->stride_w > 0 && d->pad_t >= 0 && d->pad_l >= 0,
             "%s: non-positive dimension", who);
  PF_REQUIRE((d->c & 3) == 0 && d->k == d->c, "%s: depthwise needs C %% 4 == 0 and k == c (depth multiplier 1)", who);
  PF_REQUIRE(d->r * d->s <= kMaxTaps, "%s: at most %d taps", who, kMaxTaps);
  *g = DwGeom{d->n, d->h, d->w, d->c, d->r, d->s, d->p, d->q, d->stride_h, d->stride_w, d->pad_t, d->pad_l};
  return PF_OK;
}

inline unsigned dw_grid(int64_t items) {
  int64_t want = (items + NT - 1) / NT;
  const int64_t cap = (int64_t)PF_NUM_SMS * 8;
  if (want < 1) want = 1;
  return (unsigned)(want < cap ? want : cap);
}

inline int dw_splits(const DwGeom& g, int* pps) {
  const int npix = g.N * g.P * g.Q;
  const int ctiles = (g.C + 127) / 128;
  int splits = (4 * PF_NUM_SMS + ctiles - 1) / ctiles;
  const int max_by_pix = (npix + 63) / 64;
  if (splits > max_by_pix) splits = max_by_pix;
  if (splits > PF_DWCONV_MAX_SPLITS) splits = PF_DWCONV_MAX_SPLITS;
  if (splits < 1) splits = 1;
  *pps = (npix + splits - 1) / splits;
  return (npix + *pps - 1) / *pps;
}
}  // namespace

extern "C" {

int pf_dwconv_fwd(const pf_conv_desc* d, const float* x_dev, const float* w_dev, float* y_dev, void* stream) {
  DwGeom g;
  int rc = dw_geom(d, &g, "pf_dwconv_fwd");
  if (rc) return rc;
  PF_REQUIRE(x_dev && w_dev && y_dev, "pf_dwconv_fwd: null pointer");
  const unsigned grid = dw_grid((int64_t)g.N * g.P * g.Q * (g.C >> 2));
  if (dw_is3x3(g) && dw_rows(g)) {
    g_last_variant = PF_DW_FWD_ROWS;
    dw3x3s1_fwd_rows_kernel<<<dw_grid((int64_t)g.N * ((g.P + kRB - 1) / kRB) * g.Q * (g.C >> 2)), NT, 0, (cudaStream_t)stream>>>(
        x_dev, w_dev, g, y_dev);
  } else if (dw_is3x3(g) && g.sh == 1) {
    g_last_variant = PF_DW_FWD_3X3_S1;
    dw3x3_fwd_kernel<1><<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, w_dev, g, y_dev);
  } else if (dw_is3x3(g)) {
    g_last_variant = PF_DW_FWD_3X3_S2;
    dw3x3_fwd_kernel<2><<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, w_dev, g, y_dev);
  } else {
    g_last_variant = PF_DW_FWD_GENERIC;
    dw_fwd_kernel<<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, w_dev, g, y_dev);
  }
  PF_CHECK_LAUNCH("pf_dwconv_fwd");
  return PF_OK;
}

int pf_dwconv_dgrad(const pf_conv_desc* d, const float* dy_dev, const float* w_dev, int accumulate, float* dx_dev,
                    void* stream) {
  DwGeom g;
  int rc = dw_geom(d, &g, "pf_dwconv_dgrad");
  if (rc) return rc;
  PF_REQUIRE(dy_dev && w_dev && dx_dev, "pf_dwconv_dgrad: null pointer");
  const unsigned grid = dw_grid((int64_t)g.N * g.H * g.W * (g.C >> 2));
  if (dw_is3x3(g) && dw_rows(g)) {
    g_last_variant = PF_DW_DGRAD_ROWS;
    dw3x3s1_dgrad_rows_kernel<<<dw_grid((int64_t)g.N * ((g.H + kRB - 1) / kRB) * g.W * (g.C >> 2)), NT, 0, (cudaStream_t)stream>>>(
        dy_dev, w_dev, g, accumulate, dx_dev);
  } else if (dw_is3x3(g) && g.sh == 1) {
    g_last_variant = PF_DW_DGRAD_3X3_S1;
    dw3x3_dgrad_kernel<1><<<grid, NT, 0, (cudaStream_t)stream>>>(dy_dev, w_dev, g, accumulate, dx_dev);
  } else if (dw_is3x3(g) && g.pt == g.pl && g.pt <= 1 && dw_rows_enabled()) {
    const unsigned gb = dw_grid((int64_t)g.N * ((g.H + 1) / 2) * ((g.W + 1) / 2) * (g.C >> 2));
    g_last_variant = g.pt == 0 ? PF_DW_DGRAD_BLOCK_P0 : PF_DW_DGRAD_BLOCK_P1;
    if (g.pt == 0) dw3x3s2_dgrad_block_kernel<0><<<gb, NT, 0, (cudaStream_t)stream>>>(dy_dev, w_dev, g, accumulate, dx_dev);
    else dw3x3s2_dgrad_block_kernel<1><<<gb, NT, 0, (cudaStream_t)stream>>>(dy_dev, w_dev, g, accumulate, dx_dev);
  } else if (dw_is3x3(g)) {
    g_last_variant = PF_DW_DGRAD_3X3_S2;
    dw3x3_dgrad_kernel<2><<<grid, NT, 0, (cudaStream_t)stream>>>(dy_dev, w_dev, g, accumulate, dx_dev);
  } else {
    g_last_variant = PF_DW_DGRAD_GENERIC;
    dw_dgrad_kernel<<<grid, NT, 0, (cudaStream_t)stream>>>(dy_dev, w_dev, g, accumulate, dx_dev);
  }
  PF_CHECK_LAUNCH("pf_dwconv_dgrad");
  return PF_OK;
}

int64_t pf_dwconv_wgrad_workspace_bytes(const pf_conv_desc* d) {
  DwGeom g;
  if (!d || dw_geom(d, &g, "pf_dwconv_wgrad_workspace_bytes")) return 0;
  int pps;
  const int splits = dw_splits(g, &pps);
  return (int64_t)splits * g.R * g.S * g.C * 4;
}

int pf_dwconv_wgrad(const pf_conv_desc* d, const float* x_dev, const float* dy_dev, float* ws_dev, float* dw_dev,
                    void* stream) {
  DwGeom g;
  int rc = dw_geom(d, &g, "pf_dwconv_wgrad");
  if (rc) return rc;
  PF_REQUIRE(x_dev && dy_dev && ws_dev && dw_dev, "pf_dwconv_wgrad: null pointer");
  int pps;
  const int splits = dw_splits(g, &pps);
  dim3 grid((g.C + 127) / 128, splits);
  cudaStream_t st = (cudaStream_t)stream;
  if (dw_is3x3(g) && dw_rows(g)) {
    // same number of splits, over (image, row block, column) items instead of pixels
    const int nitems = g.N * ((g.P + kRB - 1) / kRB) * g.Q;
    const int ips = (nitems + splits - 1) / splits;
    g_last_variant = PF_DW_WGRAD_ROWS;
    dw3x3s1_wgrad_rows_kernel<<<grid, NT, 0, st>>>(x_dev, dy_dev, g, ips, ws_dev);
  } else if (dw_is3x3(g) && g.sh == 1) {
    g_last_variant = PF_DW_WGRAD_3X3_S1;
    dw3x3_wgrad_partial_kernel<1><<<grid, NT, 0, st>>>(x_dev, dy_dev, g, pps, ws_dev);
  } else if (dw_is3x3(g)) {
    g_last_variant = PF_DW_WGRAD_3X3_S2;
    dw3x3_wgrad_partial_kernel<2><<<grid, NT, 0, st>>>(x_dev, dy_dev, g, pps, ws_dev);
  } else {
    g_last_variant = PF_DW_WGRAD_GENERIC;
    dw_wgrad_partial_kernel<<<grid, NT, 0, st>>>(x_dev, dy_dev, g, pps, ws_dev);
  }
  PF_CHECK_LAUNCH("pf_dwconv_wgrad/partial");
  const int n = g.R * g.S * g.C;
  dw_wgrad_final_kernel<<<(n + NT - 1) / NT, NT, 0, st>>>(ws_dev, n, splits, dw_dev);
  PF_CHECK_LAUNCH("pf_dwconv_wgrad/final");
  return PF_OK;
}

int pf_dwconv_last_variant(void) { return g_last_variant; }

int pf_dwconv_u8_supported(const pf_conv_desc* d) {
  if (!d || d->n <= 0 || d->h <= 0 || d->w <= 0 || d->c <= 0 || d->r <= 0 || d->s <= 0 || d->p <= 0 || d->q <= 0 ||
      d->pad_t < 0 || d->pad_l < 0)
    return 0;
  return d->k == d->c && d->c % kU8Ch == 0 && d->c <= 65536 && d->r * d->s <= kMaxTaps && (d->stride_h == 1 || d->stride_h == 2) &&
         (d->stride_w == 1 || d->stride_w == 2) && (int64_t)d->n * d->h * d->w * d->c < (1ll << 31) &&
         (int64_t)d->n * d->p * d->q * d->c < (1ll << 31);
}

int pf_dwconv_u8_fwd(const pf_conv_desc* d, const pf_tc_act* x, const pf_tc_wt* w, float* y_dev, void* stream) {
  const char* who = "pf_dwconv_u8_fwd";
  PF_REQUIRE(d && x && w && x->plane0 && x->hdr && w->plane0 && w->alpha && w->beta && y_dev, "%s: null pointer", who);
  PF_REQUIRE(x->plane1 == nullptr && w->plane1 == nullptr, "%s: u8 operands have one plane", who);
  PF_REQUIRE(w->bits >= 1 && w->bits <= 8, "%s: u8 weight levels need 1..8 bits", who);
  PF_REQUIRE(pf_dwconv_u8_supported(d),
             "%s: needs depth multiplier 1, C %% 16 == 0, at most %d taps, strides 1 or 2 and < 2^31 elements", who,
             kMaxTaps);
  PF_REQUIRE((((uintptr_t)x->plane0 | (uintptr_t)w->plane0 | (uintptr_t)y_dev) & 15) == 0 &&
                 (!w->per_channel || (((uintptr_t)w->alpha | (uintptr_t)w->beta) & 15) == 0) &&
                 ((uintptr_t)x->hdr & 7) == 0,
             "%s: 16-byte alignment required (per-channel scales: 16, header: 8)", who);
  const DwGeom g{d->n, d->h, d->w, d->c, d->r, d->s, d->p, d->q, d->stride_h, d->stride_w, d->pad_t, d->pad_l};
  const DwU8Epi e{w->alpha, w->beta, x->hdr, w->per_channel ? 1 : 0, 1.f / (float)((1 << w->bits) - 1)};
  const uint8_t* xl = reinterpret_cast<const uint8_t*>(x->plane0);
  const uint8_t* wl = reinterpret_cast<const uint8_t*>(w->plane0);
  const int64_t c16 = g.C / kU8Ch;
  cudaStream_t st = (cudaStream_t)stream;
  // at least C / 16 threads take items (the grid-stride loop keeps each thread on its channels)
  auto grid = [&](int64_t items) {
    const int64_t want = ((items > c16 ? items : c16) + kU8NT - 1) / kU8NT, cap = (int64_t)PF_NUM_SMS * 16;
    return (unsigned)(want < cap ? want : cap);
  };
  if (g.R == 3 && g.S == 3 && g.sh == g.sw && g.P >= kU8RB) {
    const int64_t items = (int64_t)g.N * ((g.P + kU8RB - 1) / kU8RB) * g.Q * c16;
    if (g.sh == 1) dw3x3_u8_fwd_rows_kernel<1, kU8RB><<<grid(items), kU8NT, 0, st>>>(xl, wl, e, g, y_dev);
    else dw3x3_u8_fwd_rows_kernel<2, kU8RB><<<grid(items), kU8NT, 0, st>>>(xl, wl, e, g, y_dev);
  } else {
    dw_u8_fwd_kernel<<<grid((int64_t)g.N * g.P * g.Q * c16), kU8NT, 0, st>>>(xl, wl, e, g, y_dev);
  }
  PF_CHECK_LAUNCH(who);
  return PF_OK;
}

}  // extern "C"
