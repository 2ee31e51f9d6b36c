// pf_conv.cu — fp32 implicit-GEMM convolution (forward, dgrad, wgrad) on the CUDA cores.
//
// This is the EXACT-fp32 conv path: it reproduces tf.nn.conv2d / tf.matmul in fp32
// (/root/reference/learners/uniform_quantization/utils.py:92-104 re-creates every conv on the
// fake-quantized weight; autodiff supplies dgrad/wgrad, learner.py:247) with fp32 FFMA
// accumulation, and is the on-device reference the tensor-core path (pf_conv_tc.cu) is checked against.
// It also covers the shapes the tensor-core path does not take (Cin=3 first layers, Cout=10/1001
// dense layers).  NHWC activations x HWIO kernels, so the weight is already the row-major
// [K = R*S*Cin, Cout] B operand and the output is the row-major [M = N*P*Q, Cout] C operand.
//
// One kernel template serves the three passes:
//   fwd  : M = N*P*Q,   Ng = Cout, K = R*S*Cin ;  A = im2col(x) gathered on the fly, B = w
//   dgrad: M = N*H*W,   Ng = Cin,  K = R*S*Cout;  A = gathered dy,                  B = w^T (HWOI)
//   wgrad: M = R*S*Cin, Ng = Cout, K = N*P*Q   ;  A = im2col(x)^T,                  B = dy  (split-K)
// Tile 128x64x16, 256 threads, 8x4 register tile per thread, register-staged double buffering.
#include "pf_common.cuh"

namespace {

constexpr int BM = 128, BN = 64, BK = 16, NT = 256;
constexpr int APAD = 4;

struct Geom {
  int N, H, W, C, K, R, S, P, Q, sh, sw, pt, pl;
};

enum { kFwd = 0, kDgrad = 1, kWgrad = 2 };

struct Epi {
  float* out;         // fwd: y ; dgrad: dx ; wgrad: partial workspace or dw
  const float* bias;  // fwd only, may be null
  int relu;           // fwd only
  int accumulate;     // dgrad: dx += ; wgrad (single split): unused
};

// ---- A operand: element (m, k) of the implicit matrix, 4 consecutive k (fwd/dgrad) or m (wgrad)
template <int MODE>
struct ALoader {
  const float* __restrict__ src;
  Geom g;
  int M, K;
};

__device__ __forceinline__ float4 ldg4_or_zero(const float* p, bool ok) {
  return ok ? __ldg(reinterpret_cast<const float4*>(p)) : make_float4(0.f, 0.f, 0.f, 0.f);
}

template <int MODE, bool VEC>
__global__ void __launch_bounds__(NT)
igemm_kernel(const float* __restrict__ asrc, const float* __restrict__ bsrc, Geom g, int M, int Ng,
             int K, int k_per_split, Epi ep) {
  __shared__ __align__(16) float As[2][BK][BM + APAD];
  __shared__ __align__(16) float Bs[2][BK][BN];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int kbeg = blockIdx.z * k_per_split;
  const int kend = min(K, kbeg + k_per_split);

  // ---------------- per-thread A-load coordinates
  // fwd/dgrad: 2 float4 along k: row = l/4, kvec = l%4 ; wgrad: 2 float4 along m: mvec = l%32, pix = l/32
  int a_row[2], a_kv[2];
  int a_n[2], a_y0[2], a_x0[2];  // fwd: (n, ih0, iw0); dgrad: (n, ih+pt, iw+pl); wgrad: (r, q, c) in y0,x0,n
  bool a_ok[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int l = tid + i * NT;
    if (MODE == kWgrad) {
      a_row[i] = (l & 31) * 4;  // m offset in tile
      a_kv[i] = l >> 5;         // pixel offset in k-tile
      const int m = m0 + a_row[i];
      a_ok[i] = m < M;
      const int rq = m / g.C;
      a_n[i] = m - rq * g.C;  // c
      a_y0[i] = rq / g.S;     // r
      a_x0[i] = rq - a_y0[i] * g.S;  // q
    } else {
      a_row[i] = l >> 2;
      a_kv[i] = (l & 3) * 4;
      const int m = m0 + a_row[i];
      a_ok[i] = m < M;
      const int hw = (MODE == kFwd) ? g.P * g.Q : g.H * g.W;
      const int wq = (MODE == kFwd) ? g.Q : g.W;
      const int n = m / hw;
      const int rem = m - n * hw;
      const int y = rem / wq, x = rem - y * wq;
      a_n[i] = n;
      if (MODE == kFwd) {
        a_y0[i] = y * g.sh - g.pt;
        a_x0[i] = x * g.sw - g.pl;
      } else {
        a_y0[i] = y + g.pt;
        a_x0[i] = x + g.pl;
      }
    }
  }
  // B: 1 float4: krow = tid/16, nvec = tid%16
  const int b_k = tid >> 4, b_n = (tid & 15) * 4;

  auto load_a = [&](int k0, float4* va) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (MODE == kWgrad) {
        const int pix = k0 + a_kv[i];
        if (a_ok[i] && pix < kend) {
          const int pq = g.P * g.Q;
          const int n = pix / pq;
          const int rem = pix - n * pq;
          const int oh = rem / g.Q, ow = rem - oh * g.Q;
          if (VEC) {
            const int ih = oh * g.sh - g.pt + a_y0[i], iw = ow * g.sw - g.pl + a_x0[i];
            const bool ok = ih >= 0 && ih < g.H && iw >= 0 && iw < g.W;
            const float4 t = ldg4_or_zero(asrc + (((size_t)n * g.H + ih) * g.W + iw) * g.C + a_n[i], ok);
            v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int m = m0 + a_row[i] + j;
              if (m < M) {
                const int rq = m / g.C, c = m - rq * g.C;
                const int r = rq / g.S, q = rq - r * g.S;
                const int ih = oh * g.sh - g.pt + r, iw = ow * g.sw - g.pl + q;
                if (ih >= 0 && ih < g.H && iw >= 0 && iw < g.W)
                  v[j] = __ldg(asrc + (((size_t)n * g.H + ih) * g.W + iw) * g.C + c);
              }
            }
          }
        }
      } else {
        const int CC = (MODE == kFwd) ? g.C : g.K;  // channels of the gathered tensor
        const int k = k0 + a_kv[i];
        if (a_ok[i] && k < kend) {
          if (VEC) {
            const int rq = k / CC, c = k - rq * CC;
            const int r = rq / g.S, q = rq - r * g.S;
            if (MODE == kFwd) {
              const int ih = a_y0[i] + r, iw = a_x0[i] + q;
              const bool ok = ih >= 0 && ih < g.H && iw >= 0 && iw < g.W;
              const float4 t = ldg4_or_zero(asrc + (((size_t)a_n[i] * g.H + ih) * g.W + iw) * g.C + c, ok);
              v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
            } else {
              const int th = a_y0[i] - r, tw = a_x0[i] - q;
              const int oh = th / g.sh, ow = tw / g.sw;
              const bool ok = th >= 0 && tw >= 0 && oh * g.sh == th && ow * g.sw == tw && oh < g.P && ow < g.Q;
              const float4 t = ldg4_or_zero(asrc + (((size_t)a_n[i] * g.P + oh) * g.Q + ow) * g.K + c, ok);
              v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int kk = k + j;
              if (kk < kend) {
                const int rq = kk / CC, c = kk - rq * CC;
                const int r = rq / g.S, q = rq - r * g.S;
                if (MODE == kFwd) {
                  const int ih = a_y0[i] + r, iw = a_x0[i] + q;
                  if (ih >= 0 && ih < g.H && iw >= 0 && iw < g.W)
                    v[j] = __ldg(asrc + (((size_t)a_n[i] * g.H + ih) * g.W + iw) * g.C + c);
                } else {
                  const int th = a_y0[i] - r, tw = a_x0[i] - q;
                  const int oh = th / g.sh, ow = tw / g.sw;
                  if (th >= 0 && tw >= 0 && oh * g.sh == th && ow * g.sw == tw && oh < g.P && ow < g.Q)
                    v[j] = __ldg(asrc + (((size_t)a_n[i] * g.P + oh) * g.Q + ow) * g.K + c);
                }
              }
            }
          }
        }
      }
      va[i] = make_float4(v[0], v[1], v[2], v[3]);
    }
  };
  auto load_b = [&](int k0) -> float4 {
    const int k = k0 + b_k, n = n0 + b_n;
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < kend) {
      const float* p = bsrc + (size_t)k * Ng + n;
      if (VEC) {
        if (n < Ng) t = __ldg(reinterpret_cast<const float4*>(p));
      } else {
        if (n + 0 < Ng) t.x = __ldg(p + 0);
        if (n + 1 < Ng) t.y = __ldg(p + 1);
        if (n + 2 < Ng) t.z = __ldg(p + 2);
        if (n + 3 < Ng) t.w = __ldg(p + 3);
      }
    }
    return t;
  };
  auto store_a = [&](int buf, const float4* va) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (MODE == kWgrad) {
        *reinterpret_cast<float4*>(&As[buf][a_kv[i]][a_row[i]]) = va[i];
      } else {
        As[buf][a_kv[i] + 0][a_row[i]] = va[i].x;
        As[buf][a_kv[i] + 1][a_row[i]] = va[i].y;
        As[buf][a_kv[i] + 2][a_row[i]] = va[i].z;
        As[buf][a_kv[i] + 3][a_row[i]] = va[i].w;
      }
    }
  };

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int tm = (tid >> 4) * 8, tn = (tid & 15) * 4;
  float4 va[2], vb;
  load_a(kbeg, va);
  vb = load_b(kbeg);
  store_a(0, va);
  *reinterpret_cast<float4*>(&Bs[0][b_k][b_n]) = vb;
  __syncthreads();
  int buf = 0;
  for (int k0 = kbeg; k0 < kend; k0 += BK) {
    const bool more = k0 + BK < kend;
    if (more) {
      load_a(k0 + BK, va);
      vb = load_b(k0 + BK);
    }
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][tm]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][tm + 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][kk][tn]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    if (more) {
      store_a(buf ^ 1, va);
      *reinterpret_cast<float4*>(&Bs[buf ^ 1][b_k][b_n]) = vb;
    }
    __syncthreads();
    buf ^= 1;
  }

  // ---------------- epilogue: C[m][n] row-major with leading dimension Ng
  float* out = ep.out + (MODE == kWgrad ? (size_t)blockIdx.z * M * Ng : 0);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + tm + i;
    if (m >= M) continue;
    const int n = n0 + tn;
    float v[4] = {acc[i][0], acc[i][1], acc[i][2], acc[i][3]};
    float* p = out + (size_t)m * Ng + n;
    if (MODE == kFwd) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (ep.bias && n + j < Ng) v[j] = __fadd_rn(v[j], __ldg(ep.bias + n + j));
        if (ep.relu) v[j] = fmaxf(v[j], 0.f);
      }
    }
    if (VEC && n + 3 < Ng) {
      float4 o = make_float4(v[0], v[1], v[2], v[3]);
      if (MODE == kDgrad && ep.accumulate) {
        const float4 old = *reinterpret_cast<const float4*>(p);
        o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w;
      }
      *reinterpret_cast<float4*>(p) = o;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n + j < Ng) p[j] = (MODE == kDgrad && ep.accumulate) ? p[j] + v[j] : v[j];
    }
  }
}

// dw[i] = sum_s partial[s][i]  (fixed order: deterministic)
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ partial, float* __restrict__ out, int64_t n, int splits) {
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int z = 0; z < splits; ++z) s += partial[(size_t)z * n + i];
  out[i] = s;
}

// HWIO [R,S,C,K] -> HWOI [R,S,K,C]
__global__ void __launch_bounds__(256)
hwio_to_hwoi_kernel(const float* __restrict__ w, float* __restrict__ wt, int RS, int C, int K) {
  __shared__ float tile[32][33];
  const int rs = blockIdx.z;
  const int c0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, k = k0 + tx;
    tile[j][tx] = (c < C && k < K) ? w[((size_t)rs * C + c) * K + k] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int k = k0 + j, c = c0 + tx;
    if (c < C && k < K) wt[((size_t)rs * K + k) * C + c] = tile[tx][j];
  }
}

// cols[m][k] = x[n, oh*sh - pt + r, ow*sw - pl + s, c], k = (r*S + s)*C + c; zero for padding taps and
// for k in [R*S*C, kpad).  Used to turn a conv whose Cin is not a multiple of 16 (the 7x7x3 / 5x5x3 /
// 3x3x3 first layers) into a 1x1 conv over kpad channels that the tensor-core path accepts.
__global__ void __launch_bounds__(256)
im2col_kernel(const float* __restrict__ x, Geom g, int M, int K, int kpad, float* __restrict__ cols) {
  const int kv = kpad >> 2;
  const int64_t total = (int64_t)M * kv;
  const int64_t stride = (int64_t)gridDim.x * 256;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += stride) {
    const int m = (int)(i / kv);
    const int k0 = (int)(i - (int64_t)m * kv) << 2;
    const int pq = g.P * g.Q;
    const int n = m / pq;
    const int rem = m - n * pq;
    const int oh = rem / g.Q, ow = rem - oh * g.Q;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + j;
      v[j] = 0.f;
      if (k < K) {
        const int rs = k / g.C, c = k - rs * g.C;
        const int r = rs / g.S, q = rs - r * g.S;
        const int ih = oh * g.sh - g.pt + r, iw = ow * g.sw - g.pl + q;
        if (ih >= 0 && ih < g.H && iw >= 0 && iw < g.W) v[j] = __ldg(x + (((size_t)n * g.H + ih) * g.W + iw) * g.C + c);
      }
    }
    *reinterpret_cast<float4*>(cols + (size_t)m * kpad + k0) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// im2col straight into split-bf16 operand planes (the 1x1 tensor-core conv's input format): one 16-byte chunk
// (8 k-values) per thread per plane, consecutive threads -> consecutive chunks of a row; the k -> (r, s, c)
// decode comes from a shared-memory table, the row decode uses two divisions per 8 outputs.
__global__ void __launch_bounds__(256)
im2col_planes_kernel(const float* __restrict__ x, Geom g, int M, int K, int kpad, void* __restrict__ hi,
                     void* __restrict__ lo) {
  extern __shared__ int s_tab[];                 // per k: (r << 20) | (q << 10) | c, or -1 beyond K
  for (int k = threadIdx.x; k < kpad; k += 256) {
    int e = -1;
    if (k < K) {
      const int rs = k / g.C, c = k - rs * g.C;
      const int r = rs / g.S, q = rs - r * g.S;
      e = (r << 20) | (q << 10) | c;
    }
    s_tab[k] = e;
  }
  __syncthreads();
  const int kc = kpad >> 3;
  const int64_t total = (int64_t)M * kc;
  const int64_t stride = (int64_t)gridDim.x * 256;
  const int pq = g.P * g.Q;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += stride) {
    const int m = (int)(i / kc);
    const int k0 = (int)(i - (int64_t)m * kc) << 3;
    const int n = m / pq;
    const int rem = m - n * pq;
    const int oh = rem / g.Q, ow = rem - oh * g.Q;
    const int ih0 = oh * g.sh - g.pt, iw0 = ow * g.sw - g.pl;
    const float* xn = x + (size_t)n * g.H * g.W * g.C;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int e = s_tab[k0 + j];
      const int ih = ih0 + (e >> 20), iw = iw0 + ((e >> 10) & 1023);
      v[j] = (e >= 0 && ih >= 0 && ih < g.H && iw >= 0 && iw < g.W) ? __ldg(xn + ((size_t)ih * g.W + iw) * g.C + (e & 1023)) : 0.f;
    }
    const int64_t o = (int64_t)m * kpad + k0;
    pf_st_planes4(hi, lo, o, make_float4(v[0], v[1], v[2], v[3]));
    pf_st_planes4(hi, lo, o + 4, make_float4(v[4], v[5], v[6], v[7]));
  }
}

// Space-to-depth of a stride-2 first layer (7x7x3 stem): x'[n][y'][x'][(dy*2+dx)*C + c] = x[n][2y'+dy-pt][2x'+dx-pl][c]
// (zero outside the image, zero in the padding channels), written straight as split-bf16 operand planes.  The
// stride-2 RxS conv over C channels then IS a stride-1 ceil(R/2) x ceil(S/2) conv over 4C (-> cpad) channels, which the
// tensor-core kernels take directly: no [N*P*Q, R*S*C] column matrix (2 GB at B = 256) is ever materialised.
__global__ void __launch_bounds__(256)
s2d_planes_kernel(const float* __restrict__ x, int N, int H, int W, int C, int pt, int pl, int HP, int WP, int cpad,
                  void* __restrict__ hi, void* __restrict__ lo) {
  const int c4 = cpad >> 2;
  const int64_t total = (int64_t)N * HP * WP * c4;
  const int64_t stride = (int64_t)gridDim.x * 256;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += stride) {
    const int ch0 = (int)(i % c4) << 2;
    int64_t t = i / c4;
    const int xq = (int)(t % WP); t /= WP;
    const int yq = (int)(t % HP);
    const int n = (int)(t / HP);
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ch = ch0 + j;
      v[j] = 0.f;
      if (ch < 4 * C) {
        const int blk = ch / C, c = ch - blk * C;
        const int ih = 2 * yq + (blk >> 1) - pt, iw = 2 * xq + (blk & 1) - pl;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W) v[j] = __ldg(x + (((size_t)n * H + ih) * W + iw) * C + c);
      }
    }
    pf_st_planes4(hi, lo, i << 2, make_float4(v[0], v[1], v[2], v[3]));
  }
}

// dst[j][:] = idx[j] >= 0 ? src[idx[j]][:] : 0 — re-arranges a small weight (gradient) matrix by rows
__global__ void __launch_bounds__(256)
gather_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ idx, int n_rows, int row_len,
                   float* __restrict__ dst) {
  const int64_t total = (int64_t)n_rows * row_len;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    const int j = (int)(i / row_len), e = (int)(i - (int64_t)j * row_len);
    const int s = idx[j];
    dst[i] = s >= 0 ? src[(size_t)s * row_len + e] : 0.f;
  }
}

int check_geom(const pf_conv_desc* d, Geom* g, const char* who) {
  PF_REQUIRE(d != nullptr, "%s: null descriptor", who);
  PF_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0 && d->c > 0 && d->k > 0 && d->r > 0 && d->s > 0 &&
                 d->p > 0 && d->q > 0 && d->stride_h > 0 && d->stride_w > 0 && d->pad_t >= 0 && d->pad_l >= 0,
             "%s: non-positive dimension in conv descriptor", who);
  PF_REQUIRE((int64_t)(d->p - 1) * d->stride_h - d->pad_t + d->r - 1 < d->h + d->r &&
                 (int64_t)d->n * d->h * d->w < (1ll << 31) && (int64_t)d->n * d->p * d->q < (1ll << 31) &&
                 (int64_t)d->r * d->s * d->c < (1ll << 31) && (int64_t)d->r * d->s * d->k < (1ll << 31),
             "%s: conv descriptor out of range", who);
  *g = Geom{d->n, d->h, d->w, d->c, d->k, d->r, d->s, d->p, d->q, d->stride_h, d->stride_w, d->pad_t, d->pad_l};
  return PF_OK;
}

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

extern "C" {

int pf_im2col(const pf_conv_desc* d, const float* x_dev, int kpad, float* cols_dev, void* stream) {
  Geom g;
  int rc = check_geom(d, &g, "pf_im2col");
  if (rc) return rc;
  const int K = g.R * g.S * g.C;
  PF_REQUIRE(x_dev && cols_dev && kpad >= K && (kpad & 3) == 0 && ((uintptr_t)cols_dev & 15) == 0,
             "pf_im2col: kpad must be a multiple of 4 >= R*S*C and cols 16-byte aligned");
  const int M = g.N * g.P * g.Q;
  int64_t blocks = ((int64_t)M * (kpad >> 2) + 255) / 256;
  if (blocks > PF_NUM_SMS * 16) blocks = PF_NUM_SMS * 16;
  im2col_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x_dev, g, M, K, kpad, cols_dev);
  PF_CHECK_LAUNCH("pf_im2col");
  return PF_OK;
}

int pf_im2col_planes(const pf_conv_desc* d, const float* x_dev, int kpad, void* cols_hi_dev, void* cols_lo_dev,
                     void* stream) {
  Geom g;
  int rc = check_geom(d, &g, "pf_im2col_planes");
  if (rc) return rc;
  const int K = g.R * g.S * g.C, M = g.N * g.P * g.Q;
  PF_REQUIRE(x_dev && cols_hi_dev && cols_lo_dev, "pf_im2col_planes: null pointer");
  PF_REQUIRE(kpad >= K && kpad % 8 == 0 && kpad <= 8192, "pf_im2col_planes: kpad must be a multiple of 8 in [R*S*C, 8192]");
  PF_REQUIRE(g.R < 1024 && g.S < 1024 && g.C < 1024, "pf_im2col_planes: filter / channel extent too large");
  PF_REQUIRE((((uintptr_t)cols_hi_dev | (uintptr_t)cols_lo_dev) & 15) == 0, "pf_im2col_planes: planes must be 16-byte aligned");
  int64_t blocks = ((int64_t)M * (kpad >> 3) + 255) / 256;
  if (blocks > PF_NUM_SMS * 16) blocks = PF_NUM_SMS * 16;
  im2col_planes_kernel<<<(unsigned)blocks, 256, kpad * sizeof(int), (cudaStream_t)stream>>>(x_dev, g, M, K, kpad, cols_hi_dev,
                                                                                           cols_lo_dev);
  PF_CHECK_LAUNCH("pf_im2col_planes");
  return PF_OK;
}

int pf_s2d_planes(const float* x_dev, int n, int h, int w, int c, int pad_t, int pad_l, int hp, int wp, int cpad,
                  void* hi_dev, void* lo_dev, void* stream) {
  PF_REQUIRE(n > 0 && h > 0 && w > 0 && c > 0 && hp > 0 && wp > 0 && pad_t >= 0 && pad_l >= 0, "pf_s2d_planes: bad shape");
  PF_REQUIRE(cpad % 8 == 0 && cpad >= 4 * c, "pf_s2d_planes: cpad must be a multiple of 8 and >= 4*C");
  PF_REQUIRE(x_dev && hi_dev && lo_dev, "pf_s2d_planes: null pointer");
  PF_REQUIRE((((uintptr_t)hi_dev | (uintptr_t)lo_dev) & 15) == 0, "pf_s2d_planes: planes must be 16-byte aligned");
  const int64_t total = (int64_t)n * hp * wp * (cpad >> 2);
  int64_t blocks = (total + 255) / 256;
  if (blocks > PF_NUM_SMS * 16) blocks = PF_NUM_SMS * 16;
  s2d_planes_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x_dev, n, h, w, c, pad_t, pad_l, hp, wp, cpad, hi_dev,
                                                                       lo_dev);
  PF_CHECK_LAUNCH("pf_s2d_planes");
  return PF_OK;
}

int pf_gather_rows(const float* src_dev, const int32_t* idx_dev, int n_rows, int row_len, float* dst_dev, void* stream) {
  PF_REQUIRE(n_rows >= 0 && row_len > 0, "pf_gather_rows: bad shape");
  if (n_rows == 0) return PF_OK;
  PF_REQUIRE(src_dev && idx_dev && dst_dev, "pf_gather_rows: null pointer");
  int64_t blocks = ((int64_t)n_rows * row_len + 255) / 256;
  if (blocks > PF_NUM_SMS * 8) blocks = PF_NUM_SMS * 8;
  gather_rows_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(src_dev, idx_dev, n_rows, row_len, dst_dev);
  PF_CHECK_LAUNCH("pf_gather_rows");
  return PF_OK;
}

int pf_conv2d_fwd(const pf_conv_desc* d, const float* x_dev, const float* w_dev, const float* bias_dev,
                  int relu, float* y_dev, void* stream) {
  Geom g;
  int rc = check_geom(d, &g, "pf_conv2d_fwd");
  if (rc) return rc;
  PF_REQUIRE(x_dev && w_dev && y_dev, "pf_conv2d_fwd: null pointer");
  const int M = g.N * g.P * g.Q, Ng = g.K, K = g.R * g.S * g.C;
  dim3 grid((M + BM - 1) / BM, (Ng + BN - 1) / BN, 1);
  Epi ep{y_dev, bias_dev, relu, 0};
  const bool vec = (g.C % 4 == 0) && (g.K % 4 == 0) && aligned16(x_dev) && aligned16(w_dev) && aligned16(y_dev);
  if (vec)
    igemm_kernel<kFwd, true><<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, w_dev, g, M, Ng, K, K, ep);
  else
    igemm_kernel<kFwd, false><<<grid, NT, 0, (cudaStream_t)stream>>>(x_dev, w_dev, g, M, Ng, K, K, ep);
  PF_CHECK_LAUNCH("pf_conv2d_fwd");
  return PF_OK;
}

int pf_conv2d_dgrad(const pf_conv_desc* d, const float* dy_dev, const float* w_dev, float* wt_ws_dev,
                    int accumulate, float* dx_dev, void* stream) {
  Geom g;
  int rc = check_geom(d, &g, "pf_conv2d_dgrad");
  if (rc) return rc;
  PF_REQUIRE(dy_dev && w_dev && wt_ws_dev && dx_dev, "pf_conv2d_dgrad: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  // B operand = w^T per tap: HWOI, a [R*S*Cout, Cin] row-major matrix
  dim3 tg((g.K + 31) / 32, (g.C + 31) / 32, g.R * g.S);
  hwio_to_hwoi_kernel<<<tg, 256, 0, st>>>(w_dev, wt_ws_dev, g.R * g.S, g.C, g.K);
  PF_CHECK_LAUNCH("pf_conv2d_dgrad/transpose");
  const int M = g.N * g.H * g.W, Ng = g.C, K = g.R * g.S * g.K;
  dim3 grid((M + BM - 1) / BM, (Ng + BN - 1) / BN, 1);
  Epi ep{dx_dev, nullptr, 0, accumulate};
  const bool vec = (g.C % 4 == 0) && (g.K % 4 == 0) && aligned16(dy_dev) && aligned16(wt_ws_dev) && aligned16(dx_dev);
  if (vec)
    igemm_kernel<kDgrad, true><<<grid, NT, 0, st>>>(dy_dev, wt_ws_dev, g, M, Ng, K, K, ep);
  else
    igemm_kernel<kDgrad, false><<<grid, NT, 0, st>>>(dy_dev, wt_ws_dev, g, M, Ng, K, K, ep);
  PF_CHECK_LAUNCH("pf_conv2d_dgrad");
  return PF_OK;
}

int64_t pf_conv2d_wgrad_workspace_bytes(const pf_conv_desc* d) {
  if (!d) return 0;
  const int64_t M = (int64_t)d->r * d->s * d->c, Ng = d->k;
  return (int64_t)PF_CONV_WGRAD_MAX_SPLITS * M * Ng * 4;
}

int pf_conv2d_wgrad(const pf_conv_desc* d, const float* x_dev, const float* dy_dev, float* ws_dev,
                    float* dw_dev, void* stream) {
  Geom g;
  int rc = check_geom(d, &g, "pf_conv2d_wgrad");
  if (rc) return rc;
  PF_REQUIRE(x_dev && dy_dev && dw_dev && ws_dev, "pf_conv2d_wgrad: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int M = g.R * g.S * g.C, Ng = g.K, K = g.N * g.P * g.Q;
  const int tiles = ((M + BM - 1) / BM) * ((Ng + BN - 1) / BN);
  int splits = (4 * PF_NUM_SMS + tiles - 1) / tiles;
  const int max_by_k = (K + 4 * BK - 1) / (4 * BK);
  if (splits > max_by_k) splits = max_by_k;
  if (splits > PF_CONV_WGRAD_MAX_SPLITS) splits = PF_CONV_WGRAD_MAX_SPLITS;
  if (splits < 1) splits = 1;
  int kps = (K + splits - 1) / splits;
  kps = (kps + BK - 1) / BK * BK;
  splits = (K + kps - 1) / kps;
  dim3 grid((M + BM - 1) / BM, (Ng + BN - 1) / BN, splits);
  Epi ep{splits == 1 ? dw_dev : ws_dev, nullptr, 0, 0};
  const bool vec = (g.C % 4 == 0) && (g.K % 4 == 0) && aligned16(x_dev) && aligned16(dy_dev) &&
                   aligned16(dw_dev) && aligned16(ws_dev);
  if (vec)
    igemm_kernel<kWgrad, true><<<grid, NT, 0, st>>>(x_dev, dy_dev, g, M, Ng, K, kps, ep);
  else
    igemm_kernel<kWgrad, false><<<grid, NT, 0, st>>>(x_dev, dy_dev, g, M, Ng, K, kps, ep);
  PF_CHECK_LAUNCH("pf_conv2d_wgrad");
  if (splits > 1) {
    const int64_t n = (int64_t)M * Ng;
    splitk_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws_dev, dw_dev, n, splits);
    PF_CHECK_LAUNCH("pf_conv2d_wgrad/reduce");
  }
  return PF_OK;
}

}  // extern "C"
