// pf_conv_tc.cu — convolution forward / dgrad / wgrad on the Hopper tensor cores (warpgroup MMA, wgmma).
//
// The one genuine dense contraction of the step (SURVEY §8 a4: tf.nn.conv2d re-created on the
// quantized weight, /root/reference/learners/uniform_quantization/utils.py:92-104, and its dgrad).
// The tensor cores have no fp32 x fp32 MMA, and the parity bar is fp32 (1e-5 on losses), so operands are split
//     x = hi + lo,  hi = bf16(x), lo = bf16(x - hi)         (representation error 2^-18)
// and every k-slice issues three bf16 MMAs into ONE fp32 register accumulator:
//     D += A_hi*B_hi + A_hi*B_lo + A_lo*B_hi               (the lo*lo term, 2^-18 relative, is dropped)
//
// Implicit GEMM, both operands K-major:  D[M x N] = A[M x K] * B[N x K]^T
//   fwd  : M = N*P*Q pixels, N = Cout, K = R*S*Cin;  A = im2col(x) gathered on the fly; B = w^T
//   dgrad: M = N*H*W pixels, N = Cin,  K = R*S*Cout; A = gathered dy;                  B = w as [Cin][(r,s,cout)]
// B is pre-split / pre-transposed once per step by pf_conv2d_tc_prep_weight (weights change every
// step; 20 B per weight).  The activation operand comes either as fp32 NHWC (converted to the split
// representation by the producer warps on the fly) or as PRE-SPLIT bf16 planes written by the kernel that
// produced the tensor (BN-apply / activation quantizer / BN-backward): then the producers are pure
// cp.async copies into the 128B-swizzled tiles.  Kernel structure: see conv_tc_persist_kernel below.
#include "pf_conv_tc.cuh"

namespace pfconv {
int tc_geom(const pf_conv_desc* d, TcGeom* g, const char* who) {
  PF_REQUIRE(d != nullptr, "%s: null descriptor", who);
  PF_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0 && d->c > 0 && d->k > 0 && d->r > 0 && d->s > 0 && d->p > 0 &&
                 d->q > 0 && d->stride_h > 0 && d->stride_w > 0 && d->pad_t >= 0 && d->pad_l >= 0,
             "%s: non-positive dimension in conv descriptor", who);
  *g = TcGeom{d->n, d->h, d->w, d->c, d->k, d->r, d->s, d->p, d->q, d->stride_h, d->stride_w, d->pad_t, d->pad_l};
  return PF_OK;
}

static pf_tc_plan g_last_plan;            // seq == 0: nothing recorded yet
void record_plan(const pf_tc_plan& p) {
  const int seq = g_last_plan.seq + 1;
  g_last_plan = p;
  g_last_plan.seq = seq;
}
}  // namespace pfconv

namespace {
using namespace pfconv;

constexpr int kMaxStages = 4;

__device__ __forceinline__ void split4(const float4 v, uint2& hi, uint2& lo) { pf_split4(v, hi, lo); }

// =============================================================================================
// PERSISTENT, warp-specialised fwd / dgrad kernel.  One CTA per SM loops over output tiles;
//   warps 0-7   two MMA warpgroups (wgmma, 64 rows each) that also run the epilogue (registers -> shared
//               accumulator tile -> coalesced global; bias / ReLU / residual / accumulate) while the producers
//               already fill the next tile's stages;
//   warps 8-15  producers (A gather + fp32 -> split-bf16 conversion with a register ping-pong that runs
//               across tile boundaries; B via cp.async).
// BN goes up to 128 (the accumulator registers of a warpgroup).  When one n-tile covers all output channels and
// the whole split weight matrix fits next to >= 2 A stages, B is loaded ONCE per CTA and stays resident
// ("B-stationary": every 1x1 layer of the early stages, K <= 256).
// MODE 2 = dgrad of a strided convolution decomposed into stride_h*stride_w pixel-parity classes: the rows of
// a tile all belong to one class (h = ph + sh*h', w = pw + sw*w'), and only the filter taps that can reach that
// class are visited, so no MMA multiplies structural zeros (the gather-with-divisibility-test formulation of
// MODE 1 wastes 3/4 of the tensor-core work of a 3x3 stride-2 layer).
constexpr int kMaxClasses = 4;
constexpr int kMaxTaps = 9;
struct TcClass {
  int tile_begin, Mc, Hc, Wc, ph, pw, ntaps, pad_;
  FastDiv d_hw, d_w;
  int8_t eh[kMaxTaps + 3], ew[kMaxTaps + 3], tap[kMaxTaps + 3];
};
struct TcP {
  TcGeom g;
  int M, Ng, Kdim, Kpad, BN, nk, n_stages, n_bslots, b_stationary, m_tiles, n_tiles, total_tiles;
  int accumulate, relu, ncls, cblocks, ring;
  FastDiv d_hw, d_w, d_cc, d_s, d_ntiles, d_cblocks;
  TcClass cls[kMaxClasses];
};

constexpr int kProdWarps = 8;
constexpr int kThreadsP = (kMmaWarps + kProdWarps) * 32;   // 512

template <int MODE>
__device__ __forceinline__ int tile_class(const TcP& p, int mt) {
  int ci = 0;
  if (MODE == 2) {
#pragma unroll
    for (int j = 1; j < kMaxClasses; ++j)
      if (j < p.ncls && mt >= p.cls[j].tile_begin) ci = j;
  }
  return ci;
}

template <int MODE, bool PLANES, int BN, bool BNO = false>
__global__ void __launch_bounds__(kThreadsP, 1)
conv_tc_persist_kernel(const float* __restrict__ src, const __nv_bfloat16* __restrict__ a_hi_g,
                       const __nv_bfloat16* __restrict__ a_lo_g, const __nv_bfloat16* __restrict__ b_hi,
                       const __nv_bfloat16* __restrict__ b_lo, float* __restrict__ out,
                       const float* __restrict__ bias, const float* __restrict__ residual,
                       const __grid_constant__ TcP p, const __grid_constant__ pf_tc_bn_out bn) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const TcGeom& g = p.g;
  const uint32_t a_bytes = TM * 128, b_bytes = (uint32_t)BN * 128;
  uint8_t* smem_a = smem;                                           // n_stages x (hi, lo)
  uint8_t* smem_b = smem + (size_t)p.n_stages * 2 * a_bytes;        // n_bslots x (hi, lo)
  float* acc_s = reinterpret_cast<float*>(smem_b + (size_t)p.n_bslots * 2 * b_bytes);
  long long* rowoff_all = reinterpret_cast<long long*>(acc_s + TM * acc_pitch(BN));
  uint8_t* ring_all = reinterpret_cast<uint8_t*>(rowoff_all + kMmaWarps * 32);   // p.ring: 8 warps x kRingDepth slots
  __shared__ uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int s = 0; s < p.n_stages; ++s) {
      mbar_init(&full_bar[s], kProdWarps * 32);
      mbar_init(&empty_bar[s], kMmaWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int first_tile = blockIdx.x, tile_step = gridDim.x;

  if (warp >= kMmaWarps) {
    // =================================== producers ===================================
    const int pt_ = tid - kMmaWarps * 32;
    const int l8 = pt_ & 7, rgrp = pt_ >> 3;          // 32-byte slice of the row, row group (rows rgrp + 32*i)
    const int CC = (MODE == 0) ? g.C : g.K;           // channels of the gathered tensor
    const uint32_t chunk_off = (((uint32_t)l8) ^ (uint32_t)(rgrp & 7)) << 4;
    auto tile_nk = [&](int tile) -> int {
      if (MODE != 2) return p.nk;
      const int mt = (int)fdiv((uint32_t)tile, p.d_ntiles);
      return p.cls[tile_class<MODE>(p, mt)].ntaps * p.cblocks;
    };
    // element offsets (-1: zero row) of this thread's 4 rows of A for k-stage ks of `tile`: this lane's 8-channel
    // chunk (l8) lies inside one filter tap (channel counts are multiples of 16)
    auto a_offsets = [&](int tile, int ks, long long (&off)[4]) {
      const int mt = (int)fdiv((uint32_t)tile, p.d_ntiles);
#pragma unroll
      for (int i = 0; i < 4; ++i) off[i] = -1;
      if (MODE != 2) {
        const int kk = ks * BK + l8 * 8;
        const int tap = (int)fdiv((uint32_t)kk, p.d_cc);
        const int c = kk - tap * CC;
        const int r = (int)fdiv((uint32_t)tap, p.d_s), q = tap - r * g.S;
        const int hw = (MODE == 0) ? g.P * g.Q : g.H * g.W;
        const int wq = (MODE == 0) ? g.Q : g.W;
        const bool unit_stride = g.sh == 1 && g.sw == 1;
        if (kk < p.Kdim) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int m = mt * TM + rgrp + 32 * i;
            if (m < p.M) {
              const int n_ = (int)fdiv((uint32_t)m, p.d_hw);
              const int rem = m - n_ * hw;
              const int y = (int)fdiv((uint32_t)rem, p.d_w), x = rem - y * wq;
              if (MODE == 0) {
                const int ih = y * g.sh - g.pt + r, iw = x * g.sw - g.pl + q;
                if (ih >= 0 && ih < g.H && iw >= 0 && iw < g.W) off[i] = (((long long)n_ * g.H + ih) * g.W + iw) * g.C + c;
              } else {
                const int th = y + g.pt - r, tw = x + g.pl - q;
                if (th >= 0 && tw >= 0) {
                  if (unit_stride) {
                    if (th < g.P && tw < g.Q) off[i] = (((long long)n_ * g.P + th) * g.Q + tw) * g.K + c;
                  } else {
                    const int oh = th / g.sh, ow = tw / g.sw;
                    if (oh * g.sh == th && ow * g.sw == tw && oh < g.P && ow < g.Q)
                      off[i] = (((long long)n_ * g.P + oh) * g.Q + ow) * g.K + c;
                  }
                }
              }
            }
          }
        }
      } else {
        const TcClass& k = p.cls[tile_class<MODE>(p, mt)];
        const int tap_i = (int)fdiv((uint32_t)ks, p.d_cblocks);
        const int c = (ks - tap_i * p.cblocks) * BK + l8 * 8;
        const int eh = k.eh[tap_i], ew = k.ew[tap_i];
        const int hwc = k.Hc * k.Wc;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int mc = (mt - k.tile_begin) * TM + rgrp + 32 * i;
          if (mc < k.Mc) {
            const int n_ = (int)fdiv((uint32_t)mc, k.d_hw);
            const int rem = mc - n_ * hwc;
            const int y = (int)fdiv((uint32_t)rem, k.d_w), x = rem - y * k.Wc;
            const int oh = y + eh, ow = x + ew;
            if (oh >= 0 && oh < g.P && ow >= 0 && ow < g.Q) off[i] = (((long long)n_ * g.P + oh) * g.Q + ow) * g.K + c;
          }
        }
      }
    };
    auto issue_loads_a = [&](int tile, int ks, float4 (&av)[8]) {
      long long off[4];
      a_offsets(tile, ks, off);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        av[2 * i] = off[i] >= 0 ? __ldg(reinterpret_cast<const float4*>(src + off[i])) : make_float4(0.f, 0.f, 0.f, 0.f);
        av[2 * i + 1] = off[i] >= 0 ? __ldg(reinterpret_cast<const float4*>(src + off[i]) + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    };
    uint32_t it = 0;                                   // global k-stage counter of this CTA (ring position)
    auto issue_b = [&](int tile, int ks, bool first, uint32_t s) {
      if (!p.b_stationary || first) {
        const int mt = (int)fdiv((uint32_t)tile, p.d_ntiles);
        const int n0 = (tile - mt * p.n_tiles) * BN;
        uint8_t* sb = smem_b + (size_t)(p.b_stationary ? ks : (int)s) * 2 * b_bytes;
        size_t kcol;
        if (MODE == 2) {
          const TcClass& k = p.cls[tile_class<MODE>(p, mt)];
          const int tap_i = (int)fdiv((uint32_t)ks, p.d_cblocks);
          kcol = (size_t)k.tap[tap_i] * g.K + (size_t)(ks - tap_i * p.cblocks) * BK + l8 * 8;
        } else {
          kcol = (size_t)ks * BK + l8 * 8;
        }
        for (int br = rgrp; br < BN; br += 32) {
          const bool ok = n0 + br < p.Ng;
          const size_t off = (size_t)(ok ? n0 + br : 0) * p.Kpad + kcol;
          const uint32_t dst = smem_u32(sb + (size_t)br * 128 + chunk_off);
          const uint32_t nbytes = ok ? 16u : 0u;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(b_hi + off), "r"(nbytes) : "memory");
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + b_bytes), "l"(b_lo + off), "r"(nbytes) : "memory");
        }
      }
    };
    auto do_stage = [&](int tile, int ks, bool first, const float4 (&av)[8]) {
      const uint32_t s = it % (uint32_t)p.n_stages;
      mbar_wait(&empty_bar[s], ((it / (uint32_t)p.n_stages) & 1u) ^ 1u);   // slot free?
      uint8_t* sa = smem_a + (size_t)s * 2 * a_bytes;
      issue_b(tile, ks, first, s);
      asm volatile("cp.async.commit_group;" ::: "memory");
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint2 h0, l0, h1, l1;
        split4(av[2 * i], h0, l0);
        split4(av[2 * i + 1], h1, l1);
        uint8_t* rowp = sa + (size_t)(rgrp + 32 * i) * 128 + chunk_off;
        *reinterpret_cast<uint4*>(rowp) = make_uint4(h0.x, h0.y, h1.x, h1.y);
        *reinterpret_cast<uint4*>(rowp + a_bytes) = make_uint4(l0.x, l0.y, l1.x, l1.y);
      }
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      fence_proxy_async_smem();   // generic-proxy + cp.async writes -> visible to the tensor core (async proxy)
      mbar_arrive(&full_bar[s]);
      ++it;
    };
    if (PLANES) {
      // pre-split operand: both tiles are plain cp.async copies; the stage's barrier arrival fires when this
      // thread's copies have landed, so the producers only ever wait for a free slot
      for (int tile = first_tile; tile < p.total_tiles; tile += tile_step) {
        const int nkt = tile_nk(tile);
        for (int ks = 0; ks < nkt; ++ks, ++it) {
          const uint32_t s = it % (uint32_t)p.n_stages;
          mbar_wait(&empty_bar[s], ((it / (uint32_t)p.n_stages) & 1u) ^ 1u);
          long long off[4];
          a_offsets(tile, ks, off);
          const uint32_t sa = smem_u32(smem_a + (size_t)s * 2 * a_bytes);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint32_t dst = sa + (uint32_t)(rgrp + 32 * i) * 128 + chunk_off;
            const uint32_t nb = off[i] >= 0 ? 16u : 0u;
            const size_t o = off[i] >= 0 ? (size_t)off[i] : 0;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(a_hi_g + o), "r"(nb) : "memory");
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + a_bytes), "l"(a_lo_g + o), "r"(nb) : "memory");
          }
          issue_b(tile, ks, tile == first_tile, s);
          asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(&full_bar[s])) : "memory");
        }
      }
      asm volatile("cp.async.wait_all;" ::: "memory");
    } else {
    // flat (tile, k-stage) iteration with a two-deep register ping-pong
    int t0 = first_tile, k0 = 0, nk0 = (t0 < p.total_tiles) ? tile_nk(t0) : 0;
    while (t0 < p.total_tiles && nk0 == 0) { t0 += tile_step; nk0 = (t0 < p.total_tiles) ? tile_nk(t0) : 0; }
    auto advance = [&](int& t, int& k, int& nkt) {
      if (++k >= nkt) {
        k = 0;
        do {
          t += tile_step;
          nkt = (t < p.total_tiles) ? tile_nk(t) : 0;
        } while (t < p.total_tiles && nkt == 0);     // zero-tap classes have no main loop
      }
    };
    if (t0 < p.total_tiles) {
      float4 a0[8], a1[8];
      issue_loads_a(t0, k0, a0);
      while (true) {
        int t1 = t0, k1 = k0, nk1 = nk0;
        advance(t1, k1, nk1);
        const bool v1 = t1 < p.total_tiles;
        if (v1) issue_loads_a(t1, k1, a1);
        do_stage(t0, k0, t0 == first_tile, a0);
        if (!v1) break;
        int t2 = t1, k2 = k1, nk2 = nk1;
        advance(t2, k2, nk2);
        const bool v2 = t2 < p.total_tiles;
        if (v2) issue_loads_a(t2, k2, a0);
        do_stage(t1, k1, t1 == first_tile, a1);
        if (!v2) break;
        t0 = t2; k0 = k2; nk0 = nk2;
      }
    }
    }
  } else {
    // ============================ MMA warpgroups + epilogue (warps 0-7) ============================
    const int wg = warp >> 2;                // rows [64 wg, 64 wg + 64) of the tile
    long long* rowoff = rowoff_all + warp * 32;
    const float* extra = residual ? residual : (p.accumulate ? out : nullptr);
    uint32_t it = 0;
    for (int tile = first_tile; tile < p.total_tiles; tile += tile_step) {
      const int mt = (int)fdiv((uint32_t)tile, p.d_ntiles);
      const int n0 = (tile - mt * p.n_tiles) * BN;
      int nk = p.nk;
      if (MODE == 2) nk = p.cls[tile_class<MODE>(p, mt)].ntaps * p.cblocks;
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      uint32_t prev = 0;
      for (int ks = 0; ks < nk; ++ks, ++it) {
        const uint32_t s = it % (uint32_t)p.n_stages;
        mbar_wait(&full_bar[s], (it / (uint32_t)p.n_stages) & 1u);
        if (PLANES) fence_proxy_async_smem();   // cp.async writes -> visible to the tensor core (async proxy)
        const uint32_t a_hi = smem_u32(smem_a + (size_t)s * 2 * a_bytes) + (uint32_t)wg * 64 * 128, a_lo = a_hi + a_bytes;
        const uint32_t bh = smem_u32(smem_b + (size_t)(p.b_stationary ? ks : (int)s) * 2 * b_bytes), bl = bh + b_bytes;
        wg_mma_stage<BN, 0, 2, 2>(acc, a_hi, a_lo, bh, bl, 32, 32, 16, 1024, 16, 1024);
        wgmma_wait<1>(acc);                      // the previous stage's MMAs have completed: release it
        if (ks > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = s;
      }
      wgmma_wait<0>(acc);
      if (nk > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      long long off = -1;                    // global element offset of this lane's row (-1: beyond the problem)
      const int row = (warp & 3) * 32 + lane;
      if (MODE != 2) {
        const int m = mt * TM + row;
        if (m < p.M) off = (long long)m * p.Ng;
      } else {
        const TcClass& k = p.cls[tile_class<MODE>(p, mt)];
        const int mc = (mt - k.tile_begin) * TM + row;
        if (mc < k.Mc) {
          const int hwc = k.Hc * k.Wc;
          const int n_ = (int)fdiv((uint32_t)mc, k.d_hw);
          const int rem = mc - n_ * hwc;
          const int y = (int)fdiv((uint32_t)rem, k.d_w), x = rem - y * k.Wc;
          off = (((long long)n_ * g.H + (k.ph + y * g.sh)) * g.W + (k.pw + x * g.sw)) * g.C;
        }
      }
      if (BNO) {
        // wg_tile_to_smem, and between its barriers the folded batch norm's constants of the tile's columns, in the shared
        // memory after the ring (the J table space of epi_fixed_bytes, which this kernel does not use otherwise)
        float* bn_tab = reinterpret_cast<float*>(ring_all + (p.ring ? kMmaWarps * kRingDepth * kRingSlotBytes : 0));
        named_bar_sync(1, kMmaWarps * 32);
        wgmma_store_acc<BN>(acc, acc_s, acc_pitch(BN), 64 * (tid >> 7), tid & 127);
        bn_table(bn, bn_tab, n0, BN, p.Ng, tid, kMmaWarps * 32);
        named_bar_sync(1, kMmaWarps * 32);
        epilogue_tile_a<0, true>(acc_s, warp, off, rowoff, out, extra, bias, p.relu, n0, BN, p.Ng, lane,
                                 p.ring ? ring_all + (size_t)warp * kRingDepth * kRingSlotBytes : nullptr, EpiAff{},
                                 0.f, nullptr, bn, bn_tab);
      } else {
        wg_tile_to_smem<BN>(acc, acc_s, tid);
        epilogue_tile(acc_s, warp, off, rowoff, out, extra, bias, p.relu, n0, BN, p.Ng, lane,
                      p.ring ? ring_all + (size_t)warp * kRingDepth * kRingSlotBytes : nullptr);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// fp32 -> split bf16 planes (hi = bf16(x), lo = bf16(x - hi)); 8 elements per thread, HBM-bound (8 B/element).
__global__ void __launch_bounds__(256)
split_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int64_t n8) {
  const int64_t stride = (int64_t)gridDim.x * 256;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n8; i += stride) {
    const float4 a = pf_ld_stream(src + i * 8), b = pf_ld_stream(src + i * 8 + 4);
    uint2 h0, l0, h1, l1;
    split4(a, h0, l0);
    split4(b, h1, l1);
    *reinterpret_cast<uint4*>(hi + i * 8) = make_uint4(h0.x, h0.y, h1.x, h1.y);
    *reinterpret_cast<uint4*>(lo + i * 8) = make_uint4(l0.x, l0.y, l1.x, l1.y);
  }
}

// ---------------------------------------------------------------------------------------------
// wgrad v4: persistent, warp-specialised, operands read from PRE-SPLIT bf16 planes with cp.async straight into
// the swizzled MN-major tiles (no register staging, no conversion in the loop; completion is signalled by
// cp.async.mbarrier.arrive so producers never wait for data, only for a free stage).  Work unit = (kf tile of
// 128, cout tile of BN <= 128, pixel range); units are ordered range-major so that the CTAs running together
// read the same pixels.  Epilogue: the shared epilogue_tile() into partial[split][kf][cout].
struct WgP {
  TcGeom g;
  int Mtot, Npix, pps, splits, BN, m_tiles, n_tiles, tiles, total_units, n_stages;
  FastDiv d_pq, d_q, d_c, d_s, d_tiles, d_ntiles;
};

template <int BN>
__global__ void __launch_bounds__(kThreadsP, 1)
conv_tc_wgrad_persist_kernel(const __nv_bfloat16* __restrict__ x_hi, const __nv_bfloat16* __restrict__ x_lo,
                             const __nv_bfloat16* __restrict__ dy_hi, const __nv_bfloat16* __restrict__ dy_lo,
                             float* __restrict__ partial, const __grid_constant__ WgP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const TcGeom& g = p.g;
  const uint32_t a_bytes = BK * TM * 2, b_bytes = (uint32_t)BK * BN * 2;   // one bf16 tile
  const uint32_t stage_bytes = 2 * a_bytes + 2 * b_bytes;
  float* acc_s = reinterpret_cast<float*>(smem + (size_t)p.n_stages * stage_bytes);
  long long* rowoff_all = reinterpret_cast<long long*>(acc_s + TM * acc_pitch(BN));
  __shared__ uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int s = 0; s < p.n_stages; ++s) {
      mbar_init(&full_bar[s], kProdWarps * 32);
      mbar_init(&empty_bar[s], kMmaWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int mbA = TM / 64, mbB = BN / 64;
  struct Unit {
    int split, m0, n0, pbeg, nk;
  };
  auto decode = [&](int u) -> Unit {
    Unit r;
    r.split = (int)fdiv((uint32_t)u, p.d_tiles);
    const int t = u - r.split * p.tiles;
    const int mt = (int)fdiv((uint32_t)t, p.d_ntiles);
    r.m0 = mt * TM;
    r.n0 = (t - mt * p.n_tiles) * BN;
    r.pbeg = r.split * p.pps;
    const int pend = min(p.Npix, r.pbeg + p.pps);
    r.nk = (pend - r.pbeg + BK - 1) / BK;
    return r;
  };

  if (warp >= kMmaWarps) {
    // =================================== producers ===================================
    const int pt_ = tid - kMmaWarps * 32;
    const int l16 = pt_ & 15, pg = pt_ >> 4;           // 16-byte chunk of the 128-wide MN extent, pixel group
    const uint32_t k8 = (uint32_t)(pg & 7);            // (pixel & 7) of every pixel of this thread (pixels pg + 16*i)
    const uint32_t a_mblk = (uint32_t)(l16 >> 3), chunk = (uint32_t)(l16 & 7);
    const uint32_t swz = (chunk ^ k8) << 4;
    const int pq = g.P * g.Q;
    uint32_t it = 0;
    for (int u = blockIdx.x; u < p.total_units; u += gridDim.x) {
      const Unit un = decode(u);
      const int pend = min(p.Npix, un.pbeg + p.pps);
      // A: kf = m0 + 8*l16 .. +7 lies inside one filter tap (Cin % 16 == 0): decode is stage-invariant
      const int kf = un.m0 + l16 * 8;
      const bool a_ok = kf < p.Mtot;
      const int a_tap = (int)fdiv((uint32_t)kf, p.d_c), a_c = kf - a_tap * g.C;
      const int a_r = (int)fdiv((uint32_t)a_tap, p.d_s), a_q = a_tap - a_r * g.S;
      for (int ks = 0; ks < un.nk; ++ks, ++it) {
        const uint32_t s = it % (uint32_t)p.n_stages;
        mbar_wait(&empty_bar[s], ((it / (uint32_t)p.n_stages) & 1u) ^ 1u);
        const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes), sb = sa + 2 * a_bytes;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int pix = un.pbeg + ks * BK + pg + 16 * i;
          const uint32_t kb = (uint32_t)((pg >> 3) + 2 * i);
          size_t aoff = 0, boff = 0;
          uint32_t an = 0, bn = 0;
          if (pix < pend) {
            const int pn = (int)fdiv((uint32_t)pix, p.d_pq);
            const int rem = pix - pn * pq;
            const int oh = (int)fdiv((uint32_t)rem, p.d_q), ow = rem - oh * g.Q;
            const int ih = oh * g.sh - g.pt + a_r, iw = ow * g.sw - g.pl + a_q;
            if (a_ok && ih >= 0 && ih < g.H && iw >= 0 && iw < g.W) {
              aoff = (((size_t)pn * g.H + ih) * g.W + iw) * g.C + a_c;
              an = 16;
            }
            boff = (size_t)pix * g.K;
            bn = 16;
          }
          const uint32_t da = sa + (kb * (uint32_t)(mbA * 8) + a_mblk * 8 + k8) * 128 + swz;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(da), "l"(x_hi + aoff), "r"(an) : "memory");
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(da + a_bytes), "l"(x_lo + aoff), "r"(an) : "memory");
          for (int e = l16 * 8; e < BN; e += 128) {
            const int co = un.n0 + e;
            const uint32_t nb = (co < g.K) ? bn : 0u;
            const size_t bo = nb ? boff + co : 0;
            const uint32_t db = sb + (kb * (uint32_t)(mbB * 8) + (uint32_t)(e >> 6) * 8 + k8) * 128 + swz;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(db), "l"(dy_hi + bo), "r"(nb) : "memory");
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(db + b_bytes), "l"(dy_lo + bo), "r"(nb) : "memory");
          }
        }
        // the barrier arrival fires when every cp.async issued so far by this thread has landed
        asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(&full_bar[s])) : "memory");
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else {
    // ============================ MMA warpgroups + epilogue: D rows = kf, columns = cout ============================
    const int wg = warp >> 2;                // kf rows [64 wg, 64 wg + 64) = MN block wg of the A tile
    const uint32_t sbo_a = (uint32_t)mbA * 1024u, sbo_b = (uint32_t)mbB * 1024u;
    long long* rowoff = rowoff_all + warp * 32;
    uint32_t it = 0;
    for (int u = blockIdx.x; u < p.total_units; u += gridDim.x) {
      const Unit un = decode(u);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      uint32_t prev = 0;
      for (int ks = 0; ks < un.nk; ++ks, ++it) {
        const uint32_t s = it % (uint32_t)p.n_stages;
        mbar_wait(&full_bar[s], (it / (uint32_t)p.n_stages) & 1u);
        fence_proxy_async_smem();      // cp.async (generic proxy) writes -> visible to the tensor core (async proxy)
        const uint32_t base = smem_u32(smem + (size_t)s * stage_bytes);
        const uint32_t a_hi = base + (uint32_t)wg * 1024u, a_lo = a_hi + a_bytes, bh = base + 2 * a_bytes, bl = bh + b_bytes;
        // MN-major: LBO = stride between 64-wide MN blocks, SBO = stride between 8-pixel groups; 16 pixels per MMA
        wg_mma_stage<BN, 1, 2, 2>(acc, a_hi, a_lo, bh, bl, 2 * sbo_a, 2 * sbo_b, 1024, sbo_a, 1024, sbo_b);
        wgmma_wait<1>(acc);
        if (ks > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = s;
      }
      wgmma_wait<0>(acc);
      if (un.nk > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      const int em = un.m0 + (warp & 3) * 32 + lane;
      const long long off = em < p.Mtot ? ((long long)un.split * p.Mtot + em) * g.K : -1;
      wg_tile_to_smem<BN>(acc, acc_s, tid);
      epilogue_tile(acc_s, warp, off, rowoff, partial, nullptr, nullptr, 0, un.n0, BN, g.K, lane);
    }
  }
}

__global__ void __launch_bounds__(256)
tc_splitk_reduce_kernel(const float* __restrict__ partial, float* __restrict__ out, int64_t n, int splits) {
  const int64_t i = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 4;
  if (i >= n) return;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int z = 0; z < splits; ++z) {
    const float4 v = *reinterpret_cast<const float4*>(partial + (size_t)z * n + i);
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
  }
  *reinterpret_cast<float4*>(out + i) = s;
}

// ---- weight preparation: fp32 HWIO [R,S,C,K] -> split bf16, K-major for both passes
//   fwd  : [K (cout)][Kpad_f],  k = (r*S + s)*C + c
//   dgrad: [C (cin) ][Kpad_d],  k = (r*S + s)*K + co
__global__ void __launch_bounds__(256)
tc_prep_weight_kernel(const float* __restrict__ w, int RS, int C, int K, int kpad_f, int kpad_d,
                      __nv_bfloat16* __restrict__ f_hi, __nv_bfloat16* __restrict__ f_lo,
                      __nv_bfloat16* __restrict__ d_hi, __nv_bfloat16* __restrict__ d_lo) {
  const int64_t total = (int64_t)RS * C * K;
  const int64_t stride = (int64_t)gridDim.x * 256;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += stride) {
    const int co = (int)(i % K);
    const int64_t t = i / K;
    const int c = (int)(t % C);
    const int rs = (int)(t / C);
    const float v = __ldg(w + i);
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    const __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
    const size_t fo = (size_t)co * kpad_f + (size_t)rs * C + c;
    f_hi[fo] = h;
    f_lo[fo] = l;
    if (d_hi) {
      const size_t dof = (size_t)c * kpad_d + (size_t)rs * K + co;
      d_hi[dof] = h;
      d_lo[dof] = l;
    }
  }
}

// multi-tensor form: one launch prepares every conv kernel of a network (53 launches of 10-15 us each in the
// ResNet-50 step otherwise); work items are flat chunks of the weight tensors (kind-0 pf_work)
// One work item = a 32 (k = (r,s,c) rows of the HWIO matrix) x 64 (cout) tile: rows are read coalesced, the dgrad
// copy [cin][(r,s,cout)] keeps the source's contiguity and is written directly, the fwd copy [cout][k] is the
// transpose and goes through shared memory so that its stores are 64-byte row segments instead of scattered
// 2-byte writes (the element-wise version ran at 1.5 TB/s).  work.start = first k row, work.c0 = first cout.
__global__ void __launch_bounds__(256)
tc_prep_weights_multi_kernel(const pf_tc_prep_seg* __restrict__ segs, const pf_work* __restrict__ work) {
  __shared__ __nv_bfloat16 sh_h[64][34], sh_l[64][34];
  const pf_work wk = work[blockIdx.x];
  const pf_tc_prep_seg sg = segs[wk.seg];
  const int C = sg.c, K = sg.k, KR = sg.rs * sg.c;
  const int k0 = (int)wk.start, co0 = wk.c0;
  __nv_bfloat16* f_hi = (__nv_bfloat16*)sg.fwd_hi;
  __nv_bfloat16* f_lo = (__nv_bfloat16*)sg.fwd_lo;
  __nv_bfloat16* d_hi = (__nv_bfloat16*)sg.dgrad_hi;
  __nv_bfloat16* d_lo = (__nv_bfloat16*)sg.dgrad_lo;
  {
    const int co = co0 + (threadIdx.x & 63);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int kr = (threadIdx.x >> 6) + 4 * j, kidx = k0 + kr;
      __nv_bfloat16 h = __float2bfloat16_rn(0.f), l = h;
      if (kidx < KR && co < K) {
        float v = __ldg(sg.w + (size_t)kidx * K + co);
        float level = 0.f;
        if (sg.q_bits > 0) {
          // the weight quantizer's op chain (pf_uq.cu: uq_weight_apply_kernel) on the unquantized kernel
          const int b = sg.q_ncols == 1 ? 0 : co;
          const float kq = pf_uq_kf(sg.q_bits);
          v = pf_fake_quant_lv(v, __ldg(sg.q_alpha + b), __ldg(sg.q_beta + b), kq, __ldg(sg.q_ralpha + b), __frcp_rn(kq), level);
        }
        h = __float2bfloat16_rn(v);
        l = __float2bfloat16_rn(v - __bfloat162float(h));
        if (d_hi) {
          const int rs = kidx / C, c = kidx - rs * C;
          const size_t dof = (size_t)c * sg.kpad_d + (size_t)rs * K + co;
          d_hi[dof] = h;
          d_lo[dof] = l;
        }
        if (sg.q_bits > 0) h = __float2bfloat16_rn(level - (float)(1 << (sg.q_bits - 1)));   // exact: |.| <= 128
      }
      sh_h[threadIdx.x & 63][kr] = h;
      sh_l[threadIdx.x & 63][kr] = l;
    }
  }
  __syncthreads();
  {
    const int kr = threadIdx.x & 31, kidx = k0 + kr;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int cl = (threadIdx.x >> 5) + 8 * j, co = co0 + cl;
      if (kidx < KR && co < K) {
        const size_t fo = (size_t)co * sg.kpad_f + kidx;
        f_hi[fo] = sh_h[cl][kr];
        if (sg.q_bits == 0) f_lo[fo] = sh_l[cl][kr];
      }
    }
  }
}

template <int MODE>
int launch_persist(const TcGeom& g, TcP& p, const float* src, const void* a_hi, const void* a_lo, const void* b_hi,
                   const void* b_lo, float* out, const float* bias, const float* residual, cudaStream_t st,
                   const char* who, const pf_tc_bn_out* bn) {
  const int Ng = p.Ng;
  // ---- tile width: the widest the warpgroup accumulators allow
  int BN = Ng >= 128 ? 128 : (Ng >= 64 ? 64 : (Ng >= 32 ? 32 : 16));
  const int forced = env_int("PF_TC_BN", 0);           // development knob
  if (forced >= 16 && forced <= kMaxBN && forced <= ((Ng + 15) / 16) * 16 && (forced & (forced - 1)) == 0) BN = forced;
  // the folded batch norm's epilogue at BN = 128 does not fit the 128 registers per thread of this 512-thread kernel
  if (bn && BN > 64) BN = 64;
  p.BN = BN;
  p.n_tiles = (Ng + BN - 1) / BN;
  p.total_tiles = p.m_tiles * p.n_tiles;
  p.d_ntiles = make_fastdiv((uint32_t)p.n_tiles);
  // ---- shared memory plan
  const int a_stage = 2 * TM * 128, b_slot = 2 * BN * 128;
  const int fixed = epi_fixed_bytes(BN);
  const int budget = kSmemLimit - fixed;
  int max_nk = p.nk;
  if (MODE == 2) {
    max_nk = 0;
    for (int c = 0; c < p.ncls; ++c) max_nk = std::max(max_nk, p.cls[c].ntaps * p.cblocks);
  }
  // the epilogue's residual / accumulate operand goes through a cp.async ring when the stages leave room for it
  const int ring_bytes = kMmaWarps * kRingDepth * kRingSlotBytes;
  const bool has_extra = residual != nullptr || p.accumulate;
  int budget_r = budget;
  p.ring = 0;
  if (has_extra && env_int("PF_TC_RING", 1) && BN >= 64) {
    const int b2 = budget - ring_bytes;
    const bool stat_ok = MODE != 2 && p.n_tiles == 1 && p.nk <= kMaxStages * 4 && (int64_t)p.nk * b_slot + 2 * a_stage <= b2;
    if (stat_ok || b2 / (a_stage + b_slot) >= 2) {
      p.ring = 1;
      budget_r = b2;
    }
  }
  p.b_stationary = 0;
  if (MODE != 2 && p.n_tiles == 1 && p.nk <= kMaxStages * 4 && (int64_t)p.nk * b_slot + 2 * a_stage <= budget_r &&
      env_int("PF_TC_STATIONARY", 1)) {
    p.b_stationary = 1;
    p.n_bslots = p.nk;
    p.n_stages = std::min(kMaxStages, (budget_r - p.nk * b_slot) / a_stage);
  } else {
    p.n_stages = std::min(kMaxStages, budget_r / (a_stage + b_slot));
    p.n_bslots = p.n_stages;
  }
  PF_REQUIRE(p.n_stages >= 2 || max_nk <= 1, "%s: shared-memory plan failed (BN %d)", who, BN);
  if (p.n_stages < 1) p.n_stages = 1;
  const size_t smem = (size_t)p.n_stages * a_stage + (size_t)p.n_bslots * b_slot + fixed + (p.ring ? ring_bytes : 0);
  const int grid = std::min(p.total_tiles, PF_NUM_SMS);
  record_plan(pf_tc_plan{0, 0, MODE == 0 ? 0 : 1, MODE == 2, BN, 0, 2, 2, a_hi == nullptr, p.ring ? kRingDepth : 0,
                         p.b_stationary, p.n_stages, p.total_tiles, grid, 0, 0});
  if (p.total_tiles == 0) return PF_OK;
  cudaError_t err = cudaSuccess;
  pf_tc_bn_out bn_p{};             // the folded batch norm (BNO kernels only)
  if (bn) bn_p = *bn;
  with_bn(BN, [&](auto bn_c) {
    constexpr int B = decltype(bn_c)::value;
    if (a_hi) {
      auto kern = conv_tc_persist_kernel<MODE, true, B>;
      if constexpr (MODE == 0 && B <= 64)
        if (bn) kern = conv_tc_persist_kernel<0, true, B, true>;
      err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (err == cudaSuccess)
        kern<<<grid, kThreadsP, smem, st>>>(nullptr, (const __nv_bfloat16*)a_hi, (const __nv_bfloat16*)a_lo,
                                            (const __nv_bfloat16*)b_hi, (const __nv_bfloat16*)b_lo, out, bias, residual, p,
                                            bn_p);
    } else {
      auto kern = conv_tc_persist_kernel<MODE, false, B>;
      if constexpr (MODE == 0 && B <= 64)
        if (bn) kern = conv_tc_persist_kernel<0, false, B, true>;
      err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (err == cudaSuccess)
        kern<<<grid, kThreadsP, smem, st>>>(src, nullptr, nullptr, (const __nv_bfloat16*)b_hi, (const __nv_bfloat16*)b_lo,
                                            out, bias, residual, p, bn_p);
    }
  });
  PF_CUDA(err);
  PF_CHECK_LAUNCH(who);
  return PF_OK;
}

template <int MODE>
int launch_tc(const TcGeom& g, const float* src, const void* a_hi, const void* a_lo, const void* b_hi, const void* b_lo,
              float* out, int accumulate, const float* bias, int relu, const float* residual, cudaStream_t st,
              const char* who, const pf_tc_bn_out* bn = nullptr) {
  const int64_t M64 = (MODE == 0) ? (int64_t)g.N * g.P * g.Q : (int64_t)g.N * g.H * g.W;
  PF_REQUIRE(M64 < (1ll << 31), "%s: too many rows", who);
  TcP p;
  memset(&p, 0, sizeof(p));
  p.g = g;
  p.M = (int)M64;
  p.Ng = (MODE == 0) ? g.K : g.C;
  p.Kdim = (MODE == 0) ? g.R * g.S * g.C : g.R * g.S * g.K;
  p.Kpad = pad64(p.Kdim);
  p.nk = p.Kpad / BK;
  p.accumulate = accumulate;
  p.relu = relu;
  const int CC = (MODE == 0) ? g.C : g.K;
  const int hw = (MODE == 0) ? g.P * g.Q : g.H * g.W, wq = (MODE == 0) ? g.Q : g.W;
  p.d_hw = make_fastdiv((uint32_t)hw);
  p.d_w = make_fastdiv((uint32_t)wq);
  p.d_cc = make_fastdiv((uint32_t)CC);
  p.d_s = make_fastdiv((uint32_t)g.S);
  p.cblocks = std::max(1, g.K / BK);
  p.d_cblocks = make_fastdiv((uint32_t)p.cblocks);
  p.m_tiles = (p.M + TM - 1) / TM;
  if (MODE == 1 && (g.sh > 1 || g.sw > 1) && g.sh * g.sw <= kMaxClasses && g.R * g.S <= kMaxTaps && g.K % BK == 0 &&
      env_int("PF_TC_CLASSES", 1)) {
    // pixel-parity classes of the strided dgrad
    int tiles = 0;
    for (int ph = 0; ph < g.sh; ++ph)
      for (int pw = 0; pw < g.sw; ++pw) {
        if (ph >= g.H || pw >= g.W) continue;
        TcClass& k = p.cls[p.ncls];
        k.ph = ph;
        k.pw = pw;
        k.Hc = (g.H - ph + g.sh - 1) / g.sh;
        k.Wc = (g.W - pw + g.sw - 1) / g.sw;
        k.Mc = g.N * k.Hc * k.Wc;
        k.tile_begin = tiles;
        k.d_hw = make_fastdiv((uint32_t)(k.Hc * k.Wc));
        k.d_w = make_fastdiv((uint32_t)k.Wc);
        k.ntaps = 0;
        for (int r = 0; r < g.R; ++r) {
          const int nh = ph + g.pt - r;
          if (((nh % g.sh) + g.sh) % g.sh != 0) continue;
          for (int q = 0; q < g.S; ++q) {
            const int nw = pw + g.pl - q;
            if (((nw % g.sw) + g.sw) % g.sw != 0) continue;
            k.eh[k.ntaps] = (int8_t)(nh / g.sh);
            k.ew[k.ntaps] = (int8_t)(nw / g.sw);
            k.tap[k.ntaps] = (int8_t)(r * g.S + q);
            ++k.ntaps;
          }
        }
        if (k.ntaps == 0 && accumulate) continue;      // dx += 0: nothing to do for this class
        tiles += (k.Mc + TM - 1) / TM;
        ++p.ncls;
      }
    p.m_tiles = tiles;
    return launch_persist<2>(g, p, src, a_hi, a_lo, b_hi, b_lo, out, bias, residual, st, who, nullptr);
  }
  return launch_persist<MODE>(g, p, src, a_hi, a_lo, b_hi, b_lo, out, bias, residual, st, who, bn);
}

// ---------------------------------------------------------------------------------------------
// u8 forward for the shapes the TMA-fed u8 kernel does not take (Cin or Cout a multiple of 16 but not of 64): both
// operands are the quantizers' unsigned 8-bit levels (pf_conv2d_u8_fwd), activations [N, H, W, Cin], weights
// [Cout][R*S*Cin].  The structure is conv_tc_persist_kernel's with pre-made operands: warps 8-15 copy each k-stage with
// cp.async straight into 128B-swizzled tiles (one 16-byte chunk = 16 channels of one filter tap, so any Cin % 16 == 0
// decodes per chunk; chunks past R*S*Cin are zero-filled), warps 0-7 are two m64 warpgroups.  A k-stage is 128 levels
// per row, i.e. four k32 slices at the 32-byte steps the bf16 kernel's k16 slices take; each slice is one
// u8 x u8 -> s32 wgmma, so S = sum q_a q_w is exact.  The epilogue is the TMA u8 kernel's: AFF 2 with weight centre 0
// (the rank-1 term from the channel sums J), bias, ReLU, residual and optionally the folded inference batch norm.
constexpr int BKU = 128;                         // u8 levels per k-stage and row
struct U8P {
  TcGeom g;
  int M, Ng, Kdim, nk, n_stages, n_tiles, total_tiles, relu, nseg;
  FastDiv d_hw, d_w, d_c, d_s, d_ntiles;
  EpiAff aff;
  const pf_tc_act_hdr* hdr;
  const float* csum;
};

// J of one GEMM row: the sum of the stored activation levels under the row's filter window (origin
// (oh0, ow0), R x S taps) from the per-pixel channel-segment sums `cimg` of the row's image (src_h x src_w pixels x
// nseg).  The (tap, segment) terms are independent loads, issued four at a time (branch-free; the terms are integers
// below 2^24, so the order of the additions does not change the result).  The TMA-fed u8 kernel forms the same sum in
// its consumer.
__device__ __forceinline__ float window_level_sum(const float* __restrict__ cimg, int nseg, int R, int S, FastDiv d_s,
                                                  int src_h, int src_w, int oh0, int ow0) {
  const int total = R * S * nseg;
  auto term = [&](int u) -> float {
    if (u >= total) return 0.f;
    const int t = u / nseg, g = u - t * nseg;
    const int r = (int)fdiv((uint32_t)t, d_s), s_ = t - r * S;
    const int ih = oh0 + r, iw = ow0 + s_;
    const bool ok = (unsigned)ih < (unsigned)src_h && (unsigned)iw < (unsigned)src_w;
    return ok ? __ldg(cimg + ((size_t)ih * src_w + iw) * nseg + g) : 0.f;
  };
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  for (int u = 0; u < total; u += 4) {
    const float v0 = term(u), v1 = term(u + 1), v2 = term(u + 2), v3 = term(u + 3);
    a0 += v0; a1 += v1; a2 += v2; a3 += v3;
  }
  return (a0 + a1) + (a2 + a3);
}

template <int BN, bool BNO>
__global__ void __launch_bounds__(kThreadsP, 1)
conv_u8_persist_kernel(const uint8_t* __restrict__ a_g, const uint8_t* __restrict__ b_g, float* __restrict__ out,
                       const float* __restrict__ bias, const float* __restrict__ residual,
                       const __grid_constant__ U8P p, const __grid_constant__ pf_tc_bn_out bn) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const TcGeom& g = p.g;
  constexpr uint32_t a_bytes = TM * BKU, b_bytes = (uint32_t)BN * BKU, stage_bytes = a_bytes + b_bytes;
  float* acc_s = reinterpret_cast<float*>(smem + (size_t)p.n_stages * stage_bytes);
  long long* rowoff_all = reinterpret_cast<long long*>(acc_s + TM * acc_pitch(BN));
  float* jrow_all = reinterpret_cast<float*>(rowoff_all + kMmaWarps * 32);
  float* aff_tab = jrow_all + kMmaWarps * 32;    // e1 at c, e2 at 256 + c; BNO: bn_table at 512
  __shared__ uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int s = 0; s < p.n_stages; ++s) {
      mbar_init(&full_bar[s], kProdWarps * 32);
      mbar_init(&empty_bar[s], kMmaWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int first_tile = blockIdx.x, tile_step = gridDim.x;

  if (warp >= kMmaWarps) {
    // ============ producers: thread = 16-byte chunk l8 of rows rgrp + 32 i (A) and rgrp + 32 j < BN (B) ============
    const int pt_ = tid - kMmaWarps * 32;
    const int l8 = pt_ & 7, rgrp = pt_ >> 3;
    const uint32_t chunk_off = (((uint32_t)l8) ^ (uint32_t)(rgrp & 7)) << 4;
    uint32_t it = 0;
    for (int tile = first_tile; tile < p.total_tiles; tile += tile_step) {
      const int mt = (int)fdiv((uint32_t)tile, p.d_ntiles);
      const int n0 = (tile - mt * p.n_tiles) * BN;
      // this thread's rows of A: (image, window origin), or -1 past the last row
      int img[4], oh[4], ow[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int m = mt * TM + rgrp + 32 * i;
        img[i] = -1;
        if (m < p.M) {
          img[i] = (int)fdiv((uint32_t)m, p.d_hw);
          const int rem = m - img[i] * g.P * g.Q;
          const int y = (int)fdiv((uint32_t)rem, p.d_w);
          oh[i] = y * g.sh - g.pt;
          ow[i] = (rem - y * g.Q) * g.sw - g.pl;
        }
      }
      for (int ks = 0; ks < p.nk; ++ks, ++it) {
        const uint32_t s = it % (uint32_t)p.n_stages;
        mbar_wait(&empty_bar[s], ((it / (uint32_t)p.n_stages) & 1u) ^ 1u);
        const int kk = ks * BKU + l8 * 16;
        const bool kok = kk < p.Kdim;
        const int tap = (int)fdiv((uint32_t)kk, p.d_c), c = kk - tap * g.C;
        const int r = (int)fdiv((uint32_t)tap, p.d_s), q = tap - r * g.S;
        const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes), sb = sa + a_bytes;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int ih = oh[i] + r, iw = ow[i] + q;
          const bool ok = kok && img[i] >= 0 && (unsigned)ih < (unsigned)g.H && (unsigned)iw < (unsigned)g.W;
          const size_t o = ok ? (((size_t)img[i] * g.H + ih) * g.W + iw) * g.C + c : 0;
          const uint32_t dst = sa + (uint32_t)(rgrp + 32 * i) * BKU + chunk_off;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(a_g + o), "r"(ok ? 16u : 0u) : "memory");
        }
        for (int br = rgrp; br < BN; br += 32) {
          const bool ok = kok && n0 + br < p.Ng;
          const size_t o = ok ? (size_t)(n0 + br) * p.Kdim + kk : 0;
          const uint32_t dst = sb + (uint32_t)br * BKU + chunk_off;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(b_g + o), "r"(ok ? 16u : 0u) : "memory");
        }
        // the barrier arrival fires when every cp.async issued so far by this thread has landed
        asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(&full_bar[s])) : "memory");
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else {
    // ============================ MMA warpgroups + epilogue (warps 0-7) ============================
    const int wg = warp >> 2;
    long long* rowoff = rowoff_all + warp * 32;
    float* jrow = jrow_all + warp * 32;
    // u8 levels stand for scale * level only when the tensor's minimum is 0 (header: 1 plane); otherwise the output
    // is NaN rather than silently wrong
    float a_s = __ldg(&p.hdr->scale);
    if (__ldg(&p.hdr->nplanes) != 1) a_s = __int_as_float(0x7fc00000);
    uint32_t it = 0;
    for (int tile = first_tile; tile < p.total_tiles; tile += tile_step) {
      const int mt = (int)fdiv((uint32_t)tile, p.d_ntiles);
      const int n0 = (tile - mt * p.n_tiles) * BN;
      int acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0;
      uint32_t prev = 0;
      for (int ks = 0; ks < p.nk; ++ks, ++it) {
        const uint32_t s = it % (uint32_t)p.n_stages;
        mbar_wait(&full_bar[s], (it / (uint32_t)p.n_stages) & 1u);
        fence_proxy_async_smem();              // cp.async writes -> visible to the tensor core (async proxy)
        const uint32_t base = smem_u32(smem + (size_t)s * stage_bytes);
        const uint32_t a0 = base + (uint32_t)wg * 64 * BKU, b0 = base + a_bytes;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BKU / 32; ++kk)
          WgmmaU8<BN>::mma(acc, make_smem_desc(a0 + kk * 32, 16, 1024), make_smem_desc(b0 + kk * 32, 16, 1024));
        wgmma_commit();
        wgmma_wait<1>(acc);                    // the previous stage's MMAs have completed: release it
        if (ks > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = s;
      }
      wgmma_wait<0>(acc);
      if (p.nk > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      const int m = mt * TM + (warp & 3) * 32 + lane;
      long long off = -1;
      float my_j = 0.f;
      if (m < p.M) {
        off = (long long)m * p.Ng;
        const int im = (int)fdiv((uint32_t)m, p.d_hw);
        const int rem = m - im * g.P * g.Q;
        const int y = (int)fdiv((uint32_t)rem, p.d_w), x = rem - y * g.Q;
        my_j = window_level_sum(p.csum + (size_t)im * g.H * g.W * p.nseg, p.nseg, g.R, g.S, p.d_s, g.H, g.W,
                                y * g.sh - g.pt, x * g.sw - g.pl);
      }
      // the accumulator tile and the columns' constants (e1 = s_a alpha_c / k_w, e2 = s_a beta_c; weight centre 0)
      named_bar_sync(1, kMmaWarps * 32);
      wgmma_store_acc<BN>(acc, acc_s, acc_pitch(BN), 64 * wg, tid & 127);
      for (int c = tid; c < BN; c += kMmaWarps * 32) {
        const bool cok = n0 + c < p.Ng;
        const int bi = p.aff.per_channel ? n0 + c : 0;
        const float al = cok ? __ldg(p.aff.w_alpha + bi) : 0.f, be = cok ? __ldg(p.aff.w_beta + bi) : 0.f;
        aff_tab[c] = al * p.aff.w_rk * a_s;
        aff_tab[256 + c] = be * a_s;
      }
      if (BNO) bn_table(bn, aff_tab + 512, n0, BN, p.Ng, tid, kMmaWarps * 32);
      named_bar_sync(1, kMmaWarps * 32);
      epilogue_tile_a<2, BNO>(acc_s, warp, off, rowoff, out, residual, bias, p.relu, n0, BN, p.Ng, lane, nullptr, p.aff,
                              my_j, jrow, bn, aff_tab);
    }
  }
}

int launch_u8(const TcGeom& g, const pf_tc_act& a, const pf_tc_wt& w, float* out, const float* bias, int relu,
              const float* residual, const pf_tc_bn_out* bn, cudaStream_t st, const char* who) {
  const int64_t M64 = (int64_t)g.N * g.P * g.Q;
  PF_REQUIRE(M64 < (1ll << 31), "%s: too many rows", who);
  U8P p;
  memset(&p, 0, sizeof(p));
  p.g = g;
  p.M = (int)M64;
  p.Ng = g.K;
  p.Kdim = g.R * g.S * g.C;
  p.nk = (p.Kdim + BKU - 1) / BKU;
  p.relu = relu;
  p.nseg = a.nseg;
  p.d_hw = make_fastdiv((uint32_t)(g.P * g.Q));
  p.d_w = make_fastdiv((uint32_t)g.Q);
  p.d_c = make_fastdiv((uint32_t)g.C);
  p.d_s = make_fastdiv((uint32_t)g.S);
  p.aff.w_alpha = w.alpha;
  p.aff.w_beta = w.beta;
  p.aff.per_channel = w.per_channel;
  p.aff.w_rk = 1.f / (float)((1 << w.bits) - 1);
  p.aff.w_centre = 0.f;
  p.hdr = a.hdr;
  p.csum = a.csum;
  // tile width: the widest the accumulators allow; the folded batch norm's epilogue does not fit the registers of this
  // 512-thread kernel beside a 128-wide tile (as in launch_persist)
  int BN = g.K >= 128 ? 128 : (g.K >= 64 ? 64 : (g.K >= 32 ? 32 : 16));
  if (bn && BN > 64) BN = 64;
  p.n_tiles = (g.K + BN - 1) / BN;
  p.total_tiles = (int)((M64 + TM - 1) / TM) * p.n_tiles;
  p.d_ntiles = make_fastdiv((uint32_t)p.n_tiles);
  const int stage = (TM + BN) * BKU;
  const int fixed = epi_fixed_bytes(BN) + (512 + 4 * kMaxBN) * 4;   // + e1 / e2 and the batch norm's constants
  p.n_stages = std::min(kMaxStages, (kSmemLimit - fixed) / stage);
  PF_REQUIRE(p.n_stages >= 2, "%s: shared-memory plan failed (BN %d)", who, BN);
  const size_t smem = (size_t)p.n_stages * stage + fixed;
  const int grid = std::min(p.total_tiles, PF_NUM_SMS);
  record_plan(pf_tc_plan{0, 0, 0, 0, BN, 2, 1, 1, 0, 0, 0, p.n_stages, p.total_tiles, grid, 0, 0});
  if (p.total_tiles == 0) return PF_OK;
  pf_tc_bn_out bn_p{};
  if (bn) bn_p = *bn;
  cudaError_t err = cudaSuccess;
  with_bn(BN, [&](auto bn_c) {
    constexpr int B = decltype(bn_c)::value;
    auto kern = conv_u8_persist_kernel<B, false>;
    if constexpr (B <= 64)
      if (bn) kern = conv_u8_persist_kernel<B, true>;
    err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err == cudaSuccess)
      kern<<<grid, kThreadsP, smem, st>>>((const uint8_t*)a.plane0, (const uint8_t*)w.plane0, out, bias, residual, p, bn_p);
  });
  PF_CUDA(err);
  PF_CHECK_LAUNCH(who);
  return PF_OK;
}

// multi-tensor split-K reduction: the partials of every wgrad of a step in ONE launch (kind-0 work items)
__global__ void __launch_bounds__(256)
tc_splitk_reduce_multi_kernel(const pf_tc_reduce_seg* __restrict__ segs, const pf_work* __restrict__ work) {
  const pf_work wk = work[blockIdx.x];
  const pf_tc_reduce_seg sg = segs[wk.seg];
  for (int64_t i = wk.start + (int64_t)threadIdx.x * 4; i < wk.start + wk.count; i += 1024) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int z = 0; z < sg.splits; ++z) {
      const float4 v = *reinterpret_cast<const float4*>(sg.partial + (size_t)z * sg.n + i);
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    *reinterpret_cast<float4*>(sg.out + i) = a;
  }
}

inline int64_t wg_align(int64_t b) { return (b + 255) / 256 * 256; }

// tile width, split-K factor and stage count of the persistent wgrad
inline void wgrad_plan(const TcGeom& g, WgP* pp) {
  WgP& p = *pp;
  memset(&p, 0, sizeof(p));
  p.g = g;
  p.Mtot = g.R * g.S * g.C;
  p.Npix = g.N * g.P * g.Q;
  int BN = g.K >= 128 ? 128 : 64;
  const int forced = env_int("PF_TC_WGRAD_BN", 0);
  if ((forced == 64 || forced == 128) && forced <= g.K) BN = forced;
  p.BN = BN;
  p.m_tiles = (p.Mtot + TM - 1) / TM;
  p.n_tiles = (g.K + BN - 1) / BN;
  p.tiles = p.m_tiles * p.n_tiles;
  // enough units to fill the SMs a few times over, but at least 8 k-stages (512 pixels) per unit
  // (rounded DOWN: total units just under a whole number of waves over the SMs)
  int splits = (env_int("PF_TC_WGRAD_WAVES", 1) * PF_NUM_SMS) / p.tiles;
  const int max_by_k = (p.Npix + 8 * BK - 1) / (8 * BK);
  splits = std::max(1, std::min(std::min(splits, max_by_k), PF_CONV_TC_WGRAD_MAX_SPLITS));
  int pps = (p.Npix + splits - 1) / splits;
  pps = (pps + BK - 1) / BK * BK;
  p.pps = pps;
  p.splits = (p.Npix + pps - 1) / pps;
  p.total_units = p.tiles * p.splits;
  const int fixed = epi_fixed_bytes(BN);
  p.n_stages = std::max(1, std::min(kMaxStages, (kSmemLimit - fixed) / (2 * BK * TM * 2 + 2 * BK * BN * 2)));
  p.d_pq = make_fastdiv((uint32_t)(g.P * g.Q));
  p.d_q = make_fastdiv((uint32_t)g.Q);
  p.d_c = make_fastdiv((uint32_t)g.C);
  p.d_s = make_fastdiv((uint32_t)g.S);
  p.d_tiles = make_fastdiv((uint32_t)p.tiles);
  p.d_ntiles = make_fastdiv((uint32_t)p.n_tiles);
}

}  // namespace

extern "C" {

int pf_conv2d_tc_supported(const pf_conv_desc* d) {
  if (!d) return 0;
  return (d->c % 16 == 0) && (d->k % 16 == 0) && d->c >= 16 && d->k >= 16;
}

int64_t pf_conv2d_tc_weight_elems(const pf_conv_desc* d, int dgrad) {
  if (!d) return 0;
  if (dgrad) return (int64_t)d->c * pad64((int64_t)d->r * d->s * d->k);
  return (int64_t)d->k * pad64((int64_t)d->r * d->s * d->c);
}

int pf_conv2d_tc_prep_weight(const pf_conv_desc* d, const float* w_dev, void* fwd_hi_dev, void* fwd_lo_dev,
                             void* dgrad_hi_dev, void* dgrad_lo_dev, void* stream) {
  TcGeom g;
  int rc = tc_geom(d, &g, "pf_conv2d_tc_prep_weight");
  if (rc) return rc;
  PF_REQUIRE(w_dev && fwd_hi_dev && fwd_lo_dev, "pf_conv2d_tc_prep_weight: null pointer");
  PF_REQUIRE((dgrad_hi_dev == nullptr) == (dgrad_lo_dev == nullptr), "pf_conv2d_tc_prep_weight: dgrad buffers come in pairs");
  const int kpf = pad64((int64_t)g.R * g.S * g.C), kpd = pad64((int64_t)g.R * g.S * g.K);
  cudaStream_t st = (cudaStream_t)stream;
  // padding columns must be zero: the buffers are zero-filled once by the caller at allocation time
  const int64_t total = (int64_t)g.R * g.S * g.C * g.K;
  int64_t blocks = (total + 255) / 256;
  if (blocks > PF_NUM_SMS * 8) blocks = PF_NUM_SMS * 8;
  tc_prep_weight_kernel<<<(unsigned)blocks, 256, 0, st>>>(w_dev, g.R * g.S, g.C, g.K, kpf, kpd,
                                                         (__nv_bfloat16*)fwd_hi_dev, (__nv_bfloat16*)fwd_lo_dev,
                                                         (__nv_bfloat16*)dgrad_hi_dev, (__nv_bfloat16*)dgrad_lo_dev);
  PF_CHECK_LAUNCH("pf_conv2d_tc_prep_weight");
  return PF_OK;
}

int pf_conv2d_tc_prep_weights_multi(const pf_tc_prep_seg* segs_dev, const pf_work* work_dev, int n_work, void* stream) {
  PF_REQUIRE(n_work >= 0, "pf_conv2d_tc_prep_weights_multi: n_work < 0");
  if (n_work == 0) return PF_OK;
  PF_REQUIRE(segs_dev && work_dev, "pf_conv2d_tc_prep_weights_multi: null pointer");
  tc_prep_weights_multi_kernel<<<(unsigned)n_work, 256, 0, (cudaStream_t)stream>>>(segs_dev, work_dev);
  PF_CHECK_LAUNCH("pf_conv2d_tc_prep_weights_multi");
  return PF_OK;
}

static int check_bn_out(const pf_tc_bn_out* bn, const char* who) {
  PF_REQUIRE(bn->mean && bn->var && bn->gamma && bn->beta && (bn->y || bn->hi), "%s: batch norm: null pointer", who);
  PF_REQUIRE((bn->hi == nullptr) == (bn->lo == nullptr), "%s: batch norm: planes come in pairs", who);
  PF_REQUIRE(bn->eps >= 0.f && bn->act >= 0 && bn->act <= 2, "%s: batch norm: eps < 0 or act not in 0..2", who);
  PF_REQUIRE((((uintptr_t)bn->mean | (uintptr_t)bn->var | (uintptr_t)bn->gamma | (uintptr_t)bn->beta |
               (uintptr_t)bn->y) & 15) == 0 && (((uintptr_t)bn->hi | (uintptr_t)bn->lo) & 7) == 0,
             "%s: batch norm: alignment", who);
  return PF_OK;
}

static int tc_fwd_impl(const pf_conv_desc* d, const float* x_dev, const void* x_hi, const void* x_lo, const void* w_hi_dev,
                       const void* w_lo_dev, const float* bias_dev, int relu, const float* residual_dev, float* y_dev,
                       void* stream, const char* who, const pf_tc_bn_out* bn = nullptr) {
  TcGeom g;
  int rc = tc_geom(d, &g, who);
  if (rc) return rc;
  PF_REQUIRE(pf_conv2d_tc_supported(d), "%s: Cin and Cout must be multiples of 16", who);
  PF_REQUIRE((x_dev || (x_hi && x_lo)) && w_hi_dev && w_lo_dev && y_dev, "%s: null pointer", who);
  PF_REQUIRE((((uintptr_t)x_dev | (uintptr_t)x_hi | (uintptr_t)x_lo | (uintptr_t)y_dev | (uintptr_t)w_hi_dev |
               (uintptr_t)w_lo_dev | (uintptr_t)residual_dev | (uintptr_t)bias_dev) & 15) == 0,
             "%s: 16-byte alignment required", who);
  if (bn) {
    rc = check_bn_out(bn, who);
    if (rc) return rc;
  }
  if (x_hi && conv_tma_eligible(0, g)) {
    const pf_tc_act a{x_hi, x_lo, nullptr, nullptr, 0, 0};
    const pf_tc_wt w{w_hi_dev, w_lo_dev, nullptr, nullptr, 0, 0};
    return conv_tma_launch(0, g, a, w, y_dev, 0, bias_dev, relu, residual_dev, (cudaStream_t)stream, who, bn);
  }
  return launch_tc<0>(g, x_dev, x_hi, x_lo, w_hi_dev, w_lo_dev, y_dev, 0, bias_dev, relu, residual_dev,
                      (cudaStream_t)stream, who, bn);
}

static int tc_dgrad_impl(const pf_conv_desc* d, const float* dy_dev, const void* dy_hi, const void* dy_lo,
                         const void* wd_hi_dev, const void* wd_lo_dev, int accumulate, float* dx_dev, void* stream,
                         const char* who) {
  TcGeom g;
  int rc = tc_geom(d, &g, who);
  if (rc) return rc;
  PF_REQUIRE(pf_conv2d_tc_supported(d), "%s: Cin and Cout must be multiples of 16", who);
  PF_REQUIRE((dy_dev || (dy_hi && dy_lo)) && wd_hi_dev && wd_lo_dev && dx_dev, "%s: null pointer", who);
  PF_REQUIRE((((uintptr_t)dy_dev | (uintptr_t)dy_hi | (uintptr_t)dy_lo | (uintptr_t)dx_dev | (uintptr_t)wd_hi_dev |
               (uintptr_t)wd_lo_dev) & 15) == 0, "%s: 16-byte alignment required", who);
  if (dy_hi && conv_tma_eligible(1, g)) {
    const pf_tc_act a{dy_hi, dy_lo, nullptr, nullptr, 0, 0};
    const pf_tc_wt w{wd_hi_dev, wd_lo_dev, nullptr, nullptr, 0, 0};
    return conv_tma_launch(1, g, a, w, dx_dev, accumulate, nullptr, 0, nullptr, (cudaStream_t)stream, who);
  }
  return launch_tc<1>(g, dy_dev, dy_hi, dy_lo, wd_hi_dev, wd_lo_dev, dx_dev, accumulate, nullptr, 0, nullptr,
                      (cudaStream_t)stream, who);
}

int pf_conv2d_tc_fwd(const pf_conv_desc* d, const float* x_dev, const void* w_hi_dev, const void* w_lo_dev,
                     const float* bias_dev, int relu, const float* residual_dev, float* y_dev, void* stream) {
  PF_REQUIRE(x_dev != nullptr, "pf_conv2d_tc_fwd: null pointer");
  return tc_fwd_impl(d, x_dev, nullptr, nullptr, w_hi_dev, w_lo_dev, bias_dev, relu, residual_dev, y_dev, stream,
                     "pf_conv2d_tc_fwd");
}

int pf_conv2d_tc_fwd_planes(const pf_conv_desc* d, const void* x_hi_dev, const void* x_lo_dev, const void* w_hi_dev,
                            const void* w_lo_dev, const float* bias_dev, int relu, const float* residual_dev,
                            float* y_dev, void* stream) {
  PF_REQUIRE(x_hi_dev && x_lo_dev, "pf_conv2d_tc_fwd_planes: null pointer");
  return tc_fwd_impl(d, nullptr, x_hi_dev, x_lo_dev, w_hi_dev, w_lo_dev, bias_dev, relu, residual_dev, y_dev, stream,
                     "pf_conv2d_tc_fwd_planes");
}

int pf_conv2d_tc_fwd_bn(const pf_conv_desc* d, const float* x_dev, const void* w_hi_dev, const void* w_lo_dev,
                        const float* bias_dev, int relu, const float* residual_dev, float* y_dev, const pf_tc_bn_out* bn,
                        void* stream) {
  PF_REQUIRE(x_dev != nullptr && bn != nullptr, "pf_conv2d_tc_fwd_bn: null pointer");
  return tc_fwd_impl(d, x_dev, nullptr, nullptr, w_hi_dev, w_lo_dev, bias_dev, relu, residual_dev, y_dev, stream,
                     "pf_conv2d_tc_fwd_bn", bn);
}

int pf_conv2d_tc_fwd_planes_bn(const pf_conv_desc* d, const void* x_hi_dev, const void* x_lo_dev, const void* w_hi_dev,
                               const void* w_lo_dev, const float* bias_dev, int relu, const float* residual_dev,
                               float* y_dev, const pf_tc_bn_out* bn, void* stream) {
  PF_REQUIRE(x_hi_dev && x_lo_dev && bn, "pf_conv2d_tc_fwd_planes_bn: null pointer");
  return tc_fwd_impl(d, nullptr, x_hi_dev, x_lo_dev, w_hi_dev, w_lo_dev, bias_dev, relu, residual_dev, y_dev, stream,
                     "pf_conv2d_tc_fwd_planes_bn", bn);
}

int pf_conv2d_tc_dgrad(const pf_conv_desc* d, const float* dy_dev, const void* wd_hi_dev, const void* wd_lo_dev,
                       int accumulate, float* dx_dev, void* stream) {
  PF_REQUIRE(dy_dev != nullptr, "pf_conv2d_tc_dgrad: null pointer");
  return tc_dgrad_impl(d, dy_dev, nullptr, nullptr, wd_hi_dev, wd_lo_dev, accumulate, dx_dev, stream, "pf_conv2d_tc_dgrad");
}

int pf_conv2d_tc_dgrad_planes(const pf_conv_desc* d, const void* dy_hi_dev, const void* dy_lo_dev, const void* wd_hi_dev,
                              const void* wd_lo_dev, int accumulate, float* dx_dev, void* stream) {
  PF_REQUIRE(dy_hi_dev && dy_lo_dev, "pf_conv2d_tc_dgrad_planes: null pointer");
  return tc_dgrad_impl(d, nullptr, dy_hi_dev, dy_lo_dev, wd_hi_dev, wd_lo_dev, accumulate, dx_dev, stream,
                       "pf_conv2d_tc_dgrad_planes");
}

int pf_conv2d_tc_wgrad_supported(const pf_conv_desc* d) {
  if (!d) return 0;
  return (d->c % 16 == 0) && (d->k % 64 == 0) && d->c >= 16;
}

int64_t pf_conv2d_tc_wgrad_workspace_bytes(const pf_conv_desc* d) {
  TcGeom g;
  if (!d || tc_geom(d, &g, "pf_conv2d_tc_wgrad_workspace_bytes")) return 0;
  WgP p;
  wgrad_plan(g, &p);
  // split-K partials + the split-bf16 planes of x and dy
  return (int64_t)p.splits * p.Mtot * g.K * 4 + wg_align((int64_t)g.N * g.H * g.W * g.C * 4) +
         wg_align((int64_t)g.N * g.P * g.Q * g.K * 4);
}

int64_t pf_conv2d_tc_wgrad_planes_workspace_bytes(const pf_conv_desc* d) {
  TcGeom g;
  if (!d || tc_geom(d, &g, "pf_conv2d_tc_wgrad_planes_workspace_bytes")) return 0;
  WgP p;
  wgrad_plan(g, &p);
  return (int64_t)p.splits * p.Mtot * g.K * 4;
}

int pf_conv2d_tc_wgrad_splits(const pf_conv_desc* d) {
  TcGeom g;
  if (!d || tc_geom(d, &g, "pf_conv2d_tc_wgrad_splits")) return 0;
  WgP p;
  wgrad_plan(g, &p);
  return p.splits;
}

int pf_conv2d_tc_wgrad_reduce_multi(const pf_tc_reduce_seg* segs_dev, const pf_work* work_dev, int n_work, void* stream) {
  PF_REQUIRE(n_work >= 0, "pf_conv2d_tc_wgrad_reduce_multi: n_work < 0");
  if (n_work == 0) return PF_OK;
  PF_REQUIRE(segs_dev && work_dev, "pf_conv2d_tc_wgrad_reduce_multi: null pointer");
  tc_splitk_reduce_multi_kernel<<<(unsigned)n_work, 256, 0, (cudaStream_t)stream>>>(segs_dev, work_dev);
  PF_CHECK_LAUNCH("pf_conv2d_tc_wgrad_reduce_multi");
  return PF_OK;
}

int pf_split_bf16(const float* src_dev, void* hi_dev, void* lo_dev, int64_t n, void* stream) {
  PF_REQUIRE(n >= 0 && n % 8 == 0, "pf_split_bf16: n must be a non-negative multiple of 8");
  if (n == 0) return PF_OK;
  PF_REQUIRE(src_dev && hi_dev && lo_dev, "pf_split_bf16: null pointer");
  PF_REQUIRE((((uintptr_t)src_dev | (uintptr_t)hi_dev | (uintptr_t)lo_dev) & 15) == 0, "pf_split_bf16: 16-byte alignment required");
  int64_t blocks = (n / 8 + 255) / 256;
  if (blocks > PF_NUM_SMS * 16) blocks = PF_NUM_SMS * 16;
  split_bf16_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(src_dev, (__nv_bfloat16*)hi_dev, (__nv_bfloat16*)lo_dev, n / 8);
  PF_CHECK_LAUNCH("pf_split_bf16");
  return PF_OK;
}

static int tc_wgrad_impl(const pf_conv_desc* d, const pf_tc_act& x, const pf_tc_act& dy, float* ws_dev, float* dw_dev,
                         void* stream, const char* who) {
  TcGeom g;
  int rc = tc_geom(d, &g, who);
  if (rc) return rc;
  PF_REQUIRE(pf_conv2d_tc_wgrad_supported(d), "%s: needs Cin %% 16 == 0 and Cout %% 64 == 0", who);
  PF_REQUIRE(x.plane0 && dy.plane0 && dy.plane1 && ws_dev, "%s: null pointer", who);
  PF_REQUIRE((((uintptr_t)x.plane0 | (uintptr_t)x.plane1 | (uintptr_t)dy.plane0 | (uintptr_t)dy.plane1 | (uintptr_t)ws_dev |
               (uintptr_t)dw_dev) & 15) == 0, "%s: 16-byte alignment required", who);
  PF_REQUIRE((int64_t)g.N * g.P * g.Q < (1ll << 31), "%s: too many pixels", who);
  WgP p;
  wgrad_plan(g, &p);
  cudaStream_t st = (cudaStream_t)stream;
  float* partial = (p.splits == 1 && dw_dev) ? dw_dev : ws_dev;
  if (conv_tma_eligible(2, g)) {
    rc = conv_tma_wgrad_launch(g, x, dy, p.BN, p.pps, p.splits, partial, st, who);
    if (rc) return rc;
  } else {
    PF_REQUIRE(x.hdr == nullptr && x.plane1 != nullptr, "%s: quantizer-level operands need the TMA kernels (Cin %% 64 == 0)", who);
    const size_t smem = (size_t)p.n_stages * (2 * BK * TM * 2 + 2 * BK * p.BN * 2) + epi_fixed_bytes(p.BN);
    const int grid = std::min(p.total_units, PF_NUM_SMS);
    record_plan(pf_tc_plan{0, 0, 2, 0, p.BN, 0, 2, 2, 0, 0, 0, p.n_stages, p.total_units, grid, p.splits, p.pps});
    auto kern = p.BN == 128 ? conv_tc_wgrad_persist_kernel<128> : conv_tc_wgrad_persist_kernel<64>;
    PF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, kThreadsP, smem, st>>>((const __nv_bfloat16*)x.plane0, (const __nv_bfloat16*)x.plane1,
                                        (const __nv_bfloat16*)dy.plane0, (const __nv_bfloat16*)dy.plane1, partial, p);
    PF_CHECK_LAUNCH(who);
  }
  if (p.splits > 1 && dw_dev) {
    const int64_t n = (int64_t)p.Mtot * g.K;
    tc_splitk_reduce_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, st>>>(ws_dev, dw_dev, n, p.splits);
    PF_CHECK_LAUNCH(who);
  }
  return PF_OK;
}

int pf_conv2d_tc_wgrad_planes(const pf_conv_desc* d, const void* x_hi_dev, const void* x_lo_dev, const void* dy_hi_dev,
                              const void* dy_lo_dev, float* ws_dev, float* dw_dev, void* stream) {
  PF_REQUIRE(x_hi_dev && x_lo_dev, "pf_conv2d_tc_wgrad_planes: null pointer");
  const pf_tc_act x{x_hi_dev, x_lo_dev, nullptr, nullptr, 0, 0}, dy{dy_hi_dev, dy_lo_dev, nullptr, nullptr, 0, 0};
  return tc_wgrad_impl(d, x, dy, ws_dev, dw_dev, stream, "pf_conv2d_tc_wgrad_planes");
}

int pf_conv2d_tc_wgrad_ex(const pf_conv_desc* d, const pf_tc_act* x, const pf_tc_act* dy, float* ws_dev, float* dw_dev,
                          void* stream) {
  PF_REQUIRE(x && dy, "pf_conv2d_tc_wgrad_ex: null operand");
  return tc_wgrad_impl(d, *x, *dy, ws_dev, dw_dev, stream, "pf_conv2d_tc_wgrad_ex");
}

int pf_conv2d_tc_last_plan(pf_tc_plan* out) {
  PF_REQUIRE(out != nullptr, "pf_conv2d_tc_last_plan: null pointer");
  PF_REQUIRE(g_last_plan.seq > 0, "pf_conv2d_tc_last_plan: no tensor-core conv launch recorded yet");
  *out = g_last_plan;
  return PF_OK;
}

int pf_conv2d_tc_set_feed(int mode) {
  conv_tma_set_feed(mode);
  return PF_OK;
}

int pf_conv2d_tc_tma_supported(const pf_conv_desc* d, int pass) {
  TcGeom g;
  if (!d || pass < 0 || pass > 2 || tc_geom(d, &g, "pf_conv2d_tc_tma_supported")) return 0;
  if (pass == 2) return pf_conv2d_tc_wgrad_supported(d) && conv_tma_eligible(2, g);
  return pf_conv2d_tc_supported(d) && conv_tma_eligible(pass, g);
}

int pf_conv2d_tc_fwd_ex(const pf_conv_desc* d, const pf_tc_act* x, const pf_tc_wt* w, const float* bias_dev, int relu,
                        const float* residual_dev, float* y_dev, void* stream) {
  const char* who = "pf_conv2d_tc_fwd_ex";
  PF_REQUIRE(x && w && x->plane0 && w->plane0 && y_dev, "%s: null pointer", who);
  const bool plain = x->hdr == nullptr && x->plane1 != nullptr && w->alpha == nullptr && w->plane1 != nullptr;
  if (plain)
    return tc_fwd_impl(d, nullptr, x->plane0, x->plane1, w->plane0, w->plane1, bias_dev, relu, residual_dev, y_dev, stream, who);
  TcGeom g;
  int rc = tc_geom(d, &g, who);
  if (rc) return rc;
  PF_REQUIRE(pf_conv2d_tc_supported(d) && conv_tma_eligible(0, g),
             "%s: quantizer-level operands need the TMA kernels (Cin %% 64 == 0)", who);
  PF_REQUIRE((((uintptr_t)x->plane0 | (uintptr_t)x->plane1 | (uintptr_t)w->plane0 | (uintptr_t)w->plane1 | (uintptr_t)y_dev |
               (uintptr_t)residual_dev | (uintptr_t)bias_dev | (uintptr_t)w->alpha | (uintptr_t)w->beta) & 15) == 0,
             "%s: 16-byte alignment required", who);
  return conv_tma_launch(0, g, *x, *w, y_dev, 0, bias_dev, relu, residual_dev, (cudaStream_t)stream, who);
}

int pf_conv2d_u8_supported(const pf_conv_desc* d) {
  TcGeom g;
  if (!d || tc_geom(d, &g, "pf_conv2d_u8_supported")) return 0;
  return conv_tma_u8_eligible(g);
}

// the cp.async-fed u8 kernel: channel counts that are multiples of 16, and K = R*S*Cin small enough for the exact s32
// sum (K * 255^2 < 2^31)
static bool u8_narrow_eligible(const TcGeom& g) {
  return g.C % 16 == 0 && g.K % 16 == 0 && (int64_t)g.R * g.S * g.C <= 32768;
}

int pf_conv2d_u8_narrow_supported(const pf_conv_desc* d) {
  TcGeom g;
  if (!d || tc_geom(d, &g, "pf_conv2d_u8_narrow_supported")) return 0;
  return conv_tma_u8_eligible(g) || u8_narrow_eligible(g);
}

int pf_conv2d_u8_fwd(const pf_conv_desc* d, const pf_tc_act* x, const pf_tc_wt* w, const float* bias_dev, int relu,
                     const float* residual_dev, float* y_dev, const pf_tc_bn_out* bn, void* stream) {
  const char* who = "pf_conv2d_u8_fwd";
  PF_REQUIRE(x && w && x->plane0 && x->hdr && x->csum && w->plane0 && w->alpha && w->beta && y_dev, "%s: null pointer", who);
  PF_REQUIRE(x->plane1 == nullptr && w->plane1 == nullptr, "%s: u8 operands have one plane", who);
  PF_REQUIRE(x->nseg == (d ? (d->c + 127) / 128 : 0), "%s: nseg must be ceil(Cin / 128)", who);
  TcGeom g;
  int rc = tc_geom(d, &g, who);
  if (rc) return rc;
  const bool tma = conv_tma_u8_eligible(g);
  PF_REQUIRE(tma || u8_narrow_eligible(g),
             "%s: needs Cin %% 16 == 0, Cout %% 16 == 0 and R*S*Cin <= 32768 (or Cin, Cout %% 64 == 0, strides <= 8 and "
             "filters <= 16)", who);
  PF_REQUIRE((((uintptr_t)x->plane0 | (uintptr_t)w->plane0 | (uintptr_t)y_dev | (uintptr_t)residual_dev |
               (uintptr_t)bias_dev | (uintptr_t)w->alpha | (uintptr_t)w->beta) & 15) == 0 &&
                 ((uintptr_t)x->hdr & 7) == 0,
             "%s: 16-byte alignment required (header: 8)", who);
  if (bn) {
    rc = check_bn_out(bn, who);
    if (rc) return rc;
  }
  if (tma) return conv_tma_launch(0, g, *x, *w, y_dev, 0, bias_dev, relu, residual_dev, (cudaStream_t)stream, who, bn, true);
  PF_REQUIRE(w->bits >= 1 && w->bits <= 8, "%s: weight levels need 1..8 bits", who);
  return launch_u8(g, *x, *w, y_dev, bias_dev, relu, residual_dev, bn, (cudaStream_t)stream, who);
}

int pf_conv2d_tc_dgrad_ex(const pf_conv_desc* d, const pf_tc_act* dy, const pf_tc_wt* wd, int accumulate, float* dx_dev,
                          void* stream) {
  const char* who = "pf_conv2d_tc_dgrad_ex";
  PF_REQUIRE(dy && wd && dy->plane0 && wd->plane0 && dx_dev, "%s: null pointer", who);
  // pass 1 reduces over output channels: per-channel weight scales vary along the reduction, so weight levels have no
  // column-epilogue form (and the dgrad weight copies are split planes of the quantized values anyway)
  PF_REQUIRE(wd->alpha == nullptr, "%s: weight levels are not supported in dgrad; pass split-bf16 weight planes", who);
  const bool plain = dy->hdr == nullptr && dy->plane1 != nullptr && wd->plane1 != nullptr;
  if (plain)
    return tc_dgrad_impl(d, nullptr, dy->plane0, dy->plane1, wd->plane0, wd->plane1, accumulate, dx_dev, stream, who);
  TcGeom g;
  int rc = tc_geom(d, &g, who);
  if (rc) return rc;
  PF_REQUIRE(pf_conv2d_tc_supported(d) && conv_tma_eligible(1, g),
             "%s: quantizer-level operands need the TMA kernels (unit stride, Cout %% 64 == 0)", who);
  return conv_tma_launch(1, g, *dy, *wd, dx_dev, accumulate, nullptr, 0, nullptr, (cudaStream_t)stream, who);
}

int pf_conv2d_tc_wgrad(const pf_conv_desc* d, const float* x_dev, const float* dy_dev, float* ws_dev,
                       float* dw_dev, void* stream) {
  TcGeom g;
  int rc = tc_geom(d, &g, "pf_conv2d_tc_wgrad");
  if (rc) return rc;
  PF_REQUIRE(pf_conv2d_tc_wgrad_supported(d), "pf_conv2d_tc_wgrad: needs Cin %% 16 == 0 and Cout %% 64 == 0");
  PF_REQUIRE(x_dev && dy_dev && ws_dev && dw_dev, "pf_conv2d_tc_wgrad: null pointer");
  PF_REQUIRE((((uintptr_t)x_dev | (uintptr_t)dy_dev | (uintptr_t)ws_dev | (uintptr_t)dw_dev) & 15) == 0,
             "pf_conv2d_tc_wgrad: 16-byte alignment required");
  const int64_t np64 = (int64_t)g.N * g.P * g.Q;
  PF_REQUIRE(np64 < (1ll << 31), "pf_conv2d_tc_wgrad: too many pixels");
  // split both operands into bf16 planes inside the workspace, then the persistent planes kernel
  WgP p;
  wgrad_plan(g, &p);
  const int64_t nx = (int64_t)g.N * g.H * g.W * g.C, ny = np64 * g.K;
  uint8_t* base = reinterpret_cast<uint8_t*>(ws_dev) + (int64_t)p.splits * p.Mtot * g.K * 4;
  __nv_bfloat16* xh = reinterpret_cast<__nv_bfloat16*>(base);
  __nv_bfloat16* xl = xh + nx;
  __nv_bfloat16* yh = reinterpret_cast<__nv_bfloat16*>(base + wg_align(nx * 4));
  __nv_bfloat16* yl = yh + ny;
  rc = pf_split_bf16(x_dev, xh, xl, nx, stream);
  if (rc) return rc;
  rc = pf_split_bf16(dy_dev, yh, yl, ny, stream);
  if (rc) return rc;
  return pf_conv2d_tc_wgrad_planes(d, xh, xl, yh, yl, ws_dev, dw_dev, stream);
}

}  // extern "C"
