// pf_conv_tc.cuh — pieces shared by the wgmma convolution kernels (pf_conv_tc.cu: cp.async-fed, any channel
// count that is a multiple of 16; pf_conv_tma.cu: TMA-fed, channel counts that are multiples of 64):
// tile constants, geometry, exact division by runtime constants, the warpgroup main loop and the epilogue.
#pragma once
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "pf_common.cuh"
#include "pf_tc_common.cuh"

namespace pfconv {
using namespace pftc;

constexpr int TM = 128;      // GEMM rows per CTA (two m64 warpgroups)
constexpr int BK = 64;       // bf16 elements per k-stage (= one 128-byte swizzled row)
constexpr int kSmemLimit = 232448;   // 227 KB opt-in maximum of dynamic shared memory per CTA on sm_90

struct TcGeom {
  int N, H, W, C, K, R, S, P, Q, sh, sw, pt, pl;
};

struct FastDiv {
  uint32_t mul, shift;
};
inline FastDiv make_fastdiv(uint32_t d) {   // exact for 0 <= n < 2^31 (Granlund-Montgomery round-up method)
  FastDiv f;
  uint32_t s = 0;
  while ((1ull << s) < d) ++s;
  f.shift = s;
  f.mul = (uint32_t)((((1ull << 32) * ((1ull << s) - d)) / d) + 1);
  return f;
}
__device__ __forceinline__ uint32_t fdiv(uint32_t n, FastDiv f) { return (__umulhi(n, f.mul) + n) >> f.shift; }

inline int pad64(int64_t k) { return (int)((k + 63) / 64 * 64); }
inline int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return (v && *v) ? atoi(v) : dflt;
}
int tc_geom(const pf_conv_desc* d, TcGeom* g, const char* who);

// ---------------------------------------------------------------------------------------------------------
// Main loop and epilogue warps.  Warps 0-7 of every tensor-core kernel are two warpgroups.  In the cooperative kernels
// (cp.async-fed, TMA wgrad) warpgroup g issues the wgmma of GEMM rows [64 g, 64 g + 64) of the 128 x BN tile into
// registers; at the end of a tile both write their accumulators into one fp32 tile in shared memory (row pitch BN + 4
// floats), and the same 8 warps then run the epilogue from there: warp w owns rows [32 (w % 4), 32 (w % 4) + 32) and
// every other 32-column chunk starting at chunk w / 4.  The producers (cp.async warps or the TMA thread) keep filling
// the next tile's stages meanwhile.  The TMA fwd / dgrad kernel is a ping-pong instead (pf_conv_tma.cu): each
// warpgroup owns whole tiles and runs their epilogue alone, under the other warpgroup's MMAs.
constexpr int kMmaWarps = 8;
constexpr int kMaxBN = 128;                                    // 64 accumulator registers per thread and warpgroup
__host__ __device__ constexpr int acc_pitch(int BN) { return BN + 4; }
__host__ __device__ constexpr int acc_tile_bytes(int BN) { return TM * acc_pitch(BN) * 4; }
// accumulator tile + per-warp row-offset and J tables
__host__ __device__ constexpr int epi_fixed_bytes(int BN) { return 1024 + acc_tile_bytes(BN) + kMmaWarps * 32 * (8 + 4) + 256; }

// The MMAs of one 16-wide k-slice of one m64 row block:  A0 B0 (+ A0 B1 when NB == 2) (+ A1 B0 when NA == 2)  of the
// bf16 planes (hi / lo, or integer levels).  The plane counts are template parameters: a run-time test between two
// wgmmas makes ptxas end the chain there and re-arm the accumulator registers with an injected warpgroup.arrive (C7519).
template <int BN, int TMN, int NA, int NB>
__device__ __forceinline__ void wg_mma_kslice(float (&acc)[BN / 2], uint64_t da0, uint64_t da1, uint64_t db0,
                                              uint64_t db1) {
  Wgmma<BN>::template mma<TMN, TMN>(acc, da0, db0);
  if (NB == 2) Wgmma<BN>::template mma<TMN, TMN>(acc, da0, db1);
  if (NA == 2) Wgmma<BN>::template mma<TMN, TMN>(acc, da1, db0);
}

// One k-stage of MMAs of warpgroup `wg` (wtid = thread index inside the warpgroup is implied): per 16-wide k-slice
// the plane products of wg_mma_kslice.  a0 / a1 / b0 / b1 are the shared-memory addresses of the planes; a_kstep /
// b_kstep the byte step of one 16-wide k-slice; lbo / sbo the descriptor strides.
template <int BN, int TMN, int NA, int NB>
__device__ __forceinline__ void wg_mma_stage(float (&acc)[BN / 2], uint32_t a0, uint32_t a1, uint32_t b0, uint32_t b1,
                                             uint32_t a_kstep, uint32_t b_kstep, uint32_t lbo_a, uint32_t sbo_a,
                                             uint32_t lbo_b, uint32_t sbo_b) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < BK / 16; ++kk)
    wg_mma_kslice<BN, TMN, NA, NB>(acc, make_smem_desc(a0 + kk * a_kstep, lbo_a, sbo_a),
                                   make_smem_desc(a1 + kk * a_kstep, lbo_a, sbo_a),
                                   make_smem_desc(b0 + kk * b_kstep, lbo_b, sbo_b),
                                   make_smem_desc(b1 + kk * b_kstep, lbo_b, sbo_b));
  wgmma_commit();
}

// End of a tile's main loop: wait for the last MMAs, release their stage, and hand the accumulator to the epilogue
// through the shared tile.  Named barrier 1 spans the 8 MMA warps: the first one keeps this tile's stores behind the
// previous tile's epilogue reads, the second makes the stores visible to every epilogue warp.
template <int BN>
__device__ __forceinline__ void wg_tile_to_smem(float (&acc)[BN / 2], float* acc_s, int tid) {
  named_bar_sync(1, kMmaWarps * 32);
  wgmma_store_acc<BN>(acc, acc_s, acc_pitch(BN), 64 * (tid >> 7), tid & 127);
  named_bar_sync(1, kMmaWarps * 32);
}

// Epilogue of one 128 x BN accumulator tile by one warp: rows of this warp are `acc` + i * pitch (i < 32); the warp's
// lanes write 128-byte row segments to global.
// `extra` (residual / accumulate operand, same indexing as `out`) is prefetched one 32-column chunk ahead.
// EXTRA: 0 = none; 1 = extra operand prefetched one chunk ahead in registers; 2 = extra operand streamed through a
// per-warp cp.async ring in shared memory, kRingDepth chunks (4 KB each) in flight per warp.
// AFF: the accumulator holds a product of INTEGER quantizer levels (SURVEY §7 hard part 1b): with
//   qw[k,c] = s_c (n[k,c] - centre) + o_c,   qa[m,k] = s_a j[m,k]          (s_c = alpha_c / k_w, o_c = beta_c + centre s_c)
// the convolution of the fake-quantized tensors is   s_a s_c * sum_k j (n - centre)  +  s_a o_c * J[m],
// J[m] = sum of the activation levels under the filter window of output row m (computed by the row's thread from
// per-pixel channel sums and handed in as `my_j`).  AFF 1: only the scalar s_a (weight gradient: j (x) dy).
// BNO (forward; AFF 0, or AFF 2 of the u8 kernel): after the fp32 store to `out`, the same register value also goes through the inference
// batch norm `bn` (pf_b200.h: pf_tc_bn_out) with pf_bn_apply_eval's op chain, and is stored as split-bf16 planes and /
// or fp32: the BN pass that would re-read `out` is folded into this one.  The tile's column constants come in `aff_tab`
// (bn_table: rstd, mean, gamma, beta of column c at c, BN + c, 2 BN + c, 3 BN + c; with AFF 2 they follow e1 / e2
// at aff_tab + 512), formed by the kernel before the
// epilogue: __frsqrt_rn has a called slow path, which inside the chunk loop would make ptxas save the loop's live
// registers to local memory.  BNO loads the residual at each chunk instead of one chunk ahead (the second buffer would
// not fit the registers beside the constants), and stores `out` with evict-first stores: nothing reads it soon, while
// the post-BN planes are read by the next convolution.
constexpr int kRingDepth = 4;
constexpr int kRingSlotBytes = 32 * 32 * 4;

struct EpiAff {
  const float* w_alpha;    // per-bucket alpha = (max - min) + 1e-10 of the weight quantizer (device)
  const float* w_beta;     // per-bucket beta = min
  const float* a_scale;    // device scalar: value of one activation level (or 1 for split-bf16 planes); null = 1
  int per_channel;         // 1: bucket = output channel, 0: one bucket per layer
  float w_rk, w_centre;    // 1 / (2^bits - 1), level subtracted from the stored weight levels
};

template <int EXTRA, int AFF, int RD = kRingDepth, bool BNO = false>
__device__ __forceinline__ void epilogue_tile_t(const float* __restrict__ acc, int pitch, long long my_row_off,
                                                long long* __restrict__ rowoff, float* __restrict__ out,
                                                const float* __restrict__ extra, const float* __restrict__ bias,
                                                int relu, int n0, int BN, int Ng, int lane, uint8_t* ring,
                                                const EpiAff& aff, float my_j, float* __restrict__ jrow,
                                                int c_begin, int c_step, const float* __restrict__ aff_tab,
                                                const pf_tc_bn_out& bn) {
  // aff_tab (AFF == 2, TMA-fed kernels): the tile's per-column epilogue constants e1[c] (at c) and e2[c] (at 256 + c)
  // in shared memory, computed once per tile column range instead of being re-derived from global memory per chunk
  // c_begin / c_step: this warp handles the 32-column chunks c_begin, c_begin + c_step, ...
  rowoff[lane] = my_row_off;
  if (AFF == 2) jrow[lane] = my_j;
  __syncwarp();
  const int csub = (lane & 7) * 4, rsub = lane >> 3;
  int ro[8];                                     // this lane's 8 rows (4*u + rsub) of the warp's 32, in float4 units
  float jr[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const long long o = rowoff[4 * u + rsub];
    ro[u] = o < 0 ? -1 : (int)(o >> 2);          // row offsets are multiples of 4 elements (channel counts % 16 == 0)
    jr[u] = (AFF == 2) ? jrow[4 * u + rsub] : 0.f;
  }
  __syncwarp();                                  // rowoff / jrow are rewritten by the next tile
  const float a_s = (AFF && aff.a_scale && !(AFF == 2 && aff_tab)) ? __ldg(aff.a_scale) : 1.f;
  auto load_extra = [&](int c0, float4 (&xv)[8]) {
    const int cv = c0 + csub;
    const bool cok = cv < BN && n0 + cv + 3 < Ng;
#pragma unroll
    for (int u = 0; u < 8; ++u)
      xv[u] = (cok && ro[u] >= 0) ? *reinterpret_cast<const float4*>(extra + ((size_t)ro[u] << 2) + n0 + cv)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  // ring: every lane copies exactly the 16-byte pieces it will read back itself (no cross-lane hand-off); one
  // commit group per chunk, empty groups past the end keep the wait_group count uniform
  const uint32_t ring_u32 = (EXTRA == 2) ? smem_u32(ring) : 0u;
  auto ring_issue = [&](int c0, int it) {
    if (c0 < BN) {
      const int cv = c0 + csub;
      const bool cok = cv < BN && n0 + cv + 3 < Ng;
      const uint32_t slot = ring_u32 + (uint32_t)(it & (RD - 1)) * kRingSlotBytes;
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const bool ok = cok && ro[u] >= 0;
        const float* src = ok ? extra + ((size_t)ro[u] << 2) + n0 + cv : extra;
        const uint32_t dst = slot + (uint32_t)(((4 * u + rsub) * 32 + csub) * 4);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16u : 0u) : "memory");
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  float4 xa[8], xb[8];                           // dead (eliminated) unless EXTRA == 1
  if (EXTRA == 1 && !BNO) load_extra(c_begin, xa);
  if (EXTRA == 2) {
#pragma unroll
    for (int c = 0; c < RD; ++c) ring_issue(c_begin + c_step * c, c);
  }
  int it = 0;
  for (int c0 = c_begin; c0 < BN; c0 += c_step, ++it) {
    // rows 4*u + (lane >> 3), 16-byte chunk (lane & 7): 8 lanes write one row's 128 contiguous bytes
    const int cv = c0 + csub;
    const bool cok = cv < BN && n0 + cv + 3 < Ng;
    float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias && cok) bb = __ldg(reinterpret_cast<const float4*>(bias + n0 + cv));
    float4 e1 = make_float4(a_s, a_s, a_s, a_s), e2 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (AFF == 2 && aff_tab) {
      if (cv < BN) {
        e1 = *reinterpret_cast<const float4*>(aff_tab + cv);
        e2 = *reinterpret_cast<const float4*>(aff_tab + 256 + cv);
      }
    } else if (AFF == 2) {
      float4 al, be;
      if (aff.per_channel) {
        al = cok ? __ldg(reinterpret_cast<const float4*>(aff.w_alpha + n0 + cv)) : make_float4(0.f, 0.f, 0.f, 0.f);
        be = cok ? __ldg(reinterpret_cast<const float4*>(aff.w_beta + n0 + cv)) : make_float4(0.f, 0.f, 0.f, 0.f);
      } else {
        const float a0 = __ldg(aff.w_alpha), b0 = __ldg(aff.w_beta);
        al = make_float4(a0, a0, a0, a0);
        be = make_float4(b0, b0, b0, b0);
      }
      const float sx = al.x * aff.w_rk, sy = al.y * aff.w_rk, sz = al.z * aff.w_rk, sw_ = al.w * aff.w_rk;
      e1 = make_float4(sx * a_s, sy * a_s, sz * a_s, sw_ * a_s);
      e2 = make_float4(fmaf(aff.w_centre, sx, be.x) * a_s, fmaf(aff.w_centre, sy, be.y) * a_s,
                       fmaf(aff.w_centre, sz, be.z) * a_s, fmaf(aff.w_centre, sw_, be.w) * a_s);
    }
    float4 brs, bmu, bga, bbe;                   // BNO: the columns' batch-norm constants (after e1 / e2 with AFF 2)
    if (BNO && cok) {
      const float* bt = AFF == 2 ? aff_tab + 512 : aff_tab;
      brs = *reinterpret_cast<const float4*>(bt + cv);
      bmu = *reinterpret_cast<const float4*>(bt + BN + cv);
      bga = *reinterpret_cast<const float4*>(bt + 2 * BN + cv);
      bbe = *reinterpret_cast<const float4*>(bt + 3 * BN + cv);
    }
    if (EXTRA == 1 && !BNO && c0 + c_step < BN) load_extra(c0 + c_step, xb);
    if (EXTRA == 1 && BNO) load_extra(c0, xa);
    if (EXTRA == 2) asm volatile("cp.async.wait_group %0;" ::"n"(RD - 1) : "memory");   // chunk c0 has landed
    const float* slot = reinterpret_cast<const float*>(ring + (size_t)(it & (RD - 1)) * kRingSlotBytes);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      float4 v[4], xr[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        v[u] = (cv < BN) ? *reinterpret_cast<const float4*>(acc + (size_t)(4 * (4 * half + u) + rsub) * pitch + cv)
                         : make_float4(0.f, 0.f, 0.f, 0.f);
        if (EXTRA == 2) xr[u] = *reinterpret_cast<const float4*>(slot + (4 * (4 * half + u) + rsub) * 32 + csub);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int uu = 4 * half + u;
        if (!cok || ro[uu] < 0) continue;
        float4 w = v[u];
        if (AFF == 1) { w.x *= e1.x; w.y *= e1.y; w.z *= e1.z; w.w *= e1.w; }
        if (AFF == 2) {
          const float j = jr[uu];
          w.x = fmaf(w.x, e1.x, j * e2.x); w.y = fmaf(w.y, e1.y, j * e2.y);
          w.z = fmaf(w.z, e1.z, j * e2.z); w.w = fmaf(w.w, e1.w, j * e2.w);
        }
        if (bias) { w.x = __fadd_rn(w.x, bb.x); w.y = __fadd_rn(w.y, bb.y); w.z = __fadd_rn(w.z, bb.z); w.w = __fadd_rn(w.w, bb.w); }
        if (relu) { w.x = fmaxf(w.x, 0.f); w.y = fmaxf(w.y, 0.f); w.z = fmaxf(w.z, 0.f); w.w = fmaxf(w.w, 0.f); }
        if (EXTRA) {   // fused residual add (resnet_model.py:199,314) or dx += (gradient accumulation)
          const float4 x = (EXTRA == 2) ? xr[u] : xa[uu];
          w.x = __fadd_rn(w.x, x.x); w.y = __fadd_rn(w.y, x.y); w.z = __fadd_rn(w.z, x.z); w.w = __fadd_rn(w.w, x.w);
        }
        if (BNO)
          __stcs(reinterpret_cast<float4*>(out + ((size_t)ro[uu] << 2) + n0 + cv), w);
        else
          *reinterpret_cast<float4*>(out + ((size_t)ro[uu] << 2) + n0 + cv) = w;
        if (BNO) {
          const int act = bn.act;
          w.x = pf_bn_act(w.x, bmu.x, brs.x, bga.x, bbe.x, act); w.y = pf_bn_act(w.y, bmu.y, brs.y, bga.y, bbe.y, act);
          w.z = pf_bn_act(w.z, bmu.z, brs.z, bga.z, bbe.z, act); w.w = pf_bn_act(w.w, bmu.w, brs.w, bga.w, bbe.w, act);
          const int64_t e = ((int64_t)ro[uu] << 2) + n0 + cv;
          if (bn.y) *reinterpret_cast<float4*>(bn.y + e) = w;
          if (bn.hi) pf_st_planes4(bn.hi, bn.lo, e, w);
        }
      }
    }
    if (EXTRA == 1 && !BNO) {
#pragma unroll
      for (int u = 0; u < 8; ++u) xa[u] = xb[u];
    }
    if (EXTRA == 2) {
      __syncwarp();                              // every lane has read the slot before it is refilled
      ring_issue(c0 + c_step * RD, it + RD);
    }
  }
  if (EXTRA == 2) asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// the folded batch norm's constants of columns [n0, n0 + BN) into `tab` (4 BN floats): rstd (formed as
// pf_bn_apply_eval forms it), mean, gamma and beta of column c at c, BN + c, 2 BN + c and 3 BN + c; thread t of `nthr`
// fills columns t, t + nthr, ...
__device__ __forceinline__ void bn_table(const pf_tc_bn_out& bn, float* tab, int n0, int BN, int Ng, int t, int nthr) {
  for (int c = t; c < BN; c += nthr) {
    const bool ok = n0 + c < Ng;
    tab[c] = ok ? __frsqrt_rn(__fadd_rn(__ldg(bn.var + n0 + c), bn.eps)) : 0.f;
    tab[BN + c] = ok ? __ldg(bn.mean + n0 + c) : 0.f;
    tab[2 * BN + c] = ok ? __ldg(bn.gamma + n0 + c) : 0.f;
    tab[3 * BN + c] = ok ? __ldg(bn.beta + n0 + c) : 0.f;
  }
}

// the epilogue of one warp over 32 rows of the accumulator tile starting at `acc`, 32-column chunks c_begin,
// c_begin + c_step, ...: picks the residual / accumulate path (none, registers, cp.async ring of depth 2 or 4)
template <int AFF, bool BNO = false>
__device__ __forceinline__ void epilogue_rows(const float* acc, int c_begin, int c_step, long long my_row_off,
                                              long long* rowoff, float* __restrict__ out, const float* __restrict__ extra,
                                              const float* __restrict__ bias, int relu, int n0, int BN, int Ng,
                                              int lane, uint8_t* ring, const EpiAff& aff, float my_j, float* jrow,
                                              const float* aff_tab, int ring_depth, const pf_tc_bn_out& bn) {
  static_assert(!BNO || AFF != 1, "the folded batch norm is an inference-mode (forward) epilogue");
  const int pitch = acc_pitch(BN);
  if (extra && ring && ring_depth == 2) epilogue_tile_t<2, AFF, 2, BNO>(acc, pitch, my_row_off, rowoff, out, extra, bias, relu, n0, BN, Ng, lane, ring, aff, my_j, jrow, c_begin, c_step, aff_tab, bn);
  else if (extra && ring) epilogue_tile_t<2, AFF, kRingDepth, BNO>(acc, pitch, my_row_off, rowoff, out, extra, bias, relu, n0, BN, Ng, lane, ring, aff, my_j, jrow, c_begin, c_step, aff_tab, bn);
  else if (extra) epilogue_tile_t<1, AFF, kRingDepth, BNO>(acc, pitch, my_row_off, rowoff, out, extra, bias, relu, n0, BN, Ng, lane, nullptr, aff, my_j, jrow, c_begin, c_step, aff_tab, bn);
  else epilogue_tile_t<0, AFF, kRingDepth, BNO>(acc, pitch, my_row_off, rowoff, out, nullptr, bias, relu, n0, BN, Ng, lane, nullptr, aff, my_j, jrow, c_begin, c_step, aff_tab, bn);
}

// the epilogue of warp `ew` (0..7) of the MMA warps: rows 32 (ew % 4) .., chunks ew / 4, ew / 4 + 2, ...
template <int AFF, bool BNO = false>
__device__ __forceinline__ void epilogue_tile_a(const float* acc_s, int ew, long long my_row_off, long long* rowoff,
                                                float* __restrict__ out, const float* __restrict__ extra,
                                                const float* __restrict__ bias, int relu, int n0, int BN, int Ng,
                                                int lane, uint8_t* ring, const EpiAff& aff, float my_j, float* jrow,
                                                const pf_tc_bn_out& bn, const float* aff_tab = nullptr,
                                                int ring_depth = kRingDepth) {
  epilogue_rows<AFF, BNO>(acc_s + (size_t)(32 * (ew & 3)) * acc_pitch(BN), 32 * (ew >> 2), 64, my_row_off, rowoff,
                          out, extra, bias, relu, n0, BN, Ng, lane, ring, aff, my_j, jrow, aff_tab, ring_depth, bn);
}
__device__ __forceinline__ void epilogue_tile(const float* acc_s, int ew, long long my_row_off, long long* rowoff,
                                              float* __restrict__ out, const float* __restrict__ extra,
                                              const float* __restrict__ bias, int relu, int n0, int BN, int Ng,
                                              int lane, uint8_t* ring = nullptr) {
  const EpiAff none{};
  const pf_tc_bn_out no_bn{};
  epilogue_tile_a<0>(acc_s, ew, my_row_off, rowoff, out, extra, bias, relu, n0, BN, Ng, lane, ring, none, 0.f, nullptr,
                     no_bn);
}

// dispatch on the tile width (the wgmma N is an immediate): f is called with std::integral_constant<int, BN>
template <class F>
inline void with_bn(int BN, F&& f) {
  switch (BN) {
    case 16: f(std::integral_constant<int, 16>()); break;
    case 32: f(std::integral_constant<int, 32>()); break;
    case 64: f(std::integral_constant<int, 64>()); break;
    default: f(std::integral_constant<int, 128>()); break;
  }
}

// ---- plan record (pf_conv2d_tc_last_plan): every launcher stores the plan it launches with, just before the launch
void record_plan(const pf_tc_plan& p);

// ---- TMA-fed kernels (pf_conv_tma.cu)
void conv_tma_set_feed(int mode);
bool conv_tma_eligible(int pass, const TcGeom& g);      // pass: 0 fwd, 1 dgrad, 2 wgrad
bool conv_tma_u8_eligible(const TcGeom& g);             // pf_conv2d_u8_fwd
// u8: forward with unsigned 8-bit activation and weight levels (pf_conv2d_u8_fwd)
int conv_tma_launch(int pass, const TcGeom& g, const pf_tc_act& a, const pf_tc_wt& w, float* out, int accumulate,
                    const float* bias, int relu, const float* residual, cudaStream_t st, const char* who,
                    const pf_tc_bn_out* bn = nullptr, bool u8 = false);
int conv_tma_wgrad_launch(const TcGeom& g, const pf_tc_act& x, const pf_tc_act& dy, int BN, int pps, int splits,
                          float* partial, cudaStream_t st, const char* who);

}  // namespace pfconv
