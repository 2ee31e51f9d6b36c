// pf_conv_tma.cu — the wgmma convolution kernels fed by the Tensor Memory Accelerator (sm_90a).
//
// Same contraction as pf_conv_tc.cu (SURVEY §8 a4: tf.nn.conv2d re-created on the quantized weight,
// /root/reference/learners/uniform_quantization/utils.py:92-104, its dgrad and wgrad), for channel counts that are
// multiples of 64.  What changes is how the operands reach shared memory and how many MMAs a product costs:
//   * the NHWC operand (x in fwd / wgrad, dy in dgrad) is fetched by ONE im2col-mode TMA load per k-stage and plane
//     (128 filter-window positions x 64 channels of one tap; the padding is TMA's out-of-bounds zero fill), the
//     K-major weight matrix / the dy matrix by tiled TMA loads — one elected thread issues them, completion is counted
//     in bytes on the stage's mbarrier.  No LSU instruction touches an operand; producer warps are gone (fwd / dgrad:
//     two ping-pong consumer warpgroups and a producer warpgroup; wgrad: two MMA + epilogue warpgroups and the TMA
//     warp), stages are as deep as shared memory allows (up to 8);
//   * an operand that is a <= 8-bit fake-quantized tensor arrives as its INTEGER LEVELS (exact in bf16): one plane
//     instead of hi + lo.  MMAs per k-slice: levels x levels 1, levels x split 2, split x split 3; the per-channel
//     scale, and the rank-1 term that the weight offset contributes, are applied by the epilogue (pf_conv_tc.cuh);
//   * the u8 forward (pf_conv2d_u8_fwd, inference): both operands are the quantizers' own UNSIGNED 8-bit levels, one
//     byte per element, K-major.  A k-stage is still 64 channels of one tap, now 64-byte rows (SWIZZLE_64B boxes and
//     descriptors), and a k-slice is one u8 x u8 -> s32 wgmma of k = 32: the integer sum of level products is exact,
//     and the same AFF 2 epilogue (weight centre 0) turns it into the fake-quantized model's output.
#include <cuda.h>

#include "pf_conv_tc.cuh"
#include "pf_tma.cuh"

namespace pfconv {
using namespace pftma;

constexpr int kTmaMaxStages = 8;
constexpr int kTmaThreads = (kMmaWarps + 1) * 32;     // wgrad: warps 0-7 MMA warpgroups + epilogue, warp 8 TMA producer

struct TmaP {
  int M, Ng, BN, nk, n_tiles, total_tiles;
  int cblocks, R, S;                       // k-stage ks -> tap = ks / cblocks (r = tap / S, q = tap % S), channel block
  int rows_hw, rows_w;                     // GEMM row m -> (image, y, x)
  int src_h, src_w;                        // gathered tensor
  int base_w, base_h, str_w, str_h, flip;  // window origin of row (y, x): (base + x * str); flip: tap offsets mirrored
  int na, nb;                              // operand planes (na: upper bound when a_hdr decides)
  int accumulate, relu, ring, stage_budget;     // ring: 0 = none, else the residual ring's depth (2 or 4)
  int chunked;                             // 1: the staging tile holds one 32-column chunk (fwd / dgrad, see the launcher)
  FastDiv d_hw, d_w, d_ntiles, d_cblocks, d_s;
  EpiAff aff;
  const pf_tc_act_hdr* a_hdr;
  const float* csum;
  int nseg;
  pf_tc_bn_out bn;                         // BNO kernels: the batch norm folded into the epilogue
};

// ---------------------------------------------------------------------------------------------------------
// fwd / dgrad (unit stride): D[M x Ng] = A[M x K] * B[Ng x K]^T, both operands K-major, 128 x BN output tiles,
// persistent CTAs, ping-pong consumers.  The TMA thread fills the stage ring for the CTA's tiles in order; consumer
// warpgroup w owns the CTA's tiles 2 j + w (j = 0, 1, ...) whole: two m64 wgmmas per k-slice and plane product, into
// two accumulator halves.  Two turns pass between the warpgroups, each through a pair of mbarriers:
//   * the mainloop turn: a warpgroup waits on the stage ring only after the other has issued its last tile's MMAs, so
//     the ring is consumed in the order it is filled (a consumer that ran ahead could take the parity of a stage's
//     earlier fill for the one it wants) and the two warpgroups' MMAs do not interleave;
//   * the epilogue turn: one fp32 staging tile serves both; a warpgroup owns it from its accumulator store to its last
//     read in the epilogue.
// So while one warpgroup runs a tile's epilogue (bias, ReLU, residual or accumulate, the levels' rank-1 term, 64 KB of
// fp32 stores at BN = 128), the other runs the next tile's MMAs.  Warpgroup 0 takes its first turns without waiting;
// every later turn waits for the other warpgroup's release of the previous one, which keeps the handoff correct for
// any number of tiles per CTA (with one tile, warpgroup 1 never waits and its releases are never read).
constexpr int kPingPongWarps = 4;        // arrivals per turn release and per stage release: one per consumer warp
// warps 0-7: the two consumer warpgroups; warps 8-11: the producer warpgroup (one thread issues the TMA loads).  A
// consumer holds a whole 128 x BN accumulator (128 registers at BN = 128), more than the 168 registers per thread
// that 384 resident threads leave; the producer warpgroup gives up all but 40 of its registers and the consumers
// raise theirs to 232 (128 x 40 + 256 x 232 <= 64 K).
constexpr int kPingPongThreads = (kMmaWarps + 4) * 32;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;

// The epilogue of a 128 x 128 tile through a staging tile of one 32-column chunk (128 x 36 floats, 18 KB instead of
// 66 KB): for each chunk, the warpgroup stores that chunk's accumulator fragments, and warp q runs the shared epilogue
// (epilogue_rows) on rows 32 q .. + 32 of it, with the chunk's columns as the tile.  The values and the op chain are
// those of the whole-tile epilogue, so the bits are too.  Only split-bf16 / bf16 tiles (AFF 0) without a residual /
// accumulate operand and without a folded batch norm take this path (the launcher decides): the whole-tile epilogue
// prefetches that operand one chunk ahead, which a chunk at a time cannot, and the batch-norm epilogue does not fit
// the registers beside the accumulator chunks still held (6.5 KB of spills).  Warpgroup-local barriers order each
// chunk's stores after the previous chunk's reads and before its own reads.
__device__ __forceinline__ void conv_tma_epilogue_chunked(float (&acc)[2][64], const TmaP& p, float* acc_s,
                                                          int n0, long long off, long long* rowoff, float* out,
                                                          const float* bias, int wg, int q, int lane) {
  constexpr int P = acc_pitch(32);
  float* r0 = acc_s + (size_t)(16 * q + (lane >> 2)) * P + 2 * (lane & 3);
#pragma unroll
  for (int ch = 0; ch < 4; ++ch) {
    if (ch > 0) named_bar_sync(2 + wg, 128);      // every warp has read the previous chunk
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = 4 * ch + jj;
        *reinterpret_cast<float2*>(r0 + (size_t)(64 * h) * P + 8 * jj) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
        *reinterpret_cast<float2*>(r0 + (size_t)(64 * h + 8) * P + 8 * jj) =
            make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
      }
    named_bar_sync(2 + wg, 128);                  // the chunk is visible to the warpgroup
    epilogue_rows<0>(acc_s + (size_t)(32 * q) * P, 0, 32, off, rowoff, out, nullptr, bias, p.relu, n0 + 32 * ch, 32,
                     p.Ng, lane, nullptr, p.aff, 0.f, nullptr, nullptr, 0, p.bn);
  }
}

template <int AFF, int BN, int NA, int NB, bool BNO, bool U8>
__device__ __forceinline__ void conv_tma_consumer(const TmaP& p, uint8_t* smem, uint32_t stage_bytes,
                                                  uint32_t n_stages, uint64_t* full_bar, uint64_t* empty_bar,
                                                  uint64_t* ml_bar, uint64_t* epi_bar, int* tab_n0, float* out,
                                                  const float* bias, const float* residual) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, q = warp & 3, wtid = tid & 127;   // epilogue rows [32 q, 32 q + 32) of the tile
  constexpr uint32_t kRow = U8 ? 64u : 128u, kATile = TM * kRow;   // bytes of one tile row / of the A tile
  const uint32_t b_bytes = (uint32_t)BN * kRow;
  float* acc_s = reinterpret_cast<float*>(smem + p.stage_budget);
  long long* rowoff_all = reinterpret_cast<long long*>(acc_s + TM * acc_pitch(p.chunked ? 32 : BN));
  float* jrow_all = reinterpret_cast<float*>(rowoff_all + kMmaWarps * 32);
  // AFF == 2: e1[256], e2[256] of the staged tile's columns; BNO: the folded batch norm's constants of them (bn_table)
  float* aff_tab = jrow_all + kMmaWarps * 32;
  uint8_t* ring_all = reinterpret_cast<uint8_t*>(aff_tab + (AFF == 2 ? 2 * 256 : 0) + (BNO ? 4 * kMaxBN : 0));
  long long* rowoff = rowoff_all + warp * 32;
  float* jrow = jrow_all + warp * 32;
  uint8_t* ring = p.ring ? ring_all + (size_t)warp * p.ring * kRingSlotBytes : nullptr;
  const float* extra = residual ? residual : (p.accumulate ? out : nullptr);
  uint32_t it = (uint32_t)wg * (uint32_t)p.nk;              // stage-ring position of this warpgroup's next tile
  for (int tile = blockIdx.x + wg * gridDim.x, j = 0; tile < p.total_tiles; tile += 2 * gridDim.x, ++j) {
    const bool wait_turn = wg == 1 || j > 0;
    const uint32_t turn_ph = (uint32_t)(wg == 1 ? j : j - 1) & 1u;
    // ---- mainloop
    if (wait_turn) mbar_wait_bounded(&ml_bar[wg], turn_ph);
    std::conditional_t<U8, int, float> acc[2][BN / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0;
    uint32_t s = it % n_stages, ph = (it / n_stages) & 1u, prev = 0;
    for (int ks = 0; ks < p.nk; ++ks) {
      mbar_wait_bounded(&full_bar[s], ph);                               // TMA bytes have landed
      const uint32_t a0 = smem_u32(smem + (size_t)s * stage_bytes), a1 = a0 + kATile;
      const uint32_t b0 = a0 + (uint32_t)NA * kATile, b1 = b0 + b_bytes;
      wgmma_fence();
      if constexpr (U8) {
        // two k32 slices of 32 bytes per 64-byte row; 8-row groups 512 bytes apart
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
          const uint64_t db = make_smem_desc(b0 + kk * 32, 16, 512, kSwizzle64B);
#pragma unroll
          for (int h = 0; h < 2; ++h)                                    // rows [64 h, 64 h + 64): 4 KB
            WgmmaU8<BN>::mma(acc[h], make_smem_desc(a0 + (uint32_t)h * 64 * 64 + kk * 32, 16, 512, kSwizzle64B), db);
        }
      } else {
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk) {
          const uint64_t db0 = make_smem_desc(b0 + kk * 32, 16, 1024), db1 = make_smem_desc(b1 + kk * 32, 16, 1024);
#pragma unroll
          for (int h = 0; h < 2; ++h) {                                  // rows [64 h, 64 h + 64): 8 KB per plane
            const uint32_t ha = (uint32_t)h * 64 * 128 + kk * 32;
            wg_mma_kslice<BN, 0, NA, NB>(acc[h], make_smem_desc(a0 + ha, 16, 1024), make_smem_desc(a1 + ha, 16, 1024),
                                         db0, db1);
          }
        }
      }
      wgmma_commit();
      wgmma_wait<1>(acc);                     // the previous stage's MMAs have completed: release it
      if (ks > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = s;
      if (++s == n_stages) { s = 0; ph ^= 1u; }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&ml_bar[wg ^ 1]);                          // every MMA of this tile is issued
    wgmma_wait<0>(acc);
    if (p.nk > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }
    it += 2u * (uint32_t)p.nk;
    // ---- epilogue
    const int mt = (int)fdiv((uint32_t)tile, p.d_ntiles);
    const int n0 = (tile - mt * p.n_tiles) * BN;
    const int m = mt * TM + q * 32 + lane;
    const long long off = m < p.M ? (long long)m * p.Ng : -1;
    float my_j = 0.f;
    if (AFF == 2 && p.csum && m < p.M) {
      // sum of the stored activation levels under this row's filter window, from the per-pixel channel sums, before
      // the epilogue turn (it needs no staging tile): the (tap, segment) terms are independent loads, issued four at a
      // time (branch-free; the terms are integers below 2^24, so the order of the additions does not change the result)
      const int img = (int)fdiv((uint32_t)m, p.d_hw);
      const int rem = m - img * p.rows_hw;
      const int y = (int)fdiv((uint32_t)rem, p.d_w), x = rem - y * p.rows_w;
      const int ow0 = p.base_w + x * p.str_w, oh0 = p.base_h + y * p.str_h;
      const int total = p.R * p.S * p.nseg;
      const float* cbase = p.csum + (size_t)img * p.src_h * p.src_w * p.nseg;
      auto term = [&](int u) -> float {
        if (u >= total) return 0.f;
        const int t = u / p.nseg, g = u - t * p.nseg;
        const int r = (int)fdiv((uint32_t)t, p.d_s), s_ = t - r * p.S;
        const int ih = oh0 + r, iw = ow0 + s_;
        const bool ok = (unsigned)ih < (unsigned)p.src_h && (unsigned)iw < (unsigned)p.src_w;
        return ok ? __ldg(cbase + ((size_t)ih * p.src_w + iw) * p.nseg + g) : 0.f;
      };
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      for (int u = 0; u < total; u += 4) {
        const float v0 = term(u), v1 = term(u + 1), v2 = term(u + 2), v3 = term(u + 3);
        a0 += v0; a1 += v1; a2 += v2; a3 += v3;
      }
      my_j = (a0 + a1) + (a2 + a3);
    }
    if (wait_turn) mbar_wait_bounded(&epi_bar[wg], turn_ph);            // the staging tile is this warpgroup's
    constexpr bool TAB = AFF == 2 || BNO;
    if constexpr (BN == 128 && AFF == 0 && !BNO && !U8) {
      if (p.chunked) {
        conv_tma_epilogue_chunked(acc, p, acc_s, n0, off, rowoff, out, bias, wg, q, lane);
        __syncwarp();
        if (lane == 0) mbar_arrive(&epi_bar[wg ^ 1]);                     // this warp's reads of the tile are done
        continue;
      }
    }
    wgmma_store_acc<BN>(acc[0], acc_s, acc_pitch(BN), 0, wtid);
    wgmma_store_acc<BN>(acc[1], acc_s, acc_pitch(BN), 64, wtid);
    const int tab_was = TAB ? *reinterpret_cast<volatile int*>(tab_n0) : 0;
    if (AFF == 2 && tab_was != n0) {
      // per-column constants of this tile's columns, when they differ from the staged table's (with one n-tile per
      // row of tiles this runs once per CTA):  e1[c] = s_a * alpha_c / k_w ,  e2[c] = s_a * (centre * alpha_c / k_w + beta_c)
      float a_s = p.aff.a_scale ? __ldg(p.aff.a_scale) : 1.f;
      // u8 levels stand for scale * level only when the tensor's minimum is 0 (header: 1 plane); otherwise the
      // activation offset has no term here, and the output is NaN rather than silently wrong
      if (U8 && __ldg(&p.a_hdr->nplanes) != 1) a_s = __int_as_float(0x7fc00000);
      for (int c = wtid; c < BN; c += 128) {
        const bool cok = n0 + c < p.Ng;
        const int bi = p.aff.per_channel ? n0 + c : 0;
        const float al = cok ? __ldg(p.aff.w_alpha + bi) : 0.f, be = cok ? __ldg(p.aff.w_beta + bi) : 0.f;
        const float sx = al * p.aff.w_rk;
        aff_tab[c] = sx * a_s;
        aff_tab[256 + c] = fmaf(p.aff.w_centre, sx, be) * a_s;
      }
    }
    if (BNO && tab_was != n0) bn_table(p.bn, aff_tab + (AFF == 2 ? 512 : 0), n0, BN, p.Ng, wtid, 128);
    named_bar_sync(2 + wg, 128);                       // the staged tile (and table) are visible to the warpgroup
    if (TAB && tab_was != n0 && wtid == 0) *reinterpret_cast<volatile int*>(tab_n0) = n0;
    epilogue_rows<AFF, BNO>(acc_s + (size_t)(32 * q) * acc_pitch(BN), 0, 32, off, rowoff, out, extra, bias, p.relu, n0,
                            BN, p.Ng, lane, ring, p.aff, my_j, jrow, TAB ? aff_tab : nullptr, p.ring, p.bn);
    __syncwarp();
    if (lane == 0) mbar_arrive(&epi_bar[wg ^ 1]);                         // this warp's reads of the tile are done
  }
}

template <int AFF, int BN, bool BNO = false, bool U8 = false>
__global__ void __launch_bounds__(kPingPongThreads, 1)
conv_tma_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                const __grid_constant__ CUtensorMap tmB0, const __grid_constant__ CUtensorMap tmB1,
                float* __restrict__ out, const float* __restrict__ bias, const float* __restrict__ residual,
                const __grid_constant__ TmaP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  __shared__ uint64_t full_bar[kTmaMaxStages], empty_bar[kTmaMaxStages], ml_bar[2], epi_bar[2];
  __shared__ int tab_n0;                              // first column of the column table in shared memory (-1: none)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int na = p.na;
  if (p.a_hdr) na = (__ldg(&p.a_hdr->nplanes) == 2) ? 2 : 1;
  const int nb = p.nb;
  constexpr uint32_t kRow = U8 ? 64u : 128u, kATile = TM * kRow;
  const uint32_t b_bytes = (uint32_t)BN * kRow;
  const uint32_t stage_bytes = (uint32_t)na * kATile + (uint32_t)nb * b_bytes;
  const uint32_t n_stages = min((uint32_t)kTmaMaxStages, (uint32_t)p.stage_budget / stage_bytes);

  if (tid == 0) {
    for (int s = 0; s < kTmaMaxStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kPingPongWarps);
    }
    for (int w = 0; w < 2; ++w) {
      mbar_init(&ml_bar[w], kPingPongWarps);
      mbar_init(&epi_bar[w], kPingPongWarps);
    }
    tab_n0 = -1;
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kMmaWarps) {
    // =================================== TMA producer (one thread) ===================================
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kMmaWarps && lane == 0) {
      prefetch_map(&tmA0);
      prefetch_map(&tmB0);
      if (na == 2) prefetch_map(&tmA1);
      if (nb == 2) prefetch_map(&tmB1);
      uint32_t s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int mt = (int)fdiv((uint32_t)tile, p.d_ntiles);
        const int n0 = (tile - mt * p.n_tiles) * BN;
        const int m0 = mt * TM;
        const int img = (int)fdiv((uint32_t)m0, p.d_hw);
        const int rem = m0 - img * p.rows_hw;
        const int y = (int)fdiv((uint32_t)rem, p.d_w), x = rem - y * p.rows_w;
        const int cw = p.base_w + x * p.str_w, ch = p.base_h + y * p.str_h;
        for (int ks = 0; ks < p.nk; ++ks) {
          mbar_wait_bounded(&empty_bar[s], ph ^ 1u);                     // slot free?
          const int tap = (int)fdiv((uint32_t)ks, p.d_cblocks);
          const int cb = ks - tap * p.cblocks;
          const int r = (int)fdiv((uint32_t)tap, p.d_s), q = tap - r * p.S;
          const uint32_t ow = (uint32_t)(p.flip ? p.S - 1 - q : q), oh = (uint32_t)(p.flip ? p.R - 1 - r : r);
          const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
          const uint32_t sb = sa + (uint32_t)na * kATile;
          mbar_arrive_expect_tx(&full_bar[s], stage_bytes);
          load_im2col(sa, &tmA0, &full_bar[s], cb * BK, cw, ch, img, ow, oh);
          if (na == 2) load_im2col(sa + kATile, &tmA1, &full_bar[s], cb * BK, cw, ch, img, ow, oh);
          load_2d(sb, &tmB0, &full_bar[s], ks * BK, n0);
          if (nb == 2) load_2d(sb + b_bytes, &tmB1, &full_bar[s], ks * BK, n0);
          if (++s == n_stages) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    // ==================== two ping-pong consumer warpgroups (warps 0-3, 4-7): MMAs + epilogue ====================
    // the plane counts are fixed for the whole launch: one straight-line mainloop per combination
    setmaxnreg_inc<kConsumerRegs>();
#define PF_TMA_CONSUMER(NA_, NB_)                                                                                    \
  conv_tma_consumer<AFF, BN, NA_, NB_, BNO, U8>(p, smem, stage_bytes, n_stages, full_bar, empty_bar, ml_bar, epi_bar, \
                                                &tab_n0, out, bias, residual)
    if constexpr (U8) {
      PF_TMA_CONSUMER(1, 1);
    } else {
      if (na == 2) {
        if (nb == 2) PF_TMA_CONSUMER(2, 2);
        else PF_TMA_CONSUMER(2, 1);
      } else {
        if (nb == 2) PF_TMA_CONSUMER(1, 2);
        else PF_TMA_CONSUMER(1, 1);
      }
    }
#undef PF_TMA_CONSUMER
  }
}

// ---------------------------------------------------------------------------------------------------------
// wgrad: dW[kf x cout] = X[pixels x kf]^T * dY[pixels x cout], both operands MN-major in shared memory
// ([64-wide MN block][pixel][128 B], exactly what a 64-channel x 64-pixel TMA box with SWIZZLE_128B writes).
// Work unit = (kf tile of 128 = two 64-channel blocks, cout tile of BN, pixel range); split-K partials as in
// pf_conv_tc.cu.  x arrives through an im2col-mode map (64 window positions x 64 channels of the tap the block
// belongs to), dy through a tiled map.
struct WgTmaP {
  TcGeom g;
  int Mtot, Npix, pps, splits, BN, n_tiles, tiles, total_units;
  int na, nb, stage_budget;
  FastDiv d_pq, d_q, d_c, d_s, d_tiles, d_ntiles;
  EpiAff aff;
  const pf_tc_act_hdr* x_hdr;
};
constexpr uint32_t kWgBlockBytes = BK * 128;   // one 64 (MN) x 64 (pixels) block

template <int AFF, int BN>
__global__ void __launch_bounds__(kTmaThreads, 1)
conv_tma_wgrad_kernel(const __grid_constant__ CUtensorMap tmX0, const __grid_constant__ CUtensorMap tmX1,
                      const __grid_constant__ CUtensorMap tmY0, const __grid_constant__ CUtensorMap tmY1,
                      float* __restrict__ partial, const __grid_constant__ WgTmaP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  __shared__ uint64_t full_bar[kTmaMaxStages], empty_bar[kTmaMaxStages];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const TcGeom& g = p.g;
  const int nblkB = BN / 64;
  int na = p.na;
  if (p.x_hdr) na = (__ldg(&p.x_hdr->nplanes) == 2) ? 2 : 1;
  const int nb = p.nb;
  const uint32_t a_bytes = 2 * kWgBlockBytes, b_bytes = (uint32_t)nblkB * kWgBlockBytes;
  const uint32_t stage_bytes = (uint32_t)na * a_bytes + (uint32_t)nb * b_bytes;
  const uint32_t n_stages = min((uint32_t)kTmaMaxStages, (uint32_t)p.stage_budget / stage_bytes);
  float* acc_s = reinterpret_cast<float*>(smem + p.stage_budget);
  long long* rowoff_all = reinterpret_cast<long long*>(acc_s + TM * acc_pitch(BN));
  float* jrow_all = reinterpret_cast<float*>(rowoff_all + kMmaWarps * 32);
  if (tid == 0) {
    for (int s = 0; s < kTmaMaxStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kMmaWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
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

  if (warp == kMmaWarps) {
    if (lane == 0) {
      prefetch_map(&tmX0);
      prefetch_map(&tmY0);
      if (na == 2) prefetch_map(&tmX1);
      if (nb == 2) prefetch_map(&tmY1);
      const int pq = g.P * g.Q;
      uint32_t s = 0, ph = 0;
      for (int u = blockIdx.x; u < p.total_units; u += gridDim.x) {
        const Unit un = decode(u);
        // the two 64-row blocks of the kf tile: each lies inside one filter tap (Cin % 64 == 0)
        int c0[2], tr[2], tq[2], nvalid = 0;
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int kf = un.m0 + 64 * b;
          const int tap = (int)fdiv((uint32_t)kf, p.d_c);
          c0[b] = kf - tap * g.C;
          tr[b] = (int)fdiv((uint32_t)tap, p.d_s);
          tq[b] = tap - tr[b] * g.S;
          if (kf < p.Mtot) nvalid = b + 1;
        }
        const uint32_t tx = (uint32_t)na * (uint32_t)nvalid * kWgBlockBytes + (uint32_t)nb * b_bytes;
        for (int ks = 0; ks < un.nk; ++ks) {
          mbar_wait_bounded(&empty_bar[s], ph ^ 1u);
          const int pix0 = un.pbeg + ks * BK;
          const int pn = (int)fdiv((uint32_t)pix0, p.d_pq);
          const int rem = pix0 - pn * pq;
          const int oh = (int)fdiv((uint32_t)rem, p.d_q), ow = rem - oh * g.Q;
          const int cw = ow * g.sw - g.pl, ch = oh * g.sh - g.pt;
          const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
          const uint32_t sb = sa + (uint32_t)na * a_bytes;
          mbar_arrive_expect_tx(&full_bar[s], tx);
          for (int b = 0; b < nvalid; ++b) {
            load_im2col(sa + b * kWgBlockBytes, &tmX0, &full_bar[s], c0[b], cw, ch, pn, (uint32_t)tq[b], (uint32_t)tr[b]);
            if (na == 2)
              load_im2col(sa + a_bytes + b * kWgBlockBytes, &tmX1, &full_bar[s], c0[b], cw, ch, pn, (uint32_t)tq[b],
                          (uint32_t)tr[b]);
          }
          for (int j = 0; j < nblkB; ++j) {
            load_2d(sb + j * kWgBlockBytes, &tmY0, &full_bar[s], un.n0 + 64 * j, pix0);
            if (nb == 2) load_2d(sb + b_bytes + j * kWgBlockBytes, &tmY1, &full_bar[s], un.n0 + 64 * j, pix0);
          }
          if (++s == n_stages) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    // MMA warpgroups + epilogue: warpgroup wg multiplies kf rows [64 wg, 64 wg + 64) = MN block wg of the x tile;
    // the plane counts are fixed for the whole launch: one straight-line mainloop per combination
    const int wg = warp >> 2, q = warp & 3;
    long long* rowoff = rowoff_all + warp * 32;
    float* jrow = jrow_all + warp * 32;
    auto consume = [&](auto na_c, auto nb_c) {
    constexpr int NA = decltype(na_c)::value, NB = decltype(nb_c)::value;
    uint32_t s = 0, ph = 0;
    for (int u = blockIdx.x; u < p.total_units; u += gridDim.x) {
      const Unit un = decode(u);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      uint32_t prev = 0;
      for (int ks = 0; ks < un.nk; ++ks) {
        mbar_wait_bounded(&full_bar[s], ph);
        const uint32_t base = smem_u32(smem + (size_t)s * stage_bytes);
        const uint32_t a0 = base + (uint32_t)wg * kWgBlockBytes, a1 = a0 + a_bytes;
        const uint32_t b0 = base + (uint32_t)NA * a_bytes, b1 = b0 + b_bytes;
        // MN-major: LBO = stride between 64-wide MN blocks (8 KB), SBO = stride between 8-pixel groups (1 KB);
        // one MMA consumes 16 pixels = 2 KB
        wg_mma_stage<BN, 1, NA, NB>(acc, a0, a1, b0, b1, 2048, 2048, kWgBlockBytes, 1024, kWgBlockBytes, 1024);
        wgmma_wait<1>(acc);
        if (ks > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = s;
        if (++s == n_stages) { s = 0; ph ^= 1u; }
      }
      wgmma_wait<0>(acc);
      if (un.nk > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      const int em = un.m0 + q * 32 + lane;
      const long long off = em < p.Mtot ? ((long long)un.split * p.Mtot + em) * g.K : -1;
      wg_tile_to_smem<BN>(acc, acc_s, tid);
      epilogue_tile_a<AFF>(acc_s, warp, off, rowoff, partial, nullptr, nullptr, 0, un.n0, BN, g.K, lane, nullptr, p.aff,
                           0.f, jrow, pf_tc_bn_out{});
    }
    };
    using one = std::integral_constant<int, 1>;
    using two = std::integral_constant<int, 2>;
    if (na == 2) {
      if (nb == 2) consume(two(), two());
      else consume(two(), one());
    } else {
      if (nb == 2) consume(one(), two());
      else consume(one(), one());
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// host side
static int g_feed_override = -1;          // pf_conv2d_tc_set_feed: 0 = cp.async kernels, 1 = TMA kernels, -1 = PF_TC_FEED / default
void conv_tma_set_feed(int mode) { g_feed_override = mode < 0 ? -1 : (mode ? 1 : 0); }
static bool tma_enabled() {
  if (g_feed_override >= 0) return g_feed_override == 1;
  static int on = -1;
  if (on < 0) {
    const char* v = getenv("PF_TC_FEED");
    on = !(v && strcmp(v, "lsu") == 0);
  }
  return on == 1;
}

bool conv_tma_eligible(int pass, const TcGeom& g) {
  if (!tma_enabled()) return false;
  if (pass == 0) return g.C % 64 == 0 && g.K % 16 == 0 && g.sh <= 8 && g.sw <= 8 && g.R <= 16 && g.S <= 16;
  if (pass == 1) return g.K % 64 == 0 && g.C % 16 == 0 && g.sh == 1 && g.sw == 1 && g.R <= 16 && g.S <= 16;
  return g.C % 64 == 0 && g.K % 64 == 0 && g.sh <= 8 && g.sw <= 8;
}

// the u8 forward of these shapes runs here, the other shapes pf_conv2d_u8_narrow_supported takes run the cp.async-fed
// u8 kernel (pf_conv_tc.cu): only the shape decides, not the feed setting
bool conv_tma_u8_eligible(const TcGeom& g) {
  return g.C % 64 == 0 && g.K % 64 == 0 && g.sh <= 8 && g.sw <= 8 && g.R <= 16 && g.S <= 16;
}

static int pick_bn(int Ng) {
  int BN = Ng >= 128 ? 128 : (Ng >= 64 ? 64 : (Ng >= 32 ? 32 : 16));
  const int forced = env_int("PF_TC_BN", 0);
  if (forced >= 16 && forced <= kMaxBN && forced <= ((Ng + 15) / 16) * 16 && (forced & (forced - 1)) == 0) BN = forced;
  return BN;
}

#define PF_TMA_ENCODE(call, who)                                                               \
  do {                                                                                         \
    const int e__ = (call);                                                                    \
    if (e__ != 0) {                                                                            \
      pf_set_error("%s: tensor-map encoding failed (%d): %s", who, e__, #call);                \
      return PF_ERR_INVALID_ARG;                                                               \
    }                                                                                          \
  } while (0)

// pass 0: fwd (a = x planes, b = [Cout][Kpad] weights); pass 1: unit-stride dgrad (a = dy planes, b = [Cin][Kpad_d])
int conv_tma_launch(int pass, const TcGeom& g, const pf_tc_act& a, const pf_tc_wt& w, float* out, int accumulate,
                    const float* bias, int relu, const float* residual, cudaStream_t st, const char* who,
                    const pf_tc_bn_out* bn, bool u8) {
  TmaP p;
  memset(&p, 0, sizeof(p));
  const int CC = pass == 0 ? g.C : g.K;
  const int Hs = pass == 0 ? g.H : g.P, Ws = pass == 0 ? g.W : g.Q;      // gathered tensor
  const int Ho = pass == 0 ? g.P : g.H, Wo = pass == 0 ? g.Q : g.W;      // GEMM rows
  const int64_t M64 = (int64_t)g.N * Ho * Wo;
  PF_REQUIRE(M64 < (1ll << 31), "%s: too many rows", who);
  p.M = (int)M64;
  p.Ng = pass == 0 ? g.K : g.C;
  const int Kdim = g.R * g.S * CC;
  p.nk = Kdim / BK;
  p.cblocks = CC / BK;
  p.R = g.R;
  p.S = g.S;
  p.rows_hw = Ho * Wo;
  p.rows_w = Wo;
  p.src_h = Hs;
  p.src_w = Ws;
  if (pass == 0) {
    p.base_w = -g.pl; p.base_h = -g.pt; p.str_w = g.sw; p.str_h = g.sh; p.flip = 0;
  } else {
    p.base_w = g.pl - (g.S - 1); p.base_h = g.pt - (g.R - 1); p.str_w = 1; p.str_h = 1; p.flip = 1;
  }
  p.accumulate = accumulate;
  p.relu = relu;
  const int m_tiles = (p.M + TM - 1) / TM;
  // u8: the tile widths that have an s32 wgmma instantiated (output channels are multiples of 64)
  const int BN = u8 ? (p.Ng >= 128 ? 128 : 64) : pick_bn(p.Ng);
  p.BN = BN;
  p.n_tiles = (p.Ng + BN - 1) / BN;
  p.total_tiles = m_tiles * p.n_tiles;
  p.d_hw = make_fastdiv((uint32_t)p.rows_hw);
  p.d_w = make_fastdiv((uint32_t)p.rows_w);
  p.d_ntiles = make_fastdiv((uint32_t)p.n_tiles);
  p.d_cblocks = make_fastdiv((uint32_t)p.cblocks);
  p.d_s = make_fastdiv((uint32_t)g.S);
  p.na = a.plane1 ? 2 : 1;
  p.nb = w.plane1 ? 2 : 1;
  p.a_hdr = a.hdr;
  PF_REQUIRE(a.hdr == nullptr || a.plane1 != nullptr || u8, "%s: an operand with a device header needs both planes",
             who);
  int aff = 0;
  PF_REQUIRE(!u8 || (pass == 0 && w.alpha != nullptr && a.hdr != nullptr && a.plane1 == nullptr && w.plane1 == nullptr &&
                      p.Ng % 64 == 0),
             "%s: u8 operands are a forward pass of activation levels with a header and weight levels", who);
  if (w.alpha) {
    PF_REQUIRE(w.beta != nullptr && w.bits >= 1 && w.bits <= 8, "%s: weight levels need alpha, beta and 1..8 bits", who);
    PF_REQUIRE(a.csum != nullptr && a.nseg >= 1, "%s: weight levels need the operand's channel sums", who);
    aff = 2;
    p.aff.w_alpha = w.alpha;
    p.aff.w_beta = w.beta;
    p.aff.per_channel = w.per_channel;
    p.aff.w_rk = 1.f / (float)((1 << w.bits) - 1);
    p.aff.w_centre = u8 ? 0.f : (float)(1 << (w.bits - 1));      // u8 weight levels are stored as they are
    p.aff.a_scale = a.hdr ? &a.hdr->scale : nullptr;
    p.csum = a.csum;
    p.nseg = a.nseg;
  } else if (a.hdr) {
    aff = 1;
    p.aff.a_scale = &a.hdr->scale;
  }
  PF_REQUIRE(bn == nullptr || (pass == 0 && (aff == 0 || u8)), "%s: the folded batch norm needs a split-bf16 or u8 forward",
             who);
  if (bn) p.bn = *bn;
  // ---- shared memory: [stages][accumulator tile, row offsets, J, column constants][residual ring]
  const int row_bytes = u8 ? 64 : 128;                  // one k-stage row: 64 channels of bf16 or of u8
  const int stage_max = (p.na * TM + p.nb * BN) * row_bytes;
  const bool has_extra = residual != nullptr || accumulate;
  const int aff_tab_bytes = (aff == 2 ? 2 * 256 * 4 : 0) + (bn ? 4 * kMaxBN * 4 : 0);   // the tile's per-column constants
  const int epi_bytes = epi_fixed_bytes(BN) + aff_tab_bytes;
  // the residual / accumulate operand streams through a per-warp cp.async ring of 4 (else 2) 4 KB chunks when the
  // pipeline keeps enough stages beside it: 3, or nk + 1 for the short reductions of the 1x1 layers (a 64 -> 256 layer
  // has ONE k-stage per tile: two stages already let the next tile's loads fly during this tile's MMAs)
  int budget = (kSmemLimit - epi_bytes) / 1024 * 1024;
  int ring_bytes = 0;
  p.ring = 0;
  if (has_extra && env_int("PF_TC_RING", 1) && BN >= 64) {
    const int need = std::min(3, p.nk + 1);
    for (int depth = kRingDepth; depth >= 2 && !p.ring; depth >>= 1) {
      const int rb = kMmaWarps * depth * kRingSlotBytes;
      if ((budget - rb) / stage_max >= need) {
        p.ring = depth;
        ring_bytes = rb;
      }
    }
    if (p.ring) budget = (kSmemLimit - epi_bytes - ring_bytes) / 1024 * 1024;
  }
  // a split-bf16 / bf16 128 x 128 tile without a residual / accumulate operand or a folded batch norm goes through the
  // staging tile one 32-column chunk at a time when the 48 KB saved buy the pipeline another stage the k-loop can use
  // (split x split: 3 stages instead of 2)
  int used_epi = epi_bytes;
  p.chunked = 0;
  if (BN == 128 && aff == 0 && !bn && !has_extra && p.nk >= 3) {
    const int chunk_epi = epi_fixed_bytes(32);
    const int chunk_budget = (kSmemLimit - chunk_epi) / 1024 * 1024;
    if (budget / stage_max < 3 && chunk_budget / stage_max > budget / stage_max) {
      p.chunked = 1;
      budget = chunk_budget;
      used_epi = chunk_epi;
    }
  }
  PF_REQUIRE(budget / stage_max >= 2 || p.nk <= 1, "%s: shared-memory plan failed (BN %d)", who, BN);
  p.stage_budget = budget;
  const size_t smem = (size_t)budget + used_epi + (p.ring ? ring_bytes : 0);
  const int grid = std::min(p.total_tiles, PF_NUM_SMS);
  record_plan(pf_tc_plan{0, 1, pass, 0, BN, aff, p.na, p.nb, 0, p.ring, 0, budget, p.total_tiles, grid, 0, 0});
  if (p.total_tiles == 0) return PF_OK;
  // ---- tensor maps
  alignas(64) CUtensorMap tA0, tA1, tB0, tB1;
  const int Kpad = pad64(Kdim);
  if (u8) {
    PF_TMA_ENCODE(encode_im2col_u8(&tA0, a.plane0, g.N, Hs, Ws, CC, p.base_w, p.base_h, Wo, Ho, p.str_w, p.str_h, BK, TM), who);
    PF_TMA_ENCODE(encode_2d_u8(&tB0, w.plane0, (uint64_t)Kpad, (uint64_t)p.Ng, (uint64_t)Kpad, BK, (uint32_t)BN), who);
    auto kern = BN == 128 ? (bn ? conv_tma_kernel<2, 128, true, true> : conv_tma_kernel<2, 128, false, true>)
                          : (bn ? conv_tma_kernel<2, 64, true, true> : conv_tma_kernel<2, 64, false, true>);
    PF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, kPingPongThreads, smem, st>>>(tA0, tA0, tB0, tB0, out, bias, residual, p);
    PF_CHECK_LAUNCH(who);
    return PF_OK;
  }
  PF_TMA_ENCODE(encode_im2col_bf16(&tA0, a.plane0, g.N, Hs, Ws, CC, p.base_w, p.base_h, Wo, Ho, p.str_w, p.str_h, BK, TM), who);
  if (a.plane1)
    PF_TMA_ENCODE(encode_im2col_bf16(&tA1, a.plane1, g.N, Hs, Ws, CC, p.base_w, p.base_h, Wo, Ho, p.str_w, p.str_h, BK, TM), who);
  else
    tA1 = tA0;
  PF_TMA_ENCODE(encode_2d_bf16(&tB0, w.plane0, (uint64_t)Kpad, (uint64_t)p.Ng, (uint64_t)Kpad, BK, (uint32_t)BN), who);
  if (w.plane1)
    PF_TMA_ENCODE(encode_2d_bf16(&tB1, w.plane1, (uint64_t)Kpad, (uint64_t)p.Ng, (uint64_t)Kpad, BK, (uint32_t)BN), who);
  else
    tB1 = tB0;
  cudaError_t err = cudaSuccess;
  with_bn(BN, [&](auto bn_c) {
    constexpr int B = decltype(bn_c)::value;
    auto kern = bn ? conv_tma_kernel<0, B, true>
                   : (aff == 2 ? conv_tma_kernel<2, B> : (aff == 1 ? conv_tma_kernel<1, B> : conv_tma_kernel<0, B>));
    err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err == cudaSuccess) kern<<<grid, kPingPongThreads, smem, st>>>(tA0, tA1, tB0, tB1, out, bias, residual, p);
  });
  PF_CUDA(err);
  PF_CHECK_LAUNCH(who);
  return PF_OK;
}

int conv_tma_wgrad_launch(const TcGeom& g, const pf_tc_act& x, const pf_tc_act& dy, int BN, int pps, int splits,
                          float* partial, cudaStream_t st, const char* who) {
  WgTmaP p;
  memset(&p, 0, sizeof(p));
  p.g = g;
  p.Mtot = g.R * g.S * g.C;
  p.Npix = g.N * g.P * g.Q;
  p.BN = BN;
  p.pps = pps;
  p.splits = splits;
  const int m_tiles = (p.Mtot + TM - 1) / TM;
  p.n_tiles = (g.K + BN - 1) / BN;
  p.tiles = m_tiles * p.n_tiles;
  p.total_units = p.tiles * p.splits;
  p.d_pq = make_fastdiv((uint32_t)(g.P * g.Q));
  p.d_q = make_fastdiv((uint32_t)g.Q);
  p.d_c = make_fastdiv((uint32_t)g.C);
  p.d_s = make_fastdiv((uint32_t)g.S);
  p.d_tiles = make_fastdiv((uint32_t)p.tiles);
  p.d_ntiles = make_fastdiv((uint32_t)p.n_tiles);
  p.na = x.plane1 ? 2 : 1;
  p.nb = dy.plane1 ? 2 : 1;
  p.x_hdr = x.hdr;
  PF_REQUIRE(x.hdr == nullptr || x.plane1 != nullptr, "%s: an operand with a device header needs both planes", who);
  PF_REQUIRE(dy.hdr == nullptr, "%s: the gradient operand is always split-bf16", who);
  int aff = 0;
  if (x.hdr) {
    aff = 1;
    p.aff.a_scale = &x.hdr->scale;
  }
  const int stage_max = p.na * 2 * (int)kWgBlockBytes + p.nb * (BN / 64) * (int)kWgBlockBytes;
  const int budget = (kSmemLimit - epi_fixed_bytes(BN)) / 1024 * 1024;
  PF_REQUIRE(budget / stage_max >= 2, "%s: shared-memory plan failed (BN %d)", who, BN);
  p.stage_budget = budget;
  const size_t smem = (size_t)budget + epi_fixed_bytes(BN);
  const int grid = std::min(p.total_units, PF_NUM_SMS);
  record_plan(pf_tc_plan{0, 1, 2, 0, BN, aff, p.na, p.nb, 0, 0, 0, budget, p.total_units, grid, splits, pps});
  if (p.total_units == 0) return PF_OK;
  alignas(64) CUtensorMap tX0, tX1, tY0, tY1;
  PF_TMA_ENCODE(encode_im2col_bf16(&tX0, x.plane0, g.N, g.H, g.W, g.C, -g.pl, -g.pt, g.Q, g.P, g.sw, g.sh, BK, BK), who);
  if (x.plane1)
    PF_TMA_ENCODE(encode_im2col_bf16(&tX1, x.plane1, g.N, g.H, g.W, g.C, -g.pl, -g.pt, g.Q, g.P, g.sw, g.sh, BK, BK), who);
  else
    tX1 = tX0;
  PF_TMA_ENCODE(encode_2d_bf16(&tY0, dy.plane0, (uint64_t)g.K, (uint64_t)p.Npix, (uint64_t)g.K, BK, BK), who);
  if (dy.plane1)
    PF_TMA_ENCODE(encode_2d_bf16(&tY1, dy.plane1, (uint64_t)g.K, (uint64_t)p.Npix, (uint64_t)g.K, BK, BK), who);
  else
    tY1 = tY0;
  auto kern = BN == 128 ? (aff == 1 ? conv_tma_wgrad_kernel<1, 128> : conv_tma_wgrad_kernel<0, 128>)
                        : (aff == 1 ? conv_tma_wgrad_kernel<1, 64> : conv_tma_wgrad_kernel<0, 64>);
  PF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, kTmaThreads, smem, st>>>(tX0, tX1, tY0, tY1, partial, p);
  PF_CHECK_LAUNCH(who);
  return PF_OK;
}

}  // namespace pfconv
