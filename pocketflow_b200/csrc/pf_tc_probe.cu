// pf_tc_probe.cu — single-CTA wgmma GEMM used to validate the descriptor / swizzle conventions of
// pf_tc_common.cuh on real hardware (tests/test_tc_gpu.py).  D[128 x N] = A * B^T for bf16 operands:
//   mode 0: A [128][K], B [N][K]   both K-major   (conv fwd / dgrad operand layout)
//   mode 1: A [K][128], B [K][N]   both MN-major  (conv wgrad operand layout)
// LBO/SBO are arguments so that one GPU run can sweep the candidates.
#include "pf_common.cuh"
#include "pf_tc_common.cuh"

namespace {
using namespace pftc;

constexpr int TM = 128, BK = 64;

// one warpgroup; the two 64-row halves of D are computed one after the other (A half h starts 8 KB (mode 0) or one
// MN block = lbo_a (mode 1) into the A tile)
template <int N>
__global__ void __launch_bounds__(128)
tc_probe_kernel(const __nv_bfloat16* __restrict__ A, const __nv_bfloat16* __restrict__ B, float* __restrict__ D,
                int K, int mode, uint32_t lbo_a, uint32_t sbo_a, uint32_t lbo_b, uint32_t sbo_b,
                uint32_t kstep_a, uint32_t kstep_b) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = smem;              // 128 x 64 bf16 = 16 KB
  uint8_t* sB = smem + 16384;      // up to 256 x 64 bf16 = 32 KB
  const int tid = threadIdx.x;
  for (int h = 0; h < 2; ++h) {
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    for (int k0 = 0; k0 < K; k0 += BK) {
      // ---- fill the operand tiles (generic proxy)
      if (mode == 0) {
        for (int e = tid; e < TM * BK; e += 128) {
          const int r = e / BK, k = e % BK;
          *reinterpret_cast<__nv_bfloat16*>(sA + sw128_offset(r, k)) = A[(size_t)r * K + k0 + k];
        }
        for (int e = tid; e < N * BK; e += 128) {
          const int r = e / BK, k = e % BK;
          *reinterpret_cast<__nv_bfloat16*>(sB + sw128_offset(r, k)) = B[(size_t)r * K + k0 + k];
        }
      } else {
        // MN-major: tile[kb = k/8][mb = m/64][k8 = k%8] rows of 64 MN-contiguous elements (128 B)
        for (int e = tid; e < TM * BK; e += 128) {
          const int k = e / TM, m = e % TM;
          const uint32_t row = (uint32_t)((k >> 3) * (TM / 64) * 8 + (m >> 6) * 8 + (k & 7));
          *reinterpret_cast<__nv_bfloat16*>(sA + sw128_offset(row, m & 63)) = A[(size_t)(k0 + k) * TM + m];
        }
        for (int e = tid; e < N * BK; e += 128) {
          const int k = e / N, n = e % N;
          const uint32_t row = (uint32_t)((k >> 3) * (N / 64) * 8 + (n >> 6) * 8 + (k & 7));
          *reinterpret_cast<__nv_bfloat16*>(sB + sw128_offset(row, n & 63)) = B[(size_t)(k0 + k) * N + n];
        }
      }
      fence_proxy_async_smem();
      __syncthreads();
      const uint32_t a_half = smem_u32(sA) + (uint32_t)h * (mode == 0 ? 64u * 128u : lbo_a);
      wgmma_fence();
      for (int kk = 0; kk < BK / 16; ++kk) {
        const uint64_t da = make_smem_desc(a_half + kk * kstep_a, lbo_a, sbo_a);
        const uint64_t db = make_smem_desc(smem_u32(sB) + kk * kstep_b, lbo_b, sbo_b);
        if (mode == 0) Wgmma<N>::template mma<0, 0>(acc, da, db);
        else Wgmma<N>::template mma<1, 1>(acc, da, db);
      }
      wgmma_commit();
      wgmma_wait<0>(acc);
      __syncthreads();             // the tiles are refilled next
    }
    wgmma_store_acc<N>(acc, D, N, 64 * h, tid);
  }
}
}  // namespace

extern "C" int pf_tc_probe(const void* a_dev, const void* b_dev, float* d_dev, int n, int k, int mode,
                           uint32_t lbo_a, uint32_t sbo_a, uint32_t lbo_b, uint32_t sbo_b, uint32_t kstep_a,
                           uint32_t kstep_b, void* stream) {
  PF_REQUIRE(a_dev && b_dev && d_dev, "pf_tc_probe: null pointer");
  PF_REQUIRE(n >= 16 && n <= 256 && (n & (n - 1)) == 0 && k > 0 && k % 64 == 0, "pf_tc_probe: bad shape");
  PF_REQUIRE(mode == 0 || (mode == 1 && n % 64 == 0), "pf_tc_probe: bad mode");
  const int smem = 16384 + 32768 + 1024;
  auto kern = n == 16 ? tc_probe_kernel<16> : n == 32 ? tc_probe_kernel<32> : n == 64 ? tc_probe_kernel<64>
            : n == 128 ? tc_probe_kernel<128> : tc_probe_kernel<256>;
  PF_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kern<<<1, 128, smem, (cudaStream_t)stream>>>((const __nv_bfloat16*)a_dev, (const __nv_bfloat16*)b_dev, d_dev, k, mode,
                                               lbo_a, sbo_a, lbo_b, sbo_b, kstep_a, kstep_b);
  PF_CHECK_LAUNCH("pf_tc_probe");
  return PF_OK;
}
