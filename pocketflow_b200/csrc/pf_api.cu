// pf_api.cu — error reporting, launch accounting, small utilities of libpf_b200.so.
#include <stdarg.h>

#include <atomic>

#include "pf_common.cuh"

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void pf_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void pf_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

extern "C" {

int pf_abi_version(void) { return PF_B200_ABI_VERSION; }
const char* pf_last_error(void) { return g_err; }
int64_t pf_launch_count(void) { return g_launches.load(); }
void pf_launch_count_reset(void) { g_launches.store(0); }

}  // extern "C"

int pf_num_sms() {
  static int cached[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] <= 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 1;
    cached[dev] = n;
  }
  return cached[dev];
}

extern "C" {

int pf_sm_count(int* out) {
  PF_REQUIRE(out != nullptr, "pf_sm_count: null out");
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    pf_set_error("pf_sm_count: no CUDA device: %s", cudaGetErrorString(e));
    return PF_ERR_NO_DEVICE;
  }
  PF_CUDA(cudaDeviceGetAttribute(out, cudaDevAttrMultiProcessorCount, dev));
  return PF_OK;
}

__global__ void pf_fill_u32_kernel(uint32_t* p, int64_t n, uint32_t v) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) p[i] = v;
}

__global__ void pf_minmax_reset_kernel(uint32_t* p, int64_t n_pairs) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_pairs) {
    p[2 * i] = 0xFFFFFFFFu;
    p[2 * i + 1] = 0u;
  }
}

int pf_minmax_reset(uint32_t* pairs_dev, int64_t n_pairs, void* stream) {
  PF_REQUIRE(n_pairs >= 0 && (pairs_dev != nullptr || n_pairs == 0), "pf_minmax_reset: bad arguments");
  if (n_pairs == 0) return PF_OK;
  pf_minmax_reset_kernel<<<(unsigned)((n_pairs + 255) / 256), 256, 0, (cudaStream_t)stream>>>(pairs_dev, n_pairs);
  PF_CHECK_LAUNCH("pf_minmax_reset");
  return PF_OK;
}

int pf_fill_u32(uint32_t* p_dev, int64_t n, uint32_t value, void* stream) {
  PF_REQUIRE(n >= 0 && (p_dev != nullptr || n == 0), "pf_fill_u32: bad arguments");
  if (n == 0) return PF_OK;
  int64_t blocks = (n + 255) / 256;
  if (blocks > PF_NUM_SMS * 8) blocks = PF_NUM_SMS * 8;
  pf_fill_u32_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(p_dev, n, value);
  PF_CHECK_LAUNCH("pf_fill_u32");
  return PF_OK;
}

}  // extern "C"
