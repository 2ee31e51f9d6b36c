// pf_tma.cuh — Tensor Memory Accelerator plumbing for the wgmma convolution kernels (sm_90a):
//   host : CUtensorMap encoding (tiled 2-D for the weight / gradient matrices, im2col 4-D for NHWC activations)
//          through the driver entry points fetched with cudaGetDriverEntryPoint (no link against libcuda);
//   device: cp.async.bulk.tensor wrappers (SASS: UTMALDG), mbarrier transaction counts, a bounded mbarrier wait.
// Parameter conventions of the im2col mode follow cuda.h (cuTensorMapEncodeIm2col) and were cross-checked against
// cute/atom/copy_traits_sm90_im2col.hpp of the vendored CUTLASS headers (corner arrays in W,H order; coordinates
// {c, w, h, n} = position of the filter window's first tap for the first pixel of the column, offsets {s, r}).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "pf_tc_common.cuh"

namespace pftma {

// ------------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

inline void* driver_entry(const char* name) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess)
    return nullptr;
  return fn;
}

// Drivers up to CUDA 13.1 mis-encode descriptors of tensors smaller than 128 KiB (bit 21 of the second quadword must be
// cleared) — the same fix-up CUTLASS applies after every encode call.
inline void small_tensor_fixup(CUtensorMap* m, uint64_t tensor_bytes) {
  static int drv = -1;
  if (drv < 0) cudaDriverGetVersion(&drv);
  if (drv <= 13010 && tensor_bytes < 131072) reinterpret_cast<uint64_t*>(m)[1] &= ~(1ull << 21);
}

// matrix [rows][cols] of `esize`-byte elements (cols contiguous, row pitch `pitch_elems`), box = box_cols x box_rows,
// swizzled rows of box_cols * esize bytes (128: SWIZZLE_128B, 64: SWIZZLE_64B).  Out-of-range rows / columns of a box
// read as zero.
inline int encode_2d(CUtensorMap* m, CUtensorMapDataType dtype, uint32_t esize, CUtensorMapSwizzle swizzle,
                     const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_elems, uint32_t box_cols,
                     uint32_t box_rows) {
  static EncodeTiledFn fn = (EncodeTiledFn)driver_entry("cuTensorMapEncodeTiled");
  if (!fn) return -1;
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {pitch_elems * esize};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(m, dtype, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return (int)r;
  small_tensor_fixup(m, rows * pitch_elems * esize);
  return 0;
}
// bf16, SWIZZLE_128B (box_cols * 2 bytes <= 128)
inline int encode_2d_bf16(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_elems,
                          uint32_t box_cols, uint32_t box_rows) {
  return encode_2d(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, CU_TENSOR_MAP_SWIZZLE_128B, base, cols, rows, pitch_elems,
                   box_cols, box_rows);
}
// unsigned 8-bit levels, SWIZZLE_64B (box_cols = 64)
inline int encode_2d_u8(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_elems,
                        uint32_t box_cols, uint32_t box_rows) {
  return encode_2d(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, CU_TENSOR_MAP_SWIZZLE_64B, base, cols, rows, pitch_elems,
                   box_cols, box_rows);
}

// NHWC tensor [n][h][w][c] of `esize`-byte elements in im2col mode: a load fetches `pixels` consecutive positions of the filter-window
// origin (walking w, then h, then n, in steps of str_w / str_h inside the bounding box) x `channels` channels of the
// pixel at origin + (off_w, off_h); positions outside the tensor read as zero (the convolution's padding).
//   base_w / base_h : coordinate of the window origin of output position 0 (forward: -pad; dgrad: pad - (S-1))
//   out_w / out_h   : number of window positions per row / column (the bounding box is sized to exactly that)
inline int encode_im2col(CUtensorMap* m, CUtensorMapDataType dtype, uint32_t esize, CUtensorMapSwizzle swizzle,
                         const void* base, int n, int h, int w, int c, int base_w, int base_h, int out_w, int out_h,
                         int str_w, int str_h, uint32_t channels, uint32_t pixels) {
  static EncodeIm2colFn fn = (EncodeIm2colFn)driver_entry("cuTensorMapEncodeIm2col");
  if (!fn) return -1;
  const cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  const cuuint64_t strides[3] = {(cuuint64_t)c * esize, (cuuint64_t)w * c * esize, (cuuint64_t)h * w * c * esize};
  const int lower[2] = {base_w, base_h};
  // the box spans window origins base .. base + (out - 1) * stride: upper corner offset is relative to (dim - 1)
  const int upper[2] = {(out_w - 1) * str_w + base_w + 1 - w, (out_h - 1) * str_h + base_h + 1 - h};
  if (lower[0] < -128 || lower[0] > 127 || lower[1] < -128 || lower[1] > 127 || upper[0] < -128 || upper[0] > 127 ||
      upper[1] < -128 || upper[1] > 127 || str_w > 8 || str_h > 8)
    return -2;
  const cuuint32_t estr[4] = {1, (cuuint32_t)str_w, (cuuint32_t)str_h, 1};
  const CUresult r = fn(m, dtype, 4, const_cast<void*>(base), dims, strides, lower, upper, channels, pixels, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return (int)r;
  small_tensor_fixup(m, (uint64_t)n * h * w * c * esize);
  return 0;
}
inline int encode_im2col_bf16(CUtensorMap* m, const void* base, int n, int h, int w, int c, int base_w, int base_h,
                              int out_w, int out_h, int str_w, int str_h, uint32_t channels, uint32_t pixels) {
  return encode_im2col(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, CU_TENSOR_MAP_SWIZZLE_128B, base, n, h, w, c, base_w,
                       base_h, out_w, out_h, str_w, str_h, channels, pixels);
}
inline int encode_im2col_u8(CUtensorMap* m, const void* base, int n, int h, int w, int c, int base_w, int base_h,
                            int out_w, int out_h, int str_w, int str_h, uint32_t channels, uint32_t pixels) {
  return encode_im2col(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, CU_TENSOR_MAP_SWIZZLE_64B, base, n, h, w, c, base_w,
                       base_h, out_w, out_h, str_w, str_h, channels, pixels);
}

// ------------------------------------------------------------------------------------------------ device
#ifdef __CUDACC__
__device__ __forceinline__ void prefetch_map(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(pftc::smem_u32(bar)), "r"(bytes) : "memory");
}
// 2-D tiled load: box at (col, row) -> smem (128B-swizzled rows), completion counted on `bar`
__device__ __forceinline__ void load_2d(uint32_t dst, const CUtensorMap* m, uint64_t* bar, int col, int row) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(pftc::smem_u32(bar)), "r"(col), "r"(row)
      : "memory");
}
// 4-D im2col load: `pixels` window origins starting at (w, h, n), channels [c, c + channels), tap offset (off_w, off_h)
__device__ __forceinline__ void load_im2col(uint32_t dst, const CUtensorMap* m, uint64_t* bar, int c, int w, int h, int n,
                                            uint32_t off_w, uint32_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], "
      "{%7, %8};" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(pftc::smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"((uint16_t)off_w),
      "h"((uint16_t)off_h)
      : "memory");
}
#endif

}  // namespace pftma
