// pf_jpeg.cu — baseline JPEG decoding on the device, bit for bit with libjpeg-turbo's default decompression (the
// library behind Pillow's decode_jpeg in datasets/ilsvrc12_dataset.py): Huffman decoding, the jidctint.c ("islow")
// integer IDCT, jdsample.c's fancy (triangle) upsampling and jdcolor.c's fixed-point YCbCr -> RGB, written straight
// into the crop window the input pipeline asked for.
//
// The host parses every header (datasets/jpeg.py) and hands over one pf_jpeg_desc per image: only files the device
// supports get one (8-bit, one interleaved sequential Huffman scan, grey or YCbCr with luma sampling 1x1, 2x1, 2x2 and
// chroma 1x1).  Three launches:
//   1. entropy decode, one thread per image: int16 zig-zag coefficients of every block of the MCU rows the crop needs,
//      in MCU order, into the caller's workspace.  Every read is bounded by the image's own segment; a code that is
//      not in the table, a run past coefficient 63, bits taken past the segment's data or a wrong restart marker set
//      status[i] and end that image (the host then decodes it, so whatever libjpeg does with such data is kept).
//   2. dequantise + islow IDCT of the MCU window the crop needs (upsampling context included), one thread per block,
//      in place: the block's 64 samples overwrite the first 64 bytes of its 128-byte coefficient slot.
//   3. upsample + colour-convert + crop, one thread per output pixel.
// All per-image, per-block and per-pixel arithmetic is in __host__ __device__ functions; compiled with
// -DPF_JPEG_HOST_TEST the same source exports pf_test_jpeg_decode_host, a plain loop over them that tests run on the
// CPU against Pillow.  That loop is never part of libpf_b200.so.
#ifndef PF_JPEG_HOST_TEST
#include "pf_common.cuh"
#else
#include <stdint.h>
#include <string.h>
#include "pf_b200.h"
#endif

namespace {

enum { JPEG_OK = 0, JPEG_BAD_CODE = 1, JPEG_OUT_OF_DATA = 2, JPEG_BAD_RESTART = 3, JPEG_BAD_RUN = 4, JPEG_BAD_DESC = 5 };

// ------------------------------------------------------------------------------------------- entropy decoding
// MSB-first bit buffer over one entropy-coded segment.  Stuffed 0xFF00 is a 0xFF data byte, 0xFF fill bytes before a
// marker are skipped (jdhuff.c jpeg_fill_bit_buffer).  At a marker or at the segment's end the buffer is padded with
// zero bits, as libjpeg does; taking a padding bit is an anomaly here (`real` counts the data bits still buffered).
struct BitReader {
  const uint8_t* p;
  int64_t pos, end;
  uint64_t buf;
  int bits, real;
  int marker;        // marker code met (0: none yet); p[pos] is then the byte after it
};

__host__ __device__ inline void br_init(BitReader& b, const uint8_t* p, int64_t pos, int64_t end) {
  b.p = p;
  b.pos = pos;
  b.end = end;
  b.buf = 0;
  b.bits = b.real = 0;
  b.marker = 0;
}

__host__ __device__ inline void br_fill(BitReader& b) {
  while (b.bits <= 56) {
    int c = 0;
    if (!b.marker && b.pos < b.end) {
      c = b.p[b.pos++];
      if (c == 0xFF) {
        int m = 0xFF;
        while (m == 0xFF && b.pos < b.end) m = b.p[b.pos++];
        if (m == 0xFF) {               // the segment ends inside fill bytes
          b.marker = 0x100;
          c = 0;
        } else if (m == 0) {
          c = 0xFF;
        } else {
          b.marker = m;
          c = 0;
        }
      }
      if (!b.marker) b.real += 8;
    }
    b.buf = (b.buf << 8) | (uint64_t)c;
    b.bits += 8;
  }
}

__host__ __device__ inline int br_peek(BitReader& b, int n) {
  if (b.bits < n) br_fill(b);
  return (int)((b.buf >> (b.bits - n)) & ((1u << n) - 1));
}

// false: the bits would come from the padding
__host__ __device__ inline bool br_skip(BitReader& b, int n) {
  if (b.real < n) return false;
  b.bits -= n;
  b.real -= n;
  return true;
}

// one Huffman symbol (jdhuff.c jpeg_huff_decode); -1: no code of <= 16 bits matches, -2: out of data
__host__ __device__ inline int huff_decode(BitReader& b, const pf_jpeg_huff& h) {
  br_fill(b);
  const int look = br_peek(b, 8);
  const int v = h.lookup[look];
  if (v) {
    if (!br_skip(b, v >> 8)) return -2;
    return v & 0xFF;
  }
  for (int l = 9; l <= 16; ++l) {
    const int code = br_peek(b, l);
    if (code <= h.maxcode[l]) {
      if (!br_skip(b, l)) return -2;
      return h.huffval[(code + h.valoffset[l]) & 0xFF];
    }
  }
  return -1;
}

// s extra bits, sign-extended (HUFF_EXTEND); s in 1..15.  *ok = false: out of data
__host__ __device__ inline int get_extend(BitReader& b, int s, bool* ok) {
  br_fill(b);
  const int r = br_peek(b, s);
  *ok = br_skip(b, s);
  return r < (1 << (s - 1)) ? r + ((-1) << s) + 1 : r;
}

__host__ __device__ inline int blocks_per_mcu(const pf_jpeg_desc& d) { return d.ncomp == 1 ? 1 : d.hs * d.vs + 2; }

// The MCU window [mcu_row0, mcu_rows) x [mcu_col0, mcu_col1] holds every block the crop reads: its luma rows and
// columns, and the chroma rows and columns the fancy upsampler reads, one neighbour each way, clamped to the plane.
// (Called once the crop is known to lie inside the image.)
__host__ __device__ inline bool window_covers_crop(const pf_jpeg_desc& d) {
  const int mh = 8 * d.vs, mw = 8 * d.hs;
  const int y1 = d.crop_y + d.crop_h - 1, x1 = d.crop_x + d.crop_w - 1;
  int r0 = d.crop_y / mh, r1 = y1 / mh, c0 = d.crop_x / mw, c1 = x1 / mw;
  if (d.ncomp == 3) {
    const int ch = (d.height + d.vs - 1) / d.vs, cw = (d.width + d.hs - 1) / d.hs;
    const int cy0 = d.crop_y / d.vs - (d.vs - 1), cy1 = y1 / d.vs + (d.vs - 1);
    const int cx0 = d.crop_x / d.hs - (d.hs - 1), cx1 = x1 / d.hs + (d.hs - 1);
    const int rr0 = (cy0 > 0 ? cy0 : 0) >> 3, rr1 = (cy1 < ch - 1 ? cy1 : ch - 1) >> 3;
    const int cc0 = (cx0 > 0 ? cx0 : 0) >> 3, cc1 = (cx1 < cw - 1 ? cx1 : cw - 1) >> 3;
    r0 = r0 < rr0 ? r0 : rr0;
    r1 = r1 > rr1 ? r1 : rr1;
    c0 = c0 < cc0 ? c0 : cc0;
    c1 = c1 > cc1 ? c1 : cc1;
  }
  return d.mcu_row0 <= r0 && r1 < d.mcu_rows && d.mcu_col0 <= c0 && c1 <= d.mcu_col1;
}

__host__ __device__ inline bool desc_ok(const pf_jpeg_desc& d) {
  const bool samp = d.ncomp == 1 ? (d.hs == 1 && d.vs == 1)
                                 : (d.ncomp == 3 && (d.hs == 1 || d.hs == 2) && (d.vs == 1 || d.vs == 2) && d.hs >= d.vs);
  if (!samp || d.height <= 0 || d.width <= 0 || d.scan_bytes < 0 || d.restart_interval < 0) return false;
  if (d.mcus_per_row != (d.width + 8 * d.hs - 1) / (8 * d.hs) || d.mcu_rows <= 0 ||
      d.mcu_rows > (d.height + 8 * d.vs - 1) / (8 * d.vs))
    return false;
  if (d.crop_h <= 0 || d.crop_w <= 0 || d.crop_y < 0 || d.crop_x < 0 || d.crop_y + d.crop_h > d.height ||
      d.crop_x + d.crop_w > d.width)
    return false;
  if (d.mcu_row0 < 0 || d.mcu_row0 >= d.mcu_rows || d.mcu_col0 < 0 || d.mcu_col1 < d.mcu_col0 ||
      d.mcu_col1 >= d.mcus_per_row)
    return false;
  for (int c = 0; c < d.ncomp; ++c)
    if (d.dc_tbl[c] < 0 || d.dc_tbl[c] > 3 || d.ac_tbl[c] < 0 || d.ac_tbl[c] > 3) return false;
  return window_covers_crop(d);
}

// Entropy-decodes one image's MCU rows [0, mcu_rows) into ws (64 int16 per block, zig-zag order).  Returns a status.
__host__ __device__ inline int jpeg_entropy_image(const uint8_t* data, const pf_jpeg_desc& d, int16_t* ws) {
  if (!desc_ok(d)) return JPEG_BAD_DESC;
  BitReader b;
  br_init(b, data + d.scan_offset, 0, d.scan_bytes);
  const int bpm = blocks_per_mcu(d);
  const int nmcu = d.mcus_per_row * d.mcu_rows;
  int pred[3] = {0, 0, 0};
  int restarts_left = d.restart_interval, next_rst = 0;
  int16_t* blk = ws + d.coef_offset;
  for (int m = 0; m < nmcu; ++m) {
    if (d.restart_interval) {
      if (restarts_left == 0) {
        // jdhuff.c process_restart: drop the buffered bits, expect RSTn right after the data bytes
        if (b.real >= 8) return JPEG_BAD_RESTART;
        if (!b.marker) {
          b.bits = b.real = 0;
          br_fill(b);
          if (b.real) return JPEG_BAD_RESTART;
        }
        if (b.marker != 0xD0 + next_rst) return JPEG_BAD_RESTART;
        br_init(b, b.p, b.pos, b.end);
        pred[0] = pred[1] = pred[2] = 0;
        next_rst = (next_rst + 1) & 7;
        restarts_left = d.restart_interval;
      }
      --restarts_left;
    }
    for (int k = 0; k < bpm; ++k, blk += 64) {
      const int c = (d.ncomp == 1 || k < d.hs * d.vs) ? 0 : k - d.hs * d.vs + 1;
      for (int z = 0; z < 64; ++z) blk[z] = 0;
      bool ok = true;
      int s = huff_decode(b, d.huff[d.dc_tbl[c]]);
      if (s < 0) return s == -1 ? JPEG_BAD_CODE : JPEG_OUT_OF_DATA;
      int diff = 0;
      if (s) {
        if (s > 15) return JPEG_BAD_CODE;
        diff = get_extend(b, s, &ok);
        if (!ok) return JPEG_OUT_OF_DATA;
      }
      pred[c] = (int)((unsigned)pred[c] + (unsigned)diff);         // 32-bit wrap, stored as JCOEF (int16)
      blk[0] = (int16_t)pred[c];
      const pf_jpeg_huff& ac = d.huff[d.ac_tbl[c]];
      for (int z = 1; z < 64; ++z) {
        const int rs = huff_decode(b, ac);
        if (rs < 0) return rs == -1 ? JPEG_BAD_CODE : JPEG_OUT_OF_DATA;
        const int r = rs >> 4, sz = rs & 15;
        if (sz) {
          z += r;
          if (z > 63) return JPEG_BAD_RUN;
          blk[z] = (int16_t)get_extend(b, sz, &ok);
          if (!ok) return JPEG_OUT_OF_DATA;
        } else {
          if (r != 15) break;                                         // EOB
          z += 15;                                                    // ZRL
        }
      }
    }
  }
  return JPEG_OK;
}

// ------------------------------------------------------------------------------------------- islow IDCT
constexpr int CONST_BITS = 13, PASS1_BITS = 2;
constexpr int64_t FIX_0_298631336 = 2446, FIX_0_390180644 = 3196, FIX_0_541196100 = 4433, FIX_0_765366865 = 6270,
                  FIX_0_899976223 = 7373, FIX_1_175875602 = 9633, FIX_1_501321110 = 12299, FIX_1_847759065 = 15137,
                  FIX_1_961570560 = 16069, FIX_2_053119869 = 16819, FIX_2_562915447 = 20995, FIX_3_072711026 = 25172;

__host__ __device__ inline int64_t descale(int64_t x, int n) { return (x + ((int64_t)1 << (n - 1))) >> n; }

// idct range_limit[x & RANGE_MASK] (jdmaster.c prepare_range_limit_table): the low 10 bits read as a signed value
// v in [-512, 511], then clamp(v + 128, 0, 255)
__host__ __device__ inline uint8_t idct_limit(int64_t x) {
  const int v = (int)(((x & 1023) ^ 512) - 512) + 128;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

__host__ __device__ inline int zigzag_index(int natural) {
  // position in zig-zag order of natural (row-major) coefficient `natural`
  const uint8_t zz[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42, 3,  8,  12, 17, 25, 30,
                          41, 43, 9,  11, 18, 24, 31, 40, 44, 53, 10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38,
                          46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};
  return zz[natural];
}

// one even/odd butterfly of jidctint.c on 8 dequantised inputs in natural order, stride 1
__host__ __device__ inline void idct_1d(const int64_t in[8], int64_t out[8], int shift_const) {
  int64_t z2 = in[2], z3 = in[6];
  int64_t z1 = (z2 + z3) * FIX_0_541196100;
  int64_t tmp2 = z1 + z3 * (-FIX_1_847759065);
  int64_t tmp3 = z1 + z2 * FIX_0_765366865;
  z2 = in[0];
  z3 = in[4];
  int64_t tmp0 = (z2 + z3) * ((int64_t)1 << CONST_BITS);
  int64_t tmp1 = (z2 - z3) * ((int64_t)1 << CONST_BITS);
  const int64_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in[7];
  tmp1 = in[5];
  tmp2 = in[3];
  tmp3 = in[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  int64_t z4 = tmp1 + tmp3;
  const int64_t z5 = (z3 + z4) * FIX_1_175875602;
  tmp0 *= FIX_0_298631336;
  tmp1 *= FIX_2_053119869;
  tmp2 *= FIX_3_072711026;
  tmp3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223;
  z2 *= -FIX_2_562915447;
  z3 *= -FIX_1_961570560;
  z4 *= -FIX_0_390180644;
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  out[0] = descale(tmp10 + tmp3, shift_const);
  out[7] = descale(tmp10 - tmp3, shift_const);
  out[1] = descale(tmp11 + tmp2, shift_const);
  out[6] = descale(tmp11 - tmp2, shift_const);
  out[2] = descale(tmp12 + tmp1, shift_const);
  out[5] = descale(tmp12 - tmp1, shift_const);
  out[3] = descale(tmp13 + tmp0, shift_const);
  out[4] = descale(tmp13 - tmp0, shift_const);
}

// dequantise + jpeg_idct_islow of one block, in place: 64 int16 zig-zag coefficients -> 64 uint8 samples (row-major)
// in the slot's first 64 bytes.  The shortcuts jidctint.c takes for all-zero AC columns / rows give the same values
// as the full butterflies, so they are not restated.
__host__ __device__ inline void idct_block(int16_t* blk, const uint16_t* quant_zz) {
  int32_t ws[64];
  for (int col = 0; col < 8; ++col) {
    int64_t in[8], out[8];
    for (int r = 0; r < 8; ++r) {
      const int z = zigzag_index(r * 8 + col);
      in[r] = (int64_t)((int32_t)blk[z] * (int32_t)quant_zz[z]);
    }
    idct_1d(in, out, CONST_BITS - PASS1_BITS);
    for (int r = 0; r < 8; ++r) ws[r * 8 + col] = (int32_t)out[r];
  }
  uint8_t* dst = (uint8_t*)blk;
  for (int row = 0; row < 8; ++row) {
    int64_t in[8], out[8];
    for (int c = 0; c < 8; ++c) in[c] = ws[row * 8 + c];
    idct_1d(in, out, CONST_BITS + PASS1_BITS + 3);
    for (int c = 0; c < 8; ++c) dst[row * 8 + c] = idct_limit(out[c]);
  }
}

// block j of image d's inverse-transformed window -> its coefficient slot and component; false: j is past the window
__host__ __device__ inline bool idct_block_at(const pf_jpeg_desc& d, int64_t j, int64_t* slot, int* comp) {
  const int bpm = blocks_per_mcu(d);
  const int64_t cols = d.mcu_col1 - d.mcu_col0 + 1;
  const int64_t per_row = cols * bpm;
  const int64_t row = j / per_row;
  if (row >= d.mcu_rows - d.mcu_row0) return false;
  const int64_t rem = j - row * per_row;
  const int64_t mcu = (row + d.mcu_row0) * d.mcus_per_row + d.mcu_col0 + rem / bpm;
  const int k = (int)(rem % bpm);
  *slot = d.coef_offset + (mcu * bpm + k) * 64;
  *comp = (d.ncomp == 1 || k < d.hs * d.vs) ? 0 : k - d.hs * d.vs + 1;
  return true;
}

// ------------------------------------------------------------------------------------------- upsample + colour
// sample (r, c) of component comp, read from its inverse-transformed block
__host__ __device__ inline int comp_sample(const int16_t* ws, const pf_jpeg_desc& d, int comp, int r, int c) {
  const int bpm = blocks_per_mcu(d);
  int64_t mcu;
  int k;
  if (comp == 0) {
    mcu = (int64_t)(r / (8 * d.vs)) * d.mcus_per_row + c / (8 * d.hs);
    k = ((r % (8 * d.vs)) >> 3) * d.hs + ((c % (8 * d.hs)) >> 3);
  } else {
    mcu = (int64_t)(r >> 3) * d.mcus_per_row + (c >> 3);
    k = d.hs * d.vs + comp - 1;
  }
  const uint8_t* s = (const uint8_t*)(ws + d.coef_offset + (mcu * bpm + k) * 64);
  return s[(r & 7) * 8 + (c & 7)];
}

// one chroma value at output pixel (y, x): jdsample.c h2v1 / h2v2 fancy upsampling (edges by replication, which is
// what the first / last column and the context rows of libjpeg's main buffer amount to); a downsampled width <= 2
// falls back to plain replication, as jinit_upsampler does
__host__ __device__ inline int chroma_at(const int16_t* ws, const pf_jpeg_desc& d, int comp, int y, int x) {
  if (d.hs == 1) return comp_sample(ws, d, comp, y, x);
  const int cw = (d.width + 1) >> 1, ch = (d.height + d.vs - 1) / d.vs;
  const int c = x >> 1, cn = (x & 1) ? (c + 1 < cw ? c + 1 : cw - 1) : (c > 0 ? c - 1 : 0);
  if (cw <= 2) return comp_sample(ws, d, comp, y / d.vs, c);
  if (d.vs == 1) {
    const int v = 3 * comp_sample(ws, d, comp, y, c) + comp_sample(ws, d, comp, y, cn);
    return (v + ((x & 1) ? 2 : 1)) >> 2;
  }
  const int r = y >> 1, rn = (y & 1) ? (r + 1 < ch ? r + 1 : ch - 1) : (r > 0 ? r - 1 : 0);
  const int here = 3 * comp_sample(ws, d, comp, r, c) + comp_sample(ws, d, comp, rn, c);
  const int next = 3 * comp_sample(ws, d, comp, r, cn) + comp_sample(ws, d, comp, rn, cn);
  return (3 * here + next + ((x & 1) ? 7 : 8)) >> 4;
}

__host__ __device__ inline uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// crop pixel (y, x) -> 3 bytes: jdcolor.c ycc_rgb_convert (SCALEBITS 16), grey replicated
__host__ __device__ inline void crop_pixel(const int16_t* ws, const pf_jpeg_desc& d, int y, int x, uint8_t* out) {
  const int yy = d.crop_y + y, xx = d.crop_x + x;
  const int lum = comp_sample(ws, d, 0, yy, xx);
  if (d.ncomp == 1) {
    out[0] = out[1] = out[2] = (uint8_t)lum;
    return;
  }
  const int cb = chroma_at(ws, d, 1, yy, xx) - 128, cr = chroma_at(ws, d, 2, yy, xx) - 128;
  const int64_t ONE_HALF = (int64_t)1 << 15;
  const int cr_r = (int)((91881 * (int64_t)cr + ONE_HALF) >> 16);
  const int cb_b = (int)((116130 * (int64_t)cb + ONE_HALF) >> 16);
  const int g = (int)((-46802 * (int64_t)cr + (-22554 * (int64_t)cb + ONE_HALF)) >> 16);
  out[0] = clamp255(lum + cr_r);
  out[1] = clamp255(lum + g);
  out[2] = clamp255(lum + cb_b);
}

__host__ __device__ inline int64_t idct_window_blocks(const pf_jpeg_desc& d) {
  return (int64_t)(d.mcu_rows - d.mcu_row0) * (d.mcu_col1 - d.mcu_col0 + 1) * blocks_per_mcu(d);
}

#ifndef PF_JPEG_HOST_TEST
// one single-thread block per image: the Huffman stream is serial, and lone threads in their own blocks spread over
// every SM (up to 32 resident blocks each) instead of idling 31 lanes of a warp
__global__ void __launch_bounds__(1)
jpeg_entropy_kernel(const uint8_t* __restrict__ data, const pf_jpeg_desc* __restrict__ desc, int16_t* __restrict__ ws,
                    int32_t* __restrict__ status) {
  const int i = blockIdx.x;
  status[i] = jpeg_entropy_image(data, desc[i], ws);
}

__global__ void __launch_bounds__(128)
jpeg_idct_kernel(const pf_jpeg_desc* __restrict__ desc, int16_t* __restrict__ ws, const int32_t* __restrict__ status) {
  const int i = blockIdx.y;
  if (status[i] != JPEG_OK) return;
  const pf_jpeg_desc& d = desc[i];
  const int64_t nblk = idct_window_blocks(d);
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < nblk; j += (int64_t)gridDim.x * blockDim.x) {
    int64_t slot;
    int comp;
    if (idct_block_at(d, j, &slot, &comp)) idct_block(ws + slot, d.quant[comp]);
  }
}

__global__ void __launch_bounds__(256)
jpeg_color_kernel(const pf_jpeg_desc* __restrict__ desc, const int16_t* __restrict__ ws,
                  const int32_t* __restrict__ status, uint8_t* __restrict__ crops) {
  const int i = blockIdx.y;
  if (status[i] != JPEG_OK) return;
  const pf_jpeg_desc& d = desc[i];
  const int64_t npix = (int64_t)d.crop_h * d.crop_w;
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < npix; p += (int64_t)gridDim.x * blockDim.x) {
    uint8_t rgb[3];
    crop_pixel(ws, d, (int)(p / d.crop_w), (int)(p % d.crop_w), rgb);
    uint8_t* o = crops + d.crop_offset + p * 3;
    o[0] = rgb[0];
    o[1] = rgb[1];
    o[2] = rgb[2];
  }
}
#endif

}  // namespace

#ifndef PF_JPEG_HOST_TEST
extern "C" int pf_jpeg_decode(const uint8_t* data_dev, const pf_jpeg_desc* desc_dev, int n, int16_t* coef_ws_dev,
                              uint8_t* crops_dev, int32_t* status_dev, void* stream) {
  PF_REQUIRE(n >= 0 && n <= 65535, "pf_jpeg_decode: n=%d", n);
  if (n == 0) return PF_OK;
  PF_REQUIRE(data_dev && desc_dev && coef_ws_dev && crops_dev && status_dev, "pf_jpeg_decode: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  jpeg_entropy_kernel<<<n, 1, 0, st>>>(data_dev, desc_dev, coef_ws_dev, status_dev);
  PF_CHECK_LAUNCH("pf_jpeg_decode/entropy");
  jpeg_idct_kernel<<<dim3(16, n), 128, 0, st>>>(desc_dev, coef_ws_dev, status_dev);
  PF_CHECK_LAUNCH("pf_jpeg_decode/idct");
  jpeg_color_kernel<<<dim3(32, n), 256, 0, st>>>(desc_dev, coef_ws_dev, status_dev, crops_dev);
  PF_CHECK_LAUNCH("pf_jpeg_decode/color");
  return PF_OK;
}
#else
// test-only: the three kernels' bodies as plain loops on the host, same functions, same order
extern "C" void pf_test_jpeg_decode_host(const uint8_t* data, const pf_jpeg_desc* desc, int n, int16_t* ws,
                                         uint8_t* crops, int32_t* status) {
  for (int i = 0; i < n; ++i) status[i] = jpeg_entropy_image(data, desc[i], ws);
  for (int i = 0; i < n; ++i) {
    if (status[i] != JPEG_OK) continue;
    const int64_t nblk = idct_window_blocks(desc[i]);
    for (int64_t j = 0; j < nblk; ++j) {
      int64_t slot;
      int comp;
      if (idct_block_at(desc[i], j, &slot, &comp)) idct_block(ws + slot, desc[i].quant[comp]);
    }
  }
  for (int i = 0; i < n; ++i) {
    if (status[i] != JPEG_OK) continue;
    const pf_jpeg_desc& d = desc[i];
    for (int64_t p = 0; p < (int64_t)d.crop_h * d.crop_w; ++p)
      crop_pixel(ws, d, (int)(p / d.crop_w), (int)(p % d.crop_w), crops + d.crop_offset + p * 3);
  }
}

extern "C" int pf_test_jpeg_desc_size(void) { return (int)sizeof(pf_jpeg_desc); }
#endif
