// Baseline JPEG encoder (include/dvc.h: dvc_encode_jpeg, dvc_colorize_videos_jpeg).  It writes the bytes of Pillow's
// Image.fromarray(x).save(f, "JPEG", quality=q) for uint8 RGB [H][W][3]: 4:2:0 YCbCr, JDCT_ISLOW, standard Huffman tables,
// no restart markers -- libjpeg-turbo's integer arithmetic restated (tests/jpeg_oracle.py restates it in numpy, stage by
// stage, and is checked against Pillow):
//   jccolor.c    rgb_ycc_convert: 16-bit fixed point, ONE_HALF and CBCR_OFFSET
//   jcprepct.c / jcsample.c   edge replication (expand_right_edge, expand_bottom_edge) and h2v2_downsample (bias 1, 2, ...)
//   jfdctint.c   jpeg_fdct_islow (CONST_BITS 13, PASS1_BITS 2)
//   jcdctmgr.c   quantize with compute_reciprocal's (reciprocal, correction, shift) of divisor q << 3
//   jccoefct.c   dummy blocks padding the last MCU column / row: zero AC, the DC of the preceding block of the MCU
//   jchuff.c     DC prediction per component in MCU order, ZRL, EOB, 0xFF 0x00 stuffing, 1-bits padding, then EOI
//
// The entropy-coded segment has no restart markers, so its blocks are coded in parallel: one thread per 8x8 block
// transforms, quantizes and counts its AC bits; one CTA per image adds the DC bits and scans the bit lengths; one thread per
// block writes its bits at its offset; the 0xFF bytes are counted per tile and scanned; the stuffed file (header, data,
// EOI) is assembled in device memory and copied to its destination with consecutive threads on consecutive bytes, so that a
// page-locked host destination receives full PCIe writes of the finished file only.  Seven launches per batch of images.
#include <stdint.h>

#include "dvc_internal.cuh"

namespace dvc {

namespace {

constexpr int kThreads = 128;
constexpr int kScanThreads = 1024;
constexpr int kTile = 32;  // bytes of entropy-coded data per thread of the 0xFF count and the stuffing copy

// ---- standard Huffman tables (JPEG Annex K.3; libjpeg jstdhuff.c), codes built at compile time -------------------------
struct HuffTable {
  uint16_t code[256];
  uint8_t len[256];
};

constexpr uint8_t kDcLumaBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
constexpr uint8_t kDcChromaBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
constexpr uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
constexpr uint8_t kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
constexpr uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
    0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
    0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
constexpr uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
constexpr uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
    0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
    0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
    0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
    0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
    0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

// canonical codes of a (bits, vals) table: jchuff.c jpeg_make_c_derived_tbl
constexpr HuffTable make_huff(const uint8_t (&bits)[16], const uint8_t* vals) {
  HuffTable t{};
  int code = 0, k = 0;
  for (int n = 1; n <= 16; ++n) {
    for (int i = 0; i < bits[n - 1]; ++i, ++k, ++code) t.code[vals[k]] = (uint16_t)code, t.len[vals[k]] = (uint8_t)n;
    code <<= 1;
  }
  return t;
}

// [0] DC luma, [1] DC chroma, [2] AC luma, [3] AC chroma
__constant__ HuffTable c_huff[4] = {make_huff(kDcLumaBits, kDcVals), make_huff(kDcChromaBits, kDcVals),
                                    make_huff(kAcLumaBits, kAcLumaVals), make_huff(kAcChromaBits, kAcChromaVals)};

// zigzag position of natural (row-major) index i
__host__ __device__ constexpr int zigzag_pos(int i) {
  const int t[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42, 3,  8,  12, 17, 25, 30,
                     41, 43, 9,  11, 18, 24, 31, 40, 44, 53, 10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38,
                     46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};
  return t[i];
}

constexpr int fix16(double x) { return (int)(x * 65536.0 + 0.5); }  // jccolor.c FIX(x), SCALEBITS 16
constexpr int kYR = fix16(0.29900), kYG = fix16(0.58700), kYB = fix16(0.11400), kCbR = fix16(0.16874), kCbG = fix16(0.33126),
              kHalf = fix16(0.5), kCrG = fix16(0.41869), kCrB = fix16(0.08131);

__device__ __forceinline__ int nbits_of(int a) { return a ? 32 - __clz(a) : 0; }  // a >= 0

// ---- stage 1: colour conversion, down-sampling, DCT, quantization, AC bit count ---------------------------------------
__device__ __forceinline__ int rgb_y(const unsigned char* p) { return (kYR * p[0] + kYG * p[1] + kYB * p[2] + (1 << 15)) >> 16; }
__device__ __forceinline__ int rgb_c(const unsigned char* p, int cr) {  // Cb (cr = 0) or Cr (cr = 1): CBCR_OFFSET + ONE_HALF - 1
  const int off = (128 << 16) + (1 << 15) - 1;
  return cr ? (kHalf * p[0] - kCrG * p[1] - kCrB * p[2] + off) >> 16 : (-kCbR * p[0] - kCbG * p[1] + kHalf * p[2] + off) >> 16;
}

// one 1-D pass of jpeg_fdct_islow over v[0], v[s], ..., v[7 s]; first = the row pass (PASS1_BITS scaling up)
template <int s, bool first>
__device__ __forceinline__ void fdct_1d(int* v) {
  constexpr int C0_298 = 2446, C0_390 = 3196, C0_541 = 4433, C0_765 = 6270, C0_899 = 7373, C1_175 = 9633, C1_501 = 12299,
                C1_847 = 15137, C1_961 = 16069, C2_053 = 16819, C2_562 = 20995, C3_072 = 25172;
  constexpr int sh = first ? 13 - 2 : 13 + 2;
  auto descale = [](int x, int n) { return (x + (1 << (n - 1))) >> n; };
  const int tmp0 = v[0] + v[7 * s], tmp7 = v[0] - v[7 * s];
  const int tmp1 = v[s] + v[6 * s], tmp6 = v[s] - v[6 * s];
  const int tmp2 = v[2 * s] + v[5 * s], tmp5 = v[2 * s] - v[5 * s];
  const int tmp3 = v[3 * s] + v[4 * s], tmp4 = v[3 * s] - v[4 * s];
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  if (first) {
    v[0] = (tmp10 + tmp11) * 4;
    v[4 * s] = (tmp10 - tmp11) * 4;
  } else {
    v[0] = descale(tmp10 + tmp11, 2);
    v[4 * s] = descale(tmp10 - tmp11, 2);
  }
  int z1 = (tmp12 + tmp13) * C0_541;
  v[2 * s] = descale(z1 + tmp13 * C0_765, sh);
  v[6 * s] = descale(z1 - tmp12 * C1_847, sh);
  z1 = tmp4 + tmp7;
  int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
  const int z5 = (z3 + z4) * C1_175;
  const int t4 = tmp4 * C0_298, t5 = tmp5 * C2_053, t6 = tmp6 * C3_072, t7 = tmp7 * C1_501;
  z1 *= -C0_899, z2 *= -C2_562;
  z3 = z3 * -C1_961 + z5, z4 = z4 * -C0_390 + z5;
  v[7 * s] = descale(t4 + z1 + z3, sh);
  v[5 * s] = descale(t5 + z2 + z4, sh);
  v[3 * s] = descale(t6 + z2 + z3, sh);
  v[s] = descale(t7 + z1 + z4, sh);
}

// Thread n of image blockIdx.y: block n in MCU order (per 16x16 MCU: Y00, Y01, Y10, Y11, Cb, Cr).  Writes the quantized
// block in zigzag order (int16 [64]) and the bits of its AC coefficients, ZRL and EOB included.
__global__ void __launch_bounds__(kThreads) jpeg_blocks_kernel(const unsigned char* __restrict__ rgb, int H, int W, JpegQuant qt,
                                                                int16_t* __restrict__ coef, int* __restrict__ acbits) {
  __shared__ uint8_t s_aclen[2][256];
  for (int i = threadIdx.x; i < 512; i += kThreads) s_aclen[i >> 8][i & 255] = c_huff[2 + (i >> 8)].len[i & 255];
  __syncthreads();
  const int mx = (W + 15) >> 4, my = (H + 15) >> 4, nblk = 6 * mx * my;
  const int n = blockIdx.x * kThreads + threadIdx.x;
  if (n >= nblk) return;
  const int b = blockIdx.y, mcu = n / 6, j = n - 6 * mcu, mcu_y = mcu / mx, mcu_x = mcu - mcu_y * mx;
  const unsigned char* img = rgb + (size_t)b * H * W * 3;
  const int t = j < 4 ? 0 : 1;
  int d[64];
  bool dummy = false;
  if (j < 4) {
    // jccoefct.c: a block past the image's block grid (nby, nbx) is a dummy with the DC of the preceding block of its MCU --
    // the block on its left, or for the bottom row of the last MCU row the MCU's block (0, 1), itself maybe a right dummy
    const int nby = (H + 7) >> 3, nbx = (W + 7) >> 3;
    const int by = 2 * mcu_y + (j >> 1), bx = 2 * mcu_x + (j & 1);
    const bool bottom = by >= nby;
    dummy = bottom || bx >= nbx;
    const int sy = min(by, nby - 1), sx = bottom ? min(2 * mcu_x + 1, nbx - 1) : min(bx, nbx - 1);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const unsigned char* row = img + (size_t)min(8 * sy + r, H - 1) * W * 3;
#pragma unroll
      for (int c = 0; c < 8; ++c) d[8 * r + c] = rgb_y(row + 3 * min(8 * sx + c, W - 1)) - 128;
    }
  } else {
    // h2v2_downsample of the edge-replicated full-resolution plane; chroma rows past ceil(H/2) repeat the last one
    const int cr = j - 4, last_cy = ((H + 1) >> 1) - 1;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int cy = min(8 * mcu_y + r, last_cy);
      const unsigned char* r0 = img + (size_t)(2 * cy) * W * 3;
      const unsigned char* r1 = img + (size_t)min(2 * cy + 1, H - 1) * W * 3;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int x0 = 3 * min(16 * mcu_x + 2 * c, W - 1), x1 = 3 * min(16 * mcu_x + 2 * c + 1, W - 1);
        const int sum = rgb_c(r0 + x0, cr) + rgb_c(r0 + x1, cr) + rgb_c(r1 + x0, cr) + rgb_c(r1 + x1, cr);
        d[8 * r + c] = ((sum + 1 + (c & 1)) >> 2) - 128;
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) fdct_1d<1, true>(d + 8 * r);
#pragma unroll
  for (int c = 0; c < 8; ++c) fdct_1d<8, false>(d + c);
  int zz[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int v = d[i], a = abs(v);
    const int q = (int)(((uint32_t)(a + qt.corr[t][i]) * qt.recip[t][i]) >> qt.shift[t][i]);
    zz[zigzag_pos(i)] = (dummy && i) ? 0 : (v < 0 ? -q : q);
  }
  int bits = 0, run = 0;
#pragma unroll
  for (int k = 1; k < 64; ++k) {
    if (zz[k] == 0) {
      ++run;
    } else {
      const int nb = nbits_of(abs(zz[k]));
      bits += (run >> 4) * s_aclen[t][0xF0] + s_aclen[t][((run & 15) << 4) + nb] + nb;
      run = 0;
    }
  }
  if (run) bits += s_aclen[t][0];
  acbits[(size_t)b * nblk + n] = bits;
  int4* dst = reinterpret_cast<int4*>(coef + ((size_t)b * nblk + n) * 64);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int4 w;
    w.x = (zz[8 * k + 0] & 0xffff) | (zz[8 * k + 1] << 16);
    w.y = (zz[8 * k + 2] & 0xffff) | (zz[8 * k + 3] << 16);
    w.z = (zz[8 * k + 4] & 0xffff) | (zz[8 * k + 5] << 16);
    w.w = (zz[8 * k + 6] & 0xffff) | (zz[8 * k + 7] << 16);
    dst[k] = w;
  }
}

// the block whose DC predicts block n's (per component in MCU order), or -1 for the first block of a component
__device__ __forceinline__ int dc_pred_block(int n) {
  const int j = n % 6;
  if (j == 1 || j == 2 || j == 3) return n - 1;
  if (n < 6) return -1;
  return j == 0 ? n - 3 : n - 6;  // Y00 follows the previous MCU's Y11; Cb / Cr the previous MCU's
}

__device__ __forceinline__ int dc_diff(const int16_t* coef, int n) {
  const int p = dc_pred_block(n);
  return coef[(size_t)n * 64] - (p >= 0 ? coef[(size_t)p * 64] : 0);
}

// ---- stages 2 and 5: per-image exclusive scan (one CTA of kScanThreads per image) -------------------------------------
// kind 0: the bit length of every block (its AC bits + its DC code and value bits) -> bit offsets, totals[0] = data bits;
//         then zeroes the data words that stage 3 ORs its bits into.
// kind 1: the 0xFF count of every tile -> offsets, totals[1] = 0xFF count.
template <int kind>
__global__ void __launch_bounds__(kScanThreads) jpeg_scan_kernel(int n, const int16_t* __restrict__ coef, const int* __restrict__ val,
                                                                  uint32_t* __restrict__ off, int64_t* __restrict__ totals,
                                                                  uint32_t* __restrict__ words, size_t words_per_image) {
  __shared__ int s_dclen[2][12];
  __shared__ uint32_t s_warp[kScanThreads / 32];
  if (kind == 0 && threadIdx.x < 24) s_dclen[threadIdx.x / 12][threadIdx.x % 12] = c_huff[threadIdx.x / 12].len[threadIdx.x % 12];
  __syncthreads();
  const int b = blockIdx.x;
  const int16_t* cf = coef + (size_t)b * n * 64;
  const int* v = val + (size_t)b * n;
  uint32_t* o = off + (size_t)b * n;
  if (kind == 1) n = min(n, (int)(((totals[(size_t)b * 4] + 7) / 8 + kTile - 1) / kTile));  // the tiles holding data
  auto item = [&](int i) -> uint32_t {
    if (kind == 1) return (uint32_t)v[i];
    const int nb = nbits_of(abs(dc_diff(cf, i)));
    return (uint32_t)(v[i] + s_dclen[i % 6 < 4 ? 0 : 1][nb] + nb);
  };
  const int per = (n + kScanThreads - 1) / kScanThreads, i0 = threadIdx.x * per, i1 = min(n, i0 + per);
  uint32_t sum = 0;
  for (int i = i0; i < i1; ++i) sum += item(i);
  // block-wide exclusive scan of the per-thread sums
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t incl = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += y;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = s_warp[lane], wi = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, wi, d);
      if (lane >= d) wi += y;
    }
    s_warp[lane] = wi - w;
  }
  __syncthreads();
  uint32_t run = s_warp[warp] + incl - sum;
  for (int i = i0; i < i1; ++i) {
    o[i] = run;
    run += item(i);
  }
  if (threadIdx.x == kScanThreads - 1) totals[(size_t)b * 4 + kind] = run;
  if (kind == 0) {
    __shared__ uint32_t s_total;
    if (threadIdx.x == kScanThreads - 1) s_total = run;
    __syncthreads();
    const size_t nw = ((size_t)s_total + 31) / 32;
    uint32_t* w = words + (size_t)b * words_per_image;
    for (size_t i = threadIdx.x; i < nw; i += kScanThreads) w[i] = 0;
  }
}

// ---- stage 3: Huffman coding of every block at its bit offset ----------------------------------------------------------
struct BitWriter {
  uint32_t* words;
  size_t w;      // word receiving the bits above the `fill` pending ones
  uint64_t acc;  // pending bits, the last `fill` of them valid
  int fill;
  __device__ __forceinline__ void put(uint32_t bits, int len) {  // len <= 16
    acc = (acc << len) | (bits & ((1u << len) - 1));
    fill += len;
    if (fill >= 32) {
      fill -= 32;
      atomicOr(words + w++, (uint32_t)(acc >> fill));
    }
  }
  __device__ __forceinline__ void flush() {
    if (fill) atomicOr(words + w, (uint32_t)(acc << (32 - fill)));
  }
};

__global__ void __launch_bounds__(kThreads) jpeg_encode_kernel(int nblk, const int16_t* __restrict__ coef, const uint32_t* __restrict__ off,
                                                                const int64_t* __restrict__ totals, uint32_t* __restrict__ words,
                                                                size_t words_per_image) {
  __shared__ uint16_t s_code[4][256];
  __shared__ uint8_t s_len[4][256];
  for (int i = threadIdx.x; i < 1024; i += kThreads) s_code[i >> 8][i & 255] = c_huff[i >> 8].code[i & 255], s_len[i >> 8][i & 255] = c_huff[i >> 8].len[i & 255];
  __syncthreads();
  const int n = blockIdx.x * kThreads + threadIdx.x;
  if (n >= nblk) return;
  const int b = blockIdx.y, t = n % 6 < 4 ? 0 : 1;
  const int16_t* cf = coef + (size_t)b * nblk * 64;
  const uint32_t p0 = off[(size_t)b * nblk + n];
  // start with the (p0 % 32) bits of the word that precede this block, as zeros
  BitWriter bw{words + (size_t)b * words_per_image, p0 >> 5, 0, (int)(p0 & 31)};
  const int diff = dc_diff(cf, n), dnb = nbits_of(abs(diff));
  bw.put(s_code[t][dnb], s_len[t][dnb]);
  if (dnb) bw.put((uint32_t)(diff < 0 ? diff - 1 : diff), dnb);
  const int4* src = reinterpret_cast<const int4*>(cf + (size_t)n * 64);
  int run = 0;
#pragma unroll
  for (int k8 = 0; k8 < 8; ++k8) {
    const int4 w4 = src[k8];
    const int pair[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
    for (int h = 0; h < 8; ++h) {
      const int k = 8 * k8 + h;
      if (k == 0) continue;
      const int v = (int16_t)(pair[h >> 1] >> (16 * (h & 1)));
      if (v == 0) {
        ++run;
        continue;
      }
      for (; run >= 16; run -= 16) bw.put(s_code[2 + t][0xF0], s_len[2 + t][0xF0]);
      const int nb = nbits_of(abs(v)), sym = (run << 4) + nb;
      bw.put(s_code[2 + t][sym], s_len[2 + t][sym]);
      bw.put((uint32_t)(v < 0 ? v - 1 : v), nb);
      run = 0;
    }
  }
  if (run) bw.put(s_code[2 + t][0], s_len[2 + t][0]);
  if (n == nblk - 1) {  // the last block pads the final byte with 1-bits
    const int pad = (int)((8 - (totals[(size_t)b * 4] & 7)) & 7);
    if (pad) bw.put((1u << pad) - 1, pad);
  }
  bw.flush();
}

__device__ __forceinline__ uint32_t data_byte(const uint32_t* w, size_t i) { return (w[i >> 2] >> (24 - 8 * (i & 3))) & 0xff; }

// ---- stage 4: 0xFF bytes per tile of the entropy-coded data -----------------------------------------------------------
__global__ void __launch_bounds__(256) jpeg_ff_count_kernel(int ntile, const int64_t* __restrict__ totals, const uint32_t* __restrict__ words,
                                                            size_t words_per_image, int* __restrict__ cnt) {
  const int i = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
  const size_t nbytes = ((size_t)totals[(size_t)b * 4] + 7) / 8;
  if ((size_t)i * kTile >= nbytes) return;
  const uint32_t* w = words + (size_t)b * words_per_image;
  int c = 0;
  for (size_t k = (size_t)i * kTile; k < min(nbytes, (size_t)(i + 1) * kTile); ++k) c += data_byte(w, k) == 0xff;
  cnt[(size_t)b * ntile + i] = c;
}

// ---- stage 6: the file in device memory: header, stuffed data, EOI; totals[2] = file size ------------------------------
__global__ void __launch_bounds__(256) jpeg_stuff_kernel(int ntile, const unsigned char* __restrict__ header, int hdr_len,
                                                         int64_t* __restrict__ totals, const uint32_t* __restrict__ words,
                                                         size_t words_per_image, const uint32_t* __restrict__ ffoff,
                                                         unsigned char* __restrict__ file, size_t file_stride) {
  const int i = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
  unsigned char* f = file + (size_t)b * file_stride;
  if (i < hdr_len) f[i] = header[i];
  const size_t nbytes = ((size_t)totals[(size_t)b * 4] + 7) / 8;
  const int used = (int)((nbytes + kTile - 1) / kTile);  // tiles holding data; ntile is the worst case
  if (i >= used) return;
  const uint32_t* w = words + (size_t)b * words_per_image;
  unsigned char* o = f + hdr_len + (size_t)i * kTile + ffoff[(size_t)b * ntile + i];
  for (size_t k = (size_t)i * kTile; k < min(nbytes, (size_t)(i + 1) * kTile); ++k) {
    const uint32_t v = data_byte(w, k);
    *o++ = (unsigned char)v;
    if (v == 0xff) *o++ = 0;
  }
  if (i == used - 1) {
    o[0] = 0xff, o[1] = 0xd9;
    totals[(size_t)b * 4 + 2] = (int64_t)(o + 2 - f);
  }
}

// ---- stage 7: the file to its destination (device or page-locked host memory), consecutive threads on consecutive bytes --
__global__ void __launch_bounds__(256) jpeg_copy_out_kernel(const unsigned char* __restrict__ file, size_t file_stride,
                                                            const int64_t* __restrict__ totals, JpegDst dst) {
  const int b = blockIdx.y;
  const size_t size = (size_t)totals[(size_t)b * 4 + 2];
  const unsigned char* f = file + (size_t)b * file_stride;
  unsigned char* o = dst.dst[b] + dst.dst_off;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < size; i += (size_t)gridDim.x * 256) o[i] = f[i];
  if (blockIdx.x == 0 && threadIdx.x == 0) dst.size[b][dst.size_off] = (int64_t)size;
}

}  // namespace

// ---- host side ---------------------------------------------------------------------------------------------------------
int64_t jpeg_blocks(int H, int W) { return 6LL * ((H + 15) / 16) * ((W + 15) / 16); }

int64_t jpeg_max_bytes(int H, int W) {
  if (H < 1 || W < 1 || H > 65535 || W > 65535 || jpeg_blocks(H, W) * kJpegMaxBlockBits >= (1LL << 31)) return -1;
  return kJpegHeaderBytes + 2 + 2 * ((jpeg_blocks(H, W) * kJpegMaxBlockBits + 7) / 8);
}

// quality scaling of jpeg_set_quality(q, force_baseline = TRUE) and the (reciprocal, correction, shift) of jcdctmgr.c
// compute_reciprocal for divisor q << 3 with 16-bit DCTELEMs; tables[2][64] receives the scaled tables (natural order)
static const int kStdQuant[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
     18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};

JpegQuant jpeg_quant(int quality, int tables[2][64]) {
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  JpegQuant q{};
  for (int t = 0; t < 2; ++t)
    for (int i = 0; i < 64; ++i) {
      const int v = std::min(255, std::max(1, (int)(((long)kStdQuant[t][i] * scale + 50) / 100)));
      tables[t][i] = v;
      const uint32_t d = (uint32_t)v << 3;
      int r = 16 + (31 - __builtin_clz(d));
      uint32_t fq = (1u << r) / d, c = d / 2;
      const uint32_t fr = (1u << r) % d;
      if (fr == 0) fq >>= 1, --r;
      else if (fr <= d / 2) ++c;
      else ++fq;
      q.recip[t][i] = (uint16_t)fq, q.corr[t][i] = (uint16_t)c, q.shift[t][i] = (uint8_t)r;
    }
  return q;
}

// SOI, APP0 JFIF 1.01 (no density unit, 1:1), DQT luma, DQT chroma (zigzag order), SOF0, DHT DC/AC luma, DC/AC chroma, SOS
void jpeg_header(int H, int W, const int tables[2][64], unsigned char out[kJpegHeaderBytes]) {
  unsigned char* p = out;
  auto seg = [&](int marker, int len) { *p++ = 0xff, *p++ = (unsigned char)marker, *p++ = (unsigned char)(len >> 8), *p++ = (unsigned char)len; };
  *p++ = 0xff, *p++ = 0xd8;
  seg(0xe0, 16);
  const unsigned char jfif[14] = {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  for (unsigned char v : jfif) *p++ = v;
  for (int t = 0; t < 2; ++t) {
    seg(0xdb, 67);
    *p++ = (unsigned char)t;
    int zz[64];
    for (int i = 0; i < 64; ++i) zz[zigzag_pos(i)] = tables[t][i];
    for (int v : zz) *p++ = (unsigned char)v;
  }
  seg(0xc0, 17);
  const unsigned char sof[15] = {8, (unsigned char)(H >> 8), (unsigned char)H, (unsigned char)(W >> 8), (unsigned char)W, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1};
  for (unsigned char v : sof) *p++ = v;
  auto dht = [&](int cls_id, const uint8_t (&bits)[16], const uint8_t* vals, int nvals) {
    seg(0xc4, 2 + 1 + 16 + nvals);
    *p++ = (unsigned char)cls_id;
    for (uint8_t v : bits) *p++ = v;
    for (int i = 0; i < nvals; ++i) *p++ = vals[i];
  };
  dht(0x00, kDcLumaBits, kDcVals, 12);
  dht(0x10, kAcLumaBits, kAcLumaVals, 162);
  dht(0x01, kDcChromaBits, kDcVals, 12);
  dht(0x11, kAcChromaBits, kAcChromaVals, 162);
  seg(0xda, 12);
  const unsigned char sos[10] = {3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0};
  for (unsigned char v : sos) *p++ = v;
}

JpegLayout jpeg_layout(int B, int H, int W) {
  JpegLayout L;
  L.nblk = jpeg_blocks(H, W);
  const size_t data_bytes = (size_t)(L.nblk * kJpegMaxBlockBits + 7) / 8;
  L.words_per_image = (data_bytes + 3) / 4 + 1;
  L.ntile = (int)((data_bytes + kTile - 1) / kTile);
  L.file_stride = ((size_t)jpeg_max_bytes(H, W) + 255) & ~(size_t)255;
  size_t o = 0;
  auto carve = [&](size_t bytes) { const size_t at = o; o += (bytes + 255) & ~(size_t)255; return at; };
  L.coef = carve((size_t)B * L.nblk * 64 * 2);
  L.acbits = carve((size_t)B * L.nblk * 4);
  L.off = carve((size_t)B * L.nblk * 4);
  L.words = carve((size_t)B * L.words_per_image * 4);
  L.cnt = carve((size_t)B * L.ntile * 4);
  L.ffoff = carve((size_t)B * L.ntile * 4);
  L.totals = carve((size_t)B * 4 * 8);
  L.header = carve(kJpegHeaderBytes);
  L.file = carve((size_t)B * L.file_stride);
  L.bytes = o;
  return L;
}

void launch_jpeg_encode(const unsigned char* rgb, int B, int H, int W, const JpegQuant& qt, unsigned char* ws, const JpegLayout& L,
                        const JpegDst& dst, cudaStream_t s) {
  int16_t* coef = (int16_t*)(ws + L.coef);
  int* acbits = (int*)(ws + L.acbits);
  uint32_t* off = (uint32_t*)(ws + L.off);
  uint32_t* words = (uint32_t*)(ws + L.words);
  int* cnt = (int*)(ws + L.cnt);
  uint32_t* ffoff = (uint32_t*)(ws + L.ffoff);
  int64_t* totals = (int64_t*)(ws + L.totals);
  unsigned char* file = ws + L.file;
  const int nblk = (int)L.nblk;
  const dim3 gblk((nblk + kThreads - 1) / kThreads, B);
  jpeg_blocks_kernel<<<gblk, kThreads, 0, s>>>(rgb, H, W, qt, coef, acbits);
  jpeg_scan_kernel<0><<<B, kScanThreads, 0, s>>>(nblk, coef, acbits, off, totals, words, L.words_per_image);
  jpeg_encode_kernel<<<gblk, kThreads, 0, s>>>(nblk, coef, off, totals, words, L.words_per_image);
  const dim3 gtile((L.ntile + 255) / 256, B);
  jpeg_ff_count_kernel<<<gtile, 256, 0, s>>>(L.ntile, totals, words, L.words_per_image, cnt);
  jpeg_scan_kernel<1><<<B, kScanThreads, 0, s>>>(L.ntile, coef, cnt, ffoff, totals, words, L.words_per_image);
  const dim3 gstuff((std::max(L.ntile, kJpegHeaderBytes) + 255) / 256, B);
  jpeg_stuff_kernel<<<gstuff, 256, 0, s>>>(L.ntile, ws + L.header, kJpegHeaderBytes, totals, words, L.words_per_image, ffoff, file,
                                           L.file_stride);
  const dim3 gcopy((unsigned)std::min<size_t>(256, (L.file_stride + 4095) / 4096), B);
  jpeg_copy_out_kernel<<<gcopy, 256, 0, s>>>(file, L.file_stride, totals, dst);
  launch_counter_add(7);
}

}  // namespace dvc
