// Exact-fp32 convolution as a flat shifted GEMM on CUDA cores (DVC_MATH_FP32).
//
// This is the first correct CUDA path and stays as the on-GPU fp32 reference that the wgmma
// (3xTF32) engine is validated against.  Replaces nn.Conv2d + bias + ReLU/LeakyReLU (+ skip add,
// + InstanceNorm statistics) at NonlocalNet.py:235-255,364-423 and ColorVidNet.py:96-143.
//
// Tile: 128 padded pixels x BN output channels x 8 input channels per step, 256 threads, 8 x (BN/16)
// accumulators per thread, register-prefetch double buffering (one __syncthreads per k-step).
#include <cuda_fp16.h>

#include "dvc_internal.cuh"

namespace dvc {

namespace {

constexpr int BM = 128;
constexpr int BK = 8;

// TWO_LEVEL: the products of every FOLD_STEPS k-steps (32 input channels of one tap, the k-block of the tensor-core
// engine) are summed in a fresh accumulator that is then folded into the running total, so the rounding-error chain
// is ~sqrt(32) + sqrt(9*Cin/32) long instead of sqrt(9*Cin) (the CPU reference's vectorised/blocked summation has a
// similarly short chain).  Folding only once per tap left chains of up to 512 products, and the T = 0.01 softmax of
// the correlation amplified the resulting feature error in the colour output beyond the reference's own fp32 noise.
constexpr int FOLD_STEPS = 32 / BK;
template <int BN, bool TWO_LEVEL>
__global__ void __launch_bounds__(256) conv_gemm_simt_kernel(const ConvParams p) {
  constexpr int TN = BN / 16;
  constexpr int BV = BN / 4;  // float4 per weight k-row
  __shared__ __align__(16) float smem[2 * BK * BM + 2 * BK * BN];
  float(*As)[BK][BM] = reinterpret_cast<float(*)[BK][BM]>(smem);
  float(*Bs)[BK][BN] = reinterpret_cast<float(*)[BK][BN]>(smem + 2 * BK * BM);

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.z;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int npix = p.Hp * p.Wp;
  const float* __restrict__ xb = p.x + (size_t)b * npix * p.Cin;

  const int a_row = tid >> 1, a_k4 = (tid & 1) * 4;
  const int b_k = tid / BV, b_n4 = (tid % BV) * 4;
  const bool b_active = tid < BK * BV;

  float acc[8][TN];
  float tot[TWO_LEVEL ? 8 : 1][TWO_LEVEL ? TN : 1];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      acc[i][j] = 0.f;
      if constexpr (TWO_LEVEL) tot[i][j] = 0.f;
    }

  const int kcs = p.Cin / BK;
  const int nk = p.taps * kcs;
  float4 ra = make_float4(0.f, 0.f, 0.f, 0.f), rb = make_float4(0.f, 0.f, 0.f, 0.f);

  auto gload = [&](int it) {
    const int tap = it / kcs;
    const int k0 = (it - tap * kcs) * BK;
    int off = 0;
    if (p.taps == 9) off = ((tap / 3 - 1) * p.Wp + (tap % 3 - 1)) * p.dil;
    const int r = m0 + a_row + off;
    if (r >= 0 && r < npix)
      ra = __ldg(reinterpret_cast<const float4*>(xb + (size_t)r * p.Cin + k0 + a_k4));
    else
      ra = make_float4(0.f, 0.f, 0.f, 0.f);
    if (b_active)
      rb = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)(tap * p.Cin + k0 + b_k) * p.CoutPad + n0 + b_n4));
  };
  auto sstore = [&](int buf) {
    As[buf][a_k4 + 0][a_row] = ra.x;
    As[buf][a_k4 + 1][a_row] = ra.y;
    As[buf][a_k4 + 2][a_row] = ra.z;
    As[buf][a_k4 + 3][a_row] = ra.w;
    if (b_active) *reinterpret_cast<float4*>(&Bs[buf][b_k][b_n4]) = rb;
  };

  gload(0);
  sstore(0);
  __syncthreads();
  for (int it = 0; it < nk; ++it) {
    const int cur = it & 1;
    if (it + 1 < nk) gload(it + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[cur][k][64 + ty * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float bb[TN];
      {
        const float4 b0 = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 4]);
        bb[0] = b0.x, bb[1] = b0.y, bb[2] = b0.z, bb[3] = b0.w;
        if constexpr (TN == 8) {
          const float4 b1 = *reinterpret_cast<const float4*>(&Bs[cur][k][64 + tx * 4]);
          bb[4] = b1.x, bb[5] = b1.y, bb[6] = b1.z, bb[7] = b1.w;
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    if constexpr (TWO_LEVEL) {
      const int kstep = (it + 1) % kcs;  // k-steps of the current tap done (0: the tap is complete)
      if (kstep % FOLD_STEPS == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) tot[i][j] += acc[i][j], acc[i][j] = 0.f;
      }
    }
    if (it + 1 < nk) sstore(cur ^ 1);
    __syncthreads();
  }
  if constexpr (TWO_LEVEL) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = tot[i][j];
  }

  // ---- epilogue: bias, skip add, activation, masked store, InstanceNorm statistics ----
  float ssum[TN], ssq[TN];
#pragma unroll
  for (int j = 0; j < TN; ++j) ssum[j] = 0.f, ssq[j] = 0.f;

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rl = (i < 4) ? (ty * 4 + i) : (64 + ty * 4 + (i - 4));
    const int pp = m0 + rl;
    if (pp >= npix) continue;
    const int yp = pp / p.Wp, xp = pp - yp * p.Wp;
    const int y = yp - p.P, x = xp - p.P;
    if (y < 0 || y >= p.H || x < 0 || x >= p.W) continue;
    if (p.stride == 2 && ((y | x) & 1)) continue;
    const int yo = y / p.stride, xo = x / p.stride;
#pragma unroll
    for (int g = 0; g < TN / 4; ++g) {
      const int c = n0 + (g == 0 ? tx * 4 : 64 + tx * 4);
      if (c >= p.Cout) continue;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = acc[i][g * 4 + j];
      if (p.bias) {
        const float4 bv = __ldg(reinterpret_cast<const float4*>(p.bias + c));
        v[0] += bv.x, v[1] += bv.y, v[2] += bv.z, v[3] += bv.w;
      }
      if (p.add) {
        const float4 av = __ldg(reinterpret_cast<const float4*>(
            p.add + (((size_t)b * p.aHp + yo + p.aP) * p.aWp + xo + p.aP) * p.aC + c));
        v[0] += av.x, v[1] += av.y, v[2] += av.z, v[3] += av.w;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (p.act == ACT_RELU) v[j] = fmaxf(v[j], 0.f);
        if (p.act == ACT_LRELU) v[j] = v[j] > 0.f ? v[j] : v[j] * p.slope;
        ssum[g * 4 + j] += v[j];
        ssq[g * 4 + j] += v[j] * v[j];
      }
      if (p.y) {
        const size_t o = (((size_t)b * p.yHp + yo + p.yP) * p.yWp + xo + p.yP) * p.yC + p.yCoff + c;
        if (p.y_lo) {  // feed a tensor-core layer: tf32 hi/lo planes
          float h[4], l[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            uint32_t u;
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v[j]));
            h[j] = __uint_as_float(u);
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v[j] - h[j]));
            l[j] = __uint_as_float(u);
          }
          *reinterpret_cast<float4*>(p.y + o) = make_float4(h[0], h[1], h[2], h[3]);
          *reinterpret_cast<float4*>(p.y_lo + o) = make_float4(l[0], l[1], l[2], l[3]);
        } else {
          *reinterpret_cast<float4*>(p.y + o) = make_float4(v[0], v[1], v[2], v[3]);
        }
      }
      if (p.nchw) {
#pragma unroll
        for (int j = 0; j < 4; ++j) p.nchw[(((size_t)b * p.Cout + c + j) * p.Ho + yo) * p.Wo + xo] = v[j];
      }
    }
  }

  if (p.stats) {  // block-level reduction over the 16 row groups, then one double atomic per column
    float* red = smem;  // [2][16][BN]
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int cl = (j < 4) ? (tx * 4 + j) : (64 + tx * 4 + (j - 4));
      red[ty * BN + cl] = ssum[j];
      red[16 * BN + ty * BN + cl] = ssq[j];
    }
    __syncthreads();
    if (tid < BN) {
      const int c = n0 + tid;
      if (c < p.Cout) {
        float s = 0.f, q = 0.f;
#pragma unroll
        for (int t = 0; t < 16; ++t) s += red[t * BN + tid], q += red[16 * BN + t * BN + tid];
        atomicAdd(&p.stats[((size_t)b * p.Cout + c) * 2 + 0], (double)s);
        atomicAdd(&p.stats[((size_t)b * p.Cout + c) * 2 + 1], (double)q);
      }
    }
  }
}

}  // namespace

void launch_conv_simt(const ConvParams& p, int B, bool two_level, cudaStream_t s) {
  const int npix = p.Hp * p.Wp;
  if (two_level) {
    dim3 grid((npix + BM - 1) / BM, p.CoutPad / 64, B);
    conv_gemm_simt_kernel<64, true><<<grid, 256, 0, s>>>(p);
  } else if (p.CoutPad % 128 == 0) {
    dim3 grid((npix + BM - 1) / BM, p.CoutPad / 128, B);
    conv_gemm_simt_kernel<128, false><<<grid, 256, 0, s>>>(p);
  } else {
    dim3 grid((npix + BM - 1) / BM, p.CoutPad / 64, B);
    conv_gemm_simt_kernel<64, false><<<grid, 256, 0, s>>>(p);
  }
  launch_counter_add(1);
}

}  // namespace dvc

// ---------------------------------------------------------------------------------------------------
// First-layer convolution (3 or 7 real input channels padded to 8; VGG conv1_1, ColorVidNet conv1_1.0):
// K = 27 / 63 is far too short for the GEMM tiling above, so one thread computes one output pixel for all output
// channels with the weights staged in shared memory (broadcast reads).  FFMA-bound: ~50 us at 480x864.
// ---------------------------------------------------------------------------------------------------
namespace dvc {
namespace {

// First layers (Cin <= 8 real channels, 3x3): one thread = 8 adjacent pixels of a row x COUT/8 channels; the eight
// lanes of an octet cover one pixel's COUT channels, so every store request writes whole 32-byte sectors, and every
// weight vector read from shared memory feeds 8 pixels (32 FMA per LDS.128).  CIN = real input channels (compile time;
// 0 = run-time `cin_real`, all 8 fetched); the row loop stays rolled so that the body fits the instruction cache (the
// fully unrolled 27 x 8-channel body was ~240 KB of SASS and stalled on instruction fetch).
// Accumulation order per output: taps outer, input channels inner, one fma chain -- identical to a scalar loop.
template <int COUT, int CIN>
__global__ void __launch_bounds__(128) conv_first_kernel(const ConvParams p, int cin_real) {
  constexpr int CG = COUT / 8;
  constexpr int NCI = (CIN > 0 && CIN <= 4) ? 4 : 8;  // input channels fetched per pixel
  constexpr int NCL = CIN > 0 ? CIN : 8;              // input channels in the unrolled body
  __shared__ __align__(16) float ws[9 * 8 * COUT];
  __shared__ float bs[COUT];
  __shared__ float s_amax[4];
  for (int i = threadIdx.x; i < 9 * 8 * COUT; i += 128) {
    const int co = i % COUT, k = i / COUT;  // k = tap * 8 + ci
    ws[i] = __ldg(p.w + (size_t)k * p.CoutPad + co);
  }
  for (int i = threadIdx.x; i < COUT; i += 128) bs[i] = p.bias ? __ldg(p.bias + i) : 0.f;
  __syncthreads();
  const int b = blockIdx.y;
  // fp16 output planes with a device-derived scale (tensor-core mode: the next layer is a 3xFP16 convolution)
  float yscale = 1.f, amax = 0.f;
  if (p.dyn.h16) {
    const int e_out = dyn_out_exponent(p.dyn);
    yscale = exp2_int(e_out);
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) p.dyn.cell_out->e = e_out;
  }
  const int g = threadIdx.x & 7;
  const int oct = (blockIdx.x * 128 + threadIdx.x) >> 3;
  const int opr = (p.W + 7) >> 3;
  const bool live = oct < p.H * opr;  // dead lanes recompute octet 0 and store nothing (the block stays converged)
  const int oc = live ? oct : 0;
  const int y = oc / opr, x0 = (oc - y * opr) * 8;
  float acc[8][CG];
#pragma unroll
  for (int px = 0; px < 8; ++px)
#pragma unroll
    for (int j = 0; j < CG; ++j) acc[px][j] = 0.f;
  const float* xb = p.x + (size_t)b * p.Hp * p.Wp * 8;
#pragma unroll 1
  for (int r = 0; r < 3; ++r) {
    float in[10][NCI];
#pragma unroll
    for (int col = 0; col < 10; ++col) {
      const int xx = x0 + p.P - 1 + col;
      float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
      if (xx < p.Wp) {
        const float* px = xb + ((size_t)(y + p.P + r - 1) * p.Wp + xx) * 8;
        v0 = __ldg(reinterpret_cast<const float4*>(px));
        if (NCI == 8) v1 = __ldg(reinterpret_cast<const float4*>(px + 4));
      }
      in[col][0] = v0.x, in[col][1] = v0.y, in[col][2] = v0.z, in[col][3] = v0.w;
      if (NCI == 8) in[col][4] = v1.x, in[col][5] = v1.y, in[col][6] = v1.z, in[col][7] = v1.w;
    }
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
#pragma unroll
      for (int ci = 0; ci < NCL; ++ci) {
        if (CIN > 0 || ci < cin_real) {
          const float4* wr = reinterpret_cast<const float4*>(ws + ((r * 3 + kx) * 8 + ci) * COUT + g * CG);
#pragma unroll
          for (int c4 = 0; c4 < CG / 4; ++c4) {
            const float4 w4 = wr[c4];
#pragma unroll
            for (int px = 0; px < 8; ++px) {
              const float a = in[px + kx][ci];
              acc[px][c4 * 4 + 0] = fmaf(a, w4.x, acc[px][c4 * 4 + 0]);
              acc[px][c4 * 4 + 1] = fmaf(a, w4.y, acc[px][c4 * 4 + 1]);
              acc[px][c4 * 4 + 2] = fmaf(a, w4.z, acc[px][c4 * 4 + 2]);
              acc[px][c4 * 4 + 3] = fmaf(a, w4.w, acc[px][c4 * 4 + 3]);
            }
          }
        }
      }
    }
  }
  float bias[CG];
#pragma unroll
  for (int j = 0; j < CG; ++j) bias[j] = bs[g * CG + j];
#pragma unroll
  for (int px = 0; px < 8; ++px) {
    if (!live || x0 + px >= p.W) continue;
    const size_t o = (((size_t)b * p.yHp + y + p.yP) * p.yWp + x0 + px + p.yP) * p.yC + p.yCoff + g * CG;
    float v[CG];
#pragma unroll
    for (int j = 0; j < CG; ++j) {
      v[j] = acc[px][j] + bias[j];
      if (p.act == ACT_RELU) v[j] = fmaxf(v[j], 0.f);
      if (p.act == ACT_LRELU) v[j] = v[j] > 0.f ? v[j] : v[j] * p.slope;
      amax = fmaxf(amax, fabsf(v[j]));
    }
    if (p.dyn.h16) {
      // |v * yscale| <= 2^15 by construction of the exponent (dvc_internal.cuh: dyn_out_exponent): no clamp needed
      uint32_t hw[CG / 2], lw[CG / 2];
#pragma unroll
      for (int j = 0; j < CG; j += 2) {
        const float a0 = v[j] * yscale, a1 = v[j + 1] * yscale;
        const __half2 h2 = __floats2half2_rn(a0, a1);
        const float2 hf = __half22float2(h2);
        const __half2 l2 = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
        hw[j / 2] = *reinterpret_cast<const uint32_t*>(&h2), lw[j / 2] = *reinterpret_cast<const uint32_t*>(&l2);
      }
      __half* hp = reinterpret_cast<__half*>(p.dyn.h16) + o;
      __half* lp = reinterpret_cast<__half*>(p.dyn.l16) + o;
      if constexpr (CG == 8) {
        *reinterpret_cast<uint4*>(hp) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        *reinterpret_cast<uint4*>(lp) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
      } else {
        *reinterpret_cast<uint2*>(hp) = make_uint2(hw[0], hw[1]);
        *reinterpret_cast<uint2*>(lp) = make_uint2(lw[0], lw[1]);
      }
    } else if (p.y_lo) {
#pragma unroll
      for (int c4 = 0; c4 < CG / 4; ++c4) {
        float h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          uint32_t u;
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v[c4 * 4 + j]));
          h[j] = __uint_as_float(u);
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v[c4 * 4 + j] - h[j]));
          l[j] = __uint_as_float(u);
        }
        *reinterpret_cast<float4*>(p.y + o + c4 * 4) = make_float4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<float4*>(p.y_lo + o + c4 * 4) = make_float4(l[0], l[1], l[2], l[3]);
      }
    } else {
#pragma unroll
      for (int c4 = 0; c4 < CG / 4; ++c4)
        *reinterpret_cast<float4*>(p.y + o + c4 * 4) = make_float4(v[c4 * 4], v[c4 * 4 + 1], v[c4 * 4 + 2], v[c4 * 4 + 3]);
    }
  }
  if (p.dyn.cell_out) block_amax_commit(amax, p.dyn.cell_out, s_amax);
}

}  // namespace

bool launch_conv_first(const ConvParams& p, int B, int cin_real, cudaStream_t s) {
  if (p.Cin != 8 || p.taps != 9 || p.dil != 1 || p.stride != 1 || p.add || p.stats || p.P < 1) return false;
  dim3 grid((p.H * ((p.W + 7) / 8) * 8 + 127) / 128, B);
  if (p.Cout == 64 && cin_real == 3)  // VGG19 conv1_1
    conv_first_kernel<64, 3><<<grid, 128, 0, s>>>(p, cin_real);
  else if (p.Cout == 64)
    conv_first_kernel<64, 0><<<grid, 128, 0, s>>>(p, cin_real);
  else if (p.Cout == 32 && cin_real == 7)  // ColorVidNet conv1_1.0
    conv_first_kernel<32, 7><<<grid, 128, 0, s>>>(p, cin_real);
  else if (p.Cout == 32)
    conv_first_kernel<32, 0><<<grid, 128, 0, s>>>(p, cin_real);
  else
    return false;
  launch_counter_add(1);
  return true;
}

}  // namespace dvc
