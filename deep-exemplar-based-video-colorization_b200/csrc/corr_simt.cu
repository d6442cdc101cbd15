// K7 on CUDA cores (DVC_MATH_FP32): fused  f = theta_hat^T phi_hat  ->  row max (similarity)  ->
// softmax_j(f / T)  ->  y = P V,  never materialising the N x N matrix.
// Replaces NonlocalNet.py:477-498 (torch.matmul, torch.max, F.softmax, torch.matmul).
//
// One CTA owns 128 query rows: its theta tile [C x 128] stays resident in shared memory for the
// whole sweep over the reference positions; phi streams through a double-buffered [8 x 128] tile.
// Each thread keeps an 8 x 8 block of scores in registers and folds it straight into per-row
// running statistics:
//   ARGMAX mode (T <= 2e-10, test.py:94): running (max, argmax, number of bit-equal maxima, sum of their V rows);
//       distinct fp32 scores differ by > 104 T there, so the reference's fp32 softmax is one-hot -- or, for
//       bit-equal maxima (duplicated exemplar columns), the plain mean of their V rows, which is what is returned.
//   SOFTMAX mode: flash-style online softmax (running max, running sum, 3 weighted colour sums).
#include <math.h>

#include "corr_tc.cuh"
#include "dvc_internal.cuh"

namespace dvc {

namespace {

constexpr int BM = 128, BN = 128, BK = 8;

template <bool SOFTMAX>
__global__ void __launch_bounds__(256) corr_simt_kernel(const CorrParams p) {
  extern __shared__ __align__(16) float smem[];
  float* As = smem;                        // [C][BM]
  float* Bs = smem + (size_t)p.C * BM;     // [2][BK][BN]
  float4* Vs = reinterpret_cast<float4*>(Bs + 2 * BK * BN);  // [BN]

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.y;
  const int bphi = (p.Bphi == 1) ? 0 : b;
  const int m0 = blockIdx.x * BM;
  const float* __restrict__ th = p.theta + (size_t)p.qsrc.at(b) * p.NA * p.C;
  const float* __restrict__ ph = p.phi + (size_t)bphi * p.NB * p.C;
  const float4* __restrict__ Vg = reinterpret_cast<const float4*>(p.V) + (size_t)bphi * p.NB;

  const int l_row = tid >> 1, l_k4 = (tid & 1) * 4;

  // resident theta tile, transposed to [k][row]
  for (int k0 = 0; k0 < p.C; k0 += BK) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m0 + l_row < p.NA) v = __ldg(reinterpret_cast<const float4*>(th + (size_t)(m0 + l_row) * p.C + k0 + l_k4));
    As[(k0 + l_k4 + 0) * BM + l_row] = v.x;
    As[(k0 + l_k4 + 1) * BM + l_row] = v.y;
    As[(k0 + l_k4 + 2) * BM + l_row] = v.z;
    As[(k0 + l_k4 + 3) * BM + l_row] = v.w;
  }

  float run_m[8], run_s[8], run_a[8][3];  // ARGMAX mode: run_s = number of maxima, run_a = sum of their V rows
  int run_i[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    run_m[i] = -INFINITY, run_s[i] = 0.f, run_i[i] = 0;
    run_a[i][0] = run_a[i][1] = run_a[i][2] = 0.f;
  }
  const float sc = 1.4426950408889634f / p.temperature;  // log2(e) / T

  const int kcs = p.C / BK;
  const int ntiles = (p.NB + BN - 1) / BN;
  const int nsteps = ntiles * kcs;
  float4 rb;
  auto gload = [&](int step) {
    const int jt = step / kcs, k0 = (step - jt * kcs) * BK;
    const int r = jt * BN + l_row;
    rb = (r < p.NB) ? __ldg(reinterpret_cast<const float4*>(ph + (size_t)r * p.C + k0 + l_k4))
                    : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  auto sstore = [&](int buf) {
    float* d = Bs + buf * BK * BN;
    d[(l_k4 + 0) * BN + l_row] = rb.x;
    d[(l_k4 + 1) * BN + l_row] = rb.y;
    d[(l_k4 + 2) * BN + l_row] = rb.z;
    d[(l_k4 + 3) * BN + l_row] = rb.w;
  };

  float acc[8][8];
  gload(0);
  sstore(0);
  if (SOFTMAX && tid < BN) Vs[tid] = (tid < p.NB) ? __ldg(Vg + tid) : make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();

  for (int step = 0; step < nsteps; ++step) {
    const int cur = step & 1;
    const int jt = step / kcs, kc = step - jt * kcs;
    if (kc == 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    }
    if (step + 1 < nsteps) gload(step + 1);
    const float* Ab = As + (size_t)kc * BK * BM;
    const float* Bb = Bs + cur * BK * BN;
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(Ab + k * BM + ty * 4);
      const float4 a1 = *reinterpret_cast<const float4*>(Ab + k * BM + 64 + ty * 4);
      const float4 b0 = *reinterpret_cast<const float4*>(Bb + k * BN + tx * 4);
      const float4 b1 = *reinterpret_cast<const float4*>(Bb + k * BN + 64 + tx * 4);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    if (kc == kcs - 1) {
      // ---- fold this 128 x 128 score tile into the running row statistics ----
      const int cbase = jt * BN;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (!SOFTMAX) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = cbase + ((j < 4) ? tx * 4 + j : 64 + tx * 4 + (j - 4));
            if (col < p.NB && acc[i][j] >= run_m[i]) {  // rare once the running maximum has settled
              const float4 v = __ldg(Vg + col);
              if (acc[i][j] > run_m[i]) {
                run_m[i] = acc[i][j], run_i[i] = col, run_s[i] = 1.f;
                run_a[i][0] = v.x, run_a[i][1] = v.y, run_a[i][2] = v.z;
              } else {
                run_i[i] = min(run_i[i], col), run_s[i] += 1.f;
                run_a[i][0] += v.x, run_a[i][1] += v.y, run_a[i][2] += v.z;
              }
            }
          }
        } else {
          float tm = run_m[i];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = cbase + ((j < 4) ? tx * 4 + j : 64 + tx * 4 + (j - 4));
            if (col < p.NB) tm = fmaxf(tm, acc[i][j]);
          }
          if (tm > -INFINITY) {
            const float r = (run_m[i] == -INFINITY) ? 0.f : exp2f((run_m[i] - tm) * sc);
            run_s[i] *= r, run_a[i][0] *= r, run_a[i][1] *= r, run_a[i][2] *= r;
            run_m[i] = tm;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int cl = (j < 4) ? tx * 4 + j : 64 + tx * 4 + (j - 4);
              if (cbase + cl < p.NB) {
                const float e = exp2f((acc[i][j] - tm) * sc);
                const float4 v = Vs[cl];
                run_s[i] += e;
                run_a[i][0] = fmaf(e, v.x, run_a[i][0]);
                run_a[i][1] = fmaf(e, v.y, run_a[i][1]);
                run_a[i][2] = fmaf(e, v.z, run_a[i][2]);
              }
            }
          }
        }
      }
    }
    if (step + 1 < nsteps) sstore(cur ^ 1);
    __syncthreads();
    if (SOFTMAX && kc == kcs - 1 && jt + 1 < ntiles) {
      // colours of the next column tile (all threads passed the barrier above, so Vs is free)
      if (tid < BN) {
        const int r = (jt + 1) * BN + tid;
        Vs[tid] = (r < p.NB) ? __ldg(Vg + r) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      __syncthreads();
    }
  }

  // ---- merge the 16 column groups of every row (As is free now) ----
  float* red = smem;  // [128 rows][16 groups][6]
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rl = (i < 4) ? (ty * 4 + i) : (64 + ty * 4 + (i - 4));
    float* r = red + ((size_t)rl * 16 + tx) * 6;
    r[0] = run_m[i];
    r[1] = run_s[i], r[2] = run_a[i][0], r[3] = run_a[i][1], r[4] = run_a[i][2];
    if (!SOFTMAX) r[5] = __int_as_float(run_i[i]);
  }
  __syncthreads();
  if (tid < BM && m0 + tid < p.NA) {
    const float* r = red + (size_t)tid * 16 * 6;
    const size_t o = (size_t)b * p.NA + m0 + tid;
    if (!SOFTMAX) {
      float m = -INFINITY;
      for (int g = 0; g < 16; ++g) m = fmaxf(m, r[g * 6]);
      int idx = 0x7fffffff;
      float cnt = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f;
      for (int g = 0; g < 16; ++g)
        if (r[g * 6] == m && r[g * 6 + 1] > 0.f) {
          cnt += r[g * 6 + 1], a0 += r[g * 6 + 2], a1 += r[g * 6 + 3], a2 += r[g * 6 + 4];
          idx = min(idx, __float_as_int(r[g * 6 + 5]));
        }
      float4 v;
      if (cnt == 1.f) {
        v = __ldg(Vg + idx);
      } else {
        const float inv = 1.f / cnt;
        v = make_float4(a0 * inv, a1 * inv, a2 * inv, 0.f);
      }
      reinterpret_cast<float4*>(p.y)[o] = make_float4(v.x, v.y, v.z, 0.f);
      p.sim[o] = m;
      if (p.argmax) p.argmax[o] = idx;
    } else {
      float m = -INFINITY;
      for (int g = 0; g < 16; ++g) m = fmaxf(m, r[g * 6]);
      float s = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f;
      int idx = 0;
      float best = -INFINITY;
      for (int g = 0; g < 16; ++g) {
        const float mg = r[g * 6];
        if (mg == -INFINITY) continue;
        const float w = exp2f((mg - m) * sc);
        s += w * r[g * 6 + 1], a0 += w * r[g * 6 + 2], a1 += w * r[g * 6 + 3], a2 += w * r[g * 6 + 4];
        if (mg > best) best = mg, idx = g;
      }
      (void)idx;
      reinterpret_cast<float4*>(p.y)[o] = make_float4(a0 / s, a1 / s, a2 / s, 0.f);
      p.sim[o] = m;
      if (p.argmax) p.argmax[o] = -1;  // not defined for a true softmax
    }
  }
}

}  // namespace

void launch_corr_simt(const CorrParams& p, cudaStream_t s) {
  const size_t smem = ((size_t)p.C * BM + 2 * BK * BN) * sizeof(float) + BN * sizeof(float4);
  dim3 grid((p.NA + BM - 1) / BM, p.B);
  static unsigned long long attr_mask = 0;  // the attribute is per device
  if (first_use_on_device(&attr_mask)) {
    cudaFuncSetAttribute(corr_simt_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(corr_simt_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  }
  if (p.temperature <= 2e-10f)
    corr_simt_kernel<false><<<grid, 256, smem, s>>>(p);
  else
    corr_simt_kernel<true><<<grid, 256, smem, s>>>(p);
  launch_counter_add(1);
}

}  // namespace dvc
