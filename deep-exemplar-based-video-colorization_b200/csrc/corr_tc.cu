// K7 on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
//   f = theta_hat^T phi_hat  ->  sim = rowmax f  ->  P = softmax_j(f / T)  ->  y = P V      (NonlocalNet.py:477-498)
//
// fp32-class accuracy from low-precision MMAs by operand splitting: x = hi + lo with hi, lo exactly
// representable in the MMA input type (tf32: 2 x 11 significant bits; bf16: 2 x 8), and
//   f ~= hi_a.hi_b + hi_a.lo_b + lo_a.hi_b           (lo.lo dropped: 2^-22 resp. 2^-16 relative)
// all three accumulated into the same fp32 register tile.  A third format, FP16X3, splits x * 2^14 into two fp16 planes
// (theta_hat / phi_hat are unit vectors, so the fixed power-of-two scale is exact and cannot overflow): the same
// 2 x 11 significant bits as tf32 at twice the MMA rate and half the operand bytes; scores come out times 2^28.
// FP16X3 is the default; DVC_MATH_TF32X3 and DVC_MATH_BF16X3 are selectable.  By default two CTAs on adjacent query
// tiles run as a 2-CTA cluster that shares the reference tile: each CTA loads half of it and multicasts it to both.
//
// Kernel structure (one CTA = 128 query rows x a range of 256-column tiles of reference positions), 384 threads:
//   warp 0        TMA producer: per k-block (128 bytes of K) loads A_hi, A_lo [128 x 128B] and B_hi, B_lo [256 x 128B]
//                 with SWIZZLE_128B into a 2-stage shared-memory ring (96 KB per stage), mbarrier expect_tx.
//   warps 4..11   two consumer warpgroups, one per 64 query rows: 4 k-steps x 3 wgmma (M64 x N256) per stage into
//                 128 fp32 registers per thread, then the epilogue on those registers: every thread owns two query
//                 rows and 64 of the tile's columns and keeps running (max, argmax) or online-softmax (max, sum, 3
//                 colour sums) statistics per row; the four threads that share a row write four partial results.
// The N x N score matrix never leaves the SM.  Column-range splits (grid.z) balance the SMs; a small merge kernel
// combines the per-split, per-thread row statistics.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cudaTypedefs.h>
#include <math.h>

#include <mutex>

#include "corr_tc.cuh"
#include "tc_common.cuh"

namespace dvc {

// ------------------------------------------------------------------------------------------------
// tensor-map encoding through the driver entry point (no link-time libcuda dependency)
// ------------------------------------------------------------------------------------------------
int encode_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols,
                   int elem_bytes, int swizzle_bytes) {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  });
  if (!fn) return -1;
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstride[1] = {cols * (uint64_t)elem_bytes};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = fn(out, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

namespace {

constexpr int BM = 128;        // query rows per CTA (two consumer warpgroups of 64)
constexpr int BN = 256;        // reference positions per score tile (= wgmma N)
constexpr int NTHREADS = 384;  // warpgroup 0: TMA producer (warp 0); warpgroups 1, 2: MMA + epilogue
constexpr int CONSUMER_WARPS = 8;
constexpr int QUADS = 4;       // threads sharing a query row (wgmma accumulator layout): partial results per row and split
// Each CTA holds the whole reference tile of a stage (in a 2-CTA cluster half of it arrives by the peer's multicast).
struct Cfg {
  static constexpr int STAGES = 2;
  static constexpr int A_BYTES = BM * 128, B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;  // 98304
  static constexpr int V_RING_BYTES = 2 * BN * 16;  // softmax epilogue: the V rows of the tile in flight, two slots
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*alignment slack*/ + 256 /*barriers*/ + V_RING_BYTES;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 1-D bulk copy global -> this CTA's shared memory, completing on a local mbarrier
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(tc::smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(tc::smem_u32(bar))
               : "memory");
}
// per (split part, row) partial statistics.  Softmax: running max m, sum s of exp weights, weighted colour sums a*.
// Argmax: max m, lowest column idx attaining it, s = NUMBER of columns whose score equals m bit for bit and a* = the sum
// of their V rows -- the reference's fp32 softmax(f / 1e-10) averages the V rows of bit-equal maxima (duplicated
// exemplar columns: letterbox bars, flat regions), NonlocalNet.py:486-497.
struct SplitOut {
  float m, s, a0, a1, a2;
  int idx;
  float pad0, pad1;
};

struct TcParams {
  int NA, NB, B, Bphi, C;
  PlaneSrc qsrc;  // batch b reads query set qsrc.at(b): rows qsrc.at(b) * NA .. + NA of the A planes
  int tiles_per_split;
  float sc;  // log2(e) / T
  const float* row_sc;  // optional per-query-row log2(e) / T_i (overrides sc): the contextual loss normalises every row by its own minimum distance
  float out_scale;  // scores in the accumulators are true scores / out_scale (2^-28 for pre-scaled fp16 operands, else 1)
  const float4* V;
  SplitOut* part;  // [nsplit * QUADS][B*NA]
};

// ---- operand split: rows [R][C] fp32 -> hi / lo planes -----------------------------------------------
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

template <int FMT>
__global__ void __launch_bounds__(256) split_planes_kernel(const float* __restrict__ src, void* __restrict__ hi,
                                                           void* __restrict__ lo, size_t n4) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(src) + i);
    const float x[4] = {v.x, v.y, v.z, v.w};
    if constexpr (FMT == 2) {
      __half h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xs = x[j] * 16384.0f;
        h[j] = __float2half_rn(xs);
        l[j] = __float2half_rn(xs - __half2float(h[j]));
      }
      reinterpret_cast<uint2*>(hi)[i] = make_uint2(
          (uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16),
          (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16));
      reinterpret_cast<uint2*>(lo)[i] = make_uint2(
          (uint32_t)__half_as_ushort(l[0]) | ((uint32_t)__half_as_ushort(l[1]) << 16),
          (uint32_t)__half_as_ushort(l[2]) | ((uint32_t)__half_as_ushort(l[3]) << 16));
    } else if constexpr (FMT == 0) {
      float h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) h[j] = tf32_rna(x[j]), l[j] = tf32_rna(x[j] - h[j]);
      reinterpret_cast<float4*>(hi)[i] = make_float4(h[0], h[1], h[2], h[3]);
      reinterpret_cast<float4*>(lo)[i] = make_float4(l[0], l[1], l[2], l[3]);
    } else {
      __nv_bfloat16 h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        h[j] = __float2bfloat16_rn(x[j]);
        l[j] = __float2bfloat16_rn(x[j] - __bfloat162float(h[j]));
      }
      reinterpret_cast<uint2*>(hi)[i] = make_uint2(
          (uint32_t)__bfloat16_as_ushort(h[0]) | ((uint32_t)__bfloat16_as_ushort(h[1]) << 16),
          (uint32_t)__bfloat16_as_ushort(h[2]) | ((uint32_t)__bfloat16_as_ushort(h[3]) << 16));
      reinterpret_cast<uint2*>(lo)[i] = make_uint2(
          (uint32_t)__bfloat16_as_ushort(l[0]) | ((uint32_t)__bfloat16_as_ushort(l[1]) << 16),
          (uint32_t)__bfloat16_as_ushort(l[2]) | ((uint32_t)__bfloat16_as_ushort(l[3]) << 16));
    }
  }
}

// ---- screened T -> 0 path: operand preparation ---------------------------------------------------------
// One warp per row of [R][256]: the fp16 hi plane of x * 2^14 (the only operand of the screening pass) and the exact
// Euclidean norm of what the plane drops, d = x - hi * 2^-14, which bounds the screening error of every score of that
// row: |f - f_screen| <= |d_a . b| + |a_hi . d_b| <= ||d_a|| ||b|| + ||a_hi|| ||d_b||  (Cauchy-Schwarz).
// nd[row] = ||d_row|| (rounded up), nh[row] = ||hi_row * 2^-14|| (rounded up); *nd_max = max over rows (float bits).
__global__ void __launch_bounds__(256) screen_planes_kernel(const float* __restrict__ src, __half* __restrict__ hi, float* __restrict__ nd,
                                                            float* __restrict__ nh, unsigned int* __restrict__ nd_max,
                                                            unsigned int* __restrict__ nh_max, int R) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= R) return;
  const float4* sp = reinterpret_cast<const float4*>(src + (size_t)warp * 256);
  float sd = 0.f, sh = 0.f;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const float4 v = __ldg(sp + k * 32 + lane);
    const float x[4] = {v.x, v.y, v.z, v.w};
    unsigned short hb[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half h = __float2half_rn(x[j] * 16384.0f);
      hb[j] = __half_as_ushort(h);
      const float hf = __half2float(h) * 6.103515625e-05f;  // exact: a power-of-two scale
      const float d = x[j] - hf;                            // exact (Sterbenz / few significant bits)
      sd = fmaf(d, d, sd), sh = fmaf(hf, hf, sh);
    }
    reinterpret_cast<uint2*>(hi + (size_t)warp * 256)[k * 32 + lane] =
        make_uint2((uint32_t)hb[0] | ((uint32_t)hb[1] << 16), (uint32_t)hb[2] | ((uint32_t)hb[3] << 16));
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) sd += __shfl_xor_sync(0xffffffffu, sd, off), sh += __shfl_xor_sync(0xffffffffu, sh, off);
  if (lane == 0) {
    // round the norms up generously (fp32 summation error of 256 non-negative terms is < 2^-15 relative)
    const float a = sqrtf(sd) * 1.0001f + 1e-12f, b = sqrtf(sh) * 1.0001f;
    nd[warp] = a, nh[warp] = b;
    atomicMax(nd_max, __float_as_uint(a));
    atomicMax(nh_max, __float_as_uint(b));
  }
}

// ---- main kernel ---------------------------------------------------------------------------------------
template <int FMT, bool SOFTMAX, int CL>
__global__ void __launch_bounds__(NTHREADS, 1)
    corr_tc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                   const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl, const TcParams p) {
  constexpr int KB = FMT == 0 ? 32 : 64;   // K elements per 128-byte k-block
  constexpr int STAGES = Cfg::STAGES, A_BYTES = Cfg::A_BYTES, B_BYTES = Cfg::B_BYTES, STAGE_BYTES = Cfg::STAGE_BYTES;
  const int crank = (CL == 2) ? (int)tc::cluster_ctarank() : 0;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full = bars;                     // [STAGES]   TMA -> MMA
  uint64_t* empty = bars + STAGES;           // [STAGES]   MMA (both CTAs of a cluster) -> TMA
  uint64_t* vfull = bars + 2 * STAGES;       // [2]        bulk copy of the tile's V rows -> epilogue (softmax)
  uint64_t* vempty = bars + 2 * STAGES + 2;  // [2]        this CTA's epilogue -> its producer (softmax)
  float4* v_ring = reinterpret_cast<float4*>(smem + STAGES * STAGE_BYTES + 256);  // [2][BN]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  const int bphi = (p.Bphi == 1) ? 0 : b;
  const int m0 = blockIdx.x * BM;
  const int ntiles_all = (p.NB + BN - 1) / BN;
  const int t0 = blockIdx.z * p.tiles_per_split;
  const int t1 = min(t0 + p.tiles_per_split, ntiles_all);
  const int ntiles = max(t1 - t0, 0);
  const int nkb = p.C / KB;

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmAh);
    tc::tma_prefetch_desc(&tmAl);
    tc::tma_prefetch_desc(&tmBh);
    tc::tma_prefetch_desc(&tmBl);
    for (int i = 0; i < STAGES; ++i) tc::mbar_init(&full[i], 1), tc::mbar_init(&empty[i], CONSUMER_WARPS * CL);
    for (int i = 0; i < 2; ++i) tc::mbar_init(&vfull[i], 1), tc::mbar_init(&vempty[i], CONSUMER_WARPS);
    tc::fence_barrier_init();
  }
  __syncthreads();
  if (CL == 2) tc::cluster_sync_all();  // the peer's barriers are initialised before any multicast or remote arrive reaches them

  if (warp < 4) {
    tc::setmaxnreg_dec<40>();
    if (warp == 0) {
      // ================= TMA producer (warp-convergent loop, one elected lane issues) =================
      int stage = 0;
      uint32_t phase = 0;
      const int arow0 = p.qsrc.at(b) * p.NA;
      for (int t = 0; t < ntiles; ++t) {
        const int col0 = bphi * p.NB + (t0 + t) * BN;
        for (int kb = 0; kb < nkb; ++kb) {
          tc::mbar_wait(&empty[stage], phase ^ 1);
          if (tc::elect_one()) {
            uint8_t* st = smem + stage * STAGE_BYTES;
            tc::mbar_arrive_expect_tx(&full[stage], STAGE_BYTES);
            tc::tma_load_2d(st, &tmAh, &full[stage], kb * KB, arow0 + m0);
            tc::tma_load_2d(st + A_BYTES, &tmAl, &full[stage], kb * KB, arow0 + m0);
            if (CL == 1) {
              tc::tma_load_2d(st + 2 * A_BYTES, &tmBh, &full[stage], kb * KB, col0);
              tc::tma_load_2d(st + 2 * A_BYTES + B_BYTES, &tmBl, &full[stage], kb * KB, col0);
            } else {  // my half of the reference positions, multicast into both CTAs of the cluster
              const int h = crank * (BN / 2);
              tc::tma_load_2d_mc(st + 2 * A_BYTES + h * 128, &tmBh, &full[stage], kb * KB, col0 + h, 3);
              tc::tma_load_2d_mc(st + 2 * A_BYTES + B_BYTES + h * 128, &tmBl, &full[stage], kb * KB, col0 + h, 3);
            }
          }
          __syncwarp();
          if (++stage == STAGES) stage = 0, phase ^= 1;
        }
        if (SOFTMAX) {
          // the V rows of this tile's columns for this CTA's epilogue; the slot was freed by the epilogue of tile t-2
          const int buf = t & 1;
          tc::mbar_wait(&vempty[buf], ((t >> 1) & 1) ^ 1);
          if (tc::elect_one()) {
            const int c0 = (t0 + t) * BN;
            const uint32_t bytes = (uint32_t)min(BN, p.NB - c0) * 16u;
            tc::mbar_arrive_expect_tx(&vfull[buf], bytes);
            bulk_load_1d(v_ring + buf * BN, p.V + (size_t)bphi * p.NB + c0, bytes, &vfull[buf]);
          }
          __syncwarp();
        }
      }
    }
  } else {
    // ================= consumers: wgmma into registers, then the epilogue on them =================
    tc::setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1, qd = lane & 3;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // local query row of slot 0 (slot 1: rl + 8)
    const uint32_t a_off = (uint32_t)(wg * 64 * 128);
    float sck[2], run_m[2] = {-INFINITY, -INFINITY};
    // argmax: number of bit-equal maxima and the sum of their V rows; softmax: weighted colour sums and the sum of weights
    float cnt[2] = {0.f, 0.f}, s0[2] = {0.f, 0.f}, s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
    int run_i[2] = {0, 0};
#pragma unroll
    for (int h = 0; h < 2; ++h)  // exponent scale in units of the (possibly pre-scaled) accumulator scores
      sck[h] = (p.row_sc ? __ldg(p.row_sc + (size_t)b * p.NA + min(m0 + rl + 8 * h, p.NA - 1)) : p.sc) * p.out_scale;
    const float4* __restrict__ Vg = p.V + (size_t)bphi * p.NB;
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int t = 0; t < ntiles; ++t) {
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        tc::mbar_wait(&full[stage], phase);
        const uint32_t sa = tc::smem_u32(smem + stage * STAGE_BYTES);
        const uint64_t dAh = tc::wg_desc_k128(sa + a_off), dAl = tc::wg_desc_k128(sa + A_BYTES + a_off);
        const uint64_t dBh = tc::wg_desc_k128(sa + 2 * A_BYTES), dBl = tc::wg_desc_k128(sa + 2 * A_BYTES + B_BYTES);
        tc::wg_fence_regs(acc);
        tc::wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint64_t adv = (uint64_t)(kk * 2);  // 32 bytes of K, in 16-byte units of the start-address field
          // small cross terms first, the dominant hi.hi term last
          tc::wgmma_fmt<FMT>(acc, dAl + adv, dBh + adv, (kb | kk) ? 1u : 0u);
          tc::wgmma_fmt<FMT>(acc, dAh + adv, dBl + adv, 1u);
          tc::wgmma_fmt<FMT>(acc, dAh + adv, dBh + adv, 1u);
        }
        tc::wg_commit();
        if (prev >= 0) {  // the previous k-block's MMAs have read their stage: hand it back
          tc::wg_wait<1>();
          tc::release_stage<CL>(&empty[prev], lane);
        }
        prev = stage;
        if (++stage == STAGES) stage = 0, phase ^= 1;
      }
      tc::wg_wait<0>();
      tc::wg_fence_regs(acc);
      tc::release_stage<CL>(&empty[prev], lane);

      const int buf = t & 1;
      if (SOFTMAX) tc::mbar_wait(&vfull[buf], (t >> 1) & 1);
      const int colbase = (t0 + t) * BN;
      const bool full_tile = colbase + BN <= p.NB;
      const float4* Vs = v_ring + buf * BN;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        // this thread's columns of the tile: 8 j + 2 qd + e, j = 0..31, e = 0, 1 (ascending)
        float cm = -INFINITY;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (full_tile || colbase + 8 * j + 2 * qd + e < p.NB) cm = fmaxf(cm, acc[4 * j + 2 * h + e]);
        if (!SOFTMAX) {
          if (cm >= run_m[h]) {  // rare once the running maximum has settled
            if (cm > run_m[h]) run_m[h] = cm, cnt[h] = 0.f, s0[h] = s1[h] = s2[h] = 0.f;
            uint64_t hit = 0;  // bit 2 j + e: column 8 j + 2 qd + e attains the maximum
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                hit |= (uint64_t)(acc[4 * j + 2 * h + e] == cm && (full_tile || colbase + 8 * j + 2 * qd + e < p.NB)) << (2 * j + e);
            while (hit) {  // ascending columns
              const int i = __ffsll((long long)hit) - 1;
              hit &= hit - 1;
              const int col = colbase + 8 * (i >> 1) + 2 * qd + (i & 1);
              if (cnt[h] == 0.f) run_i[h] = col;  // lowest index of this thread's columns attaining the maximum
              const float4 v = __ldg(Vg + col);
              cnt[h] += 1.f, s0[h] += v.x, s1[h] += v.y, s2[h] += v.z;
            }
          }
        } else {
          if (cm > run_m[h]) {
            const float sc_old = (run_m[h] == -INFINITY) ? 0.f : ex2_approx((run_m[h] - cm) * sck[h]);
            s0[h] *= sc_old, s1[h] *= sc_old, s2[h] *= sc_old, cnt[h] *= sc_old;
            run_m[h] = cm;
          }
          // weights e = 2^((f - m) * log2(e) / T); V rows come from shared memory as (a0, a1, a2, 1)
#pragma unroll
          for (int j = 0; j < BN / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int cl = 8 * j + 2 * qd + e;
              if (full_tile || colbase + cl < p.NB) {
                const float w = ex2_approx((acc[4 * j + 2 * h + e] - run_m[h]) * sck[h]);
                const float4 v = Vs[cl];
                s0[h] = fmaf(w, v.x, s0[h]), s1[h] = fmaf(w, v.y, s1[h]), s2[h] = fmaf(w, v.z, s2[h]), cnt[h] = fmaf(w, v.w, cnt[h]);
              }
            }
        }
      }
      if (SOFTMAX) {
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&vempty[buf]);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m0 + rl + 8 * h;
      if (row < p.NA) {
        SplitOut o;
        o.m = run_m[h] * p.out_scale, o.idx = run_i[h], o.pad0 = o.pad1 = 0.f;
        o.s = cnt[h], o.a0 = s0[h], o.a1 = s1[h], o.a2 = s2[h];
        p.part[((size_t)(blockIdx.z * QUADS + qd) * p.B + b) * p.NA + row] = o;
      }
    }
  }

  __syncthreads();
  if (CL == 2) tc::cluster_sync_all();  // no CTA may exit while its peer can still multicast into it or arrive on its barriers
}


// ---- screened T -> 0 path: one fp16 pass + exact re-scoring of the candidates ----------------------------------------
// At T <= 2e-10 only the row maximum matters (one-hot softmax), and a single hi.hi pass locates it up to the
// rigorous error eps_i of row i (screen_planes_kernel): every column j with f_screen(i, j) >= max_j f_screen - 2 eps_i is a
// CANDIDATE, all others are provably not the maximum.  The screening kernel keeps up to SCREEN_K candidates per (row,
// column-range split, thread of the row's quad) while it streams the tiles -- one third of the MMA work and half of the
// operand bytes of the 3-pass kernel; corr_rescore_kernel then evaluates the candidates exactly in fp32 on the CUDA cores
// (a few per row) and produces (sim, argmax, mean V of bit-equal maxima).  A list that overflows marks its part for brute force.
constexpr int SCREEN_K = 16;  // candidates kept per (row, column-range split, quad thread)

// The query tile (128 rows x 256 channels of fp16 = 64 KB) stays RESIDENT in shared memory for the CTA's whole sweep over
// the reference positions; only the reference tiles stream through the ring: half of the bytes per tile.
struct ScreenCfg {
  static constexpr int STAGES = 3;
  static constexpr int A_BYTES = BM * 128, B_BYTES = BN * 128;
  static constexpr int A_RES_BYTES = 4 * A_BYTES;        // all four k-blocks of the query tile (C = 256)
  static constexpr int STAGE_BYTES = B_BYTES;            // 32768
  // candidate lists of the consumer threads: [SCREEN_K][consumer threads][2 rows] column indices -- slot k of (thread, row)
  // lives at [k][thread][row], so dynamic slot indices never conflict on a bank and never touch local memory
  static constexpr int LT = CONSUMER_WARPS * 32 * 2;
  static constexpr int LIST_BYTES = SCREEN_K * LT * 4;
  static constexpr int SMEM_BYTES = A_RES_BYTES + STAGES * STAGE_BYTES + 1024 + 256 + LIST_BYTES;
};

struct ScreenParams {
  int NA, NB, B, Bphi, C;
  PlaneSrc qsrc;  // batch b reads query set qsrc.at(b) of the A plane and the query norms
  int tiles_per_split;
  const float* nd_a;   // [query sets * NA]   ||dropped part|| of every query row
  const float* nh_a;   //                                       ||hi part||
  const unsigned int* nd_b_max;  // float bits: max over reference rows of ||dropped part||
  const unsigned int* nh_b_max;  //             max over reference rows of ||hi part||
  float* pm;     // [parts][B*NA]            screening maximum of the part (true-score units)
  int* pcnt;     // [parts][B*NA]            number of candidates, or -1: overflow (brute-force the part's columns)
  int* pidx;     // [parts][B*NA][SCREEN_K]  candidate columns
};

// 2 * eps_i in true-score units (see screen_planes_kernel); 64 * 2^-24 covers the truncating fp32 accumulation
__device__ __forceinline__ float screen_threshold(float nd_a, float nh_a, float nd_b, float nh_b) {
  return 2.f * (nd_a * (nh_b + nd_b) + nh_a * nd_b + 4e-6f) * 1.001f;
}

template <int CL>
__global__ void __launch_bounds__(NTHREADS, 1)
    corr_screen_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmBh, const ScreenParams p) {
  using C = ScreenCfg;
  constexpr int KB = 64;
  constexpr int STAGES = C::STAGES, A_BYTES = C::A_BYTES, STAGE_BYTES = C::STAGE_BYTES, A_RES = C::A_RES_BYTES;
  const int crank = (CL == 2) ? (int)tc::cluster_ctarank() : 0;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ring = smem + A_RES;  // the resident query tile comes first, then the ring of reference tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + STAGES * STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  uint64_t* afull = bars + 2 * STAGES;
  int* s_ci = reinterpret_cast<int*>(ring + STAGES * STAGE_BYTES + 256);  // [SCREEN_K][LT] candidate columns

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  const int bphi = (p.Bphi == 1) ? 0 : b;
  const int m0 = blockIdx.x * BM;
  const int ntiles_all = (p.NB + BN - 1) / BN;
  const int t0 = blockIdx.z * p.tiles_per_split;
  const int ntiles = max(min(t0 + p.tiles_per_split, ntiles_all) - t0, 0);
  const int nkb = p.C / KB;

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmAh);
    tc::tma_prefetch_desc(&tmBh);
    for (int i = 0; i < STAGES; ++i) tc::mbar_init(&full[i], 1), tc::mbar_init(&empty[i], CONSUMER_WARPS * CL);
    tc::mbar_init(afull, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  if (CL == 2) tc::cluster_sync_all();

  if (warp < 4) {
    tc::setmaxnreg_dec<40>();
    if (warp == 0) {
      int stage = 0;
      uint32_t phase = 0;
      if (ntiles > 0 && tc::elect_one()) {  // the query tile: loaded once, resident for the whole sweep
        tc::mbar_arrive_expect_tx(afull, A_RES);
        for (int kb = 0; kb < nkb; ++kb) tc::tma_load_2d(smem + kb * A_BYTES, &tmAh, afull, kb * KB, p.qsrc.at(b) * p.NA + m0);
      }
      __syncwarp();
      for (int t = 0; t < ntiles; ++t) {
        const int col0 = bphi * p.NB + (t0 + t) * BN;
        for (int kb = 0; kb < nkb; ++kb) {
          tc::mbar_wait(&empty[stage], phase ^ 1);
          if (tc::elect_one()) {
            uint8_t* st = ring + stage * STAGE_BYTES;
            tc::mbar_arrive_expect_tx(&full[stage], STAGE_BYTES);
            if (CL == 1) {
              tc::tma_load_2d(st, &tmBh, &full[stage], kb * KB, col0);
            } else {
              const int h = crank * (BN / 2);
              tc::tma_load_2d_mc(st + h * 128, &tmBh, &full[stage], kb * KB, col0 + h, 3);
            }
          }
          __syncwarp();
          if (++stage == STAGES) stage = 0, phase ^= 1;
        }
      }
    }
  } else {
    // ================= consumers: one hi.hi pass, then the candidate search on the registers =================
    // Every 16-value chunk (8 column pairs) whose maximum comes within the threshold of the row's running maximum (a
    // "record" or a near-tie) builds a mask of its qualifying columns and appends their indices to the (thread, row)
    // list in shared memory.  Values are not kept: a record that beats the previous maximum by more than the threshold
    // disqualifies the whole list at once (every entry is <= the previous maximum); otherwise the old entries stay -- at
    // worst a few extra candidates for the exact re-scoring, never a missing one.
    tc::setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1, qd = lane & 3;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int et = threadIdx.x - 128;  // consumer thread index
    const uint32_t a_off = (uint32_t)(wg * 64 * 128);
    float thr[2], run_m[2] = {-INFINITY, -INFINITY};
    int cnt[2] = {0, 0};  // entries appended (only the first SCREEN_K are stored: cnt > SCREEN_K = overflow)
#pragma unroll
    for (int h = 0; h < 2; ++h) {  // candidate threshold in accumulator units (scores there are true scores * 2^28)
      const size_t grow = (size_t)p.qsrc.at(b) * p.NA + min(m0 + rl + 8 * h, p.NA - 1);
      thr[h] = screen_threshold(__ldg(p.nd_a + grow), __ldg(p.nh_a + grow), __uint_as_float(__ldg(p.nd_b_max)),
                                __uint_as_float(__ldg(p.nh_b_max))) * 268435456.0f;
    }
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    if (ntiles > 0) tc::mbar_wait(afull, 0);
    for (int t = 0; t < ntiles; ++t) {
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        tc::mbar_wait(&full[stage], phase);
        const uint64_t dA = tc::wg_desc_k128(tc::smem_u32(smem + kb * A_BYTES) + a_off);
        const uint64_t dB = tc::wg_desc_k128(tc::smem_u32(ring + stage * STAGE_BYTES));
        tc::wg_fence_regs(acc);
        tc::wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) tc::wgmma_f16(acc, dA + kk * 2, dB + kk * 2, (kb | kk) ? 1u : 0u);
        tc::wg_commit();
        if (prev >= 0) {
          tc::wg_wait<1>();
          tc::release_stage<CL>(&empty[prev], lane);
        }
        prev = stage;
        if (++stage == STAGES) stage = 0, phase ^= 1;
      }
      tc::wg_wait<0>();
      tc::wg_fence_regs(acc);
      tc::release_stage<CL>(&empty[prev], lane);

      const int colbase = (t0 + t) * BN;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int c = 0; c < BN / 64; ++c) {  // chunk c: column pairs j = 8c .. 8c+7, bit i <-> (j = 8c + i / 2, e = i % 2)
          float v[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int col = colbase + 8 * (8 * c + i / 2) + 2 * qd + (i & 1);
            // columns at or beyond NB hold zero-filled (TMA) or foreign operands: mask them
            v[i] = col < p.NB ? acc[4 * (8 * c + i / 2) + 2 * h + (i & 1)] : -INFINITY;
          }
          float cm = -INFINITY;
#pragma unroll
          for (int i = 0; i < 16; ++i) cm = fmaxf(cm, v[i]);
          if (cm - thr[h] > run_m[h]) cnt[h] = 0;  // a record that disqualifies every earlier entry (all <= the old maximum)
          run_m[h] = fmaxf(run_m[h], cm);
          const float lim = run_m[h] - thr[h];
          if (cm >= lim && cm > -INFINITY) {
            uint32_t mask = 0;
#pragma unroll
            for (int i = 0; i < 16; ++i) mask |= (v[i] >= lim ? 1u : 0u) << i;
            while (mask) {
              const int i = __ffs(mask) - 1;
              mask &= mask - 1;
              if (cnt[h] < SCREEN_K) s_ci[cnt[h] * C::LT + et * 2 + h] = colbase + 8 * (8 * c + i / 2) + 2 * qd + (i & 1);
              ++cnt[h];
            }
            if (cnt[h] > SCREEN_K) cnt[h] = SCREEN_K + 1;  // overflow (sticky until a disqualifying record clears the list)
          }
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m0 + rl + 8 * h;
      if (row < p.NA) {
        const size_t o = ((size_t)(blockIdx.z * QUADS + qd) * p.B + b) * p.NA + row;
        p.pm[o] = run_m[h] * 3.725290298461914e-09f;
        const bool overflow = cnt[h] > SCREEN_K;
        if (!overflow)
          for (int j = 0; j < cnt[h]; ++j) p.pidx[o * SCREEN_K + j] = s_ci[j * C::LT + et * 2 + h];
        p.pcnt[o] = overflow ? -1 : cnt[h];
      }
    }
  }

  __syncthreads();
  if (CL == 2) tc::cluster_sync_all();
}


// Exact re-scoring: one warp per query row.  fp32 dot products of the ORIGINAL fp32 operands (lane l owns dimensions
// 4l..4l+3 and 128+4l..128+4l+3, eight FMAs, then a butterfly sum that leaves the same bits in every lane), running
// (max, lowest index, number of bit-equal maxima, sum of their V rows) exactly like the 3-pass kernel's epilogue.
__global__ void __launch_bounds__(256) corr_rescore_kernel(const float* __restrict__ theta, const float* __restrict__ phi,
                                                           const float4* __restrict__ V, const ScreenParams p, int nparts,
                                                           float4* __restrict__ y, float* __restrict__ sim, int* __restrict__ argmax,
                                                           const CorrPeers peers) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int rows = p.B * p.NA;
  if (r >= rows) return;
  const int b = r / p.NA;
  const int bphi = (p.Bphi == 1) ? 0 : b;
  const float* ph = phi + (size_t)bphi * p.NB * 256;
  const float4* Vg = V + (size_t)bphi * p.NB;
  const int ra = p.qsrc.at(b) * p.NA + (r - b * p.NA);  // query row in theta and in the query norms
  const float4 a0 = __ldg(reinterpret_cast<const float4*>(theta + (size_t)ra * 256) + lane);
  const float4 a1 = __ldg(reinterpret_cast<const float4*>(theta + (size_t)ra * 256) + 32 + lane);
  auto score = [&](int col) {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(ph + (size_t)col * 256) + lane);
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(ph + (size_t)col * 256) + 32 + lane);
    float s0 = a0.x * b0.x, s1 = a1.x * b1.x;
    s0 = fmaf(a0.y, b0.y, s0), s1 = fmaf(a1.y, b1.y, s1);
    s0 = fmaf(a0.z, b0.z, s0), s1 = fmaf(a1.z, b1.z, s1);
    s0 = fmaf(a0.w, b0.w, s0), s1 = fmaf(a1.w, b1.w, s1);
    float sacc = s0 + s1;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, off);
    return sacc;
  };
  float pmax = -INFINITY;
  for (int s = 0; s < nparts; ++s) pmax = fmaxf(pmax, __ldg(p.pm + (size_t)s * rows + r));
  const float thr = screen_threshold(__ldg(p.nd_a + ra), __ldg(p.nh_a + ra), __uint_as_float(__ldg(p.nd_b_max)), __uint_as_float(__ldg(p.nh_b_max)));
  float m = -INFINITY, cnt = 0.f, t0 = 0.f, t1 = 0.f, t2 = 0.f;
  int idx = 0x7fffffff;
  auto visit = [&](int col) {
    const float f = score(col);
    if (f >= m) {
      const float4 v = __ldg(Vg + col);
      if (f > m) m = f, cnt = 0.f, t0 = t1 = t2 = 0.f, idx = col;
      idx = min(idx, col), cnt += 1.f, t0 += v.x, t1 += v.y, t2 += v.z;
    }
  };
  const int ntiles_all = (p.NB + BN - 1) / BN;
  for (int s = 0; s < nparts; ++s) {
    const size_t o = (size_t)s * rows + r;
    if (__ldg(p.pm + o) < pmax - thr) continue;  // nothing in this part can be the maximum
    const int n = __ldg(p.pcnt + o);
    if (n >= 0) {
      for (int j = 0; j < n; ++j) visit(__ldg(p.pidx + o * SCREEN_K + j));
    } else {  // overflowed list: every column of the part (column-range split x quad thread: columns with (col / 2) % 4 == qd)
      const int sp = s / QUADS, qd = s - sp * QUADS;
      const int c0 = sp * p.tiles_per_split * BN, c1 = min(min((sp + 1) * p.tiles_per_split, ntiles_all) * BN, p.NB);
      for (int col = c0 + 2 * qd; col < c1; col += 8) {
        visit(col);
        if (col + 1 < c1) visit(col + 1);
      }
    }
  }
  if (lane == 0) {
    float4 v;
    if (cnt == 1.f) {
      v = __ldg(Vg + idx);
    } else {
      const float inv = 1.f / cnt;
      v = make_float4(t0 * inv, t1 * inv, t2 * inv, 0.f);
    }
    y[r] = make_float4(v.x, v.y, v.z, 0.f);
    sim[r] = m;
    if (argmax) argmax[r] = idx;
    for (int g = 0; g < peers.n; ++g) {
      reinterpret_cast<float4*>(peers.y4[g])[peers.row0 + r] = make_float4(v.x, v.y, v.z, 0.f);
      peers.sim[g][peers.row0 + r] = m;
    }
  }
}

// ---- merge the column-range splits ----------------------------------------------------------------------
template <bool SOFTMAX>
__global__ void __launch_bounds__(256) corr_merge_kernel(const SplitOut* __restrict__ part, int nsplit, int rows, int NA,
                                                         int NB, int Bphi, float sc_all, const float* __restrict__ row_sc,
                                                         const float4* __restrict__ V, float4* __restrict__ y, float* __restrict__ sim,
                                                         int* __restrict__ argmax, float* __restrict__ denom, const CorrPeers peers) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const float sc = row_sc ? row_sc[r] : sc_all;
  const int b = r / NA;
  const float4* Vg = V + (size_t)((Bphi == 1) ? 0 : b) * NB;
  if (!SOFTMAX) {
    float m = -INFINITY;
    for (int s = 0; s < nsplit; ++s) m = fmaxf(m, part[(size_t)s * rows + r].m);
    // mean of the V rows of all bit-equal maxima (one row, exactly, when the maximum is unique)
    int idx = 0x7fffffff;
    float cnt = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int s = 0; s < nsplit; ++s) {
      const SplitOut o = part[(size_t)s * rows + r];
      if (o.m == m && o.s > 0.f) cnt += o.s, a0 += o.a0, a1 += o.a1, a2 += o.a2, idx = min(idx, o.idx);
    }
    float4 v;
    if (cnt == 1.f) {
      v = __ldg(Vg + idx);
    } else {
      const float inv = 1.f / cnt;
      v = make_float4(a0 * inv, a1 * inv, a2 * inv, 0.f);
    }
    y[r] = make_float4(v.x, v.y, v.z, 0.f);
    sim[r] = m;
    if (argmax) argmax[r] = idx;
    for (int g = 0; g < peers.n; ++g) {  // fused all-gather: the row goes to every GPU's full-size result
      reinterpret_cast<float4*>(peers.y4[g])[peers.row0 + r] = make_float4(v.x, v.y, v.z, 0.f);
      peers.sim[g][peers.row0 + r] = m;
    }
  } else {
    float m = -INFINITY;
    for (int s = 0; s < nsplit; ++s) m = fmaxf(m, part[(size_t)s * rows + r].m);
    float ssum = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int s = 0; s < nsplit; ++s) {
      const SplitOut o = part[(size_t)s * rows + r];
      if (o.m == -INFINITY) continue;
      const float w = exp2f((o.m - m) * sc);
      ssum += w * o.s, a0 += w * o.a0, a1 += w * o.a1, a2 += w * o.a2;
    }
    y[r] = make_float4(a0 / ssum, a1 / ssum, a2 / ssum, 0.f);
    sim[r] = m;
    if (denom) denom[r] = ssum;  // sum_j exp((f_ij - m_i) / T_i)
    if (argmax) argmax[r] = -1;
    for (int g = 0; g < peers.n; ++g) {
      reinterpret_cast<float4*>(peers.y4[g])[peers.row0 + r] = make_float4(a0 / ssum, a1 / ssum, a2 / ssum, 0.f);
      peers.sim[g][peers.row0 + r] = m;
    }
  }
}

int ws_get(CorrWorkspace* ws, int i, size_t bytes, void** out) {
  if (ws->cap[i] < bytes) {  // growth outside dvc_set_exemplar's reservation: a stand-alone call with a new shape
    if (ws->buf[i]) cudaFree(ws->buf[i]);
    ws->buf[i] = nullptr, ws->cap[i] = 0;
    if (i == 2 || i == 3 || i == 5) ws->phi_src = nullptr, ws->phi_version = -1;
    if (cudaMalloc(&ws->buf[i], bytes) != cudaSuccess) return -1;
    ws->cap[i] = bytes;
  }
  *out = ws->buf[i];
  return 0;
}

template <int FMT, bool SOFTMAX, int CL>
int launch_main_cl(const CUtensorMap& mAh, const CUtensorMap& mAl, const CUtensorMap& mBh, const CUtensorMap& mBl,
                   const TcParams& tp, dim3 grid, cudaStream_t s) {
  static unsigned long long attr_mask = 0;  // the attribute is per device
  if (first_use_on_device(&attr_mask)) {
    if (cudaFuncSetAttribute(corr_tc_kernel<FMT, SOFTMAX, CL>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES) != cudaSuccess)
      return -1;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid, cfg.blockDim = dim3(NTHREADS), cfg.dynamicSmemBytes = Cfg::SMEM_BYTES, cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = CL, at[0].val.clusterDim.y = 1, at[0].val.clusterDim.z = 1;
  cfg.attrs = at, cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, corr_tc_kernel<FMT, SOFTMAX, CL>, mAh, mAl, mBh, mBl, tp) == cudaSuccess ? 0 : -2;
}
template <int FMT, bool SOFTMAX>
int launch_main(const CUtensorMap& mAh, const CUtensorMap& mAl, const CUtensorMap& mBh, const CUtensorMap& mBl,
                const TcParams& tp, dim3 grid, int cl, cudaStream_t s) {
  return cl == 2 ? launch_main_cl<FMT, SOFTMAX, 2>(mAh, mAl, mBh, mBl, tp, grid, s)
                 : launch_main_cl<FMT, SOFTMAX, 1>(mAh, mAl, mBh, mBl, tp, grid, s);
}

}  // namespace

bool first_use_on_device(unsigned long long* mask) {
  static std::mutex mu;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(mu);
  const unsigned long long bit = 1ull << (dev & 63);
  if (*mask & bit) return false;
  *mask |= bit;
  return true;
}

// workspace buffer 5 of the screened path: 8 cells, then the reference-side and the query-side norms (launch_corr_tc)
static size_t screen_norm_bytes(int B, int Bphi, int NA, int NB) { return ((size_t)8 + (size_t)2 * Bphi * NB + (size_t)2 * B * NA) * 4; }

const unsigned int* corr_ws_screen_cells(const CorrWorkspace* ws) { return (const unsigned int*)ws->buf[5]; }
static size_t screen_cand_bytes(int nparts, int B, int NA) { return (size_t)nparts * B * NA * (8 + 4 * SCREEN_K); }

int corr_ws_reserve(CorrWorkspace* ws, int B, int Bphi, int NA, int NB) {
  void* d;
  const size_t ea = (size_t)B * NA * 256 * 4, ephi = (size_t)Bphi * NB * 256 * 4;  // tf32 words: the widest format
  const size_t part = (size_t)16 * QUADS * B * NA * sizeof(SplitOut);               // at most 16 column splits x 4 quad threads
  if (ws_get(ws, 0, ea, &d) || ws_get(ws, 1, ea, &d) || ws_get(ws, 2, ephi, &d) || ws_get(ws, 3, ephi, &d) || ws_get(ws, 4, part, &d) ||
      ws_get(ws, 5, screen_norm_bytes(B, Bphi, NA, NB), &d) || ws_get(ws, 6, screen_cand_bytes(16 * QUADS, B, NA), &d))
    return -1;
  return 0;
}

void corr_ws_free(CorrWorkspace* ws) {
  for (int i = 0; i < CorrWorkspace::NBUF; ++i) {
    if (ws->buf[i]) cudaFree(ws->buf[i]);
    ws->buf[i] = nullptr, ws->cap[i] = 0;
  }
  ws->phi_src = nullptr, ws->phi_version = -1;
}

template <int CL>
static int launch_screen_cl(const CUtensorMap& mA, const CUtensorMap& mB, const ScreenParams& sp, dim3 grid, cudaStream_t s) {
  static unsigned long long attr_mask = 0;
  if (first_use_on_device(&attr_mask)) {
    if (cudaFuncSetAttribute(corr_screen_kernel<CL>, cudaFuncAttributeMaxDynamicSharedMemorySize, ScreenCfg::SMEM_BYTES) != cudaSuccess)
      return -1;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid, cfg.blockDim = dim3(NTHREADS), cfg.dynamicSmemBytes = ScreenCfg::SMEM_BYTES, cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = CL, at[0].val.clusterDim.y = 1, at[0].val.clusterDim.z = 1;
  cfg.attrs = at, cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, corr_screen_kernel<CL>, mA, mB, sp) == cudaSuccess ? 0 : -2;
}

int launch_corr_tc(const CorrParams& p, int math, int cluster, int screen, CorrWorkspace* ws, long long phi_version,
                   cudaStream_t s, std::string* err) {
  auto fail = [&](const char* m) {
    if (err) *err = m;
    return -1;
  };
  const bool tf32 = (math == 1);
  const int fmt = math == 1 ? 0 : (math == 2 ? 1 : 2);  // DVC_MATH_TF32X3 / BF16X3 / FP16X3
  if (p.C < 64 || p.C % 64 || p.C > 4096) return fail("C must be a multiple of 64 (<= 4096)");
  const int eb = tf32 ? 4 : 2;
  // query rows in theta / the A planes: each query set once, however many batches read it
  const int qrows = p.qsrc.count(p.B) * p.NA;
  const size_t ea = (size_t)qrows * p.C, ephi = (size_t)p.Bphi * p.NB * p.C;
  void *Ah, *Al, *Bh, *Bl, *part;
  if (ws_get(ws, 0, ea * eb, &Ah) || ws_get(ws, 1, ea * eb, &Al) || ws_get(ws, 2, ephi * eb, &Bh) || ws_get(ws, 3, ephi * eb, &Bl))
    return fail("workspace allocation failed");

  int dev = 0, num_sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return fail("cudaDeviceGetAttribute(multiProcessorCount) failed");
  // column-range splits so that (row blocks x batch x splits) fills the SMs in whole waves
  const int cl = cluster == 2 ? 2 : 1;
  const int row_blocks = ((p.NA + BM - 1) / BM + cl - 1) / cl * cl;  // pairs: an even number of 128-row query tiles
  const int ntiles = (p.NB + BN - 1) / BN;
  int nsplit = 1;
  {
    const long ctas = (long)row_blocks * p.B;
    double best = -1.0;
    for (int sp = 1; sp <= 16 && sp <= ntiles; ++sp) {
      const int tps = (ntiles + sp - 1) / sp;
      const int eff_sp = (ntiles + tps - 1) / tps;
      const long total = ctas * eff_sp;
      const long waves = (total + num_sms - 1) / num_sms;
      const double eff = (double)total / (double)(waves * num_sms) * ((double)ntiles / (double)(tps * eff_sp)) -
                         0.01 * sp;  // mild penalty: every split re-runs the prologue
      if (eff > best) best = eff, nsplit = eff_sp;
    }
  }
  const int tps = (ntiles + nsplit - 1) / nsplit;
  nsplit = (ntiles + tps - 1) / tps;
  const bool softmax = !(p.temperature <= 2e-10f) || p.row_scale != nullptr;
  if (screen && fmt == 2 && !softmax && p.C == 256) {  // (the resident query tile of the screening kernel is sized for C = 256)
    // ---- screened T -> 0 path: hi planes + error norms, one fp16 pass, exact re-scoring of the candidates ----
    const int rows = p.B * p.NA, rphi = p.Bphi * p.NB;
    void *norms, *cand;
    const int sparts = nsplit * QUADS;
    if (ws_get(ws, 5, screen_norm_bytes(p.B, p.Bphi, p.NA, p.NB), &norms) || ws_get(ws, 6, screen_cand_bytes(sparts, p.B, p.NA), &cand))
      return fail("workspace allocation failed");
    // cells [8] | nd_b [rphi] | nh_b [rphi] | nd_a [rows] | nh_a [rows]: the reference side must not move with the query
    // row count, because a cached reference side is read again by calls with fewer query rows
    unsigned int* cells = (unsigned int*)norms;  // [0,1]: query side (unused maxima), [2,3]: reference side, [4..7]: padding
    float* nd_b = (float*)(cells + 8);
    float* nh_b = nd_b + rphi;
    float* nd_a = nh_b + rphi;
    float* nh_a = nd_a + rows;
    const bool phi_cached = phi_version >= 0 && ws->phi_src == p.phi && ws->phi_version == phi_version && ws->phi_fmt == 3 &&
                            ws->phi_elems == ephi;
    if (cudaMemsetAsync(cells, 0, (phi_cached ? 2 : 4) * sizeof(unsigned int), s) != cudaSuccess) return fail("cudaMemsetAsync failed");
    screen_planes_kernel<<<(qrows * 32 + 255) / 256, 256, 0, s>>>(p.theta, (__half*)Ah, nd_a, nh_a, cells + 0, cells + 1, qrows);
    if (!phi_cached) screen_planes_kernel<<<(rphi * 32 + 255) / 256, 256, 0, s>>>(p.phi, (__half*)Bh, nd_b, nh_b, cells + 2, cells + 3, rphi);
    launch_counter_add(phi_cached ? 1 : 2);
    ws->phi_src = phi_version >= 0 ? p.phi : nullptr, ws->phi_version = phi_version, ws->phi_fmt = 3, ws->phi_elems = ephi;
    CUtensorMap mA, mB;
    if (encode_tmap_2d(&mA, Ah, (uint64_t)qrows, p.C, BM, 64, 2) || encode_tmap_2d(&mB, Bh, (uint64_t)rphi, p.C, BN / cl, 64, 2))
      return fail("cuTensorMapEncodeTiled failed");
    ScreenParams sp;
    sp.NA = p.NA, sp.NB = p.NB, sp.B = p.B, sp.Bphi = p.Bphi, sp.C = p.C, sp.qsrc = p.qsrc, sp.tiles_per_split = tps;
    sp.nd_a = nd_a, sp.nh_a = nh_a, sp.nd_b_max = cells + 2, sp.nh_b_max = cells + 3;
    sp.pm = (float*)cand;
    sp.pcnt = (int*)(sp.pm + (size_t)sparts * rows);
    sp.pidx = sp.pcnt + (size_t)sparts * rows;
    dim3 grid(row_blocks, p.B, nsplit);
    const int rc = cl == 2 ? launch_screen_cl<2>(mA, mB, sp, grid, s) : launch_screen_cl<1>(mA, mB, sp, grid, s);
    if (rc) return fail(rc == -1 ? "cudaFuncSetAttribute(max dynamic smem) failed" : "cudaLaunchKernelEx failed");
    corr_rescore_kernel<<<(rows * 32 + 255) / 256, 256, 0, s>>>(p.theta, p.phi, reinterpret_cast<const float4*>(p.V), sp, sparts,
                                                                reinterpret_cast<float4*>(p.y), p.sim, p.argmax, p.peers);
    launch_counter_add(2);
    return 0;
  }
  const int nparts = nsplit * QUADS;  // partial rows the merge kernel combines
  if (ws_get(ws, 4, (size_t)nparts * p.B * p.NA * sizeof(SplitOut), &part)) return fail("workspace allocation failed");

  const int grid1 = num_sms * 8;
  // the reference side's planes survive from launch to launch while (pointer, version, format, size) are unchanged
  const bool phi_cached = phi_version >= 0 && ws->phi_src == p.phi && ws->phi_version == phi_version && ws->phi_fmt == fmt &&
                          ws->phi_elems == ephi;
  if (fmt == 0) {
    split_planes_kernel<0><<<grid1, 256, 0, s>>>(p.theta, Ah, Al, ea / 4);
    if (!phi_cached) split_planes_kernel<0><<<grid1, 256, 0, s>>>(p.phi, Bh, Bl, ephi / 4);
  } else if (fmt == 1) {
    split_planes_kernel<1><<<grid1, 256, 0, s>>>(p.theta, Ah, Al, ea / 4);
    if (!phi_cached) split_planes_kernel<1><<<grid1, 256, 0, s>>>(p.phi, Bh, Bl, ephi / 4);
  } else {
    split_planes_kernel<2><<<grid1, 256, 0, s>>>(p.theta, Ah, Al, ea / 4);
    if (!phi_cached) split_planes_kernel<2><<<grid1, 256, 0, s>>>(p.phi, Bh, Bl, ephi / 4);
  }
  launch_counter_add(phi_cached ? 1 : 2);
  ws->phi_src = phi_version >= 0 ? p.phi : nullptr, ws->phi_version = phi_version, ws->phi_fmt = fmt, ws->phi_elems = ephi;

  CUtensorMap mAh, mAl, mBh, mBl;
  const uint32_t boxk = tf32 ? 32 : 64;
  if (encode_tmap_2d(&mAh, Ah, (uint64_t)qrows, p.C, BM, boxk, eb) || encode_tmap_2d(&mAl, Al, (uint64_t)qrows, p.C, BM, boxk, eb) ||
      encode_tmap_2d(&mBh, Bh, (uint64_t)p.Bphi * p.NB, p.C, BN / cl, boxk, eb) ||
      encode_tmap_2d(&mBl, Bl, (uint64_t)p.Bphi * p.NB, p.C, BN / cl, boxk, eb))
    return fail("cuTensorMapEncodeTiled failed");

  TcParams tp;
  tp.NA = p.NA, tp.NB = p.NB, tp.B = p.B, tp.Bphi = p.Bphi, tp.C = p.C, tp.qsrc = p.qsrc, tp.tiles_per_split = tps;
  tp.sc = 1.4426950408889634f / p.temperature;
  tp.row_sc = p.row_scale;
  tp.out_scale = fmt == 2 ? 3.725290298461914e-09f /* 2^-28 */ : 1.0f;
  tp.V = reinterpret_cast<const float4*>(p.V);
  tp.part = reinterpret_cast<SplitOut*>(part);
  dim3 grid(row_blocks, p.B, nsplit);
  int rc;
  if (fmt == 0)
    rc = softmax ? launch_main<0, true>(mAh, mAl, mBh, mBl, tp, grid, cl, s) : launch_main<0, false>(mAh, mAl, mBh, mBl, tp, grid, cl, s);
  else if (fmt == 1)
    rc = softmax ? launch_main<1, true>(mAh, mAl, mBh, mBl, tp, grid, cl, s) : launch_main<1, false>(mAh, mAl, mBh, mBl, tp, grid, cl, s);
  else
    rc = softmax ? launch_main<2, true>(mAh, mAl, mBh, mBl, tp, grid, cl, s) : launch_main<2, false>(mAh, mAl, mBh, mBl, tp, grid, cl, s);
  if (rc) return fail(rc == -1 ? "cudaFuncSetAttribute(max dynamic smem) failed" : "cudaLaunchKernelEx failed");
  launch_counter_add(1);
  const int rows = p.B * p.NA;
  if (softmax)
    corr_merge_kernel<true><<<(rows + 255) / 256, 256, 0, s>>>(tp.part, nparts, rows, p.NA, p.NB, p.Bphi, tp.sc, p.row_scale, tp.V,
                                                                reinterpret_cast<float4*>(p.y), p.sim, p.argmax, p.denom, p.peers);
  else
    corr_merge_kernel<false><<<(rows + 255) / 256, 256, 0, s>>>(tp.part, nparts, rows, p.NA, p.NB, p.Bphi, tp.sc, nullptr, tp.V,
                                                                 reinterpret_cast<float4*>(p.y), p.sim, p.argmax, nullptr, p.peers);
  launch_counter_add(1);
  return 0;
}

}  // namespace dvc
