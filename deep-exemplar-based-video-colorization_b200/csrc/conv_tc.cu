// Convolution on the Hopper tensor cores (wgmma + TMA + mbarrier): DVC_MATH_TF32X3 (and its 3xFP16 default), and the
// one-pass DVC_MATH_FP16X1 (see P1 below).
//
// Same flat shifted GEMM as conv_simt.cu (Y[p, co] = sum_tap sum_ci X[p + off(tap), ci] W[tap][ci][co] over the
// padded pixel index p), with fp32-class accuracy from three 16/19-bit MMAs per product on hi/lo split operands
// (x = hi + lo):  lo.hi + hi.lo + hi.hi  -> one fp32 register tile.  Activations therefore live in HBM as two
// padded-NHWC planes; weights are split once at load time.  Default operand format: fp16 planes of x * 2^e with an
// exact power-of-two scale e (a host constant for tensors with a proven bound, else derived on the device from the
// measured max |input| and the weights' L1 norm: dvc_internal.cuh, DynOut); tf32 planes (fp32 words) remain for
// inputs without a known bound.
//
// Persistent kernel, one CTA per SM, 2-CTA CLUSTERS by default (two adjacent pixel tiles of the same channel tile: each
// CTA loads half of the weight tile and multicasts it to both), static round-robin over the (pixel-tile pair, channel
// tile) grid; 384 threads:
//   warp 0       TMA producer: per (tap, 128-byte k-block) loads X_hi, X_lo [BMT px x 128 B] at row offset off(tap) --
//                negative / past-the-end rows are zero-filled by TMA -- and W_hi, W_lo [BN x 128 B], SWIZZLE_128B, into
//                an mbarrier ring.
//   warps 4..11  two consumer warpgroups.  Tile 128 px x 64 / 128 channels: each warpgroup owns 64 pixels; tile 64 px x
//                256 channels: each owns 128 channels.  Per k-block 4 k-steps x 3 wgmma (the two cross terms of the whole
//                k-block first, hi.hi last) into fp32 registers; every chunk (kc k-blocks) that partial sum is added to
//                fp32 register totals with round-to-nearest adds (the tensor-core accumulation truncates) while the next
//                chunk's wgmma run into a second set of accumulator registers; then + bias,
//                + skip addend, activation, InstanceNorm statistics (shuffle reduction over the warp's pixels -> one
//                double atomic per channel and tile), measured max |y|, masked store of the interior pixels as fp32 /
//                tf32 planes / fp16 planes -- or the fused 1x1 + tanh tail of ColorVidNet instead of a store.
// The channel tile is capped by the register file: two partial sums + total of a 128 x 128 (or 64 x 256) tile take 192
// of the consumers' registers.
// Replaces nn.Conv2d (+ReLU/LeakyReLU/skip add) at NonlocalNet.py:235-255,364-423 and ColorVidNet.py:96-143.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>

#include "conv_tc.cuh"
#include "corr_tc.cuh"
#include "tc_common.cuh"

namespace dvc {

namespace {

constexpr int NTHREADS = 384;  // warpgroup 0: warp 0 TMA (1-3 idle); warpgroups 1, 2: MMA + epilogue
constexpr int CONSUMERS = 256;

// Tile geometry of a channel tile BN: pixels per tile, warpgroups along the channels, wgmma N per warpgroup
template <int BN>
struct Geo {
  static constexpr int WGN = BN == 256 ? 2 : 1;
  static constexpr int BMT = 128 / WGN;
  static constexpr int NW = BN / WGN;
  static constexpr int R = NW / 2;  // accumulator registers per thread
};

// KBY = bytes of K per pipeline stage and operand row: 128 (SWIZZLE_128B, 32 tf32 / 64 fp16) or 64 (SWIZZLE_64B).
// Every CTA holds the whole weight tile of a stage (in a cluster half of it arrives by the peer's multicast).
// P1 (one pass): a stage holds the hi planes only, so the same shared memory holds twice as many stages.
template <int BN, int KBY, bool P1 = false>
struct Cfg {
  static constexpr int PLANES = P1 ? 1 : 2;
  static constexpr int STAGES = (BN == 256 ? 2 : (BN == 128 ? 3 : 4)) * (128 / KBY) * (P1 ? 2 : 1);
  static constexpr int A_BYTES = Geo<BN>::BMT * KBY;
  static constexpr int B_BYTES = BN * KBY;
  static constexpr int STAGE_BYTES = PLANES * A_BYTES + PLANES * B_BYTES;
  // + barriers + statistics [8 consumer warps][2][BN]
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 512 + 8 * 2 * BN * 4;
};

// Row-shared taps (RS): the three horizontal taps of a 3x3 row (two of a 2x2 phase-convolution row) read pixel rows
// that differ by `dil` positions of the flat padded index, i.e. the SAME shared-memory tile shifted by dil rows.  One
// activation tile of AR = BMT + 8 rows is loaded per (tap row, k-block) and the wgmma descriptors of the taps start dil *
// 128 bytes apart: a third of the activation bytes through TMA and L2 (the weights still arrive per tap, in a ring of
// their own).
template <int BN, bool P1 = false>
struct CfgRS {
  static constexpr int PLANES = P1 ? 1 : 2;
  static constexpr int AR = Geo<BN>::BMT + 8;
  static constexpr int A_TILE = AR * 128;              // one plane (a multiple of the 1024-byte swizzle atom)
  static constexpr int A_STAGE = PLANES * A_TILE;      // hi + lo (P1: hi)
  static constexpr int B_TILE = BN * 128;
  static constexpr int B_STAGE = PLANES * B_TILE;
  static constexpr int A_STAGES = ((BN == 256) ? 2 : 3) * (P1 ? 2 : 1);
  static constexpr int B_STAGES = ((BN == 64) ? 4 : (BN == 128 ? 3 : 2)) * (P1 ? 2 : 1);
  static constexpr int RING_BYTES = A_STAGES * A_STAGE + B_STAGES * B_STAGE;
  static constexpr int SMEM_BYTES = RING_BYTES + 1024 + 512 + 8 * 2 * BN * 4;
};
constexpr int RS_SLACK = 8;  // rows of shift a row-shared activation tile allows

__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

// CL = 2: the kernel runs as 2-CTA clusters on adjacent pixel tiles of the same channel tile; each CTA loads its own
// pixel rows and half of the weight rows, multicast into both CTAs (half the weight bytes through L2 per CTA).
// F16: operands are fp16 hi/lo planes of x * 2^e (e static per tensor / layer, chosen from a proven bound so that
// nothing overflows): the same 2 x 11 significant bits as the tf32 split at twice the MMA rate, half the operand
// bytes and half as many truncating accumulations per unit of K; the epilogue multiplies by 2^-(e_x + e_w) (exact).
// P1 (DVC_MATH_FP16X1): one MMA per product, hi.hi, on the same planes -- the producer loads X_hi and W_hi only and
// the consumers issue one wgmma per k-step.  The operands are rounded to 11 significant bits (fp16 planes: the power-of-
// two scale is exact; tf32 planes: cvt.rna), as cuDNN rounds fp32 convolution operands to TF32; the products are
// exact and the accumulation is the three-pass engine's, so only the operand rounding differs from it.
template <int BN, int CL, int KBY, bool F16, bool RS = false, bool P1 = false>
__global__ void __launch_bounds__(NTHREADS, 1)
    conv_tc_kernel(const __grid_constant__ CUtensorMap tmXh, const __grid_constant__ CUtensorMap tmXl,
                   const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const ConvTcParams p) {
  using G = Geo<BN>;
  using C = Cfg<BN, KBY, P1>;
  using RC = CfgRS<BN, P1>;
  static_assert(!RS || KBY == 128, "row-shared taps use 128-byte K blocks");
  constexpr int BMT = G::BMT, R = G::R;
  constexpr int A_BYTES = C::A_BYTES;
  constexpr int RING = RS ? RC::RING_BYTES : C::STAGES * C::STAGE_BYTES;
  constexpr int NFULL = RS ? (RC::A_STAGES + RC::B_STAGES) : C::STAGES;  // "full" barriers (then as many "empty" ones)
  constexpr int KE = F16 ? KBY / 2 : KBY / 4;  // K elements per stage
  constexpr int FMT = F16 ? 2 : 0;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + RING);
  uint64_t* full = bars;  // RS: [A_STAGES] activation tiles, then [B_STAGES] weight tiles
  uint64_t* empty = bars + NFULL;
  float* s_stat = reinterpret_cast<float*>(smem + RING + 512);  // [8 consumer warps][2][BN]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = p.mtn ? p.mtn * (128 / BMT) : (p.Mtot + BMT - 1) / BMT;
  const int n_tiles = p.CoutPad / BN;
  const int crank = (CL == 2) ? (int)tc::cluster_ctarank() : 0;
  const int m_groups = (m_tiles + CL - 1) / CL;          // CL adjacent pixel tiles per work item
  const int total_items = m_groups * n_tiles;
  const int item0 = blockIdx.x / CL, item_stride = gridDim.x / CL;
  const int kbs = p.Cin / KE;
  const int nk = p.taps * kbs;
  // Each wgmma accumulation truncates; a chunk of `kc` k-blocks (12*kc accumulations) is therefore summed in the
  // accumulator registers from zero and then added -- with round-to-nearest fp32 adds -- to a register total (the
  // tensor-core analogue of conv_simt.cu's two-level accumulation).  Per 128-byte k-block the three-pass engine makes
  // 12 accumulations of which 4 (hi.hi) are full-size; the one-pass engine makes those 4 only.  Either way a chunk
  // holds 4*kc full-size truncating accumulations, so P1 keeps the chunk length and spends its halved stage size on
  // twice the ring stages.
  const int kc = p.kc * (128 / KBY);  // p.kc counts 128-byte k-blocks
  const int nchunks = (nk + kc - 1) / kc;
  // Split-K against wave quantisation: a work item is (tile, split s of S); split s sums the chunks
  // [nchunks*s/S, nchunks*(s+1)/S) on top of the register totals that split s-1 left in an fp32 workspace, so the
  // accumulation order -- and every output bit -- is the same as without splitting.  Items are ordered split-major and
  // every CTA walks its items in increasing order, so the chain of waits always ends at a split-0 item that waits for
  // nothing (all CTAs are resident: one per SM).
  const int S = p.splits;
  const int total_work = total_items * S;
  const int px0 = p.mt0 * 128;  // first pixel of this launch's tile range

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tmXh);
    tc::tma_prefetch_desc(&tmWh);
    if (!P1) {
      tc::tma_prefetch_desc(&tmXl);
      tc::tma_prefetch_desc(&tmWl);
    }
    for (int i = 0; i < NFULL; ++i) tc::mbar_init(&full[i], 1), tc::mbar_init(&empty[i], 8 * CL);  // consumer warps of the cluster
    tc::fence_barrier_init();
  }
  __syncthreads();
  if (CL == 2) tc::cluster_sync_all();  // the peer's barriers are initialised before any multicast or remote arrive reaches them

  if (warp < 4) {
    // register budget: the producer warpgroup gives its registers to the two consumer warpgroups
    tc::setmaxnreg_dec<40>();
    if (warp == 0) {
      // ================= TMA producer =================
      // The whole warp runs the loop convergently (so that addresses / coordinates are provably warp-uniform); one
      // elected lane issues the instructions.
      auto load_w = [&](uint8_t* st, uint64_t* fb, int kb, int wrow, int bbytes) {
        if (CL == 1) {
          tc::tma_load_2d(st, &tmWh, fb, kb * KE, wrow);
          if (!P1) tc::tma_load_2d(st + bbytes, &tmWl, fb, kb * KE, wrow);
        } else {  // my half of the channel rows, multicast into both CTAs
          const int h = crank * (BN / 2);
          tc::tma_load_2d_mc(st + h * KBY, &tmWh, fb, kb * KE, wrow + h, 3);
          if (!P1) tc::tma_load_2d_mc(st + bbytes + h * KBY, &tmWl, fb, kb * KE, wrow + h, 3);
        }
      };
      if constexpr (RS) {
        // k runs over (tap row ty, k-block kb, tap column tx) with tx fastest: the activation tile of (ty, kb) serves
        // its ntx taps; weights come per tap.  (No split-K in this mode: p.splits == 1.)
        const int ntx = p.rs_ntx, ngroups = nk / ntx;
        uint8_t* ringB = smem + RC::A_STAGES * RC::A_STAGE;
        int as = 0, bs = 0;
        uint32_t aph = 0, bph = 0;
        for (int work = item0; work < total_work; work += item_stride) {
          const int mg = work / n_tiles, nt = work - mg * n_tiles;
          const int m0 = px0 + (mg * CL + crank) * BMT, n0 = nt * BN;
          for (int g = 0; g < ngroups; ++g) {
            const int ty = g / kbs, kb = g - ty * kbs;
            tc::mbar_wait(&empty[as], aph ^ 1);
            if (tc::elect_one()) {
              uint8_t* st = smem + as * RC::A_STAGE;
              const int row = m0 + p.tap_off[ty * ntx];
              tc::mbar_arrive_expect_tx(&full[as], RC::A_STAGE);
              tc::tma_load_2d(st, &tmXh, &full[as], kb * KE, row);
              if (!P1) tc::tma_load_2d(st + RC::A_TILE, &tmXl, &full[as], kb * KE, row);
            }
            __syncwarp();
            if (++as == RC::A_STAGES) as = 0, aph ^= 1;
            for (int tx = 0; tx < ntx; ++tx) {
              const int tap = ty * ntx + tx;
              uint64_t* fb = &full[RC::A_STAGES + bs];
              tc::mbar_wait(&empty[RC::A_STAGES + bs], bph ^ 1);
              if (tc::elect_one()) {
                tc::mbar_arrive_expect_tx(fb, RC::B_STAGE);
                load_w(ringB + bs * RC::B_STAGE, fb, kb, tap * p.CoutPad + n0, RC::B_TILE);
              }
              __syncwarp();
              if (++bs == RC::B_STAGES) bs = 0, bph ^= 1;
            }
          }
        }
      } else {
        int stage = 0;
        uint32_t phase = 0;
        for (int work = item0; work < total_work; work += item_stride) {
          const int sp = work / total_items, item = work - sp * total_items;
          const int mg = item / n_tiles, nt = item - mg * n_tiles;
          const int m0 = px0 + (mg * CL + crank) * BMT, n0 = nt * BN;
          const int k_lo = (nchunks * sp / S) * kc, k_hi = min((nchunks * (sp + 1) / S) * kc, nk);
          for (int k = k_lo; k < k_hi; ++k) {
            const int tap = k / kbs, kb = k - tap * kbs;
            const int off = p.tap_off[tap];
            tc::mbar_wait(&empty[stage], phase ^ 1);
            if (tc::elect_one()) {
              uint8_t* st = smem + stage * C::STAGE_BYTES;
              const bool skip_lo = P1 || (p.dbg & 2) != 0;  // dbg & 2: TIMING EXPERIMENT ONLY (wrong results): do not fetch the activation lo plane
              tc::mbar_arrive_expect_tx(&full[stage], C::STAGE_BYTES - (skip_lo && !P1 ? A_BYTES : 0));
              tc::tma_load_2d(st, &tmXh, &full[stage], kb * KE, m0 + off);
              if (!skip_lo) tc::tma_load_2d(st + A_BYTES, &tmXl, &full[stage], kb * KE, m0 + off);
              load_w(st + C::PLANES * A_BYTES, &full[stage], kb, tap * p.CoutPad + n0, C::B_BYTES);
            }
            __syncwarp();
            if (++stage == C::STAGES) stage = 0, phase ^= 1;
          }
        }
      }
    }
  } else {
    // ================= consumers: wgmma into registers, then the epilogue on them =================
    tc::setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1, wl = warp & 3, qd = lane & 3;
    const int ctid = threadIdx.x - 128;            // consumer thread index
    const int cw = warp - 4;                       // consumer warp index: statistics slot
    const int ro = G::WGN == 1 ? wg * 64 : 0;      // this warpgroup's first pixel row of the tile
    const int co = G::WGN == 2 ? wg * G::NW : 0;   // this warpgroup's first channel of the tile
    const int prow = ro + wl * 16 + (lane >> 2);   // pixel row of register slot 0 (slot 1: + 8)
    const int img = p.Hp * p.Wp;
    auto epi_sync = [&]() { asm volatile("bar.sync 1, 256;" ::: "memory"); };  // the 256 consumer threads
    // device-side scales (conv -> ReLU -> conv chains on fp16 planes, dvc_internal.cuh: DynOut)
    float oscale = p.out_scale, yscale = 1.f, amax = 0.f;
    if constexpr (F16) {
      if (p.dyn.cell_in) oscale *= exp2_int(-p.dyn.cell_in->e);
      if (p.dyn.h16) {
        const int e_out = dyn_out_exponent(p.dyn);
        yscale = exp2_int(e_out);
        if (ctid == 0 && blockIdx.x == 0) p.dyn.cell_out->e = e_out;
      }
    }
    float acc0[R], acc1[R], tot[R];
    // workspace layout [tile][register][consumer thread]: coalesced hand-over of the running totals
    auto tile_of = [&](int w) {
      const int item = w % total_items, mg = item / n_tiles;
      return (mg * CL + crank) * n_tiles + (item - mg * n_tiles);
    };
    // Totals of work item w before its first chunk: -0 (the identity of the round-to-nearest adds, so the first chunk
    // lands in them bit for bit), or what split sp - 1 left in the workspace
    auto start_item = [&](int w) {
      const int sp = w / total_items;
      if (sp == 0) {
#pragma unroll
        for (int j = 0; j < R; ++j) tot[j] = -0.f;
        return;
      }
      const int tile_id = tile_of(w);
      if (ctid == 0) {
        const int want = p.epoch * 16 + sp;
        int got;
        do {
          asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(got) : "l"(p.flags + tile_id) : "memory");
        } while (got != want);
      }
      epi_sync();
      const float* wsp = p.ws + (size_t)tile_id * BN * BMT + ctid;
#pragma unroll
      for (int j = 0; j < R; ++j) tot[j] = __ldcg(wsp + (size_t)j * CONSUMERS);
    };
    // Epilogue of work item w on its totals
    auto finish_item = [&](int w) {
      const int sp = w / total_items, item = w - sp * total_items;
      const int mg = item / n_tiles, nt = item - mg * n_tiles;
      const int m0 = px0 + (mg * CL + crank) * BMT, n0 = nt * BN;
      const int tile_id = tile_of(w);
      if (sp < S - 1) {  // hand the running totals to the next split of this tile
        float* wsp = p.ws + (size_t)tile_id * BN * BMT + ctid;
#pragma unroll
        for (int j = 0; j < R; ++j) __stcg(wsp + (size_t)j * CONSUMERS, tot[j]);
        __threadfence();
        epi_sync();
        if (ctid == 0) {
          const int v = p.epoch * 16 + sp + 1;
          asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p.flags + tile_id), "r"(v) : "memory");
        }
        return;
      }

      // ---- bias, skip addend, activation, statistics, masked store ----
      // register tot[4 j + 2 h + e] = pixel row prow + 8 h, channel co + 8 j + 2 qd + e
      bool valid[2];
      int bimg[2], yo[2], xo[2];
      size_t yoff[2], aoff[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int pp = m0 + prow + 8 * h;
        valid[h] = pp < p.Mtot;
        bimg[h] = 0, yo[h] = 0, xo[h] = 0;
        if (valid[h]) {
          bimg[h] = pp / img;
          const int rem = pp - bimg[h] * img;
          const int yp = rem / p.Wp, xp = rem - yp * p.Wp;
          const int y = yp - p.P, x = xp - p.P;
          valid[h] = (y >= 0 && y < p.H && x >= 0 && x < p.W);
          if (p.stride == 2 && ((y | x) & 1)) valid[h] = false;
          yo[h] = (y / p.stride) * p.oscale + p.oa, xo[h] = (x / p.stride) * p.oscale + p.ob;
        }
        yoff[h] = valid[h] ? ((((size_t)bimg[h] * p.yHp + yo[h] + p.yP) * p.yWp + xo[h] + p.yP) * p.yC + p.yCoff) : 0;
        aoff[h] = (valid[h] && p.add) ? ((((size_t)bimg[h] * p.aHp + yo[h] + p.aP) * p.aWp + xo[h] + p.aP) * p.aC) : 0;
      }
      const int b_first = min(m0, p.Mtot - 1) / img, b_last = min(m0 + BMT - 1, p.Mtot - 1) / img;
      const bool uniform_img = (b_first == b_last);
      float fs0[2] = {0.f, 0.f}, fs1[2] = {0.f, 0.f};  // fused 1x1 tail: partial dot products over this thread's channels
#pragma unroll
      for (int j = 0; j < G::NW / 8; ++j) {
        const int chn = n0 + co + 8 * j + 2 * qd;  // channels chn, chn + 1
        if (chn >= p.Cout) continue;
        const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + chn));
        float ssum[2] = {0.f, 0.f}, ssq[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v0, v1;
          if constexpr (F16) {
            v0 = fmaf(tot[4 * j + 2 * h], oscale, bv.x), v1 = fmaf(tot[4 * j + 2 * h + 1], oscale, bv.y);
          } else {
            v0 = tot[4 * j + 2 * h] + bv.x, v1 = tot[4 * j + 2 * h + 1] + bv.y;
          }
          if (p.add && valid[h]) {
            float2 av = __ldg(reinterpret_cast<const float2*>(p.add + aoff[h] + chn));
            if (p.add_lo) {
              const float2 al = __ldg(reinterpret_cast<const float2*>(p.add_lo + aoff[h] + chn));
              av.x += al.x, av.y += al.y;
            }
            v0 += av.x, v1 += av.y;
          }
          if (p.act == ACT_RELU) v0 = fmaxf(v0, 0.f), v1 = fmaxf(v1, 0.f);
          if (p.act == ACT_LRELU) v0 = v0 > 0.f ? v0 : v0 * p.slope, v1 = v1 > 0.f ? v1 : v1 * p.slope;
          if (BN == 128 && p.fin_out) {
            const float2 w0 = __ldg(reinterpret_cast<const float2*>(p.fin_w + chn));
            const float2 w1 = __ldg(reinterpret_cast<const float2*>(p.fin_w + p.Cout + chn));
            fs0[h] += v0 * w0.x + v1 * w0.y;
            fs1[h] += v0 * w1.x + v1 * w1.y;
          }
          if (F16 && p.dyn.cell_out && valid[h]) amax = fmaxf(amax, fmaxf(fabsf(v0), fabsf(v1)));
          if (valid[h]) {
            if (F16 && p.dyn.h16) {
              const float x0 = fminf(fmaxf(v0 * yscale, -65504.f), 65504.f);
              const float x1 = fminf(fmaxf(v1 * yscale, -65504.f), 65504.f);
              const __half2 h2 = __floats2half2_rn(x0, x1);
              const float2 hf = __half22float2(h2);
              const __half2 l2 = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
              *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.dyn.h16) + yoff[h] + chn) = h2;
              *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.dyn.l16) + yoff[h] + chn) = l2;
            } else if (p.y_lo) {
              const float h0 = tf32_rna(v0), h1 = tf32_rna(v1);
              *reinterpret_cast<float2*>(p.y + yoff[h] + chn) = make_float2(h0, h1);
              *reinterpret_cast<float2*>(p.y_lo + yoff[h] + chn) = make_float2(tf32_rna(v0 - h0), tf32_rna(v1 - h1));
            } else if (p.y) {
              *reinterpret_cast<float2*>(p.y + yoff[h] + chn) = make_float2(v0, v1);
            }
          }
          if (p.stats) {
            if (uniform_img) {
              if (valid[h]) ssum[0] += v0, ssum[1] += v1, ssq[0] += v0 * v0, ssq[1] += v1 * v1;
            } else if (valid[h]) {
              atomicAdd(&p.stats[((size_t)bimg[h] * p.Cout + chn) * 2 + 0], (double)v0);
              atomicAdd(&p.stats[((size_t)bimg[h] * p.Cout + chn) * 2 + 1], (double)v0 * (double)v0);
              atomicAdd(&p.stats[((size_t)bimg[h] * p.Cout + chn + 1) * 2 + 0], (double)v1);
              atomicAdd(&p.stats[((size_t)bimg[h] * p.Cout + chn + 1) * 2 + 1], (double)v1 * (double)v1);
            }
          }
        }
        if (p.stats && uniform_img) {
          // the warp's 16 pixel rows of these two channels: butterfly over the 8 lanes that share qd (fixed order within
          // the tile; the tiles' double atomics below land in completion order, and the per-pixel double squares of tiles
          // that straddle an image boundary make the last bits of those sums depend on it)
#pragma unroll
          for (int off = 4; off <= 16; off <<= 1) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              ssum[e] += __shfl_xor_sync(0xffffffffu, ssum[e], off);
              ssq[e] += __shfl_xor_sync(0xffffffffu, ssq[e], off);
            }
          }
          if (lane < 4) {
            const int cl = co + 8 * j + 2 * qd;
            s_stat[(cw * 2 + 0) * BN + cl] = ssum[0], s_stat[(cw * 2 + 0) * BN + cl + 1] = ssum[1];
            s_stat[(cw * 2 + 1) * BN + cl] = ssq[0], s_stat[(cw * 2 + 1) * BN + cl + 1] = ssq[1];
          }
        }
      }
      if (BN == 128 && p.fin_out) {  // a pixel's 128 channels live in the 4 threads of its quad
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int off = 1; off <= 2; off <<= 1) {
            fs0[h] += __shfl_xor_sync(0xffffffffu, fs0[h], off);
            fs1[h] += __shfl_xor_sync(0xffffffffu, fs1[h], off);
          }
          if (qd == 0 && valid[h]) {
            const size_t hw = (size_t)p.H * p.W, po = (size_t)yo[h] * p.W + xo[h];
            p.fin_out[((size_t)bimg[h] * 2 + 0) * hw + po] = tanhf(fs0[h] + __ldg(p.fin_b + 0)) * 128.f;
            p.fin_out[((size_t)bimg[h] * 2 + 1) * hw + po] = tanhf(fs1[h] + __ldg(p.fin_b + 1)) * 128.f;
          }
        }
      }
      if (p.stats) {
        epi_sync();
        if (uniform_img) {
          constexpr int SLOTS = 8 / G::WGN;  // consumer warps that hold partial sums of one channel
          for (int i = ctid; i < BN; i += CONSUMERS) {
            const int chn = n0 + i;
            if (chn < p.Cout) {
              const int w0 = G::WGN == 2 ? (i / G::NW) * 4 : 0;
              double s4 = 0.0, q4 = 0.0;
              for (int sl = 0; sl < SLOTS; ++sl) s4 += (double)s_stat[((w0 + sl) * 2 + 0) * BN + i], q4 += (double)s_stat[((w0 + sl) * 2 + 1) * BN + i];
              atomicAdd(&p.stats[((size_t)b_first * p.Cout + chn) * 2 + 0], s4);
              atomicAdd(&p.stats[((size_t)b_first * p.Cout + chn) * 2 + 1], q4);
            }
          }
        }
        epi_sync();
      }
    };

    int stage = 0, as = 0, bs = 0;  // ring positions of the next k-block
    uint32_t phase = 0, aph = 0, bph = 0;
    int prev_stage = -1, prev_a = -1;  // ring stages the k-block in flight frees when retired (-1: none)
    auto retire_prev = [&]() {
      tc::release_stage<CL>(&empty[prev_stage], lane);
      if (RS && prev_a >= 0) tc::release_stage<CL>(&empty[prev_a], lane);
    };
    // Issue k-block k into the accumulator set `a` (FIRST: the first of its chunk, which overwrites `a`), then retire
    // the k-block issued before it
    auto kblock = [&](float (&a)[R], int k, bool first) {
      uint32_t sa, sb;
      uint64_t bo = 0;
      int tx = 0, ntx = 1;
      if constexpr (RS) {
        ntx = p.rs_ntx;
        const int g = k / ntx, ty = g / kbs;
        tx = k - g * ntx;
        if (tx == 0) tc::mbar_wait(&full[as], aph);  // the activation tile of this (tap row, k-block)
        tc::mbar_wait(&full[RC::A_STAGES + bs], bph);
        // the tap's rows start (tap_off[tap] - tap_off[first tap of the row]) rows into the shared tile
        // (p.dbg & 1: TIMING EXPERIMENT ONLY, wrong results -- every tap reads the tile at its aligned start)
        const int shift = (p.dbg & 1) ? 0 : p.tap_off[ty * ntx + tx] - p.tap_off[ty * ntx];
        sa = tc::smem_u32(smem + as * RC::A_STAGE) + (uint32_t)(ro + shift) * 128u;
        sb = tc::smem_u32(smem + RC::A_STAGES * RC::A_STAGE + bs * RC::B_STAGE) + (uint32_t)co * 128u;
        bo = p.rs_base_offset ? ((uint64_t)(shift & 7) << 49) : 0ull;
      } else {
        tc::mbar_wait(&full[stage], phase);
        sa = tc::smem_u32(smem + stage * C::STAGE_BYTES) + (uint32_t)ro * KBY;
        sb = tc::smem_u32(smem + stage * C::STAGE_BYTES + C::PLANES * A_BYTES) + (uint32_t)co * KBY;
      }
      constexpr uint32_t A_PLANE = RS ? RC::A_TILE : A_BYTES, B_PLANE = RS ? RC::B_TILE : C::B_BYTES;
      auto mkdesc = [](uint32_t x) { return KBY == 128 ? tc::wg_desc_k128(x) : tc::wg_desc_k64(x); };
      const uint64_t dXh = mkdesc(sa) | bo, dXl = mkdesc(sa + A_PLANE) | bo;
      const uint64_t dWh = mkdesc(sb), dWl = mkdesc(sb + B_PLANE);
      tc::wg_fence_regs(a);
      tc::wg_fence();
      if constexpr (P1) {
#pragma unroll
        for (int kk = 0; kk < KBY / 32; ++kk) {
          const uint64_t adv = (uint64_t)(kk * 2);
          tc::wgmma_fmt<FMT>(a, dXh + adv, dWh + adv, (first && kk == 0) ? 0u : 1u);
        }
      } else {
        // Every accumulation truncates the accumulator at ITS current magnitude, so the two small cross terms of the
        // whole k-block go first (while a fresh accumulator is still ~2^-11 of its final size, their truncations are
        // negligible) and the dominant hi*hi terms last: 4 instead of 12 full-size truncations per k-block.
#pragma unroll
        for (int kk = 0; kk < KBY / 32; ++kk) {
          const uint64_t adv = (uint64_t)(kk * 2);
          tc::wgmma_fmt<FMT>(a, dXl + adv, dWh + adv, (first && kk == 0) ? 0u : 1u);
          tc::wgmma_fmt<FMT>(a, dXh + adv, dWl + adv, 1u);
        }
#pragma unroll
        for (int kk = 0; kk < KBY / 32; ++kk) {
          const uint64_t adv = (uint64_t)(kk * 2);
          tc::wgmma_fmt<FMT>(a, dXh + adv, dWh + adv, 1u);
        }
      }
      tc::wg_commit();
      tc::wg_wait<1>();  // unconditional (a no-op without an older group), so ptxas sees every older group retired
      if (prev_stage >= 0) retire_prev();
      if constexpr (RS) {
        prev_stage = RC::A_STAGES + bs, prev_a = tx == ntx - 1 ? as : -1;
        if (++bs == RC::B_STAGES) bs = 0, bph ^= 1;
        if (tx == ntx - 1 && ++as == RC::A_STAGES) as = 0, aph ^= 1;
      } else {
        prev_stage = stage;
        if (++stage == C::STAGES) stage = 0, phase ^= 1;
      }
    };
    // Chunk ch into set `a`; once its first k-block is issued, the previous chunk (set `o`, PROMOTE) has been retired
    // by kblock's wgmma.wait_group 1 and is added to the totals while `a` is in flight
    auto chunk = [&](float (&a)[R], float (&o)[R], int ch, bool promote) {
      const int k0 = ch * kc, k_end = min(k0 + kc, nk);
      kblock(a, k0, true);
      if (promote) {
        tc::wg_fence_regs(o);
#pragma unroll
        for (int j = 0; j < R; ++j) tot[j] += o[j];
      }
      for (int k = k0 + 1; k < k_end; ++k) kblock(a, k, false);
    };
    // the last chunk of a work item
    auto drain = [&](float (&a)[R]) {
      tc::wg_wait<0>();
      tc::wg_fence_regs(a);
      retire_prev();
      prev_stage = -1;
#pragma unroll
      for (int j = 0; j < R; ++j) tot[j] += a[j];
    };
    for (int work = item0; work < total_work; work += item_stride) {
      const int sp = work / total_items;
      start_item(work);
      // consecutive chunks alternate between the two accumulator sets
      const int ch_lo = nchunks * sp / S, ch_hi = nchunks * (sp + 1) / S;
      for (int ch = ch_lo;;) {
        chunk(acc0, acc1, ch, ch > ch_lo);
        if (++ch == ch_hi) {
          drain(acc0);
          break;
        }
        chunk(acc1, acc0, ch, true);
        if (++ch == ch_hi) {
          drain(acc1);
          break;
        }
      }

      finish_item(work);
    }
    if (F16 && p.dyn.cell_out) warp_amax_commit(amax, p.dyn.cell_out);
  }

  __syncthreads();
  if (CL == 2) tc::cluster_sync_all();  // no CTA may exit while its peer can still multicast into it or arrive on its barriers
}

template <int BN, int CL, int KBY, bool F16, bool RS = false, bool P1 = false>
int launch_bn(const CUtensorMap& mXh, const CUtensorMap& mXl, const CUtensorMap& mWh, const CUtensorMap& mWl,
              const ConvTcParams& p, int num_sms, cudaStream_t s) {
  constexpr int SMEM = RS ? CfgRS<BN, P1>::SMEM_BYTES : Cfg<BN, KBY, P1>::SMEM_BYTES;
  static unsigned long long attr_mask = 0;  // the attribute is per device
  if (first_use_on_device(&attr_mask)) {
    if (cudaFuncSetAttribute(conv_tc_kernel<BN, CL, KBY, F16, RS, P1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM) != cudaSuccess)
      return -1;
  }
  constexpr int BMT = Geo<BN>::BMT;
  const int m_tiles = p.mtn ? p.mtn * (128 / BMT) : (p.Mtot + BMT - 1) / BMT;
  const int items = ((m_tiles + CL - 1) / CL) * (p.CoutPad / BN) * p.splits;
  const int max_groups = num_sms / CL;
  const int grid = CL * (items < max_groups ? items : max_groups);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid), cfg.blockDim = dim3(NTHREADS), cfg.dynamicSmemBytes = SMEM, cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = CL, at[0].val.clusterDim.y = 1, at[0].val.clusterDim.z = 1;
  cfg.attrs = at, cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, conv_tc_kernel<BN, CL, KBY, F16, RS, P1>, mXh, mXl, mWh, mWl, p) == cudaSuccess ? 0 : -2;
}

// the instantiation for (row-shared taps, operand format, K bytes per stage) of a channel tile / cluster / pass count
template <int BN, int CL, bool P1>
int launch_variant(bool rs, bool f16, int KBY, const CUtensorMap& mXh, const CUtensorMap& mXl, const CUtensorMap& mWh,
                   const CUtensorMap& mWl, const ConvTcParams& q, int num_sms, cudaStream_t s) {
  if (rs) return f16 ? launch_bn<BN, CL, 128, true, true, P1>(mXh, mXl, mWh, mWl, q, num_sms, s)
                     : launch_bn<BN, CL, 128, false, true, P1>(mXh, mXl, mWh, mWl, q, num_sms, s);
  if (f16) return KBY == 128 ? launch_bn<BN, CL, 128, true, false, P1>(mXh, mXl, mWh, mWl, q, num_sms, s)
                             : launch_bn<BN, CL, 64, true, false, P1>(mXh, mXl, mWh, mWl, q, num_sms, s);
  return KBY == 128 ? launch_bn<BN, CL, 128, false, false, P1>(mXh, mXl, mWh, mWl, q, num_sms, s)
                    : launch_bn<BN, CL, 64, false, false, P1>(mXh, mXl, mWh, mWl, q, num_sms, s);
}

}  // namespace

int conv_tc_pick_bn(int cout) { return cout >= 256 ? 256 : (cout > 64 ? 128 : 64); }

// Channel tile for one launch: 128 channels for layers with more than 64 (the 64 x 256 tile does the same MMA work per
// item as the 128 x 128 one but moves 320 instead of 256 operand rows per k-block, so it is only run when forced), and
// the 64-channel tile where wider tiles would not give every SM pair a work item.
static int pick_bn_for_launch(const ConvTcParams& p, int num_sms) {
  const int m_tiles = (p.Mtot + 127) / 128;
  int bn = conv_tc_pick_bn(p.Cout) > 128 ? 128 : conv_tc_pick_bn(p.Cout);
  while (bn > 64 && m_tiles * (p.CoutPad / bn) < num_sms / 2) bn >>= 1;
  return bn;
}

int launch_conv_tc(const ConvTcParams& p, const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, int num_sms,
                   cudaStream_t s, std::string* err, int* variant) {
  auto fail = [&](const char* m) {
    if (err) *err = m;
    return -1;
  };
  if (p.Cin % 32) return fail("Cin must be a multiple of 32");
  // the epilogue handles channel pairs of 8-channel groups, and its statistics shuffles need the whole warp
  if (p.Cout % 8) return fail("Cout must be a multiple of 8");
  const bool f16 = p.f16 != 0;
  const int eb = f16 ? 2 : 4;
  // a 128-byte row holds 32 tf32 / 64 fp16 channels; 32-channel fp16 layers use the 64-byte (SWIZZLE_64B) rows
  const int KBY = (p.kbytes == 64 || (f16 && p.Cin % 64)) ? 64 : 128;
  if (p.kc < 1) return fail("kc must be >= 1");
  if (p.passes != 1 && p.passes != 3) return fail("passes must be 1 or 3");
  if (p.CoutPad % conv_tc_pick_bn(p.Cout)) return fail("CoutPad must be a multiple of the channel tile");
  if (p.fin_out && (p.Cout != 128 || p.stride != 1 || p.oscale != 1 || p.stats)) return fail("fused 1x1 tail needs a plain 128-channel layer");
  const int BN = p.force_bn ? p.force_bn : (p.fin_out ? 128 : pick_bn_for_launch(p, num_sms));
  if (variant && !p.mtn) *variant = BN;
  // 2-CTA clusters when there are at least two pixel tiles per SM pair to go around
  const int CL = (p.cluster == 2 && (p.Mtot + 127) / 128 >= 2) ? 2 : 1;
  if (p.tail && !p.mtn && CL == 2 && BN == 256 && p.CoutPad == 256 && p.splits == 1) {
    // Wave quantisation: a 256-channel launch whose last round is partly empty runs its whole rounds with the 256-channel
    // tile and the remaining pixel blocks with 128-channel tiles, when those fit in one round.
    const int m_tiles = (p.Mtot + 127) / 128, pairs = (m_tiles + 1) / 2, slots = p.tail > 1 ? p.tail : num_sms / 2;
    const int full = pairs / slots, rem = pairs - full * slots;
    if (full >= 1 && rem > 0 && 2 * rem <= slots) {
      ConvTcParams q1 = p, q2 = p;
      q1.mt0 = 0, q1.mtn = 2 * full * slots, q1.force_bn = 256;
      q2.mt0 = q1.mtn, q2.mtn = m_tiles - q1.mtn, q2.force_bn = 128;
      int rc1 = launch_conv_tc(q1, x_hi, x_lo, w_hi, w_lo, num_sms, s, err, nullptr);
      if (rc1) return rc1;
      return launch_conv_tc(q2, x_hi, x_lo, w_hi, w_lo, num_sms, s, err, nullptr);
    }
  }
  ConvTcParams q = p;
  {  // split-K factor: minimise rounds(S) / S over the persistent grid (2 % penalty per extra split for the hand-over)
    const int BMT = BN == 256 ? Geo<256>::BMT : Geo<128>::BMT;
    const int m_tiles = p.mtn ? p.mtn * (128 / BMT) : (p.Mtot + BMT - 1) / BMT;
    const int tiles = ((m_tiles + CL - 1) / CL) * CL * (p.CoutPad / BN);
    // k-blocks of KBY bytes and the chunks the kernel sums them in (p.kc counts 128-byte k-blocks)
    const int nk = p.taps * (p.Cin / (KBY / eb)), kcs = p.kc * (128 / KBY);
    const int nchunks = (nk + kcs - 1) / kcs;
    int best = 1;
    if (p.ws && p.flags && p.splits != 1) {
      double best_cost = 1e30;
      for (int S = 1; S <= 8; ++S) {
        if (S > 1 && nchunks / S < 6) break;
        const int rounds = (tiles * S + num_sms - 1) / num_sms;
        const double cost = (double)rounds / S * (1.0 + 0.02 * (S - 1));
        if (cost < best_cost - 1e-9) best_cost = cost, best = S;
      }
      if (p.splits > 1) best = p.splits < nchunks ? p.splits : nchunks;  // forced (tests)
      if (best < 1) best = 1;
    }
    q.splits = best;
  }
  // row-shared taps: taps of one kernel row read the same activation tile shifted by a few rows (see CfgRS)
  bool rs = false;
  if (p.rowshare && KBY == 128 && q.splits == 1 && (p.taps == 9 || p.taps == 4)) {
    const int ntx = p.taps == 9 ? 3 : 2;
    rs = true;
    for (int t = 0; t < p.taps; ++t) {
      const int sh = p.tap_off[t] - p.tap_off[(t / ntx) * ntx];
      if (sh < 0 || sh > RS_SLACK) rs = false;
    }
    q.rs_ntx = ntx, q.rs_base_offset = p.rowshare == 2 ? 1 : 0;
  }
  CUtensorMap mXh, mXl, mWh, mWl;
  const int bmt = BN == 256 ? Geo<256>::BMT : Geo<128>::BMT;
  const int abox = rs ? bmt + RS_SLACK : bmt;
  if (encode_tmap_2d(&mXh, x_hi, (uint64_t)p.Mtot, p.Cin, abox, KBY / eb, eb, KBY) ||
      encode_tmap_2d(&mXl, x_lo, (uint64_t)p.Mtot, p.Cin, abox, KBY / eb, eb, KBY) ||
      encode_tmap_2d(&mWh, w_hi, (uint64_t)p.taps * p.CoutPad, p.Cin, BN / CL, KBY / eb, eb, KBY) ||
      encode_tmap_2d(&mWl, w_lo, (uint64_t)p.taps * p.CoutPad, p.Cin, BN / CL, KBY / eb, eb, KBY))
    return fail("cuTensorMapEncodeTiled failed");
  int rc;
  const bool one = p.passes == 1;
#define DVC_LAUNCH(BNv, CLv)                                                                             \
  rc = one ? launch_variant<BNv, CLv, true>(rs, f16, KBY, mXh, mXl, mWh, mWl, q, num_sms, s)             \
           : launch_variant<BNv, CLv, false>(rs, f16, KBY, mXh, mXl, mWh, mWl, q, num_sms, s)
  if (CL == 2) {
    if (BN == 256) { DVC_LAUNCH(256, 2); } else if (BN == 128) { DVC_LAUNCH(128, 2); } else { DVC_LAUNCH(64, 2); }
  } else {
    if (BN == 256) { DVC_LAUNCH(256, 1); } else if (BN == 128) { DVC_LAUNCH(128, 1); } else { DVC_LAUNCH(64, 1); }
  }
#undef DVC_LAUNCH
  if (rc) return fail(rc == -1 ? "cudaFuncSetAttribute(max dynamic smem) failed" : "cudaLaunchKernelEx failed");
  launch_counter_add(1);
  return 0;
}

}  // namespace dvc
