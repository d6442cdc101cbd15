// Hopper tensor-core (wgmma) convolution engine; see conv_tc.cu.
#pragma once
#include <string>

#include "dvc_internal.cuh"

namespace dvc {

struct ConvTcParams {
  int Hp, Wp, P, H, W, Cin;  // input planes: padded NHWC, Cin a multiple of 32
  int Mtot;                  // B * Hp * Wp
  int taps, stride;          // taps: number of row-shifted operands (9 for 3x3, 1 for 1x1, 4 for an up-sampling phase)
  int tap_off[9];            // their offsets in padded input pixels
  int oscale, oa, ob;        // output pixel = (y / stride) * oscale + oa, (x / stride) * oscale + ob
  int Cout, CoutPad;         // CoutPad: multiple of the channel tile (weights are zero beyond Cout)
  const float* bias;
  float* y;      // destination: fp32 plane, or the hi plane when y_lo != nullptr
  float* y_lo;
  int yHp, yWp, yP, yC, yCoff;
  const float* add;     // optional skip addend (fp32, or hi plane when add_lo != nullptr)
  const float* add_lo;
  int aHp, aWp, aP, aC;
  int act;
  float slope;
  double* stats;  // optional [B][Cout][2]
  int f16;          // operands are fp16 hi/lo planes (else tf32 planes stored as fp32 words)
  float out_scale;  // fp16 mode: 2^-(e_x + e_w), undoes the exact power-of-two operand scales
  DynOut dyn;       // fp16 mode: device-side scales (dyn.cell_in: the input exponent is added to out_scale's on the
                    // device; dyn.h16: store fp16 planes with a derived exponent; dyn.cell_out: record max |output|)
  // fused tail of ColorVidNet (ColorVidNet.py:143-144): out[b][c][y][x] = 128 * tanh(sum_ch v[ch] * fin_w[c][ch] + fin_b[c]),
  // c = 0, 1, computed from the activated outputs instead of storing them (needs Cout == 128 == the channel tile)
  const float* fin_w;
  const float* fin_b;
  float* fin_out;
  int mt0, mtn;   // range [mt0, mt0 + mtn) of 128-pixel blocks of this launch (mtn = 0: all pixels)
  int force_bn;   // channel tile of this launch (0: chosen by the launcher)
  int tail;       // 1: a two-round 256-channel launch runs its last partial round with 128-channel tiles (see launcher);
                  // > 1 (tests): same, pretending the GPU has `tail` cluster slots
  int splits;     // split-K factor S (1 = off); needs ws / flags below
  float* ws;      // [tiles][BN][128] fp32 partial totals
  int* flags;     // [tiles], value epoch*16 + (splits completed)
  int epoch;      // unique per launch sharing `flags`
  int kbytes;     // bytes of K per pipeline stage: 64 (SWIZZLE_64B, twice the stages) or 128 (SWIZZLE_128B)
  int cluster;    // 2: run as 2-CTA clusters with TMA-multicast weight tiles; 1: single CTAs
  int kc;         // 128-byte k-blocks summed in the wgmma accumulators before promotion to the fp32 register totals
  int passes;     // MMAs per product: 3 (lo.hi + hi.lo + hi.hi, fp32-class) or 1 (hi.hi only: DVC_MATH_FP16X1)
  int rowshare;   // 1 / 2: the taps of one kernel row share one activation tile in shared memory (conv_tc.cu: CfgRS); 2 also
                  // sets the descriptors' base-offset field to the row shift; 0: one activation tile per tap
  int rs_ntx, rs_base_offset;  // filled by the launcher
  int dbg;        // timing experiments (results are WRONG when set): 1 = row-shared taps without the row shift, 2 = no activation lo plane
};

int conv_tc_pick_bn(int cout);  // channel tile (64 / 128 / 256) used for `cout` output channels
// x_hi/x_lo: activation planes [Mtot][Cin]; w_hi/w_lo: weight planes [taps][CoutPad][Cin] (tf32-rounded fp32 words)
// *variant receives the channel tile chosen (64 / 128 / 256)
int launch_conv_tc(const ConvTcParams& p, const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, int num_sms,
                   cudaStream_t s, std::string* err, int* variant = nullptr);

}  // namespace dvc
