// Hopper tensor-core (wgmma) implementation of K7; see corr_tc.cu.
#pragma once
#include <string>

#include "dvc_internal.cuh"

namespace dvc {
// Operand planes and split partials of the correlation: owned by the context (one per device), grown only by
// corr_ws_reserve -- dvc_set_exemplar / dvc_exemplar_import pre-size it, so the frame loop never allocates.
struct CorrWorkspace {
  static constexpr int NBUF = 7;
  // A_hi, A_lo, B_hi, B_lo, split partials, screening norms, screening candidate lists
  void* buf[NBUF] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  size_t cap[NBUF] = {0, 0, 0, 0, 0, 0, 0};
  // the exemplar side is constant over a clip: its planes are split once per (pointer, version, format)
  const void* phi_src = nullptr;
  long long phi_version = -1;
  int phi_fmt = -1;
  size_t phi_elems = 0;
};
// reserve for B x NA query rows against Bphi x NB reference rows (any math mode, any split count); 0 on success
int corr_ws_reserve(CorrWorkspace* ws, int B, int Bphi, int NA, int NB);
void corr_ws_free(CorrWorkspace* ws);
// the 4 max cells of the screened path (float bits): [0, 1] query side, [2, 3] reference side (||dropped part||, ||hi
// part|| maxima); nullptr while the workspace is unallocated.  Debug / tests.
const unsigned int* corr_ws_screen_cells(const CorrWorkspace* ws);
// math = DVC_MATH_TF32X3 / BF16X3 / FP16X3.  Returns 0 on success, non-zero with *err set otherwise.
// cluster: 2 = 2-CTA clusters on adjacent query-row tiles sharing the multicast reference tile, 1 = single CTAs
// phi_version >= 0: the caller guarantees that p.phi's contents change only together with phi_version (the planes of
// the reference side are then reused across launches); < 0: split every launch
// screen != 0 (FP16X3, T <= 2e-10 only): one fp16 pass locates the candidates of every row's maximum within a rigorous error
// bound, which are then re-scored exactly in fp32 (corr_tc.cu); 0: the exact 3-pass kernel
int launch_corr_tc(const CorrParams& p, int math, int cluster, int screen, CorrWorkspace* ws, long long phi_version,
                   cudaStream_t s, std::string* err);
// cudaFuncSetAttribute is per device: true once per (kernel instantiation, device) -- `mask` is that kernel's static
bool first_use_on_device(unsigned long long* mask);
}  // namespace dvc
