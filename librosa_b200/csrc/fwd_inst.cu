// fwd_inst.cu — instantiates fwd_kernel for one transform size (compile with -DB2L_LOG2M=k).
#include "fwd_kernel.cuh"
#include "internal.h"

#ifndef B2L_LOG2M
#error "compile with -DB2L_LOG2M=<2..12>"
#endif

namespace b2l {
namespace {

template <int L, int TPF, int NW, int DUAL>
FwdKernel by_mode(int mode) {
  switch (mode) {
    case MODE_STFT: return fwd_kernel<L, TPF, NW, MODE_STFT, DUAL>;
    case MODE_MEL: return fwd_kernel<L, TPF, NW, MODE_MEL, DUAL>;
    case MODE_SPEC: return fwd_kernel<L, TPF, NW, MODE_SPEC, DUAL>;
    case MODE_STATS: return fwd_kernel<L, TPF, NW, MODE_STATS, DUAL>;
  }
  return nullptr;
}

// `variant`: 16 or 8 warps; 116 = 16 warps as two independent 8-warp halves (NSPLIT = 2).
template <int L>
FwdKernel variant_kernel(int variant, int mode) {
  constexpr int M = 1 << L;
  constexpr int TPF = M >= 32 ? M / 32 : 1;
  if constexpr (L >= 10) {
    if (variant == 16) return by_mode<L, TPF, 16, 1>(mode);
    if (variant == 8) return by_mode<L, TPF, 8, 1>(mode);
    if (variant == 116) return by_mode<L, TPF, 16, 2>(mode);
  } else {
    constexpr int NW = TPF > 16 ? 16 : TPF;
    if (variant == NW) return by_mode<L, TPF, NW, 1>(mode);
    if constexpr (L == 9) {
      if (variant == 116) return by_mode<L, TPF, 16, 2>(mode);
    }
  }
  return nullptr;
}

}  // namespace

#define B2L_CAT2(a, b) a##b
#define B2L_CAT(a, b) B2L_CAT2(a, b)

FwdKernel B2L_CAT(fwd_kernel_, B2L_LOG2M)(int variant, int mode) { return variant_kernel<B2L_LOG2M>(variant, mode); }

}  // namespace b2l
