// inv_inst.cu — instantiates inv_kernel for one transform size (compile with -DB2L_LOG2M=k).
#include "inv_kernel.cuh"
#include "internal.h"

#ifndef B2L_LOG2M
#error "compile with -DB2L_LOG2M=<2..12>"
#endif

namespace b2l {

#define B2L_CAT2(a, b) a##b
#define B2L_CAT(a, b) B2L_CAT2(a, b)

// `variant`: 16 or 8 warps; 116 = 16 warps as two independent 8-warp halves (DUAL).
namespace {
template <int L>
InvKernel variant_kernel(int variant) {
  constexpr int M = 1 << L;
  constexpr int TPF = M >= 32 ? M / 32 : 1;
  if constexpr (L >= 10) {
    if (variant == 16) return inv_kernel<L, TPF, 16, false>;
    if (variant == 8) return inv_kernel<L, TPF, 8, false>;
    if (variant == 116) return inv_kernel<L, TPF, 16, true>;
  } else {
    constexpr int NW = TPF > 16 ? 16 : TPF;
    if (variant == NW) return inv_kernel<L, TPF, NW, false>;
    if constexpr (L == 9) {
      if (variant == 116) return inv_kernel<L, TPF, 16, true>;
    }
  }
  return nullptr;
}
}  // namespace

InvKernel B2L_CAT(inv_kernel_, B2L_LOG2M)(int variant) { return variant_kernel<B2L_LOG2M>(variant); }

}  // namespace b2l
