// inv_inst.cu — instantiates inv_kernel for one transform size (compile with -DB2L_LOG2M=k).
#include "inv_kernel.cuh"
#include "internal.h"

#ifndef B2L_LOG2M
#error "compile with -DB2L_LOG2M=<2..11>"
#endif

namespace b2l {
namespace {
template <class K>
cudaError_t run_op(K kern, int op, int nt, const InvArgs* a, int grid, size_t smem, cudaStream_t st, int* result) {
  if (op == OP_SET_SMEM) return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (op == OP_OCCUPANCY) return cudaOccupancyMaxActiveBlocksPerMultiprocessor(result, kern, nt, smem);
  kern<<<grid, nt, smem, st>>>(*a);
  return cudaGetLastError();
}
}  // namespace

#define B2L_CAT2(a, b) a##b
#define B2L_CAT(a, b) B2L_CAT2(a, b)

// `nw`: 16 or 8 warps; 116 = 16 warps as two independent 8-warp halves (DUAL).
template <int L>
cudaError_t inv_dispatch(int op, int nw, const InvArgs* a, int grid, size_t smem, cudaStream_t st, int* result) {
  constexpr int M = 1 << L;
  constexpr int TPF = M >= 32 ? M / 32 : 1;
  if constexpr (L >= 10) {
    if (nw == 16) return run_op(inv_kernel<L, TPF, 16, false>, op, 16 * 32, a, grid, smem, st, result);
    if (nw == 8) return run_op(inv_kernel<L, TPF, 8, false>, op, 8 * 32, a, grid, smem, st, result);
    if (nw == 116) return run_op(inv_kernel<L, TPF, 16, true>, op, 16 * 32, a, grid, smem, st, result);
  } else {
    constexpr int NW = TPF > 16 ? 16 : TPF;
    if (nw == NW) return run_op(inv_kernel<L, TPF, NW, false>, op, NW * 32, a, grid, smem, st, result);
    if constexpr (L == 9) {
      if (nw == 116) return run_op(inv_kernel<L, TPF, 16, true>, op, 16 * 32, a, grid, smem, st, result);
    }
  }
  return cudaErrorInvalidValue;
}

cudaError_t B2L_CAT(inv_op_, B2L_LOG2M)(int op, int nw, const InvArgs* a, int grid, size_t smem, cudaStream_t st,
                                         int* result) {
  return inv_dispatch<B2L_LOG2M>(op, nw, a, grid, smem, st, result);
}

}  // namespace b2l
