// czt_inst.cu — instantiates czt_kernel for one transform size P = 2^B2L_LOG2M (compile with -DB2L_LOG2M=k).
#include "czt_kernel.cuh"
#include "internal.h"

#ifndef B2L_LOG2M
#error "compile with -DB2L_LOG2M=<5..12>"
#endif

namespace b2l {

#define B2L_CAT2(a, b) a##b
#define B2L_CAT(a, b) B2L_CAT2(a, b)

constexpr int L = B2L_LOG2M;
constexpr int P = 1 << L;
constexpr int TPF = P >= 32 ? P / 32 : 1;
constexpr int NW = L >= 10 ? 16 : (TPF > 16 ? 16 : TPF);   // HostFftCfg::czt_nw

CztKernel B2L_CAT(czt_kernel_, B2L_LOG2M)() { return czt_kernel<L, TPF, NW>; }
CztInvKernel B2L_CAT(czt_inv_kernel_, B2L_LOG2M)() { return czt_inv_kernel<L, TPF, NW>; }

}  // namespace b2l
