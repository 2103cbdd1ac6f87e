// b200ot — instantiations of the tensor-core kernels above D = 64 (tcwide.cuh), in a translation unit of their own so
// that they compile in parallel with b200ot_tc.cu.  The host side (plans, packs, finalizes, the b200ot_wide_* entries)
// is that of the other tensor-core operators, in b200ot_tc.cu.
#include "b200ot.h"
#include "host_util.cuh"
#include "tcwide.cuh"

namespace b200ot {

TcKernel tc_wide_kernel(int mode, bool bwd) {
  if (!bwd) {
    switch (mode) {
      case 0: return tc_wide_reduce_kernel<0>;
      case 1: return tc_wide_reduce_kernel<1>;
      case 4: return tc_wide_reduce_kernel<4>;
      case 5: return tc_wide_reduce_kernel<5>;
      case 6: return tc_wide_reduce_kernel<6>;
      default: return nullptr;
    }
  }
  switch (mode) {
    case 2: return tc_wide_bwd_kernel<2>;
    case 3: return tc_wide_bwd_kernel<3>;
    case 4: return tc_wide_bwd_kernel<4>;
    case 5: return tc_wide_bwd_kernel<5>;
    case 7: return tc_wide_bwd_kernel<7>;
    default: return nullptr;
  }
}

}  // namespace b200ot
