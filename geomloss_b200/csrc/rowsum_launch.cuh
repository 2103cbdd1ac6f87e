// b200ot — launch helpers of rowsum_partial_kernel: the CTA shape of the plan and of D, the dense or the ranges
// instantiation.
#pragma once
#include "plan.cuh"
#include "rowsum.cuh"

#include <type_traits>

namespace b200ot {

template <class C>
inline int launch_rowsum_kernel(const ReducePlan& pl, cudaStream_t st, const float* x, const float* center,
                                float scale, float clampq, const float* cols, const float* lse2, float* part,
                                int64_t N, int ntiles, int tiles_per_split, const int4* seg, const int2* pieces) {
  if (seg != nullptr)
    return launch_reduce<C>(rowsum_partial_kernel<C, true>, pl, st, x, center, scale, clampq, cols, lse2, part, N,
                            ntiles, tiles_per_split, 0, seg, pieces);
  return launch_reduce<C>(rowsum_partial_kernel<C, false>, pl, st, x, center, scale, clampq, cols, lse2, part, N,
                          ntiles, tiles_per_split, pl.last_pairs, seg, pieces);
}

// lse2: the softmin row gradient's row term (null for the kernel convolutions)
template <int MODE, int D>
static int launch_rowsum(const ReducePlan& pl, cudaStream_t st, const float* x, const float* center, float scale,
                         float clampq, const float* cols, const float* lse2, float* part, int64_t N,
                         const int4* seg = nullptr, const int2* pieces = nullptr) {
  if (pl.small) {
    using C = RowSumCfg<MODE, D, kSmallR, kSmallNT, kSmallTJ, 3, 4>;
    return launch_rowsum_kernel<C>(pl, st, x, center, scale, clampq, cols, lse2, part, N, pl.ntiles,
                                   pl.tiles_per_split, seg, pieces);
  }
  // D >= 5: one row per thread (same 512 rows per CTA) keeps the 2 x (D+1) accumulator pairs in registers
  using C = std::conditional_t<(D <= 4), RowSumCfg<MODE, D, kBigR, kBigNT, kBigTJ, 3, 2>,
                               RowSumCfg<MODE, D, 1, kBigR * kBigNT, kBigTJ, 3, 1>>;
  return launch_rowsum_kernel<C>(pl, st, x, center, scale, clampq, cols, lse2, part, N, pl.ntiles, pl.tiles_per_split,
                                 seg, pieces);
}

template <int MODE>
static int launch_rowsum_d(int D, const ReducePlan& pl, cudaStream_t st, const float* x, const float* center,
                           float scale, float clampq, const float* cols, const float* lse2, float* part, int64_t N,
                           const int4* seg = nullptr, const int2* pieces = nullptr) {
  switch (D) {
    case 1: return launch_rowsum<MODE, 1>(pl, st, x, center, scale, clampq, cols, lse2, part, N, seg, pieces);
    case 2: return launch_rowsum<MODE, 2>(pl, st, x, center, scale, clampq, cols, lse2, part, N, seg, pieces);
    case 3: return launch_rowsum<MODE, 3>(pl, st, x, center, scale, clampq, cols, lse2, part, N, seg, pieces);
    case 4: return launch_rowsum<MODE, 4>(pl, st, x, center, scale, clampq, cols, lse2, part, N, seg, pieces);
    case 5: return launch_rowsum<MODE, 5>(pl, st, x, center, scale, clampq, cols, lse2, part, N, seg, pieces);
    case 6: return launch_rowsum<MODE, 6>(pl, st, x, center, scale, clampq, cols, lse2, part, N, seg, pieces);
    case 7: return launch_rowsum<MODE, 7>(pl, st, x, center, scale, clampq, cols, lse2, part, N, seg, pieces);
    case 8: return launch_rowsum<MODE, 8>(pl, st, x, center, scale, clampq, cols, lse2, part, N, seg, pieces);
    default: return B200OT_EINVAL;
  }
}

}  // namespace b200ot
