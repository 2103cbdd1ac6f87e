// b200ot — work decomposition shared by every N x M reduction kernel (softmin, its backward,
// kernel convolutions): which tile shape, how many column splits.
#pragma once
#include <stdlib.h>

#include "host_util.cuh"

namespace b200ot {

// Tile shapes (must match the Cfg instantiations in the .cu files):
//   big   : 512 rows (256 consumer threads x 2 rows; the dense D = 3 softmin: 128 x 4), 1024-column tiles
//   small : 128 consumer threads x 1 row,   256-column tiles  — a few thousand points still spread
//           over every SM (132 on an H100 SXM)
constexpr int kBigNT = 256, kBigR = 2, kBigTJ = 1024;
constexpr int kSmallNT = 128, kSmallR = 1, kSmallTJ = 256;
constexpr int kPackPad = 1024;  // packed column buffers are padded to this many columns
constexpr int kPlanWaves = 16;  // waves (counted as 2 CTAs/SM) a launch is cut into when the problem is large enough

struct ReducePlan {
  int tj;        // columns per tile
  int rows_cta;  // rows per CTA
  int ntiles;
  int last_pairs;  // column pairs the consumers visit in the LAST tile (dense mode): M rounded up to kTailAlign, not to tj
  int tiles_per_split;
  int n_split;
  int64_t row_tiles;
  bool small;
};

// Pure function of (N, M, D) and the SM count, so that the scratch-size query, the pack stage and the
// reduction stage of the C ABI always agree.
//
// Column splits: as FEW as fill the machine for ~16 waves of 2 CTAs/SM (the SM count is read from the device).  A
// partial last wave costs little once the CTAs drift out of lock-step, while every extra CTA costs its prologue and a
// cold TMA ring — which matters most on the short column shards of the multi-GPU engine.
// consumers visit whole chunks: 32 columns = 16 column pairs.  The D = 3, 4 softmin runs 32-pair chunks and may read up
// to 16 pairs past last_pairs — neutral padding of the same tile, which the producer always loads whole
constexpr int kTailAlign = 32;

// Test hook ($B200OT_FORCE_SPLITS, tools/sanitize_smoke.py and the streaming tests): force the number of column splits of
// both the dense plan below and the tensor-core plan (make_tc_plan), e.g. 1 so that one CTA streams every column tile
// of a small problem and re-uses each stage of its ring many times.  Read on every call, like $B200OT_TC_MIN_D; the
// scratch query and the launch call the same plan function, so they stay consistent.  0 / unset: the default plan.
inline int forced_splits() {
  const char* e = getenv("B200OT_FORCE_SPLITS");
  return e ? atoi(e) : 0;
}

inline ReducePlan make_plan(int64_t N, int64_t M, int D = 3) {
  (void)D;
  ReducePlan p;
  const int big_rows = kBigNT * kBigR;
  p.small = (N < 8 * (int64_t)big_rows) || (M < 4 * kBigTJ);
  p.tj = p.small ? kSmallTJ : kBigTJ;
  p.rows_cta = p.small ? kSmallNT * kSmallR : big_rows;
  p.ntiles = (int)(round_up64(M, p.tj) / p.tj);
  // the packed buffer is padded with neutral columns up to a whole tile and the TMA producer always moves whole tiles,
  // but the consumers stop at the chunk that holds column M-1: on a 125 000-column shard that is 96 instead of 1024
  // columns in the 123rd tile (0.7 % of the kernel)
  p.last_pairs = M > 0 ? (int)(round_up64(M - (int64_t)(p.ntiles - 1) * p.tj, kTailAlign) / 2) : 0;
  p.row_tiles = ceil_div64(N, p.rows_cta);
  const int64_t target_ctas = (int64_t)num_sms() * 2 * kPlanWaves;
  int64_t want = ceil_div64(target_ctas, p.row_tiles);
  const int forced = forced_splits();
  if (forced > 0) want = forced;
  if (want < 1) want = 1;
  if (want > 64) want = 64;
  if (want > p.ntiles) want = p.ntiles;
  p.tiles_per_split = (int)ceil_div64(p.ntiles, want);
  p.n_split = (int)ceil_div64(p.ntiles, p.tiles_per_split);
  return p;
}

// Ranges mode (block-sparse / batched problems): one CTA per row segment, one column split, the pieces of a
// segment are at most one tile wide and aligned to kRangesAlign columns (a whole number of chunks of either
// tile shape: 2 * CH = 16 columns for the big shape, 8 for the small one).
constexpr int kRangesAlign = 16;
inline ReducePlan ranges_plan(int variant, int64_t n_seg) {
  ReducePlan p;
  p.small = (variant == B200OT_RANGES_SMALL);
  p.tj = p.small ? kSmallTJ : kBigTJ;
  p.rows_cta = p.small ? kSmallNT * kSmallR : kBigNT * kBigR;
  p.ntiles = 0;
  p.last_pairs = 0;
  p.tiles_per_split = 0;
  p.n_split = 1;
  p.row_tiles = n_seg;
  return p;
}

// Launch one instantiation of a partial-reduction kernel with its dynamic shared memory opt-in.
template <class C, class Kern, class... Args>
inline int launch_reduce(Kern kern, const ReducePlan& pl, cudaStream_t st, Args... args) {
  // the opt-in is per (kernel, device): set it once per device a process drives, not on every launch.  The cache is
  // keyed by the kernel's address — the dense and the ranges instantiation of one Cfg share this function template
  // instance (same pointer type), not the attribute.
  static const void* done[64][4] = {};
  int dev = -1;
  const void* key = reinterpret_cast<const void*>(kern);
  bool known = false;
  if (cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < 64)
    for (int s = 0; s < 4; ++s) known = known || (done[dev][s] == key);
  if (!known) {
    B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    if (dev >= 0 && dev < 64)
      for (int s = 0; s < 4; ++s)
        if (done[dev][s] == nullptr) {
          done[dev][s] = key;
          break;
        }
  }
  dim3 grid((unsigned)pl.row_tiles, (unsigned)pl.n_split);
  kern<<<grid, C::NT + 32, C::SMEM_BYTES, st>>>(args...);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

}  // namespace b200ot
