// b200ot — column packing kernel (shared by the softmin and kernel-conv translation units).
#pragma once
#include "common.cuh"

namespace b200ot {

// -------------------------------------------------------------------------------------------------
// pack: (M, D) columns + per-column scalars -> colpack tiles (layout: common.cuh / ColFmt)
//   coordinates  direct ? -scale*(y - c) : +scale*(y - c)
//   slot D       additive exponent term:  h_scale*(h_a + h_scale_b*h_b)  (softmin, h_a != null)
//                plus, for the expansion form (direct == 0), the fold  -|Y|^2/2;
//                with h_a == null the slot holds the fold alone (gaussian conv) or is skipped (direct conv)
//   next slot    w_j (kernel-conv weight) when w != null
// Padding columns (j >= M) are neutral: coordinates 0, additive term -inf (softmin) / weight 0 (conv).
// Gather mode (src != null; ranges mode of the reductions): slot j holds column src[j] of the inputs, or a
// neutral padding column when src[j] < 0 — this is how clusters / batch elements are aligned to chunk
// boundaries without touching the caller's arrays.
// gate != null: the pack returns at once unless *gate is set (the recomputation of a paired softmin, softmin_pair.cuh).
// -------------------------------------------------------------------------------------------------
static __global__ void pack_cols_kernel(const float* __restrict__ y, const float* __restrict__ h_a,
                                        const float* __restrict__ h_b, float h_scale_b, float h_scale,
                                        const float* __restrict__ w, const float* __restrict__ center, float scale,
                                        int direct, int D, int nf2, int64_t M, int64_t Mpad,
                                        float* __restrict__ out, const int* __restrict__ src = nullptr,
                                        const int* __restrict__ gate = nullptr) {
  if (gate != nullptr && *gate == 0) return;
  const int64_t slot = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= Mpad) return;
  float* pk = out + (slot >> 1) * (int64_t)(nf2 * 2) + (slot & 1);
  int64_t j = slot;
  if (src != nullptr && slot < M) j = src[slot];
  if (slot >= M || j < 0) {
    for (int k = 0; k < nf2; ++k) pk[2 * k] = 0.f;
    if (h_a != nullptr) pk[2 * D] = -INFINITY;
    return;
  }
  float sq = 0.f;
  for (int k = 0; k < D; ++k) {
    const float c = center ? center[k] : 0.f;
    const float v = scale * (y[j * D + k] - c);
    sq = fmaf(v, v, sq);
    pk[2 * k] = direct ? -v : v;
  }
  float add = direct ? 0.f : -0.5f * sq;
  int f = D;  // next free float2 slot of the packet
  if (h_a != nullptr) {
    float h = h_a[j];
    if (h_b != nullptr) h = fmaf(h_scale_b, h_b[j], h);
    pk[2 * f++] = fmaf(h_scale, h, add);
  } else if (!direct) {
    pk[2 * f++] = add;
  }
  if (w != nullptr) pk[2 * f++] = w[j];
  for (; f < nf2; ++f) pk[2 * f] = 0.f;
}

}  // namespace b200ot
