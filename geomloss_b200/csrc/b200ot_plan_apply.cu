// b200ot — the transport plan applied to a value matrix in one reduction:
//     out[i, k] = r_i sum_j w_ij V[j, k],   w_ij = softmax_j(h_j - |x_i - y_j|^2 / (2 eps))
// (the barycentric map V = Y, colour / label / feature transport).  The reference applies its dense plan,
// `plan @ V` (src/geomloss/ot/_ot_result.py: plan_operator); here the pairs are visited once per slab of value
// columns and never stored.  D <= 8: planapply.cuh (CUDA cores); above, or where the softmin row gradient is routed
// to them: tcapply.cuh (tensor cores), whose K-slab kernel serves 64 < D <= B200OT_MAX_D_WIDE (b200ot_wide_plan_apply).
#include "b200ot.h"
#include "host_util.cuh"
#include "plan.cuh"
#include "planapply.cuh"
#include "tcconv.cuh"

#include <type_traits>

namespace b200ot {

// one thread per (row, value column of the slab)
__global__ void plan_apply_finalize_kernel(const float* __restrict__ part, int n_part, int nacc, int kv, int k0, int K,
                                           const float* __restrict__ vmax, const float* __restrict__ row_factor,
                                           float* __restrict__ out, int64_t N) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N * kv) return;
  const int64_t i = e / kv;
  const int k = (int)(e - i * kv);
  float sw = 0.f, a = 0.f;
  for (int s = 0; s < n_part; ++s) {
    const float* row = part + ((int64_t)s * N + i) * nacc;
    sw += row[0];
    a += row[1 + k];
  }
  // a row without any weight (every exponent underflowed against its lse2) gives 0, not 0/0
  float r = sw > 0.f ? a / sw : 0.f;
  if (vmax != nullptr) r /= tc_energy_coord_scale(vmax[k0 + k]);  // a power of two: exact
  if (row_factor != nullptr) r *= row_factor[i];
  out[i * K + k0 + k] = r;
}

int plan_apply_finalize(const float* part, int n_part, int nacc, int kv, int k0, int K, const float* vmax,
                        const float* row_factor, float* out, int64_t N, cudaStream_t st) {
  plan_apply_finalize_kernel<<<(unsigned)ceil_div64(N * kv, 256), 256, 0, st>>>(part, n_part, nacc, kv, k0, K, vmax,
                                                                              row_factor, out, N);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

// value columns per CUDA-core pass: 8, or 4 for the last (or only) slab when it has at most 4 columns
static int simt_slab(int K, int k0) { return K - k0 <= 4 ? 4 : 8; }

struct SimtApplyPlan {
  ReducePlan pl;
  int64_t off_vals, off_part, total;
};
static SimtApplyPlan make_simt_apply_plan(int64_t N, int64_t M, int D, int K) {
  SimtApplyPlan a;
  a.pl = make_plan(N, M, D);
  const int kvmax = simt_slab(K, 0);
  a.off_vals = round_up64(b200ot_packed_cols_floats(M, D, 1) * 4, 256);
  a.off_part = a.off_vals + round_up64(round_up64(M, kPackPad) * kvmax * 4, 256);
  a.total = a.off_part + round_up64((int64_t)a.pl.n_split * N * (1 + kvmax) * 4, 256);
  return a;
}

template <int D, int KV>
static int launch_apply(const ReducePlan& pl, cudaStream_t st, const float* x, const float* center, float scale,
                        const float* cols, const float* vals, const float* lse2, float* part, int64_t N) {
  if (pl.small) {
    using C = PlanApplyCfg<D, KV, kSmallR, kSmallNT, kSmallTJ, 4>;
    return launch_reduce<C>(plan_apply_partial_kernel<C>, pl, st, x, center, scale, cols, vals, lse2, part, N,
                            pl.ntiles, pl.tiles_per_split, pl.last_pairs);
  }
  // two rows per thread and two CTAs per SM while 2 x (1 + KV) accumulator pairs per row fit the registers
  // (D <= 4 with the 4-column slab); otherwise one row per thread, the same 512 rows per CTA
  using C = std::conditional_t<(D <= 4 && KV == 4), PlanApplyCfg<D, KV, kBigR, kBigNT, kBigTJ, 2>,
                               PlanApplyCfg<D, KV, 1, kBigR * kBigNT, kBigTJ, 1>>;
  return launch_reduce<C>(plan_apply_partial_kernel<C>, pl, st, x, center, scale, cols, vals, lse2, part, N, pl.ntiles,
                          pl.tiles_per_split, pl.last_pairs);
}

template <int KV>
static int launch_apply_d(int D, const ReducePlan& pl, cudaStream_t st, const float* x, const float* center,
                          float scale, const float* cols, const float* vals, const float* lse2, float* part,
                          int64_t N) {
  switch (D) {
    case 1: return launch_apply<1, KV>(pl, st, x, center, scale, cols, vals, lse2, part, N);
    case 2: return launch_apply<2, KV>(pl, st, x, center, scale, cols, vals, lse2, part, N);
    case 3: return launch_apply<3, KV>(pl, st, x, center, scale, cols, vals, lse2, part, N);
    case 4: return launch_apply<4, KV>(pl, st, x, center, scale, cols, vals, lse2, part, N);
    case 5: return launch_apply<5, KV>(pl, st, x, center, scale, cols, vals, lse2, part, N);
    case 6: return launch_apply<6, KV>(pl, st, x, center, scale, cols, vals, lse2, part, N);
    case 7: return launch_apply<7, KV>(pl, st, x, center, scale, cols, vals, lse2, part, N);
    case 8: return launch_apply<8, KV>(pl, st, x, center, scale, cols, vals, lse2, part, N);
    default: return B200OT_EINVAL;
  }
}

static int plan_apply_simt(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                           const float* center, const float* lse2, const float* v, const float* row_factor, float* out,
                           int64_t N, int64_t M, int D, int K, float eps, void* scratch, cudaStream_t st) {
  const SimtApplyPlan a = make_simt_apply_plan(N, M, D, K);
  char* base = reinterpret_cast<char*>(scratch);
  float* cols = reinterpret_cast<float*>(base);
  float* vals = reinterpret_cast<float*>(base + a.off_vals);
  float* part = reinterpret_cast<float*>(base + a.off_part);
  int rc = softmin_pack_impl(y, h_a, h_b, h_scale_b, center, M, D, 2, eps, cols, st, nullptr);
  if (rc) return rc;
  const float scale = softmin_coord_scale(2, eps);
  const int64_t mpad = round_up64(M, kPackPad);
  for (int k0 = 0; k0 < K;) {
    const int kvs = simt_slab(K, k0), kv = K - k0 < kvs ? K - k0 : kvs;
    pack_values_kernel<<<(unsigned)ceil_div64(mpad, 256), 256, 0, st>>>(v, M, mpad, K, k0, kvs, vals);
    B200OT_CUDA_TRY(cudaGetLastError());
    rc = kvs == 4 ? launch_apply_d<4>(D, a.pl, st, x, center, scale, cols, vals, lse2, part, N)
                  : launch_apply_d<8>(D, a.pl, st, x, center, scale, cols, vals, lse2, part, N);
    if (rc) return rc;
    rc = plan_apply_finalize(part, a.pl.n_split, 1 + kvs, kv, k0, K, nullptr, row_factor, out, N, st);
    if (rc) return rc;
    k0 += kvs;
  }
  return B200OT_OK;
}

static bool plan_apply_dims(int64_t N, int64_t M, int D, int64_t K) {
  return N > 0 && M > 0 && tc_capable_dim(D) && K >= 1 && K <= 0x7fffffff;
}

}  // namespace b200ot

using namespace b200ot;

extern "C" {

B200OT_API int64_t b200ot_plan_apply_scratch_bytes(int64_t N, int64_t M, int32_t D, int64_t K) {
  if (!plan_apply_dims(N, M, D, K)) return 0;
  if (tc_routed(kTcSoftminBwd, D, N, M)) return tc_plan_apply_scratch_bytes(N, M, D, (int)K);
  return make_simt_apply_plan(N, M, D, (int)K).total;
}

B200OT_API int b200ot_plan_apply(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                                 const float* center, const float* lse2, const float* v, const float* row_factor,
                                 float* out, int64_t N, int64_t M, int32_t D, int64_t K, int32_t p, float eps,
                                 void* scratch, int64_t scratch_bytes, void* stream) {
  if (!x || !y || !h_a || !lse2 || !v || !out || !scratch || !plan_apply_dims(N, M, D, K) || !valid_p(p) ||
      p_exponent(p) != 2 || !(eps > 0.f))
    return B200OT_EINVAL;
  if (((uintptr_t)scratch) & 15) return B200OT_EALIGN;
  if (scratch_bytes < b200ot_plan_apply_scratch_bytes(N, M, D, K)) return B200OT_ESCRATCH;
  cudaStream_t st = (cudaStream_t)stream;
  if (tc_routed(kTcSoftminBwd, D, N, M))
    return tc_plan_apply(x, y, h_a, h_b, h_scale_b, center, lse2, v, row_factor, out, N, M, D, (int)K, eps, scratch, st);
  return plan_apply_simt(x, y, h_a, h_b, h_scale_b, center, lse2, v, row_factor, out, N, M, D, (int)K, eps, scratch,
                         st);
}

}  // extern "C"
