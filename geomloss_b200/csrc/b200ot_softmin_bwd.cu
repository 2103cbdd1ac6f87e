// b200ot — softmin backward w.r.t. the row cloud.
// Reference semantics: autograd through  -eps * logsumexp_j(h_j - C(x_i, y_j)/eps)  with the columns and
// h detached (src/geomloss/_legacy/sinkhorn_samples.py:179-185, sinkhorn_divergence.py:612-623):
//     d out_i / d x_i = sum_j w_ij dC(x_i, y_j)/dx_i,   w_ij = softmax_j(h_j - C_ij/eps)
// p = 2:  dC/dx = x - y          ->  grad_x_i = go_i (x_i - sum_j w_ij y_j)
// p = 1:  dC/dx = (x - y)/|x-y|  (zero inside the 1e-8 clamp of utils.py:61)
// The weights are re-normalised by their own sum, so rounding of the saved lse2 cancels.
#include "b200ot.h"
#include "host_util.cuh"
#include "plan.cuh"
#include "rowsum.cuh"
#include "rowsum_launch.cuh"

#include <type_traits>

namespace b200ot {

// part: (n_split, N, D+1) with [0] = sum w, [1+k] = sum w Y_k (p=2, scaled centred coords) or sum w u_k (p=1)
__global__ void softmin_bwd_finalize_kernel(const float* __restrict__ part, int n_split, const float* __restrict__ x,
                                            const float* __restrict__ center, const float* __restrict__ grad_out,
                                            float* __restrict__ grad_x, int64_t N, int D, int p, float inv_scale) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int na = D + 1;
  float sw = 0.f;
  for (int s = 0; s < n_split; ++s) sw += part[((int64_t)s * N + i) * na];
  // a row whose (block-sparse) column list is empty has no weight at all: zero gradient, not 0/0
  const float inv = sw > 0.f ? 1.0f / sw : 0.f;
  const float go = grad_out[i];
  for (int k = 0; k < D; ++k) {
    float a = 0.f;
    for (int s = 0; s < n_split; ++s) a += part[((int64_t)s * N + i) * na + 1 + k];
    float g;
    if (p == 2) {
      const float c = center ? center[k] : 0.f;
      g = (x[i * D + k] - c) - a * inv * inv_scale;  // x - ybar, both relative to the centre
    } else {
      g = a * inv;
    }
    grad_x[i * D + k] = go * g;
  }
}

// merged[e] = scale * sum_s part[s * n_elems + e]
__global__ void rowsum_merge_kernel(const float* __restrict__ part, int n_part, float* __restrict__ merged,
                                    int64_t n_elems, float scale) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_elems) return;
  float a = 0.f;
  for (int s = 0; s < n_part; ++s) a += part[(int64_t)s * n_elems + e];
  merged[e] = scale * a;
}

static int rowsum_merge(const float* part, int n_part, int width, float* merged, int64_t N, float scale,
                        cudaStream_t st) {
  const int threads = 256;
  rowsum_merge_kernel<<<(unsigned)ceil_div64(N * width, threads), threads, 0, st>>>(part, n_part, merged, N * width,
                                                                                    scale);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

int softmin_bwd_finalize_tc(const float* part, int n_part, const float* x, const float* center, const float* grad_out,
                            float* grad_x, int64_t N, int D, float eps, cudaStream_t st) {
  softmin_bwd_finalize_kernel<<<(unsigned)ceil_div64(N, 256), 256, 0, st>>>(
      part, n_part, x, center, grad_out, grad_x, N, D, 2, 1.0f / softmin_coord_scale(2, eps));
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

template <int MODE, int D>
static int launch_rowsum(const ReducePlan& pl, cudaStream_t st, const float* x, const float* center, float scale,
                         float clampq, const float* cols, const float* lse2, float* part, int64_t N,
                         const int4* tile_ptr = nullptr, const int2* tile_list = nullptr) {
  if (pl.small) {
    using C = RowSumCfg<MODE, D, kSmallR, kSmallNT, kSmallTJ, 3, 4>;
    return launch_rowsum_kernel<C>(pl, st, x, center, scale, clampq, cols, lse2, part, N,
                            pl.ntiles, pl.tiles_per_split, tile_ptr, tile_list);
  }
  // D >= 5: one row per thread (same 512 rows per CTA) keeps the 2 x (D+1) accumulator pairs in registers
  using C = std::conditional_t<(D <= 4), RowSumCfg<MODE, D, kBigR, kBigNT, kBigTJ, 3, 2>,
                               RowSumCfg<MODE, D, 1, kBigR * kBigNT, kBigTJ, 3, 1>>;
  return launch_rowsum_kernel<C>(pl, st, x, center, scale, clampq, cols, lse2, part, N, pl.ntiles,
                          pl.tiles_per_split, tile_ptr, tile_list);
}

template <int MODE>
static int launch_rowsum_d(int D, const ReducePlan& pl, cudaStream_t st, const float* x, const float* center,
                           float scale, float clampq, const float* cols, const float* lse2, float* part,
                           int64_t N, const int4* seg = nullptr, const int2* pieces = nullptr) {
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

using namespace b200ot;

extern "C" {

B200OT_API int b200ot_rowsum_merge(const float* part, int32_t n_part, int32_t width, float* merged, int64_t N,
                                   void* stream) {
  if (!part || !merged || n_part <= 0 || width <= 0 || N <= 0) return B200OT_EINVAL;
  return rowsum_merge(part, n_part, width, merged, N, 1.f, (cudaStream_t)stream);
}

B200OT_API int b200ot_softmin_bwd_partial(const float* x, const float* center, const float* cols, const float* lse2,
                                          float* part, int32_t n_split, int64_t N, int64_t M, int32_t D, int32_t p,
                                          float eps, void* stream) {
  if (!x || !cols || !lse2 || !part || N <= 0 || M <= 0 || !supported_simt_dim(D) || !valid_p(p) ||
      !(eps > 0.f))
    return B200OT_EINVAL;
  if (((uintptr_t)cols) & 15) return B200OT_EALIGN;
  const ReducePlan pl = make_plan(N, M, D);
  if (n_split != pl.n_split) return B200OT_EINVAL;
  const int pe = p_exponent(p);
  const float scale = softmin_coord_scale(pe, eps);
  const float clampq = scale * scale * cost_clamp(p);
  cudaStream_t st = (cudaStream_t)stream;
  return (pe == 2) ? launch_rowsum_d<kSoftminBwdP2>(D, pl, st, x, center, scale, clampq, cols, lse2, part, N)
                   : launch_rowsum_d<kSoftminBwdP1>(D, pl, st, x, center, scale, clampq, cols, lse2, part, N);
}

B200OT_API int b200ot_softmin_bwd_partial_ranges(const float* x, const float* center, const float* cols,
                                                 const float* lse2, const b200ot_segment* seg, int64_t n_seg,
                                                 const b200ot_piece* pieces, float* part, int64_t N, int32_t D,
                                                 int32_t p, float eps, int32_t variant, void* stream) {
  if (!x || !cols || !lse2 || !seg || !pieces || !part || N <= 0 || n_seg <= 0 || n_seg > 0x7fffffff ||
      !supported_simt_dim(D) || !valid_p(p) || !(eps > 0.f) ||
      (variant != B200OT_RANGES_BIG && variant != B200OT_RANGES_SMALL))
    return B200OT_EINVAL;
  if ((((uintptr_t)cols) & 15) || (((uintptr_t)seg) & 15) || (((uintptr_t)pieces) & 7)) return B200OT_EALIGN;
  const ReducePlan pl = ranges_plan(variant, n_seg);
  const int pe = p_exponent(p);
  const float scale = softmin_coord_scale(pe, eps);
  const float clampq = scale * scale * cost_clamp(p);
  cudaStream_t st = (cudaStream_t)stream;
  const int4* sg = reinterpret_cast<const int4*>(seg);
  const int2* pc = reinterpret_cast<const int2*>(pieces);
  return (pe == 2) ? launch_rowsum_d<kSoftminBwdP2>(D, pl, st, x, center, scale, clampq, cols, lse2, part, N, sg, pc)
                   : launch_rowsum_d<kSoftminBwdP1>(D, pl, st, x, center, scale, clampq, cols, lse2, part, N, sg, pc);
}

B200OT_API int b200ot_softmin_bwd_finalize(const float* part, int32_t n_part, const float* x, const float* center,
                                           const float* grad_out, float* grad_x, int64_t N, int32_t D, int32_t p,
                                           float eps, void* stream) {
  if (!part || n_part <= 0 || !x || !grad_out || !grad_x || N <= 0 ||
      (!supported_simt_dim(D) && !(tc_capable_dim(D) && p_exponent(p) == 2)) || !valid_p(p) || !(eps > 0.f))
    return B200OT_EINVAL;
  const int threads = 256;
  softmin_bwd_finalize_kernel<<<(unsigned)ceil_div64(N, threads), threads, 0, (cudaStream_t)stream>>>(
      part, n_part, x, center, grad_out, grad_x, N, D, p_exponent(p), 1.0f / softmin_coord_scale(p_exponent(p), eps));
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

// Runs pack + partial reduction of the row-gradient pass and leaves n_part sets of (N, D+1) sums in scratch, each
// `*scale_out` times the softmax-weighted sums (kTcPScale on the tensor-core path, common.cuh; 1 otherwise).
static int softmin_bwd_partials(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                                const float* center, const float* lse2, int64_t N, int64_t M, int32_t D, int32_t p,
                                float eps, void* scratch, int64_t scratch_bytes, void* stream, float** part_out,
                                int* n_part_out, float* scale_out) {
  const bool tc = p_exponent(p) == 2 && tc_routed(kTcSoftminBwd, D, N, M);
  if (!x || !y || !h_a || !lse2 || !scratch || N <= 0 || M <= 0 || (!supported_simt_dim(D) && !tc) || !valid_p(p) ||
      !(eps > 0.f))
    return B200OT_EINVAL;
  if (((uintptr_t)scratch) & 15) return B200OT_EALIGN;
  if (scratch_bytes < b200ot_softmin_scratch_bytes(N, M, D)) return B200OT_ESCRATCH;
  *scale_out = tc ? kTcPScale : 1.f;
  if (tc)
    return bwd_partial_tc(3, x, y, nullptr, h_a, h_b, h_scale_b, lse2, center, softmin_coord_scale(2, eps), N, M, D,
                          scratch, part_out, n_part_out, (cudaStream_t)stream);
  const ReducePlan pl = make_plan(N, M, D);
  float* cols = reinterpret_cast<float*>(scratch);
  float* part = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) +
                                         round_up64(b200ot_packed_cols_floats(M, D, 1) * 4, 256));
  int rc = softmin_pack_impl(y, h_a, h_b, h_scale_b, center, M, D, p, eps, cols, (cudaStream_t)stream, nullptr);
  if (rc) return rc;
  rc = b200ot_softmin_bwd_partial(x, center, cols, lse2, part, pl.n_split, N, M, D, p, eps, stream);
  *part_out = part;
  *n_part_out = pl.n_split;
  return rc;
}

B200OT_API int b200ot_softmin_bwd_sums(const float* x, const float* y, const float* h_a, const float* h_b,
                                       float h_scale_b, const float* center, const float* lse2, float* sums,
                                       int64_t N, int64_t M, int32_t D, int32_t p, float eps, void* scratch,
                                       int64_t scratch_bytes, void* stream) {
  if (!sums) return B200OT_EINVAL;
  float* part = nullptr;
  int n_part = 0;
  float p_scale = 1.f;
  const int rc = softmin_bwd_partials(x, y, h_a, h_b, h_scale_b, center, lse2, N, M, D, p, eps, scratch,
                                      scratch_bytes, stream, &part, &n_part, &p_scale);
  if (rc) return rc;
  // raw sums leave the library (the multi-GPU engine adds them over the column shards): undo the P scale here
  return rowsum_merge(part, n_part, D + 1, sums, N, 1.f / p_scale, (cudaStream_t)stream);
}

B200OT_API int b200ot_softmin_bwd_x(const float* x, const float* y, const float* h_a, const float* h_b,
                                    float h_scale_b, const float* center, const float* lse2, const float* grad_out,
                                    float* grad_x, int64_t N, int64_t M, int32_t D, int32_t p, float eps,
                                    void* scratch, int64_t scratch_bytes, void* stream) {
  if (!grad_out || !grad_x) return B200OT_EINVAL;
  float* part = nullptr;
  int n_part = 0;
  float p_scale = 1.f;  // cancels: the finalize divides by the row sum of P
  const int rc = softmin_bwd_partials(x, y, h_a, h_b, h_scale_b, center, lse2, N, M, D, p, eps, scratch,
                                      scratch_bytes, stream, &part, &n_part, &p_scale);
  if (rc) return rc;
  return b200ot_softmin_bwd_finalize(part, n_part, x, center, grad_out, grad_x, N, D, p, eps, stream);
}

B200OT_API int b200ot_softmin_bwd_x_batched(const float* x, const float* y, const float* h_a, const float* h_b,
                                            float h_scale_b, const float* center, const float* lse2,
                                            const float* grad_out, float* grad_x, int64_t B, int64_t N, int64_t M,
                                            int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                            void* stream) {
  if (!x || !y || !h_a || !lse2 || !grad_out || !grad_x || !scratch || !tc_batched_dims(B, N, M, D) || !valid_p(p) ||
      p_exponent(p) != 2 || !(eps > 0.f))
    return B200OT_EINVAL;
  if (((uintptr_t)scratch) & 15) return B200OT_EALIGN;
  if (scratch_bytes < b200ot_batched_scratch_bytes(B, N, M, D)) return B200OT_ESCRATCH;
  float* part = nullptr;
  int n_part = 0;
  // P carries kTcPScale, which cancels: the finalize divides by each row's sum of P
  const int rc = bwd_partial_tc(3, x, y, nullptr, h_a, h_b, h_scale_b, lse2, center, softmin_coord_scale(2, eps), N, M,
                                D, scratch, &part, &n_part, (cudaStream_t)stream, B, true);
  if (rc) return rc;
  return b200ot_softmin_bwd_finalize(part, n_part, x, center, grad_out, grad_x, B * N, D, p, eps, stream);
}

B200OT_API int b200ot_softmin_l1_bwd_x(const float* x, const float* y, const float* h_a, const float* h_b,
                                       float h_scale_b, const float* center, const float* lse2, const float* grad_out,
                                       float* grad_x, int64_t B, int64_t N, int64_t M, int32_t D, int32_t p, float eps,
                                       void* scratch, int64_t scratch_bytes, void* stream) {
  if (!x || !y || !h_a || !lse2 || !grad_out || !grad_x || !scratch || !tc_l1_args(B, N, M, D, p) || !(eps > 0.f))
    return B200OT_EINVAL;
  if (((uintptr_t)scratch) & 15) return B200OT_EALIGN;
  if (scratch_bytes < b200ot_softmin_l1_scratch_bytes(B, N, M, D)) return B200OT_ESCRATCH;
  float* part = nullptr;
  int n_part = 0;
  const float* coord_absmax = nullptr;
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = softmin_l1_tc(true, x, y, h_a, h_b, h_scale_b, center, lse2, B, N, M, D, p, eps, scratch, &part,
                               &n_part, &coord_absmax, st);
  if (rc) return rc;
  return softmin_l1_bwd_finalize(part, n_part, x, center, grad_out, grad_x, B * N, D, coord_absmax, st);
}

B200OT_API int b200ot_softmin_bwd_x_blocks(const float* x, const float* y, const float* h_a, const float* h_b,
                                           float h_scale_b, const float* center, const float* lse2,
                                           const float* grad_out, float* grad_x, int64_t N, const int32_t* row_src,
                                           int64_t n_row_slots, const int32_t* col_src, int64_t n_col_slots,
                                           const b200ot_segment* seg, int64_t n_seg, const b200ot_piece* pieces,
                                           int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                           void* stream) {
  if (!x || !y || !h_a || !lse2 || !grad_out || !grad_x || !row_src || !col_src || !scratch) return B200OT_EINVAL;
  int max_tiles = 0;
  int64_t n_pieces = 0;
  const int rc =
      blocks_check(N, n_row_slots, n_col_slots, seg, n_seg, pieces, D, p, eps, scratch, &max_tiles, &n_pieces);
  if (rc) return rc;
  if (scratch_bytes < tc_blocks_scratch_bytes(N, n_row_slots, n_col_slots, n_seg, n_pieces, max_tiles, D))
    return B200OT_ESCRATCH;
  float* part = nullptr;
  int n_part = 0;
  // P carries kTcPScale, which cancels: the finalize divides by each row's sum of P
  const int rc2 = softmin_blocks_tc(true, x, y, h_a, h_b, h_scale_b, center, lse2, N, row_src, n_row_slots, col_src,
                                    n_col_slots, seg, n_seg, pieces, n_pieces, max_tiles, D, eps, scratch, &part,
                                    &n_part, (cudaStream_t)stream);
  if (rc2) return rc2;
  return b200ot_softmin_bwd_finalize(part, n_part, x, center, grad_out, grad_x, N, D, p, eps, stream);
}

}  // extern "C"
