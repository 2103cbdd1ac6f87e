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

// Runs pack + partial reduction of the row-gradient pass and leaves *n_part sets of (N, D+1) sums in scratch at *part,
// each `*scale_out` times the softmax-weighted sums (kTcPScale on the tensor-core path, common.cuh; 1 otherwise).
static int softmin_bwd_partials(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                                const float* center, const float* lse2, int64_t N, int64_t M, int32_t D, int32_t p,
                                float eps, void* scratch, int64_t scratch_bytes, void* stream, float** part,
                                int* n_part, float* scale_out) {
  const bool tc = p_exponent(p) == 2 && tc_routed(kTcSoftminBwd, D, N, M);
  if (!x || !y || !h_a || !lse2 || !scratch || N <= 0 || M <= 0 || (!supported_simt_dim(D) && !tc) || !valid_p(p) ||
      !(eps > 0.f))
    return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, b200ot_softmin_scratch_bytes(N, M, D))) return rc;
  *scale_out = tc ? kTcPScale : 1.f;
  if (tc)
    return tc_softmin_bwd_sums(x, y, h_a, h_b, h_scale_b, center, lse2, N, M, D, p, eps, scratch, (cudaStream_t)stream,
                               part, n_part);
  const ReducePlan pl = make_plan(N, M, D);
  float* cols = reinterpret_cast<float*>(scratch);
  *part = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) +
                                   round_up64(b200ot_packed_cols_floats(M, D, 1) * 4, 256));
  *n_part = pl.n_split;
  int rc = softmin_pack_impl(y, h_a, h_b, h_scale_b, center, M, D, p, eps, cols, (cudaStream_t)stream, nullptr);
  if (rc) return rc;
  return b200ot_softmin_bwd_partial(x, center, cols, lse2, *part, pl.n_split, N, M, D, p, eps, stream);
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

}  // extern "C"
