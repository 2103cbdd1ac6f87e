// b200ot — kernel convolutions  out_i = sum_j k(x_i, y_j) w_j  and their row gradients.
// Reference semantics: the matvecs of kernel_loss (src/geomloss/_legacy/kernel_samples.py:116-137) with
//   gaussian  k = exp(-|x/s - y/s|^2 / 2)                    (kernel_samples.py:62-68)
//   laplacian k = exp(-sqrt(max(|x/s - y/s|^2, 1e-8)))       (kernel_samples.py:71-77, utils.py:56-61)
//   energy    k = -sqrt(max(|x - y|^2, 1e-8))                (kernel_samples.py:80-82)
// evaluated on the fly (never as an N x M matrix) by rowsum_partial_kernel, or on the tensor cores (b200ot_tc.cu) above
// D = 8 and wherever tc_routed sends the gaussian.
#include "b200ot.h"
#include "conv_kind.cuh"
#include "host_util.cuh"
#include "pack.cuh"
#include "plan.cuh"
#include "rowsum.cuh"
#include "rowsum_launch.cuh"
#include "tcconv.cuh"  // tc_energy_coord_scale, which the finalize kernels undo for the tensor-core energy kernel

#include <algorithm>

namespace b200ot {

// coord_absmax (tensor-core energy kernel): the sums are in coordinates scaled by tc_energy_coord_scale, undone here
__global__ void conv_fwd_finalize_kernel(const float* __restrict__ part, int n_split, float sign,
                                         float* __restrict__ out, int64_t N,
                                         const float* __restrict__ coord_absmax = nullptr) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float a = 0.f;
  for (int s = 0; s < n_split; ++s) a += part[(int64_t)s * N + i];
  if (coord_absmax != nullptr) a /= tc_energy_coord_scale(*coord_absmax);  // a power of two: exact
  out[i] = sign * a;
}

// gaussian: part (n_split, N, D+1): [0] = sum W e, [1+k] = sum W e Y_k   -> go (accY - X acc0) / (scale blur^2)
// laplacian / energy: part (n_split, N, D): sum W e u_k                    -> -go acc / blur   (energy: -go acc)
// (the tensor-core laplacian / energy sums have the gaussian's layout and are finalized as kind 0; coord_absmax: the
// energy kernel's coordinate scale, applied to X as the kernel applied it to the clouds; n_per > 0: a batch of elements
// of n_per rows each, whose weights were normalised per element, w_absmax[i / n_per])
__global__ void conv_bwd_finalize_kernel(const float* __restrict__ part, int n_split, const float* __restrict__ x,
                                         const float* __restrict__ center, const float* __restrict__ grad_out,
                                         float* __restrict__ grad_x, int64_t N, int D, int kind, float scale,
                                         float coef, const float* __restrict__ w_absmax,
                                         float* __restrict__ value_out = nullptr,
                                         const float* __restrict__ coord_absmax = nullptr, int64_t n_per = 0) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (coord_absmax != nullptr) scale *= tc_energy_coord_scale(*coord_absmax);
  float go = grad_out ? grad_out[i] : 1.f;  // no upstream gradient: the unit row gradient (value + gradient pass)
  float wmax = 1.f;
  // tensor-core path: the weights were normalised to max|w| = kTcPScale (tc_pack_kernel); all-zero weights leave
  // all-zero sums
  const float wa = w_absmax != nullptr ? w_absmax[n_per > 0 ? i / n_per : 0] : 0.f;
  if (wa > 0.f) wmax = wa / kTcPScale;
  go *= wmax;
  if (kind == B200OT_KERNEL_GAUSSIAN) {
    const int na = D + 1;
    float a0 = 0.f;
    for (int s = 0; s < n_split; ++s) a0 += part[((int64_t)s * N + i) * na];
    if (value_out) value_out[i] = wmax * a0;  // sum_j w_j k_ij: the forward value comes with the gradient sums
    for (int k = 0; k < D; ++k) {
      float a = 0.f;
      for (int s = 0; s < n_split; ++s) a += part[((int64_t)s * N + i) * na + 1 + k];
      const float c = center ? center[k] : 0.f;
      const float X = scale * (x[i * D + k] - c);
      grad_x[i * D + k] = go * coef * (a - X * a0);
    }
  } else {
    for (int k = 0; k < D; ++k) {
      float a = 0.f;
      for (int s = 0; s < n_split; ++s) a += part[((int64_t)s * N + i) * D + k];
      grad_x[i * D + k] = go * coef * a;
    }
  }
}

int conv_fwd_finalize(const float* part, int n_part, int kind, float* out, int64_t N, const float* coord_absmax,
                      cudaStream_t st) {
  conv_fwd_finalize_kernel<<<(unsigned)ceil_div64(N, 256), 256, 0, st>>>(
      part, n_part, kind_base(kind) == B200OT_KERNEL_ENERGY ? -1.f : 1.f, out, N, coord_absmax);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

int conv_bwd_finalize(const float* part, int n_part, const float* x, const float* center, const float* grad_out,
                      float* grad_x, int64_t N, int D, int kind, float scale, float coef, const float* w_absmax,
                      float* value_out, const float* coord_absmax, int64_t n_per, cudaStream_t st) {
  conv_bwd_finalize_kernel<<<(unsigned)ceil_div64(N, 256), 256, 0, st>>>(
      part, n_part, x, center, grad_out, grad_x, N, D, kind, scale, coef, w_absmax, value_out, coord_absmax, n_per);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

static int conv_pack(const float* y, const float* w, const float* center, int64_t M, int D, const ConvScales& cs,
                     float* cols, cudaStream_t st, const int* src = nullptr) {
  const int nf2 = colfmt_nf2(D, cs.extra);
  const int64_t mpad = round_up64(M, kPackPad);
  const int threads = 256;
  pack_cols_kernel<<<(unsigned)ceil_div64(mpad, threads), threads, 0, st>>>(
      y, nullptr, nullptr, 0.f, 0.f, w, center, cs.scale, cs.direct, D, nf2, M, mpad, cols, src);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

// the N x M launch of a CUDA-core kernel convolution (dense plan, or ranges when seg != null)
static int conv_partial(int kind_flags, bool bwd, const ReducePlan& pl, cudaStream_t st, const float* x,
                        const float* center, const ConvScales& cs, const float* cols, float* part, int64_t N, int D,
                        const int4* seg = nullptr, const int2* pieces = nullptr) {
  const int kind = kind_base(kind_flags);
  const float s = cs.scale, c = cs.clampq;
  if (kind == B200OT_KERNEL_GAUSSIAN)
    return bwd ? launch_rowsum_d<kGaussBwd>(D, pl, st, x, center, s, c, cols, nullptr, part, N, seg, pieces)
               : launch_rowsum_d<kGaussFwd>(D, pl, st, x, center, s, c, cols, nullptr, part, N, seg, pieces);
  if (kind == B200OT_KERNEL_LAPLACIAN)
    return bwd ? launch_rowsum_d<kLaplaceBwd>(D, pl, st, x, center, s, c, cols, nullptr, part, N, seg, pieces)
               : launch_rowsum_d<kLaplaceFwd>(D, pl, st, x, center, s, c, cols, nullptr, part, N, seg, pieces);
  return bwd ? launch_rowsum_d<kEnergyBwd>(D, pl, st, x, center, s, c, cols, nullptr, part, N, seg, pieces)
             : launch_rowsum_d<kEnergyFwd>(D, pl, st, x, center, s, c, cols, nullptr, part, N, seg, pieces);
}

static float conv_bwd_coef(int kind_flags, const ConvScales& cs, float blur) {
  const int kind = kind_base(kind_flags);
  if (kind == B200OT_KERNEL_GAUSSIAN) return 1.0f / (cs.scale * blur * blur);
  if (kind == B200OT_KERNEL_LAPLACIAN) return -1.0f / blur;
  return -1.0f;
}

}  // namespace b200ot

using namespace b200ot;

extern "C" {

B200OT_API int64_t b200ot_kernel_conv_scratch_bytes(int64_t N, int64_t M, int32_t D) {
  if (N <= 0 || M <= 0 || D <= 0) return 0;
  if (D > B200OT_MAX_D) return tc_capable_dim(D) ? tc_scratch_bytes(N, M, D) : 0;
  const ReducePlan pl = make_plan(N, M, D);
  const int64_t cols = b200ot_packed_cols_floats(M, D, 2) * 4;
  const int64_t part = (int64_t)pl.n_split * N * 4 * (D + 1);
  const int64_t simt = round_up64(cols, 256) + round_up64(part, 256);
  // (one size for every operator of the shape: the caller does not say which one it is about to run)
  return tc_any_routed(D, N, M) ? std::max(simt, tc_scratch_bytes(N, M, D)) : simt;
}

B200OT_API int b200ot_kernel_conv_finalize(const float* part, int32_t n_part, float* out, int64_t N, int32_t kind,
                                           void* stream) {
  if (!part || !out || n_part <= 0 || N <= 0 || !valid_kind(kind)) return B200OT_EINVAL;
  return conv_fwd_finalize(part, n_part, kind, out, N, nullptr, (cudaStream_t)stream);
}

B200OT_API int b200ot_kernel_conv_bwd_finalize(const float* part, int32_t n_part, const float* x, const float* center,
                                               const float* grad_out, float* grad_x, int64_t N, int32_t D,
                                               int32_t kind, float blur, void* stream) {
  if (!part || !x || !grad_out || !grad_x || n_part <= 0 || N <= 0 || !supported_simt_dim(D) || !valid_kind(kind))
    return B200OT_EINVAL;
  if (!blur_ok(kind, blur)) return B200OT_EINVAL;
  const ConvScales cs = conv_scales(kind, blur);
  return conv_bwd_finalize(part, n_part, x, center, grad_out, grad_x, N, D, kind_base(kind), cs.scale,
                           conv_bwd_coef(kind, cs, blur), nullptr, nullptr, nullptr, 0, (cudaStream_t)stream);
}

B200OT_API int b200ot_kernel_conv_pack_gather(const float* y, const float* w, const float* center,
                                              const int32_t* src_index, int64_t n_slots, int32_t D, int32_t kind,
                                              float blur, float* cols_out, void* stream) {
  if (!y || !w || !src_index || !cols_out || n_slots <= 0 || !supported_simt_dim(D) || !valid_kind(kind))
    return B200OT_EINVAL;
  if (!blur_ok(kind, blur)) return B200OT_EINVAL;
  if (((uintptr_t)cols_out) & 15) return B200OT_EALIGN;
  return conv_pack(y, w, center, n_slots, D, conv_scales(kind, blur), cols_out, (cudaStream_t)stream,
                   reinterpret_cast<const int*>(src_index));
}

// part: (N) sums (forward) or (N, width) sums (row gradients: width = D + 1 gaussian, D otherwise)
B200OT_API int b200ot_kernel_conv_partial_ranges(const float* x, const float* center, const float* cols,
                                                 const b200ot_segment* seg, int64_t n_seg,
                                                 const b200ot_piece* pieces, float* part, int64_t N, int32_t D,
                                                 int32_t kind, float blur, int32_t backward, int32_t variant,
                                                 void* stream) {
  if (!x || !cols || !seg || !pieces || !part || N <= 0 || n_seg <= 0 || n_seg > 0x7fffffff ||
      !supported_simt_dim(D) || !valid_kind(kind) ||
      (variant != B200OT_RANGES_BIG && variant != B200OT_RANGES_SMALL))
    return B200OT_EINVAL;
  if (!blur_ok(kind, blur)) return B200OT_EINVAL;
  if ((((uintptr_t)cols) & 15) || (((uintptr_t)seg) & 15) || (((uintptr_t)pieces) & 7)) return B200OT_EALIGN;
  return conv_partial(kind, backward != 0, ranges_plan(variant, n_seg), (cudaStream_t)stream, x, center,
                      conv_scales(kind, blur), cols, part, N, D, reinterpret_cast<const int4*>(seg),
                      reinterpret_cast<const int2*>(pieces));
}

// The kernel convolution of one problem.  Laplacian / energy: the tensor cores serve 8 < D <= 64 only (no measured
// cross-over below).
B200OT_API int b200ot_kernel_conv_fwd(const float* x, const float* y, const float* w, const float* center,
                                      float* out, int64_t N, int64_t M, int32_t D, int32_t kind, float blur,
                                      void* scratch, int64_t scratch_bytes, void* stream) {
  const bool tc = (kind_base(kind) == B200OT_KERNEL_GAUSSIAN) ? tc_routed(kTcConvFwd, D, N, M)
                                                              : (D > B200OT_MAX_D && tc_capable_dim(D));
  if (!x || !y || !w || !out || !scratch || N <= 0 || M <= 0 || !(supported_simt_dim(D) || tc) || !valid_kind(kind))
    return B200OT_EINVAL;
  if (!blur_ok(kind, blur)) return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, b200ot_kernel_conv_scratch_bytes(N, M, D))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (tc) return tc_kernel_conv(false, kind, x, y, w, center, nullptr, out, nullptr, N, M, D, blur, scratch, st);
  const ReducePlan pl = make_plan(N, M, D);
  const ConvScales cs = conv_scales(kind, blur);
  float* cols = reinterpret_cast<float*>(scratch);
  float* part = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) +
                                         round_up64(b200ot_packed_cols_floats(M, D, 2) * 4, 256));
  int rc = conv_pack(y, w, center, M, D, cs, cols, st);
  if (rc) return rc;
  rc = conv_partial(kind, false, pl, st, x, center, cs, cols, part, N, D);
  if (rc) return rc;
  return b200ot_kernel_conv_finalize(part, pl.n_split, out, N, kind, stream);
}

// Row gradients (and, with value_out, the forward values from the same pass: gaussian only), as b200ot_kernel_conv_fwd.
static int conv_bwd_x_impl(const float* x, const float* y, const float* w, const float* center, const float* grad_out,
                           float* grad_x, float* value_out, int64_t N, int64_t M, int32_t D, int32_t kind, float blur,
                           void* scratch, int64_t scratch_bytes, void* stream) {
  const bool gauss = kind_base(kind) == B200OT_KERNEL_GAUSSIAN;
  const bool tc = gauss ? tc_routed(kTcConvBwd, D, N, M) : (D > B200OT_MAX_D && tc_capable_dim(D));
  if (!x || !y || !w || !grad_x || !scratch || N <= 0 || M <= 0 || !(supported_simt_dim(D) || tc) || !valid_kind(kind) ||
      (value_out && !gauss))
    return B200OT_EINVAL;
  if (!blur_ok(kind, blur)) return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, b200ot_kernel_conv_scratch_bytes(N, M, D))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (tc) return tc_kernel_conv(true, kind, x, y, w, center, grad_out, grad_x, value_out, N, M, D, blur, scratch, st);
  const ReducePlan pl = make_plan(N, M, D);
  const ConvScales cs = conv_scales(kind, blur);
  float* cols = reinterpret_cast<float*>(scratch);
  float* part = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) +
                                         round_up64(b200ot_packed_cols_floats(M, D, 2) * 4, 256));
  int rc = conv_pack(y, w, center, M, D, cs, cols, st);
  if (rc) return rc;
  rc = conv_partial(kind, true, pl, st, x, center, cs, cols, part, N, D);
  if (rc) return rc;
  return conv_bwd_finalize(part, pl.n_split, x, center, grad_out, grad_x, N, D, kind_base(kind), cs.scale,
                           conv_bwd_coef(kind, cs, blur), nullptr, value_out, nullptr, 0, st);
}

B200OT_API int b200ot_kernel_conv_bwd_x(const float* x, const float* y, const float* w, const float* center,
                                        const float* grad_out, float* grad_x, int64_t N, int64_t M, int32_t D,
                                        int32_t kind, float blur, void* scratch, int64_t scratch_bytes,
                                        void* stream) {
  if (!grad_out) return B200OT_EINVAL;
  return conv_bwd_x_impl(x, y, w, center, grad_out, grad_x, nullptr, N, M, D, kind, blur, scratch, scratch_bytes,
                         stream);
}

B200OT_API int b200ot_kernel_conv_fwd_bwd_x(const float* x, const float* y, const float* w, const float* center,
                                            float* out, float* grad_unit, int64_t N, int64_t M, int32_t D,
                                            int32_t kind, float blur, void* scratch, int64_t scratch_bytes,
                                            void* stream) {
  if (!out) return B200OT_EINVAL;
  return conv_bwd_x_impl(x, y, w, center, nullptr, grad_unit, out, N, M, D, kind, blur, scratch, scratch_bytes, stream);
}

}  // extern "C"
