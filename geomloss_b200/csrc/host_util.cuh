// b200ot — host-side helpers shared by the translation units of libb200ot.so.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "b200ot.h"

namespace b200ot {

inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline int64_t round_up64(int64_t a, int64_t b) { return ceil_div64(a, b) * b; }

// Last CUDA error text seen by any entry point (process-wide, best effort; for diagnostics only).
void set_last_cuda_error(cudaError_t e, const char* where);

// SM count of the current device, cached per device ordinal.
int num_sms();

// Dimensions served by the CUDA-core (register tile) kernels that are instantiated in this build.
inline bool supported_simt_dim(int D) { return D >= 1 && D <= B200OT_MAX_D; }

// Cost exponent argument of the C ABI: 1 or 2, optionally or-ed with B200OT_P_UNCLAMPED (p = 1 only matters).
inline int p_exponent(int p) { return p & 0xff; }
inline bool valid_p(int p) {
  const int e = p & 0xff;
  return (e == 1 || e == 2) && (p & ~(0xff | B200OT_P_UNCLAMPED)) == 0;
}
// Clamp on |x-y|^2 under the square root: the reference's tensorized `distances` clamps at 1e-8 (utils.py:61);
// pykeops' Norm2 / sqrt do not (sqrt(0) = 0 with a zero gradient) — emulated by a clamp far below fp32 resolution.
inline float cost_clamp(int flags) { return (flags & B200OT_P_UNCLAMPED) ? 1e-30f : 1e-8f; }

// Coordinate scale of the softmin kernels: the log2-domain exponent is H - |X-Y|^2/2 (p = 2) or
// H - |X-Y| (p = 1) with X = scale * (x - c).
inline float softmin_coord_scale(int p, float eps) {
  return p == 2 ? sqrtf(1.4426950408889634f / eps) : 1.4426950408889634f / eps;
}

// Shared between translation units (defined in b200ot_softmin.cu).
int softmin_pack_impl(const float* y, const float* h_a, const float* h_b, float h_scale_b, const float* center,
                      int64_t M, int D, int p, float eps, float* cols_out, cudaStream_t st, const int* src,
                      const int* gate = nullptr);

// ---- the tensor-core (wgmma) path, b200ot_tc.cu ----
// The kernels serve any 1 <= D <= 64 (coordinates are zero-padded to a multiple of 16); above B200OT_MAX_D they are the
// only path, at or below it `tc_routed` decides per operator from the measured cross-over (see there).
enum TcOp { kTcSoftminFwd = 0, kTcSoftminBwd = 1, kTcConvFwd = 2, kTcConvBwd = 3 };
inline bool tc_capable_dim(int D) { return D >= 1 && D <= 64; }
bool tc_routed(int op, int D, int64_t N, int64_t M);
bool tc_any_routed(int D, int64_t N, int64_t M);  // some operator of this shape takes the tensor-core path (scratch sizing)
// Scratch of one problem of N rows x M columns, any D the tensor cores serve: enough for the softmin and kernel
// convolution passes, forward and row gradients
int64_t tc_scratch_bytes(int64_t N, int64_t M, int D);
int64_t tc_plan_apply_scratch_bytes(int64_t N, int64_t M, int D, int K);
// One problem on the tensor cores, the arguments validated by the caller.  The softmin forward leaves out / lse2_out as
// b200ot_softmin_finalize; the row-gradient sums leave *n_part sets of (N, D + 1) sums inside the scratch at *part,
// times kTcPScale (common.cuh); the kernel convolution leaves out (forward) or grad_x (bwd) in res and, with value_out,
// the forward values from the same pass (gaussian only); the plan apply leaves out (N, K) as b200ot_plan_apply.
int tc_softmin_fwd(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                   const float* center, const float* out_old, float alpha_old, float beta, float* out, float* lse2_out,
                   int64_t N, int64_t M, int D, int p, float eps, void* scratch, void* stream);
int tc_softmin_bwd_sums(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                        const float* center, const float* lse2, int64_t N, int64_t M, int D, int p, float eps,
                        void* scratch, cudaStream_t st, float** part, int* n_part);
int tc_kernel_conv(bool bwd, int kind, const float* x, const float* y, const float* w, const float* center,
                   const float* grad_out, float* res, float* value_out, int64_t N, int64_t M, int D, float blur,
                   void* scratch, cudaStream_t st);
int tc_plan_apply(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                  const float* center, const float* lse2, const float* v, const float* row_factor, float* out,
                  int64_t N, int64_t M, int D, int K, float eps, void* scratch, cudaStream_t st);
// The parameter list of tc_reduce_kernel / tc_bwd_kernel and of the wide kernels, and the wide kernel of a
// tc_reduce_kernel (bwd = false) or tc_bwd_kernel MODE, null for a mode it does not serve: instantiated in
// b200ot_wide.cu, a translation unit of its own so that it compiles next to b200ot_tc.cu
using TcKernel = void (*)(const unsigned char*, const unsigned char*, float*, int64_t, int, int, int, int, int, int,
                          float, const float*, int, int64_t, const int4*, const int2*, const int*);
TcKernel tc_wide_kernel(int mode, bool bwd);

// ---- finalize launches that both paths share, defined with their operator ----
// out = sign(kind) sum of the n_part (N) partials, the energy's coordinate scale undone when coord_absmax is given
// (b200ot_kernel_conv.cu: conv_fwd_finalize_kernel)
int conv_fwd_finalize(const float* part, int n_part, int kind, float* out, int64_t N, const float* coord_absmax,
                      cudaStream_t st);
// grad_x (and value_out) from the row-gradient sums of a kernel convolution (b200ot_kernel_conv.cu:
// conv_bwd_finalize_kernel)
int conv_bwd_finalize(const float* part, int n_part, const float* x, const float* center, const float* grad_out,
                      float* grad_x, int64_t N, int D, int kind, float scale, float coef, const float* w_absmax,
                      float* value_out, const float* coord_absmax, int64_t n_per, cudaStream_t st);
// grad_x of the N rows from the p = 2 softmin's tensor-core row-gradient sums, (n_part, N, D + 1), any D
// (b200ot_softmin_bwd.cu)
int softmin_bwd_finalize_tc(const float* part, int n_part, const float* x, const float* center, const float* grad_out,
                            float* grad_x, int64_t N, int D, float eps, cudaStream_t st);
// out[i, k0 + k] = row_factor_i (sum_s part[s, i, 1 + k]) / (sum_s part[s, i, 0]) / s_k for k < kv, part (n_part, N,
// nacc); s_k = tc_energy_coord_scale(vmax[k0 + k]) when vmax is given, row_factor_i = 1 when it is null
// (b200ot_plan_apply.cu)
int plan_apply_finalize(const float* part, int n_part, int nacc, int kv, int k0, int K, const float* vmax,
                        const float* row_factor, float* out, int64_t N, cudaStream_t st);

// The scratch checks of an entry point, in this order: EALIGN for a scratch not 16-byte aligned, ESCRATCH below `need`
inline int scratch_check(const void* scratch, int64_t scratch_bytes, int64_t need) {
  if (((uintptr_t)scratch) & 15) return B200OT_EALIGN;
  return scratch_bytes < need ? B200OT_ESCRATCH : B200OT_OK;
}

#define B200OT_STR2(x) #x
#define B200OT_STR(x) B200OT_STR2(x)
#define B200OT_CUDA_TRY(expr)                                                         \
  do {                                                                                \
    cudaError_t e__ = (expr);                                                         \
    if (e__ != cudaSuccess) {                                                         \
      ::b200ot::set_last_cuda_error(e__, __FILE__ ":" B200OT_STR(__LINE__));          \
      return B200OT_ECUDA;                                                            \
    }                                                                                 \
  } while (0)

}  // namespace b200ot
