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
                      int64_t M, int D, int p, float eps, float* cols_out, cudaStream_t st, const int* src);

// Tensor-core (wgmma) path, defined in b200ot_kernel_conv.cu.  The kernels serve any 1 <= D <= 64 (coordinates are
// zero-padded to a multiple of 16); above B200OT_MAX_D they are the only path, at or below it `tc_routed` decides per
// operator from the measured cross-over (see there).
enum TcOp { kTcSoftminFwd = 0, kTcSoftminBwd = 1, kTcConvFwd = 2, kTcConvBwd = 3 };
inline bool tc_capable_dim(int D) { return D >= 1 && D <= 64; }
bool tc_routed(int op, int D, int64_t N, int64_t M);
bool tc_any_routed(int D, int64_t N, int64_t M);  // some operator of this shape takes the tensor-core path (scratch sizing)
// Scratch of B problems of N rows x M columns (B = 1: one problem), any D the tensor cores serve: the larger of the
// forward plan and the row-gradient plan, whose rows keep D + head sums (head = 2: the p = 1 softmin)
int64_t tc_scratch_bytes(int64_t N, int64_t M, int D, int64_t B, int head);
// Shapes of the batched entry points: 8 < D <= 64 only (smaller dimensions batch through the ranges entry points)
inline bool tc_batched_dims(int64_t B, int64_t N, int64_t M, int D) {
  return B >= 1 && N > 0 && M > 0 && D > B200OT_MAX_D && tc_capable_dim(D);
}
// The p = 1 softmin on the tensor cores (b200ot_softmin_l1_*): B >= 1 elements, 8 < D <= 64, p = 1 | UNCLAMPED
inline bool tc_l1_args(int64_t B, int64_t N, int64_t M, int D, int p) {
  return tc_batched_dims(B, N, M, D) && valid_p(p) && p_exponent(p) == 1;
}
// Above D = 64 (b200ot_wide_*, tcwide.cuh): B >= 1 elements, 64 < D <= B200OT_MAX_D_WIDE
inline bool tc_wide_dims(int64_t B, int64_t N, int64_t M, int D) {
  return B >= 1 && N > 0 && M > 0 && D > 64 && D <= B200OT_MAX_D_WIDE;
}
// The parameter list of tc_reduce_kernel / tc_bwd_kernel and of the wide kernels
using TcKernel = void (*)(const unsigned char*, const unsigned char*, float*, int64_t, int, int, int, int, int, int,
                          float, const float*, int, int64_t, const int4*, const int2*, const int*);
// the wide kernel of a tc_reduce_kernel (bwd = false) or tc_bwd_kernel MODE, null for a mode it does not serve
// (b200ot_wide.cu)
TcKernel tc_wide_kernel(int mode, bool bwd);

// How the rows and columns of a tensor-core pass are laid out: one problem, a batch of B problems side by side (x
// (B,N,D), y (B,M,D), element b of the rows reduced over element b of the columns only), or one block-sparse problem.
// The p = 1 softmin runs the batch kernels only, B = 1 included.
enum class TcLayout { kOne, kBatch, kBlocks };

// A block-sparse problem (8 < D <= 64, p = 2; b200ot_*_blocks): every row cluster and every column cluster is padded
// to whole kTcBlocksTile-point tiles on its own, slot -> point through row_src / col_src (-1: padding), one segment per
// row tile.  blocks_check fills max_tiles (the longest segment in column tiles) and n_pieces (the pieces the segments
// reference).
inline bool tc_blocks_dims(int D) { return D > B200OT_MAX_D && tc_capable_dim(D); }
constexpr int kTcBlocksTile = 128;  // segment height and column alignment: the kernels' tile (kTcM = kTcBN, tcconv.cuh)
struct TcBlocks {
  const int *row_src, *col_src;
  int64_t n_row_slots, n_col_slots;
  const b200ot_segment* seg;
  int64_t n_seg;
  const b200ot_piece* pieces;
  int64_t n_pieces = 0;
  int max_tiles = 0;
};
// The checks every b200ot_*_blocks entry makes before any launch, in this order: EINVAL for a null descriptor array,
// N <= 0, n_seg <= 0, D outside (8, 64], p other than 2 (| B200OT_P_UNCLAMPED) or eps <= 0; EALIGN for misaligned
// descriptor arrays or scratch; EINVAL for descriptors off the tile grid.
int blocks_check(int64_t N, int D, int p, float eps, const void* scratch, TcBlocks& b);
int64_t tc_blocks_scratch_bytes(int64_t N, int D, const TcBlocks& b);

// A softmin on the tensor cores: B elements of N rows / M columns (TcLayout::kBlocks: B = 1, N rows, the slots in the
// TcBlocks).  p may carry B200OT_P_UNCLAMPED; lse2: the forward's, for the row gradients.
struct TcSoftmin {
  const float *x, *y, *h_a, *h_b;
  float h_scale_b;
  const float *center, *lse2;
  int64_t B, N, M;
  int D, p;
  float eps;
};
// What a pass leaves for its finalize: n_part sets of partials inside the scratch ((m, s) pairs forward, D + head sums
// per row for the row gradients), and the maxima the finalize undoes (null when the pass has none)
struct TcPass {
  float* part = nullptr;
  int n_part = 0;
  const float* w_absmax = nullptr;
  const float* coord_absmax = nullptr;
};
int softmin_pass_tc(bool bwd, TcLayout layout, const TcSoftmin& s, const TcBlocks* blocks, void* scratch,
                    cudaStream_t st, TcPass* r);
// out / lse2_out of the B N rows, as b200ot_softmin_finalize
int softmin_fwd_tc(TcLayout layout, const TcSoftmin& s, const TcBlocks* blocks, const float* out_old, float alpha_old,
                   float beta, float* out, float* lse2_out, void* scratch, void* stream);
int softmin_bwd_x_tc(TcLayout layout, const TcSoftmin& s, const TcBlocks* blocks, const float* grad_out, float* grad_x,
                     void* scratch, cudaStream_t st);
// grad_x of the N rows from the p = 2 softmin's tensor-core row-gradient sums, (n_part, N, D + 1), any D
// (b200ot_softmin_bwd.cu)
int softmin_bwd_finalize_tc(const float* part, int n_part, const float* x, const float* center, const float* grad_out,
                            float* grad_x, int64_t N, int D, float eps, cudaStream_t st);

// The plan applied to a value matrix v (M, K) (b200ot_plan_apply): the tensor-core pass (b200ot_kernel_conv.cu,
// tcapply.cuh) and the finalize both paths share (b200ot_plan_apply.cu).
int64_t plan_apply_tc_scratch_bytes(int64_t N, int64_t M, int D, int K);
int plan_apply_tc(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                  const float* center, const float* lse2, const float* v, const float* row_factor, float* out,
                  int64_t N, int64_t M, int D, int K, float eps, void* scratch, cudaStream_t st);
// out[i, k0 + k] = row_factor_i (sum_s part[s, i, 1 + k]) / (sum_s part[s, i, 0]) / s_k for k < kv, part (n_part, N,
// nacc); s_k = tc_energy_coord_scale(vmax[k0 + k]) when vmax is given, row_factor_i = 1 when it is null
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
