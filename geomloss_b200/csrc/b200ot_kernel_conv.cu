// b200ot — kernel convolutions  out_i = sum_j k(x_i, y_j) w_j  and their row gradients.
// Reference semantics: the matvecs of kernel_loss (src/geomloss/_legacy/kernel_samples.py:116-137) with
//   gaussian  k = exp(-|x/s - y/s|^2 / 2)                    (kernel_samples.py:62-68)
//   laplacian k = exp(-sqrt(max(|x/s - y/s|^2, 1e-8)))       (kernel_samples.py:71-77, utils.py:56-61)
//   energy    k = -sqrt(max(|x - y|^2, 1e-8))                (kernel_samples.py:80-82)
// evaluated on the fly (never as an N x M matrix) by rowsum_partial_kernel.
#include "b200ot.h"
#include "host_util.cuh"
#include "pack.cuh"
#include "plan.cuh"
#include "rowsum.cuh"
#include "rowsum_launch.cuh"
#include "tcbwd.cuh"
#include "tcconv.cuh"

#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <type_traits>
#include <vector>

namespace b200ot {

struct ConvScales {
  float scale;   // coordinate scale
  float clampq;  // clamp on the scaled squared distance
  int direct;
  int extra;
};

// `kind` may carry B200OT_KERNEL_UNCLAMPED (laplacian / energy with pykeops' unclamped sqrt)
static int kind_base(int kind) { return kind & 0xff; }
static bool valid_kind(int kind) {
  return kind_base(kind) >= 0 && kind_base(kind) <= 2 && (kind & ~(0xff | B200OT_KERNEL_UNCLAMPED)) == 0;
}

static ConvScales conv_scales(int kind_flags, float blur) {
  ConvScales c;
  const int kind = kind_base(kind_flags);
  const float clamp = cost_clamp(kind_flags);  // B200OT_KERNEL_UNCLAMPED == B200OT_P_UNCLAMPED
  if (kind == B200OT_KERNEL_GAUSSIAN) {
    c.scale = sqrtf(kLog2e) / blur;  // 2^(-|X-Y|^2/2) = exp(-|x-y|^2 / (2 blur^2))
    c.clampq = 0.f;
    c.direct = 0;
    c.extra = 2;
  } else if (kind == B200OT_KERNEL_LAPLACIAN) {
    c.scale = kLog2e / blur;  // 2^(-|X-Y|) = exp(-|x-y| / blur)
    c.clampq = kLog2e * kLog2e * clamp;
    c.direct = 1;
    c.extra = 1;
  } else {
    c.scale = 1.f;
    c.clampq = clamp;
    c.direct = 1;
    c.extra = 1;
  }
  return c;
}

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

// max_j |w_j| into *out (zero-initialised by the caller); bit order of non-negative floats = integer order.
// gridDim.y > 1: one maximum per batch element of n weights, out[blockIdx.y]
__global__ void absmax_kernel(const float* __restrict__ w, int64_t n, float* __restrict__ out) {
  w += (int64_t)blockIdx.y * n;
  out += blockIdx.y;
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(w[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f && !(m != m)) atomicMax(reinterpret_cast<unsigned int*>(out), __float_as_uint(m));
}

// max_k |pts[i, k] - center[k]| over the rows of a (na x D) and b (nb x D) into *out (zero-initialised by the caller)
__global__ void coord_absmax_kernel(const float* __restrict__ a, int64_t na, const float* __restrict__ b, int64_t nb,
                                    int D, const float* __restrict__ center, float* __restrict__ out) {
  float m = 0.f;
  const int64_t ta = na * D, tot = ta + nb * D;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (int64_t)gridDim.x * blockDim.x) {
    const float v = e < ta ? a[e] : b[e - ta];
    m = fmaxf(m, fabsf(v - (center ? center[e % D] : 0.f)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f && !(m != m)) atomicMax(reinterpret_cast<unsigned int*>(out), __float_as_uint(m));
}

template <int MODE, int D>
static int launch_rowsum(const ReducePlan& pl, cudaStream_t st, const float* x, const float* center, float scale,
                         float clampq, const float* cols, float* part, int64_t N, const int4* seg = nullptr,
                         const int2* pieces = nullptr) {
  if (pl.small) {
    using C = RowSumCfg<MODE, D, kSmallR, kSmallNT, kSmallTJ, 3, 4>;
    return launch_rowsum_kernel<C>(pl, st, x, center, scale, clampq, cols,
                            (const float*)nullptr, part, N, pl.ntiles, pl.tiles_per_split, seg, pieces);
  }
  // D >= 5: one row per thread (same 512 rows per CTA) keeps the 2 x (D+1) accumulator pairs in registers
  using C = std::conditional_t<(D <= 4), RowSumCfg<MODE, D, kBigR, kBigNT, kBigTJ, 3, 2>,
                               RowSumCfg<MODE, D, 1, kBigR * kBigNT, kBigTJ, 3, 1>>;
  return launch_rowsum_kernel<C>(pl, st, x, center, scale, clampq, cols, (const float*)nullptr,
                          part, N, pl.ntiles, pl.tiles_per_split, seg, pieces);
}

template <int MODE>
static int launch_rowsum_d(int D, const ReducePlan& pl, cudaStream_t st, const float* x, const float* center,
                           float scale, float clampq, const float* cols, float* part, int64_t N,
                           const int4* seg = nullptr, const int2* pieces = nullptr) {
  switch (D) {
    case 1: return launch_rowsum<MODE, 1>(pl, st, x, center, scale, clampq, cols, part, N, seg, pieces);
    case 2: return launch_rowsum<MODE, 2>(pl, st, x, center, scale, clampq, cols, part, N, seg, pieces);
    case 3: return launch_rowsum<MODE, 3>(pl, st, x, center, scale, clampq, cols, part, N, seg, pieces);
    case 4: return launch_rowsum<MODE, 4>(pl, st, x, center, scale, clampq, cols, part, N, seg, pieces);
    case 5: return launch_rowsum<MODE, 5>(pl, st, x, center, scale, clampq, cols, part, N, seg, pieces);
    case 6: return launch_rowsum<MODE, 6>(pl, st, x, center, scale, clampq, cols, part, N, seg, pieces);
    case 7: return launch_rowsum<MODE, 7>(pl, st, x, center, scale, clampq, cols, part, N, seg, pieces);
    case 8: return launch_rowsum<MODE, 8>(pl, st, x, center, scale, clampq, cols, part, N, seg, pieces);
    default: return B200OT_EINVAL;
  }
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
  if (kind == B200OT_KERNEL_GAUSSIAN)
    return bwd ? launch_rowsum_d<kGaussBwd>(D, pl, st, x, center, cs.scale, cs.clampq, cols, part, N, seg, pieces)
               : launch_rowsum_d<kGaussFwd>(D, pl, st, x, center, cs.scale, cs.clampq, cols, part, N, seg, pieces);
  if (kind == B200OT_KERNEL_LAPLACIAN)
    return bwd ? launch_rowsum_d<kLaplaceBwd>(D, pl, st, x, center, cs.scale, cs.clampq, cols, part, N, seg, pieces)
               : launch_rowsum_d<kLaplaceFwd>(D, pl, st, x, center, cs.scale, cs.clampq, cols, part, N, seg, pieces);
  return bwd ? launch_rowsum_d<kEnergyBwd>(D, pl, st, x, center, cs.scale, cs.clampq, cols, part, N, seg, pieces)
             : launch_rowsum_d<kEnergyFwd>(D, pl, st, x, center, cs.scale, cs.clampq, cols, part, N, seg, pieces);
}

static float conv_bwd_coef(int kind_flags, const ConvScales& cs, float blur) {
  const int kind = kind_base(kind_flags);
  if (kind == B200OT_KERNEL_GAUSSIAN) return 1.0f / (cs.scale * blur * blur);
  if (kind == B200OT_KERNEL_LAPLACIAN) return -1.0f / blur;
  return -1.0f;
}

// ---------------------------------------------------------------------------------------------------
// tensor-core path (gaussian, and laplacian / energy for 8 < D <= 64): see tcconv.cuh
// ---------------------------------------------------------------------------------------------------
struct TcPlan {
  int kp, nstage, n_split, tiles_per_split;
  int rtpe, ctpe;  // row / column tiles per batch element
  int64_t a_tiles, b_tiles, a_bytes, b_bytes, smem;
  int64_t off_b, off_part, off_misc, total;
};

// Which path serves an operator.  Above B200OT_MAX_D the tensor-core kernels are the only ones.  At or below it both
// exist: the CUDA-core kernels are FMA-pipe bound from D = 5 up while the tensor-core kernels run the zero-padded
// dk = 16 problem at the same rate whatever D.  Measured on an H100 80GB HBM3 (SXM, 400 W power limit) at N = M = 4e5
// (tools/ab_tc_route.py part A; CUDA-core -> tensor-core, 1e12 pairs/s):
//   softmin forward   D = 5: 2.38 -> 1.96   D = 6: 2.02 -> 1.95   D = 7: 1.85 -> 1.94   D = 8: 1.54 -> 1.87
//   gaussian forward  D = 4: 2.42 -> 2.39   D = 5: 1.77 -> 2.42   D = 6: 1.60 -> 2.45   D = 8: 1.31 -> 2.37
//   row gradients     D = 6: 1.33 / 1.22 -> 1.69 / 1.52 (softmin / gaussian); D = 8: 1.08 / 0.97 -> 1.63 / 1.49
// (at N = M = 1e5 and 3e4 the softmin forward already breaks even at D = 6, the others switch where they do at 4e5).  The
// forward operators switch at D = 7 (softmin) and D = 5 (gaussian).  The row gradients stay on the CUDA cores for every
// D <= 8 although the tensor cores are faster from D = 6: the fp16 image of P that GEMM 2 consumes costs accuracy at
// small blur in low dimension (relative difference between the two paths' gradients at eps = 1e-4 / blur = .05 in the
// same run: up to 3e-3 at D = 4, 4e-4 at D = 6..8, against ~1e-5 for the forward operators).  Problems below 8e8 pairs
// keep the CUDA-core kernels.  $B200OT_TC_MIN_D ("d" or "softmin_fwd,softmin_bwd,conv_fwd,conv_bwd")
// and $B200OT_TC_MIN_PAIRS override the defaults for A/B timing and for the parity tests of both routes — read on every
// call, never set by the bench.
static const int kTcMinDimDefault[4] = {7, 9, 5, 9};
static const double kTcMinPairsDefault = 8.0e8;

bool tc_routed(int op, int D, int64_t N, int64_t M) {
  if (!tc_capable_dim(D)) return false;
  if (D > B200OT_MAX_D) return true;
  int min_dim[4] = {kTcMinDimDefault[0], kTcMinDimDefault[1], kTcMinDimDefault[2], kTcMinDimDefault[3]};
  double min_pairs = kTcMinPairsDefault;
  if (const char* e = getenv("B200OT_TC_MIN_D")) {
    int v[4];
    const int n = sscanf(e, "%d,%d,%d,%d", &v[0], &v[1], &v[2], &v[3]);
    if (n == 1) {
      for (int k = 0; k < 4; ++k) min_dim[k] = v[0];
    } else if (n == 4) {
      for (int k = 0; k < 4; ++k) min_dim[k] = v[k];
    }
  }
  if (const char* e = getenv("B200OT_TC_MIN_PAIRS")) {
    const double v = atof(e);
    if (v >= 0.0) min_pairs = v;
  }
  return D >= min_dim[op] && (double)N * (double)M >= min_pairs;
}

bool tc_any_routed(int D, int64_t N, int64_t M) {
  for (int op = 0; op < 4; ++op)
    if (tc_routed(op, D, N, M)) return true;
  return false;
}

// Tuning of the row-gradient kernels (tcbwd.cuh), $B200OT_TC_BWD = "p_terms,epi,ldall,merge" for A/B timing and the
// variants' parity tests (the settings string of the C ABI, see b200ot.h):
//   p_terms  fp16 terms of P in GEMM 2 (PT).  PT = 1 saves a third of the GEMM-2 work but feeds GEMM 2 an 11-bit image
//            of P (every weight perturbed by <= 2^-12) — kept as a knob, not the default.  Measured on an
//            H100 80GB HBM3 (400 W) at N = M = 4e5, gaussian / softmin row gradients, ms: D = 16 119.5 / 111.9 (PT = 2)
//            against 107.7 / 91.3 (PT = 1); D = 64 260 / 222 against 229 / 196.
//   merge    hi.[Y_h | Y_l] as one N = 2 dk instruction per K step (1) or two N = dk instructions (0): the same
//            products and the same fp32 accumulation, so the choice does not change the result.
//   epi, ldall  the epilogue-warp count (8 or 16) and the single-load TMEM read-back of tensor-memory kernels.  The
//            wgmma kernels keep S and P in the registers of their two consumer warpgroups, so neither has a counterpart
//            here: both are validated and otherwise leave the kernel unchanged.
struct TcBwdTuning {
  int p_terms, epi, ldall, merge;
};
static const TcBwdTuning kTcBwdDefault = {2, 8, 0, 1};
static TcBwdTuning tc_bwd_tuning() {
  TcBwdTuning t = kTcBwdDefault;
  if (const char* e = getenv("B200OT_TC_BWD")) {
    int a, b, c, d;
    if (sscanf(e, "%d,%d,%d,%d", &a, &b, &c, &d) == 4 && (a == 1 || a == 2) && (b == 8 || b == 16) &&
        (c == 0 || c == 1) && (d == 0 || d == 1)) {
      t.p_terms = a;
      t.epi = b;
      t.ldall = c;
      t.merge = d;
    }
  }
  return t;
}

// B > 1 (the batched entry points): B problems of N rows x M columns side by side, each element padded to whole tiles on
// its own (tc_pack_kernel).  The split count is chosen for the whole grid, as without a batch, and cuts each element's
// ctpe column tiles (so it is capped at ctpe); a CTA never reads another element's columns.  B = 1 is the plan of one
// problem.
static TcPlan make_tc_plan(int64_t N, int64_t M, int D, bool bwd = false, int64_t B = 1) {
  TcPlan p;
  p.kp = tc_kp(D);
  p.rtpe = (int)ceil_div64(N, kTcM);
  p.ctpe = (int)ceil_div64(M, kTcBN);
  p.a_tiles = B * p.rtpe;
  p.b_tiles = B * p.ctpe;
  p.a_bytes = tc_a_img_bytes(p.kp);
  p.b_bytes = tc_b_img_bytes(p.kp, kTcBN);
  const int64_t bar_bytes = 256;  // mbarriers behind the column ring
  // the CTA's row image stays in shared memory; the rest of the 227 KB a block may use holds the column ring
  const int64_t avail = 227 * 1024 - bar_bytes - tc_a_span(p.kp);
  int64_t ns = avail / p.b_bytes;
  p.nstage = (int)(ns > kTcMaxStage ? kTcMaxStage : ns);
  p.smem = tc_a_span(p.kp) + p.nstage * p.b_bytes + bar_bytes;
  int64_t want = ceil_div64((int64_t)num_sms() * 4, p.a_tiles);
  const int forced = forced_splits();  // test hook (plan.cuh)
  if (forced > 0) want = forced;
  if (want < 1) want = 1;
  if (want > 64) want = 64;
  if (want > p.ctpe) want = p.ctpe;
  p.tiles_per_split = (int)ceil_div64(p.ctpe, want);
  p.n_split = (int)ceil_div64(p.ctpe, p.tiles_per_split);
  p.off_b = round_up64(p.a_tiles * p.a_bytes, 256);
  p.off_part = p.off_b + round_up64(p.b_tiles * p.b_bytes, 256);
  // partials: (m, s) pairs forward, D+1 sums per row backward
  p.off_misc = p.off_part + round_up64((int64_t)p.n_split * (bwd ? B * N * (D + 1) : kTcParts * B * N * 2) * 4, 256);
  p.total = p.off_misc + round_up64((B + 1) * 4, 256);  // [0]: energy coordinate max, [1 + b]: max|w| of element b
  return p;
}

int64_t tc_scratch_bytes(int64_t N, int64_t M, int D, int64_t B) {
  // forward and row-gradient launches split the columns differently: size for the larger of the two
  return std::max(make_tc_plan(N, M, D, false, B).total, make_tc_plan(N, M, D, true, B).total);
}

// Row gradients on the tensor-core path; `mode` is the MODE of tc_bwd_kernel (2 gaussian conv, 3 softmin p = 2,
// 4 laplacian, 5 energy; clampq and coord_absmax: see there).  Leaves n_part sets of (B N, D+1) partial sums in
// *part_out.  `batched`: B elements of N rows / M columns (make_tc_plan), the weights normalised per element.
int bwd_partial_tc(int mode, const float* x, const float* y, const float* w, const float* h_a, const float* h_b,
                   float h_scale_b, const float* lse2, const float* center, float scale, int64_t N, int64_t M, int D,
                   void* scratch, float** part_out, int* n_part_out, cudaStream_t st, const float** w_absmax_out,
                   float clampq, const float* coord_absmax, int64_t B, bool batched) {
  const TcPlan p = make_tc_plan(N, M, D, true, B);
  if (p.nstage < 1) return B200OT_EINVAL;
  unsigned char* base = reinterpret_cast<unsigned char*>(scratch);
  unsigned char* a_imgs = base;
  unsigned char* b_imgs = base + p.off_b;
  float* part = reinterpret_cast<float*>(base + p.off_part);
  float* w_absmax = nullptr;
  if (w != nullptr) {
    // P = w_j e_ij feeds an fp16 GEMM: normalise the weights to max|w| = kTcPScale (undone by the finalize kernel),
    // one maximum per batch element, so that a heavy element cannot push a light one's P into fp16's subnormal range
    w_absmax = reinterpret_cast<float*>(base + p.off_misc) + 1;
    B200OT_CUDA_TRY(cudaMemsetAsync(w_absmax, 0, B * sizeof(float), st));
    const dim3 g((unsigned)std::min<int64_t>(ceil_div64(M, 256), 1024), (unsigned)B);
    absmax_kernel<<<g, 256, 0, st>>>(w, M, w_absmax);
    B200OT_CUDA_TRY(cudaGetLastError());
  }
  if (w_absmax_out) *w_absmax_out = w_absmax;
  const int threads = 128;
  tc_pack_kernel<<<(unsigned)ceil_div64(p.a_tiles * kTcM, threads), threads, 0, st>>>(
      x, nullptr, nullptr, nullptr, 0.f, 0.f, center, scale, N, D, p.kp, kTcM, 0, a_imgs, lse2, nullptr, coord_absmax,
      B);
  B200OT_CUDA_TRY(cudaGetLastError());
  tc_pack_kernel<<<(unsigned)ceil_div64(p.b_tiles * kTcBN, threads), threads, 0, st>>>(
      y, w, h_a, h_b, h_scale_b, kLog2e, center, scale, M, D, p.kp, kTcBN, 1, b_imgs, nullptr, w_absmax,
      coord_absmax, B);
  B200OT_CUDA_TRY(cudaGetLastError());
  dim3 grid((unsigned)p.a_tiles, (unsigned)p.n_split);
  const int self_mode = (mode != 3 && x == y && N == M) ? 1 : 0;  // K_xx: exact zero exponent on the diagonal
  auto launch = [&](auto kern) -> int {
    B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    kern<<<grid, kTcThreads, (size_t)p.smem, st>>>(a_imgs, b_imgs, part, B * N, p.kp, p.ctpe, p.tiles_per_split,
                                                   p.nstage, D, self_mode, clampq, coord_absmax, p.rtpe, N, nullptr, nullptr, nullptr);
    B200OT_CUDA_TRY(cudaGetLastError());
    return B200OT_OK;
  };
  const TcBwdTuning tn = tc_bwd_tuning();
  // (MODE, PT, MERGE, padded dimension, batch) -> instantiation
  auto pick_dk = [&](auto mode_tag, auto pt_tag, auto merge_tag, auto batch_tag) -> int {
    constexpr int MODE = decltype(mode_tag)::value, PT = decltype(pt_tag)::value;
    constexpr bool MG = decltype(merge_tag)::value, BT = decltype(batch_tag)::value;
    switch (tc_dk(D)) {
      case 16: return launch(tc_bwd_kernel<MODE, PT, MG, 16, BT>);
      case 32: return launch(tc_bwd_kernel<MODE, PT, MG, 32, BT>);
      case 48: return launch(tc_bwd_kernel<MODE, PT, MG, 48, BT>);
      default: return launch(tc_bwd_kernel<MODE, PT, MG, 64, BT>);
    }
  };
  // the default variant (PT = 2, MERGE): the only one of the laplacian and energy row gradients and of every batched
  // row gradient
  using T2 = std::integral_constant<int, 2>;
  auto pick_default = [&](auto mode_tag) -> int {
    return batched ? pick_dk(mode_tag, T2{}, std::true_type{}, std::true_type{})
                   : pick_dk(mode_tag, T2{}, std::true_type{}, std::false_type{});
  };
  auto pick = [&](auto mode_tag) -> int {
    using T1 = std::integral_constant<int, 1>;
    using NB = std::false_type;
    if (batched) return pick_default(mode_tag);
    if (tn.merge)
      return tn.p_terms == 1 ? pick_dk(mode_tag, T1{}, std::true_type{}, NB{})
                             : pick_dk(mode_tag, T2{}, std::true_type{}, NB{});
    return tn.p_terms == 1 ? pick_dk(mode_tag, T1{}, std::false_type{}, NB{})
                           : pick_dk(mode_tag, T2{}, std::false_type{}, NB{});
  };
  int rc;
  switch (mode) {
    case 2: rc = pick(std::integral_constant<int, 2>{}); break;
    case 3: rc = pick(std::integral_constant<int, 3>{}); break;
    case 4: rc = pick_default(std::integral_constant<int, 4>{}); break;
    default: rc = pick_default(std::integral_constant<int, 5>{}); break;
  }
  if (rc) return rc;
  *part_out = part;
  *n_part_out = p.n_split;  // G of a CTA is complete over its column split (both column halves feed one GEMM)
  return B200OT_OK;
}

// Tensor-core softmin partials (p = 2): packs both clouds, runs the reduction, leaves n_part (m, s) sets in
// `*part_out` (inside scratch) for b200ot_softmin_finalize.  `batched`: B elements (make_tc_plan), B N rows of partials.
int softmin_partial_tc(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                       const float* center, int64_t N, int64_t M, int D, float eps, void* scratch,
                       float** part_out, int* n_part_out, cudaStream_t st, int64_t B, bool batched) {
  const TcPlan p = make_tc_plan(N, M, D, false, B);
  if (p.nstage < 1) return B200OT_EINVAL;
  unsigned char* base = reinterpret_cast<unsigned char*>(scratch);
  unsigned char* a_imgs = base;
  unsigned char* b_imgs = base + p.off_b;
  float* part = reinterpret_cast<float*>(base + p.off_part);
  const float scale = softmin_coord_scale(2, eps);
  const int threads = 128;
  tc_pack_kernel<<<(unsigned)ceil_div64(p.a_tiles * kTcM, threads), threads, 0, st>>>(
      x, nullptr, nullptr, nullptr, 0.f, 0.f, center, scale, N, D, p.kp, kTcM, 0, a_imgs, nullptr, nullptr, nullptr, B);
  B200OT_CUDA_TRY(cudaGetLastError());
  tc_pack_kernel<<<(unsigned)ceil_div64(p.b_tiles * kTcBN, threads), threads, 0, st>>>(
      y, nullptr, h_a, h_b, h_scale_b, kLog2e, center, scale, M, D, p.kp, kTcBN, 1, b_imgs, nullptr, nullptr, nullptr,
      B);
  B200OT_CUDA_TRY(cudaGetLastError());
  auto kern = batched ? tc_reduce_kernel<1, true> : tc_reduce_kernel<1>;
  B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
  dim3 grid((unsigned)p.a_tiles, (unsigned)p.n_split);
  kern<<<grid, kTcThreads, (size_t)p.smem, st>>>(a_imgs, b_imgs, part, B * N, p.kp, p.ctpe, p.tiles_per_split,
                                                 p.nstage, D, 0, 0.f, nullptr, p.rtpe, N, nullptr, nullptr, nullptr);
  B200OT_CUDA_TRY(cudaGetLastError());
  *part_out = part;
  *n_part_out = p.n_split * kTcParts;
  return B200OT_OK;
}

// ---------------------------------------------------------------------------------------------------
// Block-sparse softmins (the fine phase of the two-scale Sinkhorn above D = 8): every row cluster and every column
// cluster is padded to whole 128-point tiles on its own, slot -> point through row_src / col_src (-1: padding).  One
// segment per row tile; the host descriptors are validated here and copied into the scratch behind the partials.
// ---------------------------------------------------------------------------------------------------
static_assert(kTcBlocksTile == kTcM && kTcBlocksTile == kTcBN, "segments are one row tile, pieces whole column tiles");

int blocks_validate(int64_t n_row_slots, int64_t n_col_slots, const b200ot_segment* seg, int64_t n_seg,
                    const b200ot_piece* pieces, int* max_tiles, int64_t* n_pieces) {
  if (n_row_slots <= 0 || n_col_slots <= 0 || n_row_slots % kTcM || n_col_slots % kTcBN ||
      n_row_slots / kTcM != n_seg || n_col_slots / kTcBN > 0x7fffffff)
    return B200OT_EINVAL;
  int64_t np = 0;
  for (int64_t s = 0; s < n_seg; ++s) {
    const b200ot_segment& g = seg[s];
    if (g.row_start < 0 || g.row_start % kTcM || g.row_start >= n_row_slots || g.row_count < 1 ||
        g.row_count > kTcM || g.piece_begin < 0 || g.piece_end < g.piece_begin)
      return B200OT_EINVAL;
    np = std::max<int64_t>(np, g.piece_end);
  }
  // column tiles before piece q, so that a segment's tile count is one difference
  std::vector<int64_t> before(np + 1, 0);
  for (int64_t q = 0; q < np; ++q) {
    const b200ot_piece& c = pieces[q];
    if (c.col_start < 0 || c.col_start % kTcBN || c.col_count <= 0 || c.col_count % kTcBN ||
        (int64_t)c.col_start + c.col_count > n_col_slots)
      return B200OT_EINVAL;
    before[q + 1] = before[q] + c.col_count / kTcBN;
  }
  // every row tile belongs to exactly one segment: each live row is written once per split
  std::vector<char> seen(n_seg, 0);
  int64_t mt = 0;
  for (int64_t s = 0; s < n_seg; ++s) {
    const int64_t t = seg[s].row_start / kTcM;
    if (seen[t]) return B200OT_EINVAL;
    seen[t] = 1;
    mt = std::max(mt, before[seg[s].piece_end] - before[seg[s].piece_begin]);
  }
  if (mt > 0x7fffffff) return B200OT_EINVAL;
  *max_tiles = (int)mt;
  *n_pieces = np;
  return B200OT_OK;
}

// The plan of one block-sparse problem: images of n_row_slots / n_col_slots points, segments cut into splits the way
// make_tc_plan cuts a dense problem's column tiles (from the longest segment), then the descriptors.
static TcPlan make_tc_blocks_plan(int64_t N, int64_t n_row_slots, int64_t n_col_slots, int64_t n_seg, int64_t n_pieces,
                                  int max_tiles, int D, bool bwd) {
  TcPlan p = make_tc_plan(kTcM, kTcBN, D, bwd);
  p.a_tiles = n_row_slots / kTcM;
  p.b_tiles = n_col_slots / kTcBN;
  int64_t want = ceil_div64((int64_t)num_sms() * 4, n_seg);
  const int forced = forced_splits();  // test hook (plan.cuh)
  if (forced > 0) want = forced;
  if (want < 1) want = 1;
  if (want > 64) want = 64;
  const int mt = std::max(max_tiles, 1);
  if (want > mt) want = mt;
  p.tiles_per_split = (int)ceil_div64(mt, want);
  p.n_split = (int)ceil_div64(mt, p.tiles_per_split);
  p.off_b = round_up64(p.a_tiles * p.a_bytes, 256);
  p.off_part = p.off_b + round_up64(p.b_tiles * p.b_bytes, 256);
  p.off_misc = p.off_part + round_up64((int64_t)p.n_split * (bwd ? N * (D + 1) : kTcParts * N * 2) * 4, 256);
  p.total = p.off_misc + round_up64(n_seg * 16, 256) + round_up64(std::max<int64_t>(n_pieces, 1) * 8, 256);
  return p;
}

int64_t tc_blocks_scratch_bytes(int64_t N, int64_t n_row_slots, int64_t n_col_slots, int64_t n_seg, int64_t n_pieces,
                                int max_tiles, int D) {
  return std::max(make_tc_blocks_plan(N, n_row_slots, n_col_slots, n_seg, n_pieces, max_tiles, D, false).total,
                  make_tc_blocks_plan(N, n_row_slots, n_col_slots, n_seg, n_pieces, max_tiles, D, true).total);
}

// Pack, descriptor copy and reduction of one block-sparse softmin (bwd: the row-gradient sums, lse2 = the forward's);
// arguments already validated.  Leaves n_part partial sets of N rows in *part_out, like softmin_partial_tc (forward)
// and bwd_partial_tc (backward).
int softmin_blocks_tc(bool bwd, const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                      const float* center, const float* lse2, int64_t N, const int* row_src, int64_t n_row_slots,
                      const int* col_src, int64_t n_col_slots, const b200ot_segment* seg, int64_t n_seg,
                      const b200ot_piece* pieces, int64_t n_pieces, int max_tiles, int D, float eps, void* scratch,
                      float** part_out, int* n_part_out, cudaStream_t st) {
  const TcPlan p = make_tc_blocks_plan(N, n_row_slots, n_col_slots, n_seg, n_pieces, max_tiles, D, bwd);
  if (p.nstage < 1) return B200OT_EINVAL;
  unsigned char* base = reinterpret_cast<unsigned char*>(scratch);
  unsigned char* a_imgs = base;
  unsigned char* b_imgs = base + p.off_b;
  float* part = reinterpret_cast<float*>(base + p.off_part);
  int4* d_seg = reinterpret_cast<int4*>(base + p.off_misc);
  int2* d_pieces = reinterpret_cast<int2*>(base + p.off_misc + round_up64(n_seg * 16, 256));
  const float scale = softmin_coord_scale(2, eps);
  B200OT_CUDA_TRY(cudaMemcpyAsync(d_seg, seg, n_seg * 16, cudaMemcpyHostToDevice, st));
  if (n_pieces > 0) B200OT_CUDA_TRY(cudaMemcpyAsync(d_pieces, pieces, n_pieces * 8, cudaMemcpyHostToDevice, st));
  const int threads = 128;
  tc_pack_kernel<<<(unsigned)ceil_div64(n_row_slots, threads), threads, 0, st>>>(
      x, nullptr, nullptr, nullptr, 0.f, 0.f, center, scale, n_row_slots, D, p.kp, kTcM, 0, a_imgs,
      bwd ? lse2 : nullptr, nullptr, nullptr, 1, row_src);
  B200OT_CUDA_TRY(cudaGetLastError());
  tc_pack_kernel<<<(unsigned)ceil_div64(n_col_slots, threads), threads, 0, st>>>(
      y, nullptr, h_a, h_b, h_scale_b, kLog2e, center, scale, n_col_slots, D, p.kp, kTcBN, 1, b_imgs, nullptr, nullptr,
      nullptr, 1, col_src);
  B200OT_CUDA_TRY(cudaGetLastError());
  dim3 grid((unsigned)n_seg, (unsigned)p.n_split);
  auto launch = [&](auto kern) -> int {
    B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    kern<<<grid, kTcThreads, (size_t)p.smem, st>>>(a_imgs, b_imgs, part, N, p.kp, 0, p.tiles_per_split, p.nstage, D, 0,
                                                   0.f, nullptr, 0, 0, d_seg, d_pieces, row_src);
    B200OT_CUDA_TRY(cudaGetLastError());
    return B200OT_OK;
  };
  int rc;
  if (!bwd) {
    rc = launch(tc_reduce_kernel<1, false, true>);
  } else {
    // the default row-gradient variant (PT = 2, MERGE)
    switch (tc_dk(D)) {
      case 16: rc = launch(tc_bwd_kernel<3, 2, true, 16, false, true>); break;
      case 32: rc = launch(tc_bwd_kernel<3, 2, true, 32, false, true>); break;
      case 48: rc = launch(tc_bwd_kernel<3, 2, true, 48, false, true>); break;
      default: rc = launch(tc_bwd_kernel<3, 2, true, 64, false, true>); break;
    }
  }
  if (rc) return rc;
  *part_out = part;
  *n_part_out = bwd ? p.n_split : p.n_split * kTcParts;
  return B200OT_OK;
}

// Energy on the tensor cores: the largest centred coordinate of both clouds (of every batch element: one scale for the
// whole batch, a power of two that the finalize undoes exactly), from which every kernel of the pass derives the same
// power-of-two coordinate scale (tc_energy_coord_scale).  Kept in the scratch's misc block, [0].
static int energy_coord_absmax(const float* x, int64_t N, const float* y, int64_t M, int D, const float* center,
                               unsigned char* misc, cudaStream_t st, const float** out) {
  float* a = reinterpret_cast<float*>(misc);
  B200OT_CUDA_TRY(cudaMemsetAsync(a, 0, sizeof(float), st));
  coord_absmax_kernel<<<(unsigned)std::min<int64_t>(ceil_div64((N + M) * D, 256), 1024), 256, 0, st>>>(x, N, y, M, D,
                                                                                                       center, a);
  B200OT_CUDA_TRY(cudaGetLastError());
  *out = a;
  return B200OT_OK;
}

static int conv_fwd_tc(int kind_flags, const float* x, const float* y, const float* w, const float* center, float* out,
                       int64_t N, int64_t M, int D, float blur, void* scratch, cudaStream_t st, int64_t B = 1,
                       bool batched = false) {
  const int kind = kind_base(kind_flags);
  const int self_mode = (x == y && N == M) ? 1 : 0;  // K_xx / K_yy: the diagonal exponent is exactly 0 (tcconv.cuh)
  const TcPlan p = make_tc_plan(N, M, D, false, B);
  if (p.nstage < 1) return B200OT_EINVAL;
  unsigned char* base = reinterpret_cast<unsigned char*>(scratch);
  unsigned char* a_imgs = base;
  unsigned char* b_imgs = base + p.off_b;
  float* part = reinterpret_cast<float*>(base + p.off_part);
  // gaussian: 2^(-|X-Y|^2/2) with X = x sqrt(log2e) / blur; laplacian / energy: conv_scales' coordinates and clamp
  const ConvScales cs = conv_scales(kind_flags, blur);
  const float scale = kind == B200OT_KERNEL_GAUSSIAN ? sqrtf(kLog2e) / blur : cs.scale;
  const float* coord_absmax = nullptr;
  if (kind == B200OT_KERNEL_ENERGY) {
    const int rc = energy_coord_absmax(x, B * N, y, B * M, D, center, base + p.off_misc, st, &coord_absmax);
    if (rc) return rc;
  }
  const int threads = 128;
  tc_pack_kernel<<<(unsigned)ceil_div64(p.a_tiles * kTcM, threads), threads, 0, st>>>(
      x, nullptr, nullptr, nullptr, 0.f, 0.f, center, scale, N, D, p.kp, kTcM, 0, a_imgs, nullptr, nullptr,
      coord_absmax, B);
  B200OT_CUDA_TRY(cudaGetLastError());
  tc_pack_kernel<<<(unsigned)ceil_div64(p.b_tiles * kTcBN, threads), threads, 0, st>>>(
      y, w, nullptr, nullptr, 0.f, 0.f, center, scale, M, D, p.kp, kTcBN, 1, b_imgs, nullptr, nullptr, coord_absmax,
      B);
  B200OT_CUDA_TRY(cudaGetLastError());
  auto kern = kind == B200OT_KERNEL_GAUSSIAN ? (batched ? tc_reduce_kernel<0, true> : tc_reduce_kernel<0>)
              : kind == B200OT_KERNEL_LAPLACIAN ? (batched ? tc_reduce_kernel<4, true> : tc_reduce_kernel<4>)
                                                : (batched ? tc_reduce_kernel<5, true> : tc_reduce_kernel<5>);
  B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
  dim3 grid((unsigned)p.a_tiles, (unsigned)p.n_split);
  kern<<<grid, kTcThreads, (size_t)p.smem, st>>>(a_imgs, b_imgs, part, B * N, p.kp, p.ctpe, p.tiles_per_split,
                                                 p.nstage, D, self_mode, cs.clampq, coord_absmax, p.rtpe, N, nullptr, nullptr, nullptr);
  B200OT_CUDA_TRY(cudaGetLastError());
  conv_fwd_finalize_kernel<<<(unsigned)ceil_div64(B * N, 256), 256, 0, st>>>(
      part, p.n_split * kTcParts, kind == B200OT_KERNEL_ENERGY ? -1.f : 1.f, out, B * N, coord_absmax);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
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
  const int threads = 256;
  conv_fwd_finalize_kernel<<<(unsigned)ceil_div64(N, threads), threads, 0, (cudaStream_t)stream>>>(
      part, n_part, kind_base(kind) == B200OT_KERNEL_ENERGY ? -1.f : 1.f, out, N);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

B200OT_API int b200ot_kernel_conv_bwd_finalize(const float* part, int32_t n_part, const float* x, const float* center,
                                               const float* grad_out, float* grad_x, int64_t N, int32_t D,
                                               int32_t kind, float blur, void* stream) {
  if (!part || !x || !grad_out || !grad_x || n_part <= 0 || N <= 0 || !supported_simt_dim(D) || !valid_kind(kind))
    return B200OT_EINVAL;
  if (kind_base(kind) != B200OT_KERNEL_ENERGY && !(blur > 0.f)) return B200OT_EINVAL;
  const ConvScales cs = conv_scales(kind, blur);
  const int threads = 256;
  conv_bwd_finalize_kernel<<<(unsigned)ceil_div64(N, threads), threads, 0, (cudaStream_t)stream>>>(
      part, n_part, x, center, grad_out, grad_x, N, D, kind_base(kind), cs.scale, conv_bwd_coef(kind, cs, blur),
      (const float*)nullptr);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

B200OT_API int b200ot_kernel_conv_pack_gather(const float* y, const float* w, const float* center,
                                              const int32_t* src_index, int64_t n_slots, int32_t D, int32_t kind,
                                              float blur, float* cols_out, void* stream) {
  if (!y || !w || !src_index || !cols_out || n_slots <= 0 || !supported_simt_dim(D) || !valid_kind(kind))
    return B200OT_EINVAL;
  if (kind_base(kind) != B200OT_KERNEL_ENERGY && !(blur > 0.f)) return B200OT_EINVAL;
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
  if (kind_base(kind) != B200OT_KERNEL_ENERGY && !(blur > 0.f)) return B200OT_EINVAL;
  if ((((uintptr_t)cols) & 15) || (((uintptr_t)seg) & 15) || (((uintptr_t)pieces) & 7)) return B200OT_EALIGN;
  return conv_partial(kind, backward != 0, ranges_plan(variant, n_seg), (cudaStream_t)stream, x, center,
                      conv_scales(kind, blur), cols, part, N, D, reinterpret_cast<const int4*>(seg),
                      reinterpret_cast<const int2*>(pieces));
}

B200OT_API int b200ot_kernel_conv_fwd(const float* x, const float* y, const float* w, const float* center,
                                      float* out, int64_t N, int64_t M, int32_t D, int32_t kind, float blur,
                                      void* scratch, int64_t scratch_bytes, void* stream) {
  // laplacian / energy: the tensor cores serve 8 < D <= 64 only (no measured cross-over below)
  const bool tc = (kind_base(kind) == B200OT_KERNEL_GAUSSIAN) ? tc_routed(kTcConvFwd, D, N, M)
                                                              : (D > B200OT_MAX_D && tc_capable_dim(D));
  if (!x || !y || !w || !out || !scratch || N <= 0 || M <= 0 || (!supported_simt_dim(D) && !tc) || !valid_kind(kind))
    return B200OT_EINVAL;
  if (kind_base(kind) != B200OT_KERNEL_ENERGY && !(blur > 0.f)) return B200OT_EINVAL;
  if (((uintptr_t)scratch) & 15) return B200OT_EALIGN;
  if (scratch_bytes < b200ot_kernel_conv_scratch_bytes(N, M, D)) return B200OT_ESCRATCH;
  if (tc) return conv_fwd_tc(kind, x, y, w, center, out, N, M, D, blur, scratch, (cudaStream_t)stream);
  const ReducePlan pl = make_plan(N, M, D);
  const ConvScales cs = conv_scales(kind, blur);
  float* cols = reinterpret_cast<float*>(scratch);
  float* part = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) +
                                         round_up64(b200ot_packed_cols_floats(M, D, 2) * 4, 256));
  cudaStream_t st = (cudaStream_t)stream;
  int rc = conv_pack(y, w, center, M, D, cs, cols, st);
  if (rc) return rc;
  rc = conv_partial(kind, false, pl, st, x, center, cs, cols, part, N, D);
  if (rc) return rc;
  return b200ot_kernel_conv_finalize(part, pl.n_split, out, N, kind, stream);
}

// Row gradients on the tensor cores (and, with value_out, the forward values from the same pass: gaussian only), of one
// problem or (`batched`) of B elements of N rows / M columns.  Arguments already validated.
static int conv_bwd_tc(const float* x, const float* y, const float* w, const float* center, const float* grad_out,
                       float* grad_x, float* value_out, int64_t N, int64_t M, int32_t D, int32_t kind, float blur,
                       void* scratch, void* stream, int64_t B = 1, bool batched = false) {
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n_per = batched ? N : 0;  // rows per element: the finalize undoes each element's weight scale
  if (kind_base(kind) != B200OT_KERNEL_GAUSSIAN) {
    // grad = coef (sum_j P Y_j - X_i sum_j P) with P = w k'(d) / d scaled by 2^-kTcNormPLog2 (tcbwd.cuh): the
    // gaussian's finalize with coef = 2^kTcNormPLog2 / blur (laplacian, X = x log2e / blur) or 2^kTcNormPLog2 (energy)
    const int kb = kind_base(kind);
    const ConvScales cs = conv_scales(kind, blur);
    const float* coord_absmax = nullptr;
    if (kb == B200OT_KERNEL_ENERGY) {
      const TcPlan p = make_tc_plan(N, M, D, true, B);
      const int rc = energy_coord_absmax(x, B * N, y, B * M, D, center,
                                         reinterpret_cast<unsigned char*>(scratch) + p.off_misc, st, &coord_absmax);
      if (rc) return rc;
    }
    float* tc_part = nullptr;
    int n_part = 0;
    const float* w_absmax = nullptr;
    const int rc = bwd_partial_tc(kb == B200OT_KERNEL_LAPLACIAN ? 4 : 5, x, y, w, nullptr, nullptr, 0.f, nullptr,
                                  center, cs.scale, N, M, D, scratch, &tc_part, &n_part, st, &w_absmax, cs.clampq,
                                  coord_absmax, B, batched);
    if (rc) return rc;
    const float coef = (float)(1 << kTcNormPLog2) * (kb == B200OT_KERNEL_LAPLACIAN ? 1.0f / blur : 1.0f);
    conv_bwd_finalize_kernel<<<(unsigned)ceil_div64(B * N, 256), 256, 0, st>>>(
        tc_part, n_part, x, center, grad_out, grad_x, B * N, D, B200OT_KERNEL_GAUSSIAN, cs.scale, coef, w_absmax,
        nullptr, coord_absmax, n_per);
    B200OT_CUDA_TRY(cudaGetLastError());
    return B200OT_OK;
  }
  float* tc_part = nullptr;
  int n_part = 0;
  const float scale = sqrtf(kLog2e) / blur;
  const float* w_absmax = nullptr;
  const int rc = bwd_partial_tc(2, x, y, w, nullptr, nullptr, 0.f, nullptr, center, scale, N, M, D, scratch, &tc_part,
                                &n_part, st, &w_absmax, 0.f, nullptr, B, batched);
  if (rc) return rc;
  conv_bwd_finalize_kernel<<<(unsigned)ceil_div64(B * N, 256), 256, 0, st>>>(
      tc_part, n_part, x, center, grad_out, grad_x, B * N, D, 0, scale, 1.0f / (scale * blur * blur), w_absmax,
      value_out, nullptr, n_per);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

// Row gradients (and, with value_out, the forward values from the same pass: gaussian only).
static int conv_bwd_x_impl(const float* x, const float* y, const float* w, const float* center, const float* grad_out,
                           float* grad_x, float* value_out, int64_t N, int64_t M, int32_t D, int32_t kind, float blur,
                           void* scratch, int64_t scratch_bytes, void* stream) {
  const bool gauss = kind_base(kind) == B200OT_KERNEL_GAUSSIAN;
  const bool tc = gauss ? tc_routed(kTcConvBwd, D, N, M) : (D > B200OT_MAX_D && tc_capable_dim(D));
  if (!x || !y || !w || !grad_x || !scratch || N <= 0 || M <= 0 || (!supported_simt_dim(D) && !tc) ||
      !valid_kind(kind) || (value_out && !gauss))
    return B200OT_EINVAL;
  if (kind_base(kind) != B200OT_KERNEL_ENERGY && !(blur > 0.f)) return B200OT_EINVAL;
  if (((uintptr_t)scratch) & 15) return B200OT_EALIGN;
  if (scratch_bytes < b200ot_kernel_conv_scratch_bytes(N, M, D)) return B200OT_ESCRATCH;
  if (tc) return conv_bwd_tc(x, y, w, center, grad_out, grad_x, value_out, N, M, D, kind, blur, scratch, stream);
  const ReducePlan pl = make_plan(N, M, D);
  const ConvScales cs = conv_scales(kind, blur);
  float* cols = reinterpret_cast<float*>(scratch);
  float* part = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) +
                                         round_up64(b200ot_packed_cols_floats(M, D, 2) * 4, 256));
  cudaStream_t st = (cudaStream_t)stream;
  int rc = conv_pack(y, w, center, M, D, cs, cols, st);
  if (rc) return rc;
  rc = conv_partial(kind, true, pl, st, x, center, cs, cols, part, N, D);
  if (rc) return rc;
  conv_bwd_finalize_kernel<<<(unsigned)ceil_div64(N, 256), 256, 0, st>>>(
      part, pl.n_split, x, center, grad_out, grad_x, N, D, kind_base(kind), cs.scale, conv_bwd_coef(kind, cs, blur),
      (const float*)nullptr, value_out);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
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
  return conv_bwd_x_impl(x, y, w, center, nullptr, grad_unit, out, N, M, D, kind, blur, scratch, scratch_bytes,
                         stream);
}

// ---- batches of B problems in the tensor-core dimensions (tc_reduce_kernel / tc_bwd_kernel with BATCH) ----
B200OT_API int64_t b200ot_batched_scratch_bytes(int64_t B, int64_t N, int64_t M, int32_t D) {
  return tc_batched_dims(B, N, M, D) ? tc_scratch_bytes(N, M, D, B) : 0;
}

B200OT_API int b200ot_kernel_conv_fwd_batched(const float* x, const float* y, const float* w, const float* center,
                                              float* out, int64_t B, int64_t N, int64_t M, int32_t D, int32_t kind,
                                              float blur, void* scratch, int64_t scratch_bytes, void* stream) {
  if (!x || !y || !w || !out || !scratch || !tc_batched_dims(B, N, M, D) || !valid_kind(kind)) return B200OT_EINVAL;
  if (kind_base(kind) != B200OT_KERNEL_ENERGY && !(blur > 0.f)) return B200OT_EINVAL;
  if (((uintptr_t)scratch) & 15) return B200OT_EALIGN;
  if (scratch_bytes < b200ot_batched_scratch_bytes(B, N, M, D)) return B200OT_ESCRATCH;
  return conv_fwd_tc(kind, x, y, w, center, out, N, M, D, blur, scratch, (cudaStream_t)stream, B, true);
}

static int conv_bwd_x_batched_impl(const float* x, const float* y, const float* w, const float* center,
                                   const float* grad_out, float* grad_x, float* value_out, int64_t B, int64_t N,
                                   int64_t M, int32_t D, int32_t kind, float blur, void* scratch,
                                   int64_t scratch_bytes, void* stream) {
  if (!x || !y || !w || !grad_x || !scratch || !tc_batched_dims(B, N, M, D) || !valid_kind(kind) ||
      (value_out && kind_base(kind) != B200OT_KERNEL_GAUSSIAN))
    return B200OT_EINVAL;
  if (kind_base(kind) != B200OT_KERNEL_ENERGY && !(blur > 0.f)) return B200OT_EINVAL;
  if (((uintptr_t)scratch) & 15) return B200OT_EALIGN;
  if (scratch_bytes < b200ot_batched_scratch_bytes(B, N, M, D)) return B200OT_ESCRATCH;
  return conv_bwd_tc(x, y, w, center, grad_out, grad_x, value_out, N, M, D, kind, blur, scratch, stream, B, true);
}

B200OT_API int b200ot_kernel_conv_bwd_x_batched(const float* x, const float* y, const float* w, const float* center,
                                                const float* grad_out, float* grad_x, int64_t B, int64_t N, int64_t M,
                                                int32_t D, int32_t kind, float blur, void* scratch,
                                                int64_t scratch_bytes, void* stream) {
  if (!grad_out) return B200OT_EINVAL;
  return conv_bwd_x_batched_impl(x, y, w, center, grad_out, grad_x, nullptr, B, N, M, D, kind, blur, scratch,
                                 scratch_bytes, stream);
}

B200OT_API int b200ot_kernel_conv_fwd_bwd_x_batched(const float* x, const float* y, const float* w,
                                                    const float* center, float* out, float* grad_unit, int64_t B,
                                                    int64_t N, int64_t M, int32_t D, int32_t kind, float blur,
                                                    void* scratch, int64_t scratch_bytes, void* stream) {
  if (!out) return B200OT_EINVAL;
  return conv_bwd_x_batched_impl(x, y, w, center, nullptr, grad_unit, out, B, N, M, D, kind, blur, scratch,
                                 scratch_bytes, stream);
}

}  // extern "C"
