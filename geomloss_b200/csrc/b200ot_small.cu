// b200ot — small problems: ONE launch per symmetric Sinkhorn iteration (and one for the gradient of the final step).
//
// Reference semantics: the body of sinkhorn_loop (src/geomloss/_legacy/sinkhorn_divergence.py:468-493) — the four
// simultaneous updates
//     f_ba <- a0 f_ba + b0 softmin(eps, (x, y), b_log + g_ab/eps)      g_ab <- a0 g_ab + b0 softmin(eps, (y, x), a_log + f_ba/eps)
//     f_aa <- a0 f_aa + b0 softmin(eps, (x, x), a_log + f_aa/eps)      g_bb <- a0 g_bb + b0 softmin(eps, (y, y), b_log + g_bb/eps)
// all read the OLD potentials, so they are independent and run as the y-slices of one grid; batched inputs
// (B, N, D) are the z-slices (the reference's batched tensorized / LazyTensor reductions, sinkhorn_samples.py:70-71,
// :229-290).  This is the regime most users live in (N <= 5 000: doc/index.rst:34), where the tiled TMA kernels
// are launch-bound: 3 launches per softmin, 12 per iteration.  Here an iteration is one launch: no column packing
// (the cost is evaluated by explicit differences straight from the input arrays staged in shared memory), no
// partial (m, s) buffers (a CTA owns 32 rows and ALL columns: its four warps split the columns and merge through
// shared memory), the Sinkhorn prologue h = log_w + pot/eps and the damped / averaged epilogue fused in.
//
// Numerics: explicit differences (exact for coincident points, no expansion), log2 domain, online (max, sum) per
// thread refreshed once per 8 columns, fp32 throughout, final log in fp32 on a sum normalised into [1, 4 * 8).
#include <math.h>

#include "b200ot.h"
#include "common.cuh"
#include "host_util.cuh"

namespace b200ot {

constexpr int kSmallRows = 32;   // rows per CTA (one per lane)
#ifndef B200OT_SMALL_WARPS  // A/B builds: tools/ab_small.py
#define B200OT_SMALL_WARPS 4
#endif
#ifndef B200OT_SMALL_TILE
#define B200OT_SMALL_TILE 256
#endif
constexpr int kSmallWarps = B200OT_SMALL_WARPS;  // warps per CTA: each reduces its share of every column tile
constexpr int kSmallTile = B200OT_SMALL_TILE;    // columns staged per step
static_assert(kSmallTile % (8 * kSmallWarps) == 0 && kSmallTile % (8 * 8) == 0,
              "a warp takes whole 8-column chunks of a tile");

struct SmallProblemSet {
  // per problem q in {0: xy -> f_ba, 1: yx -> g_ab, 2: xx -> f_aa, 3: yy -> g_bb}
  const float* rows[4];
  const float* cols[4];
  const float* logw[4];   // log-weights of the column cloud
  const float* pot[4];    // potential on the column cloud (nullable: h = logw)
  const float* old[4];    // previous value of the output (nullable when alpha_old == 0)
  float* out[4];
  float* lse2[4];         // nullable
  const float* lse2_in[4];   // backward: saved lse2 of the forward final step
  const float* gout[4];      // backward: upstream gradient per row (nullable = zero)
  const float* go_scale;     // backward: per-batch-element factor on every gout (nullable = 1)
  const float* lo_hi;        // (2, D) bounding box of the batch: coordinates are taken from its mid-point (nullable)
  int nrows[4], ncols[4];
};

// Mid-point of the bounding box, subtracted from every coordinate before the scaling, as the tiled kernels do: the
// scaled differences then keep the bits of clouds that lie far from the origin (x - c is exact when x and c agree
// to within a factor of two, the rounded product of a large coordinate is not)
template <int D>
__device__ __forceinline__ void box_centre(const float* __restrict__ lo_hi, float (&C)[D]) {
#pragma unroll
  for (int d = 0; d < D; ++d) C[d] = lo_hi ? 0.5f * (lo_hi[d] + lo_hi[D + d]) : 0.f;
}

// Scaled coordinates are ROUNDED products (__fmul_rn is never contracted).  With a plain `scale * x` the compiler fuses
// the row side into the difference, df = fma(x, scale, -Y), while the column side Y = round(scale * y) went through
// shared memory: a point then sits at distance ~1e-6 (scaled) from ITSELF instead of 0.  Harmless for the values, fatal
// for the p = 1 gradient in the unclamped (pykeops) convention, where only an exact zero distance has a zero gradient:
// the self pair — the heaviest weight of the x <-> x problem — contributed a unit vector of rounding noise
// (tools/debug_p1.py: gradient off by O(1), value correct to 2e-7).
//
// log2-domain log-weight of a column: from a natural-log weight (w_linear = 0), or from the weight itself with the
// reference's floor log_weights(a)[a <= 0] = -100000 (sinkhorn_divergence.py:61-65) — saves the host four tiny
// elementwise launches per cloud
__device__ __forceinline__ float column_log2_weight(float w, int w_linear) {
  if (!w_linear) return w * kLog2e;
  return w > 0.f ? log2f(w) : -100000.0f * kLog2e;
}

template <int D, int P>
__device__ __forceinline__ float pair_exponent_small(const float (&X)[D], const float* __restrict__ c, float H,
                                                     float clampq) {
  float q = 0.f;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    const float df = X[d] - c[d];
    q = fmaf(df, df, q);
  }
  if (P == 2) return fmaf(-0.5f, q, H);
  return H - sqrt_approx(fmaxf(q, clampq));
}

// smem column tile layout: [kSmallTile][D + 1] floats, slot D = H (log2-domain additive term)
// WARPS: 4, or 8 when the grid underfills the machine (launch_iter)
template <int D, int P, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
    sinkhorn_iteration_small_kernel(SmallProblemSet S, float scale, float inv_eps_log2e, float clampq,
                                    float alpha_old, float beta_neg_eps_ln2, int w_linear) {
  constexpr int W = D + 1;
  __shared__ float tile[kSmallTile * W];
  __shared__ float2 red[WARPS][kSmallRows];
  const int q = blockIdx.y;
  const int b = blockIdx.z;
  const int nrows = S.nrows[q], ncols = S.ncols[q];
  const int row0 = blockIdx.x * kSmallRows;
  if (row0 >= nrows) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* __restrict__ rows = S.rows[q] + (int64_t)b * nrows * D;
  const float* __restrict__ cols = S.cols[q] + (int64_t)b * ncols * D;
  const float* __restrict__ logw = S.logw[q] + (int64_t)b * ncols;
  const float* __restrict__ pot = S.pot[q] ? S.pot[q] + (int64_t)b * ncols : nullptr;

  const int i = min(row0 + lane, nrows - 1);
  float X[D], C[D];
  box_centre<D>(S.lo_hi, C);
#pragma unroll
  for (int d = 0; d < D; ++d) X[d] = __fmul_rn(scale, rows[(int64_t)i * D + d] - C[d]);  // (never contracted: see above)

  float m = kNegBig, s = 0.f;
  for (int j0 = 0; j0 < ncols; j0 += kSmallTile) {
    const int nt = min(kSmallTile, ncols - j0);
    __syncthreads();
    for (int e = threadIdx.x; e < kSmallTile; e += WARPS * 32) {
      float* dst = tile + e * W;
      if (e < nt) {
        const int j = j0 + e;
#pragma unroll
        for (int d = 0; d < D; ++d) dst[d] = __fmul_rn(scale, cols[(int64_t)j * D + d] - C[d]);
        float h = column_log2_weight(logw[j], w_linear);
        if (pot) h = fmaf(pot[j], inv_eps_log2e, h);
        dst[D] = h;
      } else {
#pragma unroll
        for (int d = 0; d < D; ++d) dst[d] = 0.f;
        dst[D] = -INFINITY;
      }
    }
    __syncthreads();
    // warp w takes columns [w*64, w*64 + 64) of the tile, 8 at a time
    const int c_begin = warp * (kSmallTile / WARPS);
    const int c_end = min(c_begin + kSmallTile / WARPS, (nt + 7) & ~7);
    for (int c0 = c_begin; c0 < c_end; c0 += 8) {
      float t[8];
      float cm = kNegBig;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float* cp = tile + (c0 + c) * W;
        t[c] = pair_exponent_small<D, P>(X, cp, cp[D], clampq);
        cm = fmaxf(cm, t[c]);
      }
      if (cm > m) {
        s *= ex2_approx(m - cm);
        m = cm;
      }
      float cs = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) cs += ex2_approx(t[c] - m);
      s += cs;
    }
  }
  red[warp][lane] = make_float2(m, s);
  __syncthreads();
  if (warp == 0 && row0 + lane < nrows) {
    float mm = red[0][lane].x;
#pragma unroll
    for (int w = 1; w < WARPS; ++w) mm = fmaxf(mm, red[w][lane].x);
    float ss = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) ss += red[w][lane].y * ex2_approx(red[w][lane].x - mm);
    int e = 0;
    const float fr = frexpf(ss, &e);
    const float lse2 = ss > 0.f ? (mm + (float)e) + log2f(fr) : -INFINITY;
    const int64_t o = (int64_t)b * nrows + row0 + lane;
    if (S.lse2[q]) S.lse2[q][o] = lse2;
    float v = beta_neg_eps_ln2 * lse2;
    if (S.old[q]) v = fmaf(alpha_old, S.old[q][o], v);
    S.out[q][o] = v;
  }
}

// Gradient of the final (gradient-carrying) step w.r.t. the ROW clouds:
//   grad_rows[i] = sum over the problems that share this row cloud of  go_q[i] * sum_j w_ij dC(x_i, y_j)/dx_i,
//   w_ij = 2^(t_ij - lse2_i).   blockIdx.y = 0: rows x (problems xy and xx), 1: rows y (problems yx and yy).
template <int D, int P>
__global__ void __launch_bounds__(kSmallWarps * 32)
    sinkhorn_final_bwd_small_kernel(SmallProblemSet S, float scale, float inv_eps_log2e, float clampq,
                                    float out_scale, float* __restrict__ grad_x, float* __restrict__ grad_y,
                                    int n_terms, int w_linear) {
  constexpr int W = D + 1;
  __shared__ float tile[kSmallTile * W];
  __shared__ float red[kSmallWarps][kSmallRows][D];
  __shared__ float redw[kSmallWarps][kSmallRows];
  const int side = blockIdx.y;  // 0: x rows, 1: y rows
  const int b = blockIdx.z;
  const int nrows = S.nrows[side];
  const int row0 = blockIdx.x * kSmallRows;
  if (row0 >= nrows) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* __restrict__ rows = S.rows[side] + (int64_t)b * nrows * D;
  const int i = min(row0 + lane, nrows - 1);
  float X[D], G[D], C[D];
  box_centre<D>(S.lo_hi, C);
#pragma unroll
  for (int d = 0; d < D; ++d) {
    X[d] = __fmul_rn(scale, rows[(int64_t)i * D + d] - C[d]);  // (never contracted: see scaled_coord)
    G[d] = 0.f;
  }
  for (int term = 0; term < n_terms; ++term) {
    const int q = side + 2 * term;  // 0/1: cross terms, 2/3: self terms
    const float* go_p = S.gout[q];
    if (go_p == nullptr) continue;
    const int ncols = S.ncols[q];
    const float* __restrict__ cols = S.cols[q] + (int64_t)b * ncols * D;
    const float* __restrict__ logw = S.logw[q] + (int64_t)b * ncols;
    const float* __restrict__ pot = S.pot[q] ? S.pot[q] + (int64_t)b * ncols : nullptr;
    const float lse2 = S.lse2_in[q][(int64_t)b * nrows + i];
    const float go = go_p[(int64_t)b * nrows + i] * (S.go_scale ? S.go_scale[b] : 1.0f);
    float A[D];
    float sw = 0.f;
#pragma unroll
    for (int d = 0; d < D; ++d) A[d] = 0.f;
    for (int j0 = 0; j0 < ncols; j0 += kSmallTile) {
      const int nt = min(kSmallTile, ncols - j0);
      __syncthreads();
      for (int e = threadIdx.x; e < kSmallTile; e += kSmallWarps * 32) {
        float* dst = tile + e * W;
        if (e < nt) {
          const int j = j0 + e;
#pragma unroll
          for (int d = 0; d < D; ++d) dst[d] = __fmul_rn(scale, cols[(int64_t)j * D + d] - C[d]);
          float h = column_log2_weight(logw[j], w_linear);
          if (pot) h = fmaf(pot[j], inv_eps_log2e, h);
          dst[D] = h;
        } else {
#pragma unroll
          for (int d = 0; d < D; ++d) dst[d] = 0.f;
          dst[D] = -INFINITY;
        }
      }
      __syncthreads();
      const int c_begin = warp * (kSmallTile / kSmallWarps);
      const int c_end = min(c_begin + kSmallTile / kSmallWarps, nt);
      for (int c = c_begin; c < c_end; ++c) {
        const float* cp = tile + c * W;
        float df[D];
        float qq = 0.f;
#pragma unroll
        for (int d = 0; d < D; ++d) {
          df[d] = X[d] - cp[d];
          qq = fmaf(df[d], df[d], qq);
        }
        float w;
        if (P == 2) {
          w = ex2_approx(fmaf(-0.5f, qq, cp[D]) - lse2);
#pragma unroll
          for (int d = 0; d < D; ++d) A[d] = fmaf(w, df[d], A[d]);  // dC/dx = x - y  (scaled units)
        } else {
          const bool inside = qq < clampq;  // zero gradient inside the clamp (or at coincident points)
          const float qc = fmaxf(qq, clampq);
          const float rinv = rsqrt_approx(qc);
          w = ex2_approx(cp[D] - qc * rinv - lse2);
          const float wr = inside ? 0.f : w * rinv;
#pragma unroll
          for (int d = 0; d < D; ++d) A[d] = fmaf(wr, df[d], A[d]);  // unit vector
        }
        sw += w;
      }
    }
    // merge the four warps' partial sums of this term, then add  go * A / sw  into the row gradient
    __syncthreads();
#pragma unroll
    for (int d = 0; d < D; ++d) red[warp][lane][d] = A[d];
    redw[warp][lane] = sw;
    __syncthreads();
    if (warp == 0) {
      float tw = 0.f;
#pragma unroll
      for (int w = 0; w < kSmallWarps; ++w) tw += redw[w][lane];
      const float inv = tw > 0.f ? go / tw : 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) {
        float a = 0.f;
#pragma unroll
        for (int w = 0; w < kSmallWarps; ++w) a += red[w][lane][d];
        G[d] = fmaf(inv, a, G[d]);
      }
    }
  }
  if (warp == 0 && row0 + lane < nrows) {
    float* g = (side == 0 ? grad_x : grad_y) + ((int64_t)b * nrows + row0 + lane) * D;
    // p = 2: A is in scaled units (X - Y = scale (x - y)): dC/dx = (x - y) = A / scale;  p = 1: unit vectors
    const float k = out_scale * (P == 2 ? 1.0f / scale : 1.0f);
#pragma unroll
    for (int d = 0; d < D; ++d) g[d] = k * G[d];
  }
}

// Warps per CTA (each reduces its share of every column tile; tools/ab_small.py times 4 against 8).  One problem of a
// few thousand points is a grid of N/32 x 4 CTAs that underfills the SMs: 8 warps hide the latency of the tile loads.
// A large batch is thousands of CTAs, the machine is full and the wider CTA only adds barrier and merge cost: 4 warps.
template <int D, int P>
static void launch_iter_p(const SmallProblemSet& S, dim3 grid, float scale, float inv_eps_log2e, float clampq,
                          float alpha_old, float beta_neg_eps_ln2, int w_linear, cudaStream_t st) {
  const int64_t ctas = (int64_t)grid.x * grid.y * grid.z;
  if (ctas <= 1024)
    sinkhorn_iteration_small_kernel<D, P, 8><<<grid, 8 * 32, 0, st>>>(S, scale, inv_eps_log2e, clampq, alpha_old,
                                                                      beta_neg_eps_ln2, w_linear);
  else
    sinkhorn_iteration_small_kernel<D, P, 4><<<grid, 4 * 32, 0, st>>>(S, scale, inv_eps_log2e, clampq, alpha_old,
                                                                      beta_neg_eps_ln2, w_linear);
}

template <int D>
static int launch_iter(int pe, const SmallProblemSet& S, dim3 grid, float scale, float inv_eps_log2e, float clampq,
                       float alpha_old, float beta_neg_eps_ln2, int w_linear, cudaStream_t st) {
  if (pe == 2)
    launch_iter_p<D, 2>(S, grid, scale, inv_eps_log2e, clampq, alpha_old, beta_neg_eps_ln2, w_linear, st);
  else
    launch_iter_p<D, 1>(S, grid, scale, inv_eps_log2e, clampq, alpha_old, beta_neg_eps_ln2, w_linear, st);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

template <int D>
static int launch_bwd(int pe, const SmallProblemSet& S, dim3 grid, float scale, float inv_eps_log2e, float clampq,
                      float out_scale, float* gx, float* gy, int n_terms, int w_linear, cudaStream_t st) {
  if (pe == 2)
    sinkhorn_final_bwd_small_kernel<D, 2><<<grid, kSmallWarps * 32, 0, st>>>(S, scale, inv_eps_log2e, clampq,
                                                                             out_scale, gx, gy, n_terms, w_linear);
  else
    sinkhorn_final_bwd_small_kernel<D, 1><<<grid, kSmallWarps * 32, 0, st>>>(S, scale, inv_eps_log2e, clampq,
                                                                             out_scale, gx, gy, n_terms, w_linear);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

#define B200OT_DISPATCH_D(D, CALL)            \
  switch (D) {                                \
    case 1: return CALL(1);                   \
    case 2: return CALL(2);                   \
    case 3: return CALL(3);                   \
    case 4: return CALL(4);                   \
    case 5: return CALL(5);                   \
    case 6: return CALL(6);                   \
    case 7: return CALL(7);                   \
    case 8: return CALL(8);                   \
    default: return B200OT_EINVAL;            \
  }

// The batch is gridDim.z of the small kernels, at most 65535 elements per launch: a larger batch runs as consecutive
// launches over slices of it.  launch(b0, nb) enqueues the elements [b0, b0 + nb), every per-element array offset to b0.
constexpr int64_t kMaxGridZ = 65535;
constexpr int64_t kMaxGridX = 0x7fffffff;  // the cost kernels: one block per batch element, gridDim.x

template <class F>
static int for_batch_slices(int64_t B, F&& launch) {
  for (int64_t b0 = 0; b0 < B; b0 += kMaxGridZ) {
    const int rc = launch(b0, B - b0 < kMaxGridZ ? B - b0 : kMaxGridZ);
    if (rc != B200OT_OK) return rc;
  }
  return B200OT_OK;
}

template <class T>
static T* skip(T* p, int64_t n) {
  return p ? p + n : p;
}

// the problems of batch elements [b0, B) of S (lse2 / lse2_in point into their own [f_ba | g_ab | f_aa | g_bb] block,
// whose offsets already account for the whole batch)
static SmallProblemSet batch_slice(const SmallProblemSet& S, int64_t b0, int D) {
  SmallProblemSet T = S;
  for (int q = 0; q < 4; ++q) {
    const int64_t r = b0 * S.nrows[q], c = b0 * S.ncols[q];
    T.rows[q] = skip(S.rows[q], r * D);
    T.cols[q] = skip(S.cols[q], c * D);
    T.logw[q] = skip(S.logw[q], c);
    T.pot[q] = skip(S.pot[q], c);
    T.old[q] = skip(S.old[q], r);
    T.out[q] = skip(S.out[q], r);
    T.lse2[q] = skip(S.lse2[q], r);
    T.lse2_in[q] = skip(S.lse2_in[q], r);
    T.gout[q] = skip(S.gout[q], r);
  }
  T.go_scale = skip(S.go_scale, b0);
  return T;
}

static void fill_problems(SmallProblemSet& S, const float* x, const float* y, const float* a_log, const float* b_log,
                          const float* f_ba, const float* g_ab, const float* f_aa, const float* g_bb, int N, int M) {
  const float* rows[4] = {x, y, x, y};
  const float* cols[4] = {y, x, x, y};
  const float* logw[4] = {b_log, a_log, a_log, b_log};
  const float* pot[4] = {g_ab, f_ba, f_aa, g_bb};
  const int nr[4] = {N, M, N, M}, nc[4] = {M, N, N, M};
  for (int q = 0; q < 4; ++q) {
    S.rows[q] = rows[q];
    S.cols[q] = cols[q];
    S.logw[q] = logw[q];
    S.pot[q] = pot[q];
    S.nrows[q] = nr[q];
    S.ncols[q] = nc[q];
    S.old[q] = nullptr;
    S.out[q] = nullptr;
    S.lse2[q] = nullptr;
    S.lse2_in[q] = nullptr;
    S.gout[q] = nullptr;
  }
  S.go_scale = nullptr;
  S.lo_hi = nullptr;
}

// ---------------------------------------------------------------------------------------------------------------
// sinkhorn_cost on small clouds (sinkhorn_divergence.py:165-255, scal(batch=True) of utils.py:13-18): one block per
// batch element, fixed-order reduction (bitwise reproducible).
//   balanced    value = <a, f_ba - f_aa> + <b, g_ab - g_bb>                          (no debias: <a, f_ba> + <b, g_ab>)
//   unbalanced  value = <a, w (e^{-f_aa/rho} - e^{-f_ba/rho})> + <b, ...>,  w = rho + eps/2   (no debias: w (1 - e^{-f_ba/rho}))
// Optionally writes d value / d potential (the `go_*` inputs of b200ot_sinkhorn_final_bwd_small) and the per-point
// terms phi = d value / d a_i, psi = d value / d b_j.
// ---------------------------------------------------------------------------------------------------------------
struct SmallCostSet {
  const float* w[2];     // a (B, N), b (B, M)
  const float* cross[2]; // f_ba, g_ab
  const float* self[2];  // f_aa, g_bb (nullable: no debias)
  float* go_cross[2];    // nullable
  float* go_self[2];     // nullable
  float* term[2];        // phi, psi (nullable)
  float c_cross, c_self; // balanced mode: t = c_cross * cross - c_self * self
  int n[2];
};

__global__ void __launch_bounds__(256) sinkhorn_cost_small_kernel(SmallCostSet S, float rho, float wgt,
                                                                  float* __restrict__ value) {
  __shared__ float red[8];
  const int b = blockIdx.x;
  const bool unb = rho > 0.f;
  const float inv_rho = unb ? 1.0f / rho : 0.f;
  float acc = 0.f;
  for (int side = 0; side < 2; ++side) {
    const int n = S.n[side];
    const int64_t base = (int64_t)b * n;
    for (int i = threadIdx.x; i < n; i += 256) {
      const float w = S.w[side][base + i];
      const float fc = S.cross[side][base + i];
      const bool deb = S.self[side] != nullptr;
      const float fs = deb ? S.self[side][base + i] : 0.f;
      float t, gc, gs;
      if (unb) {
        const float ec = expf(-fc * inv_rho), es = deb ? expf(-fs * inv_rho) : 1.0f;
        t = wgt * (es - ec);
        gc = wgt * inv_rho * ec;
        gs = -wgt * inv_rho * es;
      } else {
        t = S.c_cross * fc - S.c_self * fs;
        gc = S.c_cross;
        gs = -S.c_self;
      }
      acc = fmaf(w, t, acc);
      if (S.go_cross[side]) S.go_cross[side][base + i] = w * gc;
      if (deb && S.go_self[side]) S.go_self[side][base + i] = w * gs;
      if (S.term[side]) S.term[side][base + i] = t;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) v += red[k];
    value[b] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Bounding box of two clouds (sinkhorn_divergence.py:96-112, max_diameter): lo[D], hi[D] over the rows of x and y in
// ONE launch (torch: four reductions, two elementwise kernels, a norm).  Blocks publish their partial boxes; the last
// block to finish folds them.  The ticket counter lives in the caller's scratch (zero before the first use; the last
// block puts it back to zero), so launches on different scratch buffers never share state.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kExtentBlocks = 64;

__global__ void __launch_bounds__(256) cloud_extent_kernel(const float* __restrict__ x, int64_t n,
                                                           const float* __restrict__ y, int64_t m, int D,
                                                           float* __restrict__ partial, unsigned int* ticket,
                                                           float* __restrict__ out) {
  __shared__ float slo[8][B200OT_MAX_D], shi[8][B200OT_MAX_D];
  __shared__ bool last;
  float lo[B200OT_MAX_D], hi[B200OT_MAX_D];
  for (int d = 0; d < B200OT_MAX_D; ++d) {
    lo[d] = INFINITY;
    hi[d] = -INFINITY;
  }
  const int64_t stride = (int64_t)gridDim.x * 256;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n + m; i += stride) {
    const float* pnt = i < n ? x + i * D : y + (i - n) * D;
    for (int d = 0; d < D; ++d) {
      const float v = pnt[d];
      lo[d] = fminf(lo[d], v);
      hi[d] = fmaxf(hi[d], v);
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto block_fold = [&]() {
    for (int d = 0; d < D; ++d) {
      for (int o = 16; o > 0; o >>= 1) {
        lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
        hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
      }
      if (lane == 0) {
        slo[warp][d] = lo[d];
        shi[warp][d] = hi[d];
      }
    }
    __syncthreads();
    if (threadIdx.x < D) {
      float a = slo[0][threadIdx.x], c = shi[0][threadIdx.x];
      for (int w = 1; w < 8; ++w) {
        a = fminf(a, slo[w][threadIdx.x]);
        c = fmaxf(c, shi[w][threadIdx.x]);
      }
      slo[0][threadIdx.x] = a;
      shi[0][threadIdx.x] = c;
    }
    __syncthreads();
  };
  block_fold();
  if (threadIdx.x < D) {
    partial[(blockIdx.x * 2 + 0) * B200OT_MAX_D + threadIdx.x] = slo[0][threadIdx.x];
    partial[(blockIdx.x * 2 + 1) * B200OT_MAX_D + threadIdx.x] = shi[0][threadIdx.x];
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int d = 0; d < B200OT_MAX_D; ++d) {
    lo[d] = INFINITY;
    hi[d] = -INFINITY;
  }
  for (int k = threadIdx.x; k < (int)gridDim.x; k += 256)
    for (int d = 0; d < D; ++d) {
      lo[d] = fminf(lo[d], __ldcg(&partial[(k * 2 + 0) * B200OT_MAX_D + d]));
      hi[d] = fmaxf(hi[d], __ldcg(&partial[(k * 2 + 1) * B200OT_MAX_D + d]));
    }
  __syncthreads();
  block_fold();
  if (threadIdx.x < D) {
    out[threadIdx.x] = slo[0][threadIdx.x];
    out[D + threadIdx.x] = shi[0][threadIdx.x];
  }
  if (threadIdx.x == 0) *ticket = 0;
}


// ---------------------------------------------------------------------------------------------------------------
// Kernel norms on small clouds: the three (four) matvecs of kernel_loss (kernel_samples.py:116-137) in ONE launch,
// their four row gradients in one more.
//   forward   q = 0: a_x = K(x, x) a     1: b_y = K(y, y) b     2: b_x = K(x, y) b     3: a_y = K(y, x) a
//   backward  side 0 (rows x): gx_i = c_i ( sum_j a_j d1 k(x_i, x_j) - sum_j b_j d1 k(x_i, y_j) ),  c_i = go a_i
//             side 1 (rows y): gy_j = c_j ( sum_i b_i d1 k(y_j, y_i) - sum_i a_i d1 k(y_j, x_i) ),  c_j = go b_j
// which is the gradient of  1/2 <dg(a), K_xx a> + 1/2 <dg(b), K_yy b> - <a, K_xy b>  with the reference's DoubleGrad /
// detach pattern (kernel_samples.py:43-54, :116-146).
// ---------------------------------------------------------------------------------------------------------------
struct SmallConvSet {
  const float* rows[4];
  const float* cols[4];
  const float* w[4];
  float* out[4];
  int nrows[4], ncols[4];
};

// KIND 0 gaussian: X = x sqrt(log2e)/blur, k = 2^(-|X-Y|^2/2);  1 laplacian: X = x log2e/blur, k = 2^(-|X-Y|);
// 2 energy: X = x, k = -|X-Y|
template <int D, int KIND>
__global__ void __launch_bounds__(kSmallWarps * 32)
    kernel_mmd_small_kernel(SmallConvSet S, float scale, float clampq) {
  constexpr int W = D + 1;
  __shared__ float tile[kSmallTile * W];
  __shared__ float red[kSmallWarps][kSmallRows];
  const int q = blockIdx.y, b = blockIdx.z;
  const int nrows = S.nrows[q], ncols = S.ncols[q];
  const int row0 = blockIdx.x * kSmallRows;
  if (row0 >= nrows) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* __restrict__ rows = S.rows[q] + (int64_t)b * nrows * D;
  const float* __restrict__ cols = S.cols[q] + (int64_t)b * ncols * D;
  const float* __restrict__ wts = S.w[q] + (int64_t)b * ncols;
  const int i = min(row0 + lane, nrows - 1);
  float X[D];
#pragma unroll
  for (int d = 0; d < D; ++d) X[d] = __fmul_rn(scale, rows[(int64_t)i * D + d]);  // (never contracted: see scaled_coord)
  float acc = 0.f;
  for (int j0 = 0; j0 < ncols; j0 += kSmallTile) {
    const int nt = min(kSmallTile, ncols - j0);
    __syncthreads();
    for (int e = threadIdx.x; e < kSmallTile; e += kSmallWarps * 32) {
      float* dst = tile + e * W;
      const bool live = e < nt;
#pragma unroll
      for (int d = 0; d < D; ++d) dst[d] = live ? __fmul_rn(scale, cols[(int64_t)(j0 + e) * D + d]) : 0.f;
      dst[D] = live ? wts[j0 + e] : 0.f;
    }
    __syncthreads();
    const int c_begin = warp * (kSmallTile / kSmallWarps);
    const int c_end = min(c_begin + kSmallTile / kSmallWarps, nt);
#pragma unroll 4
    for (int c = c_begin; c < c_end; ++c) {
      const float* cp = tile + c * W;
      float qq = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) {
        const float df = X[d] - cp[d];
        qq = fmaf(df, df, qq);
      }
      float k;
      if (KIND == 0) {
        k = ex2_approx(-0.5f * qq);
      } else {
        const float dist = sqrt_approx(fmaxf(qq, clampq));
        k = (KIND == 1) ? ex2_approx(-dist) : -dist;
      }
      acc = fmaf(k, cp[D], acc);
    }
  }
  red[warp][lane] = acc;
  __syncthreads();
  if (warp == 0 && row0 + lane < nrows) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kSmallWarps; ++w) t += red[w][lane];
    S.out[q][(int64_t)b * nrows + row0 + lane] = t;
  }
}

struct SmallConvBwd {
  const float* x;
  const float* y;
  const float* a;
  const float* b;
  const float* go;  // (B,) upstream gradient of the value
  float* gx;
  float* gy;
  int N, M;
};

template <int D, int KIND>
__global__ void __launch_bounds__(kSmallWarps * 32)
    kernel_mmd_bwd_small_kernel(SmallConvBwd S, float scale, float clampq, float coef) {
  constexpr int W = D + 1;
  __shared__ float tile[kSmallTile * W];
  __shared__ float red[kSmallWarps][kSmallRows][D];
  const int side = blockIdx.y, b = blockIdx.z;
  const int nrows = side == 0 ? S.N : S.M;
  const int row0 = blockIdx.x * kSmallRows;
  if (row0 >= nrows) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* __restrict__ rows = (side == 0 ? S.x : S.y) + (int64_t)b * nrows * D;
  const float* __restrict__ roww = (side == 0 ? S.a : S.b) + (int64_t)b * nrows;
  const int i = min(row0 + lane, nrows - 1);
  float X[D], A[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    X[d] = __fmul_rn(scale, rows[(int64_t)i * D + d]);  // (never contracted: see scaled_coord)
    A[d] = 0.f;
  }
  for (int term = 0; term < 2; ++term) {
    // term 0: the self term (same cloud, +), term 1: the cross term (other cloud, -)
    const bool other = (term == 1);
    const int ncols = (side == 0) != other ? S.N : S.M;
    const float* __restrict__ cols = ((side == 0) != other ? S.x : S.y) + (int64_t)b * ncols * D;
    const float* __restrict__ wts = ((side == 0) != other ? S.a : S.b) + (int64_t)b * ncols;
    const float sign = other ? -1.f : 1.f;
    for (int j0 = 0; j0 < ncols; j0 += kSmallTile) {
      const int nt = min(kSmallTile, ncols - j0);
      __syncthreads();
      for (int e = threadIdx.x; e < kSmallTile; e += kSmallWarps * 32) {
        float* dst = tile + e * W;
        const bool live = e < nt;
#pragma unroll
        for (int d = 0; d < D; ++d) dst[d] = live ? __fmul_rn(scale, cols[(int64_t)(j0 + e) * D + d]) : 0.f;
        dst[D] = live ? sign * wts[j0 + e] : 0.f;
      }
      __syncthreads();
      const int c_begin = warp * (kSmallTile / kSmallWarps);
      const int c_end = min(c_begin + kSmallTile / kSmallWarps, nt);
#pragma unroll 2
      for (int c = c_begin; c < c_end; ++c) {
        const float* cp = tile + c * W;
        float df[D];
        float qq = 0.f;
#pragma unroll
        for (int d = 0; d < D; ++d) {
          df[d] = X[d] - cp[d];
          qq = fmaf(df[d], df[d], qq);
        }
        float g;  // d1 k(x, y) = g * (X - Y) up to the constant `coef`
        if (KIND == 0) {
          g = ex2_approx(-0.5f * qq);
        } else {
          const bool inside = qq < clampq;
          const float qc = fmaxf(qq, clampq);
          const float rinv = rsqrt_approx(qc);
          g = (KIND == 1) ? ex2_approx(-qc * rinv) * rinv : rinv;
          if (inside) g = 0.f;
        }
        g *= cp[D];
#pragma unroll
        for (int d = 0; d < D; ++d) A[d] = fmaf(g, df[d], A[d]);
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int d = 0; d < D; ++d) red[warp][lane][d] = A[d];
  __syncthreads();
  if (warp == 0 && row0 + lane < nrows) {
    const float c = coef * S.go[b] * roww[row0 + lane];
    float* g = (side == 0 ? S.gx : S.gy) + ((int64_t)b * nrows + row0 + lane) * D;
#pragma unroll
    for (int d = 0; d < D; ++d) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kSmallWarps; ++w) t += red[w][lane][d];
      g[d] = c * t;
    }
  }
}

template <int D>
static int launch_mmd(int kind, const SmallConvSet& S, dim3 grid, float scale, float clampq, cudaStream_t st) {
  if (kind == B200OT_KERNEL_GAUSSIAN)
    kernel_mmd_small_kernel<D, 0><<<grid, kSmallWarps * 32, 0, st>>>(S, scale, clampq);
  else if (kind == B200OT_KERNEL_LAPLACIAN)
    kernel_mmd_small_kernel<D, 1><<<grid, kSmallWarps * 32, 0, st>>>(S, scale, clampq);
  else
    kernel_mmd_small_kernel<D, 2><<<grid, kSmallWarps * 32, 0, st>>>(S, scale, clampq);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

template <int D>
static int launch_mmd_bwd(int kind, const SmallConvBwd& S, dim3 grid, float scale, float clampq, float coef,
                          cudaStream_t st) {
  if (kind == B200OT_KERNEL_GAUSSIAN)
    kernel_mmd_bwd_small_kernel<D, 0><<<grid, kSmallWarps * 32, 0, st>>>(S, scale, clampq, coef);
  else if (kind == B200OT_KERNEL_LAPLACIAN)
    kernel_mmd_bwd_small_kernel<D, 1><<<grid, kSmallWarps * 32, 0, st>>>(S, scale, clampq, coef);
  else
    kernel_mmd_bwd_small_kernel<D, 2><<<grid, kSmallWarps * 32, 0, st>>>(S, scale, clampq, coef);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

// coordinate scale and clamp (scaled units) of a kernel kind — same conventions as b200ot_kernel_conv.cu
static void mmd_scales(int kind_flags, float blur, float* scale, float* clampq) {
  const int kind = kind_flags & 0xff;
  const float clamp = cost_clamp(kind_flags);
  if (kind == B200OT_KERNEL_GAUSSIAN) {
    *scale = sqrtf(kLog2e) / blur;
    *clampq = 0.f;
  } else if (kind == B200OT_KERNEL_LAPLACIAN) {
    *scale = kLog2e / blur;
    *clampq = kLog2e * kLog2e * clamp;
  } else {
    *scale = 1.f;
    *clampq = clamp;
  }
}

}  // namespace b200ot

using namespace b200ot;

extern "C" {

B200OT_API int b200ot_sinkhorn_iteration_small(const float* x, const float* y, const float* a_log, const float* b_log,
                                               const float* f_ba, const float* g_ab, const float* f_aa,
                                               const float* g_bb, float* f_ba_out, float* g_ab_out, float* f_aa_out,
                                               float* g_bb_out, float* lse2_out, int64_t B, int64_t N, int64_t M,
                                               int32_t D, int32_t p, float eps, float alpha_old, float beta,
                                               int32_t weights_linear, const float* lo_hi, void* stream) {
  if (!x || !y || !a_log || !b_log || !f_ba_out || !g_ab_out || B <= 0 || N <= 0 || M <= 0 ||
      N > B200OT_SMALL_MAX_POINTS || M > B200OT_SMALL_MAX_POINTS || !supported_simt_dim(D) || !valid_p(p) ||
      !(eps > 0.f) || ((f_aa_out == nullptr) != (g_bb_out == nullptr)))
    return B200OT_EINVAL;
  // old potentials: all present (an iteration) or all absent (the initialisation, h = log-weights, alpha_old = 0)
  const bool has_old = f_ba && g_ab;
  if (!has_old && (f_ba || g_ab || f_aa || g_bb || alpha_old != 0.f)) return B200OT_EINVAL;
  const bool debias = f_aa_out != nullptr;
  if (has_old && debias && (!f_aa || !g_bb)) return B200OT_EINVAL;
  SmallProblemSet S;
  fill_problems(S, x, y, a_log, b_log, f_ba, g_ab, f_aa, g_bb, (int)N, (int)M);
  S.lo_hi = lo_hi;
  const float* old[4] = {f_ba, g_ab, f_aa, g_bb};
  float* out[4] = {f_ba_out, g_ab_out, f_aa_out, g_bb_out};
  for (int q = 0; q < 4; ++q) {
    S.old[q] = (alpha_old != 0.f) ? old[q] : nullptr;
    S.out[q] = out[q];
    const int64_t off[4] = {0, B * N, B * (N + M), B * (2 * N + M)};
    S.lse2[q] = lse2_out ? lse2_out + off[q] : nullptr;
  }
  const int pe = p_exponent(p);
  const float scale = softmin_coord_scale(pe, eps);
  const float clampq = scale * scale * cost_clamp(p);
  const int64_t tiles = ceil_div64(N > M ? N : M, kSmallRows);
  const float bneg = -beta * eps * kLn2;
  cudaStream_t st = (cudaStream_t)stream;
  return for_batch_slices(B, [&](int64_t b0, int64_t nb) {
    const SmallProblemSet T = batch_slice(S, b0, D);
    const dim3 grid((unsigned)tiles, debias ? 4u : 2u, (unsigned)nb);
#define CALL(DD) launch_iter<DD>(pe, T, grid, scale, kLog2e / eps, clampq, alpha_old, bneg, weights_linear, st)
    B200OT_DISPATCH_D(D, CALL)
#undef CALL
  });
}

B200OT_API int b200ot_sinkhorn_final_bwd_small(const float* x, const float* y, const float* a_log, const float* b_log,
                                               const float* f_ba, const float* g_ab, const float* f_aa,
                                               const float* g_bb, const float* lse2, const float* go_f_ba,
                                               const float* go_g_ab, const float* go_f_aa, const float* go_g_bb,
                                               float* grad_x, float* grad_y, int64_t B, int64_t N, int64_t M,
                                               int32_t D, int32_t p, float eps, float scale_out,
                                               const float* go_scale, int32_t weights_linear, const float* lo_hi,
                                               void* stream) {
  if (!x || !y || !a_log || !b_log || !lse2 || !grad_x || !grad_y || B <= 0 || N <= 0 || M <= 0 ||
      N > B200OT_SMALL_MAX_POINTS || M > B200OT_SMALL_MAX_POINTS || !supported_simt_dim(D) || !valid_p(p) ||
      !(eps > 0.f))
    return B200OT_EINVAL;
  SmallProblemSet S;
  fill_problems(S, x, y, a_log, b_log, f_ba, g_ab, f_aa, g_bb, (int)N, (int)M);
  const float* go[4] = {go_f_ba, go_g_ab, go_f_aa, go_g_bb};
  const int64_t off[4] = {0, B * N, B * (N + M), B * (2 * N + M)};
  for (int q = 0; q < 4; ++q) {
    S.gout[q] = go[q];
    S.lse2_in[q] = lse2 + off[q];
  }
  S.go_scale = go_scale;
  S.lo_hi = lo_hi;
  const int n_terms = (go_f_aa || go_g_bb) ? 2 : 1;
  const int pe = p_exponent(p);
  const float scale = softmin_coord_scale(pe, eps);
  const float clampq = scale * scale * cost_clamp(p);
  const int64_t tiles = ceil_div64(N > M ? N : M, kSmallRows);
  cudaStream_t st = (cudaStream_t)stream;
  return for_batch_slices(B, [&](int64_t b0, int64_t nb) {
    const SmallProblemSet T = batch_slice(S, b0, D);
    float* gx = grad_x + b0 * N * D;
    float* gy = grad_y + b0 * M * D;
    const dim3 grid((unsigned)tiles, 2u, (unsigned)nb);
#define CALL(DD) launch_bwd<DD>(pe, T, grid, scale, kLog2e / eps, clampq, scale_out, gx, gy, n_terms, weights_linear, st)
    B200OT_DISPATCH_D(D, CALL)
#undef CALL
  });
}

B200OT_API int b200ot_sinkhorn_cost_small(const float* a, const float* b, const float* f_ba, const float* g_ab,
                                          const float* f_aa, const float* g_bb, int64_t B, int64_t N, int64_t M,
                                          float rho, float eps, float* value, float* go_f_ba, float* go_g_ab,
                                          float* go_f_aa, float* go_g_bb, float* phi, float* psi, void* stream) {
  if (!a || !b || !f_ba || !g_ab || !value || B <= 0 || N <= 0 || M <= 0 || B > kMaxGridX ||
      N > B200OT_SMALL_MAX_POINTS || M > B200OT_SMALL_MAX_POINTS || (f_aa == nullptr) != (g_bb == nullptr))
    return B200OT_EINVAL;
  SmallCostSet S;
  S.w[0] = a, S.w[1] = b;
  S.cross[0] = f_ba, S.cross[1] = g_ab;
  S.self[0] = f_aa, S.self[1] = g_bb;
  S.go_cross[0] = go_f_ba, S.go_cross[1] = go_g_ab;
  S.go_self[0] = go_f_aa, S.go_self[1] = go_g_bb;
  S.term[0] = phi, S.term[1] = psi;
  S.c_cross = S.c_self = 1.0f;
  S.n[0] = (int)N, S.n[1] = (int)M;
  sinkhorn_cost_small_kernel<<<(unsigned)B, 256, 0, (cudaStream_t)stream>>>(S, rho, rho > 0.f ? rho + 0.5f * eps : 0.f,
                                                                            value);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

B200OT_API int b200ot_kernel_mmd_value_small(const float* a, const float* b, const float* a_x, const float* b_y,
                                             const float* b_x, int64_t B, int64_t N, int64_t M, float* value,
                                             void* stream) {
  if (!a || !b || !a_x || !b_y || !b_x || !value || B <= 0 || N <= 0 || M <= 0 || B > kMaxGridX ||
      N > B200OT_SMALL_MAX_POINTS || M > B200OT_SMALL_MAX_POINTS)
    return B200OT_EINVAL;
  // 1/2 <a, a_x> + 1/2 <b, b_y> - <a, b_x>  =  <a, 1/2 a_x - b_x> + <b, 1/2 b_y>: coefficients (1/2, 1), the `self` slot
  // carries b_x on the a side only
  SmallCostSet S;
  S.w[0] = a, S.w[1] = b;
  S.cross[0] = a_x, S.cross[1] = b_y;
  S.self[0] = b_x, S.self[1] = nullptr;
  S.go_cross[0] = S.go_cross[1] = S.go_self[0] = S.go_self[1] = nullptr;
  S.term[0] = S.term[1] = nullptr;
  S.c_cross = 0.5f, S.c_self = 1.0f;
  S.n[0] = (int)N, S.n[1] = (int)M;
  sinkhorn_cost_small_kernel<<<(unsigned)B, 256, 0, (cudaStream_t)stream>>>(S, -1.0f, 0.f, value);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

B200OT_API int64_t b200ot_cloud_extent_scratch_bytes(void) {
  return (int64_t)kExtentBlocks * 2 * B200OT_MAX_D * 4 + 16;
}

B200OT_API int b200ot_cloud_extent(const float* x, int64_t n, const float* y, int64_t m, int32_t D, float* lo_hi,
                                   void* scratch, int64_t scratch_bytes, void* stream) {
  if (!x || !lo_hi || !scratch || n <= 0 || m < 0 || (m > 0 && !y) || D < 1 || D > B200OT_MAX_D ||
      scratch_bytes < b200ot_cloud_extent_scratch_bytes())
    return B200OT_EINVAL;
  int64_t blocks = ceil_div64(n + m, 256 * 8);
  if (blocks > kExtentBlocks) blocks = kExtentBlocks;
  float* partial = (float*)scratch;
  unsigned int* ticket = (unsigned int*)(partial + kExtentBlocks * 2 * B200OT_MAX_D);
  cloud_extent_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, n, y, m, D, partial, ticket, lo_hi);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

B200OT_API int b200ot_sinkhorn_loop_small(const float* x, const float* y, const float* a, const float* b,
                                          int32_t weights_linear, const double* eps_list, int32_t n_eps, double rho,
                                          int32_t debias, float* pots_a, float* pots_b, int32_t* result_in_a,
                                          int64_t B, int64_t N, int64_t M, int32_t D, int32_t p,
                                          const float* lo_hi, void* stream) {
  if (!eps_list || n_eps <= 0 || !pots_a || !pots_b || !result_in_a || pots_a == pots_b) return B200OT_EINVAL;
  auto view = [&](float* base, float** f_ba, float** g_ab, float** f_aa, float** g_bb) {
    *f_ba = base;
    *g_ab = base + B * N;
    *f_aa = debias ? base + B * (N + M) : nullptr;
    *g_bb = debias ? base + B * (2 * N + M) : nullptr;
  };
  auto damp = [&](double eps) { return rho > 0.0 ? 1.0 / (1.0 + eps / rho) : 1.0; };
  float *c0, *c1, *c2, *c3, *n0, *n1, *n2, *n3;
  float* cur = pots_a;
  float* nxt = pots_b;
  view(cur, &c0, &c1, &c2, &c3);
  // initialisation at the first temperature (sinkhorn_divergence.py:461-465): h = log-weights only
  int rc = b200ot_sinkhorn_iteration_small(x, y, a, b, nullptr, nullptr, nullptr, nullptr, c0, c1, c2, c3, nullptr, B, N, M,
                                           D, p, (float)eps_list[0], 0.f, (float)damp(eps_list[0]), weights_linear,
                                           lo_hi, stream);
  if (rc) return rc;
  // eps-scaling descent (:468-493): symmetric, averaged updates
  for (int i = 0; i < n_eps; ++i) {
    const double eps = eps_list[i];
    view(cur, &c0, &c1, &c2, &c3);
    view(nxt, &n0, &n1, &n2, &n3);
    rc = b200ot_sinkhorn_iteration_small(x, y, a, b, c0, c1, c2, c3, n0, n1, n2, n3, nullptr, B, N, M, D, p, (float)eps,
                                         0.5f, (float)(0.5 * damp(eps)), weights_linear, lo_hi, stream);
    if (rc) return rc;
    float* t = cur;
    cur = nxt;
    nxt = t;
  }
  *result_in_a = (cur == pots_a) ? 1 : 0;
  return B200OT_OK;
}

B200OT_API int b200ot_kernel_mmd_small(const float* x, const float* y, const float* a, const float* b, float* a_x,
                                       float* b_y, float* b_x, float* a_y, int64_t B, int64_t N, int64_t M, int32_t D,
                                       int32_t kind, float blur, void* stream) {
  const int kb = kind & 0xff;
  if (!x || !y || !a || !b || !a_x || !b_y || !b_x || B <= 0 || N <= 0 || M <= 0 ||
      N > B200OT_SMALL_MAX_POINTS || M > B200OT_SMALL_MAX_POINTS || !supported_simt_dim(D) || kb < 0 || kb > 2 ||
      (kind & ~(0xff | B200OT_KERNEL_UNCLAMPED)) != 0 || (kb != B200OT_KERNEL_ENERGY && !(blur > 0.f)))
    return B200OT_EINVAL;
  SmallConvSet S;
  const float* rows[4] = {x, y, x, y};
  const float* cols[4] = {x, y, y, x};
  const float* w[4] = {a, b, b, a};
  float* out[4] = {a_x, b_y, b_x, a_y};
  const int nr[4] = {(int)N, (int)M, (int)N, (int)M}, nc[4] = {(int)N, (int)M, (int)M, (int)N};
  for (int q = 0; q < 4; ++q) {
    S.rows[q] = rows[q];
    S.cols[q] = cols[q];
    S.w[q] = w[q];
    S.out[q] = out[q];
    S.nrows[q] = nr[q];
    S.ncols[q] = nc[q];
  }
  float scale, clampq;
  mmd_scales(kind, blur, &scale, &clampq);
  const int64_t tiles = ceil_div64(N > M ? N : M, kSmallRows);
  cudaStream_t st = (cudaStream_t)stream;
  return for_batch_slices(B, [&](int64_t b0, int64_t nb) {
    SmallConvSet T = S;
    for (int q = 0; q < 4; ++q) {
      T.rows[q] = S.rows[q] + b0 * S.nrows[q] * D;
      T.cols[q] = S.cols[q] + b0 * S.ncols[q] * D;
      T.w[q] = S.w[q] + b0 * S.ncols[q];
      T.out[q] = skip(S.out[q], b0 * S.nrows[q]);
    }
    const dim3 grid((unsigned)tiles, a_y ? 4u : 3u, (unsigned)nb);
#define CALL(DD) launch_mmd<DD>(kb, T, grid, scale, clampq, st)
    B200OT_DISPATCH_D(D, CALL)
#undef CALL
  });
}

B200OT_API int b200ot_kernel_mmd_bwd_small(const float* x, const float* y, const float* a, const float* b,
                                           const float* grad_value, float* grad_x, float* grad_y, int64_t B, int64_t N,
                                           int64_t M, int32_t D, int32_t kind, float blur, void* stream) {
  const int kb = kind & 0xff;
  if (!x || !y || !a || !b || !grad_value || !grad_x || !grad_y || B <= 0 || N <= 0 || M <= 0 ||
      N > B200OT_SMALL_MAX_POINTS || M > B200OT_SMALL_MAX_POINTS || !supported_simt_dim(D) || kb < 0 || kb > 2 ||
      (kind & ~(0xff | B200OT_KERNEL_UNCLAMPED)) != 0 || (kb != B200OT_KERNEL_ENERGY && !(blur > 0.f)))
    return B200OT_EINVAL;
  SmallConvBwd S;
  S.x = x;
  S.y = y;
  S.a = a;
  S.b = b;
  S.go = grad_value;
  S.gx = grad_x;
  S.gy = grad_y;
  S.N = (int)N;
  S.M = (int)M;
  float scale, clampq;
  mmd_scales(kind, blur, &scale, &clampq);
  // d1 k(x, y): gaussian -k (x - y)/blur^2 = -(k (X - Y)) / (scale blur^2); laplacian -k (x - y)/(blur |x - y|)
  // = -(k (X - Y)/|X - Y|) / blur; energy -(x - y)/|x - y|
  const float coef = kb == B200OT_KERNEL_GAUSSIAN ? -1.0f / (scale * blur * blur)
                                                  : (kb == B200OT_KERNEL_LAPLACIAN ? -1.0f / blur : -1.0f);
  const int64_t tiles = ceil_div64(N > M ? N : M, kSmallRows);
  cudaStream_t st = (cudaStream_t)stream;
  return for_batch_slices(B, [&](int64_t b0, int64_t nb) {
    SmallConvBwd T = S;
    T.x = x + b0 * N * D;
    T.y = y + b0 * M * D;
    T.a = a + b0 * N;
    T.b = b + b0 * M;
    T.go = grad_value + b0;
    T.gx = grad_x + b0 * N * D;
    T.gy = grad_y + b0 * M * D;
    const dim3 grid((unsigned)tiles, 2u, (unsigned)nb);
#define CALL(DD) launch_mmd_bwd<DD>(kb, T, grid, scale, clampq, coef, st)
    B200OT_DISPATCH_D(D, CALL)
#undef CALL
  });
}

}  // extern "C"
