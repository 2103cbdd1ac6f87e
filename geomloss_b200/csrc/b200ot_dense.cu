// b200ot — entropic OT on explicit cost matrices: both softmins of a symmetric Sinkhorn update from one pass over C.
// Interface contract: include/b200ot.h.  Reference semantics: softmin_dense and the symmetric loop of ot.solve_batch
// (src/geomloss/ot/_implementations/matrix.py:29-94, :620-660; ot/_abstract_solvers/sinkhorn_ot.py:259-260).
//
// Both updates of one iteration use the OLD potentials, so one read of C_ij feeds the row log-sum-exp of
//   t_ij = log2e (log b_j + g_j / eps - C_ij / eps)        (f~_i = -eps ln2 LSE2_j t_ij)
// and the column log-sum-exp of
//   u_ij = log2e (log a_i + f_i / eps - C_ij / eps)        (g~_j = -eps ln2 LSE2_i u_ij).
// Two exponentials per entry: the one-exponential identity 2^u = 2^t 2^(h_i - h_j) overflows fp32 once |f| / eps
// reaches ~100, which a small eps does at once.
//
// Layout (DESIGN.md §3.8): a CTA owns kDenseRows = 128 rows of one batch element and a contiguous range of column
// tiles (kDenseTJ = 32 columns, one per lane); each of its 8 warps holds 16 rows.  Per column tile a lane takes its
// column's 16 entries, folds them into its 16 row sums and into one column sum over the warp's rows.  The 8 warps' column sums meet in shared memory, once per tile, and leave as
// one (m, s) pair per (row tile, column); the row sums stay in registers across the CTA's whole column range and are
// merged across lanes once at the end.  Partials use the (m, s) float2 format of the other softmins, split-major,
// so b200ot_softmin_finalize is the epilogue of both directions:
//   rows:    part_row[s (B N) + b N + i],   s < n_split (column ranges)
//   columns: part_col[r (B M) + b M + j],   r < ceil(N / 128) (row tiles)
// Column partials cost 8 / (4 * 128) = 1/64 of C's bytes, row partials 2 n_split / M of them.
// Aligned C (16 bytes, M % 4 == 0) streams through a cp.async ring in shared memory; any other C (any N, M >= 1,
// any batch offset) takes scalar loads.  Both feed the same arithmetic.
#include "b200ot.h"
#include "common.cuh"
#include "host_util.cuh"

namespace b200ot {

constexpr int kDenseRows = 128;                    // rows per CTA
constexpr int kDenseWarps = 8;
constexpr int kDenseRPW = kDenseRows / kDenseWarps;  // rows per warp (= loads in flight per lane)
constexpr int kDenseTJ = 32;                       // columns per tile: one per lane
constexpr int kDenseTarget = 2048;                 // CTAs a launch aims for (~8 waves of 132 SMs x 2 CTAs)
constexpr int kDenseMinTiles = 8;                  // column tiles per CTA at least (256 columns)
// 2^64: a row term above it means the running max is outdated (the sum-guarded lazy max of softmin.cuh)
constexpr float kDenseGuard = 1.8446744e19f;

struct DensePlan {
  int64_t row_tiles, col_tiles;
  int n_split, tiles_per_split;
};

// Pure function of the shape (no device query), so that scratch sizes are reproducible on any host.
inline DensePlan dense_plan(int64_t B, int64_t N, int64_t M) {
  DensePlan p;
  p.row_tiles = ceil_div64(N, kDenseRows);
  p.col_tiles = ceil_div64(M, kDenseTJ);
  int64_t want = ceil_div64(kDenseTarget, p.row_tiles * B);
  const int64_t cap = ceil_div64(p.col_tiles, kDenseMinTiles);
  want = want < 1 ? 1 : (want > cap ? cap : want);
  p.tiles_per_split = (int)ceil_div64(p.col_tiles, want);
  p.n_split = (int)ceil_div64(p.col_tiles, p.tiles_per_split);  // every split owns at least one tile
  return p;
}

inline int64_t dense_row_part_bytes(const DensePlan& p, int64_t B, int64_t N) {
  return round_up64((int64_t)p.n_split * B * N * 8, 256);
}
inline int64_t dense_scratch_bytes(const DensePlan& p, int64_t B, int64_t N, int64_t M) {
  return dense_row_part_bytes(p, B, N) + round_up64(p.row_tiles * B * M * 8, 256);
}

// log2-domain h of one point: log2e (log_w + inv_eps * pot)
__device__ __forceinline__ float dense_h2(const float* __restrict__ log_w, const float* __restrict__ pot, int64_t k,
                                          float inv_eps) {
  return kLog2e * fmaf(inv_eps, __ldg(pot + k), __ldg(log_w + k));
}

// (m, s) <- (m, s) + (m2, s2) for two partial log2-sum-exps
__device__ __forceinline__ void merge_pair(float& m, float& s, float m2, float s2) {
  const float mm = fmaxf(m, m2);
  s = s * ex2_approx(m - mm) + s2 * ex2_approx(m2 - mm);
  m = mm;
}

// The aligned path (C 16-byte aligned, M % 4 == 0, so every row is): a kDenseStages-deep ring of 128 x 32 tiles in
// shared memory, filled by 16-byte cp.async copies kDenseStages - 1 tiles ahead of the tile being reduced, so that
// 48 KB per CTA stay in flight across the per-tile barrier.  Out-of-range rows and columns are zero-filled.
constexpr int kDenseStages = 4;
constexpr int kDenseTileFloats = kDenseRows * kDenseTJ;
constexpr int kDenseRingBytes = kDenseStages * kDenseTileFloats * 4;

__device__ __forceinline__ void dense_issue_tile(float* dst, const float* __restrict__ C, int64_t row0, int64_t N,
                                                 int64_t M, int64_t col0, int64_t nrow_b) {
  // thread t copies float4 column t % 8 of rows t / 8 + 32 q, q < 4
  const int v = threadIdx.x & 7;
#pragma unroll
  for (int q = 0; q < kDenseRows / 32; ++q) {
    const int r = (threadIdx.x >> 3) + 32 * q;
    const int64_t col = col0 + 4 * v;
    const bool ok = row0 + r < N && col < M;
    const float* src = ok ? C + (nrow_b + row0 + r) * M + col : C;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst + r * kDenseTJ + 4 * v)), "l"(src),
                 "r"(ok ? 16 : 0)
                 : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N_PENDING>
__device__ __forceinline__ void dense_wait_tiles() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N_PENDING) : "memory");
}

template <bool RING>
__global__ void __launch_bounds__(kDenseWarps * 32, 2)
    dense_pair_kernel(const float* __restrict__ C, const float* __restrict__ log_a, const float* __restrict__ log_b,
                      const float* __restrict__ f, const float* __restrict__ g, float inv_eps,
                      float2* __restrict__ part_row, float2* __restrict__ part_col, int64_t B, int64_t N, int64_t M,
                      int64_t row_tiles, int n_split, int tiles_per_split, int64_t col_tiles) {
  __shared__ float2 colbuf[2][kDenseWarps][kDenseTJ];
  extern __shared__ __align__(16) float ring[];
  int64_t blk = blockIdx.x;
  const int split = (int)(blk % n_split);
  blk /= n_split;
  const int64_t rt = blk % row_tiles;
  const int64_t b = blk / row_tiles;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i0 = rt * kDenseRows + warp * kDenseRPW;
  const bool live = i0 < N;  // a warp whose rows are all padding (small N) only takes part in the barriers
  const float sc = kLog2e * inv_eps;

  float ha[kDenseRPW], mr[kDenseRPW], sr[kDenseRPW];
#pragma unroll
  for (int k = 0; k < kDenseRPW; ++k) {
    ha[k] = i0 + k < N ? dense_h2(log_a, f, b * N + i0 + k, inv_eps) : kNegBig;
    mr[k] = kNegBig;
    sr[k] = 0.f;
  }
  const float* Cb = C + (b * N + i0) * M;
  const int64_t t0 = (int64_t)split * tiles_per_split;
  const int64_t t_end = min(t0 + tiles_per_split, col_tiles);
  if (RING) {
    for (int s = 0; s < kDenseStages; ++s) {
      if (t0 + s < t_end)
        dense_issue_tile(ring + s * kDenseTileFloats, C, rt * kDenseRows, N, M, (t0 + s) * kDenseTJ, b * N);
      else
        asm volatile("cp.async.commit_group;" ::: "memory");  // empty groups keep the count uniform
    }
    dense_wait_tiles<kDenseStages - 1>();
    __syncthreads();
  }
  for (int64_t jt = t0; jt < t_end; ++jt) {
    const int64_t j = jt * kDenseTJ + lane;
    const bool jv = j < M;
    const int slot = (int)((jt - t0) % kDenseStages);
    float mc = kNegBig, s_c = 0.f;
    if (live) {
      const float hb = jv ? dense_h2(log_b, g, b * M + j, inv_eps) : kNegBig;
      float c[kDenseRPW];
      if (RING) {
        const float* tile = ring + slot * kDenseTileFloats + warp * kDenseRPW * kDenseTJ;
#pragma unroll
        for (int k = 0; k < kDenseRPW; ++k) c[k] = tile[k * kDenseTJ + lane];
      } else {
#pragma unroll
        for (int k = 0; k < kDenseRPW; ++k) c[k] = (jv && i0 + k < N) ? __ldg(Cb + k * M + j) : 0.f;
      }
      // the column sum over this warp's rows: exact max first (its terms all share this tile)
      float u[kDenseRPW];
#pragma unroll
      for (int k = 0; k < kDenseRPW; ++k) {
        u[k] = fmaf(c[k], -sc, ha[k]);
        mc = fmaxf(mc, u[k]);
      }
#pragma unroll
      for (int k = 0; k < kDenseRPW; ++k) {
        s_c += ex2_approx(u[k] - mc);
        // the row sums: one term per tile, the running max raised only when a term exceeds it by 2^64
        const float t = fmaf(c[k], -sc, hb);
        const float e = ex2_approx(t - mr[k]);
        if (e > kDenseGuard) {
          sr[k] = fmaf(sr[k], ex2_approx(mr[k] - t), 1.f);
          mr[k] = t;
        } else {
          sr[k] += e;
        }
      }
    }
    float2* buf = colbuf[jt & 1][0];
    buf[warp * kDenseTJ + lane] = make_float2(mc, s_c);
    if (RING) dense_wait_tiles<kDenseStages - 2>();  // this thread's copies of tile jt + 1 have landed
    // colbuf complete, tile jt + 1 visible to every thread, slot of tile jt free (the double colbuf lets the next
    // tile's writes run without a second barrier)
    __syncthreads();
    if (RING) {
      if (jt + kDenseStages < t_end)
        dense_issue_tile(ring + slot * kDenseTileFloats, C, rt * kDenseRows, N, M, (jt + kDenseStages) * kDenseTJ,
                         b * N);
      else
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    if (warp == 0 && jv) {
      float m = buf[lane].x, s = buf[lane].y;
#pragma unroll
      for (int w = 1; w < kDenseWarps; ++w) merge_pair(m, s, buf[w * kDenseTJ + lane].x, buf[w * kDenseTJ + lane].y);
      part_col[rt * (B * M) + b * M + j] = make_float2(m, s);
    }
  }
  // row sums: across the 32 lanes (columns), then lane k writes row i0 + k
  if (!live) return;
#pragma unroll
  for (int k = 0; k < kDenseRPW; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      merge_pair(mr[k], sr[k], __shfl_xor_sync(0xffffffffu, mr[k], o), __shfl_xor_sync(0xffffffffu, sr[k], o));
    if (lane == k && i0 + k < N) part_row[(int64_t)split * (B * N) + b * N + i0 + k] = make_float2(mr[k], sr[k]);
  }
}

// grad_C_ij = go_f_i 2^(t_ij - lse2_row_i) + go_g_j 2^(u_ij - lse2_col_j): C read once, grad_C written once.
// One CTA: kDenseRPW rows x 256 columns of one batch element, one column per thread.
constexpr int kDenseBwdCols = 256;
__global__ void __launch_bounds__(kDenseBwdCols)
    dense_pair_bwd_kernel(const float* __restrict__ C, const float* __restrict__ log_a,
                          const float* __restrict__ log_b, const float* __restrict__ f,
                          const float* __restrict__ g, float inv_eps, const float* __restrict__ lse2_row,
                          const float* __restrict__ lse2_col, const float* __restrict__ go_f,
                          const float* __restrict__ go_g, float* __restrict__ grad_C, int64_t B, int64_t N,
                          int64_t M, int64_t row_blocks, int64_t col_blocks) {
  int64_t blk = blockIdx.x;
  const int64_t cb = blk % col_blocks;
  blk /= col_blocks;
  const int64_t rb = blk % row_blocks;
  const int64_t b = blk / row_blocks;
  const int64_t j = cb * kDenseBwdCols + threadIdx.x;
  if (j >= M) return;
  const float sc = kLog2e * inv_eps;
  const float hb = dense_h2(log_b, g, b * M + j, inv_eps);
  const float lse2_j = __ldg(lse2_col + b * M + j);
  const float wg = __ldg(go_g + b * M + j);
  const int64_t i0 = rb * kDenseRPW;
#pragma unroll 4
  for (int k = 0; k < kDenseRPW; ++k) {
    const int64_t i = i0 + k;
    if (i >= N) break;
    const int64_t r = b * N + i;
    const float c = __ldg(C + r * M + j);
    const float t = fmaf(c, -sc, hb) - __ldg(lse2_row + r);
    const float u = fmaf(c, -sc, dense_h2(log_a, f, r, inv_eps)) - lse2_j;
    grad_C[r * M + j] = __ldg(go_f + r) * ex2_approx(t) + wg * ex2_approx(u);
  }
}


// ---- row softmins only: the four Jacobi updates of SamplesLoss("sinkhorn", cost=...) (DESIGN.md section 3.9) ----
// Each matrix of a group has its own C (B, n_rows, n_cols), column log-weights and column potential; per entry
//   t_ij = log2e (log_w_j + pot_j / eps - C_ij / eps),   out_i = -eps ln2 LSE2_j t_ij   (finalize).
// No column direction, so no barrier and no column partials: a warp owns kRowsRPW rows and sweeps its split's columns
// in steps of 128 (4 consecutive columns per lane, one 16-byte load per row on the aligned path), reusing each column's
// h across its rows.  The row sums stay in registers with the sum-guarded lazy max and are merged across lanes once.
// Both load paths visit the same entries in the same order and share the arithmetic, so they return the same bits.
constexpr int kRowsRPW = 8;                         // rows per warp: 16-byte loads in flight per lane and step
constexpr int kRowsCTA = kDenseWarps * kRowsRPW;    // 64 rows per CTA
constexpr int kRowsStep = 4 * 32;                   // columns per warp step
constexpr int kRowsMinSteps = 4;                    // steps per split at least (512 columns)
constexpr int kRowsMaxGroup = 4;

struct RowsPlan {
  int64_t row_blocks, steps;
  int n_split, steps_per_split;
};

// Pure function of the shape (no device query), so that scratch sizes are reproducible on any host.
inline RowsPlan rows_plan(int64_t B, int64_t N, int64_t M) {
  RowsPlan p;
  p.row_blocks = ceil_div64(N, kRowsCTA);
  p.steps = ceil_div64(M, kRowsStep);
  int64_t want = ceil_div64(kDenseTarget, p.row_blocks * B);
  const int64_t cap = ceil_div64(p.steps, kRowsMinSteps);
  want = want < 1 ? 1 : (want > cap ? cap : want);
  p.steps_per_split = (int)ceil_div64(p.steps, want);
  p.n_split = (int)ceil_div64(p.steps, p.steps_per_split);  // every split owns at least one step
  return p;
}

inline int64_t rows_part_bytes(const RowsPlan& p, int64_t B, int64_t N) {
  return round_up64((int64_t)p.n_split * B * N * 8, 256);
}

struct RowsProblem {
  const float* C;
  const float* log_w;
  const float* pot;  // null: 0
  float2* part;      // part[s (B N) + b N + i], s < n_split
  int64_t B, N, M, row_blocks, steps, cta_begin;
  int n_split, steps_per_split, vec;
};
struct RowsGroup {
  RowsProblem p[kRowsMaxGroup];
  int n;
};

template <bool VEC>
__device__ __forceinline__ void dense_rows_reduce(const RowsProblem& d, int64_t blk, float inv_eps) {
  const int split = (int)(blk % d.n_split);
  blk /= d.n_split;
  const int64_t rb = blk % d.row_blocks;
  const int64_t b = blk / d.row_blocks;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t N = d.N, M = d.M;
  const int64_t i0 = rb * kRowsCTA + warp * kRowsRPW;
  if (i0 >= N) return;  // no barrier in this kernel: a warp of padding rows leaves at once
  const float sc = kLog2e * inv_eps;
  const float* __restrict__ Cw = d.C + (b * N + i0) * M;
  const float* __restrict__ lw = d.log_w + b * M;
  const float* __restrict__ pt = d.pot ? d.pot + b * M : nullptr;
  float mr[kRowsRPW], sr[kRowsRPW];
#pragma unroll
  for (int k = 0; k < kRowsRPW; ++k) {
    mr[k] = kNegBig;
    sr[k] = 0.f;
  }
  const int64_t s0 = (int64_t)split * d.steps_per_split;
  const int64_t s_end = min(s0 + d.steps_per_split, d.steps);
  for (int64_t s = s0; s < s_end; ++s) {
    const int64_t j0 = s * kRowsStep + 4 * lane;
    float c[kRowsRPW][4];
#pragma unroll
    for (int k = 0; k < kRowsRPW; ++k) {
      const bool rv = i0 + k < N;
      if (VEC) {  // M % 4 == 0: the lane's 4 columns are all in range or all out
        const float4 v = (rv && j0 < M) ? __ldg(reinterpret_cast<const float4*>(Cw + k * M + j0))
                                        : make_float4(0.f, 0.f, 0.f, 0.f);
        c[k][0] = v.x, c[k][1] = v.y, c[k][2] = v.z, c[k][3] = v.w;
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) c[k][q] = (rv && j0 + q < M) ? __ldg(Cw + k * M + j0 + q) : 0.f;
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int64_t j = j0 + q;
      if (j >= M) continue;
      const float h = kLog2e * (pt ? fmaf(inv_eps, __ldg(pt + j), __ldg(lw + j)) : __ldg(lw + j));
#pragma unroll
      for (int k = 0; k < kRowsRPW; ++k) {
        // one term per entry, the running max raised only when a term exceeds it by 2^64 (kDenseGuard)
        const float t = fmaf(c[k][q], -sc, h);
        const float e = ex2_approx(t - mr[k]);
        if (e > kDenseGuard) {
          sr[k] = fmaf(sr[k], ex2_approx(mr[k] - t), 1.f);
          mr[k] = t;
        } else {
          sr[k] += e;
        }
      }
    }
  }
  // across the 32 lanes, then lane k writes row i0 + k
#pragma unroll
  for (int k = 0; k < kRowsRPW; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      merge_pair(mr[k], sr[k], __shfl_xor_sync(0xffffffffu, mr[k], o), __shfl_xor_sync(0xffffffffu, sr[k], o));
    if (lane == k && i0 + k < N) d.part[(int64_t)split * (d.B * N) + b * N + i0 + k] = make_float2(mr[k], sr[k]);
  }
}

// The group's CTAs are enumerated problem after problem; the descriptors travel by value.
__global__ void __launch_bounds__(kDenseWarps * 32) dense_rows_kernel(const __grid_constant__ RowsGroup g, float inv_eps) {
  const int64_t blk = blockIdx.x;
  int k = 0;
#pragma unroll
  for (int q = 1; q < kRowsMaxGroup; ++q)
    if (q < g.n && blk >= g.p[q].cta_begin) k = q;
  const RowsProblem& d = g.p[k];
  if (d.vec)
    dense_rows_reduce<true>(d, blk - d.cta_begin, inv_eps);
  else
    dense_rows_reduce<false>(d, blk - d.cta_begin, inv_eps);
}

// grad_C_ij = go_i 2^(t_ij - lse2_i): C read once, grad_C written once; kDenseRPW rows x 256 columns per CTA.
__global__ void __launch_bounds__(kDenseBwdCols)
    dense_rows_bwd_kernel(const float* __restrict__ C, const float* __restrict__ log_w, const float* __restrict__ pot,
                          float inv_eps, const float* __restrict__ lse2, const float* __restrict__ go,
                          float* __restrict__ grad_C, int64_t N, int64_t M, int64_t row_blocks, int64_t col_blocks) {
  int64_t blk = blockIdx.x;
  const int64_t cb = blk % col_blocks;
  blk /= col_blocks;
  const int64_t rb = blk % row_blocks;
  const int64_t b = blk / row_blocks;
  const int64_t j = cb * kDenseBwdCols + threadIdx.x;
  if (j >= M) return;
  const float sc = kLog2e * inv_eps;
  const float h = kLog2e * (pot ? fmaf(inv_eps, __ldg(pot + b * M + j), __ldg(log_w + b * M + j)) : __ldg(log_w + b * M + j));
  const int64_t i0 = rb * kDenseRPW;
#pragma unroll 4
  for (int k = 0; k < kDenseRPW; ++k) {
    const int64_t i = i0 + k;
    if (i >= N) break;
    const int64_t r = b * N + i;
    const float c = __ldg(C + r * M + j);
    grad_C[r * M + j] = __ldg(go + r) * ex2_approx(fmaf(c, -sc, h) - __ldg(lse2 + r));
  }
}

}  // namespace b200ot

using namespace b200ot;

extern "C" {

B200OT_API int64_t b200ot_dense_scratch_bytes(int64_t B, int64_t N, int64_t M) {
  if (B <= 0 || N <= 0 || M <= 0) return 0;
  return dense_scratch_bytes(dense_plan(B, N, M), B, N, M);
}

B200OT_API int b200ot_dense_softmin_pair(const float* C, const float* log_a, const float* log_b, const float* f_old,
                                         const float* g_old, float inv_eps, float alpha_old, float beta, float* f_out,
                                         float* g_out, float* lse2_row, float* lse2_col, int64_t B, int64_t N,
                                         int64_t M, float eps, void* scratch, int64_t scratch_bytes, void* stream) {
  if (!C || !log_a || !log_b || !f_old || !g_old || !f_out || !g_out || !scratch || B <= 0 || N <= 0 || M <= 0 ||
      !(eps > 0.f) || !(inv_eps > 0.f))
    return B200OT_EINVAL;
  const DensePlan pl = dense_plan(B, N, M);
  if (const int rc = scratch_check(scratch, scratch_bytes, dense_scratch_bytes(pl, B, N, M))) return rc;
  const int64_t grid = pl.row_tiles * B * pl.n_split;
  if (grid > 0x7fffffff) return B200OT_EINVAL;
  float2* part_row = reinterpret_cast<float2*>(scratch);
  float2* part_col = reinterpret_cast<float2*>(reinterpret_cast<char*>(scratch) + dense_row_part_bytes(pl, B, N));
  cudaStream_t st = (cudaStream_t)stream;
  if ((((uintptr_t)C) & 15) == 0 && M % 4 == 0) {
    B200OT_CUDA_TRY(cudaFuncSetAttribute(dense_pair_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kDenseRingBytes));
    dense_pair_kernel<true><<<(unsigned)grid, kDenseWarps * 32, kDenseRingBytes, st>>>(
        C, log_a, log_b, f_old, g_old, inv_eps, part_row, part_col, B, N, M, pl.row_tiles, pl.n_split,
        pl.tiles_per_split, pl.col_tiles);
  } else {
    dense_pair_kernel<false><<<(unsigned)grid, kDenseWarps * 32, 0, st>>>(
        C, log_a, log_b, f_old, g_old, inv_eps, part_row, part_col, B, N, M, pl.row_tiles, pl.n_split,
        pl.tiles_per_split, pl.col_tiles);
  }
  B200OT_CUDA_TRY(cudaGetLastError());
  int rc = b200ot_softmin_finalize(reinterpret_cast<float*>(part_row), pl.n_split, f_old, alpha_old, beta, f_out,
                                   lse2_row, B * N, eps, stream);
  if (rc) return rc;
  return b200ot_softmin_finalize(reinterpret_cast<float*>(part_col), (int32_t)pl.row_tiles, g_old, alpha_old, beta,
                                 g_out, lse2_col, B * M, eps, stream);
}

B200OT_API int b200ot_dense_softmin_pair_bwd(const float* C, const float* log_a, const float* log_b, const float* f,
                                             const float* g, float inv_eps, const float* lse2_row,
                                             const float* lse2_col, const float* go_f, const float* go_g,
                                             float* grad_C, int64_t B, int64_t N, int64_t M, void* stream) {
  if (!C || !log_a || !log_b || !f || !g || !lse2_row || !lse2_col || !go_f || !go_g || !grad_C || B <= 0 ||
      N <= 0 || M <= 0 || !(inv_eps > 0.f))
    return B200OT_EINVAL;
  const int64_t row_blocks = ceil_div64(N, kDenseRPW), col_blocks = ceil_div64(M, kDenseBwdCols);
  const int64_t grid = B * row_blocks * col_blocks;
  if (grid > 0x7fffffff) return B200OT_EINVAL;
  dense_pair_bwd_kernel<<<(unsigned)grid, kDenseBwdCols, 0, (cudaStream_t)stream>>>(
      C, log_a, log_b, f, g, inv_eps, lse2_row, lse2_col, go_f, go_g, grad_C, B, N, M, row_blocks, col_blocks);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}


B200OT_API int64_t b200ot_dense_rows_scratch_bytes(const b200ot_dense_rows* probs, int32_t n) {
  if (!probs || n < 1 || n > B200OT_DENSE_ROWS_MAX) return 0;
  int64_t total = 0;
  for (int k = 0; k < n; ++k) {
    const b200ot_dense_rows& q = probs[k];
    if (q.B <= 0 || q.n_rows <= 0 || q.n_cols <= 0) return 0;
    total += rows_part_bytes(rows_plan(q.B, q.n_rows, q.n_cols), q.B, q.n_rows);
  }
  return total;
}

B200OT_API int b200ot_dense_softmin_rows(const b200ot_dense_rows* probs, int32_t n, float eps, float alpha_old,
                                         float beta, void* scratch, int64_t scratch_bytes, void* stream) {
  if (!probs || n < 1 || n > B200OT_DENSE_ROWS_MAX || !scratch || !(eps > 0.f)) return B200OT_EINVAL;
  RowsGroup g = {};
  g.n = n;
  int64_t grid = 0, offset = 0;
  for (int k = 0; k < n; ++k) {
    const b200ot_dense_rows& q = probs[k];
    if (!q.C || !q.log_w || (!q.out && !q.lse2) || q.B <= 0 || q.n_rows <= 0 || q.n_cols <= 0) return B200OT_EINVAL;
    const RowsPlan pl = rows_plan(q.B, q.n_rows, q.n_cols);
    RowsProblem& d = g.p[k];
    d.C = q.C, d.log_w = q.log_w, d.pot = q.pot;
    d.part = reinterpret_cast<float2*>(reinterpret_cast<char*>(scratch) + offset);
    d.B = q.B, d.N = q.n_rows, d.M = q.n_cols, d.row_blocks = pl.row_blocks, d.steps = pl.steps, d.cta_begin = grid;
    d.n_split = pl.n_split, d.steps_per_split = pl.steps_per_split;
    d.vec = (((uintptr_t)q.C) & 15) == 0 && q.n_cols % 4 == 0;
    grid += pl.row_blocks * q.B * pl.n_split;
    offset += rows_part_bytes(pl, q.B, q.n_rows);
  }
  if (grid > 0x7fffffff) return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, offset)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  dense_rows_kernel<<<(unsigned)grid, kDenseWarps * 32, 0, st>>>(g, 1.f / eps);
  B200OT_CUDA_TRY(cudaGetLastError());
  for (int k = 0; k < n; ++k) {
    const b200ot_dense_rows& q = probs[k];
    const int rc = b200ot_softmin_finalize(reinterpret_cast<const float*>(g.p[k].part), g.p[k].n_split, q.out_old,
                                           alpha_old, beta, q.out, q.lse2, q.B * q.n_rows, eps, stream);
    if (rc) return rc;
  }
  return B200OT_OK;
}

B200OT_API int b200ot_dense_softmin_rows_bwd(const float* C, const float* log_w, const float* pot, float inv_eps,
                                             const float* lse2, const float* go, float* grad_C, int64_t B, int64_t N,
                                             int64_t M, void* stream) {
  if (!C || !log_w || !lse2 || !go || !grad_C || B <= 0 || N <= 0 || M <= 0 || !(inv_eps > 0.f))
    return B200OT_EINVAL;
  const int64_t row_blocks = ceil_div64(N, kDenseRPW), col_blocks = ceil_div64(M, kDenseBwdCols);
  const int64_t grid = B * row_blocks * col_blocks;
  if (grid > 0x7fffffff) return B200OT_EINVAL;
  dense_rows_bwd_kernel<<<(unsigned)grid, kDenseBwdCols, 0, (cudaStream_t)stream>>>(C, log_w, pot, inv_eps, lse2, go,
                                                                                     grad_C, N, M, row_blocks,
                                                                                     col_blocks);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

}  // extern "C"
