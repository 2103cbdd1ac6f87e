// b200ot — one exponential for two softmin terms: the xy / yx softmins of a Jacobi Sinkhorn iteration from one pass, and
// the xx (or yy) softmin over the unordered pairs only.  D = 3, p = 2.  DESIGN.md §3.1b.
//
// Both clouds are packed by pack_cols_kernel with their own potential: y with h_y (H_j = log2e h_y,j - |Y_j|^2/2) and
// x with h_x (G_i likewise).  The plan-scale exponent
//     T_ij = X_i.Y_j + H_j + G_i = log2e (h_x,i + h_y,j - C_ij / eps)
// feeds the row sum of the xy softmin, sum_j 2^T_ij = 2^(log2e h_x,i) sum_j 2^t_ij, and the column sum of the yx
// softmin, sum_i 2^T_ij = 2^(log2e h_y,j) sum_i 2^t'_ji.  The partials are (m, s) pairs with m = -G_i - |X_i|^2/2, so
// softmin_finalize_kernel's lse2 = m + log2(sum s) is the softmin's.  No running max: sum_j 2^T_ij equals
// a_i exp((f_i - f~_i) / eps), which depends on how far the potential moves in one iteration, not on |f| / eps; the
// finalize checks that range and the caller recomputes a softmin that leaves it on the unpaired path.
//
// Work decomposition
//   Both axes are cut into blocks of whole 1024-point tiles (at most 64 blocks, so at most 64 partial slots per point).
//   An item is one (row block, column block) of one problem; a launch serves 1 to 3 problems (a pair, or a symmetric
//   softmin) with one CTA per item, the items longest first (PairLaunch): the block scheduler hands out the long items
//   first, and the launch has one tail instead of one per problem.  The producer warp streams the column tiles of the
//   item through a STAGES-deep TMA ring; each tile stays resident while the consumers sweep every row tile of the block
//   over it, the rows in registers (R per thread) as in softmin_partial_kernel.  Every item writes only its own slots,
//   so the results do not depend on the order in which the items run.
//   row sums    per thread in registers over one column tile, then added in column-tile order into the CTA's slot of
//               the row partials (slot = column block): every (slot, row) is owned by one thread of one CTA.
//   column sums per thread over its R rows, across the warp by a shuffle reduce-scatter (16 columns at a time), across
//               row tiles into the warp's own shared-memory row (fixed order), across warps once per column tile, and
//               written once per (column, slot = row block).  No atomics: the partials are reproducible bit for bit.
//   sym (x is y): only blocks (r, c) with c >= r run; a diagonal block runs the same body and writes its row sums
//               only (its column sums are the same terms again).  Rows of block r go to slot c, columns of block c to
//               slot r, so every (slot, point) is written exactly once.
#pragma once
#include "common.cuh"
#include "softmin.cuh"

namespace b200ot {

template <int R_, int NT_ = 128, int MINB_ = 4, int STAGES_ = 2>
struct PairCfg {
  static constexpr int D = 3;
  static constexpr int R = R_;            // rows per consumer thread
  static constexpr int NT = NT_;          // consumer threads
  static constexpr int MINB = MINB_;      // CTAs per SM the register budget is planned for
  static constexpr int STAGES = STAGES_;
  static constexpr int NF2 = 4;           // colfmt_nf2(3, 1): X0, X1, X2 and the potential term, per column pair
  static constexpr int TJ = 1024;         // points per tile on both axes (= kPackPad: packed buffers hold whole tiles)
  static constexpr int ROWS = NT * R;     // rows per sweep
  static constexpr int GP = 8;            // column pairs per group: 16 column values reduced across the warp at once
  static constexpr int NW = NT / 32;
  static constexpr int TILE_FLOATS = TJ / 2 * NF2 * 2;
  static constexpr int TILE_BYTES = TILE_FLOATS * 4;
  static constexpr int SMEM_BYTES = STAGES * TILE_BYTES + NW * TJ * 4 + 2 * STAGES * 8;
  static_assert(TJ % ROWS == 0 && (TJ / 2) % GP == 0 && GP == 8, "tile = whole sweeps and whole groups");
};

// first tile of block b when nt tiles are cut into nb blocks (sizes differ by at most one tile)
__host__ __device__ inline int pair_block_start(int b, int nt, int nb) { return (int)((int64_t)b * nt / nb); }
// how many of those blocks have `size` tiles (nt / nb or nt / nb + 1)
__host__ __device__ inline int pair_blocks_of_size(int size, int nt, int nb) {
  const int q = nt / nb, big = nt % nb;
  return size == q + 1 ? big : size == q ? nb - big : 0;
}
// the k-th of them in block order
__device__ inline int pair_block_of_size(int k, int size, int nt, int nb) {
  int b = 0;
  for (;; ++b)
    if (pair_block_start(b + 1, nt, nb) - pair_block_start(b, nt, nb) == size && k-- == 0) break;
  return b;
}

// One problem of a launch: a pair (rows x packed with h_x, columns y packed with h_y; row sums to part_row, column sums
// to part_col) or, with sym, one symmetric softmin (x is y, rows_pk is cols_pk, part_row is part_col).
struct PairProblem {
  const float* rows_pk;
  const float* cols_pk;
  float2* part_row;
  float2* part_col;
  int64_t N, M;
  int ntr, ntc, nbr, nbc;  // tiles and blocks of the row and column axes
  int sym;
};

constexpr int kPairMaxProblems = 3;
// The items of problem `prob` whose row block has tr tiles and column block tc tiles (sym: the unordered block pairs
// with one block of each size), items start .. start + count - 1 of the launch.  The blocks of an axis have q or q + 1
// tiles, so a problem has at most four classes.
struct PairClass {
  int prob, tr, tc, start;
};
// Passed by value: the classes are sorted by tr * tc (the item's tile pairs), largest first, a pure function of the
// shapes, so the item order needs no host synchronisation and no copy.
struct PairLaunch {
  PairProblem prob[kPairMaxProblems];
  PairClass cls[4 * kPairMaxProblems];
  int ncls, items;
};

// problem, row block and column block of item t
__device__ inline void pair_item(const PairLaunch& L, int t, int& p, int& rb, int& cb) {
  int c = 0;
  while (c + 1 < L.ncls && t >= L.cls[c + 1].start) ++c;
  const PairClass& K = L.cls[c];
  const PairProblem& P = L.prob[K.prob];
  int k = t - K.start, i, j;
  if (P.sym && K.tr == K.tc) {  // the unordered pairs i <= j of the n blocks of this size, row by row
    const int n = pair_blocks_of_size(K.tr, P.ntr, P.nbr);
    i = 0;
    while (k >= n - i) {
      k -= n - i;
      ++i;
    }
    j = i + k;
  } else {
    const int nc = pair_blocks_of_size(K.tc, P.ntc, P.nbc);
    i = k / nc;
    j = k % nc;
  }
  const int a = pair_block_of_size(i, K.tr, P.ntr, P.nbr), b = pair_block_of_size(j, K.tc, P.ntc, P.nbc);
  p = K.prob;
  rb = P.sym ? min(a, b) : a;
  cb = P.sym ? max(a, b) : b;
}

// v through an opaque move: a problem's fields indexed by it are read from the parameter space where they are used
// instead of being held in registers across the sweeps, which have none to spare (held, they spill)
__device__ __forceinline__ int opaque(int v) {
  asm volatile("mov.b32 %0, %0;" : "+r"(v));
  return v;
}

// One step of the warp's reduce-scatter of 2*O values: a lane keeps the half whose index bit O matches its lane bit O
// and adds its partner's copy of that half
template <int O, int NV>
__device__ __forceinline__ void reduce_scatter_step(float (&cv)[NV], int lane) {
  const bool hi = (lane & O) != 0;
#pragma unroll
  for (int k = 0; k < O; ++k) {
    const float send = hi ? cv[k] : cv[k + O];
    const float keep = hi ? cv[k + O] : cv[k];
    cv[k] = keep + __shfl_xor_sync(0xffffffffu, send, O);
  }
}

// One group of GP column pairs against the R rows of a thread: the row terms go to rs, and the 16 column values
// (summed over the thread's rows, then over the warp) end in lane l (and l ^ 16) as column (l & 15).
template <class C>
__device__ __forceinline__ float pair_group(const float4* __restrict__ tp, int pair0, const float (&X)[C::R][3],
                                            const float (&G)[C::R], float (&rs)[C::R], int lane) {
  constexpr int R = C::R, GP = C::GP;
  float cv[2 * GP];
  float gs[R];
#pragma unroll
  for (int c = 0; c < GP; ++c) {
    float2 S[C::NF2];
    load_packet<C::NF2>(tp, pair0 + c, S);
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float2 t = S[3];
#pragma unroll
      for (int d = 0; d < 3; ++d) t = ffma2(dup2(X[r][d]), S[d], t);
      t = fadd2(t, dup2(G[r]));
      const float ex = ex2_approx(t.x), ey = ex2_approx(t.y);
      gs[r] = (c == 0) ? ex : gs[r] + ex;
      gs[r] += ey;
      cv[2 * c] = (r == 0) ? ex : cv[2 * c] + ex;
      cv[2 * c + 1] = (r == 0) ? ey : cv[2 * c + 1] + ey;
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) rs[r] += gs[r];
  reduce_scatter_step<8>(cv, lane);
  reduce_scatter_step<4>(cv, lane);
  reduce_scatter_step<2>(cv, lane);
  reduce_scatter_step<1>(cv, lane);
  return cv[0] + __shfl_xor_sync(0xffffffffu, cv[0], 16);
}

template <class C>
__global__ void __launch_bounds__(C::NT + 32, C::MINB) softmin_pair_kernel(const __grid_constant__ PairLaunch L) {
  constexpr int R = C::R, NT = C::NT, TJ = C::TJ, STAGES = C::STAGES, GP = C::GP;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* tiles = reinterpret_cast<float*>(smem_raw);
  float* colacc = reinterpret_cast<float*>(smem_raw + STAGES * C::TILE_BYTES);  // [NW][TJ]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + STAGES * C::TILE_BYTES + C::NW * TJ * 4);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], NT);
    }
    mbar_fence_init();
  }
  __syncthreads();

  int p, rb, cb;
  pair_item(L, blockIdx.x, p, rb, cb);
  const PairProblem& P = L.prob[p];
  const int tc0 = pair_block_start(cb, P.ntc, P.nbc), nt = pair_block_start(cb + 1, P.ntc, P.nbc) - tc0;

  if (warp == 0) {
    if (lane == 0) {
      for (int k = 0; k < nt; ++k) {
        const int st = k % STAGES;
        if (k >= STAGES) mbar_wait(&empty[st], ((k / STAGES) + 1) & 1);
        mbar_arrive_expect_tx(&full[st], C::TILE_BYTES);
        tma_load_1d(tiles + st * C::TILE_FLOATS, P.cols_pk + (int64_t)(tc0 + k) * C::TILE_FLOATS, C::TILE_BYTES,
                    &full[st]);
      }
    }
    return;
  }

  const int tid = threadIdx.x - 32;
  const int cw = warp - 1;  // consumer warp
  float* myacc = colacc + cw * TJ;
  const bool cols = !P.sym || rb != cb;
  const int tr0 = pair_block_start(rb, P.ntr, P.nbr), tr1 = pair_block_start(rb + 1, P.ntr, P.nbr);
  for (int k = 0; k < nt; ++k) {
    const int st = k % STAGES;
    mbar_wait(&full[st], (k / STAGES) & 1);
    const float4* tp = reinterpret_cast<const float4*>(tiles + st * C::TILE_FLOATS);

    // sweeps counted from 0: the first-sweep test then holds no 64-bit row bounds across the groups
    for (int sw = 0; sw < (tr1 - tr0) * (TJ / C::ROWS); ++sw) {
      const int64_t row0 = (int64_t)tr0 * TJ + (int64_t)sw * C::ROWS;
      // rows of this sweep from the packed row cloud (padding rows carry G = -inf and add nothing)
      float X[R][3], G[R], rs[R];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int64_t i = row0 + tid + r * NT;
        const float* pk = L.prob[opaque(p)].rows_pk + (i >> 1) * (C::NF2 * 2) + (i & 1);
#pragma unroll
        for (int d = 0; d < 3; ++d) X[r][d] = pk[2 * d];
        G[r] = pk[6];
        rs[r] = 0.f;
      }
      const bool first_sweep = sw == 0;
#pragma unroll 1
      for (int g = 0; g < TJ / 2 / GP; ++g) {
        const float v = pair_group<C>(tp, g * GP, X, G, rs, lane);
        if (lane < 16) {
          float* a = myacc + g * 2 * GP + lane;
          *a = first_sweep ? v : *a + v;
        }
      }
      const PairProblem& Q = L.prob[opaque(p)];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int64_t i = row0 + tid + r * NT;
        if (i < Q.N) {
          float2* dst = Q.part_row + (int64_t)cb * Q.N + i;
          if (k == 0) {
            const float sq = fmaf(X[r][2], X[r][2], fmaf(X[r][1], X[r][1], X[r][0] * X[r][0]));
            *dst = make_float2(-G[r] + -0.5f * sq, rs[r]);
          } else {
            dst->y += rs[r];
          }
        }
      }
    }

    if (cols) {
      // column partials of this tile: the consumer warps' rows in a fixed order
      asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory");
      const float* tf = tiles + st * C::TILE_FLOATS;
      const PairProblem& Q = L.prob[opaque(p)];
#pragma unroll 1
      for (int jl = tid; jl < TJ; jl += NT) {
        float s = colacc[jl];
#pragma unroll
        for (int w = 1; w < C::NW; ++w) s += colacc[w * TJ + jl];
        const int64_t j = (int64_t)(tc0 + k) * TJ + jl;
        if (j < Q.M) {
          const float* pk = tf + (jl >> 1) * (C::NF2 * 2) + (jl & 1);
          const float y0 = pk[0], y1 = pk[2], y2 = pk[4];
          const float sq = fmaf(y2, y2, fmaf(y1, y1, y0 * y0));
          Q.part_col[(int64_t)rb * Q.M + j] = make_float2(-pk[6] + -0.5f * sq, s);
        }
      }
      asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory");
    }
    mbar_arrive(&empty[st]);
  }
}

}  // namespace b200ot
