// b200ot — the transport plan applied to a value matrix, D <= 8 (CUDA cores):
//     part[(split N + i)(1 + KV) + {0, 1 + k}] = sum_j e_ij {1, V_jk},   e_ij = 2^(H_j + X_i.Y_j - |X_i|^2/2 - lse2_i)
// i.e. the softmin row-gradient reduction of rowsum.cuh (kSoftminBwdP2) with the value matrix V (M, K) in the place
// the column coordinates take there.  The finalize divides by the row's own sum of e, so rounding of lse2 cancels.
//
// Same row tiles, bulk-TMA ring (full / empty mbarriers, per-thread release), colpack exponent tile and
// two-columns-per-step float2 arithmetic as rowsum_partial_kernel.  Each ring stage also carries the VALUE tile of its
// TJ columns: per column pair, KV float2 {V_k[j], V_k[j+1]} (pack_values_kernel), read with LDS.128; padding columns
// and value columns past K hold zeros.  KV is a compile-time slab of value columns (4 or 8): a wider V runs as
// ceil(K / 8) passes, each recomputing the exponent.
#pragma once
#include "common.cuh"

namespace b200ot {

// values (M, K) row-major -> value tiles of the slab of KV columns from k0: out[(pair KV + k) 2 + {0, 1}]
static __global__ void pack_values_kernel(const float* __restrict__ v, int64_t M, int64_t Mpad, int K, int k0, int KV,
                                          float* __restrict__ out) {
  const int64_t slot = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= Mpad) return;
  float* pk = out + (slot >> 1) * (int64_t)(KV * 2) + (slot & 1);
  for (int k = 0; k < KV; ++k) pk[2 * k] = (slot < M && k0 + k < K) ? v[slot * K + k0 + k] : 0.f;
}

template <int D_, int KV_, int R_, int NT_, int TJ_, int MINB_>
struct PlanApplyCfg {
  static constexpr int D = D_;
  static constexpr int KV = KV_;
  static constexpr int R = R_;
  static constexpr int NT = NT_;
  static constexpr int TJ = TJ_;
  static constexpr int MINB = MINB_;
  static constexpr int NACC = 1 + KV;
  static constexpr int NF2 = ((D + 2) / 2) * 2;  // colfmt_nf2(D, 1)
  static constexpr int TILE_FLOATS = (TJ / 2) * NF2 * 2;
  static constexpr int VTILE_FLOATS = (TJ / 2) * KV * 2;
  static constexpr int STAGE_BYTES = (TILE_FLOATS + VTILE_FLOATS) * 4;
  // as many stages (at most 3) as MINB resident CTAs leave room for in the SM's 228 KB (1 KB reserved per CTA)
  static constexpr int FIT = (228 * 1024 / MINB - 1024 - 64) / STAGE_BYTES;
  static constexpr int STAGES = FIT >= 3 ? 3 : FIT;
  static_assert(STAGES >= 2, "the ring needs two stages");
  static constexpr int ROWS_PER_CTA = NT * R;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * STAGES * 8;
};

template <class C>
__global__ void __launch_bounds__(C::NT + 32, C::MINB)
    plan_apply_partial_kernel(const float* __restrict__ x, const float* __restrict__ center, float scale,
                              const float* __restrict__ cols, const float* __restrict__ vals,
                              const float* __restrict__ lse2, float* __restrict__ part, int64_t N, int ntiles,
                              int tiles_per_split, int last_pairs) {
  constexpr int D = C::D, R = C::R, NT = C::NT, NF2 = C::NF2, STAGES = C::STAGES, NACC = C::NACC, KV = C::KV;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* tiles = reinterpret_cast<float*>(smem_raw);  // stage s: [exponent tile | value tile]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + STAGES * C::STAGE_BYTES);
  uint64_t* empty = full + STAGES;
  constexpr int STAGE_FLOATS = C::TILE_FLOATS + C::VTILE_FLOATS;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int split = blockIdx.y;
  const int64_t row0 = (int64_t)blockIdx.x * C::ROWS_PER_CTA;
  const int t0 = split * tiles_per_split;
  const int t1 = min(ntiles, t0 + tiles_per_split);
  const int nt = t1 - t0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], NT);  // every consumer thread releases the stage itself (rowsum.cuh)
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      for (int k = 0; k < nt; ++k) {
        const int st = k % STAGES;
        if (k >= STAGES) mbar_wait(&empty[st], ((k / STAGES) + 1) & 1);
        mbar_arrive_expect_tx(&full[st], C::STAGE_BYTES);
        float* dst = tiles + st * STAGE_FLOATS;
        tma_load_1d(dst, cols + (int64_t)(t0 + k) * C::TILE_FLOATS, C::TILE_FLOATS * 4, &full[st]);
        tma_load_1d(dst + C::TILE_FLOATS, vals + (int64_t)(t0 + k) * C::VTILE_FLOATS, C::VTILE_FLOATS * 4, &full[st]);
      }
    }
    return;
  }

  const int tid = threadIdx.x - 32;
  float2 X[R][D];
  float2 rt2[R];  // -|X|^2/2 - lse2, duplicated
#pragma unroll
  for (int r = 0; r < R; ++r) {
    int64_t i = row0 + tid + r * NT;
    if (i >= N) i = N - 1;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < D; ++k) {
      const float c = center ? center[k] : 0.f;
      const float v = scale * (x[i * D + k] - c);
      X[r][k] = dup2(v);
      acc = fmaf(v, v, acc);
    }
    rt2[r] = dup2(-0.5f * acc - lse2[i]);
  }

  float2 A[R][NACC];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int a = 0; a < NACC; ++a) A[r][a] = dup2(0.f);

  for (int k = 0; k < nt; ++k) {
    const int st = k % STAGES;
    const int npairs = (t0 + k + 1 == ntiles) ? last_pairs : C::TJ / 2;
    mbar_wait(&full[st], (k / STAGES) & 1);
    const float4* tp = reinterpret_cast<const float4*>(tiles + st * STAGE_FLOATS);
    const float4* vp = reinterpret_cast<const float4*>(tiles + st * STAGE_FLOATS + C::TILE_FLOATS);

    // two-level accumulation (tile sums T, then running sums A), as rowsum_partial_kernel
    float2 T[R][NACC];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int a = 0; a < NACC; ++a) T[r][a] = dup2(0.f);

#pragma unroll 2
    for (int jp = 0; jp < npairs; ++jp) {
      float2 S[NF2];
#pragma unroll
      for (int q = 0; q < NF2 / 2; ++q) {
        const float4 v = tp[jp * (NF2 / 2) + q];
        S[2 * q] = make_float2(v.x, v.y);
        S[2 * q + 1] = make_float2(v.z, v.w);
      }
      float2 V[KV];
#pragma unroll
      for (int q = 0; q < KV / 2; ++q) {
        const float4 v = vp[jp * (KV / 2) + q];
        V[2 * q] = make_float2(v.x, v.y);
        V[2 * q + 1] = make_float2(v.z, v.w);
      }
#pragma unroll
      for (int r = 0; r < R; ++r) {
        float2 t = fadd2(S[D], rt2[r]);
#pragma unroll
        for (int d = 0; d < D; ++d) t = ffma2(X[r][d], S[d], t);
        float2 e;
        e.x = ex2_approx(t.x);
        e.y = ex2_approx(t.y);
        T[r][0] = fadd2(T[r][0], e);
#pragma unroll
        for (int q = 0; q < KV; ++q) T[r][1 + q] = ffma2(e, V[q], T[r][1 + q]);
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int a = 0; a < NACC; ++a) A[r][a] = fadd2(A[r][a], T[r][a]);
    mbar_arrive(&empty[st]);  // after this thread's own last read of the stage
  }

#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int64_t i = row0 + tid + r * NT;
    if (i < N) {
#pragma unroll
      for (int a = 0; a < NACC; ++a) part[((int64_t)split * N + i) * NACC + a] = A[r][a].x + A[r][a].y;
    }
  }
}

}  // namespace b200ot
