// b200ot — softmin partial-reduction kernel (the N x M hot loop), templated on the problem shape.
//
// Replaces the reference's softmin_tensorized / softmin_online
// (src/geomloss/_legacy/sinkhorn_samples.py:32-71, :337-346): for every row i
//     lse2_i = log2 sum_j 2^( t_ij ),   t_ij = log2e * ( h_j - |x_i - y_j|^p / (p eps) )
// is accumulated online as a (running max m_i, sum s_i of 2^(t_ij - m_i)) pair, the cost being
// recomputed on the fly from the coordinates and never stored.
//
// Work decomposition
//   grid  = (row tiles, column splits); a CTA owns NT*R rows and a contiguous run of column tiles;
//   block = 1 producer warp + NT/32 consumer warps.  The producer streams packed column tiles
//           (see ColFmt in common.cuh) global -> shared with 1-D bulk TMA copies into a STAGES-deep
//           ring guarded by full/empty mbarriers; the column cloud (16 B/column at D=3) stays in L2.
//   consumer thread = R rows; for each column pair it reads the packet with broadcast LDS.128 and
//           evaluates two columns at once as float2 pairs (two FFMA each on Hopper): at D=3 / p=2 a
//           column costs 3 FFMA + 1 FADD + 1 FMNMX + 1 MUFU.EX2 + 1 FADD per row, i.e. the loop is
//           bound by the 16-lane/SM MUFU unit, not by FP32 issue.  PMASK moves a fraction of the
//           exponentials to a polynomial on the FMA pipe (ex2_poly2) to balance the two units.
//   max     the running max is LAZY: exponentials of a chunk are taken against the max known before
//           the chunk (so MUFU and FMA work interleave freely inside a warp) and the max is only
//           raised — with the chunk recomputed — when a chunk exceeds it by more than kLazy.
//   p = 2 uses the expansion  -|X-Y|^2/2 = X.Y - |Y|^2/2 - |X|^2/2  on centred, pre-scaled
//           coordinates (the -|Y|^2/2 term lives in the packed per-column slot, -|X|^2/2 is a row
//           constant added to m at the end); DIRECT evaluates differences explicitly
//           (used for p = 1 and as the accuracy cross-check for p = 2).
#pragma once
#include "common.cuh"

namespace b200ot {

// 2^x on a pair, FMA pipe only (see ex2_poly in common.cuh for the scalar derivation).  Arguments are
// clamped to [-126, 127]: below, the result is ~2^-126 (the MUFU path flushes to 0; both are far below one
// ulp of any row sum); above, 2^127 makes the chunk sum overflow the 2^64 guard of the lazy max, exactly
// like the +inf of the MUFU path, so an outdated max is always detected.
__device__ __forceinline__ float2 ex2_poly2(float2 x) {
  x.x = fminf(fmaxf(x.x, -126.0f), 127.0f);
  x.y = fminf(fmaxf(x.y, -126.0f), 127.0f);
  const float2 magic = dup2(12582912.0f);
  float2 t = fadd2(x, magic);
  float2 n = fadd2(t, dup2(-12582912.0f));
  float2 f = ffma2(n, dup2(-1.0f), x);
  float2 p = dup2(1.3264726694e-3f);
  p = ffma2(p, f, dup2(9.6715127364e-3f));
  p = ffma2(p, f, dup2(5.5507337449e-2f));
  p = ffma2(p, f, dup2(2.4022242083e-1f));
  p = ffma2(p, f, dup2(6.9314697760e-1f));
  p = ffma2(p, f, dup2(1.0f));
  float2 r;
  r.x = __int_as_float(__float_as_int(p.x) + (__float_as_int(t.x) << 23));
  r.y = __int_as_float(__float_as_int(p.y) + (__float_as_int(t.y) << 23));
  return r;
}

template <int D_, int R_, int P_, bool DIRECT_, unsigned PMASK_ = 0u, int NT_ = 256, int TJ_ = 1024,
          int STAGES_ = 3, int CH_ = 4, int MINB_ = 2, bool GUARD_ = false>
struct SoftminCfg {
  static constexpr int D = D_;            // ambient dimension
  static constexpr int R = R_;            // rows per consumer thread
  static constexpr int P = P_;            // cost exponent (1 or 2)
  static constexpr bool DIRECT = DIRECT_; // explicit differences instead of the dot-product expansion
  static constexpr unsigned PMASK = PMASK_; // bit c set: column pair c of every chunk takes the FMA-pipe exp2
  static constexpr int NT = NT_;          // consumer threads
  static constexpr int TJ = TJ_;          // columns per tile
  static constexpr int STAGES = STAGES_;
  static constexpr int CH = CH_;          // column pairs per chunk (running max refreshed once per chunk)
  static constexpr int MINB = MINB_;      // CTAs per SM the register budget is planned for
  static constexpr bool GUARD = GUARD_;   // detect an outdated max from the chunk SUM (> 2^64) instead of
                                          // tracking the chunk max with one FMNMX3 per column pair
  static constexpr int NEXTRA = 1;
  static constexpr int NF2 = ((D + NEXTRA + 1) / 2) * 2;
  static constexpr int TILE_FLOATS = (TJ / 2) * NF2 * 2;
  static constexpr int TILE_BYTES = TILE_FLOATS * 4;
  static constexpr int ROWS_PER_CTA = NT * R;
  static constexpr int SMEM_BYTES = STAGES * TILE_BYTES + 2 * STAGES * 8;
  static_assert(P == 2 || DIRECT, "p = 1 needs explicit differences");
  static_assert((TJ / 2) % CH == 0, "tile must hold a whole number of chunks");
};

// Lazy-max slack (log2 units): the running max m is only raised when a chunk exceeds it by more than
// this, so exp2 arguments stay <= kLazy and row sums stay far below FLT_MAX (M * 2^64 ~ 1e25 for M = 1e6).
constexpr float kLazy = 64.0f;

// log2-domain exponent of one column pair against one row
template <class C>
__device__ __forceinline__ float2 pair_exponent(const float2 (&X)[C::D], const float2 (&S)[C::NF2], float clampq) {
  constexpr int D = C::D;
  float2 t;
  if constexpr (!C::DIRECT) {
    t = S[D];
#pragma unroll
    for (int d = 0; d < D; ++d) t = ffma2(X[d], S[d], t);
  } else {
    float2 qq;
#pragma unroll
    for (int d = 0; d < D; ++d) {
      const float2 df = fadd2(X[d], S[d]);  // packed columns hold -Y
      qq = (d == 0) ? fmul2(df, df) : ffma2(df, df, qq);
    }
    if constexpr (C::P == 2) {
      t = ffma2(qq, dup2(-0.5f), S[D]);
    } else {
      qq.x = fmaxf(qq.x, clampq);
      qq.y = fmaxf(qq.y, clampq);
      float2 dist;
      dist.x = sqrt_approx(qq.x);
      dist.y = sqrt_approx(qq.y);
      t = ffma2(dist, dup2(-1.0f), S[D]);
    }
  }
  return t;
}

template <int NF2>
__device__ __forceinline__ void load_packet(const float4* __restrict__ tp, int pair, float2 (&S)[NF2]) {
#pragma unroll
  for (int q = 0; q < NF2 / 2; ++q) {
    const float4 v = tp[pair * (NF2 / 2) + q];
    S[2 * q] = make_float2(v.x, v.y);
    S[2 * q + 1] = make_float2(v.z, v.w);
  }
}

// RANGES = false: dense grid (row tiles x column splits).  RANGES = true: segments + pieces (b200ot.h, "ranges mode");
// a separate instantiation so that the dense kernel — the headline path — carries none of its registers
// (measured: 65 vs 72 registers, 245.2 vs 248.2 ms at N = M = 1e6 when the two shared one body).
// GATED: the kernel returns at once unless *gate is set — the recomputation of a paired softmin whose sums left the
// plan-scale range (softmin_pair.cuh), always enqueued.  The gate is the last parameter, so the other instantiations
// keep their code.
template <class C, bool RANGES, bool GATED = false>
__global__ void __launch_bounds__(C::NT + 32, C::MINB)
    softmin_partial_kernel(const float* __restrict__ x, const float* __restrict__ center, float scale,
                           float clampq, const float* __restrict__ cols, float2* __restrict__ part, int64_t N,
                           int ntiles, int tiles_per_split, int last_pairs, const int4* __restrict__ seg,
                           const int2* __restrict__ pieces, const int* __restrict__ gate) {
  if constexpr (GATED) {
    if (*gate == 0) return;
  }
  constexpr int D = C::D, R = C::R, NT = C::NT, NF2 = C::NF2, CH = C::CH, STAGES = C::STAGES;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* tiles = reinterpret_cast<float*>(smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + STAGES * C::TILE_BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int split = blockIdx.y;
  // dense mode: this CTA owns ROWS_PER_CTA rows and reduces the contiguous tile range of its split;
  // ranges mode (seg != null; block-sparse / batched problems, see b200ot.h): the CTA owns the rows of ONE
  // segment and reduces the column pieces listed for it
  constexpr bool sparse = RANGES;
  int t0, t1, nrows;
  int64_t row0;
  if (sparse) {
    const int4 sg = seg[blockIdx.x];
    row0 = sg.x;
    nrows = sg.y;
    t0 = sg.z;
    t1 = sg.w;
  } else {
    row0 = (int64_t)blockIdx.x * C::ROWS_PER_CTA;
    nrows = 0;  // (dense mode bounds its rows with N, like the round-1 kernel: no extra live registers)
    t0 = split * tiles_per_split;
    t1 = min(ntiles, t0 + tiles_per_split);
  }
  const int nt = t1 - t0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], NT);  // every consumer THREAD releases the stage itself (see below)
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ===== producer: one elected lane streams the column tiles of this CTA =====
    if (lane == 0) {
      for (int k = 0; k < nt; ++k) {
        const int st = k % STAGES;
        if (k >= STAGES) mbar_wait(&empty[st], ((k / STAGES) + 1) & 1);
        if (sparse) {
          const int2 pc = pieces[t0 + k];  // (first column, column count): both multiples of 2 * CH
          const uint32_t bytes = (uint32_t)pc.y * (NF2 * 4);
          mbar_arrive_expect_tx(&full[st], bytes);
          tma_load_1d(tiles + st * C::TILE_FLOATS, cols + (int64_t)pc.x * NF2, bytes, &full[st]);
        } else {
          mbar_arrive_expect_tx(&full[st], C::TILE_BYTES);
          tma_load_1d(tiles + st * C::TILE_FLOATS, cols + (int64_t)(t0 + k) * C::TILE_FLOATS, C::TILE_BYTES,
                      &full[st]);
        }
      }
    }
    return;
  }

  // ===== consumers =====
  const int tid = threadIdx.x - 32;
  // local row of slot r.  Dense mode: tid + r*NT (all rows live but in the last CTA).  Ranges mode: a warp owns R*32
  // CONSECUTIVE rows, so a segment of n rows keeps ceil(n / (32 R)) warps busy and the others idle — segments are
  // whole clusters cut at ROWS_PER_CTA rows, i.e. often a full CTA followed by a sliver, or a small boundary cluster
  const auto local_row = [&](int r) { return sparse ? (lane + 32 * (R * (tid >> 5) + r)) : (tid + r * NT); };
  if constexpr (sparse) {
    if (local_row(0) - lane >= nrows) {
      // idle warp: no row of the segment — keep the ring's arrival counts in step, compute nothing
      for (int k = 0; k < nt; ++k) {
        const int st = k % STAGES;
        mbar_wait(&full[st], (k / STAGES) & 1);
        mbar_arrive(&empty[st]);
      }
      return;
    }
  }

  float2 X[R][D];
  float rowc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    int64_t i = row0 + local_row(r);
    if constexpr (sparse) {
      if (local_row(r) >= nrows) i = row0 + nrows - 1;
    } else {
      if (i >= N) i = N - 1;
    }
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < D; ++k) {
      const float c = center ? center[k] : 0.f;
      const float v = scale * (x[i * D + k] - c);
      X[r][k] = dup2(v);
      acc = fmaf(v, v, acc);
    }
    rowc[r] = C::DIRECT ? 0.f : -0.5f * acc;
  }

  // running (m, s): s = sum_j 2^(t_j - m); m trails the true running max by at most kLazy
  float m[R];
  float2 nm2[R], s2[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    m[r] = kNegBig;
    nm2[r] = dup2(-kNegBig);
    s2[r] = dup2(0.f);
  }

  // ranges mode: column pairs of the next piece, fetched one piece ahead (every thread reads the same descriptor word)
  // (dense mode: whole tiles, except that the last tile of the cloud ends at the chunk holding its last column)
  int np_next = sparse ? (nt > 0 ? (pieces[t0].y >> 1) : 0) : (t0 + 1 == ntiles ? last_pairs : C::TJ / 2);

  // Max pre-pass.  Starting from m = -inf, every chunk in which some row of the warp meets a term 2^64 above its stale
  // max is computed twice, and while the nearest columns of a row are still being discovered that is most chunks: it
  // costs a CTA about one extra tile-time (seeding m with the known answer removes it).  The exponents of the first kPrePairs column pairs — FMA-pipe work,
  // no MUFU — give a starting max after which such jumps are rare.
  if (nt > 0) {
    constexpr int kPrePairs = 256;
    mbar_wait(&full[0], 0);
    const float4* tp = reinterpret_cast<const float4*>(tiles);
    const int npre = np_next < kPrePairs ? np_next : kPrePairs;
#pragma unroll 4
    for (int c = 0; c < npre; ++c) {
      float2 S[NF2];
      load_packet<NF2>(tp, c, S);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float2 t = pair_exponent<C>(X[r], S, clampq);
        m[r] = fmax3(m[r], t.x, t.y);
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) nm2[r] = dup2(-m[r]);
  }
  for (int k = 0; k < nt; ++k) {
    const int st = k % STAGES;
    const int npairs = np_next;
    if constexpr (sparse) {
      if (k + 1 < nt) np_next = pieces[t0 + k + 1].y >> 1;
    } else {
      if (t0 + k + 2 == ntiles) np_next = last_pairs;
    }
    mbar_wait(&full[st], (k / STAGES) & 1);
    const float4* tp = reinterpret_cast<const float4*>(tiles + st * C::TILE_FLOATS);

    // two-level accumulation: chunk sums -> tile sum ts2 -> running sum s2 (keeps the fp32 summation
    // error at ~sqrt(chunks per tile) + sqrt(tiles) ulps instead of sqrt(M) ulps)
    float2 ts2[R];
#pragma unroll
    for (int r = 0; r < R; ++r) ts2[r] = dup2(0.f);

#pragma unroll 1
    for (int jp = 0; jp < npairs; jp += CH) {
      // speculative pass: exponentials against the (possibly stale) max, chunk max on the side.  p = 2: the chunk sum
      // starts from the first column pair's terms (no 0 + e); p = 1 keeps the zero start (measured 2 % faster at D = 1, 2)
      constexpr bool kFirst = !C::DIRECT;
      float2 cs[R];
      float cm[R];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        if (!kFirst) cs[r] = dup2(0.f);
        cm[r] = kNegBig;
      }
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        float2 S[NF2];
        load_packet<NF2>(tp, jp + c, S);
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const float2 t = pair_exponent<C>(X[r], S, clampq);
          if constexpr (!C::GUARD) cm[r] = fmax3(cm[r], t.x, t.y);
          const float2 a = fadd2(t, nm2[r]);
          float2 e;
          if (c < 32 && ((C::PMASK >> (c & 31)) & 1u)) {
            e = ex2_poly2(a);
          } else {
            e.x = ex2_approx(a.x);
            e.y = ex2_approx(a.y);
          }
          cs[r] = (kFirst && c == 0) ? e : fadd2(cs[r], e);
        }
      }
#pragma unroll
      for (int r = 0; r < R; ++r) {
        bool stale;
        if constexpr (C::GUARD) {
          // a term above 2^kLazy (or an overflow to +inf) shows up in the chunk sum
          stale = !(cs[r].x + cs[r].y <= 1.8446744e19f);
        } else {
          stale = cm[r] > m[r] + kLazy;
        }
        if (stale) {
          // rare: the chunk overshoots the stale max — rebase the row on the chunk max and redo the chunk
          if constexpr (C::GUARD) {
            cm[r] = kNegBig;
#pragma unroll 1
            for (int c = 0; c < CH; ++c) {
              float2 S[NF2];
              load_packet<NF2>(tp, jp + c, S);
              const float2 t = pair_exponent<C>(X[r], S, clampq);
              cm[r] = fmax3(cm[r], t.x, t.y);
            }
          }
          const float sc = ex2_approx(m[r] - cm[r]);
          s2[r] = fmul2(s2[r], dup2(sc));
          ts2[r] = fmul2(ts2[r], dup2(sc));
          m[r] = cm[r];
          nm2[r] = dup2(-cm[r]);
          float2 acc = dup2(0.f);
#pragma unroll 1
          for (int c = 0; c < CH; ++c) {
            float2 S[NF2];
            load_packet<NF2>(tp, jp + c, S);
            const float2 a = fadd2(pair_exponent<C>(X[r], S, clampq), nm2[r]);
            acc.x += ex2_approx(a.x);
            acc.y += ex2_approx(a.y);
          }
          cs[r] = acc;
        }
        ts2[r] = fadd2(ts2[r], cs[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) s2[r] = fadd2(s2[r], ts2[r]);
    // release: each thread arrives after ITS OWN last read of the stage (an elected lane behind a __syncwarp() is as
    // correct, but compute-sanitizer's racecheck does not follow that hand-over and reports the refill as a WAR hazard)
    mbar_arrive(&empty[st]);
  }

#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int64_t i = row0 + local_row(r);
    const bool live = sparse ? (local_row(r) < nrows) : (i < N);
    if (live) part[(int64_t)split * N + i] = make_float2(m[r] + rowc[r], s2[r].x + s2[r].y);
  }
}

}  // namespace b200ot
