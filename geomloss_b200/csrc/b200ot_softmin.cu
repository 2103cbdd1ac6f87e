// b200ot — softmin forward: column packing, partial-reduction dispatch, merge / finalize, C ABI.
// Interface contract: include/b200ot.h.  Reference semantics: softmin_tensorized
// (src/geomloss/_legacy/sinkhorn_samples.py:32-71) with the cost routines of :26-29 /
// src/geomloss/_legacy/utils.py:26-61.
#include "b200ot.h"
#include "host_util.cuh"
#include "pack.cuh"
#include "plan.cuh"
#include "softmin.cuh"
#include "softmin_pair.cuh"

#include <string.h>

#include <algorithm>

namespace b200ot {

// -------------------------------------------------------------------------------------------------
// merge / finalize of partial (m, s) pairs
//   lse2 = M + log2( sum_s s_s 2^(m_s - M) ),  val = -eps ln2 lse2,  out = alpha_old*old + beta*val
// -------------------------------------------------------------------------------------------------
// The merge and the final log run in fp64: with the lazy running max a partial sum can be as large as
// M * 2^64, and log2f of such a value is only accurate to ulp(64) ~ 8e-6 — visible at large eps.
// This is N elements per softmin (elementwise), so the fp64 rate of the part is irrelevant.
struct MergedMS {
  float m;
  double s;
};
__device__ __forceinline__ MergedMS merge_ms(const float2* __restrict__ part, int n_part, int64_t N, int64_t i) {
  float mm = kNegBig;
  for (int s = 0; s < n_part; ++s) mm = fmaxf(mm, part[(int64_t)s * N + i].x);
  double ss = 0.0;
  for (int s = 0; s < n_part; ++s) {
    const float2 p = part[(int64_t)s * N + i];
    ss += (double)p.y * exp2((double)p.x - (double)mm);
  }
  MergedMS r;
  r.m = mm;
  r.s = ss;
  return r;
}

__global__ void softmin_merge_kernel(const float2* __restrict__ part, int n_part, float2* __restrict__ out,
                                     int64_t N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  // renormalise so that the merged pair is again (max-like reference, O(1)..O(M) sum) in fp32
  const MergedMS ms = merge_ms(part, n_part, N, i);
  int e = 0;
  const double frac = frexp(ms.s, &e);  // s = frac * 2^e, frac in [0.5, 1)
  out[i] = ms.s > 0.0 ? make_float2(ms.m + (float)e, (float)frac) : make_float2(ms.m, 0.f);
}

// kFinPlain: the epilogue of every softmin.  kFinChecked: also sets *flag when a merged sum is not finite or leaves
// [min_sum, 2^100] — the range in which the plan-scale sums of a paired softmin are exact (softmin_pair.cuh).
// kFinGated: returns at once unless *flag is set (the recomputation of such a softmin on the unpaired path).
enum { kFinPlain = 0, kFinChecked = 1, kFinGated = 2 };
template <int MODE>
__global__ void softmin_finalize_kernel(const float2* __restrict__ part, int n_part,
                                        const float* __restrict__ out_old, float alpha_old, float beta,
                                        float* __restrict__ out, float* __restrict__ lse2_out, int64_t N,
                                        float neg_eps_ln2, int* __restrict__ flag, double min_sum) {
  if constexpr (MODE == kFinGated) {
    if (*flag == 0) return;
  }
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const MergedMS ms = merge_ms(part, n_part, N, i);
  if constexpr (MODE == kFinChecked) {
    if (!(ms.s >= min_sum && ms.s <= 0x1p100)) *flag = 1;
  }
  const double lse2 = (double)ms.m + log2(ms.s);
  if (lse2_out) lse2_out[i] = (float)lse2;
  if (out) {
    double v = (double)neg_eps_ln2 * lse2 * (double)beta;
    if (out_old) v += (double)alpha_old * (double)out_old[i];
    out[i] = (float)v;
  }
}

// -------------------------------------------------------------------------------------------------
// dispatch
// -------------------------------------------------------------------------------------------------
// Dense big shape: sum-guarded lazy max, 512 rows per CTA (the plan's kBigNT * kBigR) split as NT threads x R rows.
// What matters is the length of the straight-line chunk between two max checks (longer chunks give the scheduler more
// independent MUFU work, but cost registers, and on a short column shard the tail of the last chunk) and, at D = 3, 4,
// how many shared-memory packet loads feed one MUFU.EX2: both go through the MIO queue.
//   D = 3, p = 2:  4 rows x 128 threads, 32-pair chunks, 4 CTAs/SM (94 registers);
//   D = 4, p = 2:  2 rows x 256 threads, 32-pair chunks, 3 CTAs/SM, 2-stage ring;
//   D = 1, 2:      2 x 256, 8 pairs with one polynomial exp2 in eight (so little FMA work per pair that it pays);
//   D >= 5:        2 x 256, 8 pairs, 2 CTAs/SM (no registers to spare); p = 1 (DIRECT) 2 x 256, 16 pairs.
// D = 3, 4 were chosen on an H100 SXM (700 W) by tools/bench_softmin_sm90.py: 0.85 / 0.75 of the MUFU.EX2 rate at the
// sampled clock, against 0.81 / 0.72 for the 2 x 256 / 16-pair / 3-CTA shape; an FMA-pipe share of the exponentials
// (ex2_poly2) was slower at every shape tried (DESIGN.md §3.1 has the sweep).
// Ranges mode keeps 2 x 256 and 8-pair chunks: its pieces must be multiples of 2*CH columns, and 16-slot cluster padding
// (kRangesAlign) costs less than the longer chunk gains on cluster-sized pieces.
// A/B builds (tools/ab_ops.py, tools/bench_softmin_sm90.py) override the dense shape with -DB200OT_BIG_CH (every D),
// -DB200OT_BIG_POLY (D <= 4, p = 2), -DB200OT_BIG_R / _MINB / _STAGES (D = 3, 4, p = 2).
template <int D, int P, bool DIRECT>
struct Variants {
  static constexpr bool kD34 = (D == 3 || D == 4) && P == 2 && !DIRECT;
#ifdef B200OT_BIG_CH
  static constexpr int kCH = B200OT_BIG_CH;
#else
  static constexpr int kCH = (DIRECT || D == 3 || D == 4) ? (kD34 ? 32 : 16) : 8;
#endif
#ifdef B200OT_BIG_POLY
  static constexpr unsigned kPoly = (D <= 4 && P == 2 && !DIRECT) ? B200OT_BIG_POLY : 0u;
#else
  static constexpr unsigned kPoly = (D <= 2 && P == 2 && !DIRECT) ? 0x01u : 0u;
#endif
#ifdef B200OT_BIG_R
  static constexpr int kR = kD34 ? B200OT_BIG_R : kBigR;
#else
  static constexpr int kR = (kD34 && D == 3) ? 4 : kBigR;
#endif
#ifdef B200OT_BIG_MINB
  static constexpr int kMinB = kD34 ? B200OT_BIG_MINB : (D <= 4 ? 3 : 2);
#else
  static constexpr int kMinB = (kD34 && D == 3) ? 4 : (D <= 4 ? 3 : 2);
#endif
#ifdef B200OT_BIG_STAGES
  static constexpr int kStages = kD34 ? B200OT_BIG_STAGES : 3;
#else
  static constexpr int kStages = (kD34 && D == 4) ? 2 : 3;
#endif
  using Big = SoftminCfg<D, kR, P, DIRECT, kPoly, kBigNT * kBigR / kR, kBigTJ, kStages, kCH, kMinB, true>;
  using BigRanges = SoftminCfg<D, kBigR, P, DIRECT, 0u, kBigNT, kBigTJ, 3, 8, (D <= 4 ? 3 : 2), true>;
  using Small = SoftminCfg<D, kSmallR, P, DIRECT, 0u, kSmallNT, kSmallTJ, 3, 4, 4, true>;
  static_assert(2 * BigRanges::CH <= kRangesAlign && 2 * Small::CH <= kRangesAlign,
                "ranges pieces are kRangesAlign-aligned");
};

template <class C, class CR = C>
static int launch_partial(const float* x, const float* center, float scale, float clampq, const float* cols,
                          float* part, const ReducePlan& pl, int64_t N, cudaStream_t st, const int4* seg,
                          const int2* pieces) {
  // the plan fixes rows per CTA and the shared-memory opt-in; the CTA shape (NT x R) may differ
  static_assert(C::ROWS_PER_CTA == CR::ROWS_PER_CTA && C::TJ == CR::TJ, "dense and ranges instantiations share one ReducePlan");
  if (seg != nullptr)
    return launch_reduce<CR>(softmin_partial_kernel<CR, true>, pl, st, x, center, scale, clampq, cols,
                             reinterpret_cast<float2*>(part), N, pl.ntiles, pl.tiles_per_split, 0, seg, pieces,
                             (const int*)nullptr);
  return launch_reduce<C>(softmin_partial_kernel<C, false>, pl, st, x, center, scale, clampq, cols,
                          reinterpret_cast<float2*>(part), N, pl.ntiles, pl.tiles_per_split, pl.last_pairs, seg,
                          pieces, (const int*)nullptr);
}

template <int D>
static int partial_for_d(int p, const float* x, const float* center, float scale, float clampq, const float* cols,
                         float* part, const ReducePlan& pl, int64_t N, cudaStream_t st, const int4* seg,
                         const int2* pieces) {
  if (p == 2) {
    using V = Variants<D, 2, false>;
    return pl.small ? launch_partial<typename V::Small>(x, center, scale, clampq, cols, part, pl, N, st, seg, pieces)
                    : launch_partial<typename V::Big, typename V::BigRanges>(x, center, scale, clampq, cols, part, pl, N, st, seg, pieces);
  } else {
    using V = Variants<D, 1, true>;
    return pl.small ? launch_partial<typename V::Small>(x, center, scale, clampq, cols, part, pl, N, st, seg, pieces)
                    : launch_partial<typename V::Big, typename V::BigRanges>(x, center, scale, clampq, cols, part, pl, N, st, seg, pieces);
  }
}

// `p` may carry B200OT_P_UNCLAMPED; M = number of column slots (gather mode: src maps slots to columns)
int softmin_pack_impl(const float* y, const float* h_a, const float* h_b, float h_scale_b, const float* center,
                      int64_t M, int D, int p, float eps, float* cols_out, cudaStream_t st, const int* src,
                      const int* gate) {
  const int pe = p_exponent(p);
  const int nf2 = colfmt_nf2(D, 1);
  const int64_t mpad = round_up64(M, kPackPad);
  const int threads = 256;
  pack_cols_kernel<<<(unsigned)ceil_div64(mpad, threads), threads, 0, st>>>(
      y, h_a, h_b, h_scale_b, kLog2e, nullptr, center, softmin_coord_scale(pe, eps), pe == 1 ? 1 : 0, D, nf2, M,
      mpad, cols_out, src, gate);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

static int softmin_partial_impl(const float* x, const float* center, const float* cols, float* part,
                                const ReducePlan& pl, int64_t N, int D, int p, float eps, cudaStream_t st,
                                const int4* seg = nullptr, const int2* pieces = nullptr) {
  const int pe = p_exponent(p);
  const float scale = softmin_coord_scale(pe, eps);
  // reference clamp on |x-y|^2 (utils.py:61) — or none (pykeops' Norm2) — in scaled units
  const float clampq = scale * scale * cost_clamp(p);
  switch (D) {
    case 1: return partial_for_d<1>(pe, x, center, scale, clampq, cols, part, pl, N, st, seg, pieces);
    case 2: return partial_for_d<2>(pe, x, center, scale, clampq, cols, part, pl, N, st, seg, pieces);
    case 3: return partial_for_d<3>(pe, x, center, scale, clampq, cols, part, pl, N, st, seg, pieces);
    case 4: return partial_for_d<4>(pe, x, center, scale, clampq, cols, part, pl, N, st, seg, pieces);
    case 5: return partial_for_d<5>(pe, x, center, scale, clampq, cols, part, pl, N, st, seg, pieces);
    case 6: return partial_for_d<6>(pe, x, center, scale, clampq, cols, part, pl, N, st, seg, pieces);
    case 7: return partial_for_d<7>(pe, x, center, scale, clampq, cols, part, pl, N, st, seg, pieces);
    case 8: return partial_for_d<8>(pe, x, center, scale, clampq, cols, part, pl, N, st, seg, pieces);
    default: return B200OT_EINVAL;
  }
}

// -------------------------------------------------------------------------------------------------
// paired softmins (softmin_pair.cuh): D = 3, p = 2, the dense big plan
// -------------------------------------------------------------------------------------------------
// the epilogue arguments of one softmin (b200ot_softmin_finalize)
struct SoftminOut {
  const float* out_old;
  float alpha_old, beta;
  float* out;
  float* lse2;
};

template <int MODE>
static int finalize_launch(const float2* part, int n_part, const SoftminOut& o, int64_t N, float eps, int* flag,
                           double min_sum, cudaStream_t st) {
  const int threads = 256;
  softmin_finalize_kernel<MODE><<<(unsigned)ceil_div64(N, threads), threads, 0, st>>>(
      part, n_part, o.out_old, o.alpha_old, o.beta, o.out, o.lse2, N, -eps * kLn2, flag, min_sum);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

// 8 rows per thread, 4 CTAs/SM in 96 registers
using PairC = PairCfg<8, 128, 4>;

// $B200OT_PAIR=0 (read on every call): every softmin takes the unpaired path, for A/B runs and tests
static bool pair_on() {
  const char* e = getenv("B200OT_PAIR");
  return !(e && strcmp(e, "0") == 0);
}

// The shapes the paired kernels serve: what the unpaired path would run on softmin_partial_kernel's big plan
static bool pair_shape(int64_t N, int64_t M, int D, int p) {
  return D == 3 && p_exponent(p) == 2 && !make_plan(N, M, D).small && !tc_routed(kTcSoftminFwd, D, N, M) &&
         !tc_routed(kTcSoftminFwd, D, M, N);
}

// Blocks of whole tiles along an axis of n points: as few tiles per block as keep the partial slots at 64 or fewer.
// Test hook $B200OT_PAIR_TILES: at least that many tiles per block (1: many blocks at small sizes).
static int pair_blocks(int64_t n) {
  const int nt = (int)ceil_div64(n, PairC::TJ);
  int tpb = (int)ceil_div64(nt, 64);
  const char* e = getenv("B200OT_PAIR_TILES");
  const int forced = e ? atoi(e) : 0;
  if (forced > tpb) tpb = forced;
  return (int)ceil_div64(nt, tpb);
}

// The unpaired path's scratch (b200ot_softmin_fwd at a shape the paired kernels serve)
static int64_t unpaired_bytes(int64_t N, int64_t M) {
  return round_up64(b200ot_packed_cols_floats(M, 3, 1) * 4, 256) +
         round_up64((int64_t)make_plan(N, M, 3).n_split * N * 16, 256);
}
static int64_t packed_bytes(int64_t n) { return round_up64(b200ot_packed_cols_floats(n, 3, 1) * 4, 256); }
// One softmin of a paired launch group: rows (nr points) against columns (nc points, column potential
// h_a + h_s * h_b), with its epilogue
struct PairedSoftmin {
  const float* rows;
  const float* cols;
  int64_t nr, nc;
  const float *h_a, *h_b;
  float h_s;
  SoftminOut o;
};
// Scratch: the range flags (one per softmin), then the region the paired pass uses and the recomputation reuses: each
// softmin's packed columns, then each softmin's partials
constexpr int64_t kPairFlagBytes = 256;
static int64_t paired_bytes(const int64_t (*shape)[2], int n) {
  int64_t paired = 0, unpaired = 0;
  for (int k = 0; k < n; ++k) {
    paired += packed_bytes(shape[k][1]) + round_up64((int64_t)pair_blocks(shape[k][1]) * shape[k][0] * 8, 256);
    unpaired = std::max(unpaired, unpaired_bytes(shape[k][0], shape[k][1]));
  }
  return kPairFlagBytes + std::max(paired, unpaired);
}
static int64_t sym_bytes(int64_t N) {
  const int64_t shape[1][2] = {{N, N}};
  return paired_bytes(shape, 1);
}
static int64_t pair_bytes(int64_t N, int64_t M) {
  const int64_t shape[2][2] = {{N, M}, {M, N}};
  return paired_bytes(shape, 2);
}
static int64_t step_bytes(int64_t N, int64_t M) {
  const int64_t shape[4][2] = {{N, M}, {M, N}, {N, N}, {M, M}};
  return paired_bytes(shape, 4);
}

static bool overlaps(const void* a, int64_t na, const void* b, int64_t nb) {
  if (!a || !b) return false;
  const char *pa = (const char*)a, *pb = (const char*)b;
  return pa < pb + nb * 4 && pb < pa + na * 4;
}
// An output of the group s[0..n) overlaps an input of the group or another output: the recomputation of a softmin
// reads every input after the finalizes wrote the outputs
static bool paired_aliased(const PairedSoftmin* s, int n, const float* center) {
  for (int a = 0; a < n; ++a)
    for (int fa = 0; fa < 2; ++fa) {
      const float* o = fa ? s[a].o.lse2 : s[a].o.out;
      if (overlaps(o, s[a].nr, center, 3)) return true;
      for (int b = 0; b < n; ++b) {
        const void* ins[] = {s[b].rows, s[b].cols, s[b].h_a, s[b].h_b, s[b].o.out_old};
        const int64_t lens[] = {s[b].nr * 3, s[b].nc * 3, s[b].nc, s[b].nc, s[b].nr};
        for (int k = 0; k < 5; ++k)
          if (overlaps(o, s[a].nr, ins[k], lens[k])) return true;
        for (int fb = 0; fb < 2; ++fb)
          if ((a != b || fa != fb) && overlaps(o, s[a].nr, fb ? s[b].o.lse2 : s[b].o.out, s[b].nr)) return true;
      }
    }
  return false;
}

// Today's pack -> partial -> finalize of one softmin (rows x, columns y), every launch returning at once unless *gate
// is set: bit for bit what b200ot_softmin_fwd computes on the unpaired path
static int softmin_fwd_gated(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                             const float* center, int64_t N, int64_t M, float eps, const SoftminOut& o, void* region,
                             int* gate, cudaStream_t st) {
  using C = Variants<3, 2, false>::Big;
  const ReducePlan pl = make_plan(N, M, 3);
  float* cols = reinterpret_cast<float*>(region);
  float* part = reinterpret_cast<float*>(reinterpret_cast<char*>(region) + packed_bytes(M));
  int rc = softmin_pack_impl(y, h_a, h_b, h_scale_b, center, M, 3, 2, eps, cols, st, nullptr, gate);
  if (rc) return rc;
  const float scale = softmin_coord_scale(2, eps);
  rc = launch_reduce<C>(softmin_partial_kernel<C, false, true>, pl, st, x, center, scale, scale * scale * cost_clamp(2),
                        (const float*)cols, reinterpret_cast<float2*>(part), N, pl.ntiles, pl.tiles_per_split,
                        pl.last_pairs, (const int4*)nullptr, (const int2*)nullptr, (const int*)gate);
  if (rc) return rc;
  return finalize_launch<kFinGated>(reinterpret_cast<const float2*>(part), pl.n_split, o, N, eps, gate, 0.0, st);
}

// One launch of softmin_pair_kernel over 1 to 3 problems: one CTA per item, the items longest first, so the block
// scheduler hands out the long ones first and one tail ends the launch
static int pair_launch(const PairProblem* probs, int nprob, cudaStream_t st) {
  PairLaunch L{};
  for (int p = 0; p < nprob; ++p) {
    const PairProblem& P = probs[p];
    L.prob[p] = P;
    const int qr = P.ntr / P.nbr, qc = P.ntc / P.nbc;
    for (int tr = qr + 1; tr >= qr; --tr)
      for (int tc = qc + 1; tc >= qc; --tc) {
        const int nr = pair_blocks_of_size(tr, P.ntr, P.nbr), nc = pair_blocks_of_size(tc, P.ntc, P.nbc);
        // sym: the unordered pairs within one size class, or of one block of each size (as class (q + 1, q))
        const int count = !P.sym ? nr * nc : tr == tc ? nr * (nr + 1) / 2 : tr > tc ? nr * nc : 0;
        if (count > 0) L.cls[L.ncls++] = PairClass{p, tr, tc, count};  // start holds the count until the sort
      }
  }
  // longest first (stable: ties keep problem order)
  std::stable_sort(L.cls, L.cls + L.ncls, [](const PairClass& a, const PairClass& b) { return a.tr * a.tc > b.tr * b.tc; });
  for (int c = 0; c < L.ncls; ++c) {
    const int count = L.cls[c].start;
    L.cls[c].start = L.items;
    L.items += count;
  }
  const auto kern = softmin_pair_kernel<PairC>;
  B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, PairC::SMEM_BYTES));
  kern<<<L.items, PairC::NT + 32, PairC::SMEM_BYTES, st>>>(L);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

// The softmins s[0..n) as one launch group: n = 1, one symmetric softmin (rows are columns); n = 2, a mirrored pair
// (s[1] is s[0] with rows and columns swapped); n = 4, that pair and the symmetric softmins of its rows (s[2]) and of
// its columns (s[3]).  Zero the flags; pack each softmin's columns with its potential; one paired pass; the range
// check of every sum; then the gated recomputation of each softmin that failed it, after all the checks since it reuses
// the region.  Arguments validated by the caller; scratch >= paired_bytes of the shapes.
static int paired_fwd(const PairedSoftmin* s, int n, const float* center, float eps, void* scratch, cudaStream_t st) {
  int* flags = reinterpret_cast<int*>(scratch);
  char* region = reinterpret_cast<char*>(scratch) + kPairFlagBytes;
  float* pk[4];
  float2* part[4];
  char* at = region;
  for (int k = 0; k < n; ++k) {
    pk[k] = reinterpret_cast<float*>(at);
    at += packed_bytes(s[k].nc);
  }
  for (int k = 0; k < n; ++k) {
    part[k] = reinterpret_cast<float2*>(at);
    at += round_up64((int64_t)pair_blocks(s[k].nc) * s[k].nr * 8, 256);
  }
  B200OT_CUDA_TRY(cudaMemsetAsync(flags, 0, n * sizeof(int), st));
  for (int k = 0; k < n; ++k)
    if (const int rc = softmin_pack_impl(s[k].cols, s[k].h_a, s[k].h_b, s[k].h_s, center, s[k].nc, 3, 2, eps, pk[k], st,
                                         nullptr))
      return rc;
  // a pair reads its rows from the pack of the mirrored softmin, a symmetric softmin from its own
  const auto problem = [&](int a, int b) {
    const int64_t N = s[a].nr, M = s[a].nc;
    const int ntr = (int)ceil_div64(N, PairC::TJ), ntc = (int)ceil_div64(M, PairC::TJ);
    return PairProblem{pk[b], pk[a], part[a], part[b], N, M, ntr, ntc, pair_blocks(N), pair_blocks(M), a == b};
  };
  PairProblem probs[kPairMaxProblems];
  int np = 0;
  if (n == 1) {
    probs[np++] = problem(0, 0);
  } else {
    probs[np++] = problem(0, 1);
    if (n == 4) {
      probs[np++] = problem(2, 2);
      probs[np++] = problem(3, 3);
    }
  }
  if (const int rc = pair_launch(probs, np, st)) return rc;
  // a point's merged sum must stay within [count 2^-100, 2^100]: the terms flushed below 2^-126 then weigh less
  // than 2^-26 of it (DESIGN.md §3.1b)
  for (int k = 0; k < n; ++k)
    if (const int rc = finalize_launch<kFinChecked>(part[k], pair_blocks(s[k].nc), s[k].o, s[k].nr, eps, flags + k,
                                                    (double)s[k].nc * 0x1p-100, st))
      return rc;
  for (int k = 0; k < n; ++k)
    if (const int rc = softmin_fwd_gated(s[k].rows, s[k].cols, s[k].h_a, s[k].h_b, s[k].h_s, center, s[k].nr, s[k].nc,
                                         eps, s[k].o, region, flags + k, st))
      return rc;
  return B200OT_OK;
}

}  // namespace b200ot

using namespace b200ot;

extern "C" {

B200OT_API int64_t b200ot_packed_cols_floats(int64_t M, int32_t D, int32_t extra) {
  if (M <= 0 || D <= 0 || extra < 1) return 0;
  return round_up64(M, kPackPad) / 2 * colfmt_nf2(D, extra) * 2;
}

B200OT_API int32_t b200ot_softmin_num_splits(int64_t N, int64_t M, int32_t D) {
  (void)D;
  if (N <= 0 || M <= 0) return 0;
  return make_plan(N, M, D).n_split;
}

B200OT_API int64_t b200ot_softmin_scratch_bytes(int64_t N, int64_t M, int32_t D) {
  if (N <= 0 || M <= 0 || D <= 0) return 0;
  if (D > B200OT_MAX_D) return tc_capable_dim(D) ? tc_scratch_bytes(N, M, D) : 0;
  const ReducePlan pl = make_plan(N, M, D);
  const int64_t cols = b200ot_packed_cols_floats(M, D, 1) * 4;
  // forward partials are (m, s) pairs; the backward pass keeps D+1 sums per (split, row)
  const int64_t part = (int64_t)pl.n_split * N * 4 * (D + 1 > 2 ? D + 1 : 2);
  int64_t simt = round_up64(cols, 256) + round_up64(part, 256);
  if (N == M && pair_shape(N, M, D, 2)) simt = std::max(simt, sym_bytes(N));  // x may be y: the symmetric kernel
  if (!tc_any_routed(D, N, M)) return simt;
  const int64_t tc = tc_scratch_bytes(N, M, D);
  return simt > tc ? simt : tc;
}

B200OT_API int b200ot_softmin_pack(const float* y, const float* h_a, const float* h_b, float h_scale_b,
                                   const float* center, int64_t M, int32_t D, int32_t p, float eps,
                                   float* cols_out, void* stream) {
  if (!y || !h_a || !cols_out || M <= 0 || !supported_simt_dim(D) || !valid_p(p) || !(eps > 0.f))
    return B200OT_EINVAL;
  if (((uintptr_t)cols_out) & 15) return B200OT_EALIGN;
  return softmin_pack_impl(y, h_a, h_b, h_scale_b, center, M, D, p, eps, cols_out, (cudaStream_t)stream, nullptr);
}

B200OT_API int b200ot_softmin_partial(const float* x, const float* center, const float* cols, float* part,
                                      int32_t n_split, int64_t N, int64_t M, int32_t D, int32_t p, float eps,
                                      void* stream) {
  if (!x || !cols || !part || N <= 0 || M <= 0 || !supported_simt_dim(D) || !valid_p(p) || !(eps > 0.f))
    return B200OT_EINVAL;
  if ((((uintptr_t)cols) & 15) || (((uintptr_t)part) & 7)) return B200OT_EALIGN;
  const ReducePlan pl = make_plan(N, M, D);
  if (n_split != pl.n_split) return B200OT_EINVAL;
  return softmin_partial_impl(x, center, cols, part, pl, N, D, p, eps, (cudaStream_t)stream);
}

B200OT_API void b200ot_ranges_shape(int32_t variant, int32_t* max_rows_per_segment, int32_t* max_cols_per_piece,
                                    int32_t* col_align) {
  const bool small = (variant == B200OT_RANGES_SMALL);
  if (max_rows_per_segment) *max_rows_per_segment = small ? kSmallNT * kSmallR : kBigNT * kBigR;
  if (max_cols_per_piece) *max_cols_per_piece = small ? kSmallTJ : kBigTJ;
  if (col_align) *col_align = kRangesAlign;
}

B200OT_API int b200ot_softmin_pack_gather(const float* y, const float* h_a, const float* h_b, float h_scale_b,
                                          const float* center, const int32_t* src_index, int64_t n_slots, int32_t D,
                                          int32_t p, float eps, float* cols_out, void* stream) {
  if (!y || !h_a || !src_index || !cols_out || n_slots <= 0 || !supported_simt_dim(D) || !valid_p(p) || !(eps > 0.f))
    return B200OT_EINVAL;
  if (((uintptr_t)cols_out) & 15) return B200OT_EALIGN;
  return softmin_pack_impl(y, h_a, h_b, h_scale_b, center, n_slots, D, p, eps, cols_out, (cudaStream_t)stream,
                           reinterpret_cast<const int*>(src_index));
}

B200OT_API int b200ot_softmin_partial_ranges(const float* x, const float* center, const float* cols,
                                             const b200ot_segment* seg, int64_t n_seg, const b200ot_piece* pieces,
                                             float* part, int64_t N, int32_t D, int32_t p, float eps,
                                             int32_t variant, void* stream) {
  if (!x || !cols || !seg || !pieces || !part || N <= 0 || n_seg <= 0 || n_seg > 0x7fffffff ||
      !supported_simt_dim(D) || !valid_p(p) || !(eps > 0.f) ||
      (variant != B200OT_RANGES_BIG && variant != B200OT_RANGES_SMALL))
    return B200OT_EINVAL;
  if ((((uintptr_t)cols) & 15) || (((uintptr_t)part) & 7) || (((uintptr_t)seg) & 15) || (((uintptr_t)pieces) & 7))
    return B200OT_EALIGN;
  const ReducePlan pl = ranges_plan(variant, n_seg);
  return softmin_partial_impl(x, center, cols, part, pl, N, D, p, eps, (cudaStream_t)stream,
                              reinterpret_cast<const int4*>(seg), reinterpret_cast<const int2*>(pieces));
}

B200OT_API int b200ot_softmin_merge(const float* part, int32_t n_part, float* merged, int64_t N, void* stream) {
  if (!part || !merged || n_part <= 0 || N <= 0) return B200OT_EINVAL;
  if ((((uintptr_t)part) & 7) || (((uintptr_t)merged) & 7)) return B200OT_EALIGN;
  const int threads = 256;
  softmin_merge_kernel<<<(unsigned)ceil_div64(N, threads), threads, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(part), n_part, reinterpret_cast<float2*>(merged), N);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

B200OT_API int b200ot_softmin_finalize(const float* part, int32_t n_part, const float* out_old, float alpha_old,
                                       float beta, float* out, float* lse2_out, int64_t N, float eps,
                                       void* stream) {
  if (!part || n_part <= 0 || N <= 0 || (!out && !lse2_out) || !(eps > 0.f)) return B200OT_EINVAL;
  if (((uintptr_t)part) & 7) return B200OT_EALIGN;
  const int threads = 256;
  return finalize_launch<kFinPlain>(reinterpret_cast<const float2*>(part), n_part,
                                    SoftminOut{out_old, alpha_old, beta, out, lse2_out}, N, eps, nullptr, 0.0,
                                    (cudaStream_t)stream);
}

B200OT_API int b200ot_softmin_fwd(const float* x, const float* y, const float* h_a, const float* h_b,
                                  float h_scale_b, const float* center, const float* out_old, float alpha_old,
                                  float beta, float* out, float* lse2_out, int64_t N, int64_t M, int32_t D,
                                  int32_t p, float eps, void* scratch, int64_t scratch_bytes, void* stream) {
  const bool tc = p_exponent(p) == 2 && tc_routed(kTcSoftminFwd, D, N, M);  // exponent from the tensor cores (tcconv.cuh)
  if (!x || !y || !h_a || !scratch || N <= 0 || M <= 0 || (!supported_simt_dim(D) && !tc) || !valid_p(p) ||
      !(eps > 0.f) || (!out && !lse2_out))
    return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, b200ot_softmin_scratch_bytes(N, M, D))) return rc;
  if (tc)
    return tc_softmin_fwd(x, y, h_a, h_b, h_scale_b, center, out_old, alpha_old, beta, out, lse2_out, N, M, D, p, eps,
                          scratch, stream);
  cudaStream_t st = (cudaStream_t)stream;
  const SoftminOut o{out_old, alpha_old, beta, out, lse2_out};
  if (x == y && N == M && pair_on() && pair_shape(N, M, D, p)) {
    // one exponential per unordered pair; refused when an output overlaps an input the recomputation would read
    const PairedSoftmin sym{x, x, N, N, h_a, h_b, h_scale_b, o};
    if (!paired_aliased(&sym, 1, center)) return paired_fwd(&sym, 1, center, eps, scratch, st);
  }
  const ReducePlan pl = make_plan(N, M, D);
  float* cols = reinterpret_cast<float*>(scratch);
  float* part = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) +
                                         round_up64(b200ot_packed_cols_floats(M, D, 1) * 4, 256));
  int rc = softmin_pack_impl(y, h_a, h_b, h_scale_b, center, M, D, p, eps, cols, st, nullptr);
  if (rc) return rc;
  rc = softmin_partial_impl(x, center, cols, part, pl, N, D, p, eps, st);
  if (rc) return rc;
  return b200ot_softmin_finalize(part, pl.n_split, out_old, alpha_old, beta, out, lse2_out, N, eps, stream);
}

B200OT_API int64_t b200ot_softmin_pair_scratch_bytes(int64_t N, int64_t M, int32_t D) {
  if (N <= 0 || M <= 0 || !pair_shape(N, M, D, 2)) return 0;
  return pair_bytes(N, M);
}

B200OT_API int b200ot_softmin_fwd_pair(const float* x, const float* y, const float* hy_a, const float* hy_b,
                                       float hy_scale_b, const float* out_a_old, float alpha_a_old, float beta_a,
                                       float* out_a, float* lse2_a, const float* hx_a, const float* hx_b,
                                       float hx_scale_b, const float* out_b_old, float alpha_b_old, float beta_b,
                                       float* out_b, float* lse2_b, const float* center, int64_t N, int64_t M,
                                       int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                       void* stream) {
  if (!x || !y || !hy_a || !hx_a || !scratch || N <= 0 || M <= 0 || !valid_p(p) || !(eps > 0.f) ||
      (!out_a && !lse2_a) || (!out_b && !lse2_b) || !pair_shape(N, M, D, p))
    return B200OT_EINVAL;
  const PairedSoftmin s[2] = {{x, y, N, M, hy_a, hy_b, hy_scale_b, {out_a_old, alpha_a_old, beta_a, out_a, lse2_a}},
                               {y, x, M, N, hx_a, hx_b, hx_scale_b, {out_b_old, alpha_b_old, beta_b, out_b, lse2_b}}};
  if (paired_aliased(s, 2, center)) return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, pair_bytes(N, M))) return rc;
  return paired_fwd(s, 2, center, eps, scratch, (cudaStream_t)stream);
}

B200OT_API int64_t b200ot_softmin_step_scratch_bytes(int64_t N, int64_t M, int32_t D) {
  if (N <= 0 || M <= 0 || !pair_shape(N, M, D, 2) || !pair_shape(N, N, D, 2) || !pair_shape(M, M, D, 2)) return 0;
  return step_bytes(N, M);
}

B200OT_API int b200ot_softmin_fwd_step(const float* x, const float* y, const b200ot_softmin_slot* slots,
                                       const float* center, int64_t N, int64_t M, int32_t D, int32_t p, float eps,
                                       void* scratch, int64_t scratch_bytes, void* stream) {
  if (!x || !y || !slots || !scratch || N <= 0 || M <= 0 || !valid_p(p) || !(eps > 0.f) ||
      b200ot_softmin_step_scratch_bytes(N, M, D) == 0 || !pair_shape(N, M, D, p))
    return B200OT_EINVAL;
  // xy, yx, xx, yy
  const float* rows[4] = {x, y, x, y};
  const float* cols[4] = {y, x, x, y};
  const int64_t nrows[4] = {N, M, N, M}, ncols[4] = {M, N, N, M};
  PairedSoftmin s[4];
  for (int k = 0; k < 4; ++k) {
    const b200ot_softmin_slot& q = slots[k];
    if (!q.h_a || (!q.out && !q.lse2)) return B200OT_EINVAL;
    s[k] = PairedSoftmin{rows[k], cols[k], nrows[k], ncols[k], q.h_a, q.h_b, q.h_scale_b,
                         {q.out_old, q.alpha_old, q.beta, q.out, q.lse2}};
  }
  if (paired_aliased(s, 4, center)) return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, step_bytes(N, M))) return rc;
  return paired_fwd(s, 4, center, eps, scratch, (cudaStream_t)stream);
}

}  // extern "C"
