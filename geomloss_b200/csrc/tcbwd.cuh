// b200ot — row gradients on the tensor cores: TWO chained GEMMs per column tile, FlashAttention style, both on
// wgmma with every intermediate in registers.
//
//   S_ij = X_i.Y_j - |X_i|^2/2 - |Y_j|^2/2 (+ H_j - lse2_i)          GEMM 1 (as in tcconv.cuh: fp16x2 split
//                                                                    operands, three cross products, rank-one chunk)
//   P_ij = 2^S_ij (* w_j)                                            MUFU.EX2 on the accumulator registers
//   G_ik = sum_j P_ij Y_jk                                           GEMM 2: A = P (registers), B = the SAME column
//                                                                    image read MN-major (K = column index)
//
// Reference semantics: the autograd of gaussian_kernel's matvec (src/geomloss/_legacy/kernel_samples.py:62-68,
// :116-137) and of the softmin (sinkhorn_samples.py:32-71) w.r.t. the row cloud:
//   gaussian:  d/dx_i = go_i * sum_j k_ij w_j (y_j - x_i) / blur^2 ;  softmin: d/dx_i = go_i * (x_i - sum_j p_ij y_j)
// i.e. per row the D+1 sums {sum_j P_ij, sum_j P_ij Y_jk}; the finalize kernels turn them into gradients.
//
// * The accumulator of GEMM 1 (64 x 128 per warpgroup) has, two 8-column blocks at a time, the shape of the f16 A
//   fragment of a k16 MMA step: P is packed to fp16 in the registers it was computed in and fed to GEMM 2 directly.
// * P = hi + lo (2 fp16 terms), Y = h + l (the image's two terms): G = hi.h + hi.l + lo.h, error ~2^-22 |P||Y|.
//   P is the weight times kTcPScale = 2^14 (common.cuh): softmax weights with +14 folded into the exponent through
//   the row image's rank-one chunk (r = -|X|^2/2 - lse2 + 14), or kernel values times weights normalised to
//   max|w| = 2^14 by the pack kernel; so P <= 2^14 (< 65504 while the true weight is < 4), and a weight stays in
//   fp16's normal range down to 2^-28 instead of 2^-14.  Unscaled, the ~1/M weights of a softmax over M >~ 16k
//   columns would sit on the fixed 6e-8 subnormal grid: a bias, not noise, when points repeat.  The finalize kernels
//   undo the scale (softmin: it cancels in sum P Y / sum P).
// * The column image of tcconv.cuh ([kgroup][column][8 halves], K-major for GEMM 1) is, read with k = column,
//   exactly the canonical MN-major no-swizzle layout (core matrix = 8 columns x 16 B of one 8-dim group), so
//   GEMM 2 needs no second copy of Y: only a descriptor read MN-major, LBO = 128 B (next 8 columns),
//   SBO = BN*16 B (next 8 dims).  The l term of Y follows its h term in the image, so hi.[Y_h | Y_l] is ONE
//   instruction with N = 2 dk per K step, accumulating [G_a | G_b] (added at the end); lo.Y_h is an N = dk
//   instruction into G_a alone.
#pragma once
#include "tcconv.cuh"

namespace b200ot {

// (lo, hi) fp32 -> packed f16x2, round to nearest even; element `lo` in bits 0..15
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t v) {
  return __half22float2(*reinterpret_cast<const __half2*>(&v));
}

template <int N>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t* a, uint64_t db) {
  static_assert(N == 16 || N == 32 || N == 48 || N == 64 || N == 96 || N == 128, "no wrapper for this N");
  if constexpr (N == 16) wgmma_rs_n16(d, a, db);
  if constexpr (N == 32) wgmma_rs_n32(d, a, db);
  if constexpr (N == 48) wgmma_rs_n48(d, a, db);
  if constexpr (N == 64) wgmma_rs_n64(d, a, db);
  if constexpr (N == 96) wgmma_rs_n96(d, a, db);
  if constexpr (N == 128) wgmma_rs_n128(d, a, db);
}

// MODE 2: gaussian row gradient (P = w_j 2^S, w scaled to max|w| = 2^14), MODE 3: softmin row gradient
// (P = 2^(S - lse2_i + 14): lse2 - 14 rides in the row operand's rank-one chunk).
// MODE 4 / 5: laplacian / energy row gradient, P = w_j 2^-kTcNormPLog2 k'(d) / d with k' = 2^-d (laplacian) or 1
// (energy), and P = 0 for a pair below its row's coincidence bound (tcconv.cuh; `clampq` and `coord_absmax` are read
// by these modes only).  The gradient is then coef (sum_j P_ij Y_j - X_i sum_j P_ij): the finalize of the gaussian.
// part[(split*N + row)*(D+1) + {0, 1+k}] = sum_j P_ij {1, Y_jk}
// DK = the padded dimension tc_dk(D) (N of GEMM 2 is a compile-time constant).
//
// self_mode: rows and columns are the same cloud (the K_xx term): the exponent of pair (i, i) is exactly 0, as in
// tc_reduce_kernel — matters when sum_j P_ij is used as the forward VALUE (b200ot_kernel_conv_fwd_bwd_x).
// MODE 7: p = 1 softmin row gradient (tcconv.cuh, kTcL1QLog2): P = 2^(H_j - c d_ij - lse2_i + k_i), Q = P / d_ij (0 below
// the row's coincidence bound); GEMM 2 takes Q.  part[(split*N + row)*(D+2) + {0, 1, 2+k}] = {sum P, sum Q, sum Q Y_k}
// (the coincident pairs weigh in sum P only), finalized as (X_i sum Q - sum Q Y) / sum P.
// MODE 4 / 5: P of one pair from its exponent s (the rsqrt of a pair below the bound t is discarded by the select)
template <int MODE>
__device__ __forceinline__ float tc_norm_p(float s, float t, float w) {
  const float q = -2.f * s;
  const float r = rsqrt_approx(q);
  float p = w * r;
  if constexpr (MODE == 4) p *= ex2_approx(-(q * r));
  return q < t ? 0.f : p;
}

// MODE 7: (P, Q) of one pair from its exponent s, the column's H and the row's rt = (c, k_i - lse2_i)
__device__ __forceinline__ float2 tc_l1_pq(float s, float t, float clampq, float H, float2 rt) {
  const float q = -2.f * s;
  const float d2 = q < t ? clampq : q;
  const float r = rsqrt_approx(d2);
  const float p = ex2_approx(fmaf(-rt.x, d2 * r, H) + rt.y);
  return make_float2(p, q < t ? 0.f : p * r);
}

// S -> P of one column tile, packed as the A fragments of GEMM 2 (ph[2 n8 + h] = the pair of row h in 8-column block
// n8; pl the lo terms), and the tile's contribution to the row sums (sum: P, sumq: Q for MODE 7).  The column slot,
// tile and rows as for tc_reduce_tile (tcconv.cuh).
template <int MODE>
__device__ __forceinline__ void tc_bwd_tile(float (&s)[64], const TcCta& c, int st, int kp, int k, int64_t row0,
                                            const float (&tb)[2], const float2 (&rt)[2], float clampq, int self_mode,
                                            int cq, uint32_t (&ph)[32], uint32_t (&pl)[32], float (&sum)[2],
                                            float (&sumq)[2]) {
  if constexpr (MODE != 3) {
    if (self_mode) tc_zero_diagonal(s, row0 - (int64_t)(c.t0 + k) * kTcBN, cq);
  }
  float tq[2] = {0.f, 0.f};
  const float* wts = reinterpret_cast<const float*>(c.sb + st * c.b_bytes + kTcBN * kp * 2);
  float ts[2] = {0.f, 0.f};
#pragma unroll
  for (int n8 = 0; n8 < kTcBN / 8; ++n8) {
    float2 w = make_float2(1.f, 1.f);
    if constexpr (MODE != 3) w = *reinterpret_cast<const float2*>(wts + 8 * n8 + cq);
    if constexpr (MODE == 4 || MODE == 5) {
      w.x *= 1.f / (float)(1 << kTcNormPLog2);
      w.y *= 1.f / (float)(1 << kTcNormPLog2);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float p0, p1;
      if constexpr (MODE == 7) {
        // w = (H_j, H_j+1); ts sums P, tq and GEMM 2 take Q
        const float2 pq0 = tc_l1_pq(s[4 * n8 + 2 * h], tb[h], clampq, w.x, rt[h]);
        const float2 pq1 = tc_l1_pq(s[4 * n8 + 2 * h + 1], tb[h], clampq, w.y, rt[h]);
        ts[h] += pq0.x + pq1.x;
        p0 = pq0.y;
        p1 = pq1.y;
      } else if constexpr (MODE >= 4) {
        p0 = tc_norm_p<MODE>(s[4 * n8 + 2 * h], tb[h], w.x);
        p1 = tc_norm_p<MODE>(s[4 * n8 + 2 * h + 1], tb[h], w.y);
      } else {
        p0 = ex2_approx(s[4 * n8 + 2 * h]);
        p1 = ex2_approx(s[4 * n8 + 2 * h + 1]);
      }
      if constexpr (MODE == 2) {
        p0 *= w.x;
        p1 *= w.y;
      }
      const uint32_t hh = pack_f16x2(p0, p1);
      ph[2 * n8 + h] = hh;
      const float2 hf = unpack_f16x2(hh);
      if constexpr (MODE == 7) {
        tq[h] += p0 + p1;
      } else {
        ts[h] += p0 + p1;
      }
      pl[2 * n8 + h] = pack_f16x2(p0 - hf.x, p1 - hf.y);
    }
  }
  sum[0] += ts[0];
  sum[1] += ts[1];
  if constexpr (MODE == 7) {
    sumq[0] += tq[0];
    sumq[1] += tq[1];
  }
}

// Row sums over the quad and gradient sums out: the thread's two rows of [G_a | G_b] (g, DK columns each) are the
// gradient sums of dimensions d0 .. d0 + DK - 1 (those below D are written); `heads`: also the row sums ahead of them.
template <int MODE, int DK, bool BATCH, bool BLOCKS>
__device__ __forceinline__ void tc_bwd_store(float* __restrict__ part, const float (&g)[DK], const float (&sum)[2],
                                             const float (&sumq)[2], int64_t row0, int split, int elem, int rtpe,
                                             int64_t n_local, const int* __restrict__ row_src, int64_t N, int D,
                                             int d0, bool heads, int cq) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float tot = sum[h];
    tot += __shfl_xor_sync(0xffffffffu, tot, 1);
    tot += __shfl_xor_sync(0xffffffffu, tot, 2);
    float totq = 0.f;
    if constexpr (MODE == 7) {
      totq = sumq[h];
      totq += __shfl_xor_sync(0xffffffffu, totq, 1);
      totq += __shfl_xor_sync(0xffffffffu, totq, 2);
    }
    constexpr int kHead = MODE == 7 ? 2 : 1;  // row sums ahead of the D gradient sums
    const int64_t row = tc_out_row<BATCH, BLOCKS>(row0 + 8 * h, elem, rtpe, n_local, row_src, N);
    if (row < N) {
      float* dst = part + ((int64_t)split * N + row) * (D + kHead);
      if (cq == 0 && heads) dst[0] = tot;
      if constexpr (MODE == 7) {
        if (cq == 0 && heads) dst[1] = totq;
      }
#pragma unroll
      for (int j = 0; j < DK / 2; ++j) {
        if (((j >> 1) & 1) != h) continue;
        const int c = d0 + 8 * (j >> 2) + cq + (j & 1);
        if (c < D) dst[kHead + c] = g[j] + g[j + DK / 2];
      }
    }
  }
}

// BATCH: B problems side by side, laid out and mapped to rows and column tiles as in tc_reduce_kernel (tcconv.cuh).
// BLOCKS: block-sparse softmin (MODE 3), segments, pieces and row_src as in tc_reduce_kernel; a split without a tile
// writes zero sums.
template <int MODE, int DK, bool BATCH = false, bool BLOCKS = false>
__global__ void __launch_bounds__(kTcThreads, 1)
    tc_bwd_kernel(const unsigned char* __restrict__ a_imgs, const unsigned char* __restrict__ b_imgs,
                  float* __restrict__ part, int64_t N, int kp, int ntiles_b, int tiles_per_split, int NSTAGE, int D,
                  int self_mode, float clampq, const float* __restrict__ coord_absmax, int rtpe, int64_t n_local,
                  const int4* __restrict__ bseg = nullptr, const int2* __restrict__ bpieces = nullptr,
                  const int* __restrict__ row_src = nullptr) {
  static_assert(MODE == 2 || MODE == 3 || MODE == 4 || MODE == 5 || MODE == 7, "row-gradient modes");
  static_assert(DK % 16 == 0 && DK <= 64, "padded dimension");
  static_assert(!BLOCKS || (MODE == 3 && !BATCH), "the block-sparse layout serves the softmin of one problem");
  extern __shared__ __align__(1024) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TcCta c = tc_cta_prologue<BATCH, BLOCKS>(smem, kp, NSTAGE, ntiles_b, tiles_per_split, rtpe, bseg, bpieces);
  if (warp == 4 * kTcWG) {
    tc_produce<BLOCKS>(c, a_imgs, b_imgs, bpieces, NSTAGE, lane);
    return;
  }
  // ===== consumer warpgroups =====
  const int wg = warp >> 2;
  const uint32_t a_addr = smem_u32(c.sa) + wg * 64 * 16;
  const int64_t row0 = (int64_t)c.row_tile * kTcM + wg * 64 + (warp & 3) * 16 + (lane >> 2);  // and row0 + 8
  const int cq = 2 * (lane & 3);
  float g[DK];  // [G_a | G_b]: columns 0..DK-1 in g[0 .. DK/2), DK..2DK-1 in g[DK/2 .. DK)
#pragma unroll
  for (int i = 0; i < DK; ++i) g[i] = 0.f;
  float sum[2] = {0.f, 0.f};
  float sumq[2] = {0.f, 0.f};  // MODE 7: sum_j Q_ij (sum holds sum_j P_ij)
  mbar_wait(c.bar_a, 0);
  float tb[2] = {0.f, 0.f};  // MODE 4 / 5 / 7: coincidence bound of each row
  if constexpr (MODE >= 4) tc_norm_row_bounds(tb, clampq, coord_absmax, c.sa, kp, wg, warp, lane);
  float2 rt[2] = {};  // MODE 7: (c, k_i - lse2_i) of each row
  if constexpr (MODE == 7) {
    tc_l1_rows(rt, c.sa, kp, wg, warp, lane);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int e = ((__float_as_int(tb[h]) >> 23) & 0xff) - 127;  // 2^e <= T_i < 2^(e+1): T_i is normal
      rt[h].y = (float)(kTcL1QLog2 + (e >> 1)) - rt[h].y;
    }
  }
  for (int k = 0; k < c.nt; ++k) {
    const int st = k % NSTAGE;
    mbar_wait(&c.full_b[st], (k / NSTAGE) & 1);
    const uint32_t b_addr = smem_u32(c.sb + st * c.b_bytes);
    // ---- GEMM 1: S ----
    float s[64];
    tc_exponent_gemm(s, a_addr, b_addr, DK / 8);
    wgmma_wait<0>();
    reg_fence(s);
    uint32_t ph[32], pl[32];
    tc_bwd_tile<MODE>(s, c, st, kp, k, row0, tb, rt, clampq, self_mode, cq, ph, pl, sum, sumq);
    // ---- GEMM 2: G += P . Y, K = the 128 columns of the tile, 16 per instruction ----
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kTcBN / 16; ++kk) {
      const uint64_t db = make_smem_desc(b_addr + (2 * kk) * 128, 128, kTcBN * 16);
      wgmma_rs<2 * DK>(g, &ph[4 * kk], db);
      wgmma_rs<DK>(g, &pl[4 * kk], db);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(g);
    __syncwarp();
    if (lane == 0) mbar_arrive(&c.empty_b[st]);  // the column tile may be overwritten
  }
  tc_bwd_store<MODE, DK, BATCH, BLOCKS>(part, g, sum, sumq, row0, c.split, c.elem, rtpe, n_local, row_src, N, D, 0,
                                        true, cq);
}

}  // namespace b200ot
