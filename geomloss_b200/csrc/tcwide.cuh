// b200ot — the tensor-core reductions above D = 64 (64 < D <= B200OT_MAX_D_WIDE): the operators of tcconv.cuh /
// tcbwd.cuh with the K axis of the exponent GEMM streamed in slabs.
//
// The operand images are those of tc_pack_kernel (fp16 h + l split terms, the bf16 rank-one chunk, the fp32 column
// slot), unchanged.  What changes is what stays in shared memory.  At D = 64 a CTA keeps its whole row image resident
// and streams column tiles; at dk = 256 the row image and one column stage no longer fit in 227 KB.  Here:
//   * the row image's rank-one chunk and the l1 row terms (2 chunks, 4 KB per 128 rows) stay resident: the epilogues
//     read |X|^2 (tc_norm_row_bound) and c / lse2 (tc_l1_row_terms) from it exactly as they read the whole image;
//   * the K axis is streamed in slabs of 64 dimensions (8 chunks of each split term).  A ring stage carries the row
//     slab and the column slab, 2 x 32 KB whatever D;
//   * each column tile's rank-one chunk and fp32 slot (4.5 KB) ride with the tile's LAST slab, in a slot of their own,
//     so that the epilogue finds the weights (or H_j) where the exponent was completed.
// The exponent of a column tile is the sum over its slabs of the hh, hl, lh products plus the rank-one chunk, so the
// epilogues of tc_reduce_kernel (tc_reduce_tile, tc_reduce_store) and of tc_bwd_kernel (tc_bwd_tile, tc_bwd_store)
// apply as they are, with the batch mapping of tc_cta_prologue / tc_out_row.
//
// Row gradients are D-sliced: the grid gains a slice axis (blockIdx.z), one slice per 64-dimension slab.  Each CTA
// recomputes the full-K exponent, and GEMM 2 (P . Y) runs against its own slab of Y only, which the CTA's slab order
// brings last so that it is still in the ring: the same MN-major read of the column image as tcbwd.cuh, with the
// l term 16 KB (8 chunks) behind the h term, so hi.[Y_h | Y_l] is one N = 128 instruction.  Slice 0 also writes the
// row sums (sum P; sum Q for the p = 1 softmin).  The partials have the layout of tc_bwd_kernel,
// (split, row, D + head), so the existing finalize kernels apply.
#pragma once
#include "tcbwd.cuh"

namespace b200ot {

constexpr int kTcWideSlab = 64;                                   // dimensions per K slab (and per gradient slice)
constexpr int kTcWideSlabChunks = kTcWideSlab / 8;                // 8-element chunks of one split term in a slab
constexpr int kTcWideTermBytes = kTcWideSlabChunks * kTcM * 16;   // one split term of a slab, 16 KB (kTcM == kTcBN)
constexpr int kTcWideStageBytes = 4 * kTcWideTermBytes;           // row slab [h | l], column slab [h | l]
constexpr int kTcWideTailBytes = 2 * kTcBN * 16 + kTcBN * 4;      // a column tile's two last chunks + fp32 slot
static_assert(kTcM == kTcBN, "row and column slabs share one chunk stride");

__host__ __device__ inline int tc_wide_slabs(int D) { return (tc_dk(D) + kTcWideSlab - 1) / kTcWideSlab; }
// shared memory: row tail (tc_a_span(16)), NSTAGE column tails, the mbarriers, then the ring of slabs 1024-aligned
__host__ __device__ inline int64_t tc_wide_ring_off(int nstage) {
  return ((tc_a_span(16) + (int64_t)nstage * kTcWideTailBytes + 256 + 1023) / 1024) * 1024;
}
__host__ __device__ inline int64_t tc_wide_smem(int nstage) {
  return tc_wide_ring_off(nstage) + (int64_t)nstage * kTcWideStageBytes;
}

// The coincidence bound T_i of the thread's two rows above D = 64 (tcconv.cuh derives it for D <= 64).  The exponent
// now sums 3 dk/16 + 1 MMAs in fp32 (up to 193 at dk = 1024), each rounding at the scale of |X|^2 + |Y|^2, on top of
// the 2^-21 of the split operands: |computed d^2 - d^2| <= (3 dk/16 + 9) 2^-23 (|X|^2 + |Y|^2) in the worst case, so
// for the near pairs that T_i must catch (|Y_j| ~ |X_i|), (3 dk/16 + 9) 2^-22 |X_i|^2.  T_i takes that coefficient of
// |X_i|^2 when it exceeds tcconv.cuh's 2^-17 (from dk = 128 on; 2^-14.4 at dk = 1024), with the same floor and clamp.
// |X_i|^2 is read back from tc_norm_row_bound with a zero clamp (2^-17 |X_i|^2 + 2^-14, exact to fp32 rounding).
__device__ __forceinline__ void tc_wide_row_bounds(float (&tb)[2], float& clampq, const float* coord_absmax,
                                                   const unsigned char* sa, int dk, int wg, int warp, int lane) {
  tc_norm_row_bounds(tb, clampq, coord_absmax, sa, 16, wg, warp, lane);
  const float rel = fmaxf(kTcNormRel, (float)(3 * dk / 16 + 9) * (1.f / 4194304.f));
  const int lr = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float xx = (tc_norm_row_bound(sa, 16, lr + 8 * h, 0.f) - kTcNormFloor) * (1.f / kTcNormRel);
    tb[h] = fmaxf(tb[h], fmaf(rel, xx, kTcNormFloor));
  }
}

// Slab j of a column tile in the order of slice `own`: own + 1, own + 2, ... (mod nslab), own last.  The forward
// passes own = nslab - 1 (slabs in order).
__device__ __forceinline__ int tc_wide_slab_at(int j, int own, int nslab) {
  int s = own + 1 + j;
  return s >= nslab ? s - nslab : s;
}

// The producer lane: the row tail once, then for every column tile of the CTA its slabs through the ring, the
// column tail with the last one.  VALUES (tc_wide_apply_kernel): the tile's value image of e_bytes (tile ct at
// e_imgs + ct e_bytes) rides with the last slab as well, into slot `st` of a ring of its own at e_ring, its bytes in
// that stage's expect_tx.
template <bool VALUES = false>
__device__ __forceinline__ void tc_wide_produce(const TcCta& c, const unsigned char* __restrict__ a_imgs,
                                                const unsigned char* __restrict__ b_imgs, unsigned char* ring,
                                                int kp, int own, int nslab, int NSTAGE, int lane,
                                                const unsigned char* __restrict__ e_imgs = nullptr,
                                                unsigned char* e_ring = nullptr, int e_bytes = 0) {
  if (lane != 0) return;
  const int seg = tc_dk_of_kp(kp) / 8;
  const unsigned char* arow = a_imgs + (int64_t)c.row_tile * tc_a_img_bytes(kp);
  mbar_arrive_expect_tx(c.bar_a, c.a_bytes);
  tma_load_1d(c.sa, arow + (int64_t)kTcTerms * seg * kTcM * 16, c.a_bytes, c.bar_a);
  const int tail = VALUES ? c.b_bytes + e_bytes : c.b_bytes;  // bytes that ride with a tile's last slab
  int step = 0;
  for (int k = 0; k < c.nt; ++k) {
    const unsigned char* bcol = b_imgs + (int64_t)(c.t0 + k) * tc_b_img_bytes(kp, kTcBN);
    for (int j = 0; j < nslab; ++j, ++step) {
      const int sl = tc_wide_slab_at(j, own, nslab);
      const int bytes = min(kTcWideSlabChunks, seg - kTcWideSlabChunks * sl) * kTcM * 16;
      const bool last = j == nslab - 1;
      const int st = step % NSTAGE;
      if (step >= NSTAGE) mbar_wait(&c.empty_b[st], ((step / NSTAGE) + 1) & 1);
      mbar_arrive_expect_tx(&c.full_b[st], 4 * bytes + (last ? tail : 0));
      unsigned char* dst = ring + (int64_t)st * kTcWideStageBytes;
#pragma unroll
      for (int t = 0; t < kTcTerms; ++t) {
        const int64_t off = (int64_t)(t * seg + kTcWideSlabChunks * sl) * kTcM * 16;
        tma_load_1d(dst + t * kTcWideTermBytes, arow + off, bytes, &c.full_b[st]);
        tma_load_1d(dst + (kTcTerms + t) * kTcWideTermBytes, bcol + off, bytes, &c.full_b[st]);
      }
      if (last) {
        tma_load_1d(c.sb + st * c.b_bytes, bcol + (int64_t)kTcTerms * seg * kTcBN * 16, c.b_bytes, &c.full_b[st]);
        if constexpr (VALUES)
          tma_load_1d(e_ring + (int64_t)st * e_bytes, e_imgs + (int64_t)(c.t0 + k) * e_bytes, e_bytes, &c.full_b[st]);
      }
    }
  }
}

// The exponent S of the warpgroup's 64 rows against column tile k, slab by slab (slice `own` last); returns with
// the ring stage of the last slab still held (its column tail and, for row gradients, its column slab are read
// next).  Every other stage is released as soon as its MMAs are done.
__device__ __forceinline__ int tc_wide_exponent(float (&s)[64], const TcCta& c, unsigned char* ring, int seg, int own,
                                                int nslab, int NSTAGE, int wg, int lane, int& step) {
  constexpr uint32_t kC = kTcM * 16;  // byte distance between 8-element K chunks (rows and columns alike)
  int st = 0;
  for (int j = 0; j < nslab; ++j, ++step) {
    const int sl = tc_wide_slab_at(j, own, nslab);
    const int nc = min(kTcWideSlabChunks, seg - kTcWideSlabChunks * sl);
    st = step % NSTAGE;
    mbar_wait(&c.full_b[st], (step / NSTAGE) & 1);
    const uint32_t ra = smem_u32(ring + (int64_t)st * kTcWideStageBytes) + wg * 64 * 16;
    const uint32_t cb = smem_u32(ring + (int64_t)st * kTcWideStageBytes + kTcTerms * kTcWideTermBytes);
    wgmma_fence();
#pragma unroll
    for (int prod = 0; prod < 3; ++prod) {
      const int ta = (prod == 2) ? 1 : 0, tb = (prod == 1) ? 1 : 0;  // (A term, B term): hh, hl, lh
      for (int kk = 0; kk < nc / 2; ++kk)
        wgmma_ss_n128_f16(s, make_smem_desc(ra + ta * kTcWideTermBytes + 2 * kk * kC, kC, 128),
                          make_smem_desc(cb + tb * kTcWideTermBytes + 2 * kk * kC, kC, 128),
                          j > 0 || prod > 0 || kk > 0);
    }
    if (j == nslab - 1)  // the rank-one chunk: row tail against the tile's column tail
      wgmma_ss_n128_bf16(s, make_smem_desc(smem_u32(c.sa) + wg * 64 * 16, kC, 128),
                         make_smem_desc(smem_u32(c.sb + st * c.b_bytes), kC, 128), true);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    if (j < nslab - 1) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&c.empty_b[st]);
    }
  }
  return st;
}

// Forward: tc_reduce_kernel's MODE (0 gaussian, 1 softmin, 4 laplacian, 5 energy, 6 p = 1 softmin) and partials.
// The kernel arguments are those of tc_reduce_kernel (the launch path is shared); kp is the image's, D > 64.
template <int MODE>
__global__ void __launch_bounds__(kTcThreads, 1)
    tc_wide_reduce_kernel(const unsigned char* __restrict__ a_imgs, const unsigned char* __restrict__ b_imgs,
                          float* __restrict__ part, int64_t N, int kp, int ntiles_b, int tiles_per_split, int NSTAGE,
                          int D, int self_mode, float clampq, const float* __restrict__ coord_absmax, int rtpe,
                          int64_t n_local, const int4* __restrict__, const int2* __restrict__,
                          const int* __restrict__) {
  static_assert(MODE == 0 || MODE == 1 || MODE == 4 || MODE == 5 || MODE == 6, "forward modes of tc_reduce_kernel");
  extern __shared__ __align__(1024) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // the prologue of tc_reduce_kernel with a 16-wide "image": the row tail in sa, one column tail per stage in sb
  const TcCta c = tc_cta_prologue<true, false>(smem, 16, NSTAGE, ntiles_b, tiles_per_split, rtpe, nullptr, nullptr);
  unsigned char* ring = smem + tc_wide_ring_off(NSTAGE);
  const int nslab = tc_wide_slabs(D);
  if (warp == 4 * kTcWG) {
    tc_wide_produce(c, a_imgs, b_imgs, ring, kp, nslab - 1, nslab, NSTAGE, lane);
    return;
  }
  const int wg = warp >> 2;
  const int seg = tc_dk_of_kp(kp) / 8;
  const int64_t row0 = (int64_t)c.row_tile * kTcM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  float acc[2] = {0.f, 0.f};
  float m[2] = {kNegBig, kNegBig}, srun[2] = {0.f, 0.f};
  mbar_wait(c.bar_a, 0);
  float tb[2] = {0.f, 0.f};
  if constexpr (MODE >= 4) tc_wide_row_bounds(tb, clampq, coord_absmax, c.sa, tc_dk(D), wg, warp, lane);
  float2 rt[2] = {};
  if constexpr (MODE == 6) tc_l1_rows(rt, c.sa, 16, wg, warp, lane);
  int step = 0;
  for (int k = 0; k < c.nt; ++k) {
    float s[64];
    const int st = tc_wide_exponent(s, c, ring, seg, nslab - 1, nslab, NSTAGE, wg, lane, step);
    tc_reduce_tile<MODE>(s, c, st, 16, k, row0, tb, rt, clampq, self_mode, cq, acc, m, srun);
    __syncwarp();
    if (lane == 0) mbar_arrive(&c.empty_b[st]);
  }
  tc_reduce_store<MODE, true, false>(part, acc, m, srun, row0, c.split, c.elem, rtpe, n_local, nullptr, N, lane);
}

// Row gradient: tc_bwd_kernel's MODE (2 gaussian, 3 softmin, 4 laplacian, 5 energy, 7 p = 1 softmin) with P fed to
// GEMM 2 as two fp16 terms, for the slab of dimensions blockIdx.z (see above).
template <int MODE>
__global__ void __launch_bounds__(kTcThreads, 1)
    tc_wide_bwd_kernel(const unsigned char* __restrict__ a_imgs, const unsigned char* __restrict__ b_imgs,
                       float* __restrict__ part, int64_t N, int kp, int ntiles_b, int tiles_per_split, int NSTAGE,
                       int D, int self_mode, float clampq, const float* __restrict__ coord_absmax, int rtpe,
                       int64_t n_local, const int4* __restrict__, const int2* __restrict__, const int* __restrict__) {
  static_assert(MODE == 2 || MODE == 3 || MODE == 4 || MODE == 5 || MODE == 7, "row-gradient modes of tc_bwd_kernel");
  extern __shared__ __align__(1024) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TcCta c = tc_cta_prologue<true, false>(smem, 16, NSTAGE, ntiles_b, tiles_per_split, rtpe, nullptr, nullptr);
  unsigned char* ring = smem + tc_wide_ring_off(NSTAGE);
  const int nslab = tc_wide_slabs(D);
  const int own = blockIdx.z;
  if (warp == 4 * kTcWG) {
    tc_wide_produce(c, a_imgs, b_imgs, ring, kp, own, nslab, NSTAGE, lane);
    return;
  }
  const int wg = warp >> 2;
  const int seg = tc_dk_of_kp(kp) / 8;
  const int64_t row0 = (int64_t)c.row_tile * kTcM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  float g[kTcWideSlab];  // [G_a | G_b] of the slice's 64 dimensions, as tc_bwd_kernel's g at DK = 64
#pragma unroll
  for (int i = 0; i < kTcWideSlab; ++i) g[i] = 0.f;
  float sum[2] = {0.f, 0.f}, sumq[2] = {0.f, 0.f};
  mbar_wait(c.bar_a, 0);
  float tb[2] = {0.f, 0.f};
  if constexpr (MODE >= 4) tc_wide_row_bounds(tb, clampq, coord_absmax, c.sa, tc_dk(D), wg, warp, lane);
  float2 rt[2] = {};
  if constexpr (MODE == 7) {
    tc_l1_rows(rt, c.sa, 16, wg, warp, lane);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int e = ((__float_as_int(tb[h]) >> 23) & 0xff) - 127;  // as tc_bwd_kernel
      rt[h].y = (float)(kTcL1QLog2 + (e >> 1)) - rt[h].y;
    }
  }
  int step = 0;
  for (int k = 0; k < c.nt; ++k) {
    float s[64];
    const int st = tc_wide_exponent(s, c, ring, seg, own, nslab, NSTAGE, wg, lane, step);
    uint32_t ph[32], pl[32];
    tc_bwd_tile<MODE>(s, c, st, 16, k, row0, tb, rt, clampq, self_mode, cq, ph, pl, sum, sumq);
    // GEMM 2 against the slice's column slab (the last one loaded): K = the tile's 128 columns, 16 per instruction.
    // In a partial last slab the columns of G past the slab's chunks read stale shared memory; they lie at or above
    // tc_dk(D) and are never written out.
    const uint32_t cb = smem_u32(ring + (int64_t)st * kTcWideStageBytes + kTcTerms * kTcWideTermBytes);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kTcBN / 16; ++kk) {
      const uint64_t db = make_smem_desc(cb + (2 * kk) * 128, 128, kTcBN * 16);
      wgmma_rs<2 * kTcWideSlab>(g, &ph[4 * kk], db);
      wgmma_rs<kTcWideSlab>(g, &pl[4 * kk], db);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(g);
    __syncwarp();
    if (lane == 0) mbar_arrive(&c.empty_b[st]);
  }
  tc_bwd_store<MODE, kTcWideSlab, true, false>(part, g, sum, sumq, row0, c.split, c.elem, rtpe, n_local, nullptr, N, D,
                                               own * kTcWideSlab, own == 0, cq);
}

}  // namespace b200ot
