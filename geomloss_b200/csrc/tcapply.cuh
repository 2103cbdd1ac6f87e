// b200ot — the transport plan applied to a value matrix on the tensor cores (8 < D <= 64): the two-GEMM scheme of
// tcbwd.cuh's softmin row gradient (MODE 3) with GEMM 2's B operand taken from a VALUE image instead of the column
// image.
//
//   S_ij = the softmin exponent - lse2_i + 14                      GEMM 1, tc_exponent_gemm, as tc_bwd_kernel<3>
//   P_ij = 2^S_ij = hi + lo (two fp16 terms, in registers)         tc_bwd_tile<3>
//   G_ik = sum_j P_ij s_k V_jk                                     GEMM 2: A = P, B = the value image of the tile
//   part[(split N + i)(1 + KV) + {0, 1 + k}] = {sum_j P_ij, G_ik}  tc_bwd_store
//
// Value image of a 128-column tile (tc_pack_values_kernel): [V_h | V_l], the fp16 two-term split of s_k V_jk for the
// slab's DKV value columns, stored [8-column group of V][tile column][8 halves] — read with k = tile column this is
// the canonical MN-major no-swizzle layout GEMM 2's descriptor already reads from the column image (LBO = 128 B,
// SBO = 128 x 16 B), V_l 128 DKV / 8 x 16 B behind V_h, so hi.[V_h | V_l] is one N = 2 DKV instruction and lo.V_h one
// N = DKV instruction per 16 columns.  512 DKV bytes per tile (32 KB at DKV = 64); it travels in a ring slot of its
// own next to its column tile, its bytes in the stage's expect_tx (tc_produce<.., EXTRA>).
//
// s_k is the power of two that puts max_j |V_jk| in [2^9, 2^10) (tc_energy_coord_scale, found on the device by
// col_absmax_kernel): both fp16 terms of an entry down to 2^-13 of its column's largest stay in fp16's normal
// range, whatever the unit of the column; the finalize divides by s_k exactly.
//
// Above D = 64 (tc_wide_apply_kernel): the same GEMM 2 and epilogue behind the K-slab exponent of tcwide.cuh.
#pragma once
#include "tcbwd.cuh"
#include "tcwide.cuh"

namespace b200ot {

__host__ __device__ inline int64_t tc_value_img_bytes(int dkv) { return (int64_t)kTcTerms * dkv * kTcBN * 2; }

// max_j |v[j, k]| of every column k of v (M, K) into out[k] (zero-initialised by the caller)
static __global__ void col_absmax_kernel(const float* __restrict__ v, int64_t M, int K, float* __restrict__ out) {
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float m = 0.f;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.y + threadIdx.y; j < M; j += (int64_t)gridDim.x * blockDim.y)
      m = fmaxf(m, fabsf(v[j * K + k]));
    if (m > 0.f && !(m != m)) atomicMax(reinterpret_cast<unsigned int*>(out + k), __float_as_uint(m));
  }
}

// one thread per (padded) column: its 16-byte piece of every 8-column group of both terms of the slab [k0, k0 + dkv)
static __global__ void tc_pack_values_kernel(const float* __restrict__ v, const float* __restrict__ vmax, int64_t M,
                                             int K, int k0, int dkv, int64_t ncols, unsigned char* __restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= ncols) return;
  unsigned char* img = out + (p / kTcBN) * tc_value_img_bytes(dkv);
  const int pt = (int)(p % kTcBN);
  for (int kc = 0; kc < dkv / 8; ++kc) {
    __half term[kTcTerms][8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = k0 + kc * 8 + e;
      const float val = (p < M && k < K) ? v[p * K + k] * tc_energy_coord_scale(vmax[k]) : 0.f;
      const __half h = __float2half_rn(val);
      term[0][e] = h;
      term[1][e] = __float2half_rn(val - __half2float(h));
    }
#pragma unroll
    for (int s = 0; s < kTcTerms; ++s)
      *reinterpret_cast<uint4*>(img + ((int64_t)(s * (dkv / 8) + kc) * kTcBN + pt) * 16) = pack8_f16(term[s]);
  }
}

// DKV = the padded width of the value slab (N of GEMM 2), KV <= DKV its live columns.  One problem, dense layout.
template <int DKV>
__global__ void __launch_bounds__(kTcThreads, 1)
    tc_apply_kernel(const unsigned char* __restrict__ a_imgs, const unsigned char* __restrict__ b_imgs,
                    const unsigned char* __restrict__ v_imgs, float* __restrict__ part, int64_t N, int kp,
                    int ntiles_b, int tiles_per_split, int NSTAGE, int KV) {
  static_assert(DKV % 16 == 0 && DKV <= 64, "padded slab width");
  extern __shared__ __align__(1024) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TcCta c = tc_cta_prologue<false, false>(smem, kp, NSTAGE, ntiles_b, tiles_per_split, 0, nullptr, nullptr);
  constexpr int v_bytes = kTcTerms * DKV * kTcBN * 2;
  unsigned char* sv = c.sb + NSTAGE * c.b_bytes + 256;  // the value ring, behind the mbarriers
  if (warp == 4 * kTcWG) {
    tc_produce<false, true>(c, a_imgs, b_imgs, nullptr, NSTAGE, lane, v_imgs, sv, v_bytes);
    return;
  }
  const int wg = warp >> 2;
  const int seg = tc_dk_of_kp(kp) / 8;
  const uint32_t a_addr = smem_u32(c.sa) + wg * 64 * 16;
  const int64_t row0 = (int64_t)c.row_tile * kTcM + wg * 64 + (warp & 3) * 16 + (lane >> 2);  // and row0 + 8
  const int cq = 2 * (lane & 3);
  float g[DKV];  // [G_a | G_b], as tc_bwd_kernel
#pragma unroll
  for (int i = 0; i < DKV; ++i) g[i] = 0.f;
  float sum[2] = {0.f, 0.f}, sumq[2] = {0.f, 0.f};
  const float tb[2] = {0.f, 0.f};
  const float2 rt[2] = {};
  mbar_wait(c.bar_a, 0);
  for (int k = 0; k < c.nt; ++k) {
    const int st = k % NSTAGE;
    mbar_wait(&c.full_b[st], (k / NSTAGE) & 1);
    float s[64];
    tc_exponent_gemm(s, a_addr, smem_u32(c.sb + st * c.b_bytes), seg);
    wgmma_wait<0>();
    reg_fence(s);
    uint32_t ph[32], pl[32];
    tc_bwd_tile<3>(s, c, st, kp, k, row0, tb, rt, 0.f, 0, cq, ph, pl, sum, sumq);
    // ---- GEMM 2: G += P . V, K = the 128 columns of the tile, 16 per instruction ----
    const uint32_t v_addr = smem_u32(sv + st * v_bytes);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kTcBN / 16; ++kk) {
      const uint64_t db = make_smem_desc(v_addr + (2 * kk) * 128, 128, kTcBN * 16);
      wgmma_rs<2 * DKV>(g, &ph[4 * kk], db);
      wgmma_rs<DKV>(g, &pl[4 * kk], db);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(g);
    __syncwarp();
    if (lane == 0) mbar_arrive(&c.empty_b[st]);  // column tile and value image may be overwritten
  }
  tc_bwd_store<3, DKV, false, false>(part, g, sum, sumq, row0, c.split, 0, 0, 0, nullptr, N, KV, 0, true, cq);
}

// tc_apply_kernel above D = 64 (64 < D <= B200OT_MAX_D_WIDE), with its arguments (kp is the image's): the exponent of
// tc_wide_reduce_kernel (row tail resident, slabs streamed in natural order through the ring, lse2 in the row tail as
// for tc_wide_bwd_kernel<3>), then tc_bwd_tile<3> and GEMM 2 against the value image.  Unlike the D-sliced row
// gradient, GEMM 2 reads no column slab, so one CTA per row tile and split serves every value column of the slab.
// The tile's value image rides with its last slab (tc_wide_produce<true>): one value slot per ring stage, behind the
// ring, released with that stage once GEMM 2 has read it.
template <int DKV>
__global__ void __launch_bounds__(kTcThreads, 1)
    tc_wide_apply_kernel(const unsigned char* __restrict__ a_imgs, const unsigned char* __restrict__ b_imgs,
                         const unsigned char* __restrict__ v_imgs, float* __restrict__ part, int64_t N, int kp,
                         int ntiles_b, int tiles_per_split, int NSTAGE, int KV) {
  static_assert(DKV % 16 == 0 && DKV <= 64, "padded slab width");
  extern __shared__ __align__(1024) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // the prologue with a 16-wide "image": the row tail in sa, one column tail per stage in sb (as tcwide.cuh)
  const TcCta c = tc_cta_prologue<false, false>(smem, 16, NSTAGE, ntiles_b, tiles_per_split, 0, nullptr, nullptr);
  unsigned char* ring = smem + tc_wide_ring_off(NSTAGE);
  constexpr int v_bytes = kTcTerms * DKV * kTcBN * 2;
  unsigned char* sv = ring + (int64_t)NSTAGE * kTcWideStageBytes;  // the value slots
  const int seg = tc_dk_of_kp(kp) / 8;
  const int nslab = (seg + kTcWideSlabChunks - 1) / kTcWideSlabChunks;
  if (warp == 4 * kTcWG) {
    tc_wide_produce<true>(c, a_imgs, b_imgs, ring, kp, nslab - 1, nslab, NSTAGE, lane, v_imgs, sv, v_bytes);
    return;
  }
  const int wg = warp >> 2;
  const int64_t row0 = (int64_t)c.row_tile * kTcM + wg * 64 + (warp & 3) * 16 + (lane >> 2);  // and row0 + 8
  const int cq = 2 * (lane & 3);
  float g[DKV];  // [G_a | G_b], as tc_apply_kernel
#pragma unroll
  for (int i = 0; i < DKV; ++i) g[i] = 0.f;
  float sum[2] = {0.f, 0.f}, sumq[2] = {0.f, 0.f};
  const float tb[2] = {0.f, 0.f};
  const float2 rt[2] = {};
  mbar_wait(c.bar_a, 0);
  int step = 0;
  for (int k = 0; k < c.nt; ++k) {
    float s[64];
    const int st = tc_wide_exponent(s, c, ring, seg, nslab - 1, nslab, NSTAGE, wg, lane, step);
    uint32_t ph[32], pl[32];
    tc_bwd_tile<3>(s, c, st, 16, k, row0, tb, rt, 0.f, 0, cq, ph, pl, sum, sumq);
    // ---- GEMM 2: G += P . V from the value slot of the last slab's stage ----
    const uint32_t v_addr = smem_u32(sv + st * v_bytes);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kTcBN / 16; ++kk) {
      const uint64_t db = make_smem_desc(v_addr + (2 * kk) * 128, 128, kTcBN * 16);
      wgmma_rs<2 * DKV>(g, &ph[4 * kk], db);
      wgmma_rs<DKV>(g, &pl[4 * kk], db);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(g);
    __syncwarp();
    if (lane == 0) mbar_arrive(&c.empty_b[st]);  // slab, column tail and value image may be overwritten
  }
  tc_bwd_store<3, DKV, false, false>(part, g, sum, sumq, row0, c.split, 0, 0, 0, nullptr, N, KV, 0, true, cq);
}

}  // namespace b200ot
