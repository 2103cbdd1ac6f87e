// b200ot — gaussian kernel convolution on the Hopper tensor cores (wgmma), for dimensions where -2 x.y^T is a
// real dense contraction (and, routed by tc_routed, a few below):
//     out_i = sum_j w_j exp(-|x_i - y_j|^2 / (2 blur^2)) = sum_j w_j 2^( X_i.Y_j - |X_i|^2/2 - |Y_j|^2/2 )
// Reference semantics: gaussian_kernel + the matvecs of kernel_loss
// (src/geomloss/_legacy/kernel_samples.py:62-68, :116-137).
//
// The whole exponent is produced by wgmma into registers:
//   * each operand is split into TWO fp16 terms X = h + l (22 significant bits) and stored ONCE as [h | l] along
//     K; the three cross products that matter (hh, hl, lh: error ~2^-22 |X||Y|) are formed by pointing the A and B
//     descriptors at the matching segments — no duplicated data in shared memory or L2, 3*Dk/16 MMA instructions
//     per tile, fp32 accumulation.  fp16's narrow range is harmless for centred, scaled coordinates.
//   * one extra 16-wide K chunk, issued as a BF16 instruction (fp32 range: potentials / eps reach 1e5), carries
//     the rank-one terms:  A: [1,1,1, r_h,r_m,r_l, 0..],  B: [c_h,c_m,c_l, 1,1,1, 0..] with r = -|X|^2/2,
//     c = -|Y|^2/2 split in three bf16 terms,
//   so the epilogue is  MUFU.EX2 -> FFMA with the column weight  on the accumulator registers and nothing else.
//
// Operand tiles are pre-packed in global memory by tc_pack_kernel in the exact image the wgmma descriptors
// expect (K-major, no swizzle: for every 8-element K chunk the 16-byte pieces of all rows are contiguous), so a
// row or column tile is ONE 1-D bulk-TMA copy; the column weights ride at the end of the column image.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc.cuh"

namespace b200ot {

constexpr int kTcM = 128;  // rows per CTA tile = M of the MMA

__host__ __device__ inline int tc_dk(int D) { return ((D + 15) / 16) * 16; }
constexpr int kTcTerms = 2;  // fp16 split terms per coordinate
// K extent of an operand image: the split terms + one 16-wide chunk of rank-one terms
__host__ __device__ inline int tc_kp(int D) { return kTcTerms * tc_dk(D) + 16; }
__host__ __device__ inline int tc_dk_of_kp(int kp) { return (kp - 16) / kTcTerms; }
__host__ __device__ inline int64_t tc_a_img_bytes(int kp) { return (int64_t)kTcM * kp * 2; }
// shared memory taken by the row image, rounded so that the column ring behind it starts 1024-byte aligned
__host__ __device__ inline int64_t tc_a_span(int kp) { return ((tc_a_img_bytes(kp) + 1023) / 1024) * 1024; }
// column image: bf16 operand data | fp32 weights
__host__ __device__ inline int64_t tc_b_img_bytes(int kp, int bn) { return (int64_t)bn * kp * 2 + (int64_t)bn * 4; }

// ---------------------------------------------------------------------------------------------------
// laplacian / energy kernels (MODE 4 / 5 of tc_reduce_kernel and tc_bwd_kernel): the same exponent GEMM gives
// S = -|X - Y|^2 / 2, so d^2 = -2 S, d = d^2 rsqrt(d^2) and k = 2^-d (laplacian, X = x log2e / blur) or k = d (energy).
//
// Resolution.  The split operands carry 22 bits (|X_k - h_k - l_k| <= 2^-22 |X_k|, the l.l product is dropped), the
// rank-one terms 24, and the fp32 accumulation of 3 dk/16 + 1 <= 13 MMAs rounds at the scale of |X|^2 + |Y|^2.
// Summed, |computed d^2 - d^2| <= 2^-18 (|X|^2 + |Y|^2) in the worst case (random signs make it ~2^-21).  A pair
// whose d^2 is below that bound cannot be told from a coincident one; since |Y_j| ~ |X_i| for exactly those pairs,
// the kernels test d^2 against the row's own bound
//     T_i = max(2^-17 |X_i|^2 + 2^-14, clamp)
// (2^-14: a floor in the scaled units, d < 2^-7, which also caps P below) and give such a pair the value of a
// coincident one (d = sqrt(clamp): the reference's 1e-8 clamp, or ~0 under the pykeops convention) and zero gradient.  The
// gradient of a pair has norm |w_j| for the energy and <= |w_j| / blur for the laplacian, so a pair treated this way
// moves a row gradient by at most that much; its value by at most |w_j| sqrt(T_i) (energy; laplacian: ln2 times
// that, in units of blur / log2e).  The diagonal of K_xx / K_yy is exact (tc_zero_diagonal: S = 0).
//
// Energy coordinates are unscaled on the CUDA cores.  Here they are multiplied by the power of two that puts the
// largest centred coordinate of either cloud in [2^9, 2^10): the fp16 l term of any coordinate above 2^-3 (2^-13 of
// the largest) then stays in fp16's normal range instead of on its 2^-24 subnormal grid, and |X| <= 2^13 keeps every
// operand far from fp16's 65504.  k = d is linear, so the finalize divides the sum by that power of two exactly; the
// gradient (X_i - Y_j) / d does not depend on it.
constexpr int kTcEnergyTopLog2 = 10;
constexpr float kTcNormRel = 1.0f / 131072.f;    // 2^-17: coefficient of |X_i|^2 in T_i
constexpr float kTcNormFloor = 1.0f / 16384.f;  // 2^-14: floor of T_i (scaled units)
// Row gradients: P = w_j k'(d) / d feeds an fp16 GEMM.  The pack normalises the weights to max|w| = kTcPScale = 2^14
// (as for the gaussian) and the kernel multiplies them by 2^-kTcNormPLog2, so |w| <= 2^8 and, with d >= 2^-7
// (T_i >= 2^-14), P <= 2^15 < 65504.  Energy: d <= 2^11 sqrt(64) = 2^14, so the P of a weight within 2^-8 of the
// largest stays normal (>= 2^-14).  Laplacian: P = w 2^-d / d of the largest weight stays normal up to d ~ 18
// (k ~ 2^-18); farther pairs sit on fp16's 2^-24 subnormal grid, an absolute error of 2^-25 next to P's 2^8 scale.
// The finalize undoes both scales.
constexpr int kTcNormPLog2 = 6;

// p = 1 softmin (MODE 6 forward, MODE 7 row gradient): f_i = -eps ln2 log2 sum_j 2^(H_j - c d_ij), d from the same
// exponent GEMM as the energy kernel, on the energy's coordinates (x - center times the power of two of
// tc_energy_coord_scale), so T_i, its floor and the error bound above hold as they stand.  c = log2e / (eps scale) is
// applied in the epilogue's FFMA; scaling the coordinates by log2e / eps instead would overflow fp16 at small eps and
// large coordinates.  A pair below T_i (and the diagonal of xx / yy) takes d = sqrt(clamp): 1e-4 (tensorized) or ~0
// (unclamped), the values the reference gives coincident points.  In real units the floor is d < 2^-7 / scale, at
// most 2^-16 of the largest centred coordinate.
// Row gradient: P = 2^(t_ij - lse2_i + k_i) and Q = P / d (0 below T_i) feed the sums {sum P, sum Q, sum Q Y}.  Q goes
// to an fp16 GEMM: k_i is the largest power of two with 2^k_i <= 2^kTcL1QLog2 sqrt(T_i), so Q <= 2^15 < 65504 for every
// admitted pair (P <= 2^k_i, d >= sqrt(T_i)); k_i >= 8 since T_i >= 2^-14.  A pair of softmax weight rho has
// Q = rho 2^k_i / d > rho 2^14 sqrt(T_i) / d, normal (>= 2^-14) whenever rho >= 2^-28 d / sqrt(T_i).  k_i cancels in
// the gradient (X_i sum Q - sum Q Y) / sum P, and so does the coordinate scale (a sum of unit vectors).
constexpr int kTcL1QLog2 = 15;

// power of two that maps the largest centred coordinate `amax` into [2^9, 2^10) (1 for an all-zero cloud); the
// exponent is bounded so that clamp * scale^2 stays finite
__host__ __device__ inline float tc_energy_coord_scale(float amax) {
  if (!(amax > 0.f) || !(amax <= 3.0e38f)) return 1.f;
  int e;
  frexpf(amax, &e);  // amax < 2^e
  e = kTcEnergyTopLog2 - e;
  e = e < -40 ? -40 : (e > 40 ? 40 : e);
  return ldexpf(1.f, e);
}

// ---------------------------------------------------------------------------------------------------
// pack: one thread per (padded) point; writes its 16-byte piece of every K chunk of its tile image
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 pack8_f16(const __half* src) {
  uint4 v;
  v.x = (uint32_t)__half_as_ushort(src[0]) | ((uint32_t)__half_as_ushort(src[1]) << 16);
  v.y = (uint32_t)__half_as_ushort(src[2]) | ((uint32_t)__half_as_ushort(src[3]) << 16);
  v.z = (uint32_t)__half_as_ushort(src[4]) | ((uint32_t)__half_as_ushort(src[5]) << 16);
  v.w = (uint32_t)__half_as_ushort(src[6]) | ((uint32_t)__half_as_ushort(src[7]) << 16);
  return v;
}

// v as three bf16 terms h + m + l (24 significant bits), packed in bits 0..15, 16..31 and 32..47
__device__ __forceinline__ uint64_t tc_bf16x3_bits(float v) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  const float q = v - __bfloat162float(h);
  const __nv_bfloat16 m = __float2bfloat16_rn(q);
  const __nv_bfloat16 l = __float2bfloat16_rn(q - __bfloat162float(m));
  return (uint64_t)__bfloat16_as_ushort(h) | ((uint64_t)__bfloat16_as_ushort(m) << 16) |
         ((uint64_t)__bfloat16_as_ushort(l) << 32);
}
__device__ __forceinline__ float tc_bf16_at(uint32_t word, int hi) {
  return __bfloat162float(__ushort_as_bfloat16((unsigned short)(hi ? word >> 16 : word & 0xffffu)));
}

// Column images carry, besides the split coordinates, the per-column additive exponent term
//   c_j = h_scale * (h_a[j] + h_scale_b * h_b[j]) - |Y_j|^2 / 2      (h_a null: just the fold)
// in the rank-one chunk, and the fp32 weight w_j (kernel conv) behind the bf16 data.  Padding columns get
// c = -1e38 when h_a is given (softmin: they must vanish from the log-sum-exp) and w = 0 otherwise.
// `coord_absmax` (energy kernel, see tc_energy_coord_scale): the coordinates are further multiplied by a power of two.
// Batches (`nb` elements of n points each, stored back to back): every element is padded to whole tiles on its own, so
// slot p belongs to element b = p / npad and reads point b n + (p - b npad); h_a, h_b, w and row_extra are indexed the
// same way, and the weights of element b are normalised by w_absmax[b].
// Gather (block-sparse problems, n = number of slots, a multiple of the tile): slot p reads point gather[p], or is
// padding when gather[p] < 0.
// l1 (the p = 1 softmin, MODE 6 / 7): the rank-one chunk carries -|X|^2/2 alone, as for the kernel norms.  A column's
// H_j = h_scale (h_a + h_scale_b h_b) goes to the fp32 weight slot instead (-1e38 for padding).  A row carries, in
// elements 8..13 of the rank-one chunk (zero in every column, so the GEMM never sees them), the exponent factor
// c = h_scale / (coordinate scale) and the row term row_extra (the forward's lse2), each as three bf16 terms.
static __global__ void tc_pack_kernel(const float* __restrict__ pts, const float* __restrict__ w,
                                      const float* __restrict__ h_a, const float* __restrict__ h_b,
                                      float h_scale_b, float h_scale, const float* __restrict__ center,
                                      float scale, int64_t n, int D, int kp, int tile, int is_cols,
                                      unsigned char* __restrict__ out,
                                      const float* __restrict__ row_extra = nullptr,
                                      const float* __restrict__ w_absmax = nullptr,
                                      const float* __restrict__ coord_absmax = nullptr, int64_t nb = 1,
                                      const int* __restrict__ gather = nullptr, int l1 = 0) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t npad = ((n + tile - 1) / tile) * tile;
  if (p >= npad * nb) return;
  if (coord_absmax != nullptr) scale *= tc_energy_coord_scale(*coord_absmax);
  const int64_t b = p / npad;
  const int64_t local = p - b * npad;
  int64_t src = b * n + local;
  const int64_t t = p / tile;
  const int pt = (int)(p % tile);
  const int dk = tc_dk(D);
  const int64_t img_bytes = (int64_t)tile * kp * 2 + (is_cols ? (int64_t)tile * 4 : 0);
  unsigned char* img = out + t * img_bytes;
  bool live = local < n;
  if (gather != nullptr) {
    const int g = gather[p];
    live = g >= 0;
    src = live ? g : 0;
  }
  float sq = 0.f;
  for (int kc = 0; kc < dk / 8; ++kc) {
    __half term[kTcTerms][8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int d = kc * 8 + k;
      float X = 0.f;
      if (live && d < D) X = scale * (pts[src * D + d] - (center ? center[d] : 0.f));
      X = fminf(fmaxf(X, -60000.f), 60000.f);  // fp16 range (only reached when every exponent underflows anyway)
      sq = fmaf(X, X, sq);
      const __half h = __float2half_rn(X);
      term[0][k] = h;
      term[1][k] = __float2half_rn(X - __half2float(h));
    }
#pragma unroll
    for (int s = 0; s < kTcTerms; ++s)
      *reinterpret_cast<uint4*>(img + ((int64_t)(s * (dk / 8) + kc) * tile + pt) * 16) = pack8_f16(term[s]);
  }
  // rank-one chunk (16 wide): rows [1,1,1, r_h,r_m,r_l, 0..]   columns [c_h,c_m,c_l, 1,1,1, 0..]
  {
    float r = live ? -0.5f * sq : 0.f;
    // softmin backward: exponent - lse2_i + kTcPLog2 (P = 2^14 softmax weight, common.cuh)
    if (!is_cols && row_extra != nullptr && live && !l1) r -= row_extra[src] - (float)kTcPLog2;
    if (is_cols && h_a != nullptr && !l1) {
      if (live) {
        float h = h_a[src];
        if (h_b != nullptr) h = fmaf(h_scale_b, h_b[src], h);
        r = fmaf(h_scale, h, r);
      } else {
        r = -1.0e38f;
      }
    }
    const __nv_bfloat16 rh = __float2bfloat16_rn(r);
    const float q1 = r - __bfloat162float(rh);
    const __nv_bfloat16 rm = __float2bfloat16_rn(q1);
    const __nv_bfloat16 rl = __float2bfloat16_rn(q1 - __bfloat162float(rm));
    const uint32_t one = 0x3F80u;  // bf16 1.0
    const uint32_t a = __bfloat16_as_ushort(rh), b = __bfloat16_as_ushort(rm), c = __bfloat16_as_ushort(rl);
    uint4 v;
    if (is_cols) {
      v.x = a | (b << 16);
      v.y = c | (one << 16);
      v.z = one | (one << 16);
    } else {
      v.x = one | (one << 16);
      v.y = one | (a << 16);
      v.z = b | (c << 16);
    }
    v.w = 0u;
    const int chunk = kTcTerms * (dk / 8);
    *reinterpret_cast<uint4*>(img + ((int64_t)chunk * tile + pt) * 16) = v;
    uint4 v2 = make_uint4(0u, 0u, 0u, 0u);
    if (l1 && !is_cols) {
      const uint64_t cf = tc_bf16x3_bits(h_scale / scale), le = tc_bf16x3_bits(live && row_extra ? row_extra[src] : 0.f);
      v2.x = cf & 0xffffffffu;                   // c: elements 8, 9
      v2.y = (cf >> 32) | ((le & 0xffffu) << 16);  // c: element 10, lse2: element 11
      v2.z = (uint32_t)(le >> 16);               // lse2: elements 12, 13
    }
    *reinterpret_cast<uint4*>(img + ((int64_t)(chunk + 1) * tile + pt) * 16) = v2;
  }
  if (is_cols) {
    // (row-gradient kernels feed P = w e to an fp16 GEMM: weights are normalised to |w| <= kTcPScale = 2^14, which
    // keeps P out of fp16's subnormal range; undone in the finalize)
    float wv = (live && w) ? w[src] : 0.f;
    if (w_absmax != nullptr && w_absmax[b] > 0.f) wv = (wv / w_absmax[b]) * kTcPScale;
    if (l1) {
      wv = -1.0e38f;
      if (live) {
        float h = h_a[src];
        if (h_b != nullptr) h = fmaf(h_scale_b, h_b[src], h);
        wv = h_scale * h;
      }
    }
    reinterpret_cast<float*>(img + (int64_t)tile * kp * 2)[pt] = wv;
  }
}

// ---------------------------------------------------------------------------------------------------
// the reduction kernel
// ---------------------------------------------------------------------------------------------------
constexpr int kTcBN = 128;      // columns per tile = N of the exponent GEMM
constexpr int kTcWG = 2;        // consumer warpgroups per CTA, 64 rows each (kTcM = 128 rows per CTA)
constexpr int kTcThreads = 128 * kTcWG + 32;  // + one producer warp behind the warpgroups
constexpr int kTcParts = 4;     // forward partial sets per column split: one per lane of an accumulator quad
constexpr int kTcMaxStage = 4;

// S = the exponent of the 64 rows of one warpgroup against a 128-column tile (both images in shared memory):
// the rank-one chunk first (bf16, overwrites the accumulator), then the three fp16 cross products hh, hl, lh.
// `a_addr` points at the warpgroup's first row of the row image.  Committed as one group; the caller waits.
__device__ __forceinline__ void tc_exponent_gemm(float (&s)[64], uint32_t a_addr, uint32_t b_addr, int seg) {
  constexpr uint32_t kA = kTcM * 16, kB = kTcBN * 16;  // byte distance between 8-element K chunks
  wgmma_fence();
  {
    const int c = kTcTerms * seg;
    wgmma_ss_n128_bf16(s, make_smem_desc(a_addr + c * kA, kA, 128), make_smem_desc(b_addr + c * kB, kB, 128), false);
  }
#pragma unroll
  for (int prod = 0; prod < 3; ++prod) {
    const int ta = (prod == 2) ? 1 : 0, tb = (prod == 1) ? 1 : 0;  // (A term, B term): hh, hl, lh
    for (int kk = 0; kk < seg / 2; ++kk)
      wgmma_ss_n128_f16(s, make_smem_desc(a_addr + (ta * seg + 2 * kk) * kA, kA, 128),
                        make_smem_desc(b_addr + (tb * seg + 2 * kk) * kB, kB, 128), true);
  }
  wgmma_commit();
}

// Rows and columns are the same cloud (the K_xx / K_yy terms of an MMD): the exponent of the pair (i, i) is
// -|X_i - X_i|^2/2 = 0 exactly, but the expansion X.X - |X|^2/2 - |X|^2/2 cancels three O(|x/blur|^2) numbers in
// fp32 (5e-3 at blur = .05, D = 64, where the diagonal IS the value).  `diag` = first row of this thread minus the
// tile's first column; the test is taken on one column tile in N/128.
__device__ __forceinline__ void tc_zero_diagonal(float (&s)[64], int64_t diag, int cq) {
  if (diag < -8 || diag >= kTcBN) return;
#pragma unroll
  for (int j = 0; j < 64; ++j)
    if (8 * (j >> 2) + cq + (j & 1) == diag + 8 * ((j >> 1) & 1)) s[j] = 0.f;
}

// MODE 4 / 5: |X_i|^2 of a row of the row image, from its rank-one chunk (r = -|X|^2/2 in three bf16 terms at
// elements 3..5; no row term is folded in for these modes), and the row's coincidence bound T_i (see above).
// `clampq` is the clamp on the scaled d^2, already multiplied by the energy coordinate scale squared.
__device__ __forceinline__ float tc_norm_row_bound(const unsigned char* sa, int kp, int local_row, float clampq) {
  const int chunk = kTcTerms * (tc_dk_of_kp(kp) / 8);
  const uint4 v = *reinterpret_cast<const uint4*>(sa + ((int64_t)chunk * kTcM + local_row) * 16);
  const float r = __bfloat162float(__ushort_as_bfloat16((unsigned short)(v.y >> 16))) +
                  __bfloat162float(__ushort_as_bfloat16((unsigned short)(v.z & 0xffffu))) +
                  __bfloat162float(__ushort_as_bfloat16((unsigned short)(v.z >> 16)));
  return fmaxf(fmaf(-2.f * kTcNormRel, r, kTcNormFloor), clampq);
}
// the clamp on the scaled d^2 (never below 1e-30, so that d^2 rsqrt(d^2) of a coincident pair is 0, not NaN)
__device__ __forceinline__ float tc_norm_clampq(float clampq, const float* coord_absmax) {
  if (coord_absmax != nullptr) {
    const float c = tc_energy_coord_scale(*coord_absmax);
    clampq *= c * c;
  }
  return fmaxf(clampq, 1e-30f);
}
// MODE 4 / 5: the clamp (scaled in place) and the coincidence bounds tb of the thread's two rows of the row image
__device__ __forceinline__ void tc_norm_row_bounds(float (&tb)[2], float& clampq, const float* coord_absmax,
                                                   const unsigned char* sa, int kp, int wg, int warp, int lane) {
  clampq = tc_norm_clampq(clampq, coord_absmax);
  const int lr = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  tb[0] = tc_norm_row_bound(sa, kp, lr, clampq);
  tb[1] = tc_norm_row_bound(sa, kp, lr + 8, clampq);
}
// MODE 6 / 7: the exponent factor c and the row term lse2 of a row of the row image (tc_pack_kernel's l1 layout), and
// the same for the thread's two rows
__device__ __forceinline__ float2 tc_l1_row_terms(const unsigned char* sa, int kp, int local_row) {
  const int chunk = kTcTerms * (tc_dk_of_kp(kp) / 8) + 1;
  const uint4 v = *reinterpret_cast<const uint4*>(sa + ((int64_t)chunk * kTcM + local_row) * 16);
  return make_float2(tc_bf16_at(v.x, 0) + tc_bf16_at(v.x, 1) + tc_bf16_at(v.y, 0),
                     tc_bf16_at(v.y, 1) + tc_bf16_at(v.z, 0) + tc_bf16_at(v.z, 1));
}
__device__ __forceinline__ void tc_l1_rows(float2 (&rt)[2], const unsigned char* sa, int kp, int wg, int warp,
                                           int lane) {
  const int lr = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  rt[0] = tc_l1_row_terms(sa, kp, lr);
  rt[1] = tc_l1_row_terms(sa, kp, lr + 8);
}
// The weighted value of one pair from its exponent s: 2^s (MODE 0), or k(d) with d^2 = clamp for a pair below the row
// bound t (and the diagonal), else -2 s (MODE 4 / 5)
template <int MODE>
__device__ __forceinline__ float tc_pair_value(float s, float t, float clampq) {
  if constexpr (MODE == 0) return ex2_approx(s);
  const float q = -2.f * s;
  const float d2 = q < t ? clampq : q;
  const float d = d2 * rsqrt_approx(d2);
  if constexpr (MODE == 4) return ex2_approx(-d);
  return d;
}

// BLOCKS (block-sparse problems): CTA x runs segment x = (row_start, row_count, piece_begin, piece_end) of `bseg`, one
// 128-row tile of one row cluster; its columns are the pieces [piece_begin, piece_end) of `bpieces`, (col_start,
// col_count) runs of whole column tiles.  Rows, columns and pieces are in slots, multiples of 128 (validated by the
// host).  The split's tiles are [split tps, split tps + tps) of the concatenation of the segment's pieces; `piece` /
// `off` locate the first of them.  A split past the segment's last tile has nt = 0.
struct TcBlockSpan {
  int row_tile, nt, piece, off;
};
__device__ __forceinline__ TcBlockSpan tc_block_span(const int4* __restrict__ seg, const int2* __restrict__ pieces,
                                                     int s, int split, int tps) {
  const int4 sg = seg[s];
  TcBlockSpan r;
  r.row_tile = sg.x / kTcM;
  const int first = split * tps;
  int pc = sg.z, acc = 0;
  while (pc < sg.w) {
    const int n = pieces[pc].y / kTcBN;
    if (acc + n > first) break;
    acc += n;
    ++pc;
  }
  r.piece = pc;
  r.off = first - acc;
  int total = acc;
  for (int q = pc; q < sg.w && total < first + tps; ++q) total += pieces[q].y / kTcBN;
  r.nt = max(0, min(tps, total - first));
  return r;
}

// What tc_reduce_kernel and tc_bwd_kernel share before their consumer loops.  Shared memory: the row image `sa`, the
// ring of NSTAGE column slots `sb` and the mbarriers behind it.  The CTA's work: row tile `row_tile` (of batch element
// `elem`) against the nt column tiles of split `split` from tile t0 (BLOCKS: from tile bs.off of piece bs.piece).
struct TcCta {
  unsigned char *sa, *sb;
  uint64_t *bar_a, *full_b, *empty_b;
  int a_bytes, b_bytes;
  int split, row_tile, elem, t0, nt;
  TcBlockSpan bs;
};
// Carves the shared memory, finds the CTA's tiles and initialises the barriers (the CTA's threads all call it)
template <bool BATCH, bool BLOCKS>
__device__ __forceinline__ TcCta tc_cta_prologue(unsigned char* smem, int kp, int NSTAGE, int ntiles_b,
                                                 int tiles_per_split, int rtpe, const int4* __restrict__ bseg,
                                                 const int2* __restrict__ bpieces) {
  TcCta c;
  c.a_bytes = kTcM * kp * 2;
  c.b_bytes = kTcBN * kp * 2 + kTcBN * 4;
  c.sa = smem;
  c.sb = smem + tc_a_span(kp);
  c.bar_a = reinterpret_cast<uint64_t*>(c.sb + NSTAGE * c.b_bytes);
  c.full_b = c.bar_a + 1;
  c.empty_b = c.full_b + kTcMaxStage;

  c.split = blockIdx.y;
  c.bs = TcBlockSpan{};
  if constexpr (BLOCKS) c.bs = tc_block_span(bseg, bpieces, blockIdx.x, c.split, tiles_per_split);
  c.row_tile = BLOCKS ? c.bs.row_tile : (int)blockIdx.x;
  c.elem = BATCH ? c.row_tile / rtpe : 0;
  c.t0 = c.elem * ntiles_b + c.split * tiles_per_split;
  const int t1 = min((c.elem + 1) * ntiles_b, c.t0 + tiles_per_split);
  c.nt = BLOCKS ? c.bs.nt : t1 - c.t0;

  if (threadIdx.x == 0) {
    mbar_init(c.bar_a, 1);
    for (int s = 0; s < NSTAGE; ++s) {
      mbar_init(&c.full_b[s], 1);
      mbar_init(&c.empty_b[s], 4 * kTcWG);  // every consumer warp, once its MMAs and weight reads are done
    }
    mbar_fence_init();
  }
  __syncthreads();
  return c;
}

// The TMA producer (one lane of the warp behind the warpgroups): the row image once, then the CTA's column tiles
// through the ring.  EXTRA: every column tile travels with a second image of e_bytes (tile ct at e_imgs + ct e_bytes)
// into slot `st` of a ring of its own at e_ring, its bytes in the stage's expect_tx (tcapply.cuh: the value image).
template <bool BLOCKS, bool EXTRA = false>
__device__ __forceinline__ void tc_produce(const TcCta& c, const unsigned char* __restrict__ a_imgs,
                                           const unsigned char* __restrict__ b_imgs,
                                           const int2* __restrict__ bpieces, int NSTAGE, int lane,
                                           const unsigned char* __restrict__ e_imgs = nullptr,
                                           unsigned char* e_ring = nullptr, int e_bytes = 0) {
  if (lane == 0) {
    mbar_arrive_expect_tx(c.bar_a, c.a_bytes);
    tma_load_1d(c.sa, a_imgs + (int64_t)c.row_tile * c.a_bytes, c.a_bytes, c.bar_a);
    int pc = c.bs.piece, off = c.bs.off;  // BLOCKS: position in the segment's pieces
    for (int k = 0; k < c.nt; ++k) {
      const int st = k % NSTAGE;
      if (k >= NSTAGE) mbar_wait(&c.empty_b[st], ((k / NSTAGE) + 1) & 1);
      mbar_arrive_expect_tx(&c.full_b[st], EXTRA ? c.b_bytes + e_bytes : c.b_bytes);
      int ct = c.t0 + k;
      if constexpr (BLOCKS) {
        const int2 pp = bpieces[pc];
        ct = pp.x / kTcBN + off;
        if (++off == pp.y / kTcBN) {
          ++pc;
          off = 0;
        }
      }
      tma_load_1d(c.sb + st * c.b_bytes, b_imgs + (int64_t)ct * c.b_bytes, c.b_bytes, &c.full_b[st]);
      if constexpr (EXTRA)
        tma_load_1d(e_ring + (int64_t)st * e_bytes, e_imgs + (int64_t)ct * e_bytes, e_bytes, &c.full_b[st]);
    }
  }
}

// The output row of tile row `row`: BATCH, row b n_local + local of a live row of element b; BLOCKS, row_src of the
// slot.  N for a padding row, which writes nothing.
template <bool BATCH, bool BLOCKS>
__device__ __forceinline__ int64_t tc_out_row(int64_t row, int elem, int rtpe, int64_t n_local,
                                              const int* __restrict__ row_src, int64_t N) {
  if constexpr (BATCH) {
    const int64_t local = row - (int64_t)elem * rtpe * kTcM;
    row = local < n_local ? (int64_t)elem * n_local + local : N;
  }
  if constexpr (BLOCKS) {
    const int g = row_src[row];
    row = g >= 0 ? g : N;
  }
  return row;
}

// The epilogue of tc_reduce_kernel on one column tile: the exponents s of the thread's two rows (row0 and row0 + 8)
// against the tile, turned into MODE's row sums (acc: MODE 0 / 4 / 5; the running (m, srun): MODE 1 / 6).  `wts` is
// the fp32 column slot of ring stage `st` (weights, or H_j for MODE 6) behind a column image of K extent kp; k is the
// CTA's column tile, row0 the thread's first row.
template <int MODE>
__device__ __forceinline__ void tc_reduce_tile(float (&s)[64], const TcCta& c, int st, int kp, int k, int64_t row0,
                                               const float (&tb)[2], const float2 (&rt)[2], float clampq,
                                               int self_mode, int cq, float (&acc)[2], float (&m)[2],
                                               float (&srun)[2]) {
  if constexpr (MODE == 6) {
    // the p = 1 exponent t = H_j - c d_ij in place of s, then the softmin's log-sum-exp below
    if (self_mode) tc_zero_diagonal(s, row0 - (int64_t)(c.t0 + k) * kTcBN, cq);
    const float* hs = reinterpret_cast<const float*>(c.sb + st * c.b_bytes + kTcBN * kp * 2);
#pragma unroll
    for (int n8 = 0; n8 < kTcBN / 8; ++n8) {
      const float2 hj = *reinterpret_cast<const float2*>(hs + 8 * n8 + cq);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        s[4 * n8 + 2 * h] = fmaf(-rt[h].x, tc_pair_value<5>(s[4 * n8 + 2 * h], tb[h], clampq), hj.x);
        s[4 * n8 + 2 * h + 1] = fmaf(-rt[h].x, tc_pair_value<5>(s[4 * n8 + 2 * h + 1], tb[h], clampq), hj.y);
      }
    }
  }
  if constexpr (MODE != 1 && MODE != 6) {
    if (self_mode) tc_zero_diagonal(s, row0 - (int64_t)(c.t0 + k) * kTcBN, cq);
    const float* wts = reinterpret_cast<const float*>(c.sb + st * c.b_bytes + kTcBN * kp * 2);
    float ts[2] = {0.f, 0.f};
#pragma unroll
    for (int n8 = 0; n8 < kTcBN / 8; ++n8) {
      const float2 w = *reinterpret_cast<const float2*>(wts + 8 * n8 + cq);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        ts[h] = fmaf(tc_pair_value<MODE>(s[4 * n8 + 2 * h], tb[h], clampq), w.x, ts[h]);
        ts[h] = fmaf(tc_pair_value<MODE>(s[4 * n8 + 2 * h + 1], tb[h], clampq), w.y, ts[h]);
      }
    }
    acc[0] += ts[0];
    acc[1] += ts[1];
  } else {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // the 32 exponents of row h in this tile: s[4 n8 + 2 h + e]
      float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
      for (int n8 = 0; n8 < kTcBN / 8; ++n8) {
        cs0 += ex2_approx(s[4 * n8 + 2 * h] - m[h]);
        cs1 += ex2_approx(s[4 * n8 + 2 * h + 1] - m[h]);
      }
      if (!(cs0 + cs1 <= 1.8446744e19f)) {
        // outdated max (a term above 2^64 or an overflow): rebase on this chunk's max and redo it
        float cm = s[2 * h];
#pragma unroll
        for (int n8 = 0; n8 < kTcBN / 8; ++n8) cm = fmax3(cm, s[4 * n8 + 2 * h], s[4 * n8 + 2 * h + 1]);
        srun[h] *= ex2_approx(m[h] - cm);
        m[h] = cm;
        cs0 = 0.f;
        cs1 = 0.f;
#pragma unroll
        for (int n8 = 0; n8 < kTcBN / 8; ++n8) {
          cs0 += ex2_approx(s[4 * n8 + 2 * h] - m[h]);
          cs1 += ex2_approx(s[4 * n8 + 2 * h + 1] - m[h]);
        }
      }
      srun[h] += cs0 + cs1;
    }
  }
}

// The partials of tc_reduce_kernel's two rows of the thread (layout below)
template <int MODE, bool BATCH, bool BLOCKS>
__device__ __forceinline__ void tc_reduce_store(float* __restrict__ part, const float (&acc)[2], const float (&m)[2],
                                                const float (&srun)[2], int64_t row0, int split, int elem, int rtpe,
                                                int64_t n_local, const int* __restrict__ row_src, int64_t N,
                                                int lane) {
  const int q = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t row = tc_out_row<BATCH, BLOCKS>(row0 + 8 * h, elem, rtpe, n_local, row_src, N);
    if (row < N) {
      if constexpr (MODE != 1 && MODE != 6) {
        part[((int64_t)split * kTcParts + q) * N + row] = acc[h];
      } else {
        reinterpret_cast<float2*>(part)[((int64_t)split * kTcParts + q) * N + row] = make_float2(m[h], srun[h]);
      }
    }
  }
}

// MODE 0: gaussian kernel conv  part[(split*kTcParts + q)*N + row]   = sum_j w_j 2^S_ij
// MODE 1: softmin               part2[(split*kTcParts + q)*N + row]  = (m, s) with sum_j 2^S_ij = s 2^m  (lazy max,
//         sum-guarded exactly like softmin.cuh; same partial format as softmin_partial_kernel)
// MODE 4: laplacian kernel conv  part[...] = sum_j w_j 2^-d_ij       MODE 5: energy  part[...] = sum_j w_j d_ij
//         (d_ij from the exponent as described above; `clampq` and `coord_absmax` are read by these modes only)
// MODE 6: p = 1 softmin, MODE 1's (m, s) partials of sum_j 2^(H_j - c d_ij) (d_ij as for MODE 5, H_j from the weight
//         slot, c from the row image; see kTcL1QLog2)
// (row gradients — modes 2 and 3 — are a two-GEMM kernel of their own: tcbwd.cuh)
//
// A CTA owns one 128-row tile: its row image is loaded once by TMA and stays in shared memory, the column tiles
// stream through a ring of NSTAGE slots (full / empty mbarriers, one producer lane).  Each of the two consumer
// warpgroups multiplies its 64 rows by the tile (wgmma, accumulator in registers) and turns the exponents into
// row sums in the same registers: while one warpgroup runs its exponentials the tensor cores serve the other.
// A thread holds two rows x 32 columns of every tile; q = lane % 4 picks which quarter of the columns it summed,
// and the four quarters are kept as separate partial sets (no shuffles, merged by the finalize kernels).
//
// BATCH: B problems of n_local rows against the same number of columns each, every element padded to whole tiles on
// its own (tc_pack_kernel).  Row tile r belongs to element b = r / rtpe and reads only that element's column tiles
// [b ntiles_b, (b + 1) ntiles_b) (ntiles_b = column tiles per element), cut into splits as without a batch; a live row
// (local index < n_local) writes its partials at row b n_local + local of the N = B n_local rows, padding rows write
// nothing.  Rows and columns of a self term are padded alike, so `row0 - column` still finds the diagonal.
// BLOCKS (softmin only): CTA x runs segment x (tc_block_span); row slot r writes its partials at row row_src[r], padding
// slots (row_src < 0) write nothing.  Every split writes every live row of its segment, (kNegBig, 0) when it has no
// tile, so the finalize merges without knowing the layout.
template <int MODE, bool BATCH = false, bool BLOCKS = false>
__global__ void __launch_bounds__(kTcThreads, 1)
    tc_reduce_kernel(const unsigned char* __restrict__ a_imgs, const unsigned char* __restrict__ b_imgs,
                     float* __restrict__ part, int64_t N, int kp, int ntiles_b, int tiles_per_split, int NSTAGE,
                     int D, int self_mode, float clampq, const float* __restrict__ coord_absmax, int rtpe,
                     int64_t n_local, const int4* __restrict__ bseg = nullptr,
                     const int2* __restrict__ bpieces = nullptr, const int* __restrict__ row_src = nullptr) {
  static_assert(MODE == 0 || MODE == 1 || MODE == 4 || MODE == 5 || MODE == 6, "row gradients live in tcbwd.cuh");
  static_assert(!BLOCKS || (MODE == 1 && !BATCH), "the block-sparse layout serves the softmin of one problem");
  extern __shared__ __align__(1024) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TcCta c = tc_cta_prologue<BATCH, BLOCKS>(smem, kp, NSTAGE, ntiles_b, tiles_per_split, rtpe, bseg, bpieces);
  if (warp == 4 * kTcWG) {
    tc_produce<BLOCKS>(c, a_imgs, b_imgs, bpieces, NSTAGE, lane);
    return;
  }
  // ===== consumer warpgroups: wgmma -> exp2 -> row sums =====
  const int wg = warp >> 2;
  const int seg = tc_dk_of_kp(kp) / 8;  // 8-element chunks per split term
  const uint32_t a_addr = smem_u32(c.sa) + wg * 64 * 16;
  const int64_t row0 = (int64_t)c.row_tile * kTcM + wg * 64 + (warp & 3) * 16 + (lane >> 2);  // and row0 + 8
  const int cq = 2 * (lane & 3);  // this thread's first column in every 8-column block
  float acc[2] = {0.f, 0.f};                 // MODE 0, 4, 5: weighted sums
  float m[2] = {kNegBig, kNegBig}, srun[2] = {0.f, 0.f};  // MODE 1: running (m, s)
  mbar_wait(c.bar_a, 0);
  float tb[2] = {0.f, 0.f};  // MODE 4 / 5 / 6: coincidence bound of each row
  if constexpr (MODE >= 4) tc_norm_row_bounds(tb, clampq, coord_absmax, c.sa, kp, wg, warp, lane);
  float2 rt[2] = {};  // MODE 6: (c, -) of each row
  if constexpr (MODE == 6) tc_l1_rows(rt, c.sa, kp, wg, warp, lane);
  for (int k = 0; k < c.nt; ++k) {
    const int st = k % NSTAGE;
    mbar_wait(&c.full_b[st], (k / NSTAGE) & 1);
    float s[64];
    tc_exponent_gemm(s, a_addr, smem_u32(c.sb + st * c.b_bytes), seg);
    wgmma_wait<0>();
    reg_fence(s);
    tc_reduce_tile<MODE>(s, c, st, kp, k, row0, tb, rt, clampq, self_mode, cq, acc, m, srun);
    __syncwarp();
    if (lane == 0) mbar_arrive(&c.empty_b[st]);
  }
  tc_reduce_store<MODE, BATCH, BLOCKS>(part, acc, m, srun, row0, c.split, c.elem, rtpe, n_local, row_src, N, lane);
}

}  // namespace b200ot
