// b200ot — shared device helpers (sm_90a).
//
// mbarrier / bulk-TMA wrappers, two-column float2 arithmetic and the MUFU intrinsics the
// softmin and kernel-conv kernels are built from.  Nothing here is exported.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "b200ot kernels are written for sm_90a (H100); compile with -gencode arch=compute_90a,code=sm_90a"
#endif

namespace b200ot {

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
// "minus infinity" that stays finite under (a - b): used to initialise running maxima.
constexpr float kNegBig = -1.0e30f;
// The tensor-core row gradients (tcbwd.cuh) feed 2^kTcPLog2 * P to their fp16 GEMM instead of P <= 1: the weights of
// a softmax over M columns are ~1/M, below fp16's normal range (6.1e-5) once M >~ 16k, where the fixed 6e-8 subnormal
// grid would round them with a bias.  2^14 P < 65504 (fp16's maximum) holds for P < 4.  Undone before any sum leaves
// the library: conv_bwd_finalize_kernel and b200ot_softmin_bwd_sums (softmin_bwd_finalize divides it out).
constexpr int kTcPLog2 = 14;
constexpr float kTcPScale = 16384.f;  // 2^kTcPLog2

// ---------------------------------------------------------------------------------------------
// Packed column layout ("colpack"), produced by pack_cols_kernel and consumed by every
// reduction kernel.  Columns are stored two at a time; a column-pair packet holds
//   NF2 float2 values  { v_k[j0], v_k[j0+1] },  k = 0..D-1 coordinates, k = D the per-column
//   additive term H, remaining slots zero padding so that a packet is a multiple of 16 bytes.
// A tile of TJ columns is therefore one contiguous run of TJ/2 packets: a single 1-D bulk TMA copy.
// ---------------------------------------------------------------------------------------------
// float2 slots per column-pair packet for D coordinates + `extra` per-column scalars (rounded to 16 B)
__host__ __device__ inline int colfmt_nf2(int D, int extra) { return ((D + extra + 1) / 2) * 2; }

// ---------------------------------------------------------------------------------------------
// mbarrier + 1-D bulk TMA (cp.async.bulk -> SASS UBLKCP)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}
// global -> shared bulk copy, completion signalled on `bar` (bytes multiple of 16, both 16B aligned)
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// math
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rsqrt_approx(float x) {
  float y;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sqrt_approx(float x) {
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
__device__ __forceinline__ float2 dup2(float a) { return make_float2(a, a); }

// Two columns at a time: the kernels carry column pairs as float2.  Hopper has no packed fp32 FMA, so each
// is two scalar round-to-nearest operations (the same values a packed instruction would produce).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// 2^x for x <= 0 evaluated on the FMA pipe (no MUFU): Cody-Waite split x = n + f, f in [-.5,.5],
// degree-5 minimax polynomial for 2^f (rel. err ~1.2e-7), exponent patched in with one integer add.
// Arguments below -126 flush to 0.  Used to off-load a fraction of the exponentials from the
// 16-lane/SM MUFU unit to the 128-lane/SM FMA unit.
__device__ __forceinline__ float ex2_poly(float x) {
  x = fminf(fmaxf(x, -126.0f), 127.0f);
  const float magic = 12582912.0f;  // 1.5 * 2^23
  float t = x + magic;              // round-to-nearest integer lives in the low mantissa bits
  float n = t - magic;
  float f = x - n;
  // near-minimax fit (relative error, c0 pinned to 1) — see tools/fit_ex2_poly.py
  float p = 1.3264726694e-3f;
  p = fmaf(p, f, 9.6715127364e-3f);
  p = fmaf(p, f, 5.5507337449e-2f);
  p = fmaf(p, f, 2.4022242083e-1f);
  p = fmaf(p, f, 6.9314697760e-1f);
  p = fmaf(p, f, 1.0f);
  int bits = __float_as_int(p) + (__float_as_int(t) << 23);
  return __int_as_float(bits);
}

}  // namespace b200ot
