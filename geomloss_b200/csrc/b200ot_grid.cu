// b200ot — separable soft-C-transform on regular grids (images / volumes).
// Reference semantics: softmin_grid (src/geomloss/_legacy/utils.py:190-279), called by the image Sinkhorn
// loop (src/geomloss/_legacy/sinkhorn_images.py:26-202): for a (batch, N, N[, N]) array h and the cost
// |x - y|^p / p on the pixel grid x = arange(N)/N, the softmin over the whole grid factorises into one
// 1-D log-sum-exp per axis,
//     out[.., i, ..] = log sum_j exp( in[.., j, ..] - k(x_i - x_j) ),   k(d) = d^2/(2 eps)  (p = 2),  |d|/eps  (p = 1)
// applied along every axis in turn, followed by a multiplication by -eps.
//
// One pass = one launch of grid_pass_kernel over the tensor viewed as [outer][N][inner]: a CTA loads a
// tile of 32 lines (all N entries along the axis) into shared memory with coalesced accesses — along the
// contiguous direction for the strided passes, transposed for the last axis — then every thread owns 8
// outputs of one line at a time and sweeps the N inputs (conflict-free LDS, lanes = lines): cost terms from
// exact integer offsets on the grid (a 14-entry packed table per 8 x 8 chunk), packed fp32 adds, lazy-max
// log-sum-exp in the log2 domain with the same 2^64 sum guard as softmin.cuh, 1 MUFU.EX2 per (output, input) pair.  Results are staged in a second shared tile
// and written back with the access pattern of the load, so passes run in place.
// Work per pass: N^(dim+1) pairs -> SFU-bound like the point-cloud softmin (256^3: 4.3e9 pairs, ~1 ms);
// HBM traffic 2 x 4 N^dim bytes per pass.
// b200ot_softmin_grid_axes runs the same pass on grids with their own side, pitch and periodic flag per axis (the
// PERIODIC instantiations), and b200ot_grid_plan_apply applies the plan of that softmin to K value channels
// (grid_apply_kernel below): the operators of ot.solve_grid.
#include <math.h>

#include "b200ot.h"
#include "common.cuh"
#include "host_util.cuh"

namespace b200ot {

constexpr int kGridTW = 32;  // lines per CTA tile (one per lane); 16 for N > 880, where two 32-line tiles of
                             // N x 33 floats no longer fit the 227 KB of shared memory (two lanes then share a
                             // line and split its outputs)
constexpr int kGridR = 8;  // outputs per thread per sweep
constexpr int kGridWarps = 8;

struct GridPassArgs {
  const float* h_a;      // first pass: input = in_scale * (h_a + h_scale_b * h_b); later passes read `out` in place
  const float* h_b;      // nullable
  const float* out_old;  // last pass only, nullable
  float* out;
  float h_scale_b, in_scale, alpha_old, beta, out_scale, xscale;
  int N, first, last;
  int64_t outer, inner;
};

// Offset n between two indices of an axis of side N: |n|, or the shorter way round min(|n|, N - |n|) on a periodic
// axis.  Exact in fp32 for N <= 1024.
template <bool PERIODIC>
__device__ __forceinline__ float grid_offset(float n, float Nf) {
  if (!PERIODIC) return n;
  const float a = fabsf(n);
  return fminf(a, Nf - a);
}

template <int P, int TW, bool PERIODIC>
__global__ void __launch_bounds__(kGridWarps * 32) grid_pass_kernel(GridPassArgs A) {
  constexpr int kGridTW = TW, kGridRS = TW + 1, NSUB = 32 / TW;
  extern __shared__ float smem_f[];
  float* tile = smem_f;                      // [N][33] inputs
  float* otile = smem_f + A.N * kGridRS;     // [N][33] outputs
  const int N = A.N;
  const int lane = (threadIdx.x & 31) % TW, warp = (threadIdx.x >> 5) * NSUB + (threadIdx.x & 31) / TW;
  const bool last_axis = (A.inner == 1);
  int64_t o, w0;
  int nw;  // live lines in this tile
  if (last_axis) {
    o = (int64_t)blockIdx.x * kGridTW;
    w0 = 0;
    nw = (int)min((int64_t)kGridTW, A.outer - o);
  } else {
    const int64_t tiles_in = (A.inner + kGridTW - 1) / kGridTW;
    o = blockIdx.x / tiles_in;
    w0 = (blockIdx.x % tiles_in) * kGridTW;
    nw = (int)min((int64_t)kGridTW, A.inner - w0);
  }

  // ---- load ----
  for (int idx = threadIdx.x; idx < N * kGridTW; idx += blockDim.x) {
    int j, w;
    if (last_axis) {
      w = idx / N;
      j = idx % N;
    } else {
      j = idx / kGridTW;
      w = idx % kGridTW;
    }
    float v = -INFINITY;
    if (w < nw) {
      const int64_t gi = last_axis ? ((o + w) * N + j) : ((o * N + j) * A.inner + w0 + w);
      if (A.first) {
        v = A.h_a[gi];
        if (A.h_b) v = fmaf(A.h_scale_b, A.h_b[gi], v);
        v *= A.in_scale;
      } else {
        v = A.out[gi];
      }
    }
    tile[j * kGridRS + w] = v;
  }
  __syncthreads();

  // ---- sweep: warp g owns outputs [g*per_warp, (g+1)*per_warp) of every line of the tile ----
  // A thread owns kGridR = 8 consecutive outputs of its line and sweeps the inputs 8 at a time.  The cost term of the
  // pair (output ib + r, input j0 + c) depends on n = (ib - j0) + (r - c) only: 14 packed table entries
  //     W[k] = ( -k(n), -k(n - 1) ),  n = (ib - j0) + k,  k = r - 2q in [-6, 7]        k(n) = xs^2 n^2  or  xs |n|
  // per chunk (n and n^2 are exact small integers in fp32: ONE rounding per entry) serve its 64 pairs, which are then
  // three packed instructions per two pairs — t = a + W, t - m, sum += 2^(t - m) — instead of four scalar ones per
  // pair: the loop is bound by the 64 MUFU.EX2, not by issue slots (ncu before: XU 77 %, issue 68 %).
  const float kq = (P == 2) ? -A.xscale * A.xscale : -A.xscale;
  const int per_warp = (N + kGridWarps * NSUB - 1) / (kGridWarps * NSUB);
  const int i_end = min(N, (warp + 1) * per_warp);
  for (int ib = warp * per_warp; ib < i_end; ib += kGridR) {
    float m[kGridR], s[kGridR];
#pragma unroll
    for (int r = 0; r < kGridR; ++r) {
      // reference exponent = the j = i term (a lower bound of the row max, usually within a few units of it): a
      // sweep that starts from -big climbs the whole Gaussian flank and re-bases at EVERY chunk left of i
      // (measured: 1.58 XU ops per pair instead of 1)
      m[r] = (ib + r < N) ? fmaxf(tile[(ib + r) * kGridRS + lane], kNegBig) : kNegBig;
      s[r] = 0.f;
    }
    for (int j0 = 0; j0 < N; j0 += 8) {
      float2 a2[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        a2[q].x = (j0 + 2 * q < N) ? tile[(j0 + 2 * q) * kGridRS + lane] : -INFINITY;
        a2[q].y = (j0 + 2 * q + 1 < N) ? tile[(j0 + 2 * q + 1) * kGridRS + lane] : -INFINITY;
      }
      const float2 base = dup2((float)(ib - j0));
      float2 W[14];
#pragma unroll
      for (int k = -6; k <= 7; ++k) {
        float2 n = fadd2(base, make_float2((float)k, (float)(k - 1)));
        if constexpr (PERIODIC) n = make_float2(grid_offset<true>(n.x, (float)N), grid_offset<true>(n.y, (float)N));
        if (P == 2) {
          W[k + 6] = fmul2(fmul2(n, n), dup2(kq));
        } else {
          W[k + 6] = fmul2(make_float2(fabsf(n.x), fabsf(n.y)), dup2(kq));
        }
      }
#pragma unroll
      for (int r = 0; r < kGridR; ++r) {
        const float2 nm = dup2(-m[r]);
        float2 cs2 = dup2(0.f);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 e = fadd2(fadd2(a2[q], W[r - 2 * q + 6]), nm);
          cs2 = fadd2(cs2, make_float2(ex2_approx(e.x), ex2_approx(e.y)));
        }
        float cs = cs2.x + cs2.y;
        if (!(cs <= 1.8446744e19f)) {
          // outdated max (or first chunk): rebase on this chunk's max and redo it
          float t[8];
          float cm = -INFINITY;
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            const float n = grid_offset<PERIODIC>((float)(ib + r - j0 - c), (float)N);
            const float av = (c & 1) ? a2[c >> 1].y : a2[c >> 1].x;
            t[c] = av + kq * ((P == 2) ? n * n : fabsf(n));
            cm = fmaxf(cm, t[c]);
          }
          cs = 0.f;
          if (cm > kNegBig) {  // otherwise every input of the chunk is -inf: nothing to add
            s[r] *= ex2_approx(m[r] - cm);
            m[r] = cm;
#pragma unroll
            for (int c = 0; c < 8; ++c) cs += ex2_approx(t[c] - cm);
          }
        }
        s[r] += cs;
      }
    }
#pragma unroll
    for (int r = 0; r < kGridR; ++r) {
      const int i = ib + r;
      if (i < i_end) {
        int e = 0;
        const float f = frexpf(s[r], &e);  // log2(s) = e + log2(f), f in [0.5, 1): exact exponent, accurate mantissa
        otile[i * kGridRS + lane] = (s[r] > 0.f) ? (m[r] + (float)e) + log2f(f) : -INFINITY;
      }
    }
  }
  __syncthreads();

  // ---- store (same access pattern as the load) ----
  for (int idx = threadIdx.x; idx < N * kGridTW; idx += blockDim.x) {
    int j, w;
    if (last_axis) {
      w = idx / N;
      j = idx % N;
    } else {
      j = idx / kGridTW;
      w = idx % kGridTW;
    }
    if (w >= nw) continue;
    const int64_t gi = last_axis ? ((o + w) * N + j) : ((o * N + j) * A.inner + w0 + w);
    float v = otile[j * kGridRS + w];
    if (A.last) {
      v = A.beta * (A.out_scale * v);
      if (A.out_old) v = fmaf(A.alpha_old, A.out_old[gi], v);
    }
    A.out[gi] = v;
  }
}

// ---- the plan applied to K value channels ------------------------------------------------------------------------
// Each pixel carries a state (l, s_1..s_K): weight 2^l and weighted mean s.  A pass along one axis maps it to
//     l'_i = log2 sum_j 2^(l_j - c(i, j)),      s'_i = sum_j 2^(l_j - c(i, j)) s_j / 2^(l'_i),
// c the log2-domain cost of that axis.  The Gaussian kernel factorises over the axes, so after one pass per axis l is
// the log2-sum of the full grid softmin and s the full conditional mean sum_j w_ij V_j / sum_j w_ij; every
// intermediate s is a convex combination of V, bounded by max |V| whatever the signs.  A slab of up to kGridApplyKS
// channels per launch: the pair's one MUFU.EX2 feeds the denominator and one FMA per channel; all of them share the
// lazy max and its 2^64 rebase of grid_pass_kernel.  Inputs (l and the slab's channels of all TW lines) are staged in
// shared memory; outputs are stored straight from registers, which keeps the tile at (1 + K) N (TW + 1) floats and
// lets the pass run in place (the CTA has read all of its lines before any store).
constexpr int kGridApplyKS = 4;

struct GridApplyArgs {
  const float* h_a;  // first pass: l = log2(e) (h_a + h_scale_b h_b); later passes read `ell` in place
  const float* h_b;  // nullable
  const float* v;    // first pass: channel k of the slab at v[k * vstride + pixel]; later passes read `s` in place
  float* ell;
  float* s;
  float h_scale_b, xscale;
  int N, nk, first;
  int64_t outer, inner, vstride;
};

template <int TW, bool PERIODIC>
__global__ void __launch_bounds__(kGridWarps * 32) grid_apply_kernel(GridApplyArgs A) {
  constexpr int RS = TW + 1, NSUB = 32 / TW, KS = kGridApplyKS;
  extern __shared__ float smem_f[];
  const int N = A.N, nk = A.nk;
  float* tile = smem_f;          // [N][RS] log2 weights
  float* vtile = smem_f + N * RS;  // [nk][N][RS] means
  const int lane = (threadIdx.x & 31) % TW, warp = (threadIdx.x >> 5) * NSUB + (threadIdx.x & 31) / TW;
  const bool last_axis = (A.inner == 1);
  int64_t o, w0;
  int nw;
  if (last_axis) {
    o = (int64_t)blockIdx.x * TW;
    w0 = 0;
    nw = (int)min((int64_t)TW, A.outer - o);
  } else {
    const int64_t tiles_in = (A.inner + TW - 1) / TW;
    o = blockIdx.x / tiles_in;
    w0 = (blockIdx.x % tiles_in) * TW;
    nw = (int)min((int64_t)TW, A.inner - w0);
  }
  auto index = [&](int j, int w) -> int64_t {
    return last_axis ? ((o + w) * N + j) : ((o * N + j) * A.inner + w0 + w);
  };

  for (int idx = threadIdx.x; idx < N * TW; idx += blockDim.x) {
    const int j = last_axis ? idx % N : idx / TW, w = last_axis ? idx / N : idx % TW;
    float l = -INFINITY;
    if (w < nw) {
      const int64_t gi = index(j, w);
      if (A.first) {
        l = A.h_a[gi];
        if (A.h_b) l = fmaf(A.h_scale_b, A.h_b[gi], l);
        l *= kLog2e;
      } else {
        l = A.ell[gi];
      }
    }
    tile[j * RS + w] = l;
    const float* src = A.first ? A.v : A.s;
    for (int k = 0; k < nk; ++k) vtile[(k * N + j) * RS + w] = (w < nw) ? src[k * A.vstride + index(j, w)] : 0.f;
  }
  __syncthreads();

  const float kq = -A.xscale * A.xscale, Nf = (float)N;
  const int per_warp = (N + kGridWarps * NSUB - 1) / (kGridWarps * NSUB);
  const int i_end = min(N, (warp + 1) * per_warp);
  int kk[KS];  // channel tile read for slab slot k (the last live one for the dead slots: their sums are discarded)
#pragma unroll
  for (int k = 0; k < KS; ++k) kk[k] = min(k, nk - 1) * N * RS;
  for (int ib = warp * per_warp; ib < i_end; ib += kGridR) {
    float m[kGridR], den[kGridR], num[kGridR][KS];
#pragma unroll
    for (int r = 0; r < kGridR; ++r) {
      m[r] = (ib + r < N) ? fmaxf(tile[(ib + r) * RS + lane], kNegBig) : kNegBig;  // the j = i term, as above
      den[r] = 0.f;
#pragma unroll
      for (int k = 0; k < KS; ++k) num[r][k] = 0.f;
    }
    for (int j0 = 0; j0 < N; j0 += 8) {
      float a[8], v[8][KS];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const bool in = (j0 + c < N);
        a[c] = in ? tile[(j0 + c) * RS + lane] : -INFINITY;
#pragma unroll
        for (int k = 0; k < KS; ++k) v[c][k] = in ? vtile[kk[k] + (j0 + c) * RS + lane] : 0.f;
      }
      float W[15];  // -c(i, j) for the offsets n = (ib - j0) + t, t = r - c in [-7, 7]
#pragma unroll
      for (int t = -7; t <= 7; ++t) {
        const float n = grid_offset<PERIODIC>((float)(ib - j0 + t), Nf);
        W[t + 7] = (n * n) * kq;
      }
#pragma unroll
      for (int r = 0; r < kGridR; ++r) {
        float e[8], cs = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          e[c] = ex2_approx((a[c] + W[r - c + 7]) - m[r]);
          cs += e[c];
        }
        if (!(cs <= 1.8446744e19f)) {
          // outdated max: rebase the denominator and the numerators on this chunk's max and redo it
          float cm = -INFINITY;
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            e[c] = a[c] + W[r - c + 7];
            cm = fmaxf(cm, e[c]);
          }
          cs = 0.f;
          if (cm > kNegBig) {
            const float sc = ex2_approx(m[r] - cm);
            den[r] *= sc;
#pragma unroll
            for (int k = 0; k < KS; ++k) num[r][k] *= sc;
            m[r] = cm;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              e[c] = ex2_approx(e[c] - cm);
              cs += e[c];
            }
          } else {
#pragma unroll
            for (int c = 0; c < 8; ++c) e[c] = 0.f;  // every input of the chunk is -inf
          }
        }
        den[r] += cs;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
#pragma unroll
          for (int k = 0; k < KS; ++k) num[r][k] = fmaf(e[c], v[c][k], num[r][k]);
        }
      }
    }
    if (lane < nw) {
#pragma unroll
      for (int r = 0; r < kGridR; ++r) {
        const int i = ib + r;
        if (i < i_end) {
          const int64_t gi = index(i, lane);
          int ex = 0;
          const float f = frexpf(den[r], &ex);
          const bool live = den[r] > 0.f;
          A.ell[gi] = live ? (m[r] + (float)ex) + log2f(f) : -INFINITY;
#pragma unroll
          for (int k = 0; k < KS; ++k)
            if (k < nk) A.s[k * A.vstride + gi] = live ? num[r][k] / den[r] : 0.f;
        }
      }
    }
  }
}

// ---- host: per-axis geometry --------------------------------------------------------------------------------------
// sides[d] in 1..1024, pitch[d] > 0 (finite), periodic[d] (nullable: no periodic axis), d < dim in 1..3; fills the
// element count of the whole batch.
static bool grid_geometry_ok(int64_t batch, int32_t dim, const int32_t* sides, const float* pitch, float eps,
                             int64_t* total) {
  if (batch <= 0 || dim < 1 || dim > 3 || !sides || !pitch || !(eps > 0.f) || !(eps < INFINITY)) return false;
  *total = batch;
  for (int d = 0; d < dim; ++d) {
    if (sides[d] < 1 || sides[d] > 1024 || !(pitch[d] > 0.f) || !(pitch[d] < INFINITY)) return false;
    *total *= sides[d];
  }
  return true;
}

static bool overlaps(const void* p, int64_t p_bytes, const void* q, int64_t q_bytes) {
  if (!p || !q) return false;
  const uintptr_t a = (uintptr_t)p, b = (uintptr_t)q;
  return a < b + (uintptr_t)q_bytes && b < a + (uintptr_t)p_bytes;
}

// The view [outer][N_axis][inner] of a (batch, sides...) tensor and the CTA count of a pass over it with TW lines.
struct GridPass {
  int32_t N;
  int64_t outer, inner, blocks;
};
static GridPass grid_pass_shape(int64_t total, int32_t dim, const int32_t* sides, int axis, int tw) {
  GridPass g;
  g.N = sides[axis];
  g.inner = 1;
  for (int d = axis + 1; d < dim; ++d) g.inner *= sides[d];
  g.outer = total / ((int64_t)g.N * g.inner);
  g.blocks = (g.inner == 1) ? ceil_div64(g.outer, tw) : g.outer * ceil_div64(g.inner, tw);
  return g;
}

}  // namespace b200ot

using namespace b200ot;

extern "C" {

B200OT_API int b200ot_softmin_grid(const float* h_a, const float* h_b, float h_scale_b, const float* out_old,
                                   float alpha_old, float beta, float* out, int64_t batch, int32_t N, int32_t dim,
                                   int32_t p, float eps, void* stream) {
  if (!h_a || !out || batch <= 0 || N <= 0 || N > 1024 || dim < 1 || dim > 3 || (p != 1 && p != 2) || !(eps > 0.f))
    return B200OT_EINVAL;
  if (out == h_a || out == h_b || (out_old && out == out_old)) return B200OT_EINVAL;  // passes run in place on `out`
  cudaStream_t st = (cudaStream_t)stream;
  int64_t total = batch;
  for (int d = 0; d < dim; ++d) total *= N;
  // pixel coordinates x = arange(N)/N, scaled so that the log2-domain exponent is in - (X_i - X_j)^2  (p = 2)
  // or in - |X_i - X_j|  (p = 1)                                                          (utils.py:235-242)
  const float xscale = (p == 2 ? sqrtf(kLog2e / (2.0f * eps)) : kLog2e / eps) / (float)N;
  const int tw = ((size_t)2 * N * (kGridTW + 1) * sizeof(float) <= 227 * 1024) ? kGridTW : 16;
  const size_t smem = (size_t)2 * N * (tw + 1) * sizeof(float);
  auto kern = (tw == kGridTW) ? ((p == 2) ? grid_pass_kernel<2, kGridTW, false> : grid_pass_kernel<1, kGridTW, false>)
                              : ((p == 2) ? grid_pass_kernel<2, 16, false> : grid_pass_kernel<1, 16, false>);
  B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // pass order of the reference: last axis first, then the others (the passes commute mathematically)
  for (int k = 0; k < dim; ++k) {
    const int axis = dim - 1 - k;  // 0 .. dim-1 within the (N, .., N) block
    GridPassArgs a;
    a.h_a = h_a;
    a.h_b = h_b;
    a.out_old = out_old;
    a.out = out;
    a.h_scale_b = h_scale_b;
    a.in_scale = kLog2e;
    a.alpha_old = alpha_old;
    a.beta = beta;
    a.out_scale = -eps * kLn2;
    a.xscale = xscale;
    a.N = N;
    a.first = (k == 0);
    a.last = (k == dim - 1);
    int64_t inner = 1;
    for (int d = axis + 1; d < dim; ++d) inner *= N;
    a.inner = inner;
    a.outer = total / ((int64_t)N * inner);
    const int64_t blocks = (inner == 1) ? ceil_div64(a.outer, tw) : a.outer * ceil_div64(inner, tw);
    kern<<<(unsigned)blocks, kGridWarps * 32, smem, st>>>(a);
    B200OT_CUDA_TRY(cudaGetLastError());
  }
  return B200OT_OK;
}

B200OT_API int b200ot_softmin_grid_axes(const float* h_a, const float* h_b, float h_scale_b, const float* out_old,
                                        float alpha_old, float beta, float* out, int64_t batch, int32_t dim,
                                        const int32_t* sides, const float* pitch, const int32_t* periodic, float eps,
                                        void* stream) {
  int64_t total = 0;
  if (!h_a || !out || !grid_geometry_ok(batch, dim, sides, pitch, eps, &total)) return B200OT_EINVAL;
  const int64_t bytes = total * (int64_t)sizeof(float);
  if (overlaps(out, bytes, h_a, bytes) || overlaps(out, bytes, h_b, bytes) || overlaps(out, bytes, out_old, bytes))
    return B200OT_EINVAL;  // passes run in place on `out`
  cudaStream_t st = (cudaStream_t)stream;
  const float xs = sqrtf(kLog2e / (2.0f * eps));  // log2-domain exponent - (xs h n)^2 for an offset of n pixels
  for (int k = 0; k < dim; ++k) {
    const int axis = dim - 1 - k;  // last axis first, as b200ot_softmin_grid
    const int N = sides[axis];
    const int tw = ((size_t)2 * N * (kGridTW + 1) * sizeof(float) <= 227 * 1024) ? kGridTW : 16;
    const size_t smem = (size_t)2 * N * (tw + 1) * sizeof(float);
    const bool per = periodic && periodic[axis];
    auto kern = (tw == kGridTW) ? (per ? grid_pass_kernel<2, kGridTW, true> : grid_pass_kernel<2, kGridTW, false>)
                                : (per ? grid_pass_kernel<2, 16, true> : grid_pass_kernel<2, 16, false>);
    B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const GridPass g = grid_pass_shape(total, dim, sides, axis, tw);
    GridPassArgs a;
    a.h_a = h_a;
    a.h_b = h_b;
    a.out_old = out_old;
    a.out = out;
    a.h_scale_b = h_scale_b;
    a.in_scale = kLog2e;
    a.alpha_old = alpha_old;
    a.beta = beta;
    a.out_scale = -eps * kLn2;
    a.xscale = xs * pitch[axis];
    a.N = N;
    a.first = (k == 0);
    a.last = (k == dim - 1);
    a.outer = g.outer;
    a.inner = g.inner;
    kern<<<(unsigned)g.blocks, kGridWarps * 32, smem, st>>>(a);
    B200OT_CUDA_TRY(cudaGetLastError());
  }
  return B200OT_OK;
}

B200OT_API int b200ot_grid_plan_apply(const float* h_a, const float* h_b, float h_scale_b, const float* v, float* ell,
                                      float* s, int64_t batch, int32_t K, int32_t dim, const int32_t* sides,
                                      const float* pitch, const int32_t* periodic, float eps, void* stream) {
  int64_t total = 0;
  if (!h_a || !v || !ell || !s || K <= 0 || !grid_geometry_ok(batch, dim, sides, pitch, eps, &total))
    return B200OT_EINVAL;
  const int64_t bytes = total * (int64_t)sizeof(float), vbytes = bytes * K;
  for (const void* in : {(const void*)h_a, (const void*)h_b}) {
    if (overlaps(ell, bytes, in, bytes) || overlaps(s, vbytes, in, bytes)) return B200OT_EINVAL;
  }
  if (overlaps(ell, bytes, v, vbytes) || overlaps(s, vbytes, v, vbytes) || overlaps(ell, bytes, s, vbytes))
    return B200OT_EINVAL;  // passes run in place on `ell` and `s`
  cudaStream_t st = (cudaStream_t)stream;
  const float xs = sqrtf(kLog2e / (2.0f * eps));
  // one chain of `dim` passes per slab: every chain recomputes the same l from h (bit for bit), so l needs no copy
  for (int32_t k0 = 0; k0 < K; k0 += kGridApplyKS) {
    const int nk = min(kGridApplyKS, K - k0);
    for (int k = 0; k < dim; ++k) {
      const int axis = dim - 1 - k;
      const int N = sides[axis];
      auto bytes_for = [&](int tw) { return (size_t)(1 + nk) * N * (tw + 1) * sizeof(float); };
      const int tw = bytes_for(32) <= 227 * 1024 ? 32 : bytes_for(16) <= 227 * 1024 ? 16 : 8;
      const size_t smem = bytes_for(tw);
      const bool per = periodic && periodic[axis];
      auto kern = (tw == 32) ? (per ? grid_apply_kernel<32, true> : grid_apply_kernel<32, false>)
                  : (tw == 16) ? (per ? grid_apply_kernel<16, true> : grid_apply_kernel<16, false>)
                               : (per ? grid_apply_kernel<8, true> : grid_apply_kernel<8, false>);
      B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      const GridPass g = grid_pass_shape(total, dim, sides, axis, tw);
      GridApplyArgs a;
      a.h_a = h_a;
      a.h_b = h_b;
      a.v = v + k0 * total;
      a.ell = ell;
      a.s = s + k0 * total;
      a.h_scale_b = h_scale_b;
      a.xscale = xs * pitch[axis];
      a.N = N;
      a.nk = nk;
      a.first = (k == 0);
      a.outer = g.outer;
      a.inner = g.inner;
      a.vstride = total;
      kern<<<(unsigned)g.blocks, kGridWarps * 32, smem, st>>>(a);
      B200OT_CUDA_TRY(cudaGetLastError());
    }
  }
  return B200OT_OK;
}

}  // extern "C"
