// b200ot — the tensor-core (wgmma) host path of every operator: which path serves a shape, the plans, the packs, one
// pass per operator and its finalize, and the C entries that only the tensor cores serve (the batched, p = 1, wide and
// block-sparse families).  Kernels: tcconv.cuh (forward), tcbwd.cuh (row gradients), tcwide.cuh (above D = 64,
// instantiated in b200ot_wide.cu), tcapply.cuh (the plan applied to a value matrix).
#include "b200ot.h"
#include "conv_kind.cuh"
#include "host_util.cuh"
#include "plan.cuh"
#include "tcapply.cuh"
#include "tcbwd.cuh"
#include "tcconv.cuh"
#include "tcwide.cuh"

#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

namespace b200ot {

// A launch group: `ctas` x n_split x slices CTAs over a_tiles row images and b_tiles column images, then the partials
// and a misc block in the scratch
struct TcPlan {
  int kp, nstage, n_split, tiles_per_split, slices;
  int rtpe, ctpe;  // row / column tiles per batch element (0 for a block-sparse problem)
  int64_t a_tiles, b_tiles, ctas, smem;
  int64_t off_b, off_part, off_misc, total;
};

// Which path serves an operator.  Above B200OT_MAX_D the tensor-core kernels are the only ones.  At or below it both
// exist: the CUDA-core kernels are FMA-pipe bound from D = 5 up while the tensor-core kernels run the zero-padded
// dk = 16 problem at the same rate whatever D.  Measured on an H100 80GB HBM3 (SXM, 400 W power limit) at N = M = 4e5
// (tools/ab_tc_route.py part A; CUDA-core -> tensor-core, 1e12 pairs/s):
//   softmin forward   D = 5: 2.38 -> 1.96   D = 6: 2.02 -> 1.95   D = 7: 1.85 -> 1.94   D = 8: 1.54 -> 1.87
//   gaussian forward  D = 4: 2.42 -> 2.39   D = 5: 1.77 -> 2.42   D = 6: 1.60 -> 2.45   D = 8: 1.31 -> 2.37
//   row gradients     D = 6: 1.33 / 1.22 -> 1.69 / 1.52 (softmin / gaussian); D = 8: 1.08 / 0.97 -> 1.63 / 1.49
// (at N = M = 1e5 and 3e4 the softmin forward already breaks even at D = 6, the others switch where they do at 4e5).  The
// forward operators switch at D = 7 (softmin) and D = 5 (gaussian).  The row gradients stay on the CUDA cores for every
// D <= 8 although the tensor cores are faster from D = 6: the fp16 image of P that GEMM 2 consumes costs accuracy at
// small blur in low dimension (relative difference between the two paths' gradients at eps = 1e-4 / blur = .05 in the
// same run: up to 3e-3 at D = 4, 4e-4 at D = 6..8, against ~1e-5 for the forward operators).  Problems below 8e8 pairs
// keep the CUDA-core kernels.  $B200OT_TC_MIN_D ("d" or "softmin_fwd,softmin_bwd,conv_fwd,conv_bwd")
// and $B200OT_TC_MIN_PAIRS override the defaults for A/B timing and for the parity tests of both routes — read on every
// call, never set by the bench.
static const int kTcMinDimDefault[4] = {7, 9, 5, 9};
static const double kTcMinPairsDefault = 8.0e8;

bool tc_routed(int op, int D, int64_t N, int64_t M) {
  if (!tc_capable_dim(D)) return false;
  if (D > B200OT_MAX_D) return true;
  int min_dim[4] = {kTcMinDimDefault[0], kTcMinDimDefault[1], kTcMinDimDefault[2], kTcMinDimDefault[3]};
  double min_pairs = kTcMinPairsDefault;
  if (const char* e = getenv("B200OT_TC_MIN_D")) {
    int v[4];
    const int n = sscanf(e, "%d,%d,%d,%d", &v[0], &v[1], &v[2], &v[3]);
    if (n == 1) {
      for (int k = 0; k < 4; ++k) min_dim[k] = v[0];
    } else if (n == 4) {
      for (int k = 0; k < 4; ++k) min_dim[k] = v[k];
    }
  }
  if (const char* e = getenv("B200OT_TC_MIN_PAIRS")) {
    const double v = atof(e);
    if (v >= 0.0) min_pairs = v;
  }
  return D >= min_dim[op] && (double)N * (double)M >= min_pairs;
}

bool tc_any_routed(int D, int64_t N, int64_t M) {
  for (int op = 0; op < 4; ++op)
    if (tc_routed(op, D, N, M)) return true;
  return false;
}

// The plan of a launch group: `ctas` row CTAs, each reading up to `tiles` (>= 1) column tiles.  The split count is
// chosen for the whole grid and cuts those tiles.  Behind the images: the partials of `rows` rows ((m, s) pairs forward, D+1
// sums per row backward, D+2 for the p = 1 softmin: `head` sums ahead of the D), then a misc block of misc_bytes.
// Above D = 64 the K-slab ring of tcwide.cuh, whose row gradients run `slices` CTAs per row tile and split.
static TcPlan make_tc_plan(int D, bool bwd, int64_t a_tiles, int64_t b_tiles, int64_t ctas, int64_t tiles, int64_t rows,
                           int64_t misc_bytes, int head = 1, int slices = 1) {
  TcPlan p;
  p.kp = tc_kp(D);
  p.slices = slices;
  p.rtpe = p.ctpe = 0;
  p.a_tiles = a_tiles;
  p.b_tiles = b_tiles;
  p.ctas = ctas;
  const int64_t b_bytes = tc_b_img_bytes(p.kp, kTcBN);
  if (D > 64) {
    // row tail, column tails and slab ring (tcwide.cuh): as many stages as fit, whatever D
    int ns = kTcMaxStage;
    while (ns > 0 && tc_wide_smem(ns) > 227 * 1024) --ns;
    p.nstage = ns;
    p.smem = tc_wide_smem(ns);
  } else {
    const int64_t bar_bytes = 256;  // mbarriers behind the column ring
    // the CTA's row image stays in shared memory; the rest of the 227 KB a block may use holds the column ring
    const int64_t avail = 227 * 1024 - bar_bytes - tc_a_span(p.kp);
    int64_t ns = avail / b_bytes;
    p.nstage = (int)(ns > kTcMaxStage ? kTcMaxStage : ns);
    p.smem = tc_a_span(p.kp) + p.nstage * b_bytes + bar_bytes;
  }
  int64_t want = ceil_div64((int64_t)num_sms() * 4, ctas * slices);
  const int forced = forced_splits();  // test hook (plan.cuh)
  if (forced > 0) want = forced;
  if (want < 1) want = 1;
  if (want > 64) want = 64;
  if (want > tiles) want = tiles;
  p.tiles_per_split = (int)ceil_div64(tiles, want);
  p.n_split = (int)ceil_div64(tiles, p.tiles_per_split);
  p.off_b = round_up64(a_tiles * tc_a_img_bytes(p.kp), 256);
  p.off_part = p.off_b + round_up64(b_tiles * b_bytes, 256);
  p.off_misc = p.off_part + round_up64((int64_t)p.n_split * (bwd ? rows * (D + head) : kTcParts * rows * 2) * 4, 256);
  p.total = p.off_misc + round_up64(misc_bytes, 256);
  return p;
}

// B problems of N rows x M columns side by side (B = 1: one problem), each element padded to whole tiles on its own
// (tc_pack_kernel).  The splits cut each element's ctpe column tiles, so a CTA never reads another element's columns.
// Above D = 64 the row gradients run one slice per K slab.  Misc block: [0] the energy coordinate maximum, [1 + b]
// max|w| of element b.
static TcPlan make_tc_plan(int64_t N, int64_t M, int D, bool bwd, int64_t B = 1, int head = 1) {
  const int rtpe = (int)ceil_div64(N, kTcM), ctpe = (int)ceil_div64(M, kTcBN);
  TcPlan p = make_tc_plan(D, bwd, B * rtpe, B * ctpe, B * rtpe, ctpe, B * N, (B + 1) * 4, head,
                          bwd && D > 64 ? tc_wide_slabs(D) : 1);
  p.rtpe = rtpe;
  p.ctpe = ctpe;
  return p;
}

// The scratch of B problems: the larger of the forward plan and the row-gradient plan, whose rows keep D + head sums
// (head = 2: the p = 1 softmin).  Forward and row-gradient launches split the columns differently.
static int64_t tc_scratch_bytes(int64_t N, int64_t M, int D, int64_t B, int head) {
  return std::max(make_tc_plan(N, M, D, false, B).total, make_tc_plan(N, M, D, true, B, head).total);
}

int64_t tc_scratch_bytes(int64_t N, int64_t M, int D) { return tc_scratch_bytes(N, M, D, 1, 1); }

// A block-sparse problem (8 < D <= 64, p = 2; b200ot_*_blocks): every row cluster and every column cluster is padded
// to whole kTcBlocksTile-point tiles on its own, slot -> point through row_src / col_src (-1: padding), one segment per
// row tile.  blocks_check fills max_tiles (the longest segment in column tiles) and n_pieces (the pieces the segments
// reference).
constexpr int kTcBlocksTile = 128;  // segment height and column alignment: the kernels' tile
static_assert(kTcBlocksTile == kTcM && kTcBlocksTile == kTcBN, "segments are one row tile, pieces whole column tiles");
struct TcBlocks {
  const int *row_src, *col_src;
  int64_t n_row_slots, n_col_slots;
  const b200ot_segment* seg;
  int64_t n_seg;
  const b200ot_piece* pieces;
  int64_t n_pieces = 0;
  int max_tiles = 0;
};

// The plan of one block-sparse problem: a CTA per segment, images of n_row_slots / n_col_slots points, segments cut
// into splits from the longest one.  Misc block: the segment descriptors, then the pieces.
static int64_t tc_blocks_seg_bytes(int64_t n_seg) { return round_up64(n_seg * 16, 256); }
static TcPlan make_tc_blocks_plan(int64_t N, int D, bool bwd, const TcBlocks& b) {
  return make_tc_plan(D, bwd, b.n_row_slots / kTcM, b.n_col_slots / kTcBN, b.n_seg, std::max(b.max_tiles, 1), N,
                      tc_blocks_seg_bytes(b.n_seg) + std::max<int64_t>(b.n_pieces, 1) * 8);
}

static int64_t tc_blocks_scratch_bytes(int64_t N, int D, const TcBlocks& b) {
  return std::max(make_tc_blocks_plan(N, D, false, b).total, make_tc_blocks_plan(N, D, true, b).total);
}

// What the images of a launch group hold (tc_pack_kernel): the row cloud x and the column cloud y, centred at `center`
// and multiplied by `scale`; B elements of N rows / M columns, or N / M block-sparse slots gathered through row_src /
// col_src.  Besides the coordinates: the column weights w, the softmin's column terms h_a + h_scale_b h_b and the
// softmin row gradient's row term lse2.  l1_c = log2e / eps > 0: the p = 1 softmin's layout (tc_pack_kernel's l1).
struct TcOperands {
  const float *x, *y, *center;
  float scale;
  int64_t N, M;
  int D;
  int64_t B = 1;
  const float *w = nullptr, *h_a = nullptr, *h_b = nullptr;
  float h_scale_b = 0.f;
  const float* lse2 = nullptr;
  const int *row_src = nullptr, *col_src = nullptr;
  float l1_c = 0.f;
};

// max_j |w_j| into *out (zero-initialised by the caller); bit order of non-negative floats = integer order.
// gridDim.y > 1: one maximum per batch element of n weights, out[blockIdx.y]
__global__ void absmax_kernel(const float* __restrict__ w, int64_t n, float* __restrict__ out) {
  w += (int64_t)blockIdx.y * n;
  out += blockIdx.y;
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(w[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f && !(m != m)) atomicMax(reinterpret_cast<unsigned int*>(out), __float_as_uint(m));
}

// max_k |pts[i, k] - center[k]| over the rows of a (na x D) and b (nb x D) into *out (zero-initialised by the caller)
__global__ void coord_absmax_kernel(const float* __restrict__ a, int64_t na, const float* __restrict__ b, int64_t nb,
                                    int D, const float* __restrict__ center, float* __restrict__ out) {
  float m = 0.f;
  const int64_t ta = na * D, tot = ta + nb * D;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (int64_t)gridDim.x * blockDim.x) {
    const float v = e < ta ? a[e] : b[e - ta];
    m = fmaxf(m, fabsf(v - (center ? center[e % D] : 0.f)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f && !(m != m)) atomicMax(reinterpret_cast<unsigned int*>(out), __float_as_uint(m));
}

// Packs both images of plan p.  Asked for through a non-null out pointer, it first computes into the misc block:
//   * w_absmax (row gradients): P = w_j e_ij feeds an fp16 GEMM, so the weights are normalised to max|w| = kTcPScale
//     (undone by the finalize kernel), one maximum per batch element, so that a heavy element cannot push a light
//     one's P into fp16's subnormal range;
//   * coord_absmax (energy): the largest centred coordinate of both clouds (of every batch element: one scale for the
//     whole batch, a power of two that the finalize undoes exactly), from which every kernel of the pass derives the
//     same power-of-two coordinate scale (tc_energy_coord_scale).
static int tc_pack(const TcPlan& p, unsigned char* base, const TcOperands& o, cudaStream_t st,
                   const float** w_absmax = nullptr, const float** coord_absmax = nullptr) {
  float* misc = reinterpret_cast<float*>(base + p.off_misc);
  const float* cmax = nullptr;
  if (coord_absmax) {
    B200OT_CUDA_TRY(cudaMemsetAsync(misc, 0, sizeof(float), st));
    const int64_t n = o.B * o.N, m = o.B * o.M;
    coord_absmax_kernel<<<(unsigned)std::min<int64_t>(ceil_div64((n + m) * o.D, 256), 1024), 256, 0, st>>>(
        o.x, n, o.y, m, o.D, o.center, misc);
    B200OT_CUDA_TRY(cudaGetLastError());
    cmax = *coord_absmax = misc;
  }
  const float* wmax = nullptr;
  if (w_absmax) {
    if (o.w != nullptr) {
      B200OT_CUDA_TRY(cudaMemsetAsync(misc + 1, 0, o.B * sizeof(float), st));
      const dim3 g((unsigned)std::min<int64_t>(ceil_div64(o.M, 256), 1024), (unsigned)o.B);
      absmax_kernel<<<g, 256, 0, st>>>(o.w, o.M, misc + 1);
      B200OT_CUDA_TRY(cudaGetLastError());
      wmax = misc + 1;
    }
    *w_absmax = wmax;
  }
  const int threads = 128;
  tc_pack_kernel<<<(unsigned)ceil_div64(p.a_tiles * kTcM, threads), threads, 0, st>>>(
      o.x, nullptr, nullptr, nullptr, 0.f, o.l1_c, o.center, o.scale, o.N, o.D, p.kp, kTcM, 0, base, o.lse2, nullptr, cmax,
      o.B, o.row_src, o.l1_c > 0.f);
  B200OT_CUDA_TRY(cudaGetLastError());
  tc_pack_kernel<<<(unsigned)ceil_div64(p.b_tiles * kTcBN, threads), threads, 0, st>>>(
      o.y, o.w, o.h_a, o.h_b, o.h_scale_b, kLog2e, o.center, o.scale, o.M, o.D, p.kp, kTcBN, 1, base + p.off_b, nullptr,
      wmax, cmax, o.B, o.col_src, o.l1_c > 0.f);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

// tc_reduce_kernel<FWD> (forward) or tc_bwd_kernel<BWD> at the padded dimension of D (row gradients)
template <int FWD, int BWD, bool BATCH, bool BLOCKS = false>
static TcKernel tc_kernel_of(bool bwd, int D) {
  if (!bwd) return tc_reduce_kernel<FWD, BATCH, BLOCKS>;
  switch (tc_dk(D)) {
    case 16: return tc_bwd_kernel<BWD, 16, BATCH, BLOCKS>;
    case 32: return tc_bwd_kernel<BWD, 32, BATCH, BLOCKS>;
    case 48: return tc_bwd_kernel<BWD, 48, BATCH, BLOCKS>;
    default: return tc_bwd_kernel<BWD, 64, BATCH, BLOCKS>;
  }
}

// How the rows and columns of a pass are laid out: one problem, a batch of B problems side by side (x (B,N,D), y
// (B,M,D), element b of the rows reduced over element b of the columns only), or one block-sparse problem.  The p = 1
// softmin runs the batch kernels only, B = 1 included.
enum class TcLayout { kOne, kBatch, kBlocks };

// The kernel of `mode` (the MODE of tc_reduce_kernel forward, of tc_bwd_kernel for the row gradients: 0 / 2 gaussian
// conv, 1 / 3 softmin p = 2, 4 laplacian, 5 energy, 6 / 7 softmin p = 1) for D and the layout; null for a pair that
// has none.  Above D = 64 the K-slab kernels, whatever the layout.
static TcKernel tc_kernel(int mode, bool bwd, int D, TcLayout layout) {
  if (D > 64) return tc_wide_kernel(mode, bwd);
  const bool one = layout == TcLayout::kOne, batch = layout == TcLayout::kBatch;
  switch (mode) {
    case 0:
    case 2: return one ? tc_kernel_of<0, 2, false>(bwd, D) : batch ? tc_kernel_of<0, 2, true>(bwd, D) : nullptr;
    case 1:
    case 3:
      return one     ? tc_kernel_of<1, 3, false>(bwd, D)
             : batch ? tc_kernel_of<1, 3, true>(bwd, D)
                     : tc_kernel_of<1, 3, false, true>(bwd, D);
    case 4: return one ? tc_kernel_of<4, 4, false>(bwd, D) : batch ? tc_kernel_of<4, 4, true>(bwd, D) : nullptr;
    case 5: return one ? tc_kernel_of<5, 5, false>(bwd, D) : batch ? tc_kernel_of<5, 5, true>(bwd, D) : nullptr;
    default: return batch ? tc_kernel_of<6, 7, true>(bwd, D) : nullptr;
  }
}

// What a pass leaves for its finalize: n_part sets of partials inside the scratch ((m, s) pairs forward, D + head sums
// per row for the row gradients), and the maxima the finalize undoes (null when the pass has none)
struct TcPass {
  float* part = nullptr;
  int n_part = 0;
  const float* w_absmax = nullptr;
  const float* coord_absmax = nullptr;
};

// One tensor-core pass of `mode` (tc_kernel) over B elements of o.N rows / o.M columns, or over the block-sparse
// problem `blocks` of o.N rows: plan, images, kernel and launch.  The row gradients normalise the weights (when the
// operator has any) and the energy's coordinates (modes 5, 6, 7) take a power-of-two scale from their maximum
// (tc_pack); the finalize undoes both.
static int tc_pass(int mode, bool bwd, TcLayout layout, TcOperands o, float clampq, const TcBlocks* blocks,
                   void* scratch, cudaStream_t st, TcPass* r) {
  const TcPlan p = blocks ? make_tc_blocks_plan(o.N, o.D, bwd, *blocks)
                          : make_tc_plan(o.N, o.M, o.D, bwd, o.B, mode == 7 ? 2 : 1);
  const TcKernel kern = tc_kernel(mode, bwd, o.D, layout);
  if (p.nstage < 1 || kern == nullptr) return B200OT_EINVAL;
  // K_xx / K_yy and the p = 1 xx / yy: the diagonal exponent is exact (tcconv.cuh)
  const int self_mode = (mode != 1 && mode != 3 && o.x == o.y && o.N == o.M) ? 1 : 0;
  const int64_t rows = o.B * o.N, n_local = blocks ? 0 : o.N;
  unsigned char* base = reinterpret_cast<unsigned char*>(scratch);
  const int4* seg = nullptr;
  const int2* pieces = nullptr;
  if (blocks) {
    // the host descriptors travel in the misc block
    int4* d_seg = reinterpret_cast<int4*>(base + p.off_misc);
    int2* d_pieces = reinterpret_cast<int2*>(base + p.off_misc + tc_blocks_seg_bytes(blocks->n_seg));
    B200OT_CUDA_TRY(cudaMemcpyAsync(d_seg, blocks->seg, blocks->n_seg * 16, cudaMemcpyHostToDevice, st));
    if (blocks->n_pieces > 0)
      B200OT_CUDA_TRY(cudaMemcpyAsync(d_pieces, blocks->pieces, blocks->n_pieces * 8, cudaMemcpyHostToDevice, st));
    seg = d_seg;
    pieces = d_pieces;
    o.N = blocks->n_row_slots;
    o.M = blocks->n_col_slots;
    o.row_src = blocks->row_src;
    o.col_src = blocks->col_src;
  }
  *r = TcPass{};
  int rc = tc_pack(p, base, o, st, bwd ? &r->w_absmax : nullptr, mode >= 5 ? &r->coord_absmax : nullptr);
  if (rc) return rc;
  B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
  const dim3 grid((unsigned)p.ctas, (unsigned)p.n_split, (unsigned)p.slices);
  kern<<<grid, kTcThreads, (size_t)p.smem, st>>>(base, base + p.off_b, reinterpret_cast<float*>(base + p.off_part),
                                                 rows, p.kp, p.ctpe, p.tiles_per_split, p.nstage, o.D, self_mode,
                                                 clampq, r->coord_absmax, p.rtpe, n_local, seg, pieces, o.row_src);
  B200OT_CUDA_TRY(cudaGetLastError());
  r->part = reinterpret_cast<float*>(base + p.off_part);
  // row gradients: G of a CTA is complete over its column split (both column halves feed one GEMM)
  r->n_part = bwd ? p.n_split : p.n_split * kTcParts;
  return B200OT_OK;
}

// A softmin on the tensor cores: B elements of N rows / M columns (TcLayout::kBlocks: B = 1, N rows, the slots in the
// TcBlocks).  p may carry B200OT_P_UNCLAMPED; lse2: the forward's, for the row gradients.
struct TcSoftmin {
  const float *x, *y, *h_a, *h_b;
  float h_scale_b;
  const float *center, *lse2;
  int64_t B, N, M;
  int D, p;
  float eps;
};

// The softmin, p = 2 (MODE 1 / 3) or p = 1 (MODE 6 / 7, on the energy's coordinates with the clamp of p)
static int softmin_pass_tc(bool bwd, TcLayout layout, const TcSoftmin& s, const TcBlocks* blocks, void* scratch,
                           cudaStream_t st, TcPass* r) {
  const bool l1 = p_exponent(s.p) == 1;
  TcOperands o{s.x, s.y, s.center, l1 ? 1.f : softmin_coord_scale(2, s.eps), s.N, s.M, s.D, s.B, nullptr, s.h_a, s.h_b,
               s.h_scale_b, s.lse2};
  if (l1) o.l1_c = kLog2e / s.eps;
  return tc_pass(l1 ? (bwd ? 7 : 6) : (bwd ? 3 : 1), bwd, layout, o, l1 ? cost_clamp(s.p) : 0.f, blocks, scratch, st,
                 r);
}

// out / lse2_out of the B N rows, as b200ot_softmin_finalize
static int softmin_fwd_tc(TcLayout layout, const TcSoftmin& s, const TcBlocks* blocks, const float* out_old,
                          float alpha_old, float beta, float* out, float* lse2_out, void* scratch, void* stream) {
  TcPass r;
  const int rc = softmin_pass_tc(false, layout, s, blocks, scratch, (cudaStream_t)stream, &r);
  if (rc) return rc;
  return b200ot_softmin_finalize(r.part, r.n_part, out_old, alpha_old, beta, out, lse2_out, s.B * s.N, s.eps, stream);
}

// p = 1 on the tensor cores: part (n_split, N, D+2) with [0] = sum P, [1] = sum Q, [2+k] = sum Q Y_k (tcbwd.cuh, MODE 7)
// -> grad_x = go (X_i sum Q - sum Q Y) / sum P, X = scale (x - center) with the pass's coordinate scale
__global__ void softmin_l1_bwd_finalize_kernel(const float* __restrict__ part, int n_split,
                                               const float* __restrict__ x, const float* __restrict__ center,
                                               const float* __restrict__ grad_out, float* __restrict__ grad_x,
                                               int64_t N, int D, const float* __restrict__ coord_absmax) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int na = D + 2;
  const float scale = tc_energy_coord_scale(*coord_absmax);
  float sp = 0.f, sq = 0.f;
  for (int s = 0; s < n_split; ++s) {
    sp += part[((int64_t)s * N + i) * na];
    sq += part[((int64_t)s * N + i) * na + 1];
  }
  const float go = sp > 0.f ? grad_out[i] / sp : 0.f;
  for (int k = 0; k < D; ++k) {
    float a = 0.f;
    for (int s = 0; s < n_split; ++s) a += part[((int64_t)s * N + i) * na + 2 + k];
    const float X = scale * (x[i * D + k] - (center ? center[k] : 0.f));
    grad_x[i * D + k] = go * (X * sq - a);
  }
}

static int softmin_bwd_x_tc(TcLayout layout, const TcSoftmin& s, const TcBlocks* blocks, const float* grad_out,
                            float* grad_x, void* scratch, cudaStream_t st) {
  TcPass r;
  const int rc = softmin_pass_tc(true, layout, s, blocks, scratch, st, &r);
  if (rc) return rc;
  // P carries kTcPScale (p = 2) or 2^k_i (p = 1), which cancel: both finalizes divide by each row's sum of P
  const int64_t rows = s.B * s.N;
  if (p_exponent(s.p) == 2)
    return softmin_bwd_finalize_tc(r.part, r.n_part, s.x, s.center, grad_out, grad_x, rows, s.D, s.eps, st);
  softmin_l1_bwd_finalize_kernel<<<(unsigned)ceil_div64(rows, 256), 256, 0, st>>>(r.part, r.n_part, s.x, s.center,
                                                                                  grad_out, grad_x, rows, s.D,
                                                                                  r.coord_absmax);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

// The kernel convolution of B elements of N rows / M columns on the tensor cores: out (forward) or grad_x (bwd) and,
// with value_out, the forward values from the same pass (gaussian only).  Every row-gradient kernel leaves the
// gaussian's sums: grad = coef (sum_j P Y_j - X_i sum_j P) with coef = 1 / (scale blur^2) for the gaussian; the
// laplacian and energy P = w k'(d) / d carries 2^-kTcNormPLog2 (tcbwd.cuh), so coef = 2^kTcNormPLog2 / blur (laplacian,
// X = x log2e / blur) or 2^kTcNormPLog2 (energy).  Arguments already validated.
static int conv_tc(bool bwd, TcLayout layout, int kind, const float* x, const float* y, const float* w,
                   const float* center, const float* grad_out, float* res, float* value_out, int64_t B, int64_t N,
                   int64_t M, int D, float blur, void* scratch, cudaStream_t st) {
  const int kb = kind_base(kind);
  // gaussian: 2^(-|X-Y|^2/2) with X = x sqrt(log2e) / blur; laplacian / energy: conv_scales' coordinates and clamp
  const ConvScales cs = conv_scales(kind, blur);
  const int mode = kb == B200OT_KERNEL_GAUSSIAN ? (bwd ? 2 : 0) : (kb == B200OT_KERNEL_LAPLACIAN ? 4 : 5);
  TcPass r;
  const int rc = tc_pass(mode, bwd, layout, {x, y, center, cs.scale, N, M, D, B, w}, cs.clampq, nullptr, scratch, st, &r);
  if (rc) return rc;
  if (!bwd) return conv_fwd_finalize(r.part, r.n_part, kind, res, B * N, r.coord_absmax, st);
  const float coef = kb == B200OT_KERNEL_GAUSSIAN
                         ? 1.0f / (cs.scale * blur * blur)
                         : (float)(1 << kTcNormPLog2) * (kb == B200OT_KERNEL_LAPLACIAN ? 1.0f / blur : 1.0f);
  // n_per = N: the finalize undoes each element's weight scale
  return conv_bwd_finalize(r.part, r.n_part, x, center, grad_out, res, B * N, D, B200OT_KERNEL_GAUSSIAN, cs.scale, coef,
                           r.w_absmax, value_out, r.coord_absmax, N, st);
}

// The plan applied to a value matrix (tcapply.cuh): the images and splits of the softmin row gradient's plan, one CTA
// per row tile and split whatever D (no D slices above 64: GEMM 2 reads the value image, not a column slab), and
// behind the images the partials (n_split, N, 1 + min(K, 64)), one slab's value image and the K column maxima of V.
// V wider than 64 columns runs in slabs of 64 (the last one padded to a multiple of 16), each a pass of its own over
// the pairs through the same images, partials and value image.  A ring stage holds, up to D = 64, a column tile and
// the slab's value image: at dk = 64 and 64 value columns 36.5 + 32 KB, two stages next to the 36 KB row image.  Above
// D = 64 it is a K slab of tcwide.cuh (64 KB) with a value slot of its own next to the column tail: at 64 value
// columns 14 KB (row tail, column tails, barriers) + 2 x (64 + 32) KB = 206 KB, where a third stage would take 302.
struct TcApplyPlan {
  TcPlan p;
  bool wide;
  int64_t off_v, off_vmax, total;
};
static int tc_apply_dkv(int K, int k0) { return tc_dk(std::min(64, K - k0)); }
static void tc_apply_stages(bool wide, int kp, int dkv, int* nstage, int64_t* smem) {
  const int64_t v_bytes = tc_value_img_bytes(dkv);
  if (wide) {
    int ns = kTcMaxStage;
    while (ns > 0 && tc_wide_smem(ns) + ns * v_bytes > 227 * 1024) --ns;
    *nstage = ns;
    *smem = tc_wide_smem(ns) + ns * v_bytes;
    return;
  }
  const int64_t bar_bytes = 256, b_bytes = tc_b_img_bytes(kp, kTcBN);
  const int64_t ns = (227 * 1024 - bar_bytes - tc_a_span(kp)) / (b_bytes + v_bytes);
  *nstage = (int)(ns > kTcMaxStage ? kTcMaxStage : ns);
  *smem = tc_a_span(kp) + *nstage * (b_bytes + v_bytes) + bar_bytes;
}
static TcApplyPlan make_tc_apply_plan(int64_t N, int64_t M, int D, int K) {
  TcApplyPlan a;
  const int64_t rtpe = ceil_div64(N, kTcM), ctpe = ceil_div64(M, kTcBN);
  a.p = make_tc_plan(D, true, rtpe, ctpe, rtpe, ctpe, N, 2 * 4);
  a.p.rtpe = (int)rtpe;
  a.p.ctpe = (int)ctpe;
  a.wide = D > 64;
  a.off_v = a.p.off_part + round_up64((int64_t)a.p.n_split * N * (1 + std::min(K, 64)) * 4, 256);
  a.off_vmax = a.off_v + round_up64(a.p.b_tiles * tc_value_img_bytes(tc_apply_dkv(K, 0)), 256);
  a.total = a.off_vmax + round_up64((int64_t)K * 4, 256);
  return a;
}

int64_t tc_plan_apply_scratch_bytes(int64_t N, int64_t M, int D, int K) { return make_tc_apply_plan(N, M, D, K).total; }

template <int DKV>
static int tc_apply_launch(const TcApplyPlan& a, unsigned char* base, int64_t N, int kv, cudaStream_t st) {
  int nstage;
  int64_t smem;
  tc_apply_stages(a.wide, a.p.kp, DKV, &nstage, &smem);
  if (nstage < 2) return B200OT_EINVAL;
  const auto kern = a.wide ? tc_wide_apply_kernel<DKV> : tc_apply_kernel<DKV>;
  B200OT_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((unsigned)a.p.ctas, (unsigned)a.p.n_split);
  kern<<<grid, kTcThreads, (size_t)smem, st>>>(base, base + a.p.off_b, base + a.off_v,
                                               reinterpret_cast<float*>(base + a.p.off_part), N, a.p.kp, a.p.ctpe,
                                               a.p.tiles_per_split, nstage, kv);
  B200OT_CUDA_TRY(cudaGetLastError());
  return B200OT_OK;
}

// out (N, K) = row_factor_i sum_j softmax_j(...) V_jk on the tensor-core path.  Arguments already validated.
int tc_plan_apply(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                  const float* center, const float* lse2, const float* v, const float* row_factor, float* out,
                  int64_t N, int64_t M, int D, int K, float eps, void* scratch, cudaStream_t st) {
  const TcApplyPlan a = make_tc_apply_plan(N, M, D, K);
  unsigned char* base = reinterpret_cast<unsigned char*>(scratch);
  int rc = tc_pack(a.p, base, {x, y, center, softmin_coord_scale(2, eps), N, M, D, 1, nullptr, h_a, h_b, h_scale_b, lse2},
                   st);
  if (rc) return rc;
  float* vmax = reinterpret_cast<float*>(base + a.off_vmax);
  B200OT_CUDA_TRY(cudaMemsetAsync(vmax, 0, (size_t)K * sizeof(float), st));
  col_absmax_kernel<<<(unsigned)std::min<int64_t>(ceil_div64(M, 8), 1024), dim3(32, 8), 0, st>>>(v, M, K, vmax);
  B200OT_CUDA_TRY(cudaGetLastError());
  float* part = reinterpret_cast<float*>(base + a.p.off_part);
  for (int k0 = 0; k0 < K; k0 += 64) {
    const int kv = std::min(64, K - k0), dkv = tc_apply_dkv(K, k0);
    const int64_t ncols = a.p.b_tiles * kTcBN;
    tc_pack_values_kernel<<<(unsigned)ceil_div64(ncols, 128), 128, 0, st>>>(v, vmax, M, K, k0, dkv, ncols,
                                                                           base + a.off_v);
    B200OT_CUDA_TRY(cudaGetLastError());
    rc = dkv == 16   ? tc_apply_launch<16>(a, base, N, kv, st)
         : dkv == 32 ? tc_apply_launch<32>(a, base, N, kv, st)
         : dkv == 48 ? tc_apply_launch<48>(a, base, N, kv, st)
                     : tc_apply_launch<64>(a, base, N, kv, st);
    if (rc) return rc;
    rc = plan_apply_finalize(part, a.p.n_split, 1 + kv, kv, k0, K, vmax, row_factor, out, N, st);
    if (rc) return rc;
  }
  return B200OT_OK;
}

// ---------------------------------------------------------------------------------------------------
// One problem, for the operator files that route it here (b200ot_softmin.cu, b200ot_softmin_bwd.cu,
// b200ot_kernel_conv.cu).  Arguments already validated.
// ---------------------------------------------------------------------------------------------------
int tc_softmin_fwd(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                   const float* center, const float* out_old, float alpha_old, float beta, float* out, float* lse2_out,
                   int64_t N, int64_t M, int D, int p, float eps, void* scratch, void* stream) {
  return softmin_fwd_tc(TcLayout::kOne, {x, y, h_a, h_b, h_scale_b, center, nullptr, 1, N, M, D, p, eps}, nullptr,
                        out_old, alpha_old, beta, out, lse2_out, scratch, stream);
}

int tc_softmin_bwd_sums(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                        const float* center, const float* lse2, int64_t N, int64_t M, int D, int p, float eps,
                        void* scratch, cudaStream_t st, float** part, int* n_part) {
  TcPass r;
  const int rc = softmin_pass_tc(true, TcLayout::kOne, {x, y, h_a, h_b, h_scale_b, center, lse2, 1, N, M, D, p, eps},
                                 nullptr, scratch, st, &r);
  *part = r.part;
  *n_part = r.n_part;
  return rc;
}

int tc_kernel_conv(bool bwd, int kind, const float* x, const float* y, const float* w, const float* center,
                   const float* grad_out, float* res, float* value_out, int64_t N, int64_t M, int D, float blur,
                   void* scratch, cudaStream_t st) {
  return conv_tc(bwd, TcLayout::kOne, kind, x, y, w, center, grad_out, res, value_out, 1, N, M, D, blur, scratch, st);
}

// ---------------------------------------------------------------------------------------------------
// The entries only the tensor cores serve come in families of B >= 1 elements side by side (TcLayout::kBatch).  A
// family is the dimensions it serves, the softmin exponent it takes and the sums ahead of the D in its row-gradient
// partials, which set its scratch: one size for every entry of the family.
//   batched  b200ot_*_batched      8 < D <= 64                   p = 2        head 1
//   p = 1    b200ot_softmin_l1_*   8 < D <= 64                   p = 1        head 2
//   wide     b200ot_wide_*         64 < D <= B200OT_MAX_D_WIDE   p = 1 or 2   head 2
// Every entry checks in one order: EINVAL (null pointers, shape, p or kind, eps or blur, ...), then EALIGN for the
// scratch, then ESCRATCH.
// ---------------------------------------------------------------------------------------------------
struct TcFamily {
  int d_lo, d_hi;  // d_lo < D <= d_hi
  int p;           // the softmin's exponent, 0: 1 or 2
  int head;
  bool takes_d(int D) const { return D > d_lo && D <= d_hi; }
  bool takes_p(int p_arg) const { return valid_p(p_arg) && (p == 0 || p_exponent(p_arg) == p); }
  bool dims(int64_t B, int64_t N, int64_t M, int D) const { return B >= 1 && N > 0 && M > 0 && takes_d(D); }
  int64_t scratch_bytes(int64_t B, int64_t N, int64_t M, int D) const {
    return dims(B, N, M, D) ? tc_scratch_bytes(N, M, D, B, head) : 0;
  }
};
constexpr TcFamily kTcBatched{B200OT_MAX_D, 64, 2, 1};
constexpr TcFamily kTcL1{B200OT_MAX_D, 64, 1, 2};
constexpr TcFamily kTcWide{64, B200OT_MAX_D_WIDE, 0, 2};

static int softmin_fwd_entry(const TcFamily& f, const float* x, const float* y, const float* h_a, const float* h_b,
                             float h_scale_b, const float* center, const float* out_old, float alpha_old, float beta,
                             float* out, float* lse2_out, int64_t B, int64_t N, int64_t M, int D, int p, float eps,
                             void* scratch, int64_t scratch_bytes, void* stream) {
  if (!x || !y || !h_a || !scratch || !f.dims(B, N, M, D) || !f.takes_p(p) || !(eps > 0.f) || (!out && !lse2_out))
    return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, f.scratch_bytes(B, N, M, D))) return rc;
  return softmin_fwd_tc(TcLayout::kBatch, {x, y, h_a, h_b, h_scale_b, center, nullptr, B, N, M, D, p, eps}, nullptr,
                        out_old, alpha_old, beta, out, lse2_out, scratch, stream);
}

static int softmin_bwd_x_entry(const TcFamily& f, const float* x, const float* y, const float* h_a, const float* h_b,
                               float h_scale_b, const float* center, const float* lse2, const float* grad_out,
                               float* grad_x, int64_t B, int64_t N, int64_t M, int D, int p, float eps, void* scratch,
                               int64_t scratch_bytes, void* stream) {
  if (!x || !y || !h_a || !lse2 || !grad_out || !grad_x || !scratch || !f.dims(B, N, M, D) || !f.takes_p(p) ||
      !(eps > 0.f))
    return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, f.scratch_bytes(B, N, M, D))) return rc;
  return softmin_bwd_x_tc(TcLayout::kBatch, {x, y, h_a, h_b, h_scale_b, center, lse2, B, N, M, D, p, eps}, nullptr,
                          grad_out, grad_x, scratch, (cudaStream_t)stream);
}

// The kernel convolution: out (kFwd), grad_x from grad_out (kBwdX), or out with the unit row gradient grad_x from one
// pass (kFwdBwdX, gaussian only)
enum class ConvMode { kFwd, kBwdX, kFwdBwdX };
static int conv_entry(const TcFamily& f, ConvMode mode, const float* x, const float* y, const float* w,
                      const float* center, const float* grad_out, float* out, float* grad_x, int64_t B, int64_t N,
                      int64_t M, int D, int kind, float blur, void* scratch, int64_t scratch_bytes, void* stream) {
  const bool bwd = mode != ConvMode::kFwd;
  if (!x || !y || !w || !scratch || (mode != ConvMode::kBwdX && !out) || (bwd && !grad_x) ||
      (mode == ConvMode::kBwdX && !grad_out) || !f.dims(B, N, M, D) || !valid_kind(kind) || !blur_ok(kind, blur) ||
      (mode == ConvMode::kFwdBwdX && kind_base(kind) != B200OT_KERNEL_GAUSSIAN))
    return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, f.scratch_bytes(B, N, M, D))) return rc;
  return conv_tc(bwd, TcLayout::kBatch, kind, x, y, w, center, grad_out, bwd ? grad_x : out, bwd ? out : nullptr, B, N,
                 M, D, blur, scratch, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------
// Block-sparse softmins (the fine phase of the two-scale Sinkhorn above D = 8, TcBlocks) in the batched family's
// dimensions and p.  The host descriptors are validated here and copied into the scratch behind the partials (tc_pass).
// ---------------------------------------------------------------------------------------------------
// The checks of both block-sparse entries before any launch, in this order: EINVAL for a null descriptor array,
// N <= 0, n_seg <= 0, D outside (8, 64], p other than 2 (| B200OT_P_UNCLAMPED) or eps <= 0; EALIGN for misaligned
// descriptor arrays or scratch; EINVAL for descriptors off the tile grid.  Fills b.max_tiles and b.n_pieces.
static int blocks_check(int64_t N, int D, int p, float eps, const void* scratch, TcBlocks& b) {
  const b200ot_segment* seg = b.seg;
  const b200ot_piece* pieces = b.pieces;
  const int64_t n_row_slots = b.n_row_slots, n_col_slots = b.n_col_slots, n_seg = b.n_seg;
  if (!seg || !pieces || N <= 0 || n_seg <= 0 || n_seg > 0x7fffffff || !kTcBatched.takes_d(D) ||
      !kTcBatched.takes_p(p) || !(eps > 0.f))
    return B200OT_EINVAL;
  if ((((uintptr_t)seg) & 15) || (((uintptr_t)pieces) & 7) || (((uintptr_t)scratch) & 15)) return B200OT_EALIGN;
  if (n_row_slots <= 0 || n_col_slots <= 0 || n_row_slots % kTcM || n_col_slots % kTcBN ||
      n_row_slots / kTcM != n_seg || n_col_slots / kTcBN > 0x7fffffff)
    return B200OT_EINVAL;
  int64_t np = 0;
  for (int64_t s = 0; s < n_seg; ++s) {
    const b200ot_segment& g = seg[s];
    if (g.row_start < 0 || g.row_start % kTcM || g.row_start >= n_row_slots || g.row_count < 1 ||
        g.row_count > kTcM || g.piece_begin < 0 || g.piece_end < g.piece_begin)
      return B200OT_EINVAL;
    np = std::max<int64_t>(np, g.piece_end);
  }
  // column tiles before piece q, so that a segment's tile count is one difference
  std::vector<int64_t> before(np + 1, 0);
  for (int64_t q = 0; q < np; ++q) {
    const b200ot_piece& c = pieces[q];
    if (c.col_start < 0 || c.col_start % kTcBN || c.col_count <= 0 || c.col_count % kTcBN ||
        (int64_t)c.col_start + c.col_count > n_col_slots)
      return B200OT_EINVAL;
    before[q + 1] = before[q] + c.col_count / kTcBN;
  }
  // every row tile belongs to exactly one segment: each live row is written once per split
  std::vector<char> seen(n_seg, 0);
  int64_t mt = 0;
  for (int64_t s = 0; s < n_seg; ++s) {
    const int64_t t = seg[s].row_start / kTcM;
    if (seen[t]) return B200OT_EINVAL;
    seen[t] = 1;
    mt = std::max(mt, before[seg[s].piece_end] - before[seg[s].piece_begin]);
  }
  if (mt > 0x7fffffff) return B200OT_EINVAL;
  b.max_tiles = (int)mt;
  b.n_pieces = np;
  return B200OT_OK;
}

}  // namespace b200ot

using namespace b200ot;

extern "C" {

// ---- batches of B problems, 8 < D <= 64 (tc_reduce_kernel / tc_bwd_kernel with BATCH) ----
B200OT_API int64_t b200ot_batched_scratch_bytes(int64_t B, int64_t N, int64_t M, int32_t D) {
  return kTcBatched.scratch_bytes(B, N, M, D);
}

B200OT_API int b200ot_softmin_fwd_batched(const float* x, const float* y, const float* h_a, const float* h_b,
                                          float h_scale_b, const float* center, const float* out_old, float alpha_old,
                                          float beta, float* out, float* lse2_out, int64_t B, int64_t N, int64_t M,
                                          int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                          void* stream) {
  return softmin_fwd_entry(kTcBatched, x, y, h_a, h_b, h_scale_b, center, out_old, alpha_old, beta, out, lse2_out, B,
                           N, M, D, p, eps, scratch, scratch_bytes, stream);
}

B200OT_API int b200ot_softmin_bwd_x_batched(const float* x, const float* y, const float* h_a, const float* h_b,
                                            float h_scale_b, const float* center, const float* lse2,
                                            const float* grad_out, float* grad_x, int64_t B, int64_t N, int64_t M,
                                            int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                            void* stream) {
  return softmin_bwd_x_entry(kTcBatched, x, y, h_a, h_b, h_scale_b, center, lse2, grad_out, grad_x, B, N, M, D, p, eps,
                             scratch, scratch_bytes, stream);
}

B200OT_API int b200ot_kernel_conv_fwd_batched(const float* x, const float* y, const float* w, const float* center,
                                              float* out, int64_t B, int64_t N, int64_t M, int32_t D, int32_t kind,
                                              float blur, void* scratch, int64_t scratch_bytes, void* stream) {
  return conv_entry(kTcBatched, ConvMode::kFwd, x, y, w, center, nullptr, out, nullptr, B, N, M, D, kind, blur, scratch,
                    scratch_bytes, stream);
}

B200OT_API int b200ot_kernel_conv_bwd_x_batched(const float* x, const float* y, const float* w, const float* center,
                                                const float* grad_out, float* grad_x, int64_t B, int64_t N, int64_t M,
                                                int32_t D, int32_t kind, float blur, void* scratch,
                                                int64_t scratch_bytes, void* stream) {
  return conv_entry(kTcBatched, ConvMode::kBwdX, x, y, w, center, grad_out, nullptr, grad_x, B, N, M, D, kind, blur,
                    scratch, scratch_bytes, stream);
}

B200OT_API int b200ot_kernel_conv_fwd_bwd_x_batched(const float* x, const float* y, const float* w,
                                                    const float* center, float* out, float* grad_unit, int64_t B,
                                                    int64_t N, int64_t M, int32_t D, int32_t kind, float blur,
                                                    void* scratch, int64_t scratch_bytes, void* stream) {
  return conv_entry(kTcBatched, ConvMode::kFwdBwdX, x, y, w, center, nullptr, out, grad_unit, B, N, M, D, kind, blur,
                    scratch, scratch_bytes, stream);
}

// ---- the p = 1 softmin, 8 < D <= 64 (tc_reduce_kernel<6> / tc_bwd_kernel<7>, batched flavour) ----
B200OT_API int64_t b200ot_softmin_l1_scratch_bytes(int64_t B, int64_t N, int64_t M, int32_t D) {
  return kTcL1.scratch_bytes(B, N, M, D);
}

B200OT_API int b200ot_softmin_l1_fwd(const float* x, const float* y, const float* h_a, const float* h_b,
                                     float h_scale_b, const float* center, const float* out_old, float alpha_old,
                                     float beta, float* out, float* lse2_out, int64_t B, int64_t N, int64_t M,
                                     int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                     void* stream) {
  return softmin_fwd_entry(kTcL1, x, y, h_a, h_b, h_scale_b, center, out_old, alpha_old, beta, out, lse2_out, B, N, M,
                           D, p, eps, scratch, scratch_bytes, stream);
}

B200OT_API int b200ot_softmin_l1_bwd_x(const float* x, const float* y, const float* h_a, const float* h_b,
                                       float h_scale_b, const float* center, const float* lse2, const float* grad_out,
                                       float* grad_x, int64_t B, int64_t N, int64_t M, int32_t D, int32_t p, float eps,
                                       void* scratch, int64_t scratch_bytes, void* stream) {
  return softmin_bwd_x_entry(kTcL1, x, y, h_a, h_b, h_scale_b, center, lse2, grad_out, grad_x, B, N, M, D, p, eps,
                             scratch, scratch_bytes, stream);
}

// ---- above D = 64: the K-slab tensor-core kernels (tcwide.cuh) ----
B200OT_API int64_t b200ot_wide_scratch_bytes(int64_t B, int64_t N, int64_t M, int32_t D) {
  return kTcWide.scratch_bytes(B, N, M, D);
}

B200OT_API int b200ot_wide_softmin_fwd(const float* x, const float* y, const float* h_a, const float* h_b,
                                       float h_scale_b, const float* center, const float* out_old, float alpha_old,
                                       float beta, float* out, float* lse2_out, int64_t B, int64_t N, int64_t M,
                                       int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                       void* stream) {
  return softmin_fwd_entry(kTcWide, x, y, h_a, h_b, h_scale_b, center, out_old, alpha_old, beta, out, lse2_out, B, N,
                           M, D, p, eps, scratch, scratch_bytes, stream);
}

B200OT_API int b200ot_wide_softmin_bwd_x(const float* x, const float* y, const float* h_a, const float* h_b,
                                         float h_scale_b, const float* center, const float* lse2,
                                         const float* grad_out, float* grad_x, int64_t B, int64_t N, int64_t M,
                                         int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                         void* stream) {
  return softmin_bwd_x_entry(kTcWide, x, y, h_a, h_b, h_scale_b, center, lse2, grad_out, grad_x, B, N, M, D, p, eps,
                             scratch, scratch_bytes, stream);
}

B200OT_API int b200ot_wide_kernel_conv_fwd(const float* x, const float* y, const float* w, const float* center,
                                           float* out, int64_t B, int64_t N, int64_t M, int32_t D, int32_t kind,
                                           float blur, void* scratch, int64_t scratch_bytes, void* stream) {
  return conv_entry(kTcWide, ConvMode::kFwd, x, y, w, center, nullptr, out, nullptr, B, N, M, D, kind, blur, scratch,
                    scratch_bytes, stream);
}

B200OT_API int b200ot_wide_kernel_conv_bwd_x(const float* x, const float* y, const float* w, const float* center,
                                             const float* grad_out, float* grad_x, int64_t B, int64_t N, int64_t M,
                                             int32_t D, int32_t kind, float blur, void* scratch,
                                             int64_t scratch_bytes, void* stream) {
  return conv_entry(kTcWide, ConvMode::kBwdX, x, y, w, center, grad_out, nullptr, grad_x, B, N, M, D, kind, blur,
                    scratch, scratch_bytes, stream);
}

// one problem (tcapply.cuh, tc_wide_apply_kernel); p = 2 only
B200OT_API int64_t b200ot_wide_plan_apply_scratch_bytes(int64_t N, int64_t M, int32_t D, int64_t K) {
  return kTcWide.dims(1, N, M, D) && K >= 1 && K <= 0x7fffffff ? tc_plan_apply_scratch_bytes(N, M, D, (int)K) : 0;
}

B200OT_API int b200ot_wide_plan_apply(const float* x, const float* y, const float* h_a, const float* h_b,
                                      float h_scale_b, const float* center, const float* lse2, const float* v,
                                      const float* row_factor, float* out, int64_t N, int64_t M, int32_t D, int64_t K,
                                      int32_t p, float eps, void* scratch, int64_t scratch_bytes, void* stream) {
  if (!x || !y || !h_a || !lse2 || !v || !out || !scratch || !kTcWide.dims(1, N, M, D) || K < 1 || K > 0x7fffffff ||
      !valid_p(p) || p_exponent(p) != 2 || !(eps > 0.f))
    return B200OT_EINVAL;
  if (const int rc = scratch_check(scratch, scratch_bytes, b200ot_wide_plan_apply_scratch_bytes(N, M, D, K))) return rc;
  return tc_plan_apply(x, y, h_a, h_b, h_scale_b, center, lse2, v, row_factor, out, N, M, D, (int)K, eps, scratch,
                       (cudaStream_t)stream);
}

// ---- block-sparse problems ----
B200OT_API void b200ot_blocks_shape(int32_t* rows_per_segment, int32_t* col_align) {
  if (rows_per_segment) *rows_per_segment = kTcBlocksTile;
  if (col_align) *col_align = kTcBlocksTile;
}

B200OT_API int64_t b200ot_blocks_scratch_bytes(int64_t N, int64_t n_row_slots, int64_t n_col_slots,
                                               const b200ot_segment* seg, int64_t n_seg, const b200ot_piece* pieces,
                                               int32_t D) {
  TcBlocks b{nullptr, nullptr, n_row_slots, n_col_slots, seg, n_seg, pieces};
  return blocks_check(N, D, 2, 1.f, nullptr, b) ? 0 : tc_blocks_scratch_bytes(N, D, b);
}

B200OT_API int b200ot_softmin_fwd_blocks(const float* x, const float* y, const float* h_a, const float* h_b,
                                         float h_scale_b, const float* center, const float* out_old, float alpha_old,
                                         float beta, float* out, float* lse2_out, int64_t N, const int32_t* row_src,
                                         int64_t n_row_slots, const int32_t* col_src, int64_t n_col_slots,
                                         const b200ot_segment* seg, int64_t n_seg, const b200ot_piece* pieces,
                                         int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                         void* stream) {
  if (!x || !y || !h_a || !row_src || !col_src || !scratch || (!out && !lse2_out)) return B200OT_EINVAL;
  TcBlocks b{row_src, col_src, n_row_slots, n_col_slots, seg, n_seg, pieces};
  if (const int rc = blocks_check(N, D, p, eps, scratch, b)) return rc;
  if (scratch_bytes < tc_blocks_scratch_bytes(N, D, b)) return B200OT_ESCRATCH;
  return softmin_fwd_tc(TcLayout::kBlocks, {x, y, h_a, h_b, h_scale_b, center, nullptr, 1, N, 0, D, p, eps}, &b, out_old,
                        alpha_old, beta, out, lse2_out, scratch, stream);
}

B200OT_API int b200ot_softmin_bwd_x_blocks(const float* x, const float* y, const float* h_a, const float* h_b,
                                           float h_scale_b, const float* center, const float* lse2,
                                           const float* grad_out, float* grad_x, int64_t N, const int32_t* row_src,
                                           int64_t n_row_slots, const int32_t* col_src, int64_t n_col_slots,
                                           const b200ot_segment* seg, int64_t n_seg, const b200ot_piece* pieces,
                                           int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                           void* stream) {
  if (!x || !y || !h_a || !lse2 || !grad_out || !grad_x || !row_src || !col_src || !scratch) return B200OT_EINVAL;
  TcBlocks b{row_src, col_src, n_row_slots, n_col_slots, seg, n_seg, pieces};
  if (const int rc = blocks_check(N, D, p, eps, scratch, b)) return rc;
  if (scratch_bytes < tc_blocks_scratch_bytes(N, D, b)) return B200OT_ESCRATCH;
  return softmin_bwd_x_tc(TcLayout::kBlocks, {x, y, h_a, h_b, h_scale_b, center, lse2, 1, N, 0, D, p, eps}, &b,
                          grad_out, grad_x, scratch, (cudaStream_t)stream);
}

}  // extern "C"
