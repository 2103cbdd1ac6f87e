/* b200ot.h — C ABI of the H100-native (sm_90a) Sinkhorn / kernel-MMD reduction engine.
 *
 * This is the drop-in boundary for the hot path of jeanfeydy/geomloss (reference commit 00e493f).
 * The reference has no FFI: its plugin seams are the Python callables
 *   softmin(eps, C_xy, h_y) -> f_x            (src/geomloss/_legacy/sinkhorn_divergence.py:291-303,
 *                                              implemented by softmin_tensorized / softmin_online,
 *                                              src/geomloss/_legacy/sinkhorn_samples.py:32-71,337-346)
 *   kernel matvecs of kernel_loss             (src/geomloss/_legacy/kernel_samples.py:92-146)
 * which the pykeops "online" backend lowers to one CUDA map-reduce launch per call
 * (sinkhorn_samples.py:322-334: generic_logsumexp("(B - (P * cost))", Vi(1), Vi(D), Vj(D), Vj(1), Pm(1))).
 * The functions below are what a maintainer would bind in place of that pykeops call.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to fp32 (or the stated type), row-major, contiguous;
 *     the caller owns every buffer; nothing is allocated, freed or retained by the library;
 *   - kernels are enqueued on `stream` (a cudaStream_t passed as void*) and the call returns
 *     immediately; no host synchronisation happens inside;
 *   - return value: 0 on success, a negative B200OT_E* code otherwise (never throws, never aborts);
 *   - "rows" x:(N,D) own the output, "cols" y:(M,D) are reduced over; D <= B200OT_MAX_D;
 *   - a reduction is split into two launches so that the column cloud can be packed once and
 *     reused (and so that partial results of column shards living on other GPUs can be merged):
 *         pack  ->  partial reduction  ->  finalize.
 *
 * Environment variables (read by the one-call entry points on every call; meant for A/B timing and for the parity tests
 * that hold both settings of every switch to the oracle — a deployment leaves them unset):
 *   B200OT_TC_MIN_D      "d" or "softmin_fwd,softmin_bwd,conv_fwd,conv_bwd": smallest D <= B200OT_MAX_D an operator
 *                        hands to the tensor-core kernels (default "7,9,5,9": forward softmin from 7, gaussian from 5)
 *   B200OT_TC_MIN_PAIRS  smallest N*M for that hand-over (default 8e8)
 *   B200OT_PAIR          "0": b200ot_softmin_fwd never takes the symmetric kernel (see b200ot_softmin_fwd_pair)
 *   B200OT_PAIR_TILES    test hook: at least this many 1024-point tiles per block of the paired kernels
 */
#ifndef B200OT_H_
#define B200OT_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200OT_API __attribute__((visibility("default")))
#else
#define B200OT_API
#endif

#define B200OT_VERSION 202 /* 0.2.2 */
#define B200OT_MAX_D 8     /* dimensions served by the CUDA-core (register tile) kernels of this build */

/* error codes */
#define B200OT_OK 0
#define B200OT_EINVAL -1   /* bad argument (null pointer, non-positive size, unsupported p / D / kind) */
#define B200OT_ESCRATCH -2 /* scratch buffer too small (see *_scratch_bytes) */
#define B200OT_ECUDA -3    /* a CUDA runtime call failed; see b200ot_last_cuda_error() */
#define B200OT_EALIGN -4   /* pointer not 16-byte aligned */

/* kernel kinds for b200ot_kernel_conv_* (reference: kernel_samples.py:62-82) */
#define B200OT_KERNEL_GAUSSIAN 0  /* exp(-|x-y|^2 / (2 blur^2)) */
#define B200OT_KERNEL_LAPLACIAN 1 /* exp(-sqrt(max(|x-y|^2/blur^2, 1e-8))) */
#define B200OT_KERNEL_ENERGY 2    /* -sqrt(max(|x-y|^2, 1e-8)) */

/* The reference has TWO conventions for the Euclidean norm under p = 1 / laplacian / energy:
 *   backend="tensorized":  sqrt(clamp_min(|x-y|^2, 1e-8))   (utils.py:56-61)           -> p = 1, kinds 1, 2
 *   backend="online" / "multiscale" (pykeops Norm2 / .sqrt(), sinkhorn_samples.py:303-306, utils.py:56-58):
 *                          sqrt(|x-y|^2), zero gradient at coincident points            -> flag below
 * Or the flag into `p` (softmin entry points) or `kind` (kernel_conv entry points). */
#define B200OT_P_UNCLAMPED 0x100
#define B200OT_KERNEL_UNCLAMPED 0x100

B200OT_API const char* b200ot_strerror(int code);
B200OT_API const char* b200ot_last_cuda_error(void);
B200OT_API int b200ot_version(void);

/* ---------------------------------------------------------------------------------------------
 * Softmin  —  out_i = -eps * log sum_j exp( h_j - |x_i - y_j|^p / (p * eps) ),   p in {1, 2}
 * replaces softmin_tensorized (sinkhorn_samples.py:32-71) / softmin_online (:337-346).
 * p = 1 uses sqrt(max(|x-y|^2, 1e-8)) like the reference's `distances` (utils.py:56-61);
 * p = 1 | B200OT_P_UNCLAMPED uses the pykeops convention (see above).
 * ------------------------------------------------------------------------------------------- */

/* Bytes of scratch needed by b200ot_softmin_fwd / _bwd_x for (N rows, M cols, D). */
B200OT_API int64_t b200ot_softmin_scratch_bytes(int64_t N, int64_t M, int32_t D);

/* One-call softmin:  out (N) <- alpha_old * out_old + beta * softmin(eps, (x, y), h)
 *   h_a (M), h_b (M, nullable):  h_j = h_a[j] + h_scale_b * h_b[j]
 *       (the Sinkhorn loop's  b_log + g / eps  is h_a = b_log, h_b = g, h_scale_b = 1/eps —
 *        sinkhorn_divergence.py:480-488 — fused here instead of a separate elementwise launch);
 *   out_old (N, nullable), alpha_old, beta:  the damping and the 1/2 (f + ft) averaging of
 *       sinkhorn_divergence.py:480-493 fused into the epilogue (alpha_old=0, beta=1: plain softmin);
 *   lse2_out (N, nullable): log2-domain log-sum-exp per row, saved for the backward pass;
 *   center (D, nullable): device vector subtracted from both clouds before the |x|^2 - 2x.y + |y|^2
 *       expansion (improves fp32 conditioning; any point near the data works, zeros if null);
 *   scratch: >= b200ot_softmin_scratch_bytes(N, M, D) bytes, 16-byte aligned.
 */
B200OT_API int b200ot_softmin_fwd(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                       const float* center, const float* out_old, float alpha_old, float beta, float* out,
                       float* lse2_out, int64_t N, int64_t M, int32_t D, int32_t p, float eps, void* scratch,
                       int64_t scratch_bytes, void* stream);

/* Two softmins of one Jacobi Sinkhorn iteration from one pass over the pairs: A (rows x, columns y, column potential
 * hy_a + hy_scale_b * hy_b; out_a, lse2_a: N) and B (rows y, columns x, column potential hx_a + hx_scale_b * hx_b;
 * out_b, lse2_b: M), each with the epilogue of b200ot_softmin_fwd.  One exponential 2^T_ij, T_ij = log2e (hx_i + hy_j -
 * C_ij / eps), feeds row sum i of A and column sum j of B.  A softmin whose merged sums leave the range in which that
 * is exact (a point's sum outside [count 2^-100, 2^100]: zero-weight points, potentials that move by tens of nats
 * in one step) is recomputed on the path of b200ot_softmin_fwd, bit for bit, with no host synchronisation.
 * D = 3, p = 2, and a shape b200ot_softmin_pair_scratch_bytes accepts; no output may overlap an input or another
 * output (EINVAL).  b200ot_softmin_fwd takes the symmetric variant of this kernel by itself when x == y and N == M
 * (each unordered pair evaluated once), unless $B200OT_PAIR=0.  Deterministic: no atomics on the sums.
 * scratch: >= b200ot_softmin_pair_scratch_bytes(N, M, D), which is 0 for a shape the paired kernel does not serve. */
B200OT_API int64_t b200ot_softmin_pair_scratch_bytes(int64_t N, int64_t M, int32_t D);
B200OT_API int b200ot_softmin_fwd_pair(const float* x, const float* y, const float* hy_a, const float* hy_b,
                                       float hy_scale_b, const float* out_a_old, float alpha_a_old, float beta_a,
                                       float* out_a, float* lse2_a, const float* hx_a, const float* hx_b,
                                       float hx_scale_b, const float* out_b_old, float alpha_b_old, float beta_b,
                                       float* out_b, float* lse2_b, const float* center, int64_t N, int64_t M,
                                       int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                       void* stream);

/* One softmin of b200ot_softmin_fwd_step: column potential h_a + h_scale_b * h_b (h_b nullable) and the epilogue of
 * b200ot_softmin_fwd (out_old and one of out, lse2 nullable). */
typedef struct {
  const float* h_a;
  const float* h_b;
  float h_scale_b;
  const float* out_old;
  float alpha_old, beta;
  float* out;
  float* lse2;
} b200ot_softmin_slot;

/* The four softmins of one symmetric Jacobi Sinkhorn iteration as one launch group: slots[0] rows x, columns y
 * (out: N); slots[1] rows y, columns x (M); slots[2] rows x, columns x (N); slots[3] rows y, columns y (M).  The xy / yx
 * pair of b200ot_softmin_fwd_pair and the symmetric xx and yy softmins of b200ot_softmin_fwd run as one launch of the
 * paired kernel, with the range check and recomputation of both, and give their results bit for bit.  D = 3, p = 2,
 * and a shape b200ot_softmin_step_scratch_bytes accepts (0 otherwise); no output may overlap an input or another output
 * (EINVAL).  scratch: >= b200ot_softmin_step_scratch_bytes(N, M, D), the four range flags first. */
B200OT_API int64_t b200ot_softmin_step_scratch_bytes(int64_t N, int64_t M, int32_t D);
B200OT_API int b200ot_softmin_fwd_step(const float* x, const float* y, const b200ot_softmin_slot* slots,
                                       const float* center, int64_t N, int64_t M, int32_t D, int32_t p, float eps,
                                       void* scratch, int64_t scratch_bytes, void* stream);

/* Gradient of the softmin w.r.t. the row cloud (the only gradient the reference's autograd
 * contract carries: columns and h are detached, sinkhorn_samples.py:179-185, sinkhorn_divergence.py:616-623):
 *   grad_x[i,:] = grad_out[i] * sum_j softmax_j(h_j - C_ij/eps) * dC(x_i, y_j)/dx_i
 * lse2 is the lse2_out of the matching forward call.  grad_x (N,D) is overwritten. */
B200OT_API int b200ot_softmin_bwd_x(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                         const float* center, const float* lse2, const float* grad_out, float* grad_x, int64_t N,
                         int64_t M, int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                         void* stream);

/* The softmax weights of the p = 2 softmin applied to a value matrix, in one reduction over the pairs per slab of
 * value columns (the transport plan times V: barycentric maps, colour / label / feature transport):
 *   out[i,k] = row_factor[i] * sum_j w_ij v[j,k],   w_ij = softmax_j(h_j - |x_i - y_j|^2 / (2 eps))
 *   v (M,K) row-major, any sign, K >= 1;  out (N,K) is overwritten;  row_factor (N, nullable): 1 when null;
 *   lse2 (N): the lse2_out of b200ot_softmin_fwd for the same x, y, h, center, eps.  The weights are normalised by
 *       the kernel's own sum over j, so rounding of lse2 cancels and a constant v comes back (to rounding);
 *   a column with h_j = -1e5 (the engine's log 0) contributes exactly 0;
 *   1 <= D <= 64, p = 2 only.  D <= 8 runs on the CUDA cores in slabs of 8 value columns, above on the tensor cores
 *   in slabs of 64 (routing as for b200ot_softmin_bwd_x); every slab is one pass that recomputes the exponent.
 *   scratch: >= b200ot_plan_apply_scratch_bytes(N, M, D, K) bytes, 16-byte aligned. */
B200OT_API int64_t b200ot_plan_apply_scratch_bytes(int64_t N, int64_t M, int32_t D, int64_t K);
B200OT_API int b200ot_plan_apply(const float* x, const float* y, const float* h_a, const float* h_b, float h_scale_b,
                      const float* center, const float* lse2, const float* v, const float* row_factor, float* out,
                      int64_t N, int64_t M, int32_t D, int64_t K, int32_t p, float eps, void* scratch,
                      int64_t scratch_bytes, void* stream);

/* --- the three stages of b200ot_softmin_fwd, exposed for column-sharded (multi-GPU) use --- */

/* Number of floats of a packed column buffer for M columns of dimension D with `extra` per-column
 * scalars (softmin: 1 = h; gaussian conv: 2 = -|y|^2/2 and weight; laplacian / energy conv: 1 = weight). */
B200OT_API int64_t b200ot_packed_cols_floats(int64_t M, int32_t D, int32_t extra);

/* Pack the column cloud for a softmin at temperature eps (coordinates pre-scaled, h folded into the
 * per-column term, padding columns neutral).  cols_out: b200ot_packed_cols_floats(M, D, 1) floats. */
B200OT_API int b200ot_softmin_pack(const float* y, const float* h_a, const float* h_b, float h_scale_b, const float* center,
                        int64_t M, int32_t D, int32_t p, float eps, float* cols_out, void* stream);

/* Number of column splits the partial reduction will use for (N, M, D): partials hold n_split * N pairs. */
B200OT_API int32_t b200ot_softmin_num_splits(int64_t N, int64_t M, int32_t D);

/* Partial reduction over the packed columns: part[(s*N + i)*2 + {0,1}] = (running max m, sum of
 * exp2(t - m)) in the log2 domain, for s < n_split.  This is the kernel that does the N x M work. */
B200OT_API int b200ot_softmin_partial(const float* x, const float* center, const float* cols, float* part, int32_t n_split,
                           int64_t N, int64_t M, int32_t D, int32_t p, float eps, void* stream);

/* ---- ranges mode: block-sparse and batched problems in ONE launch ------------------------------------------
 * Replaces the reference's `ranges=` argument of pykeops reductions (softmin_multiscale, sinkhorn_samples.py:445-450,
 * built by kernel_truncation :493-530 / from_matrix; kernel_multiscale, kernel_samples.py:246-256) and the batched
 * LazyTensor reduction of softmin_online_lazytensor (:229-290, a block-diagonal problem).
 *   segment  = a run of consecutive rows that share one list of column pieces (one CTA per segment):
 *              a cluster of the sorted row cloud (cut into <= max_rows_per_segment rows), or a batch element;
 *   piece    = a run of consecutive column SLOTS (col_start, col_count), both multiples of col_align,
 *              col_count <= max_cols_per_piece;
 *   slots    = the packed column buffer in gather mode: slot s holds column src_index[s] of the caller's arrays,
 *              or a neutral padding column when src_index[s] < 0 — clusters / batch elements are padded to a
 *              multiple of col_align slots so that every piece starts on a chunk boundary.
 * The reduction visits exactly the (row, column) pairs listed: bit-for-bit the blocks of the reference's ranges. */
typedef struct { int32_t row_start, row_count, piece_begin, piece_end; } b200ot_segment; /* 16-byte aligned array */
typedef struct { int32_t col_start, col_count; } b200ot_piece;                           /*  8-byte aligned array */
#define B200OT_RANGES_BIG 0   /* 512-row segments, pieces <= 1024 columns: large clusters */
#define B200OT_RANGES_SMALL 1 /* 128-row segments, pieces <= 256 columns: small clusters / small batch elements */
B200OT_API void b200ot_ranges_shape(int32_t variant, int32_t* max_rows_per_segment, int32_t* max_cols_per_piece,
                                    int32_t* col_align);

/* b200ot_softmin_pack in gather mode: cols_out holds b200ot_packed_cols_floats(n_slots, D, 1) floats. */
B200OT_API int b200ot_softmin_pack_gather(const float* y, const float* h_a, const float* h_b, float h_scale_b,
                                          const float* center, const int32_t* src_index, int64_t n_slots, int32_t D,
                                          int32_t p, float eps, float* cols_out, void* stream);

/* part: (N, 2) (m, s) pairs, one per row; rows that belong to no segment are left untouched. */
B200OT_API int b200ot_softmin_partial_ranges(const float* x, const float* center, const float* cols,
                                             const b200ot_segment* seg, int64_t n_seg, const b200ot_piece* pieces,
                                             float* part, int64_t N, int32_t D, int32_t p, float eps,
                                             int32_t variant, void* stream);

/* Collapse n_part partial (m, s) sets into one per row: merged[i*2 + {0,1}].  A rank calls this on its own
 * splits before exchanging partials with the other column shards (N*8 bytes per rank). */
B200OT_API int b200ot_softmin_merge(const float* part, int32_t n_part, float* merged, int64_t N, void* stream);

/* Merge n_part partial (m, s) sets (own splits and/or other ranks' shards, concatenated along the
 * leading axis) and apply the epilogue of b200ot_softmin_fwd. */
B200OT_API int b200ot_softmin_finalize(const float* part, int32_t n_part, const float* out_old, float alpha_old, float beta,
                            float* out, float* lse2_out, int64_t N, float eps, void* stream);

/* --- stages of b200ot_softmin_bwd_x, for column-sharded use: per-shard partial sums
 *     part[(s*N + i)*(D+1) + {0: sum_j w_ij, 1+k: sum_j w_ij * (coordinate or unit-vector term)}],
 *     which add across shards (all-reduce SUM) before the finalize --- */
B200OT_API int b200ot_softmin_bwd_partial(const float* x, const float* center, const float* cols, const float* lse2,
                                          float* part, int32_t n_split, int64_t N, int64_t M, int32_t D, int32_t p,
                                          float eps, void* stream);
/* ranges variant (see b200ot_softmin_partial_ranges): part is (N, D+1), one split */
B200OT_API int b200ot_softmin_bwd_partial_ranges(const float* x, const float* center, const float* cols,
                                                 const float* lse2, const b200ot_segment* seg, int64_t n_seg,
                                                 const b200ot_piece* pieces, float* part, int64_t N, int32_t D,
                                                 int32_t p, float eps, int32_t variant, void* stream);
/* One call: sums (N, D+1) = the merged partial sums of the row-gradient pass over ALL columns given (pack + partial +
 * merge; CUDA-core path for D <= B200OT_MAX_D, tensor-core path for p = 2 up to D = 64).  A column shard calls this
 * on its slice, all-reduces `sums` (SUM) and finishes with b200ot_softmin_bwd_finalize(n_part = 1). */
B200OT_API int b200ot_softmin_bwd_sums(const float* x, const float* y, const float* h_a, const float* h_b,
                                       float h_scale_b, const float* center, const float* lse2, float* sums,
                                       int64_t N, int64_t M, int32_t D, int32_t p, float eps, void* scratch,
                                       int64_t scratch_bytes, void* stream);
/* merged[i*width + a] = sum_s part[(s*N + i)*width + a] */
B200OT_API int b200ot_rowsum_merge(const float* part, int32_t n_part, int32_t width, float* merged, int64_t N,
                                   void* stream);
B200OT_API int b200ot_softmin_bwd_finalize(const float* part, int32_t n_part, const float* x, const float* center,
                                           const float* grad_out, float* grad_x, int64_t N, int32_t D, int32_t p,
                                           float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Kernel convolution  —  out_i = sum_j k(x_i, y_j) * w_j      (kernel_samples.py:128-137)
 * ------------------------------------------------------------------------------------------- */
/* b200ot_kernel_conv_fwd and _bwd_x additionally accept 8 < D <= 64 for every kind: that range runs on the tensor
 * cores (wgmma, fp16x2 split operands, exponent accumulated in registers; laplacian / energy take d from it, see
 * DESIGN.md section 3.3d).  For D <= B200OT_MAX_D the gaussian kernel takes the faster of the two paths per operator
 * and problem size (csrc/b200ot_tc.cu: tc_routed); laplacian / energy stay on the CUDA cores.  Results agree
 * to the tolerances of DESIGN.md section 4 either way. */
B200OT_API int64_t b200ot_kernel_conv_scratch_bytes(int64_t N, int64_t M, int32_t D);

B200OT_API int b200ot_kernel_conv_fwd(const float* x, const float* y, const float* w, const float* center, float* out,
                           int64_t N, int64_t M, int32_t D, int32_t kind, float blur, void* scratch,
                           int64_t scratch_bytes, void* stream);

/* grad_x[i,:] = grad_out[i] * sum_j w_j * d k(x_i, y_j) / d x_i   (rows only; columns via a swapped call) */
B200OT_API int b200ot_kernel_conv_bwd_x(const float* x, const float* y, const float* w, const float* center,
                             const float* grad_out, float* grad_x, int64_t N, int64_t M, int32_t D, int32_t kind,
                             float blur, void* scratch, int64_t scratch_bytes, void* stream);

/* Value AND unit row gradient from ONE pass over the N x M pairs (gaussian only; EINVAL otherwise):
 *   out[i] = sum_j k(x_i, y_j) w_j,    grad_unit[i,:] = sum_j w_j * d k(x_i, y_j) / d x_i
 * i.e. b200ot_kernel_conv_fwd and b200ot_kernel_conv_bwd_x(grad_out = 1) together: the row-gradient reduction
 * accumulates sum_j w_j k_ij anyway, so a caller that will differentiate (autograd of kernel_loss's matvecs,
 * kernel_samples.py:116-137) saves the separate forward reduction and multiplies grad_unit by its upstream gradient
 * row by row.  Same scratch size as the other two. */
B200OT_API int b200ot_kernel_conv_fwd_bwd_x(const float* x, const float* y, const float* w, const float* center,
                                 float* out, float* grad_unit, int64_t N, int64_t M, int32_t D, int32_t kind,
                                 float blur, void* scratch, int64_t scratch_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Batched problems in the tensor-core dimensions (8 < D <= 64): B independent problems of the same shape in one
 * launch group per call — the batched LazyTensor reductions of the reference (softmin_online_lazytensor,
 * sinkhorn_samples.py:229-290; kernel_loss on (B, N, D) inputs).  x (B,N,D), y (B,M,D); h_a, h_b, w (B,M); out,
 * lse2, grad_out (B,N); grad_x (B,N,D); center (D) shared by the whole batch.  Row i of element b is reduced over
 * the columns of element b only.  Arguments and results are those of the one-problem entries above, element by
 * element; p = 2 only (the p = 1 softmin has entries of its own, b200ot_softmin_l1_*); D <= 8 batches go through the
 * ranges entry points.
 * EINVAL for B < 1, D <= 8 or D > 64; scratch: b200ot_batched_scratch_bytes(B, N, M, D) bytes, 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
B200OT_API int64_t b200ot_batched_scratch_bytes(int64_t B, int64_t N, int64_t M, int32_t D);
B200OT_API int b200ot_softmin_fwd_batched(const float* x, const float* y, const float* h_a, const float* h_b,
                                          float h_scale_b, const float* center, const float* out_old, float alpha_old,
                                          float beta, float* out, float* lse2_out, int64_t B, int64_t N, int64_t M,
                                          int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                          void* stream);
B200OT_API int b200ot_softmin_bwd_x_batched(const float* x, const float* y, const float* h_a, const float* h_b,
                                            float h_scale_b, const float* center, const float* lse2,
                                            const float* grad_out, float* grad_x, int64_t B, int64_t N, int64_t M,
                                            int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                            void* stream);
B200OT_API int b200ot_kernel_conv_fwd_batched(const float* x, const float* y, const float* w, const float* center,
                                              float* out, int64_t B, int64_t N, int64_t M, int32_t D, int32_t kind,
                                              float blur, void* scratch, int64_t scratch_bytes, void* stream);
B200OT_API int b200ot_kernel_conv_bwd_x_batched(const float* x, const float* y, const float* w, const float* center,
                                                const float* grad_out, float* grad_x, int64_t B, int64_t N, int64_t M,
                                                int32_t D, int32_t kind, float blur, void* scratch,
                                                int64_t scratch_bytes, void* stream);
/* gaussian only, like b200ot_kernel_conv_fwd_bwd_x */
B200OT_API int b200ot_kernel_conv_fwd_bwd_x_batched(const float* x, const float* y, const float* w,
                                                    const float* center, float* out, float* grad_unit, int64_t B,
                                                    int64_t N, int64_t M, int32_t D, int32_t kind, float blur,
                                                    void* scratch, int64_t scratch_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * The p = 1 softmin in the tensor-core dimensions (8 < D <= 64): f_i = -eps log sum_j exp(h_j - |x_i - y_j| / eps),
 * the reference's cost |x - y| (`distances`, utils.py:56-61) in its tensorized (p = 1) or pykeops
 * (p = 1 | B200OT_P_UNCLAMPED) convention.  Batched layout, arguments and results as the batched entries above
 * (B = 1: one problem); lse2_out / lse2 in the same log2 units, so b200ot_softmin_finalize's epilogue applies.
 * EINVAL (before any launch) for null pointers, B < 1, N or M <= 0, D <= 8 or D > 64, p other than 1 or
 * 1 | B200OT_P_UNCLAMPED, eps <= 0; EALIGN for a misaligned scratch; ESCRATCH below
 * b200ot_softmin_l1_scratch_bytes(B, N, M, D) (0 for a shape these entries refuse).
 * ------------------------------------------------------------------------------------------- */
B200OT_API int64_t b200ot_softmin_l1_scratch_bytes(int64_t B, int64_t N, int64_t M, int32_t D);
B200OT_API int b200ot_softmin_l1_fwd(const float* x, const float* y, const float* h_a, const float* h_b,
                                     float h_scale_b, const float* center, const float* out_old, float alpha_old,
                                     float beta, float* out, float* lse2_out, int64_t B, int64_t N, int64_t M,
                                     int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                     void* stream);
/* grad_x (B,N,D) of <grad_out, f> with y and h constant: go_i sum_j w_ij (x_i - y_j) / |x_i - y_j| (zero for
 * coincident pairs, which keep their weight) */
B200OT_API int b200ot_softmin_l1_bwd_x(const float* x, const float* y, const float* h_a, const float* h_b,
                                       float h_scale_b, const float* center, const float* lse2, const float* grad_out,
                                       float* grad_x, int64_t B, int64_t N, int64_t M, int32_t D, int32_t p, float eps,
                                       void* scratch, int64_t scratch_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Above D = 64 (64 < D <= B200OT_MAX_D_WIDE): the p = 2 and p = 1 softmins and the three kernel convolutions,
 * forward and row gradient, on tensor-core kernels that stream the coordinates in 64-dimension slabs.  Batched layout,
 * arguments and results as the batched entries above (B = 1: one problem): the softmin entries take those of
 * b200ot_softmin_l1_* with p = 1 or 2 (| B200OT_P_UNCLAMPED), the convolutions those of b200ot_kernel_conv_*_batched
 * (kind | B200OT_KERNEL_UNCLAMPED).  EINVAL (before any launch) for null pointers, B < 1, N or M <= 0, D <= 64 or
 * D > B200OT_MAX_D_WIDE, a bad p or kind, eps <= 0, blur <= 0 (gaussian, laplacian); EALIGN for a misaligned
 * scratch; ESCRATCH below b200ot_wide_scratch_bytes(B, N, M, D) (0 for a shape these entries refuse), one size for
 * every entry of the family.
 * ------------------------------------------------------------------------------------------- */
#define B200OT_MAX_D_WIDE 1024
B200OT_API int64_t b200ot_wide_scratch_bytes(int64_t B, int64_t N, int64_t M, int32_t D);
B200OT_API int b200ot_wide_softmin_fwd(const float* x, const float* y, const float* h_a, const float* h_b,
                                       float h_scale_b, const float* center, const float* out_old, float alpha_old,
                                       float beta, float* out, float* lse2_out, int64_t B, int64_t N, int64_t M,
                                       int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                       void* stream);
B200OT_API int b200ot_wide_softmin_bwd_x(const float* x, const float* y, const float* h_a, const float* h_b,
                                         float h_scale_b, const float* center, const float* lse2,
                                         const float* grad_out, float* grad_x, int64_t B, int64_t N, int64_t M,
                                         int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                         void* stream);
B200OT_API int b200ot_wide_kernel_conv_fwd(const float* x, const float* y, const float* w, const float* center,
                                           float* out, int64_t B, int64_t N, int64_t M, int32_t D, int32_t kind,
                                           float blur, void* scratch, int64_t scratch_bytes, void* stream);
B200OT_API int b200ot_wide_kernel_conv_bwd_x(const float* x, const float* y, const float* w, const float* center,
                                             const float* grad_out, float* grad_x, int64_t B, int64_t N, int64_t M,
                                             int32_t D, int32_t kind, float blur, void* scratch,
                                             int64_t scratch_bytes, void* stream);
/* The plan applied to a value matrix above D = 64: b200ot_plan_apply's arguments, contract and results for one problem
 * (B = 1) with 64 < D <= B200OT_MAX_D_WIDE, p = 2 (| B200OT_P_UNCLAMPED), K >= 1; lse2 is the lse2_out of
 * b200ot_wide_softmin_fwd for the same x, y, h, center, eps.  One pass over the pairs per slab of 64 value columns,
 * each recomputing the full-K exponent on the K-slab kernels.  EINVAL (before any launch) for null pointers, N or
 * M <= 0, D <= 64 or D > B200OT_MAX_D_WIDE, K < 1, a bad p, eps <= 0; EALIGN for a misaligned scratch; ESCRATCH below
 * b200ot_wide_plan_apply_scratch_bytes(N, M, D, K) (0 for a shape this entry refuses). */
B200OT_API int64_t b200ot_wide_plan_apply_scratch_bytes(int64_t N, int64_t M, int32_t D, int64_t K);
B200OT_API int b200ot_wide_plan_apply(const float* x, const float* y, const float* h_a, const float* h_b,
                                      float h_scale_b, const float* center, const float* lse2, const float* v,
                                      const float* row_factor, float* out, int64_t N, int64_t M, int32_t D, int64_t K,
                                      int32_t p, float eps, void* scratch, int64_t scratch_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Explicit cost matrices: both softmins of one symmetric Sinkhorn update from ONE pass over C
 * replaces softmin_dense on C and on a contiguous copy of C^T (ot/_implementations/matrix.py:29-94, :620-660):
 *   f_out[b,i] <- alpha_old * f_old[b,i] + beta * (-eps log sum_j exp(log_b[b,j] + inv_eps g_old[b,j] - inv_eps C[b,i,j]))
 *   g_out[b,j] <- alpha_old * g_old[b,j] + beta * (-eps log sum_i exp(log_a[b,i] + inv_eps f_old[b,i] - inv_eps C[b,i,j]))
 * C (B,N,M) row-major fp32, any alignment; log_a, f_old (B,N); log_b, g_old (B,M); f_out, g_out must not alias the
 * inputs.  lse2_row (B,N), lse2_col (B,M) (nullable): the log2-domain log-sum-exps, for the backward entry.
 * Three launches: the pass over C, then b200ot_softmin_finalize for the rows and for the columns.
 * EINVAL (before any launch) for null pointers (lse2_* excepted), B, N or M <= 0, eps or inv_eps <= 0; EALIGN for a
 * scratch not 16-byte aligned; ESCRATCH below b200ot_dense_scratch_bytes(B, N, M), a pure function of the shape.
 * ------------------------------------------------------------------------------------------- */
B200OT_API int64_t b200ot_dense_scratch_bytes(int64_t B, int64_t N, int64_t M);
B200OT_API int b200ot_dense_softmin_pair(const float* C, const float* log_a, const float* log_b, const float* f_old,
                                         const float* g_old, float inv_eps, float alpha_old, float beta, float* f_out,
                                         float* g_out, float* lse2_row, float* lse2_col, int64_t B, int64_t N,
                                         int64_t M, float eps, void* scratch, int64_t scratch_bytes, void* stream);
/* Gradient of <go_f, f~> + <go_g, g~> w.r.t. C for the pair above (alpha_old = 0, beta = 1; fold a damping factor into
 * go_*), f and g the potentials the forward read and lse2_* its outputs; one pass, grad_C (B,N,M) overwritten:
 *   grad_C[b,i,j] = go_f[b,i] 2^(t_ij - lse2_row[b,i]) + go_g[b,j] 2^(u_ij - lse2_col[b,j]),
 *   t_ij = log2e (log_b[b,j] + inv_eps (g[b,j] - C[b,i,j])),  u_ij = log2e (log_a[b,i] + inv_eps (f[b,i] - C[b,i,j])).
 * EINVAL (before any launch) for null pointers, B, N or M <= 0, inv_eps <= 0. */
B200OT_API int b200ot_dense_softmin_pair_bwd(const float* C, const float* log_a, const float* log_b, const float* f,
                                             const float* g, float inv_eps, const float* lse2_row,
                                             const float* lse2_col, const float* go_f, const float* go_g,
                                             float* grad_C, int64_t B, int64_t N, int64_t M, void* stream);

/* Row softmins only, for a group of 1 to B200OT_DENSE_ROWS_MAX matrices in ONE partials launch: the Jacobi updates of
 * the Sinkhorn divergence on user-supplied cost matrices (softmin_tensorized, _legacy/sinkhorn_samples.py:32-71, on
 * C_xy, C_yx, C_xx, C_yy, which need not be transposes of one another).  Per problem k:
 *   out[b,i] <- alpha_old * out_old[b,i] + beta * (-eps log sum_j exp(log_w[b,j] + pot[b,j] / eps - C[b,i,j] / eps))
 * C (B, n_rows, n_cols) row-major fp32, any alignment (16-byte loads when C is 16-byte aligned and n_cols % 4 == 0,
 * the same bits otherwise); log_w, pot (B, n_cols); out_old, out, lse2 (B, n_rows).  pot null: 0; out_old null:
 * 0; lse2 (nullable) the log2-domain log-sum-exps for b200ot_dense_softmin_rows_bwd; out may be null when lse2 is
 * not.  out must not alias the inputs.  1 + n launches: the partials of every problem, then b200ot_softmin_finalize
 * per problem.  EINVAL (before any launch) for null pointers, n outside [1, B200OT_DENSE_ROWS_MAX], B, n_rows or
 * n_cols <= 0, eps <= 0; EALIGN for a scratch not 16-byte aligned; ESCRATCH below b200ot_dense_rows_scratch_bytes
 * (a pure function of the shapes, 0 for a group these entries refuse). */
#define B200OT_DENSE_ROWS_MAX 4
typedef struct {
  const float *C, *log_w, *pot, *out_old;
  float *out, *lse2;
  int64_t B, n_rows, n_cols;
} b200ot_dense_rows;
B200OT_API int64_t b200ot_dense_rows_scratch_bytes(const b200ot_dense_rows* probs, int32_t n);
B200OT_API int b200ot_dense_softmin_rows(const b200ot_dense_rows* probs, int32_t n, float eps, float alpha_old,
                                         float beta, void* scratch, int64_t scratch_bytes, void* stream);
/* Gradient of <go, out~> w.r.t. C for one problem of the entry above (alpha_old = 0, beta = 1: fold a damping factor
 * into go), pot the potential the forward read (nullable) and lse2 its output; one pass, grad_C (B,N,M) overwritten:
 *   grad_C[b,i,j] = go[b,i] 2^(t_ij - lse2[b,i]),   t_ij = log2e (log_w[b,j] + inv_eps (pot[b,j] - C[b,i,j])).
 * EINVAL (before any launch) for null pointers (pot excepted), B, N or M <= 0, inv_eps <= 0. */
B200OT_API int b200ot_dense_softmin_rows_bwd(const float* C, const float* log_w, const float* pot, float inv_eps,
                                             const float* lse2, const float* go, float* grad_C, int64_t B, int64_t N,
                                             int64_t M, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Block-sparse softmins in the tensor-core dimensions (8 < D <= 64, p = 2 or 2 | B200OT_P_UNCLAMPED): the fine phase
 * of the two-scale Sinkhorn with user cluster labels (sinkhorn_multiscale, sinkhorn_samples.py:547-681), the
 * counterpart of the ranges entries above, which serve D <= B200OT_MAX_D.  A separate family with its own layout:
 *   slots     every row cluster and every column cluster is padded to whole tiles of `col_align` (128) points on its
 *             own; row slot r holds row row_src[r] of x, column slot s column col_src[s] of y (-1: padding, a neutral
 *             column / a row that writes nothing).  row_src (n_row_slots) and col_src (n_col_slots) are device arrays;
 *   segment   one tile of `rows_per_segment` (128) row slots of one row cluster: row_start = the first slot (a multiple
 *             of 128), row_count = its live rows (1..128), [piece_begin, piece_end) its pieces.  Exactly one segment per
 *             row tile (n_seg = n_row_slots / 128); launch order = array order, so list the heaviest first;
 *   piece     (col_start, col_count): a run of whole column tiles (both multiples of 128);
 *   seg, pieces are HOST arrays (16- / 8-byte aligned).  Every call validates them and copies them into the scratch on
 *             `stream` (from pageable memory that copy waits for the stream's earlier work).
 * Each row is reduced over exactly the columns of its segment's pieces.  Results are indexed by row (x, lse2, out,
 * grad_x: N rows), h_a / h_b by column of y.  The column tiles of a segment are cut into splits like a dense problem's
 * ($B200OT_FORCE_SPLITS applies).
 * EINVAL (before any launch) for null pointers, N <= 0, n_seg <= 0, D <= 8 or D > 64, p other than 2, and descriptors
 * off the tile grid; EALIGN for misaligned descriptor arrays or scratch; ESCRATCH below b200ot_blocks_scratch_bytes
 * (0 for invalid descriptors).
 * ------------------------------------------------------------------------------------------- */
B200OT_API void b200ot_blocks_shape(int32_t* rows_per_segment, int32_t* col_align);
B200OT_API int64_t b200ot_blocks_scratch_bytes(int64_t N, int64_t n_row_slots, int64_t n_col_slots,
                                               const b200ot_segment* seg, int64_t n_seg, const b200ot_piece* pieces,
                                               int32_t D);
/* b200ot_softmin_fwd on the listed blocks: out, lse2_out (N), out_old, alpha_old, beta as there */
B200OT_API int b200ot_softmin_fwd_blocks(const float* x, const float* y, const float* h_a, const float* h_b,
                                         float h_scale_b, const float* center, const float* out_old, float alpha_old,
                                         float beta, float* out, float* lse2_out, int64_t N, const int32_t* row_src,
                                         int64_t n_row_slots, const int32_t* col_src, int64_t n_col_slots,
                                         const b200ot_segment* seg, int64_t n_seg, const b200ot_piece* pieces,
                                         int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                         void* stream);
/* b200ot_softmin_bwd_x on the listed blocks (lse2: the forward's) */
B200OT_API int b200ot_softmin_bwd_x_blocks(const float* x, const float* y, const float* h_a, const float* h_b,
                                           float h_scale_b, const float* center, const float* lse2,
                                           const float* grad_out, float* grad_x, int64_t N, const int32_t* row_src,
                                           int64_t n_row_slots, const int32_t* col_src, int64_t n_col_slots,
                                           const b200ot_segment* seg, int64_t n_seg, const b200ot_piece* pieces,
                                           int32_t D, int32_t p, float eps, void* scratch, int64_t scratch_bytes,
                                           void* stream);

/* --- stages of the CUDA-core kernel convolutions (D <= B200OT_MAX_D), ranges mode: truncated block-sparse
 *     MMDs (kernel_multiscale, kernel_samples.py:177-271) and batched problems.  cols: gather-packed,
 *     b200ot_packed_cols_floats(n_slots, D, 2) floats.  part: (N) sums (backward = 0) or (N, width) sums
 *     (backward = 1; width = D + 1 for the gaussian kernel, D otherwise); partial sums of column shards add. --- */
B200OT_API int b200ot_kernel_conv_pack_gather(const float* y, const float* w, const float* center,
                                              const int32_t* src_index, int64_t n_slots, int32_t D, int32_t kind,
                                              float blur, float* cols_out, void* stream);
B200OT_API int b200ot_kernel_conv_partial_ranges(const float* x, const float* center, const float* cols,
                                                 const b200ot_segment* seg, int64_t n_seg,
                                                 const b200ot_piece* pieces, float* part, int64_t N, int32_t D,
                                                 int32_t kind, float blur, int32_t backward, int32_t variant,
                                                 void* stream);
/* out_i = sign(kind) * sum_s part[s*N + i] */
B200OT_API int b200ot_kernel_conv_finalize(const float* part, int32_t n_part, float* out, int64_t N, int32_t kind,
                                           void* stream);
/* grad_x from n_part sets of (N, width) row-gradient sums */
B200OT_API int b200ot_kernel_conv_bwd_finalize(const float* part, int32_t n_part, const float* x, const float* center,
                                               const float* grad_out, float* grad_x, int64_t N, int32_t D,
                                               int32_t kind, float blur, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Small problems: one launch per symmetric Sinkhorn iteration
 * replaces the four softmin calls of the loop body of sinkhorn_loop (sinkhorn_divergence.py:468-493) — and of its
 * initialisation (:461-465) and final gradient-carrying step (:612-623) — for B stacked problems
 * x:(B,N,D) y:(B,M,D) a_log:(B,N) b_log:(B,M) with N, M <= B200OT_SMALL_MAX_POINTS, D <= B200OT_MAX_D and any B >= 1
 * (a batch above 65535 elements, the grid's z limit, is enqueued as consecutive launches over slices of it):
 *     f_ba_out <- alpha_old f_ba + beta softmin(eps, (x, y), b_log + g_ab/eps)      (B,N)
 *     g_ab_out <- alpha_old g_ab + beta softmin(eps, (y, x), a_log + f_ba/eps)      (B,M)
 *     f_aa_out <- alpha_old f_aa + beta softmin(eps, (x, x), a_log + f_aa/eps)      (B,N)   (debiasing; nullable pair)
 *     g_bb_out <- alpha_old g_bb + beta softmin(eps, (y, y), b_log + g_bb/eps)      (B,M)
 * all four reading the OLD potentials (f_ba .. g_bb all null: h = log-weights, the initialisation; alpha_old = 0).
 * a_log / b_log are natural-log weights, or the weights themselves when weights_linear = 1.
 * Outputs must not alias inputs.  lse2_out (nullable): B*(2N+2M) floats [f_ba | g_ab | f_aa | g_bb], the log2-domain
 * log-sum-exp of every row, consumed by b200ot_sinkhorn_final_bwd_small:
 *     grad_x <- scale_out * ( go_f_ba[i] d softmin_xy / d x_i + go_f_aa[i] d softmin_xx / d x_i )     (B,N,D)
 *     grad_y <- scale_out * ( go_g_ab[j] d softmin_yx / d y_j + go_g_bb[j] d softmin_yy / d y_j )     (B,M,D)
 * with columns and potentials held constant (the reference's autograd contract); f_ba .. g_bb are the potentials
 * that entered the final step; go_* nullable (zero upstream gradient).
 * lo_hi (nullable, 2*D floats on the device: minima then maxima, as written by b200ot_cloud_extent): the coordinates are
 * taken relative to the mid-point of this box before they are scaled by the temperature — pass the box of the whole
 * batch, or the costs of clouds far from the origin lose the low bits of their differences.  Every call of one descent
 * and its gradient must see the same box.
 * ------------------------------------------------------------------------------------------- */
#define B200OT_SMALL_MAX_POINTS 65536
B200OT_API int b200ot_sinkhorn_iteration_small(const float* x, const float* y, const float* a_log, const float* b_log,
                                               const float* f_ba, const float* g_ab, const float* f_aa,
                                               const float* g_bb, float* f_ba_out, float* g_ab_out, float* f_aa_out,
                                               float* g_bb_out, float* lse2_out, int64_t B, int64_t N, int64_t M,
                                               int32_t D, int32_t p, float eps, float alpha_old, float beta,
                                               int32_t weights_linear, const float* lo_hi, void* stream);
/* The whole descent in ONE host call: initialisation at eps_list[0] (potentials <- damped softmins of the log-weights)
 * followed by one averaged symmetric update per temperature of eps_list (host array of n_eps doubles) — n_eps + 1
 * launches enqueued back to back, no Python / FFI round trip between them.  rho <= 0: balanced (damping 1), else
 * damping 1/(1 + eps/rho) per temperature (sinkhorn_divergence.py:56-58).  pots_a, pots_b: two scratch sets of
 * B*(2N+2M) floats [f_ba | g_ab | f_aa | g_bb] used as ping-pong buffers; *result_in_a tells which one holds the final
 * iterate.  weights_linear = 1: a, b are the weights themselves (log taken in the kernel, -100000 floor for a <= 0). */
B200OT_API int b200ot_sinkhorn_loop_small(const float* x, const float* y, const float* a, const float* b,
                                          int32_t weights_linear, const double* eps_list, int32_t n_eps, double rho,
                                          int32_t debias, float* pots_a, float* pots_b, int32_t* result_in_a,
                                          int64_t B, int64_t N, int64_t M, int32_t D, int32_t p,
                                          const float* lo_hi, void* stream);
B200OT_API int b200ot_sinkhorn_final_bwd_small(const float* x, const float* y, const float* a_log, const float* b_log,
                                               const float* f_ba, const float* g_ab, const float* f_aa,
                                               const float* g_bb, const float* lse2, const float* go_f_ba,
                                               const float* go_g_ab, const float* go_f_aa, const float* go_g_bb,
                                               float* grad_x, float* grad_y, int64_t B, int64_t N, int64_t M,
                                               int32_t D, int32_t p, float eps, float scale_out,
                                               const float* go_scale, int32_t weights_linear, const float* lo_hi,
                                               void* stream);
/* go_scale (nullable): (B,) per-problem factor applied to every go_* — the upstream gradient of the B loss values when
 * go_* hold d value / d potential as written by b200ot_sinkhorn_cost_small.
 *
 * sinkhorn_cost (sinkhorn_divergence.py:165-255) of B stacked small problems in one launch, one value per problem:
 *     rho <= 0 (balanced):  value = <a, f_ba - f_aa> + <b, g_ab - g_bb>
 *     rho  > 0:             value = <a, w (e^{-f_aa/rho} - e^{-f_ba/rho})> + <b, w (e^{-g_bb/rho} - e^{-g_ab/rho})>,
 *                           w = rho + eps/2
 * (f_aa = g_bb = NULL: no debiasing — <a, f_ba> + <b, g_ab>, resp. w (1 - e^{-f/rho}).)  Nullable outputs: go_* =
 * d value / d potential per point, phi (B,N) / psi (B,M) = d value / d a_i, d value / d b_j. */
B200OT_API int b200ot_sinkhorn_cost_small(const float* a, const float* b, const float* f_ba, const float* g_ab,
                                          const float* f_aa, const float* g_bb, int64_t B, int64_t N, int64_t M,
                                          float rho, float eps, float* value, float* go_f_ba, float* go_g_ab,
                                          float* go_f_aa, float* go_g_bb, float* phi, float* psi, void* stream);

/* value[b] = 1/2 <a, a_x> + 1/2 <b, b_y> - <a, b_x> (kernel_samples.py:139-146) from the outputs of
 * b200ot_kernel_mmd_small, one launch, fixed summation order. */
B200OT_API int b200ot_kernel_mmd_value_small(const float* a, const float* b, const float* a_x, const float* b_y,
                                             const float* b_x, int64_t B, int64_t N, int64_t M, float* value,
                                             void* stream);

/* Bounding box of the rows of x:(n,D) and y:(m,D) (m = 0: x alone), D <= B200OT_MAX_D: lo_hi[0..D) = minima,
 * lo_hi[D..2D) = maxima — the inputs of max_diameter (sinkhorn_divergence.py:96-112) in one launch.  scratch:
 * b200ot_cloud_extent_scratch_bytes() bytes, ZERO before its first use (the kernel leaves it reusable). */
B200OT_API int64_t b200ot_cloud_extent_scratch_bytes(void);
B200OT_API int b200ot_cloud_extent(const float* x, int64_t n, const float* y, int64_t m, int32_t D, float* lo_hi,
                                   void* scratch, int64_t scratch_bytes, void* stream);

/* Kernel norms on small clouds (same size limits): the matvecs of kernel_loss (kernel_samples.py:116-137) in one launch,
 *     a_x = K(x,x) a   b_y = K(y,y) b   b_x = K(x,y) b   a_y = K(y,x) a  (a_y nullable: only needed for potentials / d/db)
 * and the gradient of  value = 1/2 <a, a_x> + 1/2 <b, b_y> - <a, b_x>  w.r.t. both clouds, with the reference's
 * DoubleGrad / detach pattern (kernel_samples.py:43-54, :116-146), scaled by grad_value[batch], in one more. */
B200OT_API int b200ot_kernel_mmd_small(const float* x, const float* y, const float* a, const float* b, float* a_x,
                                       float* b_y, float* b_x, float* a_y, int64_t B, int64_t N, int64_t M, int32_t D,
                                       int32_t kind, float blur, void* stream);
B200OT_API int b200ot_kernel_mmd_bwd_small(const float* x, const float* y, const float* a, const float* b,
                                           const float* grad_value, float* grad_x, float* grad_y, int64_t B, int64_t N,
                                           int64_t M, int32_t D, int32_t kind, float blur, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Grid softmin  —  the separable soft-C-transform on (batch, N, N[, N]) images / volumes
 * replaces softmin_grid (src/geomloss/_legacy/utils.py:190-279), the operator of the image Sinkhorn loop
 * (src/geomloss/_legacy/sinkhorn_images.py:26-202):
 *   out <- alpha_old * out_old + beta * ( -eps * LSE over the whole grid of  h - |x - y|^p / (p eps) ),
 *   h = h_a + h_scale_b * h_b (h_b nullable), pixel coordinates arange(N)/N, p in {1, 2}, dim in {1, 2, 3}.
 * `out` must not alias an input (the per-axis passes run in place on it).  N <= 1024.
 * ------------------------------------------------------------------------------------------- */
B200OT_API int b200ot_softmin_grid(const float* h_a, const float* h_b, float h_scale_b, const float* out_old,
                                   float alpha_old, float beta, float* out, int64_t batch, int32_t N, int32_t dim,
                                   int32_t p, float eps, void* stream);

/* The same softmin (p = 2 only) on a (batch, sides[0][, sides[1][, sides[2]]]) grid with its own geometry per axis:
 * side sides[d] in 1..1024, pixel pitch pitch[d] > 0, and periodic[d] != 0 for an axis that wraps around (offsets n
 * become min(|n|, N_d - |n|)); `periodic` may be NULL (no periodic axis).  The three arrays are host memory, dim long.
 *   out <- alpha_old * out_old + beta * ( -eps * LSE_j ( h_j - |x_i - y_j|^2 / (2 eps) ) ),  x = (k + 1/2) pitch.
 * `out` must not overlap an input.  One launch per axis. */
B200OT_API int b200ot_softmin_grid_axes(const float* h_a, const float* h_b, float h_scale_b, const float* out_old,
                                        float alpha_old, float beta, float* out, int64_t batch, int32_t dim,
                                        const int32_t* sides, const float* pitch, const int32_t* periodic, float eps,
                                        void* stream);

/* The plan of that softmin applied to K value channels, w_ij = exp(h_j - |x_i - y_j|^2 / (2 eps)) on the same geometry:
 *   ell_i = log2 sum_j w_ij           (so -eps ln2 ell is b200ot_softmin_grid_axes of h with beta = 1),
 *   s_ki  = sum_j w_ij v_kj / sum_j w_ij,      0 where every w_ij is 0 (ell = -inf).
 * h = h_a + h_scale_b h_b (h_b nullable), (batch, *grid); v and s are channel-major, (K, batch, *grid).  Outputs must
 * not overlap an input or each other (the passes run in place on them).  One launch per axis and per slab of 4
 * channels; no scratch. */
B200OT_API int b200ot_grid_plan_apply(const float* h_a, const float* h_b, float h_scale_b, const float* v, float* ell,
                                      float* s, int64_t batch, int32_t K, int32_t dim, const int32_t* sides,
                                      const float* pitch, const int32_t* periodic, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Pipe-ceiling micro-benchmarks (used by bench.py to measure the MUFU / FP32 roofline of the
 * device it runs on; each launches one kernel doing `iters` dependent steps per thread and
 * returns the number of operations executed per thread-step through *ops_per_thread_iter).
 * ------------------------------------------------------------------------------------------- */
#define B200OT_UBENCH_MUFU_EX2 0
#define B200OT_UBENCH_FFMA 1
#define B200OT_UBENCH_FFMA2 2
B200OT_API int b200ot_ubench(int32_t which, int32_t iters, int32_t blocks, float* sink, int32_t* ops_per_thread_iter,
                  void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200OT_H_ */
