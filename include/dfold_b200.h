/* dfold_b200 — C ABI of the sm_90a (H100) DFOLDv2 score-network hot path.
 *
 * The reference (fudan-generative-vision/dynamicPDB) is pure Python/PyTorch and has no FFI of its own; the
 * boundary a maintainer binds is this shared library (libdfold_b200.so), loaded with ctypes by
 * dynamicpdb_b200/kernels.py.  Every entry point cites the reference code it replaces (paths relative to the
 * reference checkout).  INTEGRATION.md shows the ctypes stub and the import overlay.
 *
 * Conventions
 *   - all pointers are DEVICE pointers to dense fp32 (or bf16-plane, uint16_t) arrays unless noted;
 *   - every function returns 0 on success, non-zero on error; dfold_last_error() returns the message
 *     (thread-local, valid until the next call on that thread);
 *   - `stream` is a cudaStream_t; work is enqueued, never synchronised;
 *   - no function allocates device memory; workspaces are passed in by the caller.
 */
#ifndef DFOLD_B200_H
#define DFOLD_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

const char* dfold_last_error(void);
int dfold_abi_version(void);
/* Host-side helper: *id_out = id of the CUDA-graph capture `stream` is recording into, 0 when not capturing
 * (HOST pointer). */
int dfold_capture_id(void* stream, unsigned long long* id_out);
/* Development aid: non-NULL `buf` (DEVICE, 4 x int64 per CTA) makes every following tensor-core GEMM launch record per CTA
 * {mainloop cycles, consumer wait on operand stages, producer wait on a free stage, 0};
 * NULL switches it off. */
int dfold_debug_gemm_stats(long long* buf);

/* ------------------------------------------------------------------------------------------------------------
 * Split-precision tensor-core GEMM (wgmma, bf16 x 3, fp32 accumulate in registers) and its operand preparation.
 * Replaces every nn.Linear on the path (src/model/ipa_pytorch_dynamic.py:284-305,590,757-796;
 * src/model/Dfold_network_dynamic.py:444-445; openfold/model/structure_module.py:58-59,102-110) and the
 * ConvNet's eight Conv2d(5x5) (src/model/ipa_pytorch_dynamic.py:664-706).
 * ---------------------------------------------------------------------------------------------------------- */

/* x[R,C] fp32 (row stride ld) -> bf16 planes hi = bf16(x), lo = bf16(x - hi).
 *   hi/lo     : [R][ldo], columns [C, cpad) zero-filled           (nullable pair)
 *   hi_t/lo_t : [C][ldt] (transposed), columns [R, rpad) zeroed   (nullable pair)
 * pre_relu applies max(x,0) first; gate (nullable, row stride ldg) zeroes x where gate <= 0 (ReLU backward);
 * colsum (nullable, [C], pre-zeroed) receives the column sums of the gated input (bias gradient), added in a fixed
 * order so that they are the same from run to run.  With neither plane pair requested only the column sums run. */
int dfold_split2d(const float* x, long R, long C, long ld, int pre_relu, const float* gate, long ldg,
                  uint16_t* hi, uint16_t* lo, long ldo, long cpad,
                  uint16_t* hi_t, uint16_t* lo_t, long ldt, long rpad, float* colsum, void* stream);

/* dfold_split2d with the ReLU gate of a residual layer y = relu(...) + residual: x passes where the fp32 difference
 * out - residual is > 0 (out and residual both [R] rows of stride ldg, neither nullable).  Planes and column sums are
 * those dfold_split2d gives for gate = out - residual computed beforehand. */
int dfold_split2d_residual_gate(const float* x, long R, long C, long ld, int pre_relu, const float* out,
                                const float* residual, long ldg, uint16_t* hi, uint16_t* lo, long ldo, long cpad,
                                uint16_t* hi_t, uint16_t* lo_t, long ldt, long rpad, float* colsum, void* stream);

/* Conv weight w[O][I][T] (the reference layout [C_out, C_in, 5, 5], T = 25) ->
 *   forward planes  f_hi/f_lo [T][O][ldi]           (K = input channel)
 *   dgrad planes    d_hi/d_lo [T][I][ldo], tap order flipped (nullable pair)
 * 1 <= T <= 56: a CTA stages a 32 x 32 x T tile in shared memory.  Only columns [0, I) / [0, O) of each plane row are
 * written; the caller zero-fills the padding up to ldi / ldo. */
int dfold_conv_weight_prep(const float* w, int O, int I, int T, uint16_t* f_hi, uint16_t* f_lo, long ldi,
                           uint16_t* d_hi, uint16_t* d_lo, long ldo, void* stream);

/* g[T][O][I] -> out[O][I][T]: weight gradient back to the parameter layout; accumulate != 0 adds into `out` (the shared
 * ConvNet's four weight gradients of a step land in the gradient buffer without separate add passes). */
int dfold_taps_to_param(const float* g, int O, int I, int T, float* out, int accumulate, void* stream);

/* for f in [0, F_out):
 * out[f*Nr + n, c] = act(alpha * sum_{tf,tn,k} A[f + f_start + tf - taps_f/2, n + tn - taps_n/2, k] * B[tf*taps_n+tn][c][k]
 *                        + bias[c]) + beta * residual[f*Nr + n, c]
 * A planes [F][Nr][lda] (zero outside the image: the 5x5 halo is a TMA out-of-bounds fill), B planes
 * [taps][n_out][ldb].  taps_f = taps_n = 1 is a plain linear layer (x @ W^T).  act: 0 none, 1 ReLU, 2 SiLU.
 * lda, ldb multiples of 8.  bias / residual nullable.  F_out = F, f_start = 0 is the plain convolution; F_out < F with
 * f_start = F - F_out computes only the last F_out frames (dead-frame pyramid), f_start < 0 is its data gradient. */
int dfold_gemm_bf16x3(const uint16_t* a_hi, const uint16_t* a_lo, long F, long F_out, int f_start, long Nr, long K, long lda,
                      const uint16_t* b_hi, const uint16_t* b_lo, long n_out, long ldb, int taps_f, int taps_n,
                      float* out, long ldo, const float* bias, const float* residual, long ldr,
                      float alpha, float beta, int act, void* stream);

/* dfold_gemm_bf16x3 on output tiles bn = 64 or 128 columns wide (dfold_gemm_bf16x3 picks the width itself).  Any other
 * width is rejected.  Each output element is the same one-CTA, fixed-order k loop at either width. */
int dfold_gemm_bf16x3_bn(const uint16_t* a_hi, const uint16_t* a_lo, long F, long F_out, int f_start, long Nr, long K,
                         long lda, const uint16_t* b_hi, const uint16_t* b_lo, long n_out, long ldb, int taps_f, int taps_n,
                         float* out, long ldo, const float* bias, const float* residual, long ldr,
                         float alpha, float beta, int act, int bn, void* stream);

/* Weight gradient: out[t][m][n] = alpha * sum_{f,j} A[f][j][m] * B[f + b_f_add + tf - taps_f/2][j + tn - taps_n/2][n]
 * A planes [F][Nr][lda] (gated output gradient, m = output channel), B planes [Fb][Nr][ldb] (layer input,
 * n = input channel) — the same pixel-major planes as above, consumed MN-major by the tensor core; out [taps][M][ldo]. */
int dfold_gemm_wgrad_bf16x3(const uint16_t* a_hi, const uint16_t* a_lo, long M, long lda,
                            const uint16_t* b_hi, const uint16_t* b_lo, long Nn, long ldb,
                            long F, long Fb, int b_f_add, long Nr, int taps_f, int taps_n,
                            float* out, long ldo, float alpha, void* stream);

/* dfold_gemm_wgrad_bf16x3 on output tiles bn = 64 or 128 columns wide; any other width is rejected. */
int dfold_gemm_wgrad_bf16x3_bn(const uint16_t* a_hi, const uint16_t* a_lo, long M, long lda,
                               const uint16_t* b_hi, const uint16_t* b_lo, long Nn, long ldb,
                               long F, long Fb, int b_f_add, long Nr, int taps_f, int taps_n,
                               float* out, long ldo, float alpha, int bn, void* stream);

/* dfold_gemm_bf16x3_bn over W >= 1 stacked windows of F frames each, each convolved on its own (the reference's
 * nn.Conv2d stack, src/model/ipa_pytorch_dynamic.py:664-706, run once per window, as `world_size * W` one-window ranks
 * of the released recipe train).  A planes [W][F][Nr][lda]; for w in [0, W), f in [0, F_out):
 *   out[(w*F_out + f)*Nr + n, c] = act(alpha * sum_{tf,tn,k} A[w][f + f_start + tf - taps_f/2][n + tn - taps_n/2][k]
 *                                      * B[tf*taps_n+tn][c][k] + bias[c]) + beta * residual[(w*F_out + f)*Nr + n, c]
 * with A zero outside window w (the 4-D map's out-of-bounds fill).  Every output element is the same one-CTA k loop as
 * dfold_gemm_bf16x3_bn on window w alone, so each window's result equals that call's bit for bit. */
int dfold_gemm_bf16x3_windows(const uint16_t* a_hi, const uint16_t* a_lo, long W, long F, long F_out, int f_start, long Nr,
                              long K, long lda, const uint16_t* b_hi, const uint16_t* b_lo, long n_out, long ldb,
                              int taps_f, int taps_n, float* out, long ldo, const float* bias, const float* residual,
                              long ldr, float alpha, float beta, int act, int bn, void* stream);

/* Weight gradient over W >= 1 stacked windows (src/model/ipa_pytorch_dynamic.py:664-706, the gradient of the Conv2d
 * weights summed over W windows):
 *   out[t][m][n] = alpha * sum_w sum_{f,j} A[w][f][j][m] * B[w][f + b_f_add + tf - taps_f/2][j + tn - taps_n/2][n]
 * A planes [W][F][Nr][lda], B planes [W][Fb][Nr][ldb], B zero outside window w.  One launch; the k loop runs window by
 * window with the promotion points of one F*W-frame reduction, so it differs from the sum of W per-window gradients in
 * fp32 rounding only.  bn = 64 or 128. */
int dfold_gemm_wgrad_bf16x3_windows(const uint16_t* a_hi, const uint16_t* a_lo, long M, long lda,
                                    const uint16_t* b_hi, const uint16_t* b_lo, long Nn, long ldb,
                                    long W, long F, long Fb, int b_f_add, long Nr, int taps_f, int taps_n,
                                    float* out, long ldo, float alpha, int bn, void* stream);

/* Batched K-major GEMM (no taps).  For every row tile of "frame" b in [0, n_batches), hb = b % bmod:
 *   out[(b / o_f_div) * Nr + n, hb * o_col_bstride + c] =
 *       alpha * sum_k A[b / a_f_div][n][hb * a_k_bstride + k] * B[hb * b_z_bstride][c][b_k_ofs + hb * b_k_bstride + k]
 * A planes [a_frames][Nr][lda] (a_cols valid columns), B planes [b_z][b_rows][ldb] (b_cols valid columns).
 * Used for the IPA value aggregation O = P V (src/model/ipa_pytorch_dynamic.py:452-454, written straight into the
 * concat buffer) and for dP = dO V^T in its backward. */
int dfold_gemm_bf16x3_batched(const uint16_t* a_hi, const uint16_t* a_lo, long a_frames, long Nr, long a_cols, long lda,
                              long n_batches, int bmod, int a_f_div, long a_k_bstride, long K,
                              const uint16_t* b_hi, const uint16_t* b_lo, long b_z, long b_rows, long b_cols, long ldb,
                              long b_k_ofs, long b_k_bstride, int b_z_bstride, long n_out,
                              float* out, long ldo, long out_rows, int o_f_div, long o_col_bstride, float alpha,
                              void* stream);

/* Batched MN-major GEMM (the reduction runs over ROWS of both operands).  For z in [0, zcount):
 *   out[z][m][n] = alpha * sum_{f < Fk} sum_j A[f*a_f_mul + z*a_z_mul][j][m] * B[f*b_f_mul + z*b_z_mul][j][z*b_n_zmul + n]
 * A planes: dims (M, a_mid, a_outer) with element strides (lda, a_ostride); B likewise.  Used for dV = P^T dO, dV_pts, dZ
 * in the IPA backward. */
int dfold_gemm_wgrad_bf16x3_batched(const uint16_t* a_hi, const uint16_t* a_lo, long M, long a_mid, long a_outer, long lda,
                                    long a_ostride, const uint16_t* b_hi, const uint16_t* b_lo, long b_cols, long b_mid,
                                    long b_outer, long ldb, long b_ostride, long Nn, long Fk, long Nr, int zcount,
                                    int a_f_mul, int a_z_mul, int b_f_mul, int b_z_mul, long b_n_zmul,
                                    float* out, long ldo, long out_z_stride, float alpha, void* stream);

/* Generic strided fp32 GEMM on CUDA cores for shapes below the tensor-core tile (K in {1,3,7,14}, N in {6,8,14}),
 * the once-per-sample q.k logits and the reductions of the IPA backward.
 * C[b,b2][m][n] = act(alpha * sum_k A[m][k] * B[n][k] + bias[n]) + beta * R[m][n]; strides in elements
 * (*_rs row, *_cs column, *_bs outer batch, *_bs2 inner batch).  ksplit > 1: split-K with atomic accumulation into
 * a pre-zeroed C (no bias / residual / activation; the last bits then vary from run to run). */
int dfold_sgemm(const float* A, long a_rs, long a_cs, long a_bs, long a_bs2,
                const float* B, long b_rs, long b_cs, long b_bs, long b_bs2,
                float* C, long c_rs, long c_cs, long c_bs, long c_bs2,
                const float* R, long r_rs, long r_cs, long r_bs, long r_bs2,
                const float* bias, int batch, int batch2, int M, int N, int K, float alpha, float beta, int act,
                int pre_relu, int ksplit, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Norms
 * ---------------------------------------------------------------------------------------------------------- */
/* MyLayerNorm (src/model/ipa_pytorch_dynamic.py:709-724): y = (x - mean) / sqrt(var_unbiased + eps) with ONE
 * mean / variance over all n elements, optional fused SiLU.  stats[2] = {mean, rstd}; workspace >= 2050 doubles. */
int dfold_global_layernorm_fwd(const float* x, float* y, float* stats, double* workspace, long n, float eps, int silu,
                               void* stream);
int dfold_global_layernorm_bwd(const float* x, const float* dy, const float* stats, double* workspace, float* dx,
                               long n, int silu, void* stream);
/* MyLayerNorm (src/model/ipa_pytorch_dynamic.py:709-724) applied to each of `segments` consecutive tensors of n elements
 * on its own (one window each), in one launch per pass: stats [segments][2]; workspace >= segments * 2050 doubles.
 * Each segment is reduced with the partition and order dfold_global_layernorm_fwd / _bwd use for n elements, so its
 * result equals that call's bit for bit. */
int dfold_global_layernorm_seg_fwd(const float* x, float* y, float* stats, double* workspace, long n, int segments,
                                   float eps, int silu, void* stream);
int dfold_global_layernorm_seg_bwd(const float* x, const float* dy, const float* stats, double* workspace, float* dx,
                                   long n, int segments, int silu, void* stream);
/* nn.LayerNorm / openfold LayerNorm over the last axis (openfold/model/primitives.py:170-199). stats [rows][2].
 * dw, db must be pre-zeroed; they are accumulated in a fixed order, so they are the same from run to run. */
int dfold_row_layernorm_fwd(const float* x, const float* w, const float* b, float* y, float* stats, long rows, int C,
                            float eps, void* stream);
int dfold_row_layernorm_bwd(const float* x, const float* w, const float* dy, const float* stats, float* dx, float* dw,
                            float* db, long rows, int C, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Rigid-frame algebra (openfold/utils/rigid_utils.py); quaternions are (w,x,y,z), 3x3 math in registers.
 * ---------------------------------------------------------------------------------------------------------- */
/* quat_to_rot :185-205 — [n,4] -> [n,3,3], not normalised. */
int dfold_quat_to_rot_fwd(const float* quat, float* rot, long n, void* stream);
int dfold_quat_to_rot_bwd(const float* quat, const float* drot, float* dquat, long n, void* stream);
/* Rigid.apply :1104-1116 (inverse=0: R p + t) / Rigid.invert_apply :1118-1130 (inverse=1: R^T (p - t)).
 * quat [F,N,4], trans [F,N,3], pts [F or 1][N][m][3] (pts_fstride = 0 shares one point set over all F), out [F,N,m,3]. */
int dfold_rigid_apply_fwd(const float* quat, const float* trans, const float* pts, long pts_fstride, float* out,
                          long F, long N, int m, int inverse, void* stream);
int dfold_rigid_apply_bwd(const float* quat, const float* trans, const float* pts, long pts_fstride, const float* dout,
                          float* dpts, float* dquat, float* dtrans, long F, long N, int m, int inverse, void* stream);
/* Rigid.compose_q_update_vec :1039-1063 (+ :587-616, :266-275): q' = normalise(q + m q*(0,u)), t' = t + m R(q) v,
 * upd6 = (u, v); mask [n] nullable. */
int dfold_compose_q_update_fwd(const float* quat, const float* trans, const float* upd6, const float* mask,
                               float* quat_out, float* trans_out, long n, void* stream);
int dfold_compose_q_update_bwd(const float* quat, const float* upd6, const float* mask, const float* dquat_out,
                               const float* dtrans_out, float* dquat, float* dtrans, float* dupd6, long n, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Fused invariant point attention core.
 * Replaces src/model/ipa_pytorch_dynamic.py:402-504 (dfold=1) and openfold/model/structure_module.py:315-428
 * (dfold=0): point-distance term on coordinate differences + pair bias + mask + softmax + value / value-point /
 * pair aggregation + local-frame inverse transform + norms -> the concat buffer fed to linear_out.
 *   logit0 [Fl,H,N,N]   q.k/sqrt(3C) + b/sqrt(3)        (frame stride 0 when shared by all frames)
 *   kv     [Fs,N,H,2C]  per head [K | V]                 (frame stride 0 when shared)
 *   q_pts  [F,N,H,Pq,3], kv_pts [F,N,H,Pq+Pv,3]          global-frame points
 *   pair   [Fz,N,N,Cp]                                   (frame stride 0 when shared)
 *   quat [F,N,4], trans [F,N,3], mask [F,N], gamma [H] = softplus(head_weights) * sqrt(1/(3*Pq*9/2))
 *   out_cat [F,N,D], D = H*(C + 8*Pv + Cp) (dfold) or H*(C + 4*Pv + Cp); lse [F,H,N] (saved for backward)
 * ---------------------------------------------------------------------------------------------------------- */
int dfold_ipa_attn_fwd(const float* logit0, long logit0_fstride, const float* kv, long kv_fstride, const float* q_pts,
                       const float* kv_pts, const float* pair, long pair_fstride, const float* quat, const float* trans,
                       const float* mask, const float* gamma, int F, int N, int H, int C, int Pq, int Pv, int Cp,
                       int dfold, float inf, float eps, float* out_cat, float* lse, void* stream);
/* Backward: writes d_og [F,N,H,Pv,3], delta [F,H,N], P and dS [H,F,N,N] (workspaces the caller reduces into dv / dz /
 * d-logits with dfold_sgemm), dq_pts [F,N,H,Pq,3], the key-point part of dkv_pts [F,N,H,Pq+Pv,3], dquat / dtrans of
 * the local-frame transform, and per-CTA partials of dgamma: dgamma [H][F*N], zeroed by the caller, whose row h sums to
 * d(gamma_h) (added by the caller in order: no atomics). */
int dfold_ipa_attn_bwd(const float* logit0, long logit0_fstride, const float* kv, long kv_fstride, const float* q_pts,
                       const float* kv_pts, const float* pair, long pair_fstride, const float* quat, const float* trans,
                       const float* mask, const float* gamma, int F, int N, int H, int C, int Pq, int Pv, int Cp,
                       int dfold, float inf, float eps, const float* out_cat, const float* lse, const float* dcat,
                       float* d_og, float* delta, float* P, float* dS, float* dq_pts, float* dkv_pts, float* dquat,
                       float* dtrans, float* dgamma, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Tensor-core path for the preset-A head geometry (csrc/ipa_fused.cu, csrc/ipa_v2.cu): the probabilities are
 * materialised once as bf16 hi/lo planes P[F,H,N,ldp]; O = P V, dP, dV, dV_pts, dZ run on dfold_gemm_bf16x3*_batched.
 * ---------------------------------------------------------------------------------------------------------- */
/* Fused forward core (csrc/ipa_fused.cu), frame-shared logit0 [H,N,N] and pair [N,N,Cp]: one kernel does the point
 * distances (exact fp32), the exact two-pass softmax, the pair and value-point aggregations, the local-frame transform and
 * the concat layout; p_hi / p_lo receive the bf16 hi/lo probability planes, which feed the P V GEMM and the backward GEMMs:
 * columns [0, H*C) of the concat buffer are left to dfold_gemm_bf16x3_batched.  H=8, Pq=8, Pv=12, Cp=32.
 * Replaces src/model/ipa_pytorch_dynamic.py:402-504. */
int dfold_ipa_fused_fwd(const float* logit0, const float* q_pts, const float* kv_pts, const float* pair, const float* quat,
                        const float* trans, const float* mask, const float* gamma, uint16_t* p_hi, uint16_t* p_lo, long ldp,
                        int F, int N, int H, int C, int Pq, int Pv, int Cp, int dfold, float inf, float eps, float* out_cat,
                        void* stream);
/* Development aid: per-CTA cycle counters of the next dfold_ipa_fused_fwd launches (16 x int64 per CTA; null = off). */
int dfold_debug_ipa_stats(long long* buf);
/* Epilogue backward: d_og [F,N,H,Pv,3], delta [F,H,N], dquat [F,N,4], dtrans [F,N,3]. */
int dfold_ipa_pre_bwd(const float* quat, const float* trans, int F, int N, int H, int C, int Pv, int Cp, int dfold,
                      const float* out_cat, const float* dcat, float* d_og, float* delta, float* dquat, float* dtrans,
                      void* stream);
/* dS = P (dP + d_og.v_pts + dO_pair.z - delta) [F,H,N,N] and dgamma partials [H][F*N] as dfold_ipa_attn_bwd, for Pq = 8
 * (Pv a multiple of 4); q_pts [F,N,H,Pq,3], kv_pts [F,N,H,Pq+Pv,3], p_hi / p_lo the forward's probability planes.
 * Tz = the dO_pair.z term precomputed as [N(i)][F*H][N(j)] by dfold_gemm_bf16x3_batched; Tog = the value-point term
 * d_og.v_pts precomputed as [F,H,N,N] the same way.  The caller computes the point gradients as contractions over dS. */
int dfold_ipa_ds_bwd(const float* q_pts, const float* kv_pts, const uint16_t* p_hi, const uint16_t* p_lo, long ldp, int F,
                     int N, int H, int Pq, int Pv, const float* delta, const float* dP, const float* Tz, const float* Tog,
                     float* dS, float* dgamma, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Score epilogue (csrc/epilogue.cu), one warp per residue, no [n,L] temporaries, no host synchronisation.
 * Replaces src/data/se3_diffuser.py:115-125 (calc_trans_score / calc_rot_score), src/data/utils.py:589-606
 * (quat_to_rotvec), src/data/so3_diffuser.py:274-305 (torch_score, use_cached_score=False) -> :9-49 (igso3_expansion),
 * :71-117 (score), :192-199 + :183-190 (sigma(t) snapped to the discrete grid, done on the device instead of
 * du.move_to_np(t)), src/data/r3_diffuser.py:42,169-177.
 *   q_pred / q_t [n,4] (w,x,y,z): predicted (rots_0) and noised (rots_t) rotations; x_pred / x_t [n,3] translations,
 *   x_pred BEFORE the model's unscale (divided by ipa_scale inside); t: DEVICE double scalar; sigma_grid [G] doubles;
 *   mask [n] or NULL.  rot_score [n,3] double; trans_score [n,3] double (trans_is_f64) or float.  Either output may be
 *   NULL.  Backward: d_rot_score / d_trans_score may be NULL (treated as zero); dq_pred [n,4], dx_pred [n,3].
 * ---------------------------------------------------------------------------------------------------------- */
int dfold_score_fwd(const float* q_pred, const float* q_t, const float* x_pred, const float* x_t, const double* t,
                    const double* sigma_grid, int G, double max_sigma, double min_sigma, double min_b, double max_b,
                    float r3_scale, float ipa_scale, const float* mask, int L, long n,
                    double* rot_score, void* trans_score, int trans_is_f64, void* stream);
int dfold_score_bwd(const float* q_pred, const float* q_t, const float* x_pred, const float* x_t, const double* t,
                    const double* sigma_grid, int G, double max_sigma, double min_sigma, double min_b, double max_b,
                    float r3_scale, float ipa_scale, const float* mask, int L, long n,
                    const double* d_rot_score, const void* d_trans_score, int trans_is_f64,
                    float* dq_pred, float* dx_pred, void* stream);

/* Structure epilogue: backbone frame o per-residue-type default frames o torsion rotations -> 8 rigid groups ->
 * idealised atom14 -> atom37 (openfold/utils/feats.py:165-228, src/data/all_atom.py:114-154,
 * src/model/Dfold_network_dynamic.py:574-594).  rot: [n,4] quaternion (un-normalised allowed: |q|^2 R, as
 * quat_to_rot) or, rot_is_matrix, [n,9]; alpha [n,7,2] (sin, cos); aatype [n] int64; tables as dumped from
 * openfold/np/residue_constants.py.  Outputs (each may be NULL): frames44 [n,8,4,4], atom14 [n,14,3], atom37 [n,37,3]. */
int dfold_frames_to_atoms_fwd(const float* rot, int rot_is_matrix, const float* trans, const float* alpha, const long* aatype,
                              const float* default_frames, const long* atom14_group, const float* atom14_mask,
                              const float* atom14_pos, const long* atom37_to_atom14, const float* atom37_mask,
                              float* frames44, float* atom14, float* atom37, long n, void* stream);

/* Quaternion product a (x) b (openfold/utils/rigid_utils.py:254-263); b_is_vec: b is [n,3], the pure quaternion (0, v)
 * (:266-275).  Backward: da = g (x) conj(b), db = conj(a) (x) g; da / db may be NULL. */
int dfold_quat_mul_fwd(const float* a, const float* b, float* out, long n, int b_is_vec, void* stream);
int dfold_quat_mul_bwd(const float* a, const float* b, const float* dout, float* da, float* db, long n, int b_is_vec, void* stream);
/* Rotation-matrix frames: for every left frame ia < n_a and its `rep` consecutive right operands ib = ia*rep + j
 *   rot_out[ib] = rot_a[ia] rot_b[ib]                 (rot_b / rot_out may be NULL)
 *   trans_out[ib] = rot_a[ia] trans_b[ib] + trans_a[ia]   (inverse: rot_a^T (trans_b - trans_a); trans_* may be NULL)
 * = rot_matmul :22, rot_vec_mul :82, Rotation.compose_r/apply/invert_apply :618-702, Rigid.compose :1065,
 * Rigid.apply / invert_apply :1104-1130 and the translation of Rigid.invert :1132. */
int dfold_rot_compose_fwd(const float* rot_a, const float* trans_a, const float* rot_b, const float* trans_b,
                          float* rot_out, float* trans_out, long n_a, int rep, int inverse, void* stream);
int dfold_rot_compose_bwd(const float* rot_a, const float* trans_a, const float* rot_b, const float* trans_b,
                          const float* drot_out, const float* dtrans_out, float* drot_a, float* dtrans_a,
                          float* drot_b, float* dtrans_b, long n_a, int rep, int inverse, void* stream);

/* One reverse-diffusion step t -> t - dt on the device, one block per trajectory frame (src/data/se3_diffuser.py:160-215,
 * src/data/so3_diffuser.py:329-365, src/data/r3_diffuser.py:106-157; replaces the numpy / scipy round trip of
 * se3_diffuser.py:11-29).  q_t [F,N,4], x_t [F,N,3] the current noised frames; scores as produced by dfold_score_fwd;
 * z_rot / z_trans [F,N,3] standard-normal draws (the caller owns the random stream); mask [F,N] 0/1 diffuse mask or NULL;
 * g_rot = so3 diffusion coefficient g(t), g_trans = sqrt(b(t)), b_t = b(t); centre-of-mass removal over each frame.
 * Writes unit quaternions q_out [F,N,4] (q_t (x) Exp(perturbation), right multiplication) and x_out [F,N,3]. */
int dfold_reverse_step(const float* q_t, const float* x_t, const double* rot_score, const void* trans_score, int trans_is_f64,
                       const float* z_rot, const float* z_trans, const float* mask, double g_rot, double g_trans, double b_t,
                       double dt, double noise_scale, double r3_scale, int center, int diffuse_rot, int diffuse_trans,
                       float* q_out, float* x_out, long F, long N, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Forward diffusion of a training window (csrc/diffuse.cu): the noising step of the data loader
 * (src/data/Dfold_data_loader_dynamic.py:332-349) on the device.
 * ---------------------------------------------------------------------------------------------------------- */
/* IGSO(3) inverse-cdf tables in fp64, one CTA per sigma row (src/data/so3_diffuser.py:132-180): for sigma_grid [num_sigma]
 * (discrete_sigma) and omega_j = (j+1) pi / num_omega, cdf [num_sigma][num_omega] = cumsum(pdf) / num_omega * pi with
 * pdf = igso3_expansion (:9-49, L terms) * (1 - cos omega) / pi, and score_scaling [num_sigma] = sqrt(|sum sn^2 pdf /
 * sum pdf|) / sqrt(3) with sn the score norms of :71-117.  Sums run in a fixed order: equal inputs give equal bits.
 * Needs (L + 2 num_omega) * 8 B <= 227 KB. */
int dfold_igso3_tables(const double* sigma_grid, int num_sigma, int num_omega, int L, double* cdf, double* score_scaling,
                       void* stream);
/* SE3Diffuser.forward_marginal (src/data/se3_diffuser.py:47-110) of n = F*N frames, one warp per frame: rigids_0 [n,7]
 * (w,x,y,z, trans) at time *t (device scalar) -> rigids_t [n,7] fp32 (unit quaternion with w >= 0), rot_score /
 * trans_score [n,3] fp64, *rot_scaling / *trans_scaling (device scalars).  Rotation: so3_diffuser.py:215-251, :274-327
 * (axis z_axis / |z_axis|, angle np.interp(u, cdf[sigma_idx(t)], omega), fp64 score with L terms, R_t = R_0 Exp(v));
 * translation: r3_diffuser.py:81-104, :159-177 (VP-SDE marginal and score in scaled units, x_t returned unscaled).
 * Draws are inputs: z_axis [n,3], u [n] in [0,1), z_trans [n,3], fp64.  mask [n] (0/1) or NULL: scores multiplied by it,
 * translations blended, rotations of mask-0 frames copied from rigids_0 (se3_diffuser.py:86-101).  diffuse_rot /
 * diffuse_trans = 0 keep that part of rigids_0 with zero score and scaling 1 (:65-84).  ref_mode != 0 is
 * SE3Diffuser.sample_ref (:217-280) with the dynamics layout: identity rotation and x_0 = 0, trans = z_trans /
 * r3_scale, rigids_0 / mask / scores / scalings unused.  No host reads: graph-capturable. */
int dfold_forward_marginal(const float* rigids_0, const double* z_axis, const double* u, const double* z_trans,
                           const float* mask, const double* t, const double* sigma_grid, const double* cdf,
                           const double* score_scaling, int num_sigma, int num_omega, int L, double max_sigma,
                           double min_sigma, double min_b, double max_b, float r3_scale, int diffuse_rot,
                           int diffuse_trans, int ref_mode, float* rigids_t, double* rot_score, double* trans_score,
                           double* rot_scaling, double* trans_scaling, long n, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Training loss (csrc/loss.cu), SURVEY.md 8 f3: value and gradients of Experiment.loss_fn after the model call
 * (train_DFOLD_dynamics.py:1206-1400; torsion term openfold/utils/loss.py:52-76) in one kernel.  All tensors fp64;
 * per-residue inputs are those of the LAST frame ([N,...]), the masks cover all nf frames, t / rot_scaling are device
 * scalars.  out[8] = {loss, rot, trans, torsion (normalised), rot, trans, torsion, final (per-frame)};
 * d_ang [N,7,2], d_rs [N,3], d_x [N,3] = d out[0] / d (angles, rot_score, translation).
 * ---------------------------------------------------------------------------------------------------------- */
int dfold_loss_fwd(const double* ang, const double* a_gt, const double* a_alt, const double* a_mask, const double* rs,
                   const double* gt_rot, const double* x, const double* x0, const double* res_mask, const double* fixed_mask,
                   const double* t, const double* rot_scaling, int nf, int N, double w_tor, double w_rot, double w_trans,
                   double t_thr, int rot_on, int separate, double* out, double* d_ang, double* d_rs, double* d_x, void* stream);
/* Auxiliary structure losses (csrc/aux_loss.cu), the backbone-atom MSE and the < 6 A pair-distance loss of
 * Experiment.loss_fn (train_DFOLD_dynamics.py:1316-1364, normalised as :1374-1375), over EVERY frame, in two launches and
 * no O((5N)^2) buffer.  pred_atom37 / gt_atom37 [nf,N,37,3] fp32 (atoms 0..4 = N, CA, C, CB, O read); masks [nf,N] fp64;
 * t[f * t_stride] (t_stride 0 or 1) gates frame f by t < t_bb / t < t_dm on the device.  work: nf * ceil(5N / 128) * 5
 * fp64.  out[2 + 2 nf] = {bb_atom_loss, dist_mat_loss (normalised), bb_atom_loss[nf], dist_mat_loss[nf]};
 * d_bb / d_dm [nf,N,5,3] fp64 = d out[0] / d pred and d out[1] / d pred (atoms 0..4).  nf <= 2048. */
int dfold_aux_loss_fwd(const float* pred_atom37, const float* gt_atom37, const double* res_mask, const double* fixed_mask,
                       const double* t, int t_stride, int nf, int N, double w_bb, double t_bb, double w_dm, double t_dm,
                       double w_aux, double* work, double* out, double* d_bb, double* d_dm, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Input featurisation of a trajectory window (csrc/featurize.cu), SURVEY.md 8 f4: atom37 coordinates [nf,N,37,3] ->
 * rigids_0 [nf,N,7] (backbone frame as quaternion wxyz + CA; replaces atom37_to_frames group 0 + rot_to_quat's CPU
 * eigh, openfold/data/data_transforms.py:755-842, openfold/utils/rigid_utils.py:208-227), torsion sin/cos, the
 * pi-periodic alternative and the mask [nf,N,7,(2)] in fp64 (data_transforms.py:923-1088), as the reference loader
 * computes them per sample on the host (src/data/Dfold_data_loader_dynamic.py:192-259, :323-330).
 * Tables: chi_idx [21,4,4] int64, chi_mask / chi_pi [21,4] fp32 (dynamicpdb_b200/data/residue_tables.npz).
 * ---------------------------------------------------------------------------------------------------------- */
int dfold_featurize_window(const float* pos, const float* atom_mask, const long* aatype, const long* chi_idx,
                           const float* chi_mask, const float* chi_pi, int nf, int N, float* rigids, double* tor, double* alt,
                           double* tmask, void* stream);

/* Adam (amsgrad) of the reference trainer (torch.optim.Adam(amsgrad=True), train_DFOLD_dynamics.py:412) in one pass over
 * flat fp32 buffers of n elements (n % 4 == 0); `step` is a device float, incremented by the call when tick != 0 (graph
 * capturable; a caller that updates the buffers chunk by chunk ticks once per optimizer step);
 * the gradient is multiplied by grad_scale on the fly (1 / world_size after a summing all-reduce). */
int dfold_adam_amsgrad(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq, long n,
                       float* step, int tick, float lr, float beta1, float beta2, float eps, float grad_scale, void* stream);
/* Global-norm gradient clipping, the commented-out torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm) of
 * Experiment.update_fn (train_DFOLD_dynamics.py:665), with torch's norm_type=2 and error_if_nonfinite=False, applied to the
 * data-parallel mean grad_scale * grad of a flat fp32 buffer of n elements (n % 4 == 0).  Writes the DEVICE scalars
 * total = ||grad_scale * grad||_2 (clip_grad_norm_'s return value) and coef = min(max_norm / (total + 1e-6), 1) in fp32,
 * NaN when total is NaN and 0 when it is inf, as torch computes them; the gradient is not modified.  The sum of squares
 * runs in fp64 in an order that depends on n only (the same bits on every run, device and rank).  max_norm > 0;
 * max_norm = inf gives coef 1 for any finite total.  partial: workspace of at least 1024 doubles. */
int dfold_grad_norm(const float* grad, long n, float grad_scale, float max_norm, double* partial, float* total, float* coef,
                    void* stream);
/* dfold_adam_amsgrad on the clipped gradient (grad * grad_scale) * (*coef), the order of DDP's mean followed by
 * clip_grad_norm_'s mul_(coef) (train_DFOLD_dynamics.py:665); coef is a DEVICE scalar (dfold_grad_norm's output), so no
 * extra pass over the gradient is made.  *coef == 1 gives the bits of dfold_adam_amsgrad. */
int dfold_adam_amsgrad_clip(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq, long n,
                            float* step, int tick, float lr, float beta1, float beta2, float eps, float grad_scale,
                            const float* coef, void* stream);
/* dfold_adam_amsgrad (coef NULL) or dfold_adam_amsgrad_clip (coef non-NULL) with the learning rate read from the DEVICE
 * fp32 scalar *lr (dfold_lr_schedule's output), so a captured step follows a schedule.  The same kernel: *lr equal to
 * fp32(x) gives the bits of the by-value call with lr = x. */
int dfold_adam_amsgrad_dlr(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq, long n,
                           float* step, int tick, const float* lr, float beta1, float beta2, float eps, float grad_scale,
                           const float* coef, void* stream);
/* The learning rate of AlphaFoldLRScheduler.get_lr (openfold/utils/lr_schedulers.py:64-82, imported by the reference
 * trainer, train_DFOLD_dynamics.py:56,652) at last_epoch = s = *step (the DEVICE step counter of dfold_adam_amsgrad, read
 * before the step's tick), written to the DEVICE fp32 scalar *lr by one thread:
 *   base_lr + s / warmup_no_steps * max_lr                                                          s <= warmup_no_steps
 *   max_lr * decay_factor ** ((s - start_decay_after_n_steps) // decay_every_n_steps + 1)       s > start_decay_after_n_steps
 *   max_lr                                                                                         otherwise
 * evaluated in fp64 as Python evaluates it, then rounded to fp32 once.  Needs 0 < warmup_no_steps <=
 * start_decay_after_n_steps, decay_every_n_steps > 0 and a finite max_lr > 0. */
int dfold_lr_schedule(const float* step, double base_lr, double max_lr, long warmup_no_steps, long start_decay_after_n_steps,
                      long decay_every_n_steps, double decay_factor, float* lr, void* stream);
/* One update of OpenFold's exponential moving average of the weights (ExponentialMovingAverage._update_state_dict_,
 * openfold/utils/exponential_moving_average.py:40-49, decay 0.999 in openfold/config.py:493) over flat fp32 buffers of n
 * elements (n % 4 == 0, 16-byte aligned):
 *   diff = ema - param;  diff *= one_minus_decay;  ema -= diff
 * each operation rounded to fp32 on its own (never an FMA), which gives the bits of those three torch ops when
 * one_minus_decay = fp32(1 - decay), 1 - decay taken in double as Python does.  0 <= one_minus_decay <= 1. */
int dfold_ema_update(float* ema, const float* param, long n, float one_minus_decay, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Evaluation metrics (csrc/metrics.cu), SURVEY.md 8 f6: the arithmetic of Experiment.eval_fn (train_DFOLD_dynamics.py:
 * 765-928) and compute_validation_metrics_all (:99-154) on the device.  All arithmetic is fp64; each coordinate input
 * is fp32 (flag 0) or fp64 (flag != 0) and is upcast exactly.  Sums run in a fixed order (equal inputs give equal bits);
 * no host reads, so every call is graph-capturable.
 * ---------------------------------------------------------------------------------------------------------- */
/* Experiment._calc_rot_trans_error (:1549-1568) over src/toolbox/rot_trans_error.py:7-73: pred / gt [nf][N][7]
 * (w,x,y,z, trans).  out [4][nf] = mean over residues of degrees(2 acos |clip(q_gt.q_pred)|) (both normalised), mean
 * |t_gt - t_pred| over residues and xyz (no mask), and the same two with gt[ref_frame] broadcast in place of pred
 * (the reference uses ref_frame = nf - 2).  Needs 0 <= ref_frame < nf. */
int dfold_rot_trans_error(const void* pred, int pred_f64, const void* gt, int gt_f64, int nf, int N, int ref_frame, double* out,
                          void* stream);
/* Masked atom errors over pred / gt [nf][N][A][3], mask [nf][N][A] (A >= 2, CA at column 1).  out [6][nf] = MAE and MSE
 * of eval_fn (:892-912; sum over the xyz-expanded mask, so 3 sum m, 0/0 = NaN), rmsd_all and rmsd_ca of
 * compute_validation_metrics_all (:143-146; sqrt(sum (gt m - pred m)^2 / (sum m + 1e-4))), sum m and sum m over CA.
 * drop_last_atom != 0 zeroes mask[nf-1][N-1][A-1], eval_fn's `atom_mask[-1, -1, -1] = 0.0` (:893). */
int dfold_atom_errors(const void* pred, int pred_f64, const void* gt, int gt_f64, const void* mask, int mask_f64, int nf, int N,
                      int A, int drop_last_atom, double* out, void* stream);
/* Batched Kabsch: B point sets of P points, point i of set s at p[s * set_stride + i * point_stride + 0..2] in both
 * `reference` and `coords` (point_stride >= 3), mask entries at mask[s * mask_set_stride + i * mask_point_stride].
 * Finds the proper rotation R and t minimising sum w |R coords + t - reference|^2 (Bio SVDSuperimposer as eval_fn
 * :898-909 and openfold/utils/superimposition.py:20-77 call it) with Horn's quaternion key matrix and fixed-sweep Jacobi,
 * centroids and covariance in separate passes.  mask_mode 0: w = 1; 1: w = mask (selection); 2: both coordinate sets
 * multiplied by the mask, w = 1 (compute_validation_metrics_all :113-150).  rmsd [B] = sqrt(sum w |R c + t - r|^2 /
 * sum w), from the applied transform; rot [B][9] (row-major), trans [B][3] and out_coords [B][P][3] = R coords + t may
 * be NULL.  An empty set (sum w = 0) gives rmsd NaN, R = I, t = 0 and out_coords = coords. */
int dfold_superimpose(const void* reference, int reference_f64, const void* coords, int coords_f64, long set_stride,
                      long point_stride, const void* mask, int mask_f64, long mask_set_stride, long mask_point_stride, int mask_mode,
                      int B, int P, double* rmsd, double* rot, double* trans, double* out_coords, void* stream);
/* openfold/utils/validation_metrics.py:17-36 drmsd of B structure pairs of N points (layout as dfold_superimpose):
 * out [B] = sqrt(sum_ij (|s1_i - s1_j| - |s2_i - s2_j|)^2 m_i m_j / (n (n - 1))), n = min over the B sets of sum m (N
 * without a mask; n <= 1 gives 0).  premul != 0 multiplies both structures by the mask first (compute_validation_metrics_all
 * :113-125).  partial: workspace of B * T * T doubles, T = ceil(N / 64), one fixed-order sum per 64 x 64 tile; B <= 65535. */
int dfold_drmsd(const void* s1, int s1_f64, const void* s2, int s2_f64, long set_stride, long point_stride, const void* mask,
                int mask_f64, long mask_set_stride, long mask_point_stride, int premul, int B, int N, double* partial, double* out,
                void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Trajectory rollout (csrc/rollout.cu), SURVEY.md 8 f7: the per-step bookkeeping of Experiment.eval_extension
 * (train_DFOLD_dynamics.py:931-1000) on the device.
 * ---------------------------------------------------------------------------------------------------------- */
/* One step of the rollout loop, replacing :993-996 (atom_traj.append(atom_pred[-1:]), rigid_traj.append(rigid_pred[-1:]),
 * valid_feats['rigids_0'] = cat(rigid_pred[1:], rigid_pred[-1:])).  rigid_pred [nf][N][7] and atom37 [nf][N][A][3] are the
 * network's prediction (fp32); rigids_0 [nf][N][7] is shifted in place; `step` is a DEVICE int64 counter s.  With
 * 0 <= s < L: rigid_traj[s] ([L][N][7]) = rigid_pred[nf-1], atom_traj[s] ([L][N][A][3]) = atom37[nf-1], rigids_0[f] =
 * rigid_pred[min(f+1, nf-1)], then s += 1; otherwise nothing is written.  One launch of one CTA, no host reads, so a
 * captured graph of (forward, advance) replays every step.  Needs nf >= 2, N, A, L >= 1 and rigid_pred disjoint from
 * rigids_0. */
int dfold_rollout_advance(const float* rigid_pred, const float* atom37, float* rigids_0, float* rigid_traj, float* atom_traj,
                          long long* step, int nf, int N, int A, int L, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DFOLD_B200_H */
