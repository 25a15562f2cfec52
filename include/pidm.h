/* libpidm -- C ABI of the H100-native physics-informed-diffusion hot path.
 *
 * The reference (jhbastek/PhysicsInformedDiffusionModels) has no FFI: its boundary is the Python class
 * surface used by main.py / sample.py (SURVEY.md section 8b).  This header is the operator interface those
 * classes are re-implemented on: plain pointers + sizes, no torch types.  Every entry point
 *   - takes raw DEVICE pointers borrowed from the caller (caller keeps them alive; nothing is allocated
 *     inside except through caller-provided workspaces),
 *   - launches on the `stream` argument (a cudaStream_t passed as void*), never synchronises,
 *   - returns 0 on success, non-zero on error with a message in pidm_last_error().
 * Activations are NHWC ([B, H*W, C]); `dtype` is PIDM_F32 (0) or PIDM_BF16 (1) and names the ACTIVATION /
 * packed-weight storage type; statistics, parameters, gradients of parameters and all reductions are fp32.
 * Each declaration cites the reference code it replaces (paths relative to the reference repository).
 */
#ifndef PIDM_H_
#define PIDM_H_

#ifdef __cplusplus
extern "C" {
#endif

#ifndef PIDM_F32
#define PIDM_F32 0
#define PIDM_BF16 1
#endif

const char* pidm_last_error(void);
int pidm_version(void);

/* ---- diffusion element-wise ops ------------------------------------------------------------------------- */
/* q_sample: x_t = sqrt(abar_t) x0 + sqrt(1-abar_t) eps.   src/denoising_utils.py:373-378 and inline :633-638 */
int pidm_qsample(const float* x0, const float* noise, const long long* t, const float* sqrt_ab,
                 const float* sqrt_1mab, float* xt, int B, int per_sample, void* stream);
/* ancestral step: out = coef1*x0_pred + coef2*x_t + sigma*z.   src/denoising_utils.py:441-455 */
int pidm_posterior_step(const float* x_t, const float* x0_pred, const float* z, float* out, float coef1, float coef2,
                        float sigma, long long n, void* stream);
/* out = a_b*x + b_b*y + c_b*z with per-sample coefficients [B]: the eta=0 DDIM jump of ddim_sample_x0
 * (src/denoising_utils.py:755-785) collapses to this form */
int pidm_axpby_per_sample(const float* a, const float* x, const float* b, const float* y, const float* c,
                          const float* z, float* out, int B, int per_sample, void* stream);
/* per-sample coefficients of the deterministic DDIM jump t -> t_next (src/denoising_utils.py:755-781, eta = 0):
 * x' = coef_x0 * x0_pred + coef_x * x  (coef_x0 = 0, coef_x = 1 where t == t_next); tables are the diff_dict entries */
int pidm_ddim_coefs(const long long* t, const long long* t_next, const float* posterior_mean_coef1,
                    const float* posterior_mean_coef2, const float* sqrt_recip_alphas, const float* noise_mean_coeff,
                    const float* alphas_prod, float* coef_x0, float* coef_x, int B, void* stream);
/* out = x * *alpha_dev  (chain-rule scaling of a precomputed gradient by the upstream scalar; out may alias x) */
int pidm_scale(const float* x, const float* alpha_dev, float* out, long long n, void* stream);

/* ---- toy study (main_toy.py, src/denoising_toy_utils.py:436-511): PIDM loss algebra on [B,D] points ---------- */
/* data term c_data*mean_b(w_b*mean_D(target-output)^2) with w_b = p2[t_b] (p2_loss_weight != NULL) or 1; Gaussian NLL of the
 * residual / inequality values with the log-likelihood clamped at -27.631 (:381); lambda*mean(opt).  ineq / opt may be
 * NULL.  sums7 = data, residual, inequality, optimisation terms, mean|r|, mean(ineq), mean(opt); gradients overwritten. */
int pidm_toy_pidm_loss(const float* target, const float* output, const float* residual, const float* ineq,
                       const float* opt, const long long* t, const float* p2_loss_weight,
                       const float* posterior_var_clipped, float c_data, float c_residual, float c_ineq, float lambda_opt,
                       float* sums7, float* grad_output, float* grad_residual, float* grad_ineq, float* grad_opt, int B,
                       int D, void* stream);

/* ---- Darcy residual (src/residuals_darcy.py:134-183 + src/grad_utils.py:64-146) ------------------------- */
/* The last int argument of the four Darcy entry points below is a flags word:
 *   PIDM_DARCY_PIXELS_AT_BOUNDARY  h = domain_length / (P-1) (else domain_length / P)
 *   PIDM_DARCY_PERIODIC            bcs='periodic' (src/grad_utils.py:76-81): every pixel uses the central second-order
 *                                  stencil and neighbours wrap around the plane; h is unchanged, and the bc_x0 / bc_x1
 *                                  channels are still written on rows 0 / P-1 and columns 0 / P-1, from the wrapped p_0 / p_1.
 * 0 and 1 keep their old meaning (pixels_at_boundary false / true); unknown bits are rejected. */
#define PIDM_DARCY_PIXELS_AT_BOUNDARY 1
#define PIDM_DARCY_PERIODIC 2
/* x0hat [B,2,P,P] fp32 NCHW (p, K); f_s [P*P]; residual [B,P*P,3] = (eq_0, bc_x0, bc_x1).  P must be 64. */
int pidm_darcy_residual_fwd(const float* x0hat, const float* f_s, float* residual, int B, int pixels,
                            float domain_length, int reverse_d1, int flags, void* stream);
/* vector-Jacobian product of the above: grad_x0hat [B,2,P,P] = J^T grad_residual */
int pidm_darcy_residual_bwd(const float* x0hat, const float* f_s, const float* grad_residual, float* grad_x0hat, int B,
                            int pixels, float domain_length, int reverse_d1, int flags, void* stream);
/* one derivative field of u [planes,P,P]: mode 0..4 = d_d0, d_d1, d_d00, d_d11, d_d01 (StencilGradients.forward,
 * src/grad_utils.py:161-175; second-order, one-sided at the boundary), OR PIDM_FD_PERIODIC for the wrapped central
 * stencil at every pixel (periodic=True, src/grad_utils.py:76-81) */
#define PIDM_FD_PERIODIC 8
int pidm_fd_stencil(const float* u, float* out, int planes, int pixels, int mode, float d0, float d1, void* stream);
/* Fused PIDM loss (src/denoising_utils.py:669-692): sums3 = {c_data*mean_b(p2[t] mse_b), mean(c_res*0.5 r^2/var_t),
 * mean|r|}; optionally the gradient of (sums3[0]+sums3[1]) w.r.t. x0hat (residual operand) and model_out (data
 * operand; pass the same pointer twice in 'mean' mode, then only grad_x0hat is written).  The residual is never
 * materialised.  The gradient pointers take one of three forms, any other is rejected before a launch:
 *   grad_x0hat = grad_model_out = NULL                  loss only (either model_out);
 *   grad_x0hat set, grad_model_out = NULL               model_out == x0hat: the data gradient is added into grad_x0hat;
 *   grad_x0hat and grad_model_out both set              model_out != x0hat. */
int pidm_darcy_pidm_loss(const float* x0hat, const float* model_out, const float* target, const float* f_s,
                         const long long* t, const float* p2_loss_weight, const float* posterior_var_clipped,
                         float c_data, float c_residual, float* sums3, float* grad_x0hat, float* grad_model_out, int B,
                         int pixels, float domain_length, int reverse_d1, int flags, void* stream);
/* CoCoGen step size (src/residuals_darcy.py:218-231): max_dr_dp[b] = largest entry (signed, as torch.max) of the Jacobian
 * d residual / d p of sample b -- evaluated analytically from the stencil coefficients and K, the reference materialises
 * the 12288 x 4096 Jacobian per sample with vmap(jacfwd). */
int pidm_darcy_jacobian_max(const float* x0hat, float* max_dr_dp, int B, int pixels, float domain_length, int reverse_d1,
                            int flags, void* stream);
/* CoCoGen corrections (src/residuals_darcy.py:209-240, applied `steps` times), one launch for the batch.  x [B,2,P,P]
 * fp32 (p, K) is updated in place: every active sample gets `steps` corrections
 *   p <- p - (1e-6 / min(max_dr_dp, 1e12)) * d(sum r^2)/dp,
 * and residual [B,P*P,3] receives the residual of the corrected fields.  Sample b is active when t == NULL or
 * t[b] < n_active (t [B] int64 on the device, so a captured graph can predicate on the time index); an inactive
 * sample is neither read nor written.  steps = 0 only evaluates the residual.  No allocation, no host synchronisation. */
int pidm_darcy_cocogen(float* x, const float* f_s, float* residual, const long long* t, int n_active, int steps, int B,
                       int pixels, float domain_length, int reverse_d1, int flags, void* stream);
/* Residual-gradient guidance (src/residuals_darcy.py:116-120): cond = d (sum|r(x_t)|) / n_norm / d x_t, the residual
 * evaluated on x_t [B,2,P,P] itself, written in the b_xy_c layout [B,P*P,2] fp32 the network takes.  sign(0) = 0.  n_norm
 * is the count the mean divides by: B*P*P*3, or world*B*P*P*3 for a shard of a global batch. */
int pidm_darcy_abs_residual_grad(const float* x_t, const float* f_s, float* cond, int B, long long n_norm, int pixels,
                                 float domain_length, int reverse_d1, int flags, void* stream);

/* ---- Darcy training-data generation (src/darcy_data_generation.py), fp64, P = 64 --------------------------- */
/* KLE permeability (:63-78, :131-133): K[b] = exp(phi_s z[b]); phi_s [q, P*P] = [sqrt(lambda_k) phi_k], z [B, q],
 * K [B, P*P].  The sum runs over k in ascending order, one sample per column of the grid: K[b] depends on z[b] only. */
int pidm_darcy_gen_kle(const double* phi_s, const double* z, double* K, int B, int q, int pixels, void* stream);
/* bytes of workspace pidm_darcy_gen_solve needs for B samples (about 6.5 MB per sample); -1 on bad arguments */
long long pidm_darcy_gen_workspace_bytes(int B, int pixels);
/* pressure for given K [B, P*P] (:135-165): p = lstsq([A; BC; w^T], [f_s; 0; 0]) computed as the normal equations with
 * node 0 pinned (banded fp64 Cholesky, half-bandwidth 3P+3) followed by p -= (w^T p) / (w^T 1).  f_s [P*P] fp64.
 * Outputs (each may be NULL): p [B, P*P] fp64; res [B] = mean |M p - b| over the P*P + 4P + 1 rows (:163-165, fp64);
 * batch [B, 2, P, P] fp32 = (p, K).  h = domain_length / (P-1) with PIDM_DARCY_PIXELS_AT_BOUNDARY in flags (trapezoid
 * weights {1,2,4} h^2/4), else domain_length / P (plain mean); reverse_dy: h1 = -h and the y BC rows +D1 | -D1 (:149-152).
 * stages: PIDM_DARCY_GEN_ASSEMBLE | _FACTOR | _POST, run in that order (PIDM_DARCY_GEN_ALL for a solve); the workspace
 * carries the band and right-hand side between them.  Workspace layout, fp64: band [B, P*P, 3P+4] first, band[b][r][d] =
 * N[r][r-d] (d = 0 .. 3P+3; entries of negative column r - d < 0 are written 0 by the assembly and never read after it),
 * then rhs [B, P*P] = A^T f_s; the factorisation overwrites band with L (same layout) and rhs with y = L^-1 rhs. */
#define PIDM_DARCY_GEN_ASSEMBLE 1
#define PIDM_DARCY_GEN_FACTOR 2
#define PIDM_DARCY_GEN_POST 4
#define PIDM_DARCY_GEN_ALL 7
int pidm_darcy_gen_solve(const double* K, const double* f_s, double* p, double* res, float* batch, void* workspace,
                         long long workspace_bytes, int B, int pixels, double domain_length, int reverse_dy, int flags,
                         int stages, void* stream);

/* ---- layout ------------------------------------------------------------------------------------------- */
/* image_to_b_xy_c (src/denoising_utils.py:36-42) fused with the dtype change + channel padding */
int pidm_nchw_to_nhwc(const float* src, void* dst, int B, int C, int HW, int Cpad, int dtype, void* stream);
/* emb_conv[0] + GELU of the residual-gradient guidance branch (src/unet_model.py:520-524,585-603):
 * out[b,hw,:] = GELU_erf(W0 cond[b,hw,:] + b0) as NHWC activations [B,HW,C] (dtype), cond [B,HW,2] fp32, W0 [C,2], b0 [C]
 * fp32.  null_mask [B] (bool bytes, may be NULL = none): those samples take cond = 0 (cond is not read), i.e. GELU(b0).
 * C % 8 == 0 and C / 8 divides 32. */
int pidm_cond_embed_fwd(const float* cond, const unsigned char* null_mask, const float* w0, const float* b0, void* out,
                        int B, int HW, int C, int dtype, void* stream);
/* its weight gradient from dg = d loss / d out [B,HW,C] (dtype): the pre-activation is recomputed;
 * dW0 [C,2] += sum dz * cond, db0 [C] += sum dz (fp32, accumulated: block partials + global reductions) */
int pidm_cond_embed_wgrad(const float* cond, const unsigned char* null_mask, const float* w0, const float* b0,
                          const void* dg, float* dw0, float* db0, int B, int HW, int C, int dtype, void* stream);
/* torch.cat((x, skip), dim=1) on NHWC rows and its backward (src/unet_model.py:606,612) */
int pidm_concat_channels(const void* a, const void* b, void* out, long long rows, int Ca, int Cb, int dtype, void* stream);
int pidm_split_channels(const void* g, void* ga, void* gb, long long rows, int Ca, int Cb, int dtype, void* stream);
/* circular padding (Unet3D(padding_mode='circular'), src/unet_model.py:161-199): y [B, H+2h, W+2h, C] is x [B,H,W,C]
 * with a halo of h = 1..3 pixels wrapped around both spatial axes, y[b,i,j] = x[b, (i-h) mod H, (j-h) mod W], copied
 * bit for bit in 16-byte units (C * sizeof(dtype) % 16 == 0, 16-byte aligned pointers).  A circular convolution is the
 * valid (pad 0) convolution of this copy; see pidm_conv2d_tc_general for the transposed gather. */
int pidm_wrap_pad_nhwc(const void* x, void* y, int B, int H, int W, int C, int halo, int dtype, void* stream);

/* ---- convolutions as implicit GEMM (src/unet_model.py:163,197,227,253,275,279,453,517) ------------------- */
/* Packed weights: Wp[n][tap*Cin + c] in the activation dtype, built by pidm_pack_weights from the framework
 * layout through strides.  PackEntry (56 bytes, see pidm_pack_entry_size):
 *   { const float* src; void* dst; long long s_n, s_c; int N, C, Cpad, taps, flip, pad_; }
 *   src index = n*s_n + c*s_c + (flip ? taps-1-tap : tap) */
int pidm_pack_entry_size(void);
int pidm_pack_weights(const void* table_dev, int n_entries, int dtype, void* stream);
/* Forward AND dgrad operand of a layer from one read of its weights (layers with Cin % 32 == 0, Cout % 32 == 0,
 * <= 16 taps); one CTA per 32 x 32 channel block.  PackPairEntry (64 bytes, see pidm_pack_pair_entry_size):
 *   { const float* src; void* dst_f; void* dst_d (may be null); long long s_co, s_ci; int Cout, Cin, taps, flip;
 *     int tile0, pad_; }
 *   src index = co*s_co + ci*s_ci + tap;  dst_f[co][tap*Cin + ci];  dst_d[ci][(flip ? taps-1-tap : tap)*Cout + co]
 *   entry e owns blocks [tile0, tile0 + (Cout/32)*(Cin/32)); tile_map_dev[i] = index of the entry that owns block i;
 *   one launch packs blocks [tile_base, tile_base + n_tiles). */
int pidm_pack_pair_entry_size(void);
int pidm_pack_weights_pairs(const void* table_dev, const int* tile_map_dev, int tile_base, int n_tiles, int max_taps,
                            int dtype, void* stream);
/* y[b,oh,ow,n] = sum A(m,k) Wp[n,k] + bias[n] + residual;  transposed=0: A gathers x at (oh*s-p+r, ow*s-p+q);
 * transposed=1: at ((oh+p-r)/s, (ow+p-q)/s) when divisible (ConvTranspose forward / strided-conv dgrad).
 * CUDA-core fp32-accumulate kernel for every geometry (parity anchor + layers the tensor-core kernel skips). */
int pidm_conv2d_simt(const void* x, const void* w_packed, const float* bias, const void* residual, void* y, int B,
                     int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride, int pad,
                     int transposed, int dtype, void* stream);
/* dW (framework layout, index n*w_stride_n + c*w_stride_c + tap) += sum_m dy[m,n] A(m,tap,c); dbias[n] += sum_m dy */
int pidm_conv2d_wgrad_simt(const void* x, const void* dy, float* dw, float* dbias, int B, int H, int W, int Cin,
                           int Cin_real, int Ho, int Wo, int Cout, int KH, int KW, int stride, int pad, int transposed,
                           long long w_stride_n, long long w_stride_c, int dtype, void* stream);
/* wgmma + TMA implicit-GEMM convolution, bf16 operands, fp32 register accumulation; same contract as pidm_conv2d_simt
 * (requires Cin % 32 == 0, Cout % 32 == 0): stride-1/2 regular convolution (input sampled through TMA elementStrides) and the
 * stride-2 transposed gather (ConvTranspose forward / dgrad of the stride-2 conv) as 4 output-parity classes over the
 * Ho/2 x Wo/2 grid, Ho = 2(H-1) - 2 pad + KH.  pad = KH/2 - 1 is the zero-padded layer (Ho = 2H); an input with a wrapped
 * 1-pixel halo (pidm_wrap_pad_nhwc, H = Ho/2 + 2) and pad = KH/2 + 1 is the circular one.
 * gn_sums (optional, [B, gn_groups, 2]): per-(sample, group) sum and sum of squares of the fp32 output, accumulated in
 * the epilogue so that the following GroupNorm needs no statistics pass.  It is zeroed here (one memset node) unless
 * gn_sums_zeroed != 0, i.e. the caller hands in a slice of a buffer it has already cleared. */
int pidm_conv2d_tc_general(const void* x, const void* w_packed, const float* bias, const void* residual, void* y, int B,
                           int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride, int pad,
                           int transposed, float* gn_sums, int gn_groups, int gn_sums_zeroed, void* stream);
int pidm_conv2d_tc_general_supported(int B, int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride,
                                     int pad, int transposed);
/* plan the tensor-core convolution picks for a supported geometry (test / tuning aid): out[10] = {BN, BK, row-group
 * staging, resident weights, ring stages, total tiles, grid (persistent CTAs), TN, TH, TW} */
int pidm_conv2d_tc_plan(int B, int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride, int pad,
                        int transposed, int* out);
/* wgrad on the tensor cores (wgmma): D[(tap,cA)][cB] = sum over grid pixels g of a[a_stride*g - pad + tap][cA] * b[g][cB], MN-major
 * (pixel-strided) TMA operands, split over pixel ranges, red.global.add into dw[cA*s_row + cB*s_col + tap] (fp32,
 * ACCUMULATED).  Regular conv: a = x, b = dy.  ConvTranspose: a = dy (a_stride 2), b = x.  Rows cA >= CA_real (channel
 * padding) are dropped.  Circular layers pass the halo'd copy of a (pidm_wrap_pad_nhwc) with pad 0; the 3x3 stride-1
 * case takes the tap-complete kernel both with (HA = GH, pad 1) and with (HA = GH + 2, pad 0). */
int pidm_conv2d_wgrad_tc(const void* a, const void* b, float* dw, int B, int HA, int WA, int CA, int CA_real, int GH,
                         int GW, int CB, int KH, int KW, int a_stride, int pad, long long s_row, long long s_col,
                         void* stream);
int pidm_conv2d_wgrad_tc_supported(int B, int GH, int GW, int CA, int CB, int KH, int KW, int a_stride);
/* plan of a pidm_conv2d_wgrad_tc call with the same integer arguments (test / tuning aid): out[12] = {tap-complete 3x3
 * kernel (1) or generic (0), NP, AA, AB, pixel splits, pixel tiles per split, pixel tiles, CTAs per split, row-group
 * staging (3x3 kernel), pixel tile TN, TH, TW} */
int pidm_conv2d_wgrad_tc_plan(int B, int HA, int WA, int CA, int CA_real, int GH, int GW, int CB, int KH, int KW,
                              int a_stride, int pad, long long s_row, long long s_col, int* out);
/* out[c] += sum_m x[m][c]: bias gradients (column sums of an NHWC tensor) */
int pidm_colsum(const void* x, float* out, long long M, int C, int dtype, void* stream);

/* ---- normalisations ------------------------------------------------------------------------------------ */
/* Block.forward tail: GroupNorm(G) -> *(scale+1)+shift -> SiLU (src/unet_model.py:233-241).  scale_shift [B,2C] or NULL.
 * residual (optional, same shape as y) is added after the SiLU: the `h + x` of a ResnetBlock whose res_conv is the
 * identity (:262).  sums [B,G,2] (sum, sum of squares) is written here and consumed by the backward.
 * With n = HW * C/G, s = sums[b][g][0], ss = sums[b][g][1]:  mean = s / n,  var = max(ss / n - mean^2, 0)  (biased, clamped),
 * rstd = 1 / sqrt(var + eps),  y = silu(((x - mean) rstd gamma + beta)(scale + 1) + shift) (+ residual).  The sums are fp32, so
 * the variance carries a relative error of about 2^-24 (1 + mean^2 / var): a group whose mean is tens of standard deviations
 * away from zero loses that many digits (DESIGN.md section 2 has the measured figures).  A constant group has var = 0 up to
 * that cancellation, hence rstd between 1 / sqrt(eps) and 1 / sqrt(eps + 2^-22 mean^2), and x - mean within 2^-23 |mean|. */
int pidm_groupnorm_silu_fwd(const void* x, const float* gamma, const float* beta, const float* scale_shift,
                            const void* residual, void* y, float* sums, int stats_precomputed, int B, int HW, int C, int G,
                            float eps, int dtype, void* stream);
/* workspace: float[B*C*2]; dgamma/dbeta ACCUMULATE; d_scale_shift [B,2C] overwritten (may be NULL);
 * dbias_of_producer (may be NULL): column sums of dx ACCUMULATED = bias gradient of the convolution that produced x. */
int pidm_groupnorm_silu_bwd(const void* x, const void* dy, const float* sums, const float* gamma, const float* beta,
                            const float* scale_shift, void* dx, float* dgamma, float* dbeta, float* d_scale_shift,
                            float* dbias_of_producer, float* workspace, int B, int HW, int C, int G, float eps,
                            int dtype, void* stream);
/* What the two GroupNorm entry points launch for a shape (test aid): out[10] = {statistics chunks, statistics block, apply
 * chunks, apply grid rules that fired (bit 0 shrink the unroll, bit 1 halve, bit 2 one wave and loop), backward path
 * (0 two-launch fallback, 1 / 2 piece kernel with 1 / 2 vectors per thread, 3 packed, 4 streaming), channel slab, threads,
 * cluster size, pixel rows per CTA, vectors per thread}; the last five are 0 on the fallback path. */
int pidm_groupnorm_plan(int B, int HW, int C, int G, int dtype, int* out);
/* channel LayerNorm, gain only, biased variance (src/unet_model.py:201-210); dgamma ACCUMULATES */
int pidm_layernorm_c_fwd(const void* x, const float* gamma, void* y, long long M, int C, float eps, int dtype, void* stream);
int pidm_layernorm_c_bwd(const void* x, const void* dy, const float* gamma, void* dx, float* dgamma,
                         const void* dx_residual /* optional: added to dx (skip-connection gradient) */, long long M, int C,
                         float eps, int dtype, void* stream);

/* ---- attention ------------------------------------------------------------------------------------------ */
/* SpatialLinearAttention core between to_qkv and to_out (src/unet_model.py:286-297), dim_head = 32.
 * qkv [B,N,3*heads*32]; out [B,N,heads*32]; ctx [B,heads,32,32], kmax/kzinv [B,heads,32] kept for backward. */
/* The whole linear-attention block at the 32-channel levels (C = 32, 8 heads, bf16):
 * y = residual + b_out + to_out(attention(to_qkv(xn))), with to_qkv a 1x1 32 -> 768 projection without bias and to_out
 * a 1x1 256 -> 32 projection (reference unet_model.py:275-297 and the Residual wrapper's `+ x`).  q, k, v are recomputed
 * per head on the tensor cores from xn = PreNorm(x), and neither the attention output nor its gradient [B,N,256] is
 * materialised: forward multiplies each head's output tile by its 32 columns of W_out on chip, backward recomputes
 * dout_h = dy W_out[:, 32h:32h+32] per head from dy.  Neither qkv nor dqkv [B,N,768] is materialised either.
 *   xn, residual, y, dy, dxn: [B,N,32] bf16.  w_qkv: packed to_qkv weights [768][32] bf16 (pidm_pack_weights).
 *   w_out: packed forward to_out weights [32][256] bf16 (pidm_pack_weights, row = output channel).  b_out: [32] fp32.
 *   fwd: y is WRITTEN; ctx [B,8,32,32] and kmax / kzinv [B,8,32] are WRITTEN and kept for backward; workspace holds
 *   pidm_linattn_block_workspace_floats(B, N) floats of scratch.
 *   bwd: dxn is WRITTEN (the gradient w.r.t. xn through to_qkv only: the residual's gradient is dy itself); dctx
 *   [B,8,32,32] is WRITTEN and read again by wgrad.
 *   wgrad: ACCUMULATES the to_qkv weight gradient into grad_w_qkv (element [n][c] at n * qkv_stride_n + c * qkv_stride_c)
 *   and the to_out weight gradient into grad_w_out (element [c][j] at c * out_stride_n + j * out_stride_c), both fp32.
 *   The bias gradient (column sums of dy) is left to pidm_colsum. */
int pidm_linattn_block_supported(int C, int heads, int N, int dtype);
int pidm_linattn_block_workspace_floats(int B, int N);
/* pixel chunking of the block's launches (test aid): out[5] = {statistics chunks, ctx / fwd / bwd / wgrad pixels per
 * CTA} */
int pidm_linattn_block_plan(int B, int N, int* out);
int pidm_linattn_block_fwd(const void* xn, const void* w_qkv, const void* w_out, const float* b_out, const void* residual,
                           void* y, float* ctx, float* kmax, float* kzinv, float* workspace, int B, int N, void* stream);
int pidm_linattn_block_bwd(const void* xn, const void* w_qkv, const void* w_out, const void* dy, const float* ctx,
                           const float* kmax, const float* kzinv, void* dxn, float* dctx, int B, int N, void* stream);
int pidm_linattn_block_wgrad(const void* xn, const void* w_qkv, const void* w_out, const void* dy, const float* ctx,
                             const float* dctx, const float* kmax, const float* kzinv, float* grad_w_qkv,
                             long long qkv_stride_n, long long qkv_stride_c, float* grad_w_out, long long out_stride_n,
                             long long out_stride_c, int B, int N, void* stream);
/* Standalone linear attention (every layer that is not the 32-channel block), s = 32^-1/2, per sample and head h with
 * q, k, v the head's [N][32] slices of qkv:
 *   out[n, h*32+e] = s * sum_d softmax_d(q[n,:])[d] * ctx[h][d][e]
 *   ctx[h][d][e]   = sum_n exp(k[n,d] - kmax[h][d]) * kzinv[h][d] * v[n,e] / N     (so ctx includes 1/(Z_d N))
 *   kmax[b, h*32+d] = max_n k[n,d];   kzinv[b, h*32+d] = 1 / sum_n exp(k[n,d] - kmax)
 * fwd WRITES out, ctx, kmax and kzinv; workspace holds pidm_linattn_workspace_floats(B, N, heads) floats of scratch.
 * bwd WRITES dqkv from qkv, dout and the forward's ctx / kmax / kzinv (heads a multiple of 4); dctx_scratch
 * [B,heads,32,32] is scratch. */
int pidm_linattn_workspace_floats(int B, int N, int heads);
int pidm_linattn_fwd(const void* qkv, void* out, float* ctx, float* kmax, float* kzinv, float* workspace, int B, int N,
                     int heads, int dtype, void* stream);
int pidm_linattn_bwd(const void* qkv, const void* dout, const float* ctx, const float* kmax, const float* kzinv,
                     void* dqkv, float* dctx_scratch, int B, int N, int heads, int dtype, void* stream);
/* What pidm_linattn_fwd / _bwd launch for a shape (test aid): out[8] = {forward path (0 one CTA per (sample, head),
 * 1 mma.sync, 2 SIMT), backward path (0 mma.sync, 1 SIMT, -1 shape refused), statistics chunks, statistics rows per
 * chunk, SIMT context rows per chunk, SIMT context chunks, mma.sync pixels per CTA, mma.sync chunks per sample}. */
int pidm_linattn_plan(int B, int N, int heads, int dtype, int* out);
/* mid-block softmax attention over <= 64 tokens (src/unet_model.py:341-367) */
int pidm_attn_fwd(const void* qkv, void* out, int B, int n_tokens, int heads, int dtype, void* stream);
int pidm_attn_bwd(const void* qkv, const void* dout, void* dqkv, int B, int n_tokens, int heads, int dtype, void* stream);

/* ---- time conditioning (fp32) --------------------------------------------------------------------------- */
/* SinusoidalPosEmb + time_mlp (src/unet_model.py:147-159,464-469); also returns SiLU(temb) for the block MLPs */
int pidm_time_embed_fwd(const long long* t, const float* W1, const float* b1, const float* W2, const float* b2,
                        float* emb, float* h1, float* temb, float* silu_t, int B, int dim, int td, void* stream);
/* workspace float[2*B*td]; parts: bit 1 = activation gradients into the workspace, bit 0 = weight / bias gradients from
 * it (ACCUMULATED) -- the second half only feeds the optimizer and may be issued on another stream after the first. */
int pidm_time_embed_bwd(const float* d_silu_t, const float* emb, const float* h1, const float* temb, const float* W2,
                        float* dW1, float* db1, float* dW2, float* db2, float* workspace, int B, int dim, int td,
                        int parts, void* stream);
/* every ResnetBlock.mlp Linear in one launch (src/unet_model.py:246-249,258-262).  MlpEntry (56 bytes):
 *   { const float* W; const float* b; float* dW; float* db; float* out; const float* dout; int n, pad_; }
 *   out_e[b, j] = b_e[j] + W_e[j,:] . silu_t[b,:] ;  backward accumulates dW_e, db_e and overwrites d_silu_t. */
int pidm_mlp_entry_size(void);
int pidm_block_mlps_fwd(const void* table_dev, int n_entries, int max_rows, const float* silu_t, int B, int td,
                        void* stream);
/* parts: bit 0 = weight / bias gradients, bit 1 = input gradient d_silu_t (independent halves) */
int pidm_block_mlps_bwd(const void* table_dev, int n_entries, int max_rows, const float* silu_t, float* d_silu_t, int B,
                        int td, int parts, void* stream);

/* ---- output head: final 1x1 conv to NCHW fp32 (+ sigmoid on the last channel) src/unet_model.py:517,619-621 */
int pidm_head_fwd(const void* x, const float* w, const float* bias, float* y, int B, int HW, int C, int O,
                  int sigmoid_last, int dtype, void* stream);
int pidm_head_bwd(const void* x, const float* w, const float* y, const float* dy, void* dx, float* dw, float* db, int B,
                  int HW, int C, int O, int sigmoid_last, int dtype, void* stream);

/* ---- step glue on flat buffers (main.py:163-166,178-183; src/denoising_utils.py:163-205) ----------------- */
/* out[0] += sum x^2, deterministic (fixed summation order).  workspace: float[1185] zero-initialised once by the caller. */
int pidm_sumsq(const float* x, long long n, float* out, float* workspace, void* stream);
/* Adam (torch.optim.Adam semantics, bias corrections evaluated in double) + global-norm clip + EMA shadow, one pass.
 * step: 1-based host step count, ignored when step_counter_dev != NULL (device counter, incremented by the call).
 * ema_first_step: 0 = no EMA update; k >= 1 = update the shadow from the k-th step on (main.py:178 => ema_start+2). */
int pidm_adam_ema_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, float* ema_shadow, long long n,
                       float lr, double beta1, double beta2, float eps, int step, int* step_counter_dev,
                       const float* grad_norm_sq_dev, float grad_scale, float max_norm, float ema_mu,
                       int ema_first_step, int zero_grad, void* stream);
/* a[i] <-> b[i] for i < n, in place, one pass (ema.ema / ema.restore of main.py:183,316 on the flat weight and EMA
 * buffers: two calls restore every bit, and no pointer into either buffer changes).  n % 4 == 0 and both pointers
 * 16-byte aligned, else an error is returned and nothing is launched. */
int pidm_swap_f32(float* a, float* b, long long n, void* stream);

/* ---- mechanics residual, matrix-free (src/residuals_mechanics_K.py:166-274) ------------------------------ */
/* u [B,2,65,65] nodal displacements, rho [B,64,64], bcs [B,4,65,65] = (bc_x, bc_y, load_x, load_y), KE [8,8].
 * residual [B,8450] = K(rho) u - f with BC rows replaced by identity rows; compliance [B] = u^T K u. */
int pidm_mechanics_residual_fwd(const float* u, const float* rho, const float* bcs, const float* KE, float* residual,
                                float* compliance, int B, int nel, void* stream);
int pidm_mechanics_residual_bwd(const float* u, const float* rho, const float* bcs, const float* KE,
                                const float* grad_residual, const float* grad_compliance, float* grad_u, float* grad_rho,
                                float* workspace /* float[B*2*(nel+1)^2] */, int B, int nel, void* stream);
/* Fused PIDM loss of the mechanics branch + its gradients (src/denoising_utils.py:669-710), one launch:
 * u [B,2,n] displacements on the (nel+1)^2 node grid, rho [B,nel,nel], x0 [B,3,n] = (disp_x, disp_y, E) data target,
 * residual [B,2n], compliance [B], vf [B].  sums6 (zeroed here) = data, residual, inequality, optimisation loss terms,
 * mean|r|, mean_b(mean(rho_b) - vf_b).  grad_u / grad_rho / grad_residual / grad_compliance are overwritten, or all four
 * are NULL: loss only (every CTA adds the same per-sample contributions to the sums, with atomics in any order, so
 * the sums agree bitwise for B = 1 and to the order of the additions otherwise); any other combination is rejected
 * before a launch. */
int pidm_mech_pidm_loss(const float* u, const float* rho, const float* x0, const float* residual, const float* compliance,
                        const float* vf, const long long* t, const float* p2_loss_weight,
                        const float* posterior_var_clipped, float c_data, float c_residual, float c_ineq,
                        float lambda_opt, float* sums6, float* grad_u, float* grad_rho, float* grad_residual,
                        float* grad_compliance, int B, int nel, void* stream);
/* bilinear resize, align_corners=False, antialias=False (resize_image, src/residuals_mechanics_K.py:10-21) */
int pidm_bilinear_resize_fwd(const float* x, float* y, int planes, int in, int out, void* stream);
int pidm_bilinear_resize_bwd(const float* dy, float* dx, int planes, int in, int out, void* stream);
/* conditional sampling of the topology-optimisation model, the two per-step pieces around the network call:
 * U-Net input out [B,3+nc,P,P] = (bilinear resize of x [B,3,P+1,P+1] to P, the nc constant planes [B,nc,P,P]) */
int pidm_mech_sample_input(const float* x, const float* planes, float* out, int B, int nc, int P, void* stream);
/* x_out [B,3,P+1,P+1] = c1[t_b] model_out + c2[t_b] x + sigma[t_b] z, model_out = (bilinear P -> P+1 of y[:, :2],
 * y[:, 2] zero-padded), y [B,3,P,P]; t [B] on the device indexes the tables.  x_out may alias x. */
int pidm_mech_posterior_step(const float* y, const float* x, const float* z, const long long* t, const float* coef1,
                             const float* coef2, const float* sigma, float* x_out, int B, int P, void* stream);
/* Jacobi-PCG of K(rho) u = f on the free dofs (u = 0 on the Dirichlet dofs), one CTA per sample, one launch for the
 * whole solve: rho [B,nel,nel], bcs [B,4,nel+1,nel+1], KE [8,8].  Stops at ||r||/||f|| < tol (fp64) or max_iter.
 * Writes u [B,2,nel+1,nel+1], iters [B] and the final relative residual relres [B].  (nel+1)^2 <= 4608. */
int pidm_mech_fem_pcg(const float* rho, const float* bcs, const float* KE, float* u, int* iters, double* relres,
                      double tol, int max_iter, int B, int nel, void* stream);
/* fm [B] = 1 unless the pixels rho > 0.5 form exactly one 8-connected component (reference :369-380) */
int pidm_mech_floating_material(const float* rho, long long* fm, int B, int nel, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PIDM_H_ */
