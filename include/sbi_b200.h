/* sbi_b200 -- C ABI of the H100-native hot path of sbi (density-estimator training and
 * posterior evaluation).  Plain pointers and sizes only; no torch types.
 *
 * Every pointer named d_* is a DEVICE pointer (sm_90a), every h_* a HOST pointer.
 * `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 * All functions return 0 on success, a negative SBI_E* code on argument errors, or a
 * positive cudaError_t value if a CUDA call failed.  Nothing here synchronises unless the
 * name ends in _host (those take host buffers and block until the result is on the host).
 *
 * Reference interface replaced (file:line under /root/reference):
 *   sbi/neural_nets/estimators/nflows_flow.py:77-97   NFlowsFlow.log_prob   -> sbi_b200_nsf_logprob
 *   sbi/neural_nets/estimators/nflows_flow.py:99-109  NFlowsFlow.loss + autograd backward
 *                                                      (trainers/base.py:1171-1187)  -> sbi_b200_nsf_vjp
 *   sbi/neural_nets/estimators/nflows_flow.py:111-128 NFlowsFlow.sample     -> sbi_b200_nsf_inverse
 *   sbi/neural_nets/estimators/nflows_flow.py:42-75   inverse_transform     -> sbi_b200_nsf_logprob (z_out)
 *   sbi/neural_nets/ratio_estimators.py:132-154      RatioEstimator.forward -> sbi_b200_ratio_forward (resnet),
 *                                                      sbi_b200_ratio_mlp_forward (mlp, linear)
 *   sbi/inference/trainers/base.py:1181-1187          clip_grad_norm_ + Adam.step -> sbi_b200_reduce_partials,
 *                                                                                  sbi_b200_adam_clip_step
 */
#ifndef SBI_B200_H
#define SBI_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SBI_B200_ABI_VERSION 1

#define SBI_EINVAL (-1)   /* bad argument */
#define SBI_ESMEM (-2)    /* model does not fit the shared-memory budget of one CTA */
#define SBI_ENOGPU (-3)   /* no sm_90 device */

/* per-layer descriptor table: SBI_NSF_LAYER_STRIDE ints per coupling layer */
#define SBI_NSF_LAYER_STRIDE 64
#define SBI_NSF_MAX_BLOCKS 8
enum {
  SBI_L_NID = 0,      /* number of identity (conditioner-input) features */
  SBI_L_NTR = 1,      /* number of transformed features */
  SBI_L_W0 = 2,       /* float offset: initial layer  [Hp][Cp+IDp], columns = [ctx | id] */
  SBI_L_B0 = 3,
  SBI_L_WF = 4,       /* final layer [n_tr*PR][Hp]; feature f owns rows f*PR .. f*PR+3K-2 */
  SBI_L_BF = 5,
  SBI_L_LU_LOWER = 6, /* nflows LULinear params, native shapes */
  SBI_L_LU_UPPER = 7,
  SBI_L_LU_DIAG = 8,
  SBI_L_LU_BIAS = 9,
  SBI_L_FEAT = 10,    /* offset into feat_tab: n_id identity features then n_tr transformed */
  SBI_L_HAS_LU = 11,
  SBI_L_BC0 = 12,     /* head == SBI_NSF_MOG: second bias of the initial layer (MADE's context_layer.bias) */
  SBI_L_BLK0 = 16     /* per residual block b, 6 ints at SBI_L_BLK0+6*b: W1,B1,W2,B2,WC,BC */
};
/* what the conditioner's outputs parameterise (`head`):
 *   SBI_NSF_SPLINE (0): rational-quadratic coupling transform + LULinear per layer, N(0, I) base (`nsf`)
 *   SBI_NSF_MOG    (1): `made`: ONE masked residual conditioner (nflows MADE, masks folded into the packed
 *                       weights) whose outputs are, per feature, M x (logit, mean, unconstrained std) of a
 *                       mixture of Gaussians; log q = sum_f log MoG_f(z_f), no base density
 *                       (sbi/neural_nets/net_builders/flow.py:37-112, sbi/utils/nn_utils.py:133-201:
 *                       MADEMoGWrapper prepends a dummy feature, so D here = features + 1 and feature 0
 *                       -- whose input the caller sets to 0 -- is excluded from the likelihood). */
#define SBI_NSF_SPLINE 0
#define SBI_NSF_MOG 1

/* Neural spline flow (sbi `posterior_nn("nsf")` / `likelihood_nn("nsf")`,
 * reference builder sbi/neural_nets/net_builders/flow.py:333-460). */
typedef struct {
  int32_t D, C, H, NB, KB, T;      /* input dim, context dim, hidden, res-blocks, bins, layers */
  int32_t Dp, Cp, IDp, Hp, PR;     /* padded: round4(D), round4(C), round4(max n_id), round4(H), round4(3KB-1) */
  int32_t TRmax;                   /* max transformed features over layers */
  int32_t nf_chunk;                /* features per final-layer weight chunk */
  int32_t rpc0, rpc1, rpc2;        /* rows per weight chunk: initial, hidden, hidden+context (GLU) */
  int32_t wcap, nbuf;              /* weight ring: floats per slot, slots */
  int32_t n_params;                /* floats in d_params */
  float tail_bound, inv_sqrt_h, min_bw, min_bh, min_d, edge_raw;
  int32_t head, M;                 /* SBI_NSF_SPLINE / SBI_NSF_MOG; mixture components (PR = round4(3M)) */
  int32_t cond_mlp;                /* 1: the conditioner is the context-only MLP of the 1-D flow (flow.py:401-408,
                                    * ContextSplineMap :1419-1478): relu(W0 ctx + b0), then NB applications of ONE
                                    * shared hidden layer (W at SBI_L_BLK0, bias at +1) with relu, then the final layer */
  float mog_eps;                   /* std = softplus(.) + mog_eps */
  float ld_zscore;                 /* sum_d log|scale_d| of the input z-score transform */
  const float* d_params;           /* packed parameters (see sbi_b200/pack.py) */
  const int32_t* d_layer_tab;      /* T * SBI_NSF_LAYER_STRIDE */
  const int32_t* d_feat_tab;
  const float* d_stats;            /* [shift(Dp) | scale(Dp) | ctx_mean(Cp) | ctx_std(Cp)] */
} sbi_nsf_model;

/* Optional outputs / inputs of the row kernels; any pointer may be NULL. */
typedef struct {
  const float* d_input;            /* (R, D) row-major, or the gather source when d_index != NULL */
  const float* d_cond;             /* (R, C) row-major, (1, C) when cond_shared, or gather source */
  const int64_t* d_index;          /* (R,) row indices into d_input/d_cond (device-resident data set) */
  int64_t R;
  int32_t cond_shared;             /* 1: one condition row for all R rows (posterior at x_o) */
} sbi_rows;

int sbi_b200_abi_version(void);
int sbi_b200_device_ok(void);      /* 1 if device 0 is sm_90, else 0 */

/* log q(input | cond) for R rows.  d_logp (R,) ; d_noise (R, D) optional (the base-space
 * point z, i.e. NFlowsFlow.inverse_transform). */
int sbi_b200_nsf_logprob(const sbi_nsf_model* m, const sbi_rows* rows, float* d_logp,
                         float* d_noise, void* stream);

/* Vector-Jacobian product of sum_r g_r * log q_r: forward + backward in one kernel.
 *   d_gout (R,) upstream gradient per row, or NULL with g_const used for every row.
 *   d_logp (R,) optional forward output.
 *   d_gpart  (n_part, n_params) per-CTA partial parameter gradients (written, not
 *            accumulated); n_part = sbi_b200_nsf_vjp_parts(R).
 *   d_ginput (R, D), d_gcond (R, C) optional input / condition gradients.
 *   d_loss_acc optional: [0] += sum_r -logp_r , [1] += #non-finite rows.              */
int sbi_b200_nsf_vjp_parts(int64_t R);
int sbi_b200_nsf_vjp(const sbi_nsf_model* m, const sbi_rows* rows, const float* d_gout,
                     float g_const, float* d_logp, float* d_gpart, float* d_ginput,
                     float* d_gcond, float* d_loss_acc, void* stream);

/* x = flow^{-1}(noise | cond): sampling path.  d_noise (R, D) -> d_out (R, D);
 * d_logabsdet (R,) optional = log|det d x / d noise|. */
int sbi_b200_nsf_inverse(const sbi_nsf_model* m, const sbi_rows* rows, float* d_out,
                         float* d_logabsdet, void* stream);

/* `made` sampling (MixtureOfGaussiansMADE.sample, D sequential conditioner passes): d_input of `rows` holds
 * standard-normal draws (R, D), d_uniform (R, D) uniforms in [0, 1) that select the mixture components
 * (inverse CDF); d_out (R, D) samples in the ORIGINAL space (column 0 is the wrapper's dummy feature). */
int sbi_b200_made_sample(const sbi_nsf_model* m, const sbi_rows* rows, const float* d_uniform, float* d_out,
                         void* stream);

/* grad[p] = sum_i gpart[i][p]  (i < n_part) */
int sbi_b200_reduce_partials(const float* d_gpart, int n_part, int64_t n_params, float* d_grad,
                             void* stream);

/* Same, additionally emitting one partial of sum(grad^2) per reduction block (d_sumsq_part,
 * sbi_b200_sumsq_blocks(n_params) floats; masked-out entries excluded) so that the clip norm needs
 * no second pass over the gradient (single-GPU path; after an all-reduce the norm must be retaken). */
int sbi_b200_sumsq_blocks(int64_t n_params);
int sbi_b200_reduce_partials_norm(const float* d_gpart, int n_part, int64_t n_params, float* d_grad,
                                  const uint8_t* d_mask, float* d_sumsq_part, void* stream);

/* Epoch statistics of a validation pass (sbi/inference/trainers/base.py:1195-1225 followed by
 * assert_all_finite): d_out2[0] = -sum of the finite entries of d_logp (n), d_out2[1] = number of
 * non-finite entries.  One launch, fixed summation order. */
int sbi_b200_nll_stats(const float* d_logp, int64_t n, float* d_out2, void* stream);

/* clip_grad_norm_(max_norm) + Adam (torch defaults, no weight decay), in place.
 *   d_state: [m (n) | v (n)] ; d_step: int32 device counter (incremented here);
 *   grad_scale multiplies the gradient first (e.g. 1/world_size after an all-reduce);
 *   d_mask optional (n,) uint8: 0 = frozen entry (padding / structural zero).
 *   max_norm <= 0 disables clipping. */
int sbi_b200_adam_clip_step(float* d_params, const float* d_grad, float* d_state,
                            int32_t* d_step, const uint8_t* d_mask, int64_t n, float lr,
                            float beta1, float beta2, float eps, float max_norm,
                            float grad_scale, void* stream);
/* as above, taking the gradient's sum of squares from d_sumsq_part (n_sumsq partials) instead of
 * recomputing it */
int sbi_b200_adam_clip_step_norm(float* d_params, const float* d_grad, float* d_state,
                                 int32_t* d_step, const uint8_t* d_mask, int64_t n, float lr,
                                 float beta1, float beta2, float eps, float max_norm,
                                 float grad_scale, const float* d_sumsq_part, int n_sumsq,
                                 void* stream);

/* ---- tensor-core bulk evaluation of the NSF (wgmma tf32, 3xTF32 split, fp32 accumulation).
 * Same function as sbi_b200_nsf_logprob (NFlowsFlow.log_prob,
 * sbi/neural_nets/estimators/nflows_flow.py:77-97) for large row counts: the ResidualNet linears
 * (nflows ResidualNet; call site sbi/neural_nets/net_builders/flow.py:411-419) run on the tensor
 * cores, 128 rows per thread block, everything else (spline, LU, base density) per thread.
 *
 * The linears' weights are re-packed from the flat parameter buffer into d_tcw by
 * sbi_b200_nsf_tc_pack (call it whenever d_params changed): per coupling layer a sequence of
 * stages [hi | lo], each half a concatenation of K-major no-swizzle wgmma operand blocks
 * [K/4 slabs][N rows][4 floats] (hi = tf32-rounded weight, lo = weight - hi).
 *   d_src   (n_words,) gather map built by the host (sbi_b200/pack.py NsfLayout.tc_plan):
 *           -1 -> 0 ; s >= 0 -> hi(params[s]) ; s <= -2 -> lo(params[-2-s])
 *   d_tab   T * SBI_NSF_TC_STRIDE ints; per layer: [0] number of stages, [1] round8(n_id),
 *           then 4 ints per stage s at 4+4s: float offset into d_tcw, floats (hi+lo), N of the
 *           main block, aux (final-layer passes: first feature | n_features << 16).
 *           Stage order: initial layer, per block (Wc, W1, W2), final-layer passes of <= 2
 *           spline features (32 rows per feature).
 * Supported when H == 50, H + C <= 64, n_id <= 48, 3*KB-1 <= 32 and the shared-memory plan fits
 * (sbi_b200_nsf_tc_supported); callers use sbi_b200_nsf_logprob otherwise. */
#define SBI_NSF_TC_STRIDE 192
#define SBI_NSF_TC_MAX_STAGES 46
typedef struct {
  int32_t n_words;                 /* floats in d_tcw / entries in d_src */
  int32_t stage_cap;               /* floats of the largest stage (hi + lo) */
  const int32_t* d_src;
  const int32_t* d_tab;
  float* d_tcw;
} sbi_nsf_tc;

int sbi_b200_nsf_tc_supported(const sbi_nsf_model* m, const sbi_nsf_tc* tc);
int sbi_b200_nsf_tc_pack(const sbi_nsf_model* m, const sbi_nsf_tc* tc, void* stream);
int sbi_b200_nsf_logprob_tc(const sbi_nsf_model* m, const sbi_nsf_tc* tc, const sbi_rows* rows,
                            float* d_logp, float* d_noise, void* stream);
/* sampling direction on the same machinery: as sbi_b200_nsf_inverse (NFlowsFlow.sample,
 * sbi/neural_nets/estimators/nflows_flow.py:111-128) */
int sbi_b200_nsf_inverse_tc(const sbi_nsf_model* m, const sbi_nsf_tc* tc, const sbi_rows* rows,
                            float* d_out, float* d_logabsdet, void* stream);

/* ---- tensor-core training step (csrc/nsf_tc.cu forward sweep with activation save + csrc/nsf_vjp_tc.cu
 * backward sweep): the parameter gradients of  sum_r g_r log q(input_r | cond_r)  -- what
 * sbi_b200_nsf_vjp computes with d_ginput == d_gcond == NULL, i.e. NFlowsFlow.loss + autograd backward of a
 * training batch (sbi/neural_nets/estimators/nflows_flow.py:99-109, sbi/inference/trainers/base.py:1171-1180)
 * -- with every conditioner linear (forward, input gradient, weight gradient) on wgmma tf32.
 *   tc_fwd: operand plan of the forward linears (pack.NsfLayout.tc_plan), as for sbi_b200_nsf_logprob_tc;
 *   tc_bwd: operand plan of the transposed linears (pack.NsfLayout.tc_bwd_plan), same descriptor format;
 *           both must have been packed from the current parameters (sbi_b200_nsf_tc_pack);
 *   d_gpart: (sbi_b200_nsf_vjp_tc_parts(R), n_params) partial gradients, reduce with sbi_b200_reduce_partials;
 *   d_save : caller-owned activation scratch of at least sbi_b200_nsf_vjp_tc_save_bytes(m, R) bytes
 *            (one slab per 128-row tile in flight: 3 KB per row and layer);
 *   d_logp (R) and d_loss_acc (2: sum of -log q over finite rows, number of non-finite rows) optional. */
int sbi_b200_nsf_vjp_tc_supported(const sbi_nsf_model* m, const sbi_nsf_tc* tc_fwd, const sbi_nsf_tc* tc_bwd);
int sbi_b200_nsf_vjp_tc_parts(int64_t R);
int64_t sbi_b200_nsf_vjp_tc_save_bytes(const sbi_nsf_model* m, int64_t R);
int sbi_b200_nsf_vjp_tc(const sbi_nsf_model* m, const sbi_nsf_tc* tc_fwd, const sbi_nsf_tc* tc_bwd,
                        const sbi_rows* rows, const float* d_gout, float g_const, float* d_logp,
                        float* d_gpart, float* d_loss_acc, float* d_save, int64_t save_bytes, void* stream);
/* The same step plus the condition gradient d_gcond (R, C) of sum_r g_r log q_r in raw condition space (the
 * context columns of every layer's initial linear and the GLU context linear of every residual block, accumulated
 * per row over the layers; one writer per entry, repeated calls are bit-identical).  The parameter partials are
 * those of sbi_b200_nsf_vjp_tc.  The instantiation adds no shared memory, so _cond_supported applies the same layout
 * check as sbi_b200_nsf_vjp_tc_supported; models it declines run sbi_b200_nsf_vjp with d_gcond. */
int sbi_b200_nsf_vjp_tc_cond_supported(const sbi_nsf_model* m, const sbi_nsf_tc* tc_fwd, const sbi_nsf_tc* tc_bwd);
int sbi_b200_nsf_vjp_tc_cond(const sbi_nsf_model* m, const sbi_nsf_tc* tc_fwd, const sbi_nsf_tc* tc_bwd,
                             const sbi_rows* rows, const float* d_gout, float g_const, float* d_logp,
                             float* d_gpart, float* d_loss_acc, float* d_gcond, float* d_save, int64_t save_bytes,
                             void* stream);

/* ---- masked autoregressive flow (sbi `posterior_nn("maf")`, reference builder
 * sbi/neural_nets/net_builders/flow.py:115-209: T x [MaskedAffineAutoregressiveTransform(MADE,
 * feed-forward blocks, tanh) + RandomPermutation], z-scored input, standardised context).
 * Masked weights are stored already multiplied by their masks. */
#define SBI_MAF_LAYER_STRIDE 32
#define SBI_MAF_AFFINE 0
#define SBI_MAF_RQS 1
enum {
  SBI_M_W0 = 0,   /* [Hp][Dp] masked initial layer */
  SBI_M_B0 = 1,
  SBI_M_WC = 2,   /* [Hp][Cp] context layer */
  SBI_M_BC = 3,
  SBI_M_WF = 4,   /* [OUTp][Hp] masked final layer; rows OUTM*d .. OUTM*d+OUTM-1 parameterise feature d */
  SBI_M_BF = 5,
  SBI_M_PERM = 6, /* offset into perm_tab: perm[D] then inverse perm[D] */
  SBI_M_BLK0 = 8  /* per feed-forward block b: W at SBI_M_BLK0+2b ([Hp][Hp] masked), bias at +1 */
};
typedef struct {
  int32_t D, C, H, NB, T;
  int32_t Dp, Cp, Hp, OUTp;
  int32_t rpc0, rpc1, rpcf;        /* rows per weight chunk: initial(+context), hidden, final */
  int32_t wcap, nbuf, n_params;
  int32_t scale_softplus;          /* 1: softplus(s)+1e-3 (what sbi's maf computes), 0: sigmoid(s+2)+1e-3 */
  /* element-wise transform the MADE parameterises (`head`):
   *   SBI_MAF_AFFINE (0): OUTM = 2, row 2d = unconstrained scale, 2d+1 = shift (`maf`, flow.py:115-209)
   *   SBI_MAF_RQS    (1): OUTM = 3*KB-1 raw spline parameters per feature, linear tails (`maf_rqs`,
   *                       flow.py:212-330: MaskedPiecewiseRationalQuadraticAutoregressiveTransform) */
  int32_t head, KB, OUTM;
  float tail_bound, min_w, min_h, min_d, isq;
  float ld_zscore;
  const float* d_params;
  const int32_t* d_layer_tab;      /* T * SBI_MAF_LAYER_STRIDE */
  const int32_t* d_perm_tab;
  const float* d_stats;            /* [shift(Dp) | scale(Dp) | ctx_mean(Cp) | ctx_std(Cp)] */
} sbi_maf_model;

/* same contracts as the sbi_b200_nsf_* entry points */
int sbi_b200_maf_logprob(const sbi_maf_model* m, const sbi_rows* rows, float* d_logp,
                         float* d_noise, void* stream);
int sbi_b200_maf_vjp_parts(int64_t R);
int sbi_b200_maf_vjp(const sbi_maf_model* m, const sbi_rows* rows, const float* d_gout,
                     float g_const, float* d_logp, float* d_gpart, float* d_ginput,
                     float* d_gcond, float* d_loss_acc, void* stream);
int sbi_b200_maf_inverse(const sbi_maf_model* m, const sbi_rows* rows, float* d_out,
                         float* d_logabsdet, void* stream);

/* ---- ratio estimator: NRE `classifier_nn("resnet")` (reference builder
 * sbi/neural_nets/net_builders/classifier.py:172-235 -> nflows ResidualNet(in=Dt+Dx, out=1,
 * hidden, context=None, num_blocks, relu); wrapper sbi/neural_nets/ratio_estimators.py:132-150:
 * logit = net(cat(standardize(theta), standardize(x)))). */
enum {
  SBI_R_W0 = 0, SBI_R_B0 = 1,   /* [Hp][Dtp+Dxp], columns = [theta | pad | x | pad] */
  SBI_R_WF = 2, SBI_R_BF = 3,   /* [4][Hp] (row 0 is the logit) */
  SBI_R_BLK0 = 4                /* per block b: W1,B1,W2,B2 at SBI_R_BLK0 + 4b */
};
typedef struct {
  int32_t Dt, Dx, H, NB;
  int32_t Dtp, Dxp, Hp;
  int32_t rpc0, rpc1;
  int32_t wcap, nbuf, n_params;
  const float* d_params;
  const int32_t* d_tab;           /* SBI_R_* offsets */
  const float* d_stats;           /* [theta_mean(Dtp) | theta_std(Dtp) | x_mean(Dxp) | x_std(Dxp)] */
} sbi_ratio_model;

/* rows of (theta, x) pairs: pair r = (theta[ti[r]], x[xi[r]]); NULL index = identity;
 * x_shared = 1: every pair uses x row 0 (potential at a fixed observation). */
typedef struct {
  const float* d_theta;
  const float* d_x;
  const int64_t* d_theta_index;
  const int64_t* d_x_index;
  int64_t R;
  int32_t x_shared;
} sbi_pairs;

/* unnormalised log-ratio logits (R,) -- RatioEstimator.forward, ratio_estimators.py:132-154 */
int sbi_b200_ratio_forward(const sbi_ratio_model* m, const sbi_pairs* pairs, float* d_logits,
                           void* stream);
/* VJP of sum_r g_r logit_r: d_gpart (n_part, n_params) per-CTA partial parameter gradients,
 * d_gtheta (R, Dt) optional gradient wrt the theta of each pair; d_logits optional. */
int sbi_b200_ratio_vjp_parts(int64_t R);
int sbi_b200_ratio_vjp(const sbi_ratio_model* m, const sbi_pairs* pairs, const float* d_gout,
                       float* d_logits, float* d_gpart, float* d_gtheta, void* stream);
/* the same VJP with both input gradients: d_gtheta (R, Dt) and d_gx (R, Dx) per pair, each optional
 * (NULL = not wanted), divided by the side's std (1 where an embedding net standardises in torch).
 * d_gpart, d_logits and d_gtheta are bit-identical with and without d_gx. */
int sbi_b200_ratio_vjp_inputs(const sbi_ratio_model* m, const sbi_pairs* pairs, const float* d_gout,
                              float* d_logits, float* d_gpart, float* d_gtheta, float* d_gx, void* stream);
/* per-row sums of per-pair rows (gradients of gathered rows): d_out (n_rows, width) with
 * out[j] = sum_{k in [row_ptr[j], row_ptr[j+1])} gpair[order[k]], added in k order by one owner per
 * entry (no atomics: repeat calls are bit-identical); d_order NULL = consecutive segments (order[k] = k).
 * d_row_ptr (n_rows + 1,) int64, non-decreasing. */
int sbi_b200_pair_rows_sum(const float* d_gpair, int32_t width, const int64_t* d_order,
                           const int64_t* d_row_ptr, int64_t n_rows, float* d_out, void* stream);

/* ---- ratio estimator: NRE `classifier_nn("mlp")` and `classifier_nn("linear")` (reference builders
 * sbi/neural_nets/net_builders/classifier.py:49-169):
 *   mlp:    logit = Linear(H,1)(relu(N(Linear(H,H)(relu(N(Linear(Dt+Dx,H)(u)))))))
 *   linear: logit = Linear(Dt+Dx,1)(u)
 * with u = cat(standardize(theta), standardize(x)) and N = nn.LayerNorm(H) (biased variance over the
 * H features of a row, eps `ln_eps`, affine) or nn.Identity.  NL = number of hidden layers (2 or 0). */
enum {
  SBI_RM_W0 = 0, SBI_RM_B0 = 1,    /* hidden layer l at 4l: Linear [Hp][Kp] (Kp = Dtp+Dxp for l = 0, Hp after; */
  SBI_RM_G0 = 2, SBI_RM_BE0 = 3,   /*   columns of layer 0 = [theta | pad | x | pad]), LayerNorm gamma, beta [Hp] */
  SBI_RM_WF = 8, SBI_RM_BF = 9     /* output layer [4][Hp], or [4][Dtp+Dxp] when NL = 0 (row 0 is the logit) */
};
enum { SBI_RM_NORM_NONE = 0, SBI_RM_NORM_LAYER = 1 };
typedef struct {
  int32_t Dt, Dx, H, NL;
  int32_t Dtp, Dxp, Hp;
  int32_t norm;                   /* SBI_RM_NORM_* */
  float ln_eps;
  int32_t rpc0, rpc1;             /* weight rows per ring chunk: layer 0 / later layers */
  int32_t wcap, nbuf, n_params;
  const float* d_params;
  const int32_t* d_tab;           /* SBI_RM_* offsets */
  const float* d_stats;           /* as sbi_ratio_model */
} sbi_ratio_mlp_model;

/* same contracts as sbi_b200_ratio_forward / _vjp_parts / _vjp.  A shape whose tile does not fit the
 * 227 KB of shared memory of one CTA returns SBI_ESMEM. */
int sbi_b200_ratio_mlp_forward(const sbi_ratio_mlp_model* m, const sbi_pairs* pairs, float* d_logits,
                               void* stream);
int sbi_b200_ratio_mlp_vjp_parts(int64_t R);
int sbi_b200_ratio_mlp_vjp(const sbi_ratio_mlp_model* m, const sbi_pairs* pairs, const float* d_gout,
                           float* d_logits, float* d_gpart, float* d_gtheta, void* stream);

/* tensor-core bulk evaluation of the classifier (same operand format and `sbi_nsf_tc` descriptor as
 * the NSF path: d_tab holds ONE stage list: initial layer, per block (W1, W2), final layer as an
 * N = 16 block whose row 0 is the weight vector; [1] = round8(Dt + Dx)).  Supported when H == 50 and
 * Dt + Dx <= 56.  Gather map: sbi_b200/pack.py RatioLayout.tc_plan. */
int sbi_b200_ratio_tc_supported(const sbi_ratio_model* m, const sbi_nsf_tc* tc);
int sbi_b200_ratio_tc_pack(const sbi_ratio_model* m, const sbi_nsf_tc* tc, void* stream);
int sbi_b200_ratio_forward_tc(const sbi_ratio_model* m, const sbi_nsf_tc* tc, const sbi_pairs* pairs,
                              float* d_logits, void* stream);

/* ---- lock-step vectorized slice sampler (state machine of
 * sbi/samplers/mcmc/slice_numpy.py:412-587 `SliceSamplerVectorized.run`): one thread per chain,
 * chain state resident in HBM, one launch per lock-step between two potential evaluations.
 * Coordinate-wise slice sampling with stepping-out (bracket width tuned as the running mean of the
 * bracket sizes during the first `tuning` sweeps) and shrinkage; random dimension order per sweep. */
enum { SBI_SLICE_BEGIN = 0, SBI_SLICE_LOWER = 1, SBI_SLICE_UPPER = 2, SBI_SLICE_SAMPLE = 3, SBI_SLICE_DONE = 4 };
typedef struct {
  int32_t C, D;                 /* chains, dimensions */
  int32_t num_samples, tuning;  /* sweeps to record per chain, tuning sweeps before recording */
  double init_width, max_width;
  uint64_t seed;
  double* d_x;                  /* (C, D) current position (in/out) */
  double* d_width;              /* (C, D) */
  int32_t* d_order;             /* (C, D) */
  int32_t* d_istate;            /* (C, 4): state, i, t, - */
  double* d_fstate;             /* (C, 8): cxi, wi, lx, ux, xi, logu, -, - */
  void* d_rng;                  /* (C, 64 bytes) Philox state */
  double* d_samples;            /* (C, num_samples, D) */
} sbi_slice_chains;

/* initialise chain state from d_x; writes the first parameters to evaluate into d_params (C, D) f32 */
int sbi_b200_slice_init(const sbi_slice_chains* s, float* d_params, void* stream);
/* one lock-step: consume d_logp (C,) evaluated at d_params, advance every chain, write the next
 * d_params; d_n_done[0] = number of chains in state DONE after this step */
int sbi_b200_slice_step(const sbi_slice_chains* s, const float* d_logp, float* d_params,
                        int32_t* d_n_done, void* stream);

/* ---- lock-step HMC / NUTS (`mcmc_method="hmc_pyro"` / `"nuts_pyro"`): one thread per chain, one
 * launch per lock-step, one leapfrog step per chain per lock-step.  Every chain runs its own
 * adaptation (dual-averaged step size, diagonal mass matrix over Stan's windows).  Between two
 * lock-steps the host evaluates log p and its gradient at d_params.  Layouts are column-per-chain
 * so that the threads of a warp touch consecutive words:
 *   d_vec    (SBI_HMC_NV0 + 4 * max_tree_depth, D, C) f64 working vectors (csrc/hmc.cu),
 *   d_istate (SBI_HMC_NI, C) i32, d_fstate (SBI_HMC_NF0 + 2 * max_tree_depth, C) f64,
 *   d_normal (D, C) f64 and d_uniform (max_tree_depth + 1, C) f64: this lock-step's draws.
 * Random numbers: a chain draws a fresh momentum from d_normal (at most once per lock-step); the
 * direction of a new doubling is d_uniform[0] < 0.5 (right); the progressive-sampling choice of the
 * merge that forms a 2^(k+1)-leaf subtree uses d_uniform[1 + k]; the top-level NUTS choice and the
 * HMC Metropolis test use d_uniform[max_tree_depth].  Other entries are left unused. */
#define SBI_HMC_NV0 11
#define SBI_HMC_NI 14
#define SBI_HMC_NF0 10
#define SBI_HMC_MAX_TREE_DEPTH 30
#define SBI_HMC_MAX_WINDOWS 64
#define SBI_HMC_TRACE_SCALARS 5
enum { SBI_HMC_NUTS = 0, SBI_HMC_HMC = 1 };
enum { SBI_HMC_PHASE_INIT = 0, SBI_HMC_PHASE_FIND = 1, SBI_HMC_PHASE_TRAJ = 2, SBI_HMC_PHASE_DONE = 3 };
typedef struct {
  int32_t C, D;
  int32_t algo;                       /* SBI_HMC_NUTS or SBI_HMC_HMC */
  int32_t max_tree_depth;             /* NUTS doublings per transition, 1..SBI_HMC_MAX_TREE_DEPTH */
  int32_t warmup, num_samples;        /* adapted transitions, then recorded transitions */
  int32_t adapt_step_size, adapt_mass_matrix;
  int32_t n_windows;                  /* adaptation windows: window w ends at transition win_end[w] */
  int32_t win_end[SBI_HMC_MAX_WINDOWS];
  double step_size;                   /* initial step size */
  double target_accept, trajectory_length;
  double* d_z;                        /* (C, D) position: initial state in, last state out */
  double* d_vec;
  int32_t* d_istate;
  double* d_fstate;
  const double* d_normal;
  const double* d_uniform;
  const float* d_logp;                /* (C,) log p at d_params (written by the host) */
  const float* d_grad;                /* (C, D) d log p / d params (written by the host) */
  float* d_params;                    /* (C, D) next point to evaluate (written by the kernel) */
  double* d_samples;                  /* (C, num_samples, D) recorded positions */
  double* d_trace;                    /* optional (C, warmup + num_samples, 2 D + 5): position, inverse
                                         mass, tree depth, leapfrog steps, divergent, accept stat, step
                                         size of every transition (the last two sets as used by it) */
} sbi_hmc_chains;

/* initialise the chain state (unit inverse mass, initial step size) and write d_z to d_params */
int sbi_b200_hmc_init(const sbi_hmc_chains* s, void* stream);
/* one lock-step: consume d_logp / d_grad at d_params and this lock-step's draws, advance every chain
 * by one potential evaluation, write the next d_params; d_n_done[0] = chains that are done */
int sbi_b200_hmc_step(const sbi_hmc_chains* s, int32_t* d_n_done, void* stream);

/* ---- flow matching (FMPE): VectorFieldMLP behind FlowMatchingEstimator
 * (net: sbi/neural_nets/net_builders/vector_field_nets.py:610-719, sinusoidal time embedding
 * :367-421; estimator: sbi/neural_nets/estimators/flowmatching_estimator.py:205-347). */
#define SBI_FM_MAX_LAYERS 12
enum {
  SBI_F_WI = 0, SBI_F_BI = 1,    /* input_layer        [Hp][Dp] */
  SBI_F_WC = 2, SBI_F_BC = 3,    /* condition_layer    [Hp][Cp] */
  SBI_F_WM = 4, SBI_F_BM = 5,    /* input_merge_layer  [Hp][2Hp], columns = [input emb | cond emb] */
  SBI_F_WT = 6, SBI_F_BT = 7,    /* time_linear_layer  [Hp][TEp] */
  SBI_F_WO = 8, SBI_F_BO = 9,    /* output_layer       [Dp][Hp] */
  SBI_F_LAYER0 = 12              /* per hidden layer i: W, B, LN gamma, LN beta at SBI_F_LAYER0 + 4i */
};
typedef struct {
  int32_t D, C, H, NL, TE;          /* theta dim, (embedded) condition dim, hidden, layers, time-emb dim */
  int32_t Dp, Cp, Hp, TEp;
  int32_t rpc_i, rpc_c, rpc_m, rpc_t, rpc_h, rpc_o;   /* rows per weight chunk of each matrix */
  int32_t wcap, nbuf, n_params;
  float noise_scale;                /* sigma_min = 1e-3 */
  float ln_eps;
  int32_t raw;                      /* 1: the bare network (score estimators): d_input is already the network
                                     * input, d_time the value fed to the time embedding, outputs are the raw
                                     * network outputs -- no flow-matching noising / standardisation / rescaling */
  int32_t pad_;
  const float* d_params;
  const int32_t* d_tab;
  const float* d_stats;             /* [mean_0(Dp) | std_0(Dp) | ctx_mean(Cp) | ctx_std(Cp) | div_term(TEp/2)] */
} sbi_fm_model;

/* v(theta_t, t; x) in ORIGINAL space (FlowMatchingEstimator.forward :205-268): d_theta (R,D),
 * d_cond (R,C) or (1,C) when cond_shared, d_time (R,) or (1,) when time_shared -> d_v (R,D). */
int sbi_b200_fm_forward(const sbi_fm_model* m, const sbi_rows* rows, const float* d_time,
                        int32_t time_shared, float* d_v, void* stream);
/* the same velocity field and its exact divergence sum_i dv_i/dtheta_i (d_div (R,); d_v optional): the
 * right-hand side of the augmented neural ODE behind `VectorFieldPosterior.log_prob`
 * (sbi/samplers/ode_solvers/zuko_ode.py:80-124 -> zuko FreeFormJacobianTransform(exact=True);
 * sbi/inference/potentials/vector_field_potential.py:145-212).  With m->raw the kernel writes the DIAGONAL of the bare
 * network's input Jacobian instead, d_div (R, D): the caller (score estimators) weights it per dimension. */
int sbi_b200_fm_forward_div(const sbi_fm_model* m, const sbi_rows* rows, const float* d_time,
                            int32_t time_shared, float* d_v, float* d_div, void* stream);
/* flow-matching loss of a batch and its parameter gradient (FlowMatchingEstimator.loss :270-347
 * + backward): rows = (theta_0, x) pairs, d_time (R,) in [0,1], d_eps (R,D) ~ N(0,I).
 * d_loss (R,) optional; d_gpart (n_part, n_params) partial gradients of sum_r g_r * loss_r. */
int sbi_b200_fm_vjp_parts(int64_t R);
int sbi_b200_fm_loss_vjp(const sbi_fm_model* m, const sbi_rows* rows, const float* d_time,
                         const float* d_eps, const float* d_gout, float g_const, float* d_loss,
                         float* d_gpart, float* d_loss_acc, void* stream);
/* the same, plus the gradient of sum_r g_r * loss_r with respect to the condition rows as given in d_cond:
 * d_gcond (R, C), through condition_layer and the in-kernel z-score (an embedding net's output when the caller
 * embeds the condition itself with identity statistics).  One writer per entry: repeated calls are bit-identical.
 * sbi_b200_fm_loss_vjp is this call with d_gcond == NULL. */
int sbi_b200_fm_loss_vjp_cond(const sbi_fm_model* m, const sbi_rows* rows, const float* d_time,
                              const float* d_eps, const float* d_gout, float g_const, float* d_loss,
                              float* d_gpart, float* d_loss_acc, float* d_gcond, void* stream);

/* Introspection, no device work: the weight-pipeline plan (ring depth, chunk rows, shared memory) that a launch of
 * kernel 0 (sbi_b200_fm_forward), 1 (sbi_b200_fm_loss_vjp / sbi_b200_fm_net_vjp) or 2 (sbi_b200_fm_forward_div)
 * uses for this model: out10 = [nbuf, wcap, rpc_i, rpc_c, rpc_m, rpc_t, rpc_h, rpc_o, dynamic smem bytes, output
 * rows per thread].  The launches re-chunk the caller's plan to fill the 227 KB of shared memory. */
int sbi_b200_fm_plan(const sbi_fm_model* m, int32_t kernel, int32_t* out10);

/* Parameter gradient of the bare network for a given upstream gradient d_dout (R, D) of its outputs (m->raw must
 * be 1): the backward of `ConditionalScoreEstimator.forward` (sbi/neural_nets/estimators/score_estimator.py:149-215)
 * through the VectorFieldMLP; everything around the network (time-dependent z-scoring, the Gaussian skip term, the
 * denoising-score-matching loss with its control variate, :230-316) is element-wise host code.
 * d_gpart (sbi_b200_fm_vjp_parts(R), n_params) receives per-CTA partial gradients. */
int sbi_b200_fm_net_vjp(const sbi_fm_model* m, const sbi_rows* rows, const float* d_time, const float* d_dout,
                        float* d_gpart, void* stream);

/* ---- adaptive Dormand-Prince 5(4) with the step control on the device (csrc/ode.cu), replacing the
 * host-side loop of the solver the reference delegates to (zuko.utils.odeint; call sites
 * sbi/samplers/ode_solvers/zuko_ode.py:80-124, sbi/inference/posteriors/vector_field_posterior.py:436-505).
 * The state is a flat fp32 vector of n entries; d_k holds the 7 stage derivatives (7 x n).  One step =
 * k_0 given (first-same-as-last), for i = 1..6: sbi_b200_ode_stage(i) then the caller's right-hand side at
 * time d_ctrl->t_stage into k_i; then sbi_b200_ode_error_commit.  Before the first step: stage 0 (copies y,
 * sets t_stage = t) and the right-hand side into k_0.  The host only polls d_ctrl->done. */
typedef struct {
  float t, h, t1, dir;      /* clock, signed step, end time, +1 / -1 */
  float atol, rtol;
  float t_stage;            /* time of the stage just prepared (input of the right-hand side) */
  float en;                 /* error norm of the last step */
  int32_t nfe, nsteps, naccept;
  int32_t done;             /* 0 running, 1 reached t1, 2 max_steps exhausted */
  int32_t max_steps;
  int32_t pad_[3];
} sbi_ode_ctrl;
int sbi_b200_ode_red_size(int64_t n);        /* floats of scratch the error reduction needs */
int sbi_b200_ode_stage(const float* d_y, const float* d_k, float* d_yi, int64_t n, int32_t stage,
                       sbi_ode_ctrl* d_ctrl, void* stream);
int sbi_b200_ode_error_commit(float* d_y, float* d_k, float* d_y5, float* d_red, int64_t n,
                              sbi_ode_ctrl* d_ctrl, void* stream);

/* One Euler-Maruyama step of the reverse SDE of the flow-matching estimator (csrc/ode.cu; reference
 * sbi/samplers/score/predictors.py:112-120 on flowmatching_estimator.py:374-469): d_theta (n = R*D) is
 * updated in place from the velocity d_v at time ts[i-1] and the normal draw d_z; d_ctrl = [current time,
 * step index i] (floats) is advanced to ts[i], i+1, so that a captured step can be replayed. */
int sbi_b200_sde_em_step(float* d_theta, const float* d_v, const float* d_z, int64_t n, const float* d_ts,
                         float* d_ctrl, float eta, float noise_scale, float t_eff, void* stream);

/* ---- rejection sampling: accept / reject + order-preserving compaction of one batch of proposals
 * (csrc/compact.cu; reference sbi/samplers/rejection/rejection.py:170-200, `keep = exp(potential - scaled
 * proposal log-prob) > u; candidates[keep]`).  Accepted rows are appended, in proposal order, at
 * d_out[*d_count ...] (rows past `cap` are dropped but counted), their global proposal indices
 * (index_base + position) at d_out_idx (optional); *d_count is advanced on the device.
 * d_scratch: sbi_b200_reject_scratch_ints(n) int32. */
int64_t sbi_b200_reject_scratch_ints(int64_t n);
int sbi_b200_reject_compact(const float* d_cand, int32_t D, const float* d_log_target, const float* d_log_scaled,
                            const float* d_u, int64_t n, int64_t index_base, float* d_out, int64_t* d_out_idx,
                            int64_t cap, int32_t* d_count, int32_t* d_scratch, void* stream);

/* ---- sampling-importance-resampling: one categorical draw per group of K proposals (csrc/compact.cu; reference
 * sbi/samplers/importance/sir.py:59-63).  Candidates are (groups*K, D) rows; per group g, lw_k = log_target_k -
 * log_proposal_k (fp32), w = softmax(lw), and the selected candidate is the first k with cumsum(w)_k >= u_g.  A
 * group selects nothing when its softmax is NaN (a NaN or +inf log weight, or all -inf) or when the cumulative
 * weights never reach u_g.  Selected rows are appended, in group order, at d_out[*d_count ...] (rows past `cap`
 * are dropped but counted), their global group indices (index_base + g) at d_out_idx (optional); *d_count is
 * advanced on the device.  d_scratch: sbi_b200_sir_scratch_ints(groups) int32. */
int64_t sbi_b200_sir_scratch_ints(int64_t groups);
int sbi_b200_sir_select(const float* d_cand, int32_t D, const float* d_log_target, const float* d_log_proposal,
                        const float* d_u, int64_t groups, int32_t K, int64_t index_base, float* d_out,
                        int64_t* d_out_idx, int64_t cap, int32_t* d_count, int32_t* d_scratch, void* stream);

/* ---- MMD misspecification test (csrc/mmd.cu; reference sbi/diagnostics/misspecification.py:19-110) ----------------
 * S index sets over the rows of d_z (R, D) fp32.  Set s takes rows d_idx[s*L + i] (int32, in [0, R)): its first
 * nx_s rows form X and the next ny_s rows form Y (d_nxy: (S, 2) int32, nx_s <= max_nx, ny_s <= max_ny,
 * nx_s + ny_s <= L <= SBI_MMD_MAX_ROWS, S <= SBI_MMD_MAX_SETS).  Unless `given_bw`, the bandwidth d_bw[s] is
 * written as the exact lower median of the nx_s*ny_s X-Y distances (NaN for an empty X or Y); with `given_bw` it is
 * read.  d_mmd[s] (fp64) receives the biased or, with `unbiased`, the reference's unbiased RBF MMD
 * (K = exp(-d^2 / (2 h^2))); a null d_mmd computes the bandwidths only.  d_ws: sbi_b200_mmd_ws_bytes(S) bytes.
 * The launch sequence does not depend on S, and a set's results depend only on its own rows. */
#define SBI_MMD_MAX_ROWS 65536
#define SBI_MMD_MAX_SETS 65536
int64_t sbi_b200_mmd_ws_bytes(int32_t S);
int sbi_b200_mmd(const float* d_z, int64_t R, int32_t D, const int32_t* d_idx, int32_t L, const int32_t* d_nxy,
                 int32_t S, int32_t max_nx, int32_t max_ny, int32_t unbiased, int32_t given_bw, float* d_bw,
                 double* d_mmd, void* d_ws, void* stream);
/* out (nx, ny) = exp(-|x_i - y_j|^2 / (2 bandwidth^2)) for x (nx, D), y (ny, D) fp32. */
int sbi_b200_rbf_matrix(const float* d_x, int64_t nx, const float* d_y, int64_t ny, int32_t D, double bandwidth,
                        float* d_out, void* stream);

/* ---- L-C2ST classifiers (csrc/lc2st.cu; reference sbi/diagnostics/lc2st.py with scikit-learn's
 * MLPClassifier(solver="adam", activation="relu")).  A network maps F = dim_theta + dim_x inputs through L ReLU
 * hidden layers to one logistic output p = P(class 1).  Parameters are packed per model in sklearn's order:
 * coefs_[0] (F x H[0], row-major), intercepts_[0], coefs_[1], intercepts_[1], ..., coefs_[L] (H[L-1] x 1),
 * intercepts_[L]; P counts them.  Envelope: F <= SBI_LC2ST_MAX_F, 1 <= L <= SBI_LC2ST_MAX_HIDDEN, every width
 * <= SBI_LC2ST_MAX_WIDTH, and the model's weights and gradient fit one CTA's shared memory with 8-row tiles
 * (sbi_b200_lc2st_plan returns SBI_ESMEM otherwise). */
#define SBI_LC2ST_MAX_HIDDEN 4
#define SBI_LC2ST_MAX_F 64
#define SBI_LC2ST_MAX_WIDTH 256
typedef struct {
  int32_t F, L;
  int32_t H[SBI_LC2ST_MAX_HIDDEN];
  int32_t P;
} sbi_lc2st_net;

/* sklearn's hyperparameters.  batch_size < 1 selects min(200, n_train); the float fields are the float32 values
 * numpy applies (one_minus_beta* = float32(1 - beta) computed in float64), the double fields the Python floats. */
typedef struct {
  int32_t max_iter, n_iter_no_change, early_stopping, shuffle, batch_size;
  float beta1, beta2, one_minus_beta1, one_minus_beta2, eps, alpha;
  double lr_d, beta1_d, beta2_d, tol;
} sbi_lc2st_opt;

/* One model of a training launch.  Its samples are entries row0 .. row0 + n_train + n_val - 1 of d_rows (pairs
 * (theta row, x row) of the shared tables) and d_labels (0 or 1): the n_train training samples, then the n_val
 * validation samples.  Epoch `e` visits training sample d_order[order0 + e * n_train + i] at position i, or, with
 * order0 < 0, a keyed bijection of [0, n_train) drawn from (key, e) on the device (identity when !shuffle). */
typedef struct {
  int64_t row0;
  int32_t n_train, n_val;
  int64_t order0;
  uint64_t key;
} sbi_lc2st_job;

/* out3 = {training tile rows, evaluation tile rows, padded parameter count}; SBI_ESMEM when a model does not fit. */
int sbi_b200_lc2st_plan(const sbi_lc2st_net* net, int32_t* out3);
/* floats of the training workspace of M models (Adam moments and best weights) */
int64_t sbi_b200_lc2st_ws_floats(const sbi_lc2st_net* net, int32_t M);
/* Train M models to completion in one launch (one CTA each).  d_params (M, P): initial parameters in, final ones
 * out (the best-validation ones when early_stopping).  Per model: d_n_iter = n_iter_, d_val_curve /
 * d_loss_curve (M, max_iter) float64 = validation accuracy / epoch loss per epoch run, d_best = the best
 * validation score (early stopping) or the best loss. */
int sbi_b200_lc2st_train(const sbi_lc2st_net* net, const sbi_lc2st_opt* opt, const sbi_lc2st_job* d_jobs, int32_t M,
                         const float* d_theta, int32_t dt, const float* d_x, int32_t dx, const int32_t* d_rows,
                         const float* d_labels, const int32_t* d_order, float* d_params, float* d_ws,
                         int32_t* d_n_iter, double* d_val_curve, double* d_loss_curve, double* d_best, void* stream);
/* row chunks of an evaluation over S rows (the length of d_part per classifier) */
int sbi_b200_lc2st_eval_chunks(const sbi_lc2st_net* net, int64_t S);
/* Evaluate C classifiers of E consecutive parameter sets each (d_params: (C*E, P)) on S rows [theta_s, x]: theta
 * from d_theta (G, S, dt) at block d_group[c] (block 0 when d_group is NULL), x = d_x (dx) for every row.
 * d_prob (C, S) = mean over members of 1 - p; d_score (C) = sum_s (prob - 0.5)^2 / S in float64; d_part:
 * (C, sbi_b200_lc2st_eval_chunks(net, S)) doubles of scratch. */
int sbi_b200_lc2st_eval(const sbi_lc2st_net* net, const float* d_params, int32_t C, int32_t E, const float* d_theta,
                        int32_t dt, int64_t S, const int32_t* d_group, const float* d_x, int32_t dx, float* d_prob,
                        double* d_part, double* d_score, void* stream);

/* ---- multi-GPU: gradient sum over NVLink peer memory (csrc/peer.cu), replacing the NCCL all-reduce +
 * norm pass of the data-parallel step (reference semantics: clip_grad_norm_ + Adam on the summed
 * gradient, sbi/inference/trainers/base.py:1181-1187).  Each rank allocates a symmetric buffer
 * (`peer_alloc`), exports its IPC handle (64 bytes) to the other ranks of the node, imports theirs, and
 * then calls `peer_sum` once per step with the table of all ranks' buffers (own buffer at [rank]):
 * d_grad_out = sum over ranks (fixed rank order) of d_grad_local, plus sbi_b200_peer_blocks(n) partials
 * of sum(g^2) for sbi_b200_adam_clip_step_norm.  The step number that tags the flags is read from the
 * exchange's own device counter inside the symmetric buffer (d_step == NULL; advanced by the kernel, never
 * rewound) or from d_step[0] (a caller-owned counter, e.g. the optimizer's), so the launch can sit in a
 * CUDA graph. */
int64_t sbi_b200_peer_bytes(int64_t n_params);
int sbi_b200_peer_blocks(int64_t n_params);
void* sbi_b200_peer_alloc(int64_t n_params);
int sbi_b200_peer_free(void* p);
int sbi_b200_peer_export(void* p, void* handle64);
void* sbi_b200_peer_import(const void* handle64);
int sbi_b200_peer_close(void* p);
int sbi_b200_peer_sum(const float* d_grad_local, void* const* h_peer_ptrs, int world, int rank,
                      int64_t n_params, float* d_grad_out, const uint8_t* d_mask, float* d_sumsq_part,
                      const int32_t* d_step, void* stream);
int sbi_b200_peer_error(const void* p, int64_t n_params);

/* ---- host-buffer entry points (the end-to-end path a CPU caller binds) ------------------
 * Device staging / optimizer buffers are owned by the caller and passed in a workspace;
 * h_* buffers should be pinned for full PCIe bandwidth.  These calls copy host->device,
 * run the kernels, copy the result device->host and block until it has landed. */
typedef struct {
  float* d_input;        /* (cap_rows, D) staging */
  float* d_cond;         /* (cap_rows, C) staging */
  float* d_logp;         /* (cap_rows) */
  float* d_gpart;        /* (sbi_b200_nsf_vjp_parts(cap_rows), n_params), zero-initialised once */
  float* d_grad;         /* (n_params) */
  float* d_state;        /* (2*n_params) Adam m | v */
  int32_t* d_step;       /* (2) */
  const uint8_t* d_mask; /* (n_params) or NULL */
  float* d_loss_acc;     /* (2) */
  int64_t cap_rows;
  float* d_sumsq;        /* (sbi_b200_sumsq_blocks(n_params)) scratch for the clip norm, or NULL */
  /* optional: run the step's forward+backward on the tensor cores (sbi_b200_nsf_vjp_tc); all NULL / 0
   * selects the SIMT kernel.  tc_pack covers both operand plans (one sbi_b200_nsf_tc_pack launch per
   * step re-packs them from the just-updated parameters); d_gpart must then hold
   * sbi_b200_nsf_vjp_tc_parts(B) slabs and d_save sbi_b200_nsf_vjp_tc_save_bytes(m, B) bytes. */
  const sbi_nsf_tc* tc_pack;
  const sbi_nsf_tc* tc_fwd;
  const sbi_nsf_tc* tc_bwd;
  float* d_save;
  int64_t save_bytes;
} sbi_train_ws;

/* One optimisation step on a host batch (replaces one iteration of
 * sbi/inference/trainers/base.py:1171-1187 incl. the batch `.to(device)` of
 * npe_base.py:722-726): loss = mean_r -log q(theta_r | x_r); h_loss_out[0] = sum_r -log q,
 * h_loss_out[1] = number of non-finite rows. */
int sbi_b200_nsf_train_step_host(const sbi_nsf_model* m, const sbi_train_ws* ws,
                                 const float* h_input, const float* h_cond, int64_t B, float lr,
                                 float beta1, float beta2, float eps, float max_norm,
                                 float* h_loss_out, void* stream);

/* Pipelined variant: enqueues step i (H2D of its pinned host batch, kernels, D2H of its loss) and
 * returns after step i-1 has completed, handing back step i-1's result in h_loss_prev[2] (NaN on
 * the first call).  Every step still carries its own H2D + D2H; the host just prepares batch i+1
 * while the device runs step i.  The caller alternates between two pinned host batch buffers
 * (buffer i%2 may be rewritten once call i+1 has returned).  `pipe` from sbi_b200_pipe_create. */
void* sbi_b200_pipe_create(void);
void sbi_b200_pipe_destroy(void* pipe);
int sbi_b200_nsf_train_step_host_async(const sbi_nsf_model* m, const sbi_train_ws* ws, void* pipe,
                                       const float* h_input, const float* h_cond, int64_t B, float lr,
                                       float beta1, float beta2, float eps, float max_norm,
                                       float* h_loss_prev, void* stream);
/* wait for the last enqueued step and return its result in h_loss_last[2] */
int sbi_b200_pipe_drain(void* pipe, float* h_loss_last);

/* Data-parallel pipelined host step (one process per GPU): as sbi_b200_nsf_train_step_host_async, with the
 * gradient sum over NVLink peer memory (sbi_b200_peer_sum, exchange-owned step counter) between the
 * partial-gradient reduction and clip+Adam; rows of all ranks form one global batch of B * world rows
 * (reference semantics: one optimizer step on the mean loss of the global batch,
 * sbi/inference/trainers/base.py:1171-1187).  ws->d_sumsq must hold sbi_b200_peer_blocks(n_params) floats. */
typedef struct {
  void* const* h_peer_ptrs;   /* (world) symmetric buffers, own buffer at [rank] (host array) */
  int world, rank;
  float* d_grad_local;        /* (n_params) scratch for this rank's reduced gradient */
} sbi_peer_ctx;
int sbi_b200_nsf_train_step_host_async_dp(const sbi_nsf_model* m, const sbi_train_ws* ws, void* pipe,
                                          const sbi_peer_ctx* peer, const float* h_input, const float* h_cond,
                                          int64_t B, float lr, float beta1, float beta2, float eps,
                                          float max_norm, float* h_loss_prev, void* stream);

/* log q(input_r | cond) for R host rows (cond: (R,C), or (1,C) when cond_shared). */
int sbi_b200_nsf_logprob_host(const sbi_nsf_model* m, const sbi_train_ws* ws,
                              const float* h_input, const float* h_cond, int64_t R,
                              int cond_shared, float* h_logp, void* stream);

/* same through the tensor-core kernel (sbi_b200_nsf_logprob_tc), in chunks whose host<->device
 * copies overlap the kernels of their neighbours; re-packs tc->d_tcw first. */
int sbi_b200_nsf_logprob_host_tc(const sbi_nsf_model* m, const sbi_nsf_tc* tc, const sbi_train_ws* ws,
                                 const float* h_input, const float* h_cond, int64_t R,
                                 int cond_shared, float* h_logp, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SBI_B200_H */
