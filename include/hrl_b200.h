/*
 * hrl_b200.h -- C ABI of the H100-native (sm_90a) HandyRL learner hot path.
 *
 * The reference (DeNA/HandyRL) is pure Python and has no FFI layer; the seam this
 * header introduces is the operator level underneath these reference functions:
 *
 *   hrl_loss_fwd_bwd      <- handyrl/train.py:176-184 (mask epilogue of forward_prediction)
 *                            handyrl/train.py:218-267 (compute_loss)
 *                            handyrl/train.py:189-215 (compose_losses)
 *                            handyrl/losses.py:16-80  (monte_carlo / temporal_difference / upgo / vtrace)
 *                            + the autograd pass of train.py:369 restricted to those ops
 *   hrl_loss_fwd_bwd_diag <- the same pass + learner diagnostics sums (importance ratios, advantages, value fit);
 *                            no reference counterpart
 *   hrl_loss_fwd          <- the forward half alone: compute_loss (train.py:189-267) on held-out data, no update
 *   hrl_compute_target   <- handyrl/losses.py:63-80  (compute_target, stand-alone)
 *   hrl_peer_allreduce_sumsq <- the gradient exchange nn.DataParallel does implicitly (train.py:339-340), as a
 *                            fused peer-memory kernel
 *   hrl_grad_sumsq /
 *   hrl_clip_adam_step    <- handyrl/train.py:370-371 (clip_grad_norm_(params, 4.0) + Adam.step,
 *                            Adam(lr, weight_decay=1e-5) of train.py:331)
 *   hrl_lamb_plan /
 *   hrl_clip_lamb_step    <- the same clip + LAMB (Adam with per-tensor trust ratios) in place of Adam; opt-in, no
 *                            reference counterpart
 *   hrl_muon_plan /
 *   hrl_clip_muon_step    <- the same clip + Muon (momentum orthogonalised by Newton-Schulz iterations) on the weight
 *                            matrices, Adam on the other words; opt-in, no reference counterpart
 *   hrl_step_commit       <- with the guard of hrl_clip_adam_step: the same step, rejected on the device when its loss
 *                            or gradient is not finite; no reference counterpart
 *   hrl_weight_ema        <- a per-step moving average of the weights; no reference counterpart (scripts/aux_swa.py
 *                            averages epoch checkpoints)
 *   hrl_gather_pad        <- handyrl/train.py:33-124  (make_batch: window slice + pad + collate)
 *   hrl_gather_pad_sym    <- the same gather with each window rotated / mirrored by a board-symmetry table; no
 *                            reference counterpart
 *   hrl_replay_sample /
 *   hrl_replay_priority_update <- prioritised replay: Batcher.select_episode's recency law (train.py:291-315) times a
 *                            per-episode priority, with importance weights; no reference counterpart
 *   hrl_distill_fwd_bwd   <- an annealed KL(teacher || student) term on the trained policy rows ("kickstarting"), launched
 *                            after hrl_loss_fwd_bwd; no reference counterpart
 *   hrl_value_bins_expect /
 *   hrl_value_bins_fwd_bwd <- categorical value / return heads (two-hot or HL-Gauss targets, cross-entropy) in place of
 *                            the squared-error / smooth-L1 terms of compose_losses (train.py:204-206); opt-in, no
 *                            reference counterpart
 *   hrl_gemm_tf32x3       <- the Linear/Conv contractions of the user's net inside train.py:142-146 (+ autograd, :369)
 *
 * Conventions
 *   - plain C, no torch types; every pointer is a DEVICE pointer unless stated;
 *   - the caller owns every buffer (inputs, outputs, workspace); the library allocates nothing;
 *   - kernels are enqueued on the stream handed in (a cudaStream_t passed as void*), no
 *     internal synchronisation, safe to capture in a CUDA graph;
 *   - return value 0 = success, negative = HrlStatus error; hrl_last_error() gives the text
 *     for the calling thread.  Nothing throws across this boundary.
 *   - tensors are contiguous, batch-major exactly as make_batch emits them
 *     (B, T, P|Pa, ...) fp32, `action` int64 (train.py:44-45, 111-124).
 */
#ifndef HRL_B200_H_
#define HRL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HRL_ABI_VERSION 3

typedef enum {
    HRL_OK = 0,
    HRL_ERR_BAD_ARG = -1,      /* null pointer, bad dimension, unknown algorithm id        */
    HRL_ERR_WORKSPACE = -2,    /* workspace missing or smaller than hrl_*_workspace_bytes   */
    HRL_ERR_UNSUPPORTED = -3,  /* shape outside what the kernels were built for             */
    HRL_ERR_CUDA = -4          /* a CUDA runtime call failed; see hrl_last_error()          */
} HrlStatus;

/* target algorithms, the strings of config.yaml `policy_target` / `value_target`
 * (reference config.yaml:26-27, losses.py:68-78) */
typedef enum { HRL_MC = 0, HRL_TD = 1, HRL_UPGO = 2, HRL_VTRACE = 3 } HrlAlgo;

/* index of each reduced scalar in HrlLossArgs.losses */
enum { HRL_LOSS_P = 0, HRL_LOSS_V = 1, HRL_LOSS_R = 2, HRL_LOSS_ENT = 3, HRL_LOSS_TOTAL = 4,
       HRL_LOSS_DCNT = 5, HRL_NUM_LOSS = 6 };

/*
 * One fused forward+backward pass of the loss over a replay batch.
 *
 * Dimensions: B windows, T = burn_in + forward steps, P players on the value side,
 * Pa players on the policy side (1 for the turn-alternating layout, else P; train.py:65-68),
 * A actions (A <= 1024 and P <= 64 are built; larger values return HRL_ERR_UNSUPPORTED).  Steps t < burn_in are
 * excluded from every loss term and receive zero gradients (train.py:220-222).
 */
/* Kernel selection and tuning of hrl_loss_fwd_bwd.  All zero = the library's own choice (what production uses);
 * the fields exist so that tests and profiling can force every code path WITHOUT process-global state (the library
 * reads no environment variables). */
typedef struct HrlLossTuning {
    int32_t variant;     /* 0 auto | 1 rows, direct loads | 2 rows, cp.async-staged | 3 bulk (TMA, wide rows) |
                            4 element-parallel | 5 lane-group (A <= 32); inapplicable variants fall back to rows */
    int32_t recurrence;  /* 0 auto (serial below 96 steps) | 1 serial loops | 2 parallel suffix scan           */
    int32_t cluster;     /* bulk kernel: CTAs per window, 0 auto | 1 | 2 | 4 | 8                               */
    int32_t consumers;   /* bulk kernel: row-reducing warps per CTA, 0 = 16                                    */
    int32_t threads;     /* threads per CTA for the other variants, 0 auto                                     */
    int32_t unstaged;    /* rows kernel: 1 = recompute masked logits instead of staging them in shared memory  */
    long long *trace;    /* device buffer of >= 32 clock64 stamps written by CTA 0 (debugging), or NULL        */
} HrlLossTuning;

typedef struct HrlLossArgs {
    int32_t B, T, P, Pa, A;
    int32_t burn_in;
    int32_t value_target;        /* HrlAlgo, used for targets (train.py:257-258)            */
    int32_t policy_target;       /* HrlAlgo, used for advantages (train.py:260-262)         */
    int32_t two_player_zero_sum; /* turn_based_training && P == 2 (train.py:243)            */
    float lambda;                /* args['lambda']                                           */
    float gamma;                 /* args['gamma'] (return stream; the value stream uses 1)   */
    float entropy_regularization;
    float entropy_regularization_decay;

    /* raw net outputs (before the mask epilogue) */
    const float *policy_raw;     /* (B,T,Pa,A)                                               */
    const float *value_raw;      /* (B,T,Pa)   or NULL when the net has no value head        */
    const float *return_raw;     /* (B,T,Pa)   or NULL when the net has no return head       */

    /* replay batch */
    const float *action_mask;    /* (B,T,Pa,A) 0 legal / 1e32 illegal                        */
    const int64_t *action;       /* (B,T,Pa)                                                 */
    const float *selected_prob;  /* (B,T,Pa)   behaviour probability                         */
    const float *reward;         /* (B,T,P)                                                  */
    const float *ret;            /* (B,T,P)    batch['return']                               */
    const float *turn_mask;      /* (B,T,P)                                                  */
    const float *observation_mask; /* (B,T,P)                                                */
    const float *episode_mask;   /* (B,T)                                                    */
    const float *progress;       /* (B,T)                                                    */
    const float *outcome;        /* (B,P)                                                    */

    /* outputs */
    float *dpolicy_raw;          /* (B,T,Pa,A) d total / d policy_raw                        */
    float *dvalue_raw;           /* (B,T,Pa)   or NULL iff value_raw is NULL                 */
    float *dreturn_raw;          /* (B,T,Pa)   or NULL iff return_raw is NULL                */
    float *losses;               /* [HRL_NUM_LOSS] p, v, r, ent, total, dcnt (sums)          */

    /* optional per-element taps for parity tests; each may be NULL */
    float *tap_target_value;     /* (B,T,P) targets['value']  (t >= burn_in, 0 before)       */
    float *tap_target_return;    /* (B,T,P) targets['return']                                */
    float *tap_advantage;        /* (B,T,P) total_advantages broadcast to P (train.py:265)   */
    float *tap_logp;             /* (B,T,Pa) log pi(a) * episode_mask (train.py:232)         */
    float *tap_rho;              /* (B,T,Pa) clipped importance ratio (train.py:237)         */
    float *tap_entropy;          /* (B,T,Pa) policy entropy per row (train.py:208)           */

    void *workspace;             /* >= hrl_loss_workspace_bytes(...) bytes, 256-byte aligned;
                                    its first 64 bytes must be zero on the first call and are
                                    left zero by every call                                  */
    size_t workspace_bytes;
    HrlLossTuning tuning;        /* zero-initialise for the defaults                         */
    int32_t io_bf16;             /* 1: policy_raw and dpolicy_raw hold bf16 (same shapes): 8 instead of 12 bytes per action
                                    move through HBM.  Wide rows only (256 < A <= 512, A % 8 == 0); everything in between --
                                    masks, softmax statistics, targets, the gradient before its final rounding -- stays fp32, so
                                    the losses equal those of the fp32 call on the widened logits bit for bit              */
    int32_t external_heads;      /* heads whose loss another kernel computes (categorical heads, hrl_value_bins_fwd_bwd):
                                    bit 0 value, bit 1 return.  For such a head the pass still reads its raw output (the
                                    expectation) to form targets, advantages and the diagnostics sums, but adds no term to
                                    losses[HRL_LOSS_V|R] (left 0) or the total, never writes its gradient -- whose pointer must
                                    be NULL -- and requires its tap_target_* (where the cross-entropy kernel reads the targets).
                                    0 = every present head is a scalar regression, as before.  It fills the padding before
                                    window_weight: the struct keeps its size and every other offset                     */
    const float *window_weight;  /* (B) importance weight of each window (prioritised replay), or NULL = 1.  It multiplies every
                                    per-cell loss term of window b (policy, value, return, entropy, entropy regulariser) and
                                    their gradients; dcnt and the diagnostics sums stay unweighted.  Weights of exactly 1
                                    give losses and gradients bit-identical to NULL                                       */
} HrlLossArgs;

/* Bytes of workspace hrl_loss_fwd_bwd needs for these dimensions (host call, no GPU work). */
size_t hrl_loss_workspace_bytes(int32_t B, int32_t T, int32_t P, int32_t Pa, int32_t A);

/* Enqueue the fused loss pass.  `stream` is a cudaStream_t. */
int hrl_loss_fwd_bwd(const HrlLossArgs *args, void *stream);

/* The forward half of hrl_loss_fwd_bwd (held-out validation losses): the same struct, workspace, shapes (bf16 logits included)
 * and choice of kernel, with the gradient phase compiled out.  Writes `losses` (bit-identical to hrl_loss_fwd_bwd on the
 * same inputs) and the taps that are given; dpolicy_raw, dvalue_raw and dreturn_raw may be NULL and are never written.
 * window_weight is ignored: held-out losses are never weighted. */
int hrl_loss_fwd(const HrlLossArgs *args, void *stream);

/*
 * Learner diagnostics (opt-in): additive sums, so that shards add up and the sums can ride the gradient all-reduce.
 * The loss pass sums over trained cells (t >= burn_in), column i = (b, t, p), tm = turn_mask, om = observation_mask,
 * q = the column's policy row (0 when Pa == 1, else p):
 *   n_pol     sum tm                                 (== HRL_LOSS_DCNT)
 *   rho       sum tm * rho, rho = exp(l) UNclipped,  l = log pi(a) * em - log(clamp(mu, 1e-16, 1)) * em   (em = episode_mask)
 *   rho_clip  sum tm * [rho > 1]                     (samples the V-Trace / UPGO clip at 1 acts on)
 *   logr      sum tm * l         logr2  sum tm * l^2 (-logr / n_pol estimates KL(mu || pi))
 *   adv       sum tm * Adv       adv2   sum tm * Adv^2   (Adv = the clipped-rho total advantage, train.py:265)
 *   n_val     sum om             (value head only; the value / return sums stay 0 without their head)
 *   tv, tv2   sum om * tgt_v, sum om * tgt_v^2         ev, ev2   sum om * (tgt_v - v), sum om * (tgt_v - v)^2, v = value_raw * om
 *   tr, tr2, er, er2   the same for the return head
 * The optimiser step sums g, g^2, [g > max_norm] and 1 per step, g = the pre-clip global gradient norm.
 */
enum { HRL_DIAG_N_POL = 0, HRL_DIAG_RHO = 1, HRL_DIAG_RHO_CLIP = 2, HRL_DIAG_LOGR = 3, HRL_DIAG_LOGR2 = 4, HRL_DIAG_ADV = 5,
       HRL_DIAG_ADV2 = 6, HRL_DIAG_N_VAL = 7, HRL_DIAG_TV = 8, HRL_DIAG_TV2 = 9, HRL_DIAG_EV = 10, HRL_DIAG_EV2 = 11,
       HRL_DIAG_TR = 12, HRL_DIAG_TR2 = 13, HRL_DIAG_ER = 14, HRL_DIAG_ER2 = 15,
       HRL_NUM_LOSS_DIAG = 16,                                   /* the sums of the loss pass come first */
       HRL_DIAG_GNORM = 16, HRL_DIAG_GNORM2 = 17, HRL_DIAG_GCLIP = 18, HRL_DIAG_STEPS = 19,
       HRL_NUM_DIAG = 20 };

/* Workspace of hrl_loss_fwd_bwd_diag (>= hrl_loss_workspace_bytes; same zero-header rule). */
size_t hrl_loss_diag_workspace_bytes(int32_t B, int32_t T, int32_t P, int32_t Pa, int32_t A);

/* hrl_loss_fwd_bwd with the diagnostics sums accumulated in the same pass: the same kernels with the extra block sums
 * compiled in, folded by the last CTA in a fixed order in fp64.  Losses and gradients are bit-identical to
 * hrl_loss_fwd_bwd.  diag: HRL_NUM_DIAG device floats, overwritten (the optimiser entries with 0). */
int hrl_loss_fwd_bwd_diag(const HrlLossArgs *args, float *diag, void *stream);

/*
 * Stand-alone compute_target (losses.py:63-80) on (B,T,P) columns.
 *   values   (B,T,P) or NULL  -> targets = advantages = returns (losses.py:64-66)
 *   returns  (B,Tr,P) with Tr == T or Tr == 1 (the (B,1,P,1) outcome of train.py:254)
 *   rewards  (B,T,P) or NULL (= 0)
 *   rhos, cs (B,T,Pr) with Pr == P or Pr == 1 (broadcast over players)
 *   masks    (B,T,P)
 *   targets, advantages (B,T,P) outputs
 */
int hrl_compute_target(int32_t algo, int32_t B, int32_t T, int32_t P, int32_t Tr, int32_t Pr,
                       const float *values, const float *returns, const float *rewards,
                       float lambda, float gamma, const float *rhos, const float *cs,
                       const float *masks, float *targets, float *advantages, void *stream);

/*
 * Optimiser step on one flat fp32 parameter bucket (train.py:370-371).
 *
 * hrl_grad_sumsq writes per-block partial sums of grad^2 into `partials`
 * (hrl_sumsq_num_partials() floats); hrl_clip_adam_step reduces them in a fixed order,
 * applies clip_grad_norm_(max_norm) and one Adam step with L2 weight decay
 * (torch.optim.Adam semantics: grad += wd * param before the moments).
 *
 * `lr` and `step` live on the device so that a captured CUDA graph stays valid while
 * the learner changes the learning rate every epoch (train.py:383-384); the kernel
 * increments *step.
 */
int32_t hrl_sumsq_num_partials(void);
int hrl_grad_sumsq(const float *grad, int64_t n, float *partials, void *stream);
int hrl_clip_adam_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq,
                       int64_t n, const float *partials, const float *lr, int64_t *step,
                       double max_norm, double beta1, double beta2, double eps, double weight_decay,
                       float *grad_norm_out /* may be NULL */, double *diag_accum /* may be NULL */,
                       const float *tail, int32_t n_tail, int32_t *skip /* may be NULL */, void *stream);
/*
 * diag_accum != NULL: the same launch also adds g, g^2, [g > max_norm] and 1 (g = the pre-clip norm) to diag_accum[0..3]
 * (device doubles, the HRL_DIAG_GNORM .. HRL_DIAG_STEPS entries of a diagnostics accumulator).
 *
 * skip != NULL: the guarded step (opt-in; a batch carrying a NaN or Inf must not poison the learner).  The step is rejected
 * when the pre-clip norm -- the fp64 fold of the fp32 partials -- is not finite, or when one of tail[0 .. n_tail) is not
 * finite (tail: the loss sums in the reduced bucket).  A finite gradient whose fp32 sum of squares overflows makes a
 * partial Inf, so it is rejected too.  Every block folds the same partials and reads the same tail, so all blocks (and all
 * ranks of a sharded learner, which see the same reduced bucket) decide alike without communicating.
 *   accepted: the arithmetic of the unguarded step, bit for bit;
 *   rejected: param, exp_avg, exp_avg_sq and diag_accum are not written, and *step is not incremented.
 * *grad_norm_out is written either way.  *skip (device int32) is set to 1 when rejected, 0 when accepted.  skip == NULL:
 * tail and n_tail are ignored and every step is taken.
 */

/*
 * LAMB on the same bucket (opt-in; You et al., 2020, Algorithm 2): Adam's moments with one trust ratio per parameter tensor,
 * so that each tensor's relative step is bounded by lr * lr_scale whatever the batch size.  With t the step count after this
 * step, c the clip coefficient of hrl_clip_adam_step (same partials, same fold) and w the weights before the step:
 *     g = c * grad                          (no weight_decay * w term here, unlike hrl_clip_adam_step)
 *     m = m + (g - m)(1 - beta1);   v = beta2 v + (1 - beta2) g^2          (fp32, hrl_clip_adam_step's order)
 *     u = (m / (1 - beta1^t)) / (sqrt(v) / sqrt(1 - beta2^t) + eps) + weight_decay * w
 *     r_i = |w_i| / |u_i| over the words of tensor i when both are > 0, else 1
 *     w <- w - (lr * lr_scale * r_i) * u
 * Tensor i is words [off_i, off_i + numel_i) of the bucket, in order; words outside every tensor (padding) are not touched.
 *
 * hrl_lamb_plan (host, no device work): cuts tensors of numel[0 .. n_tensors) words, laid out back to back from word 0, into
 * chunks of at most 1024 words that never cross a tensor, and returns their count (a negative HrlStatus on error:
 * HRL_ERR_BAD_ARG for numel NULL, n_tensors <= 0 or a numel <= 0).  plan != NULL (a host buffer of 5 int64 per chunk)
 * receives, per chunk in bucket order, {first word, words, tensor index, the tensor's first chunk, the tensor's chunk count}.
 *
 * hrl_clip_lamb_step: three launches -- the moments, u (into `update`, n floats of scratch) and per-chunk fp64 sums of w^2
 * and u^2 (into chunk_sums, 2 * n_chunks doubles); the ratios (each folded from its tensor's chunk sums in a fixed order, so
 * repeated launches, graph replays and ranks give identical bits) and the weight update; then *step += 1.  `plan` is
 * hrl_lamb_plan's table (n_chunks entries) copied to the device.  partials, lr, step, grad_norm_out, diag_accum, tail,
 * n_tail and skip mean what they mean for hrl_clip_adam_step, and the guard rejects on the same condition: a rejected step
 * writes neither param, the moments, update, chunk_sums, ratio nor diag_accum, and does not count.  ratio != NULL (device
 * floats, one per tensor) receives each tensor's r_i.  HRL_ERR_BAD_ARG: a required pointer NULL, n <= 0, n_chunks <= 0,
 * tail NULL with n_tail > 0 under the guard, or lr_scale not finite and > 0.
 */
int64_t hrl_lamb_plan(const int64_t *numel, int32_t n_tensors, int64_t *plan /* may be NULL */);
int hrl_clip_lamb_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, float *update, int64_t n,
                       const int64_t *plan, int32_t n_chunks, double *chunk_sums, const float *partials, const float *lr,
                       int64_t *step, double max_norm, double beta1, double beta2, double eps, double weight_decay,
                       double lr_scale, float *grad_norm_out /* may be NULL */, double *diag_accum /* may be NULL */,
                       const float *tail, int32_t n_tail, int32_t *skip /* may be NULL */, float *ratio /* may be NULL */,
                       void *stream);

/*
 * Muon on the same bucket (opt-in): each weight matrix's Nesterov momentum, orthogonalised by five Newton-Schulz
 * iterations, replaces Adam's step on that matrix; every other word takes hrl_clip_adam_step's update bit for bit.  A tensor
 * of shape (r, ...) is viewed as the r x k matrix, k = numel / r.  It is Muon-owned (HRL_MUON_MATRIX) when it has two or
 * more dimensions, min(r, k) >= 2 and the matrix fits one CTA: with m <= n its sides and m_p, n_p those rounded up to 16,
 * m_p <= 128 and m_p * n_p <= 128 * 576.  A matrix with min(r, k) >= 2 outside that is HRL_MUON_TOO_LARGE and takes Adam,
 * as does everything else (HRL_MUON_ADAM).  With c the clip coefficient of hrl_clip_adam_step, lr the device's learning
 * rate and W, M a Muon-owned matrix and its momentum (the exp_avg words; its exp_avg_sq words are not touched):
 *     G = c * grad;   M <- 0.95 M + G;   N = G + 0.95 M                       (fp32, each product and sum rounded)
 *     X = N / (|N|_F + 1e-7) as bf16, transposed when r > k so that X is m x n
 *     5 times:  A = bf16(X X^T);  B = bf16(b A + c A A);  X = bf16(a X + B X)   (a, b, c) = (3.4445, -4.7750, 2.0315)
 *     O = X (transposed back);   W <- W - lr (s O + weight_decay W),   s = fp32(lr_scale * 0.2 * sqrt(max(r, k)))
 * The products take bf16 operands (round to nearest even) and accumulate in fp32 on the tensor cores.
 *
 * hrl_muon_plan (host, no device work): tensors t < n_tensors of ndim[t] dimensions dims[...] (the shapes back to back; a
 * scalar has ndim 0), laid out back to back from word 0.  kind[t] receives its HrlMuonKind and counts[0..1] the numbers of
 * matrices and of Adam spans.  mats != NULL (4 int64 per matrix) receives {first word, r, k, transposed} per Muon-owned
 * tensor in bucket order; spans != NULL (2 int64 per span) receives {first word, words}: the Adam-owned words in runs of
 * adjacent tensors, cut into pieces of at most 4096.  HRL_ERR_BAD_ARG: a NULL pointer, n_tensors <= 0, ndim < 0 or an empty
 * dimension.
 *
 * hrl_clip_muon_step: two launches -- one CTA per matrix and one per Adam span of hrl_muon_plan's tables (copied to the
 * device), then *step += 1; the same count as hrl_clip_adam_step.  Fixed-order reductions and no atomics: repeated launches,
 * graph replays and ranks give identical bits.  partials, lr, step, grad_norm_out, diag_accum, tail, n_tail and skip mean
 * what they mean for hrl_clip_adam_step, and the guard rejects on the same condition: a rejected step writes neither param,
 * the moments, ortho nor diag_accum, and does not count.  ortho != NULL (n device floats) receives O at each matrix's words.
 * HRL_ERR_BAD_ARG: a required pointer NULL, n <= 0, an empty plan, tail NULL with n_tail > 0 under the guard, or lr_scale
 * not finite and > 0.
 */
typedef enum { HRL_MUON_ADAM = 0, HRL_MUON_MATRIX = 1, HRL_MUON_TOO_LARGE = 2 } HrlMuonKind;
int hrl_muon_plan(const int64_t *dims, const int32_t *ndim, int32_t n_tensors, int32_t *kind, int32_t *counts,
                  int64_t *mats /* may be NULL */, int64_t *spans /* may be NULL */);
int hrl_clip_muon_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t n, const int64_t *mats,
                       int32_t n_mats, const int64_t *spans, int32_t n_spans, const float *partials, const float *lr,
                       int64_t *step, double max_norm, double beta1, double beta2, double eps, double weight_decay,
                       double lr_scale, float *grad_norm_out /* may be NULL */, double *diag_accum /* may be NULL */,
                       const float *tail, int32_t n_tail, int32_t *skip /* may be NULL */, float *ortho /* may be NULL */,
                       void *stream);

/*
 * The accumulation that follows a guarded step, in one launch that reads *skip:
 *   accepted: accum[i] += (double)tail[i] for i < n_tail (the step's bucket tail: the epoch's loss sums, then the
 *             distillation and loss-pass diagnostics sums when they are on);
 *   rejected: *skip_count += 1, and nbytes bytes of `saved` are copied back to `state` (the buffers -- BatchNorm running
 *             statistics, num_batches_tracked -- as they were before the step's forward moved them).
 * skip_count must not lie in accum[0 .. n_tail).  state and saved are 16-byte aligned; nbytes may be 0.
 */
int hrl_step_commit(const int32_t *skip, const float *tail, int32_t n_tail, double *accum, double *skip_count,
                    void *state, const void *saved, int64_t nbytes, void *stream);

/*
 * Moving average of the learner's weights (opt-in, no reference counterpart; reference scripts/aux_swa.py averages
 * epoch checkpoints instead).  Enqueued after the optimiser step, on the n fp32 words of the learner's state -- the
 * parameters (zero pad included) and the fp32 buffers (BatchNorm running statistics):
 *     avg[i] <- fmaf(w, state[i] - avg[i], avg[i]),   w = max(1 - decay, 1 / t)   (fp32),   t = *step
 * where *step is the optimiser's step counter after this step's increment (hrl_clip_adam_step), read on the device so
 * that a captured CUDA graph replays correctly.  The first step (t = 1, w = 1) stores state[i] exactly and early steps
 * form an equal running mean; seeded != 0 (an average resumed from a saved one) uses w = 1 - decay from its first step.  Elementwise and
 * deterministic; avg and state 16-byte aligned, any n > 0, decay in (0, 1).  After a guarded step (skip != NULL, the
 * flag of hrl_clip_adam_step) nothing is written when *skip says the step was rejected.
 */
int hrl_weight_ema(float *avg, const float *state, int64_t n, const int64_t *step, float decay, int32_t seeded,
                   const int32_t *skip /* may be NULL */, void *stream);

/*
 * Gradient accumulation (opt-in; a batch trained as k micro-batches with one optimiser step): the fused loss pass of
 * micro-batch i leaves its sums in row i of a (k, ld) buffer, and one launch folds them into the bucket tail:
 *     out[j] = (float) sum_{i = 0..k-1} (double) rows[i*ld + j]      for j < n,
 * in that fixed order (bit-reproducible), rounded once.  out may not overlap rows.
 */
int hrl_sum_rows(const float *rows, int32_t k, int64_t ld, int32_t n, float *out, void *stream);

/*
 * Multi-GPU form of the same step: one-shot all-reduce (SUM) of the flat gradient bucket over NVLink peer
 * memory, fused with the sum-of-squares partials hrl_clip_adam_step consumes (replaces NCCL all-reduce +
 * hrl_grad_sumsq).  Every rank reads every rank's bucket directly (P2P loads through NVSwitch), adds them in
 * rank order -- all ranks get bit-identical sums -- and writes the result to `out_sum`.
 *   peer_buckets  device array [world] of pointers: this process's mapping of rank r's bucket (index r);
 *                 each bucket holds n floats followed by 2*world uint32 flags (zero-initialised once)
 *   flag_offset   index (in 32-bit words from the bucket start) of the flags
 *   n, n_norm     floats to reduce; the first n_norm of them (the gradients proper, not the loss sums riding in
 *                 the tail) enter the sum of squares
 *   epoch, ticket device uint32, zero-initialised once; maintained by the kernel (CUDA-graph safe)
 *   status        device uint32, zero-initialised once; set to 1 (and left there) if a peer rank did not arrive
 *                 within 20 s -- the kernel then gives up instead of spinning forever and its sums are invalid
 * Ranks synchronise inside the kernel with release/acquire flags at system scope: "my gradients are ready"
 * before the loads, "I am done reading" after them, so the next step may overwrite the bucket.
 */
int hrl_peer_allreduce_sumsq(float *out_sum, const float *const *peer_buckets, int64_t flag_offset, int32_t world,
                             int32_t rank, int64_t n, int64_t n_norm, float *partials, uint32_t *epoch, uint32_t *ticket,
                             uint32_t *status, void *stream);

/*
 * fp32-accurate matrix product on the tensor cores (wgmma.mma_async .tf32 with the 3xTF32 hi/lo split, fp32
 * accumulation in registers) -- the dense contractions of the user's net (fastnet.py runs a convolution over a
 * tiny board as one such product per direction), i.e. what torch.nn.functional.linear / conv2d and their autograd
 * do inside reference train.py:142-146, 369.
 *     C[M x N] = A_op[M x K] * B_op[N x K]^T (+ bias[N])
 *   a_kmajor / b_kmajor  1: element (row, k) of the operand at  row * ld + k  (reduction dimension contiguous)
 *                        0: at  k * ld + row  (the operand is stored transposed, e.g. reduce over samples)
 *   splits               K slices computed by separate CTAs into `workspace` (hrl_gemm_workspace_floats floats) and
 *                        summed in a fixed order (deterministic); 1 = no split, workspace may be NULL.  A split
 *                        product takes no bias and needs ldc == N; with C == NULL the slice partials
 *                        (hrl_gemm_effective_splits of them, M*N floats apart) are left in the workspace.
 * Relative error ~1e-6 of sum_k |a||b| (plain fp32 summation is ~1e-7 * sqrt(K)); NOT the 1e-3 of single-pass TF32.
 */
size_t hrl_gemm_workspace_floats(int64_t M, int64_t N, int64_t K, int32_t splits);
int32_t hrl_gemm_effective_splits(int64_t K, int32_t splits);   /* slices really produced (whole 32-element chunks) */
int hrl_gemm_tf32x3(const float *A, int64_t lda, int32_t a_kmajor, const float *B, int64_t ldb, int32_t b_kmajor,
                    const float *bias, float *C, int64_t ldc, int64_t M, int64_t N, int64_t K, int32_t splits,
                    float *workspace, void *stream);

/*
 * The same product with the elementwise neighbours of a conv -> BatchNorm -> ReLU tower fused into it, so that a layer of
 * the user's net is ONE launch per direction (forward / input gradient / weight gradient) instead of a product plus
 * separate normalisation, activation and reduction passes over the (samples x features) activations:
 *   operand transform   v = x * p[f] + y * q[f] + r[f], optionally clamped at 0, applied while the operand is staged:
 *                       BatchNorm-apply + ReLU of the previous layer (x = its raw output, p = gamma*rstd, r = beta - mean*p),
 *                       or the BatchNorm backward dY = dZ*p + Y*q + r (x = dZ, y = Y).  f = the reduction index, or the
 *                       operand row when feature_is_row (transposed operands of the weight-gradient product).
 *   epilogues           RELU: C = max(acc + bias, 0).  STATS: C = acc and per-column sum / sum of squares of C - ep_mean
 *                       over the tile (BatchNorm batch statistics of this layer's output, shifted by a pivot near the
 *                       mean so that they do not cancel; ep_mean NULL = no shift).  MASK_STATS: C = acc * (z > 0) with
 *                       z = y*scale + shift of the pre-activation y (ReLU backward) and per-column sums of C and
 *                       C * (y - mean) * rstd (the two batch sums of the BatchNorm backward).
 * Column sums land in col_partials[row_tile][2][N] (row_tile = ceil(M/128) tiles, summed by hrl_bn_finalize_*).
 */
typedef struct HrlGemmOperand {
    const float *ptr;            /* the operand as it lies in memory                                   */
    const float *ptr2;           /* optional second source with the same layout (y above), or NULL     */
    const float *p, *q, *r;      /* per-feature constants, NULL = plain operand (q only with ptr2)     */
    int64_t ld;
    int32_t kmajor;              /* 1: element (row,k) at row*ld + k; 0: at k*ld + row                 */
    int32_t relu;
    int32_t feature_is_row;
    int32_t packed;              /* B only: ptr is an hrl_board_pack image (weights pre-split into TF32 hi/lo halves and
                                    pre-swizzled, one contiguous block per 32-element chunk: staged by ONE bulk copy)  */
} HrlGemmOperand;

typedef enum { HRL_GEMM_EP_STORE = 0, HRL_GEMM_EP_RELU = 1, HRL_GEMM_EP_STATS = 2, HRL_GEMM_EP_MASK_STATS = 3 } HrlGemmEpilogue;

typedef struct HrlGemmArgs {
    HrlGemmOperand a, b;         /* C[M x N] = A_op[M x K] * B_op[N x K]^T                            */
    const float *bias;           /* per column, or NULL                                                */
    float *C;
    int64_t ldc, M, N, K;
    int32_t splits;              /* as hrl_gemm_tf32x3 (plain epilogue only)                           */
    int32_t epilogue;            /* HrlGemmEpilogue                                                    */
    float *workspace;
    const float *ep_y;           /* MASK_STATS: pre-activation tile (M x N)                            */
    int64_t ep_ldy;
    const float *ep_scale, *ep_shift;   /* per column; NULL = 1 / 0                                    */
    const float *ep_mean, *ep_rstd;     /* per column; MASK_STATS: NULL = second sum is sum(C * y);
                                           STATS: ep_mean = the pivot of the sums, ep_rstd unused     */
    float *col_partials;         /* [ceil(M/128)][2][N] floats, or NULL                                */
    /* Convolution over a board as an implicit product (replaces cuDNN's fp32 SIMT kernels for the stride-1 "same" / wrap-around
     * convolutions of the board nets: reference geister.py:18-56 ConvLSTM cells, hungry_geese.py:20-37 TorusConv2d).  Activations
     * are channels-last: a row is a pixel, ld its stride in floats.  conv_off[cell * taps + tap] = (cell the tap reads) - cell, or
     * HRL_CONV_OUTSIDE under zero padding; wrap-around boards have no outside (hrl_conv_geometry fills it).
     *   conv_mode 1  forward / input gradient: A = input pixels (M = pixels, a.ld >= conv_cin), B = hrl_conv_pack image, K = taps *
     *                (conv_cin padded to a multiple of 32); the input gradient is the same product of dy with the adjoint image.
     *   conv_mode 2  weight gradient: A = dy [pixels][Cout] (kmajor 0), B = input [pixels][conv_cin] (kmajor 0), N = taps * conv_cin,
     *                K = pixels, split over K slices; hrl_conv_wgrad_reduce sums the slices into the (Cout, Cin, kh, kw) gradient. */
    const int16_t *conv_off;
    int32_t conv_mode, conv_hw, conv_taps, conv_cin;
    /* conv_mode 2 over several (dy, x) pairs that share ONE weight -- a recurrent cell applied at every time step: segments > 0,
     * seg_a[i] / seg_b[i] (host arrays of device pointers, at most 64) replace a.ptr / b.ptr, every pair has K pixels and gets
     * `splits` K slices; C must be NULL, the (segments * effective splits) slice partials stay in the workspace for
     * hrl_conv_wgrad_reduce2.  conv_ones_row = 1 appends a B row of ones: N = taps * conv_cin + 1, and the last column of the result is
     * sum_pixels dy = the bias gradient. */
    const float *const *seg_a;
    const float *const *seg_b;
    int32_t segments, conv_ones_row;
    /* bf16 != 0: the product on bf16 operands (0 = 3xTF32, as hrl_gemm_tf32x3).  Each operand element goes through its
     * transform in fp32 (fmaf, optional ReLU) and is then rounded to the nearest bf16, ties to even; the products of the
     * rounded operands are exact in fp32 and accumulate in fp32 registers (wgmma .f32.bf16.bf16, k16).  Bias, epilogues,
     * statistics sums, split-K partials and the ones row are fp32 as in the 3xTF32 form.  Relative error of an output
     * ~2^-8 of sum_k |a||b| (each operand within 2^-9 relative), not the ~1e-6 of 3xTF32.  A packed B must then be a bf16
     * image: hrl_board_pack_many / _pivot with HrlPackJob.bf16, or hrl_conv_pack_bf16. */
    int32_t bf16;
} HrlGemmArgs;

#define HRL_CONV_OUTSIDE (-32768)
/* table (H*W*kh*kw int16, host memory) of the neighbour offsets above; wrap != 0: the board is a torus */
int hrl_conv_geometry(int32_t H, int32_t W, int32_t kh, int32_t kw, int32_t wrap, int16_t *table);
/* weights (Cout, Cin, kh, kw) -> packed B images (zero them once): forward (rows = Cout, reduction = tap-major, Cin padded to 32)
 * and adjoint (rows = Cin, reduction = flipped tap, Cout padded to 32).  Either may be NULL. */
size_t hrl_conv_pack_floats(int32_t rows, int32_t channels, int32_t taps);
int hrl_conv_pack(const float *w, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw, float *image_fwd, float *image_adj, void *stream);
/* The same images for HrlGemmArgs.bf16 products: bf16 weights (round to nearest even), [chunk][n_pad rows][64 bytes,
 * SWIZZLE_64B: 16-byte slot j of row r at j ^ ((r >> 1) & 3)].  Each takes hrl_conv_pack_floats(...) / 4 floats. */
int hrl_conv_pack_bf16(const float *w, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw, float *image_fwd, float *image_adj,
                       void *stream);
/* dw[co][ci][a][b] = sum over slices of partials[s][co][(a*kw+b)*Cin + ci]  (fixed order) */
int hrl_conv_wgrad_reduce(const float *partials, int32_t splits, float *dw, int32_t Cout, int32_t Cin, int32_t taps, void *stream);
/* the same over partial rows of `ncols` floats (taps*Cin, or taps*Cin + 1 with the ones row: column taps*Cin -> db[co], may be NULL);
 * accumulate != 0 adds to dw / db instead of overwriting them */
int hrl_conv_wgrad_reduce2(const float *partials, int32_t splits, int32_t ncols, float *dw, float *db, int32_t Cout, int32_t Cin, int32_t taps,
                           int32_t accumulate, void *stream);

int hrl_gemm_fused(const HrlGemmArgs *args, void *stream);

/*
 * Glue of a fused conv -> BatchNorm -> ReLU tower over a tiny board (handyrl_b200/tower.py: the architecture of the
 * reference's SimpleConv2dModel, envs/tictactoe.py:52-69, with every layer ONE hrl_gemm_fused launch per direction).
 *   hrl_bn_finalize_fwd   col_partials [tiles][2][C*HW] (column sum / sum of squares from the STATS epilogue) -> batch
 *                         statistics.  mean_col is read first: on entry it holds the pivot that product subtracted (its
 *                         ep_mean, equal over each channel's columns; zeros for unshifted sums); then it receives the
 *                         batch mean.  Statistics of nn.BatchNorm2d in training mode (running stats with `momentum`, unbiased running
 *                         variance, num_batches_tracked += 1) and per-COLUMN mean / rstd / scale = gamma*rstd /
 *                         shift = beta - mean*scale (each C*HW floats) for the next product's operand transform
 *   hrl_bn_finalize_bwd   col_partials (column sums of dZ and dZ*xhat from the MASK_STATS epilogue) -> dgamma, dbeta and
 *                         the per-column constants of dY = dZ*p + Y*q + r.  gamma == NULL: only dbeta (a plain bias).
 *   hrl_heads_fwd / _bwd  squeeze outputs pre (M, ld), columns [pmaps*cells | vmaps*cells | rmaps*cells] -> LeakyReLU(slope)
 *                         -> policy = . Wp^T (A x pmaps*cells), value = tanh(. Wv^T), return = . Wr^T; the backward
 *                         writes dpre and the gradients of Wp / Wv / Wr and of the squeeze biases (fixed-order sums;
 *                         workspace: hrl_heads_num_blocks(M) * (A*pin + vin + rin + maps) floats).
 *   accumulate (hrl_bn_finalize_bwd, hrl_heads_bwd): 0 writes the parameter gradients (dgamma, dbeta; dWp, dWv, dWr
 *                         and the squeeze-bias gradients); != 0 ADDS them to what those buffers hold (each fp32 result
 *                         rounded first), for the micro-batches after the first of a gradient-accumulation step.  dpre and
 *                         p_col / q_col / r_col are written either way.
 */
int hrl_bn_finalize_fwd(const float *col_partials, int32_t tiles, int32_t C, int32_t HW, int64_t rows, const float *gamma,
                        const float *beta, float eps, float momentum, float *running_mean, float *running_var,
                        int64_t *batches_tracked, float *mean_col, float *rstd_col, float *scale_col, float *shift_col, void *stream);
int hrl_bn_finalize_bwd(const float *col_partials, int32_t tiles, int32_t C, int32_t HW, int64_t rows, const float *gamma,
                        const float *mean_col, const float *rstd_col, float *dgamma, float *dbeta, float *p_col, float *q_col,
                        float *r_col, int32_t accumulate, void *stream);
int32_t hrl_heads_num_blocks(int64_t M);
int hrl_heads_fwd(const float *pre, int64_t ld, int64_t M, int32_t cells, int32_t pmaps, int32_t vmaps, int32_t rmaps, int32_t A,
                  float slope, const float *Wp, const float *Wv, const float *Wr, float *policy, float *value, float *ret, void *stream);
int hrl_heads_bwd(const float *pre, int64_t ld, int64_t M, int32_t cells, int32_t pmaps, int32_t vmaps, int32_t rmaps, int32_t A,
                  float slope, const float *Wp, const float *Wv, const float *Wr, const float *value, const float *dpolicy,
                  const float *dvalue, const float *dret, float *dpre, float *dWp, float *dWv, float *dWr, float *dbias_p,
                  float *dbias_v, float *dbias_r, float *workspace, int32_t accumulate, void *stream);

/*
 * Weight of a stride-1 "same" convolution (Cout,Cin,kh,kw; odd kernel, zero padding) <-> the dense matrix
 * (Cout*H*W, Cin*H*W) that applies it to an H x W board stored NCHW (fastnet.BoardConv2d), and the adjoint map
 * dense-gradient -> weight-gradient.  dense[(o,q),(i,p)] = w[o,i,a,b] where tap (a,b) makes output cell q read input
 * cell p, 0 if no tap does.  hrl_board_fold sums `splits` dense gradients `split_stride` floats apart (the K-slice
 * partials a split hrl_gemm_tf32x3 leaves in its workspace when called with C == NULL; 1 for a single matrix).
 */
int hrl_board_expand(const float *w, float *dense, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw, int32_t H, int32_t W,
                     void *stream);
/*
 * hrl_board_pack: the same dense matrix, written directly as the B-operand images of hrl_gemm_fused (HrlGemmOperand.packed)
 * for the forward product (rows = output features (o,q), reduction = input features (i,p)) and for the input-gradient
 * product (rows = input features, reduction = output features).  Image layout: [chunk of 32 reduction elements][hi | lo]
 * [n_pad rows][128 bytes, 16-byte slots XOR-swizzled by the row], n_pad = hrl_gemm_padded_rows(rows of the operand);
 * row0 / k0 place several convolutions side by side in one operand (e.g. the policy / value squeeze convolutions).
 * Padding rows and the reduction tail must be zero: zero the images once, they are never written.
 */
/* Profiling / test hook of hrl_gemm_fused, process-global and NOT thread safe (default 0 = the product path):
 * 1 = skip the MMAs, 2 = skip the operand loads (timing attribution, scripts/gemm_breakdown.py).
 * Results with 1 or 2 set are garbage by design. */
void hrl_gemm_set_debug(int mode);
int32_t hrl_gemm_padded_rows(int64_t N);
size_t hrl_board_pack_floats(int64_t rows, int64_t K);      /* floats of an image with `rows` operand rows over K */
int hrl_board_pack(const float *w, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw, int32_t H, int32_t W, float *image_fwd,
                   int32_t fwd_rows, int32_t fwd_row0, float *image_bwd, int32_t bwd_rows, int32_t bwd_k0, void *stream);
/* Batched forms: up to HRL_MAX_BOARD_JOBS convolutions in ONE launch (a net packs all its layers' weights once per step, and
 * folds all its weight gradients once per backward pass).  bias / bias_cells (optional, both or neither): the convolution's
 * bias replicated per cell, bias_cells[c*H*W + q] = bias[c] -- the per-column bias of the dense product. */
#define HRL_MAX_BOARD_JOBS 8
typedef struct HrlPackJob {
    const float *w;
    int32_t Cout, Cin, kh, kw, H, W;
    float *image_fwd;
    int32_t fwd_rows, fwd_row0;
    float *image_bwd;
    int32_t bwd_rows, bwd_k0;
    const float *bias;
    float *bias_cells;
    /* != 0: write the images of HrlGemmArgs.bf16 products instead -- bf16 weights (round to nearest even), [chunk][n_pad rows]
     * [64 bytes, SWIZZLE_64B: 16-byte slot j of row r at j ^ ((r >> 1) & 3)], hrl_board_pack_floats(...) / 4 floats */
    int32_t bf16;
} HrlPackJob;
typedef struct HrlFoldJob {
    const float *ddense;
    int32_t splits;
    int64_t split_stride;
    float *dw;
    int32_t Cout, Cin, kh, kw, H, W;
    /* != 0: add the folded gradient to dw (its fp32 sum over the slices and taps rounded first) instead of storing it --
     * micro-batches after the first of a gradient-accumulation step.  0 (what hrl_board_fold passes) stores. */
    int32_t accumulate;
} HrlFoldJob;
int hrl_board_pack_many(const HrlPackJob *jobs, int32_t n_jobs, void *stream);
/* The same launch (0..HRL_MAX_BOARD_JOBS jobs) plus the pivots of the STATS epilogue's shifted BatchNorm sums for 0..HRL_MAX_BOARD_JOBS
 * layers of C channels over HW cells (fused tower: the pivot is layer l's ep_mean and the mean_col hrl_bn_finalize_fwd reads):
 * pivot_col[l][c*HW + h] = running_mean[l][c] where running_mean^2 > 1024 * running_var (|mean| / std > 32: unshifted fp32
 * sums would start to lose the variance), else 0 (the sums stay those of the unshifted statistics, bit for bit).
 * running_mean / running_var / pivot_col: host arrays of `layers` device pointers. */
int hrl_board_pack_many_pivot(const HrlPackJob *jobs, int32_t n_jobs, const float *const *running_mean, const float *const *running_var,
                              float *const *pivot_col, int32_t layers, int32_t C, int32_t HW, void *stream);
int hrl_board_fold_many(const HrlFoldJob *jobs, int32_t n_jobs, void *stream);
int hrl_board_fold(const float *ddense, int32_t splits, int64_t split_stride, float *dw, int32_t Cout, int32_t Cin, int32_t kh,
                   int32_t kw, int32_t H, int32_t W, void *stream);

/*
 * Recurrent nets (SURVEY.md 8 f-3).  ConvLSTM gate arithmetic (reference geister.py:49-56): gates (N,4C,S) in the order
 * i, f, o, g are the cell's convolution output; c' = sig(f) c + sig(i) tanh(g), h' = sig(o) tanh(c').  The backward
 * recomputes the activations from `gates` and `c_prev`; dh / dc_out may be NULL (no gradient from that side).
 */
int hrl_lstm_gates_fwd(const float *gates, const float *c_prev, float *h_out, float *c_out, int64_t N, int32_t C, int32_t S,
                       void *stream);
int hrl_lstm_gates_bwd(const float *gates, const float *c_prev, const float *dh, const float *dc_out, float *dgates,
                       float *dc_prev, int64_t N, int32_t C, int32_t S, void *stream);

/*
 * Hidden-state masking of the recurrent time loop (reference train.py:152-158, 173) on a hidden leaf h (B,P,R):
 *   visible: out = h * om[b,p]            (sum_players = 0, out (B,P,R))
 *            out = sum_p h * om[b,p]      (sum_players = 1, out (B,R): turn-alternating batches)
 *   blend:   out = h (1 - om) + h_new om  (h_new (B,Pn,R), Pn == P or 1)
 * om points at observation_mask[:, t] = element (b,p) at om[b * om_stride + p].
 */
int hrl_hidden_visible_fwd(const float *h, const float *om, int64_t om_stride, float *out, int64_t B, int32_t P, int32_t R,
                           int32_t sum_players, void *stream);
int hrl_hidden_visible_bwd(const float *dout, const float *om, int64_t om_stride, float *dh, int64_t B, int32_t P, int32_t R,
                           int32_t sum_players, void *stream);
int hrl_hidden_blend_fwd(const float *h, const float *nh, const float *om, int64_t om_stride, float *out, int64_t B, int32_t P,
                         int32_t Pn, int32_t R, void *stream);
int hrl_hidden_blend_bwd(const float *dout, const float *om, int64_t om_stride, float *dh, float *dnh, int64_t B, int32_t P,
                         int32_t Pn, int32_t R, void *stream);

/*
 * Train-mode BatchNorm over (N, C, HW) fp32 activations with small HW -- used by the small-board rewrite of the user's
 * net (the nets of reference envs normalise (N,32,3,3) / (N,C,6,6) tensors; cuDNN / ATen launch one CTA per channel
 * there).  Semantics of nn.BatchNorm2d in training mode: biased variance for the normalisation, unbiased for
 * running_var, running stats updated with `momentum` (pass NULL for both to skip).  mean / rstd (C floats each) are
 * saved for the backward.  channels_last = 1: x / y / dy / dx are (N, H, W, C) in memory (torch.channels_last), e.g. the
 * activations between cuDNN's NHWC convolutions.  workspace: hrl_bn_workspace_floats(N, C, HW, channels_last) floats.
 */
size_t hrl_bn_workspace_floats(int64_t N, int32_t C, int32_t HW, int32_t channels_last);
int hrl_bn_train_fwd(const float *x, const float *gamma, const float *beta, float *y, float *mean, float *rstd,
                     float *running_mean, float *running_var, int64_t N, int32_t C, int32_t HW, int32_t channels_last, float eps, float momentum,
                     float *workspace, void *stream);
int hrl_bn_train_bwd(const float *x, const float *dy, const float *gamma, const float *mean, const float *rstd, float *dx,
                     float *dgamma, float *dbeta, int64_t N, int32_t C, int32_t HW, int32_t channels_last, float *workspace,
                     void *stream);

/*
 * Replay gather/pad: the device form of make_batch (train.py:33-124).
 *
 * Episodes are kept decoded in flat device arrays ("replay store"), one row per step:
 *   per step s and player p (value side, Ps players):  obs_mask, turn_mask(=selected_prob present),
 *   selected_prob, action, value, reward, return; per step: action_mask rows, observation rows.
 * A window descriptor selects [start, end) of one episode and where it lands in [0, T).
 */
typedef struct HrlWindow {
    int64_t first_step;   /* row of the episode's step 0 in the store                          */
    int32_t start, end;   /* window [start, end) in episode steps (train.py:305-306)           */
    int32_t train_start;  /* first trained step (train.py:304); pad_before = burn_in-(train_start-start) */
    int32_t total;        /* episode length, for progress = step / total (train.py:89)        */
    int32_t outcome_row;  /* row in the store's outcome table                                  */
    int32_t player;       /* solo training (train.py:57-58): the one store player batched; else 0 */
} HrlWindow;

typedef struct HrlGatherArgs {
    int32_t B, T, P, Pa, A;
    int32_t Ps;                   /* players per step in the store (P == Ps, or P == 1 for solo) */
    int32_t burn_in;
    int32_t obs_elems;            /* floats per observation (flattened leaf)                   */
    int32_t turn_alternating;     /* Pa == 1 layout: pick the turn player's row (train.py:65-66) */
    const HrlWindow *windows;     /* [B] device                                                */

    /* replay store, S = total stored steps */
    const float *st_obs;          /* (S,Ps,obs_elems) zero where the player did not observe     */
    const float *st_prob;         /* (S,Ps) 1.0 where absent                                   */
    const int32_t *st_action;     /* (S,Ps) 0 where absent                                     */
    const float *st_amask;        /* (S,Ps,A) 1e32 where absent                                 */
    const float *st_value;        /* (S,Ps)                                                    */
    const float *st_reward;       /* (S,Ps)                                                    */
    const float *st_return;       /* (S,Ps)                                                    */
    const uint8_t *st_flags;      /* (S,Ps) bit0 = acted (turn_mask), bit1 = observed           */
    const int32_t *st_turn;       /* (S)   index of the step's first turn player (train.py:66)         */
    const float *st_outcome;      /* (E,Ps)                                                    */

    /* batch outputs, layouts of train.py:114-124 */
    float *observation;           /* (B,T,Pa,obs_elems)                                        */
    float *selected_prob;         /* (B,T,Pa)                                                  */
    float *value;                 /* (B,T,P)                                                   */
    int64_t *action;              /* (B,T,Pa)                                                  */
    float *outcome;               /* (B,P)                                                     */
    float *reward;                /* (B,T,P)                                                   */
    float *ret;                   /* (B,T,P)                                                   */
    float *episode_mask;          /* (B,T)                                                     */
    float *turn_mask;             /* (B,T,P)                                                   */
    float *observation_mask;      /* (B,T,P)                                                   */
    float *action_mask;           /* (B,T,Pa,A)                                                */
    float *progress;              /* (B,T)                                                     */
} HrlGatherArgs;

int hrl_gather_pad(const HrlGatherArgs *args, void *stream);

/*
 * Replay gather/pad with board-symmetry augmentation: hrl_gather_pad, with window b written through transform sym[b]
 * of K permutation tables.  For a live cell of window b, with k = sym[b]:
 *   observation[e]  = stored observation[obs_src[k][e]]     e < obs_elems (the concatenated flat leaves)
 *   action_mask[a]  = stored action_mask[act_src[k][a]]     a < A
 *   action          = act_dst[k][stored action]             (an action outside [0, A) is copied unchanged)
 * act_src[k] is the inverse permutation of act_dst[k].  Pad cells and every other batch tensor are bit-identical to
 * hrl_gather_pad's; every batch byte is still written exactly once, and copies are exact.
 *
 * The kernel trusts the tables and sym: every row must be a permutation of [0, obs_elems) / [0, A), and
 * 0 <= sym[b] < K (the caller checks the values on the host before uploading them).  1 <= K <= HRL_SYM_MAX_TRANSFORMS.
 */
#define HRL_SYM_MAX_TRANSFORMS 64
int hrl_gather_pad_sym(const HrlGatherArgs *args,
                       const int32_t *sym,      /* [B] device: transform of each window, 0 <= sym[b] < K */
                       const int32_t *obs_src,  /* [K][obs_elems] device (may be NULL when obs_elems == 0) */
                       const int32_t *act_src,  /* [K][A] device: new action-mask slot <- stored slot */
                       const int32_t *act_dst,  /* [K][A] device: stored action -> new action */
                       int32_t K, void *stream);

/*
 * Prioritised replay (opt-in, no reference counterpart).  Every slot of the replay's episode directory (a ring of `ring`
 * slots; the live episodes are slots (head + i) % ring, i = 0 the oldest of `count`) holds a priority prio[s] and the serial
 * of the episode that priority belongs to, prio_serial[s].
 *
 * hrl_replay_sample draws B windows on the device, in one launch:
 *   - a live slot whose directory serial differs from prio_serial is a new episode: prio = *max_prio, prio_serial = its serial;
 *   - episode i is drawn with probability (i+1) * prio^alpha / sum (fp64 prefix sum in a fixed order, binary search);
 *   - inside it the window is placed as the host sampler places it: train_start uniform on [0, 1 + max(0, steps - forward)),
 *     start = max(0, train_start - burn_in), end = min(train_start + forward, steps), a uniform player when solo != 0;
 *   - windows[b], win_slot[b], win_serial[b] and win_weight[b] = B * p_b^(-alpha*beta) / sum_b' p_b'^(-alpha*beta).
 * The random numbers are Philox4x32-10 (curand) with key `seed`, one 128-bit block per window at counter
 * (b, counter_lo, counter_hi, 0): the same seed, counter and priorities give the same windows.
 */
typedef struct HrlReplaySampleArgs {
    int32_t B;                    /* windows to draw                                                            */
    int32_t ring;                 /* directory slots                                                            */
    int32_t head, count;          /* oldest live slot and live episodes (count >= 1, count < ring)              */
    int32_t burn_in, forward_steps;
    int32_t Ps;                   /* players per step in the store                                              */
    int32_t solo;                 /* 1: draw HrlWindow.player uniformly in [0, Ps); 0: player = 0               */
    float alpha, beta;            /* alpha >= 0, 0 <= beta <= 1                                                  */
    uint64_t seed;                /* Philox key                                                                 */
    uint64_t counter;             /* Philox counter of this batch (one per batch)                               */
    const int64_t *dir;           /* [ring][4] device mirror of the directory: first_step, steps, outcome_row, serial */
    float *prio;                  /* [ring]                                                                     */
    int64_t *prio_serial;         /* [ring]                                                                     */
    const float *max_prio;        /* [1]                                                                        */
    double *workspace;            /* [ring] prefix sums                                                         */
    HrlWindow *windows;           /* [B] out: the gather's descriptors                                          */
    int32_t *win_slot;            /* [B] out: directory slot of each window                                     */
    int64_t *win_serial;          /* [B] out: episode serial of each window                                     */
    float *win_weight;            /* [B] out: importance weights, mean 1                                        */
} HrlReplaySampleArgs;

int hrl_replay_sample(const HrlReplaySampleArgs *args, void *stream);

/*
 * The priority update that ends a prioritised step, in one launch.  Window b's priority over its trained cells
 * (t >= burn_in), tm = turn_mask (B,T,P), adv = the loss pass's tap_advantage (B,T,P):
 *     q_b = sum(tm * |adv|) / sum(tm) + epsilon      (fp32, fixed order; no priority when sum(tm) == 0)
 * prio[win_slot[b]] becomes the largest q_b of the windows on that slot -- only where prio_serial[slot] == win_serial[b]
 * (win_serial < 0: the window is ignored) -- and *max_prio rises to the largest q_b written.  skip (the guarded optimiser's
 * flag, or NULL): when *skip != 0 nothing is written.
 */
int hrl_replay_priority_update(int32_t B, int32_t T, int32_t P, int32_t burn_in, const float *tap_advantage,
                               const float *turn_mask, float epsilon, const int32_t *win_slot, const int64_t *win_serial,
                               float *prio, const int64_t *prio_serial, float *max_prio, const int32_t *skip, void *stream);

/*
 * Policy distillation from a teacher net ("kickstarting"): an annealed KL(teacher || student) term on the policy rows the fused
 * loss trains, launched right after hrl_loss_fwd_bwd on the same batch.  Row (b, t, q) of the (B,T,Pa,A) logits, trained when
 * t >= burn_in (or T == 1), f = sum_p turn_mask[b,t,p] when Pa == 1, else turn_mask[b,t,q] (the mask epilogue's own factor):
 *     zS = f * student - action_mask         zT = f * teacher - action_mask
 *     kl = sum_rows w_b * f * sum_a pT * (log pT - log pS)      pT = softmax(zT), pS = softmax(zS); terms with pT == 0 add 0
 *     c  = coef * max(0, 1 - n / anneal_steps)                   (coef when anneal_steps == 0; n = *step_count at launch)
 * w_b = window_weight[b] (1 when NULL).  sums = [kl, c * kl] (overwritten); when c > 0, losses[HRL_LOSS_TOTAL] += c * kl and
 * dpolicy_raw += c * w_b * f * f * (pS - pT) on trained rows with w_b * f != 0; when c == 0 neither is written.  Rows of weight 0
 * are never read.  Block partials are folded in fp64 in a fixed order by the last CTA, which resets the workspace counter:
 * repeated launches and graph replays give identical bits.  Pa must be 1 or P, A <= 1024, P <= 64; io_bf16 logits are
 * refused (HRL_ERR_UNSUPPORTED).
 */
typedef struct HrlDistillArgs {
    int32_t B, T, P, Pa, A;
    int32_t burn_in;
    const float *policy_raw;      /* (B,T,Pa,A) the student's raw logits (what hrl_loss_fwd_bwd read)          */
    const float *teacher_raw;     /* (B,T,Pa,A) the teacher's raw logits on the same batch                      */
    const float *action_mask;     /* (B,T,Pa,A) 0 legal / 1e32 illegal                                          */
    const float *turn_mask;       /* (B,T,P)                                                                    */
    const float *window_weight;   /* (B) importance weights (prioritised replay), or NULL = 1                   */
    const int64_t *step_count;    /* [1] the optimiser's step count before this step                           */
    float coef;                   /* c0 >= 0                                                                    */
    int64_t anneal_steps;         /* N >= 0; 0 = constant coefficient                                           */
    float *dpolicy_raw;           /* (B,T,Pa,A) added to                                                        */
    float *losses;                /* [HRL_NUM_LOSS] of the loss pass: only the total is added to               */
    float *sums;                  /* [2] out: kl, c * kl                                                        */
    void *workspace;              /* >= hrl_distill_workspace_bytes(...), first 64 bytes zero on the first call  */
    size_t workspace_bytes;
    int32_t io_bf16;              /* must be 0                                                                  */
} HrlDistillArgs;

size_t hrl_distill_workspace_bytes(int32_t B, int32_t T, int32_t P, int32_t Pa, int32_t A);
int hrl_distill_fwd_bwd(const HrlDistillArgs *args, void *stream);

/*
 * Categorical value heads (opt-in): a value or return head that outputs K logits per row, a distribution over K bins, trained
 * by cross-entropy against a two-hot or HL-Gauss target distribution.  Row (b, t, q) of the (B,T,Pa,K) logits z:
 *   bins         D = (high - low) / (K - 1), centres c_k = low + k D, edges e_k = low + (k - 1/2) D   (k = 0 .. K)
 *   transform    s(y) = sign(y) log(1 + |y|) when symlog, else y;   s^-1(m) = sign(m) (exp|m| - 1)
 *   expectation  p = softmax(z),  v = s^-1(sum_k p_k c_k)                     (what the fused loss reads as the head's output)
 *   target       x = clamp(s(y), low, high) for a target y (the loss pass's tap_target_value / _return)
 *                sigma == 0 (two-hot): j = min(floor((x - low) / D), K - 2), u = (x - c_j) / D, pi_j = 1 - u, pi_j+1 = u
 *                sigma > 0 (HL-Gauss): pi_k = [Phi((e_k+1 - x) / sigma) - Phi((e_k - x) / sigma)] /
 *                                             [Phi((e_K - x) / sigma) - Phi((e_0 - x) / sigma)]
 *   loss         over trained columns (b, t, p) -- t >= burn_in, or T == 1 -- with q = p when Pa == P, else 0:
 *                L = sum w_b om_btp (-sum_k pi_k(y_btp) log p_k(z_btq)),  dz_btq = sum_p w_b om_btp (p - pi(y_btp))
 *                om = observation_mask, w_b = window_weight[b] (1 when NULL); rows not trained get dz = 0.
 *
 * hrl_value_bins_expect   logits -> expect (B,T,Pa), every row.
 * hrl_value_bins_fwd_bwd  one head per launch: dlogits (overwritten; rows of weight 0 are zero and never read),
 *                         losses[HRL_LOSS_V] (head 0) or losses[HRL_LOSS_R] (head 1) = L, losses[HRL_LOSS_TOTAL] += L.
 *                         dlogits == NULL: the forward-only form (held-out losses), which ignores window_weight.
 *                         Block partials are folded in fp64 in a fixed order by the last CTA, which resets the workspace
 *                         counter: repeated launches and graph replays give identical bits.
 * Both: 2 <= K <= 1024, P <= 64, Pa = 1 or P (else HRL_ERR_UNSUPPORTED); low < high finite, sigma finite >= 0 (HRL_ERR_BAD_ARG).
 */
typedef struct HrlValueBinsArgs {
    int32_t B, T, P, Pa, K;
    int32_t burn_in;
    float low, high;              /* the centres span [low, high] (in symlog space when symlog)                */
    int32_t symlog;
    float sigma;                  /* 0 two-hot, > 0 HL-Gauss width in bin-space units                           */
    int32_t head;                 /* 0 value (losses[HRL_LOSS_V]), 1 return (losses[HRL_LOSS_R])               */
    const float *logits;          /* (B,T,Pa,K)                                                                 */
    float *expect;                /* (B,T,Pa) out of hrl_value_bins_expect                                      */
    const float *target;          /* (B,T,P) the loss pass's target tap of this head                            */
    const float *observation_mask;/* (B,T,P)                                                                    */
    const float *window_weight;   /* (B) importance weights, or NULL = 1                                        */
    float *dlogits;               /* (B,T,Pa,K) out, or NULL (forward only)                                     */
    float *losses;                /* [HRL_NUM_LOSS] of the loss pass                                            */
    void *workspace;              /* >= hrl_value_bins_workspace_bytes(...), first 64 bytes zero on the first call */
    size_t workspace_bytes;
} HrlValueBinsArgs;

size_t hrl_value_bins_workspace_bytes(int32_t B, int32_t T, int32_t P, int32_t Pa, int32_t K);
int hrl_value_bins_expect(const HrlValueBinsArgs *args, void *stream);
int hrl_value_bins_fwd_bwd(const HrlValueBinsArgs *args, void *stream);

/* Text of the last error raised on the calling thread ("" if none). */
const char *hrl_last_error(void);

/* HRL_ABI_VERSION the library was built with. */
int32_t hrl_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* HRL_B200_H_ */
