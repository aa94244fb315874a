// K1 -- fused forward+backward of the HandyRL loss over one replay batch (sm_90a).
//
// Replaces, in ONE launch and one pass over HBM:
//   handyrl/train.py:176-184  mask epilogue of forward_prediction
//   handyrl/train.py:218-267  compute_loss (log-softmax/gather, importance ratio clamp,
//                             2-player value symmetrisation, targets/advantages)
//   handyrl/losses.py:16-80   MC / TD(lambda) / UPGO / V-Trace reverse-time scans
//   handyrl/train.py:189-215  compose_losses (masked sums, entropy)
//   + the autograd pass of train.py:369 through those ops (closed-form gradients
//     w.r.t. the raw policy / value / return outputs of the net).
//
// CTA = EPB consecutive episodes (windows); all of their T x P x A data stays on chip between the
// statistics pass and the gradient pass, so every input byte is read from HBM once and every gradient
// byte written once.  Three data-movement variants share the same maths (loss_common.cuh):
//
//   rows kernel, staged I/O   small/medium rows: the episodes' logits and action masks are copied to
//                             shared memory with cp.async (all in flight at once, one DRAM round trip),
//                             rows are processed from shared memory, gradients are written back in place
//                             and leave with one coalesced copy-out.
//   rows kernel, direct       fallback for shapes that do not fit: coalesced (vector) global loads per row.
//   element kernel            small action spaces (A <= 32): one thread per logit, coalesced direct loads/stores,
//                             short row-wise passes in shared memory (latency-optimal for KB-sized windows).
//   bulk kernel               wide rows (A % 4 == 0): a 2-CTA cluster splits the window's time axis; TMA 1-D
//                             bulk copies (cp.async.bulk + mbarrier) bring each CTA's share of the logits into
//                             shared memory at once, warps reduce rows with register-prefetched action masks,
//                             exchange row statistics through DSMEM; gradients leave as bulk stores.
//
// Phases: (0) stage  (1) per-row softmax statistics  (2a-2c) targets / recurrences / per-cell terms
//         (publish six block partials; the last CTA folds them in a fixed order in fp64)
//         (3) gradients.
#include <cuda_bf16.h>

#include "loss_common.cuh"
#include <stdlib.h>

namespace hrl {

#define HRL_STAMP(i)                                                                             \
    do {                                                                                         \
        if (prm.trace && blockIdx.x == gridDim.x / 2 && threadIdx.x == 0) prm.trace[i] = clock64(); \
    } while (0)

// element index of the k-th value a lane holds: the scalar layout interleaves lanes; the vector layout
// (LPR == 32, A % 4 == 0) gives every lane float4 chunks so that a warp touches 512 contiguous bytes.
template <int LPR, bool VEC>
__device__ __forceinline__ int elem_index(int k, int lane) {
    return VEC ? ((k >> 2) * LPR + lane) * 4 + (k & 3) : k * LPR + lane;
}

__device__ __forceinline__ CtaCtx make_ctx(const LossParams &prm) {
    CtaCtx c;
    const HrlLossArgs &a = prm.a;
    c.T0 = a.T; c.P = a.P; c.Pa = a.Pa; c.A = a.A; c.bi = a.burn_in; c.Tt = prm.Tt;
    c.b0 = (prm.cluster > 1 ? blockIdx.x / prm.cluster : blockIdx.x) * prm.EPB;
    c.nE = min(prm.EPB, a.B - c.b0);
    c.tid = threadIdx.x; c.nthr = blockDim.x;
    c.nrows = c.nE * c.Tt * c.Pa; c.ncols = c.nE * c.Tt * c.P; c.ncells = c.nE * c.Tt;
    c.shP = log2_exact(c.P); c.shPa = log2_exact(c.Pa); c.shTt = log2_exact(c.Tt);
    c.t_lo = 0; c.t_hi = c.Tt;
    return c;
}

// phase 0: every small per-cell tensor of the CTA's episodes -> shared memory, asynchronously
__device__ __forceinline__ void stage_small(const LossParams &prm, const SmemLayout &L, float *smem, const CtaCtx &c) {
    const HrlLossArgs &a = prm.a;
    const int R = c.Tt * c.Pa;
    for (int i = c.tid; i < c.ncols; i += c.nthr) {
        const int e = i / (c.Tt * c.P), r = i - e * (c.Tt * c.P);
        const size_t g = ((size_t)(c.b0 + e) * c.T0 + c.bi) * c.P + r;
        cp_async4(smem + L.tm + i, a.turn_mask + g);
        cp_async4(smem + L.om + i, a.observation_mask + g);
        cp_async4(smem + L.rew + i, a.reward + g);
        cp_async4(smem + L.ret + i, a.ret + g);
    }
    for (int i = c.tid; i < c.ncells; i += c.nthr) {
        const int e = i / c.Tt, r = i - e * c.Tt;
        const size_t g = (size_t)(c.b0 + e) * c.T0 + c.bi + r;
        cp_async4(smem + L.emask + i, a.episode_mask + g);
        cp_async4(smem + L.prog + i, a.progress + g);
    }
    long long *s_act = reinterpret_cast<long long *>(smem + L.act);
    for (int i = c.tid; i < c.nrows; i += c.nthr) {
        const int e = i / R, r = i - e * R;
        const size_t g = ((size_t)(c.b0 + e) * c.T0 + c.bi) * c.Pa + r;
        if (prm.has_v) cp_async4(smem + L.vraw + i, a.value_raw + g); else smem[L.vraw + i] = 0.0f;
        if (prm.has_r) cp_async4(smem + L.rraw + i, a.return_raw + g); else smem[L.rraw + i] = 0.0f;
        cp_async4(smem + L.prob + i, a.selected_prob + g);
        cp_async8(s_act + i, a.action + g);
    }
    for (int i = c.tid; i < c.nE * c.P; i += c.nthr) cp_async4(smem + L.outcome + i, a.outcome + (size_t)c.b0 * c.P + i);
}

// burn-in steps take no part in the loss: zero gradients (train.py:220-222).  With io_bf16 the policy gradient holds bf16
// elements: zeroed as 16-bit words (zero in bf16 too), or the stores would land at twice the offset.
__device__ __forceinline__ void zero_burn_in(const LossParams &prm, const CtaCtx &c) {
    const HrlLossArgs &a = prm.a;
    if (c.bi <= 0) return;
    const int nz = c.bi * c.Pa * c.A, nzr = c.bi * c.Pa;
    for (int e = 0; e < c.nE; e++) {
        const size_t g0 = (size_t)(c.b0 + e) * c.T0 * c.Pa;
        if (a.io_bf16) {
            uint16_t *d16 = reinterpret_cast<uint16_t *>(a.dpolicy_raw) + g0 * c.A;
            for (int i = c.tid; i < nz; i += c.nthr) d16[i] = 0;
        } else {
            for (int i = c.tid; i < nz; i += c.nthr) a.dpolicy_raw[g0 * c.A + i] = 0.0f;
        }
        for (int i = c.tid; i < nzr; i += c.nthr) {
            if (prm.loss_v) a.dvalue_raw[g0 + i] = 0.0f;
            if (prm.loss_r) a.dreturn_raw[g0 + i] = 0.0f;
        }
    }
}

// raw per-row statistics of the softmax pass; the scalar tail (log, exp, ratio) runs later, one thread per row
__device__ __forceinline__ void store_row_stats(const SmemLayout &L, float *smem, int r, float za, float m, float se,
                                                float sw, float scale) {
    smem[L.za + r] = za;
    smem[L.mx + r] = m;
    smem[L.se + r] = se;
    smem[L.sw + r] = sw;
    smem[L.scale + r] = scale;
}

// phase 1b: log-sum-exp, entropy, log pi(a), clipped importance ratio -- in parallel over rows
__device__ __forceinline__ void row_epilogue(const LossParams &prm, const SmemLayout &L, float *smem, const CtaCtx &c) {
    const HrlLossArgs &a = prm.a;
    const int R = c.Tt * c.Pa;
    for (int r = c.tid; r < c.nrows; r += c.nthr) {
        const int e = (c.nE == 1) ? 0 : r / R, rr = r - e * R, t = fdiv(rr, c.Pa, c.shPa);
        const float se = smem[L.se + r], m = smem[L.mx + r];
        const float lsum = logf(se);
        const float h = lsum - smem[L.sw + r] / se;                         // entropy = ln S - W / S
        const float em = smem[L.emask + e * c.Tt + t], mu = smem[L.prob + r];
        const float lt = (smem[L.za + r] - m - lsum) * em;                  // train.py:232
        const float lb = logf(fminf(fmaxf(mu, 1e-16f), 1.0f)) * em;         // train.py:231
        const float rho = fminf(fmaxf(expf(lt - lb), 0.0f), 1.0f);          // train.py:235-238
        smem[L.logp + r] = lt;
        smem[L.rho + r] = rho;
        smem[L.ent + r] = h;
        smem[L.lsum + r] = lsum;
        if ((a.tap_logp || a.tap_rho || a.tap_entropy) && t >= c.t_lo && t < c.t_hi) {
            const size_t grow = ((size_t)(c.b0 + e) * c.T0 + c.bi) * c.Pa + rr;
            if (a.tap_logp) a.tap_logp[grow] = lt;
            if (a.tap_rho) a.tap_rho[grow] = rho;
            if (a.tap_entropy) a.tap_entropy[grow] = h;
        }
    }
}

// ======================================================================== rows kernel
// IOS: logits and action masks staged in shared memory by cp.async (rows read/written on chip only).
// DIAG (every kernel): the learner diagnostics sums are accumulated in phase 2c and folded with the losses.
// GRAD (every kernel): phase 3 is compiled in.  Without it (hrl_loss_fwd) the kernel writes the loss sums and the taps only:
// phases 0-2c, the partials and the fixed-order fold are the same code, so the sums are bit-identical.
template <int LPR, int NPL, bool VEC, bool IOS, bool DIAG, bool GRAD>
__global__ void __launch_bounds__(512) loss_rows_kernel(const LossParams prm) {
    extern __shared__ __align__(128) float smem[];
    __shared__ bool s_last;
    const HrlLossArgs &a = prm.a;
    const CtaCtx c = make_ctx(prm);
    const int P = c.P, Pa = c.Pa, A = c.A, Tt = c.Tt, T0 = c.T0, bi = c.bi, tid = c.tid, nthr = c.nthr;
    const int R = Tt * Pa, RS = prm.row_stride;
    const SmemLayout L = make_layout(prm.EPB, Tt, P, Pa, prm.stage_z, RS, IOS ? prm.EPB * R * RS : 0, -1, false, prm.scan + 1);
    const long long *s_act = reinterpret_cast<const long long *>(smem + L.act);
    HRL_STAMP(0);

    // ---------------- phase 0: stage
    stage_small(prm, L, smem, c);
    if (IOS) {
        const int per_ep = R * A;
        for (int i = tid; i < c.nE * per_ep; i += nthr) {
            const int e = i / per_ep, rem = i - e * per_ep;
            const int rr = rem / A, j = rem - rr * A;
            const size_t g = ((size_t)(c.b0 + e) * T0 + bi) * Pa * A + rem;
            const int s = (e * R + rr) * RS + j;
            cp_async4(smem + L.z + s, a.policy_raw + g);
            cp_async4(smem + L.am + s, a.action_mask + g);
        }
        cp_async_wait_all();
        __syncthreads();
    }
    HRL_STAMP(1);

    // ---------------- phase 1: per-row softmax statistics
    const int grp = tid / LPR, lane = tid % LPR, ngrp = nthr / LPR;
    for (int base = 0; base < c.nrows; base += ngrp) {
        const int r = base + grp;
        const bool valid = r < c.nrows;
        float z[NPL];
        float scale = 0.0f;
        int act = 0;
        size_t grow = 0;
        if (valid) {
            const int e = r / R, rr = r - e * R, t = rr / Pa, q = rr - t * Pa;
            const size_t cell = (size_t)(c.b0 + e) * T0 + bi + t;
            grow = cell * Pa + q;
            if (IOS) {
                const int scell = e * Tt + t;
                if (Pa == P) scale = smem[L.tm + scell * P + q];
                else for (int p = 0; p < P; p++) scale += smem[L.tm + scell * P + p];   // train.py:179-180
                act = (int)s_act[r];
            } else {
                if (Pa == P) scale = a.turn_mask[cell * P + q];
                else for (int p = 0; p < P; p++) scale += a.turn_mask[cell * P + p];
                act = (int)a.action[grow];
            }
        }
        const float *rawp = a.policy_raw + grow * A;
        const float *amp = a.action_mask + grow * A;
        float m = -INFINITY, za = -INFINITY;
        if (VEC) {
#pragma unroll
            for (int k4 = 0; k4 < NPL / 4; k4++) {
                const int j = (k4 * LPR + lane) * 4;
                float4 x = make_float4(0.f, 0.f, 0.f, 0.f), am = make_float4(INFINITY, INFINITY, INFINITY, INFINITY);
                if (valid && j < A) {
                    x = __ldcs(reinterpret_cast<const float4 *>(rawp + j));
                    am = __ldcs(reinterpret_cast<const float4 *>(amp + j));
                }
                z[k4 * 4 + 0] = x.x * scale - am.x;  // train.py:178-181
                z[k4 * 4 + 1] = x.y * scale - am.y;
                z[k4 * 4 + 2] = x.z * scale - am.z;
                z[k4 * 4 + 3] = x.w * scale - am.w;
            }
        } else {
#pragma unroll
            for (int k = 0; k < NPL; k++) {
                const int j = k * LPR + lane;
                z[k] = -INFINITY;
                if (valid && j < A) {
                    if (IOS) z[k] = smem[L.z + r * RS + j] * scale - smem[L.am + r * RS + j];
                    else z[k] = ld_stream(rawp + j) * scale - ld_stream(amp + j);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < NPL; k++) {
            if (elem_index<LPR, VEC>(k, lane) == act) za = z[k];
            m = fmaxf(m, z[k]);
        }
        m = group_max<LPR>(m);
        za = group_max<LPR>(za);
        // one exp per element: S = sum e, W = sum e * (z - m);  entropy = log S - W / S
        float se = 0.0f, sw = 0.0f;
#pragma unroll
        for (int k = 0; k < NPL; k++) {
            const int j = elem_index<LPR, VEC>(k, lane);
            if (valid && j < A) {
                const float d = z[k] - m;
                const float ex = expf(d);
                se += ex;
                sw += ex * fmaxf(d, -3.0e38f);     // e = 0 rows contribute 0, never 0 * inf
                if (prm.stage_z) smem[L.z + r * RS + j] = z[k];
            }
        }
        se = group_sum<LPR>(se);
        sw = group_sum<LPR>(sw);
        if (valid && lane == 0) store_row_stats(L, smem, r, za, m, se, sw, scale);
    }
    if (!IOS) cp_async_wait_all();
    HRL_STAMP(2);
    __syncthreads();
    baselines(prm, L, smem, c);
    row_epilogue(prm, L, smem, c);
    __syncthreads();
    HRL_STAMP(3);

    // ---------------- phase 2: targets, recurrences, per-cell terms; one warp publishes the scalars
    float part[6], dpart[DIAG ? HRL_NUM_LOSS_DIAG : 1];
    targets_and_losses<DIAG, GRAD>(prm, L, smem, c, part, dpart);
    HRL_STAMP(4);
    if (DIAG) reduce_diag(prm, L, smem, c, dpart);
    reduce_partials(L, smem, c, part);
    if ((tid >> 5) == (nthr >> 5) - 1) publish_partials(prm, L, smem, c, &s_last);
    HRL_STAMP(5);

    // ---------------- phase 3: gradients w.r.t. the raw net outputs
    for (int base = 0; GRAD && base < c.nrows; base += ngrp) {
        const int r = base + grp;
        if (r >= c.nrows) continue;  // no shuffles below: divergence is harmless
        const int e = r / R, rr = r - e * R, t = rr / Pa, q = rr - t * Pa;
        const int cell = e * Tt + t;
        const size_t grow = ((size_t)(c.b0 + e) * T0 + bi + t) * Pa + q;
        const RowFactors f = row_factors(prm, L, smem, c.b0 + e, cell, q, P, Pa);
        const float scale = smem[L.scale + r], m = smem[L.mx + r], lsum = smem[L.lsum + r], h = smem[L.ent + r];
        const int act = (int)s_act[r];
        float *outp = a.dpolicy_raw + grow * A;
        const float *rawp = a.policy_raw + grow * A;
        const float *amp = a.action_mask + grow * A;
        if (VEC) {
#pragma unroll
            for (int k4 = 0; k4 < NPL / 4; k4++) {
                const int j = (k4 * LPR + lane) * 4;
                if (j < A) {
                    float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (scale != 0.0f) {
                        float zz[4];
                        if (prm.stage_z) {
                            const float4 t4 = *reinterpret_cast<const float4 *>(smem + L.z + r * RS + j);
                            zz[0] = t4.x; zz[1] = t4.y; zz[2] = t4.z; zz[3] = t4.w;
                        } else {
                            const float4 x = *reinterpret_cast<const float4 *>(rawp + j);
                            const float4 am = *reinterpret_cast<const float4 *>(amp + j);
                            zz[0] = x.x * scale - am.x; zz[1] = x.y * scale - am.y;
                            zz[2] = x.z * scale - am.z; zz[3] = x.w * scale - am.w;
                        }
                        out.x = grad_elem(zz[0], j + 0 == act, m, lsum, h, f.w, f.k, scale);
                        out.y = grad_elem(zz[1], j + 1 == act, m, lsum, h, f.w, f.k, scale);
                        out.z = grad_elem(zz[2], j + 2 == act, m, lsum, h, f.w, f.k, scale);
                        out.w = grad_elem(zz[3], j + 3 == act, m, lsum, h, f.w, f.k, scale);
                    }
                    __stcs(reinterpret_cast<float4 *>(outp + j), out);
                }
            }
        } else {
#pragma unroll
            for (int kk = 0; kk < NPL; kk++) {
                const int j = kk * LPR + lane;
                if (j < A) {
                    float g = 0.0f;
                    if (scale != 0.0f) {
                        const float zj = prm.stage_z ? smem[L.z + r * RS + j] : (rawp[j] * scale - amp[j]);
                        g = grad_elem(zj, j == act, m, lsum, h, f.w, f.k, scale);
                    }
                    if (IOS) smem[L.z + r * RS + j] = g;      // leaves with the coalesced copy-out below
                    else st_stream(outp + j, g);
                }
            }
        }
        if (lane == 0) {
            if (prm.loss_v) a.dvalue_raw[grow] = f.gv;
            if (prm.loss_r) a.dreturn_raw[grow] = f.gr;
        }
    }
    if (IOS && GRAD) {
        __syncthreads();
        const int per_ep = R * A;
        for (int i = tid; i < c.nE * per_ep; i += nthr) {
            const int e = i / per_ep, rem = i - e * per_ep;
            const int rr = rem / A, j = rem - rr * A;
            st_stream(a.dpolicy_raw + ((size_t)(c.b0 + e) * T0 + bi) * Pa * A + rem, smem[L.z + (e * R + rr) * RS + j]);
        }
    }
    if (GRAD) zero_burn_in(prm, c);
    __syncthreads();
    if (s_last) {
        finalize_losses(prm, L, smem, c);
        if (DIAG) finalize_diag(prm, L, smem, c);
    }
    HRL_STAMP(6);
}

// ======================================================================== element kernel (small action spaces)
// One thread per ELEMENT of the (rows x A) logits block of the CTA's windows: global loads and gradient stores
// are coalesced without any staging copy, every element-wise step (masking, exp, gradient) is one short
// dependent chain per thread, and the row-wise steps (max, sums, scalar tail) are short loops over A <= 32
// values held in shared memory.  This is the latency-optimal mapping when a window is only a few KB.
template <bool DIAG, bool GRAD>
__global__ void __launch_bounds__(1024) loss_elem_kernel(const LossParams prm) {
    extern __shared__ __align__(128) float smem[];
    __shared__ bool s_last;
    const HrlLossArgs &a = prm.a;
    const CtaCtx c = make_ctx(prm);
    const int P = c.P, Pa = c.Pa, A = c.A, Tt = c.Tt, T0 = c.T0, bi = c.bi, tid = c.tid, nthr = c.nthr;
    const int R = Tt * Pa, per_ep = R * A, nelem = c.nE * per_ep;
    const SmemLayout L = make_layout(prm.EPB, Tt, P, Pa, 1, A, prm.EPB * R * A, -1, false, prm.scan + 1);
    const long long *s_act = reinterpret_cast<const long long *>(smem + L.act);
    float *s_z = smem + L.z, *s_e = smem + L.am;
    HRL_STAMP(0);

    stage_small(prm, L, smem, c);

    // ---- 1a: masked logits, one element per thread (train.py:178-181)
    for (int i = tid; i < nelem; i += nthr) {
        const int e = (c.nE == 1) ? 0 : i / per_ep, rem = i - e * per_ep;
        const int rr = rem / A, t = fdiv(rr, Pa, c.shPa), q = rr - t * Pa;
        const size_t cell = (size_t)(c.b0 + e) * T0 + bi + t;
        float scale = 0.0f;
        if (Pa == P) scale = a.turn_mask[cell * P + q];
        else for (int p = 0; p < P; p++) scale += a.turn_mask[cell * P + p];
        const size_t g = ((size_t)(c.b0 + e) * T0 + bi) * Pa * A + rem;
        s_z[i] = ld_stream(a.policy_raw + g) * scale - ld_stream(a.action_mask + g);
    }
    cp_async_wait_all();
    HRL_STAMP(1);
    __syncthreads();
    baselines(prm, L, smem, c);   // phase 2a: independent of the logits
    // ---- 1b: row max, gathered logit, scale
    for (int r = tid; r < c.nrows; r += nthr) {
        const float *zr = s_z + r * A;
        float m = zr[0];
        for (int j = 1; j < A; j++) m = fmaxf(m, zr[j]);
        const int e = (c.nE == 1) ? 0 : r / R, rr = r - e * R, t = fdiv(rr, Pa, c.shPa), q = rr - t * Pa;
        const int scell = e * Tt + t;
        float scale = 0.0f;
        if (Pa == P) scale = smem[L.tm + scell * P + q];
        else for (int p = 0; p < P; p++) scale += smem[L.tm + scell * P + p];
        smem[L.mx + r] = m;
        smem[L.za + r] = zr[(int)s_act[r]];
        smem[L.scale + r] = scale;
    }
    __syncthreads();
    // ---- 1c: exponentials, one element per thread
    for (int i = tid; i < nelem; i += nthr) {
        const int r = i / A;
        s_e[i] = expf(s_z[i] - smem[L.mx + r]);
    }
    __syncthreads();
    // ---- 1d: row sums, then the scalar tail of the row (log-sum-exp, entropy, log pi(a), clipped ratio)
    for (int r = tid; r < c.nrows; r += nthr) {
        const float *zr = s_z + r * A, *er = s_e + r * A;
        const float m = smem[L.mx + r];
        float se = 0.0f, sw = 0.0f;
        for (int j = 0; j < A; j++) {
            se += er[j];
            sw += er[j] * fmaxf(zr[j] - m, -3.0e38f);
        }
        smem[L.se + r] = se;
        smem[L.sw + r] = sw;
    }
    __syncthreads();
    row_epilogue(prm, L, smem, c);
    HRL_STAMP(2);
    __syncthreads();
    HRL_STAMP(3);

    float part[6], dpart[DIAG ? HRL_NUM_LOSS_DIAG : 1];
    targets_and_losses<DIAG, GRAD>(prm, L, smem, c, part, dpart);
    HRL_STAMP(4);
    if (DIAG) reduce_diag(prm, L, smem, c, dpart);
    reduce_partials(L, smem, c, part);
    if ((tid >> 5) == (nthr >> 5) - 1) publish_partials(prm, L, smem, c, &s_last);
    HRL_STAMP(5);

    // ---- 3a: per-row gradient factors (reusing the se / sw slots), value / return gradients
    for (int r = tid; GRAD && r < c.nrows; r += nthr) {
        const int e = (c.nE == 1) ? 0 : r / R, rr = r - e * R, t = fdiv(rr, Pa, c.shPa), q = rr - t * Pa;
        const RowFactors f = row_factors(prm, L, smem, c.b0 + e, e * Tt + t, q, P, Pa);
        smem[L.se + r] = f.w;
        smem[L.sw + r] = f.k;
        const size_t grow = ((size_t)(c.b0 + e) * T0 + bi) * Pa + rr;
        if (prm.loss_v) a.dvalue_raw[grow] = f.gv;
        if (prm.loss_r) a.dreturn_raw[grow] = f.gr;
    }
    __syncthreads();
    HRL_STAMP(18);
    // ---- 3b: gradients, one element per thread, coalesced stores
    for (int i = tid; GRAD && i < nelem; i += nthr) {
        const int e = (c.nE == 1) ? 0 : i / per_ep, rem = i - e * per_ep;
        const int r = i / A, j = i - r * A;
        const float scale = smem[L.scale + r];
        float g = 0.0f;
        if (scale != 0.0f)
            g = grad_elem(s_z[i], j == (int)s_act[r], smem[L.mx + r], smem[L.lsum + r], smem[L.ent + r], smem[L.se + r],
                          smem[L.sw + r], scale);
        st_stream(a.dpolicy_raw + ((size_t)(c.b0 + e) * T0 + bi) * Pa * A + rem, g);
    }
    HRL_STAMP(19);
    if (GRAD) zero_burn_in(prm, c);
    __syncthreads();
    if (s_last) {
        finalize_losses(prm, L, smem, c);
        if (DIAG) finalize_diag(prm, L, smem, c);
    }
    HRL_STAMP(6);
}

// ======================================================================== group kernel (small action spaces, fewer stages)
// Same job as the element kernel with fewer barrier-separated stages: RL = 2^k >= A lanes own one row, so the row
// maximum, the exponential sums and the gathered logit are warp shuffles inside the lane group (one fused stage
// instead of four), and the gradient stage recomputes the row factors per lane instead of a separate row pass.
template <int RL, bool DIAG, bool GRAD>
__global__ void __launch_bounds__(1024) loss_group_kernel(const LossParams prm) {
    extern __shared__ __align__(128) float smem[];
    __shared__ bool s_last;
    const HrlLossArgs &a = prm.a;
    const CtaCtx c = make_ctx(prm);
    const int P = c.P, Pa = c.Pa, A = c.A, Tt = c.Tt, T0 = c.T0, bi = c.bi, tid = c.tid, nthr = c.nthr;
    const int R = Tt * Pa;
    const SmemLayout L = make_layout(prm.EPB, Tt, P, Pa, 1, A, 0, -1, false, prm.scan + 1);
    const long long *s_act = reinterpret_cast<const long long *>(smem + L.act);
    float *s_z = smem + L.z;
    const int grp = tid / RL, lane = tid % RL, ngrp = nthr / RL;
    HRL_STAMP(0);

    stage_small(prm, L, smem, c);

    // ---- stage 1: masked logits + row statistics, one lane per element, reductions by shuffles
    for (int base = 0; base < c.nrows; base += ngrp) {
        const int r = base + grp;
        const bool valid = r < c.nrows, live = valid && lane < A;
        float z = -INFINITY, scale = 0.0f;
        int act = 0;
        if (valid) {
            const int e = (c.nE == 1) ? 0 : r / R, rr = r - e * R, t = fdiv(rr, Pa, c.shPa), q = rr - t * Pa;
            const size_t cell = (size_t)(c.b0 + e) * T0 + bi + t;
            if (Pa == P) scale = a.turn_mask[cell * P + q];
            else for (int p = 0; p < P; p++) scale += a.turn_mask[cell * P + p];   // train.py:179-180
            act = (int)a.action[cell * Pa + q];
            if (live) {
                const size_t g = (cell * Pa + q) * A + lane;
                z = ld_stream(a.policy_raw + g) * scale - ld_stream(a.action_mask + g);   // train.py:178-181
                s_z[r * A + lane] = z;
            }
        }
        const float m = group_max<RL>(z);
        const float za = group_max<RL>((live && lane == act) ? z : -INFINITY);
        const float d = live ? z - m : 0.0f;
        const float ex = live ? expf(d) : 0.0f;
        const float se = group_sum<RL>(ex);
        const float sw = group_sum<RL>(ex * fmaxf(d, -3.0e38f));
        if (valid && lane == 0) store_row_stats(L, smem, r, za, m, se, sw, scale);
    }
    cp_async_wait_all();
    HRL_STAMP(1);
    __syncthreads();
    baselines(prm, L, smem, c);
    row_epilogue(prm, L, smem, c);
    HRL_STAMP(2);
    __syncthreads();
    HRL_STAMP(3);

    float part[6], dpart[DIAG ? HRL_NUM_LOSS_DIAG : 1];
    targets_and_losses<DIAG, GRAD>(prm, L, smem, c, part, dpart);
    HRL_STAMP(4);
    if (DIAG) reduce_diag(prm, L, smem, c, dpart);
    reduce_partials(L, smem, c, part);
    if ((tid >> 5) == (nthr >> 5) - 1) publish_partials(prm, L, smem, c, &s_last);
    HRL_STAMP(5);

    // ---- stage 3: gradients; every lane gathers its row's factors itself (no separate row pass)
    for (int base = 0; GRAD && base < c.nrows; base += ngrp) {
        const int r = base + grp;
        if (r >= c.nrows) continue;
        const int e = (c.nE == 1) ? 0 : r / R, rr = r - e * R, t = fdiv(rr, Pa, c.shPa), q = rr - t * Pa;
        const RowFactors f = row_factors(prm, L, smem, c.b0 + e, e * Tt + t, q, P, Pa);
        const size_t grow = ((size_t)(c.b0 + e) * T0 + bi) * Pa + rr;
        if (lane < A) {
            const float scale = smem[L.scale + r];
            float g = 0.0f;
            if (scale != 0.0f)
                g = grad_elem(s_z[r * A + lane], lane == (int)s_act[r], smem[L.mx + r], smem[L.lsum + r], smem[L.ent + r], f.w, f.k, scale);
            st_stream(a.dpolicy_raw + grow * A + lane, g);
        }
        if (lane == 0) {
            if (prm.loss_v) a.dvalue_raw[grow] = f.gv;
            if (prm.loss_r) a.dreturn_raw[grow] = f.gr;
        }
    }
    HRL_STAMP(19);
    if (GRAD) zero_burn_in(prm, c);
    __syncthreads();
    if (s_last) {
        finalize_losses(prm, L, smem, c);
        if (DIAG) finalize_diag(prm, L, smem, c);
    }
    HRL_STAMP(6);
}

// ======================================================================== bulk (TMA) kernel
// Wide rows (A % 4 == 0).  A cluster of CS CTAs shares one window: CTA `crank` owns the time steps [t_lo, t_hi).
//   * thread 0 issues one TMA bulk load per chunk of NC logit rows into zbuf right at the start -- the CTA's
//     whole share (64 KB at T=64, A=512, CS=2) is in flight at once, no registers involved;
//   * every warp owns rows warp, warp+NC, ...: it reads the action mask of its NEXT row from global memory with
//     128-bit loads while it reduces the current row out of shared memory (one-row-ahead register prefetch),
//     writes the masked logits back in place, and pushes the row statistics to the peer CTA through DSMEM;
//   * after the (redundant, cheap) recurrences each warp turns its rows into gradients in place and sends every
//     row home with a bulk store.
// Shared memory is zbuf + ~14 KB, so two CTAs (32 row-reducing warps) share an SM.
template <bool DIAG, bool GRAD>
__global__ void __launch_bounds__(544, 2) loss_bulk_kernel(const LossParams prm) {
    extern __shared__ __align__(128) float smem[];
    __shared__ bool s_last;
    const HrlLossArgs &a = prm.a;
    CtaCtx c = make_ctx(prm);
    const int P = c.P, Pa = c.Pa, A = c.A, Tt = c.Tt, T0 = c.T0, bi = c.bi, tid = c.tid;
    const int CS = prm.cluster;
    const uint32_t crank = CS > 1 ? cluster_ctarank() : 0;
    const int Th = (Tt + CS - 1) / CS;
    c.t_lo = min((int)crank * Th, Tt);
    c.t_hi = min(c.t_lo + Th, Tt);
    const int r_lo = c.t_lo * Pa, R = (c.t_hi - c.t_lo) * Pa;    // R: rows owned by this CTA
    const int warp = tid >> 5, lane = tid & 31, NC = c.nthr >> 5;
    const int nchunk = (R + NC - 1) / NC;
    const SmemLayout L = make_layout(1, Tt, P, Pa, 1, A, 0, Th * Pa, false, prm.scan + 1);
    uint64_t *raw_full = reinterpret_cast<uint64_t *>(smem + L.bars);
    const long long *s_act = reinterpret_cast<const long long *>(smem + L.act);
    const size_t ep_off = (((size_t)c.b0 * T0 + bi) * Pa + r_lo) * A;   // first logit this CTA owns
    HRL_STAMP(0);

    if (tid == 0) {
        for (int i = 0; i < nchunk; i++) mbar_init(raw_full + i, 1);
        fence_mbar_init();
    }
    // small per-cell tensors first (a few KB, cp.async) so that they do not queue behind the bulk traffic
    stage_small(prm, L, smem, c);
    __syncthreads();
    // io_bf16: logits arrive (and gradients leave) as bf16 -- 8 bytes per action instead of 12 over the whole pass.  A raw row is
    // loaded into the UPPER half of its fp32 slot (one bulk load per row), widened in place by the statistics pass, and the
    // gradient row is narrowed into the LOWER half before its bulk store: no extra shared memory, no cross-row hazards.
    const bool io16 = a.io_bf16 != 0;
    if (tid == 0) {
        for (int ch = 0; ch < nchunk; ch++) {
            const int rows = min(NC, R - ch * NC);
            if (!io16) {
                const uint32_t bytes = (uint32_t)rows * A * 4;
                mbar_expect_tx(raw_full + ch, bytes);
                bulk_load(smem + L.z + (size_t)ch * NC * A, a.policy_raw + ep_off + (size_t)ch * NC * A, bytes, raw_full + ch);
            } else {
                mbar_expect_tx(raw_full + ch, (uint32_t)rows * A * 2);
                const uint16_t *src = reinterpret_cast<const uint16_t *>(a.policy_raw) + ep_off + (size_t)ch * NC * A;
                for (int r = 0; r < rows; r++)
                    bulk_load(reinterpret_cast<uint16_t *>(smem + L.z + (size_t)(ch * NC + r) * A) + A, src + (size_t)r * A, (uint32_t)A * 2,
                              raw_full + ch);
            }
        }
    }
    // action mask of this warp's first row -> registers (overlaps the wait for the staged tensors)
    float4 am_next[4];
    {
        const float *amp = a.action_mask + ep_off + (size_t)warp * A;
#pragma unroll
        for (int k4 = 0; k4 < 4; k4++) {
            const int j = (k4 * 32 + lane) * 4;
            am_next[k4] = (warp < R && j < A) ? __ldcs(reinterpret_cast<const float4 *>(amp + j)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    cp_async_wait_all();
    __syncthreads();        // staged small tensors visible to every warp
    baselines(prm, L, smem, c);   // phase 2a, while the logits are still in flight
    HRL_STAMP(1);

    // ---------------- statistics pass
    for (int ch = 0; ch < nchunk; ch++) {
        const int rr = ch * NC + warp;              // row within this CTA's share
        if (rr >= R) break;
        const int gr = r_lo + rr;                   // row within the window
        float4 am4[4];
#pragma unroll
        for (int k4 = 0; k4 < 4; k4++) am4[k4] = am_next[k4];
        if (rr + NC < R) {                          // prefetch the next row's mask
            const float *amp = a.action_mask + ep_off + (size_t)(rr + NC) * A;
#pragma unroll
            for (int k4 = 0; k4 < 4; k4++) {
                const int j = (k4 * 32 + lane) * 4;
                if (j < A) am_next[k4] = __ldcs(reinterpret_cast<const float4 *>(amp + j));
            }
        }
        const int t = fdiv(gr, Pa, c.shPa), q = gr - t * Pa;
        float scale = 0.0f;
        if (Pa == P) scale = smem[L.tm + t * P + q];
        else for (int p = 0; p < P; p++) scale += smem[L.tm + t * P + p];   // train.py:179-180
        const int act = (int)s_act[gr];
        if (ch < 4) HRL_STAMP(7 + 2 * ch);
        mbar_wait(raw_full + ch, 0);
        if (ch < 4) HRL_STAMP(8 + 2 * ch);
        float *zrow = smem + L.z + (size_t)rr * A;
        // branch-free over the lane's 16 elements (indices past A are clamped and neutralised)
        float4 z4[4];
        float m = -INFINITY;
#pragma unroll
        for (int k4 = 0; k4 < 4; k4++) {
            const int j = (k4 * 32 + lane) * 4;
            const bool ok = j < A;
            float4 x;
            if (!io16) {
                x = *reinterpret_cast<const float4 *>(zrow + (ok ? j : 0));
            } else {             // four bf16 of the raw row in the slot's upper half: a bf16 is the top half of the fp32
                const uint2 h = *reinterpret_cast<const uint2 *>(reinterpret_cast<const uint16_t *>(zrow) + A + (ok ? j : 0));
                x = make_float4(__uint_as_float(h.x << 16), __uint_as_float(h.x & 0xFFFF0000u), __uint_as_float(h.y << 16),
                                __uint_as_float(h.y & 0xFFFF0000u));
            }
            z4[k4].x = ok ? fmaf(x.x, scale, -am4[k4].x) : -INFINITY;  // train.py:178-181
            z4[k4].y = ok ? fmaf(x.y, scale, -am4[k4].y) : -INFINITY;
            z4[k4].z = ok ? fmaf(x.z, scale, -am4[k4].z) : -INFINITY;
            z4[k4].w = ok ? fmaf(x.w, scale, -am4[k4].w) : -INFINITY;
            m = fmaxf(m, fmaxf(fmaxf(z4[k4].x, z4[k4].y), fmaxf(z4[k4].z, z4[k4].w)));
        }
        __syncwarp();       // every lane has read its raw logits before anyone overwrites them
#pragma unroll
        for (int k4 = 0; k4 < 4; k4++) {
            const int j = (k4 * 32 + lane) * 4;
            if (j < A) *reinterpret_cast<float4 *>(zrow + j) = z4[k4];
        }
        m = group_max<32>(m);
        // S = sum 2^t, W = sum 2^t * t with t = (z - m) * log2(e):  entropy = ln S - ln2 * W / S
        // (z - m first: rows that are masked throughout sit at -1e32 and must cancel exactly)
        float se = 0.0f, sw = 0.0f;
#pragma unroll
        for (int k4 = 0; k4 < 4; k4++) {
            const float zz[4] = {z4[k4].x, z4[k4].y, z4[k4].z, z4[k4].w};
#pragma unroll
            for (int cc = 0; cc < 4; cc++) {
                const float tt = fmaxf((zz[cc] - m) * kLog2e, -1.0e37f);   // padding lanes / masked: 2^t == 0
                const float ex = fast_exp2(tt);
                se += ex;
                sw = fmaf(ex, tt, sw);
            }
        }
        se = group_sum<32>(se);
        sw = group_sum<32>(sw);
        __syncwarp();
        if (lane == 0) {
            const float za = zrow[act], swn = sw * kLn2;
            store_row_stats(L, smem, gr, za, m, se, swn, scale);
            for (uint32_t peer = 0; peer < (uint32_t)CS; peer++) {       // the other CTA of the cluster needs them too
                if (peer == crank) continue;
                st_peer_f32(smem + L.za + gr, peer, za);
                st_peer_f32(smem + L.mx + gr, peer, m);
                st_peer_f32(smem + L.se + gr, peer, se);
                st_peer_f32(smem + L.sw + gr, peer, swn);
                st_peer_f32(smem + L.scale + gr, peer, scale);
            }
        }
    }
    HRL_STAMP(2);
    if (CS > 1) cluster_sync_all(); else __syncthreads();     // every row statistic of the window is now local
    row_epilogue(prm, L, smem, c);
    __syncthreads();
    HRL_STAMP(3);

    float part[6], dpart[DIAG ? HRL_NUM_LOSS_DIAG : 1];
    targets_and_losses<DIAG, GRAD>(prm, L, smem, c, part, dpart);
    HRL_STAMP(4);
    if (DIAG) reduce_diag(prm, L, smem, c, dpart);
    reduce_partials(L, smem, c, part);
    if (warp == NC - 1) publish_partials(prm, L, smem, c, &s_last);
    HRL_STAMP(5);

    // ---------------- gradients: in place, one bulk store per row
    for (int rr = warp; GRAD && rr < R; rr += NC) {
        const int gr = r_lo + rr;
        const int t = fdiv(gr, Pa, c.shPa), q = gr - t * Pa;
        const size_t grow = ((size_t)c.b0 * T0 + bi + t) * Pa + q;
        const RowFactors f = row_factors(prm, L, smem, c.b0, t, q, P, Pa);
        const float scale = smem[L.scale + gr], m = smem[L.mx + gr], lsum = smem[L.lsum + gr], h = smem[L.ent + gr];
        const int act = (int)s_act[gr];
        float *zrow = smem + L.z + (size_t)rr * A;
        // dL/draw_j = scale * (-w (1[j=a] - p_j) + k p_j (lp_j + h)) = p_j * (sk * lp_j + swk) - 1[j=a] * scale * w
        const float sk = scale * f.k, swk = scale * (f.w + f.k * h);
        if (scale == 0.0f) {        // warp-uniform: rows that were not the acting player's get zero gradient
#pragma unroll
            for (int k4 = 0; k4 < 4; k4++) {
                const int j = (k4 * 32 + lane) * 4;
                if (j < A) *reinterpret_cast<float4 *>(zrow + j) = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        } else {
            float4 o4[4];
#pragma unroll
            for (int k4 = 0; k4 < 4; k4++) {
                const int j = (k4 * 32 + lane) * 4;
                const float4 t4 = *reinterpret_cast<const float4 *>(zrow + (j < A ? j : 0));
                const float zz[4] = {t4.x, t4.y, t4.z, t4.w};
                float g[4];
#pragma unroll
                for (int cc = 0; cc < 4; cc++) {
                    const float lp = fmaxf(zz[cc] - m - lsum, -1.0e37f);   // log-softmax, as the reference orders it
                    const float pj = fast_exp2(lp * kLog2e);
                    g[cc] = pj * fmaf(lp, sk, swk);
                }
                if (io16) {          // the action's own term goes in before the row is narrowed
#pragma unroll
                    for (int cc = 0; cc < 4; cc++)
                        if (j + cc == act) g[cc] -= scale * f.w;
                }
                o4[k4] = make_float4(g[0], g[1], g[2], g[3]);
            }
            if (io16) __syncwarp();      // the narrowed row overlays OTHER lanes' fp32 elements: every lane has read first
#pragma unroll
            for (int k4 = 0; k4 < 4; k4++) {
                const int j = (k4 * 32 + lane) * 4;
                if (j >= A) continue;
                if (!io16) {
                    *reinterpret_cast<float4 *>(zrow + j) = o4[k4];
                } else {
                    const __nv_bfloat162 lo = __floats2bfloat162_rn(o4[k4].x, o4[k4].y), hi = __floats2bfloat162_rn(o4[k4].z, o4[k4].w);
                    uint2 pk;
                    pk.x = *reinterpret_cast<const uint32_t *>(&lo);
                    pk.y = *reinterpret_cast<const uint32_t *>(&hi);
                    *reinterpret_cast<uint2 *>(reinterpret_cast<uint16_t *>(zrow) + j) = pk;
                }
            }
        }
        __syncwarp();
        if (lane == 0 && scale != 0.0f && !io16) zrow[act] -= scale * f.w;
        fence_proxy_async();   // generic-proxy writes -> visible to the bulk-copy engine
        __syncwarp();
        if (lane == 0) {
            if (io16) bulk_store(reinterpret_cast<uint16_t *>(a.dpolicy_raw) + grow * A, zrow, (uint32_t)A * 2);
            else bulk_store(a.dpolicy_raw + grow * A, zrow, (uint32_t)A * 4);
            if (prm.loss_v) a.dvalue_raw[grow] = f.gv;
            if (prm.loss_r) a.dreturn_raw[grow] = f.gr;
        }
    }
    if (GRAD && lane == 0) bulk_store_wait_all();
    if (GRAD && crank == 0) zero_burn_in(prm, c);
    __syncthreads();
    if (s_last) {
        finalize_losses(prm, L, smem, c);
        if (DIAG) finalize_diag(prm, L, smem, c);
    }
    HRL_STAMP(6);
}

// ======================================================================== host side
template <typename K>
static int launch_kernel(K kern, const LossParams &prm, int grid, int threads, size_t smem_bytes, cudaStream_t stream) {
    if (smem_bytes > 48 * 1024)
        HRL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    kern<<<grid, threads, smem_bytes, stream>>>(prm);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

template <bool DIAG, bool GRAD>
static int launch_bulk(const LossParams &prm, int grid, int threads, size_t smem_bytes, cudaStream_t stream) {
    HRL_CUDA_CHECK(cudaFuncSetAttribute(loss_bulk_kernel<DIAG, GRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = prm.cluster;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    HRL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, loss_bulk_kernel<DIAG, GRAD>, prm));
    return HRL_OK;
}

static int pow2_ceil(int x) {
    int p = 1;
    while (p < x) p <<= 1;
    return p;
}

// The dispatch of hrl_loss_fwd_bwd; DIAG picks the kernels with the diagnostics sums compiled in, !GRAD the forward-only
// kernels of hrl_loss_fwd (same choice of variant, launch shape and shared memory in every form).
template <bool DIAG, bool GRAD>
static int loss_fwd_bwd(const HrlLossArgs *args, float *diag, void *stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    HRL_REQUIRE(args != nullptr, HRL_ERR_BAD_ARG, "hrl_loss_fwd_bwd: args is NULL");
    const HrlLossArgs &a = *args;
    if (DIAG) {
        HRL_REQUIRE(diag != nullptr, HRL_ERR_BAD_ARG, "hrl_loss_fwd_bwd_diag: diag is NULL");
        HRL_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= loss_diag_workspace_bytes(a.B), HRL_ERR_WORKSPACE,
                    "hrl_loss_fwd_bwd_diag: workspace of %zu bytes is too small (need %zu, hrl_loss_diag_workspace_bytes)",
                    a.workspace_bytes, loss_diag_workspace_bytes(a.B));
    }
    HRL_REQUIRE(a.B > 0 && a.T > 0 && a.P > 0 && a.A > 0, HRL_ERR_BAD_ARG,
                "hrl_loss_fwd_bwd: non-positive dimension (B=%d T=%d P=%d A=%d)", a.B, a.T, a.P, a.A);
    HRL_REQUIRE(a.Pa == 1 || a.Pa == a.P, HRL_ERR_BAD_ARG, "hrl_loss_fwd_bwd: Pa must be 1 or P (Pa=%d P=%d)", a.Pa, a.P);
    HRL_REQUIRE(a.burn_in >= 0 && a.burn_in < a.T, HRL_ERR_BAD_ARG, "hrl_loss_fwd_bwd: burn_in=%d outside [0,T=%d)", a.burn_in, a.T);
    HRL_REQUIRE(a.value_target >= 0 && a.value_target <= 3 && a.policy_target >= 0 && a.policy_target <= 3,
                HRL_ERR_BAD_ARG, "hrl_loss_fwd_bwd: unknown target algorithm (value=%d policy=%d)", a.value_target, a.policy_target);
    HRL_REQUIRE(a.policy_raw && a.action_mask && a.action && a.selected_prob && a.reward && a.ret && a.turn_mask &&
                    a.observation_mask && a.episode_mask && a.progress && a.outcome,
                HRL_ERR_BAD_ARG, "hrl_loss_fwd_bwd: a required input pointer is NULL");
    HRL_REQUIRE(a.losses && (a.dpolicy_raw || !GRAD), HRL_ERR_BAD_ARG, "hrl_loss_fwd_bwd: a required output pointer is NULL");
    HRL_REQUIRE(a.external_heads >= 0 && a.external_heads <= 3, HRL_ERR_BAD_ARG, "hrl_loss_fwd_bwd: external_heads=%d outside 0..3",
                a.external_heads);
    const bool ext_v = a.external_heads & 1, ext_r = a.external_heads & 2;
    HRL_REQUIRE((!ext_v || (a.value_raw && a.tap_target_value)) && (!ext_r || (a.return_raw && a.tap_target_return)), HRL_ERR_BAD_ARG,
                "hrl_loss_fwd_bwd: an external head needs its output and its target tap");
    // a head whose loss another kernel computes has no gradient here; every other head needs both buffers
    HRL_REQUIRE(!GRAD || ((ext_v ? a.dvalue_raw == nullptr : (a.value_raw != nullptr) == (a.dvalue_raw != nullptr)) &&
                          (ext_r ? a.dreturn_raw == nullptr : (a.return_raw != nullptr) == (a.dreturn_raw != nullptr))),
                HRL_ERR_BAD_ARG, "hrl_loss_fwd_bwd: each head needs both its output and its gradient buffer (none when external)");
    HRL_REQUIRE(a.A <= 1024, HRL_ERR_UNSUPPORTED, "hrl_loss_fwd_bwd: A=%d > 1024 not built", a.A);
    HRL_REQUIRE(a.P <= 64, HRL_ERR_UNSUPPORTED, "hrl_loss_fwd_bwd: P=%d > 64 not built", a.P);

    LossParams prm;
    prm.a = a;
    prm.Tt = a.T - a.burn_in;
    prm.has_v = a.value_raw != nullptr;
    prm.has_r = a.return_raw != nullptr;
    prm.loss_v = prm.has_v && !ext_v;
    prm.loss_r = prm.has_r && !ext_r;
    prm.cluster = 1;
    prm.diag = diag;
    const HrlLossTuning &tune = a.tuning;
    HRL_REQUIRE(tune.variant >= 0 && tune.variant <= 5 && tune.recurrence >= 0 && tune.recurrence <= 2 && tune.cluster >= 0 &&
                    tune.cluster <= 8 && tune.consumers >= 0 && tune.threads >= 0 && tune.threads <= 1024 && tune.threads % 32 == 0,
                HRL_ERR_BAD_ARG, "hrl_loss_fwd_bwd: bad tuning block (zero-initialise HrlLossArgs.tuning for the defaults)");
    prm.scan = tune.recurrence ? tune.recurrence - 1 : (prm.Tt >= 96 ? 1 : 0);   // serial recurrences win below ~100 steps
    prm.trace = tune.trace;

    int dev = 0, max_smem = 0;
    HRL_CUDA_CHECK(cudaGetDevice(&dev));
    HRL_CUDA_CHECK(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const size_t smem_cap = (size_t)max_smem - 1024;
    const int R = prm.Tt * a.Pa;

    // row mapping: one thread per row while the row fits in 16 registers, then 2..32 lanes per row
    int LPR = 1;
    while (LPR < 32 && (a.A + LPR - 1) / LPR > 16) LPR <<= 1;
    const int NPL = LPR == 1 ? pow2_ceil(a.A) : (a.A > 512 ? 32 : 16);
    const bool aligned16 = ((reinterpret_cast<uintptr_t>(a.policy_raw) & 15) == 0) &&
                           ((reinterpret_cast<uintptr_t>(a.action_mask) & 15) == 0) &&
                           (!GRAD || (reinterpret_cast<uintptr_t>(a.dpolicy_raw) & 15) == 0);   // hrl_loss_fwd never writes it
    const int mode = tune.variant - 1;               // -1 auto, 0 direct, 1 staged I/O, 2 bulk, 3 element, 4 group

    // ---- bulk (TMA) kernel: wide rows
    if (LPR == 32 && a.A <= 512 && a.A % (a.io_bf16 ? 8 : 4) == 0 && aligned16 && (mode == -1 || mode == 2 || a.io_bf16)) {
        const size_t two_per_sm = 112 * 1024;     // dynamic shared memory that still lets two CTAs share an SM
        const int force_cs = tune.cluster;
        int NCmax = tune.consumers ? tune.consumers : 16;
        if (NCmax > 17) NCmax = 17;
        int best_cs = 0;
        size_t best_bytes = 0;
        // preference: (1) the whole window in one CTA if two such CTAs fit per SM; (2) a 2-CTA cluster splitting the
        // time axis so that two CTAs fit per SM; (3) the whole window in one CTA per SM
        for (int pass = 0; pass < 3 && !best_cs; pass++) {
            int cs = (pass == 1) ? 2 : 1;
            if (force_cs) {                       // tuning override (1, 2, 4 or 8 CTAs per window)
                if (pass != 1) continue;
                cs = force_cs;
            }
            if (cs > 1 && prm.Tt < cs) continue;
            const int zrows = ((prm.Tt + cs - 1) / cs) * a.Pa;
            const SmemLayout L = make_layout(1, prm.Tt, a.P, a.Pa, 1, a.A, 0, zrows, false, prm.scan + 1);
            const size_t bytes = (size_t)L.total * 4;
            const int NC = zrows < NCmax ? zrows : NCmax;
            if (bytes <= ((pass < 2) ? two_per_sm : smem_cap) && (zrows + NC - 1) / NC <= kMaxChunks) {
                best_cs = cs;
                best_bytes = bytes;
            }
        }
        if (best_cs) {
            const int zrows = ((prm.Tt + best_cs - 1) / best_cs) * a.Pa;
            const int NC = zrows < NCmax ? zrows : NCmax;
            prm.EPB = 1;
            prm.stage_z = 1;
            prm.row_stride = a.A;
            prm.cluster = best_cs;
            const int grid = a.B * best_cs;
            HRL_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= 2048 + (size_t)grid * 8 * sizeof(float), HRL_ERR_WORKSPACE,
                        "hrl_loss_fwd_bwd: workspace of %zu bytes is too small", a.workspace_bytes);
            return launch_bulk<DIAG, GRAD>(prm, grid, NC * 32, best_bytes, stream);
        }
        HRL_REQUIRE(mode != 2, HRL_ERR_UNSUPPORTED, "hrl_loss_fwd_bwd: bulk kernel forced but the window does not fit");
    }
    HRL_REQUIRE(!a.io_bf16, HRL_ERR_UNSUPPORTED,
                "hrl_loss_fwd_bwd: bf16 logits / gradients are built for the wide-row (bulk) kernel only: 256 < A <= 512, A %% 8 == 0, "
                "16-byte aligned tensors, a window that fits in shared memory (A=%d T=%d)", a.A, a.T);

    // ---- group kernel: small action spaces, RL = 2^k >= A lanes per row (default for A <= 32)
    if (a.A <= 32 && (mode == -1 || mode == 4)) {
        const int RL = pow2_ceil(a.A);
        const int lanes_ep = R * RL;
        int EPB = lanes_ep >= 256 ? 1 : (256 + lanes_ep - 1) / lanes_ep;
        if (EPB > a.B) EPB = a.B;
        const int grid0 = (a.B + EPB - 1) / EPB;
        int cap = 1024 / ((grid0 + kNumSM - 1) / kNumSM);      // keep the whole grid resident in one wave
        cap = cap / 32 * 32;
        int threads = ((EPB * lanes_ep + 31) / 32) * 32;
        if (threads > cap) threads = cap;
        if (threads > 1024) threads = 1024;
        if (threads < 64) threads = 64;
        if (tune.threads) threads = tune.threads;
        const SmemLayout L = make_layout(EPB, prm.Tt, a.P, a.Pa, 1, a.A, 0, -1, false, prm.scan + 1);
        if ((size_t)L.total * 4 <= (size_t)100 * 1024) {
            prm.EPB = EPB;
            prm.stage_z = 1;
            prm.row_stride = a.A;
            HRL_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= 2048 + (size_t)grid0 * 8 * sizeof(float), HRL_ERR_WORKSPACE,
                        "hrl_loss_fwd_bwd: workspace of %zu bytes is too small", a.workspace_bytes);
            const size_t bytes = (size_t)L.total * 4;
            switch (RL) {
                case 1: return launch_kernel(loss_group_kernel<1, DIAG, GRAD>, prm, grid0, threads, bytes, stream);
                case 2: return launch_kernel(loss_group_kernel<2, DIAG, GRAD>, prm, grid0, threads, bytes, stream);
                case 4: return launch_kernel(loss_group_kernel<4, DIAG, GRAD>, prm, grid0, threads, bytes, stream);
                case 8: return launch_kernel(loss_group_kernel<8, DIAG, GRAD>, prm, grid0, threads, bytes, stream);
                case 16: return launch_kernel(loss_group_kernel<16, DIAG, GRAD>, prm, grid0, threads, bytes, stream);
                default: return launch_kernel(loss_group_kernel<32, DIAG, GRAD>, prm, grid0, threads, bytes, stream);
            }
        }
    }

    // ---- element kernel: small action spaces
    if (LPR <= 2 && (mode == -1 || mode == 3)) {
        const int per_ep = R * a.A;
        int EPB = per_ep >= 256 ? 1 : (256 + per_ep - 1) / per_ep;
        if (EPB > a.B) EPB = a.B;
        // one thread per element, but never so many that the grid needs a second wave (64 regs/thread):
        // the CTAs are latency-bound, residency is what gives throughput
        const int grid0 = (a.B + EPB - 1) / EPB;
        int cap = 1024 / ((grid0 + kNumSM - 1) / kNumSM);
        cap = cap / 32 * 32;
        int threads = ((EPB * per_ep + 31) / 32) * 32;
        if (threads > cap) threads = cap;
        if (threads > 1024) threads = 1024;
        if (threads < 64) threads = 64;
        if (tune.threads) threads = tune.threads;
        const SmemLayout L = make_layout(EPB, prm.Tt, a.P, a.Pa, 1, a.A, EPB * per_ep, -1, false, prm.scan + 1);
        if ((size_t)L.total * 4 <= (size_t)100 * 1024) {
            prm.EPB = EPB;
            prm.stage_z = 1;
            prm.row_stride = a.A;
            const int grid = (a.B + EPB - 1) / EPB;
            HRL_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= 2048 + (size_t)grid * 8 * sizeof(float), HRL_ERR_WORKSPACE,
                        "hrl_loss_fwd_bwd: workspace of %zu bytes is too small", a.workspace_bytes);
            return launch_kernel(loss_elem_kernel<DIAG, GRAD>, prm, grid, threads, (size_t)L.total * 4, stream);
        }
    }

    // ---- rows kernel
    const long lanes = (long)R * LPR;       // lanes that have work in the row phases of one episode
    int threads, EPB;
    if (lanes >= 64) {
        EPB = 1;
        threads = 64;
        while (threads * 2 <= lanes && threads < 256) threads *= 2;
    } else {
        threads = 64;
        EPB = (int)(64 / lanes);
        if (EPB > a.B) EPB = a.B;
    }
    if (tune.threads) threads = tune.threads;
    prm.EPB = EPB;
    const int grid = (a.B + EPB - 1) / EPB;
    const bool vec = (LPR == 32) && (a.A % 4 == 0) && aligned16;
    // staged I/O when both the logits and the masks of the CTA's episodes fit comfortably (>= 2 CTAs per SM)
    prm.row_stride = (LPR == 1 && a.A % 2 == 0) ? a.A + 1 : a.A;
    const size_t io_floats = (size_t)EPB * R * prm.row_stride;
    // staging through cp.async pays for narrow rows; from 16 lanes per row on (A > 128) direct coalesced loads and
    // stores are faster (Geister shape, A=214: 35 us direct vs 41 us staged)
    bool ios = !vec && ((mode == -1 && LPR < 16) || mode == 1);
    prm.stage_z = tune.unstaged ? 0 : 1;
    SmemLayout L = make_layout(EPB, prm.Tt, a.P, a.Pa, 1, prm.row_stride, (int)io_floats, -1, false, prm.scan + 1);
    if (ios && (size_t)L.total * 4 > (mode == 1 ? smem_cap : (size_t)100 * 1024)) ios = false;
    if (ios) {
        prm.stage_z = 1;
    } else {
        prm.row_stride = a.A;
        L = make_layout(EPB, prm.Tt, a.P, a.Pa, prm.stage_z, a.A, 0, -1, false, prm.scan + 1);
        if ((size_t)L.total * 4 > smem_cap) {
            prm.stage_z = 0;
            L = make_layout(EPB, prm.Tt, a.P, a.Pa, 0, a.A, 0, -1, false, prm.scan + 1);
        }
    }
    const size_t smem_bytes = (size_t)L.total * 4;
    HRL_REQUIRE(smem_bytes <= smem_cap, HRL_ERR_UNSUPPORTED,
                "hrl_loss_fwd_bwd: T=%d P=%d needs %zu bytes of shared memory (> %d)", a.T, a.P, smem_bytes, max_smem);
    HRL_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= 2048 + (size_t)grid * 8 * sizeof(float), HRL_ERR_WORKSPACE,
                "hrl_loss_fwd_bwd: workspace of %zu bytes is too small (need %zu)", a.workspace_bytes,
                2048 + (size_t)grid * 8 * sizeof(float));

#define HRL_CASE(l, n, v, s) \
    if (LPR == l && NPL == n && vec == v && ios == s) return launch_kernel(loss_rows_kernel<l, n, v, s, DIAG, GRAD>, prm, grid, threads, smem_bytes, stream);
#define HRL_CASE2(l, n) HRL_CASE(l, n, false, false) HRL_CASE(l, n, false, true)
    HRL_CASE2(1, 1) HRL_CASE2(1, 2) HRL_CASE2(1, 4) HRL_CASE2(1, 8) HRL_CASE2(1, 16)
    HRL_CASE2(2, 16) HRL_CASE2(4, 16) HRL_CASE2(8, 16) HRL_CASE2(16, 16) HRL_CASE2(32, 16)
    HRL_CASE(32, 16, true, false)
    HRL_CASE2(32, 32) HRL_CASE(32, 32, true, false)      // 512 < A <= 1024
#undef HRL_CASE2
#undef HRL_CASE
    set_error("hrl_loss_fwd_bwd: no kernel for LPR=%d NPL=%d", LPR, NPL);
    return HRL_ERR_UNSUPPORTED;
}

}  // namespace hrl

extern "C" size_t hrl_loss_workspace_bytes(int32_t B, int32_t, int32_t, int32_t, int32_t) {
    return hrl::loss_workspace_base_bytes(B);   // header (ticket) + up to eight CTAs (a cluster) per window
}

extern "C" size_t hrl_loss_diag_workspace_bytes(int32_t B, int32_t, int32_t, int32_t, int32_t) {
    return hrl::loss_diag_workspace_bytes(B);   // + the diagnostics partials of up to eight CTAs per window
}

extern "C" int hrl_loss_fwd_bwd(const HrlLossArgs *args, void *stream) { return hrl::loss_fwd_bwd<false, true>(args, nullptr, stream); }

extern "C" int hrl_loss_fwd_bwd_diag(const HrlLossArgs *args, float *diag, void *stream) {
    return hrl::loss_fwd_bwd<true, true>(args, diag, stream);
}

extern "C" int hrl_loss_fwd(const HrlLossArgs *args, void *stream) { return hrl::loss_fwd_bwd<false, false>(args, nullptr, stream); }
