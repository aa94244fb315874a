// Device-side building blocks shared by the fused loss kernels (loss_kernel.cu).
#pragma once
#include "common.cuh"
#include <math.h>

namespace hrl {

struct LossParams {
    HrlLossArgs a;
    int Tt;       // trained steps = T - burn_in
    int EPB;      // episodes per CTA
    int stage_z;  // masked logits kept in shared memory between the statistics and the gradient phase
    int has_v, has_r;
    int loss_v, loss_r;   // the head's regression sum and gradient are written here (not an external categorical head)
    int row_stride;   // floats between consecutive rows of the staged logits (>= A)
    int scan;             // recurrences as a parallel suffix scan (long windows) instead of a serial loop per column
    int cluster;          // CTAs per window (bulk kernel): 1, or 2 = thread-block cluster splitting the time axis
    long long *trace;  // optional per-phase clock64 stamps of one CTA (HRL_LOSS_TRACE, debugging only)
    float *diag;       // HRL_NUM_DIAG diagnostics sums (kernels built with DIAG only)
};

// workspace: [2048-byte header (ticket) | 8 floats per CTA, up to eight CTAs per window | diagnostics: kDiagStride floats per CTA]
constexpr int kDiagStride = HRL_NUM_LOSS_DIAG;
__host__ __device__ inline size_t loss_workspace_base_bytes(int B) { return 2048 + 8 * (size_t)(B > 0 ? B : 0) * 8 * sizeof(float); }
__host__ __device__ inline size_t loss_diag_workspace_bytes(int B) {
    return loss_workspace_base_bytes(B) + 8 * (size_t)(B > 0 ? B : 0) * kDiagStride * sizeof(float);
}

// shared-memory carve-up, in floats
struct SmemLayout {
    int emask, prog;                                        // [cells]
    int tm, om, rew, ret, wterm, dv, dr;                    // [cols]
    int vb, lamv, rout, lamr;                               // [cols] recurrence inputs
    int coef;                                               // [4 kinds][cols] float4 recurrence coefficients
    int rec;                                                // [4 kinds][cols] recurrence state per step
    int se, sw, za;                                         // [rows] raw row statistics (sum exp, sum exp*d, z[action])
    int outcome;                                            // [EPB*P]
    int logp, rho, ent, mx, lsum, scale, vraw, rraw, prob;  // [rows]
    int act;                                                // [rows] int64 (2 floats each)
    int red;                                                // [12*32]
    int bars;                                               // mbarriers of the bulk loads, 8-byte aligned
    int z;                                                  // [rows*row_stride] if staged
    int am;                                                 // staged action mask: [rows*row_stride] or ring
    int total;
};

enum { kMaxChunks = 64, kMaxStages = 8 };

// alias_coef: the recurrence coefficient/state arrays (used only between the statistics and the gradient phase)
// share storage with the action-mask ring (used only during the statistics phase)
__host__ __device__ inline SmemLayout make_layout(int EPB, int Tt, int P, int Pa, int stage_z, int row_stride,
                                                  int am_floats, int z_rows = -1, bool alias_coef = false,
                                                  int coef_buffers = 2) {
    SmemLayout L;
    int cells = EPB * Tt, cols = cells * P, rows = cells * Pa, o = 0;
    L.emask = o; o += cells;
    L.prog = o; o += cells;
    L.tm = o; o += cols;
    L.om = o; o += cols;
    L.rew = o; o += cols;
    L.ret = o; o += cols;
    L.wterm = o; o += cols;
    L.dv = o; o += cols;
    L.dr = o; o += cols;
    L.vb = o; o += cols;
    L.lamv = o; o += cols;
    L.rout = o; o += cols;
    L.lamr = o; o += cols;
    L.outcome = o; o += EPB * P;
    L.logp = o; o += rows;
    L.rho = o; o += rows;
    L.ent = o; o += rows;
    L.mx = o; o += rows;
    L.lsum = o; o += rows;
    L.scale = o; o += rows;
    L.vraw = o; o += rows;
    L.rraw = o; o += rows;
    L.prob = o; o += rows;
    L.se = o; o += rows;
    L.sw = o; o += rows;
    L.za = o; o += rows;
    o = (o + 1) & ~1;
    L.act = o; o += 2 * rows;
    o = (o + 3) & ~3;
    L.red = o; o += 12 * 32;    // 6 x 32 floats for the block reduce, reused as 6 x 32 doubles by the final fold
    L.bars = o; o += 2 * (kMaxChunks + 2 * kMaxStages);
    o = (o + 31) & ~31;   // 128-byte alignment for the bulk-copy destinations
    L.z = o;
    if (stage_z) o += (z_rows >= 0 ? z_rows : rows) * row_stride;
    o = (o + 31) & ~31;
    L.am = o;
    if (alias_coef && am_floats >= 36 * cols) {
        L.coef = o;
        L.rec = o + 32 * cols;
        o += am_floats;
    } else {
        o += am_floats;
        o = (o + 3) & ~3;
        L.coef = o; o += coef_buffers * 4 * 4 * cols;   // (two for the scan) x 4 kinds x float4
        L.rec = o; o += 4 * cols;
    }
    L.total = o;
    return L;
}

// ---------------------------------------------------------------- async copy primitives
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void cp_async4(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async8(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// TMA 1-D bulk copies (SASS: UBLKCP); sizes and addresses are multiples of 16 bytes
__device__ __forceinline__ void bulk_load(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_store(void *gdst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
                 "r"(bytes)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void bulk_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// thread-block cluster primitives (distributed shared memory)
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void st_peer_f32(const float *local, uint32_t rank, float v) {
    uint32_t addr;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(addr) : "r"(smem_u32(local)), "r"(rank));
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// 2^x on the SFU (MUFU.EX2, max relative error 2^-22); callers fold log2(e) into the argument with one FMA
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// ---------------------------------------------------------------- recurrences (losses.py:16-60)
// The time recursions are split in three: (2a) per-step coefficients, in parallel; (2b) the loop-carried
// part only -- one FMA (V-Trace), two FMAs (TD) or two FMAs + max (UPGO) per step, one 16-byte shared-memory
// load and one store; (2c) targets / advantages / loss terms from the recurrence state, in parallel.
//
//   TD / UPGO (losses.py:20-42):  G_t = r_t + g * mix,  mix = (1-l') v' + l' G_{t+1}  [UPGO: max(v', mix)]
//        coef = { l', (1-l') v', v', r_t }      (primes: step t+1)         state: G_t
//   V-Trace (losses.py:45-60):    acc_t = delta_t + (g l' rho_t) acc_{t+1}
//        coef = { g l' rho_t, delta_t, -, - }                              state: acc_t   (vs_t = acc_t + v_t)
struct CtaCtx {
    int T0, P, Pa, A, bi, Tt;
    int b0, nE, tid, nthr;
    int nrows, ncols, ncells;
    int shP, shPa, shTt;   // log2 when the divisor is a power of two, else -1 (index math without integer division)
    int t_lo, t_hi;        // time steps whose loss terms this CTA accounts for (a cluster splits the window)
};

__host__ __device__ inline int log2_exact(int d) {
    int s = 0;
    while ((1 << s) < d) s++;
    return (1 << s) == d ? s : -1;
}
__device__ __forceinline__ int fdiv(int x, int d, int sh) { return sh >= 0 ? (x >> sh) : (x / d); }


// Every reverse-time step of the three recurrences is a map  x -> max(a, b + c*x)  with c >= 0:
//   TD      G_t   = r + g((1-l')v' + l' G_{t+1})            a = -big, b = r + g(1-l')v', c = g l'
//   UPGO    G_t   = r + g max(v', (1-l')v' + l' G_{t+1})    a = r + g v', b, c as TD
//   V-Trace acc_t = delta_t + (g l' rho_t) acc_{t+1}        a = -big, b = delta_t,       c = g l' rho_t
// Such maps are closed under composition,
//   (f o h)(x) = max(a_f, b_f + c_f a_h, b_f + c_f b_h + c_f c_h x),
// so the value of every step is obtained with a parallel suffix scan over t (Kogge-Stone, log2 T rounds, one
// thread per (kind, column, step)) instead of a T-step serial loop.  The scan reassociates the arithmetic:
// results differ from the sequential order by a few ulp (covered by the 1e-5 parity bar, tested at full size).
constexpr float kNegBig = -3.0e38f;

// ---- serial form (default for short windows): coefficients per step, then one minimal loop per column
__device__ __forceinline__ void fill_coef(int algo, float4 *coef, int Tt, int P, int t, float gamma, float v_next,
                                          float lam_next, float r_t, float v_t, float rho_t, float boot) {
    // coef is the column's array (stride P float4 between steps)
    float4 c4;
    if (algo == HRL_VTRACE) {
        const bool last = (t == Tt - 1);
        const float delta = rho_t * (r_t + gamma * (last ? boot : v_next) - v_t);   // losses.py:48
        c4 = make_float4(last ? 0.0f : gamma * lam_next * rho_t, delta, 0.f, 0.f);
    } else {
        c4 = make_float4(lam_next, (1.0f - lam_next) * v_next, v_next, r_t);
    }
    coef[(size_t)t * P] = c4;
}

__device__ __forceinline__ void run_recurrence(int algo, int Tt, int P, const float4 *__restrict__ coef, float gamma,
                                               float boot, float *__restrict__ state) {
    if (algo == HRL_VTRACE) {
        float acc = 0.0f;
#pragma unroll 4
        for (int t = Tt - 1; t >= 0; t--) {
            const float4 c4 = coef[(size_t)t * P];
            acc = fmaf(c4.x, acc, c4.y);
            state[t * P] = acc;
        }
    } else {
        const bool up = (algo == HRL_UPGO);
        float G = boot;
        state[(Tt - 1) * P] = G;
#pragma unroll 4
        for (int t = Tt - 2; t >= 0; t--) {
            const float4 c4 = coef[(size_t)t * P];
            float mix = fmaf(c4.x, G, c4.y);
            if (up) mix = fmaxf(c4.z, mix);
            G = fmaf(gamma, mix, c4.w);
            state[t * P] = G;
        }
    }
}



__device__ __forceinline__ float4 step_map(int algo, bool last, float gamma, float v_next, float lam_next, float r_t,
                                           float v_t, float rho_t, float boot) {
    if (algo == HRL_VTRACE) {
        const float delta = rho_t * (r_t + gamma * (last ? boot : v_next) - v_t);          // losses.py:48
        return make_float4(kNegBig, delta, last ? 0.0f : gamma * lam_next * rho_t, 0.f);    // losses.py:53
    }
    if (last) return make_float4(kNegBig, 0.0f, 1.0f, 0.f);                                 // identity: G_{T-1} = returns[:, -1]
    const float b = r_t + gamma * ((1.0f - lam_next) * v_next);
    const float a = (algo == HRL_UPGO) ? r_t + gamma * v_next : kNegBig;                    // losses.py:38
    return make_float4(a, b, gamma * lam_next, 0.f);
}

__device__ __forceinline__ float4 compose_maps(const float4 f, const float4 h) {     // f after h
    return make_float4(fmaxf(f.x, fmaf(f.z, h.x, f.y)), fmaf(f.z, h.y, f.y), f.z * h.z, 0.f);
}

// phase 2a: per-(cell, player) baselines (train.py:241-248) and lambda mixing (losses.py:71).  Needs only the staged
// small tensors, so the kernels run it while the logits are still in flight; callers barrier before phase 2b.
__device__ __forceinline__ void baselines(const LossParams &prm, const SmemLayout &L, float *smem, const CtaCtx &c) {
    const HrlLossArgs &a = prm.a;
    const int P = c.P, Pa = c.Pa, Tt = c.Tt;
    const bool sym = a.two_player_zero_sum && P == 2;
    for (int i = c.tid; i < c.ncols; i += c.nthr) {
        const int cell = fdiv(i, P, c.shP), p = i - cell * P;
        const int e = (c.nE == 1) ? 0 : fdiv(cell, Tt, c.shTt);
        const int q = (Pa == P) ? p : 0;
        const float em = smem[L.emask + cell];
        const float om = smem[L.om + i];
        const float vout = smem[L.vraw + cell * Pa + q] * om;      // train.py:184
        float vb = vout, vm = om;
        if (sym) {  // train.py:243-247
            const int po = 1 - p, qo = (Pa == P) ? po : 0;
            const float omo = smem[L.om + cell * P + po];
            const float vo = -(smem[L.vraw + cell * Pa + qo] * omo);
            vb = (vout * om + vo * omo) / (om + omo + 1e-8f);
            vm = fminf(fmaxf(om + omo, 0.0f), 1.0f);
        }
        smem[L.vb + i] = vb * em + smem[L.outcome + e * P + p] * (1.0f - em);   // train.py:248
        smem[L.lamv + i] = a.lambda + (1.0f - a.lambda) * (1.0f - vm);
        smem[L.rout + i] = smem[L.rraw + cell * Pa + q] * om;
        smem[L.lamr + i] = a.lambda + (1.0f - a.lambda) * (1.0f - om);
    }
}

// phases 2b/2c: from per-row statistics (logp, rho, ent in smem) and the baselines of phase 2a to per-cell gradient
// factors and the six loss partial sums of this thread.  Caller must __syncthreads() before (statistics and
// baselines visible) and after.  DIAG: also the HRL_NUM_LOSS_DIAG diagnostics partial sums of this thread in dpart
// (separate accumulators: the order of every loss sum is that of the plain kernels).  GRAD: the training pass, which applies
// HrlLossArgs.window_weight; the forward-only pass (held-out losses) is never weighted and compiles the weight out.
template <bool DIAG, bool GRAD>
__device__ __forceinline__ void targets_and_losses(const LossParams &prm, const SmemLayout &L, float *smem, const CtaCtx &c,
                                                   float part[6], float *dpart) {
    const HrlLossArgs &a = prm.a;
    const int P = c.P, Pa = c.Pa, Tt = c.Tt;
    const int vt = a.value_target, pt = a.policy_target;
    const bool two = (pt != vt);
    const float gam = a.gamma;
    float4 *coef = reinterpret_cast<float4 *>(smem + L.coef);
    const int cstride = c.ncols;   // float4 per kind

    if (prm.trace && blockIdx.x == gridDim.x / 2 && c.tid == 0) prm.trace[15] = clock64();
    // ---- 2b: the recurrences as a parallel suffix scan; one thread per (kind, cell, player).
    //      kinds: 0 value/value_target, 1 return/value_target, 2 value/policy_target, 3 return/policy_target
    const int nkind = two ? 4 : 2;
    const int njob = nkind * c.ncols;
    float4 *bufA = coef, *bufB = coef + (size_t)4 * cstride;
    int *info = reinterpret_cast<int *>(smem + L.rec);     // step index of each job during the scan (rec is written after it)
    for (int job = c.tid; job < njob; job += c.nthr) {
        const int kind = job / c.ncols, i = job - kind * c.ncols;
        const bool rs = kind & 1;
        const int algo = (kind >= 2) ? pt : vt;
        if (!(rs ? prm.has_r : prm.has_v) || algo == HRL_MC) continue;
        const int cell = fdiv(i, P, c.shP), p = i - cell * P;
        const int e = (c.nE == 1) ? 0 : fdiv(cell, Tt, c.shTt), t = cell - e * Tt;
        const bool lastt = (t == Tt - 1);
        const int q = (Pa == P) ? p : 0;
        const int vb = rs ? L.rout : L.vb, lm = rs ? L.lamr : L.lamv;
        const float v_next = lastt ? 0.0f : smem[vb + i + P], lam_next = lastt ? 0.0f : smem[lm + i + P];
        const float boot = rs ? smem[L.ret + (e * Tt + Tt - 1) * P + p] : smem[L.outcome + e * P + p];
        if (prm.scan) {
            bufA[job] = step_map(algo, lastt, rs ? gam : 1.0f, v_next, lam_next, rs ? smem[L.rew + i] : 0.0f, smem[vb + i],
                                 smem[L.rho + cell * Pa + q], boot);
            info[job] = t;      // job table for the scan rounds: no index arithmetic inside them
        } else {
            fill_coef(algo, coef + (size_t)kind * cstride + (size_t)e * Tt * P + p, Tt, P, t, rs ? gam : 1.0f, v_next, lam_next,
                      rs ? smem[L.rew + i] : 0.0f, smem[vb + i], smem[L.rho + cell * Pa + q], boot);
        }
    }
    if (!prm.scan) {
        __syncthreads();
        // serial form: job = (column, kind), kind k runs in warp k (the kinds proceed concurrently)
        const int warp_id = c.tid >> 5, lane_id = c.tid & 31, nwarps = c.nthr >> 5;
        const int ncolumn = c.nE * P;
        for (int kind = warp_id; kind < nkind; kind += nwarps) {
            const bool rs = kind & 1;
            const int algo = (kind >= 2) ? pt : vt;
            if (!(rs ? prm.has_r : prm.has_v) || algo == HRL_MC) continue;
            for (int col = lane_id; col < ncolumn; col += 32) {
                const int e = fdiv(col, P, c.shP), p = col - e * P;
                const size_t base = (size_t)e * Tt * P + p;
                const float boot = rs ? smem[L.ret + (e * Tt + Tt - 1) * P + p] : smem[L.outcome + e * P + p];
                run_recurrence(algo, Tt, P, coef + (size_t)kind * cstride + base, rs ? gam : 1.0f, boot,
                               smem + L.rec + (size_t)kind * c.ncols + base);
            }
        }
        __syncthreads();
    } else {
    for (int job = c.tid; job < njob; job += c.nthr) {      // skipped jobs (MC / absent head) never compose
        const int kind = job / c.ncols;
        const int algo = (kind >= 2) ? pt : vt;
        if (!((kind & 1) ? prm.has_r : prm.has_v) || algo == HRL_MC) info[job] = Tt;
    }
    __syncthreads();
    if (prm.trace && blockIdx.x == gridDim.x / 2 && c.tid == 0) prm.trace[16] = clock64();
    for (int d = 1; d < Tt; d <<= 1) {              // uniform trip count: every thread reaches every barrier
        for (int job = c.tid; job < njob; job += c.nthr) {
            float4 f = bufA[job];
            if (info[job] + d < Tt) f = compose_maps(f, bufA[job + d * P]);       // same column, d steps later
            bufB[job] = f;
        }
        __syncthreads();
        float4 *tmp = bufA; bufA = bufB; bufB = tmp;
    }
    // the composed map of steps t..T-1 applied to the terminal value: G_t (TD/UPGO, x = returns[:, -1]) or acc_t (V-Trace, x = 0)
    for (int job = c.tid; job < njob; job += c.nthr) {
        const int kind = job / c.ncols, i = job - kind * c.ncols;
        const bool rs = kind & 1;
        const int algo = (kind >= 2) ? pt : vt;
        if (!(rs ? prm.has_r : prm.has_v) || algo == HRL_MC) continue;
        const int cell = fdiv(i, P, c.shP), p = i - cell * P;
        const int e = (c.nE == 1) ? 0 : fdiv(cell, Tt, c.shTt);
        const float x0 = (algo == HRL_VTRACE) ? 0.0f : (rs ? smem[L.ret + (e * Tt + Tt - 1) * P + p] : smem[L.outcome + e * P + p]);
        const float4 f = bufA[job];
        smem[L.rec + job] = fmaxf(f.x, fmaf(f.z, x0, f.y));
    }
    __syncthreads();
    }   // scan

    if (prm.trace && blockIdx.x == gridDim.x / 2 && c.tid == 0) prm.trace[17] = clock64();
    // ---- 2c: targets, advantages, per-cell loss terms and gradient factors, one job per (cell, player)
    float Lp = 0.f, Lv = 0.f, Lr = 0.f, Lent = 0.f, Lreg = 0.f, dcnt = 0.f;
    if (DIAG) {
#pragma unroll
        for (int k = 0; k < HRL_NUM_LOSS_DIAG; k++) dpart[k] = 0.f;
    }
    for (int i = c.tid; i < c.ncols; i += c.nthr) {
        const int cell = fdiv(i, P, c.shP), p = i - cell * P;
        const int e = (c.nE == 1) ? 0 : fdiv(cell, Tt, c.shTt), t = cell - e * Tt;
        const bool lastt = (t == Tt - 1);
        const int inext = i + P;
        const int q = (Pa == P) ? p : 0, row = cell * Pa + q;
        const float om = smem[L.om + i], tm = smem[L.tm + i];
        const float rho = smem[L.rho + row];
        const float oc = smem[L.outcome + e * P + p];
        float tg[2] = {0.f, 0.f}, ad[2] = {0.f, 0.f};
#pragma unroll
        for (int rs = 0; rs < 2; rs++) {
            const bool has = rs ? prm.has_r : prm.has_v;
            const int vbo = rs ? L.rout : L.vb;
            const float v_t = smem[vbo + i];
            const float r_t = rs ? smem[L.rew + i] : 0.0f, g = rs ? gam : 1.0f;
            const float ret_t = rs ? smem[L.ret + i] : oc;
            const float boot = rs ? smem[L.ret + (e * Tt + Tt - 1) * P + p] : oc;
#pragma unroll
            for (int pass = 0; pass < 2; pass++) {
                if (pass == 1 && !two) break;
                const int algo = pass ? pt : vt, kind = rs + 2 * pass;
                const float *st = smem + L.rec + (size_t)kind * c.ncols;
                float tgt, adv;
                if (!has) { tgt = ret_t; adv = ret_t; }                                    // losses.py:64-66
                else if (algo == HRL_MC) { tgt = ret_t; adv = ret_t - v_t; }               // losses.py:16-17
                else if (algo == HRL_VTRACE) {
                    tgt = st[i] + v_t;                                                     // losses.py:56
                    const float vs_next = lastt ? boot : st[inext] + smem[vbo + inext];
                    adv = r_t + g * vs_next - v_t;                                         // losses.py:57-58
                } else { tgt = st[i]; adv = tgt - v_t; }
                if (pass == 0) tg[rs] = tgt;
                ad[rs] = adv;
            }
        }
        const float tot_adv = rho * (ad[0] + ad[1]);                            // train.py:265
        const float own = (t >= c.t_lo && t < c.t_hi) ? 1.0f : 0.0f;            // cluster: each cell is summed once
        // importance weight of the window (prioritised replay): it scales each loss term once, after the term is formed,
        // so a weight of exactly 1 changes no bit; dcnt and the diagnostics stay unweighted.  The gradient factors take it
        // in row_factors.
        const float wb = (GRAD && a.window_weight) ? __ldg(a.window_weight + c.b0 + e) : 1.0f;
        smem[L.wterm + i] = tot_adv * tm;
        Lp += own * (-smem[L.logp + row] * tot_adv * tm * wb);                  // train.py:202
        float dv = 0.f, dr = 0.f;
        if (prm.has_v) {                                                        // train.py:204
            const float d = smem[L.vraw + row] * om - tg[0];
            Lv += own * (d * d * om * wb);
            dv = d * om * om;
        }
        if (prm.has_r) {                                                        // train.py:206 smooth_l1, beta 1
            const float d = smem[L.rout + i] - tg[1], adf = fabsf(d);
            Lr += own * ((adf < 1.0f ? 0.5f * d * d : adf - 0.5f) * om * wb);
            dr = fminf(fmaxf(d, -1.0f), 1.0f) * om * om;
        }
        smem[L.dv + i] = dv;
        smem[L.dr + i] = dr;
        const float h = smem[L.ent + row] * tm;                                 // train.py:208
        Lent += own * (h * wb);
        Lreg += own * (h * (1.0f - smem[L.prog + cell] * (1.0f - a.entropy_regularization_decay)) * wb);   // train.py:212
        dcnt += own * tm;
        if (DIAG && own != 0.0f) {
            // the log ratio exactly as row_epilogue forms it before the exp and the clip (train.py:231-238)
            const float em = smem[L.emask + cell], mu = smem[L.prob + row];
            const float lr = smem[L.logp + row] - logf(fminf(fmaxf(mu, 1e-16f), 1.0f)) * em;
            if (tm != 0.0f) {
                dpart[HRL_DIAG_N_POL] += tm;
                dpart[HRL_DIAG_RHO] += tm * expf(lr);
                dpart[HRL_DIAG_RHO_CLIP] += lr > 0.0f ? tm : 0.0f;
                dpart[HRL_DIAG_LOGR] += tm * lr;
                dpart[HRL_DIAG_LOGR2] += tm * lr * lr;
                dpart[HRL_DIAG_ADV] += tm * tot_adv;
                dpart[HRL_DIAG_ADV2] += tm * tot_adv * tot_adv;
            }
            if (prm.has_v) {
                const float e = tg[0] - smem[L.vraw + row] * om;
                dpart[HRL_DIAG_N_VAL] += om;
                dpart[HRL_DIAG_TV] += om * tg[0];
                dpart[HRL_DIAG_TV2] += om * tg[0] * tg[0];
                dpart[HRL_DIAG_EV] += om * e;
                dpart[HRL_DIAG_EV2] += om * e * e;
            }
            if (prm.has_r) {
                const float e = tg[1] - smem[L.rout + i];
                dpart[HRL_DIAG_TR] += om * tg[1];
                dpart[HRL_DIAG_TR2] += om * tg[1] * tg[1];
                dpart[HRL_DIAG_ER] += om * e;
                dpart[HRL_DIAG_ER2] += om * e * e;
            }
        }
        if (own != 0.0f && (a.tap_target_value || a.tap_target_return || a.tap_advantage)) {
            const size_t gcol = ((size_t)(c.b0 + e) * c.T0 + c.bi + t) * P + p;
            if (a.tap_target_value) a.tap_target_value[gcol] = tg[0];
            if (a.tap_target_return) a.tap_target_return[gcol] = tg[1];
            if (a.tap_advantage) a.tap_advantage[gcol] = tot_adv;
        }
    }
    part[0] = Lp; part[1] = Lv; part[2] = Lr; part[3] = Lent; part[4] = Lreg; part[5] = dcnt;
}

// Block-reduce the six partial sums into shared memory (all threads), then let ONE warp publish them while
// the rest of the CTA goes on to the gradient phase: the fence + ticket latency is off the critical path.
__device__ __forceinline__ void reduce_partials(const SmemLayout &L, float *smem, const CtaCtx &c, const float part[6]) {
    const int warp = c.tid >> 5, wl = c.tid & 31;
#pragma unroll
    for (int i = 0; i < 6; i++) {
        float v = warp_sum(part[i]);
        if (wl == 0) smem[L.red + i * 32 + warp] = v;
    }
    __syncthreads();
}

// called by one full warp; *s_flag becomes true iff this CTA was the last one to publish.
// Lane 0 stores the six partials and takes the ticket with ONE acq_rel atomic: its own stores are ordered
// before the ticket by the release half, no separate (slower) fence is needed.
__device__ __forceinline__ void publish_partials(const LossParams &prm, const SmemLayout &L, const float *smem, const CtaCtx &c,
                                                 bool *s_flag) {
    const int lane = c.tid & 31, nwarp = (c.nthr + 31) >> 5;
    unsigned int *counter = reinterpret_cast<unsigned int *>(prm.a.workspace);
    float *partials = reinterpret_cast<float *>(reinterpret_cast<char *>(prm.a.workspace) + 2048);
    float v = 0.f;
    if (lane < 6)
        for (int w2 = 0; w2 < nwarp; w2++) v += smem[L.red + lane * 32 + w2];
    float vals[6];
#pragma unroll
    for (int i = 0; i < 6; i++) vals[i] = __shfl_sync(0xffffffffu, v, i);
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < 6; i++) __stcg(partials + (size_t)blockIdx.x * 8 + i, vals[i]);
        unsigned int ticket;
        asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], 1;" : "=r"(ticket) : "l"(counter) : "memory");
        *s_flag = (ticket == gridDim.x - 1);
    }
}

// Executed by the last CTA only: fold all block partials in a fixed order (fp64) and write the scalars.
__device__ __forceinline__ void finalize_losses(const LossParams &prm, const SmemLayout &L, float *smem, const CtaCtx &c) {
    const int warp = c.tid >> 5, wl = c.tid & 31, nwarp = (c.nthr + 31) >> 5;
    unsigned int *counter = reinterpret_cast<unsigned int *>(prm.a.workspace);
    const float *partials = reinterpret_cast<const float *>(reinterpret_cast<const char *>(prm.a.workspace) + 2048);
    double acc[6] = {0, 0, 0, 0, 0, 0};
    for (int blk = c.tid; blk < (int)gridDim.x; blk += c.nthr) {
#pragma unroll
        for (int i = 0; i < 6; i++) acc[i] += (double)__ldcg(partials + (size_t)blk * 8 + i);
    }
    double *dred = reinterpret_cast<double *>(smem + L.red);  // 12*32 floats = 192 doubles = 6 x 32 warps
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 6; i++) {
        double v = warp_sum_d(acc[i]);
        if (wl == 0) dred[i * 32 + warp] = v;
    }
    __syncthreads();
    if (c.tid == 0) {
        double s[6];
        for (int i = 0; i < 6; i++) {
            s[i] = 0;
            for (int w2 = 0; w2 < nwarp; w2++) s[i] += dred[i * 32 + w2];
        }
        // an external (categorical) head's regression sum is left out: its cross-entropy kernel writes the head's entry
        const double lv = prm.loss_v ? 0.5 * s[1] : 0.0, lr = prm.loss_r ? s[2] : 0.0;
        float *out = prm.a.losses;
        out[HRL_LOSS_P] = (float)s[0];
        out[HRL_LOSS_V] = (float)lv;
        out[HRL_LOSS_R] = (float)lr;
        out[HRL_LOSS_ENT] = (float)s[3];
        out[HRL_LOSS_TOTAL] = (float)(s[0] + lv + lr - (double)prm.a.entropy_regularization * s[4]);  // train.py:211-213
        out[HRL_LOSS_DCNT] = (float)s[5];
        *counter = 0u;  // leave the workspace ready for the next launch
    }
}

// ---- diagnostics (DIAG kernels only): their own block reduction, publish and fixed-order fp64 fold
__device__ __forceinline__ float *diag_partials(const LossParams &prm) {
    return reinterpret_cast<float *>(reinterpret_cast<char *>(prm.a.workspace) + loss_workspace_base_bytes(prm.a.B));
}

// All threads: block-reduce dpart (8 sums per round through the reduction scratch) and store this CTA's partials.  Each
// storing thread fences before the barrier, so the partials are visible device-wide before the publishing warp takes its
// ticket.  Ends with a barrier: the scratch is free for reduce_partials.
__device__ __forceinline__ void reduce_diag(const LossParams &prm, const SmemLayout &L, float *smem, const CtaCtx &c,
                                           const float *dpart) {
    const int warp = c.tid >> 5, wl = c.tid & 31, nwarp = (c.nthr + 31) >> 5;
    float *out = diag_partials(prm) + (size_t)blockIdx.x * kDiagStride;
#pragma unroll
    for (int r0 = 0; r0 < HRL_NUM_LOSS_DIAG; r0 += 8) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const float v = warp_sum(dpart[r0 + i]);
            if (wl == 0) smem[L.red + i * 32 + warp] = v;
        }
        __syncthreads();
        if (c.tid < 8) {
            float s = 0.f;
            for (int w2 = 0; w2 < nwarp; w2++) s += smem[L.red + c.tid * 32 + w2];
            __stcg(out + r0 + c.tid, s);
            __threadfence();
        }
        __syncthreads();
    }
}

// Last CTA only (after finalize_losses): fold every CTA's diagnostics partials in a fixed order in fp64, write prm.diag.
__device__ __forceinline__ void finalize_diag(const LossParams &prm, const SmemLayout &L, float *smem, const CtaCtx &c) {
    const int warp = c.tid >> 5, wl = c.tid & 31, nwarp = (c.nthr + 31) >> 5;
    const float *partials = diag_partials(prm);
    double acc[HRL_NUM_LOSS_DIAG];
#pragma unroll
    for (int i = 0; i < HRL_NUM_LOSS_DIAG; i++) acc[i] = 0.0;
    for (int blk = c.tid; blk < (int)gridDim.x; blk += c.nthr) {
#pragma unroll
        for (int i = 0; i < HRL_NUM_LOSS_DIAG; i++) acc[i] += (double)__ldcg(partials + (size_t)blk * kDiagStride + i);
    }
    double *dred = reinterpret_cast<double *>(smem + L.red);   // 6 x 32 doubles: four sums per round
#pragma unroll
    for (int r0 = 0; r0 < HRL_NUM_LOSS_DIAG; r0 += 4) {
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const double v = warp_sum_d(acc[r0 + i]);
            if (wl == 0) dred[i * 32 + warp] = v;
        }
        __syncthreads();
        if (c.tid < 4) {
            double s = 0.0;
            for (int w2 = 0; w2 < nwarp; w2++) s += dred[c.tid * 32 + w2];
            prm.diag[r0 + c.tid] = (float)s;
        }
    }
    if (c.tid < HRL_NUM_DIAG - HRL_NUM_LOSS_DIAG) prm.diag[HRL_NUM_LOSS_DIAG + c.tid] = 0.0f;   // the optimiser's entries
}

// per-row gradient factors gathered from the per-cell terms (sum over players when Pa == 1), times the importance weight
// of window b (the global window index: `cell` is CTA-local -- e * Tt + t, or t alone where a window spans a cluster)
struct RowFactors {
    float w, k, gv, gr;
};
__device__ __forceinline__ RowFactors row_factors(const LossParams &prm, const SmemLayout &L, const float *smem, int b, int cell,
                                                  int q, int P, int Pa) {
    RowFactors f = {0.f, 0.f, 0.f, 0.f};
    if (Pa == P) {
        f.w = smem[L.wterm + cell * P + q];
        f.k = smem[L.tm + cell * P + q];
        f.gv = smem[L.dv + cell * P + q];
        f.gr = smem[L.dr + cell * P + q];
    } else {
        for (int p = 0; p < P; p++) {
            f.w += smem[L.wterm + cell * P + p];
            f.k += smem[L.tm + cell * P + p];
            f.gv += smem[L.dv + cell * P + p];
            f.gr += smem[L.dr + cell * P + p];
        }
    }
    f.w *= smem[L.emask + cell];
    f.k *= prm.a.entropy_regularization * (1.0f - smem[L.prog + cell] * (1.0f - prm.a.entropy_regularization_decay));
    if (prm.a.window_weight) {
        const float wb = __ldg(prm.a.window_weight + b);
        f.w *= wb;
        f.k *= wb;
        f.gv *= wb;
        f.gr *= wb;
    }
    return f;
}

// dL/dz_j for one element (closed form, SURVEY.md section 7), times d z / d raw = scale
__device__ __forceinline__ float grad_elem(float zj, bool is_act, float m, float lsum, float h, float w, float k, float scale) {
    const float lp = zj - m - lsum;
    const float pj = expf(lp);
    float dz = -w * ((is_act ? 1.0f : 0.0f) - pj);
    if (pj > 0.0f) dz += k * pj * (lp + h);
    return dz * scale;
}

}  // namespace hrl
