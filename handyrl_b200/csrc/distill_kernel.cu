// Policy distillation term (hrl_distill_fwd_bwd, include/hrl_b200.h): KL(teacher || student) over the policy rows the fused
// loss trains, its gradient added to the loss pass's dpolicy_raw, annealed by the optimiser's step count on the device.
//
// A group of L lanes (L = the power of two >= A, 4 <= L <= 32) owns one row, so one warp takes 32 / L rows at once and the
// loads of a group are consecutive along A.  A row is read three times (maxima; sums of exponentials and the KL numerator;
// the gradient), the second and third from L1 / L2.  Each group's weighted KL goes to its leader lane in fp64; the warps of a
// CTA are summed in warp order, and the last CTA folds the block partials in a fixed order and resets the counter.
#include "common.cuh"

namespace hrl {
namespace {

constexpr int kDistillThreads = 256;
constexpr int kDistillWarps = kDistillThreads / 32;
constexpr int kDistillMaxGrid = kNumSM * 8;
constexpr size_t kDistillHeader = 256;      // the completion counter (zero between launches), then the block partials

struct DistillParams {
    int T, P, Pa, A, burn_in;
    int64_t rows;
    const float *__restrict__ s;
    const float *__restrict__ te;
    const float *__restrict__ m;
    const float *__restrict__ tm;
    const float *__restrict__ ww;
    const int64_t *__restrict__ step;
    float coef;
    int64_t anneal;
    float *__restrict__ dp;
    float *__restrict__ losses;
    float *__restrict__ sums;
    unsigned int *counter;
    double *partials;
};

__device__ __forceinline__ float distill_coef(float coef, int64_t anneal, const int64_t *step) {
    if (anneal <= 0) return coef;
    const double frac = 1.0 - (double)(*step) / (double)anneal;
    return frac > 0.0 ? (float)((double)coef * frac) : 0.f;
}

template <int L>
__global__ void __launch_bounds__(kDistillThreads) distill_kernel(DistillParams p) {
    constexpr int G = 32 / L;                               // rows per warp
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane / L, gl = lane % L;
    const float c = distill_coef(p.coef, p.anneal, p.step);
    const int64_t stride = (int64_t)gridDim.x * kDistillWarps * G;
    double acc = 0.0;                                       // leader lanes: the weighted KL of their rows
    for (int64_t base = ((int64_t)blockIdx.x * kDistillWarps + warp) * G; base < p.rows; base += stride) {
        const int64_t row = base + sub;
        float f = 0.f, w = 0.f;
        if (row < p.rows) {
            const int64_t bt = row / p.Pa;
            const int t = (int)(bt % p.T);
            const int64_t b = bt / p.T;
            if (!(p.burn_in > 0 && p.T > 1 && t < p.burn_in)) {
                const float *tm = p.tm + bt * p.P;
                if (p.Pa == 1) {
                    for (int q = 0; q < p.P; q++) f += tm[q];
                } else {
                    f = tm[row % p.Pa];
                }
                w = p.ww != nullptr ? p.ww[b] : 1.f;
            }
        }
        const bool on = w * f != 0.f;                       // rows of weight 0 are never read: they add exactly 0
        const int64_t off = row * p.A;
        float ms = -INFINITY, mt = -INFINITY;
        for (int a = gl; a < p.A; a += L) {
            if (on) {
                const float mk = p.m[off + a];
                ms = fmaxf(ms, f * p.s[off + a] - mk);
                mt = fmaxf(mt, f * p.te[off + a] - mk);
            }
        }
        ms = group_max<L>(ms);
        mt = group_max<L>(mt);
        float ss = 0.f, st = 0.f, x = 0.f;
        for (int a = gl; a < p.A; a += L) {
            if (on) {
                const float mk = p.m[off + a];
                const float zs = f * p.s[off + a] - mk, zt = f * p.te[off + a] - mk;
                const float et = expf(zt - mt);
                ss += expf(zs - ms);
                st += et;
                if (et > 0.f) x += et * (zt - zs);
            }
        }
        ss = group_sum<L>(ss);
        st = group_sum<L>(st);
        x = group_sum<L>(x);
        if (on) {
            const float lse_s = ms + logf(ss), lse_t = mt + logf(st);
            const float kl = x / st - lse_t + lse_s;
            if (gl == 0) acc += (double)(w * f) * (double)kl;
            if (c > 0.f) {
                const float g = c * w * f * f, rs = 1.f / ss, rt = 1.f / st;
                for (int a = gl; a < p.A; a += L) {
                    const float mk = p.m[off + a];
                    const float ps = expf(f * p.s[off + a] - mk - ms) * rs, pt = expf(f * p.te[off + a] - mk - mt) * rt;
                    p.dp[off + a] += g * (ps - pt);
                }
            }
        }
    }

    __shared__ double warp_part[kDistillWarps];
    __shared__ bool last;
    acc = warp_sum_d(acc);
    if (lane == 0) warp_part[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < kDistillWarps; i++) s += warp_part[i];
        p.partials[blockIdx.x] = s;
        __threadfence();
        last = atomicAdd(p.counter, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last || warp != 0) return;
    __threadfence();
    double s = 0.0;
    for (int i = lane; i < (int)gridDim.x; i += 32) s += __ldcg(p.partials + i);
    s = warp_sum_d(s);
    if (lane == 0) {
        const float term = c > 0.f ? (float)((double)c * s) : 0.f;
        p.sums[0] = (float)s;
        p.sums[1] = term;
        if (c > 0.f) p.losses[HRL_LOSS_TOTAL] += term;
        *p.counter = 0u;
    }
}

int distill_grid(int64_t rows, int A) {
    const int L = A <= 4 ? 4 : A <= 8 ? 8 : A <= 16 ? 16 : 32;
    const int64_t per_cta = (int64_t)kDistillWarps * (32 / L);
    const int64_t need = (rows + per_cta - 1) / per_cta;
    return (int)(need < kDistillMaxGrid ? need : kDistillMaxGrid);
}

}  // namespace
}  // namespace hrl

extern "C" size_t hrl_distill_workspace_bytes(int32_t B, int32_t T, int32_t P, int32_t Pa, int32_t A) {
    (void)P;
    if (B <= 0 || T <= 0 || Pa <= 0 || A <= 0) return hrl::kDistillHeader;
    return hrl::kDistillHeader + sizeof(double) * (size_t)hrl::distill_grid((int64_t)B * T * Pa, A);
}

extern "C" int hrl_distill_fwd_bwd(const HrlDistillArgs *a, void *stream) {
    HRL_REQUIRE(a != nullptr, HRL_ERR_BAD_ARG, "hrl_distill_fwd_bwd: NULL args");
    HRL_REQUIRE(a->B > 0 && a->T > 0 && a->P > 0 && a->Pa > 0 && a->A > 0 && a->burn_in >= 0, HRL_ERR_BAD_ARG,
                "hrl_distill_fwd_bwd: bad dimensions B=%d T=%d P=%d Pa=%d A=%d burn_in=%d", a->B, a->T, a->P, a->Pa, a->A,
                a->burn_in);
    HRL_REQUIRE(!a->io_bf16, HRL_ERR_UNSUPPORTED, "hrl_distill_fwd_bwd: bf16 logits are not supported");
    HRL_REQUIRE(a->Pa == 1 || a->Pa == a->P, HRL_ERR_UNSUPPORTED, "hrl_distill_fwd_bwd: Pa=%d is neither 1 nor P=%d", a->Pa, a->P);
    HRL_REQUIRE(a->A <= 1024 && a->P <= 64, HRL_ERR_UNSUPPORTED, "hrl_distill_fwd_bwd: A=%d P=%d outside A <= 1024, P <= 64",
                a->A, a->P);
    HRL_REQUIRE(a->coef >= 0.f && a->coef <= 3.4e38f && a->anneal_steps >= 0, HRL_ERR_BAD_ARG,
                "hrl_distill_fwd_bwd: coef must be finite and >= 0, anneal_steps >= 0");
    HRL_REQUIRE(a->policy_raw && a->teacher_raw && a->action_mask && a->turn_mask && a->step_count && a->dpolicy_raw &&
                a->losses && a->sums, HRL_ERR_BAD_ARG, "hrl_distill_fwd_bwd: NULL pointer");
    const size_t need = hrl_distill_workspace_bytes(a->B, a->T, a->P, a->Pa, a->A);
    HRL_REQUIRE(a->workspace && a->workspace_bytes >= need && (reinterpret_cast<uintptr_t>(a->workspace) & 255) == 0,
                HRL_ERR_WORKSPACE, "hrl_distill_fwd_bwd: workspace of %zu bytes (256-aligned) needed", need);

    hrl::DistillParams p;
    p.T = a->T; p.P = a->P; p.Pa = a->Pa; p.A = a->A; p.burn_in = a->burn_in;
    p.rows = (int64_t)a->B * a->T * a->Pa;
    p.s = a->policy_raw; p.te = a->teacher_raw; p.m = a->action_mask; p.tm = a->turn_mask; p.ww = a->window_weight;
    p.step = a->step_count; p.coef = a->coef; p.anneal = a->anneal_steps;
    p.dp = a->dpolicy_raw; p.losses = a->losses; p.sums = a->sums;
    char *ws = static_cast<char *>(a->workspace);
    p.counter = reinterpret_cast<unsigned int *>(ws);
    p.partials = reinterpret_cast<double *>(ws + hrl::kDistillHeader);
    const int grid = hrl::distill_grid(p.rows, a->A);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (a->A <= 4) hrl::distill_kernel<4><<<grid, hrl::kDistillThreads, 0, s>>>(p);
    else if (a->A <= 8) hrl::distill_kernel<8><<<grid, hrl::kDistillThreads, 0, s>>>(p);
    else if (a->A <= 16) hrl::distill_kernel<16><<<grid, hrl::kDistillThreads, 0, s>>>(p);
    else hrl::distill_kernel<32><<<grid, hrl::kDistillThreads, 0, s>>>(p);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}
