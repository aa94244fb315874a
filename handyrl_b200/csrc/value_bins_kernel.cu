// Categorical value heads (hrl_value_bins_expect / hrl_value_bins_fwd_bwd, include/hrl_b200.h): the expectation of a head's
// K-bin distribution, which the fused loss reads in place of a scalar head, and the cross-entropy against the two-hot or
// HL-Gauss distribution of the loss pass's targets, with its gradient with respect to the logits.
//
// A group of L lanes (L = the power of two >= K, 4 <= L <= 32) owns one row, so one warp takes 32 / L rows at once and the
// loads of a group are consecutive along K.  The cross-entropy reads a row three times (maximum; sum of exponentials; loss
// and gradient), the second and third from L1 / L2.  Each group's weighted loss goes to its leader lane in fp64; the warps of
// a CTA are summed in warp order, and the last CTA folds the block partials in a fixed order and resets the counter.
#include "common.cuh"

namespace hrl {
namespace {

constexpr int kBinsThreads = 256;
constexpr int kBinsWarps = kBinsThreads / 32;
constexpr int kBinsMaxGrid = kNumSM * 8;
constexpr size_t kBinsHeader = 256;         // the completion counter (zero between launches), then the block partials

struct BinsParams {
    int T, P, Pa, K, burn_in;
    int64_t rows;
    float low, high, delta, sigma;
    int symlog;
    const float *__restrict__ z;
    float *__restrict__ v;
    const float *__restrict__ y;
    const float *__restrict__ om;
    const float *__restrict__ ww;
    float *__restrict__ dz;
    float *__restrict__ losses;
    int head;
    unsigned int *counter;
    double *partials;
};

__device__ __forceinline__ float symlog_fwd(float y) { return copysignf(log1pf(fabsf(y)), y); }
__device__ __forceinline__ float symlog_inv(float m) { return copysignf(expm1f(fabsf(m)), m); }

// Phi(b) - Phi(a) for a <= b, from the tail that does not cancel: Phi(u) = erfc(-u / sqrt 2) / 2
__device__ __forceinline__ float cdf_diff(float a, float b) {
    constexpr float r = 0.70710678118654752f;
    if (a >= 0.f) return 0.5f * (erfcf(a * r) - erfcf(b * r));
    return 0.5f * (erfcf(-b * r) - erfcf(-a * r));
}

// the target distribution of one column: two-hot (j, u) or the HL-Gauss centre and normaliser
struct Target {
    float x, u, norm;
    int j;
};

__device__ __forceinline__ Target make_target(const BinsParams &p, float y) {
    float x = p.symlog ? symlog_fwd(y) : y;
    x = fminf(fmaxf(x, p.low), p.high);
    Target t;
    t.x = x;
    if (p.sigma == 0.f) {
        int j = (int)floorf((x - p.low) / p.delta);
        j = min(max(j, 0), p.K - 2);
        t.j = j;
        t.u = (x - fmaf((float)j, p.delta, p.low)) / p.delta;
        t.norm = 1.f;
    } else {
        t.j = 0;
        t.u = 0.f;
        const float e0 = p.low - 0.5f * p.delta, eK = p.high + 0.5f * p.delta;
        t.norm = cdf_diff((e0 - x) / p.sigma, (eK - x) / p.sigma);
    }
    return t;
}

__device__ __forceinline__ float target_prob(const BinsParams &p, const Target &t, int k) {
    if (p.sigma == 0.f) return k == t.j ? 1.f - t.u : (k == t.j + 1 ? t.u : 0.f);
    const float ek = fmaf((float)k - 0.5f, p.delta, p.low);
    return cdf_diff((ek - t.x) / p.sigma, (ek + p.delta - t.x) / p.sigma) / t.norm;
}

template <int L>
__global__ void __launch_bounds__(kBinsThreads) bins_expect_kernel(BinsParams p) {
    constexpr int G = 32 / L;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane / L, gl = lane % L;
    const int64_t stride = (int64_t)gridDim.x * kBinsWarps * G;
    for (int64_t base = ((int64_t)blockIdx.x * kBinsWarps + warp) * G; base < p.rows; base += stride) {
        const int64_t row = base + sub;
        const bool on = row < p.rows;
        const int64_t off = row * p.K;
        float m = -INFINITY;
        for (int k = gl; k < p.K; k += L)
            if (on) m = fmaxf(m, p.z[off + k]);
        m = group_max<L>(m);
        float se = 0.f, sc = 0.f;
        for (int k = gl; k < p.K; k += L) {
            if (on) {
                const float e = expf(p.z[off + k] - m);
                se += e;
                sc = fmaf(e, fmaf((float)k, p.delta, p.low), sc);
            }
        }
        se = group_sum<L>(se);
        sc = group_sum<L>(sc);
        if (on && gl == 0) {
            const float mean = sc / se;
            p.v[row] = p.symlog ? symlog_inv(mean) : mean;
        }
    }
}

template <int L, bool GRAD>
__global__ void __launch_bounds__(kBinsThreads) bins_ce_kernel(BinsParams p) {
    constexpr int G = 32 / L;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane / L, gl = lane % L;
    const int64_t stride = (int64_t)gridDim.x * kBinsWarps * G;
    double acc = 0.0;                                       // leader lanes: the weighted cross-entropy of their rows
    for (int64_t base = ((int64_t)blockIdx.x * kBinsWarps + warp) * G; base < p.rows; base += stride) {
        const int64_t row = base + sub;
        // the row's columns: p = q (Pa == P) or every player (Pa == 1), each weighted w_b * om
        float wsum = 0.f, wb = 0.f;
        int64_t col0 = 0;
        int ncol = 0;
        if (row < p.rows) {
            const int64_t bt = row / p.Pa;
            const int t = (int)(bt % p.T);
            const int64_t b = bt / p.T;
            if (!(p.burn_in > 0 && p.T > 1 && t < p.burn_in)) {
                wb = (GRAD && p.ww != nullptr) ? p.ww[b] : 1.f;
                ncol = p.Pa == 1 ? p.P : 1;
                col0 = bt * p.P + (p.Pa == 1 ? 0 : row % p.Pa);
                for (int c = 0; c < ncol; c++) wsum += wb * p.om[col0 + c];
            }
        }
        const int64_t off = row * p.K;
        bool on = false;                                    // a column of nonzero weight: rows of weight 0 are never read
        for (int c = 0; c < ncol; c++) on = on || wb * p.om[col0 + c] != 0.f;
        if (!on) {
            if (GRAD && row < p.rows)
                for (int k = gl; k < p.K; k += L) p.dz[off + k] = 0.f;
            // the group still takes part in the shuffles below
        }
        float m = -INFINITY;
        for (int k = gl; k < p.K; k += L)
            if (on) m = fmaxf(m, p.z[off + k]);
        m = group_max<L>(m);
        float se = 0.f;
        for (int k = gl; k < p.K; k += L)
            if (on) se += expf(p.z[off + k] - m);
        se = group_sum<L>(se);
        const float lse = m + logf(se);
        float ce = 0.f;                                     // sum_c w om_c sum_k pi_k(y_c) log p_k  (negated below)
        for (int k = gl; k < p.K; k += L) {
            if (on) {
                const float lp = p.z[off + k] - lse;
                float g = 0.f;
                for (int c = 0; c < ncol; c++) {
                    const float wc = wb * p.om[col0 + c];
                    if (wc == 0.f) continue;
                    const Target tg = make_target(p, p.y[col0 + c]);
                    const float pi = target_prob(p, tg, k);
                    ce = fmaf(wc * pi, lp, ce);
                    g = fmaf(wc, pi, g);
                }
                if (GRAD) p.dz[off + k] = fmaf(wsum, expf(lp), -g);
            }
        }
        ce = group_sum<L>(ce);
        if (on && gl == 0) acc -= (double)ce;
    }

    __shared__ double warp_part[kBinsWarps];
    __shared__ bool last;
    acc = warp_sum_d(acc);
    if (lane == 0) warp_part[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < kBinsWarps; i++) s += warp_part[i];
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
        const float l = (float)s;
        p.losses[p.head ? HRL_LOSS_R : HRL_LOSS_V] = l;
        p.losses[HRL_LOSS_TOTAL] += l;
        *p.counter = 0u;
    }
}

int bins_lanes(int K) { return K <= 4 ? 4 : K <= 8 ? 8 : K <= 16 ? 16 : 32; }

int bins_grid(int64_t rows, int K) {
    const int64_t per_cta = (int64_t)kBinsWarps * (32 / bins_lanes(K));
    const int64_t need = (rows + per_cta - 1) / per_cta;
    return (int)(need < kBinsMaxGrid ? need : kBinsMaxGrid);
}

int bins_params(const HrlValueBinsArgs *a, const char *name, bool ce, BinsParams &p) {
    HRL_REQUIRE(a != nullptr, HRL_ERR_BAD_ARG, "%s: NULL args", name);
    HRL_REQUIRE(a->B > 0 && a->T > 0 && a->P > 0 && a->Pa > 0 && a->K > 0 && a->burn_in >= 0, HRL_ERR_BAD_ARG,
                "%s: bad dimensions B=%d T=%d P=%d Pa=%d K=%d burn_in=%d", name, a->B, a->T, a->P, a->Pa, a->K, a->burn_in);
    HRL_REQUIRE(a->Pa == 1 || a->Pa == a->P, HRL_ERR_UNSUPPORTED, "%s: Pa=%d is neither 1 nor P=%d", name, a->Pa, a->P);
    HRL_REQUIRE(a->K >= 2 && a->K <= 1024 && a->P <= 64, HRL_ERR_UNSUPPORTED, "%s: K=%d P=%d outside 2 <= K <= 1024, P <= 64", name,
                a->K, a->P);
    HRL_REQUIRE(isfinite(a->low) && isfinite(a->high) && a->low < a->high && isfinite(a->sigma) && a->sigma >= 0.f, HRL_ERR_BAD_ARG,
                "%s: need finite low < high and a finite sigma >= 0 (low=%g high=%g sigma=%g)", name, a->low, a->high, a->sigma);
    HRL_REQUIRE(a->head == 0 || a->head == 1, HRL_ERR_BAD_ARG, "%s: head=%d is neither 0 (value) nor 1 (return)", name, a->head);
    HRL_REQUIRE(a->logits && (ce ? (a->target && a->observation_mask && a->losses) : a->expect != nullptr), HRL_ERR_BAD_ARG,
                "%s: NULL pointer", name);
    p.T = a->T; p.P = a->P; p.Pa = a->Pa; p.K = a->K; p.burn_in = a->burn_in;
    p.rows = (int64_t)a->B * a->T * a->Pa;
    p.low = a->low;
    p.high = a->high;
    p.delta = (a->high - a->low) / (float)(a->K - 1);
    p.sigma = a->sigma;
    p.symlog = a->symlog != 0;
    p.z = a->logits; p.v = a->expect; p.y = a->target; p.om = a->observation_mask; p.ww = a->window_weight;
    p.dz = a->dlogits; p.losses = a->losses; p.head = a->head;
    p.counter = nullptr;
    p.partials = nullptr;
    return HRL_OK;
}

}  // namespace
}  // namespace hrl

extern "C" size_t hrl_value_bins_workspace_bytes(int32_t B, int32_t T, int32_t P, int32_t Pa, int32_t K) {
    (void)P;
    if (B <= 0 || T <= 0 || Pa <= 0 || K <= 0) return hrl::kBinsHeader;
    return hrl::kBinsHeader + sizeof(double) * (size_t)hrl::bins_grid((int64_t)B * T * Pa, K);
}

extern "C" int hrl_value_bins_expect(const HrlValueBinsArgs *a, void *stream) {
    hrl::BinsParams p;
    const int st = hrl::bins_params(a, "hrl_value_bins_expect", false, p);
    if (st != HRL_OK) return st;
    const int grid = hrl::bins_grid(p.rows, p.K);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    switch (hrl::bins_lanes(p.K)) {
        case 4: hrl::bins_expect_kernel<4><<<grid, hrl::kBinsThreads, 0, s>>>(p); break;
        case 8: hrl::bins_expect_kernel<8><<<grid, hrl::kBinsThreads, 0, s>>>(p); break;
        case 16: hrl::bins_expect_kernel<16><<<grid, hrl::kBinsThreads, 0, s>>>(p); break;
        default: hrl::bins_expect_kernel<32><<<grid, hrl::kBinsThreads, 0, s>>>(p); break;
    }
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_value_bins_fwd_bwd(const HrlValueBinsArgs *a, void *stream) {
    hrl::BinsParams p;
    const int st = hrl::bins_params(a, "hrl_value_bins_fwd_bwd", true, p);
    if (st != HRL_OK) return st;
    const size_t need = hrl_value_bins_workspace_bytes(a->B, a->T, a->P, a->Pa, a->K);
    HRL_REQUIRE(a->workspace && a->workspace_bytes >= need && (reinterpret_cast<uintptr_t>(a->workspace) & 255) == 0,
                HRL_ERR_WORKSPACE, "hrl_value_bins_fwd_bwd: workspace of %zu bytes (256-aligned) needed", need);
    char *ws = static_cast<char *>(a->workspace);
    p.counter = reinterpret_cast<unsigned int *>(ws);
    p.partials = reinterpret_cast<double *>(ws + hrl::kBinsHeader);
    const int grid = hrl::bins_grid(p.rows, p.K);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
#define HRL_BINS_LAUNCH(L)                                                                       \
    if (p.dz) hrl::bins_ce_kernel<L, true><<<grid, hrl::kBinsThreads, 0, s>>>(p);                \
    else hrl::bins_ce_kernel<L, false><<<grid, hrl::kBinsThreads, 0, s>>>(p);
    switch (hrl::bins_lanes(p.K)) {
        case 4: HRL_BINS_LAUNCH(4) break;
        case 8: HRL_BINS_LAUNCH(8) break;
        case 16: HRL_BINS_LAUNCH(16) break;
        default: HRL_BINS_LAUNCH(32) break;
    }
#undef HRL_BINS_LAUNCH
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}
