// Small kernels between the fused tensor-core products of a conv -> BatchNorm -> ReLU tower over a tiny board
// (handyrl_b200/tower.py; the architecture of the reference's SimpleConv2dModel, envs/tictactoe.py:52-69):
//
//   hrl_bn_finalize_fwd   column sums of a layer's output less a pivot (written by hrl_gemm_fused, epilogue STATS, pivot =
//                         ep_mean = mean_col as it is on entry) -> per-channel batch
//                         mean / biased variance -> running statistics (nn.BatchNorm2d semantics) and, per COLUMN of the
//                         (samples x C*HW) activation matrix, the constants the next product's operand transform applies:
//                         scale = gamma*rstd, shift = beta - mean*scale (plus mean and rstd for the backward)
//   hrl_bn_finalize_bwd   column sums of dZ and dZ*xhat (epilogue MASK_STATS) -> dgamma, dbeta and the per-column constants
//                         of dY = dZ*p + Y*q + r (the BatchNorm backward as an operand transform); with `accumulate` it adds
//                         dgamma / dbeta to what they hold (micro-batches after the first of a gradient-accumulation step)
//   hrl_heads_fwd / _bwd  the 1x1-conv "squeeze" outputs (already a product) -> LeakyReLU -> bias-free Linear policy /
//                         tanh value / return heads, and their backward including the parameter gradients
#include <math.h>

#include "common.cuh"

namespace hrl {

__device__ __forceinline__ void block_sum2(double &s, double &q) {
    __shared__ double rs_[32], rq_[32];
    s = warp_sum_d(s);
    q = warp_sum_d(q);
    const int w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    if ((threadIdx.x & 31) == 0) { rs_[w] = s; rq_[w] = q; }
    __syncthreads();
    s = 0.0; q = 0.0;
    for (int i = 0; i < nw; i++) { s += rs_[i]; q += rq_[i]; }     // every thread: same fixed order
    __syncthreads();
}

// one CTA per channel; the sums are of y - K with the pivot K = mean_col[c * HW] on entry (the caller keeps it equal over a
// channel's columns), read before mean_col is overwritten
__global__ void __launch_bounds__(256) bn_tower_finalize_fwd_kernel(const float *__restrict__ partials, int tiles, int C, int HW, double count,
                                                                    const float *__restrict__ gamma, const float *__restrict__ beta, float eps,
                                                                    float momentum, float *__restrict__ running_mean,
                                                                    float *__restrict__ running_var, long long *__restrict__ batches_tracked,
                                                                    float *__restrict__ mean_col, float *__restrict__ rstd_col,
                                                                    float *__restrict__ scale_col, float *__restrict__ shift_col) {
    const int c = blockIdx.x, N = C * HW;
    const double K = (double)mean_col[c * HW];  // (block_sum2's barriers order this read before the stores below)
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < tiles * HW; i += blockDim.x) {
        const int t = i / HW, h = i - t * HW;
        s += (double)partials[((long long)t * 2 + 0) * N + c * HW + h];
        q += (double)partials[((long long)t * 2 + 1) * N + c * HW + h];
    }
    block_sum2(s, q);
    const double d = s / count, m = K + d;
    double var = q / count - d * d;              // biased: what F.batch_norm normalises with
    if (var < 0.0) var = 0.0;
    const float mf = (float)m, rs = (float)(1.0 / sqrt(var + (double)eps));
    const float sc = gamma[c] * rs, sh = beta[c] - mf * sc;
    for (int h = threadIdx.x; h < HW; h += blockDim.x) {
        mean_col[c * HW + h] = mf;
        rstd_col[c * HW + h] = rs;
        scale_col[c * HW + h] = sc;
        shift_col[c * HW + h] = sh;
    }
    if (threadIdx.x == 0) {
        if (running_mean) {
            running_mean[c] = (1.0f - momentum) * running_mean[c] + momentum * mf;
            running_var[c] = (1.0f - momentum) * running_var[c] + momentum * (float)(var * count / fmax(count - 1.0, 1.0));
        }
        if (c == 0 && batches_tracked) *batches_tracked += 1;
    }
}

__global__ void __launch_bounds__(256) bn_tower_finalize_bwd_kernel(const float *__restrict__ partials, int tiles, int C, int HW, double count,
                                                                    const float *__restrict__ gamma, const float *__restrict__ mean_col,
                                                                    const float *__restrict__ rstd_col, float *__restrict__ dgamma,
                                                                    float *__restrict__ dbeta, float *__restrict__ p_col,
                                                                    float *__restrict__ q_col, float *__restrict__ r_col, int accumulate) {
    const int c = blockIdx.x, N = C * HW;
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < tiles * HW; i += blockDim.x) {
        const int t = i / HW, h = i - t * HW;
        s += (double)partials[((long long)t * 2 + 0) * N + c * HW + h];
        q += (double)partials[((long long)t * 2 + 1) * N + c * HW + h];
    }
    block_sum2(s, q);
    if (threadIdx.x == 0) {
        dbeta[c] = accumulate ? dbeta[c] + (float)s : (float)s;                          // sum dZ
        if (dgamma) dgamma[c] = accumulate ? dgamma[c] + (float)q : (float)q;            // sum dZ * xhat
    }
    if (gamma != nullptr) {
        const float mu = mean_col[c * HW], rs = rstd_col[c * HW];
        const float p = gamma[c] * rs;
        const float mean_dz = (float)(s / count), mean_dzx = (float)(q / count);
        const float qq = -p * rs * mean_dzx, rr = p * (rs * mu * mean_dzx - mean_dz);
        for (int h = threadIdx.x; h < HW; h += blockDim.x) {
            p_col[c * HW + h] = p;
            q_col[c * HW + h] = qq;
            r_col[c * HW + h] = rr;
        }
    }
}

// ---- heads.  pre: (M, ld) squeeze outputs, columns [policy maps * cells | value maps * cells | return maps * cells].
constexpr int kHeadMaxIn = 64, kHeadMaxA = 32;

struct HeadsDims {
    int cells, pin, vin, rin, A;       // pin = policy maps * cells etc. (vin / rin may be 0)
};

__global__ void __launch_bounds__(128) heads_fwd_kernel(const float *__restrict__ pre, long long ld, long long M, HeadsDims d, float slope,
                                                        const float *__restrict__ Wp, const float *__restrict__ Wv,
                                                        const float *__restrict__ Wr, float *__restrict__ policy,
                                                        float *__restrict__ value, float *__restrict__ ret) {
    __shared__ float sWp[kHeadMaxA * kHeadMaxIn], sWv[kHeadMaxIn], sWr[kHeadMaxIn];
    for (int i = threadIdx.x; i < d.A * d.pin; i += blockDim.x) sWp[i] = Wp[i];
    for (int i = threadIdx.x; i < d.vin; i += blockDim.x) sWv[i] = Wv[i];
    for (int i = threadIdx.x; i < d.rin; i += blockDim.x) sWr[i] = Wr[i];
    __syncthreads();
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= M) return;
    const float *x = pre + row * ld;
    float h[kHeadMaxIn];
#pragma unroll 4
    for (int j = 0; j < d.pin; j++) { const float v = __ldg(x + j); h[j] = v > 0.f ? v : v * slope; }
    for (int a = 0; a < d.A; a++) {
        float s = 0.f;
        for (int j = 0; j < d.pin; j++) s = fmaf(h[j], sWp[a * d.pin + j], s);
        policy[row * d.A + a] = s;
    }
    if (d.vin) {
        float s = 0.f;
        for (int j = 0; j < d.vin; j++) { const float v = __ldg(x + d.pin + j); s = fmaf(v > 0.f ? v : v * slope, sWv[j], s); }
        value[row] = tanhf(s);
    }
    if (d.rin) {
        float s = 0.f;
        for (int j = 0; j < d.rin; j++) { const float v = __ldg(x + d.pin + d.vin + j); s = fmaf(v > 0.f ? v : v * slope, sWr[j], s); }
        ret[row] = s;
    }
}

// backward: dpre (M, ld) and per-block partial sums of the parameter gradients:
//   [dWp (A*pin) | dWv (vin) | dWr (rin) | dbias per squeeze map (pin+vin+rin)/cells]
// phase 1: a thread per row writes dpre and leaves its activated squeeze outputs h, its dpre and its head gradients in
// shared memory; phase 2: a thread per OUTPUT sums its 128 row products from there (fixed order, no shuffle trees).
__global__ void __launch_bounds__(128) heads_bwd_kernel(const float *__restrict__ pre, long long ld, long long M, HeadsDims d, float slope,
                                                        const float *__restrict__ Wp, const float *__restrict__ Wv,
                                                        const float *__restrict__ Wr, const float *__restrict__ value,
                                                        const float *__restrict__ dpolicy, const float *__restrict__ dvalue,
                                                        const float *__restrict__ dret, float *__restrict__ dpre,
                                                        float *__restrict__ partials, int n_out) {
    __shared__ float sWp[kHeadMaxA * kHeadMaxIn], sWv[kHeadMaxIn], sWr[kHeadMaxIn];
    extern __shared__ float sh[];                  // h [nin][129] | g [nin][129] | dp [A+2][129]   (row index fastest, padded)
    constexpr int S = 129;
    const int nin = d.pin + d.vin + d.rin;
    float *sh_h = sh, *sh_g = sh + nin * S, *sh_d = sh + 2 * nin * S;
    for (int i = threadIdx.x; i < d.A * d.pin; i += blockDim.x) sWp[i] = Wp[i];
    for (int i = threadIdx.x; i < d.vin; i += blockDim.x) sWv[i] = Wv[i];
    for (int i = threadIdx.x; i < d.rin; i += blockDim.x) sWr[i] = Wr[i];
    __syncthreads();
    const int tr = threadIdx.x;
    const long long row = (long long)blockIdx.x * blockDim.x + tr;
    const bool live = row < M;
    const float *x = pre + (live ? row : 0) * ld;
    float dp[kHeadMaxA];
    for (int a = 0; a < d.A; a++) {
        dp[a] = live ? __ldg(dpolicy + row * d.A + a) : 0.f;
        sh_d[a * S + tr] = dp[a];
    }
    float dvp = 0.f, drp = 0.f;
    if (d.vin && live) { const float v = __ldg(value + row); dvp = __ldg(dvalue + row) * (1.f - v * v); }
    if (d.rin && live) drp = __ldg(dret + row);
    sh_d[d.A * S + tr] = dvp;
    sh_d[(d.A + 1) * S + tr] = drp;
    for (int j = 0; j < nin; j++) {
        const float v = live ? __ldg(x + j) : 0.f;
        float g;                                   // gradient wrt the activated squeeze output j
        if (j < d.pin) {
            g = 0.f;
            for (int a = 0; a < d.A; a++) g = fmaf(dp[a], sWp[a * d.pin + j], g);
        } else if (j < d.pin + d.vin) {
            g = dvp * sWv[j - d.pin];
        } else {
            g = drp * sWr[j - d.pin - d.vin];
        }
        const float gp = live ? g * (v > 0.f ? 1.f : slope) : 0.f;
        if (live) dpre[row * ld + j] = gp;
        sh_h[j * S + tr] = live ? (v > 0.f ? v : v * slope) : 0.f;
        sh_g[j * S + tr] = gp;
    }
    __syncthreads();
    const int n_w = d.A * d.pin + d.vin + d.rin;
    for (int o = threadIdx.x; o < n_out; o += blockDim.x) {
        float s = 0.f;
        if (o < n_w) {                              // a Linear weight: sum_rows (head gradient) * (activated input)
            int grad_row, j;
            if (o < d.A * d.pin) { grad_row = o / d.pin; j = o - grad_row * d.pin; }
            else if (o < d.A * d.pin + d.vin) { grad_row = d.A; j = d.pin + (o - d.A * d.pin); }
            else { grad_row = d.A + 1; j = d.pin + d.vin + (o - d.A * d.pin - d.vin); }
            const float *gd = sh_d + grad_row * S, *hh = sh_h + j * S;
            for (int r = 0; r < 128; r++) s = fmaf(gd[r], hh[r], s);
        } else {                                    // a squeeze bias: sum over rows and the map's cells of dpre
            const int map = o - n_w;
            for (int cell = 0; cell < d.cells; cell++) {
                const float *gg = sh_g + (map * d.cells + cell) * S;
                for (int r = 0; r < 128; r++) s += gg[r];
            }
        }
        partials[(long long)blockIdx.x * n_out + o] = s;
    }
}

// out[i] = sum over blocks of partials[block][i] in a fixed order, scattered to up to 8 destination ranges (accumulate: added to
// what the ranges hold, the fp64 sum rounded to fp32 first)
struct ScatterPlan {
    float *dst[8];
    int begin[8];       // first index of the range in the partial vector; range k covers [begin[k], begin[k+1])
    int n;              // ranges
    int total;
};

__global__ void heads_fold_kernel(const float *__restrict__ partials, int blocks, ScatterPlan plan, int accumulate) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= plan.total) return;
    double s = 0.0;
    for (int b = 0; b < blocks; b++) s += (double)partials[(long long)b * plan.total + i];
    int k = 0;
    while (k + 1 < plan.n && i >= plan.begin[k + 1]) k++;
    float *d = plan.dst[k] + (i - plan.begin[k]);
    *d = accumulate ? *d + (float)s : (float)s;
}

}  // namespace hrl

using namespace hrl;

extern "C" int hrl_bn_finalize_fwd(const float *col_partials, int32_t tiles, int32_t C, int32_t HW, int64_t rows, const float *gamma,
                                   const float *beta, float eps, float momentum, float *running_mean, float *running_var,
                                   int64_t *batches_tracked, float *mean_col, float *rstd_col, float *scale_col, float *shift_col,
                                   void *stream) {
    HRL_REQUIRE(col_partials && gamma && beta && mean_col && rstd_col && scale_col && shift_col && tiles > 0 && C > 0 && HW > 0 && rows > 0,
                HRL_ERR_BAD_ARG, "hrl_bn_finalize_fwd: NULL pointer or bad shape");
    HRL_REQUIRE((running_mean == nullptr) == (running_var == nullptr), HRL_ERR_BAD_ARG, "hrl_bn_finalize_fwd: running statistics come in pairs");
    bn_tower_finalize_fwd_kernel<<<C, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        col_partials, tiles, C, HW, (double)rows * HW, gamma, beta, eps, momentum, running_mean, running_var,
        reinterpret_cast<long long *>(batches_tracked), mean_col, rstd_col, scale_col, shift_col);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_bn_finalize_bwd(const float *col_partials, int32_t tiles, int32_t C, int32_t HW, int64_t rows, const float *gamma,
                                   const float *mean_col, const float *rstd_col, float *dgamma, float *dbeta, float *p_col, float *q_col,
                                   float *r_col, int32_t accumulate, void *stream) {
    HRL_REQUIRE(col_partials && dbeta && tiles > 0 && C > 0 && HW > 0 && rows > 0, HRL_ERR_BAD_ARG, "hrl_bn_finalize_bwd: NULL pointer or bad shape");
    HRL_REQUIRE(gamma == nullptr || (mean_col && rstd_col && dgamma && p_col && q_col && r_col), HRL_ERR_BAD_ARG,
                "hrl_bn_finalize_bwd: with gamma, every BatchNorm output is required");
    bn_tower_finalize_bwd_kernel<<<C, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(col_partials, tiles, C, HW, (double)rows * HW, gamma,
                                                                                       mean_col, rstd_col, dgamma, dbeta, p_col, q_col, r_col,
                                                                                       accumulate ? 1 : 0);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

static int heads_dims(int32_t cells, int32_t pmaps, int32_t vmaps, int32_t rmaps, int32_t A, HeadsDims &d) {
    d.cells = cells; d.pin = pmaps * cells; d.vin = vmaps * cells; d.rin = rmaps * cells; d.A = A;
    HRL_REQUIRE(cells > 0 && pmaps > 0 && vmaps >= 0 && rmaps >= 0 && A > 0 && A <= kHeadMaxA && d.pin <= kHeadMaxIn && d.vin <= kHeadMaxIn &&
                    d.rin <= kHeadMaxIn && d.pin + d.vin + d.rin <= kHeadMaxIn,
                HRL_ERR_UNSUPPORTED, "hrl_heads: head sizes outside the built range (A <= %d, squeeze outputs <= %d)", kHeadMaxA, kHeadMaxIn);
    return HRL_OK;
}

extern "C" int32_t hrl_heads_num_blocks(int64_t M) { return (int32_t)((M + 127) / 128); }

extern "C" int hrl_heads_fwd(const float *pre, int64_t ld, int64_t M, int32_t cells, int32_t pmaps, int32_t vmaps, int32_t rmaps, int32_t A,
                             float slope, const float *Wp, const float *Wv, const float *Wr, float *policy, float *value, float *ret,
                             void *stream) {
    HeadsDims d;
    if (int e = heads_dims(cells, pmaps, vmaps, rmaps, A, d)) return e;
    HRL_REQUIRE(pre && Wp && policy && M > 0 && (!vmaps || (Wv && value)) && (!rmaps || (Wr && ret)), HRL_ERR_BAD_ARG, "hrl_heads_fwd: NULL pointer");
    heads_fwd_kernel<<<hrl_heads_num_blocks(M), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(pre, ld, M, d, slope, Wp, Wv, Wr, policy, value, ret);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_heads_bwd(const float *pre, int64_t ld, int64_t M, int32_t cells, int32_t pmaps, int32_t vmaps, int32_t rmaps, int32_t A,
                             float slope, const float *Wp, const float *Wv, const float *Wr, const float *value, const float *dpolicy,
                             const float *dvalue, const float *dret, float *dpre, float *dWp, float *dWv, float *dWr, float *dbias_p,
                             float *dbias_v, float *dbias_r, float *workspace, int32_t accumulate, void *stream_) {
    HeadsDims d;
    if (int e = heads_dims(cells, pmaps, vmaps, rmaps, A, d)) return e;
    HRL_REQUIRE(pre && Wp && dpolicy && dpre && dWp && dbias_p && workspace && M > 0 && (!vmaps || (Wv && value && dvalue && dWv && dbias_v)) &&
                    (!rmaps || (Wr && dret && dWr && dbias_r)),
                HRL_ERR_BAD_ARG, "hrl_heads_bwd: NULL pointer");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const int n_out = A * d.pin + d.vin + d.rin + pmaps + vmaps + rmaps;
    const int blocks = hrl_heads_num_blocks(M);
    const size_t sh_bytes = (size_t)(2 * (d.pin + d.vin + d.rin) + A + 2) * 129 * sizeof(float);
    if (sh_bytes > 40 * 1024)
        HRL_CUDA_CHECK(cudaFuncSetAttribute(heads_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh_bytes));
    heads_bwd_kernel<<<blocks, 128, sh_bytes, stream>>>(pre, ld, M, d, slope, Wp, Wv, Wr, value, dpolicy, dvalue, dret, dpre, workspace, n_out);
    HRL_CUDA_CHECK(cudaGetLastError());
    ScatterPlan plan;
    int k = 0, at = 0;
    plan.dst[k] = dWp; plan.begin[k++] = at; at += A * d.pin;
    if (vmaps) { plan.dst[k] = dWv; plan.begin[k++] = at; at += d.vin; }
    if (rmaps) { plan.dst[k] = dWr; plan.begin[k++] = at; at += d.rin; }
    plan.dst[k] = dbias_p; plan.begin[k++] = at; at += pmaps;
    if (vmaps) { plan.dst[k] = dbias_v; plan.begin[k++] = at; at += vmaps; }
    if (rmaps) { plan.dst[k] = dbias_r; plan.begin[k++] = at; at += rmaps; }
    plan.n = k;
    plan.total = at;
    heads_fold_kernel<<<(at + 127) / 128, 128, 0, stream>>>(workspace, blocks, plan, accumulate ? 1 : 0);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}
