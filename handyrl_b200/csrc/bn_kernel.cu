// Train-mode BatchNorm over (N, C, HW) activations with tiny HW (board games), for the small-board net rewrite
// (handyrl_b200/fastnet.py).  PyTorch's and cuDNN's spatial BatchNorm kernels launch one CTA per channel -- 32 CTAs
// on a 132-SM part, most of the GPU idle -- or decompose into ~14 elementwise/reduction launches.
// Here every pass streams the tensor once with fully coalesced accesses: thread = one column j of the (N, C*HW)
// matrix, CTA = (256 columns) x (a slab of rows).
//   forward : stats partials -> per-channel mean / rstd (+ running stats, as nn.BatchNorm2d) -> normalise
//   backward: partials of sum(dy), sum(dy * xhat) -> per-channel dbeta / dgamma -> dx
// The forward sums are shifted by a per-channel pivot K_c = the channel's value in row 0: var = E[(x-K)^2] - E[x-K]^2.
// Unshifted fp32 sums of x and x^2 lose the variance to cancellation once |mean| / std reaches the hundreds; shifted, the
// sums are of size std and the variance keeps fp32 accuracy whatever the mean (DESIGN.md, "BatchNorm statistics").
#include "common.cuh"

namespace hrl {

constexpr int kBnCols = 256;

__global__ void __launch_bounds__(kBnCols) bn_partials_kernel(const float *__restrict__ x, const float *__restrict__ dy,
                                                              const float *__restrict__ mean, const float *__restrict__ rstd,
                                                              int64_t N, int CHW, int HW, int rows_per_slab,
                                                              float *__restrict__ p0, float *__restrict__ p1, int C) {
    // forward (dy == nullptr): p0 = sum (x-K), p1 = sum (x-K)^2;  backward: p0 = sum dy, p1 = sum dy * xhat
    const int j = blockIdx.x * kBnCols + threadIdx.x;
    if (j >= CHW) return;
    const int64_t r0 = (int64_t)blockIdx.y * rows_per_slab, r1 = min(N, r0 + rows_per_slab);
    const int c = (j / HW) % C;              // NCHW: j = c*HW + h;  channels-last (HW passed as 1): j = f*C + c
    float a = 0.f, b = 0.f;
    if (dy == nullptr) {
        const float K = __ldg(x + c * HW);   // the pivot: row 0, the channel's first column
#pragma unroll 4
        for (int64_t r = r0; r < r1; r++) {
            const float v = __ldg(x + r * CHW + j) - K;
            a += v;
            b = fmaf(v, v, b);
        }
    } else {
        const float m = mean[c], rs = rstd[c];
#pragma unroll 4
        for (int64_t r = r0; r < r1; r++) {
            const float g = __ldg(dy + r * CHW + j);
            const float xh = (__ldg(x + r * CHW + j) - m) * rs;
            a += g;
            b = fmaf(g, xh, b);
        }
    }
    p0[(int64_t)blockIdx.y * CHW + j] = a;
    p1[(int64_t)blockIdx.y * CHW + j] = b;
}

// one CTA per channel folds the partials (slabs x HW columns) in fp64 and adds the pivot x[c * cmul] back to the mean
__global__ void __launch_bounds__(256) bn_finalize_fwd_kernel(const float *__restrict__ x, const float *__restrict__ p0, const float *__restrict__ p1, int slabs,
                                                              int CHW, int reps, int cmul, int istride, double count, float eps, float momentum,
                                                              float *__restrict__ mean, float *__restrict__ rstd,
                                                              float *__restrict__ running_mean, float *__restrict__ running_var) {
    const int c = blockIdx.x;
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < slabs * reps; i += blockDim.x) {        // the channel's columns: c*cmul + h*istride, h < reps
        const int sl = i / reps, h = i - sl * reps;
        s += (double)p0[(int64_t)sl * CHW + c * cmul + h * istride];
        q += (double)p1[(int64_t)sl * CHW + c * cmul + h * istride];
    }
    __shared__ double rs_[8], rq_[8];
    s = warp_sum_d(s);
    q = warp_sum_d(q);
    if ((threadIdx.x & 31) == 0) { rs_[threadIdx.x >> 5] = s; rq_[threadIdx.x >> 5] = q; }
    __syncthreads();
    if (threadIdx.x == 0) {
        s = 0.0; q = 0.0;
        for (int w = 0; w < 8; w++) { s += rs_[w]; q += rq_[w]; }
        const double d = s / count, m = (double)x[c * cmul] + d;
        double var = q / count - d * d;          // biased, as F.batch_norm normalises with
        if (var < 0.0) var = 0.0;
        mean[c] = (float)m;
        rstd[c] = (float)(1.0 / sqrt(var + (double)eps));
        if (running_mean) {
            running_mean[c] = (1.0f - momentum) * running_mean[c] + momentum * (float)m;
            running_var[c] = (1.0f - momentum) * running_var[c] + momentum * (float)(var * count / fmax(count - 1.0, 1.0));
        }
    }
}

__global__ void __launch_bounds__(256) bn_finalize_bwd_kernel(const float *__restrict__ p0, const float *__restrict__ p1, int slabs,
                                                              int CHW, int reps, int cmul, int istride, float *__restrict__ dbeta,
                                                              float *__restrict__ dgamma) {
    const int c = blockIdx.x;
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < slabs * reps; i += blockDim.x) {        // the channel's columns: c*cmul + h*istride, h < reps
        const int sl = i / reps, h = i - sl * reps;
        s += (double)p0[(int64_t)sl * CHW + c * cmul + h * istride];
        q += (double)p1[(int64_t)sl * CHW + c * cmul + h * istride];
    }
    __shared__ double rs_[8], rq_[8];
    s = warp_sum_d(s);
    q = warp_sum_d(q);
    if ((threadIdx.x & 31) == 0) { rs_[threadIdx.x >> 5] = s; rq_[threadIdx.x >> 5] = q; }
    __syncthreads();
    if (threadIdx.x == 0) {
        s = 0.0; q = 0.0;
        for (int w = 0; w < 8; w++) { s += rs_[w]; q += rq_[w]; }
        dbeta[c] = (float)s;
        dgamma[c] = (float)q;
    }
}

// forward: y = (x - mean) * rstd * gamma + beta  (x - mean first: x * scale + (beta - mean * scale) cancels when |mean| >> std)
// backward: dx = gamma * rstd * (dy - dbeta/M - xhat * dgamma/M)
__global__ void __launch_bounds__(kBnCols) bn_apply_kernel(const float *__restrict__ x, const float *__restrict__ dy,
                                                           const float *__restrict__ gamma, const float *__restrict__ beta,
                                                           const float *__restrict__ mean, const float *__restrict__ rstd,
                                                           const float *__restrict__ dbeta, const float *__restrict__ dgamma,
                                                           float inv_count, int64_t N, int CHW, int HW, int rows_per_slab,
                                                           float *__restrict__ out, int C) {
    const int j = blockIdx.x * kBnCols + threadIdx.x;
    if (j >= CHW) return;
    const int c = (j / HW) % C;
    const int64_t r0 = (int64_t)blockIdx.y * rows_per_slab, r1 = min(N, r0 + rows_per_slab);
    const float m = mean[c], rs = rstd[c], g = gamma ? gamma[c] : 1.0f;
    if (dy == nullptr) {
        const float scale = rs * g, b = beta ? beta[c] : 0.0f;
#pragma unroll 4
        for (int64_t r = r0; r < r1; r++) __stcs(out + r * CHW + j, fmaf(__ldg(x + r * CHW + j) - m, scale, b));
    } else {
        const float k = g * rs, mb = dbeta[c] * inv_count, mg = dgamma[c] * inv_count;
#pragma unroll 4
        for (int64_t r = r0; r < r1; r++) {
            const float xh = (__ldg(x + r * CHW + j) - m) * rs;
            __stcs(out + r * CHW + j, k * (__ldg(dy + r * CHW + j) - mb - xh * mg));
        }
    }
}

static void bn_grid(int64_t N, int CHW, int &slabs, int &rows_per_slab, dim3 &grid) {
    const int col_blocks = (CHW + kBnCols - 1) / kBnCols;
    slabs = (int)((N + 63) / 64);
    const int want = (8 * kNumSM + col_blocks - 1) / col_blocks;       // ~8 CTAs per SM
    if (slabs > want) slabs = want;
    if (slabs < 1) slabs = 1;
    rows_per_slab = (int)((N + slabs - 1) / slabs);
    slabs = (int)((N + rows_per_slab - 1) / rows_per_slab);
    grid = dim3(col_blocks, slabs);
}

// the (rows x cols) matrix the passes stream, for NCHW (rows = N, cols = C*HW, column j = c*HW + h) or channels-last
// activations (N*HW pixels of C contiguous channels, folded F pixels to a row so that a CTA's 256 threads all have a
// column: rows = N*HW/F, cols = F*C, column j = f*C + c)
struct BnShape {
    int64_t rows;
    int cols, cdiv, reps, cmul, istride;
};

static BnShape bn_shape(int64_t N, int C, int HW, int channels_last) {
    BnShape b;
    if (!channels_last) {
        b.rows = N; b.cols = C * HW; b.cdiv = HW; b.reps = HW; b.cmul = HW; b.istride = 1;
    } else {
        int F = 1;
        while (F * 2 * C <= kBnCols && (N * HW) % (F * 2) == 0) F *= 2;
        b.rows = N * HW / F; b.cols = F * C; b.cdiv = 1; b.reps = F; b.cmul = 1; b.istride = C;
    }
    return b;
}

}  // namespace hrl

extern "C" size_t hrl_bn_workspace_floats(int64_t N, int32_t C, int32_t HW, int32_t channels_last) {
    int slabs, rps;
    dim3 grid;
    const hrl::BnShape b = hrl::bn_shape(N, C, HW, channels_last);
    hrl::bn_grid(b.rows, b.cols, slabs, rps, grid);
    return (size_t)2 * slabs * b.cols;
}

extern "C" int hrl_bn_train_fwd(const float *x, const float *gamma, const float *beta, float *y, float *mean, float *rstd,
                                float *running_mean, float *running_var, int64_t N, int32_t C, int32_t HW, int32_t channels_last,
                                float eps, float momentum, float *workspace, void *stream_) {
    using namespace hrl;
    HRL_REQUIRE(x && y && mean && rstd && workspace, HRL_ERR_BAD_ARG, "hrl_bn_train_fwd: NULL pointer");
    HRL_REQUIRE(N > 0 && C > 0 && HW > 0 && (running_mean == nullptr) == (running_var == nullptr), HRL_ERR_BAD_ARG,
                "hrl_bn_train_fwd: bad dimensions");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
    const BnShape b = bn_shape(N, C, HW, channels_last);
    int slabs, rps;
    dim3 grid;
    bn_grid(b.rows, b.cols, slabs, rps, grid);
    float *p0 = workspace, *p1 = workspace + (size_t)slabs * b.cols;
    bn_partials_kernel<<<grid, kBnCols, 0, s>>>(x, nullptr, nullptr, nullptr, b.rows, b.cols, b.cdiv, rps, p0, p1, C);
    bn_finalize_fwd_kernel<<<C, 256, 0, s>>>(x, p0, p1, slabs, b.cols, b.reps, b.cmul, b.istride, (double)N * HW, eps, momentum, mean, rstd,
                                             running_mean, running_var);
    bn_apply_kernel<<<grid, kBnCols, 0, s>>>(x, nullptr, gamma, beta, mean, rstd, nullptr, nullptr, 0.0f, b.rows, b.cols, b.cdiv, rps, y, C);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_bn_train_bwd(const float *x, const float *dy, const float *gamma, const float *mean, const float *rstd, float *dx,
                                float *dgamma, float *dbeta, int64_t N, int32_t C, int32_t HW, int32_t channels_last, float *workspace,
                                void *stream_) {
    using namespace hrl;
    HRL_REQUIRE(x && dy && mean && rstd && dx && dgamma && dbeta && workspace, HRL_ERR_BAD_ARG, "hrl_bn_train_bwd: NULL pointer");
    HRL_REQUIRE(N > 0 && C > 0 && HW > 0, HRL_ERR_BAD_ARG, "hrl_bn_train_bwd: bad dimensions");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
    const BnShape b = bn_shape(N, C, HW, channels_last);
    int slabs, rps;
    dim3 grid;
    bn_grid(b.rows, b.cols, slabs, rps, grid);
    float *p0 = workspace, *p1 = workspace + (size_t)slabs * b.cols;
    bn_partials_kernel<<<grid, kBnCols, 0, s>>>(x, dy, mean, rstd, b.rows, b.cols, b.cdiv, rps, p0, p1, C);
    bn_finalize_bwd_kernel<<<C, 256, 0, s>>>(p0, p1, slabs, b.cols, b.reps, b.cmul, b.istride, dbeta, dgamma);
    bn_apply_kernel<<<grid, kBnCols, 0, s>>>(x, dy, gamma, nullptr, mean, rstd, dbeta, dgamma, 1.0f / ((float)N * HW), b.rows, b.cols, b.cdiv,
                                             rps, dx, C);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}
