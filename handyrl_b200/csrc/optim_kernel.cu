// K3 -- clip_grad_norm_(4.0) + Adam(weight_decay) on one flat fp32 bucket
// (handyrl/train.py:370-371 with the optimiser of train.py:331).
//
// Two launches so that the global norm is a true grid-wide reduction without cooperative
// launch: hrl_grad_sumsq writes kPartials block partials (fixed grid => fixed summation order
// => bit-reproducible), hrl_clip_adam_step has every block fold those partials itself and
// then update its slice.  lr and the step counter are read from device memory so a captured
// CUDA graph keeps working while the host changes the learning rate (train.py:383-384).
#include "common.cuh"

namespace hrl {

constexpr int kPartials = 2 * kNumSM;  // 264 blocks: two per SM
constexpr int kOptThreads = 256;

__global__ void __launch_bounds__(kOptThreads) grad_sumsq_kernel(const float *__restrict__ g, int64_t n,
                                                                  float *__restrict__ partials) {
    float acc = 0.f;
    const int64_t n4 = n >> 2;
    const float4 *g4 = reinterpret_cast<const float4 *>(g);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 v = g4[i];
        acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    if (blockIdx.x == 0)
        for (int64_t i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) acc += g[i] * g[i];
    __shared__ float red[kOptThreads / 32];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < kOptThreads / 32; w++) s += red[w];
        partials[blockIdx.x] = s;
    }
}

// DIAG: block 0 also adds g, g^2, [g > max_norm], 1 to diag[0..3] (learner diagnostics, include/hrl_b200.h)
template <bool DIAG>
__global__ void __launch_bounds__(kOptThreads) clip_adam_kernel(
    float *__restrict__ param, const float *__restrict__ grad, float *__restrict__ exp_avg,
    float *__restrict__ exp_avg_sq, int64_t n, const float *__restrict__ partials, const float *__restrict__ lr_p,
    int64_t *step_p, double max_norm_d, double beta1_d, double beta2_d, double eps_d, double wd_d,
    float *grad_norm_out, double *diag) {
    const float max_norm = (float)max_norm_d, beta2 = (float)beta2_d, eps = (float)eps_d, wd = (float)wd_d;
    // every block folds the partial sums in the same order -> identical clip coefficient everywhere
    __shared__ double red[kOptThreads / 32];
    __shared__ float s_coef;
    double acc = 0.0;
    for (int i = threadIdx.x; i < kPartials; i += blockDim.x) acc += (double)partials[i];
    acc = warp_sum_d(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < kOptThreads / 32; w++) s += red[w];
        float total_norm = (float)sqrt(s);
        float coef = max_norm / (total_norm + 1e-6f);  // torch clip_grad_norm_
        s_coef = fminf(coef, 1.0f);
        if (blockIdx.x == 0 && grad_norm_out) *grad_norm_out = total_norm;
        if (DIAG && blockIdx.x == 0) {
            diag[0] += (double)total_norm;
            diag[1] += (double)total_norm * (double)total_norm;
            diag[2] += total_norm > max_norm ? 1.0 : 0.0;
            diag[3] += 1.0;
        }
    }
    __syncthreads();
    const float coef = s_coef;
    const int64_t t = *step_p + 1;
    const float lr = *lr_p;
    const double bc1 = 1.0 - pow(beta1_d, (double)t);
    const double bc2 = 1.0 - pow(beta2_d, (double)t);
    const float step_size = (float)((double)lr / bc1);
    const float bc2_sqrt = (float)sqrt(bc2);
    const float omb1 = (float)(1.0 - beta1_d), omb2 = (float)(1.0 - beta2_d);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float p = param[i];
        float g = grad[i] * coef;
        g = g + wd * p;
        float m = exp_avg[i], v = exp_avg_sq[i];
        m = m + (g - m) * omb1;
        v = v * beta2 + omb2 * g * g;
        float denom = sqrtf(v) / bc2_sqrt + eps;
        param[i] = p - step_size * (m / denom);
        exp_avg[i] = m;
        exp_avg_sq[i] = v;
    }
}

// ---- one-shot all-reduce over NVLink peer memory, fused with the sum-of-squares partials -------------------
__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 ld_peer_f4(const float *p) {   // never served from a stale cache line
    float4 v;
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}

constexpr int kMaxWorld = 16;
constexpr unsigned long long kPeerTimeoutNs = 20ull * 1000 * 1000 * 1000;   // a rank that never arrives must not hang the GPU

__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// spin until *flag >= e; gives up after kPeerTimeoutNs (or at once when another wait already gave up) and raises *status
__device__ __forceinline__ void wait_flag(const uint32_t *flag, uint32_t e, uint32_t *status) {
    if (ld_acquire_sys(flag) >= e) return;
    const unsigned long long t0 = global_ns();
    while (ld_acquire_sys(flag) < e) {
        if (*reinterpret_cast<volatile uint32_t *>(status) != 0u) return;
        if (global_ns() - t0 > kPeerTimeoutNs) {
            atomicExch(status, 1u);
            return;
        }
    }
}

__global__ void __launch_bounds__(kOptThreads) peer_allreduce_sumsq_kernel(
    float *__restrict__ out, const float *const *__restrict__ peers, int64_t flag_offset, int world, int rank, int64_t n,
    int64_t n_norm, float *__restrict__ partials, uint32_t *epoch_p, uint32_t *ticket_p, uint32_t *status) {
    __shared__ const float *s_peer[kMaxWorld];
    __shared__ uint32_t s_epoch;
    if (threadIdx.x < world) s_peer[threadIdx.x] = peers[threadIdx.x];
    __syncthreads();
    uint32_t *my_flags = reinterpret_cast<uint32_t *>(const_cast<float *>(s_peer[rank])) + flag_offset;
    if (threadIdx.x == 0) {
        const uint32_t e = *epoch_p + 1;        // read by every block before the last block bumps it (ticket below)
        s_epoch = e;
        if (blockIdx.x == 0)                    // "my gradients are ready" -> slot [rank] of every rank's flags
            for (int p = 0; p < world; p++)
                st_release_sys(reinterpret_cast<uint32_t *>(const_cast<float *>(s_peer[p])) + flag_offset + rank, e);
        for (int p = 0; p < world; p++)         // wait until every rank's gradients are ready (epochs only grow)
            wait_flag(my_flags + p, e, status);
    }
    __syncthreads();

    float acc = 0.f;
    const int64_t n4 = n >> 2;                  // n is a multiple of 4 (FlatAdam pads the bucket)
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 s = ld_peer_f4(s_peer[0] + 4 * i);
        for (int r = 1; r < world; r++) {       // fixed rank order: bit-identical sums on every rank
            const float4 v = ld_peer_f4(s_peer[r] + 4 * i);
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
        reinterpret_cast<float4 *>(out)[i] = s;
        if (4 * i < n_norm) acc += s.x * s.x + s.y * s.y + s.z * s.z + s.w * s.w;
    }
    __shared__ float red[kOptThreads / 32];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < kOptThreads / 32; w++) s += red[w];
        partials[blockIdx.x] = s;
        __threadfence();
        if (atomicAdd(ticket_p, 1u) == gridDim.x - 1) {      // last block: every block of this rank has finished reading
            const uint32_t e = s_epoch;
            *ticket_p = 0u;
            for (int p = 0; p < world; p++)                  // "I am done reading" -> slot [world + rank]
                st_release_sys(reinterpret_cast<uint32_t *>(const_cast<float *>(s_peer[p])) + flag_offset + world + rank, e);
            for (int p = 0; p < world; p++)                  // nobody still reads MY bucket -> the next step may overwrite it
                wait_flag(my_flags + world + p, e, status);
            *epoch_p = e;
        }
    }
}

// the step counter is bumped by a 1-thread epilogue so that every block of clip_adam_kernel
// reads the same value regardless of scheduling
__global__ void bump_step_kernel(int64_t *step_p) { *step_p += 1; }

// moving average of the learner's state after the optimiser step: a <- fmaf(w, x - a, a),
// w = 1 - decay once seeded, else max(1 - decay, 1 / t) with t = *step_p.  w == 1 (the first step)
// stores x itself: fmaf(1, x - a, a) would round x - a.  Purely elementwise, so every element sees
// the same arithmetic whatever the grid.
__device__ __forceinline__ float ema_update(float a, float x, float w) { return w == 1.f ? x : fmaf(w, x - a, a); }

__global__ void __launch_bounds__(kOptThreads) weight_ema_kernel(float *__restrict__ avg, const float *__restrict__ state, int64_t n,
                                                                 const int64_t *__restrict__ step_p, float decay, int seeded) {
    const float keep = 1.f - decay;
    const int64_t t = *step_p;
    const float w = seeded ? keep : fmaxf(keep, 1.f / (float)(t > 1 ? t : 1));
    const int64_t n4 = n >> 2;
    float4 *a4 = reinterpret_cast<float4 *>(avg);
    const float4 *x4 = reinterpret_cast<const float4 *>(state);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 a = a4[i];
        const float4 x = x4[i];
        a.x = ema_update(a.x, x.x, w);
        a.y = ema_update(a.y, x.y, w);
        a.z = ema_update(a.z, x.z, w);
        a.w = ema_update(a.w, x.w, w);
        a4[i] = a;
    }
    if (blockIdx.x == 0)
        for (int64_t i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) avg[i] = ema_update(avg[i], state[i], w);
}

}  // namespace hrl

extern "C" int32_t hrl_sumsq_num_partials(void) { return hrl::kPartials; }

extern "C" int hrl_peer_allreduce_sumsq(float *out_sum, const float *const *peer_buckets, int64_t flag_offset, int32_t world,
                                        int32_t rank, int64_t n, int64_t n_norm, float *partials, uint32_t *epoch, uint32_t *ticket,
                                        uint32_t *status, void *stream) {
    using namespace hrl;
    HRL_REQUIRE(out_sum && peer_buckets && partials && epoch && ticket && status, HRL_ERR_BAD_ARG, "hrl_peer_allreduce_sumsq: NULL pointer");
    HRL_REQUIRE(world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world, HRL_ERR_BAD_ARG,
                "hrl_peer_allreduce_sumsq: bad world/rank (%d/%d)", world, rank);
    HRL_REQUIRE(n > 0 && (n & 3) == 0 && (n_norm & 3) == 0 && n_norm <= n && flag_offset >= n, HRL_ERR_BAD_ARG, "hrl_peer_allreduce_sumsq: n must be a positive multiple of 4 and the flags must follow the data");
    // the whole grid must be co-resident (blocks spin on peer flags): 264 blocks x 256 threads (two per SM) always are
    peer_allreduce_sumsq_kernel<<<kPartials, kOptThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        out_sum, peer_buckets, flag_offset, world, rank, n, n_norm, partials, epoch, ticket, status);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_grad_sumsq(const float *grad, int64_t n, float *partials, void *stream) {
    using namespace hrl;
    HRL_REQUIRE(grad && partials && n > 0, HRL_ERR_BAD_ARG, "hrl_grad_sumsq: NULL pointer or n <= 0");
    HRL_REQUIRE((reinterpret_cast<uintptr_t>(grad) & 15) == 0, HRL_ERR_BAD_ARG, "hrl_grad_sumsq: grad must be 16-byte aligned");
    grad_sumsq_kernel<<<kPartials, kOptThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(grad, n, partials);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

namespace hrl {
template <bool DIAG>
static int clip_adam_step(const char *name, float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t n,
                          const float *partials, const float *lr, int64_t *step, double max_norm, double beta1, double beta2,
                          double eps, double weight_decay, float *grad_norm_out, double *diag, void *stream) {
    HRL_REQUIRE(param && grad && exp_avg && exp_avg_sq && partials && lr && step && n > 0, HRL_ERR_BAD_ARG,
                "%s: NULL pointer or n <= 0", name);
    HRL_REQUIRE(!DIAG || diag, HRL_ERR_BAD_ARG, "%s: diag_accum is NULL", name);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    int grid = (int)((n + kOptThreads - 1) / kOptThreads);
    if (grid > kPartials) grid = kPartials;
    clip_adam_kernel<DIAG><<<grid, kOptThreads, 0, s>>>(param, grad, exp_avg, exp_avg_sq, n, partials, lr, step, max_norm,
                                                        beta1, beta2, eps, weight_decay, grad_norm_out, diag);
    HRL_CUDA_CHECK(cudaGetLastError());
    bump_step_kernel<<<1, 1, 0, s>>>(step);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}
}  // namespace hrl

extern "C" int hrl_clip_adam_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t n,
                                  const float *partials, const float *lr, int64_t *step, double max_norm, double beta1,
                                  double beta2, double eps, double weight_decay, float *grad_norm_out, void *stream) {
    return hrl::clip_adam_step<false>("hrl_clip_adam_step", param, grad, exp_avg, exp_avg_sq, n, partials, lr, step, max_norm,
                                      beta1, beta2, eps, weight_decay, grad_norm_out, nullptr, stream);
}

extern "C" int hrl_clip_adam_step_diag(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t n,
                                       const float *partials, const float *lr, int64_t *step, double max_norm, double beta1,
                                       double beta2, double eps, double weight_decay, float *grad_norm_out, double *diag_accum,
                                       void *stream) {
    return hrl::clip_adam_step<true>("hrl_clip_adam_step_diag", param, grad, exp_avg, exp_avg_sq, n, partials, lr, step,
                                     max_norm, beta1, beta2, eps, weight_decay, grad_norm_out, diag_accum, stream);
}

extern "C" int hrl_weight_ema(float *avg, const float *state, int64_t n, const int64_t *step, float decay, int32_t seeded,
                              void *stream) {
    using namespace hrl;
    HRL_REQUIRE(avg && state && step && n > 0, HRL_ERR_BAD_ARG, "hrl_weight_ema: NULL pointer or n <= 0");
    HRL_REQUIRE(((reinterpret_cast<uintptr_t>(avg) | reinterpret_cast<uintptr_t>(state)) & 15) == 0, HRL_ERR_BAD_ARG,
                "hrl_weight_ema: avg and state must be 16-byte aligned");
    HRL_REQUIRE(decay > 0.f && decay < 1.f, HRL_ERR_BAD_ARG, "hrl_weight_ema: decay must lie in (0, 1), got %g", (double)decay);
    const int64_t n4 = n >> 2;
    int64_t grid = (n4 + kOptThreads - 1) / kOptThreads;
    if (grid < 1) grid = 1;                     // n < 4: block 0 does the tail alone
    if (grid > 4 * kNumSM) grid = 4 * kNumSM;
    weight_ema_kernel<<<(int)grid, kOptThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(avg, state, n, step, decay,
                                                                                             seeded ? 1 : 0);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}
