// K3 -- clip_grad_norm_(4.0) + Adam(weight_decay) on one flat fp32 bucket
// (handyrl/train.py:370-371 with the optimiser of train.py:331).
//
// Two launches so that the global norm is a true grid-wide reduction without cooperative
// launch: hrl_grad_sumsq writes kPartials block partials (fixed grid => fixed summation order
// => bit-reproducible), hrl_clip_adam_step has every block fold those partials itself and
// then update its slice.  lr and the step counter are read from device memory so a captured
// CUDA graph keeps working while the host changes the learning rate (train.py:383-384).
#include "optim_common.cuh"

namespace hrl {

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
// GUARD: the step is rejected when the fp64 fold of the partials or one of tail[0..n_tail) is not finite.  Every block
// folds the same partials in the same order and reads the same tail, so every block reaches the same decision on its
// own; a rejected step writes neither param, the moments nor diag.  Block 0 writes the decision to *skip.
template <bool DIAG, bool GUARD>
__global__ void __launch_bounds__(kOptThreads) clip_adam_kernel(
    float *__restrict__ param, const float *__restrict__ grad, float *__restrict__ exp_avg,
    float *__restrict__ exp_avg_sq, int64_t n, const float *__restrict__ partials, const float *__restrict__ lr_p,
    int64_t *step_p, double max_norm_d, double beta1_d, double beta2_d, double eps_d, double wd_d,
    float *grad_norm_out, double *diag, const float *__restrict__ tail, int n_tail, int32_t *skip) {
    // every block folds the partial sums in the same order -> identical clip coefficient everywhere
    float coef;
    bool reject;
    clip_prologue<DIAG, GUARD>(partials, (float)max_norm_d, grad_norm_out, diag, tail, n_tail, skip, coef, reject);
    if (reject) return;
    const AdamConsts a = adam_consts(lr_p, step_p, beta1_d, beta2_d, eps_d, wd_d);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        adam_word(param, grad, exp_avg, exp_avg_sq, i, coef, a);
}

// ---- LAMB (You et al., 2020, Algorithm 2) on the same bucket: Adam's moments, one trust ratio per parameter tensor --------
// The bucket is cut into chunks of at most kLambChunk words that never cross a tensor (hrl_lamb_plan); block c of both
// launches owns chunk c.  Launch A updates the moments, writes the update direction u to a scratch bucket and the chunk's
// fp64 sums of w^2 and u^2; launch B folds the sums of its tensor's chunks in a fixed order (so every block of a tensor, every
// replay and every rank gets the same ratio) and applies w -= lr * lr_scale * r * u.
constexpr int kLambChunk = 1024;   // words per chunk: 4 per thread of a kOptThreads block
constexpr int kLambPlanWords = 5;  // int64 per chunk: start, length, tensor, that tensor's first chunk and chunk count

// DIAG, GUARD: as clip_adam_kernel, whose global-norm fold, clip coefficient and guard decision this prologue repeats word
// for word; a rejected step writes neither param, the moments, update, chunk_sums nor diag.
template <bool DIAG, bool GUARD>
__global__ void __launch_bounds__(kOptThreads) clip_lamb_moments_kernel(
    const float *__restrict__ param, const float *__restrict__ grad, float *__restrict__ exp_avg,
    float *__restrict__ exp_avg_sq, float *__restrict__ update, const int64_t *__restrict__ plan, double *__restrict__ chunk_sums,
    const float *__restrict__ partials, const int64_t *step_p, double max_norm_d, double beta1_d, double beta2_d, double eps_d,
    double wd_d, float *grad_norm_out, double *diag, const float *__restrict__ tail, int n_tail, int32_t *skip) {
    const float beta2 = (float)beta2_d, eps = (float)eps_d, wd = (float)wd_d;
    __shared__ double red[kOptThreads / 32];
    float coef;
    bool reject;
    clip_prologue<DIAG, GUARD>(partials, (float)max_norm_d, grad_norm_out, diag, tail, n_tail, skip, coef, reject);
    if (reject) return;
    const int64_t t = *step_p + 1;
    const float bc1 = (float)(1.0 - pow(beta1_d, (double)t));
    const float bc2_sqrt = (float)sqrt(1.0 - pow(beta2_d, (double)t));
    const float omb1 = (float)(1.0 - beta1_d), omb2 = (float)(1.0 - beta2_d);
    const int64_t start = plan[kLambPlanWords * blockIdx.x], len = plan[kLambPlanWords * blockIdx.x + 1];
    double ww = 0.0, uu = 0.0;
    for (int64_t i = start + threadIdx.x; i < start + len; i += blockDim.x) {
        const float p = param[i];
        const float g = grad[i] * coef;              // no wd * p here: LAMB adds the decay to the update direction
        float m = exp_avg[i], v = exp_avg_sq[i];
        m = m + (g - m) * omb1;
        v = v * beta2 + omb2 * g * g;
        const float u = (m / bc1) / (sqrtf(v) / bc2_sqrt + eps) + wd * p;
        exp_avg[i] = m;
        exp_avg_sq[i] = v;
        update[i] = u;
        ww += (double)p * (double)p;
        uu += (double)u * (double)u;
    }
    ww = block_sum_d(ww, red);
    uu = block_sum_d(uu, red);
    if (threadIdx.x == 0) {
        chunk_sums[2 * blockIdx.x] = ww;
        chunk_sums[2 * blockIdx.x + 1] = uu;
    }
}

// GUARD: nothing happens when *skip says launch A rejected the step.  ratio (may be NULL): r of tensor i -> ratio[i].
template <bool GUARD>
__global__ void __launch_bounds__(kOptThreads) lamb_apply_kernel(float *__restrict__ param, const float *__restrict__ update,
                                                                 const int64_t *__restrict__ plan,
                                                                 const double *__restrict__ chunk_sums, const float *__restrict__ lr_p,
                                                                 double lr_scale, float *ratio, const int32_t *skip) {
    if (GUARD && *skip) return;
    const int64_t *me = plan + kLambPlanWords * blockIdx.x;
    const int64_t start = me[0], len = me[1], tensor = me[2], first = me[3], count = me[4];
    __shared__ double red[kOptThreads / 32];
    __shared__ float s_step;
    double ww = 0.0, uu = 0.0;          // thread t: chunks first + t, first + t + blockDim.x, ... -- the same split in every block
    for (int64_t j = first + threadIdx.x; j < first + count; j += blockDim.x) {
        ww += chunk_sums[2 * j];
        uu += chunk_sums[2 * j + 1];
    }
    ww = block_sum_d(ww, red);
    uu = block_sum_d(uu, red);
    if (threadIdx.x == 0) {
        const double r = (ww > 0.0 && uu > 0.0) ? sqrt(ww) / sqrt(uu) : 1.0;
        s_step = (float)((double)*lr_p * lr_scale * r);
        if (ratio && blockIdx.x == first) ratio[tensor] = (float)r;
    }
    __syncthreads();
    const float step = s_step;
    for (int64_t i = start + threadIdx.x; i < start + len; i += blockDim.x) param[i] = param[i] - step * update[i];
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
// guarded form: a rejected step is not counted
__global__ void bump_step_guarded_kernel(int64_t *step_p, const int32_t *skip) { *step_p += *skip ? 0 : 1; }

int launch_bump_step(int64_t *step, const int32_t *skip, cudaStream_t stream) {
    if (skip)
        bump_step_guarded_kernel<<<1, 1, 0, stream>>>(step, skip);
    else
        bump_step_kernel<<<1, 1, 0, stream>>>(step);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

// After a guarded optimiser step.  Accepted: accum[i] += (double)tail[i], i < n_tail (one rounding, as ATen's fp64 add_
// of an fp32 tensor).  Rejected: *skip_count += 1, and the saved bytes go back to `state` (the buffers the forward moved).
__global__ void __launch_bounds__(kOptThreads) step_commit_kernel(const int32_t *__restrict__ skip, const float *__restrict__ tail,
                                                                  int n_tail, double *__restrict__ accum, double *__restrict__ skip_count,
                                                                  uint8_t *__restrict__ state, const uint8_t *__restrict__ saved,
                                                                  int64_t nbytes) {
    if (*skip == 0) {
        if (blockIdx.x == 0)
            for (int i = threadIdx.x; i < n_tail; i += blockDim.x) accum[i] = accum[i] + (double)tail[i];
        return;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *skip_count += 1.0;
    const int64_t n16 = nbytes >> 4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (int64_t)gridDim.x * blockDim.x)
        reinterpret_cast<uint4 *>(state)[i] = reinterpret_cast<const uint4 *>(saved)[i];
    if (blockIdx.x == 0)
        for (int64_t i = (n16 << 4) + threadIdx.x; i < nbytes; i += blockDim.x) state[i] = saved[i];
}

// the loss-pass sums of a gradient-accumulation step: out[j] = fp32(sum over rows i = 0..k-1, in order, of (double)rows[i*ld + j])
__global__ void sum_rows_kernel(const float *__restrict__ rows, int k, int64_t ld, int n, float *__restrict__ out) {
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        double s = 0.0;
        for (int i = 0; i < k; i++) s += (double)rows[(int64_t)i * ld + j];
        out[j] = (float)s;
    }
}

// moving average of the learner's state after the optimiser step: a <- fmaf(w, x - a, a),
// w = 1 - decay once seeded, else max(1 - decay, 1 / t) with t = *step_p.  w == 1 (the first step)
// stores x itself: fmaf(1, x - a, a) would round x - a.  Purely elementwise, so every element sees
// the same arithmetic whatever the grid.
__device__ __forceinline__ float ema_update(float a, float x, float w) { return w == 1.f ? x : fmaf(w, x - a, a); }

// GUARD: nothing happens when *skip says the optimiser step was rejected
template <bool GUARD>
__global__ void __launch_bounds__(kOptThreads) weight_ema_kernel(float *__restrict__ avg, const float *__restrict__ state, int64_t n,
                                                                 const int64_t *__restrict__ step_p, float decay, int seeded,
                                                                 const int32_t *__restrict__ skip) {
    if (GUARD && *skip) return;
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

extern "C" int hrl_clip_adam_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t n,
                                  const float *partials, const float *lr, int64_t *step, double max_norm, double beta1,
                                  double beta2, double eps, double weight_decay, float *grad_norm_out, double *diag_accum,
                                  const float *tail, int32_t n_tail, int32_t *skip, void *stream) {
    using namespace hrl;
    HRL_REQUIRE(param && grad && exp_avg && exp_avg_sq && partials && lr && step && n > 0, HRL_ERR_BAD_ARG,
                "hrl_clip_adam_step: NULL pointer or n <= 0");
    HRL_REQUIRE(!skip || (n_tail >= 0 && (tail || n_tail == 0)), HRL_ERR_BAD_ARG,
                "hrl_clip_adam_step: tail is NULL with n_tail > 0, or n_tail < 0");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    int grid = (int)((n + kOptThreads - 1) / kOptThreads);
    if (grid > kPartials) grid = kPartials;
    auto kernel = diag_accum ? (skip ? clip_adam_kernel<true, true> : clip_adam_kernel<true, false>)
                             : (skip ? clip_adam_kernel<false, true> : clip_adam_kernel<false, false>);
    kernel<<<grid, kOptThreads, 0, s>>>(param, grad, exp_avg, exp_avg_sq, n, partials, lr, step, max_norm, beta1, beta2, eps,
                                        weight_decay, grad_norm_out, diag_accum, tail, n_tail, skip);
    HRL_CUDA_CHECK(cudaGetLastError());
    return launch_bump_step(step, skip, s);
}

extern "C" int64_t hrl_lamb_plan(const int64_t *numel, int32_t n_tensors, int64_t *plan) {
    using namespace hrl;
    HRL_REQUIRE(numel && n_tensors > 0, HRL_ERR_BAD_ARG, "hrl_lamb_plan: numel is NULL or n_tensors <= 0");
    int64_t chunks = 0, off = 0;
    for (int32_t i = 0; i < n_tensors; i++) {
        HRL_REQUIRE(numel[i] > 0, HRL_ERR_BAD_ARG, "hrl_lamb_plan: tensor %d has %lld words", i, (long long)numel[i]);
        const int64_t first = chunks, count = (numel[i] + kLambChunk - 1) / kLambChunk;
        for (int64_t s = 0; s < numel[i]; s += kLambChunk, chunks++) {
            if (plan) {
                int64_t *c = plan + kLambPlanWords * chunks;
                c[0] = off + s;
                c[1] = numel[i] - s < kLambChunk ? numel[i] - s : kLambChunk;
                c[2] = i;
                c[3] = first;
                c[4] = count;
            }
        }
        off += numel[i];
    }
    HRL_REQUIRE(chunks <= INT32_MAX, HRL_ERR_UNSUPPORTED, "hrl_lamb_plan: %lld chunks", (long long)chunks);
    return chunks;
}

extern "C" int hrl_clip_lamb_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, float *update, int64_t n,
                                  const int64_t *plan, int32_t n_chunks, double *chunk_sums, const float *partials, const float *lr,
                                  int64_t *step, double max_norm, double beta1, double beta2, double eps, double weight_decay,
                                  double lr_scale, float *grad_norm_out, double *diag_accum, const float *tail, int32_t n_tail,
                                  int32_t *skip, float *ratio, void *stream) {
    using namespace hrl;
    HRL_REQUIRE(param && grad && exp_avg && exp_avg_sq && update && plan && chunk_sums && partials && lr && step && n > 0 &&
                    n_chunks > 0,
                HRL_ERR_BAD_ARG, "hrl_clip_lamb_step: NULL pointer, n <= 0 or n_chunks <= 0");
    HRL_REQUIRE(!skip || (n_tail >= 0 && (tail || n_tail == 0)), HRL_ERR_BAD_ARG,
                "hrl_clip_lamb_step: tail is NULL with n_tail > 0, or n_tail < 0");
    HRL_REQUIRE(lr_scale > 0.0 && isfinite(lr_scale), HRL_ERR_BAD_ARG, "hrl_clip_lamb_step: lr_scale must be finite and > 0, got %g",
                lr_scale);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    auto moments = diag_accum ? (skip ? clip_lamb_moments_kernel<true, true> : clip_lamb_moments_kernel<true, false>)
                              : (skip ? clip_lamb_moments_kernel<false, true> : clip_lamb_moments_kernel<false, false>);
    moments<<<n_chunks, kOptThreads, 0, s>>>(param, grad, exp_avg, exp_avg_sq, update, plan, chunk_sums, partials, step, max_norm,
                                             beta1, beta2, eps, weight_decay, grad_norm_out, diag_accum, tail, n_tail, skip);
    HRL_CUDA_CHECK(cudaGetLastError());
    auto apply = skip ? lamb_apply_kernel<true> : lamb_apply_kernel<false>;
    apply<<<n_chunks, kOptThreads, 0, s>>>(param, update, plan, chunk_sums, lr, lr_scale, ratio, skip);
    HRL_CUDA_CHECK(cudaGetLastError());
    return launch_bump_step(step, skip, s);
}

extern "C" int hrl_step_commit(const int32_t *skip, const float *tail, int32_t n_tail, double *accum, double *skip_count,
                               void *state, const void *saved, int64_t nbytes, void *stream) {
    using namespace hrl;
    HRL_REQUIRE(skip && skip_count && n_tail >= 0 && nbytes >= 0, HRL_ERR_BAD_ARG,
                "hrl_step_commit: skip or skip_count is NULL, or a negative size");
    HRL_REQUIRE(n_tail == 0 || (tail && accum), HRL_ERR_BAD_ARG, "hrl_step_commit: tail or accum is NULL with n_tail > 0");
    HRL_REQUIRE(nbytes == 0 || (state && saved), HRL_ERR_BAD_ARG, "hrl_step_commit: state or saved is NULL with nbytes > 0");
    HRL_REQUIRE(((reinterpret_cast<uintptr_t>(state) | reinterpret_cast<uintptr_t>(saved)) & 15) == 0, HRL_ERR_BAD_ARG,
                "hrl_step_commit: state and saved must be 16-byte aligned");
    int64_t grid = ((nbytes >> 4) + kOptThreads - 1) / kOptThreads;
    if (grid < 1) grid = 1;
    if (grid > 4 * kNumSM) grid = 4 * kNumSM;
    step_commit_kernel<<<(int)grid, kOptThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        skip, tail, n_tail, accum, skip_count, static_cast<uint8_t *>(state), static_cast<const uint8_t *>(saved), nbytes);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_weight_ema(float *avg, const float *state, int64_t n, const int64_t *step, float decay, int32_t seeded,
                              const int32_t *skip, void *stream) {
    using namespace hrl;
    HRL_REQUIRE(avg && state && step && n > 0, HRL_ERR_BAD_ARG, "hrl_weight_ema: NULL pointer or n <= 0");
    HRL_REQUIRE(((reinterpret_cast<uintptr_t>(avg) | reinterpret_cast<uintptr_t>(state)) & 15) == 0, HRL_ERR_BAD_ARG,
                "hrl_weight_ema: avg and state must be 16-byte aligned");
    HRL_REQUIRE(decay > 0.f && decay < 1.f, HRL_ERR_BAD_ARG, "hrl_weight_ema: decay must lie in (0, 1), got %g", (double)decay);
    const int64_t n4 = n >> 2;
    int64_t grid = (n4 + kOptThreads - 1) / kOptThreads;
    if (grid < 1) grid = 1;                     // n < 4: block 0 does the tail alone
    if (grid > 4 * kNumSM) grid = 4 * kNumSM;
    auto kernel = skip ? weight_ema_kernel<true> : weight_ema_kernel<false>;
    kernel<<<(int)grid, kOptThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(avg, state, n, step, decay, seeded ? 1 : 0,
                                                                                  skip);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_sum_rows(const float *rows, int32_t k, int64_t ld, int32_t n, float *out, void *stream) {
    HRL_REQUIRE(rows && out && k >= 1 && n >= 1 && ld >= n, HRL_ERR_BAD_ARG, "hrl_sum_rows: NULL pointer or bad shape");
    hrl::sum_rows_kernel<<<1, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(rows, k, ld, n, out);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}
