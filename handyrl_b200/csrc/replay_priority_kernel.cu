// Prioritised replay on the device: the sampler (hrl_replay_sample) and the priority update that ends a step
// (hrl_replay_priority_update).  See include/hrl_b200.h for the law; handyrl_b200/priority.py holds the host references.
//
// Both kernels are one CTA of 1024 threads.  The sampler's work is a prefix sum over at most a few hundred thousand
// directory slots and B binary searches; the update reduces B windows of (T - burn_in) * P cells.  One CTA keeps every sum
// in a fixed order without a second launch or a grid-wide ticket, and both stay off the step's critical bandwidth.
#include "common.cuh"
// Philox4x32-10 of curand's header-only device API (the generator's own header: curand_kernel.h would also pull in
// ~200 KB of precalculated tables of the other generators)
#include <curand_philox4x32_x.h>

namespace hrl {

constexpr int kPrioThreads = 1024;
constexpr int kPrioWarps = kPrioThreads / 32;
constexpr int kMaxPrioBatch = 8192;      // the update keeps one float per window in shared memory

__device__ __forceinline__ double warp_inclusive_scan_d(double v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
    }
    return v;
}

// Block sum of one double per thread: a fixed shuffle tree per warp, then warp 0 adds the warp sums in order.
__device__ __forceinline__ double block_sum_d(double v, double *s_red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum_d(v);
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += s_red[w];
        s_red[32] = s;
    }
    __syncthreads();
    return s_red[32];
}

__global__ void __launch_bounds__(kPrioThreads) replay_sample_kernel(const HrlReplaySampleArgs g) {
    __shared__ double s_red[33];
    __shared__ double s_off[kPrioWarps];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int count = g.count, ring = g.ring;
    const double alpha = (double)g.alpha;
    const float maxp = *g.max_prio;
    double *cdf = g.workspace;

    // ---- 1: weight of episode i = (i+1) * p^alpha, new slots first set to max_prio; inclusive prefix sums in fp64.
    //         Each warp scans a contiguous run of slots 32 at a time (coalesced), then the runs are offset in warp order.
    const int per_warp = (((count + kPrioWarps - 1) / kPrioWarps) + 31) & ~31;
    const int w0 = min(count, warp * per_warp), w1 = min(count, w0 + per_warp);
    double carry = 0.0;
    for (int base = w0; base < w1; base += 32) {
        const int i = base + lane;
        double v = 0.0;
        if (i < w1) {
            const int s = (int)(((int64_t)g.head + i) % ring);
            const int64_t serial = g.dir[(size_t)s * 4 + 3];
            float p;
            if (g.prio_serial[s] != serial) {          // an episode this sampler has not seen: it starts at max_prio
                p = maxp;
                g.prio[s] = p;
                g.prio_serial[s] = serial;
            } else {
                p = g.prio[s];
            }
            v = (double)(i + 1) * pow((double)p, alpha);
        }
        const double incl = warp_inclusive_scan_d(v, lane);
        if (i < w1) cdf[i] = carry + incl;
        carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) s_red[warp] = carry;
    __syncthreads();
    if (tid == 0) {
        double acc = 0.0;
        for (int w = 0; w < kPrioWarps; w++) {
            s_off[w] = acc;
            acc += s_red[w];
        }
    }
    __syncthreads();
    if (warp > 0)
        for (int i = w0 + lane; i < w1; i += 32) cdf[i] += s_off[warp];
    __syncthreads();
    const double total = cdf[count - 1];

    // ---- 2: one Philox block per window: episode (53-bit uniform, binary search), window start, solo player
    const uint2 key = make_uint2((uint32_t)g.seed, (uint32_t)(g.seed >> 32));
    const double nab = -alpha * (double)g.beta;
    double xs = 0.0;
    for (int b = tid; b < g.B; b += kPrioThreads) {
        const uint4 r = curand_Philox4x32_10(make_uint4((uint32_t)b, (uint32_t)g.counter, (uint32_t)(g.counter >> 32), 0u), key);
        const double u = (double)((((uint64_t)r.x) << 21) | (r.y >> 11)) * 0x1p-53 * total;
        int lo = 0, hi = count - 1;               // the first i with cdf[i] > u
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (cdf[mid] > u) hi = mid; else lo = mid + 1;
        }
        const int s = (int)(((int64_t)g.head + lo) % ring);
        const int64_t *d = g.dir + (size_t)s * 4;
        const int steps = (int)d[1];
        const int n = 1 + max(0, steps - g.forward_steps);
        const int ts = (int)(((uint64_t)r.z * (uint64_t)n) >> 32);           // uniform on [0, n)
        HrlWindow w;
        w.first_step = d[0];
        w.train_start = ts;
        w.start = max(0, ts - g.burn_in);
        w.end = min(ts + g.forward_steps, steps);
        w.total = steps;
        w.outcome_row = (int)d[2];
        w.player = g.solo ? (int)(((uint64_t)r.w * (uint64_t)g.Ps) >> 32) : 0;
        g.windows[b] = w;
        g.win_slot[b] = s;
        g.win_serial[b] = d[3];
        xs += pow((double)g.prio[s], nab);
    }

    // ---- 3: importance weights, normalised to mean 1 over the batch
    const double sum = block_sum_d(xs, s_red);
    for (int b = tid; b < g.B; b += kPrioThreads)
        g.win_weight[b] = (float)((double)g.B * pow((double)g.prio[g.win_slot[b]], nab) / sum);
}

__global__ void __launch_bounds__(kPrioThreads) priority_update_kernel(int B, int T, int P, int burn_in, const float *__restrict__ adv,
                                                                      const float *__restrict__ tm, float eps,
                                                                      const int32_t *__restrict__ win_slot,
                                                                      const int64_t *__restrict__ win_serial, float *prio,
                                                                      const int64_t *__restrict__ prio_serial, float *max_prio,
                                                                      const int32_t *skip) {
    if (skip != nullptr && *skip != 0) return;           // a rejected step writes nothing
    __shared__ float s_q[kMaxPrioBatch];
    __shared__ float s_max[kPrioWarps];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = (T - burn_in) * P;

    // q_b = sum(tm |adv|) / sum(tm) + eps over the trained cells, one warp per window (lane-strided sums, fixed tree);
    // -1 marks a window that gives no priority (no trained turn, or a non-finite value)
    for (int b = warp; b < B; b += kPrioWarps) {
        const size_t base = ((size_t)b * T + burn_in) * P;
        float sa = 0.f, st = 0.f;
        for (int j = lane; j < n; j += 32) {
            const float m = tm[base + j];
            sa += m * fabsf(adv[base + j]);
            st += m;
        }
        sa = warp_sum(sa);
        st = warp_sum(st);
        if (lane == 0) {
            const float q = sa / st + eps;
            s_q[b] = (st != 0.f && isfinite(q)) ? q : -1.0f;
        }
    }
    __syncthreads();
    // a slot is written only for the episode its priority belongs to; several windows on one slot resolve to their
    // largest q: the claimed slots are cleared, then take an integer max of the (positive) float bits -- order-free
    for (int b = tid; b < B; b += kPrioThreads) {
        const int64_t serial = win_serial[b];
        if (s_q[b] < 0.f || serial < 0 || prio_serial[win_slot[b]] != serial) s_q[b] = -1.0f;
        else prio[win_slot[b]] = 0.0f;
    }
    __syncthreads();
    float mx = 0.0f;
    for (int b = tid; b < B; b += kPrioThreads) {
        const float q = s_q[b];
        if (q < 0.f) continue;
        atomicMax(reinterpret_cast<int *>(prio + win_slot[b]), __float_as_int(q));
        mx = fmaxf(mx, q);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) s_max[warp] = mx;
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < kPrioWarps; w++) mx = fmaxf(mx, s_max[w]);
        if (mx > *max_prio) *max_prio = mx;
    }
}

}  // namespace hrl

extern "C" int hrl_replay_sample(const HrlReplaySampleArgs *args, void *stream) {
    using namespace hrl;
    HRL_REQUIRE(args != nullptr, HRL_ERR_BAD_ARG, "hrl_replay_sample: args is NULL");
    const HrlReplaySampleArgs &g = *args;
    HRL_REQUIRE(g.B > 0 && g.ring > 1 && g.count >= 1 && g.count < g.ring && g.head >= 0 && g.head < g.ring, HRL_ERR_BAD_ARG,
                "hrl_replay_sample: B=%d ring=%d head=%d count=%d out of range", g.B, g.ring, g.head, g.count);
    HRL_REQUIRE(g.burn_in >= 0 && g.forward_steps > 0 && g.Ps > 0, HRL_ERR_BAD_ARG,
                "hrl_replay_sample: burn_in=%d forward_steps=%d Ps=%d", g.burn_in, g.forward_steps, g.Ps);
    HRL_REQUIRE(g.alpha >= 0.f && g.beta >= 0.f && g.beta <= 1.f, HRL_ERR_BAD_ARG,
                "hrl_replay_sample: alpha=%g beta=%g outside alpha >= 0, 0 <= beta <= 1", (double)g.alpha, (double)g.beta);
    HRL_REQUIRE(g.dir && g.prio && g.prio_serial && g.max_prio && g.workspace && g.windows && g.win_slot && g.win_serial &&
                    g.win_weight, HRL_ERR_BAD_ARG, "hrl_replay_sample: a pointer is NULL");
    replay_sample_kernel<<<1, kPrioThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(g);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_replay_priority_update(int32_t B, int32_t T, int32_t P, int32_t burn_in, const float *tap_advantage,
                                          const float *turn_mask, float epsilon, const int32_t *win_slot, const int64_t *win_serial,
                                          float *prio, const int64_t *prio_serial, float *max_prio, const int32_t *skip,
                                          void *stream) {
    using namespace hrl;
    HRL_REQUIRE(B > 0 && B <= kMaxPrioBatch && T > 0 && P > 0 && burn_in >= 0 && burn_in < T, HRL_ERR_BAD_ARG,
                "hrl_replay_priority_update: B=%d (at most %d) T=%d P=%d burn_in=%d", B, kMaxPrioBatch, T, P, burn_in);
    HRL_REQUIRE(epsilon > 0.f, HRL_ERR_BAD_ARG, "hrl_replay_priority_update: epsilon=%g must be > 0", (double)epsilon);
    HRL_REQUIRE(tap_advantage && turn_mask && win_slot && win_serial && prio && prio_serial && max_prio, HRL_ERR_BAD_ARG,
                "hrl_replay_priority_update: a pointer is NULL");
    priority_update_kernel<<<1, kPrioThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        B, T, P, burn_in, tap_advantage, turn_mask, epsilon, win_slot, win_serial, prio, prio_serial, max_prio, skip);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}
