// Shared helpers for the sm_90a kernels of the HandyRL learner hot path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/hrl_b200.h"

namespace hrl {

void set_error(const char *fmt, ...);

#define HRL_CUDA_CHECK(expr)                                                              \
    do {                                                                                  \
        cudaError_t err__ = (expr);                                                       \
        if (err__ != cudaSuccess) {                                                       \
            hrl::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(err__),     \
                           __FILE__, __LINE__);                                           \
            return HRL_ERR_CUDA;                                                          \
        }                                                                                 \
    } while (0)

#define HRL_REQUIRE(cond, code, ...)        \
    do {                                    \
        if (!(cond)) {                      \
            hrl::set_error(__VA_ARGS__);    \
            return (code);                  \
        }                                   \
    } while (0)

constexpr int kNumSM = 132;  // H100 SXM

// reductions over a power-of-two group of W adjacent lanes (W <= 32)
template <int W>
__device__ __forceinline__ float group_max(float v) {
#pragma unroll
    for (int o = W / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o, W));
    return v;
}
template <int W>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
    for (int o = W / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, W);
    return v;
}
__device__ __forceinline__ float warp_sum(float v) { return group_sum<32>(v); }
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// the 3xTF32 split: hi = v with the 13 low mantissa bits cleared (exactly a TF32 number), lo = v - hi (exact)
__device__ __forceinline__ void split_tf32(float v, float &hi, float &lo) {
    hi = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
    lo = v - hi;
}

// streaming global accesses: data touched exactly once should not displace L1 lines
__device__ __forceinline__ float ld_stream(const float *p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream(float *p, float v) { __stcs(p, v); }

// asynchronous 16-byte global -> shared copies (cp.async.cg: L2 only), one commit group per call of cp_async_commit
__device__ __forceinline__ void cp_async16(uint32_t dst, const float *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

}  // namespace hrl
