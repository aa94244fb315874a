// What the optimiser kernels on the flat fp32 bucket share (csrc/optim_kernel.cu: Adam, LAMB; csrc/muon_kernel.cu: Muon):
// the clip + guard prologue that folds hrl_grad_sumsq's partials, Adam's per-word update and a fixed-order block sum.
#pragma once
#include "common.cuh"

namespace hrl {

constexpr int kPartials = 2 * kNumSM;  // 264 blocks: two per SM
constexpr int kOptThreads = 256;

__device__ __forceinline__ double block_sum_d(double x, double *red) {   // fixed order; red: kOptThreads / 32 doubles
    x = warp_sum_d(x);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < kOptThreads / 32; w++) s += red[w];
    __syncthreads();
    return s;
}

// Every block folds the partial sums in the same order -> the same clip coefficient (torch clip_grad_norm_) and, with
// GUARD, the same decision everywhere: the step is rejected when the fp64 fold or one of tail[0..n_tail) is not finite, and
// block 0 writes the decision to *skip.  DIAG: block 0 of an accepted step adds g, g^2, [g > max_norm], 1 to diag[0..3].
// Block 0 writes the pre-clip norm to *grad_norm_out (may be NULL).  Called by every thread of a kOptThreads block.
template <bool DIAG, bool GUARD>
__device__ __forceinline__ void clip_prologue(const float *__restrict__ partials, float max_norm, float *grad_norm_out, double *diag,
                                              const float *__restrict__ tail, int n_tail, int32_t *skip, float &coef, bool &reject) {
    __shared__ double red[kOptThreads / 32];
    __shared__ float s_coef;
    __shared__ int s_reject;
    double acc = 0.0;
    for (int i = threadIdx.x; i < kPartials; i += blockDim.x) acc += (double)partials[i];
    acc = warp_sum_d(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < kOptThreads / 32; w++) s += red[w];
        float total_norm = (float)sqrt(s);
        float c = max_norm / (total_norm + 1e-6f);  // torch clip_grad_norm_
        s_coef = fminf(c, 1.0f);
        if (blockIdx.x == 0 && grad_norm_out) *grad_norm_out = total_norm;
        bool rej = false;
        if (GUARD) {
            rej = !isfinite(s);                      // also a finite gradient whose fp32 sum of squares overflowed
            for (int i = 0; i < n_tail; i++) rej |= !isfinite(tail[i]);
            s_reject = rej ? 1 : 0;
            if (blockIdx.x == 0) *skip = rej ? 1 : 0;
        }
        if (DIAG && blockIdx.x == 0 && !rej) {
            diag[0] += (double)total_norm;
            diag[1] += (double)total_norm * (double)total_norm;
            diag[2] += total_norm > max_norm ? 1.0 : 0.0;
            diag[3] += 1.0;
        }
    }
    __syncthreads();
    coef = s_coef;
    reject = GUARD && s_reject;
}

// Adam's constants for the step that makes the count *step_p + 1, and its update of word i (hrl_clip_adam_step)
struct AdamConsts {
    float step_size, bc2_sqrt, omb1, omb2, beta2, eps, wd;
};

__device__ __forceinline__ AdamConsts adam_consts(const float *__restrict__ lr_p, const int64_t *step_p, double beta1_d,
                                                  double beta2_d, double eps_d, double wd_d) {
    const int64_t t = *step_p + 1;
    const float lr = *lr_p;
    const double bc1 = 1.0 - pow(beta1_d, (double)t);
    const double bc2 = 1.0 - pow(beta2_d, (double)t);
    return {(float)((double)lr / bc1), (float)sqrt(bc2), (float)(1.0 - beta1_d), (float)(1.0 - beta2_d), (float)beta2_d,
            (float)eps_d, (float)wd_d};
}

__device__ __forceinline__ void adam_word(float *__restrict__ param, const float *__restrict__ grad, float *__restrict__ exp_avg,
                                          float *__restrict__ exp_avg_sq, int64_t i, float coef, const AdamConsts &a) {
    float p = param[i];
    float g = grad[i] * coef;
    g = g + a.wd * p;
    float m = exp_avg[i], v = exp_avg_sq[i];
    m = m + (g - m) * a.omb1;
    v = v * a.beta2 + a.omb2 * g * g;
    float denom = sqrtf(v) / a.bc2_sqrt + a.eps;
    param[i] = p - a.step_size * (m / denom);
    exp_avg[i] = m;
    exp_avg_sq[i] = v;
}

// *step += 1 after the step's other launches (every block of the step reads the count before), or with the guard += 0
// when *skip says the step was rejected (csrc/optim_kernel.cu)
int launch_bump_step(int64_t *step, const int32_t *skip, cudaStream_t stream);

}  // namespace hrl
