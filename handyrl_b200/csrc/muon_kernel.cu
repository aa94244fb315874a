// clip_grad_norm_ + Muon on the flat fp32 bucket (opt-in; no reference counterpart): each weight matrix's Nesterov
// momentum is orthogonalised by five Newton-Schulz iterations on bf16 tensor-core products, the other words take Adam.
//
// One launch after hrl_grad_sumsq.  Block b < n_mats owns matrix b of the host plan (hrl_muon_plan) and does its whole
// step in one CTA: the clip prologue of clip_adam_kernel, the momentum, X0 = N / (|N|_F + 1e-7) into shared memory as bf16
// (m x n with m <= n, transposed when the matrix is tall), then five times
//     A = X X^T;  B = b A + c A A;  X = a X + B X
// with mma.sync m16n8k16 (bf16 operands rounded to nearest even, fp32 accumulation), and the weight update.  A and B are
// symmetric, so only their 16 x 16 blocks on and above the diagonal are computed and each is mirrored below: both are
// exactly symmetric in bf16, and A A is A A^T.  X is updated in place one 8-column panel per warp: a column panel of
// B X needs only the same panel of X, which the warp reads in full before it writes.  Blocks b >= n_mats each take one
// span of Adam-owned words with hrl_clip_adam_step's arithmetic (adam_word).  No atomics and fixed-order reductions: every
// launch, graph replay and rank gives the same bits.
#include <cuda_bf16.h>

#include "optim_common.cuh"

namespace hrl {

typedef __nv_bfloat16 bf16;

// The one-CTA envelope: the smaller side m and the larger n, each padded to 16, with m_p <= 128 and m_p * n_p <= 128 * 576
// (Geister's ConvLSTM gates, the largest matrix of the shipped nets).  Shared memory: X (m_p rows of n_p + 8 bf16), A and B
// (m_p rows of m_p + 8 bf16 each); the 8 extra bf16 per row put the rows of a fragment load in different banks.
constexpr int kMuonMaxSide = 128;
constexpr int kMuonMaxElems = 128 * 576;
constexpr int kMuonRowPad = 8;
constexpr int kMuonSmemBytes =
    (int)sizeof(bf16) * (kMuonMaxElems + kMuonRowPad * kMuonMaxSide + 2 * kMuonMaxSide * (kMuonMaxSide + kMuonRowPad));
static_assert(kMuonSmemBytes + 1024 <= 227 * 1024, "Muon's envelope does not fit one CTA's shared memory");
constexpr int kMuonMatWords = 4;    // int64 per matrix of the plan: first word, r, k, transposed
constexpr int kMuonSpanWords = 2;   // int64 per Adam span: first word, words
constexpr int kMuonSpan = 4096;     // words per Adam span at most: 16 per thread
constexpr int kWarps = kOptThreads / 32;

constexpr float kMuonMu = 0.95f;
constexpr float kNsA = 3.4445f, kNsB = -4.7750f, kNsC = 2.0315f;

__device__ __forceinline__ int pad16(int x) { return (x + 15) & ~15; }

__device__ __forceinline__ uint32_t ld_pair(const bf16 *p) { return *reinterpret_cast<const uint32_t *>(p); }
__device__ __forceinline__ uint32_t pack_pair(bf16 lo, bf16 hi) {
    return (uint32_t)__bfloat16_as_ushort(lo) | ((uint32_t)__bfloat16_as_ushort(hi) << 16);
}

// D[16 x 8] += A[16 x 16] B[16 x 8], bf16 operands, fp32 accumulators
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// the A fragment of rows r0..r0+15, columns k0..k0+15 of a row-major bf16 matrix S (stride ss)
__device__ __forceinline__ void frag_a(uint32_t (&a)[4], const bf16 *S, int ss, int r0, int k0, int g, int q) {
    const bf16 *p = S + (r0 + g) * ss + k0 + 2 * q;
    a[0] = ld_pair(p);
    a[1] = ld_pair(p + 8 * ss);
    a[2] = ld_pair(p + 8);
    a[3] = ld_pair(p + 8 * ss + 8);
}

// D <- bf16(e_coef * E + S S^T) over m_p x m_p, S m_p x kdim (stride ss).  E (stride sd, may be NULL: D <- bf16(S S^T)) is
// symmetric.  Each warp takes 16 x 16 blocks (bi <= bj) in turn and writes every element of the upper triangle to (i, j)
// and (j, i).
__device__ __forceinline__ void sym_product(const bf16 *S, int ss, int kdim, int mp, bf16 *D, int sd, const bf16 *E, float e_coef,
                                            float c_coef) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const int nb = mp >> 4;
    for (int blk = warp; blk < nb * (nb + 1) / 2; blk += kWarps) {
        int bi = 0, rem = blk;
        while (rem >= nb - bi) {
            rem -= nb - bi;
            bi++;
        }
        const int bj = bi + rem;
        float acc[2][4] = {};
        for (int k0 = 0; k0 < kdim; k0 += 16) {
            uint32_t a[4];
            frag_a(a, S, ss, 16 * bi, k0, g, q);
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const bf16 *p = S + (16 * bj + 8 * h + g) * ss + k0 + 2 * q;
                const uint32_t b[2] = {ld_pair(p), ld_pair(p + 8)};
                mma_bf16(acc[h], a, b);
            }
        }
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int i = 16 * bi + g + (e >= 2 ? 8 : 0), j = 16 * bj + 8 * h + 2 * q + (e & 1);
                if (bi == bj && i > j) continue;
                float v = acc[h][e];
                if (E) v = __fadd_rn(__fmul_rn(e_coef, __bfloat162float(E[i * sd + j])), __fmul_rn(c_coef, v));
                const bf16 r = __float2bfloat16_rn(v);
                D[i * sd + j] = r;
                D[j * sd + i] = r;
            }
    }
}

// X <- bf16(a X + B X) in place, X m_p x n_p (stride sx), B m_p x m_p (stride sb): warp w owns the 8-column panels
// w, w + kWarps, ...; it reads the whole panel (all m_p rows) into its accumulators before it writes any of it
__device__ __forceinline__ void ns_update(bf16 *X, int sx, int mp, int np, const bf16 *B, int sb) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const int mt = mp >> 4;
    for (int c0 = 8 * warp; c0 < np; c0 += 8 * kWarps) {
        float acc[kMuonMaxSide / 16][4] = {};
        for (int k0 = 0; k0 < mp; k0 += 16) {
            const bf16 *p = X + (k0 + 2 * q) * sx + c0 + g;       // B operand: X[k0 + k][c0 + n]
            const uint32_t b[2] = {pack_pair(p[0], p[sx]), pack_pair(p[8 * sx], p[9 * sx])};
#pragma unroll
            for (int t = 0; t < kMuonMaxSide / 16; t++)
                if (t < mt) {
                    uint32_t a[4];
                    frag_a(a, B, sb, 16 * t, k0, g, q);
                    mma_bf16(acc[t], a, b);
                }
        }
#pragma unroll
        for (int t = 0; t < kMuonMaxSide / 16; t++)
            if (t < mt)
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int i = 16 * t + g + (e >= 2 ? 8 : 0), j = c0 + 2 * q + (e & 1);
                    acc[t][e] = __fadd_rn(__fmul_rn(kNsA, __bfloat162float(X[i * sx + j])), acc[t][e]);
                }
        __syncwarp();
#pragma unroll
        for (int t = 0; t < kMuonMaxSide / 16; t++)
            if (t < mt)
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int i = 16 * t + g + (e >= 2 ? 8 : 0), j = c0 + 2 * q + (e & 1);
                    X[i * sx + j] = __float2bfloat16_rn(acc[t][e]);
                }
    }
}

// M <- mu M + g;  N <- g + mu M  (g the clipped gradient word; two roundings each, no contraction)
__device__ __forceinline__ float nesterov(float g, float m_old, float &m_new) {
    m_new = __fadd_rn(__fmul_rn(kMuonMu, m_old), g);
    return __fadd_rn(g, __fmul_rn(kMuonMu, m_new));
}

// DIAG, GUARD: as clip_adam_kernel; a rejected step writes neither param, the moments, ortho nor diag.
template <bool DIAG, bool GUARD>
__global__ void __launch_bounds__(kOptThreads, 1) clip_muon_kernel(
    float *__restrict__ param, const float *__restrict__ grad, float *__restrict__ exp_avg, float *__restrict__ exp_avg_sq,
    const int64_t *__restrict__ mats, int n_mats, const int64_t *__restrict__ spans, const float *__restrict__ partials,
    const float *__restrict__ lr_p, const int64_t *step_p, double max_norm_d, double beta1_d, double beta2_d, double eps_d,
    double wd_d, double lr_scale, float *grad_norm_out, double *diag, const float *__restrict__ tail, int n_tail, int32_t *skip,
    float *__restrict__ ortho) {
    float coef;
    bool reject;
    clip_prologue<DIAG, GUARD>(partials, (float)max_norm_d, grad_norm_out, diag, tail, n_tail, skip, coef, reject);
    if (reject) return;
    if ((int)blockIdx.x >= n_mats) {
        const int64_t *sp = spans + kMuonSpanWords * (blockIdx.x - n_mats);
        const AdamConsts a = adam_consts(lr_p, step_p, beta1_d, beta2_d, eps_d, wd_d);
        for (int64_t i = sp[0] + threadIdx.x; i < sp[0] + sp[1]; i += blockDim.x) adam_word(param, grad, exp_avg, exp_avg_sq, i, coef, a);
        return;
    }
    extern __shared__ __align__(16) uint8_t muon_smem[];
    __shared__ double red[kWarps];
    const int64_t *me = mats + kMuonMatWords * blockIdx.x;
    const int64_t off = me[0];
    const int r = (int)me[1], k = (int)me[2], words = r * k;
    const bool tr = me[3] != 0;
    const int mp = pad16(tr ? k : r), np = pad16(tr ? r : k), sx = np + kMuonRowPad, sa = mp + kMuonRowPad;
    bf16 *X = reinterpret_cast<bf16 *>(muon_smem), *A = X + mp * sx, *B = A + mp * sa;
    // the padding of X stays zero through the iterations: A, B and B X have zero rows and columns there
    for (int i = threadIdx.x; i < mp * sx / 2; i += blockDim.x) reinterpret_cast<uint32_t *>(X)[i] = 0u;
    double ss = 0.0;
    for (int i = threadIdx.x; i < words; i += blockDim.x) {
        float m;
        const float nv = nesterov(grad[off + i] * coef, exp_avg[off + i], m);
        ss += (double)nv * (double)nv;
    }
    ss = block_sum_d(ss, red);
    const float inv = (float)(1.0 / (sqrt(ss) + 1e-7));
    for (int i = threadIdx.x; i < words; i += blockDim.x) {
        float m;
        const float nv = nesterov(grad[off + i] * coef, exp_avg[off + i], m);
        exp_avg[off + i] = m;
        const int row = i / k, col = i - row * k;
        X[tr ? col * sx + row : row * sx + col] = __float2bfloat16_rn(nv * inv);
    }
    __syncthreads();
    for (int it = 0; it < 5; it++) {
        sym_product(X, sx, np, mp, A, sa, nullptr, 0.f, 1.f);
        __syncthreads();
        sym_product(A, sa, mp, mp, B, sa, A, kNsB, kNsC);
        __syncthreads();
        ns_update(X, sx, mp, np, B, sa);
        __syncthreads();
    }
    const float lr = *lr_p, wd = (float)wd_d;
    const float scale = (float)(lr_scale * 0.2 * sqrt((double)(r > k ? r : k)));
    for (int i = threadIdx.x; i < words; i += blockDim.x) {
        const int row = i / k, col = i - row * k;
        const float o = __bfloat162float(X[tr ? col * sx + row : row * sx + col]);
        if (ortho) ortho[off + i] = o;
        const float p = param[off + i];
        param[off + i] = __fsub_rn(p, __fmul_rn(lr, __fadd_rn(__fmul_rn(scale, o), __fmul_rn(wd, p))));
    }
}

}  // namespace hrl

extern "C" int hrl_muon_plan(const int64_t *dims, const int32_t *ndim, int32_t n_tensors, int32_t *kind, int32_t *counts,
                             int64_t *mats, int64_t *spans) {
    using namespace hrl;
    HRL_REQUIRE(dims && ndim && kind && counts && n_tensors > 0, HRL_ERR_BAD_ARG,
                "hrl_muon_plan: dims, ndim, kind or counts is NULL, or n_tensors <= 0");
    int64_t off = 0, run = -1, n_mats = 0, n_spans = 0;       // run: the first word of the Adam-owned words not yet in a span
    const int64_t *d = dims;
    auto close_run = [&](int64_t end) {
        for (int64_t s = run; run >= 0 && s < end; s += kMuonSpan, n_spans++)
            if (spans) {
                spans[kMuonSpanWords * n_spans] = s;
                spans[kMuonSpanWords * n_spans + 1] = end - s < kMuonSpan ? end - s : kMuonSpan;
            }
        run = -1;
    };
    for (int32_t t = 0; t < n_tensors; t++) {
        HRL_REQUIRE(ndim[t] >= 0, HRL_ERR_BAD_ARG, "hrl_muon_plan: tensor %d has %d dimensions", t, ndim[t]);
        int64_t numel = 1;
        for (int32_t j = 0; j < ndim[t]; j++) {
            HRL_REQUIRE(d[j] > 0, HRL_ERR_BAD_ARG, "hrl_muon_plan: tensor %d has an empty dimension", t);
            numel *= d[j];
        }
        const int64_t r = ndim[t] >= 2 ? d[0] : 1, k = numel / r;
        const int64_t m = r < k ? r : k, n = r < k ? k : r;
        const int64_t mp = (m + 15) / 16 * 16, np = (n + 15) / 16 * 16;
        kind[t] = HRL_MUON_ADAM;
        if (ndim[t] >= 2 && m >= 2) kind[t] = mp <= kMuonMaxSide && mp * np <= kMuonMaxElems ? HRL_MUON_MATRIX : HRL_MUON_TOO_LARGE;
        if (kind[t] == HRL_MUON_MATRIX) {
            close_run(off);
            if (mats) {
                int64_t *e = mats + kMuonMatWords * n_mats;
                e[0] = off;
                e[1] = r;
                e[2] = k;
                e[3] = r > k ? 1 : 0;
            }
            n_mats++;
        } else if (run < 0) {
            run = off;
        }
        off += numel;
        d += ndim[t];
    }
    close_run(off);
    HRL_REQUIRE(n_mats + n_spans <= INT32_MAX, HRL_ERR_UNSUPPORTED, "hrl_muon_plan: %lld blocks", (long long)(n_mats + n_spans));
    counts[0] = (int32_t)n_mats;
    counts[1] = (int32_t)n_spans;
    return HRL_OK;
}

extern "C" int hrl_clip_muon_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t n,
                                  const int64_t *mats, int32_t n_mats, const int64_t *spans, int32_t n_spans,
                                  const float *partials, const float *lr, int64_t *step, double max_norm, double beta1,
                                  double beta2, double eps, double weight_decay, double lr_scale, float *grad_norm_out,
                                  double *diag_accum, const float *tail, int32_t n_tail, int32_t *skip, float *ortho,
                                  void *stream) {
    using namespace hrl;
    HRL_REQUIRE(param && grad && exp_avg && exp_avg_sq && partials && lr && step && n > 0 && n_mats >= 0 && n_spans >= 0 &&
                    n_mats + n_spans > 0 && (mats || n_mats == 0) && (spans || n_spans == 0),
                HRL_ERR_BAD_ARG, "hrl_clip_muon_step: NULL pointer, n <= 0 or an empty plan");
    HRL_REQUIRE(!skip || (n_tail >= 0 && (tail || n_tail == 0)), HRL_ERR_BAD_ARG,
                "hrl_clip_muon_step: tail is NULL with n_tail > 0, or n_tail < 0");
    HRL_REQUIRE(lr_scale > 0.0 && isfinite(lr_scale), HRL_ERR_BAD_ARG, "hrl_clip_muon_step: lr_scale must be finite and > 0, got %g",
                lr_scale);
    static void (*const kernels[4])(float *, const float *, float *, float *, const int64_t *, int, const int64_t *,
                                    const float *, const float *, const int64_t *, double, double, double, double, double,
                                    double, float *, double *, const float *, int, int32_t *, float *) = {
        clip_muon_kernel<false, false>, clip_muon_kernel<false, true>, clip_muon_kernel<true, false>, clip_muon_kernel<true, true>};
    static uint64_t attribute_set = 0;          // one bit per device: the dynamic shared-memory limit is set once
    int dev = 0;
    HRL_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 64 || !((attribute_set >> dev) & 1u)) {
        for (auto kern : kernels)
            HRL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMuonSmemBytes));
        if (dev < 64) attribute_set |= 1ull << dev;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    kernels[(diag_accum ? 2 : 0) + (skip ? 1 : 0)]<<<n_mats + n_spans, kOptThreads, n_mats ? kMuonSmemBytes : 0, s>>>(
        param, grad, exp_avg, exp_avg_sq, mats, n_mats, spans, partials, lr, step, max_norm, beta1, beta2, eps, weight_decay,
        lr_scale, grad_norm_out, diag_accum, tail, n_tail, skip, ortho);
    HRL_CUDA_CHECK(cudaGetLastError());
    return launch_bump_step(step, skip, s);
}
