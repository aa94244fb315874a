// Weight-gradient products on warp-level tensor-core MMAs, operands read as they lie in memory (sm_90a).
//
//   C[M x N] = sum_k A_op[k][m] * B_op[k][n]      A stored [K][M] (a.ld), B stored [K][N] (b.ld), both "MN-major"
//
// The learner's weight gradients reduce over samples, and both operands are activations stored sample-major.  wgmma takes
// tf32 operands K-major only, so the wgmma kernel (gemm_common.cuh) transposes them on their way through registers.  Here
// the fragments of mma.sync.m16n8k8 .tf32 come from registers, and a thread can load them from any shared-memory layout:
//   * staging: every 32-sample chunk is copied raw, [32 samples][tile columns] per source, by 16-byte cp.async into
//     shared memory with rows padded to 104 / 296 floats (== 8 mod 32 words: the fragment loads below hit 32 distinct
//     banks).  Three stages; cp.async.wait_group + one __syncthreads per chunk, no mbarrier, no TMA;
//   * fragments: a thread needs rows g, g + 8 of an m16 tile (g = lane / 4) at k = t, t + 4 (t = lane % 4).  Fragment row
//     g holds tile row 2g and row g + 8 holds 2g + 1 (columns of B likewise: n8 tile j, column g = column 2g + j of its n16
//     pair), so one 8-byte ld.shared fetches two fragment elements and the accumulators of a thread cover 4 consecutive
//     output columns of 2 consecutive rows (16-byte stores).  Which hardware lane computes an output does not change it;
//   * operand transform on fragment load: x*p + y*q + r (A: the BatchNorm backward of two sources) or x*p + r (B: the
//     previous layer's BatchNorm-apply) with per-row constants held in registers, optional ReLU, then the hi/lo split of
//     split_tf32 (common.cuh), so the tensor core gets the values the wgmma kernel gives it.  Per k8 step the three
//     products run in the wgmma kernel's order: a_lo*b_hi, a_hi*b_lo, a_hi*b_hi;
//   * tile: 96 rows x 288 columns x one K slice of `chunks_per_split` chunks, 12 warps of 48 x 48 (2 x 6), 72 fp32
//     accumulators a thread.  A warp whose rows or columns lie past the operand skips its MMAs: a 27-row product pays for
//     32 rows, not 128;
//   * output: the K slice's partial, straight from the accumulators into the split-K workspace [split][M][N] (or C when
//     there is one slice), the layout hrl_board_fold_many and sum_partials_kernel read.
#include <cuda_runtime.h>
#include <stdint.h>

#include "gemm_wgrad.cuh"

namespace hrl {
namespace {

constexpr int kThreads = 384;              // 12 warps: 2 (rows) x 6 (columns) of 48 x 48 outputs each
constexpr int kTileM = 96, kTileN = 288;
constexpr int kWarpM = 48, kWarpN = 48;
constexpr int kChunk = 32;                 // samples per stage (the K slices are whole chunks, as in the wgmma kernel)
constexpr int kStages = 3;
constexpr int kLdA = kTileM + 8;           // shared row strides in floats, == 8 (mod 32)
constexpr int kLdB = kTileN + 8;
constexpr int kStageFloats = 2 * kChunk * kLdA + kChunk * kLdB;      // [A | A's second source | B]
constexpr size_t kSmemBytes = (size_t)kStages * kStageFloats * 4;
static_assert(kLdA % 32 == 8 && kLdB % 32 == 8, "conflict-free fragment loads need row strides == 8 (mod 32) words");

struct Operand {
    const float *ptr, *ptr2;               // [K][ld] sources (ptr2: second source, kind 2 only)
    const float *p, *q, *r;                // per-row constants (kinds 1 and 2)
    long long ld;
    int relu;
};

struct Params {
    Operand a, b;                          // A: kind 0, 1 or 2; B: kind 0 or 1
    float *C;
    long long ldc, c_split_stride;
    int M, N, K, chunks_per_split;
    int debug;
};

// operand kinds (template parameters): 0 = plain, 1 = x*p + r, 2 = x*p + y*q + r (two sources)
template <int KIND>
__device__ __forceinline__ float transform(float x, float y, float p, float q, float r, bool relu) {
    if (KIND == 0) return x;
    const float v = KIND == 2 ? fmaf(x, p, fmaf(y, q, r)) : fmaf(x, p, r);
    return relu ? fmaxf(v, 0.f) : v;
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const float (&a)[4], float b0, float b1) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
          "r"(__float_as_uint(b0)), "r"(__float_as_uint(b1)));
}

// per-row constants of this thread's 6 rows of an operand (rows 16 i + 2 g + e of the warp's 48, i < 3, e < 2): p, q, r
// as the transform uses them.  Rows past the operand get zeros (their outputs are not stored).
template <int KIND, bool IS_A>
__device__ __forceinline__ void load_consts(const Operand &op, int row0, int rows, float (&p)[6], float (&q)[6], float (&r)[6]) {
#pragma unroll
    for (int u = 0; u < 6; u++) {
        const int row = row0 + 16 * (u >> 1) + (u & 1);
        p[u] = q[u] = r[u] = 0.f;
        if (KIND == 0 || row >= rows) continue;
        p[u] = __ldg(op.p + row);
        r[u] = __ldg(op.r + row);
        if (op.q != nullptr) q[u] = __ldg(op.q + row);
        // the wgmma kernel forms a single-source A as x*p + (0*q + r), a single-source B as x*p + r
        if (KIND == 1 && IS_A) r[u] = fmaf(0.f, q[u], r[u]);
    }
}

// one 32-sample chunk of this warp's 48 x 48 outputs from shared stage `st`.  TAIL: the chunk runs past K; samples
// k >= k_left contribute exact zeros (as in the wgmma kernel).
template <int AK, int BK, bool TAIL>
__device__ __forceinline__ void mma_chunk(float (&acc)[3][6][4], const float *st, int mw, int nw, int g, int t, int k_left,
                                          const float (&pa)[6], const float (&qa)[6], const float (&ra)[6], bool relu_a,
                                          const float (&pb)[6], const float (&qb)[6], const float (&rb)[6], bool relu_b) {
    const float *sa = st, *sa2 = st + kChunk * kLdA, *sb = st + 2 * kChunk * kLdA;
#pragma unroll
    for (int ks = 0; ks < kChunk / 8; ks++) {
        const int k0 = 8 * ks + t, k1 = k0 + 4;
        const bool v0 = !TAIL || k0 < k_left, v1 = !TAIL || k1 < k_left;
        float ahi[3][4], alo[3][4];
#pragma unroll
        for (int i = 0; i < 3; i++) {
            const int m = mw + 16 * i + 2 * g;
            const float2 x0 = *reinterpret_cast<const float2 *>(sa + k0 * kLdA + m);
            const float2 x1 = *reinterpret_cast<const float2 *>(sa + k1 * kLdA + m);
            float2 y0 = make_float2(0.f, 0.f), y1 = y0;
            if (AK == 2) {
                y0 = *reinterpret_cast<const float2 *>(sa2 + k0 * kLdA + m);
                y1 = *reinterpret_cast<const float2 *>(sa2 + k1 * kLdA + m);
            }
            const int u = 2 * i;
            float v[4] = {transform<AK>(x0.x, y0.x, pa[u], qa[u], ra[u], relu_a), transform<AK>(x0.y, y0.y, pa[u + 1], qa[u + 1], ra[u + 1], relu_a),
                          transform<AK>(x1.x, y1.x, pa[u], qa[u], ra[u], relu_a), transform<AK>(x1.y, y1.y, pa[u + 1], qa[u + 1], ra[u + 1], relu_a)};
            if (TAIL) {
                if (!v0) v[0] = v[1] = 0.f;
                if (!v1) v[2] = v[3] = 0.f;
            }
#pragma unroll
            for (int e = 0; e < 4; e++) split_tf32(v[e], ahi[i][e], alo[i][e]);
        }
#pragma unroll
        for (int jp = 0; jp < 3; jp++) {
            const int n = nw + 16 * jp + 2 * g;
            const float2 z0 = *reinterpret_cast<const float2 *>(sb + k0 * kLdB + n);
            const float2 z1 = *reinterpret_cast<const float2 *>(sb + k1 * kLdB + n);
            const int u = 2 * jp;
            // element [j][h]: n8 tile j of the pair, fragment register h (k = t + 4 h)
            float v[2][2] = {{transform<BK>(z0.x, 0.f, pb[u], qb[u], rb[u], relu_b), transform<BK>(z1.x, 0.f, pb[u], qb[u], rb[u], relu_b)},
                             {transform<BK>(z0.y, 0.f, pb[u + 1], qb[u + 1], rb[u + 1], relu_b),
                              transform<BK>(z1.y, 0.f, pb[u + 1], qb[u + 1], rb[u + 1], relu_b)}};
            if (TAIL) {
                if (!v0) v[0][0] = v[1][0] = 0.f;
                if (!v1) v[0][1] = v[1][1] = 0.f;
            }
            float bhi[2][2], blo[2][2];
#pragma unroll
            for (int j = 0; j < 2; j++)
#pragma unroll
                for (int h = 0; h < 2; h++) split_tf32(v[j][h], bhi[j][h], blo[j][h]);
            // small terms first, as the wgmma kernel: a_lo*b_hi, a_hi*b_lo, a_hi*b_hi
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = 0; j < 2; j++) mma_tf32(acc[i][2 * jp + j], alo[i], bhi[j][0], bhi[j][1]);
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = 0; j < 2; j++) mma_tf32(acc[i][2 * jp + j], ahi[i], blo[j][0], blo[j][1]);
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = 0; j < 2; j++) mma_tf32(acc[i][2 * jp + j], ahi[i], bhi[j][0], bhi[j][1]);
        }
    }
}

template <int AK, int BK>
__global__ void __launch_bounds__(kThreads, 1) gemm_wgrad_kernel(const Params p) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int m0 = blockIdx.x * kTileM, n0 = blockIdx.y * kTileN, split = blockIdx.z;
    const int mw = (warp & 1) * kWarpM, nw = (warp >> 1) * kWarpN;          // the warp's outputs inside the tile
    const bool active = m0 + mw < p.M && n0 + nw < p.N;
    const int total_chunks = (p.K + kChunk - 1) / kChunk;
    const int c_begin = split * p.chunks_per_split, c_end = min(total_chunks, c_begin + p.chunks_per_split);

    float pa[6], qa[6], ra[6], pb[6], qb[6], rb[6];
    load_consts<AK, true>(p.a, m0 + mw + 2 * g, p.M, pa, qa, ra);
    load_consts<BK, false>(p.b, n0 + nw + 2 * g, p.N, pb, qb, rb);
    const bool relu_a = AK != 0 && p.a.relu, relu_b = BK != 0 && p.b.relu;

    // raw copies of chunk c into stage s: 16-byte groups of 4 columns; rows past K and groups past the operand are skipped
    // (the tail is masked when the fragments are loaded, and columns past the operand only reach outputs that are not stored)
    const uint32_t smem_base = (uint32_t)__cvta_generic_to_shared(smem);
    auto issue = [&](int c, int s) {
        if (c < c_end && (p.debug & 3) != 2) {
            const int k0 = c * kChunk;
            const uint32_t st = smem_base + (uint32_t)s * kStageFloats * 4;
            constexpr int kGroupsA = kTileM / 4, kGroupsB = kTileN / 4;
#pragma unroll
            for (int u = 0; u < kChunk * kGroupsA / kThreads; u++) {
                const int i = tid + u * kThreads, k = i / kGroupsA, col = 4 * (i - k * kGroupsA);
                if (k0 + k < p.K && m0 + col < p.M) {
                    const long long off = (long long)(k0 + k) * p.a.ld + m0 + col;
                    const uint32_t dst = st + (uint32_t)(k * kLdA + col) * 4;
                    cp_async16(dst, p.a.ptr + off);
                    if (AK == 2) cp_async16(dst + kChunk * kLdA * 4, p.a.ptr2 + off);
                }
            }
#pragma unroll
            for (int u = 0; u < kChunk * kGroupsB / kThreads; u++) {
                const int i = tid + u * kThreads, k = i / kGroupsB, col = 4 * (i - k * kGroupsB);
                if (k0 + k < p.K && n0 + col < p.N)
                    cp_async16(st + (uint32_t)(2 * kChunk * kLdA + k * kLdB + col) * 4, p.b.ptr + (long long)(k0 + k) * p.b.ld + n0 + col);
            }
        }
        cp_async_commit();          // one group per chunk, empty or not: the wait below counts groups
    };

    float acc[3][6][4];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 6; j++)
#pragma unroll
            for (int e = 0; e < 4; e++) acc[i][j][e] = 0.f;

#pragma unroll
    for (int s = 0; s < kStages - 1; s++) issue(c_begin + s, s);
    for (int c = c_begin; c < c_end; c++) {
        const int it = c - c_begin;
        cp_async_wait<kStages - 2>();       // this chunk's copies (by this thread) have landed
        __syncthreads();                    // ... and everybody's; the stage read in the previous iteration is free again
        issue(c + kStages - 1, (it + kStages - 1) % kStages);
        if (active && (p.debug & 3) != 1) {
            const float *st = smem + (it % kStages) * kStageFloats;
            const int k_left = p.K - c * kChunk;
            if (k_left >= kChunk)
                mma_chunk<AK, BK, false>(acc, st, mw, nw, g, t, k_left, pa, qa, ra, relu_a, pb, qb, rb, relu_b);
            else
                mma_chunk<AK, BK, true>(acc, st, mw, nw, g, t, k_left, pa, qa, ra, relu_a, pb, qb, rb, relu_b);
        }
    }
    cp_async_wait<0>();

    // accumulator (i, n8 tile j) register e: row 16 i + 2 g + e / 2, column 16 (j / 2) + 4 t + 2 (e % 2) + j % 2 of the warp's
    // 48 x 48 -> per row and n16 pair, 4 consecutive columns
    if (!active) return;
    float *Cg = p.C + (long long)split * p.c_split_stride;
    const bool vec = (p.ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(Cg) & 15) == 0);
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int m = m0 + mw + 16 * i + 2 * g + h;
            if (m >= p.M) continue;
            float *row = Cg + (long long)m * p.ldc;
#pragma unroll
            for (int jp = 0; jp < 3; jp++) {
                const int n = n0 + nw + 16 * jp + 4 * t;
                const float v[4] = {acc[i][2 * jp][2 * h], acc[i][2 * jp + 1][2 * h], acc[i][2 * jp][2 * h + 1], acc[i][2 * jp + 1][2 * h + 1]};
                if (vec && n + 3 < p.N) {
                    *reinterpret_cast<float4 *>(row + n) = make_float4(v[0], v[1], v[2], v[3]);
                } else {
#pragma unroll
                    for (int e = 0; e < 4; e++)
                        if (n + e < p.N) row[n + e] = v[e];
                }
            }
        }
    }
}

template <int AK, int BK>
int launch(const Params &p, dim3 grid, cudaStream_t stream) {
    HRL_CUDA_CHECK(cudaFuncSetAttribute(gemm_wgrad_kernel<AK, BK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
    gemm_wgrad_kernel<AK, BK><<<grid, kThreads, kSmemBytes, stream>>>(p);
    return HRL_OK;
}

template <int AK>
int launch_b(const Params &p, int bk, dim3 grid, cudaStream_t stream) {
    return bk == 0 ? launch<AK, 0>(p, grid, stream) : launch<AK, 1>(p, grid, stream);
}

bool aligned16(const void *ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

int kind_of(const HrlGemmOperand &o) { return o.p == nullptr ? 0 : o.ptr2 == nullptr ? 1 : 2; }

}  // namespace

bool gemm_wgrad_applies(const HrlGemmArgs &g) {
    auto fits = [](const HrlGemmOperand &o) {
        return !o.kmajor && !o.packed && (o.p == nullptr || o.feature_is_row) && o.ld % 4 == 0 && aligned16(o.ptr) &&
               (o.ptr2 == nullptr || aligned16(o.ptr2));
    };
    return !g.bf16 && g.conv_mode == 0 && g.segments == 0 && g.epilogue == HRL_GEMM_EP_STORE && g.bias == nullptr && fits(g.a) &&
           fits(g.b) && g.b.ptr2 == nullptr;
}

int launch_gemm_wgrad(const HrlGemmArgs &g, int chunks_per_split, int splits, float *C, long long ldc, long long c_split_stride,
                      int debug, cudaStream_t stream) {
    Params p;
    auto operand = [](const HrlGemmOperand &o) {
        Operand r;
        r.ptr = o.ptr; r.ptr2 = o.ptr2; r.p = o.p; r.q = o.q; r.r = o.r; r.ld = o.ld; r.relu = o.relu ? 1 : 0;
        return r;
    };
    p.a = operand(g.a);
    p.b = operand(g.b);
    p.C = C; p.ldc = ldc; p.c_split_stride = c_split_stride;
    p.M = (int)g.M; p.N = (int)g.N; p.K = (int)g.K; p.chunks_per_split = chunks_per_split;
    p.debug = debug;
    const dim3 grid((unsigned)((g.M + kTileM - 1) / kTileM), (unsigned)((g.N + kTileN - 1) / kTileN), (unsigned)splits);
    const int ak = kind_of(g.a), bk = kind_of(g.b);
    return ak == 0 ? launch_b<0>(p, bk, grid, stream) : ak == 1 ? launch_b<1>(p, bk, grid, stream) : launch_b<2>(p, bk, grid, stream);
}

}  // namespace hrl
