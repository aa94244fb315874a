// The fused tower's forward and input-gradient products on wgmma with A from registers (sm_90a).
//
//   C[M x N] = A_op[M x K] * B[N x K]^T      A K-major fp32 (one or two sources), B a packed hrl_board_pack image, N <= 288
//
// The general wgmma kernel (gemm_common.cuh) stages A through registers one chunk at a time: load, transform, split into
// hi / lo, store both halves swizzled, two CTA barriers, then the MMAs.  Only one chunk of A is in flight, and at the
// tower's shape there is one 128-row tile per SM, so the global-load latency is exposed in every chunk.  Here:
//   * tile and warps as in the wgmma kernel: 128 rows x 288 columns, 4 warpgroups, warpgroup wg owns rows 64 (wg & 1) ...
//     and columns 144 (wg >> 1) ..., 72 fp32 accumulators a thread; the epilogue is the wgmma kernel's (gemm_epilogue);
//   * A staging: every 32-element chunk is copied raw by 16-byte cp.async into shared rows padded to 36 floats, several
//     chunks ahead (3 stages for one source; 2 for two sources, the input gradient's dZ and Y).  A fragment load of
//     (row 16 w + g, k t) hits bank (4 g + t) mod 32: 32 distinct banks.  Copies stay inside the operand (rows < M, 16-byte
//     groups below K, which with ld % 4 == 0 is below min(ld, round_up(K, 4))); rows >= M and k >= K are zeroed when the
//     fragments are formed;
//   * B staging: the packed image's chunk (hi | lo, 128-byte swizzled rows) by one cp.async.bulk on an mbarrier, 2 stages.
//     Chunk c + 1's copy is issued as soon as all four warpgroups have finished chunk c - 1's MMAs (a named barrier), one
//     chunk ahead of its use;
//   * fragments: per k8 step a thread loads its four A elements (rows g, g + 8 of its warp's 16, k = t, t + 4: the .tf32
//     register fragment of wgmma), applies the wgmma kernel's transform fmaf(x, p, fmaf(y, q, r)) (y = 0 for one source)
//     with per-reduction-index constants (for one source copied to shared memory once), the optional ReLU and the tail
//     zeroing, then split_tf32's truncating hi / lo split, and issues a_lo*b_hi, a_hi*b_lo, a_hi*b_hi -- the wgmma kernel's values, chunks, k8 steps and product order
//     into the same accumulators, so the outputs are the same bits.  One wgmma group per k8 step; the fragment registers
//     are double-buffered (a group's A registers must not change until it has completed: wait_group 1 before a buffer
//     is written again).
// Shared memory: 2 x 73,728 B of B + 3 x 18,432 B (one source) or 2 x 2 x 18,432 B (two sources) of A = 202,752 / 221,184 B,
// plus 1 KB of alignment; the epilogue tile reuses it once every copy has landed.
#include <cuda_runtime.h>
#include <stdint.h>

#include "gemm_common.cuh"
#include "gemm_tower.cuh"

namespace hrl {
namespace {

constexpr int kNW = 144;                                   // MMA width of a warpgroup: a tile of 288 padded columns
constexpr int kLdA = kChunkK + 4;                          // shared row stride of a raw A chunk in floats (== 4 mod 32)
constexpr uint32_t kBHalf = 2 * kNW * kChunkK * 4;         // one half (hi or lo) of a packed chunk: 288 rows x 128 bytes
constexpr uint32_t kBStage = 2 * kBHalf;
constexpr int kBStages = 2;
constexpr uint32_t kAStage = kTileM * kLdA * 4;            // one source's raw chunk
static_assert(kLdA % 32 == 4, "conflict-free fragment loads need a row stride == 4 (mod 32) words");
constexpr int kMaxConstK = 512;                            // reduction length of a transformed A (constants held in shared memory)

// operand kinds (template parameter): 0 = plain, 1 = x*p + r (optional ReLU), 2 = x*p + y*q + r (two sources)
template <int KIND>
struct Ring {
    static constexpr int sources = KIND == 2 ? 2 : 1;
    static constexpr int stages = KIND == 2 ? 2 : 3;
    static constexpr size_t smem = 1024 + (size_t)kBStages * kBStage + (size_t)stages * sources * kAStage;
};
// the epilogue's tile and column-sum scratch (n_pad 288: 7 row passes) fit into the stages
static_assert(1024 + ((size_t)kTileM * (2 * kNW + 4) + 2 * 7 * 2 * kNW) * 4 <= Ring<0>::smem, "epilogue tile");
static_assert(Ring<2>::smem + 3 * kMaxConstK * 4 + 64 <= 232448, "shared memory of one block");

// D[64 x 144] += A[64 x 8] * B[144 x 8]^T: A from registers (the .tf32 fragment: rows g, g + 8, k t, t + 4), B in shared memory
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[72], const float (&a)[4], uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %77, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n144k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}, {%72, %73, %74, %75}, %76, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
                   "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
                 : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
                   "l"(b_desc), "r"(1)
                 : "memory");
}

template <int KIND>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_tower_kernel(const GemmParams p) {
    using R = Ring<KIND>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);      // swizzle atoms need 1024-byte alignment
    __shared__ __align__(8) uint64_t full[kBStages];       // the stage's B bulk copy has landed
    // kind 1: p, q, r of A's transform over the whole reduction, read once here rather than from global memory in every k8
    // step, where each chunk's first read missed L1 and its latency sat between the wgmma groups.  (The two-source kind
    // keeps the per-step __ldg: with this copy its results changed, for a reason not yet found.)
    __shared__ float a_consts[KIND == 1 ? 3 : 1][KIND == 1 ? kMaxConstK : 1];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, g = lane >> 2, t = lane & 3;
    const int m0 = blockIdx.x * kTileM;
    const int rows_a = min(kTileM, p.M - m0);
    const int chunks = (p.K + kChunkK - 1) / kChunkK;
    const uint32_t b_ring = smem_u32(smem), a_ring = b_ring + kBStages * kBStage;

    if (tid == 0) {
        for (int s = 0; s < kBStages; s++) mbar_init(smem_u32(&full[s]), 1);      // one arrive.expect_tx per use
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    auto issue_b = [&](int c) {            // thread 0: chunk c of the packed image into stage c % 2
        const uint32_t bar = smem_u32(&full[c % kBStages]);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(kBStage) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                         b_ring + (uint32_t)(c % kBStages) * kBStage),
                     "l"(reinterpret_cast<const uint8_t *>(p.b.ptr) + (size_t)c * kBStage), "r"(kBStage), "r"(bar)
                     : "memory");
    };
    // raw copies of A's chunk c into stage c % stages: 8 consecutive threads = the 128 bytes of one row's chunk
    auto issue_a = [&](int c) {
        if (c < chunks && (p.debug & 3) != 2) {
            const int k0 = c * kChunkK;
            const uint32_t st = a_ring + (uint32_t)(c % R::stages) * R::sources * kAStage;
#pragma unroll
            for (int u = 0; u < kTileM * 8 / kGemmThreads; u++) {
                const int i = tid + u * kGemmThreads, row = i >> 3, k = k0 + 4 * (i & 7);
                if (row < rows_a && k < p.K) {
                    const long long off = (long long)(m0 + row) * p.a.ld + k;
                    const uint32_t dst = st + (uint32_t)(row * kLdA + 4 * (i & 7)) * 4;
                    cp_async16(dst, p.a.ptr + off);
                    if (KIND == 2) cp_async16(dst + kAStage, p.a.ptr2 + off);
                }
            }
        }
        cp_async_commit();                 // one group per chunk, empty or not: the wait below counts groups
    };

    if (tid == 0) {
        issue_b(0);
        if (chunks > 1) issue_b(1);
    }
#pragma unroll
    for (int c = 0; c < R::stages - 1; c++) issue_a(c);
    if (KIND == 1) {                       // (visible after the first chunk's __syncthreads)
        for (int k = tid; k < p.K; k += kGemmThreads) {
            a_consts[0][k] = __ldg(p.a.p + k);
            a_consts[1 % (KIND == 1 ? 3 : 1)][k] = p.a.q != nullptr ? __ldg(p.a.q + k) : 0.f;
            a_consts[2 % (KIND == 1 ? 3 : 1)][k] = __ldg(p.a.r + k);
        }
    }

    float acc[kNW / 2];
#pragma unroll
    for (int i = 0; i < kNW / 2; i++) acc[i] = 0.f;
    float a_hi[2][4], a_lo[2][4];                          // fragment registers, double-buffered across the k8 steps

    const int ra = (wg & 1) * 64 + (warp & 3) * 16 + g;    // the thread's fragment rows ra, ra + 8 inside the tile
    const bool live0 = ra < rows_a, live1 = ra + 8 < rows_a;
    const uint32_t b_wg = (uint32_t)(wg >> 1) * kNW * 128;  // the warpgroup's 144 B rows inside a half
    for (int c = 0; c < chunks; c++) {
        cp_async_wait<R::stages - 2>();    // this chunk's copies (by this thread) have landed
        __syncthreads();                   // ... and everybody's; the A stage read in the previous chunk is free again
        issue_a(c + R::stages - 1);
        const int k0 = c * kChunkK, k_left = p.K - k0;
        const float *sa = reinterpret_cast<const float *>(smem + kBStages * kBStage + (size_t)(c % R::stages) * R::sources * kAStage) + ra * kLdA;
        const uint32_t b_hi = b_ring + (uint32_t)(c % kBStages) * kBStage + b_wg, b_lo = b_hi + kBHalf;
        mbar_wait(smem_u32(&full[c % kBStages]), (c / kBStages) & 1);
        // k8 steps in pairs, one fragment buffer each: fully unrolled, ptxas hoists the next steps' loads and runs out of
        // registers (it then serialises the wgmma chain, C7512)
#pragma unroll 1
        for (int ks2 = 0; ks2 < kChunkK / 8; ks2 += 2)
#pragma unroll
        for (int buf = 0; buf < 2; buf++) {
            const int ks = ks2 + buf;
            // elements e: (row ra + 8 (e & 1), k 8 ks + t + 4 (e >> 1)) -- the fragment order a0..a3
            float v[4];
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int k = 8 * ks + t + 4 * (e >> 1), o = 8 * kLdA * (e & 1) + k;
                const float x = sa[o];
                float y = 0.f, pc = 0.f, qc = 0.f, rc = 0.f;
                if (KIND == 1 && k < k_left) {
                    pc = a_consts[0][k0 + k];
                    qc = a_consts[1 % (KIND == 1 ? 3 : 1)][k0 + k];
                    rc = a_consts[2 % (KIND == 1 ? 3 : 1)][k0 + k];
                } else if (KIND == 2 && k < k_left) {
                    pc = __ldg(p.a.p + k0 + k);
                    rc = __ldg(p.a.r + k0 + k);
                    if (p.a.q != nullptr) qc = __ldg(p.a.q + k0 + k);
                }
                if (KIND == 2) y = sa[o + kAStage / 4];
                float w = x;
                if (KIND != 0) {
                    w = fmaf(x, pc, fmaf(y, qc, rc));
                    if (p.a.relu) w = fmaxf(w, 0.f);
                }
                v[e] = (k < k_left && ((e & 1) ? live1 : live0)) ? w : 0.f;
            }
            // the group that read this buffer (two k8 steps back) has completed; the values pass through an empty asm after
            // the wait, so that the split writing the buffer cannot be scheduled before it
            wgmma_wait<1>();
#pragma unroll
            for (int e = 0; e < 4; e++) asm volatile("" : "+f"(v[e]));
#pragma unroll
            for (int e = 0; e < 4; e++) split_tf32(v[e], a_hi[buf][e], a_lo[buf][e]);
            if ((p.debug & 3) != 1) {
                wgmma_fence();
                wgmma_tf32_rs(acc, a_lo[buf], wgmma_desc(b_hi + 32 * ks));
                wgmma_tf32_rs(acc, a_hi[buf], wgmma_desc(b_lo + 32 * ks));
                wgmma_tf32_rs(acc, a_hi[buf], wgmma_desc(b_hi + 32 * ks));
                wgmma_commit();
            }
            // after this step's wait every product of chunk c - 1 has completed in this warpgroup: once all four have
            // arrived, thread 0 refills chunk c - 1's B stage with chunk c + 1
            if (ks == 1 && c >= 1 && c + 1 < chunks) {
                if (warp == 0) {
                    asm volatile("bar.sync 2, %0;" ::"n"(kGemmThreads) : "memory");
                    if (tid == 0) issue_b(c + 1);
                } else {
                    asm volatile("bar.arrive 2, %0;" ::"n"(kGemmThreads) : "memory");
                }
            }
        }
    }
    wgmma_wait_all(acc);
    cp_async_wait<0>();

    gemm_epilogue<kNW>(p, acc, smem, m0, rows_a, 0, p.N, 0);
}

template <int KIND>
int launch(const GemmParams &p, cudaStream_t stream) {
    HRL_CUDA_CHECK(cudaFuncSetAttribute(gemm_tower_kernel<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Ring<KIND>::smem));
    gemm_tower_kernel<KIND><<<(unsigned)((p.M + kTileM - 1) / kTileM), kGemmThreads, Ring<KIND>::smem, stream>>>(p);
    return HRL_OK;
}

bool aligned16(const void *ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

}  // namespace

bool gemm_tower_applies(const HrlGemmArgs &g) {
    const HrlGemmOperand &a = g.a;
    return !g.bf16 && g.conv_mode == 0 && g.segments == 0 && g.splits <= 1 && a.kmajor && !a.packed && a.ld % 4 == 0 &&
           aligned16(a.ptr) && (a.ptr2 == nullptr || aligned16(a.ptr2)) && (a.p == nullptr || (!a.feature_is_row && (a.ptr2 != nullptr || g.K <= kMaxConstK))) &&
           g.b.packed &&
           g.N > kMaxN - 32 && g.N <= kMaxN;
}

int launch_gemm_tower(const GemmParams &p, cudaStream_t stream) {
    if (p.a.p == nullptr) return launch<0>(p, stream);
    return p.a.ptr2 == nullptr ? launch<1>(p, stream) : launch<2>(p, stream);
}

}  // namespace hrl
