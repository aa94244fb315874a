// Shared body of the tensor-core GEMM (csrc/gemm_kernel.cu: 3xTF32, the default; csrc/gemm_bf16_kernel.cu: bf16 operands).
// The including translation unit names the kernel template, its operand precision and its launcher:
//     #define HRL_GEMM_KERNEL gemm_tf32x3_kernel / gemm_bf16_kernel      template <A_K, B_K, PACKED, NW>
//     #define HRL_GEMM_BF16   false / true                               the constexpr BF16 inside the body
//     #define HRL_GEMM_LAUNCH launch_gemm_tf32x3 / launch_gemm_bf16      the MMA-width dispatch over its instantiations
// so that each unit instantiates only its own precision (17 widths x 6 operand layouts) from one kernel text and one width
// table, and the 3xTF32 kernels are the same __global__ function as before the bf16 form existed (a __device__ body behind a
// wrapper kernel changes their register allocation).
//
// bf16 form (HrlGemmArgs.bf16): operands are staged as in the 3xTF32 form -- global -> registers -> fp32 transform (fmaf,
// optional ReLU) -- then rounded to nearest even bf16 (__float2bfloat16_rn) and stored once, K-major SWIZZLE_64B (a
// 32-element chunk of a row = 64 bytes).  A stage is [B | A] (a quarter of the 3xTF32 stage's bytes), a packed B image is
// [chunk][n_pad rows][64 bytes] (one bulk copy per stage), and a chunk is 2 wgmma m64nNk16 .f32.bf16.bf16 per warpgroup into the
// same fp32 accumulators; the epilogues are shared.  A product of two bf16 values is exact in fp32, so the result is the
// fp32-accumulated product of the rounded operands.
// A unit that defines none (csrc/gemm_tower_kernel.cu) gets the shared pieces only: operand layout, wgmma helpers, epilogue.
#pragma once
#if defined(HRL_GEMM_KERNEL) != defined(HRL_GEMM_BF16) || defined(HRL_GEMM_KERNEL) != defined(HRL_GEMM_LAUNCH)
#error "define all of HRL_GEMM_KERNEL, HRL_GEMM_BF16 and HRL_GEMM_LAUNCH before including gemm_common.cuh, or none"
#endif
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace hrl {

constexpr int kGemmThreads = 512;   // 4 warpgroups: operand loaders, MMA issuers and epilogue at once
constexpr int kTileM = 128;
constexpr int kMaxN = 288;          // columns of one CTA tile (shared memory: 2 stages of hi/lo operands)
constexpr int kChunkK = 32;         // reduction elements per shared-memory stage
constexpr int kStages = 2;
constexpr int kItemsA = kTileM * 8 / kGemmThreads;

constexpr int kMaxSegments = 64;     // (dy, x) pairs of one segmented weight-gradient product

struct GemmOperand {
    const float *ptr, *ptr2;        // ptr2: optional second source with the same layout (operand = x*p + y*q + r), or NULL
    const float *p, *q, *r;         // per-feature constants of the operand transform, or NULL (plain operand)
    long long ld;
    int kmajor;                     // 1: element (row,k) at row*ld + k ; 0: at k*ld + row
    int relu;                       // clamp the transformed operand at 0
    int feature_is_row;             // constants indexed by the operand's row (else by the reduction index k)
    int packed;                     // B only: ptr is the hrl_board_pack image [chunk][hi|lo][n_pad rows][128 B swizzled]
};

struct GemmParams {
    GemmOperand a, b;
    const float *bias;
    float *C;
    long long ldc;
    long long c_split_stride;       // elements between the partial outputs of consecutive K slices
    int M, N, K;
    int chunks_per_split;
    int epilogue;                   // HrlGemmEpilogue
    const float *ep_y;              // masked epilogue: the pre-activation tile (M x N, leading dimension ep_ldy)
    long long ep_ldy;
    const float *ep_scale, *ep_shift, *ep_mean, *ep_rstd;     // per column, may be NULL
    float *col_partials;            // [row tiles][2][N] column sums of the epilogues that produce statistics
    int debug;                      // profiling only: 1 = no MMAs, 2 = no loads/stores
    // convolution over a board as an implicit product (no im2col in memory).  conv_off[pos * taps + tap] = (cell read by kernel
    // tap `tap` at output cell `pos`) - pos, or kConvOutside (zero padding); wrap-around boards simply have no outside.
    //   mode 1 (forward / input gradient): A rows are pixels of a channels-last tensor (ld = pixel stride), the reduction runs over
    //           (tap, channel) with every tap's channels padded to whole 32-element chunks -- chunk c reads tap c / cpt.
    //   mode 2 (weight gradient): the reduction runs over pixels, B row n is (tap, channel) = (n / cin, n % cin) of the shifted input.
    const short *conv_off;
    int conv_mode, conv_hw, conv_taps, conv_cin, conv_cpt;
    // mode 2 over several (dy, x) pairs that share one weight (a recurrent cell applied at every time step): K slice `split`
    // reads pair split / seg_splits -- ONE product per weight and backward pass instead of one per application
    int seg_splits;                 // 0 = one pair (a.ptr / b.ptr)
    int conv_ones;                  // 1: one more B row, all ones: its output column is sum_pixels dy = the bias gradient
    const float *seg_a[kMaxSegments], *seg_b[kMaxSegments];
};

constexpr short kConvOutside = -32768;
constexpr int kConvMaxTable = 256 * 9;     // cells x taps

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!ok);
}

// shared-memory matrix descriptor of wgmma, K-major, 128-byte swizzle (start >> 4 | LBO >> 4 << 16 | SBO >> 4 << 32 |
// layout SWIZZLE_128B = 1 << 62).  A row of the tile is the 128 bytes (32 reduction elements) of one chunk; 8-row groups
// are 1024 bytes apart (SBO); inside a group the 16-byte slot j of row r sits at slot j ^ (r & 7) (Swizzle<3,4,3>).  LBO is
// not used by swizzled K-major layouts (set to 1).  The k-step inside the chunk is selected by advancing the start
// address by 32 bytes; every tile base is 1024-byte aligned (base offset 0).
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t addr) {
    return (uint64_t)((addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// the same for bf16 operands: a row of the tile is the 64 bytes (32 reduction elements) of one chunk, SWIZZLE_64B (layout 2 << 62):
// 8-row groups are 512 bytes apart (SBO); inside a group the 16-byte slot j of row r sits at slot j ^ ((r >> 1) & 3)
// (Swizzle<2,4,3>).  The k16 step inside the chunk advances the start address by 32 bytes; tile bases are 512-byte aligned.
__device__ __forceinline__ uint64_t wgmma_desc_sw64(uint32_t addr) {
    return (uint64_t)((addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(512 >> 4) << 32) | (2ull << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }

// the last wait: every accumulator passes through an empty asm after it, so that no read of them is scheduled before it
template <int NACC>
__device__ __forceinline__ void wgmma_wait_all(float (&d)[NACC]) {
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < NACC; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] += A[64 x 8] * B[N x 8]^T, both operands in shared memory (tf32, K-major).  The instruction shape is part of
// the opcode: one specialisation per width, each naming exactly its N / 2 accumulators a thread.
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc);
template <>
__device__ __forceinline__ void wgmma_tf32<8>(float (&d)[4], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n8k8.f32.tf32.tf32 {%0, %1, %2, %3}, %4, %5, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<16>(float (&d)[8], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<24>(float (&d)[12], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %14, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n24k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11}, %12, %13, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<40>(float (&d)[20], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %22, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n40k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19}, %20, %21, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<48>(float (&d)[24], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<56>(float (&d)[28], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %30, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n56k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27}, %28, %29, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<72>(float (&d)[36], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %38, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n72k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35}, %36, %37, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<80>(float (&d)[40], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n80k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<88>(float (&d)[44], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %46, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n88k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43}, %44, %45, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<96>(float (&d)[48], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<104>(float (&d)[52], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %54, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n104k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51}, %52, %53, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<112>(float (&d)[56], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n112k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<120>(float (&d)[60], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %62, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n120k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59}, %60, %61, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
                   "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<144>(float (&d)[72], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %74, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n144k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}, %72, %73, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
                   "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}

// D[64 x N] += A[64 x 16] * B[N x 16]^T, bf16 operands in shared memory (K-major: the two transpose immediates are 0),
// fp32 accumulators with the fragment of the tf32 form.
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc);
template <>
__device__ __forceinline__ void wgmma_bf16<8>(float (&d)[4], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<16>(float (&d)[8], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<24>(float (&d)[12], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %14, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n24k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11}, %12, %13, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<32>(float (&d)[16], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<40>(float (&d)[20], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %22, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n40k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19}, %20, %21, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<48>(float (&d)[24], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<56>(float (&d)[28], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %30, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n56k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27}, %28, %29, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<72>(float (&d)[36], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %38, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n72k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35}, %36, %37, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<80>(float (&d)[40], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<88>(float (&d)[44], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %46, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n88k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43}, %44, %45, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<96>(float (&d)[48], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<104>(float (&d)[52], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %54, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n104k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51}, %52, %53, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<112>(float (&d)[56], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n112k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<120>(float (&d)[60], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %62, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n120k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59}, %60, %61, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
                   "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}
template <>
__device__ __forceinline__ void wgmma_bf16<144>(float (&d)[72], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %74, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n144k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}, %72, %73, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
                   "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
                   "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
                   "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
                 : "l"(a_desc), "l"(b_desc), "r"(1)
                 : "memory");
}

// one stage of the 3xTF32 product for this warpgroup's quarter of the tile: small terms first, a_lo*b_hi + a_hi*b_lo + a_hi*b_hi.
// The width is a compile-time constant of the kernel: with a runtime choice between widths ptxas cannot keep the
// accumulators in fixed registers across the cases and serialises the chain with injected warpgroup.arrive (C7519).
template <int N>
__device__ __forceinline__ void mma_stage(float (&d)[N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
#pragma unroll
    for (int ks = 0; ks < kChunkK / 8; ks++) {
        wgmma_tf32<N>(d, wgmma_desc(a_lo + 32 * ks), wgmma_desc(b_hi + 32 * ks));
        wgmma_tf32<N>(d, wgmma_desc(a_hi + 32 * ks), wgmma_desc(b_lo + 32 * ks));
        wgmma_tf32<N>(d, wgmma_desc(a_hi + 32 * ks), wgmma_desc(b_hi + 32 * ks));
    }
}

// one stage of the bf16 product: 2 k16 steps per 32-element chunk
template <int N>
__device__ __forceinline__ void mma_stage_bf16(float (&d)[N / 2], uint32_t a, uint32_t b) {
#pragma unroll
    for (int ks = 0; ks < kChunkK / 16; ks++) wgmma_bf16<N>(d, wgmma_desc_sw64(a + 32 * ks), wgmma_desc_sw64(b + 32 * ks));
}

// 4 transformed fp32 elements -> 4 bf16, round to nearest even (element k at the lower address)
__device__ __forceinline__ uint2 pack_bf16x4(const float4 v) {
    const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    return make_uint2(*reinterpret_cast<const uint32_t *>(&lo), *reinterpret_cast<const uint32_t *>(&hi));
}

__device__ __forceinline__ void split_tf32(const float4 v, float4 &hi, float4 &lo) {
    split_tf32(v.x, hi.x, lo.x);
    split_tf32(v.y, hi.y, lo.y);
    split_tf32(v.z, hi.z, lo.z);
    split_tf32(v.w, hi.w, lo.w);
}

// ---- operand loaders.  Every thread owns a fixed set of "items" (one row x 4 consecutive reduction elements = one 16-byte
// shared-memory slot per split half, K-major SWIZZLE_128B: a row's chunk = 128 bytes, slot j of row r at j ^ (r & 7)); their
// coordinates follow from the thread index (the kernel derives them again in every chunk), each chunk advances the pointers.
// (An operand stored [K][rows] is transposed by the loads -- 4 scalar loads per item, coalesced along the rows: wgmma takes
//  tf32 operands K-major only.)
// Item (B operand): 32-bit offsets -- the host bounds b.ld below 2^22.  ItemA (A operand): 64-bit offsets (any ld).
// The row is the row inside the tile (< 288); the tile's first row is added by the caller.
template <typename Off>
struct ItemT {             // three (B) or four (A) registers per item (a thread holds up to 5 B and 2 A items)
    Off off;               // first of the 4 elements in chunk 0, relative to the tile's first element
    uint32_t slot;         // byte offset of the 16-byte slot inside an operand half: row * 128 + ((j ^ (row & 7)) << 4)
    uint32_t meta;         // k | live << 9 | row << 10;  k = 4 * j: offset of the quad inside a chunk, row: for per-row constants
    __device__ __forceinline__ int k() const { return (int)(meta & 63u); }
    __device__ __forceinline__ bool live() const { return (meta >> 9) & 1u; }
    __device__ __forceinline__ int row() const { return (int)(meta >> 10); }
};
using Item = ItemT<int>;
using ItemA = ItemT<long long>;

template <bool KMAJOR, typename It = Item, bool BF16 = false>
__device__ __forceinline__ It make_item(int i, int n_items, long long ld, int rows_pad, int rows) {
    It it;
    int row, j;
    if (KMAJOR) {           // 8 consecutive lanes = the 128 contiguous bytes of one row's chunk: one cache line per quarter
        row = i >> 3;       // warp in global memory, and (swizzle) 8 distinct 16-byte slots in shared memory
        j = i & 7;
    } else {                // consecutive lanes = consecutive rows: coalesced along the contiguous dimension, and the swizzle
        j = i / rows_pad;   // spreads 8 consecutive rows of one slot column over 8 distinct slots
        row = i - j * rows_pad;
    }
    const bool live = i < n_items && row < rows;
    it.meta = (uint32_t)(4 * j) | ((live ? 1u : 0u) << 9) | ((uint32_t)row << 10);
    if constexpr (BF16)     // 8 bytes of the 64-byte row, SWIZZLE_64B: 16-byte slot j / 2 at (j / 2) ^ ((row >> 1) & 3), half j % 2
        it.slot = (uint32_t)row * 64u + (uint32_t)((((j >> 1) ^ ((row >> 1) & 3)) << 4) | ((j & 1) << 3));
    else
        it.slot = (uint32_t)row * 128u + (uint32_t)((j ^ (row & 7)) << 4);
    it.off = (decltype(it.off))(KMAJOR ? (long long)row * ld + 4 * j : (long long)(4 * j) * ld + row);
    if (i >= n_items) it.slot = 0xFFFFFFFFu;
    return it;
}

template <bool KMAJOR, typename It>
__device__ __forceinline__ float4 load_item(const It &it, const float *base, long long ld, bool vec, long long advance, int k_left) {
    // k_left = reduction elements from this chunk's start to the end of the operand (>= 32 in every chunk but the last)
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!it.live()) return v;
    const float *q = base + it.off + advance;
    if (k_left >= kChunkK) {                     // interior chunk: no per-element bounds
        if (KMAJOR) {
            if (vec) return __ldg(reinterpret_cast<const float4 *>(q));
            v.x = __ldg(q); v.y = __ldg(q + 1); v.z = __ldg(q + 2); v.w = __ldg(q + 3);
        } else {
            v.x = __ldg(q); v.y = __ldg(q + ld); v.z = __ldg(q + 2 * ld); v.w = __ldg(q + 3 * ld);
        }
        return v;
    }
    const long long st = KMAJOR ? 1 : ld;          // last, partial chunk
    const int k = it.k();
    if (k + 0 < k_left) v.x = __ldg(q);
    if (k + 1 < k_left) v.y = __ldg(q + st);
    if (k + 2 < k_left) v.z = __ldg(q + 2 * st);
    if (k + 3 < k_left) v.w = __ldg(q + 3 * st);
    return v;
}

// weight gradient of a convolution (conv_mode 2): the item's row is (tap, channel) = (off >> 16, off & 0xFFFF), its 4 reduction
// elements are 4 consecutive pixels; each reads the pixel's tap neighbour (or nothing outside the board).  `src` is the chunk's
// table [32 pixels][taps] of source pixels (-1 = outside / past the end), computed once per chunk by the producers together.
__device__ __forceinline__ float4 load_item_conv(const Item &it, const float *base, long long ld, int k0, const GemmParams &p,
                                                 const int *src) {
    float r[4] = {0.f, 0.f, 0.f, 0.f};
    if (it.live()) {
        const int ci = it.off & 0xFFFF, tap = it.off >> 16;
        if (tap >= p.conv_taps) {                    // the ones row (bias gradient)
#pragma unroll
            for (int e = 0; e < 4; e++) r[e] = (k0 + it.k() + e < p.K) ? 1.f : 0.f;
        } else {
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int sp = src[(it.k() + e) * p.conv_taps + tap];
                if (sp >= 0) r[e] = __ldg(base + (long long)sp * ld + ci);
            }
        }
    }
    return make_float4(r[0], r[1], r[2], r[3]);
}

// operand transform v = x*p[f] + y*q[f] + r[f] (relu optional) on the 4 elements of an item; elements outside the operand
// (dead rows, reduction tail) stay exactly zero.  f = the operand row (row_base + the item's row), or the reduction index k0 + k + e.
template <typename It>
__device__ __forceinline__ float4 transform_item(const GemmOperand &op, const It &it, float4 x, float4 y, int k0, int k_left,
                                                 long long row_base) {
    if (op.p == nullptr || !it.live()) return x;
    float4 pp, qq = make_float4(0.f, 0.f, 0.f, 0.f), rr;
    const int k = it.k();
    if (op.feature_is_row) {
        const long long row = row_base + it.row();
        const float a = __ldg(op.p + row), c = __ldg(op.r + row);
        pp = make_float4(a, a, a, a);
        rr = make_float4(c, c, c, c);
        if (op.q != nullptr) { const float bq = __ldg(op.q + row); qq = make_float4(bq, bq, bq, bq); }
    } else {
        const int f = k0 + k;
        if (k + 3 < k_left) {                      // k0 and k are multiples of 4: aligned vector loads of the constants
            pp = __ldg(reinterpret_cast<const float4 *>(op.p + f));
            rr = __ldg(reinterpret_cast<const float4 *>(op.r + f));
            if (op.q != nullptr) qq = __ldg(reinterpret_cast<const float4 *>(op.q + f));
        } else {
            pp = rr = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k + 0 < k_left) { pp.x = __ldg(op.p + f); rr.x = __ldg(op.r + f); if (op.q) qq.x = __ldg(op.q + f); }
            if (k + 1 < k_left) { pp.y = __ldg(op.p + f + 1); rr.y = __ldg(op.r + f + 1); if (op.q) qq.y = __ldg(op.q + f + 1); }
            if (k + 2 < k_left) { pp.z = __ldg(op.p + f + 2); rr.z = __ldg(op.r + f + 2); if (op.q) qq.z = __ldg(op.q + f + 2); }
        }
    }
    float4 v;
    v.x = fmaf(x.x, pp.x, fmaf(y.x, qq.x, rr.x));
    v.y = fmaf(x.y, pp.y, fmaf(y.y, qq.y, rr.y));
    v.z = fmaf(x.z, pp.z, fmaf(y.z, qq.z, rr.z));
    v.w = fmaf(x.w, pp.w, fmaf(y.w, qq.w, rr.w));
    if (op.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    if (k + 0 >= k_left) v.x = 0.f;
    if (k + 1 >= k_left) v.y = 0.f;
    if (k + 2 >= k_left) v.z = 0.f;
    if (k + 3 >= k_left) v.w = 0.f;
    return v;
}

// ---- epilogue of the wgmma kernels (the general one below and gemm_tower_kernel): the accumulators of warpgroup wg cover
// rows 64 (wg & 1) ... and columns NW (wg >> 1) ... of the tile at (m0, n0); registers -> shared-memory tile (padded rows) ->
// coalesced global stores into K slice `split`'s output.
template <int NW>
__device__ __forceinline__ void gemm_epilogue(const GemmParams &p, float (&acc)[NW / 2], uint8_t *smem, int m0, int rows_a, int n0,
                                              int n_here, int split) {
    constexpr int n_pad = 2 * NW, nw = NW;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    // (a thread holds 2 columns of 2 rows per 8-column group: storing from registers would scatter every warp instruction)
    //   HRL_GEMM_EP_RELU        C = max(acc, 0)
    //   HRL_GEMM_EP_STATS       C = acc, plus per-column sum and sum of squares of acc - mean over the tile's rows (mean = the
    //                           pivot ep_mean, or 0: shifted sums keep the variance when |mean| >> std)
    //   HRL_GEMM_EP_MASK_STATS  C = acc * (z > 0) with z = y*scale+shift of the pre-activation tile y (the ReLU
    //                           backward), plus per-column sums of C and of C * xhat, xhat = (y - mean) * rstd
    //                           (the two batch sums the BatchNorm backward needs)
    float *Cg = p.C + (long long)split * p.c_split_stride;
    const int ldt = n_pad + 4;                           // row stride = 16 (mod 128) bytes: conflict-free 16-byte stores
    float *tile = reinterpret_cast<float *>(smem);       // the stages are free once the last MMAs have completed
    const int ep = p.epilogue;
    // copy-out mapping: a thread owns ONE group of 4 columns (its constants and column sums live in 16 registers) and the
    // rows my_r, my_r + rpp, ...; consecutive threads = consecutive 16 bytes of a row, then of the next row
    const bool vec_c = (p.ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(Cg) & 15) == 0) && (n0 % 4 == 0) && (n_here % 4 == 0);
    const int cols4 = n_here >> 2;
    // rows per pass; capped by the column-sum scratch the host sized for the widest tile (a narrower last tile would take more)
    const int rpp = vec_c ? min(kGemmThreads / cols4, kGemmThreads / max(1, (n_pad - 12) / 4)) : 1;
    const int my_r = vec_c ? tid / cols4 : 0, my_c4 = tid - my_r * cols4;
    const bool mine = vec_c && my_r < rpp;
    const bool masked = ep == HRL_GEMM_EP_MASK_STATS;
    const bool vec_y = masked && (p.ep_ldy % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.ep_y) & 15) == 0);
    constexpr int kAhead = 4;                              // rows of the pre-activation tile in flight per thread
    float4 yq[kAhead];
    auto load_y = [&](int r) -> float4 {
        const float *yp = p.ep_y + (long long)(m0 + r) * p.ep_ldy + n0 + 4 * my_c4;
        if (vec_y) return __ldg(reinterpret_cast<const float4 *>(yp));
        return make_float4(__ldg(yp), __ldg(yp + 1), __ldg(yp + 2), __ldg(yp + 3));
    };
    if (masked && mine) {
#pragma unroll
        for (int u = 0; u < kAhead; u++) {
            const int r = my_r + u * rpp;
            yq[u] = r < rows_a ? load_y(r) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    __syncthreads();                                     // every warpgroup is done with the stages
    {
        // accumulator fragment of m64nN: register 4 j + i holds row 16 (warp % 4) + lane / 4 + 8 (i / 2), column 8 j + 2 (lane % 4) + i % 2
        const int r0 = (wg & 1) * 64 + (warp & 3) * 16 + (lane >> 2);
        const int cb = (wg >> 1) * nw + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < NW / 8; j++) {
            const int col = cb + 8 * j;
            float b0 = 0.f, b1 = 0.f;
            if (p.bias != nullptr) {
                if (col < n_here) b0 = __ldg(p.bias + n0 + col);
                if (col + 1 < n_here) b1 = __ldg(p.bias + n0 + col + 1);
            }
            *reinterpret_cast<float2 *>(tile + r0 * ldt + col) = make_float2(acc[4 * j] + b0, acc[4 * j + 1] + b1);
            *reinterpret_cast<float2 *>(tile + (r0 + 8) * ldt + col) = make_float2(acc[4 * j + 2] + b0, acc[4 * j + 3] + b1);
        }
    }
    __syncthreads();
    {
        const bool stats = (ep == HRL_GEMM_EP_STATS || masked) && p.col_partials != nullptr;
        float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
        if (mine) {
            float k_sc[4] = {1.f, 1.f, 1.f, 1.f}, k_sh[4] = {0.f, 0.f, 0.f, 0.f}, k_mu[4] = {0.f, 0.f, 0.f, 0.f}, k_rs[4] = {1.f, 1.f, 1.f, 1.f};
            if (masked || ep == HRL_GEMM_EP_STATS) {
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int col = n0 + 4 * my_c4 + e;
                    if (p.ep_scale) k_sc[e] = __ldg(p.ep_scale + col);
                    if (p.ep_shift) k_sh[e] = __ldg(p.ep_shift + col);
                    if (p.ep_mean) k_mu[e] = __ldg(p.ep_mean + col);
                    if (p.ep_rstd) k_rs[e] = __ldg(p.ep_rstd + col);
                }
            }
            for (int r0 = my_r; r0 < rows_a; r0 += kAhead * rpp) {
#pragma unroll
                for (int u = 0; u < kAhead; u++) {
                    const int r = r0 + u * rpp;
                    if (r >= rows_a) break;
                    float4 v = reinterpret_cast<const float4 *>(tile + r * ldt)[my_c4];
                    if (ep == HRL_GEMM_EP_RELU) {
                        v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
                    } else if (ep == HRL_GEMM_EP_STATS) {
                        const float d[4] = {v.x - k_mu[0], v.y - k_mu[1], v.z - k_mu[2], v.w - k_mu[3]};
#pragma unroll
                        for (int e = 0; e < 4; e++) {
                            s1[e] += d[e];
                            s2[e] = fmaf(d[e], d[e], s2[e]);
                        }
                    } else if (masked) {
                        const float4 y = yq[u];
                        const int rn = r + kAhead * rpp;
                        if (rn < rows_a) yq[u] = load_y(rn);              // the row this slot serves next
                        const float yv[4] = {y.x, y.y, y.z, y.w};
                        float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                        for (int e = 0; e < 4; e++) {
                            const float z = fmaf(yv[e], k_sc[e], k_sh[e]);
                            const float d = z > 0.f ? vv[e] : 0.f;
                            const float xh = (yv[e] - k_mu[e]) * k_rs[e];
                            vv[e] = d;
                            s1[e] += d;
                            s2[e] = fmaf(d, xh, s2[e]);
                        }
                        v = make_float4(vv[0], vv[1], vv[2], vv[3]);
                    }
                    reinterpret_cast<float4 *>(Cg + (long long)(m0 + r) * p.ldc + n0)[my_c4] = v;
                }
            }
        } else if (!vec_c) {
            for (int r = warp; r < rows_a; r += kGemmThreads / 32) {
                const float *src = tile + r * ldt;
                float *dst = Cg + (long long)(m0 + r) * p.ldc + n0;
                for (int c1 = lane; c1 < n_here; c1 += 32) dst[c1] = (ep == HRL_GEMM_EP_RELU) ? fmaxf(src[c1], 0.f) : src[c1];
            }
        }
        if (stats) {       // (the statistics epilogues require vec_c: checked by the host)
            // per-thread column sums -> shared memory (behind the tile) -> fixed-order sum over the row passes -> global partials
            float *red = tile + kTileM * ldt;                 // [rpp][2][n_pad]
            if (mine) {
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    red[(my_r * 2 + 0) * n_pad + 4 * my_c4 + e] = s1[e];
                    red[(my_r * 2 + 1) * n_pad + 4 * my_c4 + e] = s2[e];
                }
            }
            __syncthreads();
            for (int i = tid; i < 2 * n_here; i += kGemmThreads) {
                const int which = i / n_here, col = i - which * n_here;
                float acc = 0.f;
                for (int w = 0; w < rpp; w++) acc += red[(w * 2 + which) * n_pad + col];
                p.col_partials[((long long)blockIdx.x * 2 + which) * p.N + n0 + col] = acc;
            }
        }
    }
}

#ifdef HRL_GEMM_KERNEL
// A and B go global -> registers -> (transform, hi/lo split) -> shared memory; a packed B image arrives by one bulk copy a
// stage.  Each thread owns kItemsA items of the A tile (coalesced: 8 consecutive lanes = the 128 bytes of one k-major row,
// or consecutive rows of a transposed one) and ITEMS_B items of the B tile.  NW = the MMA width of a warpgroup = half the
// tile's padded column count n_pad (one instantiation per width the host dispatches).
template <bool A_K, bool B_K, bool PACKED, int NW>
__global__ void __launch_bounds__(kGemmThreads, 1) HRL_GEMM_KERNEL(const GemmParams p) {
    constexpr bool BF16 = HRL_GEMM_BF16;
    constexpr int n_pad = 2 * NW, nw = NW;
    constexpr int ITEMS_B = PACKED ? 1 : (n_pad * 8 + kGemmThreads - 1) / kGemmThreads;
    // B items loaded ahead of the stage barrier; the rest of the 5 items of the widest tiles are loaded after it, so that
    // at most 3 B float4s (plus the A items) are in flight next to the 72 accumulators
    constexpr int kItemsB1 = ITEMS_B < 3 ? ITEMS_B : 3;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);      // swizzle atoms need 1024-byte alignment
    __shared__ __align__(8) uint64_t bars[kStages];     // packed B: the stage's bulk copy has landed
    __shared__ float b_consts[2][kMaxN];     // per-row constants of a single-source B transform (no registers, no per-chunk loads)
    __shared__ float a_consts[3][kTileM];    // the same for A (one or two sources): p, q, r of the tile's rows
    __shared__ short conv_off_s[kConvMaxTable];
    __shared__ int conv_src_s[2][kChunkK * 9];      // conv_mode 2: source pixel of (pixel of the chunk, tap), two chunks in flight

    const int tid = threadIdx.x, warp = tid >> 5;
    const int m0 = blockIdx.x * kTileM;
    const int n0 = blockIdx.y * kMaxN;
    const int split = blockIdx.z;
    const int n_here = min(kMaxN, p.N - n0);
    const int rows_a = min(kTileM, p.M - m0);
    const int total_chunks = (p.K + kChunkK - 1) / kChunkK;
    const int seg = p.seg_splits ? split / p.seg_splits : 0;
    const int c_begin = (p.seg_splits ? split - seg * p.seg_splits : split) * p.chunks_per_split;
    const float *a_base = p.seg_splits ? p.seg_a[seg] : p.a.ptr, *b_base = p.seg_splits ? p.seg_b[seg] : p.b.ptr;
    const int c_end = min(total_chunks, c_begin + p.chunks_per_split);

    // shared-memory stage: [B_hi | B_lo | A_hi | A_lo], each [rows][128 B] with the 16-byte slots of a row swizzled;
    // bf16: [B | A], each [rows][64 B]
    constexpr uint32_t kElem = BF16 ? 2 : 4, kHalves = BF16 ? 1 : 2;
    const uint32_t b_bytes = (uint32_t)n_pad * kChunkK * kElem;
    const uint32_t a_bytes = (uint32_t)kTileM * kChunkK * kElem;
    const uint32_t stage_bytes = kHalves * (b_bytes + a_bytes);
    const uint32_t smem_base = smem_u32(smem);

    if (PACKED && tid == 0) {
        for (int s = 0; s < kStages; s++) mbar_init(smem_u32(&bars[s]), 1);      // one arrive.expect_tx per use
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (p.conv_mode != 0)
        for (int i = tid; i < p.conv_hw * p.conv_taps; i += kGemmThreads) conv_off_s[i] = p.conv_off[i];
    // single-source transform with per-row constants (the weight gradient's activation operand)
    const bool b_rows = !PACKED && p.b.p != nullptr && p.b.feature_is_row && p.b.ptr2 == nullptr;
    if (b_rows) {
        for (int i = tid; i < kMaxN; i += kGemmThreads) {
            const bool in = i < n_here;
            b_consts[0][i] = in ? __ldg(p.b.p + n0 + i) : 1.f;
            b_consts[1][i] = in ? __ldg(p.b.r + n0 + i) : 0.f;
        }
    }
    // per-row constants of the A transform (the weight gradient's BatchNorm-backward operand)
    const bool a_rows = p.a.p != nullptr && p.a.feature_is_row;
    if (a_rows) {
        for (int i = tid; i < kTileM; i += kGemmThreads) {
            const bool in = i < rows_a;
            a_consts[0][i] = in ? __ldg(p.a.p + m0 + i) : 1.f;
            a_consts[1][i] = in && p.a.q ? __ldg(p.a.q + m0 + i) : 0.f;
            a_consts[2][i] = in ? __ldg(p.a.r + m0 + i) : 0.f;
        }
    }
    __syncthreads();

    // ---- A items.  conv_mode 1: the row is a pixel, the chunk belongs to one kernel tap -> the source is the tap's neighbour
    const float *Ag = a_base + (A_K ? (long long)m0 * p.a.ld : (long long)m0);
    const long long a2 = p.a.ptr2 ? (p.a.ptr2 - p.a.ptr) : 0;
    const bool vec_a = A_K && (p.a.ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(a_base) & 15) == 0) &&
                       (!p.a.ptr2 || (reinterpret_cast<uintptr_t>(p.a.ptr2) & 15) == 0);
    // The items' coordinates are derived from the thread index again in every chunk (a few integer operations; `t` passes
    // through an empty asm so that the compiler cannot hoist them out of the loop): held across the loop they would take
    // 3-4 registers an item, and the instantiations with 5 B items and 72 accumulators would spill.
    auto items_a = [&](int t, ItemA (&ia)[kItemsA]) {
#pragma unroll
        for (int u = 0; u < kItemsA; u++) ia[u] = make_item<A_K, ItemA, BF16>(t + u * kGemmThreads, kTileM * 8, p.a.ld, kTileM, rows_a);
    };
    int conv_pos[kItemsA];
    {
        ItemA ia[kItemsA];
        items_a(tid, ia);
#pragma unroll
        for (int u = 0; u < kItemsA; u++) conv_pos[u] = A_K && p.conv_mode == 1 ? (int)(((long long)m0 + ia[u].row()) % p.conv_hw) : 0;
    }

    // ---- B items
    const long long off_b = B_K ? (long long)n0 * p.b.ld : (long long)n0;
    const float *Bg = b_base + off_b;
    const long long b2 = p.b.ptr2 ? (p.b.ptr2 - p.b.ptr) : 0;
    const bool vec_b = B_K && (p.b.ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.b.ptr) & 15) == 0) &&
                       (!p.b.ptr2 || (reinterpret_cast<uintptr_t>(p.b.ptr2) & 15) == 0);
    auto items_b = [&](int t, Item (&ib)[ITEMS_B]) {
#pragma unroll
        for (int u = 0; u < ITEMS_B; u++) {
            ib[u] = make_item<B_K, Item, BF16>(t + u * kGemmThreads, n_pad * 8, p.b.ld, n_pad, n_here);
            if (!PACKED && !B_K && p.conv_mode == 2) {          // row n -> (tap, channel)
                const int n = n0 + ib[u].row(), tap = n / p.conv_cin;
                ib[u].off = (n - tap * p.conv_cin) | (tap << 16);
            }
        }
    };

    // ---- this warpgroup's quarter of the tile: rows 64 (wg & 1) ..., columns nw (wg >> 1) ...
    const int wg = warp >> 2;
    float acc[NW / 2];
#pragma unroll
    for (int i = 0; i < NW / 2; i++) acc[i] = 0.f;

    for (int c = c_begin; c < c_end; c++) {
        const int it = c - c_begin, s = it % kStages;
        const int k0 = c * kChunkK;
        const int k_left = p.K - k0;
        const long long adv_b = B_K ? (long long)k0 : (long long)k0 * p.b.ld;
        if (!PACKED && !B_K && p.conv_mode == 2) {
            // source pixels of this chunk, once for all items: conv_src_s[it & 1][pixel][tap] (double-buffered: the readers of
            // the previous chunk are past their loads before anybody reaches this chunk's barrier)
            if (tid < kChunkK * p.conv_taps) {
                const int kkl = tid / p.conv_taps, tap = tid - kkl * p.conv_taps, kk = k0 + kkl;
                const short o = conv_off_s[(kk % p.conv_hw) * p.conv_taps + tap];
                conv_src_s[it & 1][tid] = (kk < p.K && o != kConvOutside) ? kk + o : -1;
            }
            asm volatile("bar.sync 1, %0;" ::"n"(kGemmThreads) : "memory");
        }
        int t = tid;
        asm volatile("" : "+r"(t));
        ItemA ia[kItemsA];
        Item ib[ITEMS_B];
        items_a(t, ia);
        items_b(t, ib);
        float4 va[kItemsA], vb[ITEMS_B];
        // B items [u0, u1): global -> registers, transform
        auto load_b = [&](int u0, int u1) {
#pragma unroll
            for (int u = u0; u < u1; u++)
                vb[u] = (!B_K && p.conv_mode == 2) ? load_item_conv(ib[u], b_base, p.b.ld, k0, p, conv_src_s[it & 1])
                                                   : load_item<B_K>(ib[u], Bg, p.b.ld, vec_b, adv_b, k_left);
            if (b_rows) {
#pragma unroll
                for (int u = u0; u < u1; u++) {
                    if (!ib[u].live()) continue;
                    const float pc = b_consts[0][ib[u].row()], rc = b_consts[1][ib[u].row()];
                    float4 v;
                    v.x = fmaf(vb[u].x, pc, rc); v.y = fmaf(vb[u].y, pc, rc); v.z = fmaf(vb[u].z, pc, rc); v.w = fmaf(vb[u].w, pc, rc);
                    if (p.b.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
                    if (k_left < kChunkK) {                  // the reduction tail stays exactly zero
                        const int k = ib[u].k();
                        if (k + 0 >= k_left) v.x = 0.f;
                        if (k + 1 >= k_left) v.y = 0.f;
                        if (k + 2 >= k_left) v.z = 0.f;
                        if (k + 3 >= k_left) v.w = 0.f;
                    }
                    vb[u] = v;
                }
            } else if (p.b.p != nullptr) {
#pragma unroll
                for (int u = u0; u < u1; u++) {
                    const float4 y = p.b.ptr2 ? load_item<B_K>(ib[u], Bg, p.b.ld, vec_b, adv_b + b2, k_left) : make_float4(0.f, 0.f, 0.f, 0.f);
                    vb[u] = transform_item(p.b, ib[u], vb[u], y, k0, k_left, n0);
                }
            }
        };
        // B items [u0, u1): hi/lo split (or bf16 rounding) -> shared memory
        auto store_b = [&](uint8_t *stp, int u0, int u1) {
#pragma unroll
            for (int u = u0; u < u1; u++) {
                if constexpr (BF16) {
                    if (ib[u].slot != 0xFFFFFFFFu) *reinterpret_cast<uint2 *>(stp + ib[u].slot) = pack_bf16x4(vb[u]);
                } else if (ib[u].slot != 0xFFFFFFFFu) {
                    float4 h4, l4;
                    split_tf32(vb[u], h4, l4);
                    *reinterpret_cast<float4 *>(stp + ib[u].slot) = h4;
                    *reinterpret_cast<float4 *>(stp + b_bytes + ib[u].slot) = l4;
                }
            }
        };
        if ((p.debug & 3) != 2) {
            // all the loads first (one exposed latency per chunk, not one per item), then the transforms
            if (A_K && p.conv_mode == 1) {          // (the host requires a k-major A for convolutions)
                const int tap = c / p.conv_cpt, ch0 = (c - tap * p.conv_cpt) * kChunkK;      // first channel of the chunk
#pragma unroll
                for (int u = 0; u < kItemsA; u++) {
                    const short o = conv_off_s[conv_pos[u] * p.conv_taps + tap];
                    va[u] = o == kConvOutside ? make_float4(0.f, 0.f, 0.f, 0.f)
                                              : load_item<true>(ia[u], Ag, p.a.ld, vec_a, (long long)o * p.a.ld + ch0, p.conv_cin - ch0);
                }
            } else {
                const long long adv_a = A_K ? (long long)k0 : (long long)k0 * p.a.ld;
#pragma unroll
                for (int u = 0; u < kItemsA; u++) va[u] = load_item<A_K>(ia[u], Ag, p.a.ld, vec_a, adv_a, k_left);
                if (a_rows) {
#pragma unroll
                    for (int u = 0; u < kItemsA; u++) {
                        const float4 y = p.a.ptr2 ? load_item<A_K>(ia[u], Ag, p.a.ld, vec_a, adv_a + a2, k_left) : make_float4(0.f, 0.f, 0.f, 0.f);
                        if (!ia[u].live()) continue;
                        const int r = ia[u].row();
                        const float pc = a_consts[0][r], qc = a_consts[1][r], rc = a_consts[2][r];
                        float4 v;
                        v.x = fmaf(va[u].x, pc, fmaf(y.x, qc, rc));
                        v.y = fmaf(va[u].y, pc, fmaf(y.y, qc, rc));
                        v.z = fmaf(va[u].z, pc, fmaf(y.z, qc, rc));
                        v.w = fmaf(va[u].w, pc, fmaf(y.w, qc, rc));
                        if (p.a.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
                        if (k_left < kChunkK) {                  // the reduction tail stays exactly zero
                            const int k = ia[u].k();
                            if (k + 0 >= k_left) v.x = 0.f;
                            if (k + 1 >= k_left) v.y = 0.f;
                            if (k + 2 >= k_left) v.z = 0.f;
                            if (k + 3 >= k_left) v.w = 0.f;
                        }
                        va[u] = v;
                    }
                } else if (p.a.p != nullptr) {
#pragma unroll
                    for (int u = 0; u < kItemsA; u++) {
                        const float4 y = p.a.ptr2 ? load_item<A_K>(ia[u], Ag, p.a.ld, vec_a, adv_a + a2, k_left) : make_float4(0.f, 0.f, 0.f, 0.f);
                        va[u] = transform_item(p.a, ia[u], va[u], y, k0, k_left, m0);
                    }
                }
            }
            if (!PACKED) load_b(0, kItemsB1);
        }
        // the stage is free once every warpgroup's products of chunk it - kStages have completed
        wgmma_wait<kStages - 1>();
        asm volatile("bar.sync 1, %0;" ::"n"(kGemmThreads) : "memory");
        uint8_t *stp = smem + s * stage_bytes;
        if (PACKED && tid == 0) {           // weights: one bulk copy of the stage's pre-split, pre-swizzled image
            const uint32_t bar = smem_u32(&bars[s]);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(kHalves * b_bytes) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                             smem_base + s * stage_bytes),
                         "l"(reinterpret_cast<const uint8_t *>(p.b.ptr) + (size_t)c * kHalves * b_bytes), "r"(kHalves * b_bytes), "r"(bar)
                         : "memory");
        }
        if ((p.debug & 3) != 2) {
            asm volatile("" : "+r"(t));           // the slots again: cheaper than holding them across the barrier
            items_a(t, ia);
            items_b(t, ib);
#pragma unroll
            for (int u = 0; u < kItemsA; u++) {
                if constexpr (BF16) {
                    if (ia[u].slot != 0xFFFFFFFFu) *reinterpret_cast<uint2 *>(stp + b_bytes + ia[u].slot) = pack_bf16x4(va[u]);
                } else if (ia[u].slot != 0xFFFFFFFFu) {
                    float4 h4, l4;
                    split_tf32(va[u], h4, l4);
                    *reinterpret_cast<float4 *>(stp + 2 * b_bytes + ia[u].slot) = h4;
                    *reinterpret_cast<float4 *>(stp + 2 * b_bytes + a_bytes + ia[u].slot) = l4;
                }
            }
            if (!PACKED) {
                store_b(stp, 0, kItemsB1);
                load_b(kItemsB1, ITEMS_B);          // the second pass of the widest tiles (while the previous chunk's MMAs run)
                store_b(stp, kItemsB1, ITEMS_B);
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores -> visible to the tensor core
        asm volatile("bar.sync 1, %0;" ::"n"(kGemmThreads) : "memory");    // the stage is full
        if (PACKED) mbar_wait(smem_u32(&bars[s]), (it / kStages) & 1);
        if ((p.debug & 3) != 1) {
            const uint32_t st = smem_base + s * stage_bytes;
            if constexpr (BF16) {
                const uint32_t a_st = st + b_bytes + (uint32_t)(wg & 1) * 64 * 64, b_st = st + (uint32_t)(wg >> 1) * nw * 64;
                wgmma_fence();
                mma_stage_bf16<NW>(acc, a_st, b_st);
            } else {
                const uint32_t a_hi = st + 2 * b_bytes + (uint32_t)(wg & 1) * 64 * 128, b_hi = st + (uint32_t)(wg >> 1) * nw * 128;
                wgmma_fence();
                mma_stage<NW>(acc, a_hi, a_hi + a_bytes, b_hi, b_hi + b_bytes);
            }
            wgmma_commit();
        }
    }
    wgmma_wait_all(acc);

    gemm_epilogue<NW>(p, acc, smem, m0, rows_a, n0, n_here, split);
}

template <bool A_K, bool B_K, bool PACKED, int NW>
static int launch_gemm(const GemmParams &p, dim3 grid, size_t smem_bytes, cudaStream_t stream) {
    HRL_CUDA_CHECK(cudaFuncSetAttribute(HRL_GEMM_KERNEL<A_K, B_K, PACKED, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    HRL_GEMM_KERNEL<A_K, B_K, PACKED, NW><<<grid, kGemmThreads, smem_bytes, stream>>>(p);
    return HRL_OK;
}

// the operand layouts of one MMA width (a packed B image is k-major)
template <int NW>
static int launch_gemm_width(const GemmParams &p, dim3 grid, size_t smem_bytes, cudaStream_t stream) {
    if (p.b.packed) return p.a.kmajor ? launch_gemm<true, true, true, NW>(p, grid, smem_bytes, stream)
                                      : launch_gemm<false, true, true, NW>(p, grid, smem_bytes, stream);
    if (p.a.kmajor) return p.b.kmajor ? launch_gemm<true, true, false, NW>(p, grid, smem_bytes, stream)
                                      : launch_gemm<true, false, false, NW>(p, grid, smem_bytes, stream);
    return p.b.kmajor ? launch_gemm<false, true, false, NW>(p, grid, smem_bytes, stream)
                      : launch_gemm<false, false, false, NW>(p, grid, smem_bytes, stream);
}

int HRL_GEMM_LAUNCH(const GemmParams &p, int nw, dim3 grid, size_t smem_bytes, cudaStream_t stream) {
    switch (nw) {                 // the MMA width of a warpgroup: half of n_pad, a multiple of 16 up to 256, then 288
    case 8: return launch_gemm_width<8>(p, grid, smem_bytes, stream);
    case 16: return launch_gemm_width<16>(p, grid, smem_bytes, stream);
    case 24: return launch_gemm_width<24>(p, grid, smem_bytes, stream);
    case 32: return launch_gemm_width<32>(p, grid, smem_bytes, stream);
    case 40: return launch_gemm_width<40>(p, grid, smem_bytes, stream);
    case 48: return launch_gemm_width<48>(p, grid, smem_bytes, stream);
    case 56: return launch_gemm_width<56>(p, grid, smem_bytes, stream);
    case 64: return launch_gemm_width<64>(p, grid, smem_bytes, stream);
    case 72: return launch_gemm_width<72>(p, grid, smem_bytes, stream);
    case 80: return launch_gemm_width<80>(p, grid, smem_bytes, stream);
    case 88: return launch_gemm_width<88>(p, grid, smem_bytes, stream);
    case 96: return launch_gemm_width<96>(p, grid, smem_bytes, stream);
    case 104: return launch_gemm_width<104>(p, grid, smem_bytes, stream);
    case 112: return launch_gemm_width<112>(p, grid, smem_bytes, stream);
    case 120: return launch_gemm_width<120>(p, grid, smem_bytes, stream);
    case 128: return launch_gemm_width<128>(p, grid, smem_bytes, stream);
    case 144: return launch_gemm_width<144>(p, grid, smem_bytes, stream);
    default: HRL_REQUIRE(false, HRL_ERR_BAD_ARG, "hrl_gemm_fused: no kernel for an MMA width of %d columns", nw);
    }
}
#endif  // HRL_GEMM_KERNEL

// the entry points of the two precisions (csrc/gemm_kernel.cu, csrc/gemm_bf16_kernel.cu): launch the kernel of MMA width nw
// for p's operand layouts
int launch_gemm_tf32x3(const GemmParams &p, int nw, dim3 grid, size_t smem_bytes, cudaStream_t stream);
int launch_gemm_bf16(const GemmParams &p, int nw, dim3 grid, size_t smem_bytes, cudaStream_t stream);

}  // namespace hrl
