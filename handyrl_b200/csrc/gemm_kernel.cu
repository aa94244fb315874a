// fp32-accurate GEMM on the Hopper tensor cores (wgmma, sm_90a) for the dense contractions of the user's net.
//
//   C[M x N] = A_op[M x K] * B_op[N x K]^T  (+ bias[N])           all fp32 in global memory
//
// north_star: "tensor cores only for the model's Linear/Conv layers where they are dense contractions".  The nets of
// the reference's board games (handyrl/envs/tictactoe.py:52-69, geister.py:101-167) convolve over boards of a few cells;
// fastnet.py runs such a layer as ONE dense matrix product per direction (forward, input gradient, weight gradient),
// which cuBLAS executes as SIMT SGEMM because the learner's contract is fp32 (1e-5 of the reference).  Here the same
// product runs on wgmma.mma_async .tf32 with the 3xTF32 split
//       a = a_hi + a_lo,  a_hi = a with the 13 low mantissa bits cleared (exactly a TF32 number), a_lo = a - a_hi (exact)
//       a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi                     (dropped: a_lo*b_lo ~ 2^-22 |a||b|)
// accumulated in fp32 registers: fp32-class accuracy (relative error ~1e-6 of |a||b| sums, tests/test_gemm_gpu.py)
// at tensor-core speed.
//
// Structure (one CTA = one 128-row tile of C x up to 288 columns x one slice of K; 16 warps = 4 warpgroups):
//   * every thread loads operand data: global fp32 -> registers -> (transform, hi/lo split) -> shared memory in the
//     K-major SWIZZLE_128B layout wgmma reads (one 128-byte row per operand row and chunk, 16-byte slots XOR-swizzled by
//     the row: conflict-free 16-byte stores both for row-contiguous and for transposing loads); either operand may be
//     stored with its reduction dimension contiguous ("k-major") or strided (transposed on the fly: the weight-gradient
//     product reduces over samples).  Packed weight images (hrl_board_pack) arrive pre-split by one bulk copy per stage;
//   * two shared-memory stages of 32 reduction elements [B_hi | B_lo | A_hi | A_lo]: the loads of chunk c+1 are in flight
//     while the tensor cores work on chunk c (TMA tensor maps are not used: the operands need the hi/lo split on their way in);
//   * warpgroup w owns the accumulators of rows 64 (w & 1) ... + 63 and columns n_pad/2 (w >> 1) ... (72 fp32 registers a
//     thread at the widest tile) and issues 3 x 4 asynchronous wgmma per stage; the epilogue stages the tile through shared
//     memory for coalesced stores.
// The kernel body lives in gemm_common.cuh, shared with the opt-in bf16-operand form (HrlGemmArgs.bf16,
// csrc/gemm_bf16_kernel.cu); this unit instantiates the 3xTF32 kernels only.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#define HRL_GEMM_KERNEL gemm_tf32x3_kernel     // the kernel template gemm_common.cuh defines, its operand precision and launcher
#define HRL_GEMM_BF16 false
#define HRL_GEMM_LAUNCH launch_gemm_tf32x3
#include "gemm_common.cuh"
#include "gemm_tower.cuh"
#include "gemm_wgrad.cuh"

// profiling / test hook (include/hrl_b200.h): 1 = no MMAs, 2 = no operand loads
static int g_gemm_debug = 0;
extern "C" void hrl_gemm_set_debug(int v) { g_gemm_debug = v; }

namespace hrl {

// fixed-order sum of the K-slice partials: out[i] = sum_s partials[s][i]  (deterministic)
__global__ void sum_partials_kernel(const float *__restrict__ partials, int splits, long long n, long long stride, float *__restrict__ out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float s = partials[i];
        for (int k = 1; k < splits; k++) s += partials[(long long)k * stride + i];
        out[i] = s;
    }
}

}  // namespace hrl


extern "C" size_t hrl_gemm_workspace_floats(int64_t M, int64_t N, int64_t K, int32_t splits) {
    (void)K;
    return splits > 1 ? (size_t)splits * (size_t)M * (size_t)N : 0;
}

// how many K slices a request for `splits` really produces (whole 32-element chunks per slice, no empty slice)
extern "C" int32_t hrl_gemm_effective_splits(int64_t K, int32_t splits) {
    const int total_chunks = (int)((K + hrl::kChunkK - 1) / hrl::kChunkK);
    if (splits < 1) splits = 1;
    if (splits > total_chunks) splits = total_chunks;
    const int per = (total_chunks + splits - 1) / splits;
    return (total_chunks + per - 1) / per;
}

extern "C" int hrl_gemm_fused(const HrlGemmArgs *args, void *stream_) {
    using namespace hrl;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    HRL_REQUIRE(args != nullptr, HRL_ERR_BAD_ARG, "hrl_gemm_fused: args is NULL");
    const HrlGemmArgs &g = *args;
    const int64_t M = g.M, N = g.N, K = g.K;
    int splits = g.splits;
    HRL_REQUIRE(g.a.ptr && g.b.ptr && (g.C || ((splits > 1 || g.segments > 0) && g.workspace)), HRL_ERR_BAD_ARG, "hrl_gemm_fused: NULL pointer");
    HRL_REQUIRE(M > 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 22) && K < (1ll << 31) && g.b.ld < (1ll << 22), HRL_ERR_BAD_ARG,
                "hrl_gemm_fused: bad dimensions (M=%lld N=%lld K=%lld)", (long long)M, (long long)N, (long long)K);
    HRL_REQUIRE(g.conv_mode >= 0 && g.conv_mode <= 2, HRL_ERR_BAD_ARG, "hrl_gemm_fused: conv_mode is 0, 1 or 2");
    if (g.conv_mode != 0) {
        HRL_REQUIRE(g.conv_off && g.conv_hw > 0 && g.conv_taps > 0 && g.conv_cin > 0 && g.conv_cin < 65536 &&
                        (long long)g.conv_hw * g.conv_taps <= hrl::kConvMaxTable && g.a.p == nullptr && g.b.p == nullptr && g.splits >= 1,
                    HRL_ERR_BAD_ARG, "hrl_gemm_fused: convolution geometry (at most 256 cells x 9 taps, plain operands)");
        if (g.conv_mode == 1)
            HRL_REQUIRE(g.b.packed && g.a.kmajor && g.a.ld >= g.conv_cin && g.a.ld % 4 == 0 && (reinterpret_cast<uintptr_t>(g.a.ptr) & 15) == 0 &&
                            M % g.conv_hw == 0 && K == (int64_t)g.conv_taps * ((g.conv_cin + kChunkK - 1) / kChunkK) * kChunkK && g.splits == 1,
                        HRL_ERR_UNSUPPORTED,
                        "hrl_gemm_fused: convolution forward needs a packed B image over taps x (channels padded to 32), 16-byte aligned "
                        "pixel rows and whole boards");
        else
            HRL_REQUIRE(!g.b.packed && !g.a.kmajor && !g.b.kmajor && g.b.ld >= g.conv_cin &&
                            N == (int64_t)g.conv_taps * g.conv_cin + (g.conv_ones_row ? 1 : 0) && K % g.conv_hw == 0,
                        HRL_ERR_UNSUPPORTED,
                        "hrl_gemm_fused: convolution weight gradient reduces over whole boards of pixels, N = taps x channels (+ 1 with the ones row)");
    }
    HRL_REQUIRE(g.segments >= 0 && g.segments <= hrl::kMaxSegments &&
                    (g.segments == 0 || (g.conv_mode == 2 && g.seg_a && g.seg_b && g.workspace && g.C == nullptr)),
                HRL_ERR_BAD_ARG, "hrl_gemm_fused: up to %d segments, of a convolution weight gradient left as slice partials in the workspace",
                hrl::kMaxSegments);
    HRL_REQUIRE(!g.conv_ones_row || g.conv_mode == 2, HRL_ERR_BAD_ARG, "hrl_gemm_fused: the ones row belongs to the convolution weight gradient");
    HRL_REQUIRE((g.conv_mode == 1 || g.a.ld >= (g.a.kmajor ? K : M)) && (g.b.packed || g.conv_mode == 2 || g.b.ld >= (g.b.kmajor ? K : N)) &&
                    (g.C == nullptr || g.ldc >= N),
                HRL_ERR_BAD_ARG, "hrl_gemm_fused: leading dimension smaller than the row length");
    HRL_REQUIRE(!g.a.packed && (!g.b.packed || (N <= hrl::kMaxN && g.b.p == nullptr && (reinterpret_cast<uintptr_t>(g.b.ptr) & 15) == 0)),
                HRL_ERR_BAD_ARG, "hrl_gemm_fused: only an untransformed B operand of at most 288 rows can be a packed image");
    HRL_REQUIRE((g.a.p == nullptr) == (g.a.r == nullptr) && (g.b.p == nullptr) == (g.b.r == nullptr) &&
                    (g.a.ptr2 == nullptr || (g.a.p && g.a.q)) && (g.b.ptr2 == nullptr || (g.b.p && g.b.q)),
                HRL_ERR_BAD_ARG, "hrl_gemm_fused: an operand transform needs p and r (and q with a second source)");
    HRL_REQUIRE(g.epilogue >= HRL_GEMM_EP_STORE && g.epilogue <= HRL_GEMM_EP_MASK_STATS, HRL_ERR_BAD_ARG, "hrl_gemm_fused: unknown epilogue");
    HRL_REQUIRE(g.epilogue != HRL_GEMM_EP_MASK_STATS || (g.ep_y != nullptr && g.ep_ldy >= N && (g.ep_mean == nullptr) == (g.ep_rstd == nullptr)),
                HRL_ERR_BAD_ARG, "hrl_gemm_fused: the masked epilogue needs the pre-activation tile");
    HRL_REQUIRE(g.epilogue < HRL_GEMM_EP_STATS || (N % 4 == 0 && g.ldc % 4 == 0 && (reinterpret_cast<uintptr_t>(g.C) & 15) == 0 && g.col_partials),
                HRL_ERR_UNSUPPORTED, "hrl_gemm_fused: the statistics epilogues need N and ldc multiples of 4, a 16-byte aligned C and col_partials");
    const int total_chunks = (int)((K + kChunkK - 1) / kChunkK);
    if (splits < 1) splits = 1;
    if (splits > total_chunks) splits = total_chunks;
    HRL_REQUIRE((splits == 1 && g.segments == 0) || (g.workspace != nullptr && g.bias == nullptr && g.epilogue == HRL_GEMM_EP_STORE), HRL_ERR_WORKSPACE,
                "hrl_gemm_fused: a split-K product needs a workspace of hrl_gemm_workspace_floats() floats, no bias and the plain epilogue");
    const int n_tiles = (int)((N + kMaxN - 1) / kMaxN);
    const int n_widest = (int)(N < kMaxN ? N : kMaxN);
    int n_pad = (n_widest + 15) / 16 * 16;
    if (n_pad > 256) n_pad = (n_pad + 31) / 32 * 32;

    GemmParams p;
    auto operand = [](const HrlGemmOperand &o) {
        GemmOperand r;
        r.ptr = o.ptr; r.ptr2 = o.ptr2; r.p = o.p; r.q = o.q; r.r = o.r; r.ld = o.ld;
        r.kmajor = o.kmajor ? 1 : 0; r.relu = o.relu ? 1 : 0; r.feature_is_row = o.feature_is_row ? 1 : 0; r.packed = o.packed ? 1 : 0;
        return r;
    };
    p.a = operand(g.a);
    p.b = operand(g.b);
    p.bias = g.bias;
    p.M = (int)M; p.N = (int)N; p.K = (int)K;
    p.chunks_per_split = (total_chunks + splits - 1) / splits;
    p.epilogue = g.epilogue;
    p.ep_y = g.ep_y; p.ep_ldy = g.ep_ldy;
    p.ep_scale = g.ep_scale; p.ep_shift = g.ep_shift; p.ep_mean = g.ep_mean; p.ep_rstd = g.ep_rstd;
    p.col_partials = g.col_partials;
    p.debug = g_gemm_debug & 63;
    p.conv_off = g.conv_off; p.conv_mode = g.conv_mode; p.conv_hw = g.conv_hw; p.conv_taps = g.conv_taps; p.conv_cin = g.conv_cin;
    p.conv_cpt = (g.conv_cin + kChunkK - 1) / kChunkK;
    splits = (total_chunks + p.chunks_per_split - 1) / p.chunks_per_split;      // no empty slices
    p.seg_splits = 0;
    p.conv_ones = g.conv_ones_row ? 1 : 0;
    if (g.segments > 0) {              // every (dy, x) pair gets `splits` K slices of its own
        p.seg_splits = splits;
        for (int i = 0; i < g.segments; i++) { p.seg_a[i] = g.seg_a[i]; p.seg_b[i] = g.seg_b[i]; }
        splits *= g.segments;
    }
    if (splits > 1 || g.segments > 0) {
        p.C = g.workspace; p.ldc = N; p.c_split_stride = M * N;
    } else {
        p.C = g.C; p.ldc = g.ldc; p.c_split_stride = 0;
    }
    // a stage: hi | lo halves of fp32-sized elements (3xTF32), or one bf16 copy of each operand
    size_t smem_bytes = 1024 + (size_t)kStages * (g.bf16 ? ((size_t)n_pad + kTileM) * kChunkK * 2
                                                         : 2 * (size_t)n_pad * kChunkK * 4 + 2 * (size_t)kTileM * kChunkK * 4);
    const size_t red_rows = (size_t)kGemmThreads / (size_t)((n_pad - 12) / 4 > 0 ? (n_pad - 12) / 4 : 1);      // copy-out row passes (as the kernel)
    const size_t ep_bytes = 1024 + ((size_t)kTileM * (n_pad + 4) + 2 * red_rows * (size_t)n_pad) * 4;      // epilogue tile + column-sum scratch
    if (smem_bytes < ep_bytes) smem_bytes = ep_bytes;
    const dim3 grid((unsigned)((M + kTileM - 1) / kTileM), (unsigned)n_tiles, (unsigned)splits);
    int st;
    // the tower's forward and input gradients (K-major A, a packed 288-column weight image) run on the kernel that stages A
    // raw, several chunks ahead; weight gradients (both operands stored [K][rows]) on the mma.sync kernel that reads them
    // untransposed
    if (gemm_tower_applies(g)) st = launch_gemm_tower(p, stream);
    else if (gemm_wgrad_applies(g)) st = launch_gemm_wgrad(g, p.chunks_per_split, splits, p.C, p.ldc, p.c_split_stride, p.debug, stream);
    else if (g.bf16) st = launch_gemm_bf16(p, n_pad / 2, grid, smem_bytes, stream);
    else st = launch_gemm_tf32x3(p, n_pad / 2, grid, smem_bytes, stream);
    if (st != HRL_OK) return st;
    HRL_CUDA_CHECK(cudaGetLastError());
    if (splits > 1 && g.C != nullptr) {       // C == NULL: the caller consumes the slice partials itself (hrl_board_fold)
        const long long n = (long long)M * N;
        HRL_REQUIRE(g.ldc == N, HRL_ERR_UNSUPPORTED, "hrl_gemm_fused: split-K output must be dense (ldc == N)");
        int blocks = (int)((n + 255) / 256);
        if (blocks > 1184) blocks = 1184;
        sum_partials_kernel<<<blocks, 256, 0, stream>>>(g.workspace, splits, n, n, g.C);
        HRL_CUDA_CHECK(cudaGetLastError());
    }
    return HRL_OK;
}

extern "C" int hrl_gemm_tf32x3(const float *A, int64_t lda, int32_t a_kmajor, const float *B, int64_t ldb, int32_t b_kmajor,
                               const float *bias, float *C, int64_t ldc, int64_t M, int64_t N, int64_t K, int32_t splits,
                               float *workspace, void *stream) {
    HrlGemmArgs g;
    memset(&g, 0, sizeof(g));
    g.a.ptr = A; g.a.ld = lda; g.a.kmajor = a_kmajor;
    g.b.ptr = B; g.b.ld = ldb; g.b.kmajor = b_kmajor;
    g.bias = bias; g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = K; g.splits = splits; g.workspace = workspace;
    g.epilogue = HRL_GEMM_EP_STORE;
    return hrl_gemm_fused(&g, stream);
}
