// The bf16 form of the tensor-core GEMM (HrlGemmArgs.bf16, an opt-in of the learner: train_args['tensor_cores'] = 'bf16').
// Same body as the 3xTF32 kernels (csrc/gemm_common.cuh), same widths and operand layouts, so that every product the default
// path runs has a bf16 form: both operands are rounded to bf16 after their fp32 transform and a chunk of 32 reduction elements
// is 2 wgmma .bf16 per warpgroup (3xTF32: 12) on a quarter of the shared-memory bytes.
#define HRL_GEMM_KERNEL gemm_bf16_kernel
#define HRL_GEMM_BF16 true
#include "gemm_common.cuh"

namespace hrl {

template <bool A_K, bool B_K, bool PACKED, int NW>
static int launch_bf16(const GemmParams &p, dim3 grid, size_t smem_bytes, cudaStream_t stream) {
    HRL_CUDA_CHECK(cudaFuncSetAttribute(gemm_bf16_kernel<A_K, B_K, PACKED, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    gemm_bf16_kernel<A_K, B_K, PACKED, NW><<<grid, kGemmThreads, smem_bytes, stream>>>(p);
    return HRL_OK;
}

template <int NW>
static int launch_bf16_width(const GemmParams &p, dim3 grid, size_t smem_bytes, cudaStream_t stream) {
    if (p.b.packed) return p.a.kmajor ? launch_bf16<true, true, true, NW>(p, grid, smem_bytes, stream)
                                      : launch_bf16<false, true, true, NW>(p, grid, smem_bytes, stream);
    if (p.a.kmajor) return p.b.kmajor ? launch_bf16<true, true, false, NW>(p, grid, smem_bytes, stream)
                                      : launch_bf16<true, false, false, NW>(p, grid, smem_bytes, stream);
    return p.b.kmajor ? launch_bf16<false, true, false, NW>(p, grid, smem_bytes, stream)
                      : launch_bf16<false, false, false, NW>(p, grid, smem_bytes, stream);
}

int launch_gemm_bf16(const GemmParams &p, int nw, dim3 grid, size_t smem_bytes, cudaStream_t stream) {
    switch (nw) {                 // the MMA widths of the 3xTF32 dispatch (csrc/gemm_kernel.cu)
    case 8: return launch_bf16_width<8>(p, grid, smem_bytes, stream);
    case 16: return launch_bf16_width<16>(p, grid, smem_bytes, stream);
    case 24: return launch_bf16_width<24>(p, grid, smem_bytes, stream);
    case 32: return launch_bf16_width<32>(p, grid, smem_bytes, stream);
    case 40: return launch_bf16_width<40>(p, grid, smem_bytes, stream);
    case 48: return launch_bf16_width<48>(p, grid, smem_bytes, stream);
    case 56: return launch_bf16_width<56>(p, grid, smem_bytes, stream);
    case 64: return launch_bf16_width<64>(p, grid, smem_bytes, stream);
    case 72: return launch_bf16_width<72>(p, grid, smem_bytes, stream);
    case 80: return launch_bf16_width<80>(p, grid, smem_bytes, stream);
    case 88: return launch_bf16_width<88>(p, grid, smem_bytes, stream);
    case 96: return launch_bf16_width<96>(p, grid, smem_bytes, stream);
    case 104: return launch_bf16_width<104>(p, grid, smem_bytes, stream);
    case 112: return launch_bf16_width<112>(p, grid, smem_bytes, stream);
    case 120: return launch_bf16_width<120>(p, grid, smem_bytes, stream);
    case 128: return launch_bf16_width<128>(p, grid, smem_bytes, stream);
    case 144: return launch_bf16_width<144>(p, grid, smem_bytes, stream);
    default: HRL_REQUIRE(false, HRL_ERR_BAD_ARG, "hrl_gemm_fused: no bf16 kernel for an MMA width of %d columns", nw);
    }
}

}  // namespace hrl
