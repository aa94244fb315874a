// The weight-gradient product of the fused tower on warp-level mma.sync (csrc/gemm_wgrad_kernel.cu): both operands stored
// [K][rows] ("MN-major", kmajor = 0), reduced over K.  hrl_gemm_fused (csrc/gemm_kernel.cu) routes the calls this kernel
// covers to it and every other call to the wgmma kernel.
#pragma once
#include <cuda_runtime.h>

#include "common.cuh"

namespace hrl {

// true when this kernel computes the call: both operands MN-major and not packed, per-row (or no) operand transforms, no
// second source for B, 16-byte aligned sources and rows, no convolution geometry, no segments, the plain epilogue, no bias,
// 3xTF32 (not bf16)
bool gemm_wgrad_applies(const HrlGemmArgs &g);

// C[split] (ldc, split stride c_split_stride) = the product over the 32-element chunks [split * chunks_per_split, ...) of K;
// debug: 1 = no MMAs, 2 = no operand copies (profiling)
int launch_gemm_wgrad(const HrlGemmArgs &g, int chunks_per_split, int splits, float *C, long long ldc, long long c_split_stride,
                      int debug, cudaStream_t stream);

}  // namespace hrl
