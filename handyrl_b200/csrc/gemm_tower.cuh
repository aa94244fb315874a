// The fused tower's forward and input-gradient products (csrc/gemm_tower_kernel.cu): a K-major fp32 A operand times a packed
// 3xTF32 weight image of 257..288 rows, on wgmma with A from registers.  hrl_gemm_fused (csrc/gemm_kernel.cu) routes the
// calls this kernel covers to it, before the weight-gradient kernel and the general wgmma kernel.
#pragma once
#include <cuda_runtime.h>

#include "common.cuh"

namespace hrl {

struct GemmParams;

// true when this kernel computes the call: 3xTF32 (not bf16), no convolution geometry, no segments, one K slice; A K-major,
// not packed, 16-byte aligned sources and rows, no transform or one per reduction index (feature_is_row 0; K <= 512 for one
// source);
// B a packed image with 257 <= N <= 288 (a tile of 288 padded columns)
bool gemm_tower_applies(const HrlGemmArgs &g);

// C = A_op * B^T with the epilogue of p (the wgmma kernel's GemmParams, one K slice); p.debug: 1 = no MMAs, 2 = no A copies
int launch_gemm_tower(const GemmParams &p, cudaStream_t stream);

}  // namespace hrl
