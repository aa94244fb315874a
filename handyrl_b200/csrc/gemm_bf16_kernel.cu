// The bf16 form of the tensor-core GEMM (HrlGemmArgs.bf16, an opt-in of the learner: train_args['tensor_cores'] = 'bf16').
// Same body as the 3xTF32 kernels (csrc/gemm_common.cuh), same widths and operand layouts, so that every product the default
// path runs has a bf16 form: both operands are rounded to bf16 after their fp32 transform and a chunk of 32 reduction elements
// is 2 wgmma .bf16 per warpgroup (3xTF32: 12) on a quarter of the shared-memory bytes.
#define HRL_GEMM_KERNEL gemm_bf16_kernel
#define HRL_GEMM_BF16 true
#define HRL_GEMM_LAUNCH launch_gemm_bf16
#include "gemm_common.cuh"
