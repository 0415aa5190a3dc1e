/* Entry points of the TEST library libb200seg_test.so (csrc/test_*.cu): not part of the product ABI (include/b200seg.h). */
#pragma once
#include <stdint.h>
#include "../../include/b200seg.h"
#ifdef __cplusplus
extern "C" {
#endif
/* Slow, obviously-correct CUDA-core direct convolution with the numerics contract of b200seg_conv2d_fwd (bf16 operands,
 * fp32 accumulate, one rounding): the on-device cross-check of the GPU op tests. */
int b200seg_conv2d_fwd_direct(const b200seg_conv_desc* d, const void* x, const void* w_ohwi, const float* bias,
                              void* y, void* stream);
#ifdef __cplusplus
}
#endif
