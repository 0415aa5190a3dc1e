// TEST LIBRARY (libb200seg_test.so, not the product): writes the keep mask of the fused element-wise dropout
// (dropout.cuh) so that tests can hand a reference exactly the bits the BatchNorm kernels used.
#include "ptx.cuh"
#include "launch.h"
#include "../../include/b200seg.h"
#include "probe.h"
#include "dropout.cuh"

namespace b200seg {

__global__ void dropout_keep_mask_kernel(const unsigned long long* __restrict__ seed, int pass, long long n8,
                                         uint8_t* __restrict__ mask) {
  pdl_sync();
  const unsigned long long s = *seed;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < n8; g += (long long)gridDim.x * blockDim.x) {
    const uint32_t keep = dropout_keep8(s, pass, g * 8);
#pragma unroll
    for (int j = 0; j < 8; ++j) mask[g * 8 + j] = (uint8_t)((keep >> j) & 1u);
  }
}

}  // namespace b200seg

using namespace b200seg;

extern "C" int b200seg_dropout_keep_mask(const uint64_t* seed, int32_t pass, int64_t npix, int32_t c, uint8_t* mask,
                                         void* stream) {
  if (!seed || !mask || npix <= 0 || c <= 0 || c % 8) return B200SEG_E_BADARG;
  const long long n8 = npix * (c / 8);
  long long blocks = (n8 + 255) / 256;
  if (blocks > B200SEG_MAX_CTAS * 16) blocks = B200SEG_MAX_CTAS * 16;
  launch_k(dropout_keep_mask_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream,
           (const unsigned long long*)seed, (int)pass, n8, mask);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}
