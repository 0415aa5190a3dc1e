// TEST LIBRARY (libb200seg_test.so, not the product): a CUDA-core direct convolution with the same numerics contract as
// the wgmma path (bf16 operands, fp32 accumulate, one final rounding), the on-device cross-check of tests/test_gpu_ops.py.
#include "ptx.cuh"
#include "launch.h"
#include "../../include/b200seg.h"
#include "probe.h"
#include <cuda_bf16.h>

namespace b200seg {

__global__ void direct_conv_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                   const float* __restrict__ bias, void* __restrict__ y, int N, int H, int W, int Cin,
                                   int Cout, int K, int S, int P, int Ho, int Wo, int x_ld, int y_ld, int out_fp32) {
  pdl_sync();
  const size_t total = (size_t)N * Ho * Wo * Cout;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int co = idx % Cout;
    const size_t pix = idx / Cout;
    const int wo = pix % Wo;
    const int ho = (pix / Wo) % Ho;
    const int n = pix / ((size_t)Wo * Ho);
    float acc = 0.f;
    for (int kh = 0; kh < K; ++kh) {
      const int hi = ho * S + kh - P;
      if (hi < 0 || hi >= H) continue;
      for (int kw = 0; kw < K; ++kw) {
        const int wi = wo * S + kw - P;
        if (wi < 0 || wi >= W) continue;
        const __nv_bfloat16* xp = x + (((size_t)n * H + hi) * W + wi) * x_ld;
        const __nv_bfloat16* wp = w + ((size_t)co * K * K + kh * K + kw) * Cin;
        for (int ci = 0; ci < Cin; ++ci) acc += __bfloat162float(xp[ci]) * __bfloat162float(wp[ci]);
      }
    }
    if (bias) acc += bias[co];
    if (out_fp32) reinterpret_cast<float*>(y)[pix * y_ld + co] = acc;
    else reinterpret_cast<__nv_bfloat16*>(y)[pix * y_ld + co] = __float2bfloat16_rn(acc);
  }
}

}  // namespace b200seg

using namespace b200seg;

extern "C" int b200seg_conv2d_fwd_direct(const b200seg_conv_desc* d, const void* x, const void* w_ohwi,
                                         const float* bias, void* y, void* stream) {
  if (!d || !x || !w_ohwi || !y) return B200SEG_E_BADARG;
  const int Ho = (d->h + 2 * d->pad - d->ksize) / d->stride + 1;
  const int Wo = (d->w + 2 * d->pad - d->ksize) / d->stride + 1;
  const size_t total = (size_t)d->n * Ho * Wo * d->cout;
  int blocks = (int)((total + 255) / 256);
  if (blocks > B200SEG_MAX_CTAS * 16) blocks = B200SEG_MAX_CTAS * 16;
  launch_k(direct_conv_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x,
           (const __nv_bfloat16*)w_ohwi, d->has_bias ? bias : nullptr, y, d->n, d->h, d->w, d->cin, d->cout, d->ksize,
           d->stride, d->pad, Ho, Wo, d->x_ld, d->y_ld, d->out_fp32);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}

