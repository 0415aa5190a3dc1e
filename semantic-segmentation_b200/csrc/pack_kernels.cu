// Weight repacking from the fp32 OIHW master copies (reference checkpoint layout, SURVEY.md §8b "State") into the
// kernels' bf16 operand layouts; ABI version / build info.
#include "ptx.cuh"
#include "launch.h"
#include "../../include/b200seg.h"
#include <cuda_bf16.h>

namespace b200seg {

__global__ void pack_weight_kernel(const float* __restrict__ w, int O, int I, int K, __nv_bfloat16* __restrict__ ohwi,
                                   __nv_bfloat16* __restrict__ dgrad, int Opad) {
  // No programmatic trigger here: the convolution kernels read their (static) weights BEFORE griddepcontrol.wait, so a
  // kernel that writes weights must be fully complete before any successor starts (plain stream order).
  pdl_wait();
  const int taps = K * K;
  const size_t total = (size_t)O * I * taps;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    // idx enumerates OIHW
    const int t = idx % taps;
    const int i = (idx / taps) % I;
    const int o = idx / ((size_t)taps * I);
    const __nv_bfloat16 v = __float2bfloat16_rn(w[idx]);
    if (ohwi) ohwi[((size_t)o * taps + t) * I + i] = v;
    if (dgrad) dgrad[((size_t)i * taps + (taps - 1 - t)) * Opad + o] = v;   // pad columns stay zero (caller memset)
  }
  __threadfence();   // the packed weights are device-visible before this block exits (successors read them pre-wait)
}

// All weights of the model in ONE launch: block b repacks kPackChunk consecutive OIHW elements of item blk_item[b]
// (fp32 master -> bf16 forward operand [O][taps][I_dst] and data-gradient operand [I_dst][taps flipped][o_pad], and the
// plane-ordered images of both when planes[blk_item[b]] names them).
constexpr int kPackChunk = 4096;
__global__ void __launch_bounds__(256)
pack_weights_kernel(const b200seg_pack_item* __restrict__ items, const b200seg_pack_planes* __restrict__ planes,
                    const int32_t* __restrict__ blk_item, const int32_t* __restrict__ blk_start, int which) {
  pdl_wait();     // no programmatic trigger: see pack_weight_kernel
  const b200seg_pack_item it = items[blk_item[blockIdx.x]];
  const b200seg_pack_planes pl = planes ? planes[blk_item[blockIdx.x]] : b200seg_pack_planes{nullptr, nullptr, 0, 0};
  const float* __restrict__ w = reinterpret_cast<const float*>(it.w_oihw);
  __nv_bfloat16* __restrict__ ohwi = (which & 1) ? reinterpret_cast<__nv_bfloat16*>(it.w_ohwi) : nullptr;
  __nv_bfloat16* __restrict__ dgrad = (which & 2) ? reinterpret_cast<__nv_bfloat16*>(it.w_dgrad) : nullptr;
  __nv_bfloat16* __restrict__ pf = (which & 1) ? reinterpret_cast<__nv_bfloat16*>(pl.fwd) : nullptr;
  __nv_bfloat16* __restrict__ pd = (which & 2) ? reinterpret_cast<__nv_bfloat16*>(pl.dgrad) : nullptr;
  const uint32_t taps = (uint32_t)(it.ksize * it.ksize), I = (uint32_t)it.i, Id = (uint32_t)it.i_dst;
  const uint32_t g_fwd = (Id + 15) / 16 * 2, g_dgrad = ((uint32_t)it.o + 15) / 16 * 2;   // planes per tap
  const uint32_t total = (uint32_t)it.o * I * taps;
  const uint32_t j0 = (uint32_t)blk_start[blockIdx.x];
#pragma unroll 4
  for (uint32_t tt = threadIdx.x; tt < (uint32_t)kPackChunk; tt += 256) {
    const uint32_t idx = j0 + tt;
    if (idx >= total) break;
    const uint32_t t = idx % taps;
    const uint32_t i = (idx / taps) % I;
    const uint32_t o = idx / (taps * I);
    const __nv_bfloat16 v = __float2bfloat16_rn(w[idx]);
    if (ohwi) ohwi[((size_t)o * taps + t) * Id + i] = v;
    if (dgrad) dgrad[((size_t)i * taps + (taps - 1 - t)) * it.o_pad + o] = v;
    // plane-ordered images (include/b200seg.h): [tap][Cin / 8][rows][8]
    if (pf) pf[(((size_t)t * g_fwd + i / 8) * pl.rows_fwd + o) * 8 + i % 8] = v;
    if (pd) pd[(((size_t)(taps - 1 - t) * g_dgrad + o / 8) * pl.rows_dgrad + i) * 8 + o % 8] = v;
  }
  __threadfence();
}

}  // namespace b200seg

using namespace b200seg;

extern "C" int32_t b200seg_pack_chunk(void) { return kPackChunk; }

extern "C" int b200seg_pack_weights(const b200seg_pack_item* items, const int32_t* blk_item, const int32_t* blk_start,
                                    int32_t n_blocks, int32_t which, void* stream) {
  if (!items || !blk_item || !blk_start || n_blocks <= 0 || which < 1 || which > 3) return B200SEG_E_BADARG;
  cudaError_t e = launch_k(pack_weights_kernel, dim3(n_blocks), dim3(256), 0, (cudaStream_t)stream, items,
                           (const b200seg_pack_planes*)nullptr, blk_item, blk_start, (int)which);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_pack_weights_planes(const b200seg_pack_item* items, const b200seg_pack_planes* planes,
                                           const int32_t* blk_item, const int32_t* blk_start, int32_t n_blocks,
                                           int32_t which, void* stream) {
  if (!items || !planes || !blk_item || !blk_start || n_blocks <= 0 || which < 1 || which > 3) return B200SEG_E_BADARG;
  cudaError_t e = launch_k(pack_weights_kernel, dim3(n_blocks), dim3(256), 0, (cudaStream_t)stream, items, planes,
                           blk_item, blk_start, (int)which);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_abi_version(void) { return 1; }
extern "C" const char* b200seg_build_info(void) { return "b200seg sm_90a " __DATE__ " " __TIME__; }

extern "C" int b200seg_pack_weight(const float* w_oihw, int32_t o, int32_t i, int32_t ksize, void* w_ohwi,
                                   void* w_dgrad, int32_t o_pad, void* stream) {
  if (w_dgrad && o_pad < o) return B200SEG_E_BADARG;
  if (!w_oihw || o <= 0 || i <= 0 || (ksize != 1 && ksize != 3)) return B200SEG_E_BADARG;
  const size_t total = (size_t)o * i * ksize * ksize;
  int blocks = (int)((total + 255) / 256);
  if (blocks > B200SEG_MAX_CTAS * 8) blocks = B200SEG_MAX_CTAS * 8;
  launch_k(pack_weight_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, w_oihw, o, i, ksize,
           (__nv_bfloat16*)w_ohwi, (__nv_bfloat16*)w_dgrad, o_pad);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}
