// Shared pieces of the two forward / data-gradient convolution kernels (conv_igemm.cu, conv3x3_halo.cu):
//   * the MMA of one K = 16 step over all N columns of a warpgroup tile (64 rows x 16 * nb16 columns), and
//   * the epilogue of a warpgroup tile straight from the wgmma accumulator fragment (ptx.cuh).
#pragma once
#include <cuda_bf16.h>
#include "ptx.cuh"
#include "bn_fold.cuh"

namespace b200seg {

// Columns [0, 16 * nb16) of acc (NB = 16-column blocks the kernel build holds): one MMA per 64-column group, narrower for
// the tail. b64 = descriptor distance between 64-column groups of the B operand (16-byte units).
template <int NB, int TA, int TB>
__device__ __forceinline__ void wgmma_row(float (&acc)[NB * 8], int nb16, uint64_t a, uint64_t b, uint32_t b64,
                                          uint32_t scale_d) {
#pragma unroll
  for (int j = 0; j < NB; j += 4) {
    const uint64_t bj = b + (uint64_t)((j / 4) * b64);
    if (j + 4 <= nb16) wgmma_n64<TA, TB>(&acc[8 * j], a, bj, scale_d);
    else if (j + 3 == nb16) wgmma_n48<TA, TB>(&acc[8 * j], a, bj, scale_d);
    else if (j + 2 == nb16) wgmma_n32<TA, TB>(&acc[8 * j], a, bj, scale_d);
    else if (j + 1 == nb16) wgmma_n16<TA, TB>(&acc[8 * j], a, bj, scale_d);
  }
}

// Sum over the 8 rows a warp holds per column pair (lanes with equal lane % 4): afterwards lanes 0-3 hold the totals.
__device__ __forceinline__ float col_reduce(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  return v;
}

struct ConvEpi {
  void* y;
  const float* bias;                  // nullable
  const __nv_bfloat16* addend;        // nullable
  int y_ld, addend_ld, out_fp32, Cout, emit_stats, cout_pad;
};

// Epilogue of a warpgroup tile (columns n0 + [0, 16 * nb16); the thread's two rows at pix[r]): bias, BN affine, addend,
// ReLU, store; sums / sums of squares of the STORED values into this warp's my_stats[2][cout_pad].
template <int NB>
__device__ __forceinline__ void conv_epilogue(const float (&acc)[NB * 8], int nb16, int n0, const bool (&valid)[2],
                                              const size_t (&pix)[2], const ConvEpi& e, const BnFoldDev& fold,
                                              float* my_stats, uint32_t lane) {
  const bool affine = fold.accum == nullptr && fold.scale != nullptr;   // evaluation: BN folded into the epilogue
#pragma unroll
  for (int c = 0; c < 2 * NB; ++c) {
    if (c >= 2 * nb16 || n0 + 8 * c >= e.Cout) break;     // warp-uniform
    const int col = n0 + 8 * c + 2 * (int)(lane & 3);
    const bool cv[2] = {col < e.Cout, col + 1 < e.Cout};
    float bi[2] = {0.f, 0.f}, sc[2] = {1.f, 1.f}, sh[2] = {0.f, 0.f};
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      if (!cv[q]) continue;
      if (e.bias) bi[q] = __ldg(e.bias + col + q);
      if (affine) { sc[q] = __ldg(fold.scale + col + q); sh[q] = __ldg(fold.shift + col + q); }
    }
    float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float v[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        v[q] = acc[4 * c + 2 * r + q] + bi[q];
        if (affine && cv[q]) v[q] = v[q] * sc[q] + sh[q];
        if (e.addend != nullptr && valid[r] && cv[q]) v[q] += __bfloat162float(e.addend[pix[r] * e.addend_ld + col + q]);
        if (affine && fold.relu) v[q] = fmaxf(v[q], 0.f);
      }
      if (!valid[r]) continue;
      if (e.out_fp32) {
        float* dst = reinterpret_cast<float*>(e.y) + pix[r] * e.y_ld + col;
        if (cv[0]) dst[0] = v[0];
        if (cv[1]) dst[1] = v[1];
        continue;
      }
      const uint32_t pk = pack_bf16x2(v[0], v[1]);
      __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(e.y) + pix[r] * e.y_ld + col;
      if (cv[1]) *reinterpret_cast<uint32_t*>(dst) = pk;
      else if (cv[0]) dst[0] = __float2bfloat16_rn(v[0]);
      const float lo = cv[0] ? bf16_lo(pk) : 0.f, hi = cv[1] ? bf16_hi(pk) : 0.f;
      s1[0] += lo; s1[1] += hi;
      s2[0] += lo * lo; s2[1] += hi * hi;
    }
    if (e.emit_stats) {
#pragma unroll
      for (int q = 0; q < 2; ++q) { s1[q] = col_reduce(s1[q]); s2[q] = col_reduce(s2[q]); }
      if (lane < 4) {
        my_stats[col] += s1[0];
        my_stats[col + 1] += s1[1];
        my_stats[e.cout_pad + col] += s2[0];
        my_stats[e.cout_pad + col + 1] += s2[1];
      }
    }
  }
}

// Slots of the previous MMA group, freed once it has completed (wgmma_wait<1> after the next commit).
struct PendingRelease {
  uint64_t* bar0 = nullptr;
  uint64_t* bar1 = nullptr;
  __device__ __forceinline__ void release(bool leader) {
    if (leader) {
      if (bar0) mbar_arrive(bar0);
      if (bar1) mbar_arrive(bar1);
    }
    bar0 = bar1 = nullptr;
  }
};

}  // namespace b200seg
