// BatchNorm statistics of a convolution, accumulated in its epilogue ("deferred" finalisation): every CTA adds its
// per-channel (sum, sum of squares) of the values it STORED to the layer's fp64 cells (red.global.add.f64). The BatchNorm
// apply pass that consumes the layer folds the totals into scale / shift in its prologue (b200seg_bn_apply_cells), so
// neither a finaliser launch nor a grid-wide synchronisation sits between the convolution and its consumer. The cells are
// zeroed by the caller once per step. A sum of <= B200SEG_MAX_GRID fp32 partials in fp64 is exact unless their magnitudes
// differ by more than 2^20, so the order of the adds does not change the result in practice. SyncBN keeps the separate
// finaliser (the cross-GPU exchange lives there).
#pragma once
#include <cstdint>

namespace b200seg {

struct BnFoldDev {
  double* accum;            // [2][cout_pad] fp64 cells; nullptr = no deferred statistics
  float* scale;
  float* shift;
  int relu;                 // affine-epilogue mode only (below)
};
// Affine-epilogue mode (evaluation: BatchNorm from running statistics folded into the convolution, accum == nullptr and
// scale != nullptr): the epilogue stores relu?(acc * scale[c] + shift[c] (+ addend)) - one launch per conv + BN (+ residual)
// + ReLU instead of three (b200seg_conv2d_fwd_affine). A convolution bias is folded into shift by the caller.

// Per-CTA statistics of a convolution: one [2][cout_pad] slot per epilogue warp (two warpgroups of four), summed in slot order.
constexpr int kStatSlots = 8;
// Called by ALL threads of the CTA after its last tile (s_stats = [kStatSlots][2][cout_pad] sums in shared memory,
// already synchronised). The consumer of the layer reads the cells after this grid has completed (stream order /
// griddepcontrol.wait), so nothing here waits for the adds.
__device__ __forceinline__ void bn_fold_tail(const BnFoldDev& f, const float* s_stats, int cout_pad) {
  for (int i = threadIdx.x; i < 2 * cout_pad; i += blockDim.x) {
    float v = 0.f;
    for (int s = 0; s < kStatSlots; ++s) v += s_stats[2 * s * cout_pad + i];
    atomicAdd(f.accum + i, (double)v);
  }
}

}  // namespace b200seg
