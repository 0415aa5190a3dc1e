// BatchNorm statistics finalisation folded into the tail of the producing convolution ("last CTA done"):
// every CTA adds its per-channel (sum, sum of squares) of the values it STORED to a per-layer fp64 accumulator
// (red.global.add.f64: order-independent up to fp64 rounding, 1e-16), takes a ticket, and the CTA that draws the last
// ticket turns the totals into scale / shift / mean / invstd (+ the batch statistics for the running-stat update) and
// clears accumulator and ticket for the next launch. Replaces one bn_finalize launch (a pure latency chain of ~10 us
// between every convolution and its consumer) per BatchNorm layer and scale pass; arithmetic identical to
// bn_finalize_kernel (bn_kernels.cu). SyncBN keeps the separate finaliser (the cross-GPU exchange lives there).
// Deferred variant (counter == nullptr, the default of the training step): the CTAs only add their sums to the cells; the
// BatchNorm apply pass that consumes the layer folds the totals in its prologue (b200seg_bn_apply_cells), so neither a
// finaliser launch nor a last-CTA tail sits between the convolution and its consumer. The cells are zeroed by the caller
// once per step. A sum of <= B200SEG_MAX_GRID fp32 partials in fp64 is exact unless their magnitudes differ by more than 2^20, so
// the order of the adds does not change the result in practice.
#pragma once
#include <cstdint>

namespace b200seg {

struct BnFoldDev {
  double* accum;            // [2][cout_pad] fp64, all zero between launches; nullptr = disabled
  unsigned* counter;        // zero between launches
  const float* gamma;
  const float* beta;
  float* scale;
  float* shift;
  float* mean;
  float* invstd;
  float* batch_out;         // [2*C] = [mean | unbiased var] or nullptr
  float* running_mean;      // nullable (then batch_out carries the deferred update)
  float* running_var;
  long long* nbt;
  float eps, momentum, count;
  int C;
  int relu;                 // affine-epilogue mode only (below)
};
// Affine-epilogue mode (evaluation: BatchNorm from running statistics folded into the convolution, accum == nullptr and
// scale != nullptr): the epilogue stores relu?(acc * scale[c] + shift[c] (+ addend)) - one launch per conv + BN (+ residual)
// + ReLU instead of three (b200seg_conv2d_fwd_affine). A convolution bias is folded into shift by the caller.

// Per-CTA statistics of a convolution: one [2][cout_pad] slot per epilogue warp (two warpgroups of four), summed in slot order.
constexpr int kStatSlots = 8;
// Called by ALL threads of the CTA after its last tile (s_stats = [kStatSlots][2][cout_pad] sums in shared memory,
// already synchronised; s_ticket_p = one free word of the CTA's dynamic shared memory). Returns after the layer's parameters are written if this CTA drew the last ticket.
__device__ __forceinline__ void bn_fold_tail(const BnFoldDev& f, const float* s_stats, int cout_pad,
                                             volatile unsigned* s_ticket_p) {
  const int nthreads = blockDim.x;
  for (int i = threadIdx.x; i < 2 * cout_pad; i += nthreads) {
    float v = 0.f;
    for (int s = 0; s < kStatSlots; ++s) v += s_stats[2 * s * cout_pad + i];
    atomicAdd(f.accum + i, (double)v);
  }
  // Only the threads that added to the accumulator fence (their adds must be visible before the ticket is drawn): a
  // fence in the epilogue threads would also wait for their outstanding output stores, which nobody here depends on.
  // Deferred mode (counter == nullptr): the consumer of the layer (bn_apply_kernel's prologue) turns the totals into the
  // parameters; nothing to wait for here - the adds are complete when this grid is (stream order / griddepcontrol.wait).
  if (f.counter == nullptr) return;
  if ((int)threadIdx.x < 2 * cout_pad) __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) *s_ticket_p = atomicAdd(f.counter, 1u);
  __syncthreads();
  if (*s_ticket_p != gridDim.x - 1) return;
  __threadfence();                       // the other CTAs' accumulator updates are visible (they fenced before their ticket)
  const double count = (double)f.count;
  for (int c = threadIdx.x; c < cout_pad; c += nthreads) {
    const double s1 = __ldcg(f.accum + c), s2 = __ldcg(f.accum + cout_pad + c);
    f.accum[c] = 0.0;
    f.accum[cout_pad + c] = 0.0;
    if (c >= f.C) continue;
    const double mean = s1 / count;
    double var = s2 / count - mean * mean;
    if (var < 0.0) var = 0.0;
    const float invstd = (float)(1.0 / sqrt(var + (double)f.eps));
    const float g_ = f.gamma ? f.gamma[c] : 1.f, b_ = f.beta ? f.beta[c] : 0.f;
    f.scale[c] = g_ * invstd;
    f.shift[c] = b_ - (float)mean * g_ * invstd;
    f.mean[c] = (float)mean;
    f.invstd[c] = invstd;
    const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
    if (f.running_mean) {
      f.running_mean[c] = (1.f - f.momentum) * f.running_mean[c] + f.momentum * (float)mean;
      f.running_var[c] = (1.f - f.momentum) * f.running_var[c] + f.momentum * (float)unbiased;
    }
    if (f.batch_out) {
      f.batch_out[c] = (float)mean;
      f.batch_out[f.C + c] = (float)unbiased;
    }
  }
  if (threadIdx.x == 0) {
    *f.counter = 0u;
    if (f.nbt) *f.nbt += 1;
  }
}

}  // namespace b200seg
