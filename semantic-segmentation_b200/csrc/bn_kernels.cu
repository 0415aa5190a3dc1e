// Training-mode BatchNorm around the tensor-core convolutions (reference: Norm2d -> torch.nn.BatchNorm2d /
// apex SyncBatchNorm, network/mynn.py:18-24; eps 1e-5, momentum 0.1, biased variance to normalise, unbiased for the
// running estimate). All kernels are HBM-bound streaming passes over NHWC bf16 with 16-byte vector accesses.
//
//   forward : conv epilogue partials -> bn_finalize (scale/shift/mean/invstd + running stats) -> bn_apply
//             z = relu?( (y*scale + shift [+ residual]) ) [* post_scale[n][c]]          (Dropout2d folded in post_scale)
//   backward: bn_bwd_reduce (sum g, sum g*xhat per channel; g = dz * (mask>0)) -> bn_bwd_finalize (dgamma, dbeta, c1, c2)
//             -> bn_bwd_apply  dy = gamma*invstd*(g - c1 - xhat*c2)  [and g written out for the residual branch]
#include "ptx.cuh"
#include "launch.h"
#include "../../include/b200seg.h"
#include "vec.cuh"
#include "conv_common.h"
#include <cstring>

namespace b200seg {

// ------------------------------------------------------------------------------------------------ forward
constexpr int kFinSlices = 16;
// Sum rows slice, slice+16, ... of a [G][pitch] partial table for channel c (first statistic at +c, second at +off2+c).
__device__ __forceinline__ void fold_rows(const float* __restrict__ partials, int G, int pitch, int off2, int c,
                                          int slice, double& a1, double& a2) {
  int g = slice;
  for (; g + 3 * kFinSlices < G; g += 4 * kFinSlices) {
    const float* p0 = partials + (size_t)g * pitch + c;
    const float u0 = p0[0], v0 = p0[off2];
    const float u1 = p0[(size_t)kFinSlices * pitch], v1 = p0[(size_t)kFinSlices * pitch + off2];
    const float u2 = p0[(size_t)2 * kFinSlices * pitch], v2 = p0[(size_t)2 * kFinSlices * pitch + off2];
    const float u3 = p0[(size_t)3 * kFinSlices * pitch], v3 = p0[(size_t)3 * kFinSlices * pitch + off2];
    a1 += (double)u0; a1 += (double)u1; a1 += (double)u2; a1 += (double)u3;
    a2 += (double)v0; a2 += (double)v1; a2 += (double)v2; a2 += (double)v3;
  }
  for (; g < G; g += kFinSlices) {
    a1 += (double)partials[(size_t)g * pitch + c];
    a2 += (double)partials[(size_t)g * pitch + off2 + c];
  }
}

// ---------------------------------------------------------------- SyncBN exchange over NVLink peer memory
// Replaces apex.parallel.SyncBatchNorm's per-layer all_gather / all_reduce (SURVEY.md §2b collective C2, config.py:216-225)
// with a one-shot exchange fused into the finalisers: every rank stores its two per-channel sums (fp64) straight into
// every peer's mailbox (P2P stores through NVSwitch), publishes a step-numbered flag with release semantics, waits for
// the flags of all ranks in its OWN mailbox and folds the ranks in rank order (bitwise identical result on every GPU).
// mail[parity][exchange][rank][2][C] doubles; flags[exchange][rank][block] uint32 (monotonic step numbers).
struct SyncArgs {
  double* const* mail_peers;      // device array [world] of every rank's mailbox base (own entry = local pointer)
  unsigned* const* flag_peers;    // device array [world] of every rank's flag base
  const unsigned* step;           // device step counter (incremented once per training step)
  long long mail_off;             // this exchange's offset inside one parity half, in doubles
  long long parity_stride;        // doubles per parity half
  int flag_off;                   // this exchange's offset in the flag array
  int world, rank;
  volatile int* beacon;           // optional host-mapped int32[8]: {entered: flag_off, step, 0, 0, left: flag_off, step}
};

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ double ld_volatile_f64(const double* p) {
  double v;
  asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

// The exchange is split over two kernels so that NOTHING that waits for a peer holds more than one warp of an SM:
//   sync_post  (tail of the finaliser, 512-thread blocks): store my sums into every peer's mailbox, publish the flags,
//              exit - never waits;
//   sync_wait_fold (bn_sync_finish_kernel / bn_bwd_sync_finish_kernel: ONE WARP per 32 channels, no shared memory):
//              poll my own flags, fold the ranks in rank order, write the layer's parameters.
// Why: a persistent tensor-core convolution takes a whole SM per CTA (up to 60 K registers, 226 KB of shared memory) and
// owns its tiles statically. A 512-thread spinning finaliser (27 K registers + 8 KB) on one SM keeps that SM's CTA of a
// convolution on ANOTHER stream from starting, so that convolution never completes - and when the peer is waiting for
// exactly that convolution's statistics while its own spinner blocks the convolution this rank waits for, the two GPUs
// deadlock (observed at 1024x2048: rank 0 spinning in the 1.0x stem exchange, rank 1 in the 0.5x attention head's).
// A one-warp waiter (<= 1.3 K registers, 1 KB reserved shared memory) fits next to any CTA of the library (the
// planners leave B200SEG_SYNC_SMEM_RESERVE bytes free per SM in SyncBN mode), so every launched kernel whose stream
// predecessors are done can always be scheduled, which is what the ordering argument in DESIGN.md needs.
__device__ __forceinline__ void sync_post(const SyncArgs& sy, int C, int c, bool owner, double s1, double s2) {
  const unsigned step = *sy.step;
  const long long base = (long long)(step & 1u) * sy.parity_stride + sy.mail_off;
  if (sy.beacon && blockIdx.x == 0 && threadIdx.x == 0) {   // post-mortem aid: which exchange this rank posted last
    sy.beacon[0] = sy.flag_off;
    sy.beacon[1] = (int)step;
  }
  if (owner) {
    for (int r = 0; r < sy.world; ++r) {
      double* dst = sy.mail_peers[r] + base + (long long)sy.rank * 2 * C;
      dst[c] = s1;
      dst[C + c] = s2;
    }
    __threadfence_system();
  }
  __syncthreads();
  const int nblk = gridDim.x;
  if (threadIdx.x == 0)
    for (int r = 0; r < sy.world; ++r)
      st_release_sys(sy.flag_peers[r] + sy.flag_off + sy.rank * nblk + blockIdx.x, step);
}

// One warp, lane = channel blockIdx.x * 32 + lane. Returns the sums over all ranks (rank order: bitwise identical on
// every GPU) for lanes with c < C.
__device__ __forceinline__ void sync_wait_fold(const SyncArgs& sy, int C, int c, double& s1, double& s2) {
  const unsigned step = *sy.step;
  const long long base = (long long)(step & 1u) * sy.parity_stride + sy.mail_off;
  const int nblk = gridDim.x;
  const unsigned* myflags = sy.flag_peers[sy.rank] + sy.flag_off + blockIdx.x;
  const double* mymail = sy.mail_peers[sy.rank] + base;
  const int lane = threadIdx.x;
  // lane r < world polls rank r's flag; flags are monotonic step numbers: a peer that is already one step ahead (it wrote
  // step + 1 into the OTHER parity half) must not be waited for, so compare by order, not by equality
  if (lane < sy.world) {
    unsigned spins = 0;
    unsigned long long t0 = 0;
    while ((int)(ld_acquire_sys(myflags + lane * nblk) - step) < 0) {
      if ((++spins & 0xFFFFu) == 0) {            // a lost peer traps after 180 s instead of hanging the GPU
        unsigned long long now;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(now));
        if (t0 == 0) t0 = now;
        else if (now - t0 > 180000000000ull) __trap();
      }
    }
  }
  __syncwarp();
  __threadfence_system();
  double t1 = 0.0, t2 = 0.0;
  if (c < C) {
    for (int r = 0; r < sy.world; ++r) {
      t1 += ld_volatile_f64(mymail + (long long)r * 2 * C + c);
      t2 += ld_volatile_f64(mymail + (long long)r * 2 * C + C + c);
    }
  }
  s1 = t1;
  s2 = t2;
  if (sy.beacon && blockIdx.x == 0 && lane == 0) {   // ... and which one it completed last
    sy.beacon[4] = sy.flag_off;
    sy.beacon[5] = (int)step;
  }
}

// scale / shift / mean / invstd (+ running statistics or the deferred batch statistics) of channel c from the totals
__device__ __forceinline__ void bn_write_params(double s1, double s2, float count, int c, int C, const float* gamma,
                                                const float* beta, float eps, float momentum, float* running_mean,
                                                float* running_var, float* scale, float* shift, float* mean_out,
                                                float* invstd_out, float* batch_stats_out) {
  const double mean = s1 / count;
  double var = s2 / count - mean * mean;
  if (var < 0.0) var = 0.0;
  const float invstd = (float)(1.0 / sqrt(var + (double)eps));
  const float g_ = gamma ? gamma[c] : 1.f, b_ = beta ? beta[c] : 0.f;
  scale[c] = g_ * invstd;
  shift[c] = b_ - (float)mean * g_ * invstd;
  mean_out[c] = (float)mean;
  invstd_out[c] = invstd;
  const double unbiased = count > 1.f ? var * (double)count / ((double)count - 1.0) : var;
  if (running_mean) {
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mean;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
  if (batch_stats_out) {   // deferred running-stat update (bn_running_update_kernel): [mean C | unbiased var C]
    batch_stats_out[c] = (float)mean;
    batch_stats_out[C + c] = (float)unbiased;
  }
}

// SyncBN, second half: one warp per 32 channels waits for every rank's sums and writes the layer's parameters. Its
// dependents (the BN apply pass ...) are released only AFTER the exchange: a successor that became resident early (PDL)
// would hold registers / shared memory on many SMs while this warp waits for a peer.
__global__ void __launch_bounds__(32)
bn_sync_finish_kernel(int C, float count, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                      float momentum, float* __restrict__ running_mean, float* __restrict__ running_var,
                      float* __restrict__ scale, float* __restrict__ shift, float* __restrict__ mean_out,
                      float* __restrict__ invstd_out, float* __restrict__ batch_stats_out, const SyncArgs sy) {
  pdl_wait();
  const int c = blockIdx.x * 32 + threadIdx.x;
  double s1, s2;
  sync_wait_fold(sy, C, c, s1, s2);
  pdl_launch();
  if (c < C)
    bn_write_params(s1, s2, count * (float)sy.world, c, C, gamma, beta, eps, momentum, running_mean, running_var, scale,
                    shift, mean_out, invstd_out, batch_stats_out);
}

__global__ void __launch_bounds__(32 * kFinSlices)
bn_finalize_kernel(const float* __restrict__ partials, int G, int C, int Cpad, float count,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                   float momentum, float* __restrict__ running_mean, float* __restrict__ running_var,
                                   long long* __restrict__ num_batches_tracked, float* __restrict__ scale,
                                   float* __restrict__ shift, float* __restrict__ mean_out,
                                   float* __restrict__ invstd_out, float* __restrict__ batch_stats_out,
                                   const SyncArgs sy) {
  pdl_wait();
  pdl_launch();     // the only dependent in SyncBN mode is the one-warp bn_sync_finish_kernel (it never blocks anything)
  // block = 32 channels x 16 slices of the G partial rows (coalesced 128-byte reads, four independent rows in flight per
  // thread: the kernel is a pure latency chain otherwise), then a fixed-order fold -> deterministic
  __shared__ double sh1[kFinSlices][32], sh2[kFinSlices][32];
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  if (blockIdx.x == 0 && threadIdx.x == 0 && num_batches_tracked) *num_batches_tracked += 1;
  double a1 = 0.0, a2 = 0.0;
  if (c < C) fold_rows(partials, G, 2 * Cpad, Cpad, c, slice, a1, a2);
  sh1[slice][lane] = a1;
  sh2[slice][lane] = a2;
  __syncthreads();
  double s1 = 0.0, s2 = 0.0;
  if (slice == 0 && c < C)
    for (int k = 0; k < kFinSlices; ++k) { s1 += sh1[k][lane]; s2 += sh2[k][lane]; }
  if (sy.world > 1) {            // SyncBN: post my sums to every rank; bn_sync_finish_kernel completes the layer
    sync_post(sy, C, c, slice == 0 && c < C, s1, s2);
    return;
  }
  if (slice != 0 || c >= C) return;
  bn_write_params(s1, s2, count, c, C, gamma, beta, eps, momentum, running_mean, running_var, scale, shift, mean_out,
                  invstd_out, batch_stats_out);
}

// Running-statistics update of ALL BatchNorm layers of a step in one pass. The scale passes of the multi-scale step run
// concurrently on different streams, so their finalisers only store the batch statistics; this kernel then applies the
// momentum updates in the reference's order (low-resolution pass first, network/ocrnet.py:278-281):
//   r <- (1-m) r + m b_pass0 ;  r <- (1-m) r + m b_pass1.   running / batch buffers share one flat layout.
__global__ void bn_running_update_kernel(float* __restrict__ running, const float* __restrict__ b0,
                                         const float* __restrict__ b1, long long n, float momentum,
                                         long long* __restrict__ nbt, int n_layers, int n_passes) {
  pdl_sync();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    float r = running[i];
    r = (1.f - momentum) * r + momentum * b0[i];
    if (b1) r = (1.f - momentum) * r + momentum * b1[i];
    running[i] = r;
  }
  if (nbt && i < n_layers) nbt[i] += n_passes;
}

// Multi-tensor SGD with momentum and weight decay (torch.optim.SGD semantics, loss/optimizer.py:43-60): one launch for all
// parameters of a group. Block b updates kSgdChunk consecutive elements of items[blk_item[b]].
constexpr int kSgdChunk = 4096;
__global__ void __launch_bounds__(256)
sgd_step_kernel(const b200seg_sgd_item* __restrict__ items, const int32_t* __restrict__ blk_item,
                const int32_t* __restrict__ blk_start, float lr, float momentum, float dampening, float weight_decay,
                int nesterov, int first_step) {
  pdl_sync();
  const b200seg_sgd_item it = items[blk_item[blockIdx.x]];
  float* __restrict__ p = reinterpret_cast<float*>(it.param);
  const float* __restrict__ g = reinterpret_cast<const float*>(it.grad);
  float* __restrict__ m = reinterpret_cast<float*>(it.momentum_buf);
  const long long j0 = blk_start[blockIdx.x];
#pragma unroll 4
  for (int t = threadIdx.x; t < kSgdChunk; t += 256) {
    const long long j = j0 + t;
    if (j >= it.numel) break;
    const float w = p[j];
    float d = g[j] + weight_decay * w;
    if (momentum != 0.f) {
      const float b = first_step ? d : momentum * m[j] + (1.f - dampening) * d;
      m[j] = b;
      d = nesterov ? d + momentum * b : b;
    }
    p[j] = w - lr * d;
  }
}

// dst += src (fp32): folds the low-resolution pass' private parameter-gradient buffer into the step's gradient.
__global__ void accum_f32_kernel(float* __restrict__ dst, const float* __restrict__ src, long long n4) {
  pdl_sync();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 a = reinterpret_cast<float4*>(dst)[i];
    const float4 b = reinterpret_cast<const float4*>(src)[i];
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    reinterpret_cast<float4*>(dst)[i] = a;
  }
}

// Eval-mode: scale/shift from the running statistics.
__global__ void bn_eval_params_kernel(int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                      const float* __restrict__ running_mean, const float* __restrict__ running_var,
                                      float* __restrict__ scale, float* __restrict__ shift) {
  pdl_sync();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float invstd = rsqrtf(running_var[c] + eps);
  const float g_ = gamma[c];
  scale[c] = g_ * invstd;
  shift[c] = beta[c] - running_mean[c] * g_ * invstd;
}

// Deferred finalisation of the producing convolution's statistics (bn_fold.cuh, counter == nullptr): every block of the
// apply pass turns the fp64 totals into scale / shift for itself; block 0 also publishes the layer's parameters (the
// backward pass reads mean / invstd, fuse layers scale / shift) and the batch / running statistics. cells == nullptr:
// scale / shift come from bn_finalize (SyncBN, evaluation, statistics that did not come from a convolution epilogue).
struct BnLazy {
  const double* cells;      // [2][cpad] = per-channel sum | sum of squares
  int cpad;
  float count, eps, momentum;
  const float* gamma;
  const float* beta;
  float* mean_out;          // [C] each; scale / shift outputs are the kernel's own scale / shift arguments
  float* invstd_out;
  float* batch_stats_out;   // [2*C] or nullptr
  float* running_mean;      // nullable
  float* running_var;
  long long* nbt;
};

__global__ void __launch_bounds__(256)
bn_apply_kernel(const __nv_bfloat16* __restrict__ y, int y_ld, float* __restrict__ scale,
                float* __restrict__ shift, const __nv_bfloat16* __restrict__ res, int res_ld,
                const float* __restrict__ post_scale, int relu, __nv_bfloat16* __restrict__ z, int z_ld,
                long long npix, int hw, int C, const BnLazy lazy) {
  pdl_sync();
  extern __shared__ float s_par[];   // [2][C]
  if (lazy.cells != nullptr) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const double s1 = lazy.cells[c], s2 = lazy.cells[lazy.cpad + c];
      if (blockIdx.x == 0) {         // same arithmetic as below: every block derives identical values
        bn_write_params(s1, s2, lazy.count, c, C, lazy.gamma, lazy.beta, lazy.eps, lazy.momentum, lazy.running_mean,
                        lazy.running_var, scale, shift, lazy.mean_out, lazy.invstd_out, lazy.batch_stats_out);
      }
      const double mean = s1 / lazy.count;
      double var = s2 / lazy.count - mean * mean;
      if (var < 0.0) var = 0.0;
      const float invstd = (float)(1.0 / sqrt(var + (double)lazy.eps));
      const float g_ = lazy.gamma ? lazy.gamma[c] : 1.f, b_ = lazy.beta ? lazy.beta[c] : 0.f;
      s_par[c] = g_ * invstd;
      s_par[C + c] = b_ - (float)mean * g_ * invstd;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && lazy.nbt) *lazy.nbt += 1;
  } else {
    for (int i = threadIdx.x; i < C; i += blockDim.x) { s_par[i] = scale[i]; s_par[C + i] = shift[i]; }
  }
  __syncthreads();
  const int groups = C >> 3;
  const long long total = npix * groups;
  const long long stride = (long long)gridDim.x * blockDim.x;
  constexpr int U = 4;               // 16-byte vectors in flight per thread and tensor (the pass is pure latency otherwise)
  for (long long base = (long long)blockIdx.x * blockDim.x + threadIdx.x; base < total; base += U * stride) {
    uint4 yv[U], rv[U];
    long long pix[U];
    int c0[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long idx = base + u * stride;
      const long long pp = idx / groups;
      pix[u] = pp;
      c0[u] = (int)(idx - pp * groups) << 3;
      if (idx < total) {
        yv[u] = *reinterpret_cast<const uint4*>(y + pp * y_ld + c0[u]);
        if (res) rv[u] = *reinterpret_cast<const uint4*>(res + pp * res_ld + c0[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (base + u * stride >= total) break;
      float v[8];
      unpack8(yv[u], v);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = v[j] * s_par[c0[u] + j] + s_par[C + c0[u] + j];
      if (res) {
        float r[8];
        unpack8(rv[u], r);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += r[j];
      }
      if (relu) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.f);
      }
      if (post_scale) {
        const float* ps = post_scale + (pix[u] / hw) * C + c0[u];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] *= ps[j];
      }
      store8(z + pix[u] * z_ld + c0[u], v);
    }
  }
  pdl_launch_late();
}

// ------------------------------------------------------------------------------------------------ backward
struct BnBwdFold {          // in-launch finalisation of bn_bwd_reduce (accum == nullptr: partial table + bn_bwd_finalize)
  double* accum;            // [2][C] fp64, zero between launches
  unsigned* counter;
  float* dgamma;
  float* dbeta;
  float* c1;
  float* c2;
  float count;
};

// Thread (r, cg): r-th pixel row of the block, 8-channel group cg. blockDim.x = groups * rows.
__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ dz, int dz_ld, const __nv_bfloat16* __restrict__ mask,
                     int mask_ld, const float* __restrict__ post_scale, const __nv_bfloat16* __restrict__ y, int y_ld,
                     const float* __restrict__ mean, const float* __restrict__ invstd, long long npix, int hw, int C,
                     int rows, float* __restrict__ partials, const BnBwdFold fold) {
  pdl_sync();
  extern __shared__ float s_red[];   // [rows][groups][16]
  const int groups = C >> 3;
  const int cg = threadIdx.x % groups, r = threadIdx.x / groups;
  const int c0 = cg << 3;
  float m[8], is[8], s1[8], s2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { m[j] = mean[c0 + j]; is[j] = invstd[c0 + j]; s1[j] = 0.f; s2[j] = 0.f; }
  if (r < rows) {
    constexpr int U = 4;             // pixels in flight per thread (three 16-byte loads each): the pass is latency bound otherwise
    const long long pstride = (long long)gridDim.x * rows;
    for (long long p0 = (long long)blockIdx.x * rows + r; p0 < npix; p0 += U * pstride) {
      uint4 gq[U], mq[U], yq[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long pix = p0 + u * pstride;
        if (pix < npix) {
          gq[u] = *reinterpret_cast<const uint4*>(dz + pix * dz_ld + c0);
          if (mask) mq[u] = *reinterpret_cast<const uint4*>(mask + pix * mask_ld + c0);
          yq[u] = *reinterpret_cast<const uint4*>(y + pix * y_ld + c0);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long pix = p0 + u * pstride;
        if (pix >= npix) break;
        float g[8], yv[8];
        unpack8(gq[u], g);
        if (post_scale) {
          const float* ps = post_scale + (pix / hw) * C + c0;
#pragma unroll
          for (int j = 0; j < 8; ++j) g[j] *= ps[j];
        }
        if (mask) {
          float mk[8];
          unpack8(mq[u], mk);
#pragma unroll
          for (int j = 0; j < 8; ++j) g[j] = mk[j] > 0.f ? g[j] : 0.f;
        }
        unpack8(yq[u], yv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s1[j] += g[j];
          s2[j] += g[j] * (yv[j] - m[j]) * is[j];
        }
      }
    }
    float* dst = s_red + ((size_t)r * groups + cg) * 16;
#pragma unroll
    for (int j = 0; j < 8; ++j) { dst[j] = s1[j]; dst[8 + j] = s2[j]; }
  }
  pdl_launch_late();
  __syncthreads();
  // deterministic in-block reduction over rows
  for (int i = threadIdx.x; i < groups * 16; i += blockDim.x) {
    const int g_ = i / 16, k = i % 16;
    float acc = 0.f;
    for (int rr = 0; rr < rows; ++rr) acc += s_red[((size_t)rr * groups + g_) * 16 + k];
    const int c = g_ * 8 + (k & 7);
    if (fold.accum != nullptr) atomicAdd(fold.accum + (k >> 3) * C + c, (double)acc);
    else partials[(size_t)blockIdx.x * 2 * C + (k >> 3) * C + c] = acc;
  }
  if (fold.accum == nullptr || fold.counter == nullptr) return;   // counter == nullptr: bn_bwd_apply folds the cells
  // In-launch finalisation (per-GPU statistics): the last CTA to finish turns the fp64 totals into dgamma / dbeta
  // (accumulated) and the two mean terms of the input gradient, and clears the cells (see bn_fold.cuh for the pattern).
  __shared__ unsigned s_ticket;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_ticket = atomicAdd(fold.counter, 1u);
  __syncthreads();
  if (s_ticket != gridDim.x - 1) return;
  __threadfence();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const double s1 = __ldcg(fold.accum + c), s2 = __ldcg(fold.accum + C + c);
    fold.accum[c] = 0.0;
    fold.accum[C + c] = 0.0;
    if (fold.dbeta) fold.dbeta[c] += (float)s1;
    if (fold.dgamma) fold.dgamma[c] += (float)s2;
    fold.c1[c] = (float)(s1 / (double)fold.count);
    fold.c2[c] = (float)(s2 / (double)fold.count);
  }
  if (threadIdx.x == 0) *fold.counter = 0u;
}

__global__ void __launch_bounds__(32 * kFinSlices)
bn_bwd_finalize_kernel(const float* __restrict__ partials, int G, int C, float count,
                       float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ c1,
                       float* __restrict__ c2, const SyncArgs sy) {
  pdl_wait();
  pdl_launch();                     // SyncBN: the dependent is the one-warp bn_bwd_sync_finish_kernel
  __shared__ double sh1[kFinSlices][32], sh2[kFinSlices][32];
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  double a1 = 0.0, a2 = 0.0;
  if (c < C) fold_rows(partials, G, 2 * C, C, c, slice, a1, a2);
  sh1[slice][lane] = a1;
  sh2[slice][lane] = a2;
  __syncthreads();
  double s1 = 0.0, s2 = 0.0;
  if (slice == 0 && c < C) {
    for (int k = 0; k < kFinSlices; ++k) { s1 += sh1[k][lane]; s2 += sh2[k][lane]; }
    // parameter gradients stay LOCAL sums (the data-parallel gradient all-reduce averages them like every other grad)
    if (dbeta) dbeta[c] += (float)s1;
    if (dgamma) dgamma[c] += (float)s2;
  }
  if (sy.world > 1) {            // SyncBN backward: the mean terms run over the global batch (bn_bwd_sync_finish_kernel)
    sync_post(sy, C, c, slice == 0 && c < C, s1, s2);
    return;
  }
  if (slice != 0 || c >= C) return;
  c1[c] = (float)(s1 / count);
  c2[c] = (float)(s2 / count);
}

__global__ void __launch_bounds__(32)
bn_bwd_sync_finish_kernel(int C, float count, float* __restrict__ c1, float* __restrict__ c2, const SyncArgs sy) {
  pdl_wait();
  const int c = blockIdx.x * 32 + threadIdx.x;
  double s1, s2;
  sync_wait_fold(sy, C, c, s1, s2);
  pdl_launch();
  if (c < C) {
    const double n = (double)count * (double)sy.world;
    c1[c] = (float)(s1 / n);
    c2[c] = (float)(s2 / n);
  }
}

__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ dz, int dz_ld, const __nv_bfloat16* __restrict__ mask,
                    int mask_ld, const float* __restrict__ post_scale, const __nv_bfloat16* __restrict__ y, int y_ld,
                    const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                    const float* __restrict__ c1, const float* __restrict__ c2, __nv_bfloat16* __restrict__ dy, int dy_ld,
                    __nv_bfloat16* __restrict__ g_out, int g_ld, int g_accumulate, long long npix, int hw, int C,
                    const double* __restrict__ cells, float count, float* __restrict__ dgamma,
                    float* __restrict__ dbeta) {
  pdl_sync();
  extern __shared__ float s_par[];   // [5][C]: mean, invstd, gamma*invstd, c1, c2
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    s_par[i] = mean[i];
    s_par[C + i] = invstd[i];
    s_par[2 * C + i] = (gamma ? gamma[i] : 1.f) * invstd[i];
    if (cells != nullptr) {          // deferred finalisation of bn_bwd_reduce's totals ([2][C] fp64): see BnLazy
      const double s1 = cells[i], s2 = cells[C + i];
      s_par[3 * C + i] = (float)(s1 / (double)count);
      s_par[4 * C + i] = (float)(s2 / (double)count);
      if (blockIdx.x == 0) {         // parameter gradients: local sums, accumulated once
        if (dbeta) dbeta[i] += (float)s1;
        if (dgamma) dgamma[i] += (float)s2;
      }
    } else {
      s_par[3 * C + i] = c1[i];
      s_par[4 * C + i] = c2[i];
    }
  }
  __syncthreads();
  const int groups = C >> 3;
  const long long total = npix * groups;
  const long long stride = (long long)gridDim.x * blockDim.x;
  constexpr int U = 3;               // 16-byte vectors in flight per thread and tensor
  for (long long base = (long long)blockIdx.x * blockDim.x + threadIdx.x; base < total; base += U * stride) {
    uint4 gq[U], mq[U], yq[U], oq[U];
    long long pixs[U];
    int c0s[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long idx = base + u * stride;
      const long long pix = idx / groups;
      pixs[u] = pix;
      c0s[u] = (int)(idx - pix * groups) << 3;
      if (idx < total) {
        gq[u] = *reinterpret_cast<const uint4*>(dz + pix * dz_ld + c0s[u]);
        if (mask) mq[u] = *reinterpret_cast<const uint4*>(mask + pix * mask_ld + c0s[u]);
        yq[u] = *reinterpret_cast<const uint4*>(y + pix * y_ld + c0s[u]);
        if (g_out && g_accumulate) oq[u] = *reinterpret_cast<const uint4*>(g_out + pix * g_ld + c0s[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (base + u * stride >= total) break;
      const long long pix = pixs[u];
      const int c0 = c0s[u];
      float g[8], yv[8], o[8];
      unpack8(gq[u], g);
      if (post_scale) {
        const float* ps = post_scale + (pix / hw) * C + c0;
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] *= ps[j];
      }
      if (mask) {
        float mk[8];
        unpack8(mq[u], mk);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] = mk[j] > 0.f ? g[j] : 0.f;
      }
      unpack8(yq[u], yv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xhat = (yv[j] - s_par[c0 + j]) * s_par[C + c0 + j];
        o[j] = s_par[2 * C + c0 + j] * (g[j] - s_par[3 * C + c0 + j] - xhat * s_par[4 * C + c0 + j]);
      }
      store8(dy + pix * dy_ld + c0, o);
      if (g_out) {
        if (g_accumulate) {
          float old[8];
          unpack8(oq[u], old);
#pragma unroll
          for (int j = 0; j < 8; ++j) g[j] += old[j];
        }
        store8(g_out + pix * g_ld + c0, g);
      }
    }
  }
  pdl_launch_late();
}

// dst = (accumulate ? dst : 0) + src * (mask > 0)    (ReLU backward into a fan-out gradient)
__global__ void __launch_bounds__(256)
masked_accum_kernel(const __nv_bfloat16* __restrict__ src, int src_ld, const __nv_bfloat16* __restrict__ mask,
                    int mask_ld, __nv_bfloat16* __restrict__ dst, int dst_ld, int accumulate, long long npix, int C) {
  pdl_sync();
  const int groups = C >> 3;
  const long long total = npix * groups;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long pix = idx / groups;
    const int c0 = (int)(idx - pix * groups) << 3;
    float g[8];
    load8(src + pix * src_ld + c0, g);
    if (mask) {
      float mk[8];
      load8(mask + pix * mask_ld + c0, mk);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = mk[j] > 0.f ? g[j] : 0.f;
    }
    if (accumulate) {
      float old[8];
      load8(dst + pix * dst_ld + c0, old);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] += old[j];
    }
    store8(dst + pix * dst_ld + c0, g);
  }
  pdl_launch_late();
}

// Grid of the element-wise passes: one 256-thread block per 256 x ew_items 16-byte items (the kernels keep several
// independent items in flight per thread only when the grid leaves them more than one), capped at ew_ctas_per_sm x SMs.
static inline int ew_grid(long long total_threads) {
  const long long per = 256LL * (tune().ew_items > 0 ? tune().ew_items : 1);
  long long b = (total_threads + per - 1) / per;
  const long long cap = (long long)B200SEG_MAX_CTAS * (tune().ew_ctas_per_sm > 0 ? tune().ew_ctas_per_sm : 8);
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

}  // namespace b200seg

using namespace b200seg;

static int make_sync(const b200seg_bn_sync* s, SyncArgs* out) {
  SyncArgs sy;
  sy.mail_peers = nullptr; sy.flag_peers = nullptr; sy.step = nullptr;
  sy.mail_off = 0; sy.parity_stride = 0; sy.flag_off = 0; sy.world = 1; sy.rank = 0; sy.beacon = nullptr;
  if (s && s->world > 1) {
    if (!s->mail_peers || !s->flag_peers || !s->step || s->rank < 0 || s->rank >= s->world) return B200SEG_E_BADARG;
    sy.mail_peers = (double* const*)s->mail_peers;
    sy.flag_peers = (unsigned* const*)s->flag_peers;
    sy.step = (const unsigned*)s->step;
    sy.mail_off = s->mail_offset; sy.parity_stride = s->parity_stride; sy.flag_off = s->flag_offset;
    sy.world = s->world; sy.rank = s->rank;
    sy.beacon = (volatile int*)s->beacon;
  }
  *out = sy;
  return 0;
}

#define CHECK_LAUNCH()                      \
  do {                                      \
    cudaError_t e_ = cudaGetLastError();    \
    return e_ == cudaSuccess ? 0 : (int)e_; \
  } while (0)

extern "C" int b200seg_bn_finalize(const float* partials, int32_t grid, int32_t c, int32_t cpad, float count,
                                   const float* gamma, const float* beta, float eps, float momentum,
                                   float* running_mean, float* running_var, int64_t* num_batches_tracked, float* scale,
                                   float* shift, float* mean, float* invstd, float* batch_stats_out,
                                   const b200seg_bn_sync* sync, void* stream) {
  if (!partials || !scale || !shift || !mean || !invstd || c <= 0 || grid <= 0) return B200SEG_E_BADARG;
  SyncArgs sy;
  if (int rc = make_sync(sync, &sy)) return rc;
  launch_k(bn_finalize_kernel, dim3((c + 31) / 32), dim3(32 * kFinSlices), 0, (cudaStream_t)stream, partials, grid, c,
           cpad, count, gamma, beta, eps, momentum, running_mean, running_var, (long long*)num_batches_tracked, scale,
           shift, mean, invstd, batch_stats_out, sy);
  if (sy.world > 1) {
    cudaError_t e0 = cudaGetLastError();
    if (e0 != cudaSuccess) return (int)e0;
    launch_k(bn_sync_finish_kernel, dim3((c + 31) / 32), dim3(32), 0, (cudaStream_t)stream, (int)c, count, gamma, beta,
             eps, momentum, running_mean, running_var, scale, shift, mean, invstd, batch_stats_out, sy);
  }
  CHECK_LAUNCH();
}

extern "C" int b200seg_bn_running_update(float* running, const float* batch_pass0, const float* batch_pass1,
                                         int64_t n, float momentum, int64_t* num_batches_tracked, int32_t n_layers,
                                         int32_t n_passes, void* stream) {
  if (!running || !batch_pass0 || n <= 0 || n_layers > n) return B200SEG_E_BADARG;
  launch_k(bn_running_update_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, running,
           batch_pass0, batch_pass1, (long long)n, momentum, (long long*)num_batches_tracked, n_layers, n_passes);
  CHECK_LAUNCH();
}

extern "C" int b200seg_accum_f32(float* dst, const float* src, int64_t n, void* stream) {
  if (!dst || !src || n <= 0 || (n & 3) || (reinterpret_cast<uintptr_t>(dst) & 15) ||
      (reinterpret_cast<uintptr_t>(src) & 15))
    return B200SEG_E_BADARG;
  launch_k(accum_f32_kernel, dim3(B200SEG_MAX_CTAS * 8), dim3(256), 0, (cudaStream_t)stream, dst, src, (long long)(n / 4));
  CHECK_LAUNCH();
}

extern "C" int b200seg_bn_eval_params(int32_t c, const float* gamma, const float* beta, float eps,
                                      const float* running_mean, const float* running_var, float* scale, float* shift,
                                      void* stream) {
  if (!gamma || !beta || !running_mean || !running_var || !scale || !shift) return B200SEG_E_BADARG;
  launch_k(bn_eval_params_kernel, dim3((c + 127) / 128), dim3(128), 0, (cudaStream_t)stream, c, gamma, beta, eps,
           running_mean, running_var, scale, shift);
  CHECK_LAUNCH();
}

extern "C" int b200seg_bn_apply(const void* y, int32_t y_ld, const float* scale, const float* shift, const void* res,
                                int32_t res_ld, const float* post_scale, int32_t relu, void* z, int32_t z_ld,
                                int64_t npix, int32_t hw, int32_t c, void* stream) {
  if (!y || !z || !scale || !shift || c % 8 || y_ld % 8 || z_ld % 8 || (res && res_ld % 8)) return B200SEG_E_BADARG;
  BnLazy lazy;
  memset(&lazy, 0, sizeof(lazy));
  launch_k(bn_apply_kernel, dim3(ew_grid(npix * (c / 8))), dim3(256), 2 * c * sizeof(float), (cudaStream_t)stream,
           (const __nv_bfloat16*)y, y_ld, const_cast<float*>(scale), const_cast<float*>(shift),
           (const __nv_bfloat16*)res, res_ld, post_scale, relu, (__nv_bfloat16*)z, z_ld, npix, hw, c, lazy);
  CHECK_LAUNCH();
}

extern "C" int b200seg_bn_apply_cells(const void* y, int32_t y_ld, const b200seg_bn_fold* f, const void* res,
                                      int32_t res_ld, const float* post_scale, int32_t relu, void* z, int32_t z_ld,
                                      int64_t npix, int32_t hw, int32_t c, void* stream) {
  if (!y || !z || !f || c % 8 || y_ld % 8 || z_ld % 8 || (res && res_ld % 8)) return B200SEG_E_BADARG;
  if (!f->accum || !f->scale || !f->shift || !f->mean || !f->invstd || f->c != c || f->count <= 0.f ||
      (reinterpret_cast<uintptr_t>(f->accum) & 7))
    return B200SEG_E_BADARG;
  BnLazy lazy;
  lazy.cells = f->accum; lazy.cpad = (c + 15) / 16 * 16;
  lazy.count = f->count; lazy.eps = f->eps; lazy.momentum = f->momentum;
  lazy.gamma = f->gamma; lazy.beta = f->beta; lazy.mean_out = f->mean; lazy.invstd_out = f->invstd;
  lazy.batch_stats_out = f->batch_stats_out; lazy.running_mean = f->running_mean; lazy.running_var = f->running_var;
  lazy.nbt = (long long*)f->num_batches_tracked;
  launch_k(bn_apply_kernel, dim3(ew_grid(npix * (c / 8))), dim3(256), 2 * c * sizeof(float), (cudaStream_t)stream,
           (const __nv_bfloat16*)y, y_ld, f->scale, f->shift, (const __nv_bfloat16*)res, res_ld, post_scale, relu,
           (__nv_bfloat16*)z, z_ld, npix, hw, c, lazy);
  CHECK_LAUNCH();
}

static inline void reduce_shape(int c, int* rows, int* threads) {
  const int groups = c / 8;
  int r = 256 / groups;
  if (r < 1) r = 1;
  *rows = r;
  *threads = groups * r;
}

extern "C" int32_t b200seg_bn_bwd_grid(int64_t npix, int32_t c) {
  int rows, threads;
  reduce_shape(c, &rows, &threads);
  const long long per = (long long)rows * (tune().red_items > 0 ? tune().red_items : 1);
  long long b = (npix + per - 1) / per;
  const long long cap = (long long)B200SEG_MAX_CTAS * (tune().red_ctas_per_sm > 0 ? tune().red_ctas_per_sm : 2);
  return (int32_t)(b < cap ? (b > 0 ? b : 1) : cap);
}

static int bn_bwd_reduce_launch(const void* dz, int32_t dz_ld, const void* mask, int32_t mask_ld,
                                const float* post_scale, const void* y, int32_t y_ld, const float* mean,
                                const float* invstd, int64_t npix, int32_t hw, int32_t c, float* partials,
                                const BnBwdFold& fold, void* stream) {
  if (!dz || !y || !mean || !invstd || (!partials && !fold.accum) || c % 8 || c > 2048) return B200SEG_E_BADARG;
  int rows, threads;
  reduce_shape(c, &rows, &threads);
  if (threads > 256) return B200SEG_E_BADARG;
  const int grid = b200seg_bn_bwd_grid(npix, c);
  const size_t smem = (size_t)rows * (c / 8) * 16 * sizeof(float);
  launch_k(bn_bwd_reduce_kernel, dim3(grid), dim3(threads), smem, (cudaStream_t)stream, (const __nv_bfloat16*)dz,
           dz_ld, (const __nv_bfloat16*)mask, mask_ld, post_scale, (const __nv_bfloat16*)y, y_ld, mean, invstd, npix,
           hw, c, rows, partials, fold);
  CHECK_LAUNCH();
}

extern "C" int b200seg_bn_bwd_reduce(const void* dz, int32_t dz_ld, const void* mask, int32_t mask_ld,
                                     const float* post_scale, const void* y, int32_t y_ld, const float* mean,
                                     const float* invstd, int64_t npix, int32_t hw, int32_t c, float* partials,
                                     void* stream) {
  BnBwdFold fold;
  memset(&fold, 0, sizeof(fold));
  return bn_bwd_reduce_launch(dz, dz_ld, mask, mask_ld, post_scale, y, y_ld, mean, invstd, npix, hw, c, partials, fold,
                              stream);
}

extern "C" int b200seg_bn_bwd_reduce_finalize(const void* dz, int32_t dz_ld, const void* mask, int32_t mask_ld,
                                              const float* post_scale, const void* y, int32_t y_ld, const float* mean,
                                              const float* invstd, int64_t npix, int32_t hw, int32_t c, double* accum,
                                              uint32_t* counter, float* dgamma, float* dbeta, float* c1, float* c2,
                                              void* stream) {
  if (!accum || !counter || !c1 || !c2 || (reinterpret_cast<uintptr_t>(accum) & 7)) return B200SEG_E_BADARG;
  BnBwdFold fold;
  fold.accum = accum; fold.counter = counter; fold.dgamma = dgamma; fold.dbeta = dbeta; fold.c1 = c1; fold.c2 = c2;
  fold.count = (float)npix;
  return bn_bwd_reduce_launch(dz, dz_ld, mask, mask_ld, post_scale, y, y_ld, mean, invstd, npix, hw, c, nullptr, fold,
                              stream);
}

extern "C" int b200seg_bn_bwd_finalize(const float* partials, int32_t grid, int32_t c, float count, float* dgamma,
                                       float* dbeta, float* c1, float* c2, const b200seg_bn_sync* sync, void* stream) {
  if (!partials || !c1 || !c2) return B200SEG_E_BADARG;
  SyncArgs sy;
  if (int rc = make_sync(sync, &sy)) return rc;
  launch_k(bn_bwd_finalize_kernel, dim3((c + 31) / 32), dim3(32 * kFinSlices), 0, (cudaStream_t)stream, partials,
           grid, c, count, dgamma, dbeta, c1, c2, sy);
  if (sy.world > 1) {
    cudaError_t e0 = cudaGetLastError();
    if (e0 != cudaSuccess) return (int)e0;
    launch_k(bn_bwd_sync_finish_kernel, dim3((c + 31) / 32), dim3(32), 0, (cudaStream_t)stream, (int)c, count, c1, c2, sy);
  }
  CHECK_LAUNCH();
}

extern "C" int b200seg_bn_bwd_apply(const void* dz, int32_t dz_ld, const void* mask, int32_t mask_ld,
                                    const float* post_scale, const void* y, int32_t y_ld, const float* mean,
                                    const float* invstd, const float* gamma, const float* c1, const float* c2, void* dy,
                                    int32_t dy_ld, void* g_out, int32_t g_ld, int32_t g_accumulate, int64_t npix,
                                    int32_t hw, int32_t c, void* stream) {
  if (!dz || !y || !dy || !mean || !invstd || !c1 || !c2 || c % 8) return B200SEG_E_BADARG;
  launch_k(bn_bwd_apply_kernel, dim3(ew_grid(npix * (c / 8))), dim3(256), 5 * c * sizeof(float), (cudaStream_t)stream,
           (const __nv_bfloat16*)dz, dz_ld, (const __nv_bfloat16*)mask, mask_ld, post_scale, (const __nv_bfloat16*)y,
           y_ld, mean, invstd, gamma, c1, c2, (__nv_bfloat16*)dy, dy_ld, (__nv_bfloat16*)g_out, g_ld, g_accumulate,
           npix, hw, c, (const double*)nullptr, 0.f, (float*)nullptr, (float*)nullptr);
  CHECK_LAUNCH();
}

// BatchNorm backward with deferred finalisation: bn_bwd_reduce adds its per-block sums to `cells` ([2][c] fp64, zeroed by
// the caller once per step), bn_bwd_apply folds them in its prologue (and accumulates dgamma / dbeta): two launches
// instead of three, nothing between the reduction and the gradient pass. Per-GPU statistics only.
extern "C" int b200seg_bn_bwd_cells(const void* dz, int32_t dz_ld, const void* mask, int32_t mask_ld,
                                    const float* post_scale, const void* y, int32_t y_ld, const float* mean,
                                    const float* invstd, const float* gamma, float* dgamma, float* dbeta, double* cells,
                                    void* dy, int32_t dy_ld, void* g_out, int32_t g_ld, int32_t g_accumulate,
                                    int64_t npix, int32_t hw, int32_t c, void* stream) {
  if (!dz || !y || !dy || !mean || !invstd || !cells || c % 8 || (reinterpret_cast<uintptr_t>(cells) & 7))
    return B200SEG_E_BADARG;
  BnBwdFold fold;
  memset(&fold, 0, sizeof(fold));
  fold.accum = cells;                 // counter == nullptr: cells only
  fold.count = (float)npix;
  if (int rc = bn_bwd_reduce_launch(dz, dz_ld, mask, mask_ld, post_scale, y, y_ld, mean, invstd, npix, hw, c, nullptr,
                                    fold, stream))
    return rc;
  launch_k(bn_bwd_apply_kernel, dim3(ew_grid(npix * (c / 8))), dim3(256), 5 * c * sizeof(float), (cudaStream_t)stream,
           (const __nv_bfloat16*)dz, dz_ld, (const __nv_bfloat16*)mask, mask_ld, post_scale, (const __nv_bfloat16*)y,
           y_ld, mean, invstd, gamma, (const float*)nullptr, (const float*)nullptr, (__nv_bfloat16*)dy, dy_ld,
           (__nv_bfloat16*)g_out, g_ld, g_accumulate, npix, hw, c, (const double*)cells, (float)npix, dgamma, dbeta);
  CHECK_LAUNCH();
}

extern "C" int b200seg_masked_accum(const void* src, int32_t src_ld, const void* mask, int32_t mask_ld, void* dst,
                                    int32_t dst_ld, int32_t accumulate, int64_t npix, int32_t c, void* stream) {
  if (!src || !dst || c % 8) return B200SEG_E_BADARG;
  launch_k(masked_accum_kernel, dim3(ew_grid(npix * (c / 8))), dim3(256), 0, (cudaStream_t)stream,
           (const __nv_bfloat16*)src, src_ld, (const __nv_bfloat16*)mask, mask_ld, (__nv_bfloat16*)dst, dst_ld,
           accumulate, npix, c);
  CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------- peer memory (SyncBN)
extern "C" int b200seg_p2p_alloc(size_t bytes, void** dev_ptr, uint8_t* handle64) {
  if (!dev_ptr || !handle64 || bytes == 0) return B200SEG_E_BADARG;
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) return (int)e;
  e = cudaMemset(p, 0, bytes);
  if (e != cudaSuccess) { cudaFree(p); return (int)e; }
  cudaIpcMemHandle_t h;
  e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { cudaFree(p); return (int)e; }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  memcpy(handle64, &h, 64);
  *dev_ptr = p;
  return 0;
}
extern "C" int b200seg_p2p_open(const uint8_t* handle64, void** dev_ptr) {
  if (!handle64 || !dev_ptr) return B200SEG_E_BADARG;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  cudaError_t e = cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess);
  return e == cudaSuccess ? 0 : (int)e;
}
extern "C" int b200seg_p2p_close(void* dev_ptr) {
  cudaError_t e = cudaIpcCloseMemHandle(dev_ptr);
  return e == cudaSuccess ? 0 : (int)e;
}
extern "C" int b200seg_p2p_free(void* dev_ptr) {
  cudaError_t e = cudaFree(dev_ptr);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int32_t b200seg_sgd_chunk(void) { return kSgdChunk; }

extern "C" int b200seg_sgd_step(const b200seg_sgd_item* items, const int32_t* blk_item, const int32_t* blk_start,
                                int32_t n_blocks, float lr, float momentum, float dampening, float weight_decay,
                                int32_t nesterov, int32_t first_step, void* stream) {
  if (!items || !blk_item || !blk_start || n_blocks <= 0) return B200SEG_E_BADARG;
  launch_k(sgd_step_kernel, dim3(n_blocks), dim3(256), 0, (cudaStream_t)stream, items, blk_item, blk_start, lr,
           momentum, dampening, weight_decay, (int)nesterov, (int)first_step);
  CHECK_LAUNCH();
}
