// Weight-gradient convolution as a wgmma GEMM with both operands MN-major (pixels are the reduction dimension):
//
//   dW[co][ci][kh][kw] += sum_{n,ho,wo} dy[n,ho,wo,co] * x[n, ho*s+kh-p, wo*s+kw-p, ci]
//
//   A = dy  [pixels][cout]  -> M = 128 output channels (two 64-channel SWIZZLE_128B blocks of 128 pixel-rows), one
//                              block per consumer warpgroup
//   B = x   [pixels][cin]   -> N <= 256 input channels (64-channel blocks), one shifted TMA box per filter tap
//   D[tap]  = fp32 accumulators in registers, taps of a group side by side (taps_in_group * N <= 256 columns)
//
// Work unit = (M tile, N tile, tap group, pixel split). Units are distributed round-robin over a persistent grid; each
// unit reduces its share of the pixels in registers. The gradient accumulator is fp32 in the kernels' [Cout][tap][Cin]
// ("OHWI") layout, so an accumulator row is a contiguous run of input channels:
//   * splits == 1 (low-resolution / wide layers: enough (tile, tap-group) items to fill the SMs): exactly one unit owns
//     every gradient element, which it adds with fire-and-forget reductions — no workspace, no second kernel,
//     deterministic;
//   * splits  > 1 (high-resolution narrow layers): units store fp32 slabs and wgrad_reduce_kernel sums the splits in a
//     fixed order (deterministic) with coalesced float4 traffic.
// The decomposition (N tile width, taps per group, splits) is picked per layer by a small cost model (wgrad_plan).
//
// MMA issue: the kernel is instantiated per W16 = min(Cin, ntile_w) / 16 (1 .. 16) and its tap loop is unrolled up to
// the most taps a unit can hold (min(9, 16 / W16)), so every MMA's width (W16 / 4 n64 MMAs and at most one n16/n32/n48
// tail) and accumulator offset (tap * W16 * 16 columns) are compile-time constants. Only the unit's tap count (a short
// last tap group) is tested at run time, between the (pixel tile, tap) MMA groups; nothing branches between an MMA and
// the commit of its group. So ptxas keeps the accumulators in registers without spills and keeps one group in flight
// under the next (wgmma_wait<1>); tests/test_wgrad_sass.py checks the compiled code for both. The last N tile of a
// multi-tile layer (720 channels: 256, 256, 208) runs the full W16 width and drops the extra columns in the epilogue
// (2.6% more MMA work over the weight gradients of the two-scale 1024x2048 step).
// The step folds the OHWI accumulators into the OIHW master gradients once, at the end (grad_fold_kernel).
// Replaces cuDNN convolution_backward (weight part) behind every nn.Conv2d listed in SURVEY.md §2b K1-K5.
#include "ptx.cuh"
#include "tma_host.h"
#include "launch.h"
#include "conv_common.h"
#include "conv_epi.cuh"
#include "../../include/b200seg.h"
#include <utility>

namespace b200seg {

struct WgradParams {
  int N, Ho, Wo, Cout, Cin;
  int ksize, stride, pad, taps, dil;
  int TH, TW, tiles_h, tiles_w, pix_tiles;
  int m_tiles, n_tiles, tap_groups, taps_per_group, splits, total_units;
  int nblocksB_max;
  int ntile_w;           // N tile width in channels (64, 128 or 256)
  int unit_n;            // accumulator row pitch of a unit slab (= min(ntile_w, Cin))
  long long unit_stride; // floats per unit slab
  int a_slot_bytes, b_slot_bytes, b_slots;
  int direct;            // splits == 1: units add straight into the gradient accumulator
};

constexpr int kWThreads = 288;       // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int kABlock = 128 * 128;   // 128 pixel rows x 64 channels bf16
constexpr int kMaxBSlots = 6;
constexpr int kWAccCols = 256;       // accumulator columns per consumer thread row (128 registers)

// one MN-major MMA of width 16 * w (w <= 4 blocks: inside one 64-channel swizzle atom). Every call site passes a
// compile-time w (fully unrolled loops), so the selection folds away.
__device__ __forceinline__ void wgmma_mn(float* d, int w, uint64_t a, uint64_t b, uint32_t scale_d) {
  if (w >= 4) wgmma_n64<1, 1>(d, a, b, scale_d);
  else if (w == 3) wgmma_n48<1, 1>(d, a, b, scale_d);
  else if (w == 2) wgmma_n32<1, 1>(d, a, b, scale_d);
  else wgmma_n16<1, 1>(d, a, b, scale_d);
}

// W16 = Nmax / 16: 16-column blocks of one tap's accumulator (Nmax = min(Cin, ntile_w), the unit slab's row pitch).
// p is a __grid_constant__ so the lambdas can capture it by reference without a stack copy.
template <int W16>
__global__ void __launch_bounds__(kWThreads, 1)
wgrad_igemm_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX,
                   const __grid_constant__ WgradParams p, float* __restrict__ ws, float* __restrict__ dw) {
  constexpr int kMaxTaps = kWAccCols / 16 / W16 < 9 ? kWAccCols / 16 / W16 : 9;   // taps of one unit (ksize <= 3)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_base = smem;                               // 2 slots
  uint8_t* b_base = smem + 2 * p.a_slot_bytes;          // b_slots
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_base + (size_t)p.b_slots * p.b_slot_bytes);
  uint64_t* a_full = bars;              // [2]
  uint64_t* a_empty = bars + 2;         // [2]
  uint64_t* b_full = bars + 4;          // [kMaxBSlots]
  uint64_t* b_empty = bars + 4 + kMaxBSlots;

  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmDy);
    tma_prefetch_desc(&tmX);
    for (int s = 0; s < 2; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 2); }
    for (int s = 0; s < p.b_slots; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_sync();   // the prologue above overlapped the previous kernel; global memory is touched only below

  // unit decode helpers (identical in every role)
  auto decode = [&](int unit, int& m_tile, int& n_tile, int& tg, int& split) {
    split = unit % p.splits;
    int item = unit / p.splits;
    tg = item % p.tap_groups; item /= p.tap_groups;
    n_tile = item % p.n_tiles;
    m_tile = item / p.n_tiles;
  };

  if (warp == 8) {
    if (elect_one()) {   // one elected lane runs the whole producer loop (TMA operands stay in uniform registers)
      int a_slot = 0, b_slot = 0;
      uint32_t a_phase = 0, b_phase = 0;
      for (int unit = blockIdx.x; unit < p.total_units; unit += gridDim.x) {
        int m_tile, n_tile, tg, split;
        decode(unit, m_tile, n_tile, tg, split);
        const int n0 = n_tile * p.ntile_w;
        const int nblk = min(p.ntile_w / 64, (p.Cin - n0 + 63) / 64);
        const int tap0 = tg * p.taps_per_group, tap1 = min(p.taps, tap0 + p.taps_per_group);
        const bool a_two = (p.Cout - m_tile * 128) > 64;      // second 64-channel dy block holds real channels
        for (int t = split; t < p.pix_tiles; t += p.splits) {
          const int tw_i = t % p.tiles_w;
          const int th_i = (t / p.tiles_w) % p.tiles_h;
          const int img = t / (p.tiles_w * p.tiles_h);
          mbar_wait(&a_empty[a_slot], a_phase ^ 1);
          uint8_t* sa = a_base + (size_t)a_slot * p.a_slot_bytes;
          mbar_arrive_expect_tx(&a_full[a_slot], (a_two ? 2 : 1) * kABlock);
          tma_load_4d(&tmDy, &a_full[a_slot], sa, m_tile * 128, tw_i * p.TW, th_i * p.TH, img);
          if (a_two)
            tma_load_4d(&tmDy, &a_full[a_slot], sa + kABlock, m_tile * 128 + 64, tw_i * p.TW, th_i * p.TH, img);
          if (++a_slot == 2) { a_slot = 0; a_phase ^= 1; }
          for (int tap = tap0; tap < tap1; ++tap) {
            const int kh = tap / p.ksize, kw = tap - kh * p.ksize;
            mbar_wait(&b_empty[b_slot], b_phase ^ 1);
            uint8_t* sb = b_base + (size_t)b_slot * p.b_slot_bytes;
            mbar_arrive_expect_tx(&b_full[b_slot], nblk * kABlock);
            for (int b = 0; b < nblk; ++b)
              tma_load_4d(&tmX, &b_full[b_slot], sb + (size_t)b * kABlock, n0 + b * 64,
                          tw_i * p.TW * p.stride + kw * p.dil - p.pad, th_i * p.TH * p.stride + kh * p.dil - p.pad,
                          img);
            if (++b_slot == p.b_slots) { b_slot = 0; b_phase ^= 1; }
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ------------------------------------------------------------------ consumers: MMA + epilogue
    const uint32_t g = warp >> 2;              // warpgroup: output channels 64g .. 64g + 63 of the M tile
    const bool leader = (threadIdx.x & 127) == 0;
    // 16 pixels per K step = 2048 B of both operands; 8-pixel groups 1024 B apart; 64-channel atoms kABlock apart
    const uint64_t tmpl = make_smem_desc(0, kABlock, 1024, 1);
    const uint32_t a0 = smem_u32(a_base) + g * kABlock, b0 = smem_u32(b_base);
    // thread rows: output channels co0 (+8); block (tap tl, 16 columns c): columns 16c + 8h + 2(lane % 4) + {0, 1}
    const int row0 = (int)(g * 64 + (warp & 3) * 16 + (lane >> 2));
    int a_slot = 0, b_slot = 0;
    uint32_t a_phase = 0, b_phase = 0;
    for (int unit = blockIdx.x; unit < p.total_units; unit += gridDim.x) {
      int m_tile, n_tile, tg, split;
      decode(unit, m_tile, n_tile, tg, split);
      const int n0 = n_tile * p.ntile_w;
      const int Nn = min(p.ntile_w, p.Cin - n0);         // multiple of 16; < 16 * W16 only in the last N tile
      const int tap0 = tg * p.taps_per_group, ntaps = min(p.taps, tap0 + p.taps_per_group) - tap0;
      const bool active = g == 0 || (p.Cout - m_tile * 128) > 64;   // this warpgroup's dy block holds real channels
      // Each MMA spans all W16 blocks even in a narrower last N tile: an output column depends on its own B column
      // only, so the columns >= Nn (stale or zero-filled shared memory) are computed and dropped by the epilogue.
      float acc[kMaxTaps * W16 * 8];
      uint32_t pend_b = 0, pend_a = 0;   // empty barriers of the group still in flight (shared addresses, 0: none)
      uint32_t started = 0;
      for (int t = split; t < p.pix_tiles; t += p.splits) {
        mbar_wait(&a_full[a_slot], a_phase);
        const uint64_t ad = tmpl + (uint64_t)((a0 + (uint32_t)a_slot * (uint32_t)p.a_slot_bytes) >> 4);
#pragma unroll
        for (int tl = 0; tl < kMaxTaps; ++tl) {
          if (tl >= ntaps) break;
          mbar_wait(&b_full[b_slot], b_phase);
          const uint64_t bd = tmpl + (uint64_t)((b0 + (uint32_t)b_slot * (uint32_t)p.b_slot_bytes) >> 4);
          if (active) {
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; ++k) {
#pragma unroll
              for (int c = 0; c < W16; c += 4)
                wgmma_mn(&acc[8 * (tl * W16 + c)], W16 - c, ad + (uint64_t)(k * 128),
                         bd + (uint64_t)(k * 128 + (c >> 2) * (kABlock >> 4)), started | (uint32_t)k);
            }
            wgmma_commit();
            wgmma_wait<1>();
          }
          if (leader && pend_b) mbar_arrive_at(pend_b);
          if (leader && pend_a) mbar_arrive_at(pend_a);
          pend_b = smem_u32(&b_empty[b_slot]);
          pend_a = tl == ntaps - 1 ? smem_u32(&a_empty[a_slot]) : 0u;
          if (++b_slot == p.b_slots) { b_slot = 0; b_phase ^= 1; }
        }
        if (++a_slot == 2) { a_slot = 0; a_phase ^= 1; }
        started = 1;
      }
      wgmma_wait<0>();
      if (leader && pend_b) mbar_arrive_at(pend_b);
      if (leader && pend_a) mbar_arrive_at(pend_a);
      if (!started || !active) continue;
#pragma unroll
      for (int tl = 0; tl < kMaxTaps; ++tl) {
        if (tl >= ntaps) break;
#pragma unroll
        for (int c = 0; c < W16; ++c) {
          if (c * 16 >= Nn) break;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int col = c * 16 + 8 * h + 2 * (int)(lane & 3);
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              const int row = row0 + 8 * r, co = m_tile * 128 + row;
              if (co >= p.Cout) continue;
              const float v0 = acc[8 * (tl * W16 + c) + 4 * h + 2 * r], v1 = acc[8 * (tl * W16 + c) + 4 * h + 2 * r + 1];
              if (p.direct) {
                // the only unit that touches these gradient elements: a fire-and-forget reduction
                red_add_v2(dw + ((size_t)co * p.taps + tap0 + tl) * p.Cin + n0 + col, v0, v1);
              } else {
                // per-unit slab [tap_local][128 rows][unit_n] fp32, summed by wgrad_reduce_kernel
                float2* dst = reinterpret_cast<float2*>(ws + (size_t)unit * p.unit_stride +
                                                        ((size_t)tl * 128 + row) * p.unit_n + col);
                *dst = make_float2(v0, v1);
              }
            }
          }
        }
      }
    }
    if (g == 0 && leader) pdl_launch_late();
  }
}

// dw[co][tap][ci] += sum over the pixel splits of the unit slabs, splits summed in a fixed order (deterministic).
// One thread block = 32 consecutive float4 of an item's [tap_local][row][col] index space (coalesced 512-byte slab reads)
// x 8 slices of the split range; the 8 partial sums are folded in slice order.
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const WgradParams p, const float* __restrict__ ws, float* __restrict__ dw, int blocks_per_item) {
  __shared__ float4 sh[8][32];
  pdl_sync();
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
  const int item = blockIdx.x / blocks_per_item, chunk = blockIdx.x - item * blocks_per_item;
  int it = item;
  const int tg = it % p.tap_groups; it /= p.tap_groups;
  const int n_tile = it % p.n_tiles;
  const int m_tile = it / p.n_tiles;
  const int n0 = n_tile * p.ntile_w;
  const int Nn = min(p.ntile_w, p.Cin - n0);
  const int rows = min(128, p.Cout - m_tile * 128);
  const int tap0 = tg * p.taps_per_group, ntap = min(p.taps, tap0 + p.taps_per_group) - tap0;
  const int c4 = Nn >> 2;                               // float4 per accumulator row
  const int f = chunk * 32 + lane;                      // float4 index inside [ntap][rows][c4]
  const bool live = f < ntap * rows * c4;
  int tl = 0, row = 0, col4 = 0;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (live) {
    col4 = f % c4;
    row = (f / c4) % rows;
    tl = f / (c4 * rows);
    const float4* src = reinterpret_cast<const float4*>(ws + (size_t)item * p.splits * p.unit_stride +
                                                        ((size_t)tl * 128 + row) * p.unit_n) + col4;
    const size_t stride4 = (size_t)p.unit_stride >> 2;
    float4 a0 = acc, a1 = acc;
    int s_ = slice;
    for (; s_ + 8 < p.splits; s_ += 16) {
      const float4 u = src[(size_t)s_ * stride4], v = src[(size_t)(s_ + 8) * stride4];
      a0.x += u.x; a0.y += u.y; a0.z += u.z; a0.w += u.w;
      a1.x += v.x; a1.y += v.y; a1.z += v.z; a1.w += v.w;
    }
    if (s_ < p.splits) {
      const float4 u = src[(size_t)s_ * stride4];
      a0.x += u.x; a0.y += u.y; a0.z += u.z; a0.w += u.w;
    }
    acc = make_float4(a0.x + a1.x, a0.y + a1.y, a0.z + a1.z, a0.w + a1.w);
  }
  sh[slice][lane] = acc;
  pdl_launch_late();
  __syncthreads();
  if (slice == 0 && live) {
    float4 t = sh[0][lane];
#pragma unroll
    for (int k = 1; k < 8; ++k) { const float4 u = sh[k][lane]; t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w; }
    float4* dst = reinterpret_cast<float4*>(dw + ((size_t)(m_tile * 128 + row) * p.taps + tap0 + tl) * p.Cin + n0) + col4;
    float4 o = *dst;
    o.x += t.x; o.y += t.y; o.z += t.z; o.w += t.w;
    *dst = o;
  }
}

// Folds the step's gradient accumulators into the step gradient (see b200seg_grad_fold in the header):
//   conv weights : dst[co][ci][tap] (OIHW master layout) (+)= acc_a[co][tap][ci] + acc_b[co][tap][ci]   (OHWI accumulators)
//   vectors      : dst[i] (+)= acc_a[i] + acc_b[i]
// One block = up to kFoldChunk consecutive elements of one parameter: coalesced write (or read-modify-write) of dst,
// transposed gather from the accumulators (each accumulator element is read, and cleared, by exactly one thread).
constexpr int kFoldChunk = 4096;
__global__ void __launch_bounds__(256)
grad_fold_kernel(float* __restrict__ dst, float* __restrict__ acc_a, float* __restrict__ acc_b,
                 const b200seg_grad_seg* __restrict__ segs, const int32_t* __restrict__ blk_seg,
                 const int32_t* __restrict__ blk_start, int mode) {
  pdl_sync();
  const bool clear = mode & 1, overwrite = mode & 2;
  const b200seg_grad_seg sg = segs[blk_seg[blockIdx.x]];
  const uint32_t numel = (uint32_t)sg.cout * sg.cin * sg.taps;     // a parameter has < 2^31 elements
  const uint32_t j0 = (uint32_t)blk_start[blockIdx.x];
  const uint32_t len = (uint32_t)(sg.cin * sg.taps), taps = (uint32_t)sg.taps, scin = (uint32_t)sg.src_cin;
  const uint32_t slen = scin * taps;
  float* a = acc_a ? acc_a + sg.src_offset : nullptr;
  float* b = acc_b ? acc_b + sg.src_offset : nullptr;
  float* d = dst + sg.offset;
  for (int t0 = threadIdx.x; t0 < kFoldChunk; t0 += 4 * 256) {   // four elements in flight per thread
    uint32_t js[4], srcs[4];
    float v[4];
    bool ok[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const uint32_t j = j0 + t0 + u * 256;
      ok[u] = j < numel;
      uint32_t src = j;
      if (taps > 1 || scin != (uint32_t)sg.cin) {
        const uint32_t r = j / len;
        const uint32_t jj = j - r * len;
        const uint32_t ci = jj / taps, tap = jj - ci * taps;
        src = r * slen + tap * scin + ci;
      }
      js[u] = j; srcs[u] = src;
      v[u] = 0.f;
      if (ok[u]) {
        if (!overwrite) v[u] = d[j];
        if (a) v[u] += a[src];
        if (b) v[u] += b[src];
      }
    }
    // The clearing stores must not be issued while loads of the same addresses are still in flight (a store that
    // chases an outstanding load miss to the same line serialises the memory pipeline: measured 25x slower).
    asm volatile("" ::"f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (!ok[u]) continue;
      d[js[u]] = v[u];
      if (clear) {
        if (a) a[srcs[u]] = 0.f;
        if (b) b[srcs[u]] = 0.f;
      }
    }
  }
}

// dst = (accumulate ? dst : 0) + (*scale_dev * scale_const) * src   (gradient publish, see the header)
__global__ void __launch_bounds__(256)
publish_grads_kernel(float* __restrict__ dst, const float* __restrict__ src, long long n4,
                     const float* __restrict__ scale_dev, float scale_const, int accumulate) {
  pdl_sync();
  const float sc = (scale_dev ? *scale_dev : 1.f) * scale_const;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 b = reinterpret_cast<const float4*>(src)[i];
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (accumulate) a = reinterpret_cast<float4*>(dst)[i];
    a.x += sc * b.x; a.y += sc * b.y; a.z += sc * b.z; a.w += sc * b.w;
    reinterpret_cast<float4*>(dst)[i] = a;
  }
}

}  // namespace b200seg

using namespace b200seg;

using WgradKernel = void (*)(CUtensorMap, CUtensorMap, WgradParams, float*, float*);
template <int... I>
static WgradKernel wgrad_kernel(int w16, std::integer_sequence<int, I...>) {
  static constexpr WgradKernel k[] = {wgrad_igemm_kernel<I + 1>...};
  return k[w16 - 1];
}

static int wgrad_grid(const WgradParams& p) { return p.total_units < B200SEG_MAX_CTAS ? p.total_units : B200SEG_MAX_CTAS; }

// Decomposition, B-ring depth and dynamic shared memory of one launch (host only; also reported by
// b200seg_conv2d_wgrad_plan_info, so the query and the launch cannot disagree).
static int wgrad_plan(const b200seg_conv_desc* d, WgradParams& p, size_t& smem_bytes) {
  if (!d) return B200SEG_E_BADARG;
  const int dil = d->dilation > 1 ? d->dilation : 1;
  if (!((d->ksize == 1 && d->pad == 0 && dil == 1) || (d->ksize == 3 && d->pad == dil))) return B200SEG_E_BADARG;
  if (d->stride != 1 && d->stride != 2) return B200SEG_E_BADARG;
  if (dil > 1 && d->stride != 1) return B200SEG_E_BADARG;
  if (d->cin % 16 || d->x_ld % 8) return B200SEG_E_BADARG;
  p.N = d->n; p.Cout = d->cout; p.Cin = d->cin;
  p.ksize = d->ksize; p.stride = d->stride; p.pad = d->pad; p.taps = d->ksize * d->ksize; p.dil = dil;
  p.Ho = (d->h + 2 * d->pad - dil * (d->ksize - 1) - 1) / d->stride + 1;
  p.Wo = (d->w + 2 * d->pad - dil * (d->ksize - 1) - 1) / d->stride + 1;
  p.TW = 16; p.TH = 8;
  if (p.Wo <= 8) { p.TW = 8; p.TH = 16; }
  p.tiles_w = (p.Wo + p.TW - 1) / p.TW;
  p.tiles_h = (p.Ho + p.TH - 1) / p.TH;
  p.pix_tiles = d->n * p.tiles_h * p.tiles_w;
  p.m_tiles = (d->cout + 127) / 128;
  const bool a_two = d->cout > 64;

  // Decomposition search. Clock estimates per 128-pixel tile of one unit: tensor issue (M=128: the MN-major dy read of
  // 4 KB per K=16 step bounds a narrow MMA at ~32 clk) against L2->smem fill at ~64 B/clk; a split run pays the slab
  // round trip through HBM (~3 KB/clk) and a second kernel.
  double best = 0;
  int best_w = 0, best_tpg = 0, best_splits = 0;
  const int widths[3] = {64, 128, 256};
  for (int wi = 0; wi < 3; ++wi) {
    const int ntw = widths[wi];
    if (wi > 0 && d->cin <= widths[wi - 1]) continue;        // same tiling as the narrower candidate
    const int n_tiles = (d->cin + ntw - 1) / ntw;
    const int Nmax = d->cin < ntw ? d->cin : ntw;
    const int nblk = (Nmax + 63) / 64;
    int tpg_max = kWAccCols / Nmax;
    if (tpg_max > p.taps) tpg_max = p.taps;
    for (int tg = (p.taps + tpg_max - 1) / tpg_max; tg <= p.taps; ++tg) {
      const int tpg = (p.taps + tg - 1) / tg;
      if ((p.taps + tpg - 1) / tpg != tg) continue;
      const int items = p.m_tiles * n_tiles * tg;
      int sp_max = B200SEG_MAX_CTAS / items;
      if (sp_max > p.pix_tiles) sp_max = p.pix_tiles;
      if (sp_max < 1) sp_max = 1;
      const double mma = (double)tpg * 8.0 * (Nmax / 2 > 32 ? Nmax / 2 : 32);
      const double bytes = (a_two ? 32768.0 : 16384.0) + (double)tpg * nblk * 16384.0;
      const double per_tile = mma > bytes / 64.0 ? mma : bytes / 64.0;
      if (tune().wgrad_min_clk > 0) {     // every unit reduces at least wgrad_min_clk modelled clocks of pixel tiles
        int sp_w = (int)((double)p.pix_tiles * per_tile / (double)tune().wgrad_min_clk);
        if (sp_w < 1) sp_w = 1;
        if (sp_w < sp_max) sp_max = sp_w;
      }
      for (int pass = 0; pass < 2; ++pass) {
        const int splits = pass == 0 ? 1 : sp_max;
        if (pass == 1 && sp_max == 1) break;
        const double tiles_per_unit = (double)((p.pix_tiles + splits - 1) / splits);
        const double unit = tiles_per_unit * per_tile + (double)tpg * Nmax * 4.0 + 1500.0;
        const double waves = (double)(((long long)items * splits + B200SEG_MAX_CTAS - 1) / B200SEG_MAX_CTAS);
        double cost = waves * unit;
        if (splits > 1) {
          const double slab = (double)items * splits * tpg * (d->cout < 128 ? d->cout : 128) * Nmax * 4.0;
          cost += 6000.0 + 2.0 * slab / 3000.0;
        }
        if (best_w == 0 || cost < best) { best = cost; best_w = ntw; best_tpg = tpg; best_splits = splits; }
      }
    }
  }
  if (best_w == 0) return B200SEG_E_BADARG;
  p.ntile_w = best_w;
  p.n_tiles = (d->cin + p.ntile_w - 1) / p.ntile_w;
  const int Nmax = d->cin < p.ntile_w ? d->cin : p.ntile_w;
  p.taps_per_group = best_tpg;
  p.tap_groups = (p.taps + best_tpg - 1) / best_tpg;
  p.splits = best_splits;
  p.direct = best_splits == 1 ? 1 : 0;
  const int items = p.m_tiles * p.n_tiles * p.tap_groups;
  p.total_units = items * p.splits;
  p.nblocksB_max = (Nmax + 63) / 64;
  p.unit_n = Nmax;
  p.unit_stride = (long long)p.taps_per_group * 128 * Nmax;
  p.a_slot_bytes = 2 * kABlock;
  p.b_slot_bytes = p.nblocksB_max * kABlock;
  const size_t fixed = 1024 + 2 * (size_t)p.a_slot_bytes + (4 + 2 * kMaxBSlots) * 8 + 16;
  const size_t budget = (size_t)227 * 1024 - smem_reserve();
  int bs = (int)((budget - fixed) / p.b_slot_bytes);
  if (bs > kMaxBSlots) bs = kMaxBSlots;
  if (bs < 2) return B200SEG_E_BADARG;
  p.b_slots = bs;
  smem_bytes = fixed + (size_t)bs * p.b_slot_bytes;
  if (smem_bytes < 120 * 1024) smem_bytes = 120 * 1024;      // one CTA per SM
  return 0;
}

extern "C" int b200seg_conv2d_wgrad_plan_info(const b200seg_conv_desc* d, int32_t* out) {
  WgradParams p;
  size_t smem_bytes;
  if (!out) return B200SEG_E_BADARG;
  if (int rc = wgrad_plan(d, p, smem_bytes)) return rc;
  out[0] = p.ntile_w; out[1] = p.n_tiles; out[2] = p.taps_per_group; out[3] = p.tap_groups; out[4] = p.splits;
  out[5] = p.m_tiles; out[6] = p.total_units; out[7] = wgrad_grid(p);
  out[8] = p.b_slots; out[9] = (int32_t)smem_bytes;
  return 0;
}

extern "C" size_t b200seg_conv2d_wgrad_ws_bytes(const b200seg_conv_desc* d) {
  WgradParams p;
  size_t smem_bytes;
  if (wgrad_plan(d, p, smem_bytes) != 0) return 0;
  if (p.direct) return 16;   // no slabs: the workspace is not touched (a non-zero size keeps callers' allocation uniform)
  return (size_t)p.total_units * p.unit_stride * sizeof(float);
}

extern "C" int b200seg_conv2d_wgrad(const b200seg_conv_desc* d, const void* x, const void* dy, int32_t dy_ld,
                                    float* dw_ohwi, void* workspace, size_t ws_bytes, void* stream) {
  if (!d || !x || !dy || !dw_ohwi) return B200SEG_E_BADARG;
  if (dy_ld % 8 || dy_ld < 8) return B200SEG_E_BADARG;
  WgradParams p;
  size_t smem_bytes;
  int rc0 = wgrad_plan(d, p, smem_bytes);
  if (rc0) return rc0;
  if (reinterpret_cast<uintptr_t>(dw_ohwi) & 15) return B200SEG_E_BADARG;
  if (!p.direct) {
    if (!workspace || ws_bytes < (size_t)p.total_units * p.unit_stride * sizeof(float)) return B200SEG_E_BADARG;
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return B200SEG_E_BADARG;
  }

  CUtensorMap tmDy, tmX;
  {
    uint64_t dims[4] = {(uint64_t)((d->cout + 7) / 8 * 8), (uint64_t)p.Wo, (uint64_t)p.Ho, (uint64_t)d->n};
    uint64_t strides[3] = {(uint64_t)dy_ld * 2, (uint64_t)p.Wo * dy_ld * 2, (uint64_t)p.Ho * p.Wo * dy_ld * 2};
    uint32_t box[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, 1};
    int rc = encode_bf16(&tmDy, dy, 4, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  {
    uint64_t dims[4] = {(uint64_t)d->cin, (uint64_t)d->w, (uint64_t)d->h, (uint64_t)d->n};
    uint64_t strides[3] = {(uint64_t)d->x_ld * 2, (uint64_t)d->w * d->x_ld * 2, (uint64_t)d->h * d->w * d->x_ld * 2};
    uint32_t box[4] = {64, (uint32_t)(p.TW * d->stride), (uint32_t)(p.TH * d->stride), 1};
    uint32_t es[4] = {1, (uint32_t)d->stride, (uint32_t)d->stride, 1};
    int rc = encode_bf16(&tmX, x, 4, dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  const int w16 = p.unit_n / 16;                  // 1 .. 16 (the planner caps the N tile at kWAccCols columns)
  const WgradKernel kernel = wgrad_kernel(w16, std::make_integer_sequence<int, kWAccCols / 16>());
  static bool attr_set[kWAccCols / 16] = {};
  if (!attr_set[w16 - 1]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return (int)e;
    attr_set[w16 - 1] = true;
  }
  cudaError_t e = launch_k(kernel, dim3(wgrad_grid(p)), dim3(kWThreads), smem_bytes, (cudaStream_t)stream, tmDy, tmX, p,
                           (float*)workspace, dw_ohwi);
  if (e != cudaSuccess) return (int)e;
  if (p.direct) return 0;
  const int items = p.m_tiles * p.n_tiles * p.tap_groups;
  const int rows_max = p.Cout < 128 ? p.Cout : 128;
  const int f_max = p.taps_per_group * rows_max * (p.unit_n / 4);
  const int bpi = (f_max + 31) / 32;
  e = launch_k(wgrad_reduce_kernel, dim3(items * bpi), dim3(256), 0, (cudaStream_t)stream, p, (const float*)workspace,
               dw_ohwi, bpi);
  return e == cudaSuccess ? 0 : (int)e;
}

/* number of kernels b200seg_conv2d_wgrad launches for this shape (1: direct, 2: split + reduce) */
extern "C" int32_t b200seg_conv2d_wgrad_launches(const b200seg_conv_desc* d) {
  WgradParams p;
  size_t smem_bytes;
  if (wgrad_plan(d, p, smem_bytes) != 0) return 0;
  return p.direct ? 1 : 2;
}

extern "C" int32_t b200seg_grad_fold_chunk(void) { return kFoldChunk; }

extern "C" int b200seg_grad_fold(float* dst, float* acc_a, float* acc_b, const b200seg_grad_seg* segs,
                                 const int32_t* blk_seg, const int32_t* blk_start, int32_t n_blocks, int32_t mode,
                                 void* stream) {
  if (!dst || (!acc_a && !acc_b) || !segs || !blk_seg || !blk_start || n_blocks <= 0) return B200SEG_E_BADARG;
  cudaError_t e = launch_k(grad_fold_kernel, dim3(n_blocks), dim3(256), 0, (cudaStream_t)stream, dst, acc_a, acc_b,
                           segs, blk_seg, blk_start, (int)mode);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_publish_grads(float* dst, const float* src, int64_t n, const float* scale_dev, float scale_const,
                                     int32_t accumulate, void* stream) {
  if (!dst || !src || n <= 0 || (n & 3) || (reinterpret_cast<uintptr_t>(dst) & 15) ||
      (reinterpret_cast<uintptr_t>(src) & 15))
    return B200SEG_E_BADARG;
  cudaError_t e = launch_k(publish_grads_kernel, dim3(B200SEG_MAX_CTAS * 8), dim3(256), 0, (cudaStream_t)stream, dst, src,
                           (long long)(n / 4), scale_dev, scale_const, (int)accumulate);
  return e == cudaSuccess ? 0 : (int)e;
}
