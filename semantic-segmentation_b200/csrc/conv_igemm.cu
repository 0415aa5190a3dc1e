// Implicit-GEMM convolution for sm_90a.
//
//   GEMM view:  D[pixels, cout] = sum over (tap, cin-chunk) A[pixels, chunk] * B[cout, chunk]^T
//   A operand:  NHWC activations fetched by 4-D tiled TMA boxes (chunk x TW x TH x 1). A filter tap is a shifted
//               box; out-of-image coordinates are zero-filled by the TMA unit, which *is* the im2col padding.
//               Stride-2 convolutions use the tensor map's element strides.
//   B operand:  bf16 weights [cout][tap][cin] through a 3-D map (chunk x 1 x BN).
//   MMA:        wgmma, M = 128 pixels (TH x TW patch) split over two consumer warpgroups of 64 rows, N = BN <= 256,
//               K = 16 per instruction, fp32 accumulators in registers.
//   Epilogue:   conv_epi.cuh, from the registers; BatchNorm sums of the *stored* values kept per warp (fixed order).
//   Schedule:   persistent CTAs, round-robin tiles; 288 threads: warps 0-7 consumers, warp 8 TMA producer.
//   Launch:     programmatic dependent launch (launch.h): the prologue overlaps the previous kernel's tail.
#include <cstdio>
#include <cstring>
#include "ptx.cuh"
#include <cstdlib>
#include "tma_host.h"
#include "launch.h"
#include "../../include/b200seg.h"
#include "conv_common.h"
#include "bn_fold.cuh"
#include "conv_epi.cuh"

namespace b200seg {

struct ConvKParams {
  int N, Ho, Wo, Cout;          // Ho/Wo: full output extent (addressing)
  int sub_H, sub_W;             // extent of the output sub-lattice this launch covers (== Ho/Wo unless strided dgrad)
  int in_stride;                // input sampling stride (forward conv stride; 1 for data gradients)
  int out_stride, out_off_h, out_off_w;   // output lattice: row = r*out_stride + out_off_h
  int ntaps;
  int tap_dh[9], tap_dw[9], tap_w[9];     // input offset and weight-tap index per filter tap
  int cchunks, KC, BN, n_tiles;
  int TH, TW, tiles_h, tiles_w, total_tiles;
  int y_ld, out_fp32, has_bias, emit_stats, cout_pad, addend_ld;
  int layout_type, sbo;
  int a_bytes, b_bytes, stage_bytes, nstages;
};

constexpr int kThreads = 288;
constexpr int kMaxStages = 8;
constexpr size_t kHalfSmBudget = 115712;   // (228 KB - 2 x 1 KB reserved) / 2: two CTAs per SM (see conv3x3_halo.cu)

// OCC: CTAs per SM; the two-per-SM build holds at most 128 accumulator columns (64 registers per consumer thread).
template <int OCC>
__global__ void __launch_bounds__(kThreads, OCC)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const ConvKParams p, void* __restrict__ y, const float* __restrict__ bias,
                  float* __restrict__ stats_partials, const __nv_bfloat16* __restrict__ addend, const BnFoldDev fold) {
  constexpr int NB = OCC == 2 ? 8 : 16;    // 16-column accumulator blocks
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages][A|B] (1024-aligned) | barriers | ticket | stats[kStatSlots][2][cout_pad]
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stage_base = smem;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)p.nstages * p.stage_bytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kMaxStages;
  uint32_t* ticket = reinterpret_cast<uint32_t*>(bars + 2 * kMaxStages);
  float* s_stats = reinterpret_cast<float*>(ticket + 4);

  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < p.nstages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    fence_barrier_init();
  }
  if (p.emit_stats) {
    for (int i = threadIdx.x; i < kStatSlots * 2 * p.cout_pad; i += kThreads) s_stats[i] = 0.f;
  }
  __syncthreads();
  pdl_sync();   // the prologue above overlapped the previous kernel; global memory is touched only below

  const int kblocks = p.ntaps * p.cchunks;

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer (one elected lane)
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int m_tile = tile / p.n_tiles, n_tile = tile - m_tile * p.n_tiles;
        const int tw_i = m_tile % p.tiles_w;
        const int th_i = (m_tile / p.tiles_w) % p.tiles_h;
        const int img = m_tile / (p.tiles_w * p.tiles_h);
        const int h0 = th_i * p.TH * p.in_stride;
        const int w0 = tw_i * p.TW * p.in_stride;
        const int n0 = n_tile * p.BN;
        for (int t = 0; t < p.ntaps; ++t)
          for (int cc = 0; cc < p.cchunks; ++cc) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = stage_base + (size_t)stage * p.stage_bytes;
            uint8_t* sb = sa + p.a_bytes;
            mbar_arrive_expect_tx(&full_bar[stage], p.a_bytes + p.b_bytes);
            tma_load_4d(&tmA, &full_bar[stage], sa, cc * p.KC, w0 + p.tap_dw[t], h0 + p.tap_dh[t], img);
            tma_load_3d(&tmB, &full_bar[stage], sb, cc * p.KC, p.tap_w[t], n0);
            if (++stage == p.nstages) { stage = 0; phase ^= 1; }
          }
      }
    }
    __syncwarp();
  } else {
    // ------------------------------------------------------------------ consumers: MMA + epilogue
    const uint32_t g = warp >> 2;              // warpgroup: pixel rows 64g .. 64g + 63 of the tile
    const bool leader = (threadIdx.x & 127) == 0;
    float* my_stats = s_stats + (size_t)warp * 2 * p.cout_pad;
    const uint64_t tmpl = make_smem_desc(0, 16, p.sbo, p.layout_type);
    const uint32_t s0 = smem_u32(stage_base);
    const uint32_t a_off = g * (uint32_t)(p.a_bytes / 2);
    const uint32_t b64 = (uint32_t)(64 * p.KC * 2) >> 4;
    const int ksteps = p.KC >> 4;
    const int nb16 = p.BN >> 4;
    ConvEpi e{y, p.has_bias ? bias : nullptr, addend, p.y_ld, p.addend_ld, p.out_fp32, p.Cout, p.emit_stats, p.cout_pad};
    float acc[NB * 8];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      PendingRelease pend;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = s0 + (uint32_t)stage * (uint32_t)p.stage_bytes;
        const uint64_t adesc = tmpl + (uint64_t)((sa + a_off) >> 4);
        const uint64_t bdesc = tmpl + (uint64_t)((sa + (uint32_t)p.a_bytes) >> 4);
        wgmma_fence();
        // advancing K by 16 bf16 = 32 bytes inside the swizzle atom: +2 in the 16-byte-unit address field
        for (int k = 0; k < ksteps; ++k)
          wgmma_row<NB, 0, 0>(acc, nb16, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), b64, (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();
        pend.release(leader);
        pend.bar0 = &empty_bar[stage];
        if (++stage == p.nstages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      pend.release(leader);
      if (tile + (int)gridDim.x >= p.total_tiles && g == 0 && (threadIdx.x & 127) == 0)
        pdl_launch_late();    // every MMA of this CTA is done: only the last epilogue and the statistics remain

      const int m_tile = tile / p.n_tiles, n_tile = tile - m_tile * p.n_tiles;
      const int tw_i = m_tile % p.tiles_w;
      const int th_i = (m_tile / p.tiles_w) % p.tiles_h;
      const int img = m_tile / (p.tiles_w * p.tiles_h);
      bool valid[2];
      size_t pix[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int m = (int)(g * 64 + (warp & 3) * 16 + (lane >> 2)) + 8 * r;   // accumulator row == pixel of the tile
        const int th = m / p.TW, tw = m - th * p.TW;
        const int hs = th_i * p.TH + th, ws = tw_i * p.TW + tw;
        valid[r] = (hs < p.sub_H) && (ws < p.sub_W);
        const int ho = hs * p.out_stride + p.out_off_h, wo = ws * p.out_stride + p.out_off_w;
        pix[r] = ((size_t)img * p.Ho + ho) * p.Wo + wo;
      }
      conv_epilogue<NB>(acc, nb16, n_tile * p.BN, valid, pix, e, fold, my_stats, lane);
    }
  }

  __syncthreads();
  if (p.emit_stats) {
    if (fold.accum != nullptr) {
      bn_fold_tail(fold, s_stats, p.cout_pad, ticket);          // statistics finalised by the last CTA of this launch
    } else {
      float* out = stats_partials + (size_t)blockIdx.x * 2 * p.cout_pad;
      for (int i = threadIdx.x; i < 2 * p.cout_pad; i += kThreads) {
        float v = 0.f;
        for (int s = 0; s < kStatSlots; ++s) v += s_stats[2 * s * p.cout_pad + i];
        out[i] = v;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------- host side
// Geometry of one launch: an implicit GEMM over an output lattice of sub_h x sub_w pixels per image.
struct LaunchGeom {
  int n, in_h, in_w, in_c, in_ld;       // operand A tensor
  int out_h, out_w, out_c, out_ld;      // full output tensor
  int sub_h, sub_w, in_stride, out_stride, out_off_h, out_off_w;
  int ntaps, tap_dh[9], tap_dw[9], tap_w[9], wtaps;   // wtaps = taps dimension of the weight tensor
  int out_fp32, has_bias, emit_stats, force_kc;
};

static bool coresident_enabled() {
  static const bool on = []() { const char* e = getenv("B200SEG_CORESIDENT"); return !(e && e[0] == '0'); }();
  return on;
}

static int plan_geom(const LaunchGeom& g, ConvPlan* pl) {
  if (g.n <= 0 || g.sub_h <= 0 || g.sub_w <= 0) return B200SEG_E_BADARG;
  if (g.in_c % 8 || g.in_ld % 8 || g.in_ld < g.in_c) return B200SEG_E_BADARG;
  if (g.out_c <= 0 || g.out_ld < g.out_c) return B200SEG_E_BADARG;
  if (!g.out_fp32 && (g.out_ld % 8)) return B200SEG_E_BADARG;
  pl->Ho = g.sub_h; pl->Wo = g.sub_w;
  // channel chunk / swizzle width: the widest of {64, 32, 16} that tiles cin without waste (zero-fill covers 720 and 48).
  int KC = 64;
  if (g.in_c % 64 != 0) {
    if (g.in_c % 32 == 0 && g.in_c < 256) KC = 32;
    else if (g.in_c == 16) KC = 16;
    else KC = 64;   // remainder chunk is zero-filled by TMA on both operands
  }
  if (g.force_kc == 16 || g.force_kc == 32 || g.force_kc == 64) KC = g.force_kc;   // test hook
  pl->KC = KC;
  pl->cchunks = (g.in_c + KC - 1) / KC;
  int TW = 16, TH = 8;
  if (g.sub_w <= 8) { TW = 8; TH = 16; }
  pl->TW = TW; pl->TH = TH;
  pl->tiles_w = (g.sub_w + TW - 1) / TW;
  pl->tiles_h = (g.sub_h + TH - 1) / TH;
  // N tile: every (tap, chunk) stage refetches its 128 x KC activation box from L2, so a tile costs about
  // k16 x (64 + BN/2) clocks (L2->smem fill of A and B at ~64 B/clk); pick the Cout split that minimises waves x tile.
  {
    const int cout16 = (g.out_c + 15) / 16 * 16;
    const int m_tiles = g.n * pl->tiles_h * pl->tiles_w;
    const int k16 = g.ntaps * pl->cchunks * (KC / 16);
    int best_nt = 0;
    double best = 0;
    for (int nt = 1; nt <= 16; ++nt) {
      const int BN = ((cout16 / 16 + nt - 1) / nt) * 16;
      if (BN > 256) continue;
      if ((cout16 + BN - 1) / BN != nt) continue;
      const long long tiles = (long long)m_tiles * nt;
      // rounds per SM (co-resident CTAs share the tensor pipe: latency hiding, not throughput)
      const double waves = (double)((tiles + B200SEG_MAX_CTAS - 1) / B200SEG_MAX_CTAS);
      const double cost = waves * k16 * (64.0 + BN / 2) + 8.0 * BN + 2000.0 + 64.0 * nt;
      if (best_nt == 0 || cost < best) { best = cost; best_nt = nt; }
      if (BN <= 16) break;
    }
    pl->n_tiles = best_nt;
    pl->BN = ((cout16 / 16 + best_nt - 1) / best_nt) * 16;
    pl->cout_pad = cout16;     // row pitch of the statistics partials (independent of the tiling)
  }
  pl->total_tiles = g.n * pl->tiles_h * pl->tiles_w * pl->n_tiles;
  pl->a_bytes = 128 * KC * 2;
  pl->b_bytes = pl->BN * KC * 2;
  pl->stage_bytes = (pl->a_bytes + pl->b_bytes + 1023) / 1024 * 1024;
  pl->acc_regs = pl->BN / 2;
  size_t fixed = 1024 /*align slack*/ + 2 * kMaxStages * 8 + 16 + (size_t)kStatSlots * 2 * pl->cout_pad * 4;
  // two CTAs per SM for narrow Cout tiles (<= 128 accumulator columns = 64 registers per consumer thread, half of the
  // shared memory each), so that CTAs of different launches overlap their fill / drain latencies on one SM; else one CTA
  // with the deepest ring
  int occ = (coresident_enabled() && pl->BN <= 128) ? 2 : 1;
  int nst = 0;
  for (; occ >= 1; --occ) {
    const size_t budget = (occ == 2 ? kHalfSmBudget : (size_t)227 * 1024) - fixed - (size_t)smem_reserve() / occ;
    nst = (int)(budget / pl->stage_bytes);
    if (nst > kMaxStages) nst = kMaxStages;
    if (nst >= (occ == 2 ? 3 : 2)) break;
  }
  if (occ < 1) return B200SEG_E_BADARG;
  pl->nstages = nst;
  pl->occ = occ;
  pl->smem_bytes = fixed + (size_t)nst * pl->stage_bytes;
  if (occ == 1 && pl->smem_bytes < 120 * 1024) pl->smem_bytes = 120 * 1024;   // one CTA per SM
  const int slots = occ == 2 ? B200SEG_MAX_GRID : B200SEG_MAX_CTAS;
  {
    const int k16 = g.ntaps * pl->cchunks * (KC / 16);
    pl->grid = conv_grid_for(pl->total_tiles, slots, (double)k16 * (64.0 + pl->BN / 2));
  }
  return 0;
}

static inline int conv_dil(const b200seg_conv_desc* d) { return d->dilation > 1 ? d->dilation : 1; }
static inline int conv_out(int in, const b200seg_conv_desc* d) {
  return (in + 2 * d->pad - conv_dil(d) * (d->ksize - 1) - 1) / d->stride + 1;
}

static LaunchGeom fwd_geom(const b200seg_conv_desc* d) {
  LaunchGeom g{};
  const int dil = conv_dil(d);
  g.n = d->n; g.in_h = d->h; g.in_w = d->w; g.in_c = d->cin; g.in_ld = d->x_ld;
  g.out_h = conv_out(d->h, d);
  g.out_w = conv_out(d->w, d);
  g.out_c = d->cout; g.out_ld = d->y_ld;
  g.sub_h = g.out_h; g.sub_w = g.out_w;
  g.in_stride = d->stride; g.out_stride = 1; g.out_off_h = g.out_off_w = 0;
  g.ntaps = d->ksize * d->ksize; g.wtaps = g.ntaps;
  for (int kh = 0; kh < d->ksize; ++kh)
    for (int kw = 0; kw < d->ksize; ++kw) {
      const int t = kh * d->ksize + kw;
      g.tap_dh[t] = kh * dil - d->pad; g.tap_dw[t] = kw * dil - d->pad; g.tap_w[t] = t;
    }
  g.out_fp32 = d->out_fp32; g.has_bias = d->has_bias; g.emit_stats = d->emit_stats; g.force_kc = d->reserved;
  return g;
}

static bool desc_ok(const b200seg_conv_desc* d) {
  if (!d || d->n <= 0 || d->h <= 0 || d->w <= 0) return false;
  const int dil = d->dilation > 1 ? d->dilation : 1;
  if (!((d->ksize == 1 && d->pad == 0 && dil == 1) || (d->ksize == 3 && d->pad == dil))) return false;
  if (d->stride != 1 && d->stride != 2) return false;
  if (dil > 1 && d->stride != 1) return false;       // dilated layers of the path are all stride 1
  return true;
}

static int g_smem_reserve = 0;
int smem_reserve() { return g_smem_reserve; }

static int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return (e && e[0]) ? atoi(e) : dflt;
}
const Tune& tune() {
  static const Tune t = {env_int("B200SEG_CONV_MIN_CLK", 0),    env_int("B200SEG_WGRAD_MIN_CLK", 0),
                         env_int("B200SEG_EW_ITEMS", 8),        env_int("B200SEG_EW_CTAS_PER_SM", 8),
                         env_int("B200SEG_RED_ITEMS", 8),       env_int("B200SEG_RED_CTAS_PER_SM", 2),
                         env_int("B200SEG_RS_ITEMS", 1)};
  return t;
}
// grid of a persistent convolution launch: every CTA gets at least conv_min_clk modelled clocks of tiles
static int conv_grid(long long total_tiles, int slots, double tile_clk) {
  long long g = total_tiles < slots ? total_tiles : slots;
  const int min_clk = tune().conv_min_clk;
  if (min_clk > 0) {
    long long want = (long long)((double)total_tiles * tile_clk / (double)min_clk + 0.999);
    if (want < 1) want = 1;
    if (want < g) g = want;
  }
  return (int)g;
}
int conv_grid_for(long long total_tiles, int slots, double tile_clk) { return conv_grid(total_tiles, slots, tile_clk); }

int conv_plan(const b200seg_conv_desc* d, ConvPlan* pl) {
  if (!desc_ok(d)) return B200SEG_E_BADARG;
  return plan_geom(fwd_geom(d), pl);
}

int make_bn_fold(const b200seg_bn_fold* f, int cout, BnFoldDev* out) {
  BnFoldDev d;
  memset(&d, 0, sizeof(d));
  if (f) {
    if (!f->accum || f->c != cout || (reinterpret_cast<uintptr_t>(f->accum) & 7)) return B200SEG_E_BADARG;
    // counter == NULL: deferred mode, only the cells are touched (see bn_fold.cuh)
    if (f->counter && (!f->scale || !f->shift || !f->mean || !f->invstd || f->count <= 0.f)) return B200SEG_E_BADARG;
    d.accum = f->accum; d.counter = f->counter; d.gamma = f->gamma; d.beta = f->beta;
    d.scale = f->scale; d.shift = f->shift; d.mean = f->mean; d.invstd = f->invstd; d.batch_out = f->batch_stats_out;
    d.running_mean = f->running_mean; d.running_var = f->running_var; d.nbt = (long long*)f->num_batches_tracked;
    d.eps = f->eps; d.momentum = f->momentum; d.count = f->count; d.C = f->c;
  }
  *out = d;
  return 0;
}

static int launch_geom(const LaunchGeom& g, const void* a, const void* w, const float* bias, void* out,
                       float* stats_partials, int32_t* stats_grid, const void* addend, int addend_ld,
                       cudaStream_t stream, const b200seg_bn_fold* fold = nullptr, const BnFoldDev* affine = nullptr) {
  ConvPlan pl;
  int rc = plan_geom(g, &pl);
  if (rc) return rc;
  if (!a || !w || !out) return B200SEG_E_BADARG;
  if (g.has_bias && !bias) return B200SEG_E_BADARG;
  if (g.emit_stats && ((!stats_partials && !fold) || g.out_fp32)) return B200SEG_E_BADARG;
  BnFoldDev fd;
  if (int frc = make_bn_fold(g.emit_stats ? fold : nullptr, g.out_c, &fd)) return frc;
  if (affine) {                       // evaluation: BatchNorm folded into the epilogue (no statistics)
    if (g.emit_stats) return B200SEG_E_BADARG;
    fd = *affine;
  }
  if ((reinterpret_cast<uintptr_t>(a) & 15) || (reinterpret_cast<uintptr_t>(w) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(addend) & 15))
    return B200SEG_E_BADARG;
  if (addend && (addend_ld % 8)) return B200SEG_E_BADARG;

  CUtensorMap tmA, tmB;
  {
    uint64_t dims[4] = {(uint64_t)g.in_c, (uint64_t)g.in_w, (uint64_t)g.in_h, (uint64_t)g.n};
    uint64_t strides[3] = {(uint64_t)g.in_ld * 2, (uint64_t)g.in_w * g.in_ld * 2,
                           (uint64_t)g.in_h * g.in_w * g.in_ld * 2};
    uint32_t box[4] = {(uint32_t)pl.KC, (uint32_t)(pl.TW * g.in_stride), (uint32_t)(pl.TH * g.in_stride), 1};
    uint32_t es[4] = {1, (uint32_t)g.in_stride, (uint32_t)g.in_stride, 1};
    rc = encode_bf16(&tmA, a, 4, dims, strides, box, es, swizzle_for_bytes(pl.KC * 2));
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {(uint64_t)g.in_c, (uint64_t)g.wtaps, (uint64_t)g.out_c};
    uint64_t strides[2] = {(uint64_t)g.in_c * 2, (uint64_t)g.wtaps * g.in_c * 2};
    uint32_t box[3] = {(uint32_t)pl.KC, 1, (uint32_t)pl.BN};
    rc = encode_bf16(&tmB, w, 3, dims, strides, box, nullptr, swizzle_for_bytes(pl.KC * 2));
    if (rc) return rc;
  }
  ConvKParams p;
  p.N = g.n; p.Ho = g.out_h; p.Wo = g.out_w; p.Cout = g.out_c;
  p.sub_H = g.sub_h; p.sub_W = g.sub_w;
  p.in_stride = g.in_stride; p.out_stride = g.out_stride; p.out_off_h = g.out_off_h; p.out_off_w = g.out_off_w;
  p.ntaps = g.ntaps;
  for (int t = 0; t < 9; ++t) { p.tap_dh[t] = g.tap_dh[t]; p.tap_dw[t] = g.tap_dw[t]; p.tap_w[t] = g.tap_w[t]; }
  p.cchunks = pl.cchunks; p.KC = pl.KC; p.BN = pl.BN; p.n_tiles = pl.n_tiles;
  p.TH = pl.TH; p.TW = pl.TW; p.tiles_h = pl.tiles_h; p.tiles_w = pl.tiles_w; p.total_tiles = pl.total_tiles;
  p.y_ld = g.out_ld; p.out_fp32 = g.out_fp32; p.has_bias = g.has_bias; p.emit_stats = g.emit_stats;
  p.cout_pad = pl.cout_pad; p.addend_ld = addend_ld;
  p.layout_type = pl.KC == 64 ? 1 : (pl.KC == 32 ? 2 : 3);   // 128B / 64B / 32B swizzle
  p.sbo = 8 * pl.KC * 2;
  p.a_bytes = pl.a_bytes; p.b_bytes = pl.b_bytes; p.stage_bytes = pl.stage_bytes; p.nstages = pl.nstages;

  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_igemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(conv_igemm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHalfSmBudget);
    if (e != cudaSuccess) return (int)e;
    // two CTAs per SM need (almost) the whole 228 KB as shared memory: ask for the maximum carve-out explicitly
    e = cudaFuncSetAttribute(conv_igemm_kernel<2>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  if (stats_grid) *stats_grid = pl.grid;
  cudaError_t e =
      pl.occ == 2 ? launch_k(conv_igemm_kernel<2>, dim3(pl.grid), dim3(kThreads), pl.smem_bytes, stream, tmA, tmB, p, out,
                             bias, stats_partials, (const __nv_bfloat16*)addend, fd)
                  : launch_k(conv_igemm_kernel<1>, dim3(pl.grid), dim3(kThreads), pl.smem_bytes, stream, tmA, tmB, p, out,
                             bias, stats_partials, (const __nv_bfloat16*)addend, fd);
  return e == cudaSuccess ? 0 : (int)e;
}

int conv_igemm_occupancy(int occ_variant, int smem_bytes) {
  int nb = -1;
  cudaFuncSetAttribute(conv_igemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  cudaFuncSetAttribute(conv_igemm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHalfSmBudget);
  cudaFuncSetAttribute(conv_igemm_kernel<2>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaError_t e = occ_variant == 2
      ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, conv_igemm_kernel<2>, kThreads, (size_t)smem_bytes)
      : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, conv_igemm_kernel<1>, kThreads, (size_t)smem_bytes);
  return e == cudaSuccess ? nb : -(int)e;
}

void conv_igemm_occupancy_report() {
  conv_igemm_occupancy(2, 1024);
  for (int v = 2; v >= 1; --v) {
    cudaFuncAttributes a;
    if (v == 2) cudaFuncGetAttributes(&a, conv_igemm_kernel<2>); else cudaFuncGetAttributes(&a, conv_igemm_kernel<1>);
    printf("conv_igemm_kernel<%d>: regs %d static smem %zu local %zu maxThreads %d maxDynSmem %d carveout %d\n  blocks/SM by dyn smem:",
           v, a.numRegs, a.sharedSizeBytes, a.localSizeBytes, a.maxThreadsPerBlock, a.maxDynamicSharedSizeBytes,
           a.preferredShmemCarveout);
    for (int kb = 0; kb <= 112; kb += 16) printf(" %dK:%d", kb, conv_igemm_occupancy(v, kb * 1024));
    printf("\n");
  }
}

int conv3x3_halo_launch(int n, int h, int w, int cin, int in_ld, const void* in, int cout, const void* wts,
                        const float* bias, void* out, int out_ld, float* stats_partials, int32_t* stats_grid,
                        const void* addend, int addend_ld, int emit_stats, cudaStream_t stream,
                        const b200seg_bn_fold* fold = nullptr, const BnFoldDev* affine = nullptr);
int conv3x3_halo_plan_info(int n, int h, int w, int cin, int cout, int32_t* out);

}  // namespace b200seg

using namespace b200seg;

extern "C" size_t b200seg_conv2d_stats_elems(const b200seg_conv_desc* d) {
  ConvPlan pl;
  if (conv_plan(d, &pl) != 0) return 0;
  return (size_t)B200SEG_MAX_GRID * 2 * ((d->cout + 15) / 16 * 16);   // [grid <= B200SEG_MAX_GRID][2][roundup16(cout)]
}

// Host-only: the launch plan of a forward (which = 0) or stride-1 data-gradient (which = 1) convolution, for tests and
// tuning scripts. out[10] = {kernel (1 halo / 0 per-tap), BN, n_tiles, grid, dynamic smem bytes, ring depth, CTAs per SM,
// accumulator registers per consumer thread, resident weights (halo), weight slots (halo)}.
extern "C" int b200seg_conv2d_plan_info(const b200seg_conv_desc* d, int32_t which, int32_t* out) {
  if (!desc_ok(d) || !out || which < 0 || which > 1) return B200SEG_E_BADARG;
  if (which == 1 && d->stride != 1) return B200SEG_E_BADARG;
  const bool halo_fwd = d->ksize == 3 && d->stride == 1 && !d->out_fp32 && d->cout % 16 == 0 && d->reserved == 0;
  const bool halo_bwd = d->ksize == 3 && d->cin % 16 == 0 && d->reserved == 0;
  if (which == 0 && halo_fwd) return conv3x3_halo_plan_info(d->n, d->h, d->w, d->cin, d->cout, out);
  if (which == 1 && halo_bwd) return conv3x3_halo_plan_info(d->n, d->h, d->w, (d->cout + 7) / 8 * 8, d->cin, out);
  LaunchGeom g = fwd_geom(d);
  if (which == 1) {          // same GEMM shape with the channel roles swapped (taps and lattice as the forward)
    g.in_c = (d->cout + 7) / 8 * 8; g.in_ld = g.in_c; g.out_c = d->cin; g.out_ld = d->cin;
    g.out_fp32 = 0; g.has_bias = 0; g.emit_stats = 0;
  }
  ConvPlan pl;
  if (int rc = plan_geom(g, &pl)) return rc;
  out[0] = 0; out[1] = pl.BN; out[2] = pl.n_tiles; out[3] = pl.grid; out[4] = (int32_t)pl.smem_bytes; out[5] = pl.nstages;
  out[6] = pl.occ; out[7] = pl.acc_regs; out[8] = 0; out[9] = 0;
  return 0;
}

extern "C" int b200seg_conv2d_fwd(const b200seg_conv_desc* d, const void* x, const void* w_ohwi, const float* bias,
                                  void* y, float* stats_partials, int32_t* stats_grid, void* stream) {
  if (!desc_ok(d)) return B200SEG_E_BADARG;
  if (d->ksize == 3 && d->stride == 1 && !d->out_fp32 && d->cout % 16 == 0 && d->reserved == 0 && conv_dil(d) == 1) {
    if (d->emit_stats && !stats_partials) return B200SEG_E_BADARG;
    // halo-tile kernel: the input is read once per tile instead of once per filter tap (conv3x3_halo.cu)
    return conv3x3_halo_launch(d->n, d->h, d->w, d->cin, d->x_ld, x, d->cout, w_ohwi, d->has_bias ? bias : nullptr, y,
                               d->y_ld, stats_partials, stats_grid, nullptr, 0, d->emit_stats, (cudaStream_t)stream);
  }
  return launch_geom(fwd_geom(d), x, w_ohwi, bias, y, stats_partials, stats_grid, nullptr, 0, (cudaStream_t)stream);
}

extern "C" int b200seg_set_smem_reserve(int32_t bytes) {
  if (bytes < 0 || bytes > 64 * 1024) return B200SEG_E_BADARG;
  g_smem_reserve = (bytes + 1023) / 1024 * 1024;
  return 0;
}

extern "C" int b200seg_conv2d_fwd_bn(const b200seg_conv_desc* d, const void* x, const void* w_ohwi, const float* bias,
                                     void* y, const b200seg_bn_fold* fold, void* stream) {
  if (!desc_ok(d) || !fold || !d->emit_stats || d->out_fp32) return B200SEG_E_BADARG;
  if (d->ksize == 3 && d->stride == 1 && d->cout % 16 == 0 && d->reserved == 0 && conv_dil(d) == 1)
    return conv3x3_halo_launch(d->n, d->h, d->w, d->cin, d->x_ld, x, d->cout, w_ohwi, d->has_bias ? bias : nullptr, y,
                               d->y_ld, nullptr, nullptr, nullptr, 0, 1, (cudaStream_t)stream, fold);
  return launch_geom(fwd_geom(d), x, w_ohwi, bias, y, nullptr, nullptr, nullptr, 0, (cudaStream_t)stream, fold);
}

// Forward convolution with a residual addend in the epilogue: y = conv(x) (+ bias) + addend, statistics of the stored sum.
// The identity-mapping blocks of WideResNet-38 (network/wider_resnet.py:170-183 `out.add_(shortcut)`) feed that sum into
// the next block's pre-activation BatchNorm, so the batch statistics come for free from this epilogue.
extern "C" int b200seg_conv2d_fwd_add(const b200seg_conv_desc* d, const void* x, const void* w_ohwi, const float* bias,
                                      const void* addend, int32_t addend_ld, void* y, float* stats_partials,
                                      int32_t* stats_grid, void* stream) {
  if (!desc_ok(d) || !addend || d->out_fp32) return B200SEG_E_BADARG;
  if (d->emit_stats && !stats_partials) return B200SEG_E_BADARG;
  if (d->ksize == 3 && d->stride == 1 && d->cout % 16 == 0 && d->reserved == 0 && conv_dil(d) == 1)
    return conv3x3_halo_launch(d->n, d->h, d->w, d->cin, d->x_ld, x, d->cout, w_ohwi, d->has_bias ? bias : nullptr, y,
                               d->y_ld, stats_partials, stats_grid, addend, addend_ld, d->emit_stats, (cudaStream_t)stream);
  return launch_geom(fwd_geom(d), x, w_ohwi, bias, y, stats_partials, stats_grid, addend, addend_ld, (cudaStream_t)stream);
}

// Evaluation: y = relu?(conv(x) * scale[co] + shift[co] (+ addend)) in the convolution epilogue (BatchNorm from running
// statistics, residual sum and ReLU of network/hrnetv2.py:50-66,86-106 in one launch). bf16 output, no statistics.
extern "C" int b200seg_conv2d_fwd_affine(const b200seg_conv_desc* d, const void* x, const void* w_ohwi,
                                         const float* scale, const float* shift, int32_t relu, const void* addend,
                                         int32_t addend_ld, void* y, void* stream) {
  if (!desc_ok(d) || !scale || !shift || d->out_fp32 || d->emit_stats || d->has_bias) return B200SEG_E_BADARG;
  BnFoldDev fd;
  memset(&fd, 0, sizeof(fd));
  fd.scale = const_cast<float*>(scale);
  fd.shift = const_cast<float*>(shift);
  fd.relu = relu ? 1 : 0;
  fd.C = d->cout;
  if (d->ksize == 3 && d->stride == 1 && d->cout % 16 == 0 && d->reserved == 0 && conv_dil(d) == 1)
    return conv3x3_halo_launch(d->n, d->h, d->w, d->cin, d->x_ld, x, d->cout, w_ohwi, nullptr, y, d->y_ld, nullptr,
                               nullptr, addend, addend_ld, 0, (cudaStream_t)stream, nullptr, &fd);
  return launch_geom(fwd_geom(d), x, w_ohwi, nullptr, y, nullptr, nullptr, addend, addend_ld, (cudaStream_t)stream,
                     nullptr, &fd);
}

// Data gradient. d describes the FORWARD convolution. dx[n,h,w,cin] = sum_taps dy[...] * W  (+ addend).
//   stride 1: one launch, a 3x3 (or 1x1) convolution of dy with the flipped, transposed weights;
//   stride 2: four launches, one per output parity class (a,b): dx[2u+a, 2v+b] only receives the taps with
//             kh = a+1 (mod 2), kw = b+1 (mod 2), read from dy[u + (a+1-kh)/2, v + (b+1-kw)/2].
extern "C" int b200seg_conv2d_dgrad(const b200seg_conv_desc* d, const void* dy, int32_t dy_ld, const void* w_dgrad,
                                    const void* addend, int32_t addend_ld, void* dx, int32_t dx_ld, void* stream) {
  if (!desc_ok(d)) return B200SEG_E_BADARG;
  const int Ho = conv_out(d->h, d);
  const int Wo = conv_out(d->w, d);
  const int K = d->ksize, taps = K * K;
  const int dil = conv_dil(d);
  LaunchGeom g{};
  g.n = d->n; g.in_h = Ho; g.in_w = Wo; g.in_c = (d->cout + 7) / 8 * 8; g.in_ld = dy_ld;
  g.out_h = d->h; g.out_w = d->w; g.out_c = d->cin; g.out_ld = dx_ld;
  g.in_stride = 1; g.wtaps = taps;
  g.out_fp32 = 0; g.has_bias = 0; g.emit_stats = 0; g.force_kc = d->reserved;
  if (d->stride == 1 && K == 3 && d->cin % 16 == 0 && d->reserved == 0 && dil == 1)
    return conv3x3_halo_launch(d->n, d->h, d->w, g.in_c, dy_ld, dy, d->cin, w_dgrad, nullptr, dx, dx_ld, nullptr, nullptr,
                               addend, addend_ld, 0, (cudaStream_t)stream);
  if (d->stride == 1) {
    g.sub_h = d->h; g.sub_w = d->w; g.out_stride = 1; g.out_off_h = g.out_off_w = 0;
    g.ntaps = taps;
    for (int kh = 0; kh < K; ++kh)
      for (int kw = 0; kw < K; ++kw) {
        const int t = kh * K + kw;
        g.tap_dh[t] = d->pad - kh * dil; g.tap_dw[t] = d->pad - kw * dil; g.tap_w[t] = taps - 1 - t;
      }
    return launch_geom(g, dy, w_dgrad, nullptr, dx, nullptr, nullptr, addend, addend_ld, (cudaStream_t)stream);
  }
  if (K == 1) {
    // 1x1 stride-2 (WideResNet-38 proj_conv of mod4.block1): only the even lattice receives a gradient. The caller hands
    // in dx either zero-filled or as the in-place accumulation target (addend == dx); the odd lattice is left untouched.
    if (addend != nullptr && addend != dx) return B200SEG_E_BADARG;
    g.sub_h = (d->h + 1) / 2; g.sub_w = (d->w + 1) / 2;
    g.out_stride = 2; g.out_off_h = 0; g.out_off_w = 0;
    g.ntaps = 1; g.tap_dh[0] = 0; g.tap_dw[0] = 0; g.tap_w[0] = 0;
    return launch_geom(g, dy, w_dgrad, nullptr, dx, nullptr, nullptr, addend, addend_ld, (cudaStream_t)stream);
  }
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      g.sub_h = (d->h - a + 1) / 2; g.sub_w = (d->w - b + 1) / 2;
      if (g.sub_h <= 0 || g.sub_w <= 0) continue;
      g.out_stride = 2; g.out_off_h = a; g.out_off_w = b;
      g.ntaps = 0;
      for (int kh = 0; kh < 3; ++kh) {
        if (((a + 1 - kh) & 1) != 0) continue;
        for (int kw = 0; kw < 3; ++kw) {
          if (((b + 1 - kw) & 1) != 0) continue;
          g.tap_dh[g.ntaps] = (a + 1 - kh) / 2; g.tap_dw[g.ntaps] = (b + 1 - kw) / 2;
          g.tap_w[g.ntaps] = taps - 1 - (kh * 3 + kw);
          ++g.ntaps;
        }
      }
      int rc = launch_geom(g, dy, w_dgrad, nullptr, dx, nullptr, nullptr, addend, addend_ld, (cudaStream_t)stream);
      if (rc) return rc;
    }
  return 0;
}
