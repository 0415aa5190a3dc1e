// 3x3 / stride-1 / pad-1 convolution (forward and data gradient) with ONE halo tile per (pixel tile, channel chunk).
//
// The generic kernel (conv_igemm.cu) fetches a shifted 128-pixel box per filter tap, i.e. it reads the input 9 times
// from L2 — the limiter of HRNet's 48/96-channel high-resolution branch, which is HBM-bound on paper. Here the TMA unit
// brings a (16+2) x (8+2) pixel halo tile of a 64-channel chunk into shared memory ONCE, and the nine taps are nine
// wgmma shared-memory descriptors into that same tile. The tile is stored without swizzle as eight planes of 8 channels
// ([channel group][18][10][8 channels], 16 bytes per pixel of a plane, one TMA box of 8 channels per plane), so every
// 8-pixel run of a plane is one 8 x 16-byte core matrix at any pixel offset:
//     start = plane + (kh*10 + kw) * 16 B,   SBO = 10 * 16 B (next tile row),   LBO = plane pitch (next channel group)
// The weights use the same no-swizzle layout ([channel group][BN][8 channels]).
//
// Roles (288 threads): warps 0-7 = two consumer warpgroups (tile rows 0-7 / 8-15: MMA + epilogue), warp 8 = TMA producer.
// Weights: resident in shared memory for the whole persistent CTA when they fit (C <= 96: the HBM-bound layers), else
// streamed per (chunk, tap) through an mbarrier ring. The Cout tile (BN) is chosen per launch by a small cost model so
// that low-resolution layers still spread over the SMs (a 16x32x384 layer has 4 pixel tiles but 6 x 64-wide Cout tiles).
// Replaces cuDNN fwd/dgrad behind the 3x3 stride-1 convolutions of network/hrnetv2.py:31-34 (BasicBlock), :76
// (Bottleneck), network/ocrnet.py:54-57 (conv3x3_ocr) and network/utils.py:348-356 (attention head).
#include <cstdio>
#include "ptx.cuh"
#include "bn_fold.cuh"
#include "conv_common.h"
#include "conv_epi.cuh"
#include "tma_host.h"
#include "launch.h"
#include "../../include/b200seg.h"
#include <cstdlib>

namespace b200seg {

struct HaloParams {
  int N, H, W, Cin, Cout;      // H, W: spatial size (same for input and output)
  int cchunks;                 // ceil(Cin / 64)
  int ksteps_last;             // K=16 steps in the last chunk
  int BN, n_tiles, cout_pad;   // cout_pad = roundup16(Cout): row pitch of the statistics partials
  int tiles_h, tiles_w, total_tiles;
  int y_ld, has_bias, emit_stats, addend_ld;
  int resident;                // weights stay in smem for the CTA lifetime
  int a_slots, b_slots;        // ring depths (b_slots unused when resident)
  int b_tile_bytes;            // BN * 128 rounded to 1024
};

constexpr int kHThreads = 288;
constexpr int kASlotBytes = 24576;     // 8 planes x 2944 B = 23552, padded to a 1024 multiple
constexpr int kHaloW = 10, kHaloH = 18, kTW = 8, kTH = 16;
constexpr int kPlaneBytes = kHaloH * kHaloW * 16;   // one 8-channel plane of the halo tile (2880 B)
constexpr int kPlane = 2944;                         // plane pitch: TMA destinations are 128-byte aligned
constexpr int kMaxASlots = 4, kMaxBSlots2 = 8;

// OCC: CTAs per SM; the two-per-SM build holds at most 128 accumulator columns (64 registers per consumer thread).
template <int OCC>
__global__ void __launch_bounds__(kHThreads, OCC)
conv3x3_halo_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const HaloParams p, __nv_bfloat16* __restrict__ y, const float* __restrict__ bias,
                    float* __restrict__ stats_partials, const __nv_bfloat16* __restrict__ addend, const BnFoldDev fold) {
  constexpr int NB = OCC == 2 ? 8 : 16;    // 16-column accumulator blocks
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_base = smem;
  uint8_t* b_base = smem + (size_t)p.a_slots * kASlotBytes;
  const int b_tiles_total = p.resident ? 9 * p.cchunks : p.b_slots;
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_base + (size_t)b_tiles_total * p.b_tile_bytes);
  uint64_t* a_full = bars;                         // [kMaxASlots]
  uint64_t* a_empty = bars + kMaxASlots;
  uint64_t* b_full = bars + 2 * kMaxASlots;        // [kMaxBSlots2] (resident: only [0])
  uint64_t* b_empty = b_full + kMaxBSlots2;
  uint32_t* ticket = reinterpret_cast<uint32_t*>(b_empty + kMaxBSlots2);
  float* s_stats = reinterpret_cast<float*>(ticket + 4);   // [kStatSlots][2][cout_pad]

  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < p.a_slots; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 2); }
    for (int s = 0; s < kMaxBSlots2; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 2); }
    fence_barrier_init();
  }
  if (p.emit_stats)
    for (int i = threadIdx.x; i < kStatSlots * 2 * p.cout_pad; i += kHThreads) s_stats[i] = 0.f;
  __syncthreads();
  // Resident weights are static for the whole step (written by the pack kernels, which never trigger a programmatic
  // launch): fetch them while the previous kernel on the stream is still draining.
  if (warp == 8 && p.resident) {
    if (elect_one()) {
      mbar_arrive_expect_tx(&b_full[0], 9 * p.cchunks * p.b_tile_bytes);
      for (int cc = 0; cc < p.cchunks; ++cc)
        for (int t = 0; t < 9; ++t)
          for (int j = 0; j < 8; ++j)
            tma_load_3d(&tmB, &b_full[0], b_base + (size_t)(cc * 9 + t) * p.b_tile_bytes + j * p.BN * 16, cc * 64 + 8 * j,
                        t, 0);
    }
    __syncwarp();
  }
  pdl_sync();   // everything above overlapped the previous kernel's tail; activations are touched only below

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer (one elected lane)
    if (elect_one()) {
      int a_slot = 0, b_slot = 0;
      uint32_t a_phase = 0, b_phase = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int m_tile = tile / p.n_tiles, n_tile = tile - m_tile * p.n_tiles;
        const int tw_i = m_tile % p.tiles_w;
        const int th_i = (m_tile / p.tiles_w) % p.tiles_h;
        const int img = m_tile / (p.tiles_w * p.tiles_h);
        for (int cc = 0; cc < p.cchunks; ++cc) {
          mbar_wait(&a_empty[a_slot], a_phase ^ 1);
          mbar_arrive_expect_tx(&a_full[a_slot], 8 * kPlaneBytes);
          for (int j = 0; j < 8; ++j)
            tma_load_4d(&tmA, &a_full[a_slot], a_base + (size_t)a_slot * kASlotBytes + j * kPlane, cc * 64 + 8 * j,
                        tw_i * kTW - 1, th_i * kTH - 1, img);
          if (++a_slot == p.a_slots) { a_slot = 0; a_phase ^= 1; }
          if (!p.resident) {
            for (int t = 0; t < 9; ++t) {
              mbar_wait(&b_empty[b_slot], b_phase ^ 1);
              mbar_arrive_expect_tx(&b_full[b_slot], p.b_tile_bytes);
              for (int j = 0; j < 8; ++j)
                tma_load_3d(&tmB, &b_full[b_slot], b_base + (size_t)b_slot * p.b_tile_bytes + j * p.BN * 16,
                            cc * 64 + 8 * j, t, n_tile * p.BN);
              if (++b_slot == p.b_slots) { b_slot = 0; b_phase ^= 1; }
            }
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ------------------------------------------------------------------ consumers: MMA + epilogue
    const uint32_t g = warp >> 2;               // warpgroup: tile rows 8g .. 8g + 7
    const bool leader = (threadIdx.x & 127) == 0;
    float* my_stats = s_stats + (size_t)warp * 2 * p.cout_pad;
    const uint64_t a_tmpl = make_smem_desc(0, kPlane, kHaloW * 16, 0);
    const uint64_t b_tmpl = make_smem_desc(0, p.BN * 16, 128, 0);
    const uint32_t a0 = smem_u32(a_base) + g * 8 * kHaloW * 16, b0 = smem_u32(b_base);
    const uint32_t b64 = (64 * 16) >> 4;                  // 64 weight rows of 16 bytes
    const uint32_t bk16 = (uint32_t)(2 * p.BN * 16) >> 4;  // next K = 16 step: two channel-group planes
    const uint32_t ak16 = (2 * kPlane) >> 4;
    const int nb16 = p.BN >> 4;
    const int last = p.cchunks - 1;
    ConvEpi e{y, p.has_bias ? bias : nullptr, addend, p.y_ld, p.addend_ld, 0, p.Cout, p.emit_stats, p.cout_pad};
    float acc[NB * 8];
    int a_slot = 0, b_slot = 0;
    uint32_t a_phase = 0, b_phase = 0;
    if (p.resident) mbar_wait(&b_full[0], 0);
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      PendingRelease pend;
      for (int cc = 0; cc <= last; ++cc) {
        mbar_wait(&a_full[a_slot], a_phase);
        const uint64_t ad = a_tmpl + (uint64_t)((a0 + (uint32_t)a_slot * kASlotBytes) >> 4);
        const int ks = (cc == last) ? p.ksteps_last : 4;
        if (p.resident) {
          wgmma_fence();
          for (int t = 0; t < 9; ++t) {
            const int kh = t / 3, kw = t - kh * 3;
            const uint64_t at = ad + (uint64_t)(kh * kHaloW + kw);     // (kh*10 + kw) pixels of 16 B
            const uint64_t bt = b_tmpl + (uint64_t)((b0 + (uint32_t)(cc * 9 + t) * (uint32_t)p.b_tile_bytes) >> 4);
            for (int k = 0; k < ks; ++k)
              wgmma_row<NB, 0, 0>(acc, nb16, at + (uint64_t)(k * ak16), bt + (uint64_t)(k * bk16), b64, (cc | t | k) != 0);
          }
          wgmma_commit();
          wgmma_wait<1>();
          pend.release(leader);
          pend.bar0 = &a_empty[a_slot];
        } else {
          for (int t = 0; t < 9; ++t) {
            const int kh = t / 3, kw = t - kh * 3;
            mbar_wait(&b_full[b_slot], b_phase);
            const uint64_t at = ad + (uint64_t)(kh * kHaloW + kw);
            const uint64_t bt = b_tmpl + (uint64_t)((b0 + (uint32_t)b_slot * (uint32_t)p.b_tile_bytes) >> 4);
            wgmma_fence();
            for (int k = 0; k < ks; ++k)
              wgmma_row<NB, 0, 0>(acc, nb16, at + (uint64_t)(k * ak16), bt + (uint64_t)(k * bk16), b64, (cc | t | k) != 0);
            wgmma_commit();
            wgmma_wait<1>();
            pend.release(leader);
            pend.bar0 = &b_empty[b_slot];
            if (t == 8) pend.bar1 = &a_empty[a_slot];
            if (++b_slot == p.b_slots) { b_slot = 0; b_phase ^= 1; }
          }
        }
        if (++a_slot == p.a_slots) { a_slot = 0; a_phase ^= 1; }
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
        const int ho = th_i * kTH + (m >> 3), wo = tw_i * kTW + (m & 7);
        valid[r] = (ho < p.H) && (wo < p.W);
        pix[r] = ((size_t)img * p.H + ho) * p.W + wo;
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
      for (int i = threadIdx.x; i < 2 * p.cout_pad; i += kHThreads) {
        float v = 0.f;
        for (int s = 0; s < kStatSlots; ++s) v += s_stats[2 * s * p.cout_pad + i];
        out[i] = v;
      }
    }
  }
}

// Cout tile width: minimise (waves x per-tile clocks) with per-tile clocks = max(tensor issue, L2->smem fill).
// A narrow tile costs ~32 clocks per MMA regardless of N (the A operand read from shared memory bounds it).
// Two CTAs may share an SM when their Cout tile needs at most 128 accumulator columns (64 registers per consumer thread)
// and half of the shared memory: CTAs of DIFFERENT launches (the 0.5x and 1.0x
// passes, the HRNet branch streams, a PDL successor's prologue) then overlap their fill/drain latencies on one SM, and a
// 256-tile layer runs as one round of 264 slots instead of two rounds of 132. B200SEG_CORESIDENT=0 restores one CTA/SM.
static bool halo_coresident_enabled() {
  static const bool on = []() { const char* e = getenv("B200SEG_CORESIDENT"); return !(e && e[0] == '0'); }();
  return on;
}
constexpr size_t kHalfSmBudget = 115712;   // (228 KB - 2 x 1 KB reserved) / 2

// Shared-memory layout of a CTA for a given Cout tile: returns the CTAs per SM it allows (2, 1, or 0 = does not fit).
struct HaloSmem { int resident, a_slots, b_slots; size_t bytes; };
static int halo_smem_layout(int BN, int n_tiles, int cchunks, int cout_pad, HaloSmem& L) {
  const size_t b_tile = (size_t)(BN * 128 + 1023) / 1024 * 1024;
  const size_t fixed = 1024 + (2 * kMaxASlots + 2 * kMaxBSlots2) * 8 + 16 + (size_t)kStatSlots * 2 * cout_pad * 4;
  const size_t resident_bytes = (size_t)9 * cchunks * b_tile;
  for (int occ = (halo_coresident_enabled() && BN <= 128) ? 2 : 1; occ >= 1; --occ) {
    const size_t budget = (occ == 2 ? kHalfSmBudget : (size_t)227 * 1024) - fixed - (size_t)smem_reserve() / occ;
    if (n_tiles == 1 && resident_bytes + 2 * (size_t)kASlotBytes <= budget) {
      const int as_ = (int)((budget - resident_bytes) / kASlotBytes);
      L.resident = 1; L.a_slots = as_ > kMaxASlots ? kMaxASlots : as_; L.b_slots = 0;
      L.bytes = fixed + resident_bytes + (size_t)L.a_slots * kASlotBytes;
      return occ;
    }
    if (budget < 2 * (size_t)kASlotBytes + 2 * b_tile) continue;
    int bs = (int)((budget - 2 * (size_t)kASlotBytes) / b_tile);
    if (bs > kMaxBSlots2) bs = kMaxBSlots2;
    if (occ == 2 && bs < 4) continue;        // a two-deep weight ring starves the tensor pipe: take the whole SM instead
    L.resident = 0; L.a_slots = 2; L.b_slots = bs;
    L.bytes = fixed + 2 * (size_t)kASlotBytes + (size_t)bs * b_tile;
    return occ;
  }
  return 0;
}

static int halo_pick_ntiles(int m_tiles, int cout, int cchunks, int k16) {
  int best_nt = 0;
  double best = 0;
  const int cout_pad = (cout + 15) / 16 * 16;
  for (int nt = 1; nt <= 16; ++nt) {
    const int BN = ((cout + nt - 1) / nt + 15) / 16 * 16;
    if (BN > 256) continue;
    if ((cout + BN - 1) / BN != nt) continue;          // same split as a smaller nt
    HaloSmem L;
    if (halo_smem_layout(BN, nt, cchunks, cout_pad, L) == 0) continue;
    // Rounds are counted per SM, not per CTA slot: two co-resident CTAs share one tensor pipe and one L2->smem path, so
    // co-residency hides latency but adds no throughput; the tiling is the one measured with one CTA per SM.
    const long long tiles = (long long)m_tiles * nt;
    const double waves = (double)((tiles + B200SEG_MAX_CTAS - 1) / B200SEG_MAX_CTAS);
    const double mma = (double)k16 * (BN / 2 > 32 ? BN / 2 : 32);
    const double fill = ((double)cchunks * kHaloH * kHaloW * 128 + (double)k16 * 32.0 * BN) / 64.0;
    const double cost = waves * (mma > fill ? mma : fill) + 8.0 * BN + 2000.0 + 64.0 * nt;
    if (best_nt == 0 || cost < best) { best = cost; best_nt = nt; }
    if (BN <= 16) break;
  }
  return best_nt ? best_nt : 1;
}

// Host launcher shared by forward and stride-1 data gradient. `in` is the A-operand tensor [n,h,w,cin_ext] (pitch in_ld),
// w is [cout][9][cin_ext] bf16. Returns B200SEG_E_BADARG when the shape is not eligible (caller falls back to the
// generic per-tap kernel). The statistics partials are [grid][2][roundup16(cout)].
// Tiling / shared-memory / occupancy decisions of one launch (host only; also reported by b200seg_conv2d_plan_info).
static int halo_plan(int n, int h, int w, int cin, int cout, HaloParams& p, size_t& smem_bytes, int& grid, int& occ) {
  if (cin % 8 || cout % 16) return B200SEG_E_BADARG;
  p.N = n; p.H = h; p.W = w; p.Cin = cin; p.Cout = cout;
  p.cchunks = (cin + 63) / 64;
  const int rem = cin - (p.cchunks - 1) * 64;
  p.ksteps_last = (rem + 15) / 16;
  p.tiles_w = (w + kTW - 1) / kTW;
  p.tiles_h = (h + kTH - 1) / kTH;
  const int m_tiles = n * p.tiles_h * p.tiles_w;
  const int k16 = 9 * ((p.cchunks - 1) * 4 + p.ksteps_last);
  p.n_tiles = halo_pick_ntiles(m_tiles, cout, p.cchunks, k16);
  p.BN = ((cout + p.n_tiles - 1) / p.n_tiles + 15) / 16 * 16;
  p.cout_pad = (cout + 15) / 16 * 16;
  p.total_tiles = m_tiles * p.n_tiles;
  p.b_tile_bytes = (p.BN * 128 + 1023) / 1024 * 1024;
  HaloSmem L;
  occ = halo_smem_layout(p.BN, p.n_tiles, p.cchunks, p.cout_pad, L);
  if (occ >= 1) { p.resident = L.resident; p.a_slots = L.a_slots; p.b_slots = L.b_slots; smem_bytes = L.bytes; }
  if (occ < 1) return B200SEG_E_BADARG;
  // one CTA per SM unless the co-resident configuration was chosen (occupancy is bounded by shared memory and registers)
  if (occ == 1 && smem_bytes < 120 * 1024) smem_bytes = 120 * 1024;
  const int slots = occ == 2 ? B200SEG_MAX_GRID : B200SEG_MAX_CTAS;
  grid = conv_grid_for(p.total_tiles, slots, (double)k16 * (p.BN / 2 > 32 ? p.BN / 2 : 32));
  return 0;
}

// {kernel 1 = halo, BN, n_tiles, grid, smem bytes, ring depth (A slots), CTAs per SM, accumulator registers per consumer
// thread, resident weights, B slots}
int conv3x3_halo_plan_info(int n, int h, int w, int cin, int cout, int32_t* out) {
  HaloParams p;
  size_t smem_bytes;
  int grid, occ;
  if (int rc = halo_plan(n, h, w, cin, cout, p, smem_bytes, grid, occ)) return rc;
  out[0] = 1; out[1] = p.BN; out[2] = p.n_tiles; out[3] = grid; out[4] = (int32_t)smem_bytes; out[5] = p.a_slots;
  out[6] = occ; out[7] = p.BN / 2; out[8] = p.resident; out[9] = p.b_slots;
  return 0;
}

int make_bn_fold(const b200seg_bn_fold* f, int cout, BnFoldDev* out);
int conv3x3_halo_launch(int n, int h, int w, int cin, int in_ld, const void* in, int cout, const void* wts,
                        const float* bias, void* out, int out_ld, float* stats_partials, int32_t* stats_grid,
                        const void* addend, int addend_ld, int emit_stats, cudaStream_t stream,
                        const b200seg_bn_fold* fold, const BnFoldDev* affine) {
  if (in_ld % 8 || out_ld % 8) return B200SEG_E_BADARG;
  BnFoldDev fd;
  if (int frc = make_bn_fold(emit_stats ? fold : nullptr, cout, &fd)) return frc;
  if (affine) {                       // evaluation: BatchNorm folded into the epilogue (no statistics)
    if (emit_stats) return B200SEG_E_BADARG;
    fd = *affine;
  }
  if (emit_stats && !stats_partials && !fold) return B200SEG_E_BADARG;
  HaloParams p;
  size_t smem_bytes;
  int grid, occ;
  if (int rc = halo_plan(n, h, w, cin, cout, p, smem_bytes, grid, occ)) return rc;
  p.y_ld = out_ld; p.has_bias = bias != nullptr; p.emit_stats = emit_stats; p.addend_ld = addend_ld;
  if (stats_grid) *stats_grid = grid;
  if (!in || !wts || !out) return B200SEG_E_BADARG;
  if ((reinterpret_cast<uintptr_t>(in) & 15) || (reinterpret_cast<uintptr_t>(wts) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(addend) & 15) || (addend && addend_ld % 8))
    return B200SEG_E_BADARG;
  CUtensorMap tmA, tmB;
  {   // one box = one 8-channel plane of the halo tile
    uint64_t dims[4] = {(uint64_t)cin, (uint64_t)w, (uint64_t)h, (uint64_t)n};
    uint64_t strides[3] = {(uint64_t)in_ld * 2, (uint64_t)w * in_ld * 2, (uint64_t)h * w * in_ld * 2};
    uint32_t box[4] = {8, (uint32_t)kHaloW, (uint32_t)kHaloH, 1};
    int rc = encode_bf16(&tmA, in, 4, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
  }
  {   // one box = one 8-channel plane (BN rows x 16 bytes) of one tap
    uint64_t dims[3] = {(uint64_t)cin, 9, (uint64_t)cout};
    uint64_t strides[2] = {(uint64_t)cin * 2, (uint64_t)9 * cin * 2};
    uint32_t box[3] = {8, 1, (uint32_t)p.BN};
    int rc = encode_bf16(&tmB, wts, 3, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv3x3_halo_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(conv3x3_halo_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHalfSmBudget);
    if (e != cudaSuccess) return (int)e;
    // two CTAs per SM need (almost) the whole 228 KB as shared memory: ask for the maximum carve-out explicitly
    e = cudaFuncSetAttribute(conv3x3_halo_kernel<2>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  cudaError_t e =
      occ == 2 ? launch_k(conv3x3_halo_kernel<2>, dim3(grid), dim3(kHThreads), smem_bytes, stream, tmA, tmB, p,
                          (__nv_bfloat16*)out, bias, stats_partials, (const __nv_bfloat16*)addend, fd)
               : launch_k(conv3x3_halo_kernel<1>, dim3(grid), dim3(kHThreads), smem_bytes, stream, tmA, tmB, p,
                          (__nv_bfloat16*)out, bias, stats_partials, (const __nv_bfloat16*)addend, fd);
  return e == cudaSuccess ? 0 : (int)e;
}


// Diagnostics: CTAs per SM the runtime grants the co-resident (OCC = 2) and the full-SM (OCC = 1) build of the two
// convolution kernels for a given dynamic shared-memory size (registers, shared-memory carve-out, barriers all included).
int conv_igemm_occupancy(int occ_variant, int smem_bytes);
int conv3x3_halo_occupancy(int occ_variant, int smem_bytes) {
  int nb = -1;
  cudaFuncSetAttribute(conv3x3_halo_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  cudaFuncSetAttribute(conv3x3_halo_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHalfSmBudget);
  cudaFuncSetAttribute(conv3x3_halo_kernel<2>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaError_t e = occ_variant == 2
      ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, conv3x3_halo_kernel<2>, kHThreads, (size_t)smem_bytes)
      : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, conv3x3_halo_kernel<1>, kHThreads, (size_t)smem_bytes);
  return e == cudaSuccess ? nb : -(int)e;
}

template <typename K>
static void occupancy_report_one(const char* name, K kernel, int threads) {
  cudaFuncAttributes a;
  if (cudaFuncGetAttributes(&a, kernel) != cudaSuccess) { printf("%s: cudaFuncGetAttributes failed\n", name); return; }
  printf("%s: regs %d static smem %zu local %zu maxThreads %d maxDynSmem %d carveout %d\n  blocks/SM by dyn smem:", name,
         a.numRegs, a.sharedSizeBytes, a.localSizeBytes, a.maxThreadsPerBlock, a.maxDynamicSharedSizeBytes,
         a.preferredShmemCarveout);
  for (int kb = 0; kb <= 112; kb += 16) {
    int nb = -1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, threads, (size_t)kb * 1024);
    printf(" %dK:%d", kb, nb);
  }
  printf("\n");
}
void conv_igemm_occupancy_report();
}  // namespace b200seg

// Diagnostics (stdout): what the runtime knows about the convolution kernels and the SM (tools/gpu_occupancy.py).
extern "C" void b200seg_debug_occupancy_report(void) {
  cudaDeviceProp pr;
  int dev = 0;
  cudaGetDevice(&dev);
  cudaGetDeviceProperties(&pr, dev);
  printf("device %s: SMs %d regs/SM %d regs/block %d smem/SM %zu smem/block optin %zu reserved smem/block %zu "
         "max blocks/SM %d max threads/SM %d\n", pr.name, pr.multiProcessorCount, pr.regsPerMultiprocessor,
         pr.regsPerBlock, pr.sharedMemPerMultiprocessor, pr.sharedMemPerBlockOptin, pr.reservedSharedMemPerBlock,
         pr.maxBlocksPerMultiProcessor, pr.maxThreadsPerMultiProcessor);
  b200seg::conv3x3_halo_occupancy(2, 1024);     // sets the attributes of both builds
  b200seg::occupancy_report_one("conv3x3_halo_kernel<2>", b200seg::conv3x3_halo_kernel<2>, b200seg::kHThreads);
  b200seg::occupancy_report_one("conv3x3_halo_kernel<1>", b200seg::conv3x3_halo_kernel<1>, b200seg::kHThreads);
  b200seg::conv_igemm_occupancy_report();
  fflush(stdout);
}

extern "C" int32_t b200seg_debug_occupancy(int32_t kernel, int32_t occ_variant, int32_t smem_bytes) {
  if (occ_variant != 1 && occ_variant != 2) return B200SEG_E_BADARG;
  return kernel == 1 ? b200seg::conv3x3_halo_occupancy(occ_variant, smem_bytes)
                     : b200seg::conv_igemm_occupancy(occ_variant, smem_bytes);
}
