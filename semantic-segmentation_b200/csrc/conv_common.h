#pragma once
#include <cstddef>
#include <cstdint>
struct b200seg_conv_desc;
namespace b200seg {
struct ConvPlan {
  int Ho, Wo;
  int KC, cchunks;
  int BN, n_tiles, cout_pad;
  int TH, TW, tiles_h, tiles_w, total_tiles, grid;
  int a_bytes, b_bytes, stage_bytes, nstages;
  int acc_regs, occ;     // fp32 accumulator registers per consumer thread (BN / 2), CTAs per SM
  size_t smem_bytes;
};
int conv_plan(const b200seg_conv_desc* d, ConvPlan* pl);
// Shared memory per SM the tensor-core kernels leave unused (b200seg_set_smem_reserve): in SyncBN mode a few one-warp
// waiter CTAs (1 KB of reserved shared memory each) must fit next to ANY convolution CTA, see bn_kernels.cu.
int smem_reserve();

// Launch-width tuning, read once from the environment (defaults: see tune() in conv_igemm.cu). The two-scale step keeps
// 8+ independent kernel chains in flight, so SM occupancy rather than the latency of one chain bounds it (B200SEG_DRY
// replays the captured program with empty kernels to show its launch / dependency floor). A launch that spreads a small
// layer over every SM pays
// its per-CTA fixed cost (prologue, pipeline fill, drain) once per SM or twice; these knobs give every CTA a minimum amount of
// work instead, so narrow launches of different streams run side by side.
struct Tune {
  int conv_min_clk;      // B200SEG_CONV_MIN_CLK: modelled tensor clocks of work per convolution CTA (0: widest grid)
  int wgrad_min_clk;     // B200SEG_WGRAD_MIN_CLK: the same per weight-gradient work unit (bounds the pixel splits)
  int ew_items;          // B200SEG_EW_ITEMS: 16-byte items per thread of the element-wise BatchNorm passes
  int ew_ctas_per_sm;    // B200SEG_EW_CTAS_PER_SM: grid cap of those passes (x SMs)
  int red_items;         // B200SEG_RED_ITEMS: pixel rows per thread of bn_bwd_reduce
  int red_ctas_per_sm;   // B200SEG_RED_CTAS_PER_SM
  int rs_items;          // B200SEG_RS_ITEMS: items per thread of the resample / fuse / accumulate passes
};
const Tune& tune();
// grid of a persistent convolution launch: min(tiles, slots), narrowed so that every CTA gets at least
// tune().conv_min_clk modelled clocks of work (tile_clk per tile)
int conv_grid_for(long long total_tiles, int slots, double tile_clk);
}  // namespace b200seg
