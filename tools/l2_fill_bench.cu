// L2 -> shared-memory fill rate of the convolution weight (B operand) loads, with and without 2-CTA TMA multicast.
// One producer warp streams the weight tiles of one Cout tile through a ring of shared-memory slots in the box shapes
// the kernels use (conv3x3_halo_kernel: eight {8 channels, 1 tap, BN rows} planes, no swizzle; conv_igemm_kernel: one
// {64 channels, 1 tap, BN rows} box, 128-byte swizzle); one consumer warp releases each slot as soon as it has landed, so
// the loop runs at the rate the memory system delivers. With multicast each CTA of a 2-CTA cluster issues half of every
// tile to both CTAs (halo: four planes; igemm: BN / 2 rows) and a slot is refilled once both CTAs have released it.
// planes: the halo tile from the plane-ordered weight image ([tap][Cin/8][Cout rows][8], include/b200seg.h), one 1-D
// cp.async.bulk of BN x 16 contiguous bytes per plane into the same shared-memory image as the halo boxes.
// Built and run by tools/gpu_l2_fill_bench.py:
//   l2_fill_bench <halo|igemm|planes> <cin> <cout> <BN> <CTAs per SM> <multicast 0|1> <tiles per CTA> [ring slots]
// prints one JSON line.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../semantic-segmentation_b200/csrc/ptx.cuh"
#include "../semantic-segmentation_b200/csrc/tma_host.h"

using namespace b200seg;

struct FillParams {
  int halo, planes, cin, BN, n_tiles, k_tiles, slots, tile_bytes, iters, multicast, cout_rows;
};

// ---------------------------------------------------------------- 2-CTA clusters (valid in a launch without clusters too)
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at the same shared-memory offset in the other CTA of the cluster
__device__ __forceinline__ void mbar_arrive_peer(uint32_t bar) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(bar), "r"(cluster_ctarank() ^ 1u));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// mc: the box goes to the same shared-memory offset of both CTAs, each signalled on the barrier at bar's offset
__device__ __forceinline__ void load_3d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2, bool mc) {
  if (mc)
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4, %5}], [%2], %6;"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "h"((uint16_t)3)
        : "memory");
  else
    tma_load_3d(m, bar, dst, c0, c1, c2);
}

__global__ void __launch_bounds__(64) l2_fill_kernel(const __grid_constant__ CUtensorMap tm, const FillParams p,
                                                      const uint8_t* __restrict__ image) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + (size_t)p.slots * p.tile_bytes);
  uint64_t* empty = full + 8;
  const int cs = p.multicast ? 2 : 1;
  const uint32_t rank = cluster_ctarank();
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.slots; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], cs); }
    fence_barrier_init();
  }
  cluster_sync();
  const int n0 = ((int)(blockIdx.x / cs) % p.n_tiles) * p.BN;
  if (threadIdx.x < 32) {
    if (elect_one()) {
      for (int i = 0; i < p.iters; ++i) {
        const int s = i % p.slots, k = i % p.k_tiles, cc = k / 9, t = k - cc * 9;
        mbar_wait(&empty[s], ((i / p.slots) & 1) ^ 1);
        mbar_arrive_expect_tx(&full[s], p.tile_bytes);
        uint8_t* dst = ring + (size_t)s * p.tile_bytes;
        if (p.planes) {
          const int G = (p.cin + 63) / 64 * 8;   // the benchmark's image carries every plane of the last chunk
          for (int j = 0; j < 8; ++j)
            bulk_load(dst + j * p.BN * 16, image + ((size_t)(t * G + 8 * cc + j) * p.cout_rows + n0) * 16, p.BN * 16,
                      &full[s]);
        } else if (p.halo) {
          for (int j = p.multicast ? 4 * (int)rank : 0, je = p.multicast ? j + 4 : 8; j < je; ++j)
            load_3d(&tm, &full[s], dst + j * p.BN * 16, cc * 64 + 8 * j, t, n0, p.multicast);
        } else {
          const int rows = p.BN / cs;
          for (int h = p.multicast ? (int)rank : 0, he = p.multicast ? h + 1 : 1; h < he; ++h)
            load_3d(&tm, &full[s], dst + h * rows * 128, cc * 64, t, n0 + h * rows, p.multicast);
        }
      }
    }
    __syncwarp();
  } else if (threadIdx.x == 32) {
    for (int i = 0; i < p.iters; ++i) {
      const int s = i % p.slots;
      mbar_wait(&full[s], (i / p.slots) & 1);
      mbar_arrive(&empty[s]);
      if (p.multicast) mbar_arrive_peer(smem_u32(&empty[s]));
    }
  }
  cluster_sync();
}

#define CK(x)                                                                         \
  do {                                                                                \
    cudaError_t e_ = (x);                                                             \
    if (e_ != cudaSuccess) {                                                          \
      fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_));                        \
      return 1;                                                                       \
    }                                                                                 \
  } while (0)

int main(int argc, char** argv) {
  if (argc != 8 && argc != 9) {
    fprintf(stderr, "usage: %s <halo|igemm|planes> <cin> <cout> <BN> <ctas per SM> <multicast> <tiles per CTA> [slots]\n",
            argv[0]);
    return 2;
  }
  FillParams p{};
  p.planes = strcmp(argv[1], "planes") == 0;
  p.halo = p.planes || strcmp(argv[1], "halo") == 0;
  p.cin = atoi(argv[2]);
  const int cout = atoi(argv[3]), occ = atoi(argv[5]);
  p.BN = atoi(argv[4]);
  p.multicast = atoi(argv[6]);
  p.iters = atoi(argv[7]);
  const int taps = p.halo ? 9 : 1;
  p.n_tiles = (cout + p.BN - 1) / p.BN;
  p.k_tiles = taps * ((p.cin + 63) / 64);
  p.tile_bytes = p.BN * 128;   // 64 channels x BN rows of bf16
  const size_t smem = occ == 2 ? 110 * 1024 : 200 * 1024;
  p.slots = (int)((smem - 1024 - 128) / p.tile_bytes);
  if (p.slots > 8) p.slots = 8;
  if (argc == 9) p.slots = atoi(argv[8]);
  if ((p.planes && (p.multicast || p.cin % 8)) || p.slots < 1 || (size_t)p.slots * p.tile_bytes + 1024 + 128 > smem) {
    fprintf(stderr, "planes: no multicast and cin a multiple of 8; the ring must fit in shared memory\n");
    return 2;
  }
  // plane image: Cout rows padded so that the last Cout tile's runs stay inside the allocation
  p.cout_rows = p.n_tiles * p.BN;
  void* w = nullptr;
  const size_t wbytes =
      p.planes ? (size_t)p.cout_rows * taps * ((p.cin + 63) / 64 * 64) * 2 : (size_t)cout * taps * p.cin * 2;
  CK(cudaMalloc(&w, wbytes));
  CK(cudaMemset(w, 0x3c, wbytes));
  CUtensorMap tm;
  const uint64_t dims[3] = {(uint64_t)p.cin, (uint64_t)taps, (uint64_t)cout};
  const uint64_t strides[2] = {(uint64_t)p.cin * 2, (uint64_t)taps * p.cin * 2};
  const uint32_t box_halo[3] = {8, 1, (uint32_t)p.BN};
  const uint32_t box_igemm[3] = {64, 1, (uint32_t)(p.BN / (p.multicast ? 2 : 1))};
  if (int rc = encode_bf16(&tm, w, 3, dims, strides, p.halo ? box_halo : box_igemm, nullptr,
                           p.halo ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B)) {
    fprintf(stderr, "tensor map: %d\n", rc);
    return 1;
  }
  CK(cudaFuncSetAttribute(l2_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaDeviceProp pr;
  CK(cudaGetDeviceProperties(&pr, 0));
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  cfg.blockDim = dim3(64);
  cfg.dynamicSmemBytes = smem;
  int grid = occ * pr.multiProcessorCount;
  if (p.multicast) {
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cfg.gridDim = dim3(grid);
    int clusters = 0;
    CK(cudaOccupancyMaxActiveClusters(&clusters, l2_fill_kernel, &cfg));
    if (2 * clusters < grid) grid = 2 * clusters;
  }
  cfg.gridDim = dim3(grid);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  const uint8_t* image = p.planes ? static_cast<const uint8_t*>(w) : nullptr;
  CK(cudaLaunchKernelEx(&cfg, l2_fill_kernel, tm, p, image));   // warm-up: brings the weights into L2
  CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int r = 0; r < 5; ++r) {
    CK(cudaEventRecord(e0));
    CK(cudaLaunchKernelEx(&cfg, l2_fill_kernel, tm, p, image));
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (ms < best) best = ms;
  }
  int clk_khz = 0;
  CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0));
  const double smem_bytes = (double)grid * p.iters * p.tile_bytes;   // bytes landed in shared memory
  const double l2_bytes = smem_bytes / (p.multicast ? 2 : 1);         // bytes read from L2
  const double s = best * 1e-3;
  const int sms = pr.multiProcessorCount;
  printf("{\"kind\": \"%s\", \"cin\": %d, \"cout\": %d, \"BN\": %d, \"ctas_per_sm\": %d, \"multicast\": %d, "
         "\"grid\": %d, \"slots\": %d, \"tile_bytes\": %d, \"weight_bytes\": %zu, \"ms\": %.4f, "
         "\"smem_fill_TBps\": %.3f, \"l2_read_TBps\": %.3f, \"smem_fill_B_per_clk_per_sm\": %.2f, "
         "\"l2_read_B_per_clk_per_sm\": %.2f, \"max_sm_clock_mhz\": %d}\n",
         p.planes ? "planes" : p.halo ? "halo" : "igemm", p.cin, cout, p.BN, occ, p.multicast, grid, p.slots, p.tile_bytes, wbytes, best,
         smem_bytes / s / 1e12, l2_bytes / s / 1e12, smem_bytes / s / (clk_khz * 1e3) / sms,
         l2_bytes / s / (clk_khz * 1e3) / sms, clk_khz / 1000);
  CK(cudaFree(w));
  return 0;
}
