// Kernel launch helper: every launch carries the programmatic-stream-serialization attribute (PDL) so the next kernel's
// prologue overlaps this kernel's body (see ptx.cuh pdl_*). Works under stream capture (the edge becomes a programmatic
// graph dependency).
#pragma once
#include <cuda_runtime.h>
#include <cstdlib>

namespace b200seg {

// B200SEG_DRY (measurement only): every launch of the library becomes an empty kernel that keeps
// the stream / programmatic dependency structure: 1 = one warp, 2 = the real grid and block dimensions (no shared
// memory). A captured step then replays at the launch-and-dependency floor of its program; results are garbage.
inline int dry_mode() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("B200SEG_DRY");
    v = e ? atoi(e) : 0;
  }
  return v;
}
static __global__ void dry_noop_kernel() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                            Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (const int dry = dry_mode()) {
    if (dry == 1) { cfg.gridDim = dim3(1); cfg.blockDim = dim3(32); }
    cfg.dynamicSmemBytes = 0;
    return cudaLaunchKernelEx(&cfg, dry_noop_kernel);
  }
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace b200seg
