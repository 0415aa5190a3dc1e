// Device-side training input pipeline (SURVEY.md §8 row f4): the reference's per-sample transform chain on the decoded
// uint8 frame, bit-exact with Pillow's arithmetic (host side, table construction and citations: b200seg/augment.py).
//
//   aug_resize_crop_kernel      RandomSizeAndCrop + RandomCrop padding + RandomHorizontallyFlip
//                               (transforms/joint_transforms.py:433-472, :143-182, :276-281): Pillow's two-pass BICUBIC
//                               resampler (22-bit fixed-point taps, the horizontal pass rounded to uint8 before the
//                               vertical one) evaluated only inside the crop window; NEAREST + label-id lookup for the
//                               mask (datasets/base_loader.py:177-181); padding = black / ignore label.
//   aug_luma_sum_kernel         mean grey level for ImageEnhance.Contrast (sum of the L conversion after the jitter ops that
//                               precede the contrast op)
//   aug_color_normalize_kernel  ColorJitter ops in their drawn order (transforms/transforms.py:297-362: Image.blend in
//                               fp32 with Pillow's truncation / clipping, HSV hue shift with Pillow's float / double
//                               promotions) -> ToTensor (/255) -> Normalize ((v - mean) / std), fp32 CHW
//
// All three are HBM / L2-bound byte kernels (6 MB of uint8 in, 25 MB of fp32 out per 1024x2048 crop): one thread per
// output pixel, coalesced stores; the gather of the resampler reads each source pixel from L1/L2 (neighbouring outputs share
// their taps).
#include <cstdint>
#include "ptx.cuh"
#include "launch.h"
#include "augment_ops.cuh"
#include "../../include/b200seg.h"

namespace b200seg {

constexpr int kAugBits = 22;     // Pillow: PRECISION_BITS = 32 - 8 - 2

__device__ __forceinline__ int aug_clip8(int v) {
  v >>= kAugBits;                // arithmetic shift (floor), like Pillow's lookup index
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

struct AugGeom {
  int src_h, src_w;              // decoded frame
  int out_h, out_w;              // crop
  int win_y0, win_x0;            // first output row / column (before the flip) that shows a resized pixel
  int n_y, n_x;                  // rows / columns of the window (table extents)
  int ksize_v, ksize_h;
  int flip, ignore_label;
};

__global__ void __launch_bounds__(256)
aug_resize_crop_kernel(const AugGeom g, const uint8_t* __restrict__ src, const uint8_t* __restrict__ src_mask,
                       const int32_t* __restrict__ kk_h, const int32_t* __restrict__ bounds_h,
                       const int32_t* __restrict__ kk_v, const int32_t* __restrict__ bounds_v,
                       const int32_t* __restrict__ near_x, const int32_t* __restrict__ near_y,
                       const uint8_t* __restrict__ id_lut, uint8_t* __restrict__ out_rgb,
                       long long* __restrict__ out_label) {
  pdl_sync();
  const long long total = (long long)g.out_h * g.out_w;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int oy = (int)(idx / g.out_w), oxf = (int)(idx - (long long)oy * g.out_w);
    const int ox = g.flip ? g.out_w - 1 - oxf : oxf;      // column of the un-flipped crop this output column shows
    const int wy = oy - g.win_y0, wx = ox - g.win_x0;
    int r = 0, gr = 0, b = 0;
    long long lab = g.ignore_label;
    if (wy >= 0 && wy < g.n_y && wx >= 0 && wx < g.n_x) {
      const int y0 = bounds_v[2 * wy], ny = bounds_v[2 * wy + 1];
      const int x0 = bounds_h[2 * wx], nx = bounds_h[2 * wx + 1];
      const int32_t* kh = kk_h + (size_t)wx * g.ksize_h;
      const int32_t* kv = kk_v + (size_t)wy * g.ksize_v;
      int v0 = 1 << (kAugBits - 1), v1 = v0, v2 = v0;
      for (int ky = 0; ky < ny; ++ky) {
        const uint8_t* row = src + ((size_t)(y0 + ky) * g.src_w + x0) * 3;
        int h0 = 1 << (kAugBits - 1), h1 = h0, h2 = h0;
        for (int kx = 0; kx < nx; ++kx) {
          const int c = __ldg(kh + kx);
          h0 += (int)row[3 * kx] * c;
          h1 += (int)row[3 * kx + 1] * c;
          h2 += (int)row[3 * kx + 2] * c;
        }
        const int cv = __ldg(kv + ky);      // the horizontal pass is stored as uint8 before the vertical one
        v0 += aug_clip8(h0) * cv;
        v1 += aug_clip8(h1) * cv;
        v2 += aug_clip8(h2) * cv;
      }
      r = aug_clip8(v0); gr = aug_clip8(v1); b = aug_clip8(v2);
      const uint8_t m = src_mask[(size_t)near_y[wy] * g.src_w + near_x[wx]];
      lab = id_lut ? id_lut[m] : m;
    }
    uint8_t* o = out_rgb + (size_t)idx * 3;
    o[0] = (uint8_t)r; o[1] = (uint8_t)gr; o[2] = (uint8_t)b;
    out_label[idx] = lab;
  }
}

__global__ void __launch_bounds__(256)
aug_luma_sum_kernel(const AugColor c, int n_before, const uint8_t* __restrict__ rgb, long long npix,
                    unsigned long long* __restrict__ sum) {
  pdl_sync();
  unsigned long long acc = 0;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < npix;
       idx += (long long)gridDim.x * blockDim.x) {
    int r = rgb[idx * 3], g = rgb[idx * 3 + 1], b = rgb[idx * 3 + 2];
    aug_apply_ops(c, 0, n_before, 0, r, g, b);
    acc += (unsigned long long)aug_luma(r, g, b);
  }
  for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  __shared__ unsigned long long sh[8];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int i = 0; i < 8; ++i) t += sh[i];
    atomicAdd(sum, t);          // integer sum: exact and order independent
  }
}

__global__ void __launch_bounds__(256)
aug_color_normalize_kernel(const AugColor c, const uint8_t* __restrict__ rgb, int h, int w,
                           const unsigned long long* __restrict__ luma_sum, float* __restrict__ out) {
  pdl_sync();
  const long long npix = (long long)h * w;
  int mean = 0;
  if (luma_sum) mean = (int)((double)(*luma_sum) / (double)npix + 0.5);     // int(ImageStat.Stat(L).mean[0] + 0.5)
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < npix;
       idx += (long long)gridDim.x * blockDim.x) {
    int r = rgb[idx * 3], g = rgb[idx * 3 + 1], b = rgb[idx * 3 + 2];
    aug_apply_ops(c, 0, c.n_ops, mean, r, g, b);
    // ToTensor: uint8 -> float / 255; Normalize: (v - mean) / std  (IEEE fp32 division, like ATen on the CPU)
    out[idx] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)r, 255.f), c.mean[0]), c.std[0]);
    out[npix + idx] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)g, 255.f), c.mean[1]), c.std[1]);
    out[2 * npix + idx] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)b, 255.f), c.mean[2]), c.std[2]);
  }
}

}  // namespace b200seg

using namespace b200seg;

extern "C" int b200seg_aug_resize_crop(const b200seg_aug_geom* d, const uint8_t* src_rgb, const uint8_t* src_mask,
                                       const int32_t* kk_h, const int32_t* bounds_h, const int32_t* kk_v,
                                       const int32_t* bounds_v, const int32_t* near_x, const int32_t* near_y,
                                       const uint8_t* id_lut, uint8_t* out_rgb, int64_t* out_label, void* stream) {
  if (!d || !src_rgb || !src_mask || !out_rgb || !out_label) return B200SEG_E_BADARG;
  if (d->src_h <= 0 || d->src_w <= 0 || d->out_h <= 0 || d->out_w <= 0 || d->n_y < 0 || d->n_x < 0)
    return B200SEG_E_BADARG;
  if (d->n_y > 0 && d->n_x > 0 && (!kk_h || !bounds_h || !kk_v || !bounds_v || !near_x || !near_y || d->ksize_h <= 0 ||
                                   d->ksize_v <= 0))
    return B200SEG_E_BADARG;
  AugGeom g;
  g.src_h = d->src_h; g.src_w = d->src_w; g.out_h = d->out_h; g.out_w = d->out_w;
  g.win_y0 = d->win_y0; g.win_x0 = d->win_x0; g.n_y = d->n_y; g.n_x = d->n_x;
  g.ksize_v = d->ksize_v; g.ksize_h = d->ksize_h; g.flip = d->flip; g.ignore_label = d->ignore_label;
  const long long total = (long long)d->out_h * d->out_w;
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)B200SEG_MAX_CTAS * 16) blocks = (long long)B200SEG_MAX_CTAS * 16;
  cudaError_t e = launch_k(aug_resize_crop_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, g, src_rgb,
                           src_mask, kk_h, bounds_h, kk_v, bounds_v, near_x, near_y, id_lut, out_rgb,
                           (long long*)out_label);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_aug_color_normalize(const b200seg_aug_color* c, const uint8_t* rgb, int32_t h, int32_t w,
                                           uint64_t* luma_sum_ws, float* out_chw, void* stream) {
  if (!c || !rgb || !out_chw || h <= 0 || w <= 0 || c->n_ops < 0 || c->n_ops > 4) return B200SEG_E_BADARG;
  AugColor k;
  k.n_ops = c->n_ops;
  int contrast_at = -1;
  for (int i = 0; i < 4; ++i) {
    k.kind[i] = i < c->n_ops ? c->kind[i] : 0;
    k.factor[i] = i < c->n_ops ? c->factor[i] : 1.f;
    k.hue_shift[i] = i < c->n_ops ? (c->hue_shift[i] & 255) : 0;
    if (i < c->n_ops) {
      if (c->kind[i] < 0 || c->kind[i] > 3) return B200SEG_E_BADARG;
      if (c->kind[i] == 1) { if (contrast_at >= 0) return B200SEG_E_BADARG; contrast_at = i; }
    }
  }
  for (int i = 0; i < 3; ++i) { k.mean[i] = c->mean[i]; k.std[i] = c->std[i]; }
  const long long npix = (long long)h * w;
  long long blocks = (npix + 255) / 256;
  if (blocks > (long long)B200SEG_MAX_CTAS * 16) blocks = (long long)B200SEG_MAX_CTAS * 16;
  if (contrast_at >= 0) {
    if (!luma_sum_ws) return B200SEG_E_BADARG;
    cudaError_t e0 = cudaMemsetAsync(luma_sum_ws, 0, sizeof(uint64_t), (cudaStream_t)stream);
    if (e0 != cudaSuccess) return (int)e0;
    e0 = launch_k(aug_luma_sum_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, k, contrast_at, rgb,
                  npix, (unsigned long long*)luma_sum_ws);
    if (e0 != cudaSuccess) return (int)e0;
  }
  cudaError_t e = launch_k(aug_color_normalize_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, k, rgb,
                           (int)h, (int)w, contrast_at >= 0 ? (const unsigned long long*)luma_sum_ws : nullptr, out_chw);
  return e == cudaSuccess ? 0 : (int)e;
}
