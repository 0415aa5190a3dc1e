// RandAugment on the device input pipeline (SURVEY.md §8 row f4): the 14 ops of datasets/randaugment.py augment_list()
// applied to the uint8 crop and its int64 label map between aug_resize_crop_kernel and aug_color_normalize_kernel,
// bit-exact with Pillow 12 (host side - the draws, the affine matrices, the static LUTs: b200seg/augment.py).
//
//   aug_affine_kernel     ShearX / ShearY / TranslateX / TranslateY (Image.transform AFFINE: BILINEAR image, NEAREST labels)
//                         and Rotate (Image.rotate: NEAREST both). NEAREST follows Pillow's ImagingTransformAffine: per-axis
//                         source tables when the matrix has no shear terms (ImagingScaleAffine's double accumulation,
//                         tabulated on the host), else 16.16 fixed point (affine_fixed). BILINEAR is ImagingGenericTransform
//                         with bilinear_filter32RGB, in double without contraction. Outside the source: black / label 255.
//   aug_hist_kernel       per-channel 256-bin histogram (AutoContrast, Equalize)
//   aug_hist_lut_kernel   ImageOps.autocontrast / ImageOps.equalize LUT from that histogram (one block per channel)
//   aug_point_kernel      Image.point with a [3][256] LUT: Invert, Solarize, Posterize and the two histogram LUTs
//   aug_enhance_kernel    ImageEnhance Brightness / Color (the jitter's blends, augment_ops.cuh) and Sharpness (SMOOTH 3x3
//                         fused with the blend; border pixels keep their value)
//
// All are byte kernels bound by HBM / L2: one thread per output pixel, coalesced stores, ping-pong between two buffers.
#include <cstdint>
#include "ptx.cuh"
#include "launch.h"
#include "augment_ops.cuh"
#include "../../include/b200seg.h"

namespace b200seg {

struct AugAffine {
  int h, w;
  int bilinear, scale;
  int fixed[6];
  int label_fill;
  double a[6];
};

// Pillow's BILINEAR(v, a, b, d): a + (b - a) * d in double
__device__ __forceinline__ double aug_lerp(double a, double b, double d) { return __dadd_rn(a, __dmul_rn(__dsub_rn(b, a), d)); }

__global__ void __launch_bounds__(256)
aug_affine_kernel(const AugAffine d, const uint8_t* __restrict__ src, const long long* __restrict__ src_label,
                  const int32_t* __restrict__ tab_x, const int32_t* __restrict__ tab_y, uint8_t* __restrict__ out,
                  long long* __restrict__ out_label) {
  pdl_sync();
  const long long total = (long long)d.h * d.w;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(idx / d.w), x = (int)(idx - (long long)y * d.w);
    int xi, yi;                        // NEAREST source pixel
    if (d.scale) {
      xi = tab_x[x];
      yi = tab_y[y];
    } else {                           // affine_fixed: xx = a2 + y * a1 + x * a0 in 32-bit integers
      const unsigned xx = (unsigned)d.fixed[2] + (unsigned)y * (unsigned)d.fixed[1] + (unsigned)x * (unsigned)d.fixed[0];
      const unsigned yy = (unsigned)d.fixed[5] + (unsigned)y * (unsigned)d.fixed[4] + (unsigned)x * (unsigned)d.fixed[3];
      xi = (int)xx >> 16;
      yi = (int)yy >> 16;
    }
    const bool inside = xi >= 0 && xi < d.w && yi >= 0 && yi < d.h;
    out_label[idx] = inside ? src_label[(size_t)yi * d.w + xi] : (long long)d.label_fill;
    int v[3] = {0, 0, 0};
    if (d.bilinear) {
      // affine_transform(): the pixel centre mapped in double, then bilinear_filter32RGB
      const double xin = (double)x + 0.5, yin = (double)y + 0.5;
      double X = __dadd_rn(__dadd_rn(__dmul_rn(d.a[0], xin), __dmul_rn(d.a[1], yin)), d.a[2]);
      double Y = __dadd_rn(__dadd_rn(__dmul_rn(d.a[3], xin), __dmul_rn(d.a[4], yin)), d.a[5]);
      if (!(X < 0.0 || X >= (double)d.w || Y < 0.0 || Y >= (double)d.h)) {
        X = __dsub_rn(X, 0.5);
        Y = __dsub_rn(Y, 0.5);
        const int x0 = (int)floor(X), y0 = (int)floor(Y);
        const double dx = __dsub_rn(X, (double)x0), dy = __dsub_rn(Y, (double)y0);
        const int xa = min(max(x0, 0), d.w - 1), xb = min(max(x0 + 1, 0), d.w - 1);
        const uint8_t* r0 = src + (size_t)min(max(y0, 0), d.h - 1) * d.w * 3;
        const bool has_r1 = y0 + 1 >= 0 && y0 + 1 < d.h;
        const uint8_t* r1 = src + (size_t)(has_r1 ? y0 + 1 : 0) * d.w * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const double v1 = aug_lerp((double)r0[xa * 3 + c], (double)r0[xb * 3 + c], dx);
          const double v2 = has_r1 ? aug_lerp((double)r1[xa * 3 + c], (double)r1[xb * 3 + c], dx) : v1;
          v[c] = (int)aug_lerp(v1, v2, dy);
        }
      }
    } else if (inside) {
      const uint8_t* p = src + ((size_t)yi * d.w + xi) * 3;
      v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
    }
    uint8_t* o = out + (size_t)idx * 3;
    o[0] = (uint8_t)v[0]; o[1] = (uint8_t)v[1]; o[2] = (uint8_t)v[2];
  }
}

__global__ void __launch_bounds__(256)
aug_hist_kernel(const uint8_t* __restrict__ rgb, long long npix, unsigned* __restrict__ hist) {
  __shared__ unsigned sh[768];
  for (int i = threadIdx.x; i < 768; i += blockDim.x) sh[i] = 0;
  pdl_sync();
  __syncthreads();
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < npix;
       idx += (long long)gridDim.x * blockDim.x) {
    atomicAdd(&sh[rgb[idx * 3]], 1u);
    atomicAdd(&sh[256 + rgb[idx * 3 + 1]], 1u);
    atomicAdd(&sh[512 + rgb[idx * 3 + 2]], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 768; i += blockDim.x)
    if (sh[i]) atomicAdd(hist + i, sh[i]);
}

// kind 0: ImageOps.autocontrast (cutoff 0): lut[i] = clip(int(i * scale + offset)), scale = 255.0 / (hi - lo),
//         offset = -lo * scale over the first / last non-empty bins; identity when hi <= lo.
// kind 1: ImageOps.equalize: step = (sum - h[last non-empty]) // 255, lut[i] = (step // 2 + sum(h[:i])) // step;
//         identity when at most one bin is non-empty or step == 0. Image.point clips the LUT to 255.
__global__ void __launch_bounds__(256)
aug_hist_lut_kernel(int kind, const unsigned* __restrict__ hist, int32_t* __restrict__ lut) {
  __shared__ long long below[256];
  __shared__ unsigned h[256];
  __shared__ int s_lo, s_hi, s_nonzero;
  pdl_sync();
  const int c = blockIdx.x, i = threadIdx.x;
  h[i] = hist[c * 256 + i];
  __syncthreads();
  if (i == 0) {
    int lo = -1, hi = -1, nonzero = 0;
    long long run = 0;
    for (int j = 0; j < 256; ++j) {
      below[j] = run;
      run += h[j];
      if (h[j]) { if (lo < 0) lo = j; hi = j; ++nonzero; }
    }
    s_lo = lo; s_hi = hi; s_nonzero = nonzero;
  }
  __syncthreads();
  const int lo = s_lo, hi = s_hi;
  int v = i;
  if (kind == 0) {
    if (hi > lo) {
      const double scale = __ddiv_rn(255.0, (double)(hi - lo));
      const double offset = __dmul_rn(-(double)lo, scale);
      v = (int)__dadd_rn(__dmul_rn((double)i, scale), offset);
      v = v < 0 ? 0 : (v > 255 ? 255 : v);
    }
  } else if (s_nonzero > 1) {
    const long long step = below[hi] / 255;      // below[hi]: every sample but those of the last non-empty bin
    if (step) {
      const long long q = (step / 2 + below[i]) / step;
      v = q > 255 ? 255 : (int)q;
    }
  }
  lut[c * 256 + i] = v;
}

__global__ void __launch_bounds__(256)
aug_point_kernel(const uint8_t* __restrict__ src, long long npix, const int32_t* __restrict__ lut,
                 uint8_t* __restrict__ dst) {
  __shared__ uint8_t sl[768];
  pdl_sync();
  for (int i = threadIdx.x; i < 768; i += blockDim.x) sl[i] = (uint8_t)lut[i];
  __syncthreads();
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < npix;
       idx += (long long)gridDim.x * blockDim.x) {
    const uint8_t* s = src + idx * 3;
    uint8_t* o = dst + idx * 3;
    o[0] = sl[s[0]]; o[1] = sl[256 + s[1]]; o[2] = sl[512 + s[2]];
  }
}

// kind: B200SEG_AUG_ENHANCE_*. Brightness / Color are the jitter's brightness / saturation blends (one-op AugColor).
__global__ void __launch_bounds__(256)
aug_enhance_kernel(int kind, float factor, const uint8_t* __restrict__ src, int h, int w, uint8_t* __restrict__ dst) {
  pdl_sync();
  AugColor c{};
  c.n_ops = 1;
  c.kind[0] = kind == B200SEG_AUG_ENHANCE_COLOR ? 2 : 0;
  c.factor[0] = factor;
  const long long npix = (long long)h * w;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < npix;
       idx += (long long)gridDim.x * blockDim.x) {
    const uint8_t* s = src + idx * 3;
    int r = s[0], g = s[1], b = s[2];
    if (kind != B200SEG_AUG_ENHANCE_SHARPNESS) {
      aug_apply_ops(c, 0, 1, 0, r, g, b);
    } else {
      const int y = (int)(idx / w), x = (int)(idx - (long long)y * w);
      if (y > 0 && y < h - 1 && x > 0 && x < w - 1) {
        // ImageFilter.SMOOTH: (1 1 1 / 1 5 1 / 1 1 1) / 13, rounded. Pillow sums fp32 taps; the exact sum is never within
        // 1/26 of a rounding boundary, so the integer form round(tot / 13) gives the same byte.
        int v[3] = {r, g, b};
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
          int tot = 4 * v[ch];
#pragma unroll
          for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) tot += s[((long long)dy * w + dx) * 3 + ch];
          v[ch] = aug_blend((2 * tot + 13) / 26, v[ch], factor);
        }
        r = v[0]; g = v[1]; b = v[2];
      }
    }
    uint8_t* o = dst + idx * 3;
    o[0] = (uint8_t)r; o[1] = (uint8_t)g; o[2] = (uint8_t)b;
  }
}

inline unsigned aug_blocks(long long n, long long cap) {
  long long blocks = (n + 255) / 256;
  return (unsigned)(blocks > cap ? cap : blocks);
}

}  // namespace b200seg

using namespace b200seg;

extern "C" int b200seg_aug_affine(const b200seg_aug_affine_desc* d, const uint8_t* src_rgb, const int64_t* src_label,
                                  const int32_t* tab_x, const int32_t* tab_y, uint8_t* out_rgb, int64_t* out_label,
                                  void* stream) {
  if (!d || !src_rgb || !src_label || !out_rgb || !out_label || d->h <= 0 || d->w <= 0) return B200SEG_E_BADARG;
  if (d->scale && (!tab_x || !tab_y)) return B200SEG_E_BADARG;
  if (src_rgb == out_rgb || src_label == out_label) return B200SEG_E_BADARG;     // a gather: never in place
  AugAffine k;
  k.h = d->h; k.w = d->w; k.bilinear = d->bilinear; k.scale = d->scale; k.label_fill = d->label_fill;
  for (int i = 0; i < 6; ++i) { k.fixed[i] = d->fixed[i]; k.a[i] = d->a[i]; }
  const long long total = (long long)d->h * d->w;
  cudaError_t e = launch_k(aug_affine_kernel, dim3(aug_blocks(total, (long long)B200SEG_MAX_CTAS * 16)), dim3(256), 0,
                           (cudaStream_t)stream, k, src_rgb, (const long long*)src_label, tab_x, tab_y, out_rgb,
                           (long long*)out_label);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_aug_hist_lut(int32_t kind, const uint8_t* rgb, int64_t npix, uint32_t* hist_ws, int32_t* lut,
                                    void* stream) {
  if (!rgb || !hist_ws || !lut || npix <= 0 || (kind != 0 && kind != 1)) return B200SEG_E_BADARG;
  cudaError_t e = cudaMemsetAsync(hist_ws, 0, 768 * sizeof(uint32_t), (cudaStream_t)stream);
  if (e != cudaSuccess) return (int)e;
  // a few CTAs per SM: each merges its 768 shared-memory bins into the global histogram once
  e = launch_k(aug_hist_kernel, dim3(aug_blocks(npix, (long long)B200SEG_MAX_CTAS * 4)), dim3(256), 0,
               (cudaStream_t)stream, rgb, (long long)npix, (unsigned*)hist_ws);
  if (e != cudaSuccess) return (int)e;
  e = launch_k(aug_hist_lut_kernel, dim3(3), dim3(256), 0, (cudaStream_t)stream, (int)kind, (const unsigned*)hist_ws, lut);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_aug_point(const uint8_t* src_rgb, int64_t npix, const int32_t* lut, uint8_t* out_rgb,
                                 void* stream) {
  if (!src_rgb || !lut || !out_rgb || npix <= 0) return B200SEG_E_BADARG;
  cudaError_t e = launch_k(aug_point_kernel, dim3(aug_blocks(npix, (long long)B200SEG_MAX_CTAS * 16)), dim3(256), 0,
                           (cudaStream_t)stream, src_rgb, (long long)npix, lut, out_rgb);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_aug_enhance(int32_t kind, float factor, const uint8_t* src_rgb, int32_t h, int32_t w,
                                   uint8_t* out_rgb, void* stream) {
  if (!src_rgb || !out_rgb || h <= 0 || w <= 0) return B200SEG_E_BADARG;
  if (kind != B200SEG_AUG_ENHANCE_BRIGHTNESS && kind != B200SEG_AUG_ENHANCE_COLOR && kind != B200SEG_AUG_ENHANCE_SHARPNESS)
    return B200SEG_E_BADARG;
  if (kind == B200SEG_AUG_ENHANCE_SHARPNESS && src_rgb == out_rgb) return B200SEG_E_BADARG;   // reads neighbours
  const long long npix = (long long)h * w;
  cudaError_t e = launch_k(aug_enhance_kernel, dim3(aug_blocks(npix, (long long)B200SEG_MAX_CTAS * 16)), dim3(256), 0,
                           (cudaStream_t)stream, (int)kind, factor, src_rgb, (int)h, (int)w, out_rgb);
  return e == cudaSuccess ? 0 : (int)e;
}
