// Pooling / broadcast glue of the DeepLabV3+ / WideResNet-38 path (SURVEY.md §8(f) row f2), NHWC bf16, 16-byte accesses:
//   maxpool3x3s2_fwd / _bwd   nn.MaxPool2d(3, stride=2, padding=1) between mod1/mod2 and mod2/mod3
//                             (network/wider_resnet.py:347-349,423-428); backward in gather form with the argmax recomputed
//                             (first maximum in row-major window order, like ATen)
//   channel_stats             per-channel sum / sum of squares of an activation (batch statistics of a pre-activation
//                             BatchNorm whose input does not come out of a convolution epilogue)
//   spatial_sum               per-image, per-channel sum over the pixels (x scale): ASPP image pooling
//                             (nn.AdaptiveAvgPool2d(1), network/utils.py:194-210) and the adjoint of the broadcast below
//   broadcast_pixels          out[n,h,w,c] (=|+=) scale * v[n,c]: bilinear Upsample of a 1x1 map is a broadcast; with
//                             scale = 1/P and accumulate it is the adjoint of the image pooling
#include "ptx.cuh"
#include "launch.h"
#include "../../include/b200seg.h"
#include "vec.cuh"

namespace b200seg {

static inline int pool_grid(long long total_threads) {
  long long b = (total_threads + 255) / 256;
  const long long cap = (long long)B200SEG_MAX_CTAS * 8;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

__global__ void __launch_bounds__(256)
maxpool3x3s2_fwd_kernel(const __nv_bfloat16* __restrict__ x, int x_ld, int N, int H, int W, int C,
                        __nv_bfloat16* __restrict__ y, int y_ld, int Ho, int Wo) {
  pdl_sync();
  const int groups = C >> 3;
  const long long total = (long long)N * Ho * Wo * groups;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long pix = idx / groups;
    const int c0 = (int)(idx - pix * groups) << 3;
    const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho), n = (int)(pix / ((long long)Wo * Ho));
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
    for (int kh = 0; kh < 3; ++kh) {
      const int h = 2 * ho - 1 + kh;
      if (h < 0 || h >= H) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int w = 2 * wo - 1 + kw;
        if (w < 0 || w >= W) continue;
        float v[8];
        load8(x + (((long long)n * H + h) * W + w) * x_ld + c0, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = v[j] > m[j] ? v[j] : m[j];
      }
    }
    store8(y + pix * y_ld + c0, m);
  }
}

// dx[n,h,w,c] (=|+=) sum over the <= 4 windows containing (h, w) of dy[window] * [argmax(window) == (h, w)]
__global__ void __launch_bounds__(256)
maxpool3x3s2_bwd_kernel(const __nv_bfloat16* __restrict__ x, int x_ld, const __nv_bfloat16* __restrict__ dy, int dy_ld,
                        int N, int H, int W, int C, int Ho, int Wo, __nv_bfloat16* __restrict__ dx, int dx_ld,
                        int accumulate) {
  pdl_sync();
  const int groups = C >> 3;
  const long long total = (long long)N * H * W * groups;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long pix = idx / groups;
    const int c0 = (int)(idx - pix * groups) << 3;
    const int w = (int)(pix % W), h = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // windows (ho, wo) with 2*ho - 1 <= h <= 2*ho + 1
    for (int ho = (h - 1 + 1) / 2; ho <= (h + 1) / 2; ++ho) {
      if (ho < 0 || ho >= Ho || h < 2 * ho - 1 || h > 2 * ho + 1) continue;
      for (int wo = (w - 1 + 1) / 2; wo <= (w + 1) / 2; ++wo) {
        if (wo < 0 || wo >= Wo || w < 2 * wo - 1 || w > 2 * wo + 1) continue;
        // recompute the window's argmax per channel: the first maximum in (kh, kw) order wins
        float m[8];
        int am[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { m[j] = -INFINITY; am[j] = -1; }
        for (int kh = 0; kh < 3; ++kh) {
          const int hh = 2 * ho - 1 + kh;
          if (hh < 0 || hh >= H) continue;
          for (int kw = 0; kw < 3; ++kw) {
            const int ww = 2 * wo - 1 + kw;
            if (ww < 0 || ww >= W) continue;
            float v[8];
            load8(x + (((long long)n * H + hh) * W + ww) * x_ld + c0, v);
#pragma unroll
            for (int j = 0; j < 8; ++j)
              if (v[j] > m[j]) { m[j] = v[j]; am[j] = kh * 3 + kw; }
          }
        }
        const int mine = (h - (2 * ho - 1)) * 3 + (w - (2 * wo - 1));
        float g[8];
        load8(dy + (((long long)n * Ho + ho) * Wo + wo) * dy_ld + c0, g);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += am[j] == mine ? g[j] : 0.f;
      }
    }
    if (accumulate) {
      float old[8];
      load8(dx + pix * dx_ld + c0, old);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += old[j];
    }
    store8(dx + pix * dx_ld + c0, acc);
  }
}

// partials[block][2][C]: per-channel sum / sum of squares of the block's pixels (rows x 8-channel groups per block,
// fixed-order fold over the rows -> deterministic); same layout the convolution epilogues emit.
__global__ void __launch_bounds__(256)
channel_stats_kernel(const __nv_bfloat16* __restrict__ x, int x_ld, long long npix, int C, int rows,
                     float* __restrict__ partials) {
  pdl_sync();
  extern __shared__ float s_cs[];   // [rows][groups][16]
  const int groups = C >> 3;
  const int cg = threadIdx.x % groups, r = threadIdx.x / groups;
  const int c0 = cg << 3;
  float s1[8], s2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { s1[j] = 0.f; s2[j] = 0.f; }
  if (r < rows) {
    for (long long pix = (long long)blockIdx.x * rows + r; pix < npix; pix += (long long)gridDim.x * rows) {
      float v[8];
      load8(x + pix * x_ld + c0, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s1[j] += v[j]; s2[j] += v[j] * v[j]; }
    }
    float* dst = s_cs + ((size_t)r * groups + cg) * 16;
#pragma unroll
    for (int j = 0; j < 8; ++j) { dst[j] = s1[j]; dst[8 + j] = s2[j]; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < groups * 16; i += blockDim.x) {
    const int g_ = i / 16, k = i % 16;
    float acc = 0.f;
    for (int rr = 0; rr < rows; ++rr) acc += s_cs[((size_t)rr * groups + g_) * 16 + k];
    partials[(size_t)blockIdx.x * 2 * C + (k >> 3) * C + g_ * 8 + (k & 7)] = acc;
  }
}

// part[n][split][C] fp32 = sum over the split's pixels of x[n, pix, c]
__global__ void __launch_bounds__(256)
spatial_sum_partial_kernel(const __nv_bfloat16* __restrict__ x, int x_ld, int P, int C, int splits,
                           float* __restrict__ part) {
  pdl_sync();
  const int groups = C >> 3;
  const int n = blockIdx.z, split = blockIdx.y;
  const int g0 = blockIdx.x * 8;                      // 8 channel groups (64 channels) per block
  const int cg = g0 + (threadIdx.x & 7), lane = threadIdx.x >> 3;   // 32 pixel lanes
  __shared__ float sh[32][8][8];
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (cg < groups) {
    const int p0 = (int)((long long)P * split / splits), p1 = (int)((long long)P * (split + 1) / splits);
    for (int p = p0 + lane; p < p1; p += 32) {
      float v[8];
      load8(x + ((long long)n * P + p) * x_ld + cg * 8, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) sh[lane][threadIdx.x & 7][j] = acc[j];
  __syncthreads();
  if (threadIdx.x < 64) {
    const int g_ = threadIdx.x >> 3, j = threadIdx.x & 7;
    if (g0 + g_ < groups) {
      float t = 0.f;
      for (int l = 0; l < 32; ++l) t += sh[l][g_][j];
      part[((size_t)n * splits + split) * C + (g0 + g_) * 8 + j] = t;
    }
  }
}

// out[n][c] (bf16, =|+=) scale * sum over splits of part[n][split][c]
__global__ void spatial_sum_fold_kernel(const float* __restrict__ part, int N, int C, int splits, float scale,
                                        __nv_bfloat16* __restrict__ out, int out_ld, int accumulate) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  const int n = i / C, c = i - n * C;
  float t = 0.f;
  for (int s = 0; s < splits; ++s) t += part[((size_t)n * splits + s) * C + c];
  t *= scale;
  __nv_bfloat16* o = out + (size_t)n * out_ld + c;
  if (accumulate) t += __bfloat162float(*o);
  *o = __float2bfloat16_rn(t);
}

__global__ void __launch_bounds__(256)
broadcast_pixels_kernel(const __nv_bfloat16* __restrict__ v, int v_ld, int N, int P, int C, float scale,
                        __nv_bfloat16* __restrict__ out, int out_ld, int accumulate) {
  pdl_sync();
  const int groups = C >> 3;
  const long long total = (long long)N * P * groups;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long pix = idx / groups;
    const int c0 = (int)(idx - pix * groups) << 3;
    const int n = (int)(pix / P);
    float a[8];
    load8(v + (size_t)n * v_ld + c0, a);
    if (accumulate) {
      float o[8];
      load8(out + pix * out_ld + c0, o);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] = o[j] + scale * a[j];
    } else if (scale != 1.f) {
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] *= scale;
    }
    store8(out + pix * out_ld + c0, a);
  }
}

}  // namespace b200seg

using namespace b200seg;

#define POOL_RET(e) return (e) == cudaSuccess ? 0 : (int)(e)

extern "C" int b200seg_maxpool3x3s2_fwd(const void* x, int32_t x_ld, int32_t n, int32_t h, int32_t w, int32_t c, void* y,
                                        int32_t y_ld, void* stream) {
  if (!x || !y || c % 8 || x_ld % 8 || y_ld % 8 || h < 1 || w < 1) return B200SEG_E_BADARG;
  const int ho = (h + 2 - 3) / 2 + 1, wo = (w + 2 - 3) / 2 + 1;
  cudaError_t e = launch_k(maxpool3x3s2_fwd_kernel, dim3(pool_grid((long long)n * ho * wo * (c / 8))), dim3(256), 0,
                           (cudaStream_t)stream, (const __nv_bfloat16*)x, (int)x_ld, (int)n, (int)h, (int)w, (int)c,
                           (__nv_bfloat16*)y, (int)y_ld, ho, wo);
  POOL_RET(e);
}

extern "C" int b200seg_maxpool3x3s2_bwd(const void* x, int32_t x_ld, const void* dy, int32_t dy_ld, int32_t n, int32_t h,
                                        int32_t w, int32_t c, void* dx, int32_t dx_ld, int32_t accumulate, void* stream) {
  if (!x || !dy || !dx || c % 8 || x_ld % 8 || dy_ld % 8 || dx_ld % 8) return B200SEG_E_BADARG;
  const int ho = (h + 2 - 3) / 2 + 1, wo = (w + 2 - 3) / 2 + 1;
  cudaError_t e = launch_k(maxpool3x3s2_bwd_kernel, dim3(pool_grid((long long)n * h * w * (c / 8))), dim3(256), 0,
                           (cudaStream_t)stream, (const __nv_bfloat16*)x, (int)x_ld, (const __nv_bfloat16*)dy, (int)dy_ld,
                           (int)n, (int)h, (int)w, (int)c, ho, wo, (__nv_bfloat16*)dx, (int)dx_ld, (int)accumulate);
  POOL_RET(e);
}

static void stats_shape(int c, int* rows, int* threads) {
  const int groups = c / 8;
  int r = 256 / groups;
  if (r < 1) r = 1;
  if (r > 32) r = 32;
  *rows = r;
  *threads = groups * r > 32 ? ((groups * r + 31) / 32) * 32 : 32;
}

extern "C" int32_t b200seg_channel_stats_grid(int64_t npix, int32_t c) {
  int rows, threads;
  stats_shape(c, &rows, &threads);
  long long b = (npix + rows - 1) / rows;
  return (int32_t)(b < B200SEG_MAX_CTAS ? (b > 0 ? b : 1) : B200SEG_MAX_CTAS);
}

/* partials: fp32 [grid][2][c] with grid = b200seg_channel_stats_grid(npix, c): feed b200seg_bn_finalize(cpad = c) */
extern "C" int b200seg_channel_stats(const void* x, int32_t x_ld, int64_t npix, int32_t c, float* partials, void* stream) {
  if (!x || !partials || c % 8 || c > 2048 || x_ld % 8) return B200SEG_E_BADARG;
  int rows, threads;
  stats_shape(c, &rows, &threads);
  if (threads > 256) return B200SEG_E_BADARG;
  const int grid = b200seg_channel_stats_grid(npix, c);
  cudaError_t e = launch_k(channel_stats_kernel, dim3(grid), dim3(threads), (size_t)rows * (c / 8) * 16 * sizeof(float),
                           (cudaStream_t)stream, (const __nv_bfloat16*)x, (int)x_ld, (long long)npix, (int)c, rows,
                           partials);
  POOL_RET(e);
}

extern "C" int32_t b200seg_spatial_sum_splits(int32_t p) {
  int s = p / 2048;
  return s < 1 ? 1 : (s > 64 ? 64 : s);
}

/* out[n][c] (bf16, pitch out_ld, =|+=) scale * sum_pixels x[n][pix][c]; ws: fp32 [n][splits][c] */
extern "C" int b200seg_spatial_sum(const void* x, int32_t x_ld, int32_t n, int32_t p, int32_t c, float scale, float* ws,
                                   void* out, int32_t out_ld, int32_t accumulate, void* stream) {
  if (!x || !ws || !out || c % 8 || x_ld % 8 || n < 1 || p < 1) return B200SEG_E_BADARG;
  const int splits = b200seg_spatial_sum_splits(p);
  cudaError_t e = launch_k(spatial_sum_partial_kernel, dim3((c / 8 + 7) / 8, splits, n), dim3(256), 0,
                           (cudaStream_t)stream, (const __nv_bfloat16*)x, (int)x_ld, (int)p, (int)c, splits, ws);
  if (e != cudaSuccess) return (int)e;
  e = launch_k(spatial_sum_fold_kernel, dim3((n * c + 255) / 256), dim3(256), 0, (cudaStream_t)stream, (const float*)ws,
               (int)n, (int)c, splits, scale, (__nv_bfloat16*)out, (int)out_ld, (int)accumulate);
  POOL_RET(e);
}

extern "C" int b200seg_broadcast_pixels(const void* v, int32_t v_ld, int32_t n, int32_t p, int32_t c, float scale,
                                        void* out, int32_t out_ld, int32_t accumulate, void* stream) {
  if (!v || !out || c % 8 || v_ld % 8 || out_ld % 8) return B200SEG_E_BADARG;
  cudaError_t e = launch_k(broadcast_pixels_kernel, dim3(pool_grid((long long)n * p * (c / 8))), dim3(256), 0,
                           (cudaStream_t)stream, (const __nv_bfloat16*)v, (int)v_ld, (int)n, (int)p, (int)c, scale,
                           (__nv_bfloat16*)out, (int)out_ld, (int)accumulate);
  POOL_RET(e);
}
