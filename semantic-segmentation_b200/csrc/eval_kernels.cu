// Eval-mode output assembly (network/ocrnet.py:185-262,289-327): full-resolution fp32 NCHW prediction / attention maps
// and the hierarchical multi-scale blend. HBM-bound elementwise / bilinear passes over [N,C,H,W] fp32 maps.
//   resize_to_nchw   NHWC fp32 [n,h,w,ld] (logit heads, 19+1 pad; or 1-channel attention logits with optional sigmoid)
//                    -> NCHW fp32 [n,C,H,W], bilinear align_corners=False (mynn.Upsample / scale_as)
//   resize_nchw      NCHW -> NCHW bilinear (scale_as between full-resolution maps of different scales)
//   blend            out = a*x + (1-a)*y   |  out = x + (1-a)*y   |  out = a*x      (a: [n,1,H,W] broadcast over C)
#include "ptx.cuh"
#include "launch.h"
#include "../../include/b200seg.h"
#include "vec.cuh"

namespace b200seg {

__global__ void __launch_bounds__(256)
resize_to_nchw_kernel(const float* __restrict__ src, int ld, int n, int h, int w, int C, int apply_sigmoid,
                      float* __restrict__ dst, int H, int W) {
  pdl_sync();
  const long long total = (long long)n * C * H * W;
  const float sy = (float)h / (float)H, sx = (float)w / (float)W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(idx % W);
    const int Y = (int)((idx / W) % H);
    const int c = (int)((idx / ((long long)W * H)) % C);
    const int b = (int)(idx / ((long long)W * H * C));
    int y0, y1, x0, x1;
    float ly, lx;
    bilinear_src(Y, sy, h, y0, y1, ly);
    bilinear_src(X, sx, w, x0, x1, lx);
    const float* base = src + (size_t)b * h * w * ld + c;
    float v00 = base[((size_t)y0 * w + x0) * ld], v01 = base[((size_t)y0 * w + x1) * ld];
    float v10 = base[((size_t)y1 * w + x0) * ld], v11 = base[((size_t)y1 * w + x1) * ld];
    if (apply_sigmoid) {
      v00 = 1.f / (1.f + expf(-v00)); v01 = 1.f / (1.f + expf(-v01));
      v10 = 1.f / (1.f + expf(-v10)); v11 = 1.f / (1.f + expf(-v11));
    }
    dst[idx] = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
  }
}

__global__ void __launch_bounds__(256)
resize_nchw_kernel(const float* __restrict__ src, int planes, int h, int w, float* __restrict__ dst, int H, int W) {
  pdl_sync();
  const long long total = (long long)planes * H * W;
  const float sy = (float)h / (float)H, sx = (float)w / (float)W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(idx % W);
    const int Y = (int)((idx / W) % H);
    const long long pl = idx / ((long long)W * H);
    int y0, y1, x0, x1;
    float ly, lx;
    bilinear_src(Y, sy, h, y0, y1, ly);
    bilinear_src(X, sx, w, x0, x1, lx);
    const float* base = src + pl * h * w;
    dst[idx] = (1.f - ly) * ((1.f - lx) * base[(size_t)y0 * w + x0] + lx * base[(size_t)y0 * w + x1]) +
               ly * ((1.f - lx) * base[(size_t)y1 * w + x0] + lx * base[(size_t)y1 * w + x1]);
  }
}

// mode 0: a*x + (1-a)*y ; mode 1: x + (1-a)*y ; mode 2: a*x
__global__ void __launch_bounds__(256)
blend_kernel(const float* __restrict__ a, const float* __restrict__ x, const float* __restrict__ y,
             float* __restrict__ out, int n, int C, long long hw, int mode) {
  pdl_sync();
  const long long total = (long long)n * C * hw;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long p = idx % hw;
    const int b = (int)(idx / (hw * C));
    const float av = a[(size_t)b * hw + p];
    float r;
    if (mode == 0) r = av * x[idx] + (1.f - av) * y[idx];
    else if (mode == 1) r = x[idx] + (1.f - av) * y[idx];
    else r = av * x[idx];
    out[idx] = r;
  }
}

static inline int egrid(long long total) {
  long long b = (total + 255) / 256;
  const long long cap = (long long)B200SEG_MAX_CTAS * 16;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// out (=|+=) pred, optionally mirrored along W: the flip / multi-scale averaging loop of eval_minibatch
// (utils/trnval_utils.py:116-160) without leaving the device.
__global__ void __launch_bounds__(256)
accum_pred_kernel(const float* __restrict__ pred, float* __restrict__ out, long long planes_h, int W, int flip,
                  int accumulate) {
  pdl_sync();
  const long long total = planes_h * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % W);
    const long long row = idx / W;
    const float v = pred[row * W + (flip ? W - 1 - x : x)];
    out[idx] = accumulate ? out[idx] + v : v;
  }
}

// Evaluation tail (utils/trnval_utils.py:160-196, utils/misc.py:50-85): softmax over the classes of the averaged
// prediction, max probability + argmax per pixel, and the C x C confusion histogram hist[gt][pred] += 1 over the pixels
// with 0 <= gt < C. Integer counters (block-local shared histogram, then 64-bit global atomics): order independent.
__global__ void __launch_bounds__(256)
argmax_hist_kernel(const float* __restrict__ pred, int n, int C, long long hw, float scale,
                   const long long* __restrict__ labels, long long* __restrict__ pred_out,
                   float* __restrict__ maxprob_out, unsigned long long* __restrict__ hist) {
  pdl_sync();
  extern __shared__ unsigned int s_hist[];     // [C*C]
  for (int i = threadIdx.x; i < C * C; i += blockDim.x) s_hist[i] = 0u;
  __syncthreads();
  const long long total = (long long)n * hw;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long b = idx / hw, p = idx - b * hw;
    const float* src = pred + (size_t)b * C * hw + p;
    float m = src[0] * scale;
    int arg = 0;
    for (int c = 1; c < C; ++c) {
      const float v = src[(size_t)c * hw] * scale;
      if (v > m) { m = v; arg = c; }          // first maximum wins, like torch.max
    }
    float sum = 0.f;
    for (int c = 0; c < C; ++c) sum += expf(src[(size_t)c * hw] * scale - m);
    if (pred_out) pred_out[idx] = arg;
    if (maxprob_out) maxprob_out[idx] = 1.f / sum;
    if (labels && hist) {
      const long long gt = labels[idx];
      if (gt >= 0 && gt < C) atomicAdd(&s_hist[(int)gt * C + arg], 1u);
    }
  }
  __syncthreads();
  if (hist)
    for (int i = threadIdx.x; i < C * C; i += blockDim.x)
      if (s_hist[i]) atomicAdd(&hist[i], (unsigned long long)s_hist[i]);
}

}  // namespace b200seg

using namespace b200seg;

extern "C" int b200seg_resize_to_nchw(const float* src_nhwc, int32_t ld, int32_t n, int32_t h, int32_t w, int32_t c,
                                      int32_t apply_sigmoid, float* dst_nchw, int32_t H, int32_t W, void* stream) {
  if (!src_nhwc || !dst_nchw || c > ld) return B200SEG_E_BADARG;
  launch_k(resize_to_nchw_kernel, dim3(egrid((long long)n * c * H * W)), dim3(256), 0, (cudaStream_t)stream, src_nhwc,
           ld, n, h, w, c, apply_sigmoid, dst_nchw, H, W);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_resize_nchw(const float* src, int32_t planes, int32_t h, int32_t w, float* dst, int32_t H,
                                   int32_t W, void* stream) {
  if (!src || !dst) return B200SEG_E_BADARG;
  launch_k(resize_nchw_kernel, dim3(egrid((long long)planes * H * W)), dim3(256), 0, (cudaStream_t)stream, src,
           planes, h, w, dst, H, W);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_blend(const float* a, const float* x, const float* y, float* out, int32_t n, int32_t c,
                             int64_t hw, int32_t mode, void* stream) {
  if (!a || !x || !out || (mode != 2 && !y) || mode < 0 || mode > 2) return B200SEG_E_BADARG;
  launch_k(blend_kernel, dim3(egrid((long long)n * c * hw)), dim3(256), 0, (cudaStream_t)stream, a, x, y, out, n, c,
           hw, mode);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_accum_pred(const float* pred, float* out, int32_t n, int32_t c, int32_t h, int32_t w,
                                  int32_t flip, int32_t accumulate, void* stream) {
  if (!pred || !out || n <= 0 || c <= 0 || h <= 0 || w <= 0) return B200SEG_E_BADARG;
  cudaError_t e = launch_k(accum_pred_kernel, dim3(egrid((long long)n * c * h * w)), dim3(256), 0, (cudaStream_t)stream,
                           pred, out, (long long)n * c * h, (int)w, (int)flip, (int)accumulate);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_argmax_hist(const float* pred_nchw, int32_t n, int32_t c, int64_t hw, float scale,
                                   const int64_t* labels, int64_t* pred_out, float* maxprob_out, int64_t* hist,
                                   void* stream) {
  if (!pred_nchw || n <= 0 || c <= 0 || c > 64 || hw <= 0 || (hist && !labels)) return B200SEG_E_BADARG;
  cudaError_t e = launch_k(argmax_hist_kernel, dim3(egrid((long long)n * hw)), dim3(256),
                           (size_t)c * c * sizeof(unsigned), (cudaStream_t)stream, pred_nchw, (int)n, (int)c,
                           (long long)hw, scale, (const long long*)labels, (long long*)pred_out, maxprob_out,
                           (unsigned long long*)hist);
  return e == cudaSuccess ? 0 : (int)e;
}
