// Multi-resolution plumbing of HRNet as single fused passes over NHWC bf16 (HBM-bound, 16-byte vector accesses):
//   fuse_fwd           y = relu?( sum_j term_j ), term_j = [scale_j*]x_j[+shift_j] sampled bilinearly when x_j is coarser.
//                      One kernel replaces the reference's per-term BN + F.interpolate + add + ReLU launches
//                      (network/hrnetv2.py:230-254) and, with a channel-offset output view, the final upsample+concat
//                      (network/hrnetv2.py:438-447). BN's affine map commutes with bilinear interpolation (weights sum to 1).
//   upsample_adjoint   gl = U^T (g * (mask>0)) in gather form: the exact adjoint of the align_corners=False bilinear
//                      operator U (incl. its border clamping), used by the backward of both call sites above.
//   image_prep         NCHW fp32 image -> NHWC bf16 padded to 16 channels, with the ResizeX bilinear rescale
//                      (network/mynn.py:102-114; scale 0.5 == 2x2 mean) folded in.
#include "ptx.cuh"
#include "launch.h"
#include "conv_common.h"
#include "../../include/b200seg.h"
#include "vec.cuh"

namespace b200seg {

struct FuseTerm {
  const __nv_bfloat16* x;
  const float* scale;   // per-channel (or null)
  const float* shift;
  int ld, h, w;         // source pitch / spatial size
};
struct FuseParams {
  FuseTerm t[4];
  int nterms;
  int N, H, W, C;
  int relu;
};

__global__ void __launch_bounds__(256)
fuse_fwd_kernel(const FuseParams p, __nv_bfloat16* __restrict__ out, int out_ld) {
  pdl_sync();
  const int groups = p.C >> 3;
  const long long total = (long long)p.N * p.H * p.W * groups;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long pix = idx / groups;
    const int c0 = (int)(idx - pix * groups) << 3;
    const int X = (int)(pix % p.W);
    const int Y = (int)((pix / p.W) % p.H);
    const int n = (int)(pix / ((long long)p.W * p.H));
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll 1
    for (int ti = 0; ti < p.nterms; ++ti) {
      const FuseTerm& t = p.t[ti];
      float v[8];
      if (t.h == p.H && t.w == p.W) {
        load8(t.x + pix * t.ld + c0, v);
      } else {
        int y0, y1, x0, x1;
        float ly, lx;
        bilinear_src(Y, (float)t.h / (float)p.H, t.h, y0, y1, ly);
        bilinear_src(X, (float)t.w / (float)p.W, t.w, x0, x1, lx);
        const __nv_bfloat16* base = t.x + (long long)n * t.h * t.w * t.ld + c0;
        float v00[8], v01[8], v10[8], v11[8];
        load8(base + ((long long)y0 * t.w + x0) * t.ld, v00);
        load8(base + ((long long)y0 * t.w + x1) * t.ld, v01);
        load8(base + ((long long)y1 * t.w + x0) * t.ld, v10);
        load8(base + ((long long)y1 * t.w + x1) * t.ld, v11);
        const float hy = 1.f - ly, hx = 1.f - lx;
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = hy * (hx * v00[j] + lx * v01[j]) + ly * (hx * v10[j] + lx * v11[j]);
      }
      if (t.scale) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = v[j] * __ldg(t.scale + c0 + j) + __ldg(t.shift + c0 + j);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
    if (p.relu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaxf(acc[j], 0.f);
    }
    store8(out + pix * out_ld + c0, acc);
  }
}

// gl[n,y,x,c] = sum over fine pixels (Y,X) of w(Y,y) * w(X,x) * g[n,Y,X,c] * (mask[n,Y,X,c] > 0)
// LANES (1, 4, 16 or 32, by upsampling ratio) consecutive lanes share one (coarse pixel, 8-channel group): they stride
// over the flattened fine window and fold their partial sums with a fixed xor butterfly (deterministic). A x8 adjoint
// gathers ~256 fine pixels per output: one thread per output would be a 500-load latency chain on 12k threads.
template <int LANES>
__global__ void __launch_bounds__(256)
upsample_adjoint_kernel(const __nv_bfloat16* __restrict__ g, int g_ld, const __nv_bfloat16* __restrict__ mask,
                        int mask_ld, int N, int H, int W, int C, __nv_bfloat16* __restrict__ out, int out_ld, int h,
                        int w, int accumulate) {
  pdl_sync();
  const int groups = C >> 3;
  const long long total = (long long)N * h * w * groups;
  const float sy = (float)h / (float)H, sx = (float)w / (float)W;
  const float ry = (float)H / (float)h, rx = (float)W / (float)w;   // upsampling ratio
  const int sub = threadIdx.x % LANES;
  const long long total_padded = (total + (256 / LANES) - 1) / (256 / LANES) * (256 / LANES);
  for (long long idx = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / LANES; idx < total_padded;
       idx += (long long)gridDim.x * blockDim.x / LANES) {
    const bool live = idx < total;       // whole LANES-groups stay in the loop together (shuffles below)
    const long long idc = live ? idx : total - 1;
    const long long pix = idc / groups;
    const int c0 = (int)(idc - pix * groups) << 3;
    const int x = (int)(pix % w);
    const int y = (int)((pix / w) % h);
    const int n = (int)(pix / ((long long)w * h));
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // fine pixel Y touches coarse row y iff its source coordinate (Y + 0.5) / ry - 0.5 lies in (y - 1, y + 1), i.e.
    // Y in (ry (y - 0.5) - 0.5, ry (y + 1.5) - 0.5): 2 ry candidates (+1 on each side against rounding); the clamped
    // border rows / columns absorb everything beyond
    int Y_lo = (int)floorf(ry * (y - 0.5f) - 0.5f) - 1, Y_hi = (int)ceilf(ry * (y + 1.5f) - 0.5f) + 1;
    int X_lo = (int)floorf(rx * (x - 0.5f) - 0.5f) - 1, X_hi = (int)ceilf(rx * (x + 1.5f) - 0.5f) + 1;
    if (y == 0) Y_lo = 0;
    if (x == 0) X_lo = 0;
    if (Y_lo < 0) Y_lo = 0;
    if (X_lo < 0) X_lo = 0;
    if (Y_hi > H || y == h - 1) Y_hi = H;
    if (X_hi > W || x == w - 1) X_hi = W;
    const int wx_n = X_hi - X_lo;
    const int cells = (Y_hi - Y_lo) * wx_n;
    for (int cell = sub; cell < cells; cell += LANES) {
      const int Y = Y_lo + cell / wx_n, X = X_lo + cell % wx_n;
      int y0, y1, x0, x1;
      float ly, lx;
      bilinear_src(Y, sy, h, y0, y1, ly);
      const float wy = (y0 == y ? 1.f - ly : 0.f) + (y1 == y ? ly : 0.f);
      if (wy == 0.f) continue;
      bilinear_src(X, sx, w, x0, x1, lx);
      const float wx = (x0 == x ? 1.f - lx : 0.f) + (x1 == x ? lx : 0.f);
      if (wx == 0.f) continue;
      const long long fp = ((long long)n * H + Y) * W + X;
      float v[8];
      load8(g + fp * g_ld + c0, v);
      if (mask) {
        float mk[8];
        load8(mask + fp * mask_ld + c0, mk);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = mk[j] > 0.f ? v[j] : 0.f;
      }
      const float wgt = wy * wx;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += wgt * v[j];
    }
#pragma unroll
    for (int off = LANES / 2; off >= 1; off >>= 1) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], off);
    }
    if (sub == 0 && live) {
      if (accumulate) {
        float old[8];
        load8(out + pix * out_ld + c0, old);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += old[j];
      }
      store8(out + pix * out_ld + c0, acc);
    }
  }
}

// images fp32 NCHW [N,3,H,W] -> bf16 NHWC [N,h,w,16] (channels 3..15 zero), bilinear-resized to (h,w).
__global__ void __launch_bounds__(256)
image_prep_kernel(const float* __restrict__ img, int N, int H, int W, __nv_bfloat16* __restrict__ out, int h, int w) {
  pdl_sync();
  const long long total = (long long)N * h * w;
  const float sy = (float)H / (float)h, sx = (float)W / (float)w;
  for (long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x; pix < total;
       pix += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(pix % w);
    const int y = (int)((pix / w) % h);
    const int n = (int)(pix / ((long long)w * h));
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
    if (h == H && w == W) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = img[(((long long)n * 3 + c) * H + y) * W + x];
    } else {
      int y0, y1, x0, x1;
      float ly, lx;
      bilinear_src(y, sy, H, y0, y1, ly);
      bilinear_src(x, sx, W, x0, x1, lx);
      const float hy = 1.f - ly, hx = 1.f - lx;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float* pl = img + ((long long)n * 3 + c) * H * W;
        v[c] = hy * (hx * pl[(long long)y0 * W + x0] + lx * pl[(long long)y0 * W + x1]) +
               ly * (hx * pl[(long long)y1 * W + x0] + lx * pl[(long long)y1 * W + x1]);
      }
    }
    float z[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) z[j] = 0.f;
    store8(out + pix * 16, v);
    store8(out + pix * 16 + 8, z);
  }
}

static inline int ew_grid(long long total_threads) {
  const long long per = 256LL * (tune().rs_items > 0 ? tune().rs_items : 1);
  long long b = (total_threads + per - 1) / per;
  const long long cap = (long long)B200SEG_MAX_CTAS * 8;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

}  // namespace b200seg

using namespace b200seg;

extern "C" int b200seg_fuse_fwd(const b200seg_fuse_desc* d, void* out, int32_t out_ld, void* stream) {
  if (!d || !out || d->nterms < 1 || d->nterms > 4 || d->c % 8 || out_ld % 8) return B200SEG_E_BADARG;
  FuseParams p;
  p.nterms = d->nterms;
  p.N = d->n; p.H = d->h; p.W = d->w; p.C = d->c; p.relu = d->relu;
  for (int i = 0; i < d->nterms; ++i) {
    if (!d->term[i].x || d->term[i].ld % 8) return B200SEG_E_BADARG;
    if ((d->term[i].scale == nullptr) != (d->term[i].shift == nullptr)) return B200SEG_E_BADARG;
    p.t[i].x = (const __nv_bfloat16*)d->term[i].x;
    p.t[i].scale = d->term[i].scale;
    p.t[i].shift = d->term[i].shift;
    p.t[i].ld = d->term[i].ld; p.t[i].h = d->term[i].h; p.t[i].w = d->term[i].w;
  }
  const long long total = (long long)d->n * d->h * d->w * (d->c / 8);
  launch_k(fuse_fwd_kernel, dim3(ew_grid(total)), dim3(256), 0, (cudaStream_t)stream, p, (__nv_bfloat16*)out, out_ld);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_upsample_adjoint(const void* g, int32_t g_ld, const void* mask, int32_t mask_ld, int32_t n,
                                        int32_t H, int32_t W, int32_t c, void* out, int32_t out_ld, int32_t h, int32_t w,
                                        int32_t accumulate, void* stream) {
  if (!g || !out || c % 8 || g_ld % 8 || out_ld % 8 || h > H || w > W) return B200SEG_E_BADARG;
  const long long total = (long long)n * h * w * (c / 8);
  const int ratio = (H + h - 1) / h;
  const cudaStream_t st = (cudaStream_t)stream;
  const __nv_bfloat16 *gp = (const __nv_bfloat16*)g, *mp = (const __nv_bfloat16*)mask;
  __nv_bfloat16* op = (__nv_bfloat16*)out;
  cudaError_t e;
  if (ratio >= 8)
    e = launch_k(upsample_adjoint_kernel<32>, dim3(ew_grid(total * 32)), dim3(256), 0, st, gp, g_ld, mp, mask_ld, n,
                 H, W, c, op, out_ld, h, w, accumulate);
  else if (ratio >= 4)
    e = launch_k(upsample_adjoint_kernel<16>, dim3(ew_grid(total * 16)), dim3(256), 0, st, gp, g_ld, mp, mask_ld, n,
                 H, W, c, op, out_ld, h, w, accumulate);
  else if (ratio >= 2)
    e = launch_k(upsample_adjoint_kernel<4>, dim3(ew_grid(total * 4)), dim3(256), 0, st, gp, g_ld, mp, mask_ld, n, H,
                 W, c, op, out_ld, h, w, accumulate);
  else
    e = launch_k(upsample_adjoint_kernel<1>, dim3(ew_grid(total)), dim3(256), 0, st, gp, g_ld, mp, mask_ld, n, H, W,
                 c, op, out_ld, h, w, accumulate);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_image_prep(const float* img_nchw, int32_t n, int32_t H, int32_t W, void* out_nhwc16, int32_t h,
                                  int32_t w, void* stream) {
  if (!img_nchw || !out_nhwc16 || h <= 0 || w <= 0) return B200SEG_E_BADARG;
  launch_k(image_prep_kernel, dim3(ew_grid((long long)n * h * w)), dim3(256), 0, (cudaStream_t)stream, img_nchw, n, H,
           W, (__nv_bfloat16*)out_nhwc16, h, w);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}
