// Shared device/host pieces of the multi-scale blend + loss kernels (mscale_loss.cu, rmi_loss.cu).
#pragma once
#include "ptx.cuh"
#include "vec.cuh"
#include "../../include/b200seg.h"

namespace b200seg {

constexpr int NC = 19;      // classes
constexpr int LD = 20;      // logits pitch (floats)
constexpr int MW = 40;      // mid / gradient buffer width

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

struct Taps {
  int i00, i01, i10, i11;   // linear pixel indices within the image
  float w00, w01, w10, w11;
};
__device__ __forceinline__ Taps make_taps(int Y, int X, int H, int W, int h, int w) {
  int y0, y1, x0, x1;
  float ly, lx;
  bilinear_src(Y, (float)h / (float)H, h, y0, y1, ly);
  bilinear_src(X, (float)w / (float)W, w, x0, x1, lx);
  Taps t;
  t.i00 = y0 * w + x0; t.i01 = y0 * w + x1; t.i10 = y1 * w + x0; t.i11 = y1 * w + x1;
  const float hy = 1.f - ly, hx = 1.f - lx;
  t.w00 = hy * hx; t.w01 = hy * lx; t.w10 = ly * hx; t.w11 = ly * lx;
  return t;
}
// PyTorch evaluates h0*(w0*a + w1*b) + h1*(w0*c + w1*d); keep that association.
__device__ __forceinline__ float tap_eval(const Taps& t, float a, float b, float c, float d, float hy, float ly, float hx,
                                          float lx) {
  return hy * (hx * a + lx * b) + ly * (hx * c + lx * d);
}

struct TapW {   // separable weights kept for the PyTorch association order
  int y0, y1, x0, x1;
  float hy, ly, hx, lx;
};
__device__ __forceinline__ TapW make_tapw(int Y, int X, int H, int W, int h, int w) {
  TapW t;
  bilinear_src(Y, (float)h / (float)H, h, t.y0, t.y1, t.ly);
  bilinear_src(X, (float)w / (float)W, w, t.x0, t.x1, t.lx);
  t.hy = 1.f - t.ly; t.hx = 1.f - t.lx;
  return t;
}
__device__ __forceinline__ float interp(const TapW& t, const float* __restrict__ base, int w, int ld, int c) {
  const float a = base[((size_t)t.y0 * w + t.x0) * ld + c], b = base[((size_t)t.y0 * w + t.x1) * ld + c];
  const float cc = base[((size_t)t.y1 * w + t.x0) * ld + c], d = base[((size_t)t.y1 * w + t.x1) * ld + c];
  return t.hy * (t.hx * a + t.lx * b) + t.ly * (t.hx * cc + t.lx * d);
}

// adjoint helpers: fine index range that can touch coarse index y, and the weight of coarse y for fine Y
__device__ __forceinline__ void adj_range(int y, int h, int H, int& lo, int& hi) {
  const float r = (float)H / (float)h;
  lo = (int)floorf(r * (y - 1)) - 1;
  hi = (int)ceilf(r * (y + 2)) + 1;
  if (y == 0 || lo < 0) lo = 0;
  if (y == h - 1 || hi > H) hi = H;
}
__device__ __forceinline__ float adj_weight(int Y, int y, int h, int H) {
  int y0, y1;
  float l;
  bilinear_src(Y, (float)h / (float)H, h, y0, y1, l);
  return (y0 == y ? 1.f - l : 0.f) + (y1 == y ? l : 0.f);
}

struct MsGeom {
  int N, H, W;        // full resolution (labels)
  int Hq, Wq;         // hi-pass quarter maps
  int Hm, Wm;         // mid grid (= lo-pass input size); 0 when there is no lo pass
  int Hl, Wl;         // lo-pass quarter maps
  int nheads;         // 1 (cls only) or 2 (cls, aux)
  float w_head0, w_head1, sup_wt;
  int ignore_index;
  int loss_kind;      // 0: softmax cross-entropy heads; 1: RMILoss criterion (sigmoid BCE heads + RMI on head 0)
};

// Blended logits of head kHead (0: cls, 1: aux) at full-resolution pixel (n, Y, X):
// joint = up2(attn*lo) + (1 - up2(attn)) * up4(hi) (network/ocrnet.py:289-298); without a lo pass just up4(hi).
// hi: that head's quarter-resolution map; the head's blended lo part sits in mid channels [kHead*19, kHead*19+19).
// Same association order as the loss kernel.
template <int kHead>
__device__ __forceinline__ void joint_head(const MsGeom& g, int n, int Y, int X, const float* __restrict__ hi,
                                           const float* __restrict__ M, float (&J)[NC]) {
  const TapW th = make_tapw(Y, X, g.H, g.W, g.Hq, g.Wq);
  const size_t imq = (size_t)n * g.Hq * g.Wq;
#pragma unroll
  for (int c = 0; c < NC; ++c) J[c] = interp(th, hi + imq * LD, g.Wq, LD, c);
  if (g.Hm > 0) {
    const TapW tm = make_tapw(Y, X, g.H, g.W, g.Hm, g.Wm);
    const size_t imm = (size_t)n * g.Hm * g.Wm;
    const float oma = 1.f - interp(tm, M + imm * MW, g.Wm, MW, 2 * NC);
#pragma unroll
    for (int c = 0; c < NC; ++c) J[c] = interp(tm, M + imm * MW, g.Wm, MW, kHead * NC + c) + oma * J[c];
  }
}

static inline MsGeom to_geom(const b200seg_mscale_desc* d) {
  MsGeom g;
  g.N = d->n; g.H = d->h; g.W = d->w; g.Hq = d->hq; g.Wq = d->wq; g.Hm = d->hm; g.Wm = d->wm; g.Hl = d->hl; g.Wl = d->wl;
  g.nheads = d->nheads; g.w_head0 = d->w_head0; g.w_head1 = d->w_head1; g.sup_wt = d->sup_wt;
  g.ignore_index = d->ignore_index;
  g.loss_kind = d->loss_kind;
  return g;
}


inline int blocks_for_total(long long total, int threads, long long cap = 148LL * 16) {
  long long b = (total + threads - 1) / threads;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

}  // namespace b200seg
