// ImageEnhance / ColorJitter arithmetic on one RGB pixel, bit-exact with Pillow 12 (host side: b200seg/augment.py).
// Shared by the colour jitter of augment_kernels.cu and the Color / Brightness / Sharpness ops of randaugment_kernels.cu.
#pragma once

namespace b200seg {

struct AugColor {
  int n_ops;
  int kind[4];                   // 0 brightness, 1 contrast, 2 saturation, 3 hue
  float factor[4];               // ImageEnhance factor (Pillow casts it to float)
  int hue_shift[4];              // np.uint8(hue_factor * 255) of the hue op
  float mean[3], std[3];
};

// Pillow's ImagingBlend(im1, im2, alpha) for one 8-bit sample: in1 + alpha * (in2 - in1) in fp32
__device__ __forceinline__ int aug_blend(int in1, int in2, float alpha) {
  const float t = __fadd_rn((float)in1, __fmul_rn(alpha, (float)(in2 - in1)));
  if (alpha >= 0.f && alpha <= 1.f) return (int)t;
  return t <= 0.f ? 0 : (t >= 255.f ? 255 : (int)t);
}
__device__ __forceinline__ int aug_luma(int r, int g, int b) {      // Pillow's RGB -> L
  return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16;
}

// Pillow's rgb2hsv_row -> uint8 hue shift -> hsv2rgb_row (Convert.c; float h with the double promotions of its literals)
__device__ __forceinline__ void aug_hue(int& r, int& g, int& b, int shift) {
  const int maxc = max(r, max(g, b)), minc = min(r, min(g, b));
  int uh = 0, us = 0;
  const int uv = maxc;
  if (minc != maxc) {
    const float cr = (float)(maxc - minc);
    const float s = __fdiv_rn(cr, (float)maxc);
    const float rc = __fdiv_rn((float)(maxc - r), cr);
    const float gc = __fdiv_rn((float)(maxc - g), cr);
    const float bc = __fdiv_rn((float)(maxc - b), cr);
    float h;
    if (r == maxc) h = __fsub_rn(bc, gc);
    else if (g == maxc) h = (float)__dsub_rn(__dadd_rn(2.0, (double)rc), (double)bc);
    else h = (float)__dsub_rn(__dadd_rn(4.0, (double)gc), (double)rc);
    h = (float)fmod(__dadd_rn(__ddiv_rn((double)h, 6.0), 1.0), 1.0);
    uh = (int)__dmul_rn((double)h, 255.0);
    us = (int)__dmul_rn((double)s, 255.0);
    uh = uh < 0 ? 0 : (uh > 255 ? 255 : uh);
    us = us < 0 ? 0 : (us > 255 ? 255 : us);
  }
  uh = (uh + shift) & 255;                                         // np.uint8 addition wraps
  if (us == 0) { r = g = b = uv; return; }
  const float hf = __fdiv_rn(__fmul_rn((float)uh, 6.0f), 255.0f);
  const float fi = floorf(hf);
  const float f = __fsub_rn(hf, fi);
  const float fs = __fdiv_rn((float)us, 255.0f);
  const float vf = (float)uv;
  auto rnd = [](float x) { const int q = (int)floor((double)x + 0.5); return q < 0 ? 0 : (q > 255 ? 255 : q); };
  const int p = rnd(__fmul_rn(vf, __fsub_rn(1.0f, fs)));
  const int q = rnd(__fmul_rn(vf, __fsub_rn(1.0f, __fmul_rn(fs, f))));
  const int t = rnd(__fmul_rn(vf, __fsub_rn(1.0f, __fmul_rn(fs, __fsub_rn(1.0f, f)))));
  switch (((int)fi) % 6) {
    case 0: r = uv; g = t; b = p; break;
    case 1: r = q; g = uv; b = p; break;
    case 2: r = p; g = uv; b = t; break;
    case 3: r = p; g = q; b = uv; break;
    case 4: r = t; g = p; b = uv; break;
    default: r = uv; g = p; b = q; break;
  }
}

// ops [first, last) of the chain; `mean` is the grey level of the contrast op (only read when that op is in range)
__device__ __forceinline__ void aug_apply_ops(const AugColor& c, int first, int last, int mean, int& r, int& g, int& b) {
  for (int i = first; i < last; ++i) {
    const float a = c.factor[i];
    switch (c.kind[i]) {
      case 0: r = aug_blend(0, r, a); g = aug_blend(0, g, a); b = aug_blend(0, b, a); break;
      case 1: r = aug_blend(mean, r, a); g = aug_blend(mean, g, a); b = aug_blend(mean, b, a); break;
      case 2: { const int l = aug_luma(r, g, b); r = aug_blend(l, r, a); g = aug_blend(l, g, a); b = aug_blend(l, b, a); break; }
      default: aug_hue(r, g, b, c.hue_shift[i]); break;
    }
  }
}

}  // namespace b200seg
