// Hierarchical multi-scale attention blend + per-pixel cross-entropy, forward and backward, without ever
// materialising a full-resolution [N,19,H,W] fp32 logit tensor.
//
// Reference semantics (network/ocrnet.py:170-183,264-319; twin network/mscale.py:182-220; loss/utils.py:133-134):
//   per scale pass  : cls/aux/attn at 1/4 of the pass input, bilinearly upsampled x4 (Upsample, fp32, align_corners=False)
//   two-scale blend : p_lo = attn * cls_lo  at the lo-pass input size ("mid" grid), then scale_as (x2) to full size;
//                     joint = up2(p_lo) + (1 - up2(attn)) * cls_hi      (same for aux)
//   loss            : OCR_ALPHA * CE(joint_aux) + CE(joint_cls) [+ w * CE(up2(cls_lo_x4)) + w * CE(cls_hi_x4)]
// The two cascaded upsamples are kept separate (x4 then x2), exactly like the reference (SURVEY §7 hard part 5).
//
// Kernels (C = 19 classes, logits fp32 [pixels][20], class-gradient outputs bf16 [pixels][32] zero padded):
//   mid_fwd      lo quarter maps -> mid buffer M[m][40] = {attn4*cls4 (19), attn4*aux4 (19), attn4, 0} (+ cls4 for the
//                supervised term)
//   loss_fwd     per full-res pixel: gather 4 mid taps + 4 hi taps, blend, log-softmax / NLL for each head, write the
//                per-pixel gradients w.r.t. the hi path (Ghi), the lo path (Glo) and block-partial loss sums
//   hi_bwd       adjoint of the x4 upsample: Ghi -> d cls_hi, d aux_hi
//   mid_bwd      adjoint of the x2 upsample + product rule at the mid grid -> D[m][40]
//   lo_bwd       adjoint of the x4 upsample on the lo pass -> d cls_lo, d aux_lo, d attn_logit (through the sigmoid)
#include "ptx.cuh"
#include "launch.h"
#include "../../include/b200seg.h"
#include "vec.cuh"
#include "mscale_common.cuh"

namespace b200seg {

// ------------------------------------------------------------------------------------------------ mid_fwd
__global__ void __launch_bounds__(256)
mid_fwd_kernel(const MsGeom g, const float* __restrict__ lo_cls, const float* __restrict__ lo_aux,
               const float* __restrict__ lo_attn, float* __restrict__ M, float* __restrict__ M2) {
  pdl_sync();
  const long long total = (long long)g.N * g.Hm * g.Wm;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(idx % g.Wm), Y = (int)((idx / g.Wm) % g.Hm), n = (int)(idx / ((long long)g.Wm * g.Hm));
    const TapW t = make_tapw(Y, X, g.Hm, g.Wm, g.Hl, g.Wl);
    const size_t img = (size_t)n * g.Hl * g.Wl;
    const float* at = lo_attn + img;
    const float a00 = sigmoidf_(at[t.y0 * g.Wl + t.x0]), a01 = sigmoidf_(at[t.y0 * g.Wl + t.x1]);
    const float a10 = sigmoidf_(at[t.y1 * g.Wl + t.x0]), a11 = sigmoidf_(at[t.y1 * g.Wl + t.x1]);
    const float A4 = t.hy * (t.hx * a00 + t.lx * a01) + t.ly * (t.hx * a10 + t.lx * a11);
    float* out = M + idx * MW;
    const float* cb = lo_cls + img * LD;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const float v = interp(t, cb, g.Wl, LD, c);
      out[c] = A4 * v;
      if (M2) M2[idx * LD + c] = v;
    }
    if (g.nheads > 1) {
      const float* ab = lo_aux + img * LD;
#pragma unroll
      for (int c = 0; c < NC; ++c) out[NC + c] = A4 * interp(t, ab, g.Wl, LD, c);
    } else {
#pragma unroll
      for (int c = 0; c < NC; ++c) out[NC + c] = 0.f;
    }
    out[2 * NC] = A4;
    out[2 * NC + 1] = 0.f;
  }
}

// log-softmax / NLL of one 19-vector; returns nll (0 if invalid) and overwrites J with (softmax - onehot) * coef
__device__ __forceinline__ float ce_grad(float (&J)[NC], int label, bool valid, float coef) {
  float m = J[0];
#pragma unroll
  for (int c = 1; c < NC; ++c) m = fmaxf(m, J[c]);
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < NC; ++c) s += expf(J[c] - m);
  const float lse = m + logf(s);
  float nll = 0.f;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const float pr = expf(J[c] - lse);
    if (c == label) nll = lse - J[c];
    J[c] = valid ? (pr - (c == label ? 1.f : 0.f)) * coef : 0.f;
  }
  return valid ? nll : 0.f;
}

// RMILoss criterion, pointwise part (loss/rmi.py:88-96): binary cross-entropy with logits against the one-hot target,
// summed over the 19 classes of a valid pixel; overwrites J with (sigmoid - onehot) * coef. P (optional) receives sigmoid.
__device__ __forceinline__ float bce_grad(float (&J)[NC], int label, bool valid, float coef, float* P) {
  float loss = 0.f;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const float z = J[c];
    const float y = c == label ? 1.f : 0.f;
    const float sp = fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)));
    const float pr = sigmoidf_(z);
    if (P) P[c] = pr;
    loss += sp;
    J[c] = valid ? (pr - y) * coef : 0.f;
  }
  return valid ? loss : 0.f;
}
constexpr float kRmiLambda = 0.5f;     // cfg.LOSS / RMILoss(loss_weight_lambda=0.5), loss/rmi.py:48

__device__ __forceinline__ void store_row40(__nv_bfloat16* dst, const float (&a)[NC], const float (&b)[NC], float e38,
                                            float e39) {
  float v[MW];
#pragma unroll
  for (int c = 0; c < NC; ++c) { v[c] = a[c]; v[NC + c] = b[c]; }
  v[38] = e38; v[39] = e39;
#pragma unroll
  for (int q = 0; q < 5; ++q) {
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = v[q * 8 + j];
    store8(dst + q * 8, o);
  }
}

// ------------------------------------------------------------------------------------------------ loss_fwd
// partial[block][4] = sums of nll over valid pixels for {cls head, aux head, supervised lo, supervised hi}
__global__ void __launch_bounds__(128)
loss_fwd_kernel(const MsGeom g, const long long* __restrict__ labels, const float* __restrict__ inv_count,
                const float* __restrict__ hi_cls, const float* __restrict__ hi_aux, const float* __restrict__ M,
                const float* __restrict__ M2, __nv_bfloat16* __restrict__ Ghi, __nv_bfloat16* __restrict__ Glo,
                __nv_bfloat16* __restrict__ Gsup, float* __restrict__ partial, const float* __restrict__ rmi_dpr,
                int Hp, int Wp) {
  pdl_sync();
  const long long total = (long long)g.N * g.H * g.W;
  const bool has_lo = g.Hm > 0;
  const bool rmi = g.loss_kind == 1;
  const float icnt = *inv_count;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(idx % g.W), Y = (int)((idx / g.W) % g.H), n = (int)(idx / ((long long)g.W * g.H));
    const long long lab64 = labels[idx];
    const bool valid = lab64 != (long long)g.ignore_index;
    const int label = valid ? (int)lab64 : -1;
    const TapW th = make_tapw(Y, X, g.H, g.W, g.Hq, g.Wq);
    const size_t imq = (size_t)n * g.Hq * g.Wq;
    float hc[NC], ha[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) hc[c] = interp(th, hi_cls + imq * LD, g.Wq, LD, c);
    if (g.nheads > 1) {
#pragma unroll
      for (int c = 0; c < NC; ++c) ha[c] = interp(th, hi_aux + imq * LD, g.Wq, LD, c);
    } else {
#pragma unroll
      for (int c = 0; c < NC; ++c) ha[c] = 0.f;
    }
    float oma = 1.f;   // 1 - up2(attn)
    float Jc[NC], Ja[NC];
    TapW tm;
    size_t imm = 0;
    if (has_lo) {
      tm = make_tapw(Y, X, g.H, g.W, g.Hm, g.Wm);
      imm = (size_t)n * g.Hm * g.Wm;
      const float Aup = interp(tm, M + imm * MW, g.Wm, MW, 2 * NC);
      oma = 1.f - Aup;
#pragma unroll
      for (int c = 0; c < NC; ++c) Jc[c] = interp(tm, M + imm * MW, g.Wm, MW, c) + oma * hc[c];
      if (g.nheads > 1) {
#pragma unroll
        for (int c = 0; c < NC; ++c) Ja[c] = interp(tm, M + imm * MW, g.Wm, MW, NC + c) + oma * ha[c];
      }
    } else {
#pragma unroll
      for (int c = 0; c < NC; ++c) { Jc[c] = hc[c]; Ja[c] = ha[c]; }
    }
    if (rmi) {
      // head 0: lambda * BCE + (1 - lambda) * RMI; the RMI gradient arrives per 4x4 pooling cell (rmi_loss.cu):
      // d probs / d z = mask * p (1 - p), avg-pool adjoint = 1/16 (loss/rmi.py:99-111)
      float P[NC];
      acc[0] += bce_grad(Jc, label, valid, g.w_head0 * kRmiLambda * icnt, P);
      if (rmi_dpr != nullptr && valid) {
        const float* dp = rmi_dpr + (((size_t)n * Hp + ((Y + 2) >> 2)) * Wp + ((X + 2) >> 2)) * LD;
#pragma unroll
        for (int c = 0; c < NC; ++c) Jc[c] += dp[c] * 0.0625f * P[c] * (1.f - P[c]);
      }
      if (g.nheads > 1) acc[1] += bce_grad(Ja, label, valid, g.w_head1 * icnt, nullptr);   // aux head: do_rmi=False
    } else {
      acc[0] += ce_grad(Jc, label, valid, g.w_head0 * icnt);
      if (g.nheads > 1) acc[1] += ce_grad(Ja, label, valid, g.w_head1 * icnt);
    }
    if (g.nheads <= 1) {
#pragma unroll
      for (int c = 0; c < NC; ++c) Ja[c] = 0.f;
    }
    // lo-path gradients: dP = gJ, dA = -sum hi*gJ
    if (has_lo) {
      float gA = 0.f;
#pragma unroll
      for (int c = 0; c < NC; ++c) gA -= hc[c] * Jc[c] + ha[c] * Ja[c];
      store_row40(Glo + idx * MW, Jc, Ja, gA, 0.f);
    }
    // hi-path gradients: (1 - Aup) * gJ (+ supervised term on the hi prediction alone)
    float gh[NC], gha[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) { gh[c] = oma * Jc[c]; gha[c] = oma * Ja[c]; }
    if (g.sup_wt != 0.f) {
      float S[NC];
#pragma unroll
      for (int c = 0; c < NC; ++c) S[c] = hc[c];
      acc[3] += rmi ? bce_grad(S, label, valid, g.sup_wt * icnt, nullptr) : ce_grad(S, label, valid, g.sup_wt * icnt);
#pragma unroll
      for (int c = 0; c < NC; ++c) gh[c] += S[c];
      if (has_lo) {
#pragma unroll
        for (int c = 0; c < NC; ++c) S[c] = interp(tm, M2 + imm * LD, g.Wm, LD, c);
        acc[2] += rmi ? bce_grad(S, label, valid, g.sup_wt * icnt, nullptr) : ce_grad(S, label, valid, g.sup_wt * icnt);
        float z[NC];
#pragma unroll
        for (int c = 0; c < NC; ++c) z[c] = 0.f;
        store_row40(Gsup + idx * MW, S, z, 0.f, 0.f);
      }
    }
    store_row40(Ghi + idx * MW, gh, gha, 0.f, oma);
  }
  __shared__ float s_acc[4][4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float a = acc[k];
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
    if (lane == 0) s_acc[warp][k] = a;
  }
  __syncthreads();
  if (threadIdx.x < 4)
    partial[(size_t)blockIdx.x * 4 + threadIdx.x] =
        (s_acc[0][threadIdx.x] + s_acc[1][threadIdx.x]) + (s_acc[2][threadIdx.x] + s_acc[3][threadIdx.x]);
}

// loss = icnt * (w0*s0 + w1*s1 + sup*(s2 + s3)); also returns the four mean NLLs
__global__ void loss_finalize_kernel(const float* __restrict__ partial, int nblocks, const float* __restrict__ inv_count,
                                     float w0, float w1, float sup, float* __restrict__ out,
                                     const float* __restrict__ rmi_terms, int n_rmi) {
  pdl_sync();
  __shared__ double s[4][32];
  double a[4] = {0, 0, 0, 0};
  for (int b = threadIdx.x; b < nblocks; b += 32)
    for (int k = 0; k < 4; ++k) a[k] += (double)partial[(size_t)b * 4 + k];
  for (int k = 0; k < 4; ++k) s[k][threadIdx.x] = a[k];
  __syncthreads();
  if (threadIdx.x == 0) {
    double t[4] = {0, 0, 0, 0};
    for (int k = 0; k < 4; ++k)
      for (int i = 0; i < 32; ++i) t[k] += s[k][i];
    const double ic = (double)*inv_count;
    double r = 0.0;                          // (1 - lambda) * w0 * sum_c mean_n(rmi_nc) / 9, already scaled per term
    for (int i = 0; i < n_rmi; ++i) r += (double)rmi_terms[i];
    out[0] = (float)(ic * (w0 * t[0] + w1 * t[1] + sup * (t[2] + t[3])) + r);
    for (int k = 0; k < 4; ++k) out[1 + k] = (float)(ic * t[k]);
    out[5] = (float)r;
  }
}

__global__ void count_valid_kernel(const long long* __restrict__ labels, long long total, int ignore_index,
                                   unsigned long long* __restrict__ counter) {
  pdl_sync();
  unsigned int c = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    c += labels[i] != (long long)ignore_index;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(counter, (unsigned long long)c);   // integer: order independent
}
__global__ void inv_count_kernel(const unsigned long long* __restrict__ counter, float* __restrict__ inv_count,
                                 int plus_one) {
  pdl_sync();
  // CE: mean over non-ignored pixels (all-ignored -> inf/NaN like the reference); RMILoss: sum / (valid + 1), rmi.py:95
  *inv_count = 1.f / ((float)(*counter) + (plus_one ? 1.f : 0.f));
}

// ------------------------------------------------------------------------------------------------ hi_bwd
// d hi[q][c] = sum_X w(X,q) * Ghi[X][c]     (one thread per quarter pixel and head)
__global__ void __launch_bounds__(128)
hi_bwd_kernel(const MsGeom g, const __nv_bfloat16* __restrict__ Ghi, __nv_bfloat16* __restrict__ d_cls,
              __nv_bfloat16* __restrict__ d_aux) {
  pdl_sync();
  const long long total = (long long)g.N * g.Hq * g.Wq * g.nheads;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int head = (int)(idx % g.nheads);
    const long long q = idx / g.nheads;
    const int x = (int)(q % g.Wq), y = (int)((q / g.Wq) % g.Hq), n = (int)(q / ((long long)g.Wq * g.Hq));
    float acc[24];
#pragma unroll
    for (int c = 0; c < 24; ++c) acc[c] = 0.f;
    int Ylo, Yhi, Xlo, Xhi;
    adj_range(y, g.Hq, g.H, Ylo, Yhi);
    adj_range(x, g.Wq, g.W, Xlo, Xhi);
    for (int Y = Ylo; Y < Yhi; ++Y) {
      const float wy = adj_weight(Y, y, g.Hq, g.H);
      if (wy == 0.f) continue;
      for (int X = Xlo; X < Xhi; ++X) {
        const float wx = adj_weight(X, x, g.Wq, g.W);
        if (wx == 0.f) continue;
        const __nv_bfloat16* src = Ghi + (((size_t)n * g.H + Y) * g.W + X) * MW;
        const float wgt = wy * wx;
        // head 0 occupies [0,19), head 1 [19,38): read the three 8-wide groups covering the head
        const int base = head == 0 ? 0 : 16;
        float v[24];
        float t8[8];
        load8(src + base, t8);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = t8[j];
        load8(src + base + 8, t8);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[8 + j] = t8[j];
        load8(src + base + 16, t8);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[16 + j] = t8[j];
#pragma unroll
        for (int c = 0; c < 24; ++c) acc[c] += wgt * v[c];
      }
    }
    // head 0: channels acc[0..18]; head 1: acc[3..21]
    float o[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) o[c] = 0.f;
    if (head == 0) {
#pragma unroll
      for (int c = 0; c < NC; ++c) o[c] = acc[c];
    } else {
#pragma unroll
      for (int c = 0; c < NC; ++c) o[c] = acc[c + 3];
    }
    __nv_bfloat16* dst = (head == 0 ? d_cls : d_aux) + q * 32;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float t8[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) t8[j] = o[k * 8 + j];
      store8(dst + k * 8, t8);
    }
  }
}

// ------------------------------------------------------------------------------------------------ mid_bwd
// D[m][c] = A4[m] * dP[m][c] (+ supervised d cls4), D[m][38] = sum_c C4[m][c]*dP[m][c] + dA[m]
__global__ void __launch_bounds__(128)
mid_bwd_kernel(const MsGeom g, const __nv_bfloat16* __restrict__ Glo, const __nv_bfloat16* __restrict__ Gsup,
               const float* __restrict__ lo_cls, const float* __restrict__ lo_aux, const float* __restrict__ M,
               float* __restrict__ D) {
  pdl_sync();
  const long long total = (long long)g.N * g.Hm * g.Wm;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % g.Wm), y = (int)((idx / g.Wm) % g.Hm), n = (int)(idx / ((long long)g.Wm * g.Hm));
    float dP[MW];
    float dS[24];
#pragma unroll
    for (int c = 0; c < MW; ++c) dP[c] = 0.f;
#pragma unroll
    for (int c = 0; c < 24; ++c) dS[c] = 0.f;
    int Ylo, Yhi, Xlo, Xhi;
    adj_range(y, g.Hm, g.H, Ylo, Yhi);
    adj_range(x, g.Wm, g.W, Xlo, Xhi);
    for (int Y = Ylo; Y < Yhi; ++Y) {
      const float wy = adj_weight(Y, y, g.Hm, g.H);
      if (wy == 0.f) continue;
      for (int X = Xlo; X < Xhi; ++X) {
        const float wx = adj_weight(X, x, g.Wm, g.W);
        if (wx == 0.f) continue;
        const size_t fp = ((size_t)n * g.H + Y) * g.W + X;
        const float wgt = wy * wx;
#pragma unroll
        for (int k = 0; k < 5; ++k) {
          float t8[8];
          load8(Glo + fp * MW + k * 8, t8);
#pragma unroll
          for (int j = 0; j < 8; ++j) dP[k * 8 + j] += wgt * t8[j];
        }
        if (Gsup) {
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            float t8[8];
            load8(Gsup + fp * MW + k * 8, t8);
#pragma unroll
            for (int j = 0; j < 8; ++j) dS[k * 8 + j] += wgt * t8[j];
          }
        }
      }
    }
    const float A4 = M[idx * MW + 2 * NC];
    const TapW t = make_tapw(y, x, g.Hm, g.Wm, g.Hl, g.Wl);
    const size_t img = (size_t)n * g.Hl * g.Wl;
    float dA = dP[2 * NC];
    float* out = D + idx * MW;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const float C4 = interp(t, lo_cls + img * LD, g.Wl, LD, c);
      dA += C4 * dP[c];
      out[c] = A4 * dP[c] + dS[c];
    }
    if (g.nheads > 1) {
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const float C4 = interp(t, lo_aux + img * LD, g.Wl, LD, c);
        dA += C4 * dP[NC + c];
        out[NC + c] = A4 * dP[NC + c];
      }
    } else {
#pragma unroll
      for (int c = 0; c < NC; ++c) out[NC + c] = 0.f;
    }
    out[2 * NC] = dA;
    out[2 * NC + 1] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------------ lo_bwd
__global__ void __launch_bounds__(128)
lo_bwd_kernel(const MsGeom g, const float* __restrict__ D, const float* __restrict__ lo_attn,
              __nv_bfloat16* __restrict__ d_cls, __nv_bfloat16* __restrict__ d_aux, __nv_bfloat16* __restrict__ d_attn) {
  pdl_sync();
  const long long total = (long long)g.N * g.Hl * g.Wl;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % g.Wl), y = (int)((idx / g.Wl) % g.Hl), n = (int)(idx / ((long long)g.Wl * g.Hl));
    float acc[MW];
#pragma unroll
    for (int c = 0; c < MW; ++c) acc[c] = 0.f;
    int Ylo, Yhi, Xlo, Xhi;
    adj_range(y, g.Hl, g.Hm, Ylo, Yhi);
    adj_range(x, g.Wl, g.Wm, Xlo, Xhi);
    for (int Y = Ylo; Y < Yhi; ++Y) {
      const float wy = adj_weight(Y, y, g.Hl, g.Hm);
      if (wy == 0.f) continue;
      for (int X = Xlo; X < Xhi; ++X) {
        const float wx = adj_weight(X, x, g.Wl, g.Wm);
        if (wx == 0.f) continue;
        const float4* src = reinterpret_cast<const float4*>(D + (((size_t)n * g.Hm + Y) * g.Wm + X) * MW);
        const float wgt = wy * wx;
#pragma unroll
        for (int k = 0; k < 10; ++k) {
          const float4 v = src[k];
          acc[k * 4] += wgt * v.x; acc[k * 4 + 1] += wgt * v.y; acc[k * 4 + 2] += wgt * v.z; acc[k * 4 + 3] += wgt * v.w;
        }
      }
    }
    float o[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) o[c] = c < NC ? acc[c] : 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float t8[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) t8[j] = o[k * 8 + j];
      store8(d_cls + idx * 32 + k * 8, t8);
    }
    if (g.nheads > 1) {
#pragma unroll
      for (int c = 0; c < 32; ++c) o[c] = c < NC ? acc[NC + c] : 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float t8[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) t8[j] = o[k * 8 + j];
        store8(d_aux + idx * 32 + k * 8, t8);
      }
    }
    const float s = sigmoidf_(lo_attn[idx]);
    float t8[8] = {acc[2 * NC] * s * (1.f - s), 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    store8(d_attn + idx * 8, t8);
  }
}

static inline int blocks_for(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = (long long)B200SEG_MAX_CTAS * 16;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace b200seg

using namespace b200seg;

#define RET_LAUNCH()                        \
  do {                                      \
    cudaError_t e_ = cudaGetLastError();    \
    return e_ == cudaSuccess ? 0 : (int)e_; \
  } while (0)

extern "C" int32_t b200seg_mscale_loss_blocks(const b200seg_mscale_desc* d) {
  return blocks_for((long long)d->n * d->h * d->w, 128);
}

extern "C" int b200seg_count_valid(const int64_t* labels, int64_t total, int32_t ignore_index, int32_t plus_one,
                                   uint64_t* counter_ws, float* inv_count, void* stream) {
  if (!labels || !counter_ws || !inv_count) return B200SEG_E_BADARG;
  cudaError_t e = cudaMemsetAsync(counter_ws, 0, sizeof(uint64_t), (cudaStream_t)stream);
  if (e != cudaSuccess) return (int)e;
  launch_k(count_valid_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, (cudaStream_t)stream,
           (const long long*)labels, total, ignore_index, (unsigned long long*)counter_ws);
  launch_k(inv_count_kernel, dim3(1), dim3(1), 0, (cudaStream_t)stream, (const unsigned long long*)counter_ws,
           inv_count, (int)plus_one);
  RET_LAUNCH();
}

extern "C" int b200seg_mscale_mid_fwd(const b200seg_mscale_desc* d, const float* lo_cls, const float* lo_aux,
                                      const float* lo_attn_logit, float* mid, float* mid_sup, void* stream) {
  if (!d || !lo_cls || !lo_attn_logit || !mid || d->hm <= 0 || (d->nheads > 1 && !lo_aux)) return B200SEG_E_BADARG;
  launch_k(mid_fwd_kernel, dim3(blocks_for((long long)d->n * d->hm * d->wm, 256)), dim3(256), 0, (cudaStream_t)stream,
           to_geom(d), lo_cls, lo_aux, lo_attn_logit, mid, mid_sup);
  RET_LAUNCH();
}

extern "C" int b200seg_mscale_loss_fwd(const b200seg_mscale_desc* d, const int64_t* labels, const float* inv_count,
                                       const float* hi_cls, const float* hi_aux, const float* mid, const float* mid_sup,
                                       void* g_hi, void* g_lo, void* g_sup, float* partial_ws, float* loss_out,
                                       const float* rmi_dpr, const float* rmi_terms, int32_t n_rmi_terms,
                                       void* stream) {
  if (!d || !labels || !inv_count || !hi_cls || !g_hi || !partial_ws || !loss_out) return B200SEG_E_BADARG;
  if (d->nheads > 1 && !hi_aux) return B200SEG_E_BADARG;
  if (d->hm > 0 && (!mid || !g_lo)) return B200SEG_E_BADARG;
  if (d->sup_wt != 0.f && d->hm > 0 && (!mid_sup || !g_sup)) return B200SEG_E_BADARG;
  if (d->loss_kind != 0 && d->loss_kind != 1) return B200SEG_E_BADARG;
  if (n_rmi_terms > 0 && !rmi_terms) return B200SEG_E_BADARG;
  const int nb = b200seg_mscale_loss_blocks(d);
  const int Hp = d->h / 4 + 1, Wp = d->w / 4 + 1;     // avg_pool2d(kernel 4, stride 4, padding 2) output size
  launch_k(loss_fwd_kernel, dim3(nb), dim3(128), 0, (cudaStream_t)stream, to_geom(d), (const long long*)labels,
           inv_count, hi_cls, hi_aux, mid, mid_sup, (__nv_bfloat16*)g_hi, (__nv_bfloat16*)g_lo, (__nv_bfloat16*)g_sup,
           partial_ws, rmi_dpr, Hp, Wp);
  launch_k(loss_finalize_kernel, dim3(1), dim3(32), 0, (cudaStream_t)stream, partial_ws, nb, inv_count,
           d->loss_kind == 1 ? d->w_head0 * kRmiLambda : d->w_head0, d->nheads > 1 ? d->w_head1 : 0.f, d->sup_wt,
           loss_out, rmi_terms, (int)n_rmi_terms);
  RET_LAUNCH();
}

extern "C" int b200seg_mscale_hi_bwd(const b200seg_mscale_desc* d, const void* g_hi, void* d_cls, void* d_aux,
                                     void* stream) {
  if (!d || !g_hi || !d_cls || (d->nheads > 1 && !d_aux)) return B200SEG_E_BADARG;
  launch_k(hi_bwd_kernel, dim3(blocks_for((long long)d->n * d->hq * d->wq * d->nheads, 128)), dim3(128), 0,
           (cudaStream_t)stream, to_geom(d), (const __nv_bfloat16*)g_hi, (__nv_bfloat16*)d_cls,
           (__nv_bfloat16*)d_aux);
  RET_LAUNCH();
}

extern "C" int b200seg_mscale_lo_bwd(const b200seg_mscale_desc* d, const void* g_lo, const void* g_sup,
                                     const float* lo_cls, const float* lo_aux, const float* lo_attn_logit,
                                     const float* mid, float* dmid_ws, void* d_cls, void* d_aux, void* d_attn,
                                     void* stream) {
  if (!d || !g_lo || !lo_cls || !lo_attn_logit || !mid || !dmid_ws || !d_cls || !d_attn || d->hm <= 0)
    return B200SEG_E_BADARG;
  const MsGeom g = to_geom(d);
  launch_k(mid_bwd_kernel, dim3(blocks_for((long long)d->n * d->hm * d->wm, 128)), dim3(128), 0, (cudaStream_t)stream,
           g, (const __nv_bfloat16*)g_lo, d->sup_wt != 0.f ? (const __nv_bfloat16*)g_sup : nullptr, lo_cls, lo_aux,
           mid, dmid_ws);
  launch_k(lo_bwd_kernel, dim3(blocks_for((long long)d->n * d->hl * d->wl, 128)), dim3(128), 0, (cudaStream_t)stream,
           g, dmid_ws, lo_attn_logit, (__nv_bfloat16*)d_cls, (__nv_bfloat16*)d_aux, (__nv_bfloat16*)d_attn);
  RET_LAUNCH();
}
