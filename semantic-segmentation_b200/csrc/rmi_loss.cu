// Region Mutual Information loss head (loss/rmi.py:70-215, loss/rmi_utils.py:15-56,95-107) on the blended class logits,
// forward and backward, without materialising a full-resolution probability tensor or the fp64 [N,19,9,130305] stacks.
//
// Reference semantics (RMILoss.forward_sigmoid + rmi_lower_bound; radius 3, avg-pool 4/4/pad 2, _IS_SUM, lambda 0.5):
//   probs = sigmoid(logits) * mask + 1e-6 ; la = avg_pool(onehot*mask), pr = avg_pool(probs)            [n,19,H/4+1,W/4+1]
//   la_v, pr_v = the nine shifted (H/4-1) x (W/4-1) views of la / pr, flattened over positions, mean-centred   (fp64)
//   appro = la_cov - la_pr (pr_cov + aI)^-1 la_pr^T ; rmi[n,c] = sum log diag chol(appro + aI) ; a = 5e-4
//   loss_rmi = sum_c mean_n rmi[n,c] / 9 ; criterion = 0.5 * BCE + 0.5 * loss_rmi
//
// Kernels:
//   rmi_pool     one thread per pooling cell: blends the 16 full-resolution logits of the cell from the quarter-resolution
//                maps (same arithmetic as the loss kernel), accumulates sigmoid probabilities and label counts
//   rmi_moments  per (image, class, position chunk): the 18 x 18 second-moment matrix of [la_v ; pr_v] and the 18 sums in
//                fp64 (thread = one matrix row, 14 positions in flight per block, fixed-order folds -> deterministic)
//   rmi_solve    per (image, class): covariances, the two 9x9 Cholesky factorisations / inverses in fp64, the RMI value
//                and the closed-form gradient of it w.r.t. every position vector:  d rmi / d pr_v(pos) = G1 pr_v + G2 la_v
//                with  Bbar = 1/2 (appro+aI)^-1,  T = la_pr (pr_cov+aI)^-1,  G1 = 2 T^T Bbar T,  G2 = -2 (Bbar T)^T
//   rmi_grad     adjoint of the nine-view gather in fp64: gradient w.r.t. the pooled probabilities, consumed by loss_fwd_kernel
//                (which applies the avg-pool adjoint 1/16 and sigmoid' per full-resolution pixel).
#include "mscale_common.cuh"
#include "launch.h"

namespace b200seg {

constexpr int kHalf = 9;             // radius * radius
constexpr int kV = 18;               // [la_v ; pr_v]
constexpr int kGroups = 14;          // positions in flight per block (14 * 18 = 252 threads)
constexpr int kChunks = 48;          // position chunks per (image, class)
constexpr int kGPitch = 180;         // doubles per (image, class) gradient record: G1[81] G2[81] mu_la[9] mu_pr[9]
constexpr float kClipMin = 1e-6f;
constexpr double kPosAlpha = 5e-4;

// kHead 0: the main prediction (pr_pool and la_pool); kHead 1: the auxiliary prediction under cfg.LOSS.OCR_AUX_RMI
// (pr_pool only: the label pool is the same for both heads).
template <int kHead>
__global__ void __launch_bounds__(128)
rmi_pool_kernel(const MsGeom g, const long long* __restrict__ labels, const float* __restrict__ hi_cls,
                const float* __restrict__ M, float* __restrict__ pr_pool, float* __restrict__ la_pool, int Hp, int Wp) {
  pdl_sync();
  const long long total = (long long)g.N * Hp * Wp;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(idx % Wp), i = (int)((idx / Wp) % Hp), n = (int)(idx / ((long long)Wp * Hp));
    float ap[NC], al[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) { ap[c] = 0.f; al[c] = 0.f; }
    for (int dy = 0; dy < 4; ++dy) {
      const int Y = 4 * i - 2 + dy;
      if (Y < 0 || Y >= g.H) continue;                 // zero padding (count_include_pad: the divisor stays 16)
      for (int dx = 0; dx < 4; ++dx) {
        const int X = 4 * j - 2 + dx;
        if (X < 0 || X >= g.W) continue;
        const long long lab = labels[((long long)n * g.H + Y) * g.W + X];
        const bool valid = lab != (long long)g.ignore_index && lab >= 0 && lab < NC;
        float J[NC];
        joint_head<kHead>(g, n, Y, X, hi_cls, M, J);
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          ap[c] += (valid ? sigmoidf_(J[c]) : 0.f) + kClipMin;
          if (kHead == 0) al[c] += (valid && (int)lab == c) ? 1.f : 0.f;
        }
      }
    }
    float* po = pr_pool + idx * LD;
#pragma unroll
    for (int c = 0; c < NC; ++c) po[c] = ap[c] * 0.0625f;
    po[NC] = 0.f;
    if (kHead == 0) {
      float* lo = la_pool + idx * LD;
#pragma unroll
      for (int c = 0; c < NC; ++c) lo[c] = al[c] * 0.0625f;
      lo[NC] = 0.f;
    }
  }
}

// partial[((n*19 + c) * kChunks + chunk)][18][19]: row i = sum over the chunk's positions of v_i * [v_0..v_17, 1]
__global__ void __launch_bounds__(256)
rmi_moments_kernel(const float* __restrict__ pr_pool, const float* __restrict__ la_pool, int Hp, int Wp,
                   double* __restrict__ partial) {
  pdl_sync();
  extern __shared__ double sh_m[];    // [kGroups][kV][kV + 1]
  const int chunk = blockIdx.x, c = blockIdx.y, n = blockIdx.z;
  const int nh = Hp - 2, nw = Wp - 2;
  const int Mpos = nh * nw;
  const int p0 = (int)((long long)Mpos * chunk / kChunks), p1 = (int)((long long)Mpos * (chunk + 1) / kChunks);
  const int i = threadIdx.x % kV, grp = threadIdx.x / kV;
  double acc[kV + 1];
#pragma unroll
  for (int k = 0; k <= kV; ++k) acc[k] = 0.0;
  if (grp < kGroups) {
    const float* mine = (i < kHalf ? la_pool : pr_pool);
    const int ti = i < kHalf ? i : i - kHalf;
    const int oy = ti / 3, ox = ti - oy * 3;
    for (int pos = p0 + grp; pos < p1; pos += kGroups) {
      const int py = pos / nw, px = pos - py * nw;
      const size_t base = (((size_t)n * Hp + py) * Wp + px) * LD + c;
      const double vi = (double)mine[base + ((size_t)oy * Wp + ox) * LD];
#pragma unroll
      for (int t = 0; t < kHalf; ++t) {
        const size_t o = base + ((size_t)(t / 3) * Wp + (t % 3)) * LD;
        acc[t] += vi * (double)la_pool[o];
        acc[kHalf + t] += vi * (double)pr_pool[o];
      }
      acc[kV] += vi;
    }
    double* dst = sh_m + ((size_t)grp * kV + i) * (kV + 1);
#pragma unroll
    for (int k = 0; k <= kV; ++k) dst[k] = acc[k];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < kV * (kV + 1); e += blockDim.x) {
    double s = 0.0;
    for (int gq = 0; gq < kGroups; ++gq) s += sh_m[(size_t)gq * kV * (kV + 1) + e];
    partial[((size_t)(n * NC + c) * kChunks + chunk) * kV * (kV + 1) + e] = s;
  }
}

// 9x9 lower Cholesky factor and its inverse (single thread, fp64)
__device__ void chol_inv9(const double* A, double* L, double* Li) {
  for (int j = 0; j < kHalf; ++j) {
    double d = A[j * kHalf + j];
    for (int k = 0; k < j; ++k) d -= L[j * kHalf + k] * L[j * kHalf + k];
    d = sqrt(d);
    L[j * kHalf + j] = d;
    for (int i = j + 1; i < kHalf; ++i) {
      double s = A[i * kHalf + j];
      for (int k = 0; k < j; ++k) s -= L[i * kHalf + k] * L[j * kHalf + k];
      L[i * kHalf + j] = s / d;
    }
    for (int i = 0; i < j; ++i) L[i * kHalf + j] = 0.0;
  }
  for (int j = 0; j < kHalf; ++j) {          // forward substitution column by column: L * Li = I
    for (int i = 0; i < kHalf; ++i) {
      if (i < j) { Li[i * kHalf + j] = 0.0; continue; }
      double s = (i == j) ? 1.0 : 0.0;
      for (int k = j; k < i; ++k) s -= L[i * kHalf + k] * Li[k * kHalf + j];
      Li[i * kHalf + j] = s / L[i * kHalf + i];
    }
  }
}

// grid (19, N), 96 threads. scale = w_head0 * (1 - lambda) / (N * 9): d loss / d rmi[n,c].
__global__ void __launch_bounds__(96)
rmi_solve_kernel(const double* __restrict__ partial, int Hp, int Wp, float scale, double* __restrict__ G,
                 float* __restrict__ rmi_terms) {
  pdl_sync();
  __shared__ double S[kV][kV + 1], mu[kV];
  __shared__ double ll[81], lp[81], A[81], L[81], Li[81], Ainv[81], T[81], B[81], Bbar[81], U[81], Abar[81];
  __shared__ double rmi_val;
  const int c = blockIdx.x, n = blockIdx.y, tid = threadIdx.x;
  const double Mpos = (double)(Hp - 2) * (double)(Wp - 2);
  for (int e = tid; e < kV * (kV + 1); e += blockDim.x) {
    double s = 0.0;
    const double* src = partial + (size_t)(n * NC + c) * kChunks * kV * (kV + 1) + e;
    for (int ch = 0; ch < kChunks; ++ch) s += src[(size_t)ch * kV * (kV + 1)];
    S[e / (kV + 1)][e % (kV + 1)] = s;
  }
  __syncthreads();
  if (tid < kV) mu[tid] = S[tid][kV] / Mpos;
  __syncthreads();
  const int r = tid / kHalf, q = tid % kHalf;
  const bool m81 = tid < 81;
  if (m81) {
    ll[tid] = S[r][q] - Mpos * mu[r] * mu[q];
    lp[tid] = S[r][kHalf + q] - Mpos * mu[r] * mu[kHalf + q];
    A[tid] = S[kHalf + r][kHalf + q] - Mpos * mu[kHalf + r] * mu[kHalf + q] + (r == q ? kPosAlpha : 0.0);
  }
  __syncthreads();
  if (tid == 0) chol_inv9(A, L, Li);
  __syncthreads();
  if (m81) { double s = 0.0; for (int k = 0; k < kHalf; ++k) s += Li[k * kHalf + r] * Li[k * kHalf + q]; Ainv[tid] = s; }
  __syncthreads();
  if (m81) { double s = 0.0; for (int k = 0; k < kHalf; ++k) s += lp[r * kHalf + k] * Ainv[k * kHalf + q]; T[tid] = s; }
  __syncthreads();
  if (m81) {
    double s = ll[tid] + (r == q ? kPosAlpha : 0.0);
    for (int k = 0; k < kHalf; ++k) s -= T[r * kHalf + k] * lp[q * kHalf + k];
    B[tid] = s;
  }
  __syncthreads();
  if (tid == 0) {
    chol_inv9(B, L, Li);
    double v = 0.0;
    for (int k = 0; k < kHalf; ++k) v += log(L[k * kHalf + k] + 1e-8);
    rmi_val = v;
  }
  __syncthreads();
  if (m81) { double s = 0.0; for (int k = 0; k < kHalf; ++k) s += Li[k * kHalf + r] * Li[k * kHalf + q]; Bbar[tid] = 0.5 * s; }
  __syncthreads();
  if (m81) { double s = 0.0; for (int k = 0; k < kHalf; ++k) s += Bbar[r * kHalf + k] * T[k * kHalf + q]; U[tid] = s; }
  __syncthreads();
  if (m81) { double s = 0.0; for (int k = 0; k < kHalf; ++k) s += T[k * kHalf + r] * U[k * kHalf + q]; Abar[tid] = s; }
  __syncthreads();
  // The gradient is a difference of large terms (entries of G ~ 1/alpha): it stays in fp64 and rmi_grad applies it to
  // the CENTRED position vectors (an fp32  G1 pr + G2 la + g0  loses every significant digit).
  double* out = G + (size_t)(n * NC + c) * kGPitch;
  if (m81) {
    out[tid] = 2.0 * Abar[tid] * (double)scale;                     // G1[t][j], t = r, j = q
    out[81 + tid] = -2.0 * U[q * kHalf + r] * (double)scale;        // G2[t][j] = Cbar[j][t]
  }
  if (tid < kV) out[162 + tid] = mu[tid];
  if (tid == 0) rmi_terms[n * NC + c] = (float)(rmi_val * (double)scale);
}

// dpr[n][i][j][c] = sum over the (<= 9) positions whose 3x3 view contains cell (i, j) as tap t of
//                   sum_t' G1[t][t'] (pr(pos + t') - mu_pr[t']) + G2[t][t'] (la(pos + t') - mu_la[t'])        (fp64)
__global__ void __launch_bounds__(256)
rmi_grad_kernel(const float* __restrict__ pr_pool, const float* __restrict__ la_pool, const double* __restrict__ G,
                int Hp, int Wp, float* __restrict__ dpr) {
  pdl_sync();
  extern __shared__ double sG[];     // [19][kGPitch]
  const int n = blockIdx.y;
  for (int e = threadIdx.x; e < NC * kGPitch; e += blockDim.x) sG[e] = G[(size_t)n * NC * kGPitch + e];
  __syncthreads();
  const int nh = Hp - 2, nw = Wp - 2;
  const long long total = (long long)Hp * Wp * LD;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % LD);
    const long long cell = idx / LD;
    const int j = (int)(cell % Wp), i = (int)(cell / Wp);
    double acc = 0.0;
    if (c < NC) {
      const double* g1 = sG + c * kGPitch;
      const double* g2 = g1 + 81;
      const double* mul = g1 + 162;
      const double* mup = g1 + 171;
      for (int y = 0; y < 3; ++y) {
        const int py = i - y;
        if (py < 0 || py >= nh) continue;
        for (int x = 0; x < 3; ++x) {
          const int px = j - x;
          if (px < 0 || px >= nw) continue;
          const int t = y * 3 + x;
          const size_t base = (((size_t)n * Hp + py) * Wp + px) * LD + c;
#pragma unroll
          for (int tt = 0; tt < kHalf; ++tt) {
            const size_t o = base + ((size_t)(tt / 3) * Wp + (tt % 3)) * LD;
            acc += g1[t * kHalf + tt] * ((double)pr_pool[o] - mup[tt]) + g2[t * kHalf + tt] * ((double)la_pool[o] - mul[tt]);
          }
        }
      }
    }
    dpr[(size_t)n * Hp * Wp * LD + idx] = (float)acc;
  }
}

}  // namespace b200seg

using namespace b200seg;

extern "C" size_t b200seg_rmi_ws_bytes(int32_t n) {
  return (size_t)n * NC * kChunks * kV * (kV + 1) * sizeof(double);
}

extern "C" int b200seg_rmi_pool(const b200seg_mscale_desc* d, const int64_t* labels, const float* hi_cls, const float* mid,
                                float* pr_pool, float* la_pool, void* stream) {
  if (!d || !labels || !hi_cls || !pr_pool || !la_pool || (d->hm > 0 && !mid)) return B200SEG_E_BADARG;
  if (d->h < 12 || d->w < 12) return B200SEG_E_BADARG;     // at least one 3x3 view of pooled cells
  const int Hp = d->h / 4 + 1, Wp = d->w / 4 + 1;
  cudaError_t e = launch_k(rmi_pool_kernel<0>, dim3(blocks_for_total((long long)d->n * Hp * Wp, 128)), dim3(128), 0,
                           (cudaStream_t)stream, to_geom(d), (const long long*)labels, hi_cls, mid, pr_pool, la_pool,
                           Hp, Wp);
  return e == cudaSuccess ? 0 : (int)e;
}

extern "C" int b200seg_rmi_pool_aux(const b200seg_mscale_desc* d, const int64_t* labels, const float* hi_aux,
                                    const float* mid, float* pr_pool, void* stream) {
  if (!d || !labels || !hi_aux || !pr_pool || d->nheads < 2 || (d->hm > 0 && !mid)) return B200SEG_E_BADARG;
  if (d->h < 12 || d->w < 12) return B200SEG_E_BADARG;
  const int Hp = d->h / 4 + 1, Wp = d->w / 4 + 1;
  cudaError_t e = launch_k(rmi_pool_kernel<1>, dim3(blocks_for_total((long long)d->n * Hp * Wp, 128)), dim3(128), 0,
                           (cudaStream_t)stream, to_geom(d), (const long long*)labels, hi_aux, mid, pr_pool,
                           (float*)nullptr, Hp, Wp);
  return e == cudaSuccess ? 0 : (int)e;
}

/* moments -> solve -> gradient w.r.t. the pooled probabilities. scale = w_head0 * (1 - lambda) / (n * 9). */
extern "C" int b200seg_rmi_solve_grad(int32_t n, int32_t h, int32_t w, const float* pr_pool, const float* la_pool,
                                      float scale, void* ws, size_t ws_bytes, double* G, float* rmi_terms, float* dpr,
                                      void* stream) {
  if (n <= 0 || !pr_pool || !la_pool || !ws || !G || !rmi_terms || !dpr) return B200SEG_E_BADARG;
  if (ws_bytes < b200seg_rmi_ws_bytes(n) || (reinterpret_cast<uintptr_t>(ws) & 7) ||
      (reinterpret_cast<uintptr_t>(G) & 7))
    return B200SEG_E_BADARG;
  const int Hp = h / 4 + 1, Wp = w / 4 + 1;
  if (Hp < 3 || Wp < 3) return B200SEG_E_BADARG;
  const size_t smem = (size_t)kGroups * kV * (kV + 1) * sizeof(double);
  cudaError_t e = launch_k(rmi_moments_kernel, dim3(kChunks, NC, n), dim3(256), smem, (cudaStream_t)stream, pr_pool,
                           la_pool, Hp, Wp, (double*)ws);
  if (e != cudaSuccess) return (int)e;
  e = launch_k(rmi_solve_kernel, dim3(NC, n), dim3(96), 0, (cudaStream_t)stream, (const double*)ws, Hp, Wp, scale, G,
               rmi_terms);
  if (e != cudaSuccess) return (int)e;
  e = launch_k(rmi_grad_kernel, dim3(blocks_for_total((long long)Hp * Wp * LD, 256), n), dim3(256),
               (size_t)NC * kGPitch * sizeof(double), (cudaStream_t)stream, pr_pool, la_pool, (const double*)G, Hp,
               Wp, dpr);
  return e == cudaSuccess ? 0 : (int)e;
}
