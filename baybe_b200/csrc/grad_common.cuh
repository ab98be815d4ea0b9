// grad_common.cuh -- device code of the gradient kernels (k_acq_grad, k_objective_grad, k_acq_grad_large, ...).
//
// One warp per point, on the CUDA cores in fp32.  With a = x * scale + shift and b_i the scaled training rows
// (train_m2 = -2 b):
//   k_i = s_f^2 kappa(|a - b_i|^2),  gk_i = 2 s_f^2 dkappa/dt,  v = L^-1 k,  u = L^-T v
// and the partial derivatives of the acquisition value with respect to mu, var and the pending cross covariances c_p
// go back through k_i with
//   dA/dk_i = s_y A_mu alpha_i - 2 s_y^2 A_var u_i - s_y^2 sum_p A_c[p] beta_p,i,   da/dx = scale.
#pragma once

#include <math.h>

#include "acq_math.cuh"
#include "common.cuh"

namespace bb {

constexpr int kGradMaxNPad = 256;
constexpr unsigned kFull = 0xffffffffu;

// kernel value k(t) and dk/dt of the scaled squared distance t (the family's constant is folded into the scale)
template <int FAMILY>
__device__ __forceinline__ void kernel_and_slope(float t, float& k, float& dkdt) {
  t = fmaxf(t, 0.f);
  if constexpr (FAMILY == BB_KERNEL_RBF) {
    k = exp2f(-t);
    dkdt = -kLn2 * k;
  } else {
    const float s = sqrtf(t), e = expf(-s);
    if constexpr (FAMILY == BB_KERNEL_MATERN12) {
      k = e;
      dkdt = s > 0.f ? -0.5f * e / s : 0.f;  // kappa'(r)/r taken as 0 at r = 0
    } else if constexpr (FAMILY == BB_KERNEL_MATERN32) {
      k = (1.f + s) * e;
      dkdt = -0.5f * e;
    } else {
      k = (1.f + s + t * (1.f / 3.f)) * e;
      dkdt = -(1.f + s) * e * (1.f / 6.f);
    }
  }
}

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

__device__ __forceinline__ float sigmoidf_(float t) { return 1.f / (1.f + expf(-t)); }

// sigmoid'(t) = e / (1 + e)^2, e = exp(-t): no cancellation in 1 - sigmoid(t) where sigmoid(t) is near 1
__device__ __forceinline__ float dsigmoidf_(float t) {
  const float e = expf(-t);
  return isinf(e) ? 0.f : e / ((1.f + e) * (1.f + e));
}

// d/dt log(softplus(t) + 0.1 / (1 + t^2)) and the value inside the log
__device__ __forceinline__ float dlog_fatplus_t(float t) {
  const float q = 1.f / fmaf(t, t, 1.f);
  const float sp = fmaxf(t, 0.f) + ((fabsf(t) < 30.f) ? log1pf(expf(-fabsf(t))) : 0.f);
  return (sigmoidf_(t) - 0.2f * (t * q) * q) / (sp + 0.1f * q);
}

// partial derivatives (A_mu, A_sd) of the analytic kinds, float64
__device__ __forceinline__ void analytic_partials(const bb_acq_spec& a, float mu, float var, double& dmu,
                                                  double& dsd) {
  const double a1 = (double)a.obj_scale, aa = fabs(a1);
  const double m = a1 * (double)mu + (double)a.obj_shift;
  const double s = aa * sqrt((double)var);
  dmu = 0.0;
  dsd = 0.0;
  switch (a.kind) {
    case BB_ACQ_PM: dmu = a1; return;
    case BB_ACQ_PSTD: dsd = a.maximize ? aa : -aa; return;
    case BB_ACQ_UCB: dmu = a1; dsd = sqrt((double)a.beta) * aa; return;
    default: break;
  }
  const double u = (m - (double)a.best_f) / s;
  if (a.kind == BB_ACQ_EI) {
    dmu = a1 * norm_cdf(u);
    dsd = aa * norm_pdf(u);
  } else if (a.kind == BB_ACQ_LOGEI) {
    // Phi(u) / h(u) = exp(log Phi(u) - log h(u)), h(u) = phi(u) + u Phi(u): never formed as a ratio
    const double log_Phi = u > -1.0 ? log(norm_cdf(u))
                                    : log(0.5 * erfcx(-u * 0.7071067811865476)) - 0.5 * u * u;
    const double r = exp(log_Phi - log_ei_helper(u));
    dmu = a1 * r / s;
    dsd = aa * (1.0 - u * r) / s;
  } else {  // PI
    dmu = a1 * norm_pdf(u) / s;
    dsd = -aa * u * norm_pdf(u) / s;
  }
}

// The kernel row of the point a (a_w: its d scaled coordinates): k_w[i] = k_i, gk_w[i] = gk_i (0 past n); returns
// this lane's part of k . alpha.
template <int FAMILY>
__device__ __forceinline__ float kernel_row_warp(const float* a_w, const float* train_m2, const float* alpha, int n,
                                                 int n_pad, int d, int d_pad, float sf2, float* k_w, float* gk_w,
                                                 int lane) {
  float ka = 0.f;
  for (int i = lane; i < n_pad; i += 32) {
    float t = 0.f;
    for (int j = 0; j < d; ++j) {
      const float df = a_w[j] + 0.5f * __ldg(train_m2 + (size_t)i * d_pad + j);
      t = fmaf(df, df, t);
    }
    float k, dk;
    kernel_and_slope<FAMILY>(t, k, dk);
    k = i < n ? sf2 * k : 0.f;
    k_w[i] = k;
    gk_w[i] = i < n ? 2.f * sf2 * dk : 0.f;
    ka = fmaf(k, __ldg(alpha + i), ka);
  }
  return ka;
}

// v = L^-1 k, 32 rows at a time: each lane takes every 32nd column of the 32 rows (coalesced loads of L^-1) and a
// reduce-scatter over the warp leaves row j0 + l in lane l.  Returns this lane's part of |v|^2.
__device__ __forceinline__ float linv_apply_warp(const float* linv, int n_pad, const float* k_w, float* v_w,
                                                 int lane) {
  float vv = 0.f;
  for (int j0 = 0; j0 < n_pad; j0 += 32) {
    float r[32];
#pragma unroll
    for (int q = 0; q < 32; ++q) r[q] = 0.f;
    for (int i0 = 0; i0 <= j0; i0 += 32) {
      const float ki = k_w[i0 + lane];
      const float* Lr = linv + (size_t)j0 * n_pad + i0 + lane;
#pragma unroll
      for (int q = 0; q < 32; ++q) r[q] = fmaf(__ldg(Lr + (size_t)q * n_pad), ki, r[q]);
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {  // reduce-scatter: lane l ends with row j0 + l
      const bool up = (lane & off) != 0;
#pragma unroll
      for (int q = 0; q < off; ++q) {
        const float send = up ? r[q] : r[q + off];
        const float keep = up ? r[q + off] : r[q];
        r[q] = keep + __shfl_xor_sync(kFull, send, off);
      }
    }
    v_w[j0 + lane] = r[0];
    vv = fmaf(r[0], r[0], vv);
  }
  return vv;
}

// u_i = (L^-T v)_i for column i of the 32-column block starting at i0 (lane l owns column i0 + l: no reduction)
__device__ __forceinline__ float linvt_apply_col(const float* linv, int n_pad, const float* v_w, int i0, int i) {
  float u = 0.f;
  for (int j = i0; j < n_pad; ++j) u = fmaf(__ldg(linv + (size_t)j * n_pad + i), v_w[j], u);
  return u;
}

// ---- one model per target with P pending points (k_objective_grad, k_hvi_grad) ------------------------------------
// A target's model as the multi-target gradient kernels read it.
struct GradTarget {
  const float *cand_scale, *cand_shift, *train_m2, *alpha, *linv, *mean_const;
  const float* pend_beta;  // [P][n_pad]
  int n, n_pad;
  float y_mean, y_std, sf2;
};

// A target's slice of a warp's scratch: a [d_pad] | k, gk, v [n_pad] | c, L^-1 c, gkp, A_c [32] (gkp: 2 s_f^2 dk/dt
// of k(x, x_p); A_c: dA/dc_p).
struct TargetScratch {
  float *a, *k, *gk, *v, *c, *r, *gkp, *ac;
};

// Forward pass of one target for the point x (its d raw coordinates), P pending points with rows pend_x [P][d] and
// L_PP^-1 plinv [P][P]: fills the scratch (A_c zeroed) and returns, in every lane, mu, var and
// sd = sqrt(max(var - |L^-1 c|^2, 0)); the return value says whether the variance clamp is inactive (it passes no
// gradient when it is).
template <int FAMILY>
__device__ __forceinline__ bool target_forward_warp(const GradTarget& md, const float* x, int d, int dp, int P,
                                                    const float* pend_x, const float* plinv, const TargetScratch& t,
                                                    float& mu, float& var, float& sd, int lane) {
  for (int j = lane; j < dp; j += 32)
    t.a[j] = j < d ? fmaf(__ldg(x + j), __ldg(md.cand_scale + j), __ldg(md.cand_shift + j)) : 0.f;
  __syncwarp();
  const float ka =
      warp_sum(kernel_row_warp<FAMILY>(t.a, md.train_m2, md.alpha, md.n, md.n_pad, d, dp, md.sf2, t.k, t.gk, lane));
  __syncwarp();
  const float vv = warp_sum(linv_apply_warp(md.linv, md.n_pad, t.k, t.v, lane));
  const float sy = md.y_std, sy2 = sy * sy;
  const float vt = md.sf2 - vv;
  mu = fmaf(sy, __ldg(md.mean_const) + ka, md.y_mean);
  var = sy2 * fmaxf(vt, 1e-10f);
  float cr = 0.f;  // lane q < P: c_q
  for (int q = 0; q < P; ++q) {
    float kb = 0.f;
    for (int i = lane; i < md.n_pad; i += 32) kb = fmaf(t.k[i], __ldg(md.pend_beta + (size_t)q * md.n_pad + i), kb);
    kb = warp_sum(kb);
    if (lane == q) cr = kb;
  }
  float g = 0.f;
  if (lane < P) {
    float tt = 0.f;
    for (int j = 0; j < d; ++j) {
      const float b = fmaf(__ldg(pend_x + (size_t)lane * d + j), __ldg(md.cand_scale + j), __ldg(md.cand_shift + j));
      const float df = t.a[j] - b;
      tt = fmaf(df, df, tt);
    }
    float k, dk;
    kernel_and_slope<FAMILY>(tt, k, dk);
    cr = sy2 * (md.sf2 * k - cr);
    g = 2.f * md.sf2 * dk;
  }
  t.c[lane] = lane < P ? cr : 0.f;
  t.gkp[lane] = g;
  t.ac[lane] = 0.f;
  // r = L^-1 c (lane i: r_i), as pending_r2_warp forms it
  float r = 0.f;
  for (int k = 0; k < P; ++k) {
    const float ck = __shfl_sync(kFull, cr, k);
    if (lane < P && k <= lane) r = fmaf(__ldg(plinv + lane * P + k), ck, r);
  }
  t.r[lane] = lane < P ? r : 0.f;
  const float r2 = warp_sum(lane < P ? r * r : 0.f);
  sd = P > 0 ? sqrtf(fmaxf(var - r2, 0.f)) : sqrtf(var);
  __syncwarp();
  return vt > 1e-10f;
}

// sd = sqrt(max(var - |r|^2, 0)), r = L^-1 c, with A_sd = dA/dsd summed over the warp: returns A_var = A_sd / (2 sd)
// and adds -A_sd L^-T r / sd to A_c (lanes < P).
__device__ __forceinline__ float target_sd_adjoint(float a_sd, float sd, int P, const float* plinv,
                                                   const TargetScratch& t, int lane) {
  const float f = sd > 0.f ? a_sd / sd : 0.f;
  if (lane < P) {
    float lt = 0.f;
    for (int i = lane; i < P; ++i) lt = fmaf(__ldg(plinv + i * P + lane), t.r[i], lt);
    t.ac[lane] = fmaf(-f, lt, t.ac[lane]);
  }
  return 0.5f * f;
}

// Reverse pass through the kernel row: k_i <- gk_i dA/dk_i with
// dA/dk_i = s_y A_mu alpha_i - 2 s_y^2 A_var u_i - s_y^2 sum_p A_c[p] beta_p,i (lanes over columns).
__device__ __forceinline__ void target_row_adjoint(const GradTarget& md, float a_mu, float a_var, int P,
                                                   const TargetScratch& t, int lane) {
  const float sy = md.y_std, sy2 = sy * sy;
  const float k_mu = sy * a_mu, k_var = -2.f * sy2 * a_var;
  for (int i0 = 0; i0 < md.n_pad; i0 += 32) {
    const int i = i0 + lane;
    const float u = linvt_apply_col(md.linv, md.n_pad, t.v, i0, i);
    float kb = fmaf(k_mu, __ldg(md.alpha + i), k_var * u);
    for (int q = 0; q < P; ++q) kb = fmaf(-sy2 * t.ac[q], __ldg(md.pend_beta + (size_t)q * md.n_pad + i), kb);
    t.k[i] = t.gk[i] * kb;
  }
}

// dA/da_j of one target after target_row_adjoint: the training rows' terms and the direct k(x, x_p) term (multiply
// by cand_scale[j] for dA/dx_j).
__device__ __forceinline__ float target_col_grad(const GradTarget& md, int j, int d, int dp, int P,
                                                 const float* pend_x, const TargetScratch& t) {
  const float sy2 = md.y_std * md.y_std;
  const float aj = t.a[j];
  float g = 0.f;
  for (int i = 0; i < md.n; ++i) g = fmaf(t.k[i], aj + 0.5f * __ldg(md.train_m2 + (size_t)i * dp + j), g);
  for (int q = 0; q < P; ++q) {
    const float b = fmaf(__ldg(pend_x + (size_t)q * d + j), __ldg(md.cand_scale + j), __ldg(md.cand_shift + j));
    g = fmaf(sy2 * t.ac[q] * t.gkp[q], aj - b, g);
  }
  return g;
}

// Floats of one warp's scratch for M targets: M TargetScratch slices, the sample chunk's adjoints [32][M] and 32
// per-target scalars (mu | var | sd | A_var, 8 each).
__host__ __device__ inline int target_warp_floats(int M, int n_pad, int d_pad) {
  return (M * (d_pad + 3 * n_pad + 4 * 32) + 32 * M + 32 + 3) & ~3;
}

// Target m's slice of the scratch that starts at wb, laid out as k_objective_grad lays it out.
__device__ __forceinline__ TargetScratch target_scratch(float* wb, int M, int m, int np, int dp) {
  TargetScratch t;
  t.a = wb + m * dp;
  t.k = wb + M * dp + m * np;
  t.gk = wb + M * (dp + np) + m * np;
  t.v = wb + M * (dp + 2 * np) + m * np;
  float* c0 = wb + M * (dp + 3 * np);
  t.c = c0 + m * 32;
  t.r = c0 + M * 32 + m * 32;
  t.gkp = c0 + 2 * M * 32 + m * 32;
  t.ac = c0 + 3 * M * 32 + m * 32;
  return t;
}

// ---- one CTA of 256 threads per point (k_acq_grad_large in gradlarge.cu, k_objective_grad_large in objgradlarge.cu) -
// Each piece is one model's; the caller synchronises the CTA between them.  Every per-element sum runs in the order of
// the warp-per-point pieces above (kernel_row_warp, linv_apply_warp, linvt_apply_col), so on the shapes both mappings
// take (d < 32) v, u and the pending products agree bit for bit.
constexpr int kCtaThreads = 256;
constexpr int kCtaWarps = kCtaThreads / 32;

// block b of nb in snake order over the warps: round r gives warp w block r W + w (r even) or r W + W - 1 - w (r odd)
__device__ __forceinline__ int snake_block(int r, int warp) {
  return r * kCtaWarps + ((r & 1) ? kCtaWarps - 1 - warp : warp);
}

// The kernel row of the point a (a_w: its d scaled coordinates): k_w[i] = k_i, gk_w[i] = gk_i (0 past n).  A thread per
// training row for d < 32, a warp per row (lanes over columns) from d = 32 on, so that wide rows are read coalesced.
template <int FAMILY>
__device__ __forceinline__ void kernel_row_cta(const float* a_w, const float* train_m2, int n, int n_pad, int d,
                                               int d_pad, float sf2, float* k_w, float* gk_w) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (d < 32) {
    for (int i = threadIdx.x; i < n_pad; i += blockDim.x) {
      float t = 0.f;
      for (int j = 0; j < d; ++j) {
        const float df = a_w[j] + 0.5f * __ldg(train_m2 + (size_t)i * d_pad + j);
        t = fmaf(df, df, t);
      }
      float k, dk;
      kernel_and_slope<FAMILY>(t, k, dk);
      k_w[i] = i < n ? sf2 * k : 0.f;
      gk_w[i] = i < n ? 2.f * sf2 * dk : 0.f;
    }
  } else {
    for (int i = warp; i < n_pad; i += kCtaWarps) {
      float t = 0.f;
      if (i < n)
        for (int j = lane; j < d; j += 32) {
          const float df = a_w[j] + 0.5f * __ldg(train_m2 + (size_t)i * d_pad + j);
          t = fmaf(df, df, t);
        }
      t = warp_sum(t);
      float k, dk;
      kernel_and_slope<FAMILY>(t, k, dk);
      if (lane == 0) {
        k_w[i] = i < n ? sf2 * k : 0.f;
        gk_w[i] = i < n ? 2.f * sf2 * dk : 0.f;
      }
    }
  }
}

// v = L^-1 k: the warps take the 32-row blocks of the lower triangle in snake order, so that each reads about the same
// share of it; each block as linv_apply_warp forms it.  The same pass forms kb_s[q] = k . beta_q of the P pending
// points (warp q mod 8).
__device__ __forceinline__ void linv_apply_cta(const float* linv, int n_pad, const float* k_w, float* v_w, int P,
                                               const float* pend_beta, float* kb_s) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nb = n_pad >> 5;
  const int rounds = (nb + kCtaWarps - 1) / kCtaWarps;
  for (int r = 0; r < rounds; ++r) {
    const int jb = snake_block(r, warp);
    if (jb >= nb) continue;
    const int j0 = jb << 5;
    float rr[32];
#pragma unroll
    for (int q = 0; q < 32; ++q) rr[q] = 0.f;
    for (int i0 = 0; i0 <= j0; i0 += 32) {
      const float ki = k_w[i0 + lane];
      const float* Lr = linv + (size_t)j0 * n_pad + i0 + lane;
#pragma unroll
      for (int q = 0; q < 32; ++q) rr[q] = fmaf(__ldg(Lr + (size_t)q * n_pad), ki, rr[q]);
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {  // reduce-scatter: lane l ends with row j0 + l
      const bool up = (lane & off) != 0;
#pragma unroll
      for (int q = 0; q < off; ++q) {
        const float send = up ? rr[q] : rr[q + off];
        const float keep = up ? rr[q + off] : rr[q];
        rr[q] = keep + __shfl_xor_sync(kFull, send, off);
      }
    }
    v_w[j0 + lane] = rr[0];
  }
  for (int q = warp; q < P; q += kCtaWarps) {
    float kb = 0.f;
    for (int i = lane; i < n_pad; i += 32) kb = fmaf(k_w[i], __ldg(pend_beta + (size_t)q * n_pad + i), kb);
    kb = warp_sum(kb);
    if (lane == 0) kb_s[q] = kb;
  }
}

// u = L^-T v over the 32-column blocks in snake order (lane l owns column i0 + l, no reduction), folded with the slope
// into the kernel row: k_w[i] = gk_i dA/dk_i, dA/dk_i = k_mu alpha_i + k_var u_i - sum_q acs[q] beta_q,i (k_mu = s_y
// A_mu, k_var = -2 s_y^2 A_var, acs[q] = s_y^2 A_c[q]).
__device__ __forceinline__ void linvt_fold_cta(const float* linv, const float* alpha, int n_pad, const float* v_w,
                                               const float* gk_w, float k_mu, float k_var, int P,
                                               const float* pend_beta, const float* acs, float* k_w) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nb = n_pad >> 5;
  const int rounds = (nb + kCtaWarps - 1) / kCtaWarps;
  for (int r = 0; r < rounds; ++r) {
    const int ib = snake_block(r, warp);
    if (ib >= nb) continue;
    const int i0 = ib << 5, i = i0 + lane;
    float u = 0.f;
    for (int j = i0; j < n_pad; ++j) u = fmaf(__ldg(linv + (size_t)j * n_pad + i), v_w[j], u);
    float kb = fmaf(k_mu, __ldg(alpha + i), k_var * u);
    for (int q = 0; q < P; ++q) kb = fmaf(-acs[q], __ldg(pend_beta + (size_t)q * n_pad + i), kb);
    k_w[i] = gk_w[i] * kb;
  }
}

// Reverse pass through the folded kernel row, first half: with G = 256 / d row groups of d threads (d < 256), group g
// sums the rows i = g mod G of column j into part[g d + j].  Every thread of the CTA calls it (it synchronises).
__device__ __forceinline__ void row_groups_cta(const float* k_w, const float* a_w, const float* train_m2, int n, int d,
                                               int d_pad, float* part) {
  const int G = d < kCtaThreads ? kCtaThreads / d : 1;
  if (G > 1) {
    const int j = threadIdx.x % d, g = threadIdx.x / d;
    if (g < G) {
      const float aj = a_w[j];
      float acc = 0.f;
      for (int i = g; i < n; i += G) acc = fmaf(k_w[i], aj + 0.5f * __ldg(train_m2 + (size_t)i * d_pad + j), acc);
      part[g * d + j] = acc;
    }
    __syncthreads();
  }
}

// Second half: dA/da_j, the row groups summed in order (or the rows in order, one thread per column, for d >= 256),
// plus the direct terms acs[q] gkp[q] (a_j - b_qj) of k(x, x_p).  Multiply by cand_scale[j] for dA/dx_j.
__device__ __forceinline__ float col_grad_cta(int j, const float* k_w, const float* a_w, const float* train_m2, int n,
                                              int d, int d_pad, const float* part, int P, const float* pend_x,
                                              const float* cand_scale, const float* cand_shift, const float* acs,
                                              const float* gkp) {
  const int G = d < kCtaThreads ? kCtaThreads / d : 1;
  const float aj = a_w[j];
  float g = 0.f;
  if (G > 1) {
    for (int r = 0; r < G; ++r) g += part[r * d + j];
  } else {
    for (int i = 0; i < n; ++i) g = fmaf(k_w[i], aj + 0.5f * __ldg(train_m2 + (size_t)i * d_pad + j), g);
  }
  for (int q = 0; q < P; ++q) {
    const float b = fmaf(__ldg(pend_x + (size_t)q * d + j), __ldg(cand_scale + j), __ldg(cand_shift + j));
    g = fmaf(acs[q] * gkp[q], aj - b, g);
  }
  return g;
}

// ---- single-target value and partials at one point (k_acq_grad in grad.cu, k_acq_grad_large in gradlarge.cu) ------

// Column means of the base samples z [S][zs] (lane k < 1 + P: column k) and, for P = 0, the mean of column 0 in every
// lane and mean |z - mean z| (zdev).
__device__ __forceinline__ void sample_means_warp(const float* z, int zs, int S, int P, float& zb, float& zdev,
                                                  int lane) {
  zb = 0.f;
  zdev = 0.f;
  if (lane < P + 1) {
    for (int s = 0; s < S; ++s) zb += z[s * zs + lane];
    zb /= (float)S;
  }
  if (P == 0) {
    float sz = 0.f;
    for (int s = lane; s < S; s += 32) sz += z[s * zs];
    const float zm = warp_sum(sz) / (float)S;
    float sa = 0.f;
    for (int s = lane; s < S; s += 32) sa += fabsf(z[s * zs] - zm);
    zdev = warp_sum(sa) / (float)S;
    zb = zm;  // same value in every lane
  }
}

// One warp's scratch for acq_point_partials: lv, mP, moP, A_c [32] | L22, dA/dL22 [P][P] | two [32][1 + P] sample
// chunks.
struct AcqScratch {
  float *lv, *mP, *moP, *ac, *Lw, *Lb, *Wc, *Wm;
};

__host__ __device__ inline int acq_scratch_floats(int P) { return 4 * 32 + 2 * P * P + 2 * 32 * (P + 1); }

__device__ __forceinline__ AcqScratch acq_scratch(float* w, int P) {
  AcqScratch s;
  s.lv = w;
  s.mP = w + 32;
  s.moP = w + 64;
  s.ac = w + 96;
  s.Lw = w + 128;
  s.Lb = s.Lw + P * P;
  s.Wc = s.Lb + P * P;
  s.Wm = s.Wc + 32 * (P + 1);
  return s;
}

// The acquisition value at one point from its moments mu, var and (lane q < P) cross covariances c_q with the P
// pending points, and its partial derivatives A_mu (g_mu), A_var (g_var, before the variance clamp) and A_c (w.ac,
// lanes < P).  Analytic kinds (S = 0): the closed forms in float64.  Monte Carlo kinds with base samples z [S][zs],
// zb / zdev from sample_means_warp: without pending points the sums of k_fused's epilogue; with them k_acq_joint's
// value (Cholesky of [[var, c^T], [c, Sigma_PP]], candidate first, with its jitter escalation) and the reverse pass
// through that Cholesky, dA/dA22 = sym(L22^-T Phi(L22^T dL22) L22^-1) / 2 (as torch's cholesky backward).  Every lane
// returns the same value, g_mu and g_var; a failed factorisation gives a NaN value and zero partials.
__device__ __forceinline__ void acq_point_partials(const bb_acq_spec& a, float mu, float var, float cr, int P,
                                                   const float* pend_mu, const float* pend_cov, const float* z, int zs,
                                                   int S, float zb, float zdev, const AcqScratch& w, float& value,
                                                   float& g_mu, float& g_var, int lane) {
  const int Q = P + 1;
  const bool is_mc = a.kind <= BB_ACQ_QPI;
  const float a1 = a.obj_scale, a0 = a.obj_shift;
  const float ucb_c = sqrtf(a.beta * 1.5707963267948966f);
  g_mu = 0.f;
  g_var = 0.f;
  if (!is_mc) {
    value = analytic_value(a, mu, var);
    double dmu, dsd;
    analytic_partials(a, mu, var, dmu, dsd);
    g_mu = (float)dmu;
    g_var = (float)(dsd / (2.0 * sqrt((double)var)));
  } else if (P == 0) {
    float c0, c1;
    mc_coef(a, mu, var, c0, c1);
    const float sd = sqrtf(var);
    float s0 = 0.f, s1 = 0.f, h0 = 0.f, h1 = 0.f;  // value sums; sums of d(term)/dt and d(term)/dt * z
    for (int s = lane; s < S; s += 32) {
      const float zz = z[s * zs], t = fmaf(c1, zz, c0);
      float g = 0.f;
      if (a.kind == BB_ACQ_QLOGEI) {
        const float q = 1.f / fmaf(t, t, 1.f);
        s0 += fmaxf(t, 0.f) + ((fabsf(t) < 30.f) ? log1pf(expf(-fabsf(t))) : 0.f);
        s1 += q;
        g = sigmoidf_(t) - 0.2f * (t * q) * q;
      } else if (a.kind == BB_ACQ_QEI) {
        s0 += fmaxf(t, 0.f);
        g = t > 0.f ? 1.f : 0.f;
      } else if (a.kind == BB_ACQ_QPI) {
        s0 += sigmoidf_(t);
        g = dsigmoidf_(t);
      }
      h0 += g;
      h1 = fmaf(g, zz, h1);
    }
    s0 = warp_sum(s0);
    s1 = warp_sum(s1);
    h0 = warp_sum(h0);
    h1 = warp_sum(h1);
    value = mc_finalize(a, mu, var, s0, s1, S, zb, zdev);
    float d_mu, d_sd;
    if (a.kind == BB_ACQ_QSR || a.kind == BB_ACQ_QUCB) {
      d_mu = a1;
      d_sd = a1 * zb + (a.kind == BB_ACQ_QUCB ? ucb_c * fabsf(a1) * zdev : 0.f);
    } else {
      const float inv_tau = a.kind == BB_ACQ_QLOGEI ? 1.f / a.tau_relu : a.kind == BB_ACQ_QPI ? 1.f / a.tau_pi : 1.f;
      const float norm = a.kind == BB_ACQ_QLOGEI ? 1.f / (s0 + 0.1f * s1) : 1.f / (float)S;
      d_mu = a1 * inv_tau * h0 * norm;
      d_sd = a1 * inv_tau * h1 * norm;
    }
    g_mu = d_mu;
    g_var = d_sd / (2.f * sd);
  } else {
    float *lv = w.lv, *mP = w.mP, *moP = w.moP, *Lw = w.Lw, *Lb = w.Lb, *Wc = w.Wc, *Wm = w.Wm;
    // ---- k_acq_joint's forward: Cholesky of the joint covariance, candidate first ----
    float sd = 0.f;
    bool ok = false;
    for (int attempt = 0; attempt < 4 && !ok; ++attempt) {
      const float jit = attempt == 0 ? 0.f : 1e-6f * __powf(10.f, (float)(attempt - 1));
      sd = sqrtf(var + jit);
      const float li = cr / sd;
      __syncwarp();
      if (lane < P) {
        lv[lane] = li;
        mP[lane] = __ldg(pend_mu + lane);
      }
      __syncwarp();
      if (lane < P)
        for (int j = 0; j <= lane; ++j)
          Lw[lane * P + j] = __ldg(pend_cov + lane * P + j) - li * lv[j] + (j == lane ? jit : 0.f);
      __syncwarp();
      bool fail = !(var + jit > 0.f);
      for (int j = 0; j < P; ++j) {
        const float dj = Lw[j * P + j];
        if (!(dj > 0.f)) {
          fail = true;
          break;
        }
        const float sj = sqrtf(dj);
        __syncwarp();
        if (lane == j) Lw[j * P + j] = sj;
        if (lane > j && lane < P) Lw[lane * P + j] /= sj;
        __syncwarp();
        if (lane > j && lane < P) {
          const float lij = Lw[lane * P + j];
          for (int k = j + 1; k <= lane; ++k) Lw[lane * P + k] -= lij * Lw[k * P + j];
        }
        __syncwarp();
      }
      ok = !fail;
    }
    __syncwarp();
    const float zb0 = __shfl_sync(kFull, zb, 0);
    {
      float ym = (lane < P) ? fmaf(lv[lane], zb0, mP[lane]) : 0.f;
      for (int j = 0; j < P; ++j) {
        const float zbj = __shfl_sync(kFull, zb, 1 + j);
        if (lane < P && j <= lane) ym = fmaf(Lw[lane * P + j], zbj, ym);
      }
      if (lane < P) moP[lane] = fmaf(a1, ym, a0);
      __syncwarp();
    }
    const float mo_c = fmaf(a1, fmaf(sd, zb0, mu), a0);
    // per-sample terms of point i (0: the candidate) from its objective o
    auto term = [&](int i, float o) -> float {
      if (a.kind == BB_ACQ_QLOGEI) return logf(a.tau_relu) + log_fatplus_t((o - a.best_f) / a.tau_relu);
      if (a.kind == BB_ACQ_QEI) return fmaxf(o - a.best_f, 0.f);
      if (a.kind == BB_ACQ_QSR) return o;
      if (a.kind == BB_ACQ_QPI) return 1.0f / (1.0f + __expf(-(o - a.best_f) / a.tau_pi));
      const float m = i == 0 ? mo_c : moP[i - 1];
      return m + ucb_c * fabsf(o - m);
    };
    auto sample_obj = [&](const float* zr, int i) -> float {  // o of point i >= 1 in sample zr
      float y = fmaf(lv[i - 1], zr[0], mP[i - 1]);
      const float* Li = Lw + (i - 1) * P;
      for (int j = 0; j < i; ++j) y = fmaf(Li[j], zr[1 + j], y);
      return fmaf(a1, y, a0);
    };
    // pass 1: the value, exactly as k_acq_joint forms it
    float run_max = -INFINITY, run_sum = 0.f;
    for (int s = lane; s < S; s += 32) {
      const float* zr = z + s * zs;
      float li_arr[BB_MAX_PENDING + 1];
      float red = term(0, fmaf(a1, fmaf(sd, zr[0], mu), a0));
      li_arr[0] = red;
      for (int i = 1; i < Q; ++i) {
        const float val = term(i, sample_obj(zr, i));
        li_arr[i] = val;
        red = fmaxf(red, val);
      }
      if (a.kind == BB_ACQ_QLOGEI) lse_push(fatmax_q(li_arr, Q, red, a.tau_max), run_max, run_sum);
      else run_sum += red;
    }
    float lse = 0.f;
    if (a.kind == BB_ACQ_QLOGEI) {
      lse_warp_combine(run_max, run_sum);
      lse = run_max + logf(run_sum);
      value = lse - logf((float)S);
    } else {
      value = warp_sum(run_sum) / (float)S;
    }
    // pass 2: per-sample weights dA/dy_i in chunks of 32 samples, accumulated into dA/d(mu, sd, l, L22)
    float acc_l = 0.f, acc_m = 0.f, acc_wm = 0.f, acc_mu = 0.f, acc_sd = 0.f;
    for (int e = lane; e < P * P; e += 32) Lb[e] = 0.f;
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      __syncwarp();
      for (int i = 0; i < Q; ++i) {
        Wc[lane * Q + i] = 0.f;
        Wm[lane * Q + i] = 0.f;
      }
      if (s < S) {
        const float* zr = z + s * zs;
        float ob[BB_MAX_PENDING + 1], li_arr[BB_MAX_PENDING + 1];
        ob[0] = fmaf(a1, fmaf(sd, zr[0], mu), a0);
        float red = term(0, ob[0]);
        li_arr[0] = red;
        int imax = 0;
        for (int i = 1; i < Q; ++i) {
          ob[i] = sample_obj(zr, i);
          const float val = term(i, ob[i]);
          li_arr[i] = val;
          if (val > red) {
            red = val;
            imax = i;
          }
        }
        float w_s = 1.f / (float)S;  // dA/d(reduced sample)
        if (a.kind == BB_ACQ_QLOGEI) {
          const float fm = fatmax_q(li_arr, Q, red, a.tau_max);
          w_s = expf(fm - lse);
          const float inv = 1.0f / (2.0f * a.tau_max);
          float ssum = 0.f;
          for (int k = 0; k < Q; ++k) {
            const float wk = fmaf(red - li_arr[k], inv, 1.0f);
            ssum += 1.0f / (wk * wk);
          }
          float rest = 0.f;
          for (int k = 0; k < Q; ++k) {
            const float wk = fmaf(red - li_arr[k], inv, 1.0f);
            const float dk = 1.0f / (wk * wk * wk) / ssum;
            rest += dk;
            Wc[lane * Q + k] = dk;
          }
          Wc[lane * Q + imax] += 1.f - rest;
          for (int k = 0; k < Q; ++k)
            Wc[lane * Q + k] *= w_s * a1 * dlog_fatplus_t((ob[k] - a.best_f) / a.tau_relu) / a.tau_relu;
        } else {
          float d;
          const float o = ob[imax];
          if (a.kind == BB_ACQ_QEI) d = o - a.best_f > 0.f ? 1.f : 0.f;
          else if (a.kind == BB_ACQ_QSR) d = 1.f;
          else if (a.kind == BB_ACQ_QPI) {
            d = dsigmoidf_((o - a.best_f) / a.tau_pi) / a.tau_pi;
          } else {
            const float m = imax == 0 ? mo_c : moP[imax - 1];
            const float sgn = o > m ? 1.f : (o < m ? -1.f : 0.f);
            d = ucb_c * sgn;
            Wm[lane * Q + imax] = w_s * a1 * (1.f - d);
          }
          Wc[lane * Q + imax] = w_s * a1 * d;
        }
      }
      __syncwarp();
      const int ns = min(32, S - s0);
      for (int t = 0; t < ns; ++t) {
        const float* zr = z + (s0 + t) * zs;
        const float* wr = Wc + t * Q;
        if (lane < P) {
          const float wt = wr[1 + lane];
          acc_l = fmaf(wt, zr[0], acc_l);
          acc_wm += Wm[t * Q + 1 + lane];
          float* Lbr = Lb + lane * P;
          for (int j = 0; j <= lane; ++j) Lbr[j] = fmaf(wt, zr[1 + j], Lbr[j]);
        } else if (lane == P) {
          acc_mu += wr[0];
          acc_sd = fmaf(wr[0], zr[0], acc_sd);
          acc_m += Wm[t * Q];
        }
      }
    }
    __syncwarp();
    // qUCB: the sample means carry weight too (they depend on the inputs like a sample with z = column means)
    if (a.kind == BB_ACQ_QUCB) {
      if (lane < P) acc_l = fmaf(acc_wm, zb0, acc_l);
      for (int j = 0; j < P; ++j) {  // column j + 1's mean sits in lane j + 1
        const float zbj = __shfl_sync(kFull, zb, 1 + j);
        if (lane < P && j <= lane) Lb[lane * P + j] = fmaf(acc_wm, zbj, Lb[lane * P + j]);
      }
      if (lane == P) {
        acc_mu += acc_m;
        acc_sd = fmaf(acc_m, zb0, acc_sd);
      }
    }
    __syncwarp();
    // ---- back through the Cholesky of A22 = Sigma_PP - l l^T + jit I ----
    float* Mw = Wc;  // [P][P] tril(L22^T dL22)
    if (lane < P)
      for (int j = 0; j <= lane; ++j) {
        float m = 0.f;
        for (int k = lane; k < P; ++k) m = fmaf(Lw[k * P + lane], Lb[k * P + j], m);
        Mw[lane * P + j] = m;
      }
    __syncwarp();
    // w = L22^-1 l (forward substitution), lane i holds w_i
    float res = lane < P ? lv[lane] : 0.f, wv = 0.f;
    for (int j = 0; j < P; ++j) {
      const float wj = __shfl_sync(kFull, res, j) / Lw[j * P + j];
      if (lane == j) wv = wj;
      if (lane > j && lane < P) res = fmaf(-Lw[lane * P + j], wj, res);
    }
    // h = G w, G = (tril(M) + tril(M, -1)^T) / 2
    float hv = 0.f;
    for (int j = 0; j < P; ++j) {
      const float wj = __shfl_sync(kFull, wv, j);
      if (lane < P) hv = fmaf(j <= lane ? Mw[lane * P + j] : Mw[j * P + lane], wj, hv);
    }
    hv *= 0.5f;
    // q = L22^-T h (back substitution), lane i holds q_i
    res = hv;
    float qv = 0.f;
    for (int j = P - 1; j >= 0; --j) {
      const float qj = __shfl_sync(kFull, res, j) / Lw[j * P + j];
      if (lane == j) qv = qj;
      if (lane < j) res = fmaf(-Lw[j * P + lane], qj, res);
    }
    const float lbar = lane < P ? acc_l - 2.f * qv : 0.f;
    // l = c / sd: A_c = lbar / sd, and sd picks up -sum_i lbar_i l_i / sd
    const float sd_l = warp_sum(lane < P ? lbar * lv[lane] : 0.f);
    const float mu_bar = __shfl_sync(kFull, acc_mu, P), sd_bar = __shfl_sync(kFull, acc_sd, P) - sd_l / sd;
    g_mu = mu_bar;
    g_var = sd_bar / (2.f * sd);
    if (lane < P) w.ac[lane] = lbar / sd;
    if (!ok) {
      value = __int_as_float(0x7fc00000);
      g_mu = g_var = 0.f;
      if (lane < P) w.ac[lane] = 0.f;
    }
    __syncwarp();
  }
}

}  // namespace bb
