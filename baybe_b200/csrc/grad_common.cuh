// grad_common.cuh -- device code of the gradient kernels (k_acq_grad in grad.cu, k_objective_grad in objgrad.cu).
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

}  // namespace bb
