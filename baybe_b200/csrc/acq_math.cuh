// acq_math.cuh -- acquisition-function arithmetic shared by the fused kernel and the
// stand-alone scoring kernels.  Restates botorch's q=1 Monte-Carlo and analytic acquisition
// functions (classes selected by name at /root/reference/baybe/acquisition/base.py:162-181,
// arguments assembled at baybe/acquisition/_builder.py:195-265); objective o = a*y + b
// (baybe/objectives/single.py:66-91).
//
// qLogEI identity used here: logmeanexp_s(log fatplus(x_s)) == log(mean_s fatplus(x_s)), so the
// per-sample log/exp pair of the reference formulation is replaced by one sum of
// fatplus(x)/tau = softplus(t) + 0.1/(1+t^2), t = x/tau, followed by a single log.
#pragma once

#include "common.cuh"

namespace bb {

// softplus(t) - max(t,0) = log1p(exp(-|t|)); only matters for |t| < 30 in fp32 sums.
__device__ __forceinline__ float softplus_tail(float abs_t) {
  float e = fast_ex2(-kLog2e * abs_t);
  return log1pf(e);
}

// log(fatplus(x, tau) / tau) = log(softplus(t) + 0.1/(1+t^2)) at t = x/tau (botorch fatplus, alpha = 0.1).
__device__ __forceinline__ float log_fatplus_t(float t) {
  const float sp = fmaxf(t, 0.f) + ((fabsf(t) < 30.f) ? softplus_tail(fabsf(t)) : 0.f);
  return logf(sp + 0.1f / fmaf(t, t, 1.0f));
}

// One Monte-Carlo sample contributes to two running sums; t = c0 + c1 * z_s with
//   qLogEI: t = (o_s - best_f)/tau_relu ; s0 += softplus(t) ; s1 += 1/(1+t^2)
//   qEI   : t = o_s - best_f            ; s0 += relu(t)
//   qPI   : t = (o_s - best_f)/tau_pi   ; s0 += sigmoid(t)
//   qUCB, qSR: closed form from the sample statistics mean(z), mean(|z - mean z|); no per-sample work.
__device__ __forceinline__ void mc_coef(const bb_acq_spec& a, float mu, float var, float& c0,
                                        float& c1) {
  const float mo = fmaf(a.obj_scale, mu, a.obj_shift);
  const float so = a.obj_scale * sqrtf(var);  // signed: o_s = mo + so * z_s
  float inv_tau = 1.0f;
  if (a.kind == BB_ACQ_QLOGEI) inv_tau = 1.0f / a.tau_relu;
  if (a.kind == BB_ACQ_QPI) inv_tau = 1.0f / a.tau_pi;
  c0 = (mo - a.best_f) * inv_tau;
  c1 = so * inv_tau;
}

template <int KIND>
__device__ __forceinline__ void mc_term(float t, float& s0, float& s1) {
  if constexpr (KIND == BB_ACQ_QLOGEI) {
    s0 += fmaxf(t, 0.f);
    s1 += fast_rcp(fmaf(t, t, 1.0f));
    if (fabsf(t) < 30.f) s0 += softplus_tail(fabsf(t));
  } else if constexpr (KIND == BB_ACQ_QEI) {
    s0 += fmaxf(t, 0.f);
  } else if constexpr (KIND == BB_ACQ_QPI) {
    s0 += fast_rcp(1.0f + fast_ex2(-kLog2e * t));
  }
}

template <int KIND>
__device__ __forceinline__ void mc_partial_kind(float c0, float c1, const float4* __restrict__ z4,
                                                int n4, float& s0, float& s1) {
  if constexpr (KIND == BB_ACQ_QLOGEI) {
    // fast path for all four samples, one rarely-taken correction branch per group of four
    float s0b = 0.f, s1b = 0.f;
#pragma unroll 2
    for (int i = 0; i < n4; ++i) {
      const float4 z = z4[i];
      const float t0 = fmaf(c1, z.x, c0), t1 = fmaf(c1, z.y, c0);
      const float t2 = fmaf(c1, z.z, c0), t3 = fmaf(c1, z.w, c0);
      s0 += fmaxf(t0, 0.f);
      s0b += fmaxf(t1, 0.f);
      s0 += fmaxf(t2, 0.f);
      s0b += fmaxf(t3, 0.f);
      s1 += fast_rcp(fmaf(t0, t0, 1.0f));
      s1b += fast_rcp(fmaf(t1, t1, 1.0f));
      s1 += fast_rcp(fmaf(t2, t2, 1.0f));
      s1b += fast_rcp(fmaf(t3, t3, 1.0f));
      const float tmin = fminf(fminf(fabsf(t0), fabsf(t1)), fminf(fabsf(t2), fabsf(t3)));
      if (tmin < 30.f) {
        if (fabsf(t0) < 30.f) s0 += softplus_tail(fabsf(t0));
        if (fabsf(t1) < 30.f) s0 += softplus_tail(fabsf(t1));
        if (fabsf(t2) < 30.f) s0 += softplus_tail(fabsf(t2));
        if (fabsf(t3) < 30.f) s0 += softplus_tail(fabsf(t3));
      }
    }
    s0 += s0b;
    s1 += s1b;
  } else {
    for (int i = 0; i < n4; ++i) {
      const float4 z = z4[i];
      mc_term<KIND>(fmaf(c1, z.x, c0), s0, s1);
      mc_term<KIND>(fmaf(c1, z.y, c0), s0, s1);
      mc_term<KIND>(fmaf(c1, z.z, c0), s0, s1);
      mc_term<KIND>(fmaf(c1, z.w, c0), s0, s1);
    }
  }
}

// Partial sums over part `part` of `nparts` equal shares of the S base samples in shared memory
// (S / nparts must be a multiple of 4).
__device__ __forceinline__ void mc_partial(const bb_acq_spec& a, float mu, float var,
                                           const float* __restrict__ z_s, int S, int part,
                                           int nparts, float& s0, float& s1) {
  s0 = 0.f;
  s1 = 0.f;
  float c0, c1;
  mc_coef(a, mu, var, c0, c1);
  const int per = S / nparts;
  const float4* z4 = reinterpret_cast<const float4*>(z_s + part * per);
  const int n4 = per >> 2;
  if (a.kind == BB_ACQ_QLOGEI) mc_partial_kind<BB_ACQ_QLOGEI>(c0, c1, z4, n4, s0, s1);
  else if (a.kind == BB_ACQ_QEI) mc_partial_kind<BB_ACQ_QEI>(c0, c1, z4, n4, s0, s1);
  else if (a.kind == BB_ACQ_QPI) mc_partial_kind<BB_ACQ_QPI>(c0, c1, z4, n4, s0, s1);
}

// ------------------------------------------------------------------------------------------
// qLogEI, tabulated fat-tail sum (q = 1, shared base samples).
// With x_s = (o_s - best_f)/tau = c0 + c1 z_s, tau = 1e-6 and zeta = sign(c1) z sorted descending, a candidate
// with at most 8 improving samples (x_(9) <= 0: nearly every row of a discrete space) splits its sum
//   sum_s fatplus(x_s)/tau = [16 largest zeta: exact terms]  +  c1^-2 H(w),   w = -c0/|c1| >= zeta_(9),
//   H(w) = sum_{s > 16} (zeta_(s) - w)^-2      (those samples sit at x <= -1024: softplus = 0, 1/(1+x^2) = x^-2).
// H is ONE function of one variable for every candidate: it is tabulated once per CTA as
// F(v) = H(w) (w - zeta_(9) + 1)^2 over v = 1/(w - zeta_(9) + 1) in [0,1] (linear interpolation, 512 intervals,
// relative error < 1e-5; the nearest pole zeta_(17) stays >= 0.25 away).  Rows outside the envelope take the
// exact sum over all S samples (mc_row_exact_warp).
// Table region (1024 floats): [0..512] F | [520..535] top-16 zeta (descending) | [536] table valid |
//                             [544..799] scratch for the callers (exact (s0, s1) per row).
// ------------------------------------------------------------------------------------------
constexpr int kMcNT = 512, kMcTop = 520, kMcOk = 536, kMcRows = 544, kMcK = 16, kMcJ = 8;

__host__ __device__ __forceinline__ bool mc_table_applicable(int has_acq, const bb_acq_spec& a, int S) {
  return has_acq && a.kind == BB_ACQ_QLOGEI && S >= 64 && (S & 63) == 0 && S <= 512;
}

// Called by EVERY thread of the CTA (contains __syncthreads); z_s: the S base samples in shared memory.
__device__ __forceinline__ void mc_table_setup(float* __restrict__ tab, const float* __restrict__ z_s, int S,
                                               float sgn) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (warp == 0) {  // sixteen largest zeta: S/32 values per lane, sixteen rounds of warp arg-max
    float vals[16];
    const int per_lane = S >> 5;
#pragma unroll
    for (int j = 0; j < 16; ++j) vals[j] = j < per_lane ? sgn * z_s[j * 32 + lane] : -INFINITY;
    for (int k = 0; k < kMcK; ++k) {
      float m = -INFINITY;
      int mj = 0;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (vals[j] > m) {
          m = vals[j];
          mj = j;
        }
      float wm = m;
      for (int o = 16; o > 0; o >>= 1) wm = fmaxf(wm, __shfl_xor_sync(0xffffffffu, wm, o));
      const unsigned who = __ballot_sync(0xffffffffu, m == wm);
      if (lane == (int)(__ffs(who) - 1)) {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (j == mj) vals[j] = -INFINITY;
      }
      if (lane == 0) tab[kMcTop + k] = wm;
    }
  }
  __syncthreads();
  const float thr = tab[kMcTop + kMcK - 1], w0 = tab[kMcTop + kMcJ];
  if (warp == 1) {  // ties at the threshold would make "top 16" ambiguous: then every row takes the exact path
    int cnt = 0;
    for (int e = lane; e < S; e += 32) cnt += (sgn * z_s[e] >= thr) ? 1 : 0;
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) tab[kMcOk] = (cnt == kMcK) ? 1.f : 0.f;
  }
  for (int j = tid; j <= kMcNT; j += blockDim.x) {
    float f = (float)(S - kMcK);
    if (j > 0) {
      const float a = (float)kMcNT / (float)j;  // a = w - zeta_(9) + 1 = 1/v
      const float w = w0 - 1.0f + a;
      const float cut = thr - w;  // zeta < thr  <=>  zeta - w < cut
      float acc0 = 0.f, acc1 = 0.f;
#pragma unroll 4
      for (int e = 0; e < S; e += 2) {
        const float d0 = fmaf(sgn, z_s[e], -w), d1 = fmaf(sgn, z_s[e + 1], -w);
        const float r0 = fast_rcp(d0 * d0), r1 = fast_rcp(d1 * d1);
        acc0 += d0 < cut ? r0 : 0.f;
        acc1 += d1 < cut ? r1 : 0.f;
      }
      f = (acc0 + acc1) * a * a;
    }
    tab[j] = f;
  }
  __syncthreads();
}

// The same table built by a GRID once per call (rebuilding it in each persistent CTA of a full-size launch costs more
// than it saves): every CTA repeats the cheap top-16 step, warp w of CTA b then fills entry 8 b + w with a
// lane-parallel sum (fixed order: lane partials over e = lane, lane + 32, ..., xor-tree).  CTA 0 also stores the
// top-16 block and the validity flag.  out: kMcRows floats in global memory.
__device__ __forceinline__ void mc_table_grid_part(float* __restrict__ tab, const float* __restrict__ z_s, int S,
                                                   float sgn, float* __restrict__ out) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // the scoring kernel that follows on the stream may start its prologue now; it synchronises on this grid's
  // completion (griddepcontrol.wait) before it reads `out`
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (warp == 0) {
    float vals[16];
    const int per_lane = S >> 5;
#pragma unroll
    for (int j = 0; j < 16; ++j) vals[j] = j < per_lane ? sgn * z_s[j * 32 + lane] : -INFINITY;
    for (int k = 0; k < kMcK; ++k) {
      float m = -INFINITY;
      int mj = 0;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (vals[j] > m) {
          m = vals[j];
          mj = j;
        }
      float wm = m;
      for (int o = 16; o > 0; o >>= 1) wm = fmaxf(wm, __shfl_xor_sync(0xffffffffu, wm, o));
      const unsigned who = __ballot_sync(0xffffffffu, m == wm);
      if (lane == (int)(__ffs(who) - 1)) {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (j == mj) vals[j] = -INFINITY;
      }
      if (lane == 0) tab[kMcTop + k] = wm;
    }
  }
  __syncthreads();
  const float thr = tab[kMcTop + kMcK - 1], w0 = tab[kMcTop + kMcJ];
  if (blockIdx.x == 0) {
    if (warp == 1) {
      int cnt = 0;
      for (int e = lane; e < S; e += 32) cnt += (sgn * z_s[e] >= thr) ? 1 : 0;
      for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      if (lane == 0) out[kMcOk] = (cnt == kMcK) ? 1.f : 0.f;
    }
    if (tid < kMcK) out[kMcTop + tid] = tab[kMcTop + tid];
  }
  const int j = blockIdx.x * (blockDim.x >> 5) + warp;
  if (j <= kMcNT) {
    float f = (float)(S - kMcK);
    if (j > 0) {
      const float a = (float)kMcNT / (float)j;
      const float w = w0 - 1.0f + a;
      const float cut = thr - w;
      float acc = 0.f;
      for (int e = lane; e < S; e += 32) {
        const float d0 = fmaf(sgn, z_s[e], -w);
        acc += d0 < cut ? fast_rcp(d0 * d0) : 0.f;
      }
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      f = acc * a * a;
    }
    if (lane == 0) out[j] = f;
  }
}

// (s0, s1) of one row from the table; false (and s0 = s1 = 0) if the row lies outside the envelope.
__device__ __forceinline__ bool mc_row_fast(const float* __restrict__ tab, float c0, float c1, float& s0,
                                            float& s1) {
  const float ac1 = fabsf(c1);
  const float t9 = fmaf(ac1, tab[kMcTop + kMcJ], c0);        // 9th largest x_s of this row
  const float t17 = fmaf(ac1, tab[kMcTop + kMcK - 1], c0);   // bounds every tabulated sample from above
  const bool fast = tab[kMcOk] != 0.f && ac1 > 1e-30f && t9 <= 0.f && t17 <= -1024.f;
  s0 = 0.f;
  s1 = 0.f;
  if (fast) {
    float tmin = 1e30f;
#pragma unroll
    for (int k = 0; k < kMcK; ++k) {
      const float t = fmaf(ac1, tab[kMcTop + k], c0);
      s0 += fmaxf(t, 0.f);
      s1 += fast_rcp(fmaf(t, t, 1.0f));
      tmin = fminf(tmin, fabsf(t));
    }
    if (tmin < 30.f) {  // a sample within 30 tau of the incumbent: softplus differs from relu there (rare)
      for (int k = 0; k < kMcK; ++k) {
        const float t = fabsf(fmaf(ac1, tab[kMcTop + k], c0));
        if (t < 30.f) s0 += softplus_tail(t);
      }
    }
    const float inv = 1.0f / ac1;
    const float a = fmaf(-t9, inv, 1.0f);  // w - zeta_(9) + 1 >= 1, no cancellation
    const float v = 1.0f / a;
    const float x = v * (float)kMcNT;
    const int i = min((int)x, kMcNT - 1);
    const float fr = x - (float)i;
    const float f0 = tab[i], f1 = tab[i + 1];
    const float q = v * inv;
    s1 = fmaf(fmaf(fr, f1 - f0, f0), q * q, s1);
  }
  return fast;
}

// Exact (s0, s1) of one row by a whole warp: lane l takes samples l, l+32, ...; fixed reduction order, so a row's
// value does not depend on where it is evaluated.  Result in every lane.
__device__ __forceinline__ void mc_row_exact_warp(const float* __restrict__ z_s, int S, float c0, float c1, int lane,
                                                  float& a0, float& a1) {
  float b0 = 0.f, b1 = 0.f;
  a0 = 0.f;
  a1 = 0.f;
  for (int e = lane; e < S; e += 64) {  // S is a multiple of 64 on this path; two independent chains
    const float t = fmaf(c1, z_s[e], c0), u = fmaf(c1, z_s[e + 32], c0);
    a0 += fmaxf(t, 0.f);
    b0 += fmaxf(u, 0.f);
    a1 += fast_rcp(fmaf(t, t, 1.0f));
    b1 += fast_rcp(fmaf(u, u, 1.0f));
    if (fminf(fabsf(t), fabsf(u)) < 30.f) {
      if (fabsf(t) < 30.f) a0 += softplus_tail(fabsf(t));
      if (fabsf(u) < 30.f) b0 += softplus_tail(fabsf(u));
    }
  }
  a0 += b0;
  a1 += b1;
  for (int o = 16; o > 0; o >>= 1) {
    a0 += __shfl_xor_sync(0xffffffffu, a0, o);
    a1 += __shfl_xor_sync(0xffffffffu, a1, o);
  }
}

__device__ __forceinline__ float mc_finalize(const bb_acq_spec& a, float mu, float var, float s0,
                                             float s1, int S, float z_mean, float zdev_mean) {
  const float sd = sqrtf(var);
  const float mo = fmaf(a.obj_scale, mu, a.obj_shift);
  const float so = a.obj_scale * sd;
  switch (a.kind) {
    case BB_ACQ_QLOGEI:
      return logf(a.tau_relu) + logf((s0 + 0.1f * s1) / (float)S);
    case BB_ACQ_QEI:
    case BB_ACQ_QPI:
      return s0 / (float)S;
    case BB_ACQ_QSR:
      return fmaf(so, z_mean, mo);
    default:  // qUCB: mean_s( m + sqrt(beta*pi/2) |o_s - m| ) with m = mean_s o_s, the SAMPLE mean (botorch
              // qUpperConfidenceBound._sample_forward: mean = obj.mean(dim=0)); zdev_mean = mean_s |z_s - mean z|
      return fmaf(sqrtf(a.beta * 1.5707963267948966f) * fabsf(so), zdev_mean, fmaf(so, z_mean, mo));
  }
}

// Analytic acquisition functions with an affine posterior transform (_builder.py:224-236).
// Evaluated in float64: one evaluation per candidate, far off the critical path.
__device__ __forceinline__ double norm_pdf(double u) {
  return exp(-0.5 * u * u) * 0.3989422804014327;
}
__device__ __forceinline__ double norm_cdf(double u) { return 0.5 * erfc(-u * 0.7071067811865476); }
__device__ __forceinline__ double log1mexp_d(double x) {
  return (x > -0.6931471805599453) ? log(-expm1(x)) : log1p(-exp(x));
}
__device__ __forceinline__ double log_ei_helper(double u) {
  // botorch _log_ei_helper: log(phi(u) + u Phi(u)), stable in the left tail
  if (u > -1.0) return log(norm_pdf(u) + u * norm_cdf(u));
  const double log_phi = -0.5 * (u * u + 1.8378770664093453);
  if (u > -1e6) {
    double w = log(erfcx(-u * 0.7071067811865476) * fabs(u)) + 0.22579135264472744;
    return log_phi + log1mexp_d(w);
  }
  return log_phi - 2.0 * log(fabs(u));
}

__device__ __forceinline__ float analytic_value(const bb_acq_spec& a, float mu, float var) {
  const double m = (double)a.obj_scale * (double)mu + (double)a.obj_shift;
  const double s = fabs((double)a.obj_scale) * sqrt((double)var);
  switch (a.kind) {
    case BB_ACQ_PM:
      return (float)m;
    case BB_ACQ_PSTD:
      return (float)(a.maximize ? s : -s);
    case BB_ACQ_UCB:
      return (float)(m + sqrt((double)a.beta) * s);
    default:
      break;
  }
  const double u = (m - (double)a.best_f) / s;
  if (a.kind == BB_ACQ_EI) return (float)(s * (norm_pdf(u) + u * norm_cdf(u)));
  if (a.kind == BB_ACQ_LOGEI) return (float)(log_ei_helper(u) + log(s));
  return (float)norm_cdf(u);  // PI
}

}  // namespace bb
