// grad.cu -- value and gradient of a single-target acquisition function at P points (bb_acq_grad).
//
// Replaces the autograd pass of the reference's continuous optimiser: optimize_acqf's L-BFGS-B on
// acqf(X).backward() (baybe/recommenders/pure/bayesian/botorch/continuous.py:184) and the same inside
// optimize_acqf_mixed with the discrete features held fixed (botorch/hybrid.py:110).
//
// One warp per point, all on the CUDA cores in fp32 (the analytic kinds' closed forms in float64, as
// analytic_value).  With a = x * scale + shift (bb_model's d_cand_scale / d_cand_shift) and b_i the scaled training
// rows:
//   k_i = s_f^2 kappa(|a - b_i|),  v = L^-1 k,  u = L^-T v,
//   mu = y_mean + s_y (c + k . alpha),  var = s_y^2 max(s_f^2 - |v|^2, 1e-10),
//   c_p = s_y^2 (k(x, x_p) - k . beta_p)                          (pending points p)
// and, with A_mu, A_var, A_c[p] the partial derivatives of the acquisition value,
//   dA/dk_i = s_y A_mu alpha_i - 2 s_y^2 A_var u_i - s_y^2 sum_p A_c[p] beta_p,i
//   grad_x A = (sum_i dA/dk_i dk_i/da + s_y^2 sum_p A_c[p] dk(x, x_p)/da) * scale.
// v is formed 32 rows at a time: each lane takes every 32nd column of the 32 rows (coalesced loads of L^-1) and a
// reduce-scatter over the warp leaves row j0 + l in lane l; u needs no reduction (lane l owns column i0 + l).
// The value and its partials at a point come from acq_point_partials (grad_common.cuh, shared with k_acq_grad_large).
// With pending points the value is k_acq_joint's (acq.cu): the Cholesky of [[var, c^T], [c, Sigma_PP]] with the
// candidate first, the same jitter escalation and the same join of the pending points' terms.  Its reverse pass
// accumulates dA/dL22 over the samples and goes back through the (1+p) Cholesky with
//   dA/dA22 = sym(L22^-T Phi(L22^T dL22) L22^-1) / 2  (as torch's cholesky backward),  A22 = Sigma_PP - l l^T,
// so only dA/dl = -2 (dA/dA22) l is needed: two triangular solves and one matrix-vector product per point.
// Every reduction has a fixed order and nothing is accumulated atomically: repeated calls are bit-identical.
#include "fused_common.cuh"
#include "grad_common.cuh"

namespace bb {

constexpr int kGradThreads = 128;  // four points per block
constexpr int kGradWarps = kGradThreads / 32;

struct GradParams {
  bb_acq_spec a;
  const float* x;  // [N][d]
  int64_t N;
  const float *cand_scale, *cand_shift, *train_m2, *alpha, *linv;
  int n, n_pad, d, d_pad;
  const float* mean_const;  // [1]
  float y_mean, y_std, sf2;
  int P;
  const float *pend_x, *pend_beta, *pend_mu, *pend_cov;  // [P][d], [P][n_pad], [P], [P][P]
  const float* z;                                          // [S][1+P]
  int S;
  float* value;  // [N]
  float* grad;   // [N][d]
};

// per-warp scratch in floats: a | k (then dA/dk_i * dk_i/dt) | gk | v | gkp [32] | acq_point_partials' scratch
// (4 x 32 vectors | L22 | dL22 | 2 x sample chunk)
__host__ __device__ inline int grad_warp_floats(int n_pad, int d_pad, int P) {
  return (d_pad + 3 * n_pad + 5 * 32 + 2 * P * P + 2 * 32 * (P + 1) + 3) & ~3;
}

template <int FAMILY>
__global__ void __launch_bounds__(kGradThreads) k_acq_grad(const GradParams p) {
  extern __shared__ __align__(16) float smem_g[];
  const int P = p.P, Q = P + 1, zs = Q | 1;
  const bool is_mc = p.a.kind <= BB_ACQ_QPI;
  const int S = is_mc ? p.S : 0;
  float* z_s = smem_g;  // [S][zs]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* wb = z_s + ((S * zs + 3) & ~3) + warp * grad_warp_floats(p.n_pad, p.d_pad, P);
  float* a_w = wb;
  float* k_w = a_w + p.d_pad;
  float* gk_w = k_w + p.n_pad;
  float* v_w = gk_w + p.n_pad;
  float* gkp = v_w + p.n_pad;                 // [32] 2 s_f^2 dk/dt of k(x, x_p)
  const AcqScratch w = acq_scratch(gkp + 32, P);  // acq_point_partials' scratch
  for (int e = threadIdx.x; e < S * Q; e += blockDim.x) {
    const int s = e / Q, k = e - s * Q;
    z_s[s * zs + k] = __ldg(p.z + e);
  }
  __syncthreads();
  const bb_acq_spec a = p.a;
  const float sy = p.y_std, sy2 = sy * sy;
  float zb = 0.f, zdev = 0.f;  // column means of the base samples and, for q = 1, mean |z - mean z|
  if (is_mc) sample_means_warp(z_s, zs, S, P, zb, zdev, lane);
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = warp_global; c < p.N; c += nwarps) {
    // ---- forward: a, k, mu, v, var, cross ----
    // (grad_common.cuh's kernel_row_warp, linv_apply_warp and linvt_apply_col are these passes; called from here
    // they change this kernel's register allocation, so its SASS would no longer be the one measured)
    for (int j = lane; j < p.d_pad; j += 32)
      a_w[j] = j < p.d ? fmaf(__ldg(p.x + c * p.d + j), __ldg(p.cand_scale + j), __ldg(p.cand_shift + j)) : 0.f;
    __syncwarp();
    float ka = 0.f;
    for (int i = lane; i < p.n_pad; i += 32) {
      float t = 0.f;
      for (int j = 0; j < p.d; ++j) {
        const float df = a_w[j] + 0.5f * __ldg(p.train_m2 + (size_t)i * p.d_pad + j);
        t = fmaf(df, df, t);
      }
      float k, dk;
      kernel_and_slope<FAMILY>(t, k, dk);
      k = i < p.n ? p.sf2 * k : 0.f;
      k_w[i] = k;
      gk_w[i] = i < p.n ? 2.f * p.sf2 * dk : 0.f;
      ka = fmaf(k, __ldg(p.alpha + i), ka);
    }
    ka = warp_sum(ka);
    __syncwarp();
    float vv = 0.f;
    for (int j0 = 0; j0 < p.n_pad; j0 += 32) {
      float r[32];
#pragma unroll
      for (int q = 0; q < 32; ++q) r[q] = 0.f;
      for (int i0 = 0; i0 <= j0; i0 += 32) {
        const float ki = k_w[i0 + lane];
        const float* Lr = p.linv + (size_t)j0 * p.n_pad + i0 + lane;
#pragma unroll
        for (int q = 0; q < 32; ++q) r[q] = fmaf(__ldg(Lr + (size_t)q * p.n_pad), ki, r[q]);
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
    vv = warp_sum(vv);
    const float vt = p.sf2 - vv;
    const bool var_free = vt > 1e-10f;  // the clamp passes no gradient
    const float mu = fmaf(sy, __ldg(p.mean_const) + ka, p.y_mean);
    const float var = sy2 * fmaxf(vt, 1e-10f);
    float cr = 0.f;  // lane p < P: c_p
    for (int q = 0; q < P; ++q) {
      float kb = 0.f;
      for (int i = lane; i < p.n_pad; i += 32) kb = fmaf(k_w[i], __ldg(p.pend_beta + (size_t)q * p.n_pad + i), kb);
      kb = warp_sum(kb);
      if (lane == q) cr = kb;
    }
    if (lane < P) {
      float t = 0.f;
      for (int j = 0; j < p.d; ++j) {
        const float b = fmaf(__ldg(p.pend_x + (size_t)lane * p.d + j), __ldg(p.cand_scale + j), __ldg(p.cand_shift + j));
        const float df = a_w[j] - b;
        t = fmaf(df, df, t);
      }
      float k, dk;
      kernel_and_slope<FAMILY>(t, k, dk);
      cr = sy2 * (p.sf2 * k - cr);
      gkp[lane] = 2.f * p.sf2 * dk;
    }
    __syncwarp();
    // ---- value and its partial derivatives (A_mu, A_var, A_c) ----
    float value, g_mu, g_var;
    acq_point_partials(a, mu, var, cr, P, p.pend_mu, p.pend_cov, z_s, zs, S, zb, zdev, w, value, g_mu, g_var,
                       lane);
    if (!var_free) g_var = 0.f;
    // ---- dA/dk_i, folded with dk_i/dt into k_w: coef_i = gk_i dA/dk_i ----
    const float k_mu = sy * g_mu, k_var = -2.f * sy2 * g_var;
    for (int i0 = 0; i0 < p.n_pad; i0 += 32) {
      const int i = i0 + lane;
      float u = 0.f;
      for (int j = i0; j < p.n_pad; ++j) u = fmaf(__ldg(p.linv + (size_t)j * p.n_pad + i), v_w[j], u);
      float kb = fmaf(k_mu, __ldg(p.alpha + i), k_var * u);
      for (int q = 0; q < P; ++q) kb = fmaf(-sy2 * w.ac[q], __ldg(p.pend_beta + (size_t)q * p.n_pad + i), kb);
      k_w[i] = gk_w[i] * kb;
    }
    __syncwarp();
    // ---- gradient: lanes over columns ----
    for (int j = lane; j < p.d; j += 32) {
      const float aj = a_w[j];
      float g = 0.f;
      for (int i = 0; i < p.n; ++i) g = fmaf(k_w[i], aj + 0.5f * __ldg(p.train_m2 + (size_t)i * p.d_pad + j), g);
      for (int q = 0; q < P; ++q) {
        const float b = fmaf(__ldg(p.pend_x + (size_t)q * p.d + j), __ldg(p.cand_scale + j), __ldg(p.cand_shift + j));
        g = fmaf(sy2 * w.ac[q] * gkp[q], aj - b, g);
      }
      p.grad[c * p.d + j] = g * __ldg(p.cand_scale + j);
    }
    if (lane == 0) p.value[c] = value;
    __syncwarp();
  }
}

}  // namespace bb

using namespace bb;

extern "C" int bb_acq_grad(const bb_model* m, const bb_acq_spec* a, const float* d_x, int64_t N, int32_t n_pending,
                           const float* d_pend_x, const float* d_pend_beta, const float* d_pend_mu,
                           const float* d_pend_cov, const float* d_z, int32_t S, float* d_value, float* d_grad,
                           void* stream) {
  BB_CHECK_ARG(m && m->abi_version == BB_ABI_VERSION, "bb_acq_grad: model struct missing or ABI mismatch");
  BB_CHECK_ARG(a != nullptr, "bb_acq_grad: acquisition spec is null");
  BB_CHECK_ARG(a->kind >= BB_ACQ_QLOGEI && a->kind <= BB_ACQ_PSTD, "bb_acq_grad: acquisition kind %d is not one of "
               "the single-target kinds", a->kind);
  BB_CHECK_SUPPORTED(!m->wide, "bb_acq_grad: wide-feature models are not supported");
  BB_CHECK_SUPPORTED(m->task_col < 0, "bb_acq_grad: models with a task parameter are not supported");
  BB_CHECK_SUPPORTED(m->n_pad <= kGradMaxNPad, "bb_acq_grad: n_pad=%d above %d is not supported", m->n_pad,
                     kGradMaxNPad);
  BB_CHECK_ARG(N >= 0, "bb_acq_grad: negative point count");
  const bool is_mc = a->kind <= BB_ACQ_QPI;
  BB_CHECK_ARG(n_pending >= 0 && n_pending <= BB_MAX_PENDING, "bb_acq_grad: n_pending=%d outside [0,%d]", n_pending,
               BB_MAX_PENDING);
  BB_CHECK_ARG(n_pending == 0 || is_mc, "bb_acq_grad: pending points need a Monte Carlo acquisition function");
  BB_CHECK_ARG(!is_mc || (S >= 1 && S <= kMaxSamples), "bb_acq_grad: S=%d outside [1,%d]", S, kMaxSamples);
  BB_CHECK_ARG(!is_mc || d_z != nullptr, "bb_acq_grad: null base samples");
  BB_CHECK_ARG(n_pending == 0 || (d_pend_x && d_pend_beta && d_pend_mu && d_pend_cov),
               "bb_acq_grad: null pending buffer");
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_x && d_value && d_grad, "bb_acq_grad: null buffer");
  GradParams p;
  p.a = *a;
  p.x = d_x;
  p.N = N;
  p.cand_scale = m->d_cand_scale;
  p.cand_shift = m->d_cand_shift;
  p.train_m2 = m->d_train_m2;
  p.alpha = m->d_alpha;
  p.linv = m->d_linv32;
  p.n = m->n;
  p.n_pad = m->n_pad;
  p.d = m->d;
  p.d_pad = m->d_pad;
  p.y_mean = m->y_mean;
  p.y_std = m->y_std;
  p.P = n_pending;
  p.pend_x = d_pend_x;
  p.pend_beta = d_pend_beta;
  p.pend_mu = d_pend_mu;
  p.pend_cov = d_pend_cov;
  p.z = d_z;
  p.S = is_mc ? S : 0;
  p.value = d_value;
  p.grad = d_grad;
  p.sf2 = m->prior_scale;  // single task: the prior variance s_f^2
  int sms, max_smem;
  int rc = device_limits(&sms, &max_smem);
  if (rc != BB_OK) return rc;
  p.mean_const = m->d_mean_const;
  const int zs = (n_pending + 1) | 1;
  const size_t smem = ((size_t)((p.S * zs + 3) & ~3) + (size_t)kGradWarps * grad_warp_floats(p.n_pad, p.d_pad,
                                                                                             n_pending)) * 4;
  BB_CHECK_SUPPORTED(smem <= (size_t)max_smem, "bb_acq_grad: S*(1+n_pending)=%d too large for shared memory",
                     p.S * zs);
  int64_t blocks = (N + kGradWarps - 1) / kGradWarps;
  if (blocks > (int64_t)sms * 8) blocks = (int64_t)sms * 8;
  return dispatch_family<true>(m->family, [&](auto fam) {
    BB_SMEM_OPTIN_ONCE(k_acq_grad<decltype(fam)::value>);
    k_acq_grad<decltype(fam)::value><<<(int)blocks, kGradThreads, smem, (cudaStream_t)stream>>>(p);
    BB_LAUNCH_CHECK();
    return BB_OK;
  });
}
