// gradlarge.cu -- value and gradient of a single-target acquisition function for any single-task model
// (bb_acq_grad_large): n_pad up to 1024 and wide-feature models, which bb_acq_grad (grad.cu) does not take.
//
// It computes what bb_acq_grad computes (see grad.cu for the formulas), with a mapping suited to long kernel rows:
// one CTA of 256 threads per point, grid-striding over the points.
//   1. The CTA forms the kernel row k and its slope gk over n: a thread per training row for d < 32, a warp per row
//      (lanes over columns) from d = 32 on, so that wide rows are read coalesced.
//   2. v = L^-1 k: the warps take the 32-row blocks of the lower triangle of L^-1 (fp32, d_linv32), each block as
//      bb_acq_grad's warp forms it (coalesced loads, a reduce-scatter over the warp).  The blocks go to the warps in
//      a snake order, so that each warp reads about the same share of the triangle.  The same pass forms each pending
//      point's k . beta_p (warp p mod 8).
//   3. One warp forms mu, var and the cross covariances c_p and calls acq_point_partials (grad_common.cuh) for the
//      value and A_mu, A_var, A_c.
//   4. u = L^-T v: the warps take the 32-column blocks (lane l owns column i0 + l, no reduction), again in snake
//      order, and fold dA/dk_i with gk_i into the kernel row.
//   5. The reverse pass through the kernel row to dA/dx: threads over (row group, column), then a sum over the row
//      groups in a fixed order.
// Every per-element sum of steps 2 to 4 runs in bb_acq_grad's order, so on the shapes both take, v, u, mu and var
// agree bit for bit when the kernel row does (d < 32).  Base samples sit in shared memory when S (1 + P) fits beside
// the point's scratch, else they are read from global memory (L2).  No float atomics: repeated calls are
// bit-identical.
#include <stdlib.h>

#include "fused_common.cuh"
#include "grad_common.cuh"

namespace bb {

constexpr int kLargeMaxNPad = BB_MAX_TRAIN;

struct GradLargeParams {
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
  int z_smem;  // base samples copied to shared memory (row stride (1 + P) | 1), else read in place (stride 1 + P)
  float* value;  // [N]
  float* grad;   // [N][d]
};

// per-CTA scratch in floats: a [d_pad] | k (then gk dA/dk), gk, v [n_pad] | c_p, k . beta_p, gkp, 4 scalars [32] |
// acq_point_partials' scratch | the column-gradient partials [kCtaThreads]
__host__ __device__ inline int grad_large_floats(int n_pad, int d_pad, int P) {
  return (d_pad + 3 * n_pad + 4 * 32 + acq_scratch_floats(P) + kCtaThreads + 3) & ~3;
}

template <int FAMILY>
__global__ void __launch_bounds__(kCtaThreads) k_acq_grad_large(const GradLargeParams p) {
  extern __shared__ __align__(16) float smem_l[];
  const int P = p.P, Q = P + 1;
  const bool is_mc = p.a.kind <= BB_ACQ_QPI;
  const int S = is_mc ? p.S : 0;
  const int zs = p.z_smem ? (Q | 1) : Q;
  float* z_s = smem_l;  // [S][zs] when p.z_smem
  float* a_w = z_s + (p.z_smem ? ((S * zs + 3) & ~3) : 0);
  float* k_w = a_w + p.d_pad;
  float* gk_w = k_w + p.n_pad;
  float* v_w = gk_w + p.n_pad;
  float* cr_s = v_w + p.n_pad;  // [32] c_p, then (after the middle) A_c[p] s_y^2
  float* kb_s = cr_s + 32;      // [32] k . beta_p
  float* gkp = kb_s + 32;       // [32] 2 s_f^2 dk/dt of k(x, x_p)
  float* sc = gkp + 32;         // [4] k_mu, k_var
  const AcqScratch w = acq_scratch(sc + 32, P);
  float* part = sc + 32 + acq_scratch_floats(P);  // [kCtaThreads]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* z = p.z_smem ? z_s : p.z;
  if (p.z_smem) {
    for (int e = threadIdx.x; e < S * Q; e += blockDim.x) {
      const int s = e / Q, k = e - s * Q;
      z_s[s * zs + k] = __ldg(p.z + e);
    }
    __syncthreads();
  }
  const bb_acq_spec a = p.a;
  const float sy = p.y_std, sy2 = sy * sy;
  float zb = 0.f, zdev = 0.f;  // warp 0 only
  if (is_mc && warp == 0) sample_means_warp(z, zs, S, P, zb, zdev, lane);
  for (int64_t c = blockIdx.x; c < p.N; c += gridDim.x) {
    // ---- 1. a, the kernel row and its slope ----
    for (int j = threadIdx.x; j < p.d_pad; j += blockDim.x)
      a_w[j] = j < p.d ? fmaf(__ldg(p.x + c * p.d + j), __ldg(p.cand_scale + j), __ldg(p.cand_shift + j)) : 0.f;
    __syncthreads();
    kernel_row_cta<FAMILY>(a_w, p.train_m2, p.n, p.n_pad, p.d, p.d_pad, p.sf2, k_w, gk_w);
    __syncthreads();
    // ---- 2. v = L^-1 k over row blocks, and k . beta_p ----
    linv_apply_cta(p.linv, p.n_pad, k_w, v_w, P, p.pend_beta, kb_s);
    __syncthreads();
    // ---- 3. one warp: mu, var, c_p, the value and its partials ----
    if (warp == 0) {
      float ka = 0.f;
      for (int i = lane; i < p.n_pad; i += 32) ka = fmaf(k_w[i], __ldg(p.alpha + i), ka);
      ka = warp_sum(ka);
      float vv = 0.f;
      for (int j0 = 0; j0 < p.n_pad; j0 += 32) vv = fmaf(v_w[j0 + lane], v_w[j0 + lane], vv);
      vv = warp_sum(vv);
      const float vt = p.sf2 - vv;
      const bool var_free = vt > 1e-10f;  // the clamp passes no gradient
      const float mu = fmaf(sy, __ldg(p.mean_const) + ka, p.y_mean);
      const float var = sy2 * fmaxf(vt, 1e-10f);
      float cr = 0.f;  // lane q < P: c_q
      if (lane < P) {
        float t = 0.f;
        for (int j = 0; j < p.d; ++j) {
          const float b =
              fmaf(__ldg(p.pend_x + (size_t)lane * p.d + j), __ldg(p.cand_scale + j), __ldg(p.cand_shift + j));
          const float df = a_w[j] - b;
          t = fmaf(df, df, t);
        }
        float k, dk;
        kernel_and_slope<FAMILY>(t, k, dk);
        cr = sy2 * (p.sf2 * k - kb_s[lane]);
        gkp[lane] = 2.f * p.sf2 * dk;
      }
      float value, g_mu, g_var;
      acq_point_partials(a, mu, var, cr, P, p.pend_mu, p.pend_cov, z, zs, S, zb, zdev, w, value, g_mu, g_var, lane);
      if (!var_free) g_var = 0.f;
      if (lane < P) cr_s[lane] = sy2 * w.ac[lane];
      if (lane == 0) {
        sc[0] = sy * g_mu;
        sc[1] = -2.f * sy2 * g_var;
        p.value[c] = value;
      }
    }
    __syncthreads();
    // ---- 4. u = L^-T v over column blocks; k_w[i] <- gk_i dA/dk_i ----
    linvt_fold_cta(p.linv, p.alpha, p.n_pad, v_w, gk_w, sc[0], sc[1], P, p.pend_beta, cr_s, k_w);
    __syncthreads();
    // ---- 5. dA/dx: row groups x columns, then the groups summed in order ----
    row_groups_cta(k_w, a_w, p.train_m2, p.n, p.d, p.d_pad, part);
    for (int j = threadIdx.x; j < p.d; j += blockDim.x) {
      const float g = col_grad_cta(j, k_w, a_w, p.train_m2, p.n, p.d, p.d_pad, part, P, p.pend_x, p.cand_scale,
                                   p.cand_shift, cr_s, gkp);
      p.grad[c * p.d + j] = g * __ldg(p.cand_scale + j);
    }
    __syncthreads();
  }
}

}  // namespace bb

using namespace bb;

extern "C" int bb_acq_grad_large(const bb_model* m, const bb_acq_spec* a, const float* d_x, int64_t N,
                                 int32_t n_pending, const float* d_pend_x, const float* d_pend_beta,
                                 const float* d_pend_mu, const float* d_pend_cov, const float* d_z, int32_t S,
                                 float* d_value, float* d_grad, void* stream) {
  BB_CHECK_ARG(m && m->abi_version == BB_ABI_VERSION, "bb_acq_grad_large: model struct missing or ABI mismatch");
  BB_CHECK_ARG(a != nullptr, "bb_acq_grad_large: acquisition spec is null");
  BB_CHECK_ARG(a->kind >= BB_ACQ_QLOGEI && a->kind <= BB_ACQ_PSTD, "bb_acq_grad_large: acquisition kind %d is not one "
               "of the single-target kinds", a->kind);
  BB_CHECK_SUPPORTED(m->task_col < 0, "bb_acq_grad_large: models with a task parameter are not supported");
  BB_CHECK_SUPPORTED(m->n_pad <= kLargeMaxNPad, "bb_acq_grad_large: n_pad=%d above %d is not supported", m->n_pad,
                     kLargeMaxNPad);
  BB_CHECK_ARG(N >= 0, "bb_acq_grad_large: negative point count");
  const bool is_mc = a->kind <= BB_ACQ_QPI;
  BB_CHECK_ARG(n_pending >= 0 && n_pending <= BB_MAX_PENDING, "bb_acq_grad_large: n_pending=%d outside [0,%d]",
               n_pending, BB_MAX_PENDING);
  BB_CHECK_ARG(n_pending == 0 || is_mc,
               "bb_acq_grad_large: pending points need a Monte Carlo acquisition function");
  BB_CHECK_ARG(!is_mc || (S >= 1 && S <= kMaxSamples), "bb_acq_grad_large: S=%d outside [1,%d]", S, kMaxSamples);
  BB_CHECK_ARG(!is_mc || d_z != nullptr, "bb_acq_grad_large: null base samples");
  BB_CHECK_ARG(n_pending == 0 || (d_pend_x && d_pend_beta && d_pend_mu && d_pend_cov),
               "bb_acq_grad_large: null pending buffer");
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_x && d_value && d_grad, "bb_acq_grad_large: null buffer");
  GradLargeParams p;
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
  p.mean_const = m->d_mean_const;
  p.y_mean = m->y_mean;
  p.y_std = m->y_std;
  p.sf2 = m->prior_scale;  // single task: the prior variance s_f^2
  p.P = n_pending;
  p.pend_x = d_pend_x;
  p.pend_beta = d_pend_beta;
  p.pend_mu = d_pend_mu;
  p.pend_cov = d_pend_cov;
  p.z = d_z;
  p.S = is_mc ? S : 0;
  p.value = d_value;
  p.grad = d_grad;
  int sms, max_smem;
  int rc = device_limits(&sms, &max_smem);
  if (rc != BB_OK) return rc;
  const size_t scratch = (size_t)grad_large_floats(p.n_pad, p.d_pad, n_pending) * 4;
  BB_CHECK_SUPPORTED(scratch <= (size_t)max_smem, "bb_acq_grad_large: d_pad=%d, n_pad=%d and n_pending=%d too large "
                     "for shared memory", p.d_pad, p.n_pad, n_pending);
  const int zs = (n_pending + 1) | 1;
  const size_t z_bytes = (size_t)((p.S * zs + 3) & ~3) * 4;
  // Real shapes leave the base samples in global memory only with d_pad in the tens of thousands;
  // BB_ACQ_GRAD_LARGE_Z_GLOBAL=1 takes that path at any shape, so that tests can hold it to the shared-memory one.
  const char* z_global = getenv("BB_ACQ_GRAD_LARGE_Z_GLOBAL");
  p.z_smem = scratch + z_bytes <= (size_t)max_smem && !(z_global && z_global[0] == '1') ? 1 : 0;
  const size_t smem = scratch + (p.z_smem ? z_bytes : 0);
  int64_t blocks = N;
  if (blocks > (int64_t)sms * 8) blocks = (int64_t)sms * 8;
  return dispatch_family<true>(m->family, [&](auto fam) {
    BB_SMEM_OPTIN_ONCE(k_acq_grad_large<decltype(fam)::value>);
    k_acq_grad_large<decltype(fam)::value><<<(int)blocks, kCtaThreads, smem, (cudaStream_t)stream>>>(p);
    BB_LAUNCH_CHECK();
    return BB_OK;
  });
}
