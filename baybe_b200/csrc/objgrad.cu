// objgrad.cu -- value and gradient of the acquisition value of an objective that is not affine in its targets
// (bb_objective_grad), for the continuous optimiser: the value bb_objective_score reports, and its gradient with
// respect to the raw comp-rep rows.
//
// Per point x, target m (one model each: partial measurements give the models their own n, scaling and
// hyper-parameters) and base sample s, as in objective.cu:
//   y_ms = mu_m + c_m . w_ms + sd_m z_ms,   sd_m = sqrt(max(var_m - |L_m^-1 c_m|^2, 0)),
//   t_ms = program_m(y_ms),   o_s = scalarise(t_s),   A = acquisition over the o_s joined with the pending terms,
// with mu_m, var_m and c_m (the cross covariances with the pending points) formed from x as in grad.cu.
//
// Reverse pass:
//   1. Sample pass (lanes over samples; objective_point_partials in objective_common.cuh, shared with
//      k_objective_grad_large): dA/do_s from the kind's term and the join (qLogEI: the fat terms, the fatmax
//      with tau_max and the logsumexp; the hard max of the other kinds; qUCB also through the sample mean), do/dt_m
//      from the scalariser (GEOM_MEAN: o w_m / (t_m + eps)), dt/dy from the program run on dual numbers (value,
//      d/dy) on the same 4-entry stack as objective.cu's run_program.  Reduced into A_mu[m] = sum_s dA/dy_ms,
//      A_sd[m] = sum_s dA/dy_ms z_ms and A_c[m][p] = sum_s dA/dy_ms w_msp (in chunks of 32 samples: lane p
//      takes column p, so the loads of w coalesce).  Then sd_m takes A_var[m] = A_sd / (2 sd) and
//      A_c[m] -= A_sd L^-T (L^-1 c) / sd.  Kinks follow torch autograd: a clamp passes the gradient on its closed
//      interval, where picks the selected branch and a max gives it to its first maximal entry (the candidate first).
//      The analytic kinds (MEAN over affine targets, no pending points) take analytic_partials on the Gaussian
//      moments sum_m w_m (a_m mu_m + b_m), sum_m (w_m a_m)^2 var_m.
//   2. Per target, back through the kernel row (grad_common.cuh):
//      dA/dk_i = s_y A_mu alpha_i - 2 s_y^2 A_var u_i - s_y^2 sum_p A_c[p] beta_p,i, then dk/dt, then the direct
//      k(x, x_p) term; the gradient is the sum over the targets in target order.
// Each target's a, k, dk/dt and v = L^-1 k stay in the warp's shared scratch from the forward to the reverse pass
// (DESIGN.md section 4.3).  Every reduction has a fixed order and nothing is accumulated atomically: repeated calls
// are bit-identical.
#include <math.h>

#include "fused_common.cuh"
#include "grad_common.cuh"
#include "objective_common.cuh"
#include "score_common.cuh"

namespace bb {

constexpr int kObjGradThreads = 128;  // four points per block
constexpr int kObjGradWarps = kObjGradThreads / 32;

struct ObjGradModel {
  const float *cand_scale, *cand_shift, *train_m2, *alpha, *linv, *mean_const;
  const float* pend_beta;  // [P][n_pad]
  int n, n_pad;
  float y_mean, y_std, sf2;
};

struct ObjGradParams {
  bb_objective obj;
  bb_acq_spec a;
  ObjGradModel mdl[BB_OBJ_MAX_TARGETS];
  int M, d, d_pad, n_pad;  // n_pad: the largest over the targets (the scratch stride)
  const float* x;          // [N][d]
  int64_t N;
  int P;
  const float *pend_x, *plinv, *w, *pend;  // [P][d], [M][P][P], [M][S][P], [S][P]
  const float* z;                          // [S][M(1+P)]
  int S;
  float* value;  // [N]
  float* grad;   // [N][d]
};

// per-warp scratch in floats: per target a | k (then dA/dk_i * dk_i/dt) | gk | v | c | L^-1 c | gkp | A_c, then the
// sample chunk's adjoints [32][M] and 4 x 8 per-target scalars
__host__ __device__ inline int objgrad_warp_floats(int M, int n_pad, int d_pad) {
  return (M * (d_pad + 3 * n_pad + 4 * 32) + 32 * M + 32 + 3) & ~3;
}

template <int FAMILY>
__global__ void __launch_bounds__(kObjGradThreads) k_objective_grad(const __grid_constant__ ObjGradParams p) {
  extern __shared__ __align__(16) float smem_og[];
  const int M = p.M, P = p.P, Q = P + 1;
  const bb_acq_spec& a = p.a;
  const int S = a.kind >= BB_ACQ_UCB ? 0 : p.S;  // analytic kinds take no base samples
  float* zc = smem_og;  // [S][M] candidate base samples
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int np = p.n_pad, dp = p.d_pad;
  float* wb = zc + ((S * M + 3) & ~3) + warp * objgrad_warp_floats(M, np, dp);
  float* a_w = wb;                 // [M][d_pad]
  float* k_w = a_w + M * dp;       // [M][n_pad]
  float* gk_w = k_w + M * np;      // [M][n_pad]
  float* v_w = gk_w + M * np;      // [M][n_pad]
  float* cw = v_w + M * np;        // [M][32] c_m
  float* rw = cw + M * 32;         // [M][32] L_m^-1 c_m
  float* gkp = rw + M * 32;        // [M][32] 2 s_f^2 dk/dt of k(x, x_p)
  float* acw = gkp + M * 32;       // [M][32] A_c[m][p]
  float* gc = acw + M * 32;        // [32][M] dA/dy of the current chunk's samples
  float* sc = gc + 32 * M;         // mu | var | sd | A_var, 8 each
  float* mu_s = sc;
  float* var_s = sc + 8;
  float* sd_s = sc + 16;
  float* gvar_s = sc + 24;
  for (int e = threadIdx.x; e < S * M; e += blockDim.x) {
    const int s = e / M, m = e - s * M;
    zc[e] = __ldg(p.z + (size_t)s * (M * Q) + m * Q + P);
  }
  __syncthreads();
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = warp_global; c < p.N; c += nwarps) {
    // ---- forward, per target: a, k, mu, v, var, c, L^-1 c, sd ----
    float gmu[BB_OBJ_MAX_TARGETS];
    bool vfree[BB_OBJ_MAX_TARGETS];
#pragma unroll
    for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
      vfree[m] = false;
      if (m >= M) continue;
      const ObjGradModel& md = p.mdl[m];
      float* am = a_w + m * dp;
      float* km = k_w + m * np;
      float* gkm = gk_w + m * np;
      float* vm = v_w + m * np;
      for (int j = lane; j < dp; j += 32)
        am[j] = j < p.d ? fmaf(__ldg(p.x + c * p.d + j), __ldg(md.cand_scale + j), __ldg(md.cand_shift + j)) : 0.f;
      __syncwarp();
      const float ka = warp_sum(kernel_row_warp<FAMILY>(am, md.train_m2, md.alpha, md.n, md.n_pad, p.d, dp, md.sf2, km,
                                                        gkm, lane));
      __syncwarp();
      const float vv = warp_sum(linv_apply_warp(md.linv, md.n_pad, km, vm, lane));
      const float sy = md.y_std, sy2 = sy * sy;
      const float vt = md.sf2 - vv;
      vfree[m] = vt > 1e-10f;  // the clamp passes no gradient
      const float mu = fmaf(sy, __ldg(md.mean_const) + ka, md.y_mean);
      const float var = sy2 * fmaxf(vt, 1e-10f);
      float cr = 0.f;  // lane q < P: c_q
      for (int q = 0; q < P; ++q) {
        float kb = 0.f;
        for (int i = lane; i < md.n_pad; i += 32) kb = fmaf(km[i], __ldg(md.pend_beta + (size_t)q * md.n_pad + i), kb);
        kb = warp_sum(kb);
        if (lane == q) cr = kb;
      }
      float g = 0.f;
      if (lane < P) {
        float t = 0.f;
        for (int j = 0; j < p.d; ++j) {
          const float b = fmaf(__ldg(p.pend_x + (size_t)lane * p.d + j), __ldg(md.cand_scale + j),
                               __ldg(md.cand_shift + j));
          const float df = am[j] - b;
          t = fmaf(df, df, t);
        }
        float k, dk;
        kernel_and_slope<FAMILY>(t, k, dk);
        cr = sy2 * (md.sf2 * k - cr);
        g = 2.f * md.sf2 * dk;
      }
      cw[m * 32 + lane] = lane < P ? cr : 0.f;
      gkp[m * 32 + lane] = g;
      acw[m * 32 + lane] = 0.f;
      // r = L^-1 c (lane i: r_i), as pending_r2_warp forms it
      const float* Lm = p.plinv + (size_t)m * P * P;
      float r = 0.f;
      for (int k = 0; k < P; ++k) {
        const float ck = __shfl_sync(kFull, cr, k);
        if (lane < P && k <= lane) r = fmaf(__ldg(Lm + lane * P + k), ck, r);
      }
      rw[m * 32 + lane] = lane < P ? r : 0.f;
      const float r2 = warp_sum(lane < P ? r * r : 0.f);
      if (lane == 0) {
        mu_s[m] = mu;
        var_s[m] = var;
        sd_s[m] = P > 0 ? sqrtf(fmaxf(var - r2, 0.f)) : sqrtf(var);
        gvar_s[m] = 0.f;
      }
      __syncwarp();
    }
    // ---- the value and its partials A_mu, A_var, A_c (objective_common.cuh) ----
    const float value = objective_point_partials(p.obj, a, M, P, S, zc, p.w, p.pend, p.plinv, mu_s, var_s, sd_s, cw, rw,
                                                 acw, gc, gvar_s, gmu, lane);
    // ---- per target: dA/dk_i folded with dk_i/dt into k_w, then the gradient (lanes over columns) ----
#pragma unroll
    for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
      if (m >= M) continue;
      const ObjGradModel& md = p.mdl[m];
      const float sy = md.y_std, sy2 = sy * sy;
      const float gv = vfree[m] ? gvar_s[m] : 0.f;
      const float k_mu = sy * gmu[m], k_var = -2.f * sy2 * gv;
      float* km = k_w + m * np;
      const float* gkm = gk_w + m * np;
      const float* vm = v_w + m * np;
      for (int i0 = 0; i0 < md.n_pad; i0 += 32) {
        const int i = i0 + lane;
        const float u = linvt_apply_col(md.linv, md.n_pad, vm, i0, i);
        float kb = fmaf(k_mu, __ldg(md.alpha + i), k_var * u);
        for (int q = 0; q < P; ++q) kb = fmaf(-sy2 * acw[m * 32 + q], __ldg(md.pend_beta + (size_t)q * md.n_pad + i), kb);
        km[i] = gkm[i] * kb;
      }
    }
    __syncwarp();
    for (int j = lane; j < p.d; j += 32) {
      float gsum = 0.f;
      for (int m = 0; m < M; ++m) {
        const ObjGradModel& md = p.mdl[m];
        const float sy2 = md.y_std * md.y_std;
        const float aj = a_w[m * dp + j];
        const float* km = k_w + m * np;
        float g = 0.f;
        for (int i = 0; i < md.n; ++i) g = fmaf(km[i], aj + 0.5f * __ldg(md.train_m2 + (size_t)i * dp + j), g);
        for (int q = 0; q < P; ++q) {
          const float b = fmaf(__ldg(p.pend_x + (size_t)q * p.d + j), __ldg(md.cand_scale + j), __ldg(md.cand_shift + j));
          g = fmaf(sy2 * acw[m * 32 + q] * gkp[m * 32 + q], aj - b, g);
        }
        gsum = fmaf(g, __ldg(md.cand_scale + j), gsum);
      }
      p.grad[c * p.d + j] = gsum;
    }
    if (lane == 0) p.value[c] = value;
    __syncwarp();
  }
}

}  // namespace bb

using namespace bb;

extern "C" int bb_objective_grad(const bb_model* const* models, int32_t n_targets, const bb_acq_spec* a,
                                 const bb_objective* obj, const float* d_x, int64_t N, int32_t n_pending,
                                 const float* d_pend_x, const float* const* d_pend_beta, const float* d_linv,
                                 const float* d_w, const float* d_pend_terms, const float* d_z, int32_t S,
                                 float* d_value, float* d_grad, void* stream) {
  static const char* fn = "bb_objective_grad";
  BB_CHECK_ARG(models != nullptr, "bb_objective_grad: model array is null");
  BB_CHECK_SUPPORTED(n_targets >= 1 && n_targets <= BB_OBJ_MAX_TARGETS, "bb_objective_grad: n_targets=%d outside [1,%d]",
                     n_targets, BB_OBJ_MAX_TARGETS);
  BB_CHECK_ARG(a != nullptr, "bb_objective_grad: acquisition spec is null");
  BB_CHECK_ARG(obj != nullptr, "bb_objective_grad: objective is null");
  BB_CHECK_ARG(obj->n_targets == n_targets, "bb_objective_grad: objective of %d targets for %d models", obj->n_targets,
               n_targets);
  const int M = n_targets;
  for (int m = 0; m < M; ++m) {
    const bb_model* md = models[m];
    BB_CHECK_ARG(md && md->abi_version == BB_ABI_VERSION, "bb_objective_grad: model %d missing or ABI mismatch", m);
    BB_CHECK_SUPPORTED(!md->wide, "bb_objective_grad: model %d: wide-feature models are not supported", m);
    BB_CHECK_SUPPORTED(md->task_col < 0, "bb_objective_grad: model %d: models with a task parameter are not supported",
                       m);
    BB_CHECK_SUPPORTED(md->n_pad <= kGradMaxNPad, "bb_objective_grad: model %d: n_pad=%d above %d is not supported", m,
                       md->n_pad, kGradMaxNPad);
    BB_CHECK_ARG(md->d == models[0]->d && md->d_pad == models[0]->d_pad && md->family == models[0]->family,
                 "bb_objective_grad: model %d differs from model 0 in d or kernel family", m);
  }
  const int rc_obj = check_objective(fn, a, obj);
  if (rc_obj != BB_OK) return rc_obj;
  const bool analytic = a->kind >= BB_ACQ_UCB;
  BB_CHECK_ARG(N >= 0, "bb_objective_grad: negative point count");
  BB_CHECK_ARG(n_pending >= 0 && n_pending <= BB_MAX_PENDING, "bb_objective_grad: n_pending=%d outside [0,%d]",
               n_pending, BB_MAX_PENDING);
  BB_CHECK_ARG(!analytic || n_pending == 0, "bb_objective_grad: analytic kinds take no pending points");
  BB_CHECK_ARG(analytic || (S >= 1 && S <= kMaxSamples), "bb_objective_grad: S=%d outside [1,%d]", S, kMaxSamples);
  BB_CHECK_ARG(analytic || d_z != nullptr, "bb_objective_grad: null base samples");
  bool pend_ok = n_pending == 0 || (d_pend_x && d_pend_beta && d_linv && d_w && d_pend_terms);
  for (int m = 0; pend_ok && n_pending > 0 && m < M; ++m) pend_ok = d_pend_beta[m] != nullptr;
  BB_CHECK_ARG(pend_ok, "bb_objective_grad: pending points need rows, beta per model, linv, w and pending terms");
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_x && d_value && d_grad, "bb_objective_grad: null buffer");
  ObjGradParams p;
  p.obj = *obj;
  p.a = *a;
  p.M = M;
  p.d = models[0]->d;
  p.d_pad = models[0]->d_pad;
  p.n_pad = 0;
  for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
    ObjGradModel& g = p.mdl[m];
    g = ObjGradModel{};
    if (m >= M) continue;
    const bb_model* md = models[m];
    g.cand_scale = md->d_cand_scale;
    g.cand_shift = md->d_cand_shift;
    g.train_m2 = md->d_train_m2;
    g.alpha = md->d_alpha;
    g.linv = md->d_linv32;
    g.mean_const = md->d_mean_const;
    g.pend_beta = n_pending > 0 ? d_pend_beta[m] : nullptr;
    g.n = md->n;
    g.n_pad = md->n_pad;
    g.y_mean = md->y_mean;
    g.y_std = md->y_std;
    g.sf2 = md->prior_scale;  // single task: the prior variance s_f^2
    p.n_pad = md->n_pad > p.n_pad ? md->n_pad : p.n_pad;
  }
  p.x = d_x;
  p.N = N;
  p.P = n_pending;
  p.pend_x = d_pend_x;
  p.plinv = d_linv;
  p.w = d_w;
  p.pend = d_pend_terms;
  p.z = d_z;
  p.S = analytic ? 0 : S;
  p.value = d_value;
  p.grad = d_grad;
  int sms, max_smem;
  int rc = device_limits(&sms, &max_smem);
  if (rc != BB_OK) return rc;
  const size_t smem = ((size_t)((p.S * M + 3) & ~3) + (size_t)kObjGradWarps * objgrad_warp_floats(M, p.n_pad, p.d_pad)) *
                      4;
  BB_CHECK_SUPPORTED(smem <= (size_t)max_smem, "bb_objective_grad: %zu bytes of shared memory above %d", smem,
                     max_smem);
  int64_t blocks = (N + kObjGradWarps - 1) / kObjGradWarps;
  if (blocks > (int64_t)sms * 8) blocks = (int64_t)sms * 8;
  return dispatch_family<true>(models[0]->family, [&](auto fam) {
    BB_SMEM_OPTIN_ONCE(k_objective_grad<decltype(fam)::value>);
    k_objective_grad<decltype(fam)::value><<<(int)blocks, kObjGradThreads, smem, (cudaStream_t)stream>>>(p);
    BB_LAUNCH_CHECK();
    return BB_OK;
  });
}
