// objgradlarge.cu -- value and gradient of the acquisition value of an objective that is not affine in its targets
// (bb_objective_grad_large) for any mix of single-task models: n_pad up to 1024 and wide-feature models, which
// bb_objective_grad (objgrad.cu) does not take.
//
// It computes what bb_objective_grad computes (see objgrad.cu for the formulas), with gradlarge.cu's mapping: one CTA
// of 256 threads per point, grid-striding over the points.  Per point:
//   1. For each target in target order: the CTA forms a = x scale + shift, the kernel row k and its slope gk
//      (kernel_row_cta), then v = L^-1 k over snake-ordered row blocks and k . beta_p (linv_apply_cta); one warp then
//      forms mu, var, c_p, L_PP^-1 c and sd as k_objective_grad does.  k is dropped after this step (one buffer
//      serves every target); gk and v stay for the reverse pass.
//   2. One warp runs the sample pass (or the analytic partials): objective_point_partials (objective_common.cuh), the
//      same function k_objective_grad calls, for the value, A_mu[m], A_var[m] and A_c[m][p].
//   3. For each target: u = L^-T v over snake-ordered column blocks folded into gk dA/dk (linvt_fold_cta), then the
//      reverse pass to dA/dx (row_groups_cta, col_grad_cta), added into the gradient in target order.
// Every per-element sum of steps 1 and 2 runs in k_objective_grad's order, so on the shapes both take (d < 32,
// n_pad <= 256) the values agree bit for bit.  The candidate's base samples [S][M] sit in shared memory.  No float
// atomics: repeated calls are bit-identical.
#include <math.h>

#include "fused_common.cuh"
#include "grad_common.cuh"
#include "objective_common.cuh"

namespace bb {

struct ObjGradLargeModel {
  const float *cand_scale, *cand_shift, *train_m2, *alpha, *linv, *mean_const;
  const float* pend_beta;  // [P][n_pad]
  int n, n_pad, off;       // off: the model's offset in the gk and v scratch (the n_pad of the targets before it)
  float y_mean, y_std, sf2;
};

struct ObjGradLargeParams {
  bb_objective obj;
  bb_acq_spec a;
  ObjGradLargeModel mdl[BB_OBJ_MAX_TARGETS];
  int M, d, d_pad;
  int n_max, n_sum;  // the largest n_pad and the sum of the n_pad over the targets
  const float* x;    // [N][d]
  int64_t N;
  int P;
  const float *pend_x, *plinv, *w, *pend;  // [P][d], [M][P][P], [M][S][P], [S][P]
  const float* z;                          // [S][M(1+P)]
  int S;
  float* value;  // [N]
  float* grad;   // [N][d]
};

// per-CTA scratch in floats: the candidate's base samples [S][M] | k (then gk dA/dk) [n_max] | dA/dx [d_pad] | the
// column-gradient partials [kCtaThreads] | c, L^-1 c, gkp, A_c (then s_y^2 A_c) [M][32] | k . beta_p [32] | the sample
// chunk's adjoints [32][M] | mu, var, sd, A_var, A_mu, free variance [8] each | a [M][d_pad] | gk, v [n_sum] each
__host__ __device__ inline size_t objgrad_large_floats(int M, int S, int n_max, int n_sum, int d_pad) {
  return (size_t)((S * M + 3) & ~3) + n_max + d_pad + kCtaThreads + 4 * 32 * M + 32 + 32 * M + 48 +
         (size_t)M * d_pad + 2 * (size_t)n_sum;
}

template <int FAMILY>
__global__ void __launch_bounds__(kCtaThreads) k_objective_grad_large(const __grid_constant__ ObjGradLargeParams p) {
  extern __shared__ __align__(16) float smem_ol[];
  const int M = p.M, P = p.P, Q = P + 1;
  const bb_acq_spec& a = p.a;
  const int S = a.kind >= BB_ACQ_UCB ? 0 : p.S;  // analytic kinds take no base samples
  const int dp = p.d_pad;
  float* zc = smem_ol;                        // [S][M] candidate base samples
  float* k_w = zc + ((S * M + 3) & ~3);       // [n_max] the current target's kernel row, then gk dA/dk
  float* gacc = k_w + p.n_max;                // [d_pad] dA/dx summed over the targets
  float* part = gacc + dp;                    // [kCtaThreads]
  float* cw = part + kCtaThreads;             // [M][32] c_m
  float* rw = cw + M * 32;                    // [M][32] L_m^-1 c_m
  float* gkp = rw + M * 32;                   // [M][32] 2 s_f^2 dk/dt of k(x, x_p)
  float* acw = gkp + M * 32;                  // [M][32] A_c[m][p], then s_y^2 A_c[m][p]
  float* kb_s = acw + M * 32;                 // [32] k . beta_p of the current target
  float* gc = kb_s + 32;                      // [32][M]
  float* sc = gc + 32 * M;                    // mu | var | sd | A_var | A_mu | free variance, 8 each; after
                                              // step 2 A_var -> -2 s_y^2 A_var, A_mu -> s_y A_mu
  float* a_w = sc + 48;                       // [M][d_pad]
  float* gk_w = a_w + M * dp;                 // [n_sum]
  float* v_w = gk_w + p.n_sum;                // [n_sum]
  float* mu_s = sc;
  float* var_s = sc + 8;
  float* sd_s = sc + 16;
  float* gvar_s = sc + 24;
  float* gmu_s = sc + 32;
  float* vfree_s = sc + 40;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int e = threadIdx.x; e < S * M; e += blockDim.x) {
    const int s = e / M, m = e - s * M;
    zc[e] = __ldg(p.z + (size_t)s * (M * Q) + m * Q + P);
  }
  for (int64_t c = blockIdx.x; c < p.N; c += gridDim.x) {
    // ---- 1. forward, per target: a, k, gk, v, then (one warp) mu, var, c, L^-1 c, sd ----
    for (int m = 0; m < M; ++m) {
      const ObjGradLargeModel& md = p.mdl[m];
      float* am = a_w + m * dp;
      float* gkm = gk_w + md.off;
      float* vm = v_w + md.off;
      for (int j = threadIdx.x; j < dp; j += blockDim.x)
        am[j] = j < p.d ? fmaf(__ldg(p.x + c * p.d + j), __ldg(md.cand_scale + j), __ldg(md.cand_shift + j)) : 0.f;
      __syncthreads();  // also: warp 0 is done with the previous target's k and k . beta_p
      kernel_row_cta<FAMILY>(am, md.train_m2, md.n, md.n_pad, p.d, dp, md.sf2, k_w, gkm);
      __syncthreads();
      linv_apply_cta(md.linv, md.n_pad, k_w, vm, P, md.pend_beta, kb_s);
      __syncthreads();
      if (warp == 0) {
        float ka = 0.f;
        for (int i = lane; i < md.n_pad; i += 32) ka = fmaf(k_w[i], __ldg(md.alpha + i), ka);
        ka = warp_sum(ka);
        float vv = 0.f;
        for (int j0 = 0; j0 < md.n_pad; j0 += 32) vv = fmaf(vm[j0 + lane], vm[j0 + lane], vv);
        vv = warp_sum(vv);
        const float sy = md.y_std, sy2 = sy * sy;
        const float vt = md.sf2 - vv;
        const float mu = fmaf(sy, __ldg(md.mean_const) + ka, md.y_mean);
        const float var = sy2 * fmaxf(vt, 1e-10f);
        float cr = 0.f, g = 0.f;  // lane q < P: c_q
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
          cr = sy2 * (md.sf2 * k - kb_s[lane]);
          g = 2.f * md.sf2 * dk;
        }
        cw[m * 32 + lane] = lane < P ? cr : 0.f;
        gkp[m * 32 + lane] = g;
        acw[m * 32 + lane] = 0.f;
        // r = L^-1 c (lane i: r_i), as k_objective_grad forms it
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
          vfree_s[m] = vt > 1e-10f ? 1.f : 0.f;  // the clamp passes no gradient
        }
        __syncwarp();
      }
    }
    __syncthreads();
    // ---- 2. one warp: the value and its partials A_mu, A_var, A_c ----
    if (warp == 0) {
      float gmu[BB_OBJ_MAX_TARGETS];
      const float value = objective_point_partials(p.obj, a, M, P, S, zc, p.w, p.pend, p.plinv, mu_s, var_s, sd_s, cw,
                                                   rw, acw, gc, gvar_s, gmu, lane);
      __syncwarp();
      for (int m = 0; m < M; ++m) {
        const float sy = p.mdl[m].y_std, sy2 = sy * sy;
        if (lane < P) acw[m * 32 + lane] *= sy2;
        if (lane == 0) {
          gmu_s[m] = sy * gmu[m];
          gvar_s[m] = vfree_s[m] != 0.f ? -2.f * sy2 * gvar_s[m] : 0.f;
        }
      }
      if (lane == 0) p.value[c] = value;
    }
    __syncthreads();
    // ---- 3. per target: u = L^-T v folded into gk dA/dk, then dA/dx added in target order ----
    for (int m = 0; m < M; ++m) {
      const ObjGradLargeModel& md = p.mdl[m];
      const float* am = a_w + m * dp;
      linvt_fold_cta(md.linv, md.alpha, md.n_pad, v_w + md.off, gk_w + md.off, gmu_s[m], gvar_s[m], P, md.pend_beta,
                     acw + m * 32, k_w);
      __syncthreads();
      row_groups_cta(k_w, am, md.train_m2, md.n, p.d, dp, part);
      for (int j = threadIdx.x; j < p.d; j += blockDim.x) {
        const float g = col_grad_cta(j, k_w, am, md.train_m2, md.n, p.d, dp, part, P, p.pend_x, md.cand_scale,
                                     md.cand_shift, acw + m * 32, gkp + m * 32);
        gacc[j] = fmaf(g, __ldg(md.cand_scale + j), m == 0 ? 0.f : gacc[j]);
      }
      __syncthreads();  // the next target overwrites k and the partials
    }
    for (int j = threadIdx.x; j < p.d; j += blockDim.x) p.grad[c * p.d + j] = gacc[j];
  }
}

}  // namespace bb

using namespace bb;

extern "C" int bb_objective_grad_large(const bb_model* const* models, int32_t n_targets, const bb_acq_spec* a,
                                       const bb_objective* obj, const float* d_x, int64_t N, int32_t n_pending,
                                       const float* d_pend_x, const float* const* d_pend_beta, const float* d_linv,
                                       const float* d_w, const float* d_pend_terms, const float* d_z, int32_t S,
                                       float* d_value, float* d_grad, void* stream) {
  static const char* fn = "bb_objective_grad_large";
  BB_CHECK_ARG(models != nullptr, "bb_objective_grad_large: model array is null");
  BB_CHECK_SUPPORTED(n_targets >= 1 && n_targets <= BB_OBJ_MAX_TARGETS,
                     "bb_objective_grad_large: n_targets=%d outside [1,%d]", n_targets, BB_OBJ_MAX_TARGETS);
  BB_CHECK_ARG(a != nullptr, "bb_objective_grad_large: acquisition spec is null");
  BB_CHECK_ARG(obj != nullptr, "bb_objective_grad_large: objective is null");
  BB_CHECK_ARG(obj->n_targets == n_targets, "bb_objective_grad_large: objective of %d targets for %d models",
               obj->n_targets, n_targets);
  const int M = n_targets;
  for (int m = 0; m < M; ++m) {
    const bb_model* md = models[m];
    BB_CHECK_ARG(md && md->abi_version == BB_ABI_VERSION, "bb_objective_grad_large: model %d missing or ABI mismatch",
                 m);
    BB_CHECK_SUPPORTED(md->task_col < 0,
                       "bb_objective_grad_large: model %d: models with a task parameter are not supported", m);
    BB_CHECK_SUPPORTED(md->n_pad <= BB_MAX_TRAIN, "bb_objective_grad_large: model %d: n_pad=%d above %d is not "
                       "supported", m, md->n_pad, BB_MAX_TRAIN);
    BB_CHECK_ARG(md->d == models[0]->d && md->d_pad == models[0]->d_pad && md->family == models[0]->family,
                 "bb_objective_grad_large: model %d differs from model 0 in d or kernel family", m);
  }
  const int rc_obj = check_objective(fn, a, obj);
  if (rc_obj != BB_OK) return rc_obj;
  const bool analytic = a->kind >= BB_ACQ_UCB;
  BB_CHECK_ARG(N >= 0, "bb_objective_grad_large: negative point count");
  BB_CHECK_ARG(n_pending >= 0 && n_pending <= BB_MAX_PENDING, "bb_objective_grad_large: n_pending=%d outside [0,%d]",
               n_pending, BB_MAX_PENDING);
  BB_CHECK_ARG(!analytic || n_pending == 0, "bb_objective_grad_large: analytic kinds take no pending points");
  BB_CHECK_ARG(analytic || (S >= 1 && S <= kMaxSamples), "bb_objective_grad_large: S=%d outside [1,%d]", S,
               kMaxSamples);
  BB_CHECK_ARG(analytic || d_z != nullptr, "bb_objective_grad_large: null base samples");
  bool pend_ok = n_pending == 0 || (d_pend_x && d_pend_beta && d_linv && d_w && d_pend_terms);
  for (int m = 0; pend_ok && n_pending > 0 && m < M; ++m) pend_ok = d_pend_beta[m] != nullptr;
  BB_CHECK_ARG(pend_ok, "bb_objective_grad_large: pending points need rows, beta per model, linv, w and pending terms");
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_x && d_value && d_grad, "bb_objective_grad_large: null buffer");
  ObjGradLargeParams p;
  p.obj = *obj;
  p.a = *a;
  p.M = M;
  p.d = models[0]->d;
  p.d_pad = models[0]->d_pad;
  p.n_max = 0;
  p.n_sum = 0;
  for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
    ObjGradLargeModel& g = p.mdl[m];
    g = ObjGradLargeModel{};
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
    g.off = p.n_sum;
    g.y_mean = md->y_mean;
    g.y_std = md->y_std;
    g.sf2 = md->prior_scale;  // single task: the prior variance s_f^2
    p.n_max = md->n_pad > p.n_max ? md->n_pad : p.n_max;
    p.n_sum += md->n_pad;
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
  const size_t smem = objgrad_large_floats(M, p.S, p.n_max, p.n_sum, p.d_pad) * 4;
  BB_CHECK_SUPPORTED(smem <= (size_t)max_smem, "bb_objective_grad_large: M=%d targets with n_pad up to %d (%d in all), "
                     "d_pad=%d and P=%d need %zu bytes of shared memory, above %d", M, p.n_max, p.n_sum, p.d_pad,
                     n_pending, smem, max_smem);
  int64_t blocks = N;
  if (blocks > (int64_t)sms * 8) blocks = (int64_t)sms * 8;
  return dispatch_family<true>(models[0]->family, [&](auto fam) {
    BB_SMEM_OPTIN_ONCE(k_objective_grad_large<decltype(fam)::value>);
    k_objective_grad_large<decltype(fam)::value><<<(int)blocks, kCtaThreads, smem, (cudaStream_t)stream>>>(p);
    BB_LAUNCH_CHECK();
    return BB_OK;
  });
}
