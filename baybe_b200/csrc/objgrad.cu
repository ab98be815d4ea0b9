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
//   1. Sample pass (lanes over samples): dA/do_s from the kind's term and the join (qLogEI: the fat terms, the fatmax
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
constexpr float kObjGeomEps = 2.220446049250313e-16f;  // as objective.cu

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

// The program of objective.cu's run_program on dual numbers: returns t, and dt/dy in dt.
__device__ __forceinline__ float run_program_dual(const bb_obj_instr* prog, int n, float y, float& dt) {
  float x = y, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  float dx = 1.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;
  for (int i = 0; i < n; ++i) {
    const int op = prog[i].op;
    const float a0 = prog[i].arg[0], a1 = prog[i].arg[1], a2 = prog[i].arg[2];
    switch (op) {
      case BB_OBJ_AFFINE:
        x = fmaf(x, a0, a1);
        dx *= a0;
        break;
      case BB_OBJ_CONST:
        x = a0;
        dx = 0.f;
        break;
      case BB_OBJ_CLAMP:  // the gradient passes on the closed interval, like torch.clamp
        if (x < a0) {
          x = a0;
          dx = 0.f;
        } else if (x > a1) {
          x = a1;
          dx = 0.f;
        }
        break;
      case BB_OBJ_TWO_SIDED: {
        const float d = x - a2;
        const bool left = x < a2;
        const float sl = left ? a0 : a1;
        x = sl != 0.f ? d * sl : 0.f;
        dx = sl != 0.f ? dx * sl : 0.f;
        break;
      }
      case BB_OBJ_BELL: {
        const float u = (x - a0) / a1;
        x = expf(-(u * u) * 0.5f);
        dx *= -x * u / a1;
        break;
      }
      case BB_OBJ_LOG:
        dx /= x;
        x = logf(x);
        break;
      case BB_OBJ_EXP:
        x = expf(x);
        dx *= x;
        break;
      case BB_OBJ_POW_INT:  // torch's pow backward: exponent * x^(exponent - 1), zero for exponent 0
        dx = a0 != 0.f ? dx * a0 * powf(x, a0 - 1.f) : 0.f;
        x = powf(x, a0);
        break;
      case BB_OBJ_SIGMOID: {
        const float e = expf(a1 * (x - a0));
        x = 1.0f / (1.0f + e);
        dx *= isinf(e) ? 0.f : -a1 * e / ((1.f + e) * (1.f + e));
        break;
      }
      case BB_OBJ_DUP_INPUT:
        s3 = s2;
        s2 = s1;
        s1 = x;
        d3 = d2;
        d2 = d1;
        d1 = dx;
        x = y;
        dx = 1.f;
        break;
      case BB_OBJ_ADD:
        x = s1 + x;
        dx = d1 + dx;
        s1 = s2;
        s2 = s3;
        d1 = d2;
        d2 = d3;
        break;
      default:  // BB_OBJ_MUL (opcodes are validated on the host)
        dx = fmaf(d1, x, s1 * dx);
        x = s1 * x;
        s1 = s2;
        s2 = s3;
        d1 = d2;
        d2 = d3;
        break;
    }
  }
  dt = dx;
  return x;
}

template <int FAMILY>
__global__ void __launch_bounds__(kObjGradThreads) k_objective_grad(const __grid_constant__ ObjGradParams p) {
  extern __shared__ __align__(16) float smem_og[];
  const int M = p.M, P = p.P, Q = P + 1;
  const bb_acq_spec& a = p.a;
  const int kind = a.kind;
  const bool analytic = kind >= BB_ACQ_UCB;
  const int S = analytic ? 0 : p.S;
  const int scal = p.obj.scalarizer;
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
  const float ucb_c = sqrtf(a.beta * 1.5707963267948966f);
  const float inv_relu = 1.0f / a.tau_relu;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = warp_global; c < p.N; c += nwarps) {
    // ---- forward, per target: a, k, mu, v, var, c, L^-1 c, sd ----
    float gmu[BB_OBJ_MAX_TARGETS];
    bool vfree[BB_OBJ_MAX_TARGETS];
#pragma unroll
    for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
      gmu[m] = 0.f;
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
    float value;
    if (analytic) {
      // MEAN over affine targets: the scalarised posterior is Gaussian (objective.cu)
      float mean = 0.f, var = 0.f;
#pragma unroll
      for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
        if (m < M) {
          const bool aff = p.obj.n_ops[m] > 0;
          const float am = p.obj.weight[m] * (aff ? p.obj.prog[m][0].arg[0] : 1.0f);
          const float bm = p.obj.weight[m] * (aff ? p.obj.prog[m][0].arg[1] : 0.0f);
          mean += fmaf(am, mu_s[m], bm);
          var = fmaf(am * am, var_s[m], var);
        }
      }
      bb_acq_spec u = a;
      u.obj_scale = 1.0f;
      u.obj_shift = 0.0f;
      value = analytic_value(u, mean, var);
      double dmu, dsd;
      analytic_partials(u, mean, var, dmu, dsd);
      const float dvar = (float)(dsd / (2.0 * sqrt((double)var)));
#pragma unroll
      for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
        if (m < M) {
          const bool aff = p.obj.n_ops[m] > 0;
          const float am = p.obj.weight[m] * (aff ? p.obj.prog[m][0].arg[0] : 1.0f);
          gmu[m] = (float)dmu * am;
          if (lane == 0) gvar_s[m] = dvar * am * am;
        }
      }
      __syncwarp();
    } else {
      // the objective of sample s (valid s only) and do/dy_m
      auto sample_o = [&](int s, float (&dody)[BB_OBJ_MAX_TARGETS]) -> float {
        float acc = 0.f, o = 0.f;
        float tt[BB_OBJ_MAX_TARGETS];
#pragma unroll
        for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
          tt[m] = 0.f;
          dody[m] = 0.f;
          if (m < M) {
            float dm = 0.f;
            const float* wr = p.w + ((size_t)m * S + s) * P;
            for (int j = 0; j < P; ++j) dm = fmaf(cw[m * 32 + j], __ldg(wr + j), dm);
            const float y = mu_s[m] + dm + sd_s[m] * zc[s * M + m];
            float dt;
            const float t = run_program_dual(p.obj.prog[m], p.obj.n_ops[m], y, dt);
            tt[m] = t;
            dody[m] = dt;
            if (scal == BB_OBJ_SCALAR_NONE) o = t;
            else if (scal == BB_OBJ_SCALAR_MEAN) acc = fmaf(p.obj.weight[m], t, acc);
            else acc = fmaf(p.obj.weight[m], logf(t + kObjGeomEps), acc);
          }
        }
        if (scal == BB_OBJ_SCALAR_MEAN) o = acc;
        else if (scal == BB_OBJ_SCALAR_GEOM_MEAN) o = expf(acc);
#pragma unroll
        for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
          if (scal == BB_OBJ_SCALAR_MEAN) dody[m] *= p.obj.weight[m];
          else if (scal == BB_OBJ_SCALAR_GEOM_MEAN) dody[m] *= o * p.obj.weight[m] / (tt[m] + kObjGeomEps);
        }
        return o;
      };
      // the candidate's term of a sample and its derivative d(term)/do (qUCB: the direct part)
      auto term_of = [&](float o, float mo, float& dterm) -> float {
        if (kind == BB_ACQ_QLOGEI) {
          dterm = dlog_fatplus_t((o - a.best_f) * inv_relu) * inv_relu;
          return logf(a.tau_relu) + log_fatplus_t((o - a.best_f) * inv_relu);
        }
        if (kind == BB_ACQ_QEI) {
          dterm = o - a.best_f >= 0.f ? 1.f : 0.f;
          return fmaxf(o - a.best_f, 0.f);
        }
        if (kind == BB_ACQ_QSR) {
          dterm = 1.f;
          return o;
        }
        if (kind == BB_ACQ_QPI) {
          dterm = dsigmoidf_((o - a.best_f) / a.tau_pi) / a.tau_pi;
          return 1.0f / (1.0f + __expf(-(o - a.best_f) / a.tau_pi));
        }
        const float sg = o > mo ? 1.f : (o < mo ? -1.f : 0.f);
        dterm = ucb_c * sg;
        return mo + ucb_c * fabsf(o - mo);
      };
      // the candidate's share of the join of its term with the pending terms: dA/d(term) up to the sample weight
      float li_arr[BB_MAX_PENDING + 1];
      auto join_share = [&](float term, int s, float& joined) -> float {
        joined = join_terms(term, p.pend + (size_t)s * P, P, li_arr, kind == BB_ACQ_QLOGEI, a.tau_max);
        float mx = term;
        for (int j = 1; j <= P; ++j) mx = fmaxf(mx, li_arr[j]);
        const bool first = term >= mx;  // the candidate comes first among equal maxima
        if (kind != BB_ACQ_QLOGEI) return first ? 1.f : 0.f;
        const float inv = 1.0f / (2.0f * a.tau_max);
        float ssum = 0.f, rest = 0.f;
        for (int k = 0; k <= P; ++k) {
          const float wk = fmaf(mx - li_arr[k], inv, 1.0f);
          ssum += 1.0f / (wk * wk);
        }
        for (int k = 0; k <= P; ++k) {
          const float wk = fmaf(mx - li_arr[k], inv, 1.0f);
          rest += 1.0f / (wk * wk * wk) / ssum;
        }
        const float w0 = fmaf(mx - term, inv, 1.0f);
        return 1.0f / (w0 * w0 * w0) / ssum + (first ? 1.f - rest : 0.f);
      };
      float dody[BB_OBJ_MAX_TARGETS];
      float mo = 0.f;  // qUCB: the sample mean of o
      if (kind == BB_ACQ_QUCB) {
        float so = 0.f;
        for (int s = lane; s < S; s += 32) so += sample_o(s, dody);
        mo = warp_sum(so) / (float)S;
      }
      // pass 1: the value, as k_objective forms it (qUCB: also the weight its sample mean carries)
      float s0a = 0.f, s1a = 0.f, run_max = -INFINITY, run_sum = 0.f, kmo = 0.f;
      for (int s = lane; s < S; s += 32) {
        const float o = sample_o(s, dody);
        if (kind == BB_ACQ_QLOGEI && P == 0) {
          mc_term<BB_ACQ_QLOGEI>((o - a.best_f) * inv_relu, s0a, s1a);
          continue;
        }
        float dterm, joined;
        const float term = term_of(o, mo, dterm);
        const float share = join_share(term, s, joined);
        if (kind == BB_ACQ_QLOGEI) lse_push(joined, run_max, run_sum);
        else s0a += joined;
        if (kind == BB_ACQ_QUCB) kmo += share * (1.f - dterm);
      }
      float lse = 0.f, norm = 1.f / (float)S;
      if (kind == BB_ACQ_QLOGEI && P == 0) {
        s0a = warp_sum(s0a);
        s1a = warp_sum(s1a);
        value = logf(a.tau_relu) + logf((s0a + 0.1f * s1a) / (float)S);
        norm = 1.f / (s0a + 0.1f * s1a);
      } else if (kind == BB_ACQ_QLOGEI) {
        lse_warp_combine(run_max, run_sum);
        lse = run_max + logf(run_sum);
        value = lse - logf((float)S);
      } else {
        value = warp_sum(s0a) / (float)S;
      }
      kmo = warp_sum(kmo) / ((float)S * (float)S);  // dA/do_s through the sample mean, the same for every s
      // pass 2: dA/dy_ms in chunks of 32 samples, reduced into A_mu, A_sd (lanes) and A_c (lane p: column p)
      float amu[BB_OBJ_MAX_TARGETS], asd[BB_OBJ_MAX_TARGETS];
#pragma unroll
      for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) amu[m] = asd[m] = 0.f;
      for (int s0 = 0; s0 < S; s0 += 32) {
        const int s = s0 + lane;
        float g = 0.f;
        if (s < S) {
          const float o = sample_o(s, dody);
          if (kind == BB_ACQ_QLOGEI && P == 0) {
            const float t = (o - a.best_f) * inv_relu;
            const float q = 1.f / fmaf(t, t, 1.f);
            g = (sigmoidf_(t) - 0.2f * (t * q) * q) * norm * inv_relu;
          } else {
            float dterm, joined;
            const float term = term_of(o, mo, dterm);
            const float share = join_share(term, s, joined);
            const float ws = kind == BB_ACQ_QLOGEI ? expf(joined - lse) : 1.f / (float)S;
            g = ws * share * dterm + (kind == BB_ACQ_QUCB ? kmo : 0.f);
          }
        }
        __syncwarp();
#pragma unroll
        for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
          if (m < M) {
            const float gm = s < S ? g * dody[m] : 0.f;
            gc[lane * M + m] = gm;
            amu[m] += gm;
            if (s < S) asd[m] = fmaf(gm, zc[s * M + m], asd[m]);
          }
        }
        __syncwarp();
        if (lane < P) {
          const int ns = min(32, S - s0);
          for (int m = 0; m < M; ++m) {
            float acc = acw[m * 32 + lane];
            const float* wr = p.w + ((size_t)m * S + s0) * P + lane;
            for (int t = 0; t < ns; ++t) acc = fmaf(gc[t * M + m], __ldg(wr + (size_t)t * P), acc);
            acw[m * 32 + lane] = acc;
          }
        }
      }
      __syncwarp();
      // sd_m = sqrt(max(var_m - |r_m|^2, 0)), r_m = L_m^-1 c_m: A_var = A_sd / (2 sd), A_c -= A_sd L_m^-T r_m / sd
#pragma unroll
      for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
        if (m < M) {
          gmu[m] = warp_sum(amu[m]);
          const float a_sd = warp_sum(asd[m]);
          const float sd = sd_s[m];
          const float f = sd > 0.f ? a_sd / sd : 0.f;
          if (lane < P) {
            const float* Lm = p.plinv + (size_t)m * P * P;
            float lt = 0.f;
            for (int i = lane; i < P; ++i) lt = fmaf(__ldg(Lm + i * P + lane), rw[m * 32 + i], lt);
            acw[m * 32 + lane] = fmaf(-f, lt, acw[m * 32 + lane]);
          }
          if (lane == 0) gvar_s[m] = 0.5f * f;
        }
      }
      __syncwarp();
    }
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
