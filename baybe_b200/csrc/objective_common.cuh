// objective_common.cuh -- host checks of a compiled objective (bb_objective), shared by bb_objective_score
// (objective.cu), bb_objective_grad (objgrad.cu) and bb_objective_grad_large (objgradlarge.cu); `fn` prefixes every
// message.  Then the device code of the objective's value and partials at one point, shared by the two gradient kernels.
#pragma once

#include <math.h>

#include "common.cuh"
#include "grad_common.cuh"
#include "score_common.cuh"

namespace bb {

// Dry run of one program on the host: opcodes, op count and stack depth (BB_OBJ_MAX_STACK).
static inline int check_program(const char* fn, const bb_objective* obj, int m) {
  const int n = obj->n_ops[m];
  BB_CHECK_SUPPORTED(n >= 0 && n <= BB_OBJ_MAX_OPS, "%s: target %d has %d ops outside [0,%d]", fn, m, n,
                     BB_OBJ_MAX_OPS);
  int depth = 1;
  for (int i = 0; i < n; ++i) {
    const bb_obj_instr& in = obj->prog[m][i];
    BB_CHECK_ARG(in.op >= BB_OBJ_AFFINE && in.op <= BB_OBJ_MUL, "%s: target %d op %d: unknown opcode %d", fn, m, i,
                 in.op);
    if (in.op == BB_OBJ_DUP_INPUT) ++depth;
    if (in.op == BB_OBJ_ADD || in.op == BB_OBJ_MUL) {
      BB_CHECK_ARG(depth >= 2, "%s: target %d op %d pops an empty stack", fn, m, i);
      --depth;
    }
    BB_CHECK_SUPPORTED(depth <= BB_OBJ_MAX_STACK, "%s: target %d op %d: stack depth %d above %d", fn, m, i, depth,
                       BB_OBJ_MAX_STACK);
    if (in.op == BB_OBJ_POW_INT)
      BB_CHECK_SUPPORTED(in.arg[0] == rintf(in.arg[0]), "%s: target %d op %d: non-integer power %g", fn, m, i,
                         (double)in.arg[0]);
  }
  BB_CHECK_ARG(depth == 1, "%s: target %d leaves %d stack entries (need 1)", fn, m, depth);
  return BB_OK;
}

// The acquisition kind and its temperatures, the target count, the scalariser, every program and weight, and the
// analytic kinds' envelope (MEAN over affine targets: the scalarised posterior must stay Gaussian).  a, obj non-null.
static inline int check_objective(const char* fn, const bb_acq_spec* a, const bb_objective* obj) {
  BB_CHECK_ARG(a->kind >= BB_ACQ_QLOGEI && a->kind <= BB_ACQ_PSTD,
               "%s: kind %d is not a single-objective acquisition function", fn, a->kind);
  const bool analytic = a->kind >= BB_ACQ_UCB;
  BB_CHECK_ARG(!(a->kind == BB_ACQ_QLOGEI) || (a->tau_relu > 0.f && a->tau_max > 0.f),
               "%s: qLogEI needs tau_relu > 0 and tau_max > 0", fn);
  BB_CHECK_ARG(!(a->kind == BB_ACQ_QPI) || a->tau_pi > 0.f, "%s: qPI needs tau_pi > 0", fn);
  const int M = obj->n_targets;
  BB_CHECK_SUPPORTED(M >= 1 && M <= BB_OBJ_MAX_TARGETS, "%s: n_targets=%d outside [1,%d]", fn, M, BB_OBJ_MAX_TARGETS);
  BB_CHECK_ARG(obj->scalarizer >= BB_OBJ_SCALAR_NONE && obj->scalarizer <= BB_OBJ_SCALAR_GEOM_MEAN,
               "%s: unknown scalarizer %d", fn, obj->scalarizer);
  BB_CHECK_ARG((obj->scalarizer == BB_OBJ_SCALAR_NONE) == (M == 1),
               "%s: scalarizer NONE is for exactly one target (got %d targets)", fn, M);
  for (int m = 0; m < M; ++m) {
    const int rc = check_program(fn, obj, m);
    if (rc != BB_OK) return rc;
    BB_CHECK_ARG(isfinite(obj->weight[m]), "%s: weight %d is not finite", fn, m);
  }
  if (analytic) {
    BB_CHECK_SUPPORTED(obj->scalarizer == BB_OBJ_SCALAR_MEAN,
                       "%s: analytic kinds need MEAN scalarisation (the posterior must stay Gaussian)", fn);
    for (int m = 0; m < M; ++m)
      BB_CHECK_SUPPORTED(obj->n_ops[m] == 0 || (obj->n_ops[m] == 1 && obj->prog[m][0].op == BB_OBJ_AFFINE),
                         "%s: analytic kinds need affine targets (target %d is not)", fn, m);
  }
  return BB_OK;
}


// ---- the objective's value and partials at one point (k_objective_grad, k_objective_grad_large) --------------------
// Device code: only translation units with kernels that use it instantiate it.

constexpr float kObjGeomEps = 2.220446049250313e-16f;  // as objective.cu

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

// The acquisition value of the objective at one point from its M targets' moments, and the partials the reverse pass
// needs (objgrad.cu's header gives the formulas).  Inputs: mu_s, var_s, sd_s [M]; cw [M][32] the cross covariances
// c_m with the P pending points and rw [M][32] = L_m^-1 c_m; zc [S][M] the candidate's base samples; w [M][S][P],
// pend [S][P] and plinv [M][P][P] as bb_objective_score takes them.  Outputs: the value and gmu[m] = A_mu in every
// lane, gvar_s[m] = A_var (before the variance clamp) and acw [M][32] = A_c (accumulated: the caller zeroes it).
// gc [32][M] is scratch.  Analytic kinds (S = 0): MEAN over affine targets, Gaussian.  One warp; every lane calls it.
__device__ __forceinline__ float objective_point_partials(const bb_objective& obj, const bb_acq_spec& a, int M, int P,
                                                          int S, const float* zc, const float* w, const float* pend,
                                                          const float* plinv, const float* mu_s, const float* var_s,
                                                          const float* sd_s, const float* cw, const float* rw,
                                                          float* acw, float* gc, float* gvar_s,
                                                          float (&gmu)[BB_OBJ_MAX_TARGETS], int lane) {
  const int kind = a.kind;
  const bool analytic = kind >= BB_ACQ_UCB;
  const int scal = obj.scalarizer;
  const float ucb_c = sqrtf(a.beta * 1.5707963267948966f);
  const float inv_relu = 1.0f / a.tau_relu;
#pragma unroll
  for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) gmu[m] = 0.f;
  float value;
  if (analytic) {
    // MEAN over affine targets: the scalarised posterior is Gaussian (objective.cu)
    float mean = 0.f, var = 0.f;
#pragma unroll
    for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
      if (m < M) {
        const bool aff = obj.n_ops[m] > 0;
        const float am = obj.weight[m] * (aff ? obj.prog[m][0].arg[0] : 1.0f);
        const float bm = obj.weight[m] * (aff ? obj.prog[m][0].arg[1] : 0.0f);
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
        const bool aff = obj.n_ops[m] > 0;
        const float am = obj.weight[m] * (aff ? obj.prog[m][0].arg[0] : 1.0f);
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
          const float* wr = w + ((size_t)m * S + s) * P;
          for (int j = 0; j < P; ++j) dm = fmaf(cw[m * 32 + j], __ldg(wr + j), dm);
          const float y = mu_s[m] + dm + sd_s[m] * zc[s * M + m];
          float dt;
          const float t = run_program_dual(obj.prog[m], obj.n_ops[m], y, dt);
          tt[m] = t;
          dody[m] = dt;
          if (scal == BB_OBJ_SCALAR_NONE) o = t;
          else if (scal == BB_OBJ_SCALAR_MEAN) acc = fmaf(obj.weight[m], t, acc);
          else acc = fmaf(obj.weight[m], logf(t + kObjGeomEps), acc);
        }
      }
      if (scal == BB_OBJ_SCALAR_MEAN) o = acc;
      else if (scal == BB_OBJ_SCALAR_GEOM_MEAN) o = expf(acc);
#pragma unroll
      for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
        if (scal == BB_OBJ_SCALAR_MEAN) dody[m] *= obj.weight[m];
        else if (scal == BB_OBJ_SCALAR_GEOM_MEAN) dody[m] *= o * obj.weight[m] / (tt[m] + kObjGeomEps);
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
      joined = join_terms(term, pend + (size_t)s * P, P, li_arr, kind == BB_ACQ_QLOGEI, a.tau_max);
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
          const float* wr = w + ((size_t)m * S + s0) * P + lane;
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
          const float* Lm = plinv + (size_t)m * P * P;
          float lt = 0.f;
          for (int i = lane; i < P; ++i) lt = fmaf(__ldg(Lm + i * P + lane), rw[m * 32 + i], lt);
          acw[m * 32 + lane] = fmaf(-f, lt, acw[m * 32 + lane]);
        }
        if (lane == 0) gvar_s[m] = 0.5f * f;
      }
    }
    __syncwarp();
  }
  return value;
}

}  // namespace bb
