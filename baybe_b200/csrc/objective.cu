// objective.cu -- acquisition values of objectives that are not affine in the modelled targets, one candidate per warp.
//
// Reference: the MC acquisition functions apply objective.to_botorch() to posterior samples
// (/root/reference/baybe/acquisition/_builder.py:211-254): per target the oriented transformation
// (objectives/base.py:130-150; desirability orients minimised targets as 1 - y, desirability.py:206-215), then the
// desirability scalariser (desirability.py:229-264: LinearMCObjective(normalised weights) or the weighted geometric
// mean exp(sum_m w_m log(t_m + eps)), eps = 2^-52, desirability.py:41-70).  Per candidate x and base sample s:
//   y_m = mu_m + c_m . w_{m,s} + sqrt(max(var_m - |L_m^-1 c_m|^2, 0)) z_{s, m(1+P)+P}    (c = 0 without pending points)
//   t_m = program_m(y_m),   o_s = scalarise(t)
// and the acquisition value over the o_s (qLogEI / qEI / qPI / qSR / qUCB), joined with the pending points' per-sample
// terms (computed once per round on the host, baybe_b200/objectives.py) by max, or fatmax for qLogEI.  The programs are
// a kernel parameter (bb_objective, 4.2 KB): every lane runs the same opcode, and two streams never share state.
//
// Mapping (DESIGN.md section 4.3, score_common.cuh): one warp per candidate, lane l takes samples l, l+32, ...; the
// S x M candidate base samples sit in shared memory.
#include <math.h>

#include "score_common.cuh"

namespace bb {

struct ObjParams : ScoreParams {  // C = P pending points; w: [M][S][P]
  bb_objective obj;
  bb_acq_spec a;
  const float* pend;  // [S][P] pending terms
};

constexpr int kObjThreads = 256;
constexpr float kGeomEps = 2.220446049250313e-16f;  // torch.finfo(float64).eps, exact in fp32

// Postfix program over y: x is the top of the evaluation stack, s1..s3 the entries below it (BB_OBJ_MAX_STACK = 4).
__device__ __forceinline__ float run_program(const bb_obj_instr* prog, int n, float y) {
  float x = y, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  for (int i = 0; i < n; ++i) {
    const int op = prog[i].op;
    const float a0 = prog[i].arg[0], a1 = prog[i].arg[1], a2 = prog[i].arg[2];
    switch (op) {
      case BB_OBJ_AFFINE: x = fmaf(x, a0, a1); break;
      case BB_OBJ_CONST: x = a0; break;
      case BB_OBJ_CLAMP: x = x < a0 ? a0 : (x > a1 ? a1 : x); break;  // NaN stays NaN, like torch.clamp
      case BB_OBJ_TWO_SIDED: {
        const float d = x - a2;
        x = (x < a2) ? (a0 != 0.f ? d * a0 : 0.f) : (a1 != 0.f ? d * a1 : 0.f);
        break;
      }
      case BB_OBJ_BELL: {
        const float u = (x - a0) / a1;
        x = expf(-(u * u) * 0.5f);
        break;
      }
      case BB_OBJ_LOG: x = logf(x); break;
      case BB_OBJ_EXP: x = expf(x); break;
      case BB_OBJ_POW_INT: x = powf(x, a0); break;
      case BB_OBJ_SIGMOID: x = 1.0f / (1.0f + expf(a1 * (x - a0))); break;
      case BB_OBJ_DUP_INPUT:
        s3 = s2;
        s2 = s1;
        s1 = x;
        x = y;
        break;
      case BB_OBJ_ADD:
        x = s1 + x;
        s1 = s2;
        s2 = s3;
        break;
      default:  // BB_OBJ_MUL (opcodes are validated on the host)
        x = s1 * x;
        s1 = s2;
        s2 = s3;
        break;
    }
  }
  return x;
}

__global__ void __launch_bounds__(kObjThreads) k_objective(const __grid_constant__ ObjParams p) {
  extern __shared__ __align__(16) float smem_o[];
  const int M = p.obj.n_targets, P = p.C, S = p.S, Q = P + 1;
  float* zc = smem_o;          // [S][M] candidate base samples
  float* linv = zc + S * M;    // [M][P][P]
  for (int e = threadIdx.x; e < S * M; e += blockDim.x) {
    const int s = e / M, m = e - s * M;
    zc[e] = __ldg(p.z + (size_t)s * (M * Q) + m * Q + P);
  }
  for (int e = threadIdx.x; e < M * P * P; e += blockDim.x) linv[e] = __ldg(p.linv + e);
  __syncthreads();

  const bb_acq_spec& a = p.a;
  const int kind = a.kind;
  const bool analytic = kind >= BB_ACQ_UCB;
  const int scal = p.obj.scalarizer;
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const float ucb_c = sqrtf(a.beta * 1.5707963267948966f);
  long long best = kEmptyKey;
  for (int64_t i = warp_global; i < p.N; i += nwarps) {
    // not warp_cond_moments: M is known only at run time here, and the analytic kinds take sd = var
    float mu[BB_OBJ_MAX_TARGETS], sd[BB_OBJ_MAX_TARGETS], cm[BB_OBJ_MAX_TARGETS];
#pragma unroll
    for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
      mu[m] = sd[m] = cm[m] = 0.f;
      if (m < M) {
        mu[m] = __ldg(p.mu + m * p.N + i);
        const float v = __ldg(p.var + m * p.N + i);
        float r2 = 0.f;
        if (P > 0) {
          cm[m] = (lane < P) ? __ldg(p.cross + ((size_t)m * p.N + i) * P + lane) : 0.f;
          r2 = pending_r2_warp(cm[m], linv + m * P * P, P, lane);
        }
        sd[m] = analytic ? v : sqrtf(fmaxf(v - r2, 0.f));
      }
    }
    float result;
    if (analytic) {
      // MEAN over affine targets: the scalarised posterior is Gaussian (desirability.py:311-320)
      float mean = 0.f, var = 0.f;
#pragma unroll
      for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
        if (m < M) {
          const bool aff = p.obj.n_ops[m] > 0;
          const float am = p.obj.weight[m] * (aff ? p.obj.prog[m][0].arg[0] : 1.0f);
          const float bm = p.obj.weight[m] * (aff ? p.obj.prog[m][0].arg[1] : 0.0f);
          mean += fmaf(am, mu[m], bm);
          var = fmaf(am * am, sd[m], var);
        }
      }
      bb_acq_spec u = a;
      u.obj_scale = 1.0f;
      u.obj_shift = 0.0f;
      result = analytic_value(u, mean, var);
    } else {
      // the objective of this lane's sample s (0 for s >= S, which no sum reads)
      auto sample_o = [&](int s) -> float {
        const bool valid = s < S;
        float acc = 0.f, o = 0.f;
#pragma unroll
        for (int m = 0; m < BB_OBJ_MAX_TARGETS; ++m) {
          if (m < M) {  // every lane takes part in the shuffles
            const float dm = P > 0 ? pending_cw_warp(cm[m], p.w + ((size_t)m * S + (valid ? s : 0)) * P, P) : 0.f;
            const float zz = valid ? zc[s * M + m] : 0.f;
            const float t = run_program(p.obj.prog[m], p.obj.n_ops[m], mu[m] + dm + sd[m] * zz);
            if (scal == BB_OBJ_SCALAR_NONE) o = t;
            else if (scal == BB_OBJ_SCALAR_MEAN) acc = fmaf(p.obj.weight[m], t, acc);
            else acc = fmaf(p.obj.weight[m], logf(t + kGeomEps), acc);
          }
        }
        if (scal == BB_OBJ_SCALAR_MEAN) o = acc;
        else if (scal == BB_OBJ_SCALAR_GEOM_MEAN) o = expf(acc);
        return o;
      };
      float mo = 0.f;  // qUCB: the SAMPLE mean of o (botorch qUpperConfidenceBound: obj.mean(dim=0))
      if (kind == BB_ACQ_QUCB) {
        float so = 0.f;
        for (int s0 = 0; s0 < S; s0 += 32) {
          const float o = sample_o(s0 + lane);
          if (s0 + lane < S) so += o;
        }
        for (int o = 16; o > 0; o >>= 1) so += __shfl_xor_sync(0xffffffffu, so, o);
        mo = so / (float)S;
      }
      const float inv_relu = 1.0f / a.tau_relu;
      float s0a = 0.f, s1a = 0.f;               // qLogEI without pending points: the mc_term sums; else plain sum
      float run_max = -INFINITY, run_sum = 0.f;  // qLogEI with pending points: online logsumexp
      float li_arr[BB_MAX_PENDING + 1];
      for (int s0 = 0; s0 < S; s0 += 32) {
        const int s = s0 + lane;
        const float o = sample_o(s);
        if (s >= S) continue;
        if (kind == BB_ACQ_QLOGEI && P == 0) {
          mc_term<BB_ACQ_QLOGEI>((o - a.best_f) * inv_relu, s0a, s1a);
          continue;
        }
        float term;
        if (kind == BB_ACQ_QLOGEI) term = logf(a.tau_relu) + log_fatplus_t((o - a.best_f) * inv_relu);
        else if (kind == BB_ACQ_QEI) term = fmaxf(o - a.best_f, 0.f);
        else if (kind == BB_ACQ_QSR) term = o;
        else if (kind == BB_ACQ_QPI) term = 1.0f / (1.0f + __expf(-(o - a.best_f) / a.tau_pi));
        else term = mo + ucb_c * fabsf(o - mo);
        term = join_terms(term, p.pend + (size_t)s * P, P, li_arr, kind == BB_ACQ_QLOGEI, a.tau_max);
        if (kind == BB_ACQ_QLOGEI) lse_push(term, run_max, run_sum);
        else s0a += term;
      }
      if (kind == BB_ACQ_QLOGEI && P == 0) {
        for (int o = 16; o > 0; o >>= 1) {
          s0a += __shfl_xor_sync(0xffffffffu, s0a, o);
          s1a += __shfl_xor_sync(0xffffffffu, s1a, o);
        }
        result = logf(a.tau_relu) + logf((s0a + 0.1f * s1a) / (float)S);
      } else if (kind == BB_ACQ_QLOGEI) {
        lse_warp_combine(run_max, run_sum);
        result = run_max + logf(run_sum) - logf((float)S);
      } else {
        for (int o = 16; o > 0; o >>= 1) s0a += __shfl_xor_sync(0xffffffffu, s0a, o);
        result = s0a / (float)S;
      }
    }
    warp_offer_best(p, i, result, lane, best);
  }
  block_flush_best<kObjThreads>(best, p.key);
}

// Dry run of one program on the host: opcodes, op count and stack depth (BB_OBJ_MAX_STACK).
static int check_program(const bb_objective* obj, int m) {
  const int n = obj->n_ops[m];
  BB_CHECK_SUPPORTED(n >= 0 && n <= BB_OBJ_MAX_OPS, "bb_objective_score: target %d has %d ops outside [0,%d]", m, n,
                     BB_OBJ_MAX_OPS);
  int depth = 1;
  for (int i = 0; i < n; ++i) {
    const bb_obj_instr& in = obj->prog[m][i];
    BB_CHECK_ARG(in.op >= BB_OBJ_AFFINE && in.op <= BB_OBJ_MUL, "bb_objective_score: target %d op %d: unknown opcode %d",
                 m, i, in.op);
    if (in.op == BB_OBJ_DUP_INPUT) ++depth;
    if (in.op == BB_OBJ_ADD || in.op == BB_OBJ_MUL) {
      BB_CHECK_ARG(depth >= 2, "bb_objective_score: target %d op %d pops an empty stack", m, i);
      --depth;
    }
    BB_CHECK_SUPPORTED(depth <= BB_OBJ_MAX_STACK, "bb_objective_score: target %d op %d: stack depth %d above %d", m, i,
                       depth, BB_OBJ_MAX_STACK);
    if (in.op == BB_OBJ_POW_INT)
      BB_CHECK_SUPPORTED(in.arg[0] == rintf(in.arg[0]), "bb_objective_score: target %d op %d: non-integer power %g", m,
                         i, (double)in.arg[0]);
  }
  BB_CHECK_ARG(depth == 1, "bb_objective_score: target %d leaves %d stack entries (need 1)", m, depth);
  return BB_OK;
}

}  // namespace bb

using namespace bb;

extern "C" int bb_objective_score(const bb_acq_spec* a, const bb_objective* obj, int64_t N, const float* d_mu,
                                  const float* d_var, int32_t n_pending, const float* d_cross, const float* d_linv,
                                  const float* d_w, const float* d_pend_terms, const float* d_z, int32_t S,
                                  const uint8_t* d_keep, float* d_score, int64_t* d_best_key, int64_t index_offset,
                                  void* stream) {
  BB_CHECK_ARG(a != nullptr, "bb_objective_score: acquisition spec is null");
  BB_CHECK_ARG(obj != nullptr, "bb_objective_score: objective is null");
  BB_CHECK_ARG(a->kind >= BB_ACQ_QLOGEI && a->kind <= BB_ACQ_PSTD,
               "bb_objective_score: kind %d is not a single-objective acquisition function", a->kind);
  const bool analytic = a->kind >= BB_ACQ_UCB;
  BB_CHECK_ARG(!(a->kind == BB_ACQ_QLOGEI) || (a->tau_relu > 0.f && a->tau_max > 0.f),
               "bb_objective_score: qLogEI needs tau_relu > 0 and tau_max > 0");
  BB_CHECK_ARG(!(a->kind == BB_ACQ_QPI) || a->tau_pi > 0.f, "bb_objective_score: qPI needs tau_pi > 0");
  const int M = obj->n_targets;
  BB_CHECK_SUPPORTED(M >= 1 && M <= BB_OBJ_MAX_TARGETS, "bb_objective_score: n_targets=%d outside [1,%d]", M,
                     BB_OBJ_MAX_TARGETS);
  BB_CHECK_ARG(obj->scalarizer >= BB_OBJ_SCALAR_NONE && obj->scalarizer <= BB_OBJ_SCALAR_GEOM_MEAN,
               "bb_objective_score: unknown scalarizer %d", obj->scalarizer);
  BB_CHECK_ARG((obj->scalarizer == BB_OBJ_SCALAR_NONE) == (M == 1),
               "bb_objective_score: scalarizer NONE is for exactly one target (got %d targets)", M);
  for (int m = 0; m < M; ++m) {
    const int rc = check_program(obj, m);
    if (rc != BB_OK) return rc;
    BB_CHECK_ARG(isfinite(obj->weight[m]), "bb_objective_score: weight %d is not finite", m);
  }
  if (analytic) {
    BB_CHECK_SUPPORTED(obj->scalarizer == BB_OBJ_SCALAR_MEAN,
                       "bb_objective_score: analytic kinds need MEAN scalarisation (the posterior must stay Gaussian)");
    for (int m = 0; m < M; ++m)
      BB_CHECK_SUPPORTED(obj->n_ops[m] == 0 || (obj->n_ops[m] == 1 && obj->prog[m][0].op == BB_OBJ_AFFINE),
                         "bb_objective_score: analytic kinds need affine targets (target %d is not)", m);
  }
  const int rc = check_score_args("bb_objective_score", "n_pending", N, index_offset, n_pending, S, !analytic,
                                  d_best_key);
  if (rc != BB_OK) return rc;
  BB_CHECK_ARG(!analytic || n_pending == 0, "bb_objective_score: analytic kinds take no pending points");
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_mu && d_var && (analytic || d_z), "bb_objective_score: null buffer");
  BB_CHECK_ARG(n_pending == 0 || (d_cross && d_linv && d_w && d_pend_terms),
               "bb_objective_score: pending points need cross, linv, w and pending terms");
  ObjParams p;
  p.N = N;
  p.mu = d_mu;
  p.var = d_var;
  p.cross = d_cross;
  p.linv = d_linv;
  p.w = d_w;
  p.z = d_z;
  p.keep = d_keep;
  p.score = d_score;
  p.key = reinterpret_cast<long long*>(d_best_key);
  p.index_offset = index_offset;
  p.C = n_pending;
  p.S = analytic ? 0 : S;
  p.obj = *obj;
  p.a = *a;
  p.pend = d_pend_terms;
  // at most 32 KB of candidate samples (S = 1024, M = 8) + 30 KB of L^-1 (M = 8, P = 31)
  const size_t smem = ((size_t)p.S * M + (size_t)M * n_pending * n_pending) * 4;
  return launch_warp_per_candidate<k_objective, kObjThreads, 4>(p, smem, (cudaStream_t)stream);
}
