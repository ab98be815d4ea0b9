// nei.cu -- noisy expected improvement (qNEI / qLogNEI) of every candidate of a discrete space, one candidate per warp.
//
// Reference: qNoisyExpectedImprovement / qLogNoisyExpectedImprovement (/root/reference/baybe/acquisition/acqfs.py:
// 226-243) with X_baseline = the measured rows (acquisition/_builder.py:319-324), pruned on the host
// (baybe_b200/noisy.py).  The conditioning set C = [kept baseline; pending; rest of the q-batch] is sampled jointly on
// the host in float64; the candidate is sampled conditionally on it (DESIGN.md section 2):
//   y_s = mu + c . w_s + sqrt(max(var - |L_C^-1 c|^2, 0)) z_{s,|C|},   o_s = a y_s + b,
// c = Sigma_{x,C} (bb_posterior's cross covariance), L_C L_C^T = Sigma_CC, w_s = L_C^-T z_{s,0..|C|-1}.  With the
// per-sample incumbent g_s (max of o over baseline and pending) and the per-sample terms of the rest of the batch:
//   qNEI    : value = mean_s max(relu(o_s - g_s), terms_s)
//   qLogNEI : value = logmeanexp_s fatmax(log tau_relu + log fatplus((o_s - g_s) / tau_relu), terms_s)   (tau_max)
// Mapping as k_hvi / k_objective (score_common.cuh).
#include <math.h>

#include "score_common.cuh"

namespace bb {

struct NeiParams : ScoreParams {  // M = 1; w: [C][S] sample-minor
  const float* g;      // [S]
  const float* terms;  // [S][Q]
  int Q;
  float a, b, tau_relu, tau_max;
};

constexpr int kNeiThreads = 256;

template <bool LOG>
__global__ void __launch_bounds__(kNeiThreads) k_nei(const NeiParams p) {
  extern __shared__ __align__(16) float smem_n[];
  const int C = p.C, S = p.S, Q = p.Q;
  float* zc = smem_n;     // [S] candidate base samples
  float* gs = zc + S;     // [S] incumbents
  float* linv = gs + S;   // [C][C]
  for (int e = threadIdx.x; e < S; e += blockDim.x) {
    zc[e] = __ldg(p.z + (size_t)e * (C + 1) + C);
    gs[e] = __ldg(p.g + e);
  }
  for (int e = threadIdx.x; e < C * C; e += blockDim.x) linv[e] = __ldg(p.linv + e);
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const float inv_tr = 1.0f / p.tau_relu, log_tr = logf(p.tau_relu);
  long long best = kEmptyKey;
  float li[BB_MAX_PENDING + 1];
  for (int64_t i = warp_global; i < p.N; i += nwarps) {
    float mu[1], sd[1], cm[1];
    warp_cond_moments<1>(p, linv, C, i, lane, mu, sd, cm);
    float run_max = -INFINITY, run_sum = 0.f;  // LOG: logsumexp over samples; else the plain sum
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      const bool valid = s < S;
      const float dm = C > 0 ? warp_cond_shift<true>(p.w, cm[0], 0, valid ? s : 0, C, S) : 0.f;
      if (!valid) continue;
      const float u = fmaf(p.a, mu[0] + dm + sd[0] * zc[s], p.b) - gs[s];
      float term = LOG ? log_tr + log_fatplus_t(u * inv_tr) : fmaxf(u, 0.f);
      if (Q > 0) term = join_terms(term, p.terms + (size_t)s * Q, Q, li, LOG, p.tau_max);
      if (LOG) lse_push(term, run_max, run_sum);
      else run_sum += term;
    }
    float result;
    if (LOG) {
      lse_warp_combine(run_max, run_sum);
      result = run_max + logf(run_sum) - logf((float)S);
    } else {
      for (int o = 16; o > 0; o >>= 1) run_sum += __shfl_xor_sync(0xffffffffu, run_sum, o);
      result = run_sum / (float)S;
    }
    warp_offer_best(p, i, result, lane, best);
  }
  block_flush_best<kNeiThreads>(best, p.key);
}

}  // namespace bb

using namespace bb;

extern "C" int bb_nei_score(int32_t log_nei, float obj_scale, float obj_shift, float tau_relu, float tau_max, int64_t N,
                            const float* d_mu, const float* d_var, int32_t n_cond, const float* d_cross,
                            const float* d_linv, const float* d_w, const float* d_z, int32_t S, const float* d_g,
                            int32_t n_batch, const float* d_batch_terms, const uint8_t* d_keep, float* d_score,
                            int64_t* d_best_key, int64_t index_offset, void* stream) {
  BB_CHECK_ARG(log_nei == 0 || log_nei == 1, "bb_nei_score: log_nei=%d is not 0 or 1", log_nei);
  BB_CHECK_ARG(isfinite(obj_scale) && isfinite(obj_shift), "bb_nei_score: objective scale/shift not finite");
  BB_CHECK_ARG(!log_nei || (tau_relu > 0.f && tau_max > 0.f), "bb_nei_score: qLogNEI needs tau_relu > 0 and tau_max > 0");
  const int rc = check_score_args("bb_nei_score", "n_cond", N, index_offset, n_cond, S, true, d_best_key);
  if (rc != BB_OK) return rc;
  BB_CHECK_ARG(n_batch >= 0 && n_batch <= n_cond, "bb_nei_score: n_batch=%d outside [0,n_cond=%d]", n_batch, n_cond);
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_mu && d_var && d_z && d_g, "bb_nei_score: null buffer");
  BB_CHECK_ARG(n_cond == 0 || (d_cross && d_linv && d_w), "bb_nei_score: conditioning points need cross, linv and w");
  BB_CHECK_ARG(n_batch == 0 || d_batch_terms, "bb_nei_score: batch points need their terms");
  NeiParams p{};
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
  p.C = n_cond;
  p.S = S;
  p.g = d_g;
  p.terms = d_batch_terms;
  p.Q = n_batch;
  p.a = obj_scale;
  p.b = obj_shift;
  p.tau_relu = log_nei ? tau_relu : 1.0f;
  p.tau_max = log_nei ? tau_max : 1.0f;
  // at most 8 KB of samples and incumbents (S = 1024) + 3.8 KB of L^-1 (31 points): below the 48 KB default
  const size_t smem = (2 * (size_t)S + (size_t)n_cond * n_cond) * 4;
  cudaStream_t st = (cudaStream_t)stream;
  return log_nei ? launch_warp_per_candidate<k_nei<true>, kNeiThreads, 4>(p, smem, st)
                 : launch_warp_per_candidate<k_nei<false>, kNeiThreads, 4>(p, smem, st);
}
