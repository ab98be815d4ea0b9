// parego.cu -- qLogNParEGO of every candidate of a discrete space over M in [2, 8] targets, one candidate per warp.
//
// Reference: qLogNParEGO (/root/reference/baybe/acquisition/acqfs.py:328-336) with X_baseline = the measured rows
// (acquisition/_builder.py:319-324); the host (baybe_b200/parego.py) draws the simplex weights, folds the
// normalisation and the weights into one affine map per target, prunes the baseline on the Chebyshev scalarisation and
// samples the conditioning set C = [kept baseline; pending; rest of the q-batch] jointly per target in float64
// (DESIGN.md section 2).  Per target m the candidate is sampled conditionally on C:
//   y_m,s = mu_m + c_m . w_m,s + sqrt(max(var_m - |L_C,m^-1 c_m|^2, 0)) z_{s, m(|C|+1)+|C|},   p_m,s = W_m y_m,s + V_m,
// and scalarised by the augmented Chebyshev form cheb_s = min_m p_m,s + alpha sum_m p_m,s.  With the per-sample
// incumbent g_s (max of cheb over baseline and pending points) and the per-sample terms of the rest of the batch:
//   value = logmeanexp_s fatmax(log tau_relu + log fatplus((cheb_s - g_s) / tau_relu), terms_s)   (tau_max)
// Mapping as k_nei (score_common.cuh).  M is a template parameter, so the per-target moments of a candidate (mu, sd
// and the lane's entry of c) stay in registers across the sample loop.
#include <math.h>

#include "score_common.cuh"

namespace bb {

struct ParegoParams : ScoreParams {  // w: [M][C][S] sample-minor
  const float* g;      // [S]
  const float* terms;  // [S][Q]
  int Q;
  float alpha, tau_relu, tau_max;
  float wt[BB_OBJ_MAX_TARGETS], off[BB_OBJ_MAX_TARGETS];  // p_m = wt_m y_m + off_m
};

constexpr int kParegoThreads = 256;
// three resident blocks per SM: the bound keeps every instantiation at <= 80 registers with no spill (without it,
// ptxas spills around the slow-path calls of sqrtf and the divisions at M = 2, 3, 4 and 7), and the grid is capped at
// the same three blocks per SM so that no block waits for a second wave
constexpr int kParegoBlocksPerSM = 3;

struct ParegoSmem {
  float* zc;    // [M][S] the candidate's base samples, target-major so that a warp's loads hit 32 banks
  float* gs;    // [S] incumbents
  float* linv;  // [M][C][C]
};

static __host__ __device__ size_t carve_parego(uint8_t* base, int M, int S, int C, ParegoSmem& s) {
  SmemCarver c{base};
  s.zc = c.take<float>((size_t)M * S * 4);
  s.gs = c.take<float>((size_t)S * 4);
  s.linv = c.take<float>((size_t)M * C * C * 4);
  return c.bytes;
}

template <int M>
__global__ void __launch_bounds__(kParegoThreads, kParegoBlocksPerSM) k_parego(const ParegoParams p) {
  extern __shared__ __align__(16) uint8_t smem_pe[];
  const int C = p.C, S = p.S, Q = p.Q;
  ParegoSmem sm;
  carve_parego(smem_pe, M, S, C, sm);
  const int zld = M * (C + 1);
  for (int e = threadIdx.x; e < M * S; e += blockDim.x) {
    const int m = e / S, s = e - m * S;
    sm.zc[e] = __ldg(p.z + (size_t)s * zld + m * (C + 1) + C);
  }
  for (int e = threadIdx.x; e < S; e += blockDim.x) sm.gs[e] = __ldg(p.g + e);
  for (int e = threadIdx.x; e < M * C * C; e += blockDim.x) sm.linv[e] = __ldg(p.linv + e);
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const float inv_tr = 1.0f / p.tau_relu, log_tr = logf(p.tau_relu);
  long long best = kEmptyKey;
  float li[BB_MAX_PENDING + 1];
  for (int64_t i = warp_global; i < p.N; i += nwarps) {
    float mu[M], sd[M], cm[M];
    warp_cond_moments<M>(p, sm.linv, C, i, lane, mu, sd, cm);
    float run_max = -INFINITY, run_sum = 0.f;  // online logsumexp over the samples
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      const bool valid = s < S;
      const int sv = valid ? s : 0;
      float pmin = INFINITY, psum = 0.f;
#pragma unroll
      for (int m = 0; m < M; ++m) {
        const float dm = C > 0 ? warp_cond_shift<true>(p.w, cm[m], m, sv, C, S) : 0.f;
        const float pm = fmaf(p.wt[m], mu[m] + dm + sd[m] * sm.zc[m * S + sv], p.off[m]);
        pmin = fminf(pmin, pm);
        psum += pm;
      }
      if (!valid) continue;
      const float u = fmaf(p.alpha, psum, pmin) - sm.gs[s];
      float term = log_tr + log_fatplus_t(u * inv_tr);
      if (Q > 0) term = join_terms(term, p.terms + (size_t)s * Q, Q, li, true, p.tau_max);
      lse_push(term, run_max, run_sum);
    }
    lse_warp_combine(run_max, run_sum);
    const float result = run_max + logf(run_sum) - logf((float)S);
    warp_offer_best(p, i, result, lane, best);
  }
  block_flush_best<kParegoThreads>(best, p.key);
}

template <int M>
static int launch_parego(const ParegoParams& p, cudaStream_t st) {
  // at most 32 KB of candidate samples + 4 KB of incumbents (S = 1024, M = 8) + 30.75 KB of L^-1 (M = 8, |C| = 31)
  ParegoSmem s;
  const size_t smem = carve_parego(nullptr, M, p.S, p.C, s);
  return launch_warp_per_candidate<k_parego<M>, kParegoThreads, kParegoBlocksPerSM>(p, smem, st);
}

}  // namespace bb

using namespace bb;

extern "C" int bb_parego_score(int32_t n_targets, const float* weight, const float* offset, float alpha,
                               float tau_relu, float tau_max, int64_t N, const float* d_mu, const float* d_var,
                               int32_t n_cond, const float* d_cross, const float* d_linv, const float* d_w,
                               const float* d_z, int32_t S, const float* d_g, int32_t n_batch,
                               const float* d_batch_terms, const uint8_t* d_keep, float* d_score,
                               int64_t* d_best_key, int64_t index_offset, void* stream) {
  BB_CHECK_SUPPORTED(n_targets >= 2 && n_targets <= BB_OBJ_MAX_TARGETS, "bb_parego_score: n_targets=%d outside [2,%d]",
                     n_targets, BB_OBJ_MAX_TARGETS);
  BB_CHECK_ARG(weight != nullptr && offset != nullptr, "bb_parego_score: null scalarisation weights or offsets");
  for (int m = 0; m < n_targets; ++m)
    BB_CHECK_ARG(isfinite(weight[m]) && isfinite(offset[m]),
                 "bb_parego_score: scalarisation weight/offset of target %d not finite", m);
  BB_CHECK_ARG(isfinite(alpha), "bb_parego_score: alpha not finite");
  BB_CHECK_ARG(tau_relu > 0.f && tau_max > 0.f, "bb_parego_score: needs tau_relu > 0 and tau_max > 0");
  const int rc = check_score_args("bb_parego_score", "n_cond", N, index_offset, n_cond, S, true, d_best_key);
  if (rc != BB_OK) return rc;
  BB_CHECK_ARG(n_batch >= 0 && n_batch <= n_cond, "bb_parego_score: n_batch=%d outside [0,n_cond=%d]", n_batch,
               n_cond);
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_mu && d_var && d_z && d_g, "bb_parego_score: null buffer");
  BB_CHECK_ARG(n_cond == 0 || (d_cross && d_linv && d_w),
               "bb_parego_score: conditioning points need cross, linv and w");
  BB_CHECK_ARG(n_batch == 0 || d_batch_terms, "bb_parego_score: batch points need their terms");
  ParegoParams p{};
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
  p.alpha = alpha;
  p.tau_relu = tau_relu;
  p.tau_max = tau_max;
  for (int m = 0; m < n_targets; ++m) {
    p.wt[m] = weight[m];
    p.off[m] = offset[m];
  }
  cudaStream_t st = (cudaStream_t)stream;
  switch (n_targets) {
    case 2: return launch_parego<2>(p, st);
    case 3: return launch_parego<3>(p, st);
    case 4: return launch_parego<4>(p, st);
    case 5: return launch_parego<5>(p, st);
    case 6: return launch_parego<6>(p, st);
    case 7: return launch_parego<7>(p, st);
    default: return launch_parego<8>(p, st);
  }
}
