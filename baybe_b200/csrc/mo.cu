// mo.cu -- hypervolume-improvement scoring for Pareto objectives (qEHVI / qLogEHVI), one candidate per warp.
//
// Reference: qExpectedHypervolumeImprovement / qLogExpectedHypervolumeImprovement
// (/root/reference/baybe/acquisition/acqfs.py:430-465) with the reference point and the box decomposition of the
// posterior-mean front set up by acquisition/_builder.py:286-317.  The decompositions are built on the host
// (baybe_b200/multiobjective.py); this kernel evaluates, per candidate x and base sample s, the improvement of
// the sample y_s(x) over the non-dominated cells [l_c, u_c) (u = +inf: no upper bound):
//   qEHVI    : HVI_s = sum_c prod_m max(min(y_m, u_cm) - l_cm, 0),                score = mean_s HVI_s
//   qLogEHVI : log HVI_s = logsumexp_c sum_m log fatplus(fatmin(y_m, u_cm) - l_cm),  score = logmeanexp_s
// (tau_relu / tau_max from bb_acq_spec).  fatmin(y, +inf) evaluates to y exactly, so no smoothing is applied
// against an open side.  With P pending points the cells are those of F u P_s, one decomposition per sample, and
// the candidate sample is conditional on the pending samples (DESIGN.md section 2):
//   y_m = a_m (mu_m + c_m . w_{m,s} + sqrt(max(var_m - |L_m^-1 c_m|^2, 0)) z_{s, m(1+P)+P}) + b_m,
// c_m = Sigma_{x,P} of target m, L_m L_m^T = K_PP (pending Cholesky), w_{m,s} = L_m^-T z_{s, m(1+P) .. m(1+P)+P-1}.
// |L^-1 c|^2 is a sum of squares: no cancellation against var for nearly collinear pending points.
#include <math.h>

#include "score_common.cuh"

namespace bb {

struct HviParams : ScoreParams {  // C = P pending points; w: [M][S][P]
  const float *lower, *upper;  // [n_dec][cells][M]
  const int32_t* n_cells;      // [n_dec]
  int cells, n_dec;            // cell stride, decompositions (1, or S with pending points)
  float tau_relu, tau_max;
  float a[BB_HVI_MAX_TARGETS], b[BB_HVI_MAX_TARGETS];
};

// botorch fatminimum(y, u) = -fatmax(-y, -u) = min(y, u) - tau log(1 + (1 + |y - u| / (2 tau))^-2); exactly y for u = +inf
__device__ __forceinline__ float fatmin_f(float y, float u, float half_inv_tau, float tau) {
  const float w = fmaf(fabsf(y - u), half_inv_tau, 1.0f);
  return fminf(y, u) - tau * __logf(1.0f + 1.0f / (w * w));
}

constexpr int kHviThreads = 256;

template <int M, bool LOG>
__global__ void __launch_bounds__(kHviThreads) k_hvi(const HviParams p) {
  extern __shared__ __align__(16) float smem_h[];
  // float offsets by hand, not SmemCarver: placing the same buffers through it makes ptxas give k_hvi<3, false> 40
  // registers and spill, and k_hvi<4, true> 48 registers and 84 B of spills
  const int P = p.C, S = p.S, Q = P + 1;
  float* zc = smem_h;              // [S][M] candidate base samples
  float* linv = zc + S * M;        // [M][P][P]
  float* cl = linv + M * P * P;    // [cells][M] bounds of the single decomposition (P = 0)
  float* cu = cl + p.cells * M;
  for (int e = threadIdx.x; e < S * M; e += blockDim.x) {
    const int s = e / M, m = e - s * M;
    zc[e] = __ldg(p.z + (size_t)s * (M * Q) + m * Q + P);
  }
  for (int e = threadIdx.x; e < M * P * P; e += blockDim.x) linv[e] = __ldg(p.linv + e);
  const bool shared_cells = p.n_dec == 1;
  const int nc0 = shared_cells ? min(__ldg(p.n_cells), p.cells) : 0;
  for (int e = threadIdx.x; e < nc0 * M; e += blockDim.x) {
    cl[e] = __ldg(p.lower + e);
    cu[e] = __ldg(p.upper + e);
  }
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const float inv_tr = 1.0f / p.tau_relu, half_inv_tm = 0.5f / p.tau_max, tm = p.tau_max;
  long long best = kEmptyKey;
  for (int64_t i = warp_global; i < p.N; i += nwarps) {
    float mu[M], sd[M], cm[M];
    warp_cond_moments<M>(p, linv, P, i, lane, mu, sd, cm);
    float run_max = -INFINITY, run_sum = 0.f;  // LOG: logsumexp over samples; else the plain sum
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      const bool valid = s < S;
      float y[M];
#pragma unroll
      for (int m = 0; m < M; ++m) {
        float dm = 0.f;
        if (P > 0) dm = warp_cond_shift<false>(p.w, cm[m], m, valid ? s : 0, P, S);
        const float zz = valid ? zc[s * M + m] : 0.f;
        y[m] = fmaf(p.a[m], mu[m] + dm + sd[m] * zz, p.b[m]);
      }
      if (!valid) continue;
      const float *L = cl, *U = cu;
      int nc = nc0;
      if (!shared_cells) {
        nc = min(__ldg(p.n_cells + s), p.cells);
        L = p.lower + (size_t)s * p.cells * M;
        U = p.upper + (size_t)s * p.cells * M;
      }
      if (LOG) {
        float cmax = -INFINITY, csum = 0.f;
        for (int c = 0; c < nc; ++c) {
          float t = 0.f;
#pragma unroll
          for (int m = 0; m < M; ++m) {
            const float f = fatmin_f(y[m], U[c * M + m], half_inv_tm, tm);
            t += log_fatplus_t((f - L[c * M + m]) * inv_tr);
          }
          lse_push(t, cmax, csum);
        }
        if (cmax > -INFINITY) lse_push(cmax + __logf(csum), run_max, run_sum);
      } else {
        float acc = 0.f;
        for (int c = 0; c < nc; ++c) {
          float prod = 1.f;
#pragma unroll
          for (int m = 0; m < M; ++m) prod *= fmaxf(fminf(y[m], U[c * M + m]) - L[c * M + m], 0.f);
          acc += prod;
        }
        run_sum += acc;
      }
    }
    float result;
    if (LOG) {
      lse_warp_combine(run_max, run_sum);
      // the M log(tau_relu) of every cell term is added once
      result = run_max + logf(run_sum) - logf((float)S) + (float)M * logf(p.tau_relu);
    } else {
      for (int o = 16; o > 0; o >>= 1) run_sum += __shfl_xor_sync(0xffffffffu, run_sum, o);
      result = run_sum / (float)S;
    }
    warp_offer_best(p, i, result, lane, best);
  }
  block_flush_best<kHviThreads>(best, p.key);
}

template <int M, bool LOG>
static int launch_hvi(const HviParams& p, cudaStream_t st) {
  // at most 48 KB + 15 KB: S*M samples and, for P = 0 only, 2*cells*M bounds (S = cells = 1024, M = 4), or with
  // P = 31 the S*M samples and M*P*P entries of L^-1
  const size_t smem = ((size_t)p.S * M + (size_t)M * p.C * p.C + (p.n_dec == 1 ? 2 * (size_t)p.cells * M : 0)) * 4;
  return launch_warp_per_candidate<k_hvi<M, LOG>, kHviThreads, 4>(p, smem, st);
}

}  // namespace bb

using namespace bb;

extern "C" int bb_hvi_score(const bb_acq_spec* a, int32_t n_targets, const float* obj_scale, const float* obj_shift,
                            int64_t N, const float* d_mu, const float* d_var, int32_t n_pending, const float* d_cross,
                            const float* d_linv, const float* d_w, const float* d_z, int32_t S, const float* d_lower,
                            const float* d_upper, const int32_t* d_n_cells, int32_t cell_stride,
                            const uint8_t* d_keep, float* d_score, int64_t* d_best_key, int64_t index_offset,
                            void* stream) {
  BB_CHECK_ARG(a != nullptr, "bb_hvi_score: acquisition spec is null");
  BB_CHECK_ARG(a->kind == BB_ACQ_QEHVI || a->kind == BB_ACQ_QLOGEHVI,
               "bb_hvi_score: kind %d is not a hypervolume acquisition function", a->kind);
  BB_CHECK_ARG(!(a->kind == BB_ACQ_QLOGEHVI) || (a->tau_relu > 0.f && a->tau_max > 0.f),
               "bb_hvi_score: qLogEHVI needs tau_relu > 0 and tau_max > 0");
  BB_CHECK_SUPPORTED(n_targets >= 2 && n_targets <= BB_HVI_MAX_TARGETS,
                     "bb_hvi_score: n_targets=%d outside [2,%d]", n_targets, BB_HVI_MAX_TARGETS);
  BB_CHECK_ARG(obj_scale != nullptr && obj_shift != nullptr, "bb_hvi_score: null objective scale/shift");
  const int rc = check_score_args("bb_hvi_score", "n_pending", N, index_offset, n_pending, S, true, d_best_key);
  if (rc != BB_OK) return rc;
  BB_CHECK_SUPPORTED(cell_stride >= 1 && cell_stride <= BB_HVI_MAX_CELLS,
                     "bb_hvi_score: cell_stride=%d outside [1,%d]", cell_stride, BB_HVI_MAX_CELLS);
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_mu && d_var && d_z && d_lower && d_upper && d_n_cells, "bb_hvi_score: null buffer");
  BB_CHECK_ARG(n_pending == 0 || (d_cross && d_linv && d_w), "bb_hvi_score: pending points need cross, linv and w");
  HviParams p{};
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
  p.S = S;
  p.lower = d_lower;
  p.upper = d_upper;
  p.n_cells = d_n_cells;
  p.cells = cell_stride;
  p.n_dec = n_pending == 0 ? 1 : S;
  p.tau_relu = a->tau_relu;
  p.tau_max = a->tau_max;
  for (int m = 0; m < n_targets; ++m) {
    p.a[m] = obj_scale[m];
    p.b[m] = obj_shift[m];
  }
  cudaStream_t st = (cudaStream_t)stream;
  const bool lg = a->kind == BB_ACQ_QLOGEHVI;
  switch (n_targets) {
    case 2: return lg ? launch_hvi<2, true>(p, st) : launch_hvi<2, false>(p, st);
    case 3: return lg ? launch_hvi<3, true>(p, st) : launch_hvi<3, false>(p, st);
    default: return lg ? launch_hvi<4, true>(p, st) : launch_hvi<4, false>(p, st);
  }
}
