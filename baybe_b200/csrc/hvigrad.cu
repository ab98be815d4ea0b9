// hvigrad.cu -- value and gradient of the hypervolume improvement of a Pareto objective (qEHVI / qLogEHVI,
// bb_hvi_grad), for the continuous optimiser: the value bb_hvi_score (mo.cu) reports, and its gradient with respect to
// the raw comp-rep rows.
//
// Per point x, target m (one model each, with its own n, scaling and hyper-parameters) and base sample s, as in mo.cu:
//   y_ms = a_m (mu_m + c_m . w_ms + sd_m z_ms) + b_m,   sd_m = sqrt(max(var_m - |L_m^-1 c_m|^2, 0)),
//   qEHVI    : h_s = HVI_s = sum_c prod_m max(min(y_m, u_cm) - l_cm, 0),                    A = mean_s h_s
//   qLogEHVI : h_s = logsumexp_c sum_m log fatplus(fatmin(y_m, u_cm) - l_cm),                A = logmeanexp_s h_s
// over the cells of the one decomposition (P = 0) or of sample s's decomposition (P > 0), with mu_m, var_m and c_m
// (the cross covariances with the pending points) formed from x as in grad.cu.
//
// Reverse pass:
//   1. Second sample pass (lanes over samples; the cell terms are recomputed, not stored): dA/dh_s (1/S, or the
//      softmax weight exp(h_s - A') of the logmeanexp) times dh_s/dy_ms:
//        qEHVI    : sum_c 1[l_cm < y_m < u_cm] prod_{m' != m} max(min(y_m', u_cm') - l_cm', 0),
//        qLogEHVI : sum_c softmax_c (d log fatplus / dt)(fatmin(y_m, u_cm) - l_cm) dfatmin/dy (ties of min split the
//                   gradient in half, as torch.minimum does),
//      times a_m.  Reduced into A_mu[m], A_sd[m] and A_c[m][p] in chunks of 32 samples as in objgrad.cu; then
//      A_var = A_sd / (2 sd) and A_c -= A_sd L^-T (L^-1 c) / sd.
//   2. Per target, back through the kernel row (grad_common.cuh):
//      dA/dk_i = s_y A_mu alpha_i - 2 s_y^2 A_var u_i - s_y^2 sum_p A_c[p] beta_p,i, then dk/dt, then the direct
//      k(x, x_p) term; the gradient is the sum over the targets in target order.
// The per-target forward and reverse passes are grad_common.cuh's, shared with objgrad.cu's kernel in substance
// (DESIGN.md section 4.3).  Every reduction has a fixed order and nothing is accumulated atomically: repeated calls
// are bit-identical.
#include <math.h>

#include "fused_common.cuh"
#include "grad_common.cuh"
#include "score_common.cuh"

namespace bb {

constexpr int kHviGradThreads = 128;  // four points per block
constexpr int kHviGradWarps = kHviGradThreads / 32;

struct HviGradParams {
  GradTarget mdl[BB_HVI_MAX_TARGETS];
  float a[BB_HVI_MAX_TARGETS], b[BB_HVI_MAX_TARGETS];
  int d, d_pad, n_pad;  // n_pad: the largest over the targets (the scratch stride)
  const float* x;       // [N][d]
  int64_t N;
  int P;
  const float *pend_x, *plinv, *w;  // [P][d], [M][P][P], [M][S][P]
  const float* z;                   // [S][M(1+P)]
  int S;
  const float *lower, *upper;  // [n_dec][cells][M], n_dec = 1 (P = 0) or S
  const int32_t* n_cells;      // [n_dec]
  int cells;
  int log;  // qLogEHVI
  float tau_relu, tau_max;
  float* value;  // [N]
  float* grad;   // [N][d]
};

// dfatmin(y, u)/dy, fatmin as acq_math.cuh's fatmin_f: the min's share (1/2 at a tie) plus the smoothing's
// sign(y - u) / (w (w^2 + 1)), w = 1 + |y - u| / (2 tau); 1 for u = +inf
__device__ __forceinline__ float dfatmin_f(float y, float u, float half_inv_tau) {
  const float w = fmaf(fabsf(y - u), half_inv_tau, 1.0f);
  const float dmin = y < u ? 1.f : (y > u ? 0.f : 0.5f);
  const float sg = y > u ? 1.f : (y < u ? -1.f : 0.f);
  return dmin + sg / (w * fmaf(w, w, 1.f));
}

// h_s of one sample over its nc cells [L, U) (k_hvi's cell loop; qLogEHVI without the M log tau_relu, -inf without
// cells)
template <int M>
__device__ __forceinline__ float sample_h(const float (&y)[M], const float* L, const float* U, int nc, bool log,
                                         float inv_tr, float half_inv_tm, float tm) {
  if (log) {
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
    return cmax > -INFINITY ? cmax + __logf(csum) : -INFINITY;
  }
  float acc = 0.f;
  for (int c = 0; c < nc; ++c) {
    float prod = 1.f;
#pragma unroll
    for (int m = 0; m < M; ++m) prod *= fmaxf(fminf(y[m], U[c * M + m]) - L[c * M + m], 0.f);
    acc += prod;
  }
  return acc;
}

// dh_s/dy_m of one sample into g (h: sample_h of the same sample)
template <int M>
__device__ __forceinline__ void sample_dh(const float (&y)[M], const float* L, const float* U, int nc, bool log,
                                          float h, float inv_tr, float half_inv_tm, float tm, float (&g)[M]) {
#pragma unroll
  for (int m = 0; m < M; ++m) g[m] = 0.f;
  if (log) {
    if (!(h > -INFINITY)) return;
    for (int c = 0; c < nc; ++c) {
      float t = 0.f, dl[M];
#pragma unroll
      for (int m = 0; m < M; ++m) {
        const float u = (fatmin_f(y[m], U[c * M + m], half_inv_tm, tm) - L[c * M + m]) * inv_tr;
        t += log_fatplus_t(u);
        dl[m] = dlog_fatplus_t(u) * inv_tr * dfatmin_f(y[m], U[c * M + m], half_inv_tm);
      }
      const float wc = __expf(t - h);  // the cell's softmax weight
#pragma unroll
      for (int m = 0; m < M; ++m) g[m] = fmaf(wc, dl[m], g[m]);
    }
    return;
  }
  for (int c = 0; c < nc; ++c) {
    float side[M];
#pragma unroll
    for (int m = 0; m < M; ++m) side[m] = fmaxf(fminf(y[m], U[c * M + m]) - L[c * M + m], 0.f);
#pragma unroll
    for (int m = 0; m < M; ++m) {
      if (!(L[c * M + m] < y[m] && y[m] < U[c * M + m])) continue;
      float o = 1.f;
#pragma unroll
      for (int k = 0; k < M; ++k)
        if (k != m) o *= side[k];
      g[m] += o;
    }
  }
}

template <int FAMILY, int M>
__global__ void __launch_bounds__(kHviGradThreads) k_hvi_grad(const __grid_constant__ HviGradParams p) {
  extern __shared__ __align__(16) float smem_hg[];
  const int P = p.P, Q = P + 1, S = p.S;
  const bool log = p.log != 0;
  const bool shared_cells = P == 0;
  const int cstride = shared_cells ? ((p.cells * M + 3) & ~3) : 0;
  float* zc = smem_hg;                   // [S][M] candidate base samples
  float* cl = zc + ((S * M + 3) & ~3);  // [cells][M] bounds of the single decomposition (P = 0)
  float* cu = cl + cstride;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int np = p.n_pad, dp = p.d_pad;
  float* wb = cu + cstride + warp * target_warp_floats(M, np, dp);
  float* gc = wb + M * (dp + 3 * np + 4 * 32);  // [32][M] dA/dy of the current chunk's samples
  for (int e = threadIdx.x; e < S * M; e += blockDim.x) {
    const int s = e / M, m = e - s * M;
    zc[e] = __ldg(p.z + (size_t)s * (M * Q) + m * Q + P);
  }
  const int nc0 = shared_cells ? min(__ldg(p.n_cells), p.cells) : 0;
  for (int e = threadIdx.x; e < nc0 * M; e += blockDim.x) {
    cl[e] = __ldg(p.lower + e);
    cu[e] = __ldg(p.upper + e);
  }
  __syncthreads();
  const float inv_tr = 1.0f / p.tau_relu, half_inv_tm = 0.5f / p.tau_max, tm = p.tau_max;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = warp_global; c < p.N; c += nwarps) {
    // ---- forward, per target: a, k, mu, v, var, c, L^-1 c, sd ----
    float mu[M], sd[M];
    bool vfree[M];
#pragma unroll
    for (int m = 0; m < M; ++m) {
      float var;
      vfree[m] = target_forward_warp<FAMILY>(p.mdl[m], p.x + c * p.d, p.d, dp, P, p.pend_x,
                                             p.plinv + (size_t)m * P * P, target_scratch(wb, M, m, np, dp), mu[m],
                                             var, sd[m], lane);
    }
    // sample s's oriented y and its cells
    auto sample_y = [&](int s, float (&y)[M]) {
#pragma unroll
      for (int m = 0; m < M; ++m) {
        const float* cm = wb + M * (dp + 3 * np) + m * 32;
        const float* wr = p.w + ((size_t)m * S + s) * P;
        float dm = 0.f;
        for (int j = 0; j < P; ++j) dm = fmaf(cm[j], __ldg(wr + j), dm);
        y[m] = fmaf(p.a[m], mu[m] + dm + sd[m] * zc[s * M + m], p.b[m]);
      }
    };
    auto cells_of = [&](int s, const float*& L, const float*& U) -> int {
      if (shared_cells) {
        L = cl;
        U = cu;
        return nc0;
      }
      L = p.lower + (size_t)s * p.cells * M;
      U = p.upper + (size_t)s * p.cells * M;
      return min(__ldg(p.n_cells + s), p.cells);
    };
    // pass 1: the value, as k_hvi forms it
    float run_max = -INFINITY, run_sum = 0.f;
    for (int s = lane; s < S; s += 32) {
      float y[M];
      sample_y(s, y);
      const float *L, *U;
      const int nc = cells_of(s, L, U);
      const float h = sample_h<M>(y, L, U, nc, log, inv_tr, half_inv_tm, tm);
      if (log) lse_push(h, run_max, run_sum);
      else run_sum += h;
    }
    float value, lse = 0.f;
    if (log) {
      lse_warp_combine(run_max, run_sum);
      lse = run_max + logf(run_sum);
      // the M log(tau_relu) of every cell term is added once
      value = lse - logf((float)S) + (float)M * logf(p.tau_relu);
    } else {
      value = warp_sum(run_sum) / (float)S;
    }
    // pass 2: dA/dy_ms in chunks of 32 samples, reduced into A_mu, A_sd (lanes) and A_c (lane p: column p)
    float amu[M], asd[M];
#pragma unroll
    for (int m = 0; m < M; ++m) amu[m] = asd[m] = 0.f;
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      float g[M];
#pragma unroll
      for (int m = 0; m < M; ++m) g[m] = 0.f;
      if (s < S) {
        float y[M];
        sample_y(s, y);
        const float *L, *U;
        const int nc = cells_of(s, L, U);
        const float h = log ? sample_h<M>(y, L, U, nc, true, inv_tr, half_inv_tm, tm) : 0.f;
        sample_dh<M>(y, L, U, nc, log, h, inv_tr, half_inv_tm, tm, g);
        const float dadh = log ? (h > -INFINITY && lse > -INFINITY ? expf(h - lse) : 0.f) : 1.f / (float)S;
#pragma unroll
        for (int m = 0; m < M; ++m) g[m] *= dadh * p.a[m];
      }
      __syncwarp();
#pragma unroll
      for (int m = 0; m < M; ++m) {
        gc[lane * M + m] = g[m];
        amu[m] += g[m];
        if (s < S) asd[m] = fmaf(g[m], zc[s * M + m], asd[m]);
      }
      __syncwarp();
      if (lane < P) {
        const int ns = min(32, S - s0);
#pragma unroll
        for (int m = 0; m < M; ++m) {
          float* ac = wb + M * (dp + 3 * np) + 3 * M * 32 + m * 32;
          float acc = ac[lane];
          const float* wr = p.w + ((size_t)m * S + s0) * P + lane;
          for (int t = 0; t < ns; ++t) acc = fmaf(gc[t * M + m], __ldg(wr + (size_t)t * P), acc);
          ac[lane] = acc;
        }
      }
    }
    __syncwarp();
    // sd_m = sqrt(max(var_m - |r_m|^2, 0)): A_var and the sd's share of A_c, then back through each kernel row
    float gmu[M], gvar[M];
#pragma unroll
    for (int m = 0; m < M; ++m) {
      gmu[m] = warp_sum(amu[m]);
      const float a_sd = warp_sum(asd[m]);
      gvar[m] = target_sd_adjoint(a_sd, sd[m], P, p.plinv + (size_t)m * P * P, target_scratch(wb, M, m, np, dp), lane);
    }
    __syncwarp();
#pragma unroll
    for (int m = 0; m < M; ++m)
      target_row_adjoint(p.mdl[m], gmu[m], vfree[m] ? gvar[m] : 0.f, P, target_scratch(wb, M, m, np, dp), lane);
    __syncwarp();
    for (int j = lane; j < p.d; j += 32) {
      float gsum = 0.f;
#pragma unroll
      for (int m = 0; m < M; ++m) {
        const float g = target_col_grad(p.mdl[m], j, p.d, dp, P, p.pend_x, target_scratch(wb, M, m, np, dp));
        gsum = fmaf(g, __ldg(p.mdl[m].cand_scale + j), gsum);
      }
      p.grad[c * p.d + j] = gsum;
    }
    if (lane == 0) p.value[c] = value;
    __syncwarp();
  }
}

template <int FAMILY, int M>
static int launch_hvi_grad(const HviGradParams& p, size_t smem, int64_t blocks, cudaStream_t st) {
  BB_SMEM_OPTIN_ONCE((k_hvi_grad<FAMILY, M>));
  k_hvi_grad<FAMILY, M><<<(int)blocks, kHviGradThreads, smem, st>>>(p);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

}  // namespace bb

using namespace bb;

extern "C" int bb_hvi_grad(const bb_model* const* models, int32_t n_targets, const bb_acq_spec* a,
                           const float* obj_scale, const float* obj_shift, const float* d_x, int64_t N,
                           int32_t n_pending, const float* d_pend_x, const float* const* d_pend_beta,
                           const float* d_linv, const float* d_w, const float* d_z, int32_t S, const float* d_lower,
                           const float* d_upper, const int32_t* d_n_cells, int32_t cell_stride, float* d_value,
                           float* d_grad, void* stream) {
  BB_CHECK_ARG(a != nullptr, "bb_hvi_grad: acquisition spec is null");
  BB_CHECK_ARG(a->kind == BB_ACQ_QEHVI || a->kind == BB_ACQ_QLOGEHVI,
               "bb_hvi_grad: kind %d is not a hypervolume acquisition function", a->kind);
  BB_CHECK_ARG(!(a->kind == BB_ACQ_QLOGEHVI) || (a->tau_relu > 0.f && a->tau_max > 0.f),
               "bb_hvi_grad: qLogEHVI needs tau_relu > 0 and tau_max > 0");
  BB_CHECK_SUPPORTED(n_targets >= 2 && n_targets <= BB_HVI_MAX_TARGETS, "bb_hvi_grad: n_targets=%d outside [2,%d]",
                     n_targets, BB_HVI_MAX_TARGETS);
  BB_CHECK_ARG(models != nullptr, "bb_hvi_grad: model array is null");
  BB_CHECK_ARG(obj_scale != nullptr && obj_shift != nullptr, "bb_hvi_grad: null objective scale/shift");
  const int M = n_targets;
  for (int m = 0; m < M; ++m) {
    const bb_model* md = models[m];
    BB_CHECK_ARG(md && md->abi_version == BB_ABI_VERSION, "bb_hvi_grad: model %d missing or ABI mismatch", m);
    BB_CHECK_SUPPORTED(!md->wide, "bb_hvi_grad: model %d: wide-feature models are not supported", m);
    BB_CHECK_SUPPORTED(md->task_col < 0, "bb_hvi_grad: model %d: models with a task parameter are not supported", m);
    BB_CHECK_SUPPORTED(md->n_pad <= kGradMaxNPad, "bb_hvi_grad: model %d: n_pad=%d above %d is not supported", m,
                       md->n_pad, kGradMaxNPad);
    BB_CHECK_ARG(md->d == models[0]->d && md->d_pad == models[0]->d_pad && md->family == models[0]->family,
                 "bb_hvi_grad: model %d differs from model 0 in d or kernel family", m);
  }
  BB_CHECK_ARG(N >= 0, "bb_hvi_grad: negative point count");
  BB_CHECK_ARG(n_pending >= 0 && n_pending <= BB_MAX_PENDING, "bb_hvi_grad: n_pending=%d outside [0,%d]", n_pending,
               BB_MAX_PENDING);
  BB_CHECK_ARG(S >= 1 && S <= kMaxSamples, "bb_hvi_grad: S=%d outside [1,%d]", S, kMaxSamples);
  BB_CHECK_SUPPORTED(cell_stride >= 1 && cell_stride <= BB_HVI_MAX_CELLS, "bb_hvi_grad: cell_stride=%d outside [1,%d]",
                     cell_stride, BB_HVI_MAX_CELLS);
  bool pend_ok = n_pending == 0 || (d_pend_x && d_pend_beta && d_linv && d_w);
  for (int m = 0; pend_ok && n_pending > 0 && m < M; ++m) pend_ok = d_pend_beta[m] != nullptr;
  BB_CHECK_ARG(pend_ok, "bb_hvi_grad: pending points need rows, beta per model, linv and w");
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_x && d_z && d_lower && d_upper && d_n_cells && d_value && d_grad, "bb_hvi_grad: null buffer");
  HviGradParams p{};
  p.d = models[0]->d;
  p.d_pad = models[0]->d_pad;
  p.n_pad = 0;
  for (int m = 0; m < M; ++m) {
    const bb_model* md = models[m];
    GradTarget& g = p.mdl[m];
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
    p.a[m] = obj_scale[m];
    p.b[m] = obj_shift[m];
  }
  p.x = d_x;
  p.N = N;
  p.P = n_pending;
  p.pend_x = d_pend_x;
  p.plinv = d_linv;
  p.w = d_w;
  p.z = d_z;
  p.S = S;
  p.lower = d_lower;
  p.upper = d_upper;
  p.n_cells = d_n_cells;
  p.cells = cell_stride;
  p.log = a->kind == BB_ACQ_QLOGEHVI;
  p.tau_relu = a->kind == BB_ACQ_QLOGEHVI ? a->tau_relu : 1.0f;
  p.tau_max = a->kind == BB_ACQ_QLOGEHVI ? a->tau_max : 1.0f;
  p.value = d_value;
  p.grad = d_grad;
  int sms, max_smem;
  int rc = device_limits(&sms, &max_smem);
  if (rc != BB_OK) return rc;
  const size_t cells = n_pending == 0 ? 2 * (size_t)((cell_stride * M + 3) & ~3) : 0;
  const size_t smem =
      ((size_t)((S * M + 3) & ~3) + cells + (size_t)kHviGradWarps * target_warp_floats(M, p.n_pad, p.d_pad)) * 4;
  BB_CHECK_SUPPORTED(smem <= (size_t)max_smem, "bb_hvi_grad: %zu bytes of shared memory above %d", smem, max_smem);
  int64_t blocks = (N + kHviGradWarps - 1) / kHviGradWarps;
  if (blocks > (int64_t)sms * 8) blocks = (int64_t)sms * 8;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_family<true>(models[0]->family, [&](auto fam) {
    constexpr int F = decltype(fam)::value;
    switch (M) {
      case 2: return launch_hvi_grad<F, 2>(p, smem, blocks, st);
      case 3: return launch_hvi_grad<F, 3>(p, smem, blocks, st);
      default: return launch_hvi_grad<F, 4>(p, smem, blocks, st);
    }
  });
}
