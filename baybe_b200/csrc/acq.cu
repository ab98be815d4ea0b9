// acq.cu -- stand-alone acquisition scoring and selection kernels:
//   k_acq_moments : q=1 score from (mu, var); warp per candidate, base samples in registers,
//                   warp-shuffle reduction (SURVEY.md K6)
//   k_acq_joint   : joint MC score of [x*; pending] per candidate (sequential greedy, K9)
//   k_argmax / top-k (K7)
// Reference: botorch MC acquisition forward + optimize_acqf_discrete's argmax, reached from
// /root/reference/baybe/recommenders/pure/bayesian/botorch/discrete.py:124-126.
#include <math.h>

#include "acq_math.cuh"
#include "common.cuh"

namespace bb {

// ------------------------------------------------------------------------------------------
// q = 1 from moments
// ------------------------------------------------------------------------------------------
constexpr int kZPerLane = 32;  // S <= 1024

template <int KIND>
__device__ __forceinline__ void lane_terms(const float (&z)[kZPerLane], int nz_full, int nz_tail_lanes,
                                           int lane, float c0, float c1, float& s0, float& s1) {
#pragma unroll
  for (int k = 0; k < kZPerLane; ++k) {
    if (k < nz_full || (k == nz_full && lane < nz_tail_lanes)) mc_term<KIND>(fmaf(c1, z[k], c0), s0, s1);
  }
}

__global__ void __launch_bounds__(256) k_acq_moments(const bb_acq_spec a, const float* __restrict__ mu,
                                                    const float* __restrict__ var, int64_t N,
                                                    const float* __restrict__ zg, int S,
                                                    float* __restrict__ score) {
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const bool is_mc = a.kind <= BB_ACQ_QPI;
  if (!is_mc) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N;
         i += (int64_t)gridDim.x * blockDim.x)
      score[i] = analytic_value(a, mu[i], var[i]);
    return;
  }
  // each lane keeps samples lane, lane+32, ... in registers for the whole kernel
  float z[kZPerLane];
  const int nz_full = S >> 5, nz_tail_lanes = S & 31;
  float sz = 0.f, sa = 0.f;
#pragma unroll
  for (int k = 0; k < kZPerLane; ++k) {
    const int s = k * 32 + lane;
    z[k] = (s < S) ? __ldg(zg + s) : 0.f;
    sz += z[k];
  }
  for (int o = 16; o > 0; o >>= 1) sz += __shfl_xor_sync(0xffffffffu, sz, o);
  const float z_mean = sz / (float)S;
  // qUCB centres on the SAMPLE mean (botorch qUpperConfidenceBound._sample_forward: mean = obj.mean(dim=0))
#pragma unroll
  for (int k = 0; k < kZPerLane; ++k)
    if (k * 32 + lane < S) sa += fabsf(z[k] - z_mean);
  for (int o = 16; o > 0; o >>= 1) sa += __shfl_xor_sync(0xffffffffu, sa, o);
  const float zdev_mean = sa / (float)S;
  for (int64_t i = warp_global; i < N; i += nwarps) {
    const float m = __ldg(mu + i), v = __ldg(var + i);
    float c0, c1, s0 = 0.f, s1 = 0.f;
    mc_coef(a, m, v, c0, c1);
    if (a.kind == BB_ACQ_QLOGEI) lane_terms<BB_ACQ_QLOGEI>(z, nz_full, nz_tail_lanes, lane, c0, c1, s0, s1);
    else if (a.kind == BB_ACQ_QEI) lane_terms<BB_ACQ_QEI>(z, nz_full, nz_tail_lanes, lane, c0, c1, s0, s1);
    else if (a.kind == BB_ACQ_QPI) lane_terms<BB_ACQ_QPI>(z, nz_full, nz_tail_lanes, lane, c0, c1, s0, s1);
    for (int o = 16; o > 0; o >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, o);
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    }
    if (lane == 0) score[i] = mc_finalize(a, m, v, s0, s1, S, z_mean, zdev_mean);
  }
}

// ------------------------------------------------------------------------------------------
// joint [x*; pending] scoring
// ------------------------------------------------------------------------------------------
struct JointParams {
  bb_acq_spec a;
  const float *mu, *var, *cross;
  int64_t N;
  const float *pend_mu, *pend_cov;
  int P;
  const float* z;  // [S][1+P]
  int S;
  float* score;
};

__device__ __forceinline__ float log_fatplus_f(float x, float tau) {
  // log( tau * (softplus(t) + 0.1/(1+t^2)) ), t = x/tau
  return logf(tau) + log_fatplus_t(x / tau);
}

__global__ void __launch_bounds__(256) k_acq_joint(const JointParams p) {
  extern __shared__ __align__(16) float smem_j[];
  const int P = p.P, Q = P + 1;
  const int zs = Q | 1;  // odd row stride: conflict-free per-lane sample rows
  float* z_s = smem_j;                      // [S][zs]
  float* wbase = z_s + (size_t)p.S * zs;    // per warp: L [P][P], l [P], muP [P]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per_warp = P * P + 3 * P + 2;
  float* Lw = wbase + warp * per_warp;
  float* lv = Lw + P * P;
  float* mP = lv + P;
  float* moP = mP + P;  // qUCB: sample mean of every pending point's objective
  for (int e = threadIdx.x; e < p.S * Q; e += blockDim.x) {
    int s = e / Q, k = e - s * Q;
    z_s[s * zs + k] = __ldg(p.z + e);
  }
  __syncthreads();
  const bb_acq_spec a = p.a;
  const float ucb_c = sqrtf(a.beta * 1.5707963267948966f);
  // column means of the base samples (lane k: column k): the sample mean of an objective is affine in them
  float zb = 0.f;
  if (lane < Q) {
    for (int s = 0; s < p.S; ++s) zb += z_s[s * zs + lane];
    zb /= (float)p.S;
  }
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = warp_global; c < p.N; c += nwarps) {
    const float mu_c = __ldg(p.mu + c);
    float var_c = __ldg(p.var + c);
    const float cr = (lane < P) ? __ldg(p.cross + c * P + lane) : 0.f;
    // ---- Cholesky of the joint covariance, candidate first: L = [[sd,0],[l, chol(S22)]] ----
    float sd = 0.f;
    bool ok = false;
    for (int attempt = 0; attempt < 4 && !ok; ++attempt) {
      // linear_operator psd_safe_cholesky (float32 settings): plain, then 1e-6 * 10^i
      const float jit = attempt == 0 ? 0.f : 1e-6f * __powf(10.f, (float)(attempt - 1));
      sd = sqrtf(var_c + jit);
      const float li = cr / sd;
      __syncwarp();
      if (lane < P) {
        lv[lane] = li;
        mP[lane] = __ldg(p.pend_mu + lane);
      }
      __syncwarp();
      if (lane < P)
        for (int j = 0; j <= lane; ++j)
          Lw[lane * P + j] = __ldg(p.pend_cov + lane * P + j) - li * lv[j] + (j == lane ? jit : 0.f);
      __syncwarp();
      bool fail = !(var_c + jit > 0.f);
      for (int j = 0; j < P; ++j) {
        const float dj = Lw[j * P + j];
        if (!(dj > 0.f)) {
          fail = true;
          break;
        }
        const float sj = sqrtf(dj);
        __syncwarp();
        if (lane == j) Lw[j * P + j] = sj;
        if (lane > j && lane < P) Lw[lane * P + j] /= sj;
        __syncwarp();
        if (lane > j && lane < P) {
          const float lij = Lw[lane * P + j];
          for (int k = j + 1; k <= lane; ++k) Lw[lane * P + k] -= lij * Lw[k * P + j];
        }
        __syncwarp();
      }
      ok = !fail;
    }
    __syncwarp();
    // ---- Monte-Carlo over the shared base samples ----
    const float a1 = a.obj_scale, a0 = a.obj_shift;
    // qUCB: botorch centres |o_s - mean| on the sample mean over s (obj.mean(dim=0)) of every point
    const float zb0 = __shfl_sync(0xffffffffu, zb, 0);
    {
      float ym = (lane < P) ? fmaf(lv[lane], zb0, mP[lane]) : 0.f;
      for (int j = 0; j < P; ++j) {
        const float zbj = __shfl_sync(0xffffffffu, zb, 1 + j);
        if (lane < P && j <= lane) ym = fmaf(Lw[lane * P + j], zbj, ym);
      }
      if (lane < P) moP[lane] = fmaf(a1, ym, a0);
      __syncwarp();
    }
    const float mo_c = fmaf(a1, fmaf(sd, zb0, mu_c), a0);
    float run_max = -INFINITY, run_sum = 0.f;  // qLogEI: online logsumexp; others: plain sum
    for (int s = lane; s < p.S; s += 32) {
      const float* zr = z_s + s * zs;
      const float z0 = zr[0];
      float o = fmaf(a1, fmaf(sd, z0, mu_c), a0);
      float li_arr[BB_MAX_PENDING + 1];
      float red;  // per-sample reduction over the q = 1+P points
      if (a.kind == BB_ACQ_QLOGEI) {
        li_arr[0] = log_fatplus_f(o - a.best_f, a.tau_relu);
        red = li_arr[0];
      } else if (a.kind == BB_ACQ_QEI) red = fmaxf(o - a.best_f, 0.f);
      else if (a.kind == BB_ACQ_QSR) red = o;
      else if (a.kind == BB_ACQ_QPI) red = 1.0f / (1.0f + __expf(-(o - a.best_f) / a.tau_pi));
      else red = mo_c + ucb_c * fabsf(o - mo_c);
      for (int i = 0; i < P; ++i) {
        float y = fmaf(lv[i], z0, mP[i]);
        const float* Li = Lw + i * P;
        for (int j = 0; j <= i; ++j) y = fmaf(Li[j], zr[1 + j], y);
        o = fmaf(a1, y, a0);
        float val;
        if (a.kind == BB_ACQ_QLOGEI) {
          val = log_fatplus_f(o - a.best_f, a.tau_relu);
          li_arr[i + 1] = val;
        } else if (a.kind == BB_ACQ_QEI) val = fmaxf(o - a.best_f, 0.f);
        else if (a.kind == BB_ACQ_QSR) val = o;
        else if (a.kind == BB_ACQ_QPI) val = 1.0f / (1.0f + __expf(-(o - a.best_f) / a.tau_pi));
        else {
          const float mo_i = moP[i];
          val = mo_i + ucb_c * fabsf(o - mo_i);
        }
        red = fmaxf(red, val);
      }
      if (a.kind == BB_ACQ_QLOGEI) {
        // fatmax over the q points: M + tau * log sum (1 + (M - li)/(2 tau))^-2
        float ssum = 0.f;
        const float inv = 1.0f / (2.0f * a.tau_max);
        for (int k = 0; k < Q; ++k) {
          const float w = fmaf(red - li_arr[k], inv, 1.0f);
          ssum += 1.0f / (w * w);
        }
        const float li = red + a.tau_max * logf(ssum);
        if (li > run_max) {
          run_sum = run_sum * __expf(run_max - li) + 1.0f;
          run_max = li;
        } else {
          run_sum += __expf(li - run_max);
        }
      } else {
        run_sum += red;
      }
    }
    float result;
    if (a.kind == BB_ACQ_QLOGEI) {
      for (int o2 = 16; o2 > 0; o2 >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, run_max, o2);
        const float os = __shfl_xor_sync(0xffffffffu, run_sum, o2);
        const float nm = fmaxf(run_max, om);
        float acc = 0.f;
        if (run_max > -INFINITY) acc += run_sum * __expf(run_max - nm);
        if (om > -INFINITY) acc += os * __expf(om - nm);
        run_max = nm;
        run_sum = acc;
      }
      result = run_max + logf(run_sum) - logf((float)p.S);
    } else {
      for (int o2 = 16; o2 > 0; o2 >>= 1) run_sum += __shfl_xor_sync(0xffffffffu, run_sum, o2);
      result = run_sum / (float)p.S;
    }
    if (lane == 0) p.score[c] = ok ? result : __int_as_float(0x7fc00000);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------
// arg-max / top-k
// ------------------------------------------------------------------------------------------
__global__ void k_key_init(long long* key) { key[0] = kEmptyKey; }

__global__ void __launch_bounds__(256) k_argmax(const float* __restrict__ score,
                                                const uint8_t* __restrict__ keep, int64_t N,
                                                int64_t index_offset, long long* __restrict__ key) {
  __shared__ long long red[8];
  long long best = kEmptyKey;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float s = score[i];
    if ((keep == nullptr || keep[i] != 0) && !(s != s)) {
      const long long k = pack_key(s, (uint32_t)(i + index_offset));
      best = k > best ? k : best;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const long long other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other > best ? other : best;
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long b = red[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) b = red[w] > b ? red[w] : b;
    if (b != kEmptyKey) atomicMax(key, b);
  }
}

__device__ __forceinline__ void decode_key(long long key, float& val, long long& idx) {
  if (key == kEmptyKey) {
    val = -INFINITY;
    idx = -1;
    return;
  }
  int32_t s = (int32_t)(key >> 32);
  s ^= (s >> 31) & 0x7fffffff;
  val = __int_as_float(s);
  idx = (long long)(0xffffffffu - (uint32_t)(key & 0xffffffffLL));
}

__global__ void k_key_decode(const long long* key, bb_best* out) {
  float v;
  long long i;
  decode_key(key[0], v, i);
  out->val = v;
  out->pad_ = 0;
  out->idx = i;
}

__global__ void k_mask_init(const uint8_t* __restrict__ keep, uint8_t* __restrict__ mask, int64_t N) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N;
       i += (int64_t)gridDim.x * blockDim.x)
    mask[i] = keep ? keep[i] : (uint8_t)1;
}

__global__ void k_topk_step(long long* key, int slot, float* vals, long long* idx, uint8_t* mask) {
  float v;
  long long i;
  decode_key(key[0], v, i);
  vals[slot] = v;
  idx[slot] = i;
  if (i >= 0) mask[i] = 0;
  key[0] = kEmptyKey;
}

static int grid_for(int64_t N, int block, int cap) {
  int64_t g = (N + block - 1) / block;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace bb

using namespace bb;

static int check_acq(const bb_acq_spec* a) {
  BB_CHECK_ARG(a != nullptr, "acquisition spec is null");
  BB_CHECK_ARG(a->kind >= BB_ACQ_QLOGEI && a->kind <= BB_ACQ_PSTD, "unknown acquisition kind %d",
               a->kind);
  return BB_OK;
}

extern "C" int bb_acq_score(const bb_acq_spec* a, const float* d_mu, const float* d_var, int64_t N,
                            const float* d_z, int32_t S, float* d_score, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  int rc = check_acq(a);
  if (rc != BB_OK) return rc;
  BB_CHECK_ARG(N >= 0, "negative candidate count");
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_mu && d_var && d_score, "bb_acq_score: null buffer");
  const bool is_mc = a->kind <= BB_ACQ_QPI;
  BB_CHECK_ARG(!is_mc || (d_z != nullptr && S >= 1 && S <= 32 * kZPerLane),
               "bb_acq_score: MC kinds need base samples, 1 <= S <= %d (got %d)", 32 * kZPerLane, S);
  int grid = is_mc ? grid_for(N * 32, 256, kSMs * 8) : grid_for(N, 256, kSMs * 8);
  k_acq_moments<<<grid, 256, 0, stream>>>(*a, d_mu, d_var, N, d_z, is_mc ? S : 0, d_score);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

extern "C" int bb_acq_score_joint(const bb_acq_spec* a, const float* d_mu, const float* d_var,
                                  const float* d_cross, int64_t N, const float* d_pend_mu,
                                  const float* d_pend_cov, int32_t P, const float* d_z, int32_t S,
                                  float* d_score, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  int rc = check_acq(a);
  if (rc != BB_OK) return rc;
  BB_CHECK_ARG(a->kind <= BB_ACQ_QPI,
               "bb_acq_score_joint: pending points need a Monte Carlo acquisition function");
  BB_CHECK_ARG(P >= 1 && P <= BB_MAX_PENDING, "bb_acq_score_joint: n_pending=%d outside [1,%d]", P,
               BB_MAX_PENDING);
  BB_CHECK_ARG(S >= 1 && S <= 1024, "bb_acq_score_joint: S=%d outside [1,1024]", S);
  BB_CHECK_ARG(N >= 0, "negative candidate count");
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_mu && d_var && d_cross && d_pend_mu && d_pend_cov && d_z && d_score,
               "bb_acq_score_joint: null buffer");
  JointParams p;
  p.a = *a;
  p.mu = d_mu;
  p.var = d_var;
  p.cross = d_cross;
  p.N = N;
  p.pend_mu = d_pend_mu;
  p.pend_cov = d_pend_cov;
  p.P = P;
  p.z = d_z;
  p.S = S;
  p.score = d_score;
  const int zs = (P + 1) | 1;
  size_t smem = ((size_t)S * zs + 8 * (size_t)(P * P + 3 * P + 2)) * 4;
  int dev = 0, max_smem = 0;
  BB_CUDA(cudaGetDevice(&dev));
  BB_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  BB_CHECK_SUPPORTED(smem <= (size_t)max_smem, "bb_acq_score_joint: S*(1+P) too large for shared memory");
  BB_CUDA(cudaFuncSetAttribute(k_acq_joint, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = grid_for(N * 32, 256, kSMs * 2);
  k_acq_joint<<<grid, 256, smem, stream>>>(p);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

extern "C" int bb_best_init(int64_t* d_best_key, void* stream) {
  BB_CHECK_ARG(d_best_key != nullptr, "bb_best_init: null key");
  k_key_init<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<long long*>(d_best_key));
  BB_LAUNCH_CHECK();
  return BB_OK;
}

extern "C" int bb_argmax(const float* d_score, const uint8_t* d_keep, int64_t N,
                         int64_t index_offset, int64_t* d_best_key, void* stream) {
  BB_CHECK_ARG(d_best_key != nullptr && (d_score != nullptr || N == 0), "bb_argmax: null buffer");
  BB_CHECK_ARG(N >= 0 && N + index_offset < 0xffffffffLL, "bb_argmax: index outside 32-bit key range");
  if (N == 0) return BB_OK;
  k_argmax<<<grid_for(N, 256, kSMs * 8), 256, 0, (cudaStream_t)stream>>>(
      d_score, d_keep, N, index_offset, reinterpret_cast<long long*>(d_best_key));
  BB_LAUNCH_CHECK();
  return BB_OK;
}

extern "C" int bb_best_decode(const int64_t* d_best_key, bb_best* d_out, void* stream) {
  BB_CHECK_ARG(d_best_key && d_out, "bb_best_decode: null buffer");
  k_key_decode<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<const long long*>(d_best_key), d_out);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

extern "C" int bb_topk(const float* d_score, const uint8_t* d_keep, int64_t N, int32_t k,
                       float* d_vals, int64_t* d_idx, uint8_t* d_scratch_mask,
                       int64_t* d_scratch_key, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  BB_CHECK_ARG(d_score && d_vals && d_idx && d_scratch_mask && d_scratch_key, "bb_topk: null buffer");
  BB_CHECK_ARG(k >= 1 && N >= 1 && N < 0xffffffffLL, "bb_topk: need k >= 1 and 1 <= N < 2^32");
  const int grid = grid_for(N, 256, kSMs * 8);
  k_mask_init<<<grid, 256, 0, stream>>>(d_keep, d_scratch_mask, N);
  BB_LAUNCH_CHECK();
  k_key_init<<<1, 1, 0, stream>>>(reinterpret_cast<long long*>(d_scratch_key));
  BB_LAUNCH_CHECK();
  for (int i = 0; i < k; ++i) {
    k_argmax<<<grid, 256, 0, stream>>>(d_score, d_scratch_mask, N, 0,
                                       reinterpret_cast<long long*>(d_scratch_key));
    BB_LAUNCH_CHECK();
    k_topk_step<<<1, 1, 0, stream>>>(reinterpret_cast<long long*>(d_scratch_key), i, d_vals,
                                     reinterpret_cast<long long*>(d_idx), d_scratch_mask);
    BB_LAUNCH_CHECK();
  }
  return BB_OK;
}

// ------------------------------------------------------------------------------------------------------------
// qNEI / qLogNEI-style noisy improvement of ONE new point per row, conditional on joint samples of a conditioning
// set C = [baseline; pending] (SURVEY.md 8f-2: acquisition/acqfs.py:227-240, X_baseline from _builder.py:319-324).
// With the joint Cholesky taken in the order [C ; x], the sample path of the new point is
//   f_x,s = mu_x + r_x . Z_C[s,:] + sqrt(max(var_x - |r_x|^2, 0)) z_x,s ,      r_x = Sigma_xC L_C^-T ,
// and the value of x is  mean_s relu( o(f_x,s) - g_s ),  g_s = max(o over the samples of C)  (the marginal gain of
// adding x to the pending set; the part that does not depend on x is added by the caller).
// d_out row i = [ Delta_i[0..S) = r_i . Z_C^T | r_i[0..m) ]  (one GEMM of the caller: Sigma_XC @ [W | L_C^-T]).
// One warp per row: |r|^2 by a shuffle reduction, then the S samples in lane-strided order (fixed order).
// ------------------------------------------------------------------------------------------------------------
namespace bb {
__global__ void __launch_bounds__(256) k_nei_reduce(const float* __restrict__ out, int64_t ld, int S, int m,
                                                    const float* __restrict__ mu, const float* __restrict__ var,
                                                    const float* __restrict__ zx, const float* __restrict__ g,
                                                    float obj_scale, float obj_shift, int64_t N,
                                                    float* __restrict__ score) {
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp0; i < N; i += nwarps) {
    const float* row = out + i * ld;
    float r2 = 0.f;
    for (int j = lane; j < m; j += 32) {
      const float r = row[S + j];
      r2 = fmaf(r, r, r2);
    }
    for (int o = 16; o > 0; o >>= 1) r2 += __shfl_xor_sync(0xffffffffu, r2, o);
    const float sc = sqrtf(fmaxf(var[i] - r2, 0.f));
    const float m0 = mu[i];
    float acc = 0.f;
    for (int s = lane; s < S; s += 32) {
      const float f = m0 + row[s] + sc * zx[s];
      acc += fmaxf(fmaf(obj_scale, f, obj_shift) - g[s], 0.f);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) score[i] = acc / (float)S;
  }
}
}  // namespace bb

extern "C" int bb_nei_reduce(const float* d_out, int64_t ld, int32_t S, int32_t m, const float* d_mu,
                             const float* d_var, const float* d_zx, const float* d_g, float obj_scale,
                             float obj_shift, int64_t N, float* d_score, void* stream) {
  BB_CHECK_ARG(N >= 0 && S >= 1 && m >= 0 && ld >= (int64_t)S + m, "bb_nei_reduce: bad shape (N=%lld S=%d m=%d ld=%lld)",
               (long long)N, S, m, (long long)ld);
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_out && d_mu && d_var && d_zx && d_g && d_score, "bb_nei_reduce: null buffer");
  const int64_t want = (N * 32 + 255) / 256;
  const int grid = (int)(want < (int64_t)kSMs * 16 ? want : (int64_t)kSMs * 16);
  bb::k_nei_reduce<<<grid, 256, 0, (cudaStream_t)stream>>>(d_out, ld, S, m, d_mu, d_var, d_zx, d_g, obj_scale, obj_shift,
                                                         N, d_score);
  BB_LAUNCH_CHECK();
  return BB_OK;
}
