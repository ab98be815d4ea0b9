// score_common.cuh -- scaffolding of the warp-per-candidate scoring kernels (k_hvi, k_objective, k_nei, k_parego).
//
// One warp scores one candidate: lane l takes base samples l, l+32, ..., and the launch runs a grid-stride loop over
// the candidates.  What the four kernels share lives here: the common part of their parameters, the candidate's
// moments conditional on the conditioning points, the join of a sample's term with the other points' terms, the
// arg-max epilogue, the host checks of the shared arguments and the launch.  Every reduction over lanes is a fixed
// xor tree, so a row's value does not depend on where it runs.
#pragma once

#include "acq_math.cuh"
#include "common.cuh"

namespace bb {

// The arguments every scoring kernel reads; each kernel's params struct derives from it and adds its own fields.
struct ScoreParams {
  int64_t N;
  const float *mu, *var;  // [M][N]
  const float* cross;     // [M][N][C]
  const float* linv;      // [M][C][C] L_C^-1 per target, row-major
  const float* w;         // [M][S][C] (k_hvi, k_objective) or sample-minor [M][C][S] (k_nei, k_parego)
  const float* z;         // [S][M(C+1)]
  const uint8_t* keep;
  float* score;
  long long* key;
  int64_t index_offset;
  int C, S;  // conditioning (pending) points, base samples
};

// Conditional moments of candidate i for targets 0..M-1 given the C = p.C points: mu[m], sd[m] = sqrt(max(var_m -
// |L_m^-1 c_m|^2, 0)) and this lane's entry cm[m] of c_m (0 for lanes >= C).  linv: the [M][C][C] factors in shared
// memory.  Every lane takes part in the shuffles.  C comes from the kernel's local copy rather than through `p`: read
// through the reference, ptxas allocates k_hvi<3, false> 40 registers and spills.
template <int M>
__device__ __forceinline__ void warp_cond_moments(const ScoreParams& p, const float* linv, int C, int64_t i, int lane,
                                                  float (&mu)[M], float (&sd)[M], float (&cm)[M]) {
#pragma unroll
  for (int m = 0; m < M; ++m) {
    const int64_t row = (int64_t)m * p.N + i;
    mu[m] = __ldg(p.mu + row);
    float r2 = 0.f;
    cm[m] = 0.f;
    if (C > 0) {
      cm[m] = (lane < C) ? __ldg(p.cross + row * C + lane) : 0.f;
      r2 = pending_r2_warp(cm[m], linv + m * C * C, C, lane);
    }
    sd[m] = sqrtf(fmaxf(__ldg(p.var + row) - r2, 0.f));
  }
}

// c_m . w_{m,s} of target m and this lane's sample s (callers pass 0 for lanes past S, which every lane must reach for
// the shuffles), with C conditioning points and S samples.  SAMPLE_MINOR picks the w layout: [M][C][S] (stride S,
// loads coalesce across the warp) or [M][S][C] (stride 1).
template <bool SAMPLE_MINOR>
__device__ __forceinline__ float warp_cond_shift(const float* w, float cm, int m, int s, int C, int S) {
  if (SAMPLE_MINOR) return pending_cw_warp(cm, w + (size_t)m * C * S + s, C, S);
  return pending_cw_warp(cm, w + ((size_t)m * S + s) * C, C);
}

// A sample's term joined with the per-sample terms tr[0..Q) of the other points of the batch: their hard maximum,
// or with FAT botorch's fatmax (tau_max).  li: scratch of BB_MAX_PENDING + 1 floats.
__device__ __forceinline__ float join_terms(float term, const float* tr, int Q, float* li, bool fat, float tau_max) {
  float mx = term;
  li[0] = term;
  for (int j = 0; j < Q; ++j) {
    const float v = __ldg(tr + j);
    li[j + 1] = v;
    mx = fmaxf(mx, v);
  }
  return fat ? fatmax_q(li, Q + 1, mx, tau_max) : mx;
}

// Lane 0 stores candidate i's value and offers it to the warp's running best key (kept rows only, NaN skipped).
__device__ __forceinline__ void warp_offer_best(const ScoreParams& p, int64_t i, float result, int lane,
                                                long long& best) {
  if (lane == 0) {
    if (p.score) p.score[i] = result;
    if ((p.keep == nullptr || p.keep[i] != 0) && !(result != result)) {
      const long long k = pack_key(result, (uint32_t)(i + p.index_offset));
      best = k > best ? k : best;
    }
  }
}

// The block's best key over its warps, merged into *key by one atomicMax (called by every thread of the block).
template <int THREADS>
__device__ __forceinline__ void block_flush_best(long long best, long long* key) {
  __shared__ long long red[THREADS / 32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long b = red[0];
    for (int w = 1; w < THREADS / 32; ++w) b = red[w] > b ? red[w] : b;
    if (b != kEmptyKey) atomicMax(key, b);
  }
}

// Host checks of the shared arguments, in this order: the 32-bit key range, the conditioning count (`noun`: n_cond or
// n_pending), S (unless `check_S` is false: analytic kinds take no samples) and the best key.
static inline int check_score_args(const char* fn, const char* noun, int64_t N, int64_t index_offset, int n_cond,
                                   int S, bool check_S, const int64_t* d_best_key) {
  BB_CHECK_ARG(N >= 0 && N + index_offset < 0xffffffffLL && index_offset >= 0, "%s: index outside 32-bit key range",
               fn);
  BB_CHECK_ARG(n_cond >= 0 && n_cond <= BB_MAX_PENDING, "%s: %s=%d outside [0,%d]", fn, noun, n_cond, BB_MAX_PENDING);
  BB_CHECK_ARG(!check_S || (S >= 1 && S <= 1024), "%s: S=%d outside [1,1024]", fn, S);
  BB_CHECK_ARG(d_best_key != nullptr, "%s: null best key", fn);
  return BB_OK;
}

// One warp per candidate, capped at BLOCKS_PER_SM resident blocks per SM (the grid-stride loop covers the rest); the
// kernel is opted in to the full dynamic shared memory once per device.
template <auto KERNEL, int THREADS, int BLOCKS_PER_SM, class Params>
static int launch_warp_per_candidate(const Params& p, size_t smem, cudaStream_t st) {
  BB_SMEM_OPTIN_ONCE(KERNEL);
  int64_t blocks = (p.N + THREADS / 32 - 1) / (THREADS / 32);
  if (blocks > kSMs * BLOCKS_PER_SM) blocks = kSMs * BLOCKS_PER_SM;
  KERNEL<<<(int)blocks, THREADS, smem, st>>>(p);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

}  // namespace bb
