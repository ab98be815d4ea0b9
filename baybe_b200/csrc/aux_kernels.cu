// aux_kernels.cu -- kernels around the fused hot path that share its K-assembly core:
//   k_kmat   : stand-alone K(X*, X) (fp32 out; the HBM-bound kernel of SURVEY.md K2)
//   k_cross  : posterior covariance of every candidate with the pending points (K9 prologue)
//   k_simt   : test-only fp32 SIMT posterior (direct-difference distances, no tensor cores)
#include "assemble.cuh"
#include "fused_common.cuh"
#include "common.cuh"

namespace bb {

constexpr int kAuxThreads = 512;
constexpr int kKsStride = 68;  // floats per staged row: 64 + 4 keeps STS.128 conflict-free

struct AuxParams {
  const void* x;
  int layout;
  int64_t N, ldx;
  int num_tiles;
  const float *cand_scale, *cand_shift, *train_m2, *train_sq, *task_covar;
  const int32_t* train_task;
  int n, n_pad, d, d_pad, n_chunks, task_col, n_tasks, scaled;
  float y_std;
  // kmat
  float* kout;
  int64_t ldk;
  // cross
  const float *pend_x, *pend_beta;
  int P;
  float* cross;
  // simt
  const float *alpha, *mean_const, *linv32;
  float y_mean;
  float *mu, *var;
};

// Shared memory of k_kmat and k_cross: the assembly core's buffers, then each kernel's own.
struct AuxSmem {
  float4 *xt4, *a_s;
  float *tsq, *tcov, *cscale, *cshift;
  int32_t *ttask, *cand_task;
  float* ks;  // k_kmat: [128][kKsStride] staged output rows
  float *cross_s, *psq;  // k_cross: [128][32] partial sums, [32] squared norms of the pending rows
  float4* pxt4;          // k_cross: [dq][32] pending rows, pair-interleaved like the training rows
  int32_t* ptask;        // k_cross: [32]
};

static __host__ __device__ SmemCarver carve_asm(uint8_t* base, const AuxParams& p, AuxSmem& s) {
  SmemCarver c{base};
  s.xt4 = c.take<float4>((size_t)p.n_pad * p.d_pad * 4);
  s.tsq = c.take<float>((size_t)p.n_pad * 4);
  s.ttask = c.take<int32_t>((size_t)p.n_pad * 4);
  s.a_s = c.take<float4>((size_t)kTileM * p.d_pad * 8);  // duplicated candidate values
  s.tcov = c.take<float>(kMaxTasks * kMaxTasks * 4);
  s.cand_task = c.take<int32_t>(kTileM * 4);
  s.cscale = c.take<float>((size_t)p.d_pad * 4);
  s.cshift = c.take<float>((size_t)p.d_pad * 4);
  return c;
}

static __host__ __device__ size_t carve_kmat(uint8_t* base, const AuxParams& p, AuxSmem& s) {
  SmemCarver c = carve_asm(base, p, s);
  s.ks = c.take<float>((size_t)kTileM * kKsStride * 4);
  return c.bytes;
}

static __host__ __device__ size_t carve_cross(uint8_t* base, const AuxParams& p, AuxSmem& s) {
  SmemCarver c = carve_asm(base, p, s);
  s.cross_s = c.take<float>(kTileM * 32 * 4);
  s.pxt4 = c.take<float4>((size_t)32 * p.d_pad * 4);
  s.psq = c.take<float>(32 * 4);
  s.ptask = c.take<int32_t>(32 * 4);
  return c.bytes;
}

// How the assembly core (sm) and the candidate staging (sc) see the shared buffers.
struct AuxCore {
  AsmSmem sm;
  StageCtx sc;
};

// Loads the model data of the assembly core into shared memory.
__device__ __forceinline__ AuxCore aux_setup(const AuxSmem& s, const AuxParams& p, int tid, int nthreads) {
  const int dq = p.d_pad >> 2;
  load_train_rows(s.xt4, p.train_m2, p.n_pad, dq, tid, nthreads);
  for (int e = tid; e < p.d_pad; e += nthreads) {
    s.cscale[e] = __ldg(p.cand_scale + e);
    s.cshift[e] = __ldg(p.cand_shift + e);
  }
  for (int e = tid; e < p.n_pad; e += nthreads) {
    s.tsq[e] = __ldg(p.train_sq + e);
    s.ttask[e] = __ldg(p.train_task + e);
  }
  for (int e = tid; e < p.n_tasks * p.n_tasks; e += nthreads) s.tcov[e] = __ldg(p.task_covar + e);
  for (int e = tid; e < kTileM; e += nthreads) s.cand_task[e] = 0;
  AuxCore r;
  r.sm.xt4 = s.xt4;
  r.sm.tsq = s.tsq;
  r.sm.ttask = s.ttask;
  r.sm.tcov = s.tcov;
  r.sm.a_s = s.a_s;
  r.sm.cand_task = s.cand_task;
  r.sm.dq = dq;
  r.sm.np = p.n_pad;
  r.sm.T = p.n_tasks;
  r.sm.scaled = p.scaled != 0;
  r.sc.x = p.x;
  r.sc.layout = p.layout;
  r.sc.N = p.N;
  r.sc.ldx = p.ldx;
  r.sc.d = p.d;
  r.sc.task_col = p.task_col;
  r.sc.cscale = s.cscale;
  r.sc.cshift = s.cshift;
  r.sc.groups = nthreads / kTileM;
  r.sc.gated = false;
  r.sc.code_table = nullptr;
  r.sc.code_table_ld = 0;
  return r;
}

// ------------------------------------------------------------------------------------------
// K(X*, X): tile of 128 candidates, 64 training points at a time, staged through shared
// memory so that every global store is a full 256-byte row segment.
// ------------------------------------------------------------------------------------------
template <int FAMILY>
__global__ void __launch_bounds__(kAuxThreads, 1) k_kmat(const AuxParams p) {
  extern __shared__ __align__(16) uint8_t smem_aux[];
  const int tid = threadIdx.x;
  AuxSmem s;
  carve_kmat(smem_aux, p, s);
  const AuxCore core = aux_setup(s, p, tid, kAuxThreads);
  const AsmSmem& sm = core.sm;
  const StageCtx& sc = core.sc;
  float* ks = s.ks;
  __syncthreads();
  const int mp = tid & 63, g = tid >> 6;
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(p.kout) & 15) == 0) && ((p.ldk & 3) == 0);
  StageRegs regs;
  if ((int)blockIdx.x < p.num_tiles) stage_prefetch(sc, sm.dq, (int64_t)blockIdx.x * kTileM, tid, regs);
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int64_t row0 = (int64_t)tile * kTileM;
    stage_commit(sc, sm.a_s, sm.cand_task, sm.T, sm.dq, row0, tid, regs);
    __syncthreads();
    if (tile + (int)gridDim.x < p.num_tiles)
      stage_prefetch(sc, sm.dq, (int64_t)(tile + gridDim.x) * kTileM, tid, regs);
    const float an0 = cand_sqnorm(sm, mp), an1 = cand_sqnorm(sm, mp + 64);
    for (int c = 0; c < p.n_chunks; ++c) {
      float k0[8], k1[8];
      assemble_2x8<FAMILY>(sm, mp, mp + 64, an0, an1, c * kChunk + g * 8, k0, k1);
      float4* d0 = reinterpret_cast<float4*>(ks + mp * kKsStride + g * 8);
      float4* d1 = reinterpret_cast<float4*>(ks + (mp + 64) * kKsStride + g * 8);
      d0[0] = make_float4(k0[0], k0[1], k0[2], k0[3]);
      d0[1] = make_float4(k0[4], k0[5], k0[6], k0[7]);
      d1[0] = make_float4(k1[0], k1[1], k1[2], k1[3]);
      d1[1] = make_float4(k1[4], k1[5], k1[6], k1[7]);
      __syncthreads();
      const int c4 = tid & 15;
      const int i = c * kChunk + c4 * 4;
#pragma unroll
      for (int rr = 0; rr < 4; ++rr) {
        const int r = (tid >> 4) + rr * 32;
        const int64_t row = row0 + r;
        if (row < p.N && i < p.n) {
          const float4 v = *reinterpret_cast<const float4*>(ks + r * kKsStride + c4 * 4);
          float* dst = p.kout + row * p.ldk + i;
          if (vec_ok && i + 3 < p.n) {
            *reinterpret_cast<float4*>(dst) = v;
          } else {
            dst[0] = v.x;
            if (i + 1 < p.n) dst[1] = v.y;
            if (i + 2 < p.n) dst[2] = v.z;
            if (i + 3 < p.n) dst[3] = v.w;
          }
        }
      }
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------------------------------
// cross[row][p] = y_std^2 * ( k(x*, p) - sum_i k(x*, x_i) beta_p[i] ),  beta_p = K^-1 k(X, p)
// ------------------------------------------------------------------------------------------
template <int FAMILY>
__global__ void __launch_bounds__(256, 1) k_cross(const AuxParams p) {
  extern __shared__ __align__(16) uint8_t smem_aux[];
  const int tid = threadIdx.x;
  AuxSmem s;
  carve_cross(smem_aux, p, s);
  const AuxCore core = aux_setup(s, p, tid, 256);
  const AsmSmem& sm = core.sm;
  const StageCtx& sc = core.sc;
  float* cross_s = s.cross_s;
  float4* pxt4 = s.pxt4;
  float* psq = s.psq;
  int32_t* ptask = s.ptask;
  // scaled pending rows, laid out like the training rows (-2 b, quad-major) + squared norms
  for (int e = tid; e < 32 * p.d_pad; e += 256) {
    int pp = e / p.d_pad, j = e - pp * p.d_pad;
    float b = 0.f;
    if (pp < p.P && j < p.d)
      b = fmaf(__ldg(p.pend_x + (size_t)pp * p.d + j), __ldg(p.cand_scale + j), __ldg(p.cand_shift + j));
    reinterpret_cast<float*>(pxt4)[xt_float_index(32, pp, j)] = -2.0f * b;
  }
  __syncthreads();
  if (tid < 32) {
    float s = 0.f;
    for (int j = 0; j < p.d_pad; ++j) {
      float b = -0.5f * reinterpret_cast<float*>(pxt4)[xt_float_index(32, tid, j)];
      s = fmaf(b, b, s);
    }
    psq[tid] = s;
    int t = 0;
    if (p.task_col >= 0 && tid < p.P)
      t = min(max(__float2int_rn(__ldg(p.pend_x + (size_t)tid * p.d + p.task_col)), 0), p.n_tasks - 1);
    ptask[tid] = t;
  }
  __syncthreads();
  const int mp = tid & 63, g = tid >> 6;  // g in 0..3: quarter of the training points
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int64_t row0 = (int64_t)tile * kTileM;
    {
      StageRegs regs;
      stage_prefetch(sc, sm.dq, row0, tid, regs);
      stage_commit(sc, sm.a_s, sm.cand_task, sm.T, sm.dq, row0, tid, regs);
    }
    for (int e = tid; e < kTileM * 32; e += 256) cross_s[e] = 0.f;
    __syncthreads();
    const float an0 = cand_sqnorm(sm, mp), an1 = cand_sqnorm(sm, mp + 64);
    float acc0[BB_MAX_PENDING + 1], acc1[BB_MAX_PENDING + 1];
#pragma unroll
    for (int pp = 0; pp <= BB_MAX_PENDING; ++pp) {
      acc0[pp] = 0.f;
      acc1[pp] = 0.f;
    }
    const int octets = p.n_pad >> 3;
    for (int o = g; o < octets; o += 4) {
      float k0[8], k1[8];
      assemble_2x8<FAMILY>(sm, mp, mp + 64, an0, an1, o * 8, k0, k1);
#pragma unroll
      for (int pp = 0; pp <= BB_MAX_PENDING; ++pp) {
        if (pp < p.P) {
          const float4* b4 = reinterpret_cast<const float4*>(p.pend_beta + (size_t)pp * p.n_pad + o * 8);
          const float4 ba = __ldg(b4), bb2 = __ldg(b4 + 1);
          acc0[pp] -= k0[0] * ba.x + k0[1] * ba.y + k0[2] * ba.z + k0[3] * ba.w + k0[4] * bb2.x +
                      k0[5] * bb2.y + k0[6] * bb2.z + k0[7] * bb2.w;
          acc1[pp] -= k1[0] * ba.x + k1[1] * ba.y + k1[2] * ba.z + k1[3] * ba.w + k1[4] * bb2.x +
                      k1[5] * bb2.y + k1[6] * bb2.z + k1[7] * bb2.w;
        }
      }
    }
    // prior term k(x*, p): group g handles pending octet g (P <= 32)
    {
      AsmSmem ps = sm;
      ps.xt4 = pxt4;
      ps.np = 32;
      ps.tsq = psq;
      ps.ttask = ptask;
      float k0[8], k1[8];
      assemble_2x8<FAMILY>(ps, mp, mp + 64, an0, an1, g * 8, k0, k1);
#pragma unroll
      for (int ii = 0; ii < 8; ++ii) {
        const int pp = g * 8 + ii;
#pragma unroll
        for (int q2 = 0; q2 <= BB_MAX_PENDING; ++q2)
          if (q2 == pp) {
            acc0[q2] += k0[ii];
            acc1[q2] += k1[ii];
          }
      }
    }
    // deterministic reduction over the four groups
    for (int gg = 0; gg < 4; ++gg) {
      if (g == gg) {
#pragma unroll
        for (int pp = 0; pp <= BB_MAX_PENDING; ++pp) {
          if (pp < p.P) {
            cross_s[mp * 32 + pp] += acc0[pp];
            cross_s[(mp + 64) * 32 + pp] += acc1[pp];
          }
        }
      }
      __syncthreads();
    }
    const float s2 = p.y_std * p.y_std;
    for (int e = tid; e < kTileM * p.P; e += 256) {
      int r = e / p.P, pp = e - r * p.P;
      int64_t row = row0 + r;
      if (row < p.N) p.cross[row * p.P + pp] = s2 * cross_s[r * 32 + pp];
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// test-only SIMT posterior: 32 candidates per CTA, direct-difference distances, fp32 FMA
// contraction with the dense fp32 copy of L^-1.
// ------------------------------------------------------------------------------------------
struct SimtSmem {
  float *ks, *xa, *red;
  int* ct;
};

static __host__ __device__ size_t carve_simt(uint8_t* base, const AuxParams& p, SimtSmem& s) {
  SmemCarver c{base};
  s.ks = c.take<float>((size_t)32 * (p.n_pad + 1) * 4);  // [32][n_pad+1]
  s.xa = c.take<float>((size_t)32 * p.d_pad * 4);        // [32][d_pad]
  s.ct = c.take<int>(32 * 4);                            // [32]
  s.red = c.take<float>(8 * 32 * 2 * 4);                 // [8][32][2]
  return c.bytes;
}

template <int FAMILY>
__global__ void __launch_bounds__(256, 1) k_simt(const AuxParams p) {
  extern __shared__ __align__(16) uint8_t smem_aux[];
  const int tid = threadIdx.x;
  SimtSmem s;
  carve_simt(smem_aux, p, s);
  float *ks = s.ks, *xa = s.xa, *red = s.red;
  int* ct = s.ct;
  const int64_t row0 = (int64_t)blockIdx.x * 32;
  for (int e = tid; e < 32 * p.d_pad; e += 256) {
    int r = e / p.d_pad, j = e - r * p.d_pad;
    int64_t row = row0 + r;
    const float xv = (j < p.d && row < p.N) ? load_x_any(p.x, p.layout, row, j, p.ldx) : 0.f;
    xa[e] = (j < p.d) ? fmaf(xv, __ldg(p.cand_scale + j), __ldg(p.cand_shift + j)) : 0.f;
    if (j == p.task_col) ct[r] = min(max(__float2int_rn(xv), 0), p.n_tasks - 1);
  }
  if (p.task_col < 0 && tid < 32) ct[tid] = 0;
  __syncthreads();
  for (int e = tid; e < 32 * p.n_pad; e += 256) {
    int r = e & 31, i = e >> 5;
    float t = 0.f;
    for (int j = 0; j < p.d_pad; ++j) {
      float diff = xa[r * p.d_pad + j] + 0.5f * __ldg(p.train_m2 + (size_t)i * p.d_pad + j);
      t = fmaf(diff, diff, t);
    }
    float k = (i < p.n) ? kernel_from_t<FAMILY>(t) : 0.f;
    if (p.scaled) k *= __ldg(p.task_covar + ct[r] * p.n_tasks + __ldg(p.train_task + i));
    ks[r * (p.n_pad + 1) + i] = k;
  }
  __syncthreads();
  const int r = tid & 31, jg = tid >> 5;
  float ss = 0.f, ms = 0.f;
  for (int j = jg; j < p.n; j += 8) {
    float v = 0.f;
    for (int i = 0; i <= j; ++i)
      v = fmaf(ks[r * (p.n_pad + 1) + i], __ldg(p.linv32 + (size_t)j * p.n_pad + i), v);
    ss = fmaf(v, v, ss);
    ms = fmaf(ks[r * (p.n_pad + 1) + j], __ldg(p.alpha + j), ms);
  }
  red[(jg * 32 + r) * 2] = ss;
  red[(jg * 32 + r) * 2 + 1] = ms;
  __syncthreads();
  if (tid < 32) {
    float s = 0.f, m = 0.f;
    for (int gg = 0; gg < 8; ++gg) {
      s += red[(gg * 32 + tid) * 2];
      m += red[(gg * 32 + tid) * 2 + 1];
    }
    int64_t row = row0 + tid;
    if (row < p.N) {
      float kss = p.scaled ? __ldg(p.task_covar + ct[tid] * p.n_tasks + ct[tid]) : 1.0f;
      float vt = fmaxf(kss - s, 1e-10f);
      p.mu[row] = fmaf(p.y_std, __ldg(p.mean_const + ct[tid]) + m, p.y_mean);
      p.var[row] = p.y_std * p.y_std * vt;
    }
  }
}

// Candidate checks (check_candidates) and the model fields of AuxParams.  These kernels read the four float layouts
// only: bit-packed rows are rejected as an invalid layout even for a wide-feature model.
static int fill_params(AuxParams& p, const bb_model* m, const void* d_x, int32_t layout, int64_t N,
                       int64_t ldx) {
  BB_CHECK_ARG(layout != BB_BITS_U8, "bit-packed candidates are not read by this entry point");
  const int rc = check_candidates(m, d_x, layout, N, ldx);
  if (rc != BB_OK) return rc;
  memset(&p, 0, sizeof(p));
  p.x = d_x;
  p.layout = layout;
  p.N = N;
  p.ldx = ldx;
  p.num_tiles = (int)((N + kTileM - 1) / kTileM);
  p.cand_scale = m->d_cand_scale;
  p.cand_shift = m->d_cand_shift;
  p.train_m2 = m->d_train_m2;
  p.train_sq = m->d_train_sq;
  p.task_covar = m->d_task_covar;
  p.train_task = m->d_train_task;
  p.n = m->n;
  p.n_pad = m->n_pad;
  p.d = m->d;
  p.d_pad = m->d_pad;
  p.n_chunks = m->n_chunks;
  p.task_col = m->task_col;
  p.n_tasks = m->n_tasks;
  p.scaled = model_scaled(m) ? 1 : 0;
  p.y_std = m->y_std;
  p.y_mean = m->y_mean;
  p.alpha = m->d_alpha;
  p.mean_const = m->d_mean_const;
  p.linv32 = m->d_linv32;
  return BB_OK;
}

int launch_cross(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx,
                 const float* d_pend_x, const float* d_pend_beta, int32_t P, float* d_cross,
                 cudaStream_t stream) {
  AuxParams p;
  int rc = fill_params(p, m, d_x, layout, N, ldx);
  if (rc != BB_OK) return rc;
  BB_CHECK_ARG(d_pend_x && d_pend_beta && d_cross, "pending buffers are null");
  BB_CHECK_ARG(P >= 1 && P <= BB_MAX_PENDING, "n_pending=%d outside [1,%d]", P, BB_MAX_PENDING);
  if (N == 0) return BB_OK;
  p.pend_x = d_pend_x;
  p.pend_beta = d_pend_beta;
  p.P = P;
  p.cross = d_cross;
  int sms, max_smem;
  rc = device_limits(&sms, &max_smem);
  if (rc != BB_OK) return rc;
  AuxSmem unused;
  const size_t smem = carve_cross(nullptr, p, unused);
  BB_CHECK_SUPPORTED(smem <= (size_t)max_smem, "shared-memory budget exceeded (%zu bytes)", smem);
  const int grid = p.num_tiles < sms ? p.num_tiles : sms;
  return dispatch_family<true>(m->family, [&](auto fam) {
    BB_SMEM_OPTIN_ONCE(k_cross<decltype(fam)::value>);
    k_cross<decltype(fam)::value><<<grid, 256, smem, stream>>>(p);
    BB_LAUNCH_CHECK();
    return BB_OK;
  });
}

}  // namespace bb

using namespace bb;

extern "C" int bb_kernel_matrix(const bb_model* m, const void* d_x, int32_t layout, int64_t N,
                                int64_t ldx, float* d_k, int64_t ldk, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const bool wide = m && m->abi_version == BB_ABI_VERSION && m->wide;  // K-chunked tensor-core path (wide.cu)
  AuxParams p;
  int rc = wide ? check_candidates(m, d_x, layout, N, ldx) : fill_params(p, m, d_x, layout, N, ldx);
  if (rc != BB_OK) return rc;
  BB_CHECK_ARG(d_k != nullptr || N == 0, "bb_kernel_matrix: output pointer is null");
  BB_CHECK_ARG(ldk >= m->n, "bb_kernel_matrix: ldk=%lld smaller than n=%d", (long long)ldk, m->n);
  if (N == 0) return BB_OK;
  if (wide) return launch_kmat_wide(m, d_x, layout, N, ldx, d_k, ldk, N, m->n, stream);
  {  // tensor-core distances + TMA tensor stores (fused.cu: k_kmat_tma) where the model and the output allow
    bool handled = false;
    rc = try_kmat_tma(m, d_x, layout, N, ldx, d_k, ldk, stream, &handled);
    if (rc != BB_OK || handled) return rc;
  }
  p.kout = d_k;
  p.ldk = ldk;
  int sms, max_smem;
  rc = device_limits(&sms, &max_smem);
  if (rc != BB_OK) return rc;
  AuxSmem unused;
  const size_t smem = carve_kmat(nullptr, p, unused);
  BB_CHECK_SUPPORTED(smem <= (size_t)max_smem, "shared-memory budget exceeded (%zu bytes)", smem);
  // several waves of small tiles balance better than one persistent CTA per SM for this
  // store-bound kernel: 2 CTAs per SM worth of grid, grid-stride over the tiles.
  const int grid = p.num_tiles < 2 * sms ? p.num_tiles : 2 * sms;
  return dispatch_family<true>(m->family, [&](auto fam) {
    BB_SMEM_OPTIN_ONCE(k_kmat<decltype(fam)::value>);
    k_kmat<decltype(fam)::value><<<grid, kAuxThreads, smem, stream>>>(p);
    BB_LAUNCH_CHECK();
    return BB_OK;
  });
}

extern "C" int bb_debug_posterior_simt(const bb_model* m, const void* d_x, int32_t layout,
                                       int64_t N, int64_t ldx, float* d_mu, float* d_var,
                                       void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  AuxParams p;
  int rc = fill_params(p, m, d_x, layout, N, ldx);
  if (rc != BB_OK) return rc;
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_mu && d_var, "bb_debug_posterior_simt: output pointers are null");
  p.mu = d_mu;
  p.var = d_var;
  SimtSmem unused;
  const size_t smem = carve_simt(nullptr, p, unused);
  const int grid = (int)((N + 31) / 32);
  return dispatch_family<true>(m->family, [&](auto fam) {
    BB_SMEM_OPTIN_ONCE(k_simt<decltype(fam)::value>);
    k_simt<decltype(fam)::value><<<grid, 256, smem, stream>>>(p);
    BB_LAUNCH_CHECK();
    return BB_OK;
  });
}
