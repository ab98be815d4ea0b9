// nipvgrad.cu -- value and gradient of qNIPV's integrated variance reduction at P points (bb_nipv_phi, bb_nipv_grad),
// for the continuous optimiser on continuous and hybrid spaces.
//
// Notation of nipv.cu, standardised units.  X: the training rows (Cholesky factor L), C: the conditioning set
// (pending points and the earlier points of a greedy batch, observed with noise), L_C L_C^T = K_D(C,C) + diag s_n^2(C):
//   phi(a)  = [ L^-1 k(X,a) ; L_C^-1 k_D(C,a) ]         r = n + |C| entries,  k_D(C,a) = k(C,a) - beta_C^T k(X,a)
//   e_m(x)  = k(m,x) - phi(m) . phi(x),   s(x) = k(x,x) - |phi(x)|^2 + s_n^2,   IVR(x) = sum_m e_m^2 / s
// With a_m = 2 e_m / s,  g = sum_m a_m phi(m),  h = sum_m a_m d k(m,x)/dx  and J_x = d phi(x) / dx:
//   grad IVR = h - J_x^T ( g - (2 IVR / s) phi(x) )
// J_x^T w is one reverse pass: u = L_C^-T w_C; training row i gets (L^-T w_X)_i - (beta_C^T u)_i, C row c gets u_c,
// and the result is sum_row coeff_row * dk(row, x)/dx.  k(x,x) and s_n^2 do not depend on x (single-task models).
//
// Four kernels, all fp32 on the CUDA cores:
//   k_nipv_image     (bb_nipv_phi) phi of 64 integration points per CTA, k_nipv_phi's arithmetic (nipv.cu) without the
//                    fp16 split or the power-of-two scale, written dimension-major [r][M] and followed by the scaled
//                    coordinates [d][M]: consecutive threads read consecutive m in the pair pass.  Built once per
//                    greedy step.
//   k_nipv_grad_x    one warp per point: k(X,x), phi(x) (the grad_common.cuh row passes) and s.
//   k_nipv_grad_m    kNgCtas CTAs, each over a contiguous range of 64-point chunks of the image; per 16-point tile, the
//                    chunk's phi and coordinates are staged in shared memory with coalesced loads, pass 1 forms e_{m,p}
//                    (dot over r, direct d-deep distance, kernel and slope), pass 2 accumulates g, h and sum e^2 with
//                    one thread per entry.  Per-CTA partials go to the workspace.
//   k_nipv_grad_fin  one CTA per point: the partials summed in CTA order, then the reverse pass.
// No float atomics and fixed reduction orders: repeated calls are bit-identical.
#include <math.h>

#include "fused_common.cuh"
#include "grad_common.cuh"

namespace bb {

constexpr int kNgMaxTrain = 256;
constexpr int kNgThreads = 256;
constexpr int kNgChunk = 64;       // integration points per staged chunk
constexpr int kNgLd = kNgChunk + 1;  // shared-memory row stride of a chunk: conflict-free column walks
constexpr int kNgTile = 16;        // points per pass over the image
constexpr int kNgCtas = 264;       // CTAs of the pair pass (2 x 132 SMs); fixed, so the partition never depends on the device
constexpr int kNgXThreads = 128;   // k_nipv_grad_x: four points per block

// ---- bb_nipv_phi ------------------------------------------------------------------------------------------------
struct NipvImageParams {
  const float* xm;  // [M][d] raw rows
  int64_t M;
  const float *cand_scale, *cand_shift, *train_m2, *linv32;
  int n, n_pad, d, d_pad, C;
  float sf2, inv_y_std;
  const float* cross;   // [M][C] original units
  const float* linv_c;  // [C][C] original units
  float* img;           // [(n + C + d)][M]
};

template <int FAMILY>
__global__ void __launch_bounds__(kNgThreads) k_nipv_image(const NipvImageParams p) {
  extern __shared__ __align__(16) float smem_img[];
  float* xa = smem_img;              // [64][d_pad]
  float* ks = xa + 64 * p.d_pad;     // [64][n_pad + 1]
  const int tid = threadIdx.x;
  const int64_t row0 = (int64_t)blockIdx.x * 64;
  const int r_all = p.n + p.C;
  for (int e = tid; e < 64 * p.d_pad; e += kNgThreads) {
    const int j = e >> 6, r = e & 63;
    const int64_t row = row0 + r;
    const float xv = (j < p.d && row < p.M) ? __ldg(p.xm + row * p.d + j) : 0.f;
    const float a = (j < p.d) ? fmaf(xv, __ldg(p.cand_scale + j), __ldg(p.cand_shift + j)) : 0.f;
    xa[r * p.d_pad + j] = a;
    if (j < p.d && row < p.M) p.img[(int64_t)(r_all + j) * p.M + row] = a;
  }
  __syncthreads();
  for (int e = tid; e < 64 * p.n_pad; e += kNgThreads) {
    const int r = e & 63, i = e >> 6;
    float t = 0.f;
    for (int j = 0; j < p.d_pad; ++j) {
      const float diff = xa[r * p.d_pad + j] + 0.5f * __ldg(p.train_m2 + (size_t)i * p.d_pad + j);
      t = fmaf(diff, diff, t);
    }
    ks[r * (p.n_pad + 1) + i] = (i < p.n) ? kernel_from_t<FAMILY>(t) * p.sf2 : 0.f;
  }
  __syncthreads();
  const int r = tid & 63;
  const int64_t row = row0 + r;
  const bool valid = row < p.M;
  for (int j = tid >> 6; j < p.n; j += kNgThreads / 64) {
    float v = 0.f;
    for (int i = 0; i <= j; ++i) v = fmaf(ks[r * (p.n_pad + 1) + i], __ldg(p.linv32 + (size_t)j * p.n_pad + i), v);
    if (valid) p.img[(int64_t)j * p.M + row] = v;
  }
  if (tid < 64 && valid) {
    for (int j = 0; j < p.C; ++j) {
      float v = 0.f;
      for (int i = 0; i <= j; ++i) v = fmaf(__ldg(p.linv_c + j * p.C + i), __ldg(p.cross + row * p.C + i), v);
      p.img[(int64_t)(p.n + j) * p.M + row] = v * p.inv_y_std;
    }
  }
}

// ---- bb_nipv_grad -----------------------------------------------------------------------------------------------
// Per point, R = r + d + 1 floats: phi(x) [r] | scaled coordinates [d] | s (the x pass), and the same layout for the
// partial sums of the pair pass: g [r] | h [d] | sum e^2.
struct NipvGradParams {
  const float* x;    // [P][d] raw rows
  int64_t P, M;
  const float* img;  // [(r + d)][M]
  const float *cand_scale, *cand_shift, *train_m2, *alpha, *linv32;
  int n, n_pad, d, d_pad, C, R, n_ctas;
  float sf2, y_std, y_var, prior_var, noise;
  const float *cond_x, *cond_beta, *linv_c;  // [C][d], [C][n_pad], [C][C] (L_C^-1, original units)
  float* xinfo;  // [P][R]
  float* part;   // [n_ctas][P][R]
  float* value;  // [P]
  float* grad;   // [P][d]
};

__host__ __device__ inline int nipv_grad_x_warp_floats(int n_pad, int d_pad) {
  return (d_pad + 3 * n_pad + 32 + 3) & ~3;
}

template <int FAMILY>
__global__ void __launch_bounds__(kNgXThreads) k_nipv_grad_x(const NipvGradParams p) {
  extern __shared__ __align__(16) float smem_gx[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t pt = (int64_t)blockIdx.x * (kNgXThreads / 32) + warp;
  if (pt >= p.P) return;
  float* a_w = smem_gx + warp * nipv_grad_x_warp_floats(p.n_pad, p.d_pad);
  float* k_w = a_w + p.d_pad;
  float* gk_w = k_w + p.n_pad;
  float* v_w = gk_w + p.n_pad;
  float* kd_w = v_w + p.n_pad;  // [32] k_D(C, x)
  for (int j = lane; j < p.d_pad; j += 32)
    a_w[j] = j < p.d ? fmaf(__ldg(p.x + pt * p.d + j), __ldg(p.cand_scale + j), __ldg(p.cand_shift + j)) : 0.f;
  __syncwarp();
  kernel_row_warp<FAMILY>(a_w, p.train_m2, p.alpha, p.n, p.n_pad, p.d, p.d_pad, p.sf2, k_w, gk_w, lane);
  __syncwarp();
  const float vv = warp_sum(linv_apply_warp(p.linv32, p.n_pad, k_w, v_w, lane));
  float kb_mine = 0.f;
  for (int c = 0; c < p.C; ++c) {
    float kb = 0.f;
    for (int i = lane; i < p.n_pad; i += 32) kb = fmaf(k_w[i], __ldg(p.cond_beta + (size_t)c * p.n_pad + i), kb);
    kb = warp_sum(kb);
    if (lane == c) kb_mine = kb;
  }
  if (lane < p.C) {
    float t = 0.f;
    for (int j = 0; j < p.d; ++j) {
      const float b = fmaf(__ldg(p.cond_x + (size_t)lane * p.d + j), __ldg(p.cand_scale + j), __ldg(p.cand_shift + j));
      const float df = a_w[j] - b;
      t = fmaf(df, df, t);
    }
    float k, dk;
    kernel_and_slope<FAMILY>(t, k, dk);
    kd_w[lane] = p.sf2 * k - kb_mine;
  }
  __syncwarp();
  float pc = 0.f;
  if (lane < p.C) {
    for (int i = 0; i <= lane; ++i) pc = fmaf(__ldg(p.linv_c + lane * p.C + i), kd_w[i], pc);
    pc *= p.y_std;  // L_C^-1 in standardised units
  }
  const float qq = warp_sum(pc * pc);
  float* out = p.xinfo + pt * p.R;
  for (int j = lane; j < p.n; j += 32) out[j] = v_w[j];
  if (lane < p.C) out[p.n + lane] = pc;
  const int r = p.n + p.C;
  for (int j = lane; j < p.d; j += 32) out[r + j] = a_w[j];
  if (lane == 0) out[r + p.d] = fmaxf(p.prior_var - vv - qq, 0.f) + p.noise;
}

__host__ __device__ inline size_t nipv_grad_m_smem(int r, int d, int R) {
  return sizeof(float) * ((size_t)(r + d) * kNgLd + (size_t)kNgTile * R + (size_t)3 * kNgTile * kNgLd);
}

template <int FAMILY>
__global__ void __launch_bounds__(kNgThreads, 1) k_nipv_grad_m(const NipvGradParams p) {
  extern __shared__ __align__(16) float smem_gm[];
  const int r = p.n + p.C, rd = r + p.d, R = p.R;
  float* ph = smem_gm;                    // [r + d][kNgLd] the chunk: phi rows, then coordinate rows
  float* xs = ph + (size_t)rd * kNgLd;    // [kNgTile][R] the tile's x-pass rows
  float* A = xs + kNgTile * R;            // [kNgTile][kNgLd] a_{m,p} = 2 e / s
  float* Cc = A + kNgTile * kNgLd;        // [kNgTile][kNgLd] a_{m,p} * dk/dt-slope
  float* E2 = Cc + kNgTile * kNgLd;       // [kNgTile][kNgLd] e^2
  const int tid = threadIdx.x;
  const int64_t n_chunks = (p.M + kNgChunk - 1) / kNgChunk;
  const int64_t c_begin = n_chunks * blockIdx.x / p.n_ctas, c_end = n_chunks * (blockIdx.x + 1) / p.n_ctas;
  const int ml = tid & 63, pg = tid >> 6;
  for (int64_t t0 = 0; t0 < p.P; t0 += kNgTile) {
    const int np = (int)min((int64_t)kNgTile, p.P - t0);
    __syncthreads();
    for (int e = tid; e < kNgTile * R; e += kNgThreads) {
      const int q = e / R;
      xs[e] = q < np ? p.xinfo[(t0 + q) * R + (e - q * R)] : 0.f;
    }
    float acc0[kNgTile], acc1[kNgTile];
#pragma unroll
    for (int q = 0; q < kNgTile; ++q) acc0[q] = acc1[q] = 0.f;
    for (int64_t ch = c_begin; ch < c_end; ++ch) {
      const int64_t m0 = ch * kNgChunk;
      __syncthreads();  // the previous chunk's pass 2 is done with ph, A, Cc, E2
      for (int e = tid; e < rd * kNgChunk; e += kNgThreads) {
        const int row = e >> 6, col = e & 63;
        const int64_t m = m0 + col;
        ph[row * kNgLd + col] = m < p.M ? __ldg(p.img + (int64_t)row * p.M + m) : 0.f;
      }
      __syncthreads();
      // pass 1: e_{m,p} for m = ml and p = pg + 4 q
      {
        const bool mvalid = m0 + ml < p.M;
        float dot[4] = {0.f, 0.f, 0.f, 0.f};
        for (int j = 0; j < r; ++j) {
          const float f = ph[j * kNgLd + ml];
#pragma unroll
          for (int q = 0; q < 4; ++q) dot[q] = fmaf(f, xs[(pg + 4 * q) * R + j], dot[q]);
        }
        float t[4] = {0.f, 0.f, 0.f, 0.f};
        for (int k = 0; k < p.d; ++k) {
          const float c = ph[(r + k) * kNgLd + ml];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float df = xs[(pg + 4 * q) * R + r + k] - c;
            t[q] = fmaf(df, df, t[q]);
          }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int pp = pg + 4 * q;
          float kv, dk;
          kernel_and_slope<FAMILY>(t[q], kv, dk);
          const float e = p.sf2 * kv - dot[q];
          const bool on = mvalid && pp < np;
          const float am = on ? 2.f * e / xs[pp * R + rd] : 0.f;
          A[pp * kNgLd + ml] = am;
          Cc[pp * kNgLd + ml] = am * 2.f * p.sf2 * dk;
          E2[pp * kNgLd + ml] = on ? e * e : 0.f;
        }
      }
      __syncthreads();
      // pass 2: entry e of every point of the tile, summed over the chunk's 64 points in order
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int e = tid + h * kNgThreads;
        if (e > rd) continue;
        float* acc = h ? acc1 : acc0;
        if (e < r) {
          const float* row = ph + e * kNgLd;
          for (int m = 0; m < kNgChunk; ++m) {
            const float f = row[m];
#pragma unroll
            for (int q = 0; q < kNgTile; ++q) acc[q] = fmaf(A[q * kNgLd + m], f, acc[q]);
          }
        } else if (e < rd) {
          const float* row = ph + e * kNgLd;
          for (int m = 0; m < kNgChunk; ++m) {
            const float f = row[m];
#pragma unroll
            for (int q = 0; q < kNgTile; ++q) acc[q] = fmaf(Cc[q * kNgLd + m], xs[q * R + e] - f, acc[q]);
          }
        } else {
          for (int m = 0; m < kNgChunk; ++m) {
#pragma unroll
            for (int q = 0; q < kNgTile; ++q) acc[q] += E2[q * kNgLd + m];
          }
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int e = tid + h * kNgThreads;
      if (e >= R) continue;
      const float* acc = h ? acc1 : acc0;
#pragma unroll
      for (int q = 0; q < kNgTile; ++q)
        if (q < np) p.part[((int64_t)blockIdx.x * p.P + t0 + q) * R + e] = acc[q];
    }
  }
}

template <int FAMILY>
__global__ void __launch_bounds__(kNgThreads) k_nipv_grad_fin(const NipvGradParams p) {
  extern __shared__ __align__(16) float smem_gf[];
  const int r = p.n + p.C, rd = r + p.d, R = p.R;
  float* tot = smem_gf;             // [R]: g then w = g - (2 IVR / s) phi(x) | h | sum e^2
  float* coef = tot + R;            // [n_pad] coefficients of the training rows
  float* uc = coef + p.n_pad;       // [32] u = L_C^-T w_C (standardised), then its coefficients
  float* cb = uc + 32;              // [C][d] scaled conditioning rows
  const int tid = threadIdx.x;
  const int64_t pt = blockIdx.x;
  const float* xi = p.xinfo + pt * R;
  for (int e = tid; e < R; e += kNgThreads) {
    float s = 0.f;
    for (int c = 0; c < p.n_ctas; ++c) s += p.part[((int64_t)c * p.P + pt) * R + e];
    tot[e] = s;
  }
  for (int e = tid; e < p.C * p.d; e += kNgThreads) {
    const int j = e % p.d;
    cb[e] = fmaf(__ldg(p.cond_x + e), __ldg(p.cand_scale + j), __ldg(p.cand_shift + j));
  }
  __syncthreads();
  const float s = xi[rd];
  const float ivr = tot[rd] / s;
  const float fac = 2.f * ivr / s;
  for (int j = tid; j < r; j += kNgThreads) tot[j] = fmaf(-fac, xi[j], tot[j]);
  __syncthreads();
  if (tid < p.C) {
    float u = 0.f;
    for (int k = tid; k < p.C; ++k) u = fmaf(__ldg(p.linv_c + k * p.C + tid), tot[p.n + k], u);
    uc[tid] = u * p.y_std;
  }
  __syncthreads();
  const float* a = xi + r;
  for (int i = tid; i < p.n; i += kNgThreads) {
    float c = 0.f;
    for (int j = i; j < p.n; ++j) c = fmaf(__ldg(p.linv32 + (size_t)j * p.n_pad + i), tot[j], c);
    for (int q = 0; q < p.C; ++q) c = fmaf(-__ldg(p.cond_beta + (size_t)q * p.n_pad + i), uc[q], c);
    float t = 0.f;
    for (int j = 0; j < p.d; ++j) {
      const float df = a[j] + 0.5f * __ldg(p.train_m2 + (size_t)i * p.d_pad + j);
      t = fmaf(df, df, t);
    }
    float k, dk;
    kernel_and_slope<FAMILY>(t, k, dk);
    coef[i] = c * 2.f * p.sf2 * dk;
  }
  __syncthreads();
  if (tid < p.C) {
    float t = 0.f;
    for (int j = 0; j < p.d; ++j) {
      const float df = a[j] - cb[tid * p.d + j];
      t = fmaf(df, df, t);
    }
    float k, dk;
    kernel_and_slope<FAMILY>(t, k, dk);
    uc[tid] *= 2.f * p.sf2 * dk;
  }
  __syncthreads();
  for (int j = tid; j < p.d; j += kNgThreads) {
    const float aj = a[j];
    float g = tot[r + j];
    for (int i = 0; i < p.n; ++i) g = fmaf(-coef[i], aj + 0.5f * __ldg(p.train_m2 + (size_t)i * p.d_pad + j), g);
    for (int c = 0; c < p.C; ++c) g = fmaf(-uc[c], aj - cb[c * p.d + j], g);
    p.grad[pt * p.d + j] = g * __ldg(p.cand_scale + j) * p.y_var;
  }
  if (tid == 0) p.value[pt] = ivr * p.y_var;
}

static int nipv_grad_model_checks(const char* fn, const bb_model* m) {
  BB_CHECK_ARG(m && m->abi_version == BB_ABI_VERSION, "%s: model struct missing or ABI mismatch", fn);
  BB_CHECK_SUPPORTED(!m->wide, "%s: wide-feature models are not supported", fn);
  BB_CHECK_SUPPORTED(m->task_col < 0, "%s: models with a task parameter are not supported", fn);
  BB_CHECK_SUPPORTED(m->n <= kNgMaxTrain && m->n_pad <= kGradMaxNPad, "%s: n=%d training points, at most %d supported",
                     fn, m->n, kNgMaxTrain);
  return BB_OK;
}

}  // namespace bb

using namespace bb;

extern "C" int bb_nipv_phi(const bb_model* m, const float* d_xm, int64_t M, int32_t n_cond, const float* d_cross_m,
                           const float* d_linv, float* d_img, void* stream) {
  int rc = nipv_grad_model_checks("bb_nipv_phi", m);
  if (rc != BB_OK) return rc;
  BB_CHECK_ARG(M >= 1 && M < 0x7fffffffLL, "bb_nipv_phi: M=%lld integration points outside [1,2^31)", (long long)M);
  BB_CHECK_ARG(n_cond >= 0 && n_cond <= BB_MAX_PENDING, "bb_nipv_phi: n_cond=%d outside [0,%d]", n_cond,
               BB_MAX_PENDING);
  BB_CHECK_ARG(d_xm && d_img, "bb_nipv_phi: null buffer");
  BB_CHECK_ARG(n_cond == 0 || (d_cross_m && d_linv), "bb_nipv_phi: conditioning points need cross_m and linv");
  int sms, max_smem;
  rc = device_limits(&sms, &max_smem);
  if (rc != BB_OK) return rc;
  const size_t smem = sizeof(float) * ((size_t)64 * m->d_pad + (size_t)64 * (m->n_pad + 1));
  BB_CHECK_SUPPORTED(smem <= (size_t)max_smem, "bb_nipv_phi: %zu bytes of shared memory above the %d available", smem,
                     max_smem);
  NipvImageParams p{};
  p.xm = d_xm;
  p.M = M;
  p.cand_scale = m->d_cand_scale;
  p.cand_shift = m->d_cand_shift;
  p.train_m2 = m->d_train_m2;
  p.linv32 = m->d_linv32;
  p.n = m->n;
  p.n_pad = m->n_pad;
  p.d = m->d;
  p.d_pad = m->d_pad;
  p.C = n_cond;
  p.sf2 = m->prior_scale;
  p.inv_y_std = 1.0f / m->y_std;
  p.cross = d_cross_m;
  p.linv_c = d_linv;
  p.img = d_img;
  return dispatch_family<true>(m->family, [&](auto fam) {
    BB_SMEM_OPTIN_ONCE(k_nipv_image<decltype(fam)::value>);
    k_nipv_image<decltype(fam)::value><<<(unsigned)((M + 63) / 64), kNgThreads, smem, (cudaStream_t)stream>>>(p);
    BB_LAUNCH_CHECK();
    return BB_OK;
  });
}

extern "C" int bb_nipv_grad(const bb_model* m, const float* noise, float prior_var, const float* d_x, int64_t P,
                            const float* d_img, int64_t M, int32_t n_cond, const float* d_cond_x,
                            const float* d_cond_beta, const float* d_linv, float* d_value, float* d_grad, void* d_ws,
                            size_t ws_bytes, void* stream) {
  int rc = nipv_grad_model_checks("bb_nipv_grad", m);
  if (rc != BB_OK) return rc;
  BB_CHECK_ARG(P >= 1 && P < 0x7fffffffLL, "bb_nipv_grad: P=%lld points outside [1,2^31)", (long long)P);
  BB_CHECK_ARG(M >= 1 && M < 0x7fffffffLL, "bb_nipv_grad: M=%lld integration points outside [1,2^31)", (long long)M);
  BB_CHECK_ARG(n_cond >= 0 && n_cond <= BB_MAX_PENDING, "bb_nipv_grad: n_cond=%d outside [0,%d]", n_cond,
               BB_MAX_PENDING);
  BB_CHECK_ARG(noise != nullptr, "bb_nipv_grad: null noise");
  BB_CHECK_ARG(isfinite(noise[0]) && noise[0] >= 0.f, "bb_nipv_grad: noise not finite and >= 0");
  BB_CHECK_ARG(isfinite(prior_var) && prior_var > 0.f, "bb_nipv_grad: prior_var must be finite and > 0");
  BB_CHECK_ARG(d_x && d_img && d_value && d_grad && d_ws, "bb_nipv_grad: null buffer");
  BB_CHECK_ARG(n_cond == 0 || (d_cond_x && d_cond_beta && d_linv),
               "bb_nipv_grad: conditioning points need cond_x, cond_beta and linv");
  const int r = m->n + n_cond, R = r + m->d + 1;
  const int64_t n_chunks = (M + kNgChunk - 1) / kNgChunk;
  const int n_ctas = (int)(n_chunks < kNgCtas ? n_chunks : kNgCtas);
  const size_t need = sizeof(float) * (size_t)P * R * (size_t)(1 + n_ctas);
  BB_CHECK_ARG(ws_bytes >= need, "bb_nipv_grad: workspace of %zu bytes, need at least %zu", ws_bytes, need);
  int sms, max_smem;
  rc = device_limits(&sms, &max_smem);
  if (rc != BB_OK) return rc;
  const size_t smem_x = sizeof(float) * (kNgXThreads / 32) * nipv_grad_x_warp_floats(m->n_pad, m->d_pad);
  const size_t smem_m = nipv_grad_m_smem(r, m->d, R);
  const size_t smem_f = sizeof(float) * ((size_t)R + m->n_pad + 32 + (size_t)n_cond * m->d);
  BB_CHECK_SUPPORTED(smem_m <= (size_t)max_smem && smem_x <= (size_t)max_smem,
                     "bb_nipv_grad: %zu bytes of shared memory above the %d available", smem_m, max_smem);
  NipvGradParams p{};
  p.x = d_x;
  p.P = P;
  p.M = M;
  p.img = d_img;
  p.cand_scale = m->d_cand_scale;
  p.cand_shift = m->d_cand_shift;
  p.train_m2 = m->d_train_m2;
  p.alpha = m->d_alpha;
  p.linv32 = m->d_linv32;
  p.n = m->n;
  p.n_pad = m->n_pad;
  p.d = m->d;
  p.d_pad = m->d_pad;
  p.C = n_cond;
  p.R = R;
  p.n_ctas = n_ctas;
  p.sf2 = m->prior_scale;
  p.y_std = m->y_std;
  p.y_var = m->y_std * m->y_std;
  p.prior_var = prior_var;
  p.noise = noise[0] < 1e-4f ? 1e-4f : noise[0];  // MIN_INFERRED_NOISE_LEVEL, as bb_nipv_score
  p.cond_x = d_cond_x;
  p.cond_beta = d_cond_beta;
  p.linv_c = d_linv;
  p.xinfo = static_cast<float*>(d_ws);
  p.part = p.xinfo + (size_t)P * R;
  p.value = d_value;
  p.grad = d_grad;
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_family<true>(m->family, [&](auto fam) {
    constexpr int F = decltype(fam)::value;
    BB_SMEM_OPTIN_ONCE(k_nipv_grad_x<F>);
    BB_SMEM_OPTIN_ONCE(k_nipv_grad_m<F>);
    k_nipv_grad_x<F><<<(unsigned)((P + 3) / 4), kNgXThreads, smem_x, st>>>(p);
    BB_LAUNCH_CHECK();
    k_nipv_grad_m<F><<<(unsigned)n_ctas, kNgThreads, smem_m, st>>>(p);
    BB_LAUNCH_CHECK();
    k_nipv_grad_fin<F><<<(unsigned)P, kNgThreads, smem_f, st>>>(p);
    BB_LAUNCH_CHECK();
    return BB_OK;
  });
}
