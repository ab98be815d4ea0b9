// model.cu -- training-side caches (SURVEY.md K8): K(X,X)+noise, Cholesky, L^-1, alpha, and the
// tensor-core image of L^-1.  Everything here runs once per fitted model, in float64, on the GPU.
//
// Replaces what gpytorch's DefaultPredictionStrategy computes lazily on the first posterior
// call of botorch.models.SingleTaskGP (reference entry: GaussianProcessSurrogate._posterior,
// /root/reference/baybe/surrogates/gaussian_process/core.py:268-269; model built at :331-339).
#include <math.h>
#include <stdarg.h>
#include <string.h>

#include <vector>

#include <stdlib.h>

#include "common.cuh"

namespace bb {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

// ------------------------------------------------------------------------------------------
// blob layout
// ------------------------------------------------------------------------------------------
struct BlobLayout {
  size_t cand_scale, cand_shift, train_m2, train_sq, alpha, train_task, task_covar, mean_const,
      rimg, linv, alpha64, xn64, linv32, kmat, resid, noise_row, tcov64, cnorm, pend_norm, pend_w64, flags,
      wimg, wimg_bits, wnorm_bits, wsrc, wide_ws, pend_img, pend_norm2, pend_task, kpend_ws, mc_table, timg_b, total;
  int ts;  // K extent (32 or 64) of the augmented training image of the tensor-core distances, 0: none
  int n_pad, d_pad, n_chunks, n_tiles;
  int wide, d_wide;
  int64_t wide_ws_rows;
};

// The CUDA-core assembly keeps the scaled training rows in shared memory (n_pad*d_pad*4 <= 56 KB);
// anything larger takes the K-chunked tensor-core path of wide.cu.
constexpr size_t kResidentTrainBytes = 56 * 1024;
// K* workspace of the wide path: whole waves of 128-row work items over the 132 SMs of an H100, as many as keep the
// block within 40 MB of the 50 MB L2 (at least one wave: from n_pad = 640 on, one wave alone is larger than that)
constexpr int64_t kWideWave = 132 * 128;
constexpr size_t kWideWsBytes = (size_t)40 << 20;
static int64_t wide_ws_rows(int n_pad) {
  const int64_t waves = (int64_t)(kWideWsBytes / ((size_t)n_pad * 4)) / kWideWave;
  return (waves < 1 ? 1 : waves) * kWideWave;
}

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static BlobLayout make_layout(int n, int d, int T) {
  BlobLayout L;
  L.n_pad = round_up(n, kChunk);
  L.d_pad = round_up(d, 4);
  L.n_chunks = L.n_pad / kChunk;
  L.n_tiles = L.n_chunks * (L.n_chunks + 1) / 2;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 1024);
    return o;
  };
  L.cand_scale = take(sizeof(float) * L.d_pad);
  L.cand_shift = take(sizeof(float) * L.d_pad);
  L.train_m2 = take(sizeof(float) * (size_t)L.n_pad * L.d_pad);
  L.train_sq = take(sizeof(float) * L.n_pad);
  L.alpha = take(sizeof(float) * L.n_pad);
  L.train_task = take(sizeof(int32_t) * L.n_pad);
  L.task_covar = take(sizeof(float) * T * T);
  L.mean_const = take(sizeof(float) * T);
  L.rimg = take((size_t)L.n_tiles * 16384);
  L.linv = take(sizeof(double) * (size_t)n * n);
  L.alpha64 = take(sizeof(double) * n);
  L.xn64 = take(sizeof(double) * (size_t)n * d);
  L.linv32 = take(sizeof(float) * (size_t)L.n_pad * L.n_pad);
  L.kmat = take(sizeof(double) * (size_t)n * n);
  L.resid = take(sizeof(double) * n * 2);
  L.noise_row = take(sizeof(double) * n);
  L.tcov64 = take(sizeof(double) * (T * T + d));
  L.cnorm = take(sizeof(float) * 2 * d);
  L.pend_norm = take(sizeof(double) * BB_MAX_PENDING * d);
  L.pend_w64 = take(sizeof(double) * BB_MAX_PENDING * n);
  L.flags = take(64);
  L.wide = ((size_t)L.n_pad * L.d_pad * 4 > kResidentTrainBytes || L.n_pad > 512) ? 1 : 0;
  L.d_wide = round_up(d, 32);
  L.wimg = L.wimg_bits = L.wnorm_bits = L.wsrc = L.wide_ws = 0;
  L.pend_img = L.pend_norm2 = L.pend_task = L.kpend_ws = L.mc_table = 0;
  L.wide_ws_rows = 0;
  if (L.wide) {
    const size_t img = (size_t)L.n_pad * L.d_wide * 2 * 3;
    L.wimg = take(img);
    L.wimg_bits = take(img);
    L.wnorm_bits = take(sizeof(float) * L.n_pad);
    L.wsrc = take(sizeof(float) * (size_t)L.n_pad * L.d_wide);
    L.wide_ws_rows = wide_ws_rows(L.n_pad);
    L.wide_ws = take(sizeof(float) * (size_t)L.wide_ws_rows * L.n_pad);
    L.pend_img = take((size_t)64 * L.d_wide * 2 * 3);
    L.pend_norm2 = take(sizeof(float) * 64);
    L.pend_task = take(sizeof(int32_t) * 64);
    L.kpend_ws = take(sizeof(float) * (size_t)L.wide_ws_rows * 64);
    L.mc_table = take(sizeof(float) * 1024);
  }
  // k_fused with tensor-core distances: augmented training-row image
  // (n_pad <= 256; K = 32 for d <= 30, K = 64 for d <= 62: the last two K columns carry |a|^2 + |b|^2)
  L.ts = L.n_pad > 256 ? 0 : d <= 30 ? 32 : d <= 62 ? 64 : 0;
  L.timg_b = 0;
  if (L.ts) {
    L.timg_b = take((size_t)3 * L.n_pad * L.ts * 2);
    if (!L.wide) L.mc_table = take(sizeof(float) * 1024);  // per-call qLogEI table (k_mc_table_grid)
  }
  L.total = off;
  return L;
}

// ------------------------------------------------------------------------------------------
// float64 kernel function on the normalised inputs (direct differences: exact in float64)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ double kernel_f64(int family, double r2) {
  if (family == BB_KERNEL_RBF) return exp(-0.5 * r2);
  double r = sqrt(fmax(r2, 1e-30));
  if (family == BB_KERNEL_MATERN12) return exp(-r);
  if (family == BB_KERNEL_MATERN32) {
    double s = 1.7320508075688772 * r;
    return (1.0 + s) * exp(-s);
  }
  double s = 2.23606797749979 * r;
  return (1.0 + s + (5.0 / 3.0) * r2) * exp(-s);
}

// d_aux: [T*T] task covariance (prior scale folded in; 1x1 = prior scale without tasks),
// followed by [d] inverse lengthscales (0 for inactive columns / the task column).
__device__ __forceinline__ double k_pair_f64(const double* __restrict__ xa,
                                             const double* __restrict__ xb, int d,
                                             const double* __restrict__ inv_ls, int family) {
  double r2 = 0.0;
  for (int j = 0; j < d; ++j) {
    double u = (xa[j] - xb[j]) * inv_ls[j];
    r2 += u * u;
  }
  return kernel_f64(family, r2);
}

__global__ void k_train_gram(const double* __restrict__ xn, const int32_t* __restrict__ task,
                             const double* __restrict__ aux, const double* __restrict__ noise_row,
                             int n, int d, int T, int family, double jitter,
                             double* __restrict__ K) {
  const double* tcov = aux;
  const double* inv_ls = aux + T * T;
  int i = blockIdx.y * blockDim.y + threadIdx.y;
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || j >= n) return;
  double k;
  if (i == j) {
    k = 1.0;  // x1 is x2: gpytorch sets the self-distance diagonal to exactly 0
  } else {
    k = k_pair_f64(xn + (size_t)i * d, xn + (size_t)j * d, d, inv_ls, family);
  }
  k *= tcov[task[i] * T + task[j]];
  if (i == j) k += noise_row[i] + jitter;
  K[(size_t)i * n + j] = k;
}

// ---- blocked float64 Cholesky / triangular inverse (32 x 32 blocks, many CTAs) -------------------
// n <= 512 makes these launch-latency sized problems: a single-CTA unblocked factorisation took 12 ms at
// n = 512 (and the thread-per-column inverse 14 ms), which dominated every bb_model_build and every
// objective evaluation of the hyper-parameter fit; the blocked forms take a few hundred microseconds.
constexpr int kNB = 32;

// Panel step at column j0, part 1: factor the (already updated) 32 x 32 diagonal block in place (one CTA).
__global__ void __launch_bounds__(1024) k_chol_diag(double* __restrict__ A, int n, int j0, int* __restrict__ fail) {
  __shared__ double D[kNB][kNB + 1];
  __shared__ int bad;
  const int tx = threadIdx.x, ty = threadIdx.y;  // (column, row) inside the block
  const int gi = j0 + ty, gj = j0 + tx;
  D[ty][tx] = (gi < n && gj < n && tx <= ty) ? A[(size_t)gi * n + gj] : (tx == ty ? 1.0 : 0.0);
  if (tx == 0 && ty == 0) bad = 0;
  __syncthreads();
  for (int j = 0; j < kNB; ++j) {
    if (tx == j && ty == j) {
      double dj = D[j][j];
      if (!(dj > 0.0)) {
        bad = 1;
        dj = 1.0;
      }
      D[j][j] = sqrt(dj);
    }
    __syncthreads();
    if (tx == j && ty > j) D[ty][j] /= D[j][j];
    __syncthreads();
    if (tx > j && tx <= ty) D[ty][tx] -= D[ty][j] * D[tx][j];
    __syncthreads();
  }
  if (gi < n && gj < n) A[(size_t)gi * n + gj] = (tx <= ty) ? D[ty][tx] : 0.0;
  if (tx == 0 && ty == 0 && bad) fail[0] = 1;
}

// Part 2: CTA b solves its 32-row slab below the diagonal block:  X L11^T = A21.
__global__ void __launch_bounds__(1024) k_chol_trsm(double* __restrict__ A, int n, int j0) {
  __shared__ double D[kNB][kNB + 1], S[kNB][kNB + 1];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int gi = j0 + ty, gj = j0 + tx;
  D[ty][tx] = (gi < n && gj < n && tx <= ty) ? A[(size_t)gi * n + gj] : (tx == ty ? 1.0 : 0.0);
  const int ri = j0 + kNB * (1 + blockIdx.x) + ty;
  S[ty][tx] = (ri < n && gj < n) ? A[(size_t)ri * n + gj] : 0.0;
  __syncthreads();
  for (int c = 0; c < kNB; ++c) {
    if (tx == c) {
      double sv = S[ty][c];
      for (int k = 0; k < c; ++k) sv -= S[ty][k] * D[c][k];
      S[ty][c] = sv / D[c][c];
    }
    __syncthreads();
  }
  if (ri < n && gj < n) A[(size_t)ri * n + gj] = S[ty][tx];
}

// Trailing update after the panel at j0: A22 -= L21 L21^T (lower blocks only).
__global__ void __launch_bounds__(1024) k_chol_update(double* __restrict__ A, int n, int j0) {
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bj > bi) return;
  __shared__ double P[kNB][kNB + 1], Q[kNB][kNB + 1];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int i0 = j0 + kNB * (1 + bi), k0 = j0 + kNB * (1 + bj);
  P[ty][tx] = (i0 + ty < n && j0 + tx < n) ? A[(size_t)(i0 + ty) * n + j0 + tx] : 0.0;
  Q[ty][tx] = (k0 + ty < n && j0 + tx < n) ? A[(size_t)(k0 + ty) * n + j0 + tx] : 0.0;
  __syncthreads();
  const int gi = i0 + ty, gj = k0 + tx;
  if (gi < n && gj < n && gj <= gi) {
    double sv = 0.0;
#pragma unroll 8
    for (int k = 0; k < kNB; ++k) sv += P[ty][k] * Q[tx][k];
    A[(size_t)gi * n + gj] -= sv;
  }
}

__global__ void k_zero_upper(double* __restrict__ A, int n) {
  const int i = blockIdx.y * blockDim.y + threadIdx.y, k = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && k < n && k > i) A[(size_t)i * n + k] = 0.0;
}

// In-place lower Cholesky of the n x n row-major matrix A; fail[0] != 0 on a non-positive pivot; the strict
// upper triangle is zeroed so that A is exactly L.
static int launch_cholesky(double* A, int n, int* fail, cudaStream_t stream) {
  BB_CUDA(cudaMemsetAsync(fail, 0, sizeof(int), stream));
  const int nb = (n + kNB - 1) / kNB;
  for (int p = 0; p < nb; ++p) {
    k_chol_diag<<<1, dim3(kNB, kNB), 0, stream>>>(A, n, p * kNB, fail);
    BB_LAUNCH_CHECK();
    if (p + 1 < nb) {
      k_chol_trsm<<<nb - p - 1, dim3(kNB, kNB), 0, stream>>>(A, n, p * kNB);
      BB_LAUNCH_CHECK();
      k_chol_update<<<dim3(nb - p - 1, nb - p - 1), dim3(kNB, kNB), 0, stream>>>(A, n, p * kNB);
      BB_LAUNCH_CHECK();
    }
  }
  k_zero_upper<<<dim3((n + 15) / 16, (n + 15) / 16), dim3(16, 16), 0, stream>>>(A, n);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

// X = L^-1 (lower triangular).  Step 1: inverses of the diagonal blocks (one CTA each).
__global__ void __launch_bounds__(1024) k_trinv_diag(const double* __restrict__ L, int n, double* __restrict__ X) {
  __shared__ double D[kNB][kNB + 1], V[kNB][kNB + 1];
  const int tx = threadIdx.x, ty = threadIdx.y, j0 = blockIdx.x * kNB;
  const int gi = j0 + ty, gj = j0 + tx;
  D[ty][tx] = (gi < n && gj < n && tx <= ty) ? L[(size_t)gi * n + gj] : (tx == ty ? 1.0 : 0.0);
  V[ty][tx] = 0.0;
  __syncthreads();
  if (ty == 0) {  // thread tx owns column c = tx of the inverse
    const int c = tx;
    V[c][c] = 1.0 / D[c][c];
    for (int i = c + 1; i < kNB; ++i) {
      double sv = 0.0;
      for (int k = c; k < i; ++k) sv += D[i][k] * V[k][c];
      V[i][c] = -sv / D[i][i];
    }
  }
  __syncthreads();
  if (gi < n && gj < n) X[(size_t)gi * n + gj] = V[ty][tx];
}

// Step 2: block column J per CTA:  X_IJ = -X_II * sum_{K=J}^{I-1} L_IK X_KJ  for I = J+1.. (X_II from step 1).
__global__ void __launch_bounds__(1024) k_trinv_offdiag(const double* __restrict__ L, int n, double* X) {
  __shared__ double Ls[kNB][kNB + 1], Xs[kNB][kNB + 1], Ts[kNB][kNB + 1];
  const int tx = threadIdx.x, ty = threadIdx.y, J = blockIdx.x;
  const int nb = (n + kNB - 1) / kNB;
  const int gj = J * kNB + tx;
  for (int I = 0; I < J; ++I) {  // blocks above the diagonal are zero
    const int gi = I * kNB + ty;
    if (gi < n && gj < n) X[(size_t)gi * n + gj] = 0.0;
  }
  for (int I = J + 1; I < nb; ++I) {
    const int gi = I * kNB + ty;
    double acc = 0.0;
    for (int K = J; K < I; ++K) {
      const int lk = K * kNB + tx, xk = K * kNB + ty;
      Ls[ty][tx] = (gi < n && lk < n) ? L[(size_t)gi * n + lk] : 0.0;
      Xs[ty][tx] = (xk < n && gj < n) ? X[(size_t)xk * n + gj] : 0.0;
      __syncthreads();
#pragma unroll 8
      for (int k = 0; k < kNB; ++k) acc += Ls[ty][k] * Xs[k][tx];
      __syncthreads();
    }
    Ts[ty][tx] = acc;
    const int dk = I * kNB + tx;  // X_II (lower triangular)
    Ls[ty][tx] = (gi < n && dk < n && tx <= ty) ? X[(size_t)gi * n + dk] : 0.0;
    __syncthreads();
    double v = 0.0;
    for (int k = 0; k <= ty; ++k) v += Ls[ty][k] * Ts[k][tx];
    if (gi < n && gj < n) X[(size_t)gi * n + gj] = -v;
    __syncthreads();  // X_IJ is read (as X_KJ) by the next block rows
  }
}

static int launch_tri_inverse(const double* L, int n, double* X, cudaStream_t stream) {
  const int nb = (n + kNB - 1) / kNB;
  k_trinv_diag<<<nb, dim3(kNB, kNB), 0, stream>>>(L, n, X);
  BB_LAUNCH_CHECK();
  k_trinv_offdiag<<<nb, dim3(kNB, kNB), 0, stream>>>(L, n, X);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

// u = Linv r ; alpha = Linv^T u   (single CTA, n <= 1024 threads)
__global__ void k_alpha(const double* __restrict__ Linv, const double* __restrict__ resid, int n,
                        double* __restrict__ u, double* __restrict__ alpha64,
                        float* __restrict__ alpha32) {
  int t = threadIdx.x;
  if (t < n) {
    double s = 0.0;
    for (int i = 0; i <= t; ++i) s += Linv[(size_t)t * n + i] * resid[i];
    u[t] = s;
  }
  __syncthreads();
  if (t < n) {
    double s = 0.0;
    for (int j = t; j < n; ++j) s += Linv[(size_t)j * n + t] * u[j];
    alpha64[t] = s;
    alpha32[t] = (float)s;
  }
}

__global__ void k_absmax(const double* __restrict__ X, size_t count, double* __restrict__ out) {
  __shared__ double red[256];
  double m = 0.0;
  for (size_t e = threadIdx.x; e < count; e += blockDim.x) m = fmax(m, fabs(X[e]));
  red[threadIdx.x] = m;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = red[0];
}

// fp16 hi/lo image of (scale * L^-1) laid out as the sequence of B-operand tiles the MMA warp
// consumes: for K chunk c (training points 64c..64c+63) and N sub-block s >= c (columns
// 64s..64s+63 of D), one 16 KB tile [hi 8 KB | lo 8 KB], each [64 n-rows][64 k] fp16, K-major,
// 128-byte swizzled.  B[n=j][k=i] = Linv[j][i] so that D[m][j] = sum_i K*[m][i] Linv[j][i].
__global__ void k_build_rimg(const double* __restrict__ Linv, int n, int n_chunks, double scale,
                             uint8_t* __restrict__ rimg, float* __restrict__ linv32, int n_pad) {
  int tile = blockIdx.x;
  // decode (c, s) from the linear tile index: tiles are ordered c-major, s = c..C-1
  int c = 0, rem = tile;
  while (rem >= n_chunks - c) {
    rem -= n_chunks - c;
    ++c;
  }
  int s = c + rem;
  uint8_t* base = rimg + (size_t)tile * 16384;
  for (int e = threadIdx.x; e < 64 * 64; e += blockDim.x) {
    int r = e >> 6, kk = e & 63;
    int j = s * 64 + r, i = c * 64 + kk;
    double v = (j < n && i < n && i <= j) ? Linv[(size_t)j * n + i] * scale : 0.0;
    float vf = (float)v;
    __half hi = __float2half_rn(vf);
    __half lo = __float2half_rn((float)(v - (double)__half2float(hi)));
    uint32_t off = sw128_offset((uint32_t)r, (uint32_t)(kk >> 3)) + (uint32_t)(kk & 7) * 2u;
    *reinterpret_cast<__half*>(base + off) = hi;
    *reinterpret_cast<__half*>(base + 8192 + off) = lo;
  }
  // fp32 dense copy, zero padded (the strict upper triangle stays zero from the blob memset)
  for (int e = threadIdx.x; e < 64 * 64; e += blockDim.x) {
    int r = e >> 6, kk = e & 63;
    int j = s * 64 + r, i = c * 64 + kk;
    double v = (j < n && i < n && i <= j) ? Linv[(size_t)j * n + i] : 0.0;
    linv32[(size_t)j * n_pad + i] = (float)v;
  }
}

// Augmented training-row image of the tensor-core distances (k_fused, k_kmat_tma): three panels [hi | mid | lo] of
// [n_pad rows][K2 k] fp16 (K2 = 32: 64-byte rows, SWIZZLE_64B; K2 = 64: 128-byte rows, SWIZZLE_128B):
//     k < d: scale_b * (-2 b_ij); k = K2 - 2: q_one (pairs with |a|^2 * P in the candidate tile);
//     k = K2 - 1: |b_i|^2 * q_sq (pairs with P1).  Rows i >= n are zero.
template <int K2>
__global__ void k_build_timg_b(const float* __restrict__ train_m2, const float* __restrict__ train_sq, int n, int n_pad,
                               int d, int d_pad, float scale_b, float q_one, float q_sq, uint8_t* __restrict__ img) {
  const uint32_t split = (uint32_t)n_pad * K2 * 2u;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n_pad * K2; e += gridDim.x * blockDim.x) {
    const int i = e / K2, j = e % K2;
    float v = 0.f;
    if (i < n) {
      if (j < d) v = train_m2[(size_t)i * d_pad + j] * scale_b;
      else if (j == K2 - 2) v = q_one;
      else if (j == K2 - 1) v = train_sq[i] * q_sq;
    }
    const __half h = __float2half_rn(v);
    const float r1 = v - __half2float(h);
    const __half m = __float2half_rn(r1);
    const __half l = __float2half_rn(r1 - __half2float(m));
    const uint32_t o = swk_offset<K2>((uint32_t)i, (uint32_t)(j >> 3)) + (uint32_t)(j & 7) * 2u;
    *reinterpret_cast<__half*>(img + o) = h;
    *reinterpret_cast<__half*>(img + split + o) = m;
    *reinterpret_cast<__half*>(img + 2 * split + o) = l;
  }
}
// K-chunked fp16 hi/mid/lo image of scale * src[n_pad][d_wide] for wide.cu: per (256-row half,
// 32-column K stage) `panels` panels [hi | mid (| lo)], each [ncols rows][32 fp16], 64-byte rows,
// SWIZZLE_64B, 8-row groups contiguous -- one contiguous bulk copy per stage.
__global__ void k_build_wimg(const float* __restrict__ src, int n_pad, int d_wide, float scale,
                             int panels, uint8_t* __restrict__ img) {
  const int n_kc = d_wide / 32;
  const size_t total = (size_t)n_pad * d_wide;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int i = (int)(e / d_wide), k = (int)(e - (size_t)i * d_wide);
    const int half = i >> 8, il = i & 255;
    const int ncols = min(256, n_pad - half * 256);
    const int kc = k >> 5, kl = k & 31;
    const size_t panel = (size_t)ncols * 64;
    const size_t base = (size_t)half * n_kc * ((size_t)panels * 256 * 64) + (size_t)kc * panels * panel;
    const uint32_t off = swk_offset<32>((uint32_t)il, (uint32_t)(kl >> 3)) + (uint32_t)(kl & 7) * 2u;
    const float v = src[e] * scale;
    const __half h = __float2half_rn(v);
    const float r1 = v - __half2float(h);
    const __half m = __float2half_rn(r1);
    const __half l = __float2half_rn(r1 - __half2float(m));
    *reinterpret_cast<__half*>(img + base + off) = h;
    *reinterpret_cast<__half*>(img + base + panel + off) = m;
    if (panels > 2) *reinterpret_cast<__half*>(img + base + 2 * panel + off) = l;
  }
}

// ------------------------------------------------------------------------------------------
// pending-point statistics (float64 math, fp32 outputs)
// ------------------------------------------------------------------------------------------
// one CTA per pending point p: kx = k(X, p) ; w = Linv kx ; beta = Linv^T w ; mu = c + kx.alpha
__global__ void k_pending_w(const float* __restrict__ pend_x, int P, int n, int n_pad, int d,
                            int T, int family, int task_col, const double* __restrict__ xn,
                            const int32_t* __restrict__ ttask, const double* __restrict__ aux,
                            const float* __restrict__ cand_norm /* [2*d]: lo, inv_range */,
                            const double* __restrict__ Linv, const double* __restrict__ alpha64,
                            const float* __restrict__ mean_const, float y_mean, float y_std,
                            float* __restrict__ beta_out, float* __restrict__ mu_out,
                            double* __restrict__ pn_out /* [P*d] normalised pending */,
                            double* __restrict__ w_out /* [P*n] */) {
  extern __shared__ double sh[];
  double* pn = sh;           // [d]
  double* kx = sh + d;       // [n]
  double* w = sh + d + n;    // [n]
  __shared__ double red[256];
  int p = blockIdx.x, tid = threadIdx.x;
  const double* tcov = aux;
  const double* inv_ls = aux + T * T;
  for (int j = tid; j < d; j += blockDim.x) {
    double x = (double)pend_x[(size_t)p * d + j];
    double v = (j == task_col) ? x : (x - (double)cand_norm[j]) * (double)cand_norm[d + j];
    pn[j] = v;
    pn_out[(size_t)p * d + j] = v;
  }
  __syncthreads();
  int tp = (task_col >= 0) ? min(max((int)llrint(pn[task_col]), 0), T - 1) : 0;
  double part = 0.0;
  for (int i = tid; i < n; i += blockDim.x) {
    double k = k_pair_f64(pn, xn + (size_t)i * d, d, inv_ls, family) * tcov[tp * T + ttask[i]];
    kx[i] = k;
    part += k * alpha64[i];
  }
  red[tid] = part;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) red[tid] += red[tid + s];
    __syncthreads();
  }
  if (tid == 0) mu_out[p] = y_mean + y_std * (float)((double)mean_const[tp] + red[0]);
  for (int j = tid; j < n; j += blockDim.x) {
    double s = 0.0;
    for (int i = 0; i <= j; ++i) s += Linv[(size_t)j * n + i] * kx[i];
    w[j] = s;
    w_out[(size_t)p * n + j] = s;
  }
  __syncthreads();
  for (int i = tid; i < n_pad; i += blockDim.x) {
    double s = 0.0;
    if (i < n)
      for (int j = i; j < n; ++j) s += Linv[(size_t)j * n + i] * w[j];
    beta_out[(size_t)p * n_pad + i] = (float)s;
  }
}

// cov[p][q] = (k(p,q) - w_p . w_q) * y_std^2, float64
__global__ void k_pending_cov(const double* __restrict__ pn, const double* __restrict__ w, int P,
                              int n, int d, int T, int family, int task_col,
                              const double* __restrict__ aux, float y_std,
                              float* __restrict__ cov) {
  int p = blockIdx.x, q = threadIdx.x;
  if (q >= P) return;
  const double* tcov = aux;
  const double* inv_ls = aux + T * T;
  int tp = (task_col >= 0) ? min(max((int)llrint(pn[(size_t)p * d + task_col]), 0), T - 1) : 0;
  int tq = (task_col >= 0) ? min(max((int)llrint(pn[(size_t)q * d + task_col]), 0), T - 1) : 0;
  double k = (p == q) ? 1.0 : k_pair_f64(pn + (size_t)p * d, pn + (size_t)q * d, d, inv_ls, family);
  k *= tcov[tp * T + tq];
  double s = 0.0;
  for (int j = 0; j < n; ++j) s += w[(size_t)p * n + j] * w[(size_t)q * n + j];
  cov[p * P + q] = (float)((k - s) * (double)y_std * (double)y_std);
}

}  // namespace bb

using namespace bb;

extern "C" int bb_abi_version(void) { return BB_ABI_VERSION; }
extern "C" const char* bb_last_error(void) { return bb::last_error(); }

extern "C" size_t bb_model_blob_bytes(int32_t n, int32_t d, int32_t n_tasks) {
  if (n <= 0 || d <= 0 || n_tasks <= 0) return 0;
  return make_layout(n, d, n_tasks).total;
}

extern "C" int bb_model_build(const bb_model_desc* desc, void* d_blob, size_t blob_bytes,
                              bb_model* out, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  BB_CHECK_ARG(desc && d_blob && out, "bb_model_build: null argument");
  const int n = desc->n, d = desc->d, T = desc->n_tasks;
  BB_CHECK_ARG(n >= 1 && d >= 1 && T >= 1, "bb_model_build: n, d, n_tasks must be positive");
  BB_CHECK_SUPPORTED(n <= BB_MAX_TRAIN,
                     "bb_model_build: n=%d training points exceeds this build's limit of %d", n,
                     BB_MAX_TRAIN);
  BB_CHECK_ARG(desc->family >= 0 && desc->family <= 3, "bb_model_build: unknown kernel family %d",
               desc->family);
  BB_CHECK_ARG(desc->task_col >= -1 && desc->task_col < d, "bb_model_build: bad task_col");
  BB_CHECK_ARG((desc->task_col >= 0) == (desc->task_covar != nullptr) || T == 1,
               "bb_model_build: task_col and task_covar must be given together");
  BB_CHECK_ARG(desc->train_x && desc->train_y && desc->lower && desc->upper && desc->lengthscale &&
                   desc->noise && desc->mean_const,
               "bb_model_build: null array in descriptor");
  BB_CHECK_ARG(((uintptr_t)d_blob & 1023) == 0, "bb_model_build: blob must be 1024-byte aligned");
  BlobLayout L = make_layout(n, d, T);
  if (blob_bytes < bb_model_blob_bytes(n, d, T)) {
    set_error("bb_model_build: blob of %zu bytes is smaller than the required %zu", blob_bytes,
              bb_model_blob_bytes(n, d, T));
    return BB_ERR_WORKSPACE;
  }
  // ---- host-side parameter packing (float64): Normalize / Standardize / ARD folding ----
  const double kfam = desc->family == BB_KERNEL_MATERN52   ? 5.0
                      : desc->family == BB_KERNEL_MATERN32 ? 3.0
                      : desc->family == BB_KERNEL_MATERN12 ? 1.0
                                                           : 0.5 * 1.4426950408889634;
  const double sq_kfam = sqrt(kfam);
  std::vector<double> lo(d), inv_range(d), inv_ls(d), centre(d, 0.0), xn((size_t)n * d);
  for (int j = 0; j < d; ++j) {
    double r = desc->upper[j] - desc->lower[j];
    if (fabs(r) < 1e-8) r = 1.0;  // botorch Normalize(min_range = 1e-8): degenerate range -> 1
    lo[j] = desc->lower[j];
    inv_range[j] = 1.0 / r;
    double ls = desc->lengthscale[j];
    inv_ls[j] = (j == desc->task_col || !(ls > 0.0)) ? 0.0 : 1.0 / ls;
    if (j == desc->task_col) {
      lo[j] = 0.0;
      inv_range[j] = 1.0;
    }
  }
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < d; ++j) {
      double v = (desc->train_x[(size_t)i * d + j] - lo[j]) * inv_range[j];
      xn[(size_t)i * d + j] = v;
      centre[j] += v / n;
    }
  std::vector<int32_t> ttask(L.n_pad, 0);
  if (desc->task_col >= 0)
    for (int i = 0; i < n; ++i) {
      long t = lrint(xn[(size_t)i * d + desc->task_col]);
      BB_CHECK_ARG(t >= 0 && t < T, "bb_model_build: training task id %ld outside [0,%d)", t, T);
      ttask[i] = (int32_t)t;
    }
  double y_mean = 0.0, y_std = 1.0;
  for (int i = 0; i < n; ++i) y_mean += desc->train_y[i] / n;
  if (n > 1) {
    double ss = 0.0;
    for (int i = 0; i < n; ++i) ss += (desc->train_y[i] - y_mean) * (desc->train_y[i] - y_mean);
    y_std = sqrt(ss / (n - 1));
    if (!(y_std >= 1e-8)) y_std = 1.0;  // botorch Standardize min_stdv
  }
  const double prior_scale = desc->has_outputscale ? desc->outputscale : 1.0;
  std::vector<double> aux(T * T + d);
  for (int a = 0; a < T; ++a)
    for (int b = 0; b < T; ++b)
      aux[a * T + b] = prior_scale * (desc->task_covar ? desc->task_covar[a * T + b] : 1.0);
  for (int j = 0; j < d; ++j) aux[T * T + j] = inv_ls[j];
  std::vector<double> resid(n), noise_row(n);
  for (int i = 0; i < n; ++i) {
    double nz = desc->noise[ttask[i]];
    noise_row[i] = nz < 1e-4 ? 1e-4 : nz;  // MIN_INFERRED_NOISE_LEVEL
    resid[i] = (desc->train_y[i] - y_mean) / y_std - desc->mean_const[ttask[i]];
  }
  // fp32 candidate transform a_j = x_j*scale_j + shift_j and the (-2 x) scaled training rows
  std::vector<float> cscale(L.d_pad, 0.f), cshift(L.d_pad, 0.f), tm2((size_t)L.n_pad * L.d_pad, 0.f),
      tsq(L.n_pad, 0.f), tcov32(T * T), mean32(T), cnorm(2 * d);
  for (int j = 0; j < d; ++j) {
    double g = inv_ls[j] * sq_kfam;
    cscale[j] = (float)(inv_range[j] * g);
    cshift[j] = (float)(-(lo[j] * inv_range[j] + centre[j]) * g);
    cnorm[j] = (float)lo[j];
    cnorm[d + j] = (float)inv_range[j];
  }
  for (int i = 0; i < n; ++i) {
    double sq = 0.0;
    for (int j = 0; j < d; ++j) {
      float b = (float)((xn[(size_t)i * d + j] - centre[j]) * inv_ls[j] * sq_kfam);
      tm2[(size_t)i * L.d_pad + j] = -2.0f * b;
      sq += (double)b * (double)b;
    }
    tsq[i] = (float)sq;
  }
  // power-of-two scales for the fp16 split images of the distance GEMM (only used for d_pad <= 64)
  float a_abs_max = 1e-30f, b_abs_max = 1e-30f;
  for (int j = 0; j < d; ++j) {
    a_abs_max = fmaxf(a_abs_max, fmaxf(fabsf((float)desc->lower[j] * cscale[j] + cshift[j]),
                                       fabsf((float)desc->upper[j] * cscale[j] + cshift[j])));
  }
  for (size_t e = 0; e < tm2.size(); ++e) b_abs_max = fmaxf(b_abs_max, fabsf(tm2[e]));
  if (!(a_abs_max > 1e-6f)) a_abs_max = 1.0f;
  if (!(b_abs_max > 1e-6f)) b_abs_max = 1.0f;
  const float dist_scale_a = ldexpf(1.0f, (int)floorf(log2f(4000.0f / a_abs_max)));   // 16x head-room
  const float dist_scale_b = ldexpf(1.0f, (int)floorf(log2f(30000.0f / b_abs_max)));
  // padded training rows: zero kernel contribution is guaranteed by zero rows of L^-1 / alpha
  for (int a = 0; a < T * T; ++a) tcov32[a] = (float)aux[a];
  for (int a = 0; a < T; ++a) mean32[a] = (float)desc->mean_const[a];

  uint8_t* B = (uint8_t*)d_blob;
  BB_CUDA(cudaMemsetAsync(B, 0, L.total, stream));
  auto up = [&](size_t off, const void* src, size_t bytes) {
    return cudaMemcpyAsync(B + off, src, bytes, cudaMemcpyHostToDevice, stream);
  };
  BB_CUDA(up(L.cand_scale, cscale.data(), cscale.size() * 4));
  BB_CUDA(up(L.cand_shift, cshift.data(), cshift.size() * 4));
  BB_CUDA(up(L.train_m2, tm2.data(), tm2.size() * 4));
  BB_CUDA(up(L.train_sq, tsq.data(), tsq.size() * 4));
  BB_CUDA(up(L.train_task, ttask.data(), ttask.size() * 4));
  BB_CUDA(up(L.task_covar, tcov32.data(), tcov32.size() * 4));
  BB_CUDA(up(L.mean_const, mean32.data(), mean32.size() * 4));
  BB_CUDA(up(L.xn64, xn.data(), xn.size() * 8));
  BB_CUDA(up(L.resid, resid.data(), resid.size() * 8));
  BB_CUDA(up(L.noise_row, noise_row.data(), noise_row.size() * 8));
  BB_CUDA(up(L.tcov64, aux.data(), aux.size() * 8));
  BB_CUDA(up(L.cnorm, cnorm.data(), cnorm.size() * 4));
  BB_CUDA(cudaStreamSynchronize(stream));  // host vectors above go out of scope only after this

  double* dK = (double*)(B + L.kmat);
  double* dLinv = (double*)(B + L.linv);
  int* dflag = (int*)(B + L.flags);
  double* dmax = (double*)(B + L.flags + 16);
  int tries = 0;
  double jitter = 0.0;
  for (;; ++tries) {
    // linear_operator psd_safe_cholesky: plain, then 1e-8, 1e-7, 1e-6 (float64)
    jitter = tries == 0 ? 0.0 : 1e-8 * pow(10.0, tries - 1);
    dim3 blk(16, 16), grd((n + 15) / 16, (n + 15) / 16);
    k_train_gram<<<grd, blk, 0, stream>>>((const double*)(B + L.xn64),
                                          (const int32_t*)(B + L.train_task),
                                          (const double*)(B + L.tcov64),
                                          (const double*)(B + L.noise_row), n, d, T, desc->family,
                                          jitter, dK);
    BB_LAUNCH_CHECK();
    {
      const int rc_chol = launch_cholesky(dK, n, dflag, stream);
      if (rc_chol != BB_OK) return rc_chol;
    }
    int flag = 0;
    BB_CUDA(cudaMemcpyAsync(&flag, dflag, sizeof(int), cudaMemcpyDeviceToHost, stream));
    BB_CUDA(cudaStreamSynchronize(stream));
    if (flag == 0) break;
    if (tries == 3) {
      set_error("bb_model_build: K + noise*I is not positive definite (jitter up to 1e-6 tried)");
      return BB_ERR_NOT_PD;
    }
  }
  {
    const int rc_inv = launch_tri_inverse(dK, n, dLinv, stream);
    if (rc_inv != BB_OK) return rc_inv;
  }
  k_alpha<<<1, 1024, 0, stream>>>(dLinv, (const double*)(B + L.resid), n,
                                  (double*)(B + L.resid) + n, (double*)(B + L.alpha64),
                                  (float*)(B + L.alpha));
  BB_LAUNCH_CHECK();
  k_absmax<<<1, 256, 0, stream>>>(dLinv, (size_t)n * n, dmax);
  BB_LAUNCH_CHECK();
  double amax = 0.0;
  BB_CUDA(cudaMemcpyAsync(&amax, dmax, sizeof(double), cudaMemcpyDeviceToHost, stream));
  BB_CUDA(cudaStreamSynchronize(stream));
  if (!(amax > 0.0) || !isfinite(amax)) {
    set_error("bb_model_build: L^-1 has no finite non-zero entries (max |.| = %g)", amax);
    return BB_ERR_NOT_PD;
  }
  // power-of-two scale so that max |scale * Linv| lies in [2^13, 2^14): well inside fp16 range
  int e;
  frexp(amax, &e);  // amax = f * 2^e, f in [0.5,1)
  double scale = ldexp(1.0, 14 - e);
  k_build_rimg<<<L.n_tiles, 256, 0, stream>>>(dLinv, n, L.n_chunks, scale, B + L.rimg,
                                              (float*)(B + L.linv32), L.n_pad);
  BB_LAUNCH_CHECK();

  // ---- augmented training image of the tensor-core distances and its power-of-two scales ----
  // A2 = [sa * a | asq * P | P1], Bt = [sb * (-2b) | Q1 | bsq * Q] with sa*sb = P*Q1 = P1*Q = G, so that the
  // distance GEMM accumulates D = G * (|a|^2 + |b|^2 - 2 a.b) = G * t.  All fp16 operands stay below 2^15.
  float ts_sa = 0.f, ts_aug_sq = 0.f, ts_aug_one = 0.f, ts_g = 0.f, ts_kscale = 1.f;
  if (L.ts) {
    double asq_max = 0.0, bsq_max = 1e-30;
    for (int j = 0; j < d; ++j) {
      const double aj = fmax(fabs((double)desc->lower[j] * cscale[j] + cshift[j]),
                             fabs((double)desc->upper[j] * cscale[j] + cshift[j]));
      asq_max += aj * aj;
    }
    for (int i = 0; i < n; ++i) bsq_max = fmax(bsq_max, (double)tsq[i]);
    if (!(asq_max > 1e-12)) asq_max = 1.0;
    const int e_p = (int)floor(log2(30000.0 / asq_max));                 // P  = 2^e_p
    const int e_q = (int)floor(log2(30000.0 / bsq_max));                 // Q  = 2^e_q
    const int e_sb = (int)floor(log2(30000.0 / (double)b_abs_max));      // sb = 2^e_sb
    const int e_sa_max = (int)floor(log2(16000.0 / (double)a_abs_max));  // sa <= 2^e_sa_max
    int e_g = e_sb + e_sa_max;                                           // G = 2^e_g
    if (e_g > 15 + e_p) e_g = 15 + e_p;                                  // Q1 = G / P  <= 2^15
    if (e_g > 15 + e_q) e_g = 15 + e_q;                                  // P1 = G / Q  <= 2^15
    if (e_g & 1) --e_g;                                                  // sqrt(G) exact
    ts_sa = ldexpf(1.0f, e_g - e_sb);
    ts_aug_sq = ldexpf(1.0f, e_p);
    ts_aug_one = ldexpf(1.0f, e_g - e_q);
    ts_g = ldexpf(1.0f, -e_g);
    const float q_one = ldexpf(1.0f, e_g - e_p), q_sq = ldexpf(1.0f, e_q), ts_sb = ldexpf(1.0f, e_sb);
    // K* scale: largest kernel value (prior scale x task covariance) times ts_kscale stays below 2^15
    double kmax = 0.0;
    for (int a = 0; a < T * T; ++a) kmax = fmax(kmax, fabs(aux[a]));
    if (!(kmax > 0.0)) kmax = 1.0;
    int e_k = (int)floor(log2(30000.0 / kmax));
    if (e_k > 10) e_k = 10;
    ts_kscale = ldexpf(1.0f, e_k);
    if (L.ts == 32)
      k_build_timg_b<32><<<32, 256, 0, stream>>>((const float*)(B + L.train_m2), (const float*)(B + L.train_sq), n,
                                                 L.n_pad, d, L.d_pad, ts_sb, q_one, q_sq, B + L.timg_b);
    else
      k_build_timg_b<64><<<32, 256, 0, stream>>>((const float*)(B + L.train_m2), (const float*)(B + L.train_sq), n,
                                                 L.n_pad, d, L.d_pad, ts_sb, q_one, q_sq, B + L.timg_b);
    BB_LAUNCH_CHECK();
  }

  float dist_scale_w = 1.0f, dist_scale_p = 1.0f, dist_scale_wp = 1.0f;
  if (L.wide) {
    // pending points lie inside the scaling bounds like candidates: bound their operand magnitudes there
    float wp_max = 1e-30f;
    for (int j = 0; j < d; ++j) {
      const float aj = fmaxf(fabsf((float)desc->lower[j] * cscale[j] + cshift[j]),
                             fabsf((float)desc->upper[j] * cscale[j] + cshift[j]));
      wp_max = fmaxf(wp_max, fabsf(cscale[j]) * (2.0f * aj + fabsf(cscale[j]) + 2.0f * fabsf(cshift[j])));
    }
    dist_scale_p = ldexpf(1.0f, (int)floorf(log2f(30000.0f / (2.0f * a_abs_max))));
    dist_scale_wp = ldexpf(1.0f, (int)floorf(log2f(30000.0f / wp_max)));
    // float layouts: B = -2 b (same numbers as d_train_m2, K-chunked)
    std::vector<float> src((size_t)L.n_pad * L.d_wide, 0.f);
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < d; ++j) src[(size_t)i * L.d_wide + j] = tm2[(size_t)i * L.d_pad + j];
    BB_CUDA(up(L.wsrc, src.data(), src.size() * 4));
    k_build_wimg<<<296, 256, 0, stream>>>((const float*)(B + L.wsrc), L.n_pad, L.d_wide, dist_scale_b,
                                          3, B + L.wimg);
    BB_LAUNCH_CHECK();
    BB_CUDA(cudaStreamSynchronize(stream));
    // bit-packed layout: t = sum_j x_j W_ij + c_i with a_j = s_j x_j + h_j, x_j in {0,1}
    std::vector<float> cvec(L.n_pad, 0.f);
    float w_abs_max = 1e-30f;
    for (int i = 0; i < n; ++i) {
      double c = (double)tsq[i];
      for (int j = 0; j < d; ++j) {
        const double sj = cscale[j], hj = cshift[j], m2 = tm2[(size_t)i * L.d_pad + j];
        const float w = (float)(sj * (m2 + sj + 2.0 * hj));
        src[(size_t)i * L.d_wide + j] = w;
        w_abs_max = fmaxf(w_abs_max, fabsf(w));
        c += hj * (m2 + hj);
      }
      cvec[i] = (float)c;
    }
    if (!(w_abs_max > 1e-6f)) w_abs_max = 1.0f;
    dist_scale_w = ldexpf(1.0f, (int)floorf(log2f(30000.0f / w_abs_max)));
    BB_CUDA(up(L.wsrc, src.data(), src.size() * 4));
    BB_CUDA(up(L.wnorm_bits, cvec.data(), cvec.size() * 4));
    k_build_wimg<<<296, 256, 0, stream>>>((const float*)(B + L.wsrc), L.n_pad, L.d_wide, dist_scale_w,
                                          2, B + L.wimg_bits);
    BB_LAUNCH_CHECK();
    BB_CUDA(cudaStreamSynchronize(stream));
  }

  memset(out, 0, sizeof(*out));
  out->abi_version = BB_ABI_VERSION;
  out->n = n;
  out->n_pad = L.n_pad;
  out->d = d;
  out->d_pad = L.d_pad;
  out->family = desc->family;
  out->task_col = desc->task_col;
  out->n_tasks = T;
  out->n_chunks = L.n_chunks;
  out->jitter_tries = tries;
  out->jitter = jitter;
  out->y_mean = (float)y_mean;
  out->y_std = (float)y_std;
  out->prior_scale = (float)prior_scale;
  out->r_scale = (float)scale;
  out->d_blob = d_blob;
  out->blob_bytes = blob_bytes;
  out->d_cand_scale = (const float*)(B + L.cand_scale);
  out->d_cand_shift = (const float*)(B + L.cand_shift);
  out->d_train_m2 = (const float*)(B + L.train_m2);
  out->d_train_sq = (const float*)(B + L.train_sq);
  out->d_alpha = (const float*)(B + L.alpha);
  out->d_train_task = (const int32_t*)(B + L.train_task);
  out->d_task_covar = (const float*)(B + L.task_covar);
  out->d_mean_const = (const float*)(B + L.mean_const);
  out->d_rimg = B + L.rimg;
  out->d_linv = dLinv;
  out->d_alpha64 = (const double*)(B + L.alpha64);
  out->d_xn64 = (const double*)(B + L.xn64);
  out->d_linv32 = (const float*)(B + L.linv32);
  out->dist_scale_a = dist_scale_a;
  out->dist_scale_b = dist_scale_b;
  if (L.ts) {
    out->d_timg_b = B + L.timg_b;
    out->dist_k = L.ts;
    if (!L.wide) out->d_mc_table = (float*)(B + L.mc_table);
    out->ts_sa = ts_sa;
    out->ts_aug_sq = ts_aug_sq;
    out->ts_aug_one = ts_aug_one;
    out->ts_g = ts_g;
    out->ts_kscale = ts_kscale;
  }
  out->wide = L.wide;
  out->d_wide = L.d_wide;
  if (L.wide) {
    out->d_wimg = B + L.wimg;
    out->d_wimg_bits = B + L.wimg_bits;
    out->d_wnorm_bits = (const float*)(B + L.wnorm_bits);
    out->d_wide_ws = (float*)(B + L.wide_ws);
    out->d_pend_img = B + L.pend_img;
    out->d_pend_norm = (float*)(B + L.pend_norm2);
    out->d_pend_task = (int32_t*)(B + L.pend_task);
    out->d_kpend_ws = (float*)(B + L.kpend_ws);
    out->d_mc_table = (float*)(B + L.mc_table);
    out->dist_scale_p = dist_scale_p;
    out->dist_scale_wp = dist_scale_wp;
    out->wide_ws_rows = L.wide_ws_rows;
    out->dist_scale_w = dist_scale_w;
  }
  BB_CUDA(cudaStreamSynchronize(stream));
  return BB_OK;
}

extern "C" int bb_pending_stats(const bb_model* m, const float* d_pend_x, int32_t P,
                                float* d_pend_beta, float* d_pend_mu, float* d_pend_cov,
                                void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  BB_CHECK_ARG(m && d_pend_x && d_pend_beta && d_pend_mu && d_pend_cov,
               "bb_pending_stats: null argument");
  BB_CHECK_ARG(m->abi_version == BB_ABI_VERSION, "bb_pending_stats: ABI mismatch");
  BB_CHECK_ARG(P >= 1 && P <= BB_MAX_PENDING, "bb_pending_stats: n_pending=%d outside [1,%d]", P,
               BB_MAX_PENDING);
  BlobLayout L = make_layout(m->n, m->d, m->n_tasks);
  uint8_t* B = (uint8_t*)m->d_blob;
  double* pn = (double*)(B + L.pend_norm);  // normalised pending rows (scratch inside the blob)
  double* w64 = (double*)(B + L.pend_w64);
  size_t shm = sizeof(double) * (m->d + 2 * m->n);
  k_pending_w<<<P, 256, shm, stream>>>(d_pend_x, P, m->n, m->n_pad, m->d, m->n_tasks, m->family,
                                       m->task_col, m->d_xn64, m->d_train_task,
                                       (const double*)(B + L.tcov64), (const float*)(B + L.cnorm),
                                       m->d_linv, m->d_alpha64, m->d_mean_const, m->y_mean,
                                       m->y_std, d_pend_beta, d_pend_mu, pn, w64);
  BB_LAUNCH_CHECK();
  k_pending_cov<<<P, 32, 0, stream>>>(pn, w64, P, m->n, m->d, m->n_tasks, m->family, m->task_col,
                                      (const double*)(B + L.tcov64), m->y_std, d_pend_cov);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

// ------------------------------------------------------------------------------------------
// MAP-fit objective on device (SURVEY.md 8f-1): exact marginal log likelihood of the GP that
// GaussianProcessSurrogate._fit hands to botorch.fit.fit_gpytorch_mll
// (/root/reference/baybe/surrogates/gaussian_process/core.py:331-341, criterion
// components/fit_criterion.py:22-41) and its gradient, float64.  The priors are closed-form in theta
// and stay on the host, as does the L-BFGS-B driver (scipy, like botorch's scipy_minimize).
//   theta = [ lengthscale[d] | noise | mean constant | B[T*T] task covariance (outputscale folded in) ]
//   mll   = -1/2 r^T K^-1 r - 1/2 log|K| - n/2 log 2 pi ,  r = y - c
//   d mll / d theta_p = 1/2 tr((alpha alpha^T - K^-1) dK/dtheta_p) ,  d mll / dc = sum(alpha)
// ------------------------------------------------------------------------------------------
namespace {

struct FitLayout {
  size_t xn, y, task, theta, K, Linv, Kinv, alpha, resid, partial, out, alpha32, flag, wmat, loovec, total;
  int nblk, np;
};

FitLayout fit_layout(int n, int d, int T) {
  FitLayout L;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return o;
  };
  L.np = d + 2 + T * T;
  L.nblk = (int)(((size_t)n * n + 1023) / 1024);
  L.xn = take(sizeof(double) * (size_t)n * d);
  L.y = take(sizeof(double) * n);
  L.task = take(sizeof(int32_t) * n);
  L.theta = take(sizeof(double) * L.np);
  L.K = take(sizeof(double) * (size_t)n * n);
  L.Linv = take(sizeof(double) * (size_t)n * n);
  L.Kinv = take(sizeof(double) * (size_t)n * n);
  L.alpha = take(sizeof(double) * n);
  L.resid = take(sizeof(double) * n * 2);
  L.partial = take(sizeof(double) * (size_t)L.nblk * L.np);
  L.out = take(sizeof(double) * (L.np + 1));
  L.alpha32 = take(sizeof(float) * n);
  L.flag = take(64);
  L.wmat = take(sizeof(double) * (size_t)n * n);   // leave-one-out criterion: 2 dF/dK
  L.loovec = take(sizeof(double) * 4 * n);          // kappa | w | u | v
  L.total = off;
  return L;
}

// d k / d(r^2) of the stationary kernels (r2 > 0)
__device__ __forceinline__ double dkernel_f64(int family, double r2) {
  if (family == BB_KERNEL_RBF) return -0.5 * exp(-0.5 * r2);
  const double r = sqrt(fmax(r2, 1e-300));
  if (family == BB_KERNEL_MATERN12) return r2 > 1e-24 ? -exp(-r) / (2.0 * r) : 0.0;
  if (family == BB_KERNEL_MATERN32) return -1.5 * exp(-1.7320508075688772 * r);
  const double s = 2.23606797749979 * r;
  return -(5.0 / 6.0) * (1.0 + s) * exp(-s);
}

__global__ void k_fit_gram(const double* __restrict__ xn, const int32_t* __restrict__ task,
                           const double* __restrict__ theta, const double* __restrict__ y, int n, int d,
                           int T, int family, double* __restrict__ K, double* __restrict__ resid) {
  const int i = blockIdx.y * blockDim.y + threadIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || j >= n) return;
  const double* B = theta + d + 2;
  double k = 1.0;
  if (i != j) {
    double r2 = 0.0;
    for (int c = 0; c < d; ++c) {
      const double u = (xn[(size_t)i * d + c] - xn[(size_t)j * d + c]) / theta[c];
      r2 += u * u;
    }
    k = kernel_f64(family, r2);
  }
  k *= B[task[i] * T + task[j]];
  if (i == j) {
    k += theta[d];
    resid[i] = y[i] - theta[d + 1];
  }
  K[(size_t)i * n + j] = k;
}

// K^-1 = L^-T L^-1
__global__ void k_fit_kinv(const double* __restrict__ Linv, int n, double* __restrict__ Kinv) {
  const int i = blockIdx.y * blockDim.y + threadIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || k >= n) return;
  double s = 0.0;
  for (int m = max(i, k); m < n; ++m) s += Linv[(size_t)m * n + i] * Linv[(size_t)m * n + k];
  Kinv[(size_t)i * n + k] = s;
}

__device__ __forceinline__ double block_sum_256(double v, double* red) {
  const int t = threadIdx.x;
  red[t] = v;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (t < s) red[t] += red[t + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// per-block partial gradients over 1024 (i,k) pairs; fixed summation order (deterministic)
__global__ void __launch_bounds__(256) k_fit_grad(const double* __restrict__ xn, const int32_t* __restrict__ task,
                                                  const double* __restrict__ theta, const double* __restrict__ alpha,
                                                  const double* __restrict__ Kinv, int n, int d, int T, int family,
                                                  double* __restrict__ partial,
                                                  const double* __restrict__ wmat) {  // null: exact MLL
  __shared__ double red[256];
  const double* B = theta + d + 2;
  const int np = d + 2 + T * T;
  double g[4], hb[4];  // 1/2 W B dk/dr2 ; 1/2 W kbase
  int pi[4], pk[4];
  double gn = 0.0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const size_t e = (size_t)blockIdx.x * 1024 + q * 256 + threadIdx.x;
    g[q] = hb[q] = 0.0;
    pi[q] = pk[q] = 0;
    if (e < (size_t)n * n) {
      const int i = (int)(e / n), k = (int)(e - (size_t)i * n);
      pi[q] = i;
      pk[q] = k;
      const double W = wmat != nullptr ? wmat[e] : alpha[i] * alpha[k] - Kinv[e];
      if (i == k) {
        gn += 0.5 * W;
        hb[q] = 0.5 * W;
      } else {
        double r2 = 0.0;
        for (int c = 0; c < d; ++c) {
          const double u = (xn[(size_t)i * d + c] - xn[(size_t)k * d + c]) / theta[c];
          r2 += u * u;
        }
        hb[q] = 0.5 * W * kernel_f64(family, r2);
        g[q] = 0.5 * W * B[task[i] * T + task[k]] * dkernel_f64(family, r2);
      }
    }
  }
  double* out = partial + (size_t)blockIdx.x * np;
  for (int c = 0; c < d; ++c) {
    const double il = 1.0 / theta[c];
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const double dl = xn[(size_t)pi[q] * d + c] - xn[(size_t)pk[q] * d + c];
      s += g[q] * dl * dl;
    }
    const double tot = block_sum_256(-2.0 * s * il * il * il, red);  // d r2 / d l_c = -2 delta^2 / l_c^3
    if (threadIdx.x == 0) out[c] = tot;
  }
  {
    const double tot = block_sum_256(gn, red);
    if (threadIdx.x == 0) {
      out[d] = tot;
      out[d + 1] = 0.0;
    }
  }
  for (int ab = 0; ab < T * T; ++ab) {
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (hb[q] != 0.0 && task[pi[q]] * T + task[pk[q]] == ab) s += hb[q];
    const double tot = block_sum_256(s, red);
    if (threadIdx.x == 0) out[d + 2 + ab] = tot;
  }
}

__global__ void k_fit_final(const double* __restrict__ partial, int nblk, int np, const double* __restrict__ resid,
                            const double* __restrict__ alpha, const double* __restrict__ Linv, int n, int d,
                            double* __restrict__ out) {
  __shared__ double red[256];
  for (int p = threadIdx.x; p < np; p += blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += partial[(size_t)b * np + p];
    out[1 + p] = s;
  }
  double quad = 0.0, logd = 0.0, sa = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    quad += resid[i] * alpha[i];
    logd += log(Linv[(size_t)i * n + i]);  // = -log L_ii
    sa += alpha[i];
  }
  quad = block_sum_256(quad, red);
  logd = block_sum_256(logd, red);
  sa = block_sum_256(sa, red);
  __syncthreads();
  if (threadIdx.x == 0) {
    out[0] = -0.5 * quad + logd - 0.5 * n * 1.8378770664093453;
    out[1 + d + 1] = sa;
  }
}

// ---- leave-one-out pseudo-likelihood (gpytorch LeaveOneOutPseudoLikelihood; the reference's criterion for
// transfer-learning search spaces, presets/baybe.py:270-281, components/fit_criterion.py:22-41) ----
//   kappa_i = [K^-1]_ii,  sigma_i^2 = 1/kappa_i,  y_i - mu_i = alpha_i / kappa_i
//   F = sum_i ( 1/2 log kappa_i - 1/2 alpha_i^2 / kappa_i ) - n/2 log 2 pi
//   dF = 1/2 sum_ab W_ab dK_ab,  W = -2 K^-1 diag(w) K^-1 + v alpha^T + alpha v^T,
//        w_i = 1/(2 kappa_i) + alpha_i^2 / (2 kappa_i^2),  u_i = alpha_i / kappa_i,  v = K^-1 u;   dF/dc = sum_i v_i
__global__ void k_loo_prep(const double* __restrict__ Kinv, const double* __restrict__ alpha, int n,
                           double* __restrict__ vec) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double kap = Kinv[(size_t)i * n + i], a = alpha[i];
    vec[i] = kap;
    vec[n + i] = 0.5 / kap + 0.5 * a * a / (kap * kap);
    vec[2 * n + i] = a / kap;
  }
}
__global__ void k_loo_v(const double* __restrict__ Kinv, int n, double* __restrict__ vec) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int m = 0; m < n; ++m) s += Kinv[(size_t)i * n + m] * vec[2 * n + m];
    vec[3 * n + i] = s;
  }
}
__global__ void k_loo_wmat(const double* __restrict__ Kinv, const double* __restrict__ alpha,
                           const double* __restrict__ vec, int n, double* __restrict__ wmat) {
  const int i = blockIdx.y * blockDim.y + threadIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || k >= n) return;
  double s = 0.0;
  for (int m = 0; m < n; ++m) s += Kinv[(size_t)i * n + m] * vec[n + m] * Kinv[(size_t)m * n + k];
  wmat[(size_t)i * n + k] = -2.0 * s + vec[3 * n + i] * alpha[k] + alpha[i] * vec[3 * n + k];
}
__global__ void k_fit_final_loo(const double* __restrict__ partial, int nblk, int np, const double* __restrict__ alpha,
                                const double* __restrict__ vec, int n, int d, double* __restrict__ out) {
  __shared__ double red[256];
  for (int p = threadIdx.x; p < np; p += blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += partial[(size_t)b * np + p];
    out[1 + p] = s;
  }
  double f = 0.0, sv = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double kap = vec[i], a = alpha[i];
    f += 0.5 * log(kap) - 0.5 * a * a / kap;
    sv += vec[3 * n + i];
  }
  f = block_sum_256(f, red);
  sv = block_sum_256(sv, red);
  __syncthreads();
  if (threadIdx.x == 0) {
    out[0] = f - 0.5 * n * 1.8378770664093453;
    out[1 + d + 1] = sv;
  }
}

}  // namespace

extern "C" size_t bb_fit_workspace_bytes(int32_t n, int32_t d, int32_t n_tasks) {
  if (n <= 0 || d <= 0 || n_tasks <= 0) return 0;
  return fit_layout(n, d, n_tasks).total;
}

extern "C" int bb_fit_setup(void* d_ws, size_t ws_bytes, int32_t n, int32_t d, int32_t n_tasks,
                            const double* xn, const double* y, const int32_t* task, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  BB_CHECK_ARG(d_ws && xn && y, "bb_fit_setup: null argument");
  BB_CHECK_ARG(n >= 1 && d >= 1 && n_tasks >= 1, "bb_fit_setup: n, d, n_tasks must be positive");
  BB_CHECK_SUPPORTED(n <= BB_MAX_TRAIN, "bb_fit_setup: n=%d exceeds this build's limit of %d", n, BB_MAX_TRAIN);
  BB_CHECK_SUPPORTED(n_tasks <= 16, "bb_fit_setup: at most 16 tasks supported");
  BB_CHECK_ARG(n_tasks == 1 || task != nullptr, "bb_fit_setup: task ids missing");
  const FitLayout L = fit_layout(n, d, n_tasks);
  if (ws_bytes < L.total) {
    set_error("bb_fit_setup: workspace of %zu bytes is smaller than the required %zu", ws_bytes, L.total);
    return BB_ERR_WORKSPACE;
  }
  uint8_t* W = (uint8_t*)d_ws;
  BB_CUDA(cudaMemsetAsync(W, 0, L.total, stream));
  BB_CUDA(cudaMemcpyAsync(W + L.xn, xn, sizeof(double) * (size_t)n * d, cudaMemcpyHostToDevice, stream));
  BB_CUDA(cudaMemcpyAsync(W + L.y, y, sizeof(double) * n, cudaMemcpyHostToDevice, stream));
  if (task) {
    for (int i = 0; i < n; ++i)
      BB_CHECK_ARG(task[i] >= 0 && task[i] < n_tasks, "bb_fit_setup: task id %d outside [0,%d)", task[i], n_tasks);
    BB_CUDA(cudaMemcpyAsync(W + L.task, task, sizeof(int32_t) * n, cudaMemcpyHostToDevice, stream));
  }
  BB_CUDA(cudaStreamSynchronize(stream));
  return BB_OK;
}

static int fit_eval_impl(void* d_ws, int32_t n, int32_t d, int32_t n_tasks, int32_t family, const double* theta,
                         double* value, double* grad, int32_t* not_pd, void* stream_, bool loo) {
  cudaStream_t stream = (cudaStream_t)stream_;
  BB_CHECK_ARG(d_ws && theta && value && grad && not_pd, "bb_fit_eval: null argument");
  BB_CHECK_ARG(family >= 0 && family <= 3, "bb_fit_eval: unknown kernel family %d", family);
  const FitLayout L = fit_layout(n, d, n_tasks);
  uint8_t* W = (uint8_t*)d_ws;
  for (int c = 0; c < d; ++c) BB_CHECK_ARG(theta[c] > 0.0, "bb_fit_eval: lengthscale %d is not positive", c);
  BB_CUDA(cudaMemcpyAsync(W + L.theta, theta, sizeof(double) * L.np, cudaMemcpyHostToDevice, stream));
  const double* dtheta = (const double*)(W + L.theta);
  double* dK = (double*)(W + L.K);
  double* dLinv = (double*)(W + L.Linv);
  double* dresid = (double*)(W + L.resid);
  dim3 blk(16, 16), grd((n + 15) / 16, (n + 15) / 16);
  k_fit_gram<<<grd, blk, 0, stream>>>((const double*)(W + L.xn), (const int32_t*)(W + L.task), dtheta,
                                      (const double*)(W + L.y), n, d, n_tasks, family, dK, dresid);
  BB_LAUNCH_CHECK();
  int rc_f = launch_cholesky(dK, n, (int*)(W + L.flag), stream);
  if (rc_f != BB_OK) return rc_f;
  rc_f = launch_tri_inverse(dK, n, dLinv, stream);
  if (rc_f != BB_OK) return rc_f;
  k_alpha<<<1, 1024, 0, stream>>>(dLinv, dresid, n, dresid + n, (double*)(W + L.alpha), (float*)(W + L.alpha32));
  BB_LAUNCH_CHECK();
  k_fit_kinv<<<grd, blk, 0, stream>>>(dLinv, n, (double*)(W + L.Kinv));
  BB_LAUNCH_CHECK();
  const double* wmat = nullptr;
  if (loo) {
    double* vec = (double*)(W + L.loovec);
    k_loo_prep<<<(n + 255) / 256, 256, 0, stream>>>((const double*)(W + L.Kinv), (const double*)(W + L.alpha), n, vec);
    BB_LAUNCH_CHECK();
    k_loo_v<<<(n + 63) / 64, 64, 0, stream>>>((const double*)(W + L.Kinv), n, vec);
    BB_LAUNCH_CHECK();
    k_loo_wmat<<<grd, blk, 0, stream>>>((const double*)(W + L.Kinv), (const double*)(W + L.alpha), vec, n,
                                        (double*)(W + L.wmat));
    BB_LAUNCH_CHECK();
    wmat = (const double*)(W + L.wmat);
  }
  k_fit_grad<<<L.nblk, 256, 0, stream>>>((const double*)(W + L.xn), (const int32_t*)(W + L.task), dtheta,
                                         (const double*)(W + L.alpha), (const double*)(W + L.Kinv), n, d, n_tasks,
                                         family, (double*)(W + L.partial), wmat);
  BB_LAUNCH_CHECK();
  if (loo)
    k_fit_final_loo<<<1, 256, 0, stream>>>((const double*)(W + L.partial), L.nblk, L.np, (const double*)(W + L.alpha),
                                           (const double*)(W + L.loovec), n, d, (double*)(W + L.out));
  else
    k_fit_final<<<1, 256, 0, stream>>>((const double*)(W + L.partial), L.nblk, L.np, dresid,
                                       (const double*)(W + L.alpha), dLinv, n, d, (double*)(W + L.out));
  BB_LAUNCH_CHECK();
  std::vector<double> out(L.np + 1);
  int flag = 0;
  BB_CUDA(cudaMemcpyAsync(out.data(), W + L.out, sizeof(double) * (L.np + 1), cudaMemcpyDeviceToHost, stream));
  BB_CUDA(cudaMemcpyAsync(&flag, W + L.flag, sizeof(int), cudaMemcpyDeviceToHost, stream));
  BB_CUDA(cudaStreamSynchronize(stream));
  *not_pd = flag;
  *value = out[0];
  for (int p = 0; p < L.np; ++p) grad[p] = out[1 + p];
  return BB_OK;
}

// value[0] = mll, grad[np] = d mll / d theta (np = d + 2 + T*T); *not_pd != 0 when K is not positive
// definite at this theta (value/grad are then unspecified).  Synchronises the stream.
extern "C" int bb_fit_eval(void* d_ws, int32_t n, int32_t d, int32_t n_tasks, int32_t family,
                           const double* theta, double* value, double* grad, int32_t* not_pd, void* stream) {
  return fit_eval_impl(d_ws, n, d, n_tasks, family, theta, value, grad, not_pd, stream, false);
}

// Same contract for the leave-one-out pseudo-likelihood (the reference's fit criterion when the search space has
// a task parameter: presets/baybe.py:270-281 -> gpytorch.mlls.LeaveOneOutPseudoLikelihood).
extern "C" int bb_fit_eval_loo(void* d_ws, int32_t n, int32_t d, int32_t n_tasks, int32_t family,
                               const double* theta, double* value, double* grad, int32_t* not_pd, void* stream) {
  return fit_eval_impl(d_ws, n, d, n_tasks, family, theta, value, grad, not_pd, stream, true);
}
