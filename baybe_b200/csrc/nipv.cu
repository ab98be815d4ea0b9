// nipv.cu -- integrated posterior variance reduction (qNIPV) of every candidate of a discrete space over a fixed set of
// integration points, with the pair products on warpgroup MMAs.
//
// Reference: qNegIntegratedPosteriorVariance (/root/reference/baybe/acquisition/acqfs.py:28-138); set-up on the host
// by baybe_b200/nipv.py.  With C the conditioning set (pending points and the other points of a q-batch, observed with
// noise) and k_D the posterior covariance given the training data,
//   k_C(a,b) = k(a,b) - phi(a) . phi(b),   phi(a) = [ L^-1 k(X,a) ; L_C^-1 k_D(C,a) ]   (standardised units)
//   IVR(x)   = sum_m k_C(m,x)^2 / (k_C(x,x) + sigma_n^2(x))
// and qNIPV(x | C) = -(1/M) [ sum_m k_C(m,m) - IVR(x) ]; the host adds the candidate-independent sum.
//
// Two kernels per block of rows:
//   k_nipv_phi    phi of 64 rows per CTA on the CUDA cores (fp32, the form of k_simt), multiplied by a power of two
//                 and written as fp16 hi/lo 128B-swizzled K-major tiles of 64 columns (r_pad = n + |C| rounded up to
//                 64), plus the rows' scaled coordinates (dimension-major), task ids and, for candidates,
//                 1 / (k_C(x,x) + sigma_n^2(x)).
//   k_nipv_pairs  one CTA per 128 candidates, two warpgroups of 64 rows.  The candidates' phi tiles stay in shared
//                 memory; the integration points' tiles stream through a ring of four 64-column chunks (bulk copies,
//                 one mbarrier per slot).  Per 64 integration points a warpgroup accumulates phi_x . phi_m with three
//                 m64n64k16 MMAs per k16 step (hi.hi + hi.lo + lo.hi, fp32), then keeps in registers the direct
//                 d-deep distance (CUDA cores), the kernel value, the task factor, the subtraction and the square,
//                 summed per row.  The four lanes of a row join by a fixed xor tree; each row has one owner, which adds
//                 the block's sum to the previous blocks' in block order.  No float atomics: the output is
//                 bit-identical from run to run.
#include <math.h>

#include <algorithm>

#include "fused_common.cuh"
#include "score_common.cuh"

namespace bb {

constexpr int kNipvMaxTrain = 256;
constexpr int kNipvThreads = 256;
constexpr uint32_t kNipvChunkBytes = 16384;  // 64 rows x 64 columns, [hi 8 KB | lo 8 KB]
constexpr int kNipvRing = 4;
constexpr int kNipvRowAlign = 128;

struct NipvPhiParams {
  const float* x;  // [rows][d] raw comp-rep, row-major
  int64_t rows, ld_out;  // valid rows; allocated rows of the block (coords / task / inv_den stride)
  const float *cand_scale, *cand_shift, *train_m2, *task_covar, *linv32;
  const int32_t* train_task;
  int n, n_pad, d, d_pad, task_col, n_tasks, scaled, C, r_pad, n_kc;
  const float* cross;  // [rows][C] original units (nullable when C = 0)
  const float* linv_c; // [C][C]
  const float* var;    // [rows] original units (candidates; null for integration points)
  float inv_y_std, inv_y_var, sphi;
  float noise[kMaxTasks];
  uint8_t* img;
  float* coords;
  int32_t* task;
  float* inv_den;
};

__host__ __device__ inline size_t nipv_phi_smem(int d_pad, int n_pad, int r_pad) {
  return sizeof(float) * ((size_t)64 * d_pad + (size_t)64 * (n_pad + 1) + (size_t)64 * (r_pad + 1)) + 64 * 4;
}

template <int FAMILY>
__global__ void __launch_bounds__(kNipvThreads) k_nipv_phi(const NipvPhiParams p) {
  extern __shared__ __align__(16) float smem_phi[];
  float* xa = smem_phi;                         // [64][d_pad]
  float* ks = xa + 64 * p.d_pad;                // [64][n_pad + 1]
  float* ph = ks + 64 * (p.n_pad + 1);          // [64][r_pad + 1]
  int* ct = reinterpret_cast<int*>(ph + 64 * (p.r_pad + 1));  // [64]
  const int tid = threadIdx.x;
  const int64_t row0 = (int64_t)blockIdx.x * 64;
  if (tid < 64) ct[tid] = 0;
  __syncthreads();
  for (int e = tid; e < 64 * p.d_pad; e += kNipvThreads) {
    const int r = e / p.d_pad, j = e - r * p.d_pad;
    const int64_t row = row0 + r;
    const float xv = (j < p.d && row < p.rows) ? __ldg(p.x + row * p.d + j) : 0.f;
    const float a = (j < p.d) ? fmaf(xv, __ldg(p.cand_scale + j), __ldg(p.cand_shift + j)) : 0.f;
    xa[e] = a;
    if (j < p.d) p.coords[(int64_t)j * p.ld_out + row] = a;
    if (j == p.task_col) ct[r] = min(max(__float2int_rn(xv), 0), p.n_tasks - 1);
  }
  __syncthreads();
  if (tid < 64) p.task[row0 + tid] = ct[tid];
  for (int e = tid; e < 64 * p.n_pad; e += kNipvThreads) {
    const int r = e & 63, i = e >> 6;
    float t = 0.f;
    for (int j = 0; j < p.d_pad; ++j) {
      const float diff = xa[r * p.d_pad + j] + 0.5f * __ldg(p.train_m2 + (size_t)i * p.d_pad + j);
      t = fmaf(diff, diff, t);
    }
    float k = (i < p.n) ? kernel_from_t<FAMILY>(t) : 0.f;
    if (p.scaled) k *= __ldg(p.task_covar + ct[r] * p.n_tasks + __ldg(p.train_task + i));
    ks[r * (p.n_pad + 1) + i] = k;
  }
  __syncthreads();
  const int r = tid & 63;
  for (int j = tid >> 6; j < p.n; j += kNipvThreads / 64) {
    float v = 0.f;
    for (int i = 0; i <= j; ++i) v = fmaf(ks[r * (p.n_pad + 1) + i], __ldg(p.linv32 + (size_t)j * p.n_pad + i), v);
    ph[r * (p.r_pad + 1) + j] = v * p.sphi;
  }
  if (tid < 64) {
    const int64_t row = row0 + r;
    const bool valid = row < p.rows;
    float q = 0.f;
    for (int j = 0; j < p.C; ++j) {
      float v = 0.f;
      if (valid)
        for (int i = 0; i <= j; ++i) v = fmaf(__ldg(p.linv_c + j * p.C + i), __ldg(p.cross + row * p.C + i), v);
      v *= p.inv_y_std;
      q = fmaf(v, v, q);
      ph[r * (p.r_pad + 1) + p.n + j] = v * p.sphi;
    }
    for (int j = p.n + p.C; j < p.r_pad; ++j) ph[r * (p.r_pad + 1) + j] = 0.f;
    if (p.inv_den != nullptr) {
      const float kxx = valid ? fmaxf(__ldg(p.var + row) * p.inv_y_var - q, 0.f) : 0.f;
      p.inv_den[row] = 1.0f / (kxx + p.noise[ct[r]]);
    }
  }
  __syncthreads();
  // fp16 hi/lo image: tile blockIdx.x, chunk kc = [hi 8 KB | lo 8 KB], row r at 128 B, 16-byte unit c16 swizzled
  const int units = p.r_pad / 8;
  uint8_t* tile = p.img + (size_t)blockIdx.x * p.n_kc * kNipvChunkBytes;
  for (int e = tid; e < 64 * units; e += kNipvThreads) {
    const int rr = e / units, u = e - rr * units;
    const float* src = ph + rr * (p.r_pad + 1) + u * 8;
    uint4 hi, lo;
    split_pair(src[0], src[1], hi.x, lo.x);
    split_pair(src[2], src[3], hi.y, lo.y);
    split_pair(src[4], src[5], hi.z, lo.z);
    split_pair(src[6], src[7], hi.w, lo.w);
    uint8_t* chunk = tile + (size_t)(u >> 3) * kNipvChunkBytes;
    const uint32_t off = sw128_offset((uint32_t)rr, (uint32_t)(u & 7));
    *reinterpret_cast<uint4*>(chunk + off) = hi;
    *reinterpret_cast<uint4*>(chunk + 8192 + off) = lo;
  }
}

struct NipvPairParams {
  const uint8_t *img_a, *img_b;
  const float *xa, *xb;        // scaled coordinates, [d][lda] / [d][ldb]
  const int32_t *ta, *tb;
  const float* inv_den;        // [lda]
  float* sums;                 // [lda] running sums over the integration blocks
  const float* task_covar;
  int64_t lda, ldb, na, nb;    // allocated / valid rows of the candidate and integration blocks
  int n_kc, d, n_tasks, scaled, first, last;
  float inv_s2, out_scale;
  const uint8_t* keep;
  float* score;
  long long* key;
  int64_t index_offset;
};

__host__ __device__ inline size_t nipv_pair_smem(int n_kc) {
  return (size_t)(2 * n_kc + kNipvRing) * kNipvChunkBytes + 8 * (kNipvRing + 1) + 1024;
}

template <int FAMILY>
__global__ void __launch_bounds__(kNipvThreads, 1) k_nipv_pairs(const NipvPairParams p) {
  extern __shared__ __align__(1024) uint8_t smem_pairs[];
  uint8_t* base = smem_pairs + ((1024u - (smem_u32(smem_pairs) & 1023u)) & 1023u);
  const int n_kc = p.n_kc;
  uint8_t* sa = base;                                      // [2 warpgroups][n_kc] chunks of this CTA's candidates
  uint8_t* ring = sa + (size_t)2 * n_kc * kNipvChunkBytes;  // [kNipvRing] chunks of integration points
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + (size_t)kNipvRing * kNipvChunkBytes);  // ring slots, then A
  const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  const int64_t tile_a = blockIdx.x;
  const int steps = (int)((p.nb + 63) / 64) * n_kc;
  if (tid == 0) {
    for (int i = 0; i <= kNipvRing; ++i) mbar_init(&bars[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    const uint8_t* src = p.img_a + (size_t)tile_a * 2 * n_kc * kNipvChunkBytes;
    mbar_expect_tx(&bars[kNipvRing], 2u * n_kc * kNipvChunkBytes);
    for (int c = 0; c < 2 * n_kc; ++c)
      bulk_g2s(sa + (size_t)c * kNipvChunkBytes, src + (size_t)c * kNipvChunkBytes, kNipvChunkBytes, &bars[kNipvRing]);
    for (int s = 0; s < kNipvRing - 1 && s < steps; ++s) {
      mbar_expect_tx(&bars[s], kNipvChunkBytes);
      bulk_g2s(ring + (size_t)s * kNipvChunkBytes, p.img_b + (size_t)s * kNipvChunkBytes, kNipvChunkBytes, &bars[s]);
    }
  }
  // this thread's accumulator rows (two) and columns (16 per 64-column tile): see wgmma_64x64
  const int64_t row0 = tile_a * 128 + wg * 64 + 16 * warp + (lane >> 2);
  const int t_row0 = __ldg(p.ta + row0), t_row1 = __ldg(p.ta + row0 + 8);
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  float rs0 = 0.f, rs1 = 0.f;
  mbar_wait(&bars[kNipvRing], 0);
  int kc = 0;
  int64_t col_base = 0;
  for (int s = 0; s < steps; ++s) {
    const int slot = s & (kNipvRing - 1);
    if (s > 0) __syncthreads();  // every warpgroup has finished step s - 1: its slot may be refilled
    if (tid == 0 && s + kNipvRing - 1 < steps) {
      const int ns = (s + kNipvRing - 1) & (kNipvRing - 1);
      mbar_expect_tx(&bars[ns], kNipvChunkBytes);
      bulk_g2s(ring + (size_t)ns * kNipvChunkBytes, p.img_b + (size_t)(s + kNipvRing - 1) * kNipvChunkBytes,
               kNipvChunkBytes, &bars[ns]);
    }
    mbar_wait(&bars[slot], (uint32_t)(s / kNipvRing) & 1u);
    const uint32_t a_hi = smem_u32(sa + (size_t)(wg * n_kc + kc) * kNipvChunkBytes), a_lo = a_hi + 8192;
    const uint32_t b_hi = smem_u32(ring + (size_t)slot * kNipvChunkBytes), b_lo = b_hi + 8192;
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      wgmma_64x64(acc, make_wg_desc<64>(a_hi + 32 * kk), make_wg_desc<64>(b_hi + 32 * kk));
      wgmma_64x64(acc, make_wg_desc<64>(a_hi + 32 * kk), make_wg_desc<64>(b_lo + 32 * kk));
      wgmma_64x64(acc, make_wg_desc<64>(a_lo + 32 * kk), make_wg_desc<64>(b_hi + 32 * kk));
    }
    wg_commit();
    wg_wait<0>();
    if (++kc < n_kc) continue;
    // one 64-column tile of phi_x . phi_m is complete: k_C = k * task - acc / sphi^2, summed squared per row
    kc = 0;
    float t[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) t[i] = 0.f;
    const int c0 = 2 * (lane & 3);
    for (int k = 0; k < p.d; ++k) {
      const float a0 = __ldg(p.xa + (int64_t)k * p.lda + row0), a1 = __ldg(p.xa + (int64_t)k * p.lda + row0 + 8);
      const float* bk = p.xb + (int64_t)k * p.ldb + col_base + c0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(bk + 8 * j));
        float u;
        u = a0 - b.x; t[4 * j + 0] = fmaf(u, u, t[4 * j + 0]);
        u = a0 - b.y; t[4 * j + 1] = fmaf(u, u, t[4 * j + 1]);
        u = a1 - b.x; t[4 * j + 2] = fmaf(u, u, t[4 * j + 2]);
        u = a1 - b.y; t[4 * j + 3] = fmaf(u, u, t[4 * j + 3]);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int64_t col = col_base + 8 * j + c0 + e;
        if (col >= p.nb) continue;
        float f0 = 1.f, f1 = 1.f;
        if (p.scaled) {
          const int tc = __ldg(p.tb + col);
          f0 = __ldg(p.task_covar + t_row0 * p.n_tasks + tc);
          f1 = __ldg(p.task_covar + t_row1 * p.n_tasks + tc);
        }
        const float k0 = fmaf(-acc[4 * j + e], p.inv_s2, kernel_from_t<FAMILY>(t[4 * j + e]) * f0);
        const float k1 = fmaf(-acc[4 * j + 2 + e], p.inv_s2, kernel_from_t<FAMILY>(t[4 * j + 2 + e]) * f1);
        rs0 = fmaf(k0, k0, rs0);
        rs1 = fmaf(k1, k1, rs1);
      }
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    col_base += 64;
  }
  rs0 += __shfl_xor_sync(0xffffffffu, rs0, 1);
  rs1 += __shfl_xor_sync(0xffffffffu, rs1, 1);
  rs0 += __shfl_xor_sync(0xffffffffu, rs0, 2);
  rs1 += __shfl_xor_sync(0xffffffffu, rs1, 2);
  long long best = kEmptyKey;
  if ((lane & 3) == 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t row = row0 + 8 * h;
      if (row >= p.na) continue;
      const float sum = (p.first ? 0.f : p.sums[row]) + (h ? rs1 : rs0);
      if (!p.last) {
        p.sums[row] = sum;
        continue;
      }
      const float v = sum * __ldg(p.inv_den + row) * p.out_scale;
      if (p.score) p.score[row] = v;
      if ((p.keep == nullptr || p.keep[row] != 0) && !(v != v)) {
        const long long k = pack_key(v, (uint32_t)(row + p.index_offset));
        best = k > best ? k : best;
      }
    }
  }
  if (!p.last) return;
  for (int o = 16; o > 0; o >>= 1) {
    const long long other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other > best ? other : best;
  }
  block_flush_best<kNipvThreads>(best, p.key);
}

// power of two that puts max |phi| = sqrt(prior_var) near 2^10: fp16 hi/lo keep 22 bits of the large entries and the
// small ones stay above the fp16 subnormal range
static float nipv_phi_scale(float prior_var) {
  int e = 0;
  frexpf(1024.0f / sqrtf(prior_var), &e);
  return ldexpf(1.0f, e - 1);
}

template <int FAMILY>
static int nipv_run(const bb_model* m, const float* noise, float prior_var, const float* d_x, int64_t N,
                    const float* d_xm, int64_t M, const float* d_var, int32_t C, const float* d_cross_x,
                    const float* d_cross_m, const float* d_linv, const uint8_t* d_keep, float* d_score,
                    int64_t* d_best_key, int64_t index_offset, void* d_ws, size_t ws_bytes, cudaStream_t st) {
  const int r_pad = round_up(m->n + C, 64), n_kc = r_pad / 64;
  const size_t row_bytes = (size_t)4 * r_pad + (size_t)4 * m->d + 12;
  const int64_t rows_fit = (int64_t)(ws_bytes / row_bytes);
  const int64_t na_all = (N + kNipvRowAlign - 1) / kNipvRowAlign * kNipvRowAlign;
  const int64_t mb_all = (M + kNipvRowAlign - 1) / kNipvRowAlign * kNipvRowAlign;
  int64_t lda = na_all, ldb = mb_all;
  if (lda + ldb > rows_fit) {
    lda = std::min(na_all, std::max<int64_t>(kNipvRowAlign, rows_fit / 2 / kNipvRowAlign * kNipvRowAlign));
    ldb = std::min(mb_all, (rows_fit - lda) / kNipvRowAlign * kNipvRowAlign);
  }
  // carve: images first (16 KB chunks), then floats
  uint8_t* w = static_cast<uint8_t*>(d_ws);
  uint8_t* img_a = w;
  uint8_t* img_b = img_a + (size_t)lda * r_pad * 4;
  float* xa = reinterpret_cast<float*>(img_b + (size_t)ldb * r_pad * 4);
  float* xb = xa + (size_t)lda * m->d;
  int32_t* ta = reinterpret_cast<int32_t*>(xb + (size_t)ldb * m->d);
  int32_t* tb = ta + lda;
  float* inv_den = reinterpret_cast<float*>(tb + ldb);
  float* sums = inv_den + lda;

  NipvPhiParams ph{};
  ph.cand_scale = m->d_cand_scale;
  ph.cand_shift = m->d_cand_shift;
  ph.train_m2 = m->d_train_m2;
  ph.task_covar = m->d_task_covar;
  ph.linv32 = m->d_linv32;
  ph.train_task = m->d_train_task;
  ph.n = m->n;
  ph.n_pad = m->n_pad;
  ph.d = m->d;
  ph.d_pad = m->d_pad;
  ph.task_col = m->task_col;
  ph.n_tasks = m->n_tasks;
  ph.scaled = model_scaled(m) ? 1 : 0;
  ph.C = C;
  ph.r_pad = r_pad;
  ph.n_kc = n_kc;
  ph.linv_c = d_linv;
  ph.inv_y_std = 1.0f / m->y_std;
  ph.inv_y_var = 1.0f / (m->y_std * m->y_std);
  const float sphi = nipv_phi_scale(prior_var);
  ph.sphi = sphi;
  for (int t = 0; t < m->n_tasks; ++t) ph.noise[t] = noise[t] < 1e-4f ? 1e-4f : noise[t];  // MIN_INFERRED_NOISE_LEVEL

  NipvPairParams pp{};
  pp.img_a = img_a;
  pp.img_b = img_b;
  pp.xa = xa;
  pp.xb = xb;
  pp.ta = ta;
  pp.tb = tb;
  pp.inv_den = inv_den;
  pp.sums = sums;
  pp.task_covar = m->d_task_covar;
  pp.lda = lda;
  pp.ldb = ldb;
  pp.n_kc = n_kc;
  pp.d = m->d;
  pp.n_tasks = m->n_tasks;
  pp.scaled = ph.scaled;
  pp.inv_s2 = 1.0f / (sphi * sphi);
  pp.out_scale = m->y_std * m->y_std;
  pp.key = reinterpret_cast<long long*>(d_best_key);

  const size_t phi_smem = nipv_phi_smem(m->d_pad, m->n_pad, r_pad);
  const size_t pair_smem = nipv_pair_smem(n_kc);
  BB_SMEM_OPTIN_ONCE(k_nipv_phi<FAMILY>);
  BB_SMEM_OPTIN_ONCE(k_nipv_pairs<FAMILY>);
  auto phi = [&](const float* x, int64_t rows, int64_t ld, const float* cross, const float* var, uint8_t* img,
                 float* coords, int32_t* task, float* den) {
    ph.x = x;
    ph.rows = rows;
    ph.ld_out = ld;
    ph.cross = cross;
    ph.var = var;
    ph.img = img;
    ph.coords = coords;
    ph.task = task;
    ph.inv_den = den;
    const int64_t tiles = (rows + kNipvRowAlign - 1) / kNipvRowAlign * (kNipvRowAlign / 64);
    k_nipv_phi<FAMILY><<<(unsigned)tiles, kNipvThreads, phi_smem, st>>>(ph);
    BB_LAUNCH_CHECK();
    return BB_OK;
  };
  for (int64_t c0 = 0; c0 < N; c0 += lda) {
    const int64_t na = std::min(lda, N - c0);
    int rc = phi(d_x + c0 * m->d, na, lda, C ? d_cross_x + c0 * C : nullptr, d_var + c0, img_a, xa, ta, inv_den);
    if (rc != BB_OK) return rc;
    for (int64_t m0 = 0; m0 < M; m0 += ldb) {
      const int64_t nb = std::min(ldb, M - m0);
      if (c0 == 0 || ldb < M) {  // one integration block: its tiles serve every candidate block
        rc = phi(d_xm + m0 * m->d, nb, ldb, C ? d_cross_m + m0 * C : nullptr, nullptr, img_b, xb, tb, nullptr);
        if (rc != BB_OK) return rc;
      }
      pp.na = na;
      pp.nb = nb;
      pp.first = m0 == 0;
      pp.last = m0 + ldb >= M;
      pp.keep = d_keep ? d_keep + c0 : nullptr;
      pp.score = d_score ? d_score + c0 : nullptr;
      pp.index_offset = index_offset + c0;
      k_nipv_pairs<FAMILY><<<(unsigned)((na + 127) / 128), kNipvThreads, pair_smem, st>>>(pp);
      BB_LAUNCH_CHECK();
    }
  }
  return BB_OK;
}

}  // namespace bb

using namespace bb;

extern "C" int bb_nipv_score(const bb_model* m, const float* noise, float prior_var, const float* d_x, int64_t N,
                             const float* d_xm, int64_t M, const float* d_var, int32_t n_cond, const float* d_cross_x,
                             const float* d_cross_m, const float* d_linv, const uint8_t* d_keep, float* d_score,
                             int64_t* d_best_key, int64_t index_offset, void* d_ws, size_t ws_bytes, void* stream) {
  int rc = check_candidates(m, d_x, BB_ROW_MAJOR_F32, N, m ? m->d : 0);
  if (rc != BB_OK) return rc;
  BB_CHECK_SUPPORTED(!m->wide, "bb_nipv_score: wide-feature models are not supported (n_pad*d_pad*4 > 56 KB)");
  BB_CHECK_SUPPORTED(m->n <= kNipvMaxTrain, "bb_nipv_score: n=%d training points, at most %d supported", m->n,
                     kNipvMaxTrain);
  rc = check_score_args("bb_nipv_score", "n_cond", N, index_offset, n_cond, 1, false, d_best_key);
  if (rc != BB_OK) return rc;
  BB_CHECK_ARG(M >= 1 && M < 0x7fffffffLL, "bb_nipv_score: M=%lld integration points outside [1,2^31)", (long long)M);
  BB_CHECK_ARG(noise != nullptr, "bb_nipv_score: null noise");
  for (int t = 0; t < m->n_tasks; ++t)
    BB_CHECK_ARG(isfinite(noise[t]) && noise[t] >= 0.f, "bb_nipv_score: noise[%d] not finite and >= 0", t);
  BB_CHECK_ARG(isfinite(prior_var) && prior_var > 0.f, "bb_nipv_score: prior_var must be finite and > 0");
  if (N == 0) return BB_OK;
  BB_CHECK_ARG(d_xm && d_var && d_ws, "bb_nipv_score: null buffer");
  BB_CHECK_ARG(n_cond == 0 || (d_cross_x && d_cross_m && d_linv),
               "bb_nipv_score: conditioning points need both cross covariances and linv");
  const int r_pad = round_up(m->n + n_cond, 64);
  const size_t need = (size_t)2 * kNipvRowAlign * ((size_t)4 * r_pad + (size_t)4 * m->d + 12);
  if (ws_bytes < need) {
    set_error("bb_nipv_score: workspace of %zu bytes, need at least %zu", ws_bytes, need);
    return BB_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_family<true>(m->family, [&](auto fam) {
    return nipv_run<decltype(fam)::value>(m, noise, prior_var, d_x, N, d_xm, M, d_var, n_cond, d_cross_x, d_cross_m,
                                         d_linv, d_keep, d_score, d_best_key, index_offset, d_ws, ws_bytes, st);
  });
}
