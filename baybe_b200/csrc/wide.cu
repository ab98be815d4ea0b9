// wide.cu -- K(X*, X) for WIDE feature spaces (d in the hundreds or thousands: substance fingerprints,
// BASELINE config 4) on the tensor cores, and the two-stage scoring path built on it.
//
//   stage 1  k_kmat_wg   t[m][i] = |a_m|^2 + |b_i|^2 - 2 a_m.b_i  with the inner product as a
//                        K-looped warpgroup-MMA GEMM (fp16 split operands, fp32 accumulators in
//                        registers), Matern/RBF epilogue, K* block -> workspace sized to stay in L2 up to n_pad = 576 (or the
//                        caller's matrix for bb_kernel_matrix)
//   stage 2  k_fused<PRE> (fused.cu) posterior GEMM + acquisition + arg-max reading that K* block
//
// Candidate layouts: the four float layouts (operand split hi/mid/lo, six products, error 2^-33)
// and BB_BITS_U8 -- bit-packed binary fingerprints.  For bits x in {0,1}^d the whole scaled squared
// distance is LINEAR in x:  t = sum_j x_j W_ij + c_i,  W_ij = s_j (-2 b_ij + s_j + 2 h_j),
// c_i = |b_i|^2 + sum_j h_j (-2 b_ij + h_j)   (a_j = s_j x_j + h_j), so the A operand is the exact
// 0/1 matrix (one fp16 panel, no split) and only W is split (hi/mid: W takes at most two distinct
// values per column, 2^-22 relative is ample): two products.
//
// Work item = 128 candidates x <= 128 training columns: each consumer warpgroup stages its 64 candidate
// rows and holds a 64 x 128 fp32 accumulator (64 registers per thread); both share every B slice.  Warp
// roles as in fused.cu.
//
// Reference path replaced: gpytorch Kernel.forward over the comp-rep of a SubstanceParameter space
// (baybe/kernels/base.py, parameters/substance.py comp_df), reached from SingleTaskGP.posterior
// (surrogates/gaussian_process/core.py).
#include "fused_common.cuh"

namespace bb {

constexpr int kWTileM = 128;   // candidates per work item
constexpr int kWHalfN = 256;   // training columns per block of the B image
constexpr int kWItemN = 128;   // training columns per work item
constexpr int kWK = 32;        // fp16 per K stage: 64-byte rows, SWIZZLE_64B
constexpr uint32_t kWPanelA = kWTileM * kWK * 2;  // 8 KB: 128 rows x 64 B; a stage holds [hi | mid | lo] (floats) or [0/1] (bits)
constexpr uint32_t kWPanelB = kWItemN * kWK * 2;  // 8 KB: 128 rows x 64 B; a stage holds [hi | mid | lo] (floats) or [hi | mid] (bits)

struct WideParams {
  const void* x;
  int layout;
  int64_t N, ldx;
  int d, n, n_pad, n_halves, n_kc;
  const float *cand_scale, *cand_shift;  // [d]
  const uint8_t* wimg;                   // B image: per (256-column block, K stage) [hi|mid|lo] swizzled panels
  const float* wnorm;                    // [n_pad] additive per-training-row term (|b|^2 or c_i)
  float a_scale, inv_scale;
  const int32_t* train_task;
  const float* task_covar;
  int task_col, n_tasks, scaled;
  float* out;
  int64_t ldk, out_rows;
  int out_cols, vec_ok, bits_vec;
  int num_items, stages;
};

struct WideSmem {
  uint8_t* ring;
  float *wnorm_s, *tcov;
  double* an_part;  // [2 K halves][128 rows], float64: |a|^2 sums d terms
  int32_t* ttask;
  uint64_t *full, *empty;
};

template <bool BITS>
__host__ __device__ inline size_t wide_carve(uint8_t* base, const WideParams& p, WideSmem& s) {
  constexpr uint32_t kStage = (BITS ? 1 : 3) * kWPanelA + (BITS ? 2 : 3) * kWPanelB;
  SmemCarver c{base};
  s.ring = c.take<uint8_t>((size_t)p.stages * kStage, 1024);  // swizzled panels
  s.wnorm_s = c.take<float>((size_t)p.n_pad * 4);
  s.ttask = c.take<int32_t>((size_t)p.n_pad * 4);
  s.an_part = c.take<double>(2 * kWTileM * 8);
  s.tcov = c.take<float>(kMaxTasks * kMaxTasks * 4);
  s.full = c.take<uint64_t>(16 * 8);  // [<=4]
  s.empty = s.full + 4;               // [<=4]
  return c.bytes;
}

// 16 consecutive features k0..k0+15 of one candidate row as fp32 (0 beyond d / beyond N).
__device__ __forceinline__ void wide_load16(const WideParams& p, int64_t row, int k0, float (&v)[16]) {
#pragma unroll
  for (int e = 0; e < 16; ++e) v[e] = 0.f;
  if (row >= p.N || k0 >= p.d) return;
  switch (p.layout) {
    case BB_ROW_MAJOR_F32: {
      const float* ptr = reinterpret_cast<const float*>(p.x) + row * p.ldx + k0;
      if (k0 + 16 <= p.d && (reinterpret_cast<uintptr_t>(ptr) & 15) == 0) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 f = __ldg(reinterpret_cast<const float4*>(ptr) + q);
          v[4 * q] = f.x;
          v[4 * q + 1] = f.y;
          v[4 * q + 2] = f.z;
          v[4 * q + 3] = f.w;
        }
      } else {
#pragma unroll
        for (int e = 0; e < 16; ++e)
          if (k0 + e < p.d) v[e] = __ldg(ptr + e);
      }
      return;
    }
    case BB_COL_MAJOR_F32:
#pragma unroll
      for (int e = 0; e < 16; ++e)
        if (k0 + e < p.d) v[e] = load_x<BB_COL_MAJOR_F32>(p.x, row, k0 + e, p.ldx);
      return;
    case BB_ROW_MAJOR_F64:
#pragma unroll
      for (int e = 0; e < 16; ++e)
        if (k0 + e < p.d) v[e] = load_x<BB_ROW_MAJOR_F64>(p.x, row, k0 + e, p.ldx);
      return;
    default:
#pragma unroll
      for (int e = 0; e < 16; ++e)
        if (k0 + e < p.d) v[e] = load_x<BB_COL_MAJOR_F64>(p.x, row, k0 + e, p.ldx);
      return;
  }
}

// 16 feature bits k0..k0+15 (k0 a multiple of 16) of one bit-packed candidate row.
__device__ __forceinline__ uint32_t wide_load_bits16(const WideParams& p, int64_t row, int k0) {
  if (row >= p.N || k0 >= p.d) return 0u;
  const uint8_t* ptr = reinterpret_cast<const uint8_t*>(p.x) + row * p.ldx + (k0 >> 3);
  uint32_t b = __ldg(ptr);
  if (k0 + 8 < p.d) b |= (uint32_t)__ldg(ptr + 1) << 8;
  const int valid = p.d - k0;  // bits beyond d are padding of the last byte
  if (valid < 16) b &= (1u << valid) - 1u;
  return b;
}

template <int FAMILY, bool BITS>
__global__ void __launch_bounds__(kWideThreads, 1) k_kmat_wg(const WideParams p) {
  constexpr int PA = BITS ? 1 : 3;
  constexpr int PB = BITS ? 2 : 3;  // W of the bit-linear form has <= 2 distinct values per column: hi+mid (2^-22) suffices
  constexpr uint32_t kStageA = PA * kWPanelA;
  constexpr uint32_t kStage = kStageA + PB * kWPanelB;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  WideSmem s;
  wide_carve<BITS>(smem_raw, p, s);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0 && (smem_u32(smem_raw) & 1023u) != 0u) __trap();

  if (tid == 0) {
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&s.full[i], kConsumerThreads / 32 + 1);  // 8 staging warps + the producer's expect_tx
      mbar_init(&s.empty[i], kConsumerWGs);
    }
    fence_mbar_init();
  }
  for (int e = tid; e < p.n_pad; e += kWideThreads) {
    s.wnorm_s[e] = __ldg(p.wnorm + e);
    s.ttask[e] = __ldg(p.train_task + e);
  }
  for (int e = tid; e < p.n_tasks * p.n_tasks; e += kWideThreads) s.tcov[e] = __ldg(p.task_covar + e);
  __syncthreads();

  if (warp < kWarpProducer) {
    // =====================================================================================
    // consumer warpgroups: stage the A operand (candidate rows -> fp16 panels), issue the MMAs of each
    // K stage (the next stage is staged while they run), then the epilogue from the accumulators
    // =====================================================================================
    const int wg = warp >> 2, t = tid & 127;
    const int r = 64 * wg + (t & 63), kh = t >> 6;  // staging: row of the item, 16-feature half of the stage
    const int ra = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // accumulator rows ra, ra + 8
    uint32_t st = 0, ph = 0;
    for (int item = blockIdx.x; item < p.num_items; item += gridDim.x) {
      const int tile = item / p.n_halves, half = item - tile * p.n_halves;
      const int64_t row0 = (int64_t)tile * kWTileM;
      const int64_t row = row0 + r;
      const int ncols = min(kWItemN, p.n_pad - half * kWItemN);
      float acc[2][32];
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
      double an = 0.0;
      float cur[16];
      uint32_t curb = 0;
      // bit rows 16-byte aligned: one 128-bit load covers four K stages and is issued four stages ahead
      uint4 cur4 = make_uint4(0u, 0u, 0u, 0u), nxt4 = cur4;
      const uint4* brow = nullptr;
      if constexpr (BITS) {
        if (p.bits_vec) {
          if (row < p.N) brow = reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.x) + row * p.ldx);
          if (brow != nullptr) {
            cur4 = __ldg(brow);
            if (p.n_kc > 4) nxt4 = __ldg(brow + 1);
          }
        } else {
          curb = wide_load_bits16(p, row, kh * 16);
        }
      }
      else wide_load16(p, row, kh * 16, cur);
      uint32_t st_prev = 0;
      for (int kc = 0; kc < p.n_kc; ++kc) {
        const int k0 = kc * kWK + kh * 16;
        uint4 pk[PA][2];
        if constexpr (BITS) {
          if (p.bits_vec) {
            const int sub = kc & 3;
            const uint32_t word = sub == 0 ? cur4.x : sub == 1 ? cur4.y : sub == 2 ? cur4.z : cur4.w;
            curb = (word >> (kh * 16)) & 0xffffu;
            if (sub == 3) {
              cur4 = nxt4;
              if (brow != nullptr && kc + 5 < p.n_kc) nxt4 = __ldg(brow + ((kc + 5) >> 2));
            }
          }
          uint32_t w[8];
#pragma unroll
          for (int e = 0; e < 8; ++e)
            w[e] = (((curb >> (2 * e)) & 1u) * 0x3C00u) | (((curb >> (2 * e + 1)) & 1u) * 0x3C000000u);
          pk[0][0] = make_uint4(w[0], w[1], w[2], w[3]);
          pk[0][1] = make_uint4(w[4], w[5], w[6], w[7]);
          if (!p.bits_vec && kc + 1 < p.n_kc) curb = wide_load_bits16(p, row, k0 + kWK);
        } else {
          float a[16];
#pragma unroll
          for (int e = 0; e < 16; ++e) {
            const int k = k0 + e;
            const float sc = (k < p.d) ? __ldg(p.cand_scale + k) : 0.f;
            const float sh = (k < p.d) ? __ldg(p.cand_shift + k) : 0.f;
            const float v = fmaf(cur[e], sc, sh);
            an = fma((double)v, (double)v, an);
            a[e] = v * p.a_scale;
          }
          if (kc + 1 < p.n_kc) wide_load16(p, row, k0 + kWK, cur);  // next stage's loads fly under the split
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint2 h0, m0, l0, h1, m1, l1;
            const float q0[4] = {a[8 * h], a[8 * h + 1], a[8 * h + 2], a[8 * h + 3]};
            const float q1[4] = {a[8 * h + 4], a[8 * h + 5], a[8 * h + 6], a[8 * h + 7]};
            split3_quad(q0, h0, m0, l0);
            split3_quad(q1, h1, m1, l1);
            pk[0][h] = make_uint4(h0.x, h0.y, h1.x, h1.y);
            pk[PA > 1 ? 1 : 0][h] = make_uint4(m0.x, m0.y, m1.x, m1.y);
            pk[PA > 2 ? 2 : 0][h] = make_uint4(l0.x, l0.y, l1.x, l1.y);
          }
        }
        mbar_wait(&s.empty[st], ph ^ 1u);  // the MMAs that read this stage last time are done
        uint8_t* sa = s.ring + (size_t)st * kStage;
#pragma unroll
        for (int pa = 0; pa < PA; ++pa) {
          *reinterpret_cast<uint4*>(sa + pa * kWPanelA + swk_offset<kWK>((uint32_t)r, (uint32_t)(kh * 2))) = pk[pa][0];
          *reinterpret_cast<uint4*>(sa + pa * kWPanelA + swk_offset<kWK>((uint32_t)r, (uint32_t)(kh * 2 + 1))) = pk[pa][1];
        }
        fence_proxy_async();  // generic-proxy writes -> visible to the tensor-core (async) proxy
        __syncwarp();
        if (lane == 0) mbar_arrive(&s.full[st]);
        mbar_wait(&s.full[st], ph);  // both warpgroups' rows staged, B slice landed
        {
          const uint32_t a_base = smem_u32(sa) + (uint32_t)wg * (64u * kWK * 2), b_base = smem_u32(sa) + kStageA;
          const uint32_t bsplit = kWPanelB;
          wg_fence();
#pragma unroll
          for (int kk = 0; kk < 2; ++kk) {
            const uint64_t ko = (uint64_t)(kk * 2);  // 16 fp16 = 32 bytes
            const uint64_t a_h = make_wg_desc<kWK>(a_base) + ko;
            const uint64_t a_md = make_wg_desc<kWK>(a_base + (PA > 1 ? kWPanelA : 0)) + ko;
            const uint64_t a_l = make_wg_desc<kWK>(a_base + (PA > 2 ? 2 * kWPanelA : 0)) + ko;
            // both 64-column halves always: a uniform issue (no serialisation); columns beyond ncols read stale
            // rows of the stage and are never stored
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              {
                const uint32_t bj = b_base + (uint32_t)j * (64u * kWK * 2);
                const uint64_t b_h = make_wg_desc<kWK>(bj) + ko, b_m = make_wg_desc<kWK>(bj + bsplit) + ko;
                if constexpr (BITS) {
                  wgmma_64x64(acc[j], a_h, b_h);
                  wgmma_64x64(acc[j], a_h, b_m);
                } else {
                  const uint64_t b_l = make_wg_desc<kWK>(bj + 2 * bsplit) + ko;
                  wgmma_64x64(acc[j], a_h, b_h);
                  wgmma_64x64(acc[j], a_h, b_m);
                  wgmma_64x64(acc[j], a_md, b_h);
                  wgmma_64x64(acc[j], a_h, b_l);
                  wgmma_64x64(acc[j], a_l, b_h);
                  wgmma_64x64(acc[j], a_md, b_m);
                }
              }
            }
          }
          wg_commit();
        }
        // the previous stage's MMAs are done: release it (this stage's run while the next one is staged)
        wg_wait<1>();
        if (kc > 0 && t == 0) mbar_arrive(&s.empty[st_prev]);
        st_prev = st;
        if (++st == (uint32_t)p.stages) {
          st = 0;
          ph ^= 1u;
        }
      }
      wg_wait<0>();
      if (t == 0) mbar_arrive(&s.empty[st_prev]);
      s.an_part[kh * kWTileM + r] = an;
      bar_wg(wg);  // an_part of this warpgroup's rows complete

      // ---- epilogue: t -> k(t) -> K* block ----
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int rl = ra + 8 * hr;
        const int64_t grow = row0 + rl;
        const float an_r = (float)(s.an_part[rl] + s.an_part[kWTileM + rl]);
        int ct = 0;
        if (p.scaled && p.task_col >= 0 && grow < p.N) {
          const float tv = load_x_any(p.x, p.layout, grow, p.task_col, p.ldx);
          ct = min(max(__float2int_rn(tv), 0), p.n_tasks - 1);
        }
        const float* tcrow = s.tcov + ct * p.n_tasks;
        if (grow >= p.out_rows) continue;
        float* dst = p.out + grow * p.ldk;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if (j * 64 >= ncols) break;  // warp-uniform
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const int i0 = half * kWItemN + j * 64 + 8 * q + 2 * (lane & 3);
            float k[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float tt = fmaf(acc[j][4 * q + 2 * hr + e], p.inv_scale, an_r + s.wnorm_s[i0 + e]);
              float kv = kernel_from_t<FAMILY>(tt);
              if (p.scaled) kv *= tcrow[s.ttask[i0 + e]];
              k[e] = (i0 + e < p.n) ? kv : 0.f;
            }
            if (p.vec_ok && i0 + 2 <= p.out_cols) {
              *reinterpret_cast<float2*>(dst + i0) = make_float2(k[0], k[1]);
            } else {
              if (i0 < p.out_cols) dst[i0] = k[0];
              if (i0 + 1 < p.out_cols) dst[i0 + 1] = k[1];
            }
          }
        }
      }
      bar_wg(wg);  // an_part is rewritten by the next item
    }
  } else {
    // =====================================================================================
    // producer: one bulk copy (TMA engine) per K stage of the B image
    // =====================================================================================
    if (elect_one()) {
      uint32_t st = 0, ph = 0;
      for (int item = blockIdx.x; item < p.num_items; item += gridDim.x) {
        // columns [128 h, 128 h + ncols) = rows sub * 128.. of each panel of 256-column block h / 2
        const int half = item % p.n_halves, blk = half >> 1, sub = half & 1;
        const int ncols = min(kWItemN, p.n_pad - half * kWItemN);
        const int bcols = min(kWHalfN, p.n_pad - blk * kWHalfN);
        const uint32_t pbytes = (uint32_t)bcols * (kWK * 2), bytes = (uint32_t)ncols * (kWK * 2);
        const uint8_t* src = p.wimg + (size_t)blk * p.n_kc * (PB * 2 * kWPanelB) + (size_t)sub * kWPanelB;
        for (int kc = 0; kc < p.n_kc; ++kc) {
          mbar_wait_relaxed(&s.empty[st], ph ^ 1u);
          mbar_expect_tx(&s.full[st], (uint32_t)PB * bytes);
#pragma unroll
          for (int pb = 0; pb < PB; ++pb)
            bulk_g2s(s.ring + (size_t)st * kStage + kStageA + pb * kWPanelB, src + (size_t)(kc * PB + pb) * pbytes,
                     bytes, &s.full[st]);
          if (++st == (uint32_t)p.stages) {
            st = 0;
            ph ^= 1u;
          }
        }
      }
    }
  }
}

template <int FAMILY, bool BITS>
static int launch_kmat_one(WideParams& p, int sms, int max_smem, cudaStream_t stream) {
  p.stages = 4;
  WideSmem unused;
  const size_t smem = wide_carve<BITS>(nullptr, p, unused);
  BB_CHECK_SUPPORTED(smem <= (size_t)max_smem, "wide kernel-matrix path: shared-memory budget exceeded (%zu bytes)", smem);
  BB_SMEM_OPTIN_ONCE((k_kmat_wg<FAMILY, BITS>));
  const int grid = p.num_items < sms ? p.num_items : sms;
  k_kmat_wg<FAMILY, BITS><<<grid, kWideThreads, smem, stream>>>(p);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

// Column set of a K(X*, .) launch: the training rows (model images) or the pending points (scratch images).
struct WideColumns {
  const uint8_t* wimg;
  const float* wnorm;
  const int32_t* task;
  int n, n_pad;
  float inv_scale;
};

static int launch_kmat_cols(const bb_model* m, const WideColumns& c, const void* d_x, int32_t layout, int64_t N,
                            int64_t ldx, float* d_out, int64_t ldk, int64_t out_rows, int out_cols,
                            cudaStream_t stream) {
  const bool bits = layout == BB_BITS_U8;
  WideParams p;
  memset(&p, 0, sizeof(p));
  p.x = d_x;
  p.layout = layout;
  p.N = N;
  p.ldx = ldx;
  p.d = m->d;
  p.n = c.n;
  p.n_pad = c.n_pad;
  p.n_halves = (c.n_pad + kWItemN - 1) / kWItemN;
  p.n_kc = m->d_wide / kWK;
  p.cand_scale = m->d_cand_scale;
  p.cand_shift = m->d_cand_shift;
  p.wimg = c.wimg;
  p.wnorm = c.wnorm;
  p.a_scale = bits ? 1.0f : m->dist_scale_a;
  p.inv_scale = c.inv_scale;
  p.train_task = c.task;
  p.task_covar = m->d_task_covar;
  p.task_col = m->task_col;
  p.n_tasks = m->n_tasks;
  p.scaled = model_scaled(m) ? 1 : 0;
  p.out = d_out;
  p.ldk = ldk;
  p.out_rows = out_rows;
  p.out_cols = out_cols;
  p.vec_ok = ((ldk & 1) == 0 && (reinterpret_cast<uintptr_t>(d_out) & 7) == 0) ? 1 : 0;
  p.num_items = (int)((N + kWTileM - 1) / kWTileM) * p.n_halves;
  p.bits_vec = (bits && (ldx & 15) == 0 && (reinterpret_cast<uintptr_t>(d_x) & 15) == 0 && (m->d & 127) == 0) ? 1 : 0;
  int max_smem = 0, sms = 0;
  {
    const int rc_lim = device_limits(&sms, &max_smem);
    if (rc_lim != BB_OK) return rc_lim;
  }
  return dispatch_family<false>(m->family, [&](auto fam) {
    constexpr int F = decltype(fam)::value;
    return bits ? launch_kmat_one<F, true>(p, sms, max_smem, stream) : launch_kmat_one<F, false>(p, sms, max_smem, stream);
  });
}

static int wide_checks(const bb_model* m, int32_t layout) {
  BB_CHECK_SUPPORTED(m->wide != 0, "model has no wide-feature images");
  BB_CHECK_SUPPORTED(m->family != BB_KERNEL_MATERN12,
                     "Matern-1/2 is not supported on the wide-feature path (GEMM-form distances are "
                     "singular at r = 0)");
  BB_CHECK_SUPPORTED(!(layout == BB_BITS_U8 && m->task_col >= 0), "bit-packed candidates cannot carry a task column");
  return BB_OK;
}

// K(X*[0..N), X) -> d_out[row * ldk + i]; rows < out_rows and columns < out_cols are written.
int launch_kmat_wide(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx,
                     float* d_out, int64_t ldk, int64_t out_rows, int out_cols, cudaStream_t stream) {
  const int rc = wide_checks(m, layout);
  if (rc != BB_OK) return rc;
  const bool bits = layout == BB_BITS_U8;
  WideColumns c;
  c.wimg = reinterpret_cast<const uint8_t*>(bits ? m->d_wimg_bits : m->d_wimg);
  c.wnorm = bits ? m->d_wnorm_bits : m->d_train_sq;
  c.task = m->d_train_task;
  c.n = m->n;
  c.n_pad = m->n_pad;
  c.inv_scale = bits ? 1.0f / m->dist_scale_w : 1.0f / (m->dist_scale_a * m->dist_scale_b);
  return launch_kmat_cols(m, c, d_x, layout, N, ldx, d_out, ldk, out_rows, out_cols, stream);
}

// ------------------------------------------------------------------------------------------
// pending points (sequential greedy, K9 prologue) on the wide path: the <= 31 pending rows become a
// 64-column "training set" of their own -- k(x*, pending) comes out of the same tensor-core kernel --
// and the posterior cross-covariance  cov(x*, p_j) = k(x*, p_j) - K*(x*) . beta_j  is a small CUDA-core
// contraction over the K* block that is already in the workspace.
// ------------------------------------------------------------------------------------------
// One CTA per pending row pp < 64 (rows >= P are zero): operand image (float form: -2 b; bit-linear form:
// W = s (-2 b + s + 2 h)), additive norm term, task id.
__global__ void __launch_bounds__(256) k_build_pend_img(const float* __restrict__ pend_x, int P, int d, int d_wide,
                                                        const float* __restrict__ cscale, const float* __restrict__ cshift,
                                                        int bits, float scale, int task_col, int n_tasks,
                                                        uint8_t* __restrict__ img, float* __restrict__ norm,
                                                        int32_t* __restrict__ task) {
  __shared__ double red[256];
  const int pp = blockIdx.x, panels = bits ? 2 : 3;
  const size_t panel = 64 * 64;  // bytes: 64 rows x 32 fp16
  double acc = 0.0;
  for (int k = threadIdx.x; k < d_wide; k += blockDim.x) {
    float b = 0.f, sk = 0.f, hk = 0.f;
    if (pp < P && k < d) {
      sk = __ldg(cscale + k);
      hk = __ldg(cshift + k);
      b = fmaf(__ldg(pend_x + (size_t)pp * d + k), sk, hk);
    }
    float v;
    if (bits) {
      v = sk * (-2.0f * b + sk + 2.0f * hk);
      acc += (double)b * b + (double)hk * (-2.0 * (double)b + (double)hk);
    } else {
      v = -2.0f * b;
      acc += (double)b * b;
    }
    v *= scale;
    const int kc = k >> 5, kl = k & 31;
    const size_t base = (size_t)kc * panels * panel;
    const uint32_t off = swk_offset<32>((uint32_t)pp, (uint32_t)(kl >> 3)) + (uint32_t)(kl & 7) * 2u;
    const __half h = __float2half_rn(v);
    const float r1 = v - __half2float(h);
    const __half mid = __float2half_rn(r1);
    *reinterpret_cast<__half*>(img + base + off) = h;
    *reinterpret_cast<__half*>(img + base + panel + off) = mid;
    if (panels > 2) *reinterpret_cast<__half*>(img + base + 2 * panel + off) = __float2half_rn(r1 - __half2float(mid));
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if ((int)threadIdx.x < st) red[threadIdx.x] += red[threadIdx.x + st];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    norm[pp] = pp < P ? (float)red[0] : 0.f;
    int t = 0;
    if (task_col >= 0 && pp < P)
      t = min(max(__float2int_rn(__ldg(pend_x + (size_t)pp * d + task_col)), 0), n_tasks - 1);
    task[pp] = t;
  }
}

// cross[row][j] = y_std^2 * ( kpend[row][j] - sum_i kstar[row][i] beta[j][i] ): one warp per candidate row.
__global__ void __launch_bounds__(256) k_cross_pre(const float* __restrict__ kstar, const float* __restrict__ kpend,
                                                   const float* __restrict__ beta, int P, int n_pad, int64_t nrows,
                                                   float s2, float* __restrict__ cross) {
  extern __shared__ float beta_s[];  // [P][n_pad]
  for (int e = threadIdx.x; e < P * n_pad; e += blockDim.x) beta_s[e] = __ldg(beta + e);
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  for (int64_t row = (int64_t)blockIdx.x * wpb + wib; row < nrows; row += (int64_t)gridDim.x * wpb) {
    float acc[BB_MAX_PENDING];
#pragma unroll
    for (int j = 0; j < BB_MAX_PENDING; ++j) acc[j] = 0.f;
    const float* kr = kstar + row * n_pad;
    for (int i = lane; i < n_pad; i += 32) {
      const float kv = kr[i];
#pragma unroll
      for (int j = 0; j < BB_MAX_PENDING; ++j)
        if (j < P) acc[j] = fmaf(kv, beta_s[j * n_pad + i], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < BB_MAX_PENDING; ++j) {
      if (j < P) {
        float v = acc[j];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) cross[row * P + j] = s2 * (kpend[row * 64 + j] - v);
      }
    }
  }
}

// Scratch images of the pending rows (once per bb_posterior call).
int launch_pend_images(const bb_model* m, int32_t layout, const float* d_pend_x, int32_t P, cudaStream_t stream) {
  const bool bits = layout == BB_BITS_U8;
  k_build_pend_img<<<64, 256, 0, stream>>>(d_pend_x, P, m->d, m->d_wide, m->d_cand_scale, m->d_cand_shift, bits ? 1 : 0,
                                           bits ? m->dist_scale_wp : m->dist_scale_p, m->task_col, m->n_tasks,
                                           reinterpret_cast<uint8_t*>(m->d_pend_img), m->d_pend_norm, m->d_pend_task);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

// One block of candidates: k(x*, pending) through k_kmat_wg, then the cross-covariances from the K* block
// that launch_kmat_wide left in the workspace.
int launch_cross_wide(const bb_model* m, const void* d_x, int32_t layout, int64_t nb, int64_t ldx,
                      const float* d_pend_beta, int32_t P, float* d_cross_blk, cudaStream_t stream) {
  const bool bits = layout == BB_BITS_U8;
  WideColumns c;
  c.wimg = reinterpret_cast<const uint8_t*>(m->d_pend_img);
  c.wnorm = m->d_pend_norm;
  c.task = m->d_pend_task;
  c.n = P;
  c.n_pad = 64;
  c.inv_scale = bits ? 1.0f / m->dist_scale_wp : 1.0f / (m->dist_scale_a * m->dist_scale_p);
  const int64_t rows_pad = (nb + 255) / 256 * 256;
  int rc = launch_kmat_cols(m, c, d_x, layout, nb, ldx, m->d_kpend_ws, 64, rows_pad, 64, stream);
  if (rc != BB_OK) return rc;
  const size_t smem = (size_t)P * m->n_pad * sizeof(float);
  BB_SMEM_OPTIN_ONCE(k_cross_pre);
  int sms = 0, max_smem = 0;
  rc = device_limits(&sms, &max_smem);
  if (rc != BB_OK) return rc;
  k_cross_pre<<<sms * 4, 256, smem, stream>>>(m->d_wide_ws, m->d_kpend_ws, d_pend_beta, P, m->n_pad, nb,
                                              m->y_std * m->y_std, d_cross_blk);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

}  // namespace bb
