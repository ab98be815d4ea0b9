// assemble.cuh -- the K(X*, X) assembly core shared by the fused scoring kernel (A operand of the
// wgmma GEMM), the stand-alone kernel-matrix kernel and the pending cross-covariance kernel.
//
// Restates gpytorch MaternKernel/RBFKernel.forward + Distance._sq_dist (constructed by the
// reference at /root/reference/baybe/kernels/base.py:173-178): scaled squared distance in the
// "GEMM form" |a|^2 + |b|^2 - 2 a.b on mean-centred inputs, clamped at 0, then the family's
// closed form.  Normalisation (botorch Normalize, gaussian_process/core.py:301-305), centring,
// the ARD 1/lengthscale and the family constant (5, 3, 1, log2(e)/2) are folded into one
// per-column scale/shift applied when the candidate tile is staged in shared memory.
// Matern-1/2 is not differentiable in r^2 at 0, so for that family the distance is formed from
// direct differences (exact near coincident points) at twice the FMA cost.
//
// Register tile: one thread = 2 candidates x 8 training points.  Training rows are stored
// pair-interleaved and the candidate values duplicated so that every operand pair comes straight
// out of an LDS.128.
#pragma once

#include "common.cuh"

namespace bb {

// Shared-memory resident model data needed by the assembly core.
// Layouts (dq = d_pad/4 dimension quads, np = number of training rows, multiple of 8):
//   xt4 [dq][np] float4.  For the training pair (i, i+1), i even, and quad jc:
//         xt4[jc*np + i]   = { b_i[4jc],   b_i+1[4jc],   b_i[4jc+1], b_i+1[4jc+1] }
//         xt4[jc*np + i+1] = { b_i[4jc+2], b_i+1[4jc+2], b_i[4jc+3], b_i+1[4jc+3] }
//       where b = -2 x scaled training row.
//   a_s [dq][2][128] float4.  For candidate m and quad jc:
//         a_s[(2jc  )*128 + m] = { a[4jc],   a[4jc],   a[4jc+1], a[4jc+1] }
//         a_s[(2jc+1)*128 + m] = { a[4jc+2], a[4jc+2], a[4jc+3], a[4jc+3] }
struct AsmSmem {
  const float4* xt4;
  const float* tsq;      // [np] squared norms of the scaled training rows
  const int32_t* ttask;  // [np] task ids of the training rows
  const float* tcov;     // [T*T] task covariance (prior scale folded in)
  float4* a_s;
  int32_t* cand_task;    // [128]
  int dq;
  int np;
  int T;
  bool scaled;           // task covariance / prior scale must be applied
};

// Float index of element (training row i, column j) inside the pair-interleaved xt4 layout.
__host__ __device__ __forceinline__ int xt_float_index(int np, int i, int j) {
  const int jc = j >> 2, comp = j & 3;
  return ((jc * np + (i & ~1) + (comp >> 1)) << 2) + ((comp & 1) << 1) + (i & 1);
}

// Copy the [np][d_pad] row-major global training block into the pair-interleaved shared layout.
__device__ __forceinline__ void load_train_rows(float4* xt4_s, const float* __restrict__ g, int np,
                                                int dq, int t, int nthreads) {
  const float4* src = reinterpret_cast<const float4*>(g);
  const int pairs = np >> 1;
  for (int e = t; e < pairs * dq; e += nthreads) {
    const int ip = e / dq, jc = e - ip * dq;
    const float4 b0 = __ldg(src + (size_t)(2 * ip) * dq + jc);
    const float4 b1 = __ldg(src + (size_t)(2 * ip + 1) * dq + jc);
    xt4_s[jc * np + 2 * ip] = make_float4(b0.x, b1.x, b0.y, b1.y);
    xt4_s[jc * np + 2 * ip + 1] = make_float4(b0.z, b1.z, b0.w, b1.w);
  }
}

// ------------------------------------------------------------------------------------------
// Candidate staging: thread (r = t & 127, jg = t >> 7) owns row r and the dimension quads
// jg, jg + groups, ...; at most kStageQuads quads per thread are prefetched into registers.
// ------------------------------------------------------------------------------------------
constexpr int kStageQuads = 2;

struct StageRegs {
  float4 v[kStageQuads];
};

template <int LAYOUT>
__device__ __forceinline__ float4 load_quad(const void* __restrict__ x, int64_t row, int j0, int d,
                                            int64_t ldx, bool row_ok) {
  float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!row_ok) return q;
  if constexpr (LAYOUT == BB_ROW_MAJOR_F32) {
    const float* p = reinterpret_cast<const float*>(x) + row * ldx + j0;
    if (j0 + 3 < d && ((reinterpret_cast<uintptr_t>(p) & 15) == 0)) {
      q = __ldg(reinterpret_cast<const float4*>(p));
    } else {
      if (j0 < d) q.x = __ldg(p);
      if (j0 + 1 < d) q.y = __ldg(p + 1);
      if (j0 + 2 < d) q.z = __ldg(p + 2);
      if (j0 + 3 < d) q.w = __ldg(p + 3);
    }
  } else {
    if (j0 < d) q.x = load_x<LAYOUT>(x, row, j0, ldx);
    if (j0 + 1 < d) q.y = load_x<LAYOUT>(x, row, j0 + 1, ldx);
    if (j0 + 2 < d) q.z = load_x<LAYOUT>(x, row, j0 + 2, ldx);
    if (j0 + 3 < d) q.w = load_x<LAYOUT>(x, row, j0 + 3, ldx);
  }
  return q;
}

// Rows that arrive while the kernel runs (gated host pass) are read with ld.global.cg: coherent at L2, where the
// copy engine's writes land; ld.global.nc (__ldg) presumes data that is constant for the kernel's lifetime.
// Level-coded rows (kLayoutCodes4: two columns per byte, low nibble = even column; kLayoutCodes8: one byte per
// column) index the per-column value table [d][table_ld].
__device__ __forceinline__ float4 load_quad_gated(const void* __restrict__ x, int layout, int64_t row, int j0, int d,
                                                  int64_t ldx, bool row_ok, const float* __restrict__ table,
                                                  int table_ld) {
  float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!row_ok || j0 >= d) return q;
  if (layout == kLayoutCodes4) {
    const uint8_t* c = reinterpret_cast<const uint8_t*>(x) + row * ldx + (j0 >> 1);
    const uint32_t b0 = __ldcg(c), b1 = (j0 + 2 < d) ? (uint32_t)__ldcg(c + 1) : 0u;
    const float* t = table + (size_t)j0 * table_ld;
    q.x = __ldg(t + (b0 & 15u));
    if (j0 + 1 < d) q.y = __ldg(t + table_ld + (b0 >> 4));
    if (j0 + 2 < d) q.z = __ldg(t + 2 * table_ld + (b1 & 15u));
    if (j0 + 3 < d) q.w = __ldg(t + 3 * table_ld + (b1 >> 4));
  } else if (layout == kLayoutCodes8) {
    const uint8_t* c = reinterpret_cast<const uint8_t*>(x) + row * ldx + j0;
    const float* t = table + (size_t)j0 * table_ld;
    q.x = __ldg(t + __ldcg(c));
    if (j0 + 1 < d) q.y = __ldg(t + table_ld + __ldcg(c + 1));
    if (j0 + 2 < d) q.z = __ldg(t + 2 * table_ld + __ldcg(c + 2));
    if (j0 + 3 < d) q.w = __ldg(t + 3 * table_ld + __ldcg(c + 3));
  } else {  // row-major fp32
    const float* ptr = reinterpret_cast<const float*>(x) + row * ldx + j0;
    if (j0 + 3 < d && ((reinterpret_cast<uintptr_t>(ptr) & 15) == 0)) return __ldcg(reinterpret_cast<const float4*>(ptr));
    q.x = __ldcg(ptr);
    if (j0 + 1 < d) q.y = __ldcg(ptr + 1);
    if (j0 + 2 < d) q.z = __ldcg(ptr + 2);
    if (j0 + 3 < d) q.w = __ldcg(ptr + 3);
  }
  return q;
}

__device__ __forceinline__ float4 load_quad_any(const void* __restrict__ x, int layout, int64_t row,
                                                int j0, int d, int64_t ldx, bool row_ok) {
  switch (layout) {
    case BB_ROW_MAJOR_F32: return load_quad<BB_ROW_MAJOR_F32>(x, row, j0, d, ldx, row_ok);
    case BB_COL_MAJOR_F32: return load_quad<BB_COL_MAJOR_F32>(x, row, j0, d, ldx, row_ok);
    case BB_ROW_MAJOR_F64: return load_quad<BB_ROW_MAJOR_F64>(x, row, j0, d, ldx, row_ok);
    default: return load_quad<BB_COL_MAJOR_F64>(x, row, j0, d, ldx, row_ok);
  }
}

struct StageCtx {
  const void* x;
  int layout;
  int64_t N, ldx;
  int d, task_col;
  const float* cscale;  // shared [d_pad]
  const float* cshift;
  int groups;           // nthreads / 128
  bool gated;           // rows published while the kernel runs (level codes or row-major fp32)
  const float* code_table;
  int code_table_ld;
};

__device__ __forceinline__ float4 stage_load_quad(const StageCtx& c, int64_t row, int jq, bool row_ok) {
  if (c.gated) return load_quad_gated(c.x, c.layout, row, jq * 4, c.d, c.ldx, row_ok, c.code_table, c.code_table_ld);
  return load_quad_any(c.x, c.layout, row, jq * 4, c.d, c.ldx, row_ok);
}

// Issue the global loads of tile `row0` (first kStageQuads quads of this thread) into registers.
__device__ __forceinline__ void stage_prefetch(const StageCtx& c, int dq, int64_t row0, int t,
                                               StageRegs& regs) {
  const int r = t & (kTileM - 1), jg = t >> 7;
  const int64_t row = row0 + r;
  const bool ok = row < c.N;
#pragma unroll
  for (int u = 0; u < kStageQuads; ++u) {
    const int jq = jg + u * c.groups;
    regs.v[u] = (jq < dq) ? stage_load_quad(c, row, jq, ok) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__device__ __forceinline__ void stage_store_quad(const StageCtx& c, float4* a_s, int32_t* cand_task,
                                                 int T, int r, int jq, float4 q) {
  const int j0 = jq * 4;
  if (c.task_col >= j0 && c.task_col < j0 + 4) {
    const float tv = (c.task_col == j0) ? q.x : (c.task_col == j0 + 1) ? q.y : (c.task_col == j0 + 2) ? q.z : q.w;
    cand_task[r] = min(max(__float2int_rn(tv), 0), T - 1);
  }
  const float ax = fmaf(q.x, c.cscale[j0], c.cshift[j0]);  // padded dims: scale = shift = 0
  const float ay = fmaf(q.y, c.cscale[j0 + 1], c.cshift[j0 + 1]);
  const float az = fmaf(q.z, c.cscale[j0 + 2], c.cshift[j0 + 2]);
  const float aw = fmaf(q.w, c.cscale[j0 + 3], c.cshift[j0 + 3]);
  a_s[(2 * jq) * kTileM + r] = make_float4(ax, ax, ay, ay);
  a_s[(2 * jq + 1) * kTileM + r] = make_float4(az, az, aw, aw);
}

// Store the prefetched quads, then load+store any remaining quads (large d) directly.
__device__ __forceinline__ void stage_commit(const StageCtx& c, float4* a_s, int32_t* cand_task,
                                             int T, int dq, int64_t row0, int t,
                                             const StageRegs& regs) {
  const int r = t & (kTileM - 1), jg = t >> 7;
#pragma unroll
  for (int u = 0; u < kStageQuads; ++u) {
    const int jq = jg + u * c.groups;
    if (jq < dq) stage_store_quad(c, a_s, cand_task, T, r, jq, regs.v[u]);
  }
  const int64_t row = row0 + r;
  for (int jq = jg + kStageQuads * c.groups; jq < dq; jq += c.groups)
    stage_store_quad(c, a_s, cand_task, T, r, jq, stage_load_quad(c, row, jq, row < c.N));
}

__device__ __forceinline__ float cand_sqnorm(const AsmSmem& sm, int m) {
  float s = 0.0f;
  for (int h = 0; h < 2 * sm.dq; ++h) {
    const float4 a = sm.a_s[h * kTileM + m];
    s = fmaf(a.x, a.x, fmaf(a.z, a.z, s));
  }
  return s;
}

// Kernel values of candidates (m0, m1) against the 8 training points i0..i0+7 (i0 % 8 == 0).
template <int FAMILY>
__device__ __forceinline__ void assemble_2x8(const AsmSmem& sm, int m0, int m1, float an0,
                                             float an1, int i0, float (&k0)[8], float (&k1)[8]) {
  constexpr bool kDirect = (FAMILY == BB_KERNEL_MATERN12);
  float t0[8], t1[8];
  {
    float acc0[8], acc1[8];
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) {
      const float t = kDirect ? 0.f : sm.tsq[i0 + ii];
      acc0[ii] = kDirect ? 0.f : t + an0;
      acc1[ii] = kDirect ? 0.f : t + an1;
    }
    const float4* xt = sm.xt4 + i0;
    const float4* a0p = sm.a_s + m0;
    const float4* a1p = sm.a_s + m1;
#pragma unroll 1
    for (int jc = 0; jc < sm.dq; ++jc) {
      const float4 A00 = a0p[0], A01 = a0p[kTileM];  // {x,x,y,y}, {z,z,w,w}
      const float4 A10 = a1p[0], A11 = a1p[kTileM];
#pragma unroll
      for (int ip = 0; ip < 4; ++ip) {
        const float4 P0 = xt[2 * ip], P1 = xt[2 * ip + 1];
        const float bx[2] = {P0.x, P0.y}, by[2] = {P0.z, P0.w}, bz[2] = {P1.x, P1.y}, bw[2] = {P1.z, P1.w};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ii = 2 * ip + h;
          if constexpr (kDirect) {
            float e;
            e = fmaf(0.5f, bx[h], A00.x); acc0[ii] = fmaf(e, e, acc0[ii]);
            e = fmaf(0.5f, by[h], A00.z); acc0[ii] = fmaf(e, e, acc0[ii]);
            e = fmaf(0.5f, bz[h], A01.x); acc0[ii] = fmaf(e, e, acc0[ii]);
            e = fmaf(0.5f, bw[h], A01.z); acc0[ii] = fmaf(e, e, acc0[ii]);
            e = fmaf(0.5f, bx[h], A10.x); acc1[ii] = fmaf(e, e, acc1[ii]);
            e = fmaf(0.5f, by[h], A10.z); acc1[ii] = fmaf(e, e, acc1[ii]);
            e = fmaf(0.5f, bz[h], A11.x); acc1[ii] = fmaf(e, e, acc1[ii]);
            e = fmaf(0.5f, bw[h], A11.z); acc1[ii] = fmaf(e, e, acc1[ii]);
          } else {
            acc0[ii] = fmaf(A00.x, bx[h], fmaf(A00.z, by[h], fmaf(A01.x, bz[h], fmaf(A01.z, bw[h], acc0[ii]))));
            acc1[ii] = fmaf(A10.x, bx[h], fmaf(A10.z, by[h], fmaf(A11.x, bz[h], fmaf(A11.z, bw[h], acc1[ii]))));
          }
        }
      }
      xt += sm.np;
      a0p += 2 * kTileM;
      a1p += 2 * kTileM;
    }
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) {
      t0[ii] = acc0[ii];
      t1[ii] = acc1[ii];
    }
  }
#pragma unroll
  for (int ii = 0; ii < 8; ++ii) {
    k0[ii] = kernel_from_t<FAMILY>(t0[ii]);
    k1[ii] = kernel_from_t<FAMILY>(t1[ii]);
  }
  if (sm.scaled) {
    const float* r0 = sm.tcov + sm.cand_task[m0] * sm.T;
    const float* r1 = sm.tcov + sm.cand_task[m1] * sm.T;
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) {
      const int tt = sm.ttask[i0 + ii];
      k0[ii] *= r0[tt];
      k1[ii] *= r1[tt];
    }
  }
}

}  // namespace bb
