// fused.cu -- the scoring kernel and its launcher: per tile of 128 candidates
//   K* = k(X*, X)                       distances on the tensor cores (augmented fp16-split GEMM, K = 32 / 64) where
//                                       the model has the augmented training image, else on the CUDA cores (fp32
//                                       GEMM form); Matern/RBF epilogue on the CUDA cores
//   mu~ = c + K* alpha                  CUDA cores (fp32, folded into the K* pass)
//   V = K* L^-T                         warpgroup MMAs (wgmma), fp16 hi/lo split x3, fp32 accumulators in
//                                       registers, lower-triangular structure of L^-1 skipped tile-wise
//   var~ = k** - |V|^2 ; un-standardise  from the accumulator registers
//   q=1 acquisition value (MC or analytic) + running arg-max
// K* never leaves the SM.  One persistent CTA per SM:
//   warpgroups 0, 1   rows 0-63 / 64-127 of the tile: assemble their K* rows chunk by chunk (64 training
//                     points), write the fp16 hi/lo chunk to shared memory and issue the MMAs of that chunk;
//                     the next chunk is assembled while those MMAs run.  Then moments and acquisition.
//   warpgroup 2       bulk-copy (TMA engine) producer of the L^-1 tiles (one elected thread; 24 registers, so
//                     that a consumer thread can hold 240)
// A warpgroup holds a 64 x 256 panel of V (128 fp32 registers per thread); a model with n_pad > 256 takes several
// column panels per tile, each re-forming the K* chunks it needs (chunk c feeds sub-blocks s >= c).  The consumer
// warpgroups are independent within a tile; on the tensor-core path they alternate their MMA issue (ping-pong), so
// that one forms kernel values while the other's MMAs run.
//
// Reference path replaced: one chunk loop of botorch.optim.optimize_acqf_discrete
// (baybe/recommenders/pure/bayesian/botorch/discrete.py) = acqf(X[chunk].unsqueeze(-2)) ->
// SingleTaskGP.posterior (surrogates/gaussian_process/core.py) -> qLogExpectedImprovement.forward
// (class chosen in acquisition/base.py).
#include <cuda.h>
#include <stdlib.h>

#include "assemble.cuh"
#include "fused_common.cuh"

namespace bb {

// Tensor-core distances: K extent K2 = 32 (d <= 30) or 64 (d <= 62), the data columns followed by |a|^2 P and P1 in the
// last two; one fp16 panel of 64 candidate rows is 64 x K2 x 2 bytes.
template <int K2>
__host__ __device__ constexpr uint32_t tc_panel() { return 64u * K2 * 2u; }

// Everything the kernel keeps in shared memory, carved from the dynamic allocation.
struct FusedSmem {
  uint8_t *ring_b, *abuf;
  float4* xt4;
  float *tsq, *alpha_s;
  int32_t* ttask;
  float4* a_s;
  float *z_s, *mean_part, *var_part, *mc_part, *tcov, *meanc;
  int32_t* cand_task;
  float *cscale_s, *cshift_s;
  uint8_t *bt, *a2;  // tensor-core distances: training image, per-warpgroup candidate panels
  float* an_x;       // [2][128] |a|^2 halves of the candidate rows
  uint64_t *b_full, *b_empty;
  long long* best_red;
  float* zstat;
  volatile unsigned* ready_cache;
};

// stages_b = number of L^-1 tiles in flight; returns the byte count
static __host__ __device__ size_t carve_fused(uint8_t* base, const FusedParams& p, FusedSmem& s) {
  SmemCarver c{base};
  s.ring_b = c.take<uint8_t>((size_t)p.stages_b * kStageBBytes, 1024);  // swizzled tiles first
  s.abuf = c.take<uint8_t>(p.tc ? 0 : (size_t)kConsumerWGs * kABytes, 1024);
  s.bt = c.take<uint8_t>((size_t)3 * p.n_pad * p.tc * 2, 1024);
  s.a2 = c.take<uint8_t>((size_t)kConsumerWGs * 3 * 64 * p.tc * 2, 1024);
  s.an_x = c.take<float>(p.tc ? 2 * kTileM * 4 : 0);
  s.xt4 = c.take<float4>(p.tc ? 0 : (size_t)p.n_pad * p.d_pad * 4);
  s.tsq = c.take<float>((size_t)p.n_pad * 4);
  s.alpha_s = c.take<float>((size_t)p.n_pad * 4);
  s.ttask = c.take<int32_t>((size_t)p.n_pad * 4);
  s.a_s = c.take<float4>(p.tc ? 0 : (size_t)kTileM * p.d_pad * 8);  // duplicated candidate values
  s.z_s = c.take<float>(kMaxSamples * 4);
  s.mean_part = c.take<float>(4 * kTileM * 4);  // [4 octet groups][128]
  s.var_part = c.take<float>(kTileM * 4);
  s.mc_part = c.take<float>(1024 * 4);  // qLogEI table + exact rows, or [2 groups][128][2]
  s.tcov = c.take<float>(kMaxTasks * kMaxTasks * 4);
  s.meanc = c.take<float>(kMaxTasks * 4);
  s.cand_task = c.take<int32_t>(kTileM * 4);
  s.cscale_s = c.take<float>((size_t)p.d_pad * 4);
  s.cshift_s = c.take<float>((size_t)p.d_pad * 4);
  s.b_full = c.take<uint64_t>(2 * kMaxStagesB * 8);
  s.b_empty = s.b_full + kMaxStagesB;
  s.best_red = c.take<long long>(4 * 8);
  s.zstat = c.take<float>(16);  // mean z, mean |z - mean z|, then the gated pass's row counts
  s.ready_cache = reinterpret_cast<volatile unsigned*>(s.zstat + 2);
  return c.bytes;
}

static size_t fused_smem_bytes(const FusedParams& p) {
  FusedSmem unused;
  return carve_fused(nullptr, p, unused);
}

// Position of L^-1 tile (chunk c, sub-block sb >= c) in the c-major image of C chunks.
__host__ __device__ __forceinline__ size_t rimg_tile(int c, int sb, int C) {
  return (size_t)c * C - (size_t)c * (c - 1) / 2 + (size_t)(sb - c);
}

// Gated pass: block until the copy stream has published the rows of `tile` (acquire at system scope: the data
// was written by the copy engine before the counter).  Bounded: after ~2 s the status word is raised and the
// kernel carries on (the host reports the pass as failed) -- a missing publication must not hang the GPU.
// One thread per warpgroup polls and hands the value to the warpgroup's other threads through its word of shared
// memory; it is kept in a register, since publications run far ahead of the tiles.  Called by the 128 threads of
// warpgroup wg (t: thread within the warpgroup), so neither warpgroup waits for the other.
__device__ __forceinline__ unsigned wait_rows(const FusedParams& p, volatile unsigned* cache_s, int tile, unsigned have,
                                              int wg, int t) {
  const long long last = (long long)(tile + 1) * kTileM;
  const unsigned need = (unsigned)(last < p.N ? last : p.N);
  if (have >= need) return have;
  if (t == 0) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p.ready_rows) : "memory");
    if (v < need) {
      unsigned long long t0, t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      while (true) {
        __nanosleep(256);
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p.ready_rows) : "memory");
        if (v >= need) break;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > 2000000000ull) {
          if (p.gate_status != nullptr) *p.gate_status = 1;
          v = 0xffffffffu;  // give up waiting for good: the pass is reported as failed
          break;
        }
      }
    }
    cache_s[wg] = v;
  }
  bar_wg(wg);  // also orders the other threads' loads of the rows behind thread 0's acquire
  const unsigned v = cache_s[wg];
  bar_wg(wg);  // the word may be rewritten by the next call
  return v;
}

// Tensor-core distances: warpgroup `wg` writes its 64 candidate rows of the tile at row0 as [sa a | |a|^2 P | P1] in
// fp16 hi/mid/lo panels of K2 columns (a2w: three panels).  Thread t (r = t & 63, h = t >> 6) owns row r and the
// dimension quads h K2/8 .. (h + 1) K2/8 - 1; the owner of the last quad appends |a|^2 P and P1.  Called by the 128
// threads of the warpgroup; ends with the panels visible to the tensor cores.
template <int K2>
__device__ __forceinline__ void tc_stage_rows(const FusedParams& p, const StageCtx& sc, int64_t row0, int wg, int t,
                                              uint8_t* a2w, float* an_x, int32_t* cand_task, const float* cscale,
                                              const float* cshift) {
  constexpr int QT = K2 / 8, QL = K2 / 4 - 1;  // quads per thread, last quad
  constexpr uint32_t kPanel = tc_panel<K2>();
  const int r = t & 63, h = t >> 6, tr = 64 * wg + r;
  const int64_t row = row0 + tr;
  const int dq = p.d_pad >> 2;
  float an = 0.f, al[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int u = 0; u < QT; ++u) {
    const int jq = QT * h + u, j0 = 4 * jq;
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    if (jq < dq) {
      const float4 q = stage_load_quad(sc, row, jq, row < p.N);
      if (p.task_col >= j0 && p.task_col < j0 + 4) {
        const float tv = (p.task_col == j0) ? q.x : (p.task_col == j0 + 1) ? q.y : (p.task_col == j0 + 2) ? q.z : q.w;
        cand_task[tr] = min(max(__float2int_rn(tv), 0), p.n_tasks - 1);
      }
      a[0] = fmaf(q.x, cscale[j0], cshift[j0]);
      a[1] = fmaf(q.y, cscale[j0 + 1], cshift[j0 + 1]);
      a[2] = fmaf(q.z, cscale[j0 + 2], cshift[j0 + 2]);
      a[3] = fmaf(q.w, cscale[j0 + 3], cshift[j0 + 3]);
      an = fmaf(a[0], a[0], fmaf(a[1], a[1], fmaf(a[2], a[2], fmaf(a[3], a[3], an))));
#pragma unroll
      for (int e = 0; e < 4; ++e) a[e] *= p.ts_sa;  // exact: power of two
    }
    if (jq == QL) {
#pragma unroll
      for (int e = 0; e < 4; ++e) al[e] = a[e];
    } else {
      uint2 hi, mid, lo;
      split3_quad(a, hi, mid, lo);
      const uint32_t off = swk_offset<K2>((uint32_t)r, (uint32_t)(jq >> 1)) + (uint32_t)(jq & 1) * 8u;
      *reinterpret_cast<uint2*>(a2w + off) = hi;
      *reinterpret_cast<uint2*>(a2w + kPanel + off) = mid;
      *reinterpret_cast<uint2*>(a2w + 2 * kPanel + off) = lo;
    }
  }
  an_x[h * kTileM + tr] = an;
  bar_wg(wg);
  if (h == 1) {
    al[2] = (an_x[tr] + an_x[kTileM + tr]) * p.ts_aug_sq;
    al[3] = p.ts_aug_one;
    uint2 hi, mid, lo;
    split3_quad(al, hi, mid, lo);
    const uint32_t off = swk_offset<K2>((uint32_t)r, (uint32_t)(QL >> 1)) + 8u;
    *reinterpret_cast<uint2*>(a2w + off) = hi;
    *reinterpret_cast<uint2*>(a2w + kPanel + off) = mid;
    *reinterpret_cast<uint2*>(a2w + 2 * kPanel + off) = lo;
  }
  fence_proxy_async();
  bar_wg(wg);
}

// D[64 x 64] = A2 (a warpgroup's 64 rows) . Bt(64 training rows)^T: six fp16 split products over K2 (issued and
// committed, not waited for).  The five small split products go first, while the accumulator is still small, and the
// hi x hi products last: the fp32 accumulator, which holds terms of size |a|^2 + |b|^2 that cancel down to t, is then
// rounded at that size K2 / 16 times instead of 6 K2 / 16 times (the distance error that matters near r = 0).
template <int K2>
__device__ __forceinline__ void tc_distances(float (&dacc)[32], uint32_t a2_addr, uint32_t bt_addr, uint32_t bsplit) {
  constexpr uint32_t kPanel = tc_panel<K2>();
#pragma unroll
  for (int i = 0; i < 32; ++i) dacc[i] = 0.f;
  wg_fence();
#pragma unroll
  for (int kk = 0; kk < K2 / 16; ++kk) {
    const uint64_t ko = (uint64_t)(kk * 2);
    const uint64_t ah = make_wg_desc<K2>(a2_addr) + ko, am = make_wg_desc<K2>(a2_addr + kPanel) + ko,
                   al = make_wg_desc<K2>(a2_addr + 2 * kPanel) + ko;
    const uint64_t bh = make_wg_desc<K2>(bt_addr) + ko, bm = make_wg_desc<K2>(bt_addr + bsplit) + ko,
                   bl = make_wg_desc<K2>(bt_addr + 2 * bsplit) + ko;
    wgmma_64x64(dacc, ah, bm);
    wgmma_64x64(dacc, am, bh);
    wgmma_64x64(dacc, ah, bl);
    wgmma_64x64(dacc, al, bh);
    wgmma_64x64(dacc, am, bm);
  }
  // formed again from the two addresses: keeping the first loop's 64-bit descriptors live costs spills at K2 = 64
  asm volatile("" : "+r"(a2_addr), "+r"(bt_addr));
#pragma unroll
  for (int kk = 0; kk < K2 / 16; ++kk) {
    const uint64_t ko = (uint64_t)(kk * 2);
    wgmma_64x64(dacc, make_wg_desc<K2>(a2_addr) + ko, make_wg_desc<K2>(bt_addr) + ko);
  }
  wg_commit();
}

// The chunk loop of one tile with the schedule fixed at compile time: a tensor-core model without task kernel or output
// scale whose V is one panel of NC = n_chunks sub-blocks.  The same MMAs and the same sums in the same order as the
// run-time loops of k_fused, as straight-line code: an MMA turn is wait, fence, the chunk's (NC - c) x 12 V MMAs, the
// next chunk's distances, hand-over; ring slots and operand descriptors are worked out before the turn is asked for.
// Called by the 128 threads of warpgroup wg; `ring` is the warpgroup's position in the ring of L^-1 tiles.
template <int FAMILY, int K2, int NC>
__device__ __forceinline__ void tc_chunks_fixed(const FusedParams& p, const FusedSmem& s, int wg, int t, int lane,
                                                int it, uint32_t a2_addr, uint32_t ring_addr, RingPos& ring,
                                                float& mean0, float& mean1, float& vq0, float& vq1) {
  const uint32_t bt_addr = smem_u32(s.bt), bsplit = (uint32_t)p.n_pad * K2 * 2u;
  const uint32_t stages = (uint32_t)p.stages_b;
  const float* alpha_t = s.alpha_s + 2 * (lane & 3);
  float acc[NC][32];
#pragma unroll
  for (int j = 0; j < NC; ++j)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
  float dacc[32];
  uint32_t slot[NC];    // ring slots of the chunk whose V MMAs are in flight: sub-block c + q reads slot[q]
  uint64_t b_desc[NC];  // and the descriptors of their hi halves
  mma_turn_wait(wg);  // the tile's first turn: the distances of chunk 0
  if (t == 0) trace_ev(p, it, 100 * wg + kEvTurnBegin);
  tc_distances<K2>(dacc, a2_addr, bt_addr, bsplit);
  mma_turn_pass(wg);
  if (t == 0) trace_ev(p, it, 100 * wg + kEvTurnEnd);
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    wg_wait<0>();  // the distances of chunk c, and the V MMAs of chunk c - 1: release their L^-1 tiles
    if (c > 0 && t == 0)
#pragma unroll
      for (int q = 0; q <= NC - c; ++q) mbar_arrive(&s.b_empty[slot[q]]);
    // kernel values in the accumulator layout = the A-fragment layout of the V MMAs
    uint32_t ahi[4][4], alo[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = 8 * kk + 2 * q;
        const float k0 = kernel_from_t<FAMILY>(dacc[i] * p.ts_g), k1 = kernel_from_t<FAMILY>(dacc[i + 1] * p.ts_g);
        const float2 al = *reinterpret_cast<const float2*>(alpha_t + c * kChunk + 8 * (i >> 2));
        const float mp = fmaf(k0, al.x, k1 * al.y);
        if ((q & 1) != 0) mean1 += mp;  // accumulator rows ra + 8
        else mean0 += mp;
        split_pair(k0 * p.ts_kscale, k1 * p.ts_kscale, ahi[kk][q], alo[kk][q]);
      }
#pragma unroll
    for (int q = 0; q < NC - c; ++q) {
      slot[q] = ring.slot;
      b_desc[q] = make_wg_desc<64>(ring_addr + ring.slot * kStageBBytes);
      mbar_wait(&s.b_full[ring.slot], ring.phase);
      ring.advance(stages);
    }
    mma_turn_wait(wg);
    if (t == 0) trace_ev(p, it, 100 * wg + kEvTurnBegin);
    wg_fence();
    // V[:, sb] += K*[:, chunk c] Linv[sb, chunk c]^T for the sub-blocks sb >= c
#pragma unroll
    for (int j = c; j < NC; ++j)
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint64_t b_hi = b_desc[j - c] + (uint64_t)(kk * 2), b_lo = b_hi + (8192u >> 4);
        wgmma_64x64_rs(acc[j], ahi[kk], b_hi);
        wgmma_64x64_rs(acc[j], ahi[kk], b_lo);
        wgmma_64x64_rs(acc[j], alo[kk], b_hi);
      }
    wg_commit();
    if (c + 1 < NC) tc_distances<K2>(dacc, a2_addr, bt_addr + (uint32_t)(c + 1) * tc_panel<K2>(), bsplit);
    mma_turn_pass(wg);
    if (t == 0) trace_ev(p, it, 100 * wg + kEvTurnEnd);
  }
  wg_wait<0>();
  if (t == 0) mbar_arrive(&s.b_empty[slot[0]]);
#pragma unroll
  for (int j = 0; j < NC; ++j)
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      vq0 = fmaf(acc[j][i], acc[j][i], fmaf(acc[j][i + 1], acc[j][i + 1], vq0));
      vq1 = fmaf(acc[j][i + 2], acc[j][i + 2], fmaf(acc[j][i + 3], acc[j][i + 3], vq1));
    }
}

// PRE = true (wide-feature path): the K* block was materialised by k_kmat_wg (wide.cu) and is read from
// p.kpre instead of being assembled here; FAMILY is then irrelevant.
// TCK = 32 / 64 (n_pad <= 256, d <= 62, Matern-3/2, -5/2, RBF): the distances of a chunk come from an augmented GEMM on
// the tensor cores, and its accumulator, converted to kernel values in registers, is the register A operand of the
// chunk's V MMAs.  Otherwise the distances run on the CUDA cores and the K* chunk goes through shared memory.
// NC = 1..4 (tensor-core path only): the model has n_chunks = NC, one V panel and neither task kernel nor output scale,
// and its chunk loop is tc_chunks_fixed; NC = 0: the run-time loops below.
template <int FAMILY, bool PRE, int TCK, int NC = 0>
__global__ void __launch_bounds__(kFusedThreads, 1) k_fused(const FusedParams p) {
  constexpr bool TC = TCK > 0;
  static_assert(NC == 0 || (TC && !PRE && NC <= kPanelSB), "a fixed chunk schedule is one panel of the tensor-core path");
  constexpr int K2 = TC ? TCK : 32;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  FusedSmem s;
  carve_fused(smem_raw, p, s);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int C = p.n_chunks;
  const int dq = p.d_pad >> 2;
  if (tid == 0 && (smem_u32(smem_raw) & 1023u) != 0u) __trap();  // swizzled tiles need 1024-B alignment

  // ---- one-time setup ----
  if (tid == 0) {
    for (int i = 0; i < p.stages_b; ++i) {
      mbar_init(&s.b_full[i], 1);
      mbar_init(&s.b_empty[i], kConsumerWGs);
    }
    fence_mbar_init();
  }
  // model data resident in shared memory for the whole kernel
  if constexpr (TC) {
    const uint4* src = reinterpret_cast<const uint4*>(p.timg_b);
    uint4* dst = reinterpret_cast<uint4*>(s.bt);
    for (int e = tid; e < 3 * p.n_pad * K2 * 2 / 16; e += kFusedThreads) dst[e] = __ldg(src + e);
    for (int e = tid; e < 4 * kTileM; e += kFusedThreads) s.mean_part[e] = 0.f;  // only group 0 is written
    fence_proxy_async();  // read by the tensor cores
  } else if constexpr (!PRE) {
    load_train_rows(s.xt4, p.train_m2, p.n_pad, dq, tid, kFusedThreads);
  }
  for (int e = tid; e < p.d_pad; e += kFusedThreads) {
    s.cscale_s[e] = __ldg(p.cand_scale + e);
    s.cshift_s[e] = __ldg(p.cand_shift + e);
  }
  for (int e = tid; e < p.n_pad; e += kFusedThreads) {
    s.tsq[e] = __ldg(p.train_sq + e);
    s.alpha_s[e] = __ldg(p.alpha + e);
    s.ttask[e] = __ldg(p.train_task + e);
  }
  for (int e = tid; e < p.n_tasks * p.n_tasks; e += kFusedThreads) s.tcov[e] = __ldg(p.task_covar + e);
  for (int e = tid; e < p.n_tasks; e += kFusedThreads) s.meanc[e] = __ldg(p.mean_const + e);
  for (int e = tid; e < kTileM; e += kFusedThreads) s.cand_task[e] = 0;
  if (p.has_acq && p.z != nullptr)
    for (int e = tid; e < p.S; e += kFusedThreads) s.z_s[e] = __ldg(p.z + e);
  __syncthreads();
  if (p.has_acq && warp == 0) {
    float sz = 0.f, sa = 0.f;
    for (int e = lane; e < p.S; e += 32) sz += s.z_s[e];
    for (int o = 16; o > 0; o >>= 1) sz += __shfl_xor_sync(0xffffffffu, sz, o);
    const float zm = sz / (float)p.S;
    for (int e = lane; e < p.S; e += 32) sa += fabsf(s.z_s[e] - zm);  // qUCB: deviations from the SAMPLE mean
    for (int o = 16; o > 0; o >>= 1) sa += __shfl_xor_sync(0xffffffffu, sa, o);
    if (lane == 0) {
      s.zstat[0] = zm;
      s.zstat[1] = sa / (float)p.S;
    }
  }

  // qLogEI: tabulated fat-tail sum (acq_math.cuh).  Built once per call by k_mc_table(_grid) where a launch has
  // many CTAs (rebuilding it in every persistent CTA costs more than it saves), else here.
  const bool fast_mc = p.mc_table != nullptr || (!PRE && mc_table_applicable(p.has_acq, p.acq, p.S));
  if (p.mc_table != nullptr) {
    asm volatile("griddepcontrol.wait;" ::: "memory");  // the table kernel may still be running (dependent launch)
    for (int e = tid; e < kMcRows; e += kFusedThreads) s.mc_part[e] = __ldcg(p.mc_table + e);
    __syncthreads();
  } else if (fast_mc) {
    mc_table_setup(s.mc_part, s.z_s, p.S, p.acq.obj_scale < 0.f ? -1.f : 1.f);
  }

  if (warp < kWarpProducer) {
    // =====================================================================================
    // consumer warpgroups
    // =====================================================================================
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = warp >> 2, t = tid & 127;
    const int mp = t & 31, g = t >> 5;           // assembly: rows m0 = 64 wg + mp and m0 + 32, octets g, g + 4
    const int m0 = 64 * wg + mp, m1 = m0 + 32;
    const int row_e = 64 * wg + (t & 63), sg = t >> 6;  // epilogue: candidate row of the warpgroup, sample group
    const int ra = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // accumulator rows ra, ra + 8
    AsmSmem sm;
    sm.xt4 = s.xt4;
    sm.tsq = s.tsq;
    sm.ttask = s.ttask;
    sm.tcov = s.tcov;
    sm.a_s = s.a_s;
    sm.cand_task = s.cand_task;
    sm.dq = dq;
    sm.np = p.n_pad;
    sm.T = p.n_tasks;
    sm.scaled = p.scaled != 0;
    StageCtx sc;
    sc.x = p.x;
    sc.layout = p.layout;
    sc.N = p.N;
    sc.ldx = p.ldx;
    sc.d = p.d;
    sc.task_col = p.task_col;
    sc.cscale = s.cscale_s;
    sc.cshift = s.cshift_s;
    sc.groups = kConsumerThreads / kTileM;
    sc.gated = p.ready_rows != nullptr;
    sc.code_table = p.code_table;
    sc.code_table_ld = p.code_table_ld;
    uint8_t* abuf = s.abuf + wg * kABytes;
    const uint64_t a_hi = make_wg_desc<64>(smem_u32(abuf)), a_lo = make_wg_desc<64>(smem_u32(abuf + 8192));
    const uint32_t ring_addr = smem_u32(s.ring_b);
    // L^-1 tiles consumed so far.  Run-time schedule: a count, ring slot bcount % stages_b, phase (bcount / stages_b) & 1
    // (stepping the position instead costs these instantiations more spills); fixed schedule: the position itself.
    uint32_t bcount = 0;
    RingPos ring;
    unsigned rows_have = 0;
    StageRegs regs;
    uint8_t* a2w = s.a2 + wg * 3 * tc_panel<K2>();
    if constexpr (!PRE)
      if ((int)blockIdx.x < p.num_tiles) {
        if (sc.gated) rows_have = wait_rows(p, s.ready_cache, blockIdx.x, rows_have, wg, t);
        if constexpr (!TC) stage_prefetch(sc, dq, (int64_t)blockIdx.x * kTileM, tid, regs);
      }
    long long best = kEmptyKey;
    // TC: the warpgroups take turns issuing their MMAs (distances of a chunk, V of the previous one), so that one
    // warpgroup forms its kernel values on the CUDA cores while the other's MMAs run.  Warpgroup 0 goes first.
    if constexpr (TC)
      if (wg == 1) mma_turn_pass(wg);

    int it = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
      const int64_t row0 = (int64_t)tile * kTileM;
      if (t == 0) trace_ev(p, it, 100 * wg + kEvTileStart);
      float an0 = 0.f, an1 = 0.f;
      if constexpr (PRE) {
        if (p.task_col >= 0 && tid < kTileM) {  // task id of each candidate row (mean constant, prior variance)
          const int64_t row = row0 + tid;
          const float tv = row < p.N ? load_x_any(p.x, p.layout, row, p.task_col, p.ldx) : 0.f;
          s.cand_task[tid] = min(max(__float2int_rn(tv), 0), p.n_tasks - 1);
        }
        bar_compute();
      } else if constexpr (TC) {
        tc_stage_rows<K2>(p, sc, row0, wg, t, a2w, s.an_x, s.cand_task, s.cscale_s, s.cshift_s);
      } else {
        stage_commit(sc, s.a_s, s.cand_task, p.n_tasks, dq, row0, tid, regs);
        bar_compute();
        an0 = cand_sqnorm(sm, m0);
        an1 = cand_sqnorm(sm, m1);
      }
      float mean0 = 0.f, mean1 = 0.f, vq0 = 0.f, vq1 = 0.f;
      if constexpr (NC > 0)
        tc_chunks_fixed<FAMILY, K2, NC>(p, s, wg, t, lane, it, smem_u32(a2w), ring_addr, ring, mean0, mean1, vq0, vq1);
      for (int lo = 0; lo < (NC > 0 ? 0 : C); lo += p.panel_sb) {  // the run-time schedule (none where it is fixed)
        const int hi = min(C, lo + p.panel_sb);
        const bool last_panel = hi == C;  // covers every chunk: the mean is formed here
        float acc[kPanelSB][32];
#pragma unroll
        for (int j = 0; j < kPanelSB; ++j)
#pragma unroll
          for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
        uint32_t b_prev = 0, n_prev = 0;  // tiles read by the MMAs in flight
        for (int c = 0; c < hi; ++c) {
          uint32_t ahi[4][4], alo[4][4];  // TC: the chunk's K* as the register A operand, one [4] per 16 k
          if constexpr (TC) {
            float dacc[32];
            if (c == 0) {  // the panel's first turn: distances only (later turns start with the V MMAs below)
              mma_turn_wait(wg);
              if (t == 0) trace_ev(p, it, 100 * wg + kEvTurnBegin);
            }
            tc_distances<K2>(dacc, smem_u32(a2w), smem_u32(s.bt) + (uint32_t)c * tc_panel<K2>(),
                             (uint32_t)p.n_pad * K2 * 2u);
            mma_turn_pass(wg);
            if (t == 0) trace_ev(p, it, 100 * wg + kEvTurnEnd);
            wg_wait<0>();  // also completes the previous chunk's V MMAs: release their L^-1 tiles
            if (t == 0)
              for (uint32_t q = 0; q < n_prev; ++q) mbar_arrive(&s.b_empty[(b_prev + q) % (uint32_t)p.stages_b]);
            // kernel values in the accumulator layout = the A-fragment layout of the V MMAs
            const float* tc0 = s.tcov + s.cand_task[ra] * p.n_tasks;
            const float* tc1 = s.tcov + s.cand_task[ra + 8] * p.n_tasks;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const int i = 8 * kk + 2 * q;
                const int col = c * kChunk + 8 * (i >> 2) + 2 * (lane & 3);
                const bool upper = (q & 1) != 0;  // accumulator rows ra + 8
                float k0 = kernel_from_t<FAMILY>(dacc[i] * p.ts_g), k1 = kernel_from_t<FAMILY>(dacc[i + 1] * p.ts_g);
                if (p.scaled) {
                  const float* tcr = upper ? tc1 : tc0;
                  k0 *= tcr[s.ttask[col]];
                  k1 *= tcr[s.ttask[col + 1]];
                }
                if (last_panel) {
                  const float2 al = *reinterpret_cast<const float2*>(s.alpha_s + col);
                  const float mp = fmaf(k0, al.x, k1 * al.y);
                  if (upper) mean1 += mp;
                  else mean0 += mp;
                }
                split_pair(k0 * p.ts_kscale, k1 * p.ts_kscale, ahi[kk][q], alo[kk][q]);
              }
          } else {
            uint4 h0[2], l0[2], h1[2], l1[2];
  #pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int i0 = c * kChunk + (g + 4 * u) * 8;
              float k0[8], k1[8];
              if constexpr (PRE) {
                const float4* q0 = reinterpret_cast<const float4*>(p.kpre + (row0 + m0) * p.ldk + i0);
                const float4* q1 = reinterpret_cast<const float4*>(p.kpre + (row0 + m1) * p.ldk + i0);
                const float4 x0 = __ldg(q0), x1 = __ldg(q0 + 1), y0 = __ldg(q1), y1 = __ldg(q1 + 1);
                k0[0] = x0.x; k0[1] = x0.y; k0[2] = x0.z; k0[3] = x0.w;
                k0[4] = x1.x; k0[5] = x1.y; k0[6] = x1.z; k0[7] = x1.w;
                k1[0] = y0.x; k1[1] = y0.y; k1[2] = y0.z; k1[3] = y0.w;
                k1[4] = y1.x; k1[5] = y1.y; k1[6] = y1.z; k1[7] = y1.w;
              } else {
                assemble_2x8<FAMILY>(sm, m0, m1, an0, an1, i0, k0, k1);
              }
              if (last_panel) {
                const float4 al0 = *reinterpret_cast<const float4*>(s.alpha_s + i0);
                const float4 al1 = *reinterpret_cast<const float4*>(s.alpha_s + i0 + 4);
                const float al[8] = {al0.x, al0.y, al0.z, al0.w, al1.x, al1.y, al1.z, al1.w};
  #pragma unroll
                for (int ii = 0; ii < 8; ++ii) {
                  mean0 = fmaf(k0[ii], al[ii], mean0);
                  mean1 = fmaf(k1[ii], al[ii], mean1);
                }
              }
              split_pair(k0[0], k0[1], h0[u].x, l0[u].x);
              split_pair(k0[2], k0[3], h0[u].y, l0[u].y);
              split_pair(k0[4], k0[5], h0[u].z, l0[u].z);
              split_pair(k0[6], k0[7], h0[u].w, l0[u].w);
              split_pair(k1[0], k1[1], h1[u].x, l1[u].x);
              split_pair(k1[2], k1[3], h1[u].y, l1[u].y);
              split_pair(k1[4], k1[5], h1[u].z, l1[u].z);
              split_pair(k1[6], k1[7], h1[u].w, l1[u].w);
            }
            // the previous chunk's MMAs are done: the A buffer and their L^-1 tiles are free
            wg_wait<0>();
            if (t == 0)
              for (uint32_t q = 0; q < n_prev; ++q) mbar_arrive(&s.b_empty[(b_prev + q) % (uint32_t)p.stages_b]);
            bar_wg(wg);
  #pragma unroll
            for (int u = 0; u < 2; ++u) {
              const uint32_t o0 = sw128_offset((uint32_t)mp, (uint32_t)(g + 4 * u));
              const uint32_t o1 = sw128_offset((uint32_t)(mp + 32), (uint32_t)(g + 4 * u));
              *reinterpret_cast<uint4*>(abuf + o0) = h0[u];
              *reinterpret_cast<uint4*>(abuf + 8192 + o0) = l0[u];
              *reinterpret_cast<uint4*>(abuf + o1) = h1[u];
              *reinterpret_cast<uint4*>(abuf + 8192 + o1) = l1[u];
            }
            fence_proxy_async();  // generic-proxy writes -> visible to the tensor-core (async) proxy
            bar_wg(wg);
          }
          // V[:, sb] += K*[:, chunk c] Linv[sb, chunk c]^T for the panel's sub-blocks sb >= c
          const int s0 = c > lo ? c : lo;
          const uint32_t n_c = (uint32_t)(hi - s0);
          for (uint32_t q = 0; q < n_c; ++q) {
            const uint32_t idx = bcount + q;
            mbar_wait(&s.b_full[idx % (uint32_t)p.stages_b], (idx / (uint32_t)p.stages_b) & 1u);
          }
          if constexpr (TC) {  // this turn also issues the next chunk's distances (or ends after the last V MMAs)
            mma_turn_wait(wg);
            if (t == 0) trace_ev(p, it, 100 * wg + kEvTurnBegin);
          }
          wg_fence();
#pragma unroll
          for (int j = 0; j < kPanelSB; ++j) {
            const int sb = lo + j;
            if (sb >= s0 && sb < hi) {
              const uint32_t st = (bcount + (uint32_t)(sb - s0)) % (uint32_t)p.stages_b;
              const uint32_t b_addr = ring_addr + st * kStageBBytes;
              const uint64_t b_hi = make_wg_desc<64>(b_addr), b_lo = make_wg_desc<64>(b_addr + 8192);
#pragma unroll
              for (int kk = 0; kk < 4; ++kk) {
                const uint64_t ko = (uint64_t)(kk * 2);  // 16 fp16 = 32 bytes = 2 x 16-byte units
                if constexpr (TC) {
                  wgmma_64x64_rs(acc[j], ahi[kk], b_hi + ko);
                  wgmma_64x64_rs(acc[j], ahi[kk], b_lo + ko);
                  wgmma_64x64_rs(acc[j], alo[kk], b_hi + ko);
                } else {
                  wgmma_64x64(acc[j], a_hi + ko, b_hi + ko);
                  wgmma_64x64(acc[j], a_hi + ko, b_lo + ko);
                  wgmma_64x64(acc[j], a_lo + ko, b_hi + ko);
                }
              }
            }
          }
          wg_commit();
          if constexpr (TC)
            if (c == hi - 1) {
              mma_turn_pass(wg);
              if (t == 0) trace_ev(p, it, 100 * wg + kEvTurnEnd);
            }
          b_prev = bcount;
          n_prev = n_c;
          bcount += n_c;
        }
        wg_wait<0>();
        if (t == 0)
          for (uint32_t q = 0; q < n_prev; ++q) mbar_arrive(&s.b_empty[(b_prev + q) % (uint32_t)p.stages_b]);
#pragma unroll
        for (int j = 0; j < kPanelSB; ++j)
          if (lo + j < hi)
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
              vq0 = fmaf(acc[j][i], acc[j][i], fmaf(acc[j][i + 1], acc[j][i + 1], vq0));
              vq1 = fmaf(acc[j][i + 2], acc[j][i + 2], fmaf(acc[j][i + 3], acc[j][i + 3], vq1));
            }
      }
      if (t == 0) trace_ev(p, it, 100 * wg + kEvChunksDone);
      // |V|^2 per row: the four lanes of a quad hold the row's columns
      vq0 += __shfl_xor_sync(0xffffffffu, vq0, 1);
      vq0 += __shfl_xor_sync(0xffffffffu, vq0, 2);
      vq1 += __shfl_xor_sync(0xffffffffu, vq1, 1);
      vq1 += __shfl_xor_sync(0xffffffffu, vq1, 2);
      if ((lane & 3) == 0) {
        s.var_part[ra] = vq0;
        s.var_part[ra + 8] = vq1;
      }
      if constexpr (TC) {  // rows ra, ra + 8: the four lanes of a quad hold the row's columns
        mean0 += __shfl_xor_sync(0xffffffffu, mean0, 1);
        mean0 += __shfl_xor_sync(0xffffffffu, mean0, 2);
        mean1 += __shfl_xor_sync(0xffffffffu, mean1, 1);
        mean1 += __shfl_xor_sync(0xffffffffu, mean1, 2);
        if ((lane & 3) == 0) {
          s.mean_part[ra] = mean0;
          s.mean_part[ra + 8] = mean1;
        }
      } else {
        s.mean_part[g * kTileM + m0] = mean0;
        s.mean_part[g * kTileM + m1] = mean1;
      }
      // global loads of the next tile fly while the epilogue runs
      if constexpr (!PRE)
        if (tile + (int)gridDim.x < p.num_tiles) {
          if (sc.gated) rows_have = wait_rows(p, s.ready_cache, tile + gridDim.x, rows_have, wg, t);
          if constexpr (!TC) stage_prefetch(sc, dq, (int64_t)(tile + gridDim.x) * kTileM, tid, regs);
        }
      bar_wg(wg);

      // ---- epilogue of the warpgroup's 64 rows (two threads per row): moments in original units, acquisition,
      // arg-max ----
      const int ct = s.cand_task[row_e];
      float msum = s.meanc[ct];
#pragma unroll
      for (int gg = 0; gg < 4; ++gg) msum += s.mean_part[gg * kTileM + row_e];
      const float vsum = s.var_part[row_e];
      const float kss = p.scaled ? s.tcov[ct * p.n_tasks + ct] : 1.0f;
      const float var_t = fmaxf(kss - vsum * p.inv_r_scale2, 1e-10f);
      const float mu = fmaf(p.y_std, msum, p.y_mean);
      const float var = p.y_std * p.y_std * var_t;
      const int64_t row = row0 + row_e;
      const bool in_range = row < p.N;
      if (sg == 0 && in_range) {
        if (p.mu) p.mu[row] = mu;
        if (p.var) p.var[row] = var;
      }
      if (p.has_acq) {
        const bool is_mc = p.acq.kind <= BB_ACQ_QPI;
        float s0f = 0.f, s1f = 0.f;
        bool fast_ok = true;
        if (is_mc && fast_mc) {
          // every thread of the row evaluates the table; rows outside its envelope get the exact sum from one
          // of the two warps that share the row group (they see the same ballot; rank % 2 picks the warp)
          float c0, c1;
          mc_coef(p.acq, mu, var, c0, c1);
          fast_ok = mc_row_fast(s.mc_part, c0, c1, s0f, s1f);
          unsigned need = __ballot_sync(0xffffffffu, !fast_ok);
          for (int rank = 0; need != 0u; ++rank) {
            const int b = __ffs(need) - 1;
            need &= need - 1u;
            if ((rank & 1) != sg) continue;
            const float cb0 = __shfl_sync(0xffffffffu, c0, b), cb1 = __shfl_sync(0xffffffffu, c1, b);
            float a0, a1;
            mc_row_exact_warp(s.z_s, p.S, cb0, cb1, lane, a0, a1);
            if (lane == b) {
              s.mc_part[kMcRows + row_e] = a0;
              s.mc_part[kMcRows + kTileM + row_e] = a1;
            }
          }
        } else if (is_mc) {
          float s0, s1;
          mc_partial(p.acq, mu, var, s.z_s, p.S, sg, 2, s0, s1);
          *reinterpret_cast<float2*>(s.mc_part + (sg * kTileM + row_e) * 2) = make_float2(s0, s1);
        }
        bar_wg(wg);
        if (sg == 0) {
          float score;
          if (is_mc) {
            float s0 = 0.f, s1 = 0.f;
            if (fast_mc) {
              s0 = fast_ok ? s0f : s.mc_part[kMcRows + row_e];
              s1 = fast_ok ? s1f : s.mc_part[kMcRows + kTileM + row_e];
            } else {
#pragma unroll
              for (int gg = 0; gg < 2; ++gg) {
                const float2 pr = *reinterpret_cast<const float2*>(s.mc_part + (gg * kTileM + row_e) * 2);
                s0 += pr.x;
                s1 += pr.y;
              }
            }
            score = mc_finalize(p.acq, mu, var, s0, s1, p.S, s.zstat[0], s.zstat[1]);
          } else {
            score = analytic_value(p.acq, mu, var);
          }
          if (in_range) {
            if (p.score) p.score[row] = score;
            const bool ok = (p.keep == nullptr || p.keep[row] != 0) && !(score != score);
            if (ok) {
              const long long key = pack_key(score, (uint32_t)(row + p.index_offset));
              best = key > best ? key : best;
            }
          }
        }
      }
      // the warpgroup's shared partials are rewritten by its next tile; the CUDA-core paths also stage the next
      // tile's candidate rows (PRE: task ids) for both warpgroups at once
      if constexpr (TC) bar_wg(wg);
      else bar_compute();
      if (t == 0) trace_ev(p, it, 100 * wg + kEvEpilogueDone);
    }
    if constexpr (TC)
      if (wg == 0) mma_turn_wait(wg);  // consumes warpgroup 1's hand-over after its last turn

    // ---- CTA-level arg-max ----
    if (p.best_key != nullptr && p.has_acq) {
      if (sg == 0) {  // warps 0, 1 of each warpgroup
        for (int o = 16; o > 0; o >>= 1) {
          const long long other = __shfl_xor_sync(0xffffffffu, best, o);
          best = other > best ? other : best;
        }
        if (lane == 0) s.best_red[2 * wg + (warp & 1)] = best;
      }
      bar_compute();
      if (tid == 0) {
        long long b = s.best_red[0];
        for (int w = 1; w < 4; ++w) b = s.best_red[w] > b ? s.best_red[w] : b;
        if (b != kEmptyKey) atomicMax(p.best_key, b);
      }
    }
  } else {
    // =====================================================================================
    // producer: stream the fp16 image of L^-1 (B operand) through the TMA engine, in the order the
    // consumers read it: per tile, per column panel, per chunk c, sub-blocks sb >= c of the panel
    // =====================================================================================
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kWarpProducer && elect_one()) {
      RingPos ring;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x)
        for (int lo = 0; lo < C; lo += p.panel_sb) {
          const int hi = min(C, lo + p.panel_sb);
          for (int c = 0; c < hi; ++c)
            for (int sb = c > lo ? c : lo; sb < hi; ++sb, ring.advance((uint32_t)p.stages_b)) {
              const uint32_t st = ring.slot;
              mbar_wait_relaxed(&s.b_empty[st], ring.phase ^ 1u);
              mbar_expect_tx(&s.b_full[st], kStageBBytes);
              bulk_g2s(s.ring_b + (size_t)st * kStageBBytes, p.rimg + rimg_tile(c, sb, C) * kStageBBytes, kStageBBytes,
                       &s.b_full[st]);
            }
        }
    }
  }
}

// ------------------------------------------------------------------------------------------
// bb_kernel_matrix for models with the augmented training image: per 128-row tile and 64-column chunk, the distances
// on the tensor cores (tc_distances), the kernel values in the accumulator registers, and the 64 x 64 fp32 tile
// stored through the TMA engine (cp.async.bulk.tensor, 128B-swizzled boxes of 64 rows x 32 columns; the tensor map
// clips rows >= N and columns >= n).  Two output buffers per warpgroup: a tile is written while the previous
// store still reads the other.
// ------------------------------------------------------------------------------------------
struct KmatSmem {
  uint8_t *bt, *a2, *out;
  float *an_x, *cscale, *cshift, *tcov;
  int32_t *cand_task, *ttask;
};

// Every buffer on a 1024-byte boundary, as the swizzled tiles and TMA boxes need.
static __host__ __device__ size_t kmat_carve(uint8_t* base, const FusedParams& p, KmatSmem& s) {
  SmemCarver c{base};
  s.out = c.take<uint8_t>((size_t)kConsumerWGs * 2 * 16384, 1024);
  s.bt = c.take<uint8_t>((size_t)3 * p.n_pad * p.tc * 2, 1024);
  s.a2 = c.take<uint8_t>((size_t)kConsumerWGs * 3 * 64 * p.tc * 2, 1024);
  s.an_x = c.take<float>(2 * kTileM * 4, 1024);
  s.cscale = c.take<float>((size_t)p.d_pad * 4, 1024);
  s.cshift = c.take<float>((size_t)p.d_pad * 4, 1024);
  s.tcov = c.take<float>(kMaxTasks * kMaxTasks * 4, 1024);
  s.cand_task = c.take<int32_t>(kTileM * 4, 1024);
  s.ttask = c.take<int32_t>((size_t)p.n_pad * 4, 1024);
  return c.bytes;
}

template <int FAMILY, int K2>
__global__ void __launch_bounds__(kConsumerThreads, 1) k_kmat_tma(const FusedParams p,
                                                                  const __grid_constant__ CUtensorMap tm) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  KmatSmem s;
  kmat_carve(smem_raw, p, s);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, t = tid & 127;
  if (tid == 0 && (smem_u32(smem_raw) & 1023u) != 0u) __trap();
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.timg_b);
    uint4* dst = reinterpret_cast<uint4*>(s.bt);
    for (int e = tid; e < 3 * p.n_pad * K2 * 2 / 16; e += kConsumerThreads) dst[e] = __ldg(src + e);
  }
  for (int e = tid; e < p.d_pad; e += kConsumerThreads) {
    s.cscale[e] = __ldg(p.cand_scale + e);
    s.cshift[e] = __ldg(p.cand_shift + e);
  }
  for (int e = tid; e < p.n_pad; e += kConsumerThreads) s.ttask[e] = __ldg(p.train_task + e);
  for (int e = tid; e < p.n_tasks * p.n_tasks; e += kConsumerThreads) s.tcov[e] = __ldg(p.task_covar + e);
  for (int e = tid; e < kTileM; e += kConsumerThreads) s.cand_task[e] = 0;
  fence_proxy_async();  // the training image is read by the tensor cores
  __syncthreads();

  StageCtx sc;
  sc.x = p.x;
  sc.layout = p.layout;
  sc.N = p.N;
  sc.ldx = p.ldx;
  sc.d = p.d;
  sc.task_col = p.task_col;
  sc.cscale = s.cscale;
  sc.cshift = s.cshift;
  sc.groups = kConsumerThreads / kTileM;
  sc.gated = false;
  sc.code_table = nullptr;
  sc.code_table_ld = 0;
  uint8_t* a2w = s.a2 + wg * 3 * tc_panel<K2>();
  const uint32_t bsplit = (uint32_t)p.n_pad * K2 * 2u;
  const int rq = 16 * (warp & 3) + (lane >> 2);  // accumulator rows rq, rq + 8 of the warpgroup's 64
  uint32_t n_stores = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int64_t row0 = (int64_t)tile * kTileM;
    tc_stage_rows<K2>(p, sc, row0, wg, t, a2w, s.an_x, s.cand_task, s.cscale, s.cshift);
    const float* tc0 = s.tcov + s.cand_task[64 * wg + rq] * p.n_tasks;
    const float* tc1 = s.tcov + s.cand_task[64 * wg + rq + 8] * p.n_tasks;
    for (int c = 0; c < p.n_chunks; ++c, ++n_stores) {
      float dacc[32];
      tc_distances<K2>(dacc, smem_u32(a2w), smem_u32(s.bt) + (uint32_t)c * tc_panel<K2>(), bsplit);
      wg_wait<0>();
      uint8_t* ob = s.out + (size_t)(wg * 2 + (n_stores & 1)) * 16384;
      if (t == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");  // the store two back has read ob
      bar_wg(wg);
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int r = rq + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (lane & 3);
        const float* tcr = (i >> 1) & 1 ? tc1 : tc0;
        float k0 = kernel_from_t<FAMILY>(dacc[i] * p.ts_g), k1 = kernel_from_t<FAMILY>(dacc[i + 1] * p.ts_g);
        if (p.scaled) {
          k0 *= tcr[s.ttask[c * kChunk + col]];
          k1 *= tcr[s.ttask[c * kChunk + col + 1]];
        }
        // 128B-swizzled box layout: 16-byte chunk index XOR (row mod 8)
        const uint32_t o = (uint32_t)(col >> 5) * 8192u + (uint32_t)r * 128u +
                           ((((uint32_t)(col & 31) >> 2) ^ ((uint32_t)r & 7u)) << 4) + (uint32_t)(col & 3) * 4u;
        *reinterpret_cast<float2*>(ob + o) = make_float2(k0, k1);
      }
      fence_proxy_async();  // generic-proxy writes -> visible to the TMA engine
      bar_wg(wg);
      if (t == 0) {
        const uint64_t map = reinterpret_cast<uint64_t>(&tm);
        const int y = (int)(row0 + 64 * wg);
#pragma unroll
        for (int b = 0; b < 2; ++b)
          asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];"
                       ::"l"(map), "r"(c * kChunk + 32 * b), "r"(y), "r"(smem_u32(ob + b * 8192))
                       : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    }
  }
  if (t == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

template <int FAMILY, int K2>
static int launch_kmat_tma_one(const FusedParams& p, const CUtensorMap& tm, int grid, size_t smem, cudaStream_t stream) {
  BB_SMEM_OPTIN_ONCE((k_kmat_tma<FAMILY, K2>));
  k_kmat_tma<FAMILY, K2><<<grid, kConsumerThreads, smem, stream>>>(p, tm);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

// FusedParams of a launch over candidates x: the candidate and model fields (acquisition and outputs: the caller's).
// The tensor-core distance fields are set where the model has the augmented training image (p.tc = model_tc_k).
static FusedParams fused_params(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx) {
  FusedParams p;
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
  p.alpha = m->d_alpha;
  p.task_covar = m->d_task_covar;
  p.mean_const = m->d_mean_const;
  p.train_task = m->d_train_task;
  p.rimg = reinterpret_cast<const uint8_t*>(m->d_rimg);
  p.n_pad = m->n_pad;
  p.d = m->d;
  p.d_pad = m->d_pad;
  p.n_chunks = m->n_chunks;
  p.task_col = m->task_col;
  p.n_tasks = m->n_tasks;
  p.y_mean = m->y_mean;
  p.y_std = m->y_std;
  p.inv_r_scale2 = 1.0f / (m->r_scale * m->r_scale);
  p.scaled = model_scaled(m) ? 1 : 0;
  p.tc = model_tc_k(m);
  if (p.tc) {
    p.timg_b = reinterpret_cast<const uint8_t*>(m->d_timg_b);
    p.ts_sa = m->ts_sa;
    p.ts_aug_sq = m->ts_aug_sq;
    p.ts_aug_one = m->ts_aug_one;
    p.ts_g = m->ts_g;
    p.ts_kscale = m->ts_kscale;
    p.inv_r_scale2 /= m->ts_kscale * m->ts_kscale;  // |V|^2 of ts_kscale K*
  }
  return p;
}

// bb_kernel_matrix front door of k_kmat_tma, after check_candidates: *handled = false when the model or the output is
// outside its envelope (no tensor-core distances, ldk not a multiple of 4 or d_k not 16-byte aligned).
int try_kmat_tma(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx, float* d_k, int64_t ldk,
                 cudaStream_t stream, bool* handled) {
  *handled = false;
  if (model_tc_k(m) == 0 || layout == BB_BITS_U8 || (ldk & 3) != 0 || (reinterpret_cast<uintptr_t>(d_k) & 15) != 0)
    return BB_OK;
  const FusedParams p = fused_params(m, d_x, layout, N, ldx);
  int sms = 0, max_smem = 0;
  int rc = device_limits(&sms, &max_smem);
  if (rc != BB_OK) return rc;
  KmatSmem unused;
  const size_t smem = kmat_carve(nullptr, p, unused);
  if (smem > (size_t)max_smem) return BB_OK;
  static EncodeTiledFn encode = nullptr;
  if (encode == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    BB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    BB_CHECK_SUPPORTED(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled is not available");
    encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  CUtensorMap tm;
  const cuuint64_t gdim[2] = {(cuuint64_t)m->n, (cuuint64_t)N};
  const cuuint64_t gstride[1] = {(cuuint64_t)ldk * 4};
  const cuuint32_t box[2] = {32, 64};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = encode(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, d_k, gdim, gstride, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return BB_ERR_CUDA;
  }
  const int grid = p.num_tiles < sms ? p.num_tiles : sms;
  rc = dispatch_family<false>(m->family, [&](auto fam) {
    constexpr int F = decltype(fam)::value;
    return p.tc == 32 ? launch_kmat_tma_one<F, 32>(p, tm, grid, smem, stream)
                      : launch_kmat_tma_one<F, 64>(p, tm, grid, smem, stream);
  });
  if (rc == BB_OK) *handled = true;
  return rc;
}

// The qLogEI table of acq_math.cuh for one set of base samples, built once per call (one CTA) into the model blob.
__global__ void __launch_bounds__(512) k_mc_table(const float* __restrict__ z, int S, float sgn,
                                                  float* __restrict__ out) {
  __shared__ float z_s[512];
  __shared__ float tab[kMcRows];
  for (int e = threadIdx.x; e < S; e += blockDim.x) z_s[e] = __ldg(z + e);
  __syncthreads();
  mc_table_setup(tab, z_s, S, sgn);
  for (int e = threadIdx.x; e < kMcRows; e += blockDim.x) out[e] = tab[e];
}

// Grid version: 65 CTAs x 8 warps, one table entry per warp (acq_math.cuh).
__global__ void __launch_bounds__(256) k_mc_table_grid(const float* __restrict__ z, int S, float sgn,
                                                       float* __restrict__ out) {
  __shared__ float z_s[512];
  __shared__ float tab[kMcRows];
  for (int e = threadIdx.x; e < S; e += blockDim.x) z_s[e] = __ldg(z + e);
  __syncthreads();
  mc_table_grid_part(tab, z_s, S, sgn, out);
}

// Launch on `stream`.  after_table: k_mc_table_grid was launched just before, so this is a programmatic dependent
// launch: the prologue overlaps the table kernel and waits for it (griddepcontrol.wait) only before it reads it.
template <int FAMILY, bool PRE, int TC = 0, int NC = 0>
static int launch_one(const FusedParams& p, int grid, size_t smem, cudaStream_t stream, bool after_table) {
  BB_SMEM_OPTIN_ONCE((k_fused<FAMILY, PRE, TC, NC>));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3((unsigned)kFusedThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = after_table ? 1 : 0;
  BB_CUDA(cudaLaunchKernelEx(&cfg, k_fused<FAMILY, PRE, TC, NC>, p));
  return BB_OK;
}

// Tensor-core path.  The chunk schedule is fixed at compile time (NC = n_chunks) where the model has neither task
// kernel nor output scale and its V is one panel, the common case; task models, scaled models and a K = 64 model whose
// ring only holds a two-sub-block panel run the run-time loops (NC = 0), one instantiation per family and K.
template <int FAMILY, int TC>
static int launch_tc(const FusedParams& p, int grid, size_t smem, cudaStream_t stream, bool after_table) {
  static_assert(kPanelSB == 4, "one case per chunk count of a panel");
  switch (!p.scaled && p.n_chunks <= p.panel_sb ? p.n_chunks : 0) {
    case 1: return launch_one<FAMILY, false, TC, 1>(p, grid, smem, stream, after_table);
    case 2: return launch_one<FAMILY, false, TC, 2>(p, grid, smem, stream, after_table);
    case 3: return launch_one<FAMILY, false, TC, 3>(p, grid, smem, stream, after_table);
    case 4: return launch_one<FAMILY, false, TC, 4>(p, grid, smem, stream, after_table);
    default: return launch_one<FAMILY, false, TC>(p, grid, smem, stream, after_table);
  }
}

// The widest V panel (kPanelSB sub-blocks, else 2) whose ring fits, with as many L^-1 stages as fit; returns the
// stage count, 0 if nothing fits.  A chunk's MMAs wait for all of its tiles at once -- min(n_chunks, panel width) --
// so the ring needs at least that many stages (and no more: the warpgroups release a chunk's tiles before either
// waits for the next chunk's).
static int pick_stages(FusedParams& p, int max_smem) {
  for (int w = kPanelSB; w >= 2; w -= 2) {
    p.panel_sb = w;
    const int need = p.n_chunks < w ? p.n_chunks : w;
    for (int st = kMaxStagesB; st >= need && st >= 1; --st) {
      p.stages_b = st;
      if (fused_smem_bytes(p) <= (size_t)max_smem) return st;
    }
  }
  p.panel_sb = 2;
  p.stages_b = 2;
  return 0;
}

// Wide-feature models: per block of <= wide_ws_rows candidates, k_kmat_wg writes the K* block into the
// workspace inside the model blob (whole waves of work items, within 40 MB of L2 while one wave fits: n_pad <= 576) and k_fused<PRE> consumes it; both on the caller's stream.
static int launch_wide_blocks(const bb_model* m, const FusedParams& full, int sms, int max_smem,
                              const WideCross* wc, cudaStream_t stream) {
  BB_CHECK_SUPPORTED(m->d_wide_ws != nullptr && m->wide_ws_rows >= 256, "wide model without workspace");
  if (wc != nullptr) {
    const int rcp = launch_pend_images(m, full.layout, wc->pend_x, wc->P, stream);
    if (rcp != BB_OK) return rcp;
  }
  const float* mc_table = nullptr;
  if (m->d_mc_table != nullptr && mc_table_applicable(full.has_acq, full.acq, full.S)) {
    k_mc_table<<<1, 512, 0, stream>>>(full.z, full.S, full.acq.obj_scale < 0.f ? -1.f : 1.f, m->d_mc_table);
    BB_LAUNCH_CHECK();
    mc_table = m->d_mc_table;
  }
  const int64_t es = (full.layout == BB_ROW_MAJOR_F64 || full.layout == BB_COL_MAJOR_F64) ? 8 : 4;
  const bool col_major = (full.layout == BB_COL_MAJOR_F32 || full.layout == BB_COL_MAJOR_F64);
  for (int64_t b0 = 0; b0 < full.N; b0 += m->wide_ws_rows) {
    const int64_t nb = full.N - b0 < m->wide_ws_rows ? full.N - b0 : m->wide_ws_rows;
    const uint8_t* xb = reinterpret_cast<const uint8_t*>(full.x);
    if (full.layout == BB_BITS_U8) xb += b0 * full.ldx;
    else xb += col_major ? b0 * es : b0 * full.ldx * es;
    const int64_t rows_pad = (nb + 255) / 256 * 256;
    int rc = launch_kmat_wide(m, xb, full.layout, nb, full.ldx, m->d_wide_ws, m->n_pad, rows_pad, m->n_pad,
                              stream);
    if (rc != BB_OK) return rc;
    if (wc != nullptr) {
      rc = launch_cross_wide(m, xb, full.layout, nb, full.ldx, wc->pend_beta, wc->P, wc->cross + b0 * wc->P, stream);
      if (rc != BB_OK) return rc;
    }
    FusedParams p = full;
    p.x = xb;
    p.N = nb;
    p.num_tiles = (int)((nb + kTileM - 1) / kTileM);
    p.kpre = m->d_wide_ws;
    p.ldk = m->n_pad;
    p.d = 0;
    p.d_pad = 0;  // nothing of the feature dimension is staged by the K*-reading kernel
    if (p.mu) p.mu += b0;
    if (p.var) p.var += b0;
    if (p.score) p.score += b0;
    if (p.keep) p.keep += b0;
    p.index_offset = full.index_offset + b0;
    BB_CHECK_SUPPORTED(pick_stages(p, max_smem) > 0, "shared-memory budget exceeded: need %zu bytes",
                       fused_smem_bytes(p));
    p.mc_table = mc_table;
    const int grid = p.num_tiles < sms ? p.num_tiles : sms;
    rc = launch_one<BB_KERNEL_RBF, true>(p, grid, fused_smem_bytes(p), stream, false);
    if (rc != BB_OK) return rc;
  }
  return BB_OK;
}

static thread_local long long* g_trace_buf = nullptr;  // test-only; per host thread, so concurrent callers never see it
static thread_local int g_trace_cap = 0;

int launch_fused(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx,
                 const bb_acq_spec* acq, const float* d_z, int32_t S, const uint8_t* d_keep,
                 float* d_mu, float* d_var, float* d_score, int64_t* d_best_key,
                 int64_t index_offset, cudaStream_t stream, const WideCross* wc, const StreamGate* gate) {
  const bool code_rows = gate != nullptr && gate->layout >= kLayoutCodes4;
  const int rc_x = check_candidates(m, d_x, layout, N, ldx, !code_rows);
  if (rc_x != BB_OK) return rc_x;
  BB_CHECK_ARG(N + index_offset < 0xffffffffLL, "candidate index exceeds the 32-bit key range");
  if (acq) {
    BB_CHECK_ARG(acq->kind >= BB_ACQ_QLOGEI && acq->kind <= BB_ACQ_PSTD, "unknown acquisition kind %d",
                 acq->kind);
    const bool is_mc = acq->kind <= BB_ACQ_QPI;
    BB_CHECK_ARG(!is_mc || (d_z != nullptr && S >= 16 && S <= kMaxSamples && S % 16 == 0),
                 "fused MC scoring needs base samples with 16 <= S <= %d, S %% 16 == 0 (got S=%d)",
                 kMaxSamples, S);
  }
  if (N == 0) return BB_OK;

  FusedParams p = fused_params(m, d_x, layout, N, ldx);
  p.has_acq = acq ? 1 : 0;
  if (acq) p.acq = *acq;
  p.z = d_z;
  p.S = S;
  p.mu = d_mu;
  p.var = d_var;
  p.score = d_score;
  p.keep = d_keep;
  p.best_key = reinterpret_cast<long long*>(d_best_key);
  p.index_offset = index_offset;
  p.trace = g_trace_buf;
  p.trace_cap = g_trace_cap;
  if (gate != nullptr) {  // overlapped host pass: rows are published while the kernel runs
    p.ready_rows = gate->ready_rows;
    p.gate_status = gate->status;
    p.code_table = gate->code_table;
    p.code_table_ld = gate->code_table_ld;
    p.layout = gate->layout;
  }
  int max_smem = 0, sms = 0;
  {
    const int rc_lim = device_limits(&sms, &max_smem);
    if (rc_lim != BB_OK) return rc_lim;
  }
  BB_CHECK_SUPPORTED(gate == nullptr || !m->wide, "the overlapped host pass does not cover wide-feature models");
  if (m->wide) return launch_wide_blocks(m, p, sms, max_smem, wc, stream);
  if (p.tc && pick_stages(p, max_smem) == 0) {  // the resident training image does not fit: CUDA-core distances
    p.tc = 0;
    p.inv_r_scale2 *= p.ts_kscale * p.ts_kscale;
  }
  BB_CHECK_SUPPORTED(pick_stages(p, max_smem) > 0, "shared-memory budget exceeded: need %zu bytes, device allows %d",
                     fused_smem_bytes(p), max_smem);
  const int grid = p.num_tiles < sms ? p.num_tiles : sms;
  if (m->d_mc_table != nullptr && mc_table_applicable(p.has_acq, p.acq, p.S) && grid > 8) {
    // qLogEI table once per call instead of once per persistent CTA (short launches keep the in-kernel build)
    k_mc_table_grid<<<(kMcNT + 8) / 8, 256, 0, stream>>>(p.z, p.S, p.acq.obj_scale < 0.f ? -1.f : 1.f, m->d_mc_table);
    BB_LAUNCH_CHECK();
    p.mc_table = m->d_mc_table;
  }
  const size_t smem = fused_smem_bytes(p);
  const bool dep = p.mc_table != nullptr;
  if (p.tc == 0)
    return dispatch_family<true>(m->family, [&](auto fam) {
      return launch_one<decltype(fam)::value, false>(p, grid, smem, stream, dep);
    });
  return dispatch_family<false>(m->family, [&](auto fam) {
    constexpr int F = decltype(fam)::value;
    return p.tc == 32 ? launch_tc<F, 32>(p, grid, smem, stream, dep) : launch_tc<F, 64>(p, grid, smem, stream, dep);
  });
}

// Shape test of the single-launch gated pass: k_fused over non-wide models.
bool fused_gate_supported(const bb_model* m) {
  if (m == nullptr || m->wide || m->n_tasks > kMaxTasks) return false;
  FusedParams p;
  memset(&p, 0, sizeof(p));
  p.n_pad = m->n_pad;
  p.d_pad = m->d_pad;
  p.n_chunks = m->n_chunks;
  int sms = 0, max_smem = 0;
  if (device_limits(&sms, &max_smem) != BB_OK) return false;
  return pick_stages(p, max_smem) > 0;
}

}  // namespace bb

using namespace bb;

// test-only: route the next fused launches' pipeline events of CTA 0 into d_buf
// ([0] = count, then (tile*1000+event, SM clock) pairs); pass null to switch tracing off.
extern "C" int bb_debug_set_trace(int64_t* d_buf, int64_t capacity_pairs) {
  bb::g_trace_buf = reinterpret_cast<long long*>(d_buf);
  bb::g_trace_cap = (int)capacity_pairs;
  return BB_OK;
}

extern "C" int bb_score_fused(const bb_model* m, const bb_acq_spec* a, const void* d_x,
                              int32_t layout, int64_t N, int64_t ldx, const uint8_t* d_keep,
                              const float* d_z, int32_t S, float* d_score, int64_t* d_best_key,
                              int64_t index_offset, void* stream) {
  BB_CHECK_ARG(a != nullptr, "bb_score_fused: acquisition spec is null");
  return launch_fused(m, d_x, layout, N, ldx, a, d_z, S, d_keep, nullptr, nullptr, d_score,
                      d_best_key, index_offset, (cudaStream_t)stream);
}

extern "C" int bb_posterior(const bb_model* m, const void* d_x, int32_t layout, int64_t N,
                            int64_t ldx, float* d_mu, float* d_var, float* d_cross,
                            const float* d_pend_x, const float* d_pend_beta, int32_t n_pending,
                            void* stream) {
  BB_CHECK_ARG(N == 0 || (d_mu != nullptr && d_var != nullptr), "bb_posterior: output pointers are null");
  if (m && m->abi_version == BB_ABI_VERSION && m->wide && d_cross != nullptr && n_pending > 0) {
    // wide-feature models: the cross-covariances reuse each K* block while it sits in the workspace
    BB_CHECK_ARG(d_pend_x && d_pend_beta, "pending buffers are null");
    BB_CHECK_ARG(n_pending <= BB_MAX_PENDING, "n_pending=%d outside [1,%d]", n_pending, BB_MAX_PENDING);
    WideCross wc{d_pend_x, d_pend_beta, n_pending, d_cross};
    return launch_fused(m, d_x, layout, N, ldx, nullptr, nullptr, 0, nullptr, d_mu, d_var, nullptr, nullptr, 0,
                        (cudaStream_t)stream, &wc);
  }
  int rc = launch_fused(m, d_x, layout, N, ldx, nullptr, nullptr, 0, nullptr, d_mu, d_var, nullptr,
                        nullptr, 0, (cudaStream_t)stream);
  if (rc != BB_OK) return rc;
  if (d_cross != nullptr && n_pending > 0)
    return launch_cross(m, d_x, layout, N, ldx, d_pend_x, d_pend_beta, n_pending, d_cross,
                        (cudaStream_t)stream);
  return BB_OK;
}
