// fused_common.cuh -- parameters and helpers shared by the scoring kernels, and the host side every launcher uses
// (candidate checks, model-derived choices, family dispatch, the launchers' prototypes)
//   fused.cu  k_fused    distances on the tensor cores or the CUDA cores, V = K* L^-T on warpgroup MMAs (wgmma),
//                        q = 1 acquisition and arg-max; its PRE variant reads a K* block instead (wide-feature path)
//   wide.cu   k_kmat_wg  K-looped wgmma distance GEMM for wide / bit-packed feature spaces and n_pad > 512
#pragma once

#include <type_traits>

#include "acq_math.cuh"
#include "common.cuh"

namespace bb {

// Two consumer warpgroups (rows 0-63 and 64-127 of a 128-candidate tile) and one producer warpgroup, one elected
// thread of which issues the bulk copies.
constexpr int kConsumerWGs = 2;
constexpr int kConsumerThreads = kConsumerWGs * 128;  // 256
constexpr int kFusedThreads = kConsumerThreads + 128;  // + producer warpgroup
constexpr int kWarpProducer = kConsumerThreads / 32;  // 8
// Register split (setmaxnreg): 384 threads launch at 168 registers each; the producer warpgroup gives most of its
// share back so that a consumer thread can hold 240: 128 x 24 + 256 x 240 = 64,512 of the SM's 65,536.
constexpr int kProducerRegs = 24, kConsumerRegs = 240;
// 64-column sub-blocks of V held in registers at once: up to a 64 x 256 fp32 panel, 128 registers per consumer
// thread.  A model with n_pad <= 256 runs one panel, so every K* chunk is formed once per tile.  A launch uses
// kPanelSB or, where shared memory cannot hold the L^-1 tiles one chunk of such a panel needs, 2 (FusedParams).
constexpr int kPanelSB = 4;
constexpr int kMaxStagesB = 8;
// k_kmat_wg (wide.cu): two consumer warpgroups and one bulk-copy producer warp
constexpr int kWideThreads = kConsumerThreads + 32;
constexpr uint32_t kABytes = 16384;      // one warpgroup's K* chunk: [hi 8 KB | lo 8 KB], 64 rows x 64 fp16, SW128
constexpr uint32_t kStageBBytes = 16384; // one L^-1 tile: [hi 8 KB | lo 8 KB], 64 rows x 64 fp16, SW128
constexpr int kMaxTasks = 16;
constexpr int kMaxSamples = 1024;

struct FusedParams {
  // candidates
  const void* x;
  int layout;
  int64_t N, ldx;
  // model.  The order of the 4-byte scalars from num_tiles to panel_sb is not arbitrary: it places each at the 8-byte
  // parity it had when ptxas allocated the fewest spills for the K = 64 tensor-core k_fused (ptxas pairs adjacent
  // parameter words into 64-bit loads); other orders spill more.
  const float *cand_scale, *cand_shift, *train_m2, *train_sq, *alpha, *task_covar, *mean_const;
  const int32_t* train_task;
  const uint8_t* rimg;  // fp16 hi/lo image of L^-1: tiles (chunk c, sub-block s >= c), c-major
  int num_tiles;        // 128-row candidate tiles
  int n_pad, d, d_pad, n_chunks, task_col, n_tasks;
  float y_mean, y_std;
  // tensor-core distances (tc = K extent 32 / 64, 0: none): augmented training image [sb (-2b) | Q1 | |b|^2 Q] as
  // fp16 hi/mid/lo panels of n_pad rows x tc k; candidate rows become [sa a | |a|^2 P | P1], so the GEMM yields
  // t / ts_g directly
  int tc;
  float inv_r_scale2;
  int scaled;  // task kernel or output scale present
  int stages_b;  // L^-1 tiles in flight
  int panel_sb;  // V sub-blocks per column panel (kPanelSB or 2), chosen with stages_b by pick_stages
  const uint8_t* timg_b;
  float ts_sa, ts_aug_sq, ts_aug_one, ts_g;
  float ts_kscale;  // power of two applied to K* before the fp16 hi/lo split (fp16 range and resolution)
  // acquisition (has_acq == 0: posterior only)
  int has_acq;
  bb_acq_spec acq;
  const float* z;
  int S;
  // outputs (nullable)
  float *mu, *var, *score;
  const uint8_t* keep;
  long long* best_key;
  int64_t index_offset;
  const float* mc_table;  // qLogEI table built once per call by k_mc_table(_grid) (null: built in the kernel or unused)
  const float* kpre;  // wide-feature path: K* block already materialised by k_kmat_wg (else null)
  int64_t ldk;
  long long* trace;  // test-only event trace (bb_debug_set_trace); null in normal operation
  int trace_cap;
  // single-launch end-to-end pass (bb_score_fused_overlapped): rows arrive from the host WHILE the kernel runs
  const unsigned* ready_rows;  // rows [0, *ready_rows) of x have landed (published by the copy stream); null: all
  int32_t* gate_status;        // set to 1 if a tile's rows were not published within the time-out
  const float* code_table;     // level-coded layouts: value table [d][code_table_ld]
  int code_table_ld;
};

// optional request threaded through launch_fused by the overlapped host pass (null: none)
struct StreamGate {
  const unsigned* ready_rows;
  int32_t* status;
  const float* code_table;
  int code_table_ld;
  int layout;  // kLayoutCodes4 / kLayoutCodes8 / BB_ROW_MAJOR_F32
};

// Trace events of k_fused, recorded by thread 0 of consumer warpgroup wg as 100 wg + id: tile start, end of the chunk
// loop, end of the tile's epilogue, and the start (turn granted) and end (MMAs issued) of each MMA turn.
constexpr int kEvTileStart = 0, kEvChunksDone = 1, kEvEpilogueDone = 2, kEvTurnBegin = 10, kEvTurnEnd = 11;

// test-only: (event id, SM clock) pairs of CTA 0 for a few tiles, to reconstruct the pipeline timeline
__device__ __forceinline__ void trace_ev(const FusedParams& p, int it, int ev) {
  if (p.trace != nullptr && blockIdx.x == 0 && it >= 6 && it < 9) {
    const long long c = clock64();
    const unsigned long long i = atomicAdd(reinterpret_cast<unsigned long long*>(p.trace), 1ull);
    if ((long long)i < p.trace_cap) {
      p.trace[1 + 2 * i] = (long long)it * 1000 + ev;
      p.trace[2 + 2 * i] = c;
    }
  }
}

// the 256 consumer threads
__device__ __forceinline__ void bar_compute() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Ping-pong of the two consumer warpgroups' MMA issue (named barriers 4 and 5 over both warpgroups): warpgroup wg
// waits for its turn on barrier 4 + wg and hands the turn to the other one by arriving on the other's barrier.
__device__ __forceinline__ void mma_turn_wait(int wg) { asm volatile("bar.sync %0, 256;" ::"r"(4 + wg) : "memory"); }
__device__ __forceinline__ void mma_turn_pass(int wg) { asm volatile("bar.arrive %0, 256;" ::"r"(5 - wg) : "memory"); }

// Position in the ring of L^-1 tiles: the slot of the next tile and the parity of its mbarriers' current phase.
// Producer and consumers step it tile by tile (a compare and a wrap, no division by the run-time stage count).
struct RingPos {
  uint32_t slot = 0, phase = 0;
  __device__ __forceinline__ void advance(uint32_t stages) {
    if (++slot == stages) {
      slot = 0;
      phase ^= 1u;
    }
  }
};

template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }


// Wait used by the single-lane helper warps: mbarrier.try_wait with a suspend-time hint parks the
// thread in hardware until the phase completes (wake-up ~60 cycles after the arrive) instead of
// polling, so the helpers neither burn issue slots nor add sleep-granularity latency.
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  const uint32_t addr = smem_u32(bar);
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity), "r"(1000000u)
        : "memory");
  }
}

// fp16 hi/mid/lo split of four fp32 values -> three 8-byte packets.
__device__ __forceinline__ void split3_quad(const float (&x)[4], uint2& hi, uint2& mid, uint2& lo) {
  __half2 h01 = __floats2half2_rn(x[0], x[1]), h23 = __floats2half2_rn(x[2], x[3]);
  float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
  const float r0 = x[0] - f01.x, r1 = x[1] - f01.y, r2 = x[2] - f23.x, r3 = x[3] - f23.y;
  __half2 m01 = __floats2half2_rn(r0, r1), m23 = __floats2half2_rn(r2, r3);
  float2 g01 = __half22float2(m01), g23 = __half22float2(m23);
  __half2 l01 = __floats2half2_rn(r0 - g01.x, r1 - g01.y), l23 = __floats2half2_rn(r2 - g23.x, r3 - g23.y);
  hi = make_uint2(*reinterpret_cast<uint32_t*>(&h01), *reinterpret_cast<uint32_t*>(&h23));
  mid = make_uint2(*reinterpret_cast<uint32_t*>(&m01), *reinterpret_cast<uint32_t*>(&m23));
  lo = make_uint2(*reinterpret_cast<uint32_t*>(&l01), *reinterpret_cast<uint32_t*>(&l23));
}

// elect.sync: true in exactly one lane of a converged warp (the bulk-copy producers issue under it).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred px;\n\t"
      "elect.sync _|px, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, px;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------------------------------
// host side shared by every launcher
// ------------------------------------------------------------------------------------------
// Checks of a candidate matrix, made by every entry point that reads one before any CUDA call.  check_ld = false
// skips the leading-dimension check (level-coded rows of the gated host pass: ld in bytes, checked by the caller).
inline int check_candidates(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx,
                            bool check_ld = true) {
  BB_CHECK_ARG(m && m->abi_version == BB_ABI_VERSION, "model struct missing or ABI mismatch");
  BB_CHECK_ARG(d_x != nullptr || N == 0, "candidate pointer is null");
  BB_CHECK_ARG(layout >= 0 && layout <= BB_BITS_U8, "unknown candidate layout %d", layout);
  BB_CHECK_ARG(N >= 0, "negative candidate count");
  BB_CHECK_SUPPORTED(layout != BB_BITS_U8 || m->wide,
                     "bit-packed candidates need a wide-feature model (n_pad*d_pad*4 > 56 KB)");
  const bool col_major = (layout == BB_COL_MAJOR_F32 || layout == BB_COL_MAJOR_F64);
  BB_CHECK_ARG(!check_ld || (layout == BB_BITS_U8 ? ldx >= (m->d + 7) / 8 : (col_major ? ldx >= N : ldx >= m->d)),
               "leading dimension %lld too small", (long long)ldx);
  BB_CHECK_SUPPORTED(m->n_tasks <= kMaxTasks, "at most %d tasks supported", kMaxTasks);
  return BB_OK;
}

// K* is multiplied by the task covariance (task kernel or output scale present)
inline bool model_scaled(const bb_model* m) { return m->task_col >= 0 || m->prior_scale != 1.0f; }

// K extent (32 or 64) of the tensor-core distance GEMM over the augmented training image, 0 where the distances run
// on the CUDA cores.  Matern-1/2 has no such kernel: GEMM-form distances are singular at r = 0.
inline int model_tc_k(const bb_model* m) {
  const bool tc = !m->wide && m->d_timg_b != nullptr && m->family != BB_KERNEL_MATERN12 &&
                  (m->dist_k == 32 || m->dist_k == 64);
  return tc ? m->dist_k : 0;
}

// Calls f(std::integral_constant<int, FAMILY>()) for a runtime kernel family and returns its status.  With
// kMatern12 = false, Matern-1/2 is rejected instead of instantiated (the tensor-core distance kernels).
template <bool kMatern12, class F>
int dispatch_family(int family, F&& f) {
  switch (family) {
    case BB_KERNEL_MATERN12:
      if constexpr (kMatern12) {
        return f(std::integral_constant<int, BB_KERNEL_MATERN12>());
      } else {
        set_error("Matern-1/2 has no tensor-core distance kernel");
        return BB_ERR_UNSUPPORTED;
      }
    case BB_KERNEL_MATERN32: return f(std::integral_constant<int, BB_KERNEL_MATERN32>());
    case BB_KERNEL_MATERN52: return f(std::integral_constant<int, BB_KERNEL_MATERN52>());
    default: return f(std::integral_constant<int, BB_KERNEL_RBF>());
  }
}

// pending-point request threaded through launch_fused on the wide path (null members: none)
struct WideCross {
  const float* pend_x;
  const float* pend_beta;
  int32_t P;
  float* cross;
};

// fused.cu
int launch_fused(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx, const bb_acq_spec* acq,
                 const float* d_z, int32_t S, const uint8_t* d_keep, float* d_mu, float* d_var, float* d_score,
                 int64_t* d_best_key, int64_t index_offset, cudaStream_t stream, const WideCross* wc = nullptr,
                 const StreamGate* gate = nullptr);
// k_kmat_tma; *handled = false when the model or the output is outside its envelope
int try_kmat_tma(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx, float* d_k, int64_t ldk,
                 cudaStream_t stream, bool* handled);
// true when the single-launch gated pass can run this model
bool fused_gate_supported(const bb_model* m);
// aux_kernels.cu
int launch_cross(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx, const float* d_pend_x,
                 const float* d_pend_beta, int32_t P, float* d_cross, cudaStream_t stream);
// wide.cu
int launch_kmat_wide(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx,
                     float* d_out, int64_t ldk, int64_t out_rows, int out_cols, cudaStream_t stream);
int launch_pend_images(const bb_model* m, int32_t layout, const float* d_pend_x, int32_t P, cudaStream_t stream);
int launch_cross_wide(const bb_model* m, const void* d_x, int32_t layout, int64_t nb, int64_t ldx,
                      const float* d_pend_beta, int32_t P, float* d_cross_blk, cudaStream_t stream);

}  // namespace bb
