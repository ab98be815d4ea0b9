// stream.cu -- the end-to-end pass over a candidate set that lives in (pinned) HOST memory.
//
// bb_score_fused_host copies row blocks on the caller's copy stream while the previous block is expanded
// (level-coded rows: bb_decode_codes) and scored (the fused kernel) on the caller's compute stream; two staging
// slots, four events created and destroyed inside the call.  One C call per pass: the Python loop it replaces spent
// ~70 us of host time per block, more than the GPU needs for a block of 125,000 rows (60 us).
// Replaces: SubspaceDiscrete.transform + to_tensor + optimize_acqf_discrete over a host-resident comp-rep
// (baybe/recommenders/pure/bayesian/botorch/discrete.py:120-126).
#include <cuda.h>
#include <stdlib.h>

#include "fused_common.cuh"

using namespace bb;

extern "C" int bb_score_fused_host(const bb_model* m, const bb_acq_spec* a, const void* h_x, int32_t host_format,
                                   int64_t N, int64_t ld, const float* d_table, int32_t table_ld,
                                   void* const* d_stage, float* const* d_rows, int64_t block_rows,
                                   const uint8_t* d_keep, const float* d_z, int32_t S, float* d_score,
                                   int64_t* d_best_key, int64_t index_offset, void* stream_, void* copy_stream_) {
  cudaStream_t stream = (cudaStream_t)stream_, copy = (cudaStream_t)copy_stream_;
  BB_CHECK_ARG(m && m->abi_version == BB_ABI_VERSION && a, "bb_score_fused_host: model / acquisition spec missing");
  BB_CHECK_ARG(N >= 0 && block_rows >= 128 && block_rows % 128 == 0, "bb_score_fused_host: block_rows must be a positive multiple of 128");
  BB_CHECK_ARG(d_stage && d_stage[0] && d_stage[1] && d_best_key, "bb_score_fused_host: staging buffers / key missing");
  BB_CHECK_ARG(stream != copy, "bb_score_fused_host: the copy stream must differ from the compute stream");
  const int d = m->d;
  size_t row_bytes;
  int32_t dev_layout = BB_ROW_MAJOR_F32;
  int bits = 0;
  switch (host_format) {
    case BB_HOST_ROWS_F32: row_bytes = (size_t)ld * 4; dev_layout = BB_ROW_MAJOR_F32; break;
    case BB_HOST_ROWS_F64: row_bytes = (size_t)ld * 8; dev_layout = BB_ROW_MAJOR_F64; break;
    case BB_HOST_CODES4: row_bytes = (size_t)ld; bits = 4; break;
    case BB_HOST_CODES8: row_bytes = (size_t)ld; bits = 8; break;
    default: set_error("bb_score_fused_host: unknown host format %d", host_format); return BB_ERR_INVALID;
  }
  if (bits) {
    BB_CHECK_ARG(d_table && d_rows && d_rows[0] && d_rows[1], "bb_score_fused_host: value table / row buffers missing");
    BB_CHECK_ARG(ld >= (bits == 8 ? d : (d + 1) / 2), "bb_score_fused_host: code rows shorter than d columns");
  } else {
    BB_CHECK_ARG(ld >= d, "bb_score_fused_host: leading dimension smaller than d");
  }
  int rc = bb_best_init(d_best_key, stream);
  if (rc != BB_OK || N == 0) return rc;
  BB_CHECK_ARG(h_x != nullptr, "bb_score_fused_host: host matrix is null");
  cudaEvent_t ev[5];
  for (int i = 0; i < 5; ++i) BB_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
  cudaEvent_t* ready = ev;       // [2] block landed in its staging slot
  cudaEvent_t* freed = ev + 2;   // [2] staging slot consumed
  BB_CUDA(cudaEventRecord(ev[4], stream));  // staging buffers may still be in use by earlier work on `stream`
  BB_CUDA(cudaStreamWaitEvent(copy, ev[4], 0));
  rc = BB_OK;
  int b = 0;
  for (int64_t lo = 0; lo < N && rc == BB_OK; lo += block_rows, ++b) {
    const int64_t rows = (N - lo) < block_rows ? (N - lo) : block_rows;
    const int slot = b & 1;
    if (b >= 2) BB_CUDA(cudaStreamWaitEvent(copy, freed[slot], 0));
    BB_CUDA(cudaMemcpyAsync(d_stage[slot], reinterpret_cast<const uint8_t*>(h_x) + (size_t)lo * row_bytes,
                            (size_t)rows * row_bytes, cudaMemcpyHostToDevice, copy));
    BB_CUDA(cudaEventRecord(ready[slot], copy));
    BB_CUDA(cudaStreamWaitEvent(stream, ready[slot], 0));
    const void* x = d_stage[slot];
    int64_t ldx = ld;
    if (bits) {
      rc = bb_decode_codes(reinterpret_cast<const uint8_t*>(d_stage[slot]), bits, rows, d, ld, d_table, table_ld,
                           d_rows[slot], d, stream);
      if (rc != BB_OK) break;
      x = d_rows[slot];
      ldx = d;
    }
    rc = launch_fused(m, x, dev_layout, rows, ldx, a, d_z, S, d_keep ? d_keep + lo : nullptr, nullptr, nullptr,
                      d_score ? d_score + lo : nullptr, d_best_key, index_offset + lo, stream, nullptr, nullptr);
    if (rc != BB_OK) break;
    BB_CUDA(cudaEventRecord(freed[slot], stream));
  }
  for (int i = 0; i < 5; ++i) cudaEventDestroy(ev[i]);
  return rc;
}


// ------------------------------------------------------------------------------------------------------------
// bb_score_fused_overlapped -- the end-to-end pass as ONE kernel launch.
//
// The fused kernel is launched first, over all N rows of a device staging buffer that is still EMPTY; the host
// matrix then follows on the copy stream in growing row blocks, and after each block the copy stream publishes the
// number of rows that have landed (cuStreamWriteValue32 into *d_ready -- a stream-ordered memory operation, no
// kernel: every SM is occupied by the persistent scoring kernel).  The kernel's conversion warps take tiles in row
// order and wait (ld.acquire.sys) until their tile is published, so scoring proceeds at the pace of the PCIe copy
// and the pass costs max(copy, compute) plus the first block's latency, with no per-block launch, decode kernel or
// fp32 intermediate: level codes are expanded in the kernel's staging step.  Shapes outside the headline kernel's
// envelope return BB_ERR_UNSUPPORTED before anything is enqueued (callers then use bb_score_fused_host).
// ------------------------------------------------------------------------------------------------------------
typedef CUresult (*WriteValue32Fn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
// growing copy blocks: 32 k rows first (the kernel idles until they land), then x4 up to 2 M rows per block -- four
// blocks for 1M rows.  Every block costs a copy + a publication, each with its own DMA start-up latency.
constexpr int64_t kGateFirstBlock = 32768, kGateMaxBlock = 2097152;

extern "C" int bb_score_fused_overlapped(const bb_model* m, const bb_acq_spec* a, const void* h_x, int32_t host_format,
                                         int64_t N, int64_t ld, const float* d_table, int32_t table_ld, void* d_stage,
                                         int64_t stage_bytes, uint32_t* d_ready, int32_t* d_status,
                                         const uint8_t* d_keep, const float* d_z, int32_t S, float* d_score,
                                         int64_t* d_best_key, int64_t index_offset, void* stream_,
                                         void* copy_stream_) {
  cudaStream_t stream = (cudaStream_t)stream_, copy = (cudaStream_t)copy_stream_;
  BB_CHECK_ARG(m && m->abi_version == BB_ABI_VERSION && a, "bb_score_fused_overlapped: model / acquisition spec missing");
  BB_CHECK_ARG(N >= 0 && N < (1ll << 32), "bb_score_fused_overlapped: row count outside the 32-bit publication counter");
  BB_CHECK_ARG(d_stage && d_ready && d_status && d_best_key, "bb_score_fused_overlapped: staging / counter / status / key missing");
  BB_CHECK_ARG(stream != copy, "bb_score_fused_overlapped: the copy stream must differ from the compute stream");
  const int d = m->d;
  size_t row_bytes;
  StreamGate gate;
  gate.ready_rows = d_ready;
  gate.status = d_status;
  gate.code_table = d_table;
  gate.code_table_ld = table_ld;
  switch (host_format) {
    case BB_HOST_ROWS_F32: row_bytes = (size_t)ld * 4; gate.layout = BB_ROW_MAJOR_F32; gate.code_table = nullptr; break;
    case BB_HOST_CODES4: row_bytes = (size_t)ld; gate.layout = kLayoutCodes4; break;
    case BB_HOST_CODES8: row_bytes = (size_t)ld; gate.layout = kLayoutCodes8; break;
    default:
      set_error("bb_score_fused_overlapped: host format %d is not covered (float64 rows: bb_score_fused_host)", host_format);
      return BB_ERR_UNSUPPORTED;
  }
  if (gate.layout >= kLayoutCodes4) {
    const int bits = gate.layout == kLayoutCodes4 ? 4 : 8;
    BB_CHECK_ARG(d_table && table_ld >= 1 && table_ld <= (1 << bits), "bb_score_fused_overlapped: value table missing / too wide");
    BB_CHECK_ARG(ld >= (bits == 8 ? d : (d + 1) / 2), "bb_score_fused_overlapped: code rows shorter than d columns");
  } else {
    BB_CHECK_ARG(ld >= d, "bb_score_fused_overlapped: leading dimension smaller than d");
  }
  BB_CHECK_ARG((int64_t)(row_bytes * (size_t)N) <= stage_bytes, "bb_score_fused_overlapped: staging buffer too small");
  BB_CHECK_SUPPORTED(fused_gate_supported(m), "bb_score_fused_overlapped: shape outside the headline kernel's envelope");
  static WriteValue32Fn write32 = nullptr;
  if (write32 == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    BB_CUDA(cudaGetDriverEntryPoint("cuStreamWriteValue32", &fn, cudaEnableDefault, &qres));
    BB_CHECK_SUPPORTED(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuStreamWriteValue32 is not available");
    write32 = reinterpret_cast<WriteValue32Fn>(fn);
  }
  // How the copy stream publishes "rows landed":
  //   0  a 4-byte H2D copy from a constant pinned table of cumulative block ends (plain DMA, ordered behind the
  //      block's copy on the same stream): default
  //   1  cuStreamWriteValue32 (stream-ordered memory operation with a system-wide memory barrier in front)
  // Issued while earlier work is still draining on the compute stream, as in bench.py's timed loop, the write-value
  // form can serialise the pass behind that work.  BB_GATE_PUBLISH=1 selects it for diagnosis.
  static const int publish_mode = [] {
    const char* e = getenv("BB_GATE_PUBLISH");
    return (e != nullptr && e[0] == '1') ? 1 : 0;
  }();
  constexpr int kMaxBlocks = 64;
  static uint32_t* h_ends = nullptr;  // pinned, written once: cumulative ends of the growing-block schedule
  if (h_ends == nullptr) {
    uint32_t* t = nullptr;
    BB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&t), kMaxBlocks * sizeof(uint32_t), cudaHostAllocDefault));
    uint64_t end = 0, rows_k = kGateFirstBlock;
    for (int k = 0; k < kMaxBlocks; ++k) {
      end += rows_k;
      t[k] = end > 0xffffffffull ? 0xffffffffu : (uint32_t)end;  // a value >= N publishes everything
      if (rows_k < kGateMaxBlock) rows_k *= 4;
    }
    h_ends = t;
  }
  auto publish = [&](cudaStream_t st, int block, uint32_t rows_landed) -> bool {
    if (publish_mode == 0 && block >= 0 && block < kMaxBlocks)
      return cudaMemcpyAsync(d_ready, h_ends + block, sizeof(uint32_t), cudaMemcpyHostToDevice, st) == cudaSuccess;
    return write32((CUstream)st, (CUdeviceptr)(uintptr_t)d_ready, (cuuint32_t)rows_landed, 0u) == CUDA_SUCCESS;
  };
  int rc = bb_best_init(d_best_key, stream);
  if (rc != BB_OK || N == 0) return rc;
  BB_CHECK_ARG(h_x != nullptr, "bb_score_fused_overlapped: host matrix is null");
  // counter and status back to zero on the compute stream, ahead of the kernel and (through the event) of the copies
  // (every driver call counts here: the pass is ~0.3 ms of GPU work, a call ~5 us of host time)
  if (reinterpret_cast<uint8_t*>(d_status) == reinterpret_cast<uint8_t*>(d_ready) + 4) {
    BB_CUDA(cudaMemsetAsync(d_ready, 0, 8, stream));  // adjacent words: one operation
  } else {
    BB_CUDA(cudaMemsetAsync(d_status, 0, sizeof(int32_t), stream));
    BB_CUDA(cudaMemsetAsync(d_ready, 0, sizeof(uint32_t), stream));
  }
  static thread_local cudaEvent_t ev = nullptr;  // one event per host thread, re-recorded every pass
  static thread_local int ev_dev = -1;
  int dev_now = 0;
  BB_CUDA(cudaGetDevice(&dev_now));
  if (ev == nullptr || ev_dev != dev_now) {
    BB_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    ev_dev = dev_now;
  }
  BB_CUDA(cudaEventRecord(ev, stream));  // earlier readers of the staging buffer are done; the counter is reset
  BB_CUDA(cudaStreamWaitEvent(copy, ev, 0));
  rc = launch_fused(m, d_stage, BB_ROW_MAJOR_F32, N, ld, a, d_z, S, d_keep, nullptr, nullptr, d_score, d_best_key,
                    index_offset, stream, nullptr, &gate);
  if (rc != BB_OK) return rc;  // no kernel was launched: nothing waits for rows
  // block k ends at h_ends[k] (or N)
  int64_t lo = 0, rows = kGateFirstBlock;
  for (int k = 0; lo < N; ++k) {
    const int64_t n = (N - lo) < rows ? (N - lo) : rows;
    const cudaError_t e = cudaMemcpyAsync(reinterpret_cast<uint8_t*>(d_stage) + (size_t)lo * row_bytes,
                                          reinterpret_cast<const uint8_t*>(h_x) + (size_t)lo * row_bytes,
                                          (size_t)n * row_bytes, cudaMemcpyHostToDevice, copy);
    lo += n;
    // publish even after a failed copy (everything): the kernel must never be left waiting
    const bool w = (e == cudaSuccess) ? publish(copy, k, (uint32_t)lo) : publish(copy, -1, 0xffffffffu);
    if (e != cudaSuccess || !w) {
      if (!w) write32((CUstream)copy, (CUdeviceptr)(uintptr_t)d_ready, 0xffffffffu, 0u);
      set_error("bb_score_fused_overlapped: host->device copy / publication failed: %s", cudaGetErrorString(e));
      return BB_ERR_CUDA;
    }
    if (rows < kGateMaxBlock) rows *= 4;
  }
  return BB_OK;
}
