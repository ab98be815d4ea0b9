// boxdec.cu -- exact box decompositions of the region a small point set does not dominate, one per sample
// (qNoisyExpectedHypervolumeImprovement: the front itself is sampled, so every greedy round needs S of them).
//
// The decomposition is the one baybe_b200.multiobjective.box_decomposition builds on the host, box for box:
//   F    = the distinct points strictly above ref in every output that no other such point weakly dominates;
//   grid = one column per cell of the grid over the sorted distinct coordinates {ref_m} u F_m of the first M - 1
//          outputs (the last column of an output open to +inf); the column's box is [lo, hi) x [h, +inf), h = the
//          largest last output of the points that cover the column's upper corner (f_m >= hi_m for m < M - 1), else
//          ref_{M-1};
//   then the boxes that touch along output j and share every other bound are joined, for j = M - 2 down to 0.
// Every bound is a coordinate of a point or of ref, so the kernel keeps a box as small integers: for each output its
// upper index into the sorted axis (the lower index is the box's corner cell) and the index of h on the sorted last
// output.  One CTA per sample; the grid of at most 32^(M-1) cells lives in shared memory, one 32-bit word per cell.
// A merge along j is a pass over the cells: a live box whose upper face on j is the lower face of the box cornered at
// that cell (same corner on the other outputs, same upper indices and h) marks that box as a non-head; then every
// head walks its chain of non-heads (at most 32 steps) and takes the last one's upper index, and the non-heads die.
// Only comparisons and copies produce the bounds: they are the float32 points and the (rounded) float64 ref exactly.
// The hypervolume of F is summed in float64 over the finite columns before the merges.
#include <math.h>

#include "common.cuh"

namespace bb {

constexpr int kDecThreads = 512;
constexpr int kDecAxis = BB_MAX_PENDING + 1;  // ref and at most 31 points per output
constexpr uint32_t kDead = 1u << 30, kNonHead = 1u << 31;
constexpr int kHShift = 18;                   // cell word: upper index of output m at bits 6m (m < 3), h at 18

struct DecParams {
  const float* pts;       // [S][n][M]
  const int32_t* n_pts;   // [S] or null
  float* lower;           // [S][C][M]
  float* upper;
  int32_t* n_cells;       // [S]
  double* hv;             // [S]
  double ref[BB_HVI_MAX_TARGETS];
  int n, C;
};

__device__ __forceinline__ int upper_idx(uint32_t w, int m) { return (int)((w >> (6 * m)) & 63u); }

template <int M>
__global__ void __launch_bounds__(kDecThreads) k_boxdec(const DecParams p) {
  extern __shared__ __align__(16) uint32_t cell[];  // [A_0][A_1]...[A_{M-2}], the last grid output fastest
  __shared__ double axis[M][kDecAxis];
  __shared__ double ref[M];
  __shared__ float pt[kDecAxis][M];
  __shared__ uint8_t pidx[kDecAxis][M];             // front point f, output m -> index on axis m
  __shared__ uint8_t first[M][kDecAxis];
  __shared__ int keep[kDecAxis];
  __shared__ int nF, A[M];
  __shared__ int warp_live[kDecThreads / 32];
  __shared__ double red[kDecThreads / 32];
  const int s = blockIdx.x, t = threadIdx.x;
  const int n = p.n_pts ? min(max(__ldg(p.n_pts + s), 0), p.n) : p.n;
  const float* src = p.pts + (size_t)s * p.n * M;
  for (int e = t; e < n * M; e += blockDim.x) pt[e / M][e % M] = __ldg(src + e);
  if (t == 0) {  // indexed at run time below: a shared copy, not a local copy of the parameters
#pragma unroll
    for (int m = 0; m < M; ++m) ref[m] = p.ref[m];
  }
  __syncthreads();

  // the front: strictly above ref, first of its duplicates, weakly dominated by no other point
  if (t < n) {
    bool ok = true;
#pragma unroll
    for (int m = 0; m < M; ++m) ok &= (double)pt[t][m] > ref[m];
    for (int j = 0; ok && j < n; ++j) {
      if (j == t) continue;
      bool vj = true, ge = true, eq = true;
#pragma unroll
      for (int m = 0; m < M; ++m) {
        vj &= (double)pt[j][m] > ref[m];
        ge &= pt[j][m] >= pt[t][m];
        eq &= pt[j][m] == pt[t][m];
      }
      if (vj && (eq ? j < t : ge)) ok = false;
    }
    keep[t] = ok;
  }
  __syncthreads();
  if (t == 0) {
    int k = 0;
    for (int i = 0; i < n; ++i) {
      if (!keep[i]) continue;
#pragma unroll
      for (int m = 0; m < M; ++m) pt[k][m] = pt[i][m];  // k <= i: an in-place compaction
      ++k;
    }
    nF = k;
  }
  __syncthreads();

  // sorted distinct axes {ref_m} u F_m: value k = 0 is ref, k >= 1 point k - 1
  const int nv = nF + 1;
  auto value = [&](int m, int k) -> double { return k == 0 ? ref[m] : (double)pt[k - 1][m]; };
  for (int e = t; e < M * nv; e += blockDim.x) {
    const int m = e / nv, k = e - m * nv;
    const double v = value(m, k);
    bool f = true;
    for (int k2 = 0; k2 < k; ++k2) f &= value(m, k2) != v;
    first[m][k] = f;
  }
  __syncthreads();
  for (int e = t; e < M * nv; e += blockDim.x) {
    const int m = e / nv, k = e - m * nv;
    const double v = value(m, k);
    int rank = 0, distinct = 0;
    for (int k2 = 0; k2 < nv; ++k2) {
      rank += first[m][k2] && value(m, k2) < v;
      distinct += first[m][k2];
    }
    if (first[m][k]) axis[m][rank] = v;
    if (k > 0) pidx[k - 1][m] = (uint8_t)rank;
    if (k == 0) A[m] = distinct;
  }
  __syncthreads();

  // one box per grid column, and the hypervolume over the finite columns
  int G = 1;
#pragma unroll
  for (int m = 0; m < M - 1; ++m) G *= A[m];
  double acc = 0.0;
  for (int c = t; c < G; c += blockDim.x) {
    int i[M - 1];
    int r = c;
#pragma unroll
    for (int m = M - 2; m >= 0; --m) {
      i[m] = r % A[m];
      r /= A[m];
    }
    int h = 0;
    for (int f = 0; f < nF; ++f) {
      bool cov = true;
#pragma unroll
      for (int m = 0; m < M - 1; ++m) cov &= (int)pidx[f][m] > i[m];
      if (cov) h = max(h, (int)pidx[f][M - 1]);
    }
    uint32_t w = (uint32_t)h << kHShift;
    bool finite = true;
    double vol = axis[M - 1][h] - axis[M - 1][0];
#pragma unroll
    for (int m = 0; m < M - 1; ++m) {
      w |= (uint32_t)(i[m] + 1) << (6 * m);
      finite &= i[m] + 1 < A[m];
      if (i[m] + 1 < A[m]) vol *= axis[m][i[m] + 1] - axis[m][i[m]];
    }
    if (finite) acc += vol;
    cell[c] = w;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((t & 31) == 0) red[t >> 5] = acc;
  __syncthreads();  // also publishes the cells

  // joins along output j = M - 2 .. 0
  for (int j = M - 2; j >= 0; --j) {
    int stride = 1;
    for (int m = j + 1; m < M - 1; ++m) stride *= A[m];
    const int Aj = A[j];
    const uint32_t field = 63u << (6 * j), same = ((1u << (kHShift + 6)) - 1u) & ~field;
    for (int c = t; c < G; c += blockDim.x) {
      const uint32_t w = cell[c];
      if (w & kDead) continue;
      const int cj = (c / stride) % Aj, b = upper_idx(w, j);
      if (b >= Aj) continue;
      const int c2 = c + (b - cj) * stride;
      const uint32_t w2 = cell[c2];
      if (!(w2 & kDead) && ((w ^ w2) & same) == 0) atomicOr(cell + c2, kNonHead);
    }
    __syncthreads();
    for (int c = t; c < G; c += blockDim.x) {
      const uint32_t w = cell[c];
      if (w & (kDead | kNonHead)) continue;
      const int cj = (c / stride) % Aj;
      int b = upper_idx(w, j);
      while (b < Aj) {
        const uint32_t w2 = *(volatile uint32_t*)(cell + c + (b - cj) * stride);
        if (!(w2 & kNonHead)) break;
        b = upper_idx(w2, j);
      }
      if (b != upper_idx(w, j)) cell[c] = (w & ~field) | ((uint32_t)b << (6 * j));
    }
    __syncthreads();
    for (int c = t; c < G; c += blockDim.x)
      if (cell[c] & kNonHead) cell[c] = kDead;
    __syncthreads();
  }

  // the surviving boxes in cell order, decoded to float bounds: a block-wide scan of the live flags gives every box
  // its slot, so the same points always give the same layout (bb_hvi_score sums the cells in that order)
  const float inf = __int_as_float(0x7f800000);
  float* lo_s = p.lower + (size_t)s * p.C * M;
  float* up_s = p.upper + (size_t)s * p.C * M;
  const int lane = t & 31, warp = t >> 5;
  int n_boxes = 0;  // boxes in the cells before c0, the same in every thread
  for (int c0 = 0; c0 < G; c0 += kDecThreads) {
    const int c = c0 + t;
    const uint32_t w = c < G ? cell[c] : kDead;
    const bool live = !(w & kDead);
    const unsigned ballot = __ballot_sync(0xffffffffu, live);
    if (lane == 0) warp_live[warp] = __popc(ballot);
    __syncthreads();
    int slot = n_boxes + __popc(ballot & ((1u << lane) - 1u));
    for (int k = 0; k < kDecThreads / 32; ++k) {
      const int v = warp_live[k];
      slot += k < warp ? v : 0;
      n_boxes += v;
    }
    __syncthreads();  // warp_live is rewritten by the next chunk
    if (!live || slot >= p.C) continue;  // past the stride the count still grows: the caller sees the overflow
    int r = c;
#pragma unroll
    for (int m = M - 2; m >= 0; --m) {
      const int im = r % A[m], b = upper_idx(w, m);
      r /= A[m];
      lo_s[slot * M + m] = (float)axis[m][im];
      up_s[slot * M + m] = b < A[m] ? (float)axis[m][b] : inf;
    }
    lo_s[slot * M + M - 1] = (float)axis[M - 1][(w >> kHShift) & 63u];
    up_s[slot * M + M - 1] = inf;
  }
  if (t == 0) {
    double total = 0.0;
    for (int k = 0; k < kDecThreads / 32; ++k) total += red[k];
    p.n_cells[s] = n_boxes;
    p.hv[s] = total;
  }
}

template <int M>
static int launch_boxdec(const DecParams& p, int S, cudaStream_t stream) {
  size_t cells = 1;
  for (int m = 0; m < M - 1; ++m) cells *= (size_t)(p.n + 1);  // at most 32^3 words = 128 KB at M = 4
  const size_t smem = cells * 4;
  // always: without the opt-in the dynamic part may only take what the static part (about 2 KB) leaves of 48 KB
  BB_CUDA(cudaFuncSetAttribute(k_boxdec<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_boxdec<M><<<S, kDecThreads, smem, stream>>>(p);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

}  // namespace bb

using namespace bb;

extern "C" int bb_hvi_decompose(int32_t n_targets, const double* ref, int32_t S, int32_t n, const float* d_points,
                                const int32_t* d_n_points, int32_t cell_stride, float* d_lower, float* d_upper,
                                int32_t* d_n_cells, double* d_hv, void* stream) {
  BB_CHECK_SUPPORTED(n_targets >= 2 && n_targets <= BB_HVI_MAX_TARGETS,
                     "bb_hvi_decompose: n_targets=%d outside [2,%d]", n_targets, BB_HVI_MAX_TARGETS);
  BB_CHECK_ARG(ref != nullptr, "bb_hvi_decompose: null reference point");
  for (int m = 0; m < n_targets; ++m)
    BB_CHECK_ARG(isfinite(ref[m]), "bb_hvi_decompose: reference point of target %d not finite", m);
  BB_CHECK_ARG(S >= 1 && S <= 1024, "bb_hvi_decompose: S=%d outside [1,1024]", S);
  BB_CHECK_ARG(n >= 0 && n <= BB_MAX_PENDING, "bb_hvi_decompose: n=%d outside [0,%d]", n, BB_MAX_PENDING);
  BB_CHECK_SUPPORTED(cell_stride >= 1 && cell_stride <= BB_HVI_MAX_CELLS,
                     "bb_hvi_decompose: cell_stride=%d outside [1,%d]", cell_stride, BB_HVI_MAX_CELLS);
  BB_CHECK_ARG(d_lower && d_upper && d_n_cells && d_hv, "bb_hvi_decompose: null output buffer");
  BB_CHECK_ARG(n == 0 || d_points, "bb_hvi_decompose: null points");
  DecParams p{};
  p.pts = d_points;
  p.n_pts = d_n_points;
  p.lower = d_lower;
  p.upper = d_upper;
  p.n_cells = d_n_cells;
  p.hv = d_hv;
  for (int m = 0; m < n_targets; ++m) p.ref[m] = ref[m];
  p.n = n;
  p.C = cell_stride;
  cudaStream_t st = (cudaStream_t)stream;
  switch (n_targets) {
    case 2: return launch_boxdec<2>(p, S, st);
    case 3: return launch_boxdec<3>(p, S, st);
    default: return launch_boxdec<4>(p, S, st);
  }
}
