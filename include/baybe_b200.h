/*
 * baybe_b200.h -- C ABI of libbaybe_b200.so: the H100-native (sm_90a) replacement for the
 * recommend-time hot path of emdgroup/baybe (GP posterior over a full discrete candidate set
 * + acquisition scoring + arg-max / top-k).
 *
 * The reference has no FFI for this path: it calls into BoTorch/GPyTorch (Python).  Each entry
 * point below cites the reference call site whose work it replaces (paths under
 * /root/reference); INTEGRATION.md shows the ctypes binding a BayBE maintainer would add.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch types.
 *   - every pointer named d_* is a DEVICE pointer owned by the caller; the library never
 *     allocates or frees device memory and keeps no global mutable state except a
 *     thread-local error string.
 *   - every call takes the caller's CUDA stream (a cudaStream_t passed as void*), enqueues
 *     its kernels there and returns without synchronising, EXCEPT bb_model_build which
 *     synchronises the stream once (Cholesky success flag / jitter escalation).
 *   - a wide-feature model (bb_model.wide) owns scratch inside its blob (K* block, pending-point images):
 *     calls that use the same bb_model must be ordered on one stream (or serialised by the caller).
 *   - return value: BB_OK (0) or a negative bb_status; bb_last_error() gives the message.
 *     No partial results: on error the output buffers are unspecified.
 */
#ifndef BAYBE_B200_H_
#define BAYBE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BB_ABI_VERSION 4

typedef enum bb_status {
  BB_OK = 0,
  BB_ERR_INVALID = -1,     /* bad argument (shape, enum, null pointer, alignment)      */
  BB_ERR_UNSUPPORTED = -2, /* valid request outside what this build implements         */
  BB_ERR_CUDA = -3,        /* a CUDA runtime call or kernel launch failed              */
  BB_ERR_NOT_PD = -4,      /* K + noise*I not positive definite after jitter escalation */
  BB_ERR_WORKSPACE = -5    /* caller-provided buffer too small                         */
} bb_status;

/* Kernel family: baybe/kernels/basic.py:48 (MaternKernel nu), :166 (RBFKernel). */
typedef enum bb_kernel_family {
  BB_KERNEL_MATERN12 = 0,
  BB_KERNEL_MATERN32 = 1,
  BB_KERNEL_MATERN52 = 2,
  BB_KERNEL_RBF = 3
} bb_kernel_family;

/* Candidate-matrix layouts.  COL_MAJOR_F64 is what the reference hands to BoTorch today
 * (baybe/utils/dataframe.py:68-81 -> float64, strides (1,N)). */
typedef enum bb_layout {
  BB_ROW_MAJOR_F32 = 0,
  BB_COL_MAJOR_F32 = 1,
  BB_ROW_MAJOR_F64 = 2,
  BB_COL_MAJOR_F64 = 3,
  BB_BITS_U8 = 4 /* bit-packed binary features (substance fingerprints, BASELINE config 4): row r is
                    ldx BYTES at d_x + r*ldx, feature j = (byte[j>>3] >> (j&7)) & 1; wide models only */
} bb_layout;

/* Acquisition kinds, named by the reference's abbreviations (baybe/acquisition/acqfs.py). */
typedef enum bb_acq_kind {
  BB_ACQ_QLOGEI = 0, /* qLogExpectedImprovement   acqfs.py:220 */
  BB_ACQ_QEI = 1,    /* qExpectedImprovement      acqfs.py:206 */
  BB_ACQ_QUCB = 2,   /* qUpperConfidenceBound     acqfs.py:283 */
  BB_ACQ_QSR = 3,    /* qSimpleRegret             acqfs.py:190 */
  BB_ACQ_QPI = 4,    /* qProbabilityOfImprovement acqfs.py:256 */
  BB_ACQ_UCB = 5,    /* UpperConfidenceBound      acqfs.py:265 */
  BB_ACQ_EI = 6,     /* ExpectedImprovement       acqfs.py:199 */
  BB_ACQ_LOGEI = 7,  /* LogExpectedImprovement    acqfs.py:213 */
  BB_ACQ_PI = 8,     /* ProbabilityOfImprovement  acqfs.py:249 */
  BB_ACQ_PM = 9,     /* PosteriorMean             acqfs.py:162 */
  BB_ACQ_PSTD = 10,  /* PosteriorStandardDeviation acqfs.py:169 */
  BB_ACQ_QEHVI = 11,   /* qExpectedHypervolumeImprovement    acqfs.py:430 (bb_hvi_score only) */
  BB_ACQ_QLOGEHVI = 12 /* qLogExpectedHypervolumeImprovement acqfs.py:448 (bb_hvi_score only) */
} bb_acq_kind;

#define BB_MAX_PENDING 31 /* max pending points in a joint (q>1) evaluation */
#define BB_MAX_TRAIN 1024 /* max training points of this build (gpytorch switches away from exact Cholesky
                             above 800); n > 512 always takes the wide-feature path (K* block + K*-reading kernel) */

/*
 * Description of a fitted GP, i.e. what botorch.models.SingleTaskGP holds after
 * GaussianProcessSurrogate._fit (baybe/surrogates/gaussian_process/core.py:272-341).
 * All pointers are HOST pointers to float64 data (these are a few KB).
 */
typedef struct bb_model_desc {
  int32_t n;              /* training points                                              */
  int32_t d;              /* comp-rep columns (searchspace.comp_rep_columns)               */
  int32_t family;         /* bb_kernel_family                                              */
  int32_t task_col;       /* comp-rep column of the TaskParameter, or -1 (core.py:104-111) */
  int32_t n_tasks;        /* T (1 without a task parameter)                                */
  int32_t has_outputscale;/* ScaleKernel present (kernels/composite.py:21)                 */
  double outputscale;     /* s_f^2 (ignored unless has_outputscale)                        */
  const double* train_x;  /* [n*d] row-major raw comp-rep training inputs                  */
  const double* train_y;  /* [n]   raw targets                                             */
  const double* lower;    /* [d]   searchspace.scaling_bounds lower row (core.py:98-102)   */
  const double* upper;    /* [d]   upper row                                               */
  const double* lengthscale; /* [d] ARD lengthscale per column; <=0 marks an inactive column
                                (kernels/base.py:223-240); ignored for task_col            */
  const double* noise;    /* [T] likelihood noise per task (floored at 1e-4)               */
  const double* mean_const; /* [T] constant mean per task, standardised units              */
  const double* task_covar; /* [T*T] evaluated PositiveIndexKernel matrix, or NULL         */
} bb_model_desc;

/*
 * Device-resident model caches (what GPyTorch's prediction strategy caches: alpha, the
 * inverse root R = L^-T, plus our fp16 hi/lo tensor-core image of it).  Filled by
 * bb_model_build; the pointers point INTO the caller-owned blob.
 *
 * Concurrency: the caches are read-only after the build, but the blob also holds per-call SCRATCH -- the K* block
 * and pending-point images of the wide-feature path and the per-call qLogEI table (d_mc_table).  Calls that use one
 * bb_model must therefore be ordered on ONE stream (or externally serialised); two streams need two models (two
 * blobs built from the same bb_model_desc).
 */
typedef struct bb_model {
  int32_t abi_version;
  int32_t n, n_pad, d, d_pad;
  int32_t family, task_col, n_tasks;
  int32_t n_chunks;          /* n_pad / 64                                               */
  int32_t jitter_tries;      /* 0 = plain Cholesky succeeded                             */
  float y_mean, y_std;       /* Standardize(1) statistics                                */
  float prior_scale;         /* s_f^2 (1 without ScaleKernel)                            */
  float r_scale;             /* power of two folded into the fp16 image of L^-1          */
  double jitter;             /* jitter finally added to the diagonal                     */
  void* d_blob;              /* base of the caller-owned blob                            */
  size_t blob_bytes;
  const float* d_cand_scale; /* [d_pad] a_j = x_j*scale_j + shift_j (normalise, centre, 1/l) */
  const float* d_cand_shift; /* [d_pad]                                                   */
  const float* d_train_m2;   /* [n_pad*d_pad] -2 * scaled training rows (0 in padding)    */
  const float* d_train_sq;   /* [n_pad] squared norms of the scaled training rows         */
  const float* d_alpha;      /* [n_pad] K^-1 (y~ - c), fp32                               */
  const int32_t* d_train_task; /* [n_pad]                                                 */
  const float* d_task_covar; /* [T*T] fp32, prior_scale folded in                         */
  const float* d_mean_const; /* [T]                                                       */
  const void* d_rimg;        /* fp16 hi/lo swizzled tiles of L^-1 (wgmma B operand)       */
  const double* d_linv;      /* [n*n] row-major L^-1, float64                             */
  const double* d_alpha64;   /* [n]                                                       */
  const double* d_xn64;      /* [n*d] normalised training inputs, float64                 */
  const float* d_linv32;     /* [n_pad*n_pad] row-major L^-1, fp32 (zero padded)          */
  float dist_scale_a;        /* power-of-two scales folded into the fp16 images of the      */
  float dist_scale_b;        /* candidate rows (a) and training rows (b)                    */
  /* wide-feature path (n_pad*d_pad*4 > 56 KB, e.g. fingerprint spaces): K-chunked operand images of
   * the tensor-core distance GEMM and a K* workspace (whole waves, <= 40 MB up to n_pad = 640), all inside the blob */
  int32_t wide;              /* 1: scoring runs k_kmat_wg + the K*-reading posterior kernel     */
  int32_t d_wide;            /* d rounded up to 32 (K extent of the images)                     */
  const void* d_wimg;        /* fp16 hi/mid/lo image of (-2 x) scaled training rows             */
  const void* d_wimg_bits;   /* same for the bit-linear form t = sum_j x_j W_ij + c_i           */
  const float* d_wnorm_bits; /* [n_pad] c_i                                                     */
  float* d_wide_ws;          /* [wide_ws_rows * n_pad] fp32 K* block                            */
  int64_t wide_ws_rows;
  float dist_scale_w;        /* power-of-two scale folded into d_wimg_bits                      */
  int32_t pad_;
  /* wide path, pending points (sequential greedy): scratch images of <=31 pending rows as extra K columns */
  void* d_pend_img;          /* [64 rows] K-chunked split image, rebuilt per bb_posterior call          */
  float* d_pend_norm;        /* [64]                                                                    */
  int32_t* d_pend_task;      /* [64]                                                                    */
  float* d_kpend_ws;         /* [wide_ws_rows * 64] k(x*, pending) block                                */
  float dist_scale_p;        /* power-of-two scales of the pending images (float form / bit-linear form) */
  float dist_scale_wp;
  float* d_mc_table;         /* [1024] per-call qLogEI table of the K*-reading kernel (acq_math.cuh)             */
  /* tensor-core distances (n_pad <= 256, d <= 62; NULL otherwise): augmented training image
   * and the power-of-two scales folded into it */
  const void* d_timg_b;      /* training rows [-2b | q | |b|^2 q'] as hi/mid/lo panels of dist_k k (SW64 / SW128)   */
  int32_t dist_k;            /* K extent of d_timg_b: 32 (d <= 30), 64 (d <= 62), 0 = none                        */
  float ts_sa;               /* candidate rows are multiplied by ts_sa                                             */
  float ts_aug_sq;           /* K column dist_k - 2 of the candidate tile = |a|^2 * ts_aug_sq                      */
  float ts_aug_one;          /* K column dist_k - 1 of the candidate tile = ts_aug_one                             */
  float ts_g;                /* accumulator * ts_g = scaled squared distance                                       */
  float ts_kscale;           /* K* is multiplied by ts_kscale before the fp16 hi/lo split                          */
} bb_model;

/* Acquisition context built by BotorchAcquisitionFunctionBuilder.build
 * (baybe/acquisition/_builder.py:195-265). */
typedef struct bb_acq_spec {
  int32_t kind;     /* bb_acq_kind                                                        */
  int32_t maximize; /* PSTD sign (acqfs.py:169-177)                                       */
  float best_f;     /* max_i o(mu(x_i)) over training inputs (_builder.py:256-265)        */
  float beta;       /* UCB/qUCB (acqfs.py:270,288)                                        */
  float obj_scale;  /* objective o = obj_scale*y + obj_shift (objectives/single.py:66-91) */
  float obj_shift;
  float tau_relu;   /* qLogEI fatplus temperature (botorch default 1e-6)                  */
  float tau_max;    /* qLogEI fatmax temperature (botorch default 1e-2)                   */
  float tau_pi;     /* qPI sigmoid temperature (botorch default 1e-3)                     */
} bb_acq_spec;

/* (value, index) of the best candidate of one shard; idx = -1 when nothing was eligible. */
typedef struct bb_best {
  float val;
  int32_t pad_;
  int64_t idx;
} bb_best;

int bb_abi_version(void);
const char* bb_last_error(void);

/* ---- training-side caches (K8): replaces the lazily cached Cholesky / alpha / inverse root
 * of gpytorch's DefaultPredictionStrategy reached from core.py:268-269, 331-341. ---------- */
size_t bb_model_blob_bytes(int32_t n, int32_t d, int32_t n_tasks);
int bb_model_build(const bb_model_desc* desc, void* d_blob, size_t blob_bytes, bb_model* out,
                   void* stream);

/* ---- hyper-parameter fit (SURVEY.md 8f-1): value and gradient of the exact marginal log likelihood that
 * GaussianProcessSurrogate._fit maximises through botorch.fit.fit_gpytorch_mll (core.py:331-341,
 * components/fit_criterion.py:22-41), float64 on device.  theta (HOST) = [lengthscale[d] | noise | mean
 * constant | task covariance B[T*T] (outputscale folded in; [1.0] without tasks)]; xn [n*d] are the
 * normalised ACTIVE columns, y [n] the standardised targets, task [n] task ids or NULL.  The priors and the
 * L-BFGS-B driver stay on the host (baybe_b200/surrogates.py).  bb_fit_eval synchronises the stream. ---- */
size_t bb_fit_workspace_bytes(int32_t n, int32_t d, int32_t n_tasks);
int bb_fit_setup(void* d_ws, size_t ws_bytes, int32_t n, int32_t d, int32_t n_tasks, const double* xn,
                 const double* y, const int32_t* task, void* stream);
int bb_fit_eval(void* d_ws, int32_t n, int32_t d, int32_t n_tasks, int32_t family, const double* theta,
                double* value, double* grad, int32_t* not_pd, void* stream);
/* Leave-one-out pseudo-likelihood (gpytorch.mlls.LeaveOneOutPseudoLikelihood), the criterion the reference's
 * presets select when the search space has a task parameter (presets/baybe.py:270-281,
 * components/fit_criterion.py:22-41): value = sum_i log N(y_i | mu_-i, sigma_-i^2), same theta / gradient layout. */
int bb_fit_eval_loo(void* d_ws, int32_t n, int32_t d, int32_t n_tasks, int32_t family, const double* theta,
                    double* value, double* grad, int32_t* not_pd, void* stream);

/* ---- K2: K(X*, X_train), fp32 row-major [N, ldk>=n].  Replaces gpytorch
 * MaternKernel/RBFKernel/ScaleKernel/ProductKernel.forward built at
 * baybe/kernels/base.py:173-178 and components/kernel.py:337. ---------------------------- */
int bb_kernel_matrix(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx,
                     float* d_k, int64_t ldk, void* stream);

/* ---- K2-K5: marginal posterior mean / variance of every candidate, original units.
 * Replaces SingleTaskGP.posterior(X.unsqueeze(-2)) reached from
 * GaussianProcessSurrogate._posterior (core.py:268-269), Surrogate.posterior_stats
 * (surrogates/base.py:308-384).  d_cross (nullable): [N, n_pending] posterior covariance with
 * the pending points, needs d_pend_beta = K^-1 k(X, pending) [n_pending, n_pad] fp32 (from
 * bb_pending_stats) and d_pend_x [n_pending, d] raw comp-rep rows (fp32 row-major). -------- */
int bb_posterior(const bb_model* m, const void* d_x, int32_t layout, int64_t N, int64_t ldx,
                 float* d_mu, float* d_var, float* d_cross, const float* d_pend_x,
                 const float* d_pend_beta, int32_t n_pending, void* stream);

/* ---- pending-point statistics for sequential greedy (K9 prologue): for P pending rows
 * (fp32 row-major raw comp-rep) returns beta = K^-1 k(X,P) [P, n_pad], the posterior mean [P]
 * and covariance [P,P] in original units (float64 math, fp32 outputs). --------------------- */
int bb_pending_stats(const bb_model* m, const float* d_pend_x, int32_t n_pending,
                     float* d_pend_beta, float* d_pend_mu, float* d_pend_cov, void* stream);

/* ---- joint posterior of R raw rows (fp32 row-major raw comp-rep, 1 <= R <= n_pad), float64 throughout: mean d_mu [R]
 * and full covariance d_cov [R][R] of the latent function in original units -- what the reference samples from when
 * it prunes the noisy-EI baseline (botorch prune_inferior_points on the measured rows, acquisition/_builder.py:
 * 319-324).  d_beta (nullable): [R][n_pad] fp32 beta = K^-1 k(X, x_r), as bb_pending_stats gives it, so that the
 * same rows can condition bb_posterior's cross covariance without a second pass.  The caller owns the float64
 * workspace d_ws of ws_doubles >= R * (n_pad + d) entries.  Unlike forming the covariance in fp32 from
 * bb_kernel_matrix, this does not cancel at noise-level variances. */
int bb_joint_posterior(const bb_model* m, const float* d_x, int32_t R, double* d_mu, double* d_cov, float* d_beta,
                       double* d_ws, size_t ws_doubles, void* stream);

/* ---- K6: acquisition value of each candidate as its own q=1 batch from (mu, var).
 * d_z: [S] shared Sobol-normal base samples (MC kinds; ignored for analytic kinds).
 * Replaces qLogExpectedImprovement.forward etc. (class picked at acquisition/base.py:162-181). */
int bb_acq_score(const bb_acq_spec* a, const float* d_mu, const float* d_var, int64_t N,
                 const float* d_z, int32_t S, float* d_score, void* stream);

/* ---- K9: joint MC acquisition value of [x*; pending] per candidate (sequential greedy,
 * candidate first -- botorch concatenate_pending_points).  d_z: [S, 1+P] row-major. -------- */
int bb_acq_score_joint(const bb_acq_spec* a, const float* d_mu, const float* d_var,
                       const float* d_cross, int64_t N, const float* d_pend_mu,
                       const float* d_pend_cov, int32_t n_pending, const float* d_z, int32_t S,
                       float* d_score, void* stream);

/* ---- K2-K7 fused: posterior + q=1 acquisition + running arg-max, K* never leaves the SM.
 * d_keep (nullable): uint8 [N], 0 = not eligible (already recommended / excluded).
 * d_score (nullable): per-candidate scores.  d_best_key: int64 packed (score, lowest index)
 * key, must be initialised with bb_best_init; combine shards with max(), decode with
 * bb_best_decode.  Replaces one round of botorch.optim.optimize_acqf_discrete
 * (baybe/recommenders/pure/bayesian/botorch/discrete.py:124-126). ------------------------- */
int bb_score_fused(const bb_model* m, const bb_acq_spec* a, const void* d_x, int32_t layout,
                   int64_t N, int64_t ldx, const uint8_t* d_keep, const float* d_z, int32_t S,
                   float* d_score, int64_t* d_best_key, int64_t index_offset, void* stream);

/* ---- K7: arg-max / top-k over a score vector (ties -> lowest index, as torch.argmax). ---- */
int bb_best_init(int64_t* d_best_key, void* stream);
int bb_argmax(const float* d_score, const uint8_t* d_keep, int64_t N, int64_t index_offset,
              int64_t* d_best_key, void* stream);
int bb_best_decode(const int64_t* d_best_key, bb_best* d_out, void* stream);
int bb_topk(const float* d_score, const uint8_t* d_keep, int64_t N, int32_t k, float* d_vals,
            int64_t* d_idx, uint8_t* d_scratch_mask /* [N] */, int64_t* d_scratch_key, void* stream);

/* ---- multi-GPU (SURVEY.md 8e): global arg-max of a row-sharded candidate set.  Every rank owns a small buffer of
 * two key slots (int64) and two arrival counters (uint32), double-buffered by epoch parity, initialised once with
 * bb_peer_slots_init; the ranks exchange the buffers' addresses with CUDA IPC (one process per GPU, NVLink peer
 * access) and fill bb_peer_group with their own and the mapped peer pointers.  bb_allreduce_best then runs ONE warp on
 * the caller's stream: atomicMax.sys of the local packed key into every rank's slot, a system fence, a bump of
 * every rank's counter, a bounded wait for `world` arrivals at the own counter, copy-out and re-arm.  No host
 * code and no NCCL call sits between the scoring kernel and the reduced key.  `epoch` must be the same on all ranks
 * and increase by one per call; *d_status = 1 if a peer did not arrive within ~11 s (d_out_key then holds the local
 * key).  Replaces torch.argmax over the full candidate set inside botorch.optim.optimize_acqf_discrete
 * (baybe/recommenders/pure/bayesian/botorch/discrete.py:124-126) for a candidate set sharded over GPUs. */
#define BB_MAX_PEERS 8
typedef struct bb_peer_group {
  int32_t rank, world;
  int64_t* d_key[BB_MAX_PEERS];    /* [r] -> two key slots in rank r's memory (own or IPC-mapped)      */
  uint32_t* d_count[BB_MAX_PEERS]; /* [r] -> two arrival counters in rank r's memory                   */
} bb_peer_group;
int bb_peer_slots_init(int64_t* d_keys /* [2] */, uint32_t* d_counts /* [2] */, void* stream);
int bb_allreduce_best(const bb_peer_group* g, const int64_t* d_local_key, uint32_t epoch, int64_t* d_out_key,
                      int32_t* d_status, void* stream);

/* ---- level-coded candidate rows (device-resident search-space cache, SURVEY.md 8f-3): a discrete search space has
 * few distinct values per comp-rep column (the parameters' value lists, baybe/searchspace/discrete.py:529-536), so
 * the host side may ship rows as `bits`-bit level codes (4: two columns per byte, low nibble = even column; 8: one
 * byte per column; row r at d_codes + r*ld_bytes) plus a value table d_table[d][table_ld] (fp32).  Expands to
 * fp32 row-major d_out[N][ldo]; exact (the table holds the comp-rep values).  Replaces shipping the float64
 * comp-rep matrix that SubspaceDiscrete.transform builds per call (botorch/discrete.py:123). */
int bb_decode_codes(const uint8_t* d_codes, int32_t bits, int64_t N, int32_t d, int64_t ld_bytes,
                    const float* d_table, int32_t table_ld, float* d_out, int64_t ldo, void* stream);

/* ---- end-to-end pass over a HOST-resident candidate set: blocks of block_rows rows (a multiple of 128) are copied
 * on `copy_stream` into two caller-owned staging buffers (d_stage[2], each block_rows * row bytes) while the previous
 * block is expanded (level codes -> d_rows[2], each block_rows * d floats) and scored by the fused kernel on `stream`.
 * h_x should be pinned; row r starts at h_x + r * row bytes (ld in ELEMENTS for the float formats, in BYTES for the
 * code formats).  Events are created and destroyed inside the call; nothing else is allocated.  Same results as
 * bb_score_fused on the device-resident matrix. */
typedef enum bb_host_format {
  BB_HOST_ROWS_F32 = 0, /* float32 rows                                  */
  BB_HOST_ROWS_F64 = 1, /* float64 rows (what the reference holds)       */
  BB_HOST_CODES4 = 2,   /* 4-bit level codes + value table (bb_decode_codes) */
  BB_HOST_CODES8 = 3    /* 8-bit level codes + value table               */
} bb_host_format;
int bb_score_fused_host(const bb_model* m, const bb_acq_spec* a, const void* h_x, int32_t host_format, int64_t N,
                        int64_t ld, const float* d_table, int32_t table_ld, void* const* d_stage,
                        float* const* d_rows, int64_t block_rows, const uint8_t* d_keep, const float* d_z, int32_t S,
                        float* d_score, int64_t* d_best_key, int64_t index_offset, void* stream, void* copy_stream);

/* ---- the same pass as ONE kernel launch (shapes of the headline kernel: n_pad <= 256, d <= 30, S <= 512; float32
 * rows or level codes).  The fused kernel is launched first over a device staging buffer (d_stage, stage_bytes >=
 * N * row bytes) that is still empty; the host matrix follows on `copy_stream` in growing row blocks, and after every
 * block the copy stream publishes the number of rows landed into *d_ready (cuStreamWriteValue32, no kernel).  The
 * kernel takes row tiles in order and waits (ld.acquire.sys on *d_ready) until its tile is published; level codes
 * are expanded in its staging step, so there is no per-block launch, decode kernel or fp32 intermediate and the
 * pass costs max(copy, compute) + the first block's latency.  *d_status is raised to 1 if rows were not published
 * within ~2 s (the kernel never hangs; the caller must treat the pass as failed).  Returns BB_ERR_UNSUPPORTED,
 * with nothing enqueued, for shapes / formats outside the envelope: fall back to bb_score_fused_host.
 * Replaces: the same reference path as bb_score_fused_host (botorch/discrete.py:120-126). */
int bb_score_fused_overlapped(const bb_model* m, const bb_acq_spec* a, const void* h_x, int32_t host_format, int64_t N,
                              int64_t ld, const float* d_table, int32_t table_ld, void* d_stage, int64_t stage_bytes,
                              uint32_t* d_ready, int32_t* d_status, const uint8_t* d_keep, const float* d_z, int32_t S,
                              float* d_score, int64_t* d_best_key, int64_t index_offset, void* stream,
                              void* copy_stream);

/* ---- noisy expected improvement of one new point per row, conditional on joint samples of C = [baseline; pending]
 * (qNoisyExpectedImprovement, baybe/acquisition/acqfs.py:227-232; X_baseline = training inputs,
 * acquisition/_builder.py:319-324; used by the hybrid recommender, recommenders/pure/bayesian/botorch/hybrid.py:30-161).
 * d_out [N, ld >= S + m]: row i = [ r_i . Z_C^T (S values) | r_i (m values) ] with r_i = Sigma_iC L_C^-T, produced by
 * the caller's GEMM; d_mu / d_var: marginal posterior of the rows (original units); d_zx [S]: the new point's own
 * base samples; d_g [S]: per-sample incumbent max(o over the samples of C).  score_i = mean_s relu(o(mu_i +
 * out_i[s] + sqrt(max(var_i - |r_i|^2, 0)) zx_s) - g_s), o(y) = obj_scale * y + obj_shift. */
int bb_nei_reduce(const float* d_out, int64_t ld, int32_t S, int32_t m, const float* d_mu, const float* d_var,
                  const float* d_zx, const float* d_g, float obj_scale, float obj_shift, int64_t N, float* d_score,
                  void* stream);

/* ---- hypervolume improvement of one new point per candidate for a Pareto objective of M targets
 * (qExpectedHypervolumeImprovement / qLogExpectedHypervolumeImprovement, baybe/acquisition/acqfs.py:430-465; reference
 * point and partitioning from acquisition/_builder.py:286-317, both built on the host by baybe_b200/multiobjective.py).
 * Kind BB_ACQ_QEHVI or BB_ACQ_QLOGEHVI (a->tau_relu / a->tau_max smooth the latter); a->obj_scale / obj_shift are not
 * used: obj_scale[M] / obj_shift[M] (HOST arrays) orient each target, o_m = obj_scale[m] * y_m + obj_shift[m].
 *   d_mu / d_var [M][N]: marginal posterior of every candidate per target (bb_posterior, one model per target).
 *   n_pending = P in [0, BB_MAX_PENDING].  With P > 0: d_cross [M][N][P] (bb_posterior's cross covariance),
 *     d_linv [M][P][P] = L_PP^-1 (row-major, lower triangular) and d_w [M][S][P] = L_PP^-T z_P of each target (pending Cholesky L_PP L_PP^T = K_PP).
 *   d_z [S][M(1+P)]: base samples; column m(1+P)+j is pending point j of target m, column m(1+P)+P the candidate.
 *   Cells: d_lower / d_upper [n_dec][cell_stride][M], d_n_cells [n_dec] (entries above cell_stride are clamped);
 *     n_dec = 1 (one decomposition of the front F, shared by all samples) for P = 0, else S (F u P_s per sample).
 *     An upper bound of +inf leaves that side open.  cell_stride <= BB_HVI_MAX_CELLS.
 * Writes the improvement of x over the cells (the pending points' own improvement is the caller's candidate-
 * independent term) to d_score (nullable), and folds d_keep (nullable) and index_offset into *d_best_key like
 * bb_argmax (initialise with bb_best_init).  S <= 1024; 2 <= M <= BB_HVI_MAX_TARGETS. */
#define BB_HVI_MAX_TARGETS 4
#define BB_HVI_MAX_CELLS 1024
int bb_hvi_score(const bb_acq_spec* a, int32_t n_targets, const float* obj_scale, const float* obj_shift, int64_t N,
                 const float* d_mu, const float* d_var, int32_t n_pending, const float* d_cross, const float* d_linv,
                 const float* d_w, const float* d_z, int32_t S, const float* d_lower, const float* d_upper,
                 const int32_t* d_n_cells, int32_t cell_stride, const uint8_t* d_keep, float* d_score,
                 int64_t* d_best_key, int64_t index_offset, void* stream);

/* ---- exact box decompositions of S small point sets, one per sample, in the layout bb_hvi_score reads
 * (qNoisyExpectedHypervolumeImprovement, whose front is sampled: acqfs.py:468-474 via botorch's
 * qNoisyExpectedHypervolumeImprovement; set-up on the host by baybe_b200/nehvi.py).  Maximisation.
 *   ref [n_targets]: HOST array of float64, finite; 2 <= n_targets <= BB_HVI_MAX_TARGETS.
 *   d_points [S][n][n_targets] float32, n in [0, BB_MAX_PENDING]; d_n_points [S] (nullable) uses only the first
 *     d_n_points[s] points of sample s (clamped to [0, n]).  S in [1, 1024].
 * For every sample: the points strictly above ref in every output, deduplicated, reduced to the non-dominated ones;
 * one box per column of the grid over their first n_targets - 1 outputs; then boxes that touch along output j and
 * share every other bound joined, for j = n_targets - 2 down to 0 -- the same set of boxes as
 * baybe_b200.multiobjective.box_decomposition of the same points (as float64), in the order of their lower corners
 * on the grid (the same points always give the same layout).  Writes the boxes to
 * d_lower / d_upper [S][cell_stride][n_targets] (+inf: an open side), their number to d_n_cells [S] and the
 * hypervolume of the points (float64) to d_hv [S].  A count above cell_stride (<= BB_HVI_MAX_CELLS) means the
 * decomposition did not fit: that sample's boxes are incomplete and the caller must not use them. */
int bb_hvi_decompose(int32_t n_targets, const double* ref, int32_t S, int32_t n, const float* d_points,
                     const int32_t* d_n_points, int32_t cell_stride, float* d_lower, float* d_upper,
                     int32_t* d_n_cells, double* d_hv, void* stream);

/* ---- Monte-Carlo (and, for affine MEAN desirability, analytic) acquisition values of an objective that is not
 * affine in the modelled targets: DesirabilityObjective (baybe/objectives/desirability.py:229-264, weighted MEAN or
 * geometric mean of per-target transformations) and single targets with a non-affine transformation
 * (objectives/base.py:130-150), applied to posterior samples as the reference's MC acquisition functions do
 * (acquisition/_builder.py:211-254, ChainedMCObjective).  Each target m carries a postfix program over its sample
 * y_m (transformations/basic.py, composite.py; compiled on the host by baybe_b200/objectives.py), evaluated on an
 * evaluation stack of at most BB_OBJ_MAX_STACK entries whose top starts as y_m; t_m = the single entry left.
 * Then o = t_0 (NONE), sum_m w_m t_m (MEAN) or exp(sum_m w_m log(t_m + 2^-52)) (GEOM_MEAN), w normalised. */
#define BB_OBJ_MAX_TARGETS 8
#define BB_OBJ_MAX_OPS 32
#define BB_OBJ_MAX_STACK 4
typedef enum bb_obj_opcode {
  BB_OBJ_AFFINE = 0,    /* top = top * arg0 + arg1                                      (AffineTransformation)  */
  BB_OBJ_CONST = 1,     /* top = arg0                                                                         */
  BB_OBJ_CLAMP = 2,     /* top = clamp(top, arg0, arg1), +-inf leaves a side open, NaN stays (Clamping)      */
  BB_OBJ_TWO_SIDED = 3, /* d = top - arg2; top = d < 0 ? d * arg0 : d * arg1, a zero slope gives 0 (TwoSidedAffine) */
  BB_OBJ_BELL = 4,      /* top = exp(-((top - arg0) / arg1)^2 / 2)                         (BellTransformation) */
  BB_OBJ_LOG = 5,       /* top = log(top)                                           (LogarithmicTransformation) */
  BB_OBJ_EXP = 6,       /* top = exp(top)                                           (ExponentialTransformation) */
  BB_OBJ_POW_INT = 7,   /* top = top^arg0, arg0 integral                                  (PowerTransformation) */
  BB_OBJ_SIGMOID = 8,   /* top = 1 / (1 + exp(arg1 * (top - arg0)))                     (SigmoidTransformation) */
  BB_OBJ_DUP_INPUT = 9, /* push y_m (the second branch of an Additive / Multiplicative transformation)         */
  BB_OBJ_ADD = 10,      /* pop b, pop a, push a + b                                     (AdditiveTransformation) */
  BB_OBJ_MUL = 11       /* pop b, pop a, push a * b                               (MultiplicativeTransformation) */
} bb_obj_opcode;
typedef enum bb_obj_scalarizer {
  BB_OBJ_SCALAR_NONE = 0,     /* single target                                                               */
  BB_OBJ_SCALAR_MEAN = 1,     /* Scalarizer.MEAN      (LinearMCObjective(normalized_weights))                */
  BB_OBJ_SCALAR_GEOM_MEAN = 2 /* Scalarizer.GEOM_MEAN (_geometric_mean, desirability.py:41-70)              */
} bb_obj_scalarizer;
typedef struct bb_obj_instr {
  int32_t op; /* bb_obj_opcode */
  float arg[3];
} bb_obj_instr;
typedef struct bb_objective {
  int32_t n_targets;                          /* M in [1, BB_OBJ_MAX_TARGETS]                           */
  int32_t scalarizer;                         /* bb_obj_scalarizer                                      */
  int32_t n_ops[BB_OBJ_MAX_TARGETS];          /* program length per target (0: identity)                */
  float weight[BB_OBJ_MAX_TARGETS];           /* normalised weights (MEAN / GEOM_MEAN)                  */
  bb_obj_instr prog[BB_OBJ_MAX_TARGETS][BB_OBJ_MAX_OPS];
} bb_objective;

/* Kinds: BB_ACQ_QLOGEI / QEI / QPI / QSR / QUCB over the samples o_s of the objective; EI / LOGEI / PI / UCB / PM / PSTD
 * only for MEAN scalarisation with every program a single AFFINE op (or empty) and no pending point: the moments
 * sum_m w_m (a_m mu_m + b_m) and sum_m (w_m a_m)^2 var_m (desirability.py:266-320) go to the analytic formulas.
 *   d_mu / d_var [M][N]: marginal posterior of every candidate per target (bb_posterior, one model per target).
 *   d_z [S][M(1+P)]: base samples; column m(1+P)+j is pending point j of target m, column m(1+P)+P the candidate.
 *   n_pending = P in [0, BB_MAX_PENDING].  With P > 0: d_cross [M][N][P], d_linv [M][P][P] = L_PP^-1 and
 *     d_w [M][S][P] = L_PP^-T z_P per target (as bb_hvi_score): y_m = mu_m + c_m . w_{m,s} +
 *     sqrt(max(var_m - |L_m^-1 c_m|^2, 0)) z_{s, m(1+P)+P}; d_pend_terms [S][P]: the per-sample term of every pending
 *     point (qLogEI: log fatplus(o - best_f) with tau_relu; qEI: relu(o - best_f); qPI: sigmoid((o - best_f)/tau_pi);
 *     qSR: o; qUCB: m + sqrt(beta pi / 2) |o - m| with m the sample mean of that point's o).  The candidate's term
 *     joins them by max (qLogEI: fatmax with tau_max), like bb_acq_score_joint.
 * Writes the value of every candidate to d_score (nullable) and folds d_keep (nullable) and index_offset into
 * *d_best_key like bb_argmax (initialise with bb_best_init).  S in [1, 1024].  The objective is passed to the
 * kernel by value (no device copy): concurrent calls on different streams do not share state. */
int bb_objective_score(const bb_acq_spec* a, const bb_objective* obj, int64_t N, const float* d_mu, const float* d_var,
                       int32_t n_pending, const float* d_cross, const float* d_linv, const float* d_w,
                       const float* d_pend_terms, const float* d_z, int32_t S, const uint8_t* d_keep, float* d_score,
                       int64_t* d_best_key, int64_t index_offset, void* stream);

/* ---- noisy expected improvement of one new point per candidate of a discrete space (qNoisyExpectedImprovement,
 * log_nei = 0, or qLogNoisyExpectedImprovement, log_nei = 1; baybe/acquisition/acqfs.py:226-243; set-up on the host
 * by baybe_b200/noisy.py).  The conditioning set C (n_cond <= BB_MAX_PENDING points: the pruned baseline, the pending
 * points, then the n_batch other points of a q-batch) is sampled jointly by the caller:
 *   d_mu / d_var [N], d_cross [N][n_cond]: bb_posterior of the candidates with C as its pending points;
 *   d_linv [n_cond][n_cond] = L_C^-1 (row-major, lower triangular), L_C L_C^T = Sigma_CC;
 *   d_w [n_cond][S] = L_C^-T z_{s,C} stored sample-minor (entry (j, s) at j * S + s);
 *   d_z [S][n_cond + 1]: base samples, column n_cond the candidate's;
 *   d_g [S]: per-sample incumbent, the maximum of o over baseline and pending points;
 *   d_batch_terms [S][n_batch]: per-sample terms of the other batch points (nullable when n_batch = 0).
 * Per sample o_s = obj_scale * (mu + c . w_s + sqrt(max(var - |L_C^-1 c|^2, 0)) z_{s,n_cond}) + obj_shift and
 *   qNEI    : t_s = relu(o_s - g_s), joined with the batch terms by max, value = mean_s;
 *   qLogNEI : t_s = log tau_relu + log fatplus((o_s - g_s) / tau_relu), joined by fatmax (tau_max), value =
 *             logmeanexp_s.
 * Writes the value of every candidate to d_score (nullable) and folds d_keep (nullable) and index_offset into
 * *d_best_key like bb_argmax (initialise with bb_best_init).  S in [1, 1024]. */
int bb_nei_score(int32_t log_nei, float obj_scale, float obj_shift, float tau_relu, float tau_max, int64_t N,
                 const float* d_mu, const float* d_var, int32_t n_cond, const float* d_cross, const float* d_linv,
                 const float* d_w, const float* d_z, int32_t S, const float* d_g, int32_t n_batch,
                 const float* d_batch_terms, const uint8_t* d_keep, float* d_score, int64_t* d_best_key,
                 int64_t index_offset, void* stream);

/* ---- Pareto objectives by random Chebyshev scalarisation: qLogNParEGO (baybe/acquisition/acqfs.py:328-336, built
 * with X_baseline = the measured rows at acquisition/_builder.py:195-209, 319-334; set-up on the host by
 * baybe_b200/parego.py).  n_targets = M in [2, BB_OBJ_MAX_TARGETS], one model per target.  The host folds the oriented
 * target, its normalisation and the simplex weight into one affine map per target, p_m = weight[m] * y_m + offset[m]
 * (weight / offset: host arrays of M floats), and scalarises cheb = min_m p_m + alpha * sum_m p_m.  The conditioning
 * set C (n_cond <= BB_MAX_PENDING points: the pruned baseline, the pending points, then the n_batch other points of a
 * q-batch) is shared by the targets and sampled jointly per target by the caller:
 *   d_mu / d_var [M][N], d_cross [M][N][n_cond]: bb_posterior of the candidates per target model, C its pending points;
 *   d_linv [M][n_cond][n_cond] = L_C,m^-1 (row-major, lower triangular);
 *   d_w [M][n_cond][S] = L_C,m^-T z_{s,C,m} stored sample-minor (entry (m, j, s) at (m * n_cond + j) * S + s);
 *   d_z [S][M(n_cond + 1)]: base samples, column m(n_cond+1)+j conditioning point j of target m, m(n_cond+1)+n_cond
 *     the candidate's;
 *   d_g [S]: per-sample incumbent, the maximum of cheb over baseline and pending points;
 *   d_batch_terms [S][n_batch]: per-sample terms of the other batch points (nullable when n_batch = 0).
 * Per sample y_m = mu_m + c_m . w_m,s + sqrt(max(var_m - |L_C,m^-1 c_m|^2, 0)) z_{s,m(n_cond+1)+n_cond},
 *   t_s = log tau_relu + log fatplus((cheb_s - g_s) / tau_relu), joined with the batch terms by fatmax (tau_max),
 *   value = logmeanexp_s.
 * Writes the value of every candidate to d_score (nullable) and folds d_keep (nullable) and index_offset into
 * *d_best_key like bb_argmax (initialise with bb_best_init).  S in [1, 1024]. */
int bb_parego_score(int32_t n_targets, const float* weight, const float* offset, float alpha, float tau_relu,
                    float tau_max, int64_t N, const float* d_mu, const float* d_var, int32_t n_cond,
                    const float* d_cross, const float* d_linv, const float* d_w, const float* d_z, int32_t S,
                    const float* d_g, int32_t n_batch, const float* d_batch_terms, const uint8_t* d_keep,
                    float* d_score, int64_t* d_best_key, int64_t index_offset, void* stream);

/* ---- integrated posterior variance reduction for global active learning (qNegIntegratedPosteriorVariance,
 * baybe/acquisition/acqfs.py:28-138; set-up on the host by baybe_b200/nipv.py).  With C the n_cond conditioning
 * points (pending points and the other points of a q-batch, observed with noise) and k_D the posterior covariance
 * given the training data, k_C(a,b) = k_D(a,b) - k_D(a,C) (K_D(C,C) + diag sigma_n^2(C))^-1 k_D(C,b).  Writes, for
 * every candidate x, IVR(x) = sum_m k_C(m,x)^2 / (k_C(x,x) + sigma_n^2(x)) in original units over the M integration
 * points m (qNIPV(x | C) = -(1/M) [sum_m k_C(m,m) - IVR(x)]; the caller adds the candidate-independent sum).
 *   m: a non-wide model with n <= 256 training points (else BB_ERR_UNSUPPORTED); noise [n_tasks]: HOST array, the
 *     likelihood noise per task in standardised units (floored at 1e-4 as in bb_model_desc); prior_var: the largest
 *     prior variance k(a,a) over the tasks, standardised (sets the power-of-two scale of the fp16 operands).
 *   d_x [N][d], d_xm [M][d]: raw comp-rep rows, fp32 row-major (M >= 1).
 *   d_var [N]: bb_posterior's variance of the candidates (original units).
 *   n_cond in [0, BB_MAX_PENDING].  With n_cond > 0: d_cross_x [N][n_cond] and d_cross_m [M][n_cond], bb_posterior's
 *     cross covariances with C as its pending points (original units), and d_linv [n_cond][n_cond] = L_C^-1
 *     (row-major, lower triangular), L_C L_C^T = K_D(C,C) + diag sigma_n^2(C) in original units.
 *   d_ws: caller-owned workspace of ws_bytes >= 256 * (4 r_pad + 4 d + 12) bytes, r_pad = n + n_cond rounded up to
 *     64; candidates and integration points are processed in blocks of rows that fit it (all of them with
 *     (N + M + 256) * (4 r_pad + 4 d + 12) bytes), so device memory is bounded for any N and M.
 * Writes IVR to d_score (nullable) and folds d_keep (nullable) and index_offset into *d_best_key like bb_argmax
 * (initialise with bb_best_init).  Deterministic: the same inputs give bit-identical outputs. */
int bb_nipv_score(const bb_model* m, const float* noise, float prior_var, const float* d_x, int64_t N,
                  const float* d_xm, int64_t M, const float* d_var, int32_t n_cond, const float* d_cross_x,
                  const float* d_cross_m, const float* d_linv, const uint8_t* d_keep, float* d_score,
                  int64_t* d_best_key, int64_t index_offset, void* d_ws, size_t ws_bytes, void* stream);

/* ---- test-only diagnostic: plain fp32 SIMT posterior (no tensor cores), used by the GPU
 * tests to separate tensor-core-path errors from formula errors.  Not called by the product. -- */
int bb_debug_posterior_simt(const bb_model* m, const void* d_x, int32_t layout, int64_t N,
                            int64_t ldx, float* d_mu, float* d_var, void* stream);
/* test-only: record pipeline events of CTA 0 of the following fused launches into d_buf
 * ([0] = count, then capacity_pairs (tile*1000 + event id, SM clock) int64 pairs, then two counters:
 * [1 + 2*capacity_pairs] rows that took the exact qLogEI sum, [2 + 2*capacity_pairs] rows served by the
 * table -- so d_buf holds 2*capacity_pairs + 3 entries); NULL switches it off. */
int bb_debug_set_trace(int64_t* d_buf, int64_t capacity_pairs);

#ifdef __cplusplus
}
#endif
#endif /* BAYBE_B200_H_ */
