/* orx.h -- C-ABI of liborx.so: the H100 (sm_90a) implementation of the openrec.tf2
 * embedding-lookup -> pair-score -> loss -> sparse-gradient -> optimizer training step.
 *
 * The reference (ylongqi/openrec) is pure Python on TensorFlow and has NO FFI of its own;
 * each entry point below therefore cites the reference *call site* (path:line relative to the
 * reference repo) whose TensorFlow op sequence it replaces.  INTEGRATION.md shows the ctypes
 * binding a maintainer would add on the reference side.
 *
 * Conventions
 *  - plain C: pointers + sizes, no torch / CUDA types in signatures (orx_stream_t is a
 *    cudaStream_t passed as void*; NULL = the legacy default stream);
 *  - every pointer is a DEVICE pointer unless its name ends in _host;
 *  - the caller owns every buffer; the library allocates only the opaque per-device workspace
 *    held by an orx_handle_t (index hash sets and duplicate-row gradient staging, loss partials,
 *    id staging, evaluation scratch, sharded-step scratch, split-K partials, the sharded censor's dedup hash, the bag apply's compacted ids), keeps no device
 *    state outside it, and orx_destroy frees all of it.  Two handles share nothing;
 *  - all calls are asynchronous w.r.t. the host and ordered on the given stream;
 *  - the calls of one handle that build or use its own batch index (the pairwise and pointwise steps, orx_sparse_apply*,
 *    orx_censor; not orx_pairwise_prefetch's side-stream build) share its index set 0 and staging rows, so they must be
 *    ordered among themselves: one stream, or streams the caller orders with events.  A table's epoch wrap then empties
 *    it on that stream, behind every launch that used it;
 *  - return value: ORX_OK (0) or a negative orx_status; orx_last_error_string() gives the
 *    thread-local message.  There is no CPU fallback: without a CUDA device every compute
 *    entry point fails with ORX_ERR_CUDA.
 *  - tables are row-major float32 [rows, dim] with 64-bit row offsets; ids are int32.
 *  - alignment: a table, its slot rows s0 / s1, GMF's w and a gather's output may start at any 4-byte-aligned address
 *    (a view into one flat parameter buffer, say).  A call moves rows as 128-bit float4 only when every caller pointer
 *    that path reads or writes through is 16-byte aligned; otherwise it takes the entry point's scalar or generic path,
 *    with the same results (a sparse step then records STEP_GENERIC, orx_censor_shard CENSOR_SCALAR).  The one
 *    exception is orx_shard_step, which has no scalar path: it refuses local shards or slot rows off a 16-byte boundary
 *    with ORX_ERR_INVALID before any device work.
 */
#ifndef ORX_H_
#define ORX_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORX_ABI_VERSION 1
#define ORX_API __attribute__((visibility("default")))

typedef struct orx_ctx* orx_handle_t;
typedef void* orx_stream_t; /* cudaStream_t */

enum orx_status {
  ORX_OK = 0,
  ORX_ERR_INVALID = -1,     /* bad argument (null pointer, negative size, unknown enum) */
  ORX_ERR_CUDA = -2,        /* CUDA runtime error (message in orx_last_error_string) */
  ORX_ERR_UNSUPPORTED = -3, /* combination not implemented */
  ORX_ERR_NOMEM = -4        /* workspace allocation failed */
};

enum orx_pair_kind { ORX_PAIR_BPR = 0, ORX_PAIR_UCML = 1 };
enum orx_point_kind { ORX_POINT_GMF = 0, ORX_POINT_WRMF = 1 };
enum orx_score_kind { ORX_SCORE_DOT = 0, ORX_SCORE_NEG_SQDIST = 1 };

/* Optimizers = the Keras OptimizerV2 sparse-apply semantics (dedup by row, then apply once):
 *   SGD        var[r] -= lr*G
 *   ADAGRAD    acc[r] += G^2; var[r] -= lr*G/(sqrt(acc[r])+eps)          (s0 = acc, init 0.1)
 *   ADAM_LAZY  row-sparse Adam (NOT the reference's semantics; explicit opt-in)
 *   ADAM_DENSE Keras-2.0 Adam on IndexedSlices: m,v decay and var update sweep the WHOLE table
 *              every step (what `optimizers.Adam()` in tf2_examples/bpr_citeulike.py:31 does)
 *   ROWWISE_ADAGRAD  one accumulator per table row (an addition, not in the reference; explicit opt-in):
 *              acc[r] += (1/dim) * sum_j G[j]^2; var[r][j] -= lr*G[j]/(sqrt(acc[r])+eps)   (s0 = acc, float[rows])
 *              Rows the batch does not touch keep row and accumulator bit for bit.  The sum over the row runs in an
 *              order each kernel fixes, so a row referenced once in a batch updates to the same bits on every run.  A
 *              dim-1 table (the item bias among them) updates exactly as ADAGRAD does.  Dense variables
 *              (orx_dense_apply's var, the pointwise step's GMF weight w) get element-wise ADAGRAD, s0 element-wise.
 *              orx_shard_step does not take it.
 *   MOMENTUM   Keras SGD(momentum=beta1) on IndexedSlices (SparseApplyKerasMomentum), row-lazy like every kind here:
 *              a[r] = beta1*a[r] - lr*G; var[r] += a[r]                   (s0 = a, [rows, dim], init 0)
 *   NESTEROV   the same with nesterov=True: a[r] = beta1*a[r] - lr*G; var[r] += beta1*a[r] - lr*G
 *              Both take lr as given, round each product, sum and difference to float32 (no fused multiply-add), and
 *              run in every entry point that takes ADAGRAD, orx_shard_step included.  Dense variables get the same
 *              formula element-wise.  Keras SGD with momentum 0 is plain SGD: pass ORX_OPT_SGD, with no slot.
 * For Adam s0 = m, s1 = v, lr_t = lr*sqrt(1-beta2^step)/(1-beta1^step), step is 1-based.  Adagrad and Adam use the
 * sqrt.approx / rcp.approx approximations. */
enum orx_opt_kind {
  ORX_OPT_SGD = 0,
  ORX_OPT_ADAGRAD = 1,
  ORX_OPT_ADAM_LAZY = 2,
  ORX_OPT_ADAM_DENSE = 3,
  /* 4 and 7 are not assigned: every entry point refuses them as unknown kinds (ORX_ERR_INVALID), as it always has.
   * Callers use both as the unknown kind that must be refused, so the momentum pair skips 7 rather than take it. */
  ORX_OPT_ROWWISE_ADAGRAD = 5,
  ORX_OPT_MOMENTUM = 6,
  ORX_OPT_NESTEROV = 8
};

typedef struct {
  int32_t kind; /* orx_opt_kind */
  float lr, eps, beta1, beta2;
  int64_t step; /* Adam: 1-based iteration count of THIS apply */
} orx_opt_t;

/* One LatentFactor (openrec/tf2/modules/latent_factor.py:4-15) and its optimizer slots. */
typedef struct {
  float* var;   /* [rows, dim] */
  float* s0;    /* Adagrad accumulator [rows, dim] | Adam m [rows, dim] | row-wise Adagrad accumulator float[rows]
                   (4-byte alignment is enough: it is read as scalars) | momentum a [rows, dim] ; NULL for SGD */
  float* s1;    /* Adam v ; NULL otherwise */
  int64_t rows;
  int32_t dim;
} orx_table_t;

/* A LatentFactor stored in bfloat16 (the *_bf16 entry points), its optimizer slots in fp32: s0 / s1 have exactly the
 * shapes and meaning of orx_table_t's (the row-wise Adagrad accumulator is float[rows]).  var holds the [rows, dim]
 * bf16 bit patterns.  Every kernel reads a row as fp32 (the exact upcast), computes in fp32 and rounds only the final
 * store of an updated element, stochastically:
 *   Element (row, col) of table t (0 = user, 1 = item), written by the apply of optimizer step opt->step with seed
 *   sr_seed, takes 16 random bits  r = H(sr_seed, step, t, row, col) >> 16, with
 *     mix64(z)   = splitmix64's finalizer: z = (z ^ z >> 30) * 0xbf58476d1ce4e5b9; z = (z ^ z >> 27) *
 *                  0x94d049bb133111eb; z ^ z >> 31   (uint64 arithmetic)
 *     mix32(x)   = x ^= x >> 16; x *= 0x7feb352d; x ^= x >> 15; x *= 0x846ca68b; x ^ x >> 16   (uint32 arithmetic)
 *     key(t)     = (uint32)(mix64(sr_seed ^ mix64(2 * step + t)) >> 32)
 *     H          = mix32(mix32(key(t) ^ (uint32)row) + (uint32)col * 0x9e3779b9)
 *   and the stored bits are (bits(x) + r) >> 16 for the fp32 result x: a value exactly representable in bf16 is kept,
 *   any other rounds away from zero with probability equal to its distance from the bf16 value below it (in units of
 *   that ulp).  Inf is stored as is; NaN keeps sign and top mantissa bits with the quiet bit set (0x0040).  The bits
 *   depend on those five values and x only, so every kernel that may write the row (owned in the fused step, staged in
 *   the tail, swept under ADAM_DENSE) rounds it alike, with or without a prefetched index.
 * Tables whose var is not 8-byte aligned, or whose dim is not a multiple of 4, take the scalar kernels (STEP_GENERIC). */
typedef struct {
  uint16_t* var; /* [rows, dim] bf16 bits */
  float* s0;     /* as orx_table_t */
  float* s1;
  int64_t rows;
  int32_t dim;
} orx_table_bf16_t;

/* ---- context ------------------------------------------------------------------------- */
ORX_API int orx_abi_version(void);
ORX_API const char* orx_last_error_string(void); /* host, thread-local */
ORX_API int orx_create(int device, orx_handle_t* out);
ORX_API int orx_destroy(orx_handle_t h);
ORX_API int orx_device_count(int* n_out_host);
/* Blocks the host until `stream` has drained (cudaStreamSynchronize). */
ORX_API int orx_stream_synchronize(orx_handle_t h, orx_stream_t stream);
/* Test hook: place the epoch of every batch-index table of the handle (index sets 0, 1 and 2), of orx_censor_shard's
 * dedup hash and, once it has run, of orx_shard_step's own index sets (31 bits; each table takes its next epoch at its next build, and the one whose epoch
 * wraps is emptied on the stream of that build). */
ORX_API int orx_debug_set_epoch(orx_handle_t h, uint32_t epoch);
/* Test hook: the kernel variants launched by this handle's DLRM entry points (orx_mlp_layer_*, orx_interact_*, orx_cross_*) and
 * sparse steps (orx_pairwise_step, orx_pairwise_step_host, orx_pointwise_step) since the last call, oldest first, at
 * most cap of them (a ring of the last ORX_DISPATCH_LOG_CAP), then clears them.
 * Record k is rec_host[8k .. 8k+7] = {op, variant, TA, TB, M, N, K, S}: a GEMM C[M,N] = op(A)[M,K] op(B)[K,N] with the
 * operand layouts TA / TB of orx_dlrm.cu and S split-K slices (1 = no split); an interaction has M = B, N = F, K = D,
 * TA = TB = 0, S = 1.  A sparse step (one record per call) has TA = kind (orx_pair_kind / orx_point_kind), TB = optimizer
 * (orx_opt_kind), M = B, N = D, K = the CTAs/SM bound of the fused kernel's __launch_bounds__ (0: none) and S = the batch
 * index set it used: 0 = built on the caller's stream, 1 or 2 = a consumed prefetch (orx_pairwise_prefetch, or the side
 * stream of orx_pairwise_step_host).  orx_score_rank, orx_score_topk and their bf16 forms write one record per call,
 * orx_score_rank_shard one per phase-2 call and orx_score_topk_shard one per phase-1 call (fields at ORX_OP_SCORE_RANK /
 * ORX_OP_SCORE_TOPK / ORX_OP_SCORE_RANK_BF16 / ORX_OP_SCORE_TOPK_BF16 / ORX_OP_SCORE_RANK_SHARD /
 * ORX_OP_SCORE_TOPK_SHARD); orx_score_all, orx_score_rank_listed and their bf16 forms write none.
 * Host-side bookkeeping only: no device work, no synchronisation. */
enum orx_dispatch_op {
  ORX_OP_GEMM = 0,
  ORX_OP_INTERACT_FWD = 1,
  ORX_OP_INTERACT_BWD = 2,
  ORX_OP_PAIRWISE_STEP = 3,  /* orx_pairwise_step, orx_pairwise_step_host */
  ORX_OP_POINTWISE_STEP = 4, /* orx_pointwise_step */
  ORX_OP_SCORE_RANK = 5,     /* orx_score_rank: TA = orx_score_kind, TB = 0, M = Bu, N = I, K = dim, S = item splits */
  ORX_OP_SCORE_TOPK = 6,     /* orx_score_topk: TA = orx_score_kind, TB = k, M = Bu, N = I, K = dim, S = item splits */
  ORX_OP_SCORE_RANK_SHARD = 7, /* orx_score_rank_shard, phase 2 only: variant RANK_SMEM / RANK_GLOBAL of the local
                                  pass, TA = orx_score_kind, TB = rank, M = Bu, N = local items, K = dim, S = item
                                  splits (0: no local items, no pass launched) */
  ORX_OP_SCORE_TOPK_SHARD = 8, /* orx_score_topk_shard, phase 1 only: variant TOPK, TA = orx_score_kind, TB = rank,
                                  M = Bu, N = local items, K = dim, S = item splits (0: no local items, no pass) */
  ORX_OP_POINTWISE_GRAD_ROWS = 9, /* orx_pointwise_grad_rows: variant STEP (k_pgr_step, specialised on D) or
                                    STEP_GENERIC (k_pgr_generic), TA = orx_point_kind, TB = 0, M = B, N = dim, K = ld,
                                    S = 1 */
  ORX_OP_CENSOR_SHARD = 10, /* orx_censor_shard, one per call: variant CENSOR_VEC / CENSOR_SCALAR, TA = rank, TB = 0,
                               M = total ids (n_per_block * n_blocks), N = local_rows, K = dim, S = world */
  ORX_OP_CROSS = 11, /* orx_cross_fwd / orx_cross_bwd, one per call with B > 0: variant CROSS_VEC / CROSS_SCALAR,
                       TA = 0 forward / 1 backward, TB = orx_cross_mode (0 forward), M = B, N = W,
                       K = split (ORX_CROSS_FINAL, else 0), S = 1 */
  ORX_OP_PAIRWISE_STEP_BF16 = 12, /* orx_pairwise_step_bf16, orx_pairwise_step_host_bf16: the fields of
                                     ORX_OP_PAIRWISE_STEP */
  ORX_OP_POINTWISE_STEP_BF16 = 13, /* orx_pointwise_step_bf16: the fields of ORX_OP_POINTWISE_STEP */
  ORX_OP_SCORE_RANK_BF16 = 14, /* orx_score_rank_bf16: the fields of ORX_OP_SCORE_RANK (same variant and item splits
                                  as orx_score_rank on the same shapes) */
  ORX_OP_SCORE_TOPK_BF16 = 15  /* orx_score_topk_bf16: the fields of ORX_OP_SCORE_TOPK (same item splits as
                                  orx_score_topk on the same shapes) */
};
enum orx_dispatch_variant {
  ORX_VARIANT_GEMM_TMA = 0,      /* k_gemm_tma: TMA-fed wgmma 3xTF32 (orx_mlp_tc.cu) */
  ORX_VARIANT_GEMM_SIMT = 1,     /* k_gemm: fp32 SIMT tiles */
  ORX_VARIANT_INTERACT_WARP = 2, /* k_interact_{fwd,bwd}_warp: one warp per sample */
  ORX_VARIANT_INTERACT = 3,      /* k_interact_{fwd,bwd}: one CTA per sample */
  ORX_VARIANT_STEP = 4,          /* k_pair_step / k_point_step specialised on D (32, 64, 128, 256), one register buffer;
                                    tables, slot rows and w 16-byte aligned */
  ORX_VARIANT_STEP_PIPE = 5,     /* k_pair_step with the register double buffer (PIPE) */
  ORX_VARIANT_STEP_GENERIC = 6,  /* k_pair_generic / k_point_generic (fused-step mode): any D, any 4-byte-aligned table */
  ORX_VARIANT_RANK_SMEM = 7,     /* k_score_rank: thresholds and histograms of a user tile in shared memory */
  ORX_VARIANT_RANK_GLOBAL = 8,   /* k_score_rank: thresholds and histograms in the handle's global scratch */
  ORX_VARIANT_TOPK = 9,          /* k_score_topk + k_topk_merge: candidate lists in the handle's global scratch */
  ORX_VARIANT_CENSOR_VEC = 10,   /* k_censor_shard, one float4 per lane (dim % 4 == 0 && dim <= 128, tab 16-byte
                                    aligned) */
  ORX_VARIANT_CENSOR_SCALAR = 11, /* k_censor_shard, lane-strided scalar rows (any other dim, or tab off a 16-byte
                                     boundary) */
  ORX_VARIANT_CROSS_VEC = 12,     /* k_cross_fwd / k_cross_bwd, one float4 per thread */
  ORX_VARIANT_CROSS_SCALAR = 13   /* k_cross_fwd / k_cross_bwd, one float per thread (any W, any 4-byte-aligned base) */
};
#define ORX_DISPATCH_LOG_CAP 64
ORX_API int orx_debug_dispatch_log(orx_handle_t h, int32_t* rec_host, int32_t cap, int32_t* n_host);
/* Test hook: the per-triplet records a prefetch resolved for index set `set` (1 or 2, as in a dispatch record), copied
 * to the device int32[B][4] rec on `stream` once that prefetch is complete: {flags, du, dp, dn} of triplet t, flags bit 0
 * = its three ids are in range, bits 1/2/3 = the user / positive / negative row is referenced once in the batch; du /
 * dp / dn = the row's staging index, -1 for such a row (ADAM_DENSE: every row has one, bits 1-3 are 0).  The records
 * of a set last until the second prefetch after it.  ORX_ERR_INVALID when the handle has none (ORX_PAIR_RESOLVE=0 at
 * orx_create, or no prefetch yet). */
ORX_API int orx_debug_pair_records(orx_handle_t h, int32_t set, int32_t* rec, int32_t B, orx_stream_t stream);
/* Test hook: the stochastic rounding of bf16 tables (orx_table_bf16_t) applied on `stream` to the device floats x[0..n),
 * element i taken as (row0 + i / dim, i % dim) of table `table` (0 = user, 1 = item) at (sr_seed, step); the bf16 bits
 * go to the device out[0..n). */
ORX_API int orx_debug_round_bf16(orx_handle_t h, const float* x, uint16_t* out, int64_t n, int64_t row0, int32_t dim,
                                 int32_t table, uint64_t sr_seed, int64_t step, orx_stream_t stream);

/* Measurement hook (bench.py's roofline): while enabled, every 8th *_step call records CUDA events on its launch stream
 * around its launches -- orx_pairwise_step, orx_pairwise_step_host and orx_pointwise_step: [0] batch index (or the wait
 * for a prefetched one), [1] the fused gather-score-update kernel, [2] tail (ADAM_DENSE: + the Adam sweeps);
 * orx_shard_step: its six launches [0..5].  orx_profile_read waits
 * for the recorded events, returns the summed device time of the first n_phases phases (ms) and the number of steps
 * recorded since the last read, and resets the counter. */
ORX_API int orx_profile_enable(orx_handle_t h, int32_t on);
ORX_API int orx_profile_read(orx_handle_t h, float* ms_host, int32_t n_phases, int32_t* n_steps_host);

/* ---- LatentFactor ---------------------------------------------------------------------- */
/* LatentFactor.__init__ 'uniform' initializer = U(-0.05,0.05), on device, counter-based RNG
 * (latent_factor.py:8-15).  lo/hi generalise it (glorot for MLP kernels). */
ORX_API int orx_fill_uniform(orx_handle_t h, float* dst, int64_t n, float lo, float hi, uint64_t seed, orx_stream_t s);
/* LatentFactor.__call__ = Embedding.call: out[b,:] = tab[ids[b],:] (bpr.py:23-27, dlrm.py:83-85).
 * ids int32 (id_is_i64 = 0) or int64 (1).  Out-of-range ids yield zero rows and are counted in
 * *n_bad (device int32, may be NULL). */
ORX_API int orx_gather(orx_handle_t h, const float* tab, int64_t rows, int32_t dim, const void* ids, int32_t id_is_i64,
               int64_t n, float* out, int32_t* n_bad, orx_stream_t s);
/* LatentFactor.censor (latent_factor.py:17-23): for the UNIQUE ids, row /= max(||row||_2, min_norm). */
ORX_API int orx_censor(orx_handle_t h, float* tab, int64_t rows, int32_t dim, const int32_t* ids, int32_t n,
               float min_norm, orx_stream_t s);
/* LatentFactor.censor (latent_factor.py:17-23) of a ROW-SHARDED table, the kernel of UCML.censor_vec (ucml.py:44-48) on
 * sharded tables (openrec_b200.sharded.censor_vec_sharded).  Row r of the global [total_rows, dim] table lives on rank
 * r % world at local row r / world of this rank's shard tab [local_rows, dim].
 *   ids: n_blocks blocks of n_per_block GLOBAL ids, block b at ids + b * block_stride -- an all-gather of every rank's
 *        ids: censor_vec packs (u, p, n) as [3][B] per rank, so call c uses ids + c * B with n_per_block = B,
 *        block_stride = 3B, n_blocks = world; one table's censor uses [world][n] with block_stride = n.
 *   This rank censors the ids it owns, 0 <= id < total_rows and id % world == rank: over all n_per_block * n_blocks
 *   ids, each such row once, row /= max(||row||_2, min_norm) with the arithmetic of orx_censor, so the rows of every
 *   rank together equal orx_censor on the global table and the concatenated ids, bit for bit.  Other ids are skipped.
 *   local_rows may exceed the rows this rank owns (a 1-row dummy shard of a rank past the table's end is not touched).
 *   Scratch: the handle's own dedup hash (not index set 0), grown to the largest call; orx_censor_shard calls of one
 *   handle are ordered among themselves as the index-set calls are.  At most ORX_CENSOR_SHARD_MAX_IDS ids per call.
 *   One dispatch record per call (ORX_OP_CENSOR_SHARD); a call without ids or owned rows launches nothing. */
#define ORX_CENSOR_SHARD_MAX_IDS (1 << 28)
ORX_API int orx_censor_shard(orx_handle_t h, float* tab, int64_t local_rows, int32_t dim, int64_t total_rows,
                             int32_t world, int32_t rank, const int32_t* ids, int32_t n_per_block, int64_t block_stride,
                             int32_t n_blocks, float min_norm, orx_stream_t s);

/* ---- pairwise recommenders: BPR (recommenders/bpr.py:21-37 + modules/pairwise_log_loss.py:15-34)
 *      and UCML (recommenders/ucml.py:21-42) ------------------------------------------------
 * One training step == model(u,p,n) under GradientTape -> tape.gradient(c_loss*loss + c_l2*l2_loss)
 * -> optimizer.apply_gradients (tf2_examples/bpr_citeulike.py:33-39; the example passes the tuple
 * (loss, l2_loss) => c_loss = c_l2 = 1).  All rows are gathered from the PRE-step tables, duplicate
 * rows' gradients are summed, the optimizer is applied once per unique row.
 * out4 (device float[4]) = { loss, l2_loss, number of out-of-range ids, number of staged rows }.
 * user/item must have equal dim; item_bias has dim 1 and item.rows rows. */
ORX_API int orx_pairwise_step(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                      const orx_table_t* item_bias, const int32_t* uid, const int32_t* pid, const int32_t* nid,
                      int32_t B, float margin, float c_loss, float c_l2, const orx_opt_t* opt_host,
                      float* out4, orx_stream_t s);
/* Same step through HOST buffers: ids are copied host->device (pinned memory recommended) and out4 is
 * copied device->host on `s`, all inside this call's stream work (the bench's end-to-end arm). */
ORX_API int orx_pairwise_step_host(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                           const orx_table_t* item_bias, const int32_t* uid_host, const int32_t* pid_host,
                           const int32_t* nid_host, int32_t B, float margin, float c_loss, float c_l2,
                           const orx_opt_t* opt_host, float* out4_host, orx_stream_t s);
/* Pipelining hint for device-resident ids: build the batch index (the dedup hash of the step) of (uid, pid, nid) NOW, on
 * the handle's side stream, so that it runs beside whatever the step stream is doing (typically the previous step).
 * ids_ready = 1: the id buffers are already complete (pre-staged batches); 0: they are complete once the work queued so
 * far on ids_stream has run (e.g. a sampler kernel).  The next orx_pairwise_step called with exactly these pointers, B and
 * optimizer kind waits for this index instead of building its own.  One outstanding prefetch; an unconsumed one is
 * dropped.  The caller must not modify the id buffers until that step has run.  orx_pairwise_step_host pipelines the
 * same way internally (upload + index of batch t under the kernels of batch t-1). */
ORX_API int orx_pairwise_prefetch(orx_handle_t h, const orx_table_t* user, const orx_table_t* item, const int32_t* uid,
                                  const int32_t* pid, const int32_t* nid, int32_t B, int32_t opt_kind, int32_t ids_ready,
                                  orx_stream_t ids_stream);
/* Forward only: (loss, l2_loss) -> out4[0..1]  (model(u,p,n) without a tape). */
ORX_API int orx_pairwise_fwd(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                     const orx_table_t* item_bias, const int32_t* uid, const int32_t* pid, const int32_t* nid,
                     int32_t B, float margin, float* out4, orx_stream_t s);
/* Un-fused gradients in TF IndexedSlices form (values per lookup, NOT deduplicated):
 * d_user[B,D], d_pos[B,D], d_neg[B,D], d_bp[B], d_bn[B]; any may be NULL.  g_out[B] (optional) receives
 * the per-triplet loss-gradient scalar.  orx_pairwise_grad_rows (below) is the compact form used by the
 * NCCL form of the sharded step: gradients are written to the lookup's own fetched row. */
ORX_API int orx_pairwise_grad(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                      const orx_table_t* item_bias, const int32_t* uid, const int32_t* pid, const int32_t* nid,
                      int32_t B, float margin, float c_loss, float c_l2, float* d_user, float* d_pos, float* d_neg,
                      float* d_bp, float* d_bn, float* g_out, orx_stream_t s);

/* ---- bf16 user / item tables (orx_table_bf16_t) ------------------------------------------------------------------
 * orx_pairwise_step_bf16 / orx_pairwise_step_host_bf16: orx_pairwise_step / orx_pairwise_step_host on bf16 user and
 * item tables, every optimizer kind included, each updated element rounded stochastically with sr_seed and opt->step.
 * The item bias stays an fp32 orx_table_t.  A batch index built by orx_pairwise_prefetch is consumed as by the fp32
 * step (pass it orx_table_t's with the rows and dims of these tables).  One dispatch record per call, op
 * ORX_OP_PAIRWISE_STEP_BF16.  Untouched rows keep their bits, except under ADAM_DENSE (its sweep writes every row). */
ORX_API int orx_pairwise_step_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                   const orx_table_bf16_t* item, const orx_table_t* item_bias, const int32_t* uid,
                                   const int32_t* pid, const int32_t* nid, int32_t B, float margin, float c_loss,
                                   float c_l2, const orx_opt_t* opt_host, uint64_t sr_seed, float* out4, orx_stream_t s);
ORX_API int orx_pairwise_step_host_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                        const orx_table_bf16_t* item, const orx_table_t* item_bias,
                                        const int32_t* uid_host, const int32_t* pid_host, const int32_t* nid_host,
                                        int32_t B, float margin, float c_loss, float c_l2, const orx_opt_t* opt_host,
                                        uint64_t sr_seed, float* out4_host, orx_stream_t s);
/* orx_pairwise_fwd / orx_pairwise_grad on bf16 user and item tables (rows read as their exact fp32 upcast). */
ORX_API int orx_pairwise_fwd_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                  const orx_table_bf16_t* item, const orx_table_t* item_bias, const int32_t* uid,
                                  const int32_t* pid, const int32_t* nid, int32_t B, float margin, float* out4,
                                  orx_stream_t s);
ORX_API int orx_pairwise_grad_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                   const orx_table_bf16_t* item, const orx_table_t* item_bias, const int32_t* uid,
                                   const int32_t* pid, const int32_t* nid, int32_t B, float margin, float c_loss,
                                   float c_l2, float* d_user, float* d_pos, float* d_neg, float* d_bp, float* d_bn,
                                   float* g_out, orx_stream_t s);
/* orx_pointwise_step_bf16: orx_pointwise_step (below) on bf16 user and item tables, every optimizer kind included, each
 * updated element rounded stochastically with sr_seed and opt->step (table 0 = user, 1 = item).  The item bias and
 * GMF's w stay fp32 orx_table_t's.  One dispatch record per call, op ORX_OP_POINTWISE_STEP_BF16.  Untouched rows keep
 * their bits, except under ADAM_DENSE (its sweep writes every row). */
ORX_API int orx_pointwise_step_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                    const orx_table_bf16_t* item, const orx_table_t* item_bias, const orx_table_t* w,
                                    const int32_t* uid, const int32_t* iid, const float* label, int32_t B, float a,
                                    float b, int32_t use_sigmoid, float c_loss, float c_l2, const orx_opt_t* opt_host,
                                    uint64_t sr_seed, float* out4, orx_stream_t s);
/* orx_pointwise_fwd / orx_pointwise_grad on bf16 user and item tables (rows read as their exact fp32 upcast); GMF's
 * d_w included. */
ORX_API int orx_pointwise_fwd_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                   const orx_table_bf16_t* item, const orx_table_t* item_bias, const orx_table_t* w,
                                   const int32_t* uid, const int32_t* iid, const float* label, int32_t B, float a,
                                   float b, int32_t use_sigmoid, float* out4, orx_stream_t s);
ORX_API int orx_pointwise_grad_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                    const orx_table_bf16_t* item, const orx_table_t* item_bias, const orx_table_t* w,
                                    const int32_t* uid, const int32_t* iid, const float* label, int32_t B, float a,
                                    float b, int32_t use_sigmoid, float c_loss, float c_l2, float* d_user,
                                    float* d_item, float* d_bias, float* d_w, float* g_out, orx_stream_t s);
/* orx_censor on a bf16 table: row / max(||row||_2, min_norm) in fp32 from the upcast row, stored rounded to nearest
 * even (a projection, not an optimizer update). */
ORX_API int orx_censor_bf16(orx_handle_t h, uint16_t* tab, int64_t rows, int32_t dim, const int32_t* ids, int32_t n,
                            float min_norm, orx_stream_t s);

/* ---- pointwise recommenders: GMF (recommenders/gmf.py:22-34) and WRMF (recommenders/wrmf.py:21-34 +
 *      modules/pointwise_mse_loss.py:18-31) ---------------------------------------------------
 * GMF: w = the [D] kernel of Dense(1,use_bias=False) (gmf.py:19) as a 1-row orx_table_t (rows=1, dim=D);
 * WRMF: w = NULL, (a,b) label weights, use_sigmoid as PointwiseMSELoss(sigmoid=...). */
ORX_API int orx_pointwise_step(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                       const orx_table_t* item_bias, const orx_table_t* w, const int32_t* uid, const int32_t* iid,
                       const float* label, int32_t B, float a, float b, int32_t use_sigmoid, float c_loss,
                       float c_l2, const orx_opt_t* opt_host, float* out4, orx_stream_t s);
ORX_API int orx_pointwise_fwd(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                      const orx_table_t* item_bias, const orx_table_t* w, const int32_t* uid, const int32_t* iid,
                      const float* label, int32_t B, float a, float b, int32_t use_sigmoid, float* out4,
                      orx_stream_t s);
ORX_API int orx_pointwise_grad(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                       const orx_table_t* item_bias, const orx_table_t* w, const int32_t* uid, const int32_t* iid,
                       const float* label, int32_t B, float a, float b, int32_t use_sigmoid, float c_loss,
                       float c_l2, float* d_user, float* d_item, float* d_bias, float* d_w, float* g_out,
                       orx_stream_t s);

/* ---- un-fused sparse apply + multi-GPU building blocks (SURVEY 8e; the reference is single-device) ----
 * orx_sparse_apply: optimizer.apply_gradients for ONE variable given IndexedSlices (ids[n], values[n,dim]):
 * dedup by row, apply once per unique row (what Keras OptimizerV2 does for every tape.gradient result of
 * an Embedding, tf2_examples/bpr_citeulike.py:37-38).  Used by owners in the row-sharded step and by DLRM. */
ORX_API int orx_sparse_apply(orx_handle_t h, const orx_table_t* tab, const int32_t* ids, const float* values,
                             int32_t n, const orx_opt_t* opt_host, orx_stream_t s);
/* Same with strided inputs: id i = ids[i*id_stride], value row i = values + i*value_ld (DLRM: ids = sparse[:,k],
 * values = dZ[:,k,:]; the row-sharded pointwise step: one column block of its exchange rows).  Value rows may start at
 * any float: 128-bit loads are used only when dim, value_ld and values allow them.  Ids outside [0, rows), such as
 * the -1 of orx_pointwise_serve, are skipped and never enter the batch index. */
ORX_API int orx_sparse_apply_strided(orx_handle_t h, const orx_table_t* tab, const int32_t* ids, int64_t id_stride,
                                     const float* values, int64_t value_ld, int32_t n, const orx_opt_t* opt_host,
                                     orx_stream_t s);
/* orx_bag_sparse_apply: optimizer.apply_gradients for ONE table of a multi-hot DLRM feature.  Bag b of the table is
 * sparse[b*ld + col_lo .. b*ld + col_lo + L) (sparse row-major [B, ld] int32); dZ + b*dz_ld is its pooled gradient row.
 * The IndexedSlices applied hold, for every valid id (0 <= id < rows) of every bag, in (b, l) order, the row
 * (id, dZ[b]) (mode 0, sum) or (id, dZ[b] / n_b) (mode 1, mean; n_b = the bag's valid ids, IEEE division); padding
 * (id < 0) and out-of-range ids contribute nothing.  Then Keras sparse semantics as orx_sparse_apply: dedup-then-apply
 * for SGD / Adagrad / row-sparse Adam, the whole-table sweep for ADAM_DENSE.  With L = 1 and mode 0 this is
 * orx_sparse_apply_strided(ids = sparse + col_lo, id_stride = ld, values = dZ, value_ld = dz_ld).
 * Scratch: the index workspace for B*L lookups (the handle's index sets and staging rows, sized per lookup) and the
 * handle's bag buffer (4 bytes per lookup + 4 per bag).  ORX_ERR_INVALID: null handle / table / opt, a null sparse / dZ
 * with B > 0, B < 0, L < 1, col_lo < 0, col_lo + L > ld, dz_ld < dim, mode outside {0, 1}, B*L > 2^31 - 1, unknown
 * optimizer kind or missing slot rows.  B = 0 is a no-op except for the ADAM_DENSE sweep. */
ORX_API int orx_bag_sparse_apply(orx_handle_t h, const orx_table_t* tab, const int32_t* sparse, int64_t ld,
                                 int32_t col_lo, int32_t L, int32_t B, const float* dZ, int64_t dz_ld, int32_t mode,
                                 const orx_opt_t* opt_host, orx_stream_t s);
/* orx_sparse_apply_strided_bf16 / orx_bag_sparse_apply_bf16: orx_sparse_apply_strided / orx_bag_sparse_apply on a bf16
 * table (orx_table_bf16_t), with the same arguments, checks, scratch and optimizer kinds.  A touched row is read as its
 * exact fp32 upcast and each updated element rounded stochastically as orx_table_bf16_t states, as table t = 0 with
 * sr_seed and opt->step (the staged-row tail and the ADAM_DENSE sweep use the same key).  A caller with several tables
 * gives each its own seed: DLRM gives table k mix64(rounding_seed + k) (mod 2^64), distinct for every k since mix64 is a
 * bijection.  Untouched rows keep their bits, except under ADAM_DENSE (its sweep writes every row).  Alignment: rows
 * move 4 elements (8 bytes) per lane when var is 8-byte aligned, dim % 4 == 0 and the slot rows the optimizer keeps are
 * 16-byte aligned (a row-wise accumulator does not count); any other 2-byte-aligned table takes the scalar path, which
 * rounds alike. */
ORX_API int orx_sparse_apply_strided_bf16(orx_handle_t h, const orx_table_bf16_t* tab, const int32_t* ids,
                                          int64_t id_stride, const float* values, int64_t value_ld, int32_t n,
                                          const orx_opt_t* opt_host, uint64_t sr_seed, orx_stream_t s);
ORX_API int orx_bag_sparse_apply_bf16(orx_handle_t h, const orx_table_bf16_t* tab, const int32_t* sparse, int64_t ld,
                                      int32_t col_lo, int32_t L, int32_t B, const float* dZ, int64_t dz_ld,
                                      int32_t mode, const orx_opt_t* opt_host, uint64_t sr_seed, orx_stream_t s);
/* Combined form used by openrec_b200/sharded.py: each rank stores ONE local table [user rows | item rows] of
 * width ld = D+4 (item bias in column D), so a lookup is (owner, combined local row) whatever its table.
 * orx_owner_bucket_combined: ids = uid | pid | nid (n_user user ids first).  Row r lives on rank r % world at
 *   local row r / world; item lookups get the owner's user-row count added to their local row.  counts[world] =
 *   lookups per owner, send_local[n] = local rows in owner-sorted send order, slot[n] = position of lookup i in
 *   that order.
 * orx_pairwise_grad_rows: score/loss/gradients on the fetched rows (one row of width ld per lookup; slots index
 *   the same buffer); gradients overwrite d_rows at the lookup's row (bias gradient in column D, padding zero). */
ORX_API int orx_owner_bucket_combined(orx_handle_t h, const int32_t* ids, int32_t n, int32_t n_user, int64_t total_users,
                                      int32_t world, int32_t* counts, int32_t* send_local, int32_t* slot, orx_stream_t s);
ORX_API int orx_pairwise_grad_rows(orx_handle_t h, int32_t kind, const float* rows, int64_t ld, int32_t dim,
                                   const int32_t* uslot, const int32_t* pslot, const int32_t* nslot, int32_t B,
                                   float margin, float c_loss, float c_l2, float inv_B, float* d_rows, float* out4,
                                   orx_stream_t s);

/* ---- row-sharded DLRM (openrec_b200/csrc/orx_dlrm_shard.cu, openrec_b200/sharded.py ShardedDLRMStep) ----------
 * The T embedding tables form one row space: row_off[k] = sum of the vocabularies of tables 0..k-1, G = row_off[T] <=
 * 2^31 - 1.  Lookup i = b*T + k (id = sparse[i]) is valid iff 0 <= id < row_off[k+1] - row_off[k]; its global row
 * g = row_off[k] + id lives on rank g % world at local row g / world.
 * orx_lookup_bucket: sparse [B, T] int32 row-major (device), row_off_host int64 [T + 1] (host).  The unique valid
 *   global rows of the batch, in ascending (owner, local row) order -- the send order, n_uniq rows:
 *     counts[world]      unique rows owned by each rank (sum = n_uniq)
 *     send_local[j]      local row of unique row j on its owner                          (j < n_uniq; rest unspecified)
 *     slot[i]            send-order index of lookup i, or -1 for an invalid id           (all B*T entries)
 *     grp_idx[grp_off[j] .. grp_off[j+1])  the lookups of unique row j, ascending i       (rest unspecified)
 *     grp_off[n_uniq]    the number of valid lookups                                     (grp_off needs B*T + 1 entries)
 *   Limits: B*T <= 2^31 - 1, T >= 1, 1 <= world <= 1024, row_off[0] == 0 and non-decreasing (ORX_ERR_INVALID
 *   otherwise, before any device work).  B = 0 writes zero counts and grp_off[0] = 0 and launches nothing.  Scratch:
 *   the handle's own lookup buffer (about 16 bytes per lookup plus the radix sort's storage), grown on demand; the
 *   batch index sets are not touched, so an orx_sparse_apply later in the same step keeps them.
 * orx_rows_segment_sum: out[j, :] = sum of src[grp_idx[p], :] for p in [grp_off[j], grp_off[j+1]), added in that
 *   order, so repeated calls give the same bits.  src rows have stride src_ld >= dim; out is [n_uniq, dim]
 *   contiguous; float4 loads when dim, src_ld and both pointers allow, a scalar path for any dim >= 1.  grp_idx entries
 *   must index rows of src.  n_uniq = 0 is a no-op. */
ORX_API int orx_lookup_bucket(orx_handle_t h, const int32_t* sparse, int32_t B, int32_t T, const int64_t* row_off_host,
                              int32_t world, int32_t* counts, int32_t* send_local, int32_t* slot, int32_t* grp_off,
                              int32_t* grp_idx, orx_stream_t s);
ORX_API int orx_rows_segment_sum(orx_handle_t h, const float* src, int64_t src_ld, int32_t dim, const int32_t* grp_off,
                                 const int32_t* grp_idx, int32_t n_uniq, float* out, orx_stream_t s);
/* Multi-hot (bag) form of the row-sharded DLRM step.  sparse [B, C] int32 row-major holds T bags per sample: table k's
 * bag is columns col_off[k] .. col_off[k+1] (col_off_host int32 [T + 1], host, col_off[0] = 0, C = col_off[T]); lookup
 * i = b*C + c.  An id < 0 is padding; an id >= the table's vocabulary is bad; neither is pooled nor gets a gradient.
 * orx_bag_shard_lookups: rows[i] = row_off[k] + sparse[i] (the global row) for a valid id of column c in table k's bag,
 *   else -1.  rows [B, C] is the input of orx_lookup_bucket as [B*C, 1] with row_off = {0, G}: the buckets are those
 *   of the T-table call.  ORX_ERR_INVALID before any device work: null handle / host arrays, B < 0, T outside [1,
 *   ORX_BAG_MAX_TABLES], col_off[0] or row_off[0] != 0, either decreasing, C = 0, G > 2^31 - 1, B*C > 2^31 - 1, a null
 *   sparse / rows with B > 0.  B = 0 is a no-op.
 * orx_bag_segment_sum: the pooled gradient folded onto the unique rows of that bucket call: out[j, :] = the sum over p
 *   in [grp_off[j], grp_off[j+1]) of v(grp_idx[p]), added in ascending p, where v(b*C + c) = dZ[b, k(c), :] (mode 0,
 *   sum) or that row divided element-wise by n[b, k(c)] (mode 1, mean; IEEE division before the add), n being the bag's
 *   valid lookups (slot >= 0, slot from the bucket call, [B*C]; read in mode 1 only).  dZ[b, k, :] is at dZ + b*dz_ld +
 *   k*dim (dz_ld >= T*dim); out is [n_uniq, dim] contiguous.  One warp per unique row, float4 loads when dim, dz_ld and
 *   both pointers allow, a scalar path for any dim >= 1, no atomics: repeated calls give the same bits.  Scratch: the
 *   mean's B*T counts in the handle's own buffer, grown on demand.  ORX_ERR_INVALID before any device work: null handle
 *   / col_off, T outside [1, ORX_BAG_MAX_TABLES], dim < 1, B < 0, n_uniq < 0 or > B*C, mode outside {0, 1}, dz_ld <
 *   T*dim, col_off[0] != 0 or decreasing, C = 0, B*C > 2^31 - 1, and with n_uniq > 0 a null dZ / grp_off / grp_idx /
 *   out, or a null slot in mode 1.  n_uniq = 0 is a no-op. */
ORX_API int orx_bag_shard_lookups(orx_handle_t h, const int32_t* sparse, int32_t B, int32_t T,
                                  const int32_t* col_off_host, const int64_t* row_off_host, int32_t* rows,
                                  orx_stream_t s);
ORX_API int orx_bag_segment_sum(orx_handle_t h, const float* dZ, int64_t dz_ld, int32_t T, int32_t dim,
                                const int32_t* col_off_host, int32_t mode, const int32_t* slot, int32_t B,
                                const int32_t* grp_off, const int32_t* grp_idx, int32_t n_uniq, float* out,
                                orx_stream_t s);

/* ---- row-sharded GMF / WRMF (openrec_b200/csrc/orx_pointwise_shard.cu, openrec_b200/sharded.py
 * pointwise_step_sharded): the user table, the item table and the item bias are row-sharded per table (row r on rank
 * r % world at local row r / world, as orx_score_rank_shard reads them); GMF's w is replicated.  The step's exchange
 * runs over one row space built so that ownership matches that layout: with Lu = ceil(U / world), user u is global row
 * u and item i is global row world*Lu + i, i.e. orx_lookup_bucket with T = 2 and row_off = {0, world*Lu, world*Lu + I};
 * an owner's local rows < Lu are user rows, the others item rows (item local row + Lu).
 * orx_pointwise_shard_lookups: lookups [B, 2] int32 (8-byte aligned) = (uid[b], iid[b]) when 0 <= uid[b] < U and
 *   0 <= iid[b] < I, else (-1, -1) for the whole sample -- the single-device step's rule (a sample with a bad id is
 *   skipped, and none of its rows is touched), and the rejection of ids in [U, world*Lu), which orx_lookup_bucket
 *   would accept.  ORX_ERR_INVALID: B < 0, U or I outside [0, 2^31 - 1], a null pointer with B > 0.  B = 0 is a no-op.
 * orx_pointwise_serve (owner side): for each requested local row req[r], r < n, writes rows[r, 0 .. ld) = the user row
 *   req[r] (req[r] < local_users) or the item row req[r] - Lu with its bias in column dim (Lu <= req[r] < Lu +
 *   local_items), zeros elsewhere; user_local[r] / item_local[r] = the row in its own table, -1 where the request
 *   belongs to the other table (both -1 for a request outside both ranges, with a zero row).  Lu = user_rows_per_rank.
 *   ORX_ERR_INVALID: dim < 1, ld <= dim, n < 0, Lu < local_users, Lu + local_items > 2^31 - 1, a null pointer with n > 0
 *   (a shard may be null when its local row count is 0).  n = 0 is a no-op.
 * orx_pointwise_grad_rows: GMF's BCE-with-logits (kind GMF: the score (u * w) . i + bias) or WRMF's weighted squared
 *   error (kind WRMF: a, b, use_sigmoid as in orx_pointwise_step) of B samples over fetched rows: sample b reads row
 *   slot[2b] (user) and row slot[2b+1] (item, its bias in column dim) of `rows` (stride ld); a sample with a negative
 *   slot is skipped.  Writes, in lookup order, d_rows[2b] = the gradient of c_loss*loss + c_l2*l2_loss w.r.t. the user
 *   row and d_rows[2b+1] = that w.r.t. the item row with the bias gradient in column dim; padding columns and the rows
 *   of a skipped sample are zero.  out2 = {loss, l2}: the loss terms summed (GMF: times inv_B, the mean over a batch of
 *   1 / inv_B samples; the gradient is scaled alike) and 0.5 * the squares of every fetched row of a valid sample
 *   (duplicates included).  GMF: gw[dim] = this batch's part of w's gradient; with add_w_terms, c_l2 * w is added to gw
 *   and 0.5 * sum(w^2) to out2[1] -- the sharded step sets it on exactly one rank, so the sum over the ranks holds each
 *   once.  The arithmetic order is that of orx_pointwise_step's kernels; no atomics: the same inputs give the same bits.
 *   One dispatch record per call (ORX_OP_POINTWISE_GRAD_ROWS): variant STEP for dim 32 / 64 / 128 / 256 with ld % 4 == 0
 *   and 16-byte aligned rows, d_rows and w, else STEP_GENERIC.  Scratch: the handle's loss partials buffer, grown to
 *   (16 + 4 * dim (GMF)) bytes per 64 samples (a growing call synchronises the device).  ORX_ERR_INVALID: unknown kind,
 *   B < 1, dim outside [1, 1024], ld <= dim, a null rows / slot / label / d_rows / out2, GMF without w or gw, slot not
 *   8-byte aligned.
 * orx_rows_scale: x[r, k] = x[r, k] * scale[k] for r < rows, k < dim (x contiguous), one rounding per element -- the
 *   u * w of orx_score_rank / orx_score_topk with scale = w, so orx_score_rank_shard / orx_score_topk_shard on scaled
 *   xrows after phase 0's sum give GMF's scores.  rows = 0 is a no-op; ORX_ERR_INVALID: rows < 0, dim < 1, null x /
 *   scale with rows > 0. */
ORX_API int orx_pointwise_shard_lookups(orx_handle_t h, const int32_t* uid, const int32_t* iid, int32_t B,
                                        int64_t total_users, int64_t total_items, int32_t* lookups /*[B, 2]*/,
                                        orx_stream_t s);
ORX_API int orx_pointwise_serve(orx_handle_t h, const float* user_shard, const float* item_shard,
                                const float* bias_shard, int32_t dim, int64_t local_users, int64_t local_items,
                                int64_t user_rows_per_rank, const int32_t* req, int32_t n, int64_t ld,
                                float* rows /*[n, ld]*/, int32_t* user_local, int32_t* item_local, orx_stream_t s);
ORX_API int orx_pointwise_grad_rows(orx_handle_t h, int32_t kind, const float* rows, int64_t ld, int32_t dim,
                                    const int32_t* slot /*[2B]*/, const float* label, const float* w, int32_t B,
                                    float a, float b, int32_t use_sigmoid, float c_loss, float c_l2, float inv_B,
                                    int32_t add_w_terms, float* d_rows /*[2B, ld]*/, float* gw /*[dim]*/,
                                    float* out2, orx_stream_t s);
ORX_API int orx_rows_scale(orx_handle_t h, float* x, int64_t rows, int32_t dim, const float* scale, orx_stream_t s);

/* ---- row-sharded BPR / UCML step over the GPUs of one box, "home-routed" (openrec_b200/csrc/orx_shard.cu,
 * openrec_b200/sharded.py).  The reference is single-device: this is the scale-out of the same synchronous step
 * (tf2_examples/bpr_citeulike.py:33-39) and replaces the NCCL all-to-alls named in SURVEY 8(e) with peer STORES into
 * IPC-mapped mailboxes.  Row r of the user / item tables lives on rank r % world at local row r / world; a triplet is
 * computed on the rank that owns its user row.
 * orx_peer_alloc/open/close/free: cudaMalloc + CUDA IPC handle (64 bytes) so every rank can map every peer's mailboxes.
 * orx_shard_t: capacities + DEVICE arrays of `world` peer pointers, one per mailbox:
 *   tripbox int32[world][3][batch_cap]  triplets routed to me, per source rank        idbox int32[world][req_cap]
 *   got float[got_rows][dim], gotb float[got_rows]   item rows + biases for my triplets (got_rows = 2*home_cap+32*world)
 *   gin float[gin_cap][dim], ginb float[gin_cap]     gradient rows + bias gradients for rows I own
 *   meta int32[world][16]  per-peer counts / offsets / loss partials      flags int32[4*64+1] phase epochs + sticky error
 * orx_shard_sizes: element counts (4-byte words) of the eight mailboxes, in the order above.
 * orx_shard_step: the whole step in ONE call: six launches on `s`, cross-rank ordering by flag words in peer memory
 *   (no barrier launches, no collective, nothing returns to the host).  user/item/item_bias are this rank's LOCAL shards.
 *   epoch: strictly increasing per step, starting at 1.  phase_lo..phase_hi (0..5) selects a sub-range of the launches so
 *   that several virtual ranks can be stepped phase by phase on one device (the 1-GPU loopback test).
 *   next_uid / next_pid / next_nid / next_B (all NULL / 0, or all set: device pointers that stay valid until that step
 *   ran) announce the batch of step epoch + 1: its route and request then ride inside this step's apply launch, and the
 *   call for epoch + 1 -- which must pass exactly these pointers as uid / pid / nid -- issues four launches instead of six.
 *   All ranks announce, or none.  Other calls on the handle may come between steps and between phases.
 *   out4 = { loss, l2_loss (GLOBAL batch, identical on every rank), skipped triplets of this rank, staged rows }.
 *   The sticky error word flags[4*64] is 0 or: 1 a peer never arrived within timeout_ms, 2 more triplets routed to this
 *   home than home_cap, 3 / 4 request / gradient inbox too small.  SGD, Adagrad and row-sparse Adam.
 *   user / item var, s0 and s1 must be 16-byte aligned (every launch moves them as float4): a base off a 16-byte
 *   boundary returns ORX_ERR_INVALID, naming the pointer, before any device work. */
typedef struct {
  int32_t world, rank, dim, batch_cap, home_cap, req_cap, gin_cap, timeout_ms;
  void *tripbox, *idbox, *got, *gotb, *gin, *ginb, *meta, *flags;   /* DEVICE arrays of `world` pointers */
} orx_shard_t;
ORX_API int orx_peer_alloc(orx_handle_t h, int64_t bytes, void** dev_ptr_out, uint8_t* handle_out64);
ORX_API int orx_peer_open(orx_handle_t h, const uint8_t* handle64, void** dev_ptr_out);
ORX_API int orx_peer_close(orx_handle_t h, void* dev_ptr);
ORX_API int orx_peer_free(orx_handle_t h, void* dev_ptr);
ORX_API int orx_shard_sizes(const orx_shard_t* x_host, int64_t* n8_host);
ORX_API int orx_shard_step(orx_handle_t h, int32_t kind, const orx_shard_t* x_host, const orx_table_t* user,
                           const orx_table_t* item, const orx_table_t* item_bias, const int32_t* uid, const int32_t* pid,
                           const int32_t* nid, int32_t B, const int32_t* next_uid, const int32_t* next_pid,
                           const int32_t* next_nid, int32_t next_B, int64_t total_users, int64_t total_items, float margin,
                           float c_loss, float c_l2, float inv_B, const orx_opt_t* opt_host, int32_t epoch,
                           int32_t phase_lo, int32_t phase_hi, float* out4, orx_stream_t s);
/* ---- dense variables (GMF w, MLP kernels/biases): Keras dense apply ---------------------- */
ORX_API int orx_dense_apply(orx_handle_t h, float* var, float* s0, float* s1, const float* grad, int64_t n,
                    const orx_opt_t* opt_host, orx_stream_t s);

/* ---- DLRM (recommenders/dlrm.py:63-100) ----------------------------------------------------------
 * The model is composed on the host from these pieces, all with explicit leading dimensions so that the
 * stacked feature tensor, the concat of (dense_vec, interactions) and their gradients are never copied.
 * orx_gather_strided: one sparse feature's LatentFactor lookup, ids = sparse[:,k] (stride = #features),
 *   out = Z[:,k,:]                                                                   (dlrm.py:83-85)
 * orx_mlp_layer_fwd/bwd: one keras Dense(units, activation) of MLP (modules/multi_layer_perceptron.py:9-16),
 *   kernel w[in,out], act 0 none / 1 relu / 2 sigmoid; bwd overwrites dy with dL/dz and produces dw, db, dx.
 * orx_interact_fwd/bwd: SecondOrderFeatureInteraction over F features = F-1 embedding rows + the dense
 *   vector as LAST feature (modules/second_order_feature_interaction.py:12-34, dlrm.py:89-92);
 *   mode 0 = the reference's bug-compatible output (SURVEY Q1), mode 1 = strictly-lower triangle of Z Z^T.
 * orx_pred_loss: clip (dlrm.py:97-98) + keras MeanSquaredError (kind 0) / BinaryCrossentropy (kind 1)
 *   (dlrm.py:52-55,72-73); out4[0] = loss, dpred = dloss/dpred. */
ORX_API int orx_gather_strided(orx_handle_t h, const float* tab, int64_t rows, int32_t dim, const int32_t* ids,
                               int64_t id_stride, int64_t n, float* out, int64_t out_ld, int32_t* n_bad,
                               orx_stream_t s);
/* orx_bag_gather: the multi-hot form of the T gathers in ONE launch -- each sparse feature is a bag of ids pooled by a sum
 *   (mode 0) or a mean (mode 1).  sparse [B, ld] int32 row-major (device); tabs_host[k] / rows_host[k] (host arrays) =
 *   table k [rows, dim]; col_off_host[T + 1] (host): table k's bag for sample b is sparse[b*ld + col_off[k] ..
 *   b*ld + col_off[k+1]).  Writes Z[b, k, :] at out + b*out_ld + k*dim.  An id < 0 is padding; an id >= rows[k] is
 *   counted in *n_bad (device, optional) and adds nothing.  Sum: the valid rows added in column order in fp32, starting
 *   from the first valid row (a one-id bag copies its row bit for bit, as orx_gather_strided); mean: that sum / the
 *   bag's valid ids (IEEE division); a bag without a valid id pools to the zero row.  float4 accesses when dim, out_ld,
 *   out and every table allow them, a scalar path for any dim >= 1.  No atomics on Z: the same inputs give the same bits.
 *   ORX_ERR_INVALID before any device work: null handle / host arrays / table, a null sparse / out with B > 0, T outside
 *   [1, ORX_BAG_MAX_TABLES], dim < 1, B < 0, ld < 1, rows[k] < 1, col_off decreasing or outside [0, ld], out_ld < T*dim,
 *   mode outside {0, 1}.  B = 0 is a no-op. */
#define ORX_BAG_MAX_TABLES 63   /* T + 1 features (the dense vector last) must fit orx_interact_* (64) */
ORX_API int orx_bag_gather(orx_handle_t h, const float* const* tabs_host, const int64_t* rows_host, int32_t T,
                           int32_t dim, const int32_t* sparse, int64_t ld, const int32_t* col_off_host, int32_t B,
                           int32_t mode, float* out, int64_t out_ld, int32_t* n_bad, orx_stream_t s);
/* orx_gather_strided_bf16 / orx_bag_gather_bf16: orx_gather_strided / orx_bag_gather on bf16 tables (uint16_t bits;
 *   every table of orx_bag_gather_bf16 is bf16), with the same arguments and checks.  Rows are widened exactly and
 *   pooled in fp32 in the same column order, so out and *n_bad are those of the fp32 call on the fp32 upcast of the
 *   tables, bit for bit.  Alignment: a lane moves 4 columns as one 8-byte load when dim % 4 == 0, out_ld % 4 == 0, out
 *   is 16-byte aligned and every table 8-byte aligned; any other 2-byte-aligned table takes the scalar path (same bits). */
ORX_API int orx_gather_strided_bf16(orx_handle_t h, const uint16_t* tab, int64_t rows, int32_t dim, const int32_t* ids,
                                    int64_t id_stride, int64_t n, float* out, int64_t out_ld, int32_t* n_bad,
                                    orx_stream_t s);
ORX_API int orx_bag_gather_bf16(orx_handle_t h, const uint16_t* const* tabs_host, const int64_t* rows_host, int32_t T,
                                int32_t dim, const int32_t* sparse, int64_t ld, const int32_t* col_off_host, int32_t B,
                                int32_t mode, float* out, int64_t out_ld, int32_t* n_bad, orx_stream_t s);
ORX_API int orx_mlp_layer_fwd(orx_handle_t h, const float* x, int64_t ldx, int32_t B, int32_t in, const float* w,
                              const float* bias, int32_t out, int32_t act, float* y, int64_t ldy, orx_stream_t s);
ORX_API int orx_mlp_layer_bwd(orx_handle_t h, const float* x, int64_t ldx, const float* y, int64_t ldy, const float* w,
                              int32_t B, int32_t in, int32_t out, int32_t act, float* dy, int64_t lddy, float* dx,
                              int64_t lddx, float* dw, float* db, orx_stream_t s);
ORX_API int orx_interact_fwd(orx_handle_t h, const float* emb, int64_t emb_ld, const float* dense, int64_t dense_ld,
                             int32_t B, int32_t F, int32_t D, int32_t self_interaction, int32_t mode, float* out,
                             int64_t out_ld, orx_stream_t s);
ORX_API int orx_interact_bwd(orx_handle_t h, const float* emb, int64_t emb_ld, const float* dense, int64_t dense_ld,
                             const float* dout, int64_t dout_ld, int32_t B, int32_t F, int32_t D,
                             int32_t self_interaction, int32_t mode, float* demb, int64_t demb_ld, float* ddense,
                             int64_t ddense_ld, orx_stream_t s);
ORX_API int orx_pred_loss(orx_handle_t h, const float* pred, const float* label, int32_t B, int32_t kind,
                          float clip_threshold, float* pred_out, float* dpred, float* out4, orx_stream_t s);
/* DCN-v2 cross network (arch_interaction_op = "cross"; Wang et al. 2021, tfrs.layers.dcn.Cross): x0 [B, W] is the cross
 * input, layer l computes y_l = U_l (V_l^T x_l) + b_l (or K_l x_l + b_l at full rank) with orx_mlp_layer_fwd and
 * x_{l+1} = x0 * y_l + x_l with orx_cross_fwd.  The backward walks the layers top first with G = dL/dx_{l+1}:
 *   orx_cross_bwd(ORX_CROSS_TOP)   (layer L-1)  dy = G * x0, A = G * y                      (P not read, G not written)
 *   orx_cross_bwd(ORX_CROSS_MID)   (layer l)    G <- G + P_{l+1}, dy = G * x0, A <- A + G * y
 *   orx_cross_bwd(ORX_CROSS_FINAL)              dL/dx0 = G + P_0 + A: columns [0, split) to dx_lo, [split, W) to dx_hi
 * where dy = dL/dy_l feeds orx_mlp_layer_bwd of U_l and V_l, whose dx is P_l = dL/dx_l through the projection.  G and
 * A are updated in place.  All operands are row-major with explicit leading dimensions (>= their widths); each element
 * is rounded once per operation (products and a * b + c as one fused multiply-add), no atomics: the same inputs give
 * the same bits.  float4 accesses when W, every leading dimension the mode uses, split (FINAL) and every base it
 * touches allow them, a scalar path for any W >= 1.  One dispatch record per call (ORX_OP_CROSS).
 *   orx_cross_fwd: out = x0 * y + xl (out may not alias the inputs).
 *   orx_cross_bwd: TOP reads G, x0, y and writes dy, A; MID reads G, P, x0, y, A and writes G, dy, A; FINAL reads G, P, A
 *   and writes dx_lo / dx_hi (dx_hi at column 0 of its rows); arguments a mode does not use may be null.
 * ORX_ERR_INVALID before any device work: a null handle or a null operand the mode uses, B < 0, W < 1, a leading
 * dimension below its width, an unknown mode, split outside [0, W].  B = 0 is a no-op. */
enum orx_cross_mode { ORX_CROSS_TOP = 0, ORX_CROSS_MID = 1, ORX_CROSS_FINAL = 2 };
ORX_API int orx_cross_fwd(orx_handle_t h, const float* x0, int64_t ld_x0, const float* xl, int64_t ld_xl, const float* y,
                          int64_t ld_y, int32_t B, int32_t W, float* out, int64_t ld_out, orx_stream_t s);
ORX_API int orx_cross_bwd(orx_handle_t h, int32_t mode, int32_t B, int32_t W, float* G, int64_t ld_G, const float* P,
                          int64_t ld_P, const float* x0, int64_t ld_x0, const float* y, int64_t ld_y, float* A,
                          int64_t ld_A, float* dy, int64_t ld_dy, int32_t split, float* dx_lo, int64_t ld_lo,
                          float* dx_hi, int64_t ld_hi, orx_stream_t s);

/* ---- inference: full-catalogue scoring (bpr.py:39-43, wrmf.py:36-40, ucml.py:50-53, gmf.py:36-41)
 * scores[Bu, I] = user_rows . item^T + bias   (DOT; GMF passes user_rows pre-multiplied by w via `scale`)
 *               = -||user_row - item||^2 + bias (NEG_SQDIST).  scale may be NULL, and so may item_bias (no bias).
 * A uid outside [0, U) scores as a zero user row: 0 + bias (DOT), -||item||^2 + bias (NEG_SQDIST). */
ORX_API int orx_score_all(orx_handle_t h, int32_t kind, const float* user_tab, int64_t U, const int32_t* uid, int32_t Bu,
                  const float* scale, const float* item_tab, const float* item_bias, int64_t I, int32_t dim,
                  float* scores, orx_stream_t s);

/* ---- scoring on bf16 tables: orx_score_all_bf16, orx_score_rank_bf16, orx_score_rank_listed_bf16 and
 * orx_score_topk_bf16 take the user and item tables as bf16 bits (uint16_t) and are otherwise their fp32 forms.
 * Each element is widened to fp32 exactly as it is read; scale, item_bias, the arithmetic and its order are fp32 and
 * unchanged.  So every output (scores, auc / ndcg / recall, top_items, top_scores, NaN and +-inf included) equals the
 * fp32 form called on the fp32 upcast of the two tables, bit for bit.  The refusals, size limits, bad-uid rule, CSR
 * rules, scratch, determinism and dispatch fields are those of the fp32 form (orx_score_rank_bf16 logs
 * ORX_OP_SCORE_RANK_BF16, orx_score_topk_bf16 ORX_OP_SCORE_TOPK_BF16, the other two nothing).  Alignment: a table at
 * any 2-byte-aligned address is accepted and gives the same bits; with dim % 4 == 0 and both tables 8-byte aligned the
 * catalogue passes of orx_score_rank_bf16 / orx_score_topk_bf16 load 4 columns at a time, which is faster.  No
 * sharded form takes bf16 tables. */
ORX_API int orx_score_all_bf16(orx_handle_t h, int32_t kind, const uint16_t* user_tab, int64_t U, const int32_t* uid,
                               int32_t Bu, const float* scale, const uint16_t* item_tab, const float* item_bias,
                               int64_t I, int32_t dim, float* scores, orx_stream_t s);

/* ---- device-side samplers (SURVEY 8f N3; semantics of openrec/tf2/data/dataset.py:7-58 + data/utils.py:82-87,102-116).
 * orx_sampler_t: the interaction records, the random permutations of the current and of the next epoch (records are
 * consumed in permutation order and never dropped: a batch that crosses the end of an epoch continues in perm_next),
 * `cursor` = records of the current epoch already consumed, and the users' positives as a CSR with sorted rows.
 * Every draw is a pure function of (seed, stream_pos + slot): stream_pos = samples emitted before this batch.
 *   orx_sample_pairwise     : slot b = record b from the cursor + one uniform negative rejected while positive for the user
 *   orx_sample_stratified   : per slot a coin: the next record (label 1) with probability pos_ratio, else a uniform
 *                             unobserved (user, item) pair (label 0); *n_pos_out (device) = records consumed by the batch
 *   orx_sample_per_positive : the stream "record, then `quota` distinct items != its positive" cut at stream_pos; the
 *                             cursor must point at the record of the group that contains stream_pos. */
typedef struct {
  const int32_t *rec_user, *rec_item;     /* [n_records] */
  const int64_t *perm_cur, *perm_next;    /* [n_records] each */
  int64_t cursor, n_records;
  const int64_t* csr_off;                 /* [total_users + 1] */
  const int32_t* csr_items;               /* [n_records], sorted inside each user's range */
  int32_t total_users, total_items;
} orx_sampler_t;
ORX_API int orx_sample_pairwise(orx_handle_t h, const orx_sampler_t* sd_host, uint64_t seed, int64_t stream_pos, int32_t B,
                                int32_t* uid, int32_t* pid, int32_t* nid, orx_stream_t s);
ORX_API int orx_sample_stratified(orx_handle_t h, const orx_sampler_t* sd_host, uint64_t seed, int64_t stream_pos, int32_t B,
                                  float pos_ratio, int32_t* uid, int32_t* iid, float* label, int32_t* n_pos_out,
                                  orx_stream_t s);
ORX_API int orx_sample_per_positive(orx_handle_t h, const orx_sampler_t* sd_host, uint64_t seed, int64_t stream_pos, int32_t B,
                                    int32_t quota, int32_t* uid, int32_t* iid, float* label, orx_stream_t s);

/* ---- ranking metrics (openrec/tf2/metrics/ranking_metrics.py:8-69), one row per user --------
 * pos/excl are uint8 masks [R, I]; at[] (host) the cut-offs; outputs auc[R], ndcg[R,n_at], recall[R,n_at]
 * (any may be NULL). */
#define ORX_MAX_AT 8 /* cut-offs of orx_rank_metrics / orx_score_rank */
ORX_API int orx_rank_metrics(orx_handle_t h, const float* pred, const uint8_t* pos, const uint8_t* excl, int32_t R,
                     int64_t I, const int32_t* at_host, int32_t n_at, float* auc, float* ndcg, float* recall,
                     orx_stream_t s);

/* ---- fused catalogue evaluation: orx_score_all + orx_rank_metrics in one call, without the [Bu, I] score matrix or
 * the dense masks (openrec_b200/tf2/metrics/evaluator.py).
 * For batch row b, u = uid[b]: positives = pos_items[pos_off[u] .. pos_off[u+1]), excluded = excl_items[excl_off[u] ..
 * excl_off[u+1]) (excl_off may be NULL = nothing excluded).  Each row sorted and unique; entries outside [0, I) are
 * ignored.  u outside [0, U): zero user row and empty lists.  Results equal orx_score_all followed by orx_rank_metrics
 * on the masks these lists describe.  max_pos (host) bounds every positive row length; a row longer than max_pos gets
 * NaN in all its outputs.  auc / ndcg / recall may each be NULL.  kind, scale, item_bias and the bad-uid rule are those
 * of orx_score_all; at most ORX_MAX_AT cut-offs.  Scratch of about 20 * Bu * (max_pos + 1) bytes comes from the
 * handle (its own allocation, grown on demand: a growing call synchronises the device). */
ORX_API int orx_score_rank(orx_handle_t h, int32_t kind, const float* user_tab, int64_t U, const int32_t* uid,
                           int32_t Bu, const float* scale, const float* item_tab, const float* item_bias, int64_t I,
                           int32_t dim, const int64_t* pos_off, const int32_t* pos_items, const int64_t* excl_off,
                           const int32_t* excl_items, int32_t max_pos, const int32_t* at_host, int32_t n_at,
                           float* auc, float* ndcg, float* recall, orx_stream_t s);
/* orx_score_rank on bf16 tables (see orx_score_all_bf16): bit-equal to orx_score_rank on their fp32 upcast. */
ORX_API int orx_score_rank_bf16(orx_handle_t h, int32_t kind, const uint16_t* user_tab, int64_t U, const int32_t* uid,
                                int32_t Bu, const float* scale, const uint16_t* item_tab, const float* item_bias,
                                int64_t I, int32_t dim, const int64_t* pos_off, const int32_t* pos_items,
                                const int64_t* excl_off, const int32_t* excl_items, int32_t max_pos,
                                const int32_t* at_host, int32_t n_at, float* auc, float* ndcg, float* recall,
                                orx_stream_t s);

/* ---- sharded catalogue evaluation: orx_score_rank over row-sharded user / item tables (the layout of orx_shard_step:
 * row r of every table lives on rank r % world at local row r / world), each rank counting over its own item rows
 * (openrec_b200/sharded.py score_rank_sharded, RankingEvaluator on ShardedBPR / ShardedUCML).
 * orx_rowshard_t: the geometry; local_* = ceil((total - rank) / world), which may be 0.
 * The call runs one phase.  Between phases the caller replaces each exchange buffer with its element-wise integer SUM
 * over all ranks (an all-reduce on the int32 / int64 words); every phase writes every element of the buffer it
 * produces, so no buffer needs clearing.  With P = max_pos + 1, and sizes from orx_score_rank_shard_sizes
 * (n3 = {Bu * dim, Bu * P, Bu * P} elements):
 *   phase 0 reads the user shard and writes xrows[b] = the bits of user row uid[b] if this rank owns it, else 0;
 *   phase 1 reads the summed xrows and writes xpred[b, q] = the bits of the score of the q-th positive of uid[b] in
 *           [0, total_items) if this rank owns that item, else 0 (all 0 for a row longer than max_pos);
 *   phase 2 reads the summed xrows and xpred, scores this rank's item rows and writes xcnt[b, 0] = its AUC count and
 *           xcnt[b, 1..n] = its rank-histogram hits, both after taking back its own items of pos u excl (two's
 *           complement; a partial may be negative), the rest of the row 0;
 *   phase 3 reads the summed xcnt and writes auc / ndcg / recall (each may be NULL).
 * Exactly one rank contributes a non-zero word to each element of xrows and xpred, so the integer sum carries the float
 * bits unchanged (-0.0, NaN payloads, +-inf), which a float sum would not.  uid holds global user ids; the CSR lists are
 * the global lists of orx_score_rank, present on every rank.  Phase 3's outputs equal orx_score_rank on the global
 * tables (scale NULL): AUC and Recall bit for bit, NDCG within one float32 ulp; the bad-uid rule, ignored list
 * entries, max_pos, excl_off == NULL and the cut-offs are those of orx_score_rank.
 * Item row i is read only at local row i / world on the rank i % world, and only for i < total_items: a rank without
 * items (local_items == 0) may pass a 1-row dummy shard that is never read, and launches no empty grid.
 * No handle state crosses a phase boundary: one handle may serve several ranks, with any call between phases.  Phase 2
 * uses the evaluation scratch of orx_score_rank and writes one dispatch record (ORX_OP_SCORE_RANK_SHARD).
 * ORX_ERR_INVALID before any device work: local_* that disagree with (total, world, rank), rank outside [0, world),
 * phase outside [0, 3], the size limits of orx_score_rank, a null buffer the phase reads or writes.  Bu = 0 is a no-op.
 * There is no scale argument: a scaled score (GMF) scales the summed xrows in place with orx_rows_scale between phase 0
 * and phase 1, which gives orx_score_rank's scores with scale = w bit for bit. */
typedef struct {
  int32_t world, rank;               /* row r of every table lives on rank r % world at local row r / world */
  int64_t total_users, total_items;  /* global U, I */
  int64_t local_users, local_items;  /* rows of this rank's shards */
} orx_rowshard_t;
ORX_API int orx_score_rank_shard_sizes(int32_t Bu, int32_t dim, int32_t max_pos, int64_t* n3_host);
ORX_API int orx_score_rank_shard(orx_handle_t h, int32_t kind, int32_t phase, const orx_rowshard_t* g_host,
                                 const float* user_shard, const float* item_shard, const float* bias_shard,
                                 int32_t dim, const int32_t* uid, int32_t Bu, const int64_t* pos_off,
                                 const int32_t* pos_items, const int64_t* excl_off, const int32_t* excl_items,
                                 int32_t max_pos, const int32_t* at_host, int32_t n_at, int32_t* xrows /*[Bu, dim]*/,
                                 int32_t* xpred /*[Bu, P]*/, int64_t* xcnt /*[Bu, P]*/, float* auc, float* ndcg,
                                 float* recall, orx_stream_t s);

/* ---- listed-candidate evaluation: AUC / NDCG / Recall of datasets with explicit negatives, each user ranked against
 * its listed items only (the sampled-metrics protocol: a user's held-out positives against about 100 listed negatives;
 * openrec_b200/tf2/metrics/evaluator.py CandidateEvaluator).  No pass over the catalogue: the work is one item row per
 * listed entry and positive.
 * For batch row b, u = uid[b]: three CSR rows indexed by user id, positives P (pos_off / pos_items), listed items L
 * (neg_off / neg_items) and exclusions E (excl_off / excl_items; excl_off may be NULL = E empty), each sorted and
 * unique, entries outside [0, I) ignored.  Results equal orx_score_all followed by orx_rank_metrics on the masks
 * Dataset.evaluation builds for such a dataset: pos = P, excl = ~(P u L) u E.  So:
 *   AUC    = sum over the eval items i in L \ P \ E of #{p in P : pred_p >= s_i}, over |P| * |L \ P \ E| (a row with no
 *            eval item gets 0 / 0 = NaN);
 *   sp     = expf(score) on (P u L) \ E and 0 elsewhere; rank_p = #{i : sp_i > sp_p}; NDCG / Recall from rank_p;
 *   a positive in E keeps its pred for AUC and has sp 0; a listed item that is also a positive is a positive.
 * AUC and Recall are bit-equal to those of orx_score_all + orx_rank_metrics, and to orx_score_rank called with the
 * exclusion rows ~(P u L) u E; NDCG equals them within one float32 ulp (float64 sums in another order).  kind, scale,
 * item_bias, the bad-uid rule, max_pos, the cut-offs, the scratch and the size limits are those of orx_score_rank; the
 * call writes no dispatch record.
 * ORX_ERR_INVALID before any device work: the refusals of orx_score_rank, and neg_off NULL.  Bu = 0 is a no-op.  The
 * scratch is orx_score_rank's own allocation, so a call between orx_pairwise_prefetch and its step leaves the
 * prefetched index alone. */
ORX_API int orx_score_rank_listed(orx_handle_t h, int32_t kind, const float* user_tab, int64_t U, const int32_t* uid,
                                  int32_t Bu, const float* scale, const float* item_tab, const float* item_bias,
                                  int64_t I, int32_t dim, const int64_t* pos_off, const int32_t* pos_items,
                                  const int64_t* neg_off, const int32_t* neg_items, const int64_t* excl_off,
                                  const int32_t* excl_items, int32_t max_pos, const int32_t* at_host, int32_t n_at,
                                  float* auc, float* ndcg, float* recall, orx_stream_t s);
/* orx_score_rank_listed on bf16 tables (see orx_score_all_bf16): bit-equal to orx_score_rank_listed on their fp32
 * upcast; no dispatch record. */
ORX_API int orx_score_rank_listed_bf16(orx_handle_t h, int32_t kind, const uint16_t* user_tab, int64_t U,
                                       const int32_t* uid, int32_t Bu, const float* scale, const uint16_t* item_tab,
                                       const float* item_bias, int64_t I, int32_t dim, const int64_t* pos_off,
                                       const int32_t* pos_items, const int64_t* neg_off, const int32_t* neg_items,
                                       const int64_t* excl_off, const int32_t* excl_items, int32_t max_pos,
                                       const int32_t* at_host, int32_t n_at, float* auc, float* ndcg, float* recall,
                                       orx_stream_t s);
/* orx_score_rank_listed over row-sharded tables: the four phases, buffers (sizes from orx_score_rank_shard_sizes),
 * exchange and geometry rules of orx_score_rank_shard.  Phases 0 and 1 are its phases 0 and 1; phase 2 writes
 * xcnt[b, 0] = the AUC count of the eval items this rank owns and xcnt[b, 1..n] the rank hits of the listed items and
 * positives outside E that it owns; phase 3 reads the summed xcnt and writes auc / ndcg / recall, counting the eval
 * items from the global lists.  Phase 3's outputs equal orx_score_rank_listed on the global tables (scale NULL): AUC and
 * Recall bit for bit, NDCG within one float32 ulp.  No handle state crosses a phase boundary.  ORX_ERR_INVALID before
 * any device work: the refusals of orx_score_rank_shard, and (Bu > 0) neg_off NULL.  Bu = 0 is a no-op.  GMF scales the
 * summed xrows with orx_rows_scale between phase 0 and phase 1. */
ORX_API int orx_score_rank_listed_shard(orx_handle_t h, int32_t kind, int32_t phase, const orx_rowshard_t* g_host,
                                        const float* user_shard, const float* item_shard, const float* bias_shard,
                                        int32_t dim, const int32_t* uid, int32_t Bu, const int64_t* pos_off,
                                        const int32_t* pos_items, const int64_t* neg_off, const int32_t* neg_items,
                                        const int64_t* excl_off, const int32_t* excl_items, int32_t max_pos,
                                        const int32_t* at_host, int32_t n_at, int32_t* xrows /*[Bu, dim]*/,
                                        int32_t* xpred /*[Bu, P]*/, int64_t* xcnt /*[Bu, P]*/, float* auc,
                                        float* ndcg, float* recall, orx_stream_t s);

/* ---- catalogue top-K retrieval: each batch row's k best unseen items in one fused pass, without the [Bu, I] score
 * matrix (openrec_b200/tf2/recommenders/retriever.py; closest reference: openrec/tf1's FastDotProductServer).
 * Scores and conventions are those of orx_score_all, unchanged: the score of (b, i) with kind, scale and item_bias as
 * there; a uid outside [0, U) scores as a zero user row and has an empty exclusion list.  Exclusion lists follow the
 * CSR conventions of orx_score_rank: row u = excl_items[excl_off[u] .. excl_off[u+1]), sorted and unique, entries
 * outside [0, I) ignored, excl_off == NULL meaning nothing is excluded.
 * Eligible items: item i is eligible for row b when 0 <= i < I, i is not in uid[b]'s exclusion row, and its score is
 * not NaN.
 * Order: row b of the output is the first k eligible items in the total order "score descending, then item id
 * ascending".  Scores compare as floats, so -0.0 == +0.0, and -inf is a valid score.
 * Padding: when fewer than k items are eligible, the remaining slots hold item -1 and score -inf.
 * Score values: top_scores[b, j] equals the orx_score_all value of (uid[b], top_items[b, j]) bit for bit, except that
 * a -0.0 may come back as +0.0.  top_scores may be NULL.
 * Argument limits: 1 <= k <= ORX_MAX_TOPK, and k > I is allowed.  Bu = 0 is a no-op.  The other size checks are those
 * of orx_score_rank.
 * Determinism: the result does not depend on the number of item splits, on how many other users share the call, or on
 * the order of atomics, so the same inputs give the same bits on every call and every handle.
 * Scratch: 8 * Bu * S * (k + 1024) + 4 * Bu * S bytes (plus 512 bytes of alignment), S = the item splits of the
 * dispatch record (one wave of CTAs over the SMs divided among the ceil(Bu / 128) user tiles, at least 1 and at most
 * ceil(I / 128)), from the handle's evaluation scratch of
 * orx_score_rank: its own allocation, grown on demand (a growing call synchronises the device), so a call between
 * orx_pairwise_prefetch and its step leaves the prefetched index alone. */
#define ORX_MAX_TOPK 1024
ORX_API int orx_score_topk(orx_handle_t h, int32_t kind, const float* user_tab, int64_t U, const int32_t* uid,
                           int32_t Bu, const float* scale, const float* item_tab, const float* item_bias, int64_t I,
                           int32_t dim, const int64_t* excl_off, const int32_t* excl_items, int32_t k,
                           int32_t* top_items /*[Bu, k]*/, float* top_scores /*[Bu, k], may be NULL*/, orx_stream_t s);
/* orx_score_topk on bf16 tables (see orx_score_all_bf16): bit-equal to orx_score_topk on their fp32 upcast, with the
 * same item splits and scratch. */
ORX_API int orx_score_topk_bf16(orx_handle_t h, int32_t kind, const uint16_t* user_tab, int64_t U, const int32_t* uid,
                                int32_t Bu, const float* scale, const uint16_t* item_tab, const float* item_bias,
                                int64_t I, int32_t dim, const int64_t* excl_off, const int32_t* excl_items, int32_t k,
                                int32_t* top_items /*[Bu, k]*/, float* top_scores /*[Bu, k], may be NULL*/,
                                orx_stream_t s);

/* ---- sharded top-K retrieval: orx_score_topk over row-sharded user / item tables (orx_rowshard_t, the layout of
 * orx_score_rank_shard), each rank keeping the k best of its own item rows (openrec_b200/sharded.py score_topk_sharded,
 * Retriever on ShardedBPR / ShardedUCML).
 * The call runs one phase; between phases the caller replaces each exchange buffer with its element-wise integer SUM
 * over all ranks.  Buffers: xrows int32 [Bu, dim], xkeys int64 [Bu, world, k], top_items int32 [Bu, k], top_scores
 * float [Bu, k] (may be NULL).
 *   phase 0 reads the user shard and writes xrows[b] = the bits of user row uid[b] if this rank owns it, else 0 (the
 *           phase 0 of orx_score_rank_shard);
 *   phase 1 reads the summed xrows, scores this rank's item rows and writes xkeys[b, rank] = the 64-bit keys of its k
 *           best eligible items of row b (score bits high, ~global item id low), sorted descending and padded with 0,
 *           and 0 into every other rank's slot of xkeys (every element written);
 *   phase 2 reads the summed xkeys and writes top_items / top_scores: the top k of the union of the ranks' keys.
 * Exactly one rank contributes a non-zero word to each element of xrows and xkeys, so the sum carries them unchanged.
 * Phase 2's outputs equal orx_score_topk on the global tables (scale NULL) bit for bit, whatever world is: the
 * eligibility, order, padding, bad-uid and exclusion-list rules are those of orx_score_topk, applied to global item
 * ids.  uid holds global user ids; the exclusion CSR is the global one, present on every rank.
 * A rank without items (local_items == 0) may pass a 1-row dummy shard: phase 1 then writes an all-zero xkeys and
 * launches no main pass.  No handle state crosses a phase boundary: phase 1 uses the scratch of orx_score_topk for its
 * own pass and merge only, so one handle may serve several ranks, with any call between phases.
 * The exchange moves 4 * Bu * dim + 8 * Bu * world * k bytes per call.
 * ORX_ERR_INVALID before any device work: the geometry checks of orx_score_rank_shard, phase outside [0, 2], k outside
 * [1, ORX_MAX_TOPK] (k > total_items is allowed), Bu * world * k > 2^31 - 1, a null buffer the phase reads or writes.
 * Bu = 0 is a no-op.  There is no scale argument: GMF scales the summed xrows with orx_rows_scale between phase 0 and
 * phase 1, as for orx_score_rank_shard. */
ORX_API int orx_score_topk_shard(orx_handle_t h, int32_t kind, int32_t phase, const orx_rowshard_t* g_host,
                                 const float* user_shard, const float* item_shard, const float* bias_shard,
                                 int32_t dim, const int32_t* uid, int32_t Bu, const int64_t* excl_off,
                                 const int32_t* excl_items, int32_t k, int32_t* xrows /*[Bu, dim]*/,
                                 int64_t* xkeys /*[Bu, world, k]*/, int32_t* top_items /*[Bu, k]*/,
                                 float* top_scores /*[Bu, k], may be NULL*/, orx_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* ORX_H_ */
