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
 *    id staging, evaluation scratch, sharded-step scratch, split-K partials), keeps no device
 *    state outside it, and orx_destroy frees all of it.  Two handles share nothing;
 *  - all calls are asynchronous w.r.t. the host and ordered on the given stream;
 *  - return value: ORX_OK (0) or a negative orx_status; orx_last_error_string() gives the
 *    thread-local message.  There is no CPU fallback: without a CUDA device every compute
 *    entry point fails with ORX_ERR_CUDA.
 *  - tables are row-major float32 [rows, dim] with 64-bit row offsets; ids are int32.
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
 * For Adam s0 = m, s1 = v, lr_t = lr*sqrt(1-beta2^step)/(1-beta1^step), step is 1-based. */
enum orx_opt_kind { ORX_OPT_SGD = 0, ORX_OPT_ADAGRAD = 1, ORX_OPT_ADAM_LAZY = 2, ORX_OPT_ADAM_DENSE = 3 };

typedef struct {
  int32_t kind; /* orx_opt_kind */
  float lr, eps, beta1, beta2;
  int64_t step; /* Adam: 1-based iteration count of THIS apply */
} orx_opt_t;

/* One LatentFactor (openrec/tf2/modules/latent_factor.py:4-15) and its optimizer slots. */
typedef struct {
  float* var;   /* [rows, dim] */
  float* s0;    /* Adagrad accumulator | Adam m ; NULL for SGD */
  float* s1;    /* Adam v ; NULL otherwise */
  int64_t rows;
  int32_t dim;
} orx_table_t;

/* ---- context ------------------------------------------------------------------------- */
ORX_API int orx_abi_version(void);
ORX_API const char* orx_last_error_string(void); /* host, thread-local */
ORX_API int orx_create(int device, orx_handle_t* out);
ORX_API int orx_destroy(orx_handle_t h);
ORX_API int orx_device_count(int* n_out_host);
/* Blocks the host until `stream` has drained (cudaStreamSynchronize). */
ORX_API int orx_stream_synchronize(orx_handle_t h, orx_stream_t stream);
/* Test hook: place the handle's batch-index epoch counter (31 bits; the wrap path empties the hash tables). */
ORX_API int orx_debug_set_epoch(orx_handle_t h, uint32_t epoch);
/* Test hook: the kernel variants launched by this handle's DLRM entry points (orx_mlp_layer_*, orx_interact_*) and
 * sparse steps (orx_pairwise_step, orx_pairwise_step_host, orx_pointwise_step) since the last call, oldest first, at
 * most cap of them (a ring of the last ORX_DISPATCH_LOG_CAP), then clears them.
 * Record k is rec_host[8k .. 8k+7] = {op, variant, TA, TB, M, N, K, S}: a GEMM C[M,N] = op(A)[M,K] op(B)[K,N] with the
 * operand layouts TA / TB of orx_dlrm.cu and S split-K slices (1 = no split); an interaction has M = B, N = F, K = D,
 * TA = TB = 0, S = 1.  A sparse step (one record per call) has TA = kind (orx_pair_kind / orx_point_kind), TB = optimizer
 * (orx_opt_kind), M = B, N = D, K = the CTAs/SM bound of the fused kernel's __launch_bounds__ (0: none) and S = the batch
 * index set it used: 0 = built on the caller's stream, 1 or 2 = a consumed prefetch (orx_pairwise_prefetch, or the side
 * stream of orx_pairwise_step_host).  orx_score_rank and orx_score_topk write one record per call (fields at
 * ORX_OP_SCORE_RANK / ORX_OP_SCORE_TOPK).
 * Host-side bookkeeping only: no device work, no synchronisation. */
enum orx_dispatch_op {
  ORX_OP_GEMM = 0,
  ORX_OP_INTERACT_FWD = 1,
  ORX_OP_INTERACT_BWD = 2,
  ORX_OP_PAIRWISE_STEP = 3,  /* orx_pairwise_step, orx_pairwise_step_host */
  ORX_OP_POINTWISE_STEP = 4, /* orx_pointwise_step */
  ORX_OP_SCORE_RANK = 5,     /* orx_score_rank: TA = orx_score_kind, TB = 0, M = Bu, N = I, K = dim, S = item splits */
  ORX_OP_SCORE_TOPK = 6      /* orx_score_topk: TA = orx_score_kind, TB = k, M = Bu, N = I, K = dim, S = item splits */
};
enum orx_dispatch_variant {
  ORX_VARIANT_GEMM_TMA = 0,      /* k_gemm_tma: TMA-fed wgmma 3xTF32 (orx_mlp_tc.cu) */
  ORX_VARIANT_GEMM_SIMT = 1,     /* k_gemm: fp32 SIMT tiles */
  ORX_VARIANT_INTERACT_WARP = 2, /* k_interact_{fwd,bwd}_warp: one warp per sample */
  ORX_VARIANT_INTERACT = 3,      /* k_interact_{fwd,bwd}: one CTA per sample */
  ORX_VARIANT_STEP = 4,          /* k_pair_step / k_point_step specialised on D (32, 64, 128, 256), one register buffer */
  ORX_VARIANT_STEP_PIPE = 5,     /* k_pair_step with the register double buffer (PIPE) */
  ORX_VARIANT_STEP_GENERIC = 6,  /* k_pair_generic / k_point_generic (fused-step mode): any D */
  ORX_VARIANT_RANK_SMEM = 7,     /* k_score_rank: thresholds and histograms of a user tile in shared memory */
  ORX_VARIANT_RANK_GLOBAL = 8,   /* k_score_rank: thresholds and histograms in the handle's global scratch */
  ORX_VARIANT_TOPK = 9           /* k_score_topk + k_topk_merge: candidate lists in the handle's global scratch */
};
#define ORX_DISPATCH_LOG_CAP 64
ORX_API int orx_debug_dispatch_log(orx_handle_t h, int32_t* rec_host, int32_t cap, int32_t* n_host);

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
 * values = dZ[:,k,:]). */
ORX_API int orx_sparse_apply_strided(orx_handle_t h, const orx_table_t* tab, const int32_t* ids, int64_t id_stride,
                                     const float* values, int64_t value_ld, int32_t n, const orx_opt_t* opt_host,
                                     orx_stream_t s);
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
 *   All ranks announce, or none.  The announced step's user index lives in the handle's index sets until that call:
 *   meanwhile (and between the phases of a step issued phase by phase) any call on the handle that would grow its
 *   workspace, orx_pairwise_prefetch / orx_pairwise_step_host, and an index-epoch take that would wrap return
 *   ORX_ERR_INVALID before any device work.  Calls that need none of these (orx_pairwise_step within the workspace,
 *   scoring, sampling) are accepted.
 *   out4 = { loss, l2_loss (GLOBAL batch, identical on every rank), skipped triplets of this rank, staged rows }.
 *   The sticky error word flags[4*64] is 0 or: 1 a peer never arrived within timeout_ms, 2 more triplets routed to this
 *   home than home_cap, 3 / 4 request / gradient inbox too small.  SGD, Adagrad and row-sparse Adam. */
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

/* ---- inference: full-catalogue scoring (bpr.py:39-43, wrmf.py:36-40, ucml.py:50-53, gmf.py:36-41)
 * scores[Bu, I] = user_rows . item^T + bias   (DOT; GMF passes user_rows pre-multiplied by w via `scale`)
 *               = -||user_row - item||^2 + bias (NEG_SQDIST).  scale may be NULL, and so may item_bias (no bias).
 * A uid outside [0, U) scores as a zero user row: 0 + bias (DOT), -||item||^2 + bias (NEG_SQDIST). */
ORX_API int orx_score_all(orx_handle_t h, int32_t kind, const float* user_tab, int64_t U, const int32_t* uid, int32_t Bu,
                  const float* scale, const float* item_tab, const float* item_bias, int64_t I, int32_t dim,
                  float* scores, orx_stream_t s);

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

#ifdef __cplusplus
}
#endif
#endif /* ORX_H_ */
