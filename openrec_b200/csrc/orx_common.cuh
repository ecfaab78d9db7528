// orx_common.cuh -- shared host/device helpers for liborx (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <functional>
#include <initializer_list>
#include <type_traits>

#include "../../include/orx.h"

// ---------------------------------------------------------------------------------------
// host: errors + context
// ---------------------------------------------------------------------------------------
void orx_set_error(const char* fmt, ...);

#define ORX_CUDA(call)                                                                         \
  do {                                                                                         \
    cudaError_t e__ = (call);                                                                  \
    if (e__ != cudaSuccess) {                                                                  \
      orx_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));     \
      return ORX_ERR_CUDA;                                                                     \
    }                                                                                          \
  } while (0)

#define ORX_REQUIRE(cond, msg)                                  \
  do {                                                          \
    if (!(cond)) {                                              \
      orx_set_error("%s: %s", __func__, msg);                   \
      return ORX_ERR_INVALID;                                   \
    }                                                           \
  } while (0)

#define ORX_LAUNCH_CHECK() ORX_CUDA(cudaGetLastError())

// Open-addressing hash index over the ids of one table for one batch ("K9").
// slot word: [63:33] epoch | [32] "seen more than once" | [31:0] id.  A slot whose epoch differs from the
// current one is EMPTY, so the table is never cleared: every step just uses a new epoch (31 bits).
struct OrxHash {
  unsigned long long* slots;  // [cap]
  int32_t* didx;              // [cap]  compact staging index of a staged row
  int32_t* did;               // [cap_rows] row id of staging index d
  int32_t* counter;           // number of staged rows
  uint32_t mask;
  int32_t shift;  // 32 - log2(cap)
  uint32_t epoch;  // current epoch, >= 1
};

// Shape of an index set for `lookups` ids: sets t.mask and t.shift, returns the slot count, the least power of two
// (>= 1024) that holds 4x the lookups.  did takes lookups + 1 entries.
uint32_t orx_hash_shape(OrxHash& t, int64_t lookups);

// 256-byte aligned bump allocation inside one buffer.  With a null base it only counts bytes (off = the size so far).
struct OrxCarve {
  char* base;
  size_t off;
  void* take(size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += (bytes + 255) & ~(size_t)255;
    return p;
  }
};

// slots | didx | did of a table for `lookups` ids (orx_hash_shape); counter and epoch are the caller's
void orx_hash_carve(OrxCarve& m, OrxHash& t, int64_t lookups);

// Start the next epoch of table t (31 bits, skipping 0), for an index build into t on `st`.  On the wrap only t's slots
// are emptied, on `st`: every launch that writes or probes t runs on `st` or is ordered before this point, so no stale
// slot can alias the epochs to come (about 65 h of back-to-back steps between wraps).
int orx_take_epoch(OrxHash& t, cudaStream_t st);

// One batch index set of the handle: user / item tables, the control words of the steps that use it and, for the
// prefetch sets 1 and 2 (pairwise batches indexed ahead on the side stream, orx_pairwise.cu), their records, events
// and what the outstanding prefetch was built for.
struct OrxIndexSet {
  OrxHash u, i;
  int32_t* ctl;   // [4] staged_u (u.counter), staged_i (i.counter), tail block ticket, bad ids: TailArgs::counters
  int4* res;      // sets 1, 2 with ORX_PAIR_RESOLVE: per-triplet records {flags, du, dp, dn} (k_index_resolve)
  cudaEvent_t done, free;   // index built / handed back by the step that consumed it
  int free_valid;
  const int32_t *uid, *pid, *nid;
  int B, mode;
  int64_t rows_u, rows_i;
};

struct orx_ctx {
  int device;
  int num_sms;
  // index workspace, one allocation (sized for cap_B lookups per table side, staging rows of g_dim floats): set 0 for
  // everything that builds its index on the caller's stream, sets 1 and 2 for prefetched pairwise batches, then the
  // staged-row gradient buffers
  int64_t cap_B;  // largest batch the workspace is sized for
  int32_t g_dim;
  void* index_ws;
  size_t index_cap;
  OrxIndexSet set[3];
  int pf_set;     // the outstanding prefetched set (1 or 2), 0 = none
  int pf_next;    // the next prefetch builds into set 1 + pf_next
  float *gu, *gi, *gb, *gw;
  // loss partials: (loss, l2) float pairs
  float* partials;
  size_t partials_cap;   // bytes
  // id staging for the *_host entry points (double buffered)
  int32_t* ids_stage[2];
  size_t stage_cap[2];   // bytes
  float* out_stage[2];
  uint32_t stage_flip;
  // measurement hook (orx_profile_*)
  int prof_on, prof_n, prof_cap;
  int prof_step;  // steps seen since orx_profile_enable: every 8th one carries the phase events
  cudaEvent_t* prof_ev;  // [prof_cap * ORX_PROF_EV]
  int32_t* bucket_cursor;  // [1024] owner-bucket scratch
  cudaStream_t side_stream;  // id upload + index build of the NEXT pairwise batch, beside the running step
  cudaEvent_t side_ev;       // "ids are final" point of orx_pairwise_prefetch on the caller's ids stream
  cudaEvent_t stage_free[2];   // id staging f free
  int stage_free_valid[2];
  int pair_resolve;        // ORX_PAIR_RESOLVE, read at orx_create: 0 = no records, a prefetched step probes the index
  void* shard_ws;         // orx_shard.cu: host bookkeeping of the row-sharded step (orx_shard_ws*)
  void* shard_scratch;     // orx_shard.cu: its local device scratch, carved by sh_layout
  size_t shard_cap;
  int32_t dispatch[ORX_DISPATCH_LOG_CAP][8];   // orx_debug_dispatch_log: ring of the last DLRM / sparse-step launches
  int64_t dispatch_n;      // records written since the last read
  void* eval_ws;           // orx_eval.cu: scratch of orx_score_rank / orx_score_topk, its own allocation
  size_t eval_cap;
  void* lookup_ws;         // orx_dlrm_shard.cu: scratch of orx_lookup_bucket (keys, scan, sort storage)
  size_t lookup_cap;
  float* splitk;           // split-K partials of the Dense-layer GEMMs and of the split column sum
  size_t splitk_cap;
  void* censor_ws;         // orx_misc.cu: the dedup hash of orx_censor_shard (slots only), its own allocation
  size_t censor_cap;
  OrxHash censor_hash;     // its slots, shape and epoch
  void* bag_ws;            // orx_sharded.cu: orx_bag_sparse_apply's compacted ids and bag counts, its own allocation
  size_t bag_cap;
  void* bag_cnt_ws;        // orx_dlrm_shard.cu: orx_bag_segment_sum's per-bag valid-id counts, its own allocation
  size_t bag_cnt_cap;
};

// Grow a workspace buffer of the handle to at least `need` bytes (*cap = its size in bytes).  Returns at once when it is
// large enough; otherwise drains the device (the old buffer may be in use on any stream), frees it and allocates the
// new one.  A failed allocation leaves *buf null and *cap 0 and returns ORX_ERR_NOMEM; a failed drain returns
// ORX_ERR_CUDA with the buffer untouched.
int orx_grow(void** buf, size_t* cap, size_t need);

// append {op, variant, TA, TB, M, N, K, S} to the handle's dispatch ring (host only)
static inline void orx_log_dispatch(orx_ctx* c, int op, int variant, int TA, int TB, int M, int N, int K, int S) {
  int32_t* r = c->dispatch[c->dispatch_n++ % ORX_DISPATCH_LOG_CAP];
  r[0] = op; r[1] = variant; r[2] = TA; r[3] = TB; r[4] = M; r[5] = N; r[6] = K; r[7] = S;
}

void orx_shard_ws_release(orx_ctx* c);
// orx_debug_set_epoch: place the epoch counters of the row-sharded step's own index sets too, once they exist
void orx_shard_set_epoch(orx_ctx* c, uint32_t epoch);

#define ORX_PROF_EV 8   // event slots per sampled step: up to 7 phases (the sharded step has seven launches)
// record phase boundary k (0..7) of the current step on `st` when profiling is enabled
// Only every 8th step is instrumented: four timing-event records per step sit between the kernels of the step that is
// being timed.  Suspected cost (not yet isolated): bench.py's un-instrumented UCML loop ran at 612 M/s against 555 M/s
// for the instrumented BPR loop in r1w although both step kernels take 71 us under ncu.
static inline bool orx_prof_sampled(const orx_ctx* c) {
  return c->prof_on && (c->prof_step & 7) == 0 && c->prof_n < c->prof_cap;
}
static inline void orx_prof_mark(orx_ctx* c, int k, cudaStream_t st) {
  if (orx_prof_sampled(c)) cudaEventRecord(c->prof_ev[c->prof_n * ORX_PROF_EV + k], st);
}
static inline void orx_prof_next(orx_ctx* c) {
  if (!c->prof_on) return;
  if (orx_prof_sampled(c)) c->prof_n++;
  c->prof_step++;
}

int orx_ensure_workspace(orx_ctx* c, int64_t B, int32_t dim);

// Runtime kind -> template argument: calls f(std::integral_constant<int, V>{}) for the V among Vs equal to v, and for the
// last of Vs when none is (every entry point validates v, with its own error message, before it dispatches).  Only the
// listed values are instantiated.
template <int V, int... Vs, typename F>
static inline auto orx_dispatch(int v, F&& f) {
  if constexpr (sizeof...(Vs) == 0) {
    return f(std::integral_constant<int, V>{});
  } else {
    if (v == V) return f(std::integral_constant<int, V>{});
    return orx_dispatch<Vs...>(v, f);
  }
}
// NESTEROV runs the MOMENTUM instances: orx_apply<MOMENTUM> picks the Nesterov form from OrxOptDev::kind, so every
// kernel has one momentum instance, not two.
template <typename F>
static inline auto orx_dispatch_opt(int opt_kind, F&& f) {
  return orx_dispatch<ORX_OPT_SGD, ORX_OPT_ADAGRAD, ORX_OPT_ADAM_LAZY, ORX_OPT_ADAM_DENSE, ORX_OPT_ROWWISE_ADAGRAD,
                      ORX_OPT_MOMENTUM>(opt_kind == ORX_OPT_NESTEROV ? ORX_OPT_MOMENTUM : opt_kind, f);
}

// an orx_opt_kind (4 and 7 are unassigned and refused: orx_dispatch_opt would otherwise run them as its last listed kind)
static inline bool orx_opt_kind_ok(int kind) {
  return (kind >= ORX_OPT_SGD && kind <= ORX_OPT_ADAM_DENSE) || kind == ORX_OPT_ROWWISE_ADAGRAD ||
         kind == ORX_OPT_MOMENTUM || kind == ORX_OPT_NESTEROV;
}
// The optimizer *o as a table of row width dim runs it: a dim-1 table under ROWWISE_ADAGRAD runs ADAGRAD (its one
// accumulator per row is the element-wise one, and the update then rounds exactly as ADAGRAD's).
static inline orx_opt_t orx_opt_dim(const orx_opt_t* o, int dim) {
  orx_opt_t r = *o;
  if (r.kind == ORX_OPT_ROWWISE_ADAGRAD && dim == 1) r.kind = ORX_OPT_ADAGRAD;
  return r;
}
// The host side of OrxOptSlots: every table carries the slot rows optimizer `kind` keeps -- s0 for every kind but SGD
// (ROWWISE_ADAGRAD: float[rows]), s1 for both Adams (ADAM_DENSE's sweep keeps m and v there).  Null tables are skipped.
bool orx_opt_slots_ok(int kind, std::initializer_list<const orx_table_t*> tabs);

// True when every pointer is 16-byte aligned (a null pointer, an absent slot row, counts as aligned).  The one rule of
// the 128-bit paths on caller memory (orx.h, Conventions): a table, slot row, dense weight or output buffer may start at
// any 4-byte-aligned address, and a call takes a float4 path only when this holds for every caller pointer that path
// reads or writes through.  Buffers the library carves itself (OrxCarve: 256-byte aligned) need no check.
template <typename... P>
static inline bool orx_aligned16(const P*... p) {
  return (((uintptr_t)0 | ... | (uintptr_t)p) & 15) == 0;
}

// True when every pointer is 8-byte aligned: the rule of a bf16 table's 4-element (8-byte) row path.
template <typename... P>
static inline bool orx_aligned8(const P*... p) {
  return (((uintptr_t)0 | ... | (uintptr_t)p) & 7) == 0;
}

// bf16 tables (orx_table_bf16_t): stochastic rounding of an update of table t (0 = user, 1 = item) at optimizer step
// `step`, as include/orx.h states it.  The per-(seed, step, t) part is taken once on the host.
__host__ __device__ inline uint32_t orx_mix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}
static inline uint64_t orx_mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}
static inline uint32_t orx_sr_table_key(uint64_t seed, int64_t step, int t) {
  return (uint32_t)(orx_mix64(seed ^ orx_mix64((uint64_t)step * 2u + (uint64_t)t)) >> 32);
}

// Grid of a grid-stride loop over n items: one thread per item, at most 32 blocks per SM, at least one block.
static inline int orx_grid_for(int64_t n, int threads, int num_sms) {
  const int64_t b = (n + threads - 1) / threads;
  const int64_t cap = (int64_t)num_sms * 32;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

// ---------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------
struct OrxOptDev {
  int32_t kind;
  float lr;    // SGD/Adagrad/momentum: lr ; Adam: bias-corrected lr_t
  float eps, beta1, beta2;   // MOMENTUM / NESTEROV: beta1 = the momentum coefficient
};

#ifdef __CUDACC__

#define ORX_FULL 0xffffffffu

// Programmatic dependent launch (sm_90+): a kernel launched with orx_launch_pdl may become resident while its
// predecessor on the stream is still draining; it must execute orx_pdl_wait() before it touches anything the predecessor
// wrote (a no-op when launched normally).  The predecessor calls orx_pdl_trigger() once a block has finished its main
// loop: the dependent grid is released when every block has triggered or exited, so launch latency and grid drain overlap.
__device__ __forceinline__ void orx_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void orx_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

bool orx_pdl_enabled();   // ORX_PDL=0 turns the attribute off (A/B measurements)

template <typename... KArgs, typename... Args>
static inline cudaError_t orx_launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                         Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = orx_pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

__device__ __forceinline__ uint32_t orx_hash32(uint32_t id, int shift) { return (id * 2654435769u) >> shift; }

#define ORX_DUP_BIT (1ull << 32)
__device__ __forceinline__ unsigned long long orx_slot_word(uint32_t epoch, int32_t id) {
  return ((unsigned long long)epoch << 33) | (unsigned long long)(uint32_t)id;
}

// Insert one id.  mode 0: rows get a staging index when they are seen the SECOND time (duplicates only);
// mode 1: on the FIRST occurrence (ADAM_DENSE stages every row); mode 2: never (pure dedup, censor).
// Returns 0 if this call was the first occurrence of the id in this epoch, else 1.
__device__ __forceinline__ uint32_t orx_hash_insert(const OrxHash& t, int32_t id, int mode) {
  const unsigned long long mine = orx_slot_word(t.epoch, id);
  uint32_t h = orx_hash32((uint32_t)id, t.shift);
  while (true) {
    unsigned long long w = __ldcg(t.slots + h);
    if ((uint32_t)(w >> 33) != t.epoch) {   // empty or stale: try to claim it
      const unsigned long long old = atomicCAS(t.slots + h, w, mine);
      if (old == w) {
        if (mode == 1) {
          const int d = atomicAdd(t.counter, 1);
          t.didx[h] = d;
          t.did[d] = id;
        }
        return 0u;
      }
      w = old;                              // somebody else claimed it meanwhile (same epoch by construction)
    }
    if ((w & ~ORX_DUP_BIT) == mine) {
      if (!(w & ORX_DUP_BIT)) {
        const unsigned long long old = atomicOr(t.slots + h, ORX_DUP_BIT);
        if (mode == 0 && !(old & ORX_DUP_BIT)) {   // this call made the row "shared": give it a staging slot
          const int d = atomicAdd(t.counter, 1);
          t.didx[h] = d;
          t.did[d] = id;
        }
      }
      return 1u;
    }
    h = (h + 1) & t.mask;
  }
}

// Loads at L2 evict-last priority, for the small random-access structures a step re-reads long after they were last
// touched (batch index, item bias + its slots) while it streams row traffic many times the L2 through the cache.  The
// policy is a per-access hint (createpolicy + .L2::cache_hint, carried in the uniform memory descriptor: no per-thread
// register); it configures no L2 set-aside, and the lines stay evictable.
__device__ __forceinline__ unsigned long long orx_ld_keep(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("{.reg .b64 pol; createpolicy.fractional.L2::evict_last.b64 pol, 1.0;\n"
               " ld.global.nc.L2::cache_hint.u64 %0, [%1], pol;}" : "=l"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ int32_t orx_ld_keep(const int32_t* p) {
  int32_t v;
  asm volatile("{.reg .b64 pol; createpolicy.fractional.L2::evict_last.b64 pol, 1.0;\n"
               " ld.global.nc.L2::cache_hint.b32 %0, [%1], pol;}" : "=r"(v) : "l"(p));
  return v;
}
// not .nc: the step that reads an item bias also writes it
__device__ __forceinline__ float orx_ld_keep(const float* p) {
  float v;
  asm volatile("{.reg .b64 pol; createpolicy.fractional.L2::evict_last.b64 pol, 1.0;\n"
               " ld.global.cg.L2::cache_hint.f32 %0, [%1], pol;}" : "=f"(v) : "l"(p));
  return v;
}

// Lookup.  Returns 0 = absent, 1 = present once, 2 = present more than once; *d = staging index if the row
// has one (duplicates in mode 0, every row in mode 1).
// DUP_ONLY (mode-0 indexes): the staging index is read only for a row present more than once, the only rows that have
// one, and *d = -1 otherwise; this saves a dependent random load per probe of a row seen once.  Callers that read *d of
// rows present once (mode 1: ADAM_DENSE stages every row) keep the default.
// KEEP: probe at L2 evict-last priority (orx_ld_keep), for kernels that stream table rows beside the probes.
template <bool DUP_ONLY = false, bool KEEP = false>
__device__ __forceinline__ uint32_t orx_hash_find(const OrxHash& t, int32_t id, int32_t* d) {
  const unsigned long long mine = orx_slot_word(t.epoch, id);
  uint32_t h = orx_hash32((uint32_t)id, t.shift);
  while (true) {
    const unsigned long long w = KEEP ? orx_ld_keep(t.slots + h) : __ldg(t.slots + h);
    if ((w & ~ORX_DUP_BIT) == mine) {
      const bool dup = (w & ORX_DUP_BIT) != 0;
      *d = (!DUP_ONLY || dup) ? (KEEP ? orx_ld_keep(t.didx + h) : __ldg(t.didx + h)) : -1;
      return dup ? 2u : 1u;
    }
    if ((uint32_t)(w >> 33) != t.epoch) {
      *d = -1;
      return 0u;
    }
    h = (h + 1) & t.mask;
  }
}

template <int W>
__device__ __forceinline__ float orx_group_sum(float v) {
#pragma unroll
  for (int o = W / 2; o > 0; o >>= 1) v += __shfl_xor_sync(ORX_FULL, v, o);
  return v;
}

__device__ __forceinline__ float4 orx_ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void orx_st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
// Table rows of the sparse steps (embedding rows and their optimizer-slot rows) at L2 evict-first priority
// (ld/st.global.cs -> LDG/STG.E.EF.128: no policy register).  A BPR step at the default bench size streams ~370 MB of
// random 512-byte rows through the 50 MB L2 of an H100, each read once and written once, so a row line is never hit
// again before it leaves.  Marking them evict-first leaves the L2 to what IS reused over the step: the batch index sets,
// item bias + its slots, and the compact staging rows (those stay at normal priority).
__device__ __forceinline__ float4 orx_ld4_stream(const float* p) { return __ldcs(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void orx_st4_stream(float* p, float4 v) { __stcs(reinterpret_cast<float4*>(p), v); }
// Row element access by storage type: a float table (every fp32 path, which these leave as it was) or a bf16 table held
// as its uint16_t bits.  A bf16 row moves 4 elements per lane as one 8-byte access (the table 8-byte aligned), widened
// to a float4 on load; all arithmetic is fp32, and only the store rounds: stochastically, with the row key
// rk = orx_sr_row(table key, row) and the element's column (orx_bf16_sr).  The float forms ignore rk and col.
__device__ __forceinline__ float orx_bf16_up(uint32_t b) { return __uint_as_float(b << 16); }
__device__ __forceinline__ uint32_t orx_sr_row(uint32_t kt, int64_t row) { return orx_mix32(kt ^ (uint32_t)row); }
__device__ __forceinline__ uint32_t orx_bf16_sr(float v, uint32_t rk, int col) {
  const uint32_t u = __float_as_uint(v);
  if ((u & 0x7f800000u) == 0x7f800000u) return (u >> 16) | ((u & 0x007fffffu) ? 0x40u : 0u);   // Inf; NaN stays NaN
  return (u + (orx_mix32(rk + (uint32_t)col * 0x9e3779b9u) >> 16)) >> 16;
}
// round to nearest even (assign, censor): not an optimizer update
__device__ __forceinline__ uint32_t orx_bf16_rne(float v) {
  const uint32_t u = __float_as_uint(v);
  if ((u & 0x7f800000u) == 0x7f800000u) return (u >> 16) | ((u & 0x007fffffu) ? 0x40u : 0u);
  return (u + 0x7fffu + ((u >> 16) & 1u)) >> 16;
}
__device__ __forceinline__ float orx_ld1(const float* p) { return *p; }
__device__ __forceinline__ float orx_ld1(const uint16_t* p) { return orx_bf16_up(*p); }
__device__ __forceinline__ void orx_st1(float* p, float v, uint32_t, int) { *p = v; }
__device__ __forceinline__ void orx_st1(uint16_t* p, float v, uint32_t rk, int col) {
  *p = (uint16_t)orx_bf16_sr(v, rk, col);
}
__device__ __forceinline__ float4 orx_bf16x4_up(uint2 b) {
  return make_float4(orx_bf16_up(b.x & 0xffffu), orx_bf16_up(b.x >> 16), orx_bf16_up(b.y & 0xffffu),
                     orx_bf16_up(b.y >> 16));
}
__device__ __forceinline__ uint2 orx_bf16x4_sr(float4 v, uint32_t rk, int col) {
  return make_uint2(orx_bf16_sr(v.x, rk, col) | (orx_bf16_sr(v.y, rk, col + 1) << 16),
                    orx_bf16_sr(v.z, rk, col + 2) | (orx_bf16_sr(v.w, rk, col + 3) << 16));
}
// 4 bf16 elements as one 8-byte load (p 8-byte aligned), widened exactly
__device__ __forceinline__ float4 orx_ld4(const uint16_t* p) {
  return orx_bf16x4_up(*reinterpret_cast<const uint2*>(p));
}
__device__ __forceinline__ float4 orx_ld4_stream(const uint16_t* p) {
  return orx_bf16x4_up(__ldcs(reinterpret_cast<const uint2*>(p)));
}
// Cache-global (ld.global.cg) row loads of the pointwise step: the float form is the plain __ldcg of a float4.
__device__ __forceinline__ float4 orx_ld4_cg(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 orx_ld4_cg(const uint16_t* p) {
  return orx_bf16x4_up(__ldcg(reinterpret_cast<const uint2*>(p)));
}
__device__ __forceinline__ void orx_st4_stream(float* p, float4 v, uint32_t, int) { orx_st4_stream(p, v); }
__device__ __forceinline__ void orx_st4_stream(uint16_t* p, float4 v, uint32_t rk, int col) {
  __stcs(reinterpret_cast<uint2*>(p), orx_bf16x4_sr(v, rk, col));
}
__device__ __forceinline__ void orx_st4_cg(float* p, float4 v, uint32_t, int) {
  __stcg(reinterpret_cast<float4*>(p), v);
}
__device__ __forceinline__ void orx_st4_cg(uint16_t* p, float4 v, uint32_t rk, int col) {
  __stcg(reinterpret_cast<uint2*>(p), orx_bf16x4_sr(v, rk, col));
}

// one 128-bit fire-and-forget reduction (REDG.E.ADD.F32x4 on sm_90+)
__device__ __forceinline__ void orx_red4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// log(sigmoid(y)) and sigmoid(-y), the stable forms TF uses (SURVEY 8a-G).
__device__ __forceinline__ void orx_logsig(float y, float* logsig, float* sig_neg) {
  float e = expf(-fabsf(y));
  *logsig = fminf(y, 0.f) - log1pf(e);
  *sig_neg = (y >= 0.f) ? e / (1.f + e) : 1.f / (1.f + e);
}
__device__ __forceinline__ float orx_sigmoid(float y) {
  float e = expf(-fabsf(y));
  return (y >= 0.f) ? 1.f / (1.f + e) : e / (1.f + e);
}


// MUFU approximations (max rel. error ~2^-22): the IEEE sqrtf + division of Adagrad/Adam cost ~25
// instructions per element and made the fused step issue-bound (ncu r1a: 553 warp-inst per triplet).
// The induced error on an updated parameter is < 1e-9 absolute at the reference's value ranges.
__device__ __forceinline__ float orx_sqrt_fast(float x) {
  float r;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float orx_rcp_fast(float x) {
  float r;
  asm("rcp.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// Which optimizer-slot rows an update reads and writes: S0 = Adagrad accumulator / Adam m / momentum a, S1 = Adam v,
// both one element per table element.  STAGE_ONLY: ADAM_DENSE updates no row in a step kernel; every row is staged and the sweep
// (k_adam_sweep) applies Adam to the table.  ROW: ROWWISE_ADAGRAD keeps S0 as one scalar per row (s0[id]) and no S1;
// a row's update needs the sum of its squared gradient first (orx_row_scale).  ELEM: the optimizer of the dim-1 and
// dense variables a kernel updates beside its rows (the item bias, GMF's w): element-wise ADAGRAD for ROW.
template <int OPT>
struct OrxOptSlots {
  static constexpr bool S0 = (OPT == ORX_OPT_ADAGRAD || OPT == ORX_OPT_ADAM_LAZY || OPT == ORX_OPT_MOMENTUM);
  static constexpr bool S1 = (OPT == ORX_OPT_ADAM_LAZY);
  static constexpr bool STAGE_ONLY = (OPT == ORX_OPT_ADAM_DENSE);
  static constexpr bool ROW = (OPT == ORX_OPT_ROWWISE_ADAGRAD);
  static constexpr int ELEM = ROW ? ORX_OPT_ADAGRAD : OPT;
};

// Row-wise Adagrad of one row of width D whose squared gradient sums to ss: acc += ss / D, and the row's factor
// 1 / (sqrt(acc) + eps), with the approximations of ADAGRAD.  Each element then moves by lr * g * factor
// (orx_row_apply4 / orx_row_apply1), the order in which ADAGRAD rounds lr * g * rcp(...).
__device__ __forceinline__ float orx_row_scale(float& acc, float ss, int D, const OrxOptDev& o) {
  acc = acc + ss / (float)D;
  return orx_rcp_fast(orx_sqrt_fast(acc) + o.eps);
}
__device__ __forceinline__ float orx_sq4(float4 g) { return g.x * g.x + g.y * g.y + g.z * g.z + g.w * g.w; }
__device__ __forceinline__ float4 orx_row_apply4(float4 w, float4 g, float f, const OrxOptDev& o) {
  return make_float4(w.x - o.lr * g.x * f, w.y - o.lr * g.y * f, w.z - o.lr * g.z * f, w.w - o.lr * g.w * f);
}
__device__ __forceinline__ float orx_row_apply1(float w, float g, float f, const OrxOptDev& o) {
  return w - o.lr * g * f;
}

// One optimizer update of one scalar.  OPT is an orx_opt_kind (ADAM_DENSE never reaches here:
// its rows are staged and swept).
// MOMENTUM serves NESTEROV too, told apart by o.kind (a kernel parameter: uniform over the grid).  Its products, sum
// and differences are rounded one by one, in the order of SparseApplyKerasMomentum, so that no path contracts them
// into a fused multiply-add of its own choosing: every kernel rounds a row's update alike.
template <int OPT>
__device__ __forceinline__ float orx_apply(float w, float g, float& s0, float& s1, const OrxOptDev& o) {
  static_assert(OPT != ORX_OPT_ROWWISE_ADAGRAD, "a row-wise row is updated through orx_row_scale");
  if (OPT == ORX_OPT_SGD) {
    return w - o.lr * g;
  } else if (OPT == ORX_OPT_ADAGRAD) {
    s0 = s0 + g * g;
    return w - o.lr * g * orx_rcp_fast(orx_sqrt_fast(s0) + o.eps);
  } else if (OPT == ORX_OPT_MOMENTUM) {
    const float lg = __fmul_rn(o.lr, g);
    s0 = __fsub_rn(__fmul_rn(o.beta1, s0), lg);
    return __fadd_rn(w, o.kind == ORX_OPT_NESTEROV ? __fsub_rn(__fmul_rn(o.beta1, s0), lg) : s0);
  } else {
    s0 = o.beta1 * s0 + (1.f - o.beta1) * g;
    s1 = o.beta2 * s1 + (1.f - o.beta2) * g * g;
    return w - o.lr * s0 * orx_rcp_fast(orx_sqrt_fast(s1) + o.eps);
  }
}

template <int OPT>
__device__ __forceinline__ float4 orx_apply4(float4 w, float4 g, float4& s0, float4& s1, const OrxOptDev& o) {
  float4 r;
  r.x = orx_apply<OPT>(w.x, g.x, s0.x, s1.x, o);
  r.y = orx_apply<OPT>(w.y, g.y, s0.y, s1.y, o);
  r.z = orx_apply<OPT>(w.z, g.z, s0.z, s1.z, o);
  r.w = orx_apply<OPT>(w.w, g.w, s0.w, s1.w, o);
  return r;
}

// One float4 (elements off..off+3) of a sample's gradient for table row `id`: a row that only this sample references
// (`own`) gets the optimizer in registers -- value w, the caller's slot registers s0 / s1 updated in place -- and row and
// slots are written back with a 128-bit store (STREAM: evict-first, orx_st4_stream; else __stcg); any other row's
// gradient is red.add'ed into its staging row d of G.  The addresses are formed inside each branch from the ids: taking
// precomputed row pointers changes the register allocation of the step kernels.
// T: the table's storage (float or bf16 bits); kt its rounding key (orx_sr_row), unused for float.
template <int OPT, bool STREAM, typename T>
__device__ __forceinline__ void orx_own_or_stage4(bool own, T* W, float* P0, float* P1, int id, float* G, int d,
                                                  int D, int off, float4 w, float4 g, float4& s0, float4& s1,
                                                  const OrxOptDev& o, uint32_t kt = 0) {
  typedef OrxOptSlots<OPT> SL;
  auto st = [](auto* p, float4 v, uint32_t rk, int col) {
    if (STREAM) orx_st4_stream(p, v, rk, col);
    else orx_st4_cg(p, v, rk, col);
  };
  if (!SL::STAGE_ONLY && own) {
    const int64_t i = (int64_t)id * D + off;
    st(W + i, orx_apply4<OPT>(w, g, s0, s1, o), orx_sr_row(kt, id), off);
    if (SL::S0) st(P0 + i, s0, 0u, 0);
    if (SL::S1) st(P1 + i, s1, 0u, 0);
  } else {
    orx_red4(G + (int64_t)d * D + off, g);
  }
}

// The ROWWISE_ADAGRAD form of orx_own_or_stage4: an owned row moves by its factor f (orx_row_scale, taken by the caller
// over the whole row) and has no slot row here -- the caller stores its accumulator once.
template <bool STREAM, typename T>
__device__ __forceinline__ void orx_own_or_stage4_row(bool own, T* W, int id, float* G, int d, int D, int off,
                                                      float4 w, float4 g, float f, const OrxOptDev& o,
                                                      uint32_t kt = 0) {
  if (own) {
    const float4 r = orx_row_apply4(w, g, f, o);
    if (STREAM) orx_st4_stream(W + (int64_t)id * D + off, r, orx_sr_row(kt, id), off);
    else orx_st4_cg(W + (int64_t)id * D + off, r, orx_sr_row(kt, id), off);
  } else {
    orx_red4(G + (int64_t)d * D + off, g);
  }
}

// One element of a variable (*W, current value w) and of its optimizer slots (*P0, *P1; read only when OPT has them):
// load the slots, apply the optimizer with gradient g, store value and slots.  (Sites that load with a cache operator
// or hold the slots in registers call orx_apply.)
template <int OPT>
__device__ __forceinline__ void orx_update1(float* W, float* P0, float* P1, float w, float g, const OrxOptDev& o) {
  typedef OrxOptSlots<OPT> SL;
  float s0 = SL::S0 ? *P0 : 0.f, s1 = SL::S1 ? *P1 : 0.f;
  *W = orx_apply<OPT>(w, g, s0, s1, o);
  if (SL::S0) *P0 = s0;
  if (SL::S1) *P1 = s1;
}
// The same on an element of a table of storage T, rounded with row key rk at column col (orx_st1).
template <int OPT, typename T>
__device__ __forceinline__ void orx_update1(T* W, float* P0, float* P1, float w, float g, const OrxOptDev& o,
                                            uint32_t rk, int col) {
  typedef OrxOptSlots<OPT> SL;
  float s0 = SL::S0 ? *P0 : 0.f, s1 = SL::S1 ? *P1 : 0.f;
  orx_st1(W, orx_apply<OPT>(w, g, s0, s1, o), rk, col);
  if (SL::S0) *P0 = s0;
  if (SL::S1) *P1 = s1;
}

// Keras dense Adam (ADAM_DENSE) of element i, m = M, v = V: IEEE sqrtf and division, as the reference computes it.
__device__ __forceinline__ void orx_adam_dense1(float* W, float* M, float* V, int64_t i, float g, const OrxOptDev& o) {
  const float mm = o.beta1 * M[i] + (1.f - o.beta1) * g;
  const float vv = o.beta2 * V[i] + (1.f - o.beta2) * g * g;
  M[i] = mm;
  V[i] = vv;
  W[i] = W[i] - o.lr * mm / (sqrtf(vv) + o.eps);
}
// The same on a bf16 table (element i at column col of the row with key rk).
__device__ __forceinline__ void orx_adam_dense1(uint16_t* W, float* M, float* V, int64_t i, float g, const OrxOptDev& o,
                                                uint32_t rk, int col) {
  const float mm = o.beta1 * M[i] + (1.f - o.beta1) * g;
  const float vv = o.beta2 * V[i] + (1.f - o.beta2) * g * g;
  M[i] = mm;
  V[i] = vv;
  orx_st1(W + i, orx_ld1(W + i) - o.lr * mm / (sqrtf(vv) + o.eps), rk, col);
}
__device__ __forceinline__ void orx_adam_dense1(float* W, float* M, float* V, int64_t i, float g, const OrxOptDev& o,
                                                uint32_t, int) {
  orx_adam_dense1(W, M, V, i, g, o);
}

// One (loss, l2) float partial per block of 8 warps at partials[2 * blockIdx.x], warps summed in a fixed order.
__device__ __forceinline__ void orx_block_partial(float loss, float l2, float* partials) {
  __shared__ float sred[8][2];
  loss = orx_group_sum<32>(loss);
  l2 = orx_group_sum<32>(l2);
  if ((threadIdx.x & 31) == 0) {
    sred[threadIdx.x >> 5][0] = loss;
    sred[threadIdx.x >> 5][1] = l2;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float l = 0.f, q = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      l += sred[w][0];
      q += sred[w][1];
    }
    partials[2 * blockIdx.x] = l;
    partials[2 * blockIdx.x + 1] = q;
  }
}

// One (loss, l2) float partial per warp at partials[2 * warp], warp = the global warp index.
__device__ __forceinline__ void orx_warp_partial(float loss, float l2, float* partials) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  loss = orx_group_sum<32>(loss);
  l2 = orx_group_sum<32>(l2);
  if ((threadIdx.x & 31) == 0) {
    partials[2 * warp] = loss;
    partials[2 * warp + 1] = l2;
  }
}

// Deterministic (loss, l2) totals of n float pairs (loss, l2) for one 256-thread block: each thread sums a fixed stride
// in float64, adds the squares of sq[0..nsq) to its l2 share (GMF weight), then a fixed-order tree.  Every thread of the
// block calls it and gets the totals in *l / *q.
__device__ __forceinline__ void orx_block_sum_partials(const float* partials, int n, const float* sq, int nsq,
                                                       double* l, double* q) {
  __shared__ double sh[2][256];
  double sl = 0.0, sq2 = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    sl += (double)__ldcg(partials + 2 * i);
    sq2 += (double)__ldcg(partials + 2 * i + 1);
  }
  if (sq)
    for (int e = threadIdx.x; e < nsq; e += blockDim.x) sq2 += (double)sq[e] * (double)sq[e];
  sh[0][threadIdx.x] = sl;
  sh[1][threadIdx.x] = sq2;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      sh[0][threadIdx.x] += sh[0][threadIdx.x + s];
      sh[1][threadIdx.x] += sh[1][threadIdx.x + s];
    }
    __syncthreads();
  }
  *l = sh[0][0];
  *q = sh[1][0];
}

#endif  // __CUDACC__

// What every sparse-step kernel (step and tail) reads: the user, item and item-bias tables with their optimizer slots
// (item and bias null for orx_sparse_apply), the row width, the optimizer, the batch's index sets and the handle's
// staging rows.  PairArgs, PointArgs and TailArgs derive from it.
struct SparseArgs {
  float *U, *Us0, *Us1;
  float *I, *Is0, *Is1;
  float *Bv, *Bs0, *Bs1;
  float *gu, *gi, *gb;
  OrxHash hu, hi;
  OrxOptDev opt;
  int D;
  uint32_t srk[2];   // bf16 tables: the rounding keys of the user / item table (orx_sr_table_key); unused for float
};

// Arguments of the shared tail kernel (staged rows -> optimizer, loss reduction).
struct TailArgs : SparseArgs {
  const float* partials;
  int n_partials;
  float loss_scale;  // BPR: 1/B (mean), UCML: 1 (sum)
  int32_t* counters;
  float* out4;
  // GMF dense weight (pointwise tail only)
  float *W, *Ws0, *Ws1, *gw;
  float c_l2;
};

#ifdef __CUDACC__
// The staged rows of a step: the nu staged user rows (a.hu) and ni staged item rows (a.hi, with the item bias) get the
// optimizer once each from their summed gradient, and the staging rows are zeroed (ADAM_DENSE: zeroed only, the sweep
// has applied them).  Every thread of the grid calls it.
// The tail is a chain of dependent round trips (counters -> row id -> rows) over a few thousand rows, i.e. latency,
// not bandwidth.  A warp therefore takes FOUR staged rows at once, eight lanes per row (a quarter-warp still covers
// 128 contiguous bytes per access), and issues all of a row's loads before the first use: 12 independent 128-bit
// loads per lane in flight at D = 128.  Table and slot rows evict-first, staging rows (G) at normal priority: the
// step's red.adds left them in L2.
// VEC: the table and slot rows of a are 16-byte aligned (orx_aligned16, decided by the launcher); with D % 4 == 0 the rows
// then move as float4, else lane-strided scalars.
template <int OPT, bool VEC, typename T = float>
__device__ __forceinline__ void orx_tail_rows(const TailArgs& a, int nu, int ni) {
  typedef OrxOptSlots<OPT> SL;
  constexpr bool ZERO_ONLY = SL::STAGE_ONLY;
  const int lane = threadIdx.x & 31;
  const int gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int D = a.D;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  const int sub = lane >> 3, sl = lane & 7;
  for (int r0 = gwarp * 4; r0 < nu + ni; r0 += nwarps * 4) {
    const int r = r0 + sub;
    const bool on = r < nu + ni;
    const bool is_u = on && r < nu;
    const int d = on ? (is_u ? r : r - nu) : 0;
    const int id = on ? (is_u ? a.hu.did[d] : a.hi.did[d]) : 0;
    float* G = (is_u ? a.gu : a.gi) + (int64_t)d * D;
    T* W = reinterpret_cast<T*>(is_u ? a.U : a.I) + (int64_t)id * D;
    const uint32_t rk = orx_sr_row(a.srk[is_u ? 0 : 1], id);
    float* P0 = (is_u ? a.Us0 : a.Is0) + (int64_t)id * D;
    float* P1 = (is_u ? a.Us1 : a.Is1) + (int64_t)id * D;
    if (VEC && (D & 3) == 0) {  // 128-bit path: float4 index sl + 8k
      const int nq = D >> 2;
      for (int e0 = 0; e0 < nq; e0 += 32) {
        float4 g[4], w[4], s0v[4], s1v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int e = e0 + sl + 8 * k;
          const bool ld = on && e < nq;
          g[k] = ld ? __ldcg(reinterpret_cast<const float4*>(G) + e) : z4;
          w[k] = (ld && !ZERO_ONLY) ? orx_ld4_stream(W + 4 * e) : z4;
          s0v[k] = (ld && SL::S0) ? orx_ld4_stream(P0 + 4 * e) : z4;
          s1v[k] = (ld && SL::S1) ? orx_ld4_stream(P1 + 4 * e) : z4;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int e = e0 + sl + 8 * k;
          if (!on || e >= nq) continue;
          if (!ZERO_ONLY) {
            orx_st4_stream(W + 4 * e, orx_apply4<OPT>(w[k], g[k], s0v[k], s1v[k], a.opt), rk, 4 * e);
            if (SL::S0) orx_st4_stream(P0 + 4 * e, s0v[k]);
            if (SL::S1) orx_st4_stream(P1 + 4 * e, s1v[k]);
          }
          __stcg(reinterpret_cast<float4*>(G) + e, z4);
        }
      }
    } else if (on) {
      for (int e = sl; e < D; e += 8) {
        if (!ZERO_ONLY) orx_update1<OPT>(W + e, P0 + e, P1 + e, orx_ld1(W + e), G[e], a.opt, rk, e);
        G[e] = 0.f;
      }
    }
    if (on && !is_u && sl == 0) {     // the item bias of the staged row
      if (!ZERO_ONLY) orx_update1<OPT>(a.Bv + id, a.Bs0 + id, a.Bs1 + id, a.Bv[id], a.gb[d], a.opt);
      a.gb[d] = 0.f;
    }
  }
  // (the hash tables are not cleared: the next step uses a new epoch)
}

// orx_tail_rows under ROWWISE_ADAGRAD: the same eight lanes per staged row take the sum of the row's squared gradient
// first -- lane sl over float4 (scalar) indices sl, sl + 8, ... in order, then the fixed 8-lane tree -- and only then
// apply: a second pass over G, which the step's red.adds left in L2.  The row's accumulator s0[id] is one scalar; the
// item bias gets element-wise ADAGRAD.
template <bool VEC, typename T = float>
__device__ __forceinline__ void orx_tail_rows_rowwise(const TailArgs& a, int nu, int ni) {
  const int lane = threadIdx.x & 31;
  const int gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int D = a.D;
  const bool vec = VEC && (D & 3) == 0;
  const int nq = D >> 2;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  const int sub = lane >> 3, sl = lane & 7;
  for (int r0 = gwarp * 4; r0 < nu + ni; r0 += nwarps * 4) {   // warp-uniform: the 8-lane sums below see every lane
    const int r = r0 + sub;
    const bool on = r < nu + ni;
    const bool is_u = on && r < nu;
    const int d = on ? (is_u ? r : r - nu) : 0;
    const int id = on ? (is_u ? a.hu.did[d] : a.hi.did[d]) : 0;
    float* G = (is_u ? a.gu : a.gi) + (int64_t)d * D;
    T* W = reinterpret_cast<T*>(is_u ? a.U : a.I) + (int64_t)id * D;
    const uint32_t rk = orx_sr_row(a.srk[is_u ? 0 : 1], id);
    float* P0 = (is_u ? a.Us0 : a.Is0) + id;
    float ss = 0.f, acc = 0.f;
    if (on) {
      acc = __ldcg(P0);
      if (vec) {
        for (int e = sl; e < nq; e += 8) ss += orx_sq4(__ldcg(reinterpret_cast<const float4*>(G) + e));
      } else {
        for (int e = sl; e < D; e += 8) ss += G[e] * G[e];
      }
    }
    ss = orx_group_sum<8>(ss);
    const float f = orx_row_scale(acc, ss, D, a.opt);
    if (on) {
      if (sl == 0) __stcg(P0, acc);
      if (vec) {
        for (int e0 = 0; e0 < nq; e0 += 32) {   // as orx_tail_rows: a chunk's loads before its first use
          float4 g[4], w[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int e = e0 + sl + 8 * k;
            g[k] = e < nq ? __ldcg(reinterpret_cast<const float4*>(G) + e) : z4;
            w[k] = e < nq ? orx_ld4_stream(W + 4 * e) : z4;
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int e = e0 + sl + 8 * k;
            if (e >= nq) continue;
            orx_st4_stream(W + 4 * e, orx_row_apply4(w[k], g[k], f, a.opt), rk, 4 * e);
            __stcg(reinterpret_cast<float4*>(G) + e, z4);
          }
        }
      } else {
        for (int e = sl; e < D; e += 8) {
          orx_st1(W + e, orx_row_apply1(orx_ld1(W + e), G[e], f, a.opt), rk, e);
          G[e] = 0.f;
        }
      }
      if (!is_u && sl == 0) {   // the item bias of the staged row
        orx_update1<ORX_OPT_ADAGRAD>(a.Bv + id, a.Bs0 + id, nullptr, a.Bv[id], a.gb[d], a.opt);
        a.gb[d] = 0.f;
      }
    }
  }
}
#endif  // __CUDACC__

OrxOptDev orx_opt_to_dev(const orx_opt_t* o);
int orx_launch_index_build_strided(orx_ctx* c, const int32_t* a, int64_t stride, int64_t rows, int32_t n,
                                   bool stage_all, cudaStream_t st);
// The shared arguments of a step over user / item / bias (item and bias may be null) with index set ix, the handle's
// staging rows and optimizer o.  A derived block takes them as its first initializer: TailArgs ta = {s}; zeroes every
// other field.
SparseArgs orx_sparse_args(const orx_ctx* c, const orx_table_t* user, const orx_table_t* item, const orx_table_t* bias,
                           const OrxIndexSet& ix, const OrxOptDev& o);
// The tables of a pairwise or pointwise step, fused or not: user, item and item bias present, user / item dims that
// agree, int32 row ids, and the slot rows optimizer opt_kind keeps -- also on w, GMF's dense weight, when it is given.
int orx_check_step_tables(const orx_table_t* user, const orx_table_t* item, const orx_table_t* bias,
                          const orx_table_t* w, int opt_kind);
// Grid of every sparse-step kernel over B samples: 256 threads, 8 samples per warp.  A kernel writes at most one
// (loss, l2) partial per warp, so 8 * orx_step_blocks(B) partials hold any step's.
static inline int orx_step_blocks(int B) { return ((B + 7) / 8 + 7) / 8; }
// What a family's step kernel launch reports back: the (loss, l2) partials it writes and, for the dispatch record, the
// orx_dispatch_variant launched and its CTAs/SM bound (0 if none).
struct OrxStepLaunch {
  int n_partials, variant, minb;
};
// A family's step kernel, launched on the driver's stream with the shared arguments (index sets chosen) and the
// handle's partials; res = the per-triplet records of a consumed prefetch (k_index_resolve), else null.
typedef std::function<int(const SparseArgs& s, const int4* res, float* partials, OrxStepLaunch* out)> OrxStepKernel;
// One fused pairwise or pointwise step on st: validate, workspace, partials, batch index (a pairwise batch, nid != null,
// takes its prefetched index when one matches), profile marks 0..3, kernel(...), dispatch record {op, variant, kind,
// opt, B, D, minb, index set}, ADAM_DENSE sweeps, tail (loss scaled by loss_scale into out4; w: GMF's dense weight,
// updated with c_l2, or null), and the prefetched set handed back.
int orx_sparse_step(orx_ctx* c, int op, int kind, const orx_table_t* user, const orx_table_t* item,
                    const orx_table_t* bias, const orx_table_t* w, const int32_t* uid, const int32_t* iid,
                    const int32_t* nid, int B, const orx_opt_t* opt, float loss_scale, float c_l2, float* out4,
                    const OrxStepKernel& kernel, cudaStream_t st, const uint32_t* srk = nullptr);
// srk (orx_sparse_step, orx_launch_adam_sweeps): the user / item tables are bf16 (orx_table_bf16_t, var passed as the
// float* of the orx_table_t) with these rounding keys (orx_sr_table_key); null = float tables.
// A bf16 table as the orx_table_t the shared host code takes: var carries the bf16 rows' address, and every kernel that
// reads it is instantiated for uint16_t storage.  A null table stays null (the shared checks refuse it).
static inline const orx_table_t* orx_bf16_table(const orx_table_bf16_t* b, orx_table_t* t) {
  if (!b) return nullptr;
  *t = {reinterpret_cast<float*>(b->var), b->s0, b->s1, b->rows, b->dim};
  return t;
}
// The un-fused forward / gradient kernel of a family over B samples: launch(partials, blocks) on st with the handle's
// partials, then, when out4 is given, the (loss, l2) partials reduced into it, the loss scaled by loss_scale.
int orx_sparse_unfused(orx_ctx* c, int B, float loss_scale, float* out4,
                       const std::function<void(float* partials, int blocks)>& launch, cudaStream_t st);
// ADAM_DENSE: Keras dense Adam over every row of user / item / bias (item and bias may be null), a row's summed gradient
// taken from its side's table of index set ix and staging rows.  Runs before the tail, which zeroes the staging rows.
int orx_launch_adam_sweeps(orx_ctx* c, const orx_table_t* user, const orx_table_t* item, const orx_table_t* bias,
                           const OrxIndexSet& ix, const OrxOptDev& o, cudaStream_t st, const uint32_t* srk = nullptr);
// k_sparse_tail over ta, its 128-bit row path chosen by the alignment of ta's table and slot rows (orx_aligned16).
// bf16: the user / item tables of ta are bf16 (ta.srk), whose 8-byte row path needs 8-byte aligned rows.
int orx_launch_tail(orx_ctx* c, const TailArgs& ta, int opt_kind, cudaStream_t st, bool bf16 = false);
int orx_launch_reduce_partials(const float* partials, int n, float loss_scale, float* out4, cudaStream_t st);
// index of n samples (a[t], b0[t]) or (a[t], b0[t], b1[t]); only samples whose ids are all in range are inserted
int orx_launch_index_build(orx_ctx* c, const int32_t* a, int64_t rows_a, const int32_t* b0, const int32_t* b1,
                           int64_t rows_b, int32_t n, int mode /* orx_hash_insert mode: 0 | 1 */, cudaStream_t st);
