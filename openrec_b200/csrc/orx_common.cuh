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

struct orx_ctx {
  int device;
  int num_sms;
  // index workspace (sized for cap_B lookups per table side)
  int64_t cap_B;  // largest batch the workspace is sized for
  OrxHash hu, hi;      // index set 0: everything that builds its index on the caller's stream
  OrxHash pf_u[2], pf_i[2];  // index sets 1, 2: pairwise batches indexed ahead on the side stream (orx_pairwise.cu)
  int32_t* counters;  // [16]: per index set k at 4k: staged_u, staged_i, ticket, bad ids; 12.. spare
  // staged-row gradient buffers
  float *gu, *gi, *gb, *gw;
  int64_t g_rows_u, g_rows_i;
  int32_t g_dim;
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
  cudaEvent_t pf_done[2], pf_free[2], stage_free[2];   // prefetched index k built / handed back; id staging f free
  int pf_free_valid[2], stage_free_valid[2];
  int pf_valid, pf_set, pf_next, pf_B, pf_mode;        // the one outstanding prefetched index and what it was built for
  const int32_t *pf_uid, *pf_pid, *pf_nid;
  int64_t pf_rows_u, pf_rows_i;
  uint32_t epoch;          // hash epoch of the last step, in [1, 2^31)
  void* shard_ws;          // orx_shard.cu: host bookkeeping of the row-sharded step (orx_shard_ws*)
  void* shard_scratch;     // orx_shard.cu: its local device scratch, carved by sh_layout
  size_t shard_cap;
  int32_t dispatch[ORX_DISPATCH_LOG_CAP][8];   // orx_debug_dispatch_log: ring of the last DLRM / sparse-step launches
  int64_t dispatch_n;      // records written since the last read
  void* eval_ws;           // orx_eval.cu: scratch of orx_score_rank / orx_score_topk, its own allocation
  size_t eval_cap;
  float* splitk;           // split-K partials of the Dense-layer GEMMs and of the split column sum
  size_t splitk_cap;
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

// Start a new hash epoch (once per step, before the index build; `st` = the stream the step runs on).
// A slot word holds 31 epoch bits: epochs live in [1, 2^31) and on wrap every table is zeroed on `st`, so a stale
// slot can never alias the current epoch (about 65 h of back-to-back steps between wraps).
int orx_next_epoch(orx_ctx* c, cudaStream_t st);
void orx_shard_ws_release(orx_ctx* c);
// true while a row-sharded step on this handle has an index that must survive until its next orx_shard_step call (an
// announced batch's user index, built inside the previous step's apply launch; or a step issued phase by phase).
// Workspace growth, a prefetch and an epoch wrap are refused meanwhile: each would empty or overwrite that index.
bool orx_shard_holds_index(const orx_ctx* c);

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
template <typename F>
static inline auto orx_dispatch_opt(int opt_kind, F&& f) {
  return orx_dispatch<ORX_OPT_SGD, ORX_OPT_ADAGRAD, ORX_OPT_ADAM_LAZY, ORX_OPT_ADAM_DENSE>(opt_kind, f);
}

// an orx_opt_kind
static inline bool orx_opt_kind_ok(int kind) { return kind >= ORX_OPT_SGD && kind <= ORX_OPT_ADAM_DENSE; }
// The host side of OrxOptSlots: every table carries the slot rows optimizer `kind` keeps -- s0 for every kind but SGD,
// s1 for both Adams (ADAM_DENSE's sweep keeps m and v there).  Null tables are skipped.
bool orx_opt_slots_ok(int kind, std::initializer_list<const orx_table_t*> tabs);

// ---------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------
struct OrxOptDev {
  int32_t kind;
  float lr;    // SGD/Adagrad: lr ; Adam: bias-corrected lr_t
  float eps, beta1, beta2;
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

// Which optimizer-slot rows an update reads and writes: S0 = Adagrad accumulator / Adam m, S1 = Adam v.  STAGE_ONLY:
// ADAM_DENSE updates no row in a step kernel; every row is staged and the sweep (k_adam_sweep) applies Adam to the table.
template <int OPT>
struct OrxOptSlots {
  static constexpr bool S0 = (OPT == ORX_OPT_ADAGRAD || OPT == ORX_OPT_ADAM_LAZY);
  static constexpr bool S1 = (OPT == ORX_OPT_ADAM_LAZY);
  static constexpr bool STAGE_ONLY = (OPT == ORX_OPT_ADAM_DENSE);
};

// One optimizer update of one scalar.  OPT is an orx_opt_kind (ADAM_DENSE never reaches here:
// its rows are staged and swept).
template <int OPT>
__device__ __forceinline__ float orx_apply(float w, float g, float& s0, float& s1, const OrxOptDev& o) {
  if (OPT == ORX_OPT_SGD) {
    return w - o.lr * g;
  } else if (OPT == ORX_OPT_ADAGRAD) {
    s0 = s0 + g * g;
    return w - o.lr * g * orx_rcp_fast(orx_sqrt_fast(s0) + o.eps);
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
template <int OPT, bool STREAM>
__device__ __forceinline__ void orx_own_or_stage4(bool own, float* W, float* P0, float* P1, int id, float* G, int d,
                                                  int D, int off, float4 w, float4 g, float4& s0, float4& s1,
                                                  const OrxOptDev& o) {
  typedef OrxOptSlots<OPT> SL;
  auto st = [](float* p, float4 v) {
    if (STREAM) orx_st4_stream(p, v);
    else __stcg(reinterpret_cast<float4*>(p), v);
  };
  if (!SL::STAGE_ONLY && own) {
    const int64_t i = (int64_t)id * D + off;
    st(W + i, orx_apply4<OPT>(w, g, s0, s1, o));
    if (SL::S0) st(P0 + i, s0);
    if (SL::S1) st(P1 + i, s1);
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

// Keras dense Adam (ADAM_DENSE) of element i, m = M, v = V: IEEE sqrtf and division, as the reference computes it.
__device__ __forceinline__ void orx_adam_dense1(float* W, float* M, float* V, int64_t i, float g, const OrxOptDev& o) {
  const float mm = o.beta1 * M[i] + (1.f - o.beta1) * g;
  const float vv = o.beta2 * V[i] + (1.f - o.beta2) * g * g;
  M[i] = mm;
  V[i] = vv;
  W[i] = W[i] - o.lr * mm / (sqrtf(vv) + o.eps);
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
template <int OPT>
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
    float* W = (is_u ? a.U : a.I) + (int64_t)id * D;
    float* P0 = (is_u ? a.Us0 : a.Is0) + (int64_t)id * D;
    float* P1 = (is_u ? a.Us1 : a.Is1) + (int64_t)id * D;
    if ((D & 3) == 0) {  // 128-bit path: float4 index sl + 8k
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
            orx_st4_stream(W + 4 * e, orx_apply4<OPT>(w[k], g[k], s0v[k], s1v[k], a.opt));
            if (SL::S0) orx_st4_stream(P0 + 4 * e, s0v[k]);
            if (SL::S1) orx_st4_stream(P1 + 4 * e, s1v[k]);
          }
          __stcg(reinterpret_cast<float4*>(G) + e, z4);
        }
      }
    } else if (on) {
      for (int e = sl; e < D; e += 8) {
        if (!ZERO_ONLY) orx_update1<OPT>(W + e, P0 + e, P1 + e, W[e], G[e], a.opt);
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
#endif  // __CUDACC__

OrxOptDev orx_opt_to_dev(const orx_opt_t* o);
int orx_launch_index_build_strided(orx_ctx* c, const int32_t* a, int64_t stride, int64_t rows, int32_t n,
                                   bool stage_all, cudaStream_t st);
// The shared arguments of a step over user / item / bias (item and bias may be null) with index sets hu / hi, the
// handle's staging rows and optimizer o.  A derived block takes them as its first initializer: TailArgs ta = {s};
// zeroes every other field.
SparseArgs orx_sparse_args(const orx_ctx* c, const orx_table_t* user, const orx_table_t* item, const orx_table_t* bias,
                           const OrxHash& hu, const OrxHash& hi, const OrxOptDev& o);
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
// handle's partials.
typedef std::function<int(const SparseArgs& s, float* partials, OrxStepLaunch* out)> OrxStepKernel;
// One fused pairwise or pointwise step on st: validate, workspace, partials, batch index (a pairwise batch, nid != null,
// takes its prefetched index when one matches), profile marks 0..3, kernel(...), dispatch record {op, variant, kind,
// opt, B, D, minb, index set}, ADAM_DENSE sweeps, tail (loss scaled by loss_scale into out4; w: GMF's dense weight,
// updated with c_l2, or null), and the prefetched set handed back.
int orx_sparse_step(orx_ctx* c, int op, int kind, const orx_table_t* user, const orx_table_t* item,
                    const orx_table_t* bias, const orx_table_t* w, const int32_t* uid, const int32_t* iid,
                    const int32_t* nid, int B, const orx_opt_t* opt, float loss_scale, float c_l2, float* out4,
                    const OrxStepKernel& kernel, cudaStream_t st);
// The un-fused forward / gradient kernel of a family over B samples: launch(partials, blocks) on st with the handle's
// partials, then, when out4 is given, the (loss, l2) partials reduced into it, the loss scaled by loss_scale.
int orx_sparse_unfused(orx_ctx* c, int B, float loss_scale, float* out4,
                       const std::function<void(float* partials, int blocks)>& launch, cudaStream_t st);
// ADAM_DENSE: Keras dense Adam over every row of user / item / bias (item and bias may be null), a row's summed gradient
// taken from its side's index set (hu / hi) and staging rows.  Runs before the tail, which zeroes the staging rows.
int orx_launch_adam_sweeps(orx_ctx* c, const orx_table_t* user, const orx_table_t* item, const orx_table_t* bias,
                           const OrxHash& hu, const OrxHash& hi, const OrxOptDev& o, cudaStream_t st);
int orx_launch_tail(orx_ctx* c, const TailArgs& ta, int opt_kind, cudaStream_t st);
int orx_launch_reduce_partials(const float* partials, int n, float loss_scale, float* out4, cudaStream_t st);
// index of n samples (a[t], b0[t]) or (a[t], b0[t], b1[t]); only samples whose ids are all in range are inserted
int orx_launch_index_build(orx_ctx* c, const int32_t* a, int64_t rows_a, const int32_t* b0, const int32_t* b1,
                           int64_t rows_b, int32_t n, int mode /* orx_hash_insert mode: 0 | 1 */, cudaStream_t st);
