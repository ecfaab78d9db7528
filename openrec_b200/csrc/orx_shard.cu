// orx_shard.cu -- the row-sharded BPR / UCML training step over the GPUs of one NVSwitch box, "home-routed" form
// (SURVEY 8e, BASELINE configs[4]; the reference is single-device: tf2_examples/bpr_citeulike.py:33-39 is the step).
//
// Partitioning: row r of the user table and of the item table (+ item bias, + optimizer slots) lives on rank r % R at
// local row r / R.  A triplet (u, p, n) is COMPUTED on the rank that owns its user row (its "home"), so the user row
// never crosses NVLink: per triplet two item rows travel in and two gradient rows travel out (the first version moved
// three each way).  Every table access is local; everything that crosses NVLink is a peer STORE of a contiguous,
// 16-byte-aligned D-float row (512 B at D = 128) or of a coalesced run of 4-byte words into a small mailbox mapped
// through CUDA IPC.  No collective, no host sync, no count ever visits the host.
//
// One step on rank `me` = six launches on one stream; cross-rank ordering is by flag words in peer memory, written by
// the LAST block of the producing kernel (release, system scope) and polled by EVERY block of the consuming kernel
// (acquire) -- there are no barrier launches:
//
//   k_sh_route    source : bucket my B triplets by home = u % R, store (u / R, p, n) into the homes' tripbox      -> flag 0
//   k_sh_request  home   : [wait 0] my T triplets: index the user ids (dedup hash), bucket the 2T item lookups by
//                          owner = id % R, store id / R into the owners' idbox, publish counts + where the rows go  -> flag 1
//   k_sh_serve    owner  : [wait 1] for every requested id: index it (dedup hash of ALL ranks' lookups), read the LOCAL
//                          row and bias, store them into the home's `got` / `gotb` (owner-sorted, so a source's rows
//                          land contiguously: 8 rows = 4 KB + one 32 B run of biases), publish the gradient-inbox bases -> flag 2
//   k_sh_compute  home   : [wait 2] score + loss + gradients per triplet; the USER row is updated right here (owned rows
//                          in registers, duplicated rows through the staging buffer -- the single-GPU scheme); the two
//                          item gradient rows (+ one 4-byte bias gradient each) are stored into their owners' `gin` /
//                          `ginb`; the last block sends this rank's (loss, l2) partial to every rank                   -> flag 3
//   k_sh_apply    owner  : [wait 3] rows requested once: optimizer straight from the gradient row; duplicated rows are
//                          summed in the staging buffer
//   k_sh_tail     both   : staged user and item rows -> optimizer; out4 = GLOBAL (loss, l2_loss), identical on every rank
//
// All gathers of a step read pre-step values: item rows are only written by k_sh_apply / k_sh_tail, which follow
// the rank's own k_sh_serve on the stream; user rows are read and written by the one triplet that owns them, shared ones
// only in k_sh_tail.  Mailbox reuse across steps needs no extra synchronisation (proof per buffer in DESIGN.md 7).
//
// Prologue: a caller that announces the NEXT batch (next_uid / next_pid / next_nid of orx_shard_step) gets that step's
// route and request as two extra block roles inside THIS step's k_sh_apply launch: two of the four cross-rank handoffs of
// a step -- ~20-35 us each of launch, fence and flag latency with no bandwidth behind them -- run under the HBM-bound
// apply, and the announced step is four launches (serve, compute, apply, tail).  Safety per buffer at ShProArgs.
//
// phase_lo / phase_hi of orx_shard_step select a sub-range of the six launches, so that R "virtual ranks" can share ONE
// device and ONE stream (tests/test_gpu_shard_loopback.py): phase k is issued for every rank before phase k + 1, every
// flag is already set when its consumer runs, and the exact kernels of the multi-GPU step are exercised on a 1-GPU box.
#include <stdlib.h>
#include <string.h>

#include "orx_common.cuh"
#include "orx_pair.cuh"

#define SH_MAX_R 64
#define SH_META 16     // int32 words per peer in a meta mailbox
#define SH_NPH 4       // flag words per peer
#define SH_ERR_WORD (SH_NPH * SH_MAX_R)
#define SH_IDX_BITS 24

// meta[X][r * SH_META + k], written by rank r into rank X's mailbox:
enum { SH_M_TRIPS = 0,    // triplets r routed to X                                  (k_sh_route)
       SH_M_REQS = 1,     // item rows home r requests from owner X                  (k_sh_request)
       SH_M_GOTOFF = 2,   // first row of r's `got` that owner X fills               (k_sh_request)
       SH_M_GINBASE = 3,  // first row of owner r's `gin` that home X fills, -1 = overflow (k_sh_serve)
       SH_M_LOSS = 4, SH_M_L2 = 5 };   // r's partial sums, float bits                (k_sh_compute)

// local control words (ShardWs::ctl)
enum { SH_C_CURH = 0, SH_C_CURO = SH_MAX_R, SH_C_GOFF = 2 * SH_MAX_R, SH_C_RCO = 3 * SH_MAX_R + 1,
       SH_C_DONE = 4 * SH_MAX_R + 1, SH_C_T = SH_C_DONE + 8, SH_C_NREQ = SH_C_T + 1, SH_C_ACUR = SH_C_T + 2,
       SH_C_BAD = SH_C_T + 4 /* + step parity */, SH_C_WORDS = SH_C_T + 8 };

struct ShardHost {   // mirrors orx_shard_t (include/orx.h)
  int32_t world, rank, dim, batch_cap, home_cap, req_cap, gin_cap, timeout_ms;
  void *tripbox, *idbox, *got, *gotb, *gin, *ginb, *meta, *flags;
};

struct ShardDev {
  int world, rank, D, batch_cap, home_cap, req_cap, gin_cap, got_rows;
  unsigned long long timeout_ns;
  int32_t* const* tripbox;   // [world] int32 [world][3][batch_cap]
  int32_t* const* idbox;     // [world] int32 [world][req_cap]
  float* const* got;         // [world] float [got_rows][D]
  float* const* gotb;        // [world] float [got_rows]
  float* const* gin;         // [world] float [gin_cap][D]
  float* const* ginb;        // [world] float [gin_cap]
  int32_t* const* meta;      // [world] int32 [world][SH_META]
  int32_t* const* flags;     // [world] int32 [SH_NPH][SH_MAX_R] + error word
};

struct ShardWs {       // per-handle local scratch
  int32_t* trip_u;     // [home_cap]      local user row of home triplet t
  int32_t* slot;       // [2 * home_cap]  (owner << 24 | index in my bucket for that owner) of lookup 2t + q, -1 = dropped
  int32_t* req;        // [gin_cap]       local item row requested as gradient-inbox row j (-1 = padding / invalid)
  int32_t* ctl;        // [SH_C_WORDS]
};

static inline int sh_got_rows(int home_cap, int world) { return 2 * home_cap + 32 * world; }

__device__ __forceinline__ int sh_bucket_of(const int32_t* off, int R, int p) {   // first r with off[r + 1] > p
  int lo = 0, hi = R - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (off[mid + 1] > p) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// rank of this lane's key inside a shared-memory counter array, warp-aggregated: one atomicAdd per distinct key and warp
// instruction instead of one per lane (with R = 2..8 owners every lane of a block hits the same few words, and
// same-address shared atomics serialise: 20 us of a 64-block kernel in the first version, profiles/r2f).
__device__ __forceinline__ int sh_rank_add(int32_t* cnt, int key, bool active) {
  const unsigned act = __ballot_sync(ORX_FULL, active);
  int rk = 0;
  if (active) {
    const unsigned peers = __match_any_sync(act, key);
    const int leader = __ffs(peers) - 1;
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == leader) base = atomicAdd(&cnt[key], __popc(peers));
    base = __shfl_sync(peers, base, leader);
    rk = base + __popc(peers & ((1u << lane) - 1u));
  }
  return rk;
}

__device__ __forceinline__ unsigned long long sh_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// every block of a consumer: wait until all ranks have published `epoch` for `phase` in MY flag words
__device__ __forceinline__ void sh_wait(const ShardDev& x, int phase, int epoch) {
  if ((int)threadIdx.x < x.world) {
    int32_t* mine = x.flags[x.rank];
    const int32_t* f = mine + phase * SH_MAX_R + threadIdx.x;
    const unsigned long long t0 = sh_now();
    unsigned spins = 0;
    while (true) {
      int32_t v;
      asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
      if (v >= epoch) break;
      if ((++spins & 63u) == 0u) {
        if (*(volatile int32_t*)(mine + SH_ERR_WORD) != 0) break;       // somebody already gave up: do not stack timeouts
        if (sh_now() - t0 > x.timeout_ns) {                             // a peer never arrived: sticky error, no hang
          atomicCAS(mine + SH_ERR_WORD, 0, 1);
          break;
        }
        __nanosleep(64);
      }
    }
  }
  __syncthreads();
}

// every block of a producer, at its very end: the last block publishes `epoch` for `phase` to every rank.
// `publish()` (all threads of the last block) stores the producer's per-peer meta words first.
// Ordering: each block orders its (peer) stores before its ticket with a GPU-scope fence; the last block, having observed
// every ticket, issues the one SYSTEM-scope fence in front of the flag stores.  Fences are cumulative (PTX memory model:
// causality order is transitive over morally-strong edges of different scopes), so a peer that acquires the flag sees
// every block's stores.  A system fence per block cost ~5 us at the end of every launch (profiles/r2g).
template <typename F>
__device__ __forceinline__ void sh_arrive(const ShardDev& x, int32_t* done, int nblk, int phase, int epoch, F publish) {
  __shared__ bool sh_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();                            // this block's stores are ordered before its ticket (GPU scope)
    sh_last = (atomicAdd(done, 1) == nblk - 1);
    __threadfence();
  }
  __syncthreads();
  if (!sh_last) return;
  publish();
  __syncthreads();
  if (threadIdx.x == 0) *done = 0;
  if ((int)threadIdx.x < x.world) {
    __threadfence_system();
    int32_t* remote = x.flags[threadIdx.x] + phase * SH_MAX_R + x.rank;
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(remote), "r"(epoch) : "memory");
  }
}

// ---------------------------------------------------------------------------------------
// phase 0: triplets -> homes.  A "role": the body of k_sh_route, and of the first blocks of the PREVIOUS step's k_sh_apply
// when the caller announced this batch there (see "prologue" in the file header).  bid / nblk = this block among the
// role's blocks; par = step parity (epoch & 1) of the skipped-triplet counter.
// ---------------------------------------------------------------------------------------
struct ShRouteArgs {
  const int32_t *uid, *pid, *nid;
  int B;
  int64_t U, I;
};

__device__ __forceinline__ void sh_route_role(const ShardDev& x, const ShardWs& w, const ShRouteArgs& r, int epoch, int bid, int nblk) {
  __shared__ int32_t cnt[SH_MAX_R], base[SH_MAX_R];
  const int R = x.world;
  if ((int)threadIdx.x < R) cnt[threadIdx.x] = 0;
  __syncthreads();
  int h[4], rk[4];
  int32_t uu[4], pp[4], nn[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = bid * 1024 + k * 256 + threadIdx.x;
    h[k] = -1;
    bool ok = false;
    if (i < r.B) {
      const int32_t u = r.uid[i], p = r.pid[i], n = r.nid[i];
      // a triplet with ANY id out of range is skipped as a whole, like the single-GPU step (orx_pairwise.cu)
      ok = u >= 0 && (int64_t)u < r.U && p >= 0 && (int64_t)p < r.I && n >= 0 && (int64_t)n < r.I;
      if (ok) {
        h[k] = u % R;
        uu[k] = u / R; pp[k] = p; nn[k] = n;
      } else {
        atomicAdd(w.ctl + SH_C_BAD + (epoch & 1), 1);
      }
    }
    rk[k] = sh_rank_add(cnt, ok ? h[k] : 0, ok);
  }
  __syncthreads();
  if ((int)threadIdx.x < R) base[threadIdx.x] = cnt[threadIdx.x] ? atomicAdd(w.ctl + SH_C_CURH + threadIdx.x, cnt[threadIdx.x]) : 0;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (h[k] < 0) continue;
    const int idx = base[h[k]] + rk[k];                      // < B <= batch_cap
    int32_t* box = x.tripbox[h[k]] + (int64_t)x.rank * 3 * x.batch_cap;
    box[idx] = uu[k];
    box[x.batch_cap + idx] = pp[k];
    box[2 * x.batch_cap + idx] = nn[k];
  }
  sh_arrive(x, w.ctl + SH_C_DONE + 0, nblk, 0, epoch, [&]() {
    if ((int)threadIdx.x < R) {
      const int q = threadIdx.x;
      x.meta[q][SH_META * x.rank + SH_M_TRIPS] = __ldcg(w.ctl + SH_C_CURH + q);
      w.ctl[SH_C_CURH + q] = 0;
    }
  });
}

__global__ void __launch_bounds__(256) k_sh_route(ShardDev x, ShardWs w, ShRouteArgs r, int epoch) {
  orx_pdl_wait();
  sh_route_role(x, w, r, epoch, blockIdx.x, gridDim.x);
  orx_pdl_trigger();
}

// ---------------------------------------------------------------------------------------
// phase 1: home: index my user rows, item lookups -> owners (a role, like phase 0)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void sh_request_role(const ShardDev& x, const ShardWs& w, const OrxHash& hu, int epoch, int bid, int nblk) {
  __shared__ int32_t toff[SH_MAX_R + 1], cnt[SH_MAX_R], base[SH_MAX_R], goff[SH_MAX_R + 1];
  __shared__ int T_sh;
  const int R = x.world, me = x.rank;
  sh_wait(x, 0, epoch);
  if (threadIdx.x == 0) {
    const int32_t* m = x.meta[me];
    int acc = 0;
    for (int s = 0; s < R; ++s) {
      int c = __ldcg(m + SH_META * s + SH_M_TRIPS);
      c = c < 0 ? 0 : (c > x.batch_cap ? x.batch_cap : c);
      toff[s] = acc;
      acc += c;
    }
    toff[R] = acc;
    if (acc > x.home_cap) { atomicCAS(x.flags[me] + SH_ERR_WORD, 0, 2); acc = x.home_cap; }   // more triplets than this home was built for
    T_sh = acc;
  }
  __syncthreads();
  const int T = T_sh;
  const int32_t* box = x.tripbox[me];
  for (int c0 = bid * 512; c0 < T; c0 += nblk * 512) {
    if ((int)threadIdx.x < R) cnt[threadIdx.x] = 0;
    __syncthreads();
    int o[4], rk[4];
    int32_t lid[4];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int t = c0 + k * 256 + threadIdx.x;
      o[2 * k] = o[2 * k + 1] = 0;
      int32_t u = -1;
      if (t < T) {
        const int s = sh_bucket_of(toff, R, t);
        const int32_t* b = box + (int64_t)s * 3 * x.batch_cap + (t - toff[s]);
        u = __ldcg(b);
        const int32_t p = __ldcg(b + x.batch_cap), n = __ldcg(b + 2 * x.batch_cap);
        w.trip_u[t] = u;
        o[2 * k] = p % R; lid[2 * k] = p / R;
        o[2 * k + 1] = n % R; lid[2 * k + 1] = n / R;
      }
      rk[2 * k] = sh_rank_add(cnt, o[2 * k], t < T);
      rk[2 * k + 1] = sh_rank_add(cnt, o[2 * k + 1], t < T);
      if (t < T) orx_hash_insert(hu, u, 0);
    }
    __syncthreads();
    if ((int)threadIdx.x < R) base[threadIdx.x] = cnt[threadIdx.x] ? atomicAdd(w.ctl + SH_C_CURO + threadIdx.x, cnt[threadIdx.x]) : 0;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int t = c0 + k * 256 + threadIdx.x;
      if (t >= T) continue;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int e = 2 * k + q;
        const int idx = base[o[e]] + rk[e];
        if (idx < x.req_cap) {
          x.idbox[o[e]][(int64_t)me * x.req_cap + idx] = lid[e];
          w.slot[2 * t + q] = (o[e] << SH_IDX_BITS) | idx;
        } else {
          w.slot[2 * t + q] = -1;
          atomicCAS(x.flags[me] + SH_ERR_WORD, 0, 3);     // one owner got more requests than its idbox holds
        }
      }
    }
    __syncthreads();
  }
  sh_arrive(x, w.ctl + SH_C_DONE + 1, nblk, 1, epoch, [&]() {
    if (threadIdx.x == 0) {
      int acc = 0;
      for (int r = 0; r < R; ++r) {
        int c = __ldcg(w.ctl + SH_C_CURO + r);
        c = c > x.req_cap ? x.req_cap : c;
        w.ctl[SH_C_RCO + r] = c;
        w.ctl[SH_C_GOFF + r] = goff[r] = acc;
        acc += (c + 31) & ~31;                 // a source's rows start on a 32-row boundary: bias runs stay 128 B aligned
        w.ctl[SH_C_CURO + r] = 0;
      }
      w.ctl[SH_C_GOFF + R] = goff[R] = acc;
      w.ctl[SH_C_T] = T;
    }
    __syncthreads();
    if ((int)threadIdx.x < R) {
      const int r = threadIdx.x;
      int32_t* m = x.meta[r] + SH_META * me;
      m[SH_M_REQS] = w.ctl[SH_C_RCO + r];
      m[SH_M_GOTOFF] = goff[r];
    }
  });
}

__global__ void __launch_bounds__(256) k_sh_request(ShardDev x, ShardWs w, OrxHash hu, int epoch) {
  orx_pdl_wait();
  sh_request_role(x, w, hu, epoch, blockIdx.x, gridDim.x);
  orx_pdl_trigger();
}

// ---------------------------------------------------------------------------------------
// phase 2: owner: requested rows -> homes
// ---------------------------------------------------------------------------------------
template <int NQ>
__global__ void __launch_bounds__(256) k_sh_serve(ShardDev x, ShardWs w, const float* __restrict__ item,
                                                  const float* __restrict__ ibias, int64_t rows, OrxHash hi, int epoch) {
  __shared__ int32_t rc[SH_MAX_R], goff[SH_MAX_R], gbase[SH_MAX_R + 1];
  __shared__ int total_sh;
  const int R = x.world, me = x.rank, D = x.D, nq = D >> 2;
  orx_pdl_wait();
  sh_wait(x, 1, epoch);
  if (threadIdx.x == 0) {
    const int32_t* m = x.meta[me];
    int acc = 0;
    for (int h = 0; h < R; ++h) {
      int c = __ldcg(m + SH_META * h + SH_M_REQS);
      c = c < 0 ? 0 : (c > x.req_cap ? x.req_cap : c);
      int g = __ldcg(m + SH_META * h + SH_M_GOTOFF);
      if (g < 0 || g + c > x.got_rows) { g = 0; c = 0; }
      rc[h] = c;
      goff[h] = g;
      gbase[h] = acc;
      acc += (c + 31) & ~31;
    }
    gbase[R] = acc;
    if (acc > x.gin_cap) {              // my gradient inbox cannot take this batch: sticky error, serve what fits
      atomicCAS(x.flags[me] + SH_ERR_WORD, 0, 4);
      acc = x.gin_cap & ~31;
    }
    total_sh = acc;
  }
  __syncthreads();
  const int total = total_sh;
  if (blockIdx.x == 0) {
    if ((int)threadIdx.x < R) x.meta[threadIdx.x][SH_META * me + SH_M_GINBASE] = gbase[threadIdx.x];
    if (threadIdx.x == 0) w.ctl[SH_C_NREQ] = total;
  }
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  const int32_t* box = x.idbox[me];
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  // a warp moves 8 consecutive inbox rows per iteration (same source: bases are multiples of 32): lanes 0..7 resolve
  // ids, index them and move the biases (one 32 B run); then all 8 rows are loaded before the first peer store
  for (int j0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 8; j0 < total; j0 += nw * 8) {
    const int h = sh_bucket_of(gbase, R, j0);
    const int idx0 = j0 - gbase[h];
    if (idx0 >= rc[h]) {                 // pure padding
      if (lane < 8) w.req[j0 + lane] = -1;
      continue;
    }
    int32_t my_id = -1;
    bool valid = false;
    if (lane < 8) {
      valid = idx0 + lane < rc[h];
      int32_t id = valid ? __ldcg(box + (int64_t)h * x.req_cap + idx0 + lane) : -1;
      if (id < 0 || (int64_t)id >= rows) id = -1;
      my_id = id;
    }
    const unsigned vmask = __ballot_sync(ORX_FULL, valid) & 0xffu;
    float* dst0 = x.got[h] + (int64_t)(goff[h] + idx0) * D;
    float4 v[8][NQ];
#pragma unroll
    for (int k = 0; k < 8; ++k) {     // all eight rows in flight before anything that stalls (the index inserts below)
      const int32_t id = __shfl_sync(ORX_FULL, my_id, k);
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int e = q * 32 + lane;
        v[k][q] = (id >= 0 && e < nq) ? __ldcg(reinterpret_cast<const float4*>(item + (int64_t)id * D) + e) : z4;
      }
    }
    if (lane < 8) {
      w.req[j0 + lane] = my_id;
      const float b = my_id >= 0 ? __ldcg(ibias + my_id) : 0.f;
      if (my_id >= 0) orx_hash_insert(hi, my_id, 0);
      if (valid) x.gotb[h][goff[h] + idx0 + lane] = b;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (!((vmask >> k) & 1u)) continue;
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int e = q * 32 + lane;
        if (e < nq) reinterpret_cast<float4*>(dst0 + (int64_t)k * D)[e] = v[k][q];
      }
    }
  }
  orx_pdl_trigger();
  sh_arrive(x, w.ctl + SH_C_DONE + 2, gridDim.x, 2, epoch, [&]() {});
}

// ---------------------------------------------------------------------------------------
// phase 3: home: score, user update, item gradient rows -> owners
// ---------------------------------------------------------------------------------------
struct ShCompArgs {
  float *U, *Us0, *Us1;     // local user shard + slots
  OrxHash hu;
  float* gu;                // user staging [.., D]
  float margin, c_loss, c_l2, inv_B, loss_scale;
  OrxOptDev opt;
  float* partials;          // [2 * warps of the grid]
};

template <int KIND, int OPT, int NQ>
__global__ void __launch_bounds__(256) k_sh_compute(ShardDev x, ShardWs w, ShCompArgs a, int epoch) {
  typedef OrxOptSlots<OPT> SL;
  constexpr int TPW = NQ == 1 ? 4 : (NQ == 2 ? 2 : 1);     // triplets in flight per warp
  __shared__ int32_t goff[SH_MAX_R], gbase[SH_MAX_R];
  const int R = x.world, me = x.rank, D = x.D, nq = D >> 2;
  orx_pdl_wait();
  sh_wait(x, 2, epoch);
  if ((int)threadIdx.x < R) {
    goff[threadIdx.x] = w.ctl[SH_C_GOFF + threadIdx.x];
    gbase[threadIdx.x] = __ldcg(x.meta[me] + SH_META * threadIdx.x + SH_M_GINBASE);
  }
  __syncthreads();
  const int T = w.ctl[SH_C_T];
  const int lane = threadIdx.x & 31;
  const int gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const float* got = x.got[me];
  const float* gotb = x.gotb[me];
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float loss_acc = 0.f, l2_acc = 0.f;
  for (int t0 = gwarp * TPW; t0 < T; t0 += nw * TPW) {
    // lanes 0..TPW-1: ids, positions, destinations and the user-row probe of triplet t0 + lane
    int my_u = -1, my_du = -1, my_own = 0, my_pp = 0, my_pn = 0;
    float* my_dp = nullptr;
    float* my_dn = nullptr;
    float* my_bdp = nullptr;
    float* my_bdn = nullptr;
    float my_bp = 0.f, my_bn = 0.f;
    if (lane < TPW && t0 + lane < T) {
      const int t = t0 + lane;
      const int32_t sp = w.slot[2 * t], sn = w.slot[2 * t + 1];
      if (sp >= 0 && sn >= 0) {
        my_u = w.trip_u[t];
        const int op = sp >> SH_IDX_BITS, ip = sp & ((1 << SH_IDX_BITS) - 1);
        const int on = sn >> SH_IDX_BITS, in = sn & ((1 << SH_IDX_BITS) - 1);
        my_pp = goff[op] + ip;
        my_pn = goff[on] + in;
        if (gbase[op] >= 0 && gbase[op] + ip < x.gin_cap) {
          my_dp = x.gin[op] + (int64_t)(gbase[op] + ip) * D;
          my_bdp = x.ginb[op] + gbase[op] + ip;
        }
        if (gbase[on] >= 0 && gbase[on] + in < x.gin_cap) {
          my_dn = x.gin[on] + (int64_t)(gbase[on] + in) * D;
          my_bdn = x.ginb[on] + gbase[on] + in;
        }
        my_bp = __ldcg(gotb + my_pp);
        my_bn = __ldcg(gotb + my_pn);
        my_own = orx_hash_find(a.hu, my_u, &my_du) == 1u;
      }
    }
    float4 u[TPW][NQ], p[TPW][NQ], n[TPW][NQ], us0[TPW][NQ], us1[TPW][NQ];
    int uu[TPW];
#pragma unroll
    for (int k = 0; k < TPW; ++k) {
      uu[k] = __shfl_sync(ORX_FULL, my_u, k);
      const int pp = __shfl_sync(ORX_FULL, my_pp, k), pn = __shfl_sync(ORX_FULL, my_pn, k);
      const int own = __shfl_sync(ORX_FULL, my_own, k);
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int e = q * 32 + lane;
        const bool on = uu[k] >= 0 && e < nq;
        u[k][q] = on ? __ldcg(reinterpret_cast<const float4*>(a.U + (int64_t)uu[k] * D) + e) : z4;
        p[k][q] = on ? __ldcg(reinterpret_cast<const float4*>(got + (int64_t)pp * D) + e) : z4;
        n[k][q] = on ? __ldcg(reinterpret_cast<const float4*>(got + (int64_t)pn * D) + e) : z4;
        us0[k][q] = (SL::S0 && on && own) ? __ldcg(reinterpret_cast<const float4*>(a.Us0 + (int64_t)uu[k] * D) + e) : z4;
        us1[k][q] = (SL::S1 && on && own) ? __ldcg(reinterpret_cast<const float4*>(a.Us1 + (int64_t)uu[k] * D) + e) : z4;
      }
    }
#pragma unroll
    for (int k = 0; k < TPW; ++k) {
      if (uu[k] < 0) continue;                       // warp-uniform
      float s1 = 0.f, s2 = 0.f, sq = 0.f;
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        if (KIND == ORX_PAIR_BPR) {
          s1 += dot4(u[k][q], p[k][q]);
          s2 += dot4(u[k][q], n[k][q]);
        } else {
          s1 += sqd4(u[k][q], p[k][q]);
          s2 += sqd4(u[k][q], n[k][q]);
        }
        sq += dot4(u[k][q], u[k][q]) + dot4(p[k][q], p[k][q]) + dot4(n[k][q], n[k][q]);
      }
      l2_acc += sq;
      s1 = orx_group_sum<32>(s1);
      s2 = orx_group_sum<32>(s2);
      const float bp = __shfl_sync(ORX_FULL, my_bp, k), bn = __shfl_sync(ORX_FULL, my_bn, k);
      float lt, g;
      pair_score<KIND>(s1, s2, bp, bn, a.margin, a.c_loss, a.inv_B, &lt, &g);
      if (lane == 0) loss_acc += lt;
      const int own = __shfl_sync(ORX_FULL, my_own, k);
      const int du = __shfl_sync(ORX_FULL, my_du, k);
      float* dp = reinterpret_cast<float*>(__shfl_sync(ORX_FULL, (unsigned long long)my_dp, k));
      float* dn = reinterpret_cast<float*>(__shfl_sync(ORX_FULL, (unsigned long long)my_dn, k));
      const int pp = __shfl_sync(ORX_FULL, my_pp, k), pn = __shfl_sync(ORX_FULL, my_pn, k);
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int e = q * 32 + lane;
        if (e >= nq) continue;
        float4 gu, gp, gn;
        pair_row_grads<KIND>(g, a.c_l2, u[k][q], p[k][q], n[k][q], &gu, &gp, &gn);
        if (dp) reinterpret_cast<float4*>(dp)[e] = gp;           // peer stores: the item gradient rows
        if (dn) reinterpret_cast<float4*>(dn)[e] = gn;
        // own: the only reference of this user row in the global batch
        orx_own_or_stage4<OPT, false>(own, a.U, a.Us0, a.Us1, uu[k], a.gu, du, D, 4 * e, u[k][q], gu, us0[k][q],
                                      us1[k][q], a.opt);
      }
      {                         // bias gradient of the positive item: BPR +g, UCML -g; the negative gets the opposite sign
        float* bdp = reinterpret_cast<float*>(__shfl_sync(ORX_FULL, (unsigned long long)my_bdp, k));
        float* bdn = reinterpret_cast<float*>(__shfl_sync(ORX_FULL, (unsigned long long)my_bdn, k));
        const float gb = (KIND == ORX_PAIR_BPR) ? g : -g;
        if (lane == 0) {        // one 4-byte peer store each, at the inbox row of the gradient row
          if (bdp) *bdp = gb;
          if (bdn) *bdn = -gb;
        }
      }
    }
  }
  orx_pdl_trigger();
  orx_warp_partial(loss_acc, l2_acc, a.partials);
  // The LAST block to finish reduces this rank's (loss, l2) partials, sends the pair to every rank and releases flag 3.
  sh_arrive(x, w.ctl + SH_C_DONE + 3, gridDim.x, 3, epoch, [&]() {
    double l, q;                                       // deterministic (fixed order, double) reduction of my partials
    orx_block_sum_partials(a.partials, (int)((gridDim.x * blockDim.x) >> 5), nullptr, 0, &l, &q);
    if ((int)threadIdx.x < R) {
      int32_t* m = x.meta[threadIdx.x] + SH_META * me;
      m[SH_M_LOSS] = __float_as_int((float)(l * (double)a.loss_scale));
      m[SH_M_L2] = __float_as_int((float)(0.5 * q));
    }
  });
}

// ---------------------------------------------------------------------------------------
// phase 4: owner: gradient inbox -> item rows
// ---------------------------------------------------------------------------------------
struct ShApplyArgs {
  float *I, *Is0, *Is1;     // local item shard + slots
  float *Bv, *Bs0, *Bs1;    // local item bias [rows] + slots
  OrxHash hi;
  float *gi, *gb;           // item staging rows / biases
  OrxOptDev opt;
};

// The prologue of the NEXT step (its route and request roles) rides in the first blocks of this launch when the caller
// announced the next batch: apply is HBM-bound and needs no NVLink, the two roles are short and latency-bound (two
// cross-rank handoffs), so they hide completely under it.  What they write is dead or private by now: tripbox / idbox /
// the TRIPS, REQS and GOTOFF meta words were last read by request / serve of THIS step, which every rank finished before
// any rank's compute -- and so before any rank's apply -- could start; trip_u / slot / the control words were last read
// by this rank's compute; the user index of the next step is a second hash set (tail of this step still reads this one).
struct ShProArgs {
  int n_route, n_request;   // blocks of each role (0 = no prologue in this launch)
  int epoch;                // of the announced step
  ShRouteArgs r;
  OrxHash hu;               // user index of the announced step
};

template <int OPT, int NQ>
__global__ void __launch_bounds__(256) k_sh_apply(ShardDev x, ShardWs w, ShApplyArgs a, ShProArgs pro, int epoch) {
  typedef OrxOptSlots<OPT> SL;
  constexpr int GRP = NQ == 1 ? 4 : (NQ == 2 ? 2 : 1);   // rows whose loads are issued together
  const int me = x.rank, D = x.D, nq = D >> 2;
  orx_pdl_wait();
  if ((int)blockIdx.x < pro.n_route) {                    // block-uniform role dispatch
    sh_route_role(x, w, pro.r, pro.epoch, blockIdx.x, pro.n_route);
    orx_pdl_trigger();
    return;
  }
  if ((int)blockIdx.x < pro.n_route + pro.n_request) {
    sh_request_role(x, w, pro.hu, pro.epoch, blockIdx.x - pro.n_route, pro.n_request);
    orx_pdl_trigger();
    return;
  }
  sh_wait(x, 3, epoch);
  const int n = w.ctl[SH_C_NREQ];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float* gin = x.gin[me];
  const float* ginb = x.ginb[me];
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  __shared__ int chunk_sh;
  // 64-row chunks handed out by a counter: blocks that start late (behind the prologue blocks) just take fewer chunks
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) chunk_sh = atomicAdd(w.ctl + SH_C_ACUR, 1);
    __syncthreads();
    const int j0 = chunk_sh * 64 + wid * 8;
    if (chunk_sh * 64 >= n) break;
    if (j0 >= n) continue;
    int32_t my_id = -1;
    int my_d = -1, my_own = 0;
    if (lane < 8) {
      my_id = w.req[j0 + lane];
      if (my_id >= 0) {
        my_own = orx_hash_find(a.hi, my_id, &my_d) == 1u;
        const float gbv = __ldcg(ginb + j0 + lane);
        if (my_own) {            // bias of a row requested once: lane-parallel, straight from the inbox
          float s0v = SL::S0 ? __ldcg(a.Bs0 + my_id) : 0.f, s1v = SL::S1 ? __ldcg(a.Bs1 + my_id) : 0.f;
          __stcg(a.Bv + my_id, orx_apply<OPT>(__ldcg(a.Bv + my_id), gbv, s0v, s1v, a.opt));
          if (SL::S0) __stcg(a.Bs0 + my_id, s0v);
          if (SL::S1) __stcg(a.Bs1 + my_id, s1v);
        } else {
          atomicAdd(a.gb + my_d, gbv);
        }
      }
    }
    if (__ballot_sync(ORX_FULL, my_id >= 0) == 0u) continue;
#pragma unroll
    for (int k0 = 0; k0 < 8; k0 += GRP) {
      float4 g[GRP][NQ], wv[GRP][NQ], s0v[GRP][NQ], s1v[GRP][NQ];
      int id[GRP], own[GRP], d[GRP];
#pragma unroll
      for (int k = 0; k < GRP; ++k) {
        id[k] = __shfl_sync(ORX_FULL, my_id, k0 + k);
        own[k] = __shfl_sync(ORX_FULL, my_own, k0 + k);
        d[k] = __shfl_sync(ORX_FULL, my_d, k0 + k);
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
          const int e = q * 32 + lane;
          const bool on = id[k] >= 0 && e < nq;
          g[k][q] = on ? __ldcg(reinterpret_cast<const float4*>(gin + (int64_t)(j0 + k0 + k) * D) + e) : z4;
          const bool ld = on && own[k];
          wv[k][q] = ld ? __ldcg(reinterpret_cast<const float4*>(a.I + (int64_t)id[k] * D) + e) : z4;
          s0v[k][q] = (SL::S0 && ld) ? __ldcg(reinterpret_cast<const float4*>(a.Is0 + (int64_t)id[k] * D) + e) : z4;
          s1v[k][q] = (SL::S1 && ld) ? __ldcg(reinterpret_cast<const float4*>(a.Is1 + (int64_t)id[k] * D) + e) : z4;
        }
      }
#pragma unroll
      for (int k = 0; k < GRP; ++k) {
        if (id[k] < 0) continue;
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
          const int e = q * 32 + lane;
          if (e >= nq) continue;
          orx_own_or_stage4<OPT, false>(own[k], a.I, a.Is0, a.Is1, id[k], a.gi, d[k], D, 4 * e, wv[k][q], g[k][q],
                                        s0v[k][q], s1v[k][q], a.opt);
        }
      }
    }
  }
  orx_pdl_trigger();
}

// staged (duplicated) user and item rows -> optimizer, once per unique row, staging re-zeroed: the rows of the
// single-GPU tail (orx_tail_rows); global (loss, l2) from the meta mailbox; counters reset.
template <int OPT>
__global__ void __launch_bounds__(256) k_sh_tail(ShardDev x, ShardWs w, TailArgs a, int par) {
  orx_pdl_wait();
  const int nu = *a.hu.counter, ni = *a.hi.counter;
  orx_tail_rows<OPT>(a, nu, ni);
  if (blockIdx.x == 0 && threadIdx.x == 0) {    // every rank adds the R pairs it holds in rank order: bit-identical totals
    const int32_t* m = x.meta[x.rank];
    float l = 0.f, q = 0.f;
    for (int r = 0; r < x.world; ++r) {
      l += __int_as_float(__ldcg(m + SH_META * r + SH_M_LOSS));
      q += __int_as_float(__ldcg(m + SH_META * r + SH_M_L2));
    }
    a.out4[0] = l;
    a.out4[1] = q;
    a.out4[2] = (float)w.ctl[SH_C_BAD + par];
    a.out4[3] = (float)(nu + ni);
    w.ctl[SH_C_BAD + par] = 0;
    w.ctl[SH_C_ACUR] = 0;
  }
  __shared__ bool last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last = (atomicAdd(a.counters + 2, 1) == (int)gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    *a.hu.counter = 0;
    *a.hi.counter = 0;
    a.counters[2] = 0;
  }
}

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
struct orx_shard_ws {
  ShardWs w;                         // carved from the handle's shard_scratch by sh_layout
  int home_cap, gin_cap, got_rows;
  const void* occ_fn[32];            // sh_ctas_per_sm: resident CTAs per SM of each persistent kernel launched so far
  int occ[32], n_occ;
  // prologue bookkeeping, per step parity: which step's route / request were issued, with which index epochs and ids
  int32_t pro_route[2], pro_request[2];
  uint32_t ep_u[2], ep_i[2];
  const int32_t *ids_u[2], *ids_p[2], *ids_n[2];
  int32_t ids_B[2];
  int32_t serve_epoch, tail_epoch;   // last step whose serve / tail was issued (different = a step's item index is live)
  const void* owner;                 // the model (its flag mailbox) this bookkeeping belongs to
};

// ---- IPC-exportable device memory: every rank maps every other rank's mailboxes (cudaIpc*, one box, NVLink) ----
extern "C" int orx_peer_alloc(orx_handle_t h, int64_t bytes, void** dev_ptr_out, uint8_t* handle_out64) {
  ORX_REQUIRE(h != nullptr && dev_ptr_out && handle_out64 && bytes > 0, "bad arguments");
  ORX_CUDA(cudaSetDevice(h->device));
  void* p = nullptr;
  ORX_CUDA(cudaMalloc(&p, (size_t)bytes));
  ORX_CUDA(cudaMemset(p, 0, (size_t)bytes));
  ORX_CUDA(cudaDeviceSynchronize());
  cudaIpcMemHandle_t hd;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  ORX_CUDA(cudaIpcGetMemHandle(&hd, p));
  memcpy(handle_out64, &hd, 64);
  *dev_ptr_out = p;
  return ORX_OK;
}

extern "C" int orx_peer_open(orx_handle_t h, const uint8_t* handle64, void** dev_ptr_out) {
  ORX_REQUIRE(h != nullptr && dev_ptr_out && handle64, "bad arguments");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaIpcMemHandle_t hd;
  memcpy(&hd, handle64, 64);
  void* p = nullptr;
  ORX_CUDA(cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
  *dev_ptr_out = p;
  return ORX_OK;
}

extern "C" int orx_peer_close(orx_handle_t h, void* dev_ptr) {
  ORX_REQUIRE(h != nullptr, "null handle");
  if (dev_ptr) ORX_CUDA(cudaIpcCloseMemHandle(dev_ptr));
  return ORX_OK;
}

extern "C" int orx_peer_free(orx_handle_t h, void* dev_ptr) {
  ORX_REQUIRE(h != nullptr, "null handle");
  if (dev_ptr) ORX_CUDA(cudaFree(dev_ptr));
  return ORX_OK;
}

// resident CTAs per SM of a 256-thread kernel (cached per kernel in the workspace, i.e. for the handle's device):
// persistent grids are sized to exactly one wave
static int sh_ctas_per_sm(orx_shard_ws* s, const void* fn, int cap) {
  for (int i = 0; i < s->n_occ; ++i)
    if (s->occ_fn[i] == fn) return s->occ[i] < cap ? s->occ[i] : cap;
  int nb = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, fn, 256, 0) != cudaSuccess || nb < 1) nb = 1;
  if (s->n_occ < 32) { s->occ_fn[s->n_occ] = fn; s->occ[s->n_occ++] = nb; }
  return nb < cap ? nb : cap;
}

// The local scratch (trip_u | slot | req | ctl) inside one allocation; with base == nullptr only the size is computed.
static size_t sh_layout(char* base, int home_cap, int gin_cap, ShardWs* w) {
  size_t off = 0;
  auto take = [&](size_t words) {
    int32_t* p = base ? reinterpret_cast<int32_t*>(base + off) : nullptr;
    off += (sizeof(int32_t) * words + 255) & ~(size_t)255;
    return p;
  };
  w->trip_u = take((size_t)home_cap);
  w->slot = take(2 * (size_t)home_cap);
  w->req = take((size_t)gin_cap);
  w->ctl = take(SH_C_WORDS);
  return off;
}

// the device scratch stays with the handle (shard_scratch, freed by orx_destroy)
void orx_shard_ws_release(orx_ctx* c) {
  delete (orx_shard_ws*)c->shard_ws;
  c->shard_ws = nullptr;
}

// A route issued for a step whose tail has not been issued yet: that step's user index lives in pf_u[its parity]
bool orx_shard_holds_index(const orx_ctx* c) {
  const orx_shard_ws* s = (const orx_shard_ws*)c->shard_ws;
  return s && (s->pro_route[0] > s->tail_epoch || s->pro_route[1] > s->tail_epoch);
}

static int shard_ws_ensure(orx_ctx* c, const ShardHost* x, cudaStream_t st) {
  orx_shard_ws* s = (orx_shard_ws*)c->shard_ws;
  const int got_rows = sh_got_rows(x->home_cap, x->world);
  if (s && s->home_cap >= x->home_cap && s->gin_cap >= x->gin_cap && s->got_rows >= got_rows) return ORX_OK;
  // a new layout starts afresh: zeroed bookkeeping and control words
  orx_shard_ws_release(c);
  c->shard_ws = s = new orx_shard_ws();
  int rc = orx_grow(&c->shard_scratch, &c->shard_cap, sh_layout(nullptr, x->home_cap, x->gin_cap, &s->w));
  if (rc) return rc;
  sh_layout(static_cast<char*>(c->shard_scratch), x->home_cap, x->gin_cap, &s->w);
  ORX_CUDA(cudaMemsetAsync(s->w.ctl, 0, sizeof(int32_t) * SH_C_WORDS, st));
  s->home_cap = x->home_cap;
  s->gin_cap = x->gin_cap;
  s->got_rows = got_rows;
  return ORX_OK;
}

static int shard_check(orx_handle_t h, const ShardHost* x) {
  ORX_REQUIRE(h != nullptr && x != nullptr, "null handle / descriptor");
  ORX_REQUIRE(x->world >= 1 && x->world <= SH_MAX_R && x->rank >= 0 && x->rank < x->world, "bad world / rank");
  ORX_REQUIRE(x->dim >= 4 && (x->dim & 3) == 0 && x->dim <= 512, "dim must be a multiple of 4 in [4, 512]");
  ORX_REQUIRE(x->batch_cap > 0 && x->home_cap > 0 && x->req_cap > 0 && x->gin_cap >= 32 && x->timeout_ms > 0, "bad capacities");
  ORX_REQUIRE(x->req_cap < (1 << SH_IDX_BITS), "req_cap must stay below 2^24");
  ORX_REQUIRE(x->tripbox && x->idbox && x->got && x->gotb && x->gin && x->ginb && x->meta && x->flags, "null mailbox pointer table");
  return ORX_OK;
}

static ShardDev shard_to_dev(const ShardHost* x) {
  ShardDev d;
  d.world = x->world; d.rank = x->rank; d.D = x->dim; d.batch_cap = x->batch_cap; d.home_cap = x->home_cap;
  d.req_cap = x->req_cap; d.gin_cap = x->gin_cap; d.got_rows = sh_got_rows(x->home_cap, x->world);
  d.timeout_ns = (unsigned long long)x->timeout_ms * 1000000ull;
  d.tripbox = (int32_t* const*)x->tripbox; d.idbox = (int32_t* const*)x->idbox;
  d.got = (float* const*)x->got; d.gotb = (float* const*)x->gotb;
  d.gin = (float* const*)x->gin; d.ginb = (float* const*)x->ginb;
  d.meta = (int32_t* const*)x->meta; d.flags = (int32_t* const*)x->flags;
  return d;
}

extern "C" int orx_shard_sizes(const orx_shard_t* xs, int64_t* n8_host) {
  const ShardHost* x = (const ShardHost*)xs;
  ORX_REQUIRE(x != nullptr && n8_host != nullptr, "null pointer");
  ORX_REQUIRE(x->world >= 1 && x->world <= SH_MAX_R && x->dim > 0 && x->batch_cap > 0 && x->home_cap > 0 && x->req_cap > 0 &&
              x->gin_cap > 0, "bad descriptor");
  const int64_t got_rows = sh_got_rows(x->home_cap, x->world);
  n8_host[0] = (int64_t)x->world * 3 * x->batch_cap;        // tripbox int32
  n8_host[1] = (int64_t)x->world * x->req_cap;              // idbox int32
  n8_host[2] = got_rows * x->dim;                           // got float
  n8_host[3] = got_rows;                                    // gotb float
  n8_host[4] = (int64_t)x->gin_cap * x->dim;                // gin float
  n8_host[5] = x->gin_cap;                                  // ginb float
  n8_host[6] = (int64_t)x->world * SH_META;                 // meta int32
  n8_host[7] = SH_ERR_WORD + 1;                             // flags int32
  return ORX_OK;
}

// runtime -> template arguments of the sharded kernels: the optimizers the sharded step supports (it rejects ADAM_DENSE)
// and the row-width classes NQ (float4 per lane: D <= 128, 256, 512)
template <typename F>
static inline auto sh_dispatch_opt(int opt_kind, F&& f) {
  return orx_dispatch<ORX_OPT_SGD, ORX_OPT_ADAGRAD, ORX_OPT_ADAM_LAZY>(opt_kind, f);
}
template <typename F>
static inline auto sh_dispatch_nq(int nq, F&& f) {
  return orx_dispatch<1, 2, 4>(nq <= 32 ? 1 : (nq <= 64 ? 2 : 4), f);
}

// two fresh index epochs (user set of the step, item set of the step).  A 31-bit wrap empties every table of the handle
// after draining the device (orx_next_epoch), which must not happen while another step's index is live: `may_drain` says
// whether it may; returns 1 (and takes nothing) when it may not and the wrap is near.
static int shard_take_epochs(orx_ctx* c, cudaStream_t st, bool may_drain, uint32_t* eu, uint32_t* ei) {
  if (c->epoch >= 0x7ffffff0u) {
    if (!may_drain) return 1;
    c->epoch = 0x7fffffffu;      // wrap now, at a step boundary: both epochs come from after the wrap
  }
  int rc;
  if ((rc = orx_next_epoch(c, st))) return rc;
  *eu = c->epoch;
  if ((rc = orx_next_epoch(c, st))) return rc;
  *ei = c->epoch;
  return ORX_OK;
}

// One step (or a sub-range of its six launches: phases 0 route, 1 request, 2 serve, 3 compute, 4 apply, 5 tail); see the
// file header.  out4 = { loss, l2_loss, skipped triplets (ids out of range), staged rows }, the first two GLOBAL and
// identical on every rank.
//
// next_uid / next_pid / next_nid / next_B (all-or-none, device pointers that stay valid until that step ran) ANNOUNCE the
// batch of step epoch + 1: its route and request ride inside this step's apply launch (ShProArgs), and the call for
// epoch + 1 -- which must pass exactly these pointers -- starts at serve.  Every rank must announce or none (a rank that
// does not would have its peers' next request wait for a route that comes a step later: slower, not wrong).
// Phases 0 and 1 of a step may also be issued explicitly ahead of phases 4 and 5 of the step before (the 1-GPU loopback
// does: fused roles of R virtual ranks on one stream would wait for each other).
extern "C" int orx_shard_step(orx_handle_t h, int32_t kind, const orx_shard_t* xs, const orx_table_t* user,
                              const orx_table_t* item, const orx_table_t* item_bias, const int32_t* uid, const int32_t* pid,
                              const int32_t* nid, int32_t B, const int32_t* next_uid, const int32_t* next_pid,
                              const int32_t* next_nid, int32_t next_B, int64_t total_users, int64_t total_items, float margin,
                              float c_loss, float c_l2, float inv_B, const orx_opt_t* opt, int32_t epoch, int32_t phase_lo,
                              int32_t phase_hi, float* out4, orx_stream_t s) {
  const ShardHost* x = (const ShardHost*)xs;
  int rc = shard_check(h, x);
  if (rc) return rc;
  ORX_REQUIRE(kind == ORX_PAIR_BPR || kind == ORX_PAIR_UCML, "unknown pairwise kind");
  ORX_REQUIRE(user && item && item_bias && user->var && item->var && item_bias->var && opt && out4, "null pointer");
  ORX_REQUIRE(user->dim == x->dim && item->dim == x->dim && item_bias->dim == 1 && item_bias->rows == item->rows, "table shapes");
  ORX_REQUIRE(B > 0 && B <= x->batch_cap && uid && pid && nid, "bad batch (larger than the mailboxes were built for?)");
  const bool announce = next_uid != nullptr;
  ORX_REQUIRE(announce == (next_pid != nullptr) && announce == (next_nid != nullptr), "next_uid / next_pid / next_nid: all or none");
  if (announce) ORX_REQUIRE(next_B > 0 && next_B <= x->batch_cap, "bad announced batch");
  ORX_REQUIRE(total_users > 0 && total_items > 0 && epoch > 0 && epoch < 0x7ffffffe, "bad totals / epoch");
  ORX_REQUIRE(phase_lo >= 0 && phase_hi <= 5 && phase_lo <= phase_hi, "bad phase range");
  ORX_REQUIRE(opt->kind == ORX_OPT_SGD || opt->kind == ORX_OPT_ADAGRAD || opt->kind == ORX_OPT_ADAM_LAZY,
              "the sharded step supports SGD, Adagrad and row-sparse Adam");
  ORX_REQUIRE(orx_opt_slots_ok(opt->kind, {user, item, item_bias}), "optimizer slot rows missing");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  // index hashes + staging: user side <= home_cap lookups, item side <= gin_cap lookups
  const int64_t need = x->home_cap > (x->gin_cap + 1) / 2 ? x->home_cap : (x->gin_cap + 1) / 2;
  if ((rc = orx_ensure_workspace(h, need, x->dim))) return rc;
  if ((rc = shard_ws_ensure(h, x, st))) return rc;
  orx_shard_ws* S = (orx_shard_ws*)h->shard_ws;
  if (S->owner != x->flags) {        // another model on this handle (each has its own mailboxes): its steps start afresh
    ORX_REQUIRE(S->serve_epoch == S->tail_epoch && S->pro_route[0] <= S->tail_epoch && S->pro_route[1] <= S->tail_epoch,
                "another sharded model on this handle has a step in flight or an announced batch outstanding");
    memset(S->pro_route, 0, sizeof(S->pro_route));
    memset(S->pro_request, 0, sizeof(S->pro_request));
    S->serve_epoch = S->tail_epoch = 0;
    S->owner = x->flags;
  }
  ORX_REQUIRE(!h->pf_valid, "this handle has an index prefetched by orx_pairwise_prefetch outstanding (the sharded step uses the same index sets)");
  const ShardWs& w = S->w;
  const ShardDev xd = shard_to_dev(x);
  const int par = epoch & 1;
  const OrxOptDev od = orx_opt_to_dev(opt);
  const int nq = x->dim >> 2;
  // compute grid <= 4 CTAs/SM x 8 warps, one (loss, l2) pair each
  if ((rc = orx_grow((void**)&h->partials, &h->partials_cap, sizeof(float) * 2 * (size_t)(h->num_sms * 4 * 8)))) return rc;
  const int route_blocks = (B + 1023) / 1024;
  int request_blocks = (x->home_cap + 511) / 512;
  if (request_blocks > h->num_sms) request_blocks = h->num_sms;

  // phases 0 / 1: unless this step's prologue was already issued (announced in the previous call, or explicitly)
  if (phase_lo == 0 && S->pro_route[par] != epoch) {
    if ((rc = shard_take_epochs(h, st, S->serve_epoch == S->tail_epoch, &S->ep_u[par], &S->ep_i[par])) != ORX_OK) {
      if (rc == 1) { orx_set_error("orx_shard_step: index epochs are about to wrap; issue this step's route after the previous step's tail"); return ORX_ERR_INVALID; }
      return rc;
    }
    S->ids_u[par] = uid; S->ids_p[par] = pid; S->ids_n[par] = nid; S->ids_B[par] = B;
  }
  if (S->pro_route[par] == epoch || phase_lo == 0)      // whichever way the prologue was issued: it must be for THIS batch
    ORX_REQUIRE(S->ids_u[par] == uid && S->ids_p[par] == pid && S->ids_n[par] == nid && S->ids_B[par] == B,
                "this step's batch differs from the one its route was issued for (announced as next_* in the previous call)");
  OrxHash hu = h->pf_u[par];
  hu.epoch = S->ep_u[par];
  OrxHash hi = h->hi;
  hi.epoch = S->ep_i[par];

  ShCompArgs ca;
  ca.U = user->var; ca.Us0 = user->s0; ca.Us1 = user->s1; ca.hu = hu; ca.gu = h->gu;
  ca.margin = margin; ca.c_loss = c_loss; ca.c_l2 = c_l2; ca.inv_B = inv_B; ca.opt = od; ca.partials = h->partials;
  ca.loss_scale = kind == ORX_PAIR_BPR ? inv_B : 1.f;
  ShApplyArgs aa;
  aa.I = item->var; aa.Is0 = item->s0; aa.Is1 = item->s1;
  aa.Bv = item_bias->var; aa.Bs0 = item_bias->s0; aa.Bs1 = item_bias->s1;
  aa.hi = hi; aa.gi = h->gi; aa.gb = h->gb; aa.opt = od;
  const bool whole = phase_lo == 0 && phase_hi == 5;     // the measurement hook follows whole steps only
  for (int ph = phase_lo; ph <= phase_hi; ++ph) {
    if (whole) orx_prof_mark(h, ph, st);
    switch (ph) {
      case 0: {
        if (S->pro_route[par] == epoch) break;           // rode in the previous step's apply launch
        ShRouteArgs ra;
        ra.uid = uid; ra.pid = pid; ra.nid = nid; ra.B = B; ra.U = total_users; ra.I = total_items;
        ORX_CUDA(orx_launch_pdl(k_sh_route, dim3(route_blocks), dim3(256), 0, st, xd, w, ra, epoch));
        S->pro_route[par] = epoch;
        break;
      }
      case 1:
        if (S->pro_request[par] == epoch) break;
        ORX_REQUIRE(S->pro_route[par] == epoch, "phase 1 before phase 0");
        ORX_CUDA(orx_launch_pdl(k_sh_request, dim3(request_blocks), dim3(256), 0, st, xd, w, hu, epoch));
        S->pro_request[par] = epoch;
        break;
      case 2:
        ORX_REQUIRE(S->pro_request[par] == epoch, "phase 2 before this step's phases 0 and 1");
        sh_dispatch_nq(nq, [&](auto Q) {
          auto kern = k_sh_serve<decltype(Q)::value>;
          orx_launch_pdl(kern, dim3(h->num_sms * sh_ctas_per_sm(S, (const void*)kern, 4)), dim3(256), 0, st, xd, w,
                         (const float*)item->var, (const float*)item_bias->var, (int64_t)item->rows, hi, epoch);
        });
        S->serve_epoch = epoch;
        break;
      case 3:
        orx_dispatch<ORX_PAIR_BPR, ORX_PAIR_UCML>(kind, [&](auto K) {
          sh_dispatch_opt(opt->kind, [&](auto O) {
            sh_dispatch_nq(nq, [&](auto Q) {
              auto kern = k_sh_compute<decltype(K)::value, decltype(O)::value, decltype(Q)::value>;
              orx_launch_pdl(kern, dim3(h->num_sms * sh_ctas_per_sm(S, (const void*)kern, 4)), dim3(256), 0, st, xd, w,
                             ca, epoch);
            });
          });
        });
        break;
      case 4: {
        ShProArgs pro;
        memset(&pro, 0, sizeof(pro));
        const int np = par ^ 1;
        if (announce && S->pro_route[np] != epoch + 1 &&
            shard_take_epochs(h, st, false, &S->ep_u[np], &S->ep_i[np]) == ORX_OK) {
          pro.n_route = (next_B + 1023) / 1024;
          pro.n_request = request_blocks;
          pro.epoch = epoch + 1;
          pro.r.uid = next_uid; pro.r.pid = next_pid; pro.r.nid = next_nid; pro.r.B = next_B;
          pro.r.U = total_users; pro.r.I = total_items;
          pro.hu = h->pf_u[np];
          pro.hu.epoch = S->ep_u[np];
          S->ids_u[np] = next_uid; S->ids_p[np] = next_pid; S->ids_n[np] = next_nid; S->ids_B[np] = next_B;
          S->pro_route[np] = S->pro_request[np] = epoch + 1;
        }
        sh_dispatch_opt(opt->kind, [&](auto O) {
          sh_dispatch_nq(nq, [&](auto Q) {
            auto kern = k_sh_apply<decltype(O)::value, decltype(Q)::value>;
            const int g = h->num_sms * sh_ctas_per_sm(S, (const void*)kern, 4) + pro.n_route + pro.n_request;
            orx_launch_pdl(kern, dim3(g), dim3(256), 0, st, xd, w, aa, pro, epoch);
          });
        });
        break;
      }
      case 5: {
        const int g = h->num_sms * 4;   // the grid of k_sparse_tail
        TailArgs ta = {orx_sparse_args(h, user, item, item_bias, hu, hi, od)};
        ta.counters = h->counters;   // [2]: the tail's block ticket
        ta.out4 = out4;
        sh_dispatch_opt(opt->kind, [&](auto O) {
          orx_launch_pdl(k_sh_tail<decltype(O)::value>, dim3(g), dim3(256), 0, st, xd, w, ta, par);
        });
        S->tail_epoch = epoch;
        break;
      }
    }
    ORX_LAUNCH_CHECK();
  }
  if (whole) {
    orx_prof_mark(h, 6, st);
    orx_prof_next(h);
  }
  return ORX_OK;
}
