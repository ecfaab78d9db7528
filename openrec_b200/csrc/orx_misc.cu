// orx_misc.cu -- LatentFactor init / gather / censor, dense optimizer apply, full-catalogue scoring,
// ranking metrics.
#include "orx_common.cuh"

// ---------------------------------------------------------------------------------------
// LatentFactor.__init__ initializer (latent_factor.py:8-15): U(lo,hi) from a counter-based hash
// (TF's RNG stream is not reproducible across frameworks; only the distribution matters).
// lo + (hi - lo) * u can round up to hi for u < 1 (e.g. [1, 2) at u = 1 - 2^-24): such a value is clamped to the
// largest float below hi, so the range stays half-open.  Values below hi keep their bits.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__global__ void k_fill_uniform(float* dst, int64_t n, float lo, float hi, uint64_t seed) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float top = nextafterf(hi, lo);   // largest float below hi
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint64_t r = splitmix64(seed * 0xD1342543DE82EF95ull + (uint64_t)i);
    const float u = (float)(r >> 40) * (1.0f / 16777216.0f);  // [0,1)
    dst[i] = fminf(lo + (hi - lo) * u, top);
  }
}

extern "C" int orx_fill_uniform(orx_handle_t h, float* dst, int64_t n, float lo, float hi, uint64_t seed,
                                orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && dst != nullptr && n >= 0, "null handle/dst or negative n");
  if (n == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  int64_t blocks = (n + 1023) / 1024;
  if (blocks > (int64_t)h->num_sms * 16) blocks = (int64_t)h->num_sms * 16;
  k_fill_uniform<<<(int)blocks, 256, 0, (cudaStream_t)s>>>(dst, n, lo, hi, seed);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// LatentFactor.__call__ (Embedding.call): out[b,:] = tab[ids[b],:]
// ---------------------------------------------------------------------------------------
// VEC: tab and out are 16-byte aligned (orx_gather decides); with D % 4 == 0 the rows then move as float4.  The row
// shape is tested here, so that the VEC instance compiles to what the kernel was before the pointer gate.
template <typename IdT, bool VEC>
__global__ void __launch_bounds__(256) k_gather(const float* __restrict__ tab, int64_t rows, int D,
                                                const IdT* __restrict__ ids, int64_t n, float* __restrict__ out,
                                                int32_t* n_bad) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const bool vec = VEC && (D & 3) == 0;
  for (int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n; b += nw) {
    const int64_t id = (int64_t)ids[b];
    const bool ok = id >= 0 && id < rows;
    if (!ok && lane == 0 && n_bad) atomicAdd(n_bad, 1);
    if (vec) {
      const float4* src = reinterpret_cast<const float4*>(tab + id * D);
      float4* dst = reinterpret_cast<float4*>(out + b * D);
      for (int e = lane; e < D / 4; e += 32) dst[e] = ok ? __ldg(src + e) : make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      for (int e = lane; e < D; e += 32) out[b * D + e] = ok ? __ldg(tab + id * D + e) : 0.f;
    }
  }
}

extern "C" int orx_gather(orx_handle_t h, const float* tab, int64_t rows, int32_t dim, const void* ids,
                          int32_t id_is_i64, int64_t n, float* out, int32_t* n_bad, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && tab, "null pointer");
  ORX_REQUIRE(rows > 0 && dim > 0 && n >= 0, "bad sizes");
  if (n == 0) return ORX_OK;                   // an empty lookup: ids and out may be NULL (empty tensors)
  ORX_REQUIRE(ids && out, "null pointer");
  ORX_CUDA(cudaSetDevice(h->device));
  int64_t blocks = (n + 7) / 8;
  if (blocks > (int64_t)h->num_sms * 32) blocks = (int64_t)h->num_sms * 32;
  orx_dispatch<0, 1>(orx_aligned16(tab, out) ? 1 : 0, [&](auto V) {
    constexpr bool VEC = decltype(V)::value == 1;
    cudaStream_t st = (cudaStream_t)s;
    if (id_is_i64) k_gather<int64_t, VEC><<<(int)blocks, 256, 0, st>>>(tab, rows, dim, (const int64_t*)ids, n, out, n_bad);
    else k_gather<int32_t, VEC><<<(int)blocks, 256, 0, st>>>(tab, rows, dim, (const int32_t*)ids, n, out, n_bad);
  });
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// LatentFactor.censor (latent_factor.py:17-23), "K10": unique ids via the batch hash (the first
// warp to insert an id owns the row), row <- row / max(||row||, min_norm).
// ---------------------------------------------------------------------------------------
// The censor of up to 8 rows of one warp: lane k < 8 holds row k in my_id (-1: none; other lanes' values are not read).
// VEC (tab 16-byte aligned, decided by the launcher) && D % 4 == 0 && D <= 128: one float4 per lane, all 8 rows loaded
// before the first norm is reduced; otherwise one row at a time, lane-strided.  Every lane of the warp calls it.  (The
// row shape is tested here rather than passed in: so k_censor<true> compiles to the same SASS as k_censor did before
// the function was factored out of it.)
// T = uint16_t: a bf16 table, scalar path only (VEC false), each result stored rounded to nearest even.
template <bool VEC, typename T = float>
__device__ __forceinline__ void orx_censor_rows8(T* tab, int D, int32_t my_id, float min_norm) {
  const int lane = threadIdx.x & 31;
  if (VEC && (D & 3) == 0 && D <= 128) {
    const int nq = D >> 2;
    float4 v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int32_t id = __shfl_sync(ORX_FULL, my_id, k);
      v[k] = (id >= 0 && lane < nq) ? __ldcg(reinterpret_cast<const float4*>(tab + (int64_t)id * D) + lane)
                                    : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int32_t id = __shfl_sync(ORX_FULL, my_id, k);
      if (id < 0) continue;
      float sq = v[k].x * v[k].x + v[k].y * v[k].y + v[k].z * v[k].z + v[k].w * v[k].w;
      sq = orx_group_sum<32>(sq);
      const float den = fmaxf(sqrtf(sq), min_norm);
      if (lane < nq)
        __stcg(reinterpret_cast<float4*>(tab + (int64_t)id * D) + lane,
               make_float4(v[k].x / den, v[k].y / den, v[k].z / den, v[k].w / den));
    }
  } else {
    for (int k = 0; k < 8; ++k) {
      const int32_t id = __shfl_sync(ORX_FULL, my_id, k);
      if (id < 0) continue;
      T* row = tab + (int64_t)id * D;
      float sq = 0.f;
      for (int e = lane; e < D; e += 32) sq += orx_ld1(row + e) * orx_ld1(row + e);
      sq = orx_group_sum<32>(sq);
      const float den = fmaxf(sqrtf(sq), min_norm);
      for (int e = lane; e < D; e += 32) {
        if constexpr (std::is_same<T, float>::value) row[e] = row[e] / den;
        else row[e] = (uint16_t)orx_bf16_rne(orx_ld1(row + e) / den);
      }
    }
  }
}

// A warp takes 8 ids per iteration: lanes 0..7 load the ids and claim the rows in the hash in parallel, then (128-bit path)
// all 8 rows are loaded before the first norm is reduced -- one row per warp left the kernel latency-bound (id -> hash ->
// row -> reduce -> divide -> store: 23 us for 65 536 ids at D = 128, three of them per UCML step).
template <bool VEC, typename T = float>
__global__ void __launch_bounds__(256) k_censor(T* tab, int64_t rows, int D, const int32_t* __restrict__ ids,
                                                int n, float min_norm, OrxHash hsh) {
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int b0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 8; b0 < n; b0 += nw * 8) {
    int32_t my_id = -1;
    if (lane < 8 && b0 + lane < n) {
      const int32_t id = ids[b0 + lane];
      if (id >= 0 && (int64_t)id < rows && orx_hash_insert(hsh, id, 2) == 0u) my_id = id;   // first claim owns the row
    }
    orx_censor_rows8<VEC, T>(tab, D, my_id, min_norm);
  }
}

// LatentFactor.censor on a row-sharded table: this rank censors the ids it owns (id % world == rank, local row
// id / world) among n GLOBAL ids laid out in blocks of n_per_block, block b at ids + b * block_stride (an all-gather of
// every rank's ids).  Only about one id in `world` is owned, so a warp reads `chunk` = min(32, 8 world) consecutive ids
// at once (coalesced; about 8 owned ones, and k_censor's 8 ids per warp at world 1), the owned lanes claim their local
// row in the dedup hash, and the first claims are compacted into a per-warp queue; every 8 queued rows, and once at the
// end, go through orx_censor_rows8, the arithmetic of k_censor.
template <bool VEC>
__global__ void __launch_bounds__(256) k_censor_shard(float* tab, int D, int64_t total_rows, int world, int rank,
                                                      const int32_t* __restrict__ ids, int n_per_block,
                                                      int64_t block_stride, int n, int chunk, float min_norm,
                                                      OrxHash hsh) {
  __shared__ int32_t queue[8][40];   // < 8 rows left over + up to 32 new claims
  int32_t* q = queue[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  int qn = 0;
  for (int t0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * chunk; t0 < n; t0 += nw * chunk) {
    const int t = t0 + lane;
    int32_t row = -1;
    if (lane < chunk && t < n) {
      const int32_t id = ids[(int64_t)(t / n_per_block) * block_stride + t % n_per_block];
      if (id >= 0 && (int64_t)id < total_rows && id % world == rank && orx_hash_insert(hsh, id / world, 2) == 0u)
        row = id / world;                                                          // first claim owns the row
    }
    const unsigned claim = __ballot_sync(ORX_FULL, row >= 0);
    if (row >= 0) q[qn + __popc(claim & ((1u << lane) - 1u))] = row;
    __syncwarp();
    const int queued = qn + __popc(claim);
    int head = 0;
    for (; queued - head >= 8; head += 8) orx_censor_rows8<VEC>(tab, D, lane < 8 ? q[head + lane] : -1, min_norm);
    const int32_t rest = lane < queued - head ? q[head + lane] : -1;   // the < 8 rows left move to the queue's front
    __syncwarp();
    if (lane < queued - head) q[lane] = rest;
    __syncwarp();
    qn = queued - head;
  }
  if (qn > 0) orx_censor_rows8<VEC>(tab, D, lane < qn ? q[lane] : -1, min_norm);
}


// T = uint16_t: orx_censor_bf16
template <typename T>
static int censor_impl(orx_handle_t h, T* tab, int64_t rows, int32_t dim, const int32_t* ids, int32_t n,
                       float min_norm, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && tab && ids, "null pointer");
  ORX_REQUIRE(rows > 0 && dim > 0 && n >= 0, "bad sizes");
  if (n == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  int rc = orx_ensure_workspace(h, n, h->g_dim > 0 ? h->g_dim : 1);
  if (rc) return rc;
  OrxIndexSet& ix = h->set[0];
  if ((rc = orx_take_epoch(ix.u, st))) return rc;   // the dedup hash needs no clearing: a new epoch empties it
  int blocks = (n + 63) / 64;                 // 8 warps x 8 ids per block and iteration
  if (blocks > h->num_sms * 8) blocks = h->num_sms * 8;
  if constexpr (std::is_same<T, uint16_t>::value) k_censor<false, T><<<blocks, 256, 0, st>>>(tab, rows, dim, ids, n, min_norm, ix.u);
  else if (orx_aligned16(tab)) k_censor<true><<<blocks, 256, 0, st>>>(tab, rows, dim, ids, n, min_norm, ix.u);
  else k_censor<false><<<blocks, 256, 0, st>>>(tab, rows, dim, ids, n, min_norm, ix.u);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

extern "C" int orx_censor(orx_handle_t h, float* tab, int64_t rows, int32_t dim, const int32_t* ids, int32_t n,
                          float min_norm, orx_stream_t s) {
  return censor_impl(h, tab, rows, dim, ids, n, min_norm, s);
}

extern "C" int orx_censor_bf16(orx_handle_t h, uint16_t* tab, int64_t rows, int32_t dim, const int32_t* ids, int32_t n,
                               float min_norm, orx_stream_t s) {
  return censor_impl(h, tab, rows, dim, ids, n, min_norm, s);
}

// The dedup hash of orx_censor_shard is the handle's censor_ws: slots only (mode-2 inserts stage nothing), as many as
// orx_hash_shape gives for the largest call so far, all of them in use (so the epoch wrap's clear covers every slot that
// may hold an old epoch).  It grows on the caller's stream; its epoch carries over, a zeroed slot being empty in any.
static int censor_hash_for(orx_ctx* c, int64_t lookups, cudaStream_t st) {
  OrxHash shape;
  const uint32_t cap = orx_hash_shape(shape, lookups);
  OrxCarve m = {nullptr, 0};
  m.take(sizeof(unsigned long long) * cap);
  if (m.off <= c->censor_cap) return ORX_OK;
  c->censor_hash.slots = nullptr;
  int rc = orx_grow(&c->censor_ws, &c->censor_cap, m.off);
  if (rc) return rc;
  m = {static_cast<char*>(c->censor_ws), 0};
  c->censor_hash.slots = (unsigned long long*)m.take(sizeof(unsigned long long) * cap);
  c->censor_hash.mask = shape.mask;
  c->censor_hash.shift = shape.shift;
  ORX_CUDA(cudaMemsetAsync(c->censor_ws, 0, c->censor_cap, st));
  return ORX_OK;
}

extern "C" int orx_censor_shard(orx_handle_t h, float* tab, int64_t local_rows, int32_t dim, int64_t total_rows,
                                int32_t world, int32_t rank, const int32_t* ids, int32_t n_per_block,
                                int64_t block_stride, int32_t n_blocks, float min_norm, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(world >= 1 && rank >= 0 && rank < world, "need world >= 1 and 0 <= rank < world");
  ORX_REQUIRE(dim > 0 && total_rows >= 0 && local_rows >= 0 && n_per_block >= 0 && n_blocks >= 0, "bad sizes");
  const int64_t owned = total_rows > rank ? (total_rows - rank + world - 1) / world : 0;
  ORX_REQUIRE(local_rows >= owned, "local_rows is below the number of rows this rank owns");
  ORX_REQUIRE(n_blocks <= 1 || block_stride >= n_per_block, "blocks overlap (block_stride < n_per_block)");
  const int64_t n = (int64_t)n_per_block * n_blocks;
  ORX_REQUIRE(n <= ORX_CENSOR_SHARD_MAX_IDS, "more than ORX_CENSOR_SHARD_MAX_IDS ids in one call");
  ORX_REQUIRE((n == 0 || ids) && (owned == 0 || tab), "null pointer");
  const bool aligned = orx_aligned16(tab);
  const bool vec = aligned && (dim & 3) == 0 && dim <= 128;   // orx_censor_rows8's 128-bit path
  orx_log_dispatch(h, ORX_OP_CENSOR_SHARD, vec ? ORX_VARIANT_CENSOR_VEC : ORX_VARIANT_CENSOR_SCALAR, rank, 0, (int)n,
                   (int)(local_rows < INT32_MAX ? local_rows : INT32_MAX), dim, world);
  if (n == 0 || owned == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  int rc = censor_hash_for(h, n, st);
  if (rc) return rc;
  if ((rc = orx_take_epoch(h->censor_hash, st))) return rc;
  const int chunk = world >= 4 ? 32 : 8 * world;   // ids per warp and iteration: about 8 of them owned
  int64_t blocks = (n + 8 * chunk - 1) / (8 * chunk);
  if (blocks > (int64_t)h->num_sms * 8) blocks = (int64_t)h->num_sms * 8;
  orx_dispatch<0, 1>(aligned ? 1 : 0, [&](auto V) {
    k_censor_shard<decltype(V)::value == 1><<<(int)blocks, 256, 0, st>>>(
        tab, dim, total_rows, world, rank, ids, n_per_block, block_stride, (int)n, chunk, min_norm, h->censor_hash);
  });
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// Keras dense apply for dense variables (GMF w, MLP kernels / biases)
// ---------------------------------------------------------------------------------------
template <int OPT>
__global__ void k_dense_apply(float* var, float* s0, float* s1, const float* __restrict__ grad, int64_t n,
                              OrxOptDev o) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    orx_update1<OPT>(var + i, s0 + i, s1 + i, var[i], grad[i], o);
}

extern "C" int orx_dense_apply(orx_handle_t h, float* var, float* s0, float* s1, const float* grad, int64_t n,
                               const orx_opt_t* opt, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && var && grad && opt, "null pointer");
  ORX_REQUIRE(n >= 0, "negative n");
  if (n == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  const OrxOptDev o = orx_opt_to_dev(opt);
  int64_t blocks = (n + 255) / 256;
  if (blocks > (int64_t)h->num_sms * 16) blocks = (int64_t)h->num_sms * 16;
  cudaStream_t st = (cudaStream_t)s;
  ORX_REQUIRE(orx_opt_kind_ok(opt->kind), "unknown optimizer kind");
  const orx_table_t t = {var, s0, s1, n, 1};
  ORX_REQUIRE(orx_opt_slots_ok(opt->kind, {&t}), "optimizer slot rows missing");
  // ADAM_DENSE runs as ADAM_LAZY: identical on a dense variable; ROWWISE_ADAGRAD as ADAGRAD: a dense variable keeps an
  // element-wise accumulator (orx.h); NESTEROV as MOMENTUM, which reads the form from o.kind
  const int kind = opt->kind == ORX_OPT_ADAM_DENSE ? ORX_OPT_ADAM_LAZY
                   : opt->kind == ORX_OPT_ROWWISE_ADAGRAD ? ORX_OPT_ADAGRAD
                   : opt->kind == ORX_OPT_NESTEROV ? ORX_OPT_MOMENTUM : opt->kind;
  orx_dispatch<ORX_OPT_SGD, ORX_OPT_ADAGRAD, ORX_OPT_ADAM_LAZY, ORX_OPT_MOMENTUM>(kind, [&](auto O) {
    k_dense_apply<decltype(O)::value><<<(int)blocks, 256, 0, st>>>(var, s0, s1, grad, n, o);
  });
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// inference: scores[Bu, I]  (bpr.py:39-43, wrmf.py:36-40, ucml.py:50-53, gmf.py:36-41), "K11".
// 64 users x 64 items per block, D consumed in chunks of 16 through shared memory; 4x4 per thread.  Tab: the tables'
// storage, float or bf16 bits widened exactly by orx_ld1 (orx_score_all_bf16); scale, bias and scores are fp32.
// ---------------------------------------------------------------------------------------
template <int KIND, typename Tab>
__global__ void __launch_bounds__(256) k_score_all(const Tab* __restrict__ user_tab, int64_t U,
                                                   const int32_t* __restrict__ uid, int Bu,
                                                   const float* __restrict__ scale, const Tab* __restrict__ item_tab,
                                                   const float* __restrict__ bias, int64_t I, int D,
                                                   float* __restrict__ scores) {
  constexpr int T = 64, KC = 16;
  __shared__ float su[KC][T + 1], si[KC][T + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t i0 = (int64_t)blockIdx.x * T;
  const int u0 = blockIdx.y * T;
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
  for (int k0 = 0; k0 < D; k0 += KC) {
    for (int e = threadIdx.x; e < T * KC; e += 256) {
      const int r = e / KC, k = e % KC;
      float uv = 0.f, iv = 0.f;
      if (k0 + k < D) {
        if (u0 + r < Bu) {
          const int32_t id = uid[u0 + r];
          if (id >= 0 && (int64_t)id < U) {
            uv = orx_ld1(user_tab + (int64_t)id * D + k0 + k);
            if (scale) uv *= scale[k0 + k];
          }
        }
        if (i0 + r < I) iv = orx_ld1(item_tab + (i0 + r) * D + k0 + k);
      }
      su[k][r] = uv;
      si[k][r] = iv;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      if (k0 + k < D) {
        float uu[4], ii[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) uu[a] = su[k][ty * 4 + a];
#pragma unroll
        for (int b = 0; b < 4; ++b) ii[b] = si[k][tx + 16 * b];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            if (KIND == ORX_SCORE_DOT) acc[a][b] += uu[a] * ii[b];
            else acc[a][b] -= (uu[a] - ii[b]) * (uu[a] - ii[b]);
          }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int u = u0 + ty * 4 + a;
    if (u >= Bu) continue;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int64_t i = i0 + tx + 16 * b;
      if (i < I) scores[(int64_t)u * I + i] = acc[a][b] + (bias ? bias[i] : 0.f);
    }
  }
}

template <typename T>
static int score_all_impl(orx_handle_t h, int32_t kind, const T* user_tab, int64_t U, const int32_t* uid, int32_t Bu,
                          const float* scale, const T* item_tab, const float* item_bias, int64_t I, int32_t dim,
                          float* scores, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && user_tab && uid && item_tab && scores, "null pointer");
  ORX_REQUIRE(kind == ORX_SCORE_DOT || kind == ORX_SCORE_NEG_SQDIST, "unknown score kind");
  ORX_REQUIRE(U > 0 && I > 0 && dim > 0 && Bu >= 0, "bad sizes");
  if (Bu == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  dim3 grid((unsigned)((I + 63) / 64), (unsigned)((Bu + 63) / 64));
  cudaStream_t st = (cudaStream_t)s;
  if (kind == ORX_SCORE_DOT)
    k_score_all<ORX_SCORE_DOT><<<grid, 256, 0, st>>>(user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, scores);
  else
    k_score_all<ORX_SCORE_NEG_SQDIST><<<grid, 256, 0, st>>>(user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim,
                                                            scores);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

extern "C" int orx_score_all(orx_handle_t h, int32_t kind, const float* user_tab, int64_t U, const int32_t* uid,
                             int32_t Bu, const float* scale, const float* item_tab, const float* item_bias, int64_t I,
                             int32_t dim, float* scores, orx_stream_t s) {
  return score_all_impl(h, kind, user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, scores, s);
}

extern "C" int orx_score_all_bf16(orx_handle_t h, int32_t kind, const uint16_t* user_tab, int64_t U, const int32_t* uid,
                                  int32_t Bu, const float* scale, const uint16_t* item_tab, const float* item_bias,
                                  int64_t I, int32_t dim, float* scores, orx_stream_t s) {
  return score_all_impl(h, kind, user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, scores, s);
}

// ---------------------------------------------------------------------------------------
// ranking metrics (openrec/tf2/metrics/ranking_metrics.py:8-69), one block per user row.
//   AUC    = #{(e,p): pred_e <= pred_p, e in eval, p in pos} / (n_pos*n_eval),  eval = !(pos|excl)
//   s      = exp(pred) * !excl ;  rank_p = #{i: s_i > s_p}
//   NDCG@k = sum_p [rank_p<k] / log2(rank_p+2)   (no ideal-DCG normaliser, SURVEY Q10)
//   Recall@k = #{p: rank_p<k} / n_pos
// ---------------------------------------------------------------------------------------
#define ORX_MAX_AT 8
struct RankArgs {
  const float* pred;
  const uint8_t *pos, *excl;
  int R;
  int64_t I;
  int at[ORX_MAX_AT];
  int n_at;
  float *auc, *ndcg, *recall;
};

__global__ void __launch_bounds__(256) k_rank_metrics(const RankArgs a) {
  constexpr int TILE = 1024;
  __shared__ int s_idx[TILE];
  __shared__ int s_n, s_npos, s_neval;
  __shared__ unsigned long long s_auc;
  __shared__ double s_dcg[ORX_MAX_AT];
  __shared__ int s_hit[ORX_MAX_AT];
  const int r = blockIdx.x;
  const float* pred = a.pred + (int64_t)r * a.I;
  const uint8_t* pos = a.pos + (int64_t)r * a.I;
  const uint8_t* excl = a.excl + (int64_t)r * a.I;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  if (threadIdx.x == 0) {
    s_npos = 0;
    s_neval = 0;
    s_auc = 0ull;
  }
  if (threadIdx.x < ORX_MAX_AT) {
    s_dcg[threadIdx.x] = 0.0;
    s_hit[threadIdx.x] = 0;
  }
  __syncthreads();
  int np = 0, ne = 0;
  for (int64_t i = threadIdx.x; i < a.I; i += blockDim.x) {
    np += pos[i] ? 1 : 0;
    ne += (pos[i] || excl[i]) ? 0 : 1;
  }
  atomicAdd(&s_npos, np);
  atomicAdd(&s_neval, ne);
  for (int64_t t0 = 0; t0 < a.I; t0 += TILE) {
    __syncthreads();
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int64_t i = t0 + threadIdx.x; i < t0 + TILE && i < a.I; i += blockDim.x)
      if (pos[i]) s_idx[atomicAdd(&s_n, 1)] = (int)i;
    __syncthreads();
    for (int q = warp; q < s_n; q += nwarp) {
      const int p = s_idx[q];
      const float pp = pred[p];
      const float sp = expf(pp) * (excl[p] ? 0.f : 1.f);
      unsigned int c_auc = 0, c_rank = 0;
      for (int64_t i = lane; i < a.I; i += 32) {
        const float pi = pred[i];
        const bool ex = excl[i] != 0;
        if (!(pos[i] || ex) && pi <= pp) ++c_auc;
        const float si = expf(pi) * (ex ? 0.f : 1.f);
        if (si > sp) ++c_rank;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        c_auc += __shfl_xor_sync(ORX_FULL, c_auc, o);
        c_rank += __shfl_xor_sync(ORX_FULL, c_rank, o);
      }
      if (lane == 0) {
        atomicAdd(&s_auc, (unsigned long long)c_auc);
        const float ra = (float)c_rank;
        const float rec = 1.f / (logf(ra + 2.f) / logf(2.0f));
        for (int k = 0; k < a.n_at; ++k)
          if (ra < (float)a.at[k]) {
            atomicAdd(&s_dcg[k], (double)rec);
            atomicAdd(&s_hit[k], 1);
          }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && a.auc) a.auc[r] = (float)s_auc / (float)((long long)s_npos * (long long)s_neval);
  if (threadIdx.x < a.n_at) {
    if (a.ndcg) a.ndcg[(int64_t)r * a.n_at + threadIdx.x] = (float)s_dcg[threadIdx.x];
    if (a.recall) a.recall[(int64_t)r * a.n_at + threadIdx.x] = (float)s_hit[threadIdx.x] / (float)s_npos;
  }
}

extern "C" int orx_rank_metrics(orx_handle_t h, const float* pred, const uint8_t* pos, const uint8_t* excl, int32_t R,
                                int64_t I, const int32_t* at_host, int32_t n_at, float* auc, float* ndcg,
                                float* recall, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && pred && pos && excl, "null pointer");
  ORX_REQUIRE(R >= 0 && I > 0 && n_at >= 0 && n_at <= ORX_MAX_AT, "bad sizes (at most 8 cut-offs)");
  ORX_REQUIRE(n_at == 0 || at_host, "null cut-offs");
  if (R == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  RankArgs a;
  a.pred = pred; a.pos = pos; a.excl = excl; a.R = R; a.I = I; a.n_at = n_at;
  for (int k = 0; k < ORX_MAX_AT; ++k) a.at[k] = k < n_at ? at_host[k] : 0;
  a.auc = auc; a.ndcg = ndcg; a.recall = recall;
  k_rank_metrics<<<R, 256, 0, (cudaStream_t)s>>>(a);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}
