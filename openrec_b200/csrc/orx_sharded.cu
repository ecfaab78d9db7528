// orx_sharded.cu -- building blocks of the row-sharded (multi-GPU) step and of un-fused sparse applies:
//   * orx_owner_bucket_combined : counting-sort the lookups of a batch by owner rank (row r lives on rank r % R,
//                        local row r / R) -> send order, per-owner counts, inverse permutation ("K9" bucket half)
//   * orx_sparse_apply : Keras OptimizerV2 sparse apply of IndexedSlices (ids[n], values[n,D]) to one table:
//                        dedup by row (batch hash), rows hit once are updated straight from their value row,
//                        duplicated rows are summed in the staging buffer and updated once by the steps' staged-row
//                        tail, k_sparse_tail ("K8").
// The reference has no multi-device code (SURVEY 2.1); the partitioning follows SURVEY 8(e).
#include "orx_common.cuh"

// ---------------------------------------------------------------------------------------
// owner bucketing: three tiny kernels (histogram, single-block scan, scatter)
// ---------------------------------------------------------------------------------------
__global__ void k_owner_hist(const int32_t* __restrict__ ids, int n, int R, int32_t* counts) {
  extern __shared__ int32_t sh[];
  for (int r = threadIdx.x; r < R; r += blockDim.x) sh[r] = 0;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int32_t id = ids[i];
    atomicAdd(&sh[id >= 0 ? id % R : 0], 1);
  }
  __syncthreads();
  for (int r = threadIdx.x; r < R; r += blockDim.x)
    if (sh[r]) atomicAdd(counts + r, sh[r]);
}

__global__ void k_owner_scan(const int32_t* counts, int R, int32_t* cursor) {
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int r = 0; r < R; ++r) {
      cursor[r] = acc;
      acc += counts[r];
    }
  }
}

// slot[i] = position of lookup i in the owner-sorted send order; send_local[slot] = local row on the owner.
// Positions are reserved per BLOCK (shared-memory ranks, one global atomic per block and owner): with only R
// cursors, one global atomic per lookup serialises (measured 158 us for 196k lookups at R = 2).
// Lookups i >= n_user are item lookups whose local row is offset by the owner's user-row count (U users in all).
__global__ void __launch_bounds__(256) k_owner_scatter(const int32_t* __restrict__ ids, int n, int n_user, int64_t U,
                                                       int R, int32_t* cursor, int32_t* __restrict__ send_local,
                                                       int32_t* __restrict__ slot) {
  extern __shared__ int32_t sh[];   // [R] counts then [R] bases
  int32_t* cnt = sh;
  int32_t* base = sh + R;
  for (int r = threadIdx.x; r < R; r += blockDim.x) cnt[r] = 0;
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int32_t id = -1;
  int r = 0, rank_in_block = 0;
  if (i < n) {
    id = ids[i];
    r = id >= 0 ? id % R : 0;
    rank_in_block = atomicAdd(&cnt[r], 1);
  }
  __syncthreads();
  for (int q = threadIdx.x; q < R; q += blockDim.x) base[q] = cnt[q] ? atomicAdd(cursor + q, cnt[q]) : 0;
  __syncthreads();
  if (i < n) {
    const int s = base[r] + rank_in_block;
    const int32_t user_rows_on_r = (i >= n_user) ? (int32_t)((U - r + R - 1) / R) : 0;
    send_local[s] = id >= 0 ? id / R + user_rows_on_r : -1;
    slot[i] = s;
  }
}

extern "C" int orx_owner_bucket_combined(orx_handle_t h, const int32_t* ids, int32_t n, int32_t n_user,
                                         int64_t total_users, int32_t world, int32_t* counts, int32_t* send_local,
                                         int32_t* slot, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && ids && counts && send_local && slot, "null pointer");
  ORX_REQUIRE(n >= 0 && n_user >= 0 && n_user <= n && world >= 1 && world <= 1024 && total_users > 0, "bad sizes");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  ORX_CUDA(cudaMemsetAsync(counts, 0, sizeof(int32_t) * world, st));
  if (n == 0) return ORX_OK;
  int blocks = (n + 255) / 256;
  if (blocks > h->num_sms * 4) blocks = h->num_sms * 4;
  k_owner_hist<<<blocks, 256, sizeof(int32_t) * world, st>>>(ids, n, world, counts);
  ORX_LAUNCH_CHECK();
  k_owner_scan<<<1, 32, 0, st>>>(counts, world, h->bucket_cursor);
  ORX_LAUNCH_CHECK();
  k_owner_scatter<<<(n + 255) / 256, 256, 2 * sizeof(int32_t) * world, st>>>(ids, n, n_user, total_users, world,
                                                                             h->bucket_cursor, send_local, slot);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// generic sparse apply
// ---------------------------------------------------------------------------------------
template <int OPT>
__global__ void __launch_bounds__(256) k_sparse_apply(float* var, float* s0, float* s1, int64_t rows, int D,
                                                      const int32_t* __restrict__ ids, int64_t id_stride,
                                                      const float* __restrict__ vals, int64_t val_ld, int n,
                                                      OrxHash hsh, float* gstage, OrxOptDev o) {
  typedef OrxOptSlots<OPT> SL;
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  // a warp takes 8 consecutive pairs per iteration; lanes 0..7 load the ids and probe the hash in parallel
  for (int b0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 8; b0 < n; b0 += nw * 8) {
  int32_t my_id = -1;
  int my_d = -1;
  uint32_t my_c = 0;
  if (lane < 8 && b0 + lane < n) {
    my_id = ids[(int64_t)(b0 + lane) * id_stride];
    if (my_id < 0 || (int64_t)my_id >= rows) my_id = -1;
    else my_c = orx_hash_find(hsh, my_id, &my_d);
  }
#pragma unroll 2
  for (int k = 0; k < 8; ++k) {
  const int b = b0 + k;
  if (b >= n) break;
  const int32_t id = __shfl_sync(ORX_FULL, my_id, k);
  const uint32_t c = __shfl_sync(ORX_FULL, my_c, k);
  const int d = __shfl_sync(ORX_FULL, my_d, k);
  if (id < 0) continue;
  const float* v = vals + (int64_t)b * val_ld;
  const bool own = !SL::STAGE_ONLY && c == 1u;
  if (((D & 3) == 0) && ((val_ld & 3) == 0)) {   // 128-bit path: all loads of the row first, then the math, then the stores
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e = lane * 4; e < D; e += 128) {
      const int64_t off = (int64_t)id * D + e;
      const float4 g = __ldcg(reinterpret_cast<const float4*>(v + e));
      const float4 wv = own ? __ldcg(reinterpret_cast<const float4*>(var + off)) : z4;
      float4 a = (SL::S0 && own) ? __ldcg(reinterpret_cast<const float4*>(s0 + off)) : z4;
      float4 bb = (SL::S1 && own) ? __ldcg(reinterpret_cast<const float4*>(s1 + off)) : z4;
      orx_own_or_stage4<OPT, false>(own, var, s0, s1, id, gstage, d, D, e, wv, g, a, bb, o);
    }
  } else {
    for (int e = lane; e < D; e += 32) {
      const int64_t off = (int64_t)id * D + e;
      if (own) orx_update1<OPT>(var + off, s0 + off, s1 + off, var[off], v[e], o);
      else atomicAdd(gstage + (int64_t)d * D + e, v[e]);
    }
  }
  }
  }
}

static int sparse_apply_impl(orx_handle_t h, const orx_table_t* tab, const int32_t* ids, int64_t id_stride,
                             const float* values, int64_t value_ld, int32_t n, const orx_opt_t* opt, orx_stream_t s);

extern "C" int orx_sparse_apply(orx_handle_t h, const orx_table_t* tab, const int32_t* ids, const float* values,
                                int32_t n, const orx_opt_t* opt, orx_stream_t s) {
  ORX_REQUIRE(tab != nullptr, "null table");
  return sparse_apply_impl(h, tab, ids, 1, values, tab->dim, n, opt, s);
}

extern "C" int orx_sparse_apply_strided(orx_handle_t h, const orx_table_t* tab, const int32_t* ids, int64_t id_stride,
                                        const float* values, int64_t value_ld, int32_t n, const orx_opt_t* opt,
                                        orx_stream_t s) {
  ORX_REQUIRE(tab != nullptr && id_stride >= 1 && value_ld >= tab->dim, "bad strides");
  return sparse_apply_impl(h, tab, ids, id_stride, values, value_ld, n, opt, s);
}

static int sparse_apply_impl(orx_handle_t h, const orx_table_t* tab, const int32_t* ids, int64_t id_stride,
                             const float* values, int64_t value_ld, int32_t n, const orx_opt_t* opt, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && tab && tab->var && opt, "null pointer");
  ORX_REQUIRE(n >= 0 && tab->rows > 0 && tab->dim > 0, "bad sizes");
  ORX_REQUIRE(orx_opt_kind_ok(opt->kind), "unknown optimizer kind");
  ORX_REQUIRE(orx_opt_slots_ok(opt->kind, {tab}), "optimizer slot rows missing");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  const bool dense = opt->kind == ORX_OPT_ADAM_DENSE;
  if (n == 0 && !dense) return ORX_OK;
  ORX_REQUIRE(n == 0 || (ids && values), "null ids/values");
  const int D = tab->dim;
  int rc = orx_ensure_workspace(h, n > 0 ? n : 1, D);
  if (rc) return rc;
  const OrxOptDev o = orx_opt_to_dev(opt);
  // the user-side hash / staging pair serves as "the" table here
  if (n > 0) {
    if ((rc = orx_launch_index_build_strided(h, ids, id_stride, tab->rows, n, dense, st))) return rc;
    const int blocks = (n + 63) / 64;   // 8 warps x 8 pairs per block and iteration
    orx_dispatch_opt(opt->kind, [&](auto O) {
      k_sparse_apply<decltype(O)::value><<<blocks, 256, 0, st>>>(tab->var, tab->s0, tab->s1, tab->rows, D, ids, id_stride,
                                                                 values, value_ld, n, h->hu, h->gu, o);
    });
    ORX_LAUNCH_CHECK();
  }
  if (dense && (rc = orx_launch_adam_sweeps(h, tab, nullptr, nullptr, h->hu, h->hi, o, st))) return rc;
  // staged rows: the shared tail with no item side and no loss
  TailArgs ta = {orx_sparse_args(h, tab, nullptr, nullptr, h->hu, h->hi, o)};
  ta.counters = h->counters;
  return orx_launch_tail(h, ta, opt->kind, st);
}
