// orx_sharded.cu -- building blocks of the row-sharded (multi-GPU) step and of un-fused sparse applies:
//   * orx_owner_bucket_combined : counting-sort the lookups of a batch by owner rank (row r lives on rank r % R,
//                        local row r / R) -> send order, per-owner counts, inverse permutation ("K9" bucket half)
//   * orx_sparse_apply : Keras OptimizerV2 sparse apply of IndexedSlices (ids[n], values[n,D]) to one table:
//                        dedup by row (batch hash), rows hit once are updated straight from their value row,
//                        duplicated rows are summed in the staging buffer and updated once by the steps' staged-row
//                        tail, k_sparse_tail ("K8").
//   * orx_bag_sparse_apply : the same for one table's multi-hot bag lookups (the bag's pooled gradient row, / its valid
//                        id count for a mean, as each valid id's value row).
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
// One warp's ROWWISE_ADAGRAD update of table row id from value row v (each element divided by nb): a row seen once in
// the batch (own, warp-uniform) takes the sum of its squared gradient first -- lane-strided in order, then the xor tree
// -- before its first store (a warp holds a row as lane * 4 ... e += 128, so D > 128 takes two passes over v); any other
// row is added into its staging row d.  vec: var moves 4 elements per lane (float4, or 8 bytes of bf16) and the value
// rows as float4 (s0[id] is one scalar).  T: the table's storage; an owned bf16 row is rounded with orx_sr_row(kt, id).
template <typename T>
__device__ __forceinline__ void orx_apply_row_rowwise(bool vec, bool own, T* var, float* s0, int id, float* gstage,
                                                      int d, int D, const float* v, float nb, const OrxOptDev& o,
                                                      uint32_t kt) {
  const int lane = threadIdx.x & 31;
  auto val4 = [&](int e) {
    const float4 g = __ldcg(reinterpret_cast<const float4*>(v + e));
    return nb == 1.f ? g : make_float4(g.x / nb, g.y / nb, g.z / nb, g.w / nb);
  };
  auto val1 = [&](int e) { return nb == 1.f ? v[e] : v[e] / nb; };
  if (!own) {
    if (vec) {
      for (int e = lane * 4; e < D; e += 128) orx_red4(gstage + (int64_t)d * D + e, val4(e));
    } else {
      for (int e = lane; e < D; e += 32) atomicAdd(gstage + (int64_t)d * D + e, val1(e));
    }
    return;
  }
  float ss = 0.f;
  if (vec) {
    for (int e = lane * 4; e < D; e += 128) ss += orx_sq4(val4(e));
  } else {
    for (int e = lane; e < D; e += 32) ss += val1(e) * val1(e);
  }
  ss = orx_group_sum<32>(ss);
  float acc = s0[id];
  const float f = orx_row_scale(acc, ss, D, o);
  T* w = var + (int64_t)id * D;
  if (vec) {
    for (int e = lane * 4; e < D; e += 128)
      orx_own_or_stage4_row<false>(true, var, id, gstage, d, D, e, orx_ld4_cg(w + e), val4(e), f, o, kt);
  } else {
    const uint32_t rk = orx_sr_row(kt, id);
    for (int e = lane; e < D; e += 32) orx_st1(w + e, orx_row_apply1(orx_ld1(w + e), val1(e), f, o), rk, e);
  }
  if (lane == 0) s0[id] = acc;
}

// VEC: var, s0 and s1 are 16-byte aligned (sparse_apply_vec decides); the row shape and the value rows are tested here,
// so that the VEC instance compiles to what the kernel was before the table gate.  Under ROWWISE_ADAGRAD only var is
// (s0 is float[rows], read as scalars).
// T: the table's storage, float or bf16 bits (uint16_t: VEC means var 8-byte aligned; an owned row is read as its exact
// fp32 upcast and stored rounded with the row key orx_sr_row(kt, id)); slots and staging rows are float either way.
template <int OPT, bool VEC, typename T = float>
__global__ void __launch_bounds__(256) k_sparse_apply(T* var, float* s0, float* s1, int64_t rows, int D,
                                                      const int32_t* __restrict__ ids, int64_t id_stride,
                                                      const float* __restrict__ vals, int64_t val_ld, int n,
                                                      OrxHash hsh, float* gstage, OrxOptDev o, uint32_t kt) {
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
// bf16 under ROWWISE_ADAGRAD: not unrolled (unrolled, 16 bytes spill around the division's slow-path call)
#pragma unroll (SL::ROW && !std::is_same<T, float>::value ? 1 : 2)
  for (int k = 0; k < 8; ++k) {
  const int b = b0 + k;
  if (b >= n) break;
  const int32_t id = __shfl_sync(ORX_FULL, my_id, k);
  const uint32_t c = __shfl_sync(ORX_FULL, my_c, k);
  const int d = __shfl_sync(ORX_FULL, my_d, k);
  if (id < 0) continue;
  const float* v = vals + (int64_t)b * val_ld;
  const bool own = !SL::STAGE_ONLY && c == 1u;
  if constexpr (SL::ROW) {
    orx_apply_row_rowwise(VEC && ((D & 3) == 0) && ((val_ld & 3) == 0) && (((uintptr_t)vals & 15) == 0), own, var, s0,
                          id, gstage, d, D, v, 1.f, o, kt);
    continue;
  } else
  // 128-bit path (value rows 16-byte aligned: a strided view may start mid-row): all loads of the row first, then the
  // math, then the stores
  if (VEC && ((D & 3) == 0) && ((val_ld & 3) == 0) && (((uintptr_t)vals & 15) == 0)) {
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e = lane * 4; e < D; e += 128) {
      const int64_t off = (int64_t)id * D + e;
      const float4 g = __ldcg(reinterpret_cast<const float4*>(v + e));
      const float4 wv = own ? orx_ld4_cg(var + off) : z4;
      float4 a = (SL::S0 && own) ? __ldcg(reinterpret_cast<const float4*>(s0 + off)) : z4;
      float4 bb = (SL::S1 && own) ? __ldcg(reinterpret_cast<const float4*>(s1 + off)) : z4;
      orx_own_or_stage4<OPT, false>(own, var, s0, s1, id, gstage, d, D, e, wv, g, a, bb, o, kt);
    }
  } else {
    const uint32_t rk = orx_sr_row(kt, id);
    for (int e = lane; e < D; e += 32) {
      const int64_t off = (int64_t)id * D + e;
      if (own) orx_update1<OPT, T>(var + off, s0 + off, s1 + off, orx_ld1(var + off), v[e], o, rk, e);
      else atomicAdd(gstage + (int64_t)d * D + e, v[e]);
    }
  }
  }
  }
}

static int sparse_apply_impl(orx_handle_t h, const orx_table_t* tab, const int32_t* ids, int64_t id_stride,
                             const float* values, int64_t value_ld, int32_t n, const orx_opt_t* opt, orx_stream_t s,
                             const uint32_t* srk = nullptr);

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

extern "C" int orx_sparse_apply_strided_bf16(orx_handle_t h, const orx_table_bf16_t* tab, const int32_t* ids,
                                             int64_t id_stride, const float* values, int64_t value_ld, int32_t n,
                                             const orx_opt_t* opt, uint64_t sr_seed, orx_stream_t s) {
  ORX_REQUIRE(tab != nullptr && id_stride >= 1 && value_ld >= tab->dim, "bad strides");
  ORX_REQUIRE(opt != nullptr, "null pointer");
  orx_table_t t;
  const uint32_t srk = orx_sr_table_key(sr_seed, opt->step, 0);
  return sparse_apply_impl(h, orx_bf16_table(tab, &t), ids, id_stride, values, value_ld, n, opt, s, &srk);
}

// The checks every un-fused sparse apply makes before any device work.
static int sparse_apply_check(orx_handle_t h, const orx_table_t* tab, int64_t n, const orx_opt_t* opt) {
  ORX_REQUIRE(h != nullptr && tab && tab->var && opt, "null pointer");
  ORX_REQUIRE(n >= 0 && tab->rows > 0 && tab->dim > 0, "bad sizes");
  ORX_REQUIRE(orx_opt_kind_ok(opt->kind), "unknown optimizer kind");
  ORX_REQUIRE(orx_opt_slots_ok(opt->kind, {tab}), "optimizer slot rows missing");
  return ORX_OK;
}

// The 4-element row path of an apply's table: a table may start anywhere (orx.h); its rows need a 16-byte (float) or
// 8-byte (bf16) boundary, its slot rows 16 bytes; a row-wise accumulator is read as scalars and does not count.
static bool sparse_apply_vec(const orx_table_t* tab, int opt_kind, bool bf16) {
  const bool rows_ok = bf16 ? orx_aligned8(tab->var) : orx_aligned16(tab->var);
  return opt_kind == ORX_OPT_ROWWISE_ADAGRAD ? rows_ok : rows_ok && orx_aligned16(tab->s0, tab->s1);
}

// The rest of an un-fused sparse apply of n lookups whose ids are ids[i * id_stride]: the batch index (mode 1 under
// ADAM_DENSE), apply(o) -- the launch that updates the rows seen once and stages the others --, the ADAM_DENSE sweeps
// and the staged-row tail.  The caller has checked the arguments and made the workspace hold n lookups.  srk: a bf16
// table (var passed as the float* of the orx_table_t) whose updates round with the table key *srk; null: a float table.
template <typename Apply>
static int sparse_apply_run(orx_handle_t h, const orx_table_t* tab, const int32_t* ids, int64_t id_stride, int32_t n,
                            const orx_opt_t* opt, cudaStream_t st, const uint32_t* srk, Apply&& apply) {
  const bool dense = opt->kind == ORX_OPT_ADAM_DENSE;
  const OrxOptDev o = orx_opt_to_dev(opt);
  int rc;
  // the user-side hash / staging pair serves as "the" table here
  if (n > 0) {
    if ((rc = orx_launch_index_build_strided(h, ids, id_stride, tab->rows, n, dense, st))) return rc;
    apply(o);
    ORX_LAUNCH_CHECK();
  }
  if (dense && (rc = orx_launch_adam_sweeps(h, tab, nullptr, nullptr, h->set[0], o, st, srk))) return rc;
  // staged rows: the shared tail with no item side and no loss
  TailArgs ta = {orx_sparse_args(h, tab, nullptr, nullptr, h->set[0], o)};
  ta.counters = h->set[0].ctl;
  if (srk) ta.srk[0] = *srk;
  return orx_launch_tail(h, ta, opt->kind, st, srk != nullptr);
}

static int sparse_apply_impl(orx_handle_t h, const orx_table_t* tab, const int32_t* ids, int64_t id_stride,
                             const float* values, int64_t value_ld, int32_t n, const orx_opt_t* opt, orx_stream_t s,
                             const uint32_t* srk) {
  int rc = sparse_apply_check(h, tab, n, opt);
  if (rc) return rc;
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  if (n == 0 && opt->kind != ORX_OPT_ADAM_DENSE) return ORX_OK;
  ORX_REQUIRE(n == 0 || (ids && values), "null ids/values");
  const int D = tab->dim;
  if ((rc = orx_ensure_workspace(h, n > 0 ? n : 1, D))) return rc;
  const orx_opt_t od = orx_opt_dim(opt, D);
  opt = &od;
  const bool vec = sparse_apply_vec(tab, od.kind, srk != nullptr);
  return sparse_apply_run(h, tab, ids, id_stride, n, opt, st, srk, [&](const OrxOptDev& o) {
    const int blocks = (n + 63) / 64;   // 8 warps x 8 pairs per block and iteration
    orx_dispatch_opt(opt->kind, [&](auto O) {
      orx_dispatch<0, 1>(vec ? 1 : 0, [&](auto V) {
        constexpr int OPT = decltype(O)::value;
        constexpr bool VEC = decltype(V)::value == 1;
        if (srk)
          k_sparse_apply<OPT, VEC, uint16_t><<<blocks, 256, 0, st>>>(
              reinterpret_cast<uint16_t*>(tab->var), tab->s0, tab->s1, tab->rows, D, ids, id_stride, values, value_ld,
              n, h->set[0].u, h->gu, o, *srk);
        else
          k_sparse_apply<OPT, VEC><<<blocks, 256, 0, st>>>(tab->var, tab->s0, tab->s1, tab->rows, D, ids, id_stride,
                                                          values, value_ld, n, h->set[0].u, h->gu, o, 0u);
      });
    });
  });
}

// ---------------------------------------------------------------------------------------
// bag-aware sparse apply (multi-hot DLRM features): lookup i = (b, l) = (i / L, i % L) of one table
// ---------------------------------------------------------------------------------------
// ids_c[b*L + l] = sparse[b*ld + col_lo + l] when it is a valid row, else -1; cnt[b] = the bag's valid ids (mean only).
// One warp per bag, 32 ids at a time.
__global__ void __launch_bounds__(256) k_bag_ids(const int32_t* __restrict__ sparse, int64_t ld, int col_lo, int L,
                                                 int B, int64_t rows, int32_t* __restrict__ ids_c,
                                                 float* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < B; b += nw) {
    int n = 0;
    for (int c = 0; c < L; c += 32) {
      int32_t id = -1;
      if (c + lane < L) {
        id = sparse[(int64_t)b * ld + col_lo + c + lane];
        if (id >= rows) id = -1;
        ids_c[(int64_t)b * L + c + lane] = id < 0 ? -1 : id;
      }
      n += __popc(__ballot_sync(ORX_FULL, id >= 0));
    }
    if (cnt && lane == 0) cnt[b] = (float)n;
  }
}

// k_sparse_apply's update over compacted bag lookups: value row i / L, divided by cnt[i / L] for a mean (cnt != null).
// A separate kernel so that k_sparse_apply's parameter block, and with it its register allocation, stays as it is.
// VEC: var, s0 and s1 are 16-byte aligned (sparse_apply_vec decides); the row shape and the value rows are tested
// here, as in k_sparse_apply.  T and kt as in k_sparse_apply.
template <int OPT, bool VEC, typename T = float>
__global__ void __launch_bounds__(256) k_bag_apply(T* var, float* s0, float* s1, int D,
                                                   const int32_t* __restrict__ ids, int L,
                                                   const float* __restrict__ vals, int64_t val_ld,
                                                   const float* __restrict__ cnt, int n, OrxHash hsh, float* gstage,
                                                   OrxOptDev o, uint32_t kt) {
  typedef OrxOptSlots<OPT> SL;
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  const bool vec = VEC && ((D & 3) == 0) && ((val_ld & 3) == 0) && (((uintptr_t)vals & 15) == 0);
  for (int b0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 8; b0 < n; b0 += nw * 8) {
  int32_t my_id = -1;
  int my_d = -1;
  uint32_t my_c = 0;
  float my_nb = 1.f;
  if (lane < 8 && b0 + lane < n) {
    my_id = ids[b0 + lane];
    if (my_id >= 0) {
      my_c = orx_hash_find(hsh, my_id, &my_d);
      if (cnt) my_nb = cnt[(b0 + lane) / L];
    }
  }
#pragma unroll 2
  for (int k = 0; k < 8; ++k) {
  const int b = b0 + k;
  if (b >= n) break;
  const int32_t id = __shfl_sync(ORX_FULL, my_id, k);
  const uint32_t c = __shfl_sync(ORX_FULL, my_c, k);
  const int d = __shfl_sync(ORX_FULL, my_d, k);
  const float nb = __shfl_sync(ORX_FULL, my_nb, k);
  if (id < 0) continue;
  const float* v = vals + (int64_t)(b / L) * val_ld;
  const bool own = !SL::STAGE_ONLY && c == 1u;
  if constexpr (SL::ROW) {
    orx_apply_row_rowwise(vec, own, var, s0, id, gstage, d, D, v, cnt ? nb : 1.f, o, kt);
    continue;
  } else
  if (vec) {
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e = lane * 4; e < D; e += 128) {
      const int64_t off = (int64_t)id * D + e;
      float4 g = __ldcg(reinterpret_cast<const float4*>(v + e));
      if (cnt) g = make_float4(g.x / nb, g.y / nb, g.z / nb, g.w / nb);
      const float4 wv = own ? orx_ld4_cg(var + off) : z4;
      float4 a = (SL::S0 && own) ? __ldcg(reinterpret_cast<const float4*>(s0 + off)) : z4;
      float4 bb = (SL::S1 && own) ? __ldcg(reinterpret_cast<const float4*>(s1 + off)) : z4;
      orx_own_or_stage4<OPT, false>(own, var, s0, s1, id, gstage, d, D, e, wv, g, a, bb, o, kt);
    }
  } else {
    const uint32_t rk = orx_sr_row(kt, id);
    for (int e = lane; e < D; e += 32) {
      const int64_t off = (int64_t)id * D + e;
      const float g = cnt ? v[e] / nb : v[e];
      if (own) orx_update1<OPT, T>(var + off, s0 + off, s1 + off, orx_ld1(var + off), g, o, rk, e);
      else atomicAdd(gstage + (int64_t)d * D + e, g);
    }
  }
  }
  }
}

// srk as in sparse_apply_run
static int bag_sparse_apply_impl(orx_handle_t h, const orx_table_t* tab, const int32_t* sparse, int64_t ld,
                                 int32_t col_lo, int32_t L, int32_t B, const float* dZ, int64_t dz_ld, int32_t mode,
                                 const orx_opt_t* opt, orx_stream_t s, const uint32_t* srk) {
  const int64_t n64 = (int64_t)B * L;
  int rc = sparse_apply_check(h, tab, B, opt);
  if (rc) return rc;
  ORX_REQUIRE(L >= 1 && col_lo >= 0 && (int64_t)col_lo + L <= ld, "bag columns outside [0, ld)");
  ORX_REQUIRE(dz_ld >= tab->dim && (mode == 0 || mode == 1), "dz_ld < dim / unknown mode");
  ORX_REQUIRE(n64 <= 0x7fffffff, "B * L > 2^31 - 1");
  ORX_REQUIRE(B == 0 || (sparse && dZ), "null sparse / dZ");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  if (B == 0 && opt->kind != ORX_OPT_ADAM_DENSE) return ORX_OK;
  const int n = (int)n64, D = tab->dim;
  if ((rc = orx_ensure_workspace(h, n > 0 ? n : 1, D))) return rc;
  int32_t* ids_c = nullptr;
  float* cnt = nullptr;
  if (n > 0) {
    OrxCarve m = {nullptr, 0};
    m.take(sizeof(int32_t) * (size_t)n);
    m.take(sizeof(float) * (size_t)B);
    if ((rc = orx_grow(&h->bag_ws, &h->bag_cap, m.off))) return rc;
    m = {static_cast<char*>(h->bag_ws), 0};
    ids_c = (int32_t*)m.take(sizeof(int32_t) * (size_t)n);
    cnt = mode == 1 ? (float*)m.take(sizeof(float) * (size_t)B) : nullptr;
    int blocks = (B + 7) / 8;
    if (blocks > h->num_sms * 32) blocks = h->num_sms * 32;
    k_bag_ids<<<blocks, 256, 0, st>>>(sparse, ld, col_lo, L, B, tab->rows, ids_c, cnt);
    ORX_LAUNCH_CHECK();
  }
  const orx_opt_t od = orx_opt_dim(opt, D);
  opt = &od;
  const bool vec = sparse_apply_vec(tab, od.kind, srk != nullptr);
  return sparse_apply_run(h, tab, ids_c, 1, n, opt, st, srk, [&](const OrxOptDev& o) {
    const int blocks = (n + 63) / 64;
    orx_dispatch_opt(opt->kind, [&](auto O) {
      orx_dispatch<0, 1>(vec ? 1 : 0, [&](auto V) {
        constexpr int OPT = decltype(O)::value;
        constexpr bool VEC = decltype(V)::value == 1;
        if (srk)
          k_bag_apply<OPT, VEC, uint16_t><<<blocks, 256, 0, st>>>(reinterpret_cast<uint16_t*>(tab->var), tab->s0,
                                                                  tab->s1, D, ids_c, L, dZ, dz_ld, cnt, n,
                                                                  h->set[0].u, h->gu, o, *srk);
        else
          k_bag_apply<OPT, VEC><<<blocks, 256, 0, st>>>(tab->var, tab->s0, tab->s1, D, ids_c, L, dZ, dz_ld, cnt, n,
                                                       h->set[0].u, h->gu, o, 0u);
      });
    });
  });
}

extern "C" int orx_bag_sparse_apply(orx_handle_t h, const orx_table_t* tab, const int32_t* sparse, int64_t ld,
                                    int32_t col_lo, int32_t L, int32_t B, const float* dZ, int64_t dz_ld, int32_t mode,
                                    const orx_opt_t* opt, orx_stream_t s) {
  return bag_sparse_apply_impl(h, tab, sparse, ld, col_lo, L, B, dZ, dz_ld, mode, opt, s, nullptr);
}

extern "C" int orx_bag_sparse_apply_bf16(orx_handle_t h, const orx_table_bf16_t* tab, const int32_t* sparse,
                                         int64_t ld, int32_t col_lo, int32_t L, int32_t B, const float* dZ,
                                         int64_t dz_ld, int32_t mode, const orx_opt_t* opt, uint64_t sr_seed,
                                         orx_stream_t s) {
  ORX_REQUIRE(opt != nullptr, "null pointer");
  orx_table_t t;
  const uint32_t srk = orx_sr_table_key(sr_seed, opt->step, 0);
  return bag_sparse_apply_impl(h, orx_bf16_table(tab, &t), sparse, ld, col_lo, L, B, dZ, dz_ld, mode, opt, s, &srk);
}
