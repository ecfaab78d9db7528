// orx_dlrm_shard.cu -- the two kernels of the row-sharded DLRM step (openrec_b200/sharded.py, ShardedDLRMStep):
//   * orx_lookup_bucket    : the [B, T] id batch -> its unique valid global rows in (owner, local row) order, per-owner
//                            counts, each lookup's index in that order and each unique row's lookups (a CSR)
//   * orx_rows_segment_sum : the per-lookup embedding gradient rows folded onto those unique rows, in a fixed order
// The T tables are one concatenated row space: global row g = row_off[k] + id lives on rank g % R at local row g / R.
// Deduplicating before the exchange is what keeps small, hot tables cheap: a feature with vocabulary 3 sends 3 rows per
// step instead of one per sample.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "orx_common.cuh"

namespace {

struct LookupWs {
  int64_t* row_off;     // [T + 1]
  uint32_t* keys_in;    // [n] owner * L + local row, or the invalid key R * L
  uint32_t* keys;       // [n] sorted
  int32_t* iota;        // [n] lookup indices, then the head flags of the sorted keys
  int32_t* incl;        // [n] inclusive scan of the head flags: 1 + the send-order index of a valid position
  int32_t* ostart;      // [R + 1] send-order index of each owner's first unique row
  void* tmp;            // CUB storage of the sort and of the scan
  size_t tmp_bytes;
};

size_t lookup_layout(char* base, int64_t n, int T, int R, size_t tmp_bytes, LookupWs* w) {
  OrxCarve m = {base, 0};
  w->row_off = reinterpret_cast<int64_t*>(m.take(sizeof(int64_t) * (size_t)(T + 1)));
  w->keys_in = reinterpret_cast<uint32_t*>(m.take(sizeof(uint32_t) * (size_t)n));
  w->keys = reinterpret_cast<uint32_t*>(m.take(sizeof(uint32_t) * (size_t)n));
  w->iota = reinterpret_cast<int32_t*>(m.take(sizeof(int32_t) * (size_t)n));
  w->incl = reinterpret_cast<int32_t*>(m.take(sizeof(int32_t) * (size_t)n));
  w->ostart = reinterpret_cast<int32_t*>(m.take(sizeof(int32_t) * (size_t)(R + 1)));
  w->tmp = m.take(tmp_bytes);
  w->tmp_bytes = tmp_bytes;
  return m.off;
}

}  // namespace

// key of lookup i = b * T + k: a valid id maps to owner * L + local row (L = ceil(G / R) local rows at most per rank), so
// the keys sort by owner, then by local row; an invalid id gets R * L, past every valid key
__global__ void __launch_bounds__(256) k_lb_keys(const int32_t* __restrict__ sparse, int64_t n, int T,
                                                 const int64_t* __restrict__ row_off, int R, uint32_t L,
                                                 uint32_t* __restrict__ keys, int32_t* __restrict__ iota) {
  const uint32_t invalid = (uint32_t)R * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % T);
    const int32_t id = sparse[i];
    const int64_t lo = row_off[k];
    uint32_t key = invalid;
    if (id >= 0 && lo + id < row_off[k + 1]) {
      const int64_t g = lo + id;
      key = (uint32_t)(g % R) * L + (uint32_t)(g / R);
    }
    keys[i] = key;
    iota[i] = (int32_t)i;
  }
}

// head flag of sorted position p: the first position of a valid key
__global__ void __launch_bounds__(256) k_lb_heads(const uint32_t* __restrict__ keys, int64_t n, uint32_t invalid,
                                                  int32_t* __restrict__ head) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t key = keys[p];
    head[p] = key != invalid && (p == 0 || keys[p - 1] != key) ? 1 : 0;
  }
}

// slot, grp_off, send_local and the owners' first unique rows from the sorted keys and the scanned heads
__global__ void __launch_bounds__(256) k_lb_scatter(const uint32_t* __restrict__ keys, const int32_t* __restrict__ idx,
                                                    const int32_t* __restrict__ incl, int64_t n, int R, uint32_t L,
                                                    int32_t* __restrict__ slot, int32_t* __restrict__ grp_off,
                                                    int32_t* __restrict__ send_local, int32_t* __restrict__ ostart) {
  const uint32_t invalid = (uint32_t)R * L;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t key = keys[p];
    const bool prev_valid = p > 0 && keys[p - 1] != invalid;
    if (key == invalid) {
      slot[idx[p]] = -1;
      if (p == 0 || prev_valid) {              // the first invalid position: p valid lookups before it
        grp_off[p == 0 ? 0 : incl[p - 1]] = (int32_t)p;
        for (int q = p == 0 ? 0 : (int)(keys[p - 1] / L) + 1; q <= R; ++q) ostart[q] = p == 0 ? 0 : incl[p - 1];
      }
      continue;
    }
    const int32_t j = incl[p] - 1;
    slot[idx[p]] = j;
    const int owner = (int)(key / L);
    if (!prev_valid || keys[p - 1] != key) {   // head of unique row j
      grp_off[j] = (int32_t)p;
      send_local[j] = (int32_t)(key - (uint32_t)owner * L);
      const int prev_owner = prev_valid ? (int)(keys[p - 1] / L) : -1;
      for (int q = prev_owner + 1; q <= owner; ++q) ostart[q] = j;
    }
    if (p == n - 1) {                          // every lookup valid: close the last segment and the owner list
      grp_off[j + 1] = (int32_t)n;
      for (int q = owner + 1; q <= R; ++q) ostart[q] = j + 1;
    }
  }
}

__global__ void k_lb_counts(const int32_t* __restrict__ ostart, int R, int32_t* __restrict__ counts) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < R; r += gridDim.x * blockDim.x)
    counts[r] = ostart[r + 1] - ostart[r];
}

extern "C" int orx_lookup_bucket(orx_handle_t h, const int32_t* sparse, int32_t B, int32_t T, const int64_t* row_off_host,
                                 int32_t world, int32_t* counts, int32_t* send_local, int32_t* slot, int32_t* grp_off,
                                 int32_t* grp_idx, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && row_off_host && counts && grp_off, "null pointer");
  ORX_REQUIRE(B >= 0 && T >= 1 && world >= 1 && world <= 1024, "bad sizes");
  ORX_REQUIRE((int64_t)B * T <= INT32_MAX, "B * T exceeds 2^31 - 1 lookups");
  ORX_REQUIRE(row_off_host[0] == 0, "row_off[0] must be 0");
  for (int k = 0; k < T; ++k) ORX_REQUIRE(row_off_host[k + 1] >= row_off_host[k], "row_off must be non-decreasing");
  const int64_t G = row_off_host[T];
  ORX_REQUIRE(G <= INT32_MAX, "the concatenated tables exceed 2^31 - 1 rows");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  const int64_t n = (int64_t)B * T;
  ORX_CUDA(cudaMemsetAsync(counts, 0, sizeof(int32_t) * world, st));
  ORX_CUDA(cudaMemsetAsync(grp_off, 0, sizeof(int32_t), st));
  if (n == 0) return ORX_OK;
  ORX_REQUIRE(sparse && send_local && slot && grp_idx, "null pointer");
  const uint32_t L = (uint32_t)((G + world - 1) / world);
  const uint32_t invalid = (uint32_t)world * L;   // <= G + world - 1 < 2^32 - 1
  int bits = 1;
  while (bits < 32 && (invalid >> bits) != 0) ++bits;

  size_t sort_bytes = 0, scan_bytes = 0;
  ORX_CUDA(cub::DeviceRadixSort::SortPairs((void*)nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                           (const int32_t*)nullptr, (int32_t*)nullptr, (int)n, 0, bits, st));
  ORX_CUDA(cub::DeviceScan::InclusiveSum((void*)nullptr, scan_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, (int)n,
                                         st));
  LookupWs w;
  const size_t tmp_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
  const int rc = orx_grow(&h->lookup_ws, &h->lookup_cap, lookup_layout(nullptr, n, T, world, tmp_bytes, &w));
  if (rc != ORX_OK) return rc;
  lookup_layout(static_cast<char*>(h->lookup_ws), n, T, world, tmp_bytes, &w);
  ORX_CUDA(cudaMemcpyAsync(w.row_off, row_off_host, sizeof(int64_t) * (size_t)(T + 1), cudaMemcpyHostToDevice, st));

  const int grid = orx_grid_for(n, 256, h->num_sms);
  k_lb_keys<<<grid, 256, 0, st>>>(sparse, n, T, w.row_off, world, L, w.keys_in, w.iota);
  ORX_LAUNCH_CHECK();
  size_t bytes = w.tmp_bytes;   // radix sort is stable: a unique row's lookups stay in ascending i
  ORX_CUDA(cub::DeviceRadixSort::SortPairs(w.tmp, bytes, w.keys_in, w.keys, w.iota, grp_idx, (int)n, 0, bits, st));
  k_lb_heads<<<grid, 256, 0, st>>>(w.keys, n, invalid, w.iota);
  ORX_LAUNCH_CHECK();
  bytes = w.tmp_bytes;
  ORX_CUDA(cub::DeviceScan::InclusiveSum(w.tmp, bytes, w.iota, w.incl, (int)n, st));
  k_lb_scatter<<<grid, 256, 0, st>>>(w.keys, grp_idx, w.incl, n, world, L, slot, grp_off, send_local, w.ostart);
  ORX_LAUNCH_CHECK();
  k_lb_counts<<<(world + 255) / 256, 256, 0, st>>>(w.ostart, world, counts);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// One warp per unique row j: out[j] = sum of src rows grp_idx[grp_off[j] .. grp_off[j + 1]), added in that order (the
// loads of U consecutive rows are issued together, the adds stay sequential), so every call gives the same bits.
template <bool VEC>
__global__ void __launch_bounds__(256) k_rows_segment_sum(const float* __restrict__ src, int64_t ld, int dim,
                                                          const int32_t* __restrict__ grp_off,
                                                          const int32_t* __restrict__ grp_idx, int n_uniq,
                                                          float* __restrict__ out) {
  constexpr int U = 4;
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n_uniq; j += warps) {
    const int32_t p0 = grp_off[j], p1 = grp_off[j + 1];
    float* o = out + j * (int64_t)dim;
    if (VEC) {
      for (int e = lane * 4; e < dim; e += 128) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        int32_t p = p0;
        for (; p + U <= p1; p += U) {
          float4 v[U];
#pragma unroll
          for (int u = 0; u < U; ++u) v[u] = __ldg(reinterpret_cast<const float4*>(src + (int64_t)grp_idx[p + u] * ld + e));
#pragma unroll
          for (int u = 0; u < U; ++u) {
            acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w;
          }
        }
        for (; p < p1; ++p) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(src + (int64_t)grp_idx[p] * ld + e));
          acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        *reinterpret_cast<float4*>(o + e) = acc;
      }
    } else {
      for (int e = lane; e < dim; e += 32) {
        float acc = 0.f;
        int32_t p = p0;
        for (; p + U <= p1; p += U) {
          float v[U];
#pragma unroll
          for (int u = 0; u < U; ++u) v[u] = __ldg(src + (int64_t)grp_idx[p + u] * ld + e);
#pragma unroll
          for (int u = 0; u < U; ++u) acc += v[u];
        }
        for (; p < p1; ++p) acc += __ldg(src + (int64_t)grp_idx[p] * ld + e);
        o[e] = acc;
      }
    }
  }
}

extern "C" int orx_rows_segment_sum(orx_handle_t h, const float* src, int64_t src_ld, int32_t dim, const int32_t* grp_off,
                                    const int32_t* grp_idx, int32_t n_uniq, float* out, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null pointer");
  ORX_REQUIRE(dim >= 1 && src_ld >= dim && n_uniq >= 0, "bad sizes");
  if (n_uniq == 0) return ORX_OK;
  ORX_REQUIRE(src && grp_off && grp_idx && out, "null pointer");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  const bool vec = (dim & 3) == 0 && (src_ld & 3) == 0 && orx_aligned16(src, out);
  int64_t blocks = ((int64_t)n_uniq + 7) / 8;
  const int64_t cap = (int64_t)h->num_sms * 64;
  if (blocks > cap) blocks = cap;
  if (vec) k_rows_segment_sum<true><<<(int)blocks, 256, 0, st>>>(src, src_ld, dim, grp_off, grp_idx, n_uniq, out);
  else k_rows_segment_sum<false><<<(int)blocks, 256, 0, st>>>(src, src_ld, dim, grp_off, grp_idx, n_uniq, out);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// Multi-hot (bag) form of the sharded DLRM step.  sparse [B, C] holds T bags per sample, table k's bag being columns
// col_off[k] .. col_off[k+1]; lookup i = b*C + c.  orx_bag_shard_lookups maps every id to its global row (the input of
// an orx_lookup_bucket call with one column and row_off = {0, G}), orx_bag_segment_sum folds the pooled gradient rows
// onto the unique rows that bucket call found.
// ---------------------------------------------------------------------------------------
struct BagShardCols {   // kernel parameter block, copied to shared memory by each block
  int32_t col_off[ORX_BAG_MAX_TABLES + 1];
  int64_t row_off[ORX_BAG_MAX_TABLES + 1];
};

// the table of column c: the largest k < T with col_off[k] <= c (an empty bag is never chosen)
__device__ __forceinline__ int bag_table_of(const int32_t* s_col, int T, int c) {
  int lo = 0, hi = T - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (s_col[mid] <= c) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(256) k_bag_shard_lookups(const __grid_constant__ BagShardCols bc, int T, int C,
                                                           const int32_t* __restrict__ sparse, int64_t n,
                                                           int32_t* __restrict__ rows) {
  __shared__ int32_t s_col[ORX_BAG_MAX_TABLES + 1];
  __shared__ int64_t s_row[ORX_BAG_MAX_TABLES + 1];
  for (int t = threadIdx.x; t <= T; t += blockDim.x) {
    s_col[t] = bc.col_off[t];
    s_row[t] = bc.row_off[t];
  }
  __syncthreads();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = bag_table_of(s_col, T, (int)(i % C));
    const int32_t id = sparse[i];
    const int64_t lo = s_row[k];
    rows[i] = id >= 0 && lo + id < s_row[k + 1] ? (int32_t)(lo + id) : -1;
  }
}

extern "C" int orx_bag_shard_lookups(orx_handle_t h, const int32_t* sparse, int32_t B, int32_t T,
                                     const int32_t* col_off_host, const int64_t* row_off_host, int32_t* rows,
                                     orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && col_off_host && row_off_host, "null pointer");
  ORX_REQUIRE(B >= 0 && T >= 1 && T <= ORX_BAG_MAX_TABLES, "B < 0 or T outside [1, ORX_BAG_MAX_TABLES]");
  ORX_REQUIRE(col_off_host[0] == 0 && row_off_host[0] == 0, "col_off[0] and row_off[0] must be 0");
  BagShardCols bc;
  for (int k = 0; k < T; ++k) {
    ORX_REQUIRE(col_off_host[k + 1] >= col_off_host[k] && row_off_host[k + 1] >= row_off_host[k],
                "col_off / row_off must be non-decreasing");
    bc.col_off[k] = col_off_host[k];
    bc.row_off[k] = row_off_host[k];
  }
  bc.col_off[T] = col_off_host[T];
  bc.row_off[T] = row_off_host[T];
  const int32_t C = col_off_host[T];
  ORX_REQUIRE(C >= 1, "no bag columns");
  ORX_REQUIRE(row_off_host[T] <= INT32_MAX, "the concatenated tables exceed 2^31 - 1 rows");
  ORX_REQUIRE((int64_t)B * C <= INT32_MAX, "B * C exceeds 2^31 - 1 lookups");
  if (B == 0) return ORX_OK;
  ORX_REQUIRE(sparse && rows, "null sparse / rows");
  ORX_CUDA(cudaSetDevice(h->device));
  const int64_t n = (int64_t)B * C;
  k_bag_shard_lookups<<<orx_grid_for(n, 256, h->num_sms), 256, 0, (cudaStream_t)s>>>(bc, T, C, sparse, n, rows);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// cnt[b*T + k] = the valid lookups (slot >= 0) of bag (b, k), as a float.  One warp per bag, 32 columns at a time.
__global__ void __launch_bounds__(256) k_bag_counts(const __grid_constant__ BagShardCols bc, int T, int C,
                                                    const int32_t* __restrict__ slot, int64_t bags,
                                                    float* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < bags; w += nw) {
    const int64_t b = w / T;
    const int k = (int)(w - b * T);
    const int32_t* sl = slot + b * C;
    int n = 0;
    for (int c = bc.col_off[k]; c < bc.col_off[k + 1]; c += 32)
      n += __popc(__ballot_sync(ORX_FULL, c + lane < bc.col_off[k + 1] && __ldg(sl + c + lane) >= 0));
    if (lane == 0) cnt[w] = (float)n;
  }
}

template <bool VEC>
__device__ __forceinline__ float4 seg_ld(const float* p) {
  if (VEC) return __ldg(reinterpret_cast<const float4*>(p));
  return make_float4(__ldg(p), 0.f, 0.f, 0.f);
}

// One warp per unique row j: out[j] = the sum over p in [grp_off[j], grp_off[j+1]) of lookup grp_idx[p]'s gradient row,
// dZ[b, k(c), :] (divided by the bag's valid count for a mean, before the add), added in ascending p.  The lookups are
// decoded 32 at a time, one per lane, and handed out by shuffle; U row loads are issued before they are added.
// VEC: a lane holds one float4 of a 128-float column chunk, else one float of a 32-float chunk; wider rows take several
// chunks, each decoding the lookups again.  No atomics: every call gives the same bits.
template <bool VEC>
__global__ void __launch_bounds__(256) k_bag_segment_sum(const __grid_constant__ BagShardCols bc, int T, int C,
                                                         const float* __restrict__ dz, int64_t dz_ld, int dim,
                                                         const float* __restrict__ cnt,
                                                         const int32_t* __restrict__ grp_off,
                                                         const int32_t* __restrict__ grp_idx, int n_uniq,
                                                         float* __restrict__ out) {
  constexpr int U = 4, W = VEC ? 4 : 1;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  __shared__ int32_t s_col[ORX_BAG_MAX_TABLES + 1];
  for (int t = threadIdx.x; t <= T; t += blockDim.x) s_col[t] = bc.col_off[t];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n_uniq; j += warps) {
    const int32_t p0 = grp_off[j], p1 = grp_off[j + 1];
    float* o = out + j * (int64_t)dim;
    for (int e0 = 0; e0 < dim; e0 += 32 * W) {
      const int e = e0 + lane * W;
      const bool on = e < dim;
      float4 acc = z4;
      for (int32_t pb = p0; pb < p1; pb += 32) {
        const int m = min(32, p1 - pb);
        int64_t src = 0;
        float nb = 1.f;
        if (lane < m) {
          const int32_t i = __ldg(grp_idx + pb + lane);
          const int32_t b = i / C;
          const int c = i - b * C;
          const int k = bag_table_of(s_col, T, c);
          src = (int64_t)b * dz_ld + (int64_t)k * dim;
          if (cnt) nb = __ldg(cnt + (int64_t)b * T + k);
        }
        for (int q = 0; q < m; q += U) {   // warp-uniform
          float4 v[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int64_t r = __shfl_sync(ORX_FULL, src, (q + u) & 31);
            v[u] = (q + u < m && on) ? seg_ld<VEC>(dz + r + e) : z4;
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const float d = __shfl_sync(ORX_FULL, nb, (q + u) & 31);
            if (q + u >= m) break;
            if (cnt) v[u] = make_float4(v[u].x / d, v[u].y / d, v[u].z / d, v[u].w / d);
            acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w;
          }
        }
      }
      if (!on) continue;
      if (VEC) *reinterpret_cast<float4*>(o + e) = acc;
      else o[e] = acc.x;
    }
  }
}

extern "C" int orx_bag_segment_sum(orx_handle_t h, const float* dZ, int64_t dz_ld, int32_t T, int32_t dim,
                                   const int32_t* col_off_host, int32_t mode, const int32_t* slot, int32_t B,
                                   const int32_t* grp_off, const int32_t* grp_idx, int32_t n_uniq, float* out,
                                   orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && col_off_host, "null pointer");
  ORX_REQUIRE(T >= 1 && T <= ORX_BAG_MAX_TABLES, "T outside [1, ORX_BAG_MAX_TABLES]");
  ORX_REQUIRE(dim >= 1 && B >= 0 && n_uniq >= 0 && (mode == 0 || mode == 1), "bad sizes / mode");
  ORX_REQUIRE(dz_ld >= (int64_t)T * dim, "dz_ld < T * dim");
  ORX_REQUIRE(col_off_host[0] == 0, "col_off[0] must be 0");
  BagShardCols bc;
  for (int k = 0; k < T; ++k) {
    ORX_REQUIRE(col_off_host[k + 1] >= col_off_host[k], "col_off must be non-decreasing");
    bc.col_off[k] = col_off_host[k];
    bc.row_off[k] = 0;
  }
  bc.col_off[T] = col_off_host[T];
  bc.row_off[T] = 0;
  const int32_t C = col_off_host[T];
  ORX_REQUIRE(C >= 1, "no bag columns");
  ORX_REQUIRE((int64_t)B * C <= INT32_MAX, "B * C exceeds 2^31 - 1 lookups");
  ORX_REQUIRE(n_uniq <= (int64_t)B * C, "more unique rows than lookups");
  if (n_uniq == 0) return ORX_OK;
  ORX_REQUIRE(dZ && grp_off && grp_idx && out && (mode == 0 || slot), "null pointer");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  float* cnt = nullptr;
  if (mode == 1) {
    const int64_t bags = (int64_t)B * T;
    const int rc = orx_grow(&h->bag_cnt_ws, &h->bag_cnt_cap, sizeof(float) * (size_t)bags);
    if (rc != ORX_OK) return rc;
    cnt = static_cast<float*>(h->bag_cnt_ws);
    int64_t blocks = (bags + 7) / 8;
    if (blocks > (int64_t)h->num_sms * 32) blocks = (int64_t)h->num_sms * 32;
    k_bag_counts<<<(int)blocks, 256, 0, st>>>(bc, T, C, slot, bags, cnt);
    ORX_LAUNCH_CHECK();
  }
  const bool vec = (dim & 3) == 0 && (dz_ld & 3) == 0 && orx_aligned16(dZ, out);
  int64_t blocks = ((int64_t)n_uniq + 7) / 8;
  const int64_t cap = (int64_t)h->num_sms * 64;
  if (blocks > cap) blocks = cap;
  if (vec)
    k_bag_segment_sum<true><<<(int)blocks, 256, 0, st>>>(bc, T, C, dZ, dz_ld, dim, cnt, grp_off, grp_idx, n_uniq, out);
  else
    k_bag_segment_sum<false><<<(int)blocks, 256, 0, st>>>(bc, T, C, dZ, dz_ld, dim, cnt, grp_off, grp_idx, n_uniq, out);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}
