// orx_pointwise_shard.cu -- the pointwise-specific kernels of the row-sharded GMF / WRMF step
// (openrec_b200/sharded.py pointwise_step_sharded) and the scale of the sharded GMF score:
//   * orx_pointwise_shard_lookups : (uid, iid) -> the [B, 2] lookup matrix of orx_lookup_bucket, a bad sample -> (-1, -1)
//   * orx_pointwise_serve         : owner side, one exchange row of width ld per requested local row (user row, or item
//                                   row with its bias in column dim; zero padding) and the per-table local ids
//   * orx_pointwise_grad_rows     : score, loss and the per-lookup gradient rows over the fetched rows, GMF's [dim]
//                                   gradient partial of w, in a fixed order (no atomics: the same bits on every call)
//   * orx_rows_scale              : x[r, k] = x[r, k] * scale[k] with one rounding (GMF's u * w of the shard phases)
// The row space of the exchange: user u is global row u, item i is global row R*Lu + i (Lu = ceil(U / R)), so user and
// item row ownership is that of the per-table layout (row r on rank r % R at local row r / R) and the owner's local
// rows < Lu are user rows, the rest item rows (item local row + Lu).
#include "orx_common.cuh"

__global__ void __launch_bounds__(256) k_pw_lookups(const int32_t* __restrict__ uid, const int32_t* __restrict__ iid,
                                                    int B, int64_t U, int64_t I, int32_t* __restrict__ out) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < B; t += gridDim.x * blockDim.x) {
    const int32_t u = uid[t], i = iid[t];
    const bool ok = u >= 0 && (int64_t)u < U && i >= 0 && (int64_t)i < I;
    reinterpret_cast<int2*>(out)[t] = ok ? make_int2(u, i) : make_int2(-1, -1);
  }
}

extern "C" int orx_pointwise_shard_lookups(orx_handle_t h, const int32_t* uid, const int32_t* iid, int32_t B,
                                           int64_t total_users, int64_t total_items, int32_t* lookups,
                                           orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(B >= 0 && total_users >= 0 && total_items >= 0 && total_users <= INT32_MAX && total_items <= INT32_MAX,
              "bad sizes");
  if (B == 0) return ORX_OK;
  ORX_REQUIRE(uid && iid && lookups, "null pointer");
  ORX_REQUIRE(((uintptr_t)lookups & 7) == 0, "lookups must be 8-byte aligned");
  ORX_CUDA(cudaSetDevice(h->device));
  k_pw_lookups<<<orx_grid_for(B, 256, h->num_sms), 256, 0, (cudaStream_t)s>>>(uid, iid, B, total_users,
                                                                              total_items, lookups);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// One thread per (request, column group of VW floats); column 0's thread also writes the two local ids.
template <int VW>
__global__ void __launch_bounds__(256) k_pw_serve(const float* __restrict__ user, const float* __restrict__ item,
                                                  const float* __restrict__ bias, int dim, int64_t local_users,
                                                  int64_t local_items, int64_t Lu, const int32_t* __restrict__ req,
                                                  int64_t n, int64_t ld, float* __restrict__ out,
                                                  int32_t* __restrict__ user_local, int32_t* __restrict__ item_local) {
  const int64_t cols = ld / VW;
  for (int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; x < n * cols; x += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = x / cols;
    const int c = (int)(x - r * cols) * VW;
    const int32_t q = req[r];
    const bool is_u = q >= 0 && q < local_users;
    const bool is_i = q >= Lu && q - Lu < local_items;
    float v[VW];
#pragma unroll
    for (int k = 0; k < VW; ++k) {
      const int e = c + k;
      float val = 0.f;
      if (e < dim) {
        if (is_u) val = user[(int64_t)q * dim + e];
        else if (is_i) val = item[(q - Lu) * dim + e];
      } else if (e == dim && is_i) {
        val = bias[q - Lu];
      }
      v[k] = val;
    }
    if (VW == 4) *reinterpret_cast<float4*>(out + r * ld + c) = make_float4(v[0], v[1], v[2], v[3]);
    else out[r * ld + c] = v[0];
    if (c == 0) {
      user_local[r] = is_u ? q : -1;
      item_local[r] = is_i ? (int32_t)(q - Lu) : -1;
    }
  }
}

extern "C" int orx_pointwise_serve(orx_handle_t h, const float* user_shard, const float* item_shard,
                                   const float* bias_shard, int32_t dim, int64_t local_users, int64_t local_items,
                                   int64_t user_rows_per_rank, const int32_t* req, int32_t n, int64_t ld,
                                   float* rows, int32_t* user_local, int32_t* item_local, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(dim >= 1 && ld >= (int64_t)dim + 1 && n >= 0 && local_users >= 0 && local_items >= 0, "bad sizes");
  ORX_REQUIRE(user_rows_per_rank >= local_users && user_rows_per_rank + local_items <= INT32_MAX,
              "user_rows_per_rank must cover this rank's user rows, and local rows must fit int32");
  if (n == 0) return ORX_OK;
  ORX_REQUIRE(req && rows && user_local && item_local, "null pointer");
  ORX_REQUIRE((local_users == 0 || user_shard) && (local_items == 0 || (item_shard && bias_shard)), "null shard");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  const bool vec = (ld & 3) == 0 && orx_aligned16(rows);
  const int64_t work = (int64_t)n * (vec ? ld / 4 : ld);
  const int grid = orx_grid_for(work, 256, h->num_sms);
  if (vec)
    k_pw_serve<4><<<grid, 256, 0, st>>>(user_shard, item_shard, bias_shard, dim, local_users, local_items,
                                        user_rows_per_rank, req, n, ld, rows, user_local, item_local);
  else
    k_pw_serve<1><<<grid, 256, 0, st>>>(user_shard, item_shard, bias_shard, dim, local_users, local_items,
                                        user_rows_per_rank, req, n, ld, rows, user_local, item_local);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// per-lookup gradient rows
// ---------------------------------------------------------------------------------------
struct PgrArgs {
  const float* rows;      // fetched rows [*, ld]: user row, or item row with the bias in column D
  int64_t ld;
  const int32_t* slot;    // [2B]: row of lookup 2b (user) / 2b + 1 (item) in rows, -1 for a skipped sample
  const float* label;
  const float* W;         // GMF's w [D], else null
  int B, D;
  float wa, wb, c_loss, c_l2, inv_B;
  int use_sigmoid;
  float* d_rows;          // [2B, ld]
  float* gw_part;         // GMF: [blocks, D] per-block partials of w's gradient
  float* partials;        // (loss, l2) per warp
};

// point_score of orx_pointwise.cu, on this file's argument block
template <int KIND>
__device__ __forceinline__ void pgr_score(float s, float bias, float label, const PgrArgs& a, float* lt, float* g) {
  if (KIND == ORX_POINT_GMF) {
    const float z = s + bias;
    *lt = fmaxf(z, 0.f) - z * label + log1pf(expf(-fabsf(z)));
    *g = a.c_loss * (orx_sigmoid(z) - label) * a.inv_B;
  } else {
    float pred = s + bias;
    if (a.use_sigmoid) pred = orx_sigmoid(pred);
    const float wgt = (a.wa - a.wb) * label + a.wb;
    const float diff = label - pred;
    *lt = wgt * diff * diff;
    float d = a.c_loss * -2.f * wgt * diff;
    if (a.use_sigmoid) d = d * pred * (1.f - pred);
    *g = d;
  }
}

// The warps' [D] partials of w's gradient (sgw[warp][D]) summed in warp order into this block's row of gw_part.
__device__ __forceinline__ void pgr_block_gw(const float* sgw, int D, float* gw_part) {
  __syncthreads();
  for (int e = threadIdx.x; e < D; e += blockDim.x) {
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) acc += sgw[w * D + e];
    gw_part[(int64_t)blockIdx.x * D + e] = acc;
  }
}

// k_point_step's lane groups and arithmetic order: a group of G lanes per sample, float4 loads, CH samples per warp.
template <int KIND, int D, int CH>
__global__ void __launch_bounds__(256) k_pgr_step(const PgrArgs a) {
  constexpr int G = (D / 4 < 32) ? D / 4 : 32;
  constexpr int K = D / (4 * G);
  constexpr int TPW = 32 / G;
  constexpr bool GMF = (KIND == ORX_POINT_GMF);
  __shared__ __align__(16) float sgw[GMF ? 8 * D : 1];

  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int grp = lane / G, gl = lane % G;
  const int t = warp * CH + lane;
  int su = -1, si = -1;
  float bi = 0.f, lab = 0.f;
  if (lane < CH && t < a.B) {
    const int2 sl = reinterpret_cast<const int2*>(a.slot)[t];
    lab = a.label[t];
    if (sl.x >= 0 && sl.y >= 0) {
      su = sl.x;
      si = sl.y;
      bi = __ldg(a.rows + (int64_t)si * a.ld + D);
    }
  }
  float4 w[K], gwacc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    w[k] = GMF ? __ldg(reinterpret_cast<const float4*>(a.W + (k * G + gl) * 4)) : make_float4(1.f, 1.f, 1.f, 1.f);
    gwacc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float loss_acc = 0.f, l2_acc = 0.f;
#pragma unroll 1
  for (int j = 0; j < CH; j += TPW) {
    const int src = j + grp;
    const int uu = __shfl_sync(ORX_FULL, su, src), ii = __shfl_sync(ORX_FULL, si, src);
    const float bj = __shfl_sync(ORX_FULL, bi, src), lj = __shfl_sync(ORX_FULL, lab, src);
    const int ts = warp * CH + src;
    const bool in = ts < a.B;
    const bool v = uu >= 0;
    float4 u[K], it[K];
    float s = 0.f, sq = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int off = (k * G + gl) * 4;
      u[k] = v ? __ldg(reinterpret_cast<const float4*>(a.rows + (int64_t)uu * a.ld + off)) : z4;
      it[k] = v ? __ldg(reinterpret_cast<const float4*>(a.rows + (int64_t)ii * a.ld + off)) : z4;
      s += w[k].x * u[k].x * it[k].x + w[k].y * u[k].y * it[k].y + w[k].z * u[k].z * it[k].z +
           w[k].w * u[k].w * it[k].w;
      sq += u[k].x * u[k].x + u[k].y * u[k].y + u[k].z * u[k].z + u[k].w * u[k].w + it[k].x * it[k].x +
            it[k].y * it[k].y + it[k].z * it[k].z + it[k].w * it[k].w;
    }
    l2_acc += sq;
    s = orx_group_sum<G>(s);
    float lt = 0.f, g = 0.f;
    pgr_score<KIND>(s, bj, lj, a, &lt, &g);
    if (!v) { lt = 0.f; g = 0.f; }
    if (gl == 0) loss_acc += lt;
    if (in) {
      float* du = a.d_rows + (int64_t)(2 * ts) * a.ld;
      float* di = du + a.ld;
      const float c2 = a.c_l2;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int off = (k * G + gl) * 4;
        float4 gu = z4, gi = z4;
        if (v) {
          gu.x = g * w[k].x * it[k].x + c2 * u[k].x; gu.y = g * w[k].y * it[k].y + c2 * u[k].y;
          gu.z = g * w[k].z * it[k].z + c2 * u[k].z; gu.w = g * w[k].w * it[k].w + c2 * u[k].w;
          gi.x = g * w[k].x * u[k].x + c2 * it[k].x; gi.y = g * w[k].y * u[k].y + c2 * it[k].y;
          gi.z = g * w[k].z * u[k].z + c2 * it[k].z; gi.w = g * w[k].w * u[k].w + c2 * it[k].w;
          if (GMF) {
            gwacc[k].x += g * u[k].x * it[k].x; gwacc[k].y += g * u[k].y * it[k].y;
            gwacc[k].z += g * u[k].z * it[k].z; gwacc[k].w += g * u[k].w * it[k].w;
          }
        }
        *reinterpret_cast<float4*>(du + off) = gu;
        *reinterpret_cast<float4*>(di + off) = gi;
      }
      for (int e = D + gl; e < a.ld; e += G) {   // bias gradient in column D of the item row, zero padding
        du[e] = 0.f;
        di[e] = e == D ? g : 0.f;
      }
    }
  }
  if (GMF) {
#pragma unroll
    for (int k = 0; k < K; ++k) {   // the TPW groups of the warp hold the same elements: fold them, lane order fixed
#pragma unroll
      for (int o = G; o < 32; o <<= 1) {
        gwacc[k].x += __shfl_xor_sync(ORX_FULL, gwacc[k].x, o);
        gwacc[k].y += __shfl_xor_sync(ORX_FULL, gwacc[k].y, o);
        gwacc[k].z += __shfl_xor_sync(ORX_FULL, gwacc[k].z, o);
        gwacc[k].w += __shfl_xor_sync(ORX_FULL, gwacc[k].w, o);
      }
      if (grp == 0) *reinterpret_cast<float4*>(sgw + wib * D + (k * G + gl) * 4) = gwacc[k];
    }
    pgr_block_gw(sgw, D, a.gw_part);
  }
  orx_warp_partial(loss_acc, l2_acc, a.partials);
}

// Any D and ld: one warp per sample, 8 samples per warp; GMF's warp partials of w's gradient in dynamic shared memory.
template <int KIND>
__global__ void __launch_bounds__(256) k_pgr_generic(const PgrArgs a) {
  extern __shared__ float sgw_dyn[];
  constexpr bool GMF = (KIND == ORX_POINT_GMF);
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int D = a.D;
  float* sgw = sgw_dyn + wib * D;
  if (GMF)
    for (int d = lane; d < D; d += 32) sgw[d] = 0.f;
  float loss_acc = 0.f, l2_acc = 0.f;
  for (int j = 0; j < 8; ++j) {
    const int t = warp * 8 + j;
    if (t >= a.B) break;
    const int2 sl = reinterpret_cast<const int2*>(a.slot)[t];
    const bool ok = sl.x >= 0 && sl.y >= 0;
    const float* ur = a.rows + (int64_t)(ok ? sl.x : 0) * a.ld;
    const float* ir = a.rows + (int64_t)(ok ? sl.y : 0) * a.ld;
    float s = 0.f, sq = 0.f;
    if (ok) {
      for (int d = lane; d < D; d += 32) {
        const float u = ur[d], it = ir[d], w = GMF ? a.W[d] : 1.f;
        s += w * u * it;
        sq += u * u + it * it;
      }
    }
    l2_acc += sq;
    s = orx_group_sum<32>(s);
    float lt = 0.f, g = 0.f;
    if (ok) pgr_score<KIND>(s, ir[D], a.label[t], a, &lt, &g);
    if (lane == 0) loss_acc += lt;
    float* du = a.d_rows + (int64_t)(2 * t) * a.ld;
    float* di = du + a.ld;
    const float c2 = a.c_l2;
    for (int d = lane; d < D; d += 32) {
      float gu = 0.f, gi = 0.f;
      if (ok) {
        const float u = ur[d], it = ir[d], w = GMF ? a.W[d] : 1.f;
        gu = g * w * it + c2 * u;
        gi = g * w * u + c2 * it;
        if (GMF) sgw[d] += g * u * it;
      }
      du[d] = gu;
      di[d] = gi;
    }
    for (int e = D + lane; e < a.ld; e += 32) {
      du[e] = 0.f;
      di[e] = e == D ? g : 0.f;
    }
  }
  if (GMF) pgr_block_gw(sgw_dyn, D, a.gw_part);
  orx_warp_partial(loss_acc, l2_acc, a.partials);
}

// One warp per element e of w's gradient: the blocks' partials summed lane-strided, then a fixed tree (GMF); block 0
// also reduces the (loss, l2) partials in float64 and, with add_w, adds c_l2 * w[e] and 0.5 * sum(w^2).
__global__ void __launch_bounds__(256) k_pgr_finish(const float* partials, int n_partials, const float* gw_part,
                                                    int n_blocks, int D, const float* W, int add_w, float c_l2,
                                                    float loss_scale, float* gw, float* out2) {
  if (blockIdx.x == 0) {
    double l, q;
    orx_block_sum_partials(partials, n_partials, add_w ? W : nullptr, add_w ? D : 0, &l, &q);
    if (threadIdx.x == 0) {
      out2[0] = (float)(l * (double)loss_scale);
      out2[1] = (float)(0.5 * q);
    }
  }
  if (!gw) return;
  const int lane = threadIdx.x & 31;
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (e >= D) return;
  float acc = 0.f;
  for (int b = lane; b < n_blocks; b += 32) acc += gw_part[(int64_t)b * D + e];
  acc = orx_group_sum<32>(acc);
  if (lane == 0) gw[e] = add_w ? acc + c_l2 * W[e] : acc;
}

extern "C" int orx_pointwise_grad_rows(orx_handle_t h, int32_t kind, const float* rows, int64_t ld, int32_t dim,
                                       const int32_t* slot, const float* label, const float* w, int32_t B, float a,
                                       float b, int32_t use_sigmoid, float c_loss, float c_l2, float inv_B,
                                       int32_t add_w_terms, float* d_rows, float* gw, float* out2, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(kind == ORX_POINT_GMF || kind == ORX_POINT_WRMF, "unknown pointwise kind");
  ORX_REQUIRE(B > 0 && dim >= 1 && dim <= 1024 && ld >= (int64_t)dim + 1,
              "bad sizes (B >= 1, 1 <= dim <= 1024, ld > dim: the bias lives in column dim)");
  ORX_REQUIRE(rows && slot && label && d_rows && out2, "null pointer");
  ORX_REQUIRE(kind == ORX_POINT_WRMF || (w && gw), "GMF needs w and gw");
  ORX_REQUIRE(((uintptr_t)slot & 7) == 0, "slot must be 8-byte aligned");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  const bool gmf = kind == ORX_POINT_GMF;
  const int blocks = orx_step_blocks(B);
  const size_t part_bytes = sizeof(float) * 2 * 8 * (size_t)blocks;
  const size_t gw_bytes = gmf ? sizeof(float) * (size_t)dim * (size_t)blocks : 0;
  int rc = orx_grow((void**)&h->partials, &h->partials_cap, part_bytes + gw_bytes);
  if (rc) return rc;
  PgrArgs pa = {};
  pa.rows = rows; pa.ld = ld; pa.slot = slot; pa.label = label; pa.W = gmf ? w : nullptr;
  pa.B = B; pa.D = dim; pa.wa = a; pa.wb = b; pa.c_loss = c_loss; pa.c_l2 = c_l2; pa.inv_B = inv_B;
  pa.use_sigmoid = use_sigmoid; pa.d_rows = d_rows; pa.partials = h->partials;
  pa.gw_part = gmf ? h->partials + 2 * 8 * (size_t)blocks : nullptr;
  const bool vec = (dim == 32 || dim == 64 || dim == 128 || dim == 256) && (ld & 3) == 0 &&
                   orx_aligned16(rows, d_rows, gmf ? w : nullptr);
  const int variant = vec ? ORX_VARIANT_STEP : ORX_VARIANT_STEP_GENERIC;
  orx_dispatch<ORX_POINT_GMF, ORX_POINT_WRMF>(kind, [&](auto K) {
    constexpr int KD = decltype(K)::value;
    if (!vec) {
      k_pgr_generic<KD><<<blocks, 256, KD == ORX_POINT_GMF ? sizeof(float) * 8 * dim : 0, st>>>(pa);
      return;
    }
    switch (dim) {
      case 32: k_pgr_step<KD, 32, 8><<<blocks, 256, 0, st>>>(pa); break;
      case 64: k_pgr_step<KD, 64, 8><<<blocks, 256, 0, st>>>(pa); break;
      case 128: k_pgr_step<KD, 128, 8><<<blocks, 256, 0, st>>>(pa); break;
      default: k_pgr_step<KD, 256, 8><<<blocks, 256, 0, st>>>(pa); break;
    }
  });
  ORX_LAUNCH_CHECK();
  const int fin = gmf ? (dim + 7) / 8 : 1;
  k_pgr_finish<<<fin, 256, 0, st>>>(h->partials, 8 * blocks, pa.gw_part, blocks, dim, pa.W, gmf && add_w_terms, c_l2,
                                    gmf ? inv_B : 1.f, gmf ? gw : nullptr, out2);
  ORX_LAUNCH_CHECK();
  orx_log_dispatch(h, ORX_OP_POINTWISE_GRAD_ROWS, variant, kind, 0, B, dim, (int)(ld > INT32_MAX ? INT32_MAX : ld), 1);
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// x[r, k] *= scale[k], rounded once (__fmul_rn: no contraction with a later add)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_rows_scale(float* __restrict__ x, int64_t n, int dim,
                                                    const float* __restrict__ scale) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    x[i] = __fmul_rn(x[i], scale[i % dim]);
}

extern "C" int orx_rows_scale(orx_handle_t h, float* x, int64_t rows, int32_t dim, const float* scale,
                              orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(rows >= 0 && dim >= 1, "bad sizes");
  if (rows == 0) return ORX_OK;
  ORX_REQUIRE(x && scale, "null pointer");
  ORX_CUDA(cudaSetDevice(h->device));
  const int64_t n = rows * dim;
  k_rows_scale<<<orx_grid_for(n, 256, h->num_sms), 256, 0, (cudaStream_t)s>>>(x, n, dim, scale);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}
