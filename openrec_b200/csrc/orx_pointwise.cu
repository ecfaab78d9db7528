// orx_pointwise.cu -- GMF / WRMF fused training step (K3/K4).
//
// Reference path replaced: openrec/tf2/recommenders/gmf.py:22-34, wrmf.py:21-34,
// modules/pointwise_mse_loss.py:18-31 + tape.gradient + apply_gradients.
// Same three launches as the pairwise step (index -> step -> tail), run by orx_sparse_step; GMF's dense [D] weight
// gets its batch-summed gradient through shared-memory + one global reduction per block and is
// updated by the tail.
#include "orx_common.cuh"

struct PointArgs : SparseArgs {
  const float* W;  // GMF weight [D] (pre-step) or null
  float* gw;       // staged dense gradient of W
  int64_t rowsU, rowsI;
  const int32_t *uid, *iid;
  const float* label;
  int B;
  float wa, wb, c_loss, c_l2, inv_B;
  int use_sigmoid;
  float* partials;
  // un-fused outputs (grad kernel only)
  float *d_user, *d_item, *d_bias, *g_out;
};

// (loss term, dloss/dscore scalar).  GMF: BCE-with-logits mean (gmf.py:28-29) ; WRMF: weighted SSE
// (pointwise_mse_loss.py:22-31).
template <int KIND>
__device__ __forceinline__ void point_score(float s, float bias, float label, const PointArgs& a, float* lt,
                                            float* g) {
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

// T: the storage of the user and item tables, float or bf16 bits (uint16_t; rows 8-byte aligned, read as their exact
// fp32 upcast and rounded on store with the keys a.srk).  Slot rows, the item bias and GMF's w are float either way.
template <int KIND, int OPT, int D, int CH, typename T = float>
__global__ void __launch_bounds__(256) k_point_step(const PointArgs a) {
  constexpr int G = (D / 4 < 32) ? D / 4 : 32;
  constexpr int K = D / (4 * G);
  constexpr int TPW = 32 / G;
  typedef OrxOptSlots<OPT> SL;
  typedef OrxOptSlots<SL::ELEM> BL;   // the item bias's optimizer (element-wise)
  constexpr bool GMF = (KIND == ORX_POINT_GMF);
  __shared__ float sgw[GMF ? D : 1];

  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int grp = lane / G, gl = lane % G;
  const int t = warp * CH + lane;
  if (GMF) {
    for (int e = threadIdx.x; e < D; e += blockDim.x) sgw[e] = 0.f;
    __syncthreads();
  }

  int u_id = 0, i_id = 0, du = -1, di = -1, flags = 0;
  float bi = 0.f, bs0 = 0.f, bs1 = 0.f, lab = 0.f;
  if (lane < CH && t < a.B) {
    u_id = a.uid[t];
    i_id = a.iid[t];
    lab = a.label[t];
    if (u_id >= 0 && u_id < a.rowsU && i_id >= 0 && i_id < a.rowsI) {
      const uint32_t cu = orx_hash_find(a.hu, u_id, &du);
      const uint32_t ci = orx_hash_find(a.hi, i_id, &di);
      bi = __ldcg(a.Bv + i_id);
      flags = 1;
      if (!SL::STAGE_ONLY) {
        flags |= (cu == 1u ? 2 : 0) | (ci == 1u ? 4 : 0);
        if (BL::S0 && (flags & 4)) bs0 = __ldcg(a.Bs0 + i_id);
        if (BL::S1 && (flags & 4)) bs1 = __ldcg(a.Bs1 + i_id);
      }
    }
  }
  float4 w[K], gwacc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    w[k] = GMF ? *reinterpret_cast<const float4*>(a.W + (k * G + gl) * 4) : make_float4(1.f, 1.f, 1.f, 1.f);
    gwacc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  }

  float loss_acc = 0.f, l2_acc = 0.f, g_own = 0.f;
#pragma unroll 1
  for (int j = 0; j < CH; j += TPW) {
    const int src = j + grp;
    const int fl = __shfl_sync(ORX_FULL, flags, src);
    const int uu = __shfl_sync(ORX_FULL, u_id, src), ii = __shfl_sync(ORX_FULL, i_id, src);
    const int duj = __shfl_sync(ORX_FULL, du, src), dij = __shfl_sync(ORX_FULL, di, src);
    const float bj = __shfl_sync(ORX_FULL, bi, src), lj = __shfl_sync(ORX_FULL, lab, src);
    const bool v = fl & 1;
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 u[K], it[K], us0[K], is0[K], us1[K], is1[K];
    float s = 0.f, sq = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int off = (k * G + gl) * 4;
      u[k] = v ? orx_ld4_cg(reinterpret_cast<const T*>(a.U) + (int64_t)uu * D + off) : z4;
      it[k] = v ? orx_ld4_cg(reinterpret_cast<const T*>(a.I) + (int64_t)ii * D + off) : z4;
      if (SL::S0) {
        us0[k] = (fl & 2) ? __ldcg(reinterpret_cast<const float4*>(a.Us0 + (int64_t)uu * D + off)) : z4;
        is0[k] = (fl & 4) ? __ldcg(reinterpret_cast<const float4*>(a.Is0 + (int64_t)ii * D + off)) : z4;
      }
      if (SL::S1) {
        us1[k] = (fl & 2) ? __ldcg(reinterpret_cast<const float4*>(a.Us1 + (int64_t)uu * D + off)) : z4;
        is1[k] = (fl & 4) ? __ldcg(reinterpret_cast<const float4*>(a.Is1 + (int64_t)ii * D + off)) : z4;
      }
      s += w[k].x * u[k].x * it[k].x + w[k].y * u[k].y * it[k].y + w[k].z * u[k].z * it[k].z +
           w[k].w * u[k].w * it[k].w;
      sq += u[k].x * u[k].x + u[k].y * u[k].y + u[k].z * u[k].z + u[k].w * u[k].w + it[k].x * it[k].x +
            it[k].y * it[k].y + it[k].z * it[k].z + it[k].w * it[k].w;
    }
    l2_acc += sq;
    s = orx_group_sum<G>(s);
    float lt = 0.f, g = 0.f;
    point_score<KIND>(s, bj, lj, a, &lt, &g);
    if (!v) { lt = 0.f; g = 0.f; }
    if (gl == 0) loss_acc += lt;
#pragma unroll
    for (int q = 0; q < TPW; ++q) {
      const float val = __shfl_sync(ORX_FULL, g, q * G);
      if (lane == j + q) g_own = val;
    }
    if constexpr (SL::ROW) {
      // each row's sum of squared gradients over its G lanes before the apply, outside `if (v)` (per triplet group)
      const float c2 = a.c_l2;
      auto grads = [&](int k, float4& gu, float4& gi) {
        gu = make_float4(g * w[k].x * it[k].x + c2 * u[k].x, g * w[k].y * it[k].y + c2 * u[k].y,
                         g * w[k].z * it[k].z + c2 * u[k].z, g * w[k].w * it[k].w + c2 * u[k].w);
        gi = make_float4(g * w[k].x * u[k].x + c2 * it[k].x, g * w[k].y * u[k].y + c2 * it[k].y,
                         g * w[k].z * u[k].z + c2 * it[k].z, g * w[k].w * u[k].w + c2 * it[k].w);
      };
      float su = 0.f, si = 0.f;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        float4 gu, gi;
        grads(k, gu, gi);
        su += orx_sq4(gu);
        si += orx_sq4(gi);
      }
      su = orx_group_sum<G>(su);
      si = orx_group_sum<G>(si);
      float ua = (fl & 2) ? __ldcg(a.Us0 + uu) : 0.f, ia = (fl & 4) ? __ldcg(a.Is0 + ii) : 0.f;
      const float fu = orx_row_scale(ua, su, D, a.opt), fi = orx_row_scale(ia, si, D, a.opt);
      if (v) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
          const int off = (k * G + gl) * 4;
          float4 gu, gi;
          grads(k, gu, gi);
          if (GMF) {
            gwacc[k].x += g * u[k].x * it[k].x; gwacc[k].y += g * u[k].y * it[k].y;
            gwacc[k].z += g * u[k].z * it[k].z; gwacc[k].w += g * u[k].w * it[k].w;
          }
          orx_own_or_stage4_row<false>(fl & 2, reinterpret_cast<T*>(a.U), uu, a.gu, duj, D, off, u[k], gu, fu, a.opt,
                                       a.srk[0]);
          orx_own_or_stage4_row<false>(fl & 4, reinterpret_cast<T*>(a.I), ii, a.gi, dij, D, off, it[k], gi, fi, a.opt,
                                       a.srk[1]);
        }
        if (gl == 0) {
          if (fl & 2) __stcg(a.Us0 + uu, ua);
          if (fl & 4) __stcg(a.Is0 + ii, ia);
        }
      }
    } else if (v) {
      const float c2 = a.c_l2;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int off = (k * G + gl) * 4;
        float4 gu, gi;
        gu.x = g * w[k].x * it[k].x + c2 * u[k].x; gu.y = g * w[k].y * it[k].y + c2 * u[k].y;
        gu.z = g * w[k].z * it[k].z + c2 * u[k].z; gu.w = g * w[k].w * it[k].w + c2 * u[k].w;
        gi.x = g * w[k].x * u[k].x + c2 * it[k].x; gi.y = g * w[k].y * u[k].y + c2 * it[k].y;
        gi.z = g * w[k].z * u[k].z + c2 * it[k].z; gi.w = g * w[k].w * u[k].w + c2 * it[k].w;
        if (GMF) {
          gwacc[k].x += g * u[k].x * it[k].x; gwacc[k].y += g * u[k].y * it[k].y;
          gwacc[k].z += g * u[k].z * it[k].z; gwacc[k].w += g * u[k].w * it[k].w;
        }
        orx_own_or_stage4<OPT, false>(fl & 2, reinterpret_cast<T*>(a.U), a.Us0, a.Us1, uu, a.gu, duj, D, off, u[k], gu,
                                      us0[k], us1[k], a.opt, a.srk[0]);
        orx_own_or_stage4<OPT, false>(fl & 4, reinterpret_cast<T*>(a.I), a.Is0, a.Is1, ii, a.gi, dij, D, off, it[k], gi,
                                      is0[k], is1[k], a.opt, a.srk[1]);
      }
    }
  }
  if (flags & 1) {
    if (flags & 4) {
      __stcg(a.Bv + i_id, orx_apply<SL::ELEM>(bi, g_own, bs0, bs1, a.opt));
      if (BL::S0) __stcg(a.Bs0 + i_id, bs0);
      if (BL::S1) __stcg(a.Bs1 + i_id, bs1);
    } else {
      atomicAdd(a.gb + di, g_own);
    }
  }
  if (GMF) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int off = (k * G + gl) * 4;
      atomicAdd(&sgw[off + 0], gwacc[k].x);
      atomicAdd(&sgw[off + 1], gwacc[k].y);
      atomicAdd(&sgw[off + 2], gwacc[k].z);
      atomicAdd(&sgw[off + 3], gwacc[k].w);
    }
    __syncthreads();
    for (int e = threadIdx.x; e < D; e += blockDim.x) atomicAdd(a.gw + e, sgw[e]);
  }
  orx_warp_partial(loss_acc, l2_acc, a.partials);
}

// Any dim; MODE 0 = fused step, 1 = forward / explicit (un-fused) gradients.  T as in k_point_step.
template <int KIND, int OPT, int MODE, typename T = float>
__global__ void __launch_bounds__(256) k_point_generic(const PointArgs a) {
  constexpr bool STAGE_ONLY = OrxOptSlots<OPT>::STAGE_ONLY;
  constexpr bool GMF = (KIND == ORX_POINT_GMF);
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int D = a.D;
  float loss_acc = 0.f, l2_acc = 0.f;
  for (int j = 0; j < 8; ++j) {
    const int t = warp * 8 + j;
    if (t >= a.B) break;
    const int uu = a.uid[t], ii = a.iid[t];
    const bool ok = uu >= 0 && uu < a.rowsU && ii >= 0 && ii < a.rowsI;
    T* ur = reinterpret_cast<T*>(a.U) + (int64_t)uu * D;
    T* ir = reinterpret_cast<T*>(a.I) + (int64_t)ii * D;
    float s = 0.f, sq = 0.f;
    if (ok) {
      for (int d = lane; d < D; d += 32) {
        const float u = orx_ld1(ur + d), it = orx_ld1(ir + d), w = GMF ? a.W[d] : 1.f;
        s += w * u * it;
        sq += u * u + it * it;
      }
    }
    l2_acc += sq;
    s = orx_group_sum<32>(s);
    float lt = 0.f, g = 0.f;
    const float bi = ok ? a.Bv[ii] : 0.f;
    if (ok) point_score<KIND>(s, bi, a.label[t], a, &lt, &g);
    if (lane == 0) loss_acc += lt;
    int du = -1, di = -1;
    bool fu = false, fi = false;
    if (MODE == 0 && ok) {
      const uint32_t cu = orx_hash_find(a.hu, uu, &du);
      const uint32_t ci = orx_hash_find(a.hi, ii, &di);
      fu = !STAGE_ONLY && cu == 1u;
      fi = !STAGE_ONLY && ci == 1u;
    }
    const float c2 = a.c_l2;
    if constexpr (OrxOptSlots<OPT>::ROW) {   // MODE 0 only: each owned row's squared-gradient sum, then the apply
      if (!ok) continue;   // warp-uniform
      const uint32_t rku = orx_sr_row(a.srk[0], uu), rki = orx_sr_row(a.srk[1], ii);
      float su = 0.f, si = 0.f;
      for (int d = lane; d < D; d += 32) {
        const float u = orx_ld1(ur + d), it = orx_ld1(ir + d), w = GMF ? a.W[d] : 1.f;
        const float gu = g * w * it + c2 * u, gi = g * w * u + c2 * it;
        su += gu * gu;
        si += gi * gi;
      }
      su = orx_group_sum<32>(su);
      si = orx_group_sum<32>(si);
      float ua = fu ? a.Us0[uu] : 0.f, ia = fi ? a.Is0[ii] : 0.f;
      const float xu = orx_row_scale(ua, su, D, a.opt), xi = orx_row_scale(ia, si, D, a.opt);
      for (int d = lane; d < D; d += 32) {
        const float u = orx_ld1(ur + d), it = orx_ld1(ir + d), w = GMF ? a.W[d] : 1.f;
        const float gu = g * w * it + c2 * u, gi = g * w * u + c2 * it;
        if (GMF && a.gw) atomicAdd(a.gw + d, g * u * it);
        if (fu) orx_st1(ur + d, orx_row_apply1(u, gu, xu, a.opt), rku, d);
        else atomicAdd(a.gu + (int64_t)du * D + d, gu);
        if (fi) orx_st1(ir + d, orx_row_apply1(it, gi, xi, a.opt), rki, d);
        else atomicAdd(a.gi + (int64_t)di * D + d, gi);
      }
      if (lane == 0) {
        if (fu) a.Us0[uu] = ua;
        if (fi) a.Is0[ii] = ia;
        if (fi) orx_update1<ORX_OPT_ADAGRAD>(a.Bv + ii, a.Bs0 + ii, nullptr, bi, g, a.opt);
        else atomicAdd(a.gb + di, g);
      }
      continue;
    } else {
    if (MODE == 0 ? ok : (a.d_user || a.d_item || a.gw)) {
      const uint32_t rku = orx_sr_row(a.srk[0], uu), rki = orx_sr_row(a.srk[1], ii);
      for (int d = lane; d < D; d += 32) {
        float gu = 0.f, gi = 0.f;
        if (ok) {
          const float u = orx_ld1(ur + d), it = orx_ld1(ir + d), w = GMF ? a.W[d] : 1.f;
          gu = g * w * it + c2 * u;
          gi = g * w * u + c2 * it;
          if (GMF && a.gw) atomicAdd(a.gw + d, g * u * it);
          if (MODE == 0) {
            const int64_t ou = (int64_t)uu * D + d, oi = (int64_t)ii * D + d;
            if (fu) orx_update1<OPT>(ur + d, a.Us0 + ou, a.Us1 + ou, u, gu, a.opt, rku, d);
            else atomicAdd(a.gu + (int64_t)du * D + d, gu);
            if (fi) orx_update1<OPT>(ir + d, a.Is0 + oi, a.Is1 + oi, it, gi, a.opt, rki, d);
            else atomicAdd(a.gi + (int64_t)di * D + d, gi);
          }
        }
        if (MODE == 1) {
          const int64_t o = (int64_t)t * D + d;
          if (a.d_user) a.d_user[o] = gu;
          if (a.d_item) a.d_item[o] = gi;
        }
      }
    }
    if (lane == 0) {
      if (MODE == 0 && ok) {
        if (fi) orx_update1<OPT>(a.Bv + ii, a.Bs0 + ii, a.Bs1 + ii, bi, g, a.opt);
        else atomicAdd(a.gb + di, g);
      }
      if (MODE == 1) {
        if (a.d_bias) a.d_bias[t] = g;
        if (a.g_out) a.g_out[t] = g;
      }
    }
    }
  }
  orx_warp_partial(loss_acc, l2_acc, a.partials);
}

// adds 0.5*sum(w^2) to out4[1] (gmf.py:31-32) and, for the explicit-gradient path, c_l2*w to d_w
__global__ void k_gmf_w_terms(const float* W, int D, float* out4, float* d_w, float c_l2) {
  __shared__ float sh[256];
  float q = 0.f;
  for (int e = threadIdx.x; e < D; e += blockDim.x) {
    q += W[e] * W[e];
    if (d_w) d_w[e] += c_l2 * W[e];
  }
  sh[threadIdx.x] = q;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0 && out4) out4[1] += 0.5f * sh[0];
}

// T = uint16_t: bf16 user / item tables, which take the same variants.
template <int KIND, int OPT, typename T = float>
static int launch_point_kind_opt(const PointArgs& pa, cudaStream_t st, OrxStepLaunch* out) {
  const int blocks = orx_step_blocks(pa.B);
  *out = {8 * blocks, ORX_VARIANT_STEP, 0};
  // k_point_step moves table rows as 4-element vectors (float4, or 8 bytes of bf16), slot rows and GMF's w as float4: a
  // base off the boundary its row path needs takes k_point_generic (a row-wise accumulator is read as scalars and does
  // not count)
  constexpr bool BF = std::is_same<T, uint16_t>::value;
  const bool rows_ok = BF ? orx_aligned8(pa.U, pa.I) : orx_aligned16(pa.U, pa.I);
  const bool vec = OrxOptSlots<OPT>::ROW ? rows_ok && orx_aligned16(pa.W)
                                         : rows_ok && orx_aligned16(pa.Us0, pa.Us1, pa.Is0, pa.Is1, pa.W);
  switch (vec ? pa.D : 0) {
    case 32: k_point_step<KIND, OPT, 32, 8, T><<<blocks, 256, 0, st>>>(pa); break;
    case 64: k_point_step<KIND, OPT, 64, 8, T><<<blocks, 256, 0, st>>>(pa); break;
    case 128: k_point_step<KIND, OPT, 128, 8, T><<<blocks, 256, 0, st>>>(pa); break;
    case 256: k_point_step<KIND, OPT, 256, 8, T><<<blocks, 256, 0, st>>>(pa); break;
    default:
      out->variant = ORX_VARIANT_STEP_GENERIC;
      k_point_generic<KIND, OPT, 0, T><<<blocks, 256, 0, st>>>(pa);
      break;
  }
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// The kernel arguments of a pointwise batch (shared part s); no gw, partials or un-fused outputs.
static PointArgs point_args(const SparseArgs& s, const orx_table_t* dense_w, const orx_table_t* user,
                            const orx_table_t* item, const int32_t* uid, const int32_t* iid, const float* label, int B,
                            float a, float b, int use_sigmoid, float c_loss, float c_l2) {
  PointArgs pa = {s};
  pa.W = dense_w ? dense_w->var : nullptr;
  pa.rowsU = user->rows; pa.rowsI = item->rows;
  pa.uid = uid; pa.iid = iid; pa.label = label; pa.B = B;
  pa.wa = a; pa.wb = b; pa.c_loss = c_loss; pa.c_l2 = c_l2; pa.inv_B = 1.0f / (float)B;
  pa.use_sigmoid = use_sigmoid;
  return pa;
}

// srk: bf16 user / item tables with these rounding keys (their var passed as float*), null: float tables
static int pointwise_step_impl(orx_ctx* h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                               const orx_table_t* item_bias, const orx_table_t* w, const int32_t* uid,
                               const int32_t* iid, const float* label, int32_t B, float a, float b,
                               int32_t use_sigmoid, float c_loss, float c_l2, const orx_opt_t* opt, float* out4,
                               cudaStream_t st, const uint32_t* srk = nullptr) {
  ORX_REQUIRE(label != nullptr, "empty batch or null inputs");
  ORX_REQUIRE(kind == ORX_POINT_GMF || kind == ORX_POINT_WRMF, "unknown pointwise kind");
  ORX_REQUIRE(kind == ORX_POINT_WRMF || w, "GMF needs w with dim == D");
  const orx_table_t* dense_w = (kind == ORX_POINT_GMF) ? w : nullptr;
  orx_opt_t od;
  if (opt && user) {   // dim-1 rows under ROWWISE_ADAGRAD run (and are recorded) as ADAGRAD
    od = orx_opt_dim(opt, user->dim);
    opt = &od;
  }
  const auto kernel = [&](const SparseArgs& sa, const int4* /*res: pairwise only*/, float* partials, OrxStepLaunch* out) {
    PointArgs pa = point_args(sa, dense_w, user, item, uid, iid, label, B, a, b, use_sigmoid, c_loss, c_l2);
    pa.partials = partials;
    pa.gw = dense_w ? h->gw : nullptr;
    return orx_dispatch<ORX_POINT_GMF, ORX_POINT_WRMF>(kind, [&](auto K) {
      return orx_dispatch_opt(opt->kind, [&](auto O) {
        if (srk) return launch_point_kind_opt<decltype(K)::value, decltype(O)::value, uint16_t>(pa, st, out);
        return launch_point_kind_opt<decltype(K)::value, decltype(O)::value>(pa, st, out);
      });
    });
  };
  return orx_sparse_step(h, srk ? ORX_OP_POINTWISE_STEP_BF16 : ORX_OP_POINTWISE_STEP, kind, user, item, item_bias,
                         dense_w, uid, iid, nullptr, B, opt, dense_w ? 1.0f / (float)B : 1.0f, c_l2, out4, kernel, st,
                         srk);
}

extern "C" int orx_pointwise_step(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                                  const orx_table_t* item_bias, const orx_table_t* w, const int32_t* uid,
                                  const int32_t* iid, const float* label, int32_t B, float a, float b,
                                  int32_t use_sigmoid, float c_loss, float c_l2, const orx_opt_t* opt, float* out4,
                                  orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_CUDA(cudaSetDevice(h->device));
  return pointwise_step_impl(h, kind, user, item, item_bias, w, uid, iid, label, B, a, b, use_sigmoid, c_loss, c_l2,
                             opt, out4, (cudaStream_t)s);
}

extern "C" int orx_pointwise_step_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                       const orx_table_bf16_t* item, const orx_table_t* item_bias,
                                       const orx_table_t* w, const int32_t* uid, const int32_t* iid,
                                       const float* label, int32_t B, float a, float b, int32_t use_sigmoid,
                                       float c_loss, float c_l2, const orx_opt_t* opt, uint64_t sr_seed, float* out4,
                                       orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(opt != nullptr, "null opt/out");
  ORX_CUDA(cudaSetDevice(h->device));
  orx_table_t tu, ti;
  const uint32_t srk[2] = {orx_sr_table_key(sr_seed, opt->step, 0), orx_sr_table_key(sr_seed, opt->step, 1)};
  return pointwise_step_impl(h, kind, orx_bf16_table(user, &tu), orx_bf16_table(item, &ti), item_bias, w, uid, iid,
                             label, B, a, b, use_sigmoid, c_loss, c_l2, opt, out4, (cudaStream_t)s, srk);
}

static int point_fwd_grad(orx_ctx* h, int kind, const orx_table_t* user, const orx_table_t* item,
                          const orx_table_t* bias, const orx_table_t* w, const int32_t* uid, const int32_t* iid,
                          const float* label, int B, float a, float b, int use_sigmoid, float c_loss, float c_l2,
                          float* d_user, float* d_item, float* d_bias, float* d_w, float* g_out, float* out4,
                          cudaStream_t st, bool bf16 = false) {
  ORX_REQUIRE(B > 0 && uid && iid && label, "empty batch or null inputs");
  ORX_REQUIRE(kind == ORX_POINT_GMF || kind == ORX_POINT_WRMF, "unknown pointwise kind");
  ORX_REQUIRE(kind == ORX_POINT_WRMF || w, "GMF needs w with dim == D");
  const orx_table_t* dense_w = (kind == ORX_POINT_GMF) ? w : nullptr;
  int rc = orx_check_step_tables(user, item, bias, dense_w, ORX_OPT_SGD);
  if (rc) return rc;
  const SparseArgs s = orx_sparse_args(h, user, item, bias, h->set[0], OrxOptDev{});
  PointArgs pa = point_args(s, dense_w, user, item, uid, iid, label, B, a, b, use_sigmoid, c_loss, c_l2);
  pa.d_user = d_user; pa.d_item = d_item; pa.d_bias = d_bias; pa.g_out = g_out;
  if (dense_w && d_w) {
    ORX_CUDA(cudaMemsetAsync(d_w, 0, sizeof(float) * user->dim, st));
    pa.gw = d_w;
  }
  const auto launch = [&](float* partials, int blocks) {
    pa.partials = partials;
    orx_dispatch<ORX_POINT_GMF, ORX_POINT_WRMF>(kind, [&](auto K) {
      if (bf16) k_point_generic<decltype(K)::value, ORX_OPT_SGD, 1, uint16_t><<<blocks, 256, 0, st>>>(pa);
      else k_point_generic<decltype(K)::value, ORX_OPT_SGD, 1><<<blocks, 256, 0, st>>>(pa);
    });
  };
  if ((rc = orx_sparse_unfused(h, B, dense_w ? pa.inv_B : 1.f, out4, launch, st))) return rc;
  if (dense_w && (out4 || d_w)) {
    k_gmf_w_terms<<<1, 256, 0, st>>>(w->var, user->dim, out4, d_w, c_l2);
    ORX_LAUNCH_CHECK();
  }
  return ORX_OK;
}

extern "C" int orx_pointwise_fwd(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                                 const orx_table_t* item_bias, const orx_table_t* w, const int32_t* uid,
                                 const int32_t* iid, const float* label, int32_t B, float a, float b,
                                 int32_t use_sigmoid, float* out4, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && out4 != nullptr, "null handle/out");
  ORX_CUDA(cudaSetDevice(h->device));
  return point_fwd_grad(h, kind, user, item, item_bias, w, uid, iid, label, B, a, b, use_sigmoid, 1.f, 1.f, nullptr,
                        nullptr, nullptr, nullptr, nullptr, out4, (cudaStream_t)s);
}

extern "C" int orx_pointwise_grad(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                                  const orx_table_t* item_bias, const orx_table_t* w, const int32_t* uid,
                                  const int32_t* iid, const float* label, int32_t B, float a, float b,
                                  int32_t use_sigmoid, float c_loss, float c_l2, float* d_user, float* d_item,
                                  float* d_bias, float* d_w, float* g_out, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_CUDA(cudaSetDevice(h->device));
  return point_fwd_grad(h, kind, user, item, item_bias, w, uid, iid, label, B, a, b, use_sigmoid, c_loss, c_l2, d_user,
                        d_item, d_bias, d_w, g_out, nullptr, (cudaStream_t)s);
}

extern "C" int orx_pointwise_fwd_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                      const orx_table_bf16_t* item, const orx_table_t* item_bias, const orx_table_t* w,
                                      const int32_t* uid, const int32_t* iid, const float* label, int32_t B, float a,
                                      float b, int32_t use_sigmoid, float* out4, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && out4 != nullptr, "null handle/out");
  ORX_CUDA(cudaSetDevice(h->device));
  orx_table_t tu, ti;
  return point_fwd_grad(h, kind, orx_bf16_table(user, &tu), orx_bf16_table(item, &ti), item_bias, w, uid, iid, label, B,
                        a, b, use_sigmoid, 1.f, 1.f, nullptr, nullptr, nullptr, nullptr, nullptr, out4, (cudaStream_t)s,
                        true);
}

extern "C" int orx_pointwise_grad_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                       const orx_table_bf16_t* item, const orx_table_t* item_bias,
                                       const orx_table_t* w, const int32_t* uid, const int32_t* iid,
                                       const float* label, int32_t B, float a, float b, int32_t use_sigmoid,
                                       float c_loss, float c_l2, float* d_user, float* d_item, float* d_bias,
                                       float* d_w, float* g_out, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_CUDA(cudaSetDevice(h->device));
  orx_table_t tu, ti;
  return point_fwd_grad(h, kind, orx_bf16_table(user, &tu), orx_bf16_table(item, &ti), item_bias, w, uid, iid, label, B,
                        a, b, use_sigmoid, c_loss, c_l2, d_user, d_item, d_bias, d_w, g_out, nullptr, (cudaStream_t)s,
                        true);
}
