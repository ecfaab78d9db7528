// orx_pairwise.cu -- BPR / UCML fused training step (K1/K2), its batch index (K9), the tail and the step driver shared
// with orx_pointwise.cu.
//
// Reference path replaced (paths relative to the reference repo):
//   openrec/tf2/recommenders/bpr.py:21-37, ucml.py:21-42, modules/pairwise_log_loss.py:15-34
//   + tape.gradient + optimizer.apply_gradients (tf2_examples/bpr_citeulike.py:33-39).
//
// Synchronous-batch semantics in three launches on one stream:
//   1. k_index_build : hash every id of the batch's valid triplets; rows hit more than once get a "staging" slot.
//   2. k_pair_step   : per triplet gather u,p,n (128-bit loads), score, loss, per-sample gradient.
//        * a row referenced exactly once in the batch is owned by its triplet: optimizer applied
//          in registers, row + slots written back once (read once, written once == algorithmic bytes);
//        * a row referenced more than once is NEVER written here: its per-sample gradient is
//          red.global.add'ed into the compact staging buffer (so every gather sees pre-step values).
//   3. k_sparse_tail : optimizer for the staged rows (once per unique row), staging re-zeroed, deterministic loss
//                      reduction.  The hash is not cleared: the next step's index uses a new epoch.
// k_pair_step is specialised on D = 32, 64, 128, 256; k_pair_generic takes any D, as the fused step (MODE 0) and as the
// forward / un-fused gradients (MODE 1).
#include "orx_common.cuh"
#include "orx_pair.cuh"

// ---------------------------------------------------------------------------------------
// K9: batch index
// ---------------------------------------------------------------------------------------
// Sample t of the batch is (a[t], b0[t]) (pointwise) or (a[t], b0[t], b1[t]) (pairwise); one thread per id.  Every bad
// id is counted.  A good id is inserted only when the whole sample is good: the step skips a sample with a bad id, so a
// row that only skipped samples reference must not be staged (the tail would apply the optimizer to it with g = 0, which
// moves an Adam row).
__global__ void k_index_build(OrxHash hu, OrxHash hi, const int32_t* __restrict__ a, int64_t rows_a,
                              const int32_t* __restrict__ b0, const int32_t* __restrict__ b1, int64_t rows_b, int n,
                              int stage_all, int32_t* bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (b1 ? 3 : 2) * n) return;
  const int t = i < n ? i : (i < 2 * n ? i - n : i - 2 * n);
  const int32_t ia = a[t], ib0 = b0[t], ib1 = b1 ? b1[t] : 0;
  const bool ga = ia >= 0 && (int64_t)ia < rows_a, gb0 = ib0 >= 0 && (int64_t)ib0 < rows_b,
             gb1 = ib1 >= 0 && (int64_t)ib1 < rows_b;
  const bool all = ga && gb0 && gb1;
  if (i < n) {
    if (!ga) atomicAdd(bad, 1);
    else if (all) orx_hash_insert(hu, ia, stage_all);
  } else {
    const bool g = i < 2 * n ? gb0 : gb1;
    if (!g) atomicAdd(bad, 1);
    else if (all) orx_hash_insert(hi, i < 2 * n ? ib0 : ib1, stage_all);
  }
}

__global__ void k_index_build_strided(OrxHash hu, const int32_t* __restrict__ a, int64_t stride, int64_t rows, int n,
                                       int stage_all, int32_t* bad) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int32_t id = a[(int64_t)i * stride];
    if (id >= 0 && (int64_t)id < rows) orx_hash_insert(hu, id, stage_all);
    else atomicAdd(bad, 1);
  }
}

int orx_launch_index_build_strided(orx_ctx* c, const int32_t* a, int64_t stride, int64_t rows, int32_t n,
                                   bool stage_all, cudaStream_t st) {
  if (n <= 0) return ORX_OK;
  int rc = orx_next_epoch(c, st);
  if (rc) return rc;
  k_index_build_strided<<<(n + 255) / 256, 256, 0, st>>>(c->hu, a, stride, rows, n, stage_all ? 1 : 0, c->counters + 3);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

int orx_launch_index_build(orx_ctx* c, const int32_t* a, int64_t rows_a, const int32_t* b0, const int32_t* b1,
                           int64_t rows_b, int32_t n, int mode, cudaStream_t st) {
  const int total = (b1 ? 3 : 2) * n;
  if (total <= 0) return ORX_OK;
  int rc = orx_next_epoch(c, st);
  if (rc) return rc;
  k_index_build<<<(total + 255) / 256, 256, 0, st>>>(c->hu, c->hi, a, rows_a, b0, b1, rows_b, n, mode, c->counters + 3);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// K1/K2: fused step
// ---------------------------------------------------------------------------------------
template <int K, bool S0, bool S1>
struct TripRegs {
  float4 u[K], p[K], n[K];
  float4 us0[K], ps0[K], ns0[K];  // dead arrays are eliminated when the optimizer has no such slot
  float4 us1[K], ps1[K], ns1[K];
  int fl, uu, pp, nn, du, dp, dn;
  float bp, bn;
};

// flags: bit0 triplet valid, bit1/2/3 user/pos/neg row owned by this triplet (fast path)
//
// One warp owns CH consecutive triplets.  Order of issue inside a warp (latency first):
//   ids (coalesced, lanes < CH) -> variable rows of the first one/two triplet groups (they need only
//   the ids) -> hash probes + bias loads (lanes < CH, overlap the row loads) -> slot rows of the first
//   groups -> steady state: process one register buffer while the other's 128-bit loads are in flight.
// L2 priority: table and slot rows are loaded and stored evict-first (orx_ld4_stream / orx_st4_stream); the probes and
// the item bias + slot loads are evict-last (orx_ld_keep), the staging red.adds and the bias stores normal, so that the
// index, the bias and the staging rows are still in L2 when they are reused.
template <int KIND, int OPT, int D, int CH, int MINB, bool PIPE>
__global__ void __launch_bounds__(256, MINB) k_pair_step(const PairArgs a) {
  constexpr int G = (D / 4 < 32) ? D / 4 : 32;  // lanes per triplet
  constexpr int K = D / (4 * G);                // float4 per lane per row
  constexpr int TPW = 32 / G;                   // triplets in flight per warp
  typedef OrxOptSlots<OPT> SL;
  static_assert(CH % TPW == 0, "chunk must be a multiple of the triplets per warp");
  typedef TripRegs<K, SL::S0, SL::S1> Regs;

  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int grp = lane / G, gl = lane % G;
  const int t = warp * CH + lane;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  orx_pdl_wait();

  // ---- ids of triplet t (lanes < CH)
  int u_id = 0, p_id = 0, n_id = 0, du = -1, dp = -1, dn = -1, flags = 0;
  if (lane < CH && t < a.B) {
    u_id = a.uid[t];
    p_id = a.pid[t];
    n_id = a.nid[t];
    flags = (u_id >= 0 && u_id < a.rowsU && p_id >= 0 && p_id < a.rowsI && n_id >= 0 && n_id < a.rowsI) ? 1 : 0;
  }

  // variable rows: need ids + the valid bit only
  auto load_var = [&](int j, Regs& r) {
    const int src = j + grp;
    r.fl = __shfl_sync(ORX_FULL, flags, src) & 1;
    r.uu = __shfl_sync(ORX_FULL, u_id, src);
    r.pp = __shfl_sync(ORX_FULL, p_id, src);
    r.nn = __shfl_sync(ORX_FULL, n_id, src);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int off = (k * G + gl) * 4;
      r.u[k] = r.fl ? orx_ld4_stream(a.U + (int64_t)r.uu * D + off) : z4;
      r.p[k] = r.fl ? orx_ld4_stream(a.I + (int64_t)r.pp * D + off) : z4;
      r.n[k] = r.fl ? orx_ld4_stream(a.I + (int64_t)r.nn * D + off) : z4;
    }
  };
  Regs ra, rb;
  load_var(0, ra);
  if (PIPE && TPW < CH) load_var(TPW, rb);

  // ---- hash probes + item_bias (lanes < CH), overlapping the row loads above; L2 evict-last (orx_ld_keep)
  float bp = 0.f, bn = 0.f, bps0 = 0.f, bps1 = 0.f, bns0 = 0.f, bns1 = 0.f;
  if (flags & 1) {
    const uint32_t cu = orx_hash_find<!SL::STAGE_ONLY, true>(a.hu, u_id, &du);
    const uint32_t cp = orx_hash_find<!SL::STAGE_ONLY, true>(a.hi, p_id, &dp);
    const uint32_t cn = orx_hash_find<!SL::STAGE_ONLY, true>(a.hi, n_id, &dn);
    bp = orx_ld_keep(a.Bv + p_id);
    bn = orx_ld_keep(a.Bv + n_id);
    if (!SL::STAGE_ONLY) {
      flags |= (cu == 1u ? 2 : 0) | (cp == 1u ? 4 : 0) | (cn == 1u ? 8 : 0);
      if (SL::S0) {
        if (flags & 4) bps0 = orx_ld_keep(a.Bs0 + p_id);
        if (flags & 8) bns0 = orx_ld_keep(a.Bs0 + n_id);
      }
      if (SL::S1) {
        if (flags & 4) bps1 = orx_ld_keep(a.Bs1 + p_id);
        if (flags & 8) bns1 = orx_ld_keep(a.Bs1 + n_id);
      }
    }
  }

  // optimizer-slot rows + staging indices: need the probe results
  auto load_slots = [&](int j, Regs& r) {
    const int src = j + grp;
    r.fl = __shfl_sync(ORX_FULL, flags, src);
    r.du = __shfl_sync(ORX_FULL, du, src);
    r.dp = __shfl_sync(ORX_FULL, dp, src);
    r.dn = __shfl_sync(ORX_FULL, dn, src);
    r.bp = __shfl_sync(ORX_FULL, bp, src);
    r.bn = __shfl_sync(ORX_FULL, bn, src);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int off = (k * G + gl) * 4;
      if (SL::S0) {
        r.us0[k] = (r.fl & 2) ? orx_ld4_stream(a.Us0 + (int64_t)r.uu * D + off) : z4;
        r.ps0[k] = (r.fl & 4) ? orx_ld4_stream(a.Is0 + (int64_t)r.pp * D + off) : z4;
        r.ns0[k] = (r.fl & 8) ? orx_ld4_stream(a.Is0 + (int64_t)r.nn * D + off) : z4;
      }
      if (SL::S1) {
        r.us1[k] = (r.fl & 2) ? orx_ld4_stream(a.Us1 + (int64_t)r.uu * D + off) : z4;
        r.ps1[k] = (r.fl & 4) ? orx_ld4_stream(a.Is1 + (int64_t)r.pp * D + off) : z4;
        r.ns1[k] = (r.fl & 8) ? orx_ld4_stream(a.Is1 + (int64_t)r.nn * D + off) : z4;
      }
    }
  };
  load_slots(0, ra);
  if (PIPE && TPW < CH) load_slots(TPW, rb);

  float loss_acc = 0.f, l2_acc = 0.f, g_own = 0.f;

  auto process = [&](int j, Regs& r) {
    float s1 = 0.f, s2 = 0.f, sq = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (KIND == ORX_PAIR_BPR) {
        s1 += dot4(r.u[k], r.p[k]);
        s2 += dot4(r.u[k], r.n[k]);
      } else {
        s1 += sqd4(r.u[k], r.p[k]);
        s2 += sqd4(r.u[k], r.n[k]);
      }
      sq += dot4(r.u[k], r.u[k]) + dot4(r.p[k], r.p[k]) + dot4(r.n[k], r.n[k]);
    }
    l2_acc += sq;  // invalid triplets contribute exact zeros
    s1 = orx_group_sum<G>(s1);
    s2 = orx_group_sum<G>(s2);
    float lt, g;
    pair_score<KIND>(s1, s2, r.bp, r.bn, a.margin, a.c_loss, a.inv_B, &lt, &g);
    const bool v = r.fl & 1;
    if (!v) { lt = 0.f; g = 0.f; }
    if (gl == 0) loss_acc += lt;
    // bias gradient of the positive item: BPR +g, UCML -a  (negative item gets the opposite sign)
    const float gbias = (KIND == ORX_PAIR_BPR) ? g : -g;
#pragma unroll
    for (int q = 0; q < TPW; ++q) {
      const float val = __shfl_sync(ORX_FULL, gbias, q * G);
      if (lane == j + q) g_own = val;
    }
    if (v) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int off = (k * G + gl) * 4;
        float4 gu, gp, gn;
        pair_row_grads<KIND>(g, a.c_l2, r.u[k], r.p[k], r.n[k], &gu, &gp, &gn);
        orx_own_or_stage4<OPT, true>(r.fl & 2, a.U, a.Us0, a.Us1, r.uu, a.gu, r.du, D, off, r.u[k], gu, r.us0[k],
                                     r.us1[k], a.opt);
        orx_own_or_stage4<OPT, true>(r.fl & 4, a.I, a.Is0, a.Is1, r.pp, a.gi, r.dp, D, off, r.p[k], gp, r.ps0[k],
                                     r.ps1[k], a.opt);
        orx_own_or_stage4<OPT, true>(r.fl & 8, a.I, a.Is0, a.Is1, r.nn, a.gi, r.dn, D, off, r.n[k], gn, r.ns0[k],
                                     r.ns1[k], a.opt);
      }
    }
  };

  if (PIPE) {
#pragma unroll 1
    for (int j = 0; j < CH; j += 2 * TPW) {
      process(j, ra);
      if (j + 2 * TPW < CH) {
        load_var(j + 2 * TPW, ra);
        load_slots(j + 2 * TPW, ra);
      }
      if (j + TPW < CH) {
        process(j + TPW, rb);
        if (j + 3 * TPW < CH) {
          load_var(j + 3 * TPW, rb);
          load_slots(j + 3 * TPW, rb);
        }
      }
    }
  } else {
#pragma unroll 1
    for (int j = 0; j < CH; j += TPW) {
      if (j > 0) {
        load_var(j, ra);
        load_slots(j, ra);
      }
      process(j, ra);
    }
  }

  orx_pdl_trigger();
  // ---- item_bias: lane-parallel, one lane per triplet of the chunk
  if (flags & 1) {
    if (flags & 4) {
      __stcg(a.Bv + p_id, orx_apply<OPT>(bp, g_own, bps0, bps1, a.opt));
      if (SL::S0) __stcg(a.Bs0 + p_id, bps0);
      if (SL::S1) __stcg(a.Bs1 + p_id, bps1);
    } else {
      atomicAdd(a.gb + dp, g_own);
    }
    if (flags & 8) {
      __stcg(a.Bv + n_id, orx_apply<OPT>(bn, -g_own, bns0, bns1, a.opt));
      if (SL::S0) __stcg(a.Bs0 + n_id, bns0);
      if (SL::S1) __stcg(a.Bs1 + n_id, bns1);
    } else {
      atomicAdd(a.gb + dn, -g_own);
    }
  }

  // ---- one (loss, l2) partial per block, fixed order => deterministic
  orx_block_partial(loss_acc, l2_acc, a.partials);
}

// Any D (e.g. the example's D=50): one triplet per warp-iteration, lanes stride the row.  MODE 0 = fused step (launched
// with PDL), 1 = forward / explicit (un-fused) gradients into a.d_* / a.g_out (OPT = SGD, unread), table or row form.
// A skipped triplet (bad id) contributes nothing and, in MODE 1, gets zero gradients and g_out = 0.
template <int KIND, int OPT, int MODE>
__global__ void __launch_bounds__(256) k_pair_generic(const PairArgs a) {
  constexpr bool STAGE_ONLY = OrxOptSlots<OPT>::STAGE_ONLY;
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int D = a.D;
  const bool row_form = MODE == 1 && a.ld != 0;
  const int64_t ld = row_form ? a.ld : D;
  float loss_acc = 0.f, l2_acc = 0.f;
  orx_pdl_wait();
  for (int j = 0; j < 8; ++j) {
    const int t = warp * 8 + j;
    if (t >= a.B) break;
    const int uu = a.uid[t], pp = a.pid[t], nn = a.nid[t];
    const bool ok = uu >= 0 && uu < a.rowsU && pp >= 0 && pp < a.rowsI && nn >= 0 && nn < a.rowsI;
    float* ur = a.U + (int64_t)uu * ld;
    float* pr = a.I + (int64_t)pp * ld;
    float* nr = a.I + (int64_t)nn * ld;
    float s1 = 0.f, s2 = 0.f, sq = 0.f, bp = 0.f, bn = 0.f, lt = 0.f, g = 0.f;
    if (ok) {
      for (int d = lane; d < D; d += 32) {
        const float u = ur[d], p = pr[d], n = nr[d];
        if (KIND == ORX_PAIR_BPR) {
          s1 += u * p;
          s2 += u * n;
        } else {
          s1 += (u - p) * (u - p);
          s2 += (u - n) * (u - n);
        }
        sq += u * u + p * p + n * n;
      }
      bp = row_form ? pr[D] : a.Bv[pp];
      bn = row_form ? nr[D] : a.Bv[nn];
    }
    l2_acc += sq;
    s1 = orx_group_sum<32>(s1);
    s2 = orx_group_sum<32>(s2);
    if (ok) pair_score<KIND>(s1, s2, bp, bn, a.margin, a.c_loss, a.inv_B, &lt, &g);
    if (lane == 0) loss_acc += lt;
    const float gbias = (KIND == ORX_PAIR_BPR) ? g : -g;
    if (MODE == 0) {
      if (!ok) continue;
      int du, dp, dn;
      const uint32_t cu = orx_hash_find<!STAGE_ONLY>(a.hu, uu, &du);
      const uint32_t cp = orx_hash_find<!STAGE_ONLY>(a.hi, pp, &dp);
      const uint32_t cn = orx_hash_find<!STAGE_ONLY>(a.hi, nn, &dn);
      const bool fu = !STAGE_ONLY && cu == 1u, fp = !STAGE_ONLY && cp == 1u, fn = !STAGE_ONLY && cn == 1u;
      for (int d = lane; d < D; d += 32) {
        const float u = ur[d], p = pr[d], n = nr[d];
        float gu, gp, gn;
        pair_grads1<KIND>(g, a.c_l2, u, p, n, &gu, &gp, &gn);
        const int64_t ou = (int64_t)uu * D + d, op = (int64_t)pp * D + d, on = (int64_t)nn * D + d;
        if (fu) orx_update1<OPT>(ur + d, a.Us0 + ou, a.Us1 + ou, u, gu, a.opt);
        else atomicAdd(a.gu + (int64_t)du * D + d, gu);
        if (fp) orx_update1<OPT>(pr + d, a.Is0 + op, a.Is1 + op, p, gp, a.opt);
        else atomicAdd(a.gi + (int64_t)dp * D + d, gp);
        if (fn) orx_update1<OPT>(nr + d, a.Is0 + on, a.Is1 + on, n, gn, a.opt);
        else atomicAdd(a.gi + (int64_t)dn * D + d, gn);
      }
      if (lane == 0) {
        if (fp) orx_update1<OPT>(a.Bv + pp, a.Bs0 + pp, a.Bs1 + pp, bp, gbias, a.opt);
        else atomicAdd(a.gb + dp, gbias);
        if (fn) orx_update1<OPT>(a.Bv + nn, a.Bs0 + nn, a.Bs1 + nn, bn, -gbias, a.opt);
        else atomicAdd(a.gb + dn, -gbias);
      }
      continue;
    }
    if (a.d_user || a.d_pos || a.d_neg) {
      for (int d = lane; d < D; d += 32) {
        float gu = 0.f, gp = 0.f, gn = 0.f;
        if (ok) pair_grads1<KIND>(g, a.c_l2, ur[d], pr[d], nr[d], &gu, &gp, &gn);
        if (row_form) {
          if (ok) {
            a.d_user[(int64_t)uu * ld + d] = gu;
            a.d_pos[(int64_t)pp * ld + d] = gp;
            a.d_neg[(int64_t)nn * ld + d] = gn;
          }
        } else {
          const int64_t o = (int64_t)t * D + d;
          if (a.d_user) a.d_user[o] = gu;
          if (a.d_pos) a.d_pos[o] = gp;
          if (a.d_neg) a.d_neg[o] = gn;
        }
      }
    }
    if (lane == 0) {
      if (row_form) {
        if (ok) {   // column D = bias gradient (items) / 0 (users); remaining padding columns = 0
          for (int64_t c = D; c < ld; ++c) {
            a.d_user[(int64_t)uu * ld + c] = 0.f;
            a.d_pos[(int64_t)pp * ld + c] = c == D ? gbias : 0.f;
            a.d_neg[(int64_t)nn * ld + c] = c == D ? -gbias : 0.f;
          }
        }
      } else {
        if (a.d_bp) a.d_bp[t] = gbias;
        if (a.d_bn) a.d_bn[t] = -gbias;
      }
      if (a.g_out) a.g_out[t] = g;
    }
  }
  orx_warp_partial(loss_acc, l2_acc, a.partials);
}

// ---------------------------------------------------------------------------------------
// ADAM_DENSE sweep: Keras-2.0 Adam on IndexedSlices touches EVERY row (SURVEY Q5, "K12").
// One warp per table row; the row's summed gradient comes from the staging buffer via the hash.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_adam_sweep(float* var, float* m, float* v, int64_t rows, int D, OrxHash h,
                                                    const float* gstage, OrxOptDev o) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += nw) {
    int d = -1;
    uint32_t c = 0;
    if (lane == 0) c = orx_hash_find(h, (int32_t)r, &d);
    c = __shfl_sync(ORX_FULL, c, 0);
    d = __shfl_sync(ORX_FULL, d, 0);
    for (int e = lane; e < D; e += 32)
      orx_adam_dense1(var, m, v, r * D + e, c ? gstage[(int64_t)d * D + e] : 0.f, o);
  }
}

// ---------------------------------------------------------------------------------------
// tail: staged rows -> optimizer (once per unique row), zero staging, clear hash, reduce loss
// ---------------------------------------------------------------------------------------

// ta.I == nullptr: no item side (orx_sparse_apply: one table, in the user-side index set); ta.out4 == nullptr: no loss.
template <int OPT>
__global__ void __launch_bounds__(256) k_sparse_tail(const TailArgs a) {
  __shared__ bool last;
  orx_pdl_wait();
  const int nu = *a.hu.counter, ni = a.I ? *a.hi.counter : 0;
  orx_tail_rows<OPT>(a, nu, ni);

  if (blockIdx.x == 0 && a.out4) {
    // deterministic loss reduction; GMF: l2_loss also holds 0.5*sum(w^2) of the PRE-step weight (gmf.py:31-32)
    double l, q;
    orx_block_sum_partials(a.partials, a.n_partials, a.W, a.W ? a.D : 0, &l, &q);
    if (threadIdx.x == 0) {
      a.out4[0] = (float)(l * (double)a.loss_scale);
      a.out4[1] = (float)(0.5 * q);
      a.out4[2] = (float)a.counters[3];
      a.out4[3] = (float)(nu + ni);
    }
    // GMF dense weight: grad = gw + c_l2*w  (gmf.py:31-32), Keras dense apply
    if (a.W) {
      for (int e = threadIdx.x; e < a.D; e += blockDim.x) {
        const float g = a.gw[e] + a.c_l2 * a.W[e];
        if (OrxOptSlots<OPT>::STAGE_ONLY) orx_adam_dense1(a.W, a.Ws0, a.Ws1, e, g, a.opt);
        else orx_update1<OPT>(a.W + e, a.Ws0 + e, a.Ws1 + e, a.W[e], g, a.opt);
        a.gw[e] = 0.f;
      }
    }
  }
  // last block to finish resets the counters (every block has read them by then)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int tk = atomicAdd(a.counters + 2, 1);
    last = (tk == (int)gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x < 4) a.counters[threadIdx.x] = 0;
}

int orx_launch_tail(orx_ctx* c, const TailArgs& ta, int opt_kind, cudaStream_t st) {
  const int grid = c->num_sms * 4;  // ~1-2 staged rows per warp: the tail is a latency chain, not bandwidth
  orx_dispatch_opt(opt_kind, [&](auto O) {
    orx_launch_pdl(k_sparse_tail<decltype(O)::value>, dim3(grid), dim3(256), 0, st, ta);
  });
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

int orx_launch_adam_sweeps(orx_ctx* c, const orx_table_t* user, const orx_table_t* item, const orx_table_t* bias,
                           const OrxHash& hu, const OrxHash& hi, const OrxOptDev& o, cudaStream_t st) {
  struct { const orx_table_t* t; int D; const OrxHash* h; const float* g; } sw[3] = {
      {user, user->dim, &hu, c->gu}, {item, user->dim, &hi, c->gi}, {bias, 1, &hi, c->gb}};
  for (const auto& s : sw) {
    if (!s.t) continue;
    int64_t blocks = (s.t->rows + 7) / 8;
    const int64_t cap = (int64_t)c->num_sms * 16;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    k_adam_sweep<<<(int)blocks, 256, 0, st>>>(s.t->var, s.t->s0, s.t->s1, s.t->rows, s.D, *s.h, s.g, o);
    ORX_LAUNCH_CHECK();
  }
  return ORX_OK;
}

SparseArgs orx_sparse_args(const orx_ctx* c, const orx_table_t* user, const orx_table_t* item, const orx_table_t* bias,
                           const OrxHash& hu, const OrxHash& hi, const OrxOptDev& o) {
  SparseArgs s = {};
  s.U = user->var; s.Us0 = user->s0; s.Us1 = user->s1;
  if (item) { s.I = item->var; s.Is0 = item->s0; s.Is1 = item->s1; }
  if (bias) { s.Bv = bias->var; s.Bs0 = bias->s0; s.Bs1 = bias->s1; }
  s.D = user->dim; s.opt = o; s.hu = hu; s.hi = hi;
  s.gu = c->gu; s.gi = c->gi; s.gb = c->gb;
  return s;
}

int orx_check_step_tables(const orx_table_t* user, const orx_table_t* item, const orx_table_t* bias,
                          const orx_table_t* w, int opt_kind) {
  ORX_REQUIRE(user && item && bias, "null table");
  ORX_REQUIRE(user->var && item->var && bias->var, "null table storage");
  ORX_REQUIRE(user->dim == item->dim && user->dim > 0, "user/item dims must match and be positive");
  ORX_REQUIRE(bias->dim == 1 && bias->rows == item->rows, "item_bias must be [item.rows, 1]");
  ORX_REQUIRE(user->rows > 0 && item->rows > 0 && user->rows <= 0x7fffffffLL && item->rows <= 0x7fffffffLL,
              "row counts must fit int32 ids");
  ORX_REQUIRE(!w || (w->var && w->dim == user->dim), "GMF needs w with dim == D");
  ORX_REQUIRE(orx_opt_slots_ok(opt_kind, {user, item, bias, w}), "optimizer slot rows missing");
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// host dispatch
// ---------------------------------------------------------------------------------------
// D = 128 runs 4 CTAs/SM with a single register buffer (64 registers): the fastest of the variants A/B-tested in
// profiles r1b/r1c/r2a (2-3 CTAs/SM with a register double-buffer, a cp.async shared-memory ring, and a
// "last arriver applies" form without the tail launch were all slower and are gone).  Re-checked on H100 SXM (700 W)
// with the L2 priorities of k_pair_step in place, BPR Adagrad at the bench shape: CH = 16 measured the same as CH = 8,
// 3 CTAs/SM was 1 % slower, and the register double-buffer (PIPE) 1-2 % slower at 2 or 3 CTAs/SM.
template <int KIND, int OPT>
static int launch_pair_step_kind_opt(const PairArgs& pa, cudaStream_t st, OrxStepLaunch* out) {
  constexpr bool LAZY = (OPT == ORX_OPT_ADAM_LAZY);  // 9 rows per triplet: no register double-buffer
  const int blocks = orx_step_blocks(pa.B);
  // k_pair_step writes one (loss, l2) partial per block, k_pair_generic one per warp
  auto go = [&](auto kern, int variant, int minb, int n_partials) {
    *out = {n_partials, variant, minb};
    orx_launch_pdl(kern, dim3(blocks), dim3(256), 0, st, pa);
  };
  constexpr int PV = LAZY ? ORX_VARIANT_STEP : ORX_VARIANT_STEP_PIPE;
  switch (pa.D) {
    case 32: go(k_pair_step<KIND, OPT, 32, 8, 2, !LAZY>, PV, 2, blocks); break;
    case 64: go(k_pair_step<KIND, OPT, 64, 8, 2, !LAZY>, PV, 2, blocks); break;
    case 128:
      if constexpr (LAZY) go(k_pair_step<KIND, OPT, 128, 8, 3, false>, ORX_VARIANT_STEP, 3, blocks);
      else go(k_pair_step<KIND, OPT, 128, 8, 4, false>, ORX_VARIANT_STEP, 4, blocks);
      break;
    case 256: go(k_pair_step<KIND, OPT, 256, 8, 2, !LAZY>, PV, 2, blocks); break;
    default: go(k_pair_generic<KIND, OPT, 0>, ORX_VARIANT_STEP_GENERIC, 0, 8 * blocks); break;
  }
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// ---- pipelined batch index ------------------------------------------------------------------------------------------
// The index of a batch depends only on its ids, so it can be built while the PREVIOUS step's kernels still run: on the
// context's side stream, into one of two "prefetch" index sets (hash tables + counters) that alternate -- set 0 stays
// with everything that builds its index on the caller's stream (pointwise / DLRM / censor / sharded / un-prefetched
// pairwise steps).  The step that consumes a prefetched index waits for it with an event; the set is handed back with
// an event recorded behind that step's tail.
static int side_stream_ensure(orx_ctx* c) {
  if (c->side_stream) return ORX_OK;
  ORX_CUDA(cudaStreamCreateWithFlags(&c->side_stream, cudaStreamNonBlocking));
  ORX_CUDA(cudaEventCreateWithFlags(&c->side_ev, cudaEventDisableTiming));
  for (int i = 0; i < 2; ++i) {
    ORX_CUDA(cudaEventCreateWithFlags(&c->pf_done[i], cudaEventDisableTiming));
    ORX_CUDA(cudaEventCreateWithFlags(&c->pf_free[i], cudaEventDisableTiming));
    ORX_CUDA(cudaEventCreateWithFlags(&c->stage_free[i], cudaEventDisableTiming));
    c->pf_free_valid[i] = c->stage_free_valid[i] = 0;
  }
  return ORX_OK;
}

// a prefetched index nobody consumed: wait for it, reset its counters (the hash itself dies with its epoch)
static int prefetch_drop(orx_ctx* c, cudaStream_t st) {
  if (!c->pf_valid) return ORX_OK;
  const int k = c->pf_set;
  ORX_CUDA(cudaStreamWaitEvent(st, c->pf_done[k], 0));
  ORX_CUDA(cudaMemsetAsync(c->counters + 4 * (1 + k), 0, sizeof(int32_t) * 4, st));
  ORX_CUDA(cudaEventRecord(c->pf_free[k], st));
  c->pf_free_valid[k] = 1;
  c->pf_valid = 0;
  return ORX_OK;
}

// Build the index of (uid, pid, nid) on the side stream.  `after` (may be null) is an event the build must wait for
// (the caller's "ids are final" point); the ids themselves may also be produced on the side stream (host upload).
static int prefetch_issue(orx_ctx* c, const int32_t* uid, const int32_t* pid, const int32_t* nid, int B, int64_t rows_u,
                          int64_t rows_i, int mode) {
  const int k = c->pf_next;
  c->pf_next ^= 1;
  cudaStream_t ss = c->side_stream;
  if (c->pf_free_valid[k]) ORX_CUDA(cudaStreamWaitEvent(ss, c->pf_free[k], 0));   // the step that last used set k is done
  int rc = orx_next_epoch(c, ss);
  if (rc) return rc;
  c->pf_u[k].epoch = c->pf_i[k].epoch = c->epoch;
  k_index_build<<<(3 * B + 255) / 256, 256, 0, ss>>>(c->pf_u[k], c->pf_i[k], uid, rows_u, pid, nid, rows_i, B, mode,
                                                     c->counters + 4 * (1 + k) + 3);
  ORX_LAUNCH_CHECK();
  ORX_CUDA(cudaEventRecord(c->pf_done[k], ss));
  c->pf_valid = 1; c->pf_set = k; c->pf_uid = uid; c->pf_pid = pid; c->pf_nid = nid; c->pf_B = B;
  c->pf_rows_u = rows_u; c->pf_rows_i = rows_i; c->pf_mode = mode;
  return ORX_OK;
}

extern "C" int orx_pairwise_prefetch(orx_handle_t h, const orx_table_t* user, const orx_table_t* item, const int32_t* uid,
                                     const int32_t* pid, const int32_t* nid, int32_t B, int32_t opt_kind, int32_t ids_ready,
                                     orx_stream_t ids_stream) {
  ORX_REQUIRE(h != nullptr && user && item && uid && pid && nid && B > 0, "bad arguments");
  ORX_REQUIRE(orx_opt_kind_ok(opt_kind), "unknown optimizer kind");
  ORX_REQUIRE(!orx_shard_holds_index(h), "a sharded step's announced batch holds this handle's index sets (a prefetch "
                                         "would overwrite one) until its orx_shard_step call");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t is = (cudaStream_t)ids_stream;
  int rc = orx_ensure_workspace(h, B, user->dim);
  if (rc) return rc;
  if ((rc = side_stream_ensure(h))) return rc;
  if ((rc = prefetch_drop(h, is))) return rc;
  if (!ids_ready) {   // the ids are final once everything queued on ids_stream so far has run
    ORX_CUDA(cudaEventRecord(h->side_ev, is));
    ORX_CUDA(cudaStreamWaitEvent(h->side_stream, h->side_ev, 0));
  }
  return prefetch_issue(h, uid, pid, nid, B, user->rows, item->rows, opt_kind == ORX_OPT_ADAM_DENSE ? 1 : 0);
}

int orx_sparse_step(orx_ctx* c, int op, int kind, const orx_table_t* user, const orx_table_t* item,
                    const orx_table_t* bias, const orx_table_t* w, const int32_t* uid, const int32_t* iid,
                    const int32_t* nid, int B, const orx_opt_t* opt, float loss_scale, float c_l2, float* out4,
                    const OrxStepKernel& kernel, cudaStream_t st) {
  ORX_REQUIRE(opt != nullptr && out4 != nullptr, "null opt/out");
  ORX_REQUIRE(orx_opt_kind_ok(opt->kind), "unknown optimizer kind");
  ORX_REQUIRE(B > 0 && uid && iid, "empty batch or null ids");
  int rc = orx_check_step_tables(user, item, bias, w, opt->kind);
  if (rc) return rc;
  const int D = user->dim;
  if ((rc = orx_ensure_workspace(c, B, D))) return rc;
  const bool dense = opt->kind == ORX_OPT_ADAM_DENSE;
  if ((rc = orx_grow((void**)&c->partials, &c->partials_cap, sizeof(float) * 2 * 8 * (size_t)orx_step_blocks(B))))
    return rc;
  orx_prof_mark(c, 0, st);
  // index: a matching prefetched one (side stream, possibly still running), else built here on the caller's stream
  int set = 0;
  if (nid && c->pf_valid && c->pf_uid == uid && c->pf_pid == iid && c->pf_nid == nid && c->pf_B == B &&
      c->pf_rows_u == user->rows && c->pf_rows_i == item->rows && c->pf_mode == (dense ? 1 : 0)) {
    set = 1 + c->pf_set;
    ORX_CUDA(cudaStreamWaitEvent(st, c->pf_done[c->pf_set], 0));
    c->pf_valid = 0;
  } else {
    if (nid && (rc = prefetch_drop(c, st))) return rc;
    if ((rc = orx_launch_index_build(c, uid, user->rows, iid, nid, item->rows, B, dense ? 1 : 0, st))) return rc;
  }
  const OrxHash& HU = set ? c->pf_u[set - 1] : c->hu;
  const OrxHash& HI = set ? c->pf_i[set - 1] : c->hi;
  orx_prof_mark(c, 1, st);
  const SparseArgs s = orx_sparse_args(c, user, item, bias, HU, HI, orx_opt_to_dev(opt));
  OrxStepLaunch L = {};
  if ((rc = kernel(s, c->partials, &L))) return rc;
  orx_log_dispatch(c, op, L.variant, kind, opt->kind, B, D, L.minb, set);
  orx_prof_mark(c, 2, st);
  if (dense && (rc = orx_launch_adam_sweeps(c, user, item, bias, HU, HI, s.opt, st))) return rc;
  TailArgs ta = {s};
  ta.partials = c->partials; ta.n_partials = L.n_partials; ta.loss_scale = loss_scale;
  ta.counters = c->counters + 4 * set; ta.out4 = out4;
  if (w) {
    ta.W = w->var; ta.Ws0 = w->s0; ta.Ws1 = w->s1; ta.gw = c->gw; ta.c_l2 = c_l2;
  }
  rc = orx_launch_tail(c, ta, opt->kind, st);
  if (set) {   // the prefetch set is free again once this tail has run
    ORX_CUDA(cudaEventRecord(c->pf_free[set - 1], st));
    c->pf_free_valid[set - 1] = 1;
  }
  orx_prof_mark(c, 3, st);
  orx_prof_next(c);
  return rc;
}

// The kernel arguments of a pairwise batch (shared part s) over user / item rows rows_u / rows_i; no un-fused outputs.
static PairArgs pair_args(const SparseArgs& s, int64_t rows_u, int64_t rows_i, const int32_t* uid, const int32_t* pid,
                          const int32_t* nid, int B, float margin, float c_loss, float c_l2, float inv_B) {
  PairArgs pa = {s};
  pa.rowsU = rows_u; pa.rowsI = rows_i;
  pa.uid = uid; pa.pid = pid; pa.nid = nid; pa.B = B;
  pa.margin = margin; pa.c_loss = c_loss; pa.c_l2 = c_l2; pa.inv_B = inv_B;
  return pa;
}

static int pairwise_step_impl(orx_ctx* c, int kind, const orx_table_t* user, const orx_table_t* item,
                              const orx_table_t* bias, const int32_t* uid, const int32_t* pid, const int32_t* nid,
                              int B, float margin, float c_loss, float c_l2, const orx_opt_t* opt, float* out4,
                              cudaStream_t st) {
  ORX_REQUIRE(kind == ORX_PAIR_BPR || kind == ORX_PAIR_UCML, "unknown pairwise kind");
  ORX_REQUIRE(nid != nullptr, "empty batch or null ids");
  const float inv_B = 1.0f / (float)B;
  const auto kernel = [&](const SparseArgs& s, float* partials, OrxStepLaunch* out) {
    PairArgs pa = pair_args(s, user->rows, item->rows, uid, pid, nid, B, margin, c_loss, c_l2, inv_B);
    pa.partials = partials;
    return orx_dispatch<ORX_PAIR_BPR, ORX_PAIR_UCML>(kind, [&](auto K) {
      return orx_dispatch_opt(opt->kind, [&](auto O) {
        return launch_pair_step_kind_opt<decltype(K)::value, decltype(O)::value>(pa, st, out);
      });
    });
  };
  return orx_sparse_step(c, ORX_OP_PAIRWISE_STEP, kind, user, item, bias, nullptr, uid, pid, nid, B, opt,
                         kind == ORX_PAIR_BPR ? inv_B : 1.0f, c_l2, out4, kernel, st);
}

extern "C" int orx_pairwise_step(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                                 const orx_table_t* item_bias, const int32_t* uid, const int32_t* pid,
                                 const int32_t* nid, int32_t B, float margin, float c_loss, float c_l2,
                                 const orx_opt_t* opt, float* out4, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_CUDA(cudaSetDevice(h->device));
  return pairwise_step_impl(h, kind, user, item, item_bias, uid, pid, nid, B, margin, c_loss, c_l2, opt, out4,
                            (cudaStream_t)s);
}

// Host-buffer form: the upload of this batch's ids and its index build run on the side stream, i.e. under the previous
// step's kernels whenever the caller enqueues ahead of the GPU; the step kernels and the read-back of out4 stay on `s`.
// The id staging buffers alternate; buffer f is reused only after the step that read it has finished (stage_free[f]).
extern "C" int orx_pairwise_step_host(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                                      const orx_table_t* item_bias, const int32_t* uid_host, const int32_t* pid_host,
                                      const int32_t* nid_host, int32_t B, float margin, float c_loss, float c_l2,
                                      const orx_opt_t* opt, float* out4_host, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(B > 0 && uid_host && pid_host && nid_host && out4_host && user && item && opt, "empty batch or null host buffers");
  ORX_REQUIRE(!orx_shard_holds_index(h), "a sharded step's announced batch holds this handle's index sets (this entry "
                                         "point prefetches into one) until its orx_shard_step call");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  int rc;
  for (int i = 0; i < 2; ++i)
    if ((rc = orx_grow((void**)&h->ids_stage[i], &h->stage_cap[i], sizeof(int32_t) * 3 * (size_t)B))) return rc;
  if ((rc = orx_ensure_workspace(h, B, user->dim))) return rc;
  if ((rc = side_stream_ensure(h))) return rc;
  if ((rc = prefetch_drop(h, st))) return rc;
  const uint32_t f = (h->stage_flip++) & 1u;
  int32_t* ids = h->ids_stage[f];
  cudaStream_t ss = h->side_stream;
  if (h->stage_free_valid[f]) ORX_CUDA(cudaStreamWaitEvent(ss, h->stage_free[f], 0));
  // three copies: the caller's arrays are separate (pinned) allocations even when they happen to be adjacent
  ORX_CUDA(cudaMemcpyAsync(ids, uid_host, sizeof(int32_t) * B, cudaMemcpyHostToDevice, ss));
  ORX_CUDA(cudaMemcpyAsync(ids + B, pid_host, sizeof(int32_t) * B, cudaMemcpyHostToDevice, ss));
  ORX_CUDA(cudaMemcpyAsync(ids + 2 * (int64_t)B, nid_host, sizeof(int32_t) * B, cudaMemcpyHostToDevice, ss));
  if ((rc = prefetch_issue(h, ids, ids + B, ids + 2 * (int64_t)B, B, user->rows, item->rows,
                           opt->kind == ORX_OPT_ADAM_DENSE ? 1 : 0)))
    return rc;
  rc = pairwise_step_impl(h, kind, user, item, item_bias, ids, ids + B, ids + 2 * (int64_t)B, B, margin, c_loss, c_l2,
                          opt, h->out_stage[f], st);
  if (rc) return rc;
  ORX_CUDA(cudaEventRecord(h->stage_free[f], st));
  h->stage_free_valid[f] = 1;
  ORX_CUDA(cudaMemcpyAsync(out4_host, h->out_stage[f], sizeof(float) * 4, cudaMemcpyDeviceToHost, st));
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// forward only / explicit gradients (un-fused; parity tests and the lazy-handle fallback)
// ---------------------------------------------------------------------------------------
__global__ void k_reduce_partials(const float* partials, int n, float loss_scale, float* out4) {
  double l, q;
  orx_block_sum_partials(partials, n, nullptr, 0, &l, &q);
  if (threadIdx.x == 0) {
    out4[0] = (float)(l * (double)loss_scale);
    out4[1] = (float)(0.5 * q);
    out4[2] = 0.f;
    out4[3] = 0.f;
  }
}

int orx_launch_reduce_partials(const float* partials, int n, float loss_scale, float* out4, cudaStream_t st) {
  k_reduce_partials<<<1, 256, 0, st>>>(partials, n, loss_scale, out4);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

int orx_sparse_unfused(orx_ctx* c, int B, float loss_scale, float* out4,
                       const std::function<void(float* partials, int blocks)>& launch, cudaStream_t st) {
  const int blocks = orx_step_blocks(B);
  int rc = orx_grow((void**)&c->partials, &c->partials_cap, sizeof(float) * 2 * 8 * (size_t)blocks);
  if (rc) return rc;
  launch(c->partials, blocks);
  ORX_LAUNCH_CHECK();
  if (!out4) return ORX_OK;
  return orx_launch_reduce_partials(c->partials, 8 * blocks, loss_scale, out4, st);
}

// k_pair_generic MODE 1 over the batch of pa (kind already validated) and, when out4 is given, its (loss, l2) reduced
// into out4: the loss scaled by inv_B for BPR (mean), summed for UCML.
static int pair_unfused(orx_ctx* c, int kind, PairArgs pa, float* out4, cudaStream_t st) {
  const auto launch = [&](float* partials, int blocks) {
    pa.partials = partials;
    orx_dispatch<ORX_PAIR_BPR, ORX_PAIR_UCML>(kind, [&](auto K) {
      k_pair_generic<decltype(K)::value, ORX_OPT_SGD, 1><<<blocks, 256, 0, st>>>(pa);
    });
  };
  return orx_sparse_unfused(c, pa.B, kind == ORX_PAIR_BPR ? pa.inv_B : 1.f, out4, launch, st);
}

static int pair_fwd_grad(orx_ctx* c, int kind, const orx_table_t* user, const orx_table_t* item,
                         const orx_table_t* bias, const int32_t* uid, const int32_t* pid, const int32_t* nid, int B,
                         float margin, float c_loss, float c_l2, float* d_user, float* d_pos, float* d_neg,
                         float* d_bp, float* d_bn, float* g_out, float* out4, cudaStream_t st) {
  ORX_REQUIRE(kind == ORX_PAIR_BPR || kind == ORX_PAIR_UCML, "unknown pairwise kind");
  ORX_REQUIRE(B > 0 && uid && pid && nid, "empty batch or null ids");
  int rc = orx_check_step_tables(user, item, bias, nullptr, ORX_OPT_SGD);
  if (rc) return rc;
  const SparseArgs s = orx_sparse_args(c, user, item, bias, c->hu, c->hi, OrxOptDev{});
  PairArgs a = pair_args(s, user->rows, item->rows, uid, pid, nid, B, margin, c_loss, c_l2, 1.0f / (float)B);
  a.d_user = d_user; a.d_pos = d_pos; a.d_neg = d_neg; a.d_bp = d_bp; a.d_bn = d_bn; a.g_out = g_out;
  return pair_unfused(c, kind, a, out4, st);
}

extern "C" int orx_pairwise_fwd(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                                const orx_table_t* item_bias, const int32_t* uid, const int32_t* pid,
                                const int32_t* nid, int32_t B, float margin, float* out4, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && out4 != nullptr, "null handle/out");
  ORX_CUDA(cudaSetDevice(h->device));
  return pair_fwd_grad(h, kind, user, item, item_bias, uid, pid, nid, B, margin, 1.f, 1.f, nullptr, nullptr, nullptr,
                       nullptr, nullptr, nullptr, out4, (cudaStream_t)s);
}

extern "C" int orx_pairwise_grad(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                                 const orx_table_t* item_bias, const int32_t* uid, const int32_t* pid,
                                 const int32_t* nid, int32_t B, float margin, float c_loss, float c_l2, float* d_user,
                                 float* d_pos, float* d_neg, float* d_bp, float* d_bn, float* g_out, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_CUDA(cudaSetDevice(h->device));
  return pair_fwd_grad(h, kind, user, item, item_bias, uid, pid, nid, B, margin, c_loss, c_l2, d_user, d_pos, d_neg,
                       d_bp, d_bn, g_out, nullptr, (cudaStream_t)s);
}

extern "C" int orx_pairwise_grad_rows(orx_handle_t h, int32_t kind, const float* rows, int64_t ld, int32_t dim,
                                      const int32_t* uslot, const int32_t* pslot, const int32_t* nslot, int32_t B,
                                      float margin, float c_loss, float c_l2, float inv_B, float* d_rows, float* out4,
                                      orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && rows && uslot && pslot && nslot && d_rows && out4, "null pointer");
  ORX_REQUIRE(kind == ORX_PAIR_BPR || kind == ORX_PAIR_UCML, "unknown pairwise kind");
  ORX_REQUIRE(B > 0 && dim > 0 && ld > dim, "bad sizes (ld must exceed dim: the bias lives in column dim)");
  ORX_CUDA(cudaSetDevice(h->device));
  SparseArgs r = {};
  r.U = r.I = const_cast<float*>(rows);   // read only in MODE 1
  r.D = dim;
  PairArgs a = pair_args(r, 3 * (int64_t)B, 3 * (int64_t)B, uslot, pslot, nslot, B, margin, c_loss, c_l2, inv_B);
  a.d_user = a.d_pos = a.d_neg = d_rows;
  a.ld = ld;
  return pair_unfused(h, kind, a, out4, (cudaStream_t)s);
}
