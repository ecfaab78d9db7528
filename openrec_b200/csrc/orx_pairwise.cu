// orx_pairwise.cu -- BPR / UCML fused training step (K1/K2), its batch index (K9), the tail and the step driver shared
// with orx_pointwise.cu.
//
// Reference path replaced (paths relative to the reference repo):
//   openrec/tf2/recommenders/bpr.py:21-37, ucml.py:21-42, modules/pairwise_log_loss.py:15-34
//   + tape.gradient + optimizer.apply_gradients (tf2_examples/bpr_citeulike.py:33-39).
//
// Synchronous-batch semantics in three launches on one stream:
//   1. k_index_build : hash every id of the batch's valid triplets; rows hit more than once get a "staging" slot.
//      A batch prefetched on the side stream (orx_pairwise_prefetch, orx_pairwise_step_host) is also resolved there:
//      k_index_resolve writes each triplet's probe answers as one record {flags, du, dp, dn}, which k_pair_step
//      reads in place of probing the index.
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

// The probe answers of a prefetched pairwise batch, once its index (hu, hi) is complete: one thread per triplet writes
// res[t] = {flags, du, dp, dn} exactly as k_pair_step's probes would find them -- flags bit 0: the three ids are in range;
// bits 1/2/3: the user / pos / neg row is referenced once in the batch (owned by this triplet); du / dp / dn: staging
// index, -1 for an owned row.  Mode 1 (ADAM_DENSE) stages every row: all three indices, no owned bits.  An invalid
// triplet gets {0, -1, -1, -1}.
__global__ void k_index_resolve(OrxHash hu, OrxHash hi, const int32_t* __restrict__ uid, const int32_t* __restrict__ pid,
                                const int32_t* __restrict__ nid, int64_t rows_u, int64_t rows_i, int n, int mode,
                                int4* __restrict__ res) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int32_t u = uid[t], p = pid[t], q = nid[t];
  int4 r = make_int4(0, -1, -1, -1);
  if (u >= 0 && (int64_t)u < rows_u && p >= 0 && (int64_t)p < rows_i && q >= 0 && (int64_t)q < rows_i) {
    if (mode == 1) {
      orx_hash_find(hu, u, &r.y);
      orx_hash_find(hi, p, &r.z);
      orx_hash_find(hi, q, &r.w);
      r.x = 1;
    } else {
      const uint32_t cu = orx_hash_find<true>(hu, u, &r.y);
      const uint32_t cp = orx_hash_find<true>(hi, p, &r.z);
      const uint32_t cn = orx_hash_find<true>(hi, q, &r.w);
      r.x = 1 | (cu == 1u ? 2 : 0) | (cp == 1u ? 4 : 0) | (cn == 1u ? 8 : 0);
    }
  }
  res[t] = r;
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
  OrxIndexSet& s = c->set[0];
  int rc = orx_take_epoch(s.u, st);
  if (rc) return rc;
  k_index_build_strided<<<(n + 255) / 256, 256, 0, st>>>(s.u, a, stride, rows, n, stage_all ? 1 : 0, s.ctl + 3);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

int orx_launch_index_build(orx_ctx* c, const int32_t* a, int64_t rows_a, const int32_t* b0, const int32_t* b1,
                           int64_t rows_b, int32_t n, int mode, cudaStream_t st) {
  const int total = (b1 ? 3 : 2) * n;
  if (total <= 0) return ORX_OK;
  OrxIndexSet& s = c->set[0];
  int rc;
  if ((rc = orx_take_epoch(s.u, st)) || (rc = orx_take_epoch(s.i, st))) return rc;
  k_index_build<<<(total + 255) / 256, 256, 0, st>>>(s.u, s.i, a, rows_a, b0, b1, rows_b, n, mode, s.ctl + 3);
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
  float uacc, pacc, nacc;         // ROWWISE_ADAGRAD: the rows' accumulators (one scalar per row)
  int fl, uu, pp, nn, du, dp, dn;
};

// flags: bit0 triplet valid, bit1/2/3 user/pos/neg row owned by this triplet (fast path)
//
// One warp owns CH consecutive triplets.  Order of issue inside a warp (latency first):
//   ids (coalesced, lanes < CH) -> variable rows of the first one/two triplet groups (they need only
//   the ids) -> hash probes + bias loads (lanes < CH, overlap the row loads) -> slot rows of the first
//   groups -> steady state: process one register buffer while the other's 128-bit loads are in flight.
//   With a.res (a prefetched batch) the ids come with their record, so there are no probes: the slot rows of the first
//   groups follow their variable rows and the bias loads without waiting for anything.
// L2 priority: table and slot rows are loaded and stored evict-first (orx_ld4_stream / orx_st4_stream); the probes and
// the item bias + slot loads are evict-last (orx_ld_keep), the staging red.adds and the bias stores normal, so that the
// index, the bias and the staging rows are still in L2 when they are reused.
// T: the storage of the user and item tables, float or bf16 bits (uint16_t; rows 8-byte aligned, rounded on store with
// the keys a.srk).  Slot rows, item bias and staging rows are float either way.
template <int KIND, int OPT, int D, int CH, int MINB, bool PIPE, typename T = float>
__global__ void __launch_bounds__(256, MINB) k_pair_step(const PairArgs a) {
  constexpr int G = (D / 4 < 32) ? D / 4 : 32;  // lanes per triplet
  constexpr int K = D / (4 * G);                // float4 per lane per row
  constexpr int TPW = 32 / G;                   // triplets in flight per warp
  typedef OrxOptSlots<OPT> SL;
  typedef OrxOptSlots<SL::ELEM> BL;             // the item bias's optimizer (element-wise)
  static_assert(CH % TPW == 0, "chunk must be a multiple of the triplets per warp");
  typedef TripRegs<K, SL::S0, SL::S1> Regs;

  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int grp = lane / G, gl = lane % G;
  const int t = warp * CH + lane;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  orx_pdl_wait();

  // ---- ids of triplet t (lanes < CH), and its record when the index was resolved ahead (a.res)
  int u_id = 0, p_id = 0, n_id = 0, du = -1, dp = -1, dn = -1, flags = 0;
  if (lane < CH && t < a.B) {
    u_id = a.uid[t];
    p_id = a.pid[t];
    n_id = a.nid[t];
    if (a.res) {
      const int4 r = __ldcs(a.res + t);
      flags = r.x;
      du = r.y;
      dp = r.z;
      dn = r.w;
    } else {
      flags = (u_id >= 0 && u_id < a.rowsU && p_id >= 0 && p_id < a.rowsI && n_id >= 0 && n_id < a.rowsI) ? 1 : 0;
    }
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
      r.u[k] = r.fl ? orx_ld4_stream(reinterpret_cast<const T*>(a.U) + (int64_t)r.uu * D + off) : z4;
      r.p[k] = r.fl ? orx_ld4_stream(reinterpret_cast<const T*>(a.I) + (int64_t)r.pp * D + off) : z4;
      r.n[k] = r.fl ? orx_ld4_stream(reinterpret_cast<const T*>(a.I) + (int64_t)r.nn * D + off) : z4;
    }
  };
  Regs ra, rb;
  load_var(0, ra);
  if (PIPE && TPW < CH) load_var(TPW, rb);

  // ---- hash probes (no a.res) + item_bias (lanes < CH), overlapping the row loads above; L2 evict-last (orx_ld_keep)
  float bp = 0.f, bn = 0.f, bps0 = 0.f, bps1 = 0.f, bns0 = 0.f, bns1 = 0.f;
  if (flags & 1) {
    uint32_t cu = 0, cp = 0, cn = 0;
    if (!a.res) {
      cu = orx_hash_find<!SL::STAGE_ONLY, true>(a.hu, u_id, &du);
      cp = orx_hash_find<!SL::STAGE_ONLY, true>(a.hi, p_id, &dp);
      cn = orx_hash_find<!SL::STAGE_ONLY, true>(a.hi, n_id, &dn);
    }
    bp = orx_ld_keep(a.Bv + p_id);
    bn = orx_ld_keep(a.Bv + n_id);
    if (!SL::STAGE_ONLY) {
      if (!a.res) flags |= (cu == 1u ? 2 : 0) | (cp == 1u ? 4 : 0) | (cn == 1u ? 8 : 0);
      if (BL::S0) {
        if (flags & 4) bps0 = orx_ld_keep(a.Bs0 + p_id);
        if (flags & 8) bns0 = orx_ld_keep(a.Bs0 + n_id);
      }
      if (BL::S1) {
        if (flags & 4) bps1 = orx_ld_keep(a.Bs1 + p_id);
        if (flags & 8) bns1 = orx_ld_keep(a.Bs1 + n_id);
      }
    }
  }

  // optimizer-slot rows + staging indices: need the probe results (or the record).  The item bias is shuffled only where
  // the score needs it, so that no row load waits for a bias load.
  auto load_slots = [&](int j, Regs& r) {
    const int src = j + grp;
    r.fl = __shfl_sync(ORX_FULL, flags, src);
    r.du = __shfl_sync(ORX_FULL, du, src);
    r.dp = __shfl_sync(ORX_FULL, dp, src);
    r.dn = __shfl_sync(ORX_FULL, dn, src);
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
    if (SL::ROW) {
      r.uacc = (r.fl & 2) ? __ldcg(a.Us0 + r.uu) : 0.f;
      r.pacc = (r.fl & 4) ? __ldcg(a.Is0 + r.pp) : 0.f;
      r.nacc = (r.fl & 8) ? __ldcg(a.Is0 + r.nn) : 0.f;
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
    pair_score<KIND>(s1, s2, __shfl_sync(ORX_FULL, bp, j + grp), __shfl_sync(ORX_FULL, bn, j + grp), a.margin, a.c_loss,
                     a.inv_B, &lt, &g);
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
    if constexpr (SL::ROW) {
      // each row's sum of squared gradients over its G lanes (k in order, then the fixed xor tree), taken outside
      // `if (v)`: v is per triplet group, the shuffles need the whole warp.  An invalid triplet's gradients are zeros.
      float su = 0.f, sp = 0.f, sn = 0.f;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        float4 gu, gp, gn;
        pair_row_grads<KIND>(g, a.c_l2, r.u[k], r.p[k], r.n[k], &gu, &gp, &gn);
        su += orx_sq4(gu);
        sp += orx_sq4(gp);
        sn += orx_sq4(gn);
      }
      su = orx_group_sum<G>(su);
      sp = orx_group_sum<G>(sp);
      sn = orx_group_sum<G>(sn);
      const float fu = orx_row_scale(r.uacc, su, D, a.opt), fp = orx_row_scale(r.pacc, sp, D, a.opt),
                  fn = orx_row_scale(r.nacc, sn, D, a.opt);
      if (v) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
          const int off = (k * G + gl) * 4;
          float4 gu, gp, gn;
          pair_row_grads<KIND>(g, a.c_l2, r.u[k], r.p[k], r.n[k], &gu, &gp, &gn);
          orx_own_or_stage4_row<true>(r.fl & 2, reinterpret_cast<T*>(a.U), r.uu, a.gu, r.du, D, off, r.u[k], gu, fu,
                                      a.opt, a.srk[0]);
          orx_own_or_stage4_row<true>(r.fl & 4, reinterpret_cast<T*>(a.I), r.pp, a.gi, r.dp, D, off, r.p[k], gp, fp,
                                      a.opt, a.srk[1]);
          orx_own_or_stage4_row<true>(r.fl & 8, reinterpret_cast<T*>(a.I), r.nn, a.gi, r.dn, D, off, r.n[k], gn, fn,
                                      a.opt, a.srk[1]);
        }
        if (gl == 0) {
          if (r.fl & 2) __stcg(a.Us0 + r.uu, r.uacc);
          if (r.fl & 4) __stcg(a.Is0 + r.pp, r.pacc);
          if (r.fl & 8) __stcg(a.Is0 + r.nn, r.nacc);
        }
      }
    } else if (v) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int off = (k * G + gl) * 4;
        float4 gu, gp, gn;
        pair_row_grads<KIND>(g, a.c_l2, r.u[k], r.p[k], r.n[k], &gu, &gp, &gn);
        orx_own_or_stage4<OPT, true>(r.fl & 2, reinterpret_cast<T*>(a.U), a.Us0, a.Us1, r.uu, a.gu, r.du, D, off,
                                     r.u[k], gu, r.us0[k], r.us1[k], a.opt, a.srk[0]);
        orx_own_or_stage4<OPT, true>(r.fl & 4, reinterpret_cast<T*>(a.I), a.Is0, a.Is1, r.pp, a.gi, r.dp, D, off,
                                     r.p[k], gp, r.ps0[k], r.ps1[k], a.opt, a.srk[1]);
        orx_own_or_stage4<OPT, true>(r.fl & 8, reinterpret_cast<T*>(a.I), a.Is0, a.Is1, r.nn, a.gi, r.dn, D, off,
                                     r.n[k], gn, r.ns0[k], r.ns1[k], a.opt, a.srk[1]);
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
      __stcg(a.Bv + p_id, orx_apply<SL::ELEM>(bp, g_own, bps0, bps1, a.opt));
      if (BL::S0) __stcg(a.Bs0 + p_id, bps0);
      if (BL::S1) __stcg(a.Bs1 + p_id, bps1);
    } else {
      atomicAdd(a.gb + dp, g_own);
    }
    if (flags & 8) {
      __stcg(a.Bv + n_id, orx_apply<SL::ELEM>(bn, -g_own, bns0, bns1, a.opt));
      if (BL::S0) __stcg(a.Bs0 + n_id, bns0);
      if (BL::S1) __stcg(a.Bs1 + n_id, bns1);
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
// T as in k_pair_step (MODE 1 of a bf16 table: the table form only).
template <int KIND, int OPT, int MODE, typename T = float>
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
    T* ur = reinterpret_cast<T*>(a.U) + (int64_t)uu * ld;
    T* pr = reinterpret_cast<T*>(a.I) + (int64_t)pp * ld;
    T* nr = reinterpret_cast<T*>(a.I) + (int64_t)nn * ld;
    const uint32_t rku = orx_sr_row(a.srk[0], uu), rkp = orx_sr_row(a.srk[1], pp), rkn = orx_sr_row(a.srk[1], nn);
    float s1 = 0.f, s2 = 0.f, sq = 0.f, bp = 0.f, bn = 0.f, lt = 0.f, g = 0.f;
    if (ok) {
      for (int d = lane; d < D; d += 32) {
        const float u = orx_ld1(ur + d), p = orx_ld1(pr + d), n = orx_ld1(nr + d);
        if (KIND == ORX_PAIR_BPR) {
          s1 += u * p;
          s2 += u * n;
        } else {
          s1 += (u - p) * (u - p);
          s2 += (u - n) * (u - n);
        }
        sq += u * u + p * p + n * n;
      }
      bp = row_form ? orx_ld1(pr + D) : a.Bv[pp];
      bn = row_form ? orx_ld1(nr + D) : a.Bv[nn];
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
      if constexpr (OrxOptSlots<OPT>::ROW) {
        // each owned row's sum of squared gradients first (lane-strided, then the xor tree: ok is warp-uniform), then
        // the apply in a second pass over the rows
        float su = 0.f, sp = 0.f, sn = 0.f;
        for (int d = lane; d < D; d += 32) {
          float gu, gp, gn;
          pair_grads1<KIND>(g, a.c_l2, orx_ld1(ur + d), orx_ld1(pr + d), orx_ld1(nr + d), &gu, &gp, &gn);
          su += gu * gu;
          sp += gp * gp;
          sn += gn * gn;
        }
        su = orx_group_sum<32>(su);
        sp = orx_group_sum<32>(sp);
        sn = orx_group_sum<32>(sn);
        float au = fu ? a.Us0[uu] : 0.f, ap = fp ? a.Is0[pp] : 0.f, an = fn ? a.Is0[nn] : 0.f;
        const float xu = orx_row_scale(au, su, D, a.opt), xp = orx_row_scale(ap, sp, D, a.opt),
                    xn = orx_row_scale(an, sn, D, a.opt);
        for (int d = lane; d < D; d += 32) {
          const float u = orx_ld1(ur + d), p = orx_ld1(pr + d), n = orx_ld1(nr + d);
          float gu, gp, gn;
          pair_grads1<KIND>(g, a.c_l2, u, p, n, &gu, &gp, &gn);
          if (fu) orx_st1(ur + d, orx_row_apply1(u, gu, xu, a.opt), rku, d);
          else atomicAdd(a.gu + (int64_t)du * D + d, gu);
          if (fp) orx_st1(pr + d, orx_row_apply1(p, gp, xp, a.opt), rkp, d);
          else atomicAdd(a.gi + (int64_t)dp * D + d, gp);
          if (fn) orx_st1(nr + d, orx_row_apply1(n, gn, xn, a.opt), rkn, d);
          else atomicAdd(a.gi + (int64_t)dn * D + d, gn);
        }
        if (lane == 0) {
          if (fu) a.Us0[uu] = au;
          if (fp) a.Is0[pp] = ap;
          if (fn) a.Is0[nn] = an;
          if (fp) orx_update1<ORX_OPT_ADAGRAD>(a.Bv + pp, a.Bs0 + pp, nullptr, bp, gbias, a.opt);
          else atomicAdd(a.gb + dp, gbias);
          if (fn) orx_update1<ORX_OPT_ADAGRAD>(a.Bv + nn, a.Bs0 + nn, nullptr, bn, -gbias, a.opt);
          else atomicAdd(a.gb + dn, -gbias);
        }
      } else {
        for (int d = lane; d < D; d += 32) {
          const float u = orx_ld1(ur + d), p = orx_ld1(pr + d), n = orx_ld1(nr + d);
          float gu, gp, gn;
          pair_grads1<KIND>(g, a.c_l2, u, p, n, &gu, &gp, &gn);
          const int64_t ou = (int64_t)uu * D + d, op = (int64_t)pp * D + d, on = (int64_t)nn * D + d;
          if (fu) orx_update1<OPT>(ur + d, a.Us0 + ou, a.Us1 + ou, u, gu, a.opt, rku, d);
          else atomicAdd(a.gu + (int64_t)du * D + d, gu);
          if (fp) orx_update1<OPT>(pr + d, a.Is0 + op, a.Is1 + op, p, gp, a.opt, rkp, d);
          else atomicAdd(a.gi + (int64_t)dp * D + d, gp);
          if (fn) orx_update1<OPT>(nr + d, a.Is0 + on, a.Is1 + on, n, gn, a.opt, rkn, d);
          else atomicAdd(a.gi + (int64_t)dn * D + d, gn);
        }
        if (lane == 0) {
          if (fp) orx_update1<OPT>(a.Bv + pp, a.Bs0 + pp, a.Bs1 + pp, bp, gbias, a.opt);
          else atomicAdd(a.gb + dp, gbias);
          if (fn) orx_update1<OPT>(a.Bv + nn, a.Bs0 + nn, a.Bs1 + nn, bn, -gbias, a.opt);
          else atomicAdd(a.gb + dn, -gbias);
        }
      }
      continue;
    }
    if (a.d_user || a.d_pos || a.d_neg) {
      for (int d = lane; d < D; d += 32) {
        float gu = 0.f, gp = 0.f, gn = 0.f;
        if (ok) pair_grads1<KIND>(g, a.c_l2, orx_ld1(ur + d), orx_ld1(pr + d), orx_ld1(nr + d), &gu, &gp, &gn);
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
// T: the table's storage; kt its rounding key (bf16).
template <typename T>
__global__ void __launch_bounds__(256) k_adam_sweep(T* var, float* m, float* v, int64_t rows, int D, OrxHash h,
                                                    const float* gstage, OrxOptDev o, uint32_t kt) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += nw) {
    int d = -1;
    uint32_t c = 0;
    if (lane == 0) c = orx_hash_find(h, (int32_t)r, &d);
    c = __shfl_sync(ORX_FULL, c, 0);
    d = __shfl_sync(ORX_FULL, d, 0);
    const uint32_t rk = orx_sr_row(kt, r);
    for (int e = lane; e < D; e += 32)
      orx_adam_dense1(var, m, v, r * D + e, c ? gstage[(int64_t)d * D + e] : 0.f, o, rk, e);
  }
}

// ---------------------------------------------------------------------------------------
// tail: staged rows -> optimizer (once per unique row), zero staging, clear hash, reduce loss
// ---------------------------------------------------------------------------------------

// ta.I == nullptr: no item side (orx_sparse_apply: one table, in the user-side index set); ta.out4 == nullptr: no loss.
// T: the storage of the user / item tables (float, or bf16 bits with VEC meaning 8-byte aligned rows).
template <int OPT, bool VEC, typename T = float>
__global__ void __launch_bounds__(256) k_sparse_tail(const TailArgs a) {
  __shared__ bool last;
  orx_pdl_wait();
  const int nu = *a.hu.counter, ni = a.I ? *a.hi.counter : 0;
  if constexpr (OrxOptSlots<OPT>::ROW) orx_tail_rows_rowwise<VEC, T>(a, nu, ni);
  else orx_tail_rows<OPT, VEC, T>(a, nu, ni);

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
    // GMF dense weight: grad = gw + c_l2*w  (gmf.py:31-32), Keras dense apply (element-wise ADAGRAD under ROWWISE)
    if (a.W) {
      for (int e = threadIdx.x; e < a.D; e += blockDim.x) {
        const float g = a.gw[e] + a.c_l2 * a.W[e];
        if (OrxOptSlots<OPT>::STAGE_ONLY) orx_adam_dense1(a.W, a.Ws0, a.Ws1, e, g, a.opt);
        else orx_update1<OrxOptSlots<OPT>::ELEM>(a.W + e, a.Ws0 + e, a.Ws1 + e, a.W[e], g, a.opt);
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

int orx_launch_tail(orx_ctx* c, const TailArgs& ta, int opt_kind, cudaStream_t st, bool bf16) {
  const int grid = c->num_sms * 4;  // ~1-2 staged rows per warp: the tail is a latency chain, not bandwidth
  // a row-wise accumulator is read as scalars: only the table rows decide; bf16 rows move 8 bytes at a time
  const bool rows_ok = bf16 ? orx_aligned8(ta.U, ta.I) : orx_aligned16(ta.U, ta.I);
  const bool vec = opt_kind == ORX_OPT_ROWWISE_ADAGRAD ? rows_ok : rows_ok && orx_aligned16(ta.Us0, ta.Us1, ta.Is0, ta.Is1);
  orx_dispatch_opt(opt_kind, [&](auto O) {
    orx_dispatch<0, 1>(vec ? 1 : 0, [&](auto V) {
      if (bf16)
        orx_launch_pdl(k_sparse_tail<decltype(O)::value, decltype(V)::value == 1, uint16_t>, dim3(grid), dim3(256), 0,
                       st, ta);
      else
        orx_launch_pdl(k_sparse_tail<decltype(O)::value, decltype(V)::value == 1>, dim3(grid), dim3(256), 0, st, ta);
    });
  });
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

int orx_launch_adam_sweeps(orx_ctx* c, const orx_table_t* user, const orx_table_t* item, const orx_table_t* bias,
                           const OrxIndexSet& ix, const OrxOptDev& o, cudaStream_t st, const uint32_t* srk) {
  struct { const orx_table_t* t; int D; const OrxHash* h; const float* g; int k; } sw[3] = {
      {user, user->dim, &ix.u, c->gu, 0}, {item, user->dim, &ix.i, c->gi, 1}, {bias, 1, &ix.i, c->gb, -1}};
  for (const auto& s : sw) {
    if (!s.t) continue;
    int64_t blocks = (s.t->rows + 7) / 8;
    const int64_t cap = (int64_t)c->num_sms * 16;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    if (srk && s.k >= 0)   // a bf16 user / item table (the bias is float)
      k_adam_sweep<<<(int)blocks, 256, 0, st>>>(reinterpret_cast<uint16_t*>(s.t->var), s.t->s0, s.t->s1, s.t->rows,
                                                s.D, *s.h, s.g, o, srk[s.k]);
    else
      k_adam_sweep<<<(int)blocks, 256, 0, st>>>(s.t->var, s.t->s0, s.t->s1, s.t->rows, s.D, *s.h, s.g, o, 0u);
    ORX_LAUNCH_CHECK();
  }
  return ORX_OK;
}

SparseArgs orx_sparse_args(const orx_ctx* c, const orx_table_t* user, const orx_table_t* item, const orx_table_t* bias,
                           const OrxIndexSet& ix, const OrxOptDev& o) {
  SparseArgs s = {};
  s.U = user->var; s.Us0 = user->s0; s.Us1 = user->s1;
  if (item) { s.I = item->var; s.Is0 = item->s0; s.Is1 = item->s1; }
  if (bias) { s.Bv = bias->var; s.Bs0 = bias->s0; s.Bs1 = bias->s1; }
  s.D = user->dim; s.opt = o; s.hu = ix.u; s.hi = ix.i;
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
// T = uint16_t: bf16 user / item tables, which take the same variants (and, like fp32, k_pair_generic when a table's
// base is off the boundary its row path needs: 8 bytes for bf16 rows, 16 for float slot rows).
template <int KIND, int OPT, typename T = float>
static int launch_pair_step_kind_opt(const PairArgs& pa, cudaStream_t st, OrxStepLaunch* out) {
  constexpr bool LAZY = (OPT == ORX_OPT_ADAM_LAZY);  // 9 rows per triplet: no register double-buffer
  const int blocks = orx_step_blocks(pa.B);
  // k_pair_step writes one (loss, l2) partial per block, k_pair_generic one per warp
  auto go = [&](auto kern, int variant, int minb, int n_partials) {
    *out = {n_partials, variant, minb};
    orx_launch_pdl(kern, dim3(blocks), dim3(256), 0, st, pa);
  };
  // MOMENTUM (NESTEROV too) keeps ADAGRAD's slot rows, but under -Xptxas -v ADAGRAD's D = 128 bound (four CTAs/SM,
  // 64 registers) spills it, and so does PIPE at D = 256 (as it spills ADAGRAD).
  // It therefore takes PIPE at D = 32 and 64, three CTAs/SM at D = 128 and one register buffer at D = 256: no spills.
  constexpr bool MOM = (OPT == ORX_OPT_MOMENTUM);
  constexpr int PV = LAZY ? ORX_VARIANT_STEP : ORX_VARIANT_STEP_PIPE;
  // k_pair_step moves table and slot rows as float4: a table or slot base off a 16-byte boundary takes k_pair_generic.
  // ROWWISE_ADAGRAD reads its accumulators as scalars, so only the tables decide; it holds three accumulator scalars
  // (and the rows' gradients over the row sum) where ADAGRAD holds 3K float4 slot registers, and takes ADAGRAD's
  // variants: PIPE at D = 32, 64, 256, four CTAs/SM without PIPE at D = 128 (no spills under -Xptxas -v).
  // bf16 rows add the rounding's hashes to the live values: under -Xptxas -v ADAGRAD spills at four CTAs/SM at D = 128
  // and with PIPE at D = 256, and LAZY at three CTAs/SM at D = 128.  bf16 ADAGRAD therefore takes MOMENTUM's variants
  // and bf16 LAZY two CTAs/SM at D = 128.
  constexpr bool BF = std::is_same<T, uint16_t>::value;
  constexpr bool ADA = (OPT == ORX_OPT_ADAGRAD);
  const bool rows_ok = BF ? orx_aligned8(pa.U, pa.I) : orx_aligned16(pa.U, pa.I);
  const bool vec = OrxOptSlots<OPT>::ROW ? rows_ok : rows_ok && orx_aligned16(pa.Us0, pa.Us1, pa.Is0, pa.Is1);
  switch (vec ? pa.D : 0) {
    case 32: go(k_pair_step<KIND, OPT, 32, 8, 2, !LAZY, T>, PV, 2, blocks); break;
    case 64: go(k_pair_step<KIND, OPT, 64, 8, 2, !LAZY, T>, PV, 2, blocks); break;
    case 128:
      if constexpr (BF && LAZY) go(k_pair_step<KIND, OPT, 128, 8, 2, false, T>, ORX_VARIANT_STEP, 2, blocks);
      else if constexpr (LAZY || MOM || (BF && ADA)) go(k_pair_step<KIND, OPT, 128, 8, 3, false, T>, ORX_VARIANT_STEP, 3, blocks);
      else go(k_pair_step<KIND, OPT, 128, 8, 4, false, T>, ORX_VARIANT_STEP, 4, blocks);
      break;
    case 256:
      if constexpr (MOM || (BF && ADA)) go(k_pair_step<KIND, OPT, 256, 8, 2, false, T>, ORX_VARIANT_STEP, 2, blocks);
      else go(k_pair_step<KIND, OPT, 256, 8, 2, !LAZY, T>, PV, 2, blocks);
      break;
    default: go(k_pair_generic<KIND, OPT, 0, T>, ORX_VARIANT_STEP_GENERIC, 0, 8 * blocks); break;
  }
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// ---- pipelined batch index ------------------------------------------------------------------------------------------
// The index of a batch depends only on its ids, so it can be built while the PREVIOUS step's kernels still run: on the
// context's side stream, into one of the handle's two prefetch index sets (1 and 2, alternating) -- set 0 stays with
// everything that builds its index on the caller's stream (pointwise / censor / sparse apply / un-prefetched pairwise
// steps; the row-sharded step keeps index sets of its own, orx_shard.cu).  The step that consumes a prefetched set waits
// for its `done` event; the set is handed back with its `free` event, recorded behind that step's tail.  A set's epoch
// is taken on the side stream after that wait, so a wrap empties its tables behind every step that used them.
static int side_stream_ensure(orx_ctx* c) {
  if (c->side_stream) return ORX_OK;
  ORX_CUDA(cudaStreamCreateWithFlags(&c->side_stream, cudaStreamNonBlocking));
  ORX_CUDA(cudaEventCreateWithFlags(&c->side_ev, cudaEventDisableTiming));
  for (int i = 0; i < 2; ++i) {
    OrxIndexSet& s = c->set[1 + i];
    ORX_CUDA(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    ORX_CUDA(cudaEventCreateWithFlags(&s.free, cudaEventDisableTiming));
    ORX_CUDA(cudaEventCreateWithFlags(&c->stage_free[i], cudaEventDisableTiming));
    s.free_valid = c->stage_free_valid[i] = 0;
  }
  return ORX_OK;
}

// a prefetched index nobody consumed: wait for it, reset its control words (the hash itself dies with its epoch)
static int prefetch_drop(orx_ctx* c, cudaStream_t st) {
  if (!c->pf_set) return ORX_OK;
  OrxIndexSet& s = c->set[c->pf_set];
  ORX_CUDA(cudaStreamWaitEvent(st, s.done, 0));
  ORX_CUDA(cudaMemsetAsync(s.ctl, 0, sizeof(int32_t) * 4, st));
  ORX_CUDA(cudaEventRecord(s.free, st));
  s.free_valid = 1;
  c->pf_set = 0;
  return ORX_OK;
}

// Build the index of (uid, pid, nid) on the side stream.  `after` (may be null) is an event the build must wait for
// (the caller's "ids are final" point); the ids themselves may also be produced on the side stream (host upload).
static int prefetch_issue(orx_ctx* c, const int32_t* uid, const int32_t* pid, const int32_t* nid, int B, int64_t rows_u,
                          int64_t rows_i, int mode) {
  const int k = 1 + c->pf_next;
  c->pf_next ^= 1;
  OrxIndexSet& s = c->set[k];
  cudaStream_t ss = c->side_stream;
  if (s.free_valid) ORX_CUDA(cudaStreamWaitEvent(ss, s.free, 0));   // the step that last used set k is done
  int rc;
  if ((rc = orx_take_epoch(s.u, ss)) || (rc = orx_take_epoch(s.i, ss))) return rc;
  k_index_build<<<(3 * B + 255) / 256, 256, 0, ss>>>(s.u, s.i, uid, rows_u, pid, nid, rows_i, B, mode, s.ctl + 3);
  ORX_LAUNCH_CHECK();
  if (s.res) {   // the probe answers too: the step then reads one record per triplet (done follows them)
    k_index_resolve<<<(B + 255) / 256, 256, 0, ss>>>(s.u, s.i, uid, pid, nid, rows_u, rows_i, B, mode, s.res);
    ORX_LAUNCH_CHECK();
  }
  ORX_CUDA(cudaEventRecord(s.done, ss));
  c->pf_set = k;
  s.uid = uid; s.pid = pid; s.nid = nid; s.B = B; s.rows_u = rows_u; s.rows_i = rows_i; s.mode = mode;
  return ORX_OK;
}

extern "C" int orx_pairwise_prefetch(orx_handle_t h, const orx_table_t* user, const orx_table_t* item, const int32_t* uid,
                                     const int32_t* pid, const int32_t* nid, int32_t B, int32_t opt_kind, int32_t ids_ready,
                                     orx_stream_t ids_stream) {
  ORX_REQUIRE(h != nullptr && user && item && uid && pid && nid && B > 0, "bad arguments");
  ORX_REQUIRE(orx_opt_kind_ok(opt_kind), "unknown optimizer kind");
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

// test hook: the first B records k_index_resolve wrote for prefetch set `set` (1 or 2), copied to rec on s once that
// set's prefetch is complete
extern "C" int orx_debug_pair_records(orx_handle_t h, int32_t set, int32_t* rec, int32_t B, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && rec && (set == 1 || set == 2) && B > 0, "bad arguments");
  const OrxIndexSet& x = h->set[set];
  ORX_REQUIRE(x.res && h->side_stream && B <= h->cap_B,
              "no records of that many triplets (ORX_PAIR_RESOLVE=0, no prefetch yet, or B beyond the workspace)");
  ORX_CUDA(cudaSetDevice(h->device));
  ORX_CUDA(cudaStreamWaitEvent((cudaStream_t)s, x.done, 0));
  ORX_CUDA(cudaMemcpyAsync(rec, x.res, sizeof(int4) * (size_t)B, cudaMemcpyDeviceToDevice, (cudaStream_t)s));
  return ORX_OK;
}

int orx_sparse_step(orx_ctx* c, int op, int kind, const orx_table_t* user, const orx_table_t* item,
                    const orx_table_t* bias, const orx_table_t* w, const int32_t* uid, const int32_t* iid,
                    const int32_t* nid, int B, const orx_opt_t* opt, float loss_scale, float c_l2, float* out4,
                    const OrxStepKernel& kernel, cudaStream_t st, const uint32_t* srk) {
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
  const OrxIndexSet& pf = c->set[c->pf_set];
  int set = 0;
  if (nid && c->pf_set && pf.uid == uid && pf.pid == iid && pf.nid == nid && pf.B == B && pf.rows_u == user->rows &&
      pf.rows_i == item->rows && pf.mode == (dense ? 1 : 0)) {
    set = c->pf_set;
    ORX_CUDA(cudaStreamWaitEvent(st, pf.done, 0));
    c->pf_set = 0;
  } else {
    if (nid && (rc = prefetch_drop(c, st))) return rc;
    if ((rc = orx_launch_index_build(c, uid, user->rows, iid, nid, item->rows, B, dense ? 1 : 0, st))) return rc;
  }
  OrxIndexSet& ix = c->set[set];
  orx_prof_mark(c, 1, st);
  SparseArgs s = orx_sparse_args(c, user, item, bias, ix, orx_opt_to_dev(opt));
  if (srk) { s.srk[0] = srk[0]; s.srk[1] = srk[1]; }
  OrxStepLaunch L = {};
  if ((rc = kernel(s, ix.res, c->partials, &L))) return rc;   // set 0 has no records
  orx_log_dispatch(c, op, L.variant, kind, opt->kind, B, D, L.minb, set);
  orx_prof_mark(c, 2, st);
  if (dense && (rc = orx_launch_adam_sweeps(c, user, item, bias, ix, s.opt, st, srk))) return rc;
  TailArgs ta = {s};
  ta.partials = c->partials; ta.n_partials = L.n_partials; ta.loss_scale = loss_scale;
  ta.counters = ix.ctl; ta.out4 = out4;
  if (w) {
    ta.W = w->var; ta.Ws0 = w->s0; ta.Ws1 = w->s1; ta.gw = c->gw; ta.c_l2 = c_l2;
  }
  rc = orx_launch_tail(c, ta, opt->kind, st, srk != nullptr);
  if (set) {   // the prefetch set is free again once this tail has run
    ORX_CUDA(cudaEventRecord(ix.free, st));
    ix.free_valid = 1;
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

// srk: bf16 user / item tables with these rounding keys (their var passed as float*), null: float tables
static int pairwise_step_impl(orx_ctx* c, int kind, const orx_table_t* user, const orx_table_t* item,
                              const orx_table_t* bias, const int32_t* uid, const int32_t* pid, const int32_t* nid,
                              int B, float margin, float c_loss, float c_l2, const orx_opt_t* opt, float* out4,
                              cudaStream_t st, const uint32_t* srk = nullptr) {
  ORX_REQUIRE(kind == ORX_PAIR_BPR || kind == ORX_PAIR_UCML, "unknown pairwise kind");
  ORX_REQUIRE(nid != nullptr, "empty batch or null ids");
  orx_opt_t od;
  if (opt && user) {   // dim-1 rows under ROWWISE_ADAGRAD run (and are recorded) as ADAGRAD
    od = orx_opt_dim(opt, user->dim);
    opt = &od;
  }
  const float inv_B = 1.0f / (float)B;
  const auto kernel = [&](const SparseArgs& s, const int4* res, float* partials, OrxStepLaunch* out) {
    PairArgs pa = pair_args(s, user->rows, item->rows, uid, pid, nid, B, margin, c_loss, c_l2, inv_B);
    pa.partials = partials;
    pa.res = res;   // k_pair_generic probes the index whatever res is
    return orx_dispatch<ORX_PAIR_BPR, ORX_PAIR_UCML>(kind, [&](auto K) {
      return orx_dispatch_opt(opt->kind, [&](auto O) {
        if (srk) return launch_pair_step_kind_opt<decltype(K)::value, decltype(O)::value, uint16_t>(pa, st, out);
        return launch_pair_step_kind_opt<decltype(K)::value, decltype(O)::value>(pa, st, out);
      });
    });
  };
  return orx_sparse_step(c, srk ? ORX_OP_PAIRWISE_STEP_BF16 : ORX_OP_PAIRWISE_STEP, kind, user, item, bias, nullptr,
                         uid, pid, nid, B, opt, kind == ORX_PAIR_BPR ? inv_B : 1.0f, c_l2, out4, kernel, st, srk);
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

extern "C" int orx_pairwise_step_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                      const orx_table_bf16_t* item, const orx_table_t* item_bias, const int32_t* uid,
                                      const int32_t* pid, const int32_t* nid, int32_t B, float margin, float c_loss,
                                      float c_l2, const orx_opt_t* opt, uint64_t sr_seed, float* out4, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(opt != nullptr, "null opt/out");
  ORX_CUDA(cudaSetDevice(h->device));
  orx_table_t tu, ti;
  const uint32_t srk[2] = {orx_sr_table_key(sr_seed, opt->step, 0), orx_sr_table_key(sr_seed, opt->step, 1)};
  return pairwise_step_impl(h, kind, orx_bf16_table(user, &tu), orx_bf16_table(item, &ti), item_bias, uid, pid, nid, B, margin,
                            c_loss, c_l2, opt, out4, (cudaStream_t)s, srk);
}

// Host-buffer form: the upload of this batch's ids and its index build run on the side stream, i.e. under the previous
// step's kernels whenever the caller enqueues ahead of the GPU; the step kernels and the read-back of out4 stay on `s`.
// The id staging buffers alternate; buffer f is reused only after the step that read it has finished (stage_free[f]).
static int pairwise_step_host_impl(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                                   const orx_table_t* item_bias, const int32_t* uid_host, const int32_t* pid_host,
                                   const int32_t* nid_host, int32_t B, float margin, float c_loss, float c_l2,
                                   const orx_opt_t* opt, float* out4_host, orx_stream_t s, const uint32_t* srk) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(B > 0 && uid_host && pid_host && nid_host && out4_host && user && item && opt, "empty batch or null host buffers");
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
                          opt, h->out_stage[f], st, srk);
  if (rc) return rc;
  ORX_CUDA(cudaEventRecord(h->stage_free[f], st));
  h->stage_free_valid[f] = 1;
  ORX_CUDA(cudaMemcpyAsync(out4_host, h->out_stage[f], sizeof(float) * 4, cudaMemcpyDeviceToHost, st));
  return ORX_OK;
}

extern "C" int orx_pairwise_step_host(orx_handle_t h, int32_t kind, const orx_table_t* user, const orx_table_t* item,
                                      const orx_table_t* item_bias, const int32_t* uid_host, const int32_t* pid_host,
                                      const int32_t* nid_host, int32_t B, float margin, float c_loss, float c_l2,
                                      const orx_opt_t* opt, float* out4_host, orx_stream_t s) {
  return pairwise_step_host_impl(h, kind, user, item, item_bias, uid_host, pid_host, nid_host, B, margin, c_loss, c_l2,
                                 opt, out4_host, s, nullptr);
}

extern "C" int orx_pairwise_step_host_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                           const orx_table_bf16_t* item, const orx_table_t* item_bias,
                                           const int32_t* uid_host, const int32_t* pid_host, const int32_t* nid_host,
                                           int32_t B, float margin, float c_loss, float c_l2, const orx_opt_t* opt,
                                           uint64_t sr_seed, float* out4_host, orx_stream_t s) {
  ORX_REQUIRE(opt != nullptr, "empty batch or null host buffers");
  orx_table_t tu, ti;
  const uint32_t srk[2] = {orx_sr_table_key(sr_seed, opt->step, 0), orx_sr_table_key(sr_seed, opt->step, 1)};
  return pairwise_step_host_impl(h, kind, orx_bf16_table(user, &tu), orx_bf16_table(item, &ti), item_bias, uid_host, pid_host,
                                 nid_host, B, margin, c_loss, c_l2, opt, out4_host, s, srk);
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
// bf16: the user / item tables of pa are bf16.
static int pair_unfused(orx_ctx* c, int kind, PairArgs pa, float* out4, cudaStream_t st, bool bf16 = false) {
  const auto launch = [&](float* partials, int blocks) {
    pa.partials = partials;
    orx_dispatch<ORX_PAIR_BPR, ORX_PAIR_UCML>(kind, [&](auto K) {
      if (bf16) k_pair_generic<decltype(K)::value, ORX_OPT_SGD, 1, uint16_t><<<blocks, 256, 0, st>>>(pa);
      else k_pair_generic<decltype(K)::value, ORX_OPT_SGD, 1><<<blocks, 256, 0, st>>>(pa);
    });
  };
  return orx_sparse_unfused(c, pa.B, kind == ORX_PAIR_BPR ? pa.inv_B : 1.f, out4, launch, st);
}

static int pair_fwd_grad(orx_ctx* c, int kind, const orx_table_t* user, const orx_table_t* item,
                         const orx_table_t* bias, const int32_t* uid, const int32_t* pid, const int32_t* nid, int B,
                         float margin, float c_loss, float c_l2, float* d_user, float* d_pos, float* d_neg,
                         float* d_bp, float* d_bn, float* g_out, float* out4, cudaStream_t st, bool bf16 = false) {
  ORX_REQUIRE(kind == ORX_PAIR_BPR || kind == ORX_PAIR_UCML, "unknown pairwise kind");
  ORX_REQUIRE(B > 0 && uid && pid && nid, "empty batch or null ids");
  int rc = orx_check_step_tables(user, item, bias, nullptr, ORX_OPT_SGD);
  if (rc) return rc;
  const SparseArgs s = orx_sparse_args(c, user, item, bias, c->set[0], OrxOptDev{});
  PairArgs a = pair_args(s, user->rows, item->rows, uid, pid, nid, B, margin, c_loss, c_l2, 1.0f / (float)B);
  a.d_user = d_user; a.d_pos = d_pos; a.d_neg = d_neg; a.d_bp = d_bp; a.d_bn = d_bn; a.g_out = g_out;
  return pair_unfused(c, kind, a, out4, st, bf16);
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

extern "C" int orx_pairwise_fwd_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                     const orx_table_bf16_t* item, const orx_table_t* item_bias, const int32_t* uid,
                                     const int32_t* pid, const int32_t* nid, int32_t B, float margin, float* out4,
                                     orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && out4 != nullptr, "null handle/out");
  ORX_CUDA(cudaSetDevice(h->device));
  orx_table_t tu, ti;
  return pair_fwd_grad(h, kind, orx_bf16_table(user, &tu), orx_bf16_table(item, &ti), item_bias, uid, pid, nid, B, margin, 1.f,
                       1.f, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, out4, (cudaStream_t)s, true);
}

extern "C" int orx_pairwise_grad_bf16(orx_handle_t h, int32_t kind, const orx_table_bf16_t* user,
                                      const orx_table_bf16_t* item, const orx_table_t* item_bias, const int32_t* uid,
                                      const int32_t* pid, const int32_t* nid, int32_t B, float margin, float c_loss,
                                      float c_l2, float* d_user, float* d_pos, float* d_neg, float* d_bp, float* d_bn,
                                      float* g_out, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_CUDA(cudaSetDevice(h->device));
  orx_table_t tu, ti;
  return pair_fwd_grad(h, kind, orx_bf16_table(user, &tu), orx_bf16_table(item, &ti), item_bias, uid, pid, nid, B, margin,
                       c_loss, c_l2, d_user, d_pos, d_neg, d_bp, d_bn, g_out, nullptr, (cudaStream_t)s, true);
}

// test hook: the stochastic rounding of include/orx.h applied to n floats, element i at (row0 + i / dim, i % dim)
__global__ void k_debug_round_bf16(const float* x, uint16_t* out, int64_t n, int64_t row0, int dim, uint32_t kt) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (uint16_t)orx_bf16_sr(x[i], orx_sr_row(kt, row0 + i / dim), (int)(i % dim));
}

extern "C" int orx_debug_round_bf16(orx_handle_t h, const float* x, uint16_t* out, int64_t n, int64_t row0,
                                    int32_t dim, int32_t table, uint64_t sr_seed, int64_t step, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && x && out, "null pointer");
  ORX_REQUIRE(n >= 0 && dim > 0 && row0 >= 0 && (table == 0 || table == 1), "bad arguments");
  if (n == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  k_debug_round_bf16<<<orx_grid_for(n, 256, h->num_sms), 256, 0, (cudaStream_t)s>>>(
      x, out, n, row0, dim, orx_sr_table_key(sr_seed, step, table));
  ORX_LAUNCH_CHECK();
  return ORX_OK;
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
