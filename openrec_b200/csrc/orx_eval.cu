// orx_eval.cu -- catalogue-scale evaluation and retrieval: score a batch of users against the whole item table and
// count the AUC / NDCG / Recall ranks in the same pass (orx_score_rank), or keep each user's k best items
// (orx_score_topk), from per-user CSR lists of positives and exclusions.  No [Bu, I] buffer.  Both share one tile loop
// (ev_tiles) and differ only in its epilogue.
//
// Counting identity (orx_rank_metrics' definitions, one batch row, p over its positives, i over all items):
//   AUC count = sum_{i eval} #{p : pred_p >= s_i}          rank_p = #{i : sp_i > sp_p},  sp = expf(pred) * !excl
// The main pass counts every item as if it were an eval item and not excluded: its AUC term #{p : pred_p >= s} and,
// with j = #{p : sp_p < expf(s)} over the ascending sp, one hit in hist[j] (the item ranks above the j smallest sp).
// The finish recomputes the scores of pos u excl, takes back their AUC terms and the rank hits of the excluded items
// (an excluded item's sp is 0 or NaN and never ranks above anything), and rank of the q-th smallest sp = sum_{j > q}
// hist[j].  Every score is computed by the FFMA chain of k_score_all (acc = 0, one fused multiply-add per k in
// ascending order, user value scaled first, bias added last), so the comparisons, and with them every count, equal
// those of orx_score_all + orx_rank_metrics exactly.
//
// Every count is a sum over items, so it splits over any partition of the catalogue.  orx_score_rank_shard runs the
// same kernels on row-sharded tables (item i is row i / world of rank i % world): each rank counts over its own rows
// and takes back its own items of pos u excl, the callers sum the integer counts over the ranks, and the finish reads
// the sums.  The user rows and the positives' scores reach every rank the same way, as integer sums in which exactly
// one rank contributes a non-zero word, so their bits cross unchanged.
//
// orx_score_topk_shard does the same for retrieval: each rank keeps the exact top k of its own rows (keys built from the
// global item ids), the ranks' lists cross as a summed exchange, and the merge of k_score_topk takes the top k of their
// union, which holds the global top k.
#include <cub/device/device_segmented_sort.cuh>

#include "orx_common.cuh"

namespace {

constexpr int EV_TU = 128, EV_TI = 128, EV_KC = 8, EV_NT = 256, EV_LD = EV_TU + 4;

// What the tile kernels (k_score_rank, k_score_topk) read.  Kept at this layout: their register allocation is tight.
// T: the storage of the user and item tables, float or bf16 held as its uint16_t bits (widened exactly by orx_ld1 as
// each element is read; scale, bias and every score stay fp32).  The sharded phases take float tables only.
template <typename T>
struct EvalArgsT {
  const T* user_tab;
  int64_t U;
  const int32_t* uid;
  int Bu;
  const float* scale;
  const T* item_tab;
  const float* bias;
  int64_t I;   // item rows the tile loop walks (rows of item_tab / bias)
  int D;
  const int64_t *pos_off, *excl_off;
  const int32_t *pos_items, *excl_items;
  int max_pos;
  int P;  // max_pos + 1: row stride of the threshold and histogram rows
};
using EvalArgs = EvalArgsT<float>;

// What the per-row kernels (one CTA per batch row) read on top: the catalogue, the item ownership and the exchange.
template <typename T>
struct EvalRowArgsT : EvalArgsT<T> {
  int64_t I_all;        // the catalogue: list entries in [0, I_all) count, n_eval = I_all - n - extra
  int world, rank;      // row r is local row r / world on rank r % world (1, 0: the whole table)
  const T* xrows;       // non-null: batch row b's user row is xrows[b * D ..] (uid still decides bad rows)
  const float* xpred;   // non-null: prep reads the positives' scores from xpred[b * P + q] instead of computing them
  const int64_t* neg_off;      // orx_score_rank_listed: the listed items' CSR (unused by the catalogue pass)
  const int32_t* neg_items;
};
using EvalRowArgs = EvalRowArgsT<float>;

// Scratch of one call (handle workspace).  keys_in / keys: [2][Bu][P] -- pred thresholds of row b at b * P, sp
// thresholds at (Bu + b) * P; keys holds them sorted ascending.  info[2b] = positives of row b (-1: longer than
// max_pos), info[2b + 1] = those whose pred is not NaN (the pred thresholds searched for AUC).
struct EvalWs {
  float *keys_in, *keys;
  int *seg_begin, *seg_end;
  unsigned* hist;                 // [Bu][P]
  unsigned long long* auc_cnt;    // [Bu]
  int* info;                      // [Bu][2]
  void* sort_tmp;
  size_t sort_bytes;
};

struct EvalOut {
  int at[ORX_MAX_AT];
  int n_at;
  float *auc, *ndcg, *recall;
};

// XROWS: user_tab holds one row per batch position (the summed exchange of the sharded pass), not per user id
template <bool XROWS, typename T>
__device__ __forceinline__ const T* ev_user_row(const EvalArgsT<T>& a, int b) {
  const int32_t id = a.uid[b];
  return (id >= 0 && (int64_t)id < a.U) ? a.user_tab + (int64_t)(XROWS ? b : id) * a.D : nullptr;
}
template <typename T>
__device__ __forceinline__ const T* ev_urow(const EvalRowArgsT<T>& a, int b) {
  if (!a.xrows) return ev_user_row<false>(a, b);
  const int32_t id = a.uid[b];
  return (id >= 0 && (int64_t)id < a.U) ? a.xrows + (int64_t)b * a.D : nullptr;
}

// ownership of a (user or item) id in [0, 2^31): row r lives on rank r % world at local row r / world
template <typename T>
__device__ __forceinline__ bool ev_owns(const EvalRowArgsT<T>& a, int32_t r) {
  return (uint32_t)r % (uint32_t)a.world == (uint32_t)a.rank;
}
template <typename T>
__device__ __forceinline__ int64_t ev_local(const EvalRowArgsT<T>& a, int32_t r) {
  return (uint32_t)r / (uint32_t)a.world;
}

// first position in items[lo, hi) holding a value >= v (the row is sorted)
__device__ __forceinline__ int64_t ev_lower(const int32_t* items, int64_t lo, int64_t hi, int64_t v) {
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((int64_t)items[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// The entries of user row `row` of a CSR that lie in [0, I): [*lo, *hi); *raw = the row's full length.
__device__ __forceinline__ void ev_range(const int64_t* off, const int32_t* items, int32_t row, int64_t rows, int64_t I,
                                         int64_t* lo, int64_t* hi, int64_t* raw) {
  *lo = *hi = *raw = 0;
  if (!off || row < 0 || (int64_t)row >= rows) return;
  const int64_t b = off[row], e = off[row + 1];
  *raw = e - b;
  *lo = ev_lower(items, b, e, 0);
  *hi = ev_lower(items, *lo, e, I);
}

__device__ __forceinline__ bool ev_contains(const int32_t* items, int64_t lo, int64_t hi, int32_t v) {
  const int64_t k = ev_lower(items, lo, hi, v);
  return k < hi && items[k] == v;
}

// The user value at k of the chain of k_score_all (urow nullptr: a zero row).  Explicit roundings: u * scale - i must
// not contract into one fused multiply-add.
template <typename T>
__device__ __forceinline__ float ev_uval(const EvalArgsT<T>& a, const T* urow, int k) {
  float uv = 0.f;
  if (urow) {
    uv = orx_ld1(urow + k);
    if (a.scale) uv = __fmul_rn(uv, a.scale[k]);
  }
  return uv;
}

// One step of the chain of k_score_all: acc after the term of (user value uv, item value iv).
template <int KIND>
__device__ __forceinline__ float ev_step(float acc, float uv, float iv) {
  if (KIND == ORX_SCORE_DOT) return __fmaf_rn(uv, iv, acc);
  const float d = __fsub_rn(uv, iv);
  return __fmaf_rn(-d, d, acc);
}

// One score by the chain of k_score_all, of an item i this rank owns (ev_owns).
template <int KIND, typename T>
__device__ __forceinline__ float ev_score1(const EvalRowArgsT<T>& a, const T* urow, int32_t i_global) {
  const int64_t i = ev_local(a, i_global);
  const T* irow = a.item_tab + i * a.D;
  float acc = 0.f;
  for (int k = 0; k < a.D; ++k) acc = ev_step<KIND>(acc, ev_uval(a, urow, k), orx_ld1(irow + k));
  return acc + (a.bias ? a.bias[i] : 0.f);
}

// #{q < n_auc : pth[q] >= s} over ascending thresholds with bounds pmin / pmax (n_auc = 0: pmin = +inf, pmax = -inf);
// a NaN s counts nothing (pred_e <= pred_p is false).
__device__ __forceinline__ unsigned ev_auc_count(const float* pth, int n_auc, float pmin, float pmax, float s) {
  if (!(s <= pmax)) return 0u;
  if (s <= pmin) return (unsigned)n_auc;
  int lo = 0, hi = n_auc;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (pth[mid] >= s) hi = mid;
    else lo = mid + 1;
  }
  return (unsigned)(n_auc - lo);
}

// #{q < n : sth[q] < e} over ascending thresholds with bounds smin / smax (n = 0: smin = +inf); NaN e gives 0.
__device__ __forceinline__ int ev_rank_slot(const float* sth, int n, float smin, float smax, float e) {
  if (!(e > smin)) return 0;
  if (e > smax) return n;
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sth[mid] < e) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// ---------------------------------------------------------------------------------------
// prep: one CTA per batch row.  pred_p and sp_p of every positive (sp: NaN -> +inf, which ranks 0 like NaN; a NaN pred
// is left out of the AUC search and out of the pred segment, which a comparison sort could not order), zeroed
// histogram and AUC count, and the two sort segments of the row.  With a.xpred the scores are read from the summed
// exchange, not computed.
// ---------------------------------------------------------------------------------------
// The positive and exclusion entries of batch row b in [0, I_all), and whether its positive row is longer than max_pos.
struct EvRow {
  int64_t plo, phi, elo, ehi;
  bool bad;
};

template <typename T>
__device__ __forceinline__ EvRow ev_row(const EvalRowArgsT<T>& a, int b) {
  EvRow r;
  int64_t praw, eraw;
  const int32_t u = a.uid[b];
  ev_range(a.pos_off, a.pos_items, u, a.U, a.I_all, &r.plo, &r.phi, &praw);
  ev_range(a.excl_off, a.excl_items, u, a.U, a.I_all, &r.elo, &r.ehi, &eraw);
  r.bad = praw > a.max_pos;
  return r;
}

template <int KIND, typename T>
__global__ void __launch_bounds__(EV_NT) k_eval_prep(const EvalRowArgsT<T> a, const EvalWs w) {
  __shared__ int s_nan, s_kp;
  const int b = blockIdx.x;
  const T* urow = ev_urow(a, b);
  const EvRow r = ev_row(a, b);
  const int64_t plo = r.plo, elo = r.elo, ehi = r.ehi;
  const bool bad = r.bad;
  const int n = bad ? 0 : (int)(r.phi - plo);
  float* kp = w.keys_in + (int64_t)b * a.P;
  float* ks = w.keys_in + (int64_t)(a.Bu + b) * a.P;
  if (threadIdx.x == 0) s_nan = s_kp = 0;
  __syncthreads();
  for (int q = threadIdx.x; q < n; q += blockDim.x) {
    const int32_t i = a.pos_items[plo + q];
    const float s = a.xpred ? a.xpred[(int64_t)b * a.P + q] : ev_score1<KIND>(a, urow, i);
    const bool ex = ev_contains(a.excl_items, elo, ehi, i);
    float sp = expf(s) * (ex ? 0.f : 1.f);
    if (sp != sp) sp = __int_as_float(0x7f800000);
    if (s != s) atomicAdd(&s_nan, 1);
    else kp[atomicAdd(&s_kp, 1)] = s;   // the pred segment holds the non-NaN preds only, in any order
    ks[q] = sp;
  }
  for (int j = threadIdx.x; j < a.P; j += blockDim.x) w.hist[(int64_t)b * a.P + j] = 0u;
  __syncthreads();
  if (threadIdx.x == 0) {
    w.info[2 * b] = bad ? -1 : n;
    w.info[2 * b + 1] = n - s_nan;
    w.auc_cnt[b] = 0ull;
    w.seg_begin[b] = b * a.P;
    w.seg_end[b] = b * a.P + n - s_nan;
    w.seg_begin[a.Bu + b] = (a.Bu + b) * a.P;
    w.seg_end[a.Bu + b] = (a.Bu + b) * a.P + n;
  }
}

// Sharded phase 0: xrows[b] = the bits of user row uid[b] if this rank owns it, else 0 (every element written).
__global__ void __launch_bounds__(EV_NT) k_eval_user_rows(const EvalRowArgs a, int32_t* xrows) {
  const int64_t n = (int64_t)a.Bu * a.D;
  for (int64_t e = blockIdx.x * (int64_t)EV_NT + threadIdx.x; e < n; e += (int64_t)gridDim.x * EV_NT) {
    const int b = (int)(e / a.D);
    const int32_t id = a.uid[b];
    int32_t v = 0;
    if (id >= 0 && (int64_t)id < a.U && ev_owns(a, id))
      v = __float_as_int(a.user_tab[ev_local(a, id) * a.D + (e - (int64_t)b * a.D)]);
    xrows[e] = v;
  }
}

// Sharded phase 1: xpred[b][q] = the bits of the score of row b's q-th positive in [0, I_all) if this rank owns that
// item, else 0; a row longer than max_pos is all 0 (every element written).
template <int KIND>
__global__ void __launch_bounds__(EV_NT) k_eval_pos_scores(const EvalRowArgs a, int32_t* xpred) {
  const int b = blockIdx.x;
  const float* urow = ev_urow(a, b);
  const EvRow r = ev_row(a, b);
  const int n = r.bad ? 0 : (int)(r.phi - r.plo);
  for (int q = threadIdx.x; q < a.P; q += blockDim.x) {
    int32_t v = 0;
    if (q < n) {
      const int32_t i = a.pos_items[r.plo + q];
      if (ev_owns(a, i)) v = __float_as_int(ev_score1<KIND>(a, urow, i));
    }
    xpred[(int64_t)b * a.P + q] = v;
  }
}

// ---------------------------------------------------------------------------------------
// main pass: 128 users x 128 items per tile, 8 x 8 scores per thread, D in chunks of 8 through a double-buffered
// shared tile.  A CTA takes one user tile and walks a contiguous range of item tiles; the thresholds and histograms
// of its rows sit in shared memory (USE_SMEM) or stay in the global scratch, reached through the same generic pointers.
// ---------------------------------------------------------------------------------------
template <typename T>
struct RowMeta {
  const T* urow;
  const float* pth;
  const float* sth;
  unsigned* hist;
  int n, n_auc;
  float pmin, pmax, smin, smax;
};

// rows / columns of a thread's 8 x 8 block: 4 at t * 4 and 4 at 64 + t * 4
__device__ __forceinline__ int ev_frag(int t, int x) { return (x < 4 ? 0 : 64 - 4) + t * 4 + x; }

template <int KIND, bool TAIL>
__device__ __forceinline__ void ev_mma_chunk(float (&acc)[8][8], const float (*sa)[EV_LD], const float (*sb)[EV_LD],
                                             int ty, int tx, int kn) {
#pragma unroll
  for (int k = 0; k < EV_KC; ++k) {
    if (TAIL && k >= kn) break;
    const float4 a0 = *reinterpret_cast<const float4*>(&sa[k][ty * 4]);
    const float4 a1 = *reinterpret_cast<const float4*>(&sa[k][64 + ty * 4]);
    const float4 b0 = *reinterpret_cast<const float4*>(&sb[k][tx * 4]);
    const float4 b1 = *reinterpret_cast<const float4*>(&sb[k][64 + tx * 4]);
    const float uu[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    const float ii[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int x = 0; x < 8; ++x)
#pragma unroll
      for (int y = 0; y < 8; ++y) {
        if (KIND == ORX_SCORE_DOT) {
          acc[x][y] = __fmaf_rn(uu[x], ii[y], acc[x][y]);
        } else {
          const float d = __fsub_rn(uu[x], ii[y]);
          acc[x][y] = __fmaf_rn(-d, d, acc[x][y]);
        }
      }
  }
}

// The main loop of k_score_rank and k_score_topk: the CTA's user tile against its contiguous range of item tiles
// (blockIdx.x of gridDim.x splits).  Tile row r's user row is urow_of(r) (nullptr: a zero row); D goes in chunks of 8
// through the double-buffered shared tiles sA / sB.  After each tile every thread calls epi(i0, acc): acc[x][y] is the
// score of row ev_frag(ty, x) and item i0 + ev_frag(tx, y) before the bias, by the chain of k_score_all.  Every thread
// passes a __syncthreads after epi returns and before the next tile's scores are read.
// VEC (bf16 tables only, dim % 4 == 0, both tables 8-byte aligned: ev_vec): each thread moves 4 columns of one row of
// each table as one 8-byte load, where the scalar loader makes 4 two-byte loads.  The loaders differ only in which
// thread carries which element, so the shared tiles, and every score, are the same bits.
template <int KIND, bool VEC, typename T, class UrowOf, class Epi>
__device__ __forceinline__ void ev_tiles(const EvalArgsT<T>& a, float (*sA)[EV_KC][EV_LD], float (*sB)[EV_KC][EV_LD],
                                         UrowOf urow_of, Epi epi) {
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t n_tiles = (a.I + EV_TI - 1) / EV_TI;
  const int64_t t_begin = n_tiles * blockIdx.x / gridDim.x, t_end = n_tiles * (blockIdx.x + 1) / gridDim.x;
  const int n_chunks = (a.D + EV_KC - 1) / EV_KC;
  float ru[4], ri[4];
  // chunk k0 of this tile into registers: element e = tid + 256 j is row e / 8, k e % 8; with VEC, thread tid holds
  // row tid / 2, k (tid % 2) * 4 + j
  auto load = [&](int64_t i0, int k0) {
    if constexpr (VEC) {
      const int r = tid >> 1, k = k0 + (tid & 1) * 4;
      float4 uv = make_float4(0.f, 0.f, 0.f, 0.f), iv = uv;
      if (k < a.D) {   // dim % 4 == 0: the 4 columns are all inside the row or all past it
        const T* urow = urow_of(r);
        if (urow) {
          uv = orx_ld4(urow + k);
          if (a.scale) {
            uv.x = __fmul_rn(uv.x, a.scale[k]);
            uv.y = __fmul_rn(uv.y, a.scale[k + 1]);
            uv.z = __fmul_rn(uv.z, a.scale[k + 2]);
            uv.w = __fmul_rn(uv.w, a.scale[k + 3]);
          }
        }
        if (i0 + r < a.I) iv = orx_ld4(a.item_tab + (i0 + r) * a.D + k);
      }
      ru[0] = uv.x; ru[1] = uv.y; ru[2] = uv.z; ru[3] = uv.w;
      ri[0] = iv.x; ri[1] = iv.y; ri[2] = iv.z; ri[3] = iv.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e = tid + EV_NT * j, r = e >> 3, k = k0 + (e & 7);
        float uv = 0.f, iv = 0.f;
        if (k < a.D) {
          const T* urow = urow_of(r);
          if (urow) {
            uv = orx_ld1(urow + k);
            if (a.scale) uv = __fmul_rn(uv, a.scale[k]);
          }
          if (i0 + r < a.I) iv = orx_ld1(a.item_tab + (i0 + r) * a.D + k);
        }
        ru[j] = uv;
        ri[j] = iv;
      }
    }
  };
  auto store = [&](int buf) {
    if constexpr (VEC) {   // rows tid / 2 of a warp's 16 row pairs: banks (4k + r) % 32 of the two halves are disjoint
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        sA[buf][(tid & 1) * 4 + j][tid >> 1] = ru[j];
        sB[buf][(tid & 1) * 4 + j][tid >> 1] = ri[j];
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e = tid + EV_NT * j;
        sA[buf][e & 7][e >> 3] = ru[j];
        sB[buf][e & 7][e >> 3] = ri[j];
      }
    }
  };

  for (int64_t t = t_begin; t < t_end; ++t) {
    const int64_t i0 = t * EV_TI;
    float acc[8][8];
#pragma unroll
    for (int x = 0; x < 8; ++x)
#pragma unroll
      for (int y = 0; y < 8; ++y) acc[x][y] = 0.f;
    load(i0, 0);
    store(0);
    __syncthreads();
    for (int c = 0; c < n_chunks; ++c) {
      if (c + 1 < n_chunks) load(i0, (c + 1) * EV_KC);
      const int kn = a.D - c * EV_KC;
      if (kn >= EV_KC) ev_mma_chunk<KIND, false>(acc, sA[c & 1], sB[c & 1], ty, tx, EV_KC);
      else ev_mma_chunk<KIND, true>(acc, sA[c & 1], sB[c & 1], ty, tx, kn);
      if (c + 1 < n_chunks) store((c + 1) & 1);
      __syncthreads();
    }
    epi(i0, acc);
  }
}

template <int KIND, bool XROWS, typename T, bool VEC = false>
__global__ void __launch_bounds__(EV_NT, 2) k_score_rank(const EvalArgsT<T> a, const EvalWs w, int use_smem) {
  extern __shared__ float4 ev_dyn4[];
  __shared__ __align__(16) float sA[2][EV_KC][EV_LD];
  __shared__ __align__(16) float sB[2][EV_KC][EV_LD];
  __shared__ RowMeta<T> meta[EV_TU];
  __shared__ unsigned long long s_auc[EV_TU];
  float* dyn = reinterpret_cast<float*>(ev_dyn4);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tx = tid & 15, ty = tid >> 4;
  const int u0 = blockIdx.y * EV_TU;
  const int rows = min(EV_TU, a.Bu - u0);
  const int rows_alloc = min(EV_TU, a.Bu);   // rows of the shared threshold region (the host sized it so)
  const int64_t P = a.P;

  if (tid < EV_TU) {
    RowMeta<T> m = {};
    if (tid < rows) {
      const int b = u0 + tid;
      m.urow = ev_user_row<XROWS>(a, b);
      m.n = max(w.info[2 * b], 0);
      m.n_auc = w.info[2 * b] < 0 ? 0 : w.info[2 * b + 1];
      if (use_smem) {
        m.pth = dyn + tid * P;
        m.sth = dyn + (rows_alloc + tid) * P;
        m.hist = reinterpret_cast<unsigned*>(dyn + (2 * rows_alloc + tid) * P);
      } else {
        m.pth = w.keys + (int64_t)b * P;
        m.sth = w.keys + (int64_t)(a.Bu + b) * P;
        m.hist = w.hist + (int64_t)b * P;
      }
    }
    meta[tid] = m;
    s_auc[tid] = 0ull;
  }
  __syncthreads();
  if (use_smem) {
    for (int r = warp; r < rows; r += EV_NT / 32) {
      const int b = u0 + r;
      const RowMeta<T>& m = meta[r];
      float* pth = const_cast<float*>(m.pth);
      float* sth = const_cast<float*>(m.sth);
      for (int q = lane; q < m.n; q += 32) {
        pth[q] = w.keys[(int64_t)b * P + q];
        sth[q] = w.keys[(int64_t)(a.Bu + b) * P + q];
      }
      for (int j = lane; j <= m.n; j += 32) m.hist[j] = 0u;
    }
    __syncthreads();
  }
  if (tid < rows) {
    RowMeta<T>& m = meta[tid];
    m.pmin = m.n_auc ? m.pth[0] : __int_as_float(0x7f800000);
    m.pmax = m.n_auc ? m.pth[m.n_auc - 1] : __int_as_float(0xff800000);
    m.smin = m.n ? m.sth[0] : __int_as_float(0x7f800000);
    m.smax = m.n ? m.sth[m.n - 1] : __int_as_float(0x7f800000);
  }
  __syncthreads();

  // epilogue: the AUC terms and rank hits of each tile's scores
  ev_tiles<KIND, VEC>(a, sA, sB, [&](int r) { return meta[r].urow; }, [&](int64_t i0, const float (&acc)[8][8]) {
    float bv[8];
#pragma unroll
    for (int y = 0; y < 8; ++y) {
      const int64_t i = i0 + ev_frag(tx, y);
      bv[y] = (a.bias && i < a.I) ? a.bias[i] : 0.f;
    }
#pragma unroll
    for (int x = 0; x < 8; ++x) {
      const int r = ev_frag(ty, x);
      if (r >= rows) continue;
      const RowMeta<T>& m = meta[r];
      if (m.n == 0) continue;
      unsigned long long cnt = 0ull;
#pragma unroll
      for (int y = 0; y < 8; ++y) {
        if (i0 + ev_frag(tx, y) >= a.I) continue;
        const float s = acc[x][y] + bv[y];
        cnt += ev_auc_count(m.pth, m.n_auc, m.pmin, m.pmax, s);
        const int j = ev_rank_slot(m.sth, m.n, m.smin, m.smax, expf(s));
        if (j) atomicAdd(m.hist + j, 1u);
      }
      if (cnt) atomicAdd(&s_auc[r], cnt);
    }
  });
  __syncthreads();
  for (int r = warp; r < rows; r += EV_NT / 32) {
    const RowMeta<T>& m = meta[r];
    if (use_smem)
      for (int j = 1 + lane; j <= m.n; j += 32) {
        const unsigned h = m.hist[j];
        if (h) atomicAdd(w.hist + (int64_t)(u0 + r) * P + j, h);
      }
    if (lane == 0 && s_auc[r]) atomicAdd(w.auc_cnt + u0 + r, s_auc[r]);
  }
}

// ---------------------------------------------------------------------------------------
// correction + finish: one CTA per batch row.  ev_take_back takes back the terms of pos u excl, ev_finish_row
// suffix-sums the histogram into the positives' ranks and writes auc / ndcg / recall with the formulas and conversions
// of k_rank_metrics.  k_eval_finish does both on one device; the sharded phases 2 and 3 split them (k_eval_correct on
// each rank's own items, k_eval_finish_counts on the summed counts).
// ---------------------------------------------------------------------------------------
// Block-wide over the entries of row r: adds to *s_sub the AUC terms of the positives and excluded items this rank
// owns (the main pass counted them as eval items) and takes their rank hits off hist (excluded items only: an excluded
// item's sp is 0 or NaN and never ranks above anything); adds to *s_extra the excluded items that are not positives,
// owned or not.  TAKE = false: *s_extra only (no scores, no thresholds).
template <int KIND, bool TAKE, typename T>
__device__ __forceinline__ void ev_take_back(const EvalRowArgsT<T>& a, int b, const EvRow& r, int n, int n_auc,
                                             const float* pth, const float* sth, unsigned* hist,
                                             unsigned long long* s_sub, long long* s_extra) {
  const int tid = threadIdx.x;
  const T* urow = TAKE ? ev_urow(a, b) : nullptr;
  float pmin = 0.f, pmax = 0.f, smin = 0.f, smax = 0.f;
  if (TAKE) {
    pmin = n_auc ? pth[0] : __int_as_float(0x7f800000);
    pmax = n_auc ? pth[n_auc - 1] : __int_as_float(0xff800000);
    smin = n ? sth[0] : __int_as_float(0x7f800000);
    smax = n ? sth[n - 1] : __int_as_float(0x7f800000);
  }
  unsigned long long sub = 0ull;
  long long extra = 0;
  if (TAKE)
    for (int64_t q = tid; q < n; q += blockDim.x) {          // positives: not eval items
      const int32_t i = a.pos_items[r.plo + q];
      if (!ev_owns(a, i)) continue;
      const float s = ev_score1<KIND>(a, urow, i);
      sub += ev_auc_count(pth, n_auc, pmin, pmax, s);
      if (ev_contains(a.excl_items, r.elo, r.ehi, i)) {
        const int j = ev_rank_slot(sth, n, smin, smax, expf(s));
        if (j) atomicSub(hist + j, 1u);
      }
    }
  for (int64_t q = r.elo + tid; q < r.ehi; q += blockDim.x) {  // excluded items that are not positives
    const int32_t i = a.excl_items[q];
    if (ev_contains(a.pos_items, r.plo, r.phi, i)) continue;
    ++extra;
    if (!TAKE || !ev_owns(a, i)) continue;
    const float s = ev_score1<KIND>(a, urow, i);
    sub += ev_auc_count(pth, n_auc, pmin, pmax, s);
    const int j = ev_rank_slot(sth, n, smin, smax, expf(s));
    if (j) atomicSub(hist + j, 1u);
  }
  if (sub) atomicAdd(s_sub, sub);
  if (extra) atomicAdd(reinterpret_cast<unsigned long long*>(s_extra), (unsigned long long)extra);
}

__device__ __forceinline__ void ev_nan_row(const EvalOut& o, int b) {   // a positive row longer than max_pos
  const float nan = __int_as_float(0x7fffffff);
  if (threadIdx.x == 0 && o.auc) o.auc[b] = nan;
  if (threadIdx.x < o.n_at) {
    if (o.ndcg) o.ndcg[(int64_t)b * o.n_at + threadIdx.x] = nan;
    if (o.recall) o.recall[(int64_t)b * o.n_at + threadIdx.x] = nan;
  }
}

// The outputs of row b from its final counts: auc_cnt, and hist_at(j) for j = 1..n (the rank hits).  Block-wide; every
// thread must call it.
template <typename T, class Hist>
__device__ __forceinline__ void ev_finish_row(const EvalRowArgsT<T>& a, const EvalOut& o, int b, int n, long long extra,
                                              unsigned long long auc_cnt, Hist hist_at) {
  __shared__ unsigned s_part[EV_NT];
  __shared__ unsigned s_after[EV_NT];
  __shared__ double s_dcg[ORX_MAX_AT];
  __shared__ int s_hit[ORX_MAX_AT];
  const int tid = threadIdx.x;
  if (tid < ORX_MAX_AT) {
    s_dcg[tid] = 0.0;
    s_hit[tid] = 0;
  }
  // rank of the q-th smallest sp = sum_{j > q} hist[j]: thread t owns hist[1 + t * chunk .. (t + 1) * chunk]
  const int chunk = (n + EV_NT - 1) / EV_NT;
  const int jlo = 1 + tid * chunk, jhi = min(n, (tid + 1) * chunk);
  unsigned part = 0;
  for (int j = jlo; j <= jhi; ++j) part += hist_at(j);
  s_part[tid] = part;
  __syncthreads();
  if (tid == 0) {
    unsigned run = 0;
    for (int t = EV_NT - 1; t >= 0; --t) {
      s_after[t] = run;
      run += s_part[t];
    }
  }
  __syncthreads();
  double dcg[ORX_MAX_AT];
  int hit[ORX_MAX_AT];
#pragma unroll
  for (int k = 0; k < ORX_MAX_AT; ++k) {
    dcg[k] = 0.0;
    hit[k] = 0;
  }
  unsigned run = s_after[tid];
  for (int j = jhi; j >= jlo; --j) {
    run += hist_at(j);                    // rank of position q = j - 1
    const float ra = (float)run;
    const float rec = 1.f / (logf(ra + 2.f) / logf(2.0f));
#pragma unroll
    for (int k = 0; k < ORX_MAX_AT; ++k)
      if (k < o.n_at && ra < (float)o.at[k]) {
        dcg[k] += (double)rec;
        ++hit[k];
      }
  }
#pragma unroll
  for (int k = 0; k < ORX_MAX_AT; ++k)
    if (k < o.n_at && hit[k]) {
      atomicAdd(&s_dcg[k], dcg[k]);
      atomicAdd(&s_hit[k], hit[k]);
    }
  __syncthreads();
  if (tid == 0 && o.auc) {
    const long long n_eval = a.I_all - (long long)n - extra;
    o.auc[b] = (float)auc_cnt / (float)((long long)n * n_eval);
  }
  if (tid < o.n_at) {
    if (o.ndcg) o.ndcg[(int64_t)b * o.n_at + tid] = (float)s_dcg[tid];
    if (o.recall) o.recall[(int64_t)b * o.n_at + tid] = (float)s_hit[tid] / (float)n;
  }
}

template <int KIND, typename T>
__global__ void __launch_bounds__(EV_NT) k_eval_finish(const EvalRowArgsT<T> a, const EvalWs w, const EvalOut o) {
  __shared__ unsigned long long s_sub;
  __shared__ long long s_extra;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int info = w.info[2 * b];
  if (info < 0) {
    ev_nan_row(o, b);
    return;
  }
  const int n = info;
  unsigned* hist = w.hist + (int64_t)b * a.P;
  const EvRow r = ev_row(a, b);
  if (tid == 0) {
    s_sub = 0ull;
    s_extra = 0;
  }
  __syncthreads();
  ev_take_back<KIND, true>(a, b, r, n, w.info[2 * b + 1], w.keys + (int64_t)b * a.P, w.keys + (int64_t)(a.Bu + b) * a.P,
                           hist, &s_sub, &s_extra);
  __syncthreads();
  ev_finish_row(a, o, b, n, s_extra, w.auc_cnt[b] - s_sub, [&](int j) { return hist[j]; });
}

// Sharded phase 2, after the main pass over this rank's rows: xcnt[b][0] = the row's AUC count and xcnt[b][1..n] its
// rank hits, both after taking back this rank's own items of pos u excl; the rest of the row 0 (every element written).
template <int KIND>
__global__ void __launch_bounds__(EV_NT) k_eval_correct(const EvalRowArgs a, const EvalWs w, int64_t* xcnt) {
  __shared__ unsigned long long s_sub;
  __shared__ long long s_extra;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int info = w.info[2 * b];
  const int n = max(info, 0);
  unsigned* hist = w.hist + (int64_t)b * a.P;
  if (tid == 0) {
    s_sub = 0ull;
    s_extra = 0;
  }
  __syncthreads();
  if (info >= 0)
    ev_take_back<KIND, true>(a, b, ev_row(a, b), n, w.info[2 * b + 1], w.keys + (int64_t)b * a.P,
                             w.keys + (int64_t)(a.Bu + b) * a.P, hist, &s_sub, &s_extra);
  __syncthreads();
  for (int j = tid; j < a.P; j += blockDim.x)
    xcnt[(int64_t)b * a.P + j] = j == 0 ? (int64_t)(w.auc_cnt[b] - s_sub) : j <= n ? (int64_t)hist[j] : 0;
}

// Sharded phase 3: the outputs from the counts summed over the ranks; n and extra come from the lists alone.
__global__ void __launch_bounds__(EV_NT) k_eval_finish_counts(const EvalRowArgs a, const int64_t* xcnt, const EvalOut o) {
  __shared__ long long s_extra;
  const int b = blockIdx.x;
  const EvRow r = ev_row(a, b);
  if (r.bad) {
    ev_nan_row(o, b);
    return;
  }
  const int n = (int)(r.phi - r.plo);
  if (threadIdx.x == 0) s_extra = 0;
  __syncthreads();
  ev_take_back<ORX_SCORE_DOT, false>(a, b, r, n, 0, nullptr, nullptr, nullptr, nullptr, &s_extra);
  __syncthreads();
  const int64_t* cnt = xcnt + (int64_t)b * a.P;
  ev_finish_row(a, o, b, n, s_extra, (unsigned long long)cnt[0], [&](int j) { return (unsigned)cnt[j]; });
}

// ---------------------------------------------------------------------------------------
// listed-candidate evaluation (orx_score_rank_listed): each row ranked against its listed items only.  On the masks of
// Dataset.evaluation for explicit negatives (pos = P, excl = ~(P u L) u E) an item outside (P u L) \ E has sp = 0,
// never ranks above anything and is no eval item, so every count of the catalogue pass is a sum over the lists: the
// eval items are L \ P \ E, each adding its AUC term and one rank hit, and each positive outside E adds its rank hit.
// The finish is ev_finish_row's with extra = I - n - n_eval (every item that is neither a positive nor an eval item).
// One CTA per batch row; prep and the threshold sort are those of orx_score_rank.
// ---------------------------------------------------------------------------------------
constexpr int EL_KS = 32;    // D columns of one staged slab: one 128-byte segment per item row
constexpr int EL_LD = 33;    // slab row stride, odd: thread t reading row t meets no bank conflict
constexpr int EL_UNR = 4;    // rows each warp has in flight while staging a slab

// Whether listed entry q of row r (an entry in [0, I_all)) is an eval item: neither a positive nor excluded.
template <typename T>
__device__ __forceinline__ bool el_eval_item(const EvalRowArgsT<T>& a, const EvRow& r, int64_t q) {
  const int32_t i = a.neg_items[q];
  return !ev_contains(a.pos_items, r.plo, r.phi, i) && !ev_contains(a.excl_items, r.elo, r.ehi, i);
}

// The listed entries of batch row b in [0, I_all): [*lo, *hi).
template <typename T>
__device__ __forceinline__ void el_range(const EvalRowArgsT<T>& a, int b, int64_t* lo, int64_t* hi) {
  int64_t raw;
  ev_range(a.neg_off, a.neg_items, a.uid[b], a.U, a.I_all, lo, hi, &raw);
}

// The counts of row b over the items this rank owns.  Positives outside E: one rank hit each, scored by ev_score1.
// Eval items: scored in chunks of
// EV_NT entries, thread t taking entry t; D goes in slabs of EL_KS columns staged in shared memory, one warp-wide
// 128-byte load per item row, and each thread runs the chain of ev_score1 (ascending k) over the slabs.
// xcnt == nullptr: the outputs by ev_finish_row.  Else (sharded phase 2): xcnt[b][0] = the AUC count, xcnt[b][1..n]
// the rank hits, the rest of the row 0 (every element written).
template <int KIND, typename T>
__global__ void __launch_bounds__(EV_NT, 3) k_eval_listed(const EvalRowArgsT<T> a, const EvalWs w, const EvalOut o,
                                                          int64_t* xcnt) {
  __shared__ float s_rows[EV_NT * EL_LD];
  __shared__ float s_u[EL_KS];
  __shared__ int32_t s_row[EV_NT];     // local item row of chunk entry t, -1: not scored on this rank
  __shared__ unsigned long long s_auc;
  __shared__ long long s_eval;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t P = a.P;
  const int info = w.info[2 * b];
  if (info < 0) {                      // a positive row longer than max_pos
    if (xcnt)
      for (int j = tid; j < a.P; j += EV_NT) xcnt[b * P + j] = 0;
    else
      ev_nan_row(o, b);
    return;
  }
  const int n = info, n_auc = w.info[2 * b + 1];
  const float* pth = w.keys + b * P;
  const float* sth = w.keys + (a.Bu + b) * P;
  unsigned* hist = w.hist + b * P;
  const float pmin = n_auc ? pth[0] : __int_as_float(0x7f800000);
  const float pmax = n_auc ? pth[n_auc - 1] : __int_as_float(0xff800000);
  const float smin = n ? sth[0] : __int_as_float(0x7f800000);
  const float smax = n ? sth[n - 1] : __int_as_float(0x7f800000);
  const EvRow r = ev_row(a, b);
  int64_t lo, hi;
  el_range(a, b, &lo, &hi);
  const T* urow = ev_urow(a, b);
  if (tid == 0) {
    s_auc = 0ull;
    s_eval = 0;
  }
  for (int q = tid; q < n; q += EV_NT) {
    const int32_t i = a.pos_items[r.plo + q];
    if (!ev_owns(a, i) || ev_contains(a.excl_items, r.elo, r.ehi, i)) continue;
    const int j = ev_rank_slot(sth, n, smin, smax, expf(ev_score1<KIND>(a, urow, i)));
    if (j) atomicAdd(hist + j, 1u);
  }
  unsigned long long auc = 0ull;
  long long n_eval = 0;
  for (int64_t c0 = lo; c0 < hi; c0 += EV_NT) {
    const int nc = (int)min((int64_t)EV_NT, hi - c0);
    int32_t row = -1;
    if (tid < nc && el_eval_item(a, r, c0 + tid)) {
      ++n_eval;
      const int32_t i = a.neg_items[c0 + tid];
      if (ev_owns(a, i)) row = (int32_t)ev_local(a, i);
    }
    s_row[tid] = row;
    float acc = 0.f;
    for (int k0 = 0; k0 < a.D; k0 += EL_KS) {
      const int ks = min(EL_KS, a.D - k0);
      __syncthreads();                 // s_row written; the previous slab consumed
      if (tid < ks) s_u[tid] = ev_uval(a, urow, k0 + tid);
      for (int t0 = warp; t0 < nc; t0 += (EV_NT / 32) * EL_UNR) {
        float v[EL_UNR];
#pragma unroll
        for (int x = 0; x < EL_UNR; ++x) {
          const int t = t0 + (EV_NT / 32) * x;
          const int32_t rt = t < nc ? s_row[t] : -1;
          v[x] = rt >= 0 && lane < ks ? orx_ld1(a.item_tab + (int64_t)rt * a.D + k0 + lane) : 0.f;
        }
#pragma unroll
        for (int x = 0; x < EL_UNR; ++x) {
          const int t = t0 + (EV_NT / 32) * x;
          if (t < nc) s_rows[t * EL_LD + lane] = v[x];
        }
      }
      __syncthreads();
      if (row >= 0)
        for (int k = 0; k < ks; ++k) acc = ev_step<KIND>(acc, s_u[k], s_rows[tid * EL_LD + k]);
    }
    if (row >= 0) {
      const float s = acc + (a.bias ? a.bias[row] : 0.f);
      auc += ev_auc_count(pth, n_auc, pmin, pmax, s);
      const int j = ev_rank_slot(sth, n, smin, smax, expf(s));
      if (j) atomicAdd(hist + j, 1u);
    }
  }
  __syncthreads();                     // s_auc / s_eval initialised (a row without listed items has no chunk)
  if (auc) atomicAdd(&s_auc, auc);
  if (n_eval) atomicAdd(reinterpret_cast<unsigned long long*>(&s_eval), (unsigned long long)n_eval);
  __syncthreads();
  if (xcnt) {
    for (int j = tid; j < a.P; j += EV_NT) xcnt[b * P + j] = j == 0 ? (int64_t)s_auc : j <= n ? (int64_t)hist[j] : 0;
    return;
  }
  ev_finish_row(a, o, b, n, a.I_all - n - s_eval, s_auc, [&](int j) { return hist[j]; });
}

// Sharded phase 3 of orx_score_rank_listed_shard: the outputs from the counts summed over the ranks; n and n_eval come
// from the lists alone.
__global__ void __launch_bounds__(EV_NT) k_eval_listed_finish_counts(const EvalRowArgs a, const int64_t* xcnt,
                                                                     const EvalOut o) {
  __shared__ long long s_eval;
  const int b = blockIdx.x, tid = threadIdx.x;
  const EvRow r = ev_row(a, b);
  if (r.bad) {
    ev_nan_row(o, b);
    return;
  }
  const int n = (int)(r.phi - r.plo);
  int64_t lo, hi;
  el_range(a, b, &lo, &hi);
  if (tid == 0) s_eval = 0;
  __syncthreads();
  long long n_eval = 0;
  for (int64_t q = lo + tid; q < hi; q += EV_NT) n_eval += el_eval_item(a, r, q) ? 1 : 0;
  if (n_eval) atomicAdd(reinterpret_cast<unsigned long long*>(&s_eval), (unsigned long long)n_eval);
  __syncthreads();
  const int64_t* cnt = xcnt + (int64_t)b * a.P;
  ev_finish_row(a, o, b, n, a.I_all - n - s_eval, (unsigned long long)cnt[0], [&](int j) { return (unsigned)cnt[j]; });
}

// ---------------------------------------------------------------------------------------
// top-K retrieval (orx_score_topk).  Key of an eligible (score s, item i): the order-preserving bits of s (-0 taken as
// +0) in the high word, ~i in the low word, so "score descending, then item ascending" is ">" on keys; keys are unique
// and every real key is > 0, which marks an empty slot.  NaN scores never form a key.
// ---------------------------------------------------------------------------------------
// Room of a candidate list beyond k.  A tile appends at most 128 keys to a row's list, so a list is cut back to k only
// once it holds more than k + TK_ROOM - 128 keys (and once after the CTA's last tile): every few tiles while the
// threshold warms up or when scores rise with item id, rarely after that.
constexpr int TK_ROOM = 1024;

struct TopkWs {
  unsigned long long* cand;   // [Bu][splits][k + TK_ROOM]: the candidate list of (row, item split)
  int* cnt;                   // [Bu][splits]: its length after the split's last tile (<= k)
};

__device__ __forceinline__ unsigned long long tk_key(float s, int64_t i) {
  unsigned u = __float_as_uint(s == 0.f ? 0.f : s);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | (unsigned)~(uint32_t)i;
}

__device__ __forceinline__ float tk_score(unsigned long long key) {
  const unsigned u = (unsigned)(key >> 32);
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

template <int NT>
__device__ __forceinline__ void tk_sync() {
  if (NT == 32) __syncwarp();
  else __syncthreads();
}

// The k-th largest (1 <= k <= number of keys) of a set of unique keys, found by NT threads (one warp, or the CTA) that
// visit the keys through each(fn): a radix select, 8 bits per pass from the most significant byte, with the 256-bin
// histogram hist in shared memory.  t = the thread's index in the group; s_sel: CTA-wide broadcast (NT > 32 only).
template <int NT, class Each>
__device__ unsigned long long tk_kth(Each each, int k, unsigned* hist, unsigned long long* s_sel, int t) {
  unsigned long long prefix = 0ull, mask = 0ull;
  unsigned kk = (unsigned)k;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int j = t; j < 256; j += NT) hist[j] = 0u;
    tk_sync<NT>();
    each([&](unsigned long long v) {
      if ((v & mask) == prefix) {
        const unsigned bin = (unsigned)(v >> shift) & 255u;
        if (NT == 32) {
          atomicAdd(&hist[bin], 1u);
        } else {   // CTA-wide: one atomic per distinct bin of the converged lanes (keys share their leading bytes)
          const unsigned peers = __match_any_sync(__activemask(), bin);
          if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[bin], (unsigned)__popc(peers));
        }
      }
    });
    tk_sync<NT>();
    if (t < 32) {   // the digit d with fewer than kk keys in the bins above it and at least kk from d up
      unsigned c[8], sum = 0u;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = hist[255 - 8 * t - j];
        sum += c[j];
      }
      unsigned incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_up_sync(ORX_FULL, incl, o);
        if (t >= o) incl += v;
      }
      const int src = __ffs(__ballot_sync(ORX_FULL, incl >= kk)) - 1;
      unsigned run = incl - sum, above = 0u;
      int d = 0;
      if (t == src)
        for (int j = 0; j < 8; ++j) {
          if (run + c[j] >= kk) {
            d = 255 - 8 * t - j;
            above = run;
            break;
          }
          run += c[j];
        }
      d = __shfl_sync(ORX_FULL, d, src);
      above = __shfl_sync(ORX_FULL, above, src);
      prefix |= (unsigned long long)d << shift;
      kk -= above;
      if (NT > 32 && t == 0) {
        s_sel[0] = prefix;
        s_sel[1] = kk;
      }
    }
    if (NT > 32) {
      __syncthreads();
      prefix = s_sel[0];
      kk = (unsigned)s_sel[1];
    }
    mask |= 0xffull << shift;
  }
  return prefix;
}

// Main pass: the tile loop of k_score_rank with a top-K epilogue.  Row r of the CTA's user tile keeps a threshold key
// (0 until its list is first cut) and appends every eligible key above it to its list in the scratch.  Cutting a list
// (one warp) keeps its exact top k, and the threshold becomes the k-th key.
template <typename T>
struct TkRow {
  const T* urow;
  int64_t elo, ehi;   // the row's exclusion entries in [0, I)
};

// SHARD: the tile loop walks this rank's a.I local rows of a row-sharded table (local row i is item i * world + rank of
// [0, I_all)) and takes user rows by batch position (a.user_tab = the summed exchange); keys and the exclusion lookup
// use the global item id, so keys stay unique across ranks and equal scores order by global id as on one device.
template <int KIND, bool SHARD, typename T, bool VEC = false>
__device__ __forceinline__ void tk_main(const EvalArgsT<T>& a, const TopkWs& w, int k, int world, int rank, int64_t I_all) {
  __shared__ __align__(16) float sA[2][EV_KC][EV_LD];
  __shared__ __align__(16) float sB[2][EV_KC][EV_LD];
  __shared__ TkRow<T> meta[EV_TU];
  __shared__ unsigned long long s_thr[EV_TU];
  __shared__ int s_cnt[EV_TU];
  __shared__ unsigned s_hist[EV_NT / 32][256];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tx = tid & 15, ty = tid >> 4;
  const int u0 = blockIdx.y * EV_TU;
  const int rows = min(EV_TU, a.Bu - u0);
  const int64_t C = (int64_t)k + TK_ROOM;
  auto list = [&](int r) { return w.cand + ((int64_t)(u0 + r) * gridDim.x + blockIdx.x) * C; };
  // cut every list of the tile longer than `limit` to its top k (after a __syncthreads that follows the appends); the
  // CTA's last tile cuts every list longer than k (a CTA has at least one tile: splits <= item tiles)
  const int64_t n_tiles = (a.I + EV_TI - 1) / EV_TI;
  const int64_t last_i0 = (n_tiles * (blockIdx.x + 1) / gridDim.x - 1) * EV_TI;
  auto cut = [&](int limit) {
    for (int r = warp; r < rows; r += EV_NT / 32) {
      const int n = s_cnt[r];
      if (n <= limit) continue;
      unsigned long long* keys = list(r);
      const unsigned long long t = tk_kth<32>([&](auto fn) {
        for (int q = lane; q < n; q += 32) fn(keys[q]);
      }, k, s_hist[warp], nullptr, lane);
      // keep the k keys >= t, in place: a chunk is read before any of its slots is written
      int kept = 0;
      for (int q0 = 0; q0 < n; q0 += 32) {
        const unsigned long long v = q0 + lane < n ? keys[q0 + lane] : 0ull;
        const unsigned keep = __ballot_sync(ORX_FULL, v >= t);
        if (v >= t) keys[kept + __popc(keep & ((1u << lane) - 1u))] = v;
        kept += __popc(keep);
      }
      __syncwarp();
      if (lane == 0) {
        s_thr[r] = t;
        s_cnt[r] = k;
      }
    }
  };

  if (tid < EV_TU) {
    TkRow<T> m = {};
    if (tid < rows) {
      int64_t raw;
      m.urow = ev_user_row<SHARD>(a, u0 + tid);
      ev_range(a.excl_off, a.excl_items, a.uid[u0 + tid], a.U, SHARD ? I_all : a.I, &m.elo, &m.ehi, &raw);
    }
    meta[tid] = m;
    s_thr[tid] = 0ull;
    s_cnt[tid] = 0;
  }
  __syncthreads();

  ev_tiles<KIND, VEC>(a, sA, sB, [&](int r) { return meta[r].urow; }, [&](int64_t i0, const float (&acc)[8][8]) {
    float bv[8];
#pragma unroll
    for (int y = 0; y < 8; ++y) {
      const int64_t i = i0 + ev_frag(tx, y);
      bv[y] = (a.bias && i < a.I) ? a.bias[i] : 0.f;
    }
#pragma unroll
    for (int x = 0; x < 8; ++x) {
      const int r = ev_frag(ty, x);
      if (r >= rows) continue;
      const unsigned long long thr = s_thr[r];
#pragma unroll
      for (int y = 0; y < 8; ++y) {
        const int64_t i = i0 + ev_frag(tx, y);
        const float s = acc[x][y] + bv[y];
        if (i >= a.I || s != s) continue;
        const int64_t ig = SHARD ? (int32_t)i * world + rank : i;   // a global id is < 2^31
        const unsigned long long key = tk_key(s, ig);
        if (key <= thr || ev_contains(a.excl_items, meta[r].elo, meta[r].ehi, (int32_t)ig)) continue;
        list(r)[atomicAdd(&s_cnt[r], 1)] = key;
      }
    }
    __syncthreads();
    cut(i0 == last_i0 ? k : k + TK_ROOM - EV_TI);
  });
  __syncthreads();
  if (tid < rows) w.cnt[(int64_t)(u0 + tid) * gridDim.x + blockIdx.x] = s_cnt[tid];
}

template <int KIND, typename T, bool VEC = false>
__global__ void __launch_bounds__(EV_NT, 2) k_score_topk(const EvalArgsT<T> a, const TopkWs w, int k) {
  tk_main<KIND, false, T, VEC>(a, w, k, 1, 0, a.I);
}

// Sharded phase 1's main pass (a.user_tab: the summed user rows of phase 0, by batch position).
template <int KIND>
__global__ void __launch_bounds__(EV_NT, 2) k_score_topk_shard(const EvalArgs a, const TopkWs w, int k, int world,
                                                               int rank, int64_t I_all) {
  tk_main<KIND, true>(a, w, k, world, rank, I_all);
}

// Merge of one batch row (the CTA): the top k of the union of its lists (radix select when the union is larger), sorted
// descending into s_key[0, k) (bitonic), 0 past the keys.  The lists: the row's split lists of k_score_topk (stride
// k + TK_ROOM, cnt[s] keys each), or with XIN the summed exchange of the sharded phase 1 (`lists` ranks' lists of stride
// k, each sorted descending and padded with 0).  Only real keys are counted and visited, never padding: keys are
// unique (global item ids), so at most k of them are >= the k-th and s_key cannot overflow.
template <bool XIN>
__device__ __forceinline__ void tk_merge(const unsigned long long* cand, const int* cnt, int lists, int k,
                                         unsigned long long* s_key) {
  __shared__ unsigned s_hist[256];
  __shared__ unsigned long long s_sel[2];
  __shared__ int s_n, s_m;
  const int tid = threadIdx.x;
  const int C = k + TK_ROOM;
  auto each = [&](auto fn) {   // lists * k <= 2^31: the grid has at most a few thousand CTAs; the caller checks world
    for (int e = tid; e < lists * k; e += EV_NT) {
      if (XIN) {
        if (cand[e]) fn(cand[e]);
        continue;
      }
      const int s = e / k, q = e - s * k;
      if (q < cnt[s]) fn(cand[(int64_t)s * C + q]);
    }
  };
  if (tid == 0) {
    s_n = 0;
    s_m = 0;
  }
  __syncthreads();
  int part = 0;
  if (XIN)
    for (int e = tid; e < lists * k; e += EV_NT) part += cand[e] != 0ull;
  else
    for (int s = tid; s < lists; s += EV_NT) part += cnt[s];
  if (part) atomicAdd(&s_n, part);
  __syncthreads();
  const int n = s_n;
  const unsigned long long t = n > k ? tk_kth<EV_NT>(each, k, s_hist, s_sel, tid) : 1ull;
  each([&](unsigned long long v) {
    if (v >= t) s_key[atomicAdd(&s_m, 1)] = v;
  });
  int p2 = 1;
  while (p2 < k) p2 <<= 1;
  const int m = min(n, k);
  for (int j = m + tid; j < p2; j += EV_NT) s_key[j] = 0ull;
  __syncthreads();
  for (int size = 2; size <= p2; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < p2; i += EV_NT) {
        const int j = i ^ stride;
        if (j > i) {
          const unsigned long long x = s_key[i], y = s_key[j];
          if ((x < y) == ((i & size) == 0)) {
            s_key[i] = y;
            s_key[j] = x;
          }
        }
      }
      __syncthreads();
    }
}

// Row b's merged keys decoded; slots past the eligible items get item -1, -inf.
__device__ __forceinline__ void tk_decode(const unsigned long long* s_key, int b, int k, int32_t* top_items,
                                          float* top_scores) {
  for (int j = threadIdx.x; j < k; j += EV_NT) {
    const unsigned long long key = s_key[j];
    top_items[(int64_t)b * k + j] = key ? (int32_t)~(uint32_t)key : -1;
    if (top_scores) top_scores[(int64_t)b * k + j] = key ? tk_score(key) : __int_as_float(0xff800000);
  }
}

// Merge: one CTA per batch row, over the row's split lists.
__global__ void __launch_bounds__(EV_NT) k_topk_merge(const TopkWs w, int splits, int k, int32_t* top_items,
                                                      float* top_scores) {
  __shared__ unsigned long long s_key[ORX_MAX_TOPK];
  const int b = blockIdx.x;
  tk_merge<false>(w.cand + (int64_t)b * splits * (k + TK_ROOM), w.cnt + (int64_t)b * splits, splits, k, s_key);
  tk_decode(s_key, b, k, top_items, top_scores);
}

// Sharded phase 1's local merge: this rank's top k of row b, as raw keys, into slot [b][rank] of xkeys[Bu][world][k].
__global__ void __launch_bounds__(EV_NT) k_topk_merge_local(const TopkWs w, int splits, int k, int world, int rank,
                                                            unsigned long long* xkeys) {
  __shared__ unsigned long long s_key[ORX_MAX_TOPK];
  const int b = blockIdx.x;
  tk_merge<false>(w.cand + (int64_t)b * splits * (k + TK_ROOM), w.cnt + (int64_t)b * splits, splits, k, s_key);
  unsigned long long* slot = xkeys + ((int64_t)b * world + rank) * k;
  for (int j = threadIdx.x; j < k; j += EV_NT) slot[j] = s_key[j];
}

// Sharded phase 2: row b's top k over the world ranks' lists of the summed xkeys, decoded.
__global__ void __launch_bounds__(EV_NT) k_topk_merge_ranks(const unsigned long long* xkeys, int world, int k,
                                                            int32_t* top_items, float* top_scores) {
  __shared__ unsigned long long s_key[ORX_MAX_TOPK];
  const int b = blockIdx.x;
  tk_merge<true>(xkeys + (int64_t)b * world * k, nullptr, world, k, s_key);
  tk_decode(s_key, b, k, top_items, top_scores);
}

// The call's scratch inside one allocation; with base == nullptr only the size is computed.
size_t ev_layout(char* base, int Bu, int P, size_t sort_bytes, EvalWs* w) {
  const size_t nk = (size_t)2 * Bu * P;
  OrxCarve m = {base, 0};
  w->keys_in = reinterpret_cast<float*>(m.take(sizeof(float) * nk));
  w->keys = reinterpret_cast<float*>(m.take(sizeof(float) * nk));
  w->seg_begin = reinterpret_cast<int*>(m.take(sizeof(int) * 2 * (size_t)Bu));
  w->seg_end = reinterpret_cast<int*>(m.take(sizeof(int) * 2 * (size_t)Bu));
  w->hist = reinterpret_cast<unsigned*>(m.take(sizeof(unsigned) * (size_t)Bu * P));
  w->auc_cnt = reinterpret_cast<unsigned long long*>(m.take(sizeof(unsigned long long) * (size_t)Bu));
  w->info = reinterpret_cast<int*>(m.take(sizeof(int) * 2 * (size_t)Bu));
  w->sort_tmp = m.take(sort_bytes);
  w->sort_bytes = sort_bytes;
  return m.off;
}

// Whether a call's tile loop runs the VEC loader of ev_tiles: bf16 tables, dim % 4 == 0 and both tables 8-byte
// aligned (so is every row start).  Any other table takes the scalar loader, with the same bits.
template <typename T>
bool ev_vec(const EvalArgsT<T>& a) {
  const uintptr_t bases = reinterpret_cast<uintptr_t>(a.user_tab) | reinterpret_cast<uintptr_t>(a.item_tab);
  return std::is_same<T, uint16_t>::value && a.D % 4 == 0 && bases % 8 == 0;
}

// Item splits of a grid of user tiles x item splits for kern at dyn bytes of dynamic shared memory: enough CTAs for one
// wave over the SMs, at most one item tile per CTA.
template <class Kern>
int ev_item_splits(const orx_ctx* h, Kern kern, size_t dyn, int Bu, int64_t I, int64_t* splits) {
  int per_sm = 0;
  ORX_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, EV_NT, dyn));
  if (per_sm < 1) per_sm = 1;
  const int64_t user_tiles = (Bu + EV_TU - 1) / EV_TU;
  const int64_t item_tiles = (I + EV_TI - 1) / EV_TI;
  int64_t s = ((int64_t)h->num_sms * per_sm + user_tiles - 1) / user_tiles;
  if (s > item_tiles) s = item_tiles;
  *splits = s < 1 ? 1 : s;
  return ORX_OK;
}

// The handle's evaluation scratch for Bu rows of P thresholds each.
int ev_workspace(orx_ctx* h, int Bu, int P, cudaStream_t st, EvalWs* w) {
  size_t sort_bytes = 0;
  ORX_CUDA(cub::DeviceSegmentedSort::SortKeys((void*)nullptr, sort_bytes, (const float*)nullptr, (float*)nullptr,
                                              2 * Bu * P, 2 * Bu, (const int*)nullptr, (const int*)nullptr, st));
  const int rc = orx_grow(&h->eval_ws, &h->eval_cap, ev_layout(nullptr, Bu, P, sort_bytes, w));
  if (rc != ORX_OK) return rc;
  ev_layout(static_cast<char*>(h->eval_ws), Bu, P, sort_bytes, w);
  return ORX_OK;
}

// prep and the segmented sort: every batch row's sorted thresholds, zeroed histogram and AUC count in w.
template <int KIND, typename T>
int ev_prep_sort(const EvalRowArgsT<T>& a, const EvalWs& w, cudaStream_t st) {
  k_eval_prep<KIND><<<a.Bu, EV_NT, 0, st>>>(a, w);
  ORX_LAUNCH_CHECK();
  size_t bytes = w.sort_bytes;
  ORX_CUDA(cub::DeviceSegmentedSort::SortKeys(w.sort_tmp, bytes, (const float*)w.keys_in, w.keys, 2 * a.Bu * a.P,
                                              2 * a.Bu, (const int*)w.seg_begin, (const int*)w.seg_end, st));
  return ORX_OK;
}

// prep, sort and the main pass over the a.I item rows (no main pass when a.I == 0): the thresholds, AUC counts and
// rank histograms of every batch row in w, before the take-back.  *variant / *splits: the main pass's dispatch fields
// (splits 0: not launched).
template <int KIND, bool XROWS, typename T>
int ev_count(orx_ctx* h, const EvalRowArgsT<T>& a, const EvalWs& w, cudaStream_t st, int* variant, int64_t* splits) {
  auto kern = k_score_rank<KIND, XROWS, T, false>;
  if constexpr (std::is_same<T, uint16_t>::value)
    if (ev_vec(a)) kern = k_score_rank<KIND, XROWS, T, true>;
  int optin = 0;
  ORX_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
  cudaFuncAttributes fa;
  ORX_CUDA(cudaFuncGetAttributes(&fa, kern));
  const size_t dyn_max = (size_t)optin - fa.sharedSizeBytes;
  // thresholds (pred, sp) and histogram of every row of a user tile in shared memory when they fit, for every tile
  const size_t rows_alloc = (size_t)(a.Bu < EV_TU ? a.Bu : EV_TU);
  const size_t dyn_need = 3 * sizeof(float) * rows_alloc * (size_t)a.P;
  const int use_smem = dyn_need <= dyn_max ? 1 : 0;
  const size_t dyn = use_smem ? dyn_need : 0;
  ORX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_max));
  *variant = use_smem ? ORX_VARIANT_RANK_SMEM : ORX_VARIANT_RANK_GLOBAL;
  *splits = 0;
  if (a.I > 0) {
    const int rc = ev_item_splits(h, kern, dyn, a.Bu, a.I, splits);
    if (rc != ORX_OK) return rc;
  }
  const int64_t user_tiles = (a.Bu + EV_TU - 1) / EV_TU;

  const int rc = ev_prep_sort<KIND>(a, w, st);
  if (rc != ORX_OK) return rc;
  if (*splits > 0) {
    EvalArgsT<T> t = a;
    if (XROWS) t.user_tab = a.xrows;
    kern<<<dim3((unsigned)*splits, (unsigned)user_tiles), EV_NT, dyn, st>>>(t, w, use_smem);
    ORX_LAUNCH_CHECK();
  }
  return ORX_OK;
}

// The dispatch op of an orx_score_rank / orx_score_topk call on tables of storage T.
template <typename T>
constexpr int ev_op(int op_fp32, int op_bf16) { return std::is_same<T, uint16_t>::value ? op_bf16 : op_fp32; }

template <int KIND, typename T>
int ev_launch(orx_ctx* h, const EvalRowArgsT<T>& a, const EvalWs& w, const EvalOut& o, cudaStream_t st) {
  int variant = 0;
  int64_t splits = 0;
  const int rc = ev_count<KIND, false>(h, a, w, st, &variant, &splits);
  if (rc != ORX_OK) return rc;
  k_eval_finish<KIND><<<a.Bu, EV_NT, 0, st>>>(a, w, o);
  ORX_LAUNCH_CHECK();
  orx_log_dispatch(h, ev_op<T>(ORX_OP_SCORE_RANK, ORX_OP_SCORE_RANK_BF16), variant, KIND, 0, a.Bu,
                   (int)(a.I > INT32_MAX ? INT32_MAX : a.I), a.D, (int)splits);
  return ORX_OK;
}

// Phase 0 of orx_score_rank_shard and orx_score_topk_shard: the bits of this rank's user rows of the batch.
void ev_user_rows(const EvalRowArgs& a, int32_t* xrows, cudaStream_t st) {
  const int64_t blocks = ((int64_t)a.Bu * a.D + EV_NT - 1) / EV_NT;
  k_eval_user_rows<<<(unsigned)(blocks < 4096 ? blocks : 4096), EV_NT, 0, st>>>(a, xrows);
}

// orx_score_rank_listed's counts of every batch row from the handle's evaluation scratch: its outputs (xcnt nullptr),
// or phase 2 of orx_score_rank_listed_shard (the counts into xcnt).
template <int KIND, typename T>
int el_launch(orx_ctx* h, const EvalRowArgsT<T>& a, const EvalOut& o, int64_t* xcnt, cudaStream_t st) {
  EvalWs w;
  int rc = ev_workspace(h, a.Bu, a.P, st, &w);
  if (rc != ORX_OK) return rc;
  rc = ev_prep_sort<KIND>(a, w, st);
  if (rc != ORX_OK) return rc;
  k_eval_listed<KIND><<<a.Bu, EV_NT, 0, st>>>(a, w, o, xcnt);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// One phase of orx_score_rank_shard, or with `listed` of orx_score_rank_listed_shard (arguments checked by the
// caller).  Phases 0 and 1 are the same for both.
template <int KIND>
int ev_shard_phase(orx_ctx* h, int phase, bool listed, const EvalRowArgs& a, const EvalOut& o, int32_t* xrows,
                   int32_t* xpred, int64_t* xcnt, cudaStream_t st) {
  if (phase == 0) {
    ev_user_rows(a, xrows, st);
  } else if (phase == 1) {
    k_eval_pos_scores<KIND><<<a.Bu, EV_NT, 0, st>>>(a, xpred);
  } else if (phase == 2 && listed) {
    return el_launch<KIND>(h, a, o, xcnt, st);
  } else if (phase == 3 && listed) {
    k_eval_listed_finish_counts<<<a.Bu, EV_NT, 0, st>>>(a, xcnt, o);
  } else if (phase == 2) {
    EvalWs w;
    int rc = ev_workspace(h, a.Bu, a.P, st, &w);
    if (rc != ORX_OK) return rc;
    int variant = 0;
    int64_t splits = 0;
    rc = ev_count<KIND, true>(h, a, w, st, &variant, &splits);
    if (rc != ORX_OK) return rc;
    k_eval_correct<KIND><<<a.Bu, EV_NT, 0, st>>>(a, w, xcnt);
    ORX_LAUNCH_CHECK();
    orx_log_dispatch(h, ORX_OP_SCORE_RANK_SHARD, variant, KIND, a.rank, a.Bu, (int)a.I, a.D, (int)splits);
    return ORX_OK;
  } else {
    k_eval_finish_counts<<<a.Bu, EV_NT, 0, st>>>(a, xcnt, o);
  }
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// The top-K scratch of Bu rows over `splits` item splits inside one allocation; with base == nullptr only the size.
size_t tk_layout(char* base, int Bu, int64_t splits, int k, TopkWs* w) {
  const size_t lists = (size_t)Bu * (size_t)splits;
  OrxCarve m = {base, 0};
  w->cand = reinterpret_cast<unsigned long long*>(m.take(sizeof(unsigned long long) * lists * ((size_t)k + TK_ROOM)));
  w->cnt = reinterpret_cast<int*>(m.take(sizeof(int) * lists));
  return m.off;
}

// The item splits of kern over a.I rows and the top-K scratch for them, from the handle's evaluation scratch.
template <class Kern, typename T>
int tk_workspace(orx_ctx* h, Kern kern, const EvalArgsT<T>& a, int k, int64_t* splits, TopkWs* w) {
  int rc = ev_item_splits(h, kern, 0, a.Bu, a.I, splits);
  if (rc != ORX_OK) return rc;
  rc = orx_grow(&h->eval_ws, &h->eval_cap, tk_layout(nullptr, a.Bu, *splits, k, w));
  if (rc != ORX_OK) return rc;
  tk_layout(static_cast<char*>(h->eval_ws), a.Bu, *splits, k, w);
  return ORX_OK;
}

template <int KIND, typename T>
int tk_launch(orx_ctx* h, const EvalArgsT<T>& a, int k, int32_t* top_items, float* top_scores, cudaStream_t st) {
  int64_t splits = 1;
  TopkWs w;
  auto kern = k_score_topk<KIND, T, false>;
  if constexpr (std::is_same<T, uint16_t>::value)
    if (ev_vec(a)) kern = k_score_topk<KIND, T, true>;
  const int rc = tk_workspace(h, kern, a, k, &splits, &w);
  if (rc != ORX_OK) return rc;
  const int64_t user_tiles = (a.Bu + EV_TU - 1) / EV_TU;
  kern<<<dim3((unsigned)splits, (unsigned)user_tiles), EV_NT, 0, st>>>(a, w, k);
  ORX_LAUNCH_CHECK();
  k_topk_merge<<<a.Bu, EV_NT, 0, st>>>(w, (int)splits, k, top_items, top_scores);
  ORX_LAUNCH_CHECK();
  orx_log_dispatch(h, ev_op<T>(ORX_OP_SCORE_TOPK, ORX_OP_SCORE_TOPK_BF16), ORX_VARIANT_TOPK, KIND, k, a.Bu, (int)a.I,
                   a.D, (int)splits);
  return ORX_OK;
}

// Phase 1 of orx_score_topk_shard (arguments checked by the caller): xkeys all 0, then, when this rank has item rows,
// the main pass over them and the local merge into slot [b][rank].  Only the scratch of this call is used.
template <int KIND>
int tk_shard_local(orx_ctx* h, const EvalArgs& a, int k, int world, int rank, int64_t I_all,
                   unsigned long long* xkeys, cudaStream_t st) {
  ORX_CUDA(cudaMemsetAsync(xkeys, 0, sizeof(unsigned long long) * (size_t)a.Bu * world * k, st));
  int64_t splits = 0;
  if (a.I > 0) {
    TopkWs w;
    const int rc = tk_workspace(h, k_score_topk_shard<KIND>, a, k, &splits, &w);
    if (rc != ORX_OK) return rc;
    const int64_t user_tiles = (a.Bu + EV_TU - 1) / EV_TU;
    k_score_topk_shard<KIND><<<dim3((unsigned)splits, (unsigned)user_tiles), EV_NT, 0, st>>>(a, w, k, world, rank,
                                                                                             I_all);
    ORX_LAUNCH_CHECK();
    k_topk_merge_local<<<a.Bu, EV_NT, 0, st>>>(w, (int)splits, k, world, rank, xkeys);
    ORX_LAUNCH_CHECK();
  }
  orx_log_dispatch(h, ORX_OP_SCORE_TOPK_SHARD, ORX_VARIANT_TOPK, KIND, rank, a.Bu, (int)a.I, a.D, (int)splits);
  return ORX_OK;
}

EvalOut ev_out(const int32_t* at_host, int n_at, float* auc, float* ndcg, float* recall) {
  EvalOut o;
  for (int k = 0; k < ORX_MAX_AT; ++k) o.at[k] = k < n_at ? at_host[k] : 0;
  o.n_at = n_at; o.auc = auc; o.ndcg = ndcg; o.recall = recall;
  return o;
}

// Why orx_score_rank / orx_score_rank_listed refuse their arguments, or nullptr (the size limit only for Bu > 0).
const char* ev_rank_refusal(orx_handle_t h, int32_t kind, const void* user_tab, int64_t U, const int32_t* uid,
                            int32_t Bu, const void* item_tab, int64_t I, int32_t dim, const int64_t* pos_off,
                            int32_t max_pos, const int32_t* at_host, int32_t n_at) {
  if (!(h != nullptr && user_tab && uid && item_tab && pos_off)) return "null pointer";
  if (!(kind == ORX_SCORE_DOT || kind == ORX_SCORE_NEG_SQDIST)) return "unknown score kind";
  if (!(U > 0 && I > 0 && I <= INT32_MAX && dim > 0 && Bu >= 0 && max_pos >= 0)) return "bad sizes";
  if (!(n_at >= 0 && n_at <= ORX_MAX_AT)) return "at most 8 cut-offs";
  if (!(n_at == 0 || at_host)) return "null cut-offs";
  if (Bu > 0 && 2 * (int64_t)Bu * ((int64_t)max_pos + 1) > INT32_MAX)
    return "Bu * (max_pos + 1) too large for one call: split the batch";
  return nullptr;
}

// The row arguments of a checked orx_score_rank / orx_score_rank_listed call (neg_off nullptr for the former).
template <typename T>
EvalRowArgsT<T> ev_rank_args(const T* user_tab, int64_t U, const int32_t* uid, int32_t Bu, const float* scale,
                             const T* item_tab, const float* item_bias, int64_t I, int32_t dim, const int64_t* pos_off,
                             const int32_t* pos_items, const int64_t* neg_off, const int32_t* neg_items,
                             const int64_t* excl_off, const int32_t* excl_items, int32_t max_pos) {
  EvalRowArgsT<T> a = {};
  a.user_tab = user_tab; a.U = U; a.uid = uid; a.Bu = Bu; a.scale = scale; a.item_tab = item_tab;
  a.bias = item_bias; a.I = I; a.I_all = I; a.world = 1; a.rank = 0; a.D = dim; a.pos_off = pos_off;
  a.excl_off = excl_off; a.pos_items = pos_items; a.excl_items = excl_items; a.max_pos = max_pos; a.P = max_pos + 1;
  a.neg_off = neg_off; a.neg_items = neg_items;
  return a;
}

// Why orx_score_rank_shard / orx_score_rank_listed_shard refuse their arguments, or nullptr (the size limit and the
// buffer checks only for Bu > 0).
const char* ev_shard_refusal(orx_handle_t h, int32_t kind, int32_t phase, const orx_rowshard_t* g_host,
                             const float* user_shard, const float* item_shard, int32_t dim, const int32_t* uid,
                             int32_t Bu, const int64_t* pos_off, int32_t max_pos, const int32_t* at_host, int32_t n_at,
                             const int32_t* xrows, const int32_t* xpred, const int64_t* xcnt) {
  if (!(h != nullptr && g_host != nullptr)) return "null pointer";
  if (!(kind == ORX_SCORE_DOT || kind == ORX_SCORE_NEG_SQDIST)) return "unknown score kind";
  if (!(phase >= 0 && phase <= 3)) return "phase must lie in [0, 3]";
  const orx_rowshard_t g = *g_host;
  if (!(g.world >= 1 && g.rank >= 0 && g.rank < g.world)) return "rank must lie in [0, world)";
  if (!(g.total_users > 0 && g.total_items > 0 && g.total_items <= INT32_MAX)) return "bad table sizes";
  if (!(g.local_users == (g.total_users - g.rank + g.world - 1) / g.world &&
        g.local_items == (g.total_items - g.rank + g.world - 1) / g.world))
    return "local_users / local_items disagree with (total, world, rank)";
  if (!(dim > 0 && Bu >= 0 && max_pos >= 0)) return "bad sizes";
  if (!(n_at >= 0 && n_at <= ORX_MAX_AT)) return "at most 8 cut-offs";
  if (!(n_at == 0 || at_host)) return "null cut-offs";
  if (Bu == 0) return nullptr;
  if (2 * (int64_t)Bu * ((int64_t)max_pos + 1) > INT32_MAX)
    return "Bu * (max_pos + 1) too large for one call: split the batch";
  if (!(uid && pos_off)) return "null pointer";
  if (!(phase != 0 || (user_shard && xrows))) return "phase 0 needs user_shard and xrows";
  if (!(phase != 1 || (item_shard && xrows && xpred))) return "phase 1 needs item_shard, xrows and xpred";
  if (!(phase != 2 || (item_shard && xrows && xpred && xcnt))) return "phase 2 needs item_shard, xrows, xpred, xcnt";
  if (!(phase != 3 || xcnt)) return "phase 3 needs xcnt";
  return nullptr;
}

// The row arguments of a checked sharded phase (neg_off nullptr for orx_score_rank_shard).
EvalRowArgs ev_shard_args(int32_t phase, const orx_rowshard_t& g, const float* user_shard, const float* item_shard,
                          const float* bias_shard, int32_t dim, const int32_t* uid, int32_t Bu,
                          const int64_t* pos_off, const int32_t* pos_items, const int64_t* neg_off,
                          const int32_t* neg_items, const int64_t* excl_off, const int32_t* excl_items,
                          int32_t max_pos, const int32_t* xrows, const int32_t* xpred) {
  EvalRowArgs a = {};
  a.user_tab = user_shard; a.U = g.total_users; a.uid = uid; a.Bu = Bu; a.item_tab = item_shard; a.bias = bias_shard;
  a.I = g.local_items; a.I_all = g.total_items; a.world = g.world; a.rank = g.rank; a.D = dim; a.pos_off = pos_off;
  a.excl_off = excl_off; a.pos_items = pos_items; a.excl_items = excl_items; a.max_pos = max_pos; a.P = max_pos + 1;
  a.xrows = phase >= 1 ? reinterpret_cast<const float*>(xrows) : nullptr;
  a.xpred = phase == 2 ? reinterpret_cast<const float*>(xpred) : nullptr;
  a.neg_off = neg_off; a.neg_items = neg_items;
  return a;
}

// orx_score_rank, orx_score_rank_listed and orx_score_topk on tables of storage T (float, or bf16 bits): one body for
// both forms, so the bf16 entries refuse, size and dispatch exactly as the fp32 ones.
template <typename T>
int score_rank_impl(orx_handle_t h, int32_t kind, const T* user_tab, int64_t U, const int32_t* uid, int32_t Bu,
                    const float* scale, const T* item_tab, const float* item_bias, int64_t I, int32_t dim,
                    const int64_t* pos_off, const int32_t* pos_items, const int64_t* excl_off, const int32_t* excl_items,
                    int32_t max_pos, const int32_t* at_host, int32_t n_at, float* auc, float* ndcg, float* recall,
                    orx_stream_t s) {
  const char* why = ev_rank_refusal(h, kind, user_tab, U, uid, Bu, item_tab, I, dim, pos_off, max_pos, at_host, n_at);
  ORX_REQUIRE(why == nullptr, why);
  if (Bu == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;

  EvalWs w;
  const int rc = ev_workspace(h, Bu, max_pos + 1, st, &w);
  if (rc != ORX_OK) return rc;

  const EvalRowArgsT<T> a = ev_rank_args(user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, pos_off, pos_items,
                                         nullptr, nullptr, excl_off, excl_items, max_pos);
  const EvalOut o = ev_out(at_host, n_at, auc, ndcg, recall);
  return kind == ORX_SCORE_DOT ? ev_launch<ORX_SCORE_DOT>(h, a, w, o, st)
                               : ev_launch<ORX_SCORE_NEG_SQDIST>(h, a, w, o, st);
}

template <typename T>
int score_rank_listed_impl(orx_handle_t h, int32_t kind, const T* user_tab, int64_t U, const int32_t* uid, int32_t Bu,
                           const float* scale, const T* item_tab, const float* item_bias, int64_t I, int32_t dim,
                           const int64_t* pos_off, const int32_t* pos_items, const int64_t* neg_off,
                           const int32_t* neg_items, const int64_t* excl_off, const int32_t* excl_items,
                           int32_t max_pos, const int32_t* at_host, int32_t n_at, float* auc, float* ndcg,
                           float* recall, orx_stream_t s) {
  const char* why = ev_rank_refusal(h, kind, user_tab, U, uid, Bu, item_tab, I, dim, pos_off, max_pos, at_host, n_at);
  ORX_REQUIRE(why == nullptr, why);
  ORX_REQUIRE(neg_off != nullptr, "null pointer");
  if (Bu == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  const EvalRowArgsT<T> a = ev_rank_args(user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, pos_off, pos_items,
                                         neg_off, neg_items, excl_off, excl_items, max_pos);
  const EvalOut o = ev_out(at_host, n_at, auc, ndcg, recall);
  cudaStream_t st = (cudaStream_t)s;
  return kind == ORX_SCORE_DOT ? el_launch<ORX_SCORE_DOT>(h, a, o, nullptr, st)
                               : el_launch<ORX_SCORE_NEG_SQDIST>(h, a, o, nullptr, st);
}

template <typename T>
int score_topk_impl(orx_handle_t h, int32_t kind, const T* user_tab, int64_t U, const int32_t* uid, int32_t Bu,
                    const float* scale, const T* item_tab, const float* item_bias, int64_t I, int32_t dim,
                    const int64_t* excl_off, const int32_t* excl_items, int32_t k, int32_t* top_items,
                    float* top_scores, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(kind == ORX_SCORE_DOT || kind == ORX_SCORE_NEG_SQDIST, "unknown score kind");
  ORX_REQUIRE(U > 0 && I > 0 && I <= INT32_MAX && dim > 0 && Bu >= 0, "bad sizes");
  ORX_REQUIRE(k >= 1 && k <= ORX_MAX_TOPK, "k must lie in [1, ORX_MAX_TOPK]");
  if (Bu == 0) return ORX_OK;   // before the pointer checks: an empty batch may come with NULL buffers
  ORX_REQUIRE(user_tab && uid && item_tab && top_items, "null pointer");
  ORX_CUDA(cudaSetDevice(h->device));
  EvalArgsT<T> a = {};
  a.user_tab = user_tab; a.U = U; a.uid = uid; a.Bu = Bu; a.scale = scale; a.item_tab = item_tab;
  a.bias = item_bias; a.I = I; a.D = dim; a.excl_off = excl_off; a.excl_items = excl_items;
  return kind == ORX_SCORE_DOT ? tk_launch<ORX_SCORE_DOT>(h, a, k, top_items, top_scores, (cudaStream_t)s)
                               : tk_launch<ORX_SCORE_NEG_SQDIST>(h, a, k, top_items, top_scores, (cudaStream_t)s);
}

}  // namespace

extern "C" int orx_score_rank(orx_handle_t h, int32_t kind, const float* user_tab, int64_t U, const int32_t* uid,
                              int32_t Bu, const float* scale, const float* item_tab, const float* item_bias, int64_t I,
                              int32_t dim, const int64_t* pos_off, const int32_t* pos_items, const int64_t* excl_off,
                              const int32_t* excl_items, int32_t max_pos, const int32_t* at_host, int32_t n_at,
                              float* auc, float* ndcg, float* recall, orx_stream_t s) {
  return score_rank_impl(h, kind, user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, pos_off, pos_items,
                         excl_off, excl_items, max_pos, at_host, n_at, auc, ndcg, recall, s);
}

extern "C" int orx_score_rank_bf16(orx_handle_t h, int32_t kind, const uint16_t* user_tab, int64_t U,
                                   const int32_t* uid, int32_t Bu, const float* scale, const uint16_t* item_tab,
                                   const float* item_bias, int64_t I, int32_t dim, const int64_t* pos_off,
                                   const int32_t* pos_items, const int64_t* excl_off, const int32_t* excl_items,
                                   int32_t max_pos, const int32_t* at_host, int32_t n_at, float* auc, float* ndcg,
                                   float* recall, orx_stream_t s) {
  return score_rank_impl(h, kind, user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, pos_off, pos_items,
                         excl_off, excl_items, max_pos, at_host, n_at, auc, ndcg, recall, s);
}

extern "C" int orx_score_rank_listed(orx_handle_t h, int32_t kind, const float* user_tab, int64_t U,
                                     const int32_t* uid, int32_t Bu, const float* scale, const float* item_tab,
                                     const float* item_bias, int64_t I, int32_t dim, const int64_t* pos_off,
                                     const int32_t* pos_items, const int64_t* neg_off, const int32_t* neg_items,
                                     const int64_t* excl_off, const int32_t* excl_items, int32_t max_pos,
                                     const int32_t* at_host, int32_t n_at, float* auc, float* ndcg, float* recall,
                                     orx_stream_t s) {
  return score_rank_listed_impl(h, kind, user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, pos_off, pos_items,
                                neg_off, neg_items, excl_off, excl_items, max_pos, at_host, n_at, auc, ndcg, recall, s);
}

extern "C" int orx_score_rank_listed_bf16(orx_handle_t h, int32_t kind, const uint16_t* user_tab, int64_t U,
                                          const int32_t* uid, int32_t Bu, const float* scale, const uint16_t* item_tab,
                                          const float* item_bias, int64_t I, int32_t dim, const int64_t* pos_off,
                                          const int32_t* pos_items, const int64_t* neg_off, const int32_t* neg_items,
                                          const int64_t* excl_off, const int32_t* excl_items, int32_t max_pos,
                                          const int32_t* at_host, int32_t n_at, float* auc, float* ndcg,
                                          float* recall, orx_stream_t s) {
  return score_rank_listed_impl(h, kind, user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, pos_off, pos_items,
                                neg_off, neg_items, excl_off, excl_items, max_pos, at_host, n_at, auc, ndcg, recall, s);
}

extern "C" int orx_score_topk(orx_handle_t h, int32_t kind, const float* user_tab, int64_t U, const int32_t* uid,
                              int32_t Bu, const float* scale, const float* item_tab, const float* item_bias, int64_t I,
                              int32_t dim, const int64_t* excl_off, const int32_t* excl_items, int32_t k,
                              int32_t* top_items, float* top_scores, orx_stream_t s) {
  return score_topk_impl(h, kind, user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, excl_off, excl_items, k,
                         top_items, top_scores, s);
}

extern "C" int orx_score_topk_bf16(orx_handle_t h, int32_t kind, const uint16_t* user_tab, int64_t U,
                                   const int32_t* uid, int32_t Bu, const float* scale, const uint16_t* item_tab,
                                   const float* item_bias, int64_t I, int32_t dim, const int64_t* excl_off,
                                   const int32_t* excl_items, int32_t k, int32_t* top_items, float* top_scores,
                                   orx_stream_t s) {
  return score_topk_impl(h, kind, user_tab, U, uid, Bu, scale, item_tab, item_bias, I, dim, excl_off, excl_items, k,
                         top_items, top_scores, s);
}

extern "C" int orx_score_rank_shard_sizes(int32_t Bu, int32_t dim, int32_t max_pos, int64_t* n3_host) {
  ORX_REQUIRE(n3_host != nullptr, "null pointer");
  ORX_REQUIRE(Bu >= 0 && dim > 0 && max_pos >= 0, "bad sizes");
  const int64_t P = (int64_t)max_pos + 1;
  ORX_REQUIRE(2 * (int64_t)Bu * P <= INT32_MAX, "Bu * (max_pos + 1) too large for one call: split the batch");
  n3_host[0] = (int64_t)Bu * dim;
  n3_host[1] = n3_host[2] = (int64_t)Bu * P;
  return ORX_OK;
}

extern "C" int orx_score_rank_shard(orx_handle_t h, int32_t kind, int32_t phase, const orx_rowshard_t* g_host,
                                    const float* user_shard, const float* item_shard, const float* bias_shard,
                                    int32_t dim, const int32_t* uid, int32_t Bu, const int64_t* pos_off,
                                    const int32_t* pos_items, const int64_t* excl_off, const int32_t* excl_items,
                                    int32_t max_pos, const int32_t* at_host, int32_t n_at, int32_t* xrows,
                                    int32_t* xpred, int64_t* xcnt, float* auc, float* ndcg, float* recall,
                                    orx_stream_t s) {
  const char* why = ev_shard_refusal(h, kind, phase, g_host, user_shard, item_shard, dim, uid, Bu, pos_off, max_pos,
                                     at_host, n_at, xrows, xpred, xcnt);
  ORX_REQUIRE(why == nullptr, why);
  if (Bu == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  const EvalRowArgs a = ev_shard_args(phase, *g_host, user_shard, item_shard, bias_shard, dim, uid, Bu, pos_off,
                                      pos_items, nullptr, nullptr, excl_off, excl_items, max_pos, xrows, xpred);
  const EvalOut o = ev_out(at_host, n_at, auc, ndcg, recall);
  cudaStream_t st = (cudaStream_t)s;
  return kind == ORX_SCORE_DOT ? ev_shard_phase<ORX_SCORE_DOT>(h, phase, false, a, o, xrows, xpred, xcnt, st)
                               : ev_shard_phase<ORX_SCORE_NEG_SQDIST>(h, phase, false, a, o, xrows, xpred, xcnt, st);
}

extern "C" int orx_score_rank_listed_shard(orx_handle_t h, int32_t kind, int32_t phase, const orx_rowshard_t* g_host,
                                           const float* user_shard, const float* item_shard, const float* bias_shard,
                                           int32_t dim, const int32_t* uid, int32_t Bu, const int64_t* pos_off,
                                           const int32_t* pos_items, const int64_t* neg_off, const int32_t* neg_items,
                                           const int64_t* excl_off, const int32_t* excl_items, int32_t max_pos,
                                           const int32_t* at_host, int32_t n_at, int32_t* xrows, int32_t* xpred,
                                           int64_t* xcnt, float* auc, float* ndcg, float* recall, orx_stream_t s) {
  const char* why = ev_shard_refusal(h, kind, phase, g_host, user_shard, item_shard, dim, uid, Bu, pos_off, max_pos,
                                     at_host, n_at, xrows, xpred, xcnt);
  ORX_REQUIRE(why == nullptr, why);
  if (Bu == 0) return ORX_OK;
  ORX_REQUIRE(neg_off != nullptr, "null pointer");
  ORX_CUDA(cudaSetDevice(h->device));
  const EvalRowArgs a = ev_shard_args(phase, *g_host, user_shard, item_shard, bias_shard, dim, uid, Bu, pos_off,
                                      pos_items, neg_off, neg_items, excl_off, excl_items, max_pos, xrows, xpred);
  const EvalOut o = ev_out(at_host, n_at, auc, ndcg, recall);
  cudaStream_t st = (cudaStream_t)s;
  return kind == ORX_SCORE_DOT ? ev_shard_phase<ORX_SCORE_DOT>(h, phase, true, a, o, xrows, xpred, xcnt, st)
                               : ev_shard_phase<ORX_SCORE_NEG_SQDIST>(h, phase, true, a, o, xrows, xpred, xcnt, st);
}

extern "C" int orx_score_topk_shard(orx_handle_t h, int32_t kind, int32_t phase, const orx_rowshard_t* g_host,
                                    const float* user_shard, const float* item_shard, const float* bias_shard,
                                    int32_t dim, const int32_t* uid, int32_t Bu, const int64_t* excl_off,
                                    const int32_t* excl_items, int32_t k, int32_t* xrows, int64_t* xkeys,
                                    int32_t* top_items, float* top_scores, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && g_host != nullptr, "null pointer");
  ORX_REQUIRE(kind == ORX_SCORE_DOT || kind == ORX_SCORE_NEG_SQDIST, "unknown score kind");
  ORX_REQUIRE(phase >= 0 && phase <= 2, "phase must lie in [0, 2]");
  const orx_rowshard_t g = *g_host;
  ORX_REQUIRE(g.world >= 1 && g.rank >= 0 && g.rank < g.world, "rank must lie in [0, world)");
  ORX_REQUIRE(g.total_users > 0 && g.total_items > 0 && g.total_items <= INT32_MAX, "bad table sizes");
  ORX_REQUIRE(g.local_users == (g.total_users - g.rank + g.world - 1) / g.world &&
                  g.local_items == (g.total_items - g.rank + g.world - 1) / g.world,
              "local_users / local_items disagree with (total, world, rank)");
  ORX_REQUIRE(dim > 0 && Bu >= 0, "bad sizes");
  ORX_REQUIRE(k >= 1 && k <= ORX_MAX_TOPK, "k must lie in [1, ORX_MAX_TOPK]");
  if (Bu == 0) return ORX_OK;
  ORX_REQUIRE((int64_t)Bu * g.world * k <= INT32_MAX, "Bu * world * k too large for one call: split the batch");
  ORX_REQUIRE(uid != nullptr, "null pointer");
  ORX_REQUIRE(phase != 0 || (user_shard && xrows), "phase 0 needs user_shard and xrows");
  ORX_REQUIRE(phase != 1 || (item_shard && xrows && xkeys), "phase 1 needs item_shard, xrows and xkeys");
  ORX_REQUIRE(phase != 2 || (xkeys && top_items), "phase 2 needs xkeys and top_items");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(xkeys);
  if (phase == 0) {
    EvalRowArgs a = {};
    a.user_tab = user_shard; a.U = g.total_users; a.uid = uid; a.Bu = Bu; a.D = dim; a.world = g.world;
    a.rank = g.rank;
    ev_user_rows(a, xrows, st);
  } else if (phase == 1) {
    EvalArgs a = {};
    a.user_tab = reinterpret_cast<const float*>(xrows); a.U = g.total_users; a.uid = uid; a.Bu = Bu;
    a.item_tab = item_shard; a.bias = bias_shard; a.I = g.local_items; a.D = dim; a.excl_off = excl_off;
    a.excl_items = excl_items;
    return kind == ORX_SCORE_DOT
               ? tk_shard_local<ORX_SCORE_DOT>(h, a, k, g.world, g.rank, g.total_items, keys, st)
               : tk_shard_local<ORX_SCORE_NEG_SQDIST>(h, a, k, g.world, g.rank, g.total_items, keys, st);
  } else {
    k_topk_merge_ranks<<<Bu, EV_NT, 0, st>>>(keys, g.world, k, top_items, top_scores);
  }
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}
