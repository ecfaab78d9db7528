// orx_pair.cuh -- argument block and per-sample math shared by the pairwise (BPR / UCML) kernels.
#pragma once
#include "orx_common.cuh"

struct PairArgs : SparseArgs {
  int64_t rowsU, rowsI;
  const int32_t *uid, *pid, *nid;
  int B;
  float margin, c_loss, c_l2, inv_B;
  float* partials;
  // k_pair_step of a prefetched batch: record t = {flags, du, dp, dn} of triplet t (k_index_resolve), read in place of the
  // id bounds check and the three index probes.  Null: probe the index.
  const int4* res;
  // un-fused outputs (k_pair_generic MODE 1).  ld = 0: table form, outputs indexed by triplet.  ld > D: row form
  // (orx_pairwise_grad_rows) -- U = I = fetched rows of stride ld with the item bias in column D, outputs written to the
  // lookup's own row of d_user = d_pos = d_neg.
  float *d_user, *d_pos, *d_neg, *d_bp, *d_bn, *g_out;
  int64_t ld;
};

__device__ __forceinline__ float dot4(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
__device__ __forceinline__ float sqd4(float4 a, float4 b) {
  float x = a.x - b.x, y = a.y - b.y, z = a.z - b.z, w = a.w - b.w;
  return x * x + y * y + z * z + w * w;
}
// r = s*(a-b) + c*d
__device__ __forceinline__ float4 axmb_pcd(float s, float4 a, float4 b, float c, float4 d) {
  return make_float4(s * (a.x - b.x) + c * d.x, s * (a.y - b.y) + c * d.y, s * (a.z - b.z) + c * d.z,
                     s * (a.w - b.w) + c * d.w);
}
// r = s*a + c*d
__device__ __forceinline__ float4 sa_pcd(float s, float4 a, float c, float4 d) {
  return make_float4(s * a.x + c * d.x, s * a.y + c * d.y, s * a.z + c * d.z, s * a.w + c * d.w);
}

// Per-sample score -> (loss term, gradient scalars).  BPR: x = (u.p+bp)-(u.n+bn),
// loss term = -log sigmoid(max(x,-30)), g = -(c_loss/B) sigmoid(-y) [x>=-30]  (pairwise_log_loss.py:19-32).
// UCML: h = margin - ((-|u-p|^2+bp) - (-|u-n|^2+bn)), loss term = max(h,0), a = c_loss [h>=0] (ucml.py:29-39).
template <int KIND>
__device__ __forceinline__ void pair_score(float s1, float s2, float bp, float bn, float margin, float c_loss,
                                           float inv_B, float* loss_term, float* g) {
  if (KIND == ORX_PAIR_BPR) {
    const float x = (s1 + bp) - (s2 + bn);
    const float y = fmaxf(x, -30.f);
    float ls, sn;
    orx_logsig(y, &ls, &sn);
    *loss_term = -ls;
    *g = (x >= -30.f) ? -(c_loss * inv_B) * sn : 0.f;
  } else {
    const float h = margin - (((-s1) + bp) - ((-s2) + bn));
    *loss_term = fmaxf(h, 0.f);
    *g = (h >= 0.f) ? c_loss : 0.f;
  }
}

// Row gradients from the scalar (SURVEY 8a-G).
template <int KIND>
__device__ __forceinline__ void pair_row_grads(float g, float c2, float4 u, float4 p, float4 n, float4* gu,
                                               float4* gp, float4* gn) {
  if (KIND == ORX_PAIR_BPR) {
    *gu = axmb_pcd(g, p, n, c2, u);
    *gp = sa_pcd(g, u, c2, p);
    *gn = sa_pcd(-g, u, c2, n);
  } else {
    const float t = 2.f * g;
    *gu = axmb_pcd(t, n, p, c2, u);
    *gp = axmb_pcd(t, p, u, c2, p);
    *gn = axmb_pcd(t, u, n, c2, n);
  }
}

// The same for one element of the rows.
template <int KIND>
__device__ __forceinline__ void pair_grads1(float g, float c2, float u, float p, float n, float* gu, float* gp,
                                            float* gn) {
  if (KIND == ORX_PAIR_BPR) {
    *gu = g * (p - n) + c2 * u;
    *gp = g * u + c2 * p;
    *gn = -g * u + c2 * n;
  } else {
    const float t = 2.f * g;
    *gu = t * (n - p) + c2 * u;
    *gp = t * (p - u) + c2 * p;
    *gn = t * (u - n) + c2 * n;
  }
}

