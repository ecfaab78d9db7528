// orx_dlrm.cu -- DLRM building blocks (rows a11-a13): strided per-feature gather (K5), second-order
// interaction fwd/bwd (K6), Dense layers fwd/bwd (K7, fp32 SIMT tiles -- 1e-5 parity first; the wgmma
// 3xTF32 path of orx_mlp_tc.cu takes every shape that fills a tile), prediction loss.
//
// Reference path: openrec/tf2/recommenders/dlrm.py:63-100, modules/multi_layer_perceptron.py:5-18,
// modules/second_order_feature_interaction.py:12-34.
#include "orx_common.cuh"

// ---------------------------------------------------------------------------------------
// K5: out[b*out_ld + :D] = tab[ids[b*id_stride], :D]   (dlrm.py:83-85, one call per sparse feature)
// ---------------------------------------------------------------------------------------
// Row loads of the DLRM gathers by table storage: a float row as float4 / scalar (__ldg), a bf16 row (uint16_t bits) as
// 4 elements in one 8-byte load / one 2-byte load, widened exactly.
// gather_ld4(row, q): columns 4q .. 4q + 3 of a row (16-byte / 8-byte aligned)
__device__ __forceinline__ float4 gather_ld4(const float* row, int q) {
  return __ldg(reinterpret_cast<const float4*>(row) + q);
}
__device__ __forceinline__ float4 gather_ld4(const uint16_t* row, int q) {
  return orx_bf16x4_up(__ldg(reinterpret_cast<const uint2*>(row) + q));
}
__device__ __forceinline__ float gather_ld1(const float* p) { return __ldg(p); }
__device__ __forceinline__ float gather_ld1(const uint16_t* p) { return orx_bf16_up(__ldg(p)); }

// VEC: out is 16-byte aligned and tab 16-byte (float) / 8-byte (bf16) aligned (gather_strided_impl decides); with D and
// out_ld multiples of 4 the rows then move 4 columns per lane (the row shape is tested here, as in k_gather).
// T: the table's storage, float or bf16 bits (uint16_t); out is float either way.
template <bool VEC, typename T = float>
__global__ void __launch_bounds__(256) k_gather_strided(const T* __restrict__ tab, int64_t rows, int D,
                                                        const int32_t* __restrict__ ids, int64_t id_stride, int64_t n,
                                                        float* __restrict__ out, int64_t out_ld, int32_t* n_bad) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const bool vec = VEC && ((D & 3) == 0) && ((out_ld & 3) == 0);
  for (int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n; b += nw) {
    const int64_t id = ids[b * id_stride];
    const bool ok = id >= 0 && id < rows;
    if (!ok && lane == 0 && n_bad) atomicAdd(n_bad, 1);
    if (vec) {
      const T* src = tab + id * D;
      float4* dst = reinterpret_cast<float4*>(out + b * out_ld);
      for (int e = lane; e < D / 4; e += 32) dst[e] = ok ? gather_ld4(src, e) : make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      for (int e = lane; e < D; e += 32) out[b * out_ld + e] = ok ? gather_ld1(tab + id * D + e) : 0.f;
    }
  }
}

template <typename T>
static int gather_strided_impl(orx_handle_t h, const T* tab, int64_t rows, int32_t dim, const int32_t* ids,
                               int64_t id_stride, int64_t n, float* out, int64_t out_ld, int32_t* n_bad,
                               orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && tab && ids && out, "null pointer");
  ORX_REQUIRE(rows > 0 && dim > 0 && n >= 0 && id_stride >= 1 && out_ld >= dim, "bad sizes");
  if (n == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  int64_t blocks = (n + 7) / 8;
  if (blocks > (int64_t)h->num_sms * 32) blocks = (int64_t)h->num_sms * 32;
  cudaStream_t st = (cudaStream_t)s;
  const bool vec = std::is_same<T, float>::value ? orx_aligned16(tab, out) : orx_aligned8(tab) && orx_aligned16(out);
  if (vec)
    k_gather_strided<true, T><<<(int)blocks, 256, 0, st>>>(tab, rows, dim, ids, id_stride, n, out, out_ld, n_bad);
  else
    k_gather_strided<false, T><<<(int)blocks, 256, 0, st>>>(tab, rows, dim, ids, id_stride, n, out, out_ld, n_bad);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

extern "C" int orx_gather_strided(orx_handle_t h, const float* tab, int64_t rows, int32_t dim, const int32_t* ids,
                                  int64_t id_stride, int64_t n, float* out, int64_t out_ld, int32_t* n_bad,
                                  orx_stream_t s) {
  return gather_strided_impl(h, tab, rows, dim, ids, id_stride, n, out, out_ld, n_bad, s);
}

extern "C" int orx_gather_strided_bf16(orx_handle_t h, const uint16_t* tab, int64_t rows, int32_t dim,
                                       const int32_t* ids, int64_t id_stride, int64_t n, float* out, int64_t out_ld,
                                       int32_t* n_bad, orx_stream_t s) {
  return gather_strided_impl(h, tab, rows, dim, ids, id_stride, n, out, out_ld, n_bad, s);
}

// ---------------------------------------------------------------------------------------
// K6: second-order interaction.  Features: F-1 embedding rows emb[b, f, :] (row stride emb_ld per
// feature, F-1 of them contiguous per sample) + the dense vector dense[b*dense_ld + :] as LAST feature
// (dlrm.py:89-92: sparse_emb_vecs + [dense_emb_vec]).
//   mode 0 (reference, bug-compatible, SURVEY Q1): out = row-major entries (i,j>=i [j>i if !self]) of
//           lower_tri(Z Z^T)  => only the diagonal survives;
//   mode 1 (dlrm): row-major entries (i, j<i [j<=i if self]) of Z Z^T.
// ---------------------------------------------------------------------------------------
#define ORX_MAX_F 64

__device__ __forceinline__ bool inter_selected(int mode, int self, int i, int j) {
  return mode == 0 ? (self ? j >= i : j > i) : (self ? j <= i : j < i);
}

// position of the selected entry (i,j) in the row-major enumeration of the selected entries
__device__ __forceinline__ int inter_index(int mode, int self, int F, int i, int j) {
  if (mode == 0) return self ? i * F - i * (i - 1) / 2 + (j - i) : i * (F - 1) - i * (i - 1) / 2 + (j - i - 1);
  return self ? i * (i + 1) / 2 + j : i * (i - 1) / 2 + j;
}

// sample b's features -> shared memory, [F][D+1] (the +1 keeps same-column reads of different rows conflict-free)
__device__ __forceinline__ void inter_load(const float* __restrict__ emb, int64_t emb_ld, const float* __restrict__ dense,
                                           int64_t dense_ld, int b, int F, int D, float* sz) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5, Dp = D + 1;
  for (int f = warp; f < F; f += nw) {
    const float* src = f < F - 1 ? emb + (int64_t)b * emb_ld + (int64_t)f * D : dense + (int64_t)b * dense_ld;
    for (int d = lane; d < D; d += 32) sz[f * Dp + d] = src[d];
  }
}

// One CTA per sample.  The F x F cells are dealt to the threads; a selected cell is one D-long dot product out of
// shared memory (first version: every thread walked all F*F cells with a runtime modulo per cell -- 10.4 ms at
// B = 32768, F = 27, D = 128, profiles/r1v_dlrm_launches.csv).
__global__ void __launch_bounds__(128) k_interact_fwd(const float* __restrict__ emb, int64_t emb_ld,
                                                      const float* __restrict__ dense, int64_t dense_ld, int B, int F,
                                                      int D, int self, int mode, float* __restrict__ out,
                                                      int64_t out_ld) {
  extern __shared__ float sz[];  // [F][D+1]
  const int b = blockIdx.x;
  if (b >= B) return;
  const int Dp = D + 1;
  inter_load(emb, emb_ld, dense, dense_ld, b, F, D, sz);
  __syncthreads();
  for (int c = threadIdx.x; c < F * F; c += blockDim.x) {
    const int i = c / F, j = c - i * F;
    if (!inter_selected(mode, self, i, j)) continue;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    if (mode == 1 || j == i) {  // mode 0: lower_tri(P)[i,j] with j>=i is non-zero only on the diagonal
      const float* zi = sz + i * Dp;
      const float* zj = sz + j * Dp;
      int d = 0;
      for (; d + 3 < D; d += 4) {
        a0 += zi[d] * zj[d];
        a1 += zi[d + 1] * zj[d + 1];
        a2 += zi[d + 2] * zj[d + 2];
        a3 += zi[d + 3] * zj[d + 3];
      }
      for (; d < D; ++d) a0 += zi[d] * zj[d];
    }
    out[(int64_t)b * out_ld + inter_index(mode, self, F, i, j)] = (a0 + a1) + (a2 + a3);
  }
}

// dZ = (dP + dP^T) Z restricted to the selected entries; emb part -> demb[b,f,:], dense part ADDED to ddense.
__global__ void __launch_bounds__(128) k_interact_bwd(const float* __restrict__ emb, int64_t emb_ld,
                                                      const float* __restrict__ dense, int64_t dense_ld,
                                                      const float* __restrict__ dout, int64_t dout_ld, int B, int F,
                                                      int D, int self, int mode, float* __restrict__ demb,
                                                      int64_t demb_ld, float* __restrict__ ddense,
                                                      int64_t ddense_ld) {
  extern __shared__ float sm[];  // Z [F][D+1] then dP [F][F]
  const int b = blockIdx.x;
  if (b >= B) return;
  const int Dp = D + 1;
  float* sz = sm;
  float* sp = sm + F * Dp;
  inter_load(emb, emb_ld, dense, dense_ld, b, F, D, sz);
  for (int c = threadIdx.x; c < F * F; c += blockDim.x) {
    const int i = c / F, j = c - i * F;
    float v = 0.f;
    if (inter_selected(mode, self, i, j) && (mode == 1 || j == i))
      v = dout[(int64_t)b * dout_ld + inter_index(mode, self, F, i, j)];
    sp[c] = v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int i = warp; i < F; i += nw) {
    for (int d = lane; d < D; d += 32) {
      float acc = 0.f;
      for (int j = 0; j < F; ++j) acc += (sp[i * F + j] + sp[j * F + i]) * sz[j * Dp + d];
      if (i < F - 1) demb[(int64_t)b * demb_ld + (int64_t)i * D + d] = acc;
      else ddense[(int64_t)b * ddense_ld + d] += acc;
    }
  }
}

// ---- fast path (mode 1, D % 4 == 0, D <= 128, F <= 32): ONE WARP per sample, grid-stride.
// The generic kernels above are shared-memory bound: every thread streams two D-long rows per cell (2 x 512 B of LDS per
// dot product at D = 128; 0.73 + 1.13 ms per step at B = 32768, F = 27, profiles/r1w).  Here a lane owns four columns:
//  fwd: row i stays in registers while j runs over its selected cells, so a cell costs ONE 128-bit shared load per lane +
//       4 FMAs; the 32 per-lane partials of 32 consecutive cells are summed by a transpose-reduce (31 shuffles per 32
//       cells), after which lane q holds cell q -> one coalesced 128-byte store per 32 outputs.
//  bwd: dZ_i = sum_j (dP + dP^T)[i][j] z_j.  The symmetric weights live in shared memory as W[j][i]; nine rows i are
//       accumulated at once, so a row z_j is loaded once per nine cells and its nine weights come as three broadcast
//       128-bit loads.
#define INTER_WARPS 4

__device__ __forceinline__ void inter_load_warp(const float* __restrict__ emb, int64_t emb_ld, const float* __restrict__ dense,
                                                int64_t dense_ld, int b, int F, int D, int lane, float4* sz /* [F][32] */) {
  const int nq = D >> 2;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int f = 0; f < F; ++f) {
    const float* src = f < F - 1 ? emb + (int64_t)b * emb_ld + (int64_t)f * D : dense + (int64_t)b * dense_ld;
    sz[f * 32 + lane] = lane < nq ? __ldg(reinterpret_cast<const float4*>(src) + lane) : z4;
  }
}

__global__ void __launch_bounds__(INTER_WARPS * 32) k_interact_fwd_warp(const float* __restrict__ emb, int64_t emb_ld,
                                                                        const float* __restrict__ dense, int64_t dense_ld,
                                                                        int B, int F, int D, int self,
                                                                        float* __restrict__ out, int64_t out_ld) {
  extern __shared__ float4 sz_all[];   // [INTER_WARPS][F][32]
  const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
  float4* sz = sz_all + (size_t)wi * F * 32;
  const int P = self ? F * (F + 1) / 2 : F * (F - 1) / 2;
  for (int b = blockIdx.x * INTER_WARPS + wi; b < B; b += gridDim.x * INTER_WARPS) {
    __syncwarp();
    inter_load_warp(emb, emb_ld, dense, dense_ld, b, F, D, lane, sz);
    __syncwarp();
    // cells in output order: row i = (self ? 0 : 1).., j = 0 .. i-1 (+ i if self)
    int i = self ? 0 : 1, j = 0;
    float4 zi = sz[i * 32 + lane];
    for (int p0 = 0; p0 < P; p0 += 32) {
      float v[32];
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        float part = 0.f;
        if (p0 + q < P) {                      // warp-uniform
          const float4 zj = sz[j * 32 + lane];
          part = zi.x * zj.x + zi.y * zj.y + zi.z * zj.z + zi.w * zj.w;
          ++j;
          if (j == i + (self ? 1 : 0)) {       // next row
            ++i;
            j = 0;
            if (i < F) zi = sz[i * 32 + lane];
          }
        }
        v[q] = part;
      }
      // transpose-reduce: after the five rounds lane q holds the sum over lanes of v[q]
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const bool up = lane & 16;
        const float send = up ? v[k] : v[k + 16], keep = up ? v[k + 16] : v[k];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const bool up = lane & 8;
        const float send = up ? v[k] : v[k + 8], keep = up ? v[k + 8] : v[k];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const bool up = lane & 4;
        const float send = up ? v[k] : v[k + 4], keep = up ? v[k + 4] : v[k];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
      }
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const bool up = lane & 2;
        const float send = up ? v[k] : v[k + 2], keep = up ? v[k + 2] : v[k];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
      }
      {
        const bool up = lane & 1;
        const float send = up ? v[0] : v[1], keep = up ? v[1] : v[0];
        v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
      }
      // lane l now holds cell index: bit4 of l selected the upper 16, bit3 the upper 8 of those, ... => cell l
      if (p0 + lane < P) out[(int64_t)b * out_ld + p0 + lane] = v[0];
    }
  }
}

__global__ void __launch_bounds__(INTER_WARPS * 32) k_interact_bwd_warp(const float* __restrict__ emb, int64_t emb_ld,
                                                                        const float* __restrict__ dense, int64_t dense_ld,
                                                                        const float* __restrict__ dout, int64_t dout_ld,
                                                                        int B, int F, int D, int self,
                                                                        float* __restrict__ demb, int64_t demb_ld,
                                                                        float* __restrict__ ddense, int64_t ddense_ld) {
  extern __shared__ float4 sb_all[];   // per warp: Z [F][32] float4, then W [F][36] floats (row j, columns i; 16-byte rows)
  constexpr int WLD = 36;              // >= 32 + padding so that nine-row blocks never read past a row
  const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
  const size_t per_warp = (size_t)F * 32 + (size_t)F * WLD / 4;
  float4* sz = sb_all + (size_t)wi * per_warp;
  float* sw = reinterpret_cast<float*>(sz + (size_t)F * 32);
  const int nq = D >> 2;
  for (int b = blockIdx.x * INTER_WARPS + wi; b < B; b += gridDim.x * INTER_WARPS) {
    __syncwarp();
    inter_load_warp(emb, emb_ld, dense, dense_ld, b, F, D, lane, sz);
    // W[j][i] = dP[i][j] + dP[j][i] over the selected cells (mode 1: j < i, or j <= i with self)
    for (int c = lane; c < F * WLD; c += 32) sw[c] = 0.f;
    __syncwarp();
    const int P = self ? F * (F + 1) / 2 : F * (F - 1) / 2;
    for (int p = lane; p < P; p += 32) {
      // invert p -> (i, j): rows hold i + self (self) or i (no self) cells
      int i = (int)((sqrtf(8.f * (float)p + 1.f) - 1.f) * 0.5f) + (self ? 0 : 1);
      while ((self ? i * (i + 1) / 2 : i * (i - 1) / 2) > p) --i;
      while ((self ? (i + 1) * (i + 2) / 2 : (i + 1) * i / 2) <= p) ++i;
      const int j = p - (self ? i * (i + 1) / 2 : i * (i - 1) / 2);
      const float g = dout[(int64_t)b * dout_ld + p];
      if (i == j) sw[j * WLD + i] = 2.f * g;
      else { sw[j * WLD + i] = g; sw[i * WLD + j] = g; }
    }
    __syncwarp();
    for (int i0 = 0; i0 < F; i0 += 9) {
      float4 acc[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int j = 0; j < F; ++j) {
        const float4 zj = sz[j * 32 + lane];
        const float* wr = sw + j * WLD + i0;   // nine weights W[j][i0 .. i0+8] (zero beyond F)
        float wv[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) wv[k] = wr[k];
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          acc[k].x += wv[k] * zj.x; acc[k].y += wv[k] * zj.y; acc[k].z += wv[k] * zj.z; acc[k].w += wv[k] * zj.w;
        }
      }
      if (lane < nq) {
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          const int i = i0 + k;
          if (i >= F) break;
          if (i < F - 1) {
            reinterpret_cast<float4*>(demb + (int64_t)b * demb_ld + (int64_t)i * D)[lane] = acc[k];
          } else {
            float4* dd = reinterpret_cast<float4*>(ddense + (int64_t)b * ddense_ld) + lane;
            float4 o = *dd;
            o.x += acc[k].x; o.y += acc[k].y; o.z += acc[k].z; o.w += acc[k].w;
            *dd = o;
          }
        }
      }
    }
  }
}

static bool inter_fast_ok(int F, int D, int mode, const void* a, const void* b, int64_t lda, int64_t ldb) {
  return mode == 1 && F >= 2 && F <= 32 && (D & 3) == 0 && D <= 128 && (lda & 3) == 0 && (ldb & 3) == 0 &&
         orx_aligned16(a, b);
}

extern "C" int orx_interact_fwd(orx_handle_t h, const float* emb, int64_t emb_ld, const float* dense,
                                int64_t dense_ld, int32_t B, int32_t F, int32_t D, int32_t self_interaction,
                                int32_t mode, float* out, int64_t out_ld, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && dense && out && (F == 1 || emb), "null pointer");
  ORX_REQUIRE(B >= 0 && F >= 1 && F <= ORX_MAX_F && D > 0 && (mode == 0 || mode == 1), "bad sizes/mode");
  if (B == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  if (inter_fast_ok(F, D, mode, emb ? (const void*)emb : (const void*)dense, dense, emb_ld, dense_ld)) {
    const size_t sm = sizeof(float4) * (size_t)INTER_WARPS * F * 32;
    ORX_CUDA(cudaFuncSetAttribute(k_interact_fwd_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    int grid = (B + INTER_WARPS - 1) / INTER_WARPS;
    if (grid > h->num_sms * 4) grid = h->num_sms * 4;
    k_interact_fwd_warp<<<grid, INTER_WARPS * 32, sm, (cudaStream_t)s>>>(emb, emb_ld, dense, dense_ld, B, F, D, self_interaction, out, out_ld);
    ORX_LAUNCH_CHECK();
    orx_log_dispatch(h, ORX_OP_INTERACT_FWD, ORX_VARIANT_INTERACT_WARP, 0, 0, B, F, D, 1);
    return ORX_OK;
  }
  const size_t smem = sizeof(float) * (size_t)F * (D + 1);
  ORX_REQUIRE(smem <= 200 * 1024, "F*D too large for the interaction kernel");
  if (smem > 48 * 1024) ORX_CUDA(cudaFuncSetAttribute(k_interact_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_interact_fwd<<<B, 128, smem, (cudaStream_t)s>>>(emb, emb_ld, dense, dense_ld, B, F, D, self_interaction, mode, out, out_ld);
  ORX_LAUNCH_CHECK();
  orx_log_dispatch(h, ORX_OP_INTERACT_FWD, ORX_VARIANT_INTERACT, 0, 0, B, F, D, 1);
  return ORX_OK;
}

extern "C" int orx_interact_bwd(orx_handle_t h, const float* emb, int64_t emb_ld, const float* dense,
                                int64_t dense_ld, const float* dout, int64_t dout_ld, int32_t B, int32_t F, int32_t D,
                                int32_t self_interaction, int32_t mode, float* demb, int64_t demb_ld, float* ddense,
                                int64_t ddense_ld, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && dense && dout && ddense && (F == 1 || (emb && demb)), "null pointer");
  ORX_REQUIRE(B >= 0 && F >= 1 && F <= ORX_MAX_F && D > 0 && (mode == 0 || mode == 1), "bad sizes/mode");
  if (B == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  if (inter_fast_ok(F, D, mode, emb ? (const void*)emb : (const void*)dense, dense, emb_ld, dense_ld) && (demb_ld & 3) == 0 &&
      (ddense_ld & 3) == 0 && orx_aligned16(demb ? (const void*)demb : (const void*)ddense, ddense)) {
    const size_t sm = (size_t)INTER_WARPS * (sizeof(float4) * (size_t)F * 32 + sizeof(float) * (size_t)F * 36);
    ORX_CUDA(cudaFuncSetAttribute(k_interact_bwd_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    int grid = (B + INTER_WARPS - 1) / INTER_WARPS;
    if (grid > h->num_sms * 3) grid = h->num_sms * 3;
    k_interact_bwd_warp<<<grid, INTER_WARPS * 32, sm, (cudaStream_t)s>>>(emb, emb_ld, dense, dense_ld, dout, dout_ld, B, F, D, self_interaction, demb, demb_ld, ddense, ddense_ld);
    ORX_LAUNCH_CHECK();
    orx_log_dispatch(h, ORX_OP_INTERACT_BWD, ORX_VARIANT_INTERACT_WARP, 0, 0, B, F, D, 1);
    return ORX_OK;
  }
  const size_t smem = sizeof(float) * ((size_t)F * (D + 1) + (size_t)F * F);
  ORX_REQUIRE(smem <= 200 * 1024, "F*D too large for the interaction kernel");
  if (smem > 48 * 1024) ORX_CUDA(cudaFuncSetAttribute(k_interact_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_interact_bwd<<<B, 128, smem, (cudaStream_t)s>>>(emb, emb_ld, dense, dense_ld, dout, dout_ld, B, F, D, self_interaction, mode, demb, demb_ld, ddense, ddense_ld);
  ORX_LAUNCH_CHECK();
  orx_log_dispatch(h, ORX_OP_INTERACT_BWD, ORX_VARIANT_INTERACT, 0, 0, B, F, D, 1);
  return ORX_OK;
}

// ---------------------------------------------------------------------------------------
// K7: Dense layers.  One fp32 SIMT GEMM  C[M,N] (+)= op(A)[M,K] * op(B)[K,N]  with 64x64x16 tiles and
// a 4x4 register block per thread; TA/TB select how the tile is read:
//   TA=0: A[m*lda + k]   TA=1: A[k*lda + m]      TB=0: B[k*ldb + n]   TB=1: B[n*ldb + k]
// Epilogue: + bias[n], activation (0 none, 1 relu, 2 sigmoid).
// ---------------------------------------------------------------------------------------
template <int TA, int TB>
__global__ void __launch_bounds__(256) k_gemm(const float* __restrict__ A, int64_t lda, const float* __restrict__ Bm,
                                              int64_t ldb, float* __restrict__ C, int64_t ldc, int M, int N, int K,
                                              const float* __restrict__ bias, int act, float* __restrict__ part) {
  constexpr int T = 64, KC = 16;
  __shared__ float sa[KC][T + 4], sb[KC][T + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * T, n0 = blockIdx.x * T;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  // split-K: blockIdx.z takes a KC-aligned slice of K and writes a raw partial tile (summed by k_splitk_reduce)
  const int kper = ((K + (int)gridDim.z - 1) / (int)gridDim.z + KC - 1) / KC * KC;
  const int k_lo = blockIdx.z * kper, k_hi = min(K, k_lo + kper);
  for (int k0 = k_lo; k0 < k_hi; k0 += KC) {
    for (int e = threadIdx.x; e < T * KC; e += 256) {
      int r, k;
      if (TA == 0) { r = e / KC; k = e % KC; } else { k = e / T; r = e % T; }   // keep the global read contiguous
      float v = 0.f;
      if (m0 + r < M && k0 + k < k_hi) v = TA == 0 ? A[(int64_t)(m0 + r) * lda + k0 + k] : A[(int64_t)(k0 + k) * lda + m0 + r];
      sa[k][r] = v;
    }
    for (int e = threadIdx.x; e < T * KC; e += 256) {
      int c, k;
      if (TB == 0) { k = e / T; c = e % T; } else { c = e / KC; k = e % KC; }
      float v = 0.f;
      if (n0 + c < N && k0 + k < k_hi) v = TB == 0 ? Bm[(int64_t)(k0 + k) * ldb + n0 + c] : Bm[(int64_t)(n0 + c) * ldb + k0 + k];
      sb[k][c] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = sa[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = sb[k][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += a[i] * b[j];
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx + 16 * j;
      if (n >= N) continue;
      if (gridDim.z > 1) {
        part[(size_t)blockIdx.z * (size_t)M * (size_t)N + (size_t)m * N + n] = acc[i][j];
        continue;
      }
      float v = acc[i][j] + (bias ? bias[n] : 0.f);
      if (act == 1) v = fmaxf(v, 0.f);
      else if (act == 2) v = orx_sigmoid(v);
      C[(int64_t)m * ldc + n] = v;
    }
  }
}

int orx_launch_gemm_tc(orx_ctx* h, int TA, int TB, const float* A, int64_t lda, const float* Bm, int64_t ldb, float* C,
                       int64_t ldc, int M, int N, int K, const float* bias, int act, cudaStream_t st);   // orx_mlp_tc.cu
int orx_launch_splitk_reduce(const float* part, int S, int M, int N, float* C, int64_t ldc, const float* bias, int act,
                             cudaStream_t st);

template <int TA, int TB>
static int launch_gemm(orx_ctx* h, const float* A, int64_t lda, const float* Bm, int64_t ldb, float* C, int64_t ldc, int M,
                       int N, int K, const float* bias, int act, cudaStream_t st) {
  // tensor cores (wgmma, 3xTF32) whenever the shape fills a tile reasonably and the TMA can describe the operands
  const int rc = orx_launch_gemm_tc(h, TA, TB, A, lda, Bm, ldb, C, ldc, M, N, K, bias, act, st);
  if (rc != ORX_ERR_UNSUPPORTED) return rc;
  const int tiles = ((N + 63) / 64) * ((M + 63) / 64);
  int S = 1;
  const int sms = h->num_sms;
  if (tiles < sms && K >= 1024) {   // dw of a narrow layer (13 x 512, 256 x 1): K = batch, a handful of tiles
    S = (2 * sms + tiles - 1) / tiles;
    if (S > K / 256) S = K / 256;
    if (S > 65535) S = 65535;
  }
  float* part = nullptr;
  if (S > 1) {
    const int rc2 = orx_grow((void**)&h->splitk, &h->splitk_cap, sizeof(float) * (size_t)S * (size_t)M * (size_t)N);
    if (rc2) return rc2;
    part = h->splitk;
  }
  dim3 grid((N + 63) / 64, (M + 63) / 64, S);
  k_gemm<TA, TB><<<grid, 256, 0, st>>>(A, lda, Bm, ldb, C, ldc, M, N, K, bias, act, part);
  ORX_LAUNCH_CHECK();
  orx_log_dispatch(h, ORX_OP_GEMM, ORX_VARIANT_GEMM_SIMT, TA, TB, M, N, K, S);
  if (S > 1) return orx_launch_splitk_reduce(part, S, M, N, C, ldc, bias, act, st);
  return ORX_OK;
}

// y[B,out] = act(x[B,in] @ w[in,out] + bias)     (multi_layer_perceptron.py:9-16; Keras kernel is [in,out])
extern "C" int orx_mlp_layer_fwd(orx_handle_t h, const float* x, int64_t ldx, int32_t B, int32_t in, const float* w,
                                 const float* bias, int32_t out, int32_t act, float* y, int64_t ldy, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && x && w && y, "null pointer");
  ORX_REQUIRE(B >= 0 && in > 0 && out > 0 && ldx >= in && ldy >= out && act >= 0 && act <= 2, "bad sizes");
  if (B == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  return launch_gemm<0, 0>(h, x, ldx, w, out, y, ldy, B, out, in, bias, act, (cudaStream_t)s);
}

// dz = dy * act'(y) in place; db[n] = sum_b dz[b,n]
__global__ void k_act_bwd(const float* __restrict__ y, int64_t ldy, float* __restrict__ dy, int64_t lddy, int B,
                          int N, int act) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * N) return;
  const int b = (int)(i / N), n = (int)(i % N);
  const float yv = y[(int64_t)b * ldy + n];
  float g = dy[(int64_t)b * lddy + n];
  if (act == 1) g = yv > 0.f ? g : 0.f;
  else if (act == 2) g = g * yv * (1.f - yv);
  dy[(int64_t)b * lddy + n] = g;
}

__global__ void __launch_bounds__(256) k_col_sum(const float* __restrict__ dz, int64_t ld, int B, int N,
                                                 float* __restrict__ out) {
  // block (32 cols x 8 row-lanes) over the row slice blockIdx.y; deterministic: fixed row partition, smem tree;
  // out = db when gridDim.y == 1, else the partial [gridDim.y][N] summed by k_splitk_reduce
  __shared__ float sh[8][33];
  const int n = blockIdx.x * 32 + (threadIdx.x & 31), r = threadIdx.x >> 5;
  const int per = (B + (int)gridDim.y - 1) / (int)gridDim.y;
  const int b_lo = blockIdx.y * per, b_hi = min(B, b_lo + per);
  float acc = 0.f;
  if (n < N)
    for (int b = b_lo + r; b < b_hi; b += 8) acc += dz[(int64_t)b * ld + n];
  sh[r][threadIdx.x & 31] = acc;
  __syncthreads();
  if (r == 0 && n < N) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += sh[k][threadIdx.x & 31];
    out[(size_t)blockIdx.y * N + n] = t;
  }
}

// Backward of one Dense layer.  dy (dL/dy, [B,out], ld lddy) is overwritten with dL/dz.
// dw[in,out] = x^T dz ; db[out] = colsum(dz) ; dx[B,in] = dz w^T (skipped when dx == NULL).
extern "C" int orx_mlp_layer_bwd(orx_handle_t h, const float* x, int64_t ldx, const float* y, int64_t ldy,
                                 const float* w, int32_t B, int32_t in, int32_t out, int32_t act, float* dy,
                                 int64_t lddy, float* dx, int64_t lddx, float* dw, float* db, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && x && y && w && dy && dw, "null pointer");
  ORX_REQUIRE(B > 0 && in > 0 && out > 0 && act >= 0 && act <= 2, "bad sizes");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  if (act != 0) {
    const int64_t n = (int64_t)B * out;
    k_act_bwd<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(y, ldy, dy, lddy, B, out, act);
    ORX_LAUNCH_CHECK();
  }
  if (db) {
    const int cb = (out + 31) / 32;
    int S = 1;
    if (B >= 4096) {
      S = (2 * h->num_sms + cb - 1) / cb;
      if (S > B / 256) S = B / 256;
    }
    if (S > 1) {
      int rc2 = orx_grow((void**)&h->splitk, &h->splitk_cap, sizeof(float) * (size_t)S * (size_t)out);
      if (rc2) return rc2;
      float* part = h->splitk;
      k_col_sum<<<dim3(cb, S), 256, 0, st>>>(dy, lddy, B, out, part);
      ORX_LAUNCH_CHECK();
      rc2 = orx_launch_splitk_reduce(part, S, 1, out, db, out, nullptr, 0, st);
      if (rc2) return rc2;
    } else {
      k_col_sum<<<cb, 256, 0, st>>>(dy, lddy, B, out, db);
      ORX_LAUNCH_CHECK();
    }
  }
  int rc = launch_gemm<1, 0>(h, x, ldx, dy, lddy, dw, out, in, out, B, nullptr, 0, st);   // dw = x^T dz
  if (rc) return rc;
  if (dx) rc = launch_gemm<0, 1>(h, dy, lddy, w, out, dx, lddx, B, in, out, nullptr, 0, st);   // dx = dz w^T
  return rc;
}

// ---------------------------------------------------------------------------------------
// prediction loss (dlrm.py:52-55,72-73,97-98): optional clip to [thr, 1-thr], then Keras
// MeanSquaredError (kind 0) or BinaryCrossentropy on probabilities (kind 1, eps = 1e-7 [TF-mem]).
// pred_out = clipped prediction; dpred = dloss/d(raw pred); out4[0] = loss.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_pred_loss(const float* __restrict__ pred, const float* __restrict__ label,
                                                   int B, int kind, float thr, float* __restrict__ pred_out,
                                                   float* __restrict__ dpred, float* partials) {
  __shared__ float sh[256];
  float acc = 0.f;
  const float invB = 1.f / (float)B;
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
    float p = pred[b];
    float pass = 1.f;
    if (thr > 0.f && thr < 1.f) {
      pass = (p >= thr && p <= 1.f - thr) ? 1.f : 0.f;
      p = fminf(fmaxf(p, thr), 1.f - thr);
    }
    const float y = label[b];
    float d;
    if (kind == 0) {
      acc += (y - p) * (y - p);
      d = 2.f * (p - y) * invB;
    } else {
      const float eps = 1e-7f;
      const float ph = fminf(fmaxf(p, eps), 1.f - eps);
      acc += -(y * logf(ph + eps) + (1.f - y) * logf(1.f - ph + eps));
      d = (p >= eps && p <= 1.f - eps) ? -(y / (ph + eps) - (1.f - y) / (1.f - ph + eps)) * invB : 0.f;
    }
    if (pred_out) pred_out[b] = p;
    if (dpred) dpred[b] = d * pass;
  }
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    partials[2 * blockIdx.x] = sh[0];
    partials[2 * blockIdx.x + 1] = 0.f;
  }
}

extern "C" int orx_pred_loss(orx_handle_t h, const float* pred, const float* label, int32_t B, int32_t kind,
                             float clip_threshold, float* pred_out, float* dpred, float* out4, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && pred && label && out4, "null pointer");
  ORX_REQUIRE(B > 0 && (kind == 0 || kind == 1), "bad sizes/kind");
  ORX_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)s;
  int blocks = (B + 255) / 256;
  if (blocks > 256) blocks = 256;
  const int rc = orx_grow((void**)&h->partials, &h->partials_cap, sizeof(float) * 2 * (size_t)blocks);
  if (rc) return rc;
  k_pred_loss<<<blocks, 256, 0, st>>>(pred, label, B, kind, clip_threshold, pred_out, dpred, h->partials);
  ORX_LAUNCH_CHECK();
  return orx_launch_reduce_partials(h->partials, blocks, 1.0f / (float)B, out4, st);
}

// ---------------------------------------------------------------------------------------
// Multi-hot features: Z[b, k, :] = the pooled bag of table k for sample b, all T tables in one launch.  Bag (b, k) is
// sparse[b*ld + col_off[k] .. col_off[k+1]); an id < 0 is padding, an id >= rows[k] is counted in n_bad; both add nothing.
// Sum: the valid rows added in column order, starting from the first valid row (so a bag of one id copies its row bit
// for bit, -0.0 included, like k_gather_strided); mean: that sum / the number of valid ids; no valid id: the zero row.
// ---------------------------------------------------------------------------------------
static_assert(ORX_BAG_MAX_TABLES + 1 <= ORX_MAX_F, "the pooled features and the dense vector must fit the interaction");

template <typename T>
struct BagTables {   // kernel parameter block: ~1.3 KB, read with register-indexed constant loads
  const T* tab[ORX_BAG_MAX_TABLES];
  int64_t rows[ORX_BAG_MAX_TABLES];
  int32_t col_off[ORX_BAG_MAX_TABLES + 1];
};

// One lane's load of a bag row chunk as stored (VEC: 4 columns, else 1): a float4 of a float table, the raw 8 bytes
// (uint2) of a bf16 one, so that the four loads in flight hold half the registers; bag_up widens it exactly.
template <bool VEC>
__device__ __forceinline__ float4 bag_ld(const float* p) {
  if (VEC) return __ldg(reinterpret_cast<const float4*>(p));
  return make_float4(__ldg(p), 0.f, 0.f, 0.f);
}
template <bool VEC>
__device__ __forceinline__ uint2 bag_ld(const uint16_t* p) {
  if (VEC) return __ldg(reinterpret_cast<const uint2*>(p));
  return make_uint2(__ldg(p), 0u);
}
__device__ __forceinline__ float4 bag_up(float4 v) { return v; }
__device__ __forceinline__ float4 bag_up(uint2 v) { return orx_bf16x4_up(v); }

__device__ __forceinline__ float4 bag_add(float4 a, float4 b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}

// One warp per bag, w = b*T + k (consecutive warps fill consecutive Z rows).  VEC: a lane holds one float4 of a
// 128-float column chunk, else one float of a 32-float chunk; wider rows take several chunks, each re-reading the ids.
// The ids are read 32 at a time (coalesced); a ballot gives the valid ones, which are taken four at a time: four row
// loads are issued before they are added, in column order.  S: the tables' storage, float or bf16 bits (uint16_t, rows
// widened exactly, so Z is the fp32 call's on the upcast tables bit for bit).
template <bool VEC, typename S = float>
__global__ void __launch_bounds__(256) k_bag_gather(const __grid_constant__ BagTables<S> bt, int T, int D,
                                                    const int32_t* __restrict__ sparse, int64_t ld, int64_t B,
                                                    int mean, float* __restrict__ out, int64_t out_ld,
                                                    int32_t* n_bad) {
  constexpr int W = VEC ? 4 : 1;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < B * T; w += nw) {
    const int64_t b = w / T;
    const int k = (int)(w - b * T);
    const S* tab = bt.tab[k];
    const int64_t rows = bt.rows[k];
    const int L = bt.col_off[k + 1] - bt.col_off[k];
    const int32_t* ids = sparse + b * ld + bt.col_off[k];
    float* dst = out + b * out_ld + (int64_t)k * D;
    for (int e0 = 0; e0 < D; e0 += 32 * W) {
      const int e = e0 + lane * W;
      const bool on = e < D;
      float4 acc = z4;
      int n = 0, bad = 0;
      for (int c = 0; c < L; c += 32) {
        const int32_t id = c + lane < L ? __ldg(ids + c + lane) : -1;
        uint32_t m = __ballot_sync(ORX_FULL, id >= 0 && id < rows);
        if (e0 == 0) bad += __popc(__ballot_sync(ORX_FULL, id >= rows));
        while (m) {   // warp-uniform
          int src[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            src[q] = m ? __ffs(m) - 1 : -1;
            m &= m - 1;
          }
          decltype(bag_ld<VEC>(tab)) v[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int64_t r = __shfl_sync(ORX_FULL, id, src[q] & 31);
            v[q] = (src[q] >= 0 && on) ? bag_ld<VEC>(tab + r * D + e) : decltype(bag_ld<VEC>(tab)){};
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (src[q] < 0) break;
            acc = n ? bag_add(acc, bag_up(v[q])) : bag_up(v[q]);
            ++n;
          }
        }
      }
      if (e0 == 0 && lane == 0 && bad && n_bad) atomicAdd(n_bad, bad);
      if (mean && n) {
        const float fn = (float)n;
        acc = make_float4(acc.x / fn, acc.y / fn, acc.z / fn, acc.w / fn);
      }
      if (!on) continue;
      if (VEC) *reinterpret_cast<float4*>(dst + e) = acc;
      else dst[e] = acc.x;
    }
  }
}

// VEC rule: out 16-byte aligned, every table 16-byte (float) / 8-byte (bf16) aligned, dim and out_ld multiples of 4.
template <typename S>
static int bag_gather_impl(orx_handle_t h, const S* const* tabs_host, const int64_t* rows_host, int32_t T,
                           int32_t dim, const int32_t* sparse, int64_t ld, const int32_t* col_off_host, int32_t B,
                           int32_t mode, float* out, int64_t out_ld, int32_t* n_bad, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && tabs_host && rows_host && col_off_host, "null pointer");
  ORX_REQUIRE(B == 0 || (sparse && out), "null sparse / out");
  ORX_REQUIRE(T >= 1 && T <= ORX_BAG_MAX_TABLES, "T outside [1, ORX_BAG_MAX_TABLES]");
  ORX_REQUIRE(dim >= 1 && B >= 0 && ld >= 1 && (mode == 0 || mode == 1), "bad sizes / mode");
  ORX_REQUIRE(out_ld >= (int64_t)T * dim, "out_ld < T * dim");
  ORX_REQUIRE(col_off_host[0] >= 0 && col_off_host[T] <= ld, "col_off outside [0, ld]");
  BagTables<S> bt;
  bool aligned = orx_aligned16(out);
  for (int k = 0; k < T; ++k) {
    ORX_REQUIRE(tabs_host[k] != nullptr && rows_host[k] > 0, "null table / empty vocabulary");
    ORX_REQUIRE(col_off_host[k + 1] >= col_off_host[k], "col_off decreasing");
    bt.tab[k] = tabs_host[k];
    bt.rows[k] = rows_host[k];
    bt.col_off[k] = col_off_host[k];
    aligned = aligned && (std::is_same<S, float>::value ? orx_aligned16(tabs_host[k]) : orx_aligned8(tabs_host[k]));
  }
  bt.col_off[T] = col_off_host[T];
  if (B == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  const int64_t bags = (int64_t)B * T;
  int64_t blocks = (bags + 7) / 8;
  if (blocks > (int64_t)h->num_sms * 32) blocks = (int64_t)h->num_sms * 32;
  cudaStream_t st = (cudaStream_t)s;
  if ((dim & 3) == 0 && (out_ld & 3) == 0 && aligned)
    k_bag_gather<true, S><<<(int)blocks, 256, 0, st>>>(bt, T, dim, sparse, ld, B, mode, out, out_ld, n_bad);
  else
    k_bag_gather<false, S><<<(int)blocks, 256, 0, st>>>(bt, T, dim, sparse, ld, B, mode, out, out_ld, n_bad);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

extern "C" int orx_bag_gather(orx_handle_t h, const float* const* tabs_host, const int64_t* rows_host, int32_t T,
                              int32_t dim, const int32_t* sparse, int64_t ld, const int32_t* col_off_host, int32_t B,
                              int32_t mode, float* out, int64_t out_ld, int32_t* n_bad, orx_stream_t s) {
  return bag_gather_impl(h, tabs_host, rows_host, T, dim, sparse, ld, col_off_host, B, mode, out, out_ld, n_bad, s);
}

extern "C" int orx_bag_gather_bf16(orx_handle_t h, const uint16_t* const* tabs_host, const int64_t* rows_host,
                                   int32_t T, int32_t dim, const int32_t* sparse, int64_t ld,
                                   const int32_t* col_off_host, int32_t B, int32_t mode, float* out, int64_t out_ld,
                                   int32_t* n_bad, orx_stream_t s) {
  return bag_gather_impl(h, tabs_host, rows_host, T, dim, sparse, ld, col_off_host, B, mode, out, out_ld, n_bad, s);
}
