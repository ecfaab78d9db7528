// orx_cross.cu -- the element-wise passes of the DCN-v2 cross network (Wang et al., 2021; TensorFlow Recommenders'
// tfrs.layers.dcn.Cross).  The projections y_l = U_l (V_l^T x_l) + b_l (or K_l x_l + b_l) run on orx_mlp_layer_fwd/bwd;
// these kernels do what lies between them:
//   forward   x_{l+1} = x0 * y_l + x_l
//   backward  per layer, top first: g = G (+ P), dy = g * x0, A (+)= g * y   (G <- g in place)
//   final     dL/dx0 = G + P + A, split by column into the bottom MLP's gradient and a contiguous dZ
// All passes are bandwidth bound; each element is read and written by one thread, so there are no atomics and the same
// inputs give the same bits.
#include "orx_common.cuh"

// VEC: one float4 per item (W, every leading dimension and, for the final pass, split multiples of 4, every base 16-byte
// aligned -- the launcher decides); else one float per item, any W >= 1 and any 4-byte-aligned base.
template <bool VEC>
__device__ __forceinline__ float4 cx_ld(const float* p) {
  if (VEC) return *reinterpret_cast<const float4*>(p);
  return make_float4(*p, 0.f, 0.f, 0.f);
}
template <bool VEC>
__device__ __forceinline__ void cx_st(float* p, float4 v) {
  if (VEC) *reinterpret_cast<float4*>(p) = v;
  else *p = v.x;
}
__device__ __forceinline__ float4 cx_fma(float4 a, float4 b, float4 c) {   // a * b + c, one rounding per element
  return make_float4(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y), __fmaf_rn(a.z, b.z, c.z),
                     __fmaf_rn(a.w, b.w, c.w));
}
__device__ __forceinline__ float4 cx_mul(float4 a, float4 b) {
  return make_float4(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y), __fmul_rn(a.z, b.z), __fmul_rn(a.w, b.w));
}
__device__ __forceinline__ float4 cx_add(float4 a, float4 b) {
  return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}

// Rows are dealt to blockIdx.y (grid-stride), a row's items to blockIdx.x * blockDim.x + threadIdx.x (grid-stride):
// no integer division per item.
#define CROSS_ROWS_LOOP(B, nq)                                                                \
  for (int64_t b = blockIdx.y; b < (B); b += gridDim.y)                                       \
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < (nq); q += gridDim.x * blockDim.x)

template <bool VEC>
__global__ void __launch_bounds__(256) k_cross_fwd(const float* __restrict__ x0, int64_t ld0,
                                                   const float* __restrict__ xl, int64_t ldl,
                                                   const float* __restrict__ y, int64_t ldy, int B, int W,
                                                   float* __restrict__ out, int64_t ldo) {
  constexpr int V = VEC ? 4 : 1;
  const int nq = W / V;
  CROSS_ROWS_LOOP(B, nq) {
    const int e = q * V;
    cx_st<VEC>(out + b * ldo + e, cx_fma(cx_ld<VEC>(x0 + b * ld0 + e), cx_ld<VEC>(y + b * ldy + e),
                                         cx_ld<VEC>(xl + b * ldl + e)));
  }
}

struct CrossBwdArgs {
  float* G; int64_t ldG;
  const float* P; int64_t ldP;
  const float* x0; int64_t ld0;
  const float* y; int64_t ldy;
  float* A; int64_t ldA;
  float* dy; int64_t lddy;
  int split;
  float* lo; int64_t ldlo;
  float* hi; int64_t ldhi;
};

// MODE = orx_cross_mode: TOP reads G, x0, y and writes dy, A; MID reads G, P, x0, y, A and writes G, dy, A; FINAL reads
// G, P, A and writes lo (columns < split) / hi (columns >= split, re-based at column 0).
template <int MODE, bool VEC>
__global__ void __launch_bounds__(256) k_cross_bwd(const __grid_constant__ CrossBwdArgs a, int B, int W) {
  constexpr int V = VEC ? 4 : 1;
  const int nq = W / V;
  CROSS_ROWS_LOOP(B, nq) {
    const int e = q * V;
    float4 g = cx_ld<VEC>(a.G + b * a.ldG + e);
    if (MODE != ORX_CROSS_TOP) g = cx_add(g, cx_ld<VEC>(a.P + b * a.ldP + e));
    if (MODE == ORX_CROSS_FINAL) {
      const float4 d = cx_add(g, cx_ld<VEC>(a.A + b * a.ldA + e));
      if (e < a.split) cx_st<VEC>(a.lo + b * a.ldlo + e, d);
      else cx_st<VEC>(a.hi + b * a.ldhi + (e - a.split), d);
      continue;
    }
    const float4 yv = cx_ld<VEC>(a.y + b * a.ldy + e);
    cx_st<VEC>(a.dy + b * a.lddy + e, cx_mul(g, cx_ld<VEC>(a.x0 + b * a.ld0 + e)));
    if (MODE == ORX_CROSS_TOP) {
      cx_st<VEC>(a.A + b * a.ldA + e, cx_mul(g, yv));
    } else {
      cx_st<VEC>(a.A + b * a.ldA + e, cx_fma(g, yv, cx_ld<VEC>(a.A + b * a.ldA + e)));
      cx_st<VEC>(a.G + b * a.ldG + e, g);
    }
  }
}

// 256 threads over a row's items (several blocks for a wide row), rows spread so that about 32 blocks per SM are in
// flight.
static dim3 cross_grid(const orx_ctx* h, int B, int nq) {
  const int bx = (nq + 255) / 256;
  int64_t by = (int64_t)h->num_sms * 32 / bx;
  if (by < 1) by = 1;
  if (by > B) by = B;
  if (by > 65535) by = 65535;
  return dim3((unsigned)bx, (unsigned)by);
}

static bool ld4(int64_t ld) { return (ld & 3) == 0; }

extern "C" int orx_cross_fwd(orx_handle_t h, const float* x0, int64_t ld_x0, const float* xl, int64_t ld_xl,
                             const float* y, int64_t ld_y, int32_t B, int32_t W, float* out, int64_t ld_out,
                             orx_stream_t s) {
  ORX_REQUIRE(h != nullptr && x0 && xl && y && out, "null pointer");
  ORX_REQUIRE(B >= 0 && W >= 1 && ld_x0 >= W && ld_xl >= W && ld_y >= W && ld_out >= W, "bad sizes");
  if (B == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  const bool vec = (W & 3) == 0 && ld4(ld_x0) && ld4(ld_xl) && ld4(ld_y) && ld4(ld_out) && orx_aligned16(x0, xl, y, out);
  cudaStream_t st = (cudaStream_t)s;
  if (vec)
    k_cross_fwd<true><<<cross_grid(h, B, W / 4), 256, 0, st>>>(x0, ld_x0, xl, ld_xl, y, ld_y, B, W, out, ld_out);
  else
    k_cross_fwd<false><<<cross_grid(h, B, W), 256, 0, st>>>(x0, ld_x0, xl, ld_xl, y, ld_y, B, W, out, ld_out);
  ORX_LAUNCH_CHECK();
  orx_log_dispatch(h, ORX_OP_CROSS, vec ? ORX_VARIANT_CROSS_VEC : ORX_VARIANT_CROSS_SCALAR, 0, 0, B, W, 0, 1);
  return ORX_OK;
}

extern "C" int orx_cross_bwd(orx_handle_t h, int32_t mode, int32_t B, int32_t W, float* G, int64_t ld_G,
                             const float* P, int64_t ld_P, const float* x0, int64_t ld_x0, const float* y, int64_t ld_y,
                             float* A, int64_t ld_A, float* dy, int64_t ld_dy, int32_t split, float* dx_lo,
                             int64_t ld_lo, float* dx_hi, int64_t ld_hi, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_REQUIRE(mode == ORX_CROSS_TOP || mode == ORX_CROSS_MID || mode == ORX_CROSS_FINAL, "unknown mode");
  ORX_REQUIRE(B >= 0 && W >= 1 && ld_G >= W && ld_A >= W, "bad sizes");
  ORX_REQUIRE(G && A, "null G / A");
  const bool fin = mode == ORX_CROSS_FINAL;
  if (mode != ORX_CROSS_TOP) ORX_REQUIRE(P && ld_P >= W, "null P / ld_P < W");
  if (!fin) ORX_REQUIRE(x0 && y && dy && ld_x0 >= W && ld_y >= W && ld_dy >= W, "null x0 / y / dy or ld < W");
  if (fin) {
    ORX_REQUIRE(split >= 0 && split <= W, "split outside [0, W]");
    ORX_REQUIRE(split == 0 || (dx_lo && ld_lo >= split), "null dx_lo / ld_lo < split");
    ORX_REQUIRE(split == W || (dx_hi && ld_hi >= W - split), "null dx_hi / ld_hi < W - split");
  }
  if (B == 0) return ORX_OK;
  ORX_CUDA(cudaSetDevice(h->device));
  CrossBwdArgs a{G, ld_G, mode == ORX_CROSS_TOP ? nullptr : P, ld_P, fin ? nullptr : x0, ld_x0, fin ? nullptr : y, ld_y,
                 A, ld_A, fin ? nullptr : dy, ld_dy, fin ? split : 0, fin ? dx_lo : nullptr, ld_lo,
                 fin ? dx_hi : nullptr, ld_hi};
  // the operands this mode touches (null ones count as aligned)
  bool vec = (W & 3) == 0 && ld4(ld_G) && ld4(ld_A) && orx_aligned16(a.G, a.A, a.P, a.x0, a.y, a.dy, a.lo, a.hi);
  if (mode != ORX_CROSS_TOP) vec = vec && ld4(ld_P);
  if (!fin) vec = vec && ld4(ld_x0) && ld4(ld_y) && ld4(ld_dy);
  else vec = vec && (split & 3) == 0 && (split == 0 || ld4(ld_lo)) && (split == W || ld4(ld_hi));
  const dim3 grid = cross_grid(h, B, vec ? W / 4 : W);
  cudaStream_t st = (cudaStream_t)s;
  orx_dispatch<ORX_CROSS_TOP, ORX_CROSS_MID, ORX_CROSS_FINAL>(mode, [&](auto M) {
    if (vec) k_cross_bwd<decltype(M)::value, true><<<grid, 256, 0, st>>>(a, B, W);
    else k_cross_bwd<decltype(M)::value, false><<<grid, 256, 0, st>>>(a, B, W);
  });
  ORX_LAUNCH_CHECK();
  orx_log_dispatch(h, ORX_OP_CROSS, vec ? ORX_VARIANT_CROSS_VEC : ORX_VARIANT_CROSS_SCALAR, 1, mode, B, W,
                   fin ? split : 0, 1);
  return ORX_OK;
}
