// orx_mlp_tc.cu -- Dense-layer GEMMs on the Hopper tensor cores: TMA-fed wgmma .tf32, accumulators in registers.
//
// DLRM's MLPs (openrec/tf2/modules/multi_layer_perceptron.py:5-18, recommenders/dlrm.py:34-37,87,90-95) are the one
// dense contraction on the path.  The parity bar is 1e-5 against an fp32 reference, which plain TF32 (10-bit mantissa)
// cannot meet, so every fp32 operand is split into two TF32 terms (hi = TF32(v) rounded to nearest, lo = v - hi)
// and  C += Ahi*Bhi + Ahi*Blo + Alo*Bhi  is accumulated in fp32 (3xTF32, relative error ~2^-21 per product).
//
// One CTA (three warpgroups) computes a 128 x 128 tile of  C[M,N] = op(A)[M,K] * op(B)[K,N], K in blocks of 16, with
// four rings of mbarriers between its two kinds of warpgroups:
//   warpgroup 0    converters: read a raw stage (conflict-free: swizzled 128-bit loads, or four coalesced scalars for
//                  the transposing case), split into hi / lo and store both tiles in the canonical K-major, no-swizzle
//                  wgmma layout (8-row x 16-byte core matrices, LBO 128 B, SBO 512 B) of a 3-stage operand ring --
//                  conflict-free 128-bit stores in both cases.  One lane of warp 0 is also the TMA producer:
//                  cp.async.bulk.tensor.2d loads the RAW fp32 A and B blocks of a k-block straight from the operands' own
//                  layouts (row stride = ld; out-of-range rows / k are zero-filled by the TMA) into a 4-stage raw ring,
//                  three k-blocks ahead of the conversion.  K-contiguous sources arrive as [rows][16] with the 64-byte
//                  swizzle, M/N-contiguous ones ([k][rows], e.g. w in the forward pass, x and dz in dw = x^T dz) as [16][rows].
//   warpgroups 1-2 MMA: warpgroup g owns rows 64g .. 64g+63 of the tile; per k-block 2 k-steps x 3 wgmma.m64n128k8 with
//                  both operands read from the operand ring, one k-block in flight while the next one is issued.
// The tensor core's fp32 accumulation truncates, and over hundreds of accumulations that bias grows linearly with K, so
// a wgmma accumulator only ever sums 4 k-blocks (64 K-elements, 24 MMAs) before it is added into a second set of fp32
// registers (round-to-nearest adds) and restarted.
// Epilogue through shared memory (coalesced rows, + bias, activation); split-K (blockIdx.z) for dw = x^T dz, whose K is
// the batch.  Shapes TMA cannot describe (row stride not a multiple of 16 bytes) or that are too small for a tile are
// left to the fp32 SIMT kernel of orx_dlrm.cu (ORX_ERR_UNSUPPORTED).
#include <cuda.h>
#include <stdlib.h>

#include "orx_common.cuh"

namespace {

constexpr int TM = 128, TN = 128, TK = 16;
constexpr int RAW_STAGES = 4, OP_STAGES = 3, GROUP_KB = 4;
constexpr int OP_SBO = (TK / 4) * 128;           // bytes between 8-row groups of an operand tile
constexpr int NCW = 4;                           // converter warps (warpgroup 0)
constexpr int THREADS = 3 * 128;
constexpr int RAW_A = TM * TK * 4, RAW_B = TN * TK * 4, RAW_STAGE = RAW_A + RAW_B;
constexpr int OP_A = TM * TK * 4, OP_B = TN * TK * 4, OP_STAGE = 2 * OP_A + 2 * OP_B;
constexpr int SMEM = RAW_STAGES * RAW_STAGE + OP_STAGES * OP_STAGE;   // 64 KB + 96 KB
static_assert(TM * (TN + 1) * 4 <= SMEM, "the epilogue tile must fit in the rings");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// K-major, no-swizzle shared-memory matrix descriptor of wgmma (PTX ISA: "Matrix Descriptor Format")
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);                  // start address        bits [0,14)
  d |= (uint64_t)(128 >> 4) << 16;                          // leading byte offset  bits [16,30): K-adjacent core matrices
  d |= (uint64_t)(OP_SBO >> 4) << 32;                       // stride byte offset   bits [32,46): next 8-row group
  return d;                                                 // base offset 0, layout type 0 = no swizzle (bits 62-63)
}

// D[64 x 128] (+)= A[64 x 8] * B[8 x 128]^T, TF32 in, FP32 accumulate, both operands K-major in shared memory.
// Fragment of D: register j of a thread sits at row 16 * (warp % 4) + lane / 4 + 8 * ((j >> 1) & 1),
// column 8 * (j >> 2) + 2 * (lane & 3) + (j & 1).
#define ORX_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                  "+f"(d[i + 6]), "+f"(d[i + 7])
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}\n"
      : ORX_D8(0), ORX_D8(8), ORX_D8(16), ORX_D8(24), ORX_D8(32), ORX_D8(40), ORX_D8(48), ORX_D8(56)
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
#undef ORX_D8
// the accumulator registers are written asynchronously: keep the compiler from moving their uses across the fences
__device__ __forceinline__ void fence_operands(float (&d)[64]) {
#pragma unroll
  for (int j = 0; j < 64; ++j) asm volatile("" : "+f"(d[j])::"memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tWAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// one 2-D TMA load: box at (c0 = inner coordinate, c1 = outer coordinate) -> shared memory, completion on `bar`
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(smem_dst)),
      "l"(tm), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}

// hi = TF32(v) rounded to nearest (cvt.rna: truncation would bias every product the same way and the error would grow
// linearly with K instead of with sqrt(K)); lo = v - hi exactly (|lo| <= 2^-11 |v|).  lo is handed to the tensor core as
// it is: .tf32 reads the top 19 bits, i.e. truncates lo by at most 2^-10 |lo| <= 2^-21 |v| -- the size of the
// lo*lo term 3xTF32 drops anyway, and of random sign because hi was rounded to nearest.
__device__ __forceinline__ float to_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}
__device__ __forceinline__ void split4(const float4 v, float4* hi, float4* lo) {
  hi->x = to_tf32(v.x); lo->x = v.x - hi->x;
  hi->y = to_tf32(v.y); lo->y = v.y - hi->y;
  hi->z = to_tf32(v.z); lo->z = v.z - hi->z;
  hi->w = to_tf32(v.w); lo->w = v.w - hi->w;
}

// One warp-item of the conversion: 32 (row, 4-k group) pairs of a raw tile -> hi / lo operand tiles.
//  KC = true : raw is [R rows][16 k] with the TMA 64-byte swizzle (16-byte chunk c of row r sits at chunk c ^ ((r >> 1) & 3));
//              item `wi` covers rows 8*wi .. 8*wi+7: lane -> row 8*wi + (lane & 7), k-core lane >> 3.  A quarter-warp reads
//              eight rows of one k-core (8 distinct bank groups thanks to the swizzle) and writes 128 contiguous bytes.
//  KC = false: raw is [16 k][R rows]; item `wi` covers k-core wi & 3 of rows 32*(wi >> 2) .. +31: four coalesced scalar
//              loads per lane, one 128-bit store per tile (a quarter-warp again writes 128 contiguous bytes).
// The byte offsets of an item inside a raw stage / an operand tile do not depend on the k-block: computed once per thread.
template <bool KC>
__device__ __forceinline__ void item_offsets(int R, int wi, int lane, int* src_off, int* dst_off) {
  int row, kcore;
  if (KC) {
    row = 8 * wi + (lane & 7);
    kcore = lane >> 3;
    *src_off = row * 64 + ((kcore ^ ((row >> 1) & 3)) << 4);
  } else {
    row = 32 * (wi >> 2) + lane;
    kcore = wi & 3;
    *src_off = (kcore * 4 * R + row) * 4;
  }
  *dst_off = (row >> 3) * OP_SBO + kcore * 128 + (row & 7) * 16;
}
template <bool KC, int R>
__device__ __forceinline__ void convert_item(const unsigned char* raw, int src_off, int dst_off, unsigned char* hi_tile,
                                             unsigned char* lo_tile) {
  float4 v;
  if (KC) {
    v = *reinterpret_cast<const float4*>(raw + src_off);
  } else {
    const float* p = reinterpret_cast<const float*>(raw + src_off);
    v.x = p[0];
    v.y = p[R];
    v.z = p[2 * R];
    v.w = p[3 * R];
  }
  float4 h, l;
  split4(v, &h, &l);
  *reinterpret_cast<float4*>(hi_tile + dst_off) = h;
  *reinterpret_cast<float4*>(lo_tile + dst_off) = l;
}

// TA / TB as in orx_dlrm.cu: TA = 0: A[m*lda + k]; TA = 1: A[k*lda + m]; TB = 0: B[k*ldb + n]; TB = 1: B[n*ldb + k].
template <int TA, int TB>
__global__ void __launch_bounds__(THREADS, 1)
k_gemm_tma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, float* __restrict__ C,
           int64_t ldc, int M, int N, int K, const float* __restrict__ bias, int act, float* __restrict__ part) {
  constexpr bool A_KC = TA == 0, B_KC = TB == 1;   // K-contiguous sources
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t raw_full[RAW_STAGES], raw_empty[RAW_STAGES], op_full[OP_STAGES], op_empty[OP_STAGES];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wgi = __shfl_sync(ORX_FULL, (int)threadIdx.x >> 7, 0);   // warpgroup index, visibly warp-uniform
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  unsigned char* raw_ring = smem;
  unsigned char* op_ring = smem + RAW_STAGES * RAW_STAGE;

  if (threadIdx.x == 0) {
    for (int s = 0; s < RAW_STAGES; ++s) { mbar_init(&raw_full[s], 1); mbar_init(&raw_empty[s], NCW); }
    for (int s = 0; s < OP_STAGES; ++s) { mbar_init(&op_full[s], NCW); mbar_init(&op_empty[s], 8); }   // 8 MMA warps
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  __syncthreads();

  // this CTA's range of k-blocks (split-K over blockIdx.z)
  const int nkb_all = (K + TK - 1) / TK;
  const int per = (nkb_all + (int)gridDim.z - 1) / (int)gridDim.z;
  const int kb_lo = blockIdx.z * per;
  const int nkb = max(0, min(nkb_all, kb_lo + per) - kb_lo);

  float sum[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) sum[j] = 0.f;

  if (wgi == 0) {
    // ------------------------------------------------ TMA producer (one lane) + converters
    auto load = [&](int kb) {
      const int rs = kb % RAW_STAGES;
      unsigned char* st = raw_ring + (size_t)rs * RAW_STAGE;
      const int k0 = (kb_lo + kb) * TK;
      mbar_expect_tx(&raw_full[rs], RAW_STAGE);               // a box is always delivered whole (out of range = zeros)
      if (A_KC) tma_load_2d(st, &tmA, k0, m0, &raw_full[rs]); else tma_load_2d(st, &tmA, m0, k0, &raw_full[rs]);
      if (B_KC) tma_load_2d(st + RAW_A, &tmB, k0, n0, &raw_full[rs]); else tma_load_2d(st + RAW_A, &tmB, n0, k0, &raw_full[rs]);
    };
    const bool producer = warp == 0 && lane == 0;
    if (producer)
      for (int kb = 0; kb < min(nkb, RAW_STAGES - 1); ++kb) load(kb);
    constexpr int ITEMS_A = TM / 8, ITEMS_B = TN / 8;          // warp-items per tile (32 (row, k-core) pairs each)
    constexpr int NIT = (ITEMS_A + ITEMS_B) / NCW;             // items per warp and k-block; item i of warp w is w + NCW*i
    static_assert((ITEMS_A + ITEMS_B) % NCW == 0 && ITEMS_A % NCW == 0, "items must divide evenly");
    constexpr int NIT_A = ITEMS_A / NCW;                       // the first NIT_A items of a warp belong to A, the rest to B
    int src_off[NIT], dst_off[NIT];
#pragma unroll
    for (int i = 0; i < NIT; ++i) {
      const int wi = warp + NCW * i;
      if (i < NIT_A) item_offsets<A_KC>(TM, wi, lane, &src_off[i], &dst_off[i]);
      else item_offsets<B_KC>(TN, wi - ITEMS_A, lane, &src_off[i], &dst_off[i]);
    }
    for (int kb = 0; kb < nkb; ++kb) {
      const int rs = kb % RAW_STAGES, os = kb % OP_STAGES;
      // refill the raw stage block kb-1 used (every converter warp has left it, or is about to)
      const int nk = kb + RAW_STAGES - 1;
      if (producer && nk < nkb) {
        if (nk >= RAW_STAGES) mbar_wait(&raw_empty[nk % RAW_STAGES], ((nk / RAW_STAGES) - 1) & 1);
        load(nk);
      }
      __syncwarp();
      mbar_wait(&raw_full[rs], (kb / RAW_STAGES) & 1);
      if (kb >= OP_STAGES) mbar_wait(&op_empty[os], ((kb / OP_STAGES) - 1) & 1);   // the MMAs of block kb-3 left this stage
      const unsigned char* ra = raw_ring + (size_t)rs * RAW_STAGE;
      const unsigned char* rb = ra + RAW_A;
      unsigned char* oa = op_ring + (size_t)os * OP_STAGE;
      unsigned char* ob = oa + 2 * OP_A;
#pragma unroll
      for (int i = 0; i < NIT; ++i) {
        if (i < NIT_A) convert_item<A_KC, TM>(ra, src_off[i], dst_off[i], oa, oa + OP_A);
        else convert_item<B_KC, TN>(rb, src_off[i], dst_off[i], ob, ob + OP_B);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the tensor core
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&op_full[os]);
        mbar_arrive(&raw_empty[rs]);
      }
    }
  } else {
    // ------------------------------------------------ MMA warpgroups
    const int wg = wgi - 1;                                    // rows 64*wg .. 64*wg+63 of the tile
    float acc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0.f;
    const uint32_t op0 = smem_u32(op_ring);
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&op_empty[s]);
    };
    for (int g0 = 0; g0 < nkb; g0 += GROUP_KB) {             // one accumulation group: up to GROUP_KB k-blocks
      const int g1 = min(nkb, g0 + GROUP_KB);
      for (int kb = g0; kb < g1; ++kb) {
        const int os = kb % OP_STAGES;
        mbar_wait(&op_full[os], (kb / OP_STAGES) & 1);
        const uint32_t a_hi = op0 + (uint32_t)(os * OP_STAGE + wg * 8 * OP_SBO), a_lo = a_hi + OP_A;
        const uint32_t b_hi = op0 + (uint32_t)(os * OP_STAGE + 2 * OP_A), b_lo = b_hi + OP_B;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < TK / 8; ++ks) {
          const uint32_t o = (uint32_t)(ks * 256);             // two k-cores of 128 bytes
          wgmma_tf32(acc, make_desc(a_hi + o), make_desc(b_hi + o), (kb == g0 && ks == 0) ? 0u : 1u);
          wgmma_tf32(acc, make_desc(a_hi + o), make_desc(b_lo + o), 1u);
          wgmma_tf32(acc, make_desc(a_lo + o), make_desc(b_hi + o), 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();                                       // block kb-1 has retired: its stage is free
        if (kb > g0) release((kb - 1) % OP_STAGES);
      }
      wgmma_wait<0>();
      fence_operands(acc);
      release((g1 - 1) % OP_STAGES);
#pragma unroll
      for (int j = 0; j < 64; ++j) sum[j] += acc[j];
    }
  }

  // ---- epilogue through shared memory: every MMA has completed (the last k-block waited for all of them) and every
  // TMA load has been consumed, so the rings are free: tile[128][TN + 1] floats
  __syncthreads();
  float* tile = reinterpret_cast<float*>(smem);
  if (warp >= NCW) {
    const int r0 = 16 * (warp - NCW) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 64; ++j) tile[(r0 + 8 * ((j >> 1) & 1)) * (TN + 1) + 8 * (j >> 2) + c0 + (j & 1)] = sum[j];
  }
  __syncthreads();
  const bool split = gridDim.z > 1;
  float* out = split ? part + (size_t)blockIdx.z * (size_t)M * (size_t)N : C;
  const int64_t ldo = split ? (int64_t)N : ldc;
  for (int r = warp; r < TM; r += THREADS / 32) {
    const int m = m0 + r;
    if (m >= M) break;
#pragma unroll
    for (int c = 0; c < TN; c += 32) {
      const int n = n0 + c + lane;
      if (n < N) {
        float x = tile[r * (TN + 1) + c + lane];
        if (!split) {
          x += bias ? bias[n] : 0.f;
          if (act == 1) x = fmaxf(x, 0.f);
          else if (act == 2) x = orx_sigmoid(x);
        }
        out[(int64_t)m * ldo + n] = x;
      }
    }
  }
}

// sum of split-K partials (deterministic: fixed order), + bias, activation
__global__ void __launch_bounds__(256) k_splitk_reduce(const float* __restrict__ part, int S, int M, int N, float* __restrict__ C,
                                                       int64_t ldc, const float* __restrict__ bias, int act) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * N) return;
  const int m = (int)(i / N), n = (int)(i % N);
  float x = 0.f;
  for (int z = 0; z < S; ++z) x += part[(size_t)z * (size_t)M * (size_t)N + (size_t)i];
  x += bias ? bias[n] : 0.f;
  if (act == 1) x = fmaxf(x, 0.f);
  else if (act == 2) x = orx_sigmoid(x);
  C[(int64_t)m * ldc + n] = x;
}

// ---- host: TMA descriptors (cuTensorMapEncodeTiled through the runtime's driver entry point: no -lcuda needed)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// map of one operand: `kc` = its K dimension is the contiguous one ([rows, K] with row stride ld), else [K, rows]
int make_map(CUtensorMap* tm, const float* base, int rows, int K, int64_t ld, bool kc, int tile_rows) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) { orx_set_error("cuTensorMapEncodeTiled is not available in this driver"); return ORX_ERR_CUDA; }
  cuuint64_t dims[2], strides[1];
  cuuint32_t box[2], estr[2] = {1, 1};
  if (kc) { dims[0] = (cuuint64_t)K; dims[1] = (cuuint64_t)rows; box[0] = TK; box[1] = (cuuint32_t)tile_rows; }
  else { dims[0] = (cuuint64_t)rows; dims[1] = (cuuint64_t)K; box[0] = (cuuint32_t)tile_rows; box[1] = TK; }
  strides[0] = (cuuint64_t)ld * 4;
  const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, kc ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { orx_set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return ORX_ERR_CUDA; }
  return ORX_OK;
}

template <int TA, int TB>
int launch_tma(const CUtensorMap& ta, const CUtensorMap& tb, float* C, int64_t ldc, int M, int N, int K, const float* bias,
               int act, float* part, int S, cudaStream_t st) {
  ORX_CUDA(cudaFuncSetAttribute(k_gemm_tma<TA, TB>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM + 1024));
  dim3 grid((N + TN - 1) / TN, (M + TM - 1) / TM, S);
  k_gemm_tma<TA, TB><<<grid, THREADS, SMEM + 1024, st>>>(ta, tb, C, ldc, M, N, K, bias, act, part);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

}  // namespace

int orx_launch_splitk_reduce(const float* part, int S, int M, int N, float* C, int64_t ldc, const float* bias, int act, cudaStream_t st) {
  const int64_t n = (int64_t)M * N;
  k_splitk_reduce<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(part, S, M, N, C, ldc, bias, act);
  ORX_LAUNCH_CHECK();
  return ORX_OK;
}

// C[M,N] = op(A) * op(B) (+bias, act) on wgmma; same operand conventions as launch_gemm in orx_dlrm.cu.
// Returns ORX_ERR_UNSUPPORTED for shapes that are left to the SIMT kernel: tiny N / K / M, operands the TMA cannot
// describe (base not 16-byte aligned, row stride not a multiple of 16 bytes), or TA = TB = 1, which no Dense-layer GEMM
// uses.  A launch is recorded in h's dispatch log.
int orx_launch_gemm_tc(orx_ctx* h, int TA, int TB, const float* A, int64_t lda, const float* Bm, int64_t ldb, float* C,
                       int64_t ldc, int M, int N, int K, const float* bias, int act, cudaStream_t st) {
  if (TA == 1 && TB == 1) return ORX_ERR_UNSUPPORTED;
  if (N < 16 || K < 8 || M < 64) return ORX_ERR_UNSUPPORTED;
  if ((lda & 3) || (ldb & 3) || !orx_aligned16(A, Bm)) return ORX_ERR_UNSUPPORTED;
  const int tiles = ((N + TN - 1) / TN) * ((M + TM - 1) / TM);
  const int nkb = (K + TK - 1) / TK;
  int S = 1;
  const int sms = h->num_sms;
  if (tiles < sms && nkb >= 32) {             // too few tiles for the machine and a long K: split it
    S = (2 * sms + tiles - 1) / tiles;
    if (S > nkb / 8) S = nkb / 8;             // at least 8 k-blocks (two accumulation groups) per split
    if (S < 1) S = 1;
  }
  int rc;
  float* part = nullptr;
  if (S > 1) {
    if ((rc = orx_grow((void**)&h->splitk, &h->splitk_cap, sizeof(float) * (size_t)S * (size_t)M * (size_t)N))) return rc;
    part = h->splitk;
  }
  CUtensorMap ta, tb;
  if ((rc = make_map(&ta, A, M, K, lda, TA == 0, TM))) return rc;
  if ((rc = make_map(&tb, Bm, N, K, ldb, TB == 1, TN))) return rc;
#define ORX_TMA(a, b) rc = launch_tma<a, b>(ta, tb, C, ldc, M, N, K, bias, act, part, S, st)
  if (TA == 0 && TB == 0) ORX_TMA(0, 0);
  else if (TA == 0) ORX_TMA(0, 1);
  else ORX_TMA(1, 0);
#undef ORX_TMA
  if (rc) return rc;
  orx_log_dispatch(h, ORX_OP_GEMM, ORX_VARIANT_GEMM_TMA, TA, TB, M, N, K, S);
  if (S > 1) return orx_launch_splitk_reduce(part, S, M, N, C, ldc, bias, act, st);
  return ORX_OK;
}
