// Tensor-core GEMM engine for sm_90a (wgmma) with an fp32-grade split-bf16 operand scheme:
//   D = sum over K slices of A_hi*B_hi + A_hi*B_lo + A_lo*B_hi  (2 planes, ~4e-6 vs fp64), or with 3 planes hi/mid/lo the 6
//   products of weight >= 2^-16 (fp32-grade); x = hi + lo, hi = bf16(x), lo = bf16(x - hi) (SURVEY.md section 0, fact 3).
// Weights arrive as pre-split plane images by cp.async.bulk; activations arrive as fp32 by TMA (2-D tensor maps) and are
// split into K-major SWIZZLE_128B bf16 planes in shared memory.  One kernel per job:
// * gemm_w_kernel, 2-plane layers: 2 warpgroups, a 128 x WN output tile (WN = 256 for layers wider than 128 columns, so
//   that each activation row block is read from HBM and split once), a ring of fp32 activation slices split in place.
//   The accumulators go through shared memory to the fused epilogue functor (4 consecutive columns of a row per call).
// * gemm_w3_tma_kernel, 3-plane layers: persistent, a producer warpgroup feeding two consumer warpgroups through
//   mbarriers, the epilogue applied from the accumulator fragments.
// * gemm_tn_kernel, weight gradients: a producer warpgroup splitting a ring of fp32 slices of both operands into
//   MN-major planes for two consumer warpgroups through mbarriers, split-K over the points.
// Every activation operand has a row stride of whole 16-byte units and a 16-byte-aligned base (check_tma_operand).
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_bf16.h>

#include "gemm_simt.cuh"

namespace nudf {
namespace tc {

constexpr int BM = 128;
constexpr int BN = 128;        // output columns per CTA of gemm_tn_kernel and of the narrow gemm_w_kernel tile
constexpr int BK = 64;
constexpr int THREADS = 256;   // 2 warpgroups: MMA issue, operand staging and epilogue
constexpr int A_HALF_BYTES = BM * BK * 2;   // 16 KB: one plane of a [128 x 64] operand slice
__host__ __device__ constexpr int b_plane_bytes(int wn) { return wn * BK * 2; }   // one plane of a [wn x 64] weight slice
__host__ __device__ constexpr int acc_ld(int wn) { return wn + 4; }   // floats per row of the accumulator tile in smem

__host__ __device__ inline int pad16(int n) { return (n + 15) & ~15; }
__host__ __device__ inline int pad64(int k) { return (k + 63) & ~63; }

// byte offset of element (row, k) inside a [rows x 64] bf16 K-major SWIZZLE_128B tile (tile base 1024-aligned)
__host__ __device__ inline uint32_t sw128(uint32_t row, uint32_t k) {
  return (row >> 3) * 1024u + (row & 7u) * 128u + ((((k >> 3) ^ (row & 7u)) & 7u) << 4) + ((k & 7u) << 1);
}

// gemm_tn_kernel: slices of TN_PS points, fp32 operand blocks as they lie in HBM ([point][128 columns]) in a
// TN_LAND-deep landing ring, split into a TN_STAGES-deep ring of bf16 plane stages (hi, lo of A, then of B)
constexpr int TN_PS = 32;
constexpr int TN_LAND = 4;
constexpr int TN_STAGES = 3;
constexpr int TN_THREADS = 384;                              // a producer and two consumer warpgroups
constexpr int TN_PRODUCER_REGS = 104, TN_CONSUMER_REGS = 200;
static_assert(TN_PRODUCER_REGS + 2 * TN_CONSUMER_REGS <= 65536 / 128, "register file of one SM");
constexpr uint32_t TN_F32_OPND = TN_PS * BM * 4;            // 16 KB: one operand's [32 x 128] fp32 block
constexpr uint32_t TN_F32_STAGE = 2 * TN_F32_OPND;          // A, then B
constexpr uint32_t TN_PLANE = BM * TN_PS * 2;               // 8 KB: one bf16 plane of one operand
constexpr uint32_t TN_PLANE_STAGE = 4 * TN_PLANE;
struct TnMaps { CUtensorMap a, b; };                         // gemm_tn_kernel's 2-D tensor maps of A and B
// byte offset of element (mn, k) inside a [128 x 32] bf16 MN-major SWIZZLE_128B plane (base 1024-aligned): two 64-wide
// MN blocks of 4 KB, each four 1 KB atoms of 8 points x 128 B; the 16-byte chunk index is XOR-ed with the point's row
// in its atom, as the hardware's 128B swizzle does with address bits 4-6 and 7-9
__host__ __device__ inline uint32_t sw128_mn(uint32_t mn, uint32_t k) {
  return (mn >> 6) * 4096u + (k >> 3) * 1024u + (k & 7u) * 128u + ((((mn >> 3) ^ k) & 7u) << 4) + ((mn & 7u) << 1);
}

// gemm_w_kernel (2 planes): slots of one fp32 [128 x 64] activation slice as it lies in HBM, each split in
// place into its hi and lo planes; W_RING(WN) slots beside the two weight stages
constexpr uint32_t W_SLOT = BM * BK * 4;                     // 32 KB
static_assert(W_SLOT == 2 * A_HALF_BYTES, "a slot holds exactly the two bf16 planes of its slice");
__host__ __device__ constexpr int w_ring(int wn) { return wn == 256 ? 3 : 4; }

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
// split 4 consecutive values into NP bf16 planes (packed pairs): plane p holds bf16_rn of what the planes before it
// left, r -= plane.  One paired conversion per two values and plane; the plane's values are read back from its bits.
template <int NP>
__device__ __forceinline__ void split4(const float x[4], uint2 planes[NP]) {
  float r[4] = {x[0], x[1], x[2], x[3]};
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    const uint32_t a = pack_bf16(r[0], r[1]), b = pack_bf16(r[2], r[3]);
    planes[p] = make_uint2(a, b);
    r[0] -= __uint_as_float(a << 16);
    r[1] -= __uint_as_float(a & 0xffff0000u);
    r[2] -= __uint_as_float(b << 16);
    r[3] -= __uint_as_float(b & 0xffff0000u);
  }
}
// ---- weight image --------------------------------------------------------------------------------------------------
// For operand B(n, k), n < N, k < K: n-tiles of NT rows (NT = 256 with 2 planes, 128 with 3 planes; the last tile is
// padded to a multiple of 16), k-slices of 64.  NP planes per element: p0 = bf16(x), p1 = bf16(x - p0),
// p2 = bf16(x - p0 - p1).  Image order: [n_tile][k_slice][plane][tile rows x 128 B, SWIZZLE_128B K-major].  Units: uint16.
__host__ __device__ inline int nt_of(int np) { return np == 2 ? 256 : 128; }
__host__ __device__ inline int n_tiles(int N, int np) { return (N + nt_of(np) - 1) / nt_of(np); }
__host__ __device__ inline int tile_rows(int N, int t, int np) { int r = N - nt_of(np) * t; return pad16(r < nt_of(np) ? r : nt_of(np)); }
__host__ __device__ inline int64_t tile_elems(int N, int K, int t, int np) { return (int64_t)(pad64(K) / 64) * np * tile_rows(N, t, np) * 64; }
__host__ __device__ inline int64_t tile_offset(int N, int K, int t, int np) {
  int64_t o = 0;
  for (int i = 0; i < t; ++i) o += tile_elems(N, K, i, np);
  return o;
}
__host__ __device__ inline int64_t image_elems(int N, int K, int np) { return tile_offset(N, K, n_tiles(N, np), np); }

// transposed == 0: B(n,k) = W[n*ldw + k]   (X W^T)      transposed == 1: B(n,k) = W[k*ldw + n]   (dY W)
static __device__ __forceinline__ void tc_prep_weights_body(const float* __restrict__ W, int64_t ldw, int N, int K, int transposed, int np,
                                                            uint16_t* __restrict__ img, int64_t start, int64_t stride) {
  const int Kp = pad64(K);
  const int nt = n_tiles(N, np);
  int64_t total = 0;
  for (int t = 0; t < nt; ++t) total += (int64_t)tile_rows(N, t, np) * Kp;
  for (int64_t idx = start; idx < total; idx += stride) {
    int64_t rem = idx;
    int t = 0;
    while (rem >= (int64_t)tile_rows(N, t, np) * Kp) { rem -= (int64_t)tile_rows(N, t, np) * Kp; ++t; }
    const int rows = tile_rows(N, t, np);
    const int nl = (int)(rem / Kp), k = (int)(rem - (int64_t)nl * Kp);
    const int n = t * nt_of(np) + nl;
    float x = 0.f;
    if (n < N && k < K) x = transposed ? W[(int64_t)k * ldw + n] : W[(int64_t)n * ldw + k];
    const int s = k >> 6, kl = k & 63;
    uint16_t* base = img + tile_offset(N, K, t, np) + (int64_t)s * np * rows * 64;
    const uint32_t off = sw128((uint32_t)nl, (uint32_t)kl) >> 1;
    float r = x;
    for (int p = 0; p < np; ++p) {
      __nv_bfloat16 h = __float2bfloat16_rn(r);
      base[(int64_t)p * rows * 64 + off] = __bfloat16_as_ushort(h);
      r -= __bfloat162float(h);
    }
  }
}
static __global__ void tc_prep_weights_kernel(const float* __restrict__ W, int64_t ldw, int N, int K, int transposed, int np,
                                              uint16_t* __restrict__ img) {
  tc_prep_weights_body(W, ldw, N, K, transposed, np, img, (int64_t)blockIdx.x * blockDim.x + threadIdx.x, (int64_t)gridDim.x * blockDim.x);
}


// ---- PTX wrappers --------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// p (the dynamic shared array) rounded up to 1024 bytes by an offset: rounding the pointer through an integer would
// lose its address space, and every access through the result would compile to a generic load or store with a 64-bit
// address instead of LDS / STS
__device__ __forceinline__ uint8_t* align1024(uint8_t* p) { return p + ((1024u - (smem_u32(p) & 1023u)) & 1023u); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t addr, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(addr), "r"(parity)
      : "memory");
  return ok;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  while (!mbar_try_wait(addr, parity)) {
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy smem writes -> visible to the async proxy (tensor core operand fetch)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// the box of a 2-D tensor map whose first element is (column c, row k) into shared memory, on an mbarrier
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c, int k, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c), "r"(k), "r"(smem_u32(bar))
               : "memory");
}

// wgmma smem descriptor of a K-major operand: start, LBO, SBO (16-byte units), bits 62-63 = 1 (SWIZZLE_128B); SBO = 1024 B
// (8-row atoms)
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// wgmma smem descriptor of an MN-major SWIZZLE_128B operand in gemm_tn_kernel's plane layout (sw128_mn).  The PTX ISA's
// canonical MN-major 128B-swizzle layout is ((8 x 16 B, m), (8, k)) : ((contiguous, LBO), (128 B, SBO)): an atom is 8
// K rows of 128 contiguous bytes (64 bf16 along M or N), LBO is the step between 64-wide MN blocks (4096 B here, used
// by B's 128 columns) and SBO the step between 8-point K groups (1024 B: the atoms of a block are consecutive).
__device__ __forceinline__ uint64_t make_desc_mn(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(4096 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// the threads of one warpgroup (named barrier 1; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
// the two consumer warpgroups of gemm_tn_kernel (named barrier 2)
__device__ __forceinline__ void tn_consumer_bar_sync() { asm volatile("bar.sync 2, 256;" ::: "memory"); }
template <uint32_t R> __device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R> __device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_but_one() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// keeps the compiler from moving reads of an accumulator array across the (volatile) wait that completes it
template <int N>
__device__ __forceinline__ void fence_operand(float (&d)[N]) {
#pragma unroll
  for (int q = 0; q < N; ++q) asm volatile("" : "+f"(d[q])::"memory");
}
// r + half an ulp of r with the sign of r (the exponent bits times 2^-24): a result the tensor core truncated toward zero,
// moved to the middle of its truncation interval
__device__ __forceinline__ float unbias_rz(float r) { return fmaf(__uint_as_float(__float_as_uint(r) & 0xff800000u), 0x1p-24f, r); }

// D[64 x 128] (+)= A[64 x 16] B[128 x 16]^T from shared memory, bf16 operands; both K-major (MN_MAJOR = 0) or both
// MN-major (1: the transpose immediates of A and B set, descriptors from make_desc_mn)
template <int MN_MAJOR = 0>
__device__ __forceinline__ void wgmma_128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
      "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, "
      "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %67;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate), "n"(MN_MAJOR));
}
// D[64 x 128] = A[64 x 16] B[128 x 16]^T into fresh registers: write-only outputs, so that the compiler keeps no
// earlier value of d alive
__device__ __forceinline__ void wgmma_128_fresh(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
      "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, "
      "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n"
      "}\n"
      : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]), "=f"(d[9]),
        "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]), "=f"(d[17]), "=f"(d[18]),
        "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]), "=f"(d[24]), "=f"(d[25]), "=f"(d[26]), "=f"(d[27]),
        "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31]), "=f"(d[32]), "=f"(d[33]), "=f"(d[34]), "=f"(d[35]), "=f"(d[36]),
        "=f"(d[37]), "=f"(d[38]), "=f"(d[39]), "=f"(d[40]), "=f"(d[41]), "=f"(d[42]), "=f"(d[43]), "=f"(d[44]), "=f"(d[45]),
        "=f"(d[46]), "=f"(d[47]), "=f"(d[48]), "=f"(d[49]), "=f"(d[50]), "=f"(d[51]), "=f"(d[52]), "=f"(d[53]), "=f"(d[54]),
        "=f"(d[55]), "=f"(d[56]), "=f"(d[57]), "=f"(d[58]), "=f"(d[59]), "=f"(d[60]), "=f"(d[61]), "=f"(d[62]), "=f"(d[63])
      : "l"(da), "l"(db), "r"(0u));
}

// D[64 x 256] (+)= A[64 x 16] B[256 x 16]^T, the same operands as wgmma_128 with twice the rows of B
__device__ __forceinline__ void wgmma_256(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, "
      "%25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, "
      "%71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, "
      "%94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, "
      "%114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]),
        "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
        "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]),
        "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]),
        "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]),
        "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]),
        "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]),
        "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]),
        "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]),
        "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]),
        "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]),
        "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(accumulate));
}

// The wgmma group of one 64-wide K slice, smallest products first; plane p at +p * stride, 32 B per 16-wide K step.
// With 3 planes only the five correction products (lo * hi, hi * lo, mid * mid, mid * hi, hi * mid: ~2^-8 of the result's
// scale, so the tensor core's truncation of each wgmma result to fp32 costs ~2^-32 of it); gemm_w3_tma_kernel issues each
// hi * hi step into fresh accumulators and adds them up in fp32 with round-to-nearest.
// WN (128 or 256) is the width of the weight slice and of the accumulator fragment.
template <int WN>
__device__ __forceinline__ void wgmma_n(float (&d)[WN / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (WN == 256) wgmma_256(d, da, db, accumulate);
  else wgmma_128(d, da, db, accumulate);
}
template <int NP, int WN>
__device__ __forceinline__ void mma_slice(float (&d)[WN / 2], uint32_t a, uint32_t a_stride, uint32_t b, uint32_t b_stride, bool zero_first) {
  auto desc = [](uint32_t base, uint32_t stride, int p, int j) { return make_desc(base + p * stride + 32u * j); };
#pragma unroll
  for (int j = 0; j < BK / 16; ++j) {
    const uint32_t acc0 = (zero_first && j == 0) ? 0u : 1u;
    if constexpr (NP == 2) {
      wgmma_n<WN>(d, desc(a, a_stride, 1, j), desc(b, b_stride, 0, j), acc0);
      wgmma_n<WN>(d, desc(a, a_stride, 0, j), desc(b, b_stride, 1, j), 1u);
      wgmma_n<WN>(d, desc(a, a_stride, 0, j), desc(b, b_stride, 0, j), 1u);
    } else {
      wgmma_n<WN>(d, desc(a, a_stride, 2, j), desc(b, b_stride, 0, j), acc0);   // lo * hi
      wgmma_n<WN>(d, desc(a, a_stride, 0, j), desc(b, b_stride, 2, j), 1u);     // hi * lo
      wgmma_n<WN>(d, desc(a, a_stride, 1, j), desc(b, b_stride, 1, j), 1u);     // mid * mid
      wgmma_n<WN>(d, desc(a, a_stride, 1, j), desc(b, b_stride, 0, j), 1u);     // mid * hi
      wgmma_n<WN>(d, desc(a, a_stride, 0, j), desc(b, b_stride, 1, j), 1u);     // hi * mid
    }
  }
}
// The wgmma group of one TN_PS-point slice of gemm_tn_kernel: MN-major planes (lo at +TN_PLANE), 2 KB per
// 16-point step, the products of each step in mma_slice<2>'s order
__device__ __forceinline__ void mma_slice_mn(float (&d)[64], uint32_t a, uint32_t b, bool zero_first) {
#pragma unroll
  for (int j = 0; j < TN_PS / 16; ++j) {
    const uint32_t acc0 = (zero_first && j == 0) ? 0u : 1u;
    const uint32_t aj = a + 2048u * j, bj = b + 2048u * j;
    wgmma_128<1>(d, make_desc_mn(aj + TN_PLANE), make_desc_mn(bj), acc0);
    wgmma_128<1>(d, make_desc_mn(aj), make_desc_mn(bj + TN_PLANE), 1u);
    wgmma_128<1>(d, make_desc_mn(aj), make_desc_mn(bj), 1u);
  }
}

// m64n{WN} accumulator fragment of warpgroup wg -> row-major [128 x acc_ld(WN)] fp32 tile in shared memory
template <int WN>
__device__ __forceinline__ void acc_to_smem(const float (&d)[WN / 2], float* acc_s, int wg, int wtid) {
  constexpr int LD = acc_ld(WN);
  const int r = 64 * wg + 16 * (wtid >> 5) + ((wtid & 31) >> 2);
  const int c = 2 * (wtid & 3);
#pragma unroll
  for (int g = 0; g < WN / 8; ++g) {
    *reinterpret_cast<float2*>(acc_s + r * LD + 8 * g + c) = make_float2(d[4 * g], d[4 * g + 1]);
    *reinterpret_cast<float2*>(acc_s + (r + 8) * LD + 8 * g + c) = make_float2(d[4 * g + 2], d[4 * g + 3]);
  }
}
// Fused epilogue of the [128 x WN] tile at (m0, n0): a warp covers 128 consecutive columns of a row per pass (WN / 128
// column halves per row), EPI_ROWS rows' loads in flight per warp.  Columns at or beyond n_valid_end are never passed on.
// The accumulators are in shared memory by now, so the registers are free for the loads.  The reverse, tangent and
// backward epilogues read one or two activation-sized tensors: with 8 rows per warp (half of its 16 rows per column
// half) those reads keep HBM busy, where 2 rows left it waiting.  The others read at most a bias and mostly store; they
// keep 2 rows, which measured faster for them.
template <class Epi> constexpr int epi_rows_in_flight() { return epi_family<Epi>::value == FAM_TC_OTHER ? 2 : 8; }
template <int WN, class Epi>
__device__ __forceinline__ void tile_epilogue(const float* acc_s, int64_t m0, int64_t M, int n0, int n_valid_end, const Epi& epi, int tid) {
  constexpr int LD = acc_ld(WN);
  constexpr int EPI_ROWS = epi_rows_in_flight<Epi>();
  const int cq = tid & 31;
#pragma unroll 1
  for (int h = 0; h < WN / 128; ++h) {
    const int cl = 128 * h + 4 * cq;
    const int col = n0 + cl;
    int nv = n_valid_end - col;
    nv = nv < 4 ? nv : 4;
    if (nv <= 0) break;
    for (int r0 = tid >> 5; r0 < BM; r0 += EPI_ROWS * (THREADS / 32)) {
      typename Epi::Aux aux[EPI_ROWS];
#pragma unroll
      for (int i = 0; i < EPI_ROWS; ++i) {
        const int64_t row = m0 + r0 + i * (THREADS / 32);
        if (row < M) epi.load(row, col, nv, aux[i]);
      }
#pragma unroll
      for (int i = 0; i < EPI_ROWS; ++i) {
        const int r = r0 + i * (THREADS / 32);
        const int64_t row = m0 + r;
        if (row < M) {
          const float4 t = *reinterpret_cast<const float4*>(acc_s + r * LD + cl);
          const float x[4] = {t.x, t.y, t.z, t.w};
          epi.apply(row, col, x, nv, aux[i]);
        }
      }
    }
  }
}

// splits this thread's 8 float4 of a [128 x 64] fp32 slice into hi / lo bf16 planes and writes them into the K-major SW128
// stage (16 KB per plane); thread t holds rows 16 pass + t / 16, columns 4 (t % 16) .. + 3
__device__ __forceinline__ void store_a(const float4 (&v)[BM * 16 / THREADS], uint8_t* sa, int tid) {
  const int c = tid & 15;
  const int rsub = tid >> 4;
#pragma unroll
  for (int pass = 0; pass < BM * 16 / THREADS; ++pass) {
    const float x[4] = {v[pass].x, v[pass].y, v[pass].z, v[pass].w};
    uint2 pl[2];
    split4<2>(x, pl);
    const uint32_t off = sw128((uint32_t)(pass * (THREADS / 16) + rsub), (uint32_t)(c * 4));
#pragma unroll
    for (int p = 0; p < 2; ++p) *reinterpret_cast<uint2*>(sa + p * A_HALF_BYTES + off) = pl[p];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// 2-plane layers: C[M x N] = epi( A[M x K] * B^T ),  B given as a pre-split 2-plane weight image, WN output columns per CTA.
// 1-D grid of ceil(M/128) * ceil(N/WN) CTAs with the column tile fastest: the column tiles of a row block run back to
// back, so that a second read of its activations hits L2.  Weight rows beyond the image tile (N = 217 -> 224 rows) leave
// stale shared memory in the last rows of the slice; they only feed columns >= N, which the epilogue never passes on.
// Weight slices arrive by cp.async.bulk into two stages on mbarriers.  The activations reach shared memory as they lie in
// HBM: one thread issues a 2-D TMA copy per 64-wide K slice (a [128 rows x 64 k] fp32 box, 32 KB; rows past M and
// columns past K arrive as zeros, padding columns of the row stride are never read) into a w_ring(WN)-deep ring of slots
// on mbarriers, all of them before the main loop.  While the wgmma group of slice ks runs, all threads split slice ks + 1
// in place: each reads its 8 float4 (store_a's mapping: a warp reads 512 contiguous bytes), a CTA barrier, then the
// hi / lo K-major SW128 planes go over the same 32 KB.  A slot is refilled as soon as the barrier after the wgmma group
// that read it has passed.  With K = 0 no copy is issued and the epilogue sees zero accumulators.
// ---------------------------------------------------------------------------------------------------------------
template <int WN, class Epi>
__global__ void __launch_bounds__(THREADS, 1)
gemm_w_kernel(int64_t M, int N, int K, const uint16_t* __restrict__ img, Epi epi, const __grid_constant__ CUtensorMap amap) {
  static_assert(WN == 128 || WN == 256, "a 128- or 256-column weight slice");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  const int tid = threadIdx.x, wg = tid >> 7;
  const int n_ct = (N + WN - 1) / WN;
  const int n0 = (int)(blockIdx.x % (unsigned)n_ct) * WN;
  const int64_t m0 = (int64_t)(blockIdx.x / (unsigned)n_ct) * BM;
  const int t = n0 / nt_of(2);                              // image tile of this CTA's columns
  const int rows_t = tile_rows(N, t, 2);
  const int row_in_tile = n0 - t * nt_of(2);
  int rows_h = rows_t - row_in_tile; rows_h = rows_h < WN ? rows_h : WN;   // weight rows of this CTA (multiple of 16)
  const int n_slices = pad64(K) / 64;
  constexpr uint32_t B_PLANE = b_plane_bytes(WN);
  const uint16_t* img_t = img + tile_offset(N, K, t, 2) + (int64_t)row_in_tile * 64;
  constexpr int NACC = WN / 2;
  float acc[NACC];
#pragma unroll
  for (int q = 0; q < NACC; ++q) acc[q] = 0.f;

  // [w_ring(WN) activation slots][2 weight stages of 2 planes][a barrier per slot][a barrier per weight stage]
  constexpr int NR = w_ring(WN);
  constexpr uint32_t W_STAGE = 2 * B_PLANE;
  uint8_t* wst = smem + NR * W_SLOT;
  uint64_t* afull = reinterpret_cast<uint64_t*>(wst + 2 * W_STAGE);
  uint64_t* wfull = afull + NR;
  auto issue_a = [&](int i) {                               // one thread: activation slice i into slot i % NR
    const int r = i % NR;
    mbar_arrive_expect_tx(&afull[r], W_SLOT);
    tma_load_2d(smem + r * W_SLOT, &amap, i * BK, (int)m0, &afull[r]);
  };
  auto issue_w = [&](int ks) {                              // one thread: weight slice ks into stage ks & 1
    uint8_t* st = wst + (ks & 1) * W_STAGE;
    const uint32_t wb = (uint32_t)rows_h * 128u;
    mbar_arrive_expect_tx(&wfull[ks & 1], 2 * wb);
    for (int p = 0; p < 2; ++p) bulk_g2s(st + p * B_PLANE, img_t + ((int64_t)ks * 2 + p) * rows_t * 64, wb, &wfull[ks & 1]);
  };
  auto split = [&](int i) {                                 // slice i, once landed, into hi / lo planes over its slot
    uint8_t* slot = smem + (i % NR) * W_SLOT;
    mbar_wait(&afull[i % NR], (uint32_t)((i / NR) & 1));
    float4 v[BM * 16 / THREADS];
    const float4* f = reinterpret_cast<const float4*>(slot) + (tid >> 4) * (BK / 4) + (tid & 15);
#pragma unroll
    for (int pass = 0; pass < BM * 16 / THREADS; ++pass) v[pass] = f[pass * (THREADS / 16) * (BK / 4)];
    __syncthreads();                                        // every read of the slot before the first plane store
    store_a(v, slot, tid);
  };
  if (tid == 0) {
    for (int r = 0; r < NR; ++r) mbar_init(&afull[r], 1);
    mbar_init(&wfull[0], 1);
    mbar_init(&wfull[1], 1);
    fence_barrier_init();
    if (n_slices > 0) issue_w(0);
    for (int i = 0; i < NR && i < n_slices; ++i) issue_a(i);
  }
  __syncthreads();
  if (n_slices > 0) {
    split(0);
    fence_proxy_async();
  }
  __syncthreads();
  for (int ks = 0; ks < n_slices; ++ks) {
    const int s = ks & 1;
    if (tid == 0 && ks + 1 < n_slices) issue_w(ks + 1);     // stage s ^ 1 was released by the wait + barrier of ks - 1
    mbar_wait(&wfull[s], (uint32_t)((ks >> 1) & 1));
    const uint32_t sa = smem_u32(smem + (ks % NR) * W_SLOT), sb = smem_u32(wst + s * W_STAGE);
    wg_fence();
    mma_slice<2, WN>(acc, sa + wg * (64 * 128), A_HALF_BYTES, sb, B_PLANE, ks == 0);
    wg_commit();
    if (ks + 1 < n_slices) split(ks + 1);
    wg_wait_all();
    fence_proxy_async();
    __syncthreads();
    if (tid == 0 && ks + NR < n_slices) issue_a(ks + NR);  // slot ks % NR: the group that read it has completed
  }
  float* acc_s = reinterpret_cast<float*>(smem);              // the slots and stages are free by now: every copy has landed
  acc_to_smem<WN>(acc, acc_s, wg, tid & 127);
  __syncthreads();
  tile_epilogue<WN>(acc_s, m0, M, n0, N, epi, tid);
}

// ---------------------------------------------------------------------------------------------------------------
// 3-plane layers: C[M x N] = epi( A[M x K] * B^T ), B given as a pre-split 3-plane weight image, K > 0.  Persistent:
// min(tiles, SMs) CTAs take the [128 x 128] tiles t = blockIdx.x + i * gridDim.x (column tile fastest, so the two column
// tiles of a row block run at the same time and the second read of its activations hits L2).  Three warpgroups and no
// CTA barrier after the set-up:
// * Producer (warpgroup 0, 40 registers).  One thread issues the 2-D TMA copies of each 64-wide K slice as four
//   [32 rows x 64 k] fp32 boxes into four landing quarters, each on its own mbarrier (rows past M and columns past K
//   arrive as zeros; a quarter that starts past M is not copied and splits as zeros), and the weight slice's three
//   plane copies into the stage.  The warpgroup splits each landed quarter with split4<3> in store_a's mapping into the
//   stage's K-major SWIZZLE_128B planes; once every thread has split its part of a quarter (an async proxy fence and a
//   warpgroup barrier), the quarter is refilled with the next slice's rows, which may belong to the CTA's next tile.
//   After the fourth quarter: an arrival on the stage's "full" barrier (128 arrivals plus the weight bytes).
// * Two consumers (warpgroups 1 and 2, 232 registers), each owning 64 rows of the tile.  Per slice: wait "full", issue
//   mma_slice<3> (the five correction products into an accumulator zeroed at the slice) and the four hi * hi steps
//   into fresh registers, add corrections, hh0 .. hh3 into tot in that order, and arrive on the stage's "empty"
//   barrier (256 arrivals) once the last group has completed.  The tensor core truncates a wgmma result toward zero;
//   every hi * hi result is a single truncation of 16 full-size products, so adding half an ulp of it (with its sign)
//   leaves an unbiased error.  Without that the bias of the 16 truncations per output (K = 256) adds up coherently over
//   the points of a parameter-gradient sum.  The consumers drift apart: one's adds overlap the other's products.  After the tile's last slice each consumer applies the epilogue functor to its own 64 rows straight
//   from the fragment: lane pairs swap one float2 so that each thread holds 4 consecutive columns of one row.
// Weight rows past the image tile (N = 217 -> 224 rows) and stage contents left by an earlier slice or tile reach only
// accumulator columns >= N, which are never passed to the epilogue.
// ---------------------------------------------------------------------------------------------------------------
constexpr int W3_THREADS = 384;
constexpr int W3_QROWS = 32;                                   // rows of one landing quarter
constexpr uint32_t W3_QUARTER = W3_QROWS * BK * 4;             // 8 KB
constexpr int W3_NQ = BM / W3_QROWS;
constexpr uint32_t W3_A_STAGE = 3 * A_HALF_BYTES;              // 48 KB: hi, mid, lo planes of a [128 x 64] slice
constexpr uint32_t W3_STAGE = W3_A_STAGE + 3 * b_plane_bytes(BN);   // + the weight slice's three planes: 96 KB
constexpr uint32_t W3_LAND = W3_NQ * W3_QUARTER;               // 32 KB: one fp32 slice
constexpr int W3_PRODUCER_REGS = 40, W3_CONSUMER_REGS = 232;
static_assert(W3_LAND == W_SLOT, "the landing quarters hold one fp32 slice");
static_assert(W3_PRODUCER_REGS + 2 * W3_CONSUMER_REGS <= 65536 / 128, "register file of one SM");
static_assert(BM * 16 / 128 / W3_NQ == 4, "four float4 per producer thread and quarter");

template <class Epi>
__global__ void __launch_bounds__(W3_THREADS, 1)
gemm_w3_tma_kernel(const float* __restrict__ A, int64_t M, int N, int K, const uint16_t* __restrict__ img, Epi epi,
                   const __grid_constant__ CUtensorMap amap) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* land = smem + 2 * W3_STAGE;
  uint64_t* full = reinterpret_cast<uint64_t*>(land + W3_LAND);
  uint64_t* empty = full + 2;
  uint64_t* landed = empty + 2;
  const int tid = threadIdx.x, wg = tid >> 7;
  const int n_ct = (N + BN - 1) / BN;
  const int tiles = (int)((M + BM - 1) / BM) * n_ct;
  const int n_slices = pad64(K) / 64;
  constexpr uint32_t B_PLANE = b_plane_bytes(BN);
  if (tid == 0) {
    mbar_init(&full[0], 129);
    mbar_init(&full[1], 129);
    mbar_init(&empty[0], 256);
    mbar_init(&empty[1], 256);
    for (int q = 0; q < W3_NQ; ++q) mbar_init(&landed[q], 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<W3_PRODUCER_REGS>();
    auto issue_quarter = [&](int t, int ks, int q) {         // one thread: rows 32q.. of slice ks of tile t
      const int64_t r0 = (int64_t)(t / n_ct) * BM + q * W3_QROWS;
      if (r0 < M) {
        mbar_arrive_expect_tx(&landed[q], W3_QUARTER);
        tma_load_2d(land + q * W3_QUARTER, &amap, ks * BK, (int)r0, &landed[q]);
      } else {
        mbar_arrive(&landed[q]);
      }
    };
    if (tid == 0 && (int)blockIdx.x < tiles)
      for (int q = 0; q < W3_NQ; ++q) issue_quarter(blockIdx.x, 0, q);
    const int c = tid & 15, rsub = tid >> 4;                  // store_a's mapping for 128 threads
    uint32_t g = 0;                                           // slices of this CTA so far
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
      const int64_t m0 = (int64_t)(t / n_ct) * BM;
      const int tn = t % n_ct;                                // image tile = column tile (3 planes: 128 rows)
      const int rows_t = tile_rows(N, tn, 3);
      const uint16_t* img_t = img + tile_offset(N, K, tn, 3);
      for (int ks = 0; ks < n_slices; ++ks, ++g) {
        int t1 = t, ks1 = ks + 1;                             // the slice after this one
        if (ks1 == n_slices) { ks1 = 0; t1 += gridDim.x; }
        const int s = g & 1;
        uint8_t* st = smem + s * W3_STAGE;
        mbar_wait(&empty[s], ((g >> 1) & 1) ^ 1);
        if (tid == 0) {
          const uint32_t wb = (uint32_t)rows_t * 128u;
          mbar_arrive_expect_tx(&full[s], 3 * wb);
          for (int p = 0; p < 3; ++p) bulk_g2s(st + W3_A_STAGE + p * B_PLANE, img_t + ((int64_t)ks * 3 + p) * rows_t * 64, wb, &full[s]);
        }
#pragma unroll 1
        for (int q = 0; q < W3_NQ; ++q) {
          float4 v[4];
          if (m0 + q * W3_QROWS < M) {
            mbar_wait(&landed[q], g & 1);
            const float4* f = reinterpret_cast<const float4*>(land + q * W3_QUARTER) + rsub * (BK / 4) + c;
#pragma unroll
            for (int pass = 0; pass < 4; ++pass) v[pass] = f[pass * 8 * (BK / 4)];
          } else {
#pragma unroll
            for (int pass = 0; pass < 4; ++pass) v[pass] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
#pragma unroll
          for (int pass = 0; pass < 4; ++pass) {
            const float x[4] = {v[pass].x, v[pass].y, v[pass].z, v[pass].w};
            uint2 pl[3];
            split4<3>(x, pl);
            const uint32_t off = sw128((uint32_t)(q * W3_QROWS + pass * 8 + rsub), (uint32_t)(c * 4));
#pragma unroll
            for (int p = 0; p < 3; ++p) *reinterpret_cast<uint2*>(st + p * A_HALF_BYTES + off) = pl[p];
          }
          // The refill is an async-proxy write over the quarter: every thread's reads of it must have returned (their
          // values are split and stored by now) and be ordered before it.  A barrier alone does not wait for loads in
          // flight, and refilling right after it let the TMA overwrite rows that were still being read.
          fence_proxy_async();
          wg_bar_sync();
          if (tid == 0 && t1 < tiles) issue_quarter(t1, ks1, q);
        }
        fence_proxy_async();
        mbar_arrive(&full[s]);
      }
    }
  } else {
    reg_alloc<W3_CONSUMER_REGS>();
    const int cw = wg - 1, wtid = tid & 127, lane = tid & 31;
    float acc[64], acc2[64], tot[64];
    auto hi_hi = [&](float (&d)[64], uint32_t a, uint32_t b, int j) {
      wg_fence();
      wgmma_128_fresh(d, make_desc(a + 32u * j), make_desc(b + 32u * j));
      wg_commit();
    };
    auto add_unbiased = [&](float (&d)[64]) {                 // after the wait that completes d
      fence_operand(d);
#pragma unroll
      for (int q = 0; q < 64; ++q) tot[q] += unbias_rz(d[q]);
    };
    uint32_t g = 0;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
      const int64_t m0 = (int64_t)(t / n_ct) * BM;
      const int n0 = (t % n_ct) * BN;
#pragma unroll
      for (int q = 0; q < 64; ++q) tot[q] = 0.f;
      for (int ks = 0; ks < n_slices; ++ks, ++g) {
        const int s = g & 1;
        mbar_wait(&full[s], (g >> 1) & 1);
        const uint32_t a = smem_u32(smem + s * W3_STAGE) + cw * (64 * 128), b = smem_u32(smem + s * W3_STAGE + W3_A_STAGE);
        wg_fence();
        mma_slice<3, BN>(acc, a, A_HALF_BYTES, b, B_PLANE, true);
        wg_commit();
        hi_hi(acc2, a, b, 0);
        wg_wait_but_one();
        fence_operand(acc);
#pragma unroll
        for (int q = 0; q < 64; ++q) tot[q] += acc[q];          // corrections
        hi_hi(acc, a, b, 1);
        wg_wait_but_one();
        add_unbiased(acc2);                                     // hh0
        hi_hi(acc2, a, b, 2);
        wg_wait_but_one();
        add_unbiased(acc);                                      // hh1
        hi_hi(acc, a, b, 3);
        wg_wait_but_one();
        add_unbiased(acc2);                                     // hh2
        wg_wait_all();
        mbar_arrive(&empty[s]);                                 // every group that read stage s has completed
        add_unbiased(acc);                                      // hh3
      }
      // fragment rows r, r + 8, columns 8j + 2(lane & 3) + {0, 1}: the even lane of a pair takes row r, the odd one row
      // r + 8, of the pair's 4 columns 8j + 4((lane & 3) >> 1) + {0 .. 3}
      const bool odd = lane & 1;
      const int64_t row = m0 + 64 * cw + 16 * (wtid >> 5) + (lane >> 2) + (odd ? 8 : 0);
      const int cbase = n0 + 4 * ((lane & 3) >> 1);
      // column groups whose epilogue loads are in flight together: as many as the registers of the free accumulators hold
      constexpr int EPI_G = sizeof(typename Epi::Aux) <= 4 * sizeof(float) ? 8 : 4;
#pragma unroll
      for (int j0 = 0; j0 < 16; j0 += EPI_G) {
        typename Epi::Aux aux[EPI_G];
#pragma unroll
        for (int i = 0; i < EPI_G; ++i) {
          const int col = cbase + 8 * (j0 + i);
          if (row < M && col < N) epi.load(row, col, N - col < 4 ? N - col : 4, aux[i]);
        }
#pragma unroll
        for (int i = 0; i < EPI_G; ++i) {
          const int j = j0 + i, col = cbase + 8 * j;
          const float s0 = odd ? tot[4 * j] : tot[4 * j + 2], s1 = odd ? tot[4 * j + 1] : tot[4 * j + 3];
          const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
          const float x[4] = {odd ? r0 : tot[4 * j], odd ? r1 : tot[4 * j + 1], odd ? tot[4 * j + 2] : r0, odd ? tot[4 * j + 3] : r1};
          if (row < M && col < N) epi.apply(row, col, x, N - col < 4 ? N - col : 4, aux[i]);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// C[M x N] += A[K x M]^T B[K x N]  (weight gradients; contraction over points, split over gridDim.z), row-major operands.
// grid = (ceil(M/128), ceil(N/128), splits).  Epi is the caller's epilogue with one split, EpiSplitStore into the split-K
// workspace with several.  colsum (optional): colsum[m] += sum_k A[k, m], the bias gradient, from the fp32 values the A
// split reads anyway; one writer per column and split (cs_ws: [split][M], or the output itself with one split).  Each
// column's sum has a fixed order: per k-quarter partials (points 8q + 2kq, 8q + 2kq + 1 of each 64 points, pairs added
// first, in point order), then (q0 + q1) + (q2 + q3).
//
// The operands reach shared memory as they lie in HBM, and three warpgroups share the work with no CTA barrier in the
// main loop:
// * Producer (warpgroup 0, TN_PRODUCER_REGS registers).  One thread issues a 2-D TMA copy per operand and slice (a
//   [TN_PS points x 128 columns] fp32 box, 16 KB; columns past M / N and points past K arrive as zeros) into a
//   TN_LAND-deep landing ring on one mbarrier per stage.  Once the consumers have released a plane stage ("empty"), the
//   warpgroup splits the next landed slice into it as MN-major hi / lo planes: warp w takes k-quarter w of each 8 points
//   of A, then of B, lane l columns 4l..4l+3; points past the chunk end (the next chunk's) are split as zeros.  Each
//   thread fences its plane stores for the async proxy and arrives on the stage's "full" barrier (128 arrivals).  The
//   landing stage is refilled with slice i + TN_LAND only after a warpgroup barrier: the refill is an async-proxy write
//   over it, and every thread's reads of it must have returned first (a barrier after the fence; see gemm_w3_tma_kernel).
// * Two consumers (warpgroups 1 and 2, 64 rows of the tile each).  Per slice: wait "full", issue mma_slice_mn (transpose
//   flags set) on one accumulator chain across the split's slices, then wait until only that group is in flight and
//   release the stage of the slice before it ("empty", 256 arrivals).
// Epilogue: one barrier over all 384 threads, after which every copy has landed and been split and every wgmma has
// completed; the consumers pass their accumulators through the landing ring to tile_epilogue, and the producer reduces
// its column-sum partials (written past the accumulator tile in the landing ring).
// ---------------------------------------------------------------------------------------------------------------
template <class Epi>
__global__ void __launch_bounds__(TN_THREADS, 1)
gemm_tn_kernel(int M, int N, int64_t K, int64_t k_chunk, Epi epi, float* __restrict__ colsum, float* __restrict__ cs_ws,
               const __grid_constant__ TnMaps maps) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
  const int m0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int64_t kb = (int64_t)blockIdx.z * k_chunk;
  const int64_t ke = (kb + k_chunk < K) ? kb + k_chunk : K;
  const bool do_csum = colsum != nullptr && blockIdx.y == 0;
  if (ke <= kb) return;
  uint8_t* land = smem;
  uint8_t* planes = smem + TN_LAND * TN_F32_STAGE;
  float* acc_s = reinterpret_cast<float*>(land);                               // after the main loop
  float* cs_part = acc_s + BM * acc_ld(BN);                                    // [4 k-quarters][128 columns]
  uint64_t* landed = reinterpret_cast<uint64_t*>(planes + TN_STAGES * TN_PLANE_STAGE);
  uint64_t* full = landed + TN_LAND;
  uint64_t* empty = full + TN_STAGES;
  const int n_sl = (int)((ke - kb + TN_PS - 1) / TN_PS);

  auto issue = [&](int i) {                               // one thread: slice i into landing stage i % TN_LAND
    const int r = i % TN_LAND;
    const int k0 = (int)(kb + (int64_t)i * TN_PS);
    uint8_t* st = land + r * TN_F32_STAGE;
    mbar_arrive_expect_tx(&landed[r], TN_F32_STAGE);
    tma_load_2d(st, &maps.a, m0, k0, &landed[r]);
    tma_load_2d(st + TN_F32_OPND, &maps.b, n0, k0, &landed[r]);
  };
  if (tid == 0) {
    for (int r = 0; r < TN_LAND; ++r) mbar_init(&landed[r], 1);
    for (int s = 0; s < TN_STAGES; ++s) {
      mbar_init(&full[s], 128);
      mbar_init(&empty[s], 256);
    }
    fence_barrier_init();
    for (int i = 0; i < TN_LAND && i < n_sl; ++i) issue(i);
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<TN_PRODUCER_REGS>();
    const int kq = tid >> 5;
    float csum[4] = {0.f, 0.f, 0.f, 0.f};
    for (int i = 0; i < n_sl; ++i) {
      const int r = i % TN_LAND, s = i % TN_STAGES;
      uint8_t* st = planes + s * TN_PLANE_STAGE;
      mbar_wait(&empty[s], ((i / TN_STAGES) & 1) ^ 1);
      mbar_wait(&landed[r], (i / TN_LAND) & 1);
      const int64_t left = ke - (kb + (int64_t)i * TN_PS);
      const int np = left < TN_PS ? (int)left : TN_PS;     // points of this slice inside the chunk
      const float* f = reinterpret_cast<const float*>(land + r * TN_F32_STAGE) + 4 * lane;
      // Shared-memory traffic without bank conflicts: a warp's float4 reads cover one point's 512 contiguous bytes, and
      // each half-warp's 8-byte plane stores cover all 8 16-byte chunks of one 128-byte swizzled row (64 columns of one
      // point), i.e. all 32 banks once.  All 16 reads of a thread are in flight together: the wgmma operand fetches keep
      // shared memory busy, and with fewer reads in flight the split, not the tensor core, set the pace.
      float4 v[2][TN_PS / 8][2];
#pragma unroll
      for (int opnd = 0; opnd < 2; ++opnd)
#pragma unroll
        for (int q = 0; q < TN_PS / 8; ++q)
#pragma unroll
          for (int kk = 0; kk < 2; ++kk) {
            const int p = 8 * q + 2 * kq + kk;
            v[opnd][q][kk] = p < np ? *reinterpret_cast<const float4*>(f + opnd * (TN_F32_OPND / 4) + p * BM) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
      if (do_csum)
#pragma unroll
        for (int q = 0; q < TN_PS / 8; ++q) {
          csum[0] += v[0][q][0].x + v[0][q][1].x; csum[1] += v[0][q][0].y + v[0][q][1].y;
          csum[2] += v[0][q][0].z + v[0][q][1].z; csum[3] += v[0][q][0].w + v[0][q][1].w;
        }
#pragma unroll
      for (int opnd = 0; opnd < 2; ++opnd)
#pragma unroll
        for (int q = 0; q < TN_PS / 8; ++q)
#pragma unroll
          for (int kk = 0; kk < 2; ++kk) {
            const float x[4] = {v[opnd][q][kk].x, v[opnd][q][kk].y, v[opnd][q][kk].z, v[opnd][q][kk].w};
            uint2 pl[2];
            split4<2>(x, pl);
            const uint32_t off = sw128_mn(4u * lane, (uint32_t)(8 * q + 2 * kq + kk));
            *reinterpret_cast<uint2*>(st + opnd * 2 * TN_PLANE + off) = pl[0];
            *reinterpret_cast<uint2*>(st + opnd * 2 * TN_PLANE + TN_PLANE + off) = pl[1];
          }
      fence_proxy_async();
      mbar_arrive(&full[s]);
      wg_bar_sync();                                      // every read of landing stage r has returned
      if (tid == 0 && i + TN_LAND < n_sl) issue(i + TN_LAND);
    }
    if (do_csum)                                          // the landing ring is free: the last barrier above passed
#pragma unroll
      for (int j = 0; j < 4; ++j) cs_part[kq * BM + 4 * lane + j] = csum[j];
    __syncthreads();
    if (do_csum && m0 + tid < M) {
      const float c = (cs_part[tid] + cs_part[BM + tid]) + (cs_part[2 * BM + tid] + cs_part[3 * BM + tid]);
      if (cs_ws != nullptr) cs_ws[(int64_t)blockIdx.z * M + m0 + tid] = c;
      else colsum[m0 + tid] += c;
    }
  } else {
    reg_alloc<TN_CONSUMER_REGS>();
    const int cw = wg - 1;
    float acc[64];
#pragma unroll
    for (int q = 0; q < 64; ++q) acc[q] = 0.f;
    for (int i = 0; i < n_sl; ++i) {
      const int s = i % TN_STAGES;
      mbar_wait(&full[s], (i / TN_STAGES) & 1);
      const uint32_t st = smem_u32(planes + s * TN_PLANE_STAGE);
      wg_fence();
      mma_slice_mn(acc, st + cw * 4096u, st + 2 * TN_PLANE, i == 0);
      wg_commit();
      wg_wait_but_one();
      if (i > 0) mbar_arrive(&empty[(i - 1) % TN_STAGES]);   // the group that read slice i - 1 has completed
    }
    wg_wait_all();
    fence_operand(acc);
    __syncthreads();                                      // the producer is done with the landing ring
    acc_to_smem<BN>(acc, acc_s, cw, tid & 127);
    tn_consumer_bar_sync();
    tile_epilogue<BN>(acc_s, m0, M, n0, N, epi, tid - 128);
  }
}

static inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}


// 2-D tensor map of a row-major fp32 operand [rows x cols] (row stride ld floats, a multiple of 4) in [box_rows x box_cols]
// boxes; boxes reaching past the extent arrive zero-filled there
static inline int tensor_map_2d(CUtensorMap* map, const float* X, int64_t ld, int64_t cols, int64_t rows, int box_cols, int box_rows) {
  static PFN_cuTensorMapEncodeTiled encode = nullptr;
  if (encode == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess ||
        fn == nullptr) {
      nudf::set_error("cuTensorMapEncodeTiled is not available from the driver");
      return -2;
    }
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled>(fn);
  }
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  const cuuint32_t elem[2] = {1, 1};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(X), dims, strides, box, elem,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    nudf::set_error("cuTensorMapEncodeTiled failed (%d)", (int)r);
    return -2;
  }
  return 0;
}
// An activation operand of the tensor-core kernels is read through a 2-D tensor map, which needs a row stride of whole
// 16-byte units and a 16-byte-aligned base.  The networks' layouts guarantee both (udf_net.cu, mlp_nets.cu); the
// stand-alone entry points repack an operand that lacks them (gemm_tc.cu).
static inline bool tma_operand_ok(const float* X, int64_t ld) { return (ld & 3) == 0 && aligned16(X); }
static inline int check_tma_operand(const float* X, int64_t ld) {
  if (tma_operand_ok(X, ld)) return 0;
  nudf::set_error("tensor-core operand at %p with row stride %lld floats: needs a stride of a multiple of 4 floats and a "
                  "16-byte-aligned base", (const void*)X, (long long)ld);
  return -1;
}

// gemm_w_kernel: w_ring(wn) fp32 slots, 2 weight stages of 2 planes, a barrier per slot and per stage; the accumulator
// tile reuses the slots and stages
constexpr size_t w_ring_operand_bytes(int wn) { return (size_t)w_ring(wn) * W_SLOT + 2 * 2 * (size_t)b_plane_bytes(wn); }
constexpr size_t w_ring_smem_bytes(int wn) { return w_ring_operand_bytes(wn) + (w_ring(wn) + 2) * sizeof(uint64_t) + 1024; }
static_assert(w_ring_smem_bytes(BN) <= 227 * 1024 && w_ring_smem_bytes(2 * BN) <= 227 * 1024, "one CTA per SM");
static_assert(BM * acc_ld(BN) * sizeof(float) <= w_ring_operand_bytes(BN), "accumulator tile in the slots and stages");
static_assert(BM * acc_ld(2 * BN) * sizeof(float) <= w_ring_operand_bytes(2 * BN), "accumulator tile in the slots and stages");

template <int WN, class Epi>
static inline int gemm_w_launch(const float* A, int64_t lda, int64_t M, int N, int K, const uint16_t* img, const Epi& epi, cudaStream_t st) {
  constexpr size_t smem = w_ring_smem_bytes(WN);
  static bool attr_set = false;   // per template instantiation
  if (!attr_set) {
    NUDF_CUDA_OK(cudaFuncSetAttribute(gemm_w_kernel<WN, Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  CUtensorMap amap{};
  if (int rc = tensor_map_2d(&amap, A, lda, K > 0 ? K : 1, M, BK, BM)) return rc;   // K = 0: a map no copy reads
  const unsigned grid = (unsigned)(cdiv(M, BM) * cdiv(N, WN));
  LaunchTimer lt_(epi_family<Epi>::value, st);
  gemm_w_kernel<WN, Epi><<<grid, THREADS, smem, st>>>(M, N, K, img, epi, amap);
  NUDF_LAUNCH_OK();
  return 0;
}
// gemm_w3_tma_kernel: 2 stages of the A and weight planes, the 4 landing quarters and 8 mbarriers; the epilogue runs
// from registers, so no accumulator tile has to fit beside them
constexpr size_t W3_SMEM = 2 * (size_t)W3_STAGE + W3_LAND + 8 * sizeof(uint64_t) + 1024;
static_assert(W3_SMEM <= 227 * 1024, "one CTA per SM");

template <class Epi>
static inline int gemm_w3_tma_launch(const float* A, int64_t lda, int64_t M, int N, int K, const uint16_t* img, const Epi& epi, cudaStream_t st) {
  static bool attr_set = false;   // per template instantiation
  if (!attr_set) {
    NUDF_CUDA_OK(cudaFuncSetAttribute(gemm_w3_tma_kernel<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)W3_SMEM));
    attr_set = true;
  }
  CUtensorMap amap{};
  if (int rc = tensor_map_2d(&amap, A, lda, K, M, BK, W3_QROWS)) return rc;
  const int64_t tiles = cdiv(M, BM) * cdiv(N, BN);
  const unsigned grid = (unsigned)(tiles < sm_count() ? tiles : sm_count());
  LaunchTimer lt_(epi_family<Epi>::value, st);
  gemm_w3_tma_kernel<Epi><<<grid, W3_THREADS, W3_SMEM, st>>>(A, M, N, K, img, epi, amap);
  NUDF_LAUNCH_OK();
  return 0;
}
// 2-plane layers run gemm_w_kernel, 256 columns per CTA when wider than 128 (one read and split of each activation row
// block instead of two), 128 otherwise; 3-plane layers run gemm_w3_tma_kernel, which needs K > 0.
template <int NP, class Epi>
static inline int gemm_w(const float* A, int64_t lda, int64_t M, int N, int K, const uint16_t* img, const Epi& epi, cudaStream_t st) {
  if (M <= 0 || N <= 0) return 0;
  if (int rc = check_tma_operand(A, lda)) return rc;
  if constexpr (NP == 3) {
    NUDF_REQUIRE(K > 0, "3-plane layers need K > 0");
    return gemm_w3_tma_launch<Epi>(A, lda, M, N, K, img, epi, st);
  } else {
    if (N > BN) return gemm_w_launch<2 * BN, Epi>(A, lda, M, N, K, img, epi, st);
    return gemm_w_launch<BN, Epi>(A, lda, M, N, K, img, epi, st);
  }
}

// The split of a weight-gradient contraction over its points (split-K), from the shape alone: the same inputs give the
// same partition, hence the same bits, on every device.  (M tiles x N tiles x splits) fills the 132 SMs of an H100 SXM
// once, each split has at least TN_MIN_POINTS points and a whole number of BK slices, and the per-split partial tiles
// and column sums fit the split-K workspace.  Returns the points per split.
constexpr int TN_WAVE_CTAS = 132;
constexpr int64_t TN_MIN_POINTS = 512;
static inline int64_t tn_k_chunk(int M, int N, int64_t K) {
  const int64_t tiles = cdiv(M, BM) * cdiv(N, BN);
  int64_t splits = TN_WAVE_CTAS / tiles;
  if (splits > cdiv(K, TN_MIN_POINTS)) splits = cdiv(K, TN_MIN_POINTS);
  splits = ws_splits(splits < 1 ? 1 : (int)splits, (int64_t)M * N + M);
  return round_up(cdiv(K, splits), BK);
}

// the landing ring, the plane stages and an mbarrier per landing stage plus two per plane stage; the accumulator tile
// and the column-sum partials reuse the landing ring
constexpr size_t TN_SMEM = (size_t)TN_LAND * TN_F32_STAGE + (size_t)TN_STAGES * TN_PLANE_STAGE +
                           (TN_LAND + 2 * TN_STAGES) * sizeof(uint64_t) + 1024;
static_assert((BM * acc_ld(BN) + 4 * BM) * sizeof(float) <= (size_t)TN_LAND * TN_F32_STAGE, "accumulator tile and column sums in the landing ring");
static_assert(TN_SMEM <= 227 * 1024, "one CTA per SM");

template <class Epi>
static inline int gemm_tn_launch(dim3 grid, const float* A, int64_t lda, const float* B, int64_t ldb, int M, int N, int64_t K,
                                 int64_t k_chunk, const Epi& epi, float* colsum, float* cs_ws, cudaStream_t st) {
  static bool attr_set = false;   // per template instantiation
  if (!attr_set) {
    NUDF_CUDA_OK(cudaFuncSetAttribute(gemm_tn_kernel<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TN_SMEM));
    attr_set = true;
  }
  TnMaps maps{};
  if (int rc = tensor_map_2d(&maps.a, A, lda, M, K, BM, TN_PS)) return rc;
  if (int rc = tensor_map_2d(&maps.b, B, ldb, N, K, BN, TN_PS)) return rc;
  gemm_tn_kernel<Epi><<<grid, TN_THREADS, TN_SMEM, st>>>(M, N, K, k_chunk, epi, colsum, cs_ws, maps);
  NUDF_LAUNCH_OK();
  return 0;
}
// C[M x N] += A[K x M]^T B[K x N] over row-major operands; colsum_a (optional) += the column sums of A
template <class Epi>
static inline int gemm_tn(const float* A, int64_t lda, const float* B, int64_t ldb, int M, int N, int64_t K, const Epi& epi,
                          cudaStream_t st, float* colsum_a = nullptr) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if (int rc = check_tma_operand(A, lda)) return rc;
  if (int rc = check_tma_operand(B, ldb)) return rc;
  const int64_t k_chunk = tn_k_chunk(M, N, K);
  const int splits = (int)cdiv(K, k_chunk);
  dim3 grid((unsigned)cdiv(M, BM), (unsigned)cdiv(N, BN), (unsigned)splits);
  LaunchTimer lt_(FAM_TC_WGRAD, st);
  if (splits == 1) return gemm_tn_launch(grid, A, lda, B, ldb, M, N, K, k_chunk, epi, colsum_a, nullptr, st);
  // deterministic split-K (gemm_simt.cuh): partial tiles and column sums go to the workspace, summed in split order
  float* ws = split_workspace(st);
  if (ws == nullptr) return -2;
  float* cs = ws + (int64_t)splits * M * N;
  const EpiSplitStore e{ws, (int64_t)M * N, N};
  if (int rc = gemm_tn_launch(grid, A, lda, B, ldb, M, N, K, k_chunk, e, colsum_a, cs, st)) return rc;
  if (int rc = splitk_reduce(ws, splits, M, N, epi, st)) return rc;
  return colsum_a != nullptr ? vec_reduce(cs, splits, M, colsum_a, st) : 0;
}

// several weight images in one launch: grid.y = job
struct PrepWJob { const float* W; uint16_t* img; int ldw, N, K, transposed, np; };
struct PrepWJobs { int n; PrepWJob j[64]; };
static __global__ void tc_prep_weights_jobs_kernel(const __grid_constant__ PrepWJobs jobs) {
  const PrepWJob& J = jobs.j[blockIdx.y];
  tc_prep_weights_body(J.W, J.ldw, J.N, J.K, J.transposed, J.np, J.img, (int64_t)blockIdx.x * blockDim.x + threadIdx.x,
                       (int64_t)gridDim.x * blockDim.x);
}
static inline int prep_weights_jobs(const PrepWJobs& jobs, cudaStream_t st) {
  if (jobs.n <= 0) return 0;
  int64_t mx = 0;
  for (int i = 0; i < jobs.n; ++i) {
    int64_t total = 0;
    for (int t = 0; t < n_tiles(jobs.j[i].N, jobs.j[i].np); ++t) total += (int64_t)tile_rows(jobs.j[i].N, t, jobs.j[i].np) * pad64(jobs.j[i].K);
    mx = total > mx ? total : mx;
  }
  int blocks = (int)((mx + 255) / 256);
  if (blocks > 1024) blocks = 1024;
  tc_prep_weights_jobs_kernel<<<dim3((unsigned)blocks, (unsigned)jobs.n), 256, 0, st>>>(jobs);
  NUDF_LAUNCH_OK();
  return 0;
}

static inline int prep_weights(const float* W, int64_t ldw, int N, int K, int transposed, int np, uint16_t* img, cudaStream_t st) {
  int64_t total = 0;
  for (int t = 0; t < n_tiles(N, np); ++t) total += (int64_t)tile_rows(N, t, np) * pad64(K);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  tc_prep_weights_kernel<<<blocks, 256, 0, st>>>(W, ldw, N, K, transposed, np, img);
  NUDF_LAUNCH_OK();
  return 0;
}

}  // namespace tc
}  // namespace nudf
