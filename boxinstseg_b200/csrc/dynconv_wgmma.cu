// a2 / a3 / a4: dense dynamic 1x1 convolution  out[b,i,p] = sum_c kernel[b,i,c] * feat[b,c,p]
// (K = C = 256 channels) as a TMA-fed Hopper wgmma kernel, TF32 inputs, FP32 accumulation in registers.
// Replaces the F.conv2d / einsum calls at
//   mmdet/models/dense_heads/box_solov2_head.py:209-211   (all S^2 cells, groups=B)
//   mmdet/models/dense_heads/discobox_head.py:1219        (positive kernels of one image)
//   mmdet/models/dense_heads/box2mask_head.py:345         (einsum 'bqc,bchw->bqhw')
// which run as cuDNN/cuBLAS GEMMs (cuDNN convolutions use TF32 by default on Ampere and later).
//
// GEMM view per image:  D[M = pixels, N = kernels] = A[M, K] * B[N, K]^T
//   A = feat^T : the pixel index is contiguous in memory, an "MN-major" operand.  wgmma reads TF32 operands from
//       shared memory only K-major, so A goes through registers: TMA stages [32 channels][32 pixels] boxes with the
//       128-byte swizzle, and each warp loads its A fragments with ld.shared (rounded to TF32 with cvt.rna).
//       The accumulator rows are a permutation of the tile's pixels chosen so that these loads are free of bank
//       conflicts (see a_pixel());
//   B = kernel : K-major, [row = kernel][32 channels] boxes with the 128-byte swizzle, read by wgmma through a
//       shared-memory descriptor;
//   D          : 64 pixels x BN <= 128 kernels of FP32 per consumer warpgroup, in registers.
// The op is HBM bound (each feat tile is read once: 128 KB per 128 pixels; B stays resident in shared
// memory for the whole CTA lifetime), so one CTA per SM streams pixel tiles:
//   warps 0-7: two consumer warpgroups, 64 pixels of a 128-pixel tile each (ld.shared -> wgmma -> global stores)
//   warp 8   : TMA producer (B once, then a ring of 16 KB A stages)
// synchronised with mbarriers only (full/empty per stage).
#include <cuda.h>

#include <algorithm>

#include "common.cuh"

namespace bxs {
namespace {

constexpr int BLOCK_M = 128;        // pixels per tile (two warpgroups of 64)
constexpr int MAX_N = 128;          // kernels per CTA
constexpr int BLOCK_K = 32;         // channels per stage = one 128-byte swizzle row of tf32
constexpr int MMA_K = 8;            // tf32: 32 bytes per instruction
constexpr int MAX_KBLOCKS = 8;      // C <= 256
constexpr int STAGES = 5;           // 80 KB of feat in flight per SM
constexpr int BOX_BYTES = BLOCK_K * 32 * 4;               // one [32 channels][32 pixels] TMA box: 4 KB
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 4;      // 16 KB
constexpr int B_KBLOCK_BYTES = MAX_N * BLOCK_K * 4;       // 16 KB
constexpr int NUM_THREADS = 288;    // two consumer warpgroups + one TMA warp
constexpr int CONSUMER_WARPS = 8;

struct SmemLayout {
  alignas(1024) uint8_t a[STAGES][A_STAGE_BYTES];
  alignas(1024) uint8_t b[MAX_KBLOCKS][B_KBLOCK_BYTES];
  alignas(8) uint64_t full[STAGES];
  uint64_t empty[STAGES];
  uint64_t b_full;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(x), "r"(y)
      : "memory");
}

__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint64_t* bar, void* dst, int x, int y, int z) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z)
      : "memory");
}

// wgmma shared-memory matrix descriptor of a K-major operand with the 128-byte swizzle (SM90): start >> 4,
// LBO (unused by this layout) = 1, SBO = 1 KB between groups of 8 rows >> 4 << 32, layout SWIZZLE_128B (1) << 62.
// The tile base is 1024-byte aligned; the k-th group of 8 tf32 columns starts 32 * k bytes into the swizzled row.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3fff) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous wgmma / wait pair
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

// D[64 x 32] += A[64 x 8] (registers) * B[32 x 8]^T (shared memory, K-major), TF32 in, FP32 accumulate
__device__ __forceinline__ void wgmma_rs_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1));
}
// D[64 x 64] += A[64 x 8] (registers) * B[64 x 8]^T (shared memory, K-major), TF32 in, FP32 accumulate
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1));
}
// D[64 x 128] += A[64 x 8] (registers) * B[128 x 8]^T (shared memory, K-major), TF32 in, FP32 accumulate
__device__ __forceinline__ void wgmma_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1));
}
// D[64 x 32] += A[64 x 8] * B[32 x 8]^T, both in shared memory (K-major), TF32 in, FP32 accumulate
__device__ __forceinline__ void wgmma_ss_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(1));
}
// D[64 x 64] += A[64 x 8] * B[64 x 8]^T, both in shared memory (K-major), TF32 in, FP32 accumulate
__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(1));
}
// D[64 x 128] += A[64 x 8] * B[128 x 8]^T, both in shared memory (K-major), TF32 in, FP32 accumulate
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(1));
}
// D[64 x 256] += A[64 x 8] * B[256 x 8]^T, both in shared memory (K-major), TF32 in, FP32 accumulate
__device__ __forceinline__ void wgmma_ss_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(1));
}

template <int BN>
__device__ __forceinline__ void wgmma_rs(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t bdesc) {
  if constexpr (BN == 32) wgmma_rs_n32(d, a, bdesc);
  else if constexpr (BN == 64) wgmma_rs_n64(d, a, bdesc);
  else wgmma_rs_n128(d, a, bdesc);
}
template <int BN>
__device__ __forceinline__ void wgmma_ss(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc) {
  if constexpr (BN == 32) wgmma_ss_n32(d, adesc, bdesc);
  else if constexpr (BN == 64) wgmma_ss_n64(d, adesc, bdesc);
  else if constexpr (BN == 128) wgmma_ss_n128(d, adesc, bdesc);
  else wgmma_ss_n256(d, adesc, bdesc);
}

// Pixel (inside its 32-pixel box) of accumulator row `r` (0..7) of a warp, for the row group `j` (0..3).  A warp's
// 16 accumulator rows are two groups j = 2h (rows 0-7) and j = 2h + 1 (rows 8-15) of the box; row r is pixel
// 16 (r / 4) + 4 j + r % 4.  In the 128-byte swizzled box the 16-byte chunk of pixel p in channel row k sits at
// (p / 4) ^ (k % 8), so the 8 rows x 4 channels of one fragment load touch 32 distinct banks.
__device__ __forceinline__ int a_pixel(int r, int j) { return 16 * (r >> 2) + 4 * j + (r & 3); }
__device__ __forceinline__ float lds_box(const uint8_t* box, int k, int p) {
  return *reinterpret_cast<const float*>(box + k * 128 + ((((p >> 2) ^ (k & 7))) << 4) + (p & 3) * 4);
}

// grid: (ctas_per_group, B * n_chunks).  CTA (x, g): image b = g / n_chunks, kernel chunk g % n_chunks of BN kernels,
// pixel tiles x, x + gridDim.x, ...
template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
dynconv_tf32_kernel(const __grid_constant__ CUtensorMap tm_feat, const __grid_constant__ CUtensorMap tm_kern,
                    float* __restrict__ out, int C, int P, int I, int n_chunks) {
  extern __shared__ uint8_t smem_raw[];
  SmemLayout& S = *reinterpret_cast<SmemLayout*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y / n_chunks, chunk = blockIdx.y % n_chunks;
  const int kblocks = (C + BLOCK_K - 1) / BLOCK_K;       // channels beyond C are zero-filled by the 3-D tensor map
  const int tiles_m = (P + BLOCK_M - 1) / BLOCK_M;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&S.full[s], 1); mbar_init(&S.empty[s], CONSUMER_WARPS); }
    mbar_init(&S.b_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == CONSUMER_WARPS) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_expect_tx(&S.b_full, (uint32_t)kblocks * BN * BLOCK_K * 4);
      for (int kb = 0; kb < kblocks; ++kb)
        tma_load_2d(&tm_kern, &S.b_full, S.b[kb], kb * BLOCK_K, b * I + chunk * BN);
      int stage = 0, phase = 0;
      for (int mt = blockIdx.x; mt < tiles_m; mt += gridDim.x) {
        for (int kb = 0; kb < kblocks; ++kb) {
          mbar_wait(&S.empty[stage], phase ^ 1);
          mbar_expect_tx(&S.full[stage], A_STAGE_BYTES);
#pragma unroll
          for (int g = 0; g < BLOCK_M / 32; ++g)
            tma_load_3d(&tm_feat, &S.full[stage], S.a[stage] + g * BOX_BYTES, mt * BLOCK_M + g * 32, kb * BLOCK_K, b);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: ld.shared A -> wgmma -> global =====================
    const int wg = warp >> 2, w = warp & 3, r = lane >> 2, c4 = lane & 3;
    const int box = 2 * wg + (w >> 1);             // the 32-pixel box of this warp's 16 rows
    const int p0 = a_pixel(r, 2 * (w & 1)), p1 = a_pixel(r, 2 * (w & 1) + 1);
    mbar_wait(&S.b_full, 0);
    int stage = 0, phase = 0;
    for (int mt = blockIdx.x; mt < tiles_m; mt += gridDim.x) {
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&S.full[stage], phase);
        const uint8_t* abox = S.a[stage] + box * BOX_BYTES;
        uint32_t a[BLOCK_K / MMA_K][4];
#pragma unroll
        for (int k4 = 0; k4 < BLOCK_K / MMA_K; ++k4) {
          const int k = k4 * MMA_K + c4;
          a[k4][0] = to_tf32(lds_box(abox, k, p0));
          a[k4][1] = to_tf32(lds_box(abox, k, p1));
          a[k4][2] = to_tf32(lds_box(abox, k + 4, p0));
          a[k4][3] = to_tf32(lds_box(abox, k + 4, p1));
        }
        const uint32_t b_base = smem_u32(S.b[kb]);
        wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < BLOCK_K / MMA_K; ++k4) wgmma_rs<BN>(acc, a[k4], make_desc(b_base + k4 * (MMA_K * 4)));
        wgmma_commit();
        wgmma_wait_all();
        fence_acc(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&S.empty[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      // accumulator elements 4 j .. 4 j + 3: kernels n = 8 j + 2 c4 + {0, 1} of rows r (pixel p0) and r + 8 (pixel p1)
      const int pix = mt * BLOCK_M + box * 32;
      const bool in0 = pix + p0 < P, in1 = pix + p1 < P;
      float* dst = out + ((int64_t)b * I + chunk * BN + 2 * c4) * P + pix;
      int n = chunk * BN + 2 * c4;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j, n += 8, dst += 8 * (int64_t)P) {
        if (n < I) {
          if (in0) dst[p0] = acc[4 * j];
          if (in1) dst[p1] = acc[4 * j + 2];
        }
        if (n + 1 < I) {
          if (in0) dst[P + p0] = acc[4 * j + 1];
          if (in1) dst[P + p1] = acc[4 * j + 3];
        }
      }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// row-major [rows, cols] float32 matrix, box = [box_rows, 32 floats], 128-byte swizzle, zero fill out of bounds
bool make_map(CUtensorMap* map, const float* base, int64_t rows, int64_t cols, int box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 4};
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// [batch, rows, cols] float32 tensor, box = [1, box_rows, 32 floats], 128-byte swizzle: rows beyond `rows` of a batch
// entry are OUT OF BOUNDS and read as zeros (a 2-D [batch * rows, cols] view would run into the next entry instead)
bool make_map3(CUtensorMap* map, const float* base, int64_t batch, int64_t rows, int64_t cols, int box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t strides[2] = {(cuuint64_t)cols * 4, (cuuint64_t)cols * (cuuint64_t)rows * 4};
  cuuint32_t box[3] = {32, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// kT[b, c, i] = kernels[b, i, c] for i < I, 0 for I <= i < Ipad   (the K-major B operand of d/d feat = K^T . G)
__global__ void transpose_pad_kernel(const float* __restrict__ k, float* __restrict__ kt, int I, int C, int Ipad, int64_t total) {
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx % Ipad);
    const int c = (int)((idx / Ipad) % C);
    const int64_t b = idx / ((int64_t)Ipad * C);
    kt[idx] = i < I ? __ldg(k + (b * I + i) * C + c) : 0.f;
  }
}

// =====================================================================================================================
// d/d kernel:  dK[b,i,c] = sum_p g[b,i,p] * feat[b,c,p]  -- a GEMM with a LONG reduction (K = pixels, 51 200 .. 65 536) and a
// tiny output (I x C).  Both operands are K-major (the pixel index is contiguous in g and in feat), so wgmma reads both
// from shared memory with the 128-byte swizzle.  Split-K: CTA (split, b * chunks + chunk) reduces pixels [p0, p1) of
// image b for 128 rows of g (64 per consumer warpgroup) into a 128 x C register accumulator (C <= 256 columns) and
// stores it as a partial; dynconv_wgrad_reduce sums the partials in split order (deterministic).
//   warps 0-7: two consumer warpgroups (wgmma, epilogue)
//   warp 8   : TMA producer (A = g tile 128 x 32, B = feat tile C x 32 per stage, 4 stages)
// =====================================================================================================================
constexpr int WG_STAGES = 4;
constexpr int WG_A_BYTES = 128 * BLOCK_K * 4;      // 16 KB
constexpr int WG_B_BYTES = 256 * BLOCK_K * 4;      // 32 KB

struct WgSmem {
  alignas(1024) uint8_t a[WG_STAGES][WG_A_BYTES];
  alignas(1024) uint8_t b[WG_STAGES][WG_B_BYTES];
  alignas(8) uint64_t full[WG_STAGES];
  uint64_t empty[WG_STAGES];
};

// BN: C rounded up to 32, 64, 128 or 256 (the columns beyond C are computed from unused shared memory and dropped)
template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
dynconv_wgrad_kernel(const __grid_constant__ CUtensorMap tm_g, const __grid_constant__ CUtensorMap tm_feat,
                     float* __restrict__ partial, int C, int P, int I, int chunks, int splits, int kb_per_split) {
  extern __shared__ uint8_t smem_raw[];
  WgSmem& S = *reinterpret_cast<WgSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int split = blockIdx.x, b = blockIdx.y / chunks, chunk = blockIdx.y % chunks;
  const int kb_total = (P + BLOCK_K - 1) / BLOCK_K;
  const int kb0 = split * kb_per_split, kb1 = min(kb0 + kb_per_split, kb_total);
  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; ++s) { mbar_init(&S.full[s], 1); mbar_init(&S.empty[s], CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == CONSUMER_WARPS) {
    if (lane == 0) {
      int stage = 0, phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&S.empty[stage], phase ^ 1);
        mbar_expect_tx(&S.full[stage], WG_A_BYTES + (uint32_t)C * BLOCK_K * 4);
        tma_load_3d(&tm_g, &S.full[stage], S.a[stage], kb * BLOCK_K, chunk * 128, b);       // rows >= I: zeros
        tma_load_3d(&tm_feat, &S.full[stage], S.b[stage], kb * BLOCK_K, 0, b);
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    const int wg = warp >> 2, w = warp & 3, r = lane >> 2, c4 = lane & 3;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0, phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&S.full[stage], phase);
      const uint32_t a_base = smem_u32(S.a[stage]) + wg * (64 * 128), b_base = smem_u32(S.b[stage]);
      wgmma_fence();
#pragma unroll
      for (int k4 = 0; k4 < BLOCK_K / MMA_K; ++k4)
        wgmma_ss<BN>(acc, make_desc(a_base + k4 * (MMA_K * 4)), make_desc(b_base + k4 * (MMA_K * 4)));
      wgmma_commit();
      wgmma_wait_all();
      fence_acc(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&S.empty[stage]);
      if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
    }
    // accumulator elements (i, i + 1), i even: row 16 w + r (+ 8 when i % 4 == 2), columns 8 (i / 4) + 2 c4 + {0, 1}
    const int row0 = chunk * 128 + wg * 64 + w * 16 + r;
    float* dst = partial + (((int64_t)b * splits + split) * I) * C;
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int row = row0 + ((i & 2) ? 8 : 0), n = 8 * (i >> 2) + 2 * c4;
      if (row < I && n < C) *reinterpret_cast<float2*>(dst + (int64_t)row * C + n) = make_float2(acc[i], acc[i + 1]);
    }
  }
}

__global__ void dynconv_wgrad_reduce(const float* __restrict__ partial, float* __restrict__ out, int splits, int64_t per_image,
                                     int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / per_image, r = i - b * per_image;
    const float* p = partial + b * splits * per_image + r;
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += p[(int64_t)s * per_image];          // split order: deterministic
    out[i] = acc;
  }
}

// out[b, i, p] for i in [0, I): kernels `tm_kern` ([B * I, C], boxes of BN rows), features `tm_feat` ([B, C, P])
template <int BN>
int launch_forward(const CUtensorMap& tm_feat, const CUtensorMap& tm_kern, float* out, int64_t B, int64_t C, int64_t P,
                   int64_t I, cudaStream_t st) {
  const int n_chunks = (int)ceil_div(I, BN);
  const int64_t groups = B * n_chunks;
  if (groups > 65535) return BXS_ERR_UNSUPPORTED;
  const int tiles_m = (int)ceil_div(P, BLOCK_M);
  const int per_group = std::min((int)std::max<int64_t>(1, sm_count() / groups), tiles_m);
  const size_t smem = sizeof(SmemLayout) + 1024;
  cudaFuncSetAttribute(dynconv_tf32_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dynconv_tf32_kernel<BN><<<dim3(per_group, (unsigned)groups), NUM_THREADS, smem, st>>>(tm_feat, tm_kern, out, (int)C,
                                                                                        (int)P, (int)I, n_chunks);
  return check_launch();
}

// the narrowest accumulator that holds I kernels (chunks of 128 beyond that)
inline int forward_bn(int64_t I) { return I <= 32 ? 32 : I <= 64 ? 64 : 128; }

int dynconv_forward(const float* feat3, int64_t feat_rows, const float* kern, float* out, int64_t B, int64_t C, int64_t P,
                    int64_t I, cudaStream_t st) {
  const int bn = forward_bn(I);
  CUtensorMap tm_feat, tm_kern;
  if (!make_map3(&tm_feat, feat3, B, feat_rows, P, BLOCK_K) || !make_map(&tm_kern, kern, B * I, C, bn)) {
    set_last_error(cudaErrorNotSupported);
    return BXS_ERR_LAUNCH;
  }
  if (bn == 32) return launch_forward<32>(tm_feat, tm_kern, out, B, C, P, I, st);
  if (bn == 64) return launch_forward<64>(tm_feat, tm_kern, out, B, C, P, I, st);
  return launch_forward<128>(tm_feat, tm_kern, out, B, C, P, I, st);
}

}  // namespace
}  // namespace bxs

using namespace bxs;

// feat [B,C,P], kernels [B,I,C] -> out [B,I,P] (all float32, contiguous).  Requirements of the TMA/wgmma path:
// C % 32 == 0, C <= 256, P % 4 == 0, 16-byte aligned bases.  BXS_ERR_UNSUPPORTED otherwise.
extern "C" int bxs_dynconv1x1_forward(const float* feat, const float* kernels, float* out, int64_t B, int64_t C, int64_t P,
                                      int64_t I, bxs_stream_t stream) {
  if (!feat || !kernels || !out || B <= 0 || C <= 0 || P <= 0 || I <= 0) return BXS_ERR_INVALID_ARG;
  if (C % BLOCK_K || C > BLOCK_K * MAX_KBLOCKS || P % 4 || (reinterpret_cast<uintptr_t>(feat) & 15) ||
      (reinterpret_cast<uintptr_t>(kernels) & 15) || B * C >= (int64_t(1) << 31) || B * I >= (int64_t(1) << 31))
    return BXS_ERR_UNSUPPORTED;
  return dynconv_forward(feat, C, kernels, out, B, C, P, I, as_stream(stream));
}


// ---------------------------------------------------------------------------------------
// backward of the dynamic 1x1 convolution (the autograd of box_solov2_head.py:209-211, discobox_head.py:1219,
// box2mask_head.py:345; the reference gets it from cuDNN / cuBLAS)
//   d/d feat  [B,C,P] = K^T . G : the FORWARD kernel with the roles swapped -- "feat" := g_out [B,I,P] (its rows beyond I
//       read as zeros through the 3-D tensor map), "kernels" := K^T zero-padded to a multiple of 32 instances
//       (transpose_pad_kernel, in the workspace).  I <= 256.
//   d/d kernel [B,I,C] = G . F^T : dynconv_wgrad_kernel (split-K) + dynconv_wgrad_reduce.
// workspace: bxs_dynconv1x1_backward_workspace_bytes(B, C, P, I) bytes.
// ---------------------------------------------------------------------------------------
namespace {
inline int wg_splits(int64_t B, int64_t P, int64_t I) {
  const int64_t chunks = ceil_div(I, 128), kb_total = ceil_div(P, BLOCK_K);
  int64_t s = std::max<int64_t>(1, (2 * (int64_t)sm_count()) / (B * chunks));
  s = std::min<int64_t>(s, std::max<int64_t>(1, kb_total / 8));          // at least 8 k-blocks (256 pixels) per CTA
  return (int)s;
}

template <int BN>
int launch_wgrad(const CUtensorMap& tm_g, const CUtensorMap& tm_f, float* partial, int64_t B, int64_t C, int64_t P,
                 int64_t I, int chunks, int splits, int kb_per, cudaStream_t st) {
  const size_t smem = sizeof(WgSmem) + 1024;
  cudaFuncSetAttribute(dynconv_wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dynconv_wgrad_kernel<BN><<<dim3((unsigned)splits, (unsigned)(B * chunks)), NUM_THREADS, smem, st>>>(
      tm_g, tm_f, partial, (int)C, (int)P, (int)I, chunks, splits, kb_per);
  return check_launch();
}
}  // namespace

extern "C" int64_t bxs_dynconv1x1_backward_workspace_bytes(int64_t B, int64_t C, int64_t P, int64_t I) {
  if (B <= 0 || C <= 0 || P <= 0 || I <= 0) return 0;
  const int64_t ipad = ceil_div(I, 32) * 32;
  return 4 * B * C * ipad + 1024 + 4 * B * (int64_t)wg_splits(B, P, I) * I * C + 1024;
}

extern "C" int bxs_dynconv1x1_backward(const float* feat, const float* kernels, const float* g_out, float* g_feat,
                                       float* g_kernels, void* workspace, int64_t B, int64_t C, int64_t P, int64_t I,
                                       bxs_stream_t stream) {
  if (!feat || !kernels || !g_out || (!g_feat && !g_kernels) || !workspace || B <= 0 || C <= 0 || P <= 0 || I <= 0)
    return BXS_ERR_INVALID_ARG;
  if (C % BLOCK_K || C > BLOCK_K * MAX_KBLOCKS || P % 4 || (g_feat && I > 256) || (reinterpret_cast<uintptr_t>(feat) & 15) ||
      (reinterpret_cast<uintptr_t>(g_out) & 15) || (reinterpret_cast<uintptr_t>(kernels) & 15))
    return BXS_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  const int64_t ipad = ceil_div(I, 32) * 32;
  float* kt = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(workspace) + 1023) & ~uintptr_t(1023));
  float* partial = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(kt + B * C * ipad) + 1023) & ~uintptr_t(1023));
  if (g_feat) {
    const int64_t total = B * C * ipad;
    transpose_pad_kernel<<<(unsigned)std::min<int64_t>(ceil_div(total, 256), 1024), 256, 0, st>>>(kernels, kt, (int)I, (int)C,
                                                                                                  (int)ipad, total);
    // out[b, c, p] = sum_i kT[b, c, i] * g[b, i, p]: "C" := I (zero-filled up to ipad), "I" := C
    int rc = dynconv_forward(g_out, I, kt, g_feat, B, ipad, P, C, st);
    if (rc != BXS_OK) return rc;
  }
  if (g_kernels) {
    const int chunks = (int)ceil_div(I, 128), splits = wg_splits(B, P, I);
    const int kb_total = (int)ceil_div(P, BLOCK_K), kb_per = (int)ceil_div(kb_total, splits);
    CUtensorMap tm_g, tm_f;
    if (!make_map3(&tm_g, g_out, B, I, P, 128) || !make_map3(&tm_f, feat, B, C, P, (int)C)) {
      set_last_error(cudaErrorNotSupported);
      return BXS_ERR_LAUNCH;
    }
    int rc = C <= 32    ? launch_wgrad<32>(tm_g, tm_f, partial, B, C, P, I, chunks, splits, kb_per, st)
             : C <= 64  ? launch_wgrad<64>(tm_g, tm_f, partial, B, C, P, I, chunks, splits, kb_per, st)
             : C <= 128 ? launch_wgrad<128>(tm_g, tm_f, partial, B, C, P, I, chunks, splits, kb_per, st)
                        : launch_wgrad<256>(tm_g, tm_f, partial, B, C, P, I, chunks, splits, kb_per, st);
    if (rc != BXS_OK) return rc;
    const int64_t total = B * I * C;
    dynconv_wgrad_reduce<<<(unsigned)std::min<int64_t>(ceil_div(total, 256), 1024), 256, 0, st>>>(partial, g_kernels, splits,
                                                                                                  I * C, total);
    rc = check_launch();
    if (rc != BXS_OK) return rc;
  }
  return BXS_OK;
}
