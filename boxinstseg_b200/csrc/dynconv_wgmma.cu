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
// Each pipeline loop is written once: dynconv_tf32_body (TF32 pixel streaming) and dynconv_wgrad_body (split-K weight
// gradient, TF32 or 16-bit) are driven by a job object per kernel that says where its operands and results are.  The
// host path of each product (forward, backward) is one template over the operand dtype.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cstring>
#include <type_traits>

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

// elements of one 128-byte swizzle row, the K-block of every TMA box: 32 floats or 64 16-bit values
template <typename T>
constexpr int KBLOCK = 128 / (int)sizeof(T);

// the operand dtypes: tensor-map data type, and the rounding of an FP32 result to the dtype (the identity for float)
template <typename T>
struct Operand;
template <>
struct Operand<float> {
  static constexpr CUtensorMapDataType tma = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  static __device__ __forceinline__ float round(float x) { return x; }
};
template <>
struct Operand<__half> {
  static constexpr CUtensorMapDataType tma = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  static __device__ __forceinline__ __half round(float x) { return __float2half_rn(x); }
};
template <>
struct Operand<__nv_bfloat16> {
  static constexpr CUtensorMapDataType tma = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  static __device__ __forceinline__ __nv_bfloat16 round(float x) { return __float2bfloat16_rn(x); }
};

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
// the MMA of dynconv_wgrad_body for TF32 operands
struct Tf32Mma {
  template <int BN>
  static __device__ __forceinline__ void mma(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc) {
    wgmma_ss<BN>(d, adesc, bdesc);
  }
};

// Pixel (inside its 32-pixel box) of accumulator row `r` (0..7) of a warp, for the row group `j` (0..3).  A warp's
// 16 accumulator rows are two groups j = 2h (rows 0-7) and j = 2h + 1 (rows 8-15) of the box; row r is pixel
// 16 (r / 4) + 4 j + r % 4.  In the 128-byte swizzled box the 16-byte chunk of pixel p in channel row k sits at
// (p / 4) ^ (k % 8), so the 8 rows x 4 channels of one fragment load touch 32 distinct banks.
__device__ __forceinline__ int a_pixel(int r, int j) { return 16 * (r >> 2) + 4 * j + (r & 3); }
__device__ __forceinline__ float lds_box(const uint8_t* box, int k, int p) {
  return *reinterpret_cast<const float*>(box + k * 128 + ((((p >> 2) ^ (k & 7))) << 4) + (p & 3) * 4);
}

// The pixel-streaming loop of the positive-cell forward and d/d operand kernels (dynconv_tf32_kernel writes it out; see
// there).  `job` says where its operands and results are:
//   job.C, job.P, job.I  : channels (the reduction), pixels, kernels of the job's problem
//   job.kmap, job.krow<BN>(): B = rows [krow, krow + BN) of the 2-D kernel map, K-blocks of 32 channels, resident
//   job.load_a(bar, dst, pixel, kb): the [32 channels][32 pixels] box of K-block kb at `pixel`
//   job.kvalid(kb)       : channels of K-block kb that hold data; the box's other rows are read as 0
//   job.template store<BN>(acc, mt, box, p0, p1, c4): the accumulator rows of a warp (see DenseOut::store)
// The job is built from `args` (the kernel's parameters) by Job's constructor.
template <int BN, class Job, class... Args>
__device__ __forceinline__ void dynconv_tf32_body(const Args&... args) {
  extern __shared__ uint8_t smem_raw[];
  SmemLayout& S = *reinterpret_cast<SmemLayout*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const Job job(args...);
  const int kblocks = (job.C + BLOCK_K - 1) / BLOCK_K;   // channels beyond C are zero-filled by the 3-D tensor map
  const int tiles_m = (job.P + BLOCK_M - 1) / BLOCK_M;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&S.full[s], 1); mbar_init(&S.empty[s], CONSUMER_WARPS); }
    mbar_init(&S.b_full, 1);
    fence_mbarrier_init();
  }
  __syncthreads();
  if (warp == CONSUMER_WARPS) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_expect_tx(&S.b_full, (uint32_t)kblocks * BN * BLOCK_K * 4);
      for (int kb = 0; kb < kblocks; ++kb)
        tma_load_2d(job.kmap, &S.b_full, S.b[kb], kb * BLOCK_K, job.template krow<BN>());
      int stage = 0, phase = 0;
      for (int mt = blockIdx.x; mt < tiles_m; mt += gridDim.x) {
        for (int kb = 0; kb < kblocks; ++kb) {
          mbar_wait(&S.empty[stage], phase ^ 1);
          mbar_expect_tx(&S.full[stage], A_STAGE_BYTES);
#pragma unroll
          for (int g = 0; g < BLOCK_M / 32; ++g)
            job.load_a(&S.full[stage], S.a[stage] + g * BOX_BYTES, mt * BLOCK_M + g * 32, kb);
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
        const int kv = job.kvalid(kb);
        uint32_t a[BLOCK_K / MMA_K][4];
#pragma unroll
        for (int k4 = 0; k4 < BLOCK_K / MMA_K; ++k4) {
          const int k = k4 * MMA_K + c4;
          a[k4][0] = k < kv ? to_tf32(lds_box(abox, k, p0)) : 0u;
          a[k4][1] = k < kv ? to_tf32(lds_box(abox, k, p1)) : 0u;
          a[k4][2] = k + 4 < kv ? to_tf32(lds_box(abox, k + 4, p0)) : 0u;
          a[k4][3] = k + 4 < kv ? to_tf32(lds_box(abox, k + 4, p1)) : 0u;
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
      job.template store<BN>(acc, mt, box, p0, p1, c4);
    }
  }
}

// the epilogue of a [B,I,P] output (image b, kernel chunk `chunk`), as dynconv_tf32_kernel stores it
struct DenseOut {
  float* out;
  int P, I, b, chunk;
  // accumulator elements 4 j .. 4 j + 3: kernels n = 8 j + 2 c4 + {0, 1} of rows r (pixel p0) and r + 8 (pixel p1)
  template <int BN>
  __device__ __forceinline__ void store(const float (&acc)[BN / 2], int mt, int box, int p0, int p1, int c4) const {
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
};

// grid: (ctas_per_group, B * n_chunks).  CTA (x, g): image b = g / n_chunks, kernel chunk g % n_chunks of BN kernels,
// pixel tiles x, x + gridDim.x, ...
// The loop is dynconv_tf32_body's, written out: run on dynconv_tf32_body through a job object, this kernel compiles to
// different address arithmetic and fragment-load order, and at BN = 32 it measured 1.3-2 % slower (H100 80GB HBM3,
// 700 W power limit, I = 16 at 200 x 256 pixels).
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
    fence_mbarrier_init();
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
      DenseOut{out, P, I, b, chunk}.store<BN>(acc, mt, box, p0, p1, c4);
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

// The tensor map of a row-major [batch, rows, cols] tensor of T, box = [1, box_rows, KBLOCK<T> columns = 128 bytes],
// 128-byte swizzle, zero fill out of bounds.  Rank 3: rows beyond `rows` of a batch entry are OUT OF BOUNDS and read as
// zeros (a 2-D [batch * rows, cols] view would run into the next entry instead).  Rank 2: the [rows, cols] matrix of a
// batch of 1, for kernels that issue 2-D loads.  false, with the last error set, when the driver cannot encode it.
template <typename T>
bool make_map(CUtensorMap* map, int rank, const T* base, int64_t batch, int64_t rows, int64_t cols, int box_rows) {
  EncodeTiledFn fn = encode_fn();
  const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)batch};
  const cuuint64_t strides[2] = {(cuuint64_t)cols * sizeof(T), (cuuint64_t)cols * (cuuint64_t)rows * sizeof(T)};
  const cuuint32_t box[3] = {KBLOCK<T>, (cuuint32_t)box_rows, 1}, estr[3] = {1, 1, 1};
  if (fn && fn(map, Operand<T>::tma, rank, const_cast<T*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS)
    return true;
  set_last_error(cudaErrorNotSupported);
  return false;
}

// kT[b, c, i] = kernels[b, i, c] for i < I, 0 for I <= i < Ipad   (the K-major B operand of d/d feat = K^T . G)
template <typename T>
__global__ void transpose_pad_kernel(const T* __restrict__ k, T* __restrict__ kt, int I, int C, int Ipad, int64_t total) {
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx % Ipad);
    const int c = (int)((idx / Ipad) % C);
    const int64_t b = idx / ((int64_t)Ipad * C);
    kt[idx] = i < I ? __ldg(k + (b * I + i) * C + c) : T();
  }
}

// =====================================================================================================================
// d/d kernel:  dK[b,i,c] = sum_p g[b,i,p] * feat[b,c,p]  -- a GEMM with a LONG reduction (K = pixels, 51 200 .. 65 536) and a
// tiny output (I x C).  Both operands are K-major (the pixel index is contiguous in g and in feat), so wgmma reads both
// from shared memory with the 128-byte swizzle.  Split-K: CTA (split, b * chunks + chunk) reduces pixels [p0, p1) of
// image b for 128 rows of g (64 per consumer warpgroup) into a 128 x C register accumulator (C <= 256 columns) and
// stores it as a partial; dynconv_wgrad_reduce sums the partials in split order (deterministic).  A stage holds one
// K-block of pixels, one 128-byte swizzle row: 32 pixels for TF32 operands, 64 for 16-bit ones.
//   warps 0-7: two consumer warpgroups (wgmma, epilogue)
//   warp 8   : TMA producer (A = g tile 128 rows x 128 bytes, B = feat tile C rows x 128 bytes per stage, 4 stages)
// =====================================================================================================================
constexpr int WG_STAGES = 4;
constexpr int WG_A_BYTES = 128 * 128;              // 16 KB
constexpr int WG_B_BYTES = 256 * 128;              // 32 KB

struct WgSmem {
  alignas(1024) uint8_t a[WG_STAGES][WG_A_BYTES];
  alignas(1024) uint8_t b[WG_STAGES][WG_B_BYTES];
  alignas(8) uint64_t full[WG_STAGES];
  uint64_t empty[WG_STAGES];
};

// The split-K loop of one CTA.  `job`:
//   job.C, job.kb0, job.kb1     : columns of the result (rows of B), the job's K-blocks of pixels
//   job.load_g(bar, dst, kb)    : A = 128 rows of g x 1 K-block;  job.load_f(bar, dst, kb): B = C rows x 1 K-block
//   job.template store<BN>(acc, wg, w, r, c4): the accumulator of a warp (see DenseWgJob)
// Mma::template mma<BN>(acc, adesc, bdesc): the wgmma over 32 bytes of K of both (K-major) operands, TF32 or 16-bit.
// BN: C rounded up to 32, 64, 128 or 256 (the columns beyond C are computed from unused shared memory and dropped)
template <int BN, class Mma, class Job>
__device__ __forceinline__ void dynconv_wgrad_body(const Job& job) {
  extern __shared__ uint8_t smem_raw[];
  WgSmem& S = *reinterpret_cast<WgSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; ++s) { mbar_init(&S.full[s], 1); mbar_init(&S.empty[s], CONSUMER_WARPS); }
    fence_mbarrier_init();
  }
  __syncthreads();
  if (warp == CONSUMER_WARPS) {
    if (lane == 0) {
      int stage = 0, phase = 0;
      for (int kb = job.kb0; kb < job.kb1; ++kb) {
        mbar_wait(&S.empty[stage], phase ^ 1);
        mbar_expect_tx(&S.full[stage], WG_A_BYTES + (uint32_t)job.C * 128);
        job.load_g(&S.full[stage], S.a[stage], kb);
        job.load_f(&S.full[stage], S.b[stage], kb);
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    const int wg = warp >> 2, w = warp & 3, r = lane >> 2, c4 = lane & 3;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0, phase = 0;
    for (int kb = job.kb0; kb < job.kb1; ++kb) {
      mbar_wait(&S.full[stage], phase);
      const uint32_t a_base = smem_u32(S.a[stage]) + wg * (64 * 128), b_base = smem_u32(S.b[stage]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 128 / 32; ++k) Mma::template mma<BN>(acc, make_desc(a_base + k * 32), make_desc(b_base + k * 32));
      wgmma_commit();
      wgmma_wait_all();
      fence_acc(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&S.empty[stage]);
      if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
    }
    job.template store<BN>(acc, wg, w, r, c4);
  }
}

// the dense d/d kernel: rows [128 chunk, 128 chunk + 128) of g [B,I,P] of image b = blockIdx.y / chunks, chunk =
// blockIdx.y % chunks, the pixels of split `split` = blockIdx.x in K-blocks of BK pixels
template <int BK>
struct DenseWgJob {
  const CUtensorMap* g;
  const CUtensorMap* feat;
  float* partial;
  int C, I, b, chunk, split, splits, kb0, kb1;
  __device__ __forceinline__ DenseWgJob(const CUtensorMap& tm_g, const CUtensorMap& tm_feat, float* partial_, int C_, int P,
                                        int I_, int chunks, int splits_, int kb_per_split)
      : g(&tm_g), feat(&tm_feat), partial(partial_), C(C_), I(I_), b(blockIdx.y / chunks), chunk(blockIdx.y % chunks),
        split(blockIdx.x), splits(splits_) {
    kb0 = split * kb_per_split;
    kb1 = min(kb0 + kb_per_split, (P + BK - 1) / BK);
  }
  __device__ __forceinline__ void load_g(uint64_t* bar, void* dst, int kb) const {
    tma_load_3d(g, bar, dst, kb * BK, chunk * 128, b);       // rows >= I: zeros
  }
  __device__ __forceinline__ void load_f(uint64_t* bar, void* dst, int kb) const {
    tma_load_3d(feat, bar, dst, kb * BK, 0, b);
  }
  // accumulator elements (i, i + 1), i even: row 16 w + r (+ 8 when i % 4 == 2), columns 8 (i / 4) + 2 c4 + {0, 1}
  template <int BN>
  __device__ __forceinline__ void store(const float (&acc)[BN / 2], int wg, int w, int r, int c4) const {
    const int row0 = chunk * 128 + wg * 64 + w * 16 + r;
    float* dst = partial + (((int64_t)b * splits + split) * I) * C;
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int row = row0 + ((i & 2) ? 8 : 0), n = 8 * (i >> 2) + 2 * c4;
      if (row < I && n < C) *reinterpret_cast<float2*>(dst + (int64_t)row * C + n) = make_float2(acc[i], acc[i + 1]);
    }
  }
};

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
dynconv_wgrad_kernel(const __grid_constant__ CUtensorMap tm_g, const __grid_constant__ CUtensorMap tm_feat,
                     float* __restrict__ partial, int C, int P, int I, int chunks, int splits, int kb_per_split) {
  dynconv_wgrad_body<BN, Tf32Mma>(DenseWgJob<BLOCK_K>(tm_g, tm_feat, partial, C, P, I, chunks, splits, kb_per_split));
}

// out[b, r] = the partials of image b summed in split order (deterministic), rounded to the operand dtype
template <typename T>
__global__ void dynconv_wgrad_reduce(const float* __restrict__ partial, T* __restrict__ out, int splits, int64_t per_image,
                                     int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / per_image, r = i - b * per_image;
    const float* p = partial + b * splits * per_image + r;
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += p[(int64_t)s * per_image];          // split order: deterministic
    out[i] = Operand<T>::round(acc);
  }
}

// the narrowest accumulator that holds I kernels (chunks of 128 beyond that)
inline int forward_bn(int64_t I) { return I <= 32 ? 32 : I <= 64 ? 64 : 128; }

// the grid of the pixel-streaming kernels: `groups` rows of CTAs that share the SMs, each row no wider than its `tiles`
inline dim3 persistent_grid(int64_t groups, int tiles) {
  return dim3(std::min((int)std::max<int64_t>(1, sm_count() / groups), tiles), (unsigned)groups);
}

// opts `kern` in to `smem` bytes of dynamic shared memory and launches it with NUM_THREADS threads per CTA
template <class Kernel, class... Args>
int launch(Kernel kern, dim3 grid, size_t smem, cudaStream_t st, const Args&... args) {
  if (opt_in_smem(kern, smem) != BXS_OK) return BXS_ERR_LAUNCH;
  kern<<<grid, NUM_THREADS, smem, st>>>(args...);
  return check_launch();
}

// 1-D grid of the grid-stride kernels (256 threads per CTA)
inline unsigned stride_grid(int64_t total) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(total, 256), 1024)); }

template <typename T>
inline T* align1k(void* p) { return reinterpret_cast<T*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023)); }

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace
}  // namespace bxs

using namespace bxs;


// =====================================================================================================================
// Positive-cell dynamic convolution (BoxSOLOv2's forward + boolean indexing, box_solov2_head.py:204-216, 317-320):
// level l convolves the positive cells of its kernel grid [B,C,S_l,S_l] with operand op(l) [B,C,P_op], and its result
// [n_l, P_op] holds the rows of image 0, then image 1, ..., cells ascending.  A problem is (operand o, image b); its
// kernels are the positive cells of every level of o (levels of one operand are consecutive), level by level.
//   forward   : pack (gather the problems' kernels K-major from the raw grids) + dynconv_tf32_body over the table
//   d/d operand: pack K^T per problem, each level's kernels zero-padded to 32, + dynconv_tf32_body with the roles swapped
//               (A = the level's output gradient rows, B = K^T)
//   d/d kernel: dynconv_wgrad_body per (level, image) segment + an ordered reduce into the raw [B,C,S,S] layout
// =====================================================================================================================
namespace bxs {
namespace {

constexpr int CELLS_MAX_LEVELS = 8;
constexpr int CELLS_MAX_OPS = 4;
constexpr int CELLS_MAX_IMAGES = 16;
constexpr int CELLS_MAX_PROBLEMS = CELLS_MAX_OPS * CELLS_MAX_IMAGES;
constexpr int CELLS_MAX_SEGS = CELLS_MAX_LEVELS * CELLS_MAX_IMAGES;

// The problem table, passed by value (about 3 KB of kernel parameters)
struct CellsPlan {
  CUtensorMap a[CELLS_MAX_LEVELS];        // A maps: operands (forward) or level output gradients (backward)
  CUtensorMap b[CELLS_MAX_OPS];           // B maps: packed kernels in b[0] (forward, d/d operand) or operands (d/d kernel)
  float* out[CELLS_MAX_LEVELS];           // forward: level outputs; d/d operand: operand gradients; d/d kernel: grids
  const float* kern[CELLS_MAX_LEVELS];    // raw kernel grids [B,C,S_l,S_l]
  const int32_t* cells;                   // [sum n_l] level-major, image-major, cells ascending
  int S2[CELLS_MAX_LEVELS];
  int lo[CELLS_MAX_OPS + 1];              // operand o owns levels [lo[o], lo[o+1])
  int P[CELLS_MAX_OPS];
  int start[CELLS_MAX_SEGS + 1];          // segment (l, b) = rows [start[l B + b], start[l B + b + 1]) of `cells`
  int pbase[CELLS_MAX_PROBLEMS + 1];      // problem (o, b) = packed kernel rows [pbase[o B + b], pbase[o B + b + 1])
  int chunk0[CELLS_MAX_SEGS + 1];         // first grid row of each problem (forward, d/d operand) or segment (d/d kernel)
  int n_levels, n_ops, B, C, KP, splits;
  __host__ __device__ int cnt(int l, int b) const { return start[l * B + b + 1] - start[l * B + b]; }
  __host__ __device__ int level_row(int l, int b) const { return start[l * B + b] - start[l * B]; }   // in level l's output
  __host__ __device__ int op_of(int l) const {
    int o = 0;
    while (o + 1 < n_ops && lo[o + 1] <= l) ++o;
    return o;
  }
};

__device__ __forceinline__ int find_chunk(const int* chunk0, int n, int y) {
  int i = 0;
  while (i + 1 < n && chunk0[i + 1] <= y) ++i;
  return i;
}

__device__ __forceinline__ float cell_kernel(const CellsPlan& pl, int l, int b, int i, int c) {
  const int cell = __ldg(pl.cells + pl.start[l * pl.B + b] + i);
  if (cell < 0 || cell >= pl.S2[l]) return 0.f;          // outside the grid: a zero kernel, never a stray read
  return __ldg(pl.kern[l] + ((int64_t)b * pl.C + c) * pl.S2[l] + cell);
}

// kpack[row, c], rows in problem order (the forward's K-major B operand)
__global__ void cells_pack_kernel(const __grid_constant__ CellsPlan pl, float* __restrict__ kpack, int64_t total) {
  const int np = pl.n_ops * pl.B;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int row = (int)(idx / pl.C), c = (int)(idx % pl.C);
    const int p = find_chunk(pl.pbase, np, row);
    const int o = p / pl.B, b = p % pl.B;
    int i = row - pl.pbase[p], l = pl.lo[o];
    while (l + 1 < pl.lo[o + 1] && i >= pl.cnt(l, b)) i -= pl.cnt(l++, b);
    kpack[idx] = cell_kernel(pl, l, b, i, c);
  }
}

// kT[p, c, k] (k < KP): problem p's kernels K^T, each level's kernels zero-padded to a multiple of 32
__global__ void cells_pack_t_kernel(const __grid_constant__ CellsPlan pl, float* __restrict__ kt, int64_t total) {
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int k = (int)(idx % pl.KP);
    const int c = (int)((idx / pl.KP) % pl.C), p = (int)(idx / ((int64_t)pl.KP * pl.C));
    const int o = p / pl.B, b = p % pl.B;
    float v = 0.f;
    for (int l = pl.lo[o]; l < pl.lo[o + 1]; ++l) {
      const int n = pl.cnt(l, b), n32 = (n + 31) & ~31;
      if (k < n32) {
        if (k < n) v = cell_kernel(pl, l, b, k, c);
        break;
      }
      k -= n32;
    }
    kt[idx] = v;
  }
}

// forward: problem (o, b), kernel chunk `chunk`
struct CellsFwdJob {
  const CellsPlan* pl;
  const CUtensorMap* kmap;
  int o, b, chunk, C, P, I, kbase;
  __device__ __forceinline__ CellsFwdJob(const CellsPlan& p) : pl(&p), kmap(&p.b[0]) {
    const int np = p.n_ops * p.B, q = find_chunk(p.chunk0, np, blockIdx.y);
    o = q / p.B, b = q % p.B, chunk = blockIdx.y - p.chunk0[q];
    C = p.C, P = p.P[o], kbase = p.pbase[q], I = p.pbase[q + 1] - kbase;
  }
  template <int BN>
  __device__ __forceinline__ int krow() const { return kbase + chunk * BN; }
  __device__ __forceinline__ void load_a(uint64_t* bar, void* dst, int x, int kb) const {
    tma_load_3d(&pl->a[o], bar, dst, x, kb * BLOCK_K, b);
  }
  __device__ __forceinline__ int kvalid(int) const { return BLOCK_K; }
  // kernel n of the problem -> its row of its level's output
  __device__ __forceinline__ float* row(int n) const {
    int l = pl->lo[o];
    while (l + 1 < pl->lo[o + 1] && n >= pl->cnt(l, b)) n -= pl->cnt(l++, b);
    return pl->out[l] + (int64_t)(pl->level_row(l, b) + n) * P;
  }
  template <int BN>
  __device__ __forceinline__ void store(const float (&acc)[BN / 2], int mt, int box, int p0, int p1, int c4) const {
    const int pix = mt * BLOCK_M + box * 32;
    const bool in0 = pix + p0 < P, in1 = pix + p1 < P;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = chunk * BN + 8 * j + 2 * c4;
      if (n < I) {
        float* dst = row(n) + pix;
        if (in0) dst[p0] = acc[4 * j];
        if (in1) dst[p1] = acc[4 * j + 2];
      }
      if (n + 1 < I) {
        float* dst = row(n + 1) + pix;
        if (in0) dst[p0] = acc[4 * j + 1];
        if (in1) dst[p1] = acc[4 * j + 3];
      }
    }
  }
};

// d/d operand: problem (o, b), channel chunk `chunk`; reduction over the problem's padded kernels
struct CellsDgradJob {
  const CellsPlan* pl;
  const CUtensorMap* kmap;
  int o, b, chunk, C, P, I, q;
  __device__ __forceinline__ CellsDgradJob(const CellsPlan& p, int n_chunks) : pl(&p), kmap(&p.b[0]) {
    q = blockIdx.y / n_chunks, chunk = blockIdx.y % n_chunks;
    o = q / p.B, b = q % p.B, P = p.P[o], I = p.C;
    C = 0;
    for (int l = p.lo[o]; l < p.lo[o + 1]; ++l) C += (p.cnt(l, b) + 31) & ~31;
  }
  template <int BN>
  __device__ __forceinline__ int krow() const { return q * I + chunk * BN; }
  // K-block kb = 32 gradient rows of one level, the k-th block of its (level, image) segment
  __device__ __forceinline__ int segment(int& kb) const {
    int l = pl->lo[o];
    for (;; ++l) {
      const int nk = (pl->cnt(l, b) + 31) >> 5;
      if (kb < nk || l + 1 == pl->lo[o + 1]) return l;
      kb -= nk;
    }
  }
  __device__ __forceinline__ void load_a(uint64_t* bar, void* dst, int x, int kb) const {
    const int l = segment(kb);
    tma_load_3d(&pl->a[l], bar, dst, x, pl->level_row(l, b) + kb * BLOCK_K, 0);
  }
  // rows past the segment belong to the next image (or lie outside the map): read as 0, so that nothing of another
  // image's gradient, not even an Inf or NaN, reaches this one
  __device__ __forceinline__ int kvalid(int kb) const {
    const int l = segment(kb);
    return min(BLOCK_K, pl->cnt(l, b) - kb * BLOCK_K);
  }
  template <int BN>
  __device__ __forceinline__ void store(const float (&acc)[BN / 2], int mt, int box, int p0, int p1, int c4) const {
    DenseOut{pl->out[o], P, I, b, chunk}.template store<BN>(acc, mt, box, p0, p1, c4);   // g_operand[o] [B,C,P]
  }
};

// d/d kernel: segment (l, b), row chunk `chunk` of 128 kernels, split `split` of the pixels
struct CellsWgJob {
  const CellsPlan* pl;
  float* partial;
  int l, o, b, chunk, split, C, I, kb0, kb1;
  __device__ __forceinline__ CellsWgJob(const CellsPlan& p, float* partial_) : pl(&p), partial(partial_) {
    const int s = find_chunk(p.chunk0, p.n_levels * p.B, blockIdx.y);
    l = s / p.B, b = s % p.B, chunk = blockIdx.y - p.chunk0[s], split = blockIdx.x;
    o = p.op_of(l);
    C = p.C, I = p.cnt(l, b);
    const int kb_total = (p.P[o] + BLOCK_K - 1) / BLOCK_K, kb_per = (kb_total + p.splits - 1) / p.splits;
    kb0 = split * kb_per, kb1 = min(kb0 + kb_per, kb_total);
  }
  __device__ __forceinline__ void load_g(uint64_t* bar, void* dst, int kb) const {
    tma_load_3d(&pl->a[l], bar, dst, kb * BLOCK_K, pl->level_row(l, b) + chunk * 128, 0);   // rows past I: dropped
  }
  __device__ __forceinline__ void load_f(uint64_t* bar, void* dst, int kb) const {
    tma_load_3d(&pl->b[o], bar, dst, kb * BLOCK_K, 0, b);
  }
  // partial[(grid row, split)] = [128 rows][C]
  template <int BN>
  __device__ __forceinline__ void store(const float (&acc)[BN / 2], int wg, int w, int r, int c4) const {
    const int row0 = wg * 64 + w * 16 + r;
    float* dst = partial + ((int64_t)blockIdx.y * pl->splits + split) * 128 * C;
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int row = row0 + ((i & 2) ? 8 : 0), n = 8 * (i >> 2) + 2 * c4;
      if (chunk * 128 + row < I && n < C)
        *reinterpret_cast<float2*>(dst + (int64_t)row * C + n) = make_float2(acc[i], acc[i + 1]);
    }
  }
};

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1) dynconv_cells_kernel(const __grid_constant__ CellsPlan pl) {
  dynconv_tf32_body<BN, CellsFwdJob>(pl);
}

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1) dynconv_cells_dgrad_kernel(const __grid_constant__ CellsPlan pl,
                                                                             int n_chunks) {
  dynconv_tf32_body<BN, CellsDgradJob>(pl, n_chunks);
}

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1) dynconv_cells_wgrad_kernel(const __grid_constant__ CellsPlan pl,
                                                                             float* __restrict__ partial) {
  const CellsWgJob job(pl, partial);
  dynconv_wgrad_body<BN, Tf32Mma>(job);
}

// d kernel_pred[l][b, c, cell] = the split-ordered sum of the partials of the positive cell's row, 0 for other cells.
// One thread per (level, image, cell); the row of a positive cell is found by bisection (cells ascending per segment).
__global__ void dynconv_cells_wgrad_reduce(const __grid_constant__ CellsPlan pl, const float* __restrict__ partial,
                                           int64_t total) {
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int64_t rem = idx;
    int l = 0;
    while (rem >= (int64_t)pl.B * pl.S2[l]) rem -= (int64_t)pl.B * pl.S2[l++];
    const int b = (int)(rem / pl.S2[l]), cell = (int)(rem % pl.S2[l]);
    const int32_t* seg = pl.cells + pl.start[l * pl.B + b];
    int lo = 0, hi = pl.cnt(l, b);
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (__ldg(seg + mid) < cell) lo = mid + 1; else hi = mid;
    }
    float* dst = pl.out[l] + (int64_t)b * pl.C * pl.S2[l] + cell;
    if (lo < pl.cnt(l, b) && __ldg(seg + lo) == cell) {
      const int g = pl.chunk0[l * pl.B + b] + lo / 128, r = lo % 128;
      const float* src = partial + ((int64_t)g * pl.splits * 128 + r) * pl.C;
      for (int c = 0; c < pl.C; ++c) {
        float acc = 0.f;
        for (int s = 0; s < pl.splits; ++s) acc += src[(int64_t)s * 128 * pl.C + c];      // split order: deterministic
        dst[(int64_t)c * pl.S2[l]] = acc;
      }
    } else {
      for (int c = 0; c < pl.C; ++c) dst[(int64_t)c * pl.S2[l]] = 0.f;
    }
  }
}

// Validates the host arrays and fills the sizes of the table (no device pointers, no maps).  BXS_OK or an error code.
int cells_plan(CellsPlan& pl, const int64_t* op_size, const int64_t* grid, const int64_t* level_op, const int64_t* counts,
               int64_t n_levels, int64_t n_ops, int64_t B, int64_t C) {
  if (!op_size || !grid || !level_op || !counts || n_levels <= 0 || n_ops <= 0 || B <= 0 || C <= 0)
    return BXS_ERR_INVALID_ARG;
  if (n_levels > CELLS_MAX_LEVELS || n_ops > CELLS_MAX_OPS || B > CELLS_MAX_IMAGES || C % BLOCK_K ||
      C > BLOCK_K * MAX_KBLOCKS)
    return BXS_ERR_UNSUPPORTED;
  memset(&pl, 0, sizeof(pl));
  pl.n_levels = (int)n_levels, pl.n_ops = (int)n_ops, pl.B = (int)B, pl.C = (int)C;
  for (int o = 0; o < n_ops; ++o) {
    if (op_size[o] <= 0) return BXS_ERR_INVALID_ARG;
    if (op_size[o] % 4 || op_size[o] >= (int64_t(1) << 31)) return BXS_ERR_UNSUPPORTED;
    pl.P[o] = (int)op_size[o];
  }
  int64_t total = 0;
  for (int l = 0; l < n_levels; ++l) {
    // operands in level order, each owning consecutive levels
    if (l == 0 ? level_op[0] != 0 : (level_op[l] != level_op[l - 1] && level_op[l] != level_op[l - 1] + 1))
      return BXS_ERR_INVALID_ARG;
    if (grid[l] <= 0) return BXS_ERR_INVALID_ARG;
    if (grid[l] * grid[l] * B * C >= (int64_t(1) << 31)) return BXS_ERR_UNSUPPORTED;
    pl.S2[l] = (int)(grid[l] * grid[l]);
    if (l == 0 || level_op[l] != level_op[l - 1]) pl.lo[level_op[l]] = l;
    for (int b = 0; b < B; ++b) {
      const int64_t n = counts[l * B + b];
      if (n < 0 || n > grid[l] * grid[l]) return BXS_ERR_INVALID_ARG;
      pl.start[l * B + b] = (int)total;
      total += n;
    }
  }
  if (level_op[n_levels - 1] != n_ops - 1) return BXS_ERR_INVALID_ARG;
  if (total * C >= (int64_t(1) << 31)) return BXS_ERR_UNSUPPORTED;
  pl.start[n_levels * B] = (int)total;
  pl.lo[n_ops] = (int)n_levels;
  int rows = 0;
  for (int o = 0; o < n_ops; ++o)
    for (int b = 0; b < B; ++b) {
      pl.pbase[o * B + b] = rows;
      for (int l = pl.lo[o]; l < pl.lo[o + 1]; ++l) rows += pl.cnt(l, b);
    }
  pl.pbase[n_ops * B] = rows;
  return BXS_OK;
}

// widest padded kernel count of a problem (the reduction of d/d operand)
int cells_kp(const CellsPlan& pl) {
  int kp = 0;
  for (int o = 0; o < pl.n_ops; ++o)
    for (int b = 0; b < pl.B; ++b) {
      int k = 0;
      for (int l = pl.lo[o]; l < pl.lo[o + 1]; ++l) k += (pl.cnt(l, b) + 31) & ~31;
      kp = std::max(kp, k);
    }
  return kp;
}

int cells_wgrad_splits(CellsPlan& pl) {
  int chunks = 0, kb_min = 1 << 30;
  for (int l = 0; l < pl.n_levels; ++l)
    for (int b = 0; b < pl.B; ++b) {
      pl.chunk0[l * pl.B + b] = chunks;
      chunks += (pl.cnt(l, b) + 127) / 128;
    }
  pl.chunk0[pl.n_levels * pl.B] = chunks;
  for (int o = 0; o < pl.n_ops; ++o) kb_min = std::min<int>(kb_min, (int)ceil_div(pl.P[o], BLOCK_K));
  pl.splits = (int)std::max<int64_t>(1, std::min<int64_t>((2 * (int64_t)sm_count()) / std::max(chunks, 1),
                                                          std::max(1, kb_min / (256 / BLOCK_K))));
  return chunks;
}
}  // namespace
}  // namespace bxs

extern "C" int64_t bxs_dynconv1x1_cells_forward_workspace_bytes(const int64_t* counts_host, int64_t n_levels, int64_t B,
                                                                int64_t C) {
  if (!counts_host || n_levels <= 0 || B <= 0 || C <= 0) return 0;
  int64_t total = 0;
  for (int64_t i = 0; i < n_levels * B; ++i) total += std::max<int64_t>(0, counts_host[i]);
  return total ? 4 * total * C + 1024 : 0;
}

extern "C" int bxs_dynconv1x1_cells_forward(const float* const* operands_host, const int64_t* op_size_host,
                                            const float* const* kernels_host, const int64_t* grid_host,
                                            const int64_t* level_op_host, const int64_t* counts_host, const int32_t* cells,
                                            float* const* out_host, void* workspace, int64_t n_levels, int64_t n_ops,
                                            int64_t B, int64_t C, bxs_stream_t stream) {
  CellsPlan pl;
  int rc = cells_plan(pl, op_size_host, grid_host, level_op_host, counts_host, n_levels, n_ops, B, C);
  if (rc != BXS_OK) return rc;
  const int total = pl.start[n_levels * B];
  if (total == 0) return BXS_OK;
  if (!operands_host || !kernels_host || !out_host || !cells || !workspace) return BXS_ERR_INVALID_ARG;
  for (int o = 0; o < n_ops; ++o) {
    if (!operands_host[o]) return BXS_ERR_INVALID_ARG;
    if (!aligned16(operands_host[o])) return BXS_ERR_UNSUPPORTED;
  }
  for (int l = 0; l < n_levels; ++l) {
    if (!kernels_host[l] || (!out_host[l] && pl.start[(l + 1) * B] > pl.start[l * B])) return BXS_ERR_INVALID_ARG;
    pl.kern[l] = kernels_host[l];
    pl.out[l] = out_host[l];
  }
  pl.cells = cells;
  const int bn = forward_bn([&] {
    int m = 0;
    for (int q = 0; q < n_ops * B; ++q) m = std::max(m, pl.pbase[q + 1] - pl.pbase[q]);
    return m;
  }());
  int groups = 0, tiles = 0;
  for (int q = 0; q < n_ops * B; ++q) {
    pl.chunk0[q] = groups;
    groups += (int)ceil_div(pl.pbase[q + 1] - pl.pbase[q], bn);
  }
  pl.chunk0[n_ops * B] = groups;
  if (groups > 65535) return BXS_ERR_UNSUPPORTED;
  float* kpack = align1k<float>(workspace);
  for (int o = 0; o < n_ops; ++o) {
    tiles = std::max(tiles, (int)ceil_div(pl.P[o], BLOCK_M));
    if (!make_map(&pl.a[o], 3, operands_host[o], B, C, pl.P[o], BLOCK_K)) return BXS_ERR_LAUNCH;
  }
  if (!make_map(&pl.b[0], 2, kpack, 1, total, C, bn)) return BXS_ERR_LAUNCH;
  cudaStream_t st = as_stream(stream);
  cells_pack_kernel<<<stride_grid((int64_t)total * C), 256, 0, st>>>(pl, kpack, (int64_t)total * C);
  if ((rc = check_launch()) != BXS_OK) return rc;
  const dim3 grid = persistent_grid(groups, tiles);
  auto go = [&](auto kernel) { return launch(kernel, grid, sizeof(SmemLayout) + 1024, st, pl); };
  return bn == 32 ? go(dynconv_cells_kernel<32>) : bn == 64 ? go(dynconv_cells_kernel<64>) : go(dynconv_cells_kernel<128>);
}

extern "C" int64_t bxs_dynconv1x1_cells_backward_workspace_bytes(const int64_t* op_size_host, const int64_t* grid_host,
                                                                 const int64_t* level_op_host, const int64_t* counts_host,
                                                                 int64_t n_levels, int64_t n_ops, int64_t B, int64_t C) {
  CellsPlan pl;
  if (cells_plan(pl, op_size_host, grid_host, level_op_host, counts_host, n_levels, n_ops, B, C) != BXS_OK) return 0;
  const int chunks = cells_wgrad_splits(pl);
  return 4 * (int64_t)n_ops * B * C * cells_kp(pl) + 1024 + 4 * (int64_t)chunks * pl.splits * 128 * C + 1024;
}

extern "C" int bxs_dynconv1x1_cells_backward(const float* const* operands_host, const int64_t* op_size_host,
                                             const float* const* kernels_host, const int64_t* grid_host,
                                             const int64_t* level_op_host, const int64_t* counts_host,
                                             const int32_t* cells, const float* const* g_out_host,
                                             float* const* g_operands_host, float* const* g_kernels_host, void* workspace,
                                             int64_t n_levels, int64_t n_ops, int64_t B, int64_t C, bxs_stream_t stream) {
  CellsPlan pl;
  int rc = cells_plan(pl, op_size_host, grid_host, level_op_host, counts_host, n_levels, n_ops, B, C);
  if (rc != BXS_OK) return rc;
  if (!operands_host || !kernels_host || !g_out_host || (!g_operands_host && !g_kernels_host) || !workspace ||
      (pl.start[n_levels * B] && !cells))
    return BXS_ERR_INVALID_ARG;
  pl.KP = cells_kp(pl);
  if (g_operands_host && pl.KP > 256) return BXS_ERR_UNSUPPORTED;
  for (int o = 0; o < n_ops; ++o) {
    if (!operands_host[o] || (g_operands_host && !g_operands_host[o])) return BXS_ERR_INVALID_ARG;
    if (!aligned16(operands_host[o])) return BXS_ERR_UNSUPPORTED;
  }
  for (int l = 0; l < n_levels; ++l) {
    const bool rows = pl.start[(l + 1) * B] > pl.start[l * B];
    if (!kernels_host[l] || (rows && !g_out_host[l]) || (g_kernels_host && !g_kernels_host[l])) return BXS_ERR_INVALID_ARG;
    if (rows && !aligned16(g_out_host[l])) return BXS_ERR_UNSUPPORTED;
    pl.kern[l] = kernels_host[l];
  }
  pl.cells = cells;
  cudaStream_t st = as_stream(stream);
  const int chunks = cells_wgrad_splits(pl);         // fills chunk0 / splits of the d/d kernel table
  float* kt = align1k<float>(workspace);
  float* partial = align1k<float>(kt + (int64_t)n_ops * B * C * pl.KP);
  if (g_operands_host) {
    CellsPlan d = pl;
    for (int o = 0; o < n_ops; ++o) d.out[o] = g_operands_host[o];
    if (d.KP == 0) {                                   // no positive cell at all: zero gradients
      for (int o = 0; o < n_ops; ++o)
        if (cudaMemsetAsync(d.out[o], 0, sizeof(float) * B * C * d.P[o], st) != cudaSuccess) return check_launch();
    } else {
      for (int l = 0; l < n_levels; ++l) {
        const int n = d.start[(l + 1) * B] - d.start[l * B];
        if (n && !make_map(&d.a[l], 3, g_out_host[l], 1, n, d.P[d.op_of(l)], BLOCK_K)) return BXS_ERR_LAUNCH;
      }
      const int bn = forward_bn(C), n_chunks = (int)ceil_div(C, bn);
      if (!make_map(&d.b[0], 2, kt, 1, (int64_t)n_ops * B * C, d.KP, bn)) return BXS_ERR_LAUNCH;
      const int64_t total = (int64_t)n_ops * B * C * d.KP;
      cells_pack_t_kernel<<<stride_grid(total), 256, 0, st>>>(d, kt, total);
      if ((rc = check_launch()) != BXS_OK) return rc;
      int tiles = 0;
      for (int o = 0; o < n_ops; ++o) tiles = std::max(tiles, (int)ceil_div(d.P[o], BLOCK_M));
      const dim3 grid = persistent_grid(n_ops * (int)B * n_chunks, tiles);
      auto go = [&](auto kernel) { return launch(kernel, grid, sizeof(SmemLayout) + 1024, st, d, n_chunks); };
      rc = bn == 32 ? go(dynconv_cells_dgrad_kernel<32>) : bn == 64 ? go(dynconv_cells_dgrad_kernel<64>)
                                                                     : go(dynconv_cells_dgrad_kernel<128>);
      if (rc != BXS_OK) return rc;
    }
  }
  if (g_kernels_host) {
    CellsPlan w = pl;
    for (int l = 0; l < n_levels; ++l) w.out[l] = g_kernels_host[l];
    if (chunks) {
      for (int l = 0; l < n_levels; ++l) {
        const int n = w.start[(l + 1) * B] - w.start[l * B];
        if (n && !make_map(&w.a[l], 3, g_out_host[l], 1, n, w.P[w.op_of(l)], 128)) return BXS_ERR_LAUNCH;
      }
      for (int o = 0; o < n_ops; ++o)
        if (!make_map(&w.b[o], 3, operands_host[o], B, C, w.P[o], (int)C)) return BXS_ERR_LAUNCH;
      const dim3 grid(w.splits, chunks);
      auto go = [&](auto kernel) { return launch(kernel, grid, sizeof(WgSmem) + 1024, st, w, partial); };
      rc = C <= 32    ? go(dynconv_cells_wgrad_kernel<32>)
           : C <= 64  ? go(dynconv_cells_wgrad_kernel<64>)
           : C <= 128 ? go(dynconv_cells_wgrad_kernel<128>)
                      : go(dynconv_cells_wgrad_kernel<256>);
      if (rc != BXS_OK) return rc;
    }
    int64_t total = 0;
    for (int l = 0; l < n_levels; ++l) total += B * (int64_t)w.S2[l];
    dynconv_cells_wgrad_reduce<<<stride_grid(total), 256, 0, st>>>(w, partial, total);
    if ((rc = check_launch()) != BXS_OK) return rc;
  }
  return BXS_OK;
}

// =====================================================================================================================
// 16-bit operands (FP16 or BF16, chosen at compile time), FP32 accumulation in registers: the same three products for
// callers that run in mixed precision (the reference's DiscoBox configs train under autocast), at half the bytes.
//   forward / d/d feat: A = feat^T goes from TMA straight to a shared-memory descriptor.  wgmma transposes 16-bit
//       operands itself (imm-trans-a), so A is read MN-major: [64 channels][64 pixels] boxes with the 128-byte swizzle
//       are the canonical MN-major SW128 layout (64 pixels = 128 bytes per channel row, 8-row groups 1 KB apart).
//       B = kernels, K-major [BN rows][64 channels] boxes, resident for the CTA's lifetime (<= 64 KB).  Each consumer
//       warpgroup rounds its 64 pixels x BN kernels to the operand dtype into a [kernel][64 pixels] shared-memory tile
//       and writes it out in 16-byte pieces, so every output row segment is whole 32-byte sectors.
//   d/d kernel: both operands K-major over the pixels (64 per stage); split-K with FP32 partials, reduced in split
//       order (deterministic) and rounded to the operand dtype only there.
// =====================================================================================================================
namespace bxs {
namespace {

constexpr int H_BLOCK_K = 64;                                // channels (or pixels) per stage: one 128-byte swizzle row
constexpr int H_MMA_K = 16;
constexpr int H_MAX_KBLOCKS = 4;                             // C <= 256
constexpr int H_STAGES = 6;                                  // 96 KB of feat in flight per SM
constexpr int H_BOX_BYTES = 64 * H_BLOCK_K * 2;              // [64 channels][64 pixels]: one warpgroup's A, 8 KB
constexpr int H_A_STAGE_BYTES = BLOCK_M * H_BLOCK_K * 2;     // 16 KB
constexpr int H_B_KBLOCK_BYTES = MAX_N * H_BLOCK_K * 2;      // 16 KB
constexpr int H_OUT_BYTES = MAX_N * 64 * 2;                  // [BN <= 128 kernels][64 pixels] of one warpgroup

struct HSmem {
  alignas(1024) uint8_t a[H_STAGES][H_A_STAGE_BYTES];
  alignas(1024) uint8_t b[H_MAX_KBLOCKS][H_B_KBLOCK_BYTES];
  alignas(16) uint8_t out[2][H_OUT_BYTES];
  alignas(8) uint64_t full[H_STAGES];
  uint64_t empty[H_STAGES];
  uint64_t b_full;
};

// D[64 x 32] += A[64 x 16] * B[32 x 16]^T, both in shared memory, F16 in, FP32 accumulate; TA = 1: A is MN-major
template <int TA>
__device__ __forceinline__ void wgmma_f16_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA));
}
// D[64 x 64] += A[64 x 16] * B[64 x 16]^T, both in shared memory, F16 in, FP32 accumulate; TA = 1: A is MN-major
template <int TA>
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA));
}
// D[64 x 128] += A[64 x 16] * B[128 x 16]^T, both in shared memory, F16 in, FP32 accumulate; TA = 1: A is MN-major
template <int TA>
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA));
}
// D[64 x 256] += A[64 x 16] * B[256 x 16]^T, both in shared memory, F16 in, FP32 accumulate; TA = 1: A is MN-major
template <int TA>
__device__ __forceinline__ void wgmma_f16_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA));
}
// D[64 x 32] += A[64 x 16] * B[32 x 16]^T, both in shared memory, BF16 in, FP32 accumulate; TA = 1: A is MN-major
template <int TA>
__device__ __forceinline__ void wgmma_bf16_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA));
}
// D[64 x 64] += A[64 x 16] * B[64 x 16]^T, both in shared memory, BF16 in, FP32 accumulate; TA = 1: A is MN-major
template <int TA>
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA));
}
// D[64 x 128] += A[64 x 16] * B[128 x 16]^T, both in shared memory, BF16 in, FP32 accumulate; TA = 1: A is MN-major
template <int TA>
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA));
}
// D[64 x 256] += A[64 x 16] * B[256 x 16]^T, both in shared memory, BF16 in, FP32 accumulate; TA = 1: A is MN-major
template <int TA>
__device__ __forceinline__ void wgmma_bf16_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA));
}

template <typename T, int BN, int TA>
__device__ __forceinline__ void wgmma16(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc) {
  if constexpr (std::is_same_v<T, __half>) {
    if constexpr (BN == 32) wgmma_f16_n32<TA>(d, adesc, bdesc);
    else if constexpr (BN == 64) wgmma_f16_n64<TA>(d, adesc, bdesc);
    else if constexpr (BN == 128) wgmma_f16_n128<TA>(d, adesc, bdesc);
    else wgmma_f16_n256<TA>(d, adesc, bdesc);
  } else {
    if constexpr (BN == 32) wgmma_bf16_n32<TA>(d, adesc, bdesc);
    else if constexpr (BN == 64) wgmma_bf16_n64<TA>(d, adesc, bdesc);
    else if constexpr (BN == 128) wgmma_bf16_n128<TA>(d, adesc, bdesc);
    else wgmma_bf16_n256<TA>(d, adesc, bdesc);
  }
}
// the MMA of dynconv_wgrad_body for 16-bit operands (both K-major)
template <typename T>
struct Mma16 {
  template <int BN>
  static __device__ __forceinline__ void mma(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc) {
    wgmma16<T, BN, 0>(d, adesc, bdesc);
  }
};

// wgmma shared-memory descriptor of an MN-major operand with the 128-byte swizzle (PTX ISA, canonical layouts of the
// matrix descriptor): the layout is ((64 MN elements, m), (8 K rows, k)) with the MN index contiguous, a K row every
// 128 bytes, SBO = the stride between groups of 8 K rows (1 KB here) and LBO = the stride between 64-element MN blocks.
// An m64 A operand spans a single MN block, so LBO is never stepped; it is set to the 8 KB box pitch.  The k-th step of
// 16 K rows starts 2 KB further, a whole number of swizzle atoms.
__device__ __forceinline__ uint64_t make_desc_mn(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3fff) | ((uint64_t)(H_BOX_BYTES >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}

// named barrier 1 + wg over the 128 threads of consumer warpgroup wg
__device__ __forceinline__ void warpgroup_bar(int wg) {
  if (wg == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 2, 128;" ::: "memory");
}

// the output tile of a warpgroup: row n (kernel) of 64 pixels = 128 bytes, its 16-byte chunks XOR-swizzled by n % 8 so
// that the accumulator scatter (8 pixels x 4 kernels per warp instruction) and the row read-out are free of conflicts
__device__ __forceinline__ int out_off(int n, int p) { return n * 128 + ((((p >> 3) ^ (n & 7))) << 4) + (p & 7) * 2; }

// grid: (ctas_per_group, B * n_chunks), as dynconv_tf32_kernel
template <typename T, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
dynconv_h_kernel(const __grid_constant__ CUtensorMap tm_feat, const __grid_constant__ CUtensorMap tm_kern,
                 T* __restrict__ out, int C, int P, int I, int n_chunks) {
  extern __shared__ uint8_t smem_raw[];
  HSmem& S = *reinterpret_cast<HSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y / n_chunks, chunk = blockIdx.y % n_chunks;
  const int kblocks = (C + H_BLOCK_K - 1) / H_BLOCK_K;   // channels beyond C are zero-filled by the 3-D tensor map
  const int tiles_m = (P + BLOCK_M - 1) / BLOCK_M;

  if (threadIdx.x == 0) {
    for (int s = 0; s < H_STAGES; ++s) { mbar_init(&S.full[s], 1); mbar_init(&S.empty[s], CONSUMER_WARPS); }
    mbar_init(&S.b_full, 1);
    fence_mbarrier_init();
  }
  __syncthreads();
  if (warp == CONSUMER_WARPS) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_expect_tx(&S.b_full, (uint32_t)kblocks * BN * H_BLOCK_K * 2);
      for (int kb = 0; kb < kblocks; ++kb)
        tma_load_3d(&tm_kern, &S.b_full, S.b[kb], kb * H_BLOCK_K, b * I + chunk * BN, 0);
      int stage = 0, phase = 0;
      for (int mt = blockIdx.x; mt < tiles_m; mt += gridDim.x) {
        for (int kb = 0; kb < kblocks; ++kb) {
          mbar_wait(&S.empty[stage], phase ^ 1);
          mbar_expect_tx(&S.full[stage], H_A_STAGE_BYTES);
#pragma unroll
          for (int g = 0; g < BLOCK_M / 64; ++g)
            tma_load_3d(&tm_feat, &S.full[stage], S.a[stage] + g * H_BOX_BYTES, mt * BLOCK_M + g * 64, kb * H_BLOCK_K, b);
          if (++stage == H_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: wgmma (A MN-major, B K-major) -> shared tile -> global =====================
    const int wg = warp >> 2, w = warp & 3, r = lane >> 2, c4 = lane & 3, t = threadIdx.x & 127;
    uint8_t* tile = S.out[wg];
    mbar_wait(&S.b_full, 0);
    int stage = 0, phase = 0;
    for (int mt = blockIdx.x; mt < tiles_m; mt += gridDim.x) {
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&S.full[stage], phase);
        const uint32_t a_base = smem_u32(S.a[stage] + wg * H_BOX_BYTES), b_base = smem_u32(S.b[kb]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < H_BLOCK_K / H_MMA_K; ++k)
          wgmma16<T, BN, 1>(acc, make_desc_mn(a_base + k * (H_MMA_K * 128)), make_desc(b_base + k * (H_MMA_K * 2)));
        wgmma_commit();
        wgmma_wait_all();
        fence_acc(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&S.empty[stage]);
        if (++stage == H_STAGES) { stage = 0; phase ^= 1; }
      }
      // accumulator elements 4 j .. 4 j + 3: kernels n = 8 j + 2 c4 + {0, 1} of pixels 16 w + r and 16 w + r + 8
      warpgroup_bar(wg);                       // the previous tile has been read out of `tile`
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int n = 8 * j + 2 * c4 + (e & 1), p = 16 * w + r + ((e & 2) ? 8 : 0);
          *reinterpret_cast<T*>(tile + out_off(n, p)) = Operand<T>::round(acc[4 * j + e]);
        }
      }
      warpgroup_bar(wg);
      const int pix = mt * BLOCK_M + wg * 64;
#pragma unroll
      for (int q = 0; q < BN / 16; ++q) {          // BN rows x 8 pieces of 16 bytes, 128 threads
        const int n = 16 * q + (t >> 3), ch = t & 7, i = chunk * BN + n, p = pix + ch * 8;
        if (i < I && p < P)
          *reinterpret_cast<uint4*>(out + ((int64_t)b * I + i) * P + p) = *reinterpret_cast<const uint4*>(tile + out_off(n, ch * 8));
      }
    }
  }
}

// d/d kernel, 16-bit operands: dynconv_wgrad_kernel with 64-pixel K-blocks
template <typename T, int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
dynconv_h_wgrad_kernel(const __grid_constant__ CUtensorMap tm_g, const __grid_constant__ CUtensorMap tm_feat,
                       float* __restrict__ partial, int C, int P, int I, int chunks, int splits, int kb_per_split) {
  dynconv_wgrad_body<BN, Mma16<T>>(DenseWgJob<H_BLOCK_K>(tm_g, tm_feat, partial, C, P, I, chunks, splits, kb_per_split));
}

// the envelope of the 16-bit kernels: TMA needs 16-byte row strides (P % 8) and bases; the output tile is written in
// 16-byte pieces
inline bool half_shape_ok(int64_t B, int64_t C, int64_t P, int64_t I) {
  return C % 32 == 0 && C <= H_BLOCK_K * H_MAX_KBLOCKS && P % 8 == 0 && B * C < (int64_t(1) << 31) &&
         B * I < (int64_t(1) << 31);
}
inline bool known_half(int dtype) { return dtype == BXS_F16 || dtype == BXS_BF16; }

// =====================================================================================================================
// The dense products for every operand dtype: float runs the TF32 kernels, __half and __nv_bfloat16 the 16-bit ones.
//   forward    [B,I,P] = K . F
//   d/d feat   [B,C,P] = K^T . G : the FORWARD kernel with the roles swapped -- "feat" := g_out [B,I,P] (its rows beyond
//       I read as zeros through the 3-D tensor map), "kernels" := K^T zero-padded to a multiple of 32 instances
//       (transpose_pad_kernel, in the workspace).  I <= 256.
//   d/d kernel [B,I,C] = G . F^T : the split-K wgrad kernel + dynconv_wgrad_reduce.
// (the autograd of box_solov2_head.py:209-211, discobox_head.py:1219, box2mask_head.py:345; the reference gets it from
// cuDNN / cuBLAS)
// =====================================================================================================================

// the kernels of operand dtype T
template <typename T>
struct Kernels {
  template <int BN> static constexpr auto fwd = dynconv_h_kernel<T, BN>;
  template <int BN> static constexpr auto wgrad = dynconv_h_wgrad_kernel<T, BN>;
  static constexpr size_t fwd_smem = sizeof(HSmem) + 1024;
  static constexpr int kmap_rank = 3;                 // dynconv_h_kernel loads B with 3-D TMA
};
template <>
struct Kernels<float> {
  template <int BN> static constexpr auto fwd = dynconv_tf32_kernel<BN>;
  template <int BN> static constexpr auto wgrad = dynconv_wgrad_kernel<BN>;
  static constexpr size_t fwd_smem = sizeof(SmemLayout) + 1024;
  static constexpr int kmap_rank = 2;                 // dynconv_tf32_body loads B with 2-D TMA
};

// out[b, i, p] = sum_c kern[b, i, c] * feat3[b, c, p] for c < C; rows c >= feat_rows of feat3 read as zeros
template <typename T>
int dynconv_forward(const T* feat3, int64_t feat_rows, const T* kern, T* out, int64_t B, int64_t C, int64_t P, int64_t I,
                    cudaStream_t st) {
  using K = Kernels<T>;
  const int bn = forward_bn(I), n_chunks = (int)ceil_div(I, bn);
  CUtensorMap tm_feat, tm_kern;
  if (!make_map(&tm_feat, 3, feat3, B, feat_rows, P, KBLOCK<T>) || !make_map(&tm_kern, K::kmap_rank, kern, 1, B * I, C, bn))
    return BXS_ERR_LAUNCH;
  const int64_t groups = B * n_chunks;
  if (groups > 65535) return BXS_ERR_UNSUPPORTED;
  const dim3 grid = persistent_grid(groups, (int)ceil_div(P, BLOCK_M));
  auto go = [&](auto kernel) {
    return launch(kernel, grid, K::fwd_smem, st, tm_feat, tm_kern, out, (int)C, (int)P, (int)I, n_chunks);
  };
  return bn == 32 ? go(K::template fwd<32>) : bn == 64 ? go(K::template fwd<64>) : go(K::template fwd<128>);
}

// d/d kernel split count: about 2 CTAs per SM, at least 256 pixels per CTA
inline int wg_splits(int64_t B, int64_t P, int64_t I, int block_k) {
  const int64_t chunks = ceil_div(I, 128), kb_total = ceil_div(P, block_k);
  int64_t s = std::max<int64_t>(1, (2 * (int64_t)sm_count()) / (B * chunks));
  s = std::min<int64_t>(s, std::max<int64_t>(1, kb_total / (256 / block_k)));   // at least 256 pixels per CTA
  return (int)s;
}

// the workspace of dynconv_backward<T>: K^T padded to 32 instances, then the FP32 partials of the split-K d/d kernel
template <typename T>
int64_t backward_workspace_bytes(int64_t B, int64_t C, int64_t P, int64_t I) {
  const int64_t ipad = ceil_div(I, 32) * 32;
  return (int64_t)sizeof(T) * B * C * ipad + 1024 + 4 * B * (int64_t)wg_splits(B, P, I, KBLOCK<T>) * I * C + 1024;
}

template <typename T>
int dynconv_backward(const T* feat, const T* kernels, const T* g_out, T* g_feat, T* g_kernels, void* workspace, int64_t B,
                     int64_t C, int64_t P, int64_t I, cudaStream_t st) {
  const int64_t ipad = ceil_div(I, 32) * 32;
  T* kt = align1k<T>(workspace);
  float* partial = align1k<float>(kt + B * C * ipad);
  if (g_feat) {
    const int64_t total = B * C * ipad;
    transpose_pad_kernel<<<stride_grid(total), 256, 0, st>>>(kernels, kt, (int)I, (int)C, (int)ipad, total);
    // out[b, c, p] = sum_i kT[b, c, i] * g[b, i, p]: "C" := I (zero-filled up to the K-block), "I" := C
    const int rc = dynconv_forward(g_out, I, kt, g_feat, B, ipad, P, C, st);
    if (rc != BXS_OK) return rc;
  }
  if (g_kernels) {
    const int chunks = (int)ceil_div(I, 128), splits = wg_splits(B, P, I, KBLOCK<T>);
    const int kb_per = (int)ceil_div(ceil_div(P, KBLOCK<T>), splits);
    CUtensorMap tm_g, tm_f;
    if (!make_map(&tm_g, 3, g_out, B, I, P, 128) || !make_map(&tm_f, 3, feat, B, C, P, (int)C)) return BXS_ERR_LAUNCH;
    using K = Kernels<T>;
    const dim3 grid((unsigned)splits, (unsigned)(B * chunks));
    auto go = [&](auto kernel) {
      return launch(kernel, grid, sizeof(WgSmem) + 1024, st, tm_g, tm_f, partial, (int)C, (int)P, (int)I, chunks, splits,
                    kb_per);
    };
    int rc = C <= 32    ? go(K::template wgrad<32>)
             : C <= 64  ? go(K::template wgrad<64>)
             : C <= 128 ? go(K::template wgrad<128>)
                        : go(K::template wgrad<256>);
    if (rc != BXS_OK) return rc;
    const int64_t total = B * I * C;
    dynconv_wgrad_reduce<<<stride_grid(total), 256, 0, st>>>(partial, g_kernels, splits, I * C, total);
    if ((rc = check_launch()) != BXS_OK) return rc;
  }
  return BXS_OK;
}
}  // namespace
}  // namespace bxs

// feat [B,C,P], kernels [B,I,C] -> out [B,I,P] (all float32, contiguous).  Requirements of the TMA/wgmma path:
// C % 32 == 0, C <= 256, P % 4 == 0, 16-byte aligned bases.  BXS_ERR_UNSUPPORTED otherwise.
extern "C" int bxs_dynconv1x1_forward(const float* feat, const float* kernels, float* out, int64_t B, int64_t C, int64_t P,
                                      int64_t I, bxs_stream_t stream) {
  if (!feat || !kernels || !out || B <= 0 || C <= 0 || P <= 0 || I <= 0) return BXS_ERR_INVALID_ARG;
  if (C % BLOCK_K || C > BLOCK_K * MAX_KBLOCKS || P % 4 || !aligned16(feat) || !aligned16(kernels) ||
      B * C >= (int64_t(1) << 31) || B * I >= (int64_t(1) << 31))
    return BXS_ERR_UNSUPPORTED;
  return dynconv_forward(feat, C, kernels, out, B, C, P, I, as_stream(stream));
}

// workspace: bxs_dynconv1x1_backward_workspace_bytes(B, C, P, I) bytes
extern "C" int64_t bxs_dynconv1x1_backward_workspace_bytes(int64_t B, int64_t C, int64_t P, int64_t I) {
  if (B <= 0 || C <= 0 || P <= 0 || I <= 0) return 0;
  return backward_workspace_bytes<float>(B, C, P, I);
}

extern "C" int bxs_dynconv1x1_backward(const float* feat, const float* kernels, const float* g_out, float* g_feat,
                                       float* g_kernels, void* workspace, int64_t B, int64_t C, int64_t P, int64_t I,
                                       bxs_stream_t stream) {
  if (!feat || !kernels || !g_out || (!g_feat && !g_kernels) || !workspace || B <= 0 || C <= 0 || P <= 0 || I <= 0)
    return BXS_ERR_INVALID_ARG;
  if (C % BLOCK_K || C > BLOCK_K * MAX_KBLOCKS || P % 4 || (g_feat && I > 256) || !aligned16(feat) || !aligned16(g_out) ||
      !aligned16(kernels))
    return BXS_ERR_UNSUPPORTED;
  return dynconv_backward(feat, kernels, g_out, g_feat, g_kernels, workspace, B, C, P, I, as_stream(stream));
}

extern "C" int bxs_dynconv1x1_half_forward(const void* feat, const void* kernels, void* out, int64_t B, int64_t C,
                                           int64_t P, int64_t I, int dtype, bxs_stream_t stream) {
  if (!feat || !kernels || !out || B <= 0 || C <= 0 || P <= 0 || I <= 0 || !known_half(dtype)) return BXS_ERR_INVALID_ARG;
  if (!half_shape_ok(B, C, P, I) || !aligned16(feat) || !aligned16(kernels) || !aligned16(out)) return BXS_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  if (dtype == BXS_F16)
    return dynconv_forward(static_cast<const __half*>(feat), C, static_cast<const __half*>(kernels),
                           static_cast<__half*>(out), B, C, P, I, st);
  return dynconv_forward(static_cast<const __nv_bfloat16*>(feat), C, static_cast<const __nv_bfloat16*>(kernels),
                         static_cast<__nv_bfloat16*>(out), B, C, P, I, st);
}

// the same for both 16-bit dtypes
extern "C" int64_t bxs_dynconv1x1_half_backward_workspace_bytes(int64_t B, int64_t C, int64_t P, int64_t I, int dtype) {
  if (B <= 0 || C <= 0 || P <= 0 || I <= 0 || !known_half(dtype)) return 0;
  return backward_workspace_bytes<__half>(B, C, P, I);
}

extern "C" int bxs_dynconv1x1_half_backward(const void* feat, const void* kernels, const void* g_out, void* g_feat,
                                            void* g_kernels, void* workspace, int64_t B, int64_t C, int64_t P, int64_t I,
                                            int dtype, bxs_stream_t stream) {
  if (!feat || !kernels || !g_out || (!g_feat && !g_kernels) || !workspace || B <= 0 || C <= 0 || P <= 0 || I <= 0 ||
      !known_half(dtype))
    return BXS_ERR_INVALID_ARG;
  if (!half_shape_ok(B, C, P, I) || (g_feat && I > 256) || !aligned16(feat) || !aligned16(kernels) || !aligned16(g_out) ||
      !aligned16(g_feat))
    return BXS_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  if (dtype == BXS_F16)
    return dynconv_backward(static_cast<const __half*>(feat), static_cast<const __half*>(kernels),
                            static_cast<const __half*>(g_out), static_cast<__half*>(g_feat),
                            static_cast<__half*>(g_kernels), workspace, B, C, P, I, st);
  return dynconv_backward(static_cast<const __nv_bfloat16*>(feat), static_cast<const __nv_bfloat16*>(kernels),
                          static_cast<const __nv_bfloat16*>(g_out), static_cast<__nv_bfloat16*>(g_feat),
                          static_cast<__nv_bfloat16*>(g_kernels), workspace, B, C, P, I, st);
}
