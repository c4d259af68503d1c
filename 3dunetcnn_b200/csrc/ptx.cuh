// Thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA) and its shared-memory descriptors.
// Everything here is hand-written PTX; no CUTLASS/CuTe dependency.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cuda.h>
#include <cuda_bf16.h>

namespace b200 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug turns into a trapped launch (cudaErrorLaunchFailure) after ~10 s instead of a hung GPU.
#ifndef B200_SPIN_LIMIT_CYCLES
#define B200_SPIN_LIMIT_CYCLES 20000000000ll
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t n = 0;
  while (!mbar_try_wait(bar, parity)) {
    // no printf here: a call inside the wgmma consumers' loop would make ptxas serialise every wgmma
    if (((++n) & 0x3FFF) == 0 && clock64() - t0 > B200_SPIN_LIMIT_CYCLES) asm volatile("trap;");
  }
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// TMA store (shared -> global tile, bulk async group completion)
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2, int c3,
                                             int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// predicated forms: convergent producer loops, one elected lane (elect_one(), evaluated once) issues
__device__ __forceinline__ void mbar_expect_tx_if(uint32_t issue, uint64_t* bar, uint32_t bytes) {
  asm volatile(
      "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\t"
      "@q mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}\n"
      ::"r"(smem_u32(bar)), "r"(bytes), "r"(issue)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d_if(uint32_t issue, void* smem_dst, const CUtensorMap* map, uint64_t* bar,
                                               int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %8, 0;\n\t"
      "@q cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];\n\t}\n"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3), "r"(c4), "r"(issue)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d_if(uint32_t issue, void* smem_dst, const CUtensorMap* map, uint64_t* bar,
                                               int c0, int c1, int c2) {
  asm volatile(
      "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %6, 0;\n\t"
      "@q cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n\t}\n"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(issue)
      : "memory");
}

// ----------------------------------------------------------------------------- programmatic dependent launch
// (common.cuh: launch_pdl).  pdl_wait: returns once the preceding kernel of the stream has completed and its memory operations
// are visible (immediately when this grid was not launched with the attribute).  pdl_launch_dependents: this CTA no longer
// holds back the launch of the next kernel.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ----------------------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 operands from shared memory (descriptors), fp32 accumulator in the registers of
// the four warps of a warpgroup.  Thread t of the warpgroup (warp w = t / 32, lane l) holds, for every 8-column block i,
// d[4i + 0..1] = row 16w + l/4, columns 8i + 2(l%4) + {0, 1} and d[4i + 2..3] = the same columns of row 16w + l/4 + 8.
// TA / TB = 1: the operand is MN-major (the contraction index is the slow axis of its shared-memory tile).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <int N>
struct Wgmma;
template <>
struct Wgmma<16> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <>
struct Wgmma<32> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <>
struct Wgmma<64> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <>
struct Wgmma<128> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};

// ----------------------------------------------------------------------------- wgmma shared-memory descriptors
//   bits [0,14)  start address >> 4        bits [16,30) leading-dim byte offset >> 4
//   bits [32,46) stride-dim byte offset >> 4   bits [49,52) base offset   bits [62,64) layout: 0 none, 1 SW128, 2 SW64, 3 SW32
// K-major swizzled tiles: SBO = bytes between 8-row groups (LBO unused); MN-major swizzled tiles: LBO = bytes between
// swizzle atoms along M/N, SBO = bytes between 8-row groups along K.  A K step inside a swizzle atom adds its byte offset to the
// start address (the hardware applies the swizzle on absolute address bits; tiles are 1024-byte aligned).
enum : uint32_t { GMMA_SW_NONE = 0, GMMA_SW128 = 1, GMMA_SW64 = 2, GMMA_SW32 = 3 };

__host__ __device__ constexpr uint32_t desc_hi(uint32_t sbo_bytes, uint32_t layout) {
  return ((sbo_bytes >> 4) & 0x3FFF) | ((layout & 3u) << 30);
}
__device__ __forceinline__ uint32_t desc_lo(uint32_t smem_addr, uint32_t lbo_bytes) {
  return ((smem_addr >> 4) & 0x3FFF) | (((lbo_bytes >> 4) & 0x3FFF) << 16);
}
__device__ __forceinline__ uint64_t desc_from(uint32_t lo, uint32_t hi) {
  return (static_cast<uint64_t>(hi) << 32) | lo;
}
__host__ __device__ constexpr uint32_t swizzle_for_row_bytes(int bytes) {
  return bytes >= 128 ? GMMA_SW128 : bytes >= 64 ? GMMA_SW64 : GMMA_SW32;
}

// ----------------------------------------------------------------------------- misc numeric helpers
__device__ __forceinline__ float bf16_lo_to_f(uint32_t packed) { return __uint_as_float(packed << 16); }
__device__ __forceinline__ float bf16_hi_to_f(uint32_t packed) { return __uint_as_float(packed & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// 8 consecutive channels (one 16-byte vector) of a bf16 tensor: value = hi (+ lo in split precision, lo != nullptr)
__device__ __forceinline__ void load8(const __nv_bfloat16* hi, const __nv_bfloat16* lo, long long off, float (&v)[8]) {
  uint4 a = *reinterpret_cast<const uint4*>(hi + off);
  v[0] = bf16_lo_to_f(a.x); v[1] = bf16_hi_to_f(a.x);
  v[2] = bf16_lo_to_f(a.y); v[3] = bf16_hi_to_f(a.y);
  v[4] = bf16_lo_to_f(a.z); v[5] = bf16_hi_to_f(a.z);
  v[6] = bf16_lo_to_f(a.w); v[7] = bf16_hi_to_f(a.w);
  if (lo) {
    uint4 b = *reinterpret_cast<const uint4*>(lo + off);
    v[0] += bf16_lo_to_f(b.x); v[1] += bf16_hi_to_f(b.x);
    v[2] += bf16_lo_to_f(b.y); v[3] += bf16_hi_to_f(b.y);
    v[4] += bf16_lo_to_f(b.z); v[5] += bf16_hi_to_f(b.z);
    v[6] += bf16_lo_to_f(b.w); v[7] += bf16_hi_to_f(b.w);
  }
}

// hi = bf16(v), lo = bf16(v - hi), both round-to-nearest-even
__device__ __forceinline__ void store8(__nv_bfloat16* hi, __nv_bfloat16* lo, long long off, const float (&v)[8]) {
  uint4 a;
  a.x = pack_bf16x2(v[0], v[1]); a.y = pack_bf16x2(v[2], v[3]);
  a.z = pack_bf16x2(v[4], v[5]); a.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(hi + off) = a;
  if (lo) {
    uint4 b;
    b.x = pack_bf16x2(v[0] - bf16_lo_to_f(a.x), v[1] - bf16_hi_to_f(a.x));
    b.y = pack_bf16x2(v[2] - bf16_lo_to_f(a.y), v[3] - bf16_hi_to_f(a.y));
    b.z = pack_bf16x2(v[4] - bf16_lo_to_f(a.z), v[5] - bf16_hi_to_f(a.z));
    b.w = pack_bf16x2(v[6] - bf16_lo_to_f(a.w), v[7] - bf16_hi_to_f(a.w));
    *reinterpret_cast<uint4*>(lo + off) = b;
  }
}

}  // namespace b200
