// sm_90a tensor-core plumbing: wgmma / mbarrier / bulk-copy PTX wrappers, the shared-memory descriptor
// encoding and the accumulator-fragment helpers used by the implicit-GEMM kernels.
//
// Operand layout used throughout ("panel" layout = the canonical K-major SWIZZLE_NONE /
// INTERLEAVE layout with SBO = 128 B):
//     element (row r, k)  ->  byte  (k/8) * (ROWS*16)  +  r*16  +  (k%8)*2        (bf16)
// i.e. one 16-byte K-chunk per row, rows contiguous, K-chunks ROWS*16 bytes apart.  With the
// 8-row-group stride (SBO) equal to 8*16 B the address is linear in r, so a descriptor whose
// start address is advanced by s*16 bytes addresses rows s..s+M-1: a convolution tap is a
// descriptor offset, not a data copy.  This is wgmma's canonical K-major no-swizzle layout (8 x 16-byte core
// matrices; LBO = K-direction stride, SBO = row-group stride).
//
// A warpgroup (4 warps) issues m64nNk16 MMAs: a 128-row tile is two warpgroups of 64 rows each, with the fp32
// accumulators in registers.  Fragment of thread t (warp w = t/32 of its warpgroup, lane l): d[4i + e] is row
// 16w + l/4 + 8*(e/2), column 8i + 2*(l%4) + (e%2).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace svcb {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// Bounded spin: a protocol bug traps (kernel error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  for (uint32_t spin = 0; spin < (1u << 28); ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(phase)
        : "memory");
    if (done) return;
  }
  __trap();
}

// The same wait for warps that share an SM with busy CUDA-core warps: the suspend-time hint lets the
// hardware park the thread until the phase flips (or ~20 us pass) instead of re-issuing try_wait + branch
// every few hundred cycles — in amp_s2d_link those spin instructions were 12 % of everything issued.
__device__ __forceinline__ void mbar_wait_parked(uint64_t* bar, uint32_t phase) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  for (uint32_t spin = 0; spin < (1u << 22); ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(phase), "r"(20000u)
        : "memory");
    if (done) return;
  }
  __trap();
}

// ---- proxies / bulk copy (TMA engine, 1-D)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---- descriptors
// K-major, no swizzle, SBO = 128 B; lbo_bytes = distance between consecutive 16-byte K-chunks.
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes = 128u) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;               // base_offset 0, layout_type 0 (interleave = no swizzle)
}

// ---- warpgroup MMA control
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across a wgmma.wait_group
template <int R>
__device__ __forceinline__ void wg_hold(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- wgmma wrappers, m64nNk16, bf16 x bf16 -> fp32, N = 16 .. 256 in steps of 16 (A from registers: N = 64, 96)
#define SVCB_F4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define SVCB_F8(i) SVCB_F4(i), SVCB_F4(i + 4)
#define SVCB_R8_0 "%0, %1, %2, %3, %4, %5, %6, %7"
#define SVCB_R8_8 "%8, %9, %10, %11, %12, %13, %14, %15"
#define SVCB_R8_16 "%16, %17, %18, %19, %20, %21, %22, %23"
#define SVCB_R8_24 "%24, %25, %26, %27, %28, %29, %30, %31"
#define SVCB_R8_32 "%32, %33, %34, %35, %36, %37, %38, %39"
#define SVCB_R8_40 "%40, %41, %42, %43, %44, %45, %46, %47"
#define SVCB_R8_48 "%48, %49, %50, %51, %52, %53, %54, %55"
#define SVCB_R8_56 "%56, %57, %58, %59, %60, %61, %62, %63"
#define SVCB_R8_64 "%64, %65, %66, %67, %68, %69, %70, %71"
#define SVCB_R8_72 "%72, %73, %74, %75, %76, %77, %78, %79"
#define SVCB_R8_80 "%80, %81, %82, %83, %84, %85, %86, %87"
#define SVCB_R8_88 "%88, %89, %90, %91, %92, %93, %94, %95"
#define SVCB_R8_96 "%96, %97, %98, %99, %100, %101, %102, %103"
#define SVCB_R8_104 "%104, %105, %106, %107, %108, %109, %110, %111"
#define SVCB_R8_112 "%112, %113, %114, %115, %116, %117, %118, %119"
#define SVCB_R8_120 "%120, %121, %122, %123, %124, %125, %126, %127"
template <int N, int TB> struct Wg;   // TB: B operand MN-major (1) or K-major (0)
template <int TB> struct Wg<16, TB> {
  static __device__ __forceinline__ void ss(float (&d)[8], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\nwgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {" SVCB_R8_0
                 "}, %8, %9, p, 1, 1, 0, %11;\n}\n" : SVCB_F8(0) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<24, TB> {
  static __device__ __forceinline__ void ss(float (&d)[12], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %14, 0;\nwgmma.mma_async.sync.aligned.m64n24k16.f32.bf16.bf16 {" SVCB_R8_0
                 ", %8, %9, %10, %11}, %12, %13, p, 1, 1, 0, %15;\n}\n" : SVCB_F8(0), SVCB_F4(8) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<32, TB> {
  static __device__ __forceinline__ void ss(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\nwgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8
                 "}, %16, %17, p, 1, 1, 0, %19;\n}\n" : SVCB_F8(0), SVCB_F8(8) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<48, TB> {
  static __device__ __forceinline__ void ss(float (&d)[24], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\nwgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16
                 "}, %24, %25, p, 1, 1, 0, %27;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<64, TB> {
  static __device__ __forceinline__ void ss(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\nwgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24
                 "}, %32, %33, p, 1, 1, 0, %35;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
  static __device__ __forceinline__ void rs(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\nwgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24
                 "}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<80, TB> {
  static __device__ __forceinline__ void ss(float (&d)[40], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %42, 0;\nwgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32
                 "}, %40, %41, p, 1, 1, 0, %43;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<96, TB> {
  static __device__ __forceinline__ void ss(float (&d)[48], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %50, 0;\nwgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40
                 "}, %48, %49, p, 1, 1, 0, %51;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
  static __device__ __forceinline__ void rs(float (&d)[48], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %53, 0;\nwgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40
                 "}, {%48, %49, %50, %51}, %52, p, 1, 1, %54;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<112, TB> {
  static __device__ __forceinline__ void ss(float (&d)[56], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %58, 0;\nwgmma.mma_async.sync.aligned.m64n112k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40 ", " SVCB_R8_48
                 "}, %56, %57, p, 1, 1, 0, %59;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40), SVCB_F8(48) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<128, TB> {
  static __device__ __forceinline__ void ss(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\nwgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40 ", " SVCB_R8_48 ", " SVCB_R8_56
                 "}, %64, %65, p, 1, 1, 0, %67;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40), SVCB_F8(48), SVCB_F8(56) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<144, TB> {
  static __device__ __forceinline__ void ss(float (&d)[72], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %74, 0;\nwgmma.mma_async.sync.aligned.m64n144k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40 ", " SVCB_R8_48 ", " SVCB_R8_56 ", " SVCB_R8_64
                 "}, %72, %73, p, 1, 1, 0, %75;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40), SVCB_F8(48), SVCB_F8(56), SVCB_F8(64) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<160, TB> {
  static __device__ __forceinline__ void ss(float (&d)[80], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %82, 0;\nwgmma.mma_async.sync.aligned.m64n160k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40 ", " SVCB_R8_48 ", " SVCB_R8_56 ", " SVCB_R8_64 ", " SVCB_R8_72
                 "}, %80, %81, p, 1, 1, 0, %83;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40), SVCB_F8(48), SVCB_F8(56), SVCB_F8(64), SVCB_F8(72) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<176, TB> {
  static __device__ __forceinline__ void ss(float (&d)[88], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %90, 0;\nwgmma.mma_async.sync.aligned.m64n176k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40 ", " SVCB_R8_48 ", " SVCB_R8_56 ", " SVCB_R8_64 ", " SVCB_R8_72 ", " SVCB_R8_80
                 "}, %88, %89, p, 1, 1, 0, %91;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40), SVCB_F8(48), SVCB_F8(56), SVCB_F8(64), SVCB_F8(72), SVCB_F8(80) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<192, TB> {
  static __device__ __forceinline__ void ss(float (&d)[96], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %98, 0;\nwgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40 ", " SVCB_R8_48 ", " SVCB_R8_56 ", " SVCB_R8_64 ", " SVCB_R8_72 ", " SVCB_R8_80 ", " SVCB_R8_88
                 "}, %96, %97, p, 1, 1, 0, %99;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40), SVCB_F8(48), SVCB_F8(56), SVCB_F8(64), SVCB_F8(72), SVCB_F8(80), SVCB_F8(88) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<208, TB> {
  static __device__ __forceinline__ void ss(float (&d)[104], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %106, 0;\nwgmma.mma_async.sync.aligned.m64n208k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40 ", " SVCB_R8_48 ", " SVCB_R8_56 ", " SVCB_R8_64 ", " SVCB_R8_72 ", " SVCB_R8_80 ", " SVCB_R8_88 ", " SVCB_R8_96
                 "}, %104, %105, p, 1, 1, 0, %107;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40), SVCB_F8(48), SVCB_F8(56), SVCB_F8(64), SVCB_F8(72), SVCB_F8(80), SVCB_F8(88), SVCB_F8(96) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<224, TB> {
  static __device__ __forceinline__ void ss(float (&d)[112], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %114, 0;\nwgmma.mma_async.sync.aligned.m64n224k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40 ", " SVCB_R8_48 ", " SVCB_R8_56 ", " SVCB_R8_64 ", " SVCB_R8_72 ", " SVCB_R8_80 ", " SVCB_R8_88 ", " SVCB_R8_96 ", " SVCB_R8_104
                 "}, %112, %113, p, 1, 1, 0, %115;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40), SVCB_F8(48), SVCB_F8(56), SVCB_F8(64), SVCB_F8(72), SVCB_F8(80), SVCB_F8(88), SVCB_F8(96), SVCB_F8(104) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<240, TB> {
  static __device__ __forceinline__ void ss(float (&d)[120], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %122, 0;\nwgmma.mma_async.sync.aligned.m64n240k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40 ", " SVCB_R8_48 ", " SVCB_R8_56 ", " SVCB_R8_64 ", " SVCB_R8_72 ", " SVCB_R8_80 ", " SVCB_R8_88 ", " SVCB_R8_96 ", " SVCB_R8_104 ", " SVCB_R8_112
                 "}, %120, %121, p, 1, 1, 0, %123;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40), SVCB_F8(48), SVCB_F8(56), SVCB_F8(64), SVCB_F8(72), SVCB_F8(80), SVCB_F8(88), SVCB_F8(96), SVCB_F8(104), SVCB_F8(112) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
template <int TB> struct Wg<256, TB> {
  static __device__ __forceinline__ void ss(float (&d)[128], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\nwgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {" SVCB_R8_0 ", " SVCB_R8_8 ", " SVCB_R8_16 ", " SVCB_R8_24 ", " SVCB_R8_32 ", " SVCB_R8_40 ", " SVCB_R8_48 ", " SVCB_R8_56 ", " SVCB_R8_64 ", " SVCB_R8_72 ", " SVCB_R8_80 ", " SVCB_R8_88 ", " SVCB_R8_96 ", " SVCB_R8_104 ", " SVCB_R8_112 ", " SVCB_R8_120
                 "}, %128, %129, p, 1, 1, 0, %131;\n}\n" : SVCB_F8(0), SVCB_F8(8), SVCB_F8(16), SVCB_F8(24), SVCB_F8(32), SVCB_F8(40), SVCB_F8(48), SVCB_F8(56), SVCB_F8(64), SVCB_F8(72), SVCB_F8(80), SVCB_F8(88), SVCB_F8(96), SVCB_F8(104), SVCB_F8(112), SVCB_F8(120) : "l"(da), "l"(db), "r"(acc), "n"(TB));
  }
};
#undef SVCB_R8_0
#undef SVCB_R8_8
#undef SVCB_R8_16
#undef SVCB_R8_24
#undef SVCB_R8_32
#undef SVCB_R8_40
#undef SVCB_R8_48
#undef SVCB_R8_56
#undef SVCB_R8_64
#undef SVCB_R8_72
#undef SVCB_R8_80
#undef SVCB_R8_88
#undef SVCB_R8_96
#undef SVCB_R8_104
#undef SVCB_R8_112
#undef SVCB_R8_120
#undef SVCB_F8
#undef SVCB_F4

// D (+)= A . B^T over nk K-steps of 16: A from a K-major panel (lbo_a, K step 2*lbo_a), B K-major (lbo_b)
template <int N>
__device__ __forceinline__ void wg_mma_k(float (&d)[N / 2], uint32_t a_addr, uint32_t lbo_a, uint32_t b_addr, uint32_t lbo_b, int nk,
                                         uint32_t first_acc) {
  const uint64_t da = smem_desc(a_addr, lbo_a), db = smem_desc(b_addr, lbo_b);
  const uint64_t sa = (uint64_t)((2u * lbo_a) >> 4), sb = (uint64_t)((2u * lbo_b) >> 4);
  for (int kk = 0; kk < nk; ++kk) Wg<N, 0>::ss(d, da + kk * sa, db + kk * sb, kk ? 1u : first_acc);
}

// accumulator fragment (64 x N of this warpgroup) -> row-major fp32 rows buf[row * ld + col] for the 8-column groups
// [g0, g1) (col relative to 8 * g0); rows 0..63 of the warpgroup
template <int N>
__device__ __forceinline__ void acc_to_smem(const float (&d)[N / 2], float* buf, int ld, int g0, int g1) {
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
  const int r = 16 * w + (l >> 2), c = 2 * (l & 3) - 8 * g0;
#pragma unroll
  for (int i = 0; i < N / 8; ++i) {
    if (i >= g0 && i < g1) {
      *reinterpret_cast<float2*>(buf + r * ld + 8 * i + c) = make_float2(d[4 * i], d[4 * i + 1]);
      *reinterpret_cast<float2*>(buf + (r + 8) * ld + 8 * i + c) = make_float2(d[4 * i + 2], d[4 * i + 3]);
    }
  }
}

// named barrier over `count` threads (a multiple of 32)
__device__ __forceinline__ void named_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P1;\n\telect.sync _|P1, 0xffffffff;\n\tselp.b32 %0, 1, 0, P1;\n\t}" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ int warp_uniform_idx() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

}  // namespace tc
}  // namespace svcb
