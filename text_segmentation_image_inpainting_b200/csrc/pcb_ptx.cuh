// pcb_ptx.cuh -- inline-PTX wrappers for the Hopper (sm_90a) async machinery used by the
// tensor-core kernels: mbarrier, TMA (cp.async.bulk.tensor), cp.async (LDGSTS), wgmma.
// No CUTLASS dependency: these are the raw instructions.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a pipeline bug becomes a reported error instead of a hung GPU.  `*abort_flag`
// (global memory) is set and the wait gives up after ~2 s of SM clocks; callers bail out.
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity, int *abort_flag, int code) {
    if (mbar_try_wait(bar, parity)) return true;
    const long long t0 = clock64();
    for (uint32_t it = 1;; ++it) {
        if (mbar_try_wait(bar, parity)) return true;
        if ((it & 63) == 0) {
            if (*reinterpret_cast<volatile int *>(abort_flag) != 0) return false;
            if (clock64() - t0 > 4000000000ll) break;          // ~2 s at 2 GHz
        }
    }
    atomicCAS(abort_flag, 0, code);
    return false;
}
// cp.async completion -> mbarrier: pending count +1 now, -1 when this thread's prior cp.asyncs land.
__device__ __forceinline__ void cp_async_mbar_arrive(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}

// ---------------------------------------------------------------- cp.async (LDGSTS), 16 B with zero fill
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void *src, bool valid) {
    const uint32_t sz = valid ? 16u : 0u;   // src-size 0 => 16 zero bytes are written
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
// the same through L1 (.ca): for gathers that read each source line several times within one stage
__device__ __forceinline__ void cp_async_16_ca(uint32_t dst, const void *src, bool valid) {
    const uint32_t sz = valid ? 16u : 0u;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// generic-proxy writes (st.shared / cp.async) -> async-proxy readers (TMA store, wgmma)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *m, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
// 4-D tile (channels, x, y, image): out-of-range coordinates (negative included) are zero-filled -- the conv padding
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap *m, int c0, int c1, int c2, int c3, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---------------------------------------------------------------- wgmma (Hopper warpgroup MMA)
// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 x bf16 -> fp32 register accumulators, issued by all 128 threads of one
// warpgroup.  TA / TB: 0 = K-major operand, 1 = MN-major operand.  Accumulator fragment of thread t (warp w = t / 32 of the
// warpgroup, lane l): d[i] is row 16 w + l / 4 + 8 ((i / 2) & 1), column 8 (i / 4) + 2 (l % 4) + (i & 1).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulator registers must not be touched by the compiler while MMAs are in flight
template <int R> __device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int TA, int TB> __device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1, 1, 1, %18, %19;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a_desc), "l"(b_desc), "n"(TA), "n"(TB));
}
// d may be a wider accumulator array: its first 32 registers are the 64 columns
template <int TA, int TB, int R> __device__ __forceinline__ void wgmma_m64n64(float (&d)[R], uint64_t a_desc, uint64_t b_desc) {
    static_assert(R >= 32, "m64n64 accumulator");
    asm volatile(
        "{\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1, %34, %35;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "n"(TA), "n"(TB));
}
template <int TA, int TB> __device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, %66, %67;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "n"(TA), "n"(TB));
}
// N = 256 is issued as two m64n128 halves (columns [0, 128) into d[0..63], [128, 256) into d[64..127]) over a K-major B tile
// whose rows are 128 bytes apart, so the second half starts 128 rows = 16 KB further.  One m64n256 instruction would need
// ~154 registers at once, and ptxas checks an instruction against the kernel's launch register limit (128 at 512 threads)
// even inside a setmaxnreg region; the accumulators themselves may exceed it there.
template <int N, int TA, int TB> __device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc) {
    if constexpr (N == 32) wgmma_m64n32<TA, TB>(d, a_desc, b_desc);
    else if constexpr (N == 64) wgmma_m64n64<TA, TB>(d, a_desc, b_desc);
    else if constexpr (N == 128) wgmma_m64n128<TA, TB>(d, a_desc, b_desc);
    else {
        static_assert(N == 256 && TB == 0, "wgmma tile width");
        wgmma_m64n128<TA, TB>(*reinterpret_cast<float (*)[64]>(&d[0]), a_desc, b_desc);
        wgmma_m64n128<TA, TB>(*reinterpret_cast<float (*)[64]>(&d[64]), a_desc, b_desc + (16384 >> 4));
    }
}
// ---------------------------------------------------------------- register reallocation (per warpgroup)
// setmaxnreg: all four warps of a warpgroup execute it (.sync.aligned).  dec returns registers to the CTA's pool, inc blocks
// until the pool holds enough; N is a multiple of 8 in [24, 256].
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
// named barrier over the `threads` threads of one role (id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// ---------------------------------------------------------------- descriptors
// Shared-memory matrix descriptor (64-bit), sm_90 wgmma format:
//   [ 0,14) start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4   [49,52) base offset   [62,64) layout: 0 none, 1 SWIZZLE_128B, 2 64B, 3 32B
// Tiles here are "row = 128 bytes, 8 rows = one 1024-byte swizzle atom" (what TMA SWIZZLE_128B and the
// software gather both produce):
//   K-major  operand: rows are M/N, the 128 B are 64 bf16 of K  -> SBO = 1024 (next 8 rows), LBO unused (1).
//   MN-major operand: rows are K,   the 128 B are 64 bf16 of M/N -> SBO = 1024 (next 8 k-rows),
//                                                                  LBO = byte distance to the next 64 M/N.
__host__ __device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= 1ull << 62;     // SWIZZLE_128B
    return d;
}

}  // namespace ptx
