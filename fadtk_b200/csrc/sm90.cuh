// sm_90a device primitives used by every tensor-core kernel in this library:
// mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA (wgmma.mma_async) and its shared-memory
// matrix descriptor, and the fp64 mma.sync the DMMA kernels use.
//
// Everything is inline PTX; nothing here depends on CUTLASS.  Bit layouts follow the PTX ISA
// "wgmma matrix descriptor" table.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

namespace sm90 {

// ----------------------------------------------------------------------------- misc
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(pred));
    return pred != 0;
}

// ------------------------------------------------- register redistribution (per warpgroup)
template <uint32_t kRegs> __device__ __forceinline__ void setmaxnreg_inc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs));
}
template <uint32_t kRegs> __device__ __forceinline__ void setmaxnreg_dec() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs));
}

// named barrier over `count` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// explicit shared-memory 16-B accesses by 32-bit shared address: a pointer derived from the aligned dynamic-smem base
// loses its address space, and the compiler then emits GENERIC ST.E / LD.E (long-scoreboard, slower than STS / LDS)
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts64(uint32_t addr, float x, float y) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x), "f"(y) : "memory");
}

// ------------------------------------------------------------------- fp64 tensor pipe
// {c0, c1} += a b: mma.sync m8n8k4 f64 (SASS DMMA.8x8x4), the fp64 MMA shape of sm_90a (wgmma has no f64 kind).
// Fragments: A lane -> row lane/4, k lane%4; B k lane%4, col lane/4; C row lane/4, cols 2 (lane%4) + {0, 1}.
__device__ __forceinline__ void dmma_884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// ------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
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
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// Watchdog: no wait in this library is legitimately longer than a few milliseconds; a protocol
// bug traps (-> cudaErrorLaunchFailure on the host) instead of hanging the GPU.  Kept free of
// function calls (no printf) so ptxas can give each warp role its own setmaxnreg budget.
// The retry loop is four instructions (try_wait with a suspend-time hint, counter, compare, branch): waiting warps
// share their scheduler with working ones.
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(ns) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    uint32_t spins = 0;
    while (!mbar_try_wait_hint(bar, parity, 2000u)) {          // may suspend up to 2 us per try; resumes on completion
        if (++spins > (1u << 24)) asm volatile("trap;");       // >= 0.3 s of retries
    }
}

// ------------------------------------------------------------------------- clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// index of this CTA's cluster in the (1-D) grid; a volatile read, so a caller can re-read it where it needs it instead of
// keeping one copy live through code that is short of registers
__device__ __forceinline__ uint32_t cluster_index() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
    return r;
}
// every thread of every CTA in the cluster; not .aligned, so a warp may reach it diverged
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster (that CTA may be this one)
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
    asm volatile(
        "{\n\t.reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}\n"
        ::"r"(smem_u32(bar)), "r"(cta) : "memory");
}

// generic-proxy writes to smem -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ------------------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)),
          "r"(c0), "r"(c1) : "memory");
}
// the same box into the shared memory of every CTA in `cta_mask` (bit i = cluster rank i), at the same offset, each
// completing its bytes on the mbarrier at the same offset in that CTA
__device__ __forceinline__ void tma_load_2d_multicast(void* dst, const CUtensorMap* m, uint64_t* bar,
                                                      int c0, int c1, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)),
          "r"(c0), "r"(c1), "h"(cta_mask) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)),
          "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)),
          "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// ------------------------------------------------------------------- wgmma descriptors
// Shared-memory matrix descriptor (64 bit):
//   [ 0,14) start address >> 4      [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4      [49,52) base offset (0: tiles are 1024-B aligned)
//   [62,64) layout: 1 = 128-B swizzle, 2 = 64-B swizzle, 3 = 32-B swizzle
enum : uint64_t { SWZ_NONE = 0, SWZ_128B = 1, SWZ_64B = 2, SWZ_32B = 3 };

__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes,
                                                   uint32_t sbo_bytes, uint64_t swizzle) {
    return  (uint64_t)((saddr & 0x3FFFF) >> 4)
          | ((uint64_t)(lbo_bytes >> 4) << 16)
          | ((uint64_t)(sbo_bytes >> 4) << 32)
          | (swizzle << 62);
}

// K-major operand tile written by TMA with SWIZZLE_128B: rows of 128 B (64 x 16-bit elements),
// 8-row swizzle atoms of 1024 B stacked along M/N.  LBO is unused for swizzled K-major layouts
// (encoded 1), SBO = 1024 B.  Advancing along K inside the 128-B atom = adding the byte offset to
// the start address (+32 B per 16 fp16 elements = +2 in the 16-B address field).
__device__ __forceinline__ uint64_t kmajor_sw128_desc(uint32_t saddr) {
    return make_smem_desc(saddr, 16, 1024, SWZ_128B);
}
// MN-major operand tile, SWIZZLE_128B, 16-bit elements: each K row holds 64 contiguous M/N
// elements (128 B); 8 K-rows form a 1024-B atom.  LBO = stride between successive 64-element
// blocks along M/N, SBO = stride between 8-row K groups.
__device__ __forceinline__ uint64_t mnmajor_sw128_desc(uint32_t saddr, uint32_t lbo_bytes,
                                                       uint32_t sbo_bytes) {
    return make_smem_desc(saddr, lbo_bytes, sbo_bytes, SWZ_128B);
}

// ------------------------------------------------------------------------- wgmma
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int N> __device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define FAD_WG_D64                                                                                                 \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                    \
    "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                            \
    "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                            \
    "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define FAD_WG_OUT64(d)                                                                                            \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),                \
    "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),          \
    "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),        \
    "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),        \
    "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),        \
    "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),        \
    "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),        \
    "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

// D[64 x 128] (+)= A[64 x 16] B[128 x 16]^T, fp16 operands in shared memory, fp32 accumulator in registers of the
// issuing warpgroup.  Thread t (warp w, lane l) holds rows 16 w + l / 4 + 8 i, columns 8 j + 2 (l % 4) + e in
// d[4 j + 2 i + e].  TA / TB = 1: the operand is MN-major.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " FAD_WG_D64 ", %64, %65, p, 1, 1, %67, %68;\n\t}\n"
        : FAD_WG_OUT64(d)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA), "n"(TB));
}

#define FAD_WG_D32                                                                                                 \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                    \
    "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
// D[64 x 64] (+)= A[64 x 16] B[64 x 16]^T with A in registers (fp16 pairs, the m64n16 accumulator layout: a[0] = row
// r, columns 2 (l % 4) + {0, 1}; a[1] = row r + 8; a[2] / a[3] = the same rows, columns + 8) and B MN-major in shared memory
__device__ __forceinline__ void wgmma_m64n64k16_f16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " FAD_WG_D32 ", {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}
// the same with B K-major in shared memory (B[n][k] rows of k, as the TMA boxes and kmajor_sw128_desc describe them)
__device__ __forceinline__ void wgmma_m64n64k16_f16_rs_kmajor(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc,
                                                              uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " FAD_WG_D32 ", {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}

}  // namespace sm90
