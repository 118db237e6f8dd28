// Tile memory, wgmma, mbarrier and bulk-copy PTX wrappers for sm_90a (hand-written; encodings follow the PTX ISA
// "asynchronous warpgroup level matrix" chapter: shared-memory matrix descriptor, wgmma.mma_async).
//
// Everything here serves one pattern: a 128-row tile whose rows are owned by the threads of a tile group (thread r of a
// warpgroup <-> tile row r), the A operand written row-per-thread into TILE MEMORY, the 64x64 weight matrix B resident
// in shared memory in the canonical no-swizzle K-major layout, and the fp32 accumulator D stored back into tile memory
// by the warpgroup that computed it and read row-per-thread.
//
// Tile memory is a region at the start of the kernel's dynamic shared memory, addressed like a 128-lane register file:
// taddr = (lane_base << 16) | column, 32-bit columns, and the thread of lane i of a warp accesses row lane_base + i.
// Column c of row r lives at byte (c / 4)·2048 + r·16 + (c % 4)·4: four consecutive columns of a row are one 16-byte
// word (one conflict-free STS.128 / LDS.128 per warp), and 16-bit data written as two halves per column is the
// canonical no-swizzle K-major layout of a wgmma operand (core matrix = 8 rows x 16 bytes, 8-row groups 128 bytes
// apart, K chunks of 8 halves 2048 bytes apart).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace degnn {

extern __shared__ __align__(1024) uint8_t degnn_dyn_smem[];   // the dynamic shared memory of the running kernel

namespace tmma {

constexpr uint32_t TM_COLGROUP_BYTES = 2048;                  // 4 columns x 128 rows
__host__ __device__ constexpr int tm_bytes(int ncols) { return ncols * 128 * 4; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

// shared-memory byte address of (row, column) of tile memory
__device__ __forceinline__ uint32_t tm_addr_rc(uint32_t row, uint32_t col) {
    return smem_u32(degnn_dyn_smem) + (col >> 2) * TM_COLGROUP_BYTES + row * 16u + (col & 3u) * 4u;
}
// address of the calling thread's row at taddr (lane_base << 16 | column)
__device__ __forceinline__ uint32_t tm_addr(uint32_t taddr) {
    return tm_addr_rc((taddr >> 16) + (threadIdx.x & 31u), taddr & 0xffffu);
}

// 64-bit shared-memory matrix descriptor (PTX ISA, wgmma "matrix-descriptor"):
//   [0,14) start address >> 4   [16,30) leading-dim byte offset >> 4   [32,46) stride-dim byte offset >> 4
//   [49,52) base offset = 0   [62,64) layout = 0 (no swizzle).  K-major: LBO = next K chunk, SBO = next 8 rows.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) |
           ((uint64_t)((sbo >> 4) & 0x3FFF) << 32);
}

// make generic-proxy smem writes (st.shared) visible to the async proxy (wgmma operand reads / bulk copies); for
// tile-memory stores, once the group barrier that follows has been passed
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- tile memory <-> registers, the own row, 4 / 8 / 16 consecutive columns (column offset a multiple of 4) --------------
__device__ __forceinline__ void tm_st4(uint32_t taddr, const uint32_t (&r)[4]) {
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(tm_addr(taddr)), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3])
                 : "memory");
}
__device__ __forceinline__ void tm_ld4(uint32_t taddr, uint32_t* r) {
    asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(tm_addr(taddr))
                 : "memory");
}
__device__ __forceinline__ void tm_st8(uint32_t taddr, const uint32_t (&r)[8]) {
    tm_st4(taddr, *reinterpret_cast<const uint32_t(*)[4]>(&r[0]));
    tm_st4(taddr + 4, *reinterpret_cast<const uint32_t(*)[4]>(&r[4]));
}
__device__ __forceinline__ void tm_st16(uint32_t taddr, const uint32_t (&r)[16]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) tm_st4(taddr + 4 * i, *reinterpret_cast<const uint32_t(*)[4]>(&r[4 * i]));
}
__device__ __forceinline__ void tm_ld16(uint32_t taddr, uint32_t (&r)[16]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) tm_ld4(taddr + 4 * i, &r[4 * i]);
}
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// ---- wgmma: one 64-row block of a tile, N = 64, fp16 operands, fp32 accumulators in registers ---------------------------
// Accumulator fragment of m64n64 (thread = lane l of warp w of the warpgroup): d[4j+0], d[4j+1] = row 16w + l/4,
// columns 8j + 2(l%4) + {0,1};  d[4j+2], d[4j+3] = the same columns of row 16w + l/4 + 8.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wgmma_f16_m64n64k16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31},"
        " %32, %33, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
// Same with the A operand in registers.  A fragment of m64k16 (thread = lane l of warp w, g = 16w + l/4, c = 2(l%4)):
// a[0] = row g, k = c, c+1;  a[1] = row g + 8, k = c, c+1;  a[2] = row g, k = c+8, c+9;  a[3] = row g + 8, k = c+8, c+9
// (two fp16 per register, even k in the low half).  For k-step ks these are exactly the accumulator pairs
// d[8ks .. 8ks+7] of an m64n64 result, so one GEMM's output feeds the next GEMM without leaving the registers.
// The registers are read asynchronously: they must stay untouched until wgmma_wait_all (see wgmma_keep).
// ACCUMULATE = false overwrites d (scale-d 0) and reads nothing of it.
#define DEGNN_WGMMA_RA_D(c)                                                                                             \
    c(d[0]), c(d[1]), c(d[2]), c(d[3]), c(d[4]), c(d[5]), c(d[6]), c(d[7]), c(d[8]), c(d[9]), c(d[10]), c(d[11]),      \
        c(d[12]), c(d[13]), c(d[14]), c(d[15]), c(d[16]), c(d[17]), c(d[18]), c(d[19]), c(d[20]), c(d[21]), c(d[22]),  \
        c(d[23]), c(d[24]), c(d[25]), c(d[26]), c(d[27]), c(d[28]), c(d[29]), c(d[30]), c(d[31])
#define DEGNN_WGMMA_RA_ASM(scale_d)                                                                                     \
    "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "                                                               \
    "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30," \
    "%31}, {%32,%33,%34,%35}, %36, " scale_d ", 1, 1, 0;\n"
template <bool ACCUMULATE>
__device__ __forceinline__ void wgmma_f16_m64n64k16_rA(float (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                       uint64_t b_desc) {
    if (ACCUMULATE)
        asm volatile(DEGNN_WGMMA_RA_ASM("1") : DEGNN_WGMMA_RA_D("+f")
                     : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc) : "memory");
    else
        asm volatile(DEGNN_WGMMA_RA_ASM("0") : DEGNN_WGMMA_RA_D("=f")
                     : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc) : "memory");
}
#undef DEGNN_WGMMA_RA_D
#undef DEGNN_WGMMA_RA_ASM
// Keep registers that an in-flight wgmma reads or writes alive and in place up to this point: the compiler sees the
// wgmma's register operands only at its issue, so without this it may reuse A registers or read D before the wait.
__device__ __forceinline__ void wgmma_keep(float& r) { asm volatile("" : "+f"(r)::"memory"); }
__device__ __forceinline__ void wgmma_keep(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }
// fragment of the 64-row block `mb` <-> 64 tile-memory columns starting at `col` (rows 64·mb .. 64·mb + 63)
__device__ __forceinline__ void frag_rows(int mb, uint32_t& r0, uint32_t& q) {
    const uint32_t w = (threadIdx.x >> 5) & 3u, l = threadIdx.x & 31u;
    r0 = 64u * (uint32_t)mb + 16u * w + (l >> 2);
    q = l & 3u;
}
__device__ __forceinline__ void frag_store(const float (&d)[32], uint32_t col, int mb) {
    uint32_t r0, q;
    frag_rows(mb, r0, q);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint32_t c = col + 8u * j + 2u * q;
        const uint32_t a0 = tm_addr_rc(r0, c), a1 = tm_addr_rc(r0 + 8u, c);
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(a0), "f"(d[4 * j]), "f"(d[4 * j + 1]) : "memory");
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(a1), "f"(d[4 * j + 2]), "f"(d[4 * j + 3]) : "memory");
    }
}
__device__ __forceinline__ void frag_load(float (&d)[32], uint32_t col, int mb) {
    uint32_t r0, q;
    frag_rows(mb, r0, q);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint32_t c = col + 8u * j + 2u * q;
        asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(d[4 * j]), "=f"(d[4 * j + 1]) : "r"(tm_addr_rc(r0, c)) : "memory");
        asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(d[4 * j + 2]), "=f"(d[4 * j + 3]) : "r"(tm_addr_rc(r0 + 8u, c))
                     : "memory");
    }
}

// ---- mbarrier ----------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// ---- bulk async copy global -> shared (TMA engine, no tensor map), completes on an mbarrier ----------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// ---- per-thread async copies global -> shared (LDGSTS: per-lane addresses, no registers, generic proxy) ------------
// Completion is per issuing thread (commit_group / wait_group); a thread that only reads what it copied itself needs
// no barrier.  16-byte form bypasses L1 (.cg); the 4/8-byte forms allocate in L1 (.ca is the only variant).
__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) { cp_async16(smem_u32(smem_dst), gsrc); }
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
// two adjacent fp32 added to global memory with one reduction (sm_90+), 8-byte aligned
__device__ __forceinline__ void red_add_v2(float* gdst, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(gdst), "f"(a), "f"(b) : "memory");
}

// named barrier among `nthreads` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace tmma
}  // namespace degnn
