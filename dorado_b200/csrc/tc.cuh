// sm_90a building blocks: mbarrier, TMA (cp.async.bulk.tensor), wgmma and mma.sync wrappers.
// Hand-written inline PTX; descriptor bit layouts follow the PTX ISA "matrix descriptor format" of wgmma.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace b200 {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must trap, never hang the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) {
            printf("b200: mbarrier wait timeout (block %d thread %d)\n", (int)blockIdx.x, (int)threadIdx.x);
            __trap();
        }
    }
}

// The same without the printf: a function call anywhere in a kernel that issues wgmma makes ptxas serialise the wgmma
// instructions (C7510).
__device__ __forceinline__ void mbar_wait_silent(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) __trap();
    }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
            "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
            ::"r"(smem_u32(smem_dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
            : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
            "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
            ::"r"(smem_u32(smem_dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
            : "memory");
}
// TMA store: shared::cta tile -> global through a tensor map (completion tracked by the thread's bulk async-group)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(m), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(m), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until at most N of this thread's bulk groups still have to READ their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// Bulk copy from this CTA's shared memory into the shared memory of a CTA of the cluster (addresses from mapa); the
// bytes complete on an mbarrier of the destination CTA.  Async proxy on both ends.
__device__ __forceinline__ void bulk_copy_smem_to_cluster(uint32_t dst_cluster_addr, uint32_t src_cta_addr, uint32_t bytes,
                                                          uint32_t dst_mbar_cluster_addr) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_cluster_addr), "r"(src_cta_addr), "r"(bytes), "r"(dst_mbar_cluster_addr)
                 : "memory");
}
// TMA load multicast to the CTAs of the cluster named in cta_mask: the tile lands at the same CTA-relative shared-memory
// offset in every destination and completes on the mbarrier at the same offset there.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                      uint16_t cta_mask) {
    asm volatile(
            "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
            ::"r"(smem_u32(smem_dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
            : "memory");
}
// cp.async (LDGSTS): 16 bytes global -> shared, bypassing L1; completion tracked per thread in commit groups, visible to
// other threads after cp_async_wait and a barrier
__device__ __forceinline__ void cp_async_16(uint32_t smem_dst, const void* gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// wait until at most N of this thread's cp.async groups are still in flight
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------- grid-scope flags (CTAs that are not in one cluster)
// Arrival on a counter in global memory: release at GPU scope, so that whatever the arriving thread has observed (with a
// preceding barrier, the whole CTA's stores) is visible to a thread that acquires the new value.
__device__ __forceinline__ void red_release_gpu_add(unsigned int* p, unsigned int v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ int ld_relaxed_gpu(const int* p) {
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// generic-proxy writes (st.shared) -> visible to the async proxy (wgmma / TMA reads of smem)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- warpgroup MMA (wgmma)
// Shared-memory matrix descriptor, K-major operand stored as rows of 128 B (64 fp16) with the 128-byte swizzle TMA produces
// (CU_TENSOR_MAP_SWIZZLE_128B): 8-row groups 1024 B apart.
//   [0,14)  start address >> 4      [16,30) leading byte offset >> 4 (unused for swizzled K-major; 1)
//   [32,46) stride byte offset >> 4 (1024 B between 8-row groups)   [62,64) layout type: 1 = SWIZZLE_128B
// Advancing 16 fp16 (32 B) along K inside the swizzle row is +2 in the address field.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3ffffu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 32] (+)= A[64 x 16] B[16 x 32]^T, both K-major in shared memory, fp16 in, fp32 accumulate.  Thread t of the
// warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) and columns 8 j + 2 (t % 4) (+ 1): d[4 j + {0, 1}] row r,
// d[4 j + {2, 3}] row r + 8.
__device__ __forceinline__ void wgmma_m64n32k16(float* d, uint64_t adesc, uint64_t bdesc, bool accumulate) {
    asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
            "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
              "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(adesc), "l"(bdesc), "r"((uint32_t)accumulate)
            : "memory");
}
// The same tile for E4M3 operands: D[64 x 32] (+)= A[64 x 32] B[32 x 32]^T, K-major (the only layout 8-bit wgmma takes),
// fp32 accumulate.  32 E4M3 along K are 32 B, so stepping K inside the swizzle row is +2 in the address field as for
// fp16; the accumulator fragment layout is that of wgmma_m64n32k16.
__device__ __forceinline__ void wgmma_m64n32k32_e4m3(float* d, uint64_t adesc, uint64_t bdesc, bool accumulate) {
    asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 "
            "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
              "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(adesc), "l"(bdesc), "r"((uint32_t)accumulate)
            : "memory");
}
// The same tile for int8 operands: D[64 x 32] (+)= A[64 x 32] B[32 x 32]^T, K-major, exact s32 accumulation.  Addressing
// and the accumulator fragment layout are those of the E4M3 form; the integer form takes no operand scale or transpose.
__device__ __forceinline__ void wgmma_m64n32k32_s8(int32_t* d, uint64_t adesc, uint64_t bdesc, bool accumulate) {
    asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
            "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n\t}"
            : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
              "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
            : "l"(adesc), "l"(bdesc), "r"((uint32_t)accumulate)
            : "memory");
}
// Two fp32 values to E4M3 (round to nearest even; beyond +-448 saturates to +-448, NaN stays NaN): lo in the low byte.
__device__ __forceinline__ uint16_t cvt_e4m3x2(float lo, float hi) {
    uint16_t r;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    return r;
}

// ---------------------------------------------------------------- warp MMA (mma.sync) and ldmatrix
// The latency-bound kernels (recurrence, conv2, attention) work on warp-sized tiles with the operands in registers.
// m16n8k16: a[4] = A rows (l / 4, + 8) x k pairs (2 (l % 4), + 8); b[2] = B k pairs (2 (l % 4), + 8) x column l / 4;
// c[4] = rows (l / 4, + 8) x columns 2 (l % 4) + {0, 1}.
__device__ __forceinline__ void mma_f16_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// m16n8k32 on int8, exact s32 accumulation: a[4] = A rows (l / 4, + 8) x 4 bytes of k at 4 (l % 4) (+ 16); b[2] = B 4 bytes of
// k at 4 (l % 4) (+ 16) x column l / 4; c[4] as m16n8k16.  An ldmatrix 8x8 b16 tile whose rows are 16 bytes of k gives the
// b fragment: thread l gets bytes 4 (l % 4) .. + 3 of row l / 4.
__device__ __forceinline__ void mma_s8_16832(int32_t* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// The int8 activation quantiser: round(v) to nearest even, saturated to [-128, 127] (callers pass kInt8ActScale * v with
// |v| <= 1, so -128 is never produced)
__device__ __forceinline__ int32_t cvt_rni_sat_s8(float v) {
    int32_t r;
    asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(r) : "f"(v));
    return r;
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t* r, uint32_t smem_addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t* r, uint32_t smem_addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_addr));
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "elect.sync _|p, 0xffffffff;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(pred));
    return pred != 0;
}

// byte offset of element (row, 16-byte chunk) inside a [rows x 64 fp16] SWIZZLE_128B tile
__device__ __forceinline__ uint32_t sw128_offset(int row, int chunk16) {
    return (uint32_t)(row * 128 + ((chunk16 ^ (row & 7)) << 4));
}

}  // namespace tc

// ---------------------------------------------------------------- host: tensor maps
// cuTensorMapEncodeTiled through the runtime's driver entry point (no link dependency on libcuda).  Elements are fp16, or
// bytes (E4M3 or int8) when elem_bytes == 1; a box row of 128 bytes gets the 128-byte swizzle.
CUtensorMap make_tmap_2d(const void* base, uint64_t inner, uint64_t outer, uint64_t outer_stride_bytes, uint32_t box_inner,
                         uint32_t box_outer, uint32_t elem_bytes = 2);
CUtensorMap make_tmap_3d(const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1_bytes, uint64_t s2_bytes,
                         uint32_t b0, uint32_t b1, uint32_t b2, uint32_t elem_bytes = 2);

}  // namespace b200
