// Thin inline-PTX wrappers for the sm_90a (Hopper) features the Saber kernels use:
// mbarrier, TMA (tiled + im2col), wgmma, clusters / distributed shared memory, PDL.
// Everything here is sm_90a code; there is no fallback path by design.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace b200 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n"
        ".reg .b32 %%rx;\n"
        ".reg .pred %%px;\n"
        "elect.sync %%rx|%%px, %1;\n"
        "@%%px mov.s32 %0, 1;\n"
        "}\n"
        : "+r"(pred)
        : "r"(0xffffffffu));
    return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// Shared-space-address variants (the single-thread producer / MMA loops keep everything as 32-bit
// shared addresses: no generic->shared conversions or 64-bit math on their critical path).
__device__ __forceinline__ void mbar_wait_sa(uint32_t bar_sa, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(bar_sa),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx_sa(uint32_t bar_sa, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_sa), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d_sa(const CUtensorMap* m, uint32_t bar_sa, uint32_t dst_sa, int32_t c0,
                                               int32_t c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst_sa),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_sa), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_im2col_4d_sa(const CUtensorMap* m, uint32_t bar_sa, uint32_t dst_sa,
                                                      int32_t c, int32_t w, int32_t h, int32_t n, uint16_t off_w,
                                                      uint16_t off_h) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};" ::"r"(dst_sa),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_sa), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
        : "memory");
}
// Tiled 4-D load (dims C, W, H, N of an NHWC tensor): the box lands densely as [h][w][c] rows; coordinates may be
// negative / past the edge, those elements are zero-filled -- the halo of a convolution slab.
__device__ __forceinline__ void tma_load_4d_sa(const CUtensorMap* m, uint32_t bar_sa, uint32_t dst_sa, int32_t c,
                                               int32_t w, int32_t h, int32_t n) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst_sa),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_sa), "r"(c), "r"(w), "r"(h), "r"(n)
        : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src_sa, int32_t c, int32_t w, int32_t h,
                                             int32_t n) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(src_sa), "r"(c), "r"(w), "r"(h), "r"(n)
                 : "memory");
}
// Multicast variants: the box lands at the same shared offset `dst_sa` in every CTA of `mask` (bit r = cluster rank r)
// and completes its bytes on the mbarrier at offset `bar_sa` of each of them.
__device__ __forceinline__ void tma_load_2d_mc_sa(const CUtensorMap* m, uint32_t bar_sa, uint32_t dst_sa, int32_t c0,
                                                  int32_t c1, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(dst_sa),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_sa), "r"(c0), "r"(c1), "h"(mask)
        : "memory");
}
__device__ __forceinline__ void tma_load_im2col_4d_mc_sa(const CUtensorMap* m, uint32_t bar_sa, uint32_t dst_sa,
                                                         int32_t c, int32_t w, int32_t h, int32_t n, uint16_t off_w,
                                                         uint16_t off_h, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8}, %9;" ::"r"(dst_sa),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_sa), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h), "h"(mask)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d_mc_sa(const CUtensorMap* m, uint32_t bar_sa, uint32_t dst_sa, int32_t c,
                                                  int32_t w, int32_t h, int32_t n, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(dst_sa),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_sa), "r"(c), "r"(w), "r"(h), "r"(n), "h"(mask)
        : "memory");
}
// arrive on an mbarrier given by its shared::cluster address (this CTA's or a peer's, see map_to_cta)
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cbar) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cbar) : "memory");
}
// non-blocking probe of an mbarrier phase (true: the phase with this parity has completed)
__device__ __forceinline__ bool mbar_try_wait_sa(uint32_t bar_sa, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
        "selp.u32 %0, 1, 0, P1;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar_sa), "r"(parity)
        : "memory");
    return ok != 0;
}
// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// Tiled 2-D load: box lands densely (swizzled per the tensor map) at dst.
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst,
                                            int32_t c0, int32_t c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// im2col 4-D load over an NHWC tensor (dims C,W,H,N): fetches `pixelsPerColumn`
// consecutive output pixels starting at base pixel (w,h,n) for filter offset
// (off_w, off_h), `channelsPerPixel` channels starting at c.
__device__ __forceinline__ void tma_load_im2col_4d(const CUtensorMap* m, uint64_t* bar, void* dst,
                                                   int32_t c, int32_t w, int32_t h, int32_t n,
                                                   uint16_t off_w, uint16_t off_h) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n),
        "h"(off_w), "h"(off_h)
        : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int32_t c0,
                                             int32_t c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(src)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_all() {
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// generic <-> async proxy ordering for all state spaces (a TMA load after an acquire of a flag that
// another SM released after its TMA store completed)
__device__ __forceinline__ void fence_proxy_async_all() {
    asm volatile("fence.proxy.async;" ::: "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_gpu_add(uint32_t* p, uint32_t v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA, accumulators in registers)
// KIND_TF32 is the MMA of the 3xTF32 kernels (KIND_TF32X3), which issue .tf32 wgmma on both planes.
enum MmaKind { KIND_I8 = 0, KIND_F16 = 1, KIND_TF32 = 2, KIND_TF32X3 = 3, KIND_E4M3 = 4 };

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(uint32_t (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// Shared-memory matrix descriptor (K-major operand) as (lo, hi) words:
//  lo: [0,14) start>>4  [16,30) LBO>>4      hi: [0,14) SBO>>4  [30,32) layout (1 SW128, 2 SW64, 3 SW32, 0 none)
// layout_type_for_chunk() returns the layout in the 3-bit form (2 SW128, 4 SW64, 6 SW32) used as `lt << 29`.
__device__ __forceinline__ uint64_t desc64(uint32_t lo, uint32_t hi) {
    return static_cast<uint64_t>(lo) | (static_cast<uint64_t>(hi) << 32);
}

// One wrapper per (operand type, N): the accumulator operand list of an inline-PTX wgmma has to be spelled out.
// D[64 x N] (+)= A[64 x 32 B] * B[N x 32 B]^T, both operands K-major in shared memory.
__device__ __forceinline__ void wgmma_s8_n16(uint32_t (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_u8_n16(uint32_t (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n16k32.s32.u8.s8 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_f16_n16(uint32_t (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n16(uint32_t (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_s8_n32(uint32_t (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_u8_n32(uint32_t (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_f16_n32(uint32_t (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n32(uint32_t (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_s8_n64(uint32_t (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_u8_n64(uint32_t (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k32.s32.u8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_f16_n64(uint32_t (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n64(uint32_t (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_s8_n128(uint32_t (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_u8_n128(uint32_t (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_f16_n128(uint32_t (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n128(uint32_t (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(a), "l"(b), "r"(acc));
}

__device__ __forceinline__ void wgmma_e4m3_n16(uint32_t (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n16k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_e4m3_n32(uint32_t (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_e4m3_n64(uint32_t (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_e4m3_n128(uint32_t (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(a), "l"(b), "r"(acc));
}

// Signedness of the int8 kind's A operand (activations) as a compile-time constant: a runtime choice at every wgmma puts
// each MMA in its own branch arm, behind a warpgroup.arrive that ptxas injects, and the MMAs of a k loop no longer
// issue back to back.
template <bool S>
using ASign = std::integral_constant<bool, S>;

// Runs `body(ASign<...>{})` once with the signedness the plan's instruction descriptor names: the branch is taken once
// per main loop, and the int8 kind gets one copy of the loop per signedness (the other kinds have one copy).
template <int MK, class F>
__device__ __forceinline__ void with_a_sign(bool a_signed, F&& body) {
    if constexpr (MK == KIND_I8) {
        if (a_signed) body(ASign<true>{});
        else body(ASign<false>{});
    } else {
        body(ASign<false>{});
    }
}

// D[64 x N] (+)= A * B^T for one 32-byte K slice; A_SIGNED selects s8 / u8 activations of the int8 kind.
template <int MK, int N, bool A_SIGNED>
__device__ __forceinline__ void wgmma(uint32_t (&d)[N / 2], uint64_t a, uint64_t b, ASign<A_SIGNED>, uint32_t acc) {
    if constexpr (MK == KIND_I8) {
        if constexpr (A_SIGNED) {
            if constexpr (N == 16) wgmma_s8_n16(d, a, b, acc);
            else if constexpr (N == 32) wgmma_s8_n32(d, a, b, acc);
            else if constexpr (N == 64) wgmma_s8_n64(d, a, b, acc);
            else wgmma_s8_n128(d, a, b, acc);
        } else {
            if constexpr (N == 16) wgmma_u8_n16(d, a, b, acc);
            else if constexpr (N == 32) wgmma_u8_n32(d, a, b, acc);
            else if constexpr (N == 64) wgmma_u8_n64(d, a, b, acc);
            else wgmma_u8_n128(d, a, b, acc);
        }
    } else if constexpr (MK == KIND_F16) {
        if constexpr (N == 16) wgmma_f16_n16(d, a, b, acc);
        else if constexpr (N == 32) wgmma_f16_n32(d, a, b, acc);
        else if constexpr (N == 64) wgmma_f16_n64(d, a, b, acc);
        else wgmma_f16_n128(d, a, b, acc);
    } else if constexpr (MK == KIND_E4M3) {
        if constexpr (N == 16) wgmma_e4m3_n16(d, a, b, acc);
        else if constexpr (N == 32) wgmma_e4m3_n32(d, a, b, acc);
        else if constexpr (N == 64) wgmma_e4m3_n64(d, a, b, acc);
        else wgmma_e4m3_n128(d, a, b, acc);
    } else {
        if constexpr (N == 16) wgmma_tf32_n16(d, a, b, acc);
        else if constexpr (N == 32) wgmma_tf32_n32(d, a, b, acc);
        else if constexpr (N == 64) wgmma_tf32_n64(d, a, b, acc);
        else wgmma_tf32_n128(d, a, b, acc);
    }
}

// The same with the s8 / u8 choice made at the instruction, for a loop that keeps it there (conv_persistent.cu): each
// int8 MMA then sits in its own branch arm. The other kinds need no choice.
template <int MK, int N>
__device__ __forceinline__ void wgmma(uint32_t (&d)[N / 2], uint64_t a, uint64_t b, bool a_signed, uint32_t acc) {
    if constexpr (MK == KIND_I8) {
        if (a_signed) wgmma<MK, N>(d, a, b, ASign<true>{}, acc);
        else wgmma<MK, N>(d, a, b, ASign<false>{}, acc);
    } else {
        wgmma<MK, N>(d, a, b, ASign<false>{}, acc);
    }
}

// GEMM row (within a warp's 16-row slice of a 64-row wgmma tile) and first column of the 16 accumulators this lane
// receives from acc_row16 for column group g: row (lane / 4) + 8 * ((lane / 2) & 1), columns 32 g + 16 (lane & 1).
__device__ __forceinline__ int acc_row16_row(int lane) { return (lane >> 2) + 8 * ((lane >> 1) & 1); }
__device__ __forceinline__ int acc_row16_col(int lane, int g) { return 32 * g + 16 * (lane & 1); }

// Regroups columns [32 g, 32 g + 32) of a warp's wgmma accumulator fragment (lane l holds rows l/4 and l/4 + 8,
// columns 8 j + 2 (l % 4) + {0, 1}) so that every lane ends up with 16 consecutive columns of ONE row -- the shape the
// epilogue works on. Two butterfly exchanges within each quad of lanes; all 32 lanes must call it.
// For N = 16 the lanes with (lane & 1) = 1 receive no valid columns.
template <int N>
__device__ __forceinline__ void acc_row16(const uint32_t (&d)[N / 2], int g, uint32_t (&v)[16]) {
    const int lane = threadIdx.x & 31;
    const bool b0 = lane & 1, b1 = lane & 2;
    uint32_t q[2][2][2][2];   // [row half][source lane bit 0][8-column block][element]
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int j0 = 4 * g + b, j1 = (N >= 32) ? 4 * g + 2 + b : j0;
                const uint32_t p0 = d[4 * j0 + 2 * h + e], p1 = d[4 * j1 + 2 * h + e];
                const uint32_t keep = b0 ? p1 : p0, send = b0 ? p0 : p1;
                const uint32_t recv = __shfl_xor_sync(0xffffffffu, send, 1);
                q[h][0][b][e] = b0 ? recv : keep;
                q[h][1][b][e] = b0 ? keep : recv;
            }
#pragma unroll
    for (int s0 = 0; s0 < 2; ++s0)
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const uint32_t keep = b1 ? q[1][s0][b][e] : q[0][s0][b][e], send = b1 ? q[0][s0][b][e] : q[1][s0][b][e];
                const uint32_t recv = __shfl_xor_sync(0xffffffffu, send, 2);
                v[8 * b + 2 * s0 + e] = b1 ? recv : keep;          // source lane bit 1 = 0
                v[8 * b + 2 * (2 + s0) + e] = b1 ? keep : recv;    // source lane bit 1 = 1
            }
}

// Instruction-descriptor word kept in the plans: [7,10) a_format (0 unsigned, 1 signed int8); the MMA shape and the
// other operand types are fixed by the kernel instantiation.
__host__ __device__ constexpr uint32_t make_idesc(uint32_t c_fmt, uint32_t a_fmt, uint32_t b_fmt, uint32_t M, uint32_t N) {
    return (c_fmt << 4) | (a_fmt << 7) | (b_fmt << 10) | ((N >> 3) << 17) | ((M >> 4) << 24);
}
__device__ __forceinline__ bool idesc_a_signed(uint32_t idesc) { return ((idesc >> 7) & 7u) == 1u; }

// ---------------------------------------------------------------- clusters / DSMEM
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// all threads of all CTAs of the cluster
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `local_saddr` in CTA `rank` of this cluster
__device__ __forceinline__ uint32_t map_to_cta(uint32_t local_saddr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_saddr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster_v4(uint32_t caddr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared::cluster.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(caddr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// 16-byte store into another CTA's shared memory that completes `bytes` on that CTA's mbarrier
// (both addresses shared::cluster): the receiver just waits on the barrier, no cluster-wide sync
__device__ __forceinline__ void st_async_v4(uint32_t caddr, uint32_t cbar, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
                 ::"r"(caddr), "r"(a), "r"(b), "r"(c), "r"(d), "r"(cbar) : "memory");
}
__device__ __forceinline__ void cluster_arrive() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_wait() {
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---------------------------------------------------------------- PDL
__device__ __forceinline__ void pdl_wait_prior_grid() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ void pdl_launch_dependents() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
// Kernel entry of a PDL launch: signal the dependents at once, then wait for the predecessor before touching memory,
// so launch latency and the neighbours' prologues overlap along the whole chain.
__device__ __forceinline__ void pdl_enter() {
    pdl_launch_dependents();
    pdl_wait_prior_grid();
}

}  // namespace b200
