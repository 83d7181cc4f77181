// Device-side helpers shared by the tensor-core kernels (gconv_tc.cu, conv2d_tma.cu, spconv_split.cu) on sm_90a:
// mbarrier / bulk-copy / cluster PTX wrappers, warpgroup MMA (wgmma) descriptors and issue, the hi/lo operand splits.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

#include <cstdlib>
#include <utility>

namespace tc {

constexpr int BM = 128;                  // output rows per tile: two consumer warpgroups of 64 rows each
constexpr int BK = 32;                   // fp32 elements per chunk = one 128-byte swizzle row
constexpr int A_TILE_BYTES = BM * 128;   // 16 KB (hi) ; same for lo
constexpr int CONS_THREADS = 256;        // two consumer warpgroups (warps 0-7) in every tensor-core kernel

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra.uni WAIT_DONE;\n\t"
        "bra.uni WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
// Programmatic dependent launch: a kernel launched with the programmatic-stream-serialization attribute may start
// while its predecessor in the stream is still running.  launch_dependents lets the NEXT grid be scheduled as soon
// as this grid's CTAs free their resources; wait blocks until every prerequisite grid has completed and its memory
// is visible - nothing that reads or writes global data may run before it.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma: start>>4 [0,14) | LBO>>4 [16,30) (=1, unused for
// swizzled K-major) | SBO>>4 [32,46) (=1024 B between 8-row groups) | layout type 1 = SWIZZLE_128B [62,64).
// Operand tiles are 1024-byte aligned; a K step of 32 bytes inside the swizzle row adds 2 to the start field.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// wgmma ordering: fence before the first MMA of a batch (the accumulators were written by ordinary instructions),
// commit the batch as a group, wait until at most N groups are still in flight.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] += A[64 x K] * B[K x N]^T, both operands K-major in shared memory, fp32 accumulators in registers:
// PREC 0 = kind tf32 (K = 8 per instruction), PREC 1 = f16 (K = 16).  Thread t of the warpgroup holds rows
// 16 (t / 32) + (t % 32) / 4 + 8 i and columns 8 j + 2 (t % 4) + e at d[4 j + 2 i + e].  scale_d = 0: D = A * B
// (the accumulator's previous contents are ignored).
template <int PREC, int N>
__device__ __forceinline__ void wgmma(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
template <>
__device__ __forceinline__ void wgmma<1, 16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(scale_d) : "memory");
}
template <>
__device__ __forceinline__ void wgmma<1, 32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d) : "memory");
}
template <>
__device__ __forceinline__ void wgmma<1, 64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d) : "memory");
}
template <>
__device__ __forceinline__ void wgmma<1, 128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d) : "memory");
}
template <>
__device__ __forceinline__ void wgmma<0, 16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(scale_d) : "memory");
}
template <>
__device__ __forceinline__ void wgmma<0, 32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d) : "memory");
}
template <>
__device__ __forceinline__ void wgmma<0, 64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d) : "memory");
}
template <>
__device__ __forceinline__ void wgmma<0, 128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d) : "memory");
}

// D[64 x 128] += A[64 x 16] * B[16 x 128] (f16, fp32 accumulators) with A in registers: a[0..3] is the thread's
// fragment, rows 16 (t / 32) + (t % 32) / 4 (+8 in a[1], a[3]) and k pairs 2 (t % 4) (+8 in a[2], a[3]); B is
// K-major in shared memory.  The MMA reads a[] asynchronously: the registers stay untouched until a wgmma_wait shows
// the group complete.
__device__ __forceinline__ void wgmma_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db) : "memory");
}
template <int R>
__device__ __forceinline__ void fence_regs(uint32_t (&r)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+r"(r[i])::"memory");
}
// Warpgroup register reallocation (all warps of a warpgroup execute the same one): the setmaxnreg.dec of one
// warpgroup returns registers to the SM's pool, the setmaxnreg.inc of another waits for them.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ uint4 lds_v4(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr)
                 : "memory");
    return v;
}

// One 128-byte K chunk (four K steps) of the split product x*w ~= xh*wh + (xh*wl + xl*wh): the two small products
// go to their own accumulator, which keeps the 2^-11-smaller terms out of the big one (tensor-core accumulation
// truncates; fewer accumulate steps on the big sum), and the epilogue adds the two once in fp32 RN.
// big_fresh: the chunk's first MMA overwrites `big` instead of adding to it (per-chunk partial sums).
template <int PREC, int N>
__device__ __forceinline__ void mma_chunk_x3(float (&big)[N / 2], float (&small)[N / 2], uint32_t a_hi, uint32_t a_lo,
                                             uint32_t b_hi, uint32_t b_lo, bool big_fresh = false) {
    const uint64_t dah = make_desc(a_hi), dal = make_desc(a_lo), dbh = make_desc(b_hi), dbl = make_desc(b_lo);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint64_t ko = 2ull * (uint64_t)k;
        wgmma<PREC, N>(small, dal + ko, dbh + ko, 1u);
        wgmma<PREC, N>(small, dah + ko, dbl + ko, 1u);
        wgmma<PREC, N>(big, dah + ko, dbh + ko, (k == 0 && big_fresh) ? 0u : 1u);
    }
}

// fp32 -> tf32 with round-to-nearest (the tensor core would otherwise just drop the 13 low bits, which
// biases every product the same way); lo = tf32_rn(x - hi) is then a signed residual of <= 2^-11 |x|.
__device__ __forceinline__ float tf32_rn(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    hi = tf32_rn(x);
    lo = tf32_rn(x - hi);
}

// PREC 0 = 3xTF32 (32 channels per 128-byte row, K=8 per MMA),
// PREC 1 = 3xFP16 (64 channels per row, K=16 per MMA, twice the MMA rate and half the operand bytes).
// FP16 split: hi = half_rn(x), lo = half_rn((x - hi) * 2048); the residual is scaled into the normal fp16 range,
// the "small" accumulator therefore carries a factor 2048 that the epilogue removes.  22 significand bits survive
// (vs 21 for the tf32 split).  The contract is |x| < 65520: at and above it half_rn(x) is +-inf, lo is -+inf and the
// next conv's big + small / 2048 is NaN for every output that reads x.  Every store of split planes therefore tracks
// its lo halves in an F16Range and report_f16_range() sets SASSD_FLAG_F16_RANGE in the status word (the caller raises; the FP32 precision has fp32's range).  Measured on the CPU oracle: the largest activation
// is 7.6 with the seed-0 test weights and 1.32e3 (neck.fcn.bn5) with the uncalibrated seed-1 BatchNorm.  Weights are
// checked once per load, on the host, when they are packed.
constexpr float kF16LoScale = 2048.f;
// One vote per warp and unit of work: lane 0 of a warp any of whose lanes saw an overflow sets the flag.  All 32
// lanes must call it.
__device__ __forceinline__ void report_f16_range(int* status, bool ovf) {
    if (__any_sync(0xffffffffu, ovf) && status && (threadIdx.x & 31) == 0) atomicOr(status, SASSD_FLAG_F16_RANGE);
}

template <int PREC>
struct Prec {
    static constexpr int BKC = PREC == 0 ? 32 : 64;   // input channels per pipeline chunk
    static constexpr int NF4 = BKC / 4;               // float4 loads per row per chunk
};

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ void split_f16(float x, float& hi_as_float, float& lo_scaled) {
    const __half h = __float2half_rn(x);
    hi_as_float = __half2float(h);
    lo_scaled = (x - hi_as_float) * kF16LoScale;
}

// Overflow of the split, tracked on the stored lo halves: lo = half((x - hi) * 2048) is +-inf exactly when a finite x
// overflowed (hi = +-inf; otherwise |x - hi| <= 16), and NaN when x is inf or NaN, which is not the split's fault and
// which __hmax2 passes over.  One HMNMX2 per stored pair keeps the check off the store path.
struct F16Range {
    __half2 m = __half2(__half(0.f), __half(0.f));
    __device__ __forceinline__ void add(uint32_t lo2) {
        m = __hmax2(m, __habs2(*reinterpret_cast<const __half2*>(&lo2)));
    }
    __device__ __forceinline__ bool overflowed() const {
        return __hisinf(__low2half(m)) != 0 || __hisinf(__high2half(m)) != 0;
    }
};

// two values at once: hi pair and scaled-residual pair as packed half2 words
__device__ __forceinline__ void split_f16x2(float x, float y, uint32_t& hi2, uint32_t& lo2) {
    const __half2 h = __floats2half2_rn(x, y);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn((x - hf.x) * kF16LoScale, (y - hf.y) * kF16LoScale);
    hi2 = *reinterpret_cast<const uint32_t*>(&h);
    lo2 = *reinterpret_cast<const uint32_t*>(&l);
}

// Host: launch `kern`, optionally as a programmatic dependent of the previous kernel in the stream (every kernel launched
// through here calls pdl_wait() before touching global data, so only its prologue overlaps the predecessor's tail).
// A per-capture choice: sassd_set_pdl(1) while the latency graph is captured (detectors._GraphedStep), off otherwise;
// the environment variable SASSD_PDL=0/1 is the default when sassd_set_pdl was never called.
extern int g_sassd_pdl;      // -1: not set (voxelize.cu)
inline bool pdl_enabled() {
    if (g_sassd_pdl >= 0) return g_sassd_pdl != 0;
    static const bool on = [] { const char* e = getenv("SASSD_PDL"); return e && atoi(e) != 0; }();
    return on;
}
template <class... KArgs, class... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

}  // namespace tc
