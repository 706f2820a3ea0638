// Shared device helpers for the sm_90a kernels: mbarrier / TMA / wgmma PTX wrappers, error plumbing.
// Everything here is written against the PTX ISA for sm_90a (CUDA 12.x); no CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vpt_b200.h"

namespace vpt {

// ------------------------------------------------------------------------------------------------------
// host-side error plumbing (vpt_last_error)
// ------------------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
#define VPT_CHECK(cond, ...)                 \
    do {                                     \
        if (!(cond)) {                       \
            vpt::set_error(__VA_ARGS__);     \
            return VPT_ERR_ARG;              \
        }                                    \
    } while (0)
#define VPT_CUDA(expr)                                                                   \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            vpt::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return VPT_ERR_CUDA;                                                         \
        }                                                                                \
    } while (0)
#define VPT_LAUNCH_CHECK() VPT_CUDA(cudaGetLastError())
static int g_pdl = 0;
// kernel<<<grid, block, smem, stream>>>(args...) with the programmatic-stream-serialization attribute when vpt_set_pdl(1)
template <typename... KArgs, typename... Args>
static inline void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = g_pdl ? 1 : 0;
    (void)cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);  // errors surface in the VPT_LAUNCH_CHECK() that follows
}


// device-side watchdog flag (defined by the including .cu): kernels that wait on mbarriers record a code here
// instead of hanging forever.
#ifndef VPT_NO_WATCHDOG
__device__ unsigned int g_device_error = 0;
#endif

// ------------------------------------------------------------------------------------------------------
// small device utils
// ------------------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  Every kernel that may be launched with the attribute starts with pdl_sync(): it lets the NEXT
// kernel of the stream be scheduled right away (its blocks then sit in their own pdl_sync()) and waits until the PREVIOUS kernel has
// completed and flushed its memory -- so only launch latency and block scheduling overlap, never the data flow.  Without the attribute
// both instructions are no-ops.  vpt_set_pdl(1) (default 0) makes the launchers below add the attribute (policy.GraphedAct(pdl=True);
// measured neutral on the ~130-node rollout graph, tests/test_gpu_policy.py checks that it changes no bit).
__device__ __forceinline__ void pdl_sync() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ float round_bf16(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

// ------------------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
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
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// try_wait with a suspend-time hint (ns): the warp sleeps in hardware until the phase completes or the time limit passes, instead of
// burning issue slots in a spin loop (round-2 ncu of the first-conv kernel: ~45 % of all executed instructions were BRA / SYNCS / BSSY
// of waiting warps, competing with the 12 working warps of the SM).
__device__ __forceinline__ bool mbar_try_wait_sleep(uint64_t* bar, uint32_t parity, uint32_t ns) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
        : "memory");
    return ok != 0;
}
// Waits for the phase with the given parity to complete.  A watchdog (~2 s of polling) turns a protocol bug
// into a recorded error + early exit rather than a hung GPU.
// The shared error flag lives in global memory: polling it on EVERY failed try_wait made every short wait cost at least one L2 round
// trip on an address that all waiting warps of all SMs hammer at once -- invisible next to the ~15 us tiles of the conv kernels, but
// it was most of the time of the first-conv kernel, whose tiles last ~0.5 us (round-2 measurement).  try_wait itself blocks for a
// hardware-defined interval, so the flag is now looked at once per 64 failed attempts.
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, unsigned int code) {
    if (mbar_try_wait(bar, parity)) return true;
    const long long t0 = clock64();
    for (unsigned int it = 1;; ++it) {
        if (mbar_try_wait_sleep(bar, parity, 20000u)) return true;
        if ((it & 63u) == 0u) {
            if (*(volatile unsigned int*)&g_device_error != 0u) return false;
            if (clock64() - t0 > 3000000000LL) {
                atomicCAS(&g_device_error, 0u, code);
                return false;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), tile mode, completion on an mbarrier
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"((uint64_t)m), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"((uint64_t)m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// TMA store (shared -> global, tile mode) as a bulk async-group: the issuing thread later waits for the group.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"((uint64_t)m), "r"(smem_u32(src)), "r"(c0),
                 "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {  // all but the N most recent groups have finished READING shared memory
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_all() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// multicast variant: the box lands at the same shared-memory offset (and signals the same mbarrier offset) in every
// CTA of the cluster whose bit is set in cta_mask
__device__ __forceinline__ void tma_load_2d_mc(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
            smem_u32(dst)),
        "l"((uint64_t)m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
        : "memory");
}

// ------------------------------------------------------------------------------------------------------
// thread-block clusters
// ------------------------------------------------------------------------------------------------------
// arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
    asm volatile(
        "{\n\t.reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}" ::"r"(smem_u32(bar)),
        "r"(rank)
        : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ------------------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): a warpgroup of 128 threads computes D[64 x N] (+)= A[64 x 16] * B[N x 16]^T with both operands in
// shared memory (descriptors below) and D in registers.  Fragment of m64nNk16 with fp32 accumulators: register r of warp w,
// lane l holds row 16*w + l/4 + 8*((r/2)&1), column 8*(r/4) + 2*(l%4) + (r&1).
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_reg_fence(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 64] (+)= A * B^T, bf16 inputs, fp32 accumulate.  TA / TB = 1: the operand is MN-major (its M / N index contiguous).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}

// D[64 x 128] (+)= A * B^T: one instruction reads the A slab once for all 128 columns (two n64 instructions read it twice).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}

// Warpgroup register budget (setmaxnreg): producer warpgroups give registers back, MMA warpgroups take them.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// 128-byte-swizzled operand tile (bit layout per the PTX ISA "matrix descriptor" of wgmma: start>>4 [0,14), LBO>>4 [16,30),
// SBO>>4 [32,46), base offset [49,52), swizzle mode [62,64) with 1 = SWIZZLE_128B).
//   K-major: rows of 64 bf16 (128 B), 8-row groups `sbo` = 1024 B apart; LBO unused.
//   MN-major: every K row holds 64 consecutive M/N elements (128 B), 8-K-row groups are `sbo` apart and the next 64 M/N elements
//   start `lbo` further -- i.e. TMA boxes of {64 elements (inner), K rows} stored back to back.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes = 16u, uint32_t sbo_bytes = 1024u) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)(lbo_bytes >> 4) << 16;
    d |= (uint64_t)(sbo_bytes >> 4) << 32;
    d |= (uint64_t)1 << 62;  // SWIZZLE_128B
    return d;
}

// The 64 x (NR / 2) fragment `d` (columns col0.. of the tile; NR = 32 for n64, 64 for n128) -> rows of a row-major fp32 staging tile
// `stg` [64][pitch] in shared memory.
template <int NR>
__device__ __forceinline__ void wgmma_frag_store(const float (&d)[NR], float* stg, int pitch, int col0) {
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    const int r0 = 16 * w + (l >> 2), c0 = col0 + 2 * (l & 3);
#pragma unroll
    for (int i = 0; i < NR / 4; ++i) {
        *reinterpret_cast<float2*>(stg + (size_t)r0 * pitch + c0 + 8 * i) = make_float2(d[4 * i], d[4 * i + 1]);
        *reinterpret_cast<float2*>(stg + (size_t)(r0 + 8) * pitch + c0 + 8 * i) = make_float2(d[4 * i + 2], d[4 * i + 3]);
    }
}
// One 32-column chunk (columns 32 * C .. 32 * C + 31 of the fragment: registers 16 * C .. 16 * C + 15) of the calling warp's 16 rows
// of `d` -> rows 0..15 of the warp's own row-major fp32 block `blk` [16][pitch].  Only the calling warp's rows are touched, so
// __syncwarp orders the block.  C is a template parameter: a run-time index into the fragment would put it in local memory.
template <int C, int NR>
__device__ __forceinline__ void wgmma_frag_store_chunk(const float (&d)[NR], float* blk, int pitch) {
    static_assert(16 * C + 16 <= NR, "chunk outside the fragment");
    const int l = threadIdx.x & 31;
    float* dst = blk + (size_t)(l >> 2) * pitch + 2 * (l & 3);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(d[16 * C + 4 * i], d[16 * C + 4 * i + 1]);
        *reinterpret_cast<float2*>(dst + (size_t)8 * pitch + 8 * i) = make_float2(d[16 * C + 4 * i + 2], d[16 * C + 4 * i + 3]);
    }
}
// 32 consecutive fp32 values of one staging row (16-byte aligned) as raw words
__device__ __forceinline__ void stg_ld_32(const float* src, uint32_t (&v)[32]) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const float4 x = reinterpret_cast<const float4*>(src)[q];
        v[4 * q] = __float_as_uint(x.x); v[4 * q + 1] = __float_as_uint(x.y); v[4 * q + 2] = __float_as_uint(x.z); v[4 * q + 3] = __float_as_uint(x.w);
    }
}

}  // namespace vpt
