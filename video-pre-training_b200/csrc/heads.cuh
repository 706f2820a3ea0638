// Action-head tail kernels: row log-softmax, Gumbel-max sampling, log-prob gather (lib/action_head.py:163-207).
// The head GEMM itself (Linear + bias, divided by the temperature) is vpt_gemm_bf16 with out_scale = 1/temperature.
#pragma once
#include "common.cuh"

namespace vpt {

__device__ __forceinline__ float block_max(float v) {
    __shared__ float red[32];
    v = warp_max(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    if (l == 0) red[w] = v;
    __syncthreads();
    float r = l < nw ? red[l] : -INFINITY;
    r = warp_max(r);
    __syncthreads();
    return r;  // valid in every thread of warp 0 ... broadcast below
}

__global__ void __launch_bounds__(256) log_softmax_kernel(const float* __restrict__ in, long long ld_in, int col0, int n,
                                                            float* __restrict__ out) {
    pdl_sync();
    __shared__ float bcast[2];
    const long long r = blockIdx.x;
    const float* x = in + r * ld_in + col0;
    float* y = out + r * (long long)n;
    float m = -INFINITY;
    for (int j = threadIdx.x; j < n; j += blockDim.x) m = fmaxf(m, x[j]);
    m = block_max(m);
    if (threadIdx.x == 0) bcast[0] = m;
    __syncthreads();
    m = bcast[0];
    float s = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += expf(x[j] - m);
    const float2 tot = block_sum2(s, 0.f);
    if (threadIdx.x == 0) bcast[1] = logf(tot.x);
    __syncthreads();
    const float lse = bcast[1];
    for (int j = threadIdx.x; j < n; j += blockDim.x) y[j] = (x[j] - m) - lse;
}

__global__ void __launch_bounds__(256) gumbel_argmax_kernel(const float* __restrict__ logits, const float* __restrict__ u,
                                                              long long* __restrict__ idx, int n) {
    pdl_sync();
    __shared__ float bv[32];
    __shared__ int bi[32];
    const long long r = blockIdx.x;
    const float* x = logits + r * (long long)n;
    const float* ur = u ? u + r * (long long)n : nullptr;
    float best = -INFINITY;
    int besti = 0x7fffffff;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        float v = x[j];
        if (ur) {
            float uu = ur[j];
            if (uu == 1.0f) uu = 0.999f;
            const float l1 = logf(uu);
            const float l2 = logf(-l1);
            v = v - l2;
        }
        if (besti == 0x7fffffff || v > best) {  // j ascends within a thread: strict > keeps the lowest index
            best = v;
            besti = j;
        }
    }
    // reduce (value desc, index asc)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        if (oi != 0x7fffffff && (besti == 0x7fffffff || ov > best || (ov == best && oi < besti))) {
            best = ov;
            besti = oi;
        }
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (l == 0) {
        bv[w] = best;
        bi[w] = besti;
    }
    __syncthreads();
    if (w == 0) {
        best = l < nw ? bv[l] : -INFINITY;
        besti = l < nw ? bi[l] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (oi != 0x7fffffff && (besti == 0x7fffffff || ov > best || (ov == best && oi < besti))) {
                best = ov;
                besti = oi;
            }
        }
        if (l == 0) idx[r] = besti == 0x7fffffff ? 0 : besti;
    }
}

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011): one 128-bit block of a counter under a key
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r > 0) {
            k.x += 0x9E3779B9u;
            k.y += 0xBB67AE85u;
        }
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    }
    return c;
}

// Gumbel-max with counter-based noise (batch-invariant sampling): row r's uniform for column j is word j % 4 of the Philox block of counter
// (j / 4, head, stream, step) under key (seed lo, seed hi), with (stream, step) = keys[r] (low 32 bits of each).  u = ((x >> 9) + 0.5) 2^-23
// is exact in fp32 and lies in [2^-24, 1 - 2^-24]: never 0 or 1, so every score is finite.  A row's pick depends on its logits and its key only.
__global__ void __launch_bounds__(256) gumbel_argmax_keyed_kernel(const float* __restrict__ logits, const long long* __restrict__ keys,
                                                                    unsigned long long seed, int head, long long* __restrict__ idx, int n) {
    pdl_sync();
    __shared__ float bv[32];
    __shared__ int bi[32];
    const long long r = blockIdx.x;
    const float* x = logits + r * (long long)n;
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    const uint32_t stream = (uint32_t)keys[2 * r], step = (uint32_t)keys[2 * r + 1];
    float best = -INFINITY;
    int besti = 0x7fffffff;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const uint4 blk = philox4x32_10(make_uint4((uint32_t)(j >> 2), (uint32_t)head, stream, step), key);
        const uint32_t w = (j & 3) == 0 ? blk.x : (j & 3) == 1 ? blk.y : (j & 3) == 2 ? blk.z : blk.w;
        const float u = ((float)(w >> 9) + 0.5f) * 1.1920928955078125e-7f;  // 2^-23; (w >> 9) + 0.5 needs 24 significant bits: exact
        const float v = x[j] - logf(-logf(u));
        if (besti == 0x7fffffff || v > best) {  // j ascends within a thread: strict > keeps the lowest index
            best = v;
            besti = j;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        if (oi != 0x7fffffff && (besti == 0x7fffffff || ov > best || (ov == best && oi < besti))) {
            best = ov;
            besti = oi;
        }
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (l == 0) {
        bv[w] = best;
        bi[w] = besti;
    }
    __syncthreads();
    if (w == 0) {
        best = l < nw ? bv[l] : -INFINITY;
        besti = l < nw ? bi[l] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (oi != 0x7fffffff && (besti == 0x7fffffff || ov > best || (ov == best && oi < besti))) {
                best = ov;
                besti = oi;
            }
        }
        if (l == 0) idx[r] = besti == 0x7fffffff ? 0 : besti;
    }
}

__global__ void gather_logprob_kernel(const float* __restrict__ logits, const long long* __restrict__ idx, float* __restrict__ lp,
                                      long long rows, int n, int accumulate) {
    pdl_sync();
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const float v = logits[r * n + idx[r]];
    lp[r] = accumulate ? lp[r] + v : v;
}

}  // namespace vpt

extern "C" int vpt_log_softmax(const float* in, int64_t ld_in, int32_t col0, int32_t n, float* out, int64_t rows, void* stream) {
    using namespace vpt;
    VPT_CHECK(in && out && rows > 0 && n > 0 && col0 >= 0, "vpt_log_softmax: bad arguments");
    launch_k(log_softmax_kernel, dim3((unsigned)rows), dim3(256), 0, (cudaStream_t)stream, in, ld_in, col0, n, out);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_gumbel_argmax(const float* logits, const float* u, int64_t* idx, int64_t rows, int32_t n, void* stream) {
    using namespace vpt;
    VPT_CHECK(logits && idx && rows > 0 && n > 0, "vpt_gumbel_argmax: bad arguments");
    launch_k(gumbel_argmax_kernel, dim3((unsigned)rows), dim3(256), 0, (cudaStream_t)stream, logits, u, reinterpret_cast<long long*>(idx), n);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_gumbel_argmax_keyed(const float* logits, const int64_t* keys, uint64_t seed, int32_t head, int64_t* idx, int64_t rows, int32_t n,
                                       void* stream) {
    using namespace vpt;
    VPT_CHECK(logits && keys && idx && rows > 0 && n > 0 && head >= 0, "vpt_gumbel_argmax_keyed: bad arguments");
    launch_k(gumbel_argmax_keyed_kernel, dim3((unsigned)rows), dim3(256), 0, (cudaStream_t)stream, logits, reinterpret_cast<const long long*>(keys),
             (unsigned long long)seed, (int)head, reinterpret_cast<long long*>(idx), (int)n);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_gather_logprob(const float* logits, const int64_t* idx, float* lp, int64_t rows, int32_t n, int32_t accumulate,
                                  void* stream) {
    using namespace vpt;
    VPT_CHECK(logits && idx && lp && rows > 0 && n > 0, "vpt_gather_logprob: bad arguments");
    launch_k(gather_logprob_kernel, dim3((unsigned)((rows + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, 
        logits, reinterpret_cast<const long long*>(idx), lp, rows, n, accumulate);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}
