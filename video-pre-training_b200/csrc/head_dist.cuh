// Entropy and KL divergence of the categorical action heads (policy.py, `pi_head.entropy` / `pi_head.kl_divergence`, and their
// backward for autograd), on fp32 log-prob rows [rows][ld] as `_heads` returns them, each row `width` = groups * n columns (groups > 1:
// the IDM's factored heads).  lib/action_head.py:186-220:
//
//   dist_fwd         H[r]  = -sum_j exp(lp[r][j]) * lp[r][j]                     (lq == NULL)
//                    KL[r] =  sum_j exp(lq[r][j]) * (lq[r][j] - lp[r][j])        (KL(q || p))
//   entropy_bwd      dlp[r][j] = -g[r] * exp(lp) * (lp + 1)
//   kl_bwd           dlq[r][j] =  g[r] * exp(lq) * (lq - lp + 1),   dlp[r][j] = -g[r] * exp(lq)     (either output may be NULL)
//
// The sum over the groups of a row and over their columns is one sum over the row's `width` columns.  Masked logits are -100 before the
// log-softmax (policy.py `_heads`), so every log-prob is finite and needs no special case.  One warp per row up to 1024 columns, one
// 256-thread block per row above (the 8641-wide buttons head).  Bandwidth bound: one pass over the inputs, one write of the outputs.
// Fixed-order sums, no atomics: two identical calls give identical bits.
#pragma once
#include "common.cuh"

namespace vpt {

// TPR threads per row (32 or 256), 256 threads per block
template <int TPR>
__global__ void __launch_bounds__(256) head_dist_fwd_kernel(const float* __restrict__ lp, long long ld_lp, const float* __restrict__ lq,
                                                            long long ld_lq, int width, float* __restrict__ out, long long rows) {
    constexpr int RPB = 256 / TPR;
    __shared__ float red[256 / 32];
    const int tr = threadIdx.x % TPR;
    const long long r = (long long)blockIdx.x * RPB + threadIdx.x / TPR;
    float s = 0.f;
    if (r < rows) {
        const float* pr = lp + r * ld_lp;
        if (lq == nullptr) {
#pragma unroll 4
            for (int j = tr; j < width; j += TPR) {
                const float v = __ldg(pr + j);
                s = fmaf(expf(v), v, s);
            }
            s = -s;  // (negated per thread: the fixed-order sum below gives -sum, bit for bit)
        } else {
            const float* qr = lq + r * ld_lq;
#pragma unroll 4
            for (int j = tr; j < width; j += TPR) {
                const float q = __ldg(qr + j);
                s = fmaf(expf(q), q - __ldg(pr + j), s);
            }
        }
    }
    s = warp_sum(s);
    if (TPR > 32) {  // fixed-order sum of the block's warps
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x != 0) return;
        s = 0.f;
#pragma unroll
        for (int w = 0; w < TPR / 32; ++w) s += red[w];
    } else if ((threadIdx.x & 31) != 0) {
        return;
    }
    if (r < rows) out[r] = s;
}

// lq == NULL: the entropy's backward into dp; else the KL's into dq / dp (either may be NULL)
template <int TPR>
__global__ void __launch_bounds__(256) head_dist_bwd_kernel(const float* __restrict__ lp, long long ld_lp, const float* __restrict__ lq,
                                                            long long ld_lq, const float* __restrict__ g, int width, float* __restrict__ dq,
                                                            long long ld_dq, float* __restrict__ dp, long long ld_dp, long long rows) {
    constexpr int RPB = 256 / TPR;
    const int tr = threadIdx.x % TPR;
    const long long r = (long long)blockIdx.x * RPB + threadIdx.x / TPR;
    if (r >= rows) return;
    const float gr = __ldg(g + r);
    const float* pr = lp + r * ld_lp;
    if (lq == nullptr) {
        float* o = dp + r * ld_dp;
#pragma unroll 4
        for (int j = tr; j < width; j += TPR) {
            const float v = __ldg(pr + j);
            o[j] = -gr * expf(v) * (v + 1.f);
        }
        return;
    }
    const float* qr = lq + r * ld_lq;
    float* oq = dq != nullptr ? dq + r * ld_dq : nullptr;
    float* op = dp != nullptr ? dp + r * ld_dp : nullptr;
#pragma unroll 4
    for (int j = tr; j < width; j += TPR) {
        const float q = __ldg(qr + j);
        const float gq = gr * expf(q);
        if (oq != nullptr) oq[j] = gq * (q - __ldg(pr + j) + 1.f);
        if (op != nullptr) op[j] = -gq;
    }
}

}  // namespace vpt

static int head_dist_fwd(const float* lp, int64_t ld_lp, const float* lq, int64_t ld_lq, int32_t width, float* out, int64_t rows,
                         void* stream) {
    using namespace vpt;
    if (width <= 1024) {
        head_dist_fwd_kernel<32><<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(lp, ld_lp, lq, ld_lq, width, out, rows);
    } else {
        head_dist_fwd_kernel<256><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(lp, ld_lp, lq, ld_lq, width, out, rows);
    }
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

static int head_dist_bwd(const float* lp, int64_t ld_lp, const float* lq, int64_t ld_lq, const float* g, int32_t width, float* dq,
                         int64_t ld_dq, float* dp, int64_t ld_dp, int64_t rows, void* stream) {
    using namespace vpt;
    if (width <= 1024) {
        head_dist_bwd_kernel<32><<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(lp, ld_lp, lq, ld_lq, g, width, dq, ld_dq, dp,
                                                                                              ld_dp, rows);
    } else {
        head_dist_bwd_kernel<256><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(lp, ld_lp, lq, ld_lq, g, width, dq, ld_dq, dp, ld_dp, rows);
    }
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_head_entropy(const float* logp, int64_t ld, int32_t groups, int32_t n, float* ent, int64_t rows, void* stream) {
    const int64_t width = (int64_t)groups * n;
    VPT_CHECK(logp && ent && rows > 0 && groups > 0 && n > 0 && width <= INT32_MAX && ld >= width, "vpt_head_entropy: bad arguments");
    return head_dist_fwd(logp, ld, nullptr, 0, (int32_t)width, ent, rows, stream);
}

extern "C" int vpt_head_kl(const float* logq, int64_t ld_q, const float* logp, int64_t ld_p, int32_t groups, int32_t n, float* kl, int64_t rows,
                           void* stream) {
    const int64_t width = (int64_t)groups * n;
    VPT_CHECK(logq && logp && kl && rows > 0 && groups > 0 && n > 0 && width <= INT32_MAX && ld_q >= width && ld_p >= width,
              "vpt_head_kl: bad arguments");
    return head_dist_fwd(logp, ld_p, logq, ld_q, (int32_t)width, kl, rows, stream);
}

extern "C" int vpt_head_entropy_bwd(const float* logp, int64_t ld, const float* g, int32_t groups, int32_t n, float* dlogp, int64_t ld_d,
                                    int64_t rows, void* stream) {
    const int64_t width = (int64_t)groups * n;
    VPT_CHECK(logp && g && dlogp && rows > 0 && groups > 0 && n > 0 && width <= INT32_MAX && ld >= width && ld_d >= width,
              "vpt_head_entropy_bwd: bad arguments");
    return head_dist_bwd(logp, ld, nullptr, 0, g, (int32_t)width, nullptr, 0, dlogp, ld_d, rows, stream);
}

extern "C" int vpt_head_kl_bwd(const float* logq, int64_t ld_q, const float* logp, int64_t ld_p, const float* g, int32_t groups, int32_t n,
                               float* dlogq, int64_t ld_dq, float* dlogp, int64_t ld_dp, int64_t rows, void* stream) {
    const int64_t width = (int64_t)groups * n;
    VPT_CHECK(logq && logp && g && (dlogq || dlogp) && rows > 0 && groups > 0 && n > 0 && width <= INT32_MAX && ld_q >= width && ld_p >= width &&
                  (dlogq == nullptr || ld_dq >= width) && (dlogp == nullptr || ld_dp >= width),
              "vpt_head_kl_bwd: bad arguments");
    return head_dist_bwd(logp, ld_p, logq, ld_q, g, (int32_t)width, dlogq, ld_dq, dlogp, ld_dp, rows, stream);
}
