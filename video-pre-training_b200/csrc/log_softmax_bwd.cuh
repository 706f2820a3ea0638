// Backward of the categorical heads' log-softmax for an arbitrary upstream gradient (the differentiable forward, training.py
// `_AutogradRunner`): given g = d loss / d logp of   logp = log_softmax(logits * scale)   over each group of n columns,
//
//     out[r][col0 + k*n + j] = scale * (g[r][k*n + j] - exp(logp[r][k*n + j]) * S[r][k]),   S[r][k] = sum_j g[r][k*n + j]
//                            = 0 where mask[r][k*n + j] == 0   (lib/action_head.py:170-171: a masked logit is overwritten)
//
// S sums over the masked entries too: that is what autograd through masked_fill followed by log_softmax gives.
// One warp per (row, group) for n <= 1024 (camera head, the IDM's factored heads), one 256-thread block per (row, group) above
// (the 8641-wide buttons head).  Bandwidth bound: logp and g are read once (g twice, the second pass mostly from L1), out written
// once.  Fixed-order sums, no atomics: two identical calls give identical bits.
#pragma once
#include "common.cuh"

namespace vpt {

template <int TPR>
__global__ void __launch_bounds__(256) log_softmax_bwd_kernel(const float* __restrict__ logp, long long ld_logp, const float* __restrict__ g,
                                                              long long ld_g, const uint8_t* __restrict__ mask, int groups, int n, float scale,
                                                              __nv_bfloat16* __restrict__ out, long long ld_out, int col0, long long nrg) {
    constexpr int RPB = 256 / TPR;
    __shared__ float red[256 / 32];
    const int tr = threadIdx.x % TPR;
    const long long rg = (long long)blockIdx.x * RPB + threadIdx.x / TPR;
    const bool live = rg < nrg;
    const long long r = live ? rg / groups : 0;
    const int c = live ? (int)(rg - r * groups) * n : 0;
    const float* gr = g + r * ld_g + c;
    float s = 0.f;
    if (live)
        for (int j = tr; j < n; j += TPR) s += __ldg(gr + j);
    s = warp_sum(s);  // (butterfly: every lane ends with the same bits)
    if (TPR > 32) {   // fixed-order sum of the block's warps
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
        __syncthreads();
        s = 0.f;
#pragma unroll
        for (int w = 0; w < TPR / 32; ++w) s += red[w];
    }
    if (!live) return;
    const float* lr = logp + r * ld_logp + c;
    const uint8_t* mr = mask != nullptr ? mask + r * (long long)groups * n + c : nullptr;
    __nv_bfloat16* orow = out + r * ld_out + col0 + c;
    for (int j = tr; j < n; j += TPR) {
        float v = scale * (__ldg(gr + j) - expf(__ldg(lr + j)) * s);
        if (mr != nullptr && mr[j] == 0) v = 0.f;
        orow[j] = __float2bfloat16_rn(v);
    }
}

}  // namespace vpt

extern "C" int vpt_log_softmax_bwd(const float* logp, int64_t ld_logp, const float* g, int64_t ld_g, const uint8_t* mask, int32_t groups, int32_t n,
                                   float scale, void* out, int64_t ld_out, int32_t col0, int64_t rows, void* stream) {
    using namespace vpt;
    const int64_t width = (int64_t)groups * n;
    VPT_CHECK(logp && g && out && rows > 0 && groups > 0 && n > 0 && col0 >= 0 && ld_logp >= width && ld_g >= width &&
                  ld_out >= col0 + width,
              "vpt_log_softmax_bwd: bad arguments");
    const long long nrg = (long long)rows * groups;
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
    if (n <= 1024) {
        log_softmax_bwd_kernel<32><<<(unsigned)((nrg + 7) / 8), 256, 0, (cudaStream_t)stream>>>(logp, ld_logp, g, ld_g, mask, groups, n, scale, o,
                                                                                             ld_out, col0, nrg);
    } else {
        log_softmax_bwd_kernel<256><<<(unsigned)nrg, 256, 0, (cudaStream_t)stream>>>(logp, ld_logp, g, ld_g, mask, groups, n, scale, o, ld_out,
                                                                                   col0, nrg);
    }
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}
