// Kernels of the RL fine-tuning step (video-pre-training_b200/training.py, RLTrainer): the gradient of
//     loss = L_pi + vf_coef * L_v + kl_coef * L_kl        (means over the N frames of a call)
// with respect to the temperature-scaled logits of every head and the value head's raw output.
//
//   ppo_coef        per row: ratio = exp(lp - old_lp); c = ratio * A / N, or 0 where the PPO objective is clipped
//                   ((A > 0 and ratio > 1+eps) or (A < 0 and ratio < 1-eps); a tie takes the unclipped branch); also the row's
//                   policy loss -min(ratio*A, clamp(ratio, 1-eps, 1+eps)*A) and the clipped flag (1 / 0) for the statistics.
//   rl_head_bwd     one launch per head: (c[r] * (p - onehot(a)) + k * (p - q)) * inv_temp as bf16 into the head's columns of the
//                   logits gradient, p = exp(logp), q = exp(logq) of the frozen reference policy (k * (p - q) dropped without it),
//                   and the row's KL(q || p) = sum_j q_j (logq_j - logp_j) (fixed-order sum) for the statistics.
//                   Bandwidth bound: one pass over logp (and logq), one bf16 write per column.
//                   rl_head_bwd_ent: the same with the entropy bonus, loss - ent_coef * mean H(pi): one more read of logp for the row's
//                   entropy H, then + ent_coef / N * p * (logp + H) in each column's gradient, and H per row for the statistics.
//   ewma_sums       (sum, sum of squares) of the returns in float64, one block, fixed order (all-reduced by the caller under DP).
//   value_bwd       one block: the EWMA normaliser update (lib/normalize_ewma.py:41-55, per_element_update = False) from those sums,
//                   then per row the normalised target with the UPDATED statistics, dvpred = scale * (vpred - target) as bf16 into
//                   one column of the logits gradient, and the row's squared error.
// No atomics anywhere: two identical calls give identical bits.
#pragma once
#include "common.cuh"

namespace vpt {

__global__ void __launch_bounds__(256) ppo_coef_kernel(const float* __restrict__ lp, const float* __restrict__ old_lp, const float* __restrict__ adv,
                                                       long long rows, float lo, float hi, float inv_n, float* __restrict__ c,
                                                       float* __restrict__ pi_loss, float* __restrict__ clipped) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const float a = __ldg(adv + r);
    const float ratio = expf(__ldg(lp + r) - __ldg(old_lp + r));
    const bool clip = (a > 0.f && ratio > hi) || (a < 0.f && ratio < lo);
    const float surr1 = ratio * a, surr2 = fminf(fmaxf(ratio, lo), hi) * a;
    c[r] = clip ? 0.f : surr1 * inv_n;
    pi_loss[r] = -fminf(surr1, surr2);
    clipped[r] = clip ? 1.f : 0.f;
}

// TPR threads per row (32: one warp per row for small heads; 256: one block per row), 256 threads per block.
// ENT (vpt_rl_head_bwd_ent): a first pass gives the row's entropy H = -sum_j p_j logp_j (fixed order, every thread holds it), the second
// adds e * p_j * (logp_j + H) to each column's gradient, the gradient of -ent_coef * mean H with e = ent_coef / N (skipped when e == 0:
// adding +0 would turn a -0 gradient into +0), and the row's H is written to ent (accumulated like kl).
template <int TPR, bool ENT = false>
__global__ void __launch_bounds__(256) rl_head_bwd_kernel(const float* __restrict__ logp, long long ld_logp, const float* __restrict__ logq,
                                                          long long ld_logq, const long long* __restrict__ idx, const float* __restrict__ c,
                                                          float k, float inv_temp, int n, __nv_bfloat16* __restrict__ out, long long ld_out,
                                                          int col0, float* __restrict__ kl, int accumulate, long long rows, float e = 0.f,
                                                          float* __restrict__ ent = nullptr) {
    constexpr int RPB = 256 / TPR;
    __shared__ float red[256 / 32];
    const int tr = threadIdx.x % TPR;
    const long long r = (long long)blockIdx.x * RPB + threadIdx.x / TPR;
    const bool live = r < rows;
    float h = 0.f;
    if (ENT) {
        if (live) {
            const float* lr = logp + r * ld_logp;
            for (int j = tr; j < n; j += TPR) {
                const float lpj = __ldg(lr + j);
                h = fmaf(expf(lpj), lpj, h);
            }
            h = -h;
        }
        h = warp_sum(h);  // (butterfly: every lane ends with the same bits)
        if (TPR > 32) {
            if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = h;
            __syncthreads();
            h = 0.f;
#pragma unroll
            for (int w = 0; w < TPR / 32; ++w) h += red[w];
            __syncthreads();  // every thread has read red before the KL sum below reuses it
        }
    }
    float s = 0.f;
    if (live) {
        const float* lr = logp + r * ld_logp;
        const float* qr = logq != nullptr ? logq + r * ld_logq : nullptr;
        __nv_bfloat16* orow = out + r * ld_out + col0;
        const long long a = __ldg(idx + r);
        const float cr = __ldg(c + r);
        for (int j = tr; j < n; j += TPR) {
            const float lpj = __ldg(lr + j);
            const float p = expf(lpj);
            float g = cr * (j == a ? p - 1.f : p);
            if (qr != nullptr) {
                const float lqj = __ldg(qr + j);
                const float q = expf(lqj);
                g = fmaf(k, p - q, g);
                s = fmaf(q, lqj - lpj, s);
            }
            if (ENT && e != 0.f) g = fmaf(e * p, lpj + h, g);
            orow[j] = __float2bfloat16_rn(g * inv_temp);
        }
    }
    s = warp_sum(s);
    if (TPR > 32) {  // fixed-order sum of the block's warps
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x != 0) return;
        s = 0.f;
        for (int w = 0; w < TPR / 32; ++w) s += red[w];
    } else if ((threadIdx.x & 31) != 0) {
        return;
    }
    if (live) {
        kl[r] = accumulate ? kl[r] + s : s;
        if (ENT) ent[r] = accumulate ? ent[r] + h : h;
    }
}

__global__ void __launch_bounds__(256) ewma_sums_kernel(const float* __restrict__ x, long long rows, double* __restrict__ sums) {
    __shared__ double red[2][256];
    double s = 0.0, s2 = 0.0;
    for (long long r = threadIdx.x; r < rows; r += 256) {
        const double v = (double)__ldg(x + r);
        s += v;
        s2 += v * v;
    }
    red[0][threadIdx.x] = s;
    red[1][threadIdx.x] = s2;
    __syncthreads();
    if (threadIdx.x < 2) {
        double t = 0.0;
        for (int i = 0; i < 256; ++i) t += red[threadIdx.x][i];
        sums[threadIdx.x] = t;
    }
}

__global__ void __launch_bounds__(256) value_bwd_kernel(const float* __restrict__ vpred, const float* __restrict__ ret, const double* __restrict__ sums,
                                                        double count, float* running_mean, float* running_mean_sq, float* debiasing_term,
                                                        float w, float one_minus_w, float scale, __nv_bfloat16* __restrict__ out, long long ld_out,
                                                        int col, float* __restrict__ sq_err, long long rows) {
    // the update in the reference's fp32 operation order: x.mul_(w).add_(batch_stat * (1 - w))
    const float bm = (float)(sums[0] / count), bsq = (float)(sums[1] / count);
    const float rm = __fadd_rn(__fmul_rn(running_mean[0], w), __fmul_rn(bm, one_minus_w));
    const float rsq = __fadd_rn(__fmul_rn(running_mean_sq[0], w), __fmul_rn(bsq, one_minus_w));
    const float deb = __fadd_rn(__fmul_rn(debiasing_term[0], w), one_minus_w);
    const float dc = fmaxf(deb, 1e-5f);
    const float mean = rm / dc;
    const float var = fmaxf(rsq / dc - mean * mean, 1e-2f);
    const float sd = sqrtf(var);
    for (long long r = threadIdx.x; r < rows; r += 256) {
        const float target = (__ldg(ret + r) - mean) / sd;
        const float d = __ldg(vpred + r) - target;
        out[r * ld_out + col] = __float2bfloat16_rn(scale * d);
        sq_err[r] = d * d;
    }
    __syncthreads();  // every thread has read the old statistics
    if (threadIdx.x == 0) {
        running_mean[0] = rm;
        running_mean_sq[0] = rsq;
        debiasing_term[0] = deb;
    }
}

}  // namespace vpt

extern "C" int vpt_ppo_coef(const float* lp, const float* old_lp, const float* adv, int64_t rows, float eps_lo, float eps_hi, float inv_n, float* c,
                            float* pi_loss, float* clipped, void* stream) {
    using namespace vpt;
    VPT_CHECK(lp && old_lp && adv && c && pi_loss && clipped && rows > 0 && eps_lo <= eps_hi, "vpt_ppo_coef: bad arguments");
    ppo_coef_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, (cudaStream_t)stream>>>(lp, old_lp, adv, rows, eps_lo, eps_hi, inv_n, c, pi_loss,
                                                                                     clipped);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_rl_head_bwd(const float* logp, int64_t ld_logp, const float* logq, int64_t ld_logq, const int64_t* idx, const float* c, float k,
                               float inv_temp, int32_t n, void* out, int64_t ld_out, int32_t col0, float* kl, int32_t accumulate, int64_t rows,
                               void* stream) {
    using namespace vpt;
    VPT_CHECK(logp && idx && c && out && kl && rows > 0 && n > 0 && col0 >= 0 && ld_logp >= n && ld_out >= col0 + (int64_t)n &&
                  (logq == nullptr || ld_logq >= n),
              "vpt_rl_head_bwd: bad arguments");
    const long long* ix = reinterpret_cast<const long long*>(idx);
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
    if (n <= 1024) {
        rl_head_bwd_kernel<32><<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(logp, ld_logp, logq, ld_logq, ix, c, k, inv_temp, n, o,
                                                                                           ld_out, col0, kl, accumulate, rows);
    } else {
        rl_head_bwd_kernel<256><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(logp, ld_logp, logq, ld_logq, ix, c, k, inv_temp, n, o, ld_out,
                                                                                 col0, kl, accumulate, rows);
    }
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_rl_head_bwd_ent(const float* logp, int64_t ld_logp, const float* logq, int64_t ld_logq, const int64_t* idx, const float* c,
                                   float k, float e, float inv_temp, int32_t n, void* out, int64_t ld_out, int32_t col0, float* kl, float* ent,
                                   int32_t accumulate, int64_t rows, void* stream) {
    using namespace vpt;
    VPT_CHECK(logp && idx && c && out && kl && ent && rows > 0 && n > 0 && col0 >= 0 && ld_logp >= n && ld_out >= col0 + (int64_t)n &&
                  (logq == nullptr || ld_logq >= n),
              "vpt_rl_head_bwd_ent: bad arguments");
    const long long* ix = reinterpret_cast<const long long*>(idx);
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
    if (n <= 1024) {
        rl_head_bwd_kernel<32, true><<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(logp, ld_logp, logq, ld_logq, ix, c, k,
                                                                                                 inv_temp, n, o, ld_out, col0, kl,
                                                                                                 accumulate, rows, e, ent);
    } else {
        rl_head_bwd_kernel<256, true><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(logp, ld_logp, logq, ld_logq, ix, c, k, inv_temp, n, o,
                                                                                       ld_out, col0, kl, accumulate, rows, e, ent);
    }
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_ewma_sums(const float* x, int64_t rows, double* sums, void* stream) {
    using namespace vpt;
    VPT_CHECK(x && sums && rows > 0, "vpt_ewma_sums: bad arguments");
    ewma_sums_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(x, rows, sums);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_value_bwd(const float* vpred, const float* returns, const double* sums, double count, float* running_mean, float* running_mean_sq,
                             float* debiasing_term, float w, float one_minus_w, float scale, void* out, int64_t ld_out, int32_t col, float* sq_err,
                             int64_t rows, void* stream) {
    using namespace vpt;
    VPT_CHECK(vpred && returns && sums && running_mean && running_mean_sq && debiasing_term && out && sq_err && rows > 0 && count > 0 && col >= 0 &&
                  ld_out > col,
              "vpt_value_bwd: bad arguments");
    value_bwd_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(vpred, returns, sums, count, running_mean, running_mean_sq, debiasing_term, w,
                                                          one_minus_w, scale, reinterpret_cast<__nv_bfloat16*>(out), ld_out, col,
                                                          sq_err, rows);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}
