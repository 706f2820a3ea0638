// fp32-parity precision mode (BASELINE north_star: "1e-3 rtol fp32"; the reference computes in fp32, lib/xf.py:40,55-63).
//
// The contraction work stays on the wgmma GEMM / implicit-GEMM kernel (gemm_tc.cuh): every operand is split into bf16 hi + lo
// parts and a layer is THREE accumulating launches  out = A_hi W_hi^T ; out += A_lo W_hi^T ; out = epi(out + A_hi W_lo^T)  with fp32
// accumulators in registers and an fp32 running sum in HBM (the dropped lo*lo term is 2^-18 relative).  Activations are kept in fp32
// between layers; the kernels below are the fp32 glue that the bf16 path folds into its epilogues: normalise + split, statistics,
// max-pool, residual add, and an fp32 attention.  Nothing here is performance-tuned -- this mode exists for the parity
// configurations (BASELINE configs[0] and the IDM tolerance), the bf16 path is the product.
#pragma once
#include "common.cuh"
#include "elementwise.cuh"

namespace vpt {

// (mean, rstd) per group of rows_per_group consecutive rows of an fp32 [rows][C] tensor; one block per group, fp64 accumulation
__global__ void __launch_bounds__(256) group_stats_f32_kernel(const float* __restrict__ x, float2* __restrict__ mr, long long per_group, float eps) {
    const float* gx = x + (long long)blockIdx.x * per_group;
    double s = 0.0, ss = 0.0;
    for (long long i = threadIdx.x; i < per_group; i += blockDim.x) {
        const double v = (double)gx[i];
        s += v;
        ss += v * v;
    }
    __shared__ double red[2][256];
    red[0][threadIdx.x] = s;
    red[1][threadIdx.x] = ss;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) {
            red[0][threadIdx.x] += red[0][threadIdx.x + o];
            red[1][threadIdx.x] += red[1][threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double mean = red[0][0] / (double)per_group;
        double var = red[1][0] / (double)per_group - mean * mean;
        if (var < 0.0) var = 0.0;
        mr[blockIdx.x] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
    }
}

// u = [(x - mean_g) * rstd_g] * gamma[c] + beta[c]  (each part optional)  ->  hi = bf16(u), lo = bf16(u - hi), and / or u itself
__global__ void __launch_bounds__(256) norm_split_f32_kernel(const float* __restrict__ x, const float2* __restrict__ mr, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, __nv_bfloat16* __restrict__ hi,
                                                               __nv_bfloat16* __restrict__ lo, float* __restrict__ out_f32, long long n, int C,
                                                               long long per_group) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float u = x[i];
        if (mr) {
            const float2 st = __ldg(mr + i / per_group);
            u = (u - st.x) * st.y;
        }
        const int c = (int)(i % C);
        if (gamma) u = u * __ldg(gamma + c);
        if (beta) u = u + __ldg(beta + c);
        if (hi) {
            const __nv_bfloat16 h = __float2bfloat16_rn(u);
            hi[i] = h;
            lo[i] = __float2bfloat16_rn(u - __bfloat162float(h));
        }
        if (out_f32) out_f32[i] = u;
    }
}

// out = a + b (optionally ReLU'd)
__global__ void __launch_bounds__(256) add_f32_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, long long n, int relu) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float v = a[i] + (b ? b[i] : 0.f);
        if (relu) v = fmaxf(v, 0.f);
        out[i] = v;
    }
}

// max_pool2d(kernel 3, stride 2, padding 1) on fp32 NHWC
__global__ void __launch_bounds__(256) maxpool3s2_f32_kernel(const float* __restrict__ in, float* __restrict__ out, long long F, int H, int W, int C) {
    const int Ho = H / 2, Wo = W / 2;
    const long long n = F * Ho * Wo * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        long long r = i / C;
        const int px = (int)(r % Wo);
        r /= Wo;
        const int py = (int)(r % Ho);
        const long long f = r / Ho;
        float m = -INFINITY;
        for (int dy = -1; dy <= 1; ++dy)
            for (int dx = -1; dx <= 1; ++dx) {
                const int y = 2 * py + dy, x = 2 * px + dx;
                if (y >= 0 && y < H && x >= 0 && x < W) m = fmaxf(m, in[((f * H + y) * W + x) * C + c]);
            }
        out[i] = m;
    }
}

// fp32 attention of one (batch row, head, query) per block of 128 threads (head_dim == 128), lib/xf.py:18-71 + the closed-form mask of
// lib/masked_attention.py:11-94 and the relative-position term of lib/xf.py:265-271 (see attention.cuh for the bf16 kernel).
__global__ void __launch_bounds__(128) attention_f32_kernel(const float* __restrict__ q, const float* __restrict__ fk, const float* __restrict__ fv,
                                                              const float* __restrict__ R, const float* __restrict__ b_nd, const uint8_t* __restrict__ first,
                                                              const uint8_t* __restrict__ smask, float* __restrict__ out, int B, int t, int maxlen,
                                                              int heads, int causal) {
    constexpr int DH = 128, NB = 10;
    const int T = maxlen + t;
    const int i = blockIdx.x % t, hd = (blockIdx.x / t) % heads, b = blockIdx.x / (t * heads);
    const int h = heads * DH;
    __shared__ float sq[DH];
    extern __shared__ float sp[];  // [maxlen + t] logits, then probabilities
    __shared__ float sr[NB];
    __shared__ float red[4];
    const int tid = threadIdx.x;
    sq[tid] = q[((long long)b * t + i) * h + hd * DH + tid];
    if (tid < NB && R) sr[tid] = R[((long long)b * t + i) * (NB * heads) + hd * NB + tid];
    __syncthreads();
    const bool fst = causal && first[(long long)b * t] != 0;  // only first[:, 0] is read (lib/masked_attention.py:167)
    float lmax = -INFINITY;
    for (int j = tid; j < T; j += 128) {
        const int d = (T - t + i) - j;
        bool ok = true;
        if (causal) {
            ok = d >= 0 && d < maxlen;
            if (ok && j < T - t) ok = !fst && smask != nullptr && smask[(long long)b * maxlen + j] != 0;
        }
        const float* kr = fk + ((long long)b * T + j) * h + hd * DH;
        float acc = 0.f;
        for (int e = 0; e < DH; ++e) acc = fmaf(sq[e], kr[e], acc);
        float bias = ok ? 0.f : -1e9f;                           // lib/xf.py:46
        if (causal && R && d >= 0 && d < maxlen) {
            float ex = 0.f;
            for (int n = 0; n < NB; ++n) ex = fmaf(sr[n], __ldg(b_nd + n * maxlen + d), ex);
            bias += ex;
        }
        const float lg = acc * (1.0f / DH) + bias;               // muP 1/dh scale (lib/xf.py:59)
        sp[j] = lg;
        lmax = fmaxf(lmax, lg);
    }
    lmax = warp_max(lmax);
    if ((tid & 31) == 0) red[tid >> 5] = lmax;
    __syncthreads();
    lmax = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    __syncthreads();
    float lsum = 0.f;
    for (int j = tid; j < T; j += 128) {
        const float pj = expf(sp[j] - lmax);
        sp[j] = pj;
        lsum += pj;
    }
    lsum = warp_sum(lsum);
    if ((tid & 31) == 0) red[tid >> 5] = lsum;
    __syncthreads();
    const float inv = 1.0f / (red[0] + red[1] + red[2] + red[3]);
    float o = 0.f;
    for (int j = 0; j < T; ++j) o = fmaf(sp[j], fv[((long long)b * T + j) * h + hd * DH + tid], o);
    out[((long long)b * t + i) * h + hd * DH + tid] = o * inv;
}

}  // namespace vpt

extern "C" int vpt_group_stats_f32(const float* x, float* mr, int64_t groups, int64_t per_group, float eps, void* stream) {
    using namespace vpt;
    VPT_CHECK(x && mr && groups > 0 && per_group > 0, "vpt_group_stats_f32: bad argument");
    group_stats_f32_kernel<<<(unsigned)groups, 256, 0, (cudaStream_t)stream>>>(x, reinterpret_cast<float2*>(mr), per_group, eps);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_norm_split_f32(const float* x, const float* mr, const float* gamma, const float* beta, void* hi, void* lo, float* out_f32,
                                  int64_t n, int32_t C, int64_t per_group, void* stream) {
    using namespace vpt;
    VPT_CHECK(x && n > 0 && C > 0 && (hi || out_f32) && (!hi == !lo), "vpt_norm_split_f32: bad argument");
    VPT_CHECK(!mr || per_group > 0, "vpt_norm_split_f32: per_group must be > 0 with mr");
    norm_split_f32_kernel<<<vpt_blocks_for(n, 1024, 4096), 256, 0, (cudaStream_t)stream>>>(
        x, reinterpret_cast<const float2*>(mr), gamma, beta, reinterpret_cast<__nv_bfloat16*>(hi), reinterpret_cast<__nv_bfloat16*>(lo), out_f32, n, C,
        per_group > 0 ? per_group : 1);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_add_f32(const float* a, const float* b, float* out, int64_t n, int32_t relu, void* stream) {
    using namespace vpt;
    VPT_CHECK(a && out && n > 0, "vpt_add_f32: bad argument");
    add_f32_kernel<<<vpt_blocks_for(n, 1024, 4096), 256, 0, (cudaStream_t)stream>>>(a, b, out, n, relu);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_maxpool3s2_f32(const float* in, float* out, int64_t F, int32_t H, int32_t W, int32_t C, void* stream) {
    using namespace vpt;
    VPT_CHECK(in && out && F > 0 && H % 2 == 0 && W % 2 == 0, "vpt_maxpool3s2_f32: bad argument");
    maxpool3s2_f32_kernel<<<vpt_blocks_for(F * (H / 2) * (W / 2) * C, 1024, 8192), 256, 0, (cudaStream_t)stream>>>(in, out, F, H, W, C);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_attention_f32(const float* q, const float* full_k, const float* full_v, const float* R, const float* b_nd, const uint8_t* first,
                                 const uint8_t* state_mask, float* out, int32_t B, int32_t t, int32_t maxlen, int32_t heads, int32_t causal,
                                 void* stream) {
    using namespace vpt;
    VPT_CHECK(q && full_k && full_v && out && B > 0 && t > 0 && heads > 0 && maxlen >= 0, "vpt_attention_f32: bad argument");
    const size_t smem = (size_t)(maxlen + t) * 4;  // the score row of one query
    VPT_CHECK(smem <= 200 * 1024, "vpt_attention_f32: at most %d keys per query (maxlen=%d t=%d)", 200 * 1024 / 4, maxlen, t);
    VPT_CHECK(!causal || (first && (!R || b_nd)), "vpt_attention_f32: causal attention needs `first` (and b_nd with R)");
    // Without the opt-in, static and dynamic shared memory together are limited to 48 KB: the kernel's own static arrays count too.
    static size_t static_smem = 0, attr = 0;
    if (static_smem == 0) {
        cudaFuncAttributes fa;
        VPT_CUDA(cudaFuncGetAttributes(&fa, attention_f32_kernel));
        static_smem = fa.sharedSizeBytes;
    }
    if (static_smem + smem > 48 * 1024 && smem > attr) {
        VPT_CUDA(cudaFuncSetAttribute(attention_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr = 200 * 1024;
    }
    attention_f32_kernel<<<(unsigned)(B * heads * t), 128, smem, (cudaStream_t)stream>>>(q, full_k, full_v, R, b_nd, first, state_mask, out, B, t, maxlen, heads,
                                                                                      causal);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}
