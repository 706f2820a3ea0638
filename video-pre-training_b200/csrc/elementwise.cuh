// HBM-bound helper kernels of the CNN / transformer path: statistics finalisation, max-pool, affine normalisation
// (GroupNorm(1) / LayerNorm application), KV-memory row copies, state-mask roll.  All are coalesced 16-byte-vector
// streaming kernels; grids are sized from the data (>= several waves of 148 SMs at bench sizes).
#pragma once
#include "common.cuh"

namespace vpt {

// block-wide (sum, sumsq) reduction in a fixed order (deterministic); result valid in thread 0
__device__ __forceinline__ float2 block_sum2(float s, float ss) {
    __shared__ float red[2][32];
    s = warp_sum(s);
    ss = warp_sum(ss);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    if (l == 0) {
        red[0][w] = s;
        red[1][w] = ss;
    }
    __syncthreads();
    float2 r = make_float2(0.f, 0.f);
    if (w == 0) {
        float a = l < nw ? red[0][l] : 0.f, b = l < nw ? red[1][l] : 0.f;
        a = warp_sum(a);
        b = warp_sum(b);
        r = make_float2(a, b);
    }
    __syncthreads();
    return r;
}

// ---------------------------------------------------------------------------------------------------------
// mr[g] = (mean, rstd) from float2 partials
// ---------------------------------------------------------------------------------------------------------
__global__ void stats_finalize_kernel(const float2* __restrict__ part, float2* __restrict__ mr, long long G, int n_per_group,
                                      double inv_count, float eps) {
    pdl_sync();
    // one warp per group; lanes stride over the partials, doubles for the final combination
    const long long g = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (g >= G) return;
    const int lane = threadIdx.x & 31;
    double s = 0.0, ss = 0.0;
    const float2* p = part + g * n_per_group;
    for (int i = lane; i < n_per_group; i += 32) {
        float2 v = __ldg(p + i);
        s += (double)v.x;
        ss += (double)v.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
    }
    if (lane == 0) {
        const double mean = s * inv_count;
        double var = ss * inv_count - mean * mean;
        if (var < 0.0) var = 0.0;
        mr[g] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
    }
}

// large groups (a conv frame has thousands of per-row partials): one 256-thread block per group, fixed-order tree
__global__ void __launch_bounds__(256) stats_finalize_block_kernel(const float2* __restrict__ part, float2* __restrict__ mr, int n_per_group,
                                                                     double inv_count, float eps) {
    pdl_sync();
    __shared__ double red[2][8];
    const long long g = blockIdx.x;
    const float2* p = part + g * (long long)n_per_group;
    double s = 0.0, ss = 0.0;
    for (int i = threadIdx.x; i < n_per_group; i += 256) {
        const float2 v = __ldg(p + i);
        s += (double)v.x;
        ss += (double)v.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
    }
    if ((threadIdx.x & 31) == 0) {
        red[0][threadIdx.x >> 5] = s;
        red[1][threadIdx.x >> 5] = ss;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        s = ss = 0.0;
        for (int w = 0; w < 8; ++w) {
            s += red[0][w];
            ss += red[1][w];
        }
        const double mean = s * inv_count;
        double var = ss * inv_count - mean * mean;
        if (var < 0.0) var = 0.0;
        mr[g] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
    }
}

// ---------------------------------------------------------------------------------------------------------
// max_pool2d(3, 2, 1) on non-negative NHWC bf16; 8 channels (16 B) per thread; grid = (blocks_per_frame, F)
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t bf16x2_max(uint32_t a, uint32_t b) {
    __nv_bfloat162 x = *reinterpret_cast<__nv_bfloat162*>(&a), y = *reinterpret_cast<__nv_bfloat162*>(&b);
    __nv_bfloat162 r = __hmax2(x, y);
    return *reinterpret_cast<uint32_t*>(&r);
}

// chan_part (optional, needs 256 % C8 == 0 so that a thread keeps one channel group): float2 [F][gridDim.x][C] per-CHANNEL (sum, sumsq)
// partials of the pooled values -- what the two-norm composition (vpt_norm2_fold) needs instead of a normalisation pass.
// (CHAN keeps 16 more accumulators: 48 registers -> 5 resident blocks instead of 8, and this kernel lives on loads in flight; two
//  items per trip and a 4-block bound give each thread twice the loads instead)
// One thread = one 8-channel group of a 2 x 2 block of outputs: the 5 x 5 input window is read once (6.25 loads per output instead of 9)
// and the maximum is separable -- per input row two horizontal 3-maxima, folded into the two output rows that row belongs to.
template <bool CHAN>
__global__ void __launch_bounds__(256, 2) maxpool3s2_kernel(const uint4* __restrict__ in, uint4* __restrict__ out,
                                                           float2* __restrict__ stat_part, float2* __restrict__ chan_part, int H, int W, int C8, int zp) {
    pdl_sync();
    const int Ho = H >> 1, Wo = W >> 1;
    const int ipitch = W + zp, opitch = Wo + zp;  // ZP layout: one extra zero column (and row) per frame
    const int orows = Ho + zp;
    const int nbx = (opitch + 1) >> 1, nby = (orows + 1) >> 1;
    const long long f = blockIdx.y;
    const int items = nby * nbx * C8;
    const uint4* fin = in + f * (long long)(H + zp) * ipitch * C8;
    uint4* fout = out + f * (long long)orows * opitch * C8;
    float s = 0.f, ss = 0.f;
    float cs[8], css[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) cs[j] = css[j] = 0.f;
    auto max4 = [](uint4 a, const uint4 b) {
        a.x = bf16x2_max(a.x, b.x); a.y = bf16x2_max(a.y, b.y); a.z = bf16x2_max(a.z, b.z); a.w = bf16x2_max(a.w, b.w);
        return a;
    };
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < items; i += gridDim.x * blockDim.x) {
        const int c = i % C8, bx = (i / C8) % nbx, by = i / (C8 * nbx);
        const uint4 zero = make_uint4(0, 0, 0, 0);  // inputs are >= 0 (post-ReLU), so 0 == -inf padding
        uint4 o[2][2] = {{zero, zero}, {zero, zero}};
        const int x0 = 4 * bx - 1, y0 = 4 * by - 1;
#pragma unroll
        for (int r = 0; r < 5; ++r) {
            const int y = y0 + r;
            if (y < 0 || y >= H) continue;
            const uint4* row = fin + ((long long)y * ipitch + x0) * C8 + c;
            uint4 v[5];
#pragma unroll
            for (int q = 0; q < 5; ++q) v[q] = (x0 + q >= 0 && x0 + q < W) ? __ldg(row + (long long)q * C8) : zero;
            const uint4 h0 = max4(max4(v[0], v[1]), v[2]), h1 = max4(max4(v[2], v[3]), v[4]);
            if (r <= 2) { o[0][0] = max4(o[0][0], h0); o[0][1] = max4(o[0][1], h1); }
            if (r >= 2) { o[1][0] = max4(o[1][0], h0); o[1][1] = max4(o[1][1], h1); }
        }
#pragma unroll
        for (int ry = 0; ry < 2; ++ry) {
#pragma unroll
            for (int rx = 0; rx < 2; ++rx) {
                const int oy = 2 * by + ry, ox = 2 * bx + rx;
                if (oy >= orows || ox >= opitch) continue;
                const uint4 m = (oy < Ho && ox < Wo) ? o[ry][rx] : zero;  // zero column / row of the ZP output
                fout[((long long)oy * opitch + ox) * C8 + c] = m;
                const uint32_t w4[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float a = bf16_lo(w4[q]), b = bf16_hi(w4[q]);
                    if (CHAN) {  // per-channel sums; the frame sums are their total
                        cs[2 * q] += a; css[2 * q] = fmaf(a, a, css[2 * q]);
                        cs[2 * q + 1] += b; css[2 * q + 1] = fmaf(b, b, css[2 * q + 1]);
                    } else {
                        s += a + b;
                        ss = fmaf(a, a, fmaf(b, b, ss));
                    }
                }
            }
        }
    }
    if (CHAN) {  // deterministic block reduction over the 256 / C8 threads that share a channel group
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s += cs[j];
            ss += css[j];
        }
        __shared__ float red[256 * 16];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            red[threadIdx.x * 16 + j] = cs[j];
            red[threadIdx.x * 16 + 8 + j] = css[j];
        }
        __syncthreads();
        for (int k = threadIdx.x; k < C8 * 8; k += blockDim.x) {
            const int c8 = k >> 3, j = k & 7;
            float a = 0.f, b = 0.f;
            for (int t = c8; t < 256; t += C8) {
                a += red[t * 16 + j];
                b += red[t * 16 + 8 + j];
            }
            chan_part[(f * gridDim.x + blockIdx.x) * (long long)(C8 * 8) + k] = make_float2(a, b);
        }
        __syncthreads();
    }
    if (stat_part) {
        const float2 r = block_sum2(s, ss);
        if (threadIdx.x == 0) stat_part[f * gridDim.x + blockIdx.x] = r;
    }
}

// ---------------------------------------------------------------------------------------------------------
// Two-norm composition (see vpt_norm2_fold in include/vpt_b200.h): one block per frame, fp64
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) norm2_fold_kernel(const float2* __restrict__ chan_part, int NP, int C, double npix, const float* __restrict__ gn,
                                                           const float* __restrict__ bn, const float* __restrict__ Ta, const float* __restrict__ Tb,
                                                           const float* __restrict__ Tc, const float* __restrict__ Td, int Cout, float eps,
                                                           float2* __restrict__ mrE, float* __restrict__ Ef, float* __restrict__ res_scale,
                                                           float* __restrict__ res_shift) {
    pdl_sync();
    const long long f = blockIdx.x;
    __shared__ double S[512], Q[512];
    __shared__ double red[256];
    const int t = threadIdx.x;
    double s = 0.0, q = 0.0;
    for (int c = t; c < C; c += 256) {
        double a = 0.0, b = 0.0;
        for (int p = 0; p < NP; ++p) {
            const float2 v = chan_part[(f * NP + p) * (long long)C + c];
            a += (double)v.x;
            b += (double)v.y;
        }
        S[c] = a;
        Q[c] = b;
        s += a;
        q += b;
    }
    auto block_sum = [&](double v) {
        __syncthreads();
        red[t] = v;
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) {
            if (t < o) red[t] += red[t + o];
            __syncthreads();
        }
        return red[0];
    };
    const double cnt = npix * (double)C;
    const double sum1 = block_sum(s), sq1 = block_sum(q);
    const double mu1 = sum1 / cnt;
    double var1 = sq1 / cnt - mu1 * mu1;
    if (var1 < 0.0) var1 = 0.0;
    const double rstd1 = 1.0 / sqrt(var1 + (double)eps);
    // x0 = a_c * y1 + b_c (the post-pool GroupNorm); its per-frame statistics follow from the per-channel sums
    double m0 = 0.0, e0 = 0.0;
    for (int c = t; c < C; c += 256) {
        const double a = rstd1 * (double)gn[c], b = (double)bn[c] - mu1 * a;
        m0 += a * S[c] + npix * b;
        e0 += a * a * Q[c] + 2.0 * a * b * S[c] + npix * b * b;
        res_scale[f * C + c] = (float)a;
        res_shift[f * C + c] = (float)b;
    }
    const double sum0 = block_sum(m0), sq0 = block_sum(e0);
    const double mu0 = sum0 / cnt;
    double var0 = sq0 / cnt - mu0 * mu0;
    if (var0 < 0.0) var0 = 0.0;
    const double rstd0 = 1.0 / sqrt(var0 + (double)eps);
    const double R = rstd0 * rstd1;
    if (t == 0) mrE[f] = make_float2(0.f, (float)R);
    for (int k = t; k < 9 * Cout; k += 256)
        Ef[f * 9 * Cout + k] = (float)(rstd0 * (double)Ta[k] - R * mu1 * (double)Tb[k] - rstd0 * mu0 * (double)Tc[k] + (double)Td[k]);
}

// ---------------------------------------------------------------------------------------------------------
// out = (in - mean_g) * rstd_g * gamma[c] + beta[c]; grid = (blocks_per_group, G)
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) affine_norm_kernel(const uint4* __restrict__ in, const float2* __restrict__ mr,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            uint4* __restrict__ out, float* __restrict__ out_f32,
                                                            float2* __restrict__ stat_part, long long items_per_group, int C8) {
    pdl_sync();
    const long long g = blockIdx.y;
    const float2 st = __ldg(mr + g);
    const float mean = st.x, rstd = st.y;
    const uint4* gin = in + g * items_per_group;
    uint4* gout = out + g * items_per_group;
    float s = 0.f, ss = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items_per_group; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C8) * 8;
        const uint4 v = __ldg(gin + i);
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c) + 1);
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c) + 1);
        float x[8] = {bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y), bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w)};
        const float ga[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float be[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = fmaf((x[j] - mean) * rstd, ga[j], be[j]);
        uint4 o;
        o.x = pack_bf16(x[0], x[1]); o.y = pack_bf16(x[2], x[3]); o.z = pack_bf16(x[4], x[5]); o.w = pack_bf16(x[6], x[7]);
        gout[i] = o;
        if (out_f32) {
            float4* of = reinterpret_cast<float4*>(out_f32 + (g * items_per_group + i) * 8);
            of[0] = make_float4(x[0], x[1], x[2], x[3]);
            of[1] = make_float4(x[4], x[5], x[6], x[7]);
        }
        const uint32_t w4[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float a = bf16_lo(w4[q]), b = bf16_hi(w4[q]);
            s += a + b;
            ss = fmaf(a, a, fmaf(b, b, ss));
        }
    }
    if (stat_part) {
        const float2 r = block_sum2(s, ss);
        if (threadIdx.x == 0) stat_part[g * gridDim.x + blockIdx.x] = r;
    }
}

// ZP variant: one group per frame, [H+1][W+1][C8] items; the zero row / column is rewritten as zero
__global__ void __launch_bounds__(256) affine_norm_zp_kernel(const uint4* __restrict__ in, const float2* __restrict__ mr,
                                                               const float* __restrict__ gamma, const float* __restrict__ beta,
                                                               uint4* __restrict__ out, float2* __restrict__ stat_part, int H, int W, int C8) {
    pdl_sync();
    const long long g = blockIdx.y;
    const float2 st = __ldg(mr + g);
    const float mean = st.x, rstd = st.y;
    const int Wp = W + 1;
    const long long items = (long long)(H + 1) * Wp * C8;
    const uint4* gin = in + g * items;
    uint4* gout = out + g * items;
    float s = 0.f, ss = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C8) * 8;
        const int pix = (int)(i / C8);
        const int y = pix / Wp, x = pix - y * Wp;
        if (y >= H || x >= W) {
            gout[i] = make_uint4(0, 0, 0, 0);
            continue;
        }
        const uint4 v = __ldg(gin + i);
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c) + 1);
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c) + 1);
        float xv[8] = {bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y), bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w)};
        const float ga[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float be[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) xv[j] = fmaf((xv[j] - mean) * rstd, ga[j], be[j]);
        uint4 o;
        o.x = pack_bf16(xv[0], xv[1]); o.y = pack_bf16(xv[2], xv[3]); o.z = pack_bf16(xv[4], xv[5]); o.w = pack_bf16(xv[6], xv[7]);
        gout[i] = o;
        const uint32_t w4[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float a = bf16_lo(w4[q]), b = bf16_hi(w4[q]);
            s += a + b;
            ss = fmaf(a, a, fmaf(b, b, ss));
        }
    }
    if (stat_part) {
        const float2 r = block_sum2(s, ss);
        if (threadIdx.x == 0) stat_part[g * gridDim.x + blockIdx.x] = r;
    }
}

// Same result, fewer instructions (ncu: the kernel above executes ~150 instructions per 32 bytes moved, mostly index
// arithmetic, and stops at ~72 % of HBM bandwidth): every thread keeps ONE channel vector (gamma / beta stay in registers) and
// walks pixels with an incrementally updated (y, x); threads [0, PL*C8) of a block cover PL = 256 / C8 consecutive pixels.
__global__ void __launch_bounds__(256) affine_norm_zp_rows_kernel(const uint4* __restrict__ in, const float2* __restrict__ mr,
                                                                    const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                    uint4* __restrict__ out, float2* __restrict__ stat_part, int H, int W, int C8) {
    pdl_sync();
    const long long g = blockIdx.y;
    const float2 st = __ldg(mr + g);
    const float mean = st.x, rstd = st.y;
    const int Wp = W + 1, npix = (H + 1) * Wp;
    const int PL = 256 / C8;
    const uint4* gin = in + g * (long long)npix * C8;
    uint4* gout = out + g * (long long)npix * C8;
    float s = 0.f, ss = 0.f;
    if ((int)threadIdx.x < PL * C8) {
        const int c8 = threadIdx.x % C8, pl = threadIdx.x / C8;
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c8 * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c8 * 8) + 1);
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c8 * 8)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c8 * 8) + 1);
        const float ga[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float be[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        const int dp = gridDim.x * PL;            // pixels advanced per trip
        const int dy = dp / Wp, dx = dp - dy * Wp;
        int pix = blockIdx.x * PL + pl;
        int y = pix / Wp, x = pix - y * Wp;
        // four pixels per trip with the loads issued first: one 16-byte load in flight per thread kept the kernel at ~67 % of the HBM
        // copy bandwidth (round-2 launch list: 13 ms / step for 57.6 GB); four in flight cover the ~1 us memory latency
        constexpr int U = 4;
        while (pix < npix) {
            uint4 v[U];
            int kind[U];  // 0: beyond the frame, 1: zero row / column, 2: interior
            long long idx[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                kind[u] = pix >= npix ? 0 : ((y >= H || x >= W) ? 1 : 2);
                idx[u] = (long long)pix * C8 + c8;
                if (kind[u] == 2) v[u] = __ldg(gin + idx[u]);
                pix += dp;
                x += dx;
                y += dy;
                if (x >= Wp) {
                    x -= Wp;
                    ++y;
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (kind[u] == 1) {
                    gout[idx[u]] = make_uint4(0, 0, 0, 0);
                } else if (kind[u] == 2) {
                    float xv[8] = {bf16_lo(v[u].x), bf16_hi(v[u].x), bf16_lo(v[u].y), bf16_hi(v[u].y),
                                   bf16_lo(v[u].z), bf16_hi(v[u].z), bf16_lo(v[u].w), bf16_hi(v[u].w)};
#pragma unroll
                    for (int j = 0; j < 8; ++j) xv[j] = fmaf((xv[j] - mean) * rstd, ga[j], be[j]);
                    uint4 o;
                    o.x = pack_bf16(xv[0], xv[1]); o.y = pack_bf16(xv[2], xv[3]); o.z = pack_bf16(xv[4], xv[5]); o.w = pack_bf16(xv[6], xv[7]);
                    gout[idx[u]] = o;
                    const uint32_t w4[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float a = bf16_lo(w4[q]), b = bf16_hi(w4[q]);
                        s += a + b;
                        ss = fmaf(a, a, fmaf(b, b, ss));
                    }
                }
            }
        }
    }
    if (stat_part) {
        const float2 r = block_sum2(s, ss);
        if (threadIdx.x == 0) stat_part[g * gridDim.x + blockIdx.x] = r;
    }
}

// ---------------------------------------------------------------------------------------------------------
// strided row copy with fp32 <-> bf16 conversion (KV memory load/store); 8 elements per thread
// ---------------------------------------------------------------------------------------------------------
template <bool SRC_F32, bool DST_F32>
__global__ void __launch_bounds__(256) copy_rows_kernel(const void* __restrict__ src0, const void* __restrict__ src1, long long src_bstride,
                                                          long long src_ld, long long src_off, void* __restrict__ dst0, void* __restrict__ dst1,
                                                          long long dst_bstride, long long dst_ld, long long dst_off, int rows, int cols8) {
    pdl_sync();
    // blockIdx.z selects one of two (source, destination) pairs of identical geometry (K and V of a layer in one launch)
    const void* src = blockIdx.z ? src1 : src0;
    void* dst = blockIdx.z ? dst1 : dst0;
    const int b = blockIdx.y;
    const long long n = (long long)rows * cols8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols8), c = (int)(i % cols8) * 8;
        const long long so = b * src_bstride + (src_off + r) * src_ld + c;
        const long long dofs = b * dst_bstride + (dst_off + r) * dst_ld + c;
        float x[8];
        if (SRC_F32) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(src) + so));
            const float4 bb = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(src) + so) + 1);
            x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = bb.x; x[5] = bb.y; x[6] = bb.z; x[7] = bb.w;
        } else {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(src) + so));
            x[0] = bf16_lo(v.x); x[1] = bf16_hi(v.x); x[2] = bf16_lo(v.y); x[3] = bf16_hi(v.y);
            x[4] = bf16_lo(v.z); x[5] = bf16_hi(v.z); x[6] = bf16_lo(v.w); x[7] = bf16_hi(v.w);
        }
        if (DST_F32) {
            float4* o = reinterpret_cast<float4*>(reinterpret_cast<float*>(dst) + dofs);
            o[0] = make_float4(x[0], x[1], x[2], x[3]);
            o[1] = make_float4(x[4], x[5], x[6], x[7]);
        } else {
            uint4 o;
            o.x = pack_bf16(x[0], x[1]); o.y = pack_bf16(x[2], x[3]); o.z = pack_bf16(x[4], x[5]); o.w = pack_bf16(x[6], x[7]);
            *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(dst) + dofs) = o;
        }
    }
}

__global__ void state_mask_update_kernel(const uint8_t* __restrict__ mask_in, const uint8_t* __restrict__ first, long long first_stride,
                                         uint8_t* __restrict__ mask_out, int B, int t, int maxlen) {
    pdl_sync();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * maxlen) return;
    const int b = i / maxlen, j = i % maxlen;
    const int keep = maxlen - min(t, maxlen);  // old entries that survive the roll
    uint8_t v = 1;
    if (j < keep) {
        const uint8_t old = mask_in ? mask_in[(long long)b * maxlen + j + t] : 0;
        v = (old != 0 && first[b * first_stride] == 0) ? 1 : 0;
    }
    mask_out[i] = v;
}

}  // namespace vpt

extern "C" int vpt_stats_finalize(const float* stat_part, float* mr, int64_t G, int32_t n_per_group, double count, float eps,
                                  void* stream) {
    using namespace vpt;
    VPT_CHECK(stat_part && mr && G > 0 && n_per_group > 0 && count > 0, "vpt_stats_finalize: bad arguments");
    if (n_per_group >= 512) {
        launch_k(stats_finalize_block_kernel, dim3((unsigned)G), dim3(256), 0, (cudaStream_t)stream, reinterpret_cast<const float2*>(stat_part),
                                                                                   reinterpret_cast<float2*>(mr), n_per_group, 1.0 / count, eps);
        VPT_LAUNCH_CHECK();
        return VPT_OK;
    }
    const int wpb = 8;
    const long long blocks = (G + wpb - 1) / wpb;
    launch_k(stats_finalize_kernel, dim3((unsigned)blocks), dim3(wpb * 32), 0, (cudaStream_t)stream, 
        reinterpret_cast<const float2*>(stat_part), reinterpret_cast<float2*>(mr), G, n_per_group, 1.0 / count, eps);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

static inline int vpt_blocks_for(long long items, int per_block, int cap) {
    long long b = (items + per_block - 1) / per_block;
    if (b < 1) b = 1;
    if (b > cap) b = cap;
    return (int)b;
}

// blocks per frame of the pooling kernel = entries per frame of its partial buffers.  A handful of frames (rollout: F = 1): enough blocks
// to put work on every SM (a 64 x 64 x 256 frame would otherwise be pooled by 4 blocks: 64 us of a 1.3 ms step).  Only for F <= 16: the
// partial count fixes the summation order of the statistics, and batch runs promise bit-identical rows whatever the batch size.
static inline int pool_parts(int F, int H, int W, int C, int per_block, int cap) {
    const long long items = (long long)(H / 2) * (W / 2) * (C / 8);
    int p = vpt_blocks_for(items, per_block, cap);
    if (F <= 16 && (long long)F * p < 2 * 148) {
        long long want = (2 * 148 + F - 1) / F, most = items / 256 > 0 ? items / 256 : 1;  // at least one item per thread
        if (want > most) want = most;
        if (want > 256) want = 256;
        if (want > p) p = (int)want;
    }
    return p;
}
extern "C" int vpt_pool_stat_parts(int32_t F, int32_t H, int32_t W, int32_t C) { return pool_parts(F, H, W, C, 2048, 64); }
/* With per-channel partials every block ends with a 16 KB shared-memory reduction: 4x fewer, 4x longer blocks amortise it
 * (measured: the pool was 50 % slower with the per-frame block count above). */
extern "C" int vpt_pool_chan_parts(int32_t F, int32_t H, int32_t W, int32_t C) { return pool_parts(F, H, W, C, 8192, 16); }

extern "C" int vpt_norm2_fold(const float* chan_part, int32_t NP, int32_t C, int64_t npix, const float* gamma_n, const float* beta_n, const float* Ta,
                              const float* Tb, const float* Tc, const float* Td, int32_t Cout, float eps, float* mrE, float* Ef, float* res_scale,
                              float* res_shift, int64_t F, void* stream) {
    using namespace vpt;
    VPT_CHECK(chan_part && gamma_n && beta_n && Ta && Tb && Tc && Td && mrE && Ef && res_scale && res_shift && F > 0, "vpt_norm2_fold: null argument");
    VPT_CHECK(C > 0 && C <= 512 && NP > 0 && Cout > 0, "vpt_norm2_fold: need 0 < C <= 512 (C=%d)", C);
    launch_k(norm2_fold_kernel, dim3((unsigned)F), dim3(256), 0, (cudaStream_t)stream, reinterpret_cast<const float2*>(chan_part), NP, C, (double)npix, gamma_n, beta_n, Ta, Tb,
                                                                    Tc, Td, Cout, eps, reinterpret_cast<float2*>(mrE), Ef, res_scale, res_shift);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

// plan_frames: the frame count whose blocks per frame (= statistics partials per frame) the call runs; vpt_maxpool3s2 passes F
extern "C" int vpt_maxpool3s2_plan(const void* in, void* out, float* stat_part, float* chan_part, int32_t F, int32_t H, int32_t W, int32_t C,
                                   int32_t zp, int32_t plan_frames, void* stream) {
    using namespace vpt;
    VPT_CHECK(in && out && F > 0, "vpt_maxpool3s2: null argument");
    VPT_CHECK(!chan_part || (C >= 8 && 256 % (C / 8) == 0), "vpt_maxpool3s2: per-channel partials need C/8 to divide 256 (C=%d)", C);
    VPT_CHECK(H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "vpt_maxpool3s2: need even H, W and C %% 8 == 0 (H=%d W=%d C=%d)", H, W, C);
    VPT_CHECK(F <= 65535, "vpt_maxpool3s2: at most 65535 frames per call (got %d)", F);
    VPT_CHECK(plan_frames > 0, "vpt_maxpool3s2_plan: plan_frames=%d must be > 0", plan_frames);
    dim3 grid(chan_part ? vpt_pool_chan_parts(plan_frames, H, W, C) : vpt_pool_stat_parts(plan_frames, H, W, C), F);
    if (chan_part)
        launch_k(maxpool3s2_kernel<true>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out),
                                                                      reinterpret_cast<float2*>(stat_part), reinterpret_cast<float2*>(chan_part), H, W, C / 8, zp ? 1 : 0);
    else
        launch_k(maxpool3s2_kernel<false>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out),
                                                                       reinterpret_cast<float2*>(stat_part), nullptr, H, W, C / 8, zp ? 1 : 0);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_maxpool3s2(const void* in, void* out, float* stat_part, float* chan_part, int32_t F, int32_t H, int32_t W, int32_t C, int32_t zp,
                              void* stream) {
    return vpt_maxpool3s2_plan(in, out, stat_part, chan_part, F, H, W, C, zp, F, stream);
}

extern "C" int vpt_norm_stat_parts(int32_t rows_per_group, int32_t C) {
    return vpt_blocks_for((long long)rows_per_group * (C / 8), 2048, 64);
}

extern "C" int vpt_affine_norm(const void* in, const float* mr, const float* gamma, const float* beta, void* out, float* out_f32,
                               float* stat_part, int64_t M, int32_t C, int32_t rows_per_group, void* stream) {
    using namespace vpt;
    VPT_CHECK(in && mr && gamma && beta && out, "vpt_affine_norm: null argument");
    VPT_CHECK(C % 8 == 0 && rows_per_group > 0 && M % rows_per_group == 0, "vpt_affine_norm: need C %% 8 == 0 and M %% rows_per_group == 0");
    const long long G = M / rows_per_group;
    const long long items = (long long)rows_per_group * (C / 8);
    const int bpg = vpt_norm_stat_parts(rows_per_group, C);
    // grid.y is limited to 65535: loop over slabs of groups
    for (long long g0 = 0; g0 < G; g0 += 65535) {
        const long long gn = (G - g0 < 65535) ? (G - g0) : 65535;
        dim3 grid(bpg, (unsigned)gn);
        launch_k(affine_norm_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, 
            reinterpret_cast<const uint4*>(in) + g0 * items, reinterpret_cast<const float2*>(mr) + g0, gamma, beta,
            reinterpret_cast<uint4*>(out) + g0 * items, out_f32 ? out_f32 + g0 * items * 8 : nullptr,
            stat_part ? reinterpret_cast<float2*>(stat_part) + g0 * bpg : nullptr, items, C / 8);
        VPT_LAUNCH_CHECK();
    }
    return VPT_OK;
}

extern "C" int vpt_affine_norm_zp(const void* in, const float* mr, const float* gamma, const float* beta, void* out, float* stat_part,
                                  int32_t F, int32_t H, int32_t W, int32_t C, void* stream) {
    using namespace vpt;
    VPT_CHECK(in && mr && gamma && beta && out && F > 0, "vpt_affine_norm_zp: null argument");
    VPT_CHECK(C % 8 == 0 && H > 0 && W > 0, "vpt_affine_norm_zp: need C %% 8 == 0");
    const long long items = (long long)(H + 1) * (W + 1) * (C / 8);
    const int bpg = vpt_norm_stat_parts((H + 1) * (W + 1), C);
    const bool fast = C / 8 <= 256;  // one channel vector per thread; wider rows fall back to the generic kernel
    for (long long g0 = 0; g0 < F; g0 += 65535) {
        const long long gn = (F - g0 < 65535) ? (F - g0) : 65535;
        dim3 grid(bpg, (unsigned)gn);
        if (fast)
            launch_k(affine_norm_zp_rows_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, 
                reinterpret_cast<const uint4*>(in) + g0 * items, reinterpret_cast<const float2*>(mr) + g0, gamma, beta,
                reinterpret_cast<uint4*>(out) + g0 * items, stat_part ? reinterpret_cast<float2*>(stat_part) + g0 * bpg : nullptr, H, W, C / 8);
        else
            launch_k(affine_norm_zp_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, 
                reinterpret_cast<const uint4*>(in) + g0 * items, reinterpret_cast<const float2*>(mr) + g0, gamma, beta,
                reinterpret_cast<uint4*>(out) + g0 * items, stat_part ? reinterpret_cast<float2*>(stat_part) + g0 * bpg : nullptr, H, W, C / 8);
        VPT_LAUNCH_CHECK();
    }
    return VPT_OK;
}

extern "C" int vpt_copy_rows2(const void* src, const void* src2, int32_t src_f32, int64_t src_bstride, int64_t src_ld, int64_t src_off, void* dst,
                              void* dst2, int32_t dst_f32, int64_t dst_bstride, int64_t dst_ld, int64_t dst_off, int32_t B, int32_t rows,
                              int32_t cols, void* stream);

extern "C" int vpt_copy_rows(const void* src, int32_t src_f32, int64_t src_bstride, int64_t src_ld, int64_t src_off, void* dst,
                             int32_t dst_f32, int64_t dst_bstride, int64_t dst_ld, int64_t dst_off, int32_t B, int32_t rows,
                             int32_t cols, void* stream) {
    return vpt_copy_rows2(src, nullptr, src_f32, src_bstride, src_ld, src_off, dst, nullptr, dst_f32, dst_bstride, dst_ld, dst_off, B, rows, cols, stream);
}

extern "C" int vpt_copy_rows2(const void* src, const void* src2, int32_t src_f32, int64_t src_bstride, int64_t src_ld, int64_t src_off, void* dst,
                              void* dst2, int32_t dst_f32, int64_t dst_bstride, int64_t dst_ld, int64_t dst_off, int32_t B, int32_t rows,
                              int32_t cols, void* stream) {
    using namespace vpt;
    if (rows == 0 || B == 0) return VPT_OK;
    VPT_CHECK(src && dst && B > 0 && rows > 0 && cols > 0 && (!src2 == !dst2), "vpt_copy_rows: bad arguments");
    VPT_CHECK(cols % 8 == 0 && src_ld % 8 == 0 && dst_ld % 8 == 0 && src_bstride % 8 == 0 && dst_bstride % 8 == 0,
              "vpt_copy_rows: cols / pitches must be multiples of 8");
    VPT_CHECK(B <= 65535, "vpt_copy_rows: B too large");
    dim3 grid(vpt_blocks_for((long long)rows * (cols / 8), 1024, 1024), B, src2 ? 2 : 1);
    cudaStream_t s = (cudaStream_t)stream;
#define VPT_CR(SF, DF)                                                                                                                        \
    launch_k(copy_rows_kernel<SF, DF>, dim3(grid), dim3(256), 0, s, src, src2, src_bstride, src_ld, src_off, dst, dst2, dst_bstride, dst_ld, dst_off, rows, \
                                                  cols / 8)
    if (src_f32 && dst_f32) VPT_CR(true, true);
    else if (src_f32) VPT_CR(true, false);
    else if (dst_f32) VPT_CR(false, true);
    else VPT_CR(false, false);
#undef VPT_CR
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_state_mask_update(const uint8_t* mask_in, const uint8_t* first, int64_t first_stride, uint8_t* mask_out,
                                     int32_t B, int32_t t, int32_t maxlen, void* stream) {
    using namespace vpt;
    if (maxlen == 0 || B == 0) return VPT_OK;
    VPT_CHECK(first && mask_out && B > 0 && t > 0 && maxlen > 0, "vpt_state_mask_update: bad arguments");
    const int n = B * maxlen;
    launch_k(state_mask_update_kernel, dim3((n + 255) / 256), dim3(256), 0, (cudaStream_t)stream, mask_in, first, first_stride, mask_out, B, t, maxlen);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}
