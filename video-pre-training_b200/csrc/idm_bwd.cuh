// Backward kernels that only the inverse dynamics model (IDM) step needs (video-pre-training_b200/training.py, IDMTrainer):
//
//   conv3d_t5_bwd   weight / bias gradient of the temporal pre-stage (csrc/conv3d.cuh).  The ReLU of the forward is NOT applied
//                   here: the caller passes the gradient wrt the conv3d output with the mask already applied (the norm backward
//                   of the first CNN conv in front of it runs with relu_x, which zeroes dx where the taped output is 0).
//                       dW[C][dt*3 + c] = sum_{f, pix} dy[f, pix, C] * img[f + dt - 2, pix, c]   (u8 values, taps outside [0, T)
//                       db[C]           = sum_{f, pix} dy[f, pix, C]                              of the frame's sequence skipped)
//                   Bandwidth bound (one pass over dy, 16 B per thread-pixel): a thread owns one 8-channel group and keeps its
//                   16 x 8 fp32 sums in registers; blocks write per-block partials, a second kernel sums them in a fixed order.
//                   TIN = float: fp32 frames on the uint8 scale (vpt_conv3d_t5_bwd_f32), read as floats like the u8 values.
//   conv3d_t5_dimg  image gradient of the temporal pre-stage, from the same dy (ReLU mask applied):
//                       dimg[b, s, pix, c] = sum_dt sum_C dy[b, s + 2 - dt, pix, C] * w[C][dt*3 + c]    (s + 2 - dt outside [0, T): 0)
//                   A thread owns one pixel's 8-channel group of one sequence and walks t once, keeping the five outputs s = t-2 .. t+2
//                   that dy[t] feeds in registers; s = t - 2 is complete after step t and is summed over the pixel's channel groups
//                   (lanes of one warp, xor shuffles) and written.  dy is read once, fixed-order sums, no atomics.
//   softmax_nll_bwd_grouped   factored categorical heads (IDM buttons = 20 x Discrete(2), camera = 2 x Discrete(11)): per row and
//                   group, the log-prob of the taken sub-action (summed over the groups of the row, for the loss) and
//                   (softmax - onehot) * scale into the group's columns of the logits gradient.
#pragma once
#include "common.cuh"
#include "backward.cuh"

namespace vpt {

constexpr int kC3bThreads = 256;

// grid = (blocks per frame, frame slabs); block (x, y) handles frames y, y + gridDim.y, ... and pixels blockIdx.x * ppb + lane, ...
template <typename TIN>
__global__ void __launch_bounds__(kC3bThreads) conv3d_t5_bwd_kernel(const TIN* __restrict__ img, const uint4* __restrict__ dy,
                                                                   float* __restrict__ part, long long F, int T, int H, int W, int C) {
    __shared__ float red[kC3bThreads / 32][256];  // per-warp sums of one tap k for every channel (C <= 256)
    const int C8 = C / 8, Wp = W + 1;
    const int npix = (H + 1) * Wp;
    const int cg = threadIdx.x % C8, pl = threadIdx.x / C8;  // channel group, pixel lane
    const int ppb = kC3bThreads / C8;
    const long long frame_px = (long long)H * W * 3;
    float acc[16][8];
#pragma unroll
    for (int k = 0; k < 16; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
    for (long long f = blockIdx.y; f < F; f += gridDim.y) {
        const int t = (int)(f % T);
        const TIN* fimg[5];
        bool tin[5];
#pragma unroll
        for (int dt = 0; dt < 5; ++dt) {
            const int tt = t + dt - 2;
            tin[dt] = tt >= 0 && tt < T;  // zero padding in time at both ends of the frame's own sequence
            fimg[dt] = img + (f + (tin[dt] ? dt - 2 : 0)) * frame_px;
        }
        const uint4* fdy = dy + f * (long long)npix * C8;
        for (int pix = blockIdx.x * ppb + pl; pix < npix; pix += gridDim.x * ppb) {
            const int y = pix / Wp, x = pix - y * Wp;
            if (y >= H || x >= W) continue;  // the ZP zero row / column
            float g[8];
            unpack8(__ldg(fdy + (long long)pix * C8 + cg), g);
            const int poff = (y * W + x) * 3;
#pragma unroll
            for (int dt = 0; dt < 5; ++dt) {
                if (!tin[dt]) continue;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float v = (float)__ldg(fimg[dt] + poff + c);
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[dt * 3 + c][j] = fmaf(g[j], v, acc[dt * 3 + c][j]);
                }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[15][j] += g[j];
        }
    }
    // fixed-order block reduction: lanes of the same channel group within a warp (xor shuffles), then the warps in order
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* out = part + ((long long)blockIdx.y * gridDim.x + blockIdx.x) * C * 16;
#pragma unroll  // compile-time k: acc stays in registers (a runtime index would move the 16 x 8 sums to local memory)
    for (int k = 0; k < 16; ++k) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float v = acc[k][j];
            for (int o = C8; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            acc[k][j] = v;
        }
        if (lane < C8) {  // C8 <= 32: lanes 0..C8-1 of every warp now hold the warp's sums of all C channels
#pragma unroll
            for (int j = 0; j < 8; ++j) red[warp][cg * 8 + j] = acc[k][j];
        }
        __syncthreads();
        for (int c = threadIdx.x; c < C; c += kC3bThreads) {
            float s = 0.f;
            for (int w = 0; w < kC3bThreads / 32; ++w) s += red[w][c];
            out[(long long)c * 16 + k] = s;
        }
        __syncthreads();
    }
}

// grid = (pixel blocks, B); block threads = (pixel, 8-channel group) with the C / 8 groups of a pixel in consecutive lanes
__global__ void __launch_bounds__(kC3bThreads) conv3d_t5_dimg_kernel(const uint4* __restrict__ dy, const float* __restrict__ w,
                                                                    float* __restrict__ dimg, int T, int H, int W, int C) {
    const int C8 = C / 8, ppb = kC3bThreads / C8;
    const int cg = threadIdx.x % C8;
    const int pix = blockIdx.x * ppb + threadIdx.x / C8;
    const bool live = pix < H * W;  // (a dead thread still joins the shuffles)
    const int y = live ? pix / W : 0, x = live ? pix % W : 0;
    float wr[8][15];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int k = 0; k < 15; ++k) wr[j][k] = __ldg(w + (cg * 8 + j) * 15 + k);
    const long long f0 = (long long)blockIdx.y * T;  // the sequence's first frame
    const long long npix = (long long)(H + 1) * (W + 1);
    const uint4* src = dy + (f0 * npix + (long long)y * (W + 1) + x) * C8 + cg;
    float* dst = dimg + (f0 * H * W + pix) * 3;
    float acc[5][3];  // acc[k]: output s = t - 2 + k
#pragma unroll
    for (int k = 0; k < 5; ++k) acc[k][0] = acc[k][1] = acc[k][2] = 0.f;
    uint4 nxt = live && T > 0 ? __ldg(src) : make_uint4(0, 0, 0, 0);
    for (int t = 0; t < T + 2; ++t) {
        float g[8];
        unpack8(nxt, g);
        if (t >= T) {
#pragma unroll
            for (int j = 0; j < 8; ++j) g[j] = 0.f;
        }
        if (live && t + 1 < T) nxt = __ldg(src + (long long)(t + 1) * npix * C8);
#pragma unroll
        for (int dt = 0; dt < 5; ++dt)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float a = acc[dt][c];
#pragma unroll
                for (int j = 0; j < 8; ++j) a = fmaf(g[j], wr[j][dt * 3 + c], a);
                acc[dt][c] = a;
            }
        // s = t - 2 has had all its taps: sum it over the pixel's channel groups
        float v[3] = {acc[0][0], acc[0][1], acc[0][2]};
#pragma unroll
        for (int c = 0; c < 3; ++c)
            for (int o = 1; o < C8; o <<= 1) v[c] += __shfl_xor_sync(0xffffffffu, v[c], o);
        if (live && cg == 0 && t >= 2) {
            float* o = dst + (long long)(t - 2) * H * W * 3;
            o[0] = v[0];
            o[1] = v[1];
            o[2] = v[2];
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[k][0] = acc[k + 1][0], acc[k][1] = acc[k + 1][1], acc[k][2] = acc[k + 1][2];
        acc[4][0] = acc[4][1] = acc[4][2] = 0.f;
    }
}

// dW [C][15], db [C] = fixed-order (double) sums of the per-block partials [S][C][16]
__global__ void __launch_bounds__(256) conv3d_t5_bwd_finalize_kernel(const float* __restrict__ part, float* __restrict__ dW, float* __restrict__ db,
                                                                       int S, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C * 16) return;
    double s = 0.0;
    for (int p = 0; p < S; ++p) s += (double)__ldg(part + (long long)p * C * 16 + i);
    const int c = i / 16, k = i % 16;
    if (k < 15) dW[c * 15 + k] = (float)s;
    else db[c] = (float)s;
}

// one thread per row: groups in order (the row's log-prob sum is formed in a fixed order)
__global__ void __launch_bounds__(256) softmax_nll_bwd_grouped_kernel(const float* __restrict__ logp, long long ld_logp, const long long* __restrict__ idx,
                                                                        int groups, int n, float scale, __nv_bfloat16* __restrict__ out,
                                                                        long long ld_out, int col0, float* __restrict__ lp, int accumulate,
                                                                        long long rows) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const float* lr = logp + r * ld_logp;
    __nv_bfloat16* orow = out + r * ld_out + col0;
    float s = 0.f;
    for (int gi = 0; gi < groups; ++gi) {
        const long long a = __ldg(idx + r * groups + gi);
        const float* lg = lr + gi * n;
        s += __ldg(lg + a);
        for (int j = 0; j < n; ++j) {
            float p = __expf(__ldg(lg + j));
            if (j == a) p -= 1.f;
            orow[gi * n + j] = __float2bfloat16_rn(p * scale);
        }
    }
    if (lp != nullptr) lp[r] = accumulate ? lp[r] + s : s;
}

static inline int conv3d_bwd_grid_x(int H, int W, int C) {
    long long b = ((long long)(H + 1) * (W + 1) * (C / 8) + 8 * kC3bThreads - 1) / (8 * kC3bThreads);  // >= 8 pixel passes per block
    if (b > 16) b = 16;
    if (b < 1) b = 1;
    return (int)b;
}
static inline int conv3d_bwd_grid_y(long long F) { return (int)(F < 128 ? F : 128); }

}  // namespace vpt

extern "C" int64_t vpt_conv3d_t5_bwd_workspace(int64_t F, int32_t H, int32_t W, int32_t C) {
    if (F <= 0 || H <= 0 || W <= 0 || C <= 0) return 0;
    return (int64_t)vpt::conv3d_bwd_grid_x(H, W, C) * vpt::conv3d_bwd_grid_y(F) * C * 16;
}

namespace vpt {

template <typename TIN>
static int conv3d_t5_bwd_launch(const char* fn, const TIN* img, const void* dy, float* dW, float* db, float* workspace, int32_t B, int32_t T, int32_t H,
                                int32_t W, int32_t C, void* stream) {
    VPT_CHECK(img && dy && dW && db && workspace && B > 0 && T > 0 && H > 0 && W > 0, "%s: bad arguments", fn);
    VPT_CHECK(C % 8 == 0 && C <= 256 && 256 % (C / 8) == 0, "%s: C=%d must be a multiple of 8, <= 256, with C/8 dividing 256", fn, C);
    VPT_CHECK((long long)(H + 1) * (W + 1) * (C / 8) < 2147483647LL, "%s: frame too large for 32-bit indexing", fn);
    const long long F = (long long)B * T;
    const int gx = conv3d_bwd_grid_x(H, W, C), gy = conv3d_bwd_grid_y(F);
    conv3d_t5_bwd_kernel<TIN><<<dim3(gx, gy), kC3bThreads, 0, (cudaStream_t)stream>>>(img, reinterpret_cast<const uint4*>(dy), workspace, F, T, H, W, C);
    VPT_LAUNCH_CHECK();
    conv3d_t5_bwd_finalize_kernel<<<(C * 16 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(workspace, dW, db, gx * gy, C);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

}  // namespace vpt

extern "C" int vpt_conv3d_t5_bwd(const uint8_t* img, const void* dy, float* dW, float* db, float* workspace, int32_t B, int32_t T, int32_t H, int32_t W,
                                 int32_t C, void* stream) {
    return vpt::conv3d_t5_bwd_launch("vpt_conv3d_t5_bwd", img, dy, dW, db, workspace, B, T, H, W, C, stream);
}

extern "C" int vpt_conv3d_t5_bwd_f32(const float* img, const void* dy, float* dW, float* db, float* workspace, int32_t B, int32_t T, int32_t H,
                                     int32_t W, int32_t C, void* stream) {
    return vpt::conv3d_t5_bwd_launch("vpt_conv3d_t5_bwd_f32", img, dy, dW, db, workspace, B, T, H, W, C, stream);
}

extern "C" int vpt_conv3d_t5_dimg(const void* dy, const float* w, float* dimg, int32_t B, int32_t T, int32_t H, int32_t W, int32_t C, void* stream) {
    using namespace vpt;
    VPT_CHECK(dy && w && dimg && B > 0 && B <= 65535 && T > 0 && H > 0 && W > 0, "vpt_conv3d_t5_dimg: bad arguments");
    VPT_CHECK(C % 8 == 0 && C >= 8 && C <= 256 && 32 % (C / 8) == 0, "vpt_conv3d_t5_dimg: C=%d must be 8 * a power of two, <= 256", C);
    VPT_CHECK((long long)(H + 1) * (W + 1) * (C / 8) < 2147483647LL, "vpt_conv3d_t5_dimg: frame too large for 32-bit indexing");
    const int ppb = kC3bThreads / (C / 8);
    conv3d_t5_dimg_kernel<<<dim3((unsigned)((H * W + ppb - 1) / ppb), (unsigned)B), kC3bThreads, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const uint4*>(dy), w, dimg, T, H, W, C);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_softmax_nll_bwd_grouped(const float* logp, int64_t ld_logp, const int64_t* idx, int32_t groups, int32_t n, float scale, void* out,
                                           int64_t ld_out, int32_t col0, float* lp, int32_t accumulate, int64_t rows, void* stream) {
    using namespace vpt;
    VPT_CHECK(logp && idx && out && rows > 0 && groups > 0 && n > 0 && col0 >= 0 && ld_logp >= (int64_t)groups * n &&
                  ld_out >= col0 + (int64_t)groups * n,
              "vpt_softmax_nll_bwd_grouped: bad arguments");
    softmax_nll_bwd_grouped_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        logp, ld_logp, reinterpret_cast<const long long*>(idx), groups, n, scale, reinterpret_cast<__nv_bfloat16*>(out), ld_out, col0, lp, accumulate,
        rows);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}
