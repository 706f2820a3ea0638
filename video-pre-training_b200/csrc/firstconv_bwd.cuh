// Weight / bias gradient of the fused stack-0 first convolution (csrc/firstconv.cuh: u8 -> conv3x3(3->C0)+bias -> ReLU ->
// max_pool 3/2/1).  The forward never materialises the 128x128xC0 pre-pool map, so the backward recomputes it:
//
//   thread = output channel (block = C0 threads); a block walks segments of 8 pooled pixels; the (5 x 19 x 3) u8 input
//   window of a segment is staged in shared memory as floats (double buffered, the next segment's window is fetched into
//   registers while this one is processed); per pooled pixel every thread pulls the 5x5x3 window into
//   registers, evaluates the convolution outputs of the pooling window in fp32 (6 new ones per pixel, the left column is the
//   previous pixel's right column), picks the first maximum (ReLU: only if it is > 0) and accumulates
//   dW[k] += g * patch_argmax[k],  db += g  in registers; there is no reduction across threads.  Per-block partials are summed
//   in a fixed order afterwards.  (Next step: the conv recompute and g^T * patch on mma.sync like the forward kernel.)
//   TIN = float: fp32 frames on the uint8 scale (vpt_firstconv_bwd_f32); every frame value is converted to float before use either way.
//
// Image gradient of the same layer (vpt_firstconv_dimg): d img[Y][X][c] = sum_C0 sum_(ky,kx) dpre[C0][Y-ky+1][X-kx+1] * w[C0][ky][kx][c],
// dpre = the pooled gradient routed to its window's maximum by firstconv_bwd's rule (the same fp32 FMA chain recomputes the conv, the
// first maximum in scan order takes it, only if it is > 0).  One CTA owns a 16x16 block of input pixels and every sum is in a fixed
// order: no partials, no atomics, bit-reproducible.  The block needs dpre on the 18x18 ring of conv positions around it, i.e. the
// pooled windows of a 10x10 pooled tile: 21x21 conv positions from a 23x23 input patch.  Per chunk of kFdCh channels: recompute the
// 21x21 conv map, route the 10x10 pooled gradients, gather dpre on the ring, contract with w (a thread per input pixel).
#pragma once
#include "common.cuh"

namespace vpt {

constexpr int kFbSeg = 8;                       // pooled pixels per segment
constexpr int kFbWinCols = 2 * kFbSeg + 3;      // input columns a segment touches
constexpr int kFbWinFloats = 5 * kFbWinCols * 3;

template <typename TIN, int kMaxThreads, int kMinBlocks>
__global__ void __launch_bounds__(kMaxThreads, kMinBlocks) firstconv_bwd_kernel(const TIN* __restrict__ img, const float* __restrict__ w, const float* __restrict__ bias,
                                                                const __nv_bfloat16* __restrict__ dy, float* __restrict__ ws, int F, int H, int W, int C0) {
    __shared__ float win[2][kFbWinFloats];  // double buffered: the next segment's window is fetched while this one is processed
    const int c = threadIdx.x;  // blockDim.x == C0
    const int Ho = H >> 1, Wo = W >> 1;
    const int segs_per_row = Wo / kFbSeg;
    const long long items = (long long)F * Ho * segs_per_row;
    float wr[27], dW[27];
#pragma unroll
    for (int k = 0; k < 27; ++k) {
        wr[k] = __ldg(w + c * 27 + k);
        dW[k] = 0.f;
    }
    const float bc = __ldg(bias + c);
    float db = 0.f;
    // element e of a segment's (5 x 19 x 3) window, as a float; zero outside the image (the conv's padding)
    auto fetch = [&](long long it, int e) -> float {
        const int seg = (int)(it % segs_per_row);
        const int oy = (int)((it / segs_per_row) % Ho);
        const long long f = it / ((long long)segs_per_row * Ho);
        const int ch = e % 3, col = (e / 3) % kFbWinCols, r = e / (3 * kFbWinCols);
        const int y = 2 * oy - 2 + r, x = 2 * seg * kFbSeg - 2 + col;
        return (y >= 0 && y < H && x >= 0 && x < W) ? (float)__ldg(img + ((f * H + y) * (long long)W + x) * 3 + ch) : 0.f;
    };
    constexpr int kPre = (kFbWinFloats + 63) / 64;  // window elements per thread for the smallest block (64 threads)
    float pre[kPre];
    const int npre = (kFbWinFloats + blockDim.x - 1) / blockDim.x;
    if ((long long)blockIdx.x < items) {
#pragma unroll
        for (int q = 0; q < kPre; ++q) {
            const int e = threadIdx.x + q * blockDim.x;
            pre[q] = (q < npre && e < kFbWinFloats) ? fetch(blockIdx.x, e) : 0.f;
        }
    }
    int buf = 0;
    for (long long it = blockIdx.x; it < items; it += gridDim.x, buf ^= 1) {
        const int seg = (int)(it % segs_per_row);
        const int oy = (int)((it / segs_per_row) % Ho);
        const long long f = it / ((long long)segs_per_row * Ho);
        const int ox0 = seg * kFbSeg;
        float* win_c = win[buf];
#pragma unroll
        for (int q = 0; q < kPre; ++q) {
            const int e = threadIdx.x + q * blockDim.x;
            if (q < npre && e < kFbWinFloats) win_c[e] = pre[q];
        }
        __syncthreads();  // (the other buffer was last read two iterations ago, behind the previous barrier)
        if (it + gridDim.x < items) {
#pragma unroll
            for (int q = 0; q < kPre; ++q) {
                const int e = threadIdx.x + q * blockDim.x;
                pre[q] = (q < npre && e < kFbWinFloats) ? fetch(it + gridDim.x, e) : 0.f;
            }
        }
        const __nv_bfloat16* gy = dy + ((f * (Ho + 1) + oy) * (long long)(Wo + 1) + ox0) * C0 + c;
        float prev[3] = {0.f, 0.f, 0.f};  // conv outputs of the previous pixel's right column == this pixel's left column
#pragma unroll 1
        for (int p = 0; p < kFbSeg; ++p) {
            const float g = __bfloat162float(gy[(long long)p * C0]);
            // 5 x 5 x 3 window of this pooled pixel -> registers
            float v[75];
#pragma unroll
            for (int r = 0; r < 5; ++r)
#pragma unroll
                for (int q = 0; q < 15; ++q) v[r * 15 + q] = win_c[(r * kFbWinCols + 2 * p) * 3 + q];
            // the 9 convolution outputs of the pooling window (column 0 is carried over from the previous pixel)
            float cv[9];
#pragma unroll
            for (int py = 0; py < 3; ++py) {
#pragma unroll
                for (int px = 0; px < 3; ++px) {
                    if (px == 0 && p > 0) {
                        cv[py * 3] = prev[py];
                        continue;
                    }
                    float a = bc;
#pragma unroll
                    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                        for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                            for (int ch = 0; ch < 3; ++ch) a = fmaf(wr[(ky * 3 + kx) * 3 + ch], v[(py + ky) * 15 + (px + kx) * 3 + ch], a);
                    cv[py * 3 + px] = a;
                }
            }
#pragma unroll
            for (int py = 0; py < 3; ++py) prev[py] = cv[py * 3 + 2];
            // first maximum over the positions inside the image (max_pool2d pads with -inf); ReLU: only a positive maximum counts
            float best = -INFINITY;
            int ay = 0, ax = 0;
#pragma unroll
            for (int py = 0; py < 3; ++py) {
#pragma unroll
                for (int px = 0; px < 3; ++px) {
                    const int yy = 2 * oy - 1 + py, xx = 2 * (ox0 + p) - 1 + px;
                    const bool inside = yy >= 0 && yy < H && xx >= 0 && xx < W;
                    if (inside && cv[py * 3 + px] > best) {
                        best = cv[py * 3 + px];
                        ay = py;
                        ax = px;
                    }
                }
            }
            const float ge = best > 0.f ? g : 0.f;
            db += ge;
            // dW += ge * patch(ay, ax), the patch re-read from the staged window at a per-thread offset: the 9 possible offsets
            // (ay*19 + ax)*3 words fall into 9 different banks, so the divergent addresses of a warp do not conflict
            const float* pw = win_c + ((ay * kFbWinCols) + 2 * p + ax) * 3;
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int q = 0; q < 9; ++q) dW[ky * 9 + q] = fmaf(ge, pw[ky * kFbWinCols * 3 + q], dW[ky * 9 + q]);
        }
    }
    float* o = ws + ((long long)blockIdx.x * C0 + c) * 28;
#pragma unroll
    for (int k = 0; k < 27; ++k) o[k] = dW[k];
    o[27] = db;
}

__global__ void firstconv_bwd_finalize_kernel(const float* __restrict__ ws, float* __restrict__ dW, float* __restrict__ db, int S, int C0) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over C0 * 28
    if (i >= C0 * 28) return;
    double a = 0.0;
    for (int s = 0; s < S; ++s) a += (double)__ldg(ws + (long long)s * C0 * 28 + i);
    const int c = i / 28, k = i % 28;
    if (k < 27) dW[c * 27 + k] = (float)a;
    else db[c] = (float)a;
}

constexpr int kFdThreads = 256;  // one per input pixel of the 16x16 block
constexpr int kFdCh = 8;         // channels per pass
constexpr int kFdIn = 23, kFdConv = 21, kFdPool = 10, kFdRing = 18;
static_assert(kFdConv % 3 == 0 && kFdThreads % kFdCh == 0, "firstconv_dimg: rows of three positions, one channel per thread");

template <typename TIN>
__global__ void __launch_bounds__(kFdThreads) firstconv_dimg_kernel(const TIN* __restrict__ img, const float* __restrict__ w,
                                                                     const float* __restrict__ bias, const __nv_bfloat16* __restrict__ dy,
                                                                     float* __restrict__ dimg, int H, int W, int C0) {
    extern __shared__ float fd_smem[];
    float* patch = fd_smem;                                   // [23][23][3] frame values, 0 outside the image
    float* ws = patch + kFdIn * kFdIn * 3 + 3;                // [C0][28]: w (ky,kx,c) then bias
    float* conv = ws + C0 * 28;                               // [kFdCh][21*21] pre-pool map
    float* gsel = conv + kFdCh * kFdConv * kFdConv;           // [100][kFdCh] routed pooled gradient (0: none)
    int* asel = reinterpret_cast<int*>(gsel + kFdPool * kFdPool * kFdCh);  // [100][kFdCh] window position (dy*3+dx) it went to
    float* dpre = reinterpret_cast<float*>(asel + kFdPool * kFdPool * kFdCh);  // [kFdCh][18*18]
    const int tx = W / 16, tiles = tx * (H / 16);
    const long long f = blockIdx.x / tiles;
    const int tile = (int)(blockIdx.x % tiles);
    const int Y0 = (tile / tx) * 16, X0 = (tile % tx) * 16;
    const int Ho = H / 2, Wo = W / 2;
    const TIN* fimg = img + f * (long long)H * W * 3;
    for (int i = threadIdx.x; i < kFdIn * kFdIn * 3; i += kFdThreads) {
        const int r = i / (kFdIn * 3), q = i % (kFdIn * 3);
        const int Y = Y0 - 4 + r, xb = (X0 - 4) * 3 + q;
        patch[i] = (Y >= 0 && Y < H && xb >= 0 && xb < W * 3) ? (float)__ldg(fimg + (long long)Y * W * 3 + xb) : 0.f;
    }
    for (int i = threadIdx.x; i < C0 * 28; i += kFdThreads) {
        const int c = i / 28, k = i % 28;
        ws[i] = k < 27 ? __ldg(w + c * 27 + k) : __ldg(bias + c);
    }
    const int iy = threadIdx.x / 16, ix = threadIdx.x % 16;  // this thread's input pixel
    float acc[3] = {0.f, 0.f, 0.f};
    const int py0 = Y0 / 2 - 1, px0 = X0 / 2 - 1;  // pooled tile origin
    for (int c0 = 0; c0 < C0; c0 += kFdCh) {
        __syncthreads();  // (first pass: patch / weights staged; later: the previous pass's contraction is done with dpre)
        // (1) the 21x21 pre-pool map, conv position (Y0-3+r, X0-3+q), in firstconv_bwd's FMA order.  A thread keeps one channel's
        // weights in registers for the whole pass (its channel is threadIdx.x % kFdCh for every item) and computes three neighbouring
        // positions of a row at once, so that they share the patch loads (15 per kernel row for 27 FMAs).
        {
            const int cl = threadIdx.x % kFdCh;
            float wr[28];
#pragma unroll
            for (int k = 0; k < 28; ++k) wr[k] = ws[(c0 + cl) * 28 + k];
            for (int it = threadIdx.x / kFdCh; it < kFdConv * (kFdConv / 3); it += kFdThreads / kFdCh) {
                const int r = it / (kFdConv / 3), q = (it % (kFdConv / 3)) * 3;
                float a0 = wr[27], a1 = wr[27], a2 = wr[27];
#pragma unroll
                for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                        for (int ch = 0; ch < 3; ++ch) {
                            const float wv = wr[(ky * 3 + kx) * 3 + ch];
                            const float* pp = patch + ((r + ky) * kFdIn + q + kx) * 3 + ch;
                            a0 = fmaf(wv, pp[0], a0);
                            a1 = fmaf(wv, pp[3], a1);
                            a2 = fmaf(wv, pp[6], a2);
                        }
                float* o = conv + cl * kFdConv * kFdConv + r * kFdConv + q;
                o[0] = a0;
                o[1] = a1;
                o[2] = a2;
            }
        }
        __syncthreads();
        // (2) route each pooled gradient of the 10x10 tile: the first maximum over the window's positions inside the image, if > 0
        for (int i = threadIdx.x; i < kFdPool * kFdPool * kFdCh; i += kFdThreads) {
            const int cl = i % kFdCh, pp = i / kFdCh;
            const int pr = pp / kFdPool, pc = pp % kFdPool;
            const int py = py0 + pr, px = px0 + pc;
            float g = 0.f;
            int at = -1;
            if (py >= 0 && py < Ho && px >= 0 && px < Wo) {
                float best = -INFINITY;
#pragma unroll
                for (int a = 0; a < 3; ++a)
#pragma unroll
                    for (int b = 0; b < 3; ++b) {
                        const int yy = 2 * py - 1 + a, xx = 2 * px - 1 + b;
                        const float v = conv[cl * kFdConv * kFdConv + (2 * pr + a) * kFdConv + 2 * pc + b];
                        if (yy >= 0 && yy < H && xx >= 0 && xx < W && v > best) {
                            best = v;
                            at = a * 3 + b;
                        }
                    }
                if (best > 0.f) g = __bfloat162float(dy[((f * (Ho + 1) + py) * (long long)(Wo + 1) + px) * C0 + c0 + cl]);
                else at = -1;
            }
            gsel[i] = g;
            asel[i] = at;
        }
        __syncthreads();
        // (3) dpre on the 18x18 ring (conv position (Y0-1+r, X0-1+q) = map position (r+2, q+2)): the windows that routed to it, in order
        for (int i = threadIdx.x; i < kFdCh * kFdRing * kFdRing; i += kFdThreads) {
            const int cl = i / (kFdRing * kFdRing), p = i % (kFdRing * kFdRing);
            const int cr = p / kFdRing + 2, cc = p % kFdRing + 2;
            float d = 0.f;
            for (int pr = (cr - 1) / 2; pr <= cr / 2; ++pr)
                for (int pc = (cc - 1) / 2; pc <= cc / 2; ++pc) {
                    const int j = (pr * kFdPool + pc) * kFdCh + cl;
                    if (asel[j] == (cr - 2 * pr) * 3 + (cc - 2 * pc)) d += gsel[j];
                }
            dpre[i] = d;
        }
        __syncthreads();
        // (4) d img of this thread's pixel += sum over the chunk's channels and the 3x3 taps
        for (int cl = 0; cl < kFdCh; ++cl) {
            const float* wc = ws + (c0 + cl) * 28;
            const float* dp = dpre + cl * kFdRing * kFdRing;
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float d = dp[(iy - ky + 2) * kFdRing + ix - kx + 2];
#pragma unroll
                    for (int ch = 0; ch < 3; ++ch) acc[ch] = fmaf(d, wc[(ky * 3 + kx) * 3 + ch], acc[ch]);
                }
        }
    }
    float* o = dimg + ((f * H + Y0 + iy) * (long long)W + X0 + ix) * 3;
    o[0] = acc[0];
    o[1] = acc[1];
    o[2] = acc[2];
}

static inline size_t firstconv_dimg_smem(int C0) {
    return sizeof(float) * ((size_t)kFdIn * kFdIn * 3 + 3 + (size_t)C0 * 28 + kFdCh * kFdConv * kFdConv + 2 * kFdPool * kFdPool * kFdCh +
                            kFdCh * kFdRing * kFdRing);
}

static inline int firstconv_bwd_blocks(long long F, int H, int W) {
    const long long items = F * (H / 2) * ((W / 2) / kFbSeg);
    long long s = 2LL * num_sms();
    if (s > items) s = items;
    if (s < 1) s = 1;
    return (int)s;
}

}  // namespace vpt

extern "C" int vpt_firstconv_bwd_parts(int64_t F, int32_t H, int32_t W) { return vpt::firstconv_bwd_blocks(F, H, W); }

namespace vpt {

template <typename TIN>
static int firstconv_bwd_launch(const char* fn, const TIN* img, const float* w, const float* bias, const void* dy, float* dW, float* db, float* workspace,
                                int64_t F, int32_t H, int32_t W, int32_t C0, void* stream) {
    VPT_CHECK(img && w && bias && dy && dW && db && workspace && F > 0, "%s: null argument", fn);
    VPT_CHECK(H % 2 == 0 && W % (2 * kFbSeg) == 0 && C0 % 32 == 0 && C0 >= 64 && C0 <= 256,
              "%s: need even H, W %% 16 == 0 and C0 in {64..256} a multiple of 32 (H=%d W=%d C0=%d)", fn, H, W, C0);
    const int S = firstconv_bwd_blocks(F, H, W);
    if (C0 <= 192)  // <= 170 registers per thread: two blocks per SM hide each other's barrier and window fetch
        firstconv_bwd_kernel<TIN, 192, 2><<<S, C0, 0, (cudaStream_t)stream>>>(img, w, bias, reinterpret_cast<const __nv_bfloat16*>(dy), workspace, (int)F, H, W, C0);
    else
        firstconv_bwd_kernel<TIN, 256, 1><<<S, C0, 0, (cudaStream_t)stream>>>(img, w, bias, reinterpret_cast<const __nv_bfloat16*>(dy), workspace, (int)F, H, W, C0);
    VPT_LAUNCH_CHECK();
    firstconv_bwd_finalize_kernel<<<(C0 * 28 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(workspace, dW, db, S, C0);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

template <typename TIN>
static int firstconv_dimg_launch(const TIN* img, const float* w, const float* bias, const void* dy, float* dimg, int64_t F, int32_t H, int32_t W,
                                 int32_t C0, void* stream) {
    const long long blocks = (long long)F * (H / 16) * (W / 16);
    VPT_CHECK(blocks < 2147483647LL, "vpt_firstconv_dimg: too many tiles");
    const size_t smem = firstconv_dimg_smem(C0);
    static size_t attr = 0;
    if (smem > attr) {
        VPT_CUDA(cudaFuncSetAttribute(firstconv_dimg_kernel<TIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    firstconv_dimg_kernel<TIN><<<(unsigned)blocks, kFdThreads, smem, (cudaStream_t)stream>>>(img, w, bias, reinterpret_cast<const __nv_bfloat16*>(dy),
                                                                                             dimg, H, W, C0);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

}  // namespace vpt

extern "C" int vpt_firstconv_bwd(const uint8_t* img, const float* w, const float* bias, const void* dy, float* dW, float* db, float* workspace, int64_t F,
                                 int32_t H, int32_t W, int32_t C0, void* stream) {
    return vpt::firstconv_bwd_launch("vpt_firstconv_bwd", img, w, bias, dy, dW, db, workspace, F, H, W, C0, stream);
}

extern "C" int vpt_firstconv_bwd_f32(const float* img, const float* w, const float* bias, const void* dy, float* dW, float* db, float* workspace,
                                     int64_t F, int32_t H, int32_t W, int32_t C0, void* stream) {
    return vpt::firstconv_bwd_launch("vpt_firstconv_bwd_f32", img, w, bias, dy, dW, db, workspace, F, H, W, C0, stream);
}

extern "C" int vpt_firstconv_dimg(const void* img, int32_t img_f32, const float* w, const float* bias, const void* dy, float* dimg, int64_t F,
                                  int32_t H, int32_t W, int32_t C0, void* stream) {
    using namespace vpt;
    VPT_CHECK(img && w && bias && dy && dimg && F > 0, "vpt_firstconv_dimg: null argument");
    VPT_CHECK(H % 16 == 0 && W % 16 == 0 && H >= 16 && W >= 16, "vpt_firstconv_dimg: H, W must be multiples of 16 (H=%d W=%d)", H, W);
    VPT_CHECK(C0 % kFdCh == 0 && C0 >= 8 && C0 <= 256, "vpt_firstconv_dimg: C0=%d must be a multiple of %d, <= 256", C0, kFdCh);
    return img_f32 ? firstconv_dimg_launch(static_cast<const float*>(img), w, bias, dy, dimg, F, H, W, C0, stream)
                   : firstconv_dimg_launch(static_cast<const uint8_t*>(img), w, bias, dy, dimg, F, H, W, C0, stream);
}
