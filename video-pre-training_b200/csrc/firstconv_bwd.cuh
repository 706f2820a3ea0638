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
#pragma once
#include "common.cuh"

namespace vpt {

constexpr int kFbSeg = 8;                       // pooled pixels per segment
constexpr int kFbWinCols = 2 * kFbSeg + 3;      // input columns a segment touches
constexpr int kFbWinFloats = 5 * kFbWinCols * 3;

template <int kMaxThreads, int kMinBlocks>
__global__ void __launch_bounds__(kMaxThreads, kMinBlocks) firstconv_bwd_kernel(const uint8_t* __restrict__ img, const float* __restrict__ w, const float* __restrict__ bias,
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

static inline int firstconv_bwd_blocks(long long F, int H, int W) {
    const long long items = F * (H / 2) * ((W / 2) / kFbSeg);
    long long s = 2LL * num_sms();
    if (s > items) s = items;
    if (s < 1) s = 1;
    return (int)s;
}

}  // namespace vpt

extern "C" int vpt_firstconv_bwd_parts(int64_t F, int32_t H, int32_t W) { return vpt::firstconv_bwd_blocks(F, H, W); }

extern "C" int vpt_firstconv_bwd(const uint8_t* img, const float* w, const float* bias, const void* dy, float* dW, float* db, float* workspace, int64_t F,
                                 int32_t H, int32_t W, int32_t C0, void* stream) {
    using namespace vpt;
    VPT_CHECK(img && w && bias && dy && dW && db && workspace && F > 0, "vpt_firstconv_bwd: null argument");
    VPT_CHECK(H % 2 == 0 && W % (2 * kFbSeg) == 0 && C0 % 32 == 0 && C0 >= 64 && C0 <= 256,
              "vpt_firstconv_bwd: need even H, W %% 16 == 0 and C0 in {64..256} a multiple of 32 (H=%d W=%d C0=%d)", H, W, C0);
    const int S = firstconv_bwd_blocks(F, H, W);
    if (C0 <= 192)  // <= 170 registers per thread: two blocks per SM hide each other's barrier and window fetch
        firstconv_bwd_kernel<192, 2><<<S, C0, 0, (cudaStream_t)stream>>>(img, w, bias, reinterpret_cast<const __nv_bfloat16*>(dy), workspace, (int)F, H, W, C0);
    else
        firstconv_bwd_kernel<256, 1><<<S, C0, 0, (cudaStream_t)stream>>>(img, w, bias, reinterpret_cast<const __nv_bfloat16*>(dy), workspace, (int)F, H, W, C0);
    VPT_LAUNCH_CHECK();
    firstconv_bwd_finalize_kernel<<<(C0 * 28 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(workspace, dW, db, S, C0);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}
