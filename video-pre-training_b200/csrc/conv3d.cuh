// IDM temporal pre-stage (lib/policy.py:394-403): Conv3d(3 -> C, kernel (5,1,1), pad (2,0,0)) + bias + ReLU applied per
// sample over its T frames (zero padded in time at both ends of the chunk, like the reference's per-sample loop), fused
// with the u8 -> /255 preprocessing.  K = 15 MACs per output: the stage is bounded by its bf16 output write
// (C*H*W*2 B per frame), so it is a plain streaming kernel: one thread = one pixel x 8 channels (16-byte store),
// output in the ZP layout + per-frame statistics partials for the GroupNorm of the following conv.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "elementwise.cuh"

namespace vpt {

// Round 2: the first version was instruction bound at 13x its HBM bound (8.4 ms per 512 frames, 135 ms of the 564 ms IDM step): three 64-bit
// divisions per item to decode a flat index, 30 shared-memory weight loads per item, 64 short blocks per frame that each re-gathered the
// weights.  Now a thread owns ONE 8-channel group for the whole block (its 15 x 8 weights live in registers), walks pixels with a
// 32-bit index and one 32-bit division, and a frame is 8 long blocks.
// TIN = float: fp32 frames on the uint8 scale (vpt_conv3d_t5_f32); each value is read as a float, so integer-valued frames give the
// uint8 path's results bit for bit.
template <typename TIN>
__global__ void __launch_bounds__(256, 1) conv3d_t5_kernel(const TIN* __restrict__ img, const float* __restrict__ w, const float* __restrict__ bias,
                                                             uint4* __restrict__ out, float2* __restrict__ stat_part, int T, int H, int W, int C, int out_f32) {
    extern __shared__ float c3_smem[];  // [15][C] weights (k-major so that 8 consecutive channels are contiguous) + [C] bias
    float* ws = c3_smem;
    float* bs = c3_smem + 15 * C;
    for (int i = threadIdx.x; i < 15 * C; i += blockDim.x) {
        const int k = i / C, c = i % C;
        ws[i] = __ldg(w + c * 15 + k);
    }
    for (int i = threadIdx.x; i < C; i += blockDim.x) bs[i] = __ldg(bias + i);
    __syncthreads();
    const long long f = blockIdx.y;          // frame index b*T + t
    const int t = (int)(f % T);
    const int C8 = C / 8, Wp = W + 1;
    const int npix = (H + 1) * Wp;
    const int cg = threadIdx.x % C8, c0 = cg * 8;   // this thread's channel group (256 % C8 == 0, host check)
    const int ppb = blockDim.x / C8;                // pixels per block pass
    float wr[15][8], br[8];
#pragma unroll
    for (int k = 0; k < 15; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j) wr[k][j] = ws[k * C + c0 + j];
#pragma unroll
    for (int j = 0; j < 8; ++j) br[j] = bs[c0 + j];
    // the five frames of the temporal window; outside the sequence (zero padding in time) the pointer stays on this frame and the weight of
    // the tap is zeroed, so that all 15 byte loads of a pixel are unconditional and in flight together (with a branch per tap they were five
    // dependent L2 round trips per pixel at 8 warps per SM: 6.6 ms per 512 frames)
    const TIN* fimg[5];
#pragma unroll
    for (int dt = 0; dt < 5; ++dt) {
        const int tt = t + dt - 2;
        const bool in = tt >= 0 && tt < T;
        fimg[dt] = img + (f + (in ? dt - 2 : 0)) * (long long)H * W * 3;
        if (!in) {
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int j = 0; j < 8; ++j) wr[dt * 3 + c][j] = 0.f;
        }
    }
    uint4* fout = out + f * (long long)npix * C8 * (out_f32 ? 2 : 1);  // fp32 output (precision mode): two uint4 per 8 channels
    float s = 0.f, ss = 0.f;
    const int pstep = gridDim.x * ppb;
    using LT = typename std::conditional<std::is_same<TIN, float>::value, float, uint32_t>::type;  // a loaded frame value
    auto load_px = [&](int pix, LT (&v)[15]) {  // the 15 input bytes of a pixel (zeros for the zero row / column and past the frame)
        const int y = pix / Wp, x = pix - y * Wp;
        const bool ok = pix < npix && y < H && x < W;
        const int poff = ok ? (y * W + x) * 3 : 0;
#pragma unroll
        for (int dt = 0; dt < 5; ++dt)
#pragma unroll
            for (int c = 0; c < 3; ++c) v[dt * 3 + c] = ok ? (LT)__ldg(fimg[dt] + poff + c) : (LT)0;
    };
    LT vn[15];
    int pix = blockIdx.x * ppb + threadIdx.x / C8;
    load_px(pix, vn);
    for (; pix < npix; pix += pstep) {
        LT v[15];
#pragma unroll
        for (int k = 0; k < 15; ++k) v[k] = vn[k];
        load_px(pix + pstep, vn);  // next pixel of this thread: in flight during the arithmetic below
        const int y = pix / Wp, x = pix - y * Wp;
        const int i = pix * C8 + cg;
        if (y >= H || x >= W) {
            if (out_f32) fout[2 * i] = fout[2 * i + 1] = make_uint4(0, 0, 0, 0);
            else fout[i] = make_uint4(0, 0, 0, 0);
            continue;
        }
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = br[j];
#pragma unroll
        for (int k = 0; k < 15; ++k) {
            const float vf = (float)v[k];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaf(vf, wr[k][j], acc[j]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaxf(acc[j], 0.f);
        if (out_f32) {
            fout[2 * i] = make_uint4(__float_as_uint(acc[0]), __float_as_uint(acc[1]), __float_as_uint(acc[2]), __float_as_uint(acc[3]));
            fout[2 * i + 1] = make_uint4(__float_as_uint(acc[4]), __float_as_uint(acc[5]), __float_as_uint(acc[6]), __float_as_uint(acc[7]));
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                s += acc[j];
                ss = fmaf(acc[j], acc[j], ss);
            }
            continue;
        }
        uint4 o;
        o.x = pack_bf16(acc[0], acc[1]); o.y = pack_bf16(acc[2], acc[3]); o.z = pack_bf16(acc[4], acc[5]); o.w = pack_bf16(acc[6], acc[7]);
        fout[i] = o;
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
        if (threadIdx.x == 0) stat_part[f * gridDim.x + blockIdx.x] = r;
    }
}

}  // namespace vpt

extern "C" int vpt_conv3d_stat_parts(int32_t H, int32_t W, int32_t C) { return vpt_blocks_for((long long)(H + 1) * (W + 1) * (C / 8), 32768, 8); }

namespace vpt {

template <typename TIN>
static int conv3d_t5_launch(const char* fn, const TIN* img, const float* w, const float* bias, void* out, float* stat_part, int32_t B, int32_t T,
                            int32_t H, int32_t W, int32_t C, int32_t out_f32, void* stream) {
    VPT_CHECK(img && w && bias && out && B > 0 && T > 0, "%s: null argument", fn);
    VPT_CHECK(C % 8 == 0 && C <= 512 && 256 % (C / 8) == 0, "%s: C=%d must be a multiple of 8, <= 512, with C/8 dividing 256", fn, C);
    VPT_CHECK((long long)(H + 1) * (W + 1) * (C / 8) * 2 < 2147483647LL, "%s: frame too large for 32-bit indexing", fn);
    const long long F = (long long)B * T;
    const int bpf = vpt_conv3d_stat_parts(H, W, C);
    const size_t smem = (size_t)16 * C * sizeof(float);
    for (long long f0 = 0; f0 < F; f0 += 65535 / T * T) {  // grid.y limit; slabs hold whole sequences
        long long fn_ = F - f0;
        if (fn_ > 65535 / T * T) fn_ = 65535 / T * T;
        dim3 grid(bpf, (unsigned)fn_);
        conv3d_t5_kernel<TIN><<<grid, 256, smem, (cudaStream_t)stream>>>(
            img + f0 * H * W * 3, w, bias, reinterpret_cast<uint4*>(out) + f0 * (long long)(H + 1) * (W + 1) * (C / 8) * (out_f32 ? 2 : 1),
            stat_part ? reinterpret_cast<float2*>(stat_part) + f0 * bpf : nullptr, T, H, W, C, out_f32 ? 1 : 0);
        VPT_LAUNCH_CHECK();
    }
    return VPT_OK;
}

}  // namespace vpt

extern "C" int vpt_conv3d_t5(const uint8_t* img, const float* w, const float* bias, void* out, float* stat_part, int32_t B, int32_t T,
                             int32_t H, int32_t W, int32_t C, int32_t out_f32, void* stream) {
    return vpt::conv3d_t5_launch("vpt_conv3d_t5", img, w, bias, out, stat_part, B, T, H, W, C, out_f32, stream);
}

extern "C" int vpt_conv3d_t5_f32(const float* img, const float* w, const float* bias, void* out, float* stat_part, int32_t B, int32_t T,
                                 int32_t H, int32_t W, int32_t C, int32_t out_f32, void* stream) {
    return vpt::conv3d_t5_launch("vpt_conv3d_t5_f32", img, w, bias, out, stat_part, B, T, H, W, C, out_f32, stream);
}
