// Training-time image augmentation (agent.py `augment_frames`): per frame an inverse affine warp with bilinear sampling and zero fill,
// then brightness, contrast, saturation and hue jitter with torchvision's `adjust_*` formulas, in one pass over HBM.
//
//   src u8 [F][H][W][3] -> dst u8 or fp32 (on the uint8 scale) [F][H][W][3];  params fp32 [F][10] = (A 2x3 row-major, b, c, s, h)
//
//   1. (u, v) = A . (x, y, 1) for the output pixel (x, y) (pixel centres at integer coordinates), computed in fp64 from the fp32 matrix,
//      so that the bilinear weights fx = u - floor(u), fy = v - floor(v) are exact up to their fp32 rounding.  Neighbours outside the
//      frame read 0.  p = top + fy (bot - top), top = p00 + fx (p01 - p00), bot = p10 + fx (p11 - p10), in fp32: an integer source point
//      reproduces the source byte.
//   2. b != 1: p = clamp(b p, 0, 255)
//   3. c != 1: p = clamp(c p + (1 - c) m, 0, 255), m = the frame mean of grey = 0.299 R + 0.587 G + 0.114 B of the step-2 result
//   4. s != 1: p = clamp(s p + (1 - s) g, 0, 255), g = the pixel's own grey
//   5. h != 0: RGB -> HSV on [0, 1] (torchvision's _rgb2hsv), H = (H + h) mod 1, back (_hsv2rgb), times 255, clamped
//   6. u8: round to nearest even; fp32: the clamped value.
//
// One CTA per frame.  The source frame is staged in shared memory by cp.async (48 KiB at 128 x 128; the dynamic shared-memory opt-in
// bounds the frame size, larger frames are refused).  With contrast, a first pass over the output pixels sums grey (fp32 per pixel, fp64
// sums) in a fixed order -- per-thread strided sums, a shuffle tree per warp, warps in index order -- and the second pass recomputes the
// warp and writes.  No atomics: a frame's output depends on its bytes and parameters alone, bit for bit.
#pragma once
#include "common.cuh"
#include "attention.cuh"  // cp_async16 / cp_async_wait_all

namespace vpt {

constexpr int kAugThreads = 256;

__device__ __forceinline__ float aug_clamp255(float v) { return fminf(fmaxf(v, 0.f), 255.f); }
__device__ __forceinline__ float aug_grey(float r, float g, float b) { return 0.299f * r + 0.587f * g + 0.114f * b; }

// steps 1 and 2 for output pixel (x, y): bilinear sample of the staged frame at A . (x, y, 1), zero outside, then brightness
__device__ __forceinline__ void aug_sample(const uint8_t* fr, int H, int W, const float* A, float bright, int x, int y, float (&p)[3]) {
    double u = fma((double)A[0], (double)x, fma((double)A[1], (double)y, (double)A[2]));
    double v = fma((double)A[3], (double)x, fma((double)A[4], (double)y, (double)A[5]));
    // beyond [-2, W + 1] every neighbour is outside either way; clamping keeps floor() in int range
    u = fmin(fmax(u, -2.0), (double)W + 1.0);
    v = fmin(fmax(v, -2.0), (double)H + 1.0);
    const double u0 = floor(u), v0 = floor(v);
    const float fx = (float)(u - u0), fy = (float)(v - v0);
    const int x0 = (int)u0, y0 = (int)v0;
    const bool ix0 = x0 >= 0 && x0 < W, ix1 = x0 + 1 >= 0 && x0 + 1 < W;
    const bool iy0 = y0 >= 0 && y0 < H, iy1 = y0 + 1 >= 0 && y0 + 1 < H;
    // every read stays inside the frame (clamped addresses); the masks above zero the outside neighbours
    const int xa = min(max(x0, 0), W - 1) * 3, xb = min(max(x0 + 1, 0), W - 1) * 3;
    const uint8_t* r0 = fr + min(max(y0, 0), H - 1) * W * 3;
    const uint8_t* r1 = fr + min(max(y0 + 1, 0), H - 1) * W * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float p00 = (iy0 && ix0) ? (float)r0[xa + c] : 0.f, p01 = (iy0 && ix1) ? (float)r0[xb + c] : 0.f;
        const float p10 = (iy1 && ix0) ? (float)r1[xa + c] : 0.f, p11 = (iy1 && ix1) ? (float)r1[xb + c] : 0.f;
        const float top = fmaf(fx, p01 - p00, p00), bot = fmaf(fx, p11 - p10, p10);
        p[c] = fmaf(fy, bot - top, top);
    }
    if (bright != 1.f) {
#pragma unroll
        for (int c = 0; c < 3; ++c) p[c] = aug_clamp255(bright * p[c]);
    }
}

// step 5 (torchvision adjust_hue on [0, 1]), in place on the uint8 scale
__device__ __forceinline__ void aug_hue(float (&p)[3], float hue) {
    const float k = 1.f / 255.f;
    const float r = p[0] * k, g = p[1] * k, b = p[2] * k;
    const float maxc = fmaxf(r, fmaxf(g, b)), minc = fminf(r, fminf(g, b));
    const bool eqc = maxc == minc;
    const float cr = maxc - minc;
    const float s = cr / (eqc ? 1.f : maxc);
    const float inv = 1.f / (eqc ? 1.f : cr);
    const float rc = (maxc - r) * inv, gc = (maxc - g) * inv, bc = (maxc - b) * inv;
    float h;
    if (maxc == r) h = bc - gc;
    else if (maxc == g) h = 2.f + rc - bc;
    else h = 4.f + gc - rc;
    h = h / 6.f + 1.f;
    h -= floorf(h);  // fmod(., 1) of a positive value
    h += hue;
    h -= floorf(h);  // Python's % 1.0
    const float v = maxc;
    const float h6 = h * 6.f, fi = floorf(h6), f = h6 - fi;
    int i = (int)fi % 6;
    const float pp = fminf(fmaxf(v * (1.f - s), 0.f), 1.f);
    const float q = fminf(fmaxf(v * (1.f - s * f), 0.f), 1.f);
    const float t = fminf(fmaxf(v * (1.f - s * (1.f - f)), 0.f), 1.f);
    float o0, o1, o2;
    switch (i) {
        case 0: o0 = v; o1 = t; o2 = pp; break;
        case 1: o0 = q; o1 = v; o2 = pp; break;
        case 2: o0 = pp; o1 = v; o2 = t; break;
        case 3: o0 = pp; o1 = q; o2 = v; break;
        case 4: o0 = t; o1 = pp; o2 = v; break;
        default: o0 = v; o1 = pp; o2 = q; break;
    }
    p[0] = aug_clamp255(o0 * 255.f);
    p[1] = aug_clamp255(o1 * 255.f);
    p[2] = aug_clamp255(o2 * 255.f);
}

template <bool OUT_F32>
__global__ void __launch_bounds__(kAugThreads, 4) augment_frames_kernel(const uint8_t* __restrict__ src, void* __restrict__ dst,
                                                                         const float* __restrict__ params, int H, int W) {
    extern __shared__ __align__(16) uint8_t aug_frame[];
    __shared__ double red[kAugThreads / 32];
    __shared__ float mean_s;
    const long long f = blockIdx.x;
    const int npx = H * W, nb = npx * 3;
    const uint8_t* s = src + f * nb;
    if ((reinterpret_cast<uintptr_t>(s) & 15) == 0) {
        const int n16 = nb >> 4;
        for (int i = threadIdx.x; i < n16; i += kAugThreads) cp_async16(aug_frame + 16 * i, s + 16 * i);
        asm volatile("cp.async.commit_group;" ::: "memory");
        for (int i = (n16 << 4) + threadIdx.x; i < nb; i += kAugThreads) aug_frame[i] = s[i];
        cp_async_wait_all();
    } else {
        for (int i = threadIdx.x; i < nb; i += kAugThreads) aug_frame[i] = s[i];
    }
    float A[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) A[k] = params[f * 10 + k];
    const float bright = params[f * 10 + 6], contrast = params[f * 10 + 7], sat = params[f * 10 + 8], hue = params[f * 10 + 9];
    __syncthreads();

    float cshift = 0.f;  // (1 - c) m
    if (contrast != 1.f) {
        double acc = 0.0;
        for (int i = threadIdx.x; i < npx; i += kAugThreads) {
            float p[3];
            aug_sample(aug_frame, H, W, A, bright, i % W, i / W, p);
            acc += (double)aug_grey(p[0], p[1], p[2]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane_id() == 0) red[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            double t = 0.0;
            for (int w = 0; w < kAugThreads / 32; ++w) t += red[w];
            mean_s = (float)(t / (double)npx);
        }
        __syncthreads();
        cshift = (1.f - contrast) * mean_s;
    }
    const float sshift = 1.f - sat;
    for (int i = threadIdx.x; i < npx; i += kAugThreads) {
        float p[3];
        aug_sample(aug_frame, H, W, A, bright, i % W, i / W, p);
        if (contrast != 1.f) {
#pragma unroll
            for (int c = 0; c < 3; ++c) p[c] = aug_clamp255(fmaf(contrast, p[c], cshift));
        }
        if (sat != 1.f) {
            const float g = sshift * aug_grey(p[0], p[1], p[2]);
#pragma unroll
            for (int c = 0; c < 3; ++c) p[c] = aug_clamp255(fmaf(sat, p[c], g));
        }
        if (hue != 0.f) aug_hue(p, hue);
        const long long o = (f * npx + i) * 3;
        if (OUT_F32) {
            float* d = static_cast<float*>(dst) + o;
#pragma unroll
            for (int c = 0; c < 3; ++c) d[c] = aug_clamp255(p[c]);
        } else {
            uint8_t* d = static_cast<uint8_t*>(dst) + o;
#pragma unroll
            for (int c = 0; c < 3; ++c) d[c] = (uint8_t)__float2int_rn(aug_clamp255(p[c]));
        }
    }
}

}  // namespace vpt

extern "C" int vpt_augment_max_frame_bytes(void) {
    using namespace vpt;
    int dev = 0, optin = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    static int static_bytes = -1;  // the kernel's static shared memory (reduction slots), the same in both instantiations
    if (static_bytes < 0) {
        cudaFuncAttributes fa[2];
        if (cudaFuncGetAttributes(&fa[0], augment_frames_kernel<false>) != cudaSuccess ||
            cudaFuncGetAttributes(&fa[1], augment_frames_kernel<true>) != cudaSuccess) {
            cudaGetLastError();
            return 0;
        }
        static_bytes = (int)(fa[0].sharedSizeBytes > fa[1].sharedSizeBytes ? fa[0].sharedSizeBytes : fa[1].sharedSizeBytes);
    }
    return optin - static_bytes;
}

extern "C" int vpt_augment_frames(const uint8_t* src, void* dst, int32_t out_f32, const float* params, int32_t F, int32_t H, int32_t W,
                                  void* stream) {
    using namespace vpt;
    VPT_CHECK(src && dst && params && F > 0 && H > 0 && W > 0, "vpt_augment_frames: bad arguments");
    const int cap = vpt_augment_max_frame_bytes();
    VPT_CHECK(cap > 0, "vpt_augment_frames: no CUDA device to query the shared-memory opt-in");
    const long long nb = 3LL * H * W;
    VPT_CHECK(nb <= cap, "vpt_augment_frames: a %d x %d frame (%lld bytes) does not fit the %d bytes of shared memory a CTA can opt in to",
              H, W, nb, cap);
    void (*kern)(const uint8_t*, void*, const float*, int, int) = out_f32 ? augment_frames_kernel<true> : augment_frames_kernel<false>;
    static int attr[2] = {0, 0};
    if ((int)nb > attr[out_f32 ? 1 : 0]) {
        VPT_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)nb));
        attr[out_f32 ? 1 : 0] = (int)nb;
    }
    kern<<<F, kAugThreads, (size_t)nb, (cudaStream_t)stream>>>(src, dst, params, H, W);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}
