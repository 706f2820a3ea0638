// Stack-0 first convolution, fully fused: u8 NHWC frame -> (x/255) conv3x3(3->C0)+bias -> ReLU -> max_pool(3,2,1)
// -> bf16 NHWC + per-(tile, channel) statistics partials.
//
// K = 27 is too small for a warpgroup MMA to matter (the layer is 0.75 % of the FLOPs and bounded by its epilogue / output
// write), so the contraction runs on warp-level mma.sync m16n8k16: A = the im2col view of the u8 patch (u8 values
// are exact in bf16; fragments are gathered straight from the patch in shared memory, no im2col copy), B = the fp32
// weights split as bf16 hi + bf16 lo (K = 27 + 27 -> 64), fp32 accumulate: products are exact and the result is
// fp32-accurate (SURVEY.md section 7.2: the first conv is the largest single contributor to bf16 error otherwise).
//
// One CTA = one 8x8 tile of POOLED outputs of one frame = 17x17 conv outputs (19 m16 tiles) from a 19x19x3 patch.
// ~99 KB of shared memory at C0 = 128 -> two CTAs per SM overlap one CTA's pooling with the other's MMAs.
// F32OUT (precision mode): the conv tile is kept in fp32 and the output is fp32; the channels then go through the tile 64 at a time.
// TIN = float (fp32 frames on the uint8 scale, vpt_firstconv_pool_f32): an fp32 value is not exact in bf16, so the patch is split too,
// x = x_hi + x_lo, and A = x_hi | x_hi | 1 | x_lo against B = w_hi | w_lo | bias | w_hi (x_lo * w_lo, below 2^-16 relative, dropped):
// K = 96, 6 k-steps.  The x_lo k-steps run after the other four and only for a tile whose x_lo is not all zero (a CTA-wide vote
// while the patch is staged), so integer-valued frames take exactly the uint8 path's MMAs in the same order: bit-identical outputs.
#pragma once
#include <type_traits>

#include "attention.cuh"  // ldsm_x4 / mma_bf16_16816
#include "common.cuh"

namespace vpt {

constexpr int kFcTile = 8;               // pooled outputs per tile edge
constexpr int kFcConv = 2 * kFcTile + 1; // 17 conv rows/cols
constexpr int kFcIn = kFcConv + 2;       // 19 input rows/cols
constexpr int kFcThreads = 256;
constexpr int kFcPos = kFcConv * kFcConv;        // 289 conv positions
constexpr int kFcMTiles = (kFcPos + 15) / 16;    // 19
constexpr int kFcPatchElems = kFcIn * kFcIn * 3; // 1083
constexpr int kFcPatchBytes = 2192;              // bf16 patch + one zero element, 16-byte multiple

template <typename TIN>
struct FcIn {
    static constexpr bool kF32 = std::is_same<TIN, float>::value;
    static constexpr int kKSteps = kF32 ? 6 : 4;           // k-steps of 16: x_hi (w_hi, w_lo, bias) [+ x_lo (w_hi)]
    static constexpr int kBPitch = 16 * kKSteps + 8;       // 72 / 104 bf16 per weight row (144 / 208 B: conflict-free ldmatrix)
    static constexpr int kPatches = kF32 ? 2 : 1;          // x_hi [, x_lo]
};

template <bool F32OUT, typename TIN>
__global__ void __launch_bounds__(kFcThreads, 2) firstconv_pool_kernel(const TIN* __restrict__ img, const float* __restrict__ w,
                                                                       const float* __restrict__ bias, void* __restrict__ out_,
                                                                       float2* __restrict__ stat_part, int H, int W, int C0, long long total_tiles, int zp) {
    pdl_sync();
    extern __shared__ __align__(16) uint8_t fc_smem[];
    using In = FcIn<TIN>;
    constexpr int kBPitch = In::kBPitch, kKCols = 16 * In::kKSteps;
    __nv_bfloat16* patch = reinterpret_cast<__nv_bfloat16*>(fc_smem);                                  // [19][19][3]
    __nv_bfloat16* patch_lo = reinterpret_cast<__nv_bfloat16*>(fc_smem + kFcPatchBytes);               // [19][19][3] (fp32 frames)
    __nv_bfloat16* Bs = reinterpret_cast<__nv_bfloat16*>(fc_smem + In::kPatches * kFcPatchBytes);     // [C0][kBPitch]
    using CT = typename std::conditional<F32OUT, float, __nv_bfloat16>::type;
    const int CB = F32OUT ? 64 : C0;  // channels per pass through the conv tile
    const int cpitch = CB + 8;
    CT* ctile = reinterpret_cast<CT*>(Bs + (size_t)C0 * kBPitch);                                    // [289][CB+8]
    CT* const out = reinterpret_cast<CT*>(out_);
    const int tiles_x = (W / 2) / kFcTile, tiles_y = (H / 2) / kFcTile;
    const int tiles = tiles_x * tiles_y;

    // ---- hi/lo-split weights, staged once per (persistent) CTA
    for (int i = threadIdx.x; i < C0 * kKCols; i += kFcThreads) {
        const int n = i / kKCols, k = i % kKCols;
        float v = 0.f;
        if (k >= 64) {  // fp32 frames: w_hi against x_lo
            if (k < 64 + 27) v = __ldg(w + n * 27 + k - 64);
        } else if (k < 27) {
            v = __ldg(w + n * 27 + k);
        } else if (k < 54) {
            const float x = __ldg(w + n * 27 + k - 27);
            v = x - __bfloat162float(__float2bfloat16_rn(x));
        } else if (k == 54) {  // bias rides along as two extra K columns against a constant-one A column
            v = __ldg(bias + n);
        } else if (k == 55) {
            const float x = __ldg(bias + n);
            v = x - __bfloat162float(__float2bfloat16_rn(x));
        }
        Bs[n * kBPitch + k] = __float2bfloat16_rn(v);
    }

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tg = lane & 3;
    // per-thread patch offsets of the k indices this lane feeds: k -> (ky, kx*3+c) -> ky*57 + q ; k in [27,54) repeats
    int koff[4][4];
    bool kval[4][4];
#pragma unroll
    for (int s = 0; s < 4; ++s)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int k = 16 * s + 2 * tg + (e & 1) + ((e >> 1) << 3);
            const int kk = k < 27 ? k : k - 27;
            kval[s][e] = k < 54;
            koff[s][e] = kval[s][e] ? (kk / 9) * (kFcIn * 3) + kk % 9 : 0;
        }

    // (a) patch staging without div/mod in the tile loop: each thread owns fixed patch elements; the NEXT tile's bytes are
    // prefetched into registers while the current tile is computed
    constexpr int kPE = (kFcPatchElems + kFcThreads - 1) / kFcThreads;  // 5
    int pe_row[kPE], pe_col[kPE];  // input row / byte column (x*3+c) inside the patch
#pragma unroll
    for (int j = 0; j < kPE; ++j) {
        const int i = threadIdx.x + j * kFcThreads;
        pe_row[j] = i / (kFcIn * 3);
        pe_col[j] = i % (kFcIn * 3);
    }
    TIN pre[kPE];
    auto prefetch = [&](long long tid) {
        const long long f = tid / tiles;
        const int tile = (int)(tid % tiles);
        const int Yin0 = 2 * (tile / tiles_x) * kFcTile - 2, Xin0 = 2 * (tile % tiles_x) * kFcTile - 2;
        const TIN* fimg = img + f * (long long)H * W * 3;
#pragma unroll
        for (int j = 0; j < kPE; ++j) {
            const int Y = Yin0 + pe_row[j], xb = Xin0 * 3 + pe_col[j];  // xb = X*3 + c
            const bool ok = (threadIdx.x + j * kFcThreads < kFcPatchElems) && Y >= 0 && Y < H && xb >= 0 && xb < W * 3;
            pre[j] = ok ? __ldg(fimg + (long long)Y * W * 3 + xb) : (TIN)0;
        }
    };
    if ((long long)blockIdx.x < total_tiles) prefetch(blockIdx.x);

  for (long long tid = blockIdx.x; tid < total_tiles; tid += gridDim.x) {
    const long long f = tid / tiles;
    const int tile = (int)(tid % tiles);
    const int PY0 = (tile / tiles_x) * kFcTile, PX0 = (tile % tiles_x) * kFcTile;
    // ---- stage the input patch (u8 -> bf16, exact; fp32 -> bf16 hi + bf16 lo) from the prefetched registers, then prefetch the next tile
    int any_lo = 0;  // fp32 frames: some x_lo of this tile is not zero (the x_lo k-steps run)
    if constexpr (In::kF32) {
        int nz = 0;
#pragma unroll
        for (int j = 0; j < kPE; ++j) {
            const int i = threadIdx.x + j * kFcThreads;
            if (i < kFcPatchElems) {
                const __nv_bfloat16 hi = __float2bfloat16_rn(pre[j]);
                const float lo = pre[j] - __bfloat162float(hi);
                patch[i] = hi;
                patch_lo[i] = __float2bfloat16_rn(lo);
                nz |= lo != 0.f;
            }
        }
        any_lo = __syncthreads_or(nz);
    } else {
#pragma unroll
        for (int j = 0; j < kPE; ++j) {
            const int i = threadIdx.x + j * kFcThreads;
            if (i < kFcPatchElems) patch[i] = __float2bfloat16_rn((float)pre[j]);
        }
    }
    if (tid + gridDim.x < total_tiles) prefetch(tid + gridDim.x);
    const int Ho = H / 2, Wo = W / 2, opitch = Wo + zp;  // ZP layout: one extra zero column / row
    CT* fout = out + f * (long long)(Ho + zp) * opitch * C0;
  for (int cg = 0; cg < C0; cg += CB) {
    __syncthreads();  // patch (and, first time, weights) visible; previous pass's pooling finished reading ctile

    for (int mt = warp; mt < kFcMTiles; mt += kFcThreads / 32) {
        // A fragments (rows g and g+8 of this m-tile) for the 4 k-steps, gathered from the patch
        int pos[2], pbase[2];
        bool inimg[2];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            const int p = min(mt * 16 + g + rr * 8, kFcPos - 1);
            pos[rr] = mt * 16 + g + rr * 8;
            const int cy = p / kFcConv, cx = p % kFcConv;
            pbase[rr] = (cy * kFcIn + cx) * 3;
            const int Y = 2 * PY0 - 1 + cy, X = 2 * PX0 - 1 + cx;
            inimg[rr] = (Y >= 0 && Y < H && X >= 0 && X < W);
        }
        uint32_t af[4][4];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {  // hh = 0: k, k+1 ; hh = 1: k+8, k+9
                    const uint16_t lo = kval[s][2 * hh] ? *reinterpret_cast<const uint16_t*>(patch + pbase[rr] + koff[s][2 * hh]) : (uint16_t)0;
                    const uint16_t hi = kval[s][2 * hh + 1] ? *reinterpret_cast<const uint16_t*>(patch + pbase[rr] + koff[s][2 * hh + 1]) : (uint16_t)0;
                    af[s][rr + 2 * hh] = (uint32_t)lo | ((uint32_t)hi << 16);
                }
            }
        }
        if (tg == 3) af[3][0] = af[3][1] = 0x3F803F80u;  // k = 54, 55: constant 1.0 (x the bias columns of B)

        for (int nh = cg / 64; nh < (cg + CB) / 64; ++nh) {  // 64 output channels at a time
            float acc[8][4];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll
            for (int s = 0; s < 4; ++s) {
#pragma unroll
                for (int np = 0; np < 4; ++np) {
                    uint32_t b0, b1, b2, b3;
                    const int nrow = nh * 64 + np * 16 + (lane & 7) + ((lane >> 4) << 3);
                    const int kcol = s * 16 + (((lane >> 3) & 1) << 3);
                    ldsm_x4(smem_u32(Bs + nrow * kBPitch + kcol), b0, b1, b2, b3);
                    mma_bf16_16816(acc[2 * np], af[s][0], af[s][1], af[s][2], af[s][3], b0, b1);
                    mma_bf16_16816(acc[2 * np + 1], af[s][0], af[s][1], af[s][2], af[s][3], b2, b3);
                }
            }
            if constexpr (In::kF32) {
                if (any_lo) {
                    // A = x_lo at k' = k - 64 in [0, 27): the patch offsets of k' are koff[s] of the first two k-steps (k' < 27).  One
                    // k-step's fragments at a time (4 registers), gathered after the x_hi MMAs, to keep the register pressure of the u8 path.
#pragma unroll
                    for (int s = 0; s < 2; ++s) {
                        uint32_t af_lo[4];
#pragma unroll
                        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                            for (int hh = 0; hh < 2; ++hh) {
                                const int k = 16 * s + 2 * tg + 8 * hh;  // k' of the pair's first element
                                const uint16_t lo = k < 27 ? *reinterpret_cast<const uint16_t*>(patch_lo + pbase[rr] + koff[s][2 * hh]) : (uint16_t)0;
                                const uint16_t hi = k + 1 < 27 ? *reinterpret_cast<const uint16_t*>(patch_lo + pbase[rr] + koff[s][2 * hh + 1]) : (uint16_t)0;
                                af_lo[rr + 2 * hh] = (uint32_t)lo | ((uint32_t)hi << 16);
                            }
#pragma unroll
                        for (int np = 0; np < 4; ++np) {
                            uint32_t b0, b1, b2, b3;
                            const int nrow = nh * 64 + np * 16 + (lane & 7) + ((lane >> 4) << 3);
                            const int kcol = 64 + s * 16 + (((lane >> 3) & 1) << 3);
                            ldsm_x4(smem_u32(Bs + nrow * kBPitch + kcol), b0, b1, b2, b3);
                            mma_bf16_16816(acc[2 * np], af_lo[0], af_lo[1], af_lo[2], af_lo[3], b0, b1);
                            mma_bf16_16816(acc[2 * np + 1], af_lo[0], af_lo[1], af_lo[2], af_lo[3], b2, b3);
                        }
                    }
                }
            }
            // raw pre-activation values; ReLU is applied after the max (monotone), positions outside the image hold 0
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                if (pos[rr] >= kFcPos) continue;
                CT* crow = ctile + (size_t)pos[rr] * cpitch + (nh * 64 - cg) + 2 * tg;
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const float v0 = inimg[rr] ? acc[nt][2 * rr] : 0.f;
                    const float v1 = inimg[rr] ? acc[nt][2 * rr + 1] : 0.f;
                    if constexpr (F32OUT) *reinterpret_cast<float2*>(crow + nt * 8) = make_float2(v0, v1);
                    else *reinterpret_cast<uint32_t*>(crow + nt * 8) = pack_bf16(v0, v1);
                }
            }
        }
    }
    __syncthreads();

    // ---- 3x3 / stride-2 max over the conv tile, 16 B (8 bf16 / 4 fp32 channels) per item
    if constexpr (F32OUT) {
        const int C4 = CB / 4;
        for (int i = threadIdx.x; i < kFcTile * kFcTile * C4; i += kFcThreads) {
            const int c4 = i % C4, px = (i / C4) % kFcTile, py = i / (C4 * kFcTile);
            float4 m = make_float4(0.f, 0.f, 0.f, 0.f);  // starting from 0 == applying the ReLU after the max
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    const int p = (2 * py + dy) * kFcConv + 2 * px + dx;
                    const float4 v = *reinterpret_cast<const float4*>(ctile + (size_t)p * cpitch + 4 * c4);
                    m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
                }
            *reinterpret_cast<float4*>(fout + ((long long)(PY0 + py) * opitch + PX0 + px) * C0 + cg + 4 * c4) = m;
        }
    } else {
    const int C8 = C0 / 8;
    for (int i = threadIdx.x; i < kFcTile * kFcTile * C8; i += kFcThreads) {
        const int c8 = i % C8, px = (i / C8) % kFcTile, py = i / (C8 * kFcTile);
        uint4 m = make_uint4(0, 0, 0, 0);  // starting from 0 == applying the ReLU after the max
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const int p = (2 * py + dy) * kFcConv + 2 * px + dx;
                const uint4 v = *reinterpret_cast<const uint4*>(ctile + (size_t)p * cpitch + 8 * c8);
                m.x = bf16x2_max(m.x, v.x); m.y = bf16x2_max(m.y, v.y);
                m.z = bf16x2_max(m.z, v.z); m.w = bf16x2_max(m.w, v.w);
            }
        *reinterpret_cast<uint4*>(fout + ((long long)(PY0 + py) * opitch + PX0 + px) * C0 + 8 * c8) = m;
    }
    }
  }
    if (zp) {  // edge tiles write the zero column x = Wo and the zero row y = Ho (plus the corner)
        const int C8 = C0 * (int)sizeof(CT) / 16;  // 16-byte words per pixel
        uint4* fo = reinterpret_cast<uint4*>(fout);
        const bool right = (PX0 + kFcTile == Wo), bottom = (PY0 + kFcTile == Ho);
        if (right)
            for (int i = threadIdx.x; i < kFcTile * C8; i += kFcThreads)
                fo[((long long)(PY0 + i / C8) * opitch + Wo) * C8 + (i % C8)] = make_uint4(0, 0, 0, 0);
        if (bottom)
            for (int i = threadIdx.x; i < (kFcTile + (right ? 1 : 0)) * C8; i += kFcThreads)
                fo[((long long)Ho * opitch + PX0 + i / C8) * C8 + (i % C8)] = make_uint4(0, 0, 0, 0);
    }
    __syncthreads();  // the tile's pooled outputs are visible to the whole block; ctile / patch may be reused
    if (stat_part) {  // per-channel (sum, sumsq) of the tile's pooled outputs, in a fixed order
        for (int c = threadIdx.x; c < C0; c += kFcThreads) {
            float cs = 0.f, css = 0.f;
            for (int py = 0; py < kFcTile; ++py)
                for (int px = 0; px < kFcTile; ++px) {
                    const CT o = fout[((long long)(PY0 + py) * opitch + PX0 + px) * C0 + c];
                    float v;
                    if constexpr (F32OUT) v = o;
                    else v = __bfloat162float(o);
                    cs += v;
                    css = fmaf(v, v, css);
                }
            stat_part[(f * tiles + tile) * C0 + c] = make_float2(cs, css);
        }
    }
  }
}

}  // namespace vpt

// statistics partials per frame: one per (8x8 pooled tile, channel), index tile * C0 + channel
extern "C" int vpt_firstconv_stat_parts(int32_t F, int32_t H, int32_t W, int32_t C0) {
    (void)F;
    return (H / 16) * (W / 16) * C0;
}

// Kernel choice of the C ABI.  This build has one first-convolution kernel, so every mode selects it.
extern "C" int vpt_set_firstconv_mode(int32_t mode) {
    (void)mode;
    return VPT_OK;
}

namespace vpt {

template <typename TIN>
static int firstconv_pool_launch(const char* fn, const TIN* img, const float* w, const float* bias, void* out, float* stat_part, int32_t F,
                                 int32_t H, int32_t W, int32_t C0, int32_t zp, int32_t out_f32, void* stream) {
    VPT_CHECK(img && w && bias && out && F > 0, "%s: null argument", fn);
    VPT_CHECK(H % 16 == 0 && W % 16 == 0 && H >= 16 && W >= 16, "%s: H, W must be multiples of 16 (H=%d W=%d)", fn, H, W);
    VPT_CHECK(C0 == 64 || C0 == 128 || C0 == 192 || C0 == 256, "%s: C0=%d not in {64,128,192,256}", fn, C0);
    const long long blocks = (long long)F * (H / 16) * (W / 16);
    VPT_CHECK(blocks < 2147483647LL, "%s: too many tiles", fn);
    using In = FcIn<TIN>;
    const int CB = out_f32 ? 64 : C0;
    const size_t smem = (size_t)In::kPatches * kFcPatchBytes + (size_t)C0 * In::kBPitch * 2 + (size_t)kFcPos * (CB + 8) * (out_f32 ? 4 : 2);
    void (*kern)(const TIN*, const float*, const float*, void*, float2*, int, int, int, long long, int) =
        out_f32 ? firstconv_pool_kernel<true, TIN> : firstconv_pool_kernel<false, TIN>;
    static size_t attr[2] = {0, 0};  // (one table per frame type)
    if (smem > attr[out_f32 ? 1 : 0]) {
        VPT_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr[out_f32 ? 1 : 0] = smem;
    }
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    if (per_sm > 2) per_sm = 2;
    if (per_sm < 1) per_sm = 1;
    long long grid = (long long)num_sms() * per_sm;
    if (grid > blocks) grid = blocks;
    launch_k(kern, dim3((unsigned)grid), dim3(kFcThreads), smem, (cudaStream_t)stream,
             img, w, bias, out, reinterpret_cast<float2*>(stat_part), H, W, C0, blocks, zp ? 1 : 0);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

}  // namespace vpt

extern "C" int vpt_firstconv_pool(const uint8_t* img, const float* w, const float* bias, void* out, float* stat_part, int32_t F,
                                  int32_t H, int32_t W, int32_t C0, int32_t zp, int32_t out_f32, void* stream) {
    return vpt::firstconv_pool_launch("vpt_firstconv_pool", img, w, bias, out, stat_part, F, H, W, C0, zp, out_f32, stream);
}

extern "C" int vpt_firstconv_pool_f32(const float* img, const float* w, const float* bias, void* out, float* stat_part, int32_t F,
                                      int32_t H, int32_t W, int32_t C0, int32_t zp, int32_t out_f32, void* stream) {
    return vpt::firstconv_pool_launch("vpt_firstconv_pool_f32", img, w, bias, out, stat_part, F, H, W, C0, zp, out_f32, stream);
}
