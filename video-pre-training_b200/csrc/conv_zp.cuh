// Implicit-GEMM 3x3 convolution on wgmma with the input tile REUSED across the 9 taps from shared memory.
//
// Implicit GEMM re-fetches the A tile for every tap, which makes a tensor-core convolution bound by the bytes TMA can deliver into
// one SM rather than by the tensor pipe.  This kernel removes the 9x A redundancy:
//
//   * activations live in the "ZP" layout [F][H+1][W+1][C] (bf16) whose row y=H and column x=W are zero: with one shared
//     zero row / column every 3x3 neighbour of pixel q (a linear row index over the whole tensor) is the row q + dy*(W+1) + dx,
//     so a tile of 128 consecutive rows needs ONE contiguous span of  rows + 2*(W+2)  input rows per 64 channels;
//   * the span is fetched once per 64-channel block by plain 2-D TMA (out-of-range rows are zero-filled) and all 9 taps are
//     issued as wgmmas whose A descriptors start at span + ((dy+1)*(W+1) + dx+1)*128 B (for K-major SWIZZLE_128B operands the
//     swizzle is a function of the absolute shared-memory address, so a descriptor start advanced by any multiple of 128 B reads
//     the shifted rows; tools/desc_experiment.py checks this on the GEMM kernel);
//   * weights stream through their own pipeline, one [block_n][64] tile per (channel block, tap).
//
//   warps 0..7: two wgmma warpgroups (64 rows each) + epilogue   warp 8: A-span TMA producer   warp 9: weight TMA producer
// Epilogue = GroupNorm fold (border-class tables), ReLU, residual, bf16 store in ZP layout (border rows are written as
// zeros, which maintains the layout invariant), per-row (sum, sumsq) partials for the next layer's statistics.
#pragma once
#include "common.cuh"
#include "gemm_tc.cuh"

namespace vpt {

static int g_cz_dbg = 0;

constexpr int kCzThreads = 32 * kNumEpiWarps + 64;  // 10 warps
constexpr int kCzMaxBStages = 8;

struct ConvZpParams {
    long long Q;  // total rows = F * FS
    int H, W, Wp, FS;
    int N, block_n, num_n_tiles, cin, cin_blocks;
    int a_box_rows, a_boxes, a_stage_bytes, b_stages;
    int dbg;              // experiment: 1 = epilogue skips its global stores, 2 = skips the whole epilogue body
    int bo;               // descriptor experiment: set the base-offset field of the shifted A descriptors
    long long num_m_tiles;
    const float* mr;
    const float* S1;
    const float* S2;
    int relu;
    const __nv_bfloat16* residual;
    __nv_bfloat16* out;
    float* stat_part;  // [Q][2 * num_n_tiles] float2 or null
    const float* Ef;         // [F][9][N] per-frame fold table (two-norm composition) or null
    const float* res_scale;  // [F][N] or null: residual enters as res_scale * r + res_shift
    const float* res_shift;
};

template <int BN>
__global__ void __launch_bounds__(kCzThreads, 1)
conv3x3_zp_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const ConvZpParams p) {
    pdl_sync();
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
    constexpr uint32_t b_stage_bytes = (uint32_t)BN * kBlockK * 2;
    uint8_t* smem_a = smem;                                        // 2 A-span stages
    uint8_t* smem_b = smem + 2 * (size_t)p.a_stage_bytes;          // b_stages weight tiles
    float* stg_all = reinterpret_cast<float*>(smem_b + (size_t)p.b_stages * b_stage_bytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stg_all) + kStgBytes);
    uint64_t* a_full = bars;
    uint64_t* a_empty = bars + 2;
    uint64_t* b_full = bars + 4;
    uint64_t* b_empty = bars + 4 + kCzMaxBStages;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == kNumEpiWarps && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < 2; ++i) {
            mbar_init(&a_full[i], 1);
            mbar_init(&a_empty[i], 2);  // one arrival per consumer warpgroup
        }
        for (int i = 0; i < p.b_stages; ++i) {
            mbar_init(&b_full[i], 1);
            mbar_init(&b_empty[i], 2);
        }
        fence_barrier_init();
    }
    __syncthreads();

    const long long num_tiles = p.num_m_tiles * p.num_n_tiles;
    const long long tile_begin = (long long)blockIdx.x;
    const long long tile_step = (long long)gridDim.x;
    const int halo = p.Wp + 1;  // rows before / after the tile that the taps reach

    if (warp == kNumEpiWarps) {
        if (lane == 0) {
            // ================= A-span producer =================
            int stage = 0;
            uint32_t phase = 0;
            bool ok = true;
            for (long long tile = tile_begin; tile < num_tiles && ok; tile += tile_step) {
                const long long m_tile = tile / p.num_n_tiles;
                const long long span0 = m_tile * kBlockM - halo;
                for (int cb = 0; cb < p.cin_blocks; ++cb) {
                    if (!(ok = mbar_wait(&a_empty[stage], phase ^ 1u, 0x110u))) break;
                    mbar_expect_tx(&a_full[stage], (uint32_t)p.a_stage_bytes);
                    uint8_t* sa = smem_a + (size_t)stage * p.a_stage_bytes;
                    for (int b = 0; b < p.a_boxes; ++b)
                        tma_load_2d(sa + (size_t)b * p.a_box_rows * 128, &tmA, &a_full[stage], cb * kBlockK, (int)(span0 + (long long)b * p.a_box_rows));
                    advance(stage, phase, 2);
                }
            }
        }
    } else if (warp == kNumEpiWarps + 1) {
        if (lane == 0) {
            // ================= weight producer =================
            int stage = 0;
            uint32_t phase = 0;
            bool ok = true;
            for (long long tile = tile_begin; tile < num_tiles && ok; tile += tile_step) {
                const int n0 = (int)(tile % p.num_n_tiles) * BN;
                for (int cb = 0; cb < p.cin_blocks && ok; ++cb) {
                    for (int tap = 0; tap < 9; ++tap) {
                        if (!(ok = mbar_wait(&b_empty[stage], phase ^ 1u, 0x120u))) break;
                        mbar_expect_tx(&b_full[stage], b_stage_bytes);
                        tma_load_2d(smem_b + (size_t)stage * b_stage_bytes, &tmB, &b_full[stage], tap * p.cin + cb * kBlockK, n0);
                        advance(stage, phase, p.b_stages);
                    }
                }
            }
        }
    } else {
        // ================= wgmma + epilogue (warps 0..7) =================
        const int wg = warp >> 2;                     // warpgroup: rows 64*wg .. 64*wg+63 of the tile
        const int quarter = 2 * wg + (warp & 1);
        const int grp = (warp >> 1) & 1;              // column half
        float* stg = stg_all + (size_t)wg * 64 * kStgPitch;
        const float* my_row = stg + (size_t)((warp & 1) * 32 + lane) * kStgPitch;
        const int nchunks = BN >> 5;
        const int c_begin = grp == 0 ? 0 : (nchunks + 1) >> 1;
        const int c_end = grp == 0 ? (nchunks + 1) >> 1 : nchunks;
        const int P = p.num_n_tiles * 2;
        const bool tab_vec = ((p.N & 3) == 0);
        const bool leader = (threadIdx.x & 127) == 0;
        int astage = 0, bstage = 0;
        uint32_t aphase = 0, bphase = 0;
        bool ok = true;
        for (long long tile = tile_begin; tile < num_tiles && ok; tile += tile_step) {
            const long long m_tile = tile / p.num_n_tiles;
            const int n_tile = (int)(tile % p.num_n_tiles);
            const int n0 = n_tile * BN;
            // ---- main loop: 64 rows x BN channels of this warpgroup over (channel block, tap)
            float frag[BN / 64][32];
            for (int cb = 0; cb < p.cin_blocks && ok; ++cb) {
                if (!(ok = mbar_wait(&a_full[astage], aphase, 0x310u))) break;
                const uint32_t a_base = smem_u32(smem_a + (size_t)astage * p.a_stage_bytes) + (uint32_t)wg * 64u * 128u;
                int prev = -1;
                for (int tap = 0; tap < 9; ++tap) {
                    if (!(ok = mbar_wait(&b_full[bstage], bphase, 0x320u))) break;
                    const uint32_t b_addr = smem_u32(smem_b + (size_t)bstage * b_stage_bytes);
                    const int row_off = (tap / 3) * p.Wp + (tap % 3);  // (dy+1)*Wp + (dx+1)
                    const uint32_t a_addr = a_base + (uint32_t)row_off * 128u;
                    const uint64_t a_bo = p.bo ? ((uint64_t)((a_addr >> 7) & 7u) << 49) : 0ull;
                    wgmma_fence();
                    wg_mma_kblock<false, BN>(frag, a_addr, b_addr, a_bo, (cb | tap) != 0);
                    wgmma_commit();
                    wgmma_wait<1>();
                    if (prev >= 0 && leader) mbar_arrive(&b_empty[prev]);
                    prev = bstage;
                    advance(bstage, bphase, p.b_stages);
                }
                wgmma_wait<0>();
                if (prev >= 0 && leader) mbar_arrive(&b_empty[prev]);
                if (leader) mbar_arrive(&a_empty[astage]);
                advance(astage, aphase, 2);
            }
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) wgmma_reg_fence(frag[j]);
            if (!ok) break;
            named_bar_sync(1 + wg, 128);
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) wgmma_frag_store(frag[j], stg, kStgPitch, j * 64);
            named_bar_sync(1 + wg, 128);

            const long long q = m_tile * kBlockM + quarter * 32 + lane;
            const bool row_ok = q < p.Q;
            // decode the ZP row: frame, y, x
            const long long f = q / p.FS;
            const int r = (int)(q - f * p.FS);
            const int y = r / p.Wp, x = r - y * p.Wp;
            const bool interior = row_ok && (y < p.H) && (x < p.W);
            float ga = 1.f, gb = 0.f;
            if (p.mr != nullptr && interior) {
                const float mean = __ldg(p.mr + 2 * f), rstd = __ldg(p.mr + 2 * f + 1);
                ga = rstd;
                gb = rstd * mean;
            }
            const int cy = (y == 0) ? 0 : ((y == p.H - 1) ? 2 : 1);
            const int cx = (x == 0) ? 0 : ((x == p.W - 1) ? 2 : 1);
            const int cls = interior ? cy * 3 + cx : 0;
            const float* s1row = p.S1 ? p.S1 + (size_t)cls * p.N : nullptr;
            const float* s2row = p.S2 ? p.S2 + (size_t)cls * p.N : nullptr;
            if (p.Ef) {  // per-frame fold table: out = ga * acc + Ef[f][cls][c]
                s1row = nullptr;
                s2row = p.Ef + ((size_t)(interior ? f : 0) * 9 + cls) * p.N;
            }
            const float* rarow = (p.res_scale && interior) ? p.res_scale + (size_t)f * p.N : nullptr;
            const float* rbrow = (p.res_scale && interior) ? p.res_shift + (size_t)f * p.N : nullptr;
            float st_s = 0.f, st_ss = 0.f;

            for (int c = c_begin; c < (p.dbg == 2 ? c_begin : c_end); ++c) {
                const int nb = n0 + c * 32;
                const int lim = min(32, min(BN - c * 32, p.N - nb));
                if (!row_ok || lim <= 0) continue;
                uint32_t acc[32];
                stg_ld_32(my_row + c * 32, acc);
                __nv_bfloat16* op = p.out + (size_t)q * p.N + nb;
                const bool full = (lim == 32) && ((p.N & 7) == 0);
                if (!interior) {  // zero row / column of the ZP layout
                    if (full) {
#pragma unroll
                        for (int qq = 0; qq < 4; ++qq) reinterpret_cast<uint4*>(op)[qq] = make_uint4(0, 0, 0, 0);
                    } else {
                        for (int j = 0; j < lim; ++j) op[j] = __float2bfloat16_rn(0.f);
                    }
                    continue;
                }
                float v[32];
                if (full && tab_vec) {
#pragma unroll
                    for (int qq = 0; qq < 8; ++qq) {
                        float4 a1 = s1row ? __ldg(reinterpret_cast<const float4*>(s1row + nb) + qq) : make_float4(0, 0, 0, 0);
                        float4 a2 = s2row ? __ldg(reinterpret_cast<const float4*>(s2row + nb) + qq) : make_float4(0, 0, 0, 0);
                        v[4 * qq + 0] = fmaf(ga, __uint_as_float(acc[4 * qq + 0]), fmaf(-gb, a1.x, a2.x));
                        v[4 * qq + 1] = fmaf(ga, __uint_as_float(acc[4 * qq + 1]), fmaf(-gb, a1.y, a2.y));
                        v[4 * qq + 2] = fmaf(ga, __uint_as_float(acc[4 * qq + 2]), fmaf(-gb, a1.z, a2.z));
                        v[4 * qq + 3] = fmaf(ga, __uint_as_float(acc[4 * qq + 3]), fmaf(-gb, a1.w, a2.w));
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        float a1 = 0.f, a2 = 0.f;
                        if (j < lim) {
                            if (s1row) a1 = __ldg(s1row + nb + j);
                            if (s2row) a2 = __ldg(s2row + nb + j);
                        }
                        v[j] = fmaf(ga, __uint_as_float(acc[j]), fmaf(-gb, a1, a2));
                    }
                }
                if (p.relu == 1) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
                }
                if (p.residual != nullptr) {
                    const __nv_bfloat16* rp = p.residual + (size_t)q * p.N + nb;
                    if (rarow) {
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            if (j < lim) v[j] += fmaf(__ldg(rarow + nb + j), __bfloat162float(rp[j]), __ldg(rbrow + nb + j));
                    } else if (full) {
#pragma unroll
                        for (int qq = 0; qq < 4; ++qq) {
                            uint4 rr = __ldg(reinterpret_cast<const uint4*>(rp) + qq);
                            v[8 * qq + 0] += bf16_lo(rr.x); v[8 * qq + 1] += bf16_hi(rr.x);
                            v[8 * qq + 2] += bf16_lo(rr.y); v[8 * qq + 3] += bf16_hi(rr.y);
                            v[8 * qq + 4] += bf16_lo(rr.z); v[8 * qq + 5] += bf16_hi(rr.z);
                            v[8 * qq + 6] += bf16_lo(rr.w); v[8 * qq + 7] += bf16_hi(rr.w);
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            if (j < lim) v[j] += __bfloat162float(rp[j]);
                    }
                }
                if (p.relu == 2) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
                }
                uint32_t pk[16];
#pragma unroll
                for (int j = 0; j < 16; ++j) pk[j] = pack_bf16(v[2 * j], v[2 * j + 1]);
                if (p.stat_part) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const float lo = bf16_lo(pk[j]), hi = bf16_hi(pk[j]);
                        if (2 * j < lim) { st_s += lo; st_ss = fmaf(lo, lo, st_ss); }
                        if (2 * j + 1 < lim) { st_s += hi; st_ss = fmaf(hi, hi, st_ss); }
                    }
                }
                if (p.dbg == 1) {
                    if (pk[0] == 0x12345678u) op[0] = __float2bfloat16_rn(0.f);  // keep the values live, store (almost) never
                } else if (full) {
#pragma unroll
                    for (int qq = 0; qq < 4; ++qq)
                        reinterpret_cast<uint4*>(op)[qq] = make_uint4(pk[4 * qq], pk[4 * qq + 1], pk[4 * qq + 2], pk[4 * qq + 3]);
                } else {
#pragma unroll
                    for (int j = 0; j < 32; ++j)
                        if (j < lim) op[j] = __float2bfloat16_rn(v[j]);
                }
            }
            if (p.stat_part && row_ok) reinterpret_cast<float2*>(p.stat_part)[(size_t)q * P + n_tile * 2 + grp] = make_float2(st_s, st_ss);
        }
    }
}

}  // namespace vpt

namespace vpt {
// Weight-tile width.  A handful of frames (rollout: F = 1, 1089 rows at 32 x 32): the launch is a read of the weight tensor through
// the few SMs that have a tile, so narrower weight tiles put more SMs (each fetching a slice) on it.
static inline void conv_zp_block_n(long long Q, int N, int* bn, int* nt) {
    choose_block_n(N, bn, nt);
    const long long tiles = (Q + kBlockM - 1) / kBlockM;
    if (tiles * *nt >= 64 || *bn == 64) return;
    *bn = 64;
    *nt = (N + 63) / 64;
}
}  // namespace vpt

extern "C" int vpt_conv3x3_zp(const vpt_conv_zp_args* a, void* stream) {
    using namespace vpt;
    VPT_CHECK(a && a->x && a->w && a->out, "vpt_conv3x3_zp: null operand");
    const int H = a->H, W = a->W, C = a->Cin, N = a->Cout;
    VPT_CHECK(a->F > 0 && H >= 2 && W >= 2 && C > 0 && C % 64 == 0 && N > 0 && N % 16 == 0,
              "vpt_conv3x3_zp: need F>0, H,W>=2, Cin %% 64 == 0, Cout %% 16 == 0 (F=%d H=%d W=%d Cin=%d Cout=%d)", a->F, H, W, C, N);
    // two stages of the 128 + 2*(W+2)-row input span, the fp32 staging tiles and two weight stages must fit in shared memory
    VPT_CHECK(W <= 182, "vpt_conv3x3_zp: W=%d too wide (at most 182: two input spans of 128 + 2*(W+2) rows must fit in shared memory)", W);
    VPT_CHECK(((uintptr_t)a->x & 15) == 0 && ((uintptr_t)a->w & 15) == 0 && ((uintptr_t)a->out & 15) == 0, "vpt_conv3x3_zp: pointers must be 16-byte aligned");
    ConvZpParams p;
    memset(&p, 0, sizeof(p));
    p.H = H; p.W = W; p.Wp = W + 1; p.FS = (H + 1) * (W + 1);
    p.Q = (long long)a->F * p.FS;
    VPT_CHECK(p.Q < 2147483647LL, "vpt_conv3x3_zp: too many rows for 32-bit TMA coordinates");
    p.N = N; p.cin = C; p.cin_blocks = C / 64;
    conv_zp_block_n(p.Q, N, &p.block_n, &p.num_n_tiles);
    p.num_m_tiles = (p.Q + kBlockM - 1) / kBlockM;
    const int span = kBlockM + 2 * (p.Wp + 1);
    p.a_boxes = (span + 255) / 256;
    p.a_box_rows = ((span + p.a_boxes - 1) / p.a_boxes + 7) / 8 * 8;
    VPT_CHECK(p.a_box_rows <= 256, "vpt_conv3x3_zp: span does not fit the TMA box limit");
    p.a_stage_bytes = p.a_boxes * p.a_box_rows * 128;
    const uint32_t b_stage_bytes = (uint32_t)p.block_n * kBlockK * 2;
    const size_t fixed_bytes = 1024 + 2 * (size_t)p.a_stage_bytes + kStgBytes + (4 + 2 * kCzMaxBStages) * 8;
    int bst = (int)((227 * 1024 - (long long)fixed_bytes) / b_stage_bytes);
    if (bst > kCzMaxBStages) bst = kCzMaxBStages;
    VPT_CHECK(bst >= 2, "vpt_conv3x3_zp: not enough shared memory for the weight pipeline (W=%d Cout=%d)", W, N);
    p.b_stages = bst;
    const size_t smem_bytes = fixed_bytes + (size_t)bst * b_stage_bytes;

    CUtensorMap tmA, tmB;
    {
        cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)p.Q};
        cuuint64_t strides[1] = {(cuuint64_t)C * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)p.a_box_rows};
        int r = make_tmap_bf16(&tmA, a->x, 2, dims, strides, box);
        if (r) return r;
    }
    {
        cuuint64_t dims[2] = {(cuuint64_t)9 * C, (cuuint64_t)N};
        cuuint64_t strides[1] = {(cuuint64_t)9 * C * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)p.block_n};
        int r = make_tmap_bf16(&tmB, a->w, 2, dims, strides, box);
        if (r) return r;
    }
    VPT_CHECK(!(a->mr && !a->S1 && !a->Ef), "vpt_conv3x3_zp: mr given without S1 (or Ef)");
    VPT_CHECK(!a->Ef || a->mr, "vpt_conv3x3_zp: Ef needs mr = (0, rstd) per frame");
    VPT_CHECK(!a->res_scale == !a->res_shift && (!a->res_scale || a->residual) && (!a->res_scale || N % 8 == 0),
              "vpt_conv3x3_zp: res_scale / res_shift come as a pair, with a residual, Cout %% 8 == 0");
    p.mr = a->mr; p.S1 = a->mr ? a->S1 : nullptr; p.S2 = a->S2; p.relu = a->relu;
    p.residual = reinterpret_cast<const __nv_bfloat16*>(a->residual);
    p.out = reinterpret_cast<__nv_bfloat16*>(a->out);
    p.stat_part = a->stat_part;
    p.Ef = a->Ef; p.res_scale = a->res_scale; p.res_shift = a->res_shift;
    p.dbg = g_cz_dbg;
    p.bo = g_dbg_bo > 0 ? 1 : 0;

    static bool attr_set = false;
    if (!attr_set) {
        VPT_CUDA(cudaFuncSetAttribute(conv3x3_zp_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        VPT_CUDA(cudaFuncSetAttribute(conv3x3_zp_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set = true;
    }
    const long long tiles = p.num_m_tiles * p.num_n_tiles;
    long long grid = num_sms();
    if (grid <= 0) grid = 132;
    if (grid > tiles) grid = tiles;
    if (p.block_n == 64)
        launch_k(conv3x3_zp_kernel<64>, dim3((unsigned)grid), dim3(kCzThreads), smem_bytes, (cudaStream_t)stream, tmA, tmB, p);
    else
        launch_k(conv3x3_zp_kernel<128>, dim3((unsigned)grid), dim3(kCzThreads), smem_bytes, (cudaStream_t)stream, tmA, tmB, p);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

// Kernel-variant knobs of the C ABI.  This build has one convolution kernel (no CTA-pair or operand-swapped variant), so only the
// epilogue experiment level (bits 4..7 of the pair mode, tools/conv_bench.py) has an effect; with swap mode 0 everywhere the
// swapped kernel's statistics layout never applies.
extern "C" int vpt_set_conv_pair_mode(int32_t on) {
    vpt::g_cz_dbg = (on & 0xff) >> 4;
    return VPT_OK;
}

extern "C" int vpt_set_conv_swap_mode(int32_t on) {
    (void)on;
    return VPT_OK;
}

extern "C" int64_t vpt_conv_zp_t_stat_floats(int32_t F, int32_t H, int32_t W, int32_t Cout) {
    (void)F; (void)H; (void)W; (void)Cout;
    return 0;
}

extern "C" int vpt_conv_zp_t_stats_finalize(const float* part, float* mr, int32_t F, int32_t H, int32_t W, float eps, void* stream) {
    (void)part; (void)mr; (void)F; (void)H; (void)W; (void)eps; (void)stream;
    vpt::set_error("vpt_conv_zp_t_stats_finalize: no convolution kernel of this build emits per-tile partials (vpt_conv_zp_t_stat_floats is 0)");
    return VPT_ERR_ARG;
}

extern "C" int vpt_conv_zp_stat_parts(int32_t F, int32_t H, int32_t W, int32_t Cout) {
    const long long Q = (long long)F * (H + 1) * (W + 1);
    int bn, nt;
    vpt::conv_zp_block_n(Q, Cout, &bn, &nt);
    return nt * 2;
}
