// Persistent, warp-specialised wgmma GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   warps 0..7 (two warpgroups): wgmma consumers -- warpgroup g owns rows 64g..64g+63 of the 128-row tile, accumulates them in
//                                registers, stages them through shared memory and runs the epilogue on them
//                                (norm-fold / bias / ReLU / residual -> bf16|fp32 store + statistics)
//   warp 8 (one lane)          : TMA producer -- A tile (128 rows x 64 bf16, 128B-swizzled) + B tile (block_n x 64)
//
// Convolution: the K loop runs over (tap, 64-channel block); the A tile of tap (dy,dx) is ONE 4-D TMA box of the raw
// NHWC activation tensor at pixel offset (dy,dx) -- TMA zero-fills out-of-image elements, which is exactly pad=1 --
// landing in shared memory as 128 pixel rows of 128 B, i.e. the canonical K-major SWIZZLE_128B wgmma operand.
// GroupNorm/LayerNorm on the input is folded into the epilogue (see include/vpt_b200.h).
#pragma once
#include "common.cuh"

namespace vpt {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kMaxBlockN = 128;      // wgmma accumulators of 64 x 128 per warpgroup: 64 fp32 registers per thread
constexpr int kNumEpiWarps = 8;
constexpr int kGemmThreads = 32 * kNumEpiWarps + 32;
constexpr int kMaxStages = 8;
constexpr uint32_t kStageBytesA = kBlockM * kBlockK * 2;
constexpr int kStgPitch = kMaxBlockN + 4;                       // fp32 staging row pitch (conflict-free 16-byte row reads)
constexpr uint32_t kStgBytes = 2u * 64u * kStgPitch * 4u;        // both warpgroups' 64-row staging tiles

struct GemmParams {
    int M, N, K;
    int block_n, num_m_tiles, num_n_tiles, k_iters, num_stages;
    int dbg_shift, dbg_bo;  // descriptor experiment: A rows loaded `dbg_shift` rows early, MMA start advanced to compensate
    int cluster;  // CTAs per cluster; they work on consecutive M tiles of one N tile and share the B tile by TMA multicast
    int conv, H, W, cin_blocks, px_per_frame;
    // epilogue
    const float* mr;
    int rows_per_group;
    const float* S1;
    const float* S2;
    int relu;
    float out_scale;
    const void* residual;
    int residual_f32;
    long long ld_res;
    void* out;
    int out_f32;
    long long ld_out;
    int seg_len;
    long long seg_stride, seg_off;
    float* stat_part;
    int stat_mode;
    // column segments with their own destination (fused projections); ndst == 0: the single destination above
    int ndst;
    int dst_n0[4];
    void* dst_out[4];
    long long dst_ld[4];
    int dst_f32[4];
    int dst_remap[4];
    // weight-gradient mode (kWgrad): out[split][m][tap*N + n] = sum over this split's K rows of A[k][m] * B[k + tap_shift[tap]][n]
    // (both operands MN-major: A is [K rows][M], B is [K rows][N] in memory)
    int ntaps, k_splits, k_iters_split;
    int tap_shift[9];
    long long split_stride;
};

__device__ __forceinline__ void advance(int& stage, uint32_t& phase, int num_stages) {
    if (++stage == num_stages) {
        stage = 0;
        phase ^= 1u;
    }
}

// One warpgroup's share of a 128 x BN tile: 64 rows x BN columns of the stage's operands, accumulated over one k block
// (four k16 steps) into `acc` as BN/64 fragments of 64 x 64.  A rows start at a_addr (K-major: 128-byte rows; MN-major: one
// {64 M, 64 K} box), B likewise; MN-major boxes of B are 8192 B apart.
template <bool kMN, int BN>
__device__ __forceinline__ void wg_mma_kblock(float (&acc)[BN / 64][32], uint32_t a_addr, uint32_t b_addr, uint64_t a_bo, bool accumulate) {
#pragma unroll
    for (int k = 0; k < kBlockK / 16; ++k) {
#pragma unroll
        for (int j = 0; j < BN / 64; ++j) {
            if (kMN)  // 16 K rows of 128 B per instruction
                wgmma_n64<1, 1>(acc[j], gmma_desc_sw128(a_addr + k * 2048, 8192u, 1024u), gmma_desc_sw128(b_addr + j * 8192 + k * 2048, 8192u, 1024u),
                                (uint32_t)(accumulate || k != 0));
            else
                wgmma_n64<0, 0>(acc[j], gmma_desc_sw128(a_addr + k * 32) | a_bo, gmma_desc_sw128(b_addr + j * 8192 + k * 32),
                                (uint32_t)(accumulate || k != 0));
        }
    }
}

// kWgrad: both operands are MN-major -- A = [K rows][M], B = [K rows][N] row-major activations (K = pixels / tokens), staged
// as TMA boxes of {64 columns, 64 K rows} -- the tile index additionally enumerates (K split, tap); tiles are
// [split][m_tile][tap][n_tile] and the B operand is read `tap_shift[tap]` rows further down (TMA zero-fills what falls outside
// the tensor, which is exactly the zero padding of a 3x3 convolution on the ZP layout).  cluster == 1 in this mode.
template <bool kWgrad, int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
    pdl_sync();
    extern __shared__ uint8_t smem_raw[];
    // carve: [A stages][B stages][staging][barriers]; operand tiles need 1024-byte alignment for SWIZZLE_128B
    const uint32_t raw = smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
    constexpr uint32_t stage_bytes_b = (uint32_t)BN * kBlockK * 2;
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + (size_t)p.num_stages * kStageBytesA;
    float* stg_all = reinterpret_cast<float*>(smem_b + (size_t)p.num_stages * stage_bytes_b);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stg_all) + kStgBytes);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + kMaxStages;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int CS = p.cluster;

    if (warp == kNumEpiWarps && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < p.num_stages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], (uint32_t)(2 * CS));  // one arrival per consumer warpgroup of every CTA of the cluster
        }
        fence_barrier_init();
    }
    __syncthreads();
    // peers must not multicast into / arrive on this CTA's barriers before they are initialised
    if (CS > 1) cluster_sync_all();

    const int cta_rank = CS > 1 ? (int)cluster_ctarank() : 0;
    const int cluster_id = blockIdx.x / CS, num_clusters = gridDim.x / CS;
    const uint16_t cmask = (uint16_t)((1u << CS) - 1u);
    // a "super tile" = CS consecutive M tiles of one N tile; CTA r of the cluster owns M tile group*CS + r
    const int tiles_mn = ((p.num_m_tiles + CS - 1) / CS) * p.num_n_tiles * (kWgrad ? p.ntaps : 1);
    const int num_super = tiles_mn * (kWgrad ? p.k_splits : 1);
    const int n_cols = kWgrad ? p.num_n_tiles * p.ntaps : p.num_n_tiles;  // tile columns (wgrad: [tap][n_tile])

    if (warp == kNumEpiWarps) {
        if (lane == 0) {
            // ================= TMA producer =================
            int stage = 0;
            uint32_t phase = 0;
            bool ok = true;
            const uint32_t slice_rows = (uint32_t)BN / CS, slice_bytes = stage_bytes_b / CS;
            for (int st = cluster_id; st < num_super && ok; st += num_clusters) {
                const int split = kWgrad ? st / tiles_mn : 0, sm = kWgrad ? st - split * tiles_mn : st;
                const int m_tile = (sm / n_cols) * CS + cta_rank, col = sm % n_cols;
                const int tap = kWgrad ? col / p.num_n_tiles : 0, n_tile = kWgrad ? col - tap * p.num_n_tiles : col;
                const int m0 = m_tile * kBlockM, n0 = n_tile * BN;
                int f0 = 0, y0 = 0;
                if (p.conv) {
                    f0 = m0 / p.px_per_frame;
                    y0 = (m0 % p.px_per_frame) / p.W;
                }
                const int it0 = kWgrad ? split * p.k_iters_split : 0;
                const int it1 = kWgrad ? min(p.k_iters, it0 + p.k_iters_split) : p.k_iters;
                const int bshift = kWgrad ? p.tap_shift[tap] : 0;
                for (int it = it0; it < it1; ++it) {
                    if (!(ok = mbar_wait(&empty_bar[stage], phase ^ 1u, 0x100u))) break;
                    mbar_expect_tx(&full_bar[stage], kStageBytesA + stage_bytes_b);
                    uint8_t* sa = smem_a + (size_t)stage * kStageBytesA;
                    uint8_t* sb = smem_b + (size_t)stage * stage_bytes_b;
                    if (kWgrad) {
                        tma_load_2d(sa, &tmA, &full_bar[stage], m0, it * kBlockK);
                        tma_load_2d(sa + 8192, &tmA, &full_bar[stage], m0 + 64, it * kBlockK);
#pragma unroll
                        for (int bx = 0; bx < BN / 64; ++bx)
                            tma_load_2d(sb + bx * 8192, &tmB, &full_bar[stage], n0 + bx * 64, it * kBlockK + bshift);
                        advance(stage, phase, p.num_stages);
                        continue;
                    }
                    if (p.conv) {
                        const int tap = it / p.cin_blocks, cb = it - tap * p.cin_blocks;
                        const int dy = tap / 3 - 1, dx = tap - (tap / 3) * 3 - 1;
                        tma_load_4d(sa, &tmA, &full_bar[stage], cb * kBlockK, dx, y0 + dy, f0);
                    } else {
                        tma_load_2d(sa, &tmA, &full_bar[stage], it * kBlockK, m0 - p.dbg_shift);
                    }
                    if (CS > 1)  // this CTA fetches 1/CS of the B tile and multicasts it to every CTA of the cluster
                        tma_load_2d_mc(sb + cta_rank * slice_bytes, &tmB, &full_bar[stage], it * kBlockK, n0 + cta_rank * slice_rows, cmask);
                    else
                        tma_load_2d(sb, &tmB, &full_bar[stage], it * kBlockK, n0);
                    advance(stage, phase, p.num_stages);
                }
            }
        }
    } else {
        // ================= wgmma + epilogue (warps 0..7) =================
        const int wg = warp >> 2;                     // warpgroup: rows 64*wg .. 64*wg+63 of the tile
        const int quarter = 2 * wg + (warp & 1);      // 32-row quarter this warp stores
        const int chalf = (warp >> 1) & 1;            // column half
        float* stg = stg_all + (size_t)wg * 64 * kStgPitch;
        const float* my_row = stg + (size_t)((warp & 1) * 32 + lane) * kStgPitch;
        const int nchunks = BN >> 5;
        const int c_begin = chalf == 0 ? 0 : (nchunks + 1) >> 1;
        const int c_end = chalf == 0 ? (nchunks + 1) >> 1 : nchunks;
        const int P = p.num_n_tiles * 2;
        const bool tab_vec = (p.conv == 0) || ((p.N & 3) == 0);
        const bool res_vec = ((p.ld_res & 7) == 0);
        int stage = 0;
        uint32_t phase = 0;
        bool ok = true;
        for (int st = cluster_id; st < num_super && ok; st += num_clusters) {
            const int split = kWgrad ? st / tiles_mn : 0, sm = kWgrad ? st - split * tiles_mn : st;
            const int m_tile = (sm / n_cols) * CS + cta_rank, col = sm % n_cols;
            const int tap = kWgrad ? col / p.num_n_tiles : 0, n_tile = kWgrad ? col - tap * p.num_n_tiles : col;
            const int m0 = m_tile * kBlockM, n0 = n_tile * BN;
            // ---- main loop: this warpgroup's 64 x BN accumulators
            float frag[BN / 64][32];
            int n_it = p.k_iters;
            if (kWgrad) {
                const int it0 = split * p.k_iters_split;
                n_it = min(p.k_iters, it0 + p.k_iters_split) - it0;
            }
            int prev = -1;
            for (int it = 0; it < n_it; ++it) {
                if (!(ok = mbar_wait(&full_bar[stage], phase, 0x300u))) break;
                const uint32_t a_addr = kWgrad ? smem_u32(smem_a + (size_t)stage * kStageBytesA) + (uint32_t)wg * 8192u
                                               : smem_u32(smem_a + (size_t)stage * kStageBytesA) + (uint32_t)(wg * 64 + p.dbg_shift) * 128u;
                const uint64_t a_bo = p.dbg_bo ? ((uint64_t)((a_addr >> 7) & 7u) << 49) : 0ull;
                const uint32_t b_addr = smem_u32(smem_b + (size_t)stage * stage_bytes_b);
                wgmma_fence();
                wg_mma_kblock<kWgrad, BN>(frag, a_addr, b_addr, a_bo, it != 0);
                wgmma_commit();
                wgmma_wait<1>();  // the previous k block's MMAs are done: its stage may be refilled
                if (prev >= 0 && (threadIdx.x & 127) == 0)
                    for (int r = 0; r < CS; ++r) mbar_arrive_cluster(&empty_bar[prev], (uint32_t)r);
                prev = stage;
                advance(stage, phase, p.num_stages);
            }
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) wgmma_reg_fence(frag[j]);
            if (prev >= 0 && (threadIdx.x & 127) == 0)
                for (int r = 0; r < CS; ++r) mbar_arrive_cluster(&empty_bar[prev], (uint32_t)r);
            if (!ok) break;
            // ---- accumulators -> row-major staging tile (the previous tile's epilogue has finished reading it)
            named_bar_sync(1 + wg, 128);
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) wgmma_frag_store(frag[j], stg, kStgPitch, j * 64);
            named_bar_sync(1 + wg, 128);

            const int m = m0 + quarter * 32 + lane;
            const bool row_ok = m < p.M;
            // per-row constants
            float ga = 1.f, gb = 0.f;
            if (p.mr != nullptr && row_ok) {
                const int g = m / p.rows_per_group;
                const float mean = __ldg(p.mr + 2 * g), rstd = __ldg(p.mr + 2 * g + 1);
                ga = rstd;
                gb = rstd * mean;
            }
            int cls = 0;
            if (p.conv) {
                const int pix = m % p.px_per_frame;
                const int y = pix / p.W, x = pix - y * p.W;
                const int cy = (y == 0) ? 0 : ((y == p.H - 1) ? 2 : 1);
                const int cx = (x == 0) ? 0 : ((x == p.W - 1) ? 2 : 1);
                cls = cy * 3 + cx;
            }
            const float* s1row = p.S1 ? p.S1 + (size_t)cls * p.N : nullptr;
            const float* s2row = p.S2 ? p.S2 + (size_t)cls * p.N : nullptr;
            // destination of this tile's columns (uniform per tile: segments start on tile boundaries)
            void* d_out = p.out;
            long long d_ld = p.ld_out;
            int d_f32 = p.out_f32, d_col0 = 0;
            bool d_remap = p.seg_len > 0;
            if (p.ndst > 0) {
                int sg = 0;
                for (int i = 1; i < p.ndst; ++i)
                    if (n0 >= p.dst_n0[i]) sg = i;
                d_out = p.dst_out[sg]; d_ld = p.dst_ld[sg]; d_f32 = p.dst_f32[sg]; d_col0 = p.dst_n0[sg];
                d_remap = d_remap && p.dst_remap[sg] != 0;
            }
            const bool d_vec = d_f32 ? ((d_ld & 3) == 0) : ((d_ld & 7) == 0);
            long long orow = m;
            if (d_remap) orow = (long long)(m / p.seg_len) * p.seg_stride + p.seg_off + (m % p.seg_len);
            float st_s = 0.f, st_ss = 0.f;

            for (int c = c_begin; c < c_end; ++c) {
                const int nb = n0 + c * 32;
                const int lim = min(32, min(BN - c * 32, p.N - nb));  // valid columns in this chunk
                if (!row_ok || lim <= 0) continue;
                uint32_t acc[32];
                stg_ld_32(my_row + c * 32, acc);
                float v[32];
                const bool full = (lim == 32);
                // ---- fold: v = ga*acc - gb*S1 + S2
                if (full && tab_vec) {
#pragma unroll
                    for (int q = 0; q < 8; ++q) {
                        float4 a1 = s1row ? __ldg(reinterpret_cast<const float4*>(s1row + nb) + q) : make_float4(0, 0, 0, 0);
                        float4 a2 = s2row ? __ldg(reinterpret_cast<const float4*>(s2row + nb) + q) : make_float4(0, 0, 0, 0);
                        v[4 * q + 0] = fmaf(ga, __uint_as_float(acc[4 * q + 0]), fmaf(-gb, a1.x, a2.x));
                        v[4 * q + 1] = fmaf(ga, __uint_as_float(acc[4 * q + 1]), fmaf(-gb, a1.y, a2.y));
                        v[4 * q + 2] = fmaf(ga, __uint_as_float(acc[4 * q + 2]), fmaf(-gb, a1.z, a2.z));
                        v[4 * q + 3] = fmaf(ga, __uint_as_float(acc[4 * q + 3]), fmaf(-gb, a1.w, a2.w));
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
                // ---- residual
                if (p.residual != nullptr) {
                    if (p.residual_f32) {
                        const float* rp = reinterpret_cast<const float*>(p.residual) + (size_t)m * p.ld_res + nb;
                        if (full && (p.ld_res & 3) == 0) {
#pragma unroll
                            for (int q = 0; q < 8; ++q) {
                                float4 r = __ldg(reinterpret_cast<const float4*>(rp) + q);
                                v[4 * q + 0] += r.x; v[4 * q + 1] += r.y; v[4 * q + 2] += r.z; v[4 * q + 3] += r.w;
                            }
                        } else {
#pragma unroll
                            for (int j = 0; j < 32; ++j)
                                if (j < lim) v[j] += __ldg(rp + j);
                        }
                    } else {
                        const __nv_bfloat16* rp = reinterpret_cast<const __nv_bfloat16*>(p.residual) + (size_t)m * p.ld_res + nb;
                        if (full && res_vec) {
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                uint4 r = __ldg(reinterpret_cast<const uint4*>(rp) + q);
                                v[8 * q + 0] += bf16_lo(r.x); v[8 * q + 1] += bf16_hi(r.x);
                                v[8 * q + 2] += bf16_lo(r.y); v[8 * q + 3] += bf16_hi(r.y);
                                v[8 * q + 4] += bf16_lo(r.z); v[8 * q + 5] += bf16_hi(r.z);
                                v[8 * q + 6] += bf16_lo(r.w); v[8 * q + 7] += bf16_hi(r.w);
                            }
                        } else {
#pragma unroll
                            for (int j = 0; j < 32; ++j)
                                if (j < lim) v[j] += __bfloat162float(rp[j]);
                        }
                    }
                }
                if (p.relu == 2) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
                }
                if (p.out_scale != 1.f) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) v[j] *= p.out_scale;
                }
                // ---- store (+ statistics of the stored values)
                if (d_f32) {
                    float* op = reinterpret_cast<float*>(d_out) + (size_t)orow * d_ld + (nb - d_col0);
                    if (kWgrad) op += (size_t)split * p.split_stride + (size_t)tap * p.N;
                    if (full && d_vec) {
#pragma unroll
                        for (int q = 0; q < 8; ++q)
                            reinterpret_cast<float4*>(op)[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            if (j < lim) op[j] = v[j];
                    }
                    if (p.stat_part) {
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            if (j < lim) {
                                st_s += v[j];
                                st_ss = fmaf(v[j], v[j], st_ss);
                            }
                    }
                } else {
                    __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(d_out) + (size_t)orow * d_ld + (nb - d_col0);
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
                    if (full && d_vec) {
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            reinterpret_cast<uint4*>(op)[q] = make_uint4(pk[4 * q], pk[4 * q + 1], pk[4 * q + 2], pk[4 * q + 3]);
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            if (j < lim) op[j] = __float2bfloat16_rn(v[j]);
                    }
                }
            }
            // statistics partials
            if (p.stat_part) {
                if (p.stat_mode == 1) {
                    if (row_ok)
                        reinterpret_cast<float2*>(p.stat_part)[(size_t)m * P + n_tile * 2 + chalf] = make_float2(st_s, st_ss);
                } else {
                    const float s = warp_sum(st_s), ss = warp_sum(st_ss);
                    const int g32 = (m0 + quarter * 32) >> 5;
                    if (lane == 0 && (m0 + quarter * 32) < p.M)
                        reinterpret_cast<float2*>(p.stat_part)[(size_t)g32 * P + n_tile * 2 + chalf] = make_float2(s, ss);
                }
            }
        }
    }

    // no CTA may exit while a peer can still multicast into its shared memory or arrive on its barriers
    if (CS > 1) cluster_sync_all();
}

// ------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (fn) return fn;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
        return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    return fn;
}

static int make_tmap_bf16(CUtensorMap* tm, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                          const cuuint32_t* box, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) {
        set_error("cuTensorMapEncodeTiled not available from the driver");
        return VPT_ERR_CUDA;
    }
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u)", (int)r, rank,
                  (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
        return VPT_ERR_CUDA;
    }
    return VPT_OK;
}

// N tile: 64 or 128 columns (the wgmma accumulators of a warpgroup hold 64 x block_n fp32 values)
static inline void choose_block_n(int N, int* block_n, int* n_tiles) {
    int nt = (N + kMaxBlockN - 1) / kMaxBlockN;
    int bn = (N + nt - 1) / nt;
    bn = bn <= 64 ? 64 : kMaxBlockN;
    *block_n = bn;
    *n_tiles = (N + bn - 1) / bn;
}

static int g_default_cluster = 1;
static int g_small_m_enabled = 1;
static int g_dbg_shift = 0, g_dbg_bo = 0;
static int g_num_sms = 0;
static int num_sms() {
    if (g_num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    return g_num_sms;
}

}  // namespace vpt

extern "C" int vpt_set_default_cluster(int32_t cs) {
    VPT_CHECK(cs == 1 || cs == 2 || cs == 4, "vpt_set_default_cluster: cluster size must be 1, 2 or 4");
    vpt::g_default_cluster = cs;
    return VPT_OK;
}

extern "C" int vpt_debug_set(int32_t shift, int32_t bo) {
    vpt::g_dbg_shift = shift;
    vpt::g_dbg_bo = bo;
    vpt::g_small_m_enabled = (shift == 0 && bo >= 0) ? 1 : 0;  // the descriptor experiment (and bo = -1) forces the tensor-core kernel
    return VPT_OK;
}

extern "C" int vpt_gemm_stat_parts(int32_t N) {
    int bn, nt;
    vpt::choose_block_n(N, &bn, &nt);
    return nt * 2;
}

namespace vpt {
int try_launch_gemv_small_fwd(const vpt_gemm_args* a, void* stream);
}

extern "C" int vpt_gemm_bf16(const vpt_gemm_args* a, void* stream) {
    using namespace vpt;
    VPT_CHECK(a != nullptr && a->A && a->B && a->out, "vpt_gemm_bf16: null operand");
    VPT_CHECK(a->M > 0 && a->N > 0 && a->K > 0, "vpt_gemm_bf16: bad shape M=%d N=%d K=%d", a->M, a->N, a->K);
    VPT_CHECK(a->K % 8 == 0, "vpt_gemm_bf16: K=%d must be a multiple of 8 (16-byte rows for TMA)", a->K);
    VPT_CHECK(((uintptr_t)a->A & 15) == 0 && ((uintptr_t)a->B & 15) == 0, "vpt_gemm_bf16: A/B must be 16-byte aligned");
    VPT_CHECK(a->mr == nullptr || a->rows_per_group > 0, "vpt_gemm_bf16: rows_per_group must be > 0 with mr");
    VPT_CHECK(a->stat_part == nullptr || a->stat_mode == 1 || a->stat_mode == 2, "vpt_gemm_bf16: bad stat_mode %d", a->stat_mode);
    VPT_CHECK(!(a->mr && !a->S1), "vpt_gemm_bf16: mr given without S1");
    if (g_small_m_enabled) {  // rollout path: a handful of rows -> weight-streaming kernel (csrc/gemv_small.cuh)
        const int r = try_launch_gemv_small_fwd(a, stream);
        if (r <= 0) return r;
    }
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = a->M; p.N = a->N; p.K = a->K;
    choose_block_n(a->N, &p.block_n, &p.num_n_tiles);
    if (a->ndst > 0) {  // segments start on N-tile boundaries: the largest tile width that divides every segment start
        int bn = kMaxBlockN;
        for (int i = 1; i < a->ndst && i < 4; ++i)
            if (a->dst_n0[i] % bn != 0) bn = 64;
        if (a->N <= 64) bn = 64;
        p.block_n = bn;
        p.num_n_tiles = (a->N + bn - 1) / bn;
    }
    p.num_m_tiles = (a->M + kBlockM - 1) / kBlockM;
    p.conv = a->conv;
    CUtensorMap tmA, tmB;
    if (a->conv) {
        const int H = a->H, W = a->W, C = a->Cin;
        VPT_CHECK(H >= 2 && W >= 2 && C > 0 && C % 64 == 0, "vpt_gemm_bf16(conv): need H,W >= 2 and Cin %% 64 == 0 (H=%d W=%d Cin=%d)", H, W, C);
        VPT_CHECK(a->K == 9 * C, "vpt_gemm_bf16(conv): K=%d != 9*Cin=%d", a->K, 9 * C);
        const int pxpf = H * W;
        VPT_CHECK(a->M % pxpf == 0, "vpt_gemm_bf16(conv): M=%d not a multiple of H*W=%d", a->M, pxpf);
        VPT_CHECK(128 % W == 0 && W <= 128, "vpt_gemm_bf16(conv): W=%d must divide 128", W);
        int tile_rows, tile_frames;
        if (pxpf >= 128) {
            VPT_CHECK(pxpf % 128 == 0, "vpt_gemm_bf16(conv): H*W=%d must be a multiple of 128", pxpf);
            tile_rows = 128 / W; tile_frames = 1;
        } else {
            VPT_CHECK(128 % pxpf == 0, "vpt_gemm_bf16(conv): H*W=%d must divide 128", pxpf);
            tile_rows = H; tile_frames = 128 / pxpf;
        }
        const cuuint64_t F = (cuuint64_t)(a->M / pxpf);
        cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, F};
        cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
        cuuint32_t box[4] = {64, (cuuint32_t)W, (cuuint32_t)tile_rows, (cuuint32_t)tile_frames};
        int r = make_tmap_bf16(&tmA, a->A, 4, dims, strides, box);
        if (r) return r;
        p.H = H; p.W = W; p.cin_blocks = C / 64; p.px_per_frame = pxpf;
        p.k_iters = 9 * p.cin_blocks;
    } else {
        cuuint64_t dims[2] = {(cuuint64_t)a->K, (cuuint64_t)a->M};
        cuuint64_t strides[1] = {(cuuint64_t)a->K * 2};
        cuuint32_t box[2] = {64, 128};
        int r = make_tmap_bf16(&tmA, a->A, 2, dims, strides, box);
        if (r) return r;
        p.k_iters = (a->K + kBlockK - 1) / kBlockK;
        p.px_per_frame = 1; p.W = 1; p.H = 1;
    }
    // cluster size: CTAs of a cluster share the B tile (TMA multicast), which cuts L2->SM operand traffic per FLOP
    int cs = a->cluster;
    if (cs == 0) cs = g_default_cluster;
    if (cs != 1 && cs != 2 && cs != 4) cs = 1;
    while (cs > 1 && (p.num_m_tiles < cs || p.block_n % (8 * cs) != 0)) cs >>= 1;
    p.cluster = cs;
    p.dbg_shift = g_dbg_shift; p.dbg_bo = g_dbg_bo;
    {
        cuuint64_t dims[2] = {(cuuint64_t)a->K, (cuuint64_t)a->N};
        cuuint64_t strides[1] = {(cuuint64_t)a->K * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)(p.block_n / cs)};
        int r = make_tmap_bf16(&tmB, a->B, 2, dims, strides, box);
        if (r) return r;
    }
    const uint32_t stage_bytes = kStageBytesA + (uint32_t)p.block_n * kBlockK * 2;
    const size_t fixed_bytes = 1024 + kStgBytes + 2 * kMaxStages * 8;
    int stages = (int)((227 * 1024 - fixed_bytes) / stage_bytes);
    if (stages > kMaxStages) stages = kMaxStages;
    p.num_stages = stages;
    const size_t smem_bytes = fixed_bytes + (size_t)stages * stage_bytes;
    p.mr = a->mr; p.rows_per_group = a->rows_per_group > 0 ? a->rows_per_group : 1;
    p.S1 = a->mr ? a->S1 : nullptr;
    p.S2 = a->S2;
    p.relu = a->relu; p.out_scale = a->out_scale;
    p.residual = a->residual; p.residual_f32 = a->residual_f32; p.ld_res = a->ld_res;
    p.out = a->out; p.out_f32 = a->out_f32; p.ld_out = a->ld_out;
    p.seg_len = a->seg_len; p.seg_stride = a->seg_stride; p.seg_off = a->seg_off;
    p.stat_part = a->stat_part; p.stat_mode = a->stat_mode;
    VPT_CHECK(!(a->mr && !a->S1), "vpt_gemm_bf16: mr given without S1");
    VPT_CHECK(a->ndst >= 0 && a->ndst <= 4, "vpt_gemm_bf16: ndst=%d not in 0..4", a->ndst);
    p.ndst = a->ndst;
    for (int i = 0; i < a->ndst; ++i) {
        VPT_CHECK(a->dst_out[i] != nullptr && a->dst_n0[i] % p.block_n == 0 && (i == 0 ? a->dst_n0[0] == 0 : a->dst_n0[i] > a->dst_n0[i - 1]),
                  "vpt_gemm_bf16: destination segment %d must start on an N-tile boundary (n0=%d, tile %d) in ascending order", i, a->dst_n0[i], p.block_n);
        p.dst_n0[i] = a->dst_n0[i]; p.dst_out[i] = a->dst_out[i]; p.dst_ld[i] = a->dst_ld[i]; p.dst_f32[i] = a->dst_f32[i]; p.dst_remap[i] = a->dst_remap[i];
    }
    VPT_CHECK(!(a->ndst > 0 && a->stat_part), "vpt_gemm_bf16: statistics partials are not supported with destination segments");

    static bool attr_set = false;
    if (!attr_set) {
        VPT_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<false, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        VPT_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<false, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set = true;
    }
    void (*kern)(const CUtensorMap, const CUtensorMap, const GemmParams) = p.block_n == 64 ? gemm_tc_kernel<false, 64> : gemm_tc_kernel<false, 128>;
    const int num_super = ((p.num_m_tiles + cs - 1) / cs) * p.num_n_tiles;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.blockDim = dim3(kGemmThreads);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[2];
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;  // (see pdl_sync() in common.cuh)
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    // persistent grid: as many clusters as can be co-resident (cluster size 4 strands some SMs of the uneven GPCs)
    static int max_clusters[2][5] = {{0, 0, 0, 0, 0}, {0, 0, 0, 0, 0}};
    int& mc = max_clusters[p.block_n == 64 ? 0 : 1][cs];
    if (mc == 0) {
        int n = 0;
        cfg.gridDim = dim3(num_sms() / cs * cs);
        cudaError_t e = cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
        if (e != cudaSuccess || n <= 0) {
            (void)cudaGetLastError();
            n = num_sms() / cs;
        }
        mc = n;
    }
    int clusters = mc;
    if (clusters > num_super) clusters = num_super;
    cfg.gridDim = dim3(clusters * cs);
    cfg.numAttrs = g_pdl ? 2 : 1;
    VPT_CUDA(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, p));
    return VPT_OK;
}

// ------------------------------------------------------------------------------------------------------
// weight gradients: dW[m][tap*N + n] = sum_k a[k][m] * b[k + shift[tap]][n]   (K = pixels / tokens, split over CTAs)
// ------------------------------------------------------------------------------------------------------
namespace vpt {

struct WgradPlan {
    int block_n, n_tiles, m_tiles, k_iters, splits, k_iters_split;
};

static WgradPlan wgrad_plan(int M, int N, int ntaps, long long R) {
    WgradPlan w;
    // whole 64-column TMA boxes, at most kMaxBlockN wide
    w.block_n = N <= 64 ? 64 : kMaxBlockN;
    w.n_tiles = (N + w.block_n - 1) / w.block_n;
    w.m_tiles = (M + kBlockM - 1) / kBlockM;
    w.k_iters = (int)((R + kBlockK - 1) / kBlockK);
    const int tiles = w.m_tiles * w.n_tiles * ntaps;
    int splits = (2 * num_sms() + tiles - 1) / tiles;  // ~2 work items per SM
    const int max_splits = w.k_iters / 8 > 0 ? w.k_iters / 8 : 1;  // at least 8 K iterations per item
    if (splits > max_splits) splits = max_splits;
    if (splits > 64) splits = 64;
    if (splits < 1) splits = 1;
    w.k_iters_split = (w.k_iters + splits - 1) / splits;
    w.splits = (w.k_iters + w.k_iters_split - 1) / w.k_iters_split;  // every split owns >= 1 iteration
    return w;
}

// out[i] = sum_s part[s][i] in a fixed order; 4 floats per thread
__global__ void __launch_bounds__(256) sum_splits_kernel(const float4* __restrict__ part, float4* __restrict__ out, long long n4, int splits) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 a = __ldg(part + i);
        for (int s = 1; s < splits; ++s) {
            const float4 b = __ldg(part + (long long)s * n4 + i);
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        out[i] = a;
    }
}

}  // namespace vpt

extern "C" int64_t vpt_wgrad_workspace_bytes(int32_t M, int32_t N, int32_t ntaps, int64_t R) {
    if (M <= 0 || N <= 0 || ntaps <= 0 || ntaps > 9 || R <= 0) return 0;
    const vpt::WgradPlan w = vpt::wgrad_plan(M, N, ntaps, R);
    const long long splits = w.splits;
    return splits > 1 ? (int64_t)splits * M * N * ntaps * 4 : 0;
}

extern "C" int vpt_wgrad_bf16(const void* a, int64_t lda, const void* b, int64_t ldb, int32_t M, int32_t N, int64_t R, const int32_t* shifts,
                              int32_t ntaps, float* out, void* workspace, int64_t workspace_bytes, void* stream) {
    using namespace vpt;
    VPT_CHECK(a && b && out && shifts, "vpt_wgrad_bf16: null operand");
    VPT_CHECK(M > 0 && N > 0 && R > 0 && ntaps >= 1 && ntaps <= 9, "vpt_wgrad_bf16: bad shape M=%d N=%d R=%lld ntaps=%d", M, N, (long long)R, ntaps);
    VPT_CHECK(M % 8 == 0 && N % 8 == 0 && lda % 8 == 0 && ldb % 8 == 0 && lda >= M && ldb >= N,
              "vpt_wgrad_bf16: M, N and the row strides must be multiples of 8 (M=%d N=%d lda=%lld ldb=%lld)", M, N, (long long)lda, (long long)ldb);
    VPT_CHECK(R < 2147483647LL - 4096, "vpt_wgrad_bf16: too many rows for 32-bit TMA coordinates");
    VPT_CHECK(((uintptr_t)a & 15) == 0 && ((uintptr_t)b & 15) == 0 && ((uintptr_t)out & 15) == 0, "vpt_wgrad_bf16: pointers must be 16-byte aligned");
    const WgradPlan w = wgrad_plan(M, N, ntaps, R);
    const long long out_elems = (long long)M * N * ntaps;
    VPT_CHECK(w.splits == 1 || (workspace && workspace_bytes >= (int64_t)w.splits * out_elems * 4),
              "vpt_wgrad_bf16: workspace too small (%lld bytes, need %lld)", (long long)workspace_bytes, (long long)w.splits * out_elems * 4);
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.N = N; p.K = (int)R;
    p.block_n = w.block_n; p.num_n_tiles = w.n_tiles; p.num_m_tiles = w.m_tiles;
    p.k_iters = w.k_iters; p.k_splits = w.splits; p.k_iters_split = w.k_iters_split;
    p.ntaps = ntaps;
    for (int i = 0; i < ntaps; ++i) p.tap_shift[i] = shifts[i];
    p.cluster = 1;
    p.px_per_frame = 1; p.W = 1; p.H = 1; p.rows_per_group = 1;
    p.out_scale = 1.f;
    p.out = w.splits > 1 ? workspace : (void*)out;
    p.out_f32 = 1;
    p.ld_out = (long long)N * ntaps;
    p.split_stride = out_elems;
    CUtensorMap tmA, tmB;
    {   // MN-major operands: the tensor map's inner dimension is the operand's M (N) index, its rows are K
        cuuint64_t dims[2] = {(cuuint64_t)M, (cuuint64_t)R};
        cuuint64_t strides[1] = {(cuuint64_t)lda * 2};
        cuuint32_t box[2] = {64, 64};
        int r = make_tmap_bf16(&tmA, a, 2, dims, strides, box);
        if (r) return r;
    }
    {
        cuuint64_t dims[2] = {(cuuint64_t)N, (cuuint64_t)R};
        cuuint64_t strides[1] = {(cuuint64_t)ldb * 2};
        cuuint32_t box[2] = {64, 64};
        int r = make_tmap_bf16(&tmB, b, 2, dims, strides, box);
        if (r) return r;
    }
    const uint32_t stage_bytes = kStageBytesA + (uint32_t)p.block_n * kBlockK * 2;
    const size_t fixed_bytes = 1024 + kStgBytes + 2 * kMaxStages * 8;
    int stages = (int)((227 * 1024 - fixed_bytes) / stage_bytes);
    if (stages > kMaxStages) stages = kMaxStages;
    p.num_stages = stages;
    const size_t smem_bytes = fixed_bytes + (size_t)stages * stage_bytes;
    static bool attr_set = false;
    if (!attr_set) {
        VPT_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<true, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        VPT_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<true, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set = true;
    }
    const int items = w.m_tiles * w.n_tiles * ntaps * w.splits;
    const int grid = items < num_sms() ? items : num_sms();
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kGemmThreads);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    VPT_CUDA(cudaLaunchKernelEx(&cfg, p.block_n == 64 ? gemm_tc_kernel<true, 64> : gemm_tc_kernel<true, 128>, tmA, tmB, p));
    if (w.splits > 1) {
        const long long n4 = out_elems / 4;
        long long blocks = (n4 + 255) / 256;
        if (blocks > 4096) blocks = 4096;
        sum_splits_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(workspace),
                                                                              reinterpret_cast<float4*>(out), n4, w.splits);
        VPT_LAUNCH_CHECK();
    }
    return VPT_OK;
}

// Weight-gradient kernel choice of the C ABI.  This build has one weight-gradient kernel (the MN-major mode of gemm_tc_kernel), so
// every mode selects it.
extern "C" int vpt_set_wgrad_mode(int32_t mode) {
    (void)mode;
    return VPT_OK;
}
