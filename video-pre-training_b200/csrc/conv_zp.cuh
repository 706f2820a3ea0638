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
//   warpgroups 0, 1 (warps 0..7): MMA + epilogue, ping-pong.  Each owns a whole 128-row x BN tile (one m64nBNk16 per 64-row
//       half and k16 step) and they take alternate tiles of the CTA's persistent sequence.  Named barriers let one warpgroup at a
//       time issue main-loop MMAs, so one warpgroup's epilogue runs while the other's main loop keeps the tensor pipe busy.  That
//       pair is the only synchronisation between the warpgroups: the epilogues share nothing, so both can run at once.  A span and
//       weight stages are released one MMA group late, so MMAs stay in flight across channel blocks and drain only at the end of
//       a tile.
//   warpgroup 2: warp 8 = A-span TMA producer, warp 9 = weight TMA producer (both in tile order), registers handed to the MMA
//       warpgroups with setmaxnreg.
// Epilogue = GroupNorm fold (border-class tables), ReLU, residual, bf16 store in ZP layout (border rows are written as
// zeros, which maintains the layout invariant), per-row (sum, sumsq) partials for the next layer's statistics.  One thread per
// row does the arithmetic.  The accumulators stay in registers through the epilogue; an epilogue warp takes the 32 rows its own
// fragment holds (rows 16w .. 16w+15 of each 64-row half) and passes them, 32 columns at a time, through a 32 x 32 fp32 block of
// shared memory that no other warp touches, so __syncwarp is all the epilogue needs.  The residual and the bf16 result pass
// through the same block so that global memory sees 64-byte row segments; a chunk's residual is loaded a chunk ahead (the first
// one while the tile's last MMAs drain).
#pragma once
#include "common.cuh"
#include "gemm_tc.cuh"

namespace vpt {

static int g_cz_dbg = 0;

constexpr int kCzThreads = 384;  // 3 warpgroups
constexpr int kCzMaxBStages = 8;
constexpr int kCzProducerRegs = 24, kCzMmaRegs = 240;  // setmaxnreg budget: 128 * 24 + 256 * 240 <= 64 K registers

// named barriers (0 is __syncthreads): kCzBarOrder + w = warpgroup w may issue its next main loop
constexpr int kCzBarOrder = 1;

// epilogue staging: one 32-row x 32-column fp32 block per MMA warp.  Pitch 36 floats = 144 B keeps rows 16-byte aligned and puts
// eight lanes reading consecutive rows on eight distinct 16-byte bank groups.
constexpr int kCzStgPitch = 36;
constexpr uint32_t kCzStgBytes = 8u * 32u * kCzStgPitch * 4u;

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

// One 64-row half of a tile over one k block (four k16 steps): m64nBNk16, one instruction per k16 step.
template <int BN>
__device__ __forceinline__ void cz_mma_k16(float (&acc)[BN / 2], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    if constexpr (BN == 128)
        wgmma_n128<0, 0>(acc, a_desc, b_desc, accumulate);
    else
        wgmma_n64<0, 0>(acc, a_desc, b_desc, accumulate);
}

// Chunk c (32 columns) of the calling warp's rows of both halves of a tile -> the warp's staging block, rows 0..15 from half 0 and
// 16..31 from half 1.  The switch turns the run-time chunk index into the constant register indices the fragment needs.
template <int BN>
__device__ __forceinline__ void cz_stage_chunk(const float (&frag)[2][BN / 2], int c, float* wrows) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float* blk = wrows + (size_t)h * 16 * kCzStgPitch;
        switch (c) {
            case 0: wgmma_frag_store_chunk<0>(frag[h], blk, kCzStgPitch); break;
            case 1: wgmma_frag_store_chunk<1>(frag[h], blk, kCzStgPitch); break;
            case 2: if constexpr (BN == 128) wgmma_frag_store_chunk<2>(frag[h], blk, kCzStgPitch); break;
            case 3: if constexpr (BN == 128) wgmma_frag_store_chunk<3>(frag[h], blk, kCzStgPitch); break;
        }
    }
}

template <int BN>
__global__ void __launch_bounds__(kCzThreads, 1)
conv3x3_zp_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const ConvZpParams p) {
    static_assert(BN == 64 || BN == 128, "BN is 64 or 128");
    pdl_sync();
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
    constexpr uint32_t b_stage_bytes = (uint32_t)BN * kBlockK * 2;
    uint8_t* smem_a = smem;                                        // 2 A-span stages
    uint8_t* smem_b = smem + 2 * (size_t)p.a_stage_bytes;          // b_stages weight tiles
    float* stg = reinterpret_cast<float*>(smem_b + (size_t)p.b_stages * b_stage_bytes);  // the MMA warps' staging blocks
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stg) + kCzStgBytes);
    uint64_t* a_full = bars;
    uint64_t* a_empty = bars + 2;
    uint64_t* b_full = bars + 4;
    uint64_t* b_empty = bars + 4 + kCzMaxBStages;

    const int warp = threadIdx.x >> 5;

    if (threadIdx.x == 8 * 32) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < 2; ++i) {
            mbar_init(&a_full[i], 1);
            mbar_init(&a_empty[i], 1);  // one consumer warpgroup per tile
        }
        for (int i = 0; i < p.b_stages; ++i) {
            mbar_init(&b_full[i], 1);
            mbar_init(&b_empty[i], 1);
        }
        fence_barrier_init();
    }
    __syncthreads();

    // 32-bit tile and row indices: the host keeps Q (and so every row and tile index) below 2^31
    const int num_tiles = (int)(p.num_m_tiles * p.num_n_tiles);
    const int tile_begin = (int)blockIdx.x;
    const int tile_step = (int)gridDim.x;
    const int halo = p.Wp + 1;  // rows before / after the tile that the taps reach

    if (warp >= 8) {
        setmaxnreg_dec<kCzProducerRegs>();
        if (threadIdx.x == 8 * 32) {
            // ================= A-span producer: one span per (tile, channel block), in tile order =================
            int stage = 0;
            uint32_t phase = 0;
            bool ok = true;
            for (int tile = tile_begin; tile < num_tiles && ok; tile += tile_step) {
                const int m_tile = tile / p.num_n_tiles;
                const int span0 = m_tile * kBlockM - halo;
                for (int cb = 0; cb < p.cin_blocks; ++cb) {
                    if (!(ok = mbar_wait(&a_empty[stage], phase ^ 1u, 0x110u))) break;
                    mbar_expect_tx(&a_full[stage], (uint32_t)p.a_stage_bytes);
                    uint8_t* sa = smem_a + (size_t)stage * p.a_stage_bytes;
                    for (int b = 0; b < p.a_boxes; ++b)
                        tma_load_2d(sa + (size_t)b * p.a_box_rows * 128, &tmA, &a_full[stage], cb * kBlockK, span0 + b * p.a_box_rows);
                    advance(stage, phase, 2);
                }
            }
        } else if (threadIdx.x == 9 * 32) {
            // ================= weight producer: one [BN][64] tile per (tile, channel block, tap) =================
            int stage = 0;
            uint32_t phase = 0;
            bool ok = true;
            for (int tile = tile_begin; tile < num_tiles && ok; tile += tile_step) {
                const int n0 = (tile % p.num_n_tiles) * BN;
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
        return;
    }

    // ================= MMA + epilogue: warpgroup wg owns the CTA's tiles 2i + wg of its sequence (ping-pong) =================
    setmaxnreg_inc<kCzMmaRegs>();
    const int wg = warp >> 2;
    const int lane = threadIdx.x & 31;
    // Epilogue rows follow the fragment: warp w of a warpgroup holds rows 16w .. 16w+15 of each 64-row half, and those 32 rows are
    // the ones it finishes.  Row i of the warp's staging block is tile row 64 * (i / 16) + 16w + i % 16; lane l works on row l.
    const int wrow0 = (warp & 3) * 16;
    float* wrows = stg + (size_t)warp * 32 * kCzStgPitch;
    float* my_row = wrows + (size_t)lane * kCzStgPitch;
    const int my_trow = ((lane >> 4) << 6) + wrow0 + (lane & 15);
    // the coalesced residual loads / result stores take four lanes per row, eight block rows per step, four steps
    const int seg = lane & 3;  // 16-byte piece of a 64-byte row segment
    const int seg_row0 = lane >> 2, seg_trow0 = wrow0 + seg_row0;
    const auto seg_row = [&](int k) { return seg_row0 + 8 * k; };                             // block row of step k
    const auto seg_trow = [&](int k) { return seg_trow0 + ((k >> 1) << 6) + ((k & 1) << 3); };  // and its tile row
    constexpr int nchunks = BN >> 5;
    constexpr int c_half = (nchunks + 1) >> 1;  // statistics partial 0 sums chunks [0, c_half), partial 1 the rest
    const int P = p.num_n_tiles * 2;
    // with N % 8 == 0 and 16-byte aligned bases, rows of the residual and of res_scale / res_shift are read as 16-byte vectors
    const bool res_vec = ((p.N & 7) == 0) && (((uintptr_t)p.residual | (uintptr_t)p.res_scale | (uintptr_t)p.res_shift) & 15) == 0;
    const int b_per_tile = 9 * p.cin_blocks;
    for (int s = wg; tile_begin + s * tile_step < num_tiles; s += 2) {
        const int tile = tile_begin + s * tile_step;
        const bool has_next = tile + tile_step < num_tiles;  // the other warpgroup has tile s + 1
        const int m_tile = tile / p.num_n_tiles;
        const int n_tile = tile % p.num_n_tiles;
        const int n0 = n_tile * BN;
        // this tile's place in the producers' FIFOs: both warpgroups consume them in tile order
        const long long a_it = (long long)s * p.cin_blocks, b_it = (long long)s * b_per_tile;
        int astage = (int)(a_it & 1), bstage = (int)(b_it % p.b_stages);
        uint32_t aphase = (uint32_t)((a_it >> 1) & 1), bphase = (uint32_t)((b_it / p.b_stages) & 1);

        // ---- main loop: 128 rows x BN channels over (channel block, tap); the other warpgroup's main loop goes first
        if (s > 0) named_bar_sync(kCzBarOrder + wg, 256);
        float frag[2][BN / 2];
        bool ok = true;
        int prev_b = -1, prev_a = -1;  // stages whose last MMA group is the one in flight: released after the next group's wait
        for (int cb = 0; cb < p.cin_blocks && ok; ++cb) {
            if (!(ok = mbar_wait(&a_full[astage], aphase, 0x310u))) break;
            const uint32_t a_base = smem_u32(smem_a + (size_t)astage * p.a_stage_bytes);
#pragma unroll 1
            for (int tap = 0; tap < 9; ++tap) {
                if (!(ok = mbar_wait(&b_full[bstage], bphase, 0x320u))) break;
                const uint32_t b_addr = smem_u32(smem_b + (size_t)bstage * b_stage_bytes);
                const int row_off = (tap / 3) * p.Wp + (tap % 3);  // (dy+1)*Wp + (dx+1)
                const uint32_t a_addr = a_base + (uint32_t)row_off * 128u;
                const uint64_t a_bo = p.bo ? ((uint64_t)((a_addr >> 7) & 7u) << 49) : 0ull;  // rows 64.. start 8 KB later: same phase
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kBlockK / 16; ++k) {
                    const uint32_t acc = (uint32_t)((cb | tap | k) != 0);
                    const uint64_t bd = gmma_desc_sw128(b_addr + k * 32);
                    cz_mma_k16<BN>(frag[0], gmma_desc_sw128(a_addr + k * 32) | a_bo, bd, acc);
                    cz_mma_k16<BN>(frag[1], gmma_desc_sw128(a_addr + 64u * 128u + k * 32) | a_bo, bd, acc);
                }
                wgmma_commit();
                wgmma_wait<1>();
                if ((threadIdx.x & 127) == 0) {
                    if (prev_b >= 0) mbar_arrive(&b_empty[prev_b]);
                    if (prev_a >= 0) mbar_arrive(&a_empty[prev_a]);
                }
                prev_a = -1;
                prev_b = bstage;
                advance(bstage, bphase, p.b_stages);
            }
            prev_a = astage;
            advance(astage, aphase, 2);
        }
        // every MMA of this tile is issued: the other warpgroup may start its main loop while these drain
        if (has_next) named_bar_arrive(kCzBarOrder + (wg ^ 1), 256);

        // ---- epilogue.  Full chunks of 32 columns move their global data through the warp's staging block: once every lane holds
        // its row's fp32 chunk in registers the block is free, so the residual comes in (bytes 0..63 of a row) and the bf16 result
        // goes out (bytes 64..127) as 64-byte row segments, four lanes per row, instead of one 16-byte piece per row and lane.
        // The residual is loaded into registers a chunk ahead, chunk 0's here while the MMAs drain.
        const int q0 = m_tile * kBlockM;
        const auto chunk_full = [&](int c) { return p.N - (n0 + c * 32) >= 32 && res_vec; };  // the same for every lane
        uint4 res_next[4];
        const auto res_load = [&](int c) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
                res_next[k] = q0 + seg_trow(k) < p.Q
                                  ? __ldg(reinterpret_cast<const uint4*>(p.residual + (size_t)(q0 + seg_trow(k)) * p.N + n0 + c * 32) + seg)
                                  : make_uint4(0u, 0u, 0u, 0u);
        };
        if (p.residual != nullptr && p.dbg != 2 && chunk_full(0)) res_load(0);

        wgmma_wait<0>();
#pragma unroll
        for (int h = 0; h < 2; ++h) wgmma_reg_fence(frag[h]);
        if ((threadIdx.x & 127) == 0) {
            if (prev_b >= 0) mbar_arrive(&b_empty[prev_b]);
            if (prev_a >= 0) mbar_arrive(&a_empty[prev_a]);
        }
        if (!ok) break;

        const int q = q0 + my_trow;
        const bool row_ok = q < p.Q;
        // decode the ZP row: frame, y, x
        const int f = q / p.FS;
        const int r = q - f * p.FS;
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
        float st_s0 = 0.f, st_ss0 = 0.f, st_s1 = 0.f, st_ss1 = 0.f;  // statistics partials of the two column groups

        // Chunks of 32 columns.  The arithmetic per element is the same on the full and the partial path.
#pragma unroll 1
        for (int c = 0; c < (p.dbg == 2 ? 0 : nchunks); ++c) {
            const int g = c < c_half ? 0 : 1;
            const int nb = n0 + c * 32;
            const int lim = min(32, p.N - nb);
            if (lim <= 0) break;
            const bool full = chunk_full(c);
            uint32_t acc[32];
            __syncwarp();  // the previous chunk has left the block
            cz_stage_chunk<BN>(frag, c, wrows);
            __syncwarp();
            stg_ld_32(my_row, acc);
            if (full) {
                __syncwarp();
                if (p.residual != nullptr) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if (q0 + seg_trow(k) < p.Q) reinterpret_cast<uint4*>(wrows + (size_t)seg_row(k) * kCzStgPitch)[seg] = res_next[k];
                    if (c + 1 < nchunks && chunk_full(c + 1)) res_load(c + 1);
                    __syncwarp();
                }
                if (row_ok) {
                    uint4* dst = reinterpret_cast<uint4*>(my_row + 16);
                    if (!interior) {  // zero row / column of the ZP layout
#pragma unroll
                        for (int o = 0; o < 4; ++o) dst[o] = make_uint4(0u, 0u, 0u, 0u);
                    } else {
                        float s_ = g ? st_s1 : st_s0, ss_ = g ? st_ss1 : st_ss0;
                        // eight columns at a time, from the table loads to the packed result: the other chunks' accumulators are
                        // live, so only a few loads can be in flight
#pragma unroll
                        for (int o = 0; o < 4; ++o) {
                            float v[8];
#pragma unroll
                            for (int h = 0; h < 2; ++h) {  // N % 8 == 0: the fold tables' rows are float4-aligned
                                const int qq = 2 * o + h;
                                float4 a1 = s1row ? __ldg(reinterpret_cast<const float4*>(s1row + nb) + qq) : make_float4(0, 0, 0, 0);
                                float4 a2 = s2row ? __ldg(reinterpret_cast<const float4*>(s2row + nb) + qq) : make_float4(0, 0, 0, 0);
                                v[4 * h + 0] = fmaf(ga, __uint_as_float(acc[4 * qq + 0]), fmaf(-gb, a1.x, a2.x));
                                v[4 * h + 1] = fmaf(ga, __uint_as_float(acc[4 * qq + 1]), fmaf(-gb, a1.y, a2.y));
                                v[4 * h + 2] = fmaf(ga, __uint_as_float(acc[4 * qq + 2]), fmaf(-gb, a1.z, a2.z));
                                v[4 * h + 3] = fmaf(ga, __uint_as_float(acc[4 * qq + 3]), fmaf(-gb, a1.w, a2.w));
                            }
                            if (p.relu == 1) {
#pragma unroll
                                for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.f);
                            }
                            if (p.residual != nullptr) {
                                const uint4 rr = reinterpret_cast<const uint4*>(my_row)[o];  // this row's residual, staged above
                                const float r8[8] = {bf16_lo(rr.x), bf16_hi(rr.x), bf16_lo(rr.y), bf16_hi(rr.y),
                                                     bf16_lo(rr.z), bf16_hi(rr.z), bf16_lo(rr.w), bf16_hi(rr.w)};
                                if (rarow) {
                                    const float4* ra4 = reinterpret_cast<const float4*>(rarow + nb) + 2 * o;
                                    const float4* rb4 = reinterpret_cast<const float4*>(rbrow + nb) + 2 * o;
                                    const float4 a0 = __ldg(ra4), a1 = __ldg(ra4 + 1), b0 = __ldg(rb4), b1 = __ldg(rb4 + 1);
                                    const float ra[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                                    const float rb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                                    for (int j = 0; j < 8; ++j) v[j] += fmaf(ra[j], r8[j], rb[j]);
                                } else {
#pragma unroll
                                    for (int j = 0; j < 8; ++j) v[j] += r8[j];
                                }
                            }
                            if (p.relu == 2) {
#pragma unroll
                                for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.f);
                            }
                            uint32_t pk[4];
#pragma unroll
                            for (int j = 0; j < 4; ++j) pk[j] = pack_bf16(v[2 * j], v[2 * j + 1]);
                            if (p.stat_part) {
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    const float lo = bf16_lo(pk[j]), hi = bf16_hi(pk[j]);
                                    s_ += lo; ss_ = fmaf(lo, lo, ss_);
                                    s_ += hi; ss_ = fmaf(hi, hi, ss_);
                                }
                            }
                            dst[o] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                        }
                        if (g) { st_s1 = s_; st_ss1 = ss_; } else { st_s0 = s_; st_ss0 = ss_; }
                    }
                }
                __syncwarp();
                if (p.dbg != 1) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if (q0 + seg_trow(k) < p.Q)
                            reinterpret_cast<uint4*>(p.out + (size_t)(q0 + seg_trow(k)) * p.N + nb)[seg] =
                                reinterpret_cast<const uint4*>(wrows + (size_t)seg_row(k) * kCzStgPitch + 16)[seg];
                }
                continue;
            }
            // ---- partial chunk (Cout not a multiple of the tile width / of 8): element by element, straight to global memory
            if (!row_ok) continue;
            float v[32];
            uint32_t pk[16];
            __nv_bfloat16* op = p.out + (size_t)q * p.N + nb;
            if (!interior) {
                for (int j = 0; j < lim; ++j) op[j] = __float2bfloat16_rn(0.f);
                continue;
            }
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                float a1 = 0.f, a2 = 0.f;
                if (j < lim) {
                    if (s1row) a1 = __ldg(s1row + nb + j);
                    if (s2row) a2 = __ldg(s2row + nb + j);
                }
                v[j] = fmaf(ga, __uint_as_float(acc[j]), fmaf(-gb, a1, a2));
            }
            if (p.relu == 1) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
            }
            if (p.residual != nullptr) {
                const __nv_bfloat16* rp = p.residual + (size_t)q * p.N + nb;
#pragma unroll
                for (int j = 0; j < 32; ++j)
                    if (j < lim) v[j] += rarow ? fmaf(__ldg(rarow + nb + j), __bfloat162float(rp[j]), __ldg(rbrow + nb + j)) : __bfloat162float(rp[j]);
            }
            if (p.relu == 2) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) pk[j] = pack_bf16(v[2 * j], v[2 * j + 1]);
            if (p.stat_part) {
                float s_ = g ? st_s1 : st_s0, ss_ = g ? st_ss1 : st_ss0;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const float lo = bf16_lo(pk[j]), hi = bf16_hi(pk[j]);
                    if (2 * j < lim) { s_ += lo; ss_ = fmaf(lo, lo, ss_); }
                    if (2 * j + 1 < lim) { s_ += hi; ss_ = fmaf(hi, hi, ss_); }
                }
                if (g) { st_s1 = s_; st_ss1 = ss_; } else { st_s0 = s_; st_ss0 = ss_; }
            }
            if (p.dbg != 1) {
#pragma unroll
                for (int j = 0; j < 32; ++j)
                    if (j < lim) op[j] = __float2bfloat16_rn(v[j]);
            }
        }
        if (p.stat_part && row_ok)
            reinterpret_cast<float4*>(p.stat_part)[((size_t)q * P + n_tile * 2) >> 1] = make_float4(st_s0, st_ss0, st_s1, st_ss1);
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

namespace vpt {
// plan_frames: the frame count whose launch plan (weight-tile width, hence the statistics partial layout) the call runs
static int conv3x3_zp_launch(const vpt_conv_zp_args* a, int plan_frames, void* stream) {
    VPT_CHECK(a && a->x && a->w && a->out, "vpt_conv3x3_zp: null operand");
    const int H = a->H, W = a->W, C = a->Cin, N = a->Cout;
    VPT_CHECK(a->F > 0 && H >= 2 && W >= 2 && C > 0 && C % 64 == 0 && N > 0 && N % 16 == 0,
              "vpt_conv3x3_zp: need F>0, H,W>=2, Cin %% 64 == 0, Cout %% 16 == 0 (F=%d H=%d W=%d Cin=%d Cout=%d)", a->F, H, W, C, N);
    // two stages of the 128 + 2*(W+2)-row input span, the warps' staging blocks and the weight stages share shared memory: up to
    // this width at least four 128-column weight stages fit
    VPT_CHECK(W <= 182, "vpt_conv3x3_zp: W=%d too wide (at most 182: two input spans of 128 + 2*(W+2) rows must fit in shared memory)", W);
    VPT_CHECK(((uintptr_t)a->x & 15) == 0 && ((uintptr_t)a->w & 15) == 0 && ((uintptr_t)a->out & 15) == 0, "vpt_conv3x3_zp: pointers must be 16-byte aligned");
    ConvZpParams p;
    memset(&p, 0, sizeof(p));
    p.H = H; p.W = W; p.Wp = W + 1; p.FS = (H + 1) * (W + 1);
    p.Q = (long long)a->F * p.FS;
    VPT_CHECK(p.Q <= 2147483647LL - kBlockM, "vpt_conv3x3_zp: too many rows for 32-bit row indices and TMA coordinates");
    p.N = N; p.cin = C; p.cin_blocks = C / 64;
    VPT_CHECK(plan_frames > 0, "vpt_conv3x3_zp_plan: plan_frames=%d must be > 0", plan_frames);
    conv_zp_block_n((long long)plan_frames * p.FS, N, &p.block_n, &p.num_n_tiles);
    p.num_m_tiles = (p.Q + kBlockM - 1) / kBlockM;
    const int span = kBlockM + 2 * (p.Wp + 1);
    p.a_boxes = (span + 255) / 256;
    p.a_box_rows = ((span + p.a_boxes - 1) / p.a_boxes + 7) / 8 * 8;
    VPT_CHECK(p.a_box_rows <= 256, "vpt_conv3x3_zp: span does not fit the TMA box limit");
    p.a_stage_bytes = p.a_boxes * p.a_box_rows * 128;
    const uint32_t b_stage_bytes = (uint32_t)p.block_n * kBlockK * 2;
    const size_t fixed_bytes = 1024 + 2 * (size_t)p.a_stage_bytes + kCzStgBytes + (4 + 2 * kCzMaxBStages) * 8;
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
}  // namespace vpt

extern "C" int vpt_conv3x3_zp(const vpt_conv_zp_args* a, void* stream) {
    return vpt::conv3x3_zp_launch(a, a ? a->F : 1, stream);
}

// The plan of `plan_frames` frames at any F: each output row (and its statistics partials) is computed as in a call of plan_frames frames.
extern "C" int vpt_conv3x3_zp_plan(const vpt_conv_zp_args* a, int32_t plan_frames, void* stream) {
    return vpt::conv3x3_zp_launch(a, plan_frames, stream);
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
