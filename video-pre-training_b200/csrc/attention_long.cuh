// Banded masked attention for KV memories longer than the kernels of attention.cuh / attention_bwd.cuh hold in shared memory
// (attention_memory_size 2048 -> maxlen 1920 is the reference's default).  Same semantics: query i (chunk-local) sees the keys
// j in (i, i + maxlen] of [memory | chunk], d = maxlen + i - j in [0, maxlen); memory row j only where state_mask[b][j] and not
// first[b][0]; logits q.k / 128 + R[i,:] . b_nd[:, d]; masked keys get no weight.  No shared memory here grows with maxlen.
//
//   forward        CTA = (64-query block, head, batch row), 4 warps x 16 queries, mma.sync m16n8k16 bf16 / fp32 accumulate over
//                  64-key tiles with an online softmax; the relative term is computed per tile from the queries' R rows (registers)
//                  and the 127 columns of b_nd the tile spans.  When the query blocks cannot fill the GPU (rollout: t = 1), a
//                  thread-block cluster of up to 8 CTAs splits the band; each keeps its partial (max, sum, output) in shared memory
//                  and CTA rank 0 combines them in rank order through distributed shared memory (no workspace, graph-capturable).
//   backward rows  16 queries per CTA, one warp per query, 64-key tiles of K / V staged: pass 1 writes each logit and dO.v to the
//                  P / dS workspace (indexed by d) and takes the max; pass 2 the softmax sums; pass 3 rewrites P and dS, and
//                  accumulates dR and dQ (K staged again).
//   backward keys  16 chunk keys per CTA, 64-query tiles of Q / dO staged: dK = dS^T Q / 128, dV = P^T dO (+ the state_out gradient).
//   backward mem   16 memory rows per CTA, 64-query tiles: dmem_K / dmem_V (+ the state_out gradient of the row when j >= t).
//   d b_nd         attn_bwd_bnd_kernel of attention_bwd.cuh (any maxlen, 64-bit indices).
// Every sum runs in a fixed order without atomics, so two identical calls give identical bits.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"
#include "attention.cuh"
#include "attention_bwd.cuh"

namespace vpt {

constexpr int kAlSplitMax = 8;                   // CTAs of a cluster sharing one query block's band (portable cluster size)
constexpr int kAlDist = 2 * kAttBK;              // b_nd columns staged per forward tile: 127 distances, padded to 128
constexpr int kAlNb = 10;                        // basis rows (nbasis <= 10)
constexpr int kAlPo = kAttD + 4;                 // fp32 pitch of the partial output staged for the cluster combine
constexpr int kAlKK = 64;                        // key offsets (rows kernel) / query offsets (keys, mem kernels) per staged tile
constexpr int kAlStage = kAlKK + kAbRows - 1;    // rows staged per tile: the tile's span over the CTA's 16 queries / keys

// RING: K / V / smask in the ring layout of attention.cuh (vpt_attention_ring), `off` read from ring_off[0] on the device, `rows` /
// `row_off` optional (vpt_attention_ring_rows)
template <bool RING>
__global__ void __launch_bounds__(kAttThreads) attention_long_kernel(
    const __nv_bfloat16* __restrict__ Q, const __nv_bfloat16* __restrict__ Kf, const __nv_bfloat16* __restrict__ Vf,
    const float* __restrict__ R, long long ld_r, const float* __restrict__ b_nd, const uint8_t* __restrict__ first,
    long long first_stride, const uint8_t* __restrict__ smask, __nv_bfloat16* __restrict__ out, int t, int maxlen, int heads,
    int nbasis, int nsplit, const int* __restrict__ ring_off, const int* __restrict__ rows, const int* __restrict__ row_off) {
    pdl_sync();
    extern __shared__ __align__(16) uint8_t al_smem[];
    __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(al_smem);
    __nv_bfloat16* Ks = Qs + kAttBQ * kAttPitch;
    __nv_bfloat16* Vs = Ks + kAttBK * kAttPitch;
    float* Bt = reinterpret_cast<float*>(Vs + kAttBK * kAttPitch);  // [kAlNb][kAlDist]: b_nd at d = dbase + c
    float* ML = Bt + kAlNb * kAlDist;                               // [64][2] partial (max, sum) for the cluster combine
    uint8_t* Ms = reinterpret_cast<uint8_t*>(ML + 2 * kAttBQ);      // [64] key of the tile usable?

    const int split = (int)(blockIdx.x % nsplit), qb = (int)(blockIdx.x / nsplit);  // cluster rank = split (cluster dims (nsplit,1,1))
    const int q0 = qb * kAttBQ, head = blockIdx.y, b = blockIdx.z;
    const int h = heads * kAttD;
    const int T = maxlen + t;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tg = lane & 3;
    int off = 0;
    const int rk = RING ? ring_row_of(b, rows, ring_off, row_off, maxlen, off) : b;  // row of K / V / smask
    if (RING && rk < 0) {  // inert padding row: every CTA of the cluster shares b, so all leave before the first cluster barrier
        if (split == 0) store_zero_rows(out, b, t, q0, h, head);
        return;
    }
    const long long kv_rows = RING ? maxlen : T;  // rows per batch row of K / V
    const __nv_bfloat16* Kb = Kf + (long long)rk * kv_rows * h;
    const __nv_bfloat16* Vb = Vf + (long long)rk * kv_rows * h;
    const bool mem_ok = (first[(long long)b * first_stride] == 0) && (smask != nullptr);

    load_tile_64x128(Qs, Q + (long long)b * t * h, h, q0, t, head * kAttD);
    const int iq[2] = {q0 + warp * 16 + g, q0 + warp * 16 + g + 8};
    float rr[2][kAlNb];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int n = 0; n < kAlNb; ++n)
            rr[r][n] = (n < nbasis && iq[r] < t) ? __ldg(R + ((long long)b * t + iq[r]) * ld_r + head * nbasis + n) : 0.f;
    cp_async_wait_all();
    __syncthreads();

    uint32_t qf[8][4];
    {
        const int row = warp * 16 + (lane & 15);
        const int colh = (lane >> 4) * 8;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks)
            ldsm_x4(smem_u32(Qs + row * kAttPitch + ks * 16 + colh), qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
    }

    float o[16][4];
#pragma unroll
    for (int n = 0; n < 16; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
    const float kLog2e = 1.4426950408889634f;
    const float qk_scale = 1.0f / (float)kAttD;  // muP 1/d (lib/xf.py:59)

    const int last_q = min(q0 + kAttBQ, t) - 1;
    const int j_lo = q0 + 1, j_hi = min(last_q + maxlen, T - 1);
    const int ntiles = (j_hi - j_lo + kAttBK) / kAttBK;
    const int per = (ntiles + nsplit - 1) / nsplit;
    const int tile_end = min(ntiles, (split + 1) * per);

    for (int tile = split * per; tile < tile_end; ++tile) {
        const int kb0 = j_lo + tile * kAttBK;
        __syncthreads();  // previous tile's K / V / Bt / Ms fully consumed
        if (RING) {
            load_tile_64x128_ring(Ks, Kb, h, kb0, T, head * kAttD, off, maxlen);
            load_tile_64x128_ring(Vs, Vb, h, kb0, T, head * kAttD, off, maxlen);
        } else {
            load_tile_64x128(Ks, Kb, h, kb0, T, head * kAttD);
            load_tile_64x128(Vs, Vb, h, kb0, T, head * kAttD);
        }
        const int dbase = maxlen + q0 - kb0 - (kAttBK - 1);  // distance of (query q0, key kb0 + 63)
        for (int x = threadIdx.x; x < kAlNb * kAlDist; x += kAttThreads) {
            const int n = x / kAlDist, c = x % kAlDist, d = dbase + c;
            Bt[x] = (n < nbasis && c < kAlDist - 1 && d >= 0 && d < maxlen) ? __ldg(b_nd + (long long)n * maxlen + d) : 0.f;
        }
        if (threadIdx.x < kAttBK) {
            const int j = kb0 + threadIdx.x;
            Ms[threadIdx.x] = (j >= maxlen) ? 1 : (mem_ok && smask[(long long)rk * maxlen + (RING ? ring_row(j, off, maxlen) : j)] != 0);
        }
        cp_async_wait_all();
        __syncthreads();

        float s[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                uint32_t b0, b1, b2, b3;
                const int krow = np * 16 + (lane & 7) + ((lane >> 4) << 3);
                const int kcol = ks * 16 + (((lane >> 3) & 1) << 3);
                ldsm_x4(smem_u32(Ks + krow * kAttPitch + kcol), b0, b1, b2, b3);
                mma_bf16_16816(s[2 * np], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], b0, b1);
                mma_bf16_16816(s[2 * np + 1], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], b2, b3);
            }
        }
        float bmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int n = 0; n < 8; ++n) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = e >> 1;
                const int i = iq[r];
                const int jl = n * 8 + 2 * tg + (e & 1);
                const int j = kb0 + jl;
                const int d = maxlen + i - j;
                bool ok = (i < t) && (j < T) && (d >= 0) && (d < maxlen);
                float extra = 0.f;
                if (ok) {
                    ok = Ms[jl] != 0;
                    const float* bt = Bt + (i - q0) - jl + (kAttBK - 1);
#pragma unroll
                    for (int nb = 0; nb < kAlNb; ++nb)
                        if (nb < nbasis) extra = fmaf(rr[r][nb], bt[nb * kAlDist], extra);
                }
                const float v = ok ? (s[n][e] * qk_scale + extra) * kLog2e : -INFINITY;
                s[n][e] = v;
                bmax[r] = fmaxf(bmax[r], v);
            }
        }
        float scale[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            float bm = bmax[r];
            bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 1));
            bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 2));
            const float m_new = fmaxf(mrow[r], bm);
            const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
            scale[r] = exp2f(mrow[r] - m_use);
            mrow[r] = m_new;
            float rs = 0.f;
#pragma unroll
            for (int n = 0; n < 8; ++n) {
                const float p0 = exp2f(s[n][2 * r] - m_use), p1 = exp2f(s[n][2 * r + 1] - m_use);
                s[n][2 * r] = p0;
                s[n][2 * r + 1] = p1;
                rs += p0 + p1;
            }
            rs += __shfl_xor_sync(0xffffffffu, rs, 1);
            rs += __shfl_xor_sync(0xffffffffu, rs, 2);
            lrow[r] = lrow[r] * scale[r] + rs;
        }
#pragma unroll
        for (int n = 0; n < 16; ++n) {
            o[n][0] *= scale[0]; o[n][1] *= scale[0];
            o[n][2] *= scale[1]; o[n][3] *= scale[1];
        }
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const uint32_t a0 = pack_bf16(s[2 * ks][0], s[2 * ks][1]);
            const uint32_t a1 = pack_bf16(s[2 * ks][2], s[2 * ks][3]);
            const uint32_t a2 = pack_bf16(s[2 * ks + 1][0], s[2 * ks + 1][1]);
            const uint32_t a3 = pack_bf16(s[2 * ks + 1][2], s[2 * ks + 1][3]);
#pragma unroll
            for (int np = 0; np < 8; ++np) {
                uint32_t b0, b1, b2, b3;
                const int vrow = ks * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
                const int vcol = np * 16 + ((lane >> 4) << 3);
                ldsm_x4_t(smem_u32(Vs + vrow * kAttPitch + vcol), b0, b1, b2, b3);
                mma_bf16_16816(o[2 * np], a0, a1, a2, a3, b0, b1);
                mma_bf16_16816(o[2 * np + 1], a0, a1, a2, a3, b2, b3);
            }
        }
    }

    if (nsplit == 1) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int i = iq[r];
            if (i >= t) continue;
            const float inv = 1.0f / lrow[r];
            __nv_bfloat16* op = out + ((long long)b * t + i) * h + head * kAttD;
#pragma unroll
            for (int n = 0; n < 16; ++n)
                *reinterpret_cast<uint32_t*>(op + n * 8 + 2 * tg) = pack_bf16(o[n][2 * r] * inv, o[n][2 * r + 1] * inv);
        }
        return;
    }
    // cluster combine: every CTA stages its unnormalised partial (max, sum, output); rank 0 merges ranks 0..nsplit-1 in order
    __syncthreads();  // K / V tiles consumed: the partial output reuses them
    float* Po = reinterpret_cast<float*>(Ks);  // [64][kAlPo]
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = warp * 16 + g + 8 * r;
#pragma unroll
        for (int n = 0; n < 16; ++n) {
            Po[row * kAlPo + n * 8 + 2 * tg] = o[n][2 * r];
            Po[row * kAlPo + n * 8 + 2 * tg + 1] = o[n][2 * r + 1];
        }
        if (tg == 0) {
            ML[2 * row] = mrow[r];
            ML[2 * row + 1] = lrow[r];
        }
    }
    cluster_sync_all();
    if (split == 0) {
        namespace cg = cooperative_groups;
        cg::cluster_group cl = cg::this_cluster();
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int i = iq[r];
            const int row = warp * 16 + g + 8 * r;
            float m = -INFINITY;
            for (int k = 0; k < nsplit; ++k) m = fmaxf(m, cl.map_shared_rank(ML, k)[2 * row]);
            const float m_use = (m == -INFINITY) ? 0.f : m;
            float l = 0.f, acc[16][2];
#pragma unroll
            for (int n = 0; n < 16; ++n) acc[n][0] = acc[n][1] = 0.f;
            for (int k = 0; k < nsplit; ++k) {
                const float* ml = cl.map_shared_rank(ML, k);
                const float* po = cl.map_shared_rank(Po, k) + row * kAlPo + 2 * tg;
                const float sc = exp2f(ml[2 * row] - m_use);
                l = fmaf(ml[2 * row + 1], sc, l);
#pragma unroll
                for (int n = 0; n < 16; ++n) {
                    const float2 v = *reinterpret_cast<const float2*>(po + n * 8);
                    acc[n][0] = fmaf(v.x, sc, acc[n][0]);
                    acc[n][1] = fmaf(v.y, sc, acc[n][1]);
                }
            }
            if (i < t) {
                const float inv = 1.0f / l;
                __nv_bfloat16* op = out + ((long long)b * t + i) * h + head * kAttD;
#pragma unroll
                for (int n = 0; n < 16; ++n) *reinterpret_cast<uint32_t*>(op + n * 8 + 2 * tg) = pack_bf16(acc[n][0] * inv, acc[n][1] * inv);
            }
        }
    }
    cluster_sync_all();  // no CTA leaves while rank 0 still reads its shared memory
}

// ---------------------------------------------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kAbThreads) attn_bwd_rows_long_kernel(
    const __nv_bfloat16* __restrict__ Q, const __nv_bfloat16* __restrict__ Kf, const __nv_bfloat16* __restrict__ Vf, const float* __restrict__ R,
    long long ld_r, const float* __restrict__ b_nd, const uint8_t* __restrict__ first, long long first_stride, const uint8_t* __restrict__ smask,
    const __nv_bfloat16* __restrict__ dO, __nv_bfloat16* __restrict__ out, long long ld_out, float* __restrict__ wsP, float* __restrict__ wsS, int t,
    int maxlen, int heads, int nbasis) {
    extern __shared__ __align__(16) uint8_t al_smem[];
    __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(al_smem);   // [kAlStage][pitch]: keys i0 + 1 + kk0 + r
    __nv_bfloat16* Vs = Ks + kAlStage * kAbPitch;
    __nv_bfloat16* Qs = Vs + kAlStage * kAbPitch;                    // [16][pitch]
    __nv_bfloat16* Os = Qs + kAbRows * kAbPitch;                     // dO rows
    float* Bt = reinterpret_cast<float*>(Os + kAbRows * kAbPitch);  // [kAlNb][kAlKK]: b_nd at d = maxlen - 1 - (kk0 + c)
    float* Ss = Bt + kAlNb * kAlKK;                                 // [16][kAlKK] dS of each warp's query over the tile
    uint8_t* Ms = reinterpret_cast<uint8_t*>(Ss + kAbRows * kAlKK);  // [kAlStage] staged key usable?

    const int i0 = blockIdx.x * kAbRows, head = blockIdx.y, b = blockIdx.z;
    const int h = heads * kAbD, T = maxlen + t;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const __nv_bfloat16* Kb = Kf + (long long)b * T * h;
    const __nv_bfloat16* Vb = Vf + (long long)b * T * h;
    stage_rows(Qs, Q + (long long)b * t * h, h, i0, kAbRows, t, head * kAbD);
    stage_rows(Os, dO + (long long)b * t * h, h, i0, kAbRows, t, head * kAbD);
    const bool mem_ok = (first[(long long)b * first_stride] == 0) && (smask != nullptr);
    const int i = i0 + warp;
    const bool active = i < t;  // whole warps; every warp still takes part in the block-wide barriers
    const long long row = (long long)b * t + i;
    float rr[kAlNb];
#pragma unroll
    for (int n = 0; n < kAlNb; ++n) rr[n] = (active && n < nbasis) ? __ldg(R + row * ld_r + head * nbasis + n) : 0.f;
    const long long wbase = (((long long)b * heads + head) * t + i) * maxlen;
    const __nv_bfloat16* qrow = Qs + warp * kAbPitch;
    const __nv_bfloat16* orow = Os + warp * kAbPitch;

    auto stage_tile = [&](int kk0, bool with_v) {
        __syncthreads();  // the previous tile is consumed
        stage_rows(Ks, Kb, h, i0 + 1 + kk0, kAlStage, T, head * kAbD);
        if (with_v) stage_rows(Vs, Vb, h, i0 + 1 + kk0, kAlStage, T, head * kAbD);
        for (int x = threadIdx.x; x < kAlNb * kAlKK; x += blockDim.x) {
            const int n = x / kAlKK, kk = kk0 + x % kAlKK;
            Bt[x] = (n < nbasis && kk < maxlen) ? __ldg(b_nd + (long long)n * maxlen + (maxlen - 1 - kk)) : 0.f;
        }
        for (int x = threadIdx.x; x < kAlStage; x += blockDim.x) {
            const int j = i0 + 1 + kk0 + x;
            Ms[x] = (j >= maxlen) ? 1 : (mem_ok && smask[(long long)b * maxlen + j] != 0);
        }
        __syncthreads();
    };

    // ---- pass 1: logit (-inf where masked) -> wsP, dP = dO . v -> wsS, and the row max.  Lane owns kk = kk0 + lane + 32 k.
    float mx = -INFINITY;
    for (int kk0 = 0; kk0 < maxlen; kk0 += kAlKK) {
        stage_tile(kk0, true);
        if (!active) continue;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int c = lane + 32 * k, kk = kk0 + c;
            if (kk >= maxlen) continue;
            const __nv_bfloat16* krow = Ks + (size_t)(warp + c) * kAbPitch;  // key j = i + 1 + kk
            const __nv_bfloat16* vrow = Vs + (size_t)(warp + c) * kAbPitch;
            float qk = 0.f, ov = 0.f;
#pragma unroll 4
            for (int cc = 0; cc < 16; ++cc) {
                qk += dot8(*reinterpret_cast<const uint4*>(qrow + cc * 8), *reinterpret_cast<const uint4*>(krow + cc * 8));
                ov += dot8(*reinterpret_cast<const uint4*>(orow + cc * 8), *reinterpret_cast<const uint4*>(vrow + cc * 8));
            }
            float extra = 0.f;
#pragma unroll
            for (int n = 0; n < kAlNb; ++n)
                if (n < nbasis) extra = fmaf(rr[n], Bt[n * kAlKK + c], extra);
            const float sv = Ms[warp + c] ? qk * (1.0f / (float)kAbD) + extra : -INFINITY;
            mx = fmaxf(mx, sv);
            const int d = maxlen - 1 - kk;
            wsP[wbase + d] = sv;
            wsS[wbase + d] = ov;
        }
    }
    mx = warp_max(mx);
    // ---- pass 2: the softmax denominator and delta = sum P dP (each lane re-reads what it wrote)
    float den = 0.f, num = 0.f;
    if (active) {
        for (int kk = lane; kk < maxlen; kk += 32) {
            const int d = maxlen - 1 - kk;
            const float e = __expf(wsP[wbase + d] - mx);  // 0 for a masked key; the key at d = 0 is always visible, so den > 0
            den += e;
            num = fmaf(e, wsS[wbase + d], num);
        }
    }
    den = warp_sum(den);
    num = warp_sum(num);
    const float inv = 1.f / den;
    const float delta = num * inv;
    // ---- pass 3: P, dS -> workspace; dR = dS b_nd^T; dQ = dS K / 128
    float dr[kAlNb];
#pragma unroll
    for (int n = 0; n < kAlNb; ++n) dr[n] = 0.f;
    float dq[4] = {0.f, 0.f, 0.f, 0.f};
    float* srow = Ss + warp * kAlKK;
    for (int kk0 = 0; kk0 < maxlen; kk0 += kAlKK) {
        stage_tile(kk0, false);
        if (!active) continue;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int c = lane + 32 * k, kk = kk0 + c;
            float ds = 0.f;
            if (kk < maxlen) {
                const int d = maxlen - 1 - kk;
                const float p = __expf(wsP[wbase + d] - mx) * inv;
                ds = p * (wsS[wbase + d] - delta);
                wsP[wbase + d] = p;
                wsS[wbase + d] = ds;
#pragma unroll
                for (int n = 0; n < kAlNb; ++n)
                    if (n < nbasis) dr[n] = fmaf(ds, Bt[n * kAlKK + c], dr[n]);
            }
            srow[c] = ds;
        }
        __syncwarp();
        const int nk = min(kAlKK, maxlen - kk0);
        for (int c = 0; c < nk; ++c) {
            const float ds = srow[c];
            const uint2 kv = *reinterpret_cast<const uint2*>(Ks + (size_t)(warp + c) * kAbPitch + lane * 4);
            dq[0] = fmaf(ds, bf16_lo(kv.x), dq[0]);
            dq[1] = fmaf(ds, bf16_hi(kv.x), dq[1]);
            dq[2] = fmaf(ds, bf16_lo(kv.y), dq[2]);
            dq[3] = fmaf(ds, bf16_hi(kv.y), dq[3]);
        }
    }
    if (!active) return;
#pragma unroll
    for (int n = 0; n < kAlNb; ++n) {
        if (n < nbasis) {
            const float v = warp_sum(dr[n]);
            if (lane == 0) out[row * ld_out + 3 * h + head * nbasis + n] = __float2bfloat16_rn(v);
        }
    }
    const float sc = 1.0f / (float)kAbD;
    uint2 o2;
    o2.x = pack_bf16(dq[0] * sc, dq[1] * sc);
    o2.y = pack_bf16(dq[2] * sc, dq[3] * sc);
    *reinterpret_cast<uint2*>(out + row * ld_out + head * kAbD + lane * 4) = o2;
}

// dk / dv += over the 32 staged queries [sub, sub + 32) of the tile, for the lane's 4 dims; p / ds are this lane's workspace values
__device__ __forceinline__ void al_accum32(float (&dk)[4], float (&dv)[4], const __nv_bfloat16* Qs, const __nv_bfloat16* Os, int r0, int n, float p,
                                           float ds, int lane) {
    for (int q = 0; q < n; ++q) {
        const float pp = __shfl_sync(0xffffffffu, p, q), ss = __shfl_sync(0xffffffffu, ds, q);
        const uint2 qv = *reinterpret_cast<const uint2*>(Qs + (size_t)(r0 + q) * kAbPitch + lane * 4);
        const uint2 ov = *reinterpret_cast<const uint2*>(Os + (size_t)(r0 + q) * kAbPitch + lane * 4);
        dk[0] = fmaf(ss, bf16_lo(qv.x), dk[0]); dk[1] = fmaf(ss, bf16_hi(qv.x), dk[1]);
        dk[2] = fmaf(ss, bf16_lo(qv.y), dk[2]); dk[3] = fmaf(ss, bf16_hi(qv.y), dk[3]);
        dv[0] = fmaf(pp, bf16_lo(ov.x), dv[0]); dv[1] = fmaf(pp, bf16_hi(ov.x), dv[1]);
        dv[2] = fmaf(pp, bf16_lo(ov.y), dv[2]); dv[3] = fmaf(pp, bf16_hi(ov.y), dv[3]);
    }
}

// chunk key jc is attended by the queries i = jc + dd, dd in [0, maxlen), i < t
__global__ void __launch_bounds__(kAbThreads) attn_bwd_keys_long_kernel(const __nv_bfloat16* __restrict__ Q, const __nv_bfloat16* __restrict__ dO,
                                                                         const float* __restrict__ wsP, const float* __restrict__ wsS,
                                                                         const float* __restrict__ dsk, const float* __restrict__ dsv,
                                                                         __nv_bfloat16* __restrict__ out, long long ld_out, int t, int maxlen, int heads) {
    extern __shared__ __align__(16) uint8_t al_smem[];
    __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(al_smem);  // [kAlStage][pitch]: queries jc0 + dd0 + r
    __nv_bfloat16* Os = Qs + kAlStage * kAbPitch;
    const int jc0 = blockIdx.x * kAbRows, head = blockIdx.y, b = blockIdx.z;
    const int h = heads * kAbD;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int jc = jc0 + warp;
    const bool active = jc < t;
    const long long bh = (long long)b * heads + head;
    float dk[4] = {0.f, 0.f, 0.f, 0.f}, dv[4] = {0.f, 0.f, 0.f, 0.f};
    const int dmax = min(maxlen, t - jc0);  // offsets any key of the CTA needs
    for (int dd0 = 0; dd0 < dmax; dd0 += kAlKK) {
        __syncthreads();
        stage_rows(Qs, Q + (long long)b * t * h, h, jc0 + dd0, kAlStage, t, head * kAbD);
        stage_rows(Os, dO + (long long)b * t * h, h, jc0 + dd0, kAlStage, t, head * kAbD);
        __syncthreads();
        if (!active) continue;
        for (int sub = 0; sub < kAlKK; sub += 32) {
            const int n = min(32, min(maxlen, t - jc) - (dd0 + sub));
            if (n <= 0) break;
            const int dl = dd0 + sub + lane;
            float p = 0.f, ds = 0.f;
            if (lane < n) {
                const long long w = (bh * t + jc + dl) * maxlen + dl;
                p = __ldg(wsP + w);
                ds = __ldg(wsS + w);
            }
            al_accum32(dk, dv, Qs, Os, warp + sub, n, p, ds, lane);  // staged row of query jc + dd0 + sub + q
        }
    }
    if (!active) return;
    const float sc = 1.0f / (float)kAbD;
#pragma unroll
    for (int c = 0; c < 4; ++c) dk[c] *= sc;
    const int r = jc + maxlen - t;  // this key's row of state_out (when >= 0)
    if (r >= 0) {
        const long long so = ((long long)b * maxlen + r) * h + head * kAbD + lane * 4;
        if (dsk != nullptr) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(dsk + so));
            dk[0] += g.x; dk[1] += g.y; dk[2] += g.z; dk[3] += g.w;
        }
        if (dsv != nullptr) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(dsv + so));
            dv[0] += g.x; dv[1] += g.y; dv[2] += g.z; dv[3] += g.w;
        }
    }
    const long long row = (long long)b * t + jc;
    uint2 o2;
    o2.x = pack_bf16(dk[0], dk[1]);
    o2.y = pack_bf16(dk[2], dk[3]);
    *reinterpret_cast<uint2*>(out + row * ld_out + h + head * kAbD + lane * 4) = o2;
    o2.x = pack_bf16(dv[0], dv[1]);
    o2.y = pack_bf16(dv[2], dv[3]);
    *reinterpret_cast<uint2*>(out + row * ld_out + 2 * h + head * kAbD + lane * 4) = o2;
}

// memory row j < maxlen is seen by the queries i in [0, min(j, t)) at d = maxlen + i - j where the row is visible (as attn_bwd_mem_kernel,
// with the queries staged 64 at a time)
__global__ void __launch_bounds__(kAbThreads) attn_bwd_mem_long_kernel(const __nv_bfloat16* __restrict__ Q, const __nv_bfloat16* __restrict__ dO,
                                                                        const float* __restrict__ wsP, const float* __restrict__ wsS,
                                                                        const uint8_t* __restrict__ first, long long first_stride,
                                                                        const uint8_t* __restrict__ smask, const float* __restrict__ dsk,
                                                                        const float* __restrict__ dsv, float* __restrict__ dmem_k,
                                                                        float* __restrict__ dmem_v, int t, int maxlen, int heads) {
    extern __shared__ __align__(16) uint8_t al_smem[];
    __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(al_smem);  // [kAlKK][pitch]: queries q0 + r
    __nv_bfloat16* Os = Qs + kAlKK * kAbPitch;
    const int j0 = blockIdx.x * kAbRows, head = blockIdx.y, b = blockIdx.z;
    const int h = heads * kAbD;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool mem_ok = (first[(long long)b * first_stride] == 0) && (smask != nullptr);
    const int nq = mem_ok ? min(t, min(j0 + kAbRows, maxlen) - 1) : 0;  // queries any row of this CTA is seen by
    const int j = j0 + warp;
    const bool active = j < maxlen;
    const int ni = (active && mem_ok && smask[(long long)b * maxlen + j] != 0) ? min(j, t) : 0;
    const long long bh = (long long)b * heads + head;
    float dk[4] = {0.f, 0.f, 0.f, 0.f}, dv[4] = {0.f, 0.f, 0.f, 0.f};
    for (int q0 = 0; q0 < nq; q0 += kAlKK) {
        __syncthreads();
        stage_rows(Qs, Q + (long long)b * t * h, h, q0, kAlKK, t, head * kAbD);
        stage_rows(Os, dO + (long long)b * t * h, h, q0, kAlKK, t, head * kAbD);
        __syncthreads();
        for (int sub = 0; sub < kAlKK; sub += 32) {
            const int n = min(32, ni - (q0 + sub));
            if (n <= 0) break;
            const int il = q0 + sub + lane;
            float p = 0.f, ds = 0.f;
            if (lane < n) {
                const long long w = (bh * t + il) * maxlen + (maxlen + il - j);
                p = __ldg(wsP + w);
                ds = __ldg(wsS + w);
            }
            al_accum32(dk, dv, Qs, Os, sub, n, p, ds, lane);
        }
    }
    if (!active) return;
    const float sc = 1.0f / (float)kAbD;
#pragma unroll
    for (int c = 0; c < 4; ++c) dk[c] *= sc;
    if (j >= t) {  // memory row j is row j - t of state_out (t < maxlen)
        const long long so = ((long long)b * maxlen + (j - t)) * h + head * kAbD + lane * 4;
        if (dsk != nullptr) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(dsk + so));
            dk[0] += g.x; dk[1] += g.y; dk[2] += g.z; dk[3] += g.w;
        }
        if (dsv != nullptr) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(dsv + so));
            dv[0] += g.x; dv[1] += g.y; dv[2] += g.z; dv[3] += g.w;
        }
    }
    const long long o = ((long long)b * maxlen + j) * h + head * kAbD + lane * 4;
    *reinterpret_cast<float4*>(dmem_k + o) = make_float4(dk[0], dk[1], dk[2], dk[3]);
    *reinterpret_cast<float4*>(dmem_v + o) = make_float4(dv[0], dv[1], dv[2], dv[3]);
}

// ---------------------------------------------------------------------------------------------------------------------------------
// launchers, called by vpt_attention / vpt_attention_bwd_state for the shapes their own kernels do not take
// ---------------------------------------------------------------------------------------------------------------------------------
int attention_long_fwd(const __nv_bfloat16* Q, const __nv_bfloat16* Kf, const __nv_bfloat16* Vf, const float* R, long long ld_r, const float* b_nd,
                       const uint8_t* first, long long first_stride, const uint8_t* smask, __nv_bfloat16* out, int B, int t, int maxlen, int heads,
                       int nbasis, const int* ring_off, const int* rows, const int* row_off, int plan_B, cudaStream_t stream) {
    VPT_CHECK(nbasis <= kAlNb, "vpt_attention: nbasis=%d > %d", nbasis, kAlNb);
    const size_t smem = (size_t)(kAttBQ + 2 * kAttBK) * kAttPitch * 2 + (size_t)(kAlNb * kAlDist + 2 * kAttBQ) * 4 + kAttBK;
    const bool ring = ring_off != nullptr;
    auto kernel = ring ? attention_long_kernel<true> : attention_long_kernel<false>;
    static bool attr_set[2] = {false, false};
    if (!attr_set[ring]) {
        VPT_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set[ring] = true;
    }
    const int nqb = (t + kAttBQ - 1) / kAttBQ;
    // few CTAs: split each query block's key band over a cluster.  The split is chosen for plan_B rows (B, or 1 for the batch-invariant
    // plan); it fixes the order in which a row's partial softmax sums meet
    const long long ctas = (long long)nqb * heads * plan_B;
    const int band_tiles = (maxlen + kAttBQ - 1 + kAttBK - 1) / kAttBK;  // most key tiles of one query block
    int nsplit = 1;
    if (ctas < num_sms()) nsplit = (int)min((long long)min(kAlSplitMax, band_tiles), (num_sms() + ctas - 1) / ctas);
    dim3 grid(nqb * nsplit, heads, B);
    if (nsplit == 1) {
        launch_k(kernel, grid, dim3(kAttThreads), smem, stream, Q, Kf, Vf, R, ld_r, b_nd, first, first_stride, smask, out, t, maxlen, heads, nbasis, 1,
                 ring_off, rows, row_off);
    } else {
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDim = grid;
        cfg.blockDim = dim3(kAttThreads);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = nsplit;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;  // launched without PDL: pdl_sync() is then a no-op and the launch fully ordered
        (void)cudaLaunchKernelEx(&cfg, kernel, Q, Kf, Vf, R, ld_r, b_nd, first, first_stride, smask, out, t, maxlen, heads, nbasis, nsplit, ring_off,
                                 rows, row_off);
    }
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

// the query-major and key-major passes (P / dS to the workspace, dq | dk | dv | dR to `out`)
int attention_bwd_long(const __nv_bfloat16* Q, const __nv_bfloat16* Kf, const __nv_bfloat16* Vf, const float* R, long long ld_r, const float* b_nd,
                       const uint8_t* first, long long first_stride, const uint8_t* smask, const __nv_bfloat16* dO, __nv_bfloat16* out,
                       long long ld_out, float* wsP, float* wsS, int B, int t, int maxlen, int heads, int nbasis, const float* dstate_k,
                       const float* dstate_v, cudaStream_t stream) {
    const size_t smem_rows = (size_t)(2 * kAlStage + 2 * kAbRows) * kAbPitch * 2 + (size_t)(kAlNb + kAbRows) * kAlKK * 4 + kAlStage;
    const size_t smem_keys = (size_t)(2 * kAlStage) * kAbPitch * 2;
    static bool attr_set = false;
    if (!attr_set) {
        VPT_CUDA(cudaFuncSetAttribute(attn_bwd_rows_long_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_rows));
        attr_set = true;
    }
    dim3 grid((t + kAbRows - 1) / kAbRows, heads, B);
    attn_bwd_rows_long_kernel<<<grid, kAbThreads, smem_rows, stream>>>(Q, Kf, Vf, R, ld_r, b_nd, first, first_stride, smask, dO, out, ld_out, wsP,
                                                                          wsS, t, maxlen, heads, nbasis);
    VPT_LAUNCH_CHECK();
    attn_bwd_keys_long_kernel<<<grid, kAbThreads, smem_keys, stream>>>(Q, dO, wsP, wsS, dstate_k, dstate_v, out, ld_out, t, maxlen, heads);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

// dmem_k / dmem_v from the workspace the passes above wrote
int attention_bwd_long_mem(const __nv_bfloat16* Q, const __nv_bfloat16* dO, const float* wsP, const float* wsS, const uint8_t* first,
                           long long first_stride, const uint8_t* smask, const float* dstate_k, const float* dstate_v, float* dmem_k, float* dmem_v,
                           int B, int t, int maxlen, int heads, cudaStream_t stream) {
    const size_t smem_mem = (size_t)(2 * kAlKK) * kAbPitch * 2;
    dim3 mgrid((maxlen + kAbRows - 1) / kAbRows, heads, B);
    attn_bwd_mem_long_kernel<<<mgrid, kAbThreads, smem_mem, stream>>>(Q, dO, wsP, wsS, first, first_stride, smask, dstate_k, dstate_v, dmem_k, dmem_v,
                                                                       t, maxlen, heads);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

}  // namespace vpt
