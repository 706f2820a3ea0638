// Banded masked self-attention over [KV memory | chunk] with the learned relative-position bias, flash style:
// warp-level mma.sync (m16n8k16 bf16, fp32 accumulate), online fp32 softmax, the mask and the rank-`nbasis`
// relative term computed arithmetically (never materialised).  head_dim is 128 at every VPT width.
//
//   CTA = (64-query block, head, batch row), 4 warps x 16 queries.  For query i (chunk-local) the visible keys are
//   j in (i, i + maxlen] in [memory|chunk] coordinates (d = maxlen + i - j in [0, maxlen)), so a 64-query block
//   touches at most maxlen + 63 keys.
#pragma once
#include "common.cuh"

namespace vpt {

constexpr int kAttD = 128;             // head dim
constexpr int kAttBQ = 64;             // queries per CTA
constexpr int kAttBK = 64;             // keys per block
constexpr int kAttPitch = kAttD + 8;   // bf16 elements per smem row (272 B: conflict-free ldmatrix)
constexpr int kAttThreads = 128;

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// rows [row0, row0+64) of a [rows_total][ld] bf16 matrix (128 columns starting at col0) -> smem tile, zero beyond rows_total
__device__ __forceinline__ void load_tile_64x128(__nv_bfloat16* dst, const __nv_bfloat16* src, long long ld, int row0, int rows_total,
                                                 int col0) {
    for (int i = threadIdx.x; i < 64 * 16; i += kAttThreads) {
        const int r = i >> 4, ch = i & 15;
        __nv_bfloat16* d = dst + r * kAttPitch + ch * 8;
        const int row = row0 + r;
        if (row >= 0 && row < rows_total) cp_async16(d, src + (long long)row * ld + col0 + ch * 8);
        else *reinterpret_cast<uint4*>(d) = make_uint4(0, 0, 0, 0);
    }
}

// Ring layout of the KV memory (t = 1 rollout steps, vpt_attention_ring): K / V are bf16 [B][maxlen][h] and smask u8 [B][maxlen] with
// [memory | chunk] key j at physical row (off + j) % maxlen, so the new chunk row (j = maxlen) sits at `off`, where memory key j = 0 was
// (outside the t = 1 band).  Only the row addresses change: the key order and tiling are those of the linear layout, so are the bits.
__device__ __forceinline__ int ring_row(int row, int off, int maxlen) { return (off + row) % maxlen; }

// A step of some of the ring's environments (vpt_attention_ring_rows) adds two optional device arrays: `rows` int32 [B] maps batch row b
// (Q, R, first, out) to ring row rows[b] (K, V, smask), rows[b] < 0 marking an inert padding row, and `row_off` int32 [E] adds a per-row
// offset: key j of ring row r is at physical row (off + row_off[r] + j) % maxlen.  Null pointers: ring row b, offset `off`.
// The ring row and offset of batch row b, or -1 for an inert row (RING only).
__device__ __forceinline__ int ring_row_of(int b, const int* __restrict__ rows, const int* __restrict__ ring_off, const int* __restrict__ row_off,
                                           int maxlen, int& off) {
    const int r = rows ? rows[b] : b;
    if (r >= 0) off = row_off ? (ring_off[0] + row_off[r]) % maxlen : ring_off[0];
    return r;
}

// the output rows [q0, min(q0 + 64, t)) of one head of batch row b set to zero (an inert row of a ring step: no key is read)
__device__ __forceinline__ void store_zero_rows(__nv_bfloat16* out, int b, int t, int q0, int h, int head) {
    for (int i = threadIdx.x; i < kAttBQ * (kAttD / 8); i += kAttThreads) {
        const int q = q0 + i / (kAttD / 8);
        if (q < t) *reinterpret_cast<uint4*>(out + ((long long)b * t + q) * h + head * kAttD + (i % (kAttD / 8)) * 8) = make_uint4(0, 0, 0, 0);
    }
}

// load_tile_64x128 for a ring: memory-coordinate rows [row0, row0+64), zero beyond rows_total (tiles may wrap)
__device__ __forceinline__ void load_tile_64x128_ring(__nv_bfloat16* dst, const __nv_bfloat16* src, long long ld, int row0, int rows_total,
                                                      int col0, int off, int maxlen) {
    for (int i = threadIdx.x; i < 64 * 16; i += kAttThreads) {
        const int r = i >> 4, ch = i & 15;
        __nv_bfloat16* d = dst + r * kAttPitch + ch * 8;
        const int row = row0 + r;
        if (row >= 0 && row < rows_total) cp_async16(d, src + (long long)ring_row(row, off, maxlen) * ld + col0 + ch * 8);
        else *reinterpret_cast<uint4*>(d) = make_uint4(0, 0, 0, 0);
    }
}

// RING: K / V / smask in the ring layout above, `off` read from ring_off[0] on the device, `rows` / `row_off` optional (t = 1, causal)
template <bool RING>
__global__ void __launch_bounds__(kAttThreads) attention_kernel(
    const __nv_bfloat16* __restrict__ Q, const __nv_bfloat16* __restrict__ Kf, const __nv_bfloat16* __restrict__ Vf,
    const float* __restrict__ R, long long ld_r, const float* __restrict__ b_nd, const uint8_t* __restrict__ first,
    long long first_stride, const uint8_t* __restrict__ smask, __nv_bfloat16* __restrict__ out, int t, int maxlen, int heads,
    int nbasis, int causal, const int* __restrict__ ring_off, const int* __restrict__ rows, const int* __restrict__ row_off) {
    pdl_sync();
    extern __shared__ __align__(16) uint8_t att_smem[];
    __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(att_smem);
    __nv_bfloat16* Ks = Qs + kAttBQ * kAttPitch;
    __nv_bfloat16* Vs = Ks + kAttBK * kAttPitch;
    float* Es = reinterpret_cast<float*>(Vs + kAttBK * kAttPitch);  // [64][maxlen]
    float* Bs = Es + (size_t)kAttBQ * maxlen;                        // [nbasis][maxlen]
    float* Rs = Bs + (size_t)nbasis * maxlen;                        // [64][nbasis]
    uint8_t* Ms = reinterpret_cast<uint8_t*>(Rs + kAttBQ * nbasis);  // [maxlen] memory key usable?

    const int q0 = blockIdx.x * kAttBQ, head = blockIdx.y, b = blockIdx.z;
    const int h = heads * kAttD;
    const int T = maxlen + t;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tg = lane & 3;
    const __nv_bfloat16* Qb = Q + (long long)b * t * h;
    int off = 0;
    const int rk = RING ? ring_row_of(b, rows, ring_off, row_off, maxlen, off) : b;  // row of K / V / smask
    if (RING && rk < 0) {  // inert padding row (uniform over the CTA)
        store_zero_rows(out, b, t, q0, h, head);
        return;
    }
    const long long kv_rows = RING ? maxlen : T;  // rows per batch row of K / V
    const __nv_bfloat16* Kb = Kf + (long long)rk * kv_rows * h;
    const __nv_bfloat16* Vb = Vf + (long long)rk * kv_rows * h;

    load_tile_64x128(Qs, Qb, h, q0, t, head * kAttD);
    if (causal && maxlen > 0) {
        const bool mem_ok = (first[(long long)b * first_stride] == 0) && (smask != nullptr);
        for (int j = threadIdx.x; j < maxlen; j += kAttThreads)
            Ms[j] = mem_ok ? smask[(long long)rk * maxlen + (RING ? ring_row(j, off, maxlen) : j)] : 0;
        for (int i = threadIdx.x; i < nbasis * maxlen; i += kAttThreads) Bs[i] = __ldg(b_nd + i);
        for (int i = threadIdx.x; i < kAttBQ * nbasis; i += kAttThreads) {
            const int r = i / nbasis, n = i % nbasis;
            Rs[i] = (q0 + r < t) ? __ldg(R + ((long long)b * t + q0 + r) * ld_r + head * nbasis + n) : 0.f;
        }
    }
    cp_async_wait_all();
    __syncthreads();
    if (causal && maxlen > 0) {
        for (int i = threadIdx.x; i < kAttBQ * maxlen; i += kAttThreads) {
            const int r = i / maxlen, d = i % maxlen;
            float e = 0.f;
            for (int n = 0; n < nbasis; ++n) e = fmaf(Rs[r * nbasis + n], Bs[n * maxlen + d], e);
            Es[i] = e;
        }
    }

    // Q fragments for this warp's 16 rows, all 8 k-steps
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
    int j_lo, j_hi;  // inclusive key range in [memory|chunk] coordinates
    if (causal) {
        j_lo = q0 + 1;
        j_hi = min(last_q + maxlen, T - 1);
    } else {
        j_lo = 0;
        j_hi = T - 1;
    }
    const int iq[2] = {q0 + warp * 16 + g, q0 + warp * 16 + g + 8};

    for (int kb0 = j_lo; kb0 <= j_hi; kb0 += kAttBK) {
        __syncthreads();  // previous block's K/V fully consumed (also orders the Es writes before first use)
        if (RING) {
            load_tile_64x128_ring(Ks, Kb, h, kb0, T, head * kAttD, off, maxlen);
            load_tile_64x128_ring(Vs, Vb, h, kb0, T, head * kAttD, off, maxlen);
        } else {
            load_tile_64x128(Ks, Kb, h, kb0, T, head * kAttD);
            load_tile_64x128(Vs, Vb, h, kb0, T, head * kAttD);
        }
        cp_async_wait_all();
        __syncthreads();

        // S = Q K^T  (16 x 64 per warp)
        float s[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {  // pairs of 8-key tiles
                uint32_t b0, b1, b2, b3;
                const int krow = np * 16 + (lane & 7) + ((lane >> 4) << 3);
                const int kcol = ks * 16 + (((lane >> 3) & 1) << 3);
                ldsm_x4(smem_u32(Ks + krow * kAttPitch + kcol), b0, b1, b2, b3);
                mma_bf16_16816(s[2 * np], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], b0, b1);
                mma_bf16_16816(s[2 * np + 1], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], b2, b3);
            }
        }
        // logits (log2 domain), mask, relative bias
        float bmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int n = 0; n < 8; ++n) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int rr = e >> 1;
                const int i = iq[rr];
                const int j = kb0 + n * 8 + 2 * tg + (e & 1);
                bool ok = (i < t) && (j < T);
                float extra = 0.f;
                if (causal) {
                    const int d = maxlen + i - j;
                    ok = ok && (d >= 0) && (d < maxlen);
                    if (ok) {
                        ok = (j >= maxlen) || (Ms[j] != 0);
                        extra = Es[(warp * 16 + g + rr * 8) * maxlen + d];
                    }
                }
                const float v = ok ? (s[n][e] * qk_scale + extra) * kLog2e : -INFINITY;
                s[n][e] = v;
                bmax[rr] = fmaxf(bmax[rr], v);
            }
        }
        float scale[2];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            float bm = bmax[rr];
            bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 1));
            bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 2));
            const float m_new = fmaxf(mrow[rr], bm);
            const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
            scale[rr] = exp2f(mrow[rr] - m_use);  // exp2(-inf) = 0 on the first block
            mrow[rr] = m_new;
            float rs = 0.f;
#pragma unroll
            for (int n = 0; n < 8; ++n) {
                const float p0 = exp2f(s[n][2 * rr] - m_use), p1 = exp2f(s[n][2 * rr + 1] - m_use);
                s[n][2 * rr] = p0;
                s[n][2 * rr + 1] = p1;
                rs += p0 + p1;
            }
            rs += __shfl_xor_sync(0xffffffffu, rs, 1);
            rs += __shfl_xor_sync(0xffffffffu, rs, 2);
            lrow[rr] = lrow[rr] * scale[rr] + rs;
        }
#pragma unroll
        for (int n = 0; n < 16; ++n) {
            o[n][0] *= scale[0]; o[n][1] *= scale[0];
            o[n][2] *= scale[1]; o[n][3] *= scale[1];
        }
        // O += P V   (P: 16 x 64 as A fragments; V: [key][d] read with ldmatrix.trans)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const uint32_t a0 = pack_bf16(s[2 * ks][0], s[2 * ks][1]);
            const uint32_t a1 = pack_bf16(s[2 * ks][2], s[2 * ks][3]);
            const uint32_t a2 = pack_bf16(s[2 * ks + 1][0], s[2 * ks + 1][1]);
            const uint32_t a3 = pack_bf16(s[2 * ks + 1][2], s[2 * ks + 1][3]);
#pragma unroll
            for (int np = 0; np < 8; ++np) {  // pairs of 8-wide d tiles
                uint32_t b0, b1, b2, b3;
                const int vrow = ks * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
                const int vcol = np * 16 + ((lane >> 4) << 3);
                ldsm_x4_t(smem_u32(Vs + vrow * kAttPitch + vcol), b0, b1, b2, b3);
                mma_bf16_16816(o[2 * np], a0, a1, a2, a3, b0, b1);
                mma_bf16_16816(o[2 * np + 1], a0, a1, a2, a3, b2, b3);
            }
        }
    }

    // normalise and store
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const int i = iq[rr];
        if (i >= t) continue;
        const float inv = 1.0f / lrow[rr];
        __nv_bfloat16* op = out + ((long long)b * t + i) * h + head * kAttD;
#pragma unroll
        for (int n = 0; n < 16; ++n)
            *reinterpret_cast<uint32_t*>(op + n * 8 + 2 * tg) = pack_bf16(o[n][2 * rr] * inv, o[n][2 * rr + 1] * inv);
    }
}

// attention_long.cuh: the causal forward for a KV memory whose bias table does not fit this kernel's shared memory
int attention_long_fwd(const __nv_bfloat16* Q, const __nv_bfloat16* Kf, const __nv_bfloat16* Vf, const float* R, long long ld_r, const float* b_nd,
                       const uint8_t* first, long long first_stride, const uint8_t* smask, __nv_bfloat16* out, int B, int t, int maxlen, int heads,
                       int nbasis, const int* ring_off, const int* rows, const int* row_off, int plan_B, cudaStream_t stream);

// shared memory of attention_kernel for a causal band of `maxlen` keys with `nb` basis rows (nb = 0: mask "none")
inline size_t attention_smem(int maxlen, int nb) {
    return (size_t)(kAttBQ + 2 * kAttBK) * kAttPitch * 2 + ((size_t)kAttBQ * maxlen + (size_t)nb * maxlen + (size_t)kAttBQ * nb) * 4 +
           (size_t)((maxlen + 15) / 16 * 16) + 16;
}

}  // namespace vpt

// plan_batch: the batch size whose launch plan (the long band's cluster split) the call runs; vpt_attention passes B.  attention_kernel
// itself has no batch-dependent choice: one CTA per (query block, head, batch row).
extern "C" int vpt_attention_plan(const void* Q, const void* Kf, const void* Vf, const float* R, int64_t ld_r, const float* b_nd,
                                  const uint8_t* first, int64_t first_stride, const uint8_t* smask, void* out, int32_t B, int32_t t,
                                  int32_t maxlen, int32_t heads, int32_t nbasis, int32_t causal, int32_t plan_batch, void* stream) {
    using namespace vpt;
    VPT_CHECK(plan_batch > 0, "vpt_attention_plan: plan_batch=%d must be > 0", plan_batch);
    VPT_CHECK(Q && Kf && Vf && out && B > 0 && t > 0 && heads > 0 && maxlen >= 0, "vpt_attention: bad arguments");
    if (causal) VPT_CHECK(maxlen > 0 && R && b_nd && first && nbasis > 0, "vpt_attention: causal mode needs maxlen > 0, R, b_nd, first");
    else VPT_CHECK(maxlen == 0, "vpt_attention: mask 'none' has no KV memory (maxlen must be 0)");
    VPT_CHECK(B <= 65535 && heads <= 65535, "vpt_attention: grid too large");
    const int nb = causal ? nbasis : 0;
    const size_t smem = attention_smem(maxlen, nb);
    if (smem > 227 * 1024) {  // only a causal band can be this long (mask 'none' has no memory): tile it over keys
        return attention_long_fwd(reinterpret_cast<const __nv_bfloat16*>(Q), reinterpret_cast<const __nv_bfloat16*>(Kf),
                                  reinterpret_cast<const __nv_bfloat16*>(Vf), R, ld_r, b_nd, first, first_stride, smask,
                                  reinterpret_cast<__nv_bfloat16*>(out), B, t, maxlen, heads, nb, nullptr, nullptr, nullptr, plan_batch, (cudaStream_t)stream);
    }
    static size_t attr = 0;
    if (smem > attr) {
        VPT_CUDA(cudaFuncSetAttribute(attention_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    dim3 grid((t + kAttBQ - 1) / kAttBQ, heads, B);
    launch_k(attention_kernel<false>, dim3(grid), dim3(kAttThreads), smem, (cudaStream_t)stream, 
        reinterpret_cast<const __nv_bfloat16*>(Q), reinterpret_cast<const __nv_bfloat16*>(Kf), reinterpret_cast<const __nv_bfloat16*>(Vf), R,
        ld_r, b_nd, first, first_stride, smask, reinterpret_cast<__nv_bfloat16*>(out), t, maxlen, heads, nb, causal, (const int*)nullptr,
        (const int*)nullptr, (const int*)nullptr);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_attention(const void* Q, const void* Kf, const void* Vf, const float* R, int64_t ld_r, const float* b_nd,
                             const uint8_t* first, int64_t first_stride, const uint8_t* smask, void* out, int32_t B, int32_t t,
                             int32_t maxlen, int32_t heads, int32_t nbasis, int32_t causal, void* stream) {
    return vpt_attention_plan(Q, Kf, Vf, R, ld_r, b_nd, first, first_stride, smask, out, B, t, maxlen, heads, nbasis, causal, B, stream);
}

namespace vpt {

int attention_ring(const void* Q, const void* Kr, const void* Vr, const float* R, int64_t ld_r, const float* b_nd, const uint8_t* first,
                   int64_t first_stride, const uint8_t* smask, const int32_t* ring_off, const int32_t* rows, const int32_t* row_off, void* out,
                   int32_t B, int32_t maxlen, int32_t heads, int32_t nbasis, int32_t plan_B, void* stream) {
    VPT_CHECK(plan_B > 0, "vpt_attention_ring_plan: plan_batch=%d must be > 0", plan_B);
    const size_t smem = attention_smem(maxlen, nbasis);
    if (smem > 227 * 1024) {
        return attention_long_fwd(reinterpret_cast<const __nv_bfloat16*>(Q), reinterpret_cast<const __nv_bfloat16*>(Kr),
                                  reinterpret_cast<const __nv_bfloat16*>(Vr), R, ld_r, b_nd, first, first_stride, smask,
                                  reinterpret_cast<__nv_bfloat16*>(out), B, 1, maxlen, heads, nbasis, ring_off, rows, row_off, plan_B, (cudaStream_t)stream);
    }
    static size_t attr = 0;
    if (smem > attr) {
        VPT_CUDA(cudaFuncSetAttribute(attention_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    launch_k(attention_kernel<true>, dim3(1, heads, B), dim3(kAttThreads), smem, (cudaStream_t)stream,
        reinterpret_cast<const __nv_bfloat16*>(Q), reinterpret_cast<const __nv_bfloat16*>(Kr), reinterpret_cast<const __nv_bfloat16*>(Vr), R,
        ld_r, b_nd, first, first_stride, smask, reinterpret_cast<__nv_bfloat16*>(out), 1, maxlen, heads, nbasis, 1, (const int*)ring_off,
        (const int*)rows, (const int*)row_off);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

}  // namespace vpt

extern "C" int vpt_attention_ring(const void* Q, const void* Kr, const void* Vr, const float* R, int64_t ld_r, const float* b_nd,
                                  const uint8_t* first, int64_t first_stride, const uint8_t* smask, const int32_t* ring_off, void* out, int32_t B,
                                  int32_t maxlen, int32_t heads, int32_t nbasis, void* stream) {
    using namespace vpt;
    VPT_CHECK(Q && Kr && Vr && R && b_nd && first && smask && ring_off && out && B > 0 && maxlen > 0 && heads > 0 && nbasis > 0,
              "vpt_attention_ring: bad arguments");
    VPT_CHECK(B <= 65535 && heads <= 65535, "vpt_attention_ring: grid too large");
    return attention_ring(Q, Kr, Vr, R, ld_r, b_nd, first, first_stride, smask, ring_off, nullptr, nullptr, out, B, maxlen, heads, nbasis, B, stream);
}

extern "C" int vpt_attention_ring_rows(const void* Q, const void* Kr, const void* Vr, const float* R, int64_t ld_r, const float* b_nd,
                                       const uint8_t* first, int64_t first_stride, const uint8_t* smask, const int32_t* ring_off, const int32_t* rows,
                                       const int32_t* row_off, void* out, int32_t B, int32_t maxlen, int32_t heads, int32_t nbasis, void* stream) {
    using namespace vpt;
    VPT_CHECK(Q && Kr && Vr && R && b_nd && first && smask && ring_off && out && B > 0 && maxlen > 0 && heads > 0 && nbasis > 0,
              "vpt_attention_ring_rows: bad arguments");
    VPT_CHECK(B <= 65535 && heads <= 65535, "vpt_attention_ring_rows: grid too large");
    return attention_ring(Q, Kr, Vr, R, ld_r, b_nd, first, first_stride, smask, ring_off, rows, row_off, out, B, maxlen, heads, nbasis, B, stream);
}

// vpt_attention_ring / vpt_attention_ring_rows (rows may be null) with the long band's cluster split of plan_batch rows
extern "C" int vpt_attention_ring_plan(const void* Q, const void* Kr, const void* Vr, const float* R, int64_t ld_r, const float* b_nd,
                                       const uint8_t* first, int64_t first_stride, const uint8_t* smask, const int32_t* ring_off, void* out, int32_t B,
                                       int32_t maxlen, int32_t heads, int32_t nbasis, int32_t plan_batch, void* stream) {
    using namespace vpt;
    VPT_CHECK(Q && Kr && Vr && R && b_nd && first && smask && ring_off && out && B > 0 && maxlen > 0 && heads > 0 && nbasis > 0,
              "vpt_attention_ring_plan: bad arguments");
    VPT_CHECK(B <= 65535 && heads <= 65535, "vpt_attention_ring_plan: grid too large");
    return attention_ring(Q, Kr, Vr, R, ld_r, b_nd, first, first_stride, smask, ring_off, nullptr, nullptr, out, B, maxlen, heads, nbasis, plan_batch,
                          stream);
}

extern "C" int vpt_attention_ring_rows_plan(const void* Q, const void* Kr, const void* Vr, const float* R, int64_t ld_r, const float* b_nd,
                                            const uint8_t* first, int64_t first_stride, const uint8_t* smask, const int32_t* ring_off,
                                            const int32_t* rows, const int32_t* row_off, void* out, int32_t B, int32_t maxlen, int32_t heads,
                                            int32_t nbasis, int32_t plan_batch, void* stream) {
    using namespace vpt;
    VPT_CHECK(Q && Kr && Vr && R && b_nd && first && smask && ring_off && out && B > 0 && maxlen > 0 && heads > 0 && nbasis > 0,
              "vpt_attention_ring_rows_plan: bad arguments");
    VPT_CHECK(B <= 65535 && heads <= 65535, "vpt_attention_ring_rows_plan: grid too large");
    return attention_ring(Q, Kr, Vr, R, ld_r, b_nd, first, first_stride, smask, ring_off, rows, row_off, out, B, maxlen, heads, nbasis, plan_batch,
                          stream);
}
