// Backward of the banded masked attention (csrc/attention.cuh) for the BC step.  The attention FLOPs are ~0.03 % of the
// model, so this is written for clarity on CUDA cores (fp32 FMA), not for the tensor cores:
//
//   rows kernel  (16 queries of one (batch row, head) per CTA, one warp per query; K / V band staged in shared memory)
//       recomputes the logits + softmax P, dP = dO V^T, dS = P * (dP - sum(P dP)); writes P and dS (indexed by the
//       relative distance d) to a workspace, and dQ = dS K / D, dR = dS b_nd^T to the gradient buffer
//   keys kernel  (16 chunk keys per CTA, one warp per key; Q / dO band staged in shared memory)
//       dK = dS^T Q / D, dV = P^T dO        (chunk rows; + the state_out gradient of the row, when given, before the bf16 rounding)
//   b_nd kernel  (one CTA per distance d)  d b_nd[n][d] = sum_{b,head,i} R[b,i,head,n] * dS[b,head,i,d]
//   memory kernel (16 memory rows per CTA, one warp per row; only when the state_in gradient is asked for)
//       dmem_K = dS^T Q / D, dmem_V = P^T dO over the queries that see the row (+ the state_out gradient of the row when t < maxlen)
//
// Query i (chunk-local) sees the keys j = i+1 .. i+maxlen in [memory|chunk] coordinates, d = maxlen + i - j in [0, maxlen).
// state_out = full[t : t + maxlen]: its row r is memory row t + r (r < maxlen - t) or chunk row r + t - maxlen.
#pragma once
#include "common.cuh"
#include "backward.cuh"

namespace vpt {

constexpr int kAbD = 128;                 // head dim
constexpr int kAbRows = 16;               // queries (keys) per CTA
constexpr int kAbPitch = kAbD + 8;        // bf16 elements per staged row (272 B: conflict-free 16-byte row-strided reads)
constexpr int kAbThreads = kAbRows * 32;
constexpr int kAbMaxPerLane = 4;          // maxlen <= 128

__device__ __forceinline__ float dot8(const uint4& a, const uint4& b) {
    float x[8], y[8];
    unpack8(a, x);
    unpack8(b, y);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s = fmaf(x[j], y[j], s);
    return s;
}

// rows [row0, row0+nrows) x 128 columns (from col0) of a [rows_total][ld] bf16 matrix -> smem (pitch kAbPitch), zeros outside
__device__ __forceinline__ void stage_rows(__nv_bfloat16* dst, const __nv_bfloat16* src, long long ld, int row0, int nrows, int rows_total, int col0) {
    for (int i = threadIdx.x; i < nrows * 16; i += blockDim.x) {
        const int r = i >> 4, ch = i & 15;
        const int row = row0 + r;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (row >= 0 && row < rows_total) v = __ldg(reinterpret_cast<const uint4*>(src + (long long)row * ld + col0 + ch * 8));
        *reinterpret_cast<uint4*>(dst + r * kAbPitch + ch * 8) = v;
    }
}

__global__ void __launch_bounds__(kAbThreads) attn_bwd_rows_kernel(
    const __nv_bfloat16* __restrict__ Q, const __nv_bfloat16* __restrict__ Kf, const __nv_bfloat16* __restrict__ Vf, const float* __restrict__ R,
    long long ld_r, const float* __restrict__ b_nd, const uint8_t* __restrict__ first, long long first_stride, const uint8_t* __restrict__ smask,
    const __nv_bfloat16* __restrict__ dO, __nv_bfloat16* __restrict__ out, long long ld_out, float* __restrict__ wsP, float* __restrict__ wsS, int t,
    int maxlen, int heads, int nbasis) {
    extern __shared__ __align__(16) uint8_t ab_smem[];
    const int nk = maxlen + kAbRows - 1;  // keys staged per CTA
    __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(ab_smem);
    __nv_bfloat16* Vs = Ks + (size_t)nk * kAbPitch;
    __nv_bfloat16* Qs = Vs + (size_t)nk * kAbPitch;           // [16][pitch]
    __nv_bfloat16* Os = Qs + kAbRows * kAbPitch;              // dO rows
    float* Bs = reinterpret_cast<float*>(Os + kAbRows * kAbPitch);  // [nbasis][maxlen]
    float* Ss = Bs + (size_t)nbasis * maxlen;                 // [16][maxlen] dS of each row, by key offset kk
    uint8_t* Ms = reinterpret_cast<uint8_t*>(Ss + (size_t)kAbRows * maxlen);  // [maxlen]

    const int i0 = blockIdx.x * kAbRows, head = blockIdx.y, b = blockIdx.z;
    const int h = heads * kAbD, T = maxlen + t;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j0 = i0 + 1;  // first staged key
    stage_rows(Ks, Kf + (long long)b * T * h, h, j0, nk, T, head * kAbD);
    stage_rows(Vs, Vf + (long long)b * T * h, h, j0, nk, T, head * kAbD);
    stage_rows(Qs, Q + (long long)b * t * h, h, i0, kAbRows, t, head * kAbD);
    stage_rows(Os, dO + (long long)b * t * h, h, i0, kAbRows, t, head * kAbD);
    {
        const bool mem_ok = (first[(long long)b * first_stride] == 0) && (smask != nullptr);
        for (int j = threadIdx.x; j < maxlen; j += blockDim.x) Ms[j] = mem_ok ? smask[(long long)b * maxlen + j] : 0;
        for (int i = threadIdx.x; i < nbasis * maxlen; i += blockDim.x) Bs[i] = __ldg(b_nd + i);
    }
    __syncthreads();
    const int i = i0 + warp;
    if (i >= t) return;  // no further block-wide barriers below
    const long long row = (long long)b * t + i;
    float rr[10];
#pragma unroll
    for (int n = 0; n < 10; ++n) rr[n] = n < nbasis ? __ldg(R + row * ld_r + head * nbasis + n) : 0.f;

    // ---- logits and dP for this lane's keys kk = lane + 32 k  (key j = i + 1 + kk, staged row warp + kk, d = maxlen-1-kk)
    float s[kAbMaxPerLane], dp[kAbMaxPerLane];
    bool ok[kAbMaxPerLane];
    const __nv_bfloat16* qrow = Qs + warp * kAbPitch;
    const __nv_bfloat16* orow = Os + warp * kAbPitch;
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < kAbMaxPerLane; ++k) {
        const int kk = lane + 32 * k;
        s[k] = -INFINITY;
        dp[k] = 0.f;
        ok[k] = false;
        if (kk >= maxlen) continue;
        const int j = i + 1 + kk, d = maxlen - 1 - kk;
        ok[k] = (j >= maxlen) || (Ms[j] != 0);
        const __nv_bfloat16* krow = Ks + (size_t)(warp + kk) * kAbPitch;
        const __nv_bfloat16* vrow = Vs + (size_t)(warp + kk) * kAbPitch;
        float qk = 0.f, ov = 0.f;
#pragma unroll 4
        for (int c = 0; c < 16; ++c) {
            qk += dot8(*reinterpret_cast<const uint4*>(qrow + c * 8), *reinterpret_cast<const uint4*>(krow + c * 8));
            ov += dot8(*reinterpret_cast<const uint4*>(orow + c * 8), *reinterpret_cast<const uint4*>(vrow + c * 8));
        }
        float extra = 0.f;
#pragma unroll
        for (int n = 0; n < 10; ++n)
            if (n < nbasis) extra = fmaf(rr[n], Bs[n * maxlen + d], extra);
        if (ok[k]) {
            s[k] = qk * (1.0f / (float)kAbD) + extra;
            mx = fmaxf(mx, s[k]);
        }
        dp[k] = ov;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float den = 0.f;
#pragma unroll
    for (int k = 0; k < kAbMaxPerLane; ++k) {
        s[k] = ok[k] ? __expf(s[k] - mx) : 0.f;
        den += s[k];
    }
    den = warp_sum(den);
    const float inv = 1.f / den;  // the query's own key (d = 0) is always visible, so den > 0
    float delta = 0.f;
#pragma unroll
    for (int k = 0; k < kAbMaxPerLane; ++k) {
        s[k] *= inv;
        delta = fmaf(s[k], dp[k], delta);
    }
    delta = warp_sum(delta);
    float* srow = Ss + (size_t)warp * maxlen;
    float dr[10];
#pragma unroll
    for (int n = 0; n < 10; ++n) dr[n] = 0.f;
    const long long wbase = (((long long)b * heads + head) * t + i) * maxlen;
#pragma unroll
    for (int k = 0; k < kAbMaxPerLane; ++k) {
        const int kk = lane + 32 * k;
        if (kk >= maxlen) continue;
        const int d = maxlen - 1 - kk;
        const float ds = s[k] * (dp[k] - delta);
        srow[kk] = ds;
        wsP[wbase + d] = s[k];
        wsS[wbase + d] = ds;
#pragma unroll
        for (int n = 0; n < 10; ++n)
            if (n < nbasis) dr[n] = fmaf(ds, Bs[n * maxlen + d], dr[n]);
    }
    __syncwarp();
    // ---- dR (warp reduction per basis) and dQ (lanes own 4 dims, loop over the keys)
#pragma unroll
    for (int n = 0; n < 10; ++n) {
        if (n < nbasis) {
            const float v = warp_sum(dr[n]);
            if (lane == 0) out[row * ld_out + 3 * h + head * nbasis + n] = __float2bfloat16_rn(v);
        }
    }
    float dq[4] = {0.f, 0.f, 0.f, 0.f};
    for (int kk = 0; kk < maxlen; ++kk) {
        const float ds = srow[kk];
        const uint2 kv = *reinterpret_cast<const uint2*>(Ks + (size_t)(warp + kk) * kAbPitch + lane * 4);
        dq[0] = fmaf(ds, bf16_lo(kv.x), dq[0]);
        dq[1] = fmaf(ds, bf16_hi(kv.x), dq[1]);
        dq[2] = fmaf(ds, bf16_lo(kv.y), dq[2]);
        dq[3] = fmaf(ds, bf16_hi(kv.y), dq[3]);
    }
    const float sc = 1.0f / (float)kAbD;
    uint2 o2;
    o2.x = pack_bf16(dq[0] * sc, dq[1] * sc);
    o2.y = pack_bf16(dq[2] * sc, dq[3] * sc);
    *reinterpret_cast<uint2*>(out + row * ld_out + head * kAbD + lane * 4) = o2;
}

__global__ void __launch_bounds__(kAbThreads) attn_bwd_keys_kernel(const __nv_bfloat16* __restrict__ Q, const __nv_bfloat16* __restrict__ dO,
                                                                    const float* __restrict__ wsP, const float* __restrict__ wsS,
                                                                    const float* __restrict__ dsk, const float* __restrict__ dsv,
                                                                    __nv_bfloat16* __restrict__ out, long long ld_out, int t, int maxlen, int heads) {
    extern __shared__ __align__(16) uint8_t ab_smem[];
    const int nq = maxlen + kAbRows - 1;
    __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(ab_smem);
    __nv_bfloat16* Os = Qs + (size_t)nq * kAbPitch;
    const int jc0 = blockIdx.x * kAbRows, head = blockIdx.y, b = blockIdx.z;
    const int h = heads * kAbD;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    stage_rows(Qs, Q + (long long)b * t * h, h, jc0, nq, t, head * kAbD);
    stage_rows(Os, dO + (long long)b * t * h, h, jc0, nq, t, head * kAbD);
    __syncthreads();
    const int jc = jc0 + warp;  // chunk-local key; attended by the queries i = jc + d, d in [0, maxlen)
    if (jc >= t) return;
    const long long bh = (long long)b * heads + head;
    float dk[4] = {0.f, 0.f, 0.f, 0.f}, dv[4] = {0.f, 0.f, 0.f, 0.f};
    for (int d0 = 0; d0 < maxlen; d0 += 32) {
        const int dl = d0 + lane;
        float p = 0.f, ds = 0.f;
        if (dl < maxlen && jc + dl < t) {
            const long long w = ((bh * t) + jc + dl) * maxlen + dl;
            p = __ldg(wsP + w);
            ds = __ldg(wsS + w);
        }
        const int nd = min(32, maxlen - d0);
        for (int dd = 0; dd < nd; ++dd) {
            const float pp = __shfl_sync(0xffffffffu, p, dd), ss = __shfl_sync(0xffffffffu, ds, dd);
            const int r = warp + d0 + dd;  // staged row of query i = jc + d
            const uint2 qv = *reinterpret_cast<const uint2*>(Qs + (size_t)r * kAbPitch + lane * 4);
            const uint2 ov = *reinterpret_cast<const uint2*>(Os + (size_t)r * kAbPitch + lane * 4);
            dk[0] = fmaf(ss, bf16_lo(qv.x), dk[0]); dk[1] = fmaf(ss, bf16_hi(qv.x), dk[1]);
            dk[2] = fmaf(ss, bf16_lo(qv.y), dk[2]); dk[3] = fmaf(ss, bf16_hi(qv.y), dk[3]);
            dv[0] = fmaf(pp, bf16_lo(ov.x), dv[0]); dv[1] = fmaf(pp, bf16_hi(ov.x), dv[1]);
            dv[2] = fmaf(pp, bf16_lo(ov.y), dv[2]); dv[3] = fmaf(pp, bf16_hi(ov.y), dv[3]);
        }
    }
    const float sc = 1.0f / (float)kAbD;
#pragma unroll
    for (int c = 0; c < 4; ++c) dk[c] *= sc;
    const int r = jc + maxlen - t;  // this key's row of state_out (when >= 0)
    if (r >= 0) {  // no addend at all without a state gradient: the bits stay those of the plain backward
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

// Memory row j < maxlen is seen by the queries i in [0, min(j, t)) at d = maxlen + i - j, where the row is visible (state_mask[b, j] and
// not first[b, 0]); the P / dS the rows kernel wrote for those (i, d) are all this needs.  Writes dmem_k / dmem_v fp32 [B][maxlen][h] in
// full (+ the state_out gradient of the row when j >= t).  Fixed-order sums over i, no atomics.
__global__ void __launch_bounds__(kAbThreads) attn_bwd_mem_kernel(const __nv_bfloat16* __restrict__ Q, const __nv_bfloat16* __restrict__ dO,
                                                                   const float* __restrict__ wsP, const float* __restrict__ wsS,
                                                                   const uint8_t* __restrict__ first, long long first_stride,
                                                                   const uint8_t* __restrict__ smask, const float* __restrict__ dsk,
                                                                   const float* __restrict__ dsv, float* __restrict__ dmem_k,
                                                                   float* __restrict__ dmem_v, int t, int maxlen, int heads) {
    extern __shared__ __align__(16) uint8_t ab_smem[];
    const int j0 = blockIdx.x * kAbRows, head = blockIdx.y, b = blockIdx.z;
    const int h = heads * kAbD;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool mem_ok = (first[(long long)b * first_stride] == 0) && (smask != nullptr);
    const int nq = mem_ok ? min(t, min(j0 + kAbRows, maxlen) - 1) : 0;  // queries any row of this CTA is seen by: i < j < min(j0 + 16, maxlen)
    __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(ab_smem);
    __nv_bfloat16* Os = Qs + (size_t)max(nq, 1) * kAbPitch;
    stage_rows(Qs, Q + (long long)b * t * h, h, 0, nq, t, head * kAbD);
    stage_rows(Os, dO + (long long)b * t * h, h, 0, nq, t, head * kAbD);
    __syncthreads();
    const int j = j0 + warp;
    if (j >= maxlen) return;
    const long long bh = (long long)b * heads + head;
    float dk[4] = {0.f, 0.f, 0.f, 0.f}, dv[4] = {0.f, 0.f, 0.f, 0.f};
    const int ni = (mem_ok && smask[(long long)b * maxlen + j] != 0) ? min(j, t) : 0;
    for (int i0 = 0; i0 < ni; i0 += 32) {
        const int il = i0 + lane;
        float p = 0.f, ds = 0.f;
        if (il < ni) {
            const long long w = (bh * t + il) * maxlen + (maxlen + il - j);
            p = __ldg(wsP + w);
            ds = __ldg(wsS + w);
        }
        const int n = min(32, ni - i0);
        for (int ii = 0; ii < n; ++ii) {
            const float pp = __shfl_sync(0xffffffffu, p, ii), ss = __shfl_sync(0xffffffffu, ds, ii);
            const int r = i0 + ii;  // staged row of query i
            const uint2 qv = *reinterpret_cast<const uint2*>(Qs + (size_t)r * kAbPitch + lane * 4);
            const uint2 ov = *reinterpret_cast<const uint2*>(Os + (size_t)r * kAbPitch + lane * 4);
            dk[0] = fmaf(ss, bf16_lo(qv.x), dk[0]); dk[1] = fmaf(ss, bf16_hi(qv.x), dk[1]);
            dk[2] = fmaf(ss, bf16_lo(qv.y), dk[2]); dk[3] = fmaf(ss, bf16_hi(qv.y), dk[3]);
            dv[0] = fmaf(pp, bf16_lo(ov.x), dv[0]); dv[1] = fmaf(pp, bf16_hi(ov.x), dv[1]);
            dv[2] = fmaf(pp, bf16_lo(ov.y), dv[2]); dv[3] = fmaf(pp, bf16_hi(ov.y), dv[3]);
        }
    }
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

// one CTA per distance d: db_nd[n][d] = sum over (b, head, i) of R[b,i,head,n] * dS[b,head,i,d]; fixed-order reduction
__global__ void __launch_bounds__(256) attn_bwd_bnd_kernel(const float* __restrict__ R, long long ld_r, const float* __restrict__ wsS,
                                                             float* __restrict__ db_nd, int B, int t, int maxlen, int heads, int nbasis) {
    __shared__ float red[8][10];
    const int d = blockIdx.x;
    float acc[10];
#pragma unroll
    for (int n = 0; n < 10; ++n) acc[n] = 0.f;
    const long long total = (long long)B * heads * t;
    for (long long e = threadIdx.x; e < total; e += 256) {
        const int i = (int)(e % t);
        const long long bh = e / t;
        const int head = (int)(bh % heads), b = (int)(bh / heads);
        const float ds = __ldg(wsS + e * maxlen + d);
        const float* rp = R + ((long long)b * t + i) * ld_r + head * nbasis;
#pragma unroll
        for (int n = 0; n < 10; ++n)
            if (n < nbasis) acc[n] = fmaf(ds, __ldg(rp + n), acc[n]);
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
    for (int n = 0; n < 10; ++n) {
        const float v = warp_sum(acc[n]);
        if (l == 0) red[w][n] = v;
    }
    __syncthreads();
    if (threadIdx.x < nbasis) {
        float s = 0.f;
        for (int q = 0; q < 8; ++q) s += red[q][threadIdx.x];
        db_nd[threadIdx.x * maxlen + d] = s;
    }
}

// attention_long.cuh: the backward for maxlen > 32 * kAbMaxPerLane
int attention_bwd_long(const __nv_bfloat16* Q, const __nv_bfloat16* Kf, const __nv_bfloat16* Vf, const float* R, long long ld_r, const float* b_nd,
                       const uint8_t* first, long long first_stride, const uint8_t* smask, const __nv_bfloat16* dO, __nv_bfloat16* out,
                       long long ld_out, float* wsP, float* wsS, int B, int t, int maxlen, int heads, int nbasis, const float* dstate_k,
                       const float* dstate_v, cudaStream_t stream);
int attention_bwd_long_mem(const __nv_bfloat16* Q, const __nv_bfloat16* dO, const float* wsP, const float* wsS, const uint8_t* first,
                           long long first_stride, const uint8_t* smask, const float* dstate_k, const float* dstate_v, float* dmem_k, float* dmem_v,
                           int B, int t, int maxlen, int heads, cudaStream_t stream);

}  // namespace vpt

extern "C" int vpt_attention_bwd_state(const void* Q, const void* Kf, const void* Vf, const float* R, int64_t ld_r, const float* b_nd,
                                       const uint8_t* first, int64_t first_stride, const uint8_t* smask, const void* dO, void* out, int64_t ld_out,
                                       float* db_nd, float* workspace, int32_t B, int32_t t, int32_t maxlen, int32_t heads, int32_t nbasis,
                                       const float* dstate_k, const float* dstate_v, float* dmem_k, float* dmem_v, void* stream) {
    using namespace vpt;
    VPT_CHECK(Q && Kf && Vf && R && b_nd && first && dO && out && db_nd && workspace, "vpt_attention_bwd: null argument");
    VPT_CHECK(B > 0 && B <= 65535 && t > 0 && heads > 0 && maxlen > 0 && nbasis > 0 && nbasis <= 10,
              "vpt_attention_bwd: unsupported shape (B=%d t=%d maxlen=%d heads=%d nbasis=%d)", B, t, maxlen, heads, nbasis);
    VPT_CHECK(ld_out % 4 == 0 && ld_out >= 3 * (int64_t)heads * kAbD + heads * nbasis, "vpt_attention_bwd: gradient buffer too narrow");
    VPT_CHECK((dmem_k == nullptr) == (dmem_v == nullptr), "vpt_attention_bwd_state: dmem_k and dmem_v are given together or not at all");
    for (const float* p : {dstate_k, dstate_v, (const float*)dmem_k, (const float*)dmem_v})
        VPT_CHECK(reinterpret_cast<uintptr_t>(p) % 16 == 0, "vpt_attention_bwd_state: state gradients must be 16-byte aligned");
    const size_t ws_half = (size_t)B * heads * t * maxlen;
    float* wsP = workspace;
    float* wsS = workspace + ws_half;
    if (maxlen > 32 * kAbMaxPerLane) {  // longer memories: the band-tiled kernels of attention_long.cuh
        const int rc = attention_bwd_long(reinterpret_cast<const __nv_bfloat16*>(Q), reinterpret_cast<const __nv_bfloat16*>(Kf),
                                          reinterpret_cast<const __nv_bfloat16*>(Vf), R, ld_r, b_nd, first, first_stride, smask,
                                          reinterpret_cast<const __nv_bfloat16*>(dO), reinterpret_cast<__nv_bfloat16*>(out), ld_out, wsP, wsS, B, t,
                                          maxlen, heads, nbasis, dstate_k, dstate_v, (cudaStream_t)stream);
        if (rc != VPT_OK) return rc;
        attn_bwd_bnd_kernel<<<maxlen, 256, 0, (cudaStream_t)stream>>>(R, ld_r, wsS, db_nd, B, t, maxlen, heads, nbasis);
        VPT_LAUNCH_CHECK();
        if (dmem_k == nullptr) return VPT_OK;
        return attention_bwd_long_mem(reinterpret_cast<const __nv_bfloat16*>(Q), reinterpret_cast<const __nv_bfloat16*>(dO), wsP, wsS, first,
                                      first_stride, smask, dstate_k, dstate_v, dmem_k, dmem_v, B, t, maxlen, heads, (cudaStream_t)stream);
    }
    const int nk = maxlen + kAbRows - 1;
    const size_t smem_rows = (size_t)(2 * nk + 2 * kAbRows) * kAbPitch * 2 + ((size_t)nbasis * maxlen + (size_t)kAbRows * maxlen) * 4 + maxlen + 16;
    const size_t smem_keys = (size_t)(2 * nk) * kAbPitch * 2;
    const size_t smem_mem = (size_t)(2 * max(min(t, maxlen - 1), 1)) * kAbPitch * 2;
    static bool attr_set = false;
    if (!attr_set) {
        VPT_CUDA(cudaFuncSetAttribute(attn_bwd_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPT_CUDA(cudaFuncSetAttribute(attn_bwd_keys_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        VPT_CUDA(cudaFuncSetAttribute(attn_bwd_mem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_set = true;
    }
    dim3 grid((t + kAbRows - 1) / kAbRows, heads, B);
    attn_bwd_rows_kernel<<<grid, kAbThreads, smem_rows, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(Q), reinterpret_cast<const __nv_bfloat16*>(Kf), reinterpret_cast<const __nv_bfloat16*>(Vf), R, ld_r, b_nd,
        first, first_stride, smask, reinterpret_cast<const __nv_bfloat16*>(dO), reinterpret_cast<__nv_bfloat16*>(out), ld_out, wsP, wsS, t, maxlen,
        heads, nbasis);
    VPT_LAUNCH_CHECK();
    attn_bwd_keys_kernel<<<grid, kAbThreads, smem_keys, (cudaStream_t)stream>>>(reinterpret_cast<const __nv_bfloat16*>(Q),
                                                                               reinterpret_cast<const __nv_bfloat16*>(dO), wsP, wsS, dstate_k,
                                                                               dstate_v, reinterpret_cast<__nv_bfloat16*>(out), ld_out, t, maxlen,
                                                                               heads);
    VPT_LAUNCH_CHECK();
    attn_bwd_bnd_kernel<<<maxlen, 256, 0, (cudaStream_t)stream>>>(R, ld_r, wsS, db_nd, B, t, maxlen, heads, nbasis);
    VPT_LAUNCH_CHECK();
    if (dmem_k != nullptr) {
        dim3 mgrid((maxlen + kAbRows - 1) / kAbRows, heads, B);
        attn_bwd_mem_kernel<<<mgrid, kAbThreads, smem_mem, (cudaStream_t)stream>>>(
            reinterpret_cast<const __nv_bfloat16*>(Q), reinterpret_cast<const __nv_bfloat16*>(dO), wsP, wsS, first, first_stride, smask, dstate_k,
            dstate_v, dmem_k, dmem_v, t, maxlen, heads);
        VPT_LAUNCH_CHECK();
    }
    return VPT_OK;
}

extern "C" int vpt_attention_bwd(const void* Q, const void* Kf, const void* Vf, const float* R, int64_t ld_r, const float* b_nd, const uint8_t* first,
                                 int64_t first_stride, const uint8_t* smask, const void* dO, void* out, int64_t ld_out, float* db_nd, float* workspace,
                                 int32_t B, int32_t t, int32_t maxlen, int32_t heads, int32_t nbasis, void* stream) {
    return vpt_attention_bwd_state(Q, Kf, Vf, R, ld_r, b_nd, first, first_stride, smask, dO, out, ld_out, db_nd, workspace, B, t, maxlen, heads,
                                   nbasis, nullptr, nullptr, nullptr, nullptr, stream);
}
