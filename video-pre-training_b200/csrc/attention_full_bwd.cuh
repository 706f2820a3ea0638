// Backward of the unmasked attention of the IDM (attention_mask_style "none", csrc/attention.cuh with causal = 0): no KV memory
// (maxlen = 0), every query of a chunk sees all t keys of its own chunk, logits = q.k / D (muP), no relative-position term.
// The causal kernel (attention_bwd.cuh) indexes its workspace by distance inside the band; here the band is the whole chunk, so the
// workspace is the plain [t][t] matrix per (batch row, head).  t <= 128 (the IDM's 128-frame chunks), D = 128.
//
//   rows kernel  (16 queries of one (batch row, head) per CTA, one warp per query; all t keys / values staged in shared memory)
//       recomputes the logits and the softmax P (the forward keeps no log-sum-exp; 128 keys per row make this cheap),
//       dP = dO V^T, dS = P * (dP - sum(P dP)); writes P and dS to the workspace and dQ = dS K / D to the gradient buffer
//   keys kernel  (16 keys per CTA, one warp per key; all t queries / output gradients staged)
//       dK = dS^T Q / D, dV = P^T dO
// Every output element is written by exactly one thread with a fixed summation order: no atomics, bit-reproducible.
// CUDA cores, fp32 FMA: at the 4x IDM shape (B = 4, t = 128, 32 heads) this is ~1.3 GFMA per layer, well under 1 % of the step.
#pragma once
#include "common.cuh"
#include "backward.cuh"
#include "attention_bwd.cuh"

namespace vpt {

constexpr int kAfMaxT = 128;

__global__ void __launch_bounds__(kAbThreads) attn_full_bwd_rows_kernel(const __nv_bfloat16* __restrict__ Q, const __nv_bfloat16* __restrict__ K,
                                                                         const __nv_bfloat16* __restrict__ V, const __nv_bfloat16* __restrict__ dO,
                                                                         __nv_bfloat16* __restrict__ out, long long ld_out, float* __restrict__ wsP,
                                                                         float* __restrict__ wsS, int t, int heads) {
    extern __shared__ __align__(16) uint8_t af_smem[];
    __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(af_smem);
    __nv_bfloat16* Vs = Ks + (size_t)t * kAbPitch;
    __nv_bfloat16* Qs = Vs + (size_t)t * kAbPitch;   // [16][pitch]
    __nv_bfloat16* Os = Qs + kAbRows * kAbPitch;     // dO rows
    float* Ss = reinterpret_cast<float*>(Os + kAbRows * kAbPitch);  // [16][t] dS of each row
    const int i0 = blockIdx.x * kAbRows, head = blockIdx.y, b = blockIdx.z;
    const int h = heads * kAbD;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    stage_rows(Ks, K + (long long)b * t * h, h, 0, t, t, head * kAbD);
    stage_rows(Vs, V + (long long)b * t * h, h, 0, t, t, head * kAbD);
    stage_rows(Qs, Q + (long long)b * t * h, h, i0, kAbRows, t, head * kAbD);
    stage_rows(Os, dO + (long long)b * t * h, h, i0, kAbRows, t, head * kAbD);
    __syncthreads();
    const int i = i0 + warp;
    if (i >= t) return;  // no block-wide barriers below
    const long long row = (long long)b * t + i;
    // logits and dP for this lane's keys j = lane + 32 k
    float s[kAbMaxPerLane], dp[kAbMaxPerLane];
    const __nv_bfloat16* qrow = Qs + warp * kAbPitch;
    const __nv_bfloat16* orow = Os + warp * kAbPitch;
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < kAbMaxPerLane; ++k) {
        const int j = lane + 32 * k;
        s[k] = -INFINITY;
        dp[k] = 0.f;
        if (j >= t) continue;
        const __nv_bfloat16* krow = Ks + (size_t)j * kAbPitch;
        const __nv_bfloat16* vrow = Vs + (size_t)j * kAbPitch;
        float qk = 0.f, ov = 0.f;
#pragma unroll 4
        for (int c = 0; c < 16; ++c) {
            qk += dot8(*reinterpret_cast<const uint4*>(qrow + c * 8), *reinterpret_cast<const uint4*>(krow + c * 8));
            ov += dot8(*reinterpret_cast<const uint4*>(orow + c * 8), *reinterpret_cast<const uint4*>(vrow + c * 8));
        }
        s[k] = qk * (1.0f / (float)kAbD);
        mx = fmaxf(mx, s[k]);
        dp[k] = ov;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float den = 0.f;
#pragma unroll
    for (int k = 0; k < kAbMaxPerLane; ++k) {
        s[k] = (lane + 32 * k < t) ? __expf(s[k] - mx) : 0.f;
        den += s[k];
    }
    den = warp_sum(den);
    const float inv = 1.f / den;
    float delta = 0.f;
#pragma unroll
    for (int k = 0; k < kAbMaxPerLane; ++k) {
        s[k] *= inv;
        delta = fmaf(s[k], dp[k], delta);
    }
    delta = warp_sum(delta);
    float* srow = Ss + (size_t)warp * t;
    const long long wbase = (((long long)b * heads + head) * t + i) * t;
#pragma unroll
    for (int k = 0; k < kAbMaxPerLane; ++k) {
        const int j = lane + 32 * k;
        if (j >= t) continue;
        const float ds = s[k] * (dp[k] - delta);
        srow[j] = ds;
        wsP[wbase + j] = s[k];
        wsS[wbase + j] = ds;
    }
    __syncwarp();
    // dQ: lanes own 4 dims, loop over the keys in order
    float dq[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < t; ++j) {
        const float ds = srow[j];
        const uint2 kv = *reinterpret_cast<const uint2*>(Ks + (size_t)j * kAbPitch + lane * 4);
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

__global__ void __launch_bounds__(kAbThreads) attn_full_bwd_keys_kernel(const __nv_bfloat16* __restrict__ Q, const __nv_bfloat16* __restrict__ dO,
                                                                         const float* __restrict__ wsP, const float* __restrict__ wsS,
                                                                         __nv_bfloat16* __restrict__ out, long long ld_out, int t, int heads) {
    extern __shared__ __align__(16) uint8_t af_smem[];
    __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(af_smem);
    __nv_bfloat16* Os = Qs + (size_t)t * kAbPitch;
    const int j0 = blockIdx.x * kAbRows, head = blockIdx.y, b = blockIdx.z;
    const int h = heads * kAbD;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    stage_rows(Qs, Q + (long long)b * t * h, h, 0, t, t, head * kAbD);
    stage_rows(Os, dO + (long long)b * t * h, h, 0, t, t, head * kAbD);
    __syncthreads();
    const int j = j0 + warp;
    if (j >= t) return;
    const long long bh = (long long)b * heads + head;
    float dk[4] = {0.f, 0.f, 0.f, 0.f}, dv[4] = {0.f, 0.f, 0.f, 0.f};
    for (int q0 = 0; q0 < t; q0 += 32) {
        const int ql = q0 + lane;
        float p = 0.f, ds = 0.f;
        if (ql < t) {
            const long long w = (bh * t + ql) * t + j;
            p = __ldg(wsP + w);
            ds = __ldg(wsS + w);
        }
        const int nq = min(32, t - q0);
        for (int qq = 0; qq < nq; ++qq) {
            const float pp = __shfl_sync(0xffffffffu, p, qq), ss = __shfl_sync(0xffffffffu, ds, qq);
            const int r = q0 + qq;
            const uint2 qv = *reinterpret_cast<const uint2*>(Qs + (size_t)r * kAbPitch + lane * 4);
            const uint2 ov = *reinterpret_cast<const uint2*>(Os + (size_t)r * kAbPitch + lane * 4);
            dk[0] = fmaf(ss, bf16_lo(qv.x), dk[0]); dk[1] = fmaf(ss, bf16_hi(qv.x), dk[1]);
            dk[2] = fmaf(ss, bf16_lo(qv.y), dk[2]); dk[3] = fmaf(ss, bf16_hi(qv.y), dk[3]);
            dv[0] = fmaf(pp, bf16_lo(ov.x), dv[0]); dv[1] = fmaf(pp, bf16_hi(ov.x), dv[1]);
            dv[2] = fmaf(pp, bf16_lo(ov.y), dv[2]); dv[3] = fmaf(pp, bf16_hi(ov.y), dv[3]);
        }
    }
    const float sc = 1.0f / (float)kAbD;
    const long long row = (long long)b * t + j;
    uint2 o2;
    o2.x = pack_bf16(dk[0] * sc, dk[1] * sc);
    o2.y = pack_bf16(dk[2] * sc, dk[3] * sc);
    *reinterpret_cast<uint2*>(out + row * ld_out + h + head * kAbD + lane * 4) = o2;
    o2.x = pack_bf16(dv[0], dv[1]);
    o2.y = pack_bf16(dv[2], dv[3]);
    *reinterpret_cast<uint2*>(out + row * ld_out + 2 * h + head * kAbD + lane * 4) = o2;
}

}  // namespace vpt

extern "C" int64_t vpt_attention_full_bwd_workspace(int32_t B, int32_t t, int32_t heads) { return 2LL * B * heads * t * t; }

extern "C" int vpt_attention_full_bwd(const void* Q, const void* K, const void* V, const void* dO, void* out, int64_t ld_out, float* workspace, int32_t B,
                                      int32_t t, int32_t heads, void* stream) {
    using namespace vpt;
    VPT_CHECK(Q && K && V && dO && out && workspace, "vpt_attention_full_bwd: null argument");
    VPT_CHECK(B > 0 && B <= 65535 && t > 0 && t <= kAfMaxT && heads > 0 && heads <= 65535,
              "vpt_attention_full_bwd: unsupported shape (B=%d t=%d heads=%d; t <= %d)", B, t, heads, kAfMaxT);
    VPT_CHECK(ld_out % 4 == 0 && ld_out >= 3 * (int64_t)heads * kAbD, "vpt_attention_full_bwd: gradient buffer too narrow");
    float* wsP = workspace;
    float* wsS = workspace + (size_t)B * heads * t * t;
    const size_t smem_rows = (size_t)(2 * t + 2 * kAbRows) * kAbPitch * 2 + (size_t)kAbRows * t * 4;
    const size_t smem_keys = (size_t)(2 * t) * kAbPitch * 2;
    static bool attr_set = false;
    if (!attr_set) {
        VPT_CUDA(cudaFuncSetAttribute(attn_full_bwd_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
        VPT_CUDA(cudaFuncSetAttribute(attn_full_bwd_keys_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
        attr_set = true;
    }
    dim3 grid((t + kAbRows - 1) / kAbRows, heads, B);
    attn_full_bwd_rows_kernel<<<grid, kAbThreads, smem_rows, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(Q), reinterpret_cast<const __nv_bfloat16*>(K), reinterpret_cast<const __nv_bfloat16*>(V),
        reinterpret_cast<const __nv_bfloat16*>(dO), reinterpret_cast<__nv_bfloat16*>(out), ld_out, wsP, wsS, t, heads);
    VPT_LAUNCH_CHECK();
    attn_full_bwd_keys_kernel<<<grid, kAbThreads, smem_keys, (cudaStream_t)stream>>>(reinterpret_cast<const __nv_bfloat16*>(Q),
                                                                                    reinterpret_cast<const __nv_bfloat16*>(dO), wsP, wsS,
                                                                                    reinterpret_cast<__nv_bfloat16*>(out), ld_out, t, heads);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}
