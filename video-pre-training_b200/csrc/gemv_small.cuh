// Small-M linear layer (rollout path, B*T <= 8 tokens): out = epilogue(A[M][K] . W[N][K]^T) with the same epilogue contract as
// vpt_gemm_bf16.  With one or a few rows the tensor pipe is irrelevant -- the layer is a read of the weight matrix at HBM
// speed (2x model: 497 MB per step) -- and a 128-row tensor-core tile would leave all but ceil(N/256) SMs idle.  So: one warp
// per output column, lanes stride over K with 16-byte loads of W (streamed, read once) and of the A rows (L1/L2 resident),
// fp32 FMA, warp-shuffle reduction, scalar epilogue; row statistics by a one-CTA-per-row follow-up in the same [M][P] layout.
#pragma once
#include "common.cuh"
#include "elementwise.cuh"
#include "gemm_tc.cuh"

namespace vpt {

constexpr int kGsMaxM = 8;
constexpr int kGsThreads = 256;

constexpr int kGsUnroll = 8;  // 16-byte weight loads in flight per lane (8 x 512 B per warp: what it takes to cover HBM latency with few warps)

// read-once weights: no L1 allocation, and evict-first in L2 -- the 0.5 GB weight stream of a rollout step would otherwise flush the
// activations and the CNN weights (20 MB, re-read every step) out of the 126 MB L2
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint4 ld_stream16(const uint4* p, uint64_t pol) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p), "l"(pol));
    return v;
}

// kWpc warps share one output column (each streams a contiguous 1/kWpc of the K range; partial sums meet in shared memory): used when
// N is small, so that the layer still has thousands of 16-byte loads in flight per SM (N = 256, K = 73984 `dense`: 32 CTAs otherwise).
// kGroups: blockIdx.y picks a group of kGsMaxM rows (the any-M launch); without it the one group is rows 0..M-1 and the code is the M <= 8
// launch's as it always was.  A row's sum is the same either way.
template <int kWpc, bool kGroups>
__global__ void __launch_bounds__(kGsThreads) gemv_small_kernel(const __nv_bfloat16* __restrict__ A, const __nv_bfloat16* __restrict__ W,
                                                                  const GemmParams p) {
    pdl_sync();
    __shared__ float s_part[kGsThreads / 32][kGsMaxM];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = kGroups ? blockIdx.y * kGsMaxM : 0;
    const int M = kGroups ? min(p.M - m0, kGsMaxM) : p.M, K8 = p.K >> 3;
    if (kGroups) A += (size_t)m0 * p.K;
    const uint64_t pol = l2_evict_first_policy();
    constexpr int kCols = (kGsThreads / 32) / kWpc;  // output columns per CTA
    const int kpart = warp % kWpc;
    const int chunk = ((K8 + kWpc - 1) / kWpc + 31) / 32 * 32;
    const int k_begin = kpart * chunk, k_end = min(K8, k_begin + chunk);
    for (int n0 = blockIdx.x * kCols; n0 < p.N; n0 += gridDim.x * kCols) {
        const int n = n0 + warp / kWpc;
        float acc[kGsMaxM];
#pragma unroll
        for (int m = 0; m < kGsMaxM; ++m) acc[m] = 0.f;
        if (n < p.N) {
            const uint4* wrow = reinterpret_cast<const uint4*>(W + (size_t)n * p.K);
            for (int k0 = k_begin + lane; k0 < k_end; k0 += 32 * kGsUnroll) {
                uint4 w[kGsUnroll];
#pragma unroll
                for (int u = 0; u < kGsUnroll; ++u) w[u] = (k0 + 32 * u < k_end) ? ld_stream16(wrow + k0 + 32 * u, pol) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
                for (int u = 0; u < kGsUnroll; ++u) {
                    const int k = k0 + 32 * u;
                    if (k >= k_end) break;
                    const float wf[8] = {bf16_lo(w[u].x), bf16_hi(w[u].x), bf16_lo(w[u].y), bf16_hi(w[u].y),
                                         bf16_lo(w[u].z), bf16_hi(w[u].z), bf16_lo(w[u].w), bf16_hi(w[u].w)};
#pragma unroll
                    for (int m = 0; m < kGsMaxM; ++m) {
                        if (m < M) {
                            const uint4 a = __ldg(reinterpret_cast<const uint4*>(A + (size_t)m * p.K) + k);
                            acc[m] = fmaf(bf16_lo(a.x), wf[0], acc[m]); acc[m] = fmaf(bf16_hi(a.x), wf[1], acc[m]);
                            acc[m] = fmaf(bf16_lo(a.y), wf[2], acc[m]); acc[m] = fmaf(bf16_hi(a.y), wf[3], acc[m]);
                            acc[m] = fmaf(bf16_lo(a.z), wf[4], acc[m]); acc[m] = fmaf(bf16_hi(a.z), wf[5], acc[m]);
                            acc[m] = fmaf(bf16_lo(a.w), wf[6], acc[m]); acc[m] = fmaf(bf16_hi(a.w), wf[7], acc[m]);
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int m = 0; m < kGsMaxM; ++m) acc[m] = warp_sum(acc[m]);
        if (kWpc > 1) {  // fixed-order sum of the K parts (block-uniform control flow: every warp reaches the barriers)
            if (lane == 0) {
#pragma unroll
                for (int m = 0; m < kGsMaxM; ++m) s_part[warp][m] = acc[m];
            }
            __syncthreads();
            if (kpart == 0) {
#pragma unroll
                for (int m = 0; m < kGsMaxM; ++m) {
                    float t = 0.f;
                    for (int q = 0; q < kWpc; ++q) t += s_part[warp + q][m];
                    acc[m] = t;
                }
            }
            __syncthreads();
        }
        if (n >= p.N || kpart != 0) continue;
        if (lane == 0) {
            const float s1 = p.S1 ? __ldg(p.S1 + n) : 0.f, s2 = p.S2 ? __ldg(p.S2 + n) : 0.f;
#pragma unroll
            for (int m = 0; m < kGsMaxM; ++m) {
                if (m >= M) continue;
                const int mg = m0 + m;
                float ga = 1.f, gb = 0.f;
                if (p.mr) {
                    const int g = mg / p.rows_per_group;
                    const float mean = __ldg(p.mr + 2 * g), rstd = __ldg(p.mr + 2 * g + 1);
                    ga = rstd;
                    gb = rstd * mean;
                }
                float v = fmaf(ga, acc[m], fmaf(-gb, s1, s2));
                if (p.relu == 1) v = fmaxf(v, 0.f);
                if (p.residual) {
                    v += p.residual_f32 ? reinterpret_cast<const float*>(p.residual)[(size_t)mg * p.ld_res + n]
                                        : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.residual)[(size_t)mg * p.ld_res + n]);
                }
                if (p.relu == 2) v = fmaxf(v, 0.f);
                v *= p.out_scale;
                // destination: the single one, or the column segment n falls into (fused projections, vpt_gemm_args.dst_*)
                void* d_out = p.out;
                long long d_ld = p.ld_out;
                int d_f32 = p.out_f32, d_col0 = 0;
                bool d_remap = p.seg_len > 0;
                if (p.ndst > 0) {
                    int sg = 0;
                    for (int i = 1; i < p.ndst; ++i)
                        if (n >= p.dst_n0[i]) sg = i;
                    d_out = p.dst_out[sg]; d_ld = p.dst_ld[sg]; d_f32 = p.dst_f32[sg]; d_col0 = p.dst_n0[sg];
                    d_remap = d_remap && p.dst_remap[sg] != 0;
                }
                long long orow = mg;
                if (d_remap) orow = (long long)(mg / p.seg_len) * p.seg_stride + p.seg_off + (mg % p.seg_len);
                if (d_f32) reinterpret_cast<float*>(d_out)[(size_t)orow * d_ld + (n - d_col0)] = v;
                else reinterpret_cast<__nv_bfloat16*>(d_out)[(size_t)orow * d_ld + (n - d_col0)] = __float2bfloat16_rn(v);
            }
        }
    }
}

// statistics partials of the rows just stored, in the [M][P] layout of the tensor-core kernel: slot 0 carries the whole
// row's (sum, sumsq), the other slots are zero.  One CTA per row (M <= 8, N <= a few thousand): negligible.
__global__ void __launch_bounds__(256) row_stats_small_kernel(const GemmParams p, int P) {
    pdl_sync();
    const int m = blockIdx.x;
    long long orow = m;
    if (p.seg_len > 0) orow = (long long)(m / p.seg_len) * p.seg_stride + p.seg_off + (m % p.seg_len);
    float s = 0.f, ss = 0.f;
    for (int n = threadIdx.x; n < p.N; n += blockDim.x) {
        const float v = p.out_f32 ? reinterpret_cast<const float*>(p.out)[(size_t)orow * p.ld_out + n]
                                  : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.out)[(size_t)orow * p.ld_out + n]);
        s += v;
        ss = fmaf(v, v, ss);
    }
    const float2 r = block_sum2(s, ss);
    float2* sp = reinterpret_cast<float2*>(p.stat_part) + (size_t)m * P;
    if (threadIdx.x == 0) sp[0] = r;
    for (int i = 1 + threadIdx.x; i < P; i += blockDim.x) sp[i] = make_float2(0.f, 0.f);
}

static bool gemv_small_shape_ok(const vpt_gemm_args* a) {
    return !a->conv && (a->K & 7) == 0 && !(a->stat_part && a->stat_mode != 1) && !(a->ndst > 0 && a->stat_part);
}

// Launches the weight-streaming kernel over ceil(M / 8) groups of rows.  Every row gets the accumulation order of the M <= 8 launch
// (the K split, lane-to-K mapping and combine order come from N, K and the SM count only), so its result does not depend on M.
template <bool kGroups>
static int launch_gemv_small(const vpt_gemm_args* a, void* stream) {
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = a->M; p.N = a->N; p.K = a->K;
    p.mr = a->mr; p.rows_per_group = a->rows_per_group > 0 ? a->rows_per_group : 1;
    p.S1 = a->mr ? a->S1 : nullptr; p.S2 = a->S2;
    p.relu = a->relu; p.out_scale = a->out_scale;
    p.residual = a->residual; p.residual_f32 = a->residual_f32; p.ld_res = a->ld_res;
    p.out = a->out; p.out_f32 = a->out_f32; p.ld_out = a->ld_out;
    p.seg_len = a->seg_len; p.seg_stride = a->seg_stride; p.seg_off = a->seg_off;
    p.stat_part = a->stat_part; p.stat_mode = a->stat_mode;
    p.ndst = a->ndst;
    for (int i = 0; i < a->ndst && i < 4; ++i) {
        p.dst_n0[i] = a->dst_n0[i]; p.dst_out[i] = a->dst_out[i]; p.dst_ld[i] = a->dst_ld[i]; p.dst_f32[i] = a->dst_f32[i]; p.dst_remap[i] = a->dst_remap[i];
    }
    int bn, nt;
    choose_block_n(a->N, &bn, &nt);
    const int P = nt * 2;  // == vpt_gemm_stat_parts(N)
    // one warp per column when that already gives >= ~4 CTAs per SM, else the 8 warps of a CTA share a column (K split)
    const bool split = a->N < 4 * num_sms() * (kGsThreads / 32) / 8 && a->K >= 2048;
    int grid = split ? a->N : (a->N + kGsThreads / 32 - 1) / (kGsThreads / 32);
    if (grid > 8 * 148) grid = 8 * 148;
    const int groups = (a->M + kGsMaxM - 1) / kGsMaxM;
    if (split)
        launch_k(gemv_small_kernel<kGsThreads / 32, kGroups>, dim3(grid, groups), dim3(kGsThreads), 0, (cudaStream_t)stream, reinterpret_cast<const __nv_bfloat16*>(a->A),
                                                                                          reinterpret_cast<const __nv_bfloat16*>(a->B), p);
    else
        launch_k(gemv_small_kernel<1, kGroups>, dim3(grid, groups), dim3(kGsThreads), 0, (cudaStream_t)stream, reinterpret_cast<const __nv_bfloat16*>(a->A),
                                                                            reinterpret_cast<const __nv_bfloat16*>(a->B), p);
    VPT_LAUNCH_CHECK();
    if (a->stat_part) {
        launch_k(row_stats_small_kernel, dim3(a->M), dim3(256), 0, (cudaStream_t)stream, p, P);
        VPT_LAUNCH_CHECK();
    }
    return VPT_OK;
}

// returns VPT_OK after launching, or 1 if this shape is not handled here (caller falls through to the tensor-core kernel)
static int try_launch_gemv_small(const vpt_gemm_args* a, void* stream) {
    if (a->M > kGsMaxM || !gemv_small_shape_ok(a)) return 1;
    return launch_gemv_small<false>(a, stream);
}

int try_launch_gemv_small_fwd(const vpt_gemm_args* a, void* stream) { return try_launch_gemv_small(a, stream); }

}  // namespace vpt

// The weight-streaming kernel at any M (batch-invariant inference): each row is computed as the M = 1 launch computes it.  Shapes the
// kernel does not take (conv, K % 8 != 0, stat_mode 2, destination segments with statistics) are refused, not sent elsewhere.
extern "C" int vpt_gemm_bf16_rowwise(const vpt_gemm_args* a, void* stream) {
    using namespace vpt;
    VPT_CHECK(a != nullptr && a->A && a->B && a->out, "vpt_gemm_bf16_rowwise: null operand");
    VPT_CHECK(a->M > 0 && a->N > 0 && a->K > 0, "vpt_gemm_bf16_rowwise: bad shape M=%d N=%d K=%d", a->M, a->N, a->K);
    VPT_CHECK(((uintptr_t)a->A & 15) == 0 && ((uintptr_t)a->B & 15) == 0, "vpt_gemm_bf16_rowwise: A/B must be 16-byte aligned");
    VPT_CHECK(a->mr == nullptr || a->rows_per_group > 0, "vpt_gemm_bf16_rowwise: rows_per_group must be > 0 with mr");
    VPT_CHECK(!(a->mr && !a->S1), "vpt_gemm_bf16_rowwise: mr given without S1");
    VPT_CHECK(gemv_small_shape_ok(a), "vpt_gemm_bf16_rowwise: no conv, K %% 8 == 0 (K=%d), statistics in stat_mode 1 and not with dst segments",
              a->K);
    VPT_CHECK((a->M + kGsMaxM - 1) / kGsMaxM <= 65535, "vpt_gemm_bf16_rowwise: M=%d exceeds %d rows", a->M, 65535 * kGsMaxM);
    // up to 8 rows: the M <= 8 launch itself (one group, the same kernel as vpt_gemm_bf16 runs there)
    return a->M <= kGsMaxM ? launch_gemv_small<false>(a, stream) : launch_gemv_small<true>(a, stream);
}
