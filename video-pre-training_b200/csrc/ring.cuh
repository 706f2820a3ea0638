// The KV memory as a ring (policy.py RingState): per layer K / V bf16 [E][maxlen][h] and the state mask u8 [E][maxlen], memory key j
// of environment e at physical row (off + row_off[e] + j) % maxlen, `off` one device int32 shared by every layer and `row_off` an optional
// device int32 [E] (null: all zeros).  A t = 1 step writes the new K / V row of each layer at the row's slot (ring_write), runs the
// attention on the ring (vpt_attention_ring, attention.cuh / attention_long.cuh), and finally advances `off` (ring_advance) or, for a step
// of some environments only, their `row_off` (ring_advance_rows).  No memory row is ever copied.
//
// A step of some environments takes `rows` int32 [B]: batch row b of the step is environment rows[b], or an inert padding row if
// rows[b] < 0 (it reads and writes no ring memory).  Null `rows`: batch row b is environment b.
#pragma once
#include "common.cuh"

namespace vpt {

// one CTA per batch row: K / V row b of the step -> its environment's ring slot; mask[r][slot] = 1 and, where first[b], every other slot of
// row r cleared (vpt_state_mask_update at t = 1 in ring coordinates: the rolled-in slot is the newest, the others keep their bit unless the
// episode restarts)
__global__ void __launch_bounds__(256) ring_write_kernel(const uint4* __restrict__ knew, const uint4* __restrict__ vnew, uint4* __restrict__ kring,
                                                         uint4* __restrict__ vring, uint8_t* __restrict__ mask, const uint8_t* __restrict__ first,
                                                         long long first_stride, const int* __restrict__ ring_off, const int* __restrict__ rows,
                                                         const int* __restrict__ row_off, int maxlen, int h8) {
    pdl_sync();
    const int b = blockIdx.x;
    const int r = rows ? rows[b] : b;
    if (r < 0) return;  // inert padding row
    const int off = row_off ? (ring_off[0] + row_off[r]) % maxlen : ring_off[0];
    const long long dst = ((long long)r * maxlen + off) * h8;
    for (int c = threadIdx.x; c < h8; c += blockDim.x) {
        kring[dst + c] = knew[(long long)b * h8 + c];
        vring[dst + c] = vnew[(long long)b * h8 + c];
    }
    const bool reset = first[(long long)b * first_stride] != 0;
    uint8_t* m = mask + (long long)r * maxlen;
    for (int j = threadIdx.x; j < maxlen; j += blockDim.x) {
        if (j == off) m[j] = 1;
        else if (reset) m[j] = 0;
    }
}

__global__ void ring_advance_kernel(int* __restrict__ ring_off, int maxlen) {
    pdl_sync();
    if (threadIdx.x == 0) ring_off[0] = (ring_off[0] + 1) % maxlen;
}

// row_off[rows[i]] = (row_off[rows[i]] + 1) % maxlen for every rows[i] >= 0 (the rows are distinct: no two threads share an entry)
__global__ void ring_advance_rows_kernel(int* __restrict__ row_off, const int* __restrict__ rows, int B, int maxlen) {
    pdl_sync();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
        const int r = rows[i];
        if (r >= 0) row_off[r] = (row_off[r] + 1) % maxlen;
    }
}

int ring_write(const void* knew, const void* vnew, void* kring, void* vring, uint8_t* mask, const uint8_t* first, int64_t first_stride,
               const int32_t* ring_off, const int32_t* rows, const int32_t* row_off, int32_t B, int32_t maxlen, int32_t h, void* stream) {
    launch_k(ring_write_kernel, dim3(B), dim3(256), 0, (cudaStream_t)stream, reinterpret_cast<const uint4*>(knew), reinterpret_cast<const uint4*>(vnew),
             reinterpret_cast<uint4*>(kring), reinterpret_cast<uint4*>(vring), mask, first, (long long)first_stride, (const int*)ring_off,
             (const int*)rows, (const int*)row_off, maxlen, h / 8);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

}  // namespace vpt

extern "C" int vpt_ring_write(const void* knew, const void* vnew, void* kring, void* vring, uint8_t* mask, const uint8_t* first, int64_t first_stride,
                              const int32_t* ring_off, int32_t B, int32_t maxlen, int32_t h, void* stream) {
    using namespace vpt;
    VPT_CHECK(knew && vnew && kring && vring && mask && first && ring_off && B > 0 && maxlen > 0 && h > 0, "vpt_ring_write: bad arguments");
    VPT_CHECK(h % 8 == 0, "vpt_ring_write: h = %d must be a multiple of 8", h);
    return ring_write(knew, vnew, kring, vring, mask, first, first_stride, ring_off, nullptr, nullptr, B, maxlen, h, stream);
}

extern "C" int vpt_ring_write_rows(const void* knew, const void* vnew, void* kring, void* vring, uint8_t* mask, const uint8_t* first,
                                   int64_t first_stride, const int32_t* ring_off, const int32_t* rows, const int32_t* row_off, int32_t B, int32_t maxlen,
                                   int32_t h, void* stream) {
    using namespace vpt;
    VPT_CHECK(knew && vnew && kring && vring && mask && first && ring_off && B > 0 && maxlen > 0 && h > 0, "vpt_ring_write_rows: bad arguments");
    VPT_CHECK(h % 8 == 0, "vpt_ring_write_rows: h = %d must be a multiple of 8", h);
    return ring_write(knew, vnew, kring, vring, mask, first, first_stride, ring_off, rows, row_off, B, maxlen, h, stream);
}

extern "C" int vpt_ring_advance(int32_t* ring_off, int32_t maxlen, void* stream) {
    using namespace vpt;
    VPT_CHECK(ring_off && maxlen > 0, "vpt_ring_advance: bad arguments");
    launch_k(ring_advance_kernel, dim3(1), dim3(32), 0, (cudaStream_t)stream, (int*)ring_off, maxlen);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

extern "C" int vpt_ring_advance_rows(int32_t* row_off, const int32_t* rows, int32_t B, int32_t maxlen, void* stream) {
    using namespace vpt;
    VPT_CHECK(row_off && rows && B > 0 && maxlen > 0, "vpt_ring_advance_rows: bad arguments");
    launch_k(ring_advance_rows_kernel, dim3(1), dim3(256), 0, (cudaStream_t)stream, (int*)row_off, (const int*)rows, (int)B, (int)maxlen);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}

namespace vpt {
// the sampling keys of a step of a ring (batch-invariant mode): keys[b] = (r, steps[r]) for batch row b of environment r, then steps[r] += 1;
// an inert row (r < 0) gets (-1, 0) and advances nothing.  The rows are distinct: no two threads share an entry.
__global__ void ring_noise_keys_kernel(long long* __restrict__ steps, const int* __restrict__ rows, long long* __restrict__ keys, int B) {
    pdl_sync();
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
        const int r = rows ? rows[b] : b;
        if (r < 0) {
            keys[2 * b] = -1;
            keys[2 * b + 1] = 0;
            continue;
        }
        const long long s = steps[r];
        keys[2 * b] = r;
        keys[2 * b + 1] = s;
        steps[r] = s + 1;
    }
}
}  // namespace vpt

extern "C" int vpt_ring_noise_keys(int64_t* steps, const int32_t* rows, int64_t* keys, int32_t B, void* stream) {
    using namespace vpt;
    VPT_CHECK(steps && keys && B > 0, "vpt_ring_noise_keys: bad arguments");
    launch_k(ring_noise_keys_kernel, dim3((B + 255) / 256), dim3(256), 0, (cudaStream_t)stream, reinterpret_cast<long long*>(steps), (const int*)rows,
             reinterpret_cast<long long*>(keys), (int)B);
    VPT_LAUNCH_CHECK();
    return VPT_OK;
}
