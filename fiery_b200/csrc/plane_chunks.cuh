// Loads and stores of 4-pixel chunks of a contiguous fp32 pixel run (a pixel plane, or a piece of one), shared by the plane-wise
// passes (spatial_sums.cu, batch_norm.cu).  Chunk q covers pixels 4q .. 4q + 3 of the run; pixels at or past `pixels` read as zero
// and are not written.  `vec`: the run's base is 16-byte aligned, so a whole chunk moves as one float4; otherwise, and for the
// run's last partial chunk, it moves as single floats.  Either way the values are the same: only the access width changes.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fiery {

__device__ __forceinline__ float4 load_chunk4(const float* __restrict__ p, int q, int pixels, bool vec) {
    const int i = 4 * q;
    if (vec && i + 3 < pixels) return __ldg(reinterpret_cast<const float4*>(p) + q);
    float4 v;
    v.x = __ldg(p + i);
    v.y = i + 1 < pixels ? __ldg(p + i + 1) : 0.f;
    v.z = i + 2 < pixels ? __ldg(p + i + 2) : 0.f;
    v.w = i + 3 < pixels ? __ldg(p + i + 3) : 0.f;
    return v;
}

__device__ __forceinline__ void store_chunk4(float* __restrict__ p, int q, int pixels, bool vec, float4 v) {
    const int i = 4 * q;
    if (vec && i + 3 < pixels) {
        reinterpret_cast<float4*>(p)[q] = v;
        return;
    }
    p[i] = v.x;
    if (i + 1 < pixels) p[i + 1] = v.y;
    if (i + 2 < pixels) p[i + 2] = v.z;
    if (i + 3 < pixels) p[i + 3] = v.w;
}

__device__ __forceinline__ bool aligned16_ptr(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace fiery
