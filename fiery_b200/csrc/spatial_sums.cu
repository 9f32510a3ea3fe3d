// Per-plane spatial sums of a (b, C, s, X, Y) fp32 tensor: sums[b][c][t] = sum over the X*Y pixels of plane (b, c, t).  The temporal
// block's pyramid pooling takes its spatial means from them (the pool kernel covers the whole map), and the temporal aggregation's
// backward the per-(frame, channel) sums of its output gradient.
//
// One CTA per plane, the plane's pixels read once (a bandwidth-bound pass).  The summation order depends on X*Y only: the plane is cut
// into 4-pixel chunks, thread i adds chunks i, i + 256, i + 512, ... into four accumulators (one per chunk lane), the thread's total is
// (a0 + a1) + (a2 + a3), the warps reduce by an xor butterfly and warp 0 adds the eight warp sums in ascending order.  Whether a chunk
// is read as one float4 (plane base 16-byte aligned) or as four floats changes the load only, so a plane's sum is bit-identical
// whatever its strides, its neighbours or its place in the tensor.  No atomics.
#include "common.cuh"
#include "plane_chunks.cuh"

namespace fiery {

constexpr int SS_THREADS = 256;
constexpr int SS_UNROLL = 4;                       // chunks in flight per thread
constexpr long long SS_MAX_GRID = 1ll << 30;

struct SsShape {
    long long planes, channels, frames;
    long long sb, sc, st;                          // elements
    int pixels;
};

__global__ void __launch_bounds__(SS_THREADS) spatial_sums_kernel(const SsShape s, const float* __restrict__ x, float* __restrict__ sums) {
    __shared__ float warp_sums[SS_THREADS / 32];
    const int n_chunks = (s.pixels + 3) / 4;
    for (long long plane = blockIdx.x; plane < s.planes; plane += gridDim.x) {
        const long long t = plane % s.frames, c = (plane / s.frames) % s.channels, b = plane / (s.frames * s.channels);
        const float* p = x + b * s.sb + c * s.sc + t * s.st;
        const bool vec = (reinterpret_cast<uintptr_t>(p) & 15) == 0;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        for (int q0 = threadIdx.x; q0 < n_chunks; q0 += SS_UNROLL * SS_THREADS) {
            float4 v[SS_UNROLL];
#pragma unroll
            for (int u = 0; u < SS_UNROLL; ++u) {
                const int q = q0 + u * SS_THREADS;
                if (q < n_chunks) v[u] = load_chunk4(p, q, s.pixels, vec);
            }
#pragma unroll
            for (int u = 0; u < SS_UNROLL; ++u) {
                if (q0 + u * SS_THREADS < n_chunks) {
                    a0 += v[u].x;
                    a1 += v[u].y;
                    a2 += v[u].z;
                    a3 += v[u].w;
                }
            }
        }
        float v = (a0 + a1) + (a2 + a3);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
            float total = warp_sums[0];
#pragma unroll
            for (int w = 1; w < SS_THREADS / 32; ++w) total += warp_sums[w];
            sums[plane] = total;
        }
        __syncthreads();                           // warp_sums is rewritten for the next plane
    }
}

int launch_spatial_sums(const fiery_spatial_sums_desc_t* d, const float* x, float* sums, cudaStream_t stream) {
    SsShape s;
    s.channels = d->channels;
    s.frames = d->frames;
    s.planes = static_cast<long long>(d->batch) * d->channels * d->frames;
    s.sb = d->stride_b;
    s.sc = d->stride_c;
    s.st = d->stride_t;
    s.pixels = d->pixels;
    if (s.planes == 0) return FIERY_OK;
    const unsigned grid = static_cast<unsigned>(s.planes < SS_MAX_GRID ? s.planes : SS_MAX_GRID);
    spatial_sums_kernel<<<grid, SS_THREADS, 0, stream>>>(s, x, sums);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
