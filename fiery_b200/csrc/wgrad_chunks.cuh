// The summation order of the bit-reproducible weight gradients (bev_conv_bwd.cu, temporal_entry.cu, causal_conv.cu): the pixel
// tiles, numbered in a fixed order, are cut into c = min(tiles, cap) chunks, chunk i holding tiles [i * tiles / c, (i + 1) * tiles / c);
// each chunk stores its partial and wgrad_reduce_kernel adds the partials in ascending chunk order.  The cap is a per-layer constant,
// not the SM count, so the order depends on the shape only.
#pragma once
#include "common.cuh"

namespace fiery {

constexpr int WG_MAX_CHUNKS = 128;            // the cap of the temporal entry and the causal convolution

inline int wgrad_chunks(long long tiles, int cap) { return static_cast<int>(tiles < cap ? tiles : cap); }

// out[i] (i < n) = sum of partial[c * chunk_floats + offset(i)] over the chunks c in ascending order (zeros when there are none);
// offset(i) is where output i lies in a chunk's partial
template <typename Offset>
__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, int n_chunks, size_t chunk_floats, int n, Offset offset,
                                    float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t off = offset(i);
    float acc = 0.f;
    for (int c = 0; c < n_chunks; ++c) acc += partial[c * chunk_floats + off];
    out[i] = acc;
}

template <typename Offset>
int launch_wgrad_reduce(const float* partial, int n_chunks, size_t chunk_floats, int n, Offset offset, float* out, cudaStream_t stream) {
    wgrad_reduce_kernel<<<(n + 255) / 256, 256, 0, stream>>>(partial, n_chunks, chunk_floats, n, offset, out);
    FIERY_CUDA_CHECK(cudaGetLastError());
    return FIERY_OK;
}

}  // namespace fiery
