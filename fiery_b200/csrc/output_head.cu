// The decoder's output heads after their 3x3 convolution (fiery/models/decoder.py:24-50: BatchNorm2d, ReLU, Conv2d(C, n, 1) with a
// bias) as a chain of the project's kernels (include/fiery_b200.h, fiery_output_head_*), on `maps` (X, Y) maps y with C channels:
//
//   k   = bn's coefficients of y          batch-norm statistics and finalize, no apply pass
//   out = W1 relu(fmaf(k, y)) + b1        the temporal entry's forward with the Bottleneck's BN + ReLU prologue, and b1 folded in
//                                         as one extra channel of value 1 (batch = maps, frames = 1, N = n rounded up to 8)
//
// so relu(bn(y)) never reaches memory.  The backward is two passes over y (batch_norm.cu's output-head section): the sums pass
// (the norm's gradient sums, dW1 and db1, with the 1x1's input gradient recomputed from grad_out per piece) and the apply pass (dy).
// Every reduction has a fixed order: bit-reproducible, graph-capturable, no atomics and no host synchronisation.
#include "bn_coef.cuh"

namespace fiery {

size_t temporal_entry_packed_bytes(const fiery_temporal_entry_desc_t* d);
int launch_temporal_entry_pack(const fiery_temporal_entry_desc_t* d, const float* w, float* packed, cudaStream_t stream);
int launch_output_head_entry_forward(const fiery_temporal_entry_desc_t* d, const float* x, const float* ones, const float* packed,
                                     const BnCoef* coef, float* out, cudaStream_t stream);
size_t output_head_backward_workspace_bytes(const fiery_batch_norm_desc_t* d, int n);
int launch_output_head_backward(const fiery_batch_norm_desc_t* d, const float* y, const float* g, const float* w1, int ld, int n,
                                const float* w, const float* bias, const float* mean, const float* var, float* grad_y, float* grad_bn_w,
                                float* grad_bn_b, float* grad_w, float* grad_b, void* workspace, cudaStream_t stream);

static size_t oh_align(size_t v) { return (v + 255) / 256 * 256; }

// the 1x1 as a temporal entry over (batch = maps, frames = 1) with one extra channel (the bias), the norm over (maps, C, 1, X, Y)
static fiery_temporal_entry_desc_t oh_entry(const fiery_output_head_desc_t* d) {
    fiery_temporal_entry_desc_t e{};
    e.batch = d->maps;
    e.frames = 1;
    e.pixels = d->grid_x * d->grid_y;
    e.in_channels = d->channels;
    e.extra_channels = 1;
    e.n_segments = 1;
    e.seg_channels[0] = d->n_out;
    e.in_stride_b = e.in_stride_t = static_cast<int64_t>(d->channels) * e.pixels;
    e.in_stride_c = e.pixels;
    return e;
}

static fiery_batch_norm_desc_t oh_norm(const fiery_output_head_desc_t* d) {
    fiery_batch_norm_desc_t b{};
    b.batch = d->maps;
    b.channels = d->channels;
    b.frames = 1;
    b.pixels = d->grid_x * d->grid_y;
    b.stride_b = static_cast<int64_t>(d->channels) * b.pixels;
    b.stride_c = b.stride_t = b.pixels;
    b.training = d->training;
    b.relu = 1;
    b.eps = d->eps;
    return b;
}

size_t output_head_packed_bytes(const fiery_output_head_desc_t* d) {
    const fiery_temporal_entry_desc_t e = oh_entry(d);
    return temporal_entry_packed_bytes(&e);
}

int launch_output_head_pack(const fiery_output_head_desc_t* d, const float* w, void* packed, cudaStream_t stream) {
    const fiery_temporal_entry_desc_t e = oh_entry(d);
    return launch_temporal_entry_pack(&e, w, static_cast<float*>(packed), stream);
}

// the forward's workspace: the norm's (coefficients first), then the maps' ones
size_t output_head_forward_workspace_bytes(const fiery_output_head_desc_t* d) {
    const fiery_batch_norm_desc_t b = oh_norm(d);
    return oh_align(batch_norm_workspace_bytes(&b)) + oh_align(static_cast<size_t>(d->maps) * sizeof(float));
}

__global__ void oh_ones_kernel(float* __restrict__ p, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = 1.f;
}

int launch_output_head_forward(const fiery_output_head_desc_t* d, const float* y, const void* packed, const float* bn_w, const float* bn_b,
                               const float* running_mean, const float* running_var, float* out, float* mean, float* var, void* workspace,
                               cudaStream_t stream) {
    const fiery_temporal_entry_desc_t e = oh_entry(d);
    const fiery_batch_norm_desc_t b = oh_norm(d);
    float* ones = reinterpret_cast<float*>(static_cast<char*>(workspace) + oh_align(batch_norm_workspace_bytes(&b)));
    oh_ones_kernel<<<(d->maps + 255) / 256, 256, 0, stream>>>(ones, d->maps);
    FIERY_CUDA_CHECK(cudaGetLastError());
    int rc = launch_batch_norm_coef(&b, y, bn_w, bn_b, running_mean, running_var, mean, var, workspace, stream);
    if (rc == FIERY_OK)
        rc = launch_output_head_entry_forward(&e, y, ones, static_cast<const float*>(packed), static_cast<const BnCoef*>(workspace), out,
                                              stream);
    return rc;
}

size_t output_head_backward_workspace_bytes(const fiery_output_head_desc_t* d) {
    const fiery_batch_norm_desc_t b = oh_norm(d);
    return output_head_backward_workspace_bytes(&b, d->n_out);
}

// w1: the fp32 (n, C) weight, so da is the fp32 product
int launch_output_head_backward(const fiery_output_head_desc_t* d, const float* grad_out, const float* y, const float* mean, const float* var,
                                const float* w1, const float* bn_w, const float* bn_b, float* grad_y, float* grad_bn_w, float* grad_bn_b,
                                float* grad_w, float* grad_b, void* workspace, cudaStream_t stream) {
    const fiery_batch_norm_desc_t b = oh_norm(d);
    return launch_output_head_backward(&b, y, grad_out, w1, d->channels, d->n_out, bn_w, bn_b, mean, var, grad_y, grad_bn_w, grad_bn_b,
                                       grad_w, grad_b, workspace, stream);
}

}  // namespace fiery
