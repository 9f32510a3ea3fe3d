// The batch norm's per-channel apply coefficients (batch_norm.cu), and the BN + ReLU prologue the Bottleneck's convolutions apply to
// their operand as they read it (temporal_entry.cu, causal_conv.cu, driven by bottleneck.cu).
#pragma once
#include "common.cuh"

namespace fiery {

// Per-channel coefficients the finalize writes for the apply passes.  Forward: y = fmaf(scale, x, shift).  Backward:
// dx = fmaf(scale, g', fmaf(k1, x - mean, k0)) in training, scale * g' in eval.
struct BnCoef {
    float scale, shift, mean, k1, k0;
};

// max(fmaf(scale, v, shift), 0): bit for bit the value bn_apply_kernel<RELU = true, RESIDUAL = false> writes (a NaN passes)
__device__ __forceinline__ float bn_relu_apply(const BnCoef& k, float v) {
    const float o = fmaf(k.scale, v, k.shift);
    return o < 0.f ? 0.f : o;
}

// The forward's statistics (mean_out, var_out) and apply coefficients of x, without the apply pass: the batch's in training, the
// running ones in eval (fiery_batch_norm_forward's first two steps).  The coefficients are at the start of the workspace
// (batch_norm_workspace_bytes(d) bytes) and stay valid until the next launch that uses it.
int launch_batch_norm_coef(const fiery_batch_norm_desc_t* d, const float* x, const float* w, const float* bias, const float* running_mean,
                           const float* running_var, float* mean_out, float* var_out, void* workspace, cudaStream_t stream);
size_t batch_norm_workspace_bytes(const fiery_batch_norm_desc_t* d);

// The same from a group's gathered (world, channels, 3) (n, mean, M2) triplets (fiery_batch_norm_forward_gathered without the apply
// pass): the group's statistics, count_out[0] = the group's n (may be NULL) and the coefficients at the start of the workspace.
int launch_batch_norm_coef_gathered(const fiery_batch_norm_desc_t* d, int world, const double* gathered, const float* w, const float* bias,
                                    float* mean_out, float* var_out, double* count_out, void* workspace, cudaStream_t stream);

}  // namespace fiery
