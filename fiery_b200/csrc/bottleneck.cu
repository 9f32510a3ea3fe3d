// The future prediction's Bottleneck (fiery/layers/convolutions.py:64-168, the plain variant) as one chain of the project's kernels
// (include/fiery_b200.h, fiery_bottleneck_*), on `maps` (X, Y) maps with C channels and M = C / 2:
//
//   y1 = W_down x                       temporal entry forward (batch = maps, frames = 1)
//   k1 = bn1's coefficients of y1       batch-norm statistics and finalize, no apply pass
//   y2 = conv3x3(relu(fmaf(k1, y1)))    the 3x3 forward with its BN + ReLU prologue on the landed halo
//   k2 = bn2's coefficients of y2
//   y3 = W_up relu(fmaf(k2, y2))        the entry forward with its BN + ReLU prologue on the A fragments
//   out = relu(bn3(y3)) + x             batch-norm forward with ReLU and residual
//
// so a1 = relu(bn1(y1)) and a2 = relu(bn2(y2)) never reach memory.  The backward runs the chain in reverse on y1, y2, y3 only:
// bn3's backward -> dy3; dW_up from the entry weight gradient with the bn2 prologue on its x tile; da2 = W_up^T dy3; bn2's backward
// -> dy2; dW_conv from the 3x3 weight gradient with the bn1 prologue on its x run; da1 = the 3x3 input gradient; bn1's backward -> dy1;
// dW_down; dx = W_down^T dy1 + grad_out in the entry input gradient's epilogue.  Every reduction is one of the reused kernels', so
// everything stays bit-reproducible, graph-capturable and free of atomics and host synchronisation.
#include "bn_coef.cuh"

namespace fiery {

size_t temporal_entry_packed_bytes(const fiery_temporal_entry_desc_t* d);
int launch_temporal_entry_pack(const fiery_temporal_entry_desc_t* d, const float* w, float* packed, cudaStream_t stream);
int launch_temporal_entry_forward(const fiery_temporal_entry_desc_t* d, const float* x, const float* extra, const float* packed,
                                  float* const* out, cudaStream_t stream);
int launch_temporal_entry_dgrad(const fiery_temporal_entry_desc_t* d, const float* const* gy, const float* packed, const float* bias,
                                float* gx, cudaStream_t stream);
size_t temporal_entry_wgrad_workspace_bytes(const fiery_temporal_entry_desc_t* d);
int launch_temporal_entry_wgrad(const fiery_temporal_entry_desc_t* d, const float* x, const float* extra, const float* const* gy,
                                float* gw, void* workspace, cudaStream_t stream);
int launch_bottleneck_entry_forward(const fiery_temporal_entry_desc_t* d, const float* x, const float* packed, const BnCoef* coef, float* out,
                                    cudaStream_t stream);
int launch_bottleneck_entry_dgrad(const fiery_temporal_entry_desc_t* d, const float* gy, const float* packed, const float* res, float* gx,
                                  cudaStream_t stream);
int launch_bottleneck_entry_wgrad(const fiery_temporal_entry_desc_t* d, const float* x, const BnCoef* coef, const float* gy, float* gw,
                                  void* workspace, cudaStream_t stream);
size_t causal_conv_packed_bytes(const fiery_causal_conv3d_desc_t* d);
int launch_causal_conv_pack(const fiery_causal_conv3d_desc_t* d, const float* w, float* packed, cudaStream_t stream);
int launch_causal_conv_dgrad(const fiery_causal_conv3d_desc_t* d, const float* gy, const float* packed, float* gx, cudaStream_t stream);
size_t causal_conv_wgrad_workspace_bytes(const fiery_causal_conv3d_desc_t* d);
int launch_bottleneck_conv_forward(const fiery_causal_conv3d_desc_t* d, const float* x, const float* packed, const BnCoef* coef, float* y,
                                   cudaStream_t stream);
int launch_bottleneck_conv_wgrad(const fiery_causal_conv3d_desc_t* d, const float* x, const BnCoef* coef, const float* gy, float* gw,
                                 void* workspace, cudaStream_t stream);
int launch_batch_norm_forward(const fiery_batch_norm_desc_t* d, const float* x, const float* w, const float* bias, const float* running_mean,
                              const float* running_var, const float* residual, float* y, float* mean_out, float* var_out,
                              void* workspace, cudaStream_t stream);
int launch_batch_norm_backward(const fiery_batch_norm_desc_t* d, const float* x, const float* dy, const float* w, const float* bias,
                               const float* mean, const float* var, float* dx, float* grad_w, float* grad_b, void* workspace,
                               cudaStream_t stream);

static size_t bk_align(size_t v) { return (v + 255) / 256 * 256; }

// The three stages' descriptors: the 1x1 convolutions as temporal entries over (batch = maps, frames = 1), the 3x3 as a causal
// convolution with kt = 1, the norms over (maps, channels, 1, X, Y) contiguous.
struct BkDescs {
    int C, M;
    long long P;
    fiery_temporal_entry_desc_t down, up;
    fiery_causal_conv3d_desc_t conv;
    fiery_batch_norm_desc_t bn[3];
};

static fiery_temporal_entry_desc_t bk_entry(const fiery_bottleneck_desc_t* d, int K, int n_out) {
    fiery_temporal_entry_desc_t e{};
    e.batch = d->maps;
    e.frames = 1;
    e.pixels = d->grid_x * d->grid_y;
    e.in_channels = K;
    e.n_segments = 1;
    e.seg_channels[0] = n_out;
    e.in_stride_b = e.in_stride_t = static_cast<int64_t>(K) * e.pixels;
    e.in_stride_c = e.pixels;
    return e;
}

static BkDescs bk_descs(const fiery_bottleneck_desc_t* d) {
    BkDescs s;
    s.C = d->channels;
    s.M = d->channels / 2;
    s.P = static_cast<long long>(d->grid_x) * d->grid_y;
    s.down = bk_entry(d, s.C, s.M);
    s.up = bk_entry(d, s.M, s.C);
    s.conv = fiery_causal_conv3d_desc_t{d->maps, 1, d->grid_x, d->grid_y, s.M, s.M, 1};
    const int ch[3] = {s.M, s.M, s.C};
    for (int i = 0; i < 3; ++i) {
        fiery_batch_norm_desc_t& b = s.bn[i];
        b.batch = d->maps;
        b.channels = ch[i];
        b.frames = 1;
        b.pixels = static_cast<int32_t>(s.P);
        b.stride_b = ch[i] * s.P;
        b.stride_c = b.stride_t = s.P;
        b.training = d->training;
        b.relu = 1;
        b.eps = d->eps;
    }
    return s;
}

// the pack: the down projection's entry pack, the 3x3's causal-conv pack, the up projection's entry pack, each 256-byte aligned
struct BkPack {
    size_t down, conv, up, bytes;
};
static BkPack bk_pack(const BkDescs& s) {
    BkPack p;
    p.down = 0;
    p.conv = bk_align(temporal_entry_packed_bytes(&s.down));
    p.up = p.conv + bk_align(causal_conv_packed_bytes(&s.conv));
    p.bytes = p.up + bk_align(temporal_entry_packed_bytes(&s.up));
    return p;
}

size_t bottleneck_packed_bytes(const fiery_bottleneck_desc_t* d) { return bk_pack(bk_descs(d)).bytes; }

int launch_bottleneck_pack(const fiery_bottleneck_desc_t* d, const float* w_down, const float* w_conv, const float* w_up, void* packed,
                           cudaStream_t stream) {
    const BkDescs s = bk_descs(d);
    const BkPack p = bk_pack(s);
    char* base = static_cast<char*>(packed);
    int rc = launch_temporal_entry_pack(&s.down, w_down, reinterpret_cast<float*>(base + p.down), stream);
    if (rc == FIERY_OK) rc = launch_causal_conv_pack(&s.conv, w_conv, reinterpret_cast<float*>(base + p.conv), stream);
    if (rc == FIERY_OK) rc = launch_temporal_entry_pack(&s.up, w_up, reinterpret_cast<float*>(base + p.up), stream);
    return rc;
}

// the largest batch-norm workspace of the three norms (the workspace holds the coefficients, then the pieces' partials)
static size_t bk_bn_bytes(const BkDescs& s) {
    size_t b = 0;
    for (int i = 0; i < 3; ++i) b = b > batch_norm_workspace_bytes(&s.bn[i]) ? b : batch_norm_workspace_bytes(&s.bn[i]);
    return bk_align(b);
}

size_t bottleneck_forward_workspace_bytes(const fiery_bottleneck_desc_t* d) { return bk_bn_bytes(bk_descs(d)); }

int launch_bottleneck_forward(const fiery_bottleneck_desc_t* d, const float* x, const void* packed, const float* const* norms, float* y1,
                              float* y2, float* y3, float* out, float* stats, void* workspace, cudaStream_t stream) {
    const BkDescs s = bk_descs(d);
    const BkPack p = bk_pack(s);
    const char* pk = static_cast<const char*>(packed);
    const BnCoef* coef = static_cast<const BnCoef*>(workspace);      // launch_batch_norm_coef's coefficients: the workspace's start
    float* mean[3] = {stats, stats + 2 * s.M, stats + 4 * s.M};
    auto nrm = [&](int i, int j) { return norms[4 * i + j]; };
    int rc = launch_temporal_entry_forward(&s.down, x, nullptr, reinterpret_cast<const float*>(pk + p.down), &y1, stream);
    if (rc == FIERY_OK)
        rc = launch_batch_norm_coef(&s.bn[0], y1, nrm(0, 0), nrm(0, 1), nrm(0, 2), nrm(0, 3), mean[0], mean[0] + s.M, workspace, stream);
    if (rc == FIERY_OK) rc = launch_bottleneck_conv_forward(&s.conv, y1, reinterpret_cast<const float*>(pk + p.conv), coef, y2, stream);
    if (rc == FIERY_OK)
        rc = launch_batch_norm_coef(&s.bn[1], y2, nrm(1, 0), nrm(1, 1), nrm(1, 2), nrm(1, 3), mean[1], mean[1] + s.M, workspace, stream);
    if (rc == FIERY_OK) rc = launch_bottleneck_entry_forward(&s.up, y2, reinterpret_cast<const float*>(pk + p.up), coef, y3, stream);
    if (rc == FIERY_OK)
        rc = launch_batch_norm_forward(&s.bn[2], y3, nrm(2, 0), nrm(2, 1), nrm(2, 2), nrm(2, 3), x, out, mean[2], mean[2] + s.C, workspace,
                                       stream);
    return rc;
}

// The backward's workspace: dy3 (maps, C, P); two (maps, M, P) buffers (da2 then da1, and dy2 then dy1); the batch norms' workspace;
// the forward coefficients of bn2, then bn1, recomputed from the saved statistics for the weight gradients' prologues (an eval-mode
// finalize: the same fp64 formula the forward's finalize ran on the same fp32 mean and var) with the scratch statistics they copy;
// and the largest of the three weight gradients' workspaces.
struct BkBwdWork {
    size_t dy3, a, b, bn, coef, scratch, wgrad, bytes;
};
static BkBwdWork bk_bwd_work(const BkDescs& s, int maps) {
    BkBwdWork w;
    const size_t nm = static_cast<size_t>(maps) * s.P;
    fiery_batch_norm_desc_t one = s.bn[1];
    one.batch = one.pixels = 1;
    one.training = 0;
    w.dy3 = 0;
    w.a = bk_align(nm * s.C * 4);
    w.b = w.a + bk_align(nm * s.M * 4);
    w.bn = w.b + bk_align(nm * s.M * 4);
    w.coef = w.bn + bk_bn_bytes(s);
    w.scratch = w.coef + bk_align(batch_norm_workspace_bytes(&one));
    w.wgrad = w.scratch + bk_align(2 * s.M * 4);
    size_t wg = temporal_entry_wgrad_workspace_bytes(&s.down);
    wg = wg > temporal_entry_wgrad_workspace_bytes(&s.up) ? wg : temporal_entry_wgrad_workspace_bytes(&s.up);
    wg = wg > causal_conv_wgrad_workspace_bytes(&s.conv) ? wg : causal_conv_wgrad_workspace_bytes(&s.conv);
    w.bytes = w.wgrad + bk_align(wg);
    return w;
}

size_t bottleneck_backward_workspace_bytes(const fiery_bottleneck_desc_t* d) { return bk_bwd_work(bk_descs(d), d->maps).bytes; }

int launch_bottleneck_backward(const fiery_bottleneck_desc_t* d, const float* grad_out, const float* x, const float* y1, const float* y2,
                               const float* y3, const float* stats, const void* packed, const float* const* norms, float* grad_x,
                               float* grad_w_down, float* grad_w_conv, float* grad_w_up, float* const* grad_norms, void* workspace,
                               cudaStream_t stream) {
    const BkDescs s = bk_descs(d);
    const BkPack p = bk_pack(s);
    const BkBwdWork w = bk_bwd_work(s, d->maps);
    char* ws = static_cast<char*>(workspace);
    float* dy3 = reinterpret_cast<float*>(ws + w.dy3);
    float* buf_a = reinterpret_cast<float*>(ws + w.a);
    float* buf_b = reinterpret_cast<float*>(ws + w.b);
    void* bn_ws = ws + w.bn;
    void* coef_ws = ws + w.coef;
    const BnCoef* coef = static_cast<const BnCoef*>(coef_ws);
    float* scratch = reinterpret_cast<float*>(ws + w.scratch);
    void* wg_ws = ws + w.wgrad;
    const char* pk = static_cast<const char*>(packed);
    const float* mean[3] = {stats, stats + 2 * s.M, stats + 4 * s.M};
    const float* var[3] = {mean[0] + s.M, mean[1] + s.M, mean[2] + s.C};
    auto nrm = [&](int i, int j) { return norms[4 * i + j]; };
    auto gn = [&](int i, int j) { return grad_norms[2 * i + j]; };
    // what each stage is needed for: a gradient below it
    const bool need_n1 = gn(0, 0) || gn(0, 1);
    const bool need_dy1 = grad_x || grad_w_down;
    const bool need_da1 = need_dy1 || need_n1;
    const bool need_dy2 = need_da1 || grad_w_conv;
    const bool need_da2 = need_dy2 || gn(1, 0) || gn(1, 1);
    fiery_batch_norm_desc_t eval_bn = s.bn[1];
    eval_bn.training = 0;
    eval_bn.batch = eval_bn.pixels = 1;

    int rc = launch_batch_norm_backward(&s.bn[2], y3, grad_out, nrm(2, 0), nrm(2, 1), mean[2], var[2], dy3, gn(2, 0), gn(2, 1), bn_ws, stream);
    if (rc == FIERY_OK && grad_w_up) {
        rc = launch_batch_norm_coef(&eval_bn, nullptr, nrm(1, 0), nrm(1, 1), mean[1], var[1], scratch, scratch + s.M, coef_ws, stream);
        if (rc == FIERY_OK) rc = launch_bottleneck_entry_wgrad(&s.up, y2, coef, dy3, grad_w_up, wg_ws, stream);
    }
    if (rc == FIERY_OK && need_da2)
        rc = launch_temporal_entry_dgrad(&s.up, &dy3, reinterpret_cast<const float*>(pk + p.up), nullptr, buf_a, stream);
    if (rc == FIERY_OK && need_da2)
        rc = launch_batch_norm_backward(&s.bn[1], y2, buf_a, nrm(1, 0), nrm(1, 1), mean[1], var[1], need_dy2 ? buf_b : nullptr, gn(1, 0),
                                        gn(1, 1), bn_ws, stream);
    if (rc == FIERY_OK && grad_w_conv) {
        rc = launch_batch_norm_coef(&eval_bn, nullptr, nrm(0, 0), nrm(0, 1), mean[0], var[0], scratch, scratch + s.M, coef_ws, stream);
        if (rc == FIERY_OK) rc = launch_bottleneck_conv_wgrad(&s.conv, y1, coef, buf_b, grad_w_conv, wg_ws, stream);
    }
    if (rc == FIERY_OK && need_da1) rc = launch_causal_conv_dgrad(&s.conv, buf_b, reinterpret_cast<const float*>(pk + p.conv), buf_a, stream);
    if (rc == FIERY_OK && need_da1)
        rc = launch_batch_norm_backward(&s.bn[0], y1, buf_a, nrm(0, 0), nrm(0, 1), mean[0], var[0], need_dy1 ? buf_b : nullptr, gn(0, 0),
                                        gn(0, 1), bn_ws, stream);
    const float* dy1 = buf_b;
    if (rc == FIERY_OK && grad_w_down) rc = launch_temporal_entry_wgrad(&s.down, x, nullptr, &dy1, grad_w_down, wg_ws, stream);
    if (rc == FIERY_OK && grad_x)
        rc = launch_bottleneck_entry_dgrad(&s.down, dy1, reinterpret_cast<const float*>(pk + p.down), grad_out, grad_x, stream);
    return rc;
}

}  // namespace fiery
