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
int launch_batch_norm_local_stats(const fiery_batch_norm_desc_t* d, const float* x, double* stats, void* workspace, cudaStream_t stream);
int launch_batch_norm_forward_gathered(const fiery_batch_norm_desc_t* d, int world, const double* gathered, const float* x, const float* w,
                                       const float* bias, const float* residual, float* y, float* mean_out, float* var_out,
                                       double* count_out, void* workspace, cudaStream_t stream);
int launch_batch_norm_local_grad_sums(const fiery_batch_norm_desc_t* d, const float* x, const float* dy, const float* w, const float* bias,
                                      const float* mean, const float* var, double* sums, float* grad_w, float* grad_b, void* workspace,
                                      cudaStream_t stream);
int launch_batch_norm_backward_gathered(const fiery_batch_norm_desc_t* d, int world, const double* gathered, const float* x, const float* dy,
                                        const float* w, const float* bias, const float* mean, const float* var, float* dx, void* workspace,
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

// The forward's operands as the launches below take them: the descriptors, each convolution's pack, the coefficients at the
// workspace's start (launch_batch_norm_coef's and launch_batch_norm_coef_gathered's) and each norm's mean and var in stats
struct BkFwd {
    BkDescs s;
    const float *p_down, *p_conv, *p_up;
    const BnCoef* coef;
    float *mean[3], *var[3];
};
static BkFwd bk_fwd(const fiery_bottleneck_desc_t* d, const void* packed, float* stats, void* workspace) {
    BkFwd f;
    f.s = bk_descs(d);
    const BkPack p = bk_pack(f.s);
    const char* pk = static_cast<const char*>(packed);
    f.p_down = reinterpret_cast<const float*>(pk + p.down);
    f.p_conv = reinterpret_cast<const float*>(pk + p.conv);
    f.p_up = reinterpret_cast<const float*>(pk + p.up);
    f.coef = static_cast<const BnCoef*>(workspace);
    const int M = f.s.M;
    f.mean[0] = stats, f.mean[1] = stats + 2 * M, f.mean[2] = stats + 4 * M;
    f.var[0] = f.mean[0] + M, f.var[1] = f.mean[1] + M, f.var[2] = f.mean[2] + f.s.C;
    return f;
}

int launch_bottleneck_forward(const fiery_bottleneck_desc_t* d, const float* x, const void* packed, const float* const* norms, float* y1,
                              float* y2, float* y3, float* out, float* stats, void* workspace, cudaStream_t stream) {
    const BkFwd f = bk_fwd(d, packed, stats, workspace);
    const BkDescs& s = f.s;
    auto nrm = [&](int i, int j) { return norms[4 * i + j]; };
    int rc = launch_temporal_entry_forward(&s.down, x, nullptr, f.p_down, &y1, stream);
    if (rc == FIERY_OK)
        rc = launch_batch_norm_coef(&s.bn[0], y1, nrm(0, 0), nrm(0, 1), nrm(0, 2), nrm(0, 3), f.mean[0], f.var[0], workspace, stream);
    if (rc == FIERY_OK) rc = launch_bottleneck_conv_forward(&s.conv, y1, f.p_conv, f.coef, y2, stream);
    if (rc == FIERY_OK)
        rc = launch_batch_norm_coef(&s.bn[1], y2, nrm(1, 0), nrm(1, 1), nrm(1, 2), nrm(1, 3), f.mean[1], f.var[1], workspace, stream);
    if (rc == FIERY_OK) rc = launch_bottleneck_entry_forward(&s.up, y2, f.p_up, f.coef, y3, stream);
    if (rc == FIERY_OK)
        rc = launch_batch_norm_forward(&s.bn[2], y3, nrm(2, 0), nrm(2, 1), nrm(2, 2), nrm(2, 3), x, out, f.mean[2], f.var[2], workspace,
                                       stream);
    return rc;
}

// The forward with each norm's statistics over a group, split at the norms: stage k (0..2) ends with this rank's (n, mean, M2) of
// y_{k+1} in `local`, stage k (1..3) starts with norm k's gathered finalize.  The convolutions and the last apply are the launches
// above, on the same coefficients.
int launch_bottleneck_sync_forward_stage(const fiery_bottleneck_desc_t* d, int stage, int world, const double* gathered, const float* x,
                                         const void* packed, const float* const* norms, float* y1, float* y2, float* y3, float* out,
                                         float* stats, double* counts, double* local, void* workspace, cudaStream_t stream) {
    const BkFwd f = bk_fwd(d, packed, stats, workspace);
    const BkDescs& s = f.s;
    auto nrm = [&](int i, int j) { return norms[4 * i + j]; };
    float* const y[3] = {y1, y2, y3};
    int rc = FIERY_OK;
    if (stage == 1 || stage == 2) {
        const int i = stage - 1;
        rc = launch_batch_norm_coef_gathered(&s.bn[i], world, gathered, nrm(i, 0), nrm(i, 1), f.mean[i], f.var[i], counts + i, workspace,
                                             stream);
    }
    if (rc == FIERY_OK && stage == 0) rc = launch_temporal_entry_forward(&s.down, x, nullptr, f.p_down, &y1, stream);
    if (rc == FIERY_OK && stage == 1) rc = launch_bottleneck_conv_forward(&s.conv, y1, f.p_conv, f.coef, y2, stream);
    if (rc == FIERY_OK && stage == 2) rc = launch_bottleneck_entry_forward(&s.up, y2, f.p_up, f.coef, y3, stream);
    if (rc == FIERY_OK && stage < 3) rc = launch_batch_norm_local_stats(&s.bn[stage], y[stage], local, workspace, stream);
    if (rc == FIERY_OK && stage == 3)
        rc = launch_batch_norm_forward_gathered(&s.bn[2], world, gathered, y3, nrm(2, 0), nrm(2, 1), x, out, f.mean[2], f.var[2], counts + 2,
                                                workspace, stream);
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

// The backward's operands, and what each stage is needed for (a gradient below it), from the gradients asked for
struct BkBwd {
    BkDescs s;
    const float *p_down, *p_conv, *p_up;
    float *dy3, *buf_a, *buf_b, *scratch;
    void *bn_ws, *coef_ws, *wg_ws;
    const float *mean[3], *var[3];
    fiery_batch_norm_desc_t eval_bn;
    bool need_n1, need_dy1, need_da1, need_dy2, need_da2;
};
static BkBwd bk_bwd(const fiery_bottleneck_desc_t* d, const float* stats, const void* packed, float* grad_x, float* grad_w_down,
                    float* grad_w_conv, float* const* grad_norms, void* workspace) {
    BkBwd b;
    b.s = bk_descs(d);
    const BkPack p = bk_pack(b.s);
    const BkBwdWork w = bk_bwd_work(b.s, d->maps);
    char* ws = static_cast<char*>(workspace);
    const char* pk = static_cast<const char*>(packed);
    b.p_down = reinterpret_cast<const float*>(pk + p.down);
    b.p_conv = reinterpret_cast<const float*>(pk + p.conv);
    b.p_up = reinterpret_cast<const float*>(pk + p.up);
    b.dy3 = reinterpret_cast<float*>(ws + w.dy3);
    b.buf_a = reinterpret_cast<float*>(ws + w.a);
    b.buf_b = reinterpret_cast<float*>(ws + w.b);
    b.bn_ws = ws + w.bn;
    b.coef_ws = ws + w.coef;
    b.scratch = reinterpret_cast<float*>(ws + w.scratch);
    b.wg_ws = ws + w.wgrad;
    const int M = b.s.M;
    b.mean[0] = stats, b.mean[1] = stats + 2 * M, b.mean[2] = stats + 4 * M;
    b.var[0] = b.mean[0] + M, b.var[1] = b.mean[1] + M, b.var[2] = b.mean[2] + b.s.C;
    b.eval_bn = b.s.bn[1];
    b.eval_bn.training = 0;
    b.eval_bn.batch = b.eval_bn.pixels = 1;
    b.need_n1 = grad_norms[0] || grad_norms[1];
    b.need_dy1 = grad_x || grad_w_down;
    b.need_da1 = b.need_dy1 || b.need_n1;
    b.need_dy2 = b.need_da1 || grad_w_conv;
    b.need_da2 = b.need_dy2 || grad_norms[2] || grad_norms[3];
    return b;
}

// from dy3: grad_w_up (bn2's prologue on y2) and da2 = W_up^T dy3 into buf_a, each when needed
static int bk_bwd_up(const BkBwd& b, const float* y2, const float* const* norms, float* grad_w_up, cudaStream_t stream) {
    int rc = FIERY_OK;
    if (grad_w_up) {
        rc = launch_batch_norm_coef(&b.eval_bn, nullptr, norms[4], norms[5], b.mean[1], b.var[1], b.scratch, b.scratch + b.s.M, b.coef_ws,
                                    stream);
        if (rc == FIERY_OK)
            rc = launch_bottleneck_entry_wgrad(&b.s.up, y2, static_cast<const BnCoef*>(b.coef_ws), b.dy3, grad_w_up, b.wg_ws, stream);
    }
    if (rc == FIERY_OK && b.need_da2) rc = launch_temporal_entry_dgrad(&b.s.up, &b.dy3, b.p_up, nullptr, b.buf_a, stream);
    return rc;
}

// from dy2 in buf_b: grad_w_conv (bn1's prologue on y1) and da1 = the 3x3 input gradient into buf_a, each when needed
static int bk_bwd_conv(const BkBwd& b, const float* y1, const float* const* norms, float* grad_w_conv, cudaStream_t stream) {
    int rc = FIERY_OK;
    if (grad_w_conv) {
        rc = launch_batch_norm_coef(&b.eval_bn, nullptr, norms[0], norms[1], b.mean[0], b.var[0], b.scratch, b.scratch + b.s.M, b.coef_ws,
                                    stream);
        if (rc == FIERY_OK)
            rc = launch_bottleneck_conv_wgrad(&b.s.conv, y1, static_cast<const BnCoef*>(b.coef_ws), b.buf_b, grad_w_conv, b.wg_ws, stream);
    }
    if (rc == FIERY_OK && b.need_da1) rc = launch_causal_conv_dgrad(&b.s.conv, b.buf_b, b.p_conv, b.buf_a, stream);
    return rc;
}

// from dy1 in buf_b: grad_w_down and grad_x = W_down^T dy1 + grad_out, each when asked for
static int bk_bwd_down(const BkBwd& b, const float* x, const float* grad_out, float* grad_w_down, float* grad_x, cudaStream_t stream) {
    const float* dy1 = b.buf_b;
    int rc = FIERY_OK;
    if (grad_w_down) rc = launch_temporal_entry_wgrad(&b.s.down, x, nullptr, &dy1, grad_w_down, b.wg_ws, stream);
    if (rc == FIERY_OK && grad_x) rc = launch_bottleneck_entry_dgrad(&b.s.down, dy1, b.p_down, grad_out, grad_x, stream);
    return rc;
}

int launch_bottleneck_backward(const fiery_bottleneck_desc_t* d, const float* grad_out, const float* x, const float* y1, const float* y2,
                               const float* y3, const float* stats, const void* packed, const float* const* norms, float* grad_x,
                               float* grad_w_down, float* grad_w_conv, float* grad_w_up, float* const* grad_norms, void* workspace,
                               cudaStream_t stream) {
    const BkBwd b = bk_bwd(d, stats, packed, grad_x, grad_w_down, grad_w_conv, grad_norms, workspace);
    auto nrm = [&](int i, int j) { return norms[4 * i + j]; };
    auto gn = [&](int i, int j) { return grad_norms[2 * i + j]; };
    int rc = launch_batch_norm_backward(&b.s.bn[2], y3, grad_out, nrm(2, 0), nrm(2, 1), b.mean[2], b.var[2], b.dy3, gn(2, 0), gn(2, 1),
                                        b.bn_ws, stream);
    if (rc == FIERY_OK) rc = bk_bwd_up(b, y2, norms, grad_w_up, stream);
    if (rc == FIERY_OK && b.need_da2)
        rc = launch_batch_norm_backward(&b.s.bn[1], y2, b.buf_a, nrm(1, 0), nrm(1, 1), b.mean[1], b.var[1], b.need_dy2 ? b.buf_b : nullptr,
                                        gn(1, 0), gn(1, 1), b.bn_ws, stream);
    if (rc == FIERY_OK) rc = bk_bwd_conv(b, y1, norms, grad_w_conv, stream);
    if (rc == FIERY_OK && b.need_da1)
        rc = launch_batch_norm_backward(&b.s.bn[0], y1, b.buf_a, nrm(0, 0), nrm(0, 1), b.mean[0], b.var[0], b.need_dy1 ? b.buf_b : nullptr,
                                        gn(0, 0), gn(0, 1), b.bn_ws, stream);
    if (rc == FIERY_OK) rc = bk_bwd_down(b, x, grad_out, grad_w_down, grad_x, stream);
    return rc;
}

// The backward with each norm's gradient sums over a group, split at the norms (norm 3, 2, 1 in stages 0, 1, 2): stage k (0..2) ends
// with this rank's (n, S1, S2) of its norm in `local` and the norm's own weight and bias gradients; stage k (1..3) starts with that
// norm's gathered backward, into the buffer the single-rank chain above writes, then runs the same launches up to the next norm.
int launch_bottleneck_sync_backward_stage(const fiery_bottleneck_desc_t* d, int stage, int world, const double* gathered,
                                          const float* grad_out, const float* x, const float* y1, const float* y2, const float* y3,
                                          const float* stats, const void* packed, const float* const* norms, float* grad_x,
                                          float* grad_w_down, float* grad_w_conv, float* grad_w_up, float* const* grad_norms, double* local,
                                          void* workspace, cudaStream_t stream) {
    const BkBwd b = bk_bwd(d, stats, packed, grad_x, grad_w_down, grad_w_conv, grad_norms, workspace);
    auto nrm = [&](int i, int j) { return norms[4 * i + j]; };
    auto gn = [&](int i, int j) { return grad_norms[2 * i + j]; };
    int rc = FIERY_OK;
    switch (stage) {
    case 0:
        rc = launch_batch_norm_local_grad_sums(&b.s.bn[2], y3, grad_out, nrm(2, 0), nrm(2, 1), b.mean[2], b.var[2], local, gn(2, 0),
                                               gn(2, 1), b.bn_ws, stream);
        break;
    case 1:
        rc = launch_batch_norm_backward_gathered(&b.s.bn[2], world, gathered, y3, grad_out, nrm(2, 0), nrm(2, 1), b.mean[2], b.var[2],
                                                 b.dy3, b.bn_ws, stream);
        if (rc == FIERY_OK) rc = bk_bwd_up(b, y2, norms, grad_w_up, stream);
        if (rc == FIERY_OK && b.need_da2)
            rc = launch_batch_norm_local_grad_sums(&b.s.bn[1], y2, b.buf_a, nrm(1, 0), nrm(1, 1), b.mean[1], b.var[1], local, gn(1, 0),
                                                   gn(1, 1), b.bn_ws, stream);
        break;
    case 2:
        if (!b.need_dy2) break;
        rc = launch_batch_norm_backward_gathered(&b.s.bn[1], world, gathered, y2, b.buf_a, nrm(1, 0), nrm(1, 1), b.mean[1], b.var[1],
                                                 b.buf_b, b.bn_ws, stream);
        if (rc == FIERY_OK) rc = bk_bwd_conv(b, y1, norms, grad_w_conv, stream);
        if (rc == FIERY_OK && b.need_da1)
            rc = launch_batch_norm_local_grad_sums(&b.s.bn[0], y1, b.buf_a, nrm(0, 0), nrm(0, 1), b.mean[0], b.var[0], local, gn(0, 0),
                                                   gn(0, 1), b.bn_ws, stream);
        break;
    default:
        if (!b.need_dy1) break;
        rc = launch_batch_norm_backward_gathered(&b.s.bn[0], world, gathered, y1, b.buf_a, nrm(0, 0), nrm(0, 1), b.mean[0], b.var[0],
                                                 b.buf_b, b.bn_ws, stream);
        if (rc == FIERY_OK) rc = bk_bwd_down(b, x, grad_out, grad_w_down, grad_x, stream);
    }
    return rc;
}

}  // namespace fiery
