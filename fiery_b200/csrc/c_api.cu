// extern "C" boundary of libfiery_b200.so (declared in include/fiery_b200.h).  Argument validation, TMA descriptor
// creation and launch dispatch; no torch types, no host<->device copies except where the header says so.
#include <initializer_list>
#include <stdarg.h>
#include <string.h>

#include "lift_plan.cuh"

namespace fiery {

static thread_local char g_last_error[512] = "";

int set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
    va_end(ap);
    return code;
}

int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, int rank, const void* base, const cuuint64_t* dims,
                      const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* elem_strides,
                      CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2_promotion, const char* what) {
    // cuTensorMapEncodeTiled is a driver call and needs a current context; a thread that has made no runtime call yet
    // (e.g. the autograd engine's worker on its first backward) has none, so bind the primary context once per thread.
    static thread_local bool ctx_bound = false;
    if (!ctx_bound) {
        cudaFree(nullptr);
        ctx_bound = true;
    }
    static const auto encode = []() -> decltype(&cuTensorMapEncodeTiled) {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return nullptr;
        return reinterpret_cast<decltype(&cuTensorMapEncodeTiled)>(sym);
    }();
    if (!encode) return set_error(FIERY_E_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    static const cuuint32_t unit[5] = {1, 1, 1, 1, 1};
    const CUresult r = encode(map, dtype, static_cast<cuuint32_t>(rank), const_cast<void*>(base), dims, strides_bytes, box,
                              elem_strides ? elem_strides : unit, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2_promotion,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(FIERY_E_CUDA, "cuTensorMapEncodeTiled (%s) failed with CUresult %d", what, (int)r);
    return FIERY_OK;
}

// Tensor maps of the lift's tile kernels (lift_tile.cuh: HeadMapsCols)
int encode_head_maps_cols(HeadMapsCols* maps, const void* head, const LiftParams& P, int channels_per_lane) {
    const size_t es = 4;
    // the image coordinate of a tile is absolute (frame0 * n_cameras + ...): the map spans every image up to this launch's last
    const cuuint64_t ww = P.ww, hh = P.hh, n_images = static_cast<cuuint64_t>(P.frame0 + P.n_frames) * P.n_cameras;
    const cuuint64_t plane = ww * hh * es, image = plane * P.head_channels;
    FIERY_REQUIRE((reinterpret_cast<uintptr_t>(head) & 15) == 0 && (plane * (P.use_depth ? P.D : 0)) % 16 == 0,
                  "head tensor (or its context slice) is not 16-byte aligned");
    const int cpl = channels_per_lane;
    FIERY_REQUIRE(cpl >= 1 && P.C % cpl == 0 && P.C / cpl <= 256 && hh <= 256, "column kernel: unsupported head shape");
    if (P.use_depth) {
        cuuint64_t dims[4] = {ww, static_cast<cuuint64_t>(P.D), hh, n_images};
        cuuint64_t strides[3] = {plane, ww * es, image};
        cuuint32_t box[4] = {WT, 48, static_cast<cuuint32_t>(hh), 1};
        const int rc = encode_tensor_map(&maps->depth, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, head, dims, strides, box, nullptr,
                                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "depth, 4-D");
        if (rc != FIERY_OK) return rc;
    } else {
        memset(&maps->depth, 0, sizeof(CUtensorMap));
    }
    const char* ctx_base = static_cast<const char*>(head) + plane * (P.use_depth ? P.D : 0);
    cuuint64_t dims[5] = {ww, static_cast<cuuint64_t>(P.C / cpl), static_cast<cuuint64_t>(cpl), hh, n_images};
    cuuint64_t strides[4] = {cpl * plane, plane, ww * es, image};
    cuuint32_t box[5] = {WT, static_cast<cuuint32_t>(P.C / cpl), static_cast<cuuint32_t>(cpl), static_cast<cuuint32_t>(hh), 1};
    return encode_tensor_map(&maps->ctx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, ctx_base, dims, strides, box, nullptr,
                             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "context, 5-D");
}

// NCHW output (frames, C, X*Y) as a 3-D map, innermost the pillar axis; the layout pass stores (box_pillars x C) blocks into it
int encode_bev_map(CUtensorMap* map, float* bev, long long pillars, int channels, int n_frames, int box_pillars) {
    FIERY_REQUIRE((reinterpret_cast<uintptr_t>(bev) & 15) == 0 && pillars % 4 == 0, "BEV output is not 16-byte aligned / pitched");
    FIERY_REQUIRE(channels <= 256 && box_pillars <= 256, "BEV map: box too large");
    cuuint64_t dims[3] = {static_cast<cuuint64_t>(pillars), static_cast<cuuint64_t>(channels), static_cast<cuuint64_t>(n_frames)};
    cuuint64_t strides[2] = {static_cast<cuuint64_t>(pillars) * 4, static_cast<cuuint64_t>(pillars) * channels * 4};
    cuuint32_t box[3] = {static_cast<cuuint32_t>(box_pillars), static_cast<cuuint32_t>(channels), 1};
    return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, bev, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_NONE,
                             CU_TENSOR_MAP_L2_PROMOTION_NONE, "BEV output");
}

// Head shapes the lift's kernels are built for.  The plan needs rows and depth bins that fit a tile record; the forward and backward
// tile kernels also need 64 channels and a 16-byte row pitch for their tensor maps.  The entry points check the shape once, after
// their 0-frame return; the launchers behind them rely on it.
int check_lift_geometry(const LiftParams& P) {
    FIERY_REQUIRE(P.hh >= 1 && P.hh <= PLAN_MAX_ROWS, "feat_h=%d not supported by this build (<= %d)", P.hh, PLAN_MAX_ROWS);
    FIERY_REQUIRE(P.D >= 1 && P.D <= DPAD, "depth_bins=%d not supported by this build (1..48)", P.D);
    return FIERY_OK;
}
static int check_lift_tile_shape(const LiftParams& P) {
    FIERY_REQUIRE(P.C == 64, "channels=%d not supported by this build (C must be 64)", P.C);
    FIERY_REQUIRE(P.ww % 4 == 0, "feat_w=%d must be a multiple of 4 (TMA row pitch must be 16-byte aligned)", P.ww);
    return check_lift_geometry(P);
}

// launchers defined next to their kernels (the lift's: lift_plan.cuh)
int launch_warp(int forward, int n_maps, int C, int H, int W, const float* a, long long a_stride, const float* theta,
                const unsigned char* copy_mask, float* b, long long b_stride, int nearest, cudaStream_t stream);
int launch_warp_theta(int n_seq, int T, int cumulative, const float* flow, float ex, float ey, float* theta,
                      unsigned char* copy_mask, cudaStream_t stream);
int launch_pack_conv_weights(const float* w_oihw, float* packed, cudaStream_t stream);
int launch_bev_conv(int n_frames, int H, int W, const float* x_nhwc, const float* w_packed, const float* scale, const float* shift,
                    int relu, float* y_nhwc, cudaStream_t stream);
int launch_pack_conv_weights_transposed(const float* w_oihw, float* packed, cudaStream_t stream);
int launch_bev_conv_dgrad(int n_frames, int H, int W, const float* gy_nhwc, const float* w_packed_t, float* gx_nhwc, cudaStream_t stream);
size_t bev_conv_wgrad_workspace_bytes(int n_frames, int H, int W);
int launch_bev_conv_wgrad(int n_frames, int H, int W, const float* x_nhwc, const float* gy_nhwc, float* dw_oihw, void* workspace,
                          cudaStream_t stream);
int launch_depth_layer(int n_images, int pixels, int n_out, const void* feat, int dtype, const void* weight_padded, const float* bias,
                       float* head, cudaStream_t stream);
size_t temporal_entry_packed_bytes(const fiery_temporal_entry_desc_t* d);
int launch_temporal_entry_pack(const fiery_temporal_entry_desc_t* d, const float* w, float* packed, cudaStream_t stream);
int launch_temporal_entry_forward(const fiery_temporal_entry_desc_t* d, const float* x, const float* extra, const float* packed,
                                  float* const* out, cudaStream_t stream);
int launch_temporal_entry_dgrad(const fiery_temporal_entry_desc_t* d, const float* const* gy, const float* packed, const float* bias,
                                float* gx, cudaStream_t stream);
int launch_spatial_sums(const fiery_spatial_sums_desc_t* d, const float* x, float* sums, cudaStream_t stream);
size_t temporal_entry_wgrad_workspace_bytes(const fiery_temporal_entry_desc_t* d);
int launch_temporal_entry_wgrad(const fiery_temporal_entry_desc_t* d, const float* x, const float* extra, const float* const* gy,
                                float* gw, void* workspace, cudaStream_t stream);
size_t causal_conv_packed_bytes(const fiery_causal_conv3d_desc_t* d);
size_t conv3x3_packed_bytes(const fiery_conv3x3_desc_t* d);
int launch_conv3x3_pack(const fiery_conv3x3_desc_t* d, const float* w, float* packed, cudaStream_t stream);
int launch_conv3x3(const fiery_conv3x3_desc_t* d, int dgrad, const float* in0, const float* in1, const float* packed, float* out0,
                   float* out1, cudaStream_t stream);
size_t conv3x3_wgrad_workspace_bytes(const fiery_conv3x3_desc_t* d);
int launch_conv3x3_wgrad(const fiery_conv3x3_desc_t* d, const float* x0, const float* x1, const float* gy, float* gw, void* workspace,
                         cudaStream_t stream);
size_t spatial_gru_packed_bytes(const fiery_spatial_gru_desc_t* d);
int launch_spatial_gru_pack(const fiery_spatial_gru_desc_t* d, const float* w_gates, const float* w_state, float* packed, cudaStream_t stream);
size_t spatial_gru_forward_workspace_bytes(const fiery_spatial_gru_desc_t* d);
int launch_spatial_gru_forward(const fiery_spatial_gru_desc_t* d, const float* x, const float* h0, const float* packed, const float* b_gates,
                               const float* bn_w, const float* bn_b, const float* running_mean, const float* running_var, float* out,
                               float* saved, float* means, float* vars, void* workspace, cudaStream_t stream);
size_t spatial_gru_backward_workspace_bytes(const fiery_spatial_gru_desc_t* d);
int launch_spatial_gru_backward(const fiery_spatial_gru_desc_t* d, const float* grad_out, const float* x, const float* h0, const float* out,
                                const float* saved_c, const float* means, const float* vars, const float* packed, const float* bn_w,
                                const float* bn_b, float* grad_x, float* grad_h0, float* grad_w_gates, float* grad_b_gates,
                                float* grad_w_state, float* grad_bn_w, float* grad_bn_b, void* workspace, cudaStream_t stream);
size_t batch_norm_workspace_bytes(const fiery_batch_norm_desc_t* d);
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
int launch_spatial_gru_forward_step_begin(const fiery_spatial_gru_desc_t* d, int t, const float* x, const float* h0, const float* packed,
                                          const float* b_gates, const float* out, float* saved, double* stats, void* workspace,
                                          cudaStream_t stream);
int launch_spatial_gru_forward_step_end(const fiery_spatial_gru_desc_t* d, int t, int world, const double* gathered, const float* h0,
                                        const float* bn_w, const float* bn_b, float* out, const float* saved_c, float* means, float* vars,
                                        double* count_out, void* workspace, cudaStream_t stream);
int launch_spatial_gru_backward_step_begin(const fiery_spatial_gru_desc_t* d, int t, const float* grad_out, const float* h0, const float* out,
                                           const float* saved_c, const float* means, const float* vars, const float* packed,
                                           const float* bn_w, const float* bn_b, float* grad_h0, double* sums, void* workspace,
                                           cudaStream_t stream);
int launch_spatial_gru_backward_step_end(const fiery_spatial_gru_desc_t* d, int t, int world, const double* gathered, const float* h0,
                                         const float* out, const float* saved_c, const float* means, const float* vars, const float* packed,
                                         const float* bn_w, const float* bn_b, float* grad_x, float* grad_h0, void* workspace,
                                         cudaStream_t stream);
int launch_spatial_gru_backward_weights(const fiery_spatial_gru_desc_t* d, const float* x, const float* h0, const float* out, const float* saved_c,
                                        const float* packed, float* grad_w_gates, float* grad_b_gates, float* grad_w_state, float* grad_bn_w,
                                        float* grad_bn_b, void* workspace, cudaStream_t stream);
int launch_causal_conv_pack(const fiery_causal_conv3d_desc_t* d, const float* w, float* packed, cudaStream_t stream);
size_t bottleneck_packed_bytes(const fiery_bottleneck_desc_t* d);
int launch_bottleneck_pack(const fiery_bottleneck_desc_t* d, const float* w_down, const float* w_conv, const float* w_up, void* packed,
                           cudaStream_t stream);
size_t bottleneck_forward_workspace_bytes(const fiery_bottleneck_desc_t* d);
int launch_bottleneck_forward(const fiery_bottleneck_desc_t* d, const float* x, const void* packed, const float* const* norms, float* y1,
                              float* y2, float* y3, float* out, float* stats, void* workspace, cudaStream_t stream);
size_t bottleneck_backward_workspace_bytes(const fiery_bottleneck_desc_t* d);
int launch_bottleneck_backward(const fiery_bottleneck_desc_t* d, const float* grad_out, const float* x, const float* y1, const float* y2,
                               const float* y3, const float* stats, const void* packed, const float* const* norms, float* grad_x,
                               float* grad_w_down, float* grad_w_conv, float* grad_w_up, float* const* grad_norms, void* workspace,
                               cudaStream_t stream);
int launch_bottleneck_sync_forward_stage(const fiery_bottleneck_desc_t* d, int stage, int world, const double* gathered, const float* x,
                                         const void* packed, const float* const* norms, float* y1, float* y2, float* y3, float* out,
                                         float* stats, double* counts, double* local, void* workspace, cudaStream_t stream);
int launch_bottleneck_sync_backward_stage(const fiery_bottleneck_desc_t* d, int stage, int world, const double* gathered,
                                          const float* grad_out, const float* x, const float* y1, const float* y2, const float* y3,
                                          const float* stats, const void* packed, const float* const* norms, float* grad_x,
                                          float* grad_w_down, float* grad_w_conv, float* grad_w_up, float* const* grad_norms, double* local,
                                          void* workspace, cudaStream_t stream);
size_t output_head_packed_bytes(const fiery_output_head_desc_t* d);
int launch_output_head_pack(const fiery_output_head_desc_t* d, const float* w, void* packed, cudaStream_t stream);
size_t output_head_forward_workspace_bytes(const fiery_output_head_desc_t* d);
int launch_output_head_forward(const fiery_output_head_desc_t* d, const float* y, const void* packed, const float* bn_w, const float* bn_b,
                               const float* running_mean, const float* running_var, float* out, float* mean, float* var, void* workspace,
                               cudaStream_t stream);
size_t output_head_backward_workspace_bytes(const fiery_output_head_desc_t* d);
int launch_output_head_backward(const fiery_output_head_desc_t* d, const float* grad_out, const float* y, const float* mean, const float* var,
                                const float* w1, const float* bn_w, const float* bn_b, float* grad_y, float* grad_bn_w, float* grad_bn_b,
                                float* grad_w, float* grad_b, void* workspace, cudaStream_t stream);
int launch_causal_conv_forward(const fiery_causal_conv3d_desc_t* d, const float* x, const float* packed, float* y, cudaStream_t stream);
int launch_causal_conv_dgrad(const fiery_causal_conv3d_desc_t* d, const float* gy, const float* packed, float* gx, cudaStream_t stream);
size_t causal_conv_wgrad_workspace_bytes(const fiery_causal_conv3d_desc_t* d);
int launch_causal_conv_wgrad(const fiery_causal_conv3d_desc_t* d, const float* x, const float* gy, float* gw, void* workspace,
                             cudaStream_t stream);
int vs_plan(int64_t n_rows, const int64_t* ranks, int32_t* seg, int64_t* host_n, cudaStream_t);
int vs_forward(int64_t n_rows, int channels, int64_t feat_stride, const float* feats, const int64_t* coords,
               const int32_t* seg, int64_t n_seg, float* sums, int64_t* coords_out, cudaStream_t);
int vs_backward(int64_t n_rows, int channels, const float* grad_sums, const int32_t* seg, float* grad_feats, cudaStream_t);
size_t vs_det_workspace_bytes(int64_t n_rows, int channels);
int vs_forward_det(int64_t n_rows, int channels, int64_t feat_stride, const float* feats, const int64_t* coords, const int32_t* seg,
                   float* sums, int64_t* coords_out, float* edge, cudaStream_t);

// shape-only parameters for the size queries (no pointers); false for a descriptor they answer 0 for
static bool shape_params(const fiery_lift_desc_t* d, LiftParams& P) {
    if (!d || d->n_frames < 0 || d->n_cameras < 1 || d->feat_w < 1 || d->bev_x < 1 || d->bev_y < 1) return false;
    P = LiftParams{};
    P.n_frames = d->n_frames; P.n_cameras = d->n_cameras; P.C = d->channels; P.D = d->depth_bins;
    P.hh = d->feat_h; P.ww = d->feat_w;
    P.n_wtiles = (d->feat_w + WT - 1) / WT;
    P.bev_layout = d->bev_layout;
    P.pillars = static_cast<long long>(d->bev_x) * d->bev_y;
    return true;
}

static int make_params(const fiery_lift_desc_t* d, const float* calib_a, const float* calib_b, const float* fu,
                       const float* fv, const float* fd, LiftParams& P) {
    FIERY_REQUIRE(d != nullptr, "desc is NULL");
    FIERY_REQUIRE(d->n_frames >= 0 && d->n_cameras >= 1, "bad n_frames=%d / n_cameras=%d", d->n_frames, d->n_cameras);
    FIERY_REQUIRE(d->depth_bins >= 1 && d->channels >= 1 && d->feat_h >= 1 && d->feat_w >= 1,
                  "bad head shape D=%d C=%d h=%d w=%d", d->depth_bins, d->channels, d->feat_h, d->feat_w);
    FIERY_REQUIRE(d->bev_x >= 1 && d->bev_y >= 1, "bad BEV size %dx%d", d->bev_x, d->bev_y);
    // the reference squeezes the Z axis and assigns into (C, X, Y) (fiery.py:268-271): only one height cell works
    FIERY_REQUIRE(d->bev_z == 1, "bev_z=%d: the reference path only supports a single height cell (fiery.py:269)", d->bev_z);
    FIERY_REQUIRE(static_cast<long long>(d->bev_x) * d->bev_y < (1ll << 31), "BEV grid too large");
    FIERY_REQUIRE(d->calib_mode == FIERY_CALIB_RAW || d->calib_mode == FIERY_CALIB_COMPOSED, "bad calib_mode %d", d->calib_mode);
    FIERY_REQUIRE(d->bev_layout == FIERY_BEV_NCHW || d->bev_layout == FIERY_BEV_NHWC, "bad bev_layout %d", d->bev_layout);
    FIERY_REQUIRE(d->n_frames == 0 || (calib_a && calib_b), "calibration pointer is NULL");
    FIERY_REQUIRE(fu && fv && fd, "frustum pointer is NULL");
    for (int a = 0; a < 3; ++a) FIERY_REQUIRE(d->bev_resolution[a] > 0.f, "bev_resolution[%d] must be positive", a);
    shape_params(d, P);                              // accepts every descriptor that passed the checks above
    P.use_depth = d->use_depth_distribution ? 1 : 0;
    P.head_channels = d->channels + (P.use_depth ? d->depth_bins : 0);
    P.calib_mode = d->calib_mode;
    P.calib_a = calib_a; P.calib_b = calib_b; P.fu = fu; P.fv = fv; P.fd = fd;
    P.grid = make_grid_params(*d);
    return FIERY_OK;
}

// The body of the three forward entry points: `launch` is the default or the deterministic launcher, `buffer` its scratch or
// workspace; `warped` (fiery_lift_forward_warped) requires theta and copy_mask, the others take both or neither.
static int lift_forward(decltype(&launch_lift_forward) launch, const fiery_lift_desc_t* desc, const void* head, const float* calib_a,
                        const float* calib_b, const float* fu, const float* fv, const float* fd, float* bev_out, void* buffer,
                        const void* plan, const float* theta, const uint8_t* copy_mask, bool warped, void* stream) {
    LiftParams P;
    int rc = make_params(desc, calib_a, calib_b, fu, fv, fd, P);
    if (rc != FIERY_OK) return rc;
    if (P.n_frames == 0) return FIERY_OK;
    if (warped) FIERY_REQUIRE(head && bev_out && theta && copy_mask, "head / bev_out / theta / copy_mask is NULL");
    FIERY_REQUIRE(head && bev_out, "head / bev_out is NULL");
    FIERY_REQUIRE((theta == nullptr) == (copy_mask == nullptr), "theta and copy_mask go together (the warped lift) or are both NULL");
    FIERY_REQUIRE(!theta || desc->bev_layout == FIERY_BEV_NCHW, "the warped lift writes the NCHW layout only");
    FIERY_REQUIRE(desc->head_dtype == FIERY_DTYPE_F32 || desc->head_dtype == FIERY_DTYPE_F16, "head dtype %d not supported (fp32 / fp16)",
                  desc->head_dtype);
    rc = check_lift_tile_shape(P);
    if (rc != FIERY_OK) return rc;
    return launch(P, head, desc->head_dtype, bev_out, buffer, plan, theta, copy_mask, static_cast<cudaStream_t>(stream));
}

}  // namespace fiery

using namespace fiery;

extern "C" {

FIERY_API int fiery_abi_version(void) { return FIERY_B200_ABI_VERSION; }

FIERY_API const char* fiery_last_error(void) { return g_last_error; }

FIERY_API size_t fiery_lift_plan_bytes(const fiery_lift_desc_t* d) {
    LiftParams P;
    if (!shape_params(d, P) || P.n_frames == 0) return 0;
    return plan_bytes(P.n_frames, P.n_cameras, P.n_wtiles, P.pillars);
}

FIERY_API int fiery_lift_plan(const fiery_lift_desc_t* desc, const float* calib_a, const float* calib_b, const float* frustum_u,
                              const float* frustum_v, const float* frustum_d, void* plan_out, void* stream) {
    LiftParams P;
    int rc = make_params(desc, calib_a, calib_b, frustum_u, frustum_v, frustum_d, P);
    if (rc != FIERY_OK) return rc;
    if (P.n_frames == 0) return FIERY_OK;
    FIERY_REQUIRE(plan_out != nullptr, "plan_out is NULL");
    const PlanView v = plan_view(plan_out, P.n_frames, P.n_cameras, P.n_wtiles, P.pillars, 0);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    FIERY_CUDA_CHECK(cudaMemsetAsync(const_cast<unsigned char*>(v.touched), 0, static_cast<size_t>(P.n_frames) * P.pillars, st));
    return launch_lift_plan(P, const_cast<unsigned char*>(v.tiles), const_cast<unsigned char*>(v.touched), 1, st);
}

FIERY_API size_t fiery_lift_scratch_bytes(const fiery_lift_desc_t* d) {
    LiftParams P;
    if (!shape_params(d, P) || P.n_frames == 0) return 0;
    return lift_scratch_bytes(P);
}

FIERY_API void fiery_lift_set_max_chunk_frames(int32_t n) { lift_set_max_chunk_frames(n); }

FIERY_API int fiery_lift_forward_launches(const fiery_lift_desc_t* d) {
    LiftParams P;
    if (!shape_params(d, P) || P.n_frames == 0) return 0;
    return lift_forward_launches(P);
}

FIERY_API size_t fiery_lift_workspace_bytes(const fiery_lift_desc_t* d) {
    LiftParams P;
    if (!shape_params(d, P) || P.n_frames == 0) return 0;
    const size_t relayout = (lift_backward_relayout_bytes(P) + 127) & ~static_cast<size_t>(127);
    return relayout + static_cast<size_t>(P.n_frames) * P.n_cameras * P.n_wtiles * PLAN_TILE_BYTES;
}

FIERY_API int fiery_lift_forward(const fiery_lift_desc_t* desc, const void* head, const float* calib_a, const float* calib_b,
                       const float* frustum_u, const float* frustum_v, const float* frustum_d, float* bev_out,
                       void* scratch, const void* plan, void* stream) {
    return lift_forward(launch_lift_forward, desc, head, calib_a, calib_b, frustum_u, frustum_v, frustum_d, bev_out, scratch, plan,
                        nullptr, nullptr, false, stream);
}

FIERY_API int fiery_lift_forward_warped(const fiery_lift_desc_t* desc, const void* head, const float* calib_a, const float* calib_b,
                                        const float* frustum_u, const float* frustum_v, const float* frustum_d, float* bev_out,
                                        void* scratch, const void* plan, const float* theta, const uint8_t* copy_mask, void* stream) {
    return lift_forward(launch_lift_forward, desc, head, calib_a, calib_b, frustum_u, frustum_v, frustum_d, bev_out, scratch, plan,
                        theta, copy_mask, true, stream);
}

FIERY_API size_t fiery_lift_deterministic_workspace_bytes(const fiery_lift_desc_t* d) {
    LiftParams P;
    if (!shape_params(d, P) || P.n_frames == 0) return 0;
    return lift_det_workspace_bytes(P);
}

FIERY_API int fiery_lift_forward_deterministic(const fiery_lift_desc_t* desc, const void* head, const float* calib_a,
                                               const float* calib_b, const float* frustum_u, const float* frustum_v,
                                               const float* frustum_d, float* bev_out, void* workspace, const void* plan,
                                               const float* theta, const uint8_t* copy_mask, void* stream) {
    return lift_forward(launch_lift_forward_det, desc, head, calib_a, calib_b, frustum_u, frustum_v, frustum_d, bev_out, workspace,
                        plan, theta, copy_mask, false, stream);
}

FIERY_API int fiery_lift_forward_timed(const fiery_lift_desc_t* desc, const void* head, const float* calib_a, const float* calib_b,
                                       const float* frustum_u, const float* frustum_v, const float* frustum_d, float* bev_out,
                                       void* scratch, const void* plan, void* stream, int32_t max_launches, float* host_ms,
                                       int32_t* host_kind, int32_t* host_n_launches) {
    FIERY_REQUIRE(host_ms && host_kind && host_n_launches && max_launches >= 1, "timed forward: NULL output / no room");
    LaunchTimer t;
    t.cap = max_launches < LaunchTimer::MAX ? max_launches : LaunchTimer::MAX;
    for (int i = 0; i < 2 * t.cap; ++i) FIERY_CUDA_CHECK(cudaEventCreate(&t.ev[i]));
    lift_set_timer(&t);
    const int rc = fiery_lift_forward(desc, head, calib_a, calib_b, frustum_u, frustum_v, frustum_d, bev_out, scratch, plan, stream);
    lift_set_timer(nullptr);
    cudaError_t e = cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
    *host_n_launches = t.n;
    for (int i = 0; i < t.n && rc == FIERY_OK && e == cudaSuccess; ++i) {
        host_kind[i] = t.kind[i];
        e = cudaEventElapsedTime(&host_ms[i], t.ev[2 * i], t.ev[2 * i + 1]);
    }
    for (int i = 0; i < 2 * t.cap; ++i) cudaEventDestroy(t.ev[i]);
    if (rc != FIERY_OK) return rc;
    FIERY_CUDA_CHECK(e);
    return FIERY_OK;
}

FIERY_API int fiery_lift_backward(const fiery_lift_desc_t* desc, const void* head, const float* calib_a, const float* calib_b,
                        const float* frustum_u, const float* frustum_v, const float* frustum_d, const float* grad_bev,
                        void* grad_head, float* workspace, const void* plan, void* stream) {
    LiftParams P;
    int rc = make_params(desc, calib_a, calib_b, frustum_u, frustum_v, frustum_d, P);
    if (rc != FIERY_OK) return rc;
    if (P.n_frames == 0) return FIERY_OK;
    FIERY_REQUIRE(head && grad_bev && grad_head, "head / grad_bev / grad_head is NULL");
    P.grad_bev = grad_bev;
    P.grad_head = static_cast<float*>(grad_head);
    FIERY_REQUIRE(workspace != nullptr || (desc->bev_layout == FIERY_BEV_NHWC && plan != nullptr),
                  "backward needs the workspace of fiery_lift_workspace_bytes() (NCHW grad_bev re-layout and/or the geometry plan)");
    FIERY_REQUIRE(desc->head_dtype == FIERY_DTYPE_F32, "head dtype %d not supported by this build (fp32 only)", desc->head_dtype);
    rc = check_lift_tile_shape(P);
    if (rc != FIERY_OK) return rc;
    return launch_lift_backward(P, head, workspace, plan, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_lift_point_indices(const fiery_lift_desc_t* desc, const float* calib_a, const float* calib_b,
                             const float* frustum_u, const float* frustum_v, const float* frustum_d, int64_t* idx_out,
                             uint8_t* valid_out, int32_t* pillar_out, void* stream) {
    LiftParams P;
    int rc = make_params(desc, calib_a, calib_b, frustum_u, frustum_v, frustum_d, P);
    if (rc != FIERY_OK) return rc;
    return launch_point_indices(P, idx_out, valid_out, pillar_out, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_compose_calibration(int32_t n, const float* intrinsics, const float* extrinsics, float* combined_out,
                              float* translation_out, void* stream) {
    FIERY_REQUIRE(n >= 0, "n_matrices=%d", n);
    FIERY_REQUIRE(n == 0 || (intrinsics && extrinsics && combined_out && translation_out), "NULL pointer");
    return launch_compose(n, intrinsics, extrinsics, combined_out, translation_out, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_voxels_summing_plan(int64_t n_rows, const int64_t* ranks, int32_t* segment_of_row, int64_t* host_n_segments,
                              void* stream) {
    FIERY_REQUIRE(n_rows >= 0 && n_rows < (1ll << 31), "n_rows=%lld out of range", (long long)n_rows);
    FIERY_REQUIRE(host_n_segments != nullptr, "host_n_segments is NULL");
    if (n_rows == 0) { *host_n_segments = 0; return FIERY_OK; }
    FIERY_REQUIRE(ranks && segment_of_row, "NULL pointer");
    return vs_plan(n_rows, ranks, segment_of_row, host_n_segments, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_voxels_summing_forward(int64_t n_rows, int32_t channels, int64_t feat_stride, const float* feats,
                                 const int64_t* coords, const int32_t* segment_of_row, int64_t n_segments,
                                 float* sums_out, int64_t* coords_out, void* stream) {
    FIERY_REQUIRE(n_rows >= 0 && channels >= 1 && feat_stride >= channels, "bad shape n_rows=%lld C=%d stride=%lld",
                  (long long)n_rows, channels, (long long)feat_stride);
    if (n_rows == 0) return FIERY_OK;
    FIERY_REQUIRE(feats && coords && segment_of_row && sums_out && coords_out, "NULL pointer");
    return vs_forward(n_rows, channels, feat_stride, feats, coords, segment_of_row, n_segments, sums_out, coords_out,
                      static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_voxels_summing_deterministic_workspace_bytes(int64_t n_rows, int32_t channels) {
    if (n_rows <= 0 || channels < 1) return 0;
    return vs_det_workspace_bytes(n_rows, channels);
}

FIERY_API int fiery_voxels_summing_forward_deterministic(int64_t n_rows, int32_t channels, int64_t feat_stride, const float* feats,
                                                         const int64_t* coords, const int32_t* segment_of_row, int64_t n_segments,
                                                         float* sums_out, int64_t* coords_out, void* workspace, void* stream) {
    FIERY_REQUIRE(n_rows >= 0 && channels >= 1 && feat_stride >= channels, "bad shape n_rows=%lld C=%d stride=%lld",
                  (long long)n_rows, channels, (long long)feat_stride);
    if (n_rows == 0) return FIERY_OK;
    FIERY_REQUIRE(feats && coords && segment_of_row && sums_out && coords_out, "NULL pointer");
    FIERY_REQUIRE(workspace != nullptr, "NULL workspace (fiery_voxels_summing_deterministic_workspace_bytes)");
    (void)n_segments;
    return vs_forward_det(n_rows, channels, feat_stride, feats, coords, segment_of_row, sums_out, coords_out,
                          static_cast<float*>(workspace), static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_voxels_summing_backward(int64_t n_rows, int32_t channels, const float* grad_sums, const int32_t* segment_of_row,
                                  float* grad_feats, void* stream) {
    FIERY_REQUIRE(n_rows >= 0 && channels >= 1, "bad shape");
    if (n_rows == 0) return FIERY_OK;
    FIERY_REQUIRE(grad_sums && segment_of_row && grad_feats, "NULL pointer");
    return vs_backward(n_rows, channels, grad_sums, segment_of_row, grad_feats, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_warp_features_forward(int32_t n_maps, int32_t channels, int32_t height, int32_t width, const float* x,
                                          int64_t x_map_stride, const float* theta, const uint8_t* copy_mask, float* out,
                                          int64_t out_map_stride, int32_t nearest, void* stream) {
    FIERY_REQUIRE(n_maps >= 0 && channels >= 1 && height >= 1 && width >= 1, "warp: bad shape");
    FIERY_REQUIRE(n_maps == 0 || (x && theta && out), "warp: NULL pointer");
    return launch_warp(1, n_maps, channels, height, width, x, x_map_stride, theta, copy_mask, out, out_map_stride, nearest ? 1 : 0,
                       static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_warp_features_backward(int32_t n_maps, int32_t channels, int32_t height, int32_t width, const float* grad_out,
                                           int64_t grad_out_map_stride, const float* theta, const uint8_t* copy_mask,
                                           float* grad_x, int64_t grad_x_map_stride, int32_t nearest, void* stream) {
    FIERY_REQUIRE(n_maps >= 0 && channels >= 1 && height >= 1 && width >= 1, "warp: bad shape");
    FIERY_REQUIRE(n_maps == 0 || (grad_out && theta && grad_x), "warp: NULL pointer");
    return launch_warp(0, n_maps, channels, height, width, grad_out, grad_out_map_stride, theta, copy_mask, grad_x, grad_x_map_stride,
                       nearest ? 1 : 0, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_warp_theta(int32_t n_sequences, int32_t T, int32_t cumulative, const float* flow, float spatial_extent_x,
                               float spatial_extent_y, float* theta, uint8_t* copy_mask, void* stream) {
    FIERY_REQUIRE(n_sequences >= 0 && (!cumulative || T >= 1), "warp_theta: bad shape");
    FIERY_REQUIRE(n_sequences == 0 || (flow && theta && (copy_mask || !cumulative)), "warp_theta: NULL pointer");
    return launch_warp_theta(n_sequences, T, cumulative ? 1 : 0, flow, spatial_extent_x, spatial_extent_y, theta, copy_mask,
                             static_cast<cudaStream_t>(stream));
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

FIERY_API int fiery_bev_conv_pack_weights(const float* weight_oihw, float* packed_out, void* stream) {
    FIERY_REQUIRE(weight_oihw && packed_out, "bev conv: NULL weight pointer");
    return launch_pack_conv_weights(weight_oihw, packed_out, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_bev_first_conv_forward(int32_t n_frames, int32_t height, int32_t width, const float* x_nhwc, const float* packed_weight,
                                           const float* scale, const float* shift, int32_t relu, float* y_nhwc, void* stream) {
    FIERY_REQUIRE(n_frames == 0 || (x_nhwc && packed_weight && y_nhwc), "bev conv: NULL pointer");
    FIERY_REQUIRE(n_frames >= 0 && height >= 1 && width >= 1, "bev conv: bad shape %d x %d x %d", n_frames, height, width);
    if (n_frames == 0) return FIERY_OK;
    FIERY_REQUIRE((scale == nullptr) == (shift == nullptr), "bev conv: scale and shift go together");
    FIERY_REQUIRE(aligned16(x_nhwc) && aligned16(packed_weight) && aligned16(y_nhwc), "bev conv: pointers must be 16-byte aligned");
    return launch_bev_conv(n_frames, height, width, x_nhwc, packed_weight, scale, shift, relu ? 1 : 0, y_nhwc, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_bev_conv_pack_weights_transposed(const float* weight_oihw, float* packed_out, void* stream) {
    FIERY_REQUIRE(weight_oihw && packed_out, "bev conv: NULL weight pointer");
    return launch_pack_conv_weights_transposed(weight_oihw, packed_out, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_bev_first_conv_backward_data(int32_t n_frames, int32_t height, int32_t width, const float* grad_y_nhwc,
                                                 const float* packed_weight_t, float* grad_x_nhwc, void* stream) {
    FIERY_REQUIRE(n_frames >= 0 && height >= 1 && width >= 1, "bev conv backward: bad shape %d x %d x %d", n_frames, height, width);
    if (n_frames == 0) return FIERY_OK;
    FIERY_REQUIRE(grad_y_nhwc && packed_weight_t && grad_x_nhwc, "bev conv backward: NULL pointer");
    FIERY_REQUIRE(aligned16(grad_y_nhwc) && aligned16(packed_weight_t) && aligned16(grad_x_nhwc),
                  "bev conv backward: pointers must be 16-byte aligned");
    return launch_bev_conv_dgrad(n_frames, height, width, grad_y_nhwc, packed_weight_t, grad_x_nhwc, static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_bev_first_conv_backward_weight_workspace_bytes(int32_t n_frames, int32_t height, int32_t width) {
    return bev_conv_wgrad_workspace_bytes(n_frames, height, width);
}

FIERY_API int fiery_bev_first_conv_backward_weight(int32_t n_frames, int32_t height, int32_t width, const float* x_nhwc,
                                                   const float* grad_y_nhwc, float* grad_weight_oihw, void* workspace, void* stream) {
    FIERY_REQUIRE(n_frames >= 0 && height >= 1 && width >= 1, "bev conv backward: bad shape %d x %d x %d", n_frames, height, width);
    FIERY_REQUIRE(grad_weight_oihw, "bev conv backward: NULL grad_weight");
    FIERY_REQUIRE(aligned16(grad_weight_oihw), "bev conv backward: pointers must be 16-byte aligned");
    if (n_frames > 0) {
        FIERY_REQUIRE(x_nhwc && grad_y_nhwc && workspace, "bev conv backward: NULL pointer");
        FIERY_REQUIRE(aligned16(x_nhwc) && aligned16(grad_y_nhwc) && aligned16(workspace), "bev conv backward: pointers must be 16-byte aligned");
    }
    return launch_bev_conv_wgrad(n_frames, height, width, x_nhwc, grad_y_nhwc, grad_weight_oihw, workspace, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_depth_layer_forward(int32_t n_images, int32_t pixels, int32_t n_out, const void* feat, int32_t dtype,
                                        const void* weight_padded, const float* bias, float* head_out, void* stream) {
    FIERY_REQUIRE(n_images == 0 || (feat && weight_padded && head_out), "depth layer: NULL pointer");
    // 128 = DL_M (depth_layer.cu): the rows of the padded weight matrix
    FIERY_REQUIRE(n_images >= 0 && pixels >= 1 && n_out >= 1 && n_out <= 128, "depth layer: bad shape (%d images, %d pixels, %d outputs)",
                  n_images, pixels, n_out);
    FIERY_REQUIRE(dtype >= 0 && dtype <= 2, "depth layer: dtype %d not supported (0 fp32, 1 fp16, 2 bf16)", dtype);
    if (n_images == 0) return FIERY_OK;
    FIERY_REQUIRE((static_cast<long long>(pixels) * (dtype == 0 ? 4 : 2)) % 16 == 0 && pixels % 4 == 0,
                  "depth layer: h*w = %d must give a 16-byte row pitch (and a multiple of 4)", pixels);
    FIERY_REQUIRE(aligned16(feat) && aligned16(weight_padded) && aligned16(head_out), "depth layer: pointers must be 16-byte aligned");
    return launch_depth_layer(n_images, pixels, n_out, feat, dtype, weight_padded, bias, head_out, static_cast<cudaStream_t>(stream));
}

// The temporal entry's shape limits, one place for every entry point.  The messages name the field.
static int check_temporal_entry_desc(const fiery_temporal_entry_desc_t* d) {
    FIERY_REQUIRE(d, "temporal entry: NULL desc");
    FIERY_REQUIRE(d->batch >= 0 && d->frames >= 0, "temporal entry: batch = %d, frames = %d must be >= 0", d->batch, d->frames);
    FIERY_REQUIRE(d->in_channels >= 1 && d->in_channels <= 128, "temporal entry: in_channels K = %d must be in 1..128", d->in_channels);
    FIERY_REQUIRE(d->extra_channels >= 0 && d->extra_channels <= 8, "temporal entry: extra_channels E = %d must be in 0..8",
                  d->extra_channels);
    FIERY_REQUIRE(d->n_segments >= 1 && d->n_segments <= 4, "temporal entry: n_segments = %d must be in 1..4", d->n_segments);
    int n_out = 0, n_pad = 0;
    for (int q = 0; q < d->n_segments; ++q) {
        FIERY_REQUIRE(d->seg_channels[q] >= 1 && d->seg_channels[q] <= 256, "temporal entry: seg_channels[%d] = %d must be in 1..256", q,
                      d->seg_channels[q]);
        n_out += d->seg_channels[q];
        n_pad += (d->seg_channels[q] + 7) / 8 * 8;
    }
    FIERY_REQUIRE(n_out <= 256, "temporal entry: N_out = %d output channels (sum of seg_channels) must be <= 256", n_out);
    FIERY_REQUIRE(n_pad <= 256, "temporal entry: N_out with each segment rounded up to 8 channels = %d must be <= 256", n_pad);
    FIERY_REQUIRE(d->pixels >= 1 && d->pixels % 4 == 0, "temporal entry: pixels X*Y = %d must be a positive multiple of 4 (16-byte TMA pitch)",
                  d->pixels);
    FIERY_REQUIRE(d->in_stride_b >= 0 && d->in_stride_t >= 0 && d->in_stride_c >= 0 && d->in_stride_b % 4 == 0 && d->in_stride_t % 4 == 0 &&
                  d->in_stride_c % 4 == 0, "temporal entry: input strides (%lld, %lld, %lld) must be non-negative multiples of 4 elements",
                  (long long)d->in_stride_b, (long long)d->in_stride_t, (long long)d->in_stride_c);
    return FIERY_OK;
}

FIERY_API size_t fiery_temporal_entry_packed_bytes(const fiery_temporal_entry_desc_t* desc) {
    if (check_temporal_entry_desc(desc) != FIERY_OK) return 0;
    return temporal_entry_packed_bytes(desc);
}

FIERY_API int fiery_temporal_entry_pack_weights(const fiery_temporal_entry_desc_t* desc, const float* weight, void* packed, void* stream) {
    const int rc = check_temporal_entry_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(weight && packed, "temporal entry: NULL weight pointer");
    FIERY_REQUIRE(aligned16(packed), "temporal entry: packed weights must be 16-byte aligned");
    return launch_temporal_entry_pack(desc, weight, static_cast<float*>(packed), static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_temporal_entry_forward(const fiery_temporal_entry_desc_t* desc, const float* x, const float* extra, const void* packed,
                                           float* const* out, void* stream) {
    const int rc = check_temporal_entry_desc(desc);
    if (rc != FIERY_OK) return rc;
    if (desc->batch == 0 || desc->frames == 0) return FIERY_OK;
    FIERY_REQUIRE(x && packed && out && (extra || desc->extra_channels == 0), "temporal entry: NULL pointer");
    FIERY_REQUIRE(aligned16(x) && aligned16(packed), "temporal entry: pointers must be 16-byte aligned");
    for (int q = 0; q < desc->n_segments; ++q) FIERY_REQUIRE(out[q] && aligned16(out[q]), "temporal entry: out[%d] is NULL or misaligned", q);
    return launch_temporal_entry_forward(desc, x, desc->extra_channels ? extra : nullptr, static_cast<const float*>(packed), out,
                                         static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_temporal_entry_backward_data(const fiery_temporal_entry_desc_t* desc, const float* const* grad_out, const void* packed,
                                                 float* grad_x, void* stream) {
    const int rc = check_temporal_entry_desc(desc);
    if (rc != FIERY_OK) return rc;
    if (desc->batch == 0 || desc->frames == 0) return FIERY_OK;
    FIERY_REQUIRE(grad_out && packed && grad_x, "temporal entry: NULL pointer");
    FIERY_REQUIRE(aligned16(packed) && aligned16(grad_x), "temporal entry: pointers must be 16-byte aligned");
    for (int q = 0; q < desc->n_segments; ++q)
        FIERY_REQUIRE(grad_out[q] && aligned16(grad_out[q]), "temporal entry: grad_out[%d] is NULL or misaligned", q);
    return launch_temporal_entry_dgrad(desc, grad_out, static_cast<const float*>(packed), nullptr, grad_x,
                                       static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_temporal_aggregation_forward(const fiery_temporal_entry_desc_t* desc, const float* const* paths, const void* packed,
                                                 const float* bias, float* out, void* stream) {
    const int rc = check_temporal_entry_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(desc->extra_channels == 0, "temporal aggregation: extra_channels = %d must be 0", desc->extra_channels);
    if (desc->batch == 0 || desc->frames == 0) return FIERY_OK;
    FIERY_REQUIRE(paths && packed && out, "temporal aggregation: NULL pointer");
    FIERY_REQUIRE(aligned16(packed) && aligned16(out), "temporal aggregation: pointers must be 16-byte aligned");
    for (int q = 0; q < desc->n_segments; ++q)
        FIERY_REQUIRE(paths[q] && aligned16(paths[q]), "temporal aggregation: paths[%d] is NULL or misaligned", q);
    return launch_temporal_entry_dgrad(desc, paths, static_cast<const float*>(packed), bias, out, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_spatial_sums(const fiery_spatial_sums_desc_t* desc, const float* x, float* sums, void* stream) {
    FIERY_REQUIRE(desc, "spatial sums: NULL desc");
    FIERY_REQUIRE(desc->batch >= 0 && desc->channels >= 0 && desc->frames >= 0,
                  "spatial sums: batch = %d, channels = %d, frames = %d must be >= 0", desc->batch, desc->channels, desc->frames);
    FIERY_REQUIRE(desc->pixels >= 1, "spatial sums: pixels X*Y = %d must be >= 1", desc->pixels);
    FIERY_REQUIRE(desc->stride_b >= 0 && desc->stride_c >= 0 && desc->stride_t >= 0,
                  "spatial sums: strides (%lld, %lld, %lld) must be >= 0", (long long)desc->stride_b, (long long)desc->stride_c,
                  (long long)desc->stride_t);
    if (static_cast<long long>(desc->batch) * desc->channels * desc->frames == 0) return FIERY_OK;
    FIERY_REQUIRE(x && sums, "spatial sums: NULL pointer");
    return launch_spatial_sums(desc, x, sums, static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_temporal_entry_backward_weight_workspace_bytes(const fiery_temporal_entry_desc_t* desc) {
    if (check_temporal_entry_desc(desc) != FIERY_OK) return 0;
    return temporal_entry_wgrad_workspace_bytes(desc);
}

FIERY_API int fiery_temporal_entry_backward_weight(const fiery_temporal_entry_desc_t* desc, const float* x, const float* extra,
                                                   const float* const* grad_out, float* grad_w, void* workspace, void* stream) {
    const int rc = check_temporal_entry_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(grad_w, "temporal entry: NULL grad_w");
    if (desc->batch > 0 && desc->frames > 0) {
        FIERY_REQUIRE(x && grad_out && workspace && (extra || desc->extra_channels == 0), "temporal entry: NULL pointer");
        FIERY_REQUIRE(aligned16(x) && aligned16(workspace), "temporal entry: pointers must be 16-byte aligned");
        for (int q = 0; q < desc->n_segments; ++q)
            FIERY_REQUIRE(grad_out[q] && aligned16(grad_out[q]), "temporal entry: grad_out[%d] is NULL or misaligned", q);
    }
    return launch_temporal_entry_wgrad(desc, x, desc->extra_channels ? extra : nullptr, grad_out, grad_w, workspace,
                                       static_cast<cudaStream_t>(stream));
}

// The causal convolution's shape limits, one place for every entry point.  The messages name the field.
static int check_causal_conv_desc(const fiery_causal_conv3d_desc_t* d) {
    FIERY_REQUIRE(d, "causal conv: NULL desc");
    FIERY_REQUIRE(d->batch >= 0 && d->frames >= 0, "causal conv: batch = %d, frames = %d must be >= 0", d->batch, d->frames);
    FIERY_REQUIRE(d->in_channels >= 1 && d->in_channels <= 64, "causal conv: in_channels = %d must be in 1..64", d->in_channels);
    FIERY_REQUIRE(d->out_channels >= 1 && d->out_channels <= 64, "causal conv: out_channels = %d must be in 1..64", d->out_channels);
    FIERY_REQUIRE(d->kt == 1 || d->kt == 2, "causal conv: kt = %d must be 1 or 2 (kernel (kt, 3, 3))", d->kt);
    FIERY_REQUIRE(d->grid_x >= 1, "causal conv: grid_x = %d must be >= 1", d->grid_x);
    FIERY_REQUIRE(d->grid_y >= 1 && d->grid_y % 4 == 0, "causal conv: grid_y = %d must be a positive multiple of 4 (16-byte TMA row pitch)",
                  d->grid_y);
    return FIERY_OK;
}

FIERY_API size_t fiery_causal_conv3d_packed_bytes(const fiery_causal_conv3d_desc_t* desc) {
    if (check_causal_conv_desc(desc) != FIERY_OK) return 0;
    return causal_conv_packed_bytes(desc);
}

FIERY_API int fiery_causal_conv3d_pack_weights(const fiery_causal_conv3d_desc_t* desc, const float* weight, void* packed, void* stream) {
    const int rc = check_causal_conv_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(weight && packed, "causal conv: NULL weight pointer");
    FIERY_REQUIRE(aligned16(packed), "causal conv: packed weights must be 16-byte aligned");
    return launch_causal_conv_pack(desc, weight, static_cast<float*>(packed), static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_causal_conv3d_forward(const fiery_causal_conv3d_desc_t* desc, const float* x, const void* packed, float* y, void* stream) {
    const int rc = check_causal_conv_desc(desc);
    if (rc != FIERY_OK) return rc;
    if (desc->batch == 0 || desc->frames == 0) return FIERY_OK;
    FIERY_REQUIRE(x && packed && y, "causal conv: NULL pointer");
    FIERY_REQUIRE(aligned16(x) && aligned16(packed) && aligned16(y), "causal conv: pointers must be 16-byte aligned");
    return launch_causal_conv_forward(desc, x, static_cast<const float*>(packed), y, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_causal_conv3d_backward_data(const fiery_causal_conv3d_desc_t* desc, const float* grad_y, const void* packed,
                                                float* grad_x, void* stream) {
    const int rc = check_causal_conv_desc(desc);
    if (rc != FIERY_OK) return rc;
    if (desc->batch == 0 || desc->frames == 0) return FIERY_OK;
    FIERY_REQUIRE(grad_y && packed && grad_x, "causal conv: NULL pointer");
    FIERY_REQUIRE(aligned16(grad_y) && aligned16(packed) && aligned16(grad_x), "causal conv: pointers must be 16-byte aligned");
    return launch_causal_conv_dgrad(desc, grad_y, static_cast<const float*>(packed), grad_x, static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_causal_conv3d_backward_weight_workspace_bytes(const fiery_causal_conv3d_desc_t* desc) {
    if (check_causal_conv_desc(desc) != FIERY_OK) return 0;
    return causal_conv_wgrad_workspace_bytes(desc);
}

FIERY_API int fiery_causal_conv3d_backward_weight(const fiery_causal_conv3d_desc_t* desc, const float* x, const float* grad_y,
                                                  float* grad_w, void* workspace, void* stream) {
    const int rc = check_causal_conv_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(grad_w, "causal conv: NULL grad_w");
    if (desc->batch > 0 && desc->frames > 0) {
        FIERY_REQUIRE(x && grad_y && workspace, "causal conv: NULL pointer");
        FIERY_REQUIRE(aligned16(x) && aligned16(grad_y) && aligned16(workspace), "causal conv: pointers must be 16-byte aligned");
    }
    return launch_causal_conv_wgrad(desc, x, grad_y, grad_w, workspace, static_cast<cudaStream_t>(stream));
}

// The batch norm's shape limits, one place for every entry point.  The messages name the field.  sync: the entries of a rank in a
// group (fiery_batch_norm_*_gathered and their local phases), which take training only and a rank with no or a single value.
static int check_batch_norm_desc(const fiery_batch_norm_desc_t* d, bool sync = false) {
    FIERY_REQUIRE(d, "batch norm: NULL desc");
    FIERY_REQUIRE(d->channels >= 1, "batch norm: channels = %d must be >= 1", d->channels);
    if (sync)
        FIERY_REQUIRE(d->batch >= 0 && d->frames >= 0, "batch norm: batch = %d, frames = %d must be >= 0", d->batch, d->frames);
    else
        FIERY_REQUIRE(d->batch >= 0 && d->frames >= 0 && static_cast<long long>(d->batch) * d->frames >= 1,
                      "batch norm: batch = %d, frames = %d must be >= 0 with batch * frames >= 1", d->batch, d->frames);
    FIERY_REQUIRE(d->pixels >= 1, "batch norm: pixels X*Y = %d must be >= 1", d->pixels);
    FIERY_REQUIRE(d->stride_b >= 0 && d->stride_c >= 0 && d->stride_t >= 0, "batch norm: strides (%lld, %lld, %lld) must be >= 0",
                  (long long)d->stride_b, (long long)d->stride_c, (long long)d->stride_t);
    if (sync) FIERY_REQUIRE(d->training == 1, "batch norm: training = %d must be 1 for statistics over a group", d->training);
    FIERY_REQUIRE(d->training == 0 || d->training == 1, "batch norm: training = %d must be 0 or 1", d->training);
    FIERY_REQUIRE(d->relu == 0 || d->relu == 1, "batch norm: relu = %d must be 0 or 1", d->relu);
    FIERY_REQUIRE(d->eps >= 0.0, "batch norm: eps = %g must be >= 0", d->eps);
    FIERY_REQUIRE(sync || !d->training || static_cast<long long>(d->batch) * d->frames * d->pixels >= 2,
                  "batch norm: n = batch * frames * pixels = %lld values per channel must be >= 2 in training",
                  static_cast<long long>(d->batch) * d->frames * d->pixels);
    return FIERY_OK;
}

static bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

static int check_world(int world, const double* gathered, const char* what) {
    FIERY_REQUIRE(world >= 1, "%s: world = %d must be >= 1", what, world);
    FIERY_REQUIRE(gathered, "%s: NULL gathered", what);
    FIERY_REQUIRE(aligned8(gathered), "%s: gathered must be 8-byte aligned", what);
    return FIERY_OK;
}

FIERY_API size_t fiery_batch_norm_sync_workspace_bytes(const fiery_batch_norm_desc_t* desc) {
    if (check_batch_norm_desc(desc, true) != FIERY_OK) return 0;
    return batch_norm_workspace_bytes(desc);
}

FIERY_API int fiery_batch_norm_local_stats(const fiery_batch_norm_desc_t* desc, const float* x, double* stats, void* workspace, void* stream) {
    const int rc = check_batch_norm_desc(desc, true);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE((x || desc->batch == 0 || desc->frames == 0) && stats && workspace, "batch norm: NULL x / stats / workspace");
    FIERY_REQUIRE(aligned8(stats) && aligned16(workspace), "batch norm: stats must be 8-byte and workspace 16-byte aligned");
    return launch_batch_norm_local_stats(desc, x, stats, workspace, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_batch_norm_forward_gathered(const fiery_batch_norm_desc_t* desc, int32_t world, const double* gathered, const float* x,
                                                const float* weight, const float* bias, const float* residual, float* y, float* mean_out,
                                                float* var_out, double* count_out, void* workspace, void* stream) {
    int rc = check_batch_norm_desc(desc, true);
    if (rc != FIERY_OK || (rc = check_world(world, gathered, "batch norm")) != FIERY_OK) return rc;
    const bool empty = desc->batch == 0 || desc->frames == 0;
    FIERY_REQUIRE(((x && y) || empty) && mean_out && var_out && workspace, "batch norm: NULL x / y / mean_out / var_out / workspace");
    FIERY_REQUIRE(aligned16(workspace) && (!count_out || aligned8(count_out)),
                  "batch norm: workspace must be 16-byte and count_out 8-byte aligned");
    return launch_batch_norm_forward_gathered(desc, world, gathered, x, weight, bias, residual, y, mean_out, var_out, count_out, workspace,
                                              static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_batch_norm_local_grad_sums(const fiery_batch_norm_desc_t* desc, const float* x, const float* grad_y, const float* weight,
                                               const float* bias, const float* mean, const float* var, double* sums, float* grad_weight,
                                               float* grad_bias, void* workspace, void* stream) {
    const int rc = check_batch_norm_desc(desc, true);
    if (rc != FIERY_OK) return rc;
    const bool empty = desc->batch == 0 || desc->frames == 0;
    FIERY_REQUIRE(((x && grad_y) || empty) && mean && var && sums && workspace, "batch norm: NULL x / grad_y / mean / var / sums / workspace");
    FIERY_REQUIRE(aligned8(sums) && aligned16(workspace), "batch norm: sums must be 8-byte and workspace 16-byte aligned");
    return launch_batch_norm_local_grad_sums(desc, x, grad_y, weight, bias, mean, var, sums, grad_weight, grad_bias, workspace,
                                             static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_batch_norm_backward_gathered(const fiery_batch_norm_desc_t* desc, int32_t world, const double* gathered, const float* x,
                                                 const float* grad_y, const float* weight, const float* bias, const float* mean,
                                                 const float* var, float* grad_x, void* workspace, void* stream) {
    int rc = check_batch_norm_desc(desc, true);
    if (rc != FIERY_OK || (rc = check_world(world, gathered, "batch norm")) != FIERY_OK) return rc;
    const bool empty = desc->batch == 0 || desc->frames == 0;
    FIERY_REQUIRE(((x && grad_y && grad_x) || empty) && mean && var && workspace,
                  "batch norm: NULL x / grad_y / grad_x / mean / var / workspace");
    FIERY_REQUIRE(aligned16(workspace), "batch norm: workspace must be 16-byte aligned");
    return launch_batch_norm_backward_gathered(desc, world, gathered, x, grad_y, weight, bias, mean, var, grad_x, workspace,
                                               static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_batch_norm_workspace_bytes(const fiery_batch_norm_desc_t* desc) {
    if (check_batch_norm_desc(desc) != FIERY_OK) return 0;
    return batch_norm_workspace_bytes(desc);
}

FIERY_API int fiery_batch_norm_forward(const fiery_batch_norm_desc_t* desc, const float* x, const float* weight, const float* bias,
                                       const float* running_mean, const float* running_var, const float* residual, float* y,
                                       float* mean_out, float* var_out, void* workspace, void* stream) {
    const int rc = check_batch_norm_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(x && y && mean_out && var_out && workspace, "batch norm: NULL x / y / mean_out / var_out / workspace");
    FIERY_REQUIRE(desc->training || (running_mean && running_var), "batch norm: eval mode needs running_mean and running_var");
    FIERY_REQUIRE(aligned16(workspace), "batch norm: workspace must be 16-byte aligned");
    return launch_batch_norm_forward(desc, x, weight, bias, desc->training ? nullptr : running_mean, desc->training ? nullptr : running_var,
                                     residual, y, mean_out, var_out, workspace, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_batch_norm_backward(const fiery_batch_norm_desc_t* desc, const float* x, const float* grad_y, const float* weight,
                                        const float* bias, const float* mean, const float* var, float* grad_x, float* grad_weight,
                                        float* grad_bias, void* workspace, void* stream) {
    const int rc = check_batch_norm_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(x && grad_y && mean && var && workspace, "batch norm: NULL x / grad_y / mean / var / workspace");
    FIERY_REQUIRE(aligned16(workspace), "batch norm: workspace must be 16-byte aligned");
    return launch_batch_norm_backward(desc, x, grad_y, weight, bias, mean, var, grad_x, grad_weight, grad_bias, workspace,
                                      static_cast<cudaStream_t>(stream));
}

// The spatial GRU's shape limits, one place for every entry point.  The messages name the field.
static int check_spatial_gru_desc(const fiery_spatial_gru_desc_t* d) {
    FIERY_REQUIRE(d, "spatial GRU: NULL desc");
    FIERY_REQUIRE(d->batch >= 1 && d->frames >= 1, "spatial GRU: batch = %d, frames = %d must be >= 1", d->batch, d->frames);
    FIERY_REQUIRE(d->x_frames == 1 || d->x_frames == d->frames, "spatial GRU: x_frames = %d must be 1 or frames = %d", d->x_frames, d->frames);
    FIERY_REQUIRE(d->x_channels >= 1 && d->x_channels <= 64, "spatial GRU: x_channels = %d must be in 1..64", d->x_channels);
    FIERY_REQUIRE(d->h_channels >= 1 && d->h_channels <= 64, "spatial GRU: h_channels = %d must be in 1..64", d->h_channels);
    FIERY_REQUIRE(d->grid_x >= 1, "spatial GRU: grid_x = %d must be >= 1", d->grid_x);
    FIERY_REQUIRE(d->grid_y >= 1 && d->grid_y % 4 == 0, "spatial GRU: grid_y = %d must be a positive multiple of 4 (16-byte TMA row pitch)",
                  d->grid_y);
    FIERY_REQUIRE(d->x_stride_b >= 0 && d->x_stride_t >= 0 && d->x_stride_c >= 0 && d->x_stride_b % 4 == 0 && d->x_stride_t % 4 == 0 &&
                      d->x_stride_c % 4 == 0,
                  "spatial GRU: x strides (%lld, %lld, %lld) must be non-negative multiples of 4 elements", (long long)d->x_stride_b,
                  (long long)d->x_stride_t, (long long)d->x_stride_c);
    FIERY_REQUIRE(d->training == 0 || d->training == 1, "spatial GRU: training = %d must be 0 or 1", d->training);
    FIERY_REQUIRE(d->eps >= 0.0, "spatial GRU: eps = %g must be >= 0", d->eps);
    FIERY_REQUIRE(!d->training || static_cast<long long>(d->batch) * d->grid_x * d->grid_y >= 2,
                  "spatial GRU: batch * X * Y must be >= 2 in training");
    return FIERY_OK;
}

FIERY_API size_t fiery_spatial_gru_packed_bytes(const fiery_spatial_gru_desc_t* desc) {
    if (check_spatial_gru_desc(desc) != FIERY_OK) return 0;
    return spatial_gru_packed_bytes(desc);
}

FIERY_API int fiery_spatial_gru_pack_weights(const fiery_spatial_gru_desc_t* desc, const float* w_gates, const float* w_state, void* packed,
                                             void* stream) {
    const int rc = check_spatial_gru_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(w_gates && w_state && packed, "spatial GRU: NULL weight pointer");
    FIERY_REQUIRE(aligned16(packed), "spatial GRU: packed weights must be 16-byte aligned");
    return launch_spatial_gru_pack(desc, w_gates, w_state, static_cast<float*>(packed), static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_spatial_gru_saved_bytes(const fiery_spatial_gru_desc_t* desc) {
    if (check_spatial_gru_desc(desc) != FIERY_OK) return 0;
    return 4 * sizeof(float) * static_cast<size_t>(desc->frames) * desc->batch * desc->h_channels * desc->grid_x * desc->grid_y;
}

FIERY_API size_t fiery_spatial_gru_forward_workspace_bytes(const fiery_spatial_gru_desc_t* desc) {
    if (check_spatial_gru_desc(desc) != FIERY_OK) return 0;
    return spatial_gru_forward_workspace_bytes(desc);
}

FIERY_API int fiery_spatial_gru_forward(const fiery_spatial_gru_desc_t* desc, const float* x, const float* h0, const void* packed,
                                        const float* b_gates, const float* bn_weight, const float* bn_bias, const float* running_mean,
                                        const float* running_var, float* out, void* saved, float* means, float* vars, void* workspace,
                                        void* stream) {
    const int rc = check_spatial_gru_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(x && h0 && packed && b_gates && out && saved && means && vars && workspace, "spatial GRU: NULL pointer");
    FIERY_REQUIRE(desc->training || (running_mean && running_var), "spatial GRU: eval mode needs running_mean and running_var");
    FIERY_REQUIRE(aligned16(x) && aligned16(h0) && aligned16(packed) && aligned16(out) && aligned16(saved) && aligned16(workspace),
                  "spatial GRU: pointers must be 16-byte aligned");
    return launch_spatial_gru_forward(desc, x, h0, static_cast<const float*>(packed), b_gates, bn_weight, bn_bias,
                                      desc->training ? nullptr : running_mean, desc->training ? nullptr : running_var, out,
                                      static_cast<float*>(saved), means, vars, workspace, static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_spatial_gru_backward_workspace_bytes(const fiery_spatial_gru_desc_t* desc) {
    if (check_spatial_gru_desc(desc) != FIERY_OK) return 0;
    return spatial_gru_backward_workspace_bytes(desc);
}

FIERY_API int fiery_spatial_gru_backward(const fiery_spatial_gru_desc_t* desc, const float* grad_out, const float* x, const float* h0,
                                         const float* out, const void* saved, const float* means, const float* vars, const void* packed,
                                         const float* bn_weight, const float* bn_bias, float* grad_x, float* grad_h0, float* grad_w_gates,
                                         float* grad_b_gates, float* grad_w_state, float* grad_bn_weight, float* grad_bn_bias,
                                         void* workspace, void* stream) {
    const int rc = check_spatial_gru_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(grad_out && x && h0 && out && saved && means && vars && packed && workspace, "spatial GRU: NULL pointer");
    FIERY_REQUIRE(aligned16(grad_out) && aligned16(x) && aligned16(h0) && aligned16(out) && aligned16(saved) && aligned16(packed) &&
                      aligned16(workspace) && (!grad_x || aligned16(grad_x)) && (!grad_h0 || aligned16(grad_h0)),
                  "spatial GRU: pointers must be 16-byte aligned");
    return launch_spatial_gru_backward(desc, grad_out, x, h0, out, static_cast<const float*>(saved), means, vars,
                                       static_cast<const float*>(packed), bn_weight, bn_bias, grad_x, grad_h0, grad_w_gates, grad_b_gates,
                                       grad_w_state, grad_bn_weight, grad_bn_bias, workspace, static_cast<cudaStream_t>(stream));
}

// the per-step entries' common checks: the desc in training, the step, and the 16-byte aligned pointers (NULL where allowed)
static int check_spatial_gru_step(const fiery_spatial_gru_desc_t* d, int t, std::initializer_list<const void*> required,
                                  std::initializer_list<const void*> optional) {
    const int rc = check_spatial_gru_desc(d);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(d->training == 1, "spatial GRU: training = %d must be 1 for statistics over a group", d->training);
    FIERY_REQUIRE(t >= 0 && t < d->frames, "spatial GRU: t = %d must be in 0..frames - 1 = %d", t, d->frames - 1);
    for (const void* p : required) FIERY_REQUIRE(p, "spatial GRU: NULL pointer");
    for (const void* p : required) FIERY_REQUIRE(aligned16(p), "spatial GRU: pointers must be 16-byte aligned");
    for (const void* p : optional) FIERY_REQUIRE(!p || aligned16(p), "spatial GRU: pointers must be 16-byte aligned");
    return FIERY_OK;
}

FIERY_API int fiery_spatial_gru_forward_step_begin(const fiery_spatial_gru_desc_t* desc, int32_t t, const float* x, const float* h0,
                                                   const void* packed, const float* b_gates, const float* out, void* saved, double* stats,
                                                   void* workspace, void* stream) {
    const int rc = check_spatial_gru_step(desc, t, {x, h0, packed, out, saved, workspace}, {});
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(b_gates && stats, "spatial GRU: NULL b_gates / stats");
    FIERY_REQUIRE(aligned8(stats), "spatial GRU: stats must be 8-byte aligned");
    return launch_spatial_gru_forward_step_begin(desc, t, x, h0, static_cast<const float*>(packed), b_gates, out, static_cast<float*>(saved),
                                                 stats, workspace, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_spatial_gru_forward_step_end(const fiery_spatial_gru_desc_t* desc, int32_t t, int32_t world, const double* gathered,
                                                 const float* h0, const float* bn_weight, const float* bn_bias, float* out, const void* saved,
                                                 float* means, float* vars, double* count_out, void* workspace, void* stream) {
    int rc = check_spatial_gru_step(desc, t, {h0, out, saved, workspace}, {});
    if (rc != FIERY_OK || (rc = check_world(world, gathered, "spatial GRU")) != FIERY_OK) return rc;
    FIERY_REQUIRE(means && vars, "spatial GRU: NULL means / vars");
    FIERY_REQUIRE(!count_out || aligned8(count_out), "spatial GRU: count_out must be 8-byte aligned");
    return launch_spatial_gru_forward_step_end(desc, t, world, gathered, h0, bn_weight, bn_bias, out, static_cast<const float*>(saved), means,
                                               vars, count_out, workspace, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_spatial_gru_backward_step_begin(const fiery_spatial_gru_desc_t* desc, int32_t t, const float* grad_out, const float* h0,
                                                    const float* out, const void* saved, const float* means, const float* vars,
                                                    const void* packed, const float* bn_weight, const float* bn_bias, float* grad_h0,
                                                    double* sums, void* workspace, void* stream) {
    const int rc = check_spatial_gru_step(desc, t, {grad_out, h0, out, saved, packed, workspace}, {grad_h0});
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(means && vars && sums, "spatial GRU: NULL means / vars / sums");
    FIERY_REQUIRE(aligned8(sums), "spatial GRU: sums must be 8-byte aligned");
    return launch_spatial_gru_backward_step_begin(desc, t, grad_out, h0, out, static_cast<const float*>(saved), means, vars,
                                                  static_cast<const float*>(packed), bn_weight, bn_bias, grad_h0, sums, workspace,
                                                  static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_spatial_gru_backward_step_end(const fiery_spatial_gru_desc_t* desc, int32_t t, int32_t world, const double* gathered,
                                                  const float* h0, const float* out, const void* saved, const float* means, const float* vars,
                                                  const void* packed, const float* bn_weight, const float* bn_bias, float* grad_x,
                                                  float* grad_h0, void* workspace, void* stream) {
    int rc = check_spatial_gru_step(desc, t, {h0, out, saved, packed, workspace}, {grad_x, grad_h0});
    if (rc != FIERY_OK || (rc = check_world(world, gathered, "spatial GRU")) != FIERY_OK) return rc;
    FIERY_REQUIRE(means && vars, "spatial GRU: NULL means / vars");
    return launch_spatial_gru_backward_step_end(desc, t, world, gathered, h0, out, static_cast<const float*>(saved), means, vars,
                                                static_cast<const float*>(packed), bn_weight, bn_bias, grad_x, grad_h0, workspace,
                                                static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_spatial_gru_backward_weights(const fiery_spatial_gru_desc_t* desc, const float* x, const float* h0, const float* out,
                                                 const void* saved, const void* packed, float* grad_w_gates, float* grad_b_gates,
                                                 float* grad_w_state, float* grad_bn_weight, float* grad_bn_bias, void* workspace,
                                                 void* stream) {
    const int rc = check_spatial_gru_step(desc, 0, {x, h0, out, saved, packed, workspace}, {});
    if (rc != FIERY_OK) return rc;
    return launch_spatial_gru_backward_weights(desc, x, h0, out, static_cast<const float*>(saved), static_cast<const float*>(packed),
                                               grad_w_gates, grad_b_gates, grad_w_state, grad_bn_weight, grad_bn_bias, workspace,
                                               static_cast<cudaStream_t>(stream));
}

// The 3x3 convolution's limits, one place for every entry point.  The messages name the field.
static int check_conv3x3_desc(const fiery_conv3x3_desc_t* d) {
    FIERY_REQUIRE(d, "3x3 conv: NULL desc");
    FIERY_REQUIRE(d->maps >= 1, "3x3 conv: maps = %d must be >= 1", d->maps);
    FIERY_REQUIRE(d->in_channels[0] >= 1 && d->in_channels[0] <= 64, "3x3 conv: in_channels[0] = %d must be in 1..64", d->in_channels[0]);
    FIERY_REQUIRE(d->in_channels[1] >= 0 && d->in_channels[1] <= 64, "3x3 conv: in_channels[1] = %d must be in 0..64", d->in_channels[1]);
    FIERY_REQUIRE(d->out_channels[0] >= 1 && d->out_channels[0] <= 64, "3x3 conv: out_channels[0] = %d must be in 1..64",
                  d->out_channels[0]);
    FIERY_REQUIRE(d->out_channels[1] >= 0 && d->out_channels[1] <= 64, "3x3 conv: out_channels[1] = %d must be in 0..64",
                  d->out_channels[1]);
    FIERY_REQUIRE(d->grid_x >= 1, "3x3 conv: grid_x = %d must be >= 1", d->grid_x);
    FIERY_REQUIRE(d->grid_y >= 1 && d->grid_y % 4 == 0, "3x3 conv: grid_y = %d must be a positive multiple of 4 (16-byte TMA row pitch)",
                  d->grid_y);
    return FIERY_OK;
}

FIERY_API size_t fiery_conv3x3_packed_bytes(const fiery_conv3x3_desc_t* desc) {
    if (check_conv3x3_desc(desc) != FIERY_OK) return 0;
    return conv3x3_packed_bytes(desc);
}

FIERY_API int fiery_conv3x3_pack_weights(const fiery_conv3x3_desc_t* desc, const float* weight, void* packed, void* stream) {
    const int rc = check_conv3x3_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(weight && packed && aligned16(packed), "3x3 conv: NULL weight or misaligned pack");
    return launch_conv3x3_pack(desc, weight, static_cast<float*>(packed), static_cast<cudaStream_t>(stream));
}

// a segment pair: the first always given, the second when it has channels
static int check_conv3x3_pair(const int* channels, const float* a, const float* b, const char* what) {
    FIERY_REQUIRE(a && aligned16(a), "3x3 conv: %s0 is NULL or misaligned", what);
    FIERY_REQUIRE(!channels[1] || (b && aligned16(b)), "3x3 conv: %s1 is NULL or misaligned", what);
    return FIERY_OK;
}

FIERY_API int fiery_conv3x3_forward(const fiery_conv3x3_desc_t* desc, const float* x0, const float* x1, const void* packed, float* y0,
                                    float* y1, void* stream) {
    int rc = check_conv3x3_desc(desc);
    if (rc != FIERY_OK) return rc;
    if ((rc = check_conv3x3_pair(desc->in_channels, x0, x1, "x")) != FIERY_OK) return rc;
    if ((rc = check_conv3x3_pair(desc->out_channels, y0, y1, "y")) != FIERY_OK) return rc;
    FIERY_REQUIRE(packed && aligned16(packed), "3x3 conv: NULL or misaligned pack");
    return launch_conv3x3(desc, 0, x0, x1, static_cast<const float*>(packed), y0, y1, static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_conv3x3_backward_data(const fiery_conv3x3_desc_t* desc, const float* grad_y0, const float* grad_y1, const void* packed,
                                          float* grad_x0, float* grad_x1, void* stream) {
    int rc = check_conv3x3_desc(desc);
    if (rc != FIERY_OK) return rc;
    if ((rc = check_conv3x3_pair(desc->out_channels, grad_y0, grad_y1, "grad_y")) != FIERY_OK) return rc;
    if ((rc = check_conv3x3_pair(desc->in_channels, grad_x0, grad_x1, "grad_x")) != FIERY_OK) return rc;
    FIERY_REQUIRE(packed && aligned16(packed), "3x3 conv: NULL or misaligned pack");
    return launch_conv3x3(desc, 1, grad_y0, grad_y1, static_cast<const float*>(packed), grad_x0, grad_x1, static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_conv3x3_backward_weight_workspace_bytes(const fiery_conv3x3_desc_t* desc) {
    if (check_conv3x3_desc(desc) != FIERY_OK) return 0;
    return conv3x3_wgrad_workspace_bytes(desc);
}

FIERY_API int fiery_conv3x3_backward_weight(const fiery_conv3x3_desc_t* desc, const float* x0, const float* x1, const float* grad_y,
                                            float* grad_w, void* workspace, void* stream) {
    int rc = check_conv3x3_desc(desc);
    if (rc != FIERY_OK) return rc;
    if ((rc = check_conv3x3_pair(desc->in_channels, x0, x1, "x")) != FIERY_OK) return rc;
    FIERY_REQUIRE(grad_y && aligned16(grad_y) && grad_w && workspace && aligned16(workspace),
                  "3x3 conv: NULL or misaligned grad_y / grad_w / workspace");
    return launch_conv3x3_wgrad(desc, x0, x1, grad_y, grad_w, workspace, static_cast<cudaStream_t>(stream));
}


// The Bottleneck's limits, one place for every entry point: those of the kernels it chains.  The messages name the field.
static int check_bottleneck_desc(const fiery_bottleneck_desc_t* d) {
    FIERY_REQUIRE(d, "bottleneck: NULL desc");
    FIERY_REQUIRE(d->maps >= 1, "bottleneck: maps = %d must be >= 1", d->maps);
    FIERY_REQUIRE(d->channels >= 2 && d->channels <= 128, "bottleneck: channels = %d must be in 2..128 (M = channels / 2 <= 64)",
                  d->channels);
    FIERY_REQUIRE(d->grid_x >= 1, "bottleneck: grid_x = %d must be >= 1", d->grid_x);
    FIERY_REQUIRE(d->grid_y >= 1 && d->grid_y % 4 == 0, "bottleneck: grid_y = %d must be a positive multiple of 4 (16-byte TMA row pitch)",
                  d->grid_y);
    FIERY_REQUIRE(static_cast<long long>(d->grid_x) * d->grid_y < (1ll << 31), "bottleneck: grid_x * grid_y = %lld pixels must be < 2^31",
                  static_cast<long long>(d->grid_x) * d->grid_y);
    FIERY_REQUIRE(d->training == 0 || d->training == 1, "bottleneck: training = %d must be 0 or 1", d->training);
    FIERY_REQUIRE(d->eps >= 0.0, "bottleneck: eps = %g must be >= 0", d->eps);
    FIERY_REQUIRE(!d->training || static_cast<long long>(d->maps) * d->grid_x * d->grid_y >= 2,
                  "bottleneck: maps * grid_x * grid_y = %lld values per channel must be >= 2 in training",
                  static_cast<long long>(d->maps) * d->grid_x * d->grid_y);
    return FIERY_OK;
}

FIERY_API size_t fiery_bottleneck_packed_bytes(const fiery_bottleneck_desc_t* desc) {
    if (check_bottleneck_desc(desc) != FIERY_OK) return 0;
    return bottleneck_packed_bytes(desc);
}

FIERY_API int fiery_bottleneck_pack_weights(const fiery_bottleneck_desc_t* desc, const float* w_down, const float* w_conv, const float* w_up,
                                            void* packed, void* stream) {
    const int rc = check_bottleneck_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(w_down && w_conv && w_up && packed, "bottleneck: NULL weight pointer");
    FIERY_REQUIRE(aligned16(packed), "bottleneck: packed weights must be 16-byte aligned");
    return launch_bottleneck_pack(desc, w_down, w_conv, w_up, packed, static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_bottleneck_forward_workspace_bytes(const fiery_bottleneck_desc_t* desc) {
    if (check_bottleneck_desc(desc) != FIERY_OK) return 0;
    return bottleneck_forward_workspace_bytes(desc);
}

FIERY_API int fiery_bottleneck_forward(const fiery_bottleneck_desc_t* desc, const float* x, const void* packed, const float* const* norms,
                                       float* y1, float* y2, float* y3, float* out, float* stats, void* workspace, void* stream) {
    const int rc = check_bottleneck_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(x && packed && norms && y1 && y2 && y3 && out && stats && workspace, "bottleneck: NULL pointer");
    for (int i = 0; i < 3 && !desc->training; ++i)
        FIERY_REQUIRE(norms[4 * i + 2] && norms[4 * i + 3], "bottleneck: eval mode needs norm %d's running_mean and running_var", i);
    FIERY_REQUIRE(aligned16(x) && aligned16(packed) && aligned16(y1) && aligned16(y2) && aligned16(y3) && aligned16(out) && aligned16(workspace),
                  "bottleneck: pointers must be 16-byte aligned");
    return launch_bottleneck_forward(desc, x, packed, norms, y1, y2, y3, out, stats, workspace, static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_bottleneck_backward_workspace_bytes(const fiery_bottleneck_desc_t* desc) {
    if (check_bottleneck_desc(desc) != FIERY_OK) return 0;
    return bottleneck_backward_workspace_bytes(desc);
}

FIERY_API int fiery_bottleneck_backward(const fiery_bottleneck_desc_t* desc, const float* grad_out, const float* x, const float* y1,
                                        const float* y2, const float* y3, const float* stats, const void* packed, const float* const* norms,
                                        float* grad_x, float* grad_w_down, float* grad_w_conv, float* grad_w_up, float* const* grad_norms,
                                        void* workspace, void* stream) {
    const int rc = check_bottleneck_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(grad_out && x && y1 && y2 && y3 && stats && packed && norms && grad_norms && workspace, "bottleneck: NULL pointer");
    FIERY_REQUIRE(aligned16(grad_out) && aligned16(x) && aligned16(y1) && aligned16(y2) && aligned16(y3) && aligned16(packed) &&
                      aligned16(workspace) && (!grad_x || aligned16(grad_x)),
                  "bottleneck: pointers must be 16-byte aligned");
    return launch_bottleneck_backward(desc, grad_out, x, y1, y2, y3, stats, packed, norms, grad_x, grad_w_down, grad_w_conv, grad_w_up,
                                      grad_norms, workspace, static_cast<cudaStream_t>(stream));
}

// the group stages' common checks: the desc in training, the stage, and the gathered triplets of stages 1..3
static int check_bottleneck_stage(const fiery_bottleneck_desc_t* d, int stage, int world, const double* gathered) {
    int rc = check_bottleneck_desc(d);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(d->training == 1, "bottleneck: training = %d must be 1 for statistics over a group", d->training);
    FIERY_REQUIRE(stage >= 0 && stage <= 3, "bottleneck: stage = %d must be in 0..3", stage);
    if (stage > 0 && (rc = check_world(world, gathered, "bottleneck")) != FIERY_OK) return rc;
    return FIERY_OK;
}

FIERY_API int fiery_bottleneck_sync_forward_stage(const fiery_bottleneck_desc_t* desc, int32_t stage, int32_t world, const double* gathered,
                                                  const float* x, const void* packed, const float* const* norms, float* y1, float* y2,
                                                  float* y3, float* out, float* stats, double* counts, double* local, void* workspace,
                                                  void* stream) {
    const int rc = check_bottleneck_stage(desc, stage, world, gathered);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(x && packed && norms && y1 && y2 && y3 && out && stats && workspace, "bottleneck: NULL pointer");
    FIERY_REQUIRE(aligned16(x) && aligned16(packed) && aligned16(y1) && aligned16(y2) && aligned16(y3) && aligned16(out) && aligned16(workspace),
                  "bottleneck: pointers must be 16-byte aligned");
    if (stage < 3) FIERY_REQUIRE(local, "bottleneck: NULL local");
    if (stage < 3) FIERY_REQUIRE(aligned8(local), "bottleneck: local must be 8-byte aligned");
    if (stage > 0) FIERY_REQUIRE(counts, "bottleneck: NULL counts");
    if (stage > 0) FIERY_REQUIRE(aligned8(counts), "bottleneck: counts must be 8-byte aligned");
    return launch_bottleneck_sync_forward_stage(desc, stage, world, gathered, x, packed, norms, y1, y2, y3, out, stats, counts, local, workspace,
                                                static_cast<cudaStream_t>(stream));
}

FIERY_API int fiery_bottleneck_sync_backward_stage(const fiery_bottleneck_desc_t* desc, int32_t stage, int32_t world, const double* gathered,
                                                   const float* grad_out, const float* x, const float* y1, const float* y2, const float* y3,
                                                   const float* stats, const void* packed, const float* const* norms, float* grad_x,
                                                   float* grad_w_down, float* grad_w_conv, float* grad_w_up, float* const* grad_norms,
                                                   double* local, void* workspace, void* stream) {
    const int rc = check_bottleneck_stage(desc, stage, world, gathered);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(grad_out && x && y1 && y2 && y3 && stats && packed && norms && grad_norms && workspace, "bottleneck: NULL pointer");
    FIERY_REQUIRE(aligned16(grad_out) && aligned16(x) && aligned16(y1) && aligned16(y2) && aligned16(y3) && aligned16(packed) &&
                      aligned16(workspace) && (!grad_x || aligned16(grad_x)),
                  "bottleneck: pointers must be 16-byte aligned");
    if (stage < 3) FIERY_REQUIRE(local, "bottleneck: NULL local");
    if (stage < 3) FIERY_REQUIRE(aligned8(local), "bottleneck: local must be 8-byte aligned");
    return launch_bottleneck_sync_backward_stage(desc, stage, world, gathered, grad_out, x, y1, y2, y3, stats, packed, norms, grad_x,
                                                 grad_w_down, grad_w_conv, grad_w_up, grad_norms, local, workspace,
                                                 static_cast<cudaStream_t>(stream));
}

// The output head's limits, one place for every entry point.  The messages name the field.
static int check_output_head_desc(const fiery_output_head_desc_t* d) {
    FIERY_REQUIRE(d, "output head: NULL desc");
    FIERY_REQUIRE(d->maps >= 1, "output head: maps = %d must be >= 1", d->maps);
    FIERY_REQUIRE(d->channels >= 1 && d->channels <= 128, "output head: channels = %d must be in 1..128", d->channels);
    FIERY_REQUIRE(d->n_out >= 1 && d->n_out <= 8, "output head: n_out = %d must be in 1..8", d->n_out);
    FIERY_REQUIRE(d->grid_x >= 1, "output head: grid_x = %d must be >= 1", d->grid_x);
    FIERY_REQUIRE(d->grid_y >= 1, "output head: grid_y = %d must be >= 1", d->grid_y);
    const long long P = static_cast<long long>(d->grid_x) * d->grid_y;
    FIERY_REQUIRE(P < (1ll << 31), "output head: grid_x * grid_y = %lld pixels must be < 2^31", P);
    FIERY_REQUIRE(P % 4 == 0, "output head: grid_x * grid_y = %lld pixels must be a multiple of 4 (16-byte TMA plane pitch)", P);
    FIERY_REQUIRE(d->training == 0 || d->training == 1, "output head: training = %d must be 0 or 1", d->training);
    FIERY_REQUIRE(d->eps >= 0.0, "output head: eps = %g must be >= 0", d->eps);
    FIERY_REQUIRE(!d->training || d->maps * P >= 2, "output head: maps * grid_x * grid_y = %lld values per channel must be >= 2 in training",
                  d->maps * P);
    return FIERY_OK;
}

FIERY_API size_t fiery_output_head_packed_bytes(const fiery_output_head_desc_t* desc) {
    if (check_output_head_desc(desc) != FIERY_OK) return 0;
    return output_head_packed_bytes(desc);
}

FIERY_API int fiery_output_head_pack_weights(const fiery_output_head_desc_t* desc, const float* w, void* packed, void* stream) {
    const int rc = check_output_head_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(w && packed, "output head: NULL weight pointer");
    FIERY_REQUIRE(aligned16(packed), "output head: packed weights must be 16-byte aligned");
    return launch_output_head_pack(desc, w, packed, static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_output_head_forward_workspace_bytes(const fiery_output_head_desc_t* desc) {
    if (check_output_head_desc(desc) != FIERY_OK) return 0;
    return output_head_forward_workspace_bytes(desc);
}

FIERY_API int fiery_output_head_forward(const fiery_output_head_desc_t* desc, const float* y, const void* packed, const float* bn_weight,
                                        const float* bn_bias, const float* running_mean, const float* running_var, float* out, float* mean,
                                        float* var, void* workspace, void* stream) {
    const int rc = check_output_head_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(y && packed && out && mean && var && workspace, "output head: NULL pointer");
    FIERY_REQUIRE(desc->training || (running_mean && running_var), "output head: eval mode needs running_mean and running_var");
    FIERY_REQUIRE(aligned16(y) && aligned16(packed) && aligned16(out) && aligned16(workspace), "output head: pointers must be 16-byte aligned");
    return launch_output_head_forward(desc, y, packed, bn_weight, bn_bias, running_mean, running_var, out, mean, var, workspace,
                                      static_cast<cudaStream_t>(stream));
}

FIERY_API size_t fiery_output_head_backward_workspace_bytes(const fiery_output_head_desc_t* desc) {
    if (check_output_head_desc(desc) != FIERY_OK) return 0;
    return output_head_backward_workspace_bytes(desc);
}

FIERY_API int fiery_output_head_backward(const fiery_output_head_desc_t* desc, const float* grad_out, const float* y, const float* mean,
                                         const float* var, const float* w1, const float* bn_weight, const float* bn_bias, float* grad_y,
                                         float* grad_bn_weight, float* grad_bn_bias, float* grad_w, float* grad_b, void* workspace,
                                         void* stream) {
    const int rc = check_output_head_desc(desc);
    if (rc != FIERY_OK) return rc;
    FIERY_REQUIRE(grad_out && y && mean && var && w1 && workspace, "output head: NULL pointer");
    FIERY_REQUIRE(aligned16(grad_out) && aligned16(y) && aligned16(workspace) && (!grad_y || aligned16(grad_y)),
                  "output head: pointers must be 16-byte aligned");
    return launch_output_head_backward(desc, grad_out, y, mean, var, w1, bn_weight, bn_bias, grad_y, grad_bn_weight, grad_bn_bias,
                                       grad_w, grad_b, workspace, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
