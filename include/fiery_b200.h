/*
 * fiery_b200 -- C ABI of the Hopper-native (sm_90a, H100) camera->BEV lift.
 *
 * The reference (wayveai/fiery) has no FFI: its "operator API" for this path is three Python call sites
 * (SURVEY.md section 8b).  Each entry point below replaces one of them and is what a binding for the path would
 * bind (ctypes stub: fiery_b200/_lib.py; reference-side patch: INTEGRATION.md):
 *
 *   fiery_lift_plan + fiery_lift_forward / fiery_lift_backward
 *       replace Fiery.get_geometry              fiery/models/fiery.py:193-208     (the plan: geometry once per batch)
 *             + Encoder.forward tail            fiery/models/encoder.py:98-102   (softmax x context outer product)
 *             + Fiery.projection_to_birds_eye_view   fiery/models/fiery.py:221-273
 *       i.e. the body of Fiery.calculate_birds_eye_view_features (fiery.py:275-286) after depth_layer.
 *   fiery_voxels_summing_forward / _backward
 *       replace VoxelsSumming.forward/backward  fiery/utils/geometry.py:283-314  (call site fiery.py:261)
 *   fiery_lift_point_indices
 *       exposes the integer voxel coordinates the reference computes at fiery.py:236-256 (for parity checks)
 *   fiery_compose_calibration
 *       exposes combined = R @ inverse(K), translation  (fiery.py:196,203)
 *   fiery_depth_layer_forward
 *       replaces Encoder.depth_layer (the head tensor's producer)  fiery/models/encoder.py:36,96   [SURVEY.md section 8f, next-3]
 *   fiery_bev_first_conv_forward
 *       replaces Decoder.first_conv (+ bn1 + relu in eval mode)  fiery/models/decoder.py:11,59-61   [SURVEY.md section 8f, next-2]
 *   fiery_bev_first_conv_backward_data / _weight
 *       the backward of Decoder.first_conv (what cuDNN runs for the reference's training step)
 *   fiery_warp_features_forward / _backward, fiery_warp_theta
 *       replace affine_grid + grid_sample inside warp_features  fiery/utils/geometry.py:219-220 (called from
 *       cumulative_warp_features geometry.py:225-253, call site fiery.py:143)   [SURVEY.md section 8f, next-1]
 *
 * Conventions: every pointer is a DEVICE pointer on the current CUDA device unless its name starts with
 * `host_`; tensors are dense row-major with the shapes given; `stream` is a cudaStream_t passed as void*
 * (NULL = default stream).  Calls enqueue work and return without synchronising unless stated.  Return value:
 * 0 on success, a negative FIERY_E_* code otherwise; fiery_last_error() gives the message for the calling thread.
 * There is no CPU implementation behind this ABI.
 */
#ifndef FIERY_B200_H_
#define FIERY_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FIERY_B200_ABI_VERSION 2

#if defined(__GNUC__)
#define FIERY_API __attribute__((visibility("default")))
#else
#define FIERY_API
#endif

enum {
    FIERY_OK = 0,
    FIERY_E_INVALID = -1,     /* bad argument / unsupported shape (message says which) */
    FIERY_E_CUDA = -2,        /* a CUDA runtime/driver call failed */
    FIERY_E_UNSUPPORTED = -3  /* valid request this build does not implement */
};

enum { FIERY_DTYPE_F32 = 0, FIERY_DTYPE_F16 = 1 };

/* How the camera calibration is supplied (fiery.py:193-205). */
enum {
    FIERY_CALIB_RAW = 0,       /* calib_a = intrinsics (B',n,3,3), calib_b = extrinsics (B',n,4,4); R @ K^-1 is
                                  composed on the device (LU with partial pivoting + solve, explicit fp32 order) */
    FIERY_CALIB_COMPOSED = 1   /* calib_a = combined (B',n,3,3) = R @ K^-1, calib_b = translation (B',n,3) */
};

/* Memory layout of the BEV tensor produced / consumed. Logical shape is always (B', C, X, Y) (fiery.py:225). */
enum {
    FIERY_BEV_NCHW = 0,        /* contiguous (B', C, X, Y) -- what the reference returns */
    FIERY_BEV_NHWC = 1         /* physical (B', X, Y, C): torch "channels_last" for the same logical tensor */
};

typedef struct fiery_lift_desc {
    int32_t n_frames;          /* B' = batch x time receptive field (fiery.py:278) */
    int32_t n_cameras;         /* n */
    int32_t depth_bins;        /* D, len(arange(*LIFT.D_BOUND)) (fiery.py:115) */
    int32_t channels;          /* C, MODEL.ENCODER.OUT_CHANNELS */
    int32_t feat_h, feat_w;    /* h, w = FINAL_DIM // DOWNSAMPLE (fiery.py:112) */
    int32_t bev_x, bev_y, bev_z;   /* bev_dimension (geometry.py:55); bev_z must be 1 (fiery.py:269) */
    float bev_offset[3];       /* bev_start_position - bev_resolution / 2, evaluated in fp32 (fiery.py:236) */
    float bev_resolution[3];   /* geometry.py:53 */
    float z_valid_lo, z_valid_hi; /* closed fp32 interval of (z - bev_offset[2]) for which
                                     0 <= trunc((z - bev_offset[2]) / bev_resolution[2]) < bev_z; computed
                                     exactly on the host (fiery_b200/geometry.py) */
    int32_t use_depth_distribution;  /* encoder.py:98: 1 = softmax x context, 0 = uniform depth (head has C channels) */
    int32_t head_dtype;        /* FIERY_DTYPE_* of the head tensor */
    int32_t calib_mode;        /* FIERY_CALIB_* */
    int32_t bev_layout;        /* FIERY_BEV_* */
} fiery_lift_desc_t;

FIERY_API int fiery_abi_version(void);
FIERY_API const char* fiery_last_error(void);

/*
 * Geometry plan.  Where every frustum point lands -- get_geometry (fiery.py:193-208) and the voxel index, mask and rank of
 * projection_to_birds_eye_view (fiery.py:236-256) -- depends on the calibration, the frustum and the BEV grid only, not on the head
 * tensor.  fiery_lift_plan evaluates it once for a batch of calibrations (the reference's exact fp32 operation order) and stores it
 * as pillar runs per (camera, feature column, depth), in the orders the forward and the backward kernel consume, plus one "receives
 * a point" byte per pillar.  fiery_lift_forward / fiery_lift_backward take `plan`:
 *   NULL      the geometry is evaluated inside the call (forward: in the tile kernel, under the latency of its loads; backward: by
 *             the plan kernel into the workspace);
 *   non-NULL  a buffer of fiery_lift_plan_bytes(desc) bytes filled by fiery_lift_plan with the SAME descriptor shape and the
 *             calibration of this batch -- the plan of a training step shared by its forward and backward, or one plan reused by
 *             every call while the camera rig is static.  It is only read.
 */
FIERY_API size_t fiery_lift_plan_bytes(const fiery_lift_desc_t* desc);
FIERY_API int fiery_lift_plan(const fiery_lift_desc_t* desc, const float* calib_a, const float* calib_b, const float* frustum_u,
                              const float* frustum_v, const float* frustum_d, void* plan_out, void* stream);

/* Bytes of zero-initialised device scratch fiery_lift_forward needs for FIERY_BEV_NCHW output (0 for NHWC): a
 * channel-last fp32 accumulator (chunk, X*Y, C) followed by one mark byte per pillar, where chunk <= B' is the number
 * of frames processed per pass (all of them unless the accumulator would exceed 1 GiB).
 * Invariant: the scratch must be all zero on entry; it is all zero again when the call's work completes. */
FIERY_API size_t fiery_lift_scratch_bytes(const fiery_lift_desc_t* desc);

/*
 * Forward lift.  head: (B'*n, D+C, h, w) [C channels if !use_depth_distribution], dtype head_dtype (FIERY_DTYPE_F32, or
 * FIERY_DTYPE_F16 for AMP heads: values are converted exactly to fp32 and all arithmetic is fp32, as autocast does to the
 * reference's softmax and outer product, encoder.py:99-100).
 * frustum_u (w), frustum_v (h), frustum_d (D): the separable factors of Fiery.frustum (fiery.py:109-128), fp32.
 * bev_out: (B',C,X,Y) fp32 in bev_layout.  For FIERY_BEV_NHWC the caller must pass bev_out zero-filled (the kernel
 * accumulates into it) and scratch may be NULL.
 */
FIERY_API int fiery_lift_forward(const fiery_lift_desc_t* desc, const void* head, const float* calib_a, const float* calib_b,
                       const float* frustum_u, const float* frustum_v, const float* frustum_d,
                       float* bev_out, void* scratch, const void* plan, void* stream);

/*
 * The lift followed by cumulative_warp_features (fiery/models/fiery.py:140-146, fiery/utils/geometry.py:225-253) in one chain: same
 * arguments as fiery_lift_forward (bev_layout must be FIERY_BEV_NCHW), plus the sampling maps of fiery_warp_theta for the B' frames:
 * theta (B', 2, 3) fp32 and copy_mask (B') bytes (1 = the present frame of its sequence: written as is, geometry.py:243).  Frame f of
 * bev_out is the bilinear sample (affine_grid + grid_sample, zero padding, align_corners=False) of frame f's lifted features --
 * gathered straight from the channel-last accumulator by the layout pass, so the unwarped BEV is never written or re-read
 * (3 launches per frame group instead of 2, and none of the standalone warp's).  [SURVEY.md section 8f, next-1]
 */
FIERY_API int fiery_lift_forward_warped(const fiery_lift_desc_t* desc, const void* head, const float* calib_a, const float* calib_b,
                                        const float* frustum_u, const float* frustum_v, const float* frustum_d, float* bev_out,
                                        void* scratch, const void* plan, const float* theta, const uint8_t* copy_mask, void* stream);

/*
 * Bit-reproducible forward lift (what torch.use_deterministic_algorithms(True) selects in the Python layer).  Same descriptors as
 * fiery_lift_forward: fp32 and fp16 heads, both calibration modes, NCHW and NHWC output, the uniform-depth head.  theta / copy_mask
 * non-NULL (NCHW only): the warped lift of fiery_lift_forward_warped.  plan: a plan of fiery_lift_plan for this batch, or NULL (the
 * call then builds a forward-only plan per pass into the workspace).  workspace: fiery_lift_deterministic_workspace_bytes(desc)
 * bytes; its contents on entry are irrelevant.  bev_out is fully overwritten in both layouts (NHWC needs no zero fill).
 * Summation order: every pillar of frame f is the fp32 sum of its pillar runs' partial sums (each run's sum is the register chain
 * the tile kernel computes along the image column), added one after the other in ascending (tile of frame f, run index in the
 * tile's plan record) order.  The order depends on frame f's geometry only, so a frame's BEV is bit-identical whatever other frames
 * share the call, however the call is cut into passes, with the caller's plan or the internal one, captured in a graph or not; NCHW
 * and NHWC hold the same bits, and a warped frame with its copy flag set equals the plain deterministic BEV of that frame.
 * Frames run in passes bounded like the scratch of fiery_lift_forward (fiery_lift_set_max_chunk_frames applies).  Nothing
 * synchronises with the host, so the call can be captured in a CUDA graph.
 */
FIERY_API size_t fiery_lift_deterministic_workspace_bytes(const fiery_lift_desc_t* desc);
FIERY_API int fiery_lift_forward_deterministic(const fiery_lift_desc_t* desc, const void* head, const float* calib_a,
                                               const float* calib_b, const float* frustum_u, const float* frustum_v,
                                               const float* frustum_d, float* bev_out, void* workspace, const void* plan,
                                               const float* theta, const uint8_t* copy_mask, void* stream);

/* Number of kernel launches one fiery_lift_forward call with this descriptor issues (NHWC: the tile kernel; NCHW: tile kernel
 * + layout pass per frame group; groups of frames run as concurrent chains on internal streams that are forked from and
 * joined back into `stream` with events, so the call behaves like work queued on `stream` and can be captured in a graph). */
FIERY_API int fiery_lift_forward_launches(const fiery_lift_desc_t* desc);

/* fiery_lift_forward with every kernel launch bracketed by an event pair on its own stream (profiling / bench.py's roofline): runs
 * the call, synchronises `stream`, and writes per launch the duration in milliseconds and the kind (1 tile kernel, 2 layout pass)
 * into host arrays of max_launches entries; *host_n_launches receives the count.  Launches of different chains overlap, so the
 * durations are what each kernel took while the others were running -- the launches the step really runs. */
FIERY_API int fiery_lift_forward_timed(const fiery_lift_desc_t* desc, const void* head, const float* calib_a, const float* calib_b,
                                       const float* frustum_u, const float* frustum_v, const float* frustum_d, float* bev_out,
                                       void* scratch, const void* plan, void* stream, int32_t max_launches, float* host_ms,
                                       int32_t* host_kind, int32_t* host_n_launches);

/* Test hook: caps the frames per pass (0 = default: as many as fit 1 GiB of scratch), so the multi-pass path can be exercised on
 * small batches.  Process-wide; changes fiery_lift_scratch_bytes accordingly. */
FIERY_API void fiery_lift_set_max_chunk_frames(int32_t n);

/* Bytes of device workspace fiery_lift_backward needs: the channel-last re-layout of an FIERY_BEV_NCHW grad_bev (0 for NHWC) plus
 * room for the plan records (used when plan is NULL).  Contents on entry/exit are irrelevant. */
FIERY_API size_t fiery_lift_workspace_bytes(const fiery_lift_desc_t* desc);

/*
 * Backward of the lift w.r.t. the head tensor (head_dtype must be FIERY_DTYPE_F32 in this build: widen an fp16 head first).
 * grad_bev: (B',C,X,Y) fp32 in bev_layout; grad_head: same shape and dtype as head, fully overwritten.  Calibration gets no gradient (geometry is integer, geometry.py:300).
 */
FIERY_API int fiery_lift_backward(const fiery_lift_desc_t* desc, const void* head, const float* calib_a, const float* calib_b,
                        const float* frustum_u, const float* frustum_v, const float* frustum_d,
                        const float* grad_bev, void* grad_head, float* workspace, const void* plan, void* stream);


/*
 * Integer voxel coordinates of all N = n*D*h*w points per frame, in the reference's point order
 * (camera, depth, row, column) (fiery.py:233).  idx_out: (B',N,3) int64 = trunc((p - offset)/res) (fiery.py:236-237);
 * valid_out: (B',N) uint8 (fiery.py:240-247); pillar_out: (B',N) int32 = rank (fiery.py:252-256) or -1 -- taken
 * from the same device function the lift kernels use.  Any output pointer may be NULL.
 * Where a scaled coordinate s = (p - offset)/res is NaN, +-inf or |s| >= 2^63, idx_out of that axis is unspecified (torch's .long()
 * itself gives different values on CPU and CUDA there); valid_out is 0 and pillar_out is -1 for such a point.
 */
FIERY_API int fiery_lift_point_indices(const fiery_lift_desc_t* desc, const float* calib_a, const float* calib_b,
                             const float* frustum_u, const float* frustum_v, const float* frustum_d,
                             int64_t* idx_out, uint8_t* valid_out, int32_t* pillar_out, void* stream);

/* combined (B'*n,3,3) and translation (B'*n,3) from intrinsics (B'*n,3,3) and extrinsics (B'*n,4,4). */
FIERY_API int fiery_compose_calibration(int32_t n_matrices, const float* intrinsics, const float* extrinsics,
                              float* combined_out, float* translation_out, void* stream);

/*
 * VoxelsSumming.forward (geometry.py:286-302).  feats (Nm,C) fp32 with row stride feat_stride elements,
 * coords (Nm,3) int64, ranks (Nm) int64 sorted ascending.
 * Step 1 -- fiery_voxels_summing_plan: writes segment_of_row (Nm) int32 (the index into the output each row sums
 * into) and *host_n_segments = U.  Synchronises `stream` (the reference's boolean indexing at geometry.py:295 has
 * the same host sync).  Step 2 -- fiery_voxels_summing_forward: sums_out (U,C) fp32, coords_out (U,3) int64 (coords
 * of the last row of each run, geometry.py:295).
 * Backward (geometry.py:305-314): grad_feats[i] = grad_sums[segment_of_row[i]].
 */
FIERY_API int fiery_voxels_summing_plan(int64_t n_rows, const int64_t* ranks, int32_t* segment_of_row,
                              int64_t* host_n_segments, void* stream);
FIERY_API int fiery_voxels_summing_forward(int64_t n_rows, int32_t channels, int64_t feat_stride, const float* feats,
                                 const int64_t* coords, const int32_t* segment_of_row, int64_t n_segments,
                                 float* sums_out, int64_t* coords_out, void* stream);
FIERY_API int fiery_voxels_summing_backward(int64_t n_rows, int32_t channels, const float* grad_sums,
                                  const int32_t* segment_of_row, float* grad_feats, void* stream);
/* Bit-reproducible fiery_voxels_summing_forward: the same arguments plus a workspace of
 * fiery_voxels_summing_deterministic_workspace_bytes(n_rows, channels) bytes (contents on entry irrelevant).  A run that crosses the
 * edge of a 64-row chunk is summed per chunk, and its pieces are added in chunk order (no atomics); sums_out needs no zero fill. */
FIERY_API size_t fiery_voxels_summing_deterministic_workspace_bytes(int64_t n_rows, int32_t channels);
FIERY_API int fiery_voxels_summing_forward_deterministic(int64_t n_rows, int32_t channels, int64_t feat_stride, const float* feats,
                                                         const int64_t* coords, const int32_t* segment_of_row, int64_t n_segments,
                                                         float* sums_out, int64_t* coords_out, void* workspace, void* stream);

/*
 * BEV feature warping -- the heavy part of warp_features / cumulative_warp_features (fiery/utils/geometry.py:181-253, call
 * site fiery/models/fiery.py:143-146): affine_grid + grid_sample (align_corners=False, zero padding; bilinear, or nearest
 * if `nearest` != 0) of n_maps feature maps (C, H, W) fp32 under the affine maps theta (n_maps, 2, 3).  Map m starts at
 * x + m * x_map_stride (elements); channel planes are dense (H*W).  copy_mask (n_maps bytes, may be NULL): maps with a
 * non-zero byte are copied unchanged -- the present frame of a sequence (geometry.py:243).
 * backward: grad_x[m] = adjoint of the sampling applied to grad_out[m].  grad_x is OVERWRITTEN (no zero-fill needed): the adjoint
 * runs as a gather over the output pixels that sampled each source pixel (deterministic, no atomics); for maps that are no near-rigid
 * transforms (|det| < 1/4, strong scaling, non-finite) the search covers the whole image: exact, but slow.
 */
FIERY_API int fiery_warp_features_forward(int32_t n_maps, int32_t channels, int32_t height, int32_t width, const float* x,
                                          int64_t x_map_stride, const float* theta, const uint8_t* copy_mask, float* out,
                                          int64_t out_map_stride, int32_t nearest, void* stream);
FIERY_API int fiery_warp_features_backward(int32_t n_maps, int32_t channels, int32_t height, int32_t width, const float* grad_out,
                                           int64_t grad_out_map_stride, const float* theta, const uint8_t* copy_mask,
                                           float* grad_x, int64_t grad_x_map_stride, int32_t nearest, void* stream);

/*
 * The pose algebra in front of the sampling: flow (6-DoF vectors tx,ty,tz,rx,ry,rz) -> theta (., 2, 3) for the calls above.
 * cumulative != 0 replaces the loop of cumulative_warp_features (geometry.py:241-251: pose_vec2mat :145-160, the running
 * product flow[t] @ ... @ flow[T-2], mat2pose_vec :82-107, then the theta of warp_features :197-219): flow is
 * (n_sequences, T, 6), theta (n_sequences*T, 2, 3) and copy_mask (n_sequences*T bytes, required) are written; the last frame
 * of every sequence is flagged "copy".  cumulative == 0 is the theta of a plain warp_features call: flow (n_sequences, 6),
 * T ignored, copy_mask may be NULL.  spatial_extent_x/y as in geometry.py:205-206.
 */
FIERY_API int fiery_warp_theta(int32_t n_sequences, int32_t T, int32_t cumulative, const float* flow, float spatial_extent_x,
                               float spatial_extent_y, float* theta, uint8_t* copy_mask, void* stream);

/*
 * First BEV convolution on the tensor cores (wgmma, TF32 operands, fp32 accumulation) -- Decoder.first_conv
 * (fiery/models/decoder.py:11,59): Conv2d(64, 64, kernel_size=7, stride=2, padding=3, bias=False), optionally followed by a per-channel
 * affine (bn1 folded for inference, decoder.py:60) and relu (decoder.py:61).  [SURVEY.md section 8f, next-2]
 * It consumes the lift's channel-last result directly: x_nhwc (B', H, W, 64) fp32 = FIERY_BEV_NHWC output of fiery_lift_forward;
 * y_nhwc (B', Ho, Wo, 64) fp32 with Ho = (H - 1) / 2 + 1, Wo likewise.  packed_weight: (49, 64, 64) = (tap r*7+s, out, in), made from
 * the module's (64, 64, 7, 7) weight by fiery_bev_conv_pack_weights.  scale / shift: 64 floats each, or both NULL.
 */
FIERY_API int fiery_bev_conv_pack_weights(const float* weight_oihw, float* packed_out, void* stream);
FIERY_API int fiery_bev_first_conv_forward(int32_t n_frames, int32_t height, int32_t width, const float* x_nhwc, const float* packed_weight,
                                           const float* scale, const float* shift, int32_t relu, float* y_nhwc, void* stream);

/*
 * Backward of fiery_bev_first_conv_forward without the optional affine / relu (wgmma, TF32 operands, fp32 accumulation); the
 * same shapes: x_nhwc / grad_x_nhwc (n_frames, height, width, 64) fp32, grad_y_nhwc (n_frames, Ho, Wo, 64) fp32 with
 * Ho = (height - 1) / 2 + 1, Wo likewise.  Pointers 16-byte aligned.
 *
 * fiery_bev_conv_pack_weights_transposed: the module's (64, 64, 7, 7) weight -> (49, 64, 64) = (tap r*7+s, in, out), rounded to
 * TF32 (nearest, ties away).
 * fiery_bev_first_conv_backward_data: grad_x = the input gradient (the transposed convolution of grad_y), fully overwritten (no
 * zero fill needed).  Each element is the fp32 accumulation of its taps' products in a fixed order (no atomics): bit-reproducible.
 * fiery_bev_first_conv_backward_weight: grad_weight_oihw (64, 64, 7, 7) fp32 = the weight gradient, fully overwritten (zeros when
 * n_frames == 0).  workspace: fiery_bev_first_conv_backward_weight_workspace_bytes(n_frames, height, width) bytes (0 when
 * n_frames == 0 or the shape is invalid; at most 18 x 49 x 64 x 64 x 4 bytes = 13.8 MiB); its contents on entry are irrelevant.
 * Summation order: the output pixels are cut into 16 x 8 tiles, numbered frame by frame in row-major tile order, and the tiles
 * into c = min(tiles, 18) chunks, chunk k holding tiles [k * tiles / c, (k + 1) * tiles / c).  A chunk's partial is the tensor
 * core's fp32 accumulation over its tiles in ascending order, 8 pixels per MMA; grad_weight is the fp32 sum of the c partials in
 * ascending chunk order.  The order depends on (n_frames, height, width) only, not on the device or the stream, so the result is
 * bit-reproducible and the call can be captured in a CUDA graph.  No host synchronisation.
 */
FIERY_API int fiery_bev_conv_pack_weights_transposed(const float* weight_oihw, float* packed_out, void* stream);
FIERY_API int fiery_bev_first_conv_backward_data(int32_t n_frames, int32_t height, int32_t width, const float* grad_y_nhwc,
                                                 const float* packed_weight_t, float* grad_x_nhwc, void* stream);
FIERY_API size_t fiery_bev_first_conv_backward_weight_workspace_bytes(int32_t n_frames, int32_t height, int32_t width);
FIERY_API int fiery_bev_first_conv_backward_weight(int32_t n_frames, int32_t height, int32_t width, const float* x_nhwc,
                                                   const float* grad_y_nhwc, float* grad_weight_oihw, void* workspace, void* stream);

/*
 * Encoder.depth_layer on the tensor cores -- the 1x1 convolution 128 -> D + C that produces the head tensor
 * (fiery/models/encoder.py:36,96): head_out (n_images, n_out, pixels) fp32 = weight @ feat + bias, computed by wgmma (fp16 / bf16
 * operands under AMP, TF32 for fp32 features; fp32 accumulation).  feat: (n_images, 128, pixels) with pixels = h*w, dtype 0 fp32 /
 * 1 fp16 / 2 bf16; weight_padded: (128, 128) row-major in the SAME dtype, rows >= n_out zero; bias: n_out floats or NULL.  Writing the
 * fp32 head directly removes the widening pass an AMP step otherwise needs in front of the lift.  [SURVEY.md section 8f, next-3]
 */
FIERY_API int fiery_depth_layer_forward(int32_t n_images, int32_t pixels, int32_t n_out, const void* feat, int32_t dtype,
                                        const void* weight_padded, const float* bias, float* head_out, void* stream);

/*
 * The temporal block's 1x1x1 input projections as one GEMM (TemporalBlock, fiery/layers/temporal.py:218-281): the paths'
 * conv_1x1x1_norm_activated convolutions and the projection's Conv3d read the same block input, so their n_segments (<= 4) weights,
 * stacked along the output channel, are one matrix W (N_out, K + E), N_out = sum of seg_channels, row-major fp32.  wgmma, TF32
 * operands, fp32 accumulation; W is rounded to TF32 (nearest, ties away) when packed, activations are truncated by the tensor core.
 *
 * x: the block input, element (b, t, k, p) at x[b * in_stride_b + t * in_stride_t + k * in_stride_c + p], p < pixels = X*Y, so the
 * permuted concat (b, K, s, X, Y) of a (b, s, K, X, Y) tensor and a contiguous (b, K, s, X, Y) tensor are both read as they lie.
 * extra: NULL (E = 0) or (batch, frames, E) fp32 channels that are constant over the map (the egopose): they enter the forward as the
 * bias sum_j W[o, K + j] * extra[b, t, j], computed in fp32.
 * out[q] / grad_out[q]: segment q's (batch, seg_channels[q], frames, X, Y) fp32, contiguous.
 * Limits (rejected with a message naming the field): 1 <= K <= 128; N_out <= 256, also with every segment rounded up to 8 channels;
 * 0 <= E <= 8; pixels % 4 == 0; the strides multiples of 4 elements; pointers 16-byte aligned.  batch * frames == 0 is a no-op (the
 * weight gradient is then zero).
 *
 * fiery_temporal_entry_packed_bytes / fiery_temporal_entry_pack_weights: the device pack of W that the three calls take.
 * fiery_temporal_entry_forward: out[q] fully overwritten.
 * fiery_temporal_entry_backward_data: grad_x (the K input channels, written with x's strides) = sum_q W_q^T grad_out[q].
 * fiery_temporal_entry_backward_weight: grad_w (N_out, K + E) = sum over frames and pixels of grad_out x^T (columns K + j: of the
 * extra channel j), fully overwritten.  workspace: fiery_temporal_entry_backward_weight_workspace_bytes(desc) bytes (0 for 0 frames),
 * contents irrelevant.  Summation order: the frames' pixels are cut into 64-pixel tiles, numbered frame by frame (b, then t), and the
 * tiles into c = min(tiles, 128) chunks, chunk i holding tiles [i * tiles / c, (i + 1) * tiles / c); a chunk's partial is the tensor
 * core's fp32 accumulation over its tiles in ascending order, and grad_w the fp32 sum of the partials in ascending chunk order.  The
 * order depends on (batch * frames, pixels) only: bit-reproducible, graph-capturable, no host synchronisation.
 */
typedef struct {
    int32_t batch;
    int32_t frames;
    int32_t pixels;
    int32_t in_channels;          /* K */
    int32_t extra_channels;       /* E */
    int32_t n_segments;
    int32_t seg_channels[4];
    int64_t in_stride_b, in_stride_t, in_stride_c;   /* elements */
} fiery_temporal_entry_desc_t;

FIERY_API size_t fiery_temporal_entry_packed_bytes(const fiery_temporal_entry_desc_t* desc);
FIERY_API int fiery_temporal_entry_pack_weights(const fiery_temporal_entry_desc_t* desc, const float* weight, void* packed, void* stream);
FIERY_API int fiery_temporal_entry_forward(const fiery_temporal_entry_desc_t* desc, const float* x, const float* extra, const void* packed,
                                           float* const* out, void* stream);
FIERY_API int fiery_temporal_entry_backward_data(const fiery_temporal_entry_desc_t* desc, const float* const* grad_out, const void* packed,
                                                 float* grad_x, void* stream);
FIERY_API size_t fiery_temporal_entry_backward_weight_workspace_bytes(const fiery_temporal_entry_desc_t* desc);
FIERY_API int fiery_temporal_entry_backward_weight(const fiery_temporal_entry_desc_t* desc, const float* x, const float* extra,
                                                   const float* const* grad_out, float* grad_w, void* workspace, void* stream);

/*
 * The temporal block's aggregation (TemporalBlock, fiery/layers/temporal.py:268-276) without the concat: a 1x1x1 convolution of
 * cat([path_0, .., path_{n-1}, pooled broadcast over the map], channel) is sum_q A_q path_q plus, per frame, the pooled columns' product
 * W_P v, a per-(frame, output channel) bias.  The sum is the entry's backward_data GEMM with the roles swapped:
 *   desc.in_channels = N, the aggregation's output channels; desc.seg_channels[q] = C_q, path q's channels; desc.extra_channels = 0;
 *   desc.in_stride_b / _t / _c: the strides of out (out[b * in_stride_b + t * in_stride_t + n * in_stride_c + p]);
 *   packed: fiery_temporal_entry_pack_weights of the stacked (sum C_q, N) matrix [A_0^T; ..; A_{n-1}^T].
 * paths[q]: (batch, C_q, frames, X, Y) fp32, contiguous; bias: NULL or (batch * frames, N) fp32, contiguous, row b * frames + t.
 *   out[b, n, t, p] = sum_q sum_c A_q[n, c] * paths[q][b, c, t, p] + bias[b * frames + t, n], fully overwritten.
 * wgmma, TF32 operands (the pack rounded to nearest, the paths truncated by the tensor core), fp32 accumulation; the bias is added in
 * fp32.  Limits: those of fiery_temporal_entry_desc_t (N <= 128, sum of round8(C_q) <= 256, at most 4 paths, pixels % 4 == 0, strides
 * multiples of 4 elements, pointers 16-byte aligned), and extra_channels == 0.  No workspace; batch * frames == 0 is a no-op.
 * Its backward is the entry's forward (path gradients: x = grad_out with K = N, the same pack) and backward_weight (x = grad_out,
 * grad_out[q] = paths[q]: the (sum C_q, N) transposed weight gradient), plus fiery_spatial_sums of grad_out for the bias.
 */
FIERY_API int fiery_temporal_aggregation_forward(const fiery_temporal_entry_desc_t* desc, const float* const* paths, const void* packed,
                                                 const float* bias, float* out, void* stream);

/*
 * Per-plane spatial sums: sums[(b * channels + c) * frames + t] = sum over p < pixels of x[b * stride_b + c * stride_c + t * stride_t + p]
 * for a fp32 tensor (batch, channels, frames, X, Y) whose pixel planes are contiguous (pixels = X*Y) and whose other strides are
 * arbitrary (the permuted (b, s, C, X, Y) concat, a contiguous NCDHW tensor, a channel slice).  sums: batch * channels * frames fp32,
 * fully overwritten.  Offsets in 64 bits.  Limits: batch, channels, frames >= 0 (a zero is a no-op); pixels >= 1; strides >= 0.  No
 * workspace, no alignment requirement.  Summation order: the plane is cut into 4-pixel chunks; thread i of 256 adds chunks i, i + 256,
 * ... in ascending order into one accumulator per chunk lane, its total is (lane 0 + lane 1) + (lane 2 + lane 3), the 32 threads of a
 * warp reduce by an xor butterfly (16, 8, 4, 2, 1) and the 8 warp sums are added in ascending order.  The order depends on pixels only:
 * a plane's sum is bit-identical whatever its strides or its neighbours; no atomics, graph-capturable.
 */
typedef struct {
    int32_t batch;
    int32_t channels;
    int32_t frames;
    int32_t pixels;               /* X*Y */
    int64_t stride_b, stride_c, stride_t;   /* elements */
} fiery_spatial_sums_desc_t;

FIERY_API int fiery_spatial_sums(const fiery_spatial_sums_desc_t* desc, const float* x, float* sums, void* stream);

/*
 * The temporal model's causal convolution (CausalConv3d, fiery/layers/temporal.py:65-85) without its BatchNorm and ReLU: a zero pad of
 * kt - 1 frames in front and one pixel around the map, then a bias-free Conv3d with kernel (kt, 3, 3), stride 1, dilation 1:
 *   y[b, o, t, p] = sum_{i, tau, dy, dx} W[o, i, tau, dy, dx] * x[b, i, t + tau - (kt - 1), p + (dy - 1, dx - 1)]
 * (terms outside the tensor are zero).  wgmma, TF32 operands, fp32 accumulation; W is rounded to TF32 (nearest, ties away) when
 * packed, and so are x in the forward and the weight gradient and grad_y in backward_data; grad_y in the weight gradient is
 * truncated by the tensor core.
 *
 * x / grad_x: (batch, in_channels, frames, grid_x, grid_y) fp32, contiguous; y / grad_y: (batch, out_channels, frames, grid_x, grid_y)
 * fp32, contiguous; weight / grad_w: (out_channels, in_channels, kt, 3, 3) fp32, contiguous.
 * Limits (rejected with FIERY_E_INVALID and a message naming the field): 1 <= in_channels, out_channels <= 64; kt 1 or 2; grid_x >= 1;
 * grid_y a positive multiple of 4 (16-byte TMA row pitch); pointers 16-byte aligned.  batch * frames == 0 is a no-op (the weight
 * gradient is then zero).
 *
 * fiery_causal_conv3d_packed_bytes / fiery_causal_conv3d_pack_weights: the device pack of W that forward and backward_data take.
 * fiery_causal_conv3d_forward: y fully overwritten.
 * fiery_causal_conv3d_backward_data: grad_x = the adjoint of the forward applied to grad_y, fully overwritten.
 * fiery_causal_conv3d_backward_weight: grad_w[o, i, tau, dy, dx] = sum over batch, frames and pixels of grad_y[b, o, t, p] *
 * x[b, i, t + tau - (kt - 1), p + (dy - 1, dx - 1)], fully overwritten.  workspace: fiery_causal_conv3d_backward_weight_workspace_bytes
 * (desc) bytes (0 for 0 frames), contents irrelevant.  Summation order: the pixels are cut into tiles of 32 consecutive grid_y
 * positions of one map row, numbered (b, t, x, run) with the run fastest, and the tiles into c = min(tiles, 128) chunks, chunk i
 * holding tiles [i * tiles / c, (i + 1) * tiles / c); a chunk's partial is the tensor core's fp32 accumulation over its tiles in
 * ascending order, and grad_w the fp32 sum of the partials in ascending chunk order.  The order depends on the shape only:
 * bit-reproducible, graph-capturable, no host synchronisation.
 */
typedef struct {
    int32_t batch;
    int32_t frames;
    int32_t grid_x;               /* X: map rows */
    int32_t grid_y;               /* Y: map columns, contiguous */
    int32_t in_channels;
    int32_t out_channels;
    int32_t kt;                   /* time taps: 2 for the (2, 3, 3) convolution, 1 for (1, 3, 3) */
} fiery_causal_conv3d_desc_t;

FIERY_API size_t fiery_causal_conv3d_packed_bytes(const fiery_causal_conv3d_desc_t* desc);
FIERY_API int fiery_causal_conv3d_pack_weights(const fiery_causal_conv3d_desc_t* desc, const float* weight, void* packed, void* stream);
FIERY_API int fiery_causal_conv3d_forward(const fiery_causal_conv3d_desc_t* desc, const float* x, const void* packed, float* y,
                                          void* stream);
FIERY_API int fiery_causal_conv3d_backward_data(const fiery_causal_conv3d_desc_t* desc, const float* grad_y, const void* packed,
                                                float* grad_x, void* stream);
FIERY_API size_t fiery_causal_conv3d_backward_weight_workspace_bytes(const fiery_causal_conv3d_desc_t* desc);
FIERY_API int fiery_causal_conv3d_backward_weight(const fiery_causal_conv3d_desc_t* desc, const float* x, const float* grad_y,
                                                  float* grad_w, void* workspace, void* stream);

/*
 * BatchNorm3d (the temporal model's norms, fiery/layers/temporal.py) over x (batch, channels, frames, X, Y) fp32 whose pixel planes
 * are contiguous (pixels = X*Y) and whose other strides are arbitrary, with an optional fused ReLU and an optional fused residual add.
 * Per channel c, over n = batch * frames * pixels values:
 *   training: mean and biased var of the batch;  eval: mean = running_mean[c], var = running_var[c];
 *   scale = weight[c] / sqrt(var + eps), shift = bias[c] - mean * scale, in fp64 from the fp32 mean and var, rounded once
 *   (weight NULL: 1; bias NULL: 0);
 *   y = fmaf(scale, x, shift), then max(y, 0) when relu (a NaN stays NaN), then + residual when residual is not NULL.
 * The backward, with g' = grad_y where the forward's fmaf(scale, x, shift) is not <= 0 (relu; a NaN passes, as torch's
 * threshold_backward), 0 where it is, or g' = grad_y (no relu), and
 * S1 = sum g', S2 = sum g' (x - mean):
 *   grad_bias = S1, grad_weight = S2 / sqrt(var + eps);
 *   training: grad_x = scale * (g' - S1 / n - (x - mean) * S2 / (n * (var + eps)));  eval: grad_x = scale * g'.
 * mean and var are what the forward wrote to mean_out / var_out, and the backward takes the forward's weight and bias, so its ReLU
 * mask is exactly where the forward's ReLU output was zero.  The residual's gradient is grad_y itself.
 *
 * y, residual, grad_y, grad_x: (batch, channels, frames, X, Y) fp32, contiguous.  weight, bias, running_mean, running_var, mean_out,
 * var_out, mean, var, grad_weight, grad_bias: (channels,) fp32.  Any pointer may have 4-byte alignment (16-byte aligned pixel runs
 * move as float4).  workspace: fiery_batch_norm_workspace_bytes(desc) bytes, 16-byte aligned, contents irrelevant (0 for a rejected
 * descriptor).  The backward computes what is asked for: grad_x, grad_weight and grad_bias may each be NULL.  Offsets in 64 bits.
 * Limits (FIERY_E_INVALID, the message names the field): channels >= 1; batch, frames >= 0 with batch * frames >= 1; pixels >= 1;
 * strides >= 0; training and relu 0 or 1; eps >= 0; in training n >= 2; in eval running_mean and running_var are given.
 *
 * Summation order (no atomics; the order depends on the shape only, so results are bit-reproducible whatever the strides or the
 * addresses, and graph-capturable): each pixel plane is cut into pieces of 4096 pixels, the last one shorter.  Within a piece, thread
 * i of 256 holds 4-pixel chunks i, i + 256, i + 512, i + 768, adds them in ascending order, each chunk as (p0 + p1) + (p2 + p3), the 32
 * threads of a warp reduce by an xor butterfly (16, 8, 4, 2, 1) and the 8 warp sums are added in ascending order, in fp32.  The
 * forward reduces a piece to its mean (the sum over its count) and M2 = sum (x - piece mean)^2, the backward to S1 and S2.  Per
 * channel, the pieces are merged in ascending (b, t, piece) order in fp64: Chan's formula for (count, mean, M2) in the forward, plain
 * sums in the backward.  Kernels: csrc/batch_norm.cu.
 */
typedef struct {
    int32_t batch;
    int32_t channels;
    int32_t frames;
    int32_t pixels;               /* X*Y */
    int64_t stride_b, stride_c, stride_t;   /* x's strides, elements */
    int32_t training;             /* 1: batch statistics; 0: running statistics */
    int32_t relu;                 /* 1: ReLU after the affine map */
    double eps;
} fiery_batch_norm_desc_t;

FIERY_API size_t fiery_batch_norm_workspace_bytes(const fiery_batch_norm_desc_t* desc);
FIERY_API int fiery_batch_norm_forward(const fiery_batch_norm_desc_t* desc, const float* x, const float* weight, const float* bias,
                                       const float* running_mean, const float* running_var, const float* residual, float* y,
                                       float* mean_out, float* var_out, void* workspace, void* stream);
FIERY_API int fiery_batch_norm_backward(const fiery_batch_norm_desc_t* desc, const float* x, const float* grad_y, const float* weight,
                                        const float* bias, const float* mean, const float* var, float* grad_x, float* grad_weight,
                                        float* grad_bias, void* workspace, void* stream);

/*
 * The batch norm in training with batch statistics over a group of `world` ranks (torch.nn.SyncBatchNorm), in two phases each way;
 * the caller gathers every rank's triplets between them (no collective runs in the library):
 *   forward:  fiery_batch_norm_local_stats -> stats (channels, 3) fp64 (n, mean, M2) of this rank's x, its pieces merged as
 *             fiery_batch_norm_forward merges them;  gather to gathered (world, channels, 3), rank r at [r];
 *             fiery_batch_norm_forward_gathered -> the group's mean and biased var (mean_out, var_out), y as fiery_batch_norm_forward
 *             computes it from them, and count_out[0] = the group's n (fp64, may be NULL; the running variance's unbiased factor).
 *   backward: fiery_batch_norm_local_grad_sums -> sums (channels, 3) fp64 (n, S1, S2) of this rank, and this rank's grad_weight =
 *             S2 / sqrt(var + eps), grad_bias = S1 (each may be NULL; the local sums, as torch's);  gather;
 *             fiery_batch_norm_backward_gathered -> grad_x from the group's S1, S2 and n.
 * The gathered finalize merges the ranks in ascending rank order in fp64, starting from rank 0's triplet: Chan's formula for
 * (n, mean, M2), plain sums for (n, S1, S2); a rank with n = 0 adds nothing.  Every rank computes the same numbers, and with world 1
 * they are bit for bit fiery_batch_norm_forward's / _backward's.  mean and var are the gathered forward's outputs.
 * Limits as above, except: training must be 1; batch * frames may be 0 (a rank with no values still writes its triplet) and a rank
 * may hold a single value; world >= 1.  stats, sums, gathered, count_out: 8-byte aligned.  workspace:
 * fiery_batch_norm_sync_workspace_bytes(desc), 16-byte aligned, contents irrelevant.  A group n of 0 or 1 gives NaN / 0 statistics
 * (the library cannot see the group's n on the host).
 */
FIERY_API size_t fiery_batch_norm_sync_workspace_bytes(const fiery_batch_norm_desc_t* desc);
FIERY_API int fiery_batch_norm_local_stats(const fiery_batch_norm_desc_t* desc, const float* x, double* stats, void* workspace, void* stream);
FIERY_API int fiery_batch_norm_forward_gathered(const fiery_batch_norm_desc_t* desc, int32_t world, const double* gathered, const float* x,
                                                const float* weight, const float* bias, const float* residual, float* y, float* mean_out,
                                                float* var_out, double* count_out, void* workspace, void* stream);
FIERY_API int fiery_batch_norm_local_grad_sums(const fiery_batch_norm_desc_t* desc, const float* x, const float* grad_y, const float* weight,
                                               const float* bias, const float* mean, const float* var, double* sums, float* grad_weight,
                                               float* grad_bias, void* workspace, void* stream);
FIERY_API int fiery_batch_norm_backward_gathered(const fiery_batch_norm_desc_t* desc, int32_t world, const double* gathered, const float* x,
                                                 const float* grad_y, const float* weight, const float* bias, const float* mean,
                                                 const float* var, float* grad_x, void* workspace, void* stream);

/*
 * The future prediction's SpatialGRU (fiery/layers/temporal.py:10-62) over T steps, without flow warping.  For t = 0 .. T-1, with
 * h = h0 at t = 0 and out[:, t-1] after:
 *   u = sigmoid(conv3x3([x_t, h], W_gates[:C_h]) + b_gates[:C_h] + bias_init)
 *   r = sigmoid(conv3x3([x_t, h], W_gates[C_h:]) + b_gates[C_h:] + bias_init)
 *   q = (1 - r) h,  s = conv3x3([x_t, q], W_state)  (no bias)
 *   a = max(fmaf(scale, s, shift), 0) with batch_norm's scale and shift (fiery_batch_norm_*: this step's batch statistics in
 *       training, the running ones in eval),  out[:, t] = (1 - u) h + u a
 * conv3x3 is a 3x3 convolution with zero padding 1, [.,.] a concatenation along channels (never built).  wgmma, TF32 operands
 * (weights and activations rounded to nearest when read), fp32 accumulation; the gates' sigmoid is 1 / (1 + expf(-v)).  NaN and
 * +-inf follow these formulas in IEEE arithmetic: a non-finite x or h pixel reaches every output channel of its 3x3 neighbourhood
 * (0 * NaN is NaN, zero weights included), the ReLU passes NaN, and in training a non-finite s makes its channel's statistics NaN.
 *
 * x: (batch, x_frames, x_channels, grid_x, grid_y) fp32 with contiguous pixel planes and the strides given in the desc (elements,
 * multiples of 4); x_frames 1 means one frame read for every step.  h0, grad_h0: (batch, h_channels, X, Y) contiguous.  out,
 * grad_out: (batch, frames, h_channels, X, Y) contiguous.  W_gates / grad_w_gates (2 h_channels, x_channels + h_channels, 3, 3),
 * b_gates / grad_b_gates (2 h_channels), W_state / grad_w_state (h_channels, x_channels + h_channels, 3, 3), bn_weight, bn_bias,
 * running_mean, running_var, grad_bn_weight, grad_bn_bias (h_channels): contiguous fp32.  grad_x: (batch, x_frames, x_channels, X, Y)
 * contiguous (with x_frames 1 the sum over the steps).  means / vars: (frames, h_channels), each step's mean and biased variance
 * (copies of the running ones in eval).  saved: fiery_spatial_gru_saved_bytes, u, r, q and s of every step as (frames, batch,
 * h_channels, X, Y) each; the backward reads what the forward wrote there.  Workspaces: the *_workspace_bytes, 256-byte aligned,
 * contents irrelevant.  The backward computes what is asked for: grad_x, grad_h0 and each parameter gradient may be NULL.
 * Limits (FIERY_E_INVALID, the message names the field): 1 <= x_channels, h_channels <= 64; batch, frames >= 1; x_frames 1 or
 * frames; grid_x >= 1; grid_y a positive multiple of 4; training 0 or 1; eps >= 0; in training batch * X * Y >= 2; pointers
 * 16-byte aligned.
 *
 * Summation orders (no atomics; bit-reproducible, graph-capturable): the batch statistics as fiery_batch_norm_forward on each step's
 * s; the weight gradients as fiery_causal_conv3d_backward_weight's over (batch, frames) with kt = 1; the gates' bias gradient, per
 * channel, 256 threads each adding elements i, i + 256, ... of the (frame, batch) planes in ascending order, then a halving tree;
 * grad_bn_weight / grad_bn_bias the steps' fiery_batch_norm_backward results added in ascending step order.  Kernels:
 * csrc/spatial_gru.cu, csrc/causal_conv.cu, csrc/batch_norm.cu.
 */
typedef struct {
    int32_t batch;
    int32_t frames;               /* T: steps */
    int32_t x_frames;             /* 1 or frames */
    int32_t grid_x;
    int32_t grid_y;
    int32_t x_channels;
    int32_t h_channels;
    int64_t x_stride_b, x_stride_t, x_stride_c;   /* elements */
    int32_t training;
    double eps;
    float bias_init;
} fiery_spatial_gru_desc_t;

FIERY_API size_t fiery_spatial_gru_packed_bytes(const fiery_spatial_gru_desc_t* desc);
FIERY_API int fiery_spatial_gru_pack_weights(const fiery_spatial_gru_desc_t* desc, const float* w_gates, const float* w_state, void* packed,
                                             void* stream);
FIERY_API size_t fiery_spatial_gru_saved_bytes(const fiery_spatial_gru_desc_t* desc);
FIERY_API size_t fiery_spatial_gru_forward_workspace_bytes(const fiery_spatial_gru_desc_t* desc);
FIERY_API int fiery_spatial_gru_forward(const fiery_spatial_gru_desc_t* desc, const float* x, const float* h0, const void* packed,
                                        const float* b_gates, const float* bn_weight, const float* bn_bias, const float* running_mean,
                                        const float* running_var, float* out, void* saved, float* means, float* vars, void* workspace,
                                        void* stream);
FIERY_API size_t fiery_spatial_gru_backward_workspace_bytes(const fiery_spatial_gru_desc_t* desc);
FIERY_API int fiery_spatial_gru_backward(const fiery_spatial_gru_desc_t* desc, const float* grad_out, const float* x, const float* h0,
                                         const float* out, const void* saved, const float* means, const float* vars, const void* packed,
                                         const float* bn_weight, const float* bn_bias, float* grad_x, float* grad_h0, float* grad_w_gates,
                                         float* grad_b_gates, float* grad_w_state, float* grad_bn_weight, float* grad_bn_bias,
                                         void* workspace, void* stream);

/*
 * The SpatialGRU in training with each step's batch statistics over a group of `world` ranks (its norm a SyncBatchNorm), one step
 * at a time: the caller gathers every rank's (channels, 3) fp64 triplets into (world, channels, 3) between a step's two calls, as
 * for fiery_batch_norm_local_stats / _forward_gathered and _local_grad_sums / _backward_gathered.
 *   forward, t = 0 .. T-1:  step_begin (step t's gates and state convolution; stats = this rank's (n, mean, M2) of s), then
 *                           step_end (the group's mean and var into means[t], vars[t], count_out[0] = the group's n (may be NULL),
 *                           and the blend into out[:, t]);
 *   backward, t = T-1 .. 0: step_begin (the blend's gradient; sums = this rank's (n, S1, S2) of the norm's backward), then
 *                           step_end (the norm's input gradient from the group's sums, and step t's input gradients into grad_x
 *                           and the carried state gradient);
 *   then backward_weights:  the weight gradients, the gates' bias gradient, and grad_bn_weight / grad_bn_bias, each the sum over
 *                           the steps, in ascending order, of this rank's S2 / sqrt(var + eps) and S1 (the local sums, as torch's).
 * Arguments are fiery_spatial_gru_forward's / _backward's, the same in every call of a sequence; the forward calls share one
 * fiery_spatial_gru_forward_workspace_bytes workspace and the backward calls one fiery_spatial_gru_backward_workspace_bytes workspace,
 * kept from the first call of the sequence to the last (with grad_h0 NULL, the carried gradient lives there).  With world 1 every
 * output is bit for bit fiery_spatial_gru_forward's / _backward's.  Limits as fiery_spatial_gru_*, and: training 1; 0 <= t < frames;
 * world >= 1; stats, sums, gathered, count_out 8-byte aligned.
 */
FIERY_API int fiery_spatial_gru_forward_step_begin(const fiery_spatial_gru_desc_t* desc, int32_t t, const float* x, const float* h0,
                                                   const void* packed, const float* b_gates, const float* out, void* saved, double* stats,
                                                   void* workspace, void* stream);
FIERY_API int fiery_spatial_gru_forward_step_end(const fiery_spatial_gru_desc_t* desc, int32_t t, int32_t world, const double* gathered,
                                                 const float* h0, const float* bn_weight, const float* bn_bias, float* out, const void* saved,
                                                 float* means, float* vars, double* count_out, void* workspace, void* stream);
FIERY_API int fiery_spatial_gru_backward_step_begin(const fiery_spatial_gru_desc_t* desc, int32_t t, const float* grad_out, const float* h0,
                                                    const float* out, const void* saved, const float* means, const float* vars,
                                                    const void* packed, const float* bn_weight, const float* bn_bias, float* grad_h0,
                                                    double* sums, void* workspace, void* stream);
FIERY_API int fiery_spatial_gru_backward_step_end(const fiery_spatial_gru_desc_t* desc, int32_t t, int32_t world, const double* gathered,
                                                  const float* h0, const float* out, const void* saved, const float* means, const float* vars,
                                                  const void* packed, const float* bn_weight, const float* bn_bias, float* grad_x,
                                                  float* grad_h0, void* workspace, void* stream);
FIERY_API int fiery_spatial_gru_backward_weights(const fiery_spatial_gru_desc_t* desc, const float* x, const float* h0, const float* out,
                                                 const void* saved, const void* packed, float* grad_w_gates, float* grad_b_gates,
                                                 float* grad_w_state, float* grad_bn_weight, float* grad_bn_bias, void* workspace,
                                                 void* stream);

/*
 * The spatial GRU's 3x3 convolution on its own: zero padding 1, stride 1, no bias, on `maps` independent (X, Y) maps, the input the
 * channel concatenation of two segments x0 (in_channels[0]) and x1 (in_channels[1], 0 for none), the output split into y0
 * (out_channels[0]) and y1 (out_channels[1], 0 for none), each segment its own contiguous (maps, C, X, Y) fp32 tensor:
 *   [y0, y1][m, o, p] = sum_{i, dy, dx} W[o, i, dy, dx] * [x0, x1][m, i, p + (dy - 1, dx - 1)]
 * with W (out0 + out1, in0 + in1, 3, 3).  The same kernels, packs and weight-gradient blocks fiery_spatial_gru_* runs, with plain
 * stores: TF32 operands rounded to nearest (grad_y truncated by the tensor core in the weight gradient), fp32 accumulation.
 * backward_data: [gx0, gx1] from [gy0, gy1], each overwritten.  backward_weight: grad_w from x0, x1 and grad_y, ONE contiguous
 * (maps, out0 + out1, X, Y) tensor, overwritten, in fiery_causal_conv3d_backward_weight's order (tiles over (maps, x, run), 64 output
 * channels per block).  workspace: fiery_conv3x3_backward_weight_workspace_bytes, contents irrelevant.
 * Limits (FIERY_E_INVALID): maps >= 1; 1 <= in_channels[0], out_channels[0] <= 64; 0 <= in_channels[1], out_channels[1] <= 64;
 * grid_x >= 1; grid_y a positive multiple of 4; pointers 16-byte aligned.
 */
typedef struct {
    int32_t maps;
    int32_t grid_x;
    int32_t grid_y;
    int32_t in_channels[2];
    int32_t out_channels[2];
} fiery_conv3x3_desc_t;

FIERY_API size_t fiery_conv3x3_packed_bytes(const fiery_conv3x3_desc_t* desc);
FIERY_API int fiery_conv3x3_pack_weights(const fiery_conv3x3_desc_t* desc, const float* weight, void* packed, void* stream);
FIERY_API int fiery_conv3x3_forward(const fiery_conv3x3_desc_t* desc, const float* x0, const float* x1, const void* packed, float* y0,
                                    float* y1, void* stream);
FIERY_API int fiery_conv3x3_backward_data(const fiery_conv3x3_desc_t* desc, const float* grad_y0, const float* grad_y1, const void* packed,
                                          float* grad_x0, float* grad_x1, void* stream);
FIERY_API size_t fiery_conv3x3_backward_weight_workspace_bytes(const fiery_conv3x3_desc_t* desc);
FIERY_API int fiery_conv3x3_backward_weight(const fiery_conv3x3_desc_t* desc, const float* x0, const float* x1, const float* grad_y,
                                            float* grad_w, void* workspace, void* stream);

/*
 * The future prediction's Bottleneck (fiery/layers/convolutions.py:64-168, the plain variant: out_channels = in_channels = C, a 3x3
 * convolution with padding 1 and stride 1, no projection, dropout 0) on `maps` independent (X, Y) maps, with M = C / 2 (integer
 * division, the reference's int(in_channels / 2)):
 *   y1 = W_down x                       (1x1, C -> M)
 *   y2 = conv3x3(relu(bn1(y1)))         (M -> M; the zero padding is relu(bn1(y1))'s)
 *   y3 = W_up relu(bn2(y2))             (1x1, M -> C)
 *   out = relu(bn3(y3)) + x
 * Each bn_i is fiery_batch_norm_forward's (training: this call's batch statistics; eval: the running ones), so relu(bn_i(y)) is
 * max(fmaf(scale, y, shift), 0) with its fp64-derived scale and shift.  relu(bn1(y1)) and relu(bn2(y2)) are never stored: each value
 * is computed as the next convolution reads it, exactly the fp32 value fiery_batch_norm_forward (relu 1) would write, and then
 * treated as that convolution treats its input (the 3x3 rounds it to TF32 nearest, the 1x1 lets the tensor core truncate it).  So y1
 * is fiery_temporal_entry_forward's (batch = maps, frames = 1), y2 fiery_causal_conv3d_forward's (kt = 1) on fiery_batch_norm_forward's
 * output of y1, y3 the entry's on bn2's output, out fiery_batch_norm_forward's (relu 1, residual x) of y3, bit for bit.
 *
 * The backward, from g = grad_out: dy3 = bn3's backward (relu) of (y3, g); grad_w_up from the entry weight gradient of relu(bn2(y2))
 * (computed as its tile is read) and dy3; da2 = W_up^T dy3; dy2 = bn2's backward of (y2, da2); grad_w_conv from the 3x3 weight gradient
 * of relu(bn1(y1)) (computed as its run is read) and dy2; da1 = the 3x3 input gradient of dy2; dy1 = bn1's backward of (y1, da1);
 * grad_w_down = the entry weight gradient of (x, dy1); grad_x = W_down^T dy1 + g, the add in the input gradient's epilogue (one fp32 add
 * of the same two values).  Each is bit for bit that composition of fiery_temporal_entry_*, fiery_causal_conv3d_* and
 * fiery_batch_norm_backward.  The backward computes what is asked for: grad_x, each weight gradient and each grad_norms entry may be
 * NULL (a NULL weight gradient launches nothing for it, and the stages below the last gradient asked for do not run).
 *
 * x, out, y3, grad_out, grad_x: (maps, C, X, Y) fp32, contiguous; y1, y2: (maps, M, X, Y).  W_down / grad_w_down (M, C), W_conv /
 * grad_w_conv (M, M, 3, 3), W_up / grad_w_up (C, M): fp32, contiguous (a 1x1 conv weight's trailing (1, 1) dropped).  norms: 12
 * pointers, norm i = 0, 1, 2 (M, M, C channels) at [4i .. 4i + 3]: weight, bias, running_mean, running_var; weight / bias may be NULL
 * (1 / 0); running_* are read in eval only.  grad_norms: 6 pointers, [2i] = grad weight and [2i + 1] = grad bias of norm i, each may
 * be NULL.  stats: 2 (2M + C) fp32, written by the forward and read by the backward: mean1, var1, mean2, var2 (M each), mean3, var3 (C
 * each), the biased variances (copies of the running statistics in eval).  Workspaces: the *_workspace_bytes, 16-byte aligned,
 * contents irrelevant (0 bytes for a rejected descriptor).
 * Limits (FIERY_E_INVALID, the message names the field): 2 <= channels <= 128 (M <= 64 for the 3x3 kernels, K <= 128 for the entry);
 * maps >= 1; grid_x >= 1; grid_y a positive multiple of 4 (so pixels X*Y % 4 == 0); training 0 or 1; eps >= 0; in training
 * maps * X * Y >= 2; pointers 16-byte aligned.
 *
 * Summation orders: the reused kernels' (no atomics, no host synchronisation; bit-reproducible and graph-capturable): the statistics
 * and norm gradients as fiery_batch_norm_*, the 1x1 weight gradients as fiery_temporal_entry_backward_weight's over (maps, 1 frame),
 * the 3x3's as fiery_causal_conv3d_backward_weight's with kt = 1.  Kernels: csrc/bottleneck.cu on csrc/temporal_entry.cu,
 * csrc/causal_conv.cu and csrc/batch_norm.cu.
 */
typedef struct {
    int32_t maps;                 /* N: independent maps (batch * frames) */
    int32_t grid_x;
    int32_t grid_y;
    int32_t channels;             /* C: in_channels = out_channels */
    int32_t training;             /* 1: batch statistics; 0: running statistics */
    double eps;
} fiery_bottleneck_desc_t;

FIERY_API size_t fiery_bottleneck_packed_bytes(const fiery_bottleneck_desc_t* desc);
FIERY_API int fiery_bottleneck_pack_weights(const fiery_bottleneck_desc_t* desc, const float* w_down, const float* w_conv, const float* w_up,
                                            void* packed, void* stream);
FIERY_API size_t fiery_bottleneck_forward_workspace_bytes(const fiery_bottleneck_desc_t* desc);
FIERY_API int fiery_bottleneck_forward(const fiery_bottleneck_desc_t* desc, const float* x, const void* packed, const float* const* norms,
                                       float* y1, float* y2, float* y3, float* out, float* stats, void* workspace, void* stream);
FIERY_API size_t fiery_bottleneck_backward_workspace_bytes(const fiery_bottleneck_desc_t* desc);
FIERY_API int fiery_bottleneck_backward(const fiery_bottleneck_desc_t* desc, const float* grad_out, const float* x, const float* y1,
                                        const float* y2, const float* y3, const float* stats, const void* packed, const float* const* norms,
                                        float* grad_x, float* grad_w_down, float* grad_w_conv, float* grad_w_up, float* const* grad_norms,
                                        void* workspace, void* stream);

/*
 * The Bottleneck in training with each norm's batch statistics over a group of `world` ranks (its three norms SyncBatchNorms), split
 * at the norms: the caller gathers every rank's (channels, 3) fp64 triplets `local` into `gathered` (world, channels, 3), rank r at
 * [r], between two stages, as for fiery_batch_norm_local_stats / _forward_gathered and _local_grad_sums / _backward_gathered.
 *   forward, stages 0 .. 3 in order:
 *     0: y1 = W_down x;                                                          local = this rank's (n, mean, M2) of y1 (M channels)
 *     1: bn1's gathered finalize (mean1, var1 into stats, counts[0] = the group's n); y2 = conv3x3(relu(bn1(y1)));  local of y2 (M)
 *     2: bn2's gathered finalize (mean2, var2, counts[1]); y3 = W_up relu(bn2(y2));                                local of y3 (C)
 *     3: bn3's gathered finalize (mean3, var3, counts[2]); out = relu(bn3(y3)) + x.
 *   backward, stages 0 .. s, s the deepest stage a gradient asked for needs:
 *     0: local = this rank's (n, S1, S2) of bn3's backward on (y3, grad_out); its own grad_norms[4], [5]
 *     1: dy3 = bn3's backward from the gathered sums; grad_w_up; da2 = W_up^T dy3; local of bn2's backward on (y2, da2), grad_norms[2], [3]
 *     2: dy2 = bn2's backward from the gathered sums; grad_w_conv; da1 = the 3x3 input gradient; local of bn1's, grad_norms[0], [1]
 *     3: dy1 = bn1's backward from the gathered sums; grad_w_down; grad_x = W_down^T dy1 + grad_out.
 *   s is 3 when grad_x or grad_w_down is asked for, else 2 for grad_w_conv or bn1's weight or bias, else 1 for grad_w_up or bn2's, else
 *   0: it depends on which gradients are asked for only, so every rank runs as many gathers (s; 3 in the forward).  A NULL gradient
 *   launches nothing for it, as in fiery_bottleneck_backward, and a stage past s launches nothing it does not need.
 * Each stage's computation is fiery_bottleneck_forward's / _backward's with the group's statistics and sums, and the gathered finalize
 * merges the ranks in ascending rank order (fiery_batch_norm_*_gathered), so every rank gets bit-identical statistics and counts.  The
 * norms' weight and bias gradients are each rank's own (the local sums, as torch's SyncBatchNorm).  With world 1 every output,
 * statistic and gradient is bit for bit fiery_bottleneck_forward's / _backward's: a group of one merges exactly as the single-rank
 * finalize does, and the backward's prologue coefficients come from the saved mean and var through the same eval finalize.
 * Arguments are fiery_bottleneck_forward's / _backward's, the same in every stage of a sequence; the forward's stages share one
 * fiery_bottleneck_forward_workspace_bytes workspace and the backward's one fiery_bottleneck_backward_workspace_bytes workspace, kept
 * from stage 0 to the last stage (the backward's intermediate gradients live there).  counts: 3 fp64, each norm's group n (the running
 * variance's unbiased factor).  Limits as fiery_bottleneck_*, and: training 1; 0 <= stage <= 3; world >= 1 and gathered non-NULL in
 * stages 1..3; local non-NULL in stages 0..2, counts in forward stages 1..3; gathered, local, counts 8-byte aligned.  A rank with no
 * maps is the caller's to handle (the fiery_batch_norm_* group entries take n = 0).  Summation orders: fiery_bottleneck_*'s and
 * fiery_batch_norm_*_gathered's.
 */
FIERY_API int fiery_bottleneck_sync_forward_stage(const fiery_bottleneck_desc_t* desc, int32_t stage, int32_t world, const double* gathered,
                                                  const float* x, const void* packed, const float* const* norms, float* y1, float* y2,
                                                  float* y3, float* out, float* stats, double* counts, double* local, void* workspace,
                                                  void* stream);
FIERY_API int fiery_bottleneck_sync_backward_stage(const fiery_bottleneck_desc_t* desc, int32_t stage, int32_t world, const double* gathered,
                                                   const float* grad_out, const float* x, const float* y1, const float* y2, const float* y3,
                                                   const float* stats, const void* packed, const float* const* norms, float* grad_x,
                                                   float* grad_w_down, float* grad_w_conv, float* grad_w_up, float* const* grad_norms,
                                                   double* local, void* workspace, void* stream);

/*
 * One of the decoder's output heads after its 3x3 convolution (fiery/models/decoder.py:24-50: BatchNorm2d(C), ReLU, Conv2d(C, n, 1)
 * with a bias) on `maps` independent (X, Y) maps y with C channels:
 *   a   = relu(bn(y)) = max(fmaf(scale, y, shift), 0)       bn as fiery_batch_norm_forward's (relu 1): training this call's batch
 *                                                           statistics, eval the running ones
 *   out[m, j, p] = sum_c W1[j, c] a[m, c, p] + b1[j]
 * a is never stored: each value is computed as the 1x1 reads it, exactly the fp32 value fiery_batch_norm_forward (relu 1) would write,
 * and the tensor core truncates it to TF32; W1 is rounded to TF32 (nearest) when packed, the products accumulate in fp32, and b1 is
 * added once, exactly, to the accumulator (it enters as the extra channel of a fiery_temporal_entry_forward with value 1).  So out is
 * fiery_temporal_entry_forward's (batch = maps, frames = 1, E = 1, extra = 1) on fiery_batch_norm_forward's output of y, bit for bit.
 *
 * The backward, from g = grad_out: da[m, c, p] = sum_{j < n} W1[j, c] g[m, j, p] with the fp32 W1 (w1), fmaf in ascending j, in fp32; then grad_y, grad_bn_weight, grad_bn_bias are bit for bit fiery_batch_norm_backward's (relu 1) on (y, da), with
 * scale and shift recomputed from the saved mean and var by the same fp64 formula; grad_w[j, c] = sum_{m, p} g[m, j, p] a[m, c, p] and
 * grad_b[j] = sum_{m, p} g[m, j, p], a in fp32.  da is never stored: both backward passes recompute it from g.  The backward computes
 * what is asked for: grad_y, grad_bn_weight, grad_bn_bias, grad_w and grad_b may each be NULL; the pass over y that sums runs only for
 * a gradient that needs a sum (all but grad_y in eval), the pass that writes grad_y only for grad_y.
 *
 * y, grad_y: (maps, C, X, Y) fp32, contiguous; out, grad_out: (maps, n, X, Y) fp32, contiguous.  w: (n, C + 1) fp32, W1 with b1 as its
 * last column (the pack's input); w1: (n, C) fp32, W1 alone (the backward's); grad_w (n, C), grad_b (n).  bn_weight / bn_bias may be NULL (1 / 0); running_mean / running_var are read in eval only.
 * mean, var: (C,) fp32, written by the forward (the biased variance; copies of the running statistics in eval) and read by the
 * backward.  Workspaces: the *_workspace_bytes, 16-byte aligned, contents irrelevant (0 bytes for a rejected descriptor).
 * Limits (FIERY_E_INVALID, the message names the field): 1 <= channels <= 128 (the entry's K); 1 <= n_out <= 8; maps >= 1;
 * grid_x, grid_y >= 1 with X*Y % 4 == 0 (16-byte TMA pixel-plane pitch) and X*Y < 2^31; training 0 or 1; eps >= 0; in training
 * maps * X * Y >= 2; y, out, packed, grad_out, grad_y, workspace 16-byte aligned.
 *
 * Summation orders (no atomics, no host synchronisation; bit-reproducible and graph-capturable): the statistics and the norm's
 * gradients as fiery_batch_norm_*; grad_w and grad_b over the same 4096-pixel pieces of each (m, c) plane -- a piece's partial summed
 * as fiery_batch_norm_backward sums S1 (grad_b from channel 0's pieces) -- and the partials added in ascending (m, piece) order in
 * fp64, rounded once.  Kernels: csrc/output_head.cu on csrc/temporal_entry.cu and csrc/batch_norm.cu.
 */
typedef struct {
    int32_t maps;                 /* N: independent maps (batch * frames) */
    int32_t grid_x;
    int32_t grid_y;
    int32_t channels;             /* C */
    int32_t n_out;                /* n: the 1x1's outputs */
    int32_t training;             /* 1: batch statistics; 0: running statistics */
    double eps;
} fiery_output_head_desc_t;

FIERY_API size_t fiery_output_head_packed_bytes(const fiery_output_head_desc_t* desc);
FIERY_API int fiery_output_head_pack_weights(const fiery_output_head_desc_t* desc, const float* w, void* packed, void* stream);
FIERY_API size_t fiery_output_head_forward_workspace_bytes(const fiery_output_head_desc_t* desc);
FIERY_API int fiery_output_head_forward(const fiery_output_head_desc_t* desc, const float* y, const void* packed, const float* bn_weight,
                                        const float* bn_bias, const float* running_mean, const float* running_var, float* out, float* mean,
                                        float* var, void* workspace, void* stream);
FIERY_API size_t fiery_output_head_backward_workspace_bytes(const fiery_output_head_desc_t* desc);
FIERY_API int fiery_output_head_backward(const fiery_output_head_desc_t* desc, const float* grad_out, const float* y, const float* mean,
                                         const float* var, const float* w1, const float* bn_weight, const float* bn_bias, float* grad_y,
                                         float* grad_bn_weight, float* grad_bn_bias, float* grad_w, float* grad_b, void* workspace,
                                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FIERY_B200_H_ */
